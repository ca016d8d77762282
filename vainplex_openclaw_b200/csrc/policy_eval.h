// policy_eval.h -- the device side of a policy program that both policy kernels share (policy_eval.cu: a batch of contexts,
// one warp each; policy_eval_one.cu: one context, one block): the context's texts, the leaves and a rule's program, and the
// first-match / aggregation rule of matchPolicy and aggregateMatches (src/policy-evaluator.ts:44-146).  Included by those two
// translation units only.
#pragma once
#include "kernels.h"

namespace cg {
namespace {

constexpr uint32_t kPeTexts = 64;        // slotted texts of a context kept in shared memory; past that HIT leaves walk the range
constexpr uint32_t kNoRule = 0xfffffu;

// the texts of one context that have a hit row: (slot, role), collected once per context by one warp
struct CtxTexts {
  const uint32_t* slot; const uint8_t* role; uint32_t n;    // n > kPeTexts: read the range itself
  uint32_t t0, t1;
};

// the texts [t0, t1) that have a hit row, as (slot, role) into s_slot / s_role (the first kPeTexts of them) with a ballot per
// 32 texts; one whole warp calls it.  -> their number
__device__ __forceinline__ uint32_t collect_texts(const ScanWork& w, const PolicyBatch& b, uint32_t t0, uint32_t t1, uint32_t lane, uint32_t* s_slot,
                                                  uint8_t* s_role) {
  const uint32_t below = (1u << lane) - 1u;
  uint32_t nt = 0;
  for (uint32_t i0 = t0; i0 < t1; i0 += 32) {
    const uint32_t i = i0 + lane;
    const uint32_t s = i < t1 ? w.slot_of_msg[i] : 0xffffffffu;
    const bool has = s < w.slot_cap;
    const uint32_t m = __ballot_sync(0xffffffffu, has);
    const uint32_t at = nt + __popc(m & below);
    if (has && at < kPeTexts) { s_slot[at] = s; s_role[at] = b.roles[i]; }
    nt += __popc(m);
  }
  return nt;
}

__device__ __forceinline__ bool row_bit(const ScanWork& w, uint32_t rw, uint32_t slot, uint32_t r) {
  return (w.hit[(size_t)slot * rw + (r >> 5)] >> (r & 31)) & 1u;
}

// HIT(r, q): rule r hit a text of the context whose role is q
__device__ __forceinline__ bool hit_leaf(const ScanWork& w, uint32_t rw, const PolicyBatch& b, const CtxTexts& ct, uint32_t r, uint32_t q) {
  if (ct.n <= kPeTexts) {
    for (uint32_t k = 0; k < ct.n; k++) if (ct.role[k] == q && row_bit(w, rw, ct.slot[k], r)) return true;
    return false;
  }
  for (uint32_t i = ct.t0; i < ct.t1; i++) {
    const uint32_t s = w.slot_of_msg[i];
    if (s < w.slot_cap && b.roles[i] == q && row_bit(w, rw, s, r)) return true;
  }
  return false;
}

// one rule's postfix program on a bit stack (depth <= 32, checked when the program was set)
__device__ __forceinline__ bool run_rule(const PolicyTable& pt, const ScanWork& w, uint32_t rw, const PolicyBatch& b, const CtxTexts& ct, const uint32_t* arow,
                         uint32_t at, uint32_t n_ops) {
  uint32_t st = 0;
  for (uint32_t k = 0; k < n_ops; k++) {
    const uint32_t o = pt.ops[at + k];
    switch (o & 7u) {
      case kPolOpConst: st = st << 1 | (o >> 3); break;
      case kPolOpAtom: { const uint32_t a = o >> 3; st = st << 1 | ((arow[a >> 5] >> (a & 31)) & 1u); break; }
      case kPolOpHit: st = st << 1 | (hit_leaf(w, rw, b, ct, (o >> 3) & 0x1fffffu, o >> 24) ? 1u : 0u); break;
      case kPolOpAnd: { const uint32_t t = st & 1u; st >>= 1; st &= ~1u | t; break; }
      case kPolOpOr: { const uint32_t t = st & 1u; st >>= 1; st |= t; break; }
      default: st ^= 1u; break;                                   // kPolOpNot
    }
  }
  return st & 1u;
}

// rule j of the program holds for the context: its policy's scope atom (if any) and its program hold
__device__ __forceinline__ bool rule_holds(const PolicyTable& pt, const ScanWork& w, uint32_t rw, const PolicyBatch& b, const CtxTexts& ct, const uint32_t* arow,
                                           const uint4& ri) {
  const bool t = ri.w == 0xffffffffu || ((arow[ri.w >> 5] >> (ri.w & 31)) & 1u);
  return t && run_rule(pt, w, rw, b, ct, arow, ri.x, ri.y & 0xffffffu);
}

// The walk of one context's program, 32 rules (a chunk) at a time in program order (policy order, then rule order), by one
// whole warp with lane l on rule base + l.  A lane's rule is its policy's match when it holds and no earlier rule of the same
// policy holds: within the chunk a ballot says so, across chunks the policy of the previous chunk's last rule carries whether
// it already matched.  The verdict aggregates the first matches: matched policies, any deny / 2fa / audit, and the first
// deny / 2fa whose effect has a reason.
struct PolicyWalk {
  uint32_t carry_first = 0xffffffffu, matched = 0, deny_r = kNoRule, twofa_r = kNoRule;
  bool carry_hit = false, any_deny = false, any_2fa = false, any_audit = false;

  // t: the lane's rule holds; z: the first program rule of its policy (0xffffffff past the program).  -> is it the match?
  __device__ __forceinline__ bool first(bool t, uint32_t z, uint32_t base, uint32_t n_rules, uint32_t lane) {
    const uint32_t below = (1u << lane) - 1u;
    const uint32_t tb = __ballot_sync(0xffffffffu, t);
    const uint32_t from = z > base && z != 0xffffffffu ? z - base : 0u;    // the first lane of this lane's policy
    const bool f = t && !(tb & below & ~((1u << from) - 1u)) && !(carry_hit && z == carry_first);
    // the policy of the chunk's last rule: did it match in this chunk or before?
    const uint32_t last = min(31u, n_rules - 1u - base);
    const uint32_t z_last = __shfl_sync(0xffffffffu, z, last);
    const uint32_t from_last = z_last > base ? z_last - base : 0u;
    const bool hit_last = (tb & ~((1u << from_last) - 1u)) != 0u || (carry_hit && z_last == carry_first);
    carry_first = z_last; carry_hit = hit_last;
    return f;
  }
  // first: the lane's rule is its policy's match (f: the chunk's ballot of them); y: its n_ops | action << 24 | has_reason << 26
  __device__ __forceinline__ void add(bool first, uint32_t y, uint32_t base, uint32_t f) {
    const uint32_t act = (y >> 24) & 3u, reason = (y >> 26) & 1u;
    const uint32_t fd = __ballot_sync(0xffffffffu, first && act == 3u), fdr = __ballot_sync(0xffffffffu, first && act == 3u && reason);
    const uint32_t f2 = __ballot_sync(0xffffffffu, first && act == 2u), f2r = __ballot_sync(0xffffffffu, first && act == 2u && reason);
    matched += __popc(f);
    any_deny |= fd != 0u; any_2fa |= f2 != 0u; any_audit |= __ballot_sync(0xffffffffu, first && act == 1u) != 0u;
    if (deny_r == kNoRule && fdr) deny_r = base + __ffs(fdr) - 1;
    if (twofa_r == kNoRule && f2r) twofa_r = base + __ffs(f2r) - 1;
  }
  // outcome | matched policies (saturating at 511) << 3 | deciding rule << 12 (openclaw_gov.h)
  __device__ __forceinline__ uint32_t verdict() const {
    const uint32_t outcome = any_deny ? 4u : any_2fa ? 3u : any_audit ? 2u : matched ? 1u : 0u;
    const uint32_t decide = any_deny ? deny_r : any_2fa ? twofa_r : kNoRule;
    return outcome | (min(matched, 511u) << 3) | (decide << 12);
  }
};

}  // namespace
}  // namespace cg
