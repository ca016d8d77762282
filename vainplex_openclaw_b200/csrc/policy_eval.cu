// policy_eval.cu -- whole policy rules on the device (cg_policy_eval_batch[_device], openclaw_gov.h): matchPolicy and
// aggregateMatches of src/policy-evaluator.ts:44-146 over a compiled policy program, for a batch of evaluation contexts
// whose texts a policy-mode step has just scanned.  Kept in its own translation unit: the scan kernels' code does not
// change with it.
#include <algorithm>

#include "kernels.h"

namespace cg {

namespace {

constexpr uint32_t kPeWarps = 8;         // warps (contexts in flight) per block
constexpr uint32_t kPeTexts = 64;        // slotted texts of a context kept in shared memory; past that HIT leaves walk the range
constexpr uint32_t kNoRule = 0xfffffu;

// the texts of one context that have a hit row: (slot, role), collected once per context by its warp
struct CtxTexts {
  const uint32_t* slot; const uint8_t* role; uint32_t n;    // n > kPeTexts: read the range itself
  uint32_t t0, t1;
};

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

// One warp per context, lanes over the program's rules, 32 at a time in program order (policy order, then rule order).
// A lane's rule holds when its policy's scope atom (if any) and its program hold; it is its policy's match when no earlier
// rule of the same policy holds -- within the chunk a ballot says so, across chunks the policy that straddles the boundary
// carries whether it already matched.  Then per chunk: matched policies (popc), any deny / 2fa / audit, and the first deny
// / 2fa whose effect has a reason.
//   kMode 0: verdict words.  kMode 1: verdict words and w.out_len[c] = matches of context c (w.out_len[n_ctx] = 0).
//   kMode 2: the matches of every context with some, at w.out_off[c], below cap; *count and the status.
// An incomplete step: every verdict 0xffffffff, count 0xffffffff, no match.  A context range that is decreasing or runs past
// n_texts (only a caller's HBM can hold one): verdict 0xfffffffe, no match.
template <int kMode>
__global__ void __launch_bounds__(kPeWarps * 32, 4) policy_eval_kernel(PolicyTable pt, ScanWork w, uint32_t rw, PolicyBatch b, uint32_t* __restrict__ verdicts,
                                                                   uint32_t* __restrict__ out, uint32_t cap, uint32_t* __restrict__ count) {
  __shared__ uint32_t s_slot[kPeWarps][kPeTexts];
  __shared__ uint8_t s_role[kPeWarps][kPeTexts];
  const bool incomplete = w.counters[kCtrErrors] != 0;
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
  if (kMode == 2) {
    if (gtid == 0) {
      const uint64_t total = w.out_off[b.n_ctx];
      if (incomplete) *count = 0xffffffffu;
      else {
        *count = total >= 0xffffffffull ? 0xffffffffu : (uint32_t)total;
        w.counters[kCtrResolveStatus] = total >= 0xffffffffull ? kResolveTooLarge : total > cap ? kResolveCapacity : kResolveOk;
      }
    }
    if (incomplete) return;
  } else {
    if (kMode == 1 && gtid == 0) w.out_len[b.n_ctx] = 0;
    if (incomplete) {
      for (uint32_t i = gtid; i < b.n_ctx; i += gridDim.x * blockDim.x) { verdicts[i] = 0xffffffffu; if (kMode == 1) w.out_len[i] = 0; }
      return;
    }
  }
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, below = (1u << lane) - 1u;
  for (uint32_t c = blockIdx.x * kPeWarps + wid; c < b.n_ctx; c += gridDim.x * kPeWarps) {
    if (kMode == 2 && (w.out_len[c] == 0 || w.out_off[c] >= cap)) continue;
    const uint32_t t0 = b.ctx_off[c], t1 = b.ctx_off[c + 1];
    if (t0 > t1 || t1 > b.n_texts) {
      if (kMode != 2 && lane == 0) { verdicts[c] = 0xfffffffeu; if (kMode == 1) w.out_len[c] = 0; }
      continue;
    }
    // the context's texts with a hit row, as (slot, role)
    uint32_t nt = 0;
    for (uint32_t i0 = t0; i0 < t1; i0 += 32) {
      const uint32_t i = i0 + lane;
      const uint32_t s = i < t1 ? w.slot_of_msg[i] : 0xffffffffu;
      const bool has = s < w.slot_cap;
      const uint32_t m = __ballot_sync(0xffffffffu, has);
      const uint32_t at = nt + __popc(m & below);
      if (has && at < kPeTexts) { s_slot[wid][at] = s; s_role[wid][at] = b.roles[i]; }
      nt += __popc(m);
    }
    __syncwarp();
    const CtxTexts ct{s_slot[wid], s_role[wid], nt, t0, t1};
    const uint32_t* arow = b.atoms + (size_t)c * pt.aw;
    uint32_t carry_first = 0xffffffffu, matched = 0, deny_r = kNoRule, twofa_r = kNoRule;
    bool carry_hit = false, any_deny = false, any_2fa = false, any_audit = false;
    uint64_t pos = kMode == 2 ? w.out_off[c] : 0ull;
    for (uint32_t base = 0; base < pt.n_rules; base += 32) {
      const uint32_t j = base + lane;
      uint4 ri = make_uint4(0u, 0u, 0xffffffffu, 0xffffffffu);
      bool t = false;
      if (j < pt.n_rules) {
        ri = pt.rules[j];
        t = ri.w == 0xffffffffu || ((arow[ri.w >> 5] >> (ri.w & 31)) & 1u);
        if (t) t = run_rule(pt, w, rw, b, ct, arow, ri.x, ri.y & 0xffffffu);
      }
      const uint32_t tb = __ballot_sync(0xffffffffu, t);
      const uint32_t from = ri.z > base && ri.z != 0xffffffffu ? ri.z - base : 0u;    // the first lane of this lane's policy
      const bool first = t && !(tb & below & ~((1u << from) - 1u)) && !(carry_hit && ri.z == carry_first);
      // the policy of the chunk's last rule: did it match in this chunk or before?
      const uint32_t last = min(31u, pt.n_rules - 1u - base);
      const uint32_t z_last = __shfl_sync(0xffffffffu, ri.z, last);
      const uint32_t from_last = z_last > base ? z_last - base : 0u;
      const bool hit_last = (tb & ~((1u << from_last) - 1u)) != 0u || (carry_hit && z_last == carry_first);
      carry_first = z_last; carry_hit = hit_last;
      const uint32_t f = __ballot_sync(0xffffffffu, first);
      if (kMode != 2) {
        const uint32_t act = (ri.y >> 24) & 3u, reason = (ri.y >> 26) & 1u;
        const uint32_t fd = __ballot_sync(0xffffffffu, first && act == 3u), fdr = __ballot_sync(0xffffffffu, first && act == 3u && reason);
        const uint32_t f2 = __ballot_sync(0xffffffffu, first && act == 2u), f2r = __ballot_sync(0xffffffffu, first && act == 2u && reason);
        matched += __popc(f);
        any_deny |= fd != 0u; any_2fa |= f2 != 0u; any_audit |= __ballot_sync(0xffffffffu, first && act == 1u) != 0u;
        if (deny_r == kNoRule && fdr) deny_r = base + __ffs(fdr) - 1;
        if (twofa_r == kNoRule && f2r) twofa_r = base + __ffs(f2r) - 1;
      } else {
        const uint64_t p = pos + __popc(f & below);
        if (first && p < cap) { out[2 * p] = c; out[2 * p + 1] = j; }
        pos += __popc(f);
        if (pos >= cap) break;
      }
    }
    if (kMode != 2 && lane == 0) {
      const uint32_t outcome = any_deny ? 4u : any_2fa ? 3u : any_audit ? 2u : matched ? 1u : 0u;
      const uint32_t decide = any_deny ? deny_r : any_2fa ? twofa_r : kNoRule;
      verdicts[c] = outcome | (min(matched, 511u) << 3) | (decide << 12);
      if (kMode == 1) w.out_len[c] = matched;
    }
    __syncwarp();                                                // (the next context overwrites this warp's texts)
  }
}

uint32_t pe_grid(uint32_t n_ctx, int sm_count) {
  return std::max<uint32_t>(1u, std::min<uint32_t>((uint32_t)(((uint64_t)n_ctx + kPeWarps - 1) / kPeWarps), (uint32_t)sm_count * 8u));
}

}  // namespace

int launch_policy_eval(const PolicyTable& pt, const ScanWork& w, uint32_t rw, const PolicyBatch& b, uint32_t* d_verdicts, bool counts, int sm_count,
                       cudaStream_t stream) {
  const uint32_t grid = pe_grid(b.n_ctx, sm_count);
  if (!counts) { policy_eval_kernel<0><<<grid, kPeWarps * 32, 0, stream>>>(pt, w, rw, b, d_verdicts, nullptr, 0, nullptr); return 1; }
  policy_eval_kernel<1><<<grid, kPeWarps * 32, 0, stream>>>(pt, w, rw, b, d_verdicts, nullptr, 0, nullptr);
  return 1 + launch_exclusive_scan(w.out_len, w.out_off, b.n_ctx + 1, w.scan_part, sm_count, stream);
}

int launch_policy_emit(const PolicyTable& pt, const ScanWork& w, uint32_t rw, const PolicyBatch& b, uint32_t* d_out, uint32_t cap, uint32_t* d_count,
                       int sm_count, cudaStream_t stream) {
  policy_eval_kernel<2><<<pe_grid(b.n_ctx, sm_count), kPeWarps * 32, 0, stream>>>(pt, w, rw, b, nullptr, d_out, cap, d_count);
  return 1;
}

}  // namespace cg
