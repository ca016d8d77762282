// policy_eval.cu -- whole policy rules on the device (cg_policy_eval_batch[_device], openclaw_gov.h): matchPolicy and
// aggregateMatches of src/policy-evaluator.ts:44-146 over a compiled policy program, for a batch of evaluation contexts
// whose texts a policy-mode step has just scanned.  Kept in its own translation unit: the scan kernels' code does not
// change with it.
#include <algorithm>

#include "policy_eval.h"

namespace cg {

namespace {

constexpr uint32_t kPeWarps = 8;         // warps (contexts in flight) per block

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
    const uint32_t nt = collect_texts(w, b, t0, t1, lane, s_slot[wid], s_role[wid]);
    __syncwarp();
    const CtxTexts ct{s_slot[wid], s_role[wid], nt, t0, t1};
    const uint32_t* arow = b.atoms + (size_t)c * pt.aw;
    PolicyWalk pw;
    uint64_t pos = kMode == 2 ? w.out_off[c] : 0ull;
    for (uint32_t base = 0; base < pt.n_rules; base += 32) {
      const uint32_t j = base + lane;
      uint4 ri = make_uint4(0u, 0u, 0xffffffffu, 0xffffffffu);
      bool t = false;
      if (j < pt.n_rules) {
        ri = pt.rules[j];
        t = rule_holds(pt, w, rw, b, ct, arow, ri);
      }
      const bool first = pw.first(t, ri.z, base, pt.n_rules, lane);
      const uint32_t f = __ballot_sync(0xffffffffu, first);
      if (kMode != 2) {
        pw.add(first, ri.y, base, f);
      } else {
        const uint64_t p = pos + __popc(f & below);
        if (first && p < cap) { out[2 * p] = c; out[2 * p + 1] = j; }
        pos += __popc(f);
        if (pos >= cap) break;
      }
    }
    if (kMode != 2 && lane == 0) {
      verdicts[c] = pw.verdict();
      if (kMode == 1) w.out_len[c] = pw.matched;
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
