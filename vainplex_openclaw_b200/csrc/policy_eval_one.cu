// policy_eval_one.cu -- whole policy rules for ONE evaluation context (cg_policy_eval_one, openclaw_gov.h): the same
// matchPolicy / aggregateMatches as policy_eval_kernel (the shared walk in policy_eval.h), with the whole block on the one
// context and the packed result written in place, so that the single-context path needs one kernel behind its step.  In its
// own translation unit: policy_eval.cu's kernels and launches stay as they are.
#include "policy_eval.h"

namespace cg {

namespace {

constexpr uint32_t kOneWarps = 16;                 // warps per block: each takes 32-rule chunks of the window in turn
constexpr uint32_t kOneWindow = 1024;              // program rules whose truth bits sit in shared memory at once
static_assert(kPeOneTexts <= kPeTexts, "every text of the context is collected into shared memory");

// One block.  Warp 0 collects the context's slotted texts (every text of the step) as policy_eval_kernel's warps do.  Then per
// window of kOneWindow program rules: every warp evaluates 32-rule chunks of it (scope atom and program per lane) into a truth
// word per chunk and the (first rule of its policy, effect) of each rule, in shared memory; warp 0 then walks the window's
// chunks in program order with PolicyWalk (first match per policy, carried across chunk and window seams) and writes each
// first match's program rule, up to cap, at out[kPeOneRules + i].  out[0] = the verdict word, out[1] = the matched policies,
// out[kPeOneCounters..] = the step's counter block.  An incomplete step: verdict and count 0xffffffff, no match.
__global__ void __launch_bounds__(kOneWarps * 32, 1) policy_eval_one_kernel(PolicyTable pt, ScanWork w, uint32_t rw, PolicyBatch b, uint32_t* __restrict__ out,
                                                                          uint32_t cap) {
  __shared__ uint32_t s_slot[kPeTexts];
  __shared__ uint8_t s_role[kPeTexts];
  __shared__ uint32_t s_truth[kOneWindow / 32];
  __shared__ uint2 s_rule[kOneWindow];             // per rule of the window: z (first rule of its policy), y (n_ops | effect)
  __shared__ uint32_t s_nt;
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, below = (1u << lane) - 1u;
  for (uint32_t i = threadIdx.x; i < kCounterWords; i += blockDim.x) out[kPeOneCounters + i] = w.counters[i];
  if (w.counters[kCtrErrors] != 0) {
    if (threadIdx.x == 0) out[0] = out[1] = 0xffffffffu;
    return;
  }
  if (wid == 0) {
    const uint32_t nt = collect_texts(w, b, 0, b.n_texts, lane, s_slot, s_role);
    if (lane == 0) s_nt = nt;
  }
  __syncthreads();
  const CtxTexts ct{s_slot, s_role, s_nt, 0, b.n_texts};
  PolicyWalk pw;
  uint32_t pos = 0;
  for (uint32_t w0 = 0; w0 < pt.n_rules; w0 += kOneWindow) {
    for (uint32_t k = wid; k < kOneWindow / 32; k += kOneWarps) {
      const uint32_t j = w0 + 32 * k + lane;
      uint4 ri = make_uint4(0u, 0u, 0xffffffffu, 0xffffffffu);
      bool t = false;
      if (j < pt.n_rules) {
        ri = pt.rules[j];
        t = rule_holds(pt, w, rw, b, ct, b.atoms, ri);
      }
      s_rule[32 * k + lane] = make_uint2(ri.z, ri.y);
      const uint32_t tb = __ballot_sync(0xffffffffu, t);
      if (lane == 0) s_truth[k] = tb;
    }
    __syncthreads();
    if (wid == 0) {
      for (uint32_t k = 0; k < kOneWindow / 32 && w0 + 32 * k < pt.n_rules; k++) {
        const uint32_t base = w0 + 32 * k;
        const uint2 r = s_rule[32 * k + lane];
        const bool first = pw.first((s_truth[k] >> lane) & 1u, r.x, base, pt.n_rules, lane);
        const uint32_t f = __ballot_sync(0xffffffffu, first);
        pw.add(first, r.y, base, f);
        const uint32_t p = pos + __popc(f & below);
        if (first && p < cap) out[kPeOneRules + p] = base + lane;
        pos += __popc(f);
      }
    }
    __syncthreads();                                 // (the next window overwrites the truth words)
  }
  if (threadIdx.x == 0) { out[0] = pw.verdict(); out[1] = pw.matched; }
}

}  // namespace

int launch_policy_eval_one(const PolicyTable& pt, const ScanWork& w, uint32_t rw, const PolicyBatch& b, uint32_t* d_out, uint32_t cap, cudaStream_t stream) {
  policy_eval_one_kernel<<<1, kOneWarps * 32, 0, stream>>>(pt, w, rw, b, d_out, cap);
  return 1;
}

}  // namespace cg
