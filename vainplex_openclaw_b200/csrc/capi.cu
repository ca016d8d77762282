// capi.cu -- the C ABI declared in include/openclaw_gov.h (host orchestration only; every byte of
// matching and hashing happens in the kernels of scan_kernels.cu / sha256_kernels.cu).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <dlfcn.h>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/openclaw_gov.h"
#include "dev_buffer.h"
#include "kernels.h"
#include "rulec.h"
#include "ruleset_image.h"

using namespace cg;

namespace {

thread_local std::string g_err;
std::mutex g_mu;

// Calls that share device scratch run in the order they were issued, whatever streams they are issued on.  A scratch keeps
// the stream of the call that used it last and an event recorded there behind that use.
struct IssueOrder { cudaEvent_t ev = nullptr; cudaStream_t last = nullptr; };

struct Ctx {
  bool ready = false;
  int device = 0, sm_count = 132;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaEvent_t pev[6] = {};          // profiling: before scan_kernel, after scan_kernel, confirm_kernel, resolve, verify, finalize
  bool profiling = false;
  cg_stats stats{};
  // grow-only staging in HBM
  Buf<uint8_t, false, 256> d_bytes;   // message / leaf bytes: 256 zero bytes readable in front (sha_words)
  DevBuf<uint32_t> d_off32;
  DevBuf<uint64_t> d_off64, d_words;
  DevBuf<uint32_t> d_dig[2];
  IssueOrder dig_order;           // the calls that use d_dig, on the library's stream or the caller's
  // chunked host-buffer scans: H2D of chunk c+1 and D2H of chunk c-1 overlap the kernels of chunk c
  static constexpr int kChunks = 8;
  cudaStream_t s_h2d = nullptr, s_d2h = nullptr; cudaEvent_t e_h2d[kChunks] = {}, e_done[kChunks] = {}; HostBuf<uint32_t> h_chunk_counters;
  // cg_find_matches_batch / cg_redact_batch / cg_policy_verdict_batch staging (grow-only)
  DevBuf<cg_span> d_spans;
  DevBuf<uint8_t> d_redact_out; DevBuf<uint32_t> d_redact_meta;
  DevBuf<uint32_t> d_verdicts;
  DevBuf<uint32_t> d_hits;        // cg_scan_batch's hit list: [count][(msg, rule) pairs]
  DevBuf<uint8_t> d_views;        // the host-buffer *_views calls' view ids, staged beside the offsets
  // cg_policy_eval_batch staging: text roles, context offsets, atom rows, [count][(ctx, rule) pairs]
  DevBuf<uint8_t> d_proles;
  DevBuf<uint32_t> d_pctx, d_patoms, d_pmatch;
  DevBuf<uint32_t> d_roots;       // cg_merkle_root_sharded_device: every rank's block roots (cg_comm_destroy frees them)
};
// never destroyed: no CUDA call may run from a static destructor at process exit (cg_shutdown frees what G holds)
Ctx& G = *new Ctx;

int fail(int code, const std::string& msg) { g_err = msg; return code; }
#define CU(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return cuda_fail(_e, #x); } while (0)
int require_ready() { return G.ready ? CG_OK : fail(CG_ERR_NOT_INITIALIZED, "cg_init has not been called (or no CUDA device)"); }
void count_launches(int k) { G.stats.kernel_launches += k; }

// One call's use of a scratch on st, from before its first use (before anything is grown, captured, copied or launched) to
// after its last: st first waits for the previous call's event when that call ran on another stream (rc: CG_OK or the
// error), and the event is recorded on st when the scope ends.  A null order orders nothing (the call fails its argument
// checks before it touches any scratch).
class InOrder {
 public:
  InOrder(IssueOrder* o, cudaStream_t st) : o_(o), st_(st) {
    if (o && o->last && o->last != st) { const cudaError_t e = cudaStreamWaitEvent(st, o->ev, 0); if (e != cudaSuccess) rc = cuda_fail(e, "cudaStreamWaitEvent"); }
  }
  ~InOrder() { if (o_) { cudaEventRecord(o_->ev, st_); o_->last = st_; } }
  InOrder(const InOrder&) = delete;
  InOrder& operator=(const InOrder&) = delete;
  int rc = CG_OK;
 private:
  IssueOrder* o_; cudaStream_t st_;
};

// NCCL, bound at run time (nccl_load), and the communicator of cg_comm_init
struct NcclApi {
  void* h = nullptr; void* comm = nullptr; int rank = 0, world = 1;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, cg_nccl_id, int) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
} g_nccl;

// The single-message staging block, host (pinned) and device: [offsets, 256 B][message bytes][64 zero bytes] in (kOneIn),
// [word][counters][hit row] out (kOneOut).  The span calls stage their input in their own block (kFew*) and keep the packed
// result (kOnePack bytes, layout in kernels.h) on both sides and, on the device only, the digests and the redacted bytes
// before the pack step moves them behind the spans (kOnePack each).
constexpr uint32_t kOneBytes = 16384, kOneRw = 128, kOneIn = 256 + kOneBytes + 64, kOneOut = (kOneHitRow + kOneRw) * 4;
constexpr uint32_t kOnePack = 512 * 1024;
// The span calls' staging block, host (pinned) and device: [offsets, kFewMsgs + 1][text bytes, kFewBytes][64 zero bytes],
// the offsets rebased to kFewTextAt.  The limits: 256 strings (kFewMsgs: the resolver keeps its per-message arrays in shared
// memory) and 64 KB of text (cg_policy_eval_one's limit); the _one calls keep 16 KB (kOneBytes).
constexpr uint32_t kFewBytes = 65536, kFewTextAt = 1280, kFewIn = kFewTextAt + kFewBytes + 64;
static_assert(4 * (kFewMsgs + 1) <= kFewTextAt && kFewTextAt % 256 == 0 && pack_spans_at(kFewMsgs) < 4096, "span call staging layout");
// cg_policy_eval_one's staging block, host (pinned) and device: in, [offsets, kPeOneTexts + 1][roles][atom row, kPeOneAtomWords]
// [text bytes, kPeOneBytes][64 zero bytes] at fixed places (offsets are rebased to kPeTextAt); out, kPeOneRules + kPeOneRulesCap
// words (kernels.h).  The limits: 64 texts (kPeOneTexts: the kernel keeps the text list in shared memory), 64 KB of text (a tool
// call's params or a message with its conversation history), 32 768 atoms, 4096 matched policies.
constexpr uint32_t kPeOneBytes = 65536, kPeOneAtomWords = 1024, kPeOneRulesCap = 4096;
constexpr uint32_t kPeRolesAt = 512, kPeAtomsAt = kPeRolesAt + 256, kPeTextAt = kPeAtomsAt + 4 * kPeOneAtomWords;
constexpr uint32_t kPeIn = kPeTextAt + kPeOneBytes + 64, kPeOut = 4 * (kPeOneRules + kPeOneRulesCap);
static_assert(4 * (kPeOneTexts + 1) <= kPeRolesAt && kPeOneTexts <= 256 && kPeTextAt % 256 == 0, "cg_policy_eval_one staging layout");

// A blocking call family's pinned host block and device block, of sizes fixed by the family's layout, allocated and zeroed
// by the family's first call
struct Staging {
  const size_t host_bytes, dev_bytes;
  HostBuf<uint8_t> h{}; DevBuf<uint8_t> d{};
  int ensure() {
    if (!h.get()) { if (int rc = h.alloc(host_bytes)) return rc; memset(h.get(), 0, host_bytes); }
    if (!d.get()) { if (int rc = d.alloc(dev_bytes)) return rc; CU(cudaMemset(d.get(), 0, dev_bytes)); }
    return CG_OK;
  }
};

// A call family's step graphs (cached_graph): Cap instances at most, each replayed only for the key it was recorded with
// (the family's launch arguments that are not staged data) and under the scratch generation and verify grid current then
// (a graph holds the scratch pointers, the rule set's device tables and verify_small_kernel's grid by value)
template <typename Key, int Cap>
struct GraphCache {
  struct Entry { cudaGraphExec_t exec = nullptr; int kernels = 0; uint64_t used = 0, gen = 0; int ctas = 0; Key key{}; };
  Entry e[Cap];
  uint64_t clock = 0;
  GraphCache() = default;
  GraphCache(const GraphCache&) = delete;
  GraphCache& operator=(const GraphCache&) = delete;
  ~GraphCache() { for (auto& g : e) if (g.exec) cudaGraphExecDestroy(g.exec); }
};

}  // namespace

int cg::cuda_fail(cudaError_t e, const char* what) {
  g_err = std::string(what) + ": " + cudaGetErrorString(e);
  return CG_ERR_CUDA;
}
struct cg_ruleset {
  HostImage host;
  std::vector<uint32_t> category;
  DevRuleset dev{};
  std::vector<DevBuf<uint8_t>> allocs;     // the device tables of dev and work (upload)
  DevBuf<uint8_t> rule_policy, rule_action;    // dev.rule_policy / dev.rule_action (cg_ruleset_set_policy)
  uint32_t n_sets = 0, program_words = 0;
  // the step scratch: ScanWork's buffers, grouped by the capacity that sizes them (prepare_step)
  struct {
    DevBuf<uint32_t> counters, persist;      // allocated once
    uint32_t msg_cap = 0; DevBuf<uint32_t> slot_of_msg;
    uint32_t l1_cap = 0; DevBuf<uint32_t> l1_pos, l1_fac; DevBuf<uint2> fq;
    uint32_t slot_cap = 0; DevBuf<uint32_t> slot_msg, cand, hit;
    uint32_t event_cap = 0; DevBuf<uint2> events; DevBuf<uint32_t> heavy_idx, event_pos, event_pre;
    uint32_t span_cap = 0; DevBuf<uint32_t> spans, sp_start, sp_len, sp_cat; DevBuf<uint4> sorted, sort_tmp;
    uint32_t res_cap = 0; DevBuf<uint64_t> words, out_len, out_off, scan_part; DevBuf<uint32_t> seg_cnt, seg_begin, kept_cnt, kept_begin;
    void view(ScanWork& w) const {    // (w's rule tables stay as they are)
      w.counters = counters.get(); w.persist = persist.get(); w.msg_cap = msg_cap; w.slot_of_msg = slot_of_msg.get();
      w.l1_cap = l1_cap; w.l1_pos = l1_pos.get(); w.l1_fac = l1_fac.get(); w.fq = fq.get(); w.slot_cap = slot_cap; w.slot_msg = slot_msg.get(); w.cand = cand.get(); w.hit = hit.get();
      w.event_cap = event_cap; w.events = events.get(); w.heavy_idx = heavy_idx.get(); w.event_pos = event_pos.get(); w.event_pre = event_pre.get();
      w.span_cap = span_cap; w.spans = spans.get(); w.sorted = sorted.get(); w.sort_tmp = sort_tmp.get(); w.sp_start = sp_start.get(); w.sp_len = sp_len.get(); w.sp_cat = sp_cat.get();
      w.res_cap = res_cap; w.words = words.get(); w.out_len = out_len.get(); w.out_off = out_off.get(); w.seg_cnt = seg_cnt.get(); w.seg_begin = seg_begin.get();
      w.kept_cnt = kept_cnt.get(); w.kept_begin = kept_begin.get(); w.scan_part = scan_part.get();
    }
  } scratch;
  ScanWork work{};                // scratch as the launchers take it (by value): rebuilt by every prepare_step that grows it
  IssueOrder order;               // the calls that use work and one, on the library's stream or the caller's
  uint64_t seq = 0;               // device-path batches issued so far
  // device path: every batch's counters are mirrored into a ring of pinned slots, so that a queue overflow (results of
  // that batch marked incomplete by finalize_kernel) is seen by the next call / by cg_scan_join and the scratch grows
  static constexpr int kMirror = 16;
  HostBuf<uint32_t> h_counters; cudaEvent_t e_cnt[kMirror] = {}; bool cnt_pending[kMirror] = {};
  uint32_t grow_l1 = 0, grow_slot = 0, grow_ev = 0, grow_span = 0;     // capacities learnt from overflows
  uint32_t sticky_flags = 0;      // error flags of batches since the last cg_scan_join
  uint32_t sticky_status = 0;     // 1 << span resolution status (kResolve*) of batches since the last cg_scan_join
  // verify_small_kernel's grid (CTAs per SM): one while the island matcher decides (nearly) everything, four once a step has
  // sent more than 2048 pairs to the VM (non-ASCII traffic); back to one below 256.  Part of the cached graphs' keys.
  int verify_ctas = 1;
  void size_verify_grid() { const uint32_t ev = last_counters[kCtrEvents]; if (ev > 2048u) verify_ctas = 4; else if (ev < 256u) verify_ctas = 1; }
  uint32_t last_counters[kCounterWords] = {};
  uint64_t scratch_gen = 0;       // advanced by every change to what a captured step holds (scratch buffers, DevRuleset)
  // cg_scan_batch_device's step as one CUDA graph, keyed on (d_bytes, d_offsets, d_words, n): two entries, so that callers
  // that alternate between two input/output buffer sets replay, never re-capture
  GraphCache<std::tuple<const void*, const void*, const void*, uint32_t>, 2> device_graphs;
  // The blocking calls (blocking_call), each family with its staging and its graphs over the staging's fixed addresses.
  // cg_scan_one: the message length is data, so one graph serves every message.
  struct { Staging io{kOneIn + kOneOut, kOneIn + kOneOut}; GraphCache<std::tuple<>, 1> graphs; } one;
  // cg_find_matches_one / cg_redact_one / cg_find_matches_few / cg_redact_few: the input block and the packed result, and
  // the step + resolver (+ digests and splice) + pack per (redact, string count) (the step takes the count by value)
  struct { Staging in{kFewIn, kFewIn}, pack{kOnePack, 3 * (size_t)kOnePack}; GraphCache<std::tuple<bool, uint32_t>, 16> graphs; } span;
  // cg_policy_eval_one: the step + policy_eval_one_kernel per (text count, prog_gen) (a graph holds PolicyTable by value)
  struct { Staging io{kPeIn + kPeOut, kPeIn + kPeOut}; GraphCache<std::tuple<uint32_t, uint64_t>, 8> graphs; } pone;
  // cg_ruleset_set_views: n_views rows of dev.rw words in HBM (bit r of row v = rule r is in view v); none before the first call
  DevBuf<uint32_t> view_rows; uint32_t n_views = 0;
  // cg_ruleset_set_policy_program: the program's words and one rule record per program rule (kernels.h PolicyTable) in HBM;
  // prog_gen advances with every program set (a captured graph holds the tables by value)
  DevBuf<uint32_t> prog_ops; DevBuf<uint4> prog_rules; uint32_t prog_n_rules = 0, prog_n_atoms = 0;
  uint64_t prog_gen = 0;
  ~cg_ruleset() {                 // (the buffers, graph caches and staging blocks release themselves)
    for (auto& e : e_cnt) if (e) cudaEventDestroy(e);
    if (order.ev) cudaEventDestroy(order.ev);
  }
};

namespace {

// v and pad_elems zero elements behind it into one more of the rule set's tables, or into *into (allocated anew) -> *out
template <typename T>
int upload(cg_ruleset* rs, const std::vector<T>& v, const T** out, size_t pad_elems = 4, DevBuf<uint8_t>* into = nullptr) {
  DevBuf<uint8_t>& d = into ? *into : rs->allocs.emplace_back();
  const size_t bytes = (v.size() + pad_elems) * sizeof(T);
  if (int rc = d.alloc(bytes)) return rc;
  CU(cudaMemset(d.get(), 0, bytes));
  if (!v.empty()) CU(cudaMemcpy(d.get(), v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  *out = reinterpret_cast<const T*>(d.get());
  return CG_OK;
}
// one group of scratch buffers at n elements each: all of them freed, then each allocated
template <typename... B>
int regrow(size_t n, B&... b) {
  (b.reset(), ...);
  int rc = CG_OK;
  ((rc = rc ? rc : b.alloc(n)), ...);
  return rc;
}

// What a step computes: result words only; a policy step whose per-message scratch a hit list or verdicts read afterwards;
// or a span step (raw spans for the span resolver, result words in ScanWork::words).
enum StepKind { kStepWords, kStepPolicy, kStepSpans };

// One step on device-resident input: scratch reset, gram scan (+ exact factors), resolve, verify, finalize; over no message
// only the zeroed counter block.  With views, resolve admits only the (message, rule) pairs of each message's view.
// Asynchronous.
int run_scan_device(cg_ruleset* rs, const uint8_t* d_bytes, const uint32_t* d_off, uint32_t n, uint64_t* d_words, StepKind kind, cudaStream_t st,
                    const ViewTable* views = nullptr) {
  const ScanWork& w = rs->work;
  if (!n) { CU(cudaMemsetAsync(w.counters, 0, kCounterWords * sizeof(uint32_t), st)); return CG_OK; }
  const bool spans = kind == kStepSpans;
  int k = launch_reset(rs->dev, w, n, G.sm_count, st);
  if (G.profiling) cudaEventRecord(G.pev[0], st);
  k += launch_scan(rs->dev, w, d_bytes, d_off, n, d_words, G.sm_count, st);
  if (G.profiling) cudaEventRecord(G.pev[1], st);
  k += launch_confirm(rs->dev, w, d_bytes, d_off, n, G.sm_count, st);
  if (G.profiling) cudaEventRecord(G.pev[2], st);
  k += launch_resolve(rs->dev, w, d_bytes, d_off, n, spans, G.sm_count, st, views);
  if (G.profiling) cudaEventRecord(G.pev[3], st);
  k += launch_verify(rs->dev, w, d_bytes, d_off, spans, G.sm_count, st, spans ? 4 : rs->verify_ctas);
  if (G.profiling) cudaEventRecord(G.pev[4], st);
  k += launch_finalize(rs->dev, w, d_words, n, G.sm_count, st);
  if (G.profiling) cudaEventRecord(G.pev[5], st);
  count_launches(k);
  CU(cudaGetLastError());
  return CG_OK;
}

void prepare_kernels() { static bool done = false; if (!done) { prepare_scan_kernels(); done = true; } }

// capacities a batch of n messages starts with (confirmed occurrences are rare: about one per hundred messages on chat text;
// a step without spans writes none)
void default_caps(const cg_ruleset* rs, uint32_t n, StepKind kind, uint32_t* l1, uint32_t* slot, uint32_t* ev, uint32_t* span) {
  *l1 = std::max(std::max<uint32_t>(std::max<uint32_t>(2 * n, 1u << 16), rs->work.l1_cap), rs->grow_l1);
  *slot = std::max(std::max<uint32_t>(std::max<uint32_t>(n / 4, 4096), rs->work.slot_cap), rs->grow_slot);
  *ev = std::max(std::max<uint32_t>(std::max<uint32_t>(n, 4096), rs->work.event_cap), rs->grow_ev);
  *span = kind == kStepSpans ? std::max(std::max<uint32_t>(std::max<uint32_t>(n, 4096), rs->work.span_cap), rs->grow_span) : 1;
}
// the verify grid and the scratch of a step over n messages, with per-message scratch for at least res_min items behind a
// policy step; growing waits for st (nothing may still use a replaced buffer)
int prepare_step(cg_ruleset* rs, uint32_t n, StepKind kind, cudaStream_t st, uint32_t res_min = 0) {
  rs->size_verify_grid();
  const ScanWork& w = rs->work;
  uint32_t l1, slot, ev, span;
  default_caps(rs, n, kind, &l1, &slot, &ev, &span);
  n = std::max<uint32_t>(n, 1);
  const uint32_t res = kind != kStepWords ? std::max(n, res_min) : 0;
  if (n <= w.msg_cap && l1 <= w.l1_cap && slot <= w.slot_cap && ev <= w.event_cap && span <= w.span_cap && res <= w.res_cap) return CG_OK;
  CU(cudaStreamSynchronize(st));
  rs->scratch_gen++;
  // a group's capacity is recorded once all its buffers are there; rs->work is rebuilt on every return (no freed buffer in it)
  auto& s = rs->scratch; int rc;
  struct View { cg_ruleset* rs; ~View() { rs->scratch.view(rs->work); } } view{rs};
  if (!s.counters.get()) { if ((rc = s.counters.alloc(kCounterWords)) || (rc = s.persist.alloc(4))) return rc; CU(cudaMemset(s.persist.get(), 0, 16)); CU(cudaDeviceSynchronize()); }
  if (n > s.msg_cap) { s.msg_cap = 0; if ((rc = regrow(n, s.slot_of_msg))) return rc; s.msg_cap = n; }
  if (l1 > s.l1_cap) { s.l1_cap = 0; if ((rc = regrow(l1, s.l1_pos, s.l1_fac, s.fq))) return rc; s.l1_cap = l1; }
  if (slot > s.slot_cap) {
    const size_t rows = (size_t)slot * (rs->dev.rw ? rs->dev.rw : 1);
    s.slot_cap = 0; s.slot_msg.reset();
    if ((rc = regrow(rows, s.cand, s.hit)) || (rc = s.slot_msg.alloc(slot))) return rc;
    // rows start out zero and every step clears the ones it used (reset_kernel)
    CU(cudaMemset(s.cand.get(), 0, rows * 4)); CU(cudaMemset(s.hit.get(), 0, rows * 4)); CU(cudaMemset(s.persist.get(), 0, 16)); CU(cudaDeviceSynchronize());
    s.slot_cap = slot;
  }
  if (ev > s.event_cap) { s.event_cap = 0; if ((rc = regrow(ev, s.events, s.heavy_idx, s.event_pos, s.event_pre))) return rc; s.event_cap = ev; }
  if (span > s.span_cap) {
    s.span_cap = 0; s.spans.reset();
    if ((rc = regrow(span, s.sorted, s.sort_tmp, s.sp_start, s.sp_len, s.sp_cat)) || (rc = s.spans.alloc((size_t)span * 6))) return rc;
    s.span_cap = span;
  }
  if (res > s.res_cap || (res && !s.scan_part.get())) {
    s.res_cap = 0;
    if ((rc = regrow((size_t)res + 1, s.words, s.out_len, s.out_off, s.seg_cnt, s.seg_begin, s.kept_cnt, s.kept_begin))) return rc;
    if (!s.scan_part.get() && (rc = s.scan_part.alloc(kScanPartials))) return rc;
    s.res_cap = res;
  }
  return CG_OK;
}
// what an overflowed step teaches about the capacities the next one needs
void learn_caps(cg_ruleset* rs, const uint32_t* hc) {
  const uint32_t flags = hc[kCtrErrors];
  if (flags & ERR_L1_OVERFLOW) { const uint32_t need = std::max(hc[kCtrConfirmed], hc[kCtrFlagWords]); rs->grow_l1 = std::max<uint32_t>(rs->grow_l1, std::max<uint32_t>(2 * need, need + 65536)); }
  if (flags & ERR_SLOT_OVERFLOW) rs->grow_slot = std::max<uint32_t>(rs->grow_slot, std::max<uint32_t>(2 * hc[kCtrSlots], hc[kCtrSlots] + 4096));
  if (flags & ERR_EVENT_OVERFLOW) rs->grow_ev = std::max<uint32_t>(rs->grow_ev, std::max<uint32_t>(2 * hc[kCtrEvents], hc[kCtrEvents] + 4096));
  if (flags & ERR_SPAN_OVERFLOW) rs->grow_span = std::max<uint32_t>(rs->grow_span, std::max<uint32_t>(2 * hc[kCtrRawSpans], hc[kCtrRawSpans] + 4096));
}
const char* const kVmOverflow = "matcher thread list / stack overflow on device";
// a finished step's counter block -> CG_OK, CG_ERR_TOO_LARGE, or 1 = a queue overflowed (the capacities the step needs
// have been learnt)
int absorb_counters(cg_ruleset* rs, const uint32_t* hc) {
  memcpy(rs->last_counters, hc, sizeof rs->last_counters);
  if (hc[kCtrErrors] & (ERR_VM_STACK | ERR_VM_LIST)) return fail(CG_ERR_TOO_LARGE, kVmOverflow);
  if (hc[kCtrErrors]) learn_caps(rs, hc);
  return hc[kCtrErrors] ? 1 : CG_OK;
}
// the statistics of a completed host-side step over n messages of `bytes` bytes (device calls count messages at enqueue and
// the rest in poll_mirrors)
void count_step(uint32_t n, uint64_t bytes, const uint32_t* hc) {
  G.stats.messages_scanned += n; G.stats.bytes_scanned += bytes;
  G.stats.candidate_events += hc[kCtrEvents]; G.stats.verified_pairs += hc[kCtrEvents];
}
// the kernels enqueue() puts on st, recorded as one graph (*graph: the caller's to destroy); they are counted each time an
// instance is launched, not here
template <typename Enqueue>
int record(cudaStream_t st, Enqueue&& enqueue, cudaGraph_t* graph, int* kernels) {
  cudaGraph_t g = nullptr;
  const uint64_t before = G.stats.kernel_launches;
  CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  const int rc = enqueue();
  cudaError_t e = cudaStreamEndCapture(st, &g);
  *kernels = (int)(G.stats.kernel_launches - before); G.stats.kernel_launches = before;
  if (rc != CG_OK || e != cudaSuccess) { if (g) cudaGraphDestroy(g); cudaGetLastError(); return rc != CG_OK ? rc : cuda_fail(e, "cudaStreamEndCapture"); }
  *graph = g;
  return CG_OK;
}
// *out = the cache's graph of key for the current scratch and verify grid.  On a miss enqueue() is recorded afresh on st
// into the least recently used entry, whose instance is re-targeted (cudaGraphExecUpdate: where the launch sequence is the
// same, only parameters change) and instantiated anew only when the update is refused.
template <typename Key, int Cap, typename Enqueue>
int cached_graph(cg_ruleset* rs, GraphCache<Key, Cap>& c, const Key& key, cudaStream_t st, Enqueue&& enqueue, typename GraphCache<Key, Cap>::Entry** out) {
  typename GraphCache<Key, Cap>::Entry* g = nullptr;
  for (auto& e : c.e) if (e.exec && e.key == key && e.gen == rs->scratch_gen && e.ctas == rs->verify_ctas) g = &e;
  if (!g) {
    g = &c.e[0];
    for (auto& e : c.e) if (e.used < g->used) g = &e;
    cudaGraph_t graph = nullptr;
    int kernels = 0;
    if (int rc = record(st, enqueue, &graph, &kernels)) return rc;
    cudaGraphExecUpdateResultInfo info;
    if (!g->exec || cudaGraphExecUpdate(g->exec, graph, &info) != cudaSuccess) {
      cudaGetLastError();                                     // (a refused update is not an error of the call)
      if (g->exec) { cudaGraphExecDestroy(g->exec); g->exec = nullptr; }
      const cudaError_t e = cudaGraphInstantiate(&g->exec, graph, 0);
      if (e != cudaSuccess) { cudaGraphDestroy(graph); g->exec = nullptr; return cuda_fail(e, "cudaGraphInstantiate"); }
    }
    cudaGraphDestroy(graph);
    g->key = key; g->gen = rs->scratch_gen; g->ctas = rs->verify_ctas; g->kernels = kernels;
  }
  g->used = ++c.clock;
  *out = g;
  return CG_OK;
}
// the rules of one hit row (rw words), lowest first: put(i, rule) for the i-th rule of the output while i < cap; returns nh
// plus the number of rules in the row (cg_scan_one's single row; batches build their hit list on the device)
template <typename Put>
uint32_t append_hit_row(const uint32_t* row, uint32_t rw, uint32_t nh, uint32_t cap, Put&& put) {
  for (uint32_t k = 0; k < rw; k++)
    for (uint32_t v = row[k]; v; v &= v - 1, nh++) if (nh < cap) put(nh, k * 32 + (uint32_t)__builtin_ctz(v));
  return nh;
}

int check_offsets(const uint32_t* offsets, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) if (offsets[i + 1] < offsets[i]) return fail(CG_ERR_INVALID_ARG, "offsets must be non-decreasing");
  return CG_OK;
}

// The host-buffer calls' driver: stages the batch into G.d_bytes / G.d_off32, then per attempt the step of `kind` (result
// words to G.d_words, a span step's to the scratch), the work after(scratch) enqueues behind it (-> CG_OK or an error; it
// may copy sizes to the host, never into the caller's buffers), the counter block to the host and one synchronise.  A
// queue overflow grows the scratch and runs the attempt again.  last_scan_ms times the step alone.  views (one id per message,
// checked by the caller): staged beside the offsets, the step filtered by them.  res_min: as prepare_step.
template <typename After>
int scan_host(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, StepKind kind, After&& after, const uint8_t* views = nullptr,
              uint32_t res_min = 0) {
  if (int rc = require_ready()) return rc;
  if (!rs || (n && (!bytes || !offsets))) return fail(CG_ERR_INVALID_ARG, "null argument");
  int rc;
  if (n && (rc = check_offsets(offsets, n))) return rc;
  const size_t first = n ? offsets[0] : 0, total = n ? offsets[n] : 0;
  if ((rc = G.d_bytes.grow(total + 64))) return rc;
  if ((rc = G.d_off32.grow((size_t)n + 1))) return rc;
  if ((rc = G.d_words.grow((size_t)n + 1))) return rc;
  if (views && (rc = G.d_views.grow((size_t)n + 1))) return rc;
  cudaStream_t st = G.stream;
  if (n) {
    if (total > first) CU(cudaMemcpyAsync(G.d_bytes.get() + first, bytes + first, total - first, cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(G.d_bytes.get() + total, 0, 64, st));
    CU(cudaMemcpyAsync(G.d_off32.get(), offsets, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, st));
    if (views) CU(cudaMemcpyAsync(G.d_views.get(), views, n, cudaMemcpyHostToDevice, st));
  }
  const ViewTable vt{rs->view_rows.get(), G.d_views.get(), rs->n_views};
  uint32_t hc[kCounterWords] = {};
  for (int attempt = 0; attempt < 10; attempt++) {
    if ((rc = prepare_step(rs, n, kind, st, res_min))) return rc;
    const ScanWork& w = rs->work;
    CU(cudaEventRecord(G.ev0, st));
    if ((rc = run_scan_device(rs, G.d_bytes.get(), G.d_off32.get(), n, kind == kStepSpans ? w.words : G.d_words.get(), kind, st, views ? &vt : nullptr))) return rc;
    CU(cudaEventRecord(G.ev1, st));
    if ((rc = after(w))) return rc;
    CU(cudaMemcpyAsync(hc, w.counters, kCounterWords * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    float ms = 0; cudaEventElapsedTime(&ms, G.ev0, G.ev1); G.stats.last_scan_ms = ms;
    if ((rc = absorb_counters(rs, hc)) == 1) continue;
    if (rc) return rc;
    count_step(n, total - first, hc);
    return CG_OK;
  }
  return fail(CG_ERR_CAPACITY, "candidate queues kept overflowing");
}

int ensure_copy_streams() {
  if (G.s_h2d) return CG_OK;
  const int C = Ctx::kChunks;
  CU(cudaStreamCreateWithFlags(&G.s_h2d, cudaStreamNonBlocking)); CU(cudaStreamCreateWithFlags(&G.s_d2h, cudaStreamNonBlocking));
  for (int c = 0; c < C; c++) { CU(cudaEventCreateWithFlags(&G.e_h2d[c], cudaEventDisableTiming)); CU(cudaEventCreateWithFlags(&G.e_done[c], cudaEventDisableTiming)); }
  return G.h_chunk_counters.alloc((size_t)C * kCounterWords);
}

// Words-only scan of a large host batch in kChunks pieces: the H2D copy of piece c+1 and the D2H copy of piece c-1 run
// on their own streams while the kernels of piece c run -- end to end the call then costs little more than the H2D copy
// alone.  Returns 1 when a queue overflowed somewhere (capacities have been grown; the caller re-runs in one piece).
int scan_host_chunked(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint64_t* out_words) {
  const int C = Ctx::kChunks;
  int rc;
  if ((rc = check_offsets(offsets, n))) return rc;
  const size_t total = offsets[n];
  if ((rc = G.d_bytes.grow(total + 64))) return rc;
  if ((rc = G.d_off32.grow((size_t)n + 1))) return rc;
  if ((rc = G.d_words.grow((size_t)n + 1))) return rc;
  if ((rc = ensure_copy_streams())) return rc;
  cudaStream_t st = G.stream;
  InOrder turn(&rs->order, st);
  if (turn.rc) return turn.rc;
  const uint32_t per = (n + C - 1) / C;
  CU(cudaStreamSynchronize(st));                            // (whatever still read the staging buffers is done: s_h2d does not wait for st)
  if ((rc = prepare_step(rs, per, kStepWords, st))) return rc;
  CU(cudaMemcpyAsync(G.d_off32.get(), offsets, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, G.s_h2d));
  CU(cudaMemsetAsync(G.d_bytes.get() + total, 0, 64, G.s_h2d));
  CU(cudaEventRecord(G.ev0, st));
  int used = 0;
  for (int c = 0; c < C; c++) {
    const uint32_t m0 = std::min<uint64_t>((uint64_t)c * per, n), m1 = std::min<uint64_t>((uint64_t)(c + 1) * per, n);
    if (m1 <= m0) break;
    used = c + 1;
    const size_t b0 = offsets[m0], b1 = offsets[m1];
    if (b1 > b0) CU(cudaMemcpyAsync(G.d_bytes.get() + b0, bytes + b0, b1 - b0, cudaMemcpyHostToDevice, G.s_h2d));
    CU(cudaEventRecord(G.e_h2d[c], G.s_h2d));
    CU(cudaStreamWaitEvent(st, G.e_h2d[c], 0));
    // (a piece reads up to 16 bytes past its last message -- bytes of the next piece that may still be in flight; whatever
    // it sees there cannot produce an occurrence inside its own range)
    if ((rc = run_scan_device(rs, G.d_bytes.get(), G.d_off32.get() + m0, m1 - m0, G.d_words.get() + m0, kStepWords, st))) return rc;
    CU(cudaMemcpyAsync(G.h_chunk_counters.get() + (size_t)c * kCounterWords, rs->work.counters, kCounterWords * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(G.e_done[c], st));
    CU(cudaStreamWaitEvent(G.s_d2h, G.e_done[c], 0));
    if (out_words) CU(cudaMemcpyAsync(out_words + m0, G.d_words.get() + m0, (size_t)(m1 - m0) * 8, cudaMemcpyDeviceToHost, G.s_d2h));
  }
  CU(cudaEventRecord(G.ev1, st));
  CU(cudaStreamSynchronize(st)); CU(cudaStreamSynchronize(G.s_d2h)); CU(cudaStreamSynchronize(G.s_h2d));
  float ms = 0; cudaEventElapsedTime(&ms, G.ev0, G.ev1); G.stats.last_scan_ms = ms;
  bool overflow = false;
  for (int c = 0; c < used; c++) {
    if ((rc = absorb_counters(rs, G.h_chunk_counters.get() + (size_t)c * kCounterWords)) < 0) return rc;
    overflow |= rc == 1;
  }
  if (overflow) return 1;
  for (int c = 0; c < used; c++) {
    const uint32_t m0 = c * per, m1 = std::min<uint64_t>((uint64_t)(c + 1) * per, n);
    count_step(m1 - m0, offsets[m1] - offsets[m0], G.h_chunk_counters.get() + (size_t)c * kCounterWords);
  }
  return CG_OK;
}

// device path: look at every mirrored counter block whose copy has completed
void poll_mirrors(cg_ruleset* rs, bool wait) {
  for (int i = 0; i < cg_ruleset::kMirror; i++) {
    if (!rs->cnt_pending[i]) continue;
    if (wait) cudaEventSynchronize(rs->e_cnt[i]);
    else if (cudaEventQuery(rs->e_cnt[i]) != cudaSuccess) { cudaGetLastError(); continue; }
    rs->cnt_pending[i] = false;
    const uint32_t* hc = rs->h_counters.get() + (size_t)i * kCounterWords;
    rs->sticky_flags |= hc[kCtrErrors];
    if (!hc[kCtrErrors]) rs->sticky_status |= hc[kCtrResolveStatus] ? 1u << hc[kCtrResolveStatus] : 0u;
    G.stats.spans += hc[kCtrResolved]; G.stats.sha256_items += hc[kCtrDigests]; G.stats.hits += hc[kCtrHits];     // (zero for steps without them)
    absorb_counters(rs, hc);                                // (cg_scan_join reports the flags)
  }
}

// device path: the pinned counter mirror ring (allocated by the first device-path call)
int ensure_mirrors(cg_ruleset* rs) {
  if (rs->h_counters.get()) return CG_OK;
  if (int rc = rs->h_counters.alloc((size_t)cg_ruleset::kMirror * kCounterWords)) return rc;
  for (auto& e : rs->e_cnt) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  return CG_OK;
}
// device path: copy the counter block of the batch just enqueued on st into the next mirror slot
int mirror_counters(cg_ruleset* rs, cudaStream_t st) {
  const int slot = (int)(rs->seq % cg_ruleset::kMirror);
  if (rs->cnt_pending[slot]) { cudaEventSynchronize(rs->e_cnt[slot]); poll_mirrors(rs, false); }
  CU(cudaMemcpyAsync(rs->h_counters.get() + (size_t)slot * kCounterWords, rs->work.counters, kCounterWords * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(rs->e_cnt[slot], st));
  rs->cnt_pending[slot] = true; rs->seq++;
  return CG_OK;
}

// n + 1 offsets rebased to text_at, the n strings' bytes from there on and 64 zero bytes behind them into a staging block's
// host side -> the bytes of it to copy to the device
size_t stage_texts(uint8_t* h, uint32_t text_at, const uint8_t* bytes, const uint32_t* offsets, uint32_t n) {
  const uint32_t first = n ? offsets[0] : 0, len = n ? offsets[n] - first : 0;
  uint32_t* hoff = reinterpret_cast<uint32_t*>(h);
  for (uint32_t i = 0; i <= n; i++) hoff[i] = text_at + (n ? offsets[i] - first : 0);
  if (len) memcpy(h + text_at, bytes + first, len);
  memset(h + text_at + len, 0, 64);
  return (size_t)text_at + len + 64;
}

// The blocking calls' driver, one device round trip on the library's stream: the rule set's turn, the family's staging,
// the scratch of a `kind` step over n items (res_min: as prepare_step), the graph of key from the family's cache (enqueue:
// the step over the staged input and the family's kernels behind it, recorded on a miss), the first stage(in.h) bytes of
// `in` to the device, one graph launch, `bytes` bytes at `at` of `out` back to its host side, one synchronise.  -> CG_OK,
// an error, or 1 = a queue overflowed (counter block at byte `counters` of out.h; the capacities have been learnt): take
// the batch call.
template <typename Key, int Cap, typename Stage, typename Enqueue>
int blocking_call(cg_ruleset* rs, StepKind kind, uint32_t n, uint32_t res_min, GraphCache<Key, Cap>& cache, const Key& key, Staging& in, Stage&& stage,
                  Enqueue&& enqueue, Staging& out, size_t at, size_t bytes, size_t counters) {
  cudaStream_t st = G.stream;
  InOrder turn(&rs->order, st);
  int rc;
  if ((rc = turn.rc) || (rc = in.ensure()) || (rc = out.ensure())) return rc;
  if ((rc = prepare_step(rs, n, kind, st, res_min))) return rc;
  typename GraphCache<Key, Cap>::Entry* g = nullptr;
  if ((rc = cached_graph(rs, cache, key, st, enqueue, &g))) return rc;
  CU(cudaMemcpyAsync(in.d.get(), in.h.get(), stage(in.h.get()), cudaMemcpyHostToDevice, st));
  CU(cudaGraphLaunch(g->exec, st));
  CU(cudaMemcpyAsync(out.h.get() + at, out.d.get() + at, bytes, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  count_launches(g->kernels);
  return absorb_counters(rs, reinterpret_cast<const uint32_t*>(out.h.get() + counters));
}

// cg_scan_batch_device's step replayed as one CUDA graph -- one launch per step instead of six, so the host never becomes
// the bottleneck
template <typename Step>
int replay_step(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_words, cudaStream_t st, Step&& step) {
  decltype(rs->device_graphs)::Entry* g = nullptr;
  if (int rc = cached_graph(rs, rs->device_graphs, {d_bytes, d_offsets, d_words, n}, st, step, &g)) return rc;
  CU(cudaGraphLaunch(g->exec, st));
  count_launches(g->kernels);
  return CG_OK;
}

// The device-resident calls' driver, asynchronous on st: grows the scratch first if an earlier batch overflowed, enqueues
// the step of `kind` (replayed as a graph when `graph`), the work after(scratch) enqueues behind it (-> its launch count)
// and the counter block into the mirror ring.  Result words go to d_words, or when it is null to the scratch's (looked up
// after prepare_step, which may replace that buffer).  Never waits for the device except when the scratch must grow.  views:
// the step filtered by them (never replayed as a graph).  res_min: as prepare_step.
template <typename After>
int scan_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, uint64_t* d_words, StepKind kind, cudaStream_t st,
                After&& after, bool graph = false, const ViewTable* views = nullptr, uint32_t res_min = 0) {
  InOrder turn(&rs->order, st);
  int rc;
  if ((rc = turn.rc)) return rc;
  if ((rc = ensure_mirrors(rs))) return rc;
  poll_mirrors(rs, false);                                  // (an earlier batch overflowed?  grow before this one runs)
  if ((rc = prepare_step(rs, n, kind, st, res_min))) return rc;
  if (!d_words) d_words = rs->work.words;
  const auto step = [&] { return run_scan_device(rs, (const uint8_t*)d_bytes, (const uint32_t*)d_offsets, n, d_words, kind, st, views); };
  if ((rc = graph ? replay_step(rs, d_bytes, d_offsets, n, d_words, st, step) : step())) return rc;
  count_launches(after(rs->work));
  CU(cudaGetLastError());
  G.stats.messages_scanned += n;
  return mirror_counters(rs, st);
}

// the checks every device-resident call starts with: an initialised library, a rule set and the batch in HBM (16-byte aligned)
int device_batch_args(const cg_ruleset* rs, const void* d_bytes, const void* d_offsets) {
  if (int rc = require_ready()) return rc;
  if (!rs || !d_bytes || !d_offsets) return fail(CG_ERR_INVALID_ARG, "null argument");
  if ((uintptr_t)d_bytes & 15u) return fail(CG_ERR_INVALID_ARG, "d_bytes must be 16-byte aligned");
  return CG_OK;
}

// the redacted output behind a span resolver: SHA-256 of every resolved span into d_digests, then the copy + placeholder
// splice of n messages into d_out.  The resolver set how many of each run (counters[kCtrDigests] / [kCtrSplice]: none unless
// every output fits).
int enqueue_redact_tail(const ScanWork& w, const uint8_t* d_bytes, const uint32_t* d_off, const uint32_t* d_out_offsets, uint32_t* d_digests,
                        uint8_t* d_out, uint32_t n, cudaStream_t st) {
  const int k = launch_redact_digests(d_bytes, w.sp_start, w.sp_len, w.counters + kCtrDigests, d_digests, G.sm_count, st);
  return k + launch_redact_splice(d_bytes, d_off, d_out_offsets, w.kept_begin, w.sp_start, w.sp_len, w.sp_cat, d_digests, d_out,
                                  w.counters + kCtrSplice, n, G.sm_count, st);
}

}  // namespace

extern "C" {

int cg_version(void) { return 100; }
const char* cg_last_error(void) { return g_err.c_str(); }

int cg_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int cg_init(int device) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (G.ready) return CG_OK;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) { cudaGetLastError(); return fail(CG_ERR_CUDA, "no CUDA device available (this library has no CPU fallback)"); }
  if (device >= 0) CU(cudaSetDevice(device));
  CU(cudaGetDevice(&G.device));
  cudaDeviceProp prop; CU(cudaGetDeviceProperties(&prop, G.device));
  if (prop.major != 9 || prop.minor != 0) return fail(CG_ERR_CUDA, "device is not sm_90 (kernels are built for sm_90a only)");
  G.sm_count = prop.multiProcessorCount;
  CU(cudaStreamCreateWithFlags(&G.stream, cudaStreamNonBlocking));
  CU(cudaEventCreate(&G.ev0)); CU(cudaEventCreate(&G.ev1));
  for (cudaEvent_t& e : G.pev) CU(cudaEventCreate(&e));
  CU(cudaEventCreateWithFlags(&G.dig_order.ev, cudaEventDisableTiming));

  G.ready = true;
  return CG_OK;
}

void cg_shutdown(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!G.ready) return;
  cudaDeviceSynchronize();
  if (G.s_h2d) { cudaStreamDestroy(G.s_h2d); cudaStreamDestroy(G.s_d2h); for (int c = 0; c < Ctx::kChunks; c++) { cudaEventDestroy(G.e_h2d[c]); cudaEventDestroy(G.e_done[c]); } }
  cudaEventDestroy(G.dig_order.ev);
  cudaEventDestroy(G.ev0); cudaEventDestroy(G.ev1); for (cudaEvent_t e : G.pev) cudaEventDestroy(e); cudaStreamDestroy(G.stream);
  G = Ctx();                      // (frees every buffer G held)
}

int cg_set_profiling(int on) { G.profiling = on != 0; return CG_OK; }

// device time between profiling events pev[from] and pev[to] of the most recent completed step
static int elapsed_ms(int from, int to, float* out) {
  *out = 0;
  if (cudaEventElapsedTime(out, G.pev[from], G.pev[to]) == cudaSuccess) return CG_OK;
  cudaGetLastError();
  return fail(CG_ERR_CUDA, "profiling events not recorded / not complete");
}

int cg_last_kernel_ms(float out_ms[4]) {
  // device time of scan_kernel / confirm_kernel + resolve / verify / finalize of the most recent *completed* scan step
  if (!G.ready || !out_ms) return fail(CG_ERR_INVALID_ARG, "not initialised");
  static const int ev[5] = {0, 1, 3, 4, 5};
  for (int i = 0; i < 4; i++) if (int rc = elapsed_ms(ev[i], ev[i + 1], &out_ms[i])) return rc;
  return CG_OK;
}

int cg_last_tail_ms(float out_ms[2]) {
  // confirm_kernel / resolve_kernel of the most recent completed step in profiling mode
  if (!G.ready || !out_ms) return fail(CG_ERR_INVALID_ARG, "not initialised");
  for (int i = 0; i < 2; i++) if (int rc = elapsed_ms(1 + i, 2 + i, &out_ms[i])) return rc;
  return CG_OK;
}

int cg_scan_work_counters(const cg_ruleset* rs, uint32_t out16[16]) {
  // [0] slots (messages with confirmed candidates), [1] (message, rule) pairs sent to the VM, [2] spans, [3] error flags,
  // [4] confirmed factor occurrences, [5] verify kernel's event cursor, [6] flagged grams (level 1a) -- of the last step
  // whose counters reached the host (cg_scan_batch: the call itself; device path: after cg_scan_join)
  if (!rs || !out16) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!rs->work.counters) return fail(CG_ERR_INVALID_ARG, "no scan has run");
  memcpy(out16, rs->last_counters, 64);
  if (!(rs->dev.debug_flags & 2u)) { out16[7] = rs->last_counters[kCtrPastRecheck]; out16[8] = rs->last_counters[kCtrFlagWords]; out16[9] = rs->last_counters[kCtrPairs]; }   // grams past the recheck map, flag words, (gram, entry) pairs
  return CG_OK;
}

int cg_get_stats(cg_stats* out) { if (!out) return fail(CG_ERR_INVALID_ARG, "null"); *out = G.stats; return CG_OK; }
uint64_t cg_launch_count(void) { return G.stats.kernel_launches; }

int cg_rule_check(const char* source, uint32_t source_len, uint32_t flags, char* err, uint32_t err_len) {
  CompiledRule r = compile_rule(source ? source : "", source_len, flags);
  if (err && err_len) { snprintf(err, err_len, "%s", r.error.c_str()); }
  if (r.status == RULE_OK) return CG_OK;
  g_err = r.error;
  return r.status == RULE_ERR_SYNTAX ? CG_ERR_SYNTAX : r.status == RULE_ERR_UNSUPPORTED ? CG_ERR_UNSUPPORTED : CG_ERR_TOO_LARGE;
}

int cg_ruleset_create(const cg_rule* rules, uint32_t n_rules, uint32_t options, cg_ruleset** out, int32_t* status_per_rule) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!out || (n_rules && !rules)) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (int rc = require_ready()) return rc;
  std::unique_ptr<cg_ruleset> rs(new cg_ruleset());
  CU(cudaEventCreateWithFlags(&rs->order.ev, cudaEventDisableTiming));
  std::vector<RuleSrc> src(n_rules);
  rs->category.resize(n_rules);
  for (uint32_t i = 0; i < n_rules; i++) { src[i] = RuleSrc{rules[i].source, rules[i].source_len, rules[i].flags}; rs->category[i] = rules[i].category; }
  ImageOptions io;
  io.stride = (options & 7u) == CG_OPT_STRIDE2 ? 2 : (options & 7u) == CG_OPT_STRIDE4 ? 4 : 0;
  if (const char* e = getenv("CG_BLOOM2")) io.bloom2 = atoi(e);
  std::string perr;
  if (!build_host_image(src.data(), n_rules, io, &rs->host, &perr)) return fail(CG_ERR_TOO_LARGE, perr);
  HostImage& H = rs->host;
  for (uint32_t i = 0; i < n_rules; i++) {
    int32_t st = H.rules[i].status;
    int32_t code = st == RULE_OK ? CG_OK : st == RULE_ERR_SYNTAX ? CG_ERR_SYNTAX : st == RULE_ERR_UNSUPPORTED ? CG_ERR_UNSUPPORTED : CG_ERR_TOO_LARGE;
    if (status_per_rule) status_per_rule[i] = code;
    else if (code != CG_OK) return fail(code, "rule " + std::to_string(i) + ": " + H.rules[i].error);
  }
  const Prefilter& P = H.pf;
  const std::vector<uint32_t>&prog = H.prog, &prog_off = H.prog_off, &sets = H.sets, &first = H.first;
  const std::vector<uint16_t>& ranges = H.ranges;
  rs->n_sets = H.n_sets; rs->program_words = (uint32_t)H.prog.size();
  if (P.shapes.size() > 16) return fail(CG_ERR_TOO_LARGE, "internal: more than 16 gram shapes");

  DevRuleset& d = rs->dev;
  int rc;
  const uint8_t* d_image; if ((rc = upload(rs.get(), H.image, &d_image, 16))) return rc;
  d.image = d_image; d.image_bytes = H.bm_bytes; d.stride = (uint32_t)P.stride;
  d.bm_mask = H.bm_mask; d.bloom2 = H.bloom2 ? 1u : 0u; d.rk_off = H.rk_off; d.rk_mask = H.rk_bytes - 4; d.tables_resident = H.tables_resident ? 1u : 0u;
  d.dir_off = H.dir_off; d.ent_off = H.ent_off; d.nb_shift = H.nb_shift;
  d.n_shapes = (uint32_t)P.shapes.size(); for (uint32_t k = 0; k < 16; k++) d.shapes[k] = k < d.n_shapes ? P.shapes[k] : 0;
  d.n_trig = (uint32_t)P.trig_bytes.size(); for (uint32_t t = 0; t < 2; t++) d.trig_byte[t] = t < d.n_trig ? P.trig_bytes[t] : 0;
  d.hot_c5f = 0x5f5f5f5fu; d.hot_c10 = 0x10101010u; d.hot_one = 1u;
  d.debug_flags = 0; if (const char* e = getenv("CG_SCAN_DEBUG")) d.debug_flags = (uint32_t)atoi(e);   // 1: drop flagged grams (timing experiments only, results wrong)
  if ((rc = upload(rs.get(), P.trig_offsets, &d.trig_offsets))) return rc;
  if ((rc = upload(rs.get(), P.trig_list, &d.trig_list))) return rc;
  if ((rc = upload(rs.get(), H.bucket_start, &d.bucket_start))) return rc;
  { const uint32_t* ew = nullptr; if ((rc = upload(rs.get(), H.entry_words, &ew, 8))) return rc; d.entries = reinterpret_cast<const uint2*>(ew); }
  { const uint32_t* sw = nullptr; if ((rc = upload(rs.get(), H.slot_words, &sw, 16))) return rc; d.slots = reinterpret_cast<const uint4*>(sw); }
  if ((rc = upload(rs.get(), H.group_entries, &d.group_entries))) return rc;
  d.slot_shift = H.slot_shift; d.slot_mask = H.n_slots - 1;
  {
    // confirm_kernel's tables in one block (kernels.h)
    std::vector<uint8_t> cf;
    auto put = [&](const void* p, size_t bytes, size_t pad = 0) { const uint32_t o = (uint32_t)cf.size(); cf.resize((cf.size() + bytes + pad + 15) & ~(size_t)15, 0); if (bytes) memcpy(cf.data() + o, p, bytes); return o; };
    put(H.image.data() + H.rk_off, H.rk_bytes);
    d.cf_slots_off = put(H.slot_words.data(), H.slot_words.size() * 4);
    d.cf_ge_off = put(H.group_entries.data(), H.group_entries.size() * 4, 16);
    d.cf_fac_off = put(H.factor_words.data(), H.factor_words.size() * 4, 64);
    d.cf_bs_off = put(P.bytesets.data(), P.bytesets.size() * 4, 32);
    d.cf_bytes = (uint32_t)cf.size();
    d.cf_resident = d.cf_bytes <= kConfirmTableBudget ? 1u : 0u;
    const uint8_t* dcf = nullptr; if ((rc = upload(rs.get(), cf, &dcf, 16))) return rc;
    d.cf_image = dcf;
  }
  d.n_factors = (uint32_t)P.factors.size();
  if ((rc = upload(rs.get(), H.factor_words, &d.factors, 16))) return rc;
  if ((rc = upload(rs.get(), P.bytesets, &d.bytesets, 8))) return rc;
  if ((rc = upload(rs.get(), P.always_rules, &d.always_rules))) return rc;
  d.n_always = (uint32_t)P.always_rules.size();
  if ((rc = upload(rs.get(), prog, &d.prog))) return rc;
  if ((rc = upload(rs.get(), prog_off, &d.rule_prog_off))) return rc;
  if ((rc = upload(rs.get(), sets, &d.sets, 8))) return rc;
  if ((rc = upload(rs.get(), ranges, &d.set_ranges, 8))) return rc;
  if ((rc = upload(rs.get(), first, &d.rule_first, 8))) return rc;
  if ((rc = upload(rs.get(), H.alpha, &d.rule_alpha, 8))) return rc;
  { const uint64_t* bw = nullptr; if ((rc = upload(rs.get(), H.bit_words, &bw, 8))) return rc; d.bit_words = reinterpret_cast<const unsigned long long*>(bw); }
  if ((rc = upload(rs.get(), H.bit_off, &d.bit_off))) return rc;
  { const uint64_t* fs = nullptr; if ((rc = upload(rs.get(), H.factor_skip, &fs, 8))) return rc; d.factor_skip = reinterpret_cast<const unsigned long long*>(fs); }
  d.rule_policy = nullptr; d.rule_action = nullptr;
  {
    // the span resolver's tie-break: rank of every rule in (category, rule) order
    std::vector<uint32_t> order(n_rules), rank(n_rules);
    for (uint32_t i = 0; i < n_rules; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return rs->category[a] < rs->category[b]; });
    for (uint32_t i = 0; i < n_rules; i++) rank[order[i]] = i;
    if ((rc = upload(rs.get(), rs->category, &rs->work.rule_category))) return rc;
    if ((rc = upload(rs.get(), rank, &rs->work.rule_rank))) return rc;
  }
  d.n_rules = n_rules; d.rw = (n_rules + 31) / 32; if (d.rw == 0) d.rw = 1;
  d.max_prog_len = 0; for (uint32_t i = 0; i < n_rules; i++) d.max_prog_len = std::max(d.max_prog_len, prog_off[i + 1] - prog_off[i]);
  prepare_kernels();
  *out = rs.release();
  return CG_OK;
}

void cg_ruleset_destroy(cg_ruleset* rs) { std::lock_guard<std::mutex> lk(g_mu); if (rs) { if (G.ready) cudaDeviceSynchronize(); delete rs; } }

int cg_ruleset_get_info(const cg_ruleset* rs, cg_ruleset_info* o) {
  if (!rs || !o) return fail(CG_ERR_INVALID_ARG, "null argument");
  memset(o, 0, sizeof *o);
  o->n_rules = (uint32_t)rs->host.rules.size();
  for (auto& r : rs->host.rules) if (r.status == RULE_OK) o->n_ok++;
  const Prefilter& P = rs->host.pf;
  o->n_always_candidate = (uint32_t)P.always_rules.size(); o->n_sets = rs->n_sets;
  o->stride = (uint32_t)P.stride; o->gram_keys = (uint32_t)P.keys.size(); o->gram_entries = (uint32_t)P.entries.size();
  o->factor_len = P.min_factor_len | (P.max_factor_len << 8); o->n_factors = (uint32_t)P.factors.size();
  o->image_bytes = rs->dev.image_bytes; o->bitmap_bytes = rs->host.bm_bytes; o->program_words = rs->program_words;
  o->n_triggers = (uint32_t)P.trig_bytes.size(); o->tables_resident = rs->host.tables_resident ? 1u : 0u;
  return CG_OK;
}

namespace {
int scan_batch_host(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint64_t* out_words,
                    cg_hit* out_hits, uint32_t hits_cap, uint32_t* out_nhits, const uint8_t* views);
}  // namespace

int cg_scan_batch(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint64_t* out_words,
                  cg_hit* out_hits, uint32_t hits_cap, uint32_t* out_nhits) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc;
  // large words-only batches: chunked, copies overlapped with the kernels (the hit list needs the per-batch slot tables)
  if (!out_hits && out_words && n >= (1u << 16) && G.ready && rs && bytes && offsets) {
    rc = scan_host_chunked(rs, bytes, offsets, n, out_words);
    if (rc < 0) return rc;
    if (rc == 0) {
      if (out_nhits) { uint64_t nh = 0; for (uint32_t i = 0; i < n; i++) if (out_words[i] >> 63) nh += (out_words[i] >> 32) & 0x7fffffffu; *out_nhits = (uint32_t)nh; G.stats.hits += nh; }
      return CG_OK;
    }
    // rc == 1: a queue overflowed in some piece; capacities have been raised -- run the batch in one piece below
  }
  return scan_batch_host(rs, bytes, offsets, n, out_words, out_hits, hits_cap, out_nhits, nullptr);
}

namespace {
// the one-piece path of cg_scan_batch, and cg_scan_batch_views.  The hit list on the device (as cg_scan_hits_batch_device
// builds it): counts and their scan behind the step, the total to the host, then the first min(total, hits_cap) pairs into a
// staging buffer and back
int scan_batch_host(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint64_t* out_words,
                    cg_hit* out_hits, uint32_t hits_cap, uint32_t* out_nhits, const uint8_t* views) {
  const bool want_hits = out_hits || out_nhits;
  cudaStream_t st = G.stream;
  InOrder turn(rs ? &rs->order : nullptr, st);
  if (turn.rc) return turn.rc;
  uint64_t total = 0;
  int rc = scan_host(rs, bytes, offsets, n, want_hits ? kStepPolicy : kStepWords, [&](const ScanWork& w) {
    if (!want_hits || !n) return CG_OK;
    count_launches(launch_hit_count(w, G.d_words.get(), n, G.sm_count, st));
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&total, w.out_off + n, 8, cudaMemcpyDeviceToHost, st));
    return CG_OK;
  }, views);
  if (rc) return rc;
  const uint32_t nh = (uint32_t)total, k = out_hits && !(total >> 32) ? std::min(nh, hits_cap) : 0u;
  if (out_words && n) CU(cudaMemcpyAsync(out_words, G.d_words.get(), (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  if (k) {
    if ((rc = G.d_hits.grow(2 * (size_t)k + 1))) return rc;      // [count][pairs]
    count_launches(launch_hit_emit(rs->dev, rs->work, n, G.d_hits.get() + 1, k, G.d_hits.get(), G.sm_count, st));
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(out_hits, G.d_hits.get() + 1, (size_t)k * sizeof(cg_hit), cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  if (total >> 32) { if (out_nhits) *out_nhits = 0xffffffffu; return fail(CG_ERR_TOO_LARGE, "2^32 hits or more in one batch"); }
  if (out_nhits) *out_nhits = nh;
  G.stats.hits += nh;
  if (out_hits && nh > hits_cap) return fail(CG_ERR_CAPACITY, "out_hits too small");
  return CG_OK;
}

// the host-buffer *_views calls' ids, checked before anything is staged or written
int check_views(const cg_ruleset* rs, const uint8_t* views, uint32_t n) {
  if (int rc = require_ready()) return rc;
  if (!rs || (n && !views)) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!rs->n_views) return fail(CG_ERR_INVALID_ARG, "cg_ruleset_set_views has not been called");
  for (uint32_t i = 0; i < n; i++) if (views[i] >= rs->n_views) return fail(CG_ERR_INVALID_ARG, "view id " + std::to_string(views[i]) + " of message " + std::to_string(i) + " >= n_views");
  return CG_OK;
}
}  // namespace

int cg_scan_batch_views(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, const uint8_t* views, uint32_t n, uint64_t* out_words,
                        cg_hit* out_hits, uint32_t hits_cap, uint32_t* out_nhits) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = check_views(rs, views, n)) return rc;
  return scan_batch_host(rs, bytes, offsets, n, out_words, out_hits, hits_cap, out_nhits, views);
}

namespace {
// -> CG_OK, an error, or 1 = take the general path (long message, large rule set, a queue overflowed)
int scan_one_fast(cg_ruleset* rs, const uint8_t* bytes, uint32_t len, uint64_t* out_word, uint32_t* out_rules, uint32_t rules_cap, uint32_t* out_nrules) {
  if (!G.ready || !rs || (len && !bytes) || len > kOneBytes || rs->dev.rw > kOneRw - 2 || G.profiling) return 1;
  Staging& s = rs->one.io;
  const uint32_t off[2] = {0, len};
  const int rc = blocking_call(rs, kStepWords, 1, 0, rs->one.graphs, {}, s, [&](uint8_t* h) { return stage_texts(h, 256, bytes, off, 1); }, [&] {
        const uint32_t* d_off = reinterpret_cast<const uint32_t*>(s.d.get());
        uint32_t* d_out = reinterpret_cast<uint32_t*>(s.d.get() + kOneIn); uint64_t* d_word = reinterpret_cast<uint64_t*>(s.d.get() + kOneIn + kOneOut - 8);   // (the word lands behind the hit row, then is packed to the front)
        const int r = run_scan_device(rs, s.d.get(), d_off, 1, d_word, kStepWords, G.stream);
        if (r == CG_OK) count_launches(launch_pack_one(rs->dev, rs->work, d_word, d_out, kOneRw - 2, G.stream));
        return r;
      }, s, kOneIn, (kOneHitRow + rs->dev.rw) * 4, kOneIn + 4 * kOneCounters);
  if (rc) return rc;                                             // 1: a queue overflowed, the general path retries with larger scratch
  const uint32_t* ho = reinterpret_cast<const uint32_t*>(s.h.get() + kOneIn);
  const uint32_t* hc = ho + kOneCounters;
  count_step(1, len, hc);
  if (out_word) *out_word = (uint64_t)ho[0] | ((uint64_t)ho[1] << 32);
  const uint32_t nh = append_hit_row(ho + kOneHitRow, rs->dev.rw, 0, out_rules ? rules_cap : 0, [&](uint32_t i, uint32_t r) { out_rules[i] = r; });
  if (out_nrules) *out_nrules = nh;
  G.stats.hits += nh;
  if (out_rules && nh > rules_cap) return fail(CG_ERR_CAPACITY, "out_rules too small");
  return CG_OK;
}
}  // namespace

int cg_scan_one(cg_ruleset* rs, const uint8_t* bytes, uint32_t len, uint64_t* out_word, uint32_t* out_rules, uint32_t rules_cap, uint32_t* out_nrules) {
  { std::lock_guard<std::mutex> lk(g_mu); const int frc = scan_one_fast(rs, bytes, len, out_word, out_rules, rules_cap, out_nrules); if (frc != 1) return frc; }
  uint32_t off[2] = {0, len};
  std::vector<cg_hit> hits(rules_cap ? rules_cap : 1);
  uint32_t nh = 0; uint64_t word = 0;
  int rc = cg_scan_batch(rs, bytes, off, 1, &word, out_rules ? hits.data() : nullptr, rules_cap, &nh);
  if (out_word) *out_word = word;
  if (out_nrules) *out_nrules = nh;
  if (out_rules) for (uint32_t i = 0; i < nh && i < rules_cap; i++) out_rules[i] = hits[i].rule;
  return rc;
}

namespace {
// the span resolver behind a host-buffer span step, its sizes to the host (sizes[0] resolved spans, or redacting {output
// bytes, resolved spans}).  Resolved spans land in G.d_spans; redacting, G.d_redact_meta holds [sizes, 4 words][out offsets,
// n + 1][digests, 16-byte aligned, room for every raw span: *d_digests].
int resolve_staged(const ScanWork& w, uint32_t n, bool redact, uint64_t sizes[2], uint32_t** d_digests) {
  const size_t dig_at = ((size_t)n + 1 + 4 + 3) & ~(size_t)3;
  int rc;
  if ((rc = G.d_spans.grow((size_t)w.span_cap))) return rc;
  if ((rc = G.d_redact_meta.grow(dig_at + (redact ? (size_t)w.span_cap * 8 : 0)))) return rc;
  *d_digests = G.d_redact_meta.get() + dig_at;
  const SpanOutputs o{reinterpret_cast<uint32_t*>(G.d_spans.get()), w.span_cap, G.d_redact_meta.get() + 4, ~0ull, G.d_redact_meta.get(), redact};
  count_launches(launch_span_resolve(w, G.d_off32.get(), n, o, G.sm_count, G.stream));
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(sizes, G.d_redact_meta.get(), redact ? 16 : 4, cudaMemcpyDeviceToHost, G.stream));
  return CG_OK;
}

int find_matches_host(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans,
                      const uint8_t* views) {
  InOrder turn(rs ? &rs->order : nullptr, G.stream);
  if (turn.rc) return turn.rc;
  uint64_t sizes[2] = {0, 0}; uint32_t* d_dig = nullptr;
  int rc = scan_host(rs, bytes, offsets, n, kStepSpans, [&](const ScanWork& w) { return resolve_staged(w, n, false, sizes, &d_dig); }, views);
  if (rc) return rc;
  const uint32_t outn = (uint32_t)sizes[0], k = std::min(outn, spans_cap);
  G.stats.spans += outn;
  if (out_spans && k) { CU(cudaMemcpyAsync(out_spans, G.d_spans.get(), (size_t)k * sizeof(cg_span), cudaMemcpyDeviceToHost, G.stream)); CU(cudaStreamSynchronize(G.stream)); }
  if (out_nspans) *out_nspans = outn;
  if (out_spans && outn > spans_cap) return fail(CG_ERR_CAPACITY, "out_spans too small");
  return CG_OK;
}
}  // namespace

int cg_find_matches_batch(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans) {
  std::lock_guard<std::mutex> lk(g_mu);
  return find_matches_host(rs, bytes, offsets, n, out_spans, spans_cap, out_nspans, nullptr);
}

int cg_find_matches_batch_views(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, const uint8_t* views, uint32_t n, cg_span* out_spans,
                                uint32_t spans_cap, uint32_t* out_nspans) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = check_views(rs, views, n)) return rc;
  return find_matches_host(rs, bytes, offsets, n, out_spans, spans_cap, out_nspans, views);
}

int cg_ruleset_set_policy(cg_ruleset* rs, const uint32_t* rule_policy, const uint8_t* rule_action, uint32_t n_rules) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!rs || !rule_policy || !rule_action || n_rules != rs->dev.n_rules) return fail(CG_ERR_INVALID_ARG, "one (policy, action) pair per rule of the set");
  std::vector<uint32_t> pol(rule_policy, rule_policy + n_rules), act(n_rules);
  for (uint32_t i = 0; i < n_rules; i++) {
    if (rule_action[i] > 2) return fail(CG_ERR_INVALID_ARG, "action must be 0 (allow), 1 (audit) or 2 (deny)");
    if (i && pol[i] < pol[i - 1]) return fail(CG_ERR_INVALID_ARG, "rules must be stored policy by policy (policy index non-decreasing)");
    act[i] = rule_action[i];
  }
  CU(cudaStreamSynchronize(G.stream));
  DevBuf<uint8_t> d_pol, d_act; const uint32_t *p, *a; int rc;     // (they replace the old tables once both are there)
  if ((rc = upload(rs, pol, &p, 4, &d_pol)) || (rc = upload(rs, act, &a, 4, &d_act))) return rc;
  rs->rule_policy = std::move(d_pol); rs->rule_action = std::move(d_act);
  rs->dev.rule_policy = p; rs->dev.rule_action = a;
  rs->scratch_gen++;                                        // DevRuleset is captured by value
  return CG_OK;
}

int cg_ruleset_set_views(cg_ruleset* rs, const uint32_t* rows, uint32_t n_views) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!rs || !rows) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (n_views < 1 || n_views > 256) return fail(CG_ERR_INVALID_ARG, "n_views must be 1 .. 256");
  const uint32_t n_rules = rs->dev.n_rules, rw = rs->dev.rw;
  for (uint32_t v = 0; v < n_views; v++)
    for (uint32_t k = 0; k < rw; k++) {
      const uint32_t valid = n_rules >= 32 * (k + 1) ? ~0u : n_rules > 32 * k ? (1u << (n_rules - 32 * k)) - 1u : 0u;     // bits of rules < n_rules
      if (rows[(size_t)v * rw + k] & ~valid) return fail(CG_ERR_INVALID_ARG, "view " + std::to_string(v) + " has a bit at or past n_rules");
    }
  CU(cudaStreamSynchronize(G.stream));
  rs->view_rows.reset(); rs->n_views = 0;
  if (int rc = rs->view_rows.alloc((size_t)n_views * rw)) return rc;
  CU(cudaMemcpy(rs->view_rows.get(), rows, (size_t)n_views * rw * 4, cudaMemcpyHostToDevice));
  rs->n_views = n_views;
  rs->scratch_gen++;
  return CG_OK;
}

namespace {
int verdict_host(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint32_t* out_verdicts, const uint8_t* views) {
  cudaStream_t st = G.stream;
  InOrder turn(&rs->order, st);
  if (turn.rc) return turn.rc;
  int rc = scan_host(rs, bytes, offsets, n, kStepWords, [&](const ScanWork& w) {
    if (!n) return CG_OK;
    int r;
    if ((r = G.d_verdicts.grow((size_t)n))) return r;
    CU(cudaMemsetAsync(G.d_verdicts.get(), 0, (size_t)n * 4, st));  // (verdict_kernel writes the messages that hit)
    count_launches(launch_verdicts(rs->dev, w, G.d_verdicts.get(), n, G.sm_count, st));
    CU(cudaGetLastError());
    return CG_OK;
  }, views);
  if (rc || !n) return rc;
  CU(cudaMemcpyAsync(out_verdicts, G.d_verdicts.get(), (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}
}  // namespace

int cg_policy_verdict_batch(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint32_t* out_verdicts) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!rs || !out_verdicts) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!rs->dev.rule_policy) return fail(CG_ERR_INVALID_ARG, "cg_ruleset_set_policy has not been called");
  return verdict_host(rs, bytes, offsets, n, out_verdicts, nullptr);
}

int cg_policy_verdict_batch_views(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, const uint8_t* views, uint32_t n, uint32_t* out_verdicts) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = check_views(rs, views, n)) return rc;
  if (!out_verdicts) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!rs->dev.rule_policy) return fail(CG_ERR_INVALID_ARG, "cg_ruleset_set_policy has not been called");
  return verdict_host(rs, bytes, offsets, n, out_verdicts, views);
}

namespace {
int redact_host(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint8_t* out_bytes, uint64_t out_cap,
                uint64_t* out_need, uint32_t* out_offsets, cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans, uint8_t* out_digests32,
                const uint8_t* views) {
  if (!out_offsets || (n && (!bytes || !offsets))) return fail(CG_ERR_INVALID_ARG, "null argument");
  InOrder turn(rs ? &rs->order : nullptr, G.stream);
  if (turn.rc) return turn.rc;
  uint64_t sizes[2] = {0, 0}; uint32_t* d_dig = nullptr;
  int rc = scan_host(rs, bytes, offsets, n, kStepSpans, [&](const ScanWork& w) { return resolve_staged(w, n, true, sizes, &d_dig); }, views);
  if (rc) return rc;                                        // (input bytes / offsets stay in G.d_bytes / G.d_off32)
  const uint64_t pos = sizes[0]; const uint32_t ns = (uint32_t)sizes[1];
  G.stats.spans += ns;
  if (out_need) *out_need = pos;
  if (out_nspans) *out_nspans = ns;
  const bool too_large = pos >> 32, fits = !too_large && !(out_spans && ns > spans_cap) && pos <= out_cap && out_bytes;
  cudaStream_t st = G.stream;
  if (fits && (rc = G.d_redact_out.grow((size_t)pos + 64))) return rc;
  CU(cudaMemcpyAsync(out_offsets, G.d_redact_meta.get() + 4, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost, st));
  if (fits) {
    count_launches(enqueue_redact_tail(rs->work, G.d_bytes.get(), G.d_off32.get(), G.d_redact_meta.get() + 4, d_dig, G.d_redact_out.get(), n, st));
    G.stats.sha256_items += ns;
    CU(cudaGetLastError());
    if (pos) CU(cudaMemcpyAsync(out_bytes, G.d_redact_out.get(), (size_t)pos, cudaMemcpyDeviceToHost, st));
    if (ns && out_spans) CU(cudaMemcpyAsync(out_spans, G.d_spans.get(), (size_t)ns * sizeof(cg_span), cudaMemcpyDeviceToHost, st));
    if (ns && out_digests32) CU(cudaMemcpyAsync(out_digests32, d_dig, (size_t)ns * 32, cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  if (too_large) return fail(CG_ERR_TOO_LARGE, "redacted batch exceeds 4 GiB");
  if (!fits) return fail(CG_ERR_CAPACITY, "output buffer too small (see *out_need / *out_nspans)");
  return CG_OK;
}
}  // namespace

int cg_redact_batch(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint8_t* out_bytes, uint64_t out_cap,
                    uint64_t* out_need, uint32_t* out_offsets, cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans, uint8_t* out_digests32) {
  std::lock_guard<std::mutex> lk(g_mu);
  return redact_host(rs, bytes, offsets, n, out_bytes, out_cap, out_need, out_offsets, out_spans, spans_cap, out_nspans, out_digests32, nullptr);
}

int cg_redact_batch_views(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, const uint8_t* views, uint32_t n, uint8_t* out_bytes,
                          uint64_t out_cap, uint64_t* out_need, uint32_t* out_offsets, cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans,
                          uint8_t* out_digests32) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = check_views(rs, views, n)) return rc;
  return redact_host(rs, bytes, offsets, n, out_bytes, out_cap, out_need, out_offsets, out_spans, spans_cap, out_nspans, out_digests32, views);
}

namespace {
struct OneSpanOut { cg_span* spans; uint32_t spans_cap; uint32_t* nspans; uint8_t* bytes; uint64_t out_cap; uint64_t* need; uint8_t* digests; uint32_t* offsets; };

// cg_find_matches_one / cg_redact_one (n = 1) and cg_find_matches_few / cg_redact_few on the staging block: one H2D copy,
// one graph (span-mode step over the n staged strings, one-block resolver, digests and splice when redacting, pack), one D2H
// copy of the header plus a window sized from the text length, one synchronise; a second copy and synchronise only for a
// packed result longer than the window.  Outputs, statuses and statistics are those of the batch call.  -> CG_OK, an error,
// or 1 = take the batch call (an argument the batch call rejects, no device, more than kFewMsgs strings or max_bytes of
// text, profiling, a queue overflowed, or a result longer than the packed region)
int span_few_fast(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint32_t max_bytes, bool redact, const OneSpanOut& out) {
  if (!G.ready || !rs || G.profiling || n > kFewMsgs || (n && (!bytes || !offsets)) || (redact && !out.offsets)) return 1;
  for (uint32_t i = 0; i < n; i++) if (offsets[i + 1] < offsets[i]) return 1;
  const uint32_t first = n ? offsets[0] : 0, len = n ? offsets[n] - first : 0;
  if (len > max_bytes) return 1;
  Staging& in = rs->span.in; Staging& pk = rs->span.pack;
  // the resolver's capacities on this path: every resolved span (and, redacting, its digest and the output) must fit the block
  const uint32_t at = pack_spans_at(n), room = kOnePack - at;
  // the window: the header with the offsets, 1 KB and len / 2 bytes (find-matches) or 2 x len bytes (redaction) of the packed result
  const uint32_t window = std::min<uint32_t>(kOnePack, at + 1024 + (redact ? 2 * len : len / 2));
  const int rc = blocking_call(rs, kStepSpans, n, 0, rs->span.graphs, {redact, n}, in, [&](uint8_t* h) { return stage_texts(h, kFewTextAt, bytes, offsets, n); }, [&] {
        const ScanWork& w = rs->work;
        const uint32_t* d_off = reinterpret_cast<const uint32_t*>(in.d.get());
        uint32_t* d_pack = reinterpret_cast<uint32_t*>(pk.d.get()); uint32_t* d_dig = reinterpret_cast<uint32_t*>(pk.d.get() + kOnePack); uint8_t* d_out = pk.d.get() + 2 * kOnePack;
        const int r = run_scan_device(rs, in.d.get(), d_off, n, w.words, kStepSpans, G.stream);
        if (r != CG_OK) return r;
        const SpanOutputs so{d_pack + at / 4, room / (redact ? 56u : 24u), d_pack + kPackOffsets, redact ? (uint64_t)room : 0ull, d_pack + kPackSizes, redact};
        int k = launch_span_resolve_few(w, d_off, n, so, G.stream);
        if (redact) k += enqueue_redact_tail(w, in.d.get(), d_off, d_pack + kPackOffsets, d_dig, d_out, n, G.stream);
        k += launch_span_pack_few(w, d_dig, d_out, d_pack, kOnePack, n, redact, G.stream);
        count_launches(k);
        CU(cudaGetLastError());
        return CG_OK;
      }, pk, 0, window, 4 * kPackCounters);
  if (rc) return rc;                                             // 1: a queue overflowed, the batch call retries with larger scratch
  const uint32_t* hp = reinterpret_cast<const uint32_t*>(pk.h.get());
  const uint32_t* hc = hp + kPackCounters;
  const uint32_t packed = hp[0];
  if (!packed) return 1;                                         // longer than the packed region: the batch call has room
  if (packed > window) {
    CU(cudaMemcpyAsync(pk.h.get() + window, pk.d.get() + window, packed - window, cudaMemcpyDeviceToHost, G.stream));
    CU(cudaStreamSynchronize(G.stream));
  }
  count_step(n, len, hc);
  const uint8_t* body = pk.h.get() + at;
  if (!redact) {
    const uint32_t ns = hp[kPackSizes];
    G.stats.spans += ns;
    const uint32_t k = std::min(ns, out.spans_cap);
    if (out.spans && k) memcpy(out.spans, body, (size_t)k * sizeof(cg_span));
    if (out.nspans) *out.nspans = ns;
    if (out.spans && ns > out.spans_cap) return fail(CG_ERR_CAPACITY, "out_spans too small");
    return CG_OK;
  }
  uint64_t sizes[2];
  memcpy(sizes, hp + kPackSizes, sizeof sizes);
  const uint64_t need = sizes[0]; const uint32_t ns = (uint32_t)sizes[1];
  G.stats.spans += ns;
  if (out.need) *out.need = need;
  if (out.nspans) *out.nspans = ns;
  memcpy(out.offsets, hp + kPackOffsets, ((size_t)n + 1) * 4);
  if (need >> 32) return fail(CG_ERR_TOO_LARGE, "redacted batch exceeds 4 GiB");
  if ((out.spans && ns > out.spans_cap) || need > out.out_cap || !out.bytes) return fail(CG_ERR_CAPACITY, "output buffer too small (see *out_need / *out_nspans)");
  G.stats.sha256_items += ns;
  if (need) memcpy(out.bytes, body + (size_t)ns * (sizeof(cg_span) + 32), (size_t)need);
  if (ns && out.spans) memcpy(out.spans, body, (size_t)ns * sizeof(cg_span));
  if (ns && out.digests) memcpy(out.digests, body + (size_t)ns * sizeof(cg_span), (size_t)ns * 32);
  return CG_OK;
}
}  // namespace

int cg_find_matches_one(cg_ruleset* rs, const uint8_t* bytes, uint32_t len, cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans) {
  const uint32_t off[2] = {0, len};
  { std::lock_guard<std::mutex> lk(g_mu); const int frc = span_few_fast(rs, bytes, off, 1, kOneBytes, false, OneSpanOut{out_spans, spans_cap, out_nspans, nullptr, 0, nullptr, nullptr, nullptr}); if (frc != 1) return frc; }
  return cg_find_matches_batch(rs, bytes, off, 1, out_spans, spans_cap, out_nspans);
}

int cg_redact_one(cg_ruleset* rs, const uint8_t* bytes, uint32_t len, uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_need,
                  cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans, uint8_t* out_digests32) {
  const uint32_t off[2] = {0, len};
  uint32_t out_off[2] = {0, 0};
  { std::lock_guard<std::mutex> lk(g_mu); const int frc = span_few_fast(rs, bytes, off, 1, kOneBytes, true, OneSpanOut{out_spans, spans_cap, out_nspans, out_bytes, out_cap, out_need, out_digests32, out_off}); if (frc != 1) return frc; }
  return cg_redact_batch(rs, bytes, off, 1, out_bytes, out_cap, out_need, out_off, out_spans, spans_cap, out_nspans, out_digests32);
}

int cg_find_matches_few(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans) {
  { std::lock_guard<std::mutex> lk(g_mu); const int frc = span_few_fast(rs, bytes, offsets, n, kFewBytes, false, OneSpanOut{out_spans, spans_cap, out_nspans, nullptr, 0, nullptr, nullptr, nullptr}); if (frc != 1) return frc; }
  return cg_find_matches_batch(rs, bytes, offsets, n, out_spans, spans_cap, out_nspans);
}

int cg_redact_few(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_need,
                  uint32_t* out_offsets, cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans, uint8_t* out_digests32) {
  { std::lock_guard<std::mutex> lk(g_mu); const int frc = span_few_fast(rs, bytes, offsets, n, kFewBytes, true, OneSpanOut{out_spans, spans_cap, out_nspans, out_bytes, out_cap, out_need, out_digests32, out_offsets}); if (frc != 1) return frc; }
  return cg_redact_batch(rs, bytes, offsets, n, out_bytes, out_cap, out_need, out_offsets, out_spans, spans_cap, out_nspans, out_digests32);
}

int cg_scan_batch_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_words, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = device_batch_args(rs, d_bytes, d_offsets)) return rc;
  if (!d_out_words) return fail(CG_ERR_INVALID_ARG, "null argument");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream;
  if (!n) return CG_OK;
  return scan_device(rs, d_bytes, d_offsets, n, (uint64_t*)d_out_words, kStepWords, st, [](const ScanWork&) { return 0; }, !G.profiling);
}

int cg_scan_join(cg_ruleset* rs, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!rs) return fail(CG_ERR_INVALID_ARG, "null argument");
  CU(cudaStreamSynchronize(stream ? (cudaStream_t)stream : G.stream));
  poll_mirrors(rs, true);
  const uint32_t flags = rs->sticky_flags, status = rs->sticky_status; rs->sticky_flags = rs->sticky_status = 0;
  if (flags & (ERR_VM_STACK | ERR_VM_LIST)) return fail(CG_ERR_TOO_LARGE, std::string(kVmOverflow) + " (result words of that batch are all ones)");
  if (status & (1u << kResolveTooLarge)) return fail(CG_ERR_TOO_LARGE, "redacted batch exceeds 4 GiB, or a batch has 2^32 - 1 hits or more");
  if (flags) return fail(CG_ERR_CAPACITY, "a candidate queue overflowed: the result words (or sizes) of that batch are all ones; the scratch has been grown, scan the batch again");
  if (status & (1u << kResolveCapacity)) return fail(CG_ERR_CAPACITY, "output buffer too small: the sizes a batch needs are in its d_out_sizes / d_out_nspans / d_out_nhits");
  return CG_OK;
}

namespace {
// the device-resident *_views calls' table: the rule set's rows and the caller's ids in HBM (which the host cannot check: an id
// >= n_views selects the empty view)
int device_views(const cg_ruleset* rs, const void* d_views, ViewTable* vt) {
  if (!rs->n_views) return fail(CG_ERR_INVALID_ARG, "cg_ruleset_set_views has not been called");
  if (!d_views) return fail(CG_ERR_INVALID_ARG, "null argument");
  *vt = ViewTable{rs->view_rows.get(), (const uint8_t*)d_views, rs->n_views};
  return CG_OK;
}

int find_matches_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_spans, uint32_t spans_cap,
                        void* d_out_nspans, void* stream, const ViewTable* views) {
  if (int rc = device_batch_args(rs, d_bytes, d_offsets)) return rc;
  if ((spans_cap && !d_out_spans) || !d_out_nspans) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (((uintptr_t)d_offsets | (uintptr_t)d_out_spans | (uintptr_t)d_out_nspans) & 3u) return fail(CG_ERR_INVALID_ARG, "d_offsets, d_out_spans and d_out_nspans must be 4-byte aligned");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream;
  const SpanOutputs o{(uint32_t*)d_out_spans, d_out_spans ? spans_cap : 0u, nullptr, 0, d_out_nspans, false};
  return scan_device(rs, d_bytes, d_offsets, n, nullptr, kStepSpans, st, [&](const ScanWork& w) {
    return launch_span_resolve(w, (const uint32_t*)d_offsets, n, o, G.sm_count, st);
  }, false, views);
}

int redact_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_bytes, uint64_t out_cap,
                  void* d_out_offsets, void* d_out_spans, uint32_t spans_cap, void* d_out_digests32, void* d_out_sizes, void* stream, const ViewTable* views) {
  if (int rc = device_batch_args(rs, d_bytes, d_offsets)) return rc;
  if (!d_out_offsets || !d_out_sizes || (out_cap && !d_out_bytes) || (spans_cap && (!d_out_spans || !d_out_digests32))) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (((uintptr_t)d_offsets | (uintptr_t)d_out_offsets | (uintptr_t)d_out_spans) & 3u) return fail(CG_ERR_INVALID_ARG, "d_offsets, d_out_offsets and d_out_spans must be 4-byte aligned");
  if ((uintptr_t)d_out_sizes & 7u) return fail(CG_ERR_INVALID_ARG, "d_out_sizes must be 8-byte aligned");
  if ((uintptr_t)d_out_digests32 & 15u) return fail(CG_ERR_INVALID_ARG, "d_out_digests32 must be 16-byte aligned");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream;
  const SpanOutputs o{(uint32_t*)d_out_spans, spans_cap, (uint32_t*)d_out_offsets, d_out_bytes ? out_cap : 0ull, d_out_sizes, true};
  return scan_device(rs, d_bytes, d_offsets, n, nullptr, kStepSpans, st, [&](const ScanWork& w) {
    const int k = launch_span_resolve(w, (const uint32_t*)d_offsets, n, o, G.sm_count, st);
    return k + enqueue_redact_tail(w, (const uint8_t*)d_bytes, (const uint32_t*)d_offsets, o.out_offsets, (uint32_t*)d_out_digests32,
                                   (uint8_t*)d_out_bytes, n, st);
  }, false, views);
}

// (with views, d_out_nhits = NULL, d_out_hits = NULL and hits_cap = 0: the result words alone, as cg_scan_batch_device)
int scan_hits_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_words, void* d_out_hits,
                     uint32_t hits_cap, void* d_out_nhits, void* stream, const ViewTable* views) {
  if (int rc = device_batch_args(rs, d_bytes, d_offsets)) return rc;
  const bool words_only = views && !d_out_nhits && !d_out_hits && !hits_cap;
  if (!d_out_words || (!d_out_nhits && !words_only) || (hits_cap && !d_out_hits)) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (((uintptr_t)d_offsets | (uintptr_t)d_out_hits | (uintptr_t)d_out_nhits) & 3u) return fail(CG_ERR_INVALID_ARG, "d_offsets, d_out_hits and d_out_nhits must be 4-byte aligned");
  if ((uintptr_t)d_out_words & 7u) return fail(CG_ERR_INVALID_ARG, "d_out_words must be 8-byte aligned");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream;
  uint64_t* words = (uint64_t*)d_out_words;
  if (words_only) return n ? scan_device(rs, d_bytes, d_offsets, n, words, kStepWords, st, [](const ScanWork&) { return 0; }, false, views) : CG_OK;
  if (!n) { CU(cudaMemsetAsync(d_out_nhits, 0, 4, st)); return CG_OK; }
  return scan_device(rs, d_bytes, d_offsets, n, words, kStepPolicy, st, [&](const ScanWork& w) {
    const int k = launch_hit_count(w, words, n, G.sm_count, st);
    return k + launch_hit_emit(rs->dev, w, n, (uint32_t*)d_out_hits, d_out_hits ? hits_cap : 0u, (uint32_t*)d_out_nhits, G.sm_count, st);
  }, false, views);
}

int verdict_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_verdicts, void* stream, const ViewTable* views) {
  if (int rc = device_batch_args(rs, d_bytes, d_offsets)) return rc;
  if (!d_out_verdicts) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!rs->dev.rule_policy) return fail(CG_ERR_INVALID_ARG, "cg_ruleset_set_policy has not been called");
  if (((uintptr_t)d_offsets | (uintptr_t)d_out_verdicts) & 3u) return fail(CG_ERR_INVALID_ARG, "d_offsets and d_out_verdicts must be 4-byte aligned");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream;
  if (!n) return CG_OK;
  uint32_t* verdicts = (uint32_t*)d_out_verdicts;
  CU(cudaMemsetAsync(verdicts, 0, (size_t)n * 4, st));       // (verdict_kernel writes the messages that hit)
  return scan_device(rs, d_bytes, d_offsets, n, nullptr, kStepPolicy, st, [&](const ScanWork& w) { return launch_verdicts(rs->dev, w, verdicts, n, G.sm_count, st); },
                     false, views);
}

// the checks of a device-resident *_views call, then its table
int device_views_args(const cg_ruleset* rs, const void* d_bytes, const void* d_offsets, const void* d_views, ViewTable* vt) {
  if (int rc = device_batch_args(rs, d_bytes, d_offsets)) return rc;
  return device_views(rs, d_views, vt);
}
}  // namespace

int cg_find_matches_batch_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_spans, uint32_t spans_cap,
                                 void* d_out_nspans, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  return find_matches_device(rs, d_bytes, d_offsets, n, d_out_spans, spans_cap, d_out_nspans, stream, nullptr);
}
int cg_find_matches_batch_device_views(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, const void* d_views, uint32_t n, void* d_out_spans,
                                       uint32_t spans_cap, void* d_out_nspans, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  ViewTable vt;
  if (int rc = device_views_args(rs, d_bytes, d_offsets, d_views, &vt)) return rc;
  return find_matches_device(rs, d_bytes, d_offsets, n, d_out_spans, spans_cap, d_out_nspans, stream, &vt);
}

int cg_redact_batch_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_bytes, uint64_t out_cap,
                           void* d_out_offsets, void* d_out_spans, uint32_t spans_cap, void* d_out_digests32, void* d_out_sizes, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  return redact_device(rs, d_bytes, d_offsets, n, d_out_bytes, out_cap, d_out_offsets, d_out_spans, spans_cap, d_out_digests32, d_out_sizes, stream, nullptr);
}
int cg_redact_batch_device_views(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, const void* d_views, uint32_t n, void* d_out_bytes,
                                 uint64_t out_cap, void* d_out_offsets, void* d_out_spans, uint32_t spans_cap, void* d_out_digests32, void* d_out_sizes,
                                 void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  ViewTable vt;
  if (int rc = device_views_args(rs, d_bytes, d_offsets, d_views, &vt)) return rc;
  return redact_device(rs, d_bytes, d_offsets, n, d_out_bytes, out_cap, d_out_offsets, d_out_spans, spans_cap, d_out_digests32, d_out_sizes, stream, &vt);
}

int cg_scan_hits_batch_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_words, void* d_out_hits,
                              uint32_t hits_cap, void* d_out_nhits, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  return scan_hits_device(rs, d_bytes, d_offsets, n, d_out_words, d_out_hits, hits_cap, d_out_nhits, stream, nullptr);
}
int cg_scan_hits_batch_device_views(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, const void* d_views, uint32_t n, void* d_out_words,
                                    void* d_out_hits, uint32_t hits_cap, void* d_out_nhits, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  ViewTable vt;
  if (int rc = device_views_args(rs, d_bytes, d_offsets, d_views, &vt)) return rc;
  return scan_hits_device(rs, d_bytes, d_offsets, n, d_out_words, d_out_hits, hits_cap, d_out_nhits, stream, &vt);
}

int cg_policy_verdict_batch_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_verdicts, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  return verdict_device(rs, d_bytes, d_offsets, n, d_out_verdicts, stream, nullptr);
}
int cg_policy_verdict_batch_device_views(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, const void* d_views, uint32_t n, void* d_out_verdicts,
                                         void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  ViewTable vt;
  if (int rc = device_views_args(rs, d_bytes, d_offsets, d_views, &vt)) return rc;
  return verdict_device(rs, d_bytes, d_offsets, n, d_out_verdicts, stream, &vt);
}

// ---------------------------------------------------------------------------------- policy programs

int cg_ruleset_set_policy_program(cg_ruleset* rs, const uint32_t* program, uint32_t words, uint32_t n_atoms) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!rs || !program || !words) return fail(CG_ERR_INVALID_ARG, "null argument");
  const auto bad = [](const std::string& m) { return fail(CG_ERR_INVALID_ARG, "policy program: " + m); };
  std::vector<uint4> rules;
  uint32_t at = 1;
  const uint32_t n_pol = program[0];
  for (uint32_t p = 0; p < n_pol; p++) {
    if (words - at < 2) return bad("policy " + std::to_string(p) + " runs past the end");
    const uint32_t scope = program[at], n_rules = program[at + 1];
    at += 2;
    if (scope != 0xffffffffu && scope >= n_atoms) return bad("policy " + std::to_string(p) + ": scope atom >= n_atoms");
    const uint32_t first = (uint32_t)rules.size();
    for (uint32_t r = 0; r < n_rules; r++) {
      const std::string where = "policy " + std::to_string(p) + " rule " + std::to_string(r);
      if (rules.size() >= (1u << 20) - 1) return fail(CG_ERR_TOO_LARGE, "policy program: more than 2^20 - 1 rules");
      if (words - at < 2) return bad(where + " runs past the end");
      const uint32_t head = program[at], n_ops = program[at + 1];
      at += 2;
      if (head > 7u) return bad(where + ": effect word must be action | has_reason << 2");
      if (n_ops > words - at) return bad(where + ": ops run past the end");
      if (n_ops > 0xffffffu) return fail(CG_ERR_TOO_LARGE, "policy program: " + where + " has 2^24 ops or more");
      uint32_t depth = 0;
      for (uint32_t k = 0; k < n_ops; k++) {
        const uint32_t o = program[at + k], code = o & 7u;
        if (code == kPolOpConst || code == kPolOpAtom || code == kPolOpHit) {
          if (code == kPolOpConst && (o >> 3) > 1u) return bad(where + ": CONST takes 0 or 1");
          if (code == kPolOpAtom && (o >> 3) >= n_atoms) return bad(where + ": atom >= n_atoms");
          if (code == kPolOpHit && ((o >> 3) & 0x1fffffu) >= rs->dev.n_rules) return bad(where + ": HIT rule >= the rule set's rules");
          if (++depth > 32) return fail(CG_ERR_TOO_LARGE, "policy program: " + where + " needs a stack deeper than 32");
        } else if (code == kPolOpAnd || code == kPolOpOr || code == kPolOpNot) {
          if (o >> 3) return bad(where + ": AND / OR / NOT take no operand");
          if (depth < (code == kPolOpNot ? 1u : 2u)) return bad(where + ": stack underflow");
          if (code != kPolOpNot) depth--;
        } else {
          return bad(where + ": unknown op " + std::to_string(code));
        }
      }
      if (depth != 1) return bad(where + " must leave exactly one value");
      rules.push_back(make_uint4(at, n_ops | (head & 3u) << 24 | (head >> 2) << 26, first, scope));
      at += n_ops;
    }
  }
  if (at != words) return bad("words past the last policy");
  CU(cudaStreamSynchronize(G.stream));
  rs->prog_ops.reset(); rs->prog_rules.reset(); rs->prog_n_rules = rs->prog_n_atoms = 0;
  rs->prog_gen++;                                           // (cg_policy_eval_one's graphs hold the old tables)
  int rc;
  if ((rc = rs->prog_ops.alloc(words)) || (rc = rs->prog_rules.alloc(std::max<size_t>(rules.size(), 1)))) return rc;
  CU(cudaMemcpy(rs->prog_ops.get(), program, (size_t)words * 4, cudaMemcpyHostToDevice));
  if (!rules.empty()) CU(cudaMemcpy(rs->prog_rules.get(), rules.data(), rules.size() * sizeof(uint4), cudaMemcpyHostToDevice));
  rs->prog_n_rules = (uint32_t)rules.size(); rs->prog_n_atoms = n_atoms;
  return CG_OK;
}

namespace {
PolicyTable policy_table(const cg_ruleset* rs) { return PolicyTable{rs->prog_ops.get(), rs->prog_rules.get(), rs->prog_n_rules, (rs->prog_n_atoms + 31) / 32}; }

int policy_eval_host(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, const uint8_t* roles, uint32_t n_texts, const uint32_t* ctx_offsets,
                     const uint32_t* atoms, uint32_t n_ctx, uint32_t* out_verdicts, cg_policy_match* out_matches, uint32_t matches_cap, uint32_t* out_nmatches) {
  if (int rc = require_ready()) return rc;
  if (!rs) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!rs->prog_ops.get()) return fail(CG_ERR_INVALID_ARG, "cg_ruleset_set_policy_program has not been called");
  const PolicyTable pt = policy_table(rs);
  if (!ctx_offsets || (n_texts && !roles) || (n_ctx && (!out_verdicts || (pt.aw && !atoms)))) return fail(CG_ERR_INVALID_ARG, "null argument");
  for (uint32_t c = 0; c < n_ctx; c++)
    if (ctx_offsets[c] > ctx_offsets[c + 1] || ctx_offsets[c + 1] > n_texts) return fail(CG_ERR_INVALID_ARG, "context " + std::to_string(c) + ": text range decreasing or past n_texts");
  const bool want = out_matches || out_nmatches;
  if (!n_ctx) { if (out_nmatches) *out_nmatches = 0; return CG_OK; }
  cudaStream_t st = G.stream;
  InOrder turn(&rs->order, st);
  if (turn.rc) return turn.rc;
  int rc;
  if ((rc = G.d_proles.grow((size_t)n_texts + 1))) return rc;
  if ((rc = G.d_pctx.grow((size_t)n_ctx + 1))) return rc;
  if ((rc = G.d_patoms.grow((size_t)n_ctx * pt.aw + 1))) return rc;
  if ((rc = G.d_verdicts.grow((size_t)n_ctx))) return rc;
  if (n_texts) CU(cudaMemcpyAsync(G.d_proles.get(), roles, n_texts, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(G.d_pctx.get(), ctx_offsets, ((size_t)n_ctx + 1) * 4, cudaMemcpyHostToDevice, st));
  if (pt.aw) CU(cudaMemcpyAsync(G.d_patoms.get(), atoms, (size_t)n_ctx * pt.aw * 4, cudaMemcpyHostToDevice, st));
  const PolicyBatch b{G.d_proles.get(), n_texts, G.d_pctx.get(), G.d_patoms.get(), n_ctx};
  uint64_t total = 0;
  rc = scan_host(rs, bytes, offsets, n_texts, kStepPolicy, [&](const ScanWork& w) {
    count_launches(launch_policy_eval(pt, w, rs->dev.rw, b, G.d_verdicts.get(), want, G.sm_count, st));
    CU(cudaGetLastError());
    if (want) CU(cudaMemcpyAsync(&total, w.out_off + n_ctx, 8, cudaMemcpyDeviceToHost, st));
    return CG_OK;
  }, nullptr, n_ctx);
  if (rc) return rc;
  CU(cudaMemcpyAsync(out_verdicts, G.d_verdicts.get(), (size_t)n_ctx * 4, cudaMemcpyDeviceToHost, st));
  const uint32_t k = out_matches && !(total >> 32) ? (uint32_t)std::min<uint64_t>(total, matches_cap) : 0u;
  if (want) {                                                // (emit runs whatever the count: launches do not depend on it)
    if ((rc = G.d_pmatch.grow(2 * (size_t)k + 1))) return rc;      // [count][pairs]
    count_launches(launch_policy_emit(pt, rs->work, rs->dev.rw, b, G.d_pmatch.get() + 1, k, G.d_pmatch.get(), G.sm_count, st));
    CU(cudaGetLastError());
    if (k) CU(cudaMemcpyAsync(out_matches, G.d_pmatch.get() + 1, (size_t)k * sizeof(cg_policy_match), cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  if (total >> 32) { if (out_nmatches) *out_nmatches = 0xffffffffu; return fail(CG_ERR_TOO_LARGE, "2^32 matches or more in one batch"); }
  if (out_nmatches) *out_nmatches = (uint32_t)total;
  if (out_matches && total > matches_cap) return fail(CG_ERR_CAPACITY, "out_matches too small (see *out_nmatches)");
  return CG_OK;
}

int policy_eval_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, const void* d_roles, uint32_t n_texts, const void* d_ctx_offsets,
                       const void* d_atoms, uint32_t n_ctx, void* d_out_verdicts, void* d_out_matches, uint32_t matches_cap, void* d_out_nmatches,
                       void* stream) {
  if (int rc = require_ready()) return rc;
  if (!rs) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!rs->prog_ops.get()) return fail(CG_ERR_INVALID_ARG, "cg_ruleset_set_policy_program has not been called");
  const PolicyTable pt = policy_table(rs);
  if ((n_texts && (!d_bytes || !d_offsets || !d_roles)) || !d_ctx_offsets || (n_ctx && (!d_out_verdicts || (pt.aw && !d_atoms))) ||
      (matches_cap && !d_out_matches) || (d_out_matches && !d_out_nmatches))
    return fail(CG_ERR_INVALID_ARG, "null argument");
  if ((uintptr_t)d_bytes & 15u) return fail(CG_ERR_INVALID_ARG, "d_bytes must be 16-byte aligned");
  if (((uintptr_t)d_offsets | (uintptr_t)d_ctx_offsets | (uintptr_t)d_atoms | (uintptr_t)d_out_verdicts | (uintptr_t)d_out_matches | (uintptr_t)d_out_nmatches) & 3u)
    return fail(CG_ERR_INVALID_ARG, "d_offsets, d_ctx_offsets, d_atoms and the outputs must be 4-byte aligned");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream;
  const bool want = d_out_nmatches != nullptr;
  if (!n_ctx) { if (want) CU(cudaMemsetAsync(d_out_nmatches, 0, 4, st)); return CG_OK; }
  const PolicyBatch b{(const uint8_t*)d_roles, n_texts, (const uint32_t*)d_ctx_offsets, (const uint32_t*)d_atoms, n_ctx};
  return scan_device(rs, d_bytes, d_offsets, n_texts, nullptr, kStepPolicy, st, [&](const ScanWork& w) {
    int k = launch_policy_eval(pt, w, rs->dev.rw, b, (uint32_t*)d_out_verdicts, want, G.sm_count, st);
    if (want) k += launch_policy_emit(pt, w, rs->dev.rw, b, (uint32_t*)d_out_matches, d_out_matches ? matches_cap : 0u, (uint32_t*)d_out_nmatches, G.sm_count, st);
    return k;
  }, false, nullptr, n_ctx);
}
}  // namespace

int cg_policy_eval_batch(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, const uint8_t* roles, uint32_t n_texts, const uint32_t* ctx_offsets,
                         const uint32_t* atoms, uint32_t n_ctx, uint32_t* out_verdicts, cg_policy_match* out_matches, uint32_t matches_cap, uint32_t* out_nmatches) {
  std::lock_guard<std::mutex> lk(g_mu);
  return policy_eval_host(rs, bytes, offsets, roles, n_texts, ctx_offsets, atoms, n_ctx, out_verdicts, out_matches, matches_cap, out_nmatches);
}

int cg_policy_eval_batch_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, const void* d_roles, uint32_t n_texts, const void* d_ctx_offsets,
                                const void* d_atoms, uint32_t n_ctx, void* d_out_verdicts, void* d_out_matches, uint32_t matches_cap, void* d_out_nmatches,
                                void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  return policy_eval_device(rs, d_bytes, d_offsets, d_roles, n_texts, d_ctx_offsets, d_atoms, n_ctx, d_out_verdicts, d_out_matches, matches_cap,
                            d_out_nmatches, stream);
}

namespace {
// cg_policy_eval_one on the staging block: one H2D copy, one graph (the policy-mode step over the staged texts, then
// policy_eval_one_kernel), one D2H copy of the header and as many rules as the caller can take, one synchronise.  Outputs,
// statuses and statistics are those of cg_policy_eval_batch with one context.  -> CG_OK, an error, or 1 = take the batch call
// (an argument the batch call rejects or judges, no device, profiling, more texts, bytes or atoms than the staging block
// holds, more matches than it holds and the caller wants, a queue overflowed)
int policy_one_fast(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, const uint8_t* roles, uint32_t n_texts, const uint32_t* atoms,
                    uint32_t* out_verdict, uint32_t* out_rules, uint32_t rules_cap, uint32_t* out_nrules) {
  if (!G.ready || !rs || !rs->prog_ops.get() || !out_verdict || G.profiling || n_texts > kPeOneTexts) return 1;
  if (n_texts && (!bytes || !offsets || !roles)) return 1;
  const PolicyTable pt = policy_table(rs);
  if (pt.aw > kPeOneAtomWords || (pt.aw && !atoms)) return 1;
  for (uint32_t i = 0; i < n_texts; i++) if (offsets[i + 1] < offsets[i]) return 1;
  const uint32_t first = n_texts ? offsets[0] : 0, len = n_texts ? offsets[n_texts] - first : 0;
  if (len > kPeOneBytes) return 1;
  Staging& s = rs->pone.io;
  // matches <= policies <= program rules: no more of them than the caller takes can be needed
  const uint32_t want = std::min(std::min(out_rules ? rules_cap : 0u, kPeOneRulesCap), pt.n_rules);
  const int rc = blocking_call(rs, kStepPolicy, n_texts, 1, rs->pone.graphs, {n_texts, rs->prog_gen}, s, [&](uint8_t* h) {
        if (n_texts) memcpy(h + kPeRolesAt, roles, n_texts);
        if (pt.aw) memcpy(h + kPeAtomsAt, atoms, (size_t)pt.aw * 4);
        return stage_texts(h, kPeTextAt, bytes, offsets, n_texts);
      }, [&] {
        const ScanWork& w = rs->work;
        const PolicyBatch b{s.d.get() + kPeRolesAt, n_texts, nullptr, reinterpret_cast<const uint32_t*>(s.d.get() + kPeAtomsAt), 1};
        const int r = run_scan_device(rs, s.d.get(), reinterpret_cast<const uint32_t*>(s.d.get()), n_texts, w.words, kStepPolicy, G.stream);
        if (r != CG_OK) return r;
        count_launches(launch_policy_eval_one(pt, w, rs->dev.rw, b, reinterpret_cast<uint32_t*>(s.d.get() + kPeIn), kPeOneRulesCap, G.stream));
        CU(cudaGetLastError());
        return CG_OK;
      }, s, kPeIn, 4 * ((size_t)kPeOneRules + want), kPeIn + 4 * kPeOneCounters);
  if (rc) return rc;                                             // 1: a queue overflowed, the batch call retries with larger scratch
  const uint32_t* ho = reinterpret_cast<const uint32_t*>(s.h.get() + kPeIn);
  const uint32_t* hc = ho + kPeOneCounters;
  const uint32_t nm = ho[1];
  if (out_rules && nm > kPeOneRulesCap && rules_cap > kPeOneRulesCap) return 1;
  count_step(n_texts, len, hc);
  *out_verdict = ho[0];
  if (out_nrules) *out_nrules = nm;
  if (out_rules) memcpy(out_rules, ho + kPeOneRules, (size_t)std::min(nm, rules_cap) * 4);
  if (out_rules && nm > rules_cap) return fail(CG_ERR_CAPACITY, "out_rules too small (see *out_nrules)");
  return CG_OK;
}
}  // namespace

int cg_policy_eval_one(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, const uint8_t* roles, uint32_t n_texts, const uint32_t* atoms,
                       uint32_t* out_verdict, uint32_t* out_rules, uint32_t rules_cap, uint32_t* out_nrules) {
  std::lock_guard<std::mutex> lk(g_mu);
  const int frc = policy_one_fast(rs, bytes, offsets, roles, n_texts, atoms, out_verdict, out_rules, rules_cap, out_nrules);
  if (frc != 1) return frc;
  // the batch call with one context; the match list staged here (matches <= program rules), its rules copied out as the batch
  // call writes its matches: the first rules_cap on CG_ERR_CAPACITY, none when it fails earlier (nm then stays unwritten)
  const uint32_t ctx[2] = {0, n_texts};
  const uint32_t cap = std::min(rules_cap, rs && G.ready ? rs->prog_n_rules : 0u);
  std::vector<cg_policy_match> m(out_rules ? std::max<uint32_t>(cap, 1u) : 0u);
  uint32_t nm = 0xffffffffu;
  const int rc = policy_eval_host(rs, bytes, offsets, roles, n_texts, ctx, atoms, 1, out_verdict, out_rules ? m.data() : nullptr, out_rules ? cap : 0u,
                                  out_rules || out_nrules ? &nm : nullptr);
  if (nm == 0xffffffffu) return rc;
  if (out_nrules) *out_nrules = nm;
  if (out_rules) for (uint32_t i = 0; i < nm && i < cap; i++) out_rules[i] = m[i].rule;
  return rc;
}

// ---------------------------------------------------------------------------------- SHA / Merkle

int cg_sha256_batch(const uint8_t* bytes, const uint64_t* offsets, uint32_t n, uint8_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!n) return CG_OK;
  if (!offsets || !out) return fail(CG_ERR_INVALID_ARG, "null argument");
  cudaStream_t st = G.stream;
  InOrder turn(&G.dig_order, st);
  size_t total = offsets[n]; int rc;
  if ((rc = turn.rc)) return rc;
  if ((rc = G.d_bytes.grow(total + 64))) return rc;
  if ((rc = G.d_off64.grow((size_t)n + 1))) return rc;
  if ((rc = G.d_dig[0].grow((size_t)n * 8))) return rc;
  if (total) CU(cudaMemcpyAsync(G.d_bytes.get(), bytes, total, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(G.d_off64.get(), offsets, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
  int k = launch_sha256_batch(G.d_bytes.get(), G.d_off64.get(), n, (uint8_t*)G.d_dig[0].get(), st);
  count_launches(k); G.stats.sha256_items += n;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, G.d_dig[0].get(), (size_t)n * 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}

namespace {
int empty_root(uint8_t out[32]) {
  // SHA-256("") -- computed by the same kernel, not on the CPU
  InOrder turn(&G.dig_order, G.stream);
  int rc;
  if ((rc = turn.rc)) return rc;
  if ((rc = G.d_off64.grow(2))) return rc;
  if ((rc = G.d_dig[0].grow(8))) return rc;
  if ((rc = G.d_bytes.grow(64))) return rc;
  CU(cudaMemsetAsync(G.d_off64.get(), 0, 16, G.stream));
  int k = launch_sha256_batch(G.d_bytes.get(), G.d_off64.get(), 1, (uint8_t*)G.d_dig[0].get(), G.stream);
  count_launches(k);
  CU(cudaMemcpyAsync(out, G.d_dig[0].get(), 32, cudaMemcpyDeviceToHost, G.stream));
  CU(cudaStreamSynchronize(G.stream));
  return CG_OK;
}

// One-shot trees: size_dig(n) makes room for n staged nodes in G.d_dig[0]; fold_dig folds n nodes at d_nodes (read in place,
// may be G.d_dig[0]) by at most max_levels levels, ping-ponging between G.d_dig[1] and G.d_dig[0]; *out = the folded nodes
int size_dig(uint64_t n) {
  int rc = G.d_dig[0].grow((size_t)n * 8);
  return rc ? rc : G.d_dig[1].grow((size_t)(n + 1) / 2 * 8 + 8);
}
int fold_dig(const uint32_t* d_nodes, uint64_t n, uint32_t max_levels, cudaStream_t st, const uint32_t** out) {
  count_launches(launch_merkle_fold(d_nodes, n, max_levels, G.d_dig[1].get(), G.d_dig[0].get(), st, out));
  CU(cudaGetLastError());
  return CG_OK;
}

// root of n leaves in G.d_bytes (ragged at d_off, else leaf_len bytes each) -> host; leaves and fold time last_merkle_ms
int staged_root(uint64_t n, const uint64_t* d_off, uint64_t leaf_len, uint8_t out_root[32]) {
  cudaStream_t st = G.stream; const uint32_t* d_root; int rc;
  InOrder turn(&G.dig_order, st);
  if ((rc = turn.rc)) return rc;
  if ((rc = size_dig(n))) return rc;
  CU(cudaEventRecord(G.ev0, st));
  count_launches(d_off ? launch_merkle_leaves_var(G.d_bytes.get(), d_off, n, G.d_dig[0].get(), st) : launch_merkle_leaves_fixed(G.d_bytes.get(), leaf_len, n, G.d_dig[0].get(), st));
  G.stats.merkle_leaves += n;
  if ((rc = fold_dig(G.d_dig[0].get(), n, 64, st, &d_root))) return rc;
  CU(cudaEventRecord(G.ev1, st));
  CU(cudaMemcpyAsync(out_root, d_root, 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  float ms = 0; cudaEventElapsedTime(&ms, G.ev0, G.ev1); G.stats.last_merkle_ms = ms;
  return CG_OK;
}

// roots of the aligned 2^block_log2-leaf blocks of n fixed-size leaves in device memory -> d_roots (32 bytes per block)
int block_roots(const void* d_bytes, uint64_t leaf_len, uint64_t n, uint32_t block_log2, void* d_roots, cudaStream_t st) {
  const uint32_t* d_res; int rc;
  InOrder turn(&G.dig_order, st);
  if ((rc = turn.rc)) return rc;
  if ((rc = size_dig(n))) return rc;
  count_launches(launch_merkle_leaves_fixed((const uint8_t*)d_bytes, leaf_len, n, G.d_dig[0].get(), st)); G.stats.merkle_leaves += n;
  if ((rc = fold_dig(G.d_dig[0].get(), n, block_log2, st, &d_res))) return rc;
  CU(cudaMemcpyAsync(d_roots, d_res, ((n + (1ull << block_log2) - 1) >> block_log2) * 32, cudaMemcpyDeviceToDevice, st));
  return CG_OK;
}
}  // namespace

int cg_merkle_root(const uint8_t* bytes, const uint64_t* offsets, uint64_t n, uint8_t out_root[32]) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!out_root) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (n == 0) return empty_root(out_root);
  if (!offsets) return fail(CG_ERR_INVALID_ARG, "null argument");
  size_t total = offsets[n]; int rc;
  if ((rc = G.d_bytes.grow(total + 64))) return rc;
  if ((rc = G.d_off64.grow((size_t)n + 1))) return rc;
  if (total) CU(cudaMemcpyAsync(G.d_bytes.get(), bytes, total, cudaMemcpyHostToDevice, G.stream));
  CU(cudaMemcpyAsync(G.d_off64.get(), offsets, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, G.stream));
  return staged_root(n, G.d_off64.get(), 0, out_root);
}

int cg_merkle_root_fixed(const uint8_t* bytes, uint64_t leaf_len, uint64_t n, uint8_t out_root[32]) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!out_root) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (n == 0) return empty_root(out_root);
  size_t total = (size_t)leaf_len * n; int rc;
  if ((rc = G.d_bytes.grow(total + 64))) return rc;
  if (total) CU(cudaMemcpyAsync(G.d_bytes.get(), bytes, total, cudaMemcpyHostToDevice, G.stream));
  return staged_root(n, nullptr, leaf_len, out_root);
}

int cg_merkle_block_roots_device(const void* d_bytes, uint64_t leaf_len, uint64_t n, uint32_t block_log2, void* d_out_roots, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  // (beyond 2^40 leaves per block the block count would need a shift of 64 or more: undefined, and it sizes the copy)
  if (block_log2 > 40) return fail(CG_ERR_INVALID_ARG, "block_log2 must be at most 40");
  if (!n) return CG_OK;
  if (!d_bytes || !d_out_roots) return fail(CG_ERR_INVALID_ARG, "null argument");
  return block_roots(d_bytes, leaf_len, n, block_log2, d_out_roots, stream ? (cudaStream_t)stream : G.stream);
}

int cg_merkle_fold(const uint8_t* nodes32, uint64_t m, uint8_t out_root[32]) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!out_root) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (m == 0) return empty_root(out_root);
  if (!nodes32) return fail(CG_ERR_INVALID_ARG, "null argument");
  cudaStream_t st = G.stream; const uint32_t* d_root; int rc;
  InOrder turn(&G.dig_order, st);
  if ((rc = turn.rc)) return rc;
  if ((rc = size_dig(m))) return rc;
  CU(cudaMemcpyAsync(G.d_dig[0].get(), nodes32, m * 32, cudaMemcpyHostToDevice, st));
  if ((rc = fold_dig(G.d_dig[0].get(), m, 64, st, &d_root))) return rc;
  CU(cudaMemcpyAsync(out_root, d_root, 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}

int cg_merkle_fold_device(const void* d_nodes32, uint64_t m, void* d_out_root32, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!m || !d_nodes32 || !d_out_root32) return fail(CG_ERR_INVALID_ARG, "null or empty input");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream; const uint32_t* d_root; int rc;
  InOrder turn(&G.dig_order, st);
  if ((rc = turn.rc)) return rc;
  if ((rc = size_dig(m))) return rc;
  // the fold reads the nodes in place, unless they are off the 16-byte alignment of the kernels' loads: then from a copy
  const uint32_t* d_nodes = (const uint32_t*)d_nodes32;
  if ((uintptr_t)d_nodes32 & 15) { CU(cudaMemcpyAsync(G.d_dig[0].get(), d_nodes32, m * 32, cudaMemcpyDeviceToDevice, st)); d_nodes = G.d_dig[0].get(); }
  if ((rc = fold_dig(d_nodes, m, 64, st, &d_root))) return rc;
  CU(cudaMemcpyAsync(d_out_root32, d_root, 32, cudaMemcpyDeviceToDevice, st));
  return CG_OK;
}

// ---------------------------------------------------------------------------------- Merkle log (append, frontier, proofs)
struct cg_merkle_log {
  uint64_t n = 0;                 // leaves so far; bit h of n set <=> slot h holds the root of a perfect 2^h subtree
  bool keep = false;              // keep every leaf digest in HBM (needed for inclusion proofs)
  DevBuf<uint32_t> d_slots;       // 64 x 8 words
  DevBuf<uint32_t> d_tmp;         // 65 x 8 words: [0..63] a proof folded from the leaf digests, [64] the root
  DevBuf<uint32_t> d_new;         // !keep: the current batch's leaf digests
  DevBuf<uint32_t> d_a, d_b;      // level ping-pong
  // keep: d_lvl[0] holds the n leaf digests.  tree (cg_merkle_log_create_tree): level h >= 1 holds floor(n / 2^h) nodes at d_lvl[h]
  // (node j covers leaves [j 2^h, (j + 1) 2^h)), each level sized for (leaf digest room) >> h nodes, so the store is smaller than
  // the leaf digests; d_spine: 64 x 8 words, the suffix roots of the tree size of the last proof call (log_spine)
  bool tree = false;
  DevBuf<uint32_t> d_lvl[64];
  DevBuf<uint32_t> d_spine;
  IssueOrder order;               // every call on the log, host-buffer or device-resident, on the library's stream or the caller's
  // set by the device when an append read a decreasing offset pair (that leaf went in as the empty leaf); cg_merkle_log_join
  // reports it once and from then on the log refuses every call (failed)
  DevBuf<uint32_t> d_err;
  bool failed = false;
  ~cg_merkle_log() { if (order.ev) cudaEventDestroy(order.ev); }     // (the buffers release themselves)
};

namespace {
// room in the level ping-pong for a fold of cnt > 1 nodes
int log_fold_room(cg_merkle_log* L, uint64_t cnt) {
  int rc = L->d_a.grow((size_t)(cnt + 1) / 2 * 8 + 8);
  return rc ? rc : L->d_b.grow((size_t)(cnt + 3) / 4 * 8 + 8);
}
// MTH of `cnt` consecutive leaf digests starting at d_in (level-wise, unpaired node promoted) -> d_out (32 bytes)
int log_range_root(cg_merkle_log* L, const uint32_t* d_in, uint64_t cnt, uint32_t* d_out, cudaStream_t st) {
  int rc;
  if (cnt == 1) { CU(cudaMemcpyAsync(d_out, d_in, 32, cudaMemcpyDeviceToDevice, st)); return CG_OK; }
  if ((rc = log_fold_room(L, cnt))) return rc;
  const uint32_t* d_root;
  count_launches(launch_merkle_fold(d_in, cnt, 64, L->d_a.get(), L->d_b.get(), st, &d_root));
  CU(cudaMemcpyAsync(d_out, d_root, 32, cudaMemcpyDeviceToDevice, st));
  return CG_OK;
}
int log_check(cg_merkle_log* L) {
  if (int rc = require_ready()) return rc;
  if (!L) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (L->failed) return fail(CG_ERR_INVALID_ARG, "a device append put a leaf with a decreasing offset pair into this log (reported by cg_merkle_log_join): it refuses every call");
  return CG_OK;
}
// root of the current tree -> d_tmp[64]
int log_root_device(cg_merkle_log* L, cudaStream_t st) {
  // fold the frontier from the smallest subtree upwards: r = slot[lowest]; r = node(slot[h], r) for every higher set bit
  const int lowest = __builtin_ctzll(L->n);
  ChainOperands ops{}; uint32_t nl = 0;
  for (int h = lowest + 1; h < 64; h++) if ((L->n >> h) & 1ull) ops.left[nl++] = L->d_slots.get() + 8 * h;
  count_launches(launch_merkle_chain_keep(ops, nl, L->d_slots.get() + 8 * lowest, L->d_tmp.get() + 8 * 64, st));
  return CG_OK;
}
// node j of level h of a tree log (level 0: leaf digest j)
uint32_t* log_node(cg_merkle_log* L, uint32_t h, uint64_t j) { return L->d_lvl[h].get() + 8 * (size_t)j; }

int log_new(cg_merkle_log** out, bool keep, bool tree) {
  if (int rc = require_ready()) return rc;
  if (!out) return fail(CG_ERR_INVALID_ARG, "null argument");
  std::unique_ptr<cg_merkle_log> L(new cg_merkle_log());
  L->keep = keep; L->tree = tree; int rc;
  if ((rc = L->d_slots.alloc(64 * 8)) || (rc = L->d_tmp.alloc(65 * 8)) || (rc = L->d_err.alloc(1))) return rc;
  CU(cudaMemset(L->d_slots.get(), 0, 64 * 32)); CU(cudaMemset(L->d_err.get(), 0, 4));
  CU(cudaEventCreateWithFlags(&L->order.ev, cudaEventDisableTiming));
  if (tree && (rc = L->d_spine.alloc(64 * 8))) return rc;
  *out = L.release();
  return CG_OK;
}
}  // namespace

int cg_merkle_log_create(cg_merkle_log** out, int keep_leaf_digests) {
  std::lock_guard<std::mutex> lk(g_mu);
  return log_new(out, keep_leaf_digests != 0, false);
}

int cg_merkle_log_create_tree(cg_merkle_log** out) {
  std::lock_guard<std::mutex> lk(g_mu);
  return log_new(out, true, true);
}
void cg_merkle_log_destroy(cg_merkle_log* L) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (L) { if (G.ready) { cudaStreamSynchronize(G.stream); cudaEventSynchronize(L->order.ev); } delete L; }
}
int cg_merkle_log_size(const cg_merkle_log* L, uint64_t* out_n) { if (!L || !out_n) return fail(CG_ERR_INVALID_ARG, "null argument"); *out_n = L->n; return CG_OK; }

int cg_merkle_log_restore(cg_merkle_log** out, uint64_t n, const uint8_t* frontier32, uint32_t count) {
  if (!out || (count && !frontier32) || count != (uint32_t)__builtin_popcountll(n)) return fail(CG_ERR_INVALID_ARG, "frontier must hold one digest per set bit of n");
  cg_merkle_log* made = nullptr; int rc = cg_merkle_log_create(&made, 0);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g_mu);
  std::unique_ptr<cg_merkle_log> L(made); uint32_t k = 0;  // (destroyed unless complete: *out is set on success only)
  for (int h = 63; h >= 0; h--) if ((n >> h) & 1ull) { CU(cudaMemcpy(L->d_slots.get() + 8 * h, frontier32 + 32 * (size_t)k, 32, cudaMemcpyHostToDevice)); k++; }
  L->n = n;
  *out = L.release();
  return CG_OK;
}

int cg_merkle_log_frontier(cg_merkle_log* L, uint8_t* out_frontier32, uint32_t* out_count) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!out_count) return fail(CG_ERR_INVALID_ARG, "null argument");
  InOrder turn(&L->order, G.stream);
  if ((rc = turn.rc)) return rc;
  uint32_t k = 0;
  for (int h = 63; h >= 0; h--) if ((L->n >> h) & 1ull) { if (out_frontier32) CU(cudaMemcpyAsync(out_frontier32 + 32 * (size_t)k, L->d_slots.get() + 8 * h, 32, cudaMemcpyDeviceToHost, G.stream)); k++; }
  CU(cudaStreamSynchronize(G.stream));
  *out_count = k;
  return CG_OK;
}

namespace {
// room for m more leaf digests; returns where they go
int log_digest_room(cg_merkle_log* L, uint64_t m, cudaStream_t st, uint32_t** out) {
  if (!L->keep) { if (int rc = L->d_new.grow((size_t)m * 8)) return rc; *out = L->d_new.get(); return CG_OK; }
  const uint64_t room = L->d_lvl[0].cap() / 8;
  if (L->n + m > room) {               // grow the digest store (amortised doubling), keeping what is there; a tree log's node
    const uint64_t cap = std::max<uint64_t>(L->n + m, room * 2);          // levels follow (level h holds up to cap >> h nodes)
    DevBuf<uint32_t> nl[64];
    int rc = CG_OK; cudaError_t e = cudaSuccess;
    for (uint32_t h = 0; !rc && e == cudaSuccess && h < (L->tree ? 64u : 1u) && (cap >> h); h++) {
      if ((cap >> h) <= L->d_lvl[h].cap() / 8) continue;
      if (!(rc = nl[h].alloc((size_t)(cap >> h) * 8)) && (L->n >> h)) e = cudaMemcpyAsync(nl[h].get(), L->d_lvl[h].get(), (size_t)(L->n >> h) * 32, cudaMemcpyDeviceToDevice, st);
    }
    // the copies read the old buffers and write the new ones: they are done before any buffer is freed, on failure too
    const cudaError_t s = cudaStreamSynchronize(st);
    if (rc) return rc;
    if (e != cudaSuccess || s != cudaSuccess) return cuda_fail(e != cudaSuccess ? e : s, e != cudaSuccess ? "cudaMemcpyAsync" : "cudaStreamSynchronize(st)");
    for (uint32_t h = 0; h < 64; h++) if (nl[h].get()) L->d_lvl[h] = std::move(nl[h]);
  }
  *out = L->d_lvl[0].get() + (size_t)L->n * 8;
  return CG_OK;
}
// m new leaf digests at d_dig: cut [n, n+m) into aligned perfect blocks (block size <= lowest set bit of its position),
// reduce each, carry into the frontier.  On a tree log the block's fold writes its levels into the store (its root is node
// (h, pos >> h)) and every carry makes the complete node (top, pos >> top) under the next occupied slot.  The plan depends on
// n and m only; with wait the host waits for st before the log counts the leaves (host-buffer appends), without it the
// launches stay in flight (device-resident appends: the size counts enqueued leaves).
int log_absorb(cg_merkle_log* L, const uint32_t* d_dig, uint64_t m, cudaStream_t st, bool wait = true) {
  int rc;
  uint64_t pos = L->n, rem = m;
  while (rem) {
    uint64_t s = pos ? (pos & (~pos + 1)) : (1ull << 63);
    while (s > rem) s >>= 1;
    int h = 0; while ((1ull << h) < s) h++;
    uint32_t* lv[64] = {};
    if (L->tree) for (int l = 1; l <= h; l++) lv[l] = log_node(L, l, pos >> l);
    else if (s > 1 && (rc = log_fold_room(L, s))) return rc;
    const uint32_t* acc;                                    // the block's root (a block of one leaf: the leaf digest, no launch)
    count_launches(launch_merkle_fold(d_dig + (size_t)(pos - L->n) * 8, s, 64, L->d_a.get(), L->d_b.get(), st, &acc, L->tree ? lv : nullptr));
    ChainOperands ops{}; uint32_t nl = 0; int top = h;     // slots h, h+1, ... that are occupied merge into the new subtree
    while ((pos >> top) & 1ull) { ops.left[nl] = L->d_slots.get() + 8 * top; top++; ops.keep[nl] = L->tree ? log_node(L, top, pos >> top) : nullptr; nl++; }
    if (nl) count_launches(launch_merkle_chain_keep(ops, nl, acc, L->d_slots.get() + 8 * top, st));
    else CU(cudaMemcpyAsync(L->d_slots.get() + 8 * top, acc, 32, cudaMemcpyDeviceToDevice, st));
    pos += s; rem -= s;
  }
  CU(cudaGetLastError());
  if (wait) CU(cudaStreamSynchronize(st));
  L->n += m;
  return CG_OK;
}
}  // namespace

/* room for n_leaves more leaf digests and their bytes up front (an append that has to grow the digest store pays a device
 * allocation and a copy of everything kept so far); on a log without a node store also the fold ping-pong for a block of
 * n_leaves (24 bytes per leaf), which its appends would otherwise grow themselves */
int cg_merkle_log_reserve(cg_merkle_log* L, uint64_t n_leaves, uint64_t n_bytes) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  InOrder turn(&L->order, G.stream);
  if ((rc = turn.rc)) return rc;
  uint32_t* unused;
  if (n_leaves && (rc = log_digest_room(L, n_leaves, G.stream, &unused))) return rc;
  if (n_leaves > 1 && !L->tree && (rc = log_fold_room(L, n_leaves))) return rc;     // (a tree log folds into its store)
  if (n_bytes && (rc = G.d_bytes.grow((size_t)n_bytes + 64))) return rc;
  if (n_leaves && (rc = G.d_off64.grow((size_t)n_leaves + 1))) return rc;
  return CG_OK;
}

int cg_merkle_log_append(cg_merkle_log* L, const uint8_t* bytes, const uint64_t* offsets, uint64_t m) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!m) return CG_OK;
  if (!offsets) return fail(CG_ERR_INVALID_ARG, "null argument");
  for (uint64_t i = 0; i < m; i++) if (offsets[i + 1] < offsets[i]) return fail(CG_ERR_INVALID_ARG, "offsets must be non-decreasing");
  if (L->n + m < L->n) return fail(CG_ERR_TOO_LARGE, "log size overflows 64 bits");
  cudaStream_t st = G.stream;
  InOrder turn(&L->order, st);
  if ((rc = turn.rc)) return rc;
  const size_t first = offsets[0], total = offsets[m];
  if ((rc = G.d_bytes.grow(total + 64))) return rc;
  if ((rc = G.d_off64.grow((size_t)m + 1))) return rc;
  if ((rc = ensure_copy_streams())) return rc;
  uint32_t* d_dig;                                          // where this batch's leaf digests go
  if ((rc = log_digest_room(L, m, st, &d_dig))) return rc;
  CU(cudaStreamSynchronize(st));                            // (whatever still read the staging buffer is done)
  CU(cudaMemcpyAsync(G.d_off64.get(), offsets, ((size_t)m + 1) * 8, cudaMemcpyHostToDevice, G.s_h2d));
  // the leaf bytes go over in pieces on the copy stream; the leaf kernel of piece c runs while piece c + 1 is still in flight
  const int C = (total - first) > ((size_t)4 << 20) ? Ctx::kChunks : 1;
  const uint64_t per = (m + C - 1) / C;
  for (int c = 0; c < C; c++) {
    const uint64_t m0 = std::min<uint64_t>((uint64_t)c * per, m), m1 = std::min<uint64_t>((uint64_t)(c + 1) * per, m);
    if (m1 <= m0) break;
    const size_t b0 = offsets[m0], b1 = offsets[m1];
    if (b1 > b0) CU(cudaMemcpyAsync(G.d_bytes.get() + b0, bytes + b0, b1 - b0, cudaMemcpyHostToDevice, G.s_h2d));
    CU(cudaEventRecord(G.e_h2d[c], G.s_h2d));
    CU(cudaStreamWaitEvent(st, G.e_h2d[c], 0));
    int k = launch_merkle_leaves_var(G.d_bytes.get(), G.d_off64.get() + m0, m1 - m0, d_dig + (size_t)m0 * 8, st);
    count_launches(k);
  }
  G.stats.merkle_leaves += m;
  return log_absorb(L, d_dig, m, st);
}

/* The event log as it lies on disk (src/audit-trail.ts:151-179: one JSON.stringify(record) per line, records joined with
 * "\n", a trailing "\n" per flush): the buffer is split at '\n' ON THE DEVICE, every line (without its '\n') is a leaf. */
int cg_merkle_log_append_jsonl(cg_merkle_log* L, const uint8_t* bytes, uint64_t len, uint64_t* out_lines) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (out_lines) *out_lines = 0;
  if (!len) return CG_OK;
  if (!bytes) return fail(CG_ERR_INVALID_ARG, "null argument");
  cudaStream_t st = G.stream;
  InOrder turn(&L->order, st);
  if ((rc = turn.rc)) return rc;
  const uint32_t n_pieces = (uint32_t)((len + 4095) / 4096);
  if ((rc = G.d_bytes.grow((size_t)len + 64))) return rc;
  if ((rc = G.d_off32.grow((size_t)n_pieces + 4))) return rc;          // newline counts per 4 KB piece
  if ((rc = G.d_off64.grow(2))) return rc;
  CU(cudaMemcpyAsync(G.d_bytes.get(), bytes, len, cudaMemcpyHostToDevice, st));
  uint64_t* d_total = G.d_off64.get();                           // (re-grown below once the line count is known)
  int k = launch_newline_split(G.d_bytes.get(), len, G.d_off32.get(), d_total, st);
  uint64_t n_lines = 0;
  CU(cudaMemcpyAsync(&n_lines, d_total, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (!n_lines) return CG_OK;
  if (L->n + n_lines < L->n) return fail(CG_ERR_TOO_LARGE, "log size overflows 64 bits");
  if ((rc = G.d_off64.grow((size_t)n_lines + 1))) return rc;
  k += launch_newline_starts(G.d_bytes.get(), len, G.d_off32.get(), G.d_off64.get(), n_lines, st);
  uint32_t* d_dig;
  if ((rc = log_digest_room(L, n_lines, st, &d_dig))) return rc;
  k += launch_merkle_leaves_var(G.d_bytes.get(), G.d_off64.get(), n_lines, d_dig, st, /*trim_newline=*/true);
  count_launches(k); G.stats.merkle_leaves += n_lines;
  if (out_lines) *out_lines = n_lines;
  return log_absorb(L, d_dig, n_lines, st);
}

int cg_merkle_log_root(cg_merkle_log* L, uint8_t out_root[32]) {
  {
    std::lock_guard<std::mutex> lk(g_mu);
    int rc = log_check(L); if (rc) return rc;
    if (!out_root) return fail(CG_ERR_INVALID_ARG, "null argument");
    InOrder turn(&L->order, G.stream);
    if ((rc = turn.rc)) return rc;
    if (L->n) {
      if ((rc = log_root_device(L, G.stream))) return rc;
      CU(cudaMemcpyAsync(out_root, L->d_tmp.get() + 8 * 64, 32, cudaMemcpyDeviceToHost, G.stream));
      CU(cudaStreamSynchronize(G.stream));
      return CG_OK;
    }
    return empty_root(out_root);
  }
}

namespace {
// Proofs on a tree log.  Every sibling range of RFC 6962's recursion over D[0:s] is a complete aligned node of the store or a
// suffix D[a:s] whose root is a right-to-left fold of s's frontier subtrees: the spine.  spine[h] (h a set bit of s above its
// lowest) = MTH(D[s with bits <= h cleared : s]), made by one chain over the frontier subtrees, which are stored nodes.
int log_spine(cg_merkle_log* L, uint64_t s, cudaStream_t st) {
  const int lowest = __builtin_ctzll(s);
  ChainOperands ops{}; uint32_t nl = 0;
  for (int h = lowest + 1; h < 64; h++) if ((s >> h) & 1ull) { ops.left[nl] = log_node(L, h, (s >> h) - 1); ops.keep[nl] = L->d_spine.get() + 8 * h; nl++; }
  count_launches(launch_merkle_chain_keep(ops, nl, log_node(L, lowest, (s >> lowest) - 1), nullptr, st));
  return CG_OK;
}
NodeStore log_store(cg_merkle_log* L) {
  NodeStore ns{};
  for (uint32_t h = 0; h < 64; h++) ns.lvl[h] = L->d_lvl[h].get();
  return ns;
}
// The leaf ranges [a, b) of PATH(i, D[0:size]) (RFC 6962 2.1.1; first == 0), or of PROOF(first, D[0:size]) (2.1.2; i unused),
// in proof order -- the gather kernel's rule (merkle_path_element): a consistency proof is the node (ctz first, (first - 1) >>
// ctz first) unless first is a power of two, then the path of leaf first - 1 from level ctz first up (nothing when first == size).
std::vector<std::pair<uint64_t, uint64_t>> proof_ranges(uint64_t i, uint64_t size, uint64_t first) {
  std::vector<std::pair<uint64_t, uint64_t>> r;
  uint32_t lo = 0;
  if (first) {
    if (first == size) return r;
    i = first - 1; lo = (uint32_t)__builtin_ctzll(first);
    if (first & (first - 1)) r.push_back({first - (1ull << lo), first});
  }
  for (uint64_t levels = merkle_path_levels(i, size, lo); levels; levels &= levels - 1) {
    const uint32_t l = (uint32_t)__builtin_ctzll(levels);
    const uint64_t b = ((i >> l) ^ 1ull) << l;
    r.push_back({b, b + std::min<uint64_t>(size - b, 1ull << l)});
  }
  return r;
}
// the spine of `size`, then m paths (leaf indices h_idx, or one consistency proof from `first` when h_idx is null) at `stride`
// digests each -> out_paths32 (host), their lengths -> out_lens (host, may be null).  Two launches, whatever m and size.
int log_gather(cg_merkle_log* L, const uint64_t* h_idx, uint32_t m, uint64_t size, uint64_t first, uint8_t* out_paths32, uint32_t stride,
               uint32_t* out_lens) {
  cudaStream_t st = G.stream; int rc;
  InOrder turn(&G.dig_order, st);
  if ((rc = turn.rc)) return rc;
  const size_t path_words = (size_t)m * stride * 8, lens_words = ((size_t)m + 7) / 8 * 8;
  if ((rc = G.d_dig[0].grow(path_words + lens_words))) return rc;
  if (h_idx && (rc = G.d_off64.grow((size_t)m))) return rc;
  uint32_t* d_paths = G.d_dig[0].get(); uint32_t* d_lens = d_paths + path_words;
  if (h_idx) CU(cudaMemcpyAsync(G.d_off64.get(), h_idx, (size_t)m * 8, cudaMemcpyHostToDevice, st));
  if ((rc = log_spine(L, size, st))) return rc;
  count_launches(launch_merkle_gather(log_store(L), L->d_spine.get(), size, h_idx ? G.d_off64.get() : nullptr, first, m, stride, d_paths, d_lens, G.sm_count, st));
  CU(cudaGetLastError());
  if (path_words) CU(cudaMemcpyAsync(out_paths32, d_paths, path_words * 4, cudaMemcpyDeviceToHost, st));
  if (out_lens) CU(cudaMemcpyAsync(out_lens, d_lens, (size_t)m * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}
// one proof at the log's size, whose ranges are `ranges` (proof_ranges) -> out_path32 (host): gathered from the node store on a
// tree log, else every range folded from the leaf digests.  The path of leaf *h_idx, or PROOF(first, ...) when h_idx is null.
int log_proof(cg_merkle_log* L, const std::vector<std::pair<uint64_t, uint64_t>>& ranges, const uint64_t* h_idx, uint64_t first, uint8_t* out_path32) {
  if (L->tree) return ranges.empty() ? CG_OK : log_gather(L, h_idx, 1, L->n, first, out_path32, (uint32_t)ranges.size(), nullptr);
  cudaStream_t st = G.stream; int rc;
  for (size_t i = 0; i < ranges.size(); i++)
    if ((rc = log_range_root(L, L->d_lvl[0].get() + (size_t)ranges[i].first * 8, ranges[i].second - ranges[i].first, L->d_tmp.get() + 8 * i, st))) return rc;
  if (!ranges.empty()) CU(cudaMemcpyAsync(out_path32, L->d_tmp.get(), ranges.size() * 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}
}  // namespace

int cg_merkle_log_proofs(cg_merkle_log* L, const uint64_t* indices, uint32_t m, uint64_t tree_size, uint8_t* out_paths32, uint32_t path_stride,
                         uint32_t* out_lens) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!L->tree) return fail(CG_ERR_UNSUPPORTED, "proofs at any tree size need a log made by cg_merkle_log_create_tree");
  if (tree_size == 0 || tree_size > L->n) return fail(CG_ERR_INVALID_ARG, "tree_size must be in [1, size of the log]");
  if (!m) return CG_OK;
  if (!indices || !out_lens || (path_stride && !out_paths32)) return fail(CG_ERR_INVALID_ARG, "null argument");
  for (uint32_t i = 0; i < m; i++) if (indices[i] >= tree_size) return fail(CG_ERR_INVALID_ARG, "leaf index out of range");
  const uint32_t longest = tree_size > 1 ? 64 - (uint32_t)__builtin_clzll(tree_size - 1) : 0;       // ceil(log2 tree_size)
  if (path_stride < longest) return fail(CG_ERR_CAPACITY, "path_stride is below ceil(log2 tree_size)");
  InOrder turn(&L->order, G.stream);
  if ((rc = turn.rc)) return rc;
  return log_gather(L, indices, m, tree_size, 0, out_paths32, path_stride, out_lens);
}

int cg_merkle_log_consistency_between(cg_merkle_log* L, uint64_t first_size, uint64_t second_size, uint8_t* out_path32, uint32_t path_cap, uint32_t* out_len) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!out_len) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!L->tree) return fail(CG_ERR_UNSUPPORTED, "proofs at any tree size need a log made by cg_merkle_log_create_tree");
  if (second_size == 0 || second_size > L->n || first_size == 0 || first_size > second_size)
    return fail(CG_ERR_INVALID_ARG, "need 1 <= first_size <= second_size <= size of the log");
  const uint32_t len = (uint32_t)proof_ranges(0, second_size, first_size).size();
  if (len > path_cap || (len && !out_path32)) return fail(CG_ERR_CAPACITY, "path buffer too small");
  *out_len = len;
  InOrder turn(&L->order, G.stream);
  if ((rc = turn.rc)) return rc;
  return len ? log_gather(L, nullptr, 1, second_size, first_size, out_path32, len, nullptr) : CG_OK;
}

int cg_merkle_log_proof(cg_merkle_log* L, uint64_t index, uint8_t* out_path32, uint32_t path_cap, uint32_t* out_len) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!out_len) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!L->keep) return fail(CG_ERR_UNSUPPORTED, "log was created without leaf digests (or restored from a frontier): no proofs");
  if (index >= L->n) return fail(CG_ERR_INVALID_ARG, "leaf index out of range");
  const auto ranges = proof_ranges(index, L->n, 0);
  *out_len = (uint32_t)ranges.size();
  if (ranges.size() > path_cap || (ranges.size() && !out_path32)) return fail(CG_ERR_CAPACITY, "path buffer too small");
  InOrder turn(&L->order, G.stream);
  if ((rc = turn.rc)) return rc;
  return log_proof(L, ranges, &index, 0, out_path32);
}

/* RFC 6962 2.1.2: PROOF(m, D[n]) -- the nodes that show the tree of the first m leaves is a prefix of the current one. */
int cg_merkle_log_consistency(cg_merkle_log* L, uint64_t first_size, uint8_t* out_path32, uint32_t path_cap, uint32_t* out_len) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!out_len) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!L->keep) return fail(CG_ERR_UNSUPPORTED, "log was created without leaf digests (or restored from a frontier): no proofs");
  if (first_size == 0 || first_size > L->n) return fail(CG_ERR_INVALID_ARG, "first_size must be in [1, size of the log]");
  const auto ranges = proof_ranges(0, L->n, first_size);
  *out_len = (uint32_t)ranges.size();
  if (ranges.size() > path_cap || ranges.size() > 64 || (ranges.size() && !out_path32)) return fail(CG_ERR_CAPACITY, "path buffer too small");
  InOrder turn(&L->order, G.stream);
  if ((rc = turn.rc)) return rc;
  return log_proof(L, ranges, nullptr, first_size, out_path32);
}

/* RFC 9162 2.1.4.2: *out_ok = 1 iff `path` proves that the tree with root_first over first_size leaves is a prefix of the tree
 * with root_second over second_size leaves (node hashes on the device, as everywhere in this library) */
int cg_merkle_verify_consistency(uint64_t first_size, uint64_t second_size, const uint8_t root_first[32], const uint8_t root_second[32],
                                 const uint8_t* path32, uint32_t path_len, int* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!out_ok || !root_first || !root_second || (path_len && !path32) || path_len > 64) return fail(CG_ERR_INVALID_ARG, "bad argument");
  int rc; cudaStream_t st = G.stream;
  InOrder turn(&G.dig_order, st);
  if ((rc = turn.rc)) return rc;
  if ((rc = G.d_dig[0].grow((size_t)(path_len + 4) * 8))) return rc;
  uint32_t* d_r1 = G.d_dig[0].get(); uint32_t* d_r2 = d_r1 + 8; uint32_t* d_ok = d_r2 + 8; uint32_t* d_path = d_ok + 8;
  CU(cudaMemcpyAsync(d_r1, root_first, 32, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d_r2, root_second, 32, cudaMemcpyHostToDevice, st));
  if (path_len) CU(cudaMemcpyAsync(d_path, path32, (size_t)path_len * 32, cudaMemcpyHostToDevice, st));
  int k = launch_merkle_consistency(first_size, second_size, d_r1, d_r2, d_path, path_len, d_ok, st);
  count_launches(k);
  uint32_t ok = 0;
  CU(cudaMemcpyAsync(&ok, d_ok, 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  *out_ok = (int)ok;
  return CG_OK;
}

namespace {
/* m proofs against one (tree_size, root): the leaves are hashed by the word-granular leaf kernel over the staging buffer, then
 * one thread per proof walks its path (RFC 9162 2.1.3.2).  Two launches, whatever m. */
int verify_proofs(const uint8_t* leaf_bytes, const uint64_t* leaf_offsets, const uint64_t* indices, uint32_t m, uint64_t tree_size,
                  const uint8_t* paths32, uint32_t path_stride, const uint32_t* path_lens, const uint8_t root[32], uint8_t* out_ok) {
  if (!m) return CG_OK;
  if (!leaf_offsets || !indices || !path_lens || !root || !out_ok || (path_stride && !paths32)) return fail(CG_ERR_INVALID_ARG, "null argument");
  for (uint32_t i = 0; i < m; i++) {
    if (leaf_offsets[i + 1] < leaf_offsets[i]) return fail(CG_ERR_INVALID_ARG, "offsets must be non-decreasing");
    if (path_lens[i] > 64 || path_lens[i] > path_stride) return fail(CG_ERR_INVALID_ARG, "a path is longer than 64 digests or than path_stride");
  }
  const size_t total = leaf_offsets[m];
  if (total && !leaf_bytes) return fail(CG_ERR_INVALID_ARG, "null argument");
  int rc; cudaStream_t st = G.stream;
  InOrder turn(&G.dig_order, st);
  if ((rc = turn.rc)) return rc;
  // d_dig[0]: leaf digests | root ; d_dig[1]: paths | indices | lengths | verdicts (every region a multiple of 32 bytes)
  const size_t leaf_words = (size_t)m * 8, path_words = (size_t)m * path_stride * 8, idx_words = ((size_t)m * 2 + 7) / 8 * 8,
               len_words = ((size_t)m + 7) / 8 * 8, ok_words = ((size_t)m + 31) / 32 * 8;
  if ((rc = G.d_bytes.grow(total + 64))) return rc;
  if ((rc = G.d_off64.grow((size_t)m + 1))) return rc;
  if ((rc = G.d_dig[0].grow(leaf_words + 8))) return rc;
  if ((rc = G.d_dig[1].grow(path_words + idx_words + len_words + ok_words))) return rc;
  uint32_t* d_leaf = G.d_dig[0].get(); uint32_t* d_root = d_leaf + leaf_words;
  uint32_t* d_paths = G.d_dig[1].get(); uint64_t* d_idx = reinterpret_cast<uint64_t*>(d_paths + path_words);
  uint32_t* d_lens = d_paths + path_words + idx_words; uint8_t* d_ok = reinterpret_cast<uint8_t*>(d_lens + len_words);
  if (total) CU(cudaMemcpyAsync(G.d_bytes.get(), leaf_bytes, total, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(G.d_off64.get(), leaf_offsets, ((size_t)m + 1) * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d_root, root, 32, cudaMemcpyHostToDevice, st));
  if (path_words) CU(cudaMemcpyAsync(d_paths, paths32, path_words * 4, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d_idx, indices, (size_t)m * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d_lens, path_lens, (size_t)m * 4, cudaMemcpyHostToDevice, st));
  int k = launch_merkle_leaves_var(G.d_bytes.get(), G.d_off64.get(), m, d_leaf, st);
  k += launch_merkle_verify_batch(d_leaf, d_idx, m, tree_size, d_paths, path_stride, d_lens, d_root, d_ok, G.sm_count, st);
  count_launches(k);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out_ok, d_ok, m, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}
}  // namespace

int cg_merkle_verify_proof(const uint8_t* leaf_bytes, uint64_t leaf_len, uint64_t index, uint64_t tree_size, const uint8_t* path32, uint32_t path_len,
                           const uint8_t root[32], int* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!out_ok || !root || (leaf_len && !leaf_bytes) || (path_len && !path32) || path_len > 64) return fail(CG_ERR_INVALID_ARG, "bad argument");
  const uint64_t off[2] = {0, leaf_len}; uint8_t ok = 0;
  int rc = verify_proofs(leaf_bytes, off, &index, 1, tree_size, path32, path_len, &path_len, root, &ok);
  if (!rc) *out_ok = ok;
  return rc;
}

int cg_merkle_verify_proofs(const uint8_t* leaf_bytes, const uint64_t* leaf_offsets, const uint64_t* indices, uint32_t m, uint64_t tree_size,
                            const uint8_t* paths32, uint32_t path_stride, const uint32_t* path_lens, const uint8_t root[32], uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  return verify_proofs(leaf_bytes, leaf_offsets, indices, m, tree_size, paths32, path_stride, path_lens, root, out_ok);
}

// ---------------------------------------------------------------------------------- Merkle log, device-resident
// The host twins' results from buffers in HBM, asynchronous on the caller's stream: the absorb plan, the proof ranges' spine and
// every argument the host can see are worked out on the host, so a call enqueues the twin's launches and waits only when a
// buffer has to grow.  What only the device can see (offsets, indices, path lengths in HBM) is checked by the kernels in band.
namespace {
// a pointer the kernels load from or store to with a width of `align` bytes (null passes: the callers check for null first)
int check_aligned(const void* p, uintptr_t align, const char* what) {
  if ((uintptr_t)p & (align - 1)) return fail(CG_ERR_INVALID_ARG, std::string(what) + " must be " + std::to_string(align) + "-byte aligned");
  return CG_OK;
}
cudaStream_t caller_stream(void* stream) { return stream ? (cudaStream_t)stream : G.stream; }
// m leaves in HBM hashed into the log's digest room (one launch: ragged at d_off, else leaf_len bytes each), then absorbed
// without a final synchronise
int log_append_device(cg_merkle_log* L, const uint8_t* d_bytes, const uint64_t* d_off, uint64_t leaf_len, uint64_t m, void* stream) {
  if (L->n + m < L->n) return fail(CG_ERR_TOO_LARGE, "log size overflows 64 bits");
  const cudaStream_t st = caller_stream(stream); int rc;
  InOrder turn(&L->order, st);
  if ((rc = turn.rc)) return rc;
  uint32_t* d_dig;
  if ((rc = log_digest_room(L, m, st, &d_dig))) return rc;
  count_launches(d_off ? launch_merkle_leaves_guarded(d_bytes, d_off, m, d_dig, L->d_err.get(), st) : launch_merkle_leaves_fixed(d_bytes, leaf_len, m, d_dig, st));
  G.stats.merkle_leaves += m;
  return log_absorb(L, d_dig, m, st, /*wait=*/false);
}
}  // namespace

int cg_merkle_log_append_device(cg_merkle_log* L, const void* d_bytes, const void* d_offsets, uint64_t m, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!m) return CG_OK;
  if (!d_bytes || !d_offsets) return fail(CG_ERR_INVALID_ARG, "null argument");
  if ((rc = check_aligned(d_bytes, 16, "d_bytes")) || (rc = check_aligned(d_offsets, 8, "d_offsets"))) return rc;
  return log_append_device(L, (const uint8_t*)d_bytes, (const uint64_t*)d_offsets, 0, m, stream);
}

int cg_merkle_log_append_fixed_device(cg_merkle_log* L, const void* d_bytes, uint64_t leaf_len, uint64_t m, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!m) return CG_OK;
  if (!d_bytes) return fail(CG_ERR_INVALID_ARG, "null argument");
  // (any alignment: launch_merkle_leaves_fixed takes the byte-granular kernel off the word kernel's alignment, as for
  // cg_merkle_block_roots_device)
  if (leaf_len && m > UINT64_MAX / leaf_len) return fail(CG_ERR_INVALID_ARG, "m * leaf_len overflows 64 bits");
  return log_append_device(L, (const uint8_t*)d_bytes, nullptr, leaf_len, m, stream);
}

int cg_merkle_log_root_device(cg_merkle_log* L, void* d_out_root32, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!d_out_root32) return fail(CG_ERR_INVALID_ARG, "null argument");
  const cudaStream_t st = caller_stream(stream);
  InOrder turn(&L->order, st);
  if ((rc = turn.rc)) return rc;
  if (L->n) {
    if ((rc = log_root_device(L, st))) return rc;
  } else {
    // SHA-256("") by the same kernel as the host twin's, but from the log's own scratch, never the library's staging (whose
    // other users take no turn before they write it): 16 zero bytes of d_tmp are both the offsets pair and the word it loads
    CU(cudaMemsetAsync(L->d_tmp.get(), 0, 32, st));
    count_launches(launch_sha256_batch((const uint8_t*)L->d_tmp.get(), (const uint64_t*)L->d_tmp.get(), 1, (uint8_t*)(L->d_tmp.get() + 8 * 64), st));
  }
  CU(cudaMemcpyAsync(d_out_root32, L->d_tmp.get() + 8 * 64, 32, cudaMemcpyDeviceToDevice, st));
  CU(cudaGetLastError());
  return CG_OK;
}

int cg_merkle_log_proofs_device(cg_merkle_log* L, const void* d_indices, uint32_t m, uint64_t tree_size, void* d_out_paths32, uint32_t path_stride,
                                void* d_out_lens, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!L->tree) return fail(CG_ERR_UNSUPPORTED, "proofs at any tree size need a log made by cg_merkle_log_create_tree");
  if (tree_size == 0 || tree_size > L->n) return fail(CG_ERR_INVALID_ARG, "tree_size must be in [1, size of the log]");
  if (!m) return CG_OK;
  if (!d_indices || !d_out_lens || (path_stride && !d_out_paths32)) return fail(CG_ERR_INVALID_ARG, "null argument");
  if ((rc = check_aligned(d_indices, 8, "d_indices")) || (rc = check_aligned(d_out_paths32, 16, "d_out_paths32")) ||
      (rc = check_aligned(d_out_lens, 4, "d_out_lens"))) return rc;
  const uint32_t longest = tree_size > 1 ? 64 - (uint32_t)__builtin_clzll(tree_size - 1) : 0;       // ceil(log2 tree_size)
  if (path_stride < longest) return fail(CG_ERR_CAPACITY, "path_stride is below ceil(log2 tree_size)");
  const cudaStream_t st = caller_stream(stream);
  InOrder turn(&L->order, st), dig(&G.dig_order, st);
  if ((rc = turn.rc) || (rc = dig.rc)) return rc;
  if ((rc = log_spine(L, tree_size, st))) return rc;
  count_launches(launch_merkle_gather(log_store(L), L->d_spine.get(), tree_size, (const uint64_t*)d_indices, 0, m, path_stride, (uint32_t*)d_out_paths32,
                                      (uint32_t*)d_out_lens, G.sm_count, st, /*checked=*/true));
  CU(cudaGetLastError());
  return CG_OK;
}

int cg_merkle_log_consistency_between_device(cg_merkle_log* L, uint64_t first_size, uint64_t second_size, void* d_out_path32, uint32_t path_cap,
                                             void* d_out_len, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!d_out_len) return fail(CG_ERR_INVALID_ARG, "null argument");
  if ((rc = check_aligned(d_out_len, 4, "d_out_len")) || (rc = check_aligned(d_out_path32, 16, "d_out_path32"))) return rc;
  if (!L->tree) return fail(CG_ERR_UNSUPPORTED, "proofs at any tree size need a log made by cg_merkle_log_create_tree");
  if (second_size == 0 || second_size > L->n || first_size == 0 || first_size > second_size)
    return fail(CG_ERR_INVALID_ARG, "need 1 <= first_size <= second_size <= size of the log");
  const uint32_t len = (uint32_t)proof_ranges(0, second_size, first_size).size();
  if (len > path_cap || (len && !d_out_path32)) return fail(CG_ERR_CAPACITY, "path buffer too small");
  const cudaStream_t st = caller_stream(stream);
  InOrder turn(&L->order, st), dig(&G.dig_order, st);
  if ((rc = turn.rc) || (rc = dig.rc)) return rc;
  if (!len) { CU(cudaMemsetAsync(d_out_len, 0, 4, st)); return CG_OK; }
  if ((rc = log_spine(L, second_size, st))) return rc;
  count_launches(launch_merkle_gather(log_store(L), L->d_spine.get(), second_size, nullptr, first_size, 1, len, (uint32_t*)d_out_path32, (uint32_t*)d_out_len,
                                      G.sm_count, st));
  CU(cudaGetLastError());
  return CG_OK;
}

int cg_merkle_verify_proofs_device(const void* d_leaf_bytes, const void* d_leaf_offsets, const void* d_indices, uint32_t m, uint64_t tree_size,
                                   const void* d_paths32, uint32_t path_stride, const void* d_path_lens, const void* d_root32, void* d_out_ok, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!m) return CG_OK;
  if (!d_leaf_bytes || !d_leaf_offsets || !d_indices || !d_path_lens || !d_root32 || !d_out_ok || (path_stride && !d_paths32))
    return fail(CG_ERR_INVALID_ARG, "null argument");
  int rc;
  if ((rc = check_aligned(d_leaf_bytes, 16, "d_leaf_bytes")) || (rc = check_aligned(d_leaf_offsets, 8, "d_leaf_offsets")) ||
      (rc = check_aligned(d_indices, 8, "d_indices")) || (rc = check_aligned(d_paths32, 16, "d_paths32")) ||
      (rc = check_aligned(d_path_lens, 4, "d_path_lens"))) return rc;
  const cudaStream_t st = caller_stream(stream);
  InOrder turn(&G.dig_order, st);
  if ((rc = turn.rc)) return rc;
  // d_dig[0]: leaf digests | root (the caller's root copied, so that it may have any alignment)
  if ((rc = G.d_dig[0].grow((size_t)m * 8 + 8))) return rc;
  uint32_t* d_leaf = G.d_dig[0].get(); uint32_t* d_root = d_leaf + (size_t)m * 8;
  CU(cudaMemcpyAsync(d_root, d_root32, 32, cudaMemcpyDeviceToDevice, st));
  const uint64_t* d_off = (const uint64_t*)d_leaf_offsets;
  int k = launch_merkle_leaves_guarded((const uint8_t*)d_leaf_bytes, d_off, m, d_leaf, nullptr, st);
  k += launch_merkle_verify_batch(d_leaf, (const uint64_t*)d_indices, m, tree_size, (const uint32_t*)d_paths32, path_stride, (const uint32_t*)d_path_lens,
                                  d_root, (uint8_t*)d_out_ok, G.sm_count, st, d_off);
  count_launches(k);
  CU(cudaGetLastError());
  return CG_OK;
}

int cg_merkle_log_join(cg_merkle_log* L, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  CU(cudaStreamSynchronize(caller_stream(stream)));
  CU(cudaEventSynchronize(L->order.ev));                    // (every call issued on the log has run: each one ran behind the one before)
  uint32_t err = 0;
  CU(cudaMemcpyAsync(&err, L->d_err.get(), 4, cudaMemcpyDeviceToHost, G.stream));
  CU(cudaStreamSynchronize(G.stream));
  if (err) {
    L->failed = true;
    return fail(CG_ERR_INVALID_ARG, "a device append read a decreasing offset pair: that leaf went in as the empty leaf, and the log refuses every further call");
  }
  return CG_OK;
}

// ---------------------------------------------------------------------------------- multi-GPU: one process per GPU
// The scan shards by message with no exchange at all (cg_shard_range is the split rule).  The Merkle tree has ONE exchange:
// every rank's roots of aligned 2^k-leaf blocks are all-gathered and every rank folds the same list.  NCCL is bound at run
// time (dlopen of the process's libnccl.so.2 -- the one the host framework has loaded, if any) so that a single-GPU
// deployment has no such dependency.
void cg_shard_range(uint64_t n, int rank, int world, uint64_t align, uint64_t* lo, uint64_t* hi) {
  if (align == 0) align = 1;
  if (world < 1) world = 1;
  const uint64_t blocks = (n + align - 1) / align;
  const uint64_t lo_b = (uint64_t)((unsigned __int128)blocks * (unsigned)rank / (unsigned)world), hi_b = (uint64_t)((unsigned __int128)blocks * (unsigned)(rank + 1) / (unsigned)world);
  if (lo) *lo = std::min(lo_b * align, n);
  if (hi) *hi = std::min(hi_b * align, n);
}

namespace {
int nccl_load() {
  if (g_nccl.h) return CG_OK;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return fail(CG_ERR_UNSUPPORTED, std::string("NCCL not found: ") + dlerror());
  g_nccl.GetUniqueId = (int (*)(void*))dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (int (*)(void**, int, cg_nccl_id, int))dlsym(h, "ncclCommInitRank");
  g_nccl.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(h, "ncclAllGather");
  g_nccl.CommDestroy = (int (*)(void*))dlsym(h, "ncclCommDestroy");
  g_nccl.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllGather || !g_nccl.CommDestroy) { dlclose(h); return fail(CG_ERR_UNSUPPORTED, "NCCL symbols missing"); }
  g_nccl.h = h;
  return CG_OK;
}
int nccl_fail(int rc, const char* what) { return fail(CG_ERR_CUDA, std::string(what) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "NCCL error")); }
}  // namespace

int cg_comm_unique_id(cg_nccl_id* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!out) return fail(CG_ERR_INVALID_ARG, "null argument");
  int rc = nccl_load(); if (rc) return rc;
  int r = g_nccl.GetUniqueId(out); if (r) return nccl_fail(r, "ncclGetUniqueId");
  return CG_OK;
}
int cg_comm_init(int rank, int world, const cg_nccl_id* id) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!id || world < 1 || rank < 0 || rank >= world) return fail(CG_ERR_INVALID_ARG, "bad rank / world / id");
  int rc = nccl_load(); if (rc) return rc;
  if (g_nccl.comm) { g_nccl.CommDestroy(g_nccl.comm); g_nccl.comm = nullptr; }
  int r = g_nccl.CommInitRank(&g_nccl.comm, world, *id, rank); if (r) return nccl_fail(r, "ncclCommInitRank");
  g_nccl.rank = rank; g_nccl.world = world;
  return CG_OK;
}
void cg_comm_destroy(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_nccl.comm && g_nccl.CommDestroy) { if (G.ready) cudaStreamSynchronize(G.stream); g_nccl.CommDestroy(g_nccl.comm); }
  G.d_roots.reset();
  g_nccl.comm = nullptr; g_nccl.world = 1; g_nccl.rank = 0;
}

/* Root of the tree over the leaves of ALL ranks (rank r holds leaves [lo_r, hi_r) of cg_shard_range(n_total, r, world, 2^block_log2),
 * device-resident): block roots here, one all-gather of (count, roots) per rank, the same fold on every rank.  The all-gather runs
 * outside the library lock (its first call may wait for the peers to connect) on the communicator's root buffer. */
int cg_merkle_root_sharded_device(const void* d_bytes, uint64_t leaf_len, uint64_t n_local, uint64_t n_total, uint32_t block_log2, uint8_t out_root[32], void* stream) {
  std::unique_lock<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!out_root || block_log2 > 40) return fail(CG_ERR_INVALID_ARG, "bad argument");
  const int rank = g_nccl.rank, world = g_nccl.world; void* const comm = g_nccl.comm;
  if (world > 1 && !comm) return fail(CG_ERR_NOT_INITIALIZED, "cg_comm_init has not been called");
  uint64_t lo, hi; cg_shard_range(n_total, rank, world, 1ull << block_log2, &lo, &hi);
  if (hi - lo != n_local) return fail(CG_ERR_INVALID_ARG, "n_local is not this rank's share of n_total (cg_shard_range with align = 2^block_log2)");
  if (n_local && !d_bytes) return fail(CG_ERR_INVALID_ARG, "null argument");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream;
  // every rank contributes max_blocks slots (its own roots first); the counts follow from the split rule, no second exchange
  uint64_t max_blocks = 0, total_blocks = 0; std::vector<uint64_t> nblk((size_t)world);
  for (int r = 0; r < world; r++) { uint64_t a, b; cg_shard_range(n_total, r, world, 1ull << block_log2, &a, &b); nblk[(size_t)r] = (b - a + (1ull << block_log2) - 1) >> block_log2; max_blocks = std::max(max_blocks, nblk[(size_t)r]); total_blocks += nblk[(size_t)r]; }
  if (max_blocks == 0) return empty_root(out_root);
  int rc;
  if ((rc = G.d_roots.grow((size_t)world * max_blocks * 8))) return rc;
  uint32_t* const all = G.d_roots.get(); uint32_t* const mine = all + (size_t)rank * max_blocks * 8;   // (an in-place all-gather)
  CU(cudaMemsetAsync(mine, 0, max_blocks * 32, st));
  if (n_local && (rc = block_roots(d_bytes, leaf_len, n_local, block_log2, mine, st))) return rc;
  if (world > 1) {
    lk.unlock(); const int r = g_nccl.AllGather(mine, all, max_blocks * 32, /*ncclChar*/ 0, comm, st); lk.lock();
    if (r) return nccl_fail(r, "ncclAllGather");
    // (a cg_shutdown, cg_comm_destroy or other sharded call during the gather is misuse, but must not make the fold read freed memory)
    if (!G.ready || G.d_roots.get() != all) return fail(CG_ERR_NOT_INITIALIZED, "the library or the communicator's buffer changed during the all-gather");
  }
  const uint32_t* d_root;                                   // the fold's input: the gathered roots without the empty slots
  InOrder turn(&G.dig_order, st);                           // (block_roots took its own turn: the lock was let go since)
  if ((rc = turn.rc)) return rc;
  if ((rc = size_dig(total_blocks))) return rc;
  uint32_t* d = G.d_dig[0].get();
  for (int r = 0; r < world; r++) if (nblk[(size_t)r]) { CU(cudaMemcpyAsync(d, all + (size_t)r * max_blocks * 8, nblk[(size_t)r] * 32, cudaMemcpyDeviceToDevice, st)); d += nblk[(size_t)r] * 8; }
  if ((rc = fold_dig(G.d_dig[0].get(), total_blocks, 64, st, &d_root))) return rc;
  CU(cudaMemcpyAsync(out_root, d_root, 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}

}  // extern "C"
