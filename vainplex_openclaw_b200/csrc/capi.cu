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
#include <vector>

#include "../../include/openclaw_gov.h"
#include "kernels.h"
#include "rulec.h"
#include "ruleset_image.h"

using namespace cg;

namespace {

thread_local std::string g_err;
std::mutex g_mu;

struct Ctx {
  bool ready = false;
  int device = 0, sm_count = 132;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaEvent_t pev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t pev_scan[8] = {};      // profiling: begin / end of scan_kernel for each of the (at most four) pieces of a step
  uint32_t prof_pieces = 0;
  bool profiling = false;
  cg_stats stats{};
  // grow-only staging in HBM
  uint8_t* d_bytes = nullptr; size_t cap_bytes = 0; uint8_t* d_bytes_raw = nullptr;   // d_bytes = d_bytes_raw + 256: readable in front (sha_words)
  uint32_t* d_off32 = nullptr; size_t cap_off32 = 0;
  uint64_t* d_off64 = nullptr; size_t cap_off64 = 0;
  uint64_t* d_words = nullptr; size_t cap_words = 0;
  uint32_t* d_dig[2] = {nullptr, nullptr}; size_t cap_dig[2] = {0, 0};
  // chunked host-buffer scans: H2D of chunk c+1 and D2H of chunk c-1 overlap the kernels of chunk c
  static constexpr int kChunks = 8;
  cudaStream_t s_h2d = nullptr, s_d2h = nullptr; cudaEvent_t e_h2d[kChunks] = {}, e_done[kChunks] = {}; uint32_t* h_chunk_counters = nullptr;
  // cg_find_matches_batch / cg_redact_batch / cg_policy_verdict_batch staging (grow-only)
  cg_span* d_spans = nullptr; size_t cap_spans = 0;
  uint8_t* d_redact_out = nullptr; size_t cap_redact_out = 0; uint32_t* d_redact_meta = nullptr; size_t cap_redact_meta = 0;
  uint32_t* d_verdicts = nullptr; size_t cap_verdicts = 0;
} G;

int fail(int code, const std::string& msg) { g_err = msg; return code; }
int cuda_fail(cudaError_t e, const char* what) {
  g_err = std::string(what) + ": " + cudaGetErrorString(e);
  return CG_ERR_CUDA;
}
#define CU(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return cuda_fail(_e, #x); } while (0)
int require_ready() { return G.ready ? CG_OK : fail(CG_ERR_NOT_INITIALIZED, "cg_init has not been called (or no CUDA device)"); }
void count_launches(int k) { G.stats.kernel_launches += k; }

// NCCL, bound at run time (nccl_load), and the communicator of cg_comm_init
struct NcclApi {
  void* h = nullptr; void* comm = nullptr; int rank = 0, world = 1;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, cg_nccl_id, int) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  uint32_t* d_roots = nullptr; size_t cap_roots = 0;     // cg_merkle_root_sharded_device: every rank's block roots (grow-only)
} g_nccl;
void free_shard_roots() { if (g_nccl.d_roots) cudaFree(g_nccl.d_roots); g_nccl.d_roots = nullptr; g_nccl.cap_roots = 0; }

template <typename T>
int grow(T** p, size_t* cap, size_t need_elems) {
  if (need_elems <= *cap && *p) return CG_OK;
  if (*p) cudaFree(*p);
  *p = nullptr; *cap = 0;
  size_t n = need_elems + need_elems / 4 + 64;
  cudaError_t e = cudaMalloc((void**)p, n * sizeof(T));
  if (e != cudaSuccess) { *p = nullptr; return cuda_fail(e, "cudaMalloc"); }
  *cap = n;
  return CG_OK;
}

// the staging buffer for message / leaf bytes: 256 readable bytes in front of it and 64 + slack behind what is asked for
int grow_bytes(size_t need) {
  if (need <= G.cap_bytes && G.d_bytes) return CG_OK;
  if (G.d_bytes_raw) cudaFree(G.d_bytes_raw);
  G.d_bytes_raw = G.d_bytes = nullptr; G.cap_bytes = 0;
  const size_t n = need + need / 4 + 64;
  cudaError_t e = cudaMalloc((void**)&G.d_bytes_raw, n + 512);
  if (e != cudaSuccess) { G.d_bytes_raw = nullptr; return cuda_fail(e, "cudaMalloc"); }
  cudaMemset(G.d_bytes_raw, 0, 256);
  G.d_bytes = G.d_bytes_raw + 256; G.cap_bytes = n;
  return CG_OK;
}

}  // namespace

struct cg_ruleset {
  HostImage host;
  std::vector<uint32_t> category;
  DevRuleset dev{};
  std::vector<void*> allocs;
  uint32_t n_sets = 0, program_words = 0;
  ScanWork work{};
  uint64_t seq = 0;               // device-path batches issued so far
  // device path: every batch's counters are mirrored into a ring of pinned slots, so that a queue overflow (results of
  // that batch marked incomplete by finalize_kernel) is seen by the next call / by cg_scan_join and the scratch grows
  static constexpr int kMirror = 16;
  uint32_t* h_counters = nullptr; cudaEvent_t e_cnt[kMirror] = {}; bool cnt_pending[kMirror] = {};
  uint32_t grow_l1 = 0, grow_slot = 0, grow_ev = 0, grow_span = 0;     // capacities learnt from overflows
  uint32_t sticky_flags = 0;      // error flags of batches since the last cg_scan_join
  uint32_t sticky_status = 0;     // 1 << span resolution status (kResolve*) of batches since the last cg_scan_join
  // verify_small_kernel's grid (CTAs per SM): one while the island matcher decides (nearly) everything, four once a step has
  // sent more than 2048 pairs to the VM (non-ASCII traffic); back to one below 256.  Part of the cached graphs' keys.
  int verify_ctas = 1;
  void size_verify_grid() { const uint32_t ev = last_counters[1]; if (ev > 2048u) verify_ctas = 4; else if (ev < 256u) verify_ctas = 1; }
  uint32_t last_counters[kCounterWords] = {};
  uint64_t scratch_gen = 0;       // advanced by every change to what a captured step holds (scratch buffers, DevRuleset)
  // the device-resident step replayed as one CUDA graph (keyed on its arguments, the scratch generation and the verify grid)
  struct CachedGraph { int kernels = 0; cudaGraphExec_t exec = nullptr; const void* bytes = nullptr; const void* off = nullptr; void* words = nullptr; uint32_t n = 0; uint64_t gen = 0; int ctas = 0; uint64_t used = 0; };
  // cg_scan_one: pinned staging + one device block ([offsets][message bytes] in, [word][counters][hit row] out) and the
  // step as a graph over those fixed addresses (the message length is data, so one graph serves every message)
  struct OnePath { cudaGraphExec_t exec = nullptr; uint8_t* h_pin = nullptr; uint8_t* d_buf = nullptr; uint64_t gen = 0; int ctas = 0; int kernels = 0; } one;
  CachedGraph graphs[2];          // two entries: callers that alternate between two input/output buffer sets replay, never re-capture
  uint64_t graph_clock = 0;
  ~cg_ruleset() {
    for (auto& g : graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    if (one.exec) cudaGraphExecDestroy(one.exec);
    if (one.h_pin) cudaFreeHost(one.h_pin);
    cudaFree(one.d_buf);
    if (h_counters) cudaFreeHost(h_counters);
    for (auto& e : e_cnt) if (e) cudaEventDestroy(e);
    for (void* p : allocs) cudaFree(p);
    cudaFree(work.heavy_idx); cudaFree(work.l1_pos); cudaFree(work.l1_fac); cudaFree(work.fq); cudaFree(work.slot_of_msg);
    cudaFree(work.counters); cudaFree(work.persist); cudaFree(work.slot_msg); cudaFree(work.cand); cudaFree(work.hit); cudaFree(work.events); cudaFree(work.event_pos); cudaFree(work.event_pre); cudaFree(work.spans);
    cudaFree(work.words); cudaFree(work.seg_cnt); cudaFree(work.seg_begin); cudaFree(work.kept_cnt); cudaFree(work.kept_begin); cudaFree(work.out_len); cudaFree(work.out_off);
    cudaFree(work.sorted); cudaFree(work.sort_tmp); cudaFree(work.sp_start); cudaFree(work.sp_len); cudaFree(work.sp_cat); cudaFree(work.scan_part);
  }
};

namespace {

template <typename T>
int upload(cg_ruleset* rs, const std::vector<T>& v, const T** out, size_t pad_elems = 4) {
  void* d = nullptr;
  size_t bytes = (v.size() + pad_elems) * sizeof(T);
  CU(cudaMalloc(&d, bytes));
  rs->allocs.push_back(d);
  CU(cudaMemset(d, 0, bytes));
  if (!v.empty()) CU(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  *out = reinterpret_cast<const T*>(d);
  return CG_OK;
}

// (res_msgs: messages the span resolver must have room for; 0 for a step without spans)
int ensure_work(cg_ruleset* rs, ScanWork& w, uint32_t n_msgs, uint32_t l1_cap, uint32_t slot_cap, uint32_t event_cap, uint32_t span_cap, uint32_t res_msgs) {
  rs->scratch_gen++;                                        // (prepare_step calls this only when some buffer must grow)
  if (!w.counters) { CU(cudaMalloc((void**)&w.counters, kCounterWords * sizeof(uint32_t))); CU(cudaMalloc((void**)&w.persist, 16)); CU(cudaMemset(w.persist, 0, 16)); CU(cudaDeviceSynchronize()); }
  if (n_msgs > w.msg_cap) { cudaFree(w.slot_of_msg); w.slot_of_msg = nullptr; w.msg_cap = 0; CU(cudaMalloc((void**)&w.slot_of_msg, (size_t)n_msgs * 4)); w.msg_cap = n_msgs; }
  if (l1_cap > w.l1_cap) {
    cudaFree(w.l1_pos); cudaFree(w.l1_fac); cudaFree(w.fq); w.l1_pos = w.l1_fac = nullptr; w.fq = nullptr; w.l1_cap = 0;
    CU(cudaMalloc((void**)&w.l1_pos, (size_t)l1_cap * 4)); CU(cudaMalloc((void**)&w.l1_fac, (size_t)l1_cap * 4)); CU(cudaMalloc((void**)&w.fq, (size_t)l1_cap * 8));
    w.l1_cap = l1_cap;
  }
  if (slot_cap > w.slot_cap) {
    cudaFree(w.slot_msg); cudaFree(w.cand); cudaFree(w.hit); w.slot_msg = w.cand = w.hit = nullptr; w.slot_cap = 0;
    size_t rw = rs->dev.rw ? rs->dev.rw : 1;
    CU(cudaMalloc((void**)&w.slot_msg, (size_t)slot_cap * 4));
    CU(cudaMalloc((void**)&w.cand, (size_t)slot_cap * rw * 4));
    CU(cudaMalloc((void**)&w.hit, (size_t)slot_cap * rw * 4));
    // rows start out zero and every step clears the ones it used (reset_kernel)
    CU(cudaMemset(w.cand, 0, (size_t)slot_cap * rw * 4)); CU(cudaMemset(w.hit, 0, (size_t)slot_cap * rw * 4)); CU(cudaMemset(w.persist, 0, 16)); CU(cudaDeviceSynchronize());
    w.slot_cap = slot_cap;
  }
  if (event_cap > w.event_cap) { cudaFree(w.events); cudaFree(w.event_pos); cudaFree(w.event_pre); cudaFree(w.heavy_idx); w.events = nullptr; w.event_pos = w.event_pre = w.heavy_idx = nullptr; w.event_cap = 0; CU(cudaMalloc((void**)&w.events, (size_t)event_cap * sizeof(uint2))); CU(cudaMalloc((void**)&w.heavy_idx, (size_t)event_cap * 4)); CU(cudaMalloc((void**)&w.event_pos, (size_t)event_cap * 4)); CU(cudaMalloc((void**)&w.event_pre, (size_t)event_cap * 4)); w.event_cap = event_cap; }
  if (span_cap > w.span_cap) {
    cudaFree(w.spans); cudaFree(w.sorted); cudaFree(w.sort_tmp); cudaFree(w.sp_start); cudaFree(w.sp_len); cudaFree(w.sp_cat);
    w.spans = w.sp_start = w.sp_len = w.sp_cat = nullptr; w.sorted = w.sort_tmp = nullptr; w.span_cap = 0;
    CU(cudaMalloc((void**)&w.spans, (size_t)span_cap * 24));
    CU(cudaMalloc((void**)&w.sorted, (size_t)span_cap * 16)); CU(cudaMalloc((void**)&w.sort_tmp, (size_t)span_cap * 16));
    CU(cudaMalloc((void**)&w.sp_start, (size_t)span_cap * 4)); CU(cudaMalloc((void**)&w.sp_len, (size_t)span_cap * 4)); CU(cudaMalloc((void**)&w.sp_cat, (size_t)span_cap * 4));
    w.span_cap = span_cap;
  }
  if (res_msgs > w.res_cap || (res_msgs && !w.scan_part)) {
    cudaFree(w.words); cudaFree(w.seg_cnt); cudaFree(w.seg_begin); cudaFree(w.kept_cnt); cudaFree(w.kept_begin); cudaFree(w.out_len); cudaFree(w.out_off);
    w.words = w.out_len = w.out_off = nullptr; w.seg_cnt = w.seg_begin = w.kept_cnt = w.kept_begin = nullptr; w.res_cap = 0;
    const size_t m = (size_t)res_msgs + 1;
    CU(cudaMalloc((void**)&w.words, m * 8)); CU(cudaMalloc((void**)&w.out_len, m * 8)); CU(cudaMalloc((void**)&w.out_off, m * 8));
    CU(cudaMalloc((void**)&w.seg_cnt, m * 4)); CU(cudaMalloc((void**)&w.seg_begin, m * 4)); CU(cudaMalloc((void**)&w.kept_cnt, m * 4)); CU(cudaMalloc((void**)&w.kept_begin, m * 4));
    if (!w.scan_part) CU(cudaMalloc((void**)&w.scan_part, (size_t)kScanPartials * 8));
    w.res_cap = res_msgs;
  }
  return CG_OK;
}

static uint32_t scan_pieces() { static const uint32_t k = [] { const char* e = getenv("CG_PIECES"); const int v = e ? atoi(e) : 1; return (uint32_t)(v >= 1 && v <= 4 ? v : 1); }(); return k; }
// One step on device-resident input: scratch reset, gram scan (+ exact factors), resolve, verify, finalize.  Asynchronous.
int run_scan_device(cg_ruleset* rs, const uint8_t* d_bytes, const uint32_t* d_off, uint32_t n, uint64_t* d_words, bool spans, cudaStream_t st) {
  const ScanWork& w = rs->work;
  int k = launch_reset(rs->dev, w, n, G.sm_count, st);
  if (G.profiling) cudaEventRecord(G.pev[0], st);
  // CG_PIECES = 2..4 scans the batch in pieces, each followed by its own lookup + check, so that a flagged gram is read again
  // while its piece is still in the 50 MB L2.  Every extra launch of the latency-bound kernels costs time the L2 hits have to
  // win back.  One piece unless asked otherwise.
  const uint32_t K = scan_pieces();
  if (G.profiling) G.prof_pieces = K;
  for (uint32_t piece = 0; piece < K; piece++) {
    const uint32_t m0 = (uint32_t)((uint64_t)n * piece / K), m1 = (uint32_t)((uint64_t)n * (piece + 1) / K);
    if (m1 == m0) continue;
    ScanWork wk = w; wk.q_cap = w.l1_cap / K; wk.q_slot = piece; wk.fq = w.fq + (size_t)piece * wk.q_cap;
    if (G.profiling) cudaEventRecord(G.pev_scan[2 * piece], st);
    k += launch_scan(rs->dev, wk, d_bytes, d_off + m0, m1 - m0, d_words + m0, G.sm_count, st);
    if (G.profiling) cudaEventRecord(G.pev_scan[2 * piece + 1], st);
    k += launch_confirm(rs->dev, wk, d_bytes, d_off + m0, m1 - m0, G.sm_count, st);
  }
  if (G.profiling) cudaEventRecord(G.pev[1], st);
  k += launch_resolve(rs->dev, w, d_bytes, d_off, n, spans, G.sm_count, st);
  if (G.profiling) cudaEventRecord(G.pev[2], st);
  k += launch_verify(rs->dev, w, d_bytes, d_off, spans, G.sm_count, st, spans ? 4 : rs->verify_ctas);
  if (G.profiling) cudaEventRecord(G.pev[3], st);
  k += launch_finalize(rs->dev, w, d_words, n, G.sm_count, st);
  if (G.profiling) cudaEventRecord(G.pev[4], st);
  count_launches(k);
  CU(cudaGetLastError());
  return CG_OK;
}

void prepare_kernels() { static bool done = false; if (!done) { prepare_scan_kernels(); done = true; } }

// capacities a batch of n messages starts with (confirmed occurrences are rare: about one per hundred messages on chat text;
// a step without spans writes none)
void default_caps(const cg_ruleset* rs, uint32_t n, bool spans, uint32_t* l1, uint32_t* slot, uint32_t* ev, uint32_t* span) {
  *l1 = std::max(std::max<uint32_t>(std::max<uint32_t>(2 * n, 1u << 16), rs->work.l1_cap), rs->grow_l1);
  *slot = std::max(std::max<uint32_t>(std::max<uint32_t>(n / 4, 4096), rs->work.slot_cap), rs->grow_slot);
  *ev = std::max(std::max<uint32_t>(std::max<uint32_t>(n, 4096), rs->work.event_cap), rs->grow_ev);
  *span = spans ? std::max(std::max<uint32_t>(std::max<uint32_t>(n, 4096), rs->work.span_cap), rs->grow_span) : 1;
}
// the verify grid and the scratch of a step over n messages; growing waits for st (nothing may still use a replaced buffer)
int prepare_step(cg_ruleset* rs, uint32_t n, bool spans, cudaStream_t st) {
  rs->size_verify_grid();
  const ScanWork& w = rs->work;
  uint32_t l1, slot, ev, span;
  default_caps(rs, n, spans, &l1, &slot, &ev, &span);
  n = std::max<uint32_t>(n, 1);
  const uint32_t res = spans ? n : 0;
  if (n <= w.msg_cap && l1 <= w.l1_cap && slot <= w.slot_cap && ev <= w.event_cap && span <= w.span_cap && res <= w.res_cap) return CG_OK;
  CU(cudaStreamSynchronize(st));
  return ensure_work(rs, rs->work, n, l1, slot, ev, span, res);
}
// fq is cut into four equal pieces at most: the fullest piece decides
static uint32_t queue_need(const uint32_t* hc) { uint32_t m = 0; for (int i = 24; i < 28; i++) m = std::max(m, hc[i]); return m > 0xffffffffu / scan_pieces() ? 0xffffffffu : scan_pieces() * m; }
// what an overflowed step teaches about the capacities the next one needs
void learn_caps(cg_ruleset* rs, const uint32_t* hc) {
  const uint32_t flags = hc[3];
  if (flags & ERR_L1_OVERFLOW) { const uint32_t need = std::max(hc[4], queue_need(hc)); rs->grow_l1 = std::max<uint32_t>(rs->grow_l1, std::max<uint32_t>(2 * need, need + 65536)); }
  if (flags & ERR_SLOT_OVERFLOW) rs->grow_slot = std::max<uint32_t>(rs->grow_slot, std::max<uint32_t>(2 * hc[0], hc[0] + 4096));
  if (flags & ERR_EVENT_OVERFLOW) rs->grow_ev = std::max<uint32_t>(rs->grow_ev, std::max<uint32_t>(2 * hc[1], hc[1] + 4096));
  if (flags & ERR_SPAN_OVERFLOW) rs->grow_span = std::max<uint32_t>(rs->grow_span, std::max<uint32_t>(2 * hc[2], hc[2] + 4096));
}
const char* const kVmOverflow = "matcher thread list / stack overflow on device";
// a finished step's counter block -> CG_OK, CG_ERR_TOO_LARGE, or 1 = a queue overflowed (the capacities the step needs
// have been learnt)
int absorb_counters(cg_ruleset* rs, const uint32_t* hc) {
  memcpy(rs->last_counters, hc, sizeof rs->last_counters);
  if (hc[3] & (ERR_VM_STACK | ERR_VM_LIST)) return fail(CG_ERR_TOO_LARGE, kVmOverflow);
  if (hc[3]) learn_caps(rs, hc);
  return hc[3] ? 1 : CG_OK;
}
// the kernels enqueue() puts on st, captured as one graph; they are counted each time the graph is launched, not here
template <typename Enqueue>
int capture(cudaStream_t st, Enqueue&& enqueue, cudaGraphExec_t* exec, int* kernels) {
  cudaGraph_t g = nullptr;
  const uint64_t before = G.stats.kernel_launches;
  CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  const int rc = enqueue();
  cudaError_t e = cudaStreamEndCapture(st, &g);
  *kernels = (int)(G.stats.kernel_launches - before); G.stats.kernel_launches = before;
  if (rc != CG_OK || e != cudaSuccess) { if (g) cudaGraphDestroy(g); cudaGetLastError(); return rc != CG_OK ? rc : cuda_fail(e, "cudaStreamEndCapture"); }
  e = cudaGraphInstantiate(exec, g, 0);
  cudaGraphDestroy(g);
  if (e != cudaSuccess) { *exec = nullptr; return cuda_fail(e, "cudaGraphInstantiate"); }
  return CG_OK;
}
// the rules of one hit row (rw words), lowest first: put(i, rule) for the i-th rule of the output while i < cap; returns nh
// plus the number of rules in the row
template <typename Put>
uint32_t append_hit_row(const uint32_t* row, uint32_t rw, uint32_t nh, uint32_t cap, Put&& put) {
  for (uint32_t k = 0; k < rw; k++)
    for (uint32_t v = row[k]; v; v &= v - 1, nh++) if (nh < cap) put(nh, k * 32 + (uint32_t)__builtin_ctz(v));
  return nh;
}

struct HostScan {
  std::vector<uint32_t> counters, slot_msg, hit, spans;
};

int check_offsets(const uint32_t* offsets, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) if (offsets[i + 1] < offsets[i]) return fail(CG_ERR_INVALID_ARG, "offsets must be non-decreasing");
  return CG_OK;
}

// full host-buffer scan with capacity retry; leaves words in G.d_words (a span-mode step: in the rule set's scratch)
int scan_host(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, bool spans, HostScan* hs) {
  if (int rc = require_ready()) return rc;
  if (!rs || (n && (!bytes || !offsets))) return fail(CG_ERR_INVALID_ARG, "null argument");
  int rc;
  if (n && (rc = check_offsets(offsets, n))) return rc;
  const size_t first = n ? offsets[0] : 0, total = n ? offsets[n] : 0;
  if ((rc = grow_bytes(total + 64))) return rc;
  if ((rc = grow(&G.d_off32, &G.cap_off32, (size_t)n + 1))) return rc;
  if ((rc = grow(&G.d_words, &G.cap_words, (size_t)n + 1))) return rc;
  cudaStream_t st = G.stream;
  if (n) {
    if (total > first) CU(cudaMemcpyAsync(G.d_bytes + first, bytes + first, total - first, cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(G.d_bytes + total, 0, 64, st));
    CU(cudaMemcpyAsync(G.d_off32, offsets, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, st));
  }
  hs->counters.assign(kCounterWords, 0);
  for (int attempt = 0; attempt < 10; attempt++) {
    if ((rc = prepare_step(rs, n, spans, st))) return rc;
    CU(cudaEventRecord(G.ev0, st));
    if (n) { if ((rc = run_scan_device(rs, G.d_bytes, G.d_off32, n, spans ? rs->work.words : G.d_words, spans, st))) return rc; }
    else CU(cudaMemsetAsync(rs->work.counters, 0, kCounterWords * sizeof(uint32_t), st));
    CU(cudaEventRecord(G.ev1, st));
    CU(cudaMemcpyAsync(hs->counters.data(), rs->work.counters, kCounterWords * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    float ms = 0; cudaEventElapsedTime(&ms, G.ev0, G.ev1); G.stats.last_scan_ms = ms;
    if ((rc = absorb_counters(rs, hs->counters.data())) == 1) continue;
    if (rc) return rc;
    G.stats.messages_scanned += n; G.stats.bytes_scanned += total - first;
    G.stats.candidate_events += hs->counters[1]; G.stats.verified_pairs += hs->counters[1];
    return CG_OK;
  }
  return fail(CG_ERR_CAPACITY, "candidate queues kept overflowing");
}

int ensure_copy_streams() {
  if (G.s_h2d) return CG_OK;
  const int C = Ctx::kChunks;
  CU(cudaStreamCreateWithFlags(&G.s_h2d, cudaStreamNonBlocking)); CU(cudaStreamCreateWithFlags(&G.s_d2h, cudaStreamNonBlocking));
  for (int c = 0; c < C; c++) { CU(cudaEventCreateWithFlags(&G.e_h2d[c], cudaEventDisableTiming)); CU(cudaEventCreateWithFlags(&G.e_done[c], cudaEventDisableTiming)); }
  CU(cudaMallocHost((void**)&G.h_chunk_counters, (size_t)C * kCounterWords * 4));
  return CG_OK;
}

// Words-only scan of a large host batch in kChunks pieces: the H2D copy of piece c+1 and the D2H copy of piece c-1 run
// on their own streams while the kernels of piece c run -- end to end the call then costs little more than the H2D copy
// alone.  Returns 1 when a queue overflowed somewhere (capacities have been grown; the caller re-runs in one piece).
int scan_host_chunked(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint64_t* out_words) {
  const int C = Ctx::kChunks;
  int rc;
  if ((rc = check_offsets(offsets, n))) return rc;
  const size_t total = offsets[n];
  if ((rc = grow_bytes(total + 64))) return rc;
  if ((rc = grow(&G.d_off32, &G.cap_off32, (size_t)n + 1))) return rc;
  if ((rc = grow(&G.d_words, &G.cap_words, (size_t)n + 1))) return rc;
  if ((rc = ensure_copy_streams())) return rc;
  cudaStream_t st = G.stream;
  const uint32_t per = (n + C - 1) / C;
  CU(cudaStreamSynchronize(st));                            // (whatever still read the staging buffers is done: s_h2d does not wait for st)
  if ((rc = prepare_step(rs, per, false, st))) return rc;
  CU(cudaMemcpyAsync(G.d_off32, offsets, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, G.s_h2d));
  CU(cudaMemsetAsync(G.d_bytes + total, 0, 64, G.s_h2d));
  CU(cudaEventRecord(G.ev0, st));
  int used = 0;
  for (int c = 0; c < C; c++) {
    const uint32_t m0 = std::min<uint64_t>((uint64_t)c * per, n), m1 = std::min<uint64_t>((uint64_t)(c + 1) * per, n);
    if (m1 <= m0) break;
    used = c + 1;
    const size_t b0 = offsets[m0], b1 = offsets[m1];
    if (b1 > b0) CU(cudaMemcpyAsync(G.d_bytes + b0, bytes + b0, b1 - b0, cudaMemcpyHostToDevice, G.s_h2d));
    CU(cudaEventRecord(G.e_h2d[c], G.s_h2d));
    CU(cudaStreamWaitEvent(st, G.e_h2d[c], 0));
    // (a piece reads up to 16 bytes past its last message -- bytes of the next piece that may still be in flight; whatever
    // it sees there cannot produce an occurrence inside its own range)
    if ((rc = run_scan_device(rs, G.d_bytes, G.d_off32 + m0, m1 - m0, G.d_words + m0, false, st))) return rc;
    CU(cudaMemcpyAsync(G.h_chunk_counters + (size_t)c * kCounterWords, rs->work.counters, kCounterWords * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(G.e_done[c], st));
    CU(cudaStreamWaitEvent(G.s_d2h, G.e_done[c], 0));
    if (out_words) CU(cudaMemcpyAsync(out_words + m0, G.d_words + m0, (size_t)(m1 - m0) * 8, cudaMemcpyDeviceToHost, G.s_d2h));
  }
  CU(cudaEventRecord(G.ev1, st));
  CU(cudaStreamSynchronize(st)); CU(cudaStreamSynchronize(G.s_d2h)); CU(cudaStreamSynchronize(G.s_h2d));
  float ms = 0; cudaEventElapsedTime(&ms, G.ev0, G.ev1); G.stats.last_scan_ms = ms;
  bool overflow = false;
  uint64_t events = 0;
  for (int c = 0; c < used; c++) {
    const uint32_t* hc = G.h_chunk_counters + (size_t)c * kCounterWords;
    if ((rc = absorb_counters(rs, hc)) < 0) return rc;
    overflow |= rc == 1;
    events += hc[1];
  }
  if (overflow) return 1;
  G.stats.messages_scanned += n; G.stats.bytes_scanned += total - offsets[0];
  G.stats.candidate_events += events; G.stats.verified_pairs += events;
  return CG_OK;
}

// device path: look at every mirrored counter block whose copy has completed
void poll_mirrors(cg_ruleset* rs, bool wait) {
  for (int i = 0; i < cg_ruleset::kMirror; i++) {
    if (!rs->cnt_pending[i]) continue;
    if (wait) cudaEventSynchronize(rs->e_cnt[i]);
    else if (cudaEventQuery(rs->e_cnt[i]) != cudaSuccess) { cudaGetLastError(); continue; }
    rs->cnt_pending[i] = false;
    const uint32_t* hc = rs->h_counters + (size_t)i * kCounterWords;
    rs->sticky_flags |= hc[3];
    if (!hc[3]) rs->sticky_status |= hc[16] ? 1u << hc[16] : 0u;
    G.stats.spans += hc[20]; G.stats.sha256_items += hc[21];     // (zero for words-only steps)
    absorb_counters(rs, hc);                                // (cg_scan_join reports the flags)
  }
}

// device path: the pinned counter mirror ring (allocated by the first device-path call)
int ensure_mirrors(cg_ruleset* rs) {
  if (rs->h_counters) return CG_OK;
  CU(cudaMallocHost((void**)&rs->h_counters, (size_t)cg_ruleset::kMirror * kCounterWords * 4));
  for (auto& e : rs->e_cnt) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  return CG_OK;
}
// device path: copy the counter block of the batch just enqueued on st into the next mirror slot
int mirror_counters(cg_ruleset* rs, cudaStream_t st) {
  const int slot = (int)(rs->seq % cg_ruleset::kMirror);
  if (rs->cnt_pending[slot]) { cudaEventSynchronize(rs->e_cnt[slot]); poll_mirrors(rs, false); }
  CU(cudaMemcpyAsync(rs->h_counters + (size_t)slot * kCounterWords, rs->work.counters, kCounterWords * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(rs->e_cnt[slot], st));
  rs->cnt_pending[slot] = true; rs->seq++;
  return CG_OK;
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
  for (int i = 0; i < 5; i++) CU(cudaEventCreate(&G.pev[i]));
  for (int i = 0; i < 8; i++) CU(cudaEventCreate(&G.pev_scan[i]));

  G.ready = true;
  return CG_OK;
}

void cg_shutdown(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!G.ready) return;
  cudaDeviceSynchronize();
  cudaFree(G.d_spans); cudaFree(G.d_redact_out); cudaFree(G.d_redact_meta); cudaFree(G.d_verdicts);
  if (G.h_chunk_counters) cudaFreeHost(G.h_chunk_counters);
  if (G.s_h2d) { cudaStreamDestroy(G.s_h2d); cudaStreamDestroy(G.s_d2h); for (int c = 0; c < Ctx::kChunks; c++) { cudaEventDestroy(G.e_h2d[c]); cudaEventDestroy(G.e_done[c]); } }
  cudaFree(G.d_bytes_raw); cudaFree(G.d_off32); cudaFree(G.d_off64); cudaFree(G.d_words); cudaFree(G.d_dig[0]); cudaFree(G.d_dig[1]);
  free_shard_roots();
  cudaEventDestroy(G.ev0); cudaEventDestroy(G.ev1); for (int i = 0; i < 5; i++) cudaEventDestroy(G.pev[i]); for (int i = 0; i < 8; i++) cudaEventDestroy(G.pev_scan[i]); cudaStreamDestroy(G.stream);
  G = Ctx();
}

int cg_set_profiling(int on) { G.profiling = on != 0; return CG_OK; }

int cg_last_kernel_ms(float out_ms[4]) {
  // device time of scan / confirm / verify / finalize of the most recent *completed* scan step
  if (!G.ready || !out_ms) return fail(CG_ERR_INVALID_ARG, "not initialised");
  for (int i = 0; i < 4; i++) { out_ms[i] = 0; if (cudaEventElapsedTime(&out_ms[i], G.pev[i], G.pev[i + 1]) != cudaSuccess) { cudaGetLastError(); return fail(CG_ERR_CUDA, "profiling events not recorded / not complete"); } }
  // [0] = scan_kernel alone (summed over the pieces of the step), [1] = everything else before the VM (lookup, check, resolve)
  float scan = 0;
  for (uint32_t p = 0; p < G.prof_pieces; p++) { float t = 0; if (cudaEventElapsedTime(&t, G.pev_scan[2 * p], G.pev_scan[2 * p + 1]) == cudaSuccess) scan += t; else cudaGetLastError(); }
  if (G.prof_pieces) { out_ms[1] += out_ms[0] - scan; out_ms[0] = scan; }
  return CG_OK;
}

int cg_last_tail_ms(float out_ms[2]) {
  // confirm_kernel / resolve_kernel of the most recent completed step in profiling mode (all pieces)
  if (!G.ready || !out_ms) return fail(CG_ERR_INVALID_ARG, "not initialised");
  float scan = 0, pre = 0;
  for (uint32_t p = 0; p < G.prof_pieces; p++) { float t = 0; if (cudaEventElapsedTime(&t, G.pev_scan[2 * p], G.pev_scan[2 * p + 1]) == cudaSuccess) scan += t; else cudaGetLastError(); }
  out_ms[0] = out_ms[1] = 0;
  if (cudaEventElapsedTime(&pre, G.pev[0], G.pev[1]) != cudaSuccess || cudaEventElapsedTime(&out_ms[1], G.pev[1], G.pev[2]) != cudaSuccess) { cudaGetLastError(); return fail(CG_ERR_CUDA, "profiling events not recorded / not complete"); }
  out_ms[0] = pre - scan;
  return CG_OK;
}

int cg_scan_work_counters(const cg_ruleset* rs, uint32_t out16[16]) {
  // [0] slots (messages with confirmed candidates), [1] (message, rule) pairs sent to the VM, [2] spans, [3] error flags,
  // [4] confirmed factor occurrences, [5] verify kernel's event cursor, [6] flagged grams (level 1a) -- of the last step
  // whose counters reached the host (cg_scan_batch: the call itself; device path: after cg_scan_join)
  if (!rs || !out16) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!rs->work.counters) return fail(CG_ERR_INVALID_ARG, "no scan has run");
  memcpy(out16, rs->last_counters, 64);
  if (!(rs->dev.debug_flags & 2u)) { out16[7] = rs->last_counters[19]; out16[8] = out16[9] = 0; for (int i = 0; i < 4; i++) { out16[8] += rs->last_counters[24 + i]; out16[9] += rs->last_counters[28 + i]; } }   // grams past the recheck map, flag words, (gram, entry) pairs
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
  std::vector<RuleSrc> src(n_rules);
  rs->category.resize(n_rules);
  for (uint32_t i = 0; i < n_rules; i++) { src[i] = RuleSrc{rules[i].source, rules[i].source_len, rules[i].flags}; rs->category[i] = rules[i].category; }
  ImageOptions io;
  io.stride = (options & 7u) == CG_OPT_STRIDE2 ? 2 : (options & 7u) == CG_OPT_STRIDE4 ? 4 : 0;
  if (const char* e = getenv("CG_STRIDE")) io.stride = atoi(e);
  if (const char* e = getenv("CG_BITMAP_KB")) io.bitmap_kb = (uint32_t)atoi(e);
  if (const char* e = getenv("CG_BLOOM2")) io.bloom2 = atoi(e);
  if (const char* e = getenv("CG_MAX_KEYS")) io.max_keys = (uint32_t)atoi(e);
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
    static const bool no_smem = getenv("CG_CONFIRM_SMEM") && atoi(getenv("CG_CONFIRM_SMEM")) == 0;
    d.cf_resident = (!no_smem && d.cf_bytes <= kConfirmTableBudget) ? 1u : 0u;
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
  { const uint64_t* fs = nullptr; if ((rc = upload(rs.get(), H.factor_skip, &fs, 8))) return rc; d.factor_skip = getenv("CG_NO_SKIP") ? nullptr : reinterpret_cast<const unsigned long long*>(fs); }
  if (getenv("CG_NO_BITPROG")) d.bit_words = nullptr;
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

int cg_scan_batch(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint64_t* out_words,
                  cg_hit* out_hits, uint32_t hits_cap, uint32_t* out_nhits) {
  std::lock_guard<std::mutex> lk(g_mu);
  HostScan hs;
  int rc;
  // large words-only batches: chunked, copies overlapped with the kernels (the hit list needs the per-batch slot tables)
  static const bool no_chunks = getenv("CG_NO_CHUNKS") && atoi(getenv("CG_NO_CHUNKS"));
  if (!no_chunks && !out_hits && out_words && n >= (1u << 16) && G.ready && rs && bytes && offsets) {
    rc = scan_host_chunked(rs, bytes, offsets, n, out_words);
    if (rc < 0) return rc;
    if (rc == 0) {
      if (out_nhits) { uint64_t nh = 0; for (uint32_t i = 0; i < n; i++) if (out_words[i] >> 63) nh += (out_words[i] >> 32) & 0x7fffffffu; *out_nhits = (uint32_t)nh; G.stats.hits += nh; }
      return CG_OK;
    }
    // rc == 1: a queue overflowed in some piece; capacities have been raised -- run the batch in one piece below
  }
  rc = scan_host(rs, bytes, offsets, n, false, &hs);
  if (rc) return rc;
  cudaStream_t st = G.stream;
  if (out_words && n) CU(cudaMemcpyAsync(out_words, G.d_words, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  uint32_t n_slots = hs.counters[0], rw = rs->dev.rw;
  uint32_t nh = 0;
  if ((out_hits || out_nhits) && n_slots) {
    hs.slot_msg.resize(n_slots); hs.hit.resize((size_t)n_slots * rw);
    CU(cudaMemcpyAsync(hs.slot_msg.data(), rs->work.slot_msg, (size_t)n_slots * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(hs.hit.data(), rs->work.hit, (size_t)n_slots * rw * 4, cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  if ((out_hits || out_nhits) && n_slots) {
    std::vector<uint32_t> order(n_slots);
    for (uint32_t i = 0; i < n_slots; i++) order[i] = i;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return hs.slot_msg[a] < hs.slot_msg[b]; });
    for (uint32_t oi = 0; oi < n_slots; oi++) {
      uint32_t s = order[oi];
      if (hs.slot_msg[s] == 0xffffffffu) continue;
      nh = append_hit_row(&hs.hit[(size_t)s * rw], rw, nh, out_hits ? hits_cap : 0, [&](uint32_t i, uint32_t r) { out_hits[i].msg = hs.slot_msg[s]; out_hits[i].rule = r; });
    }
  }
  if (out_nhits) *out_nhits = nh;
  G.stats.hits += nh;
  if (out_hits && nh > hits_cap) return fail(CG_ERR_CAPACITY, "out_hits too small");
  return CG_OK;
}

namespace {
constexpr uint32_t kOneBytes = 16384, kOneRw = 128, kOneIn = 256 + kOneBytes + 64, kOneOut = (2 + kCounterWords + kOneRw) * 4;
// -> CG_OK, an error, or 1 = take the general path (long message, large rule set, a queue overflowed)
int scan_one_fast(cg_ruleset* rs, const uint8_t* bytes, uint32_t len, uint64_t* out_word, uint32_t* out_rules, uint32_t rules_cap, uint32_t* out_nrules) {
  static const bool off_ = getenv("CG_ONE_FAST") && atoi(getenv("CG_ONE_FAST")) == 0;
  if (off_ || !G.ready || !rs || (len && !bytes) || len > kOneBytes || rs->dev.rw > kOneRw - 2 || G.profiling) return 1;
  cg_ruleset::OnePath& o = rs->one;
  cudaStream_t st = G.stream;
  int rc;
  if (!o.h_pin) { CU(cudaMallocHost((void**)&o.h_pin, kOneIn + kOneOut)); memset(o.h_pin, 0, kOneIn + kOneOut); CU(cudaMalloc((void**)&o.d_buf, kOneIn + kOneOut)); CU(cudaMemset(o.d_buf, 0, kOneIn + kOneOut)); }
  if ((rc = prepare_step(rs, 1, false, st))) return rc;
  const uint8_t* d_bytes = o.d_buf; const uint32_t* d_off = reinterpret_cast<const uint32_t*>(o.d_buf);
  uint32_t* d_out = reinterpret_cast<uint32_t*>(o.d_buf + kOneIn); uint64_t* d_word = reinterpret_cast<uint64_t*>(o.d_buf + kOneIn + kOneOut - 8);   // (the word lands behind the hit row, then is packed to the front)
  if (!o.exec || o.gen != rs->scratch_gen || o.ctas != rs->verify_ctas) {
    if (o.exec) { cudaGraphExecDestroy(o.exec); o.exec = nullptr; }
    if ((rc = capture(st, [&] {
          const int r = run_scan_device(rs, d_bytes, d_off, 1, d_word, false, st);
          if (r == CG_OK) count_launches(launch_pack_one(rs->dev, rs->work, d_word, d_out, kOneRw - 2, st));
          return r;
        }, &o.exec, &o.kernels))) return rc;
    o.gen = rs->scratch_gen; o.ctas = rs->verify_ctas;
  }
  uint32_t* hoff = reinterpret_cast<uint32_t*>(o.h_pin); hoff[0] = 256; hoff[1] = 256 + len;
  if (len) memcpy(o.h_pin + 256, bytes, len);
  memset(o.h_pin + 256 + len, 0, 64);
  CU(cudaMemcpyAsync(o.d_buf, o.h_pin, 256 + (size_t)len + 64, cudaMemcpyHostToDevice, st));
  CU(cudaGraphLaunch(o.exec, st));
  CU(cudaMemcpyAsync(o.h_pin + kOneIn, d_out, (2 + kCounterWords + rs->dev.rw) * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  count_launches(o.kernels);
  const uint32_t* ho = reinterpret_cast<const uint32_t*>(o.h_pin + kOneIn);
  const uint32_t* hc = ho + 2;
  if ((rc = absorb_counters(rs, hc))) return rc;                 // 1: a queue overflowed, the general path retries with larger scratch
  G.stats.messages_scanned += 1; G.stats.bytes_scanned += len; G.stats.candidate_events += hc[1]; G.stats.verified_pairs += hc[1];
  if (out_word) *out_word = (uint64_t)ho[0] | ((uint64_t)ho[1] << 32);
  const uint32_t nh = append_hit_row(ho + 2 + kCounterWords, rs->dev.rw, 0, out_rules ? rules_cap : 0, [&](uint32_t i, uint32_t r) { out_rules[i] = r; });
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
// findMatches + resolveOverlaps for a host batch: scan_host (with its retries), then the span resolver on the library stream.
// Resolved spans land in G.d_spans; redacting, G.d_redact_meta holds [sizes, 4 words][out offsets, n + 1][digests, 16-byte
// aligned, room for every raw span] and *out_offsets the output offsets.  *ns = resolved spans, *need = redacted bytes.
// Leaves the input in G.d_bytes / G.d_off32.
int resolve_host(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, bool redact, uint32_t* out_offsets,
                 uint32_t* ns, uint64_t* need, uint32_t** d_digests) {
  HostScan hs;
  int rc = scan_host(rs, bytes, offsets, n, true, &hs);
  if (rc) return rc;
  const ScanWork& w = rs->work;
  cudaStream_t st = G.stream;
  const size_t dig_at = ((size_t)n + 1 + 4 + 3) & ~(size_t)3;
  if ((rc = grow(&G.d_spans, &G.cap_spans, (size_t)w.span_cap))) return rc;
  if ((rc = grow(&G.d_redact_meta, &G.cap_redact_meta, dig_at + (redact ? (size_t)w.span_cap * 8 : 0)))) return rc;
  uint32_t* d_sizes = G.d_redact_meta; uint32_t* d_out_off = G.d_redact_meta + 4;
  *d_digests = G.d_redact_meta + dig_at;
  const SpanOutputs o{reinterpret_cast<uint32_t*>(G.d_spans), w.span_cap, d_out_off, ~0ull, d_sizes, redact};
  count_launches(launch_span_resolve(w, G.d_off32, n, o, G.sm_count, st));
  CU(cudaGetLastError());
  uint64_t sizes[2] = {0, 0};
  CU(cudaMemcpyAsync(sizes, d_sizes, redact ? 16 : 4, cudaMemcpyDeviceToHost, st));
  if (redact) CU(cudaMemcpyAsync(out_offsets, d_out_off, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  *ns = redact ? (uint32_t)sizes[1] : (uint32_t)sizes[0]; *need = redact ? sizes[0] : 0;
  G.stats.spans += *ns;
  return CG_OK;
}
}  // namespace

int cg_find_matches_batch(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans) {
  std::lock_guard<std::mutex> lk(g_mu);
  uint32_t outn = 0; uint64_t need = 0; uint32_t* d_dig = nullptr;
  int rc = resolve_host(rs, bytes, offsets, n, false, nullptr, &outn, &need, &d_dig);
  if (rc) return rc;
  const uint32_t k = std::min(outn, spans_cap);
  if (out_spans && k) { CU(cudaMemcpyAsync(out_spans, G.d_spans, (size_t)k * sizeof(cg_span), cudaMemcpyDeviceToHost, G.stream)); CU(cudaStreamSynchronize(G.stream)); }
  if (out_nspans) *out_nspans = outn;
  if (out_spans && outn > spans_cap) return fail(CG_ERR_CAPACITY, "out_spans too small");
  return CG_OK;
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
  int rc;
  if ((rc = upload(rs, pol, &rs->dev.rule_policy))) return rc;
  if ((rc = upload(rs, act, &rs->dev.rule_action))) return rc;
  rs->scratch_gen++;                                        // DevRuleset is captured by value
  return CG_OK;
}

int cg_policy_verdict_batch(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint32_t* out_verdicts) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!rs || !out_verdicts) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!rs->dev.rule_policy) return fail(CG_ERR_INVALID_ARG, "cg_ruleset_set_policy has not been called");
  HostScan hs;
  int rc = scan_host(rs, bytes, offsets, n, false, &hs);
  if (rc) return rc;
  if (!n) return CG_OK;
  if ((rc = grow(&G.d_verdicts, &G.cap_verdicts, (size_t)n))) return rc;
  uint32_t* d_verdicts = G.d_verdicts;
  cudaStream_t st = G.stream;
  CU(cudaMemsetAsync(d_verdicts, 0, (size_t)n * 4, st));
  int k = launch_verdicts(rs->dev, rs->work, d_verdicts, G.sm_count, st);
  count_launches(k);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out_verdicts, d_verdicts, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}

int cg_redact_batch(cg_ruleset* rs, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint8_t* out_bytes, uint64_t out_cap,
                    uint64_t* out_need, uint32_t* out_offsets, cg_span* out_spans, uint32_t spans_cap, uint32_t* out_nspans, uint8_t* out_digests32) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!out_offsets || (n && (!bytes || !offsets))) return fail(CG_ERR_INVALID_ARG, "null argument");
  uint32_t ns = 0; uint64_t pos = 0; uint32_t* d_dig = nullptr;
  int rc = resolve_host(rs, bytes, offsets, n, true, out_offsets, &ns, &pos, &d_dig);     // input bytes / offsets stay in G.d_bytes / G.d_off32
  if (rc) return rc;
  if (out_need) *out_need = pos;
  if (out_nspans) *out_nspans = ns;
  if (pos >> 32) return fail(CG_ERR_TOO_LARGE, "redacted batch exceeds 4 GiB");
  if ((out_spans && ns > spans_cap) || pos > out_cap || !out_bytes) return fail(CG_ERR_CAPACITY, "output buffer too small (see *out_need / *out_nspans)");
  cudaStream_t st = G.stream;
  if ((rc = grow(&G.d_redact_out, &G.cap_redact_out, (size_t)pos + 64))) return rc;
  uint8_t* d_out = G.d_redact_out;
  // device: digests and the splice itself, over the resolver's per-span arrays; it set their counts (counters[21], [22])
  const ScanWork& w = rs->work;
  int kl = launch_redact_digests(G.d_bytes, w.sp_start, w.sp_len, w.counters + 21, d_dig, G.sm_count, st);
  kl += launch_redact_splice(G.d_bytes, G.d_off32, G.d_redact_meta + 4, w.kept_begin, w.sp_start, w.sp_len, w.sp_cat, d_dig, d_out, w.counters + 22, n, G.sm_count, st);
  count_launches(kl); G.stats.sha256_items += ns;
  CU(cudaGetLastError());
  if (pos) CU(cudaMemcpyAsync(out_bytes, d_out, (size_t)pos, cudaMemcpyDeviceToHost, st));
  if (ns && out_spans) CU(cudaMemcpyAsync(out_spans, G.d_spans, (size_t)ns * sizeof(cg_span), cudaMemcpyDeviceToHost, st));
  if (ns && out_digests32) CU(cudaMemcpyAsync(out_digests32, d_dig, (size_t)ns * 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}

int cg_scan_batch_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_words, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!rs || !d_bytes || !d_offsets || !d_out_words) return fail(CG_ERR_INVALID_ARG, "null argument");
  if ((uintptr_t)d_bytes & 15u) return fail(CG_ERR_INVALID_ARG, "d_bytes must be 16-byte aligned");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream;
  if (!n) return CG_OK;
  static const bool use_graph = !(getenv("CG_NO_GRAPH") && atoi(getenv("CG_NO_GRAPH")));
  int rc;
  if ((rc = ensure_mirrors(rs))) return rc;
  // did an earlier batch overflow a queue?  (its result words say "incomplete"; grow the scratch before this one runs)
  poll_mirrors(rs, false);
  if ((rc = prepare_step(rs, n, false, st))) return rc;
  const auto enqueue = [&] { return run_scan_device(rs, (const uint8_t*)d_bytes, (const uint32_t*)d_offsets, n, (uint64_t*)d_out_words, false, st); };
  if (!use_graph || G.profiling) {
    rc = enqueue();
  } else {
    // memsets + scan + resolve + verify + finalize captured once per (arguments, scratch generation, verify grid), then
    // replayed: one launch per step instead of six, so the host never becomes the bottleneck
    cg_ruleset::CachedGraph* hit = nullptr;
    for (auto& g : rs->graphs) if (g.exec && g.bytes == d_bytes && g.off == d_offsets && g.words == d_out_words && g.n == n && g.gen == rs->scratch_gen && g.ctas == rs->verify_ctas) hit = &g;
    if (!hit) {
      hit = rs->graphs[0].used <= rs->graphs[1].used ? &rs->graphs[0] : &rs->graphs[1];       // least recently used entry
      if (hit->exec) { cudaGraphExecDestroy(hit->exec); hit->exec = nullptr; }
      if ((rc = capture(st, enqueue, &hit->exec, &hit->kernels))) return rc;
      hit->bytes = d_bytes; hit->off = d_offsets; hit->words = d_out_words; hit->n = n; hit->gen = rs->scratch_gen; hit->ctas = rs->verify_ctas;
    }
    hit->used = ++rs->graph_clock;
    CU(cudaGraphLaunch(hit->exec, st));
    count_launches(hit->kernels);
  }
  if (rc == CG_OK) {
    G.stats.messages_scanned += n;
    rc = mirror_counters(rs, st);
  }
  return rc;
}

int cg_scan_join(cg_ruleset* rs, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!rs) return fail(CG_ERR_INVALID_ARG, "null argument");
  CU(cudaStreamSynchronize(stream ? (cudaStream_t)stream : G.stream));
  poll_mirrors(rs, true);
  const uint32_t flags = rs->sticky_flags, status = rs->sticky_status; rs->sticky_flags = rs->sticky_status = 0;
  if (flags & (ERR_VM_STACK | ERR_VM_LIST)) return fail(CG_ERR_TOO_LARGE, std::string(kVmOverflow) + " (result words of that batch are all ones)");
  if (status & (1u << kResolveTooLarge)) return fail(CG_ERR_TOO_LARGE, "redacted batch exceeds 4 GiB");
  if (flags) return fail(CG_ERR_CAPACITY, "a candidate queue overflowed: the result words (or sizes) of that batch are all ones; the scratch has been grown, scan the batch again");
  if (status & (1u << kResolveCapacity)) return fail(CG_ERR_CAPACITY, "output buffer too small: the sizes a batch needs are in its d_out_sizes / d_out_nspans");
  return CG_OK;
}

namespace {
// findMatches (+ redaction) of a batch in HBM, enqueued on st: the span-mode step, the resolver, digests and splice (redact),
// then the counter block into the mirror ring.  Never waits for the device except when the scratch must grow.
int spans_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, const SpanOutputs& o, void* d_out_bytes,
                 void* d_digests, void* stream) {
  if (!rs || !d_bytes || !d_offsets || !o.sizes) return fail(CG_ERR_INVALID_ARG, "null argument");
  if ((uintptr_t)d_bytes & 15u) return fail(CG_ERR_INVALID_ARG, "d_bytes must be 16-byte aligned");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream;
  const uint8_t* bytes = (const uint8_t*)d_bytes; const uint32_t* off = (const uint32_t*)d_offsets;
  int rc;
  if ((rc = ensure_mirrors(rs))) return rc;
  poll_mirrors(rs, false);                                  // (an earlier batch overflowed?  grow before this one runs)
  if ((rc = prepare_step(rs, n, true, st))) return rc;
  const ScanWork& w = rs->work;
  if (n) { if ((rc = run_scan_device(rs, bytes, off, n, w.words, true, st))) return rc; }
  else CU(cudaMemsetAsync(w.counters, 0, kCounterWords * sizeof(uint32_t), st));
  int k = launch_span_resolve(w, off, n, o, G.sm_count, st);
  if (o.redact) {
    k += launch_redact_digests(bytes, w.sp_start, w.sp_len, w.counters + 21, (uint32_t*)d_digests, G.sm_count, st);
    k += launch_redact_splice(bytes, off, o.out_offsets, w.kept_begin, w.sp_start, w.sp_len, w.sp_cat, (const uint32_t*)d_digests,
                              (uint8_t*)d_out_bytes, w.counters + 22, n, G.sm_count, st);
  }
  count_launches(k);
  CU(cudaGetLastError());
  G.stats.messages_scanned += n;
  return mirror_counters(rs, st);
}
}  // namespace

int cg_find_matches_batch_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_spans, uint32_t spans_cap,
                                 void* d_out_nspans, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (spans_cap && !d_out_spans) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (((uintptr_t)d_offsets | (uintptr_t)d_out_spans | (uintptr_t)d_out_nspans) & 3u) return fail(CG_ERR_INVALID_ARG, "d_offsets, d_out_spans and d_out_nspans must be 4-byte aligned");
  const SpanOutputs o{(uint32_t*)d_out_spans, d_out_spans ? spans_cap : 0u, nullptr, 0, d_out_nspans, false};
  return spans_device(rs, d_bytes, d_offsets, n, o, nullptr, nullptr, stream);
}

int cg_redact_batch_device(cg_ruleset* rs, const void* d_bytes, const void* d_offsets, uint32_t n, void* d_out_bytes, uint64_t out_cap,
                           void* d_out_offsets, void* d_out_spans, uint32_t spans_cap, void* d_out_digests32, void* d_out_sizes, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!d_out_offsets || (out_cap && !d_out_bytes) || (spans_cap && (!d_out_spans || !d_out_digests32))) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (((uintptr_t)d_offsets | (uintptr_t)d_out_offsets | (uintptr_t)d_out_spans) & 3u) return fail(CG_ERR_INVALID_ARG, "d_offsets, d_out_offsets and d_out_spans must be 4-byte aligned");
  if ((uintptr_t)d_out_sizes & 7u) return fail(CG_ERR_INVALID_ARG, "d_out_sizes must be 8-byte aligned");
  if ((uintptr_t)d_out_digests32 & 15u) return fail(CG_ERR_INVALID_ARG, "d_out_digests32 must be 16-byte aligned");
  const SpanOutputs o{(uint32_t*)d_out_spans, spans_cap, (uint32_t*)d_out_offsets, d_out_bytes ? out_cap : 0ull, d_out_sizes, true};
  return spans_device(rs, d_bytes, d_offsets, n, o, d_out_bytes, d_out_digests32, stream);
}

// ---------------------------------------------------------------------------------- SHA / Merkle

int cg_sha256_batch(const uint8_t* bytes, const uint64_t* offsets, uint32_t n, uint8_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!n) return CG_OK;
  if (!offsets || !out) return fail(CG_ERR_INVALID_ARG, "null argument");
  size_t total = offsets[n]; int rc;
  if ((rc = grow_bytes(total + 64))) return rc;
  if ((rc = grow(&G.d_off64, &G.cap_off64, (size_t)n + 1))) return rc;
  if ((rc = grow(&G.d_dig[0], &G.cap_dig[0], (size_t)n * 8))) return rc;
  cudaStream_t st = G.stream;
  if (total) CU(cudaMemcpyAsync(G.d_bytes, bytes, total, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(G.d_off64, offsets, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
  int k = launch_sha256_batch(G.d_bytes, G.d_off64, n, (uint8_t*)G.d_dig[0], st);
  count_launches(k); G.stats.sha256_items += n;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, G.d_dig[0], (size_t)n * 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}

namespace {
int empty_root(uint8_t out[32]) {
  // SHA-256("") -- computed by the same kernel, not on the CPU
  int rc;
  if ((rc = grow(&G.d_off64, &G.cap_off64, 2))) return rc;
  if ((rc = grow(&G.d_dig[0], &G.cap_dig[0], 8))) return rc;
  if ((rc = grow_bytes(64))) return rc;
  CU(cudaMemsetAsync(G.d_off64, 0, 16, G.stream));
  int k = launch_sha256_batch(G.d_bytes, G.d_off64, 1, (uint8_t*)G.d_dig[0], G.stream);
  count_launches(k);
  CU(cudaMemcpyAsync(out, G.d_dig[0], 32, cudaMemcpyDeviceToHost, G.stream));
  CU(cudaStreamSynchronize(G.stream));
  return CG_OK;
}

// One-shot trees: size_dig(n) makes room for n staged nodes in G.d_dig[0]; fold_dig folds n nodes at d_nodes (read in place,
// may be G.d_dig[0]) by at most max_levels levels, ping-ponging between G.d_dig[1] and G.d_dig[0]; *out = the folded nodes
int size_dig(uint64_t n) {
  int rc = grow(&G.d_dig[0], &G.cap_dig[0], (size_t)n * 8);
  return rc ? rc : grow(&G.d_dig[1], &G.cap_dig[1], (size_t)(n + 1) / 2 * 8 + 8);
}
int fold_dig(const uint32_t* d_nodes, uint64_t n, uint32_t max_levels, cudaStream_t st, const uint32_t** out) {
  count_launches(launch_merkle_fold(d_nodes, n, max_levels, G.d_dig[1], G.d_dig[0], st, out));
  CU(cudaGetLastError());
  return CG_OK;
}

// root of n leaves in G.d_bytes (ragged at d_off, else leaf_len bytes each) -> host; leaves and fold time last_merkle_ms
int staged_root(uint64_t n, const uint64_t* d_off, uint64_t leaf_len, uint8_t out_root[32]) {
  cudaStream_t st = G.stream; const uint32_t* d_root; int rc;
  if ((rc = size_dig(n))) return rc;
  CU(cudaEventRecord(G.ev0, st));
  count_launches(d_off ? launch_merkle_leaves_var(G.d_bytes, d_off, n, G.d_dig[0], st) : launch_merkle_leaves_fixed(G.d_bytes, leaf_len, n, G.d_dig[0], st));
  G.stats.merkle_leaves += n;
  if ((rc = fold_dig(G.d_dig[0], n, 64, st, &d_root))) return rc;
  CU(cudaEventRecord(G.ev1, st));
  CU(cudaMemcpyAsync(out_root, d_root, 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  float ms = 0; cudaEventElapsedTime(&ms, G.ev0, G.ev1); G.stats.last_merkle_ms = ms;
  return CG_OK;
}

// roots of the aligned 2^block_log2-leaf blocks of n fixed-size leaves in device memory -> d_roots (32 bytes per block)
int block_roots(const void* d_bytes, uint64_t leaf_len, uint64_t n, uint32_t block_log2, void* d_roots, cudaStream_t st) {
  const uint32_t* d_res; int rc;
  if ((rc = size_dig(n))) return rc;
  count_launches(launch_merkle_leaves_fixed((const uint8_t*)d_bytes, leaf_len, n, G.d_dig[0], st)); G.stats.merkle_leaves += n;
  if ((rc = fold_dig(G.d_dig[0], n, block_log2, st, &d_res))) return rc;
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
  if ((rc = grow_bytes(total + 64))) return rc;
  if ((rc = grow(&G.d_off64, &G.cap_off64, (size_t)n + 1))) return rc;
  if (total) CU(cudaMemcpyAsync(G.d_bytes, bytes, total, cudaMemcpyHostToDevice, G.stream));
  CU(cudaMemcpyAsync(G.d_off64, offsets, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, G.stream));
  return staged_root(n, G.d_off64, 0, out_root);
}

int cg_merkle_root_fixed(const uint8_t* bytes, uint64_t leaf_len, uint64_t n, uint8_t out_root[32]) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!out_root) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (n == 0) return empty_root(out_root);
  size_t total = (size_t)leaf_len * n; int rc;
  if ((rc = grow_bytes(total + 64))) return rc;
  if (total) CU(cudaMemcpyAsync(G.d_bytes, bytes, total, cudaMemcpyHostToDevice, G.stream));
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
  if ((rc = size_dig(m))) return rc;
  CU(cudaMemcpyAsync(G.d_dig[0], nodes32, m * 32, cudaMemcpyHostToDevice, st));
  if ((rc = fold_dig(G.d_dig[0], m, 64, st, &d_root))) return rc;
  CU(cudaMemcpyAsync(out_root, d_root, 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}

int cg_merkle_fold_device(const void* d_nodes32, uint64_t m, void* d_out_root32, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!m || !d_nodes32 || !d_out_root32) return fail(CG_ERR_INVALID_ARG, "null or empty input");
  cudaStream_t st = stream ? (cudaStream_t)stream : G.stream; const uint32_t* d_root; int rc;
  if ((rc = size_dig(m))) return rc;
  // the fold reads the nodes in place, unless they are off the 16-byte alignment of the kernels' loads: then from a copy
  const uint32_t* d_nodes = (const uint32_t*)d_nodes32;
  if ((uintptr_t)d_nodes32 & 15) { CU(cudaMemcpyAsync(G.d_dig[0], d_nodes32, m * 32, cudaMemcpyDeviceToDevice, st)); d_nodes = G.d_dig[0]; }
  if ((rc = fold_dig(d_nodes, m, 64, st, &d_root))) return rc;
  CU(cudaMemcpyAsync(d_out_root32, d_root, 32, cudaMemcpyDeviceToDevice, st));
  return CG_OK;
}

// ---------------------------------------------------------------------------------- Merkle log (append, frontier, proofs)
struct cg_merkle_log {
  uint64_t n = 0;                 // leaves so far; bit h of n set <=> slot h holds the root of a perfect 2^h subtree
  bool keep = false;              // keep every leaf digest in HBM (needed for inclusion proofs)
  uint32_t* d_slots = nullptr;    // 64 x 8 words
  uint32_t* d_tmp = nullptr;      // 66 x 8 words: [0..63] gathered left operands, [64] accumulator, [65] result
  uint32_t* d_leaves = nullptr; uint64_t cap_leaves = 0;     // keep: n leaf digests
  uint32_t* d_new = nullptr; size_t cap_new = 0;             // !keep: the current batch's leaf digests
  uint32_t* d_a = nullptr; size_t cap_a = 0; uint32_t* d_b = nullptr; size_t cap_b = 0;   // level ping-pong
  ~cg_merkle_log() { cudaFree(d_slots); cudaFree(d_tmp); cudaFree(d_leaves); cudaFree(d_new); cudaFree(d_a); cudaFree(d_b); }
};

namespace {
// MTH of `cnt` consecutive leaf digests starting at d_in (level-wise, unpaired node promoted) -> d_out (32 bytes)
int log_range_root(cg_merkle_log* L, const uint32_t* d_in, uint64_t cnt, uint32_t* d_out, cudaStream_t st) {
  int rc;
  if (cnt == 1) { CU(cudaMemcpyAsync(d_out, d_in, 32, cudaMemcpyDeviceToDevice, st)); return CG_OK; }
  if ((rc = grow(&L->d_a, &L->cap_a, (size_t)(cnt + 1) / 2 * 8 + 8))) return rc;
  if ((rc = grow(&L->d_b, &L->cap_b, (size_t)(cnt + 3) / 4 * 8 + 8))) return rc;
  const uint32_t* d_root;
  count_launches(launch_merkle_fold(d_in, cnt, 64, L->d_a, L->d_b, st, &d_root));
  CU(cudaMemcpyAsync(d_out, d_root, 32, cudaMemcpyDeviceToDevice, st));
  return CG_OK;
}
int log_check(cg_merkle_log* L) {
  if (int rc = require_ready()) return rc;
  if (!L) return fail(CG_ERR_INVALID_ARG, "null argument");
  return CG_OK;
}
// root of the current tree -> d_tmp[65]
int log_root_device(cg_merkle_log* L, cudaStream_t st) {
  // fold the frontier from the smallest subtree upwards: r = slot[lowest]; r = node(slot[h], r) for every higher set bit
  uint32_t nl = 0; int lowest = -1;
  for (int h = 0; h < 64; h++) if ((L->n >> h) & 1ull) {
    if (lowest < 0) { lowest = h; continue; }
    CU(cudaMemcpyAsync(L->d_tmp + 8 * nl, L->d_slots + 8 * h, 32, cudaMemcpyDeviceToDevice, st)); nl++;
  }
  int k = launch_merkle_chain(L->d_tmp, nl, L->d_slots + 8 * lowest, L->d_tmp + 8 * 65, st);
  count_launches(k);
  return CG_OK;
}
}  // namespace

int cg_merkle_log_create(cg_merkle_log** out, int keep_leaf_digests) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!out) return fail(CG_ERR_INVALID_ARG, "null argument");
  std::unique_ptr<cg_merkle_log> L(new cg_merkle_log());
  L->keep = keep_leaf_digests != 0;
  CU(cudaMalloc((void**)&L->d_slots, 64 * 32)); CU(cudaMalloc((void**)&L->d_tmp, 66 * 32));
  CU(cudaMemset(L->d_slots, 0, 64 * 32));
  *out = L.release();
  return CG_OK;
}
void cg_merkle_log_destroy(cg_merkle_log* L) { std::lock_guard<std::mutex> lk(g_mu); if (L) { if (G.ready) cudaStreamSynchronize(G.stream); delete L; } }
int cg_merkle_log_size(const cg_merkle_log* L, uint64_t* out_n) { if (!L || !out_n) return fail(CG_ERR_INVALID_ARG, "null argument"); *out_n = L->n; return CG_OK; }

int cg_merkle_log_restore(cg_merkle_log** out, uint64_t n, const uint8_t* frontier32, uint32_t count) {
  if (!out || (count && !frontier32) || count != (uint32_t)__builtin_popcountll(n)) return fail(CG_ERR_INVALID_ARG, "frontier must hold one digest per set bit of n");
  int rc = cg_merkle_log_create(out, 0);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g_mu);
  cg_merkle_log* L = *out; uint32_t k = 0;
  for (int h = 63; h >= 0; h--) if ((n >> h) & 1ull) { CU(cudaMemcpy(L->d_slots + 8 * h, frontier32 + 32 * (size_t)k, 32, cudaMemcpyHostToDevice)); k++; }
  L->n = n;
  return CG_OK;
}

int cg_merkle_log_frontier(cg_merkle_log* L, uint8_t* out_frontier32, uint32_t* out_count) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!out_count) return fail(CG_ERR_INVALID_ARG, "null argument");
  uint32_t k = 0;
  for (int h = 63; h >= 0; h--) if ((L->n >> h) & 1ull) { if (out_frontier32) CU(cudaMemcpyAsync(out_frontier32 + 32 * (size_t)k, L->d_slots + 8 * h, 32, cudaMemcpyDeviceToHost, G.stream)); k++; }
  CU(cudaStreamSynchronize(G.stream));
  *out_count = k;
  return CG_OK;
}

namespace {
// room for m more leaf digests; returns where they go
int log_digest_room(cg_merkle_log* L, uint64_t m, cudaStream_t st, uint32_t** out) {
  int rc;
  if (L->keep) {
    if (L->n + m > L->cap_leaves) {                         // grow the digest store (amortised doubling), keeping what is there
      uint64_t cap = std::max<uint64_t>(L->n + m, L->cap_leaves * 2); uint32_t* nd = nullptr;
      CU(cudaMalloc((void**)&nd, (size_t)cap * 32));
      if (L->n) CU(cudaMemcpyAsync(nd, L->d_leaves, (size_t)L->n * 32, cudaMemcpyDeviceToDevice, st));
      CU(cudaStreamSynchronize(st)); cudaFree(L->d_leaves); L->d_leaves = nd; L->cap_leaves = cap;
    }
    *out = L->d_leaves + (size_t)L->n * 8;
  } else {
    if ((rc = grow(&L->d_new, &L->cap_new, (size_t)m * 8))) return rc;
    *out = L->d_new;
  }
  return CG_OK;
}
// m new leaf digests at d_dig: cut [n, n+m) into aligned perfect blocks (block size <= lowest set bit of its position),
// reduce each, carry into the frontier
int log_absorb(cg_merkle_log* L, const uint32_t* d_dig, uint64_t m, cudaStream_t st) {
  int rc, k;
  uint64_t pos = L->n, rem = m;
  while (rem) {
    uint64_t s = pos ? (pos & (~pos + 1)) : (1ull << 63);
    while (s > rem) s >>= 1;
    uint32_t* acc = L->d_tmp + 8 * 64;
    if ((rc = log_range_root(L, d_dig + (size_t)(pos - L->n) * 8, s, acc, st))) return rc;
    int h = 0; while ((1ull << h) < s) h++;
    uint32_t nl = 0; int top = h;                           // slots h, h+1, ... that are occupied merge into the new subtree
    while ((pos >> top) & 1ull) { CU(cudaMemcpyAsync(L->d_tmp + 8 * nl, L->d_slots + 8 * top, 32, cudaMemcpyDeviceToDevice, st)); nl++; top++; }
    if (nl) { k = launch_merkle_chain(L->d_tmp, nl, acc, L->d_slots + 8 * top, st); count_launches(k); }
    else CU(cudaMemcpyAsync(L->d_slots + 8 * top, acc, 32, cudaMemcpyDeviceToDevice, st));
    pos += s; rem -= s;
  }
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(st));
  L->n += m;
  return CG_OK;
}
}  // namespace

/* room for n_leaves more leaf digests and their bytes up front (an append that has to grow the digest store pays a device
 * allocation and a copy of everything kept so far) */
int cg_merkle_log_reserve(cg_merkle_log* L, uint64_t n_leaves, uint64_t n_bytes) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  uint32_t* unused;
  if (n_leaves && (rc = log_digest_room(L, n_leaves, G.stream, &unused))) return rc;
  if (n_bytes && (rc = grow_bytes((size_t)n_bytes + 64))) return rc;
  if (n_leaves && (rc = grow(&G.d_off64, &G.cap_off64, (size_t)n_leaves + 1))) return rc;
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
  const size_t first = offsets[0], total = offsets[m];
  if ((rc = grow_bytes(total + 64))) return rc;
  if ((rc = grow(&G.d_off64, &G.cap_off64, (size_t)m + 1))) return rc;
  if ((rc = ensure_copy_streams())) return rc;
  uint32_t* d_dig;                                          // where this batch's leaf digests go
  if ((rc = log_digest_room(L, m, st, &d_dig))) return rc;
  CU(cudaStreamSynchronize(st));                            // (whatever still read the staging buffer is done)
  CU(cudaMemcpyAsync(G.d_off64, offsets, ((size_t)m + 1) * 8, cudaMemcpyHostToDevice, G.s_h2d));
  // the leaf bytes go over in pieces on the copy stream; the leaf kernel of piece c runs while piece c + 1 is still in flight
  const int C = (total - first) > ((size_t)4 << 20) ? Ctx::kChunks : 1;
  const uint64_t per = (m + C - 1) / C;
  for (int c = 0; c < C; c++) {
    const uint64_t m0 = std::min<uint64_t>((uint64_t)c * per, m), m1 = std::min<uint64_t>((uint64_t)(c + 1) * per, m);
    if (m1 <= m0) break;
    const size_t b0 = offsets[m0], b1 = offsets[m1];
    if (b1 > b0) CU(cudaMemcpyAsync(G.d_bytes + b0, bytes + b0, b1 - b0, cudaMemcpyHostToDevice, G.s_h2d));
    CU(cudaEventRecord(G.e_h2d[c], G.s_h2d));
    CU(cudaStreamWaitEvent(st, G.e_h2d[c], 0));
    int k = launch_merkle_leaves_var(G.d_bytes, G.d_off64 + m0, m1 - m0, d_dig + (size_t)m0 * 8, st);
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
  const uint32_t n_pieces = (uint32_t)((len + 4095) / 4096);
  if ((rc = grow_bytes((size_t)len + 64))) return rc;
  if ((rc = grow(&G.d_off32, &G.cap_off32, (size_t)n_pieces + 4))) return rc;          // newline counts per 4 KB piece
  if ((rc = grow(&G.d_off64, &G.cap_off64, 2))) return rc;
  CU(cudaMemcpyAsync(G.d_bytes, bytes, len, cudaMemcpyHostToDevice, st));
  uint64_t* d_total = G.d_off64;                           // (re-grown below once the line count is known)
  int k = launch_newline_split(G.d_bytes, len, G.d_off32, d_total, st);
  uint64_t n_lines = 0;
  CU(cudaMemcpyAsync(&n_lines, d_total, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (!n_lines) return CG_OK;
  if (L->n + n_lines < L->n) return fail(CG_ERR_TOO_LARGE, "log size overflows 64 bits");
  if ((rc = grow(&G.d_off64, &G.cap_off64, (size_t)n_lines + 1))) return rc;
  k += launch_newline_starts(G.d_bytes, len, G.d_off32, G.d_off64, n_lines, st);
  uint32_t* d_dig;
  if ((rc = log_digest_room(L, n_lines, st, &d_dig))) return rc;
  k += launch_merkle_leaves_var(G.d_bytes, G.d_off64, n_lines, d_dig, st, /*trim_newline=*/true);
  count_launches(k); G.stats.merkle_leaves += n_lines;
  if (out_lines) *out_lines = n_lines;
  return log_absorb(L, d_dig, n_lines, st);
}

int cg_merkle_log_root(cg_merkle_log* L, uint8_t out_root[32]) {
  {
    std::lock_guard<std::mutex> lk(g_mu);
    int rc = log_check(L); if (rc) return rc;
    if (!out_root) return fail(CG_ERR_INVALID_ARG, "null argument");
    if (L->n) {
      if ((rc = log_root_device(L, G.stream))) return rc;
      CU(cudaMemcpyAsync(out_root, L->d_tmp + 8 * 65, 32, cudaMemcpyDeviceToHost, G.stream));
      CU(cudaStreamSynchronize(G.stream));
      return CG_OK;
    }
    return empty_root(out_root);
  }
}

int cg_merkle_log_proof(cg_merkle_log* L, uint64_t index, uint8_t* out_path32, uint32_t path_cap, uint32_t* out_len) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!out_len) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!L->keep) return fail(CG_ERR_UNSUPPORTED, "log was created without leaf digests (or restored from a frontier): no proofs");
  if (index >= L->n) return fail(CG_ERR_INVALID_ARG, "leaf index out of range");
  // RFC 6962 2.1.1: PATH(m, D[n]) -- the sibling subtree at every split on the way down, returned leaf level first
  std::vector<std::pair<uint64_t, uint64_t>> sib;
  uint64_t lo = 0, hi = L->n;
  while (hi - lo > 1) {
    uint64_t k = 1; while (k * 2 < hi - lo) k *= 2;       // largest power of two < hi - lo
    if (index < lo + k) { sib.push_back({lo + k, hi}); hi = lo + k; } else { sib.push_back({lo, lo + k}); lo = lo + k; }
  }
  *out_len = (uint32_t)sib.size();
  if (sib.size() > path_cap || (sib.size() && !out_path32)) return fail(CG_ERR_CAPACITY, "path buffer too small");
  cudaStream_t st = G.stream;
  for (size_t i = 0; i < sib.size(); i++) {
    const auto& r = sib[sib.size() - 1 - i];
    if ((rc = log_range_root(L, L->d_leaves + (size_t)r.first * 8, r.second - r.first, L->d_tmp + 8 * i, st))) return rc;
  }
  if (!sib.empty()) CU(cudaMemcpyAsync(out_path32, L->d_tmp, sib.size() * 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}

/* RFC 6962 2.1.2: PROOF(m, D[n]) -- the nodes that show the tree of the first m leaves is a prefix of the current one. */
int cg_merkle_log_consistency(cg_merkle_log* L, uint64_t first_size, uint8_t* out_path32, uint32_t path_cap, uint32_t* out_len) {
  std::lock_guard<std::mutex> lk(g_mu);
  int rc = log_check(L); if (rc) return rc;
  if (!out_len) return fail(CG_ERR_INVALID_ARG, "null argument");
  if (!L->keep) return fail(CG_ERR_UNSUPPORTED, "log was created without leaf digests (or restored from a frontier): no proofs");
  if (first_size == 0 || first_size > L->n) return fail(CG_ERR_INVALID_ARG, "first_size must be in [1, size of the log]");
  // SUBPROOF(m, D[lo:hi], b): k = largest power of two < hi - lo; m <= k: recurse left, then MTH(D[lo+k:hi]);
  // else recurse right with b = false, then MTH(D[lo:lo+k]); m == hi - lo: {} if b else {MTH(D[lo:hi])}
  std::vector<std::pair<uint64_t, uint64_t>> ranges;      // in proof order
  {
    std::vector<std::pair<uint64_t, uint64_t>> tail;       // appended after the recursion, innermost first
    uint64_t lo = 0, hi = L->n, m = first_size; bool b = true;
    while (m != hi - lo) {
      uint64_t k = 1; while (k * 2 < hi - lo) k *= 2;
      if (m <= k) { tail.push_back({lo + k, hi}); hi = lo + k; }
      else { tail.push_back({lo, lo + k}); lo += k; m -= k; b = false; }
    }
    if (!b) ranges.push_back({lo, hi});
    for (size_t i = tail.size(); i-- > 0;) ranges.push_back(tail[i]);
  }
  *out_len = (uint32_t)ranges.size();
  if (ranges.size() > path_cap || ranges.size() > 64 || (ranges.size() && !out_path32)) return fail(CG_ERR_CAPACITY, "path buffer too small");
  cudaStream_t st = G.stream;
  for (size_t i = 0; i < ranges.size(); i++)
    if ((rc = log_range_root(L, L->d_leaves + (size_t)ranges[i].first * 8, ranges[i].second - ranges[i].first, L->d_tmp + 8 * i, st))) return rc;
  if (!ranges.empty()) CU(cudaMemcpyAsync(out_path32, L->d_tmp, ranges.size() * 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}

/* RFC 9162 2.1.4.2: *out_ok = 1 iff `path` proves that the tree with root_first over first_size leaves is a prefix of the tree
 * with root_second over second_size leaves (node hashes on the device, as everywhere in this library) */
int cg_merkle_verify_consistency(uint64_t first_size, uint64_t second_size, const uint8_t root_first[32], const uint8_t root_second[32],
                                 const uint8_t* path32, uint32_t path_len, int* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!out_ok || !root_first || !root_second || (path_len && !path32) || path_len > 64) return fail(CG_ERR_INVALID_ARG, "bad argument");
  int rc; cudaStream_t st = G.stream;
  if ((rc = grow(&G.d_dig[0], &G.cap_dig[0], (size_t)(path_len + 4) * 8))) return rc;
  uint32_t* d_r1 = G.d_dig[0]; uint32_t* d_r2 = d_r1 + 8; uint32_t* d_ok = d_r2 + 8; uint32_t* d_path = d_ok + 8;
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

int cg_merkle_verify_proof(const uint8_t* leaf_bytes, uint64_t leaf_len, uint64_t index, uint64_t tree_size, const uint8_t* path32, uint32_t path_len,
                           const uint8_t root[32], int* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int rc = require_ready()) return rc;
  if (!out_ok || !root || (leaf_len && !leaf_bytes) || (path_len && !path32) || path_len > 64) return fail(CG_ERR_INVALID_ARG, "bad argument");
  int rc; cudaStream_t st = G.stream;
  if ((rc = grow_bytes((size_t)leaf_len + 64))) return rc;
  if ((rc = grow(&G.d_off64, &G.cap_off64, 2))) return rc;
  if ((rc = grow(&G.d_dig[0], &G.cap_dig[0], (size_t)(path_len + 4) * 8))) return rc;
  uint64_t off[2] = {0, leaf_len};
  if (leaf_len) CU(cudaMemcpyAsync(G.d_bytes, leaf_bytes, leaf_len, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(G.d_off64, off, 16, cudaMemcpyHostToDevice, st));
  uint32_t* d_leaf = G.d_dig[0]; uint32_t* d_root = d_leaf + 8; uint32_t* d_ok = d_root + 8; uint32_t* d_path = d_ok + 8;
  int k = launch_merkle_leaves_var(G.d_bytes, G.d_off64, 1, d_leaf, st);
  CU(cudaMemcpyAsync(d_root, root, 32, cudaMemcpyHostToDevice, st));
  if (path_len) CU(cudaMemcpyAsync(d_path, path32, (size_t)path_len * 32, cudaMemcpyHostToDevice, st));
  k += launch_merkle_verify(d_leaf, index, tree_size, d_path, path_len, d_root, d_ok, st);
  count_launches(k);
  uint32_t ok = 0;
  CU(cudaMemcpyAsync(&ok, d_ok, 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  *out_ok = (int)ok;
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
  free_shard_roots();
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
  if ((rc = grow(&g_nccl.d_roots, &g_nccl.cap_roots, (size_t)world * max_blocks * 8))) return rc;
  uint32_t* const all = g_nccl.d_roots; uint32_t* const mine = all + (size_t)rank * max_blocks * 8;   // (an in-place all-gather)
  CU(cudaMemsetAsync(mine, 0, max_blocks * 32, st));
  if (n_local && (rc = block_roots(d_bytes, leaf_len, n_local, block_log2, mine, st))) return rc;
  if (world > 1) {
    lk.unlock(); const int r = g_nccl.AllGather(mine, all, max_blocks * 32, /*ncclChar*/ 0, comm, st); lk.lock();
    if (r) return nccl_fail(r, "ncclAllGather");
    // (a cg_shutdown, cg_comm_destroy or other sharded call during the gather is misuse, but must not make the fold read freed memory)
    if (!G.ready || g_nccl.d_roots != all) return fail(CG_ERR_NOT_INITIALIZED, "the library or the communicator's buffer changed during the all-gather");
  }
  const uint32_t* d_root;                                   // the fold's input: the gathered roots without the empty slots
  if ((rc = size_dig(total_blocks))) return rc;
  uint32_t* d = G.d_dig[0];
  for (int r = 0; r < world; r++) if (nblk[(size_t)r]) { CU(cudaMemcpyAsync(d, all + (size_t)r * max_blocks * 8, nblk[(size_t)r] * 32, cudaMemcpyDeviceToDevice, st)); d += nblk[(size_t)r] * 8; }
  if ((rc = fold_dig(G.d_dig[0], total_blocks, 64, st, &d_root))) return rc;
  CU(cudaMemcpyAsync(out_root, d_root, 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return CG_OK;
}

}  // extern "C"
