// span_resolve.cu -- resolveOverlaps (registry.ts:288-316) on the device: the raw spans a span-mode step queued (in any
// order) become the resolved spans of the batch, sorted by (msg, start16), with the redacted output's sizes and offsets.
//
//   count per message -> exclusive scan -> scatter into message order -> sort each message's segment and keep greedily
//   -> exclusive scans of the kept counts (first resolved index per message) and of the output lengths -> emit
//
// Order within a message: (start16 ascending, length in UTF-16 units descending, category ascending, rule ascending); a
// span is kept iff its start16 >= the end16 of the last kept span (-1 before the first).  A rule's global-exec iteration
// never yields two matches at one start, so the key is a strict total order and the result does not depend on the order
// the raw spans were queued in.  An empty match sets last_end to its own start: empty spans at one position are all kept.
//
// Every launch geometry depends on n and the SM count only; the span count is read from device memory.
//
// A batch of a few messages (cg_find_matches_one / cg_redact_one, cg_find_matches_few / cg_redact_few) skips the chain:
// span_resolve_few_kernel runs the same stages in one block, with the per-message arrays in shared memory, through the same
// warp_sort_keep / sort_keep_segment as the segments of a batch.
#include <algorithm>
#include <cstdint>

#include "kernels.h"

namespace cg {

namespace {

constexpr int kScanBlock = 512;              // exclusive scan
constexpr uint32_t kScanPerBlock = 4096;     // elements per scan block at least
constexpr int kSortBlock = 512;              // segment sort: one warp per short segment, one block per long one
constexpr uint32_t kWarpSort = 32;           // segments up to this long: sorted in registers by one warp
constexpr uint32_t kBlockSort = 2048;        // longer ones: runs of this many sorted in shared memory, then merged in HBM

// ---------------------------------------------------------------------------------------------- exclusive scan
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* sm /*[32]*/) {
  for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  __syncthreads();                                        // (sm may still be read by a previous call)
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  T t = 0;
  for (uint32_t k = 0; k < blockDim.x / 32; k++) t += sm[k];
  return t;
}

// partial[b] = sum of block b's range
template <typename T>
__global__ void __launch_bounds__(kScanBlock) xscan_sums_kernel(const T* __restrict__ in, uint32_t count, uint32_t per, T* __restrict__ partial) {
  __shared__ T sm[32];
  const uint64_t lo = (uint64_t)blockIdx.x * per, hi = lo + per < count ? lo + per : count;
  T s = 0;
  for (uint64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) s += in[i];
  s = block_sum(s, sm);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// out[i] = sum of in[0, i): the partials of the blocks in front, then the block's own range 512 elements at a time
template <typename T>
__global__ void __launch_bounds__(kScanBlock) xscan_apply_kernel(const T* __restrict__ in, T* __restrict__ out, uint32_t count, uint32_t per,
                                                               const T* __restrict__ partial) {
  __shared__ T sm[32];
  __shared__ T warp_excl[32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T c = 0;
  for (uint32_t k = threadIdx.x; k < blockIdx.x; k += blockDim.x) c += partial[k];
  T carry = block_sum(c, sm);
  __syncthreads();                                        // (every thread has read sm before the loop writes it)
  const uint64_t lo = (uint64_t)blockIdx.x * per, hi = lo + per < count ? lo + per : count;
  for (uint64_t base = lo; base < hi; base += blockDim.x) {
    const uint64_t i = base + threadIdx.x;
    const T v = i < hi ? in[i] : (T)0;
    T incl = v;
    for (int d = 1; d < 32; d <<= 1) { const T t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (uint32_t)d) incl += t; }
    if (lane == 31) sm[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      const T wv = lane < blockDim.x / 32 ? sm[lane] : (T)0;
      T wi = wv;
      for (int d = 1; d < 32; d <<= 1) { const T t = __shfl_up_sync(0xffffffffu, wi, d); if (lane >= (uint32_t)d) wi += t; }
      warp_excl[lane] = wi - wv;
      if (lane == 31) sm[0] = wi;                         // the chunk's total (sm[] is read again only after the next barrier)
    }
    __syncthreads();
    if (i < hi) out[i] = carry + warp_excl[warp] + incl - v;
    carry += sm[0];
    __syncthreads();
  }
}

template <typename T>
int xscan(const T* d_in, T* d_out, uint32_t count, T* d_part, int sm_count, cudaStream_t stream) {
  if (count == 0) return 0;
  uint32_t blocks = (count + kScanPerBlock - 1) / kScanPerBlock;
  const uint32_t max_blocks = std::min<uint32_t>(kScanPartials, 2u * (uint32_t)sm_count);
  if (blocks > max_blocks) blocks = max_blocks;
  const uint32_t per = (uint32_t)(((uint64_t)count + blocks - 1) / blocks);
  xscan_sums_kernel<T><<<blocks, kScanBlock, 0, stream>>>(d_in, count, per, d_part);
  xscan_apply_kernel<T><<<blocks, kScanBlock, 0, stream>>>(d_in, d_out, count, per, d_part);
  return 2;
}

// ---------------------------------------------------------------------------------------------- sort keys
// (start16, ~length16, rank of the rule in (category, rule) order, raw span index): ascending = resolveOverlaps' order
__device__ __forceinline__ bool key_less(const uint4& a, const uint4& b) {
  if (a.x != b.x) return a.x < b.x;
  if (a.y != b.y) return a.y < b.y;
  if (a.z != b.z) return a.z < b.z;
  return a.w < b.w;
}
__device__ __forceinline__ uint32_t key_end(const uint4& k) { return k.x + ~k.y; }
__device__ __forceinline__ uint4 pad_key() { return make_uint4(~0u, ~0u, ~0u, ~0u); }
__device__ __forceinline__ uint4 shfl_key(const uint4& k, uint32_t src_or_mask, bool xor_mode) {
  uint4 r;
  if (xor_mode) {
    r.x = __shfl_xor_sync(0xffffffffu, k.x, src_or_mask); r.y = __shfl_xor_sync(0xffffffffu, k.y, src_or_mask);
    r.z = __shfl_xor_sync(0xffffffffu, k.z, src_or_mask); r.w = __shfl_xor_sync(0xffffffffu, k.w, src_or_mask);
  } else {
    r.x = __shfl_sync(0xffffffffu, k.x, src_or_mask); r.y = __shfl_sync(0xffffffffu, k.y, src_or_mask);
    r.z = __shfl_sync(0xffffffffu, k.z, src_or_mask); r.w = __shfl_sync(0xffffffffu, k.w, src_or_mask);
  }
  return r;
}
// elements of the sorted run a[0, len) below x (or_equal: not above x)
__device__ __forceinline__ uint32_t rank_in(const uint4* __restrict__ a, uint32_t len, const uint4& x, bool or_equal) {
  uint32_t lo = 0, hi = len;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    const uint4 y = a[mid];
    if (or_equal ? !key_less(x, y) : key_less(y, x)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// bytes the placeholder "[REDACTED:<category>:<8 hex>]" takes instead of the span (category names of sha256_kernels.cu)
__device__ __forceinline__ int64_t splice_delta(const ScanWork& w, const uint32_t* __restrict__ category, const uint4& k) {
  const uint32_t* s = w.spans + (size_t)k.w * 6;
  const uint32_t cat = category[s[1]] & 3u;
  return (int64_t)(20u + ((0x0603090au >> (8u * cat)) & 0xffu)) - (int64_t)(s[3] - s[2]);
}

// Sort the segment sorted[s0, s0 + c) (any length) and keep greedily, one block: runs of kBlockSort bitonic-sorted in shared
// memory, pairwise merges in HBM (through sort_tmp), the greedy walk by one thread.  The kept keys move to the segment's
// front.  Returns the number kept and, redacting, *delta = the bytes their placeholders add (both on every thread).
// Call from block-uniform code with blockDim.x == kSortBlock.
__device__ uint32_t sort_keep_segment(const ScanWork& w, const uint32_t* __restrict__ category, uint32_t s0, uint32_t c, int redact,
                                      long long* delta) {
  __shared__ uint4 sk[kBlockSort];
  __shared__ long long red[32];
  __shared__ uint32_t kept_sh;
  uint4* cur = w.sorted + s0; uint4* alt = w.sort_tmp + s0;
  for (uint32_t base = 0; base < c; base += kBlockSort) {             // runs of kBlockSort: bitonic sort in shared memory
    const uint32_t cc = min(kBlockSort, c - base);
    uint32_t P = 64; while (P < cc) P <<= 1;
    for (uint32_t i = threadIdx.x; i < P; i += blockDim.x) sk[i] = i < cc ? cur[base + i] : pad_key();
    __syncthreads();
    for (uint32_t k = 2; k <= P; k <<= 1)
      for (uint32_t j = k >> 1; j > 0; j >>= 1) {
        for (uint32_t i = threadIdx.x; i < P; i += blockDim.x) {
          const uint32_t p = i ^ j;
          if (p > i) {
            const uint4 a = sk[i], b = sk[p];
            if (((i & k) == 0) ? key_less(b, a) : key_less(a, b)) { sk[i] = b; sk[p] = a; }
          }
        }
        __syncthreads();
      }
    for (uint32_t i = threadIdx.x; i < cc; i += blockDim.x) cur[base + i] = sk[i];
    __syncthreads();
  }
  for (uint64_t width = kBlockSort; width < c; width *= 2) {           // pairwise merges in HBM: each key finds its place by rank
    for (uint32_t i = threadIdx.x; i < c; i += blockDim.x) {
      const uint64_t a0 = (uint64_t)i / (2 * width) * (2 * width);
      const uint32_t a1 = (uint32_t)min(a0 + width, (uint64_t)c), b1 = (uint32_t)min(a0 + 2 * width, (uint64_t)c);
      const uint4 x = cur[i];
      const uint32_t pos = i < a1 ? (i - (uint32_t)a0) + rank_in(cur + a1, b1 - a1, x, false)
                                  : (i - a1) + rank_in(cur + a0, a1 - (uint32_t)a0, x, true);
      alt[a0 + pos] = x;
    }
    __syncthreads();
    uint4* t = cur; cur = alt; alt = t;
  }
  if (threadIdx.x == 0) {                                              // the greedy walk: kept keys to the segment's front
    long long last_end = -1;
    uint32_t k = 0;
    for (uint32_t j = 0; j < c; j++) {
      const uint4 x = cur[j];
      if ((long long)x.x >= last_end) { w.sorted[s0 + k++] = x; last_end = key_end(x); }
    }
    kept_sh = k;
  }
  __syncthreads();
  const uint32_t kc = kept_sh;
  long long d = 0;
  if (redact) for (uint32_t j = threadIdx.x; j < kc; j += blockDim.x) d += splice_delta(w, category, w.sorted[s0 + j]);
  *delta = block_sum(d, red);
  return kc;
}

// The same for a segment of 1 .. kWarpSort keys, one warp: bitonic sort in registers, the greedy walk done by all lanes in
// step.  Returns the number kept and, redacting, *delta (both on every lane).  Call from warp-uniform code.
__device__ __forceinline__ uint32_t warp_sort_keep(const ScanWork& w, const uint32_t* __restrict__ category, uint32_t s0, uint32_t c, int redact,
                                                   long long* delta) {
  const uint32_t lane = threadIdx.x & 31;
  uint4 v = lane < c ? w.sorted[s0 + lane] : pad_key();
  for (uint32_t k = 2; k <= 32; k <<= 1)
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      const uint4 o = shfl_key(v, j, true);
      const bool keep_min = ((lane & j) == 0) == ((lane & k) == 0);
      if (keep_min ? key_less(o, v) : key_less(v, o)) v = o;
    }
  long long last_end = -1;
  uint32_t keep = 0;
  for (uint32_t j = 0; j < c; j++) {
    const uint32_t s = __shfl_sync(0xffffffffu, v.x, j), e = __shfl_sync(0xffffffffu, key_end(v), j);
    if ((long long)s >= last_end) { keep |= 1u << j; last_end = e; }
  }
  const bool mine = (keep >> lane) & 1u;
  long long d = 0;
  if (mine) {
    w.sorted[s0 + __popc(keep & ((1u << lane) - 1u))] = v;
    if (redact) d = splice_delta(w, category, v);
  }
  for (int k = 16; k; k >>= 1) d += __shfl_xor_sync(0xffffffffu, d, k);
  *delta = d;
  return __popc(keep);
}

// exclusive prefix sums of a[0, count) in place, one block (count <= blockDim.x, a in shared memory); part: 32 elements of
// shared memory.  Call from block-uniform code.
template <typename T>
__device__ __forceinline__ void block_xscan_small(T* a, uint32_t count, T* part) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T v = threadIdx.x < count ? a[threadIdx.x] : (T)0;
  T incl = v;
  for (int d = 1; d < 32; d <<= 1) { const T t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (uint32_t)d) incl += t; }
  if (lane == 31) part[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const T wv = lane < blockDim.x / 32 ? part[lane] : (T)0;
    T wi = wv;
    for (int d = 1; d < 32; d <<= 1) { const T t = __shfl_up_sync(0xffffffffu, wi, d); if (lane >= (uint32_t)d) wi += t; }
    part[lane] = wi - wv;
  }
  __syncthreads();
  if (threadIdx.x < count) a[threadIdx.x] = part[warp] + incl - v;
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------- kernels
__global__ void __launch_bounds__(256) span_count_kernel(ScanWork w) {
  const uint32_t ns = min(w.counters[kCtrRawSpans], w.span_cap);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) atomicAdd(&w.seg_cnt[w.spans[(size_t)i * 6]], 1u);
}

// raw span -> its message's segment (positions inside a segment in arbitrary order: the sort fixes them)
__global__ void __launch_bounds__(256) span_scatter_kernel(ScanWork w, const uint32_t* __restrict__ rank) {
  const uint32_t ns = min(w.counters[kCtrRawSpans], w.span_cap);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) {
    const uint32_t* s = w.spans + (size_t)i * 6;
    const uint32_t msg = s[0], s16 = s[4], e16 = s[5];
    const uint32_t pos = w.seg_begin[msg] + atomicSub(&w.seg_cnt[msg], 1u) - 1u;
    w.sorted[pos] = make_uint4(s16, ~(e16 - s16), rank[s[1]], i);
  }
}

// Sort every message's segment and keep greedily: the kept keys move to the front of the segment, kept_cnt[m] = how many,
// out_len[m] = the message's redacted length (redact only).
__global__ void __launch_bounds__(kSortBlock) span_sort_keep_kernel(ScanWork w, const uint32_t* __restrict__ category, const uint32_t* __restrict__ off,
                                                                    uint32_t n, int redact) {
  const uint32_t lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) { w.kept_cnt[n] = 0; w.out_len[n] = 0; }

  // short segments: one warp each, bitonic sort in registers, the greedy walk done by all lanes in step
  const uint32_t nw = gridDim.x * (blockDim.x / 32);
  for (uint32_t m = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); m < n; m += nw) {
    const uint32_t s0 = w.seg_begin[m], c = w.seg_begin[m + 1] - s0;
    if (c > kWarpSort) continue;
    const uint32_t len = off[m + 1] - off[m];
    if (c == 0) { if (lane == 0) { w.kept_cnt[m] = 0; if (redact) w.out_len[m] = len; } continue; }
    long long delta = 0;
    const uint32_t kept = warp_sort_keep(w, category, s0, c, redact, &delta);
    if (lane == 0) { w.kept_cnt[m] = kept; if (redact) w.out_len[m] = (uint64_t)((long long)len + delta); }
  }

  // long segments: one block each (block-uniform branches)
  for (uint32_t m = blockIdx.x; m < n; m += gridDim.x) {
    const uint32_t s0 = w.seg_begin[m], c = w.seg_begin[m + 1] - s0;
    if (c <= kWarpSort) continue;
    long long delta = 0;
    const uint32_t kc = sort_keep_segment(w, category, s0, c, redact, &delta);
    if (threadIdx.x == 0) { w.kept_cnt[m] = kc; if (redact) w.out_len[m] = (uint64_t)((long long)(off[m + 1] - off[m]) + delta); }
    __syncthreads();
  }
}

// The whole resolver for a batch of a few messages (n <= kFewMsgs: cg_find_matches_one / cg_redact_one and the _few calls),
// one block, with the per-message arrays in shared memory: count per message -> exclusive scan -> scatter into message order
// -> each segment sorted and kept (one warp per segment of at most kWarpSort keys, the whole block per longer one, through
// warp_sort_keep / sort_keep_segment) -> exclusive scans of the kept counts and the output lengths -> everything
// span_emit_kernel writes for n messages.  The span count is read from device memory only.
__global__ void __launch_bounds__(kSortBlock) span_resolve_few_kernel(ScanWork w, const uint32_t* __restrict__ category,
                                                                      const uint32_t* __restrict__ rank, const uint32_t* __restrict__ off,
                                                                      uint32_t n, SpanOutputs o) {
  __shared__ uint32_t seg[kFewMsgs + 1];         // raw spans per message, then the first of its segment
  __shared__ uint32_t fill[kFewMsgs];            // keys scattered into each segment so far
  __shared__ uint32_t kept[kFewMsgs + 1];        // spans kept per message, then its first resolved span
  __shared__ unsigned long long olen[kFewMsgs + 1];   // redacted bytes per message, then its output offset
  __shared__ unsigned long long part[32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool incomplete = w.counters[kCtrErrors] != 0;
  const uint32_t c = incomplete ? 0u : min(w.counters[kCtrRawSpans], w.span_cap);
  const int redact = o.redact ? 1 : 0;
  for (uint32_t m = threadIdx.x; m <= n; m += blockDim.x) { seg[m] = 0; kept[m] = 0; olen[m] = 0; if (m < n) fill[m] = 0; }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < c; i += blockDim.x) atomicAdd(&seg[w.spans[(size_t)i * 6]], 1u);
  __syncthreads();
  block_xscan_small(seg, n + 1, reinterpret_cast<uint32_t*>(part));
  for (uint32_t i = threadIdx.x; i < c; i += blockDim.x) {
    const uint32_t* s = w.spans + (size_t)i * 6;
    const uint32_t m = s[0];
    w.sorted[seg[m] + atomicAdd(&fill[m], 1u)] = make_uint4(s[4], ~(s[5] - s[4]), rank[s[1]], i);
  }
  __syncthreads();
  for (uint32_t m = warp; m < n; m += blockDim.x / 32) {              // short segments: one warp each
    const uint32_t s0 = seg[m], cm = seg[m + 1] - s0;
    if (cm > kWarpSort) continue;
    long long delta = 0;
    const uint32_t k = cm ? warp_sort_keep(w, category, s0, cm, redact, &delta) : 0u;
    if (lane == 0) { kept[m] = k; if (redact) olen[m] = (unsigned long long)((long long)(off[m + 1] - off[m]) + delta); }
  }
  __syncthreads();
  for (uint32_t m = 0; m < n; m++) {                                   // long ones: the whole block each (block-uniform)
    const uint32_t s0 = seg[m], cm = seg[m + 1] - s0;
    if (cm <= kWarpSort) continue;
    long long delta = 0;
    const uint32_t k = sort_keep_segment(w, category, s0, cm, redact, &delta);
    if (threadIdx.x == 0) { kept[m] = k; if (redact) olen[m] = (unsigned long long)((long long)(off[m + 1] - off[m]) + delta); }
  }
  __syncthreads();
  block_xscan_small(kept, n + 1, reinterpret_cast<uint32_t*>(part));
  if (redact) block_xscan_small(olen, n + 1, part);
  const uint32_t total = kept[n];
  const uint64_t need = redact ? olen[n] : 0;
  uint32_t status = kResolveOk;
  if (!incomplete) {
    if (redact && (need >> 32)) status = kResolveTooLarge;
    else if (total > o.spans_cap || (redact && need > o.out_cap)) status = kResolveCapacity;
  }
  const bool go = !incomplete && status == kResolveOk;
  for (uint32_t r = threadIdx.x; r < total; r += blockDim.x) {
    uint32_t lo = 0, hi = n;                                           // kept[lo] <= r < kept[hi]
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (kept[mid] <= r) lo = mid; else hi = mid; }
    const uint4 k = w.sorted[seg[lo] + (r - kept[lo])];
    const uint32_t* s = w.spans + (size_t)k.w * 6;
    const uint32_t rule = s[1], sb = s[2], eb = s[3];
    if (r < o.spans_cap) {
      uint32_t* d = o.spans + (size_t)r * 6;
      d[0] = lo; d[1] = rule; d[2] = sb; d[3] = eb; d[4] = s[4]; d[5] = s[5];
    }
    if (redact) { w.sp_start[r] = off[lo] + sb; w.sp_len[r] = eb - sb; w.sp_cat[r] = category[rule]; }
  }
  for (uint32_t m = threadIdx.x; m <= n; m += blockDim.x) {
    w.kept_begin[m] = kept[m];
    if (redact) { w.out_off[m] = olen[m]; o.out_offsets[m] = (uint32_t)olen[m]; }
  }
  if (threadIdx.x == 0) {
    if (redact) { uint64_t* z = reinterpret_cast<uint64_t*>(o.sizes); z[0] = incomplete ? ~0ull : need; z[1] = incomplete ? ~0ull : total; }
    else *reinterpret_cast<uint32_t*>(o.sizes) = incomplete ? ~0u : total;
    w.counters[kCtrResolveStatus] = status;
    w.counters[kCtrResolved] = incomplete ? 0u : total;
    w.counters[kCtrDigests] = go && redact ? total : 0u;
    w.counters[kCtrSplice] = go && redact ? n : 0u;
  }
}

// The few-message result made contiguous for one D2H copy (layout: kernels.h, launch_span_pack_few).  The spans, sizes and
// output offsets are already in place (the resolver wrote them there); this adds the status, the packed length, the
// counter block and, redacting, the digests and the output bytes behind the spans -- when all of it fits in pack_cap bytes.
__global__ void __launch_bounds__(512) span_pack_few_kernel(ScanWork w, const uint32_t* __restrict__ digests, const uint8_t* __restrict__ out,
                                                            uint32_t* __restrict__ packed, uint32_t pack_cap, uint32_t n, int redact) {
  const uint32_t flags = w.counters[kCtrErrors], status = w.counters[kCtrResolveStatus];
  uint32_t ns = 0; uint64_t need = 0;
  if (redact) { const uint64_t* z = reinterpret_cast<const uint64_t*>(packed + kPackSizes); need = z[0]; ns = (uint32_t)z[1]; }
  else ns = packed[kPackSizes];
  const uint32_t at = pack_spans_at(n);
  const uint64_t len = (uint64_t)at + (uint64_t)ns * 24 + (redact ? (uint64_t)ns * 32 + need : 0);
  const bool fits = !flags && status == kResolveOk && len <= pack_cap;
  if (fits && redact) {
    uint32_t* dd = packed + at / 4 + (size_t)ns * 6;
    for (uint32_t i = threadIdx.x; i < ns * 8; i += blockDim.x) dd[i] = digests[i];
    uint8_t* ob = reinterpret_cast<uint8_t*>(dd + (size_t)ns * 8);
    for (uint32_t i = threadIdx.x; i < need; i += blockDim.x) ob[i] = out[i];
  }
  if (threadIdx.x < kCounterWords) packed[kPackCounters + threadIdx.x] = w.counters[threadIdx.x];
  if (threadIdx.x == 0) { packed[0] = fits ? (uint32_t)len : 0u; packed[1] = status; }
}

// Resolved span r = the (r - kept_begin[m])-th kept key of message m; sizes, status and the output offsets.
__global__ void __launch_bounds__(256) span_emit_kernel(ScanWork w, const uint32_t* __restrict__ category, const uint32_t* __restrict__ off,
                                                        uint32_t n, SpanOutputs o) {
  const bool incomplete = w.counters[kCtrErrors] != 0;
  const uint32_t total = w.kept_begin[n];
  const uint64_t need = o.redact ? w.out_off[n] : 0;
  uint32_t status = kResolveOk;
  if (!incomplete) {
    if (o.redact && (need >> 32)) status = kResolveTooLarge;
    else if (total > o.spans_cap || (o.redact && need > o.out_cap)) status = kResolveCapacity;
  }
  const bool go = !incomplete && status == kResolveOk;
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
  for (uint32_t r = tid; r < total; r += stride) {
    uint32_t lo = 0, hi = n;                                           // kept_begin[lo] <= r < kept_begin[hi]
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (w.kept_begin[mid] <= r) lo = mid; else hi = mid; }
    const uint4 k = w.sorted[w.seg_begin[lo] + (r - w.kept_begin[lo])];
    const uint32_t* s = w.spans + (size_t)k.w * 6;
    const uint32_t rule = s[1], sb = s[2], eb = s[3];
    if (!incomplete && r < o.spans_cap) {
      uint32_t* d = o.spans + (size_t)r * 6;
      d[0] = lo; d[1] = rule; d[2] = sb; d[3] = eb; d[4] = s[4]; d[5] = s[5];
    }
    if (o.redact) { w.sp_start[r] = off[lo] + sb; w.sp_len[r] = eb - sb; w.sp_cat[r] = category[rule]; }
  }
  if (o.redact) for (uint32_t m = tid; m <= n; m += stride) o.out_offsets[m] = (uint32_t)w.out_off[m];
  if (tid == 0) {
    if (o.redact) { uint64_t* z = reinterpret_cast<uint64_t*>(o.sizes); z[0] = incomplete ? ~0ull : need; z[1] = incomplete ? ~0ull : total; }
    else *reinterpret_cast<uint32_t*>(o.sizes) = incomplete ? ~0u : total;
    w.counters[kCtrResolveStatus] = status;
    w.counters[kCtrResolved] = incomplete ? 0u : total;
    w.counters[kCtrDigests] = go && o.redact ? total : 0u;
    w.counters[kCtrSplice] = go && o.redact ? n : 0u;
  }
}

}  // namespace

int launch_exclusive_scan(const uint32_t* d_in, uint32_t* d_out, uint32_t count, uint64_t* d_part, int sm_count, cudaStream_t stream) {
  return xscan<uint32_t>(d_in, d_out, count, reinterpret_cast<uint32_t*>(d_part), sm_count, stream);
}
int launch_exclusive_scan(const uint64_t* d_in, uint64_t* d_out, uint32_t count, uint64_t* d_part, int sm_count, cudaStream_t stream) {
  return xscan<uint64_t>(d_in, d_out, count, d_part, sm_count, stream);
}

int launch_span_resolve(const ScanWork& w, const uint32_t* d_off, uint32_t n, const SpanOutputs& o, int sm_count, cudaStream_t stream) {
  int k = 0;
  cudaMemsetAsync(w.seg_cnt, 0, ((size_t)n + 1) * 4, stream);
  span_count_kernel<<<sm_count * 4, 256, 0, stream>>>(w);
  k++;
  k += launch_exclusive_scan(w.seg_cnt, w.seg_begin, n + 1, w.scan_part, sm_count, stream);
  span_scatter_kernel<<<sm_count * 4, 256, 0, stream>>>(w, w.rule_rank);
  k++;
  span_sort_keep_kernel<<<sm_count * 2, kSortBlock, 0, stream>>>(w, w.rule_category, d_off, n, o.redact ? 1 : 0);
  k++;
  k += launch_exclusive_scan(w.kept_cnt, w.kept_begin, n + 1, w.scan_part, sm_count, stream);
  if (o.redact) k += launch_exclusive_scan(w.out_len, w.out_off, n + 1, w.scan_part, sm_count, stream);
  span_emit_kernel<<<sm_count * 4, 256, 0, stream>>>(w, w.rule_category, d_off, n, o);
  k++;
  return k;
}

int launch_span_resolve_few(const ScanWork& w, const uint32_t* d_off, uint32_t n, const SpanOutputs& o, cudaStream_t stream) {
  span_resolve_few_kernel<<<1, kSortBlock, 0, stream>>>(w, w.rule_category, w.rule_rank, d_off, n, o);
  return 1;
}

int launch_span_pack_few(const ScanWork& w, const uint32_t* d_digests, const uint8_t* d_out, uint32_t* d_packed, uint32_t pack_cap, uint32_t n,
                         bool redact, cudaStream_t stream) {
  span_pack_few_kernel<<<1, 512, 0, stream>>>(w, d_digests, d_out, d_packed, pack_cap, n, redact ? 1 : 0);
  return 1;
}

}  // namespace cg
