// wide_tile_micro.cu -- scan_kernel's stride-2 probe loop at 16 and at 32 bytes per lane and tile.
// Same loop shape as the kernel: two register buffers one tile ahead, the next tile's loads pinned behind the current
// tile's first use by a run-time-zero data dependency, one flag word per lane and round, one ballot per round.  A 128 KB
// bitmap in shared memory (the size scan_kernel stages), 1024 threads per CTA, one CTA per SM, a 256 MB buffer.
//   W = 1: a lane owns one 16-byte chunk per tile (512-byte warp tiles, four tiles per round)
//   W = 2: a lane owns chunks c and c + 32 (1 KB warp tiles, two 512-byte halves loaded back to back, two tiles per round)
// What it answers: is scan_kernel bound by the bytes each warp keeps in flight?  If so, W = 2 streams clearly faster.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o wide_tile_micro wide_tile_micro.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

#define FULL 0xffffffffu
constexpr int kThreads = 1024;
constexpr uint32_t kBitmapBytes = 128 * 1024, kMult = 0x9E3779B1u;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint4 ldg_stream(const uint8_t* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t fold(uint32_t w) {
  const uint32_t z = (w & 0x5f5f5f5fu) ^ 0x10101010u;
  const uint32_t nd = __byte_perm(z + 0x70707070u, 0, 0xba98);
  return z & (nd | 0xf0f0f0f0u);
}
__device__ __forceinline__ void probe(uint32_t bm, uint32_t key, uint32_t& flags) {
  const uint32_t hi = __umulhi(key, kMult);
  const uint32_t wv = lds32(bm + (hi & (kBitmapBytes - 4u)));
  flags = __funnelshift_l(wv << (key & 31u), flags, 1);
}
// the eight stride-2 probes of one 16-byte chunk; w4 = the first word of the next chunk
__device__ __forceinline__ uint32_t probe_chunk(uint32_t bm, const uint4& v, uint32_t w4) {
  const uint32_t f0 = fold(v.x), f1 = fold(v.y), f2 = fold(v.z), f3 = fold(v.w), f4 = fold(w4);
  uint32_t flags = 0;
  probe(bm, f0, flags); probe(bm, __funnelshift_r(f0, f1, 16), flags);
  probe(bm, f1, flags); probe(bm, __funnelshift_r(f1, f2, 16), flags);
  probe(bm, f2, flags); probe(bm, __funnelshift_r(f2, f3, 16), flags);
  probe(bm, f3, flags); probe(bm, __funnelshift_r(f3, f4, 16), flags);
  return flags;
}

template <int W>
__global__ void __launch_bounds__(kThreads, 1)
probe_kernel(const uint8_t* __restrict__ text, uint32_t end_chunk, const uint32_t* __restrict__ bitmap_g, uint32_t zero, uint32_t* __restrict__ out) {
  extern __shared__ __align__(128) uint8_t smem[];
  for (uint32_t i = threadIdx.x; i < kBitmapBytes / 16; i += kThreads) reinterpret_cast<uint4*>(smem)[i] = reinterpret_cast<const uint4*>(bitmap_g)[i];
  __syncthreads();
  const uint32_t bm = smem_u32(smem), lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = kThreads / 32;
  const bool last_lane = lane == 31;
  constexpr uint32_t kTile = 32u * W;                       // chunks per warp tile
  uint32_t c = (blockIdx.x * wpb + warp) * kTile + lane;
  const uint32_t cstep = gridDim.x * wpb * kTile;
  struct Buf { uint4 v[W]; uint32_t t; };
  auto load = [&](Buf& b, uint32_t cc) {
#pragma unroll
    for (int h = 0; h < W; h++) { b.v[h] = make_uint4(0, 0, 0, 0); if (cc + 32u * h < end_chunk) b.v[h] = ldg_stream(text + (size_t)(cc + 32u * h) * 16); }
    const uint32_t tc = cc + 32u * (W - 1) + 1u;
    b.t = 0; if (last_lane && tc < end_chunk) b.t = __ldg(reinterpret_cast<const uint32_t*>(text + (size_t)tc * 16));
  };
  Buf bA, bB; load(bA, c); bB = bA;
  uint32_t acc = 0, flagged = 0, words = 0;
  auto tile = [&](const Buf& cur, Buf& nxt, uint32_t cc) {
    uint32_t ncc = cc + cstep;
    asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(ncc) : "r"(cur.v[0].x), "r"(zero));
    load(nxt, ncc);
    if (W == 1) {
      uint32_t w4 = __shfl_down_sync(FULL, cur.v[0].x, 1); if (last_lane) w4 = cur.t;
      acc = acc << 8 | probe_chunk(bm, cur.v[0], w4);
    } else {
      // first half: lane l + 1's first-half word; lane 31 takes lane 0's second-half word (chunk base + 32)
      const uint32_t wa = __shfl_sync(FULL, lane == 0 ? cur.v[W - 1].x : cur.v[0].x, (lane + 1) & 31);
      uint32_t wb = __shfl_down_sync(FULL, cur.v[W - 1].x, 1); if (last_lane) wb = cur.t;
      acc = acc << 16 | probe_chunk(bm, cur.v[0], wa) << 8 | probe_chunk(bm, cur.v[W - 1], wb);
    }
  };
#pragma unroll 1
  while (c - lane < end_chunk) {
    if (W == 1) { tile(bA, bB, c); tile(bB, bA, c + cstep); tile(bA, bB, c + 2u * cstep); tile(bB, bA, c + 3u * cstep); c += 4u * cstep; }
    else { tile(bA, bB, c); tile(bB, bA, c + cstep); c += 2u * cstep; }
    const uint32_t m = __ballot_sync(FULL, acc != 0);
    if (m) { words += lane == 0 ? __popc(m) : 0u; flagged += __popc(acc); acc = 0; }
  }
  flagged = __reduce_add_sync(FULL, flagged);
  if (lane == 0) { atomicAdd(&out[0], flagged); atomicAdd(&out[1], words); }
}

__global__ void gen_text(uint8_t* t, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t r = (uint32_t)i * 2654435761u; r ^= r >> 15; r *= 2246822519u; r ^= r >> 13; r *= 3266489917u; r ^= r >> 16;
    t[i] = (r % 7u == 0) ? ' ' : (uint8_t)('a' + (r >> 8) % 26u);
  }
}
__global__ void copy_read(const uint4* __restrict__ t, size_t n16, uint32_t* out) {
  uint32_t acc = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) { uint4 v = ldg_stream(reinterpret_cast<const uint8_t*>(t + i)); acc ^= v.x ^ v.y ^ v.z ^ v.w; }
  if (acc == 0x12345678u) out[0] = acc;
}

template <int W>
static float run(const char* name, const uint8_t* d_text, size_t bytes, const uint32_t* d_bm, uint32_t* d_out, int sms) {
  cudaFuncSetAttribute(probe_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBitmapBytes);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e9f, sum = 0.f; uint32_t cnt[2] = {0, 0};
  const int reps = 20;
  for (int r = 0; r < reps + 2; r++) {
    cudaMemset(d_out, 0, 8);
    cudaEventRecord(e0);
    probe_kernel<W><<<sms, kThreads, kBitmapBytes>>>(d_text, (uint32_t)(bytes / 16), d_bm, 0u, d_out);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (r >= 2) { sum += ms; if (ms < best) best = ms; }
  }
  cudaMemcpy(cnt, d_out, 8, cudaMemcpyDeviceToHost);
  printf("%-22s best %8.1f us  %7.1f GB/s   mean %8.1f us  %7.1f GB/s   flagged grams %u  flag words %u  (%s)\n", name, best * 1e3, bytes / (best * 1e-3) / 1e9,
         sum / reps * 1e3, bytes / (sum / reps * 1e-3) / 1e9, cnt[0], cnt[1], cudaGetErrorString(cudaGetLastError()));
  return best;
}

int main() {
  const size_t bytes = (size_t)1 << 28;      // 256 MB = 1 Mi x 256 B
  int dev = 0, sms = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  uint8_t* d_text; uint32_t *d_bm, *d_out;
  cudaMalloc(&d_text, bytes + 4096); cudaMalloc(&d_bm, kBitmapBytes); cudaMalloc(&d_out, 64);
  gen_text<<<sms * 8, 256>>>(d_text, bytes + 4096);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int r = 0; r < 3; r++) {
    cudaEventRecord(e0); copy_read<<<sms * 16, 256>>>(reinterpret_cast<const uint4*>(d_text), bytes / 16, d_out); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (r == 2) printf("grid-stride LDG.128 read (one load per thread and step; a reference, not a ceiling)  %8.1f us  %7.1f GB/s\n", ms * 1e3, bytes / (ms * 1e-3) / 1e9);
  }
  const double dens[2] = {0.003, 0.013};
  for (double d : dens) {
    std::vector<uint32_t> bm(kBitmapBytes / 4, 0);
    srand(11);
    const size_t nbits = (size_t)(d * kBitmapBytes * 8);
    for (size_t i = 0; i < nbits; i++) { uint32_t b = ((uint32_t)rand() * 32768u + (uint32_t)rand()) % (kBitmapBytes * 8); bm[b >> 5] |= 1u << (b & 31); }
    cudaMemcpy(d_bm, bm.data(), kBitmapBytes, cudaMemcpyHostToDevice);
    printf("--- bitmap density %.3f, %d SMs x %d threads\n", d, sms, kThreads);
    for (int k = 0; k < 2; k++) {                 // alternated, twice
      run<1>("stride2 16 B / lane", d_text, bytes, d_bm, d_out, sms);
      run<2>("stride2 32 B / lane", d_text, bytes, d_bm, d_out, sms);
    }
  }
  return 0;
}
