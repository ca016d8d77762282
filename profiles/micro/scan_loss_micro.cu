// scan_loss_micro.cu -- where scan_kernel loses the bare stride-2 loop's streaming rate: the kernel's extras added to the
// loop of wide_tile_micro.cu (1 KB warp tiles, two register buffers one tile ahead behind a run-time-zero dependency, 128
// KB bitmap in shared memory, 1024 threads, one CTA per SM, 256 MB = 1 Mi x 256 B, the C2 batch) one at a time, each
// configuration timed in the same run:
//   RING   per round, lanes with a non-zero flag word push (chunk, word) to a per-warp ring in shared memory; 32 entries at
//          a time go to a queue in HBM.  BLOCK: lane 0 takes the block with an atomicAdd on one address and every lane waits
//          for its result (what scan_kernel does); RESV: the block was reserved one append earlier, the atomic's result is
//          not needed until the next append, and the real entry count goes out once per warp at the end.
//   TRIG   the trigger test of scan_kernel<2, 1, ...>: one folded byte compared per word, a vote per half.
//   HEAD   a stand-in for the head check on block 0: every thread walks three chains of eight dependent global loads
//          before its loop (the 500-rule set: 1 500 checks, a few dependent loads each).
//   EARLY  the first tile's loads are issued before the wait for the bitmap (TMA bulk copy, mbarrier), not after it.
//   BAL    tiles dealt to the warps of the grid CTA-interleaved (warp w of CTA b is warp w x grid + b), so that the tiles
//          left over after the last full round go to one or two warps of every SM instead of all warps of the first CTAs.
// The bitmap is filled at random to the density that flags as many grams on this text as C2 does (about 0.8 M flag
// words per 256 MB).
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o _bin/scan_loss_micro scan_loss_micro.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

#define FULL 0xffffffffu
constexpr int kThreads = 1024;
constexpr uint32_t kBitmapBytes = 128 * 1024, kMult = 0x9E3779B1u, kRing = 64;
enum : int { RING = 1, RESV = 2, TRIG = 4, HEAD = 8, EARLY = 16, BAL = 32 };

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint4 ldg_stream(const uint8_t* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t fold_z(uint32_t w) { return (w & 0x5f5f5f5fu) ^ 0x10101010u; }
__device__ __forceinline__ uint32_t fold_key(uint32_t z) { return z & (__byte_perm(z + 0x70707070u, 0, 0xba98) | 0xf0f0f0f0u); }
__device__ __forceinline__ void probe(uint32_t bm, uint32_t key, uint32_t& flags) {
  const uint32_t hi = __umulhi(key, kMult);
  flags = __funnelshift_l(lds32(bm + (hi & (kBitmapBytes - 4u))) << (key & 31u), flags, 1);
}
__device__ __forceinline__ uint32_t differs(uint32_t z, uint32_t splat) { return (z ^ splat) + 0x7f7f7f7fu; }

__device__ __forceinline__ void mbar_wait(uint64_t* bar) {
  asm volatile("{\n.reg .pred p;\nW:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n@p bra D;\nbra W;\nD:\n}\n" ::"r"(smem_u32(bar)) : "memory");
}

template <int F>
__global__ void __launch_bounds__(kThreads, 1)
loss_kernel(const uint8_t* __restrict__ text, uint32_t end_chunk, const uint8_t* __restrict__ bitmap_g, const uint32_t* __restrict__ chain, uint32_t zero,
            uint32_t* __restrict__ ctr, uint2* __restrict__ q, uint32_t q_cap) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = kThreads / 32, lt = (1u << lane) - 1u;
  const bool last_lane = lane == 31;
  if (threadIdx.x == 0) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar))); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar)), "r"(kBitmapBytes) : "memory");
    for (uint32_t o = 0; o < kBitmapBytes; o += 32768u)
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem + o)), "l"(bitmap_g + o), "r"(32768u), "r"(smem_u32(&bar)) : "memory");
  }
  const uint32_t gw = (F & BAL) ? warp * gridDim.x + blockIdx.x : blockIdx.x * wpb + warp;
  uint32_t c = gw * 64u + lane;
  const uint32_t cstep = gridDim.x * wpb * 64u;
  struct Buf { uint4 a, b; uint32_t t; };
  auto load = [&](Buf& v, uint32_t cc) {
    v.a = make_uint4(0, 0, 0, 0); v.b = v.a; v.t = 0;
    if (cc < end_chunk) v.a = ldg_stream(text + (size_t)cc * 16);
    if (cc + 32u < end_chunk) v.b = ldg_stream(text + (size_t)(cc + 32u) * 16);
    if (last_lane && cc + 33u < end_chunk) v.t = __ldg(reinterpret_cast<const uint32_t*>(text + (size_t)(cc + 33u) * 16));
  };
  Buf bA, bB;
  if (F & EARLY) load(bA, c);
  mbar_wait(&bar);
  if (!(F & EARLY)) load(bA, c);
  bB = bA;
  uint32_t sink = 0;
  if ((F & HEAD) && blockIdx.x == 0) {
    for (int r = 0; r < 3; r++) { uint32_t p = threadIdx.x * 3u + r; for (int k = 0; k < 8; k++) p = chain[p & 65535u]; sink += p; }
  }
  const uint32_t bm = smem_u32(smem), ring = smem_u32(smem + kBitmapBytes) + warp * kRing * 8;
  const uint32_t splat = (('=' & 0x5fu) ^ 0x10u) * 0x01010101u;
  uint32_t acc = 0, h = 0, t = 0, resv = 0, real = 0; bool has_resv = false;
  auto half = [&](const uint4& v, uint32_t w4) {
    const uint32_t z0 = fold_z(v.x), z1 = fold_z(v.y), z2 = fold_z(v.z), z3 = fold_z(v.w);
    const uint32_t f0 = fold_key(z0), f1 = fold_key(z1), f2 = fold_key(z2), f3 = fold_key(z3), f4 = fold_key(fold_z(w4));
    uint32_t flags = 0;
    probe(bm, f0, flags); probe(bm, __funnelshift_r(f0, f1, 16), flags); probe(bm, f1, flags); probe(bm, __funnelshift_r(f1, f2, 16), flags);
    probe(bm, f2, flags); probe(bm, __funnelshift_r(f2, f3, 16), flags); probe(bm, f3, flags); probe(bm, __funnelshift_r(f3, f4, 16), flags);
    acc = acc << 8 | flags;
    if (F & TRIG) {
      const bool trig = (differs(z0, splat) & differs(z1, splat) & differs(z2, splat) & differs(z3, splat) & 0x80808080u) != 0x80808080u;
      if (__any_sync(FULL, trig)) { sink += trig; __syncwarp(); }
    }
  };
  auto tile = [&](const Buf& cur, Buf& nxt, uint32_t cc) {
    uint32_t ncc = cc + cstep;
    asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(ncc) : "r"(cur.a.x), "r"(zero));
    load(nxt, ncc);
    const uint32_t wa = __shfl_sync(FULL, lane == 0 ? cur.b.x : cur.a.x, (lane + 1) & 31);
    uint32_t wb = __shfl_down_sync(FULL, cur.b.x, 1); if (last_lane) wb = cur.t;
    half(cur.a, wa); half(cur.b, wb);
  };
  auto append = [&](uint32_t k) {          // k <= 32 ring entries -> the queue
    uint32_t base;
    if (F & RESV) {
      base = __shfl_sync(FULL, resv, 0); has_resv = false; real += k;
      if (base + lane < q_cap) {
        uint2 e = make_uint2(0u, 0u);
        if (lane < k) asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(e.x), "=r"(e.y) : "r"(ring + (((h + lane) & (kRing - 1)) << 3)));
        q[base + lane] = e;
      }
    } else {
      base = 0;
      if (lane == 0) base = atomicAdd(&ctr[0], k);
      base = __shfl_sync(FULL, base, 0);
      if (lane < k) {
        uint2 e;
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(e.x), "=r"(e.y) : "r"(ring + (((h + lane) & (kRing - 1)) << 3)));
        if (base + lane < q_cap) q[base + lane] = e;
      }
    }
    h += k;
  };
  uint32_t words = 0;
#pragma unroll 1
  while (c - lane < end_chunk) {
    tile(bA, bB, c); tile(bB, bA, c + cstep); c += 2u * cstep;
    const uint32_t m = __ballot_sync(FULL, acc != 0);
    if (m) {
      if (F & RING) {
        if (acc) asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(ring + (((t + __popc(m & lt)) & (kRing - 1)) << 3)), "r"(c), "r"(acc) : "memory");
        t += __popc(m);
        if ((F & RESV) && !has_resv) { if (lane == 0) resv = atomicAdd(&ctr[1], 32u); has_resv = true; }
        if (t - h >= 32u) {
          __syncwarp(); append(32u);
          if ((F & RESV) && t != h) { if (lane == 0) resv = atomicAdd(&ctr[1], 32u); has_resv = true; }
        }
      } else words += lane == 0 ? __popc(m) : 0u;
      acc = 0;
    }
  }
  __syncwarp();
  if ((F & RING) && t != h) append(t - h);
  if ((F & RESV) && lane == 0 && real) atomicAdd(&ctr[0], real);
  if (!(F & RING) && lane == 0 && words) atomicAdd(&ctr[0], words);
  if (sink == 0x12345678u) ctr[2] = sink;
}

__global__ void gen_text(uint8_t* t, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t r = (uint32_t)i * 2654435761u; r ^= r >> 15; r *= 2246822519u; r ^= r >> 13; r *= 3266489917u; r ^= r >> 16;
    t[i] = (r % 7u == 0) ? ' ' : (r % 53u == 0) ? '=' : (uint8_t)('a' + (r >> 8) % 26u);
  }
}

struct Ctx { const uint8_t* text; size_t bytes; const uint8_t* bm; const uint32_t* chain; uint32_t* ctr; uint2* q; uint32_t q_cap; int sms; };

template <int F>
static void run(const char* name, const Ctx& x, float* best_out) {
  const int smem = (int)(kBitmapBytes + 32 * kRing * 8);
  cudaFuncSetAttribute(loss_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e9f, sum = 0.f; uint32_t cnt[2] = {0, 0};
  const int reps = 30;
  for (int r = 0; r < reps + 3; r++) {
    cudaMemset(x.ctr, 0, 16);
    cudaEventRecord(e0);
    loss_kernel<F><<<x.sms, kThreads, smem>>>(x.text, (uint32_t)(x.bytes / 16), x.bm, x.chain, 0u, x.ctr, x.q, x.q_cap);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (r >= 3) { sum += ms; if (ms < best) best = ms; }
  }
  cudaMemcpy(cnt, x.ctr, 8, cudaMemcpyDeviceToHost);
  const float mean = sum / reps;
  printf("%-44s best %7.1f us %6.0f GB/s  mean %7.1f us %6.0f GB/s  flag words %u  reserved %u  (%s)\n", name, best * 1e3, x.bytes / (best * 1e-3) / 1e9,
         mean * 1e3, x.bytes / (mean * 1e-3) / 1e9, cnt[0], cnt[1], cudaGetErrorString(cudaGetLastError()));
  if (best_out) *best_out = mean;
}

int main(int argc, char** argv) {
  const double density = argc > 1 ? atof(argv[1]) : 0.0062;
  const size_t bytes = (size_t)1 << 28;
  int dev = 0, sms = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, dev);
  printf("%s, %d SMs x %d threads, 256 MB, bitmap density %.4f\n", prop.name, sms, kThreads, density);
  Ctx x; x.bytes = bytes; x.sms = sms; x.q_cap = 1u << 24;
  uint8_t* d_text; uint8_t* d_bm; uint32_t *d_chain, *d_ctr; uint2* d_q;
  cudaMalloc(&d_text, bytes + 4096); cudaMalloc(&d_bm, kBitmapBytes); cudaMalloc(&d_chain, 65536 * 4); cudaMalloc(&d_ctr, 16); cudaMalloc(&d_q, (size_t)x.q_cap * 8);
  gen_text<<<sms * 8, 256>>>(d_text, bytes + 4096);
  std::vector<uint32_t> bm(kBitmapBytes / 4, 0), ch(65536);
  srand(11);
  const size_t nbits = (size_t)(density * kBitmapBytes * 8);
  for (size_t i = 0; i < nbits; i++) { uint32_t b = ((uint32_t)rand() * 32768u + (uint32_t)rand()) % (kBitmapBytes * 8); bm[b >> 5] |= 1u << (b & 31); }
  for (uint32_t i = 0; i < 65536; i++) ch[i] = ((uint32_t)rand() * 32768u + (uint32_t)rand()) & 65535u;
  cudaMemcpy(d_bm, bm.data(), kBitmapBytes, cudaMemcpyHostToDevice); cudaMemcpy(d_chain, ch.data(), 65536 * 4, cudaMemcpyHostToDevice);
  x.text = d_text; x.bm = d_bm; x.chain = d_chain; x.ctr = d_ctr; x.q = d_q;
  for (int k = 0; k < 2; k++) {            // every configuration twice, alternated
    printf("--- pass %d\n", k + 1);
    run<0>("bare loop", x, nullptr);
    run<RING>("+ ring, blocking append", x, nullptr);
    run<RING | TRIG>("+ ring, blocking append + trigger", x, nullptr);
    run<RING | TRIG | HEAD>("+ ... + head stand-in on block 0", x, nullptr);
    run<RING | RESV | TRIG | HEAD>("  append reserved ahead", x, nullptr);
    run<RING | RESV | TRIG>("  append reserved ahead, no head", x, nullptr);
    run<RING | RESV | TRIG | EARLY>("  ... + first loads before the bitmap wait", x, nullptr);
    run<RING | RESV | TRIG | EARLY | BAL>("  ... + CTA-interleaved tiles", x, nullptr);
    run<EARLY>("bare loop, first loads before the wait", x, nullptr);
    run<BAL>("bare loop, CTA-interleaved tiles", x, nullptr);
    run<RING | RESV>("bare loop + ring, append reserved ahead", x, nullptr);
  }
  return 0;
}
