// tail_atomic_micro.cu -- what the scan step's tail pays for its single-word counters: K items, each of which takes one
// entry of a queue behind a counter word, on the grids the tail launches, every configuration timed in the same run.
//   confirm grid  132 x 1024 threads (one CTA per SM), items spread thinly over the grid-stride loop: one lane in 16 holds
//                 an item, two per 32-lane wave, as confirmed occurrences are spread over confirm_kernel's (gram, entry)
//                 pair waves.  Each item writes an 8-byte queue entry at the index the counter gave it.
//     NONE    no counter: the entry goes to a fixed place (the floor: the loop and the stores)
//     ONE     one atomicAdd per item on the one counter word (confirm_pairs before per-warp appends)
//     BALLOT  one atomicAdd per wave and warp, after a ballot
//     RING    a per-warp buffer of 32 entries in shared memory, written to the queue behind one atomicAdd whenever the next
//             wave would not fit, the rest at the end (confirm_kernel's occurrence appends)
//   resolve grid  8 x 132 x 256 threads, every 4th lane takes an item (resolve_kernel's spread), grid-stride; every item
//                 is a message of its own.  The chain resolve_kernel runs for a message's first occurrence:
//     CHAIN       volatile read of the message's slot word, atomicAdd on the slot counter, store of the slot's message,
//                 atomicCAS on the message's (distinct) slot word
//     CHAIN_WARP  the same with one atomicAdd per warp and round for all the warp's new slots
//     CHAIN_NONE  the same without the counter (slot = item index): the floor
// Counts: K = 11 k, 32 k, 110 k and 142 k (C2's hit messages at p_hit 1 %, its confirmed occurrences, hit messages at
// p_hit 10 %, occurrences of the other vocabulary; DESIGN.md §4.4).  Mean and best of 30 launches after 3, CUDA events.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o _bin/tail_atomic_micro tail_atomic_micro.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define FULL 0xffffffffu
enum : int { NONE = 0, ONE = 1, BALLOT = 2, RING = 3, CHAIN = 4, CHAIN_WARP = 5, CHAIN_NONE = 6 };
constexpr uint32_t kSpace = 16;            // confirm grid: index space per item (one lane in 16 holds one)

__device__ __forceinline__ uint32_t mix(uint32_t x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }

template <int M>
__global__ void __launch_bounds__(1024, 1) confirm_like(uint32_t k_items, uint32_t* __restrict__ ctr, uint2* __restrict__ q) {
  __shared__ uint2 buf[32][32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lt = (1u << lane) - 1u;
  const uint32_t space = k_items * kSpace, stride = gridDim.x * blockDim.x;
  uint32_t held = 0;
  auto flush = [&]() {
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(&ctr[0], held);
    base = __shfl_sync(FULL, base, 0);
    if (lane < held) q[base + lane] = buf[warp][lane];
    held = 0;
    __syncwarp();
  };
  for (uint32_t j0 = blockIdx.x * blockDim.x + threadIdx.x - lane; j0 < space; j0 += stride) {     // warp-uniform
    const uint32_t j = j0 + lane;
    const bool item = j < space && mix(j) % kSpace == 0;
    const uint2 e = make_uint2(j, mix(j + 1));
    if (M == NONE) { if (item) q[j / kSpace] = e; }
    if (M == ONE) { if (item) q[atomicAdd(&ctr[0], 1u)] = e; }
    if (M == BALLOT) {
      const uint32_t m = __ballot_sync(FULL, item);
      if (m) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&ctr[0], __popc(m));
        base = __shfl_sync(FULL, base, 0);
        if (item) q[base + __popc(m & lt)] = e;
      }
    }
    if (M == RING) {
      const uint32_t m = __ballot_sync(FULL, item);
      if (m) {
        if (held + __popc(m) > 32u) flush();
        if (item) buf[warp][held + __popc(m & lt)] = e;
        held += __popc(m);
        __syncwarp();
      }
    }
  }
  if (M == RING && held) flush();
}

template <int M>
__global__ void __launch_bounds__(256, 4) resolve_like(uint32_t k_items, uint32_t* __restrict__ ctr, uint32_t* __restrict__ slot_of, uint32_t* __restrict__ slot_msg) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x, lane = threadIdx.x & 31;
  for (uint32_t i = tid / 4, i0 = (tid - lane) / 4; i0 < k_items; i += stride / 4, i0 += stride / 4) {
    const bool item = tid % 4 == 0 && i < k_items;
    const uint32_t msg = item ? mix(i) % (k_items * 16u) : 0u;      // a message of its own (collisions are rare and harmless)
    const uint32_t s = item ? *reinterpret_cast<volatile uint32_t*>(&slot_of[msg]) : 0u;
    const bool need = item && s == 0xffffffffu;
    uint32_t mine = 0;
    if (M == CHAIN) { if (need) mine = atomicAdd(&ctr[0], 1u); }
    if (M == CHAIN_NONE) mine = i;
    if (M == CHAIN_WARP) {
      const uint32_t m = __ballot_sync(FULL, need);
      uint32_t base = 0;
      if (m) { if (lane == 0) base = atomicAdd(&ctr[0], __popc(m)); base = __shfl_sync(FULL, base, 0); }
      mine = base + __popc(m & ((1u << lane) - 1u));
    }
    if (need) {
      slot_msg[mine] = msg;
      if (atomicCAS(&slot_of[msg], 0xffffffffu, mine) != 0xffffffffu) slot_msg[mine] = 0xffffffffu;
    }
  }
}

struct Ctx { uint32_t* ctr; uint2* q; uint32_t* slot_of; uint32_t* slot_msg; int sms; };

template <int M>
static float run(const char* name, const Ctx& x, uint32_t k) {
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e9f, sum = 0.f; uint32_t cnt = 0;
  const int reps = 30;
  for (int r = 0; r < reps + 3; r++) {
    cudaMemset(x.ctr, 0, 16);
    if (M >= CHAIN) cudaMemset(x.slot_of, 0xff, (size_t)k * 16u * 4u);
    cudaEventRecord(e0);
    if (M < CHAIN) confirm_like<M><<<x.sms, 1024>>>(k, x.ctr, x.q);
    else resolve_like<M><<<x.sms * 8, 256>>>(k, x.ctr, x.slot_of, x.slot_msg);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (r >= 3) { sum += ms; if (ms < best) best = ms; }
  }
  cudaMemcpy(&cnt, x.ctr, 4, cudaMemcpyDeviceToHost);
  const float mean = sum / reps;
  printf("K %6u  %-12s mean %7.2f us  best %7.2f us  counter %7u  (%s)\n", k, name, mean * 1e3f, best * 1e3f, cnt, cudaGetErrorString(cudaGetLastError()));
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return mean * 1e3f;
}

int main() {
  int dev = 0, sms = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, dev);
  printf("%s, %d SMs; confirm grid %d x 1024 (one item per %u lanes), resolve grid %d x 256 (every 4th lane)\n", prop.name, sms, sms, kSpace, sms * 8);
  const uint32_t ks[4] = {11u << 10, 32u << 10, 110u << 10, 142u << 10};
  Ctx x; x.sms = sms;
  cudaMalloc(&x.ctr, 16); cudaMalloc(&x.q, (size_t)(142u << 10) * kSpace * 8); cudaMalloc(&x.slot_of, (size_t)(142u << 10) * 16 * 4);
  cudaMalloc(&x.slot_msg, (size_t)(142u << 10) * 4 * 2);
  for (int pass = 0; pass < 2; pass++) {           // every configuration twice, alternated
    printf("--- pass %d\n", pass + 1);
    for (uint32_t k : ks) {
      const float n0 = run<NONE>("none", x, k), a1 = run<ONE>("one/item", x, k), a2 = run<BALLOT>("one/wave", x, k), a3 = run<RING>("ring of 32", x, k);
      const float c0 = run<CHAIN_NONE>("chain none", x, k), c1 = run<CHAIN>("chain", x, k), c2 = run<CHAIN_WARP>("chain/warp", x, k);
      printf("K %6u  confirm grid: one/item %+.2f us over none (%.2f ns per item), one/wave %+.2f, ring %+.2f;  resolve chain: per item %+.2f us over none, per warp %+.2f\n",
             k, a1 - n0, (a1 - n0) * 1e3f / k, a2 - n0, a3 - n0, c1 - c0, c2 - c0);
    }
  }
  return 0;
}
