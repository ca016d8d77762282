// scan_kernels.cu -- sm_90a kernels of the message-scan hot path.
//
//   reset_kernel    start of a step: counters, slot table, the candidate / hit rows the previous step used.
//   scan_kernel     every byte of the batch buffer through the gram filter: 4-byte grams folded, hashed and tested against
//                   a bitmap in shared memory (image staged with TMA bulk copies, completion on an mbarrier); lanes with
//                   flagged grams push (chunk, flag word) to a queue in HBM, compacted with warp ballots.
//   confirm_kernel  flagged grams: reloaded, recheck map, table probes, exact factor comparison -- tables in shared memory,
//                   work handed from stage to stage in ballot-compacted waves.
//   resolve_kernel  level 2: message of every confirmed factor occurrence; RegExp.test around it by the bit-parallel
//                   island matcher (bitprog.h), or a direct hit, or a (message, rule) pair for the VM.
//                   (resolve_views_kernel: the same for the rules of each message's view only.)
//   verify_kernel   exact ECMAScript semantics for the queued pairs: a Pike VM over UTF-16 units
//                   decoded on the fly from the UTF-8 bytes (leftmost-first, global-exec
//                   iteration of registry.ts:225-236, RegExp.test of context.ts:9-25).
//   finalize_kernel per-message result words from the verified-hit bitmaps.
//
// Replaces the two hot loops of the reference: gov/src/conditions/context.ts:9-25 (rules x
// RegExp.test) and gov/src/redaction/registry.ts:212-242 (P global-exec passes per string).
#include "kernels.h"
#include "rulec.h"
#include "pike_vm.h"
#include "bitprog.h"
#include "gram_filter.h"
#include <algorithm>

namespace cg {

// ------------------------------------------------------------------------------------------
// PTX helpers: mbarrier + TMA 1-D bulk copy (global -> shared)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
// (reads that must not push the level-1b tables out of L1: the text is touched once, the tables by every thread)
__device__ __forceinline__ uint32_t ldg_stream32(const void* p) {
  uint32_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ldg_stream(const uint8_t* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

// ------------------------------------------------------------------------------------------
// level 1: the gram filter.  Position-parallel: a warp tile is 1 KB of the batch buffer made of two 512-byte halves; lane
// l owns 16-byte chunk c = tile base + l of the first half and chunk c + 32 of the second (two LDG.128, each half one
// coalesced 512-byte sweep), no per-message state, so long and ragged messages need no special handling.
//   1a  every aligned 4-byte gram (stride 4) or every even-offset gram (stride 2) is folded SWAR-style, hashed with one
//       IMAD and tested against the bitmap in shared memory (two bits of one word).  Result bits are funnel-shifted
//       into a per-lane flag word; a warp ballot decides whether anything has to be looked at.
//       Flag-word layout (flagged_gram_pos decodes it): a tile adds 2 * half_bits bits, its first half's probes above its
//       second half's, probe 0 of a half highest; a round is as many tiles as fill 32 bits (two at stride 2, four at
//       stride 4), the oldest tile highest, and the lane's queue entry carries its first-half chunk after the round.
//   1b  lanes with flagged grams push (chunk, flag word) to a per-warp ring in shared memory, which goes to a queue in HBM
//       128 entries at a time; confirm_kernel takes it from there (recheck map, level-1b lookup, exact factor, message).  Confirmed factor
//       occurrences go to the queue in HBM, one atomic each (they are rare).
// ------------------------------------------------------------------------------------------
constexpr int kScanThreads = 1024;      // 32 warps, one CTA per SM
constexpr uint32_t kAppend = 128;       // (chunk, flag word) pairs a warp collects before it appends them to the queue in HBM, one atomic
constexpr uint32_t kRing = 256;         // ring entries per warp (a power of two): fewer than kAppend + one round's 32 are ever held
constexpr uint32_t kScanRingBytes = (kScanThreads / 32) * kRing * 8;
constexpr uint32_t kTileChunks = 64;    // 16-byte chunks per warp tile: two halves of 32
// probe bits per 16-byte chunk = grams per chunk (stride 2: 8, stride 4: 4); tiles per round = 32 / (2 * half_bits)
__host__ __device__ constexpr uint32_t half_bits(uint32_t nprobe) { return 4u * nprobe; }

// the byte position of the gram behind bit `bit` of a flag word (scan_kernel's layout above).  newest = 16 x the lane's
// first-half chunk in the round's last tile = 16 x (queued chunk - cstep); cstep16 = 16 x the chunks between a warp's
// consecutive tiles (grid x warps per CTA x kTileChunks).  Probe j of a tile (first half first) is j = ~bit mod
// 2 * half_bits; a chunk's probes are stride bytes apart, so every term is a shift or a mask of the bit number.
template <int NPROBE>
__device__ __forceinline__ uint32_t flagged_gram_pos(uint32_t newest, uint32_t bit, uint32_t cstep16) {
  constexpr uint32_t hb = half_bits(NPROBE), lhb = NPROBE == 2 ? 3u : 2u, stride_shift = NPROBE == 2 ? 1u : 2u;
  static_assert(hb == 1u << lhb && (hb << stride_shift) == 16u, "half_bits probes, stride bytes apart, cover one 16-byte chunk");
  const uint32_t j = ~bit;
  return newest - (bit >> (lhb + 1u)) * cstep16 + ((j >> lhb) & 1u) * (kTileChunks / 2u * 16u) + ((j & (hb - 1u)) << stride_shift);
}

__device__ __forceinline__ uint32_t lds_u32(uint32_t saddr) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr)); return v; }

struct QueueEmit {
  const ScanWork& w;
  __device__ __forceinline__ void operator()(uint32_t t0, uint32_t f) {
    const uint32_t k = atomicAdd(&w.counters[kCtrConfirmed], 1u);
    if (k < w.l1_cap) { w.l1_pos[k] = t0; w.l1_fac[k] = f; } else atomicOr(&w.counters[kCtrErrors], ERR_L1_OVERFLOW);
  }
};

// The hot loop is bound by the integer ALU pipe (LOP3 / SHF / PRMT: 16 lanes per SM sub-partition and clock), not by
// instruction issue: constants that would cost a second LOP3 as immediates sit in registers, and additions go through
// IMAD (x * one + c, `one` a run-time 1 the compiler cannot fold) so that they execute on the FMA pipe instead.
struct HotConst { uint32_t c5f, c10, one, mask; };            // mask = bitmap bytes - 4
// z = (w & 0x5f5f5f5f) ^ 0x10101010 per byte (one LOP3); the gram key drops the low nibble of the digit bytes (z < 0x10)
__device__ __forceinline__ uint32_t fold_z(uint32_t w, const HotConst& k) {
  uint32_t z;
  asm("lop3.b32 %0, %1, %2, %3, 0x6a;" : "=r"(z) : "r"(w), "r"(k.c5f), "r"(k.c10));
  return z;
}
__device__ __forceinline__ uint32_t fold_key(uint32_t z, const HotConst& k) {
  uint32_t y, keep, f;
  asm("mad.lo.u32 %0, %1, %2, 0x70707070;" : "=r"(y) : "r"(z), "r"(k.one));
  asm("prmt.b32 %0, %1, %1, 0xba98;" : "=r"(keep) : "r"(y));                                 // sign-replicate: 0xff for non-digit bytes
  asm("lop3.b32 %0, %1, %2, 0xf0f0f0f0, 0xe0;" : "=r"(f) : "r"(z), "r"(keep));               // z & (keep | 0xf0f0f0f0)
  return f;
}
// one probe of the bitmap: word at byte address hi32(key * M) & bm_mask (one IMAD.HI on the FMA pipe, one LOP3), bit
// 31 - (key & 31) of it -- the bit index comes straight from the folded first byte, the variable shift only looks at the
// low five bits of its operand -- shifted into `flags`.  Five instructions per probe.
template <int BLOOM2>
__device__ __forceinline__ void gram_probe(uint32_t bm, const HotConst& k, uint32_t key, uint32_t& flags) {
  const uint32_t hi = __umulhi(key, kGramMult);
  const uint32_t wv = lds_u32(bm + (hi & k.mask));
  uint32_t t = wv << (key & 31u);
  if (BLOOM2) t &= wv << ((hi >> 17) & 31u);
  flags = __funnelshift_l(t, flags, 1);
}
// trigger bytes, compared in the folded domain (z): bit 7 of every byte of the result is CLEAR where z equals the splatted
// folded trigger byte (z ^ splat <= 0x5f, so adding 0x7f carries into bit 7 exactly when the byte differs; no carry across bytes)
__device__ __forceinline__ uint32_t differs(uint32_t z, uint32_t splat_z, uint32_t one) {
  uint32_t y; const uint32_t e = z ^ splat_z;
  asm("mad.lo.u32 %0, %1, %2, 0x7f7f7f7f;" : "=r"(y) : "r"(e), "r"(one));
  return y;
}

// what the rare paths need (kept out of line: the hot loop must stay small enough for the instruction cache)
struct ScanCtx { GramTables T; const uint8_t* bytes; uint32_t begin, end; };

// trigger bytes inside one 16-byte chunk: bit 8k+7 of mk_j set = byte k of word j equals a trigger byte in the folded
// domain (which merges case and bit 7), so every marked byte is compared again exactly
__device__ __forceinline__ void trigger_chunk(const DevRuleset& rs, const ScanWork& w, const ScanCtx& c, uint32_t mk0, uint32_t mk1, uint32_t mk2, uint32_t mk3, uint32_t chunk) {
  QueueEmit emit{w};
#pragma unroll 1
  for (uint32_t j = 0; j < 4; j++) {
    uint32_t mk = j == 0 ? mk0 : j == 1 ? mk1 : j == 2 ? mk2 : mk3;
    while (mk) {
      const uint32_t bitpos = 31u - __clz(mk); mk &= ~(1u << bitpos);
      const uint32_t pos = chunk * 16u + 4u * j + (bitpos >> 3);
      if (pos < c.begin || pos >= c.end) continue;
      const uint32_t by = c.bytes[pos];
      for (uint32_t t = 0; t < rs.n_trig; t++) if (by == rs.trig_byte[t]) gram_trigger(rs, c.T, t, c.bytes, c.begin, c.end, pos, emit);
    }
  }
}

template <int NPROBE, int NTRIG, int BLOOM2>
__global__ void __launch_bounds__(kScanThreads, 1)
scan_kernel(const __grid_constant__ DevRuleset rs, const __grid_constant__ ScanWork w, const uint8_t* __restrict__ bytes, const uint32_t* __restrict__ off, uint32_t n,
            uint64_t* __restrict__ words) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar;
  if (threadIdx.x == 0) { mbar_init(&bar, 1); fence_barrier_init(); }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bar, rs.image_bytes);                        // (the bitmap; everything else the rule set consists of is confirm_kernel's)
    for (uint32_t o = 0; o < rs.image_bytes; o += 32768u) {
      uint32_t len = rs.image_bytes - o < 32768u ? rs.image_bytes - o : 32768u;
      tma_bulk_g2s(smem + o, rs.image + o, len, &bar);
    }
  }
  // while the image is in flight: result words start at zero (finalize_kernel fills in the messages that hit)
  for (uint32_t i = blockIdx.x * kScanThreads + threadIdx.x; i < n; i += gridDim.x * kScanThreads) words[i] = 0ull;
  ScanCtx ctx;
  ctx.bytes = bytes; ctx.begin = off[0]; ctx.end = off[n];
  const uint32_t begin = ctx.begin, end = ctx.end;
  mbar_wait(&bar, 0);

  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = kScanThreads / 32;
  uint32_t lt = (1u << lane) - 1u; const uint32_t FULL = 0xffffffffu;
  asm volatile("" : "+r"(lt));                // (loop invariants the compiler would otherwise recompute in every iteration of the hot loop)
  const uint32_t bm = smem_u32(smem);
  const uint32_t ring1 = smem_u32(smem + rs.image_bytes) + warp * (kRing * 8);
  ctx.T.factors = rs.factors; ctx.T.bytesets = rs.bytesets; ctx.T.bucket_start = rs.bucket_start; ctx.T.entries = rs.entries;    // (triggers only)
  HotConst hk; hk.c5f = rs.hot_c5f; hk.c10 = rs.hot_c10; hk.one = rs.hot_one; hk.mask = rs.bm_mask;
  asm volatile("" : "+r"(hk.c5f), "+r"(hk.c10), "+r"(hk.one), "+r"(hk.mask));

  const uint32_t first_chunk = begin >> 4;
  uint32_t end_chunk = (end + 15u) >> 4;       // 16-byte chunks [first, end)
  // folded (z domain) trigger bytes, splatted
  uint32_t splat0 = NTRIG > 0 ? (((rs.trig_byte[0] & 0x5fu) ^ 0x10u) * 0x01010101u) : 0u, splat1 = NTRIG > 1 ? (((rs.trig_byte[1] & 0x5fu) ^ 0x10u) * 0x01010101u) : 0u;
  asm volatile("" : "+r"(splat0), "+r"(splat1));
  // this lane's first-half chunk in the warp's current tile (64 chunks = 1 KB).  Tiles are dealt round-robin to all warps of
  // the grid, CTA-interleaved (warp w of CTA b is the grid's warp w x grid + b): the tiles left over after the last full
  // round then go to one or two warps of every SM, not to every warp of the first few CTAs, whose SMs would stream a whole
  // extra tile while the others have finished.
  uint32_t c = first_chunk + (warp * gridDim.x + blockIdx.x) * kTileChunks + lane;
  uint32_t cstep = gridDim.x * wpb * kTileChunks;
  uint32_t shl_bits = hk.one << half_bits(NPROBE);
  asm volatile("" : "+r"(end_chunk), "+r"(cstep), "+r"(shl_bits));
  const bool last_lane = lane == 31;

  // a tile in registers: the lane's two chunks (c, c + 32) and, at stride 2, lane 31's first word of chunk c + 33
  struct Tile { uint4 a, b; uint32_t t; };
  auto load_tile = [&](Tile& v, uint32_t cc) {
    v.a = make_uint4(0, 0, 0, 0); v.b = make_uint4(0, 0, 0, 0); v.t = 0;
    if (cc < end_chunk) v.a = ldg_stream(bytes + (size_t)cc * 16);
    if (cc + 32u < end_chunk) v.b = ldg_stream(bytes + (size_t)(cc + 32u) * 16);
    if (NPROBE == 2 && last_lane && cc + 33u < end_chunk) v.t = __ldg(reinterpret_cast<const uint32_t*>(bytes + (size_t)(cc + 33u) * 16));
  };
  // Tiles go through two register buffers, one tile ahead: tile k consumes one buffer and, as its first action after
  // touching that data, issues both loads of tile k + 1 into the other (dead since tile k - 1 folded it).  Both halves
  // are issued together and needed together, so a tile keeps 1 KB per warp in flight behind ONE wait.
  // ptxas tracks every load of this loop on ONE scoreboard, and a wait on a scoreboard waits for everything issued on it:
  // were the next loads issued BEFORE the first use of the current data (where the scheduler hoists them if it may), each
  // tile would wait for the loads it has just issued -- the full HBM latency, exposed once per tile.  The address of the
  // next tile therefore depends on the current data (+ word * 0 with a run-time zero), which pins the order.
  // The probe results of a round's tiles (2 x 16 bits at stride 2, 4 x 8 at stride 4) are collected in one register per
  // lane; after the round every lane with a non-zero flag word pushes (its chunk, the word) to ring 1 -- one ballot per
  // round, no loop.  Halves past the end load zeros; whatever those flag is dropped by the position checks of the slow path.
  constexpr uint32_t kTilesPerRound = 32u / (2u * half_bits(NPROBE));
  static_assert(kTilesPerRound == 2 || kTilesPerRound == 4, "a round alternates the two buffers");
  uint32_t zero = hk.one - 1u;
  asm volatile("" : "+r"(zero));
  Tile tA, tB;
  load_tile(tA, c); tB.a = make_uint4(0, 0, 0, 0); tB.b = tB.a; tB.t = 0;
  uint32_t acc = 0;
  // the probes and trigger test of one 16-byte chunk (chunk number cc); w4 = the first word of chunk cc + 1 (stride 2)
  auto scan_half = [&](const uint4& cur, uint32_t w4, uint32_t cc) {
    const uint32_t z0 = fold_z(cur.x, hk), z1 = fold_z(cur.y, hk), z2 = fold_z(cur.z, hk), z3 = fold_z(cur.w, hk);
    const uint32_t f0 = fold_key(z0, hk), f1 = fold_key(z1, hk), f2 = fold_key(z2, hk), f3 = fold_key(z3, hk);
    uint32_t flags = 0;
    if (NPROBE == 2) {
      const uint32_t f4 = fold_key(fold_z(w4, hk), hk);
      gram_probe<BLOOM2>(bm, hk, f0, flags); gram_probe<BLOOM2>(bm, hk, __funnelshift_r(f0, f1, 16), flags);
      gram_probe<BLOOM2>(bm, hk, f1, flags); gram_probe<BLOOM2>(bm, hk, __funnelshift_r(f1, f2, 16), flags);
      gram_probe<BLOOM2>(bm, hk, f2, flags); gram_probe<BLOOM2>(bm, hk, __funnelshift_r(f2, f3, 16), flags);
      gram_probe<BLOOM2>(bm, hk, f3, flags); gram_probe<BLOOM2>(bm, hk, __funnelshift_r(f3, f4, 16), flags);
    } else {
      gram_probe<BLOOM2>(bm, hk, f0, flags); gram_probe<BLOOM2>(bm, hk, f1, flags);
      gram_probe<BLOOM2>(bm, hk, f2, flags); gram_probe<BLOOM2>(bm, hk, f3, flags);
    }
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(acc) : "r"(acc), "r"(shl_bits), "r"(flags));      // acc = acc << half_bits | flags, on the FMA pipe
    if (NTRIG > 0) {
      // triggers: d_j has bit 7 of a byte clear where it equals a trigger byte (folded domain)
      uint32_t d0 = differs(z0, splat0, hk.one), d1 = differs(z1, splat0, hk.one), d2 = differs(z2, splat0, hk.one), d3 = differs(z3, splat0, hk.one);
      if (NTRIG > 1) { d0 &= differs(z0, splat1, hk.one); d1 &= differs(z1, splat1, hk.one); d2 &= differs(z2, splat1, hk.one); d3 &= differs(z3, splat1, hk.one); }
      const bool trig = (d0 & d1 & d2 & d3 & 0x80808080u) != 0x80808080u;
      if (__any_sync(FULL, trig)) {
        if (trig) trigger_chunk(rs, w, ctx, ~d0 & 0x80808080u, ~d1 & 0x80808080u, ~d2 & 0x80808080u, ~d3 & 0x80808080u, cc);
        __syncwarp();
      }
    }
  };
  auto scan_tile = [&](const Tile& buf, Tile& nbuf, uint32_t cc) {
    const Tile cur = buf;
    uint32_t ncc = cc + cstep;
    asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(ncc) : "r"(cur.a.x), "r"(zero));     // (waits for the current tile's data)
    load_tile(nbuf, ncc);
    uint32_t wa = 0, wb = 0;
    if (NPROBE == 2) {
      // the odd grams' fifth word: first half, chunk cc + 1 = the next lane's first-half word, for lane 31 lane 0's
      // second-half word (chunk tile base + 32); second half, the next lane's second-half word, for lane 31 chunk cc + 33
      wa = __shfl_sync(FULL, lane == 0 ? cur.b.x : cur.a.x, (lane + 1u) & 31u);
      wb = __shfl_down_sync(FULL, cur.b.x, 1); if (last_lane) wb = cur.t;
    }
    scan_half(cur.a, wa, cc);
    scan_half(cur.b, wb, cc + 32u);
  };
  // Nothing is done about a flagged gram here: looking at one means a chain of dependent loads (the gram again, the
  // recheck map, the level-1b bucket, the factor, the text around it), and with 32 warps per SM there is nobody to hide
  // that latency behind: a slow path inside this kernel would stall the hot loop, whatever its instruction count.  The
  // flag words go to a queue in HBM, and confirm_kernel, with one thread per flag word and the whole GPU's worth of warps,
  // does the looking.  A warp appends kAppend of them at a time behind ONE atomic, whose result every lane waits for while
  // it issues no new tile, so there are few appends -- one or two per warp on C2 traffic (appends of 32 took the 5000-rule
  // scan 0.193 ms instead of 0.121).  Reserving the next block one append ahead, so that nobody waits, measured slower.
  uint32_t h1 = 0, t1 = 0;       // the ring holds [h1, t1)
  auto append = [&](uint32_t k) {                           // k entries from the ring -> the queue
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(&w.counters[kCtrFlagWords], k);
    base = __shfl_sync(FULL, base, 0);
#pragma unroll 1
    for (uint32_t j = lane; j < k; j += 32u) {
      uint32_t cw, aw;
      asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(cw), "=r"(aw) : "r"(ring1 + (((h1 + j) & (kRing - 1)) << 3)));
      if (base + j < w.l1_cap) w.fq[base + j] = make_uint2(cw, aw); else atomicOr(&w.counters[kCtrErrors], ERR_L1_OVERFLOW);
    }
    h1 += k;
  };
#pragma unroll 1
  while (c - lane < end_chunk) {                           // warp-uniform: this warp still has a tile
    scan_tile(tA, tB, c);
    scan_tile(tB, tA, c + cstep);
    if (kTilesPerRound == 4) {
      scan_tile(tA, tB, c + 2u * cstep);
      scan_tile(tB, tA, c + 3u * cstep);
    }
    c += kTilesPerRound * cstep;
    // acc: flagged_gram_pos<NPROBE>((c - cstep) * 16, bit, cstep * 16) is the gram behind each set bit
    const uint32_t m = __ballot_sync(FULL, acc != 0);
    if (m) {
      if (acc) asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(ring1 + (((t1 + __popc(m & lt)) & (kRing - 1)) << 3)), "r"(c), "r"(acc) : "memory");
      t1 += __popc(m); acc = 0;
      if (t1 - h1 >= kAppend) { __syncwarp(); append(kAppend); }
    }
  }
  __syncwarp();
  if (t1 != h1) append(t1 - h1);
}

// ------------------------------------------------------------------------------------------
// level 2: which message does every confirmed factor occurrence belong to?  Slots, candidates for the VM, direct hits.
// ------------------------------------------------------------------------------------------
constexpr uint32_t kIslandSteps = 96;      // islands the bit-parallel matcher walks itself (longer ones, and those it cannot reach the occurrence in, are the VM's)
struct SlotSink {
  const DevRuleset& rs; const ScanWork& w; uint32_t msg; uint32_t slot;
  const uint8_t* text = nullptr; uint32_t text_len = 0;       // the message (policy mode: lets candidate() decide eligible rules on the spot)
  __device__ SlotSink(const DevRuleset& r, const ScanWork& wk, uint32_t m, bool ws) : rs(r), w(wk), msg(m), slot(0xffffffffu), want_spans(ws) {}
  __device__ bool ensure_slot() {
    if (slot != 0xffffffffu) return slot < w.slot_cap;
    uint32_t s = *reinterpret_cast<volatile uint32_t*>(&w.slot_of_msg[msg]);
    if (s == 0xffffffffu) {
      uint32_t mine = atomicAdd(&w.counters[kCtrSlots], 1u);
      if (mine >= w.slot_cap) { atomicOr(&w.counters[kCtrErrors], ERR_SLOT_OVERFLOW); slot = mine; return false; }
      w.slot_msg[mine] = msg;                            // (the slot's candidate / hit rows are zero already: reset_kernel; no fence on this path)
      uint32_t old = atomicCAS(&w.slot_of_msg[msg], 0xffffffffu, mine);
      if (old == 0xffffffffu) s = mine; else { s = old; w.slot_msg[mine] = 0xffffffffu; }   // lost the race: slot stays unused
    }
    slot = s;
    return true;
  }
  // spans mode: one VM run per (message, rule), over the whole message (cand bitmap dedupes).
  // policy mode: one VM run per confirmed factor occurrence, restricted to its island.
  bool want_spans;
  __device__ void candidate(uint32_t r, uint32_t t0, uint32_t pre, uint32_t f) {
    // policy mode, rule with a bit-parallel program, ASCII island: RegExp.test around this occurrence is decided right here
    // (bitprog.h) -- no slot for a miss, no VM run for a hit
    if (!want_spans && text) {
      const uint32_t bo = rs.bit_off[r];
      if (bo != kBitProgNone) {
        if (slot == 0xffffffffu) { const uint32_t s0 = *reinterpret_cast<volatile uint32_t*>(&w.slot_of_msg[msg]); if (s0 != 0xffffffffu && s0 < w.slot_cap && ((w.hit[(size_t)s0 * rs.rw + (r >> 5)] >> (r & 31)) & 1u)) return; }   // already a hit
        const int res = island_test(rs, f, r, text, text_len, t0, pre, kIslandSteps);
        if (res == 0) return;
        if (res == 1) { direct(r); return; }
      }
    }
    if (!ensure_slot()) return;
    uint32_t bit = 1u << (r & 31);
    uint32_t old = atomicOr(&w.cand[(size_t)slot * rs.rw + (r >> 5)], bit);
    if (want_spans && (old & bit)) return;
    uint32_t e = atomicAdd(&w.counters[kCtrEvents], 1u);
    if (e < w.event_cap) {
      // a long stretch of pattern before the factor (or an unbounded one) means many start positions for the VM: such
      // runs are an order of magnitude longer than the rest and are handed out first, so that none of them starts last
      const bool heavy = !want_spans && (pre & 0xffffu) >= 24u;
      w.events[e] = make_uint2(slot, r | (heavy ? 0x80000000u : 0u)); w.event_pos[e] = t0; w.event_pre[e] = pre;
      if (heavy) w.heavy_idx[atomicAdd(&w.counters[kCtrHeavy], 1u)] = e;
    } else atomicOr(&w.counters[kCtrErrors], ERR_EVENT_OVERFLOW);
  }
  // rules without factors: one whole-message run (event_pos = 0xffffffff)
  __device__ void candidate_always(uint32_t r) {
    if (!ensure_slot()) return;
    uint32_t bit = 1u << (r & 31);
    uint32_t old = atomicOr(&w.cand[(size_t)slot * rs.rw + (r >> 5)], bit);
    if (old & bit) return;
    uint32_t e = atomicAdd(&w.counters[kCtrEvents], 1u);
    if (e < w.event_cap) { w.events[e] = make_uint2(slot, r); w.event_pos[e] = 0xffffffffu; } else atomicOr(&w.counters[kCtrErrors], ERR_EVENT_OVERFLOW);
  }
  // a confirmed exact factor already proves RegExp.test(message) for this rule
  __device__ void direct(uint32_t r) {
    if (!ensure_slot()) return;
    uint32_t bit = 1u << (r & 31);
    atomicOr(&w.cand[(size_t)slot * rs.rw + (r >> 5)], bit);
    atomicOr(&w.hit[(size_t)slot * rs.rw + (r >> 5)], bit);
  }
};

// ------------------------------------------------------------------------------------------
// Everything between "the bitmap flagged a gram" and "this (message, rule) goes to the VM" is a chain of dependent loads
// per item and keeps only a fraction of its input at every step.  Inside scan_kernel that chain would stall the hot loop
// (32 warps per SM cannot hide it); as one kernel with barriers between the steps, every step would wait for its slowest
// thread.  So it runs in launches of its own:
//   confirm_kernel  flag word -> gram positions -> gram reloaded, folded, recheck map, table probes -> exact factor  -> factor occurrences
//   resolve_kernel  message of the occurrence (no straddling), slot, island matcher / candidate for the VM / direct hit; also the
//                   occurrences of trigger bytes and of the head check, and the rules every message is a candidate for
// ------------------------------------------------------------------------------------------
// What bounds this work is not re-reading the flagged places of the batch (a random gather, profiles/micro/gather_micro.cu)
// but the number of uncoalesced loads behind each item: a gram, its recheck word and slots, then the entry, factor words,
// text words and byte-set words.  So:
//   * the tables (recheck map, slots, entries, factor words, byte sets: 127 KB at 500 rules) are staged into SHARED memory,
//     where a random word costs a bank conflict instead of an L1 tag lookup per lane; rule sets whose tables do not fit are read
//     in place (same code, generic pointers);
//   * slots are only probed for grams that passed the recheck map, and a (gram, entry) pair first compares the (up to) four
//     factor elements that follow the gram -- two text words at most -- before anything else is fetched: nine pairs in ten end there;
//   * no lane ever loops over its own items while the others wait (the first fused version did: 32 M warp instructions, two
//     thirds of them in per-lane entry and byte loops with one or two lanes active).  Flag bits become gram positions, and the
//     entries a gram hits become (position, entry) pairs, in WAVES of at most one item per lane that are compacted with a
//     ballot into a 64-entry ring per warp in shared memory; whenever a ring holds 32 items, all 32 lanes run the next stage
//     as a straight line (gram -> recheck -> probes | quick test -> whole factor).  Leftovers wait for the next wave.
//   * confirmed occurrences are as rare as one or two per wave of 32 pairs, and an atomicAdd per occurrence on the one
//     counter word queues every lane of the grid at one L2 slice: they collect in a 32-entry buffer per warp, which goes to
//     the queue behind ONE atomic whenever the next wave would not fit, and at the end.
constexpr uint32_t kCfRing = 64;                  // entries per warp and ring (a power of two): 31 leftovers + one wave of 32
constexpr uint32_t kCfOcc = 32;                   // confirmed (position, factor) pairs a warp holds before it appends them
constexpr int kCfThreads = 1024;
constexpr uint32_t kCfWarpBytes = kCfRing * (4 + 8) + kCfOcc * 8;    // gram positions (4 B), (position, entry) pairs (8 B), occurrences (8 B)
constexpr uint32_t kCfRingBytes = (kCfThreads / 32) * kCfWarpBytes;
static_assert(kCfRingBytes + kConfirmTableBudget + 1024u <= 227u * 1024u, "rings and resident tables fit the H100's opt-in shared memory per block");

struct ConfirmCtx {
  const DevRuleset& rs; const ScanWork& w; const uint8_t* bytes;
  const uint8_t* rk; const uint4* slots; const uint32_t* group_entries; const uint32_t* factors; const uint32_t* bytesets;     // shared-memory copies when they fit
  uint2* pring; uint32_t phead, ptail;          // this warp's ring of (gram position, entry) pairs
  uint2* occ; uint32_t held;                    // this warp's confirmed occurrences not yet in the queue: occ[0, held)
  uint32_t begin, end, n_shapes, passed, lane;
};
// the warp's held occurrences -> the queue (warp-uniform; the counter keeps counting past l1_cap, as every queue's does)
__device__ __forceinline__ void append_occurrences(ConfirmCtx& c) {
  uint32_t base = 0;
  if (c.lane == 0) base = atomicAdd(&c.w.counters[kCtrConfirmed], c.held);
  base = __shfl_sync(0xffffffffu, base, 0);
  if (c.lane < c.held) {
    const uint2 o = c.occ[c.lane];
    if (base + c.lane < c.w.l1_cap) { c.w.l1_pos[base + c.lane] = o.x; c.w.l1_fac[base + c.lane] = o.y; } else atomicOr(&c.w.counters[kCtrErrors], ERR_L1_OVERFLOW);
  }
  c.held = 0;
  __syncwarp();
}
__device__ __forceinline__ uint32_t byteset_bit(const uint32_t* __restrict__ bytesets, uint32_t sid, uint32_t b) { return (bytesets[(size_t)sid * 8 + (b >> 5)] >> (b & 31)) & 1u; }

// one (gram, entry) pair per lane: does the entry's factor start at the position the gram implies?  First the (up to) four
// elements that follow the gram (the factor's first four when the gram is its tail): two text words at most, and nine pairs
// in ten end there; the lanes that are left compare the whole factor (five text words at most, every element test in flight).
__device__ __forceinline__ void confirm_pairs(ConfirmCtx& c, uint2 pr, bool active) {
  uint32_t f = 0, flen = 0, qb = 0, qe = 0; int64_t t0 = 0; const uint32_t* fw = c.factors;
  bool ok = false;
  if (active) {
    const uint32_t y = c.group_entries[pr.y];
    f = y & 0xfffffu;
    const int goff = (int)((y >> 20) & 31u) - 3;
    t0 = (int64_t)pr.x - goff;
    fw = c.factors + (size_t)f * 12;          // rule, len | exact << 24, 16 x u16 set ids, pre, pre_alpha
    flen = fw[1] & 0xffu;
    ok = t0 >= (int64_t)c.begin && t0 + (int64_t)flen <= (int64_t)c.end;
    qb = (uint32_t)(goff + (int)kGramLen < 0 ? 0 : goff + (int)kGramLen); if (qb >= flen) qb = 0;
    qe = min(qb + 4u, flen);
  }
  if (ok && qe > qb) {
    const size_t qp = (size_t)t0 + qb;
    const uint32_t* tq = reinterpret_cast<const uint32_t*>(c.bytes + (qp & ~(size_t)3));
    const uint32_t q0 = __ldg(tq), q1 = ((uint32_t)qp & 3u) + (qe - qb) > 4u ? __ldg(tq + 1) : 0u;
    const uint32_t qt = __funnelshift_r(q0, q1, 8u * ((uint32_t)qp & 3u));
    uint32_t bits = 1u;
#pragma unroll
    for (uint32_t i = 0; i < 4; i++) {
      const uint32_t k = qb + i;
      if (k < qe) bits &= byteset_bit(c.bytesets, (fw[2 + (k >> 1)] >> (16 * (k & 1))) & 0xffffu, (qt >> (8 * i)) & 0xffu);
    }
    ok = bits != 0;
  }
  if (!__any_sync(0xffffffffu, ok)) return;
  if (ok && flen > qe - qb) {
    const uint32_t* tp = reinterpret_cast<const uint32_t*>(c.bytes + ((size_t)t0 & ~(size_t)3));
    const uint32_t sh = 8u * ((uint32_t)t0 & 3u);
    const uint32_t need = ((uint32_t)t0 & 3u) + flen;           // bytes from the first aligned word on (nothing past the factor's end is read)
    const uint32_t a0 = __ldg(tp), a1 = need > 4u ? __ldg(tp + 1) : 0u, a2 = need > 8u ? __ldg(tp + 2) : 0u, a3 = need > 12u ? __ldg(tp + 3) : 0u, a4 = need > 16u ? __ldg(tp + 4) : 0u;
    const uint32_t tx[4] = {__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh), __funnelshift_r(a2, a3, sh), __funnelshift_r(a3, a4, sh)};
    uint32_t bits = 1u;
#pragma unroll
    for (uint32_t k = 0; k < 16; k++) {
      if (k < flen && !(k >= qb && k < qe)) bits &= byteset_bit(c.bytesets, (fw[2 + (k >> 1)] >> (16 * (k & 1))) & 0xffffu, (tx[k >> 2] >> (8 * (k & 3))) & 0xffu);
    }
    ok = bits != 0;
  }
  const uint32_t m = __ballot_sync(0xffffffffu, ok);
  if (!m) return;
  if (c.held + __popc(m) > kCfOcc) append_occurrences(c);
  if (ok) c.occ[c.held + __popc(m & ((1u << c.lane) - 1u))] = make_uint2((uint32_t)t0, f);
  c.held += __popc(m);
  __syncwarp();
}

// one gram position per lane (active lanes only do loads; everybody takes part in the votes): gram -> recheck map -> one probe
// per shape; the entries of the groups it hits go to the pair ring in waves of at most one per lane, 32 pairs at a time leave it
__device__ __forceinline__ void confirm_gram(ConfirmCtx& c, uint32_t pos, bool active) {
  const DevRuleset& rs = c.rs;
  const uint32_t FULL = 0xffffffffu, lt = (1u << c.lane) - 1u;
  active = active && pos < c.end;
  uint32_t key = 0;
  if (active) {
    const uint32_t* p4 = reinterpret_cast<const uint32_t*>(c.bytes + (pos & ~3u));
    uint32_t gw = __ldg(p4);
    if (pos & 3u) gw = __funnelshift_r(gw, __ldg(p4 + 1), 8u * (pos & 3u));
    key = gram_fold_word(gw);
  }
  const uint32_t rh = gram_recheck_hash(key);
  const bool pass = active && ((*reinterpret_cast<const uint32_t*>(c.rk + (rh & rs.rk_mask)) << (rh >> 27)) & 0x80000000u);
  if (!__any_sync(FULL, pass)) return;
  if (pass) c.passed++;
  for (uint32_t s0 = 0; s0 < c.n_shapes; s0 += 4u) {
    uint32_t first[4], cnt[4], tot = 0;
#pragma unroll
    for (uint32_t u = 0; u < 4; u++) {
      const uint32_t s = s0 + u, km = key & rs.shapes[s & 15u];
      first[u] = 0; cnt[u] = 0;
      if (pass && s < c.n_shapes) {
        uint32_t slot = ((km ^ (s * 0x9E3779B9u)) * kGramMult2) >> rs.slot_shift;
        uint4 sl = c.slots[slot];
        while (sl.w && (sl.x != km || sl.y != s)) { slot = (slot + 1u) & rs.slot_mask; sl = c.slots[slot]; }    // (linear probing; rarely a second slot)
        first[u] = sl.z; cnt[u] = sl.w;
      }
      tot += cnt[u];
    }
    for (uint32_t j = 0;; j++) {
      const bool has = j < tot;
      const uint32_t m = __ballot_sync(FULL, has);
      if (!m) break;
      if (has) {
        uint32_t jj = j, ei;
        if (jj < cnt[0]) ei = first[0] + jj; else { jj -= cnt[0]; if (jj < cnt[1]) ei = first[1] + jj; else { jj -= cnt[1]; if (jj < cnt[2]) ei = first[2] + jj; else ei = first[3] + (jj - cnt[2]); } }
        c.pring[(c.ptail + __popc(m & lt)) & (kCfRing - 1)] = make_uint2(pos, ei);
      }
      c.ptail += __popc(m);
      __syncwarp();
      if (c.ptail - c.phead >= 32u) { const uint2 pr = c.pring[(c.phead + c.lane) & (kCfRing - 1)]; c.phead += 32u; __syncwarp(); confirm_pairs(c, pr, true); }
    }
  }
}

// An occurrence that starts less than three bytes into the scanned range has no gram in front of it: compared directly,
// here rather than in scan_kernel, where the block that did it started streaming late and set the kernel's end.  The 3 x
// n_factors checks are spread over the grid and, inside a block, over its warps (the block's j-th check goes to lane
// j / wpb of warp j mod wpb), so that no warp pays more than a few of these chains of dependent loads before its queue work.
// They find an occurrence rarely (only where a factor starts the batch), so each keeps its own atomic (QueueEmit).
__device__ __noinline__ void head_check(const DevRuleset& rs, const ScanWork& w, const uint8_t* __restrict__ bytes, uint32_t begin, uint32_t end) {
  QueueEmit emit{w};
  const uint32_t wpb = blockDim.x >> 5, t = (threadIdx.x & 31u) * wpb + (threadIdx.x >> 5);
  for (uint32_t i = t * gridDim.x + blockIdx.x; i < 3u * rs.n_factors; i += gridDim.x * blockDim.x) {
    const uint32_t f = i / 3u, t0 = begin + i % 3u;
    const uint32_t* fw = rs.factors + (size_t)f * 12;
    if (t0 < end && t0 + (fw[1] & 0xffu) <= end && factor_at(fw, rs.bytesets, bytes + t0)) emit(t0, f);
  }
}

// NPROBE as scan_kernel's: the flag-word decode is a handful of shifts and masks per bit (flagged_gram_pos)
template <int NPROBE>
__global__ void __launch_bounds__(kCfThreads, 1)
confirm_kernel(const __grid_constant__ DevRuleset rs, const __grid_constant__ ScanWork w, const uint8_t* __restrict__ bytes, const uint32_t* __restrict__ off, uint32_t n, uint32_t cstep) {
  extern __shared__ __align__(16) uint8_t cf_smem[];          // [pair rings][gram rings][occurrence buffers][tables, when resident]
  __shared__ uint32_t cta_ctr[3];                             // flagged grams, grams past the recheck map, pairs: one atomic each per CTA
  const uint32_t cstep16 = cstep * 16u;
  const uint32_t nq = (rs.debug_flags & 1u) ? 0u : min(w.counters[kCtrFlagWords], w.l1_cap);
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5, FULL = 0xffffffffu, lt = (1u << lane) - 1u;
  uint2* pring = reinterpret_cast<uint2*>(cf_smem) + warp * kCfRing;
  uint32_t* ring = reinterpret_cast<uint32_t*>(cf_smem + (size_t)wpb * kCfRing * 8) + warp * kCfRing;
  uint2* occ = reinterpret_cast<uint2*>(cf_smem + (size_t)wpb * kCfRing * 12) + warp * kCfOcc;
  if (threadIdx.x < 3) cta_ctr[threadIdx.x] = 0u;
  const uint8_t* T = rs.cf_image;
  if (rs.cf_resident) {
    uint8_t* st = cf_smem + (size_t)wpb * kCfWarpBytes;
    if (blockIdx.x * 32u * wpb < nq) {           // (a block without work does not need them)
      for (uint32_t o = threadIdx.x * 16u; o < rs.cf_bytes; o += blockDim.x * 16u) *reinterpret_cast<uint4*>(st + o) = ldg_stream(rs.cf_image + o);
    }
    T = st;
  }
  __syncthreads();
  head_check(rs, w, bytes, off[0], off[n]);
  const uint32_t gwarp = blockIdx.x * wpb + warp, nwarps = gridDim.x * wpb;
  ConfirmCtx c{rs, w, bytes, T, reinterpret_cast<const uint4*>(T + rs.cf_slots_off), reinterpret_cast<const uint32_t*>(T + rs.cf_ge_off),
               reinterpret_cast<const uint32_t*>(T + rs.cf_fac_off), reinterpret_cast<const uint32_t*>(T + rs.cf_bs_off), pring, 0u, 0u, occ, 0u,
               off[0], off[n], rs.n_shapes, 0u, lane};
  uint32_t head = 0, tail = 0, flagged = 0;
  for (uint32_t base = gwarp * 32u; base < nq; base += nwarps * 32u) {
    uint2 q = make_uint2(0u, 0u);
    if (base + lane < nq) q = w.fq[base + lane];
    // flag bits -> gram positions, one wave per bit rank (the k-th set bit of every lane's word): at most 32 new positions a wave
    uint32_t bits = q.y;
    const uint32_t newest = (q.x - cstep) * 16u;
    for (;;) {
      const uint32_t m = __ballot_sync(FULL, bits != 0);
      if (!m) break;
      if (bits) {
        const uint32_t bit = (uint32_t)__ffs((int)bits) - 1u; bits &= bits - 1u;
        ring[(tail + __popc(m & lt)) & (kCfRing - 1)] = flagged_gram_pos<NPROBE>(newest, bit, cstep16);
      }
      tail += __popc(m); flagged += lane == 0 ? __popc(m) : 0u;
      __syncwarp();
      if (tail - head >= 32u) { const uint32_t pos = ring[(head + lane) & (kCfRing - 1)]; head += 32u; __syncwarp(); confirm_gram(c, pos, true); }
    }
  }
  if (tail != head) { const bool a = lane < tail - head; const uint32_t pos = a ? ring[(head + lane) & (kCfRing - 1)] : 0u; __syncwarp(); confirm_gram(c, pos, a); }
  if (c.ptail != c.phead) { const bool a = lane < c.ptail - c.phead; const uint2 pr = a ? c.pring[(c.phead + lane) & (kCfRing - 1)] : make_uint2(0u, 0u); confirm_pairs(c, pr, a); }
  if (c.held) append_occurrences(c);
  const uint32_t passed = __reduce_add_sync(FULL, c.passed);
  if (lane == 0) { if (flagged) atomicAdd(&cta_ctr[0], flagged); if (passed) atomicAdd(&cta_ctr[1], passed); if (c.ptail) atomicAdd(&cta_ctr[2], c.ptail); }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (cta_ctr[0]) atomicAdd(&w.counters[kCtrFlagged], cta_ctr[0]);
    if (cta_ctr[1]) atomicAdd(&w.counters[kCtrPastRecheck], cta_ctr[1]);
    if (cta_ctr[2]) atomicAdd(&w.counters[kCtrPairs], cta_ctr[2]);
  }
}

// Which (message, rule) pairs may enter a slot: every pair (the calls without views), or only the rules of the message's
// view (ViewTable, kernels.h).  The test sits in front of SlotSink, so an out-of-view occurrence takes no slot, walks no
// island and queues no VM event; everything downstream reads the slot's rows only and so sees the view's rules alone.
struct AllRules { __device__ __forceinline__ bool admits(uint32_t, uint32_t) const { return true; } };
struct InView {
  ViewTable vt; uint32_t rw;
  __device__ __forceinline__ bool admits(uint32_t msg, uint32_t r) const {
    const uint32_t v = vt.ids[msg];
    return v < vt.n_views && ((vt.rows[(size_t)v * rw + (r >> 5)] >> (r & 31)) & 1u);
  }
};

template <class Filter>
__device__ __forceinline__ void resolve_occurrences(const DevRuleset& rs, const ScanWork& w, const uint8_t* __restrict__ bytes, const uint32_t* __restrict__ off,
                                                    uint32_t n, int want_spans, const Filter& filter) {
  const uint32_t n1 = min(w.counters[kCtrConfirmed], w.l1_cap);
  const uint32_t stride = gridDim.x * blockDim.x, tid = blockIdx.x * blockDim.x + threadIdx.x;
  // Occurrences take different paths of very different lengths (direct hit, island matcher of 5 .. 96 steps, slot allocation),
  // and a warp executes the union of its lanes' paths one dependent instruction after the other: with 32 occurrences per warp
  // a few warps run long dependent chains while most warp slots stay empty.  So only every `spread`-th lane takes an
  // occurrence: more warps, each with a short chain (4: what fits one wave of resident warps).
  constexpr uint32_t spread = 4;
  for (uint32_t i = tid / spread; i < n1 && tid % spread == 0; i += stride / spread) {
    const uint32_t pos = w.l1_pos[i], f = w.l1_fac[i];
    const uint32_t msg = message_of(off, n, pos);
    if (pos + (rs.factors[(size_t)f * 12 + 1] & 0xffu) > off[msg + 1]) continue;     // straddles two messages: not an occurrence
    if (!filter.admits(msg, rs.factors[(size_t)f * 12])) continue;                      // (the factor's rule: factor_confirmed's)
    SlotSink sink(rs, w, msg, want_spans != 0);
    sink.text = bytes + off[msg]; sink.text_len = off[msg + 1] - off[msg];
    factor_confirmed(rs, f, pos - off[msg], want_spans != 0, sink);
  }
  if (rs.n_always) for (uint32_t msg = tid; msg < n; msg += stride) {
    SlotSink sink(rs, w, msg, want_spans != 0);
    for (uint32_t k = 0; k < rs.n_always; k++) if (filter.admits(msg, rs.always_rules[k])) sink.candidate_always(rs.always_rules[k]);
  }
}

__global__ void __launch_bounds__(256, 4)
resolve_kernel(DevRuleset rs, ScanWork w, const uint8_t* __restrict__ bytes, const uint32_t* __restrict__ off, uint32_t n, int want_spans) {
  resolve_occurrences(rs, w, bytes, off, n, want_spans, AllRules{});
}
// the same with the views of cg_*_views: the table is an argument of its own (DevRuleset / ScanWork keep their layout).  Two
// CTAs per SM, not four: under resolve_kernel's 64-register cap this instantiation spills; at this bound it takes 92
// registers and spills nothing
__global__ void __launch_bounds__(256, 2)
resolve_views_kernel(DevRuleset rs, ScanWork w, const uint8_t* __restrict__ bytes, const uint32_t* __restrict__ off, uint32_t n, int want_spans,
                     ViewTable views) {
  resolve_occurrences(rs, w, bytes, off, n, want_spans, InView{views, rs.rw});
}

// ------------------------------------------------------------------------------------------
// level 3: exact verification by the Pike VM
// ------------------------------------------------------------------------------------------
constexpr int kVerifyThreads = 64;            // verify_large_kernel
// verify_small_kernel: VM runs diverge completely (different program, different text), so two runs in one warp cost the
// SUM of their instruction streams: one run per warp, whose lanes cooperate inside the run instead.
constexpr int kVerifyBlock = 256, kVerifyCtasPerSm = 4, kVerifySlots = kVerifyBlock / 32;     // one VM run per warp
constexpr int kSmallProg = 192;          // VM capacity that covers every built-in rule (longest: key-value-credential, 183 instructions)

struct GlobalSpanSink {
  const ScanWork& w; uint32_t msg, rule; bool lane0_only;
  __device__ void span(uint32_t sb, uint32_t eb, uint32_t s16, uint32_t e16) {
    if (lane0_only && (threadIdx.x & 31u)) return;         // warp-redundant runs (verify_small_kernel): one lane reports
    uint32_t k = atomicAdd(&w.counters[kCtrRawSpans], 1u);
    if (k < w.span_cap) { uint32_t* o = w.spans + (size_t)k * 6; o[0] = msg; o[1] = rule; o[2] = sb; o[3] = eb; o[4] = s16; o[5] = e16; }
    else atomicOr(&w.counters[kCtrErrors], ERR_SPAN_OVERFLOW);
  }
};

// thread-interleaved shared-memory VM storage: element i of thread t lives at base[i * blockDim + t]
struct SmemStore {
  static constexpr uint32_t cap = kSmallProg;
  static constexpr bool coop = true;       // one run per WARP: every lane executes it redundantly and helps where it can (pike_vm.h)
  uint16_t* mark_; uint16_t* pcs_; uint32_t* sts_; uint16_t* stk_; uint32_t stride, t;
  __device__ __forceinline__ uint16_t& mark(uint32_t i) { return mark_[i * stride + t]; }
  __device__ __forceinline__ uint16_t& pc(int L, uint32_t i) { return pcs_[(L * cap + i) * stride + t]; }
  __device__ __forceinline__ uint32_t& st(int L, uint32_t i) { return sts_[(L * cap + i) * stride + t]; }
  __device__ __forceinline__ uint16_t& stk(uint32_t i) { return stk_[i * stride + t]; }
};
constexpr int kStageMsg = 256;                       // messages up to this many bytes are staged into shared memory
constexpr size_t kVerifyVmBytes = (size_t)kVerifySlots * (kSmallProg * 2 + 2 * kSmallProg * 2 + 2 * kSmallProg * 4 + kVmStack * 2);
constexpr size_t kVerifyProgBytes = 0;      // (staging areas: measured, not worth their copy loops)
constexpr size_t kVerifyMsgBytes = 0;
constexpr size_t kVerifySmem = kVerifyVmBytes + kVerifyProgBytes + kVerifyMsgBytes;

// small programs (<= kSmallProg instructions): VM state in shared memory
template <bool SPANS>
__global__ void __launch_bounds__(kVerifyBlock, kVerifyCtasPerSm)
verify_small_kernel(DevRuleset rs, ScanWork w, const uint8_t* __restrict__ bytes, const uint32_t* __restrict__ off) {
  extern __shared__ __align__(16) uint8_t vsm[];
  const uint32_t n_events = min(w.counters[kCtrEvents], w.event_cap);
  if (n_events == 0) return;                    // (the island matcher decided everything: the common case)
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // One run per warp.  All 32 lanes execute it redundantly -- identical registers, uniform control flow, the VM
  // state in shared memory written with identical values -- so that the lanes can split the work wherever a step
  // is data-parallel (SIMD literal / class stretches, mark clearing; see pike_vm.h).  Only lane 0 reports.
  const uint32_t slot_id = warp;
  SmemStore st;
  st.stride = kVerifySlots; st.t = slot_id;
  st.sts_ = reinterpret_cast<uint32_t*>(vsm);
  st.pcs_ = reinterpret_cast<uint16_t*>(vsm + (size_t)kVerifySlots * 2 * kSmallProg * 4);
  st.mark_ = st.pcs_ + (size_t)kVerifySlots * 2 * kSmallProg;
  st.stk_ = st.mark_ + (size_t)kVerifySlots * kSmallProg;
  VMS<SmemStore> vm(rs, st);
  // events are handed out one at a time (their cost varies by two orders of magnitude): a static split leaves most
  // warps idle while a few finish their second or third long run
  const uint32_t n_heavy = min(w.counters[kCtrHeavy], n_events);
  bool heavy_phase = true;
  for (;;) {
    uint32_t e = 0;
    if (lane == 0) e = atomicAdd(&w.counters[heavy_phase ? kCtrVerifyHeavy : kCtrVerifyLight], 1u);
    e = __shfl_sync(0xffffffffu, e, 0);
    if (heavy_phase) {
      if (e >= n_heavy) { heavy_phase = false; continue; }
      e = w.heavy_idx[e];
    } else if (e >= n_events) break;
    uint2 ev = w.events[e];
    if (!heavy_phase && (ev.y >> 31)) continue;             // done (or being done) by the heavy phase
    uint32_t slot = ev.x, rule = ev.y & 0x7fffffffu;
    const uint32_t plen = rs.rule_prog_off[rule + 1] - rs.rule_prog_off[rule];
    if (plen > (uint32_t)kSmallProg) continue;          // handled by verify_large_kernel
    uint32_t msg = w.slot_msg[slot];
    GlobalSpanSink sink{w, msg, rule, true};
    const uint32_t t0 = w.event_pos[e];
    if (!SPANS && t0 != 0xffffffffu) {                  // another occurrence already proved it?  (one read, broadcast: the warp must agree)
      uint32_t hv = 0;
      if (lane == 0) hv = w.hit[(size_t)slot * rs.rw + (rule >> 5)];
      hv = __shfl_sync(0xffffffffu, hv, 0);
      if ((hv >> (rule & 31)) & 1u) continue;
    }
    const uint8_t* m = bytes + off[msg]; const uint32_t len = off[msg + 1] - off[msg];
    bool any;
    const long long tc0 = (rs.debug_flags & 2u) ? clock64() : 0;
    if (SPANS || t0 == 0xffffffffu) any = run_rule<SPANS>(vm, rs, rule, m, len, sink);
    else any = test_at_factor(vm, rs, rule, m, len, t0, w.event_pre[e]);
    __syncwarp();
    if (any && lane == 0) atomicOr(&w.hit[(size_t)slot * rs.rw + (rule >> 5)], 1u << (rule & 31));
    if ((rs.debug_flags & 2u) && lane == 0) {       // CG_SCAN_DEBUG=2: histogram of VM cycles per event behind counters[kCtrDebug] (<2^11, <2^12, ... >=2^17), the max in it
      const uint32_t cyc = (uint32_t)(clock64() - tc0);
      int bkt = 31 - __clz(cyc | 1u) - 10; bkt = bkt < 0 ? 0 : bkt > 7 ? 7 : bkt;
      atomicAdd(&w.counters[kCtrDebug + 1 + bkt], 1u); atomicMax(&w.counters[kCtrDebug], cyc);
    }
    __syncwarp();                                          // lane 0 reported; everyone together again before the next run touches shared memory
  }
  if (vm.err && lane == 0) atomicOr(&w.counters[kCtrErrors], vm.err);
}

// programs longer than kSmallProg: per-thread local arrays
template <bool SPANS>
__global__ void __launch_bounds__(kVerifyThreads)
verify_large_kernel(DevRuleset rs, ScanWork w, const uint8_t* __restrict__ bytes, const uint32_t* __restrict__ off) {
  const uint32_t n_events = min(w.counters[kCtrEvents], w.event_cap);
  VMT<kMaxProgLen> vm(rs);
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n_events; e += gridDim.x * blockDim.x) {
    uint2 ev = w.events[e];
    uint32_t slot = ev.x, rule = ev.y & 0x7fffffffu;
    uint32_t plen = rs.rule_prog_off[rule + 1] - rs.rule_prog_off[rule];
    if (plen <= (uint32_t)kSmallProg) continue;
    uint32_t msg = w.slot_msg[slot];
    GlobalSpanSink sink{w, msg, rule, false};
    const uint32_t t0 = w.event_pos[e];
    bool any;
    if (SPANS || t0 == 0xffffffffu) any = run_rule<SPANS>(vm, rs, rule, bytes + off[msg], off[msg + 1] - off[msg], sink);
    else {
      if ((w.hit[(size_t)slot * rs.rw + (rule >> 5)] >> (rule & 31)) & 1u) continue;     // another occurrence already proved it
      any = test_at_factor(vm, rs, rule, bytes + off[msg], off[msg + 1] - off[msg], t0, w.event_pre[e]);
    }
    if (any) atomicOr(&w.hit[(size_t)slot * rs.rw + (rule >> 5)], 1u << (rule & 31));
  }
  if (vm.err) atomicOr(&w.counters[kCtrErrors], vm.err);
}

// Start of a step.  The candidate / hit rows of a slot must be zero when a message takes it; clearing them there cost every
// first occurrence of a message a loop of stores and a __threadfence in the middle of resolve_kernel's dependency chain.  The
// rows the PREVIOUS step used are cleared here instead (their number survives in w.persist), together with what two memsets did.
__global__ void reset_kernel(DevRuleset rs, ScanWork w, uint32_t n) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
  const uint32_t used = min(w.persist[0], w.slot_cap) * rs.rw;
  for (uint32_t i = tid; i < used; i += stride) { w.cand[i] = 0; w.hit[i] = 0; }
  for (uint32_t i = tid; i < n; i += stride) w.slot_of_msg[i] = 0xffffffffu;
  if (tid < kCounterWords) w.counters[tid] = 0;
}

__global__ void finalize_kernel(DevRuleset rs, ScanWork w, uint64_t* __restrict__ words, uint32_t n) {
  if (blockIdx.x == 0 && threadIdx.x == 0) w.persist[0] = min(w.counters[kCtrSlots], w.slot_cap);
  // A step whose queues overflowed or whose VM ran out of space has incomplete results: every word of the batch says so
  // (in-band, so that a caller of the asynchronous device path cannot mistake them for "no hit").
  if (w.counters[kCtrErrors]) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) words[i] = kWordIncomplete;
    return;
  }
  const uint32_t n_slots = min(w.counters[kCtrSlots], w.slot_cap);
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_slots; s += gridDim.x * blockDim.x) {
    const uint32_t msg = w.slot_msg[s];
    if (msg == 0xffffffffu) continue;                    // slot lost an allocation race: unused
    uint32_t count = 0, first = 0xffffffffu;
    for (uint32_t k = 0; k < rs.rw; k++) {
      uint32_t v = w.hit[(size_t)s * rs.rw + k];
      if (v) { if (first == 0xffffffffu) first = k * 32 + (__ffs(v) - 1); count += __popc(v); }
    }
    if (count) words[msg] = (1ull << 63) | ((uint64_t)count << 32) | first;
  }
}

// Verdict of a message from its hit bitmap (aggregateMatches, policy-evaluator.ts:110-146, for messageContains rules):
// policies in priority order, per policy the FIRST matching rule counts, deny beats audit beats allow, and the first
// policy that produced the winning action is the one whose reason is reported.  Rules are stored policy by policy, so an
// ascending walk over the hit bits meets every policy's deciding rule first.
// An incomplete step (a queue overflowed, the VM failed) has no verdicts: every one of the batch is 0xffffffff, which no
// verdict can be (action 3 does not exist).
__global__ void verdict_kernel(DevRuleset rs, ScanWork w, uint32_t* __restrict__ verdicts, uint32_t n) {
  if (w.counters[kCtrErrors]) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) verdicts[i] = 0xffffffffu;
    return;
  }
  const uint32_t n_slots = min(w.counters[kCtrSlots], w.slot_cap);
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_slots; s += gridDim.x * blockDim.x) {
    const uint32_t msg = w.slot_msg[s];
    if (msg == 0xffffffffu) continue;
    uint32_t prev = 0xffffffffu, best = 0, decide = 0xfffffu, matched = 0;
    for (uint32_t k = 0; k < rs.rw; k++) {
      uint32_t v = w.hit[(size_t)s * rs.rw + k];
      while (v) {
        const uint32_t r = k * 32 + (__ffs(v) - 1); v &= v - 1;
        const uint32_t p = rs.rule_policy[r];
        if (p == prev) continue;
        prev = p; matched++;
        const uint32_t a = rs.rule_action[r];
        if (a == 2u && best != 2u) { best = 2u; decide = r; } else if (a == 1u && best == 0u) { best = 1u; decide = r; }
      }
    }
    if (matched) verdicts[msg] = best | (min(matched, 1023u) << 2) | (decide << 12);
  }
}

// The (msg, rule) hit list of a finished policy-mode step, sorted by message, then rule (cg_scan_hits_batch_device,
// cg_scan_batch): hit_count_kernel -> exclusive scan of the counts -> hit_emit_kernel.
// cnt[m] = the rules message m hit, from its result word (finalize_kernel counted them in the same hit row); cnt[n] = 0, so
// that the scan's last element is the total.
__global__ void __launch_bounds__(256) hit_count_kernel(const uint64_t* __restrict__ words, uint32_t n, uint64_t* __restrict__ cnt) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) {
    const uint64_t v = i < n ? words[i] : 0ull;
    cnt[i] = (v >> 63) ? (v >> 32) & 0x7fffffffull : 0ull;
  }
}

// One warp per 32 consecutive messages: a ballot finds the ones with hits (w.out_len = counts, w.out_off = their exclusive
// scan), then all 32 lanes write each such message's hit row together -- lane k takes row words k, k + 32, ..., and a popc
// prefix over the lanes places its rules -- so a row of 157 words (5000 rules) costs five wave steps, not one lane's walk.
// Pairs go to out (two u32 each) below position cap only.  *count = the total (0xffffffff: incomplete step, or 2^32 - 1 hits
// or more), also counters[kCtrHits] for cg_stats.hits; counters[kCtrResolveStatus] = kResolveCapacity / kResolveTooLarge past cap / 2^32 - 1.
__global__ void __launch_bounds__(256) hit_emit_kernel(DevRuleset rs, ScanWork w, uint32_t n, uint32_t* __restrict__ out, uint32_t cap,
                                                       uint32_t* __restrict__ count) {
  const bool incomplete = w.counters[kCtrErrors] != 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const uint64_t total = w.out_off[n];
    if (incomplete) *count = 0xffffffffu;
    else {
      const uint32_t t = total >= 0xffffffffull ? 0xffffffffu : (uint32_t)total;
      *count = t; w.counters[kCtrHits] = t;
      w.counters[kCtrResolveStatus] = total >= 0xffffffffull ? kResolveTooLarge : total > cap ? kResolveCapacity : kResolveOk;
    }
  }
  if (incomplete) return;
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x / 32);
  for (uint32_t g = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); (uint64_t)g * 32 < n; g += warps) {
    const uint32_t m = g * 32 + lane;
    const uint32_t c = m < n ? (uint32_t)w.out_len[m] : 0u;
    const uint64_t at = m < n ? w.out_off[m] : 0ull;
    for (uint32_t todo = __ballot_sync(0xffffffffu, c != 0 && at < cap); todo; todo &= todo - 1) {
      const uint32_t j = __ffs(todo) - 1, msg = g * 32 + j;
      uint64_t pos = __shfl_sync(0xffffffffu, at, j);
      const uint32_t* row = w.hit + (size_t)w.slot_of_msg[msg] * rs.rw;
      for (uint32_t k0 = 0; k0 < rs.rw && pos < cap; k0 += 32) {          // (pos is the same on every lane)
        uint32_t v = k0 + lane < rs.rw ? row[k0 + lane] : 0u;
        const uint32_t pc = __popc(v);
        uint32_t incl = pc;
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (uint32_t)d) incl += t; }
        for (uint64_t p = pos + (incl - pc); v && p < cap; v &= v - 1, p++) { out[2 * p] = msg; out[2 * p + 1] = (k0 + lane) * 32 + (__ffs(v) - 1); }
        pos += __shfl_sync(0xffffffffu, incl, 31);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
#define CG_FOR_SCAN_VARIANTS(X) X(1, 0, 0) X(1, 1, 0) X(1, 2, 0) X(2, 0, 0) X(2, 1, 0) X(2, 2, 0) X(1, 0, 1) X(1, 1, 1) X(1, 2, 1) X(2, 0, 1) X(2, 1, 1) X(2, 2, 1)
void prepare_scan_kernels() {
  int dev = 0, optin = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  const int kMaxSmem = (optin > 0 ? optin : 227 * 1024) - 1024;     // leave room for the kernels' static shared memory
#define CG_PREP(P, T, B) cudaFuncSetAttribute(scan_kernel<P, T, B>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
  CG_FOR_SCAN_VARIANTS(CG_PREP)
#undef CG_PREP
  cudaFuncSetAttribute(confirm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kCfRingBytes + kConfirmTableBudget));
  cudaFuncSetAttribute(confirm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kCfRingBytes + kConfirmTableBudget));
  cudaFuncSetAttribute(verify_small_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kVerifySmem);
  cudaFuncSetAttribute(verify_small_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kVerifySmem);
}

// grid of the scan for a batch of n messages (confirm_kernel decodes the queue's chunk numbers with the same value)
static uint32_t scan_grid(uint32_t n, int sm_count) {
  uint32_t grid = (uint32_t)sm_count;
  if (n < 4096) grid = std::max<uint32_t>(1u, std::min<uint32_t>(grid, n / 32u + 1u));         // tiny batches: fewer image loads
  return grid;
}
int launch_scan(const DevRuleset& rs, const ScanWork& w, const uint8_t* d_bytes, const uint32_t* d_off, uint32_t n,
                uint64_t* d_words, int sm_count, cudaStream_t stream) {
  if (n == 0) return 0;
  const size_t smem = (size_t)rs.image_bytes + kScanRingBytes;
  // the scanned range is only known on the device (off[0] .. off[n]); a warp tile is 1 KB, messages are rarely shorter than 16
  const uint32_t grid = scan_grid(n, sm_count);
  const int np = rs.stride == 2 ? 2 : 1, nt = (int)rs.n_trig, bl = rs.bloom2 ? 1 : 0;
#define CG_LAUNCH(P, T, B) if (np == P && nt == T && bl == B) scan_kernel<P, T, B><<<grid, kScanThreads, smem, stream>>>(rs, w, d_bytes, d_off, n, d_words);
  CG_FOR_SCAN_VARIANTS(CG_LAUNCH)
#undef CG_LAUNCH
  return 1;
}

int launch_confirm(const DevRuleset& rs, const ScanWork& w, const uint8_t* d_bytes, const uint32_t* d_off, uint32_t n, int sm_count, cudaStream_t stream) {
  if (n == 0) return 0;
  const uint32_t cstep = scan_grid(n, sm_count) * (uint32_t)(kScanThreads / 32) * kTileChunks;       // (the queue's chunk numbers are decoded with the scan's grid)
  const size_t smem = (size_t)kCfRingBytes + (rs.cf_resident ? rs.cf_bytes : 0u);
  if (rs.stride == 2) confirm_kernel<2><<<scan_grid(n, sm_count), kCfThreads, smem, stream>>>(rs, w, d_bytes, d_off, n, cstep);
  else confirm_kernel<1><<<scan_grid(n, sm_count), kCfThreads, smem, stream>>>(rs, w, d_bytes, d_off, n, cstep);
  return 1;
}
int launch_resolve(const DevRuleset& rs, const ScanWork& w, const uint8_t* d_bytes, const uint32_t* d_off, uint32_t n, bool want_spans, int sm_count, cudaStream_t stream,
                   const ViewTable* views) {
  if (n == 0) return 0;
  if (views) resolve_views_kernel<<<sm_count * 8, 256, 0, stream>>>(rs, w, d_bytes, d_off, n, want_spans ? 1 : 0, *views);
  else resolve_kernel<<<sm_count * 8, 256, 0, stream>>>(rs, w, d_bytes, d_off, n, want_spans ? 1 : 0);
  return 1;
}

int launch_verify(const DevRuleset& rs, const ScanWork& w, const uint8_t* d_bytes, const uint32_t* d_off,
                  bool want_spans, int sm_count, cudaStream_t stream, int ctas_per_sm) {
  int k = 1;
  const int ctas = ctas_per_sm >= 1 && ctas_per_sm <= kVerifyCtasPerSm ? ctas_per_sm : kVerifyCtasPerSm;
  if (want_spans) {
    verify_small_kernel<true><<<sm_count * ctas, kVerifyBlock, kVerifySmem, stream>>>(rs, w, d_bytes, d_off);
  } else {
    verify_small_kernel<false><<<sm_count * ctas, kVerifyBlock, kVerifySmem, stream>>>(rs, w, d_bytes, d_off);
  }
  if (rs.max_prog_len > (uint32_t)kSmallProg) {
    k++;
    if (want_spans) verify_large_kernel<true><<<sm_count * 4, kVerifyThreads, 0, stream>>>(rs, w, d_bytes, d_off);
    else verify_large_kernel<false><<<sm_count * 4, kVerifyThreads, 0, stream>>>(rs, w, d_bytes, d_off);
  }
  return k;
}

int launch_verdicts(const DevRuleset& rs, const ScanWork& w, uint32_t* d_verdicts, uint32_t n, int sm_count, cudaStream_t stream) {
  verdict_kernel<<<sm_count * 2, 256, 0, stream>>>(rs, w, d_verdicts, n);
  return 1;
}

int launch_hit_count(const ScanWork& w, const uint64_t* d_words, uint32_t n, int sm_count, cudaStream_t stream) {
  hit_count_kernel<<<sm_count * 4, 256, 0, stream>>>(d_words, n, w.out_len);
  return 1 + launch_exclusive_scan(w.out_len, w.out_off, n + 1, w.scan_part, sm_count, stream);
}
int launch_hit_emit(const DevRuleset& rs, const ScanWork& w, uint32_t n, uint32_t* d_out, uint32_t cap, uint32_t* d_count, int sm_count, cudaStream_t stream) {
  const uint32_t blocks = std::max<uint32_t>(1u, std::min<uint32_t>((uint32_t)(((uint64_t)n + 255) / 256), (uint32_t)sm_count * 4));   // 8 warps x 32 messages per block
  hit_emit_kernel<<<blocks, 256, 0, stream>>>(rs, w, n, d_out, cap, d_count);
  return 1;
}

// cg_scan_one: out = [word lo, word hi][counter block][hit row of the message, rw words] (kernels.h: kOneCounters, kOneHitRow)
__global__ void pack_one_kernel(DevRuleset rs, ScanWork w, const uint64_t* __restrict__ word, uint32_t* __restrict__ out, uint32_t rw_cap) {
  const uint32_t t = threadIdx.x;
  if (t == 0) { out[0] = (uint32_t)word[0]; out[1] = (uint32_t)(word[0] >> 32); }
  if (t < kCounterWords) out[kOneCounters + t] = w.counters[t];
  const uint32_t s = w.slot_of_msg[0];
  for (uint32_t k = t; k < rs.rw && k < rw_cap; k += blockDim.x) out[kOneHitRow + k] = (s != 0xffffffffu && s < w.slot_cap) ? w.hit[(size_t)s * rs.rw + k] : 0u;
}
int launch_pack_one(const DevRuleset& rs, const ScanWork& w, const uint64_t* d_word, uint32_t* d_out, uint32_t rw_cap, cudaStream_t stream) {
  pack_one_kernel<<<1, 64, 0, stream>>>(rs, w, d_word, d_out, rw_cap);
  return 1;
}

int launch_reset(const DevRuleset& rs, const ScanWork& w, uint32_t n, int sm_count, cudaStream_t stream) {
  reset_kernel<<<sm_count * 4, 256, 0, stream>>>(rs, w, n);
  return 1;
}

int launch_finalize(const DevRuleset& rs, const ScanWork& w, uint64_t* d_words, uint32_t n, int sm_count, cudaStream_t stream) {
  finalize_kernel<<<sm_count * 2, 256, 0, stream>>>(rs, w, d_words, n);
  return 1;
}

}  // namespace cg
