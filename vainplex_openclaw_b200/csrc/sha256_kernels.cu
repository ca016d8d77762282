// sha256_kernels.cu -- batched SHA-256 and the Proof-of-Guardrails Merkle tree (sm_90a).
//
// Replaces createHash("sha256").update(s).digest() (gov/src/util.ts:77-79, gov/src/redaction/
// vault.ts:26-28, nats/src/hooks.ts:90-94) for batches, and builds the Merkle tree the reference
// only describes (README "Proof-of-Guardrails"; RFC.md:782-800 specifies a hash chain that was
// never implemented).  Convention (frozen in oracle/sha256_merkle.c, restated in DESIGN.md):
//   leaf = SHA-256(0x00 || bytes), node = SHA-256(0x01 || L || R), unpaired node promoted.
// All 64 rounds run in registers; digests are stored in HBM as the canonical 32 big-endian bytes.
#include "kernels.h"
#include <algorithm>

namespace cg {

__constant__ uint32_t K256[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
    0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
    0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};

__device__ __forceinline__ uint32_t rotr(uint32_t x, int n) { return __funnelshift_r(x, x, n); }
__device__ __forceinline__ uint32_t bswap(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

__device__ __forceinline__ void sha_init(uint32_t h[8]) {
  h[0] = 0x6a09e667; h[1] = 0xbb67ae85; h[2] = 0x3c6ef372; h[3] = 0xa54ff53a;
  h[4] = 0x510e527f; h[5] = 0x9b05688c; h[6] = 0x1f83d9ab; h[7] = 0x5be0cd19;
}

// a + b on the FMA pipe: IMAD a, ONE, b with ONE = 1 read from constant memory at run time (a literal 1 is folded back
// into IADD3 by ptxas).  SHA-256 rounds are mostly SHF and LOP3, which must run on the integer ALU pipe while the FMA pipe
// idles; additions need not.
__constant__ uint32_t kRuntimeOne = 1;
__device__ __forceinline__ uint32_t add_fma(uint32_t a, uint32_t b) { return a * kRuntimeOne + b; }

// one compression; w[16] is clobbered (rolling message schedule, all in registers)
__device__ __forceinline__ void sha_compress(uint32_t h[8], uint32_t w[16]) {
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll
  for (int t = 0; t < 64; t++) {
    uint32_t wt;
    if (t < 16) wt = w[t];
    else {
      uint32_t w15 = w[(t - 15) & 15], w2 = w[(t - 2) & 15];
      uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ (w15 >> 3);
      uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ (w2 >> 10);
      wt = add_fma(add_fma(w[t & 15], s0), add_fma(w[(t - 7) & 15], s1));
      w[t & 15] = wt;
    }
    uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
    uint32_t ch = (e & f) ^ (~e & g);
    uint32_t t1 = add_fma(add_fma(add_fma(hh, S1), add_fma(ch, K256[t])), wt);
    uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
    uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
    uint32_t t2 = add_fma(S0, mj);
    hh = g; g = f; f = e; e = add_fma(d, t1); d = c; c = b; b = a; a = add_fma(t1, t2);
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

__device__ __forceinline__ void store_digest(uint32_t* out, const uint32_t h[8]) {
  uint4 a = make_uint4(bswap(h[0]), bswap(h[1]), bswap(h[2]), bswap(h[3]));
  uint4 b = make_uint4(bswap(h[4]), bswap(h[5]), bswap(h[6]), bswap(h[7]));
  reinterpret_cast<uint4*>(out)[0] = a; reinterpret_cast<uint4*>(out)[1] = b;
}

// generic: SHA-256 of [prefix byte if prefix >= 0] || data[0,len) ; byte-granular, any alignment
__device__ void sha_bytes(int prefix, const uint8_t* __restrict__ data, uint64_t len, uint32_t h[8]) {
  sha_init(h);
  const uint64_t p = prefix >= 0 ? 1 : 0, total = p + len;
  const uint64_t nblk = (total + 9 + 63) / 64;
  for (uint64_t blk = 0; blk < nblk; blk++) {
    uint32_t w[16];
#pragma unroll
    for (int t = 0; t < 16; t++) {
      uint32_t v = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        uint64_t idx = blk * 64 + t * 4 + k;   // index in the padded message
        uint32_t byte;
        if (idx < p) byte = (uint32_t)prefix;
        else if (idx < total) byte = data[idx - p];
        else if (idx == total) byte = 0x80;
        else byte = 0;
        v = (v << 8) | byte;
      }
      w[t] = v;
    }
    if (blk == nblk - 1) { uint64_t bits = total * 8; w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
    sha_compress(h, w);
  }
}

// The same for ragged inputs at any alignment, word-granular: the padded message is a byte stream that starts at address
// A = data - (1 if there is a prefix byte); message word m is the four bytes at A + 4m, fetched as two ALIGNED 32-bit loads
// and one funnel shift.  Only the first word (prefix byte) and the words around the end of the data (0x80, zeros, length)
// are patched.  The caller guarantees that the aligned words covering [A, data + len) are readable (up to 3 bytes before
// and 7 bytes after the data: every buffer this is called on is one of the library's own, padded on both sides).
__device__ void sha_words(int prefix, const uint8_t* __restrict__ data, uint64_t len, uint32_t h[8]) {
  sha_init(h);
  const uint32_t p = prefix >= 0 ? 1u : 0u;
  const uint64_t total = p + len, nblk = (total + 9 + 63) / 64;
  const uintptr_t A = reinterpret_cast<uintptr_t>(data) - p;
  const uint32_t* base = reinterpret_cast<const uint32_t*>(A & ~(uintptr_t)3);
  const uint32_t sh = 8u * (uint32_t)(A & 3u);
  uint32_t lo = __ldg(base);                           // aligned word holding stream byte 0
  uint64_t q = 1;                                      // next aligned word to fetch
  for (uint64_t blk = 0; blk < nblk; blk++) {
    uint32_t w[16];
#pragma unroll
    for (int t = 0; t < 16; t++) {
      const uint64_t m = blk * 16 + t, b0 = 4 * m;     // stream bytes [b0, b0 + 4)
      uint32_t v = 0;
      if (b0 < total) {
        // (the second aligned word is only touched when the stream word really straddles into it and it still holds data)
        uint32_t hi = 0;
        if (sh && b0 + 4 - (sh >> 3) < total) hi = __ldg(base + q);
        if (!sh) { v = lo; lo = (b0 + 4 < total) ? __ldg(base + q) : 0u; }
        else { v = __funnelshift_r(lo, hi, sh); lo = hi; }
        q++;
        v = bswap(v);
        if (m == 0 && p) v = (v & 0x00ffffffu) | ((uint32_t)prefix << 24);
        if (b0 + 4 > total) { const uint32_t k = (uint32_t)(total - b0); v = (v & (0xffffffffu << (32 - 8 * k))) | (0x80u << (24 - 8 * k)); }
      } else if (b0 == total) v = 0x80000000u;
      w[t] = v;
    }
    if (blk == nblk - 1) { const uint64_t bits = total * 8; w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
    sha_compress(h, w);
  }
}

__global__ void __launch_bounds__(128) sha256_batch_kernel(const uint8_t* __restrict__ bytes, const uint64_t* __restrict__ off,
                                                            uint32_t n, uint32_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t h[8];
  sha_words(-1, bytes + off[i], off[i + 1] - off[i], h);
  store_digest(out + (size_t)i * 8, h);
}

// leaf i = bytes[off[i], off[i+1]) ; with trim_newline a final '\n' of the range is not part of the leaf (JSONL lines,
// audit-trail.ts:168: records joined with "\n" plus a trailing "\n" per flush)
__global__ void __launch_bounds__(128) merkle_leaves_var_kernel(const uint8_t* __restrict__ bytes, const uint64_t* __restrict__ off,
                                                                 uint64_t n, uint32_t* __restrict__ out, int trim_newline) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t h[8];
  uint64_t b = off[i], e = off[i + 1];
  if (trim_newline && e > b && bytes[e - 1] == '\n') e--;
  sha_words(0x00, bytes + b, e - b, h);
  store_digest(out + i * 8, h);
}

// fixed-size leaves whose length is a multiple of 4 and whose base is 4-byte aligned:
// word loads, the 0x00 domain-separation byte shifts every message word by one byte.
__global__ void __launch_bounds__(128) merkle_leaves_fixed_kernel(const uint8_t* __restrict__ bytes, uint32_t leaf_words,
                                                                   uint64_t n, uint32_t* __restrict__ out) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t* leaf = reinterpret_cast<const uint32_t*>(bytes) + i * leaf_words;
  uint32_t h[8]; sha_init(h);
  const uint32_t total = 1 + leaf_words * 4;           // bytes incl. prefix
  const uint32_t nblk = (total + 9 + 63) / 64;
  uint32_t prev = 0;                                   // big-endian word preceding the current one (prefix 0x00 in its low byte)
  uint32_t widx = 0;                                   // next leaf word to consume
  for (uint32_t blk = 0; blk < nblk; blk++) {
    uint32_t w[16];
#pragma unroll
    for (int t = 0; t < 16; t++) {
      // message word m = blk*16+t covers message bytes [4m, 4m+4) = leaf bytes [4m-1, 4m+3)
      uint32_t m = blk * 16 + t;
      uint32_t cur;
      if (m < leaf_words) { cur = bswap(__ldg(leaf + widx)); widx++; }
      else if (m == leaf_words) cur = 0x80000000u >> 0;  // leaf exhausted: next byte after data is 0x80
      else cur = 0;
      // bytes: low byte of prev, then top three bytes of cur
      uint32_t v = (prev << 24) | (cur >> 8);
      if (m == leaf_words) v = (prev << 24) | 0x00800000u;
      else if (m > leaf_words) v = 0;
      w[t] = v;
      prev = cur;
    }
    if (blk == nblk - 1) { w[14] = 0; w[15] = total * 8; }
    sha_compress(h, w);
  }
  store_digest(out + i * 8, h);
}

// node = SHA-256(0x01 || L || R): 65 bytes = two blocks
__device__ __forceinline__ void merkle_node(const uint32_t l[8], const uint32_t r[8], uint32_t h[8]) {
  // l, r hold big-endian digest words (i.e. the SHA state words)
  uint32_t w[16];
  w[0] = 0x01000000u | (l[0] >> 8);
#pragma unroll
  for (int t = 1; t < 8; t++) w[t] = (l[t - 1] << 24) | (l[t] >> 8);
  w[8] = (l[7] << 24) | (r[0] >> 8);
#pragma unroll
  for (int t = 1; t < 8; t++) w[8 + t] = (r[t - 1] << 24) | (r[t] >> 8);
  sha_init(h);
  sha_compress(h, w);
  w[0] = (r[7] << 24) | 0x00800000u;
#pragma unroll
  for (int t = 1; t < 15; t++) w[t] = 0;
  w[15] = 65 * 8;
  sha_compress(h, w);
}

__device__ __forceinline__ void load_digest(const uint32_t* p, uint32_t d[8]) {
  uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
  d[0] = bswap(a.x); d[1] = bswap(a.y); d[2] = bswap(a.z); d[3] = bswap(a.w);
  d[4] = bswap(b.x); d[5] = bswap(b.y); d[6] = bswap(b.z); d[7] = bswap(b.w);
}

__global__ void __launch_bounds__(128) merkle_level_kernel(const uint32_t* __restrict__ in, uint64_t n_in, uint32_t* __restrict__ out) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t n_out = (n_in + 1) / 2;
  if (i >= n_out) return;
  if (2 * i + 1 < n_in) {
    uint32_t l[8], r[8], h[8];
    load_digest(in + 16 * i, l); load_digest(in + 16 * i + 8, r);
    merkle_node(l, r, h);
    store_digest(out + 8 * i, h);
  } else {
    reinterpret_cast<uint4*>(out + 8 * i)[0] = reinterpret_cast<const uint4*>(in + 16 * i)[0];
    reinterpret_cast<uint4*>(out + 8 * i)[1] = reinterpret_cast<const uint4*>(in + 16 * i)[1];
  }
}

// ------------------------------------------------------------------------------------------
// Merkle log helpers (append-only log: frontier carries, root fold, audit-path check) -- a handful of node hashes
// per call, run by one thread on the device (the product computes no hash on the CPU)
// ------------------------------------------------------------------------------------------
// acc = node(left[k], acc) for k = 0..n_left-1 : frontier carry chains and the root fold.  left: n_left digests.
__global__ void merkle_chain_kernel(const uint32_t* __restrict__ left, uint32_t n_left, const uint32_t* __restrict__ acc_in, uint32_t* __restrict__ acc_out) {
  if (threadIdx.x || blockIdx.x) return;
  uint32_t r[8]; load_digest(acc_in, r);
  for (uint32_t k = 0; k < n_left; k++) { uint32_t l[8], h[8]; load_digest(left + 8 * k, l); merkle_node(l, r, h);
#pragma unroll
    for (int t = 0; t < 8; t++) r[t] = h[t]; }
  store_digest(acc_out, r);
}
// RFC 9162 2.1.3.2: does `path` prove that the leaf with digest leaf32 is entry `index` of the tree of `size` leaves with root `root32`?
__global__ void merkle_verify_kernel(const uint32_t* __restrict__ leaf32, unsigned long long index, unsigned long long size,
                                     const uint32_t* __restrict__ path, uint32_t path_len, const uint32_t* __restrict__ root32, uint32_t* __restrict__ ok) {
  if (threadIdx.x || blockIdx.x) return;
  *ok = 0;
  if (index >= size) return;
  unsigned long long fn = index, sn = size - 1;
  uint32_t r[8]; load_digest(leaf32, r);
  for (uint32_t k = 0; k < path_len; k++) {
    if (sn == 0) return;
    uint32_t p[8], h[8]; load_digest(path + 8 * k, p);
    if ((fn & 1ull) || fn == sn) {
      merkle_node(p, r, h);
      if (!(fn & 1ull)) while (!(fn & 1ull) && fn != 0) { fn >>= 1; sn >>= 1; }
    } else merkle_node(r, p, h);
#pragma unroll
    for (int t = 0; t < 8; t++) r[t] = h[t];
    fn >>= 1; sn >>= 1;
  }
  if (sn != 0) return;
  uint32_t q[8]; load_digest(root32, q);
  bool eq = true;
#pragma unroll
  for (int t = 0; t < 8; t++) eq = eq && q[t] == r[t];
  *ok = eq ? 1u : 0u;
}
// RFC 9162 2.1.4.2: does `path` prove that the tree of `first` leaves with root first32 is a prefix of the tree of
// `second` leaves with root second32?
__global__ void merkle_consistency_kernel(unsigned long long first, unsigned long long second, const uint32_t* __restrict__ first32,
                                          const uint32_t* __restrict__ second32, const uint32_t* __restrict__ path, uint32_t path_len, uint32_t* __restrict__ ok) {
  if (threadIdx.x || blockIdx.x) return;
  *ok = 0;
  if (first == 0 || first > second) return;
  uint32_t f1[8], f2[8]; load_digest(first32, f1); load_digest(second32, f2);
  if (first == second) { bool eq = path_len == 0; for (int t = 0; t < 8; t++) eq = eq && f1[t] == f2[t]; *ok = eq ? 1u : 0u; return; }
  unsigned long long fn = first - 1, sn = second - 1;
  const bool pow2 = (first & (first - 1)) == 0;            // then the old root itself is the first element of the walk
  while (fn & 1ull) { fn >>= 1; sn >>= 1; }
  uint32_t fr[8], sr[8], k = 0;
  if (pow2) { for (int t = 0; t < 8; t++) fr[t] = sr[t] = f1[t]; }
  else { if (path_len == 0) return; load_digest(path, fr); for (int t = 0; t < 8; t++) sr[t] = fr[t]; k = 1; }
  for (; k < path_len; k++) {
    if (sn == 0) return;
    uint32_t c[8], h[8]; load_digest(path + 8 * k, c);
    if ((fn & 1ull) || fn == sn) {
      merkle_node(c, fr, h); for (int t = 0; t < 8; t++) fr[t] = h[t];
      merkle_node(c, sr, h); for (int t = 0; t < 8; t++) sr[t] = h[t];
      if (!(fn & 1ull)) while (!(fn & 1ull) && fn != 0) { fn >>= 1; sn >>= 1; }
    } else { merkle_node(sr, c, h); for (int t = 0; t < 8; t++) sr[t] = h[t]; }
    fn >>= 1; sn >>= 1;
  }
  bool eq = sn == 0;
  for (int t = 0; t < 8; t++) eq = eq && fr[t] == f1[t] && sr[t] == f2[t];
  *ok = eq ? 1u : 0u;
}

// Up to five tree levels inside one warp: lane i holds node i of an aligned group of 32 (fewer at the ragged end), the
// pairwise reduction runs through shuffles -- at step s the lanes with (i mod 2^(s+1)) == 0 hash their node with the one
// 2^s lanes up, an unpaired node is promoted unchanged -- and only the group's root goes back to HBM.  Used for the small
// upper levels of every tree and for the short trees of log appends, where a kernel launch per level costs more than the
// idle lanes do (the large lower levels keep every lane busy in merkle_level_kernel).
__global__ void __launch_bounds__(256) merkle_reduce_kernel(const uint32_t* __restrict__ in, uint64_t n_in, uint32_t levels, uint32_t* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31u, span = 1u << levels;                   // nodes per group (<= 32)
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t gpw = 32u >> levels;                                             // groups per warp
  const uint64_t group = warp * gpw + lane / span, n_groups = (n_in + span - 1) / span;
  const uint64_t node = group * span + (lane & (span - 1));
  bool have = group < n_groups && node < n_in;
  uint32_t d[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (have) load_digest(in + 8 * node, d);
  for (uint32_t s = 0; s < levels; s++) {
    uint32_t o[8];
#pragma unroll
    for (int t = 0; t < 8; t++) o[t] = __shfl_down_sync(0xffffffffu, d[t], 1u << s);
    const bool ohave = __shfl_down_sync(0xffffffffu, have ? 1u : 0u, 1u << s) != 0;
    if (((lane & (span - 1)) & ((2u << s) - 1u)) == 0 && have && ohave) {
      uint32_t h[8]; merkle_node(d, o, h);
#pragma unroll
      for (int t = 0; t < 8; t++) d[t] = h[t];
    }
  }
  if ((lane & (span - 1)) == 0 && have) store_digest(out + 8 * group, d);
}

// JSONL split on the device: line i of the buffer = bytes[starts[i], starts[i+1]) including its '\n' (the last line may
// lack one).  Three small kernels: newline count per 4 KB piece, exclusive scan over the pieces (one block), line starts.
constexpr uint32_t kSplitPiece = 4096;
__global__ void __launch_bounds__(256) newline_count_kernel(const uint8_t* __restrict__ bytes, uint64_t len, uint32_t* __restrict__ counts) {
  const uint64_t lo = (uint64_t)blockIdx.x * kSplitPiece, hi = lo + kSplitPiece < len ? lo + kSplitPiece : len;
  uint32_t c = 0;
  for (uint64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) c += bytes[i] == '\n';
  __shared__ uint32_t sm[8];
  for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) { uint32_t t = 0; for (int k = 0; k < 8; k++) t += sm[k]; counts[blockIdx.x] = t; }
}
__global__ void __launch_bounds__(1024) newline_scan_kernel(uint32_t* __restrict__ counts, uint32_t n_pieces, uint64_t* __restrict__ total_lines, uint64_t len, const uint8_t* __restrict__ bytes) {
  // exclusive scan in place, one block (n_pieces <= a few hundred thousand: 1 GB of JSONL is 262144 pieces)
  __shared__ uint32_t carry, warp_sum[32];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < n_pieces; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    uint32_t v = i < n_pieces ? counts[i] : 0, incl = v;
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if ((threadIdx.x & 31) >= (uint32_t)d) incl += t; }
    if ((threadIdx.x & 31) == 31) warp_sum[threadIdx.x >> 5] = incl;
    __syncthreads();
    if (threadIdx.x < 32) { uint32_t w = warp_sum[threadIdx.x], wi = w; for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, wi, d); if (threadIdx.x >= (uint32_t)d) wi += t; } warp_sum[threadIdx.x] = wi - w; }
    __syncthreads();
    const uint32_t excl = carry + warp_sum[threadIdx.x >> 5] + incl - v;
    if (i < n_pieces) counts[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total_lines = (uint64_t)carry + ((len && bytes[len - 1] != '\n') ? 1u : 0u);      // + an unterminated last line
}
__global__ void __launch_bounds__(256) newline_starts_kernel(const uint8_t* __restrict__ bytes, uint64_t len, const uint32_t* __restrict__ piece_rank, uint64_t* __restrict__ starts, uint64_t n_lines) {
  // starts[0] = 0; the line after the r-th newline (0-based) starts at its position + 1; starts[n_lines] = len
  const uint64_t lo = (uint64_t)blockIdx.x * kSplitPiece, hi = lo + kSplitPiece < len ? lo + kSplitPiece : len;
  if (blockIdx.x == 0 && threadIdx.x == 0) { starts[0] = 0; starts[n_lines] = len; }
  __shared__ uint32_t run;
  if (threadIdx.x == 0) run = piece_rank[blockIdx.x];
  __syncthreads();
  for (uint64_t b = lo; b < hi; b += blockDim.x) {                // 256 bytes at a time, in order
    const uint64_t i = b + threadIdx.x;
    const bool nl = i < hi && bytes[i] == '\n';
    const uint32_t m = __ballot_sync(0xffffffffu, nl);
    __shared__ uint32_t wcnt[8];
    if ((threadIdx.x & 31) == 0) wcnt[threadIdx.x >> 5] = __popc(m);
    __syncthreads();
    uint32_t before = run;
    for (uint32_t k = 0; k < (threadIdx.x >> 5); k++) before += wcnt[k];
    if (nl) starts[(uint64_t)before + __popc(m & ((1u << (threadIdx.x & 31)) - 1u)) + 1] = i + 1;     // (the r-th newline ends line r)
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t t = 0; for (int k = 0; k < 8; k++) t += wcnt[k]; run += t; }
    __syncthreads();
  }
}
int launch_newline_split(const uint8_t* d_bytes, uint64_t len, uint32_t* d_piece_counts, uint64_t* d_total_lines, cudaStream_t stream) {
  if (!len) return 0;
  const uint32_t n_pieces = (uint32_t)((len + kSplitPiece - 1) / kSplitPiece);
  newline_count_kernel<<<n_pieces, 256, 0, stream>>>(d_bytes, len, d_piece_counts);
  newline_scan_kernel<<<1, 1024, 0, stream>>>(d_piece_counts, n_pieces, d_total_lines, len, d_bytes);
  return 2;
}
int launch_newline_starts(const uint8_t* d_bytes, uint64_t len, const uint32_t* d_piece_rank, uint64_t* d_starts, uint64_t n_lines, cudaStream_t stream) {
  if (!len) return 0;
  const uint32_t n_pieces = (uint32_t)((len + kSplitPiece - 1) / kSplitPiece);
  newline_starts_kernel<<<n_pieces, 256, 0, stream>>>(d_bytes, len, d_piece_rank, d_starts, n_lines);
  return 1;
}
int launch_merkle_consistency(uint64_t first, uint64_t second, const uint32_t* d_first32, const uint32_t* d_second32, const uint32_t* d_path, uint32_t path_len, uint32_t* d_ok, cudaStream_t stream) {
  merkle_consistency_kernel<<<1, 32, 0, stream>>>(first, second, d_first32, d_second32, d_path, path_len, d_ok);
  return 1;
}
int launch_merkle_chain(const uint32_t* d_left, uint32_t n_left, const uint32_t* d_acc_in, uint32_t* d_acc_out, cudaStream_t stream) {
  merkle_chain_kernel<<<1, 32, 0, stream>>>(d_left, n_left, d_acc_in, d_acc_out);
  return 1;
}
int launch_merkle_verify(const uint32_t* d_leaf32, uint64_t index, uint64_t size, const uint32_t* d_path, uint32_t path_len, const uint32_t* d_root32, uint32_t* d_ok, cudaStream_t stream) {
  merkle_verify_kernel<<<1, 32, 0, stream>>>(d_leaf32, index, size, d_path, path_len, d_root32, d_ok);
  return 1;
}

// ------------------------------------------------------------------------------------------
// redacted-output assembly (RedactionEngine.applyReplacements, engine.ts:165-181, with the vault's placeholder
// "[REDACTED:<category>:<first 8 hex digits of SHA-256(match)>]", vault.ts:33-35,75-104)
// ------------------------------------------------------------------------------------------
// SHA-256 of every matched text: span i = bytes[start[i], start[i] + len[i]) for i < *ns (the count is the resolver's)
__global__ void __launch_bounds__(128) redact_digest_kernel(const uint8_t* __restrict__ bytes, const uint32_t* __restrict__ start,
                                                             const uint32_t* __restrict__ len, const uint32_t* __restrict__ ns, uint32_t* __restrict__ out) {
  const uint32_t cnt = *ns;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += gridDim.x * blockDim.x) {
    uint32_t h[8];
    sha_bytes(-1, bytes + start[i], len[i], h);
    store_digest(out + (size_t)i * 8, h);
  }
}

__constant__ char kCatName[4][12] = {"credential", "financial", "pii", "custom"};       // CATEGORY_ORDER, registry.ts:17-22
__constant__ uint8_t kCatLen[4] = {10, 9, 3, 6};

// One warp per message: the text between spans is copied, every span is replaced by its placeholder.
// span_begin[msg] .. span_begin[msg+1] index the (position-sorted, non-overlapping) spans of the message.
__global__ void __launch_bounds__(256) redact_splice_kernel(const uint8_t* __restrict__ bytes, const uint32_t* __restrict__ off,
                                                             const uint32_t* __restrict__ out_off, const uint32_t* __restrict__ span_begin,
                                                             const uint32_t* __restrict__ span_start, const uint32_t* __restrict__ span_len,
                                                             const uint32_t* __restrict__ span_cat, const uint32_t* __restrict__ digests,
                                                             uint8_t* __restrict__ out, const uint32_t* __restrict__ n_msgs) {
  const uint32_t lane = threadIdx.x & 31u, wpb = blockDim.x >> 5, n = *n_msgs;
  for (uint32_t msg = blockIdx.x * wpb + (threadIdx.x >> 5); msg < n; msg += gridDim.x * wpb) {
    const uint32_t b = off[msg], e = off[msg + 1];
    uint32_t src = b, dst = out_off[msg];
    for (uint32_t k = span_begin[msg], ke = span_begin[msg + 1]; k <= ke; k++) {
      const uint32_t stop = k < ke ? span_start[k] : e;          // copy bytes[src, stop)
      for (uint32_t i = lane; i < stop - src; i += 32u) out[dst + i] = bytes[src + i];
      dst += stop - src;
      if (k == ke) break;
      const uint32_t cat = span_cat[k] & 3u, cl = kCatLen[cat];
      // "[REDACTED:" cat ":" hhhhhhhh "]"   = 10 + cl + 1 + 8 + 1 bytes, one byte per lane
      const uint32_t plen = 20u + cl;
      if (lane < plen) {
        uint8_t ch;
        if (lane < 10u) ch = (uint8_t)"[REDACTED:"[lane];
        else if (lane < 10u + cl) ch = (uint8_t)kCatName[cat][lane - 10u];
        else if (lane == 10u + cl) ch = ':';
        else if (lane < 19u + cl) {
          const uint32_t d = lane - (11u + cl);                   // hex digit 0..7 of the digest (bytes 0..3)
          const uint32_t word = digests[(size_t)k * 8];           // stored big-endian byte order in memory: byte j = (word >> 8j) & 0xff
          const uint32_t byte = (word >> (8u * (d >> 1))) & 0xffu, nib = (d & 1u) ? (byte & 15u) : (byte >> 4);
          ch = (uint8_t)(nib < 10u ? '0' + nib : 'a' + nib - 10u);
        } else ch = ']';
        out[dst + lane] = ch;
      }
      dst += plen;
      src = span_start[k] + span_len[k];
    }
  }
}

int launch_redact_digests(const uint8_t* d_bytes, const uint32_t* d_start, const uint32_t* d_len, const uint32_t* d_ns, uint32_t* d_out,
                          int sm_count, cudaStream_t stream) {
  redact_digest_kernel<<<sm_count * 8, 128, 0, stream>>>(d_bytes, d_start, d_len, d_ns, d_out);
  return 1;
}
int launch_redact_splice(const uint8_t* d_bytes, const uint32_t* d_off, const uint32_t* d_out_off, const uint32_t* d_span_begin,
                         const uint32_t* d_span_start, const uint32_t* d_span_len, const uint32_t* d_span_cat, const uint32_t* d_digests,
                         uint8_t* d_out, const uint32_t* d_n, uint32_t n_max, int sm_count, cudaStream_t stream) {
  if (!n_max) return 0;
  const uint32_t grid = std::min<uint32_t>((n_max + 7) / 8, (uint32_t)sm_count * 8u);
  redact_splice_kernel<<<grid, 256, 0, stream>>>(d_bytes, d_off, d_out_off, d_span_begin, d_span_start, d_span_len, d_span_cat, d_digests, d_out, d_n);
  return 1;
}

int launch_sha256_batch(const uint8_t* d_bytes, const uint64_t* d_off, uint32_t n, uint8_t* d_out, cudaStream_t stream) {
  if (!n) return 0;
  sha256_batch_kernel<<<(n + 127) / 128, 128, 0, stream>>>(d_bytes, d_off, n, reinterpret_cast<uint32_t*>(d_out));
  return 1;
}
// fixed-size leaves of any length / alignment (byte-granular path)
__global__ void __launch_bounds__(128) merkle_leaves_fixed_generic_kernel(const uint8_t* __restrict__ bytes, uint64_t leaf_len,
                                                                           uint64_t n, uint32_t* __restrict__ out) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t h[8];
  sha_bytes(0x00, bytes + i * leaf_len, leaf_len, h);
  store_digest(out + i * 8, h);
}

int launch_merkle_leaves_fixed(const uint8_t* d_bytes, uint64_t leaf_len, uint64_t n, uint32_t* d_out, cudaStream_t stream) {
  if (!n) return 0;
  if (leaf_len == 0 || (leaf_len & 3) || (reinterpret_cast<uintptr_t>(d_bytes) & 3) || leaf_len > (1u << 28)) {
    merkle_leaves_fixed_generic_kernel<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(d_bytes, leaf_len, n, d_out);
    return 1;
  }
  merkle_leaves_fixed_kernel<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(d_bytes, (uint32_t)(leaf_len / 4), n, d_out);
  return 1;
}
int launch_merkle_leaves_var(const uint8_t* d_bytes, const uint64_t* d_off, uint64_t n, uint32_t* d_out, cudaStream_t stream, bool trim_newline) {
  if (!n) return 0;
  merkle_leaves_var_kernel<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(d_bytes, d_off, n, d_out, trim_newline ? 1 : 0);
  return 1;
}
static int launch_merkle_level(const uint32_t* d_in, uint64_t n_in, uint32_t* d_out, cudaStream_t stream) {
  uint64_t n_out = (n_in + 1) / 2;
  if (!n_out) return 0;
  merkle_level_kernel<<<(unsigned)((n_out + 127) / 128), 128, 0, stream>>>(d_in, n_in, d_out);
  return 1;
}
static int launch_merkle_reduce(const uint32_t* d_in, uint64_t n_in, uint32_t levels, uint32_t* d_out, cudaStream_t stream) {
  if (!n_in || levels == 0 || levels > 5) return 0;
  const uint64_t n_groups = (n_in + (1ull << levels) - 1) >> levels, warps = (n_groups + (32u >> levels) - 1) / (32u >> levels);
  merkle_reduce_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(d_in, n_in, levels, d_out);
  return 1;
}
// Above 2^15 nodes a level is one launch of merkle_level_kernel (every lane busy); from 2^15 nodes down merkle_reduce_kernel
// folds min(5, levels left under max_levels, ceil(log2 n)) levels per launch, where a launch costs more than idle lanes do.
int launch_merkle_fold(const uint32_t* d_in, uint64_t n, uint32_t max_levels, uint32_t* d_a, uint32_t* d_b, cudaStream_t stream,
                       const uint32_t** d_result) {
  int k = 0;
  const uint32_t* src = d_in; uint32_t* dst = d_a;
  for (uint32_t lv = 0; n > 1 && lv < max_levels;) {
    uint32_t step = 1;
    if (n <= (1u << 15)) { step = std::min(5u, max_levels - lv); while (step > 1 && (1ull << (step - 1)) >= n) step--; }
    k += step > 1 ? launch_merkle_reduce(src, n, step, dst, stream) : launch_merkle_level(src, n, dst, stream);
    n = (n + (1ull << step) - 1) >> step; lv += step;
    src = dst; dst = dst == d_a ? d_b : d_a;
  }
  *d_result = src;
  return k;
}

}  // namespace cg
