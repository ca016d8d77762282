// bitprog.h -- RegExp.test around a confirmed factor occurrence for the rules whose Pike program has at most 63 consuming
// instructions and no lookaround: a bit-parallel simulation of the same program (one bit per consuming instruction, bit 63
// = MATCH), one THREAD per occurrence instead of one warp per Pike-VM run.
//
// What makes the boolean answer of gov/src/conditions/context.ts:9-25 (RegExp.test per rule) independent of thread
// priorities: a match exists iff MATCH is reachable from some start position, whatever the order alternatives are tried
// in; the empty-iteration check of ECMA-262 22.2.2.3.1 step 2.b only prunes iterations that consume nothing, which
// never changes the set of end positions reachable (no backreferences, no lookaround in these programs).  So the
// program's epsilon edges are closed once, at compile time, per context of the position between two units -- the
// assertions ^ $ \b \B only look at (word boundary?, start of message?, end of message?) -- and a step is
// "accepting instructions for this byte" & "live instructions", then OR of the follow masks of what is left.
//
// ASCII only: a byte >= 0x80 inside the island hands the occurrence to the Pike VM (UTF-16 unit semantics, pike_vm.h).
// The tables are built from the rule's own Pike program (rulec.cpp output), so both matchers interpret ONE compilation.
#pragma once
#include <cstdint>
#include "kernels.h"
#include "pike_vm.h"

namespace cg {

// Table of one rule, W = 1 or 2 state words (uint64; consuming instruction k = bit k, MATCH = bit 64 W - 1):
//   W | accept[128][W] | start[32][W] | meta | rowmap[2] | behind[2] | ahead[2] | next[W] | self[W] | follow rows [n_rows][64 W][W]
//   context of the position between two units, 5 bits: word boundary, start of message, end of message, previous unit in the
//   rule's lookbehind set, next unit in its lookahead set (single-unit lookaround, one set per direction, ASCII-only sets:
//   the token-boundary guards (?<![A-Z0-9]) ... (?![A-Z0-9]) of the credential rules).  Contexts with identical follow rows
//   share one row: rowmap holds 4 bits per context.
//   meta = n_rows | W << 4 | start_same << 8 (start[] identical in every context) | has_look << 9
//   next / self = the instructions k whose follow set is, in every row, a subset of {k, k + 1}: bit k of `next` when it holds
//   k + 1 (the next unit of a literal or class run), bit k of `self` when it holds k (a loop on one unit).  Their successors
//   are a shift and a mask -- no load; only the other instructions (alternations, group loops) go through the follow rows.
constexpr uint32_t kBitProgNone = 0xffffffffu;
constexpr uint32_t kBitCtxs = 32;
CG_HD uint32_t bitprog_meta_off(uint32_t W) { return (128u + kBitCtxs) * W; }
CG_HD uint32_t bitprog_rows_off(uint32_t W) { return bitprog_meta_off(W) + 7u + 2u * W; }
CG_HD uint32_t bitprog_words(uint32_t W, uint32_t n_rows) { return bitprog_rows_off(W) + n_rows * 64u * W * W; }

// context of the position between the bytes `prev` and `next` (-1 = none; 0x80 = some non-ASCII unit)
CG_HD uint32_t bitprog_ctx(int prev, int next, bool at_start) {
  return (uint32_t)(is_word(prev) != is_word(next)) | (at_start ? 2u : 0u) | (next < 0 ? 4u : 0u);
}
CG_HD uint32_t bitprog_in128(uint64_t lo, uint64_t hi, int u) { return u < 0 || u >= 0x80 ? 0u : (uint32_t)(((u & 64) ? hi : lo) >> (u & 63)) & 1u; }

// -> 1 a match that starts in [s, t0] exists, 0 none, -1 cannot tell (non-ASCII byte in the island, or more than max_steps
// bytes to walk: ask the VM, whose warp-wide runs suit long islands better than one thread's chain of table loads).
// One thread walks the island, so what this costs is the length of its dependency chain, not its instruction count: the
// four next bytes and their accept masks are fetched together (loads that depend on the position alone), and only the
// state update is sequential -- a shift and a mask for most instructions, a follow row from L2 for the others.
// resume != nullptr: the walk starts at s with the given state and no further start positions (the compiler has already run the
// rule's program over the confirmed factor, whose elements the instructions accept as a whole or not at all: factor_skip below)
template <int W>
CG_HD int bitprog_test_w(const uint64_t* __restrict__ bp, const uint8_t* __restrict__ m, uint32_t len, uint32_t s, uint32_t t0, uint32_t max_steps, const uint64_t* __restrict__ resume = nullptr) {
  const uint64_t* accept = bp; const uint64_t* start = bp + 128 * W; const uint64_t* hd = bp + bitprog_meta_off(W); const uint64_t* rows = bp + bitprog_rows_off(W);
  const uint64_t meta = hd[0], map0 = hd[1], map1 = hd[2];
  const bool start_same = (meta >> 8) & 1u, has_look = (meta >> 9) & 1u, one_row = (meta & 15u) == 1u;
  const uint64_t lb0 = has_look ? hd[3] : 0, lb1 = has_look ? hd[4] : 0, la0 = has_look ? hd[5] : 0, la1 = has_look ? hd[6] : 0;
  uint64_t m_next[W], m_self[W], live[W], acc_cur[W], start0[W];
  constexpr uint64_t kMatch = 1ull << 63;            // of the last word
  for (int w = 0; w < W; w++) { m_next[w] = hd[7 + w]; m_self[w] = hd[7 + W + w]; }
  int prev = s > 0 ? (m[s - 1] < 0x80 ? (int)m[s - 1] : 0x80) : -1;          // (a unit >= 0x80 is not a word character, whatever it is)
  int cur = s < len ? (int)m[s] : -1;
  uint32_t ctx = bitprog_ctx(prev, cur, s == 0) | (has_look ? bitprog_in128(lb0, lb1, prev) << 3 | bitprog_in128(la0, la1, cur) << 4 : 0u);
  for (int w = 0; w < W; w++) { start0[w] = resume ? 0 : start[ctx * W + w]; live[w] = resume ? resume[w] : start0[w]; acc_cur[w] = cur >= 0 && cur < 0x80 ? accept[cur * W + w] : 0; }
  if (resume) t0 = s - 1;                        // (s >= 1: at least one factor element lies before it)
  for (uint32_t pos = s;;) {
    // the block's four "next" bytes and their accept masks
    int nb[4]; uint64_t na[4][W];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int i = 0; i < 4; i++) nb[i] = pos + 1 + i < len ? (int)m[pos + 1 + i] : -1;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int i = 0; i < 4; i++) for (int w = 0; w < W; w++) na[i][w] = nb[i] >= 0 && nb[i] < 0x80 ? accept[nb[i] * W + w] : 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int i = 0; i < 4; i++) {
      if (live[W - 1] & kMatch) return 1;
      if (cur < 0) return 0;
      if (cur >= 0x80 || pos - s >= max_steps) return -1;
      const int nxt = nb[i];
      uint64_t hit[W], carry = 0, any_hit = 0;
      for (int w = 0; w < W; w++) {
        const uint64_t h = live[w] & acc_cur[w], hn = h & m_next[w];
        live[w] = (hn << 1) | carry | (h & m_self[w]);
        carry = hn >> 63;
        hit[w] = h & ~(m_next[w] | m_self[w]); any_hit |= hit[w];
      }
      if (!start_same || any_hit) ctx = bitprog_ctx(cur, nxt < 0x80 ? nxt : 0x80, false) | (has_look ? bitprog_in128(lb0, lb1, cur) << 3 | bitprog_in128(la0, la1, nxt) << 4 : 0u);
      if (any_hit) {
        const uint32_t row = one_row ? 0u : (uint32_t)(((ctx & 16u) ? map1 : map0) >> (4 * (ctx & 15u))) & 15u;
        const uint64_t* fw = rows + (size_t)row * 64 * W * W;
        for (int w = 0; w < W; w++) {
          uint64_t hw = hit[w];
          while (hw) {
#if defined(__CUDA_ARCH__)
            const int k = __ffsll((long long)hw) - 1;
#else
            const int k = __builtin_ctzll(hw);
#endif
            hw &= hw - 1;
            for (int v = 0; v < W; v++) live[v] |= fw[(size_t)(w * 64 + k) * W + v];
          }
        }
      }
      pos++;
      if (pos <= t0) { for (int w = 0; w < W; w++) live[w] |= start_same ? start0[w] : start[ctx * W + w]; }      // a new start position (none beyond the factor occurrence)
      else { uint64_t any = 0; for (int w = 0; w < W; w++) any |= live[w]; if (!any) return 0; }
      cur = nxt;
      for (int w = 0; w < W; w++) acc_cur[w] = na[i][w];
    }
  }
}
CG_HD int bitprog_test(const uint64_t* __restrict__ bp, const uint8_t* __restrict__ m, uint32_t len, uint32_t s, uint32_t t0, uint32_t max_steps = 0xffffffffu, const uint64_t* __restrict__ resume = nullptr) {
  // (the table's first word is its width W)
  return bp[0] == 2 ? bitprog_test_w<2>(bp + 1, m, len, s, t0, max_steps, resume) : bitprog_test_w<1>(bp + 1, m, len, s, t0, max_steps, resume);
}

// one word of a 256-bit set held in eight registers
CG_HD uint32_t bitprog_sel8(const uint32_t a[8], uint32_t i) {
  const uint32_t lo = (i & 2u) ? ((i & 1u) ? a[3] : a[2]) : ((i & 1u) ? a[1] : a[0]);
  const uint32_t hi = (i & 2u) ? ((i & 1u) ? a[7] : a[6]) : ((i & 1u) ? a[5] : a[4]);
  return (i & 4u) ? hi : lo;
}

// the island's first byte: test_at_factor's start position (pike_vm.h), without the cursor (ASCII islands only matter here).
// Four bytes per round, the set in registers: the chain is the tests, not a load per byte.  Gives up `limit` bytes before t0
// (the caller then hands the occurrence to the VM: bitprog_test would not walk that far either).
CG_HD uint32_t island_start(const DevRuleset& rs, uint32_t rule, const uint8_t* __restrict__ m, uint32_t len, uint32_t t0, uint32_t pre_units, uint32_t limit = 0xffffffffu) {
  const uint32_t pa = pre_units >> 16; pre_units &= 0xffffu;
  const uint32_t* alpha = pa != 0xffffu ? rs.bytesets + (size_t)pa * 8 : rs.rule_alpha + (size_t)rule * 8;
  if (t0 > len) t0 = len;
  uint32_t s = t0;
  uint32_t floor_ = pre_units < 0xffffu ? (t0 > 3u * pre_units ? t0 - 3u * pre_units : 0u) : 0u;     // (earlier starts cannot reach the factor)
  if (limit != 0xffffffffu && t0 - floor_ > limit) floor_ = t0 - limit - (t0 > limit ? 1u : 0u);      // (one byte past the limit tells "too long" from "ends there")
  if (s <= floor_) return s;
  uint32_t a[8];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int i = 0; i < 8; i++) a[i] = alpha[i];
  for (;;) {
    uint32_t b[4];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (uint32_t i = 0; i < 4; i++) b[i] = s > floor_ + i ? m[s - 1 - i] : 0x100u;        // 0x100: stop
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (uint32_t i = 0; i < 4; i++) {
      if (b[i] > 0xffu || !((bitprog_sel8(a, b[i] >> 5) >> (b[i] & 31u)) & 1u)) return s;
      s--;
    }
  }
}


// RegExp.test around the occurrence of factor f of rule r at message offset t0: 1 / 0 / -1 (ask the VM).
// factor_skip[3 f] = L | state words: for a factor that starts its rule's matches (no pattern unit before it, no assertion in
// the rule) the compiler has run the program over the first L factor elements -- every live instruction accepts an element's
// whole byte set or none of it, so the state after them does not depend on the text -- and check_kernel has compared those
// very elements exactly: the walk resumes behind them.  A `sk-...` token costs 4 steps instead of 20.
CG_HD int island_test(const DevRuleset& rs, uint32_t f, uint32_t r, const uint8_t* __restrict__ m, uint32_t len, uint32_t t0, uint32_t pre, uint32_t max_steps) {
  const uint64_t* bp = reinterpret_cast<const uint64_t*>(rs.bit_words) + rs.bit_off[r];
  const uint64_t* resume = nullptr; uint32_t s = 0;
  if (f != 0xffffffffu) {
    const uint64_t* sk = reinterpret_cast<const uint64_t*>(rs.factor_skip) + (size_t)f * 3;
    const uint32_t L = (uint32_t)sk[0];
    if (L && t0 + L <= len) { resume = sk + 1; s = t0 + L; }
  }
  if (!resume) {
    s = island_start(rs, r, m, len, t0, pre, max_steps);
    if (max_steps != 0xffffffffu && (t0 < len ? t0 : len) - s >= max_steps) return -1;
  }
  return bitprog_test(bp, m, len, s, t0, max_steps, resume);
}

}  // namespace cg
