// tests/native/vm_harness.cpp -- TEST INFRASTRUCTURE ONLY (built into tests/native/_build/, never
// into the product library).  Runs the product's rule compiler, prefilter tables and the *same*
// Pike-VM source (csrc/pike_vm.h, compiled for the host here) on the CPU so that the CPU test tier
// (-m "not gpu") can compare them with the oracle before any GPU time is spent:
//   * compile status / program shape per rule
//   * prefilter soundness: every true (message, rule) hit must be a prefilter candidate (gram filter: gram_filter.h)
//   * exact spans of the VM == oracle/jsre.c spans
// The product path never links this file; libopenclaw_gov.so only runs the VM inside verify_kernel.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../vainplex_openclaw_b200/csrc/pike_vm.h"
#include "../../vainplex_openclaw_b200/csrc/bitprog.h"
#include "../../vainplex_openclaw_b200/csrc/gram_filter.h"
#include "../../vainplex_openclaw_b200/csrc/ruleset_image.h"

using namespace cg;

struct Harness {
  HostImage H;
  DevRuleset d{};
  GramTables T{};
  std::vector<uint2> entries;
};

struct VecSink {
  std::vector<uint32_t>* v;
  void span(uint32_t sb, uint32_t eb, uint32_t s16, uint32_t e16) { v->push_back(sb); v->push_back(eb); v->push_back(s16); v->push_back(e16); }
};

extern "C" {

void* harness_create(const char** srcs, const uint32_t* lens, const uint32_t* flags, uint32_t n, int stride, uint32_t bitmap_kb,
                     uint32_t max_keys, int32_t* status) {
  Harness* h = new Harness();
  std::vector<RuleSrc> src(n);
  for (uint32_t i = 0; i < n; i++) src[i] = RuleSrc{srcs[i], lens[i], flags[i]};
  ImageOptions io; io.stride = stride & 7; io.bloom2 = (stride >> 3) & 1; io.bitmap_kb = bitmap_kb; if (max_keys) io.max_keys = max_keys;
  std::string err;
  if (!build_host_image(src.data(), n, io, &h->H, &err)) { delete h; return nullptr; }
  for (uint32_t i = 0; i < n; i++) if (status) status[i] = h->H.rules[i].status;
  HostImage& H = h->H; DevRuleset& d = h->d;
  // pad host vectors the same way capi.cu pads the device copies
  H.sets.resize(H.sets.size() + 8, 0); H.ranges.resize(H.ranges.size() + 8, 0); H.first.resize(H.first.size() + 8, 0);
  H.factor_words.resize(H.factor_words.size() + 24, 0); H.pf.bytesets.resize(H.pf.bytesets.size() + 8, 0);
  uint32_t n_always = (uint32_t)H.pf.always_rules.size();
  H.pf.always_rules.resize(H.pf.always_rules.size() + 4, 0);
  H.pf.trig_offsets.resize(H.pf.trig_offsets.size() + 4, 0); H.pf.trig_list.resize(H.pf.trig_list.size() + 4, 0);
  for (size_t i = 0; i + 1 < H.entry_words.size(); i += 2) h->entries.push_back(make_uint2(H.entry_words[i], H.entry_words[i + 1]));
  h->entries.resize(h->entries.size() + 2, make_uint2(0, 0));
  d.image = H.image.data(); d.image_bytes = H.bm_bytes; d.stride = (uint32_t)H.pf.stride;
  d.bm_mask = H.bm_mask; d.bloom2 = H.bloom2 ? 1u : 0u; d.rk_off = H.rk_off; d.rk_mask = H.rk_bytes - 4; d.tables_resident = H.tables_resident; d.nb_shift = H.nb_shift;
  d.n_shapes = (uint32_t)H.pf.shapes.size(); for (uint32_t k = 0; k < d.n_shapes && k < 16; k++) d.shapes[k] = H.pf.shapes[k];
  d.n_trig = (uint32_t)H.pf.trig_bytes.size(); for (uint32_t q = 0; q < 2; q++) d.trig_byte[q] = q < d.n_trig ? H.pf.trig_bytes[q] : 0;
  d.trig_offsets = H.pf.trig_offsets.data(); d.trig_list = H.pf.trig_list.data();
  d.bucket_start = H.bucket_start.data(); d.entries = h->entries.data(); d.n_factors = (uint32_t)H.pf.factors.size();
  d.factors = H.factor_words.data(); d.bytesets = H.pf.bytesets.data();
  d.always_rules = H.pf.always_rules.data(); d.n_always = n_always;
  d.prog = H.prog.data(); d.rule_prog_off = H.prog_off.data(); d.sets = H.sets.data(); d.set_ranges = H.ranges.data();
  H.alpha.resize(H.alpha.size() + 8, 0);
  d.rule_first = H.first.data(); d.rule_alpha = H.alpha.data(); d.bit_words = reinterpret_cast<const unsigned long long*>(H.bit_words.data()); d.bit_off = H.bit_off.data(); d.factor_skip = reinterpret_cast<const unsigned long long*>(H.factor_skip.data()); d.n_rules = n; d.rw = (n + 31) / 32; if (!d.rw) d.rw = 1;
  h->T = GramTables{d.bucket_start, d.entries, d.factors, d.bytesets};
  return h;
}
void harness_destroy(void* p) { delete (Harness*)p; }

// info: [0]=bitmap keys [1]=n_factors [2]=stride [3]=factor len min|max<<8 [4]=n_always [5]=image_bytes [6]=program words
//       [7]=level-1b entries [8]=shapes [9]=triggers [10]=bitmap bytes [11]=tables resident
void harness_info(void* p, uint32_t* out) {
  Harness* h = (Harness*)p;
  out[0] = (uint32_t)h->H.pf.keys.size(); out[1] = (uint32_t)h->H.pf.factors.size(); out[2] = (uint32_t)h->H.pf.stride;
  out[3] = h->H.pf.min_factor_len | (h->H.pf.max_factor_len << 8);
  out[4] = h->d.n_always; out[5] = h->d.image_bytes; out[6] = (uint32_t)h->H.prog.size();
  out[7] = (uint32_t)h->H.pf.entries.size(); out[8] = (uint32_t)h->H.pf.shapes.size(); out[9] = (uint32_t)h->H.pf.trig_bytes.size();
  out[10] = h->H.bm_bytes; out[11] = h->H.tables_resident ? 1u : 0u;
}
// bytes of confirm_kernel's table block, laid out as cg_ruleset_create lays it out (capi.cu): recheck map, slots, group
// entries (+16), factor words (+64), byte sets (+32), each part rounded up to 16 bytes.  The kernel stages the block into
// shared memory when it is at most kConfirmTableBudget bytes.
uint32_t harness_confirm_bytes(void* p) {
  const HostImage& H = ((Harness*)p)->H;
  size_t n = 0;
  auto put = [&](size_t bytes, size_t pad) { n = (n + bytes + pad + 15) & ~(size_t)15; };
  put(H.rk_bytes, 0); put(H.slot_words.size() * 4, 0); put(H.group_entries.size() * 4, 16);
  put(H.factor_words.size() * 4, 64); put(H.pf.bytesets.size() * 4, 32);
  return (uint32_t)n;
}
const char* harness_rule_error(void* p, uint32_t rule) { return ((Harness*)p)->H.rules[rule].error.c_str(); }
int harness_rule_nfactors(void* p, uint32_t rule) { return (int)((Harness*)p)->H.rules[rule].factors.size(); }
int harness_rule_exact(void* p, uint32_t rule) { return ((Harness*)p)->H.rules[rule].factors_exact ? 1 : 0; }

// all matches of one rule (global exec loop); out quadruples sb,eb,s16,e16; returns count or -1 on VM overflow
int harness_find_all(void* p, uint32_t rule, const uint8_t* m, uint32_t len, uint32_t* out, uint32_t cap) {
  Harness* h = (Harness*)p;
  VM local(h->d); VM* vm = &local;
  std::vector<uint32_t> v; VecSink sink{&v};
  run_rule<true>(*vm, h->d, rule, m, len, sink);
  if (vm->err) return -1;
  uint32_t k = (uint32_t)(v.size() / 4);
  for (uint32_t i = 0; i < k && i < cap; i++) memcpy(out + 4 * i, v.data() + 4 * i, 16);
  return (int)k;
}
int harness_test(void* p, uint32_t rule, const uint8_t* m, uint32_t len) {
  Harness* h = (Harness*)p;
  VM vm(h->d);
  std::vector<uint32_t> v; VecSink sink{&v};
  bool any = run_rule<false>(vm, h->d, rule, m, len, sink);
  if (vm.err) return -1;
  return any ? 1 : 0;
}

// the scan kernel's candidate logic (gram probes, level-1b lookup, exact factor comparison -- the same CG_HD code),
// restated for one message that sits `lead` bytes into a buffer of arbitrary other bytes (the neighbouring messages
// of a batch; seeded filler here): bitmaps (rw words each) of queued candidates and of direct hits
struct BitSink {
  uint32_t* cand; uint32_t* direct_;
  std::vector<uint32_t>* occ;   // (rule, t0, pre, factor) of confirmed occurrences
  void candidate(uint32_t r, uint32_t t0 = 0xffffffffu, uint32_t pre = 0xffffffffu, uint32_t f = 0xffffffffu) { cand[r >> 5] |= 1u << (r & 31); if (occ) { occ->push_back(r); occ->push_back(t0); occ->push_back(pre); occ->push_back(f); } }
  void direct(uint32_t r) { direct_[r >> 5] |= 1u << (r & 31); }
};
struct OccEmit {
  const DevRuleset& d; BitSink& sink; uint32_t lead; bool want_spans; uint32_t* per_factor;
  void operator()(uint32_t t0, uint32_t f) { if (per_factor) per_factor[f]++; factor_confirmed(d, f, t0 - lead, want_spans, sink); }
};
// returns the number of flagged grams (level 1a)
static uint32_t scan_message(Harness* h, const uint8_t* m, uint32_t len, uint32_t lead, uint32_t seed, bool want_spans, BitSink& sink, uint32_t* per_factor) {
  const DevRuleset& d = h->d;
  std::vector<uint8_t> buf((size_t)lead + len + 48);
  uint32_t x = seed * 2654435761u + 12345u;
  for (auto& b : buf) { x = x * 1664525u + 1013904223u; b = (uint8_t)(x >> 24); }
  memcpy(buf.data() + lead, m, len);
  const uint32_t begin = lead, end = lead + len;
  OccEmit emit{d, sink, lead, want_spans, per_factor};
  uint32_t flagged = 0;
  // occurrences that start less than three bytes into the scanned range have no gram before them (scan_kernel's head check)
  if (lead < 3) for (uint32_t f = 0; f < d.n_factors; f++) for (uint32_t t0 = begin; t0 < begin + 3 && t0 < end; t0++) {
    const uint32_t* fw = d.factors + (size_t)f * 12;
    if (t0 + (fw[1] & 0xffu) <= end && factor_at(fw, d.bytesets, buf.data() + t0)) emit(t0, f);
  }
  for (uint32_t q = 0; q < end; q += d.stride) {
    uint32_t wv; memcpy(&wv, buf.data() + q, 4);
    const uint32_t key = gram_fold_word(wv);
    if (!gram_bitmap_test(d.image, key, d.bm_mask, d.bloom2 != 0)) continue;
    flagged++;
    if (!gram_recheck_test(d.image + d.rk_off, key, d.rk_mask)) continue;
    gram_lookup(d, h->T, key, buf.data(), begin, end, q, emit);
  }
  for (uint32_t ti = 0; ti < d.n_trig; ti++) for (uint32_t q = begin; q < end; q++) if (buf[q] == d.trig_byte[ti]) gram_trigger(d, h->T, ti, buf.data(), begin, end, q, emit);
  return flagged;
}
void harness_candidates(void* p, const uint8_t* m, uint32_t len, uint32_t* cand, uint32_t* direct, int want_spans, uint32_t* l1_hits, uint32_t lead, uint32_t seed) {
  Harness* h = (Harness*)p; const DevRuleset& d = h->d;
  for (uint32_t k = 0; k < d.rw; k++) { cand[k] = 0; direct[k] = 0; }
  BitSink sink{cand, direct, nullptr};
  for (uint32_t k = 0; k < d.n_always; k++) sink.candidate(d.always_rules[k]);
  uint32_t fl = scan_message(h, m, len, lead, seed, want_spans != 0, sink, nullptr);
  if (l1_hits) *l1_hits = fl;
}

static uint64_t g_bit_decided = 0, g_bit_mismatch = 0, g_bit_fallback = 0;
static uint32_t g_vm_rule[8192], g_bit_rule[8192];      // per rule: occurrences left to the VM / decided by the bit-parallel matcher
// policy-mode verification exactly as verify_*_kernel does it: for every confirmed factor occurrence
// run test_at_factor; returns the bitmap of rules that hit (direct hits included)
void harness_policy_hits(void* p, const uint8_t* m, uint32_t len, uint32_t* hits, uint32_t lead, uint32_t seed) {
  Harness* h = (Harness*)p; const DevRuleset& d = h->d;
  std::vector<uint32_t> cand(d.rw, 0), occ;
  for (uint32_t k = 0; k < d.rw; k++) hits[k] = 0;
  BitSink sink{cand.data(), hits, &occ};
  for (uint32_t k = 0; k < d.n_always; k++) sink.candidate(d.always_rules[k]);
  scan_message(h, m, len, lead, seed, false, sink, nullptr);
  VM vm(d);
  struct Null { void span(uint32_t, uint32_t, uint32_t, uint32_t) {} } ns;
  for (size_t k = 0; k + 3 < occ.size(); k += 4) {
    uint32_t r = occ[k], t0 = occ[k + 1], pre = occ[k + 2];
    if ((hits[r >> 5] >> (r & 31)) & 1u) continue;
    bool any = t0 == 0xffffffffu ? run_rule<false>(vm, d, r, m, len, ns) : test_at_factor(vm, d, r, m, len, t0, pre);
    // the bit-parallel matcher (what resolve_kernel runs for eligible rules) must say the same whenever it says anything
    if (t0 != 0xffffffffu && d.bit_off[r] != kBitProgNone) {
      const int res = island_test(d, occ[k + 3], r, m, len, t0, pre, 0xffffffffu);
      if (res >= 0) { g_bit_decided++; g_bit_rule[r & 8191]++; if ((res == 1) != any) g_bit_mismatch++; } else { g_bit_fallback++; g_vm_rule[r & 8191]++; }
    } else g_vm_rule[r & 8191]++;
    if (any) hits[r >> 5] |= 1u << (r & 31);
  }
}
void harness_rule_counts(uint32_t* vm, uint32_t* bit, uint32_t n) { for (uint32_t i = 0; i < n && i < 8192; i++) { vm[i] = g_vm_rule[i]; bit[i] = g_bit_rule[i]; } }
void harness_bitprog_stats(uint64_t* out3) { out3[0] = g_bit_decided; out3[1] = g_bit_mismatch; out3[2] = g_bit_fallback; }
uint32_t harness_bitprog_eligible(void* p) { Harness* h = (Harness*)p; uint32_t k = 0; for (uint32_t r = 0; r < h->d.n_rules; r++) k += h->d.bit_off[r] != kBitProgNone; return k; }

// The whole device pipeline restated over a packed batch exactly as scan_kernel / resolve_kernel / verify see it: head
// check at the start of the scanned range, gram probes over [off[0], off[n]) of the buffer, triggers, message_of() for every
// confirmed occurrence (occurrences straddling two messages dropped), always-candidates, island-restricted VM.
// hits: n x rw words.  The buffer must be readable for 16 bytes past off[n].
void harness_policy_hits_batch(void* p, const uint8_t* buf, const uint32_t* off, uint32_t n, uint32_t* hits) {
  Harness* h = (Harness*)p; const DevRuleset& d = h->d;
  for (size_t k = 0; k < (size_t)n * d.rw; k++) hits[k] = 0;
  if (!n) return;
  const uint32_t begin = off[0], end = off[n];
  std::vector<std::pair<uint32_t, uint32_t>> occ;       // (t0, factor)
  struct Emit { std::vector<std::pair<uint32_t, uint32_t>>* o; void operator()(uint32_t t0, uint32_t f) { o->push_back({t0, f}); } } emit{&occ};
  for (uint32_t f = 0; f < d.n_factors; f++) for (uint32_t t0 = begin; t0 < begin + 3 && t0 < end; t0++) {
    const uint32_t* fw = d.factors + (size_t)f * 12;
    if (t0 + (fw[1] & 0xffu) <= end && factor_at(fw, d.bytesets, buf + t0)) emit(t0, f);
  }
  for (uint32_t q = (begin >> 4) << 4; q < end; q += d.stride) {
    uint32_t wv; memcpy(&wv, buf + q, 4);
    const uint32_t key = gram_fold_word(wv);
    if (gram_bitmap_test(d.image, key, d.bm_mask, d.bloom2 != 0) && gram_recheck_test(d.image + d.rk_off, key, d.rk_mask)) gram_lookup(d, h->T, key, buf, begin, end, q, emit);
  }
  for (uint32_t ti = 0; ti < d.n_trig; ti++) for (uint32_t q = begin; q < end; q++) if (buf[q] == d.trig_byte[ti]) gram_trigger(d, h->T, ti, buf, begin, end, q, emit);
  VM vm(d);
  struct Null { void span(uint32_t, uint32_t, uint32_t, uint32_t) {} } ns;
  std::vector<uint32_t> cand(d.rw);
  for (auto& o : occ) {
    const uint32_t msg = message_of(off, n, o.first);
    if (o.first + (d.factors[(size_t)o.second * 12 + 1] & 0xffu) > off[msg + 1]) continue;
    uint32_t* hm = hits + (size_t)msg * d.rw;
    std::vector<uint32_t> one;
    BitSink sink{cand.data(), hm, &one};
    factor_confirmed(d, o.second, o.first - off[msg], false, sink);
    for (size_t k = 0; k + 3 < one.size(); k += 4) {
      const uint32_t r = one[k];
      if ((hm[r >> 5] >> (r & 31)) & 1u) continue;
      if (test_at_factor(vm, d, r, buf + off[msg], off[msg + 1] - off[msg], one[k + 1], one[k + 2])) hm[r >> 5] |= 1u << (r & 31);
    }
  }
  for (uint32_t msg = 0; msg < n; msg++) for (uint32_t k = 0; k < d.n_always; k++) {
    const uint32_t r = d.always_rules[k]; uint32_t* hm = hits + (size_t)msg * d.rw;
    if ((hm[r >> 5] >> (r & 31)) & 1u) continue;
    if (run_rule<false>(vm, d, r, buf + off[msg], off[msg + 1] - off[msg], ns)) hm[r >> 5] |= 1u << (r & 31);
  }
}

// debug: confirmed occurrences per factor over one message (adds into counts[n_factors]); returns flagged grams
uint32_t harness_l1_factor_counts(void* p, const uint8_t* m, uint32_t len, uint32_t* counts) {
  Harness* h = (Harness*)p; const DevRuleset& d = h->d;
  std::vector<uint32_t> cand(d.rw, 0), dir(d.rw, 0);
  BitSink sink{cand.data(), dir.data(), nullptr};
  return scan_message(h, m, len, 16, 1, false, sink, counts);
}

// flagged grams (level 1a) and confirmed occurrences over a batch of fixed-length messages laid out back to back
void harness_batch_rates(void* p, const uint8_t* data, uint64_t n_msgs, uint32_t msg_len, uint64_t* out2) {
  Harness* h = (Harness*)p; const DevRuleset& d = h->d;
  uint64_t flagged = 0, occ = 0;
  struct Cnt { uint64_t* n; void operator()(uint32_t, uint32_t) { (*n)++; } } emit{&occ};
  const uint64_t total = n_msgs * msg_len;
  for (uint64_t q = 0; q + 4 <= total; q += d.stride) {
    uint32_t wv; memcpy(&wv, data + q, 4);
    const uint32_t key = gram_fold_word(wv);
    if (!gram_bitmap_test(d.image, key, d.bm_mask, d.bloom2 != 0)) continue;
    flagged++;
    if (!gram_recheck_test(d.image + d.rk_off, key, d.rk_mask)) continue;
    gram_lookup(d, h->T, key, data, 0, (uint32_t)total, (uint32_t)q, emit);
  }
  out2[0] = flagged; out2[1] = occ;
}

// debug: print every full factor with its gram positions
void harness_dump_factors(void* p) {
  Harness* h = (Harness*)p; const Prefilter& P = h->H.pf;
  for (size_t f = 0; f < P.factors.size(); f++) {
    const FullFactor& ff = P.factors[f];
    printf("factor %zu rule %u len %d exact %d : ", f, ff.rule, ff.len, ff.exact);
    for (int k = 0; k < ff.len; k++) {
      int cnt = 0, last = -1; for (int b = 0; b < 256; b++) if ((P.bytesets[(size_t)ff.elem[k] * 8 + (b >> 5)] >> (b & 31)) & 1) { cnt++; last = b; }
      if (cnt == 1) { if (last >= 33 && last < 127) printf("%c", last); else printf("\\x%02x", last); } else printf("[%d]", cnt);
    }
    printf("  grams:");
    for (auto& e : P.entries) if (e.factor == f) printf(" off %d mask %08x", e.off, e.mask);
    printf("\n");
  }
  printf("stride %d keys %zu entries %zu shapes %zu triggers %zu always %zu bitmap %u B resident %d\n", P.stride, P.keys.size(), P.entries.size(), P.shapes.size(),
         P.trig_bytes.size(), P.always_rules.size(), h->H.bm_bytes, (int)h->H.tables_resident);
}

}  // extern "C"

// VM work statistics per rule over a batch (built with -DCG_VM_STATS only): for every confirmed occurrence that reaches
// the VM, accumulate the counters of pike_vm.h into out[rule * 8 + i], i = 0..4; out[rule * 8 + 5] = events, [6] = island start distance
#ifdef CG_VM_STATS
extern "C" unsigned long long cg_vm_stats[8] = {0, 0, 0, 0, 0, 0, 0, 0};
extern "C" void harness_vm_stats(void* p, const uint8_t* data, uint64_t n_msgs, uint32_t msg_len, unsigned long long* out) {
  Harness* h = (Harness*)p; const DevRuleset& d = h->d;
  VM vm(d);
  for (uint64_t mi = 0; mi < n_msgs; mi++) {
    const uint8_t* m = data + mi * msg_len; uint32_t len = msg_len;
    std::vector<uint32_t> cand(d.rw, 0), hits(d.rw, 0), occ;
    BitSink sink{cand.data(), hits.data(), &occ};
    scan_message(h, m, len, 16, 1, false, sink, nullptr);
    for (size_t k = 0; k + 3 < occ.size(); k += 4) {
      uint32_t r = occ[k], t0 = occ[k + 1], pre = occ[k + 2];
      if ((hits[r >> 5] >> (r & 31)) & 1u) continue;
      if (t0 == 0xffffffffu) continue;
      for (int i = 0; i < 8; i++) cg_vm_stats[i] = 0;
      bool any = test_at_factor(vm, d, r, m, len, t0, pre);
      if (any) hits[r >> 5] |= 1u << (r & 31);
      for (int i = 0; i < 5; i++) out[(size_t)r * 8 + i] += cg_vm_stats[i];
      out[(size_t)r * 8 + 5]++;
      out[(size_t)r * 8 + 6] += (pre & 0xffffu);
    }
  }
}
#endif
