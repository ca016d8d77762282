// kernels.h -- device-side structures and launchers shared by capi.cu and the .cu kernel files.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace cg {

// Everything the scan / verify kernels need to know about a compiled rule set (device pointers).
struct DevRuleset {
  // gram filter (rulec.h): the image is staged into shared memory by the scan kernel with TMA bulk copies.
  //   [0, bm_mask + 4)  bitmap ; [rk_off] recheck map ; then, when tables_resident: [dir_off] bucket_start (n_buckets + 1 words)
  //   [ent_off] level-1b entries (8 B each).  All offsets 16-byte aligned.  Factor words and byte sets stay in HBM.
  const uint8_t* image;
  uint32_t image_bytes;          // bytes scan_kernel stages: the bitmap (the rest of the image is read in place by confirm_kernel)
  uint32_t stride;               // 4: one probe per aligned word, 2: also the gram at byte offset 2 of every word
  uint32_t bm_mask, bloom2;      // bitmap word address = hi32(key * kGramMult) & bm_mask; bloom2: keys set / need two bits of the word
  uint32_t rk_off, rk_mask;      // recheck map (gram_filter.h): image offset, bytes - 4; always part of the image
  uint32_t tables_resident;      // level-1b tables are part of the image (else read through the HBM pointers below)
  uint32_t dir_off, ent_off;
  uint32_t nb_shift;             // bucket = hash >> nb_shift
  uint32_t n_shapes, shapes[16]; // distinct key masks of the level-1b entries
  uint32_t n_trig, trig_byte[2]; // single-byte triggers
  uint32_t hot_c5f, hot_c10, hot_one;   // 0x5f5f5f5f, 0x10101010, 1: run-time constants of the scan kernel's hot loop (scan_kernels.cu)
  const uint32_t* trig_offsets;  // CSR over triggers -> trig_list (factor | element index << 20)
  const uint32_t* trig_list;
  const uint32_t* bucket_start;  // HBM copies of the level-1b tables
  const uint2* entries;
  const uint4* slots;            // confirm_kernel's view of the same entries (ruleset_image.h): open-addressing table of groups
  const uint32_t* group_entries; // entry words (factor | (gram offset + 3) << 20 | shape << 25) in group order
  uint32_t slot_shift, slot_mask;
  // confirm_kernel's tables as one block ([recheck map][slots][group entries][factor words][byte sets], 16-byte aligned parts):
  // staged into shared memory when cf_resident (they fit beside the position rings), read in place otherwise
  const uint8_t* cf_image; uint32_t cf_bytes, cf_resident, cf_slots_off, cf_ge_off, cf_fac_off, cf_bs_off;
  uint32_t n_factors;
  uint32_t max_prog_len;         // longest Pike program of the set (picks the VM capacity)
  uint32_t debug_flags;          // CG_SCAN_DEBUG (experiments only): bit 0 = drop flagged grams (results wrong),
                                 //   bit 1 = histogram of VM cycles per event in counters[7..15]
  const uint32_t* factors;       // 12 words per full factor: rule, len | exact<<24, 16 x u16 set ids, max prefix units, prefix-alphabet set id
  const uint32_t* bytesets;      // 8 words per 256-bit byte set
  const uint32_t* always_rules;  // candidates for every message
  uint32_t n_always;
  const uint32_t* prog;          // all Pike programs, concatenated
  const uint32_t* rule_prog_off; // n_rules + 1
  const uint32_t* sets;          // 6 words per unit set: ascii[4], range_off, n_ranges
  const uint16_t* set_ranges;    // inclusive lo,hi pairs
  const unsigned long long* bit_words; const uint32_t* bit_off;   // bitprog.h: 139 + 64 x rows words per eligible rule, bit_off[rule] = first word or 0xffffffff
  const unsigned long long* factor_skip;   // 3 words per factor: elements the island matcher may skip | its state behind them (bitprog.h: island_test); nullptr = none
  const uint32_t* rule_first;    // 8 words per rule: first-byte bitmap
  const uint32_t* rule_alpha;    // 8 words per rule: alphabet bitmap (bytes a match can contain)
  // verdict aggregation (policy-evaluator.ts:44-146, messageContains slice): per rule its policy (index in priority order,
  // non-decreasing with the rule index) and its effect (0 allow, 1 audit, 2 deny); nullptr until cg_ruleset_set_policy
  const uint32_t* rule_policy; const uint32_t* rule_action;
  uint32_t n_rules;
  uint32_t rw;                   // bitmap words per slot = ceil(n_rules / 32)
};

// Per-call scratch in HBM.  A "slot" is one message with at least one confirmed candidate.
struct ScanWork {
  uint32_t* counters;            // 32 words: [0]=n_slots [1]=n_events [2]=n_spans [3]=error flags [4]=n_l1 (confirmed factor occurrences) [5]=verify cursor
                                 //           [6]=flagged grams (level 1a) [7..15]=debug [17]=n_heavy [18]=verify cursor (light events) [19]=grams past the recheck map
                                 //           [24..27]=flag words queued, [28..31]=(gram, entry) pairs compared, per piece of the batch
                                 //           span resolution: [16]=status (kResolve*) [20]=resolved spans [21]=digests to compute [22]=messages to splice
  uint32_t* l1_pos;              // [l1_cap] factor occurrences scan_kernel confirms itself (head check, trigger bytes): buffer offset of the
  uint32_t* l1_fac;              //          factor's first byte, factor id
  uint2* fq;                     // [l1_cap] scan_kernel's flag words: x = the lane's chunk number after the round, y = 4 tiles x 8 (4) probe bits
  uint32_t* persist;             // [4] survives the per-step reset: [0] = slots the previous step used (their candidate / hit rows are zeroed by the next step's reset_kernel)
  uint32_t* slot_of_msg;         // [n] 0xffffffff = none yet (reset per step)
  uint32_t* slot_msg;            // [slot_cap]
  uint32_t* cand;                // [slot_cap * rw]  candidate (msg,rule) pairs already queued
  uint32_t* hit;                 // [slot_cap * rw]  verified pairs
  uint2* events;                 // [event_cap]  (slot, rule | heavy << 31) for the Pike VM
  uint32_t* heavy_idx;           // [event_cap]  indices of the events expected to run long (counters[17] of them): verified first
  uint32_t* event_pos;           // [event_cap]  policy mode: message offset of the confirmed factor's first byte
  uint32_t* event_pre;           // [event_cap]  policy mode: max units of a match before that factor (0xffff = unbounded)
  uint32_t* spans;               // [span_cap * 6] msg, rule, start_byte, end_byte, start16, end16
  uint32_t l1_cap, msg_cap, slot_cap, event_cap, span_cap;
  uint32_t q_cap, q_slot;        // this launch's piece of fq (a step scans the batch in up to 4 pieces: q_slot 0..3) and its counter [24 + q_slot]
  // span resolution (span-mode steps only): [res_cap + 1] per message, [span_cap] per raw span
  uint64_t* words;               // [res_cap] result words of span-mode steps
  uint32_t* seg_cnt;             // raw spans per message (counted down again by the scatter)
  uint32_t* seg_begin;           // exclusive scan of seg_cnt: the message's segment of `sorted`
  uint32_t* kept_cnt;            // spans resolveOverlaps keeps per message
  uint32_t* kept_begin;          // exclusive scan of kept_cnt: the message's first resolved span
  uint64_t* out_len;             // redacted bytes per message
  uint64_t* out_off;             // exclusive scan of out_len
  uint4* sorted;                 // [span_cap] (start16, ~length16, rule rank, raw span index) in message order; kept keys first
  uint4* sort_tmp;               // [span_cap] merge passes of long segments
  uint32_t* sp_start;            // [span_cap] per resolved span: buffer offset of its first byte, byte length, category
  uint32_t* sp_len;              //            (redact_splice_kernel's input)
  uint32_t* sp_cat;
  uint64_t* scan_part;           // [kScanPartials] partial sums of the exclusive scans
  uint32_t res_cap;
  // per rule its category (CG_CAT_*) and its rank in (category, rule) order, uploaded with the rule set.  (Kept here, not in
  // DevRuleset: every scan kernel takes DevRuleset by value, and a larger one changes their code.)
  const uint32_t* rule_category; const uint32_t* rule_rank;
};

enum : uint32_t { ERR_EVENT_OVERFLOW = 1, ERR_SPAN_OVERFLOW = 2, ERR_VM_STACK = 4, ERR_VM_LIST = 8, ERR_SLOT_OVERFLOW = 16, ERR_L1_OVERFLOW = 32 };
// span resolution status (counters[16]); kept out of the error flags, which mean "a queue overflowed"
enum : uint32_t { kResolveOk = 0, kResolveCapacity = 1, kResolveTooLarge = 2 };
constexpr uint32_t kCounterWords = 32;
constexpr uint32_t kScanPartials = 1024;         // blocks an exclusive scan uses at most
constexpr uint32_t kConfirmTableBudget = 176u * 1024u;     // shared memory confirm_kernel may spend on its tables (beside 32 KB of rings)
constexpr uint64_t kWordIncomplete = ~0ull;      // result word of every message of a batch whose queues overflowed / whose VM failed

// launchers (all asynchronous on `stream`); return the number of kernels launched.
// scan: level 1 of the whole buffer range [off[0], off[n]); queues confirmed factor occurrences and zeroes d_words.
// d_bytes must be 16-byte aligned and readable up to 16 bytes past off[n].
int launch_scan(const DevRuleset& rs, const ScanWork& w, const uint8_t* d_bytes, const uint32_t* d_off, uint32_t n,
                uint64_t* d_words, int sm_count, cudaStream_t stream);
// per piece of the batch: flag words -> grams -> recheck map -> table probes -> exact factors (confirm_kernel)
int launch_confirm(const DevRuleset& rs, const ScanWork& w, const uint8_t* d_bytes, const uint32_t* d_off, uint32_t n, int sm_count, cudaStream_t stream);
// once per step: message, slot, candidates for the VM / direct hits / island matcher
int launch_resolve(const DevRuleset& rs, const ScanWork& w, const uint8_t* d_bytes, const uint32_t* d_off, uint32_t n, bool want_spans, int sm_count, cudaStream_t stream);
// ctas_per_sm (1 .. 4): events are handed out by an atomic cursor, so any grid is correct; an empty launch costs more at four
// CTAs per SM than at one, so the caller sizes the grid by what the previous steps sent to the VM
int launch_verify(const DevRuleset& rs, const ScanWork& w, const uint8_t* d_bytes, const uint32_t* d_off,
                  bool want_spans, int sm_count, cudaStream_t stream, int ctas_per_sm = 4);
// one verdict word per hit message: action | matched policies << 2 | deciding rule << 12 (cg_policy_verdict_batch)
int launch_verdicts(const DevRuleset& rs, const ScanWork& w, uint32_t* d_verdicts, int sm_count, cudaStream_t stream);
int launch_finalize(const DevRuleset& rs, const ScanWork& w, uint64_t* d_words, uint32_t n, int sm_count, cudaStream_t stream);
// start of a step: counters = 0, slot_of_msg = none, candidate / hit rows of the slots the previous step used = 0
int launch_reset(const DevRuleset& rs, const ScanWork& w, uint32_t n, int sm_count, cudaStream_t stream);

// single-message path: result word, counters and the message's hit row packed into one block (one D2H copy)
int launch_pack_one(const DevRuleset& rs, const ScanWork& w, const uint64_t* d_word, uint32_t* d_out, uint32_t rw_cap, cudaStream_t stream);

// raises the dynamic shared-memory limits of every kernel once (not legal inside stream capture)
void prepare_scan_kernels();

// exclusive prefix sums: out[i] = in[0] + ... + in[i - 1] for i < count (count >= 1; d_part: kScanPartials elements)
int launch_exclusive_scan(const uint32_t* d_in, uint32_t* d_out, uint32_t count, uint64_t* d_part, int sm_count, cudaStream_t stream);
int launch_exclusive_scan(const uint64_t* d_in, uint64_t* d_out, uint32_t count, uint64_t* d_part, int sm_count, cudaStream_t stream);
// where resolved spans go (device pointers).  spans: 6 words per span, the first spans_cap written; redact: out_offsets[n+1],
// and sizes = u64[2] {output bytes needed, resolved spans}, else sizes = u32[1] resolved spans; sizes are ~0 when the step
// is incomplete (a queue overflowed or the VM failed).  The status goes to counters[16]: kResolveTooLarge (redact, 4 GiB or
// more), kResolveCapacity (more spans than spans_cap, or more bytes than out_cap).
struct SpanOutputs {
  uint32_t* spans; uint32_t spans_cap;
  uint32_t* out_offsets; uint64_t out_cap;
  void* sizes;
  bool redact;
};
// resolveOverlaps of a span-mode step over n messages (d_off as scanned): a fixed number of kernels for given n and mode,
// whatever the span count.  Redact also leaves the splice's input in w.sp_* / w.kept_begin and sets counters[21] / [22] to the
// spans to digest / messages to splice (0 unless every output fits).
int launch_span_resolve(const ScanWork& w, const uint32_t* d_off, uint32_t n, const SpanOutputs& o, int sm_count, cudaStream_t stream);

// SHA-256 / Merkle
int launch_sha256_batch(const uint8_t* d_bytes, const uint64_t* d_off, uint32_t n, uint8_t* d_out, cudaStream_t stream);
// Merkle log: acc = node(left[k], acc) chains; audit-path verification
int launch_merkle_chain(const uint32_t* d_left, uint32_t n_left, const uint32_t* d_acc_in, uint32_t* d_acc_out, cudaStream_t stream);
int launch_merkle_verify(const uint32_t* d_leaf32, uint64_t index, uint64_t size, const uint32_t* d_path, uint32_t path_len, const uint32_t* d_root32, uint32_t* d_ok, cudaStream_t stream);
// redacted output: SHA-256 of every span, then copy + placeholder splice (one warp per message).  Both read their item
// count from device memory (*d_ns spans, *d_n <= n_max messages), so that the resolver decides on the device whether they run.
// d_out digests: 16-byte aligned.
int launch_redact_digests(const uint8_t* d_bytes, const uint32_t* d_start, const uint32_t* d_len, const uint32_t* d_ns, uint32_t* d_out,
                          int sm_count, cudaStream_t stream);
int launch_redact_splice(const uint8_t* d_bytes, const uint32_t* d_off, const uint32_t* d_out_off, const uint32_t* d_span_begin,
                         const uint32_t* d_span_start, const uint32_t* d_span_len, const uint32_t* d_span_cat, const uint32_t* d_digests,
                         uint8_t* d_out, const uint32_t* d_n, uint32_t n_max, int sm_count, cudaStream_t stream);
// leaf digests of fixed-size leaves: out[i] = SHA-256(0x00 || leaf_i)
int launch_merkle_leaves_fixed(const uint8_t* d_bytes, uint64_t leaf_len, uint64_t n, uint32_t* d_out, cudaStream_t stream);
// ragged leaves, word-granular: d_bytes must be one of the library's own buffers (readable 4 bytes before the first leaf and
// 8 bytes after the last); trim_newline: a final '\n' of a leaf's range is not hashed (JSONL lines)
int launch_merkle_leaves_var(const uint8_t* d_bytes, const uint64_t* d_off, uint64_t n, uint32_t* d_out, cudaStream_t stream, bool trim_newline = false);
// JSONL on the device: newline counts per 4 KB piece + their exclusive scan (d_piece_counts, *d_total_lines), then the line starts
int launch_newline_split(const uint8_t* d_bytes, uint64_t len, uint32_t* d_piece_counts, uint64_t* d_total_lines, cudaStream_t stream);
int launch_newline_starts(const uint8_t* d_bytes, uint64_t len, const uint32_t* d_piece_rank, uint64_t* d_starts, uint64_t n_lines, cudaStream_t stream);
int launch_merkle_consistency(uint64_t first, uint64_t second, const uint32_t* d_first32, const uint32_t* d_second32, const uint32_t* d_path, uint32_t path_len, uint32_t* d_ok, cudaStream_t stream);
// fold the n nodes at d_in (16-byte aligned) level by level until one is left or max_levels levels are done; the first level
// writes d_a, later ones d_b, d_a, ...; only the first reads d_in (d_b may be d_in).  *d_result = the folded nodes.
int launch_merkle_fold(const uint32_t* d_in, uint64_t n, uint32_t max_levels, uint32_t* d_a, uint32_t* d_b, cudaStream_t stream,
                       const uint32_t** d_result);

}  // namespace cg
