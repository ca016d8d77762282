/*
 * openclaw_gov.h -- C ABI of the H100-native openclaw-governance hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b): plain pointers and sizes, no C++ or
 * torch types, no exceptions, no library-owned memory handed to the caller.  The Node N-API
 * shim (napi/openclaw_gov_napi.c) and the Python ctypes binding (vainplex_openclaw_b200/
 * _native.py) bind exactly these symbols.  Each entry point names the reference interface
 * it replaces; paths are relative to packages/openclaw-governance/ of the reference.
 *
 * Error model (replaces JS exceptions caught by the failMode blocks, src/hooks.ts:232-241,
 * src/redaction/hooks.ts:193-204): every function returns CG_OK (0) or a negative code and
 * cg_last_error() holds a thread-local message.  There is NO CPU fallback: without a usable
 * CUDA device every compute call fails with CG_ERR_CUDA / CG_ERR_NOT_INITIALIZED.
 *
 * Text encoding: message bytes are UTF-8 as produced by Buffer.from(str,'utf8') (lone
 * surrogates already replaced by U+FFFD).  All span offsets are reported both in bytes and in
 * UTF-16 code units, the unit the reference's m.index / lastIndex use (registry.ts:226-231).
 */
#ifndef OPENCLAW_GOV_H
#define OPENCLAW_GOV_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CG_API __attribute__((visibility("default")))

/* ---- status codes */
#define CG_OK                   0
#define CG_ERR_INVALID_ARG     -1
#define CG_ERR_NOT_INITIALIZED -2
#define CG_ERR_CUDA            -3   /* no device / kernel or copy failed: caller applies failMode */
#define CG_ERR_SYNTAX          -4   /* `new RegExp(src)` would throw SyntaxError */
#define CG_ERR_UNSUPPORTED     -5   /* valid JS regex outside the supported subset (DESIGN.md) */
#define CG_ERR_TOO_LARGE       -6   /* rule expands past the matcher program limit */
#define CG_ERR_CAPACITY        -7   /* caller's output array too small; *out_count holds the need */
#define CG_ERR_NOMEM           -8

/* ---- rule flags / categories */
#define CG_FLAG_ICASE 1u            /* RegExp flag "i" (registry.ts:112,223) */
/* CATEGORY_ORDER of src/redaction/registry.ts:17-22 */
#define CG_CAT_CREDENTIAL 0u
#define CG_CAT_FINANCIAL  1u
#define CG_CAT_PII        2u
#define CG_CAT_CUSTOM     3u

/* ---- ruleset options: stride of the gram filter (DESIGN.md section 4) */
#define CG_OPT_STRIDE_AUTO 0u /* 4 when every factor of the set can be covered at four alignments, else 2 (default) */
#define CG_OPT_STRIDE2     2u /* probe the gram at every even byte offset */
#define CG_OPT_STRIDE4     4u /* probe every aligned 4-byte word only (rule sets of long literals) */

typedef struct cg_ruleset cg_ruleset;

typedef struct cg_rule {
  const char *source;      /* JS RegExp source, UTF-8, not NUL-terminated */
  uint32_t source_len;
  uint32_t flags;          /* CG_FLAG_* */
  uint32_t category;       /* CG_CAT_* ; only used by cg_find_matches_* ordering */
} cg_rule;

typedef struct cg_hit {     /* one (message, rule) with RegExp.test(message) === true */
  uint32_t msg;
  uint32_t rule;
} cg_hit;

typedef struct cg_span {    /* one element of PatternRegistry.findMatches()'s result */
  uint32_t msg;
  uint32_t rule;
  uint32_t start_byte, end_byte;   /* offsets into the message's UTF-8 bytes */
  uint32_t start16, end16;         /* same span in UTF-16 code units (JS indices) */
} cg_span;

typedef struct cg_ruleset_info {
  uint32_t n_rules, n_ok, n_always_candidate, n_sets;
  uint32_t stride, gram_keys, gram_entries, factor_len /* min | max<<8 */, image_bytes /* staged into shared memory per CTA */;
  uint32_t program_words, n_factors, bitmap_bytes, n_triggers, tables_resident;
} cg_ruleset_info;

typedef struct cg_stats {   /* cumulative since cg_init; surfaced by governance.status (index.ts:103-114) */
  uint64_t messages_scanned, bytes_scanned, candidate_events, verified_pairs, hits, spans;
  uint64_t sha256_items, merkle_leaves, kernel_launches;
  double last_scan_ms, last_merkle_ms;   /* device time of the last call (CUDA events) */
} cg_stats;

/* ---- lifecycle.  Replaces nothing in the reference (it has no device); called from the
 * plugin's register()/gateway_stop (index.ts:66-118).  device < 0 selects the current device. */
CG_API int cg_init(int device);
CG_API void cg_shutdown(void);
CG_API const char *cg_last_error(void);
CG_API int cg_version(void);
CG_API int cg_device_count(void);
CG_API int cg_get_stats(cg_stats *out);
CG_API uint64_t cg_launch_count(void);   /* kernels launched by this library so far */
/* measurement hooks (the reference's ScanResult.elapsedMs / evaluationUs, src/redaction/engine.ts:54,65):
 * with profiling on, CUDA events bracket each kernel of a scan step on its stream. */
CG_API int cg_set_profiling(int on);
CG_API int cg_last_tail_ms(float out_ms[2]);            /* confirm_kernel, resolve_kernel of that step (profiling mode) */
CG_API int cg_last_kernel_ms(float out_ms[4]);          /* scan, resolve, verify, finalize of the last completed step */
CG_API int cg_scan_work_counters(const cg_ruleset *rs, uint32_t out16[16]); /* slots, VM pairs, spans, flags, confirmed factor occurrences, (internal), flagged grams, reserved */

/* ---- rule-set compile.  Replaces `new RegExp(pattern)` in buildPolicyIndex
 * (src/policy-loader.ts:119-128), compileCustomPattern (src/redaction/registry.ts:249-281) and
 * the per-call `new RegExp(source,"g"+i)` of findMatches (registry.ts:222-223).
 * status_per_rule (may be NULL) receives CG_OK / CG_ERR_SYNTAX / CG_ERR_UNSUPPORTED /
 * CG_ERR_TOO_LARGE per rule; rules that failed never match.  With status_per_rule == NULL the
 * first failing rule fails the whole call. */
CG_API int cg_ruleset_create(const cg_rule *rules, uint32_t n_rules, uint32_t options,
                             cg_ruleset **out, int32_t *status_per_rule);
CG_API void cg_ruleset_destroy(cg_ruleset *rs);
CG_API int cg_ruleset_get_info(const cg_ruleset *rs, cg_ruleset_info *out);
/* one rule, no device needed: what would `new RegExp(src, flags)` do?  (validateRegex,
 * src/policy-loader.ts:15-31).  err/err_len may be NULL/0. */
CG_API int cg_rule_check(const char *source, uint32_t source_len, uint32_t flags, char *err, uint32_t err_len);

/* ---- policy-semantics scan: RegExp.test per (message, rule) -- matchesAny,
 * src/conditions/context.ts:9-25, over a batch.  Host buffers; copies are inside the call.
 *   bytes/offsets : n messages, message i = bytes[offsets[i] .. offsets[i+1])
 *   out_words[n]  : hit ? 1<<63 | (#distinct rules hit)<<32 | lowest hit rule index : 0
 *   out_hits      : optional sparse list sorted by (msg, rule); hits_cap entries available;
 *                   *out_nhits = number of hits (CG_ERR_CAPACITY when it exceeds hits_cap). */
CG_API int cg_scan_batch(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, uint32_t n,
                         uint64_t *out_words, cg_hit *out_hits, uint32_t hits_cap, uint32_t *out_nhits);
/* single message, blocking: the path for the synchronous hooks before_message_write /
 * tool_result_persist (src/hooks.ts:297-389).  out_rules receives the hit rule indices. */
CG_API int cg_scan_one(cg_ruleset *rs, const uint8_t *bytes, uint32_t len, uint64_t *out_word,
                       uint32_t *out_rules, uint32_t rules_cap, uint32_t *out_nrules);

/* ---- redaction-semantics scan: PatternRegistry.findMatches (registry.ts:212-242) including
 * resolveOverlaps (registry.ts:288-316) for every message of a batch.  Spans come back sorted
 * by (msg, start); `rule` is the index passed to cg_ruleset_create. */
CG_API int cg_find_matches_batch(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, uint32_t n,
                                 cg_span *out_spans, uint32_t spans_cap, uint32_t *out_nspans);

/* ---- verdicts instead of hit bits (SURVEY.md section 8 f3): aggregateMatches / matchPolicy of src/policy-evaluator.ts:44-146
 * for rule sets whose rules are the messageContains patterns of a policy list.  rule_policy[i] = index of rule i's policy
 * in evaluation order (priority descending; rules stored policy by policy), rule_action[i] = 0 allow / 1 audit / 2 deny.
 * Per message: per policy the first matching rule counts; deny beats audit beats allow; the first policy that produced the
 * winning action is reported.  out_verdicts[i] = action | (matched policies, saturating at 1023) << 2 | deciding rule << 12
 * (deciding rule = 0xfffff when no deny / audit rule matched; 0 = no policy matched: allow). */
CG_API int cg_ruleset_set_policy(cg_ruleset *rs, const uint32_t *rule_policy, const uint8_t *rule_action, uint32_t n_rules);
CG_API int cg_policy_verdict_batch(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, uint32_t n, uint32_t *out_verdicts);

/* ---- redacted output of a batch: RedactionEngine.scanString (src/redaction/engine.ts:74-85) = findMatches +
 * applyReplacements (engine.ts:165-181), every match replaced by the vault's default placeholder
 * "[REDACTED:<category>:<first 8 hex digits of SHA-256(match)>]" (src/redaction/vault.ts:33-35,75-104).
 *   out_bytes / out_offsets[n+1] : redacted messages, same packing as the input; *out_need = bytes needed
 *   out_spans / out_digests32    : the resolved spans (as cg_find_matches_batch) and SHA-256 of each matched text, so that
 *                                  the caller's vault can store the originals and detect the 2^-32 case in which two live
 *                                  values share hash8 and vault.store switches to the 12-digit form (vault.ts:85-104).
 * CG_ERR_CAPACITY when out_cap / spans_cap are too small (sizes in *out_need / *out_nspans). */
CG_API int cg_redact_batch(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, uint32_t n,
                           uint8_t *out_bytes, uint64_t out_cap, uint64_t *out_need, uint32_t *out_offsets,
                           cg_span *out_spans, uint32_t spans_cap, uint32_t *out_nspans, uint8_t *out_digests32);

/* ---- device-resident variant (inputs/outputs already in HBM; used by bench.py `value` and by callers that pipeline
 * their own copies).  Pointers are CUDA device pointers; `stream` is a cudaStream_t (NULL = the library's own stream);
 * asynchronous w.r.t. the host, strictly in order on `stream`.
 * d_bytes must be 16-byte aligned and readable for 16 bytes past offsets[n] (padding; any content).
 * Queue capacities: a batch that overflows an internal queue (far more candidates than usual) cannot be re-run by the
 * library (the call has long returned).  Instead EVERY result word of that batch is set to 0xffffffffffffffff
 * ("incomplete") by the device, the scratch is grown before the next call runs, and cg_scan_join reports
 * CG_ERR_CAPACITY once: scan that batch again.  (cg_scan_batch, the host-buffer call, retries by itself.) */
CG_API int cg_scan_batch_device(cg_ruleset *rs, const void *d_bytes, const void *d_offsets, uint32_t n,
                                void *d_out_words, void *stream);
/* findMatches + resolveOverlaps for a batch in HBM.  Same input rules as cg_scan_batch_device (d_bytes 16-byte aligned,
 * readable 16 bytes past offsets[n]).  d_out_spans: cg_span[spans_cap] (may be NULL when spans_cap is 0); d_out_nspans: one
 * uint32 = resolved spans of the batch.  Asynchronous and in order on `stream` like cg_scan_batch_device; its status comes
 * from cg_scan_join: CG_ERR_CAPACITY when the batch has more than spans_cap spans (the first spans_cap are written), or when
 * an internal queue overflowed (then *d_out_nspans = 0xffffffff, nothing is written, the scratch grows: issue it again). */
CG_API int cg_find_matches_batch_device(cg_ruleset *rs, const void *d_bytes, const void *d_offsets, uint32_t n,
                                        void *d_out_spans, uint32_t spans_cap, void *d_out_nspans, void *stream);
/* RedactionEngine.scanString for a batch in HBM (cg_redact_batch's packing and placeholder).  d_out_bytes: out_cap bytes;
 * d_out_offsets: uint32[n+1]; d_out_spans: cg_span[spans_cap]; d_out_digests32: 32 bytes per span, 16-byte aligned;
 * d_out_sizes: uint64[2] = {output bytes needed, resolved spans}, 8-byte aligned.  Sizes and offsets are always written;
 * spans, digests and output bytes only while they fit (no byte past out_cap or spans_cap is ever written).  cg_scan_join
 * reports CG_ERR_CAPACITY when they did not (issue again with the sizes), CG_ERR_TOO_LARGE for 4 GiB of output or more, and
 * CG_ERR_CAPACITY once after an internal queue overflow (both sizes = ~0, nothing else written; issue the batch again). */
CG_API int cg_redact_batch_device(cg_ruleset *rs, const void *d_bytes, const void *d_offsets, uint32_t n,
                                  void *d_out_bytes, uint64_t out_cap, void *d_out_offsets,
                                  void *d_out_spans, uint32_t spans_cap, void *d_out_digests32, void *d_out_sizes, void *stream);
/* Waits for `stream` and returns the status of every device-path batch (scan, find-matches, redact) issued since the
 * previous join: CG_OK, CG_ERR_CAPACITY (see above) or CG_ERR_TOO_LARGE (the VM ran out of thread-list space; words all
 * ones as well; or a redacted batch of 4 GiB or more). */
CG_API int cg_scan_join(cg_ruleset *rs, void *stream);

/* ---- SHA-256.  Replaces createHash("sha256").update(s).digest() at src/util.ts:77-79,
 * src/redaction/vault.ts:26-28 (and nats/src/hooks.ts:90-94) for a batch of n byte strings. */
CG_API int cg_sha256_batch(const uint8_t *bytes, const uint64_t *offsets, uint32_t n, uint8_t *out_digests32);

/* ---- Proof-of-Guardrails Merkle tree over event-log leaves (audit JSONL lines,
 * src/audit-trail.ts:151-179; no implementation in the reference -- convention in DESIGN.md:
 * leaf = SHA-256(0x00||bytes), node = SHA-256(0x01||L||R), unpaired node promoted, empty =
 * SHA-256("")). */
CG_API int cg_merkle_root(const uint8_t *bytes, const uint64_t *offsets, uint64_t n, uint8_t out_root[32]);
CG_API int cg_merkle_root_fixed(const uint8_t *bytes, uint64_t leaf_len, uint64_t n, uint8_t out_root[32]);
/* device-resident: fixed-size leaves in HBM -> roots of consecutive 2^block_log2-leaf blocks
 * (d_out_roots[ceil(n / 2^block_log2)][32], device memory).  Shards call this, all-gather the
 * block roots (the one collective on this path) and finish with cg_merkle_fold.
 * block_log2 must be at most 40 (as for cg_merkle_root_sharded_device): larger values return
 * CG_ERR_INVALID_ARG before any buffer is touched. */
CG_API int cg_merkle_block_roots_device(const void *d_bytes, uint64_t leaf_len, uint64_t n, uint32_t block_log2,
                                        void *d_out_roots, void *stream);
/* fold m 32-byte subtree roots (host memory) into one root with the same level-wise rule */
CG_API int cg_merkle_fold(const uint8_t *nodes32, uint64_t m, uint8_t out_root[32]);

/* ---- multi-GPU, one process per GPU (SURVEY.md section 8 e).  The scan shards by message and exchanges nothing:
 * cg_shard_range is the split rule (contiguous [lo, hi) per rank, every boundary except n a multiple of `align`).  The
 * Merkle tree exchanges once: cg_merkle_root_sharded_device reduces this rank's leaves to roots of aligned 2^block_log2-leaf
 * blocks, all-gathers them (NCCL, bound at run time with dlopen: a single-GPU process needs no NCCL) and folds the same list
 * on every rank -- the root of the single tree over all ranks' leaves.  Bootstrap: rank 0 calls cg_comm_unique_id and hands
 * the 128 bytes to the other ranks by whatever channel launched them; every rank calls cg_comm_init(rank, world, id). */
typedef struct { char internal[128]; } cg_nccl_id;
CG_API void cg_shard_range(uint64_t n, int rank, int world, uint64_t align, uint64_t *lo, uint64_t *hi);
CG_API int cg_comm_unique_id(cg_nccl_id *out);
CG_API int cg_comm_init(int rank, int world, const cg_nccl_id *id);
CG_API void cg_comm_destroy(void);
CG_API int cg_merkle_root_sharded_device(const void *d_bytes, uint64_t leaf_len, uint64_t n_local, uint64_t n_total, uint32_t block_log2,
                                         uint8_t out_root[32], void *stream);
CG_API int cg_merkle_fold_device(const void *d_nodes32, uint64_t m, void *d_out_root32, void *stream);

/* ---- append-only Merkle log over the event log (SURVEY.md section 8 f2; audit JSONL lines of src/audit-trail.ts:151-179
 * as leaves, same convention as cg_merkle_root).  The log keeps the *frontier* -- the root of one perfect subtree per
 * set bit of its size, at most 64 digests -- so that appending a batch costs O(batch) and the state that has to be
 * persisted next to the YYYY-MM-DD.jsonl file is a few hundred bytes.  With keep_leaf_digests the leaf digests stay
 * in HBM (32 bytes per leaf) and RFC 6962 audit paths can be produced.  No counterpart in the reference. */
typedef struct cg_merkle_log cg_merkle_log;
CG_API int cg_merkle_log_create(cg_merkle_log **out, int keep_leaf_digests);
CG_API void cg_merkle_log_destroy(cg_merkle_log *log);
CG_API int cg_merkle_log_append(cg_merkle_log *log, const uint8_t *bytes, const uint64_t *offsets, uint64_t n);   /* host buffers */
/* the day file itself (src/audit-trail.ts:151-179: JSON lines joined with "\n", trailing "\n" per flush): split at '\n' on the
 * device, every line without its '\n' is one leaf (an unterminated last line counts); *out_lines = leaves appended */
/* capacity for n_leaves more leaves / n_bytes of leaf bytes per append, allocated now instead of by the appends */
CG_API int cg_merkle_log_reserve(cg_merkle_log *log, uint64_t n_leaves, uint64_t n_bytes);
CG_API int cg_merkle_log_append_jsonl(cg_merkle_log *log, const uint8_t *bytes, uint64_t len, uint64_t *out_lines);
CG_API int cg_merkle_log_size(const cg_merkle_log *log, uint64_t *out_n);
CG_API int cg_merkle_log_root(cg_merkle_log *log, uint8_t out_root[32]);      /* == cg_merkle_root over every leaf appended so far */
/* frontier: one digest per set bit of the size, largest subtree first; restore() resumes a log from it (no proofs) */
CG_API int cg_merkle_log_frontier(cg_merkle_log *log, uint8_t *out_frontier32, uint32_t *out_count);
CG_API int cg_merkle_log_restore(cg_merkle_log **out, uint64_t n, const uint8_t *frontier32, uint32_t count);
/* RFC 6962 2.1.1 audit path of leaf `index` in the current tree (leaf level first); needs keep_leaf_digests */
CG_API int cg_merkle_log_proof(cg_merkle_log *log, uint64_t index, uint8_t *out_path32, uint32_t path_cap, uint32_t *out_len);
/* RFC 6962 2.1.2 consistency proof between the tree of the first first_size leaves and the current tree; needs keep_leaf_digests */
CG_API int cg_merkle_log_consistency(cg_merkle_log *log, uint64_t first_size, uint8_t *out_path32, uint32_t path_cap, uint32_t *out_len);
/* RFC 9162 2.1.4.2: *out_ok = 1 iff `path` proves that the tree (root_first, first_size) is a prefix of (root_second, second_size) */
CG_API int cg_merkle_verify_consistency(uint64_t first_size, uint64_t second_size, const uint8_t root_first[32], const uint8_t root_second[32],
                                        const uint8_t *path32, uint32_t path_len, int *out_ok);
/* RFC 9162 2.1.3.2: *out_ok = 1 iff `path` proves that leaf_bytes is entry `index` of the tree of tree_size leaves with this root */
CG_API int cg_merkle_verify_proof(const uint8_t *leaf_bytes, uint64_t leaf_len, uint64_t index, uint64_t tree_size,
                                  const uint8_t *path32, uint32_t path_len, const uint8_t root[32], int *out_ok);

#ifdef __cplusplus
}
#endif
#endif /* OPENCLAW_GOV_H */
