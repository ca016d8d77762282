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
 * surrogates already replaced by U+FFFD).  Ill-formed bytes decode as TextDecoder decodes them:
 * each maximal subpart of an ill-formed sequence becomes one U+FFFD (WHATWG Encoding, UTF-8
 * decoder), and a sequence cut at a message's end never continues into the next message.  All span offsets are reported both in bytes and in
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
 *                   *out_nhits = number of hits (CG_ERR_CAPACITY when it exceeds hits_cap; CG_ERR_TOO_LARGE at 2^32
 *                   hits or more).  Built on the device, as cg_scan_hits_batch_device builds it. */
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
/* findMatches + resolveOverlaps for one message, blocking (the synchronous hooks' path, src/redaction/hooks.ts:158-206,
 * 405-456).  Spans, *out_nspans, return code and statistics equal cg_find_matches_batch with n = 1 (span.msg = 0): on
 * CG_ERR_CAPACITY the first spans_cap spans are written.  A message of at most 16 KB costs one H2D copy, one CUDA graph,
 * one D2H copy and one synchronise (DESIGN.md section 4.5); longer ones, and the rare result too long for the staging
 * block, take the batch call's path. */
CG_API int cg_find_matches_one(cg_ruleset *rs, const uint8_t *bytes, uint32_t len,
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
/* RedactionEngine.scanString for one message, blocking: bytes, spans and digests equal cg_redact_batch with n = 1
 * (*out_need = redacted length; CG_ERR_CAPACITY with the sizes set and nothing else written when a capacity is short).
 * Same single-message path as cg_find_matches_one. */
CG_API int cg_redact_one(cg_ruleset *rs, const uint8_t *bytes, uint32_t len, uint8_t *out_bytes, uint64_t out_cap,
                         uint64_t *out_need, cg_span *out_spans, uint32_t spans_cap, uint32_t *out_nspans, uint8_t *out_digests32);
/* findMatches / scanString for the few strings of one scanned value, blocking: RedactionEngine.scan / scanValue /
 * scanStringValue (src/redaction/engine.ts:53-147) redact every string leaf of a tool result, a tool call's params or a
 * message's metadata (the hooks tool_result_persist, after_tool_call and message_sending, src/redaction/hooks.ts:158-206).
 * The contract is exactly cg_find_matches_batch's / cg_redact_batch's: signature, spans, bytes, offsets, digests, return
 * codes, argument checks, partial writes on CG_ERR_CAPACITY and statistics (except kernel_launches and last_scan_ms).  Only
 * the cost differs: up to 256 strings and 64 KB of text cost one H2D copy, one CUDA graph, one D2H copy and one synchronise
 * (DESIGN.md section 4.5), as cg_find_matches_one / cg_redact_one do for one string.  More strings or more text, profiling,
 * a queue overflow and the rare result too long for the staging block take the batch call's path. */
CG_API int cg_find_matches_few(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, uint32_t n,
                               cg_span *out_spans, uint32_t spans_cap, uint32_t *out_nspans);
CG_API int cg_redact_few(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, uint32_t n,
                         uint8_t *out_bytes, uint64_t out_cap, uint64_t *out_need, uint32_t *out_offsets,
                         cg_span *out_spans, uint32_t spans_cap, uint32_t *out_nspans, uint8_t *out_digests32);

/* ---- device-resident variant (inputs/outputs already in HBM; used by bench.py `value` and by callers that pipeline
 * their own copies).  Pointers are CUDA device pointers; `stream` is a cudaStream_t (NULL = the library's own stream);
 * asynchronous w.r.t. the host, strictly in order on `stream`.
 * Calls that share a rule set (every scan, hit-list, find-matches, redaction and verdict call on it: host-buffer,
 * single-message or device-resident) run in the order they were issued, whatever stream each one is on: a call on another
 * stream than the rule set's previous call waits for that call on the device, never on the host, and a blocking call returns
 * after it.  So do the calls that share the library's digest scratch: cg_sha256_batch, cg_merkle_root[_fixed],
 * cg_merkle_fold[_device], cg_merkle_block_roots_device, cg_merkle_root_sharded_device, the tree log's proof calls (host-buffer
 * and device-resident), the proof verifiers (cg_merkle_verify_proofs[_device], cg_merkle_verify_proof,
 * cg_merkle_verify_consistency).  So do the calls on one Merkle log (every cg_merkle_log_* call on it
 * but _size and _destroy, host-buffer or device-resident).  Other calls may overlap.
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
/* Every (message, rule) hit of a batch in HBM: the rule lists that matchesAny (src/conditions/context.ts:9-34, messageContains
 * / conversationContains and the tool-param `matches` rules), aggregateMatches (src/policy-evaluator.ts:110-146) and the
 * response gate's mustMatch / mustNotMatch (src/response-gate.ts:105-147) test per text, built on the device.  Same input rules as
 * cg_scan_batch_device.  d_out_words[n]: the result words of cg_scan_batch_device; d_out_hits: cg_hit[hits_cap] sorted by
 * (msg, rule), 4-byte aligned (may be NULL when hits_cap is 0); d_out_nhits: one uint32 = hits of the batch, 4-byte aligned.
 * Asynchronous and in order on `stream`; its status comes from cg_scan_join: CG_ERR_CAPACITY when the batch has more than
 * hits_cap hits (the first hits_cap are written), CG_ERR_TOO_LARGE at 2^32 - 1 hits or more, and CG_ERR_CAPACITY once after
 * an internal queue overflow (then *d_out_nhits = 0xffffffff, no hit is written, the scratch grows: issue the batch again).
 * n = 0 writes 0 to *d_out_nhits and enqueues nothing else. */
CG_API int cg_scan_hits_batch_device(cg_ruleset *rs, const void *d_bytes, const void *d_offsets, uint32_t n,
                                     void *d_out_words, void *d_out_hits, uint32_t hits_cap, void *d_out_nhits, void *stream);
/* cg_policy_verdict_batch for a batch in HBM (aggregateMatches / matchPolicy, src/policy-evaluator.ts:44-146): one verdict
 * (uint32, 4-byte aligned) per message into d_out_verdicts.  CG_ERR_INVALID_ARG before anything is enqueued when
 * cg_ruleset_set_policy has not been called.  Asynchronous and in order on `stream`, status from cg_scan_join; after an
 * internal queue overflow every verdict of the batch is 0xffffffff (no verdict has action 3) and the join reports
 * CG_ERR_CAPACITY once: issue the batch again. */
CG_API int cg_policy_verdict_batch_device(cg_ruleset *rs, const void *d_bytes, const void *d_offsets, uint32_t n,
                                          void *d_out_verdicts, void *stream);
/* Waits for `stream` and returns the status of every device-path batch (scan, hits, verdicts, find-matches, redact) issued
 * since the previous join: CG_OK, CG_ERR_CAPACITY (see above) or CG_ERR_TOO_LARGE (the VM ran out of thread-list space; words
 * all ones as well; a redacted batch of 4 GiB or more; a hit list of 2^32 - 1 hits or more). */
CG_API int cg_scan_join(cg_ruleset *rs, void *stream);

/* ---- per-message views of one rule set.  Which rules a text is tested against depends on where it comes from: the output
 * of an exempt tool goes through the credential built-ins only (credentialOnlyEngine, src/redaction/hooks.ts:79-81,176-178,
 * 218-222), and a policy's scope.channels / scope.excludeAgents decide whether it applies to a context
 * (src/policy-evaluator.ts:18-26).  A view is a subset of the rules of a rule set; each message of a batch carries one view
 * id.  The result for message m under view v equals what the call without views returns for m on a rule set compiled from
 * the rules of v alone (same relative order, flags, categories and policy assignment), with rule indices still those of the
 * whole set: result words count in-view rules only, hit lists hold in-view pairs, resolveOverlaps (registry.ts:288-316) runs
 * among in-view rules only (an out-of-view rule's longer match displaces nothing), redaction follows from those spans, and a
 * policy without an in-view rule never matches.  An empty view gives word 0, no hit, no span, the input bytes unchanged and
 * verdict 0.  cg_stats counts what the filtered step did.
 *
 * cg_ruleset_set_views: rows holds n_views x ceil(n_rules / 32) words, bit r of row v set = rule r is in view v.
 * 1 <= n_views <= 256; a bit at or past n_rules is CG_ERR_INVALID_ARG.  Like cg_ruleset_set_policy it waits for the library's
 * stream and replaces the rows: device-resident calls already enqueued on the caller's own streams must be joined first. */
CG_API int cg_ruleset_set_views(cg_ruleset *rs, const uint32_t *rows, uint32_t n_views);
/* Host-buffer twins: views = one id per message (host memory); otherwise the signature, outputs and statuses of the call
 * without views.  An id >= n_views, or a call before cg_ruleset_set_views, is CG_ERR_INVALID_ARG before anything is copied
 * or written.  cg_scan_batch_views runs a large words-only batch as one piece (cg_scan_batch overlaps its copies in chunks). */
CG_API int cg_scan_batch_views(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, const uint8_t *views, uint32_t n,
                               uint64_t *out_words, cg_hit *out_hits, uint32_t hits_cap, uint32_t *out_nhits);
CG_API int cg_find_matches_batch_views(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, const uint8_t *views, uint32_t n,
                                       cg_span *out_spans, uint32_t spans_cap, uint32_t *out_nspans);
CG_API int cg_redact_batch_views(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, const uint8_t *views, uint32_t n,
                                 uint8_t *out_bytes, uint64_t out_cap, uint64_t *out_need, uint32_t *out_offsets,
                                 cg_span *out_spans, uint32_t spans_cap, uint32_t *out_nspans, uint8_t *out_digests32);
CG_API int cg_policy_verdict_batch_views(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, const uint8_t *views, uint32_t n,
                                         uint32_t *out_verdicts);
/* Device-resident twins: d_views = one uint8 id per message in HBM (advance it with d_offsets for a sub-range); otherwise the
 * asynchrony, alignment rules, capacities, overflow protocol and cg_scan_join reporting of the call without views.  The host
 * cannot read the ids: an id >= n_views selects the empty view.  A call before cg_ruleset_set_views, or d_views = NULL, is
 * CG_ERR_INVALID_ARG before anything is enqueued.  cg_scan_hits_batch_device_views with d_out_hits = NULL, hits_cap = 0 and
 * d_out_nhits = NULL writes the result words alone (cg_scan_batch_device's output, launched directly, not from a graph). */
CG_API int cg_scan_hits_batch_device_views(cg_ruleset *rs, const void *d_bytes, const void *d_offsets, const void *d_views, uint32_t n,
                                           void *d_out_words, void *d_out_hits, uint32_t hits_cap, void *d_out_nhits, void *stream);
CG_API int cg_find_matches_batch_device_views(cg_ruleset *rs, const void *d_bytes, const void *d_offsets, const void *d_views, uint32_t n,
                                              void *d_out_spans, uint32_t spans_cap, void *d_out_nspans, void *stream);
CG_API int cg_redact_batch_device_views(cg_ruleset *rs, const void *d_bytes, const void *d_offsets, const void *d_views, uint32_t n,
                                        void *d_out_bytes, uint64_t out_cap, void *d_out_offsets,
                                        void *d_out_spans, uint32_t spans_cap, void *d_out_digests32, void *d_out_sizes, void *stream);
CG_API int cg_policy_verdict_batch_device_views(cg_ruleset *rs, const void *d_bytes, const void *d_offsets, const void *d_views, uint32_t n,
                                                void *d_out_verdicts, void *stream);

/* ---- whole policy rules (PolicyEvaluator.evaluate, src/policy-evaluator.ts:18-146, and the evaluators of src/conditions) for a batch of
 * evaluation contexts.  A policy PROGRAM is stored on a rule set; one call scans all texts of all contexts in one policy-mode
 * step and evaluates the program for every context on the device.
 *
 * Split of work.  Regex leaves are device leaves HIT(r, q) = "rule r of this rule set hit some text of the context whose
 * role is q": messageContains (role 0, the message), conversationContains (role 1, a conversation entry) and a tool param's
 * `matches` (role 2 + k, param key k as the caller numbers them).  Texts are included as a caller of the reference sees
 * them: an empty message is left out, every conversation entry and every string param is included, so checkMessage's
 * `!ctx.messageContent` (context.ts) and matchParam's `typeof value !== "string"` (tool.ts) hold without further leaves; an
 * invalid `matches` pattern is CONST 0 (tool.ts:39-44).  Every other test is an ATOM a, one bit per context the caller
 * computes: tool-name and agent-id globs, trustTier, channel, hasMetadata, sessionKey, param equals / contains / startsWith /
 * in, the rule gates minTrust / maxTrust, a policy's matchesScope (:18-26), time / risk / frequency.  The device evaluates
 * the boolean structure (conditions = AND, any = OR, not), the first matching rule of each policy (matchPolicy, :129-146)
 * and aggregateMatches (:44-78).  Policies are stored in evaluation order (priority, then specificity, :36-42: an order that
 * depends on the policy alone; scope only removes policies, so one global order serves every context).
 *
 * Program (uint32 words): [n_policies], then per policy [scope atom, 0xffffffff = none][n_rules], then per rule
 * [action | has_reason << 2][n_ops][n_ops op words, postfix].  action: 0 allow, 1 audit, 2 2fa, 3 deny; has_reason: the
 * effect has a non-empty reason.  Program rules are numbered 0, 1, ... across all policies in this order.  Op words (low 3
 * bits the op): CONST b = 0 | b << 3 (b = 0 or 1); ATOM a = 1 | a << 3; HIT r q = 2 | r << 3 | q << 24 (r < 2^21, q < 256);
 * AND = 3; OR = 4; NOT = 5.  An empty condition list is CONST 1, an empty `any` CONST 0.
 * cg_ruleset_set_policy_program checks that every rule leaves exactly one value, that no rule needs a stack deeper than 32
 * (CG_ERR_TOO_LARGE), that r < the rule set's rules and a < n_atoms, and at most 2^20 - 1 program rules (CG_ERR_TOO_LARGE);
 * anything else malformed is CG_ERR_INVALID_ARG.  Like cg_ruleset_set_policy it waits for the library's stream and replaces
 * the tables.
 *
 * cg_policy_eval_batch: n_texts texts (bytes / offsets as cg_scan_batch) with one role each (roles[n_texts]); context c owns
 * the texts [ctx_offsets[c], ctx_offsets[c+1]) (n_ctx + 1 offsets, non-decreasing, at most n_texts; a context may own none,
 * so n_ctx may exceed n_texts and n_texts may be 0) and atom row atoms[c * ceil(n_atoms / 32) ..] (bit a of the row = atom
 * a).  out_verdicts[c] = outcome | (matched policies, saturating at 511) << 3 | deciding program rule << 12, outcome 0 no
 * policy matched, 1 allow, 2 allow with audit, 3 2fa, 4 deny; the deciding rule is the first match of the winning action
 * (deny or 2fa) with has_reason, else 0xfffff -- the reason is the first non-empty one of that action (:51-60).
 * out_matches: the (context, program rule) of every policy that matched, sorted by (context, evaluation order) -- the
 * `matches` list of the result (engine.ts:236,249) -- the first matches_cap written; *out_nmatches = their number
 * (CG_ERR_CAPACITY past matches_cap, CG_ERR_TOO_LARGE at 2^32 - 1 or more).  out_matches and out_nmatches may both be NULL
 * (verdicts only).  A context range that is decreasing or past n_texts is CG_ERR_INVALID_ARG before anything is copied. */
typedef struct cg_policy_match { uint32_t ctx; uint32_t rule; } cg_policy_match;   /* rule = program rule index */
CG_API int cg_ruleset_set_policy_program(cg_ruleset *rs, const uint32_t *program, uint32_t words, uint32_t n_atoms);
CG_API int cg_policy_eval_batch(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, const uint8_t *roles, uint32_t n_texts,
                                const uint32_t *ctx_offsets, const uint32_t *atoms, uint32_t n_ctx, uint32_t *out_verdicts,
                                cg_policy_match *out_matches, uint32_t matches_cap, uint32_t *out_nmatches);
/* The same for a batch in HBM (d_bytes 16-byte aligned as for cg_scan_batch_device; every other pointer 4-byte aligned;
 * d_out_matches may be NULL when matches_cap is 0; d_out_nmatches = NULL: verdicts only).  Asynchronous and in order on
 * `stream`, status from cg_scan_join: CG_ERR_CAPACITY when there are more than matches_cap matches (the first matches_cap
 * are written), CG_ERR_TOO_LARGE at 2^32 - 1 or more, and CG_ERR_CAPACITY once after an internal queue overflow (then every
 * verdict is 0xffffffff, *d_out_nmatches = 0xffffffff and no match is written: issue the batch again).  The host cannot read
 * the context offsets: a context whose range is decreasing or runs past n_texts gets verdict 0xfffffffe and no match, the
 * others are unaffected.  n_ctx = 0 writes 0 to *d_out_nmatches and enqueues nothing else.  Launches: the step, then one
 * kernel (verdicts only) or count + exclusive scan + emit, on grids that depend on n_ctx and the SM count only. */
CG_API int cg_policy_eval_batch_device(cg_ruleset *rs, const void *d_bytes, const void *d_offsets, const void *d_roles, uint32_t n_texts,
                                       const void *d_ctx_offsets, const void *d_atoms, uint32_t n_ctx, void *d_out_verdicts,
                                       void *d_out_matches, uint32_t matches_cap, void *d_out_nmatches, void *stream);
/* One evaluation context, blocking: PolicyEvaluator.evaluate for the hooks that evaluate one context per event
 * (before_tool_call, message_sending; src/hooks.ts:173-290).  Returns exactly what cg_policy_eval_batch returns for the
 * context that owns all n_texts texts (ctx_offsets = {0, n_texts}) with atom row `atoms`: *out_verdict = its verdict word,
 * out_rules[i] = out_matches[i].rule (program rules of the matched policies, in evaluation order), the first rules_cap of them
 * written and *out_nrules = their number (CG_ERR_CAPACITY past rules_cap); the same argument checks, error codes and cg_stats
 * (but kernel_launches and last_scan_ms).  out_rules and out_nrules may be NULL; n_texts = 0 is valid (a tool call without
 * string params gets a verdict from its atoms).  Up to 64 texts, 64 KB of text, 32 768 atoms and 4096 matched policies (when
 * the caller wants that many), the call costs one H2D copy, one CUDA graph (the step, then one kernel), one D2H copy and one
 * synchronise (DESIGN.md section 4.8); anything larger, and a step whose internal queues overflowed, takes the batch call's
 * path.  In order with the rule set's other calls, like cg_scan_one. */
CG_API int cg_policy_eval_one(cg_ruleset *rs, const uint8_t *bytes, const uint32_t *offsets, const uint8_t *roles,
                              uint32_t n_texts, const uint32_t *atoms, uint32_t *out_verdict,
                              uint32_t *out_rules, uint32_t rules_cap, uint32_t *out_nrules);

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
/* capacity for n_leaves more leaves / n_bytes of leaf bytes per append, allocated now instead of by the appends.  On a log
 * without a node store (cg_merkle_log_create) this includes the buffers that fold a block of up to n_leaves leaves: 24 bytes per
 * leaf on top of the 32 of a kept leaf digest (a tree log folds into its store and needs none). */
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

/* ---- proofs at any tree size, in batches.  An auditor holds the root and size of an earlier day's log (the frontier
 * persisted next to YYYY-MM-DD.jsonl, src/audit-trail.ts:151-179) and asks today's log for receipts against it, as RFC 6962 /
 * CT get-proof-by-hash does with its tree_size.  A log made by cg_merkle_log_create_tree keeps its leaf digests and every
 * complete aligned node MTH(D[j 2^h, (j + 1) 2^h)) -- fewer than n more digests, filled by the appends' own folds and frontier
 * carries -- so a proof is a gather of at most 64 stored digests instead of a re-hash of the tree.  Its roots, frontiers and
 * sizes equal those of a keep_leaf_digests = 1 log, and so do its appends' kernel launches; cg_merkle_log_proof and
 * cg_merkle_log_consistency on it return the same bytes from the store.  Logs from cg_merkle_log_restore keep no nodes. */
CG_API int cg_merkle_log_create_tree(cg_merkle_log **out);
/* RFC 6962 2.1.1 PATH(index, D[0:tree_size]) for m indices; needs a log made by cg_merkle_log_create_tree.
 * tree_size <= size of the log.  Path i (leaf level first) at out_paths32 + i * path_stride * 32, its length in out_lens[i];
 * the stride's unused digests are zero.  Checked before anything is written: no node store -> CG_ERR_UNSUPPORTED; tree_size 0
 * or past the log, or an index >= tree_size -> CG_ERR_INVALID_ARG; path_stride < ceil(log2 tree_size) -> CG_ERR_CAPACITY;
 * m = 0 -> CG_OK with nothing written. */
CG_API int cg_merkle_log_proofs(cg_merkle_log *log, const uint64_t *indices, uint32_t m, uint64_t tree_size,
                                uint8_t *out_paths32, uint32_t path_stride, uint32_t *out_lens);
/* RFC 6962 2.1.2 PROOF(first_size, D[0:second_size]) with second_size <= size of the log (1 <= first_size <= second_size);
 * at most ceil(log2 second_size) + 1 digests.  Errors as for cg_merkle_log_proofs, *out_len and the path untouched. */
CG_API int cg_merkle_log_consistency_between(cg_merkle_log *log, uint64_t first_size, uint64_t second_size,
                                             uint8_t *out_path32, uint32_t path_cap, uint32_t *out_len);
/* RFC 9162 2.1.3.2 for m (leaf, index, path) triples against one (tree_size, root): out_ok[i] = 1 iff proof i holds -- exactly
 * when cg_merkle_verify_proof says so.  leaves: bytes/offsets as cg_merkle_root (ragged); paths at path_stride digests,
 * lengths in path_lens (each <= 64 and <= path_stride, else CG_ERR_INVALID_ARG). */
CG_API int cg_merkle_verify_proofs(const uint8_t *leaf_bytes, const uint64_t *leaf_offsets, const uint64_t *indices, uint32_t m,
                                   uint64_t tree_size, const uint8_t *paths32, uint32_t path_stride, const uint32_t *path_lens,
                                   const uint8_t root[32], uint8_t *out_ok);

/* ---- device-resident Merkle log calls: leaves, indices, paths and verdicts already in HBM (event records a caller built on the
 * device, proofs served to or checked for a consumer on the device).  Each call writes exactly what its host twin returns --
 * the same roots, frontier, node store, path bytes, lengths and verdicts -- and touches only the caller's device buffers and the
 * log's or the library's scratch.  Asynchronous on `stream` (NULL = the library's stream): a call waits on the host only when a
 * log or library buffer has to grow (cg_merkle_log_reserve sizes the log's buffers up front).  Calls on one log run in the order
 * they were issued, host-buffer and device-resident alike, whatever stream each is on; calls on different logs overlap.
 * cg_merkle_log_size counts the leaves enqueued so far.  Every argument the host can see is checked as the host twin checks it,
 * and pointer alignment too, before anything is enqueued (CG_ERR_INVALID_ARG): ragged byte buffers 16-byte aligned and readable
 * 16 bytes past their last offset, paths 16-byte aligned, offsets and indices 8-byte, lengths 4-byte.  What only the device can
 * see is checked in band, per item, leaving the other items alone: */
/* leaf i = d_bytes[d_offsets[i], d_offsets[i+1]) (uint64 offsets).  A decreasing pair goes in as the empty leaf without being
 * read and marks the log: cg_merkle_log_join reports CG_ERR_INVALID_ARG once, and from then on every call on the log but
 * _size and _destroy returns CG_ERR_INVALID_ARG (a log that holds a wrong leaf must not keep going quietly). */
CG_API int cg_merkle_log_append_device(cg_merkle_log *log, const void *d_bytes, const void *d_offsets /* uint64[m+1] */,
                                       uint64_t m, void *stream);
/* m leaves of leaf_len bytes each at d_bytes, any alignment (the leaves and kernels of cg_merkle_block_roots_device, e.g.
 * fixed-size event records) */
CG_API int cg_merkle_log_append_fixed_device(cg_merkle_log *log, const void *d_bytes, uint64_t leaf_len, uint64_t m, void *stream);
/* cg_merkle_log_root into 32 bytes of HBM (any alignment) */
CG_API int cg_merkle_log_root_device(cg_merkle_log *log, void *d_out_root32, void *stream);
/* cg_merkle_log_proofs from and into HBM (the same argument checks); an index >= tree_size gets length 0xffffffff and an
 * all-zero stride */
CG_API int cg_merkle_log_proofs_device(cg_merkle_log *log, const void *d_indices /* uint64[m] */, uint32_t m, uint64_t tree_size,
                                       void *d_out_paths32, uint32_t path_stride, void *d_out_lens /* uint32[m] */, void *stream);
/* cg_merkle_log_consistency_between into HBM: the path's digests at d_out_path32, its length (uint32) at *d_out_len */
CG_API int cg_merkle_log_consistency_between_device(cg_merkle_log *log, uint64_t first_size, uint64_t second_size,
                                                    void *d_out_path32, uint32_t path_cap, void *d_out_len, void *stream);
/* cg_merkle_verify_proofs from and into HBM (leaves ragged as for cg_merkle_log_append_device, root: 32 bytes, any alignment,
 * d_out_ok: one uint8 per proof).  A decreasing leaf offset pair, a path length above 64 or above path_stride, or an index >=
 * tree_size gives ok = 0 without reading that leaf or path. */
CG_API int cg_merkle_verify_proofs_device(const void *d_leaf_bytes, const void *d_leaf_offsets, const void *d_indices, uint32_t m,
                                          uint64_t tree_size, const void *d_paths32, uint32_t path_stride, const void *d_path_lens,
                                          const void *d_root32, void *d_out_ok, void *stream);
/* waits for `stream` and for every call issued on the log; CG_ERR_INVALID_ARG (once, then on every call) when a device append
 * read a decreasing offset pair, else CG_OK */
CG_API int cg_merkle_log_join(cg_merkle_log *log, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* OPENCLAW_GOV_H */
