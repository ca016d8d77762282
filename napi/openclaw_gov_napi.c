/*
 * napi/openclaw_gov_napi.c -- thin N-API (node_api.h, C ABI, ABI-stable) shim over libopenclaw_gov.so.
 *
 * This is the binding the TypeScript plugin (@vainplex/openclaw-governance, src/hooks.ts,
 * src/redaction/registry.ts) calls instead of V8 RegExp / node:crypto on the hot path (napi/gpu-backend.ts).
 * Node.js is absent from this repository's image and from the GPU box, so the addon is not built here; it compiles
 * against any Node >= 22 header set, and the CPU test tier compiles it against napi/stub/node_api.h (declarations only)
 * so that it cannot rot:
 *
 *   cc -shared -fPIC -I"$(node -p 'process.config.variables.node_prefix')/include/node" \
 *      -Iinclude napi/openclaw_gov_napi.c -Lvainplex_openclaw_b200 -lopenclaw_gov \
 *      -Wl,-rpath,'$ORIGIN' -o openclaw_gov.node
 *
 * JS surface (all synchronous -- the sync hooks before_message_write / tool_result_persist cannot
 * await, src/hooks.ts:360-365; the async bulk path wraps scanBatch in a libuv worker on the JS side):
 *   init(device?: number): void ; shutdown(): void ; stats(): {...} ; ruleCheck(source, flags?): number
 *   createRuleset(rules: {source: string, flags?: number, category?: number}[]): {handle: External, status: Int32Array}
 *   scanBatch(handle, bytes: Uint8Array, offsets: Uint32Array): {words: BigUint64Array, hits: Uint32Array}  // hits: msg,rule pairs
 *   scanOne(handle, bytes: Uint8Array): {word: bigint, rules: Uint32Array}
 *   findMatchesBatch(handle, bytes, offsets): Uint32Array  // 6 words per span: msg, rule, startByte, endByte, start16, end16
 *   redactBatch(handle, bytes, offsets): {bytes, offsets, spans, digests}  // scanString for a batch, spliced on the device
 *   findMatchesOne(handle, bytes: Uint8Array): Uint32Array  // one message, blocking: findMatchesBatch's spans for a batch of one
 *   redactOne(handle, bytes: Uint8Array): {bytes, spans, digests}  // one message, blocking: scanString spliced on the device
 *   findMatchesFew(handle, bytes, offsets): Uint32Array  // the strings of one scanned value, blocking, one device round trip
 *   redactFew(handle, bytes, offsets): {bytes, offsets, spans, digests}  //   (up to 256 strings and 64 KB): the batch calls' results
 *   setPolicy(handle, rulePolicy: Uint32Array, ruleAction: Uint8Array): void ; verdictBatch(handle, bytes, offsets): Uint32Array
 *   setViews(handle, rows: Uint32Array, nViews: number): void  // nViews rows of ceil(nRules / 32) words, bit r = rule r in the view
 *   scanBatchViews / findMatchesBatchViews / redactBatchViews / verdictBatchViews(handle, bytes, offsets, views: Uint8Array)
 *     // the batch calls above with one view id per message: each message decided on its view's rules alone
 *   setPolicyProgram(handle, program: Uint32Array, nAtoms: number): void  // whole policies (openclaw_gov.h: program layout)
 *   policyEvalBatch(handle, bytes, offsets, roles: Uint8Array, ctxOffsets: Uint32Array, atoms: Uint32Array, nAtoms: number):
 *     {verdicts: Uint32Array, matches: Uint32Array}  // one verdict per context; matches: ctx, program rule pairs
 *   policyEvalOne(handle, bytes, offsets, roles: Uint8Array, atoms: Uint32Array, nAtoms: number): {verdict: number, rules: Uint32Array}
 *     // one context owning every text, blocking, one device round trip: policyEvalBatch's verdict and program rules
 *   sha256Batch(bytes: Uint8Array, offsets: BigUint64Array): Uint8Array  // 32 bytes per item
 *   merkleRoot(bytes: Uint8Array, offsets: BigUint64Array): Uint8Array   // 32 bytes
 *   logCreate(keepLeafDigests: boolean): External ; logRestore(size: bigint, frontier: Uint8Array): External
 *   logAppend(log, bytes, offsets: BigUint64Array): void ; logAppendJsonl(log, bytes: Uint8Array): bigint (lines) ; logReserve(log, leaves, bytes)
 *   logSize(log): bigint ; logRoot(log): Uint8Array ; logFrontier(log): Uint8Array
 *   logProof(log, index: bigint): Uint8Array ; logConsistency(log, firstSize: bigint): Uint8Array      // 32 bytes per path node
 *   verifyProof(leaf: Uint8Array, index, treeSize, path: Uint8Array, root: Uint8Array): boolean
 *   verifyConsistency(firstSize, secondSize, rootFirst, rootSecond, path): boolean
 *   logCreateTree(): External  // keeps every complete subtree node: receipts against any earlier size, in batches
 *   logProofs(log, indices: BigUint64Array, treeSize): {paths: Uint8Array, lens: Uint32Array}  // stride max(1, ceil(log2 treeSize)) nodes
 *   logConsistencyBetween(log, firstSize, secondSize): Uint8Array
 *   verifyProofs(leafBytes, leafOffsets: BigUint64Array, indices: BigUint64Array, treeSize, paths, lens: Uint32Array, stride, root): Uint8Array (0/1)
 * Every failure throws a JS Error carrying cg_last_error(); the reference's try/catch + failMode
 * blocks (src/hooks.ts:232-241, src/redaction/hooks.ts:193-204) decide what happens next.
 * Offsets are validated here (non-decreasing, last one within the byte array): the C ABI trusts its caller.
 */
#include <node_api.h>
#include <stdlib.h>
#include <string.h>

#include "openclaw_gov.h"

#define NAPI_CALL(env, call) do { if ((call) != napi_ok) { napi_throw_error((env), NULL, "N-API call failed: " #call); return NULL; } } while (0)
#define CG_CALL(env, call) do { int _rc = (call); if (_rc != CG_OK) { napi_throw_error((env), NULL, cg_last_error()); return NULL; } } while (0)
#define ARGS(env, info, n) size_t argc = (n); napi_value argv[(n)]; NAPI_CALL(env, napi_get_cb_info(env, info, &argc, argv, NULL, NULL)); \
  if (argc < (n)) { napi_throw_type_error(env, NULL, "too few arguments"); return NULL; }

static void ruleset_finalize(napi_env env, void *data, void *hint) { (void)env; (void)hint; cg_ruleset_destroy((cg_ruleset *)data); }
static void log_finalize(napi_env env, void *data, void *hint) { (void)env; (void)hint; cg_merkle_log_destroy((cg_merkle_log *)data); }

/* typed array -> pointer + byte length (element size from the array type) */
static int get_ta(napi_env env, napi_value v, uint8_t **p, size_t *bytes, napi_typedarray_type want) {
  napi_typedarray_type t; napi_value ab; size_t off, len; bool is;
  if (napi_is_typedarray(env, v, &is) != napi_ok || !is) return 0;
  if (napi_get_typedarray_info(env, v, &t, &len, (void **)p, &ab, &off) != napi_ok || t != want) return 0;
  *bytes = len * (t == napi_uint8_array ? 1 : t == napi_uint32_array || t == napi_int32_array ? 4 : 8);
  return 1;
}
/* (bytes, offsets) of a batch; 32-bit offsets for scans, 64-bit for SHA / Merkle.  Returns the number of items or -1 (thrown). */
static int64_t get_batch(napi_env env, napi_value vb, napi_value vo, int wide, uint8_t **bytes, uint8_t **offs) {
  size_t nb, no;
  if (!get_ta(env, vb, bytes, &nb, napi_uint8_array) || !get_ta(env, vo, offs, &no, wide ? napi_biguint64_array : napi_uint32_array) || no == 0) {
    napi_throw_type_error(env, NULL, wide ? "expected (Uint8Array, BigUint64Array)" : "expected (Uint8Array, Uint32Array)"); return -1;
  }
  const size_t n = no / (wide ? 8 : 4) - 1;
  uint64_t prev = 0;
  for (size_t i = 0; i <= n; i++) {
    const uint64_t o = wide ? ((const uint64_t *)*offs)[i] : ((const uint32_t *)*offs)[i];
    if (o < prev || o > nb) { napi_throw_range_error(env, NULL, "offsets must be non-decreasing and end inside the byte array"); return -1; }
    prev = o;
  }
  return (int64_t)n;
}
/* the *Views calls' last argument: one view id per message (Uint8Array of n elements).  0 = thrown. */
static int get_views(napi_env env, napi_value v, int64_t n, uint8_t **ids) {
  size_t nv;
  if (!get_ta(env, v, ids, &nv, napi_uint8_array) || (int64_t)nv != n) { napi_throw_type_error(env, NULL, "views: a Uint8Array with one view id per message"); return 0; }
  if (!nv) *ids = NULL;
  return 1;
}
/* arguments (handle, bytes, offsets[, views]) of a batch call: 3 + views of them */
#define BATCH_ARGS(env, info, views) size_t argc = 4; napi_value argv[4]; NAPI_CALL(env, napi_get_cb_info(env, info, &argc, argv, NULL, NULL)); \
  if (argc < 3u + (size_t)(views)) { napi_throw_type_error(env, NULL, "too few arguments"); return NULL; }
static napi_value make_u8(napi_env env, const void *src, size_t len) {
  napi_value ab, arr; void *data;
  if (napi_create_arraybuffer(env, len, &data, &ab) != napi_ok) return NULL;
  if (len && src) memcpy(data, src, len);
  if (napi_create_typedarray(env, napi_uint8_array, len, ab, 0, &arr) != napi_ok) return NULL;
  return arr;
}
static int get_u64(napi_env env, napi_value v, uint64_t *out) {
  bool lossless; napi_valuetype t;
  if (napi_typeof(env, v, &t) != napi_ok) return 0;
  if (t == napi_bigint) return napi_get_value_bigint_uint64(env, v, out, &lossless) == napi_ok;
  double d; if (napi_get_value_double(env, v, &d) != napi_ok || d < 0) return 0;
  *out = (uint64_t)d; return 1;
}

static napi_value js_init(napi_env env, napi_callback_info info) {
  size_t argc = 1; napi_value argv[1]; int32_t dev = -1;
  NAPI_CALL(env, napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
  if (argc >= 1) napi_get_value_int32(env, argv[0], &dev);
  CG_CALL(env, cg_init(dev));
  return NULL;
}
static napi_value js_shutdown(napi_env env, napi_callback_info info) { (void)env; (void)info; cg_shutdown(); return NULL; }

static napi_value js_stats(napi_env env, napi_callback_info info) {
  (void)info; cg_stats s; napi_value out, v;
  CG_CALL(env, cg_get_stats(&s));
  NAPI_CALL(env, napi_create_object(env, &out));
#define PUT(name, val) do { NAPI_CALL(env, napi_create_double(env, (double)(val), &v)); NAPI_CALL(env, napi_set_named_property(env, out, name, v)); } while (0)
  PUT("messagesScanned", s.messages_scanned); PUT("bytesScanned", s.bytes_scanned); PUT("hits", s.hits); PUT("spans", s.spans);
  PUT("sha256Items", s.sha256_items); PUT("merkleLeaves", s.merkle_leaves); PUT("kernelLaunches", s.kernel_launches);
  PUT("lastScanMs", s.last_scan_ms); PUT("lastMerkleMs", s.last_merkle_ms);
#undef PUT
  return out;
}

static char *get_string(napi_env env, napi_value v, size_t *len) {
  if (napi_get_value_string_utf8(env, v, NULL, 0, len) != napi_ok) return NULL;
  char *buf = (char *)malloc(*len + 1);
  if (!buf) return NULL;
  if (napi_get_value_string_utf8(env, v, buf, *len + 1, len) != napi_ok) { free(buf); return NULL; }      /* lone surrogates -> U+FFFD, like Buffer.from */
  return buf;
}

static napi_value js_rule_check(napi_env env, napi_callback_info info) {
  size_t argc = 2; napi_value argv[2], out; uint32_t flags = 0; size_t len;
  NAPI_CALL(env, napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
  if (argc < 1) { napi_throw_type_error(env, NULL, "ruleCheck(source, flags?)"); return NULL; }
  if (argc >= 2) napi_get_value_uint32(env, argv[1], &flags);
  char *src = get_string(env, argv[0], &len);
  if (!src) { napi_throw_type_error(env, NULL, "ruleCheck: source must be a string"); return NULL; }
  const int rc = cg_rule_check(src, (uint32_t)len, flags, NULL, 0);
  free(src);
  NAPI_CALL(env, napi_create_int32(env, rc, &out));
  return out;
}

static napi_value js_create_ruleset(napi_env env, napi_callback_info info) {
  ARGS(env, info, 1)
  uint32_t n = 0;
  NAPI_CALL(env, napi_get_array_length(env, argv[0], &n));
  cg_rule *rules = (cg_rule *)calloc(n ? n : 1, sizeof(cg_rule));
  char **bufs = (char **)calloc(n ? n : 1, sizeof(char *));
  int bad = !rules || !bufs;
  for (uint32_t i = 0; i < n && !bad; i++) {
    napi_value r, v; size_t len = 0; bool has;
    if (napi_get_element(env, argv[0], i, &r) != napi_ok || napi_get_named_property(env, r, "source", &v) != napi_ok || !(bufs[i] = get_string(env, v, &len))) { bad = 1; break; }
    rules[i].source = bufs[i]; rules[i].source_len = (uint32_t)len;
    if (napi_has_named_property(env, r, "flags", &has) == napi_ok && has && napi_get_named_property(env, r, "flags", &v) == napi_ok) napi_get_value_uint32(env, v, &rules[i].flags);
    rules[i].category = CG_CAT_CUSTOM;
    if (napi_has_named_property(env, r, "category", &has) == napi_ok && has && napi_get_named_property(env, r, "category", &v) == napi_ok) napi_get_value_uint32(env, v, &rules[i].category);
  }
  napi_value status_ab, status, out = NULL, handle; void *status_data = NULL; cg_ruleset *rs = NULL; int rc = CG_OK;
  if (!bad) bad = napi_create_arraybuffer(env, (size_t)n * 4, &status_data, &status_ab) != napi_ok || napi_create_typedarray(env, napi_int32_array, n, status_ab, 0, &status) != napi_ok;
  if (!bad) rc = cg_ruleset_create(rules, n, CG_OPT_STRIDE_AUTO, &rs, (int32_t *)status_data);
  if (bufs) for (uint32_t i = 0; i < n; i++) free(bufs[i]);
  free(bufs); free(rules);
  if (bad) { napi_throw_type_error(env, NULL, "createRuleset([{source: string, flags?: number, category?: number}])"); return NULL; }
  if (rc != CG_OK) { napi_throw_error(env, NULL, cg_last_error()); return NULL; }
  if (napi_create_object(env, &out) != napi_ok || napi_create_external(env, rs, ruleset_finalize, NULL, &handle) != napi_ok) { cg_ruleset_destroy(rs); napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  NAPI_CALL(env, napi_set_named_property(env, out, "handle", handle));
  NAPI_CALL(env, napi_set_named_property(env, out, "status", status));
  return out;
}

static napi_value scan_batch(napi_env env, napi_callback_info info, int views) {
  BATCH_ARGS(env, info, views)
  cg_ruleset *rs; uint8_t *bytes, *offp, *ids = NULL;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  const int64_t nn = get_batch(env, argv[1], argv[2], 0, &bytes, &offp); if (nn < 0) return NULL;
  if (views && !get_views(env, argv[3], nn, &ids)) return NULL;
  const uint32_t n = (uint32_t)nn;
#define SCAN(cap) (views ? cg_scan_batch_views(rs, bytes, (const uint32_t *)offp, ids, n, (uint64_t *)wdata, tmp, (cap), &nh) \
                         : cg_scan_batch(rs, bytes, (const uint32_t *)offp, n, (uint64_t *)wdata, tmp, (cap), &nh))
  napi_value words_ab, words, hits_ab, hits, out; void *wdata, *hdata;
  NAPI_CALL(env, napi_create_arraybuffer(env, (size_t)n * 8, &wdata, &words_ab));
  NAPI_CALL(env, napi_create_typedarray(env, napi_biguint64_array, n, words_ab, 0, &words));
  uint32_t nh = 0, cap = 1024; cg_hit *tmp = (cg_hit *)malloc(sizeof(cg_hit) * cap);
  int rc = tmp ? SCAN(cap) : CG_ERR_CUDA;
  if (rc == CG_ERR_CAPACITY) { cap = nh; cg_hit *t2 = (cg_hit *)realloc(tmp, sizeof(cg_hit) * cap); if (t2) { tmp = t2; rc = SCAN(cap); } }
#undef SCAN
  if (rc != CG_OK) { free(tmp); napi_throw_error(env, NULL, cg_last_error()); return NULL; }
  if (napi_create_arraybuffer(env, (size_t)nh * 8, &hdata, &hits_ab) != napi_ok) { free(tmp); napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  memcpy(hdata, tmp, (size_t)nh * 8); free(tmp);
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint32_array, (size_t)nh * 2, hits_ab, 0, &hits));
  NAPI_CALL(env, napi_create_object(env, &out));
  NAPI_CALL(env, napi_set_named_property(env, out, "words", words));
  NAPI_CALL(env, napi_set_named_property(env, out, "hits", hits));
  return out;
}
static napi_value js_scan_batch(napi_env env, napi_callback_info info) { return scan_batch(env, info, 0); }
static napi_value js_scan_batch_views(napi_env env, napi_callback_info info) { return scan_batch(env, info, 1); }

static napi_value js_scan_one(napi_env env, napi_callback_info info) {
  ARGS(env, info, 2)
  cg_ruleset *rs; uint8_t *bytes; size_t nb; uint64_t word = 0; uint32_t nr = 0; uint32_t rules[64];
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  if (!get_ta(env, argv[1], &bytes, &nb, napi_uint8_array)) { napi_throw_type_error(env, NULL, "scanOne(handle, Uint8Array)"); return NULL; }
  CG_CALL(env, cg_scan_one(rs, bytes, (uint32_t)nb, &word, rules, 64, &nr));
  napi_value out, w, ab, arr; void *data;
  NAPI_CALL(env, napi_create_object(env, &out));
  NAPI_CALL(env, napi_create_bigint_uint64(env, word, &w));
  if (nr > 64) nr = 64;
  NAPI_CALL(env, napi_create_arraybuffer(env, (size_t)nr * 4, &data, &ab));
  memcpy(data, rules, (size_t)nr * 4);
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint32_array, nr, ab, 0, &arr));
  NAPI_CALL(env, napi_set_named_property(env, out, "word", w));
  NAPI_CALL(env, napi_set_named_property(env, out, "rules", arr));
  return out;
}

static napi_value find_matches_batch(napi_env env, napi_callback_info info, int views) {
  BATCH_ARGS(env, info, views)
  cg_ruleset *rs; uint8_t *bytes, *offp, *ids = NULL;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  const int64_t nn = get_batch(env, argv[1], argv[2], 0, &bytes, &offp); if (nn < 0) return NULL;
  if (views && !get_views(env, argv[3], nn, &ids)) return NULL;
  uint32_t n = (uint32_t)nn, ns = 0, cap = 256; cg_span *tmp = (cg_span *)malloc(sizeof(cg_span) * cap);
#define FIND(cap) (views ? cg_find_matches_batch_views(rs, bytes, (const uint32_t *)offp, ids, n, tmp, (cap), &ns) \
                         : cg_find_matches_batch(rs, bytes, (const uint32_t *)offp, n, tmp, (cap), &ns))
  int rc = tmp ? FIND(cap) : CG_ERR_CUDA;
  if (rc == CG_ERR_CAPACITY) { cap = ns; cg_span *t2 = (cg_span *)realloc(tmp, sizeof(cg_span) * cap); if (t2) { tmp = t2; rc = FIND(cap); } }
#undef FIND
  if (rc != CG_OK) { free(tmp); napi_throw_error(env, NULL, cg_last_error()); return NULL; }
  napi_value ab, arr; void *data;
  if (napi_create_arraybuffer(env, (size_t)ns * sizeof(cg_span), &data, &ab) != napi_ok) { free(tmp); napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  memcpy(data, tmp, (size_t)ns * sizeof(cg_span)); free(tmp);
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint32_array, (size_t)ns * 6, ab, 0, &arr));
  return arr;
}
static napi_value js_find_matches_batch(napi_env env, napi_callback_info info) { return find_matches_batch(env, info, 0); }
static napi_value js_find_matches_batch_views(napi_env env, napi_callback_info info) { return find_matches_batch(env, info, 1); }

static napi_value js_set_views(napi_env env, napi_callback_info info) {
  ARGS(env, info, 3)
  cg_ruleset *rs; uint8_t *rows; size_t nb; uint32_t nv = 0; cg_ruleset_info ri;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  CG_CALL(env, cg_ruleset_get_info(rs, &ri));
  /* the library reads nViews rows of exactly ceil(nRules / 32) words (one word for a set without rules) */
  const size_t row_words = ri.n_rules ? ((size_t)ri.n_rules + 31) / 32 : 1;
  if (!get_ta(env, argv[1], &rows, &nb, napi_uint32_array) || napi_get_value_uint32(env, argv[2], &nv) != napi_ok || !nv || nb != (size_t)nv * row_words * 4) {
    napi_throw_type_error(env, NULL, "setViews(handle, rows: Uint32Array of nViews x ceil(nRules / 32) words, nViews)"); return NULL;
  }
  CG_CALL(env, cg_ruleset_set_views(rs, (const uint32_t *)rows, nv));
  return NULL;
}

static napi_value js_set_policy(napi_env env, napi_callback_info info) {
  ARGS(env, info, 3)
  cg_ruleset *rs; uint8_t *pol, *act; size_t np, na;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  if (!get_ta(env, argv[1], &pol, &np, napi_uint32_array) || !get_ta(env, argv[2], &act, &na, napi_uint8_array) || np / 4 != na) { napi_throw_type_error(env, NULL, "setPolicy(handle, Uint32Array, Uint8Array) of equal lengths"); return NULL; }
  CG_CALL(env, cg_ruleset_set_policy(rs, (const uint32_t *)pol, act, (uint32_t)na));
  return NULL;
}
static napi_value verdict_batch(napi_env env, napi_callback_info info, int views) {
  BATCH_ARGS(env, info, views)
  cg_ruleset *rs; uint8_t *bytes, *offp, *ids = NULL; napi_value ab, arr; void *data;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  const int64_t nn = get_batch(env, argv[1], argv[2], 0, &bytes, &offp); if (nn < 0) return NULL;
  if (views && !get_views(env, argv[3], nn, &ids)) return NULL;
  NAPI_CALL(env, napi_create_arraybuffer(env, (size_t)nn * 4, &data, &ab));
  CG_CALL(env, views ? cg_policy_verdict_batch_views(rs, bytes, (const uint32_t *)offp, ids, (uint32_t)nn, (uint32_t *)data)
                     : cg_policy_verdict_batch(rs, bytes, (const uint32_t *)offp, (uint32_t)nn, (uint32_t *)data));
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint32_array, (size_t)nn, ab, 0, &arr));
  return arr;
}
static napi_value js_verdict_batch(napi_env env, napi_callback_info info) { return verdict_batch(env, info, 0); }
static napi_value js_verdict_batch_views(napi_env env, napi_callback_info info) { return verdict_batch(env, info, 1); }

static napi_value js_set_policy_program(napi_env env, napi_callback_info info) {
  ARGS(env, info, 3)
  cg_ruleset *rs; uint8_t *prog; size_t nb; uint32_t n_atoms = 0;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  if (!get_ta(env, argv[1], &prog, &nb, napi_uint32_array) || !nb || napi_get_value_uint32(env, argv[2], &n_atoms) != napi_ok) {
    napi_throw_type_error(env, NULL, "setPolicyProgram(handle, program: Uint32Array, nAtoms)"); return NULL;
  }
  CG_CALL(env, cg_ruleset_set_policy_program(rs, (const uint32_t *)prog, (uint32_t)(nb / 4), n_atoms));
  return NULL;
}

/* the texts, their roles, the contexts' text ranges (checked here: the C call trusts them) and ceil(nAtoms / 32) atom words
 * per context, nAtoms as given to setPolicyProgram */
static napi_value js_policy_eval_batch(napi_env env, napi_callback_info info) {
  ARGS(env, info, 7)
  cg_ruleset *rs; uint8_t *bytes, *offp, *roles, *ctxp, *atoms; size_t nr, nc, na; uint32_t n_atoms = 0;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  const int64_t nn = get_batch(env, argv[1], argv[2], 0, &bytes, &offp); if (nn < 0) return NULL;
  if (!get_ta(env, argv[3], &roles, &nr, napi_uint8_array) || (int64_t)nr != nn || !get_ta(env, argv[4], &ctxp, &nc, napi_uint32_array) || nc < 4 ||
      !get_ta(env, argv[5], &atoms, &na, napi_uint32_array) || napi_get_value_uint32(env, argv[6], &n_atoms) != napi_ok) {
    napi_throw_type_error(env, NULL, "policyEvalBatch(handle, bytes, offsets, roles: Uint8Array (one per text), ctxOffsets: Uint32Array, atoms: Uint32Array, nAtoms)"); return NULL;
  }
  const uint32_t n_ctx = (uint32_t)(nc / 4 - 1), *co = (const uint32_t *)ctxp;
  for (uint32_t c = 0; c < n_ctx; c++)
    if (co[c] > co[c + 1] || co[c + 1] > (uint64_t)nn) { napi_throw_range_error(env, NULL, "ctxOffsets must be non-decreasing and end inside the texts"); return NULL; }
  if (na != (size_t)n_ctx * ((n_atoms + 31) / 32) * 4) { napi_throw_type_error(env, NULL, "atoms: ceil(nAtoms / 32) words per context"); return NULL; }
  napi_value vab, verdicts, mab, matches, out; void *vdata, *mdata;
  NAPI_CALL(env, napi_create_arraybuffer(env, (size_t)n_ctx * 4, &vdata, &vab));
  uint32_t nm = 0, cap = 1024; cg_policy_match *tmp = (cg_policy_match *)malloc(sizeof(cg_policy_match) * cap);
#define EVAL(cap) cg_policy_eval_batch(rs, bytes, (const uint32_t *)offp, nr ? roles : NULL, (uint32_t)nn, co, na ? (const uint32_t *)atoms : NULL, n_ctx, \
                                       (uint32_t *)vdata, tmp, (cap), &nm)
  int rc = tmp ? EVAL(cap) : CG_ERR_CUDA;
  if (rc == CG_ERR_CAPACITY) { cap = nm; cg_policy_match *t2 = (cg_policy_match *)realloc(tmp, sizeof(cg_policy_match) * cap); if (t2) { tmp = t2; rc = EVAL(cap); } }
#undef EVAL
  if (rc != CG_OK) { free(tmp); napi_throw_error(env, NULL, cg_last_error()); return NULL; }
  if (napi_create_arraybuffer(env, (size_t)nm * 8, &mdata, &mab) != napi_ok) { free(tmp); napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  memcpy(mdata, tmp, (size_t)nm * 8); free(tmp);
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint32_array, n_ctx, vab, 0, &verdicts));
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint32_array, (size_t)nm * 2, mab, 0, &matches));
  NAPI_CALL(env, napi_create_object(env, &out));
  NAPI_CALL(env, napi_set_named_property(env, out, "verdicts", verdicts));
  NAPI_CALL(env, napi_set_named_property(env, out, "matches", matches));
  return out;
}

static napi_value js_sha256_batch(napi_env env, napi_callback_info info) {
  ARGS(env, info, 2)
  uint8_t *bytes, *offp; napi_value ab, arr; void *data;
  const int64_t nn = get_batch(env, argv[0], argv[1], 1, &bytes, &offp); if (nn < 0) return NULL;
  NAPI_CALL(env, napi_create_arraybuffer(env, (size_t)nn * 32, &data, &ab));
  CG_CALL(env, cg_sha256_batch(bytes, (const uint64_t *)offp, (uint32_t)nn, (uint8_t *)data));
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint8_array, (size_t)nn * 32, ab, 0, &arr));
  return arr;
}

static napi_value js_merkle_root(napi_env env, napi_callback_info info) {
  ARGS(env, info, 2)
  uint8_t *bytes, *offp, root[32];
  const int64_t nn = get_batch(env, argv[0], argv[1], 1, &bytes, &offp); if (nn < 0) return NULL;
  CG_CALL(env, cg_merkle_root(bytes, (const uint64_t *)offp, (uint64_t)nn, root));
  return make_u8(env, root, 32);
}

/* ---- append-only Merkle log over the audit JSONL (src/audit-trail.ts:151-179) */
static napi_value wrap_log(napi_env env, cg_merkle_log *L) {
  napi_value h;
  if (napi_create_external(env, L, log_finalize, NULL, &h) != napi_ok) { cg_merkle_log_destroy(L); napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  return h;
}
static napi_value js_log_create(napi_env env, napi_callback_info info) {
  size_t argc = 1; napi_value argv[1]; bool keep = true; cg_merkle_log *L = NULL;
  NAPI_CALL(env, napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
  if (argc >= 1) napi_get_value_bool(env, argv[0], &keep);
  CG_CALL(env, cg_merkle_log_create(&L, keep ? 1 : 0));
  return wrap_log(env, L);
}
static napi_value js_log_create_tree(napi_env env, napi_callback_info info) {
  (void)info; cg_merkle_log *L = NULL;
  CG_CALL(env, cg_merkle_log_create_tree(&L));
  return wrap_log(env, L);
}
static napi_value js_log_restore(napi_env env, napi_callback_info info) {
  ARGS(env, info, 2)
  uint64_t n; uint8_t *f; size_t nf; cg_merkle_log *L = NULL;
  if (!get_u64(env, argv[0], &n) || !get_ta(env, argv[1], &f, &nf, napi_uint8_array) || nf % 32) { napi_throw_type_error(env, NULL, "logRestore(size, Uint8Array of 32-byte digests)"); return NULL; }
  CG_CALL(env, cg_merkle_log_restore(&L, n, f, (uint32_t)(nf / 32)));
  return wrap_log(env, L);
}
static napi_value js_log_append(napi_env env, napi_callback_info info) {
  ARGS(env, info, 3)
  cg_merkle_log *L; uint8_t *bytes, *offp;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&L));
  const int64_t nn = get_batch(env, argv[1], argv[2], 1, &bytes, &offp); if (nn < 0) return NULL;
  CG_CALL(env, cg_merkle_log_append(L, bytes, (const uint64_t *)offp, (uint64_t)nn));
  return NULL;
}
static napi_value js_log_append_jsonl(napi_env env, napi_callback_info info) {
  ARGS(env, info, 2)
  cg_merkle_log *L; uint8_t *bytes; size_t nb; uint64_t lines = 0; napi_value out;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&L));
  if (!get_ta(env, argv[1], &bytes, &nb, napi_uint8_array)) { napi_throw_type_error(env, NULL, "logAppendJsonl(log, Uint8Array)"); return NULL; }
  CG_CALL(env, cg_merkle_log_append_jsonl(L, bytes, nb, &lines));
  NAPI_CALL(env, napi_create_bigint_uint64(env, lines, &out));
  return out;
}
static napi_value js_log_reserve(napi_env env, napi_callback_info info) {
  ARGS(env, info, 3)
  cg_merkle_log *L; uint64_t a, b;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&L));
  if (!get_u64(env, argv[1], &a) || !get_u64(env, argv[2], &b)) { napi_throw_type_error(env, NULL, "logReserve(log, leaves, bytes)"); return NULL; }
  CG_CALL(env, cg_merkle_log_reserve(L, a, b));
  return NULL;
}
static napi_value js_log_size(napi_env env, napi_callback_info info) {
  ARGS(env, info, 1)
  cg_merkle_log *L; uint64_t n = 0; napi_value out;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&L));
  CG_CALL(env, cg_merkle_log_size(L, &n));
  NAPI_CALL(env, napi_create_bigint_uint64(env, n, &out));
  return out;
}
static napi_value js_log_root(napi_env env, napi_callback_info info) {
  ARGS(env, info, 1)
  cg_merkle_log *L; uint8_t root[32];
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&L));
  CG_CALL(env, cg_merkle_log_root(L, root));
  return make_u8(env, root, 32);
}
static napi_value js_log_frontier(napi_env env, napi_callback_info info) {
  ARGS(env, info, 1)
  cg_merkle_log *L; uint8_t f[64 * 32]; uint32_t k = 0;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&L));
  CG_CALL(env, cg_merkle_log_frontier(L, f, &k));
  return make_u8(env, f, (size_t)k * 32);
}
static napi_value js_log_path(napi_env env, napi_callback_info info, int consistency) {
  ARGS(env, info, 2)
  cg_merkle_log *L; uint64_t x; uint8_t p[64 * 32]; uint32_t k = 0;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&L));
  if (!get_u64(env, argv[1], &x)) { napi_throw_type_error(env, NULL, "expected (log, index | size)"); return NULL; }
  CG_CALL(env, consistency ? cg_merkle_log_consistency(L, x, p, 64, &k) : cg_merkle_log_proof(L, x, p, 64, &k));
  return make_u8(env, p, (size_t)k * 32);
}
static napi_value js_log_proof(napi_env env, napi_callback_info info) { return js_log_path(env, info, 0); }
static napi_value js_log_consistency(napi_env env, napi_callback_info info) { return js_log_path(env, info, 1); }
static napi_value js_verify_proof(napi_env env, napi_callback_info info) {
  ARGS(env, info, 5)
  uint8_t *leaf, *path, *root; size_t nl, np, nr; uint64_t index, size; int ok = 0; napi_value out;
  if (!get_ta(env, argv[0], &leaf, &nl, napi_uint8_array) || !get_u64(env, argv[1], &index) || !get_u64(env, argv[2], &size) ||
      !get_ta(env, argv[3], &path, &np, napi_uint8_array) || !get_ta(env, argv[4], &root, &nr, napi_uint8_array) || np % 32 || nr != 32) {
    napi_throw_type_error(env, NULL, "verifyProof(leaf, index, treeSize, path, root)"); return NULL; }
  CG_CALL(env, cg_merkle_verify_proof(leaf, nl, index, size, path, (uint32_t)(np / 32), root, &ok));
  NAPI_CALL(env, napi_get_boolean(env, ok != 0, &out));
  return out;
}
/* logProofs(log, BigUint64Array indices, treeSize) -> { paths: Uint8Array (m x stride x 32, stride = max(1, ceil(log2 treeSize))), lens: Uint32Array } */
static napi_value js_log_proofs(napi_env env, napi_callback_info info) {
  ARGS(env, info, 3)
  cg_merkle_log *L; uint8_t *ip; size_t ni; uint64_t size; napi_value res, paths, lens_ab, lens; void *lens_data;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&L));
  if (!get_ta(env, argv[1], &ip, &ni, napi_biguint64_array) || !get_u64(env, argv[2], &size) || ni / 8 > UINT32_MAX) {
    napi_throw_type_error(env, NULL, "logProofs(log, BigUint64Array, treeSize)"); return NULL; }
  const uint32_t m = (uint32_t)(ni / 8);
  uint32_t stride = 1; while (stride < 64 && size > (1ull << stride)) stride++;          /* ceil(log2 treeSize), at least 1 */
  uint8_t *tmp = (uint8_t *)malloc((size_t)m * stride * 32 + 32);
  if (!tmp) { napi_throw_error(env, NULL, "out of memory"); return NULL; }
  NAPI_CALL(env, napi_create_arraybuffer(env, (size_t)m * 4 + 4, &lens_data, &lens_ab));
  int rc = cg_merkle_log_proofs(L, (const uint64_t *)ip, m, size, tmp, stride, (uint32_t *)lens_data);
  if (rc != CG_OK) { free(tmp); napi_throw_error(env, NULL, cg_last_error()); return NULL; }
  paths = make_u8(env, tmp, (size_t)m * stride * 32);
  free(tmp);
  if (!paths) { napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint32_array, m, lens_ab, 0, &lens));
  NAPI_CALL(env, napi_create_object(env, &res));
  NAPI_CALL(env, napi_set_named_property(env, res, "paths", paths)); NAPI_CALL(env, napi_set_named_property(env, res, "lens", lens));
  return res;
}
static napi_value js_log_consistency_between(napi_env env, napi_callback_info info) {
  ARGS(env, info, 3)
  cg_merkle_log *L; uint64_t a, b; uint8_t p[65 * 32]; uint32_t k = 0;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&L));
  if (!get_u64(env, argv[1], &a) || !get_u64(env, argv[2], &b)) { napi_throw_type_error(env, NULL, "logConsistencyBetween(log, firstSize, secondSize)"); return NULL; }
  CG_CALL(env, cg_merkle_log_consistency_between(L, a, b, p, 65, &k));
  return make_u8(env, p, (size_t)k * 32);
}
/* verifyProofs(leafBytes, BigUint64Array leafOffsets, BigUint64Array indices, treeSize, paths, Uint32Array lens, stride, root) -> Uint8Array */
static napi_value js_verify_proofs(napi_env env, napi_callback_info info) {
  ARGS(env, info, 8)
  uint8_t *bytes, *offp, *ip, *paths, *lp, *root; size_t ni, np, nl, nr; uint64_t size; uint32_t stride;
  const int64_t nn = get_batch(env, argv[0], argv[1], 1, &bytes, &offp); if (nn < 0) return NULL;
  if (!get_ta(env, argv[2], &ip, &ni, napi_biguint64_array) || !get_u64(env, argv[3], &size) || !get_ta(env, argv[4], &paths, &np, napi_uint8_array) ||
      !get_ta(env, argv[5], &lp, &nl, napi_uint32_array) || napi_get_value_uint32(env, argv[6], &stride) != napi_ok ||
      !get_ta(env, argv[7], &root, &nr, napi_uint8_array) || nr != 32 || ni / 8 != (size_t)nn || nl / 4 != (size_t)nn ||
      np < (size_t)nn * stride * 32 || nn > UINT32_MAX) {
    napi_throw_type_error(env, NULL, "verifyProofs(leafBytes, leafOffsets, indices, treeSize, paths, lens, stride, root)"); return NULL; }
  napi_value ab, out; void *ok;
  NAPI_CALL(env, napi_create_arraybuffer(env, (size_t)nn + 1, &ok, &ab));
  CG_CALL(env, cg_merkle_verify_proofs(bytes, (const uint64_t *)offp, (const uint64_t *)ip, (uint32_t)nn, size, paths, stride, (const uint32_t *)lp, root, (uint8_t *)ok));
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint8_array, (size_t)nn, ab, 0, &out));
  return out;
}
static napi_value js_verify_consistency(napi_env env, napi_callback_info info) {
  ARGS(env, info, 5)
  uint8_t *r1, *r2, *path; size_t n1, n2, np; uint64_t a, b; int ok = 0; napi_value out;
  if (!get_u64(env, argv[0], &a) || !get_u64(env, argv[1], &b) || !get_ta(env, argv[2], &r1, &n1, napi_uint8_array) || !get_ta(env, argv[3], &r2, &n2, napi_uint8_array) ||
      !get_ta(env, argv[4], &path, &np, napi_uint8_array) || n1 != 32 || n2 != 32 || np % 32) {
    napi_throw_type_error(env, NULL, "verifyConsistency(firstSize, secondSize, rootFirst, rootSecond, path)"); return NULL; }
  CG_CALL(env, cg_merkle_verify_consistency(a, b, r1, r2, path, (uint32_t)(np / 32), &ok));
  NAPI_CALL(env, napi_get_boolean(env, ok != 0, &out));
  return out;
}

static napi_value redact_batch(napi_env env, napi_callback_info info, int views) {
  BATCH_ARGS(env, info, views)
  cg_ruleset *rs; uint8_t *bytes, *offp, *ids = NULL;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  const int64_t nn = get_batch(env, argv[1], argv[2], 0, &bytes, &offp); if (nn < 0) return NULL;
  if (views && !get_views(env, argv[3], nn, &ids)) return NULL;
  uint32_t n = (uint32_t)nn, ns = 0, cap_spans = 256; uint64_t need = 0, cap_bytes = (uint64_t)((const uint32_t *)offp)[n] + 4096;
  napi_value off_ab, off_arr; void *off_data;
  NAPI_CALL(env, napi_create_arraybuffer(env, (size_t)(n + 1) * 4, &off_data, &off_ab));
  uint8_t *out = NULL, *dig = NULL; cg_span *spans = NULL; int rc = CG_ERR_CUDA;
  for (;;) {
    uint8_t *o2 = (uint8_t *)realloc(out, cap_bytes + 64); cg_span *s2 = (cg_span *)realloc(spans, sizeof(cg_span) * cap_spans); uint8_t *d2 = (uint8_t *)realloc(dig, (size_t)cap_spans * 32);
    if (o2) out = o2;
    if (s2) spans = s2;
    if (d2) dig = d2;
    if (!o2 || !s2 || !d2) break;
    rc = views ? cg_redact_batch_views(rs, bytes, (const uint32_t *)offp, ids, n, out, cap_bytes, &need, (uint32_t *)off_data, spans, cap_spans, &ns, dig)
               : cg_redact_batch(rs, bytes, (const uint32_t *)offp, n, out, cap_bytes, &need, (uint32_t *)off_data, spans, cap_spans, &ns, dig);
    if (rc == CG_ERR_CAPACITY && (need > cap_bytes || ns > cap_spans)) { if (need > cap_bytes) cap_bytes = need; if (ns > cap_spans) cap_spans = ns; continue; }
    break;
  }
  if (rc != CG_OK) { free(out); free(spans); free(dig); napi_throw_error(env, NULL, cg_last_error()); return NULL; }
  napi_value res = NULL, b_arr = make_u8(env, out, (size_t)need), d_arr = make_u8(env, dig, (size_t)ns * 32), s_ab, s_arr = NULL; void *p;
  int ok = b_arr && d_arr && napi_create_arraybuffer(env, (size_t)ns * sizeof(cg_span), &p, &s_ab) == napi_ok;
  if (ok) { memcpy(p, spans, (size_t)ns * sizeof(cg_span)); ok = napi_create_typedarray(env, napi_uint32_array, (size_t)ns * 6, s_ab, 0, &s_arr) == napi_ok; }
  free(out); free(spans); free(dig);
  if (!ok || napi_create_typedarray(env, napi_uint32_array, (size_t)n + 1, off_ab, 0, &off_arr) != napi_ok || napi_create_object(env, &res) != napi_ok) { napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  NAPI_CALL(env, napi_set_named_property(env, res, "bytes", b_arr)); NAPI_CALL(env, napi_set_named_property(env, res, "offsets", off_arr));
  NAPI_CALL(env, napi_set_named_property(env, res, "spans", s_arr)); NAPI_CALL(env, napi_set_named_property(env, res, "digests", d_arr));
  return res;
}
static napi_value js_redact_batch(napi_env env, napi_callback_info info) { return redact_batch(env, info, 0); }
static napi_value js_redact_batch_views(napi_env env, napi_callback_info info) { return redact_batch(env, info, 1); }

/* ---- one message, blocking: the synchronous hooks' findMatches / scanString (cg_find_matches_one / cg_redact_one) */
static uint8_t one_empty[1];                          /* the message of an empty Uint8Array */
static napi_value js_find_matches_one(napi_env env, napi_callback_info info) {
  ARGS(env, info, 2)
  cg_ruleset *rs; uint8_t *bytes; size_t nb;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  if (!get_ta(env, argv[1], &bytes, &nb, napi_uint8_array) || nb > UINT32_MAX) { napi_throw_type_error(env, NULL, "findMatchesOne(handle, Uint8Array)"); return NULL; }
  if (!nb) bytes = one_empty;                       /* an empty typed array may report NULL: the C ABI rejects a NULL message */
  uint32_t ns = 0, cap = 64; cg_span *tmp = (cg_span *)malloc(sizeof(cg_span) * cap);
  int rc = tmp ? cg_find_matches_one(rs, bytes, (uint32_t)nb, tmp, cap, &ns) : CG_ERR_NOMEM;
  if (rc == CG_ERR_CAPACITY) { cap = ns; cg_span *t2 = (cg_span *)realloc(tmp, sizeof(cg_span) * cap); if (t2) { tmp = t2; rc = cg_find_matches_one(rs, bytes, (uint32_t)nb, tmp, cap, &ns); } }
  if (rc != CG_OK) { free(tmp); napi_throw_error(env, NULL, rc == CG_ERR_NOMEM ? "out of host memory" : cg_last_error()); return NULL; }
  napi_value ab, arr; void *data;
  if (napi_create_arraybuffer(env, (size_t)ns * sizeof(cg_span), &data, &ab) != napi_ok) { free(tmp); napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  memcpy(data, tmp, (size_t)ns * sizeof(cg_span)); free(tmp);
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint32_array, (size_t)ns * 6, ab, 0, &arr));
  return arr;
}

static napi_value js_redact_one(napi_env env, napi_callback_info info) {
  ARGS(env, info, 2)
  cg_ruleset *rs; uint8_t *bytes; size_t nb;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  if (!get_ta(env, argv[1], &bytes, &nb, napi_uint8_array) || nb > UINT32_MAX) { napi_throw_type_error(env, NULL, "redactOne(handle, Uint8Array)"); return NULL; }
  if (!nb) bytes = one_empty;
  uint32_t ns = 0, cap_spans = 64; uint64_t need = 0, cap_bytes = (uint64_t)nb + 1024;
  uint8_t *out = NULL, *dig = NULL; cg_span *spans = NULL; int rc = CG_ERR_NOMEM;
  for (;;) {
    uint8_t *o2 = (uint8_t *)realloc(out, cap_bytes); cg_span *s2 = (cg_span *)realloc(spans, sizeof(cg_span) * cap_spans); uint8_t *d2 = (uint8_t *)realloc(dig, (size_t)cap_spans * 32);
    if (o2) out = o2;
    if (s2) spans = s2;
    if (d2) dig = d2;
    if (!o2 || !s2 || !d2) { rc = CG_ERR_NOMEM; break; }
    rc = cg_redact_one(rs, bytes, (uint32_t)nb, out, cap_bytes, &need, spans, cap_spans, &ns, dig);
    if (rc == CG_ERR_CAPACITY && (need > cap_bytes || ns > cap_spans)) { if (need > cap_bytes) cap_bytes = need; if (ns > cap_spans) cap_spans = ns; continue; }
    break;
  }
  if (rc != CG_OK) { free(out); free(spans); free(dig); napi_throw_error(env, NULL, rc == CG_ERR_NOMEM ? "out of host memory" : cg_last_error()); return NULL; }
  napi_value res = NULL, b_arr = make_u8(env, out, (size_t)need), d_arr = make_u8(env, dig, (size_t)ns * 32), s_ab, s_arr = NULL; void *p;
  int ok = b_arr && d_arr && napi_create_arraybuffer(env, (size_t)ns * sizeof(cg_span), &p, &s_ab) == napi_ok;
  if (ok) { memcpy(p, spans, (size_t)ns * sizeof(cg_span)); ok = napi_create_typedarray(env, napi_uint32_array, (size_t)ns * 6, s_ab, 0, &s_arr) == napi_ok; }
  free(out); free(spans); free(dig);
  if (!ok || napi_create_object(env, &res) != napi_ok) { napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  NAPI_CALL(env, napi_set_named_property(env, res, "bytes", b_arr));
  NAPI_CALL(env, napi_set_named_property(env, res, "spans", s_arr)); NAPI_CALL(env, napi_set_named_property(env, res, "digests", d_arr));
  return res;
}

/* ---- the few strings of one scanned value, blocking: RedactionEngine.scan's findMatches / scanString for all its string
 * leaves in one device round trip (cg_find_matches_few / cg_redact_few); results as findMatchesBatch / redactBatch */
static napi_value js_find_matches_few(napi_env env, napi_callback_info info) {
  BATCH_ARGS(env, info, 0)
  cg_ruleset *rs; uint8_t *bytes, *offp;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  const int64_t nn = get_batch(env, argv[1], argv[2], 0, &bytes, &offp); if (nn < 0) return NULL;
  const uint32_t n = (uint32_t)nn;
  if (!bytes) bytes = one_empty;                    /* an empty typed array may report NULL: the C ABI rejects a NULL byte buffer */
  uint32_t ns = 0, cap = 64; cg_span *tmp = (cg_span *)malloc(sizeof(cg_span) * cap);
  int rc = tmp ? cg_find_matches_few(rs, bytes, (const uint32_t *)offp, n, tmp, cap, &ns) : CG_ERR_NOMEM;
  if (rc == CG_ERR_CAPACITY) { cap = ns; cg_span *t2 = (cg_span *)realloc(tmp, sizeof(cg_span) * cap); if (t2) { tmp = t2; rc = cg_find_matches_few(rs, bytes, (const uint32_t *)offp, n, tmp, cap, &ns); } }
  if (rc != CG_OK) { free(tmp); napi_throw_error(env, NULL, rc == CG_ERR_NOMEM ? "out of host memory" : cg_last_error()); return NULL; }
  napi_value ab, arr; void *data;
  if (napi_create_arraybuffer(env, (size_t)ns * sizeof(cg_span), &data, &ab) != napi_ok) { free(tmp); napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  memcpy(data, tmp, (size_t)ns * sizeof(cg_span)); free(tmp);
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint32_array, (size_t)ns * 6, ab, 0, &arr));
  return arr;
}

static napi_value js_redact_few(napi_env env, napi_callback_info info) {
  BATCH_ARGS(env, info, 0)
  cg_ruleset *rs; uint8_t *bytes, *offp;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  const int64_t nn = get_batch(env, argv[1], argv[2], 0, &bytes, &offp); if (nn < 0) return NULL;
  const uint32_t n = (uint32_t)nn;
  if (!bytes) bytes = one_empty;
  const uint32_t *off = (const uint32_t *)offp;
  uint32_t ns = 0, cap_spans = 64; uint64_t need = 0, cap_bytes = (uint64_t)(off[n] - off[0]) + 1024;
  napi_value off_ab, off_arr; void *off_data;
  NAPI_CALL(env, napi_create_arraybuffer(env, (size_t)(n + 1) * 4, &off_data, &off_ab));
  uint8_t *out = NULL, *dig = NULL; cg_span *spans = NULL; int rc = CG_ERR_NOMEM;
  for (;;) {
    uint8_t *o2 = (uint8_t *)realloc(out, cap_bytes + 64); cg_span *s2 = (cg_span *)realloc(spans, sizeof(cg_span) * cap_spans); uint8_t *d2 = (uint8_t *)realloc(dig, (size_t)cap_spans * 32);
    if (o2) out = o2;
    if (s2) spans = s2;
    if (d2) dig = d2;
    if (!o2 || !s2 || !d2) { rc = CG_ERR_NOMEM; break; }
    rc = cg_redact_few(rs, bytes, off, n, out, cap_bytes, &need, (uint32_t *)off_data, spans, cap_spans, &ns, dig);
    if (rc == CG_ERR_CAPACITY && (need > cap_bytes || ns > cap_spans)) { if (need > cap_bytes) cap_bytes = need; if (ns > cap_spans) cap_spans = ns; continue; }
    break;
  }
  if (rc != CG_OK) { free(out); free(spans); free(dig); napi_throw_error(env, NULL, rc == CG_ERR_NOMEM ? "out of host memory" : cg_last_error()); return NULL; }
  napi_value res = NULL, b_arr = make_u8(env, out, (size_t)need), d_arr = make_u8(env, dig, (size_t)ns * 32), s_ab, s_arr = NULL; void *p;
  int ok = b_arr && d_arr && napi_create_arraybuffer(env, (size_t)ns * sizeof(cg_span), &p, &s_ab) == napi_ok;
  if (ok) { memcpy(p, spans, (size_t)ns * sizeof(cg_span)); ok = napi_create_typedarray(env, napi_uint32_array, (size_t)ns * 6, s_ab, 0, &s_arr) == napi_ok; }
  free(out); free(spans); free(dig);
  if (!ok || napi_create_typedarray(env, napi_uint32_array, (size_t)n + 1, off_ab, 0, &off_arr) != napi_ok || napi_create_object(env, &res) != napi_ok) { napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  NAPI_CALL(env, napi_set_named_property(env, res, "bytes", b_arr)); NAPI_CALL(env, napi_set_named_property(env, res, "offsets", off_arr));
  NAPI_CALL(env, napi_set_named_property(env, res, "spans", s_arr)); NAPI_CALL(env, napi_set_named_property(env, res, "digests", d_arr));
  return res;
}

/* one context owning every text (cg_policy_eval_one): the texts, their roles and ceil(nAtoms / 32) atom words, nAtoms as given to
 * setPolicyProgram -> {verdict, rules} */
static napi_value js_policy_eval_one(napi_env env, napi_callback_info info) {
  ARGS(env, info, 6)
  cg_ruleset *rs; uint8_t *bytes, *offp, *roles, *atoms; size_t nb, nr, na; uint32_t n_atoms = 0;
  NAPI_CALL(env, napi_get_value_external(env, argv[0], (void **)&rs));
  const int64_t nn = get_batch(env, argv[1], argv[2], 0, &bytes, &offp); if (nn < 0) return NULL;
  if (!get_ta(env, argv[1], &bytes, &nb, napi_uint8_array) || !get_ta(env, argv[3], &roles, &nr, napi_uint8_array) || (int64_t)nr != nn ||
      !get_ta(env, argv[4], &atoms, &na, napi_uint32_array) || napi_get_value_uint32(env, argv[5], &n_atoms) != napi_ok) {
    napi_throw_type_error(env, NULL, "policyEvalOne(handle, bytes, offsets, roles: Uint8Array (one per text), atoms: Uint32Array, nAtoms)"); return NULL;
  }
  if (na != (size_t)((n_atoms + 31) / 32) * 4) { napi_throw_type_error(env, NULL, "atoms: ceil(nAtoms / 32) words"); return NULL; }
  if (!nb) bytes = one_empty;                       /* an empty typed array may report NULL: the C ABI rejects a NULL text buffer */
  uint32_t verdict = 0, nm = 0, cap = 64; uint32_t *tmp = (uint32_t *)malloc(sizeof(uint32_t) * cap);
#define EVAL(cap) cg_policy_eval_one(rs, bytes, (const uint32_t *)offp, nr ? roles : NULL, (uint32_t)nn, na ? (const uint32_t *)atoms : NULL, &verdict, \
                                     tmp, (cap), &nm)
  int rc = tmp ? EVAL(cap) : CG_ERR_NOMEM;
  if (rc == CG_ERR_CAPACITY && nm > cap) { cap = nm; uint32_t *t2 = (uint32_t *)realloc(tmp, sizeof(uint32_t) * cap); if (t2) { tmp = t2; rc = EVAL(cap); } }
#undef EVAL
  if (rc != CG_OK) { free(tmp); napi_throw_error(env, NULL, rc == CG_ERR_NOMEM ? "out of host memory" : cg_last_error()); return NULL; }
  napi_value ab, rules, v, out; void *data;
  if (napi_create_arraybuffer(env, (size_t)nm * 4, &data, &ab) != napi_ok) { free(tmp); napi_throw_error(env, NULL, "N-API call failed"); return NULL; }
  memcpy(data, tmp, (size_t)nm * 4); free(tmp);
  NAPI_CALL(env, napi_create_typedarray(env, napi_uint32_array, nm, ab, 0, &rules));
  NAPI_CALL(env, napi_create_double(env, (double)verdict, &v));   /* (a uint32 is exact as a JS number) */
  NAPI_CALL(env, napi_create_object(env, &out));
  NAPI_CALL(env, napi_set_named_property(env, out, "verdict", v));
  NAPI_CALL(env, napi_set_named_property(env, out, "rules", rules));
  return out;
}

static napi_value module_init(napi_env env, napi_value exports) {
  napi_property_descriptor d[] = {
#define FN(name, fn) {name, NULL, fn, NULL, NULL, NULL, napi_default, NULL}
    FN("init", js_init), FN("shutdown", js_shutdown), FN("stats", js_stats), FN("ruleCheck", js_rule_check),
    FN("createRuleset", js_create_ruleset), FN("scanBatch", js_scan_batch), FN("scanOne", js_scan_one),
    FN("findMatchesBatch", js_find_matches_batch), FN("redactBatch", js_redact_batch),
    FN("findMatchesOne", js_find_matches_one), FN("redactOne", js_redact_one),
    FN("findMatchesFew", js_find_matches_few), FN("redactFew", js_redact_few),
    FN("setPolicy", js_set_policy), FN("verdictBatch", js_verdict_batch),
    FN("setViews", js_set_views), FN("scanBatchViews", js_scan_batch_views), FN("findMatchesBatchViews", js_find_matches_batch_views),
    FN("redactBatchViews", js_redact_batch_views), FN("verdictBatchViews", js_verdict_batch_views),
    FN("setPolicyProgram", js_set_policy_program), FN("policyEvalBatch", js_policy_eval_batch), FN("policyEvalOne", js_policy_eval_one),
    FN("sha256Batch", js_sha256_batch), FN("merkleRoot", js_merkle_root),
    FN("logCreate", js_log_create), FN("logRestore", js_log_restore), FN("logAppend", js_log_append), FN("logAppendJsonl", js_log_append_jsonl),
    FN("logReserve", js_log_reserve), FN("logSize", js_log_size), FN("logRoot", js_log_root), FN("logFrontier", js_log_frontier),
    FN("logProof", js_log_proof), FN("logConsistency", js_log_consistency), FN("verifyProof", js_verify_proof), FN("verifyConsistency", js_verify_consistency),
    FN("logCreateTree", js_log_create_tree), FN("logProofs", js_log_proofs), FN("logConsistencyBetween", js_log_consistency_between),
    FN("verifyProofs", js_verify_proofs),
#undef FN
  };
  if (napi_define_properties(env, exports, sizeof d / sizeof d[0], d) != napi_ok) return NULL;
  return exports;
}

NAPI_MODULE(openclaw_gov, module_init)
