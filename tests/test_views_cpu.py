"""CPU tier for per-message views (cg_ruleset_set_views and the *_views twins): the C ABI header, the library's exports and
the N-API shim bind the new symbols; the plugin maps exempt-tool flags and policy scopes to view rows as a plain
restatement does; the GPU tests' per-view oracle agrees with the oracle's policy hits filtered by view on the built-ins."""
import os
import re

import numpy as np

from test_gpu_views import ViewOracle, case_batch, view_sets
from test_gpu_parity import oracle_policy
from vainplex_openclaw_b200 import _native as N
from vainplex_openclaw_b200 import plugin as P
from vainplex_openclaw_b200.workload import BUILTIN_RULES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_TWINS = ["cg_scan_batch_views", "cg_find_matches_batch_views", "cg_redact_batch_views", "cg_policy_verdict_batch_views"]
DEVICE_TWINS = ["cg_scan_hits_batch_device_views", "cg_find_matches_batch_device_views", "cg_redact_batch_device_views",
                "cg_policy_verdict_batch_device_views"]
NEW = ["cg_ruleset_set_views"] + HOST_TWINS + DEVICE_TWINS


def test_header_exports_and_napi_bind_the_views_calls():
    hdr = open(os.path.join(ROOT, "include", "openclaw_gov.h")).read()
    for fn in NEW:
        assert re.search(r"CG_API int %s\(" % fn, hdr), fn
        assert fn in N.EXPORTS, fn
    L = N.load()
    assert all(hasattr(L, fn) for fn in NEW)
    # each twin takes the views right after the offsets and otherwise the original's parameters
    decl = lambda fn: re.sub(r"\s+", " ", re.search(r"CG_API int %s\((.*?)\);" % fn, hdr, re.S).group(1)).split(", ")
    for fn in HOST_TWINS + DEVICE_TWINS:
        orig = fn[:-len("_views")]
        a, b = decl(orig), decl(fn)
        at = 3
        assert b[:at] == a[:at] and b[at + 1:] == a[at:], fn
        assert b[at] == ("const uint8_t *views" if fn in HOST_TWINS else "const void *d_views"), fn
    src = open(os.path.join(ROOT, "napi", "openclaw_gov_napi.c")).read()
    for fn in ["cg_ruleset_set_views"] + HOST_TWINS:
        assert fn + "(" in src, fn
    for js in ("setViews", "scanBatchViews", "findMatchesBatchViews", "redactBatchViews", "verdictBatchViews"):
        assert 'FN("%s"' % js in src, js
        assert js + "(" in open(os.path.join(ROOT, "napi", "gpu-backend.ts")).read(), js
    assert "_device_views" not in src                          # JavaScript holds no device pointers


def test_view_rows_restated():
    rows = N.view_rows([[0, 5, 31, 32, 39], [], [39]], 40)
    want = np.zeros((3, 2), np.uint32)
    for v, rl in enumerate([[0, 5, 31, 32, 39], [], [39]]):
        for r in rl:
            want[v, r // 32] |= np.uint32(1 << (r % 32))
    assert np.array_equal(rows, want)


def test_credential_views_restated():
    """the redaction rule set with both views: the registry's patterns, then the credential built-ins it left out; the
    credential view holds every credential built-in, in BUILTIN_RULES order, and nothing else"""
    cred_ids = [pid for pid, cat, _s, _f in BUILTIN_RULES if cat == 0]
    for cats in (["credential", "pii", "financial"], ["pii"], ["financial", "pii"], ["credential"], []):
        reg = P.PatternRegistry(cats, [{"name": "x", "regex": "ab+c", "category": "custom"}])
        ext, full, cred = P.credential_views(reg.patterns)
        assert ext[:len(reg.patterns)] == reg.patterns and full == list(range(len(reg.patterns)))
        assert [ext[i]["id"] for i in cred] == cred_ids
        assert [p["id"] for p in ext[len(reg.patterns):]] == ([] if "credential" in cats else cred_ids)
        ce = P.PatternRegistry(["credential"], [])
        assert [(ext[i]["source"], ext[i]["flags"]) for i in cred] == [(p["source"], p["flags"]) for p in ce.patterns]


def test_scope_views_restated():
    """one view per distinct in-scope policy set of the batch, holding the patterns of those policies"""
    rng = np.random.default_rng(3)
    agents, channels = ["a", "b", "c", None], ["slack", "mail", "web", None]
    for trial in range(20):
        pols = []
        for i in range(int(rng.integers(1, 8))):
            scope = {}
            if rng.random() < 0.5:
                scope["excludeAgents"] = [a for a in agents[:3] if rng.random() < 0.4]
            if rng.random() < 0.5:
                scope["channels"] = [c for c in channels[:3] if rng.random() < 0.5]
            pols.append({"id": "p%d" % i, "scope": scope})
        pattern_policy = sorted(int(x) for x in rng.integers(0, len(pols), int(rng.integers(1, 20))))
        ctxs = [{"agentId": agents[int(rng.integers(4))], "channel": channels[int(rng.integers(4))]} for _ in range(30)]
        views, ids = P.scope_views(pols, pattern_policy, ctxs)
        for ctx, v in zip(ctxs, ids):
            ok = []
            for pi, p in enumerate(pols):
                sc = p["scope"]
                if ctx["agentId"] in sc.get("excludeAgents", []):
                    continue
                if sc.get("channels") and ctx["channel"] not in sc["channels"]:
                    continue
                ok.append(pi)
            assert views[v] == [k for k, pi in enumerate(pattern_policy) if pi in ok]
        assert sorted(set(ids)) == list(range(len(views)))


def test_per_view_oracle_equals_filtered_policy_hits(oracle):
    """words and hits of the per-view oracle == the oracle's hits over all rules filtered by each message's view (valid for
    RegExp.test, which decides every rule on its own), on the built-ins' member batch"""
    rules, _opt, msgs = case_batch(N, "builtins")
    views = view_sets(rules, seed=17)
    ids = np.random.default_rng(2).integers(0, len(views), len(msgs)).astype(np.uint8)
    words, hits, _spans = ViewOracle(oracle, rules).of(msgs, ids, views)
    data, off = N.pack(msgs)
    _, all_hits = oracle_policy(oracle, rules, data, off)
    keep = [(m, r) for m, r in all_hits if r in set(views[ids[m]])]
    assert hits == keep and len(keep) > 100
    per = {}
    for m, r in keep:
        per.setdefault(m, []).append(r)
    want = np.array([(1 << 63) | (len(per[m]) << 32) | per[m][0] if m in per else 0 for m in range(len(msgs))], np.uint64)
    assert np.array_equal(words, want)


NAPI_SET_VIEWS_HARNESS = r'''
#include <stdbool.h>
#include <stdio.h>
#include "openclaw_gov_napi.c"
/* just enough of N-API and of the C ABI for js_set_views; every other symbol stays unresolved and is never called */
enum { K_EXT, K_NUM, K_TA };
struct napi_value__ { int kind; void *ext; uint32_t u32; napi_typedarray_type t; size_t len; void *data; };
static napi_value g_argv[3]; static int g_thrown; static uint32_t g_n_rules, g_set_nv; static int g_set_calls;
napi_status napi_get_cb_info(napi_env e, napi_callback_info i, size_t *argc, napi_value *argv, napi_value *t, void **d) {
  (void)e; (void)i; (void)t; (void)d; for (size_t k = 0; k < *argc && k < 3; k++) argv[k] = g_argv[k]; *argc = 3; return napi_ok; }
napi_status napi_get_value_external(napi_env e, napi_value v, void **r) { (void)e; if (v->kind != K_EXT) return napi_invalid_arg; *r = v->ext; return napi_ok; }
napi_status napi_get_value_uint32(napi_env e, napi_value v, uint32_t *r) { (void)e; if (v->kind != K_NUM) return napi_invalid_arg; *r = v->u32; return napi_ok; }
napi_status napi_is_typedarray(napi_env e, napi_value v, bool *r) { (void)e; *r = v->kind == K_TA; return napi_ok; }
napi_status napi_get_typedarray_info(napi_env e, napi_value v, napi_typedarray_type *t, size_t *len, void **data, napi_value *ab, size_t *off) {
  (void)e; *t = v->t; *len = v->len; *data = v->data; *ab = NULL; *off = 0; return napi_ok; }
napi_status napi_throw_type_error(napi_env e, const char *c, const char *m) { (void)e; (void)c; (void)m; g_thrown = 1; return napi_ok; }
napi_status napi_throw_error(napi_env e, const char *c, const char *m) { (void)e; (void)c; (void)m; g_thrown = 1; return napi_ok; }
const char *cg_last_error(void) { return ""; }
int cg_ruleset_get_info(const cg_ruleset *rs, cg_ruleset_info *o) { (void)rs; memset(o, 0, sizeof *o); o->n_rules = g_n_rules; return CG_OK; }
int cg_ruleset_set_views(cg_ruleset *rs, const uint32_t *rows, uint32_t n) { (void)rs; (void)rows; g_set_calls++; g_set_nv = n; return CG_OK; }
/* one setViews call: rules in the set, words in the rows array, nViews -> "thrown calls nViews" */
static void one(uint32_t n_rules, size_t words, uint32_t nv) {
  static uint32_t rows[64]; static int dummy;
  struct napi_value__ h = {K_EXT, &dummy, 0, 0, 0, NULL}, r = {K_TA, NULL, 0, napi_uint32_array, words, rows}, n = {K_NUM, NULL, nv, 0, 0, NULL};
  g_argv[0] = &h; g_argv[1] = &r; g_argv[2] = &n; g_n_rules = n_rules; g_thrown = g_set_calls = 0; g_set_nv = 0;
  js_set_views(NULL, NULL);
  printf("%d %d %u\n", g_thrown, g_set_calls, g_set_nv);
}
int main(int argc, char **argv) {
  for (int i = 1; i + 2 < argc; i += 3) one((uint32_t)atoi(argv[i]), (size_t)atoi(argv[i + 1]), (uint32_t)atoi(argv[i + 2]));
  return 0;
}
'''


def test_napi_set_views_checks_the_rows_length(tmp_path):
    """setViews passes the rows to the library only when the array holds exactly nViews rows of ceil(nRules / 32) words
    (the C call has no length): shorter arrays, wider rows and a zero nViews throw before anything is read.  Runs the
    shim's js_set_views with a minimal N-API and C ABI behind it."""
    import subprocess
    src, exe = tmp_path / "set_views.c", tmp_path / "set_views"
    src.write_text(NAPI_SET_VIEWS_HARNESS)
    r = subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-I" + os.path.join(ROOT, "napi"), "-I" + os.path.join(ROOT, "napi", "stub"),
                        "-I" + os.path.join(ROOT, "include"), "-Wl,--unresolved-symbols=ignore-all", "-o", str(exe), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    cases = [(40, 1, 1), (40, 2, 1), (40, 3, 1), (40, 8, 2), (40, 4, 2), (40, 6, 2), (40, 0, 0), (32, 1, 1), (33, 1, 1),
             (33, 2, 1), (0, 1, 1), (0, 0, 1), (5000, 157, 1), (5000, 156, 1)]
    out = subprocess.run([str(exe)] + [str(x) for c in cases for x in c], capture_output=True, text=True, check=True).stdout.split("\n")
    for (n_rules, words, nv), line in zip(cases, out):
        rw = max(1, (n_rules + 31) // 32)
        ok = nv > 0 and words == nv * rw
        assert line == ("0 1 %d" % nv if ok else "1 0 0"), (n_rules, words, nv, line)


def test_python_view_ids_are_counted():
    assert list(N._ids([0, 1, 2], 3)) == [0, 1, 2]
    for bad in ([0, 1], [0, 1, 2, 3], []):
        try:
            N._ids(bad, 3)
        except ValueError:
            continue
        raise AssertionError(bad)
