"""cg_policy_eval_one without a device: declared and exported, bound by the N-API shim (with the empty-array guard) and
called by the TypeScript glue, and CG_ERR_NOT_INITIALIZED before cg_init with nothing written."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def test_declared_and_exported():
    from vainplex_openclaw_b200 import _native as N
    hdr = open(os.path.join(ROOT, "include", "openclaw_gov.h")).read()
    assert re.search(r"CG_API\s+int\s+cg_policy_eval_one\s*\(", hdr)
    assert "cg_policy_eval_one" in N.EXPORTS
    assert hasattr(N.load(), "cg_policy_eval_one")
    assert hasattr(N.Ruleset, "eval_one")
    from vainplex_openclaw_b200 import plugin as P
    assert hasattr(P.PolicyEvaluator, "verdict_one")


def test_napi_shim_binds_policy_eval_one_with_the_null_guard():
    src = open(os.path.join(ROOT, "napi", "openclaw_gov_napi.c")).read()
    assert 'FN("policyEvalOne", js_policy_eval_one)' in src
    body = src[src.index("static napi_value js_policy_eval_one("):]
    body = body[:body.index("\n}\n")]
    guard = re.search(r"if \(!nb\) bytes = (\w+);", body)
    assert guard and body.index(guard.group(0)) < body.index("cg_policy_eval_one(")
    assert re.search(r"static uint8_t %s\[1\];" % guard.group(1), src)
    ts = open(os.path.join(ROOT, "napi", "gpu-backend.ts")).read()
    assert "addon.policyEvalOne(" in ts and "policyEvalOne(handle: unknown" in ts and "class GpuPolicyEvaluator" in ts


def test_before_init_is_not_initialized_and_writes_nothing():
    # a fresh process that never calls cg_init (with or without a device: the call must not initialise anything)
    code = ("import sys, ctypes as C; sys.path.insert(0, %r)\n"
            "from vainplex_openclaw_b200 import _native as N\n"
            "L = N.load()\n"
            "v, n = C.c_uint32(7), C.c_uint32(7)\n"
            "off = (C.c_uint32 * 2)(0, 3); roles = (C.c_uint8 * 1)(0); atoms = (C.c_uint32 * 1)(0); rules = (C.c_uint32 * 4)(7, 7, 7, 7)\n"
            "a = L.cg_policy_eval_one(None, b'abc', off, roles, 1, atoms, C.byref(v), rules, 4, C.byref(n))\n"
            "b = L.cg_policy_eval_one(None, None, None, None, 0, None, C.byref(v), rules, 4, C.byref(n))\n"
            "print(a, b, v.value, n.value, list(rules))\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["-2", "-2", "7", "7", "[7,", "7,", "7,", "7]"]
