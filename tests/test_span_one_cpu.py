"""The single-message span calls (cg_find_matches_one / cg_redact_one) without a device: exported, bound by the N-API
shim, and CG_ERR_NOT_INITIALIZED before cg_init."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def test_single_message_span_calls_are_declared_and_exported():
    from vainplex_openclaw_b200 import _native as N
    hdr = open(os.path.join(ROOT, "include", "openclaw_gov.h")).read()
    for name in ("cg_find_matches_one", "cg_redact_one"):
        assert re.search(r"CG_API\s+int\s+%s\s*\(" % name, hdr), name
        assert name in N.EXPORTS
        assert hasattr(N.load(), name)


def test_napi_shim_binds_the_single_message_calls():
    src = open(os.path.join(ROOT, "napi", "openclaw_gov_napi.c")).read()
    assert "cg_find_matches_one(" in src and "cg_redact_one(" in src
    assert 'FN("findMatchesOne", js_find_matches_one)' in src and 'FN("redactOne", js_redact_one)' in src
    ts = open(os.path.join(ROOT, "napi", "gpu-backend.ts")).read()
    assert "addon.findMatchesOne(" in ts


def test_napi_shim_never_passes_null_for_an_empty_message():
    """N-API may report NULL as the data pointer of an empty typed array (TextEncoder.encode('')), and the C ABI rejects a
    NULL message whatever its length: both single-message shims substitute a real pointer before calling it"""
    src = open(os.path.join(ROOT, "napi", "openclaw_gov_napi.c")).read()
    for fn, call in (("js_find_matches_one", "cg_find_matches_one("), ("js_redact_one", "cg_redact_one(")):
        body = src[src.index("static napi_value %s(" % fn):]
        body = body[:body.index("\n}\n")]
        guard = re.search(r"if \(!nb\) bytes = (\w+);", body)
        assert guard and body.index(guard.group(0)) < body.index(call), fn
        assert re.search(r"static uint8_t %s\[1\];" % guard.group(1), src), fn


def test_single_message_calls_before_init_are_not_initialized():
    # a fresh process that never calls cg_init (with or without a device: the calls must not initialise anything)
    code = ("import sys, ctypes as C; sys.path.insert(0, %r)\n"
            "from vainplex_openclaw_b200 import _native as N\n"
            "L = N.load()\n"
            "n, need = C.c_uint32(7), C.c_uint64(7)\n"
            "spans = (C.c_uint32 * 64)(); out = (C.c_uint8 * 64)(); dig = (C.c_uint8 * 64)()\n"
            "a = L.cg_find_matches_one(None, b'abc', 3, spans, 8, C.byref(n))\n"
            "b = L.cg_redact_one(None, b'abc', 3, out, 64, C.byref(need), spans, 8, C.byref(n), dig)\n"
            "print(a, b, n.value, need.value)\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["-2", "-2", "7", "7"]
