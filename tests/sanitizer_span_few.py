"""Workload for a compute-sanitizer run over the few-string span calls (not collected by pytest): cg_find_matches_few and
cg_redact_few at 1, 2, 17, 255 and 256 strings, totals of 0 and 64 KB, empty strings, a result whose packed form is longer
than the first copy's window, a queue overflow answered through the batch path, and the capacity paths.  Every result is
checked against the batch calls.  Usage:
  compute-sanitizer --tool memcheck --error-exitcode 3 python tests/sanitizer_span_few.py"""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vainplex_openclaw_b200 import _native as N, workload as W  # noqa: E402

N.init(0)
rl = W.make_rules(120)
rs = N.Ruleset(W.rules_as_tuples(rl), strict=True)
rng = np.random.default_rng(3)
data_t, _, _ = W.make_messages(1, 65536, rl, p_hit=1.0, utf8_frac=0.15, seed=3)
src = bytes(data_t.numpy()[:65536])


def split(n, total):
    cuts = np.sort(rng.integers(0, total + 1, max(n - 1, 0)))
    b = [0] + [int(c) for c in cuts] + [total]
    return [src[b[i]:b[i + 1]] for i in range(n)]


def same(msgs):
    data, off = N.pack(msgs)
    assert [tuple(s) for s in rs.find_matches_few(data, off).tolist()] == [tuple(s) for s in rs.find_matches_batch(data, off).tolist()]
    a, b = rs.redact_few(data, off), rs.redact_batch(data, off)
    assert bytes(a[0]) == bytes(b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[3], b[3])


for n, total in ((1, 0), (1, 900), (2, 300), (17, 4000), (255, 9000), (256, 20000), (3, 65536), (256, 0)):
    same(split(n, total))
same([b"", b"1" * 600 + b" tail", b""])                                 # a packed result longer than the first window
over = N.Ruleset([(r"\d", 0, 2), ("[a-z]", 0, 3)], strict=True)
d, o = N.pack([b"7" * 2500, b"7" * 2500 + b" abcdefghij"])             # more raw spans than a fresh scratch holds
assert len(over.find_matches_few(d, o)) == len(over.find_matches_few(d, o)) == 5010
over.close()
L = N.load()
data, off = N.pack(split(9, 3000))
n, need = C.c_uint32(0), C.c_uint64(0)
oo = np.zeros(10, np.uint32)
spans, out, dig = np.zeros(24 * 4, np.uint8), np.zeros(64, np.uint8), np.zeros(32 * 4, np.uint8)
assert L.cg_find_matches_few(rs.handle, data.ctypes.data, off.ctypes.data, 9, spans.ctypes.data, 4, C.byref(n)) == N.CG_ERR_CAPACITY
assert L.cg_redact_few(rs.handle, data.ctypes.data, off.ctypes.data, 9, out.ctypes.data, 64, C.byref(need), oo.ctypes.data,
                       spans.ctypes.data, 4, C.byref(n), dig.ctypes.data) == N.CG_ERR_CAPACITY
rs.close()
print("sanitizer workload ok")
