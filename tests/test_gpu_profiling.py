"""GPU tier: profiling mode (cg_set_profiling) records events around the scan step's kernels.  With it on, the batch calls
return what they return with it off, and the event timings keep their meaning: last_kernel_ms() = (scan_kernel,
confirm_kernel + resolve, verify, finalize), last_tail_ms() = (confirm_kernel, resolve).  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from test_gpu_boundaries import device_words, hit_pairs, span_tuples
from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


def outputs(N, rs, data, off):
    """(host words, host hit pairs, spans, device words) of one batch"""
    words, hits = rs.scan_batch(data, off)
    spans = span_tuples(rs.find_matches_batch(data, off))
    dwords = device_words(N, rs, data, off)
    return words, hit_pairs(hits), spans, dwords


def check_timings(N):
    kms, tms = N.last_kernel_ms(), N.last_tail_ms()
    assert len(kms) == 4 and len(tms) == 2
    assert all(t >= 0.0 for t in kms + tms), (kms, tms)
    assert abs(kms[1] - (tms[0] + tms[1])) <= 2e-3, (kms, tms)      # ms: confirm + resolve, within 2 us
    return kms, tms


def test_profiling_keeps_outputs_and_timings(N):
    rl = W.make_rules(64)
    rs = N.Ruleset(W.rules_as_tuples(rl), strict=True)
    data_t, off_t, inj = W.make_messages(4096, 256, rl, p_hit=0.05, seed=11)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    try:
        words, hits, spans, dwords = outputs(N, rs, data, off)
        assert len(inj) and len(hits) and len(spans)
        N.set_profiling(True)
        pw, ph = rs.scan_batch(data, off)
        assert np.array_equal(pw, words) and hit_pairs(ph) == hits
        check_timings(N)
        assert span_tuples(rs.find_matches_batch(data, off)) == spans
        check_timings(N)
        assert np.array_equal(device_words(N, rs, data, off), dwords)
        check_timings(N)
    finally:
        N.set_profiling(False)
        rs.close()
