"""The workloads of test_gpu_span_boundaries.py checked with the oracle alone, without a device: the segment batches hold
the raw-span counts they claim, and the JSONL blobs the sizes, newlines, empty-line runs and long lines they claim."""
import numpy as np

from test_gpu_span_boundaries import (JSONL_BLOBS, SEG_RULES, SEG_SIZES, check_jsonl_claims, geometry, jsonl_blob, long_segment_batch,
                                      merge_passes, raw_span_counts, segment_batch)


def test_segment_batches_hold_the_raw_span_counts_they_claim(oracle):
    g = geometry(132)                                       # the SM count of an H100 SXM
    for kind in SEG_RULES:
        msgs, raw = segment_batch(kind)
        assert np.array_equal(raw_span_counts(oracle, SEG_RULES[kind], msgs), raw), kind
        assert sorted(set(raw.tolist()) - {0}) == sorted(set(SEG_SIZES) - {0})
    assert {merge_passes(g, c) for c in SEG_SIZES} == {0, 1, 2, 3}
    msgs, raw = long_segment_batch(g)
    assert np.array_equal(raw_span_counts(oracle, SEG_RULES["ties"], msgs), raw)
    assert min(int((raw[b::g.sort_blocks] > g.warp_sort).sum()) for b in range(g.sort_blocks)) >= 3


def test_jsonl_blobs_have_the_lines_they_claim(oracle):
    for name in JSONL_BLOBS:
        blob = jsonl_blob(name)
        lines = check_jsonl_claims(name, blob)
        data, off = oracle.pack(lines)
        assert len(oracle.merkle_root(data, off)) == 32
        assert int(off[-1]) + len(lines) - (0 if blob.endswith(b"\n") else 1) == len(blob)
