"""Device-resident findMatches and redaction (cg_find_matches_batch_device / cg_redact_batch_device) and the span resolver
behind them and behind the host calls: spans, output bytes, digests, sizes and statuses against the host calls, the oracle
and a Python restatement of applyReplacements.  Run on an H100: pytest -m gpu."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_parity import CATS, oracle_spans
from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu
GUARD = 0x5A
EMPTY_MATCH_RULES = [(r"sk-[a-zA-Z0-9]{20,}", 0, 0), (r"\d+", 0, 3), (r"", 0, 3), (r"^$", 0, 3), (r"a*?b", 0, 3), (r"x\b", 0, 3), (r"(?:a??)?", 0, 3)]


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


@pytest.fixture(scope="module")
def torch():
    import torch as T
    return T


def tup(spans):
    return [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in spans]


def full(spans):
    return [tuple(int(s[f]) for f in ("msg", "rule", "start_byte", "end_byte", "start16", "end16")) for s in spans]


def to_device(torch, data, off):
    """message bytes (16-byte aligned, 64 bytes of padding) and int32 offsets in HBM"""
    d = torch.from_numpy(np.concatenate([np.asarray(data, np.uint8), np.zeros(64, np.uint8)])).cuda()
    o = torch.from_numpy(np.asarray(off, np.uint32).astype(np.int32)).cuda()
    return d, o


def ragged(data_t, off_t, seed, max_len):
    buf, off0 = data_t.numpy(), off_t.numpy()
    rng = np.random.default_rng(seed)
    return [bytes(buf[int(off0[i]):int(off0[i]) + int(rng.integers(0, max_len + 1))]) for i in range(len(off0) - 1)]


class FindOut:
    """device buffers of one cg_find_matches_batch_device call, with guard words behind the capacity"""

    def __init__(self, torch, cap, guard=64):
        self.cap = cap
        self.spans = torch.full(((cap + guard) * 6,), GUARD * 0x01010101, dtype=torch.int32, device="cuda")
        self.nspans = torch.full((4,), -1, dtype=torch.int32, device="cuda")

    def issue(self, rs, d, o, n, stream=0):
        rs.find_matches_batch_device(d.data_ptr(), o.data_ptr(), n, self.spans.data_ptr(), self.cap, self.nspans.data_ptr(), stream)

    def result(self, N):
        ns = int(self.nspans[0].item()) & 0xffffffff
        raw = self.spans.cpu().numpy().view(np.uint32)
        spans = raw[:6 * min(ns, self.cap)].copy().view(N.SPAN_DTYPE)
        return ns, spans, raw[6 * self.cap:]


class RedactOut:
    """device buffers of one cg_redact_batch_device call, with guard bytes behind both capacities"""

    def __init__(self, torch, n, out_cap, spans_cap, guard=256):
        self.n, self.out_cap, self.spans_cap = n, out_cap, spans_cap
        self.out = torch.full((out_cap + guard,), GUARD, dtype=torch.uint8, device="cuda")
        self.off = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
        self.spans = torch.full(((spans_cap + 16) * 6,), GUARD * 0x01010101, dtype=torch.int32, device="cuda")
        self.dig = torch.full(((spans_cap + 16) * 32,), GUARD, dtype=torch.uint8, device="cuda")
        self.sizes = torch.full((2,), -1, dtype=torch.int64, device="cuda")

    def issue(self, rs, d, o, stream=0):
        rs.redact_batch_device(d.data_ptr(), o.data_ptr(), self.n, self.out.data_ptr(), self.out_cap, self.off.data_ptr(),
                               self.spans.data_ptr(), self.spans_cap, self.dig.data_ptr(), self.sizes.data_ptr(), stream)

    def sizes_(self):
        s = self.sizes.cpu().numpy().view(np.uint64)
        return int(s[0]), int(s[1])

    def result(self, N):
        need, ns = self.sizes_()
        out = self.out.cpu().numpy()
        spans_raw = self.spans.cpu().numpy().view(np.uint32)
        dig = self.dig.cpu().numpy()
        return (out[:need], self.off.cpu().numpy().view(np.uint32), spans_raw[:6 * ns].copy().view(N.SPAN_DTYPE),
                dig[:32 * ns].reshape(-1, 32), out[self.out_cap:], spans_raw[6 * self.spans_cap:], dig[32 * self.spans_cap:])


def find_device(N, torch, rs, data, off, cap=None):
    """one batch through cg_find_matches_batch_device; issued again while an internal queue overflows (sizes ~0)"""
    n = len(off) - 1
    d, o = to_device(torch, data, off)
    fo = FindOut(torch, cap if cap is not None else max(1024, 4 * n))
    for attempt in range(4):
        fo.issue(rs, d, o, n)
        try:
            rs.scan_join()
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
            assert (int(fo.nspans[0].item()) & 0xffffffff) == 0xffffffff
    ns, spans, guard = fo.result(N)
    assert (guard == GUARD * 0x01010101).all()
    assert ns == len(spans)
    return spans


def splice_python(msgs, rules, spans, dig):
    """applyReplacements restated: right to left, [REDACTED:<category>:<hash8>]"""
    by_msg = {}
    for s, d in zip(spans, dig):
        m = msgs[int(s["msg"])][int(s["start_byte"]):int(s["end_byte"])]
        assert bytes(d) == hashlib.sha256(m).digest()
        by_msg.setdefault(int(s["msg"]), []).append((int(s["start_byte"]), int(s["end_byte"]), CATS[rules[int(s["rule"])][2]], bytes(d).hex()[:8]))
    out = []
    for i, m in enumerate(msgs):
        e = bytearray(m)
        for a, b, cat, h8 in sorted(by_msg.get(i, []), reverse=True):
            e[a:b] = ("[REDACTED:%s:%s]" % (cat, h8)).encode()
        out.append(bytes(e))
    return out


# ------------------------------------------------------------------------------------------------ spans

SPAN_CASES = [(17, 0.0), (120, 0.0), (120, 0.1), (120, 0.2), (500, 0.0), (500, 0.1), (500, 0.2)]


@pytest.mark.parametrize("n_rules,utf8_frac", SPAN_CASES)
def test_device_spans_equal_host_and_oracle(N, torch, oracle, n_rules, utf8_frac):
    rl = W.make_rules(n_rules)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(1500, 200, rl, p_hit=0.25, utf8_frac=utf8_frac, seed=300 + n_rules + int(utf8_frac * 10))
    msgs = ragged(data_t, off_t, 7 + n_rules, 200)                     # lengths 0 .. 200, may cut a character
    data, off = N.pack(msgs)
    exp = oracle_spans(oracle, rules, data, off)
    host = rs.find_matches_batch(data, off)
    dev = find_device(N, torch, rs, data, off)
    assert tup(host) == exp and len(exp) >= 100
    assert full(dev) == full(host)
    rs.close()


def test_device_spans_small_and_dense_batches(N, torch, oracle):
    """n = 0, n = 1, every message with spans, and the empty-match rules"""
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    d0, o0 = N.pack([])
    assert len(find_device(N, torch, rs, d0, o0)) == 0
    data_t, off_t, _ = W.make_messages(1, 300, rl, p_hit=1.0, seed=21)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    dev = find_device(N, torch, rs, data, off)
    assert tup(dev) == oracle_spans(oracle, rules, data, off) and len(dev) >= 1
    data_t, off_t, _ = W.make_messages(2000, 256, rl, p_hit=1.0, seed=22)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    dev = find_device(N, torch, rs, data, off)
    assert tup(dev) == oracle_spans(oracle, rules, data, off)
    assert len(set(int(s["msg"]) for s in dev)) == 2000
    rs.close()

    rs = N.Ruleset(EMPTY_MATCH_RULES, strict=True)
    rng = np.random.default_rng(3)
    msgs = [b"", b"a", b"sk-" + b"a" * 25, b"", b"12 345", "\U0001F600".encode(), b"aab xb", b"x" * 700 + b" 9"]
    msgs += [bytes(rng.integers(32, 127, int(k), dtype=np.uint8)) for k in rng.integers(0, 90, 300)]
    msgs += [bytes(rng.integers(0, 256, int(k), dtype=np.uint8)) for k in rng.integers(0, 40, 200)]
    data, off = N.pack(msgs)
    dev = find_device(N, torch, rs, data, off, cap=100000)
    assert tup(dev) == oracle_spans(oracle, EMPTY_MATCH_RULES, data, off)
    assert full(dev) == full(rs.find_matches_batch(data, off))
    rs.close()


def test_tie_breaks_follow_category_then_rule(N, torch, oracle):
    """identical spans from rules of different categories and from two rules of one category; equal starts of different
    lengths; several empty matches at one position"""
    rules = [("abc", 0, 2), ("ab.", 0, 3), ("abc", 0, 0), ("abc", 0, 0), ("ab", 0, 1), ("a", 0, 2), ("q??", 0, 3), ("", 0, 1)]
    rs = N.Ruleset(rules, strict=True)
    msgs = [b"abc", b"xxabcabd abcabc", b"ab", b"", b"zabcz" * 50]
    data, off = N.pack(msgs)
    exp = oracle_spans(oracle, rules, data, off)
    dev = find_device(N, torch, rs, data, off)
    assert tup(dev) == exp
    assert full(dev) == full(rs.find_matches_batch(data, off))
    assert any(r == 2 for (_, r, _, _) in exp)                        # "abc" as credential wins over pii / custom / the copy
    rs.close()


def test_one_dense_message(N, torch, oracle):
    """one message holding nearly every span of the batch, beside short messages: 8 000 digits under \\d (the segment is
    sorted in runs and merged), then 36 single-digit rules of all four categories over 2 000 digits: 72 000 raw spans in
    one segment, identical spans tie-broken by (category, rule).  (Span mode costs the VM O(message length) per match, so
    the messages stay this short.)"""
    rules = [(r"\d", 0, 2), ("[a-z]+", 0, 1)]
    msgs = [b"abc 12", b"1" * 8000, b"", b"x9y"]
    data, off = N.pack(msgs)
    rs = N.Ruleset(rules, strict=True)
    exp = oracle_spans(oracle, rules, data, off)
    host = rs.find_matches_batch(data, off)                                 # (sizes the scratch: one VM pass fewer below)
    dev = find_device(N, torch, rs, data, off, cap=10000)
    assert len(exp) > 8000 and tup(dev) == exp and full(dev) == full(host)
    rs.close()
    many = [((r"\d", r"[0-9]", r"[0-5]|[6-9]")[i % 3], 0, (3 * i + 1) % 4) for i in range(36)]
    msgs = [b"a1", b"7" * 2000, b"", b"x9y"]
    data, off = N.pack(msgs)
    rs = N.Ruleset(many, strict=True)
    exp = oracle_spans(oracle, many, data, off)
    host = rs.find_matches_batch(data, off)
    dev = find_device(N, torch, rs, data, off, cap=10000)
    assert len(exp) == 2002 and tup(dev) == exp and full(dev) == full(host)
    rs.close()


# ------------------------------------------------------------------------------------------------ redaction

def test_redacted_output_equals_host_and_python(N, torch, oracle):
    rl = W.make_rules(200)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(3000, 180, rl, p_hit=0.3, utf8_frac=0.15, seed=78)
    msgs = ragged(data_t, off_t, 6, 180)
    data, off = N.pack(msgs)
    h_out, h_off, h_spans, h_dig = rs.redact_batch(data, off)
    n = len(msgs)
    d, o = to_device(torch, data, off)
    ro = RedactOut(torch, n, len(h_out) + 1000, len(h_spans) + 100)
    ro.issue(rs, d, o)
    rs.scan_join()
    out, out_off, spans, dig, g_out, g_spans, g_dig = ro.result(N)
    assert ro.sizes_() == (len(h_out), len(h_spans))
    assert tup(spans) == oracle_spans(oracle, rules, data, off) and len(spans) >= 300
    assert full(spans) == full(h_spans) and np.array_equal(dig, h_dig)
    assert np.array_equal(out_off, h_off) and np.array_equal(out, h_out)
    exp = splice_python(msgs, rules, spans, dig)
    assert [bytes(out[int(out_off[i]):int(out_off[i + 1])]) for i in range(n)] == exp
    assert (ro.out.cpu().numpy()[len(h_out):] == GUARD).all()               # nothing past `need`, nor past spans_cap
    assert (g_spans == GUARD * 0x01010101).all() and (g_dig == GUARD).all()
    rs.close()


def test_capacity_is_reported_and_nothing_written_past_it(N, torch):
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(800, 200, rl, p_hit=0.5, seed=31)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    h_out, h_off, h_spans, h_dig = rs.redact_batch(data, off)
    need, ns = len(h_out), len(h_spans)
    assert ns > 20
    n = len(off) - 1
    d, o = to_device(torch, data, off)
    for out_cap, spans_cap in ((need - 1, ns), (need, ns - 1), (0, 0)):
        ro = RedactOut(torch, n, out_cap, spans_cap)
        ro.issue(rs, d, o)
        with pytest.raises(N.GovError) as ei:
            rs.scan_join()
        assert ei.value.code == N.CG_ERR_CAPACITY
        assert ro.sizes_() == (need, ns)
        out_all = ro.out.cpu().numpy()
        assert (out_all == GUARD).all()                                     # no byte of output, digest or span past the capacities
        assert (ro.dig.cpu().numpy() == GUARD).all()
        assert np.array_equal(ro.off.cpu().numpy().view(np.uint32), h_off)
        sp = ro.spans.cpu().numpy().view(np.uint32)
        assert (sp[6 * spans_cap:] == GUARD * 0x01010101).all()
    ro = RedactOut(torch, n, need, ns)                                      # issued again with the reported sizes
    ro.issue(rs, d, o)
    rs.scan_join()
    out, out_off, spans, dig, g_out, g_spans, g_dig = ro.result(N)
    assert np.array_equal(out, h_out) and full(spans) == full(h_spans) and np.array_equal(dig, h_dig)
    assert (g_out == GUARD).all() and (g_spans == GUARD * 0x01010101).all() and (g_dig == GUARD).all()
    # find-matches: the first spans_cap spans, the true count, CG_ERR_CAPACITY
    fo = FindOut(torch, ns // 2)
    fo.issue(rs, d, o, n)
    with pytest.raises(N.GovError) as ei:
        rs.scan_join()
    assert ei.value.code == N.CG_ERR_CAPACITY
    got_ns, spans, guard = fo.result(N)
    assert got_ns == ns and full(spans) == full(h_spans)[:ns // 2] and (guard == GUARD * 0x01010101).all()
    rs.close()


def test_internal_overflow_is_reported_in_band(N, torch, oracle):
    """more raw spans than a fresh rule set's span queue holds (max(n, 4096)): sizes ~0, CG_ERR_CAPACITY once, nothing
    written; the same batch issued again is complete"""
    rules = [(r"\d", 0, 2), ("[a-z]", 0, 3)]
    msgs = [b"7" * 900 + b" abc" for _ in range(10)]
    data, off = N.pack(msgs)
    exp = oracle_spans(oracle, rules, data, off)
    assert len(exp) > 4096
    n = len(msgs)
    d, o = to_device(torch, data, off)
    rs = N.Ruleset(rules, strict=True)
    fo = FindOut(torch, 20000)
    fo.issue(rs, d, o, n)
    with pytest.raises(N.GovError) as ei:
        rs.scan_join()
    assert ei.value.code == N.CG_ERR_CAPACITY
    assert (int(fo.nspans[0].item()) & 0xffffffff) == 0xffffffff
    assert (fo.spans.cpu().numpy().view(np.uint32) == GUARD * 0x01010101).all()
    fo.issue(rs, d, o, n)
    rs.scan_join()
    ns, spans, _ = fo.result(N)
    assert tup(spans) == exp
    rs.close()
    rs = N.Ruleset(rules, strict=True)                                     # the same for the redaction call
    ro = RedactOut(torch, n, 400000, 20000)
    ro.issue(rs, d, o)
    with pytest.raises(N.GovError) as ei:
        rs.scan_join()
    assert ei.value.code == N.CG_ERR_CAPACITY
    assert ro.sizes_() == (2 ** 64 - 1, 2 ** 64 - 1)
    assert (ro.out.cpu().numpy() == GUARD).all() and (ro.dig.cpu().numpy() == GUARD).all()
    rs.scan_join()                                                           # reported once
    ro.issue(rs, d, o)
    rs.scan_join()
    out, out_off, spans, dig, _, _, _ = ro.result(N)
    assert tup(spans) == exp
    assert [bytes(out[int(out_off[i]):int(out_off[i + 1])]) for i in range(n)] == splice_python(msgs, rules, spans, dig)
    rs.close()


# ------------------------------------------------------------------------------------------------ asynchrony

def test_back_to_back_batches_on_one_stream(N, torch):
    rl = W.make_rules(500)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    st = torch.cuda.Stream()
    batches = []
    for seed in range(3):
        data_t, off_t, _ = W.make_messages(3000, 256, rl, p_hit=0.05 * (seed + 1), seed=500 + seed)
        data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
        batches.append((data, off, rs.redact_batch(data, off), rs.scan_batch(data, off, want_hits=False)[0]))
    dev = [to_device(torch, data, off) for data, off, _, _ in batches]
    finds = [FindOut(torch, len(h[2]) + 10) for _, _, h, _ in batches]
    reds = [RedactOut(torch, len(off) - 1, len(h[0]) + 10, len(h[2]) + 10) for _, off, h, _ in batches]
    words = [torch.zeros(len(off) - 1, dtype=torch.int64, device="cuda") for _, off, _, _ in batches]
    torch.cuda.synchronize()
    for (d, o), fo, ro, w in zip(dev, finds, reds, words):                  # no host wait between the batches
        n = ro.n
        rs.scan_batch_device(d.data_ptr(), o.data_ptr(), n, w.data_ptr(), st.cuda_stream)
        fo.issue(rs, d, o, n, st.cuda_stream)
        ro.issue(rs, d, o, st.cuda_stream)
    rs.scan_join(st.cuda_stream)
    for (data, off, h, ew), fo, ro, w in zip(batches, finds, reds, words):
        ns, spans, _ = fo.result(N)
        assert full(spans) == full(h[2])
        out, out_off, rspans, dig, _, _, _ = ro.result(N)
        assert np.array_equal(out, h[0]) and np.array_equal(out_off, h[1]) and full(rspans) == full(h[2]) and np.array_equal(dig, h[3])
        assert np.array_equal(w.cpu().numpy().view(np.uint64), ew)
    rs.close()


def test_launch_count_does_not_depend_on_the_span_count(N, torch):
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    quiet_t, qoff_t, _ = W.make_messages(2000, 256, rl, p_hit=0.0, seed=41)
    dense_t, doff_t, _ = W.make_messages(2000, 256, rl, p_hit=1.0, seed=42)
    q = to_device(torch, quiet_t.numpy(), qoff_t.numpy())
    dn = to_device(torch, dense_t.numpy(), doff_t.numpy())
    fo, ro = FindOut(torch, 200000), RedactOut(torch, 2000, 4 << 20, 200000)
    for attempt in range(4):                                                # warm: scratch sized for both batches
        for d, o in (q, dn):
            fo.issue(rs, d, o, 2000); ro.issue(rs, d, o)
        try:
            rs.scan_join()
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
    counts, found = {}, {}
    for name, (d, o) in (("quiet", q), ("dense", dn)):
        k0 = N.launch_count()
        fo.issue(rs, d, o, 2000)
        k1 = N.launch_count()
        ro.issue(rs, d, o)
        k2 = N.launch_count()
        rs.scan_join()
        counts[name] = (k1 - k0, k2 - k1)
        found[name] = fo.result(N)[0]
    assert found["dense"] >= 2000 and found["quiet"] < found["dense"] // 10
    assert counts["quiet"] == counts["dense"]
    rs.close()


# ------------------------------------------------------------------------------------------------ arguments, statistics

def test_argument_checks(N, torch):
    rs = N.Ruleset([("abc", 0, 2)], strict=True)
    data, off = N.pack([b"xxabc", b"abc"])
    d, o = to_device(torch, data, off)
    fo, ro = FindOut(torch, 16), RedactOut(torch, 2, 256, 16)
    L = N.load()
    with pytest.raises(N.GovError) as ei:
        rs.find_matches_batch_device(d.data_ptr() + 4, o.data_ptr(), 2, fo.spans.data_ptr(), 16, fo.nspans.data_ptr())
    assert ei.value.code == -1
    with pytest.raises(N.GovError):
        ro.issue(rs, d[4:], o)
    assert L.cg_find_matches_batch_device(None, d.data_ptr(), o.data_ptr(), 2, fo.spans.data_ptr(), 16, fo.nspans.data_ptr(), None) == -1
    assert L.cg_find_matches_batch_device(rs.handle, d.data_ptr(), o.data_ptr(), 2, None, 16, fo.nspans.data_ptr(), None) == -1
    assert L.cg_find_matches_batch_device(rs.handle, d.data_ptr(), o.data_ptr(), 2, fo.spans.data_ptr(), 16, None, None) == -1
    assert L.cg_find_matches_batch_device(rs.handle, None, o.data_ptr(), 2, fo.spans.data_ptr(), 16, fo.nspans.data_ptr(), None) == -1
    assert L.cg_redact_batch_device(rs.handle, d.data_ptr(), o.data_ptr(), 2, ro.out.data_ptr(), 256, None, ro.spans.data_ptr(), 16,
                                    ro.dig.data_ptr(), ro.sizes.data_ptr(), None) == -1
    assert L.cg_redact_batch_device(rs.handle, d.data_ptr(), o.data_ptr(), 2, ro.out.data_ptr(), 256, ro.off.data_ptr(), ro.spans.data_ptr(), 16,
                                    None, ro.sizes.data_ptr(), None) == -1
    assert L.cg_redact_batch_device(rs.handle, d.data_ptr(), o.data_ptr(), 2, ro.out.data_ptr(), 256, ro.off.data_ptr(), ro.spans.data_ptr(), 16,
                                    ro.dig.data_ptr(), None, None) == -1
    rs.scan_join()
    fo.issue(rs, d, o, 2)                                                   # the rule set is still usable
    rs.scan_join()
    assert tup(fo.result(N)[1]) == [(0, 0, 2, 5), (1, 0, 0, 3)]
    rs.close()
    # before cg_init, in a fresh process: CG_ERR_NOT_INITIALIZED
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path.insert(0, %r)\n"
            "from vainplex_openclaw_b200 import _native as N\n"
            "L = N.load()\n"
            "print(L.cg_find_matches_batch_device(None, 16, 16, 1, 16, 1, 16, None),"
            " L.cg_redact_batch_device(None, 16, 16, 1, 16, 1, 16, 16, 1, 16, 16, None))\n" % root)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["-2", "-2"]


def test_statistics_count_resolved_spans(N, torch):
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(1000, 200, rl, p_hit=0.3, seed=61)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    n = len(off) - 1
    s0 = N.stats()
    spans = rs.find_matches_batch(data, off)
    s1 = N.stats()
    out, _, rspans, _ = rs.redact_batch(data, off)
    s2 = N.stats()
    ns = len(spans)
    assert ns > 50 and len(rspans) == ns
    assert s1.spans - s0.spans == ns and s1.sha256_items == s0.sha256_items
    assert s2.spans - s1.spans == ns and s2.sha256_items - s1.sha256_items == ns
    d, o = to_device(torch, data, off)
    fo, ro = FindOut(torch, ns), RedactOut(torch, n, len(out), ns)
    fo.issue(rs, d, o, n)
    ro.issue(rs, d, o)
    s3 = N.stats()
    assert s3.messages_scanned - s2.messages_scanned == 2 * n
    rs.scan_join()
    s4 = N.stats()
    assert s4.spans - s2.spans == 2 * ns and s4.sha256_items - s2.sha256_items == ns
    rs.close()
