"""Device-resident hit lists and verdicts (cg_scan_hits_batch_device / cg_policy_verdict_batch_device) and the hit-list
kernels behind them and behind cg_scan_batch's out_hits: (msg, rule) lists against the oracle and the host call, result
words against cg_scan_batch_device, verdicts against cg_policy_verdict_batch, capacities, queue overflows, streams and edge
cases.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from test_gpu_parity import oracle_policy
from test_gpu_redact_device import to_device
from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu
GUARD = 0x5A5A5A5A
ALL_ONES = 0xffffffff


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


@pytest.fixture(scope="module")
def torch():
    import torch as T
    return T


class HitsOut:
    """device buffers of one cg_scan_hits_batch_device call, with guard words behind the capacity"""

    def __init__(self, torch, n, cap, guard=64):
        self.n, self.cap = n, cap
        self.words = torch.full((max(n, 1),), -1, dtype=torch.int64, device="cuda")
        self.hits = torch.full(((cap + guard) * 2,), GUARD, dtype=torch.int32, device="cuda")
        self.nhits = torch.full((4,), -1, dtype=torch.int32, device="cuda")

    def issue(self, rs, d, o, stream=0, null_hits=False):
        rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr(), self.n, self.words.data_ptr(), 0 if null_hits else self.hits.data_ptr(),
                                  self.cap, self.nhits.data_ptr(), stream)

    def nh(self):
        return int(self.nhits[0].item()) & 0xffffffff

    def result(self):
        """-> (count word, pairs written [(msg, rule)], guard words behind the capacity, result words)"""
        nh = self.nh()
        raw = self.hits.cpu().numpy().view(np.uint32)
        k = min(nh, self.cap)
        pairs = [tuple(int(x) for x in p) for p in raw[:2 * k].reshape(-1, 2)]
        return nh, pairs, raw[2 * self.cap:], self.words.cpu().numpy().view(np.uint64)[:self.n]


def hits_device(N, torch, rs, data, off, cap=None, stream=0):
    """one batch through cg_scan_hits_batch_device; issued again while an internal queue overflows (count ~0)"""
    n = len(off) - 1
    d, o = to_device(torch, data, off)
    ho = HitsOut(torch, n, cap if cap is not None else max(1024, 4 * n))
    for attempt in range(4):
        ho.issue(rs, d, o, stream)
        try:
            rs.scan_join(stream)
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
            assert ho.nh() == ALL_ONES
    nh, pairs, guard, words = ho.result()
    assert (guard == GUARD).all()
    assert nh == len(pairs)
    return words, pairs


def device_words(N, torch, rs, data, off):
    """the result words of cg_scan_batch_device (issued again after an overflow)"""
    n = len(off) - 1
    d, o = to_device(torch, data, off)
    out = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    for attempt in range(4):
        rs.scan_batch_device(d.data_ptr(), o.data_ptr(), n, out.data_ptr())
        try:
            rs.scan_join()
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
    return out.cpu().numpy().view(np.uint64)


def host_pairs(hits):
    return [(int(h["msg"]), int(h["rule"])) for h in hits]


def verdicts_device(N, torch, rs, data, off, stream=0):
    n = len(off) - 1
    d, o = to_device(torch, data, off)
    out = torch.full((n + 16,), GUARD, dtype=torch.int32, device="cuda")
    for attempt in range(4):
        rs.verdict_batch_device(d.data_ptr(), o.data_ptr(), n, out.data_ptr(), stream)
        try:
            rs.scan_join(stream)
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
            assert (out[:n].cpu().numpy().view(np.uint32) == ALL_ONES).all()
    got = out.cpu().numpy().view(np.uint32)
    assert (got[n:] == GUARD).all()
    return got[:n]


# ------------------------------------------------------------------------------ 1. parity

@pytest.mark.parametrize("n_rules,n", [(500, 1 << 16), (5000, 4096)])
def test_hit_list_equals_oracle_host_and_words(N, torch, oracle, n_rules, n):
    """500 rules (the 17 built-ins first) at p_hit 10 % over 64 Ki messages, and 5000 rules (157 hit words per row): the
    device list == the oracle's (msg, rule) list == cg_scan_batch's out_hits; the words == cg_scan_batch_device's."""
    rl = W.make_rules(n_rules)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(n, 256, rl, p_hit=0.10, seed=7100 + n_rules)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    if n_rules == 5000:
        # a few dense messages whose hits spread over every word of the row (the wave's later steps)
        rng = np.random.default_rng(5000)
        msgs = [bytes(data[int(off[i]):int(off[i + 1])]) for i in range(n)]
        for i in range(0, n, 409):
            picks = sorted(rng.choice(len(rl), 120, replace=False))
            msgs[i] = b" ".join(rl[int(r)]["sample"].encode() for r in picks)
        data, off = N.pack(msgs)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    words, pairs = hits_device(N, torch, rs, data, off)
    assert pairs == ehits
    assert np.array_equal(words, ewords)
    hwords, hhits = rs.scan_batch(data, off)
    assert host_pairs(hhits) == ehits and np.array_equal(hwords, ewords)
    assert np.array_equal(device_words(N, torch, rs, data, off), words)
    assert len(ehits) > n // 20
    if n_rules == 5000:
        assert max(r for _, r in ehits) >= 4900 and max(sum(1 for m, _ in ehits if m == i) for i in range(0, n, 409)) >= 100
    rs.close()


# ------------------------------------------------------------------------------ 2. capacity

def test_capacity_first_pairs_and_guard(N, torch, oracle):
    """hits_cap below the total: the first hits_cap pairs, nothing past them, *d_out_nhits = the total, CG_ERR_CAPACITY
    once and CG_OK at the next join; hits_cap = 0 with a NULL list gives the count alone."""
    rl = W.make_rules(500)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(6000, 256, rl, p_hit=0.10, seed=77)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    _, ehits = oracle_policy(oracle, rules, data, off)
    total = len(ehits)
    hits_device(N, torch, rs, data, off)                              # (scratch sized: no queue overflow below)
    d, o = to_device(torch, data, off)
    for cap in (1, 31, 32, 33, total // 2, total - 1):
        ho = HitsOut(torch, 6000, cap, guard=256)
        ho.issue(rs, d, o)
        with pytest.raises(N.GovError) as ei:
            rs.scan_join()
        assert ei.value.code == N.CG_ERR_CAPACITY
        rs.scan_join()                                                # (reported once)
        nh, pairs, guard, _ = ho.result()
        assert nh == total and pairs == ehits[:cap] and (guard == GUARD).all(), cap
    ho = HitsOut(torch, 6000, total)                                  # exactly enough
    ho.issue(rs, d, o)
    rs.scan_join()
    nh, pairs, guard, _ = ho.result()
    assert nh == total and pairs == ehits and (guard == GUARD).all()
    ho = HitsOut(torch, 6000, 0)
    ho.issue(rs, d, o, null_hits=True)
    with pytest.raises(N.GovError) as ei:
        rs.scan_join()
    assert ei.value.code == N.CG_ERR_CAPACITY
    assert ho.nh() == total and (ho.hits.cpu().numpy().view(np.uint32) == GUARD).all()
    rs.scan_join()
    # no hit at all: cap 0 and a NULL list are enough
    msgs0 = [b"plain words and nothing else %d" % i for i in range(500)]
    data0, off0 = N.pack(msgs0)
    assert oracle_policy(oracle, rules, data0, off0)[1] == []
    d0, o0 = to_device(torch, data0, off0)
    ho = HitsOut(torch, 500, 0)
    ho.issue(rs, d0, o0, null_hits=True)
    rs.scan_join()
    assert ho.nh() == 0
    with pytest.raises(N.GovError) as ei:                             # (a capacity without a list)
        rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr(), 6000, ho.words.data_ptr(), 0, 5, ho.nhits.data_ptr())
    assert ei.value.code == -1
    rs.close()


# ------------------------------------------------------------------------------ 3. queue overflow, in band

def test_queue_overflow_is_reported_in_band(N, torch, oracle):
    """A fresh rule set sized by a small batch, then 30 000 messages that all hit: the count is 0xffffffff, no pair is
    written, the join raises CG_ERR_CAPACITY; issued again the batch gives the oracle's list.  The same for verdicts,
    which are all 0xffffffff."""
    rl = W.make_rules(64)
    rules = W.rules_as_tuples(rl)
    d0_t, o0_t, _ = W.make_messages(64, 256, rl, p_hit=0.0, seed=3)
    d1_t, o1_t, _ = W.make_messages(30000, 256, rl, p_hit=1.0, seed=4)
    n1 = 30000
    _, ehits = oracle_policy(oracle, rules, d1_t.numpy(), o1_t.numpy().astype(np.uint32))
    st = torch.cuda.Stream()

    rs = N.Ruleset(rules, strict=True)
    d0, o0 = to_device(torch, d0_t.numpy(), o0_t.numpy())
    d1, o1 = to_device(torch, d1_t.numpy(), o1_t.numpy())
    small, big = HitsOut(torch, 64, 1024), HitsOut(torch, n1, 4 * n1)
    small.issue(rs, d0, o0, st.cuda_stream)
    big.issue(rs, d1, o1, st.cuda_stream)
    with pytest.raises(N.GovError) as ei:
        rs.scan_join(st.cuda_stream)
    assert ei.value.code == N.CG_ERR_CAPACITY
    nh, _, _, words = big.result()
    assert nh == ALL_ONES and (big.hits.cpu().numpy().view(np.uint32) == GUARD).all()
    assert (words == np.uint64(0xffffffffffffffff)).all()
    for attempt in range(4):                                          # (a slot overflow hides how many VM events the batch needs)
        big.issue(rs, d1, o1, st.cuda_stream)
        try:
            rs.scan_join(st.cuda_stream)
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
            assert big.nh() == ALL_ONES
    nh, pairs, guard, words = big.result()
    assert nh == len(ehits) and pairs == ehits and (guard == GUARD).all()
    assert int((words >> np.uint64(63)).sum()) >= 29000
    rs.close()

    rs = N.Ruleset(rules, strict=True)
    rng = np.random.default_rng(64)
    pol = np.sort(rng.integers(0, 20, len(rules))).astype(np.uint32)
    act = rng.integers(0, 3, len(rules)).astype(np.uint8)
    rs.set_policy(pol, act)
    vs = torch.full((64,), 7, dtype=torch.int32, device="cuda")
    vb = torch.full((n1 + 16,), GUARD, dtype=torch.int32, device="cuda")
    rs.verdict_batch_device(d0.data_ptr(), o0.data_ptr(), 64, vs.data_ptr(), st.cuda_stream)
    rs.verdict_batch_device(d1.data_ptr(), o1.data_ptr(), n1, vb.data_ptr(), st.cuda_stream)
    with pytest.raises(N.GovError) as ei:
        rs.scan_join(st.cuda_stream)
    assert ei.value.code == N.CG_ERR_CAPACITY
    got = vb.cpu().numpy().view(np.uint32)
    assert (got[:n1] == ALL_ONES).all() and (got[n1:] == GUARD).all()
    assert np.array_equal(verdicts_device(N, torch, rs, d1_t.numpy(), o1_t.numpy().astype(np.uint32), st.cuda_stream),
                          rs.verdict_batch(d1_t.numpy(), o1_t.numpy().astype(np.uint32)))
    rs.close()


# ------------------------------------------------------------------------------ 4. verdicts

def test_device_verdicts_equal_host_verdicts(N, torch):
    """random policy lists over 500 rules: cg_policy_verdict_batch_device == cg_policy_verdict_batch; without a policy the
    call is rejected before anything is enqueued"""
    rl = W.make_rules(500)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(20000, 256, rl, p_hit=0.10, seed=500)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    d, o = to_device(torch, data, off)
    out = torch.full((20000,), GUARD, dtype=torch.int32, device="cuda")
    with pytest.raises(N.GovError) as ei:
        rs.verdict_batch_device(d.data_ptr(), o.data_ptr(), 20000, out.data_ptr())
    assert ei.value.code == -1
    torch.cuda.synchronize()
    assert (out.cpu().numpy().view(np.uint32) == GUARD).all()
    rng = np.random.default_rng(4)
    for trial in range(3):
        pol = np.sort(rng.integers(0, 30 + 100 * trial, len(rules))).astype(np.uint32)
        act = rng.integers(0, 3, len(rules)).astype(np.uint8)
        rs.set_policy(pol, act)
        want = rs.verdict_batch(data, off)
        got = verdicts_device(N, torch, rs, data, off)
        assert np.array_equal(got, want), [(i, hex(a), hex(b)) for i, (a, b) in enumerate(zip(got, want)) if a != b][:5]
        assert (want != 0).sum() > 1000 and (want == 0).sum() > 1000
    rs.verdict_batch_device(d.data_ptr(), o.data_ptr(), 0, out.data_ptr())      # n = 0: nothing to do
    rs.scan_join()
    rs.close()


# ------------------------------------------------------------------------------ 5. streams and edge cases

def test_two_batches_on_one_stream_before_one_join(N, torch):
    rl = W.make_rules(500)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    st = torch.cuda.Stream()
    batches = []
    for seed in (11, 12):
        data_t, off_t, _ = W.make_messages(8000, 256, rl, p_hit=0.05, seed=seed)
        batches.append((data_t.numpy(), off_t.numpy().astype(np.uint32)))
    expect = [rs.scan_batch(dd, oo) for dd, oo in batches]
    dev = [to_device(torch, dd, oo) for dd, oo in batches]
    outs = [HitsOut(torch, 8000, 4096) for _ in batches]
    torch.cuda.synchronize()
    for rep in range(2):
        for (d, o), ho in zip(dev, outs):
            ho.issue(rs, d, o, st.cuda_stream)
        rs.scan_join(st.cuda_stream)
        for ho, (ew, eh) in zip(outs, expect):
            nh, pairs, guard, words = ho.result()
            assert pairs == host_pairs(eh) and nh == len(eh) and (guard == GUARD).all()
            assert np.array_equal(words, ew)
    rs.close()


def test_small_batches_and_empty_messages(N, torch, oracle):
    """n = 0 writes 0 to the count; n = 1 with and without hits; empty messages among messages that hit"""
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    d, o = to_device(torch, np.zeros(16, np.uint8), np.zeros(1, np.uint32))
    ho = HitsOut(torch, 0, 16)
    ho.issue(rs, d, o)
    rs.scan_join()
    assert ho.nh() == 0 and (ho.hits.cpu().numpy().view(np.uint32) == GUARD).all()
    tok = [r["sample"].encode() for r in rl[:40]]
    cases = [[b"x " + tok[3] + b" " + tok[20]], [b"nothing here"], [b""],
             [b"", tok[0], b"", b"", b" ".join(tok), b"", tok[17] + tok[39], b""]]
    for msgs in cases:
        data, off = N.pack(msgs)
        _, ehits = oracle_policy(oracle, rules, data, off)
        words, pairs = hits_device(N, torch, rs, data, off)
        assert pairs == ehits, msgs
        assert host_pairs(rs.scan_batch(data, off)[1]) == ehits
    assert len(oracle_policy(oracle, rules, *N.pack(cases[-1]))[1]) >= 40
    rs.close()


def test_launch_count_does_not_depend_on_the_hit_count(N, torch):
    rl = W.make_rules(500)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    counts = []
    for p_hit in (0.0, 1.0):
        data_t, off_t, _ = W.make_messages(4096, 256, rl, p_hit=p_hit, seed=21)
        data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
        hits_device(N, torch, rs, data, off)                          # (scratch grown for this batch)
        d, o = to_device(torch, data, off)
        ho = HitsOut(torch, 4096, 1 << 16)
        k0 = N.launch_count()
        ho.issue(rs, d, o)
        counts.append(N.launch_count() - k0)
        rs.scan_join()
        counts.append(ho.nh())
    assert counts[0] == counts[2] and counts[1] < 100 and counts[3] >= 4096
    rs.close()


def test_statistics_count_hits_as_the_host_call_does(N, torch, oracle):
    rl = W.make_rules(500)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(5000, 256, rl, p_hit=0.10, seed=31)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    _, ehits = oracle_policy(oracle, rules, data, off)
    hits_device(N, torch, rs, data, off)                              # (no overflow below)
    s0 = N.stats().hits
    hits_device(N, torch, rs, data, off)
    s1 = N.stats().hits
    rs.scan_batch(data, off)
    s2 = N.stats().hits
    assert s1 - s0 == s2 - s1 == len(ehits) > 0
    rs.close()
