"""GPU tier, structure of the device path: launch geometry that changes with the batch size, kernel variants picked from
the compiled rule set, host-side path switches (hit-row width, single-message fast path, chunked host batches, cached
graphs), the verdict kernel and the device-resident Merkle calls.  Every result is compared bit-exactly with the CPU
oracle or hashlib.  Run on an H100: pytest -m gpu."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from test_gpu_parity import oracle_policy, oracle_spans
from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu

ROUND_PER_CTA = 4 * 32 * 512        # bytes one scan CTA covers per round: four 512-byte tiles for each of its 32 warps


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def scan_grid(n, sms):
    """the scan's grid for n messages (scan_kernels.cu: one CTA per SM, fewer for batches below 4096 messages)"""
    return sms if n >= 4096 else max(1, min(sms, n // 32 + 1))


def hit_pairs(hits):
    return [(int(h["msg"]), int(h["rule"])) for h in hits]


def span_tuples(spans):
    return [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in spans]


def device_words(N, rs, data, off, stream=None):
    """cg_scan_batch_device over the whole batch -> words (host copy)"""
    import torch
    n = len(off) - 1
    d = torch.from_numpy(np.ascontiguousarray(data)).cuda()
    o = torch.from_numpy(off.astype(np.int32)).cuda()
    out = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    st = stream or torch.cuda.Stream()
    torch.cuda.synchronize()
    rs.scan_batch_device(d.data_ptr(), o.data_ptr(), n, out.data_ptr(), st.cuda_stream)
    rs.scan_join(st.cuda_stream)
    return out.cpu().numpy().view(np.uint64)


def filler(rl, length, seed):
    return W.make_messages(1, length, rl, p_hit=0.0, seed=seed)[0].numpy()[:length].copy()


# ------------------------------------------------------------------------------ A. scan step at its boundaries

class GridBatch:
    """One flat text with rule tokens planted at the first bytes, across 512-byte tile boundaries and across the round
    boundaries of every grid the batch sizes of a group can get, cut into messages without splitting a token.  A batch
    of n messages is the first n - 1 cut messages plus one last message that runs to the end of the text (trimmed so that
    the batch's length has the wanted residue mod 16) and ends with a token on its last byte."""

    def __init__(self, oracle, rl, rules, n_max, grids, total, seed):
        rng = np.random.default_rng(seed)
        self.rl, self.rules, self.oracle = rl, rules, oracle
        self.flat = filler(rl, total, seed)
        busy = np.zeros(total + 1, dtype=bool)
        samples = [r["sample"].encode() for r in rl]

        def put(at, tok):
            if at < 0 or at + len(tok) > total - 64 or busy[at:at + len(tok)].any():
                return False
            self.flat[at:at + len(tok)] = np.frombuffer(tok, dtype=np.uint8)
            busy[at:at + len(tok)] = True
            return True

        assert put(0, samples[int(rng.integers(0, len(samples)))] + b" ")
        bounds = set(range(512, min(total, 48 * 512), 512))
        for g in grids:
            bounds |= set(range(g * ROUND_PER_CTA, total, g * ROUND_PER_CTA))
        self.planted = 1
        for b in sorted(bounds):
            tok = b" " + samples[int(rng.integers(0, len(samples)))] + b" "
            self.planted += put(b - int(rng.integers(1, len(tok))), tok)
        cand = rng.choice(np.arange(1, total - 64), 2 * n_max, replace=False)
        for i in range(len(cand)):
            while busy[cand[i] - 1] and busy[cand[i]]:                     # (never inside a token)
                cand[i] += 1
        cand = np.unique(cand)
        cuts = np.sort(rng.choice(cand, n_max - 1, replace=False))
        self.cuts = np.concatenate([[0], cuts]).astype(np.int64)
        # messages 0 .. n_max - 2 are the same in every batch: their oracle results once
        data = np.concatenate([self.flat[:self.cuts[-1]], np.zeros(64, np.uint8)])
        off = self.cuts.astype(np.uint32)
        self.base_words, self.base_hits = oracle_policy(oracle, rules, data, off)
        self.samples = samples
        self.rng = rng

    def batch(self, n, residue):
        tok = b" " + self.samples[int(self.rng.integers(0, len(self.samples)))]
        start = int(self.cuts[n - 1])
        trim = (len(self.flat) + len(tok) - residue) % 16
        last = np.concatenate([self.flat[start:len(self.flat) - trim], np.frombuffer(tok, dtype=np.uint8)])
        data = np.concatenate([self.flat[:start], last, np.zeros(64, np.uint8)])
        off = np.concatenate([self.cuts[:n], [start + len(last)]]).astype(np.uint32)
        assert int(off[-1]) % 16 == residue
        lw, lh = oracle_policy(self.oracle, self.rules, np.concatenate([last, np.zeros(64, np.uint8)]),
                               np.array([0, len(last)], dtype=np.uint32))
        words = np.concatenate([self.base_words[:n - 1], lw])
        hits = [h for h in self.base_hits if h[0] < n - 1] + [(n - 1, r) for (_, r) in lh]
        return data, off, words, hits


@pytest.fixture(scope="module")
def grid_rules():
    rl = W.make_rules(40)
    return rl, W.rules_as_tuples(rl)


@pytest.mark.parametrize("group", ["small", "large"])
def test_scan_around_the_grid_rule(N, oracle, grid_rules, group):
    """n in {1, 31, 32, 33} and {4095, 4096, 4097} (the grid changes at n / 32 + 1 and at 4096), buffer lengths 0, 1 and
    15 mod 16, tokens at the head of the range, across tile and round boundaries and on the last byte: words and hit
    list of the host path and words of the device path equal the oracle's."""
    rl, rules = grid_rules
    sms = sm_count()
    ns = [1, 31, 32, 33] if group == "small" else [4095, 4096, 4097]
    grids = sorted({scan_grid(n, sms) for n in ns})
    total = max(grids) * ROUND_PER_CTA * (3 if group == "small" else 1) + 150000
    gb = GridBatch(oracle, rl, rules, max(ns), grids, total, seed=4096 + len(ns))
    assert gb.planted >= 30
    rs = N.Ruleset(rules, strict=True)
    for n in ns:
        for residue in (0, 1, 15):
            data, off, ewords, ehits = gb.batch(n, residue)
            words, hits = rs.scan_batch(data, off)
            assert np.array_equal(words, ewords), (n, residue)
            assert hit_pairs(hits) == ehits, (n, residue)
            assert np.array_equal(device_words(N, rs, data, off), ewords), (n, residue)
            assert int(ewords[-1]) >> 63 and int(ewords[0]) >> 63          # the last byte's token, the head's token
    rs.close()


def test_scan_of_a_dense_batch(N, oracle, grid_rules):
    """Traffic made of rule-literal fragments flags a gram in most 16-byte chunks: every warp's 64-entry ring wraps many
    times and flushes a remainder at the end; host and device path equal the oracle."""
    rl, rules = grid_rules
    rs = N.Ruleset(rules, strict=True)
    n, length = 33, 65536
    data_t, off_t, _ = W.make_messages(n, length, rl, p_hit=0.5, seed=55, frag_frac=1.0)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    words, hits = rs.scan_batch(data, off)
    assert np.array_equal(words, ewords) and hit_pairs(hits) == ehits
    flagged = rs.work_counters()[6]
    print("flagged grams:", flagged, "16-byte chunks:", n * length // 16)
    assert flagged >= n * length // 16 // 4
    assert np.array_equal(device_words(N, rs, data, off), ewords)
    rs.close()


LITS = [("alphabetagamma", 0, 3), ("thequickbrownfox", 0, 3), ("zeppelin_airship", 1, 3)]
R_OK, R_AT, R_HASH, R_PCT = ("ok", 0, 3), (r"\w+@\w+", 0, 3), (r"\w+#\w+", 0, 2), (r"\d+%\d+", 0, 1)


# (rule set, options) -> (stride, triggers, always-candidate rules) it must compile to; stride 4 = one probe per chunk word
VARIANTS = [
    (LITS, 4, (4, 0, 0)),
    (LITS + [R_AT], 4, (4, 1, 0)),
    (LITS + [R_AT, R_HASH], 4, (4, 2, 0)),
    (LITS + [R_AT, R_HASH, R_PCT], 4, (4, 2, 1)),          # a third uncoverable factor: every message is a candidate
    (LITS + [R_OK], 2, (2, 0, 0)),
    (LITS + [R_OK, R_AT], 2, (2, 1, 0)),
    (LITS + [R_OK, R_AT, R_HASH], 2, (2, 2, 0)),
]


@pytest.mark.parametrize("rules,options,want", VARIANTS, ids=["s%d-t%d-a%d" % v[2] for v in VARIANTS])
def test_scan_kernel_variants(N, oracle, rules, options, want):
    """Each compiled scan_kernel variant (one or two probes per chunk word x zero, one or two trigger bytes) is shown to
    be the one compiled (Ruleset.info) and its words, hits and spans equal the oracle's; trigger bytes sit at every
    alignment in the 16-byte chunks, at the head of the range and on the last byte."""
    rs = N.Ruleset(rules, options=options, strict=True)
    info = rs.info()
    assert (info.stride, info.n_triggers, info.n_always_candidate) == want
    rng = np.random.default_rng(sum(want) * 7 + len(rules))
    toks = [b"alphabetagamma", b"thequickbrownfox", b"ZEPPELIN_Airship", b"ok", b"bob@example", b"x@y", b"a1#b2", b"7#z",
            b"12%34", b"@", b"#", b"%", b"alphabetagamm", b"a@", b"#b", b"o k"]
    words = [b"lorem", b"ipsum", b"dolor", b"sit", b"amet", b"q", b"zz", b"12", b"--"]
    msgs = [b"bob@example", b"a1#b2 x", b"12%34"]                          # triggers on the first bytes of the range
    for i in range(700):
        parts = []
        for _ in range(int(rng.integers(0, 7))):
            pool = toks if rng.random() < 0.4 else words
            parts.append(pool[int(rng.integers(0, len(pool)))])
        pad = b"." * int(rng.integers(0, 16))                               # every alignment of what follows
        msgs.append(pad + b" ".join(parts))
    msgs.append(b"tail " * 5 + b"end@x")                                     # a trigger on the last byte
    data, off = N.pack(msgs)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert len({r for _, r in ehits}) == len(rules)
    w, h = rs.scan_batch(data, off)
    assert np.array_equal(w, ewords) and hit_pairs(h) == ehits
    assert span_tuples(rs.find_matches_batch(data, off)) == oracle_spans(oracle, rules, data, off)
    assert np.array_equal(device_words(N, rs, data, off), ewords)
    rs.close()


@pytest.mark.parametrize("n_rules", [1, 31, 32, 33, 63, 64, 65])
def test_hit_row_width(N, oracle, n_rules):
    """Rule counts around each multiple of 32 (the hit row's width in words): tokens of the last rule and of the rules on
    either side of every word boundary -- the words' count and lowest-rule fields, the hit list and scan_one."""
    rl = W.make_rules(n_rules)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    targets = sorted({0, n_rules - 1} | {k for k in (30, 31, 32, 33, 62, 63, 64) if k < n_rules})
    rng = np.random.default_rng(n_rules)
    body = filler(rl, 300 * 96, seed=n_rules)
    msgs = []
    for i in range(300):
        m = bytes(body[i * 96:i * 96 + int(rng.integers(0, 96))])
        for _ in range(int(rng.integers(0, 4))):
            r = targets[int(rng.integers(0, len(targets)))]
            p = int(rng.integers(0, len(m) + 1))
            m = m[:p] + b" " + rl[r]["sample"].encode() + b" " + m[p:]
        msgs.append(m)
    msgs.append(b" ".join(rl[r]["sample"].encode() for r in targets))
    data, off = N.pack(msgs)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert {r for _, r in ehits} >= set(targets)
    words, hits = rs.scan_batch(data, off)
    assert np.array_equal(words, ewords) and hit_pairs(hits) == ehits
    for i, m in enumerate(msgs):
        w1, r1 = rs.scan_one(m)
        assert w1 == int(ewords[i]) and r1 == [r for (mm, r) in ehits if mm == i], i
    rs.close()


def test_scan_one_fast_and_general_path_at_4032_rules(N, oracle):
    """cg_scan_one keeps its single-graph fast path up to 4032 rules (126 hit words); 4033 rules take the general path.
    Both equal scan_batch and the oracle, with tokens on the rules next to every word boundary at the top."""
    rl = W.make_rules(4033)
    rng = np.random.default_rng(4033)
    targets = [0, 31, 32, 4000, 4030, 4031, 4032]
    body = filler(rl, 250 * 128, seed=4033)
    msgs = []
    for i in range(250):
        m = bytes(body[i * 128:i * 128 + int(rng.integers(0, 128))])
        if i % 2:
            r = targets[int(rng.integers(0, len(targets)))]
            m += b" " + rl[r]["sample"].encode()
        msgs.append(m)
    msgs.append(b" ".join(rl[r]["sample"].encode() for r in targets))
    data, off = N.pack(msgs)
    for n_rules in (4032, 4033):
        rules = W.rules_as_tuples(rl[:n_rules])
        rs = N.Ruleset(rules, strict=True)
        ewords, ehits = oracle_policy(oracle, rules, data, off)
        assert {r for _, r in ehits} >= {r for r in targets if r < n_rules}
        words, hits = rs.scan_batch(data, off)
        assert np.array_equal(words, ewords) and hit_pairs(hits) == ehits
        for i, m in enumerate(msgs):
            w1, r1 = rs.scan_one(m)
            assert w1 == int(ewords[i]) and r1 == [r for (mm, r) in ehits if mm == i], (n_rules, i)
        rs.close()


def oracle_words_sampled(oracle, rules, data, off, step):
    """the oracle's words of every step-th message (a batch of those messages alone)"""
    idx = np.arange(0, len(off) - 1, step)
    msgs = [bytes(data[int(off[i]):int(off[i + 1])]) for i in idx]
    from vainplex_openclaw_b200._native import pack
    d, o = pack(msgs)
    return idx, oracle_policy(oracle, rules, d, o)[0]


def test_host_batch_one_piece_chunked_and_overflow_fallback(N, oracle):
    """Words-only host batches of 65536 messages or more are scanned in pieces: 65535 messages (one piece) and 65536 (the
    chunked path) give the same words for the same messages.  On a fresh rule set a batch in which every message hits
    overflows a piece's queues, and the call falls back to one piece (more kernels than the same call once the
    capacities have grown); its words equal the one-piece result and the oracle's."""
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    n = 65536
    data_t, off_t, _ = W.make_messages(n, 64, rl, p_hit=0.05, seed=65536)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    rs = N.Ruleset(rules, strict=True)
    w_one, _ = rs.scan_batch(data, off[:n], want_hits=False)              # 65535 messages
    w_chunk, _ = rs.scan_batch(data, off, want_hits=False)                # 65536 messages
    assert np.array_equal(w_one, w_chunk[:n - 1])
    idx, ew = oracle_words_sampled(oracle, rules, data, off, 17)
    assert np.array_equal(w_chunk[idx], ew)
    rs.close()

    data_t, off_t, _ = W.make_messages(n, 64, rl, p_hit=1.0, seed=65537)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    rs = N.Ruleset(rules, strict=True)
    k0 = N.launch_count()
    w_first, _ = rs.scan_batch(data, off, want_hits=False)
    k1 = N.launch_count()
    w_again, _ = rs.scan_batch(data, off, want_hits=False)
    k2 = N.launch_count()
    assert k1 - k0 > k2 - k1, (k1 - k0, k2 - k1)                          # the first call ran the pieces and then one piece
    w_hits, hits = rs.scan_batch(data, off, want_hits=True)
    assert np.array_equal(w_first, w_again) and np.array_equal(w_first, w_hits)
    assert int((w_first >> np.uint64(63)).sum()) >= 0.9 * n
    idx, ew = oracle_words_sampled(oracle, rules, data, off, 17)
    assert np.array_equal(w_first[idx], ew)
    rs.close()


def test_device_graph_cache_eviction_and_set_policy(N, oracle):
    """Three (buffer, n) configurations alternate on one rule set, so the two cached graphs are evicted over and over;
    set_policy (which drops the cached graphs) is called between device-path calls.  Every output equals the oracle's."""
    import torch
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    cfgs = []
    for k, n in enumerate((700, 1500, 3100)):
        data_t, off_t, _ = W.make_messages(n, 160, rl, p_hit=0.2, seed=700 + k)
        data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
        want, _ = oracle_policy(oracle, rules, data, off)
        d = torch.from_numpy(data).cuda()
        o = torch.from_numpy(off.astype(np.int32)).cuda()
        out = torch.full((n,), -1, dtype=torch.int64, device="cuda")
        cfgs.append((d, o, out, n, want))
    rng = np.random.default_rng(3)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for step, k in enumerate([0, 1, 2, 0, 1, 2, 2, 0, 0, 1, 2, 1]):     # misses that evict, and hits
        d, o, out, n, want = cfgs[k]
        out.fill_(-1)
        torch.cuda.synchronize()
        rs.scan_batch_device(d.data_ptr(), o.data_ptr(), n, out.data_ptr(), st.cuda_stream)
        rs.scan_join(st.cuda_stream)
        assert np.array_equal(out.cpu().numpy().view(np.uint64), want), step
        if step in (4, 7, 8):
            rs.set_policy(np.sort(rng.integers(0, 30, len(rules))), rng.integers(0, 3, len(rules)))
    rs.close()


# ------------------------------------------------------------------------------ B. verdicts against an independent aggregation

def expected_verdicts(hits, n, rule_policy, rule_action):
    """openclaw_gov.h, cg_policy_verdict_batch, applied to the oracle's hit list: per policy its first matching rule
    counts; deny beats audit beats allow; the first policy with the winning action decides; matched policies saturate
    at 1023; deciding rule 0xfffff when no deny / audit rule matched; 0 when nothing matched."""
    out = np.zeros(n, dtype=np.uint32)
    by_msg = {}
    for m, r in hits:
        by_msg.setdefault(m, []).append(r)
    for m, rs in by_msg.items():
        first = {}
        for r in sorted(rs):
            first.setdefault(int(rule_policy[r]), r)
        deciding = [(p, r) for p, r in first.items() if rule_action[r] == 2] or [(p, r) for p, r in first.items() if rule_action[r] == 1]
        action, rule = (int(rule_action[min(deciding)[1]]), min(deciding)[1]) if deciding else (0, 0xfffff)
        out[m] = action | min(len(first), 1023) << 2 | rule << 12
    return out


def test_verdicts_equal_the_oracle_aggregation(N, oracle):
    """Random policy lists over 160 rules (five hit words): messages with several tokens, only allow rules, no match."""
    rl = W.make_rules(160)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    rng = np.random.default_rng(160)
    body = filler(rl, 900 * 80, seed=160)
    msgs = []
    for i in range(900):
        m = bytes(body[i * 80:i * 80 + int(rng.integers(0, 80))])
        for _ in range(int(rng.integers(0, 5)) if i % 3 else int(i % 2)):
            r = int(rng.integers(0, len(rl)))
            m += b" " + rl[r]["sample"].encode() + b" "
        msgs.append(m)
    data, off = N.pack(msgs)
    _, ehits = oracle_policy(oracle, rules, data, off)
    for trial in range(3):
        pol = np.sort(rng.integers(0, 40 + 40 * trial, len(rules))).astype(np.uint32)
        act = rng.integers(0, 3, len(rules)).astype(np.uint8)
        rs.set_policy(pol, act)
        want = expected_verdicts(ehits, len(msgs), pol, act)
        got = rs.verdict_batch(data, off)
        assert np.array_equal(got, want), [(i, hex(a), hex(b)) for i, (a, b) in enumerate(zip(got, want)) if a != b][:5]
        kinds = [(v & 3, v != 0) for v in want.tolist()]
        assert kinds.count((2, True)) >= 20 and kinds.count((1, True)) >= 20 and kinds.count((0, True)) >= 10 and kinds.count((0, False)) >= 50
    # allow rules only: every verdict that matched says allow with deciding rule 0xfffff
    act = np.zeros(len(rules), dtype=np.uint8)
    rs.set_policy(pol, act)
    want = expected_verdicts(ehits, len(msgs), pol, act)
    assert np.array_equal(rs.verdict_batch(data, off), want)
    assert all(v == 0 or (v & 3 == 0 and v >> 12 == 0xfffff) for v in want.tolist())
    # what set_policy rejects: the wrong length, action 3, a decreasing policy index
    for bad_pol, bad_act in ((pol[:-1], act[:-1]), (pol, np.where(np.arange(len(rules)) == 77, 3, act)),
                             (np.where(np.arange(len(rules)) == 90, 0, pol + 1), act)):
        with pytest.raises(N.GovError) as ei:
            rs.set_policy(bad_pol, bad_act)
        assert ei.value.code == -1
    rs.close()


def test_verdict_matched_policies_saturate(N, oracle):
    """1100 policies whose rules all match one shared token: the matched-policies field saturates at 1023."""
    n_pol = 1100
    rules, pol = [], []
    for p in range(n_pol):
        rules.append((r"(?:zebra42|q%dx)" % p, 0, 3)); pol.append(p)
        if p % 10 == 3:
            rules.append((r"zebra4\d", 0, 3)); pol.append(p)
    rs = N.Ruleset(rules, strict=True)
    rng = np.random.default_rng(1023)
    msgs = [b"say zebra42 now", b"zebra42", b"q17x and q1099x", b"zebra4x", b"", b"nothing"] * 5
    data, off = N.pack(msgs)
    _, ehits = oracle_policy(oracle, rules, data, off)
    for trial in range(3):
        act = rng.integers(0, 3, len(rules)).astype(np.uint8)
        if trial == 1:
            act[:900] = 0                                                   # the first deny / audit comes late
        if trial == 2:
            act[:] = 0                                                      # allow only
        rs.set_policy(np.array(pol, dtype=np.uint32), act)
        want = expected_verdicts(ehits, len(msgs), pol, act)
        assert np.array_equal(rs.verdict_batch(data, off), want)
        assert (want[0] >> 2) & 1023 == 1023 and (want[2] >> 2) & 1023 == 2 and want[3] == 0
    rs.close()


# ------------------------------------------------------------------------------ C. device-resident Merkle calls

MERKLE_NS = [1, 31, 32, 33, (1 << 15) - 1, 1 << 15, (1 << 15) + 1, 100003]
_block_roots_cache = {}


def oracle_block_roots(oracle, data, leaf, n, bl):
    key = (leaf, n, bl)
    if key not in _block_roots_cache:
        b = 1 << bl
        _block_roots_cache[key] = np.stack([np.frombuffer(oracle.merkle_root_fixed(data[s * leaf:], leaf, min(b, n - s)), dtype=np.uint8)
                                            for s in range(0, n, b)])
    return _block_roots_cache[key]


@pytest.mark.parametrize("n", MERKLE_NS)
def test_merkle_block_roots_fold_and_sharded_root_on_the_device(N, oracle, n):
    """cg_merkle_block_roots_device for block sizes 2^0 .. 2^40 (the per-level kernel / warp-reduction switch at 2^15),
    word-kernel leaves (32, 48 bytes), generic-kernel leaves (37 bytes, a pointer one byte off), on a caller stream and on
    the library's stream: every block root equals the oracle's root of that block and nothing past the last root is
    written; cg_merkle_fold_device over them and cg_merkle_root_sharded_device (one rank) equal the root of all leaves."""
    import torch
    L = N.load()
    bls = sorted({0, 1, 4, 5, 6, 15, 16, 17, max(0, (n - 1).bit_length()), 40})
    caller = torch.cuda.Stream()
    for leaf, shift in ((32, 0), (48, 0), (37, 0), (32, 1)):
        data = W.make_leaves(n, leaf, seed=n + leaf).numpy()
        root = oracle.merkle_root_fixed(data, leaf, n)
        buf = torch.zeros(len(data) + 16, dtype=torch.uint8, device="cuda")
        buf[shift:shift + len(data)] = torch.from_numpy(data).cuda()
        ptr = buf.data_ptr() + shift
        for bl in bls:
            want = oracle_block_roots(oracle, data, leaf, n, bl)
            nb = want.shape[0]
            out = torch.empty((nb + 1) * 32, dtype=torch.uint8, device="cuda")
            froot = torch.empty(64, dtype=torch.uint8, device="cuda")
            for st in (caller, None):
                out.fill_(0xA5); froot.fill_(0xA5)
                torch.cuda.synchronize()
                sp = st.cuda_stream if st is not None else None
                N.check(L.cg_merkle_block_roots_device(ptr, leaf, n, bl, out.data_ptr(), sp))
                N.check(L.cg_merkle_fold_device(out.data_ptr(), nb, froot.data_ptr(), sp))
                torch.cuda.synchronize()
                got = out.cpu().numpy()
                assert np.array_equal(got[:nb * 32].reshape(nb, 32), want), (leaf, shift, bl, st is None)
                assert (got[nb * 32:] == 0xA5).all()
                fr = froot.cpu().numpy()
                assert fr[:32].tobytes() == root and (fr[32:] == 0xA5).all(), (leaf, shift, bl)
            if bl in (0, 5, 16, 40):
                assert N.merkle_root_sharded_device(ptr, leaf, n, n, bl, caller.cuda_stream) == root
    if n == 1:
        assert N.merkle_root_sharded_device(ptr, 32, 0, 0, 4) == hashlib.sha256(b"").digest()
    with pytest.raises(N.GovError) as ei:
        N.merkle_root_sharded_device(ptr, 32, n - 1, n, 4)
    assert ei.value.code == -1


def test_merkle_block_roots_reject_block_log2_beyond_40(N):
    """block_log2 above 40 is rejected before any buffer is touched (the output keeps its guard bytes)."""
    import torch
    L = N.load()
    data = torch.from_numpy(W.make_leaves(100, 32, seed=1).numpy()).cuda()
    out = torch.full((4 * 32,), 0xA5, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for bl in (41, 64):
        assert L.cg_merkle_block_roots_device(data.data_ptr(), 32, 100, bl, out.data_ptr(), None) == -1
        with pytest.raises(N.GovError) as ei:
            N.merkle_root_sharded_device(data.data_ptr(), 32, 100, 100, bl)
        assert ei.value.code == -1
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == 0xA5).all()
