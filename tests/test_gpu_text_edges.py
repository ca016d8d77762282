"""GPU tier, text edges: every call's result for a message depends on that message's bytes only, decoded as TextDecoder
decodes them.  Neighbour messages whose bytes would change each other's answers (at every residue of the edge mod 16,
across 512-byte tiles, across the pieces of the chunked host path), bytes before and behind the scanned range, stale
bytes in the host staging buffers, and ill-formed UTF-8 with U+FFFD rules -- through the host, single-message and
device-resident calls, against the oracle, Python's UTF-8 decoder, hashlib and a Python restatement of the splice.
Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from helpers import (EDGE_PAIRS, EDGE_RULES, FFFD_ATOMS, FFFD_CASES, EdgeBatch, ill_formed_corpus, ill_formed_texts,
                     random_regex, unit_starts)
from test_gpu_boundaries import VARIANTS, expected_verdicts, hit_pairs
from test_gpu_parity import oracle_policy, oracle_spans
from test_gpu_redact_device import GUARD, FindOut, RedactOut, full, splice_python, to_device, tup

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


@pytest.fixture(scope="module")
def torch():
    import torch as T
    return T


def split_msgs(data, off):
    return [bytes(data[int(off[i]):int(off[i + 1])]) for i in range(len(off) - 1)]


class Expected:
    """the oracle's answers for a batch of messages (packed alone, zero padding), and the byte offsets of its spans"""

    def __init__(self, N, oracle, rules, msgs):
        self.msgs = msgs
        data, off = N.pack(msgs)
        self.words, self.hits = oracle_policy(oracle, rules, data, off)
        self.spans = oracle_spans(oracle, rules, data, off)
        starts = {}
        self.full = []
        for m, r, s, e in self.spans:
            st = starts.setdefault(m, unit_starts(msgs[m]))
            self.full.append((m, r, st[s], st[e], s, e))


def check_redaction(msgs, rules, spans, dig, out, out_off):
    assert [bytes(out[int(out_off[i]):int(out_off[i + 1])]) for i in range(len(msgs))] == splice_python(msgs, rules, spans, dig)


def device_results(N, torch, rs, d, o, n, spans_cap=1 << 16, out_cap=None):
    """the three device-resident calls over n messages at offsets tensor o (which may start inside a larger array) of
    device buffer d -> (words, spans, (out, out_off, spans, digests))"""
    st = torch.cuda.Stream()
    words = torch.full((max(n, 1),), -1, dtype=torch.int64, device="cuda")
    fo = FindOut(torch, spans_cap)
    ro = RedactOut(torch, n, out_cap or 8 * int(d.numel()) + 4096, spans_cap)
    torch.cuda.synchronize()
    rs.scan_batch_device(d.data_ptr(), o.data_ptr(), n, words.data_ptr(), st.cuda_stream)
    fo.issue(rs, d, o, n, st.cuda_stream)
    ro.issue(rs, d, o, st.cuda_stream)
    rs.scan_join(st.cuda_stream)
    ns, spans, guard = fo.result(N)
    assert ns == len(spans) and (guard == GUARD * 0x01010101).all()
    out, out_off, rspans, dig, _, _, _ = ro.result(N)
    return words.cpu().numpy().view(np.uint64)[:n], spans, (out, out_off[:n + 1], rspans, dig)


def check_every_call(N, torch, rs, rules, data, off, exp, seed=0):
    """scan_batch, find_matches_batch, redact_batch, verdict_batch and the three device calls over one packed batch
    against the oracle's answers for its messages"""
    msgs = exp.msgs
    n = len(msgs)
    words, hits = rs.scan_batch(data, off)
    assert np.array_equal(words, exp.words)
    assert hit_pairs(hits) == exp.hits
    spans = rs.find_matches_batch(data, off)
    assert tup(spans) == exp.spans and full(spans) == exp.full
    out, out_off, rspans, dig = rs.redact_batch(data, off)
    assert full(rspans) == exp.full
    check_redaction(msgs, rules, rspans, dig, out, out_off)
    rng = np.random.default_rng(seed)
    pol = np.sort(rng.integers(0, max(2, len(rules) // 2), len(rules))).astype(np.uint32)
    act = rng.integers(0, 3, len(rules)).astype(np.uint8)
    rs.set_policy(pol, act)
    assert np.array_equal(rs.verdict_batch(data, off), expected_verdicts(exp.hits, n, pol, act))
    d, o = to_device(torch, data, off)
    dwords, dspans, (dout, dout_off, drspans, ddig) = device_results(N, torch, rs, d, o, n, out_cap=len(out) + 64)
    assert np.array_equal(dwords, exp.words)
    assert full(dspans) == exp.full and full(drspans) == exp.full
    assert np.array_equal(dout, out) and np.array_equal(dout_off, out_off) and np.array_equal(ddig, dig)


# ------------------------------------------------------------------------------------------------ A. neighbour pairs

def test_neighbour_pairs_through_every_call(N, torch, oracle):
    """Each pair split over two messages (empty messages between some) and joined in one, the edge at every residue mod
    16 and within 8 bytes of a 512-byte tile boundary: every call equals the oracle, every pair's answers are the ones
    its name says (the joined controls hit where they should), and "€" cut as E2 82 | AC is two U+FFFD and no "€"."""
    eb = EdgeBatch(EDGE_PAIRS)
    exp = Expected(N, oracle, EDGE_RULES, eb.msgs)
    eb.check_hits(set(exp.hits))
    rs = N.Ruleset(EDGE_RULES, strict=True)
    check_every_call(N, torch, rs, EDGE_RULES, eb.data, eb.off, exp, seed=1)
    euro = [i for i, p in enumerate(EDGE_PAIRS) if p[0] == "euro-split"][0]
    by_msg = {}
    for s in exp.full:
        by_msg.setdefault(s[0], []).append(s[1:])
    for pi, res, edge, li, ri in eb.split:
        if pi == euro:
            assert by_msg[li] == [(11, 0, 2, 0, 1)] and by_msg[ri] == [(11, 0, 1, 0, 1)], res
    for pi, res, edge, mi in eb.joined:
        if pi == euro:
            assert by_msg[mi] == [(10, 0, 3, 0, 1)], res
    rs.close()


# tokens of the scan-kernel variants' rules cut in two (rule source -> (left, right))
VARIANT_SPLITS = {
    "alphabetagamma": (b"alphabetag", b"amma"), "thequickbrownfox": (b"thequick", b"brownfox"), "zeppelin_airship": (b"ZEPPELIN_", b"Airship"),
    r"\w+@\w+": (b"bob@", b"example"), r"\w+#\w+": (b"a1", b"#b2"), r"\d+%\d+": (b"12%", b"34"), "ok": (b"o", b"k"),
}


@pytest.mark.parametrize("rules,options,want", VARIANTS, ids=["s%d-t%d-a%d" % v[2] for v in VARIANTS])
def test_neighbour_pairs_on_scan_kernel_variants(N, torch, oracle, rules, options, want):
    """Every compiled scan_kernel variant (one or two probes per chunk word, zero to two trigger bytes, always-candidate
    rules): each rule's token cut over two messages at every residue of the edge misses, joined it hits."""
    pairs = [("%s-split" % src, ri, *VARIANT_SPLITS[src], ri % 2, (False, False, True)) for ri, (src, _, _) in enumerate(rules)]
    eb = EdgeBatch(pairs)
    exp = Expected(N, oracle, rules, eb.msgs)
    eb.check_hits(set(exp.hits))
    rs = N.Ruleset(rules, options=options, strict=True)
    info = rs.info()
    assert (info.stride, info.n_triggers, info.n_always_candidate) == want
    check_every_call(N, torch, rs, rules, eb.data, eb.off, exp, seed=len(rules))
    rs.close()


# ------------------------------------------------------------------------------------------------ B. bytes outside the range

def pair_stream():
    """the pairs' left and right messages one after the other: every message's neighbours would change its answer"""
    return [m for p in EDGE_PAIRS for m in (p[2], p[3])]


def test_bytes_before_and_behind_the_range(N, torch, oracle):
    """The device calls on a range whose neighbours in the buffer are not padding: the bytes before offsets[0] complete the
    first message's token (or break its guard), the 16-64 bytes behind offsets[n] complete the last one's; sub-ranges of
    the pair stream take the offsets pointer past the first messages, so the bytes on both sides are real neighbours.
    Results equal the zero-padded batch of the same messages on the host calls, and the oracle."""
    rs = N.Ruleset(EDGE_RULES, strict=True)
    msgs = pair_stream()
    checked = 0
    for pre, tail in ((b"", b"\0" * 64), (b"alphabe" + b"X" * 9, b"tagamma" + b"Q" * 9), (b"\xe2\x82" + b"7" * 30, b"9" * 40 + b"\x80" * 24),
                      (b"na\xc3" * 16, b"\xaf" * 16), (b"key_" + b"a" * 60, b"a" * 64), (b"bob" * 11, b"@example" * 8)):
        assert 16 <= len(tail) <= 64
        for k, m in ((0, len(msgs)), (1, len(msgs) - 2), (2, 1), (3, 1), (5, 3), (9, 6), (16, 1), (17, 1), (18, 2), (35, 1), (36, 4)):
            sub = msgs[k:k + m]
            packed = pre + b"".join(msgs)
            off = (len(pre) + np.cumsum([0] + [len(x) for x in msgs])).astype(np.uint32)
            # behind the sub-range: the next message, then the tail; the buffer ends 16 bytes behind the range at the least
            data = np.frombuffer(packed + tail, dtype=np.uint8).copy()
            exp = Expected(N, oracle, EDGE_RULES, sub)
            zdata, zoff = N.pack(sub)
            host_spans = rs.find_matches_batch(zdata, zoff)
            h_out, h_off, h_rspans, h_dig = rs.redact_batch(zdata, zoff)
            assert tup(host_spans) == exp.spans and full(host_spans) == exp.full
            d = torch.from_numpy(data).cuda()
            o = torch.from_numpy(off.astype(np.int32)).cuda()
            words, spans, (out, out_off, rspans, dig) = device_results(N, torch, rs, d, o[k:], len(sub), out_cap=len(h_out) + 64)
            assert np.array_equal(words, exp.words), (pre, k, m)
            assert full(spans) == exp.full and full(rspans) == exp.full, (pre, k, m)
            assert np.array_equal(out, h_out) and np.array_equal(out_off, h_off) and np.array_equal(dig, h_dig), (pre, k, m)
            checked += 1
    assert checked == 66
    rs.close()


# ------------------------------------------------------------------------------------------------ C. stale staging

def test_stale_staging_bytes_on_the_host_calls(N, oracle):
    """A long batch, then a batch made of its prefix whose last message ends where the long batch's next message
    completed its token (or broke its guard): the host calls stage both batches in the same grow-only buffer.  Then the
    single-message calls, each message after a longer one whose tail would complete its token."""
    rs = N.Ruleset(EDGE_RULES, strict=True)
    pol, act = np.arange(len(EDGE_RULES), dtype=np.uint32), np.full(len(EDGE_RULES), 2, dtype=np.uint8)
    rs.set_policy(pol, act)
    msgs = [b"w" * 700] + pair_stream()
    whole = N.pack(msgs)
    for k in range(2, len(msgs), 2):                      # the prefix ends with a pair's left message
        for data, off in (whole, N.pack(msgs[:k])):
            exp = Expected(N, oracle, EDGE_RULES, split_msgs(data, off))
            words, hits = rs.scan_batch(data, off)
            assert np.array_equal(words, exp.words) and hit_pairs(hits) == exp.hits, k
            assert full(rs.find_matches_batch(data, off)) == exp.full, k
            out, out_off, rspans, dig = rs.redact_batch(data, off)
            assert full(rspans) == exp.full
            check_redaction(exp.msgs, EDGE_RULES, rspans, dig, out, out_off)
            assert np.array_equal(rs.verdict_batch(data, off), expected_verdicts(exp.hits, len(exp.msgs), pol, act))
    hits_seen = 0
    for _name, _r, left, right, _e, want in EDGE_PAIRS:
        for longer, m in ((left + right, left), (b"x" + left + right, b"x" + left), (left + right + right, left + right)):
            exp = Expected(N, oracle, EDGE_RULES, [m])
            rs.scan_one(longer); rs.find_matches_one(longer); rs.redact_one(longer)
            word, rules_hit = rs.scan_one(m)
            assert word == int(exp.words[0]) and rules_hit == [r for _, r in exp.hits], m
            rs.find_matches_one(longer)
            assert full(rs.find_matches_one(m)) == exp.full, m
            rs.redact_one(longer)
            out, spans, dig = rs.redact_one(m)
            assert full(spans) == exp.full
            assert [out] == splice_python([m], EDGE_RULES, spans, dig)
            hits_seen += bool(exp.hits)
    assert hits_seen >= 20
    rs.close()


# ------------------------------------------------------------------------------------------------ D. chunked host pieces

@pytest.mark.parametrize("n", [65536, 65543, 70001])
def test_tokens_across_the_pieces_of_the_chunked_host_path(N, oracle, n):
    """Words-only host batches of 65536 messages or more are scanned in eight pieces of ceil(n / 8) messages, each piece
    reading up to 16 bytes into the next one while that is still being copied.  At every piece edge a pair is cut (the
    pairs in turn): words equal the oracle's, each pair answers as its name says, and the joined controls placed beside
    each edge hit.  The chunked call launches more kernels than a one-piece batch of 65535 messages."""
    rs = N.Ruleset(EDGE_RULES, strict=True)
    per = -(-n // 8)
    msgs = [(b"filler %d " % i) * (1 + i % 3) for i in range(n)]
    split, joined = [], []
    for c in range(1, 8):
        name, r, left, right, _e, want = EDGE_PAIRS[(3 * c + n) % len(EDGE_PAIRS)]
        msgs[c * per - 1], msgs[c * per] = left, right
        msgs[c * per + 2] = left + right
        split.append((c * per - 1, c * per, r, want, name))
        joined.append((c * per + 2, r, want, name))
    data, off = N.pack(msgs)
    assert [c * per for c in range(1, 8)] == [e[1] for e in split] and all(e[1] < n for e in split)
    ewords, ehits = oracle_policy(oracle, EDGE_RULES, data, off)
    hs = set(ehits)
    for li, ri, r, want, name in split:
        assert ((li, r) in hs, (ri, r) in hs) == want[:2], name
    for mi, r, want, name in joined:
        assert ((mi, r) in hs) == want[2], name
    rs.scan_batch(data, off, want_hits=False)                # (sizes the scratch: the measured calls do not grow it)
    k0 = N.launch_count()
    words, _ = rs.scan_batch(data, off, want_hits=False)
    k1 = N.launch_count()
    assert np.array_equal(words, ewords)
    one, _ = rs.scan_batch(data, off[:65536], want_hits=False)
    k2 = N.launch_count()
    assert np.array_equal(one, ewords[:65535])
    assert k1 - k0 > k2 - k1, (k1 - k0, k2 - k1)
    rs.close()


# ------------------------------------------------------------------------------------------------ E. ill-formed text

def test_random_rules_on_ill_formed_text(N, torch, oracle):
    """The CPU tier's random differential on ill-formed text as one rule set through every call: words, hits, spans
    with byte offsets, redaction.  The patterns are flat sequences of quantified atoms (no groups), so that the oracle's
    backtracking stays short on these longer texts."""
    rng = np.random.default_rng(90210)
    msgs = ill_formed_texts(rng, 600, max_pieces=20) + [t for _, t, _ in FFFD_CASES] + ill_formed_corpus()
    data, off = N.pack(msgs)
    rules = []
    while len(rules) < 120:
        src = random_regex(rng, depth=2, atoms=FFFD_ATOMS)
        fl = 1 if rng.random() < 0.2 else 0
        try:
            rx = oracle.Regex(src, "i" if fl else "")
            oracle.scan_policy([rx], data, off.astype(np.uint64))
        except (oracle.RegexSyntaxError, oracle.OracleUnsupported, RuntimeError):
            continue
        if N.rule_check(src, fl) == 0:
            rules.append((src, fl, int(rng.integers(0, 4))))
    assert sum("FFFD" in r[0] for r in rules) >= 15
    exp = Expected(N, oracle, rules, msgs)
    assert len(exp.hits) >= 3000
    rs = N.Ruleset(rules, strict=True)
    check_every_call(N, torch, rs, rules, data, off, exp, seed=3)
    rs.close()


FFFD_RULES = [(src, 0, 1) for src, _, _ in FFFD_CASES] + [(r"\uFFFD{2}", 1, 0), (r"[^\x00-\x7f]+", 0, 3), (r"\W+", 0, 2), (r"\w+", 0, 3)]


def test_fffd_rules_and_redaction_on_ill_formed_text(N, torch, oracle):
    """U+FFFD literals in policy mode (the filter's factor alone used to decide them) and in span mode, on the four
    cases the filter missed and on every ill-formed sequence in context; redaction of those messages: bytes against the
    splice restated in Python, digests against hashlib over the raw span bytes.  The single-message calls agree."""
    msgs = [t for _, t, _ in FFFD_CASES] + ill_formed_corpus() + [b"pad " * k + t for k in (1, 4, 5) for _, t, _ in FFFD_CASES]
    exp = Expected(N, oracle, FFFD_RULES, msgs)
    assert all((i, i) in exp.hits for i in range(len(FFFD_CASES)))
    assert sum(1 for _, r in exp.hits if r < 5) >= 100
    rs = N.Ruleset(FFFD_RULES, strict=True)
    data, off = N.pack(msgs)
    check_every_call(N, torch, rs, FFFD_RULES, data, off, exp, seed=5)
    for i, m in enumerate(msgs):
        word, hit = rs.scan_one(m)
        assert word == int(exp.words[i]) and hit == [r for mm, r in exp.hits if mm == i], m
        mine = [(0,) + s[1:] for s in exp.full if s[0] == i]
        assert full(rs.find_matches_one(m)) == mine, m
        out, spans, dig = rs.redact_one(m)
        assert full(spans) == mine
        assert [out] == splice_python([m], FFFD_RULES, spans, dig)
    rs.close()
