"""GPU tier, the span resolver (span_resolve.cu), the redaction digests and splice and the JSONL split (sha256_kernels.cu)
past their launch boundaries.  Every launch geometry there depends on the SM count S only: each case derives its batch
from geometry(S) and asserts that the batch crosses the boundary it is named for.  Spans are compared with the C oracle
(findMatches + resolveOverlaps), redacted bytes and digests with splice_python and hashlib fed the oracle's spans, Merkle
roots with the oracle.  Every batch goes through the host calls (cg_find_matches_batch, cg_redact_batch) and the
device-resident calls (cg_find_matches_batch_device, cg_redact_batch_device); guard words follow every device output.
The workload builders are checked without a device in test_span_boundaries_cpu.py.  Run on an H100: pytest -m gpu."""
import hashlib
from types import SimpleNamespace

import numpy as np
import pytest

from helpers import oracle_regexes
from test_gpu_parity import CATS, oracle_spans
from test_gpu_redact_device import GUARD, FindOut, RedactOut, splice_python, to_device
from vainplex_openclaw_b200._native import SPAN_DTYPE, pack

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


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def geometry(S):
    """The launch constants of span_resolve.cu and sha256_kernels.cu for S SMs."""
    return SimpleNamespace(
        S=S,
        scan_block=4096,                    # xscan: one block per 4096 elements ...
        scan_blocks_max=min(1024, 2 * S),   # ... at most kScanPartials, two per SM; then each block's range grows
        warp_sort=32,                       # segments of up to 32 raw spans: one warp each, in registers
        block_sort=2048,                    # longer ones: one block each, runs of 2048 sorted, then merged in HBM
        sort_warps=32 * S,                  # span_sort_keep_kernel: 2S blocks of 512 threads
        sort_blocks=2 * S,
        stride=1024 * S,                    # span_count / span_scatter / span_emit: 4S x 256; redact_digest_kernel: 8S x 128
        splice_warps=64 * S)                # redact_splice_kernel: at most 8S blocks of 8 warps, one message per warp


def scan_split(g, count):
    """(blocks, elements per block) of launch_exclusive_scan over count elements"""
    blocks = min(-(-count // g.scan_block), g.scan_blocks_max)
    return blocks, -(-count // blocks)


def merge_passes(g, c):
    """pairwise merge passes sort_keep_segment runs over a segment of c raw spans (odd: the result is in sort_tmp)"""
    return (-(-c // g.block_sort) - 1).bit_length() if c > g.warp_sort else 0


# ------------------------------------------------------------------------------------------------ expected results

def oracle_array(oracle, rules, data, off):
    """oracle_spans as an int64 array [k, 4] of (msg, rule, start16, end16)"""
    regs = oracle_regexes(oracle, rules)
    pats = [(regs[i], CATS[rules[i][2]]) for i in range(len(rules))]
    return oracle.find_matches_batch(pats, data, off.astype(np.uint64)).astype(np.int64).reshape(-1, 4)


class Expected:
    """What a batch of ASCII messages must give: the oracle's resolved spans (start_byte = start16 in ASCII), their SHA-256
    (hashlib) and the redacted messages (splice_python).  Messages are independent, so the answer for the n messages from
    m0 is a window of these arrays (window())."""

    def __init__(self, oracle, rules, msgs):
        assert all(m.isascii() for m in msgs)
        self.msgs = msgs
        self.data, self.off = pack(msgs)
        arr = oracle_array(oracle, rules, self.data, self.off)
        sp = np.zeros(len(arr), SPAN_DTYPE)
        for col, f in enumerate(("msg", "rule", "start16", "end16")):
            sp[f] = arr[:, col]
        sp["start_byte"], sp["end_byte"] = sp["start16"], sp["end16"]
        self.spans = sp
        m, a, b = sp["msg"].tolist(), sp["start_byte"].tolist(), sp["end_byte"].tolist()
        self.dig = np.frombuffer(b"".join(hashlib.sha256(msgs[i][s:e]).digest() for i, s, e in zip(m, a, b)), np.uint8).reshape(-1, 32)
        out = splice_python(msgs, rules, sp, self.dig)
        self.out = np.frombuffer(b"".join(out), np.uint8)
        self.out_off = np.zeros(len(msgs) + 1, np.uint64)
        self.out_off[1:] = np.cumsum([len(x) for x in out])
        self.first = np.searchsorted(sp["msg"], np.arange(len(msgs) + 1))     # first span of every message
        self.counts = np.diff(self.first)                                     # resolved spans per message

    def window(self, m0, n):
        """(spans, digests, redacted bytes, output offsets) of the batch of messages m0 .. m0 + n - 1"""
        s0, s1 = self.first[m0], self.first[m0 + n]
        spans = self.spans[s0:s1].copy()
        spans["msg"] -= m0
        o = self.out_off[m0:m0 + n + 1]
        return spans, self.dig[s0:s1], self.out[int(o[0]):int(o[-1])], o - o[0]


def assert_same(what, got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.nonzero(got != want)[0] if got.ndim == 1 else np.nonzero((got != want).any(axis=tuple(range(1, got.ndim))))[0]
    assert not len(bad), (what, len(bad), int(bad[0]), got[bad[0]], want[bad[0]])


def assert_spans(what, got, want):
    assert len(got) == len(want), (what, len(got), len(want))
    for f in SPAN_DTYPE.names:
        assert_same((what, f), got[f], want[f])


def find_dev(N, torch, rs, d, o_ptr, n, cap):
    """cg_find_matches_batch_device on a batch already in HBM, offsets at o_ptr, capacity = what the batch needs (the
    guard words lie right behind the spans); issued again while an internal queue overflows (count ~0)"""
    fo = FindOut(torch, cap)
    for attempt in range(4):
        rs.find_matches_batch_device(d.data_ptr(), o_ptr, n, fo.spans.data_ptr(), cap, fo.nspans.data_ptr())
        try:
            rs.scan_join()
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
            assert (int(fo.nspans[0].item()) & 0xffffffff) == 0xffffffff
    ns, spans, guard = fo.result(N)
    assert ns == cap and (guard == GUARD * 0x01010101).all()
    return spans


def redact_dev(N, torch, rs, d, o_ptr, n, out_cap, spans_cap):
    """cg_redact_batch_device the same way, with guard words behind the output offsets too"""
    ro = RedactOut(torch, n, out_cap, spans_cap)
    ro.off = torch.full((n + 1 + 64,), -1, dtype=torch.int32, device="cuda")
    for attempt in range(4):
        rs.redact_batch_device(d.data_ptr(), o_ptr, n, ro.out.data_ptr(), out_cap, ro.off.data_ptr(), ro.spans.data_ptr(), spans_cap,
                               ro.dig.data_ptr(), ro.sizes.data_ptr())
        try:
            rs.scan_join()
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3 and ro.sizes_() == (2 ** 64 - 1, 2 ** 64 - 1), (e, ro.sizes_())
    assert ro.sizes_() == (out_cap, spans_cap)
    out, off, spans, dig, g_out, g_spans, g_dig = ro.result(N)
    assert (g_out == GUARD).all() and (g_spans == GUARD * 0x01010101).all() and (g_dig == GUARD).all()
    assert (off[n + 1:] == 0xffffffff).all()
    return out, off[:n + 1], spans, dig


def check_batch(N, torch, rs, ex, n=None, dev=None, m0=0):
    """The n messages of ex from m0 through both device calls and (m0 = 0) both host calls: spans with their byte
    offsets, resolved count, output offsets, redacted bytes and digests equal ex's."""
    n = len(ex.msgs) - m0 if n is None else n
    spans, dig, out, out_off = ex.window(m0, n)
    if m0 == 0:
        off = ex.off[:n + 1]
        assert_spans("host find", rs.find_matches_batch(ex.data, off), spans)
        h_out, h_off, h_spans, h_dig = rs.redact_batch(ex.data, off)
        assert_spans("host redact", h_spans, spans)
        assert_same("host digests", h_dig, dig)
        assert_same("host offsets", h_off, out_off)
        assert_same("host bytes", h_out, out)
    d, o = dev if dev is not None else to_device(torch, ex.data, ex.off)
    o_ptr = o.data_ptr() + 4 * m0
    assert_spans("device find", find_dev(N, torch, rs, d, o_ptr, n, len(spans)), spans)
    r_out, r_off, r_spans, r_dig = redact_dev(N, torch, rs, d, o_ptr, n, len(out), len(spans))
    assert_spans("device redact", r_spans, spans)
    assert_same("device digests", r_dig, dig)
    assert_same("device offsets", r_off, out_off)
    assert_same("device bytes", r_out, out)
    return len(spans)


# ------------------------------------------------------------------------------------------------ 1. scan blocks, warp and splice loops

SCAN_RULES = [(r"\d+", 0, 2), (r"\d\d", 0, 1), (r"[a-z]+\d", 0, 0), ("zq", 0, 3)]

# batch sizes: n(g), and what a batch of n messages crosses (the scans run over the n + 1 per-message counts)
SCAN_CASES = {
    "4095": (lambda g: g.scan_block - 1, lambda g, n: scan_split(g, n + 1) == (1, g.scan_block)),
    "4096": (lambda g: g.scan_block, lambda g, n: scan_split(g, n + 1)[0] == 2),
    "8192": (lambda g: 2 * g.scan_block, lambda g, n: scan_split(g, n + 1)[0] == 3),
    "32S": (lambda g: g.sort_warps, lambda g, n: n == g.sort_warps),
    "32S+1": (lambda g: g.sort_warps + 1, lambda g, n: n == g.sort_warps + 1),
    "64S": (lambda g: g.splice_warps, lambda g, n: n == g.splice_warps),
    "64S+1": (lambda g: g.splice_warps + 1, lambda g, n: n == g.splice_warps + 1),
    # every block of the capped grid gets exactly 4096 counts / one more (4097) / a range that is no multiple of 512 and a
    # shorter last block
    "8192S-1": (lambda g: g.scan_block * g.scan_blocks_max - 1,
                lambda g, n: scan_split(g, n + 1) == (g.scan_blocks_max, g.scan_block)),
    "8192S": (lambda g: g.scan_block * g.scan_blocks_max,
              lambda g, n: scan_split(g, n + 1) == (g.scan_blocks_max, g.scan_block + 1)),
    "8192S+5000": (lambda g: g.scan_block * g.scan_blocks_max + 5000,
                   lambda g, n: (lambda b, p: b == g.scan_blocks_max and p % 512 != 0 and n + 1 - (b - 1) * p < p)(*scan_split(g, n + 1))),
}
SUB_M0 = [1, 2, 4095, 4096, 4097]        # odd, even, either side of the first 4096-message edge of the whole batch
QUIET = b"ABCDEFGHIJKLMNOPRSTUVWXYZ -.:"  # matched by no rule of SCAN_RULES
PIECES = [b"7", b"42", b"123", b"98765", b"ab3", b"zq", b"zq7", b"k9", b"xy12", b"zqzq"]


def sub_n(g):
    return g.splice_warps + 1


def scan_edges(g, n):
    """the first count of every scan block but the first, over the n + 1 counts of a batch of n messages"""
    blocks, per = scan_split(g, n + 1)
    return [k * per for k in range(1, blocks)]


def scan_workload(g, seed):
    """Messages of 0-16 bytes (1 % of 24-60 byte ones whose redaction is shorter), spans in the first message, the last
    message of every SCAN_CASES batch, the messages on both sides of each of its scan-block edges and the first and last
    message of every sub-range.  Drawn from pools of templates, so that a million messages cost little to build."""
    rng = np.random.default_rng(seed)
    qb = np.frombuffer(QUIET, np.uint8)

    def quiet(k):
        return bytes(rng.choice(qb, k))

    quiet_pool = [b""] + [quiet(int(k)) for k in rng.integers(0, 17, 255)]
    span_pool = []
    while len(span_pool) < 2000:
        m = b"".join(quiet(int(rng.integers(0, 3))) + PIECES[int(rng.integers(0, len(PIECES)))] for _ in range(int(rng.integers(1, 4))))
        if len(m) <= 16:
            span_pool.append(m)
    long_pool = [quiet(1) + b"9" * int(k) for k in rng.integers(24, 61, 50)] + [b"q" * int(k) + b"5" for k in rng.integers(30, 60, 50)]
    forced = {0}
    for n_of, _ in SCAN_CASES.values():
        n = n_of(g)
        forced.add(n - 1)
        for e in scan_edges(g, n):
            forced |= {e - 1, e}
    for m0 in SUB_M0:
        forced |= {m0, m0 + sub_n(g) - 1}
    n_max = max(max(n_of(g) for n_of, _ in SCAN_CASES.values()), max(SUB_M0) + sub_n(g))
    pool = quiet_pool + span_pool + long_pool
    kind = rng.random(n_max)
    pick = np.where(kind < 0.45, rng.integers(0, len(quiet_pool), n_max),
                    np.where(kind < 0.99, len(quiet_pool) + rng.integers(0, len(span_pool), n_max),
                             len(quiet_pool) + len(span_pool) + rng.integers(0, len(long_pool), n_max)))
    f = np.array(sorted(x for x in forced if x < n_max))
    pick[f] = len(quiet_pool) + rng.integers(0, len(span_pool), len(f))
    return [pool[k] for k in pick.tolist()], f


@pytest.fixture(scope="module")
def scan_group(oracle, torch):
    """the largest batch of the group, its expected results (sliced for every smaller batch) and its copy in HBM"""
    g = geometry(sm_count())
    msgs, forced = scan_workload(g, seed=8192)
    ex = Expected(oracle, SCAN_RULES, msgs)
    assert (ex.counts[forced] > 0).all()
    delta = np.diff(ex.out_off.astype(np.int64)) - np.diff(ex.off.astype(np.int64))
    assert (delta < 0).sum() > 1000 and (delta > 0).sum() > 1000               # placeholders shorter and longer than the match
    print("scan group: S = %d, %d messages, %d resolved spans, %d redacted bytes" % (g.S, len(msgs), len(ex.spans), len(ex.out)))
    return SimpleNamespace(g=g, ex=ex, dev=to_device(torch, ex.data, ex.off))


@pytest.mark.parametrize("case", list(SCAN_CASES))
def test_scan_blocks_sort_warps_and_splice_warps(N, torch, scan_group, case):
    """The first n messages of the group: n around one scan block, around the grid cap of the scans (8192 S with S = 132
    on an H100 SXM), and around the warp loops of the sort (32 S) and of the splice (64 S)."""
    g, ex = scan_group.g, scan_group.ex
    n_of, crosses = SCAN_CASES[case]
    n = n_of(g)
    assert crosses(g, n), (case, n, scan_split(g, n + 1))
    c = ex.counts
    assert c[0] and c[n - 1] and all(c[e - 1] and c[e] for e in scan_edges(g, n) if e < n)
    rs = N.Ruleset(SCAN_RULES, strict=True)
    k = check_batch(N, torch, rs, ex, n, scan_group.dev)
    print("n = %d: scan %s, %d resolved spans" % (n, scan_split(g, n + 1), k))
    rs.close()


@pytest.mark.parametrize("m0", SUB_M0)
def test_device_calls_on_a_sub_range(N, torch, scan_group, m0):
    """Both device calls with d_offsets pointing at message m0 (offsets[0] != 0) of the resident batch, for a sub-batch
    that crosses the scan's first block edge and both warp loops: message indices from m0, output offsets from 0,
    digests of the right bytes."""
    g, ex = scan_group.g, scan_group.ex
    n = sub_n(g)
    assert scan_split(g, n + 1)[0] >= 2 and n > g.sort_warps and n > g.splice_warps
    assert ex.off[m0] != 0 and ex.counts[m0] and ex.counts[m0 + n - 1]
    rs = N.Ruleset(SCAN_RULES, strict=True)
    check_batch(N, torch, rs, ex, n, scan_group.dev, m0=m0)
    rs.close()


# ------------------------------------------------------------------------------------------------ 2. segment sizes

SEG_SIZES = [0, 1, 31, 32, 33, 63, 64, 65, 2047, 2048, 2049, 4096, 4097, 8192, 8193]
# one rule: c digits; ties: c / 2 digits matched alike by a pii and a financial rule (plus an "x" when c is odd), so
# (category, rule) decides the order inside every run and merge
SEG_RULES = {"one-rule": [(r"\d", 0, 2)], "ties": [(r"\d", 0, 2), (r"[0-9]", 0, 1), ("x", 0, 3)]}


def segment_message(kind, c, rng):
    if kind == "one-rule":
        return bytes(rng.integers(48, 58, c, dtype=np.uint8))
    return bytes(rng.integers(48, 58, c // 2, dtype=np.uint8)) + b"x" * (c % 2)


def segment_batch(kind):
    """a message of exactly c raw spans for every c in SEG_SIZES, a message without spans after each -> (msgs, raw spans)"""
    rng = np.random.default_rng(len(kind))
    msgs, raw = [], []
    for i, c in enumerate(SEG_SIZES):
        msgs += [segment_message(kind, c, rng), (b"", b"ab-")[i % 2]]
        raw += [c, 0]
    return msgs, np.array(raw)


def long_segment_batch(g):
    """6S + 10 messages of 33-100 raw spans (ties rules): every sort block takes three or four long segments"""
    rng = np.random.default_rng(g.S)
    raw = rng.integers(g.warp_sort + 1, 101, 6 * g.S + 10)
    return [segment_message("ties", int(c), rng) for c in raw], raw


def raw_span_counts(oracle, rules, msgs):
    """raw spans per message: every match of every rule (one rule's matches never overlap, so the oracle's resolved
    spans of a rule on its own are all of them)"""
    data, off = pack(msgs)
    cnt = np.zeros(len(msgs), np.int64)
    for r in rules:
        cnt += np.bincount([s[0] for s in oracle_spans(oracle, [r], data, off)], minlength=len(msgs))
    return cnt


@pytest.mark.parametrize("kind", list(SEG_RULES))
def test_segment_sizes(N, torch, oracle, kind):
    """Segments of exactly 0, 1, 31/32/33 (warp / block sort), 63/64/65 (bitonic padding), 2047/2048/2049 (one run / two),
    4096/4097 and 8192/8193 raw spans: one, two and three merge passes, so the result is read back from sorted and from
    sort_tmp."""
    g = geometry(sm_count())
    msgs, raw = segment_batch(kind)
    assert np.array_equal(raw_span_counts(oracle, SEG_RULES[kind], msgs), raw)
    assert {g.warp_sort, g.warp_sort + 1, g.block_sort, g.block_sort + 1} <= set(SEG_SIZES)
    assert {merge_passes(g, c) for c in SEG_SIZES} == {0, 1, 2, 3}
    ex = Expected(oracle, SEG_RULES[kind], msgs)
    assert np.array_equal(ex.counts, raw if kind == "one-rule" else raw // 2 + raw % 2)
    rs = N.Ruleset(SEG_RULES[kind], strict=True)
    check_batch(N, torch, rs, ex)
    rs.close()


def test_several_long_segments_per_sort_block(N, torch, oracle):
    g = geometry(sm_count())
    msgs, raw = long_segment_batch(g)
    assert np.array_equal(raw_span_counts(oracle, SEG_RULES["ties"], msgs), raw)
    per_block = [int((raw[b::g.sort_blocks] > g.warp_sort).sum()) for b in range(g.sort_blocks)]
    assert len(msgs) > 2 * g.S + 10 and min(per_block) >= 3
    ex = Expected(oracle, SEG_RULES["ties"], msgs)
    rs = N.Ruleset(SEG_RULES["ties"], strict=True)
    check_batch(N, torch, rs, ex)
    rs.close()


# ------------------------------------------------------------------------------------------------ 3. totals past the grid stride

STRIDE_RULES = [(r"\d", 0, 2)]


def stride_batch(g):
    """more than 2 x 1024 S resolved spans in messages of 100-140 digits, with messages without spans: a run at the
    start, one in the middle, one at the end, and runs of 1, 2 and 3 between dense messages"""
    rng = np.random.default_rng(1024)
    quiet = [b"", b"no digits here", b""]

    def dense(k):
        return [bytes(rng.integers(48, 58, int(rng.integers(100, 141)), dtype=np.uint8)) for _ in range(k)]

    half = (2 * g.stride) // 240 + 10
    msgs = quiet * 20 + dense(half) + quiet * 100
    for r in (1, 2, 3) * 10:
        msgs += dense(1) + quiet[:r]
    return msgs + dense(half) + quiet * 15


def test_span_totals_past_the_grid_stride(N, torch, oracle):
    """span_count / span_scatter / span_emit and the digest kernel loop over more than twice their grid; span_emit's
    binary search over kept_begin meets runs of messages without kept spans at the start, middle and end"""
    g = geometry(sm_count())
    msgs = stride_batch(g)
    ex = Expected(oracle, STRIDE_RULES, msgs)
    c = ex.counts
    assert len(ex.spans) > 2 * g.stride
    assert not c[:60].any() and not c[-45:].any() and c[60]
    runs = np.diff(np.nonzero(c)[0]) - 1                                  # messages without spans between two with spans
    assert {1, 2, 3} <= set(runs.tolist()) and runs.max() >= 300
    rs = N.Ruleset(STRIDE_RULES, strict=True)
    check_batch(N, torch, rs, ex)
    rs.close()


# ------------------------------------------------------------------------------------------------ 5. digest lengths

DIGEST_RULES = [("Q[a-z]*Q", 0, 0)]


def digest_batch():
    """one match per message, of every length 2 .. 200, at every start address mod 16"""
    rng = np.random.default_rng(200)
    msgs, pos = [], 0
    for length in range(2, 201):
        for a in range(16):
            m = b"." * ((a - pos) % 16) + b"Q" + bytes(rng.integers(97, 123, length - 2, dtype=np.uint8)) + b"Q" + b"." * int(rng.integers(0, 4))
            msgs.append(m)
            pos += len(m)
    return msgs


def test_redaction_digests_of_every_length_and_alignment(N, torch, oracle):
    """redact_digest_kernel's byte-granular SHA-256 (sha_bytes) across its padding edges (55/56, 63/64, 119/120, 127/128
    bytes): digests equal hashlib on both calls"""
    msgs = digest_batch()
    ex = Expected(oracle, DIGEST_RULES, msgs)
    sp = ex.spans
    length = (sp["end_byte"] - sp["start_byte"]).astype(np.int64)
    addr = ex.off[sp["msg"]].astype(np.int64) + sp["start_byte"]
    assert set(zip(length.tolist(), (addr % 16).tolist())) == {(k, a) for k in range(2, 201) for a in range(16)}
    rs = N.Ruleset(DIGEST_RULES, strict=True)
    check_batch(N, torch, rs, ex)
    rs.close()


GENERIC_LEAVES = [1, 2, 3, 53, 54, 55, 62, 63, 118, 119]     # merkle_leaves_fixed_generic_kernel (sha_bytes)
WORD_LEAVES = [52, 56, 60, 64, 116, 120]                     # merkle_leaves_fixed_kernel


def test_fixed_leaf_roots_at_the_padding_edges(N, oracle):
    """Fixed-size leaves hashed with the 0x00 prefix: the generic kernel at 55/56, 63/64 and 119/120 hashed bytes, the
    word kernel on either side of its one-block / two-block / three-block edges; roots equal the oracle's and a single
    leaf's root equals hashlib"""
    assert all(x % 4 for x in GENERIC_LEAVES) and {55, 56, 63, 64, 119, 120} <= {x + 1 for x in GENERIC_LEAVES}
    assert all(x % 4 == 0 for x in WORD_LEAVES) and {(1 + x + 9 + 63) // 64 for x in WORD_LEAVES} == {1, 2, 3}
    for leaf in GENERIC_LEAVES + WORD_LEAVES:
        for n in (1, 2, 3, 777):
            data = np.random.default_rng(leaf * 1000 + n).integers(0, 256, n * leaf + 64, dtype=np.uint8)
            root = N.merkle_root_fixed(data, leaf, n)
            assert root == oracle.merkle_root_fixed(data, leaf, n), (leaf, n)
            if n == 1:
                assert root == hashlib.sha256(b"\0" + data[:leaf].tobytes()).digest(), leaf


# ------------------------------------------------------------------------------------------------ 6. JSONL split past 1024 pieces

PIECE = 4096                                       # newline_count_kernel: one piece per block
E1, E2 = 1024 * PIECE, 2048 * PIECE                # newline_scan_kernel: 1024 pieces per iteration
JSONL_BLOBS = {
    "4MiB+1-terminated": dict(size=E1 + 1, terminated=True, iterations=2, empty_run=(E1 - 6, E1 + 1)),
    "4MiB-unterminated": dict(size=E1, terminated=False, iterations=1, newlines=(E1 - PIECE - 1, E1 - PIECE)),
    "9MB-unterminated": dict(size=9_000_000, terminated=False, iterations=3, newlines=(E1 - 1, E1, E2 - 1, E2)),
    "9MB-terminated": dict(size=9_000_001, terminated=True, iterations=3, long_line=(E1 - 5000, E1 + 3 * PIECE + 3000),
                           empty_run=(E2 - 3, E2 + 4)),
}


def jsonl_blob(name):
    """printable ASCII lines of 0-900 bytes with what JSONL_BLOBS[name] asks for: newlines at given bytes, a run of empty
    lines, a line longer than three pieces, a terminated or unterminated last line"""
    spec = JSONL_BLOBS[name]
    size = spec["size"]
    rng = np.random.default_rng(size)
    buf = rng.integers(0x20, 0x7f, size, dtype=np.uint8)
    nl = np.cumsum(rng.integers(1, 900, size // 400 + 10))
    buf[nl[nl < size]] = 10
    if "long_line" in spec:
        a, b = spec["long_line"]
        buf[a:b] = ord("x")
        buf[a - 1] = buf[b] = 10
    if "empty_run" in spec:
        a, b = spec["empty_run"]
        buf[a:b] = 10
    for p in spec.get("newlines", ()):
        buf[p] = 10
    buf[-1] = 10 if spec["terminated"] else ord("}")
    return buf.tobytes()


def jsonl_lines(blob):
    lines = blob.split(b"\n")
    return lines[:-1] if blob.endswith(b"\n") else lines


def check_jsonl_claims(name, blob):
    """the blob has the size, scan iterations, newlines, empty-line run and long line JSONL_BLOBS claims"""
    spec = JSONL_BLOBS[name]
    assert len(blob) == spec["size"] and blob.endswith(b"\n") == spec["terminated"]
    pieces = -(-len(blob) // PIECE)
    assert -(-pieces // 1024) == spec["iterations"]
    assert all(blob[p] == 10 for p in spec.get("newlines", ()))
    if "empty_run" in spec:
        a, b = spec["empty_run"]
        assert blob[a:b] == b"\n" * (b - a) and b - a >= 3
        assert any(a < e < b for e in (E1, E2))                    # newlines on both sides of a 1024-piece edge
    if "long_line" in spec:
        a, b = spec["long_line"]
        assert blob[a - 1] == 10 and blob[b] == 10 and b"\n" not in blob[a:b]
        assert b - a > 3 * PIECE and a < E1 < b
    lines = jsonl_lines(blob)
    assert len(lines) == blob.count(b"\n") + (0 if spec["terminated"] else 1)
    return lines


@pytest.mark.parametrize("name", list(JSONL_BLOBS))
def test_jsonl_split_past_1024_pieces(N, oracle, name):
    """newline_scan_kernel carries its running count from one 1024-piece iteration to the next: the line count and the
    root equal the oracle's, and so does the same blob appended in two flushes cut at a newline past piece 1024"""
    blob = jsonl_blob(name)
    lines = check_jsonl_claims(name, blob)
    data, off = oracle.pack(lines)
    want = oracle.merkle_root(data, off)
    log = N.MerkleLog(keep_leaf_digests=False)
    assert log.append_jsonl(blob) == len(lines) and log.size() == len(lines)
    assert log.root() == want
    log.close()
    cut = blob.index(b"\n", E1 + 100 if len(blob) > E1 + PIECE else len(blob) // 2) + 1
    assert cut < len(blob)
    log = N.MerkleLog(keep_leaf_digests=False)
    assert log.append_jsonl(blob[:cut]) + log.append_jsonl(blob[cut:]) == len(lines)
    assert log.root() == want
    log.close()
