"""Calls that share device scratch, issued on different streams: the scan path's calls on one rule set (its scan scratch and
single-message staging) and the SHA-256 / Merkle calls (the library's digest buffers).  They run in the order they were
issued, whatever streams they are on; every result equals the oracle's or hashlib's; and calls that share nothing do not
wait for each other.

The order is made observable by a gate: a torch stream s1 held by torch.cuda._sleep(GATE), with the first call enqueued
behind it.  GATE is 2e8 clock cycles, at least 0.1 s at the H100's top clock of 1.98 GHz and longer at a lower one, while
every call here takes a few milliseconds once a first, ungated call has sized its buffers.  A call that waits for the gated
one therefore returns with s1 finished, and a call that does not wait returns with s1 still pending.
Run on an H100: pytest -m gpu."""
import hashlib
from types import SimpleNamespace

import numpy as np
import pytest

from test_gpu_parity import oracle_policy, oracle_spans
from test_gpu_redact_device import GUARD as BYTE_GUARD, FindOut, RedactOut, ragged, splice_python, to_device, tup
from test_gpu_scan_hits_device import ALL_ONES, GUARD, HitsOut, hits_device, host_pairs
from test_gpu_views import ViewOracle, random_policy, verdicts_of
from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu
GATE = 200_000_000
N_MSGS, TILES = 2000, 33                 # the batch, and the copies of it in the batch of the chunked host path (>= 2^16 messages)
STAT_FIELDS = ("messages_scanned", "bytes_scanned", "candidate_events", "verified_pairs", "hits", "spans", "sha256_items",
               "merkle_leaves", "kernel_launches")


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


@pytest.fixture(scope="module")
def torch():
    import torch as T
    return T


def gate(torch, s1):
    with torch.cuda.stream(s1):
        torch.cuda._sleep(GATE)


def stats(N):
    s = N.stats()
    return {f: getattr(s, f) for f in STAT_FIELDS}


# ------------------------------------------------------------------------------ the batch, its expectation, the calls

def expectation(oracle, rules, msgs, data, off, pol, act, views, ids):
    words, hits = oracle_policy(oracle, rules, data, off)
    vwords, vhits, _ = ViewOracle(oracle, rules).of(msgs, ids, views)
    return SimpleNamespace(words=words, hits=hits, spans=oracle_spans(oracle, rules, data, off), verdicts=verdicts_of(hits, len(msgs), pol, act),
                           vwords=vwords, vhits=vhits)


def check_redaction(msgs, rules, E, out, out_off, spans, dig):
    """spans as the oracle's; the bytes are applyReplacements of those spans, every digest hashlib's"""
    assert tup(spans) == E.spans
    assert [bytes(out[int(out_off[i]):int(out_off[i + 1])]) for i in range(len(msgs))] == splice_python(msgs, rules, spans, dig)


class DeviceCall:
    """One device-resident call on the batch in HBM with its own output buffers: reset() fills them with guards (default
    stream), issue(stream) enqueues the call, check() asserts what it wrote against the expectation."""

    def __init__(self, kind, w, torch):
        self.kind, self.w = kind, w
        n = w.n
        if kind in ("hits", "hits_views"):
            self.out = HitsOut(torch, n, 4 * n)
        elif kind == "find":
            self.out = FindOut(torch, 4 * n)
        elif kind == "redact":
            self.out = RedactOut(torch, n, 4 * len(w.data) + 65536, 4 * n)
        else:
            self.out = None
        self.words = torch.empty(n, dtype=torch.int64, device="cuda")
        self.verdicts = torch.empty(n + 16, dtype=torch.int32, device="cuda")

    def reset(self):
        o = self.out
        self.words.fill_(-1)
        self.verdicts.fill_(GUARD)
        if isinstance(o, HitsOut):
            o.words.fill_(-1); o.hits.fill_(GUARD); o.nhits.fill_(-1)
        elif isinstance(o, FindOut):
            o.spans.fill_(BYTE_GUARD * 0x01010101); o.nspans.fill_(-1)
        elif isinstance(o, RedactOut):
            o.out.fill_(BYTE_GUARD); o.off.fill_(-1); o.spans.fill_(BYTE_GUARD * 0x01010101); o.dig.fill_(BYTE_GUARD); o.sizes.fill_(-1)

    def issue(self, stream, rs=None):
        w, o = self.w, self.out
        rs = rs or w.rs
        d, off, n = w.d, w.o, w.n
        if self.kind == "words":
            rs.scan_batch_device(d.data_ptr(), off.data_ptr(), n, self.words.data_ptr(), stream)
        elif self.kind == "hits":
            o.issue(rs, d, off, stream)
        elif self.kind == "hits_views":
            rs.scan_hits_batch_device(d.data_ptr(), off.data_ptr(), n, o.words.data_ptr(), o.hits.data_ptr(), o.cap, o.nhits.data_ptr(),
                                      stream, views=w.dv.data_ptr())
        elif self.kind == "find":
            o.issue(rs, d, off, n, stream)
        elif self.kind == "redact":
            o.issue(rs, d, off, stream)
        else:
            rs.verdict_batch_device(d.data_ptr(), off.data_ptr(), n, self.verdicts.data_ptr(), stream)

    def check(self):
        w, o, E = self.w, self.out, self.w.E
        if self.kind == "words":
            assert np.array_equal(self.words.cpu().numpy().view(np.uint64), E.words)
        elif self.kind in ("hits", "hits_views"):
            nh, pairs, guard, words = o.result()
            want_words, want_hits = (E.words, E.hits) if self.kind == "hits" else (E.vwords, E.vhits)
            assert nh == len(pairs) and pairs == want_hits and (guard == GUARD).all()
            assert np.array_equal(words, want_words)
        elif self.kind == "find":
            ns, spans, guard = o.result(w.N)
            assert ns == len(spans) and tup(spans) == E.spans and (guard == BYTE_GUARD * 0x01010101).all()
        elif self.kind == "redact":
            out, out_off, spans, dig, g_out, g_spans, g_dig = o.result(w.N)
            check_redaction(w.msgs, w.rules, E, out, out_off, spans, dig)
            assert (g_out == BYTE_GUARD).all() and (g_spans == BYTE_GUARD * 0x01010101).all() and (g_dig == BYTE_GUARD).all()
        else:
            got = self.verdicts.cpu().numpy().view(np.uint32)
            assert np.array_equal(got[:w.n], E.verdicts) and (got[w.n:] == GUARD).all()


DEVICE_CALLS = ["words", "hits", "find", "redact", "verdicts", "hits_views"]


def host_call(name, w, rs=None):
    """Run a blocking call on the batch (or one message of it) and return its check: the call returns first, so that a test
    can look at the gate before anything slow runs."""
    E, rules, msgs = w.E, w.rules, w.msgs
    rs = rs or w.rs
    i, one = w.one, w.msgs[w.one]
    want_spans = [(0, r, s, e) for (m, r, s, e) in E.spans if m == i]
    if name == "scan_batch":
        words, hits = rs.scan_batch(w.data, w.off)

        def check():
            assert np.array_equal(words, E.words) and host_pairs(hits) == E.hits
    elif name == "scan_batch_chunked":
        words, _ = rs.scan_batch(w.big_data, w.big_off, want_hits=False)

        def check():
            assert np.array_equal(words, np.tile(E.words, TILES))
    elif name == "find_matches_batch":
        spans = rs.find_matches_batch(w.data, w.off)

        def check():
            assert tup(spans) == E.spans
    elif name == "redact_batch":
        out, out_off, spans, dig = rs.redact_batch(w.data, w.off)

        def check():
            check_redaction(msgs, rules, E, out, out_off, spans, dig)
    elif name == "verdict_batch":
        verdicts = rs.verdict_batch(w.data, w.off)

        def check():
            assert np.array_equal(verdicts, E.verdicts)
    elif name == "scan_one":
        word, rl = rs.scan_one(one)

        def check():
            assert word == int(E.words[i]) and rl == [r for (m, r) in E.hits if m == i]
    elif name == "find_matches_one":
        spans = rs.find_matches_one(one)

        def check():
            assert tup(spans) == want_spans
    else:
        assert name == "redact_one"
        out, spans, dig = rs.redact_one(one)

        def check():
            assert tup(spans) == want_spans and out == splice_python([one], rules, spans, dig)[0]
    return check


HOST_CALLS = ["scan_batch", "scan_batch_chunked", "find_matches_batch", "redact_batch", "verdict_batch", "scan_one",
              "find_matches_one", "redact_one"]


@pytest.fixture(scope="module")
def world(N, torch, oracle):
    """One rule set of 120 rules with a policy and views, a ragged batch of 2000 messages (a rule's sample planted in two
    fifths of them, a tenth of the words non-ASCII) and its expectation; a second rule set of the same rules; two output sets
    for every device call; every call issued once, so that nothing below grows a buffer or captures a graph."""
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    data_t, off_t, _ = W.make_messages(N_MSGS, 200, rl, p_hit=0.4, utf8_frac=0.1, seed=2026)
    msgs = ragged(data_t, off_t, seed=2027, max_len=200)
    data, off = N.pack(msgs)
    pol, act = random_policy(rules, seed=2028)
    views = [[], list(range(len(rules))), list(range(0, len(rules), 2)), [i for i, r in enumerate(rules) if r[2] == 0]]
    ids = np.random.default_rng(2029).integers(0, len(views), N_MSGS).astype(np.uint8)
    E = expectation(oracle, rules, msgs, data, off, pol, act, views, ids)
    sets = []
    for _ in range(2):
        rs = N.Ruleset(rules, strict=True)
        rs.set_policy(pol, act)
        rs.set_views(views)
        sets.append(rs)
    d, o = to_device(torch, data, off)
    hit_msgs = {m for m, _ in E.hits} & {m for m, *_ in E.spans}
    w = SimpleNamespace(N=N, rules=rules, msgs=msgs, data=data, off=off, n=N_MSGS, E=E, rs=sets[0], rs2=sets[1], d=d, o=o,
                        dv=torch.from_numpy(np.concatenate([ids, np.zeros(16, np.uint8)])).cuda(),
                        one=min(hit_msgs), s1=torch.cuda.Stream(), s2=torch.cuda.Stream())
    w.big_data, w.big_off = N.pack(msgs * TILES)
    assert len(E.hits) > 250 and len(E.spans) > 250 and len(w.big_off) - 1 >= 1 << 16
    w.dev = {k: (DeviceCall(k, w, torch), DeviceCall(k, w, torch)) for k in DEVICE_CALLS}
    for rs in sets:
        for which, st in enumerate((w.s1, w.s2)):            # one stream at a time: nothing here overlaps
            for k in DEVICE_CALLS:
                w.dev[k][which].reset()
            torch.cuda.synchronize()
            for attempt in range(4):                          # (a queue overflow grows the scratch: issued again)
                for k in DEVICE_CALLS:
                    w.dev[k][which].issue(st.cuda_stream, rs)
                try:
                    rs.scan_join(st.cuda_stream)
                    break
                except N.GovError as e:
                    assert e.code == N.CG_ERR_CAPACITY and attempt < 3
            for k in DEVICE_CALLS:
                w.dev[k][which].check()
        for name in HOST_CALLS:
            host_call(name, w, rs)()
    torch.cuda.synchronize()
    yield w
    for rs in sets:
        rs.close()


# ------------------------------------------------------------------------------ a. ordering behind a gated call

@pytest.mark.parametrize("y", HOST_CALLS)
@pytest.mark.parametrize("x", DEVICE_CALLS)
def test_host_call_runs_after_a_device_call_on_another_stream(torch, world, x, y):
    """X on the gated stream s1, then the blocking host or single-message call Y on the same rule set (the library's
    stream): Y returns only after X has run, and both equal the oracle."""
    w = world
    X = w.dev[x][0]
    X.reset()
    torch.cuda.synchronize()
    gate(torch, w.s1)
    X.issue(w.s1.cuda_stream)
    check_y = host_call(y, w)
    x_done = w.s1.query()
    w.rs.scan_join(w.s1.cuda_stream)
    X.check()
    check_y()
    assert x_done, "%s returned before %s, issued first on another stream, had run" % (y, x)


@pytest.mark.parametrize("x", DEVICE_CALLS)
def test_device_call_runs_after_the_same_call_on_another_stream(torch, world, x):
    """X on the gated stream s1, then the same call with its own outputs on s2: once s2 is done, so is s1; both equal the
    oracle (the second output set also keeps two graphs of cg_scan_batch_device alive)."""
    w = world
    X, Y = w.dev[x]
    X.reset(); Y.reset()
    torch.cuda.synchronize()
    gate(torch, w.s1)
    X.issue(w.s1.cuda_stream)
    Y.issue(w.s2.cuda_stream)
    w.s2.synchronize()
    x_done = w.s1.query()
    w.rs.scan_join(w.s1.cuda_stream); w.rs.scan_join(w.s2.cuda_stream)
    X.check(); Y.check()
    assert x_done, "%s on s2 finished before the same call, issued first on s1, had run" % x


# ---- the digest buffers

def leaf(b):
    return hashlib.sha256(b"\x00" + b).digest()


def fold(nodes):
    """the level-wise fold of the Merkle calls: node = SHA-256(0x01 || L || R), an unpaired node moves up unchanged"""
    nodes = list(nodes)
    while len(nodes) > 1:
        nodes = [hashlib.sha256(b"\x01" + nodes[i] + nodes[i + 1]).digest() if i + 1 < len(nodes) else nodes[i] for i in range(0, len(nodes), 2)]
    return nodes[0]


@pytest.fixture(scope="module")
def merkle(N, torch, oracle):
    """fixed-size leaves and subtree roots in HBM for the device calls, ragged leaves and a tree log for the host calls, the
    expected answers from hashlib (the fold checked once against the oracle), every call issued once"""
    rng = np.random.default_rng(77)
    n, leaf_len, block_log2 = 5000, 32, 4
    leaves_fixed = W.make_leaves(n, leaf_len, seed=78).numpy()
    fixed = [leaves_fixed[i * leaf_len:(i + 1) * leaf_len].tobytes() for i in range(n)]
    hashed = [leaf(x) for x in fixed]
    B = 1 << block_log2
    m = SimpleNamespace(N=N, n=n, leaf_len=leaf_len, block_log2=block_log2, s1=torch.cuda.Stream(), s2=torch.cuda.Stream(),
                        roots_want=b"".join(fold(hashed[s:s + B]) for s in range(0, n, B)))
    assert fold(hashed) == oracle.merkle_root_fixed(leaves_fixed, leaf_len, n)
    m.d_leaves = torch.from_numpy(leaves_fixed).cuda()
    m.d_roots = torch.empty(len(m.roots_want), dtype=torch.uint8, device="cuda")
    nodes = rng.integers(0, 256, (3000, 32), dtype=np.uint8)
    m.d_nodes = torch.from_numpy(nodes.reshape(-1)).cuda()
    m.d_root = torch.empty(32, dtype=torch.uint8, device="cuda")
    m.fold_want = fold(x.tobytes() for x in nodes)
    # host calls: ragged leaves (SHA-256, root), subtree roots (fold), a tree log (audit paths, their verification)
    lens = rng.integers(0, 300, 1500)
    m.off64 = np.zeros(len(lens) + 1, dtype=np.uint64)
    m.off64[1:] = np.cumsum(lens)
    m.data = rng.integers(0, 256, int(m.off64[-1]) + 64, dtype=np.uint8)
    m.ragged = [m.data[int(m.off64[i]):int(m.off64[i + 1])].tobytes() for i in range(len(lens))]
    m.root_want = oracle.merkle_root(m.data, m.off64)
    assert m.root_want == fold(leaf(x) for x in m.ragged)
    m.nodes2 = rng.integers(0, 256, (777, 32), dtype=np.uint8)
    m.log_leaves = m.ragged[:200]
    m.log = N.MerkleLog.tree()
    m.log.append(m.log_leaves)
    m.log_root = m.log.root()
    m.idx = np.arange(0, 200, 7)
    m.paths_want = [oracle.merkle_audit_path(m.log_leaves, int(i)) for i in m.idx]
    L = N.load()
    m.block_roots = lambda st: N.check(L.cg_merkle_block_roots_device(m.d_leaves.data_ptr(), leaf_len, n, block_log2, m.d_roots.data_ptr(), st))
    m.fold_device = lambda st: N.check(L.cg_merkle_fold_device(m.d_nodes.data_ptr(), 3000, m.d_root.data_ptr(), st))
    for call in (m.block_roots, m.fold_device):
        call(m.s1.cuda_stream)
    m.s1.synchronize()
    for y in MERKLE_HOST_CALLS:
        merkle_host_call(y, m)()
    torch.cuda.synchronize()
    yield m
    m.log.close()


def merkle_host_call(name, m):
    N = m.N
    if name == "sha256_batch":
        out = N.sha256_batch(m.data, m.off64)
        return lambda: [x.tobytes() for x in out] == [hashlib.sha256(x).digest() for x in m.ragged] or pytest.fail(name)
    if name == "merkle_root":
        root = N.merkle_root(m.data, m.off64)
        return lambda: root == m.root_want or pytest.fail(name)
    if name == "merkle_fold":
        root = N.merkle_fold(m.nodes2)
        return lambda: root == fold(x.tobytes() for x in m.nodes2) or pytest.fail(name)
    if name == "log_proofs":
        paths, lens = m.log.proofs(m.idx)
        return lambda: [[paths[k, j].tobytes() for j in range(int(lens[k]))] for k in range(len(m.idx))] == m.paths_want or pytest.fail(name)
    assert name == "verify_proofs"
    paths = [list(p) for p in m.paths_want]
    paths[3] = paths[3][:-1] + [bytes(32)]                        # one proof with its last digest replaced: rejected
    ok = N.merkle_verify_proofs([m.log_leaves[int(i)] for i in m.idx], m.idx, 200, paths, m.log_root)
    return lambda: ok.tolist() == [k != 3 for k in range(len(m.idx))] or pytest.fail(name)


MERKLE_HOST_CALLS = ["sha256_batch", "merkle_root", "merkle_fold", "log_proofs", "verify_proofs"]


def merkle_device_check(m, x):
    if x == "block_roots":
        assert m.d_roots.cpu().numpy().tobytes() == m.roots_want
    else:
        assert m.d_root.cpu().numpy().tobytes() == m.fold_want


@pytest.mark.parametrize("y", MERKLE_HOST_CALLS)
@pytest.mark.parametrize("x", ["block_roots", "fold_device"])
def test_digest_call_runs_after_a_device_merkle_call_on_another_stream(torch, merkle, x, y):
    """cg_merkle_block_roots_device / cg_merkle_fold_device on the gated stream s1, then a blocking call that uses the same
    digest buffers on the library's stream: it returns only after the device call has run, and both equal hashlib."""
    m = merkle
    m.d_roots.fill_(0); m.d_root.fill_(0)
    torch.cuda.synchronize()
    gate(torch, m.s1)
    getattr(m, x)(m.s1.cuda_stream)
    check_y = merkle_host_call(y, m)
    x_done = m.s1.query()
    m.s1.synchronize()
    merkle_device_check(m, x)
    check_y()
    assert x_done, "%s returned before %s, issued first on another stream, had run" % (y, x)


# ------------------------------------------------------------------------------ b. no false serialisation

def test_calls_on_another_rule_set_do_not_wait(torch, world):
    """a gated batch on R1; host, single-message and device calls on R2 (same rules) complete while it is still held"""
    w = world
    X, Y = w.dev["hits"]
    X.reset(); Y.reset()
    torch.cuda.synchronize()
    gate(torch, w.s1)
    X.issue(w.s1.cuda_stream)
    pending = []
    for name in ("scan_batch", "redact_batch", "find_matches_one"):
        check = host_call(name, w, w.rs2)
        pending.append((name, w.s1.query()))
        check()
    Y.issue(w.s2.cuda_stream, w.rs2)
    w.s2.synchronize()
    pending.append(("device call on s2", w.s1.query()))
    w.rs.scan_join(w.s1.cuda_stream); w.rs2.scan_join(w.s2.cuda_stream)
    X.check(); Y.check()
    assert not [name for name, done in pending if done], "waited for a call on another rule set"


def test_digest_calls_do_not_wait_for_a_scan(torch, world, merkle):
    w, m = world, merkle
    X = w.dev["redact"][0]
    X.reset()
    torch.cuda.synchronize()
    gate(torch, w.s1)
    X.issue(w.s1.cuda_stream)
    pending = []
    for name in MERKLE_HOST_CALLS:
        check = merkle_host_call(name, m)
        pending.append((name, w.s1.query()))
        check()
    w.rs.scan_join(w.s1.cuda_stream)
    X.check()
    assert not [name for name, done in pending if done], "waited for a scan"


def test_scans_do_not_wait_for_a_merkle_call(torch, world, merkle):
    w, m = world, merkle
    Y = w.dev["find"][1]
    Y.reset()
    m.d_roots.fill_(0)
    torch.cuda.synchronize()
    gate(torch, m.s1)
    m.block_roots(m.s1.cuda_stream)
    pending = []
    for name in ("scan_batch", "verdict_batch", "scan_one", "redact_one"):
        check = host_call(name, w)
        pending.append((name, m.s1.query()))
        check()
    Y.issue(w.s2.cuda_stream)
    w.s2.synchronize()
    pending.append(("device call on s2", m.s1.query()))
    m.s1.synchronize(); w.rs.scan_join(w.s2.cuda_stream)
    merkle_device_check(m, "block_roots")
    Y.check()
    assert not [name for name, done in pending if done], "waited for a Merkle call"


# ------------------------------------------------------------------------------ c. ungated interleavings

def test_interleaved_calls_equal_the_same_calls_one_after_another(N, torch, world):
    """A batch of 128 copies of the batch (256 000 messages) on s1, then at once host, single-message and s2 device calls on
    the same rule set, then both streams joined: every result and the cg_stats delta equal those of the same calls issued
    one after another with a join between them."""
    w = world
    reps = 128
    big_msgs = w.msgs * reps
    bd, bo = to_device(torch, *N.pack(big_msgs))
    torch.cuda.synchronize()
    big = HitsOut(torch, len(big_msgs), len(w.E.hits) * reps + 64)
    want_hits = [(mm + k * w.n, r) for k in range(reps) for (mm, r) in w.E.hits]
    s1, s2 = w.s1.cuda_stream, w.s2.cuda_stream
    calls = ["scan_batch", "find_matches_one", "redact_batch", "scan_one", "verdict_batch", "redact_one", "find_matches_batch"]
    devs = [w.dev[k][1] for k in ("find", "redact", "verdicts", "hits_views")]

    def run(interleaved):
        for dv in devs:
            dv.reset()
        big.hits.fill_(GUARD)
        torch.cuda.synchronize()
        s0 = stats(N)
        big.issue(w.rs, bd, bo, s1)
        if not interleaved:
            w.rs.scan_join(s1)
        checks = []
        for k, name in enumerate(calls):
            checks.append(host_call(name, w))
            if k < len(devs):
                devs[k].issue(s2)
                if not interleaved:
                    w.rs.scan_join(s2)
        w.rs.scan_join(s1); w.rs.scan_join(s2)
        delta = {f: v - s0[f] for f, v in stats(N).items()}
        for check in checks:
            check()
        for dv in devs:
            dv.check()
        nh, pairs, guard, words = big.result()
        assert nh == len(pairs) and pairs == want_hits and (guard == GUARD).all()
        assert np.array_equal(words, np.tile(w.E.words, reps))
        return delta

    hits_device(N, torch, w.rs, *N.pack(big_msgs), cap=big.cap, stream=s1)     # (sizes the scratch for the large batch)
    one_by_one = run(False)
    assert run(True) == one_by_one
    assert one_by_one["messages_scanned"] == (reps + 4 + len(devs)) * w.n + 3


def test_overflow_in_an_interleaving_is_reported_once(N, torch, oracle):
    """A fresh rule set sized by a small batch, then 30 000 messages that all hit on s1 (a queue overflows), and at once
    host, single-message and s2 device calls on the same rule set: the large batch's words are all ones, every other call
    equals the oracle, and the joins report CG_ERR_CAPACITY exactly once."""
    rl = W.make_rules(64)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    d0_t, o0_t, _ = W.make_messages(64, 256, rl, p_hit=0.0, seed=3)
    d1_t, o1_t, _ = W.make_messages(30000, 256, rl, p_hit=1.0, seed=4)
    d2_t, o2_t, _ = W.make_messages(2000, 200, rl, p_hit=0.2, utf8_frac=0.1, seed=5)
    data2, off2 = d2_t.numpy(), o2_t.numpy().astype(np.uint32)
    ewords, ehits = oracle_policy(oracle, rules, data2, off2)
    hits_device(N, torch, rs, d0_t.numpy(), o0_t.numpy().astype(np.uint32), stream=s1.cuda_stream)     # (sizes the queues)
    d1, o1 = to_device(torch, d1_t.numpy(), o1_t.numpy())
    d2, o2 = to_device(torch, data2, off2)
    words1 = torch.zeros(30000, dtype=torch.int64, device="cuda")
    ho = HitsOut(torch, 2000, 4096)
    one = next(m for m, _ in ehits)
    msg = bytes(data2[int(off2[one]):int(off2[one + 1])])
    torch.cuda.synchronize()
    rs.scan_batch_device(d1.data_ptr(), o1.data_ptr(), 30000, words1.data_ptr(), s1.cuda_stream)
    ho.issue(rs, d2, o2, s2.cuda_stream)
    hwords, hhits = rs.scan_batch(data2, off2)
    word, rlist = rs.scan_one(msg)
    errors = []
    for st in (s1, s2, s1):
        try:
            rs.scan_join(st.cuda_stream)
        except N.GovError as e:
            errors.append(e.code)
    assert errors == [N.CG_ERR_CAPACITY]
    assert (words1.cpu().numpy().view(np.uint64) == np.uint64(0xffffffffffffffff)).all()
    nh, pairs, guard, dwords = ho.result()
    assert nh != ALL_ONES and pairs == ehits and (guard == GUARD).all() and np.array_equal(dwords, ewords)
    assert host_pairs(hhits) == ehits and np.array_equal(hwords, ewords)
    assert word == int(ewords[one]) and rlist == [r for m, r in ehits if m == one]
    rs.close()
