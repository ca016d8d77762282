"""GPU tier: the real kernels through the C ABI (ctypes) against the oracle and the golden vectors.
Bit-exact everywhere (integer / byte / index work).  Run on an H100: pytest -m gpu."""
import hashlib
import json
import os

import numpy as np
import pytest

from helpers import oracle_regexes, PACK_RULES, PACK_TEXTS, random_regex
from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
VECTORS = json.load(open(os.path.join(HERE, "golden", "registry_vectors.json")))["vectors"]
CATS = ["credential", "financial", "pii", "custom"]


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


def oracle_policy(O, rules, data, off):
    regs = oracle_regexes(O, rules)
    assert all(r is not None for r in regs)
    bits, words = O.scan_policy(regs, data, off.astype(np.uint64))
    hits = []
    for m in range(bits.shape[0]):
        row = np.unpackbits(bits[m], bitorder="little")[:len(rules)]
        hits += [(m, int(r)) for r in np.nonzero(row)[0]]
    return words, hits


def oracle_spans(O, rules, data, off):
    regs = oracle_regexes(O, rules)
    pats = [(regs[i], CATS[rules[i][2]]) for i in range(len(rules))]
    return [tuple(x) for x in O.find_matches_batch(pats, data, off.astype(np.uint64)).tolist()]


def test_native_library_is_the_cuda_one(N):
    assert N.load().cg_device_count() >= 1
    assert os.path.basename(N.lib_path()) == "libopenclaw_gov.so"


def test_reference_vectors_through_the_kernels(N, oracle):
    """every golden input x the reference's registry configurations, spans == oracle, checks hold"""
    from test_oracle_golden import run_checks
    configs = {}
    for v in VECTORS:
        key = json.dumps([v["categories"], v["custom"]])
        configs.setdefault(key, []).append(v)
    for key, vs in configs.items():
        cats, custom = json.loads(key)
        reg = oracle.builtin_registry(cats, custom)           # (Regex, category, id) storage order
        rules = [(r[0].source, 1 if "i" in r[0].flags else 0, CATS.index(r[1])) for r in reg]
        if not rules:
            continue
        rs = N.Ruleset(rules, strict=True)
        msgs = [N.js_utf8(v["input"]) for v in vs]
        data, off = N.pack(msgs)
        spans = rs.find_matches_batch(data, off)
        exp = oracle_spans(oracle, rules, data, off)
        got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in spans]
        assert got == exp
        for mi, v in enumerate(vs):
            u = oracle.js_units(v["input"])
            ms = [{"id": reg[r][2], "match": u[s:e].tobytes().decode("utf-16-le", "surrogatepass")} for (m, r, s, e) in got if m == mi]
            run_checks(ms, v["checks"])
        rs.close()


@pytest.mark.parametrize("n_rules,stride", [(17, 0), (17, 2), (64, 0), (120, 2), (120, 4), (500, 0), (500, 2), (2000, 0), (5000, 0)])
def test_policy_scan_equals_oracle(N, oracle, n_rules, stride):
    """stride 0 = the compiler's choice (17 built-ins: 4; larger sets: 2; 2000 / 5000 rules: level-1b tables in HBM);
    stride 4 forced on a synthetic set turns the factors no gram covers at four alignments into trigger bytes or
    always-candidate rules (spans checked too)"""
    rl = W.make_rules(n_rules)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, options=stride, strict=True)
    info = rs.info()
    assert stride == 0 or info.stride == stride
    if stride == 4:
        assert info.n_triggers + info.n_always_candidate >= 1
    n = 6000 if n_rules <= 2000 else 2500
    data_t, off_t, inj = W.make_messages(n, 256, rl, p_hit=0.05, seed=4242 + n_rules)
    data = data_t.numpy()
    off = off_t.numpy().astype(np.uint32)
    words, hits = rs.scan_batch(data, off)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert [(int(h["msg"]), int(h["rule"])) for h in hits] == ehits
    assert np.array_equal(words, ewords)
    assert len(ehits) >= len(inj)          # every injected token is a true hit
    if stride == 4:
        got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in rs.find_matches_batch(data, off)]
        assert got == oracle_spans(oracle, rules, data, off)
    rs.close()


def test_device_scan_equals_host_path(N, oracle):
    """cg_scan_batch_device: a run of different batches into separate output buffers equals the host path, batch by batch."""
    import torch
    rl = W.make_rules(500)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    n = 20000
    batches = []
    for seed in range(5):
        data_t, off_t, _ = W.make_messages(n, 256, rl, p_hit=0.03, seed=900 + seed)
        batches.append((data_t.numpy(), off_t.numpy().astype(np.uint32)))
    expect = [rs.scan_batch(d, o, want_hits=False)[0] for d, o in batches]
    ewords, _ = oracle_policy(oracle, rules, batches[0][0][:2000 * 256 + 64], batches[0][1][:2001])
    assert np.array_equal(expect[0][:2000], ewords)
    stream = torch.cuda.Stream()
    dev = [(torch.from_numpy(d).cuda(), torch.from_numpy(o.astype(np.int32)).cuda()) for d, o in batches]
    outs = [torch.full((n,), -1, dtype=torch.int64, device="cuda") for _ in batches]
    torch.cuda.synchronize()
    for rep in range(3):
        for (d, o), out in zip(dev, outs):
            rs.scan_batch_device(d.data_ptr(), o.data_ptr(), n, out.data_ptr(), stream.cuda_stream)
        rs.scan_join(stream.cuda_stream)
        stream.synchronize()
        for out, e in zip(outs, expect):
            assert np.array_equal(out.cpu().numpy().view(np.uint64), e)
            out.fill_(-1)
        torch.cuda.synchronize()
    rs.close()


def test_device_queue_overflow_is_reported_in_band(N, oracle):
    """A device-path batch that overflows a candidate queue cannot be re-run by the library: every result word of that
    batch says "incomplete" (all ones), cg_scan_join reports CG_ERR_CAPACITY once, and the same batch scanned again --
    the scratch has grown -- is complete and equals the oracle."""
    import torch
    rl = W.make_rules(64)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    st = torch.cuda.Stream()
    # a small first batch sizes the queues (>= 4096 slots / events); the next one hits in every message
    d0, o0, _ = W.make_messages(64, 256, rl, p_hit=0.0, seed=3)
    d1, o1, _ = W.make_messages(30000, 256, rl, p_hit=1.0, seed=4)
    outs = []
    for d, o in ((d0, o0), (d1, o1)):
        n = o.numel() - 1
        dd, oo = d.cuda(), o.to(torch.int32).cuda()
        out = torch.zeros(n, dtype=torch.int64, device="cuda")
        rs.scan_batch_device(dd.data_ptr(), oo.data_ptr(), n, out.data_ptr(), st.cuda_stream)
        outs.append((dd, oo, out, n))
    with pytest.raises(N.GovError) as ei:
        rs.scan_join(st.cuda_stream)
    assert ei.value.code == N.CG_ERR_CAPACITY
    assert (outs[0][2].cpu().numpy() == 0).all() or True          # (the small batch is complete, hits or not)
    assert (outs[1][2].cpu().numpy().view(np.uint64) == np.uint64(0xffffffffffffffff)).all()
    dd, oo, out, n = outs[1]
    for attempt in range(4):                                         # (a slot overflow hides how many VM events the batch needs: one more round)
        rs.scan_batch_device(dd.data_ptr(), oo.data_ptr(), n, out.data_ptr(), st.cuda_stream)
        try:
            rs.scan_join(st.cuda_stream)
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
            assert (out.cpu().numpy().view(np.uint64) == np.uint64(0xffffffffffffffff)).all()
    ewords, _ = oracle_policy(oracle, rules, d1.numpy()[:3000 * 256 + 64], o1.numpy().astype(np.uint32)[:3001])
    got = out.cpu().numpy().view(np.uint64)
    assert np.array_equal(got[:3000], ewords) and (got != np.uint64(0xffffffffffffffff)).all() and int((got >> np.uint64(63)).sum()) >= 29000
    rs.close()


def test_scanned_range_need_not_start_at_the_buffer_start(N, oracle):
    """The device path scans [offsets[0], offsets[n]) of the buffer: sub-ranges at every alignment (what the chunked host
    path does), tokens right at the first bytes of the range (no gram in front of them: the kernel's head check)."""
    import torch
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    rng = np.random.default_rng(5)
    msgs = []
    for i in range(400):
        L = int(rng.integers(0, 90))
        filler_t, _, _ = W.make_messages(1, L + 64, rl, p_hit=0.0, seed=1000 + i)
        m = bytearray(filler_t.numpy()[:L].tobytes())
        if i % 3 == 0:
            tok = rl[int(rng.integers(0, len(rl)))]["sample"].encode()
            m = bytearray(tok) + m                                  # the message starts with a token
        msgs.append(bytes(m))
    data, off = N.pack(msgs)
    ewords, _ = oracle_policy(oracle, rules, data, off)
    d = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
    o = torch.from_numpy(off.astype(np.int32)).cuda()
    st = torch.cuda.Stream()
    n_hit = 0
    for m0 in range(0, 400, 7):
        m1 = min(400, m0 + 61)
        out = torch.full((m1 - m0,), -1, dtype=torch.int64, device="cuda")
        rs.scan_batch_device(d.data_ptr(), o.data_ptr() + 4 * m0, m1 - m0, out.data_ptr(), st.cuda_stream)
        rs.scan_join(st.cuda_stream)
        got = out.cpu().numpy().view(np.uint64)
        assert np.array_equal(got, ewords[m0:m1]), m0
        n_hit += int((got >> np.uint64(63)).sum())
    assert n_hit >= 500
    with pytest.raises(N.GovError):
        rs.scan_batch_device(d.data_ptr() + 4, o.data_ptr(), 10, out.data_ptr(), st.cuda_stream)     # d_bytes must be 16-byte aligned
    rs.close()


@pytest.mark.parametrize("utf8_frac,length", [(0.2, 190), (0.0, 64), (0.1, 1024)])
def test_redaction_spans_equal_oracle(N, oracle, utf8_frac, length):
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(2500, length, rl, p_hit=0.2, utf8_frac=utf8_frac, seed=99 + length)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    spans = rs.find_matches_batch(data, off)
    got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in spans]
    assert got == oracle_spans(oracle, rules, data, off)
    # byte offsets delimit the same text as the UTF-16 offsets
    for s in spans[:200]:
        m = bytes(data[off[s["msg"]]:off[s["msg"] + 1]])
        txt = m.decode("utf-8", "replace")
        u = oracle.js_units(txt)
        a = m[s["start_byte"]:s["end_byte"]].decode("utf-8", "replace")
        b = u[s["start16"]:s["end16"]].tobytes().decode("utf-16-le", "replace")
        assert a == b
    rs.close()


def test_ragged_empty_and_edge_inputs(N, oracle):
    rules = [(r"sk-[a-zA-Z0-9]{20,}", 0, 0), (r"\d+", 0, 3), (r"", 0, 3), (r"^$", 0, 3), (r"a*?b", 0, 3), (r"x\b", 0, 3), (r"(?:a??)?", 0, 3)]
    rs = N.Ruleset(rules, strict=True)
    rng = np.random.default_rng(3)
    msgs = [b"", b"a", b"sk-" + b"a" * 25, b"", b"12 345", "😀".encode(), b"aab xb", b"x" * 700 + b" 9"]
    msgs += [bytes(rng.integers(32, 127, int(k), dtype=np.uint8)) for k in rng.integers(0, 90, 300)]
    msgs += [bytes(rng.integers(0, 256, int(k), dtype=np.uint8)) for k in rng.integers(0, 40, 200)]   # invalid UTF-8 too
    data, off = N.pack(msgs)
    words, hits = rs.scan_batch(data, off)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert [(int(h["msg"]), int(h["rule"])) for h in hits] == ehits
    assert np.array_equal(words, ewords)
    spans = rs.find_matches_batch(data, off)
    got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in spans]
    assert got == oracle_spans(oracle, rules, data, off)
    # n = 0
    d0, o0 = N.pack([])
    w0, h0 = rs.scan_batch(d0, o0)
    assert len(w0) == 0 and len(h0) == 0
    rs.close()


def test_failed_rules_never_match_and_report_status(N):
    rs = N.Ruleset([("ok+", 0, 3), ("a(b", 0, 3), (r"(x)\1", 0, 3)])
    assert list(rs.status) == [0, N.CG_ERR_SYNTAX, N.CG_ERR_UNSUPPORTED]
    data, off = N.pack([b"okkk a(b xx"])
    words, hits = rs.scan_batch(data, off)
    assert [(int(h["msg"]), int(h["rule"])) for h in hits] == [(0, 0)]
    with pytest.raises(N.GovError):
        N.Ruleset([("a(b", 0, 3)], strict=True)
    rs.close()


def test_single_long_message(N, oracle):
    rl = W.make_rules(40)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(1, 65536, rl, p_hit=1.0, seed=5)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    spans = rs.find_matches_batch(data, off)
    got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in spans]
    assert got == oracle_spans(oracle, rules, data, off)
    rs.close()


def test_long_and_ragged_messages(N, oracle):
    """The scan is position-parallel over the buffer, so message lengths do not matter to it: tokens placed on and around
    every 1 KB boundary (warp tiles are 512 bytes) must be found exactly once, for ragged lengths, through the host path
    and the device path."""
    import torch
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    rng = np.random.default_rng(99)
    lens = [5000, 3 * 1024 + 5, 2049, 100, 70000, 0, 1024, 2048, 4096 + 17, 33, 9000]
    filler_t, _, _ = W.make_messages(1, sum(lens) + 64, rl, p_hit=0.0, seed=17)
    filler = filler_t.numpy()
    msgs, pos = [], 0
    for L in lens:
        m = bytearray(filler[pos:pos + L].tobytes()); pos += L
        for b in range(1024, L, 1024):                       # a token ending / starting / straddling each boundary
            r = rl[int(rng.integers(17, len(rl)))]
            tok = (" " + r["sample"] + " ").encode()
            at = b + int(rng.integers(-len(tok) - 2, 3))
            if 0 <= at and at + len(tok) <= L:
                m[at:at + len(tok)] = tok
        msgs.append(bytes(m))
    data, off = N.pack(msgs)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert len(ehits) >= 60
    for rep in range(2):
        words, hits = rs.scan_batch(data, off)
        assert np.array_equal(words, ewords)
        assert [(int(h["msg"]), int(h["rule"])) for h in hits] == ehits
    d = torch.from_numpy(np.concatenate([data, np.zeros(64, np.uint8)])).cuda()
    o = torch.from_numpy(off.astype(np.int32)).cuda()
    out = torch.full((len(msgs),), -1, dtype=torch.int64, device="cuda")
    st = torch.cuda.Stream()
    for rep in range(3):
        rs.scan_batch_device(d.data_ptr(), o.data_ptr(), len(msgs), out.data_ptr(), st.cuda_stream)
        rs.scan_join(st.cuda_stream)
        st.synchronize()
        assert np.array_equal(out.cpu().numpy().view(np.uint64), ewords)
    spans = rs.find_matches_batch(data, off)
    got = [(int(x["msg"]), int(x["rule"]), int(x["start16"]), int(x["end16"])) for x in spans]
    assert got == oracle_spans(oracle, rules, data, off)
    # and back to a short-message batch on the same rule set
    data2_t, off2_t, _ = W.make_messages(3000, 200, rl, p_hit=0.1, seed=18)
    data2, off2 = data2_t.numpy(), off2_t.numpy().astype(np.uint32)
    w2, _ = rs.scan_batch(data2, off2)
    assert np.array_equal(w2, oracle_policy(oracle, rules, data2, off2)[0])
    rs.close()


def test_redact_batch_equals_oracle_splice(N, oracle):
    """cg_redact_batch: findMatches + applyReplacements with [REDACTED:<category>:<hash8>] (engine.ts:165-181,
    vault.ts:33-35), bytes and digests exact, on ragged UTF-8 messages."""
    import hashlib
    rl = W.make_rules(200)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    data_t, off_t, _ = W.make_messages(4000, 180, rl, p_hit=0.3, utf8_frac=0.15, seed=77)
    buf = data_t.numpy()
    off0 = off_t.numpy()
    rng = np.random.default_rng(5)
    msgs = [bytes(buf[int(off0[i]):int(off0[i]) + int(rng.integers(0, 181))]) for i in range(4000)]     # ragged, may cut a character
    data, off = N.pack(msgs)
    out, out_off, spans, dig = rs.redact_batch(data, off)
    exp_spans = oracle_spans(oracle, rules, data, off)
    got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in spans]
    assert got == exp_spans and len(got) >= 300
    by_msg = {}
    for s, d in zip(spans, dig):
        m = msgs[int(s["msg"])][int(s["start_byte"]):int(s["end_byte"])]
        assert bytes(d) == hashlib.sha256(m).digest()
        by_msg.setdefault(int(s["msg"]), []).append((int(s["start_byte"]), int(s["end_byte"]), CATS[rules[int(s["rule"])][2]], bytes(d).hex()[:8]))
    assert int(out_off[0]) == 0 and len(out) == int(out_off[-1])
    for i, m in enumerate(msgs):
        e = bytearray(m)
        for a, b, cat, h8 in sorted(by_msg.get(i, []), reverse=True):                 # right to left, as applyReplacements
            e[a:b] = ("[REDACTED:%s:%s]" % (cat, h8)).encode()
        assert bytes(out[int(out_off[i]):int(out_off[i + 1])]) == bytes(e), i
    rs.close()


# ------------------------------------------------------------------------------ SHA-256 / Merkle

def test_sha256_batch_equals_hashlib_and_oracle(N, oracle):
    rng = np.random.default_rng(11)
    msgs = [bytes(rng.integers(0, 256, int(k), dtype=np.uint8)) for k in list(range(0, 140)) + [255, 256, 257, 1000, 5000]]
    msgs += [b"abc", b"", b"Hello World!"]
    off = np.zeros(len(msgs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    data = np.frombuffer(b"".join(msgs) + b"\0" * 64, dtype=np.uint8).copy()
    out = N.sha256_batch(data, off)
    for i, m in enumerate(msgs):
        assert out[i].tobytes() == hashlib.sha256(m).digest()
    assert np.array_equal(out, oracle.sha256_batch(data, off))
    assert out[-1].tobytes().hex() == "7f83b1657ff1fc53b92dc18148a1d65dfc2d4b1fa3d677284addd200126d9069"  # gov/RFC.md:1562


@pytest.mark.parametrize("n", [0, 1, 2, 3, 5, 8, 33, 1000, 4097, 100003])
def test_merkle_root_variable_leaves(N, oracle, n):
    rng = np.random.default_rng(n + 1)
    lens = rng.integers(0, 300, n)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    data = rng.integers(0, 256, int(off[-1]) + 64, dtype=np.uint8)
    assert N.merkle_root(data, off) == oracle.merkle_root(data, off)


@pytest.mark.parametrize("n,leaf", [(1 << 16, 256), (100003, 256), (50000, 32), (7777, 64), (999, 1024), (1234, 37)])
def test_merkle_root_fixed_leaves(N, oracle, n, leaf):
    data = W.make_leaves(n, leaf).numpy()
    assert N.merkle_root_fixed(data, leaf, n) == oracle.merkle_root_fixed(data, leaf, n)


def test_merkle_fold_of_block_roots(N, oracle):
    n, leaf, k = 10000, 64, 8
    data = W.make_leaves(n, leaf).numpy()
    roots = []
    for s in range(0, n, 1 << k):
        e = min(n, s + (1 << k))
        roots.append(np.frombuffer(N.merkle_root_fixed(data[s * leaf:], leaf, e - s), dtype=np.uint8))
    assert N.merkle_fold(np.stack(roots)) == oracle.merkle_root_fixed(data, leaf, n)


def test_merkle_log_append_frontier_and_proofs(N, oracle):
    """Append-only log: the root after every append equals the one-shot tree over all leaves so far (device and oracle),
    the persisted frontier resumes the log, and RFC 6962 audit paths equal the oracle's and verify (RFC 9162 2.1.3.2)."""
    rng = np.random.default_rng(2024)
    leaves = [bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)) for _ in range(2500)]
    log = N.MerkleLog(keep_leaf_digests=True)
    assert log.root() == hashlib.sha256(b"").digest() and log.size() == 0
    done = 0
    for chunk in [1, 1, 2, 3, 5, 64, 63, 1, 256, 700, 1, 1000, 403]:
        log.append(leaves[done:done + chunk]); done += chunk
        data, off = N.pack(leaves[:done])
        assert log.size() == done
        assert log.root() == oracle.merkle_root(data, off.astype(np.uint64)) == N.merkle_root(data, off.astype(np.uint64))
        assert len(log.frontier()) == bin(done).count("1")
    assert done == 2500
    root = log.root()
    # persisted frontier -> resumed log keeps producing the same roots
    resumed = N.MerkleLog.restore(done, log.frontier())
    extra = [b"event-%d" % i for i in range(37)]
    log.append(extra); resumed.append(extra)
    assert resumed.root() == log.root() and resumed.size() == done + 37
    all_leaves = leaves + extra
    root2 = log.root()
    small = all_leaves[:77]                                  # the pure-Python oracle paths are for small trees
    slog = N.MerkleLog()
    slog.append(small)
    sroot = slog.root()
    for i in [0, 1, 31, 32, 63, 64, 75, 76]:
        p = slog.proof(i)
        assert p == oracle.merkle_audit_path(small, i)
        assert oracle.merkle_verify_path(small[i], i, len(small), p, sroot) and N.merkle_verify_proof(small[i], i, len(small), p, sroot)
    for i in [0, 1, 1234, 2047, 2048, 2499, 2500, 2536]:
        p = log.proof(i)
        assert oracle.merkle_verify_path(all_leaves[i], i, len(all_leaves), p, root2)
        assert N.merkle_verify_proof(all_leaves[i], i, len(all_leaves), p, root2)
        assert not N.merkle_verify_proof(all_leaves[i] + b"x", i, len(all_leaves), p, root2)
        assert not N.merkle_verify_proof(all_leaves[i], i, len(all_leaves), p, root)          # an older root
        if p:
            assert not N.merkle_verify_proof(all_leaves[i], i ^ 1, len(all_leaves), p, root2)
    for lg in (log, resumed, slog):
        lg.close()


def test_merkle_ct_reference_vectors_on_the_device(N, oracle):
    """The Certificate Transparency known answers (tests/golden/ct_merkle_vectors.json) through the C ABI: roots of the
    first k leaves (one-shot and incremental log), audit paths, consistency proofs, both verifiers."""
    import json
    v = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ct_merkle_vectors.json")))
    leaves = [bytes.fromhex(x) for x in v["leaves_hex"]]
    roots = [bytes.fromhex(x) for x in v["roots_hex"]]
    log = N.MerkleLog()
    for k in range(1, 9):
        data, off = N.pack(leaves[:k])
        assert N.merkle_root(data, off.astype(np.uint64)) == roots[k - 1]
        log.append(leaves[k - 1:k])
        assert log.root() == roots[k - 1]
    for c in v["inclusion"]:
        lg = N.MerkleLog(); lg.append(leaves[:c["size"]])
        p = lg.proof(c["index"])
        assert [x.hex() for x in p] == c["path_hex"]
        assert N.merkle_verify_proof(leaves[c["index"]], c["index"], c["size"], p, roots[c["size"] - 1])
        lg.close()
    for c in v["consistency"]:
        lg = N.MerkleLog(); lg.append(leaves[:c["second"]])
        p = lg.consistency(c["first"])
        assert [x.hex() for x in p] == c["path_hex"]
        assert N.merkle_verify_consistency(c["first"], c["second"], roots[c["first"] - 1], roots[c["second"] - 1], p)
        lg.close()
    log.close()


def test_merkle_consistency_proofs(N, oracle):
    """RFC 6962 2.1.2 proofs from the log equal the oracle's for every (m, n) of a small tree, and verify (device verifier,
    RFC 9162 2.1.4.2, and the oracle's); on a 70k-leaf log the proofs verify against roots recorded along the way and
    any tampering (root, path length, sizes) is rejected."""
    rng = np.random.default_rng(62)
    leaves = [bytes(rng.integers(0, 256, int(rng.integers(0, 120)), dtype=np.uint8)) for _ in range(70)]
    log = N.MerkleLog(); roots = [None]
    for x in leaves:
        log.append([x]); roots.append(log.root())
    for n in (1, 2, 3, 7, 8, 9, 33, 64, 70):
        lg = N.MerkleLog(); lg.append(leaves[:n])
        for m in range(1, n + 1):
            p = lg.consistency(m)
            assert p == oracle.merkle_consistency_proof(leaves[:n], m), (m, n)
            assert N.merkle_verify_consistency(m, n, roots[m], roots[n], p)
            assert oracle.merkle_verify_consistency(m, n, roots[m], roots[n], p)
            if m < n:
                assert not N.merkle_verify_consistency(m, n, roots[m], roots[n - 1] if n - 1 != m else roots[n][::-1], p)
                assert not N.merkle_verify_consistency(m, n, roots[m][::-1], roots[n], p)
                assert not N.merkle_verify_consistency(m, n, roots[m], roots[n], p[:-1])
                assert not N.merkle_verify_consistency(m, n, roots[m], roots[n], p + [p[-1]])
        assert not N.merkle_verify_consistency(0, n, roots[1], roots[n], [])
        lg.close()
    log.close()
    big = N.MerkleLog(); marks = {}
    n = 0
    for chunk in (1, 4095, 1, 32768, 12345, 20000):
        data = W.make_leaves(chunk, 48, seed=n + 1).numpy()
        off = (np.arange(chunk + 1, dtype=np.uint64) * 48)
        big.append_packed(data, off); n += chunk
        marks[n] = big.root()
    for m, rm in marks.items():
        p = big.consistency(m)
        assert N.merkle_verify_consistency(m, n, rm, marks[n], p) and oracle.merkle_verify_consistency(m, n, rm, marks[n], p)
        if m < n:                                            # wrong sizes: whatever RFC 9162's walk says (the oracle), mostly "no"
            for mm, nn in ((m, n - 1), (m + 1, n), (m, n + 1), (m - 1, n), (m, 2 * n)):
                assert N.merkle_verify_consistency(mm, nn, rm, marks[n], p) == oracle.merkle_verify_consistency(mm, nn, rm, marks[n], p), (mm, nn)
            assert not N.merkle_verify_consistency(m + 1, n, rm, marks[n], p)
    big.close()


def test_merkle_log_from_jsonl_bytes(N, oracle):
    """The event log as it lies on disk (JSON lines, src/audit-trail.ts:151-179): split on the device; every line without
    its newline is a leaf.  Empty lines, an unterminated last line, lines across the 4 KB pieces of the split kernel."""
    rng = np.random.default_rng(151)
    lines = [b'{"id":"%d","verdict":"allow","pad":"%s"}' % (i, b"x" * int(rng.integers(0, 900))) for i in range(3000)]
    lines[5] = b""; lines[6] = b""; lines[100] = b"y" * 9000; lines[2999] = b"tail"
    blob = b"\n".join(lines) + b"\n"
    data, off = N.pack(lines)
    want = oracle.merkle_root(data, off.astype(np.uint64))
    log = N.MerkleLog(keep_leaf_digests=False)
    assert log.append_jsonl(blob) == 3000 and log.size() == 3000 and log.root() == want
    log.close()
    log = N.MerkleLog()                                   # in flushes that end mid-file, last one unterminated
    cut = [0, 1, 4096, 4097, 50000, len(blob) - 1]
    cut = [blob.rfind(b"\n", 0, c) + 1 for c in cut] + [len(blob) - 1]
    total = 0
    for a, b in zip(cut[:-1], cut[1:]):
        total += log.append_jsonl(blob[a:b])
    assert total == 3000 and log.root() == want
    assert log.append_jsonl(b"") == 0 and log.append_jsonl(b"\n") == 1 and log.size() == 3001
    p = log.proof(100)
    assert N.merkle_verify_proof(lines[100], 100, 3001, p, log.root())
    log.close()


@pytest.mark.parametrize("n", [1, 2, 3, 31, 32, 33, 1023, 1024, 1025, 32767, 32768, 32769, 200001])
def test_merkle_subtree_reduction_sizes(N, oracle, n):
    """log roots over n leaves for n around the warp-shuffle reduction's boundaries (32 per warp, 2^15 switch to the level kernels)"""
    data = W.make_leaves(n, 40, seed=n).numpy()
    off = np.arange(n + 1, dtype=np.uint64) * 40
    log = N.MerkleLog(keep_leaf_digests=(n < 40000))
    log.append_packed(data, off)
    assert log.root() == oracle.merkle_root_fixed(data, 40, n) == N.merkle_root(data, off)
    log.close()


def test_sha256_ragged_alignment(N, oracle):
    """word-granular ragged leaves: every start alignment mod 16 x every length 0..200"""
    rng = np.random.default_rng(256)
    msgs = []
    for pad in range(16):
        msgs.append(bytes(rng.integers(0, 256, pad, dtype=np.uint8)))
        for ln in list(range(0, 70)) + [119, 120, 127, 128, 129, 200]:
            msgs.append(bytes(rng.integers(0, 256, ln, dtype=np.uint8)))
    off = np.zeros(len(msgs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    data = np.frombuffer(b"".join(msgs) + b"\0" * 64, dtype=np.uint8).copy()
    out = N.sha256_batch(data, off)
    for i, m in enumerate(msgs):
        assert out[i].tobytes() == hashlib.sha256(m).digest(), (i, len(m))
    assert N.merkle_root(data, off) == oracle.merkle_root(data, off)
    sub = off[7:]                                          # offsets[0] != 0
    assert N.merkle_root(data, sub) == oracle.merkle_root(data, sub)


def test_programs_longer_than_the_small_vm(N, oracle):
    """verify_large_kernel: rules whose Pike program exceeds the shared-memory VM's 192 instructions (and the bit-parallel
    matcher's 63) -- policy words and spans equal the oracle's."""
    rules = [(r"tok_[a-f0-9]{200}z", 0, 0), (r"(?:ab|cd|ef){70}!", 0, 1), (r"sk-[a-zA-Z0-9]{20,}", 0, 2), (r"key=[A-Z]{100}[0-9]{100}\b", 1, 3)]
    rng = np.random.default_rng(192)
    hexd = b"0123456789abcdef"
    msgs = []
    for i in range(400):
        k = i % 8
        if k == 0: body = b"tok_" + bytes(rng.choice(np.frombuffer(hexd, dtype=np.uint8), 200)) + b"z"
        elif k == 1: body = b"tok_" + bytes(rng.choice(np.frombuffer(hexd, dtype=np.uint8), 199)) + b"z"          # one short
        elif k == 2: body = b"".join([b"ab", b"cd", b"ef"][int(x)] for x in rng.integers(0, 3, 70)) + b"!"
        elif k == 3: body = b"".join([b"ab", b"cd", b"ef"][int(x)] for x in rng.integers(0, 3, 69)) + b"x!"
        elif k == 4: body = b"KEY=" + b"Q" * 100 + b"7" * 100
        elif k == 5: body = b"key=" + b"q" * 100 + b"7" * 100 + b"a"                                             # \b fails
        elif k == 6: body = b"sk-" + b"a1B2" * 6
        else: body = b"nothing to see"
        msgs.append(b"pad " * int(rng.integers(0, 5)) + body + b" tail" * int(rng.integers(0, 3)))
    rs = N.Ruleset(rules, strict=True)
    assert rs.info().program_words > 600
    data, off = N.pack(msgs)
    words, hits = rs.scan_batch(data, off)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert np.array_equal(words, ewords) and [(int(h["msg"]), int(h["rule"])) for h in hits] == ehits and len(ehits) >= 200
    spans = rs.find_matches_batch(data, off)
    got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in spans]
    assert got == oracle_spans(oracle, rules, data, off) and len(got) >= 200
    rs.close()


def test_cortex_language_packs_on_the_kernels(N, oracle):
    """The ten real language packs of openclaw-cortex as ONE rule set (70 rules, flag i on Cyrillic / Latin-1 literals, CJK,
    Hangul): the reference's own 100 anyMatch assertions through the kernels, and the policy words of the whole batch
    against the oracle."""
    c = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cortex_pack_vectors.json"), encoding="utf-8"))
    rules, where = [], {}
    for lang, cats in c["packs"].items():
        for cat, pats in cats.items():
            for p in pats:
                where.setdefault((lang, cat), []).append(len(rules))
                rules.append((p["source"], 1 if "i" in p["flags"] else 0, 3))
    rs = N.Ruleset(rules, strict=True)
    msgs = [v["text"].encode("utf-8") for v in c["vectors"]] * 20
    data, off = N.pack(msgs)
    words, hits = rs.scan_batch(data, off)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert np.array_equal(words, ewords) and [(int(h["msg"]), int(h["rule"])) for h in hits] == ehits
    by_msg = {}
    for h in hits:
        by_msg.setdefault(int(h["msg"]), set()).add(int(h["rule"]))
    for i, v in enumerate(c["vectors"]):
        assert any(r in by_msg.get(i, set()) for r in where[(v["lang"], v["category"])]) == v["expect"], (v["lang"], v["category"], v["text"])
    rs.close()


def test_non_ascii_rule_packs_on_the_kernels(N, oracle):
    """SURVEY 8 f4: CJK / Cyrillic / Hangul literal alternations, classes with CJK ranges, `.*` between literals and the
    lazy PEM block: policy words, hits and resolved spans equal the oracle's."""
    rs = N.Ruleset(PACK_RULES, strict=True)
    msgs = [t.encode("utf-8") for t in PACK_TEXTS] * 40
    data, off = N.pack(msgs)
    words, hits = rs.scan_batch(data, off)
    ewords, ehits = oracle_policy(oracle, PACK_RULES, data, off)
    assert np.array_equal(words, ewords) and [(int(h["msg"]), int(h["rule"])) for h in hits] == ehits and len(ehits) >= 400
    spans = rs.find_matches_batch(data, off)
    got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in spans]
    assert got == oracle_spans(oracle, PACK_RULES, data, off)
    rs.close()


def test_chunked_host_scan_equals_one_piece_scan(N, oracle):
    """Large words-only host batches go through the chunked path (copies overlapped with the kernels): same words as
    the one-piece path, ragged lengths, and the hit count derived from the words equals the hit list's length."""
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    n = 90000
    data_t, off_t, _ = W.make_messages(n, 96, rl, p_hit=0.05, seed=321)
    buf, off0 = data_t.numpy(), off_t.numpy()
    rng = np.random.default_rng(8)
    lens = rng.integers(0, 97, n)
    off = np.zeros(n + 1, dtype=np.uint32); off[1:] = np.cumsum(lens)
    data = np.zeros(int(off[-1]) + 64, dtype=np.uint8)
    src = np.repeat(off0[:-1].astype(np.int64), lens) + (np.arange(int(off[-1])) - np.repeat(off[:-1].astype(np.int64), lens))
    data[:int(off[-1])] = buf[src]
    w_one, hits = rs.scan_batch(data, off, want_hits=True)              # one piece (hit list requested)
    w_chunk, _ = rs.scan_batch(data, off, want_hits=False)              # chunked
    assert np.array_equal(w_one, w_chunk)
    assert int(((w_chunk >> np.uint64(32)) & np.uint64(0x7fffffff))[w_chunk >> np.uint64(63) == 1].sum()) == len(hits) >= 1000
    sub = 3000
    ewords, _ = oracle_policy(oracle, rules, data[: int(off[sub]) + 64], off[: sub + 1])
    assert np.array_equal(w_chunk[:sub], ewords)
    rs.close()


def test_random_regex_differential_on_the_kernels(N, oracle):
    """The CPU tier fuzzes the compiler + VM on the host; this is the same differential through the real kernels:
    ~250 random patterns (those both sides accept) as ONE rule set, dense / empty / astral matches, policy words + hits
    and resolved spans against the oracle."""
    rng = np.random.default_rng(777)
    alphabet = ["a", "b", "c", "1", " ", "é", "😀", "\n", "A"]
    texts = ["".join(alphabet[int(k)] for k in rng.integers(0, len(alphabet), int(rng.integers(0, 24)))) for _ in range(80)]
    texts += ["", "a", "aaaa", "abcabc", "😀", "a😀b", "1 a1"]
    msgs = [t.encode("utf-8") for t in texts]
    data, off = N.pack(msgs)
    rules = []
    for _ in range(700):
        src = random_regex(rng)
        fl = 1 if rng.random() < 0.2 else 0
        try:
            rx = oracle.Regex(src, "i" if fl else "")
            oracle.find_matches_batch([(rx, "custom")], data, off.astype(np.uint64))      # exponential backtracking -> RuntimeError
        except (oracle.RegexSyntaxError, oracle.OracleUnsupported, RuntimeError):
            continue
        if N.rule_check(src, fl) != 0:
            continue
        rules.append((src, fl, int(rng.integers(0, 4))))
        if len(rules) == 250:
            break
    assert len(rules) >= 200
    rs = N.Ruleset(rules, strict=True)
    words, hits = rs.scan_batch(data, off)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert [(int(h["msg"]), int(h["rule"])) for h in hits] == ehits and np.array_equal(words, ewords) and len(ehits) > 3000
    spans = rs.find_matches_batch(data, off)
    got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in spans]
    assert got == oracle_spans(oracle, rules, data, off)
    rs.close()


def test_single_message_path_equals_the_batch_path(N, oracle):
    """cg_scan_one (pinned staging + the step as one graph over fixed addresses) against cg_scan_batch and the oracle:
    lengths around every boundary of the fast path (0, one chunk, 16 KB, beyond -> general path), non-ASCII text,
    interleaved with batch calls that grow the scratch (the graph must be re-captured), 160 rules (five hit words)."""
    rl = W.make_rules(160)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    rng = np.random.default_rng(5)
    samples = [r["sample"].encode() for r in rl if r["sample"]]
    msgs = [b"", b"a", b"x" * 15, b"y" * 16, b"z" * 17]
    for L in (255, 256, 1000, 4096, 16383, 16384, 16385, 40000):
        body = bytes(rng.integers(97, 123, L, dtype=np.uint8))
        s = samples[int(rng.integers(0, len(samples)))]
        p = int(rng.integers(0, max(1, L - len(s))))
        msgs.append(body[:p] + s + body[p + len(s):] if L > len(s) + 2 else body)
    msgs += [("пароль sk-" + "a" * 24 + " ключ bob@example.com 4111 1111 1111 1111").encode(), samples[0] + b" " + samples[1], samples[2]]
    data, off = N.pack(msgs)
    words, hits = rs.scan_batch(data, off)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert np.array_equal(words, ewords) and [(int(h["msg"]), int(h["rule"])) for h in hits] == ehits
    for rep in range(2):
        for i, m in enumerate(msgs):
            w1, r1 = rs.scan_one(m)
            assert w1 == int(words[i]), (i, len(m))
            assert r1 == [r for (mm, r) in ehits if mm == i], (i, len(m))
        # a batch large enough to grow the scratch in between: the single-message graph is re-captured
        big, boff, _ = W.make_messages(200000 if rep == 0 else 1000, 64, rl, p_hit=0.05, seed=11)
        rs.scan_batch(big.numpy(), boff.numpy().astype(np.uint32))
    rs.close()


def test_island_matcher_features_through_the_kernels(N, oracle):
    """resolve_kernel's island matcher on the device: two-word programs (64 .. 127 consuming instructions), lookaround guards,
    resume behind the confirmed factor, islands longer than the 96 steps it walks itself (those go to the VM) -- the same
    rules and boundary texts as the CPU tier's test_island_matcher_two_words_lookaround_and_factor_skip, plus long messages."""
    rules = [
        (r"(?<![A-Z0-9])PZULOYQ[0-9A-Z]{16}(?![A-Z0-9])", 0, 3),
        (r"(?<!\d)\+?[1-9]\d{6,14}(?!\d)", 0, 3),
        (r"(?:password|passwd|pwd|secret|token|api_key|apikey)\s*[:=]\s*['\"]?[^\s'\"]{8,64}", 1, 3),
        (r"sk-ant-[a-zA-Z0-9-]{80,}", 0, 3),
        (r"hgisr[a-zA-Z0-9_-]{36,}", 0, 3),
        (r"(?<=[a-f])zq[0-9]{3}(?=[xy])", 0, 3),
        (r"\bkey_[a-z]{70,90}\b", 0, 3),
        (r"abc-[A-Za-z0-9]{16,40}", 0, 3),
        (r"[a-z]+@[a-z]+\.com", 0, 3),
    ]
    tok = "PZULOYQ" + "A1B2C3D4E5F6G7H8"
    texts = [tok, " " + tok, tok + " ", "x" + tok + ".", "X" + tok, tok + "9", "-" + tok + "-", tok[:-1], tok + tok,
             "+4915112345678", "call +4915112345678 now", "1234567", "123456", "a1234567b", "91234567890123456", "x+1234567",
             "token=abcdefgh", "TOKEN : 'abcdefghij'", "secret=short", "password = \"" + "p" * 64 + "\"", "api_key=" + "k" * 70, "pwd:1234567", "pwd:12345678",
             "sk-ant-" + "a" * 79, "sk-ant-" + "a" * 80, "say sk-ant-" + "Ab-9" * 25 + " end", "sk-ant-" + "a" * 200,
             "hgisr" + "_" * 35, "hgisr" + "_" * 36, "hgisr" + "x" * 120,
             "azq123x", "gzq123x", "fzq123y!", "azq12x", "zq123x", "azq123",
             "key_" + "a" * 69, "key_" + "a" * 70, "key_" + "a" * 90, "key_" + "a" * 91, "a key_" + "b" * 80 + " z", "xkey_" + "b" * 80,
             "abc-" + "Z" * 15, "abc-" + "Z" * 16, "abc-" + "Z" * 41, "abc-abc-" + "Q" * 16, "éabc-" + "Z" * 16, "abc-" + "Z" * 10 + "é" + "Z" * 16,
             "q" * 300 + "@example.com", "q" * 95 + "@example.com", "q" * 96 + "@example.com", "q" * 97 + "@example.com", "é" + "q" * 50 + "@example.com",
             ("lorem ipsum " * 400) + tok + (" dolor sit amet" * 300) + " token = " + "v" * 30]
    msgs = [N.js_utf8(t) for t in texts] * 3
    rs = N.Ruleset(rules, strict=True)
    data, off = N.pack(msgs)
    words, hits = rs.scan_batch(data, off)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert [(int(h["msg"]), int(h["rule"])) for h in hits] == ehits
    assert np.array_equal(words, ewords)
    assert len({r for (_, r) in ehits}) == len(rules)        # every rule hits somewhere
    for i in (0, 25, len(texts) - 1):
        assert rs.scan_one(msgs[i])[1] == [r for (m, r) in ehits if m == i]
    rs.close()


def test_vm_grid_follows_the_traffic(N, oracle):
    """verify_small_kernel's grid is sized by what the previous step sent to the VM (one CTA per SM while the island matcher
    decides everything, four above 2048 pairs): ASCII traffic, then traffic whose islands are full of non-ASCII text (the VM's),
    twice (the second time with the large grid), then ASCII again -- every batch equal to the oracle, on the host path and on
    the device path (whose cached graph is keyed on the grid)."""
    import torch
    rl = W.make_rules(120)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, strict=True)
    plain_t, poff_t, _ = W.make_messages(6000, 256, rl, p_hit=0.3, seed=21)
    heavy_t, hoff_t, _ = W.make_messages(80000, 256, rl, p_hit=1.0, seed=22, utf8_frac=1.0)
    sets = {"plain": (plain_t.numpy(), poff_t.numpy().astype(np.uint32)), "heavy": (heavy_t.numpy(), hoff_t.numpy().astype(np.uint32))}
    want = {k: oracle_policy(oracle, rules, d, o) for k, (d, o) in sets.items()}
    seen = []
    for name in ("plain", "heavy", "heavy", "plain"):
        data, off = sets[name]
        words, hits = rs.scan_batch(data, off)
        seen.append((name, rs.work_counters()[1]))
        assert np.array_equal(words, want[name][0]), name
        assert [(int(h["msg"]), int(h["rule"])) for h in hits] == want[name][1], name
    print("pairs sent to the VM per batch:", seen)        # (> 2048 switches to the large grid; either way the results must hold)
    dev = torch.device("cuda:0")
    stream = torch.cuda.Stream()
    for name in ("heavy", "plain", "heavy"):
        d, o = torch.from_numpy(sets[name][0]).to(dev), torch.from_numpy(sets[name][1].astype(np.int64)).to(torch.int32).to(dev)
        n = o.numel() - 1
        out = torch.zeros(n, dtype=torch.int64, device=dev)
        with torch.cuda.stream(stream):
            for _ in range(2):
                rs.scan_batch_device(d.data_ptr(), o.data_ptr(), n, out.data_ptr(), stream.cuda_stream)
                rs.scan_join(stream.cuda_stream)
        assert np.array_equal(out.cpu().numpy().view(np.uint64), want[name][0]), name
    rs.close()
