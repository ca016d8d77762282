"""GPU tier for cg_policy_eval_one (one evaluation context, one device round trip): its verdict and program rules equal the
restatement of policy_program fed with the oracle's hit sets (policy-slice cases, the built-ins, random policy sets, random
sets over the 500-rule C2 set with planted hits) and PolicyEvaluator.verdict_one equals verdict_batch of one context; the raw
C ABI outputs, return codes and statistics equal cg_policy_eval_batch with one context at the fast path's edges (text count,
bytes, empty texts, chunk and window seams, capacity with guard words); graphs per text count and per program; a queue
overflow answered through the batch call, with the fast path taken again afterwards; launches that do not depend on hits;
issue order behind a device-resident call on a held stream."""
import ctypes as C

import numpy as np
import pytest

import policy_program as PP
from test_gpu_policy_eval import c2_rules, to_dev
from test_gpu_redact_device import to_device
from vainplex_openclaw_b200 import plugin as P

pytestmark = pytest.mark.gpu
GUARD = 0x5a5a5a5a
MAX_TEXTS, MAX_BYTES = 64, 65536          # the fast path's limits (capi.cu kPeOneTexts / kPeOneBytes)
GATE = 200_000_000
INVALID_ARG = -1                          # CG_ERR_INVALID_ARG
STAT_FIELDS = ("messages_scanned", "bytes_scanned", "candidate_events", "verified_pairs", "hits", "spans", "sha256_items",
               "merkle_leaves", "last_merkle_ms")


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


@pytest.fixture(scope="module")
def torch():
    import torch as T
    return T


@pytest.fixture(scope="module")
def oracle_scanner(oracle):
    class OracleScanner:
        def __init__(self, rules, logger=None):
            self.rules = [([pats] if isinstance(pats, str) else list(pats)) for pats in rules]
            self.cache = {}

        def scan(self, texts):
            return [[ri for ri, pats in enumerate(self.rules) if oracle.matches_any(pats, [t], self.cache)] for t in texts]
    return OracleScanner


def stats(N):
    s = N.stats()
    return {f: getattr(s, f) for f in STAT_FIELDS}


def delta(a, b):
    return {f: b[f] - a[f] for f in STAT_FIELDS if f != "last_merkle_ms"} | {"last_merkle_ms": b["last_merkle_ms"]}


# ------------------------------------------------------------------------------------------ against the oracle

def check_set(N, policies, ctxs, oracle_scanner, other=None):
    """every context through cg_policy_eval_one against the restatement with the oracle's hit sets, and verdict_one against
    verdict_batch of that one context.  -> the number of matches seen"""
    pe = P.PolicyEvaluator(policies, other_condition=other)
    po = P.PolicyEvaluator(policies, scanner_cls=oracle_scanner, other_condition=other)
    assert pe.program.tolist() == po.program.tolist()
    rs = pe._program_ruleset()
    seen = 0
    for ctx in ctxs:
        texts, roles, ctx_off, atoms = pe.program_inputs([ctx])
        hits = po.scanner.scan(texts) if (po.scanner and texts) else [[] for _ in texts]
        words, matches = PP.restate(po.program, [set(h) for h in hits], roles, ctx_off, atoms)
        data, off = N.pack([N.js_utf8(t) for t in texts])
        assert rs.eval_one(data, off, roles, atoms[0]) == (int(words[0]), [int(j) for j in matches["rule"]]), ctx
        assert pe.verdict_one(ctx) == pe.verdict_batch([ctx])[0], ctx
        seen += len(matches)
    return seen


def test_slice_cases(N, oracle_scanner):
    for policies, ctxs in PP.slice_cases():
        check_set(N, policies, ctxs, oracle_scanner)


def test_builtins_on_tool_calls(N, oracle_scanner):
    assert check_set(N, PP.builtin_policies(), PP.tool_contexts(np.random.default_rng(5), 3000), oracle_scanner, PP.other_condition) > 500


def test_random_policy_sets(N, oracle_scanner):
    rng = np.random.default_rng(21)
    seen = 0
    for _ in range(150):
        seen += check_set(N, PP.random_policies(rng), PP.random_contexts(rng, 40), oracle_scanner, PP.other_condition)
    assert seen > 1000


def test_random_sets_over_the_c2_rules(N, oracle_scanner):
    rl = c2_rules()
    pats = [r["source"] for r in rl]
    samples = [r["sample"] for r in rl if r["sample"]]
    rng = np.random.default_rng(31)
    seen = 0
    for _ in range(20):
        pols = PP.random_policies(rng, patterns=list(rng.choice(pats, 40)), max_policies=12)
        seen += check_set(N, pols, PP.random_contexts(rng, 100, samples=samples), oracle_scanner, PP.other_condition)
    assert seen > 500


# ------------------------------------------------------------------------------------------ equal to the batch call

def raw_one(N, rs, data, off, roles, atoms, cap, want=True):
    n = len(off) - 1
    verdict, nr = C.c_uint32(GUARD), C.c_uint32(GUARD)
    rules = np.full(cap + 8, GUARD, np.uint32)
    rc = N.load().cg_policy_eval_one(rs.handle, data.ctypes.data, off.ctypes.data, roles.ctypes.data if n else None, n,
                                     atoms.ctypes.data if atoms.size else None, C.byref(verdict), rules.ctypes.data if want else None, cap,
                                     C.byref(nr) if want else None)
    assert (rules[cap:] == GUARD).all()
    return rc, verdict.value, nr.value, rules[:cap].tolist()


def raw_batch(N, rs, data, off, roles, atoms, cap, want=True):
    n = len(off) - 1
    ver = np.full(1, GUARD, np.uint32)
    m = np.zeros(cap + 8, N.POLICY_MATCH_DTYPE)
    m["ctx"], m["rule"] = GUARD, GUARD
    nm = C.c_uint32(GUARD)
    ctx = np.array([0, n], np.uint32)
    rc = N.load().cg_policy_eval_batch(rs.handle, data.ctypes.data, off.ctypes.data, roles.ctypes.data if n else None, n, ctx.ctypes.data,
                                       atoms.ctypes.data if atoms.size else None, 1, ver.ctypes.data, m.ctypes.data if want else None, cap,
                                       C.byref(nm) if want else None)
    assert (m["rule"][cap:] == GUARD).all()
    return rc, int(ver[0]), nm.value, m["rule"][:cap].tolist()


def same_as_batch(N, rs, data, off, roles, atoms, cap, want=True):
    """one call each way, outputs, return codes and cg_stats deltas compared.  -> the one-call's outputs"""
    s0 = stats(N)
    one = raw_one(N, rs, data, off, roles, atoms, cap, want)
    s1 = stats(N)
    bat = raw_batch(N, rs, data, off, roles, atoms, cap, want)
    s2 = stats(N)
    assert one == bat
    assert delta(s0, s1) == delta(s1, s2)
    return one


WORDS = ["alpha7", "beta", "gammma", "delta-42", "eps", "zeta zeta", "", "x"]


def seam_program(rng, n_rules_set, n_atoms, total=1100):
    """policies of 1..40 rules until `total` program rules, one of them straddling the 1024-rule window seam; each rule a small
    random expression over HIT(r, role) / ATOM / CONST leaves"""
    sizes = []
    while sum(sizes) < total:
        sizes.append(int(rng.integers(1, 41)))
    at = np.cumsum([0] + sizes)
    k = int(np.searchsorted(at, 1024, side="right")) - 1
    if at[k] == 1024:                                       # (the seam fell between two policies: merge them)
        sizes[k - 1] += sizes.pop(k)
    words = [len(sizes)]
    for sz in sizes:
        words += [0xffffffff if rng.random() < 0.7 else int(rng.integers(n_atoms)), sz]
        for _ in range(sz):
            def leaf():
                u = rng.random()
                if u < 0.5:
                    return [2 | int(rng.integers(n_rules_set)) << 3 | int(rng.integers(3)) << 24]
                if u < 0.85:
                    return [1 | int(rng.integers(n_atoms)) << 3]
                return [int(rng.integers(2)) << 3]
            ops = leaf()
            for _ in range(int(rng.integers(0, 3))):
                ops += leaf() + [int(rng.choice([3, 4]))]
            if rng.random() < 0.2:
                ops += [5]
            words += [int(rng.integers(4)) | (4 if rng.random() < 0.6 else 0), len(ops)] + ops
    return np.array(words, np.uint32)


def texts_case(N, rng, n, total_bytes=None):
    """n texts (one role each of 0..2) drawn from WORDS, or padded so that together they hold exactly total_bytes"""
    ts = [" ".join(rng.choice(WORDS, int(rng.integers(0, 4)))).encode() for _ in range(n)]
    if total_bytes is not None:
        per = total_bytes // max(n, 1)
        ts = [(t + b"." * per)[:per] for t in ts]
        ts[-1] += b"." * (total_bytes - per * n)
        assert sum(map(len, ts)) == total_bytes
    data, off = N.pack(ts)
    return data, off, rng.integers(0, 3, n).astype(np.uint8)


@pytest.fixture(scope="module")
def seam_case(N):
    rng = np.random.default_rng(77)
    rs = N.Ruleset([("alpha\\d", 0, 3), ("beta", 0, 3), ("gam+a", 0, 3), ("delta-\\d+", 0, 3), ("zeta", 1, 3)], strict=True)
    n_atoms = 40
    rs.set_policy_program(seam_program(rng, 5, n_atoms), n_atoms)
    return rs, rng, n_atoms


def test_edges_equal_the_batch_call(N, seam_case):
    rs, rng, n_atoms = seam_case
    counts = []
    for n, total in ((0, None), (1, None), (2, None), (MAX_TEXTS, None), (MAX_TEXTS + 1, None), (MAX_TEXTS, MAX_BYTES), (MAX_TEXTS, MAX_BYTES + 1),
                     (3, MAX_BYTES), (1, MAX_BYTES + 1)):
        for _ in range(4):
            data, off, roles = texts_case(N, rng, n, total)
            atoms = rng.integers(0, 2**32, (n_atoms + 31) // 32, dtype=np.uint64).astype(np.uint32)
            rc, v, nm, _ = same_as_batch(N, rs, data, off, roles, atoms, 2048)
            assert rc == N.CG_OK and nm != GUARD and v != GUARD
            same_as_batch(N, rs, data, off, roles, atoms, 0, want=False)
            counts.append(nm)
            if nm >= 1:
                for cap in (nm - 1, nm, nm + 1):
                    rc, _v, nm2, rules = same_as_batch(N, rs, data, off, roles, atoms, cap)
                    assert nm2 == nm and rc == (N.CG_ERR_CAPACITY if cap < nm else N.CG_OK)
                    assert rules[min(cap, nm):] == [GUARD] * (cap - min(cap, nm))
    assert max(counts) > 20                                    # (matches on both sides of the chunk and window seams)
    # empty texts, all of them or some
    for ts in ([b""] * 5, [b"", b"beta", b"", b"zeta"], [b""] * MAX_TEXTS):
        data, off = N.pack(ts)
        same_as_batch(N, rs, data, off, rng.integers(0, 3, len(ts)).astype(np.uint8), np.full((n_atoms + 31) // 32, 0xffffffff, np.uint32), 64)
    # texts that start past offset 0 of the caller's buffer
    data, off, roles = texts_case(N, rng, 10)
    off2 = (off + 37).astype(np.uint32)
    data2 = np.concatenate([np.full(37, ord("b"), np.uint8), data])
    atoms = np.zeros((n_atoms + 31) // 32, np.uint32)
    assert same_as_batch(N, rs, data2, off2, roles, atoms, 64) == raw_one(N, rs, data, off, roles, atoms, 64)


def test_argument_checks_equal_the_batch_call(N, seam_case):
    rs, rng, n_atoms = seam_case
    data, off, roles = texts_case(N, rng, 4)
    atoms = np.zeros((n_atoms + 31) // 32, np.uint32)
    L = N.load()
    ver, nr, rules = C.c_uint32(GUARD), C.c_uint32(GUARD), np.zeros(8, np.uint32)
    ctx = np.array([0, 4], np.uint32)
    bad_off = off.copy()
    bad_off[2] = bad_off[3] + 1
    for args in ((rs.handle, data.ctypes.data, off.ctypes.data, None, 4, atoms.ctypes.data),      # roles missing
                 (rs.handle, data.ctypes.data, off.ctypes.data, roles.ctypes.data, 4, None),      # atoms missing
                 (rs.handle, None, off.ctypes.data, roles.ctypes.data, 4, atoms.ctypes.data),     # bytes missing
                 (rs.handle, data.ctypes.data, bad_off.ctypes.data, roles.ctypes.data, 4, atoms.ctypes.data),   # decreasing offsets
                 (None, data.ctypes.data, off.ctypes.data, roles.ctypes.data, 4, atoms.ctypes.data)):
        a = L.cg_policy_eval_one(*args, C.byref(ver), rules.ctypes.data, 8, C.byref(nr))
        b = L.cg_policy_eval_batch(args[0], args[1], args[2], args[3], 4, ctx.ctypes.data, args[5], 1, np.zeros(1, np.uint32).ctypes.data,
                                   np.zeros(8, N.POLICY_MATCH_DTYPE).ctypes.data, 8, C.byref(C.c_uint32(0)))
        assert a == b == INVALID_ARG and ver.value == GUARD and nr.value == GUARD
    assert L.cg_policy_eval_one(rs.handle, data.ctypes.data, off.ctypes.data, roles.ctypes.data, 4, atoms.ctypes.data, None, None, 0, None) == INVALID_ARG
    fresh = N.Ruleset([("abc", 0, 3)], strict=True)                   # no program set
    assert L.cg_policy_eval_one(fresh.handle, data.ctypes.data, off.ctypes.data, roles.ctypes.data, 4, None, C.byref(ver), None, 0, None) == INVALID_ARG
    fresh.close()


# ------------------------------------------------------------------------------------------ graphs

def test_graphs_per_text_count_and_program(N, seam_case):
    rs, rng, n_atoms = seam_case
    for n in (1, 3, 1, 7, 3, 0, 64, 1, 7, 12, 3, 0, 9, 2, 5, 11, 1):
        data, off, roles = texts_case(N, rng, n)
        atoms = rng.integers(0, 2**32, (n_atoms + 31) // 32, dtype=np.uint64).astype(np.uint32)
        same_as_batch(N, rs, data, off, roles, atoms, 2048)
    r2 = N.Ruleset([("beta", 0, 3), ("alpha\\d", 0, 3)], strict=True)
    data, off = N.pack([b"alpha1 beta", b"beta"])
    roles = np.array([0, 1], np.uint8)
    deny = [1, 0xffffffff, 1, 3 | 4, 1, 2 | 0 << 3 | 0 << 24]              # deny when rule 0 hit the message
    audit = [1, 0xffffffff, 1, 1, 1, 2 | 1 << 3 | 0 << 24]                # audit when rule 1 hit the message
    r2.set_policy_program(deny, 0)
    a = raw_one(N, r2, data, off, roles, np.zeros(0, np.uint32), 8)
    r2.set_policy_program(audit, 0)
    b = raw_one(N, r2, data, off, roles, np.zeros(0, np.uint32), 8)
    assert a[:3] == (N.CG_OK, 4 | 1 << 3 | 0 << 12, 1) and b[:3] == (N.CG_OK, 2 | 1 << 3 | 0xfffff << 12, 1)
    assert b == raw_batch(N, r2, data, off, roles, np.zeros(0, np.uint32), 8)
    r2.close()


# ------------------------------------------------------------------------------------------ protocols

def step_kernels(N, torch, rs, data, off):
    """the kernels of one scan step over these texts (cg_scan_batch_device replays the step alone)"""
    d, o = to_device(torch, data, off)
    words = torch.zeros(len(off), dtype=torch.int64, device="cuda")
    rs.scan_batch_device(d.data_ptr(), o.data_ptr(), len(off) - 1, words.data_ptr())
    rs.scan_batch_device(d.data_ptr(), o.data_ptr(), len(off) - 1, words.data_ptr())
    before = N.launch_count()
    rs.scan_batch_device(d.data_ptr(), o.data_ptr(), len(off) - 1, words.data_ptr())
    rs.scan_join()
    return N.launch_count() - before


def test_queue_overflow_takes_the_batch_call_then_the_fast_path(N, torch):
    """a fresh rule set of 100 rules that share the factor "needle", over 64 texts of 1 KB made of it: 6 400 (text, rule) pairs
    for the VM (4 096 fit the fresh scratch) and far more confirmed occurrences than the 65 536 it holds.  The answer comes
    from the batch call; the next call runs the fast path's graph again."""
    srcs = [("needle\\d{0,2}[a-z]*%d" % i, 0, 3) for i in range(100)]
    rs = N.Ruleset(srcs, strict=True)
    prog = [100]
    for i in range(100):
        prog += [0xffffffff, 1, 3 | 4 if i % 7 == 0 else 1, 1, 2 | i << 3 | 0 << 24]
    rs.set_policy_program(prog, 0)
    texts = [(b"needle%d " % i) * 1024 for i in range(64)]
    texts = [t[:1024] for t in texts]
    data, off = N.pack(texts)
    assert int(off[-1]) == MAX_BYTES
    roles = np.zeros(64, np.uint8)
    atoms = np.zeros(0, np.uint32)
    before = N.launch_count()
    got = raw_one(N, rs, data, off, roles, atoms, 256)
    first = N.launch_count() - before
    c = rs.work_counters()
    assert int(c[3]) == 0 and (int(c[1]) > 4096 or int(c[4]) > 65536)     # the step that answered needed more than a fresh scratch
    want = raw_batch(N, rs, data, off, roles, atoms, 256)
    assert got == want and got[0] == N.CG_OK and got[2] > 10
    k = step_kernels(N, torch, rs, data, off)
    assert first > k + 1                                                     # the fast attempt, then the batch call's launches
    before = N.launch_count()
    assert raw_one(N, rs, data, off, roles, atoms, 256) == want
    assert N.launch_count() - before == k + 1                                # the fast path again
    rs.close()


def test_launches_are_the_step_plus_one_with_and_without_hits(N, torch, seam_case):
    rs, rng, n_atoms = seam_case
    atoms = np.zeros((n_atoms + 31) // 32, np.uint32)
    for n in (1, 5, 64):
        data, off, roles = texts_case(N, rng, n)
        blank = np.zeros_like(data)
        k = step_kernels(N, torch, rs, data, off)
        ds = []
        for dd in (data, blank, data, blank):
            raw_one(N, rs, dd, off, roles, atoms, 64)               # (a new graph is captured on first use: counted from the second call)
            before = N.launch_count()
            raw_one(N, rs, dd, off, roles, atoms, 64)
            ds.append(N.launch_count() - before)
        assert ds == [k + 1] * 4, (n, k, ds)
    data, off = N.pack([])
    raw_one(N, rs, data, off, np.zeros(0, np.uint8), atoms, 64)
    before = N.launch_count()
    raw_one(N, rs, data, off, np.zeros(0, np.uint8), atoms, 64)
    assert N.launch_count() - before == 1                            # no text: the counter block cleared, then the kernel


def test_a_device_call_on_a_held_stream_comes_first(N, torch):
    pe = P.PolicyEvaluator(PP.random_policies(np.random.default_rng(3), max_policies=10) + PP.builtin_policies(), other_condition=PP.other_condition)
    ctxs = PP.random_contexts(np.random.default_rng(4), 500)
    rs = pe._program_ruleset()
    texts, roles, ctx_off, atoms = pe.program_inputs(ctxs)
    data, off = N.pack([N.js_utf8(t) for t in texts])
    words, matches = rs.eval_batch(data, off, roles, ctx_off, atoms)
    d, o = to_device(torch, data, off)
    dr, dc, da = to_dev(torch, roles, ctx_off, atoms)
    verdicts = torch.full((len(ctxs),), GUARD, dtype=torch.int32, device="cuda")
    s1 = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(GATE)
    rs.eval_batch_device(d.data_ptr(), o.data_ptr(), dr.data_ptr(), len(off) - 1, dc.data_ptr(), da.data_ptr(), len(ctxs), verdicts.data_ptr(),
                         stream=s1.cuda_stream)
    t1, r1, c1, a1 = pe.program_inputs(ctxs[:1])
    d1, o1 = N.pack([N.js_utf8(t) for t in t1])
    got = rs.eval_one(d1, o1, r1, a1[0])
    assert s1.query()                                                # the device call had run when the one-call returned
    rs.scan_join(s1.cuda_stream)
    assert np.array_equal(verdicts.cpu().numpy().view(np.uint32), words)
    assert got == (int(words[0]), [int(j) for j in matches["rule"][matches["ctx"] == 0]])
