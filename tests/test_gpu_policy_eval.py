"""GPU tier for policy programs: PolicyEvaluator.verdict_batch (cg_policy_eval_batch) equals evaluate_batch on the
policy-slice cases, the built-ins and random policy sets (also over the 500-rule C2 set with planted hits); the host and
device twins agree; edges of the batch shape and of the stack depth; capacity with guard words; the in-band protocols
(queue overflow, bad context ranges in HBM); issue order across streams; launch counts independent of the hit count."""
import numpy as np
import pytest

import policy_program as PP
from test_gpu_redact_device import to_device
from vainplex_openclaw_b200 import plugin as P
from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu
GUARD = 0x5a5a5a5a


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


@pytest.fixture(scope="module")
def torch():
    import torch as T
    return T


def same(pe, ctxs):
    assert pe.verdict_batch(ctxs) == pe.evaluate_batch(ctxs)


def test_slice_cases(N):
    for policies, ctxs in PP.slice_cases():
        same(P.PolicyEvaluator(policies), ctxs)


def test_builtins_on_tool_calls(N):
    same(P.PolicyEvaluator(PP.builtin_policies(), other_condition=PP.other_condition), PP.tool_contexts(np.random.default_rng(5), 3000))


def test_random_policy_sets(N):
    rng = np.random.default_rng(21)
    for _ in range(150):
        same(P.PolicyEvaluator(PP.random_policies(rng), other_condition=PP.other_condition), PP.random_contexts(rng, 40))


def c2_rules():
    return [r for r in W.make_rules(500) if N_ok(r["source"])]


def N_ok(src):
    from vainplex_openclaw_b200 import _native
    return _native.rule_check(src, 0) == 0


def test_random_sets_over_the_c2_rules(N):
    """random policy sets whose regex tests are drawn from the 500-rule C2 set, contexts with its samples planted"""
    rl = c2_rules()
    pats = [r["source"] for r in rl]
    samples = [r["sample"] for r in rl if r["sample"]]
    rng = np.random.default_rng(31)
    hits = 0
    for _ in range(30):
        pe = P.PolicyEvaluator(PP.random_policies(rng, patterns=list(rng.choice(pats, 40)), max_policies=12), other_condition=PP.other_condition)
        ctxs = PP.random_contexts(rng, 200, samples=samples)
        res = pe.verdict_batch(ctxs)
        assert res == pe.evaluate_batch(ctxs)
        hits += sum(len(r["matches"]) for r in res)
    assert hits > 1000


def program_case(N, n_ctx, seed=3):
    """a rule set, a program over it and a batch of contexts: (pe, ruleset, data, off, roles, ctx_off, atoms)"""
    rng = np.random.default_rng(seed)
    pe = P.PolicyEvaluator(PP.random_policies(rng, max_policies=10) + PP.builtin_policies(), other_condition=PP.other_condition)
    ctxs = PP.random_contexts(rng, n_ctx)
    texts, roles, ctx_off, atoms = pe.program_inputs(ctxs)
    data, off = N.pack([N.js_utf8(t) for t in texts])
    rs = pe.scanner.ruleset
    rs.set_policy_program(pe.program, len(pe.atoms))
    return pe, ctxs, rs, data, off, roles, ctx_off, atoms


class EvalOut:
    """device buffers of one cg_policy_eval_batch_device call, guard words behind every output"""

    def __init__(self, torch, n_ctx, cap, guard=64):
        self.n_ctx, self.cap = n_ctx, cap
        self.verdicts = torch.full((n_ctx + guard,), GUARD, dtype=torch.int32, device="cuda")
        self.matches = torch.full(((cap + guard) * 2,), GUARD, dtype=torch.int32, device="cuda")
        self.count = torch.full((guard,), GUARD, dtype=torch.int32, device="cuda")

    def issue(self, rs, d, o, dr, n_texts, dc, da, stream=0, matches=True):
        rs.eval_batch_device(d.data_ptr(), o.data_ptr(), dr.data_ptr(), n_texts, dc.data_ptr(), da.data_ptr(), self.n_ctx, self.verdicts.data_ptr(),
                             self.matches.data_ptr() if matches else 0, self.cap if matches else 0, self.count.data_ptr() if matches else 0, stream)

    def result(self):
        v = self.verdicts.cpu().numpy().view(np.uint32)
        m = self.matches.cpu().numpy().view(np.uint32)
        c = self.count.cpu().numpy().view(np.uint32)
        nm = int(c[0])
        k = min(nm, self.cap)
        pairs = m[:2 * k].reshape(-1, 2)
        assert (v[self.n_ctx:] == GUARD).all() and (m[2 * self.cap:] == GUARD).all() and (c[1:] == GUARD).all()
        return v[:self.n_ctx], nm, [tuple(int(x) for x in p) for p in pairs]


def to_dev(torch, roles, ctx_off, atoms):
    dr = torch.from_numpy(np.concatenate([np.asarray(roles, np.uint8), np.zeros(4, np.uint8)])).cuda()
    dc = torch.from_numpy(np.asarray(ctx_off, np.uint32).view(np.int32).copy()).cuda()
    da = torch.from_numpy(np.concatenate([np.asarray(atoms, np.uint32).reshape(-1), np.zeros(1, np.uint32)]).view(np.int32)).cuda()
    return dr, dc, da


@pytest.mark.parametrize("n_ctx", [0, 1, 31, 32, 33, 4097])
def test_host_twin_equals_device_twin(N, torch, n_ctx):
    pe, ctxs, rs, data, off, roles, ctx_off, atoms = program_case(N, n_ctx)
    words, matches = rs.eval_batch(data, off, roles, ctx_off, atoms)
    assert pe.decode_verdicts(words, matches) == pe.evaluate_batch(ctxs)
    d, o = to_device(torch, data, off)
    dr, dc, da = to_dev(torch, roles, ctx_off, atoms)
    out = EvalOut(torch, n_ctx, max(len(matches), 1))
    out.issue(rs, d, o, dr, len(off) - 1, dc, da)
    rs.scan_join()
    v, nm, pairs = out.result()
    assert np.array_equal(v, words) and nm == len(matches) and pairs == [tuple(x) for x in matches.tolist()]
    w2, m2 = rs.eval_batch(data, off, roles, ctx_off, atoms, want_matches=False)
    assert np.array_equal(w2, words) and len(m2) == 0


def test_contexts_without_texts_and_many_entries(N):
    """contexts with no text, an empty message, more conversation entries than a warp keeps in shared memory; a batch with
    no text at all"""
    pols = [{"id": "c", "rules": [{"id": "r", "conditions": [{"type": "context", "conversationContains": "needle-\\d+"}], "effect": {"action": "deny", "reason": "n"}}]},
            {"id": "m", "rules": [{"id": "r", "conditions": [{"type": "context", "messageContains": "x"}], "effect": {"action": "audit"}}]},
            {"id": "t", "rules": [{"id": "r", "conditions": [{"type": "tool", "name": "exec"}], "effect": {"action": "2fa", "reason": "t"}}]}]
    pe = P.PolicyEvaluator(pols)
    ctxs = []
    for i in range(300):
        k = i % 5
        conv = ["filler %d" % j for j in range(33 if k == 1 else 100 if k == 2 else 0)]
        if k in (1, 2) and i % 2:
            conv[-1] = "needle-%d" % i
        ctxs.append({"agentId": "a", "toolName": "exec" if k == 3 else None, "messageContent": "" if k == 0 else "x y" if k == 4 else "",
                     "conversationContext": conv})
    same(pe, ctxs)
    res = pe.verdict_batch(ctxs)
    assert sum(r["action"] == "deny" for r in res) > 50
    no_text = [{"agentId": "a", "toolName": "exec" if i % 2 else "read"} for i in range(70)]
    texts, _r, _c, _a = pe.program_inputs(no_text)
    assert texts == []
    same(pe, no_text)


def test_stack_depth_32_and_deeper(N):
    rs = N.Ruleset([("abc", 0, 3)], strict=True)

    def prog(depth):
        ops = [N.POL_CONST | 1 << 3] * depth + [N.POL_AND] * (depth - 1)
        return [1, 0xffffffff, 1, 3 | 4, len(ops)] + ops
    rs.set_policy_program(prog(32), 0)
    data, off = N.pack([b"zzabczz"])
    w, m = rs.eval_batch(data, off, [0], [0, 1, 1], np.zeros((2, 0), np.uint32))
    assert (w == np.uint32(4 | 1 << 3 | 0 << 12)).all() and m.tolist() == [(0, 0), (1, 0)]
    with pytest.raises(N.GovError) as ei:
        rs.set_policy_program(prog(33), 0)
    assert ei.value.code == N.CG_ERR_TOO_LARGE
    for bad in ([1, 0xffffffff, 1, 3, 2, N.POL_CONST, N.POL_CONST],          # leaves two values
                [1, 0xffffffff, 1, 3, 1, N.POL_AND],                          # underflow
                [1, 0xffffffff, 1, 3, 1, N.POL_HIT | 1 << 3],                 # rule past the set
                [1, 0xffffffff, 1, 3, 1, N.POL_ATOM],                         # atom past n_atoms
                [1, 0, 0], [1, 0xffffffff, 1, 8, 1, N.POL_CONST], [2, 0xffffffff, 0]):
        with pytest.raises(N.GovError) as ei:
            rs.set_policy_program(bad, 0)
        assert ei.value.code == -1, bad                        # CG_ERR_INVALID_ARG
    rs.close()


def test_capacity_first_matches_and_guard(N, torch):
    pe, ctxs, rs, data, off, roles, ctx_off, atoms = program_case(N, 500, seed=9)
    words, matches = rs.eval_batch(data, off, roles, ctx_off, atoms)
    assert len(matches) > 100
    d, o = to_device(torch, data, off)
    dr, dc, da = to_dev(torch, roles, ctx_off, atoms)
    for cap in (0, 1, 37, len(matches) - 1):
        out = EvalOut(torch, 500, cap)
        out.issue(rs, d, o, dr, len(off) - 1, dc, da)
        with pytest.raises(N.GovError) as ei:
            rs.scan_join()
        assert ei.value.code == N.CG_ERR_CAPACITY
        v, nm, pairs = out.result()
        assert np.array_equal(v, words) and nm == len(matches) and pairs == [tuple(x) for x in matches.tolist()[:cap]]
    import ctypes as C
    ver = np.zeros(500, np.uint32)
    small = np.zeros(40, N.POLICY_MATCH_DTYPE)
    nm = C.c_uint32(0)
    rc = N.load().cg_policy_eval_batch(rs.handle, data.ctypes.data, off.ctypes.data, roles.ctypes.data, len(off) - 1, ctx_off.ctypes.data,
                                       atoms.ctypes.data, 500, ver.ctypes.data, small.ctypes.data, 37, C.byref(nm))
    assert rc == N.CG_ERR_CAPACITY and nm.value == len(matches) and small[:37].tolist() == matches.tolist()[:37] and (small[37:]["ctx"] == 0).all()


def test_queue_overflow_and_bad_ranges_in_band(N, torch):
    """a fresh rule set sized by a small batch, then 30 000 texts that all hit: every verdict and the count are 0xffffffff,
    no match is written, the join raises CG_ERR_CAPACITY once; issued again the results are the host's.  Context ranges that
    are decreasing or run past n_texts get 0xfffffffe, the others are unaffected."""
    rl = W.make_rules(64)
    srcs = [r["source"] for r in rl if N_ok(r["source"])]
    pols = [{"id": "p%d" % i, "rules": [{"id": "r", "conditions": [{"type": "context", "messageContains": s}], "effect": {"action": "deny", "reason": s}}]}
            for i, s in enumerate(srcs)]
    pe = P.PolicyEvaluator(pols)
    rs = pe.scanner.ruleset
    rs.set_policy_program(pe.program, len(pe.atoms))
    d1_t, o1_t, _ = W.make_messages(30000, 256, rl, p_hit=1.0, seed=4)
    data, off = d1_t.numpy(), o1_t.numpy().astype(np.uint32)
    n = 30000
    n_ctx = n // 2
    ctx_off = np.arange(0, n + 1, 2, dtype=np.uint32)
    roles = np.zeros(n, np.uint8)
    atoms = np.zeros((n_ctx, 0), np.uint32)
    d, o = to_device(torch, data, off)
    dr, dc, da = to_dev(torch, roles, ctx_off, atoms)
    st = torch.cuda.Stream()
    out = EvalOut(torch, n_ctx, 8 * n)
    out.issue(rs, d, o, dr, n, dc, da, st.cuda_stream)
    with pytest.raises(N.GovError) as ei:
        rs.scan_join(st.cuda_stream)
    assert ei.value.code == N.CG_ERR_CAPACITY
    v, nm, _pairs = out.result()
    assert (v == 0xffffffff).all() and nm == 0xffffffff and (out.matches.cpu().numpy().view(np.uint32) == GUARD).all()
    for attempt in range(4):
        out.issue(rs, d, o, dr, n, dc, da, st.cuda_stream)
        try:
            rs.scan_join(st.cuda_stream)
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
    words, matches = rs.eval_batch(data, off, roles, ctx_off, atoms)
    v, nm, pairs = out.result()
    assert np.array_equal(v, words) and nm == len(matches) and pairs == [tuple(x) for x in matches.tolist()]
    assert int(((words & 7) == 4).sum()) > n_ctx * 0.9
    bad = ctx_off.copy()
    bad[10], bad[20], bad[n_ctx] = bad[11] + 1, n + 5, n + 1          # context 10 decreasing, 19 / 20 past n_texts, the last past n_texts
    dc2 = torch.from_numpy(bad.view(np.int32).copy()).cuda()
    out2 = EvalOut(torch, n_ctx, 8 * n)
    out2.issue(rs, d, o, dr, n, dc2, da, st.cuda_stream)
    rs.scan_join(st.cuda_stream)                                      # (a bad range is reported in its verdict, not by the join)
    v2, nm2, pairs2 = out2.result()
    badc = {10, 19, 20, n_ctx - 1}
    assert all(v2[c] == 0xfffffffe for c in badc)
    keep = [c for c in range(n_ctx) if c not in badc and c != 9]
    assert np.array_equal(v2[keep], words[keep])
    rs.close()


def test_two_streams_run_in_issue_order(N, torch):
    pe, ctxs, rs, data, off, roles, ctx_off, atoms = program_case(N, 2000, seed=12)
    words, matches = rs.eval_batch(data, off, roles, ctx_off, atoms)
    d, o = to_device(torch, data, off)
    dr, dc, da = to_dev(torch, roles, ctx_off, atoms)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [EvalOut(torch, 2000, len(matches) + 1) for _ in range(6)]
    for i, out in enumerate(outs):
        out.issue(rs, d, o, dr, len(off) - 1, dc, da, (s1 if i % 2 else s2).cuda_stream)
    rs.scan_join(s1.cuda_stream)
    rs.scan_join(s2.cuda_stream)
    for out in outs:
        v, nm, pairs = out.result()
        assert np.array_equal(v, words) and nm == len(matches) and pairs == [tuple(x) for x in matches.tolist()]


def test_launch_count_and_stats_do_not_depend_on_hits(N, torch):
    """the same batch shape with no hit and with many: equal kernel launches and cg_stats deltas (but the hit counts)"""
    pe, ctxs, rs, data, off, roles, ctx_off, atoms = program_case(N, 1000, seed=14)
    d, o = to_device(torch, data, off)
    dr, dc, da = to_dev(torch, roles, ctx_off, atoms)
    blank = np.zeros_like(data)
    db, ob = to_device(torch, blank, off)
    deltas = []
    for dd, matches in ((db, True), (d, True), (db, False), (d, False)):
        out = EvalOut(torch, 1000, 100000)
        before = N.stats()
        out.issue(rs, dd, o, dr, len(off) - 1, dc, da, 0, matches)
        rs.scan_join()
        after = N.stats()
        deltas.append((after.kernel_launches - before.kernel_launches, after.messages_scanned - before.messages_scanned))
    assert deltas[0] == deltas[1] and deltas[2] == deltas[3] and deltas[0][0] >= deltas[2][0] + 3
