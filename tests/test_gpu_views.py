"""Per-message views of one rule set (cg_ruleset_set_views and the *_views twins of the batch calls): every message is
decided on the rules of its own view as if that view were a rule set of its own -- result words, hit lists, resolved spans,
redacted bytes, digests and verdicts -- against a per-view oracle, against the calls without views on rule sets compiled
from each view's rules, and, for the full view, against the calls without views including launches and statistics.
Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

from helpers import oracle_regexes
from members import build_case
from test_gpu_parity import CATS
from test_gpu_redact_device import GUARD as BYTE_GUARD, FindOut, RedactOut, full, ragged, splice_python, to_device
from test_gpu_scan_hits_device import ALL_ONES, GUARD, HitsOut
from test_gpu_scan_launches import LONG_RULES, STAT_FIELDS, measure, stats
from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu
# the long-program rules plus two rules without a factor (every message is their candidate): verify_large_kernel, and the
# always-candidate loop of resolve_kernel
ALWAYS_LONG_RULES = LONG_RULES + [(r"\d+", 0, 3), (r"x\b", 0, 3), (r"[a-z]\d", 0, 1)]


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


@pytest.fixture(scope="module")
def torch():
    import torch as T
    return T


# ------------------------------------------------------------------------------ the expectation

def view_sets(rules, seed):
    """the empty view, the full view, three singletons, a random half and its complement, the credential rules"""
    R = len(rules)
    rng = np.random.default_rng(seed)
    half = sorted(int(x) for x in rng.choice(R, R // 2, replace=False))
    comp = sorted(set(range(R)) - set(half))
    singles = sorted({0, R - 1, int(rng.integers(R))})
    cred = [i for i, r in enumerate(rules) if r[2] == 0]
    return [[], list(range(R))] + [[s] for s in singles] + [half, comp, cred]


class ViewOracle:
    """The oracle on a rule set made of one view's rules alone, rule indices mapped back to the whole set's: result words,
    (msg, rule) hits sorted, resolved spans (msg, rule, start16, end16) in findMatches order."""

    def __init__(self, O, rules):
        self.O, self.rules = O, rules
        self.regs = oracle_regexes(O, rules)
        assert all(r is not None for r in self.regs)

    def of(self, msgs, ids, views):
        n = len(msgs)
        words = np.zeros(n, dtype=np.uint64)
        hits, spans = [], [[] for _ in range(n)]
        for v, idx in enumerate(views):
            mi = [i for i in range(n) if int(ids[i]) == v]
            if not idx or not mi:
                continue
            regs = [self.regs[r] for r in idx]
            data, off = self.O.pack([msgs[i] for i in mi])
            bits, w = self.O.scan_policy(regs, data, off)
            for j, i in enumerate(mi):
                x = int(w[j])
                if x >> 63:
                    words[i] = (1 << 63) | (x & (0x7fffffff << 32)) | idx[x & 0xffffffff]
                hits += [(i, idx[int(k)]) for k in np.nonzero(np.unpackbits(bits[j], bitorder="little")[:len(idx)])[0]]
            pats = [(regs[k], CATS[self.rules[r][2]]) for k, r in enumerate(idx)]
            for m, r, s, e in self.O.find_matches_batch(pats, data, off).tolist():
                spans[mi[m]].append((mi[m], idx[r], s, e))
        return words, sorted(hits), [s for per in spans for s in per]


def verdicts_of(hits, n, pol, act):
    """aggregateMatches restated over a hit list (policy-evaluator.ts:110-146, as verdict_kernel computes it)"""
    out = np.zeros(n, dtype=np.uint32)
    by = {}
    for m, r in hits:
        by.setdefault(m, []).append(r)
    for m, rl in by.items():
        prev, best, decide, matched = None, 0, 0xfffff, 0
        for r in sorted(rl):
            if pol[r] == prev:
                continue
            prev = pol[r]
            matched += 1
            if act[r] == 2 and best != 2:
                best, decide = 2, r
            elif act[r] == 1 and best == 0:
                best, decide = 1, r
        out[m] = best | (min(matched, 1023) << 2) | (decide << 12)
    return out


def random_policy(rules, seed):
    rng = np.random.default_rng(seed)
    return np.sort(rng.integers(0, max(2, len(rules) // 4), len(rules))).astype(np.uint32), rng.integers(0, 3, len(rules)).astype(np.uint8)


# ------------------------------------------------------------------------------ every twin on one batch

def joined(N, rs, issue, check_incomplete=None):
    """issue a device call and join; issued again while an internal queue overflows"""
    for attempt in range(4):
        issue()
        try:
            rs.scan_join()
            return
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
            if check_incomplete:
                check_incomplete()


def redact_views(ro, rs, d, o, dv, stream=0):
    """RedactOut's call through cg_redact_batch_device_views"""
    rs.redact_batch_device(d.data_ptr(), o.data_ptr(), ro.n, ro.out.data_ptr(), ro.out_cap, ro.off.data_ptr(), ro.spans.data_ptr(),
                           ro.spans_cap, ro.dig.data_ptr(), ro.sizes.data_ptr(), stream, views=dv.data_ptr())


def twins(N, torch, rs, msgs, ids, host=True):
    """every *_views twin on one batch (host=False: the device-resident ones only) -> dict of results (the device ones
    checked for guard bytes / words)"""
    data, off = N.pack(msgs)
    n = len(msgs)
    ids = np.asarray(ids, dtype=np.uint8)
    r = {}
    if host:
        words, hits = rs.scan_batch(data, off, views=ids)
        r["words"], r["hits"] = words, [(int(h["msg"]), int(h["rule"])) for h in hits]
        r["spans"] = full(rs.find_matches_batch(data, off, views=ids))
        out, out_off, sp, dig = rs.redact_batch(data, off, views=ids)
        r["redact"] = (bytes(out), out_off.tolist(), full(sp), dig.tobytes())
        r["verdicts"] = rs.verdict_batch(data, off, views=ids)

    d, o = to_device(torch, data, off)
    dv = torch.from_numpy(np.concatenate([ids, np.zeros(16, np.uint8)])).cuda()
    ho = HitsOut(torch, n, max(1024, 4 * n))
    joined(N, rs, lambda: rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr(), n, ho.words.data_ptr(), ho.hits.data_ptr(), ho.cap,
                                                     ho.nhits.data_ptr(), views=dv.data_ptr()))
    nh, pairs, guard, dwords = ho.result()
    assert (guard == GUARD).all() and nh == len(pairs)
    r["d_words"], r["d_hits"] = dwords, pairs
    wo = torch.full((max(n, 1),), -1, dtype=torch.int64, device="cuda")
    joined(N, rs, lambda: rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr(), n, wo.data_ptr(), 0, 0, 0, views=dv.data_ptr()))
    r["d_words_only"] = wo.cpu().numpy().view(np.uint64)[:n]
    fo = FindOut(torch, max(1024, 8 * n))
    joined(N, rs, lambda: rs.find_matches_batch_device(d.data_ptr(), o.data_ptr(), n, fo.spans.data_ptr(), fo.cap, fo.nspans.data_ptr(),
                                                        views=dv.data_ptr()))
    ns, dspans, guard = fo.result(N)
    assert (guard == GUARD).all() and ns == len(dspans)
    r["d_spans"] = full(dspans)
    total = int(off[n]) - int(off[0]) if n else 0
    ro = RedactOut(torch, n, 8 * total + 65536, max(1024, 8 * n))
    joined(N, rs, lambda: redact_views(ro, rs, d, o, dv))
    dout, doff, dsp, ddig, g1, g2, g3 = ro.result(N)
    assert (g1 == BYTE_GUARD).all() and (g2 == GUARD).all() and (g3 == BYTE_GUARD).all()
    r["d_redact"] = (bytes(dout), doff.tolist(), full(dsp), ddig.tobytes())
    vo = torch.full((n + 16,), GUARD, dtype=torch.int32, device="cuda")
    joined(N, rs, lambda: rs.verdict_batch_device(d.data_ptr(), o.data_ptr(), n, vo.data_ptr(), views=dv.data_ptr()))
    got = vo.cpu().numpy().view(np.uint32)
    assert (got[n:] == GUARD).all()
    r["d_verdicts"] = got[:n]
    return r


def check_against(r, msgs, rules, words, hits, spans, verdicts):
    """every twin's results equal the expectation; the redaction is applyReplacements of the expected spans"""
    n = len(msgs)
    for k in ("words", "d_words", "d_words_only"):
        assert np.array_equal(r[k], words), k
    assert r["hits"] == hits and r["d_hits"] == hits
    assert [s[:2] + s[4:] for s in r["spans"]] == spans
    assert r["d_spans"] == r["spans"]
    out, out_off, rsp, dig = r["redact"]
    assert rsp == r["spans"] and r["d_redact"] == r["redact"]
    sp = np.array(rsp, dtype=np.uint32).reshape(-1, 6).copy().view(
        np.dtype([(f, np.uint32) for f in ("msg", "rule", "start_byte", "end_byte", "start16", "end16")])).reshape(-1)
    want = splice_python(msgs, rules, sp, np.frombuffer(dig, np.uint8).reshape(-1, 32))
    assert [out[out_off[i]:out_off[i + 1]] for i in range(n)] == want
    assert np.array_equal(r["verdicts"], verdicts) and np.array_equal(r["d_verdicts"], verdicts)


# ------------------------------------------------------------------------------ 1. subset equivalence against the oracle

CASES = ["builtins", "syn500-s2", "syn5000", "non-ascii", "always-long"]


def case_batch(N, name):
    """(rules, options, messages) of a case: the member batch of tests/members.py (every rule's members planted), or for
    the always-candidate / long-program set a ragged batch with hits of the long rules"""
    if name == "always-long":
        data_t, off_t, _ = W.make_messages(3000, 256, W.make_rules(17), p_hit=0.2, utf8_frac=0.1, seed=91)
        msgs = ragged(data_t, off_t, seed=92, max_len=256)
        for i in range(0, len(msgs), 37):
            msgs[i] = (b"x tok_" + b"0a" * 100 + b"z 12", b"sk-" + b"a1B2" * 6 + b" x", b"ab" * 70 + b"! q7", b"KEY=" + b"Q" * 100 + b"7" * 100)[(i // 37) % 4]
        return ALWAYS_LONG_RULES, N.OPT_STRIDE_AUTO, msgs
    case = build_case(name)
    options = {"syn500-s2": N.OPT_STRIDE2}.get(name, N.OPT_STRIDE_AUTO)
    return case.rules, options, case.members.msgs


@pytest.mark.parametrize("name", CASES)
def test_views_equal_the_oracle_on_each_views_rules(N, torch, oracle, name):
    """Random view ids per message over the empty view, the full view, singletons, a random half and its complement and
    the credential rules: words, hit lists (guard words behind them), spans, redacted bytes, offsets, digests and verdicts
    of every host-buffer and device-resident twin equal the oracle run on each view's rules alone."""
    rules, options, msgs = case_batch(N, name)
    rs = N.Ruleset(rules, options=options, strict=True)
    info = rs.info()
    if name == "syn5000":
        assert info.n_rules == 5000
    if name in ("non-ascii", "always-long"):
        assert info.n_always_candidate > 0
    views = view_sets(rules, seed=len(rules))
    rs.set_views(views)
    pol, act = random_policy(rules, seed=len(rules) + 1)
    rs.set_policy(pol, act)
    ids = np.random.default_rng(len(msgs)).integers(0, len(views), len(msgs)).astype(np.uint8)
    words, hits, spans = ViewOracle(oracle, rules).of(msgs, ids, views)
    r = twins(N, torch, rs, msgs, ids)
    check_against(r, msgs, rules, words, hits, spans, verdicts_of(hits, len(msgs), pol, act))
    # strength: every non-empty view has hits, and the full view's messages hit rules outside every other view
    hit_views = {int(ids[m]) for m, _ in hits}
    assert hit_views >= {v for v, idx in enumerate(views) if len(idx) > 1}, hit_views
    assert all(ids[m] != 0 for m, _ in hits) and all(ids[m] != 0 for m, *_ in spans)
    print("%s: %d rules, %d messages, %d hits, %d spans, %d views" % (name, len(rules), len(msgs), len(hits), len(spans), len(views)))
    rs.close()


# ------------------------------------------------------------------------------ 2. GPU against GPU

@pytest.mark.parametrize("name", ["builtins", "syn500"])
def test_each_view_equals_a_rule_set_of_its_rules(N, torch, name):
    """Each view's messages through the twins == the same messages through the calls without views on a rule set compiled
    from the view's rules (indices mapped back, the policy assignment restricted to them)."""
    rl = W.make_rules(17 if name == "builtins" else 500)
    rules = W.rules_as_tuples(rl)
    data_t, off_t, _ = W.make_messages(6000, 256, rl, p_hit=0.15, utf8_frac=0.1, seed=606)
    msgs = ragged(data_t, off_t, seed=607, max_len=256)
    rs = N.Ruleset(rules, strict=True)
    views = view_sets(rules, seed=608)
    rs.set_views(views)
    pol, act = random_policy(rules, seed=609)
    rs.set_policy(pol, act)
    ids = np.random.default_rng(610).integers(0, len(views), len(msgs)).astype(np.uint8)
    r = twins(N, torch, rs, msgs, ids)
    for v, idx in enumerate(views):
        mi = [i for i in range(len(msgs)) if ids[i] == v]
        sub_msgs = [msgs[i] for i in mi]
        sel = set(mi)
        if not idx:
            assert all(int(r["words"][i]) == 0 and r["verdicts"][i] == 0 for i in mi)
            assert not [h for h in r["hits"] if h[0] in sel] and not [s for s in r["spans"] if s[0] in sel]
            out, out_off, _, _ = r["redact"]
            assert all(out[out_off[i]:out_off[i + 1]] == msgs[i] for i in mi)
            continue
        sub = N.Ruleset([rules[i] for i in idx], strict=True)
        sub.set_policy(pol[idx], act[idx])
        data, off = N.pack(sub_msgs)
        sw, sh = sub.scan_batch(data, off)
        back = lambda w: 0 if not w >> 63 else (w & ~0xffffffff) | idx[w & 0xffffffff]
        assert [int(r["words"][i]) for i in mi] == [back(int(w)) for w in sw]
        assert [h for h in r["hits"] if h[0] in sel] == [(mi[int(h["msg"])], idx[int(h["rule"])]) for h in sh]
        remap = lambda s: (mi[s[0]], idx[s[1]]) + tuple(s[2:])
        assert [s for s in r["spans"] if s[0] in sel] == [remap(s) for s in full(sub.find_matches_batch(data, off))]
        out, out_off, sp, dig = sub.redact_batch(data, off)
        rout, roff, rsp, rdig = r["redact"]
        assert [rout[roff[i]:roff[i + 1]] for i in mi] == [bytes(out[out_off[j]:out_off[j + 1]]) for j in range(len(mi))]
        keep = [k for k, s in enumerate(rsp) if s[0] in sel]
        assert [rsp[k] for k in keep] == [remap(s) for s in full(sp)]
        assert b"".join(rdig[32 * k:32 * k + 32] for k in keep) == dig.tobytes()
        sv = sub.verdict_batch(data, off)
        vback = lambda x: x if x == 0 or (x >> 12) == 0xfffff else (x & 0xfff) | (idx[x >> 12] << 12)
        assert [int(r["verdicts"][i]) for i in mi] == [vback(int(x)) for x in sv]
        sub.close()
    rs.close()


def test_full_view_equals_the_calls_without_views(N, torch):
    """The full view: every twin's results, kernel launches and cg_stats delta equal those of the call without views."""
    rl = W.make_rules(500)
    rules = W.rules_as_tuples(rl)
    data_t, off_t, _ = W.make_messages(4000, 256, rl, p_hit=0.1, seed=620)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    n = 4000
    rs = N.Ruleset(rules, strict=True)
    rs.set_views([range(len(rules))])
    rs.set_policy(*random_policy(rules, 621))
    ids = np.zeros(n, np.uint8)
    host = [("scan", lambda v: rs.scan_batch(data, off, views=v)), ("find", lambda v: rs.find_matches_batch(data, off, views=v)),
            ("redact", lambda v: rs.redact_batch(data, off, views=v)), ("verdicts", lambda v: rs.verdict_batch(data, off, views=v))]
    for what, call in host:
        call(None)
        a = measure(N, lambda: call(None))
        b = measure(N, lambda: call(ids))
        assert a[0] == b[0] and a[1] == b[1], (what, a[:2], b[:2])
        ra, rb = (a[2] if isinstance(a[2], tuple) else (a[2],)), (b[2] if isinstance(b[2], tuple) else (b[2],))
        assert all(np.array_equal(x, y) for x, y in zip(ra, rb)), what
    d, o = to_device(torch, data, off)
    dv = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    ho = [HitsOut(torch, n, 4 * n) for _ in range(2)]
    fo = [FindOut(torch, 8 * n) for _ in range(2)]
    ro = [RedactOut(torch, n, 8 * int(off[n]) + 65536, 8 * n) for _ in range(2)]
    vo = [torch.zeros(n, dtype=torch.int32, device="cuda") for _ in range(2)]
    wo = [torch.zeros(n, dtype=torch.int64, device="cuda") for _ in range(2)]
    pv = dv.data_ptr()
    dev = [("hits", lambda k, v: rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr(), n, ho[k].words.data_ptr(), ho[k].hits.data_ptr(), ho[k].cap,
                                                             ho[k].nhits.data_ptr(), views=v), lambda k: ho[k].result()[:2]),
           ("find", lambda k, v: rs.find_matches_batch_device(d.data_ptr(), o.data_ptr(), n, fo[k].spans.data_ptr(), fo[k].cap, fo[k].nspans.data_ptr(),
                                                              views=v), lambda k: full(fo[k].result(N)[1])),
           ("redact", lambda k, v: ro[k].issue(rs, d, o) if v is None else redact_views(ro[k], rs, d, o, dv),
            lambda k: tuple(x.tobytes() for x in ro[k].result(N)[:4])),
           ("verdicts", lambda k, v: rs.verdict_batch_device(d.data_ptr(), o.data_ptr(), n, vo[k].data_ptr(), views=v),
            lambda k: vo[k].cpu().numpy().tobytes())]
    for what, call, res in dev:
        got = []
        for k, v in ((0, None), (1, pv)):
            call(k, v)
            rs.scan_join()
            torch.cuda.synchronize()
            s0 = stats(N)
            kl, dq, _ = measure(N, lambda: call(k, v))
            rs.scan_join()
            torch.cuda.synchronize()
            s1 = stats(N)
            got.append((kl, dq, {f: s1[f] - s0[f] for f in STAT_FIELDS}, res(k)))
        assert got[0][:3] == got[1][:3], (what, got[0][:3], got[1][:3])
        assert got[0][3] == got[1][3], what
    # the words-only twin: cg_scan_batch_device's words and step launches (its original replays them from a graph)
    rs.scan_batch_device(d.data_ptr(), o.data_ptr(), n, wo[0].data_ptr())
    rs.scan_join()
    kl, _, _ = measure(N, lambda: rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr(), n, wo[1].data_ptr(), 0, 0, 0, views=pv))
    rs.scan_join()
    assert kl == 6 and torch.equal(wo[0], wo[1])
    rs.close()


# ------------------------------------------------------------------------------ 3. overlap displacement

DISPLACE_RULES = [(r"sk-[a-zA-Z0-9]{20,}", 0, 0), (r"sk-[a-zA-Z0-9_-]{20,}", 0, 0),
                  (r"[a-zA-Z0-9._%+-]+@[a-zA-Z0-9.-]+\.[a-zA-Z]{2,}", 0, 2), (r"mail me at [a-z]+", 0, 3)]


def test_out_of_view_rules_displace_no_span(N, torch, oracle):
    """sk-[a-zA-Z0-9]{20,} loses its span to the longer sk-[a-zA-Z0-9_-]{20,} match, and an e-mail address to an earlier
    custom match, when all rules run; in a view without the winner the loser's span is kept and spliced."""
    key, mail = b"sk-ABCDEFGHIJKLMNOPQRSTUVWX", b"someone@example.com"
    msgs = [b"x " + key + b"_yz-123 y", b"mail me at " + mail + b" ok", b"both " + key + b"_q-9 and mail me at " + mail]
    rs = N.Ruleset(DISPLACE_RULES, strict=True)
    views = [[0, 1, 2, 3], [0, 2], [0], [2]]
    rs.set_views(views)
    rs.set_policy(np.arange(4), np.full(4, 2))
    full_spans = [s[:2] for s in full(rs.find_matches_batch(*N.pack(msgs)))]
    assert (0, 0) not in full_spans and (0, 1) in full_spans and (1, 2) not in full_spans and (1, 3) in full_spans
    ids = np.array([[v] * 3 for v in range(4)], np.uint8).reshape(-1)
    batch = msgs * 4
    words, hits, spans = ViewOracle(oracle, DISPLACE_RULES).of(batch, ids, views)
    r = twins(N, torch, rs, batch, ids)
    check_against(r, batch, DISPLACE_RULES, words, hits, spans, verdicts_of(hits, len(batch), np.arange(4), np.full(4, 2)))
    got = {(s[0], s[1]) for s in r["spans"]}
    assert {(3, 0), (5, 0), (4, 2), (5, 2), (6, 0), (8, 0), (10, 2), (11, 2)} <= got
    out, out_off, _, _ = r["redact"]
    for m in (3, 5, 6, 8):
        assert key not in out[out_off[m]:out_off[m + 1]] and b"[REDACTED:credential:" in out[out_off[m]:out_off[m + 1]]
    for m in (4, 5, 10, 11):
        assert mail not in out[out_off[m]:out_off[m + 1]] and b"[REDACTED:pii:" in out[out_off[m]:out_off[m + 1]]
    rs.close()


# ------------------------------------------------------------------------------ 4. arguments and errors

def test_arguments_and_errors(N, torch):
    L = N.load()
    rules = W.rules_as_tuples(W.make_rules(17))
    rs = N.Ruleset(rules, strict=True)
    rs.set_policy(np.arange(17), np.full(17, 1))
    msgs = [b"x " + r["sample"].encode() for r in W.make_rules(17)]
    data, off = N.pack(msgs)
    n = len(msgs)
    ids = np.zeros(n, np.uint8)
    SENT = 0x77

    def host_calls(views):
        words = np.full(n, SENT, np.uint64); hits = np.full(64, SENT, np.uint64); nh = C.c_uint32(SENT)
        spans = np.full(64 * 6, SENT, np.uint32); ns = C.c_uint32(SENT)
        out = np.full(8192, SENT, np.uint8); need = C.c_uint64(SENT); ooff = np.full(n + 1, SENT, np.uint32); dig = np.full(64 * 32, SENT, np.uint8)
        verd = np.full(n, SENT, np.uint32)
        p = views.ctypes.data
        rcs = [L.cg_scan_batch_views(rs.handle, data.ctypes.data, off.ctypes.data, p, n, words.ctypes.data, hits.ctypes.data, 32, C.byref(nh)),
               L.cg_find_matches_batch_views(rs.handle, data.ctypes.data, off.ctypes.data, p, n, spans.ctypes.data, 64, C.byref(ns)),
               L.cg_redact_batch_views(rs.handle, data.ctypes.data, off.ctypes.data, p, n, out.ctypes.data, 8000, C.byref(need), ooff.ctypes.data,
                                       spans.ctypes.data, 64, C.byref(ns), dig.ctypes.data),
               L.cg_policy_verdict_batch_views(rs.handle, data.ctypes.data, off.ctypes.data, p, n, verd.ctypes.data)]
        untouched = ((words == SENT).all() and (hits == SENT).all() and nh.value == SENT and (spans == SENT).all() and ns.value == SENT
                     and (out == SENT).all() and need.value == SENT and (ooff == SENT).all() and (dig == SENT).all() and (verd == SENT).all())
        return rcs, untouched

    # before set_views: host and device twins are rejected, nothing written
    rcs, untouched = host_calls(ids)
    assert rcs == [-1] * 4 and untouched
    d, o = to_device(torch, data, off)
    dv = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    vo = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    with pytest.raises(N.GovError) as ei:
        rs.verdict_batch_device(d.data_ptr(), o.data_ptr(), n, vo.data_ptr(), views=dv.data_ptr())
    assert ei.value.code == -1
    # set_views: bits past n_rules, n_views 0 and 257
    rows = np.zeros((257, 1), np.uint32)
    assert L.cg_ruleset_set_views(rs.handle, rows.ctypes.data, 0) == -1
    assert L.cg_ruleset_set_views(rs.handle, rows.ctypes.data, 257) == -1
    bad = np.array([[1 << 17]], np.uint32)
    assert L.cg_ruleset_set_views(rs.handle, bad.ctypes.data, 1) == -1
    assert L.cg_ruleset_set_views(rs.handle, rows.ctypes.data, 256) == 0
    # the Python binding checks what the C call cannot: the rows' width and the number of ids
    for wide in (np.zeros((1, 2), np.uint32), np.zeros((2, 0), np.uint32)):
        with pytest.raises(ValueError):
            rs.set_views(wide)
    with pytest.raises(ValueError):
        rs.scan_batch(data, off, views=np.zeros(n - 1, np.uint8))
    with pytest.raises(ValueError):
        rs.redact_batch(data, off, views=np.zeros(n + 1, np.uint8))
    rs.set_views([range(17), [3]])
    # an id out of range: host twins rejected before anything is written
    rcs, untouched = host_calls(np.array([0] * (n - 1) + [2], np.uint8))
    assert rcs == [-1] * 4 and untouched
    # device twins: an id out of range is the empty view
    ids = np.array([1, 255, 2, 0] * (n // 4 + 1), np.uint8)[:n]
    r = twins(N, torch, rs, msgs, ids, host=False)
    base_words, base_hits = rs.scan_batch(data, off)
    ew = np.array([int(base_words[i]) if ids[i] == 0 else 0 for i in range(n)], np.uint64)
    eh = [(m, x) for m, x in ((int(h["msg"]), int(h["rule"])) for h in base_hits) if ids[m] == 0 or (ids[m] == 1 and x == 3)]
    for i in range(n):
        if ids[i] == 1 and (i, 3) in eh:
            ew[i] = (1 << 63) | (1 << 32) | 3
    assert np.array_equal(r["d_words"], ew) and r["d_hits"] == eh
    empty = [i for i in range(n) if ids[i] >= 2]
    assert all(r["d_verdicts"][i] == 0 for i in empty) and not [s for s in r["d_spans"] if s[0] in empty]
    dout, doff, _, _ = r["d_redact"]
    assert all(dout[doff[i]:doff[i + 1]] == msgs[i] for i in empty)
    # set_views between calls: later calls see the new rows, calls without views are unaffected
    ids = np.zeros(n, np.uint8)
    w1, _ = rs.scan_batch(data, off, views=ids)
    rs.set_views([[3]])
    w2, _ = rs.scan_batch(data, off, views=ids)
    only3 = np.array([(1 << 63) | (1 << 32) | 3 if (i, 3) in {(int(h["msg"]), int(h["rule"])) for h in base_hits} else 0 for i in range(n)], np.uint64)
    assert np.array_equal(w1, base_words) and np.array_equal(w2, only3) and 0 < int((w2 != 0).sum()) < int((w1 != 0).sum())
    assert np.array_equal(rs.scan_batch(data, off)[0], base_words)
    rs.close()


# ------------------------------------------------------------------------------ 5. boundaries and overflow

def test_small_ragged_and_sub_range_batches(N, torch, oracle):
    """n = 0 and 1; a ragged batch of more messages than resolve_kernel's grid has threads (every message a candidate of the
    always rules); a sub-range of a device batch (d_offsets and d_views advanced together)"""
    rules = ALWAYS_LONG_RULES
    rs = N.Ruleset(rules, strict=True)
    views = view_sets(rules, seed=5)
    rs.set_views(views)
    pol, act = random_policy(rules, 6)
    rs.set_policy(pol, act)
    vo = ViewOracle(oracle, rules)
    for msgs in ([], [b"x9 sk-" + b"a1B2" * 6 + b" 77"]):
        ids = np.ones(len(msgs), np.uint8)
        words, hits, spans = vo.of(msgs, ids, views)
        check_against(twins(N, torch, rs, msgs, ids), msgs, rules, words, hits, spans, verdicts_of(hits, len(msgs), pol, act))
    rng = np.random.default_rng(7)
    n = 132 * 8 * 256 + 30011
    pool = [b"", b"x", b"ab1", b"x 42", b"no digits here", b"sk-" + b"a1B2" * 6, b"p7q x", b"ab" * 70 + b"!"]
    msgs = [pool[int(k)] for k in rng.integers(0, len(pool), n)]
    ids = rng.integers(0, len(views), n).astype(np.uint8)
    words, hits, _ = vo.of(msgs, ids, views)
    data, off = N.pack(msgs)
    w, h = rs.scan_batch(data, off, views=ids)
    assert np.array_equal(w, words) and [(int(x["msg"]), int(x["rule"])) for x in h] == hits
    d, o = to_device(torch, data, off)
    dv = torch.from_numpy(np.concatenate([ids, np.zeros(16, np.uint8)])).cuda()
    ho = HitsOut(torch, n, 4 * n)
    joined(N, rs, lambda: rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr(), n, ho.words.data_ptr(), ho.hits.data_ptr(), ho.cap,
                                                     ho.nhits.data_ptr(), views=dv.data_ptr()))
    _, pairs, _, dw = ho.result()
    assert np.array_equal(dw, words) and pairs == hits
    # sub-range [k, k + m): both pointers advanced
    k, m = 1001, 5003
    sub_w, sub_h, _ = vo.of(msgs[k:k + m], ids[k:k + m], views)
    ho = HitsOut(torch, m, 4 * m)
    joined(N, rs, lambda: rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr() + 4 * k, m, ho.words.data_ptr(), ho.hits.data_ptr(), ho.cap,
                                                     ho.nhits.data_ptr(), views=dv.data_ptr() + k))
    _, pairs, _, dw = ho.result()
    assert np.array_equal(dw, sub_w) and pairs == sub_h
    fo = FindOut(torch, 8 * m)
    joined(N, rs, lambda: rs.find_matches_batch_device(d.data_ptr(), o.data_ptr() + 4 * k, m, fo.spans.data_ptr(), fo.cap, fo.nspans.data_ptr(),
                                                        views=dv.data_ptr() + k))
    assert full(fo.result(N)[1]) == full(rs.find_matches_batch(*N.pack(msgs[k:k + m]), views=ids[k:k + m]))
    rs.close()


def test_queue_overflow_is_reported_once_then_repeats_clean(N, torch, oracle):
    """A fresh rule set sized by a small batch, then 30 000 messages that all hit, through the hit-list twin: the count is
    0xffffffff, the words all ones, the join raises CG_ERR_CAPACITY once; issued again the batch gives the per-view oracle's
    list."""
    rl = W.make_rules(64)
    rules = W.rules_as_tuples(rl)
    d0_t, o0_t, _ = W.make_messages(64, 256, rl, p_hit=0.0, seed=3)
    d1_t, o1_t, _ = W.make_messages(30000, 256, rl, p_hit=1.0, seed=4)
    n1 = 30000
    data1, off1 = d1_t.numpy(), o1_t.numpy().astype(np.uint32)
    msgs1 = [bytes(data1[int(off1[i]):int(off1[i + 1])]) for i in range(n1)]
    views = view_sets(rules, seed=8)
    ids = np.random.default_rng(9).integers(1, len(views), n1).astype(np.uint8)
    words, hits, _ = ViewOracle(oracle, rules).of(msgs1, ids, views)
    rs = N.Ruleset(rules, strict=True)
    rs.set_views(views)
    st = torch.cuda.Stream()
    d0, o0 = to_device(torch, d0_t.numpy(), o0_t.numpy())
    d1, o1 = to_device(torch, data1, off1)
    v0 = torch.zeros(80, dtype=torch.uint8, device="cuda")
    v1 = torch.from_numpy(np.concatenate([ids, np.zeros(16, np.uint8)])).cuda()
    small, big = HitsOut(torch, 64, 1024), HitsOut(torch, n1, 4 * n1)

    def issue(ho, d, o, v, n):
        rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr(), n, ho.words.data_ptr(), ho.hits.data_ptr(), ho.cap, ho.nhits.data_ptr(),
                                  st.cuda_stream, views=v.data_ptr())
    issue(small, d0, o0, v0, 64)
    issue(big, d1, o1, v1, n1)
    with pytest.raises(N.GovError) as ei:
        rs.scan_join(st.cuda_stream)
    assert ei.value.code == N.CG_ERR_CAPACITY
    nh, _, _, w = big.result()
    assert nh == ALL_ONES and (big.hits.cpu().numpy().view(np.uint32) == GUARD).all()
    assert (w == np.uint64(0xffffffffffffffff)).all()
    for attempt in range(4):
        issue(big, d1, o1, v1, n1)
        try:
            rs.scan_join(st.cuda_stream)
            break
        except N.GovError as e:
            assert e.code == N.CG_ERR_CAPACITY and attempt < 3
    nh, pairs, guard, w = big.result()
    assert nh == len(hits) and pairs == hits and (guard == GUARD).all() and np.array_equal(w, words)
    rs.close()


# ------------------------------------------------------------------------------ 6. plugin

@pytest.mark.parametrize("cats", [["credential", "pii", "financial"], ["pii", "financial"]])
def test_credential_only_strings_equal_the_credential_engine(N, cats):
    """RedactionEngine.scan_strings(inputs, credential_only=flags) == credential_engine.scan_strings on the flagged strings
    and engine.scan_strings on the others, string by string in the same order: outputs, counts, categories and the vault's
    entries -- also when the configured categories leave the credential built-ins out"""
    import json
    import os
    from vainplex_openclaw_b200 import plugin as P
    here = os.path.dirname(os.path.abspath(__file__))
    inputs = [v["input"] for v in json.load(open(os.path.join(here, "golden", "registry_vectors.json")))["vectors"]][:150]
    inputs += ["", "key sk-" + "Q1w2" * 6 + " for bob@example.com", "card 4111 1111 1111 1111 and password=Hunter2Hunter2"] * 3
    flags = [bool(x) for x in np.random.default_rng(11).integers(0, 2, len(inputs))]
    custom = [{"name": "ticket", "regex": "TCK-[0-9]{4}", "category": "custom"}]
    v1, v2 = P.RedactionVault(), P.RedactionVault()
    engine = P.RedactionEngine(P.PatternRegistry(cats, custom), v1)
    cred = P.RedactionEngine(P.PatternRegistry(["credential"], []), v1)
    combined = P.RedactionEngine(P.PatternRegistry(cats, custom), v2)
    want = [(cred if f else engine).scan_strings([s])[0] for s, f in zip(inputs, flags)]
    got = combined.scan_strings(inputs, credential_only=flags)
    assert sum(r["redactionCount"] for r in want) >= 40
    assert any(f and r["redactionCount"] for f, r in zip(flags, want)) and any(not f and "pii" in r["categories"] for f, r in zip(flags, want))
    for s, a, b in zip(inputs, want, got):
        assert (a["output"], a["redactionCount"], a["categories"]) == (b["output"], b["redactionCount"], b["categories"]), s
    strip = lambda v: {h: {k: e[k] for k in ("original", "category", "placeholder")} for h, e in v.entries.items()}
    assert strip(v1) == strip(v2) and v1.hash_index == v2.hash_index


def scoped_restatement(mp, texts, contexts):
    """matchesScope (PolicyEvaluator._matches_scope) over the policies, then evaluate_batch's aggregation of the hits of the
    in-scope policies' rules"""
    from vainplex_openclaw_b200 import plugin as P
    out = []
    for hit, ctx in zip(mp.scanner.scan(texts), contexts):
        per_policy = {}
        for h in hit:
            pi, ri = mp.index[h]
            if P.PolicyEvaluator._matches_scope(mp.policies[pi], ctx) and (pi not in per_policy or ri < per_policy[pi]):
                per_policy[pi] = ri
        action, reason = "allow", "No matching policies"
        for pi in sorted(per_policy):
            eff = mp.policies[pi]["rules"][per_policy[pi]].get("effect", {"action": "deny"})
            if eff["action"] == "deny" and action != "deny":
                action, reason = "deny", eff.get("reason", "Denied by policy %s" % mp.policies[pi]["id"])
            elif eff["action"] == "audit" and action == "allow":
                action, reason = "audit", eff.get("reason", "")
        out.append((action, reason, len(per_policy)))
    return out


def test_scoped_verdicts_equal_a_host_restatement(N):
    """MessagePolicy.verdict_batch(texts, contexts) honours every policy's scope (excludeAgents, channels) on random scoped
    policy sets, one view per distinct in-scope set; without contexts it is unchanged"""
    import random
    from vainplex_openclaw_b200 import plugin as P
    rnd = random.Random(12)
    words = ["alpha", "bravo", "charlie", "delta", "echo", "foxtrot", "golf", "hotel", "india", "juliet"]
    agents, channels = ["main", "ops", "bot", None], ["slack", "mail", "web", None]
    for trial in range(3):
        policies = []
        for pi in range(12):
            rules = [{"messageContains": [rnd.choice(words) for _ in range(rnd.randint(1, 2))],
                      "effect": {"action": rnd.choice(["deny", "audit", "allow"]), "reason": "p%d r%d" % (pi, ri)}} for ri in range(rnd.randint(1, 3))]
            scope = {}
            if rnd.random() < 0.5:
                scope["excludeAgents"] = rnd.sample(agents[:3], rnd.randint(1, 2))
            if rnd.random() < 0.5:
                scope["channels"] = rnd.sample(channels[:3], rnd.randint(1, 2))
            policies.append({"id": "pol%d" % pi, "priority": rnd.randint(0, 5) * 10, "rules": rules, "scope": scope})
        mp = P.MessagePolicy(policies)
        texts = [" ".join(rnd.choice(words + ["zulu"] * 4) for _ in range(rnd.randint(0, 8))) for _ in range(800)]
        contexts = [{"agentId": rnd.choice(agents), "channel": rnd.choice(channels)} for _ in texts]
        want = scoped_restatement(mp, texts, contexts)
        rs, calls = mp.scanner.ruleset, []
        set_views = rs.set_views
        rs.set_views = lambda v: (calls.append(v), set_views(v))
        got = mp.verdict_batch(texts, contexts)
        assert [(g["action"], g["reason"], g["matchedPolicies"]) for g in got] == want
        # the same views again: the rows stay as they are; other contexts: new rows
        assert mp.verdict_batch(texts, contexts) == got and len(calls) == 1
        half = [{"agentId": "main", "channel": "slack"}] * len(texts)
        assert [(g["action"], g["reason"], g["matchedPolicies"]) for g in mp.verdict_batch(texts, half)] == scoped_restatement(mp, texts, half)
        assert len(calls) == 2
        assert mp.verdict_batch(texts, contexts) == got and len(calls) == 3
        del rs.set_views
        assert len({w[0] for w in want}) == 3
        assert [(g["action"], g["reason"], g["matchedPolicies"]) for g in mp.verdict_batch(texts)] == \
            [(x["action"], x["reason"], len(x["matches"])) for x in mp.evaluate_batch(texts)]
