"""GPU tier, how the scan entry points drive the step: the number of kernels every host-buffer, device-resident and
single-message scan call launches, restated from the launchers, and the cg_stats delta each call leaves.  Every call is
issued once first, so that the measured call needs no retry.  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_redact_device import FindOut, RedactOut, ragged, to_device
from test_gpu_scan_hits_device import HitsOut
from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu

# verify_large_kernel runs when the set's longest Pike program exceeds 192 instructions (test_gpu_parity's long rules)
LONG_RULES = [(r"tok_[a-f0-9]{200}z", 0, 0), (r"(?:ab|cd|ef){70}!", 0, 1), (r"sk-[a-zA-Z0-9]{20,}", 0, 2), (r"key=[A-Z]{100}[0-9]{100}\b", 1, 3)]
FIND_RESOLVER, REDACT_RESOLVER, HIT_COUNT, HIT_EMIT, VERDICTS = 8, 10, 3, 1, 1
STAT_FIELDS = ("messages_scanned", "bytes_scanned", "candidate_events", "verified_pairs", "hits", "spans", "sha256_items")


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


@pytest.fixture(scope="module")
def torch():
    import torch as T
    return T


def step_launches(n, large):
    """reset, scan, confirm, resolve, verify_small, finalize (+ verify_large); a step over no message launches none"""
    return 0 if n == 0 else 6 + int(large)


def redact_tail(n):
    """digests, then the splice (no splice launch for an empty batch)"""
    return 1 + int(n > 0)


def rule_set(N, name):
    if name == "builtins":
        rl = W.make_rules(17)
        rules = W.rules_as_tuples(rl)
    else:
        rl, rules = None, LONG_RULES
    rs = N.Ruleset(rules, strict=True)
    rs.set_policy(np.arange(len(rules)), np.full(len(rules), 2))
    return rs, rl


def batches(rl):
    """n = 0, n = 1 and a ragged batch of a few thousand messages (some of them hits of the long rules)"""
    data_t, off_t, _ = W.make_messages(3000, 256, rl if rl is not None else W.make_rules(17), p_hit=0.2, utf8_frac=0.1, seed=77)
    msgs = ragged(data_t, off_t, seed=78, max_len=256)
    for i in range(0, len(msgs), 40):
        msgs[i] = (b"x tok_" + b"0a" * 100 + b"z", b"sk-" + b"a1B2" * 6, b"ab" * 70 + b"!", b"KEY=" + b"Q" * 100 + b"7" * 100)[(i // 40) % 4]
    return [[], [msgs[1] + b" sk-" + b"Z9" * 12], msgs]


def stats(N):
    s = N.stats()
    return {f: getattr(s, f) for f in STAT_FIELDS}


def measure(N, call):
    """-> (kernels launched, cg_stats delta, what call returned)"""
    s0, k0 = stats(N), N.launch_count()
    out = call()
    k1, s1 = N.launch_count(), stats(N)
    return k1 - k0, {f: s1[f] - s0[f] for f in STAT_FIELDS}, out


def host_delta(n, nbytes, wc, **extra):
    """a host-buffer call: messages and bytes of the batch, the step's VM pairs as both candidate events and verified pairs"""
    d = dict.fromkeys(STAT_FIELDS, 0)
    d.update(messages_scanned=n, bytes_scanned=nbytes, candidate_events=wc[1], verified_pairs=wc[1], **extra)
    return d


def device_delta(n, **extra):
    """a device-resident call: messages counted at enqueue, never bytes; spans, digests and hits once joined"""
    d = dict.fromkeys(STAT_FIELDS, 0)
    d.update(messages_scanned=n, **extra)
    return d


@pytest.mark.parametrize("name,large", [("builtins", False), ("long", True)])
def test_host_buffer_calls_launch_the_step_and_their_own_kernels(N, name, large):
    L = N.load()
    rs, rl = rule_set(N, name)
    for msgs in batches(rl):
        data, off = N.pack(msgs)
        n = len(msgs)
        nbytes = int(off[n]) - int(off[0])
        S = step_launches(n, large)
        words = np.zeros(max(n, 1), np.uint64)
        nh = C.c_uint32(0)

        def scan(hits, cap, with_nhits=True):
            return L.cg_scan_batch(rs.handle, data.ctypes.data, off.ctypes.data, n, words.ctypes.data,
                                   None if hits is None else hits.ctypes.data, cap, C.byref(nh) if with_nhits else None)

        # words only
        scan(None, 0, False)
        k, d, rc = measure(N, lambda: scan(None, 0, False))
        assert rc == 0 and k == S and d == host_delta(n, nbytes, rs.work_counters()), (n, k, d)
        # the count alone, then the list, then a list with no room
        k, d, rc = measure(N, lambda: scan(None, 0))
        total = nh.value
        assert rc == 0 and k == S + (HIT_COUNT if n else 0) and d == host_delta(n, nbytes, rs.work_counters(), hits=total), (n, k, d)
        hits = np.zeros(max(total, 1), N.HIT_DTYPE)
        k, d, rc = measure(N, lambda: scan(hits, total))
        assert rc == 0 and nh.value == total
        assert k == S + (HIT_COUNT + (HIT_EMIT if total else 0) if n else 0) and d == host_delta(n, nbytes, rs.work_counters(), hits=total), (n, k, d)
        k, d, rc = measure(N, lambda: scan(hits, 0))
        assert rc == (N.CG_ERR_CAPACITY if total else 0) and nh.value == total
        assert k == S + (HIT_COUNT if n else 0) and d == host_delta(n, nbytes, rs.work_counters(), hits=total), (n, k, d)
        assert total > 0 or n < 2

        # find-matches
        cap = 8 * n + 64
        spans = np.zeros(cap, N.SPAN_DTYPE)
        ns = C.c_uint32(0)
        find = lambda: L.cg_find_matches_batch(rs.handle, data.ctypes.data, off.ctypes.data, n, spans.ctypes.data, cap, C.byref(ns))
        find()
        k, d, rc = measure(N, find)
        assert rc == 0 and k == S + FIND_RESOLVER and d == host_delta(n, nbytes, rs.work_counters(), spans=ns.value), (n, k, d)
        found = ns.value

        # redaction: the tail only when the output fits, and its digests counted only then
        out_cap = 8 * nbytes + 65536
        out = np.zeros(out_cap + 64, np.uint8)
        out_off = np.zeros(n + 1, np.uint32)
        dig = np.zeros((cap, 32), np.uint8)
        need = C.c_uint64(0)

        def redact(out_cap):
            return L.cg_redact_batch(rs.handle, data.ctypes.data, off.ctypes.data, n, out.ctypes.data, out_cap, C.byref(need),
                                     out_off.ctypes.data, spans.ctypes.data, cap, C.byref(ns), dig.ctypes.data)

        redact(out_cap)
        k, d, rc = measure(N, lambda: redact(out_cap))
        assert rc == 0 and ns.value == found
        assert k == S + REDACT_RESOLVER + redact_tail(n) and d == host_delta(n, nbytes, rs.work_counters(), spans=found, sha256_items=found), (n, k, d)
        if need.value:
            k, d, rc = measure(N, lambda: redact(need.value - 1))
            assert rc == N.CG_ERR_CAPACITY and ns.value == found
            assert k == S + REDACT_RESOLVER and d == host_delta(n, nbytes, rs.work_counters(), spans=found), (n, k, d)

        # verdicts
        verdicts = np.zeros(max(n, 1), np.uint32)
        verdict = lambda: L.cg_policy_verdict_batch(rs.handle, data.ctypes.data, off.ctypes.data, n, verdicts.ctypes.data)
        k, d, rc = measure(N, verdict)
        assert rc == 0 and k == S + (VERDICTS if n else 0) and d == host_delta(n, nbytes, rs.work_counters()), (n, k, d)
    rs.close()


@pytest.mark.parametrize("name,large", [("builtins", False), ("long", True)])
def test_device_resident_calls_launch_the_step_and_their_own_kernels(N, torch, name, large):
    rs, rl = rule_set(N, name)
    for msgs in batches(rl):
        data, off = N.pack(msgs)
        n = len(msgs)
        S = step_launches(n, large)
        d, o = to_device(torch, data, off)
        words = torch.full((max(n, 1),), -1, dtype=torch.int64, device="cuda")
        ho = HitsOut(torch, n, 8 * n + 64)
        fo = FindOut(torch, 8 * n + 64)
        ro = RedactOut(torch, n, 8 * int(off[n]) + 65536, 8 * n + 64)
        verdicts = torch.zeros((max(n, 1),), dtype=torch.int32, device="cuda")
        calls = {
            "words": (lambda: rs.scan_batch_device(d.data_ptr(), o.data_ptr(), n, words.data_ptr()), S),
            "hits": (lambda: ho.issue(rs, d, o), S + HIT_COUNT + HIT_EMIT if n else 0),
            "verdicts": (lambda: rs.verdict_batch_device(d.data_ptr(), o.data_ptr(), n, verdicts.data_ptr()), S + VERDICTS if n else 0),
            "find": (lambda: fo.issue(rs, d, o, n), S + FIND_RESOLVER),
            "redact": (lambda: ro.issue(rs, d, o), S + REDACT_RESOLVER + redact_tail(n)),
        }
        for what, (call, want) in calls.items():
            call()
            rs.scan_join()
            torch.cuda.synchronize()
            s0 = stats(N)
            k, dq, _ = measure(N, call)
            rs.scan_join()
            torch.cuda.synchronize()
            s1 = stats(N)
            joined = {f: s1[f] - s0[f] for f in STAT_FIELDS}
            assert k == want, (what, n, k)
            ns = fo.result(N)[0] if what == "find" else int(ro.sizes[1].item()) if what == "redact" else 0
            assert dq == device_delta(n), (what, n, dq)
            extra = {"hits": {"hits": ho.nh()}, "find": {"spans": ns}, "redact": {"spans": ns, "sha256_items": ns}}.get(what, {})
            assert joined == device_delta(n, **extra), (what, n, joined)
    rs.close()


@pytest.mark.parametrize("name,large", [("builtins", False), ("long", True)])
def test_single_message_graphs_launch_the_step_and_their_tail(N, name, large):
    rs, rl = rule_set(N, name)
    for msg in (b"", b"nothing to see here", b"pad sk-" + b"a1B2" * 6 + b" tok_" + b"0a" * 100 + b"z mail me at someone@example.com"):
        S = step_launches(1, large)
        rs.scan_one(msg)
        k, d, (word, rules) = measure(N, lambda: rs.scan_one(msg))
        assert k == S + 1 and d == host_delta(1, len(msg), rs.work_counters(), hits=len(rules)), (msg, k, d)
        rs.find_matches_one(msg)
        k, d, spans = measure(N, lambda: rs.find_matches_one(msg))
        assert k == S + 2 and d == host_delta(1, len(msg), rs.work_counters(), spans=len(spans)), (msg, k, d)
        rs.redact_one(msg)
        k, d, (_, rspans, _) = measure(N, lambda: rs.redact_one(msg))
        assert len(rspans) == len(spans)
        assert k == S + 4 and d == host_delta(1, len(msg), rs.work_counters(), spans=len(spans), sha256_items=len(spans)), (msg, k, d)
    rs.close()
