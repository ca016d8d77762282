"""One evaluation context per call (cg_policy_eval_one) beside the paths that exist for it.

Workloads: the reference's built-ins on one tool-call context; the policy set of DESIGN §7 (the 500 C2 rules as
messageContains rules of 250 policies, plus the built-ins) on one 256-byte message with 0, 5 and 20 conversation entries of
256 bytes, with a planted hit in the message and without.  Calls, each the host-clock median of --iters calls after --warmup:
  evaluate        PolicyEvaluator.evaluate(ctx): cg_scan_batch, then the host walk
  verdict_batch   PolicyEvaluator.verdict_batch([ctx]): atoms, packing, cg_policy_eval_batch with one context
  verdict_one     PolicyEvaluator.verdict_one(ctx): atoms, packing, cg_policy_eval_one
  batch_raw       the bare ctypes call of cg_policy_eval_batch on inputs built once
  one_raw         the bare ctypes call of cg_policy_eval_one on inputs built once
  scan_one_raw    cg_scan_one on the message alone (the single-message scan, for scale)
With --profile, policy_eval_one_kernel's device time from torch.profiler instead (a run of its own; the trace is not kept).
Prints one JSON line with the card's name, power limit and max SM clock read in the same run.  Needs an H100; writes nothing.

    python profiles/policy_eval_one.py [--iters 2000] [--warmup 200] [--profile]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from hits_device import card  # noqa: E402


def median_us(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return round(float(np.median(t)) * 1e6, 1)


def workloads(N, P, W, PP):
    """-> [(name, PolicyEvaluator, ctx, message bytes)]"""
    out = []
    bpe = P.PolicyEvaluator(PP.builtin_policies(), other_condition=PP.other_condition)
    tool = {"agentId": "main", "channel": "matrix", "sessionKey": "agent:main:1", "toolName": "exec",
            "toolParams": {"command": "git push origin main", "path": "/srv/credentials/db.key"},
            "trust": {"agent": {"tier": "standard"}, "session": {"tier": "standard"}}, "conversationContext": [], "messageContent": ""}
    out.append(("builtins_tool_call", bpe, tool, b""))
    rl = [r for r in W.make_rules(500) if N.rule_check(r["source"], 0) == 0]
    pols = [{"id": "c2-%d" % i, "priority": 1, "rules": [
        {"id": "deny", "conditions": [{"type": "context", "messageContains": rl[2 * i]["source"]}], "effect": {"action": "deny", "reason": "rule %d" % (2 * i)}},
        {"id": "audit", "conditions": [{"type": "context", "messageContains": rl[2 * i + 1]["source"]}], "effect": {"action": "audit"}}]}
        for i in range(len(rl) // 2)]
    pe = P.PolicyEvaluator(pols + PP.builtin_policies(), other_condition=PP.other_condition)
    hit_t, hit_o, inj = W.make_messages(64, 256, rl, p_hit=1.0, seed=5)
    clean_t, clean_o, _ = W.make_messages(64, 256, rl, p_hit=0.0, seed=6)
    hd, ho, cd, co = hit_t.numpy(), hit_o.numpy(), clean_t.numpy(), clean_o.numpy()
    msg = lambda d, o, i: bytes(d[int(o[i]):int(o[i + 1])]).decode("utf-8", "replace")   # noqa: E731
    for conv in (0, 5, 20):
        for hit in (False, True):
            m = msg(hd, ho, 0) if hit else msg(cd, co, 0)
            ctx = {"agentId": "main", "channel": "matrix", "sessionKey": "agent:main:1", "toolName": None, "toolParams": None,
                   "trust": {"agent": {"tier": "standard"}, "session": {"tier": "standard"}},
                   "messageContent": m, "conversationContext": [msg(cd, co, 1 + k) for k in range(conv)]}
            out.append(("c2_250_policies_conv%d_%s" % (conv, "hit" if hit else "clean"), pe, ctx, N.js_utf8(m)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("policy_eval_one.py needs a CUDA device")
    import policy_program as PP
    from vainplex_openclaw_b200 import _native as N, plugin as P, workload as W
    N.init(0)
    L = N.load()
    res = {"card": card(), "iters": a.iters, "warmup": a.warmup, "workloads": {}}
    for name, pe, ctx, m in workloads(N, P, W, PP):
        assert pe.verdict_one(ctx) == pe.verdict_batch([ctx])[0]
        rs = pe._program_ruleset()
        texts, roles, ctx_off, atoms = pe.program_inputs([ctx])
        data, off = N.pack([N.js_utf8(t) for t in texts])
        n = len(texts)
        row = np.ascontiguousarray(atoms[0])
        ver, nm = np.zeros(1, np.uint32), C.c_uint32(0)
        matches = np.zeros(1024, N.POLICY_MATCH_DTYPE)
        rules = np.zeros(1024, np.uint32)
        v1 = C.c_uint32(0)
        rp, ap_, cp = roles.ctypes.data if n else None, row.ctypes.data if row.size else None, ctx_off.ctypes.data

        def batch_raw():
            assert L.cg_policy_eval_batch(rs.handle, data.ctypes.data, off.ctypes.data, rp, n, cp, ap_, 1, ver.ctypes.data, matches.ctypes.data, 1024, C.byref(nm)) == 0

        def one_raw():
            assert L.cg_policy_eval_one(rs.handle, data.ctypes.data, off.ctypes.data, rp, n, ap_, C.byref(v1), rules.ctypes.data, 1024, C.byref(nm)) == 0
        one_raw()
        batch_raw()
        w = {"texts": n, "bytes": int(off[-1]), "verdict": int(v1.value), "matches": int(nm.value)}
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            for _ in range(a.warmup):
                one_raw()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(200):
                    one_raw()
            ks = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" and "policy_eval_one_kernel" in e.key:
                    ks = {"calls": e.count, "avg_us": round(e.device_time_total / max(e.count, 1), 2)}
            w["policy_eval_one_kernel"] = ks
        else:
            w["evaluate_us"] = median_us(lambda: pe.evaluate(ctx), a.iters, a.warmup)
            w["verdict_batch_us"] = median_us(lambda: pe.verdict_batch([ctx]), a.iters, a.warmup)
            w["verdict_one_us"] = median_us(lambda: pe.verdict_one(ctx), a.iters, a.warmup)
            w["batch_raw_us"] = median_us(batch_raw, a.iters, a.warmup)
            w["one_raw_us"] = median_us(one_raw, a.iters, a.warmup)
            if m:
                sw, sn = C.c_uint64(0), C.c_uint32(0)
                srs = pe.scanner.ruleset
                w["scan_one_raw_us"] = median_us(lambda: L.cg_scan_one(srs.handle, m, len(m), C.byref(sw), rules.ctypes.data, 1024, C.byref(sn)), a.iters, a.warmup)
        res["workloads"][name] = w
    print(json.dumps(res))


if __name__ == "__main__":
    main()
