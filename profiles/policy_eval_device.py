"""Whole policy rules on the device (cg_policy_eval_batch_device) beside today's paths.

The C2 shape: 1 Mi evaluation contexts, each one 256-byte message and one `command` tool param; the policies are the
500 C2 rules as messageContains rules of 250 policies (a deny and an audit rule each) plus the reference's built-ins
(credential guard, production safeguard, rate limiter, night mode: tool-param `matches`, trust tiers, `any`, `not`,
frequency / time atoms).  Calls:
  policy_eval_device           cg_policy_eval_batch_device, verdicts only, then with the match list
  hits_device_plus_host_walk   cg_scan_hits_batch_device over the same texts, the hit list to the host, then
                               PolicyEvaluator's host walk (_evaluate) -- the walk timed on a sample of contexts and scaled
  verdict_device_slice         cg_policy_verdict_batch_device on the messageContains-only slice (messages alone)
Each: median of --iters runs, host clock around enqueue + join and CUDA events around the enqueue on the stream.  Prints
one JSON line with the card's name, power limit and max SM clock read in the same run.  Needs an H100; writes nothing.

    python profiles/policy_eval_device.py [--ctx 1048576] [--iters 20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from hits_device import card  # noqa: E402


def timed(torch, st, fn, iters):
    for _ in range(3):
        try:
            fn()
        except Exception as e:                                # (a fresh rule set's first large batch may overflow a queue: the join
            if getattr(e, "code", 0) != -7:                   # reports it once, the scratch grows and the next call runs)
                raise
    host, dev = [], []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(iters):
        t0 = time.perf_counter()
        e0.record(st)
        fn()
        e1.record(st)
        e1.synchronize()
        host.append((time.perf_counter() - t0) * 1e3)
        dev.append(e0.elapsed_time(e1))
    return {"host_ms_median": float(np.median(host)), "event_ms_median": float(np.median(dev)), "host_ms_min": min(host), "iters": iters}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctx", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--walk-sample", type=int, default=20000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("policy_eval_device.py needs a CUDA device")
    from policy_program import COMMANDS, builtin_policies, other_condition
    from vainplex_openclaw_b200 import _native as N, plugin as P, workload as W
    N.init(0)
    n = a.ctx
    rl = [r for r in W.make_rules(500) if N.rule_check(r["source"], 0) == 0]
    pols = [{"id": "c2-%d" % i, "priority": 1, "rules": [
        {"id": "deny", "conditions": [{"type": "context", "messageContains": rl[2 * i]["source"]}], "effect": {"action": "deny", "reason": "rule %d" % (2 * i)}},
        {"id": "audit", "conditions": [{"type": "context", "messageContains": rl[2 * i + 1]["source"]}], "effect": {"action": "audit"}}]}
        for i in range(len(rl) // 2)]
    pe = P.PolicyEvaluator(pols + builtin_policies(), other_condition=other_condition)
    data_t, off_t, _ = W.make_messages(n, 256, rl, p_hit=0.01, seed=1234)
    msgs = data_t.numpy()
    moff = off_t.numpy().astype(np.uint64)
    rng = np.random.default_rng(7)
    # the caller's scalar side: a few distinct (tool, agent, trust) profiles, their atom rows computed by the evaluator's helpers
    profiles = [{"agentId": ag, "channel": "matrix", "toolName": "exec", "toolParams": {"command": "x"},
                 "trust": {"agent": {"tier": t}, "session": {"tier": t}}} for ag in ("main", "unresolved") for t in ("standard", "trusted")]
    prof_rows = np.stack([pe.program_inputs([p])[3][0] for p in profiles])
    which = rng.integers(0, len(profiles), n)
    cmds = [c.encode() for c in COMMANDS]
    cmd_of = rng.integers(0, len(cmds), n)
    # texts: message i, then its command; contexts own two texts (an empty command is still a text, as evaluate_batch keeps it)
    lens = np.empty(2 * n, np.uint64)
    lens[0::2] = moff[1:] - moff[:-1]
    lens[1::2] = [len(cmds[k]) for k in cmd_of]
    off = np.zeros(2 * n + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    buf = np.zeros(int(off[-1]) + 64, np.uint8)
    for i in range(n):                                        # (setup only)
        buf[int(off[2 * i]):int(off[2 * i + 1])] = msgs[int(moff[i]):int(moff[i + 1])]
        c = cmds[cmd_of[i]]
        buf[int(off[2 * i + 1]):int(off[2 * i + 2])] = np.frombuffer(c, np.uint8) if c else []
    roles = np.zeros(2 * n, np.uint8)
    roles[1::2] = pe.param_role.get("command", 255)
    ctx_off = np.arange(0, 2 * n + 1, 2, dtype=np.uint32)
    atoms = np.ascontiguousarray(prof_rows[which])
    rs = pe.scanner.ruleset
    rs.set_policy_program(pe.program, len(pe.atoms))
    st = torch.cuda.Stream()
    dev = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x).view(dt)).cuda()
    d = dev(buf, np.uint8)
    o = dev(off.astype(np.uint32), np.int32)
    dr, dc, da = dev(np.concatenate([roles, np.zeros(4, np.uint8)]), np.uint8), dev(ctx_off, np.int32), dev(atoms.reshape(-1), np.int32)
    verdicts = torch.empty(n, dtype=torch.int32, device="cuda")
    nm = torch.empty(1, dtype=torch.int32, device="cuda")
    cap = 4 * n
    matches = torch.empty(2 * cap, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def eval_v():
        rs.eval_batch_device(d.data_ptr(), o.data_ptr(), dr.data_ptr(), 2 * n, dc.data_ptr(), da.data_ptr(), n, verdicts.data_ptr(), 0, 0, 0, st.cuda_stream)
        rs.scan_join(st.cuda_stream)

    def eval_m():
        rs.eval_batch_device(d.data_ptr(), o.data_ptr(), dr.data_ptr(), 2 * n, dc.data_ptr(), da.data_ptr(), n, verdicts.data_ptr(), matches.data_ptr(), cap,
                             nm.data_ptr(), st.cuda_stream)
        rs.scan_join(st.cuda_stream)
    res = {"policy_eval_device_verdicts": timed(torch, st, eval_v, a.iters), "policy_eval_device_matches": timed(torch, st, eval_m, a.iters)}
    k0 = N.launch_count(); eval_m(); res["policy_eval_device_matches"]["kernels"] = N.launch_count() - k0
    res["matches"] = int(nm.item()) & 0xffffffff
    v = verdicts.cpu().numpy().view(np.uint32)
    res["outcomes"] = {k: int(((v & 7) == i).sum()) for i, k in enumerate(("none", "allow", "audit", "2fa", "deny"))}
    # today's path: the hit list in HBM, to the host, then the host walk
    words = torch.empty(2 * n, dtype=torch.int64, device="cuda")
    hits = torch.empty(2 * cap, dtype=torch.int32, device="cuda")
    nh = torch.empty(1, dtype=torch.int32, device="cuda")

    def hits_once():
        rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr(), 2 * n, words.data_ptr(), hits.data_ptr(), cap, nh.data_ptr(), st.cuda_stream)
        rs.scan_join(st.cuda_stream)
        k = int(nh.item()) & 0xffffffff
        return hits[:2 * k].cpu()
    res["hits_device_plus_d2h"] = timed(torch, st, hits_once, a.iters)
    pairs = hits_once().numpy().view(np.uint32).reshape(-1, 2)
    m = min(a.walk_sample, n)
    per = [{"msg": set(), "conv": set(), "param": {"command": set()}} for _ in range(m)]
    for t, r in pairs[pairs[:, 0] < 2 * m]:
        (per[t // 2]["msg"].add(int(r)) if t % 2 == 0 else per[t // 2]["param"]["command"].add(int(r)))
    ctxs = [dict(profiles[which[i]], messageContent="m", toolParams={"command": cmds[cmd_of[i]].decode()}) for i in range(m)]
    t0 = time.perf_counter()
    walked = [pe._evaluate(ctxs[i], per[i]) for i in range(m)]
    walk_ms = (time.perf_counter() - t0) * 1e3
    res["host_walk"] = {"sample_ctx": m, "ms": walk_ms, "ms_scaled_to_all": walk_ms * n / m}
    dec = pe.decode_verdicts(v[:m], np.zeros(0, N.POLICY_MATCH_DTYPE))
    assert [r["action"] for r in dec] == [r["action"] for r in walked], "device verdicts differ from the host walk"
    # the messageContains-only slice: cg_policy_verdict_batch_device over the messages
    mp = P.MessagePolicy([{"id": p["id"], "priority": 1, "rules": [{"messageContains": r["conditions"][0]["messageContains"], "effect": r["effect"]}
                                                                    for r in p["rules"]]} for p in pols])
    mp.verdict_batch(["warm up"])
    dm, om = dev(np.concatenate([msgs, np.zeros(64, np.uint8)]), np.uint8), dev(moff.astype(np.uint32), np.int32)
    vs = torch.empty(n, dtype=torch.int32, device="cuda")

    def slice_once():
        mp.scanner.ruleset.verdict_batch_device(dm.data_ptr(), om.data_ptr(), n, vs.data_ptr(), st.cuda_stream)
        mp.scanner.ruleset.scan_join(st.cuda_stream)
    res["verdict_device_slice"] = timed(torch, st, slice_once, a.iters)
    print(json.dumps({"workload": {"contexts": n, "texts": 2 * n, "msg_bytes": 256, "program_rules": len(pe.program_rules), "atoms": len(pe.atoms)},
                      "card": card(), "results": res}))


if __name__ == "__main__":
    main()
