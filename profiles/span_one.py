"""Latency of the single-message calls the synchronous hooks make, beside the batch calls at n = 1.

Per call, host clock around the blocking call through the Python binding (the batch calls on a batch packed once),
median and p10 / p90 over --calls calls after --warm calls:
  scan_one            cg_scan_one
  find_batch_n1       cg_find_matches_batch with n = 1
  find_one            cg_find_matches_one
  redact_batch_n1     cg_redact_batch with n = 1
  redact_one          cg_redact_one
on the 17 built-in rules and the 500-rule C2 set, for a 256-byte message without a hit, one with a hit, and a 4 KB
message with hits; plus the plugin's tool_result_persist handler on a JSON tool result with 20 string leaves.
Prints one JSON line with the card's name, power limit and max SM clock read in the same run.  Needs an H100; writes nothing.

    python profiles/span_one.py [--calls 2000] [--warm 200]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from profiles.redact_device import card  # noqa: E402


def timed(fn, calls, warm):
    for _ in range(warm):
        fn()
    t = np.empty(calls)
    for i in range(calls):
        t0 = time.perf_counter()
        fn()
        t[i] = time.perf_counter() - t0
    us = t * 1e6
    return {"median_us": float(np.median(us)), "p10_us": float(np.percentile(us, 10)), "p90_us": float(np.percentile(us, 90))}


def calls_for(N, rs, msg):
    """the five calls on one message through the Python binding (the batch calls on a batch packed once)"""
    data, off = N.pack([msg])
    return {
        "scan_one": lambda: rs.scan_one(msg),
        "find_batch_n1": lambda: rs.find_matches_batch(data, off),
        "find_one": lambda: rs.find_matches_one(msg),
        "redact_batch_n1": lambda: rs.redact_batch(data, off),
        "redact_one": lambda: rs.redact_one(msg),
    }


def tool_result(W):
    """a JSON tool result of 20 string leaves, a few of them holding a secret"""
    rng = np.random.default_rng(5)
    words = ["deploy", "status", "ok", "build", "artifact", "region", "eu-west", "latency", "retry", "node", "cache", "warm"]
    leaves = {}
    for i in range(20):
        s = " ".join(words[int(k)] for k in rng.integers(0, len(words), 12))
        if i % 7 == 3:
            s += " token sk-" + "Zq9" * 10
        if i % 9 == 5:
            s += " mail bob.smith@example.com"
        leaves["field_%02d" % i] = s
    return {"toolName": "exec", "message": {"stdout": leaves}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--warm", type=int, default=200)
    a = ap.parse_args()
    from vainplex_openclaw_b200 import _native as N, plugin as P, workload as W
    N.init(0)
    results = []
    for n_rules in (17, 500):
        rl = W.make_rules(n_rules)
        rs = N.Ruleset(W.rules_as_tuples(rl), strict=True)
        msgs = {}
        for name, L, p in (("256B_no_hit", 256, 0.0), ("256B_hit", 256, 1.0), ("4KB", 4096, 1.0)):
            data_t, _, _ = W.make_messages(1, L, rl, p_hit=p, seed=11 + L)
            msgs[name] = bytes(data_t.numpy()[:L])
        for name, msg in msgs.items():
            fns = calls_for(N, rs, msg)
            spans = len(rs.find_matches_one(msg))
            row = {"rules": n_rules, "message": name, "bytes": len(msg), "spans": spans}
            for k, fn in fns.items():
                row[k] = timed(fn, a.calls, a.warm)
            k0 = N.launch_count(); fns["find_one"](); k1 = N.launch_count(); fns["find_batch_n1"](); k2 = N.launch_count()
            fns["redact_one"](); k3 = N.launch_count(); fns["redact_batch_n1"](); k4 = N.launch_count()
            row["kernels"] = {"find_one": k1 - k0, "find_batch_n1": k2 - k1, "redact_one": k3 - k2, "redact_batch_n1": k4 - k3}
            results.append(row)
        rs.close()

    class Api:
        def __init__(self):
            self.handlers, self.pluginConfig, self.logger = [], {}, P.NullLogger()

        def on(self, name, handler, opts=None):
            self.handlers.append((name, (opts or {}).get("priority"), handler))

        def registerGatewayMethod(self, name, fn):
            pass
    api = Api()
    P.GovernancePlugin().register(api)
    trp = [h for (n, p, h) in api.handlers if n == "tool_result_persist" and p == 800][0]
    ev = tool_result(W)
    assert "[REDACTED:" in trp(ev, {})["message"]
    hook = {"hook": "tool_result_persist", "string_leaves": 20, **timed(lambda: trp(ev, {}), a.calls, a.warm)}
    print(json.dumps({"card": card(), "calls": a.calls, "warm": a.warm, "results": results, "plugin": hook}))


if __name__ == "__main__":
    main()
