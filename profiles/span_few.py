"""Latency of the few-string span calls (cg_find_matches_few / cg_redact_few) beside the paths that exist for the same work.

Per call, host clock around the blocking call through the Python binding, median and p10 / p90 over --calls calls after
--warm calls (span_one.py's timed):
  n_x_redact_one   n calls of cg_redact_one, one per string
  redact_batch     cg_redact_batch on the n strings
  redact_few       cg_redact_few on the n strings
for n = 1, 5, 20, 64 and 256 short strings (64 bytes, every fourth one with a planted hit), on the 17 built-in rules and on
the 500-rule C2 set; then cg_redact_few at a string count missing from the graph cache (the calls cycle through more counts
than the cache keeps, so every call records the step again and re-targets an evicted graph).  With --handler only the
plugin's tool_result_persist handler on span_one.py's JSON tool result of 20 string leaves and on one of 200 (its leaves ten
times over), so that the parent tree's handler can be timed in the same run with --tree.
Prints one JSON line with the card's name, power limit and max SM clock read in the same run.  Needs an H100; writes nothing.

    python profiles/span_few.py [--calls 1000] [--warm 100]
    python profiles/span_few.py --handler [--tree PATH]
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, HERE)


def tool_results(tool_result, W):
    one = tool_result(W)
    leaves = one["message"]["stdout"]
    big = {"%s_%d" % (k, j): v for j in range(10) for k, v in leaves.items()}
    return {20: one, 200: {"toolName": "exec", "message": {"stdout": big}}}


def handler(a, timed, tool_result):
    from vainplex_openclaw_b200 import _native as N, plugin as P, workload as W
    N.init(0)

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
    out = []
    for leaves, ev in tool_results(tool_result, W).items():
        assert "[REDACTED:" in trp(ev, {})["message"]
        k0 = N.launch_count(); trp(ev, {}); k1 = N.launch_count()
        out.append({"hook": "tool_result_persist", "string_leaves": leaves, "kernels": k1 - k0, **timed(lambda: trp(ev, {}), a.calls, a.warm)})
    return out


def calls(a, timed):
    from vainplex_openclaw_b200 import _native as N, workload as W
    N.init(0)
    results = []
    for n_rules in (17, 500):
        rl = W.make_rules(n_rules)
        rs = N.Ruleset(W.rules_as_tuples(rl), strict=True)
        data_t, _, _ = W.make_messages(256, 64, rl, p_hit=0.25, seed=21)
        pool = [bytes(data_t.numpy()[64 * i:64 * (i + 1)]) for i in range(256)]
        for n in (1, 5, 20, 64, 256):
            msgs = pool[:n]
            data, off = N.pack(msgs)
            assert [tuple(x) for x in rs.redact_few(data, off)[2].tolist()] == [tuple(x) for x in rs.redact_batch(data, off)[2].tolist()]
            row = {"rules": n_rules, "strings": n, "bytes": int(off[-1]), "spans": len(rs.find_matches_few(data, off))}
            row["n_x_redact_one"] = timed(lambda: [rs.redact_one(m) for m in msgs], max(a.calls // n, 20), max(a.warm // n, 5))
            row["redact_batch"] = timed(lambda: rs.redact_batch(data, off), a.calls, a.warm)
            row["redact_few"] = timed(lambda: rs.redact_few(data, off), a.calls, a.warm)
            k0 = N.launch_count(); rs.redact_few(data, off); k1 = N.launch_count(); rs.redact_batch(data, off); k2 = N.launch_count()
            row["kernels"] = {"redact_few": k1 - k0, "redact_batch": k2 - k1}
            results.append(row)
        # a count missing from the graph cache on every call: 40 counts in turn (the cache keeps 16)
        sets = [N.pack(pool[:n]) for n in range(20, 60)]
        it = iter(range(1 << 30))
        miss = timed(lambda: rs.redact_few(*sets[next(it) % len(sets)]), a.calls, a.warm)
        hit = timed(lambda: rs.redact_few(*sets[0]), a.calls, a.warm)
        bat = timed(lambda: rs.redact_batch(*sets[0]), a.calls, a.warm)
        results.append({"rules": n_rules, "graph_cache": {"strings": "20..59 in turn", "redact_few_missing": miss, "redact_few_cached_20": hit,
                                                          "redact_batch_20": bat}})
        rs.close()
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--warm", type=int, default=100)
    ap.add_argument("--handler", action="store_true")
    ap.add_argument("--tree", default=None, help="import the package from this tree instead (the handler of another version)")
    a = ap.parse_args()
    if a.tree:
        sys.path.insert(0, os.path.abspath(a.tree))
    from profiles.redact_device import card
    from profiles.span_one import timed, tool_result
    res = handler(a, timed, tool_result) if a.handler else calls(a, timed)
    import vainplex_openclaw_b200
    print(json.dumps({"card": card(), "tree": os.path.dirname(os.path.dirname(os.path.abspath(vainplex_openclaw_b200.__file__))),
                      "calls": a.calls, "warm": a.warm, "results": res}))


if __name__ == "__main__":
    main()
