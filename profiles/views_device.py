"""Per-message views on the device (cg_scan_hits_batch_device_views / cg_redact_batch_device_views) beside the calls without
views and beside the alternative a caller has without them: one rule set per subset, each called on its gathered messages.

The C2 shape: 500 rules, 256-byte messages, 1 Mi messages, p_hit 1 % and 10 %.  For the hit list and for redaction:
  all      the call without views (every rule)
  full     the _views twin, every message in the view of all rules
  split    the _views twin, two views of half the rules each, assigned to the messages at random
  two_sets two rule sets compiled from the two halves, each called on its messages gathered into a batch of their own
           (the gather itself is not timed)
Each variant: host clock around enqueue + cg_scan_join and CUDA events around the same work on its stream, the median of
--iters runs, the variants interleaved run by run.  Prints one JSON line with the card's name, power limit and max SM clock
read in the same run.  Needs an H100; writes nothing.

    python profiles/views_device.py [--msgs 1048576] [--iters 20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from profiles.hits_device import card  # noqa: E402


def med(t):
    return {"ms_median": float(np.median(t)), "ms_min": float(min(t)), "ms_max": float(max(t))}


def measure(N, torch, rl, n, L, p_hit, iters):
    from vainplex_openclaw_b200 import workload as W
    rules = W.rules_as_tuples(rl)
    R = len(rules)
    rng = np.random.default_rng(99)
    half_a = sorted(int(x) for x in rng.choice(R, R // 2, replace=False))
    half_b = sorted(set(range(R)) - set(half_a))
    rs = N.Ruleset(rules, strict=True)
    rs.set_views([range(R), half_a, half_b])
    sets = [N.Ruleset([rules[i] for i in h], strict=True) for h in (half_a, half_b)]
    data_t, off_t, _ = W.make_messages(n, L, rl, p_hit=p_hit, seed=4321)
    data, off = data_t.numpy(), off_t.numpy().astype(np.uint32)
    split = rng.integers(1, 3, n).astype(np.uint8)
    st = torch.cuda.Stream()

    def dev_batch(msgs_idx):
        """a batch of the messages msgs_idx in HBM: (bytes, offsets, n)"""
        lens = (off[1:] - off[:-1])[msgs_idx].astype(np.int64)
        o = np.zeros(len(msgs_idx) + 1, np.int64); o[1:] = np.cumsum(lens)
        starts = off[:-1][msgs_idx].astype(np.int64)
        idx = (np.repeat(starts - o[:-1], lens) + np.arange(int(o[-1]))) if len(msgs_idx) else np.zeros(0, np.int64)
        buf = np.concatenate([data[idx], np.zeros(64, np.uint8)])
        return torch.from_numpy(buf).cuda(), torch.from_numpy(o.astype(np.int32)).cuda(), len(msgs_idx)

    whole = (torch.from_numpy(np.concatenate([data[:int(off[n])], np.zeros(64, np.uint8)])).cuda(), torch.from_numpy(off.astype(np.int32)).cuda(), n)
    parts = [dev_batch(np.nonzero(split == v)[0]) for v in (1, 2)]
    v_full = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    v_split = torch.from_numpy(np.concatenate([split, np.zeros(16, np.uint8)])).cuda()

    class Out:
        def __init__(self, m, nbytes):
            self.words = torch.empty(max(m, 1), dtype=torch.int64, device="cuda")
            self.hits = torch.empty(2 * 4 * max(m, 1), dtype=torch.int32, device="cuda")
            self.nh = torch.empty(1, dtype=torch.int32, device="cuda")
            self.out = torch.empty(4 * nbytes + (1 << 20), dtype=torch.uint8, device="cuda")
            self.off = torch.empty(m + 1, dtype=torch.int32, device="cuda")
            self.spans = torch.empty(6 * 4 * max(m, 1), dtype=torch.int32, device="cuda")
            self.dig = torch.empty(32 * 4 * max(m, 1), dtype=torch.uint8, device="cuda")
            self.sizes = torch.empty(2, dtype=torch.int64, device="cuda")
            self.cap = 4 * max(m, 1)

    outs = {"whole": Out(n, int(off[n])), "p1": Out(parts[0][2], parts[0][0].numel()), "p2": Out(parts[1][2], parts[1][0].numel())}
    s = st.cuda_stream

    def hits(r, b, o, views=None):
        r.scan_hits_batch_device(b[0].data_ptr(), b[1].data_ptr(), b[2], o.words.data_ptr(), o.hits.data_ptr(), o.cap, o.nh.data_ptr(), s, views=views)

    def redact(r, b, o, views=None):
        r.redact_batch_device(b[0].data_ptr(), b[1].data_ptr(), b[2], o.out.data_ptr(), o.out.numel() - 64, o.off.data_ptr(), o.spans.data_ptr(), o.cap,
                              o.dig.data_ptr(), o.sizes.data_ptr(), s, views=views)

    variants = {}
    for name, call in (("hits", hits), ("redact", redact)):
        variants[name + "/all"] = lambda call=call: call(rs, whole, outs["whole"])
        variants[name + "/full"] = lambda call=call: call(rs, whole, outs["whole"], v_full.data_ptr())
        variants[name + "/split"] = lambda call=call: call(rs, whole, outs["whole"], v_split.data_ptr())
        variants[name + "/two_sets"] = lambda call=call: (call(sets[0], parts[0], outs["p1"]), call(sets[1], parts[1], outs["p2"]))

    def join():
        rs.scan_join(s); sets[0].scan_join(s); sets[1].scan_join(s)

    # warm-up (scratch grown, modules loaded), and the results the timings stand for
    for f in variants.values():
        for _ in range(3):
            f(); join()
    check = {}
    for name in ("hits/all", "hits/full", "redact/all", "redact/full"):
        variants[name](); join()
        o = outs["whole"]
        check[name] = (o.nh.cpu().numpy().tobytes(), o.words.cpu().numpy().tobytes()) if name.startswith("hits") else \
            (o.sizes.cpu().numpy().tobytes(), o.off.cpu().numpy().tobytes(), o.out[:int(o.sizes[0].item())].cpu().numpy().tobytes())
    assert check["hits/all"] == check["hits/full"] and check["redact/all"] == check["redact/full"], "full view differs from the call without views"
    host = {k: [] for k in variants}
    dev = {k: [] for k in variants}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for it in range(iters):
        keys = list(variants) if it % 2 == 0 else list(reversed(list(variants)))
        for k in keys:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ev0.record(st)
            variants[k]()
            ev1.record(st)
            join()
            host[k].append((time.perf_counter() - t0) * 1e3)
            dev[k].append(ev0.elapsed_time(ev1))
    for r in sets:
        r.close()
    rs.close()
    return {"p_hit": p_hit, "split_sizes": [parts[0][2], parts[1][2]],
            "ms": {k: {"host": med(host[k]), "device": med(dev[k])} for k in variants}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--msgs", type=int, default=1 << 20)
    ap.add_argument("--len", type=int, default=256)
    ap.add_argument("--rules", type=int, default=500)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("views_device.py needs a CUDA device")
    from vainplex_openclaw_b200 import _native as N, workload as W
    N.init(0)
    rl = W.make_rules(a.rules)
    res = [measure(N, torch, rl, a.msgs, a.len, p, a.iters) for p in (0.01, 0.10)]
    print(json.dumps({"workload": {"rules": a.rules, "msg_bytes": a.len, "msgs": a.msgs}, "card": card(), "results": res}))


if __name__ == "__main__":
    main()
