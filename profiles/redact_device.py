"""Redaction rate from HBM (cg_redact_batch_device) beside the host-buffer call (cg_redact_batch).

The C2 shape of bench.py's extra.redact: 500 rules, 256-byte messages, 256 Ki messages, p_hit 1 % and 10 %.
  device: host clock around enqueue + cg_scan_join, many iterations after warm-up, inputs and outputs in HBM
  host:   host clock around cg_redact_batch from pinned host buffers, with cg_stats.last_scan_ms (the span-mode scan step
          alone, CUDA events) so that the share of the scan in the call is visible
Prints one JSON line with the card's name and power limit read in the same run.  Needs an H100; writes nothing.

    python profiles/redact_device.py [--msgs 262144] [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        name, power, clk = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:                                    # (the rates still stand; the card is then unknown)
        return {"error": str(e)}


def measure(N, torch, rs, rl, n, L, p_hit, iters):
    from vainplex_openclaw_b200 import workload as W
    data_t, off_t, _ = W.make_messages(n, L, rl, p_hit=p_hit, seed=1234)
    h_data = torch.empty(data_t.numel(), dtype=torch.uint8, pin_memory=True); h_data.copy_(data_t)
    h_off = torch.empty(n + 1, dtype=torch.int32, pin_memory=True); h_off.copy_(off_t)
    hd, ho = h_data.numpy(), h_off.numpy().view(np.uint32)
    # host-buffer call
    out, out_off, spans, dig = rs.redact_batch(hd, ho)
    t_host, scan_ms = [], []
    for _ in range(max(3, iters // 4)):
        t0 = time.perf_counter()
        rs.redact_batch(hd, ho)
        t_host.append(time.perf_counter() - t0)
        scan_ms.append(N.stats().last_scan_ms)
    # device-resident call
    d, o = h_data.cuda(), h_off.cuda()
    need, ns = len(out), len(spans)
    d_out = torch.empty(need + 64, dtype=torch.uint8, device="cuda")
    d_off = torch.empty(n + 1, dtype=torch.int32, device="cuda")
    d_spans = torch.empty(max(ns, 1) * 6, dtype=torch.int32, device="cuda")
    d_dig = torch.empty(max(ns, 1) * 32, dtype=torch.uint8, device="cuda")
    d_sizes = torch.empty(2, dtype=torch.int64, device="cuda")
    st = torch.cuda.Stream()
    torch.cuda.synchronize()

    def once():
        rs.redact_batch_device(d.data_ptr(), o.data_ptr(), n, d_out.data_ptr(), need, d_off.data_ptr(), d_spans.data_ptr(), ns,
                               d_dig.data_ptr(), d_sizes.data_ptr(), st.cuda_stream)
        rs.scan_join(st.cuda_stream)

    for _ in range(3):
        once()
    assert np.array_equal(d_out.cpu().numpy()[:need], out), "device output differs from the host call"
    t_dev = []
    for _ in range(iters):
        t0 = time.perf_counter()
        once()
        t_dev.append(time.perf_counter() - t0)
    k0 = N.launch_count(); once(); kernels = N.launch_count() - k0
    med_dev, med_host = float(np.median(t_dev)), float(np.median(t_host))
    return {"p_hit": p_hit, "spans": ns, "out_bytes": need,
            "device": {"msgs_per_s": n / med_dev, "ms_median": med_dev * 1e3, "ms_min": min(t_dev) * 1e3, "ms_max": max(t_dev) * 1e3,
                       "kernels_per_call": kernels, "iters": iters},
            "host": {"msgs_per_s": n / med_host, "ms_median": med_host * 1e3, "last_scan_ms_median": float(np.median(scan_ms)),
                     "scan_share": float(np.median(scan_ms)) / (med_host * 1e3), "iters": len(t_host)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--msgs", type=int, default=1 << 18)
    ap.add_argument("--len", type=int, default=256)
    ap.add_argument("--rules", type=int, default=500)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("redact_device.py needs a CUDA device")
    from vainplex_openclaw_b200 import _native as N, workload as W
    N.init(0)
    rl = W.make_rules(a.rules)
    rs = N.Ruleset(W.rules_as_tuples(rl), strict=True)
    res = [measure(N, torch, rs, rl, a.msgs, a.len, p, a.iters) for p in (0.01, 0.10)]
    print(json.dumps({"workload": {"rules": a.rules, "msg_bytes": a.len, "msgs": a.msgs}, "card": card(), "results": res}))
    rs.close()


if __name__ == "__main__":
    main()
