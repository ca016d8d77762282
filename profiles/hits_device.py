"""Hit lists from HBM (cg_scan_hits_batch_device) beside the words-only device call (cg_scan_batch_device) and the
host-buffer call (cg_scan_batch) with and without its hit list.

The C2 shape: 500 rules, 256-byte messages, 1 Mi messages, p_hit 1 % and 10 %.
  device: host clock around enqueue + cg_scan_join, many iterations after warm-up, inputs and outputs in HBM, and the
          kernels each call launches
  host:   host clock around cg_scan_batch from pinned host buffers, words only (out_hits = NULL) and with the hit list
Prints one JSON line with the card's name, power limit and max SM clock read in the same run.  Needs an H100; writes nothing.

    python profiles/hits_device.py [--msgs 1048576] [--iters 20]
"""
import argparse
import ctypes as C
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


def timed(fn, iters):
    for _ in range(3):
        fn()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return t


def summary(n, t, **extra):
    med = float(np.median(t))
    return dict({"msgs_per_s": n / med, "ms_median": med * 1e3, "ms_min": min(t) * 1e3, "ms_max": max(t) * 1e3, "iters": len(t)}, **extra)


def measure(N, torch, rs, rl, n, L, p_hit, iters):
    from vainplex_openclaw_b200 import workload as W
    data_t, off_t, _ = W.make_messages(n, L, rl, p_hit=p_hit, seed=1234)
    h_data = torch.empty(data_t.numel(), dtype=torch.uint8, pin_memory=True); h_data.copy_(data_t)
    h_off = torch.empty(n + 1, dtype=torch.int32, pin_memory=True); h_off.copy_(off_t)
    h_words = torch.empty(n, dtype=torch.int64, pin_memory=True)
    lib = N.load()
    # host-buffer call: words only, then with the hit list (room for every hit)
    nh = C.c_uint32(0)
    N.check(lib.cg_scan_batch(rs.handle, h_data.data_ptr(), h_off.data_ptr(), n, h_words.data_ptr(), None, 0, C.byref(nh)))
    total = nh.value
    h_hits = torch.empty(2 * max(total, 1), dtype=torch.int32, pin_memory=True)
    t_host_words = timed(lambda: N.check(lib.cg_scan_batch(rs.handle, h_data.data_ptr(), h_off.data_ptr(), n, h_words.data_ptr(), None, 0, C.byref(nh))), max(3, iters // 4))
    t_host_hits = timed(lambda: N.check(lib.cg_scan_batch(rs.handle, h_data.data_ptr(), h_off.data_ptr(), n, h_words.data_ptr(), h_hits.data_ptr(), total, C.byref(nh))), max(3, iters // 4))
    host_pairs = h_hits.numpy().view(np.uint32)[:2 * total].copy()
    # device-resident calls
    d, o = h_data.cuda(), h_off.cuda()
    d_words = torch.empty(n, dtype=torch.int64, device="cuda")
    d_hits = torch.empty(2 * max(total, 1), dtype=torch.int32, device="cuda")
    d_nh = torch.empty(1, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    torch.cuda.synchronize()

    def words_once():
        rs.scan_batch_device(d.data_ptr(), o.data_ptr(), n, d_words.data_ptr(), st.cuda_stream)
        rs.scan_join(st.cuda_stream)

    def hits_once():
        rs.scan_hits_batch_device(d.data_ptr(), o.data_ptr(), n, d_words.data_ptr(), d_hits.data_ptr(), total, d_nh.data_ptr(), st.cuda_stream)
        rs.scan_join(st.cuda_stream)

    t_words = timed(words_once, iters)
    k0 = N.launch_count(); words_once(); k_words = N.launch_count() - k0
    t_hits = timed(hits_once, iters)
    k0 = N.launch_count(); hits_once(); k_hits = N.launch_count() - k0
    assert (int(d_nh.item()) & 0xffffffff) == total, "device hit count differs from the host call"
    assert np.array_equal(d_hits.cpu().numpy().view(np.uint32)[:2 * total], host_pairs), "device hit list differs from the host call"
    return {"p_hit": p_hit, "hits": total,
            "device": {"scan_batch_device": summary(n, t_words, kernels_per_call=k_words),
                       "scan_hits_batch_device": summary(n, t_hits, kernels_per_call=k_hits),
                       "hits_extra_ms_median": (float(np.median(t_hits)) - float(np.median(t_words))) * 1e3},
            "host": {"scan_batch_words_only": summary(n, t_host_words), "scan_batch_with_hits": summary(n, t_host_hits)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--msgs", type=int, default=1 << 20)
    ap.add_argument("--len", type=int, default=256)
    ap.add_argument("--rules", type=int, default=500)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("hits_device.py needs a CUDA device")
    from vainplex_openclaw_b200 import _native as N, workload as W
    N.init(0)
    rl = W.make_rules(a.rules)
    rs = N.Ruleset(W.rules_as_tuples(rl), strict=True)
    res = [measure(N, torch, rs, rl, a.msgs, a.len, p, a.iters) for p in (0.01, 0.10)]
    print(json.dumps({"workload": {"rules": a.rules, "msg_bytes": a.len, "msgs": a.msgs}, "card": card(), "results": res}))
    rs.close()


if __name__ == "__main__":
    main()
