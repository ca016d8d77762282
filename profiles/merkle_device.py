"""The Merkle log's device-resident calls beside their host-buffer twins, on the same card in one run.

  append_ragged  --leaves ragged leaves (64..320 bytes) into a fresh tree log with capacity reserved: cg_merkle_log_append from
                 pinned host memory vs cg_merkle_log_append_device from HBM (+ cg_merkle_log_join), alternated
  append_c4      the same count of 32-byte records (bench.py's C4 shape): cg_merkle_log_append with uniform offsets from pinned
                 memory vs cg_merkle_log_append_fixed_device
  proofs         --proofs random indices at the full size of the ragged log: cg_merkle_log_proofs into pinned buffers vs
                 cg_merkle_log_proofs_device into HBM
  verify         the same proofs: cg_merkle_verify_proofs from pinned buffers vs cg_merkle_verify_proofs_device from HBM
Per call: the median over --reps of the host clock around a call that ends with the results in place (the host twins
synchronise; a device call is followed by a join or a stream synchronise), for the device twins the median of CUDA events
around the call on its stream, and for each twin its kernels' device time (torch.profiler, one call).  Results are checked:
equal roots, equal path bytes and lengths, every verdict 1 on both sides.  Prints one JSON line with the card's name, power
limit and max SM clock read in the same run.  Needs an H100; writes nothing.

    python profiles/merkle_device.py [--leaves 16777216] [--proofs 1048576] [--reps 5]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from profiles.merkle_proofs import kernel_ms  # noqa: E402
from profiles.redact_device import card  # noqa: E402


def timed(torch, fn, stream=None):
    """(host ms, event ms on stream or None) of one call of fn; fn leaves its results in place before it returns"""
    if stream is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
    t0 = time.perf_counter()
    fn()
    if stream is not None:
        e1.record(stream)
        e1.synchronize()
    return (time.perf_counter() - t0) * 1e3, (e0.elapsed_time(e1) if stream is not None else None)


def summary(samples):
    host = [h for h, _ in samples]
    ev = [e for _, e in samples if e is not None]
    out = {"call_ms": float(np.median(host))}
    if ev:
        out["event_ms"] = float(np.median(ev))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--leaves", type=int, default=1 << 24)
    ap.add_argument("--proofs", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    from vainplex_openclaw_b200 import _native as N
    N.init(0)
    lib = N.load()
    n, m, reps = args.leaves, args.proofs, args.reps
    s = torch.cuda.Stream()
    st = s.cuda_stream
    g = torch.Generator(device="cuda").manual_seed(42)
    lens = torch.randint(64, 321, (n,), device="cuda", generator=g)
    d_off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    d_off[1:] = torch.cumsum(lens, 0)
    total = int(d_off[-1])
    d_bytes = torch.randint(0, 256, (total + 64,), dtype=torch.uint8, device="cuda", generator=g)
    h_bytes = torch.empty(total + 64, dtype=torch.uint8, pin_memory=True); h_bytes.copy_(d_bytes)
    h_off = torch.empty(n + 1, dtype=torch.int64, pin_memory=True); h_off.copy_(d_off)
    d_c4 = torch.randint(0, 256, (n * 32 + 64,), dtype=torch.uint8, device="cuda", generator=g)
    h_c4 = torch.empty(n * 32 + 64, dtype=torch.uint8, pin_memory=True); h_c4.copy_(d_c4)
    h_c4_off = torch.arange(0, 32 * (n + 1), 32, dtype=torch.int64).pin_memory()
    torch.cuda.synchronize()
    res = {"card": card(), "leaves": n, "proofs": m, "reps": reps}

    def fresh(nbytes):
        lg = N.MerkleLog.tree()
        lg.reserve(n, nbytes + 64)
        torch.cuda.synchronize()
        return lg

    def append_pair(label, nbytes, host_call, device_call, names):
        samples, roots, keep = {"host": [], "device": []}, {}, None
        for r in range(reps + 1):                              # (the first round warms up)
            for kind in ("host", "device"):
                lg = fresh(nbytes)
                if kind == "host":
                    t = timed(torch, lambda: host_call(lg))
                else:
                    t = timed(torch, lambda: (device_call(lg), lg.join(st)), s)
                if r:
                    samples[kind].append(t)
                roots[kind] = lg.root()
                if kind == "device" and r == reps:
                    keep = lg
                else:
                    lg.close()
        assert roots["host"] == roots["device"], label
        out = {k: summary(v) for k, v in samples.items()}
        lg = fresh(nbytes)
        out["host"]["kernel_ms"] = kernel_ms(torch, lambda: host_call(lg), names)
        lg.close()
        lg = fresh(nbytes)
        out["device"]["kernel_ms"] = kernel_ms(torch, lambda: (device_call(lg), lg.join(st)), names)
        lg.close()
        out["leaves_per_s"] = {k: n / out[k]["call_ms"] * 1e3 for k in ("host", "device")}
        return out, keep

    absorb = ["merkle_reduce_kernel", "merkle_level_kernel", "merkle_chain_kernel"]
    res["append_ragged"], tree = append_pair(
        "ragged", total,
        lambda lg: N.check(lib.cg_merkle_log_append(lg.handle, h_bytes.data_ptr(), h_off.data_ptr(), n)),
        lambda lg: lg.append_device(d_bytes.data_ptr(), d_off.data_ptr(), n, st),
        ["merkle_leaves_var_kernel", "merkle_leaves_guarded_kernel"] + absorb)
    res["append_ragged"]["leaf_bytes"] = {"lengths": "64..320", "total": total}
    res["append_c4"], c4 = append_pair(
        "c4", 32 * n,
        lambda lg: N.check(lib.cg_merkle_log_append(lg.handle, h_c4.data_ptr(), h_c4_off.data_ptr(), n)),
        lambda lg: lg.append_fixed_device(d_c4.data_ptr(), 32, n, st),
        ["merkle_leaves_var_kernel", "merkle_leaves_fixed_kernel"] + absorb)
    c4.close()

    # proofs at the full size of the ragged log
    size = tree.size()
    stride = (size - 1).bit_length()
    d_idx = torch.randint(0, size, (m,), dtype=torch.int64, device="cuda", generator=g)
    h_idx = torch.empty(m, dtype=torch.int64, pin_memory=True); h_idx.copy_(d_idx)
    h_paths = torch.empty(m * stride * 32, dtype=torch.uint8, pin_memory=True)
    h_lens = torch.empty(m, dtype=torch.int32, pin_memory=True)
    d_paths = torch.empty(m * stride * 32, dtype=torch.uint8, device="cuda")
    d_lens = torch.empty(m, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def host_proofs():
        N.check(lib.cg_merkle_log_proofs(tree.handle, h_idx.data_ptr(), m, size, h_paths.data_ptr(), stride, h_lens.data_ptr()))

    def device_proofs():
        tree.proofs_device(d_idx.data_ptr(), m, size, d_paths.data_ptr(), stride, d_lens.data_ptr(), st)

    host_proofs(); device_proofs(); s.synchronize()
    assert torch.equal(h_paths.cuda(), d_paths) and torch.equal(h_lens.cuda(), d_lens)
    res["proofs"] = {"tree_size": size, "stride": stride, "path_bytes": m * stride * 32,
                     "host": summary([timed(torch, host_proofs) for _ in range(reps)]),
                     "device": summary([timed(torch, device_proofs, s) for _ in range(reps)])}
    names = ["merkle_gather_kernel", "merkle_gather_checked_kernel", "merkle_chain_kernel"]
    res["proofs"]["host"]["kernel_ms"] = kernel_ms(torch, host_proofs, names)
    res["proofs"]["device"]["kernel_ms"] = kernel_ms(torch, device_proofs, names)

    # verify the same proofs: their leaves packed on the device
    starts, ln = d_off[:-1][d_idx], lens[d_idx]
    d_voff = torch.zeros(m + 1, dtype=torch.int64, device="cuda")
    d_voff[1:] = torch.cumsum(ln, 0)
    vtotal = int(d_voff[-1])
    pos = torch.arange(vtotal, device="cuda") - torch.repeat_interleave(d_voff[:-1], ln) + torch.repeat_interleave(starts, ln)
    d_vbytes = torch.zeros(vtotal + 64, dtype=torch.uint8, device="cuda")
    d_vbytes[:vtotal] = d_bytes[pos]
    del pos
    d_root = torch.from_numpy(np.frombuffer(tree.root(), dtype=np.uint8).copy()).cuda()
    h_vbytes = torch.empty(vtotal + 64, dtype=torch.uint8, pin_memory=True); h_vbytes.copy_(d_vbytes)
    h_voff = torch.empty(m + 1, dtype=torch.int64, pin_memory=True); h_voff.copy_(d_voff)
    h_root = d_root.cpu().numpy().copy()
    h_ok = torch.empty(m, dtype=torch.uint8, pin_memory=True)
    d_ok = torch.empty(m, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def host_verify():
        N.check(lib.cg_merkle_verify_proofs(h_vbytes.data_ptr(), h_voff.data_ptr(), h_idx.data_ptr(), m, size, h_paths.data_ptr(), stride,
                                            h_lens.data_ptr(), h_root.ctypes.data, h_ok.data_ptr()))

    def device_verify():
        N.merkle_verify_proofs_device(d_vbytes.data_ptr(), d_voff.data_ptr(), d_idx.data_ptr(), m, size, d_paths.data_ptr(), stride,
                                      d_lens.data_ptr(), d_root.data_ptr(), d_ok.data_ptr(), st)

    host_verify(); device_verify(); s.synchronize()
    assert bool((h_ok == 1).all()) and bool((d_ok == 1).all())
    res["verify"] = {"tree_size": size, "leaf_bytes": vtotal,
                     "host": summary([timed(torch, host_verify) for _ in range(reps)]),
                     "device": summary([timed(torch, device_verify, s) for _ in range(reps)])}
    names = ["merkle_leaves_var_kernel", "merkle_leaves_guarded_kernel", "merkle_verify_batch_kernel", "merkle_verify_checked_kernel"]
    res["verify"]["host"]["kernel_ms"] = kernel_ms(torch, host_verify, names)
    res["verify"]["device"]["kernel_ms"] = kernel_ms(torch, device_verify, names)
    tree.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
