"""Proofs from a log that keeps its complete subtree nodes (cg_merkle_log_create_tree), beside the plain log.

On a --leaves-leaf log (ragged 64..320-byte leaves, pinned host memory, 16 appends, capacity reserved up front):
  append       leaves/s of a tree log and of a keep_leaf_digests = 1 log, alternated, median over --reps
  proofs       cg_merkle_log_proofs for --proofs random indices at the current size and at an earlier size (pinned output
               buffers): median call time over --reps calls, and the device time of the gather kernel (torch.profiler)
  one_by_one   cg_merkle_log_proof on the plain log (re-folds every sibling range) and on the tree log, --sample calls each
  verify       cg_merkle_verify_proofs for the same --proofs proofs: median call time, and the device time of the leaf and
               verify kernels
Every call's results are checked: proofs against the plain log's on a sample, every verdict 1.  Prints one JSON line with
the card's name, power limit and max SM clock read in the same run.  Needs an H100; writes nothing.

    python profiles/merkle_proofs.py [--leaves 16777216] [--proofs 1048576] [--reps 5] [--sample 16]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from profiles.redact_device import card  # noqa: E402


def median_ms(fn, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def kernel_ms(torch, fn, names):
    """device time of the named kernels in one call of fn (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for n in names:
            if n in ev.key:
                out[n] = out.get(n, 0.0) + ev.device_time_total / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--leaves", type=int, default=1 << 24)
    ap.add_argument("--proofs", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=16)
    args = ap.parse_args()
    import torch
    from vainplex_openclaw_b200 import _native as N
    N.init(0)
    lib = N.load()
    n, m = args.leaves, args.proofs
    rng = np.random.default_rng(42)
    lens = rng.integers(64, 321, n).astype(np.uint64)
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    h_bytes = torch.randint(0, 256, (int(offs[-1]) + 64,), dtype=torch.uint8).pin_memory()
    h_offs = torch.from_numpy(offs.view(np.int64)).pin_memory()
    per = n // 16

    def build(make):
        lg = make()
        lg.reserve(n, per * 320 + 64)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for c in range(16):
            N.check(lib.cg_merkle_log_append(lg.handle, h_bytes.data_ptr(), h_offs.data_ptr() + 8 * c * per, per))
        return lg, time.perf_counter() - t0

    append = {"tree": [], "plain": []}
    tree = plain = None
    for r in range(args.reps):
        for kind, make in (("tree", N.MerkleLog.tree), ("plain", lambda: N.MerkleLog(keep_leaf_digests=True))):
            lg, dt = build(make)
            append[kind].append(16 * per / dt)
            if r == args.reps - 1:
                if kind == "tree":
                    tree = lg
                else:
                    plain = lg
            else:
                lg.close()
    size = 16 * per
    assert tree.root() == plain.root() and np.array_equal(tree.frontier(), plain.frontier())
    res = {"card": card(), "leaves": size, "leaf_bytes": "ragged 64..320", "host_memory": "pinned",
           "append_leaves_per_s": {k: float(np.median(v)) for k, v in append.items()}}
    res["append_overhead_of_the_store"] = 1.0 - res["append_leaves_per_s"]["tree"] / res["append_leaves_per_s"]["plain"]

    earlier = size * 5 // 8 + 12345
    proofs = {}
    idx_all = {}
    for label, s in (("current", size), ("earlier", earlier)):
        stride = (s - 1).bit_length()
        idx = torch.from_numpy(rng.integers(0, s, m).astype(np.int64)).pin_memory()
        paths = torch.empty(m * stride * 32, dtype=torch.uint8).pin_memory()
        plens = torch.empty(m, dtype=torch.int32).pin_memory()

        def call():
            N.check(lib.cg_merkle_log_proofs(tree.handle, idx.data_ptr(), m, s, paths.data_ptr(), stride, plens.data_ptr()))
        call()
        ms = median_ms(call, args.reps)
        kern = kernel_ms(torch, call, ["merkle_gather_kernel", "merkle_chain_kernel"])
        proofs[label] = {"tree_size": s, "proofs": m, "stride": stride, "call_ms": ms, "proofs_per_s_call": m / ms * 1e3,
                         "d2h_bytes": m * stride * 32 + 4 * m, "kernel_ms": kern,
                         "proofs_per_s_gather_kernel": m / kern.get("merkle_gather_kernel", float("nan")) * 1e3}
        idx_all[label] = (s, idx, paths, plens, stride)
    res["proofs"] = proofs

    # one at a time: the plain log re-folds every sibling range, the tree log gathers
    s, idx, paths, plens, stride = idx_all["current"]
    sample = idx.numpy()[:args.sample].astype(np.uint64).tolist()
    P = paths.numpy().reshape(m, stride, 32)
    L_ = plens.numpy()
    for j, i in enumerate(sample[:4]):
        assert plain.proof(i) == [P[j, k].tobytes() for k in range(int(L_[j]))], i
    plain.proof(sample[0]); tree.proof(sample[0])
    t = {"plain": [], "tree": []}
    for i in sample:
        for kind, lg in (("plain", plain), ("tree", tree)):
            t0 = time.perf_counter(); lg.proof(i); t[kind].append((time.perf_counter() - t0) * 1e3)
    res["one_by_one_ms"] = {k: float(np.median(v)) for k, v in t.items()}
    res["one_by_one_calls"] = len(sample)

    # verify the current-size proofs in one call
    idx_np = idx.numpy().astype(np.uint64)
    vo = np.zeros(m + 1, dtype=np.uint64)
    vo[1:] = np.cumsum(lens[idx_np])
    hb = h_bytes.numpy()
    starts = offs[idx_np].astype(np.int64)
    gather = np.concatenate([np.arange(a, a + int(ln)) for a, ln in zip(starts[: min(m, 1 << 20)], lens[idx_np][: min(m, 1 << 20)])]) if m else np.zeros(0, dtype=np.int64)
    vbytes = torch.empty(int(vo[-1]) + 64, dtype=torch.uint8).pin_memory()
    vbytes.numpy()[:int(vo[-1])] = hb[gather]
    voffs = torch.from_numpy(vo.view(np.int64)).pin_memory()
    root = np.frombuffer(tree.root(), dtype=np.uint8).copy()
    ok = torch.empty(m, dtype=torch.uint8).pin_memory()

    def vcall():
        N.check(lib.cg_merkle_verify_proofs(vbytes.data_ptr(), voffs.data_ptr(), idx.data_ptr(), m, s, paths.data_ptr(), stride,
                                            plens.data_ptr(), root.ctypes.data, ok.data_ptr()))
    vcall()
    assert bool((ok.numpy() == 1).all())
    vms = median_ms(vcall, args.reps)
    vk = kernel_ms(torch, vcall, ["merkle_verify_batch_kernel", "merkle_leaves_var_kernel"])
    res["verify"] = {"proofs": m, "tree_size": s, "call_ms": vms, "proofs_per_s_call": m / vms * 1e3,
                     "h2d_bytes": int(vo[-1]) + m * stride * 32 + 12 * m, "kernel_ms": vk,
                     "proofs_per_s_verify_kernel": m / vk.get("merkle_verify_batch_kernel", float("nan")) * 1e3,
                     "node_hashes_per_proof_mean": float(L_.mean())}
    tree.close(); plain.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
