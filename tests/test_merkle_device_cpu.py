"""CPU tier of the device-resident Merkle log calls: they are declared, exported and bound; before cg_init they return
CG_ERR_NOT_INITIALIZED; and the launches each one enqueues, restated here from the host's plan (log_absorb's block cuts and
launch_merkle_fold's steps in csrc/capi.cu and csrc/sha256_kernels.cu), so that the GPU tier can hold the library to them:
  append:  one leaf launch, then the host twin's fold and chain launches (the host twin hashes its leaves in up to eight
           pieces, to overlap their copies);
  proofs:  the spine (one chain launch), then the gather;
  verify:  the leaves, then the verifier.
No device needed."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NEW_CALLS = ("cg_merkle_log_append_device", "cg_merkle_log_append_fixed_device", "cg_merkle_log_root_device", "cg_merkle_log_proofs_device",
             "cg_merkle_log_consistency_between_device", "cg_merkle_verify_proofs_device", "cg_merkle_log_join")
COPY_CHUNKS, CHUNKED_ABOVE = 8, 4 << 20      # Ctx::kChunks; a host append of more leaf bytes than this copies them in pieces


def absorb_blocks(n, m):
    """log_absorb's cut of leaves [n, n + m) into aligned perfect blocks: (position, size), each size at most the lowest set
    bit of its position"""
    out, pos, rem = [], n, m
    while rem:
        s = (pos & -pos) if pos else 1 << 63
        while s > rem:
            s >>= 1
        out.append((pos, s))
        pos += s
        rem -= s
    return out


def fold_launches(n):
    """launch_merkle_fold of n nodes to one: one launch per merkle_level_kernel level above 2^15 nodes, then
    merkle_reduce_kernel launches of up to five levels each"""
    k, lv = 0, 0
    while n > 1:
        step = 1
        if n <= 1 << 15:
            step = min(5, 64 - lv)
            while step > 1 and (1 << (step - 1)) >= n:
                step -= 1
        k += 1
        n = (n + (1 << step) - 1) >> step
        lv += step
    return k


def absorb_launches(n, m):
    """fold and chain launches of absorbing m leaves into a log of n: per block its fold, and one chain launch when the block
    carries into an occupied frontier slot (else a device copy)"""
    k = 0
    for pos, s in absorb_blocks(n, m):
        h = s.bit_length() - 1
        k += fold_launches(s) + (1 if (pos >> h) & 1 else 0)
    return k


def host_leaf_launches(m, leaf_bytes):
    """cg_merkle_log_append's leaf launches: one per non-empty piece of the copy"""
    c = COPY_CHUNKS if leaf_bytes > CHUNKED_ABOVE else 1
    per = (m + c - 1) // c
    return len([i for i in range(c) if min(i * per, m) < min((i + 1) * per, m)])


def append_device_launches(n, m):
    return (1 + absorb_launches(n, m)) if m else 0


def append_host_launches(n, m, leaf_bytes):
    return (host_leaf_launches(m, leaf_bytes) + absorb_launches(n, m)) if m else 0


def proofs_device_launches(m):
    return 2 if m else 0


def verify_device_launches(m):
    return 2 if m else 0


def test_blocks_cover_the_append_with_aligned_perfect_subtrees():
    for n in range(0, 300):
        for m in range(0, 70):
            blocks = absorb_blocks(n, m)
            assert sum(s for _, s in blocks) == m
            pos = n
            for p, s in blocks:
                assert p == pos and s & (s - 1) == 0 and p % s == 0
                pos += s


def test_fold_launches_follow_the_switch_at_two_to_the_fifteen():
    assert [fold_launches(s) for s in (1, 2, 32, 33, 1 << 10, 1 << 15)] == [0, 1, 1, 2, 2, 3]
    for k in range(16, 30):
        assert fold_launches(1 << k) == (k - 15) + 3         # one level launch per level above 2^15, then 5 + 5 + 5 levels


def test_one_leaf_at_a_time_chains_exactly_on_odd_sizes():
    for n in range(0, 1 << 12):
        assert absorb_launches(n, 1) == (n & 1)
        assert append_device_launches(n, 1) == 1 + (n & 1)


def test_device_append_saves_the_host_twins_extra_leaf_launches():
    for n, m in ((0, 1), (5, 4095), (4096, 32768), (12345, 131073), (1 << 20, 1 << 16)):
        assert append_host_launches(n, m, 0) == append_device_launches(n, m)
        assert append_host_launches(n, m, 16 << 20) - append_device_launches(n, m) == min(COPY_CHUNKS, m) - 1


def test_device_calls_are_declared_exported_and_bound():
    from vainplex_openclaw_b200 import _native as N
    hdr = open(os.path.join(ROOT, "include", "openclaw_gov.h")).read()
    for name in NEW_CALLS:
        assert re.search(r"CG_API\s+int\s+%s\s*\(" % name, hdr), name
        assert name in N.EXPORTS, name
    for meth in ("append_device", "append_fixed_device", "root_device", "proofs_device", "consistency_between_device", "join"):
        assert callable(getattr(N.MerkleLog, meth)), meth
    assert callable(N.merkle_verify_proofs_device)
    L = N.load()
    assert all(hasattr(L, name) for name in NEW_CALLS)


def test_device_calls_need_init():
    """before cg_init every new call returns CG_ERR_NOT_INITIALIZED (in a fresh process: no device is touched)"""
    code = ("import ctypes as C\nfrom vainplex_openclaw_b200 import _native as N\nL = N.load()\n"
            "print(L.cg_merkle_log_append_device(None, None, None, 1, None), L.cg_merkle_log_append_fixed_device(None, None, 32, 1, None),\n"
            "      L.cg_merkle_log_root_device(None, None, None), L.cg_merkle_log_proofs_device(None, None, 1, 1, None, 1, None, None),\n"
            "      L.cg_merkle_log_consistency_between_device(None, 1, 1, None, 1, None, None),\n"
            "      L.cg_merkle_verify_proofs_device(None, None, None, 1, 1, None, 0, None, None, None, None), L.cg_merkle_log_join(None, None))\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["-2"] * len(NEW_CALLS)
