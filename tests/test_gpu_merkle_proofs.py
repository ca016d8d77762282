"""GPU tier, proofs from a log's node store (cg_merkle_log_create_tree): audit paths and consistency proofs at any tree size,
in batches, against the oracle's RFC 6962 recursion and the CT vectors; the store filled across the fold's switch points;
the gather and batch-verify kernels past their grids; batched verification rejecting exactly what the oracle's RFC 9162 walk
rejects; errors before any output byte changes.  Run on an H100: pytest -m gpu."""
import ctypes as C
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GATHER_WARPS, GATHER_BLOCKS_PER_SM = 8, 8              # kGatherWarps, kGatherBlocksPerSm (csrc/kernels.h)
VERIFY_BLOCK, VERIFY_BLOCKS_PER_SM = 128, 16           # kProofVerifyBlock, kProofVerifyBlocksPerSm
LARGE_CHUNKS = [1, 4095, 1, 32768, 12345, 20000, 131073]


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def unpack(paths, lens):
    return [[paths[i, k].tobytes() for k in range(int(lens[i]))] for i in range(len(lens))]


def launches(N, call):
    k0 = N.launch_count()
    out = call()
    return N.launch_count() - k0, out


def ragged(rng, m, lo, hi):
    """m leaves of random lengths in [lo, hi]: (data, off64, list of bytes)"""
    lens = rng.integers(lo, hi + 1, m)
    off = np.zeros(m + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    data = rng.integers(0, 256, int(off[-1]) + 64, dtype=np.uint8)
    return data, off, [data[int(off[i]):int(off[i + 1])].tobytes() for i in range(m)]


def test_small_tree_log_matches_the_oracle_at_every_size(N, oracle):
    """70 leaves appended as 1, 1, 2, 3, 5, 17, 41: for every size s and index i < s the path equals the oracle's, and so does
    every consistency proof (m, s); all of them verify, on the device and in the oracle, against the root of the first s
    leaves (reported by a log fed one leaf at a time; at the append boundaries the tree log reports the same root)."""
    rng = np.random.default_rng(70)
    leaves = [rng.integers(0, 256, int(rng.integers(0, 121)), dtype=np.uint8).tobytes() for _ in range(70)]
    ref = N.MerkleLog(keep_leaf_digests=False)
    roots = {}
    for s in range(1, 71):
        ref.append(leaves[s - 1:s])
        roots[s] = ref.root()
    ref.close()
    log = N.MerkleLog.tree()
    try:
        size = 0
        for m in (1, 1, 2, 3, 5, 17, 41):
            log.append(leaves[size:size + m])
            size += m
            assert log.root() == roots[size] and log.size() == size
        for s in range(1, 71):
            paths, lens = log.proofs(np.arange(s), tree_size=s)
            got = unpack(paths, lens)
            for i in range(s):
                assert got[i] == oracle.merkle_audit_path(leaves[:s], i), (i, s)
                assert oracle.merkle_verify_path(leaves[i], i, s, got[i], roots[s])
            assert N.merkle_verify_proofs(leaves[:s], np.arange(s), s, (paths, lens), roots[s]).all(), s
            for m in range(1, s + 1):
                p = log.consistency_between(m, s)
                assert p == oracle.merkle_consistency_proof(leaves[:s], m), (m, s)
                assert oracle.merkle_verify_consistency(m, s, roots[m], roots[s], p)
                assert N.merkle_verify_consistency(m, s, roots[m], roots[s], p)
    finally:
        log.close()


def test_ct_vectors_from_one_tree_log(N):
    v = json.load(open(os.path.join(HERE, "golden", "ct_merkle_vectors.json")))
    leaves = [bytes.fromhex(x) for x in v["leaves_hex"]]
    roots = [bytes.fromhex(x) for x in v["roots_hex"]]
    log = N.MerkleLog.tree()
    try:
        log.append(leaves)
        assert log.root() == roots[7]
        for c in v["inclusion"]:
            paths, lens = log.proofs([c["index"]], tree_size=c["size"])
            p = unpack(paths, lens)[0]
            assert [x.hex() for x in p] == c["path_hex"], c
            assert N.merkle_verify_proofs([leaves[c["index"]]], [c["index"]], c["size"], [p], roots[c["size"] - 1]).all()
        for c in v["consistency"]:
            assert [x.hex() for x in log.consistency_between(c["first"], c["second"])] == c["path_hex"], c
    finally:
        log.close()


@pytest.fixture(scope="module")
def large(N):
    """a tree log and a keep_leaf_digests = 1 log fed the same appends across the fold's switch points (2^15 nodes, block
    sizes from 1 to 2^17), with every root, frontier and launch count compared after each append"""
    rng = np.random.default_rng(2024)
    total = sum(LARGE_CHUNKS)
    data, off, leaves = ragged(rng, total, 0, 80)
    tree, plain = N.MerkleLog.tree(), N.MerkleLog(keep_leaf_digests=True)
    roots, size = {}, 0
    for m in LARGE_CHUNKS:
        sub = off[size:size + m + 1]
        kt, _ = launches(N, lambda: tree.append_packed(data, sub))
        kp, _ = launches(N, lambda: plain.append_packed(data, sub))
        size += m
        assert kt == kp, size
        assert tree.size() == plain.size() == size
        r = tree.root()
        assert r == plain.root(), size
        assert np.array_equal(tree.frontier(), plain.frontier()), size
        roots[size] = r
    yield {"tree": tree, "plain": plain, "roots": roots, "leaves": leaves, "data": data, "off": off}
    tree.close()
    plain.close()


def edge_indices(rng, s, k=2000):
    idx = set(rng.integers(0, s, k).tolist()) | {0, s - 1}
    for b in range(s.bit_length()):
        idx |= {x for x in ((1 << b) - 1, 1 << b, (1 << b) + 1) if x < s}
    return np.array(sorted(idx), dtype=np.uint64)


def test_large_log_proofs_at_every_recorded_size(N, oracle, large):
    rng = np.random.default_rng(3)
    tree, roots, leaves = large["tree"], large["roots"], large["leaves"]
    for s, root in roots.items():
        idx = edge_indices(rng, s)
        paths, lens = tree.proofs(idx, tree_size=s)
        assert (lens <= max(1, (s - 1).bit_length())).all()
        got = unpack(paths, lens)
        for i, p in zip(idx.tolist(), got):
            assert oracle.merkle_verify_path(leaves[i], i, s, p, root), (i, s)
        assert N.merkle_verify_proofs([leaves[i] for i in idx.tolist()], idx, s, (paths, lens), root).all(), s


def test_large_log_current_size_equals_the_plain_log(N, large):
    """at the current size the batched paths equal cg_merkle_log_proof of the plain log; on the tree log cg_merkle_log_proof
    and cg_merkle_log_consistency return the plain log's bytes (from two launches each)"""
    rng = np.random.default_rng(4)
    tree, plain = large["tree"], large["plain"]
    n = tree.size()
    idx = edge_indices(rng, n, 60)
    got = unpack(*tree.proofs(idx))
    for i, p in zip(idx.tolist(), got):
        want = plain.proof(i)
        assert p == want, i
        k, q = launches(N, lambda: tree.proof(i))
        assert q == want and k == (2 if want else 0), i
    for first in sorted(set(large["roots"]) | {1, 2, 3, 4095, 4096, 4097, 1 << 15, n - 1, n}):
        want = plain.consistency(first)
        k, q = launches(N, lambda: tree.consistency(first))
        assert q == want and k == (2 if want else 0), first
        assert tree.consistency_between(first, n) == want, first


def test_batch_geometry_guards_and_launch_counts(N, large):
    """m around one warp and around one full grid of the gather and the verify kernel: results equal the one-by-one paths,
    nothing is written past out_paths32, out_lens or out_ok, and each call launches two kernels whatever m and n are"""
    L = N.load()
    tree, leaves = large["tree"], large["leaves"]
    sms = sm_count()
    g_gather = sms * GATHER_BLOCKS_PER_SM * GATHER_WARPS
    g_verify = sms * VERIFY_BLOCKS_PER_SM * VERIFY_BLOCK
    rng = np.random.default_rng(5)
    small = N.MerkleLog.tree()
    small.append([b"a", b"b", b"c"])
    try:
        for log, n in ((small, 3), (tree, tree.size())):
            stride = max(1, (n - 1).bit_length())
            for m in sorted({0, 1, 31, 32, 33, g_gather - 1, g_gather, g_gather + 1}):
                idx = rng.integers(0, n, m).astype(np.uint64)
                out = np.full(m * stride * 32 + 64, 0xA5, dtype=np.uint8)
                lens = np.full(m + 4, 0xA5A5A5A5, dtype=np.uint32)
                k, rc = launches(N, lambda: L.cg_merkle_log_proofs(log.handle, idx.ctypes.data, m, n, out.ctypes.data, stride, lens.ctypes.data))
                assert rc == 0 and k == (2 if m else 0), (n, m)
                assert (out[m * stride * 32:] == 0xA5).all() and (lens[m:] == 0xA5A5A5A5).all(), (n, m)
                if m:
                    assert (lens[:m] <= stride).all()
                    for j in sorted({0, m // 2, m - 1}):
                        i = int(idx[j])
                        assert [bytes(x) for x in out[:m * stride * 32].reshape(m, stride, 32)[j, :lens[j]]] == unpack(*log.proofs([i]))[0], (n, m, i)
                        assert not out[:m * stride * 32].reshape(m, stride, 32)[j, lens[j]:].any()
        n = tree.size()
        s = n - 7
        root = np.frombuffer(root_at(N, large, s), dtype=np.uint8).copy()
        for m in sorted({1, 31, 32, 33, g_verify - 1, g_verify, g_verify + 1}):
            idx = rng.integers(0, s, m).astype(np.uint64)
            paths, lens = tree.proofs(idx, tree_size=s)
            data, off = pack64([leaves[i] for i in idx.tolist()])
            ok = np.full(m + 16, 0xA5, dtype=np.uint8)
            k, rc = launches(N, lambda: L.cg_merkle_verify_proofs(data.ctypes.data, off.ctypes.data, idx.ctypes.data, m, s, paths.ctypes.data,
                                                                   paths.shape[1], lens.ctypes.data, root.ctypes.data, ok.ctypes.data))
            assert rc == 0 and k == 2, m
            assert (ok[:m] == 1).all() and (ok[m:] == 0xA5).all(), m
    finally:
        small.close()


def pack64(leaves):
    off = np.zeros(len(leaves) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in leaves])
    return np.frombuffer(b"".join(leaves) + b"\0" * 64, dtype=np.uint8).copy(), off


def root_at(N, large, s):
    """MTH of the first s leaves, from a plain log fed them in one append"""
    lg = N.MerkleLog(keep_leaf_digests=False)
    try:
        lg.append_packed(large["data"], large["off"][:s + 1])
        return lg.root()
    finally:
        lg.close()


def test_batched_verification_rejects_what_the_oracle_rejects(N, oracle, large):
    """100k valid proofs all hold; copies with one change each (a flipped leaf byte, index ^ 1, tree_size +- 1, a path element
    dropped or added, an older root, an index >= tree_size) give the oracle's bit on every copy"""
    tree, leaves, roots = large["tree"], large["leaves"], large["roots"]
    n = tree.size()
    rng = np.random.default_rng(6)
    idx = rng.integers(0, n, 100000).astype(np.uint64)
    paths, lens = tree.proofs(idx)
    root = roots[n]
    assert N.merkle_verify_proofs([leaves[i] for i in idx.tolist()], idx, n, (paths, lens), root).all()

    sel = rng.choice(len(idx), 2048, replace=False)
    base = [(leaves[int(idx[j])], int(idx[j]), [paths[j, k].tobytes() for k in range(int(lens[j]))]) for j in sel]
    older = roots[sorted(roots)[-2]]
    extra = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    variants = {
        "leaf": [(bytes([lf[0] ^ 1]) + lf[1:] if lf else b"\x00", i, p, n, root) for lf, i, p in base],
        "index^1": [(lf, i ^ 1, p, n, root) for lf, i, p in base],
        "size+1": [(lf, i, p, n + 1, root) for lf, i, p in base],
        "size-1": [(lf, i, p, n - 1, root) for lf, i, p in base],
        "dropped": [(lf, i, p[:-1], n, root) for lf, i, p in base],
        "added": [(lf, i, p + [extra], n, root) for lf, i, p in base],
        "older root": [(lf, i, p, n, older) for lf, i, p in base],
        "index>=size": [(lf, n + i % 3, p, n, root) for lf, i, p in base],
    }
    for name, items in variants.items():
        by_size = {}
        for k, it in enumerate(items):
            by_size.setdefault((it[3], it[4]), []).append(k)
        got = np.zeros(len(items), dtype=bool)
        for (s, r), ks in by_size.items():
            got[ks] = N.merkle_verify_proofs([items[k][0] for k in ks], [items[k][1] for k in ks], s, [items[k][2] for k in ks], r)
        want = np.array([oracle.merkle_verify_path(lf, i, s, p, r) for lf, i, p, s, r in items], dtype=bool)
        assert np.array_equal(got, want), name


def test_verification_over_every_leaf_length_and_start_offset(N, oracle):
    """leaves of every length 0..200, each batch starting k = 0..15 bytes into the staging buffer: all proofs hold, and a flipped
    last byte makes every non-empty one fail"""
    leaves = [bytes((7 * j + L) & 0xFF for j in range(L)) for L in range(201)]
    log = N.MerkleLog.tree()
    try:
        log.append(leaves)
        n, root = len(leaves), log.root()
        paths, lens = log.proofs(np.arange(n))
        for k in range(16):
            off = np.zeros(n + 1, dtype=np.uint64)
            off[1:] = np.cumsum([len(x) for x in leaves])
            off += k
            data = np.frombuffer(b"\xee" * k + b"".join(leaves) + b"\0" * 64, dtype=np.uint8).copy()
            assert N.merkle_verify_proofs((data, off), np.arange(n), n, (paths, lens), root).all(), k
            bad = data.copy()
            bad[off[1:].astype(np.int64) - 1] ^= 1                                 # last byte of every leaf (the byte before, for the empty one)
            got = N.merkle_verify_proofs((bad, off), np.arange(n), n, (paths, lens), root)
            want = [oracle.merkle_verify_path(bad[int(off[i]):int(off[i + 1])].tobytes(), i, n, unpack(paths[i:i + 1], lens[i:i + 1])[0], root)
                    for i in range(n)]
            assert got.tolist() == want, k
            assert not got[1:].any(), k
    finally:
        log.close()


def test_errors_come_before_any_output(N):
    L = N.load()
    tree = N.MerkleLog.tree()
    tree.append([b"x%d" % i for i in range(10)])
    plain = N.MerkleLog(keep_leaf_digests=True)
    plain.append([b"y"] * 4)
    nokeep = N.MerkleLog(keep_leaf_digests=False)
    nokeep.append([b"z"] * 4)
    restored = N.MerkleLog.restore(10, tree.frontier())
    try:
        def proofs(log, idx, s, stride):
            idx = np.array(idx, dtype=np.uint64)
            out = np.full(len(idx) * max(stride, 1) * 32 + 32, 0x5A, dtype=np.uint8)
            lens = np.full(len(idx) + 1, 7, dtype=np.uint32)
            k, rc = launches(N, lambda: L.cg_merkle_log_proofs(log.handle, idx.ctypes.data, len(idx), s, out.ctypes.data, stride, lens.ctypes.data))
            assert (out == 0x5A).all() and (lens == 7).all() and k == 0
            return rc

        def between(log, a, b, cap):
            out = np.full(65 * 32, 0x5A, dtype=np.uint8)
            ln = C.c_uint32(99)
            k, rc = launches(N, lambda: L.cg_merkle_log_consistency_between(log.handle, a, b, out.ctypes.data, cap, C.byref(ln)))
            assert (out == 0x5A).all() and ln.value == 99 and k == 0
            return rc

        for log in (plain, nokeep, restored):
            assert proofs(log, [0], 4, 8) == N.CG_ERR_UNSUPPORTED
            assert between(log, 1, 4, 64) == N.CG_ERR_UNSUPPORTED
        assert proofs(tree, [0], 0, 8) == -1
        assert proofs(tree, [0], 11, 8) == -1
        assert proofs(tree, [0, 5], 5, 8) == -1                       # an index >= tree_size
        assert proofs(tree, [3], 10, 3) == N.CG_ERR_CAPACITY          # ceil(log2 10) = 4
        assert proofs(tree, [], 10, 4) == 0
        for a, b in ((0, 5), (6, 5), (1, 0), (1, 11)):
            assert between(tree, a, b, 64) == -1, (a, b)
        assert between(tree, 3, 10, 1) == N.CG_ERR_CAPACITY
        ok = np.full(4, 0x5A, dtype=np.uint8)
        lens = np.array([65], dtype=np.uint32)
        paths = np.zeros(65 * 32, dtype=np.uint8)
        idx = np.zeros(1, dtype=np.uint64)
        off = np.array([0, 1], dtype=np.uint64)
        data = np.zeros(64, dtype=np.uint8)
        r = np.zeros(32, dtype=np.uint8)
        assert L.cg_merkle_verify_proofs(data.ctypes.data, off.ctypes.data, idx.ctypes.data, 1, 1, paths.ctypes.data, 65, lens.ctypes.data,
                                         r.ctypes.data, ok.ctypes.data) == -1                # a path longer than 64
        assert (ok == 0x5A).all()
        assert L.cg_merkle_verify_proofs(None, None, None, 0, 1, None, 0, None, None, None) == 0
    finally:
        for lg in (tree, plain, nokeep, restored):
            lg.close()
