"""GPU tier of the device-resident Merkle log calls: appends from HBM (ragged and fixed-size), the root, proofs, consistency
proofs and batched verification into HBM, each against the oracle and its host twin; device and host appends interleaved on
one log across the fold's switch points; the in-band answers for what only the device can check (indices past the tree,
over-long paths, decreasing offsets) leaving the other items alone; a log that took a decreasing offset pair reporting it
once at join and refusing every call after; argument checks before anything is enqueued; launch counts as the host plan
restates them (test_merkle_device_cpu); and the per-log issue order across streams, observed through a gated stream as in
test_gpu_streams.  Run on an H100: pytest -m gpu."""
from types import SimpleNamespace

import numpy as np
import pytest

from test_gpu_merkle_proofs import LARGE_CHUNKS, edge_indices, ragged, unpack
from test_merkle_device_cpu import append_device_launches, append_host_launches, proofs_device_launches, verify_device_launches

pytestmark = pytest.mark.gpu
GATE = 200_000_000                      # torch.cuda._sleep cycles: at least 0.1 s at the H100's top clock (test_gpu_streams)
GUARD = 0xAB
NOT_IN_TREE = 0xFFFFFFFF                # the length of the path of an index past the tree


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


@pytest.fixture(scope="module")
def torch():
    import torch as T
    return T


def dev(torch, arr):
    t = torch.from_numpy(np.ascontiguousarray(arr)).cuda()
    torch.cuda.synchronize()
    return t


def host(t, dtype):
    return t.cpu().numpy().view(dtype)


def launches(N, call):
    k0 = N.launch_count()
    out = call()
    return N.launch_count() - k0, out


def make_log(N, kind):
    return N.MerkleLog.tree() if kind == "tree" else N.MerkleLog(keep_leaf_digests=(kind == "keep"))


def frontier_want(oracle, data, off, n):
    """the oracle's roots of the perfect subtrees of the first n leaves, largest first"""
    out, a = [], 0
    for h in reversed(range(n.bit_length())):
        if n >> h & 1:
            out.append(oracle.merkle_root(data, off[a:a + (1 << h) + 1]))
            a += 1 << h
    return out


def check_log(oracle, log, data, off, size):
    log.join()
    assert log.size() == size
    assert log.root() == oracle.merkle_root(data, off[:size + 1]), size
    assert [x.tobytes() for x in log.frontier()] == frontier_want(oracle, data, off, size), size


def expect_gov_error(N, code, call):
    with pytest.raises(N.GovError) as e:
        call()
    assert e.value.code == code, e.value


# ------------------------------------------------------------------------------ appends

@pytest.mark.parametrize("kind", ["tree", "keep", "plain"])
def test_device_and_host_appends_interleave_on_one_log(N, torch, oracle, kind):
    """LARGE_CHUNKS (blocks from 1 to 2^17 leaves, across the fold's 2^15 switch) of ragged leaves of 0..200 bytes, device and
    host appends alternating: root and frontier equal the oracle's after every append, and each append launches what the
    host plan says"""
    rng = np.random.default_rng(11)
    data, off, _ = ragged(rng, sum(LARGE_CHUNKS), 0, 200)
    d_data, d_off = dev(torch, data), dev(torch, off)
    log = make_log(N, kind)
    size = 0
    try:
        for k, m in enumerate(LARGE_CHUNKS):
            sub = off[size:size + m + 1]
            if (k % 2 == 0) == (kind != "keep"):
                got, _ = launches(N, lambda: log.append_device(d_data.data_ptr(), d_off.data_ptr() + 8 * size, m))
                assert got == append_device_launches(size, m), (size, m)
            else:
                got, _ = launches(N, lambda: log.append_packed(data, sub))
                assert got == append_host_launches(size, m, int(sub[-1] - sub[0])), (size, m)
            size += m
            check_log(oracle, log, data, off, size)
    finally:
        log.close()


def test_ragged_leaves_at_every_alignment_from_a_fresh_allocation(N, torch, oracle):
    """every length 0..200 at every start alignment mod 16 (filler leaves in between), the first leaves at offset 0 of an
    allocation of its own (nothing readable in front of it), appended from HBM in one call and in two calls around a host
    append: the oracle's root; a single leaf at offset 0 as well"""
    lens, pos = [], 0
    for L in range(201):
        for a in range(16):
            pad = (a - pos) % 16
            if pad:
                lens.append(pad)
                pos += pad
            lens.append(L)
            pos += L
    off = np.zeros(len(lens) + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    assert lens[:2] == [0, 1] and int(off[1]) == 0              # an empty leaf and a one-byte leaf, both at offset 0
    torch.cuda.empty_cache()
    buf = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")   # larger than any cached block: a fresh segment
    data = np.random.default_rng(12).integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    buf[:len(data)].copy_(torch.from_numpy(data))
    d_off = dev(torch, off)
    torch.cuda.synchronize()
    m = len(lens)
    for split in (None, m // 3):
        log = N.MerkleLog.tree()
        try:
            if split is None:
                log.append_device(buf.data_ptr(), d_off.data_ptr(), m)
            else:
                log.append_device(buf.data_ptr(), d_off.data_ptr(), split)
                log.append_packed(data, off[split:split + 2])
                log.append_device(buf.data_ptr(), d_off.data_ptr() + 8 * (split + 1), m - split - 1)
            check_log(oracle, log, data, off, m)
        finally:
            log.close()
    one = np.array([0, 100], dtype=np.uint64)
    d_one = dev(torch, one)
    log = N.MerkleLog(keep_leaf_digests=False)
    try:
        log.append_device(buf.data_ptr(), d_one.data_ptr(), 1)
        check_log(oracle, log, data, one, 1)
    finally:
        log.close()


@pytest.mark.parametrize("leaf_len", [32, 13, 0])
def test_fixed_size_appends_from_hbm(N, torch, oracle, leaf_len):
    """C4-shaped 32-byte records (the word kernel), 13-byte leaves (the byte kernel) and empty leaves, appended in pieces: the
    oracle's root over every prefix, the launches of the host plan"""
    chunks = [16, 1008, 4096, 33344, 3]
    n = sum(chunks)
    data = np.random.default_rng(leaf_len).integers(0, 256, n * leaf_len + 64, dtype=np.uint8)
    d_data = dev(torch, data)
    log = N.MerkleLog.tree()
    size = 0
    try:
        for m in chunks:
            got, _ = launches(N, lambda: log.append_fixed_device(d_data.data_ptr() + size * leaf_len, leaf_len, m))
            assert got == append_device_launches(size, m)
            size += m
            log.join()
            assert log.root() == oracle.merkle_root_fixed(data, leaf_len, size), size
    finally:
        log.close()


def test_fixed_size_appends_at_any_alignment(N, torch, oracle):
    """fixed-size leaves need no alignment, as for cg_merkle_block_roots_device: 32-byte records from 4-byte and 1-byte aligned
    addresses (the word and the byte kernel) give the oracle's root"""
    data = np.random.default_rng(23).integers(0, 256, 4096 * 32 + 64, dtype=np.uint8)
    d_data = dev(torch, data)
    for start in (4, 3):
        log = N.MerkleLog.tree()
        try:
            log.append_fixed_device(d_data.data_ptr() + start, 32, 1000)
            log.append_fixed_device(d_data.data_ptr() + start + 1000 * 32, 32, 3000)
            log.join()
            assert log.root() == oracle.merkle_root_fixed(data[start:].copy(), 32, 4000), start
        finally:
            log.close()


def test_root_device_equals_the_host_root(N, torch, oracle):
    """the empty log's root (SHA-256 of nothing) and the root after each append, into HBM at an odd address"""
    log = N.MerkleLog.tree()
    out = torch.full((64,), GUARD, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(13)
    try:
        for m in (0, 1, 2, 5, 100):
            if m:
                log.append([rng.integers(0, 256, int(rng.integers(0, 90)), dtype=np.uint8).tobytes() for _ in range(m)])
            log.root_device(out.data_ptr() + 3)
            log.join()
            got = host(out, np.uint8)
            assert got[3:35].tobytes() == log.root() and (got[:3] == GUARD).all() and (got[35:] == GUARD).all()
    finally:
        log.close()


# ------------------------------------------------------------------------------ proofs and verification

@pytest.fixture(scope="module")
def trees(N, torch, oracle):
    """two tree logs fed the same LARGE_CHUNKS of ragged leaves, one from HBM and one from host memory; the roots at every
    append boundary"""
    rng = np.random.default_rng(2025)
    data, off, leaves = ragged(rng, sum(LARGE_CHUNKS), 0, 80)
    d_data, d_off = dev(torch, data), dev(torch, off)
    from_hbm, from_host = N.MerkleLog.tree(), N.MerkleLog.tree()
    roots, size = {}, 0
    for m in LARGE_CHUNKS:
        from_hbm.append_device(d_data.data_ptr(), d_off.data_ptr() + 8 * size, m)
        from_host.append_packed(data, off[size:size + m + 1])
        size += m
        roots[size] = oracle.merkle_root(data, off[:size + 1])
    from_hbm.join()
    t = SimpleNamespace(hbm=from_hbm, host=from_host, roots=roots, size=size, data=data, off=off, leaves=leaves)
    yield t
    from_hbm.close()
    from_host.close()


def test_a_log_filled_from_hbm_serves_the_host_filled_logs_proofs(N, trees):
    rng = np.random.default_rng(14)
    for s in trees.roots:
        idx = edge_indices(rng, s, 500)
        assert unpack(*trees.hbm.proofs(idx, tree_size=s)) == unpack(*trees.host.proofs(idx, tree_size=s)), s
        for first in sorted({f for f in (1, 2, s // 3, s - 1, s) if 1 <= f <= s}):
            assert trees.hbm.consistency_between(first, s) == trees.host.consistency_between(first, s), (first, s)


def proofs_device(N, torch, log, idx, s, stride):
    """proofs_device into guard-filled buffers: (launches, paths uint8[m, stride, 32], lens uint32[m])"""
    m = len(idx)
    d_idx = dev(torch, np.ascontiguousarray(idx, dtype=np.uint64))
    d_paths = torch.full((m * stride * 32 + 64,), GUARD, dtype=torch.uint8, device="cuda")
    d_lens = torch.full((m + 4,), -1, dtype=torch.int32, device="cuda")
    k, _ = launches(N, lambda: log.proofs_device(d_idx.data_ptr(), m, s, d_paths.data_ptr(), stride, d_lens.data_ptr()))
    log.join()
    p, lens = host(d_paths, np.uint8), host(d_lens, np.uint32)
    assert (p[m * stride * 32:] == GUARD).all() and (lens[m:] == NOT_IN_TREE).all()
    return k, p[:m * stride * 32].reshape(m, stride, 32), lens[:m]


def test_proofs_device_equal_the_host_twin(N, torch, trees):
    """at every append boundary, edge and random indices with a stride two digests wider than needed: the host twin's paths
    and lengths, the tail of every stride zero, two launches"""
    rng = np.random.default_rng(15)
    for s in sorted(trees.roots) + [3, 4097]:
        idx = edge_indices(rng, s, 3000)
        want_p, want_l = trees.host.proofs(idx, tree_size=s)
        w = want_p.shape[1]
        k, p, lens = proofs_device(N, torch, trees.hbm, idx, s, w + 2)
        assert k == proofs_device_launches(len(idx))
        assert np.array_equal(lens, want_l), s
        assert np.array_equal(p[:, :w], want_p) and not p[:, w:].any(), s


def test_indices_past_the_tree_get_the_in_band_answer(N, torch, trees):
    """indices >= tree_size (one past, far past, 2^64 - 1) among good ones: length 0xffffffff and an all-zero stride for them,
    the host twin's paths for the others"""
    s = 50000
    rng = np.random.default_rng(16)
    idx = rng.integers(0, s, 997).astype(np.uint64)
    bad = np.zeros(len(idx), dtype=bool)
    for j, v in ((0, s), (5, s + 1), (100, trees.size), (500, 2 ** 64 - 1), (996, s)):
        idx[j], bad[j] = v, True
    stride = (s - 1).bit_length()
    k, p, lens = proofs_device(N, torch, trees.hbm, idx, s, stride)
    want_p, want_l = trees.host.proofs(idx[~bad], tree_size=s)
    assert k == 2
    assert (lens[bad] == NOT_IN_TREE).all() and not p[bad].any()
    assert np.array_equal(lens[~bad], want_l) and np.array_equal(p[~bad], want_p)


def test_consistency_between_device_equals_the_host_twin(N, torch, trees):
    rng = np.random.default_rng(17)
    n = trees.size
    pairs = {(1, 1), (1, n), (n, n), (4096, 4097), (4095, 4096), (3, 70000)} | {tuple(sorted(rng.integers(1, n + 1, 2).tolist())) for _ in range(60)}
    d_path = torch.full((66 * 32,), GUARD, dtype=torch.uint8, device="cuda")
    d_len = torch.full((2,), -1, dtype=torch.int32, device="cuda")
    for first, second in sorted(pairs):
        d_path.fill_(GUARD); d_len.fill_(-1)
        want = trees.host.consistency_between(first, second)
        k, _ = launches(N, lambda: trees.hbm.consistency_between_device(first, second, d_path.data_ptr(), 65, d_len.data_ptr()))
        trees.hbm.join()
        got, ln = host(d_path, np.uint8), host(d_len, np.uint32)
        assert k == (2 if want else 0) and ln[0] == len(want) and ln[1] == NOT_IN_TREE, (first, second)
        assert [got[32 * i:32 * i + 32].tobytes() for i in range(len(want))] == want, (first, second)
        assert (got[32 * len(want):] == GUARD).all(), (first, second)


def pack_leaves(leaves):
    off = np.zeros(len(leaves) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in leaves])
    return np.frombuffer(b"".join(leaves) + b"\0" * 64, dtype=np.uint8).copy(), off


def verify_device(N, torch, data, off, idx, s, paths, lens, root, root_offset=0):
    """verify_proofs_device on copies in HBM (the root at an odd address): (launches, ok bool[m])"""
    m = len(idx)
    d_data, d_off, d_idx = dev(torch, data), dev(torch, off), dev(torch, np.ascontiguousarray(idx, dtype=np.uint64))
    d_paths, d_lens = dev(torch, np.ascontiguousarray(paths)), dev(torch, np.ascontiguousarray(lens, dtype=np.uint32))
    d_root = dev(torch, np.frombuffer(b"\0" * root_offset + root, dtype=np.uint8).copy())
    d_ok = torch.full((m + 8,), GUARD, dtype=torch.uint8, device="cuda")
    k, _ = launches(N, lambda: N.merkle_verify_proofs_device(d_data.data_ptr(), d_off.data_ptr(), d_idx.data_ptr(), m, s, d_paths.data_ptr(), paths.shape[1],
                                                             d_lens.data_ptr(), d_root.data_ptr() + root_offset, d_ok.data_ptr()))
    torch.cuda.synchronize()
    ok = host(d_ok, np.uint8)
    assert set(ok[:m].tolist()) <= {0, 1} and (ok[m:] == GUARD).all()
    return k, ok[:m].astype(bool)


@pytest.mark.parametrize("tamper", [False, True])
def test_verify_proofs_device_equals_the_host_twin(N, torch, trees, tamper):
    """proofs of random leaves at every append boundary, as they are or with a flipped path byte, a wrong index, a changed
    leaf or a shortened path in a third of them: the host twin's verdicts, two launches"""
    rng = np.random.default_rng(18 + tamper)
    for s, root in trees.roots.items():
        idx = rng.integers(0, s, 4000).astype(np.uint64)
        paths, lens = trees.host.proofs(idx, tree_size=s)
        leaves = [trees.leaves[int(i)] for i in idx]
        if tamper:
            for j in range(0, len(idx), 3):
                t = rng.integers(0, 4)
                if t == 0 and lens[j]:
                    paths[j, rng.integers(0, lens[j]), rng.integers(0, 32)] ^= 1
                elif t == 1:
                    idx[j] = (int(idx[j]) + 1) % s
                elif t == 2:
                    leaves[j] = leaves[j] + b"x"
                elif lens[j]:
                    lens[j] -= 1
        data, off = pack_leaves(leaves)
        want = N.merkle_verify_proofs((data, off), idx, s, (paths, lens), root)
        k, got = verify_device(N, torch, data, off, idx, s, paths, lens, root, root_offset=5)
        assert k == verify_device_launches(len(idx))
        assert np.array_equal(got, want), s
        assert want.all() != tamper


def test_verify_in_band_rejections_leave_the_other_proofs_alone(N, torch, trees):
    """a path length of 65, one above the stride, an index >= tree_size and a decreasing offset pair each give ok = 0 for that
    proof; every other proof gets the host twin's verdict on its own leaf"""
    s = trees.size
    root = trees.roots[s]
    rng = np.random.default_rng(20)
    m = 600
    idx = rng.integers(0, s, m).astype(np.uint64)
    paths, lens = trees.host.proofs(idx, tree_size=s)
    stride = paths.shape[1]
    wide = np.zeros((m, 70, 32), dtype=np.uint8)
    wide[:, :stride] = paths
    leaves = [trees.leaves[int(i)] for i in idx]
    data, off = pack_leaves(leaves)
    bad = np.zeros(m, dtype=bool)
    lens_dev = lens.copy()
    lens_dev[10], bad[10] = 65, True                         # above 64 (the stride is 70)
    idx_dev = idx.copy()
    idx_dev[20], bad[20] = s, True
    idx_dev[21], bad[21] = 2 ** 64 - 1, True
    j = next(j for j in range(30, m) if off[j] > 0)
    off_dev = off.copy()
    off_dev[j + 1], bad[j] = off[j] - 1, True                # proof j: [off[j], off[j] - 1), and proof j + 1 starts a byte early
    k, got = verify_device(N, torch, data, off_dev, idx_dev, s, wide, lens_dev, root)
    assert k == 2
    assert not got[bad].any()
    # the others on the host twin, each with the leaf its offsets now select (proof 31 starts earlier)
    lv = [data[int(off_dev[j]):int(off_dev[j + 1])].tobytes() if not bad[j] else b"" for j in range(m)]
    want = N.merkle_verify_proofs(lv, np.where(bad, 0, idx_dev).astype(np.uint64), s, (paths, np.where(bad, 0, lens).astype(np.uint32)), root)
    assert np.array_equal(got[~bad], want[~bad])
    assert want[~bad].sum() == (~bad).sum() - 1                # every untouched proof holds; proof j + 1 lost its leaf
    # the stride itself is a bound: a length one above a stride of 3 is rejected before the path is read
    k, got3 = verify_device(N, torch, np.zeros(64, np.uint8), np.zeros(2, np.uint64), np.zeros(1, np.uint64), 16, np.zeros((1, 3, 32), np.uint8),
                            np.array([4], np.uint32), root)
    assert k == 2 and not got3.any()


def test_a_decreasing_offset_pair_poisons_the_log(N, torch, oracle):
    """a device append whose pair 5 decreases: the leaf goes in as the empty leaf (the root enqueued behind it says so), the
    join reports CG_ERR_INVALID_ARG once, and from then on every call on the log is refused"""
    rng = np.random.default_rng(21)
    data, off, leaves = ragged(rng, 64, 1, 40)
    log = N.MerkleLog.tree()
    try:
        log.append(leaves[:10])
        bad = off[10:16].copy()
        bad[5] = bad[4] - 1                                  # leaf 14 = [off[14], off[14] - 1): decreasing
        d_data, d_off = dev(torch, data), dev(torch, bad)
        log.append_device(d_data.data_ptr(), d_off.data_ptr(), 5)
        d_root = torch.zeros(32, dtype=torch.uint8, device="cuda")
        log.root_device(d_root.data_ptr())
        assert log.size() == 15
        torch.cuda.synchronize()
        expect = leaves[:10] + [data[int(bad[j]):int(bad[j + 1])].tobytes() if bad[j + 1] >= bad[j] else b"" for j in range(5)]
        assert expect[14] == b"" and expect[:14] == leaves[:14]
        e_data, e_off = pack_leaves(expect)
        assert host(d_root, np.uint8).tobytes() == oracle.merkle_root(e_data, e_off)
        expect_gov_error(N, -1, log.join)
        d_idx = dev(torch, np.zeros(1, np.uint64))
        d_out = torch.zeros(64 * 32, dtype=torch.uint8, device="cuda")
        for call in (log.join, log.root, lambda: log.append([b"x"]), lambda: log.append_device(d_data.data_ptr(), d_off.data_ptr(), 1),
                     lambda: log.proofs([0]), lambda: log.proofs_device(d_idx.data_ptr(), 1, 1, d_out.data_ptr(), 1, d_out.data_ptr()),
                     lambda: log.root_device(d_root.data_ptr()), log.frontier, lambda: log.reserve(10)):
            expect_gov_error(N, -1, call)
        assert log.size() == 15
    finally:
        log.close()


def test_host_checkable_arguments_fail_before_anything_is_enqueued(N, torch):
    L = N.load()
    log, plain = N.MerkleLog.tree(), N.MerkleLog(keep_leaf_digests=True)
    d = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    base = d.data_ptr()
    off = dev(torch, np.arange(0, 33, dtype=np.uint64))
    try:
        log.append_device(base, off.data_ptr(), 32)
        plain.append_device(base, off.data_ptr(), 32)
        log.join(); plain.join()
        k0 = N.launch_count()
        cases = [
            (-1, lambda: L.cg_merkle_log_append_device(log.handle, base + 1, off.data_ptr(), 4, None)),       # bytes not 16-byte aligned
            (-1, lambda: L.cg_merkle_log_append_device(log.handle, base + 8, off.data_ptr(), 4, None)),
            (-1, lambda: L.cg_merkle_log_append_device(log.handle, base, off.data_ptr() + 4, 4, None)),       # offsets not 8-byte aligned
            (-1, lambda: L.cg_merkle_log_append_device(log.handle, None, off.data_ptr(), 4, None)),
            (-1, lambda: L.cg_merkle_log_append_fixed_device(log.handle, base, 1 << 40, 1 << 30, None)),       # m * leaf_len overflows
            (-1, lambda: L.cg_merkle_log_root_device(log.handle, None, None)),
            (-5, lambda: L.cg_merkle_log_proofs_device(plain.handle, base, 1, 32, base, 5, base, None)),      # no node store
            (-1, lambda: L.cg_merkle_log_proofs_device(log.handle, base, 1, 33, base, 6, base, None)),        # tree_size past the log
            (-1, lambda: L.cg_merkle_log_proofs_device(log.handle, base, 1, 0, base, 6, base, None)),
            (-7, lambda: L.cg_merkle_log_proofs_device(log.handle, base, 1, 32, base, 4, base, None)),        # stride < ceil(log2 32)
            (-1, lambda: L.cg_merkle_log_proofs_device(log.handle, base, 1, 32, base + 8, 5, base, None)),    # paths not 16-byte aligned
            (-1, lambda: L.cg_merkle_log_proofs_device(log.handle, base + 4, 1, 32, base, 5, base, None)),    # indices not 8-byte aligned
            (-1, lambda: L.cg_merkle_log_proofs_device(log.handle, base, 1, 32, base, 5, base + 2, None)),    # lengths not 4-byte aligned
            (-5, lambda: L.cg_merkle_log_consistency_between_device(plain.handle, 1, 32, base, 8, base, None)),
            (-1, lambda: L.cg_merkle_log_consistency_between_device(log.handle, 5, 4, base, 8, base, None)),
            (-7, lambda: L.cg_merkle_log_consistency_between_device(log.handle, 3, 32, base, 1, base, None)),
            (-1, lambda: L.cg_merkle_log_consistency_between_device(log.handle, 3, 32, base + 16, 8, base + 1, None)),
            (-1, lambda: L.cg_merkle_verify_proofs_device(base + 1, off.data_ptr(), base, 1, 1, base, 1, base, base, base, None)),
            (-1, lambda: L.cg_merkle_verify_proofs_device(base, off.data_ptr(), base, 1, 1, base + 8, 1, base, base, base, None)),
            (-1, lambda: L.cg_merkle_verify_proofs_device(base, off.data_ptr(), base, 1, 1, base, 1, base, None, base, None)),
        ]
        for j, (code, call) in enumerate(cases):
            assert call() == code, j
        assert N.launch_count() == k0 and log.size() == 32
        assert L.cg_merkle_log_append_device(log.handle, None, None, 0, None) == 0                           # m = 0: nothing to do
        assert L.cg_merkle_log_proofs_device(log.handle, None, 0, 32, None, 0, None, None) == 0
        assert L.cg_merkle_verify_proofs_device(None, None, None, 0, 1, None, 0, None, None, None, None) == 0
        log.join()
    finally:
        log.close()
        plain.close()


# ------------------------------------------------------------------------------ streams

def test_calls_on_one_log_run_in_issue_order_across_streams(N, torch, oracle):
    """With reserved capacity a device append behind a gated stream returns while the gate holds; calls on another log (device
    and host) return while it still holds; a host root on the same log returns after it.  Behind a second gate, a device
    proof call on the same log on another stream runs after the append.  Every result equals the oracle's."""
    rng = np.random.default_rng(22)
    data, off, leaves = ragged(rng, 3000, 0, 100)
    d_data, d_off = dev(torch, data), dev(torch, off)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    A, B = N.MerkleLog.tree(), N.MerkleLog.tree()
    d_idx = dev(torch, np.arange(0, 2500, 7, dtype=np.uint64))
    m, stride = d_idx.numel(), 12
    d_paths = torch.zeros(m * stride * 32, dtype=torch.uint8, device="cuda")
    d_lens = torch.zeros(m, dtype=torch.int32, device="cuda")

    def gate():
        with torch.cuda.stream(s1):
            torch.cuda._sleep(GATE)
    try:
        for log in (A, B):
            log.reserve(4000)
            log.append_device(d_data.data_ptr(), d_off.data_ptr(), 1000, s1.cuda_stream)     # (first calls: the kernels are loaded)
            log.proofs_device(d_idx.data_ptr(), 100, 1000, d_paths.data_ptr(), stride, d_lens.data_ptr(), s1.cuda_stream)
            log.join(s1.cuda_stream)
        torch.cuda.synchronize()
        gate()
        A.append_device(d_data.data_ptr(), d_off.data_ptr() + 8 * 1000, 1000, s1.cuda_stream)
        pending = [("device append behind the gate", s1.query())]
        B.append_device(d_data.data_ptr(), d_off.data_ptr() + 8 * 1000, 1000, s2.cuda_stream)
        s2.synchronize()
        pending.append(("device append on another log", s1.query()))
        b_root = B.root()
        pending.append(("host root of another log", s1.query()))
        a_root = A.root()
        root_after = s1.query()
        assert not [what for what, done in pending if done], "returned only after the gate: %s" % pending
        assert root_after, "the host root returned before the append issued first on the log had run"
        want = oracle.merkle_root(data, off[:2001])
        assert a_root == want and b_root == want
        torch.cuda.synchronize()
        gate()
        A.append_device(d_data.data_ptr(), d_off.data_ptr() + 8 * 2000, 500, s1.cuda_stream)
        gated = not s1.query()
        A.proofs_device(d_idx.data_ptr(), m, 2500, d_paths.data_ptr(), stride, d_lens.data_ptr(), s2.cuda_stream)
        s2.synchronize()
        proofs_after = s1.query()
        A.join(s1.cuda_stream)
        assert gated and proofs_after, "a device proof call on another stream ran before the append issued first on the log"
        lens = host(d_lens, np.uint32)
        p = host(d_paths, np.uint8).reshape(m, stride, 32)
        idx = host(d_idx, np.uint64)
        want_p, want_l = A.proofs(idx, tree_size=2500)
        assert np.array_equal(lens, want_l) and np.array_equal(p[:, :want_p.shape[1]], want_p)
        assert unpack(want_p, want_l)[3] == oracle.merkle_audit_path(leaves[:2500], int(idx[3]))
        assert A.root() == oracle.merkle_root(data, off[:2501])
    finally:
        A.close()
        B.close()


def test_an_empty_logs_device_root_leaves_the_librarys_staging_alone(N, torch, oracle):
    """the root of an empty log behind a gated stream s1, then cg_merkle_root and a host append on another log, whose offsets go
    through the library's staging on its stream: both return while the gate holds, every root equals the oracle's, and the
    empty log's root is SHA-256 of nothing"""
    rng = np.random.default_rng(24)
    data, off, _ = ragged(rng, 300, 1, 90)                  # (no empty leaf: a zeroed offsets pair would show)
    s1 = torch.cuda.Stream()
    empty, other = N.MerkleLog.tree(), N.MerkleLog.tree()
    d_root = torch.full((32,), GUARD, dtype=torch.uint8, device="cuda")
    try:
        empty.root_device(d_root.data_ptr(), s1.cuda_stream)
        empty.join(s1.cuda_stream)
        N.merkle_root(data, off)
        torch.cuda.synchronize()
        d_root.fill_(GUARD)
        torch.cuda.synchronize()
        with torch.cuda.stream(s1):
            torch.cuda._sleep(GATE)
        empty.root_device(d_root.data_ptr(), s1.cuda_stream)
        root = N.merkle_root(data, off)
        other.append_packed(data, off)
        other_root = other.root()
        pending = not s1.query()
        empty.join(s1.cuda_stream)
        want = oracle.merkle_root(data, off)
        assert root == want and other_root == want
        assert host(d_root, np.uint8).tobytes() == oracle.sha256(b"")
        assert pending, "a call that shares nothing with the empty log's root waited for it"
    finally:
        empty.close()
        other.close()
