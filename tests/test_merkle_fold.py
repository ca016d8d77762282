"""GPU tier, how the Merkle calls fold their trees: the number of kernels each entry point launches (leaf kernel plus the
fold's step rule), that cg_merkle_fold_device only reads its input, and that the sharded root gives the same answer call
after call and after cg_comm_destroy.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu

NS = [1, 2, 3, 31, 32, 33, (1 << 15) - 1, 1 << 15, (1 << 15) + 1, (1 << 15) + (1 << 14), 200001]
BLOCK_LOG2S = [0, 1, 5, 6, 16, 40]


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


def fold_launches(n, max_levels=64):
    """the fold's step rule: above 2^15 nodes one level per launch, else min(5, levels left under max_levels, ceil(log2 n))
    levels per launch; it stops at one node or after max_levels levels"""
    k = lv = 0
    while n > 1 and lv < max_levels:
        step = 1 if n > 1 << 15 else min(5, max_levels - lv, (n - 1).bit_length())
        n = (n + (1 << step) - 1) >> step
        lv += step
        k += 1
    return k


def absorb_launches(size, m):
    """a log append of m leaf digests to a log of `size` leaves: the aligned perfect blocks it is cut into are folded, and a
    block that lands on an occupied frontier slot is carried by one chain launch"""
    k, pos, rem = 0, size, m
    while rem:
        s = pos & -pos if pos else 1 << 63
        while s > rem:
            s >>= 1
        k += fold_launches(s)
        k += (pos >> (s.bit_length() - 1)) & 1
        pos += s
        rem -= s
    return k


def proof_ranges(index, size):
    """RFC 6962 2.1.1: the leaf ranges of the sibling subtrees on the way down to leaf `index`"""
    out, lo, hi = [], 0, size
    while hi - lo > 1:
        k = 1 << ((hi - lo - 1).bit_length() - 1)
        if index < lo + k:
            out.append((lo + k, hi)); hi = lo + k
        else:
            out.append((lo, lo + k)); lo += k
    return out


def launches(N, call):
    k0 = N.launch_count()
    out = call()
    return N.launch_count() - k0, out


@pytest.mark.parametrize("n", NS)
def test_merkle_entry_points_launch_the_leaf_kernel_and_the_fold_rule(N, n):
    """every one-shot Merkle call launches one leaf kernel (when it hashes leaves) plus what the step rule gives for its tree;
    all of them agree on the root"""
    import torch
    L = N.load()
    data = W.make_leaves(n, 32, seed=n).numpy()
    off = np.arange(n + 1, dtype=np.uint64) * 32
    k, root = launches(N, lambda: N.merkle_root_fixed(data, 32, n))
    assert k == 1 + fold_launches(n)
    k, r = launches(N, lambda: N.merkle_root(data, off))
    assert k == 1 + fold_launches(n) and r == root

    nodes = np.random.default_rng(n).integers(0, 256, (n, 32), dtype=np.uint8)
    k, froot = launches(N, lambda: N.merkle_fold(nodes))
    assert k == fold_launches(n)
    d_nodes = torch.from_numpy(nodes.reshape(-1)).cuda()
    d_out = torch.zeros(32, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    k, _ = launches(N, lambda: N.check(L.cg_merkle_fold_device(d_nodes.data_ptr(), n, d_out.data_ptr(), None)))
    torch.cuda.synchronize()
    assert k == fold_launches(n) and d_out.cpu().numpy().tobytes() == froot

    d_leaves = torch.from_numpy(data).cuda()
    stream = torch.cuda.Stream()
    for bl in BLOCK_LOG2S:
        nb = (n + (1 << bl) - 1) >> bl
        roots = torch.zeros(nb * 32, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        k, _ = launches(N, lambda: N.check(L.cg_merkle_block_roots_device(d_leaves.data_ptr(), 32, n, bl, roots.data_ptr(), stream.cuda_stream)))
        assert k == 1 + fold_launches(n, bl), bl
        k, r = launches(N, lambda: N.merkle_root_sharded_device(d_leaves.data_ptr(), 32, n, n, bl, stream.cuda_stream))
        assert k == 1 + fold_launches(n, bl) + fold_launches(nb) and r == root, bl
    torch.cuda.synchronize()


def test_merkle_empty_trees_launch_one_hash(N):
    """the empty tree's root is SHA-256 of nothing, one launch of the batch kernel, whichever call asks for it"""
    import torch
    d = torch.zeros(64, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for call in (lambda: N.merkle_root_fixed(np.zeros(64, dtype=np.uint8), 32, 0), lambda: N.merkle_fold(np.zeros((0, 32), dtype=np.uint8)),
                 lambda: N.merkle_root_sharded_device(d.data_ptr(), 32, 0, 0, 4)):
        assert launches(N, call)[0] == 1


@pytest.mark.parametrize("sizes", [[1], [5], [33, 31], [(1 << 15) + (1 << 14), 3], [1 << 15, (1 << 15) + 1, 2]])
def test_merkle_log_append_and_proof_launches(N, sizes):
    """a log append launches one leaf kernel plus, for every aligned block its leaves are cut into, the block's fold and a chain
    launch where the block carries into the frontier; an audit path folds every sibling range"""
    log = N.MerkleLog(keep_leaf_digests=True)
    try:
        size = 0
        for m in sizes:
            data = W.make_leaves(m, 32, seed=size + m).numpy()
            off = np.arange(m + 1, dtype=np.uint64) * 32
            k, _ = launches(N, lambda: log.append_packed(data, off))
            assert k == 1 + absorb_launches(size, m), (size, m)
            size += m
        for index in sorted({0, size // 2, size - 1}):
            k, path = launches(N, lambda: log.proof(index))
            ranges = proof_ranges(index, size)
            assert len(path) == len(ranges) and k == sum(fold_launches(hi - lo) for lo, hi in ranges), index
    finally:
        log.close()


@pytest.mark.parametrize("m", [1, 2, 33, 40000])
def test_merkle_fold_device_leaves_its_input_untouched(N, m):
    """cg_merkle_fold_device reads its nodes in place and writes none of them, from an aligned pointer and from one that is
    4 bytes off the 16-byte alignment of the kernels' loads; its root equals the host fold's"""
    import torch
    L = N.load()
    nodes = np.random.default_rng(m).integers(0, 256, m * 32, dtype=np.uint8)
    want = N.merkle_fold(nodes.reshape(m, 32))
    stream = torch.cuda.Stream()
    for shift in (0, 4):
        buf = torch.zeros(m * 32 + 16, dtype=torch.uint8, device="cuda")
        buf[shift:shift + m * 32] = torch.from_numpy(nodes).cuda()
        before = buf.cpu().numpy()
        out = torch.zeros(32, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        N.check(L.cg_merkle_fold_device(buf.data_ptr() + shift, m, out.data_ptr(), stream.cuda_stream))
        torch.cuda.synchronize()
        assert np.array_equal(buf.cpu().numpy(), before), shift
        assert out.cpu().numpy().tobytes() == want, shift


def test_merkle_sharded_root_repeats_and_survives_comm_destroy(N):
    """consecutive one-rank sharded roots on one stream give the same root, also when a call needs larger root buffers than
    the one before, and a call after cg_comm_destroy still works"""
    import torch
    n = 100003
    data = W.make_leaves(n, 32, seed=7).numpy()
    root = N.merkle_root_fixed(data, 32, n)
    d = torch.from_numpy(data).cuda()
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    assert [N.merkle_root_sharded_device(d.data_ptr(), 32, n, n, 5, stream.cuda_stream) for _ in range(5)] == [root] * 5
    assert N.merkle_root_sharded_device(d.data_ptr(), 32, n, n, 0, stream.cuda_stream) == root
    N.comm_destroy()
    assert N.merkle_root_sharded_device(d.data_ptr(), 32, n, n, 5, stream.cuda_stream) == root
    assert N.merkle_root_sharded_device(d.data_ptr(), 32, n, n, 16) == root
    with pytest.raises(N.GovError) as ei:                   # leaves without a pointer: an argument error, before any launch
        N.merkle_root_sharded_device(0, 32, n, n, 5)
    assert ei.value.code == -1
