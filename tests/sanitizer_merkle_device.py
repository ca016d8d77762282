"""Workload for a compute-sanitizer run over the device-resident Merkle log calls (not collected by pytest): the guarded leaf
kernel on leaves that start at offset 0 of an allocation of their own and end at its last byte plus the 16 readable bytes
the call asks for, and on a decreasing offset pair; the checked gather with indices past the tree; the checked verifier with
over-long path lengths, an index past the tree and a decreasing pair.  PyTorch's caching allocator is switched off, so
that every buffer is an allocation of its own and memcheck sees a read past its end.  Usage:
  PYTORCH_NO_CUDA_MEMORY_CACHING=1 compute-sanitizer --tool memcheck --error-exitcode 3 python tests/sanitizer_merkle_device.py"""
import os
import sys

os.environ.setdefault("PYTORCH_NO_CUDA_MEMORY_CACHING", "1")       # (before torch is imported)
import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vainplex_openclaw_b200 import _native as N  # noqa: E402

N.init(0)
rng = np.random.default_rng(9)
lens = rng.integers(0, 120, 3000)
off = np.zeros(len(lens) + 1, dtype=np.uint64)
off[1:] = np.cumsum(lens)
data = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
d_data = torch.from_numpy(data).cuda()                        # exactly the bytes the call may read (one cudaMalloc)
d_off = torch.from_numpy(off.view(np.int64)).cuda()
log = N.MerkleLog.tree()
log.append_device(d_data.data_ptr(), d_off.data_ptr(), 1000)
log.append_packed(data, off[1000:2001])
log.append_device(d_data.data_ptr(), d_off.data_ptr() + 8 * 2000, 1000)
log.join()
want = N.merkle_root(data, off)
assert log.root() == want

size, m = log.size(), 500
idx = rng.integers(0, size, m).astype(np.uint64)
idx[::50] = size + np.arange(10, dtype=np.uint64)               # past the tree
stride = (size - 1).bit_length()
d_idx = torch.from_numpy(idx.view(np.int64)).cuda()
d_paths = torch.empty(m * stride * 32, dtype=torch.uint8, device="cuda")
d_lens = torch.empty(m, dtype=torch.int32, device="cuda")
log.proofs_device(d_idx.data_ptr(), m, size, d_paths.data_ptr(), stride, d_lens.data_ptr())
log.join()
lens_h = d_lens.cpu().numpy().view(np.uint32)
assert (lens_h[::50] == 0xFFFFFFFF).all()

good = np.where(lens_h != 0xFFFFFFFF, idx, 0).astype(np.uint64)
leaves = [data[int(off[i]):int(off[i + 1])].tobytes() for i in good]
voff = np.zeros(m + 1, dtype=np.uint64)
voff[1:] = np.cumsum([len(x) for x in leaves])
vbytes = np.frombuffer(b"".join(leaves) + b"\0" * 16, dtype=np.uint8).copy()
voff[101] = voff[100] - 1 if voff[100] else 0                  # a decreasing pair (or an empty leaf)
lens_v = np.where(lens_h == 0xFFFFFFFF, 0, lens_h).astype(np.uint32)
lens_v[7], lens_v[8] = 65, stride + 1                         # over-long paths
idx_v = good.copy()
idx_v[9] = size
d_vbytes = torch.from_numpy(vbytes).cuda()
d_voff = torch.from_numpy(voff.view(np.int64)).cuda()
d_vidx = torch.from_numpy(idx_v.view(np.int64)).cuda()
d_vlens = torch.from_numpy(lens_v.view(np.int32)).cuda()
d_root = torch.from_numpy(np.frombuffer(want, dtype=np.uint8).copy()).cuda()
d_ok = torch.empty(m, dtype=torch.uint8, device="cuda")
N.merkle_verify_proofs_device(d_vbytes.data_ptr(), d_voff.data_ptr(), d_vidx.data_ptr(), m, size, d_paths.data_ptr(), stride, d_vlens.data_ptr(),
                              d_root.data_ptr(), d_ok.data_ptr())
torch.cuda.synchronize()
ok = d_ok.cpu().numpy()
assert not ok[[7, 8, 9]].any() and ok[1:7].all()

bad = N.MerkleLog(keep_leaf_digests=False)                    # a decreasing pair in an append: hashed without a read
boff = np.array([0, 10, 4, 20], dtype=np.uint64)
d_boff = torch.from_numpy(boff.view(np.int64)).cuda()
bad.append_device(d_data.data_ptr(), d_boff.data_ptr(), 3)
try:
    bad.join()
    raise SystemExit("the decreasing pair was not reported")
except N.GovError as e:
    assert e.code == -1
bad.close()
log.close()
print("ok", size, int(ok.sum()))
