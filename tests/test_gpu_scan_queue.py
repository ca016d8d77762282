"""GPU tier: the scan step's head check, flag-word queue and tile dealing.  The head check of the scanned range runs in
confirm_kernel, scan_kernel's warps append to the flag-word queue 128 entries at a time, and tiles are dealt to the grid's
warps CTA-interleaved.  Each case is compared with the CPU oracle.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from test_gpu_boundaries import LITS, R_AT, R_OK, device_words, hit_pairs, sm_count
from test_gpu_parity import oracle_policy

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


def lowercase_text(rng, length):
    t = rng.integers(ord("a"), ord("z") + 1, length).astype(np.uint8)
    t[rng.random(length) < 0.15] = ord(" ")
    return t


@pytest.mark.parametrize("rules,options,stride", [(LITS + [R_OK], 2, 2), (LITS + [R_AT], 4, 4)], ids=["stride2", "stride4"])
def test_factor_at_the_head_of_the_range(N, oracle, rules, options, stride):
    """A factor that starts 0, 1 or 2 bytes into the scanned range has no gram in front of it: the head check finds it, on
    the host path, the device path and scan_one, whether the batch starts at buffer offset 0 or further in."""
    rs = N.Ruleset(rules, options=options, strict=True)
    assert rs.info().stride == stride
    rng = np.random.default_rng(stride)
    for k in (0, 1, 2):
        for tok in (b"alphabetagamma", b"ZEPPELIN_Airship", b"bob@example" if stride == 4 else b"ok"):
            head = b"." * k + tok + b" " + bytes(lowercase_text(rng, 40))
            msgs = [head] + [bytes(lowercase_text(rng, int(rng.integers(0, 300)))) for _ in range(40)]
            data, off = N.pack(msgs)
            ewords, ehits = oracle_policy(oracle, rules, data, off)
            assert int(ewords[0]) >> 63, (k, tok)
            words, hits = rs.scan_batch(data, off)
            assert np.array_equal(words, ewords) and hit_pairs(hits) == ehits, (k, tok)
            assert np.array_equal(device_words(N, rs, data, off), ewords), (k, tok)
            w1, _ = rs.scan_one(head)
            assert w1 == int(ewords[0]), (k, tok)
            # the same messages behind a skipped first message: the scanned range starts at off[1], not at 0
            skip = bytes(lowercase_text(rng, 48 + k))
            d2, o2 = N.pack([skip] + msgs)
            ew2, _ = oracle_policy(oracle, rules, d2, o2)
            o_in = o2[1:].copy()
            ew_in = ew2[1:]
            words2, _ = rs.scan_batch(d2, o_in)
            assert np.array_equal(words2, ew_in), (k, tok)
            assert np.array_equal(device_words(N, rs, d2, o_in), ew_in), (k, tok)
    rs.close()


def test_flag_queue_overflow_grows_and_recovers(N, oracle):
    """A fresh rule set sized by a small batch, then a batch in which nearly every lane flags a word every round: the flag
    queue runs past its capacity, every word of that batch says "incomplete", cg_scan_join reports
    CG_ERR_CAPACITY once, and the batch scanned again (the scratch has grown) equals the oracle."""
    import torch
    rules = LITS + [R_OK]
    rs = N.Ruleset(rules, options=2, strict=True)
    rng = np.random.default_rng(77)
    st = torch.cuda.Stream()
    small = [bytes(lowercase_text(rng, 200)) for _ in range(64)]
    # rule-literal fragments end to end: grams of the literals in every 16-byte chunk
    frags = [b"alphabet", b"betagamma", b"quickbrown", b"brownfox", b"zeppelin", b"airship", b"ok", b"thequick"]
    n, length = 48, 1 << 17
    big = []
    for i in range(n):
        parts, size = [], 0
        while size < length:
            p = frags[int(rng.integers(0, len(frags)))] + (b" " if rng.random() < 0.5 else b"")
            parts.append(p); size += len(p)
        big.append(b"".join(parts)[:length])
    outs = []
    for msgs in (small, big):
        data, off = N.pack(msgs)
        dd = torch.from_numpy(np.ascontiguousarray(data)).cuda()
        oo = torch.from_numpy(off.astype(np.int32)).cuda()
        out = torch.zeros(len(msgs), dtype=torch.int64, device="cuda")
        rs.scan_batch_device(dd.data_ptr(), oo.data_ptr(), len(msgs), out.data_ptr(), st.cuda_stream)
        outs.append((data, off, dd, oo, out))
    with pytest.raises(N.GovError) as ei:
        rs.scan_join(st.cuda_stream)
    assert ei.value.code == N.CG_ERR_CAPACITY
    data, off, dd, oo, out = outs[1]
    assert (out.cpu().numpy().view(np.uint64) == np.uint64(0xffffffffffffffff)).all()
    rs.scan_batch_device(dd.data_ptr(), oo.data_ptr(), n, out.data_ptr(), st.cuda_stream)
    rs.scan_join(st.cuda_stream)                                       # (complete now: no error)
    words = out.cpu().numpy().view(np.uint64)
    ewords, _ = oracle_policy(oracle, rules, data, off)
    assert np.array_equal(words, ewords)
    assert rs.work_counters()[8] > 65536                              # real flag words: more than the first capacity
    hw, _ = rs.scan_batch(data, off)
    assert np.array_equal(hw, ewords)
    rs.close()


@pytest.mark.parametrize("extra", [1, 31, 33])
@pytest.mark.parametrize("rules,options,stride", [(LITS + [R_OK], 2, 2), (LITS + [R_AT], 4, 4)], ids=["stride2", "stride4"])
def test_tiles_left_over_after_the_last_full_round(N, oracle, rules, options, stride, extra):
    """Batches whose 1 KB tile count is one round of every warp of the grid plus 1, 31 or 33 tiles (a round is two tiles at
    stride 2, four at stride 4): tokens in the left-over tiles, at their edges and on the last byte are found, on the host
    and the device path."""
    rs = N.Ruleset(rules, options=options, strict=True)
    assert rs.info().stride == stride
    warps = sm_count() * 32
    tiles = (2 if stride == 2 else 4) * warps + extra
    total = tiles * 1024 - 5
    rng = np.random.default_rng(1000 * stride + extra)
    flat = lowercase_text(rng, total)
    toks = [b" alphabetagamma ", b" thequickbrownfox ", b" ZEPPELIN_Airship ", b" ok " if stride == 2 else b" bob@x "]
    tail = (extra + 2) * 1024
    places = list(range(total - tail, total - 40, 700)) + [int(p) for p in rng.integers(0, total - tail, 200)]
    places += [t * 1024 - 6 for t in range(tiles - extra - 1, tiles)]                   # across the left-over tiles' edges
    for p in places:
        tok = toks[int(rng.integers(0, len(toks)))]
        flat[p:p + len(tok)] = np.frombuffer(tok, dtype=np.uint8)
    end = toks[0].strip()
    flat[total - len(end):] = np.frombuffer(end, dtype=np.uint8)                        # a token on the last byte
    n = 4096
    cuts = np.sort(rng.choice(np.arange(1, total - 64), n - 1, replace=False))
    off = np.concatenate([[0], cuts, [total]]).astype(np.uint32)
    data = np.concatenate([flat, np.zeros(64, np.uint8)])
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    assert int(ewords[-1]) >> 63
    words, hits = rs.scan_batch(data, off)
    assert np.array_equal(words, ewords) and hit_pairs(hits) == ehits
    assert np.array_equal(device_words(N, rs, data, off), ewords)
    rs.close()
