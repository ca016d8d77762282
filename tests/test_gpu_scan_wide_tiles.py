"""GPU tier, scan_kernel's warp tiles: a tile is 1 KB made of two 512-byte halves (lane l owns chunk base + l and chunk
base + 32 + l), and lane 31's odd grams of the first half read lane 0's second-half word.  Rule tokens straddle every
512-byte edge of the text -- every tile edge, every half-tile seam, and so every CTA and round edge of the grids of
1, 2 and 3 CTAs the batch sizes get -- and batches end inside a first and inside a second half with a token on their
last byte.  The seam tokens are deterministic: SEAM_SAMPLES rule samples take turns, and each one crosses successive
seams at split points 1, 2, 3, ... of its token, so whichever gram the compiler registered for its factor, a seam puts
that gram on bytes 510..513 of a tile (the gram lane 31 folds from lane 0's second-half word) once the sweep is
complete; a rule's seam tokens are SEAM_SAMPLES KB apart, more than the 5 KB messages of the 80-message batches that
must catch a missed one.  At stride 2 (500 synthetic rules) and stride 4 (the 17 built-ins), words and hit lists of the
host path and words of cg_scan_batch_device equal the oracle's, also for a batch whose off[0] is not 0 and not 16-byte aligned.
Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from test_gpu_boundaries import device_words, filler, hit_pairs, scan_grid, sm_count
from test_gpu_parity import oracle_policy
from vainplex_openclaw_b200 import workload as W

pytestmark = pytest.mark.gpu

TILE, HALF, WARPS = 1024, 512, 32          # bytes per warp tile and per half; warps per scan CTA (1024 threads)
TILES_PER_ROUND = {2: 2, 4: 4}             # one 32-bit flag word per lane and round: 16 probe bits per tile at stride 2, 8 at stride 4
NS = (20, 40, 80)                          # grids of 1, 2 and 3 CTAs
ENDS = (1, 300, 511, 512, 513, 700, 1023, 0)     # batch end mod TILE: inside a first half (1 .. 512), inside a second half
PREFIX = 3 * 16 + 5                        # off[0] of the ragged batch
SEAM_SAMPLES = 12                          # rule samples the half-tile seams take turns with


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


class Text:
    """filler text with a rule token across every 512-byte edge; each batch cuts it into n messages whose last one is
    short, so that the oracle's answers for the first n - 1 messages are computed once per n"""

    def __init__(self, oracle, rl, rules, total, seed):
        self.rng = np.random.default_rng(seed)
        self.oracle, self.rules = oracle, rules
        self.samples = [r["sample"].encode() for r in rl]
        self.flat = filler(rl, total, seed)
        busy = np.zeros(total, dtype=bool)
        seam_rules = self.rng.permutation(len(self.samples))[:SEAM_SAMPLES]
        self.seam_splits = {int(r): set() for r in seam_rules}          # rule -> split points its seam tokens took
        self.seams = {int(r): 0 for r in seam_rules}                     # rule -> seams it crossed
        for b in range(HALF, total - 4096, HALF):
            if b % TILE:                                                   # a half-tile seam: the next split point of the next sample
                k = b // TILE
                r = int(seam_rules[k % len(seam_rules)])
                tok = b" " + self.samples[r] + b" "
                split = 1 + (k // len(seam_rules)) % (len(tok) - 1)
                self.seam_splits[r].add(split)
                self.seams[r] += 1
            else:
                tok = b" " + self.samples[int(self.rng.integers(0, len(self.samples)))] + b" "
                split = int(self.rng.integers(1, len(tok)))
            at = b - split
            assert not busy[at:at + len(tok)].any()
            self.flat[at:at + len(tok)] = np.frombuffer(tok, dtype=np.uint8)
            busy[at:at + len(tok)] = True
        self.free = np.nonzero(~busy[1:total - 4096])[0] + 1          # cut positions that split no token
        self.last_cut = total - 3072
        self.base = {}

    def head(self, n):
        """the first n - 1 messages (cut points, oracle words and hits), shared by every batch of n messages"""
        if n not in self.base:
            cand = self.free[self.free < self.last_cut]
            cuts = np.sort(self.rng.choice(cand, n - 2, replace=False))
            cuts = np.concatenate([[0], cuts, [self.last_cut]]).astype(np.int64)
            data = np.concatenate([self.flat[:self.last_cut], np.zeros(64, np.uint8)])
            words, hits = oracle_policy(self.oracle, self.rules, data, cuts.astype(np.uint32))
            self.base[n] = (cuts, words, hits)
        return self.base[n]

    def batch(self, n, end_mod, prefix=0):
        """n messages over the text, the last one ending with a rule token on the batch's last byte, at
        (off[n] - (off[0] & ~15)) % TILE == end_mod; prefix bytes (with a token of their own) in front of off[0]"""
        cuts, bwords, bhits = self.head(n)
        tok = b" " + self.samples[int(self.rng.integers(0, len(self.samples)))]
        tile0 = prefix & ~15
        e = self.last_cut + 1024
        e += (end_mod - (e + prefix + len(tok) - tile0)) % TILE
        last = np.concatenate([self.flat[self.last_cut:e], np.frombuffer(tok, dtype=np.uint8)])
        pre = np.frombuffer((b" " + self.samples[0] + b" ").ljust(prefix, b".")[:prefix], dtype=np.uint8)
        data = np.concatenate([pre, self.flat[:self.last_cut], last, np.zeros(64, np.uint8)])
        off = np.concatenate([cuts + prefix, [prefix + self.last_cut + len(last)]]).astype(np.uint32)
        assert (int(off[-1]) - tile0) % TILE == end_mod
        lw, lh = oracle_policy(self.oracle, self.rules, np.concatenate([last, np.zeros(64, np.uint8)]),
                               np.array([0, len(last)], dtype=np.uint32))
        words = np.concatenate([bwords, lw])
        hits = bhits + [(n - 1, r) for (_, r) in lh]
        return data, off, words, hits


CASES = {"syn500-s2": (500, 2), "builtins-s4": (17, 4)}


@pytest.mark.parametrize("name", list(CASES))
def test_wide_tiles_at_their_edges_seams_and_rounds(N, oracle, name):
    """Tokens across every tile edge, half-tile seam, CTA and round edge; batch ends at every half position; a ragged
    batch with off[0] = 53: host words and hits and device words equal the oracle's."""
    n_rules, stride = CASES[name]
    rl = W.make_rules(n_rules)
    rules = W.rules_as_tuples(rl)
    rs = N.Ruleset(rules, options=N.OPT_STRIDE2 if stride == 2 else N.OPT_STRIDE_AUTO, strict=True)
    assert rs.info().stride == stride
    sms = sm_count()
    grids = sorted({scan_grid(n, sms) for n in NS})
    assert grids == [1, 2, 3]
    round_bytes = max(grids) * WARPS * TILES_PER_ROUND[stride] * TILE
    text = Text(oracle, rl, rules, 2 * round_bytes + 8192, seed=stride * 1000 + n_rules)     # two rounds of the largest grid
    # each seam sample swept the split points 1 .. (its seams, at most its token's length - 1); most swept them all
    full = 0
    for r, splits in text.seam_splits.items():
        n_split = len(text.samples[r]) + 1
        assert splits == set(range(1, 1 + min(n_split, text.seams[r]))), r
        full += text.seams[r] >= n_split
    assert full >= SEAM_SAMPLES * 3 // 4, full
    for n in NS:
        for end_mod in ENDS:
            data, off, ewords, ehits = text.batch(n, end_mod)
            words, hits = rs.scan_batch(data, off)
            assert np.array_equal(words, ewords), (n, end_mod)
            assert hit_pairs(hits) == ehits, (n, end_mod)
            assert np.array_equal(device_words(N, rs, data, off), ewords), (n, end_mod)
            assert int(ewords[-1]) >> 63                                           # the last byte's token
            assert sum(int(w) >> 63 for w in ewords) >= 0.9 * n                   # (most messages hold several tokens)
    for end_mod in (200, 800):
        data, off, ewords, ehits = text.batch(NS[1], end_mod, prefix=PREFIX)
        assert int(off[0]) == PREFIX
        words, hits = rs.scan_batch(data, off)
        assert np.array_equal(words, ewords) and hit_pairs(hits) == ehits, end_mod
        assert np.array_equal(device_words(N, rs, data, off), ewords), end_mod
    rs.close()
