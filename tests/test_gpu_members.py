"""GPU tier: random members of every rule's language and their near misses (tests/members.py), at every residue mod 16,
across 512-byte tile edges at every offset, cut across neighbouring messages and on the last byte of the batch, through
the scan kernels of each compiled regime: words, hit lists and spans of the host, device-resident and single-message
calls against the oracle, bit-exactly.  test_members_cpu.py runs the same batches through the host harness (the
compiler and the host restatement of the kernels), so a disagreement here that the CPU tier does not show is a kernel's.
Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from helpers import Harness
from members import CASES, Expected, build_case, check_strength
from test_gpu_boundaries import hit_pairs, span_tuples
from test_gpu_redact_device import find_device, tup
from test_gpu_scan_hits_device import device_words, hits_device

pytestmark = pytest.mark.gpu

CONFIRM_TABLE_BUDGET = 176 * 1024          # kernels.h kConfirmTableBudget: confirm_kernel stages its tables up to this size
ONE_SAMPLE = 200


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


@pytest.fixture(scope="module")
def torch():
    import torch as T
    return T


_built = {}


def case_and_oracle(oracle, name):
    """(Case, Expected); the two syn500 cases share one (same rules, same members)"""
    key = "syn500" if name in ("syn500-s2", "syn500-s4") else name
    if key not in _built:
        c = build_case(name)
        _built[key] = (c, Expected(oracle, c.rules))
    return _built[key]


def check_regime(N, rs, harness_lib, name, rules, options):
    """the compiled regime the case is named for, from Ruleset.info() and, for the confirm block's size and the gram
    shapes, from the same rule set compiled by the host harness (shown to be the same compilation)"""
    info = rs.info()
    regime = (info.stride, info.n_triggers, info.n_always_candidate)
    h = Harness(harness_lib, rules, stride=options)
    hi, cf = h.info(), h.confirm_block_bytes()
    h.close()
    assert (hi["stride"], hi["triggers"], hi["n_always"], hi["keys"], hi["entries"], hi["n_factors"]) == \
        regime + (info.gram_keys, info.gram_entries, info.n_factors)
    if name == "builtins":
        assert regime == (4, 1, 0)                          # one probe per chunk word, the '@' trigger
    elif name == "syn500-s2":
        assert regime == (2, 1, 0) and hi["shapes"] == 3
        assert cf <= CONFIRM_TABLE_BUDGET                   # confirm_kernel stages its tables in shared memory
    elif name == "syn500-s4":
        assert regime == (4, 1, 0)
    elif name == "syn5000":
        # the confirm block holds 48 bytes per factor and, per gram entry, one 4-byte group entry and two or more 16-byte
        # slots (capi.cu, ruleset_image.cpp): this lower bound past the budget means the tables are read in place
        assert info.n_factors * 48 + info.gram_entries * 8 > CONFIRM_TABLE_BUDGET and cf > CONFIRM_TABLE_BUDGET
    elif name == "non-ascii":
        assert info.n_always_candidate > 0 and info.n_triggers == 2
    assert info.n_ok == len(rules)
    return regime, cf


@pytest.mark.parametrize("name", CASES)
def test_members_and_near_misses_through_the_kernels(N, torch, oracle, harness_lib, name):
    """Every batch of the case through scan_batch (words, hit list), scan_batch_device (words), scan_hits_batch_device
    (hit list, guard words behind it), find_matches_batch and find_matches_batch_device (spans), and a fixed sample of its
    messages through scan_one and find_matches_one, against the oracle.  Strength: every rule has 10 distinct
    oracle-positive members (members.UNSATISFIABLE apart), 30 % of the distinct pieces do not match the rule they were
    made from, and the near misses whose changed byte folds to the original (case bit, bit 7, digit twins) flag exactly
    the grams their members flag: they reach confirm_kernel, which has to reject them."""
    case, exp = case_and_oracle(oracle, name)
    options = {"syn500-s2": N.OPT_STRIDE2, "syn500-s4": N.OPT_STRIDE4}.get(name, N.OPT_STRIDE_AUTO)
    rs = N.Ruleset(case.rules, options=options, strict=True)
    regime, cf = check_regime(N, rs, harness_lib, name, case.rules, options)
    n_pos, n_neg = check_strength(case, exp)
    flagged, vm_pairs = {}, {}
    rng = np.random.default_rng(len(name))
    for bname, b in case.batches():
        ewords, ehits, espans = exp.of(b.msgs)
        words, hits = rs.scan_batch(b.data, b.off)
        flagged[bname], vm_pairs[bname] = rs.work_counters()[6], rs.work_counters()[1]
        assert np.array_equal(words, ewords), bname
        assert hit_pairs(hits) == ehits, bname
        assert np.array_equal(device_words(N, torch, rs, b.data, b.off), ewords), bname
        dwords, dpairs = hits_device(N, torch, rs, b.data, b.off, cap=len(ehits) + 16)
        assert dpairs == ehits and np.array_equal(dwords, ewords), bname
        assert span_tuples(rs.find_matches_batch(b.data, b.off)) == espans, bname
        assert tup(find_device(N, torch, rs, b.data, b.off, cap=len(espans) + 16)) == espans, bname
        rules_of, spans_of = {}, {}
        for mm, r in ehits:
            rules_of.setdefault(mm, []).append(r)
        for mm, r, s, e in espans:
            spans_of.setdefault(mm, []).append((0, r, s, e))
        for i in sorted(rng.choice(len(b.msgs), min(ONE_SAMPLE, len(b.msgs)), replace=False).tolist()):
            m = b.msgs[i]
            w1, r1 = rs.scan_one(m)
            assert w1 == int(ewords[i]) and r1 == rules_of.get(i, []), (bname, m)
            assert tup(rs.find_matches_one(m)) == spans_of.get(i, []), (bname, m)
        print("%s / %s: %d messages, %d bytes, %d hits, %d spans, %d flagged grams, %d VM pairs"
              % (name, bname, len(b.msgs), b.total, len(ehits), len(espans), flagged[bname], vm_pairs[bname]))
    print("%s: regime %s, confirm block %d bytes, distinct pieces matching their rule %d, not matching %d"
          % (name, regime, cf, n_pos, n_neg))
    assert flagged["members"] > 0
    # a folding near miss flags the grams of its member, no fewer: the filter passes it on and the exact comparison in
    # confirm_kernel (or the matchers behind it) must reject it
    assert set(case.folding) >= {"xor20", "xor80", "xorA0"}
    for kind, (nb, mb) in case.folding.items():
        fl = []
        for b in (nb, mb):
            words, _ = rs.scan_batch(b.data, b.off)
            assert np.array_equal(words, exp.of(b.msgs)[0]), kind
            fl.append(rs.work_counters()[6])
        nwords = exp.of(nb.msgs)[0]
        n_rejected = sum(1 for i, _ in nb.member_messages() if not int(nwords[i]) >> 63)
        print("%s / %s near misses: %d pieces, %d hitting nothing, %d flagged grams (their members: %d)"
              % (name, kind, len(nb.pieces), n_rejected, fl[0], fl[1]))
        assert fl[0] == fl[1] > 0, kind
    if name == "non-ascii":
        assert vm_pairs["members"] > 0                      # non-ASCII islands go to the VM
    rs.close()
