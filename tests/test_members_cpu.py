"""CPU tier: the member and near-miss batches of test_gpu_members.py (tests/members.py) through the host harness -- the
product's compiler, gram filter tables and matchers with the device pipeline restated on the host.  The policy pipeline
over each packed batch equals the oracle; oracle hits are gram-filter candidates; all matches of a rule on a sample
of messages equal the oracle's spans.  When the GPU tier disagrees with the oracle and this file does not, the kernel is
at fault, not the compiler."""
import numpy as np
import pytest

import members as M
from helpers import Harness, oracle_regexes

SPAN_SAMPLE = 300
# the host harness's stride option for each case (0: the compiler's choice), as cg_ruleset_create's options
STRIDE = {"builtins": 0, "syn500-s2": 2, "syn500-s4": 4, "non-ascii": 0}
# (stride, gram shapes, trigger bytes, always-candidate rules) each case compiles to
REGIME = {"builtins": (4, 5, 1, 0), "syn500-s2": (2, 3, 1, 0), "syn500-s4": (4, 5, 1, 0), "non-ascii": (2, 8, 2, 9)}
CONFIRM_TABLE_BUDGET = 176 * 1024          # kernels.h kConfirmTableBudget
FOLD_SAMPLE = 400                          # folding near misses per kind whose flagged grams are compared with their member's
CANDIDATE_SAMPLE = 1500                    # distinct hit messages per batch whose oracle hits must be gram-filter candidates

_built = {}


def case_and_oracle(oracle, name):
    key = "syn500" if name in ("syn500-s2", "syn500-s4") else name
    if key not in _built:
        c = M.build_case(name)
        _built[key] = (c, M.Expected(oracle, c.rules))
    return _built[key]


def test_generator_follows_ecmascript_semantics():
    """The generator's own sets and case variants (not the compiler's, not the oracle's)."""
    assert M.case_variants(ord("k")) == [ord("K"), ord("k")]                     # not U+212A KELVIN SIGN (its upper case is itself)
    assert ord("ſ") not in M.case_variants(ord("s"))                        # long s upper-cases to ASCII 'S': excluded
    assert sorted(M.case_variants(ord("ж"))) == [0x416, 0x436]
    assert ord("µ") in M.case_variants(ord("μ"))                       # MICRO SIGN and GREEK SMALL MU share U+039C
    assert M.case_variants(ord("ß")) == [0xdf]                                  # 'SS' is two units: ß stays itself
    lang = M.Language(r"[^\s'\"]\d\w.", 0, np.random.default_rng(0))
    neg, dig, word, dot = lang.classes
    every = lambda c: {x for lo, hi in c.ranges for x in range(lo, hi + 1)}
    assert every(dig) == set(M.DIGITS) and every(word) == set(M.WORD)
    assert every(neg) == set(M.UNIVERSE) - set(M.JS_SPACES) - {0x27, 0x22} and 0xFEFF not in every(neg)
    assert every(dot) == set(M.UNIVERSE) - M.LINE_TERMINATORS
    r = M.RuleMembers(0, r"ab[0-9]{2,4}(?:x|yz)+", 0, np.random.default_rng(1), 16)
    assert not r.coverage_gaps()
    assert set("".join(t for _, t, _ in r.members)) >= set("0123456789")    # every digit is in a member, not only drawn
    ri = M.RuleMembers(0, r"[a-f]{3}q", 1, np.random.default_rng(2), 16)
    assert not ri.coverage_gaps()
    assert set("".join(t[:3] for _, t, _ in ri.members).lower()) == set("abcdef")
    assert any(c.isupper() for _, t, _ in ri.members for c in t)                 # flag i: case variants are emitted
    assert all(t.startswith("ab") for _, t, _ in r.members)
    counts = sorted({len(t) - len(t.lstrip("ab0123456789")) for _, t, _ in r.members})
    assert counts[0] == 4 and counts[-1] == 6                                    # the repeat at its min and its max


# syn5000 compiles like syn500 (stride 2, three shapes); what sets it apart is on the device only (confirm_kernel reads
# its tables in place), and deciding its batches against 5000 rules would take the oracle alone past half a minute
@pytest.mark.parametrize("name", [c for c in M.CASES if c != "syn5000"])
def test_members_through_the_host_pipeline(oracle, harness_lib, name):
    """Every batch of the case (members, near misses, members again: total lengths 0, 1 and 15 mod 16):
    Harness.policy_hits_batch equals the oracle's (msg, rule) list; every oracle hit of a sample of the distinct hit messages
    is a candidate of the gram filter (at a lead that moves the message through the 16 residues); on a sample of (message,
    rule) pairs every match of the rule equals the oracle's.  A folding near miss flags as many grams as its member."""
    case, exp = case_and_oracle(oracle, name)
    h = Harness(harness_lib, case.rules, stride=STRIDE[name])
    assert (h.status[:len(case.rules)] == 0).all()
    info = h.info()
    assert (info["stride"], info["shapes"], info["triggers"], info["n_always"]) == REGIME[name]
    if name == "syn500-s2":
        assert h.confirm_block_bytes() <= CONFIRM_TABLE_BUDGET
    n_pos, n_neg = M.check_strength(case, exp)
    regs = oracle_regexes(oracle, case.rules)
    rng = np.random.default_rng(len(name) + 7)
    checked = set()
    for bname, b in case.batches():
        _, ehits, _ = exp.of(b.msgs)
        assert h.policy_hits_batch(b.data, b.off) == ehits, bname
        by = {}
        for m, r in ehits:
            by.setdefault(m, set()).add(r)
        for i in sorted(by)[::max(1, len(by) // CANDIDATE_SAMPLE)]:
            m = b.msgs[i]
            if m not in checked:
                checked.add(m)
                c, d, _ = h.candidates2(m, lead=16 + len(checked) % 16, seed=i)
                assert by[i] <= c | d, (bname, m, by[i] - (c | d))
        for i in rng.choice(len(b.msgs), SPAN_SAMPLE, replace=False).tolist():
            m = b.msgs[i]
            rule = int(rng.choice(sorted(by[i]))) if i in by else int(rng.integers(0, len(case.rules)))
            d, o = oracle.pack([m])
            want = [(s, e) for _, _, s, e in oracle.find_matches_batch([(regs[rule], "custom")], d, o).tolist()]
            assert [(g[2], g[3]) for g in h.find_all(rule, m)] == want, (bname, rule, m)
        print("%s / %s: %d messages, %d hits" % (name, bname, len(b.msgs), len(ehits)))
    for kind, (nb, mb) in case.folding.items():
        for pi in sorted(rng.choice(len(nb.pieces), min(FOLD_SAMPLE, len(nb.pieces)), replace=False).tolist()):
            lead = 16 + pi % 16
            near, member = (b"".join(b.pieces[pi][1:]) for b in (nb, mb))
            assert h.candidates2(near, lead=lead, seed=pi)[2] == h.candidates2(member, lead=lead, seed=pi)[2], (kind, near, member)
    print("%s: distinct pieces matching their rule %d, not matching %d, distinct hit messages checked for candidates %d"
          % (name, n_pos, n_neg, len(checked)))
    h.close()
