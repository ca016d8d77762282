"""CPU tier, text edges: a message's results depend on its own bytes only, decoded as TextDecoder decodes them.  The
product's compiler, gram filter and matchers (host harness) and the oracle against Python's UTF-8 decoder on ill-formed
input, U+FFFD literals through the whole pipeline, and the packed-batch pipeline on neighbours whose bytes would change
each other's answers.  The GPU tier (test_gpu_text_edges.py) runs the same cases through the kernels."""
import numpy as np
import pytest

from helpers import (AKIA, EDGE_PAIRS, EDGE_RULES, FFFD_ATOMS, FFFD_CASES, ILL_FORMED, EdgeBatch, Harness, decode_units,
                     ill_formed_corpus, ill_formed_texts, oracle_regexes, random_regex, unit_starts)
from vainplex_openclaw_b200 import workload as W

LINE_TERMINATORS = {0x0A, 0x0D, 0x2028, 0x2029}
WORD = set(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_")


def oracle_spans(O, rx, msgs):
    d, o = O.pack(msgs)
    out = {}
    for mi, _, s, e in O.find_matches_batch([(rx, "custom")], d, o).tolist():
        out.setdefault(mi, []).append((s, e))
    return out


def test_python_decoder_reports_maximal_subparts():
    """The reference decoder itself on the WHATWG examples: one U+FFFD per maximal subpart, with its bytes."""
    assert [(u, a, b) for u, a, b in decode_units(b"\xf0\x9f\x98a")] == [(0xfffd, 0, 3), (0x61, 3, 4)]
    assert decode_units(b"\xed\xa0\x80") == [(0xfffd, 0, 1), (0xfffd, 1, 2), (0xfffd, 2, 3)]
    assert decode_units(b"\xe0\x80\xaf") == [(0xfffd, 0, 1), (0xfffd, 1, 2), (0xfffd, 2, 3)]
    assert decode_units(b"\xf4\x90\x80\x80") == [(0xfffd, i, i + 1) for i in range(4)]
    assert decode_units(b"\xe2\x82\xac\xef\xbf\xbd") == [(0x20ac, 0, 3), (0xfffd, 3, 6)]
    assert decode_units("\U0001F600".encode()) == [(0xd83d, 0, 2), (0xde00, 2, 4)]


@pytest.mark.parametrize("kind", list(ILL_FORMED))
def test_decoders_agree_with_python_on_ill_formed_input(oracle, harness_lib, kind):
    """[^], . and \\W over every ill-formed sequence of one kind, in context: the oracle's UTF-16 spans and the harness's
    spans (UTF-16 and bytes) are the units Python's decoder produces; each replacement covers exactly its maximal
    subpart's bytes.  The policy pipeline (gram filter -> matchers) says the same."""
    rules = [("[^]", 0, 3), (".", 0, 3), (r"\W", 0, 3)]
    keep = {0: lambda u: True, 1: lambda u: u not in LINE_TERMINATORS, 2: lambda u: u >= 128 or u not in WORD}
    h = Harness(harness_lib, rules)
    assert (h.status[:3] == 0).all()
    regs = oracle_regexes(oracle, rules)
    msgs = [m for m in ill_formed_corpus() if any(s in m for s in ILL_FORMED[kind])]
    assert len(msgs) >= 8 * len(ILL_FORMED[kind])
    replacements = 0
    for ri in range(3):
        exp = oracle_spans(oracle, regs[ri], msgs)
        for mi, m in enumerate(msgs):
            units = decode_units(m)
            want = [(a, b, i, i + 1) for i, (u, a, b) in enumerate(units) if keep[ri](u)]
            assert exp.get(mi, []) == [(w[2], w[3]) for w in want], (rules[ri][0], m)
            assert h.find_all(ri, m) == want, (rules[ri][0], m)
            assert (ri in h.policy_hits(m, lead=mi % 5)) == bool(want), (rules[ri][0], m)
            replacements += sum(1 for u in units if u[0] == 0xfffd)
    assert replacements >= 3 * len(msgs)


def test_fffd_literals_match_ill_formed_input(oracle, harness_lib):
    """A rule with a literal U+FFFD matches wherever the decoder produces one, not only at EF BF BD: the four cases the
    gram filter missed (its factor was U+FFFD's own UTF-8 bytes), at every lead in front of the message."""
    for src, text, spans in FFFD_CASES:
        h = Harness(harness_lib, [(src, 0, 3)])
        assert h.status[0] == 0
        rx = oracle.Regex(src)
        assert oracle_spans(oracle, rx, [text]).get(0) == spans, src
        starts = unit_starts(text)
        assert h.find_all(0, text) == [(starts[s], starts[e], s, e) for s, e in spans], src
        for lead in (0, 1, 2, 3, 7, 16):
            assert 0 in h.candidates(text, lead=lead, seed=lead), ("filter missed", src, text, lead)
            assert h.policy_hits(text, lead=lead, seed=lead) == {0}, (src, text, lead)
        h.close()


def test_fffd_fix_leaves_rule_sets_without_fffd_unchanged(harness_lib):
    """The bench's rule sets hold no U+FFFD: they compile to the tables they compiled to before U+FFFD literals took the
    three byte shapes."""
    want = {
        17: dict(keys=14323, n_factors=23, stride=4, factor_min=2, factor_max=16, n_always=0, image_bytes=131072, prog_words=766,
                 entries=88, shapes=5, triggers=1, bitmap_bytes=131072, tables_resident=0),
        500: dict(keys=3694, n_factors=775, stride=2, factor_min=2, factor_max=16, n_always=0, image_bytes=131072, prog_words=14647,
                  entries=1548, shapes=3, triggers=1, bitmap_bytes=131072, tables_resident=0),
    }
    for n, info in want.items():
        rules = W.rules_as_tuples(W.make_rules(n))
        assert not any("\ufffd" in r[0] or "UFFFD" in r[0].upper() for r in rules)
        h = Harness(harness_lib, rules)
        assert h.info() == info, n
        h.close()


def test_random_regex_differential_on_ill_formed_text(oracle, harness_lib):
    """Random patterns (helpers.ATOMS plus U+FFFD alone and in a class; flag i on a fifth of them) on random texts made
    of ASCII, valid multi-byte characters, U+FFFD and ill-formed pieces: spans (UTF-16 and bytes) equal the oracle's,
    every true hit is a candidate of the gram filter, the policy pipeline answers RegExp.test."""
    rng = np.random.default_rng(20261016)
    msgs = ill_formed_texts(rng, 60) + [t for _, t, _ in FFFD_CASES] + [b"", b"\xef\xbf\xbd", b"\xe2\x82\xac"]
    starts = [unit_starts(m) for m in msgs]
    checked = fffd_rules = hits = 0
    for it in range(600):
        src = random_regex(rng, atoms=FFFD_ATOMS)
        fl = 1 if rng.random() < 0.2 else 0
        try:
            rx = oracle.Regex(src, "i" if fl else "")
        except (oracle.RegexSyntaxError, oracle.OracleUnsupported):
            continue
        h = Harness(harness_lib, [(src, fl, 3)])
        if int(h.status[0]) != 0:
            h.close()
            continue
        try:
            exp = oracle_spans(oracle, rx, msgs)
        except RuntimeError:          # exponential backtracking in the oracle: not a usable vector
            h.close()
            continue
        for mi, m in enumerate(msgs):
            e = exp.get(mi, [])
            got = h.find_all(0, m)
            assert [(g[2], g[3]) for g in got] == e, (src, fl, m)
            assert [(g[0], g[1]) for g in got] == [(starts[mi][s], starts[mi][t]) for s, t in e], (src, fl, m)
            if e:
                assert 0 in h.candidates(m, lead=mi % 4, seed=it), ("prefilter missed", src, fl, m)
                hits += 1
            assert (0 in h.policy_hits(m, lead=mi % 7, seed=it)) == bool(e), ("policy pipeline differs", src, fl, m)
        checked += 1
        fffd_rules += "FFFD" in src
        h.close()
    assert checked > 350 and fffd_rules > 60 and hits > 3000, (checked, fffd_rules, hits)


def oracle_hits(O, rules, data, off):
    regs = oracle_regexes(O, rules)
    bits, _ = O.scan_policy(regs, data, off.astype(np.uint64))
    return [(m, int(r)) for m in range(bits.shape[0]) for r in np.nonzero(np.unpackbits(bits[m], bitorder="little")[:len(rules)])[0]]


def test_packed_batch_pipeline_keeps_neighbours_apart(oracle, harness_lib):
    """The device pipeline restated over a packed batch (buffer-relative gram positions, head check, message lookup,
    straddle check) on the neighbour pairs at every residue of the edge, across tile boundaries: hits equal the oracle's,
    the joined controls hit.  Then the same messages with the bytes before the range and behind it filled with what
    would complete the first and the last message's tokens."""
    h = Harness(harness_lib, EDGE_RULES)
    assert (h.status[:len(EDGE_RULES)] == 0).all()
    eb = EdgeBatch(EDGE_PAIRS)
    want = oracle_hits(oracle, EDGE_RULES, eb.data, eb.off)
    eb.check_hits(set(want))
    assert h.policy_hits_batch(eb.data, eb.off) == want
    # the same messages behind a prefix and in front of a tail that complete tokens across the range's ends
    msgs = [b"tagamma", b"x", b"alphabe"]
    for pre in (b"alphabe", b"X" * 16 + b"alphabe", b"Q" * 33):
        for tail in (b"tagamma" + b"\0" * 57, b"7" * 64, b"\x80" * 64):
            d = np.frombuffer(pre + b"".join(msgs) + tail, dtype=np.uint8).copy()
            off = (len(pre) + np.cumsum([0] + [len(m) for m in msgs])).astype(np.uint32)
            assert h.policy_hits_batch(d, off) == []
    for pre, tail in ((b"X", b"Q" * 64), (b"7", b"9" * 64)):                 # the guards see the range's ends, not these bytes
        d = np.frombuffer(pre + AKIA + tail, dtype=np.uint8).copy()
        assert h.policy_hits_batch(d, np.array([len(pre), len(pre) + len(AKIA)], dtype=np.uint32)) == [(0, 0)]
    h.close()
