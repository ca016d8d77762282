"""CPU tier, the fact that proofs from a log's node store rest on: in RFC 6962's recursion over D[0:s] every sibling range
(and every element of a consistency proof) is either a complete aligned node [j 2^h, (j + 1) 2^h) or a suffix D[a:s] whose
root is the right-to-left fold F_i of s's frontier subtrees, i >= 1.  The rule the gather kernel follows (the levels of
merkle_path_levels in csrc/kernels.h, restated here) is checked against proof_ranges and the oracle's recursion for every
(index, s) and every (first, s) with s <= 2^10, and on real digests against the oracle for small s.  No device needed."""
import os
import re

from test_merkle_fold import proof_ranges

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
S_MAX = 1 << 10


def path_levels(i, s, lo=0):
    """merkle_path_levels: bit l set <=> PATH(i, D[0:s]) has an element at level l (levels >= lo only)"""
    inner = (i ^ (s - 1)).bit_length()
    below = (1 << inner) - 1
    return (below | (i & ~below)) & ~((1 << lo) - 1)


def element_range(i, s, level):
    """the sibling range of i's ancestor at `level`, cut at s"""
    b = ((i >> level) ^ 1) << level
    return b, min(b + (1 << level), s)


def gather_ranges(i, s):
    """the gather kernel's inclusion path of leaf i in the tree of s leaves: leaf level first"""
    lv = path_levels(i, s)
    return [element_range(i, s, l) for l in range(64) if lv >> l & 1]


def gather_consistency(first, s):
    """PROOF(first, D[0:s]): the node (ctz first, (first - 1) >> ctz first) unless first is a power of two, then the path of
    leaf first - 1 from level ctz(first) up"""
    if first == s:
        return []
    lo = (first & -first).bit_length() - 1
    seed = [(first - (1 << lo), first)] if first & (first - 1) else []
    lv = path_levels(first - 1, s, lo)
    return seed + [element_range(first - 1, s, l) for l in range(64) if lv >> l & 1]


def consistency_ranges(first, s):
    """the oracle's SUBPROOF recursion (oracle.merkle_consistency_proof) on leaf ranges instead of digests"""
    def sub(m, lo, hi, b):
        if m == hi - lo:
            return [] if b else [(lo, hi)]
        k = 1 << ((hi - lo - 1).bit_length() - 1)
        if m <= k:
            return sub(m, lo, lo + k, b) + [(lo + k, hi)]
        return sub(m - k, lo + k, hi, False) + [(lo, lo + k)]
    return sub(first, 0, s, True)


def frontier_starts(s):
    """start of every frontier subtree of s, largest first"""
    out, a = [], 0
    for h in reversed(range(s.bit_length())):
        if s >> h & 1:
            out.append(a)
            a += 1 << h
    return out


def classify(a, b, s):
    """('node', h, j) for a complete aligned node, ('suffix', i) for D[a:s] = F_i with i >= 1; anything else fails"""
    w = b - a
    if w & (w - 1) == 0 and a % w == 0:
        return ("node", w.bit_length() - 1, a // w)
    assert b == s, (a, b, s)
    starts = frontier_starts(s)
    assert a in starts[1:], (a, s)
    return ("suffix", starts.index(a))


def spine_slot(a, s):
    """where the gather kernel reads a suffix: spine[msb(s - a)], the fold of s's frontier subtrees under bits <= msb(s - a)"""
    w = s - a
    h = w.bit_length() - 1
    assert a == s & ~((2 << h) - 1)
    return h


def test_every_inclusion_path_is_stored_nodes_and_frontier_suffixes():
    for s in range(1, S_MAX + 1):
        for i in range(s):
            got = gather_ranges(i, s)
            want = proof_ranges(i, s)[::-1]
            assert got == want, (i, s)
            for a, b in got:
                if classify(a, b, s)[0] == "suffix":
                    spine_slot(a, s)


def test_every_consistency_proof_is_stored_nodes_and_frontier_suffixes():
    for s in range(1, S_MAX + 1):
        for first in range(1, s + 1):
            got = gather_consistency(first, s)
            assert got == consistency_ranges(first, s), (first, s)
            assert len(got) <= max(1, (s - 1).bit_length()) + 1
            for a, b in got:
                if classify(a, b, s)[0] == "suffix":
                    spine_slot(a, s)


def test_path_lengths_fit_the_documented_strides():
    for s in range(1, S_MAX + 1):
        assert max(bin(path_levels(i, s)).count("1") for i in range(s)) == (s - 1).bit_length()


def test_store_digests_give_the_oracle_proofs(oracle):
    """with real digests: complete nodes from a level-wise store, suffixes from the spine fold, for every s <= 40"""
    import random
    rng = random.Random(5)
    leaves = [bytes(rng.randrange(256) for _ in range(rng.randrange(0, 50))) for _ in range(40)]
    H = [oracle.merkle_leaf_hash(x) for x in leaves]
    levels = [H]
    while len(levels[-1]) > 1:
        prev = levels[-1]
        levels.append([oracle.merkle_node_hash(prev[2 * j], prev[2 * j + 1]) for j in range(len(prev) // 2)])
    for s in range(1, len(leaves) + 1):
        spine = {}
        bits = [h for h in range(s.bit_length()) if s >> h & 1]
        acc = levels[bits[0]][(s >> bits[0]) - 1]
        for h in bits[1:]:
            acc = oracle.merkle_node_hash(levels[h][(s >> h) - 1], acc)
            spine[h] = acc
        root = spine[bits[-1]] if len(bits) > 1 else levels[bits[0]][0]

        def digest(a, b):
            w = b - a
            if w & (w - 1) == 0:
                return levels[w.bit_length() - 1][a // w]
            return spine[spine_slot(a, s)]
        for i in range(s):
            path = [digest(a, b) for a, b in gather_ranges(i, s)]
            assert path == oracle.merkle_audit_path(leaves[:s], i), (i, s)
            assert oracle.merkle_verify_path(leaves[i], i, s, path, root)
        for first in range(1, s + 1):
            assert [digest(a, b) for a, b in gather_consistency(first, s)] == oracle.merkle_consistency_proof(leaves[:s], first), (first, s)


def test_proof_calls_are_declared_exported_and_bound():
    from vainplex_openclaw_b200 import _native as N
    hdr = open(os.path.join(ROOT, "include", "openclaw_gov.h")).read()
    shim = open(os.path.join(ROOT, "napi", "openclaw_gov_napi.c")).read()
    ts = open(os.path.join(ROOT, "napi", "gpu-backend.ts")).read()
    for name in ("cg_merkle_log_create_tree", "cg_merkle_log_proofs", "cg_merkle_log_consistency_between", "cg_merkle_verify_proofs"):
        assert re.search(r"CG_API\s+int\s+%s\s*\(" % name, hdr), name
        assert name in N.EXPORTS and name + "(" in shim, name
    for fn in ("logCreateTree", "logProofs", "logConsistencyBetween", "verifyProofs"):
        assert "addon.%s(" % fn in ts, fn


def test_proof_calls_need_init():
    """before cg_init every new call returns CG_ERR_NOT_INITIALIZED (in a fresh process: no device is touched)"""
    import subprocess
    import sys
    code = ("import ctypes as C\nfrom vainplex_openclaw_b200 import _native as N\nL = N.load()\nh = C.c_void_p()\n"
            "print(L.cg_merkle_log_create_tree(C.byref(h)), L.cg_merkle_verify_proofs(None, None, None, 1, 1, None, 0, None, None, None))\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == ["-2", "-2"]
