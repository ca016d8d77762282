"""Random members of each rule's language, their near misses, and packed batches that place them at every alignment.

The generator reads a rule's source with Python's regular-expression parser (re._parser) for its structure only and
applies ECMAScript semantics itself, so it shares no code with the product's compiler (rulec.cpp) or the oracle
(oracle/jsre.c):
  \\d, \\w      ASCII only
  \\s          the JS WhiteSpace and LineTerminator set
  .           anything but \\n, \\r, U+2028 and U+2029
  negations   [^...], \\S, \\W, \\D and . are complements over UNIVERSE: printable ASCII, tab, newline, the JS spaces, 2- and
              3-byte letters, U+FFFD and an astral character
  flag i      each unit becomes a random character with the same Canonicalize (ECMA-262, non-unicode mode: the upper case
              of a single code unit, never a non-ASCII character to an ASCII one), computed from str.upper()
Assertions (^, $, \\b, \\B, look-around) emit nothing: the neighbours put around a member satisfy or violate them, and
the oracle decides every message.  Near misses change one thing about a member; the oracle decides those too.
"""
import re._constants as K
import re._parser as P

import numpy as np

JS_SPACES = [0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x20, 0xA0, 0x1680] + list(range(0x2000, 0x200B)) + [0x2028, 0x2029, 0x202F, 0x205F, 0x3000, 0xFEFF]
LINE_TERMINATORS = {0x0A, 0x0D, 0x2028, 0x2029}
DIGITS = list(range(0x30, 0x3A))
WORD = DIGITS + list(range(0x41, 0x5B)) + list(range(0x61, 0x7B)) + [0x5F]
EXTRA = [0xE9, 0xC9, 0x416, 0x436, 0x4E2D, 0xFFFD, 0x1F600]              # é É Ж ж 中 U+FFFD 😀
UNIVERSE = sorted(set(range(0x20, 0x7F)) | set(JS_SPACES) | set(EXTRA))
SMALL_CLASS = 64                  # classes up to this size have every member drawn; larger ones their ranges' end points
UNBOUNDED_EXTRA = 12              # an unbounded repeat runs up to min + 12 ...
LONG_EXTRA = 100                  # ... and once per rule to min + 100 (islands longer than the island matcher walks)
# digits fold to the same value as these in the gram filter (case bit and bit 7 dropped, 0x30-0x3F collapsed)
DIGIT_TWINS = b":;<=>?/"


def _canonicalize(c):
    """ECMA-262 22.2.2.7.3 Canonicalize, non-unicode mode"""
    u = chr(c).upper()
    if len(u) != 1 or (c >= 128 and ord(u) < 128):
        return c
    return ord(u)


_CASE_VARIANTS = None


def case_variants(c):
    """every BMP character with c's Canonicalize (c itself included)"""
    global _CASE_VARIANTS
    if _CASE_VARIANTS is None:
        by = {}
        for x in range(0x10000):
            if not 0xD800 <= x <= 0xDFFF:
                by.setdefault(_canonicalize(x), []).append(x)
        _CASE_VARIANTS = by
    if c >= 0x10000:
        return [c]
    return _CASE_VARIANTS[_canonicalize(c)]


def _runs(points):
    """maximal ranges of consecutive code points of a sorted list"""
    out = []
    for p in points:
        if out and out[-1][1] + 1 == p:
            out[-1][1] = p
        else:
            out.append([p, p])
    return [tuple(r) for r in out]


def _merge(ranges):
    out = []
    for lo, hi in sorted(ranges):
        if out and lo <= out[-1][1] + 1:
            out[-1][1] = max(out[-1][1], hi)
        else:
            out.append([lo, hi])
    return [tuple(r) for r in out]


def _category(cat):
    """(ranges, negated) of a class escape"""
    table = {K.CATEGORY_DIGIT: (DIGITS, False), K.CATEGORY_NOT_DIGIT: (DIGITS, True), K.CATEGORY_SPACE: (JS_SPACES, False),
             K.CATEGORY_NOT_SPACE: (JS_SPACES, True), K.CATEGORY_WORD: (WORD, False), K.CATEGORY_NOT_WORD: (WORD, True)}
    if cat not in table:
        raise ValueError("class escape %r" % (cat,))
    pts, neg = table[cat]
    return _runs(sorted(pts)), neg


class CharClass:
    """One class of a rule (a bracket class, an escape, '.', a negated literal): the code points it admits, its ranges,
    the members a rule's language members must hold at least once (`required`) and those they hold so far."""

    def __init__(self, ranges, rng, label):
        self.label = label
        self.ranges = [(lo, hi) for lo, hi in _merge(ranges) if not (0xD800 <= lo and hi <= 0xDFFF)]
        self.size = sum(hi - lo + 1 for lo, hi in self.ranges)
        assert self.size > 0, label
        if self.size <= SMALL_CLASS:
            self.required = {c for lo, hi in self.ranges for c in range(lo, hi + 1)}
        else:
            self.required = set()
            for lo, hi in self.ranges:
                self.required |= {lo, hi}
                if hi - lo > 1:
                    self.required.add(int(rng.integers(lo + 1, hi)))
        self.required -= set(range(0xD800, 0xE000))
        self.queue = sorted(self.required)            # drawn first, in random order
        rng.shuffle(self.queue)
        self.emitted = set()                          # what the rule's members hold (their Canonicalize under flag i)
        self._w = np.array([hi - lo + 1 for lo, hi in self.ranges], dtype=np.float64)
        self._w /= self._w.sum()

    @classmethod
    def of(cls, items, rng, label):
        """from the items of a parsed IN node"""
        neg, pos, negs = False, [], []
        for op, av in items:
            if op == K.NEGATE:
                neg = True
            elif op == K.LITERAL:
                pos.append((av, av))
            elif op == K.RANGE:
                pos.append(tuple(av))
            elif op == K.CATEGORY:
                rs, n = _category(av)
                if n:
                    negs.append(rs)
                else:
                    pos += rs
            else:
                raise ValueError("class item %r" % (op,))
        members = set()
        for rs in negs:                                    # \S \W \D inside a class: complements over the universe
            inside = {c for lo, hi in rs for c in range(lo, hi + 1)}
            members |= {u for u in UNIVERSE if u not in inside}
        if not neg:
            return cls(pos + _runs(sorted(members)), rng, label)
        inside = members | {u for u in UNIVERSE if any(lo <= u <= hi for lo, hi in pos)}
        return cls(_runs([u for u in UNIVERSE if u not in inside]), rng, label)

    def draw(self, rng):
        if self.queue:
            c = self.queue.pop()
        else:
            lo, hi = self.ranges[int(rng.choice(len(self.ranges), p=self._w))]
            c = int(rng.integers(lo, hi + 1))
            while 0xD800 <= c <= 0xDFFF:
                c = int(rng.integers(lo, hi + 1))
        return c

    def outside(self, rng):
        """a code point just outside one of the ranges (an end point - 1 or + 1), or None"""
        cands = [x for lo, hi in self.ranges for x in (lo - 1, hi + 1)
                 if 0 <= x <= 0x10FFFF and not 0xD800 <= x <= 0xDFFF and not any(a <= x <= b for a, b in self.ranges)]
        return int(rng.choice(cands)) if cands else None

    def uncovered(self, icase):
        """required members no member of the rule holds (under flag i: none of their case variants)"""
        if icase:
            return {r for r in self.required if _canonicalize(r) not in self.emitted}
        return self.required - self.emitted


class Language:
    """A rule's source as a tree the generator walks: ('lit', cp) / ('cls', CharClass) / ('alt', [seq]) /
    ('rep', id, lo, hi, seq) / ('grp', seq) / ('nil',) -- seq is a list of nodes."""

    def __init__(self, source, flags, rng):
        self.source, self.icase, self.rng = source, bool(flags & 1), rng
        self.classes, self.repeats = [], []
        self.tree = self._conv(P.parse(source))
        self._sched = {}

    def _cls(self, ranges, label):
        c = CharClass(ranges, self.rng, label)
        self.classes.append(c)
        return ("cls", c)

    def _conv(self, sub):
        out = []
        for op, av in sub:
            if op == K.LITERAL:
                out.append(("lit", av))
            elif op == K.NOT_LITERAL:
                out.append(self._cls(_runs([u for u in UNIVERSE if u != av]), "[^%s]" % chr(av)))
            elif op == K.ANY:
                out.append(self._cls(_runs([u for u in UNIVERSE if u not in LINE_TERMINATORS]), "."))
            elif op == K.IN:
                c = CharClass.of(av, self.rng, str(av))
                self.classes.append(c)
                out.append(("cls", c))
            elif op == K.SUBPATTERN:
                out.append(("grp", self._conv(av[-1])))
            elif op == K.BRANCH:
                out.append(("alt", [self._conv(b) for b in av[1]]))
            elif op in (K.MAX_REPEAT, K.MIN_REPEAT):
                lo, hi, body = av
                rid = len(self.repeats)
                self.repeats.append((lo, None if hi == K.MAXREPEAT else hi))
                out.append(("rep", rid, lo, None if hi == K.MAXREPEAT else hi, self._conv(body)))
            elif op in (K.AT, K.ASSERT, K.ASSERT_NOT):
                out.append(("nil",))
            else:
                raise ValueError("%s: unsupported node %r" % (self.source, op))
        return out

    def _count(self, rid, lo, hi, long_mode, override):
        if override is not None and override[0] == rid and not override[2]:
            override[2] = True
            return override[1]
        top = hi if hi is not None else lo + UNBOUNDED_EXTRA
        if hi is None and long_mode[0]:
            long_mode[0] = False
            return lo + LONG_EXTRA
        k = self._sched.get(rid, 0)
        self._sched[rid] = k + 1
        want = [lo, lo + 1, top - 1, top][k] if k < 4 else int(self.rng.integers(lo, top + 1))
        return min(max(want, lo), top)

    def _walk(self, seq, out, long_mode, override):
        rng = self.rng
        for node in seq:
            kind = node[0]
            if kind == "lit":
                c = node[1]
                if self.icase:
                    v = case_variants(c)
                    c = v[int(rng.integers(0, len(v)))]
                out.append((c, None))
            elif kind == "cls":
                c = node[1].draw(rng)
                if self.icase:
                    v = case_variants(c)
                    c = v[int(rng.integers(0, len(v)))]
                out.append((c, node[1]))
            elif kind == "grp":
                self._walk(node[1], out, long_mode, override)
            elif kind == "alt":
                alts = node[1]
                # a branch whose classes still have members to draw first
                pend = [i for i, a in enumerate(alts) if self._pending(a)]
                i = pend[int(rng.integers(0, len(pend)))] if pend and rng.random() < 0.5 else int(rng.integers(0, len(alts)))
                self._walk(alts[i], out, long_mode, override)
            elif kind == "rep":
                _, rid, lo, hi, body = node
                for _ in range(self._count(rid, lo, hi, long_mode, override)):
                    self._walk(body, out, long_mode, override)

    def _pending(self, seq):
        for node in seq:
            if node[0] == "cls" and node[1].queue:
                return True
            if node[0] in ("grp",) and self._pending(node[1]):
                return True
            if node[0] == "rep" and self._pending(node[4]):
                return True
            if node[0] == "alt" and any(self._pending(a) for a in node[1]):
                return True
        return False

    def member(self, long=False, override=None):
        """-> [(code point, CharClass or None)] of one string the walk produced"""
        out = []
        self._walk(self.tree, out, [long], override)
        return out

    def pending(self):
        return any(c.queue for c in self.classes)


def text_of(units):
    return "".join(chr(c) for c, _ in units)


# neighbours of a member: nothing (the message edge), a space, a letter, a digit, '_', a non-ASCII character
CONTEXTS = ["", " ", "a", "Q", "z", "7", "0", "_", "é", "Ж", "中", "\U0001F600"]


def context(rng):
    u = rng.random()
    if u < 0.25:
        return ""
    if u < 0.5:
        return " "
    return CONTEXTS[int(rng.integers(2, len(CONTEXTS)))]


class RuleMembers:
    """members and near misses of one rule: (left, text, right) strings and (left, member bytes, right) byte strings"""

    def __init__(self, rule_index, source, flags, rng, n_members, n_near=3, max_members=96):
        self.rule = rule_index
        self.lang = Language(source, flags, rng)
        self.members = []                    # (left, text, right)
        units = []
        long_left = any(hi is None for _, hi in self.lang.repeats)
        while len(self.members) < n_members or (self.coverage_gaps() and len(self.members) < max_members):
            j = len(self.members)
            u = self.lang.member(long=(j == 1 and long_left))
            for c, cls in u:
                if cls is not None:
                    cls.emitted.add(_canonicalize(c) if self.lang.icase else c)
            if j % 5 == 2:                                 # the member is the whole message
                left, right = "", ""
            elif j % 5 in (0, 3):                          # the message edge or a space on both sides
                left, right = " "[:int(rng.integers(0, 2))], " "[:int(rng.integers(0, 2))]
            else:
                left, right = context(rng), context(rng)
            units.append(u)
            self.members.append((left, text_of(u), right))
        self.units = units
        self.near = []                       # (kind, member index, left bytes, near-miss bytes, right bytes)
        for j, (left, text, right) in enumerate(self.members):
            self.near += self._near_misses(rng, j, left, text, right, n_near)

    def coverage_gaps(self):
        """classes with required members that no member holds (what the members emitted, not what was drawn)"""
        return [(c.label, sorted(c.uncovered(self.lang.icase))[:8]) for c in self.lang.classes if c.uncovered(self.lang.icase)]

    def _near_misses(self, rng, j, left, text, right, n_near):
        L, R = left.encode(), right.encode()
        b = text.encode("utf-8")
        out = []
        kinds = ["xor", "xor", "digit", "endpoint", "repeat", "trunc"]
        for k in range(n_near):
            kind = kinds[(n_near * j + k) % len(kinds)]
            m = None
            if kind == "xor" and b:
                p = int(rng.integers(0, len(b)))
                x = int(rng.choice([0x20, 0x80, 0xA0]))
                m = b[:p] + bytes([b[p] ^ x]) + b[p + 1:]
                kind = "xor%02X" % x
            elif kind == "digit":
                ds = [i for i, x in enumerate(b) if 0x30 <= x <= 0x39]
                if ds:
                    p = ds[int(rng.integers(0, len(ds)))]
                    t = DIGIT_TWINS[int(rng.integers(0, len(DIGIT_TWINS)))]
                    m = b[:p] + bytes([t]) + b[p + 1:]
                    kind = "digit" if t != 0x2F else "digit-slash"
            elif kind == "endpoint":
                u = self.units[j]
                at = [i for i, (_, c) in enumerate(u) if c is not None]
                if at:
                    i = at[int(rng.integers(0, len(at)))]
                    x = u[i][1].outside(rng)
                    if x is not None:
                        m = (text_of(u[:i]) + chr(x) + text_of(u[i + 1:])).encode("utf-8")
            elif kind == "repeat":
                reps = [(rid, lo, hi) for rid, (lo, hi) in enumerate(self.lang.repeats) if lo > 0 or hi is not None]
                if reps:
                    rid, lo, hi = reps[int(rng.integers(0, len(reps)))]
                    cnt = lo - 1 if (lo > 0 and (hi is None or rng.random() < 0.5)) else hi + 1
                    m = text_of(self.lang.member(override=[rid, cnt, False])).encode("utf-8")
            elif kind == "trunc" and len(text) > 1:
                m = (text[1:] if rng.random() < 0.5 else text[:-1]).encode("utf-8")
            if m is None:                                  # (the kind does not apply: a one-byte change instead)
                if not b:
                    continue
                p = int(rng.integers(0, len(b)))
                m = b[:p] + bytes([b[p] ^ 0x20]) + b[p + 1:]
                kind = "xor20"
            out.append((kind, j, L, m, R))
        return out


def make_members(rules, rng, n_members=16, n_near=3, subset=None):
    """RuleMembers of every rule (or of the rule indices in `subset`); every rule must parse and every class be covered"""
    out = []
    for ri in (range(len(rules)) if subset is None else subset):
        src, fl = rules[ri][0], rules[ri][1]
        rm = RuleMembers(ri, src, fl, rng, n_members, n_near)
        assert not rm.coverage_gaps(), (src, rm.coverage_gaps())
        out.append(rm)
    return out


# ------------------------------------------------------------------------------------------------ batch layout

TILE = 512
FILLER = (b"lorem ipsum dolor sit amet consectetur adipiscing elit sed do eiusmod tempor incididunt ut labore et dolore magna "
          b"aliqua ut enim ad minim veniam quis nostrud exercitation ullamco laboris nisi ut aliquip ex ea commodo consequat ") * 8


class MembersBatch:
    """Member messages (left + member + right) laid out in one packed batch:
      - the first byte of a rule's members falls on every residue mod 16 (each rule has 16 members or more);
      - `straddle` pieces (a rule's first piece) start at edge - d of a 512-byte tile edge, for every d in 1 .. len - 1;
      - every `cut_every`-th piece is cut in two neighbouring messages (bytes of a member on both sides of the cut;
        cut_every=None: none);
      - the batch ends with a piece whose member ends on the last byte, and its length is = `residue` mod 16.
    Filler messages (slices of FILLER) between the pieces set their alignment.  pieces: [(rule, left, member, right)]
    with bytes; kind[i] says what message i is: ('piece', piece index), ('cut', piece index) or ('fill', None)."""

    def __init__(self, pieces, residue, rng, straddle=(), cut_every=11):
        data = bytearray()
        self.off, self.kind = [0], []
        self.starts = []                       # (piece index, buffer offset of the member's first byte)
        self.straddles = []                    # (piece index, tile edge, d)
        self.pieces = pieces

        def msg(b, kind):
            data.extend(b)
            self.off.append(len(data))
            self.kind.append(kind)

        def fill(k):
            if k:
                msg(FILLER[:k], ("fill", None))

        def place(pi, member_at, cut=False):
            rule, left, mem, right = pieces[pi]
            fill(member_at - len(left) - len(data))
            assert len(data) + len(left) == member_at
            self.starts.append((pi, member_at))
            whole = left + mem + right
            if cut and len(whole) > 1:
                c = int(rng.integers(1, len(whole)))
                msg(whole[:c], ("cut", pi))
                msg(whole[c:], ("cut", pi))
            else:
                msg(whole, ("piece", pi))

        res_of = {}
        for pi, (rule, left, mem, right) in enumerate(pieces[:-1]):
            k = res_of.get(rule, 0)
            res_of[rule] = k + 1
            want = (k * 7 + rule) % 16                      # a rule's pieces in turn on the 16 residues
            at = len(data) + len(left)
            place(pi, at + (want - at) % 16, cut=cut_every is not None and pi % cut_every == cut_every - 1)
        for pi in straddle:
            rule, left, mem, right = pieces[pi]
            for d in range(1, len(mem)):
                edge = -(-(len(data) + len(left) + d) // TILE) * TILE
                place(pi, edge - d)
                self.straddles.append((pi, edge, d))
        last = len(pieces) - 1
        rule, left, mem, right = pieces[last]
        pieces[last] = (rule, left, mem, b"")
        end = len(data) + len(left) + len(mem)
        place(last, len(data) + len(left) + (residue - end) % 16)
        self.total = len(data)
        self.data = np.frombuffer(bytes(data) + b"\0" * 64, dtype=np.uint8).copy()
        self.off = np.array(self.off, dtype=np.uint32)
        self.msgs = [bytes(data[self.off[i]:self.off[i + 1]]) for i in range(len(self.off) - 1)]
        self._check(residue, cut_every)

    def _check(self, residue, cut_every):
        """the layout claims"""
        assert self.total % 16 == residue and self.kind[-1] == ("piece", len(self.pieces) - 1)
        assert self.msgs[-1].endswith(self.pieces[-1][2]) and self.pieces[-1][2]
        seen = {}
        for pi, at in self.starts:
            seen.setdefault(self.pieces[pi][0], set()).add(at % 16)
            assert bytes(self.data[at:at + len(self.pieces[pi][2])]) == self.pieces[pi][2]
        count = {}
        for p in self.pieces[:-1]:
            count[p[0]] = count.get(p[0], 0) + 1
        for rule, k in count.items():
            if k >= 16:
                assert seen[rule] == set(range(16)), rule
        starts = set(self.starts)
        by = {}
        for pi, edge, d in self.straddles:
            assert edge % TILE == 0 and (pi, edge - d) in starts
            by.setdefault(pi, set()).add(d)
        for pi, ds in by.items():
            assert ds == set(range(1, len(self.pieces[pi][2]))), pi
        if cut_every is not None:
            assert sum(1 for k in self.kind if k[0] == "cut") >= 2 * (len(self.pieces) // (cut_every + 1))

    def member_messages(self):
        """(message index, piece index) of every uncut piece"""
        return [(i, k[1]) for i, k in enumerate(self.kind) if k[0] == "piece"]


# ------------------------------------------------------------------------------------------------ the rule sets and their batches

def cortex_rules():
    import json
    import os
    c = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cortex_pack_vectors.json"), encoding="utf-8"))
    return [(p["source"], 1 if "i" in p["flags"] else 0, 3) for cats in c["packs"].values() for pats in cats.values() for p in pats]


def stratified_subset(rules, k, seed, skip=17):
    """k synthetic rules (indices >= skip), the same share of each rule form (its source's first characters) as the set"""
    rng = np.random.default_rng(seed)
    forms = {}
    for i in range(skip, len(rules)):
        src = rules[i][0]
        key = "lit" if src.isalnum() else src[:3] if src[0] in "(\\" else "pre"
        forms.setdefault(key, []).append(i)
    out = []
    for key in sorted(forms):
        idx = forms[key]
        take = max(1, round(k * len(idx) / (len(rules) - skip)))
        out += sorted(rng.choice(idx, min(take, len(idx)), replace=False).tolist())
    return sorted(out)[:k] if len(out) > k else sorted(out)


# near-miss kinds whose changed byte folds to the byte it replaced in the gram filter (case bit and bit 7 dropped, digits
# and : ; < = > ? collapsed): a near miss of one of these kinds flags exactly the grams its member flags
FOLDING_KINDS = ("xor20", "xor80", "xorA0", "digit")
# rules none of whose generated members can match: \B needs a word character on both sides of "mid", and the
# neighbours put around members are word characters on both sides too rarely
UNSATISFIABLE = {r"\Bmid\B"}


class Case:
    """A rule set with a member batch and a near-miss batch (and the member pieces again, laid out anew, at a third
    residue of the total length).  For every near-miss kind of FOLDING_KINDS, `folding[kind]` = (the near misses of that
    kind, their members) as two batches with the same layout, byte for byte apart from the changed bytes."""

    def __init__(self, name, rules, options, seed, subset=None, n_members=16, n_near=3):
        self.name, self.rules, self.options = name, rules, options
        rng = np.random.default_rng(seed)
        self.rm = make_members(rules, rng, n_members=n_members, n_near=n_near, subset=subset)
        members, near = [], []
        src = {}
        for r in self.rm:
            members += [(r.rule, L.encode(), t.encode("utf-8"), R.encode()) for L, t, R in r.members]
            for kind, j, L, m, R in r.near:
                near.append((r.rule, L, m, R))
                L0, t, R0 = r.members[j]
                src.setdefault(kind, []).append(((r.rule, L, m, R), (r.rule, L0.encode(), t.encode("utf-8"), R0.encode())))
        order = rng.permutation(len(members))
        members = [members[i] for i in order]
        near = [near[i] for i in rng.permutation(len(near))]
        # every rule's longest-but-bounded member of the first few straddles a tile edge at every offset
        first = {}
        for pi, p in enumerate(members[:-1]):
            if len(p[2]) >= 2 and (p[0] not in first or len(p[2]) > len(members[first[p[0]]][2])) and len(p[2]) <= 48:
                first[p[0]] = pi
        nfirst = {}
        for pi, p in enumerate(near[:-1]):
            if 2 <= len(p[2]) <= 48 and p[0] not in nfirst:
                nfirst[p[0]] = pi
        self.members = MembersBatch(list(members), 0, rng, straddle=sorted(first.values()))
        self.near = MembersBatch(list(near), 1, rng, straddle=sorted(nfirst.values()))
        order = rng.permutation(len(members))
        self.again = MembersBatch([members[i] for i in order], 15, rng)
        self.folding = {}
        for k, kind in enumerate(FOLDING_KINDS):
            pairs = src.get(kind, [])
            if len(pairs) < 2:
                continue
            nb = MembersBatch([p[0] for p in pairs], 0, np.random.default_rng(seed + k), cut_every=None)
            mb = MembersBatch([p[1] for p in pairs], 0, np.random.default_rng(seed + k), cut_every=None)
            assert np.array_equal(nb.off, mb.off) and int((nb.data != mb.data).sum()) <= len(pairs), kind
            self.folding[kind] = (nb, mb)

    def batches(self):
        return [("members", self.members), ("near misses", self.near), ("members again", self.again)]


def build_case(name):
    from helpers import EDGE_RULES, PACK_RULES
    from vainplex_openclaw_b200 import workload as W
    if name == "builtins":
        return Case(name, W.rules_as_tuples(W.make_rules(17)), 0, seed=17, n_members=32)
    if name in ("syn500-s2", "syn500-s4"):
        return Case(name, W.rules_as_tuples(W.make_rules(500)), 2 if name.endswith("s2") else 4, seed=500)
    if name == "syn5000":
        rules = W.rules_as_tuples(W.make_rules(5000))
        # (one near miss per member: the oracle decides every message against 5000 rules)
        return Case(name, rules, 0, seed=5000, subset=list(range(17)) + stratified_subset(rules, 400, seed=5000), n_near=1)
    if name == "non-ascii":
        return Case(name, PACK_RULES + cortex_rules() + EDGE_RULES, 0, seed=92, n_members=32)
    raise KeyError(name)


CASES = ["builtins", "syn500-s2", "syn500-s4", "syn5000", "non-ascii"]


class Expected:
    """The oracle's answers for the messages of a rule set's batches, each distinct message decided once (a message's
    results depend on its own bytes only): result words, (msg, rule) hits and resolved spans (msg, rule, start16, end16)."""

    CATS = ["credential", "financial", "pii", "custom"]

    def __init__(self, O, rules):
        from helpers import oracle_regexes
        self.O, self.rules = O, rules
        self.regs = oracle_regexes(O, rules)
        assert all(r is not None for r in self.regs)
        self.pats = [(self.regs[i], self.CATS[rules[i][2]]) for i in range(len(rules))]
        self.memo = {}

    def _decide(self, msgs):
        new = sorted({m for m in msgs if m not in self.memo})
        if not new:
            return
        data, off = self.O.pack(new)
        bits, words = self.O.scan_policy(self.regs, data, off)
        spans = self.O.find_matches_batch(self.pats, data, off)
        per = [[] for _ in new]
        for m, r, s, e in spans.tolist():
            per[m].append((r, s, e))
        R = len(self.rules)
        for i, m in enumerate(new):
            hit = np.nonzero(np.unpackbits(bits[i], bitorder="little")[:R])[0].tolist()
            self.memo[m] = (int(words[i]), hit, per[i])

    def of(self, msgs):
        """-> (words uint64[n], hits [(msg, rule)], spans [(msg, rule, start16, end16)])"""
        self._decide(msgs)
        words = np.array([self.memo[m][0] for m in msgs], dtype=np.uint64)
        hits = [(i, r) for i, m in enumerate(msgs) for r in self.memo[m][1]]
        spans = [(i, r, s, e) for i, m in enumerate(msgs) for r, s, e in self.memo[m][2]]
        return words, hits, spans


def strength(case, exp):
    """-> (rules with fewer than 10 distinct oracle-positive members in the member batch, distinct pieces of the member and
    near-miss batches that match the rule they were made from, distinct pieces that do not).  A piece is one member or
    near miss with its neighbours; it counts once however often it is placed, and only if one placement is uncut."""
    pos = {r.rule: 0 for r in case.rm}
    n_pos = n_neg = 0
    for name, b in case.batches()[:2]:
        hs = set(exp.of(b.msgs)[1])
        hit = {pi: (i, b.pieces[pi][0]) in hs for i, pi in b.member_messages()}
        for pi, h in hit.items():
            n_pos += h
            n_neg += not h
            if name == "members":
                pos[b.pieces[pi][0]] += h
    return sorted(r for r, k in pos.items() if k < 10), n_pos, n_neg


def check_strength(case, exp):
    """every rule has 10 distinct positive members but exactly the UNSATISFIABLE ones of the set; 30 % of the distinct
    pieces do not match their rule -> (pieces matching, pieces not matching)"""
    weak, n_pos, n_neg = strength(case, exp)
    assert {case.rules[r][0] for r in weak} == UNSATISFIABLE & {case.rules[r.rule][0] for r in case.rm}, [case.rules[r][0] for r in weak]
    assert n_neg >= 0.3 * (n_pos + n_neg), (n_pos, n_neg)
    return n_pos, n_neg
