"""Host-side mirror of the @vainplex/openclaw-governance plugin interface for the hot path.

Node.js is not available in this image or on the GPU box, so the host layer above the C ABI is
written in Python with the reference's own names, argument meaning and error behaviour (the
TypeScript equivalent a maintainer would ship is sketched in INTEGRATION.md).  Everything that
matches or hashes goes through the C ABI (include/openclaw_gov.h) to the CUDA kernels; this file
only holds the host logic the reference also keeps on the host:

  PatternRegistry    gov/src/redaction/registry.ts:165-316   (findMatches -> cg_find_matches_one / cg_redact_one, and
                     for the strings of one scanned value cg_find_matches_few / cg_redact_few)
  RedactionVault     gov/src/redaction/vault.ts:39-258        (sha256 -> cg_sha256_batch)
  RedactionEngine    gov/src/redaction/engine.ts:38-191
  evaluate_allowlist gov/src/redaction/allowlist.ts:35-85
  validate_regex / build_regex_cache   gov/src/policy-loader.ts:12-31,88-133
  matches_any        gov/src/conditions/context.ts:9-25       (RegExp.test -> cg_scan_batch)
  MessagePolicy      gov/src/policy-evaluator.ts:44-146 (messageContains rules only: deny > audit > allow)
  register(api)      gov/index.ts:66-115, gov/src/hooks.ts:883-916, gov/src/redaction/hooks.ts:97-142

A device failure surfaces as GovError inside the same try/except blocks where the reference
catches exceptions, so `failMode` ("open" | "closed") still decides -- there is no CPU fallback.
"""
from __future__ import annotations

import json
import re
import time
from typing import Any, Callable, Dict, Iterable, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import _native as N
from .workload import BUILTIN_RULES

CATEGORY_ORDER = ("credential", "financial", "pii", "custom")
_CAT_ID = {c: i for i, c in enumerate(CATEGORY_ORDER)}
MAX_DEPTH = 20
MAX_JSON_PARSE_LENGTH = 1_000_000
_NESTED_QUANTIFIER_RE = re.compile(r"(\+|\*|\{)\)(\+|\*|\{)")
MAX_PATTERN_LENGTH = 500


class NullLogger:
    def info(self, *_a): pass
    def warn(self, *_a): pass
    def error(self, *_a): pass
    def debug(self, *_a): pass


def _js_len(s: str) -> int:
    return len(s.encode("utf-16-le", "surrogatepass")) // 2


def _slice16(s: str, a: int, b: int) -> str:
    """s.slice(a, b) with JS (UTF-16) indices."""
    if s.isascii():
        return s[a:b]
    u = s.encode("utf-16-le", "surrogatepass")
    return u[2 * a:2 * b].decode("utf-16-le", "surrogatepass")


# ------------------------------------------------------------------------------------- registry

class PatternRegistry:
    """registry.ts:165-316.  Patterns: dicts {id, category, source, flags, builtin}."""

    def __init__(self, enabled_categories: Iterable[str], custom_patterns: Sequence[dict] = (), logger=None):
        self.logger = logger or NullLogger()
        enabled = set(enabled_categories)
        self.patterns: List[dict] = []
        for pid, cat, src, fl in BUILTIN_RULES:
            cname = CATEGORY_ORDER[cat]
            if cname in enabled:
                self.patterns.append({"id": pid, "category": cname, "source": src, "flags": fl, "builtin": True})
        for cp in custom_patterns:
            # compileCustomPattern (registry.ts:249-281): syntax errors are rejected with a warning.  The
            # reference's timing-based ReDoS probe is replaced by a static check: patterns outside the
            # supported subset or over the program-size limit are rejected (no backtracking on this path).
            rc = N.rule_check(cp["regex"], 0)
            if rc != 0:
                self.logger.warn('[redaction] Custom pattern "%s" failed to compile (%d)' % (cp["name"], rc))
                continue
            self.patterns.append({"id": "custom-" + cp["name"], "category": cp["category"], "source": cp["regex"],
                                  "flags": 0, "builtin": False})
        self._ruleset = None
        self.logger.info("[redaction] Registry initialized: %d patterns (%d built-in, %d custom)" % (
            len(self.patterns), sum(p["builtin"] for p in self.patterns), sum(not p["builtin"] for p in self.patterns)))

    def get_patterns(self):
        return self.patterns

    def get_by_category(self, category: str):
        return [p for p in self.patterns if p["category"] == category]

    def is_credential_category(self, category: str) -> bool:
        return category == "credential"

    def _rs(self) -> Optional[N.Ruleset]:
        if self._ruleset is None and self.patterns:
            self._ruleset = N.Ruleset([(p["source"], p["flags"], _CAT_ID[p["category"]]) for p in self.patterns], strict=True)
        return self._ruleset

    def find_matches_batch(self, inputs: Sequence[str]) -> List[List[dict]]:
        """findMatches for many strings in one device call."""
        out: List[List[dict]] = [[] for _ in inputs]
        rs = self._rs()
        if rs is None or not inputs:
            return out
        data, off = N.pack([N.js_utf8(s) for s in inputs])
        for sp in rs.find_matches_batch(data, off):
            s = inputs[int(sp["msg"])]
            a, b = int(sp["start16"]), int(sp["end16"])
            out[int(sp["msg"])].append({"pattern": self.patterns[int(sp["rule"])], "match": _slice16(s, a, b), "start": a, "end": b})
        return out

    def find_matches(self, input, redact: bool = False):
        """findMatches for one string: one blocking device call.  The result is the list findMatches returns.

        redact=False: cg_find_matches_one.  redact=True (RedactionEngine's scanString path): cg_redact_one, which finds the
        same matches and also splices the default placeholders and hashes every match on the device; the result then carries
        that in .redacted (see Matches).  Both go through this method so that a failing device call surfaces here, where
        the reference's engine calls findMatches.

        input may also be a list of strings (the string leaves of one value RedactionEngine.scan walks): one Matches per
        string, from one blocking device call (cg_find_matches_few / cg_redact_few)."""
        if not isinstance(input, str):
            return self._find_matches_few(list(input), redact)
        rs = self._rs()
        if rs is None:
            return Matches()
        enc = N.js_utf8(input)
        if redact:
            out_bytes, spans, digests = rs.redact_one(enc)
            redacted = RedactedString(enc, out_bytes, spans, digests)
        else:
            spans, redacted = rs.find_matches_one(enc), None
        out = Matches(redacted=redacted)
        for sp in spans:
            a, b = int(sp["start16"]), int(sp["end16"])
            out.append({"pattern": self.patterns[int(sp["rule"])], "match": _slice16(input, a, b), "start": a, "end": b})
        return out


    def _find_matches_few(self, inputs: List[str], redact: bool) -> List["Matches"]:
        rs = self._rs()
        if rs is None or not inputs:
            return [Matches() for _ in inputs]
        enc = [N.js_utf8(s) for s in inputs]
        data, off = N.pack(enc)
        if redact:
            out_bytes, out_off, spans, digests = rs.redact_few(data, off)
        else:
            spans = rs.find_matches_few(data, off)
        first = np.searchsorted(spans["msg"], np.arange(len(inputs) + 1))      # (spans come sorted by (msg, start))
        res = []
        for m, s in enumerate(inputs):
            a, b = int(first[m]), int(first[m + 1])
            redacted = RedactedString(enc[m], bytes(out_bytes[int(out_off[m]):int(out_off[m + 1])]), spans[a:b], digests[a:b]) if redact else None
            out = Matches(redacted=redacted)
            for sp in spans[a:b]:
                x, y = int(sp["start16"]), int(sp["end16"])
                out.append({"pattern": self.patterns[int(sp["rule"])], "match": _slice16(s, x, y), "start": x, "end": y})
            res.append(out)
        return res


class RedactedString(NamedTuple):
    """what cg_redact_one returns for one string: its UTF-8 bytes, the redacted bytes with the default placeholders, the
    resolved spans and the SHA-256 of every match"""
    enc: bytes
    out: bytes
    spans: np.ndarray
    digests: np.ndarray


class Matches(list):
    """PatternRegistry.find_matches' result: the list findMatches returns; .redacted is the device's RedactedString when
    it was asked for (redact=True), else None."""

    def __init__(self, items=(), redacted: Optional[RedactedString] = None):
        super().__init__(items)
        self.redacted = redacted


# ------------------------------------------------------------------------------------- vault

def sha256_hex(strings: Sequence[str]) -> List[str]:
    """createHash('sha256').update(s).digest('hex') for each string (util.ts:77-79) on the device."""
    if not strings:
        return []
    enc = [N.js_utf8(s) for s in strings]
    off = np.zeros(len(enc) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(e) for e in enc])
    data = np.frombuffer(b"".join(enc) + b"\0" * 64, dtype=np.uint8).copy()
    return [bytes(d).hex() for d in N.sha256_batch(data, off)]


class RedactionVault:
    """vault.ts:39-258.  Never persisted, never logged."""

    PLACEHOLDER_RE = re.compile(r"\[REDACTED:(?:credential|pii|financial|custom):([a-f0-9]{8,12})\]")

    def __init__(self, logger=None, expiry_seconds: Optional[float] = None, clock: Callable[[], float] = time.time):
        self.logger = logger or NullLogger()
        self.expiry = 3600 if expiry_seconds is None else expiry_seconds
        self.entries: Dict[str, dict] = {}
        self.hash_index: Dict[str, List[str]] = {}
        self.clock = clock

    def _now_ms(self) -> float:
        return self.clock() * 1000.0

    def store(self, original: str, category: str, full_hash: Optional[str] = None) -> str:
        full_hash = full_hash or sha256_hex([original])[0]
        hash8 = full_hash[:8]
        now = self._now_ms()
        existing = self.entries.get(full_hash)
        if existing and existing["expiresAt"] > now:
            return existing["placeholder"]
        hs = hash8
        for h in self.hash_index.get(hash8, []):
            e = self.entries.get(h)
            if e and h != full_hash and e["expiresAt"] > now:
                hs = full_hash[:12]
                break
        placeholder = "[REDACTED:%s:%s]" % (category, hs)
        self.entries[full_hash] = {"original": original, "category": category, "placeholder": placeholder, "hash": full_hash,
                                   "createdAt": now, "expiresAt": now + self.expiry * 1000.0}
        idx = self.hash_index.setdefault(hash8, [])
        if full_hash not in idx:
            idx.append(full_hash)
        return placeholder

    def resolve_by_hash(self, hash_slice: str) -> Optional[str]:
        now = self._now_ms()
        if len(hash_slice) == 8:
            for fh in self.hash_index.get(hash_slice, []):
                e = self.entries.get(fh)
                if e and e["expiresAt"] > now and hash_slice in e["placeholder"]:
                    return e["original"]
            return None
        for fh, e in self.entries.items():
            if fh.startswith(hash_slice) and e["expiresAt"] > now and hash_slice in e["placeholder"]:
                return e["original"]
        return None

    def resolve(self, placeholder: str) -> Optional[str]:
        m = self.PLACEHOLDER_RE.search(placeholder)
        return self.resolve_by_hash(m.group(1)) if m else None

    def resolve_all(self, text: str):
        unresolved: List[str] = []

        def rep(m):
            o = self.resolve_by_hash(m.group(1))
            if o is not None:
                return o
            unresolved.append(m.group(1))
            return m.group(0)
        return {"resolved": self.PLACEHOLDER_RE.sub(rep, text), "unresolvedHashes": unresolved}

    @property
    def size(self) -> int:
        now = self._now_ms()
        return sum(1 for e in self.entries.values() if e["expiresAt"] > now)

    def evict_expired(self) -> int:
        now = self._now_ms()
        dead = [h for h, e in self.entries.items() if e["expiresAt"] <= now]
        for h in dead:
            del self.entries[h]
            lst = [x for x in self.hash_index.get(h[:8], []) if x != h]
            if lst:
                self.hash_index[h[:8]] = lst
            else:
                self.hash_index.pop(h[:8], None)
        return len(dead)

    def clear(self):
        self.entries.clear()
        self.hash_index.clear()


# ------------------------------------------------------------------------------------- engine

def credential_views(patterns: Sequence[dict]) -> Tuple[List[dict], List[int], List[int]]:
    """One rule set for both engines of the redaction hooks: the registry's patterns, then every credential built-in the
    configured categories left out.  -> (patterns of that set, the view of the registry's patterns, the view of the
    credential built-ins in BUILTIN_RULES order -- credentialOnlyEngine's rules, src/redaction/hooks.ts:79-81)."""
    ext = list(patterns)
    have = {p["id"] for p in patterns if p["builtin"]}
    for pid, cat, src, fl in BUILTIN_RULES:
        if CATEGORY_ORDER[cat] == "credential" and pid not in have:
            ext.append({"id": pid, "category": "credential", "source": src, "flags": fl, "builtin": True})
    cred = {pid for pid, cat, _s, _f in BUILTIN_RULES if CATEGORY_ORDER[cat] == "credential"}
    return ext, list(range(len(patterns))), [i for i, p in enumerate(ext) if p["builtin"] and p["id"] in cred]


class RedactionEngine:
    """engine.ts:38-191."""

    def __init__(self, registry: PatternRegistry, vault: RedactionVault):
        self.registry, self.vault = registry, vault
        self._views = None            # (rule set with the credential view, its patterns): scan_strings(credential_only=...)

    def scan_string(self, input: str):
        cats, count = set(), [0]
        out = self._redact_string(input, cats, count)
        return {"output": out, "redactionCount": count[0], "categories": cats}

    def scan(self, input: Any):
        """scan / scanValue / scanStringValue (engine.ts:53-147) in three passes: the walk records, in walk order, every string
        that scanStringValue would redact and a skeleton of the value; one device call (registry.find_matches on the list,
        cg_redact_few) finds, hashes and splices all of them; the replay stores the matches in the vault string by string in
        walk order (right to left inside each string, as applyReplacements does) and rebuilds the value.  Output, counts,
        categories and the vault equal a walk that redacts leaf by leaf.  A value without strings makes no device call; when
        the call fails nothing reaches the vault."""
        t0 = time.perf_counter()
        cats, count = set(), [0]
        leaves: List[str] = []
        skeleton = self._walk(input, set(), 0, leaves, [])
        found = self.registry.find_matches(leaves, redact=True) if leaves else []
        done = []
        for s, matches in zip(leaves, found):
            if not matches:
                done.append(s)
                continue
            r = matches.redacted
            counter = {"redactionCount": 0}
            done.append(self._store_and_splice(s, r.enc, r.out, r.spans, r.digests, cats, counter))
            count[0] += counter["redactionCount"]
        out = self._rebuild(skeleton, done)
        return {"output": out, "redactionCount": count[0], "categories": cats, "elapsedMs": (time.perf_counter() - t0) * 1e3}

    # skeleton nodes: (_LEAF, i) the i-th recorded string; (_JSON, node) a string that held JSON, dumped again; (_LIST,
    # [nodes]); (_DICT, [(key, node)]); (_KEEP, value) a value returned as it is
    _LEAF, _JSON, _LIST, _DICT, _KEEP = range(5)

    def _walk(self, value, seen, depth, leaves: List[str], keep: list):
        """scanValue's walk (engine.ts:94-126) without the redaction: the same depth limit, the same seen rule (a second
        reference to an object becomes "[Circular]") and the same JSON-in-string parse.  keep holds the parsed values, so
        that no id in seen is reused while the walk runs."""
        if depth > MAX_DEPTH or value is None:
            return (self._KEEP, value)
        if isinstance(value, str):
            t = value.lstrip()
            if _js_len(value) <= MAX_JSON_PARSE_LENGTH and (t.startswith("{") or t.startswith("[")):
                try:
                    parsed = json.loads(value)
                    if isinstance(parsed, (dict, list)):
                        keep.append(parsed)
                        return (self._JSON, self._walk(parsed, seen, depth + 1, leaves, keep))
                except ValueError:
                    pass
            leaves.append(value)
            return (self._LEAF, len(leaves) - 1)
        if isinstance(value, (list, dict)):
            if id(value) in seen:
                return (self._KEEP, "[Circular]")
            seen.add(id(value))
            if isinstance(value, list):
                return (self._LIST, [self._walk(v, seen, depth + 1, leaves, keep) for v in value])
            return (self._DICT, [(k, self._walk(v, seen, depth + 1, leaves, keep)) for k, v in value.items()])
        return (self._KEEP, value)

    def _rebuild(self, node, done: List[str]):
        kind, x = node
        if kind == self._LEAF:
            return done[x]
        if kind == self._JSON:
            return json.dumps(self._rebuild(x, done), separators=(",", ":"), ensure_ascii=False)
        if kind == self._LIST:
            return [self._rebuild(v, done) for v in x]
        if kind == self._DICT:
            return {k: self._rebuild(v, done) for k, v in x}
        return x

    def scan_strings(self, inputs: Sequence[str], credential_only: Optional[Sequence[bool]] = None) -> List[dict]:
        """scanString (engine.ts:74-85) for many strings with the splice done on the device (cg_redact_batch): matches,
        SHA-256 of every match and the redacted text come back from one call; the vault learns the originals here, in the
        same loop as scan_string (_store_and_splice), so both give scanString's result.  A string is spliced on the host,
        with the placeholders the vault returned (vault.store runs once per match), when the vault issues its 12-digit form
        (another live value shares hash8, vault.ts:85-104), when the string has a lone surrogate or a match splits a
        surrogate pair, or when several empty matches share a position (applyReplacements puts the last one first).

        credential_only: one flag per string; a flagged string is scanned as credentialOnlyEngine scans an exempt tool's
        output (the credential built-ins only, src/redaction/hooks.ts:79-81,176-178,218-222), the others as this engine
        scans them -- in one call (cg_redact_batch_views), on one rule set with a view for each."""
        patterns = self.registry.patterns
        if credential_only is not None:
            if self._views is None:
                ext, full, cred = credential_views(self.registry.patterns)
                rs = N.Ruleset([(p["source"], p["flags"], _CAT_ID[p["category"]]) for p in ext], strict=True)
                rs.set_views([full, cred])
                self._views = (rs, ext)
            rs, patterns = self._views
            views = np.array([1 if f else 0 for f in credential_only], dtype=np.uint8)
            assert len(views) == len(inputs), "one credential_only flag per string"
        else:
            rs, views = self.registry._rs(), None
        if rs is None or not inputs:
            return [{"output": s, "redactionCount": 0, "categories": set()} for s in inputs]
        enc = [N.js_utf8(s) for s in inputs]
        data, off = N.pack(enc)
        out, out_off, spans, digests = rs.redact_batch(data, off, views=views)
        res = [{"output": s, "redactionCount": 0, "categories": set()} for s in inputs]
        first = np.searchsorted(spans["msg"], np.arange(len(inputs) + 1)) if len(spans) else None
        for m in (np.unique(spans["msg"]) if len(spans) else ()):
            m = int(m)
            a, b = int(first[m]), int(first[m + 1])
            r = res[m]
            r["output"] = self._store_and_splice(inputs[m], enc[m], bytes(out[int(out_off[m]):int(out_off[m + 1])]), spans[a:b], digests[a:b],
                                                 r["categories"], r, patterns)
        return res

    def _redact_string(self, input: str, cats, count) -> str:
        """scanString's splice for one string: one blocking device call (cg_redact_one) gives the spans, the SHA-256 of every
        match and the redacted text; the vault learns the originals here."""
        matches = self.registry.find_matches(input, redact=True)
        if not matches:
            return input
        r = matches.redacted
        counter = {"redactionCount": 0}
        result = self._store_and_splice(input, r.enc, r.out, r.spans, r.digests, cats, counter)
        count[0] += counter["redactionCount"]
        return result

    def _store_and_splice(self, s: str, enc: bytes, out: bytes, spans, digests, cats, counter: dict, patterns=None) -> str:
        """applyReplacements (engine.ts:165-181) for the resolved spans of one string s (enc = its UTF-8 bytes, out = the
        device's redacted bytes): vault.store for every match, last match first, with the device's SHA-256 of the match.
        The device text is the answer unless the vault issued a placeholder other than the default 8-digit one (another live
        value shares hash8, vault.ts:85-104), or the bytes cannot stand for the JS string (a lone surrogate, a match that
        splits a surrogate pair, several empty matches at one position): then s is spliced on the host, right to left, with
        the placeholders the vault returned."""
        starts = [int(x) for x in spans["start16"]]
        order = sorted(range(len(starts)), key=lambda i: -starts[i])          # the reference's order: by start, descending, stable
        device_text = len(set(starts)) == len(starts)
        try:
            device_text = device_text and s.encode("utf-8") == enc
        except UnicodeEncodeError:
            device_text = False
        reps = []
        for i in order:
            sp = spans[i]
            a, b = starts[i], int(sp["end16"])
            match = _slice16(s, a, b)
            if N.js_utf8(match) == enc[int(sp["start_byte"]):int(sp["end_byte"])]:
                h = bytes(digests[i]).hex()
            else:                                                            # the device hashed other bytes than createHash() would
                h = sha256_hex([match])[0]
                device_text = False
            cat = (patterns or self.registry.patterns)[int(sp["rule"])]["category"]
            ph = self.vault.store(match, cat, h)
            device_text = device_text and ph == "[REDACTED:%s:%s]" % (cat, h[:8])
            reps.append((a, b, ph))
            counter["redactionCount"] += 1
            cats.add(cat)
        if device_text:
            return out.decode("utf-8", "surrogatepass")
        result = s
        for a, b, ph in reps:
            result = _slice16(result, 0, a) + ph + _slice16(result, b, _js_len(result))
        return result


def evaluate_allowlist(category: str, context: dict, allowlist: dict):
    """allowlist.ts:35-85."""
    if category == "credential":
        return {"allowed": False, "reason": "Credentials are never allowlisted"}
    if context.get("toolName") and context["toolName"] in allowlist.get("exemptTools", []):
        return {"allowed": True, "reason": 'Tool "%s" is exempt from redaction' % context["toolName"]}
    if context.get("agentId") and context["agentId"] in allowlist.get("exemptAgents", []):
        return {"allowed": True, "reason": 'Agent "%s" is exempt from outbound redaction' % context["agentId"]}
    if category == "pii" and context.get("channel") in allowlist.get("piiAllowedChannels", []) and context.get("channel"):
        return {"allowed": True, "reason": 'PII allowed on channel "%s"' % context["channel"]}
    if category == "financial" and context.get("channel") in allowlist.get("financialAllowedChannels", []) and context.get("channel"):
        return {"allowed": True, "reason": 'Financial data allowed on channel "%s"' % context["channel"]}
    return {"allowed": False, "reason": "No allowlist match"}


# ------------------------------------------------------------------------------------- policy scan

def validate_regex(pattern: str):
    """policy-loader.ts:15-31."""
    if _js_len(pattern) > MAX_PATTERN_LENGTH:
        return {"valid": False, "error": "Pattern exceeds %d chars" % MAX_PATTERN_LENGTH}
    if _NESTED_QUANTIFIER_RE.search(pattern):
        return {"valid": False, "error": "Nested quantifiers detected (ReDoS risk)"}
    rc = N.rule_check(pattern, 0)
    if rc == N.CG_ERR_SYNTAX:
        return {"valid": False, "error": "Invalid regular expression"}
    return {"valid": True}


def _escape_literal(s: str) -> str:
    return re.sub(r"([\\^$.*+?()\[\]{}|/])", r"\\\1", s)


class RuleScanner:
    """The rule-set side of matchesAny (context.ts:9-25) for a *set* of messageContains rules.

    rules: list of pattern lists (a rule matches when ANY of its patterns does).  A pattern with a
    syntax error falls back to `text.includes(pattern)` exactly like the reference (context.ts:15-17):
    it is compiled as an escaped literal.  Patterns rejected by validate_regex are still evaluated
    (context.ts:12-14 compiles them on every call)."""

    def __init__(self, rules: Sequence[Sequence[str]], logger=None):
        self.logger = logger or NullLogger()
        self.rule_of_pattern: List[int] = []
        srcs = []
        for ri, pats in enumerate(rules):
            for p in ([pats] if isinstance(pats, str) else pats):
                rc = N.rule_check(p, 0)
                if rc == N.CG_ERR_SYNTAX:
                    p = _escape_literal(p)
                elif rc != 0:
                    raise N.GovError(rc, "pattern outside the supported subset: %r" % p)
                srcs.append((p, 0, 3))
                self.rule_of_pattern.append(ri)
        self.n_rules = len(rules)
        self.ruleset = N.Ruleset(srcs, strict=True) if srcs else None

    def scan(self, texts: Sequence[str]) -> List[List[int]]:
        """-> for each text the sorted list of rule indices whose messageContains matches."""
        out: List[List[int]] = [[] for _ in texts]
        if self.ruleset is None or not texts:
            return out
        data, off = N.pack([N.js_utf8(t) for t in texts])
        _words, hits = self.ruleset.scan_batch(data, off)
        for h in hits:
            r = self.rule_of_pattern[int(h["rule"])]
            lst = out[int(h["msg"])]
            if not lst or lst[-1] != r:
                if r not in lst:
                    lst.append(r)
        for lst in out:
            lst.sort()
        return out


def matches_any(patterns, texts: Sequence[str], scanner_cache: Optional[dict] = None) -> bool:
    """context.ts:9-25 for one condition (convenience; batch callers use RuleScanner directly)."""
    lst = [patterns] if isinstance(patterns, str) else list(patterns)
    key = tuple(lst)
    sc = scanner_cache.get(key) if scanner_cache is not None else None
    if sc is None:
        sc = RuleScanner([lst])
        if scanner_cache is not None:
            scanner_cache[key] = sc
    return any(sc.scan(list(texts)))


class MessagePolicy:
    """The messageContains slice of the policy pipeline (policy-evaluator.ts:44-146): policies sorted by
    priority (desc), per policy the first matching rule counts, deny > audit > allow, first deny reason."""

    def __init__(self, policies: Sequence[dict], logger=None):
        self.policies = sorted([p for p in policies if p.get("enabled", True)], key=lambda p: -p.get("priority", 0))
        self.index = []          # (policy idx, rule idx)
        rules = []
        for pi, p in enumerate(self.policies):
            for ri, r in enumerate(p["rules"]):
                rules.append(r["messageContains"])
                self.index.append((pi, ri))
        self.scanner = RuleScanner(rules, logger)
        self._views_set = None        # the views last given to the rule set (verdict_batch with contexts)

    def evaluate_batch(self, texts: Sequence[str]) -> List[dict]:
        res = []
        for hit in self.scanner.scan(texts):
            per_policy: Dict[int, int] = {}
            for h in hit:
                pi, ri = self.index[h]
                if pi not in per_policy or ri < per_policy[pi]:
                    per_policy[pi] = ri
            action, reason, matched = "allow", "No matching policies", []
            for pi in sorted(per_policy):
                rule = self.policies[pi]["rules"][per_policy[pi]]
                eff = rule.get("effect", {"action": "deny"})
                matched.append({"policyId": self.policies[pi]["id"], "action": eff["action"]})
                if eff["action"] == "deny" and action != "deny":
                    action, reason = "deny", eff.get("reason", "Denied by policy %s" % self.policies[pi]["id"])
                elif eff["action"] == "audit" and action == "allow":
                    action, reason = "audit", eff.get("reason", "")
            res.append({"action": action, "reason": reason, "matches": matched})
        return res

    def evaluate(self, text: str) -> dict:
        return self.evaluate_batch([text])[0]

    ACTIONS = ("allow", "audit", "deny")

    def verdict_batch(self, texts: Sequence[str], contexts: Optional[Sequence[dict]] = None) -> List[dict]:
        """Same action / reason as evaluate_batch, aggregated on the device (cg_policy_verdict_batch): one verdict word
        per message comes back instead of the hit list (the `matches` list is not materialised).

        contexts: one per text; then only the policies whose scope (excludeAgents, channels: matchesScope,
        policy-evaluator.ts:18-26) admits the text's context take part -- one view per distinct in-scope policy set of the
        batch (cg_policy_verdict_batch_views)."""
        rs = self.scanner.ruleset
        if rs is None or not texts:
            return [{"action": "allow", "reason": "No matching policies", "matchedPolicies": 0} for _ in texts]
        if not getattr(self, "_policy_set", False):
            pol, act = [], []
            for pat_rule in self.scanner.rule_of_pattern:
                pi, ri = self.index[pat_rule]
                eff = self.policies[pi]["rules"][ri].get("effect", {"action": "deny"})
                pol.append(pi); act.append(self.ACTIONS.index(eff["action"]))
            rs.set_policy(pol, act)
            self._policy_set = True
        if contexts is None:
            data, off = N.pack([N.js_utf8(t) for t in texts])
            words = rs.verdict_batch(data, off).tolist()
        else:
            assert len(contexts) == len(texts), "one context per text"
            pattern_policy = [self.index[r][0] for r in self.scanner.rule_of_pattern]
            views, ids = scope_views(self.policies, pattern_policy, contexts)
            words = [0] * len(texts)
            for v0 in range(0, len(views), 256):                # (at most 256 views per call)
                sel = [i for i in range(len(texts)) if v0 <= ids[i] < v0 + 256]
                if views[v0:v0 + 256] != self._views_set:        # (set_views waits for the stream and replaces the rows)
                    rs.set_views(views[v0:v0 + 256])
                    self._views_set = views[v0:v0 + 256]
                data, off = N.pack([N.js_utf8(texts[i]) for i in sel])
                for i, w in zip(sel, rs.verdict_batch(data, off, views=[ids[i] - v0 for i in sel]).tolist()):
                    words[i] = w
        out = []
        for v in words:
            action, matched, decide = self.ACTIONS[v & 3], (v >> 2) & 1023, v >> 12
            reason = "No matching policies" if action == "allow" else ""
            if decide != 0xfffff and action != "allow":
                pi, ri = self.index[self.scanner.rule_of_pattern[decide]]
                eff = self.policies[pi]["rules"][ri].get("effect", {"action": "deny"})
                reason = eff.get("reason", "Denied by policy %s" % self.policies[pi]["id"]) if action == "deny" else eff.get("reason", "")
            out.append({"action": action, "reason": reason, "matchedPolicies": matched})
        return out


def scope_views(policies: Sequence[dict], pattern_policy: Sequence[int], contexts: Sequence[dict]) -> Tuple[List[List[int]], List[int]]:
    """The views of MessagePolicy.verdict_batch(texts, contexts): per context the policies its scope admits
    (PolicyEvaluator._matches_scope), one view per distinct set in order of first appearance, holding the patterns
    (pattern_policy[k] = policy of pattern k) of those policies.  -> (views, view id per context)"""
    seen: Dict[Tuple[int, ...], int] = {}
    views: List[List[int]] = []
    ids: List[int] = []
    for ctx in contexts:
        key = tuple(pi for pi, p in enumerate(policies) if PolicyEvaluator._matches_scope(p, ctx))
        if key not in seen:
            seen[key] = len(views)
            keep = set(key)
            views.append([k for k, pi in enumerate(pattern_policy) if pi in keep])
        ids.append(seen[key])
    return views, ids


# ------------------------------------------------------------------------------------- full policy slice

TIER_ORDINAL = {"untrusted": 0, "restricted": 1, "standard": 2, "trusted": 3, "elevated": 4}     # util.ts:201-210


def _glob_match(pattern: str, value: str) -> bool:
    """util.ts:68-74 globToRegex + test (anchored; `*` = `.*`, `?` = `.`; `.` does not match line terminators)."""
    import re
    esc = re.sub(r"[.+^${}()|\[\]\\]", lambda m: "\\" + m.group(0), pattern).replace("*", "[^\\n\\r\\u2028\\u2029]*").replace("?", "[^\\n\\r\\u2028\\u2029]")
    return re.fullmatch(esc, value) is not None


def _as_list(v) -> list:
    return v if isinstance(v, list) else [v]


class PolicyEvaluator:
    """policy-evaluator.ts:18-146 with every text test routed to the device in ONE batch per call:

      * matchesScope (:18-26: excludeAgents, channels), sortPolicies (:36-42: priority desc, then specificity
        agents 10 / channels 5 / hooks 3), matchPolicy (:128-146: first rule whose trust gates and conditions hold),
        aggregateMatches (:44-80: deny > 2fa > audit > allow, the reference's reason strings);
      * conditions: `context` (messageContains, conversationContains, channel, hasMetadata, sessionKey --
        conditions/context.ts:9-76), `tool` (name glob; params equals / contains / matches / startsWith / in --
        conditions/tool.ts:10-84), `agent` (id glob, trustTier), `any`, `not` (conditions/simple.ts:39-150); `time`, `risk`
        and `frequency` conditions are not on the scan path and are taken from a caller-supplied callback
        (`other_condition(cond, ctx) -> bool`, default False like an unknown evaluator, conditions/index.ts:44-46).

    Every regex of every policy (messageContains / conversationContains patterns, `matches` param matchers) is one rule
    of one device rule set; a call packs the message, the conversation entries and the tool-parameter strings of all its
    contexts into one batch, scans it once, and the boolean tree is evaluated on the host from the hit list."""

    def __init__(self, policies: Sequence[dict], logger=None, other_condition=None, scanner_cls=None):
        self.policies = [p for p in policies if p.get("enabled", True)]
        self.other = other_condition or (lambda cond, ctx: False)
        self.pattern_rule: Dict[str, int] = {}
        rules: List[List[str]] = []

        def reg(pat: str):
            if pat not in self.pattern_rule:
                self.pattern_rule[pat] = len(rules)
                rules.append([pat])

        def walk(cond):
            t = cond.get("type")
            if t == "context":
                for key in ("messageContains", "conversationContains"):
                    v = cond.get(key)
                    if v is not None:
                        for pat in ([v] if isinstance(v, str) else v):
                            reg(pat)
            elif t == "tool":
                for m in (cond.get("params") or {}).values():
                    if "matches" in m:
                        self.tool_matches.add(m["matches"])
            elif t == "any":
                for sub in cond.get("conditions", []):
                    walk(sub)
            elif t == "not":
                walk(cond["condition"])

        self.tool_matches = set()
        for p in self.policies:
            for r in p.get("rules", []):
                for c in r.get("conditions", []):
                    walk(c)
        # tool `matches` patterns: an invalid one never matches (tool.ts:39-44), unlike messageContains' includes() fallback
        self.tool_rule: Dict[str, int] = {}
        for pat in sorted(self.tool_matches):
            if N.rule_check(pat, 0) == 0:
                self.tool_rule[pat] = len(rules)
                rules.append([pat])
        self.scanner = (scanner_cls or RuleScanner)(rules, logger) if rules else None
        self._compile_program()
        self._program_rs = None          # the rule set verdict_batch evaluates the program on (the scanner's, or an empty one)

    # -- the policy program (cg_ruleset_set_policy_program, openclaw_gov.h): verdict_batch evaluates every policy on the device
    ACTION_CODE = {"allow": 0, "audit": 1, "2fa": 2, "deny": 3}

    def _compile_program(self) -> None:
        """Policies in evaluation order (sortPolicies, policy-evaluator.ts:36-42: it depends on the policy alone and scope
        only removes policies, so one order serves every context), each rule's gates and conditions as a postfix program over
        HIT(rule, role) leaves for the regex tests and atoms for every other test (the helpers _cond and _evaluate call).
        Sets self.program (uint32 words), self.atoms ([ctx -> bool], one per atom id), self.param_role (tool-param key ->
        role 2 + k) and self.program_rules ((policy, rule) per program rule)."""
        atom_id: Dict[tuple, int] = {}
        self.atoms: List[Callable[[dict], bool]] = []
        self.param_role: Dict[str, int] = {}

        def atom_index(key: tuple, fn) -> int:
            if key not in atom_id:
                atom_id[key] = len(self.atoms)
                self.atoms.append(fn)
            return atom_id[key]

        def atom(key: tuple, fn) -> List[int]:
            return [N.POL_ATOM | atom_index(key, fn) << 3]

        def hit(rule: int, role: int) -> List[int]:
            return [N.POL_HIT | rule << 3 | role << 24]

        def fold(parts: List[List[int]], op: int, empty: int) -> List[int]:
            if not parts:
                return [N.POL_CONST | empty << 3]
            out = list(parts[0])
            for q in parts[1:]:
                out += q + [op]
            return out

        def canon(v) -> str:
            return json.dumps(v, sort_keys=True, default=repr)

        def role_of(key: str) -> int:
            if key not in self.param_role:
                if len(self.param_role) >= 254:
                    raise ValueError("more than 254 tool-param keys with a `matches` test")
                self.param_role[key] = 2 + len(self.param_role)
            return self.param_role[key]

        def cond(c: dict) -> List[int]:
            t = c.get("type")
            parts: List[List[int]] = []
            if t == "context":
                for key, role in (("conversationContains", 1), ("messageContains", 0)):
                    if c.get(key) is not None:
                        parts.append(fold([hit(self.pattern_rule[p], role) for p in _as_list(c[key])], N.POL_OR, 0))
                if c.get("hasMetadata") is not None:
                    k = _as_list(c["hasMetadata"])
                    parts.append(atom(("hasMetadata", canon(k)), lambda ctx, k=k: self._has_metadata(k, ctx)))
                if c.get("channel") is not None:
                    k = _as_list(c["channel"])
                    parts.append(atom(("channel", canon(k)), lambda ctx, k=k: self._in_channel(k, ctx)))
                if c.get("sessionKey") is not None:
                    k = c["sessionKey"]
                    parts.append(atom(("sessionKey", k), lambda ctx, k=k: self._session_key(k, ctx)))
                return fold(parts, N.POL_AND, 1)
            if t == "tool":
                if c.get("name") is not None:
                    k = _as_list(c["name"])
                    parts.append(atom(("toolName", canon(k)), lambda ctx, k=k: self._tool_name(k, ctx)))
                if c.get("params"):
                    parts.append(atom(("hasParams",), self._has_params))
                    for key, m in c["params"].items():
                        if "matches" in m and "equals" not in m and "contains" not in m:
                            pat = m["matches"]
                            parts.append(hit(self.tool_rule[pat], role_of(key)) if pat in self.tool_rule else [N.POL_CONST])
                        else:
                            parts.append(atom(("param", key, canon(m)), lambda ctx, key=key, m=m: self._param_test(key, m, ctx)))
                return fold(parts, N.POL_AND, 1)
            if t == "agent":
                if c.get("id") is not None:
                    k = _as_list(c["id"])
                    parts.append(atom(("agentId", canon(k)), lambda ctx, k=k: self._agent_id_in(k, ctx)))
                if c.get("trustTier") is not None:
                    k = _as_list(c["trustTier"])
                    parts.append(atom(("agentTier", canon(k)), lambda ctx, k=k: self._agent_tier_in(k, ctx)))
                return fold(parts, N.POL_AND, 1)
            if t == "any":
                return fold([cond(sub) for sub in c.get("conditions", [])], N.POL_OR, 0)
            if t == "not":
                return cond(c["condition"]) + [N.POL_NOT]
            return atom(("other", canon(c)), lambda ctx, c=c: bool(self.other(c, ctx)))

        order = sorted(self.policies, key=lambda p: (-(p.get("priority") or 0), -self._specificity(p)))     # stable, as _evaluate
        words: List[int] = [len(order)]
        self.program_rules: List[Tuple[dict, dict]] = []
        for p in order:
            scope = p.get("scope") or {}
            if scope.get("excludeAgents") or scope.get("channels"):
                words.append(atom_index(("scope", canon([scope.get("excludeAgents"), scope.get("channels")])), lambda ctx, p=p: self._matches_scope(p, ctx)))
            else:
                words.append(0xffffffff)
            words.append(len(p.get("rules", [])))
            for r in p.get("rules", []):
                parts = []
                if r.get("minTrust"):
                    parts.append(atom(("minTrust", r["minTrust"]), lambda ctx, t=r["minTrust"]: self._min_trust(t, ctx)))
                if r.get("maxTrust"):
                    parts.append(atom(("maxTrust", r["maxTrust"]), lambda ctx, t=r["maxTrust"]: self._max_trust(t, ctx)))
                ops = fold(parts + [cond(c) for c in r.get("conditions", [])], N.POL_AND, 1)
                eff = r.get("effect", {"action": "allow"})
                words += [self.ACTION_CODE.get(eff.get("action"), 0) | (4 if eff.get("reason") else 0), len(ops)] + ops
                self.program_rules.append((p, r))
        self.program = np.array(words, dtype=np.uint32)

    def program_inputs(self, contexts: Sequence[dict]):
        """The texts of the contexts with their roles (evaluate_batch's inclusions; a string param whose key no `matches` test
        names feeds no leaf and is left out), the contexts' text ranges and their atom rows.
        -> (texts, roles uint8[n_texts], ctx_off uint32[n_ctx + 1], atoms uint32[n_ctx, ceil(n_atoms / 32)])"""
        texts: List[str] = []
        roles: List[int] = []
        ctx_off = np.zeros(len(contexts) + 1, dtype=np.uint32)
        atoms = np.zeros((len(contexts), (len(self.atoms) + 31) // 32), dtype=np.uint32)
        for ci, ctx in enumerate(contexts):
            if ctx.get("messageContent"):
                texts.append(ctx["messageContent"]); roles.append(0)
            for t in ctx.get("conversationContext") or []:
                texts.append(t); roles.append(1)
            for key, val in (ctx.get("toolParams") or {}).items():
                if isinstance(val, str) and key in self.param_role:
                    texts.append(val); roles.append(self.param_role[key])
            ctx_off[ci + 1] = len(texts)
            for a, fn in enumerate(self.atoms):
                if fn(ctx):
                    atoms[ci, a >> 5] |= np.uint32(1 << (a & 31))
        return texts, np.array(roles, dtype=np.uint8), ctx_off, atoms

    def decode_verdicts(self, words, matches) -> List[dict]:
        """verdict words and the (ctx, rule) match list -> what evaluate_batch returns per context (action, reason, matches;
        the reason of a deny / 2fa is the first non-empty one of that action, aggregateMatches, policy-evaluator.ts:51-60)"""
        first = np.searchsorted(np.asarray(matches["ctx"]), np.arange(len(words) + 1)) if len(matches) else np.zeros(len(words) + 1, np.int64)
        out = []
        for c, v in enumerate(int(x) for x in words):
            if v >= 0xfffffffe:
                raise N.GovError(N.CG_ERR_CAPACITY, "context %d has no verdict (0x%08x)" % (c, v))
            ms = []
            for j in matches["rule"][int(first[c]):int(first[c + 1])]:
                p, r = self.program_rules[int(j)]
                ms.append({"policyId": p["id"], "ruleId": r.get("id"), "effect": r.get("effect", {"action": "allow"}), "controls": p.get("controls") or []})
            outcome, decide = v & 7, v >> 12
            if outcome >= 3:
                action = "deny" if outcome == 4 else "2fa"
                reason = self.program_rules[decide][1]["effect"]["reason"] if decide != 0xfffff else \
                    ("Denied by governance policy" if outcome == 4 else "Requires 2FA approval")
            else:
                action = "allow"
                reason = ("No matching policies", "Allowed by governance policy", "Allowed with audit logging")[outcome]
            out.append({"action": action, "reason": reason, "matches": ms})
        return out

    def verdict_batch(self, contexts: Sequence[dict]) -> List[dict]:
        """evaluate_batch's result (action, reason, matches) with the policies evaluated on the device: one policy-mode scan of
        every text of the batch, then the program for every context (cg_policy_eval_batch); only the verdict words and the
        match list come back.  Atoms are computed here for every context (a time / risk / frequency callback is called for
        each context and condition, not only where the host walk would reach it)."""
        if not contexts:
            return []
        rs = self._program_ruleset()
        texts, roles, ctx_off, atoms = self.program_inputs(contexts)
        data, off = N.pack([N.js_utf8(t) for t in texts])
        words, matches = rs.eval_batch(data, off, roles, ctx_off, atoms)
        return self.decode_verdicts(words, matches)

    def verdict_one(self, ctx: dict) -> dict:
        """verdict_batch([ctx])[0] in one blocking device round trip (cg_policy_eval_one): the hooks that evaluate one context
        per event (before_tool_call, message_sending)."""
        rs = self._program_ruleset()
        texts, roles, _ctx_off, atoms = self.program_inputs([ctx])
        data, off = N.pack([N.js_utf8(t) for t in texts])
        word, rules = rs.eval_one(data, off, roles, atoms[0])
        matches = np.array([(0, r) for r in rules], dtype=N.POLICY_MATCH_DTYPE)
        return self.decode_verdicts(np.array([word], dtype=np.uint32), matches)[0]

    def _program_ruleset(self) -> N.Ruleset:
        """the rule set the program is evaluated on (the scanner's, or an empty one), the program set on it once"""
        if self._program_rs is None:
            rs = getattr(self.scanner, "ruleset", None) if self.scanner is not None else N.Ruleset([], strict=True)
            if rs is None:
                raise TypeError("verdict_batch needs the device RuleScanner")
            rs.set_policy_program(self.program, len(self.atoms))
            self._program_rs = rs
        return self._program_rs

    # -- one batch for all contexts
    def evaluate_batch(self, contexts: Sequence[dict]) -> List[dict]:
        texts: List[str] = []
        where: List[Tuple[int, str, object]] = []          # (context index, kind, key)
        for ci, ctx in enumerate(contexts):
            if ctx.get("messageContent"):
                texts.append(ctx["messageContent"]); where.append((ci, "msg", None))
            for k, t in enumerate(ctx.get("conversationContext") or []):
                texts.append(t); where.append((ci, "conv", k))
            for key, val in (ctx.get("toolParams") or {}).items():
                if isinstance(val, str):
                    texts.append(val); where.append((ci, "param", key))
        hits = self.scanner.scan(texts) if (self.scanner and texts) else [[] for _ in texts]
        per_ctx = [{"msg": set(), "conv": set(), "param": {}} for _ in contexts]
        for (ci, kind, key), h in zip(where, hits):
            if kind == "param":
                per_ctx[ci]["param"][key] = set(h)
            else:
                per_ctx[ci][kind].update(h)
        return [self._evaluate(ctx, per_ctx[ci]) for ci, ctx in enumerate(contexts)]

    def evaluate(self, ctx: dict) -> dict:
        return self.evaluate_batch([ctx])[0]

    # -- policy-evaluator.ts
    @staticmethod
    def _matches_scope(policy: dict, ctx: dict) -> bool:
        scope = policy.get("scope") or {}
        if ctx.get("agentId") in (scope.get("excludeAgents") or []):
            return False
        ch = scope.get("channels") or []
        if ch and (not ctx.get("channel") or ctx["channel"] not in ch):
            return False
        return True

    @staticmethod
    def _specificity(policy: dict) -> int:
        scope = policy.get("scope") or {}
        return (10 if scope.get("agents") else 0) + (5 if scope.get("channels") else 0) + (3 if scope.get("hooks") else 0)

    def _evaluate(self, ctx: dict, hit: dict) -> dict:
        applicable = [p for p in self.policies if self._matches_scope(p, ctx)]
        applicable.sort(key=lambda p: (-(p.get("priority") or 0), -self._specificity(p)))        # stable, like Array.prototype.sort
        matches = []
        for p in applicable:
            for r in p.get("rules", []):
                if r.get("minTrust") and not self._min_trust(r["minTrust"], ctx):
                    continue
                if r.get("maxTrust") and not self._max_trust(r["maxTrust"], ctx):
                    continue
                if all(self._cond(c, ctx, hit) for c in r.get("conditions", [])):
                    matches.append({"policyId": p["id"], "ruleId": r.get("id"), "effect": r.get("effect", {"action": "allow"}),
                                    "controls": p.get("controls") or []})
                    break
        deny = next((m for m in matches if m["effect"]["action"] == "deny"), None)
        twofa = next((m for m in matches if m["effect"]["action"] == "2fa"), None)
        audit = any(m["effect"]["action"] == "audit" for m in matches)
        if deny:
            return {"action": "deny", "reason": deny["effect"].get("reason") or "Denied by governance policy", "matches": matches}
        if twofa:
            return {"action": "2fa", "reason": twofa["effect"].get("reason") or "Requires 2FA approval", "matches": matches}
        if audit:
            return {"action": "allow", "reason": "Allowed with audit logging", "matches": matches}
        return {"action": "allow", "reason": "Allowed by governance policy" if matches else "No matching policies", "matches": matches}

    # -- the scalar tests of conditions/*.ts and the rule gates (matchPolicy, :135-140): _cond / _evaluate call them, and
    # each distinct one is an atom of the policy program (verdict_batch)
    @staticmethod
    def _session_tier(ctx: dict) -> int:
        return TIER_ORDINAL[((ctx.get("trust") or {}).get("session") or {}).get("tier", "standard")]

    @staticmethod
    def _min_trust(tier: str, ctx: dict) -> bool:
        return PolicyEvaluator._session_tier(ctx) >= TIER_ORDINAL[tier]

    @staticmethod
    def _max_trust(tier: str, ctx: dict) -> bool:
        return PolicyEvaluator._session_tier(ctx) <= TIER_ORDINAL[tier]

    @staticmethod
    def _has_metadata(keys, ctx: dict) -> bool:
        return all(k in (ctx.get("metadata") or {}) for k in keys)

    @staticmethod
    def _in_channel(chans, ctx: dict) -> bool:
        return bool(ctx.get("channel")) and ctx["channel"] in chans

    @staticmethod
    def _session_key(glob: str, ctx: dict) -> bool:
        return bool(ctx.get("sessionKey")) and _glob_match(glob, ctx["sessionKey"])

    @staticmethod
    def _tool_name(names, ctx: dict) -> bool:
        tn = ctx.get("toolName")
        return bool(tn) and any(_glob_match(p, tn) if ("*" in p or "?" in p) else p == tn for p in names)

    @staticmethod
    def _has_params(ctx: dict) -> bool:
        return bool(ctx.get("toolParams"))

    @staticmethod
    def _param_test(key: str, m: dict, ctx: dict) -> bool:
        """a param matcher other than `matches` (tool.ts:30-60); `matches` is a scan leaf"""
        v = (ctx.get("toolParams") or {}).get(key)
        if "equals" in m:
            return v == m["equals"] and type(v) == type(m["equals"])
        if "contains" in m:
            return isinstance(v, str) and m["contains"] in v
        if "startsWith" in m:
            return isinstance(v, str) and v.startswith(m["startsWith"])
        if "in" in m:
            return v in m["in"]
        return False

    @staticmethod
    def _agent_id_in(ids, ctx: dict) -> bool:
        aid = ctx.get("agentId", "")
        return any(_glob_match(p, aid) if ("*" in p or "?" in p) else p == aid for p in ids)

    @staticmethod
    def _agent_tier_in(tiers, ctx: dict) -> bool:
        return ((ctx.get("trust") or {}).get("agent") or {}).get("tier", "standard") in tiers

    # -- conditions/*.ts
    def _any_pattern(self, patterns, hitset) -> bool:
        return any(self.pattern_rule[p] in hitset for p in ([patterns] if isinstance(patterns, str) else patterns))

    def _cond(self, c: dict, ctx: dict, hit: dict) -> bool:
        t = c.get("type")
        if t == "context":
            if c.get("conversationContains") is not None:
                if not (ctx.get("conversationContext") or []) or not self._any_pattern(c["conversationContains"], hit["conv"]):
                    return False
            if c.get("messageContains") is not None:
                if not ctx.get("messageContent") or not self._any_pattern(c["messageContains"], hit["msg"]):
                    return False
            if c.get("hasMetadata") is not None and not self._has_metadata(_as_list(c["hasMetadata"]), ctx):
                return False
            if c.get("channel") is not None and not self._in_channel(_as_list(c["channel"]), ctx):
                return False
            if c.get("sessionKey") is not None and not self._session_key(c["sessionKey"], ctx):
                return False
            return True
        if t == "tool":
            if c.get("name") is not None and not self._tool_name(_as_list(c["name"]), ctx):
                return False
            if c.get("params"):
                if not self._has_params(ctx):
                    return False
                tp = ctx["toolParams"]
                for key, m in c["params"].items():
                    if "matches" in m and "equals" not in m and "contains" not in m:
                        v = tp.get(key)
                        ok = isinstance(v, str) and m["matches"] in self.tool_rule and self.tool_rule[m["matches"]] in hit["param"].get(key, set())
                    else:
                        ok = self._param_test(key, m, ctx)
                    if not ok:
                        return False
            return True
        if t == "agent":
            if c.get("id") is not None and not self._agent_id_in(_as_list(c["id"]), ctx):
                return False
            if c.get("trustTier") is not None and not self._agent_tier_in(_as_list(c["trustTier"]), ctx):
                return False
            return True
        if t == "any":
            return any(self._cond(sub, ctx, hit) for sub in c.get("conditions", []))
        if t == "not":
            return not self._cond(c["condition"], ctx, hit)
        return bool(self.other(c, ctx))


class ResponseGate:
    """response-gate.ts:23-176: requiredTools / mustMatch / mustNotMatch validators per agent; every mustMatch /
    mustNotMatch pattern of the configuration is one rule of one device rule set, a batch of messages is scanned once.
    An invalid pattern blocks (fail-closed, :113-118,134-139)."""

    def __init__(self, config: dict, logger=None, scanner_cls=None):
        self.config = config
        self.rule_of: Dict[str, Optional[int]] = {}
        rules = []
        for rule in config.get("rules", []):
            for v in rule.get("validators", []):
                if v["type"] in ("mustMatch", "mustNotMatch") and v["pattern"] not in self.rule_of:
                    if N.rule_check(v["pattern"], 0) == 0:
                        self.rule_of[v["pattern"]] = len(rules); rules.append([v["pattern"]])
                    else:
                        self.rule_of[v["pattern"]] = None
        self.scanner = (scanner_cls or RuleScanner)(rules, logger) if rules else None

    def validate_batch(self, items: Sequence[Tuple[str, str, Sequence[dict]]]) -> List[dict]:
        """items: (content, agentId, toolCallLog[{toolName, output}]) -> ResponseGateValidationResult per item"""
        if not self.config.get("enabled"):
            return [{"passed": True, "failedValidators": [], "reasons": []} for _ in items]
        hits = self.scanner.scan([it[0] for it in items]) if self.scanner else [[] for _ in items]
        out = []
        for (content, agent, log), h in zip(items, hits):
            hs = set(h); failed, reasons = [], []
            for rule in self.config.get("rules", []):
                ra = rule.get("agentId")
                if ra and (agent not in ra if isinstance(ra, list) else ra != agent):
                    continue
                for v in rule.get("validators", []):
                    if v["type"] == "requiredTools":
                        called = {e["toolName"] for e in log}
                        missing = [t for t in v["tools"] if t not in called]
                        if missing:
                            failed.append("requiredTools:" + ",".join(v["tools"]))
                            reasons.append(v.get("message") or "Response Gate: required tool(s) not called: " + ", ".join(missing))
                        continue
                    ri = self.rule_of[v["pattern"]]
                    if ri is None:
                        failed.append("%s:%s" % (v["type"], v["pattern"]))
                        reasons.append("Response Gate: invalid regex pattern /%s/ — blocked (fail-closed)" % v["pattern"])
                    elif v["type"] == "mustMatch" and ri not in hs:
                        failed.append("mustMatch:" + v["pattern"])
                        reasons.append(v.get("message") or "Response Gate: content does not match required pattern /%s/" % v["pattern"])
                    elif v["type"] == "mustNotMatch" and ri in hs:
                        failed.append("mustNotMatch:" + v["pattern"])
                        reasons.append(v.get("message") or "Response Gate: content matches forbidden pattern /%s/" % v["pattern"])
            res = {"passed": not failed, "failedValidators": failed, "reasons": reasons}
            if failed:
                tpl = self.config.get("fallbackMessage") or self.config.get("fallbackTemplate")
                if tpl:
                    res["fallbackMessage"] = tpl.replace("{reasons}", "; ".join(reasons)).replace("{validators}", ", ".join(failed)).replace("{agent}", agent)
            out.append(res)
        return out

    def validate(self, content: str, agent_id: str, tool_call_log: Sequence[dict]) -> dict:
        return self.validate_batch([(content, agent_id, tool_call_log)])[0]


# ------------------------------------------------------------------------------------- plugin entry

DEFAULT_REDACTION_CONFIG = {
    "enabled": True, "categories": ["credential", "pii", "financial"], "customPatterns": [], "failMode": "closed",
    "vaultExpirySeconds": 3600,
    "allowlist": {"piiAllowedChannels": [], "financialAllowedChannels": [], "exemptTools": [], "exemptAgents": []},
}


def _agent_id(ctx: Optional[dict]) -> str:
    """util.ts:140-172 (resolveAgentId), the part the hot path needs: explicit id, else `agent:<id>:...` session key."""
    ctx = ctx or {}
    if ctx.get("agentId"):
        return ctx["agentId"]
    parts = (ctx.get("sessionKey") or "").split(":")
    return parts[1] if len(parts) >= 2 and parts[0] == "agent" and parts[1] else "main"


class GovernancePlugin:
    """id / name / register(api) as in gov/index.ts:60-118 -- the part that touches the hot path."""

    id = "openclaw-governance"
    name = "OpenClaw Governance (H100 hot path)"

    def __init__(self):
        self.registry = self.vault = self.engine = self.credential_engine = self.policy = None
        self.config: dict = {}

    def register(self, api) -> None:
        cfg = dict(getattr(api, "pluginConfig", None) or {})
        self.config = cfg
        logger = getattr(api, "logger", None) or NullLogger()
        fail_mode = cfg.get("failMode", "open")
        N.init(int(cfg.get("gpu", {}).get("device", -1)))            # optional new key; default: current device
        red = {**DEFAULT_REDACTION_CONFIG, **cfg.get("redaction", {})}
        red["allowlist"] = {**DEFAULT_REDACTION_CONFIG["allowlist"], **red.get("allowlist", {})}
        self.policy = MessagePolicy([p for p in cfg.get("policies", []) if all("messageContains" in r for r in p.get("rules", []))], logger)
        self.evaluator = PolicyEvaluator([p for p in cfg.get("policies", []) if any("conditions" in r for r in p.get("rules", []))], logger)
        self.response_gate = ResponseGate(cfg["responseGate"], logger) if (cfg.get("responseGate") or {}).get("enabled") else None
        self.tool_call_log: Dict[str, List[dict]] = {}
        api.on("message_sending", self._governance_message_sending(fail_mode, logger), {"priority": 1000})
        api.on("before_tool_call", self._governance_before_tool_call(fail_mode, logger), {"priority": 1000})
        api.on("before_message_write", self._governance_before_message_write(fail_mode, logger), {"priority": 1000})
        api.on("after_tool_call", self._governance_after_tool_call(logger), {"priority": 900})
        if red["enabled"]:
            self.vault = RedactionVault(logger, red["vaultExpirySeconds"])
            self.registry = PatternRegistry(red["categories"], red["customPatterns"], logger)
            self.engine = RedactionEngine(self.registry, self.vault)
            self.credential_engine = RedactionEngine(PatternRegistry(["credential"], [], logger), self.vault)
            api.on("tool_result_persist", self._tool_result_persist(red, logger), {"priority": 800})
            api.on("after_tool_call", self._redaction_after_tool_call(red, logger), {"priority": 800})
            api.on("before_tool_call", self._redaction_before_tool_call(red, logger), {"priority": 950})
            api.on("message_sending", self._redaction_message_sending(red, logger), {"priority": 900})
            api.on("before_message_write", self._before_message_write(red, logger), {"priority": 900})
            logger.info("[redaction] Hooks registered (Layer 1 + Layer 2)")
        if hasattr(api, "registerGatewayMethod"):
            api.registerGatewayMethod("governance.status", lambda: self.status())

    def status(self) -> dict:
        s = N.stats()
        return {"gpu": {"messagesScanned": int(s.messages_scanned), "bytesScanned": int(s.bytes_scanned), "hits": int(s.hits),
                        "kernelLaunches": int(s.kernel_launches), "lastScanMs": float(s.last_scan_ms)}}

    @staticmethod
    def _eval_ctx(ctx, **extra) -> dict:
        ctx = ctx or {}
        return {"agentId": _agent_id(ctx), "channel": ctx.get("channelId") or ctx.get("channel"), "sessionKey": ctx.get("sessionKey"),
                "trust": ctx.get("trust") or {"session": {"tier": "standard"}, "agent": {"tier": "standard"}},
                "conversationContext": ctx.get("conversationContext") or [], "metadata": ctx.get("metadata") or {}, **extra}

    # gov/src/hooks.ts:173-243 (before_tool_call 1000): the tool / params conditions of the policy set; deny -> block, 2fa -> block
    # with the approval reason (the approval flow itself -- approval-2fa.ts -- is the reference's control plane)
    def _governance_before_tool_call(self, fail_mode, logger):
        def handler(event, ctx):
            try:
                ev = event or {}
                v = self.evaluator.evaluate(self._eval_ctx(ctx, toolName=ev.get("toolName"), toolParams=ev.get("params")))
                if v["action"] in ("deny", "2fa"):
                    return {"block": True, "blockReason": v["reason"]}
                return None
            except Exception as e:                      # noqa: BLE001
                logger.error("[governance] before_tool_call error: %s" % e)
                return {"block": True, "blockReason": "Governance engine error (fail-closed)"} if fail_mode == "closed" else None
        return handler

    # gov/src/hooks.ts:391-430 (after_tool_call 900): the per-session tool log the response gate reads
    def _governance_after_tool_call(self, logger):
        def handler(event, ctx):
            ev, c = event or {}, ctx or {}
            sid = c.get("sessionKey") or c.get("sessionId") or "agent:%s" % _agent_id(c)
            out = ev.get("result")
            self.tool_call_log.setdefault(sid, []).append({"toolName": ev.get("toolName"), "output": out if isinstance(out, str) else json.dumps(out, default=str)})
        return handler

    # gov/src/hooks.ts:297-389 (before_message_write 1000): response gate (mustMatch / mustNotMatch on the device, requiredTools from
    # the tool log); fallback message keeps the content's shape (:339-351)
    def _governance_before_message_write(self, fail_mode, logger):
        def handler(event, ctx):
            try:
                msg = (event or {}).get("message") or {}
                content = msg.get("content")
                if isinstance(content, list):
                    content = "\n".join(b.get("text", "") for b in content if isinstance(b, dict) and b.get("type") == "text")
                if not content or not isinstance(content, str) or self.response_gate is None:
                    return None
                c = ctx or {}
                agent = _agent_id(c)
                sid = c.get("sessionKey") or c.get("sessionId") or "agent:%s" % agent
                res = self.response_gate.validate(content, agent, self.tool_call_log.get(sid, []))
                if res["passed"]:
                    return None
                reason = "Response Gate blocked: " + "; ".join(res["reasons"])
                logger.warn("[governance] %s (agent=%s, failed=%s)" % (reason, agent, ",".join(res["failedValidators"])))
                if res.get("fallbackMessage"):
                    fb = [{"type": "text", "text": res["fallbackMessage"]}] if isinstance(msg.get("content"), list) else res["fallbackMessage"]
                    return {"message": {**msg, "content": fb}}
                return {"block": True, "blockReason": reason}
            except Exception as e:                      # noqa: BLE001
                logger.error("[governance] before_message_write error: %s" % e)
                return {"block": True, "blockReason": "Governance engine error (fail-closed)"} if fail_mode == "closed" else None
        return handler

    # gov/src/redaction/hooks.ts:208-258 (after_tool_call 800: fire-and-forget, mutates the event for audit logging)
    def _redaction_after_tool_call(self, red, logger):
        def handler(event, ctx):
            try:
                ev = event or {}
                if ev.get("result") is None:
                    return
                eng = self.credential_engine if ev.get("toolName") in red["allowlist"].get("exemptTools", []) else self.engine
                res = eng.scan(ev["result"])
                if res["redactionCount"] > 0:
                    ev["result"] = res["output"]
            except Exception as e:                      # noqa: BLE001
                logger.error("[redaction] L1 error: %s" % e)
                if red["failMode"] == "closed" and event is not None:
                    event["result"] = "[REDACTION ERROR: Tool output suppressed (fail-closed)]"
        return handler

    # gov/src/redaction/hooks.ts:260-305, 474-520 (before_tool_call 950: placeholders in tool params back to their originals)
    def _redaction_before_tool_call(self, red, logger):
        def handler(event, ctx):
            try:
                state = {"count": 0, "has": False, "unresolved": []}

                def res(v):
                    if isinstance(v, str):
                        if not RedactionVault.PLACEHOLDER_RE.search(v):
                            return v
                        state["has"] = True
                        r = self.vault.resolve_all(v)
                        state["count"] += r["resolved"] != v
                        state["unresolved"] += r["unresolvedHashes"]
                        return r["resolved"]
                    if isinstance(v, list):
                        return [res(x) for x in v]
                    if isinstance(v, dict):
                        return {k: res(x) for k, x in v.items()}
                    return v
                params = res((event or {}).get("params") or {})
                if not state["has"]:
                    return None
                if state["unresolved"]:
                    reason = "Unresolvable redacted value(s): %d placeholder(s) could not be resolved (expired or unknown)" % len(state["unresolved"])
                    logger.warn("[redaction] Vault resolution blocked: %s" % reason)
                    return {"block": True, "blockReason": reason}
                return {"params": params}
            except Exception as e:                      # noqa: BLE001
                logger.error("[redaction] Vault resolution error: %s" % e)
                return {"block": True, "blockReason": "Redaction vault error (fail-closed): %s" % e} if red["failMode"] == "closed" else None
        return handler

    # gov/src/hooks.ts:245-290
    def _governance_message_sending(self, fail_mode, logger):
        def handler(event, ctx):
            try:
                content = (event or {}).get("content")
                if not content:
                    return None
                verdict = self.policy.evaluate(content)
                if verdict["action"] == "deny":
                    return {"cancel": True}
                if self.evaluator.policies and self.evaluator.evaluate(self._eval_ctx(ctx, messageContent=content))["action"] in ("deny", "2fa"):
                    return {"cancel": True}
                return None
            except Exception as e:                      # noqa: BLE001 -- mirrors the reference's catch-all
                logger.error("[governance] message_sending error: %s" % e)
                return {"cancel": True} if fail_mode == "closed" else None
        return handler

    # gov/src/redaction/hooks.ts:307-403
    def _redaction_message_sending(self, red, logger):
        def handler(event, ctx):
            try:
                if not event or not event.get("content"):
                    return None
                scan = self.engine.scan_string(event["content"])
                if scan["redactionCount"] == 0:
                    return None
                context = {"channel": (ctx or {}).get("channelId"), "agentId": _agent_id(ctx)}
                if all(evaluate_allowlist(c, context, red["allowlist"])["allowed"] for c in scan["categories"]):
                    return None
                applied = scan["redactionCount"]
                if event.get("metadata"):
                    meta = self.engine.scan(event["metadata"])
                    if meta["redactionCount"] > 0:
                        event["metadata"].update(meta["output"])
                        applied += meta["redactionCount"]
                return {"content": scan["output"]} if applied > 0 else None
            except Exception as e:                      # noqa: BLE001
                logger.error("[redaction] L2 error: %s" % e)
                return {"cancel": True} if red["failMode"] == "closed" else None
        return handler

    # gov/src/redaction/hooks.ts:405-456 (synchronous hook)
    def _before_message_write(self, red, logger):
        def handler(event, ctx):
            try:
                if not event or not event.get("content"):
                    return None
                if _agent_id(ctx) in red["allowlist"].get("exemptAgents", []):
                    return None
                scan = self.engine.scan_string(event["content"])
                if scan["redactionCount"] == 0 or not ({"credential", "financial"} & scan["categories"]):
                    return None
                return {"content": scan["output"]}
            except Exception as e:                      # noqa: BLE001
                logger.error("[redaction] L2-sync error: %s" % e)
                return {"block": True, "blockReason": "Redaction error (fail-closed)"} if red["failMode"] == "closed" else None
        return handler

    # gov/src/redaction/hooks.ts:158-206 (synchronous hook)
    def _tool_result_persist(self, red, logger):
        def handler(event, ctx):
            try:
                message = (event or {}).get("message")
                if message is None:
                    return None
                tool = event.get("toolName") or "unknown"
                eng = self.credential_engine if tool in red["allowlist"].get("exemptTools", []) else self.engine
                scan_input = message if isinstance(message, str) else json.dumps(message, separators=(",", ":"), ensure_ascii=False)
                result = eng.scan(scan_input)
                return {"message": result["output"]} if result["redactionCount"] > 0 else None
            except Exception as e:                      # noqa: BLE001
                logger.error("[redaction] L1 persist error: %s" % e)
                return {"message": "[REDACTION ERROR: Tool output suppressed (fail-closed)]"} if red["failMode"] == "closed" else None
        return handler


plugin = GovernancePlugin()
