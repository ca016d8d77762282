"""Shared by the policy-program tests (CPU and GPU tier): a Python restatement of policy_eval_kernel's semantics (program,
hit sets, atoms -> verdict words and match list), the cases of test_policy_slice, the reference's built-in policies with
tool-call contexts, and random policy sets with contexts."""
import numpy as np

from test_policy_slice import make_ctx, tool_rule
from vainplex_openclaw_b200 import _native as N

NONE = 0xffffffff


def parse(program):
    """-> [(scope atom, [(action, has_reason, ops)])] per policy"""
    p = [int(x) for x in program]
    at, pols = 1, []
    for _ in range(p[0]):
        scope, nr = p[at], p[at + 1]
        at += 2
        rules = []
        for _ in range(nr):
            head, n = p[at], p[at + 1]
            rules.append((head & 3, head >> 2, p[at + 2:at + 2 + n]))
            at += 2 + n
        pols.append((scope, rules))
    assert at == len(p)
    return pols


def restate(program, text_hits, roles, ctx_off, atoms):
    """what cg_policy_eval_batch returns, restated: text_hits[i] = the rules text i hit.
    -> (verdict words uint32[n_ctx], POLICY_MATCH_DTYPE array)"""
    pols = parse(program)
    words, matches = [], []
    for c in range(len(ctx_off) - 1):
        texts = range(int(ctx_off[c]), int(ctx_off[c + 1]))

        def bit(a):
            return (int(atoms[c, a >> 5]) >> (a & 31)) & 1

        def run(ops):
            st = []
            for o in ops:
                code = o & 7
                if code == N.POL_CONST:
                    st.append(o >> 3)
                elif code == N.POL_ATOM:
                    st.append(bit(o >> 3))
                elif code == N.POL_HIT:
                    r, q = (o >> 3) & 0x1fffff, o >> 24
                    st.append(int(any(roles[i] == q and r in text_hits[i] for i in texts)))
                elif code == N.POL_AND:
                    b = st.pop(); st[-1] &= b
                elif code == N.POL_OR:
                    b = st.pop(); st[-1] |= b
                else:
                    st[-1] ^= 1
            assert len(st) == 1
            return st[0]
        j, found = 0, []
        for scope, rules in pols:
            first = None
            for act, reason, ops in rules:
                if first is None and (scope == NONE or bit(scope)) and run(ops):
                    first = (j, act, reason)
                j += 1
            if first:
                found.append(first)
        acts = [a for _, a, _ in found]
        outcome = 4 if 3 in acts else 3 if 2 in acts else 2 if 1 in acts else 1 if found else 0
        want = {4: 3, 3: 2}.get(outcome)
        decide = next((jj for jj, a, r in found if a == want and r), 0xfffff)
        words.append(outcome | min(len(found), 511) << 3 | decide << 12)
        matches += [(c, jj) for jj, _, _ in found]
    return np.array(words, dtype=np.uint32), np.array(matches, dtype=N.POLICY_MATCH_DTYPE)


def restated_verdicts(pe, contexts):
    """PolicyEvaluator.verdict_batch's result through the restatement, with pe's own scanner for the hit sets"""
    texts, roles, ctx_off, atoms = pe.program_inputs(contexts)
    hits = pe.scanner.scan(texts) if (pe.scanner and texts) else [[] for _ in texts]
    words, matches = restate(pe.program, [set(h) for h in hits], roles, ctx_off, atoms)
    return pe.decode_verdicts(words, matches)


# ------------------------------------------------------------------------------------------ cases

def slice_cases():
    """(policies, contexts) of test_policy_slice's policy evaluator and condition cases"""
    deny = {"action": "deny", "reason": "Denied"}
    allow_p = {"id": "allow-p", "scope": {}, "rules": [tool_rule({"action": "allow"})]}
    deny_p = {"id": "deny-p", "scope": {}, "rules": [tool_rule(deny)]}
    twofa = {"id": "t", "scope": {}, "rules": [tool_rule({"action": "2fa"})]}
    audit = {"id": "a", "scope": {"agents": ["forge"], "channels": ["matrix"]}, "rules": [tool_rule({"action": "audit"})]}
    sets = [[], [{"id": "p1", "scope": {}, "rules": [tool_rule({"action": "deny", "reason": "No exec allowed"})]}], [allow_p, deny_p],
            [{"id": "low", "scope": {}, "priority": 1, "rules": [tool_rule({"action": "allow"})]},
             {"id": "high", "scope": {}, "priority": 10, "rules": [tool_rule({"action": "deny", "reason": "High priority deny"})]}],
            [{"id": "p1", "scope": {"excludeAgents": ["forge"]}, "rules": [tool_rule(deny)]}],
            [{"id": "p1", "scope": {"channels": ["telegram"]}, "rules": [tool_rule(deny)]}],
            [{"id": "p1", "scope": {}, "rules": [tool_rule({"action": "allow"}, minTrust="trusted")]}],
            [{"id": "p1", "scope": {}, "rules": [tool_rule({"action": "deny", "reason": "Too new"}, maxTrust="restricted")]}],
            [{"id": "p1", "scope": {}, "rules": [tool_rule({"action": "audit", "level": "verbose"})]}],
            [{"id": "p1", "scope": {}, "rules": [{"id": "r1", "conditions": [{"type": "tool", "name": "exec"}, {"type": "agent", "id": "cerberus"}], "effect": deny}]}],
            [{"id": "p1", "scope": {}, "rules": [tool_rule({"action": "allow"}), tool_rule({"action": "deny", "reason": "Should not reach"}, rid="r2")]}],
            [{"id": "p1", "scope": {}, "controls": ["A.8.3"], "rules": [tool_rule({"action": "allow"})]}],
            [twofa, audit], [twofa, audit, deny_p]]
    out = [(s, [make_ctx()]) for s in sets]
    conds = [
        ({"type": "tool", "name": "exec", "params": {"command": {"matches": "git push.*(main|master)"}}},
         [dict(toolParams={"command": "git push origin main"}), dict(toolParams={"command": "git push origin dev"})]),
        ({"type": "tool", "params": {"command": {"matches": "docker.*"}}}, [{}]),
        ({"type": "tool", "params": {"command": {"matches": "[invalid"}}}, [{}]),
        ({"type": "tool", "params": {"count": {"matches": "\\d+"}}}, [dict(toolParams={"count": 42})]),
        ({"type": "tool", "params": {"elevated": {"equals": True}}}, [dict(toolParams={"elevated": True}), dict(toolParams={"elevated": False})]),
        ({"type": "tool", "params": {"command": {"startsWith": "sudo"}}}, [dict(toolParams={"command": "sudo rm -rf"})]),
        ({"type": "tool", "params": {"host": {"in": ["sandbox", "gateway"]}}}, [dict(toolParams={"host": "sandbox"}), dict(toolParams={"host": "node"})]),
        ({"type": "tool"}, [{}]),
        ({"type": "tool", "name": "exec"}, [dict(toolName=None)]),
        ({"type": "tool", "params": {"command": {"contains": "test"}}}, [dict(toolParams=None)]),
        ({"type": "tool", "name": "ex*"}, [{}]), ({"type": "tool", "name": "e?"}, [{}]),
        ({"type": "context", "conversationContains": "JIRA-\\d+"}, [{}]),
        ({"type": "context", "conversationContains": "TICKET-\\d+"}, [{}]),
        ({"type": "context", "conversationContains": "JIRA"}, [dict(conversationContext=[])]),
        ({"type": "context", "conversationContains": ["NOPE", "JIRA-\\d+"]}, [{}]),
        ({"type": "context", "messageContains": "Hello"}, [{}, dict(messageContent="")]),
        ({"type": "context", "messageContains": "a(b"}, [dict(messageContent="xx a(b yy")]),
        ({"type": "any", "conditions": [{"type": "context", "messageContains": "zzz"}, {"type": "context", "conversationContains": "JIRA"}]}, [{}]),
        ({"type": "not", "condition": {"type": "context", "messageContains": "zzz"}}, [{}]),
        ({"type": "not", "condition": {"type": "context", "messageContains": "Hel+o"}}, [{}]),
    ]
    for cond, overs in conds:
        pol = [{"id": "p", "scope": {}, "rules": [{"id": "r", "conditions": [cond], "effect": {"action": "deny", "reason": "x"}}]}]
        out.append((pol, [make_ctx(**o) for o in overs]))
    pol = [{"id": "p", "scope": {}, "rules": [{"id": "r", "conditions": [{"type": "context", "messageContains": "secret-\\d{3}"}], "effect": {"action": "deny", "reason": "leak"}}]}]
    out.append((pol, [make_ctx(messageContent="x secret-%03d y" % i if i % 3 == 0 else "nothing %d" % i) for i in range(60)]))
    return out


def builtin_policies():
    """src/builtin-policies.ts: credential guard, production safeguard, rate limiter (night mode needs the clock: its `time`
    condition is an atom like frequency)"""
    prod = [{"type": "tool", "name": "exec", "params": {"command": {"matches": "(docker push|docker-compose.*prod|systemctl.*(restart|stop|enable|disable))"}}},
            {"type": "tool", "name": "exec", "params": {"command": {"matches": "git push.*(origin|upstream).*(main|master|prod)"}}},
            {"type": "tool", "name": "gateway", "params": {"action": {"matches": "(restart|config\\.apply|update\\.run)"}}}]
    trusted = {"type": "agent", "trustTier": ["trusted", "elevated"]}
    cred_any = [{"type": "tool", "params": {"file_path": {"matches": "\\.(env|pem|key)$"}}},
                {"type": "tool", "params": {"path": {"matches": "\\.(env|pem|key)$"}}},
                {"type": "tool", "params": {"command": {"matches": "(cat|less|head|tail|cp|mv|grep|find|scp|rsync|docker\\s+cp).*\\.(env|pem|key)"}}},
                {"type": "tool", "params": {"command": {"matches": "(cp|mv|scp|rsync|docker\\s+cp).*(credentials|secrets|\\.env|\\.pem|\\.key)"}}},
                {"type": "tool", "params": {"command": {"matches": "(grep|find).*(password|token|secret|credential)"}}},
                {"type": "tool", "params": {"file_path": {"contains": "credentials"}}}, {"type": "tool", "params": {"path": {"contains": "credentials"}}},
                {"type": "tool", "params": {"file_path": {"contains": "secrets"}}}, {"type": "tool", "params": {"path": {"contains": "secrets"}}}]
    night = ["read", "memory_search", "memory_get", "web_search"]
    return [
        {"id": "builtin-night-mode", "scope": {"hooks": ["before_tool_call", "message_sending"]}, "priority": 100, "controls": ["A.7.1", "A.6.2"],
         "rules": [{"id": "allow-critical-at-night", "conditions": [{"type": "time", "after": "23:00", "before": "08:00"}, {"type": "tool", "name": night}],
                    "effect": {"action": "allow"}},
                   {"id": "deny-non-critical-at-night", "conditions": [{"type": "time", "after": "23:00", "before": "08:00"},
                                                                       {"type": "not", "condition": {"type": "tool", "name": night}}],
                    "effect": {"action": "deny", "reason": "Night mode active (23:00-08:00). Only critical operations allowed."}}]},
        {"id": "builtin-credential-guard", "scope": {"hooks": ["before_tool_call"]}, "priority": 200, "controls": ["A.8.11", "A.8.4", "A.5.33"],
         "rules": [{"id": "block-credential-read", "conditions": [{"type": "tool", "name": ["read", "exec", "write", "edit"]}, {"type": "any", "conditions": cred_any}],
                    "effect": {"action": "deny", "reason": "Credential Guard: Access to credential files is restricted"}}]},
        {"id": "builtin-production-safeguard", "scope": {"hooks": ["before_tool_call"], "excludeAgents": ["unresolved"]}, "priority": 150,
         "controls": ["A.8.31", "A.8.32", "A.8.9"],
         "rules": [{"id": "allow-production-ops-trusted", "conditions": [trusted, {"type": "any", "conditions": prod}], "effect": {"action": "allow"}},
                   {"id": "block-production-ops", "conditions": [{"type": "not", "condition": trusted}, {"type": "any", "conditions": prod}],
                    "effect": {"action": "deny", "reason": "Production Safeguard: This operation requires explicit approval (trusted+ agents only)"}}]},
        {"id": "builtin-rate-limiter", "scope": {"hooks": ["before_tool_call"]}, "priority": 50, "controls": ["A.8.6"],
         "rules": [{"id": "rate-limit-trusted", "conditions": [trusted, {"type": "frequency", "maxCount": 30, "windowSeconds": 60, "scope": "agent"}],
                    "effect": {"action": "deny", "reason": "Rate limit exceeded (30/min for trusted agents)"}},
                   {"id": "rate-limit-default", "conditions": [{"type": "not", "condition": trusted}, {"type": "frequency", "maxCount": 15, "windowSeconds": 60, "scope": "agent"}],
                    "effect": {"action": "deny", "reason": "Rate limit exceeded (15/min)"}}]},
    ]


def other_condition(cond, ctx):
    """a deterministic stand-in for time / risk / frequency: a function of the condition and the context"""
    return (len(cond.get("type", "")) + len(ctx.get("agentId") or "") + len(ctx.get("toolName") or "") + int(cond.get("maxCount", 1))) % 3 == 0


TOOLS = ["read", "exec", "write", "edit", "gateway", "web_search", "memory_get", "browser"]
COMMANDS = ["cat .env", "less id_rsa.pem", "docker push app:prod", "git push origin main", "git push upstream dev", "ls -la",
            "grep -r password .", "cp credentials.json /tmp", "systemctl restart nginx", "echo hello", "rsync secrets/ host:", ""]
PATHS = ["/etc/app/.env", "/home/u/notes.txt", "/srv/credentials/db.key", "secrets.yaml", "README.md"]


def tool_contexts(rng, n):
    """tool-call contexts (before_tool_call) for the built-ins"""
    out = []
    for _ in range(n):
        tool = TOOLS[int(rng.integers(len(TOOLS)))]
        params = {}
        if rng.random() < 0.7:
            params["command"] = COMMANDS[int(rng.integers(len(COMMANDS)))]
        if rng.random() < 0.4:
            params["file_path" if rng.random() < 0.5 else "path"] = PATHS[int(rng.integers(len(PATHS)))]
        if tool == "gateway" and rng.random() < 0.7:
            params["action"] = ["restart", "config.apply", "status", "update.run"][int(rng.integers(4))]
        if rng.random() < 0.1:
            params["count"] = int(rng.integers(100))
        tiers = ["untrusted", "restricted", "standard", "trusted", "elevated"]
        out.append({"agentId": ["main", "forge", "unresolved", "atlas"][int(rng.integers(4))], "channel": ["matrix", "slack", None][int(rng.integers(3))],
                    "sessionKey": "agent:main:%d" % int(rng.integers(5)), "toolName": tool, "toolParams": params if params or rng.random() < 0.5 else None,
                    "trust": {"agent": {"tier": tiers[int(rng.integers(5))]}, "session": {"tier": tiers[int(rng.integers(5))]}},
                    "conversationContext": [], "messageContent": ""})
    return out


# ------------------------------------------------------------------------------------------ random policy sets

PATTERNS = ["secret-\\d{3}", "JIRA-\\d+", "docker", "rm -rf", "passw(or)?d", "a(b", "\\.(env|pem|key)$", "git push.*main", "^sudo ", "token[:=]\\S+"]
SAMPLES = ["secret-123", "JIRA-77", "docker", "rm -rf /", "password", "x a(b y", "file.env", "git push origin main", "sudo ls", "token=abc"]
WORDS = ["hello", "world", "please", "deploy", "the", "service", "now", "ok"]
KEYS = ["command", "path", "host", "count", "elevated"]
AGENTS, CHANNELS, TIERS = ["main", "forge", "atlas", "cerberus"], ["matrix", "slack", "web"], ["untrusted", "restricted", "standard", "trusted", "elevated"]


def _pick(rng, xs):
    return xs[int(rng.integers(len(xs)))]


def _some(rng, xs, k=3):
    return [_pick(rng, xs) for _ in range(int(rng.integers(1, k + 1)))]


def random_condition(rng, depth, patterns=PATTERNS):
    u = rng.random() if depth < 4 else rng.random() * 0.8
    if u < 0.28:
        c = {"type": "context"}
        for key in ("messageContains", "conversationContains", "channel", "hasMetadata", "sessionKey"):
            if rng.random() < 0.35:
                c[key] = {"messageContains": lambda: _some(rng, patterns) if rng.random() < 0.5 else _pick(rng, patterns),
                          "conversationContains": lambda: _some(rng, patterns) if rng.random() < 0.5 else _pick(rng, patterns),
                          "channel": lambda: _some(rng, CHANNELS), "hasMetadata": lambda: _some(rng, ["a", "b"], 2),
                          "sessionKey": lambda: _pick(rng, ["agent:*", "agent:main:?", "x*"])}[key]()
        return c
    if u < 0.56:
        c = {"type": "tool"}
        if rng.random() < 0.6:
            c["name"] = _pick(rng, ["exec", "read", "ex*", "w?ite", ["exec", "gateway"]])
        if rng.random() < 0.6:
            params = {}
            for key in _some(rng, KEYS, 2):
                params[key] = _pick(rng, [{"matches": _pick(rng, patterns + ["[bad"])}, {"equals": _pick(rng, ["ls", 3, True])},
                                          {"contains": "o"}, {"startsWith": "sudo"}, {"in": ["ls", "sandbox", 3]}])
            c["params"] = params
        return c
    if u < 0.72:
        c = {"type": "agent"}
        if rng.random() < 0.6:
            c["id"] = _pick(rng, ["main", "f*", ["atlas", "cerberus"]])
        if rng.random() < 0.6:
            c["trustTier"] = _some(rng, TIERS, 2)
        return c
    if u < 0.8:
        return {"type": _pick(rng, ["time", "risk", "frequency"]), "maxCount": int(rng.integers(1, 5))}
    if u < 0.9:
        return {"type": "any", "conditions": [random_condition(rng, depth + 1, patterns) for _ in range(int(rng.integers(0, 4)))]}
    return {"type": "not", "condition": random_condition(rng, depth + 1, patterns)}


def random_policies(rng, patterns=PATTERNS, max_policies=6):
    pols = []
    for i in range(int(rng.integers(1, max_policies + 1))):
        scope = {}
        if rng.random() < 0.3:
            scope["excludeAgents"] = _some(rng, AGENTS, 2)
        if rng.random() < 0.3:
            scope["channels"] = _some(rng, CHANNELS, 2)
        if rng.random() < 0.2:
            scope["agents"] = ["main"]
        rules = []
        for k in range(int(rng.integers(0, 4))):
            action = _pick(rng, ["allow", "audit", "2fa", "deny"])
            eff = {"action": action}
            if action in ("deny", "2fa") or rng.random() < 0.3:
                eff["reason"] = "%s by p%d r%d" % (action, i, k)
            r = {"id": "r%d" % k, "conditions": [random_condition(rng, 1, patterns) for _ in range(int(rng.integers(0, 3)))], "effect": eff}
            if rng.random() < 0.2:
                r["minTrust"] = _pick(rng, TIERS)
            if rng.random() < 0.2:
                r["maxTrust"] = _pick(rng, TIERS)
            rules.append(r)
        pols.append({"id": "p%d" % i, "scope": scope, "priority": int(rng.integers(0, 3)), "rules": rules, "controls": ["c%d" % i]})
    return pols


def _text(rng, samples=SAMPLES):
    w = [_pick(rng, WORDS) for _ in range(int(rng.integers(0, 5)))]
    if rng.random() < 0.5:
        w.insert(int(rng.integers(len(w) + 1)), _pick(rng, samples))
    return " ".join(w)


def random_contexts(rng, n, samples=SAMPLES):
    out = []
    for _ in range(n):
        params = {}
        for key in KEYS:
            if rng.random() < 0.35:
                params[key] = _pick(rng, [_text(rng, samples), "ls", "sudo rm", 3, True, "sandbox"])
        out.append({"agentId": _pick(rng, AGENTS), "channel": _pick(rng, CHANNELS + [None]), "sessionKey": _pick(rng, ["agent:main:x", "agent:forge:y", None]),
                    "trust": {"agent": {"tier": _pick(rng, TIERS)}, "session": {"tier": _pick(rng, TIERS)}},
                    "metadata": {k: 1 for k in ["a", "b"] if rng.random() < 0.5},
                    "toolName": _pick(rng, ["exec", "read", "write", "gateway", None]), "toolParams": params if params or rng.random() < 0.5 else None,
                    "messageContent": _text(rng, samples) if rng.random() < 0.8 else "",
                    "conversationContext": [_text(rng, samples) for _ in range(int(rng.integers(0, 4)))]})
    return out
