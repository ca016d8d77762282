"""CPU tier for policy programs (cg_ruleset_set_policy_program / cg_policy_eval_batch[_device]): PolicyEvaluator's program
compiler, run through a Python restatement of the kernel's semantics with the oracle's hit sets, gives what evaluate_batch
gives -- on the policy-slice cases, the reference's built-ins and random policy sets; the launch counts restated; the
exports are in the header, the Python binding, the N-API shim and the TypeScript declarations, and the shim compiles."""
import os
import re
import subprocess

import numpy as np
import pytest

import policy_program as PP
from vainplex_openclaw_b200 import _native as N
from vainplex_openclaw_b200 import plugin as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["cg_ruleset_set_policy_program", "cg_policy_eval_batch", "cg_policy_eval_batch_device"]


@pytest.fixture(scope="module")
def oracle_scanner(oracle):
    class OracleScanner:
        def __init__(self, rules, logger=None):
            self.rules = [([pats] if isinstance(pats, str) else list(pats)) for pats in rules]
            self.cache = {}

        def scan(self, texts):
            return [[ri for ri, pats in enumerate(self.rules) if oracle.matches_any(pats, [t], self.cache)] for t in texts]
    return OracleScanner


def check(policies, contexts, scanner, other=None):
    pe = P.PolicyEvaluator(policies, scanner_cls=scanner, other_condition=other)
    assert PP.restated_verdicts(pe, contexts) == pe.evaluate_batch(contexts)
    return pe


def test_slice_cases(oracle_scanner):
    for policies, contexts in PP.slice_cases():
        check(policies, contexts, oracle_scanner)


def test_builtins_on_tool_calls(oracle_scanner):
    ctxs = PP.tool_contexts(np.random.default_rng(5), 400)
    pe = check(PP.builtin_policies(), ctxs, oracle_scanner, PP.other_condition)
    acts = [r["action"] for r in pe.evaluate_batch(ctxs)]
    assert acts.count("deny") > 40 and acts.count("allow") > 40


def test_random_policy_sets(oracle_scanner):
    rng = np.random.default_rng(11)
    decided = 0
    for _ in range(2000):
        pols = PP.random_policies(rng)
        ctxs = PP.random_contexts(rng, 6)
        pe = check(pols, ctxs, oracle_scanner, PP.other_condition)
        decided += sum(r["action"] != "allow" for r in pe.evaluate_batch(ctxs))
    assert decided > 1000


def test_empty_reason_takes_the_next_non_empty_one(oracle_scanner):
    """aggregateMatches (policy-evaluator.ts:51-60) keeps the first NON-EMPTY deny reason: a first deny without one does not
    hide a later deny's.  (evaluate_batch reports the first deny's reason or the default.)"""
    tool = [{"type": "tool", "name": "exec"}]
    pols = [{"id": "a", "priority": 2, "rules": [{"id": "r", "conditions": tool, "effect": {"action": "deny"}}]},
            {"id": "b", "priority": 1, "rules": [{"id": "r", "conditions": tool, "effect": {"action": "deny", "reason": "second"}}]},
            {"id": "c", "rules": [{"id": "r", "conditions": tool, "effect": {"action": "2fa", "reason": ""}}]}]
    pe = P.PolicyEvaluator(pols, scanner_cls=oracle_scanner)
    r = PP.restated_verdicts(pe, [PP.make_ctx(), PP.make_ctx(toolName="read")])
    assert (r[0]["action"], r[0]["reason"], [m["policyId"] for m in r[0]["matches"]]) == ("deny", "second", ["a", "b", "c"])
    assert (r[1]["action"], r[1]["reason"], r[1]["matches"]) == ("allow", "No matching policies", [])
    pe = P.PolicyEvaluator(pols[:1] + pols[2:], scanner_cls=oracle_scanner)
    assert PP.restated_verdicts(pe, [PP.make_ctx()])[0]["reason"] == "Denied by governance policy"
    pe = P.PolicyEvaluator(pols[2:], scanner_cls=oracle_scanner)
    assert PP.restated_verdicts(pe, [PP.make_ctx()])[0]["reason"] == "Requires 2FA approval"


def test_program_layout(oracle_scanner):
    """the words of a small program, written out"""
    pols = [{"id": "s", "scope": {"channels": ["matrix"]}, "rules": [
        {"id": "r0", "conditions": [], "effect": {"action": "audit"}},
        {"id": "r1", "minTrust": "trusted", "conditions": [{"type": "any", "conditions": []},
                                                           {"type": "not", "condition": {"type": "context", "messageContains": ["x", "y"]}}],
         "effect": {"action": "deny", "reason": "no"}}]},
        {"id": "t", "priority": -1, "rules": [{"id": "q", "conditions": [{"type": "tool", "params": {"command": {"matches": "z+"}}}], "effect": {"action": "2fa"}}]}]
    pe = P.PolicyEvaluator(pols, scanner_cls=oracle_scanner)
    C, A, H, AND, OR, NOT = N.POL_CONST, N.POL_ATOM, N.POL_HIT, N.POL_AND, N.POL_OR, N.POL_NOT
    want = [2,
            0, 2, 1, 1, C | 1 << 3,
            3 | 4, 8, A | 1 << 3, C, AND, H | 0 << 3, H | 1 << 3, OR, NOT, AND,
            0xffffffff, 1, 2, 3, A | 2 << 3, H | 2 << 3 | 2 << 24, AND]
    assert pe.program.tolist() == want and pe.param_role == {"command": 2} and len(pe.atoms) == 3


def test_launch_counts_restated():
    """the step, then one evaluation kernel (verdicts only) or count + exclusive scan + emit; none of it depends on hits"""
    src = open(os.path.join(ROOT, "vainplex_openclaw_b200", "csrc", "policy_eval.cu")).read()
    assert "return 1 + launch_exclusive_scan(w.out_len, w.out_off, b.n_ctx + 1" in src
    assert src.count("<<<") == 3 and src.count("<<<pe_grid(") + src.count("<<<grid,") == 3
    assert "uint32_t pe_grid(uint32_t n_ctx, int sm_count)" in src


def test_exports_and_bindings():
    hdr = open(os.path.join(ROOT, "include", "openclaw_gov.h")).read()
    for fn in NEW:
        assert re.search(r"CG_API int %s\(" % fn, hdr), fn
        assert fn in N.EXPORTS, fn
    assert "typedef struct cg_policy_match" in hdr
    L = N.load()
    assert all(hasattr(L, fn) for fn in NEW)
    assert all(hasattr(N.Ruleset, m) for m in ("set_policy_program", "eval_batch", "eval_batch_device"))
    src = open(os.path.join(ROOT, "napi", "openclaw_gov_napi.c")).read()
    ts = open(os.path.join(ROOT, "napi", "gpu-backend.ts")).read()
    for fn in NEW[:2]:
        assert fn + "(" in src, fn
    for js in ("setPolicyProgram", "policyEvalBatch"):
        assert 'FN("%s"' % js in src and js + "(" in ts, js
    assert "cg_policy_eval_batch_device" not in src              # JavaScript holds no device pointers
    assert "compilePolicyProgram" in ts


def test_napi_shim_compiles_against_the_stub(tmp_path):
    out = tmp_path / "shim.o"
    r = subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-c", "-I" + os.path.join(ROOT, "napi", "stub"),
                        "-I" + os.path.join(ROOT, "include"), "-o", str(out), os.path.join(ROOT, "napi", "openclaw_gov_napi.c")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
