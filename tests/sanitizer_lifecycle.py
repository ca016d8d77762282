"""Allocation lifecycle workload for a compute-sanitizer run (not collected by pytest; numpy only, no device buffers of its
own): every host-buffer call family, once on a batch whose candidate queues overflow so the scratch regrows; repeated
set_policy / set_views / set_policy_program; keep, no-keep, tree and restored Merkle logs grown past their first capacity;
then every handle destroyed, cg_shutdown, cg_init, one more scan and cg_shutdown.  Usage:
  compute-sanitizer --tool memcheck --leak-check full --error-exitcode 3 python tests/sanitizer_lifecycle.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vainplex_openclaw_b200 import _native as N  # noqa: E402

RULES = [(r"secret-[0-9]{4}", 0, 0), (r"tok_[a-z]{6}", 1, 1), (r"[0-9]{3}-[0-9]{2}-[0-9]{4}", 0, 2), (r"password\s*=\s*\S+", 1, 3)]
HITS = [b"secret-1234", b"TOK_abcdef", b"123-45-6789", b"password = hunter2"]
rng = np.random.default_rng(5)


def batch(n, hit_every):
    msgs = []
    for i in range(n):
        words = [bytes(rng.integers(97, 123, int(rng.integers(1, 9)), dtype=np.uint8)) for _ in range(int(rng.integers(2, 30)))]
        if hit_every and i % hit_every == 0:
            words.insert(int(rng.integers(0, len(words) + 1)), HITS[i % len(HITS)])
        msgs.append(b" ".join(words))
    return N.pack(msgs)


def leaves(n):
    return [bytes(rng.integers(0, 256, int(rng.integers(0, 100)), dtype=np.uint8)) for _ in range(n)]


N.init(0)
rs = N.Ruleset(RULES, strict=True)
small, small_off = batch(300, 7)
w0, h0 = rs.scan_batch(small, small_off)
# every message hits: more slots than a batch of this size starts with, so the step overflows, grows and runs again
big, big_off = batch(20000, 1)
w1, h1 = rs.scan_batch(big, big_off)
assert int((w1 != 0).sum()) == 20000 and len(h1) >= 20000
wide, wide_off = batch(70000, 50)                                   # the chunked words-only path
w2, _ = rs.scan_batch(wide, wide_off, want_hits=False)
spans = rs.find_matches_batch(small, small_off)
red = rs.redact_batch(small, small_off)
rs.scan_one(HITS[0] + b" and more")
rs.find_matches_one(HITS[1]); rs.redact_one(HITS[2])
rs.find_matches_few(small, small_off[:9]); rs.redact_few(small, small_off[:9])
for k in range(3):
    rs.set_policy(np.arange(len(RULES), dtype=np.uint32), np.full(len(RULES), k % 3, dtype=np.uint8))
    rs.verdict_batch(small, small_off)
    rs.set_views([[0, 1], [2, 3], list(range(len(RULES)))][: k + 1])
    ids = np.arange(300, dtype=np.uint8) % (k + 1)
    rs.scan_batch(small, small_off, views=ids); rs.find_matches_batch(small, small_off, views=ids)
    rs.redact_batch(small, small_off, views=ids); rs.verdict_batch(small, small_off, views=ids)
    # one policy, k + 1 rules: deny on a hit of rule 0 in a text of role 0, else CONST 0
    prog = [1, 0xffffffff, k + 1] + [2, 1, N.POL_HIT | (0 << 3)] + [0, 1, N.POL_CONST] * k
    rs.set_policy_program(np.array(prog, dtype=np.uint32), 0)
    roles = np.zeros(300, dtype=np.uint8)
    rs.eval_batch(small, small_off, roles, np.array([0, 100, 300], dtype=np.uint32), np.zeros(0, dtype=np.uint32))
    rs.eval_one(small, small_off[:5], roles[:4], np.zeros(0, dtype=np.uint32))

sha = N.sha256_batch(small, small_off.astype(np.uint64))
N.merkle_root(small, small_off.astype(np.uint64)); N.merkle_root_fixed(small, 16, len(small) // 16); N.merkle_fold(sha)
logs = [N.MerkleLog(True), N.MerkleLog(False), N.MerkleLog.tree()]
appends = [leaves(m) for m in (3, 70, 900, 5000)]                  # each past the digest room the one before left
for lg in logs:
    for a in appends:
        lg.append(a)
    lg.append_jsonl(b"\n".join(b'{"e": %d}' % i for i in range(3000)) + b"\n")
    lg.root()
assert logs[0].root() == logs[1].root() == logs[2].root()
assert N.merkle_verify_proof(appends[0][1], 1, logs[0].size(), logs[0].proof(1), logs[0].root())
logs[0].consistency(77)
paths, lens = logs[2].proofs(np.arange(0, 8000, 97), 8000); logs[2].consistency_between(100, 8000)
restored = N.MerkleLog.restore(logs[1].size(), logs[1].frontier())
for m in (2, 600, 4000):
    restored.append(leaves(m))
assert restored.root() != logs[1].root()
for lg in logs + [restored]:
    lg.close()
rs.close()

N.load().cg_shutdown()
N.init(0)
rs = N.Ruleset(RULES, strict=True)
w3, _ = rs.scan_batch(small, small_off)
assert np.array_equal(w3, w0)
rs.close()
N.load().cg_shutdown()
print("ok", int((w1 != 0).sum()), len(spans), len(red[2]))
