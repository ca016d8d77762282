"""GPU tier: confirm_kernel collects a warp's confirmed factor occurrences in a buffer of 32 and appends them to the queue
behind one atomic; resolve_kernel takes a slot per message and a VM event per candidate from them.  Each case is compared
with the CPU oracle, on the policy path, the span path and a call with views.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from test_gpu_boundaries import LITS, R_AT, R_OK, device_words, hit_pairs
from test_gpu_parity import oracle_policy, oracle_spans
from test_gpu_views import ViewOracle

pytestmark = pytest.mark.gpu

TOK = b"alphabetagamma"                    # rule 0: an exact factor, a direct hit in policy mode, a VM run in span mode
ERR_SLOT_OVERFLOW, ERR_L1_OVERFLOW = 16, 32
CONFIGS = [(LITS + [R_OK], 2), (LITS + [R_AT], 4)]


@pytest.fixture(scope="module")
def N():
    from vainplex_openclaw_b200 import _native
    _native.init()
    return _native


def quiet(rng, length):
    """text no rule matches: x, y and spaces"""
    t = np.where(rng.random(length) < 0.5, ord("x"), ord("y")).astype(np.uint8)
    t[rng.random(length) < 0.15] = ord(" ")
    return bytes(t)


def check_all(N, oracle, rs, rules, msgs):
    """policy words and hits (host and device path), spans, and both through views (every other message in the empty view)"""
    data, off = N.pack(msgs)
    ewords, ehits = oracle_policy(oracle, rules, data, off)
    words, hits = rs.scan_batch(data, off)
    assert np.array_equal(words, ewords) and hit_pairs(hits) == ehits
    assert np.array_equal(device_words(N, rs, data, off), ewords)
    counters = rs.work_counters()
    got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in rs.find_matches_batch(data, off)]
    assert got == oracle_spans(oracle, rules, data, off)
    views = [list(range(len(rules))), []]
    ids = np.arange(len(msgs), dtype=np.uint8) % 2
    vwords, vhits, vspans = ViewOracle(oracle, rules).of(msgs, ids, views)
    rs.set_views(views)
    w2, h2 = rs.scan_batch(data, off, views=ids)
    assert np.array_equal(w2, vwords) and hit_pairs(h2) == vhits
    s2 = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in rs.find_matches_batch(data, off, views=ids)]
    assert sorted(s2) == sorted(vspans)
    return ewords, counters


@pytest.mark.parametrize("layout", ["one message", "a message per token"])
@pytest.mark.parametrize("rules,options", CONFIGS, ids=["stride2", "stride4"])
def test_one_warps_occurrences(N, oracle, rules, options, layout):
    """0, 31, 32, 33 and 64 occurrences inside the first kilobyte of the batch: one scan warp's flag words, one confirm
    warp's buffer (empty, one short of full, full, one over, two full appends).  In one message, every lane of a resolve
    warp asks for the same message's slot; a message per token makes them claim slots apart."""
    rs = N.Ruleset(rules, options=options, strict=True)
    rng = np.random.default_rng(5)
    per_token = None
    for k in (1, 0, 31, 32, 33, 64):
        # (a quiet first message: the head check confirms an occurrence within three bytes of the range's start a second time)
        if layout == "one message":
            head = [b" " + b" ".join([TOK] * k) + b" " + quiet(rng, 30)]
        else:
            head = [b" " + TOK for _ in range(k)]
        msgs = [b"xyxy"] + head + [quiet(rng, int(rng.integers(0, 300))) for _ in range(300)]
        ewords, counters = check_all(N, oracle, rs, rules, msgs)
        hit_msgs = int((ewords >> np.uint64(63)).sum())
        assert hit_msgs == (min(k, 1) if layout == "one message" else k), k
        if k == 1:
            per_token = counters[4]
            assert per_token >= 1
        assert counters[4] == k * per_token, k                     # confirmed occurrences: every one counted once
        assert counters[0] >= hit_msgs, k                          # slots: at least one per hit message
    rs.close()


@pytest.mark.parametrize("rules,options", CONFIGS, ids=["stride2", "stride4"])
def test_messages_race_for_slots(N, oracle, rules, options):
    """Thousands of messages with several occurrences each: a message's occurrences sit in different resolve warps, which
    race for its slot; the losers' slots stay unused, and every result equals the oracle."""
    rs = N.Ruleset(rules, options=options, strict=True)
    rng = np.random.default_rng(11)
    toks = [TOK, b"thequickbrownfox", b"ZEPPELIN_Airship", b"ok" if options == 2 else b"bob@example"]
    msgs = []
    for i in range(6000):
        parts = [quiet(rng, int(rng.integers(0, 40)))]
        if rng.random() < 0.4:
            for _ in range(int(rng.integers(2, 9))):
                parts += [b" " + toks[int(rng.integers(0, len(toks)))] + b" ", quiet(rng, int(rng.integers(0, 20)))]
        msgs.append(b"".join(parts))
    ewords, counters = check_all(N, oracle, rs, rules, msgs)
    assert counters[0] >= int((ewords >> np.uint64(63)).sum())
    rs.close()


@pytest.mark.parametrize("queue", ["occurrences", "slots"])
def test_tail_queue_overflow_grows_and_recovers(N, oracle, queue):
    """A rule set whose queues a small batch sized, then a batch with more confirmed occurrences (dense tokens) or more hit
    messages (a token in each of 20 000) than they hold: every word of that batch says "incomplete", cg_scan_join reports
    CG_ERR_CAPACITY once, the counter of the overflowed queue counted all it needed, and the batch scanned again equals the
    oracle."""
    import torch
    rules = LITS + [R_OK]
    rs = N.Ruleset(rules, options=2, strict=True)
    rng = np.random.default_rng(23)
    st = torch.cuda.Stream()
    small = [quiet(rng, 200) for _ in range(64)]
    if queue == "occurrences":
        big = [b" ".join([TOK] * 6500) for _ in range(16)]        # about 104 000 occurrences; the queue holds 65 536
    else:
        big = [quiet(rng, int(rng.integers(0, 60))) + b" " + TOK + b" " + quiet(rng, 20) for _ in range(20000)]   # 4 096 slots
    outs = []
    for msgs in (small, big):
        data, off = N.pack(msgs)
        dd = torch.from_numpy(np.ascontiguousarray(data)).cuda()
        oo = torch.from_numpy(off.astype(np.int32)).cuda()
        out = torch.zeros(len(msgs), dtype=torch.int64, device="cuda")
        rs.scan_batch_device(dd.data_ptr(), oo.data_ptr(), len(msgs), out.data_ptr(), st.cuda_stream)
        outs.append((data, off, dd, oo, out))
    with pytest.raises(N.GovError) as ei:
        rs.scan_join(st.cuda_stream)
    assert ei.value.code == N.CG_ERR_CAPACITY
    failed = rs.work_counters()
    assert failed[3] & (ERR_L1_OVERFLOW if queue == "occurrences" else ERR_SLOT_OVERFLOW)
    data, off, dd, oo, out = outs[1]
    assert (out.cpu().numpy().view(np.uint64) == np.uint64(0xffffffffffffffff)).all()
    rs.scan_batch_device(dd.data_ptr(), oo.data_ptr(), len(big), out.data_ptr(), st.cuda_stream)
    rs.scan_join(st.cuda_stream)                                       # (complete now: no error)
    done = rs.work_counters()
    assert done[3] == 0
    ewords, _ = oracle_policy(oracle, rules, data, off)
    assert np.array_equal(out.cpu().numpy().view(np.uint64), ewords)
    if queue == "occurrences":
        assert failed[4] == done[4] > 65536                            # counted past the capacity, every one once
    else:
        assert failed[0] >= 20000 and done[0] >= 20000 and int((ewords >> np.uint64(63)).sum()) == 20000
    rs.close()


def test_vm_event_queue_grows(N, oracle):
    """Span mode queues one VM run per (message, rule): 8 000 hit messages on a rule set whose event queue a small batch
    sized at 4 096 runs past it; the call grows the queue, runs again, and its spans equal the oracle's."""
    rules = LITS + [R_OK]
    rs = N.Ruleset(rules, options=2, strict=True)
    rng = np.random.default_rng(29)
    small = [quiet(rng, 200) for _ in range(64)]
    d0, o0 = N.pack(small)
    assert len(rs.find_matches_batch(d0, o0)) == 0
    msgs = [quiet(rng, int(rng.integers(0, 60))) + b" " + TOK + b" " + quiet(rng, 20) for _ in range(8000)]
    data, off = N.pack(msgs)
    got = [(int(s["msg"]), int(s["rule"]), int(s["start16"]), int(s["end16"])) for s in rs.find_matches_batch(data, off)]
    assert got == oracle_spans(oracle, rules, data, off)
    assert rs.work_counters()[1] >= 8000                               # VM pairs: past the first capacity
    rs.close()
