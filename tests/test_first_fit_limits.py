"""The first-fit wave chain (KA_WAVE_FIRST_FIT) at its limits, every device result checked field by field against
fit_models.plan_waves (and models.plan_waves where the greedy rule runs too):

- the claim reset after 2^21 rounds, in all four first-fit chain instances (state in shared or global memory, with or without a
  sender), on plans of about 2.1 M rows whose load table stays under 2^29 bytes;
- the shared-memory band with senders: N + n_send = 25 600 rows of 8 bytes in shared memory, 25 601 in global memory;
- the bound Wb the device computes, seen through KA_ERR_LIMIT (a = Wb) on tables too wide for it, on both branches of its min,
  and the load-table limit of 2^30 bytes with a send table;
- walks that end at wave Wb through the chain's loop bound, and a bucket filled to exactly its budget;
- the last sender index below KA_WAVE_NO_SENDER (65 534), under both rules;
- a plan of more than 65 536 waves: the log pass over a tall table, the second summary call and three radix passes.

The device does not report Wb or its rounds. fit_models.bound and models.chain_rounds restate them, and the CPU tests here check
with them that each input reaches the edge it is named for."""
import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SEND_SUMMARY_DTYPE, WAVE_SUMMARY_DTYPE
from tests import fit_models, models, util

LIMIT = _native.KA_ERR_LIMIT
CHUNK, RESET = models.WAVE_CHUNK, models.WAVE_RESET
SMEM_ROWS = 25600            # KA_SMEM_BUDGET / KA_WAVE_FIT_ROW_BYTES: rows of chain state (claim, hint) in shared memory
TABLE_LIMIT = 1 << 30        # KA_WAVE_FIT_MAX_BYTES: the load table [N + n_send][Wb] of int64
NO_SENDER = 0xFFFF           # KA_WAVE_NO_SENDER: the largest sender index is 65 534


def bound_of(rep_off, cur, out, out_len, send):
    """fit_models.bound over the records of these rows (send: with their senders)."""
    records, senders = models.wave_records(rep_off, cur, out, out_len)
    return fit_models.bound([(g, r, 1, s if send else None) for g, (r, s) in enumerate(zip(records, senders)) if r])


def _solver(ids, rule="first_fit"):
    s = kab.Solver(0)
    s.set_brokers(*util.table(ids, 8))
    s.set_wave_rule(rule)
    return s


# ---- the claim reset -------------------------------------------------------------------------------------------------------

def reset_input(send, seed=11):
    """A plan whose chain crosses round 2^21 in a chunk of mixed rows, with a load table of at most 2^29 bytes. A serial prefix of
    1 023 x 2 048 + 1 987 records fills 2^21 - 61 rounds with a Wb near 1 000 (700 with a sender): without a sender, record i receives
    b(i mod 8 191) and b(i + 1 mod 8 191); with one, record i is led by s(i / 2 mod 6 000) and receives r((i + 1) / 2 mod 6 000),
    so records i and i + 1 share a leader or a receiver. A prefix row weighs the budget. Then a tail of random rows on other
    brokers: four hot receivers (and, with a sender, four hot leaders), weights 0 .. 2 x the budget, unchanged rows and rows
    without receivers. Its first records fill the prefix's last chunk; the next chunk starts 60 rounds before the reset and runs
    past it. Chain state: N = 25 600 (shared memory) and 25 601 brokers (global); with a sender N = 12 800 and a send table of
    12 800 or 12 801 ids."""
    rng = np.random.default_rng(seed)
    n_pre = 1023 * CHUNK + CHUNK - 1 - 60
    i = np.arange(n_pre)
    if send:
        K, B, C, N = 6000, 9, 5, 12800
        lead = 1 + (i // 2) % K
        pre_cur, pre_rep = lead.astype(np.int32), 1
        pre_new = np.stack([lead, K + 1 + ((i + 1) // 2) % K, np.full(n_pre, -1)], axis=1)
        first_free, n_tail, p_hot = 2 * K + 1, 24000, 0.25
    else:
        K, B, C, N = 8191, 7, None, SMEM_ROWS
        pre_cur, pre_rep = np.zeros(0, dtype=np.int32), 0
        pre_new = np.stack([1 + i % K, 1 + (i + 1) % K, np.full(n_pre, -1)], axis=1)
        first_free, n_tail, p_hot = K + 1, 20000, 0.3
    pool = np.arange(first_free, N + 1)
    hot, leaders = pool[:4], pool[4:8]
    cur_lists, new_lists = [], []
    for g in range(n_tail):
        c = [int(x) for x in rng.choice(pool, int(rng.integers(0, 4)), replace=False)]
        if send and c and rng.random() < 0.15:
            c[0] = int(rng.choice(leaders[~np.isin(leaders, c)]))
        u = rng.random()
        if u < 0.2:
            new = list(c)                                   # unchanged
        elif u < 0.3:
            new = c[1:] + c[:1]                             # a reorder or a drop: no receiver
        else:
            new, n = c[:1], 2 + int(rng.integers(0, 2))
            while len(new) < n:
                b = int(rng.choice(hot)) if len(new) == 1 and rng.random() < p_hot else int(rng.choice(pool))
                if b not in new and b not in c:
                    new.append(b)
        cur_lists.append(c)
        new_lists.append(new)
    t_off, t_cur = util.cur_lists(cur_lists)
    t_out, t_len = util.rows(new_lists, 3)
    budget = C if send else B
    weight = np.concatenate([np.full(n_pre, budget), rng.integers(0, 2 * budget + 1, len(t_len))]).astype(np.int64)
    rep_off = np.concatenate([np.arange(n_pre + 1, dtype=np.int64) * pre_rep, n_pre * pre_rep + t_off[1:]])
    ids, racks = util.table(np.arange(1, N + 1), 8)
    inp = dict(rep_off=rep_off, cur=np.concatenate([pre_cur, t_cur]).astype(np.int32),
               out=np.concatenate([pre_new, t_out]).astype(np.int32), out_len=np.concatenate([np.full(n_pre, 2), t_len]).astype(np.int32),
               weight=weight, B=np.int64(B), ids=ids, racks=racks)
    if send:
        inp.update(C=np.int64(C), send_smem=np.arange(1, SMEM_ROWS - N + 1, dtype=np.int32),
                   send_global=np.arange(1, SMEM_ROWS - N + 2, dtype=np.int32))
    else:
        gids, gracks = util.table(np.arange(1, N + 2), 8)
        inp.update(ids_global=gids, racks_global=gracks)
    return inp


_CASES = {}


def reset_case(form):
    """(input, records, senders or None, chain rounds, Wb) of reset_input, computed once per form."""
    if form not in _CASES:
        send = form == "send"
        inp = reset_input(send)
        records, senders = models.wave_records(inp["rep_off"], inp["cur"], inp["out"], inp["out_len"])
        senders = senders if send else None
        rounds = models.chain_rounds(records, senders)
        Wb = fit_models.bound([(g, r, 1, None if senders is None else senders[g]) for g, r in enumerate(records) if r])
        _CASES[form] = inp, records, senders, rounds, Wb
    return _CASES[form]


def _state_rows(inp, tag):
    """N + n_send of the plan with chain state in shared memory (tag "smem") or in global memory ("global")."""
    if "C" in inp:
        return len(inp["ids"]) + len(inp["send_" + tag])
    return len(inp["ids_global" if tag == "global" else "ids"])


@pytest.mark.parametrize("form", ["receive", "send"])
def test_reset_inputs_reach_the_edges(form):
    """The chain's rows sit exactly at 25 600 / 25 601; the rounds cross 2^21 inside one chunk with records and shared brokers
    or senders on both sides; Wb keeps the load table under 2^29 bytes (so the send-form prefix's Wb is not the 2.1 M a single
    leader would give)."""
    inp, records, senders, rounds, Wb = reset_case(form)
    assert [_state_rows(inp, t) for t in ("smem", "global")] == [SMEM_ROWS, SMEM_ROWS + 1]
    before, after, shared, later = models.crossing_chunk(records, senders, rounds)
    assert before >= 300 and after >= 300 and shared >= 4 and later >= 3, (before, after, shared, later)
    assert int(rounds.max()) > RESET
    assert 500 <= Wb and Wb * (SMEM_ROWS + 1) * 8 <= TABLE_LIMIT // 2, Wb


# The first-fit plans of both state placements, in a child process (util.run_child), written back to the directory given.
_CHILD = r"""
import sys
import time
import numpy as np
import kafka_assigner_b200 as kab
d = sys.argv[1]
a = dict(np.load(d + "/in.npz"))
send = "C" in a
res = {}
for tag in ("smem", "global"):
    s = kab.Solver(0)
    g = tag == "global" and not send
    s.set_brokers(a["ids_global"] if g else a["ids"], a["racks_global"] if g else a["racks"])
    s.set_wave_rule("first_fit")
    kw = dict(max_broker_out=int(a["C"]), send_brokers=a["send_" + tag]) if send else {}
    t = time.perf_counter()
    wave, summ, st = s.plan_waves(a["rep_off"], a["cur"], a["out"], a["out_len"], int(a["B"]), weight=a["weight"], **kw)
    print("%s plan_waves %.2f s" % (tag, time.perf_counter() - t))
    res[tag + "_wave"], res[tag + "_summary"], res[tag + "_status"] = wave, summ, np.array([st.code, st.a, st.b])
np.savez(d + "/out.npz", **res)
"""
CHILD_TIMEOUT = 300   # seconds: the child's two calls take about 11 s on an H100 (DESIGN.md), the model about 35 s


@pytest.fixture(scope="module", params=["receive", "send"])
def reset_plans(request, tmp_path_factory, native_lib):
    """(input, device results, model waves, model summaries) of reset_input: the device's from the child, the model's computed
    meanwhile."""
    send = request.param == "send"
    d = tmp_path_factory.mktemp("fit_" + request.param)
    inp = reset_input(send)
    np.savez(d / "in.npz", **inp)

    def expected():
        e_wave, e_summ, e_st = fit_models.plan_waves(inp["rep_off"], inp["cur"], inp["out"], inp["out_len"], inp["ids"], int(inp["B"]),
                                                     inp["weight"], (inp["send_smem"], int(inp["C"])) if send else None)
        assert e_st == (0, 0, 0)
        return e_wave, util.summary_array(e_summ, WAVE_SEND_SUMMARY_DTYPE if send else WAVE_SUMMARY_DTYPE)

    (e_wave, e_summ), out, secs = util.run_child(_CHILD, d, CHILD_TIMEOUT, expected, "the first-fit plans of " + request.param)
    print("%s: child and model %.1f s\n%s" % (request.param, secs, out))
    return inp, dict(np.load(d / "out.npz")), e_wave, e_summ


@pytest.mark.gpu
def test_plans_cross_round_2_21(reset_plans):
    """All four first-fit chain instances: every wave, W and summary field of both state placements equal the model."""
    inp, dev, e_wave, e_summ = reset_plans
    for tag in ("smem", "global"):
        assert dev[tag + "_status"].tolist() == [0, 0, 0], tag
        assert np.array_equal(dev[tag + "_wave"], e_wave), (tag, np.nonzero(dev[tag + "_wave"] != e_wave)[0][:10])
        assert len(dev[tag + "_summary"]) == len(e_summ), tag
        for f in e_summ.dtype.names:
            assert np.array_equal(dev[tag + "_summary"][f], e_summ[f]), (tag, f)


# ---- the shared-memory band with senders --------------------------------------------------------------------------------------

def send_band_input(rows):
    """6 000 random rows over 12 800 brokers, the send table those brokers padded with ids no row names to N + n_send = rows. One
    hot leader leads every tenth row (Wb is about 750, far below the 5 242 the table allows at 25 600 rows), and
    every 50th row receives only hot brokers."""
    rng = np.random.default_rng(rows)
    N, Q = 12800, 6000
    ids = np.arange(1, N + 1, dtype=np.int32)
    hot, lead = ids[-5:], int(ids[7])
    cur_lists = [[int(x) for x in rng.choice(ids, int(rng.integers(0, 4)), replace=False)] for _ in range(Q)]
    new_lists = []
    for g, c in enumerate(cur_lists):
        if g % 10 == 0:
            c[:] = [lead] + [x for x in c if x != lead][:2]
        new_lists.append([int(x) for x in rng.choice(hot if g % 50 == 0 else ids, int(rng.integers(1, 4)), replace=False)])
    send_ids = np.concatenate([ids, 10 ** 8 + np.arange(rows - 2 * N)]).astype(np.int32)
    return ids, send_ids, util.cur_lists(cur_lists), util.rows(new_lists, 3)


@pytest.mark.parametrize("rows", [SMEM_ROWS, SMEM_ROWS + 1])
def test_send_band_input(rows):
    ids, send_ids, (rep_off, cur), (out, out_len) = send_band_input(rows)
    assert len(ids) + len(send_ids) == rows
    Wb = bound_of(rep_off, cur, out, out_len, True)
    assert 300 <= Wb <= 1000 and Wb * rows * 8 <= TABLE_LIMIT, Wb


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [SMEM_ROWS, SMEM_ROWS + 1])
def test_send_band(native_lib, rows):
    ids, send_ids, (rep_off, cur), (out, out_len) = send_band_input(rows)
    s = _solver(ids)
    wave, summ, st = util.check_plan(s, rep_off, cur, out, out_len, 4, None, send_ids, 6)
    assert st.code == 0 and len(summ) > 1


# ---- the bound Wb, through KA_ERR_LIMIT --------------------------------------------------------------------------------------

WIDE = np.arange(1, 65536, dtype=np.int32)   # 65 535 brokers: the table refuses Wb > 2 048 without a send table


def refused_inputs():
    """(name, rows, send_ids or None) of plans whose load table on WIDE is over 2^30 bytes. Random rows of up to 8 receivers among
    60 brokers, some hot, so that Wb = 1 + the sum over a row (below M); and 3 000 rows all receiving the same 8 brokers, so that
    Wb = M. The send forms add leaders, some hot, whose S_s - 1 is part of the sum."""
    rng = np.random.default_rng(23)
    pool, hot = np.arange(1, 61), np.array([3, 17, 42])
    res = []
    for send in (False, True):
        cur_lists, new_lists = [], []
        for g in range(5000):
            lead = int(rng.choice([61, 62])) if send and g % 4 == 0 else int(rng.integers(61, 100))
            n = int(rng.integers(1, 9))
            new = [int(x) for x in rng.choice(pool, n, replace=False)]
            if g % 3 == 0 and not set(hot) & set(new):
                new[0] = int(rng.choice(hot))
            cur_lists.append([lead] if send else [])
            new_lists.append(new)
        res.append(("random_send" if send else "random", (util.cur_lists(cur_lists), util.rows(new_lists, 8)),
                    np.arange(61, 100, dtype=np.int32) if send else None))
        same = [int(x) for x in range(2, 10)]
        res.append(("same_eight_send" if send else "same_eight", (util.cur_lists([[1] if send else []] * 3000),
                                                                    util.rows([same] * 3000, 8)),
                    np.array([1], dtype=np.int32) if send else None))
    return res


def test_refused_inputs_are_over_the_limit():
    for name, ((rep_off, cur), (out, out_len)), send_ids in refused_inputs():
        Wb = bound_of(rep_off, cur, out, out_len, send_ids is not None)
        M = int((out_len > 0).sum())
        rows = len(WIDE) + (0 if send_ids is None else len(send_ids))
        assert Wb * rows * 8 > TABLE_LIMIT, name
        if name.startswith("same_eight"):
            assert Wb == M == 3000, name
        else:
            assert Wb < M, name
            if send_ids is not None:   # the senders' term decides Wb
                no_send = bound_of(rep_off, cur, out, out_len, False)
                assert no_send < Wb, (no_send, Wb)


@pytest.mark.gpu
def test_bound_through_the_limit(native_lib):
    """Every plan is refused with KA_ERR_LIMIT, a = the model's Wb: the device's count and bound kernels give the closed form."""
    s = _solver(WIDE)
    for name, ((rep_off, cur), (out, out_len)), send_ids in refused_inputs():
        send = {} if send_ids is None else dict(max_broker_out=5, send_brokers=send_ids)
        wave, summ, st = s.plan_waves(rep_off, cur, out, out_len, 2, **send)
        assert (st.code, st.a) == (LIMIT, bound_of(rep_off, cur, out, out_len, send_ids is not None)), (name, st.code, st.a)
        assert len(wave) == 0 and len(summ) == 0


def _led_table(n_send):
    """A send table of n_send ids: broker 1, then 10^8, 10^8 + 1, ..."""
    return np.concatenate([[1], 10 ** 8 + np.arange(n_send - 1)]).astype(np.int32)


def test_send_table_limit_sizes():
    rep_off, cur = util.cur_lists([[1]] * 2048)
    out, out_len = util.rows([[1, 2]] * 2048)
    assert bound_of(rep_off, cur, out, out_len, True) == 2048
    assert 2048 * (40 + 65496) * 8 == TABLE_LIMIT and 65497 < NO_SENDER


@pytest.mark.gpu
def test_send_table_limit(native_lib):
    """N = 40, 2 048 rows led by broker 1 and receiving broker 2: Wb = 2 048. A send table of 65 496 ids makes a load table of
    exactly 2^30 bytes, which is planned; one more id is refused with a = 2 048."""
    s = _solver(np.arange(1, 41))
    rep_off, cur = util.cur_lists([[1]] * 2048)
    out, out_len = util.rows([[1, 2]] * 2048)
    wave, summ, st = util.check_plan(s, rep_off, cur, out, out_len, 1, None, _led_table(65496), 1)
    assert st.code == 0 and wave.tolist() == list(range(1, 2049)) and len(summ) == 2048
    wave, summ, st = s.plan_waves(rep_off, cur, out, out_len, 1, max_broker_out=1, send_brokers=_led_table(65497))
    assert (st.code, st.a) == (LIMIT, 2048) and len(wave) == 0


# ---- walks that end at Wb, and the exact cap ---------------------------------------------------------------------------------

# (current lists, new lists, B, weights, sender budget C or None, first-fit waves, greedy waves)
HAND = [
    # four heavy rows fill waves 1-4 of broker 2; the weight-0 row walks up from wave 1 and stops at Wb = 5
    ([[1]] * 5, [[2]] * 5, 3, [7, 7, 7, 7, 0], None, [1, 2, 3, 4, 5], [1, 2, 3, 4, 5]),
    # every row has its own receiver: only the sender term of Wb (S_1 - 1 = 4) lets the weight-0 row reach wave 5
    ([[1]] * 5, [[1, 2], [1, 3], [1, 4], [1, 5], [1, 6]], 100, [4, 4, 4, 4, 0], 3, [1, 2, 3, 4, 5], [1, 2, 3, 4, 5]),
    # 3 + 0 fills wave 1 to exactly B, 1 + 2 wave 2; first fit puts the last weight-0 row back in wave 1
    ([[1]] * 5, [[2]] * 5, 3, [3, 0, 1, 2, 0], None, [1, 1, 2, 2, 1], [1, 1, 2, 2, 2]),
]


def _hand_args(cur_l, new_l, weight):
    rep_off, cur = util.cur_lists(cur_l)
    out, out_len = util.rows(new_l)
    return rep_off, cur, out, out_len, np.asarray(weight, dtype=np.int64)


@pytest.mark.parametrize("case", range(len(HAND)))
def test_hand_worked_models(case):
    cur_l, new_l, B, weight, C, fit, greedy = HAND[case]
    rep_off, cur, out, out_len, w = _hand_args(cur_l, new_l, weight)
    send = None if C is None else (list(range(1, 41)), C)
    ids = np.arange(1, 41)
    assert fit_models.plan_waves(rep_off, cur, out, out_len, ids, B, w, send)[0].tolist() == fit
    assert models.plan_waves(rep_off, cur, out, out_len, ids, B, w, send)[0].tolist() == greedy
    Wb = bound_of(rep_off, cur, out, out_len, C is not None)
    if case < 2:
        assert Wb == max(fit) == 5
    if case == 1:   # without the sender term the bound would be 1
        assert bound_of(rep_off, cur, out, out_len, False) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(HAND)))
def test_hand_worked(native_lib, case):
    cur_l, new_l, B, weight, C, fit, greedy = HAND[case]
    rep_off, cur, out, out_len, w = _hand_args(cur_l, new_l, weight)
    s = _solver(np.arange(1, 41))
    send_ids = None if C is None else np.arange(1, 41, dtype=np.int32)
    for rule, expect in (("first_fit", fit), ("greedy", greedy)):
        wave, _, st = util.check_plan(s, rep_off, cur, out, out_len, B, w, send_ids, C, rule)
        assert st.code == 0 and wave.tolist() == expect, rule


# ---- the last sender index ---------------------------------------------------------------------------------------------------

def last_sender_input():
    """3 000 rows over brokers 1..40, led by ids of a send table of 65 535 ids (10^8 + k): a quarter by its first id, a quarter by
    its last (index 65 534), the rest by others; rows keep or drop their leader."""
    rng = np.random.default_rng(65534)
    send_ids = (10 ** 8 + np.arange(NO_SENDER)).astype(np.int32)
    pick = rng.integers(0, 4, 3000)
    leads = np.where(pick == 0, send_ids[0], np.where(pick == 1, send_ids[-1], rng.choice(send_ids[1:-1], 3000)))
    cur_lists, new_lists = [], []
    for g, lead in enumerate(leads.tolist()):
        cur_lists.append([lead] + [int(x) for x in rng.choice(np.arange(1, 41), int(rng.integers(0, 2)), replace=False)])
        recv = [int(x) for x in rng.choice(np.arange(1, 41), int(rng.integers(1, 3)), replace=False)]
        new_lists.append([lead] + recv if g % 3 else recv)
    return send_ids, util.cur_lists(cur_lists), util.rows(new_lists, 3)


def test_last_sender_input():
    send_ids, (rep_off, cur), (out, out_len) = last_sender_input()
    assert len(send_ids) == NO_SENDER and int(send_ids[-1]) in cur.tolist()
    Wb = bound_of(rep_off, cur, out, out_len, True)
    assert Wb * (40 + NO_SENDER) * 8 <= TABLE_LIMIT and Wb <= 2046, Wb


@pytest.mark.gpu
@pytest.mark.parametrize("rule", ["first_fit", "greedy"])
def test_last_sender_index(native_lib, rule):
    send_ids, (rep_off, cur), (out, out_len) = last_sender_input()
    s = _solver(np.arange(1, 41), rule)
    for B, C in ((1, 2), (3, 4)):
        wave, summ, st = util.check_plan(s, rep_off, cur, out, out_len, B, None, send_ids, C, rule)
        assert st.code == 0 and len(summ) > 1


# ---- more than 65 536 waves --------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("send", [False, True])
def test_more_than_65536_waves(native_lib, send):
    """70 000 rows all received by broker 2 (B = 1; with a sender, all led by broker 1): W = Wb = 70 000. plan_waves makes its
    second summary call, and plan_waves_json's radix passes take three digits; every document byte for byte."""
    Q = 70000
    s = _solver(np.arange(1, 41))
    rep_off, cur = util.cur_lists([[1]] * Q)
    out, out_len = util.rows([[2]] * Q)
    send_ids = np.arange(1, 41, dtype=np.int32) if send else None
    wave, summ, st = util.check_plan(s, rep_off, cur, out, out_len, 1, None, send_ids, 1 if send else None)
    assert st.code == 0 and len(summ) == Q > kab.Solver.WAVE_SUMMARY_CAP
    names = ["tall.%d" % t for t in range(7)]
    part_off = np.arange(8, dtype=np.int64) * (Q // 7)
    kw = dict(max_broker_out=1, send_brokers=send_ids) if send else {}
    docs, d_wave, d_summ, st = s.plan_waves_json(names, part_off, None, rep_off, cur, out, out_len, 1, **kw)
    e_docs, _, _, e_wave, _, e_st = fit_models.wave_documents(names, part_off, None, rep_off, cur, out, out_len, s.broker_id, 1,
                                                              None, (list(send_ids), 1) if send else None)
    assert st.code == 0 and e_st == (0, 0, 0)
    assert np.array_equal(d_wave, e_wave) and np.array_equal(d_summ, summ)
    assert len(docs) == len(e_docs) == Q
    assert b"".join(bytes(x) for x in docs) == b"".join(e_docs) and [len(x) for x in docs] == [len(e) for e in e_docs]
