"""ka_plan_waves_send and ka_plan_waves_send_json: a wave plan that caps what each partition's leader sends per wave as well as
what each broker receives. `models.plan_waves` with `send` restates the rule of include/kassign.h as a plain loop; every wave,
W, summary and document of the device must equal it. The CPU tests pin the model on hand-worked cases and its invariants on
random inputs, the declarations, and what Solver.plan_waves / plan_waves_json hand the C ABI."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SEND_SUMMARY_DTYPE, WAVE_SUMMARY_DTYPE
from tests import models, util

FIELDS = WAVE_SEND_SUMMARY_DTYPE.names
INT64_MAX = np.iinfo(np.int64).max
BAD, LIMIT = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT


def _model(cur_lists, new_lists, B, C, weight=None, ids=range(1, 100), send_ids=range(1, 100)):
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists)
    return models.plan_waves(rep_off, cur, out, out_len, list(ids), B, weight, send=(list(send_ids), C))


def send_loads(cur_lists, new_lists, wave, weight=None):
    """{(wave, leader): [what each of its rows sends]} of a plan."""
    w = np.ones(len(wave), dtype=np.int64) if weight is None else np.asarray(weight, dtype=np.int64)
    res = {}
    for g, (old, new) in enumerate(zip(cur_lists, new_lists)):
        r = sum(b not in old for b in new)
        if r and old:
            res.setdefault((int(wave[g]), old[0]), []).append(int(w[g]) * r)
    return res


# ---- CPU -----------------------------------------------------------------------------------------------------------------

def test_symbols_are_exported_and_declared(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kassign.h")).read()
    for name, n_args in (("ka_plan_waves_send", 18), ("ka_plan_waves_send_json", 25)):
        assert hasattr(raw, name)
        res, args = _native.SYMBOLS[name]
        assert res is ctypes.c_int32 and len(args) == n_args
        assert "int32_t %s(ka_ctx* ctx," % name in header
    assert "} ka_wave_send_summary;" in header
    assert ctypes.sizeof(_native.KaWaveSendSummary) == 16 and WAVE_SEND_SUMMARY_DTYPE.itemsize == 56
    assert WAVE_SEND_SUMMARY_DTYPE.names[:5] == WAVE_SUMMARY_DTYPE.names


def test_without_a_context_is_no_device(native_lib):
    L = native_lib
    st = kab.KaStatus()
    n = ctypes.c_int32(5)
    args = (None, 0, None, None, 1, None, None, None, 1, 0, None, 1, None, ctypes.byref(n), None, None, 0)
    assert L.ka_plan_waves_send(*args, ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE
    assert st.code == _native.KA_ERR_NO_DEVICE and n.value == 0
    assert L.ka_plan_waves_send(*args, None) == BAD
    n.value = 5
    jargs = (None, 0, None, None, None, None, 1, None, None, None, 1, 0, None, 1, None, None, None, 0, None, None, ctypes.byref(n), None,
             None, 0)
    assert L.ka_plan_waves_send_json(*jargs, ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE and n.value == 0


def test_model_drained_leader_is_split():
    """Broker 1 leads 12 rows, each moving one replica to its own receiver: a receive budget alone puts them all in wave 1, a send
    budget of 5 cuts them into waves of 5."""
    cur = [[1, 2]] * 12
    new = [[2, 10 + g] for g in range(12)]
    wave, summ, st = models.plan_waves(*util.cur_lists(cur), *util.rows(new), list(range(2, 40)), 1)
    assert st == (0, 0, 0) and wave.tolist() == [1] * 12
    wave, summ, st = _model(cur, new, 1, 5)
    assert st == (0, 0, 0) and wave.tolist() == [1] * 5 + [2] * 5 + [3] * 2
    assert [(s["max_broker_out"], s["max_broker_out_id"]) for s in summ] == [(5, 1), (5, 1), (2, 1)]
    assert [(s["max_broker_in"], s["max_broker_in_id"]) for s in summ] == [(1, 10), (1, 15), (1, 20)]
    assert [s["rows"] for s in summ] == [5, 5, 2]


def test_model_hand_worked_cases():
    # a row heavier than C opens its sender's wave alone; a zero weight sends nothing and joins its sender's open wave
    wave, summ, _ = _model([[1], [1], [1], [1]], [[2], [3, 4], [5], [6]], 10, 3, weight=[1, 4, 1, 0])
    assert wave.tolist() == [1, 2, 3, 3]   # row 1 sends 8 > C: a wave of its own; row 2 cannot join it
    assert [s["max_broker_out"] for s in summ] == [1, 8, 1]
    # a broker that sends one row and receives another: separate budgets
    wave, summ, _ = _model([[1], [2], [1]], [[2], [1], [3]], 1, 1)
    assert wave.tolist() == [1, 1, 2]
    assert [(s["max_broker_in"], s["max_broker_in_id"], s["max_broker_out"], s["max_broker_out_id"]) for s in summ] == [
        (1, 1, 1, 1), (1, 3, 1, 1)]
    # an empty current list has no sender: only the receive budget applies, and the send table need not hold anything
    wave, summ, st = _model([[], [], [1]], [[2], [3], [4]], 1, 1, send_ids=[1])
    assert st == (0, 0, 0) and wave.tolist() == [1, 1, 1]
    assert [(s["max_broker_out"], s["max_broker_out_id"]) for s in summ] == [(1, 1)]
    # a row without receivers has no sender term either; nothing changed gives no wave
    assert _model([[5, 1]], [[1]], 1, 1, send_ids=[])[0].tolist() == [1]
    assert _model([[1, 2]], [[1, 2]], 1, 1)[1] == []
    # refusals: the lowest failing row; within a row the new list first
    assert _model([[1], [7], [1]], [[2], [3], [2, 2]], 1, 1, send_ids=[1])[2] == (BAD, 1, 7)
    assert _model([[7], [1]], [[200], [2]], 1, 1, send_ids=[1])[2] == (BAD, 0, 200)
    assert _model([[7], [1]], [[7, 2]], 1, 1, send_ids=[1])[2] == (BAD, 0, 7)


@pytest.mark.parametrize("seed", range(6))
def test_model_invariants(seed):
    rng = np.random.default_rng(seed)
    ids = np.arange(1, 13)
    cur_lists, new_lists = util.random_wave_case(rng, 300, 12)
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    for B, C, weight in ((1, 1, None), (2, 5, None), (10 ** 6, 3, None), (4, 10 ** 6, None), (50, 60, rng.integers(0, 40, 300)),
                         (30, 200, rng.integers(0, 80, 300))):
        wave, summ, st = models.plan_waves(rep_off, cur, out, out_len, ids, B, weight, send=(ids, C))
        assert st == (0, 0, 0)
        W = len(summ)
        assert W == (int(wave.max()) if len(wave) else 0)
        assert all(s["rows"] > 0 for s in summ) and set(wave.tolist()) - {0} == set(range(1, W + 1))
        w = np.ones(300, dtype=np.int64) if weight is None else np.asarray(weight, dtype=np.int64)
        inb = {}
        for g, (old, new) in enumerate(zip(cur_lists, new_lists)):
            for b in new:
                if b not in old:
                    inb.setdefault((int(wave[g]), b), []).append(int(w[g]))
        for ws in inb.values():
            assert sum(ws) <= B or sum(x > 0 for x in ws) == 1, ws
        for xs in send_loads(cur_lists, new_lists, wave, weight).values():
            assert sum(xs) <= C or sum(x > 0 for x in xs) == 1, xs
        # a send budget no plan reaches: no leader opens a wave, so a row's wave is the larger of ka_plan_waves's receiver term
        # and its leader's open wave (the wave of the leader's previous moved row)
        big = 8 * int(w.sum())
        wave, summ, _ = models.plan_waves(rep_off, cur, out, out_len, ids, B, weight, send=(ids, big))
        last = {}
        for g in range(300):
            r = [b for b in new_lists[g] if b not in cur_lists[g]]
            if r and cur_lists[g]:
                assert wave[g] >= last.get(cur_lists[g][0], 1)
                last[cur_lists[g][0]] = int(wave[g])
    # where no leader has two moved rows, the leaders' open waves never matter: exactly ka_plan_waves's plan
    cur_lists = [[g + 1] + c[1:] if rng.random() < 0.7 else [] for g, c in enumerate(cur_lists)]
    new_lists = [[b for b in x if b not in c[:1]] for x, c in zip(new_lists, cur_lists)]
    ids = np.arange(1, 301)
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    for B, weight in ((1, None), (3, None), (40, rng.integers(0, 30, 300))):
        wave, summ, _ = models.plan_waves(rep_off, cur, out, out_len, ids, B, weight, send=(ids, INT64_MAX))
        e_wave, e_summ, _ = models.plan_waves(rep_off, cur, out, out_len, ids, B, weight)
        assert np.array_equal(wave, e_wave) and [{k: s[k] for k in WAVE_SUMMARY_DTYPE.names} for s in summ] == e_summ


@pytest.mark.parametrize("W", [3, 100])
def test_plan_waves_with_a_send_budget_marshals_its_arguments(W):
    lib = util.FakeWaveLib(W)
    s = util.fake_solver(lib)
    out, out_len = util.rows([[1, 2], [3], [4, 5, 6], []])
    rep_off, cur = util.cur_lists([[1], [2, 3], [4], [7, 8]])
    weight = np.array([5, 0, 7, 1], dtype=np.int64)
    wave, summ, st = s.plan_waves(rep_off, cur, out, out_len, 9, weight=weight, max_broker_out=11, send_brokers=[1, 2, 4, 7])
    assert st.code == 0
    first = lib.calls[0]
    assert first["Q"] == 4 and first["stride"] == 3 and first["B"] == 9 and first["C"] == 11 and first["cap"] == 4
    assert first["send_id"].tolist() == [1, 2, 4, 7] and np.array_equal(first["weight"], weight)
    assert np.array_equal(first["rep_off"], rep_off) and np.array_equal(first["new_broker"], out.ravel())
    assert np.array_equal(wave, 1 + np.arange(4) % W)
    assert summ.dtype == WAVE_SEND_SUMMARY_DTYPE and len(summ) == W
    assert [list(x) for x in summ] == [[v * 10 + f for f in range(7)] for v in range(W)]
    assert len(lib.calls) == (2 if W > 4 else 1) and lib.calls[-1]["cap"] == max(W, 4)
    with pytest.raises(ValueError):
        s.plan_waves(rep_off, cur, out, out_len, 9, max_broker_out=11)
    with pytest.raises(ValueError):
        s.plan_waves(rep_off, cur, out, out_len, 9, send_brokers=[1])


def test_plan_waves_json_with_a_send_budget_marshals_its_arguments():
    lib = util.FakeWaveLib(3)
    s = util.fake_solver(lib)
    out, out_len = util.rows([[1, 2], [3], [4, 5, 6], []])
    rep_off, cur = util.cur_lists([[1], [2, 3], [4], [7, 8]])
    names, part_off = ["alpha", "", "bc"], [0, 3, 3, 4]
    docs, wave, summ, st = s.plan_waves_json(names, part_off, None, rep_off, cur, out, out_len, 9, max_broker_out=12,
                                             send_brokers=np.array([1, 2, 4, 7], dtype=np.int64))
    assert st.code == 0 and len(lib.calls) == 1
    c = lib.calls[0]
    assert c["T"] == 3 and c["B"] == 9 and c["C"] == 12 and c["cap"] == 4 and c["send_id"].tolist() == [1, 2, 4, 7]
    assert c["json_cap"] == models.json_bound(names, part_off, 3)
    assert [bytes(d) for d in docs] == [b"<0>", b"<1>", b"<2>"] and wave.tolist() == [1, 2, 3, 1]
    assert summ.dtype == WAVE_SEND_SUMMARY_DTYPE and [list(x) for x in summ] == [[v * 10 + f for f in range(7)] for v in range(3)]


# ---- GPU -----------------------------------------------------------------------------------------------------------------

def _check(s, rep_off, cur, out, out_len, B, C, send_ids, weight=None):
    """plan_waves with a send budget against the model, every field. Returns (wave, summary, status)."""
    wave, summ, st = s.plan_waves(rep_off, cur, out, out_len, B, weight=weight, max_broker_out=C, send_brokers=send_ids)
    e_wave, e_summ, e_st = models.plan_waves(rep_off, cur, out, out_len, s.broker_id, B, weight, send=(send_ids, C))
    assert (st.code, st.a, st.b) == e_st, ((st.code, st.a, st.b), e_st)
    if st.code == 0:
        assert np.array_equal(wave, e_wave), np.nonzero(wave != e_wave)[0][:10]
        assert [util.record_of(x, FIELDS) for x in summ] == e_summ
    return wave, summ, st


@pytest.mark.gpu
@pytest.mark.parametrize("remove", [0.0, 0.03])
def test_solve_rows(native_lib, remove):
    cl = kab.synth.make_ragged_cluster(T=4000, N=400, max_partitions=128, seed=7, remove_frac=remove)
    s, out, out_len, S = util.solved(cl)
    Q = len(out_len)
    weight = np.random.default_rng(3).integers(0, 1 << 30, Q).astype(np.int64)
    mean = int(weight.mean())
    for B, C, w in ((1, 1, None), (1, 4, None), (3, 2, None), (20, 20, None), (INT64_MAX, 1, None), (4 * mean, 4 * mean, weight),
                    (mean, 16 * mean, weight)):
        _check(s, cl.rep_off, cl.cur, out, out_len, B, C, cl.all_broker_id, w)
    for B, C, w in ((2, 2, None), (8 * mean, 2 * mean, weight)):
        util.check_wave_documents(s, cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, B, weight=w, C=C,
                                  send_ids=cl.all_broker_id)


@pytest.mark.gpu
def test_drained_brokers_send_within_the_budget(native_lib):
    """With brokers removed, a receive budget alone lets the drained leaders send far beyond C in one wave; the send budget holds
    every leader to C."""
    cl = kab.synth.make_ragged_cluster(T=4000, N=400, max_partitions=128, seed=9, remove_frac=0.03)
    s, out, out_len, S = util.solved(cl)
    B, C = 8, 8
    wave, _, st = s.plan_waves(cl.rep_off, cl.cur, out, out_len, B)
    assert st.code == 0
    lists = [cl.cur[cl.rep_off[g]:cl.rep_off[g + 1]].tolist() for g in range(len(out_len))]
    new = [out[g, :out_len[g]].tolist() for g in range(len(out_len))]
    assert max(sum(x) for x in send_loads(lists, new, wave).values()) > 4 * C
    wave, summ, st = _check(s, cl.rep_off, cl.cur, out, out_len, B, C, cl.all_broker_id)
    assert max(sum(x) for x in send_loads(lists, new, wave).values()) <= C and int(summ["max_broker_out"].max()) == C


@pytest.mark.gpu
def test_a_huge_send_budget(native_lib):
    """With C >= 8 x the sum of the weights no leader opens a wave. Where no leader has two moved rows (here: every row led by a
    broker of its own, or by nobody) the plan, every summary field of ka_plan_waves and every document are exactly those of
    ka_plan_waves / ka_plan_waves_json; on a solved cluster the device still equals the model."""
    s = kab.Solver(0)
    N = 3000
    s.set_brokers(*util.table(np.arange(1, N + 1), 8))
    rng = np.random.default_rng(12)
    Q = N
    cur_lists = [[g + 1] + [int(x) for x in rng.choice(np.arange(1, N + 1), 1)] if g % 5 else [] for g in range(Q)]
    cur_lists = [c[:1] if len(c) == 2 and c[0] == c[1] else c for c in cur_lists]
    hot = np.arange(N - 20, N + 1)
    new_lists = [[int(x) for x in rng.choice(hot if g % 2 else np.arange(1, N + 1), 2, replace=False)] for g in range(Q)]
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 2)
    weight = rng.integers(0, 1 << 20, Q).astype(np.int64)
    names, part_off = ["h%d" % t for t in range(30)], np.arange(31) * (Q // 30)
    send_ids = np.arange(1, N + 1, dtype=np.int32)
    for B, w in ((1, None), (5, None), (int(weight.mean()), weight)):
        big = 8 * (Q if w is None else int(w.sum()))
        for C in (big, INT64_MAX):
            wave, summ, st = _check(s, rep_off, cur, out, out_len, B, C, send_ids, w)
            e_wave, e_summ, e_st = s.plan_waves(rep_off, cur, out, out_len, B, weight=w)
            assert st.code == e_st.code == 0 and len(e_summ) > 1 and np.array_equal(wave, e_wave)
            assert all(np.array_equal(summ[f], e_summ[f]) for f in WAVE_SUMMARY_DTYPE.names)
        docs, _, _, _, _, st = util.check_wave_documents(s, names, part_off, None, rep_off, cur, out, out_len, B, weight=w, C=big,
                                                         send_ids=send_ids)
        e_docs, _, _, _ = s.plan_waves_json(names, part_off, None, rep_off, cur, out, out_len, B, weight=w)
        assert st.code == 0 and [bytes(d) for d in docs] == [bytes(d) for d in e_docs]
    cl = kab.synth.make_ragged_cluster(T=3000, N=300, max_partitions=128, seed=13, remove_frac=0.02)
    s, out, out_len, S = util.solved(cl)
    _check(s, cl.rep_off, cl.cur, out, out_len, 2, INT64_MAX, cl.all_broker_id)


@pytest.mark.gpu
@pytest.mark.parametrize("table", ["smem_lut", "global_lut", "bsearch", "state_in_smem", "state_in_global"])
def test_lookup_modes_and_chain_state(native_lib, table):
    """All three receiver lookup modes, and N + n_send on both sides of the chain's shared-memory limit (12 800 words of 16 bytes):
    6 400 + 6 400 in shared memory, 6 400 + 6 401 in global memory."""
    N = 6400 if table.startswith("state") else 50
    if table == "global_lut":
        ids, racks = util.table(1 + 700 * np.arange(N), 5)
    elif table == "bsearch":
        ids, racks = util.bsearch_table(N)
    else:
        ids, racks = util.table(np.arange(1, N + 1), 8)
    # the send table: the broker table and senders outside it (a drained set), n_send = N or N + 1 for the state cases
    extra = {"state_in_smem": 0, "state_in_global": 1}.get(table, 7)
    gone = np.arange(1, extra + 1) + int(ids.max())
    send_ids = np.concatenate([ids, gone]).astype(np.int32)
    s = kab.Solver(0)
    s.set_brokers(ids, racks)
    rng = np.random.default_rng(N + extra)
    Q = 20000
    leaders = np.concatenate([ids[-3:], gone]) if extra else ids[-3:]
    cur_lists = [[int(rng.choice(leaders if g % 4 == 0 else ids))] + [] for g in range(Q)]
    hot = ids[:5]
    new_lists = []
    for g, c in enumerate(cur_lists):
        pool = np.setdiff1d(hot if g % 3 == 0 else ids, c)
        new_lists.append([int(x) for x in rng.choice(pool, int(rng.integers(1, 4)), replace=False)])
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    for B, C, w in ((1, 1, None), (16, 5, None), (500, 700, rng.integers(0, 100, Q).astype(np.int64))):
        _check(s, rep_off, cur, out, out_len, B, C, send_ids, w)
    names, part_off = ["m%d" % t for t in range(40)], np.arange(41) * (Q // 40)
    util.check_wave_documents(s, names, part_off, None, rep_off, cur, out, out_len, 16, C=5, send_ids=send_ids)


@pytest.mark.gpu
def test_one_leader_is_fully_serial(native_lib):
    """Every moved row comes from broker 1, each to a receiver of its own: with C = 1 every row is a wave of its own, across the
    chain's chunks; the documents cross two radix passes."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))
    Q = 5000
    cur_lists = [[1]] * Q
    new_lists = [[1, 2 + g % 39] for g in range(Q)]
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists)
    wave, summ, st = _check(s, rep_off, cur, out, out_len, 10 ** 6, 1, [1])
    assert st.code == 0 and wave.tolist() == list(range(1, Q + 1)) and set(summ["max_broker_out_id"].tolist()) == {1}
    names, part_off = ["serial-%d" % t for t in range(7)], (np.arange(8) * Q) // 7
    docs, _, _, _, _, st = util.check_wave_documents(s, names, part_off, None, rep_off, cur, out, out_len, 10 ** 6, C=1, send_ids=[1])
    assert st.code == 0 and len(docs) == Q


def _raw(s, Q, rep_off, cur, stride, new_len, new, weight, B, n_send, send_id, C, wave, summary, send_summary, cap, n=None):
    st = kab.KaStatus()
    n = ctypes.c_int32(-7) if n is None else n
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = s._L.ka_plan_waves_send(s._h, Q, p(rep_off), p(cur), stride, p(new_len), p(new), p(weight), B, n_send, p(send_id), C, p(wave),
                                 ctypes.byref(n) if n is not False else None, p(summary), p(send_summary), cap, ctypes.byref(st))
    return rc, st, n


def _raw_json(s, T, part_off, rep_off, cur, stride, new_len, new, B, n_send, send_id, C, names, name_off, js, json_cap, doc_off, wave,
              summary, send_summary, cap):
    st = kab.KaStatus()
    n = ctypes.c_int32(-7)
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = s._L.ka_plan_waves_send_json(s._h, T, p(part_off), None, p(rep_off), p(cur), stride, p(new_len), p(new), None, B, n_send,
                                      p(send_id), C, p(names), p(name_off), p(js), json_cap, p(doc_off), p(wave), ctypes.byref(n),
                                      p(summary), p(send_summary), cap, ctypes.byref(st))
    return rc, st, n


@pytest.mark.gpu
def test_errors_and_buffers(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 21), 4))
    rng = np.random.default_rng(4)
    Q = 1000
    cur_lists, new_lists = util.random_wave_case(rng, Q, 20)
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    send = np.arange(1, 21, dtype=np.int32)
    wave, summ, ssum = np.zeros(Q, dtype=np.int32), np.zeros(Q, dtype=WAVE_SUMMARY_DTYPE), np.zeros((Q, 2), dtype=np.int64)
    keys = ("s", "Q", "rep_off", "cur", "stride", "new_len", "new", "weight", "B", "n_send", "send_id", "C", "wave", "summary",
            "send_summary", "cap")
    ok = (s, Q, rep_off, cur, 3, out_len, out, None, 2, 20, send, 3, wave, summ, ssum, Q)

    def call(n=None, **kw):
        a = dict(zip(keys, ok))
        a.update(kw)
        rc, st, n = _raw(*a.values(), n=n)
        assert rc == st.code
        if n is not False:
            assert rc == 0 or n.value == 0
        return rc, st.a, st.b

    assert call()[0] == 0
    # the checks of ka_plan_waves first, then the sender's
    assert call(stride=0, C=0)[0] == BAD and call(n=False)[0] == BAD and call(B=0, n_send=70000)[0] == BAD
    assert call(stride=9, new=np.full((Q, 9), -1, dtype=np.int32), C=0)[:2] == (LIMIT, 9)
    assert call(C=0)[0] == BAD and call(n_send=-1)[0] == BAD and call(send_id=None)[0] == BAD
    assert call(send_id=None, n_send=0, cap=0, summary=None, send_summary=None)[0] == BAD   # row 0.. have senders: device refusal
    assert call(send_summary=None)[0] == BAD and call(send_summary=None, summary=None, cap=0)[0] == 0
    unsorted = send.copy()
    unsorted[[4, 5]] = unsorted[[5, 4]]
    assert call(send_id=unsorted)[0] == BAD
    dup = send.copy()
    dup[7] = dup[6]
    assert call(send_id=dup)[0] == BAD
    many = np.arange(1, 65537, dtype=np.int32)
    assert call(n_send=65536, send_id=many)[:2] == (LIMIT, 65536)
    assert call(n_send=65535, send_id=many)[0] == 0
    # on the device: the lowest failing row, the new list before the sender
    for sids, rows, expect in ((send[send != 5], {}, None), (send, {300: [1, 99]}, (BAD, 300, 99))):
        o, ln = out.copy(), out_len.copy()
        for g, x in rows.items():
            o[g, :] = -1
            o[g, :len(x)] = x
            ln[g] = len(x)
        e = models.plan_waves(rep_off, cur, o, ln, s.broker_id, 2, send=(sids, 3))[2]
        assert e[0] == BAD and (expect is None or e == expect)
        assert call(new=o, new_len=ln, n_send=len(sids), send_id=sids) == e
    g = int(models.plan_waves(rep_off, cur, out, out_len, s.broker_id, 2, send=(send[send != 5], 3))[2][1])
    o, ln = out.copy(), out_len.copy()
    o[g, :] = -1
    o[g, :2] = [7, 7]
    ln[g] = 2
    assert call(new=o, new_len=ln, n_send=19, send_id=send[send != 5]) == (BAD, g, 7)   # its own new list comes first
    # a summary capacity below W
    e_wave, e_summ, _ = models.plan_waves(rep_off, cur, out, out_len, s.broker_id, 1, send=(send, 1))
    W = len(e_summ)
    assert W > 3
    few, few_s = np.zeros(3, dtype=WAVE_SUMMARY_DTYPE), np.zeros((3, 2), dtype=np.int64)
    rc, _, n = _raw(s, Q, rep_off, cur, 3, out_len, out, None, 1, 20, send, 1, wave, few, few_s, 3)
    assert rc == 0 and n.value == W and np.array_equal(wave, e_wave)
    assert [{f: int(x[f]) for f in WAVE_SUMMARY_DTYPE.names} | dict(max_broker_out=int(y[0]), max_broker_out_id=int(y[1]))
            for x, y in zip(few, few_s)] == e_summ[:3]
    # the documents: the sender checks after the text checks; the exact size succeeds, one byte less is KA_ERR_LIMIT
    T = 10
    topic_names = ["err-%d" % t for t in range(T)]
    names, name_off = kab.Solver.marshal_names(topic_names)
    part_off = np.arange(T + 1, dtype=np.int64) * 100
    cap = models.json_bound(topic_names, part_off, 3)
    js, doc_off = np.zeros(cap, dtype=np.uint8), np.zeros(Q + 1, dtype=np.int64)
    jok = dict(s=s, T=T, part_off=part_off, rep_off=rep_off, cur=cur, stride=3, new_len=out_len, new=out, B=2, n_send=20, send_id=send,
               C=3, names=names, name_off=name_off, js=js, json_cap=cap, doc_off=doc_off, wave=wave, summary=summ, send_summary=ssum,
               cap=Q)

    def jcall(**kw):
        a = dict(jok)
        a.update(kw)
        rc, st, n = _raw_json(*a.values())
        assert rc == st.code and (rc == 0 or n.value == 0)
        return rc, st.a, st.b

    assert jcall(js=None, C=0)[0] == BAD and jcall(doc_off=None, n_send=70000)[0] == BAD
    assert jcall(C=0)[0] == BAD and jcall(n_send=70000, send_id=np.arange(70000, dtype=np.int32))[:2] == (LIMIT, 70000)
    e_docs = models.wave_documents(topic_names, part_off, None, rep_off, cur, out, out_len, s.broker_id, 2, send=(send, 3))[0]
    size = sum(len(d) for d in e_docs)
    assert 0 < size <= cap
    assert jcall(json_cap=size - 1)[:2] == (LIMIT, size - 1)
    js[:] = 0
    assert jcall(json_cap=size)[0] == 0 and bytes(js[:size]) == b"".join(e_docs) and not js[size:].any()
    assert doc_off[:len(e_docs) + 1].tolist() == np.concatenate([[0], np.cumsum([len(d) for d in e_docs])]).tolist()
    assert jcall(n_send=19, send_id=send[send != 5])[0] == BAD


@pytest.mark.gpu
def test_context_is_untouched_and_launches_are_fixed(native_lib):
    cl = kab.synth.make_ragged_cluster(T=3000, N=400, max_partitions=128, seed=21, remove_frac=0.02)
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    args = (cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    out, out_len, _ = s.solve_ragged(*args)
    before = (s.counters(), s.last_order_plan(), s.last_stage_plan())
    n0 = s.launch_count()
    _, summ, st = s.plan_waves(cl.rep_off, cl.cur, out, out_len, 2, max_broker_out=3, send_brokers=cl.all_broker_id)
    assert st.code == 0 and len(summ) > 1 and s.launch_count() - n0 == 9
    docs, _, _, st = s.plan_waves_json(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, 2, max_broker_out=3,
                                       send_brokers=cl.all_broker_id)
    assert st.code == 0 and len(docs) > 1
    assert np.array_equal(s.counters(), before[0]) and (s.last_order_plan(), s.last_stage_plan()) == before[1:]
    again, again_len, _ = s.solve_ragged(*args)
    fresh = kab.Solver(0)
    fresh.set_brokers(cl.broker_id, cl.rack_index)
    fresh.solve_ragged(*args)
    f_out, f_len, _ = fresh.solve_ragged(*args)
    assert np.array_equal(again, f_out) and np.array_equal(again_len, f_len)

    # the plan's 9 whatever Q, W and n_send; the documents add 3 per radix pass (8 bits of W each) and 3, none when W = 0
    def launches(Q, same=False, n_send=1):
        rep_off, cur = util.cur_lists([[1]] * Q)
        o, ln = util.rows([[1 if same else 2]] * Q)
        send_ids = np.arange(1, n_send + 1, dtype=np.int32)
        n0 = s.launch_count()
        _, _, st = s.plan_waves(rep_off, cur, o, ln, 10 ** 9, max_broker_out=1, send_brokers=send_ids)
        n1 = s.launch_count()
        docs, _, _, st2 = s.plan_waves_json(["t"], [0, Q], None, rep_off, cur, o, ln, 10 ** 9, max_broker_out=1, send_brokers=send_ids)
        assert st.code == st2.code == 0 and len(docs) == (0 if same else Q)
        return n1 - n0, s.launch_count() - n1

    assert launches(100) == launches(255, n_send=30000) == (9, 9 + 3 + 3)
    assert launches(256) == launches(3000, n_send=12000) == (9, 9 + 6 + 3)
    assert launches(500, same=True) == (9, 9)


@pytest.mark.gpu
def test_cpp_host_mirror(native_lib):
    """host/test_waves_send.cpp: the SendBudget overloads of planWaves / planWavesJson keep both budgets per wave, agree with each
    other, and with a huge send budget equal the calls without one."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_WAVES_SEND_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
