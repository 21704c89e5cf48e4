"""ka_plan_waves: a reassignment cut into waves in which no broker receives more than a budget. `models.plan_waves` restates the
rule of include/kassign.h as a plain loop; every wave, summary and W of the device must equal it. The CPU tests pin the model on
hand-worked cases and its invariants on random inputs, and what Solver.plan_waves hands the C ABI."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SUMMARY_DTYPE
from tests import models, util

FIELDS = WAVE_SUMMARY_DTYPE.names
INT64_MAX = np.iinfo(np.int64).max
BAD, LIMIT = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT


def _model(cur_lists, new_lists, B, weight=None, ids=range(1, 100)):
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists)
    return models.plan_waves(rep_off, cur, out, out_len, np.asarray(list(ids)), B, weight)


# ---- CPU -----------------------------------------------------------------------------------------------------------------

def test_symbol_is_exported_and_declared(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    assert hasattr(raw, "ka_plan_waves")
    res, args = _native.SYMBOLS["ka_plan_waves"]
    assert res is ctypes.c_int32 and len(args) == 14
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kassign.h")).read()
    assert "int32_t ka_plan_waves(ka_ctx* ctx, int64_t Q," in header and "} ka_wave_summary;" in header
    assert ctypes.sizeof(_native.KaWaveSummary) == 40 and WAVE_SUMMARY_DTYPE.itemsize == 40


def test_without_a_context_is_no_device(native_lib):
    L = native_lib
    st = kab.KaStatus()
    n = ctypes.c_int32(5)
    assert L.ka_plan_waves(None, 0, None, None, 1, None, None, None, 1, None, ctypes.byref(n), None, 0,
                           ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE
    assert st.code == _native.KA_ERR_NO_DEVICE and n.value == 0
    assert L.ka_plan_waves(None, 0, None, None, 1, None, None, None, 1, None, ctypes.byref(n), None, 0, None) == BAD


@pytest.mark.parametrize("W", [3, 100])
def test_plan_waves_marshals_its_arguments(W):
    lib = util.FakeWaveLib(W)
    s = util.fake_solver(lib)
    out, out_len = util.rows([[1, 2], [3], [4, 5, 6], []])
    rep_off, cur = util.cur_lists([[1], [2, 3], [4], [7, 8]])
    weight = np.array([5, 0, 7, 1], dtype=np.int64)
    wave, summ, st = s.plan_waves(rep_off.astype(np.int32), cur.astype(np.int64), out, out_len, 9, weight=weight)
    assert st.code == 0
    first = lib.calls[0]
    assert first["Q"] == 4 and first["stride"] == 3 and first["B"] == 9 and first["cap"] == min(4, kab.Solver.WAVE_SUMMARY_CAP)
    assert np.array_equal(first["rep_off"], rep_off) and np.array_equal(first["cur"], cur)
    assert np.array_equal(first["new_len"], out_len) and np.array_equal(first["new_broker"], out.ravel())
    assert np.array_equal(first["weight"], weight) and first["wave"]
    assert np.array_equal(wave, 1 + np.arange(4) % W)
    assert summ.dtype == WAVE_SUMMARY_DTYPE and len(summ) == W
    assert [list(x) for x in summ] == [[v * 10 + f for f in range(5)] for v in range(W)]
    if W > first["cap"]:   # the rest of the summaries in a second call of capacity W (a fake plan: W beyond Q)
        assert len(lib.calls) == 2 and lib.calls[1]["cap"] == W
    else:
        assert len(lib.calls) == 1
    s.plan_waves(rep_off, cur, out, out_len, 1)
    assert lib.calls[-1]["weight"] is None


def test_model_hand_worked_unit_budget():
    cur = [[1, 2], [1, 2], [1], [2], [1, 2], [1, 2], [5], [1], [2]]
    new = [[1, 3], [3, 4], [3], [4], [2, 1], [1, 2], [4, 5], [3, 4], [3]]
    wave, summ, st = _model(cur, new, 2)
    assert st == (0, 0, 0)
    assert wave.tolist() == [1, 1, 2, 1, 1, 0, 2, 2, 3]
    assert summ == [dict(rows=4, rows_moved=3, replicas_added=4, max_broker_in=2, max_broker_in_id=3),
                    dict(rows=3, rows_moved=3, replicas_added=4, max_broker_in=2, max_broker_in_id=3),
                    dict(rows=1, rows_moved=1, replicas_added=1, max_broker_in=1, max_broker_in_id=3)]


def test_model_hand_worked_weights():
    # a row heavier than B opens its broker's wave alone; zero weights fit anywhere
    wave, summ, _ = _model([[1], [1], [1], [1]], [[2], [2], [2], [3]], 3, weight=[5, 1, 0, 0])
    assert wave.tolist() == [1, 2, 2, 1]
    assert summ == [dict(rows=2, rows_moved=2, replicas_added=5, max_broker_in=5, max_broker_in_id=2),
                    dict(rows=2, rows_moved=2, replicas_added=1, max_broker_in=1, max_broker_in_id=2)]
    wave, summ, _ = _model([[1]], [[2]], 1, weight=[0])
    assert wave.tolist() == [1] and summ == [dict(rows=1, rows_moved=1, replicas_added=0, max_broker_in=0, max_broker_in_id=-1)]
    # a row waits for the busiest of its receivers; drops and reorders only are wave 1
    wave, _, _ = _model([[1], [1], [1], [1, 2], [1, 2]], [[2], [2], [2, 3], [1], [2, 1]], 1)
    assert wave.tolist() == [1, 2, 3, 1, 1]
    # nothing changed, and no rows
    assert _model([[1, 2]], [[1, 2]], 1)[1] == [] and _model([], [], 1)[1] == []
    # errors at the first position of the lowest failing row
    assert _model([[1], [1], [1]], [[2], [3, 3], [200]], 1)[2] == (BAD, 1, 3)
    assert _model([[1], [1]], [[2], [200]], 1)[2] == (BAD, 1, 200)
    assert _model([[200]], [[200]], 1)[2] == (0, 0, 0)   # a kept broker need not be in the table


def check_invariants(cur_lists, new_lists, wave, summ, B, weight, ids):
    """The budget rule, contiguous non-empty waves, and the per-wave replicas_added summing to ka_move_summary's."""
    W = len(summ)
    assert W == (int(wave.max()) if len(wave) else 0)
    assert all(s["rows"] > 0 for s in summ) and set(wave.tolist()) - {0} == set(range(1, W + 1))
    w = np.ones(len(wave), dtype=np.int64) if weight is None else np.asarray(weight, dtype=np.int64)
    inb = {}
    for g, (old, new) in enumerate(zip(cur_lists, new_lists)):
        assert (wave[g] == 0) == (old == new)
        for b in new:
            if b not in old:
                inb.setdefault((int(wave[g]), b), []).append(int(w[g]))
    for ws in inb.values():   # beyond B only through one heavier row, with nothing else but zero weights
        assert sum(ws) <= B or sum(x > 0 for x in ws) == 1, ws
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    e = models.move_summary(out, out_len, rep_off, cur, np.asarray(ids, dtype=np.int64), weight)[0]
    assert sum(s["replicas_added"] for s in summ) == e["replicas_added"]
    if w.sum() <= B:
        assert W <= 1


@pytest.mark.parametrize("seed", range(6))
def test_model_invariants(seed):
    rng = np.random.default_rng(seed)
    ids = np.arange(1, 13)
    cur_lists, new_lists = util.random_wave_case(rng, 300, 12)
    for B, weight in ((1, None), (4, None), (10 ** 6, None), (50, rng.integers(0, 40, 300)), (30, rng.integers(0, 80, 300))):
        wave, summ, st = _model(cur_lists, new_lists, B, weight, ids)
        assert st == (0, 0, 0)
        check_invariants(cur_lists, new_lists, wave, summ, B, weight, ids)


# ---- GPU -----------------------------------------------------------------------------------------------------------------

def _check(s, rep_off, cur, out, out_len, B, weight=None, ids=None):
    """plan_waves against the model, every field. Returns (wave, summary, status)."""
    ids = s.broker_id if ids is None else ids
    wave, summ, st = s.plan_waves(rep_off, cur, out, out_len, B, weight=weight)
    e_wave, e_summ, e_st = models.plan_waves(rep_off, cur, out, out_len, ids, B, weight)
    assert (st.code, st.a, st.b) == e_st, ((st.code, st.a, st.b), e_st)
    if st.code == 0:
        assert np.array_equal(wave, e_wave), np.nonzero(wave != e_wave)[0][:10]
        assert [util.record_of(x, FIELDS) for x in summ] == e_summ
    return wave, summ, st


@pytest.mark.gpu
@pytest.mark.parametrize("remove", [0.0, 0.02, 0.2])
def test_solve_rows(native_lib, remove):
    cl = kab.synth.make_ragged_cluster(T=4000, N=400, max_partitions=128, seed=7, remove_frac=remove)
    s, out, out_len, S = util.solved(cl)
    rng = np.random.default_rng(3)
    Q = len(out_len)
    weight = rng.integers(0, 1 << 30, Q).astype(np.int64)
    for B, w in ((1, None), (3, None), (200, None), (INT64_MAX, None), (1, weight), (1 << 32, weight), (INT64_MAX, weight)):
        wave, summ, st = _check(s, cl.rep_off, cl.cur, out, out_len, B, w)
        assert st.code == 0
        if B == INT64_MAX:
            assert len(summ) <= 1
    # the waves add up to what ka_score_candidates reports for the same rows
    score, sst = s.score_ragged_candidates([(cl.broker_id, cl.rack_index)], cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off,
                                           cl.cur, -1, out_stride=S, weight=weight)
    assert sst[0].code == 0
    _, summ, _ = s.plan_waves(cl.rep_off, cl.cur, out, out_len, 1 << 32, weight=weight)
    assert int(summ["replicas_added"].sum()) == int(score[0]["replicas_added"]) > 0
    assert int(summ["rows"].sum()) == int(score[0]["rows_changed"])


@pytest.mark.gpu
def test_growing_rf_rows_of_4_to_8(native_lib):
    for drf, shape in ((5, dict(N=60, seed=16)), (8, dict(N=200, seed=19, max_partitions=64))):   # no racks: RF 8 is assignable
        cl = kab.synth.make_ragged_cluster(T=600, R=6, rack_frac=0.0, desired_rf=drf, **shape)
        s, out, out_len, S = util.solved(cl, drf)
        assert S == drf and out_len.max() == drf
        for B in (1, 7, 1000):
            _check(s, cl.rep_off, cl.cur, out, out_len, B)
            _check(s, cl.rep_off, cl.cur, out, out_len, B * 1000, np.arange(len(out_len), dtype=np.int64) % 2000)


@pytest.mark.gpu
def test_hand_built_rows(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))

    def run(cur_lists, new_lists, B, weight=None, stride=None):
        rep_off, cur = util.cur_lists(cur_lists)
        out, out_len = util.rows(new_lists, stride)
        return _check(s, rep_off, cur, out, out_len, B, None if weight is None else np.asarray(weight, dtype=np.int64))

    assert run([[1, 2], [3, 4]], [[2, 1], [4, 3]], 1)[0].tolist() == [1, 1]                   # reorder only
    assert run([[1, 2, 3], [4, 5]], [[1], []], 1)[0].tolist() == [1, 1]                      # drops only
    assert run([[1], [1], [1], [1]], [[2], [2], [2], [3]], 3, [5, 1, 0, 0])[0].tolist() == [1, 2, 2, 1]   # heavier, zero
    assert run([[3, 3], [99, 1], [], [100]], [[3, 5], [1, 6], [7, 8], []], 1)[0].tolist() == [1, 1, 1, 1]  # dup / dead / empty
    assert len(run([], [], 1)[1]) == 0                                                         # Q = 0
    wave, summ, _ = run([[1, 2]] * 50, [[1, 2]] * 50, 1)                                        # nothing changed
    assert not wave.any() and len(summ) == 0
    wave, summ, _ = run([[1]] * 5000, [[2]] * 5000, 1)                                          # fully serial, across chunks
    assert wave.tolist() == list(range(1, 5001)) and len(summ) == 5000
    eight = [[int(x) for x in 1 + (np.arange(8) + g) % 40] for g in range(3000)]                # 8 receivers per row
    run([[]] * 3000, eight, 1)
    run([[]] * 3000, eight, 5, np.arange(3000) % 4)
    rng = np.random.default_rng(2)
    cur_lists, new_lists = util.random_wave_case(rng, 20000, 40, 8)
    for B in (1, 2, 9):
        run(cur_lists, new_lists, B, stride=8)
        run(cur_lists, new_lists, B * 10, rng.integers(0, 30, 20000), stride=8)


@pytest.mark.gpu
@pytest.mark.parametrize("table", ["smem_lut", "global_lut", "bsearch", "state_in_smem", "state_in_global"])
def test_lookup_modes_and_chain_state(native_lib, table):
    N = dict(smem_lut=50, global_lut=50, bsearch=50, state_in_smem=12800, state_in_global=12801)[table]
    if table == "global_lut":
        ids, racks = util.table(1 + 700 * np.arange(N), 5)
    elif table == "bsearch":
        ids, racks = util.bsearch_table(N)
    else:
        ids, racks = util.table(np.arange(1, N + 1), 8)
    s = kab.Solver(0)
    s.set_brokers(ids, racks)
    rng = np.random.default_rng(N)
    Q = 30000
    cur_lists = [[int(x) for x in rng.choice(ids, int(rng.integers(0, 4)), replace=False)] for _ in range(Q)]
    hot = ids[-5:]   # receivers crowd on a few brokers (the chain's conflicts)
    new_lists = [[int(x) for x in rng.choice(hot if g % 3 == 0 else ids, int(rng.integers(1, 4)), replace=False)] for g in range(Q)]
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    for B, w in ((1, None), (16, None), (500, rng.integers(0, 100, Q).astype(np.int64))):
        _check(s, rep_off, cur, out, out_len, B, w)


def _raw(s, Q, rep_off, cur, stride, new_len, new, weight, B, wave, summary, cap, n=None):
    st = kab.KaStatus()
    n = ctypes.c_int32(-7) if n is None else n
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = s._L.ka_plan_waves(s._h, Q, p(rep_off), p(cur), stride, p(new_len), p(new), p(weight), B, p(wave),
                            ctypes.byref(n) if n is not False else None, p(summary), cap, ctypes.byref(st))
    return rc, st, n


@pytest.mark.gpu
def test_errors(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 21), 4))
    rng = np.random.default_rng(4)
    cur_lists, new_lists = util.random_wave_case(rng, 1000, 20)
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    wave, summ = np.zeros(1000, dtype=np.int32), np.zeros(8, dtype=WAVE_SUMMARY_DTYPE)
    ok = (s, 1000, rep_off, cur, 3, out_len, out, None, 2, wave, summ, 8)

    def call(n=None, **kw):
        a = dict(zip(("s", "Q", "rep_off", "cur", "stride", "new_len", "new", "weight", "B", "wave", "summary", "cap"), ok))
        a.update(kw)
        rc, st, n = _raw(*a.values(), n=n)
        assert rc == st.code
        if n is not False:
            assert rc == 0 or n.value == 0
        return rc, st.a, st.b

    assert call()[0] == 0
    assert call(Q=-1)[0] == BAD and call(stride=0)[0] == BAD and call(n=False)[0] == BAD and call(cap=-1)[0] == BAD
    assert call(summary=None)[0] == BAD and call(B=0)[0] == BAD
    bad_off = rep_off.copy()
    bad_off[500] = bad_off[501] + 1
    assert call(rep_off=bad_off)[0] == BAD
    shifted = rep_off + 1
    assert call(rep_off=shifted)[0] == BAD
    wide = np.full((1000, 9), -1, dtype=np.int32)
    assert call(stride=9, new=wide)[:2] == (LIMIT, 9)
    long_len = out_len.copy()
    long_len[[700, 300]] = [4, -1]
    assert call(new_len=long_len)[:2] == (BAD, 300)
    neg = np.ones(1000, dtype=np.int64)
    neg[10] = -1
    assert call(weight=neg)[0] == BAD
    edge = np.ones(1000, dtype=np.int64)
    edge[0] = INT64_MAX // 8 - 999
    assert call(weight=edge)[0] == 0
    edge[1] += 1
    assert call(weight=edge)[0] == LIMIT
    # on the device the lowest failing row wins, with the broker at the first failing position of its list
    for rows, expect in (({700: [5, 5], 300: [1, 99]}, (BAD, 300, 99)), ({700: [1, 99], 300: [2, 6, 2]}, (BAD, 300, 2)),
                         ({999: [21]}, (BAD, 999, 21)), ({0: [3, 3]}, (BAD, 0, 3))):
        o, ln = out.copy(), out_len.copy()
        for g, x in rows.items():
            o[g, :] = -1
            o[g, :len(x)] = x
            ln[g] = len(x)
        assert call(new=o, new_len=ln) == expect
        e = models.plan_waves(rep_off, cur, o, ln, s.broker_id, 2)[2]
        assert e == expect
    # Q == 0 and a cap below W
    assert call(Q=0)[0] == 0
    n = ctypes.c_int32(0)
    _check(s, rep_off, cur, out, out_len, 1)
    e_wave, e_summ, _ = models.plan_waves(rep_off, cur, out, out_len, s.broker_id, 1)
    W = len(e_summ)
    assert W > 3
    few = np.zeros(3, dtype=WAVE_SUMMARY_DTYPE)
    rc, _, n = _raw(s, 1000, rep_off, cur, 3, out_len, out, None, 1, wave, few, 3)
    assert rc == 0 and n.value == W and [util.record_of(x, FIELDS) for x in few] == e_summ[:3] and np.array_equal(wave, e_wave)
    rc, _, n = _raw(s, 1000, rep_off, cur, 3, out_len, out, None, 1, None, None, 0)
    assert rc == 0 and n.value == W


@pytest.mark.gpu
def test_context_is_untouched_and_launches_are_fixed(native_lib):
    cl = kab.synth.make_ragged_cluster(T=3000, N=400, max_partitions=128, seed=21, remove_frac=0.02)
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    args = (cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    out, out_len, _ = s.solve_ragged(*args)
    before = (s.counters(), s.last_order_plan(), s.last_stage_plan())
    n0 = s.launch_count()
    rc, _, n = _raw(s, len(out_len), cl.rep_off, cl.cur, 3, out_len, out, None, 2, np.zeros(len(out_len), dtype=np.int32), None, 0)
    n1 = s.launch_count()
    assert rc == 0 and n.value > 1
    assert np.array_equal(s.counters(), before[0]) and (s.last_order_plan(), s.last_stage_plan()) == before[1:]
    # a following solve gives the rows it gives without the call
    again, again_len, _ = s.solve_ragged(*args)
    ref = kab.Solver(0)
    ref.set_brokers(cl.broker_id, cl.rack_index)
    ref.solve_ragged(*args)
    ref_out, ref_len, _ = ref.solve_ragged(*args)
    assert np.array_equal(again, ref_out) and np.array_equal(again_len, ref_len)
    # the same launches at another size
    big = kab.synth.make_ragged_cluster(T=40000, N=400, max_partitions=128, seed=22, remove_frac=0.2)
    s2, bout, blen, _ = util.solved(big)
    m0 = s2.launch_count()   # one C call each: Solver.plan_waves makes a second one for a plan of many waves
    rc, _, n = _raw(s2, len(blen), big.rep_off, big.cur, 3, blen, bout, None, 1, np.zeros(len(blen), dtype=np.int32), None, 0)
    assert rc == 0 and n.value > 64 and s2.launch_count() - m0 == n1 - n0


@pytest.mark.gpu
def test_plans_on_its_own_device(native_lib):
    """A Solver plans on its context's device whatever device is current: here another Solver's device 0."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    cl = kab.synth.make_ragged_cluster(T=2000, N=200, max_partitions=64, seed=23, remove_frac=0.02)
    s = kab.Solver(1)
    s.set_brokers(cl.broker_id, cl.rack_index)
    out, out_len, st = s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    assert st.code == 0
    other = kab.Solver(0)   # leaves device 0 current
    other.set_brokers(cl.broker_id, cl.rack_index)
    weight = np.random.default_rng(5).integers(0, 1000, len(out_len)).astype(np.int64)
    for B, w in ((1, None), (2000, weight)):
        _, summ, st = _check(s, cl.rep_off, cl.cur, out, out_len, B, w)
        assert st.code == 0 and len(summ) > 0


@pytest.mark.gpu
def test_cpp_host_mirror(native_lib):
    """host/test_waves.cpp: every wave's document of KafkaTopicAssigner::planWaves, concatenated over the waves, holds exactly the
    changed partitions of newAssignmentJson(solveTopics(...))."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_WAVES_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
