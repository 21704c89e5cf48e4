"""KA_WAVE_FIRST_FIT: every plan call of a Context under the first-fit wave rule, each row in the earliest wave where its
receivers and its sender still have room. `fit_models.plan_waves` restates the rule of include/kassign.h; the
CPU tests check it against a search from wave 1 and its stated bounds, and what Solver.set_wave_rule hands the C ABI; every
wave, summary, document and status of the device must equal the model."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SEND_SUMMARY_DTYPE, WAVE_SUMMARY_DTYPE
from tests import fit_models, models, usage_models, util

BAD, LIMIT, NO_DEVICE = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT, _native.KA_ERR_NO_DEVICE
INT64_MAX = np.iinfo(np.int64).max


def _model(cur_lists, new_lists, B, weight=None, ids=range(1, 100), send=None, first_fit=True):
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists)
    plan = fit_models.plan_waves if first_fit else models.plan_waves
    return plan(rep_off, cur, out, out_len, np.asarray(list(ids)), B, weight, send)


def check_first_fit(cur_lists, new_lists, wave, summ, B, weight=None, send=None):
    """Every invariant include/kassign.h states for a first-fit plan: non-empty waves 1..W, every row's wave the smallest that
    fits beside the earlier rows (a search from wave 1), so every budget holds, and W <= Wb."""
    W = len(summ)
    assert W == (int(wave.max()) if len(wave) else 0)
    assert all(s["rows"] > 0 for s in summ) and set(wave.tolist()) - {0} == set(range(1, W + 1))
    C = None if send is None else send[1]
    inb, outb = {}, {}
    moved = fit_models.moved(cur_lists, new_lists, weight, send)
    for g, recv, w, s in moved:
        a = w * len(recv)

        def fits(v):
            return all(inb.get((b, v), 0) == 0 or inb[(b, v)] + w <= B for b in recv) and \
                (s is None or outb.get((s, v), 0) == 0 or outb[(s, v)] + a <= C)
        v = 1
        while not fits(v):
            v += 1
        assert wave[g] == v, (g, int(wave[g]), v)
        for b in recv:
            inb[(b, v)] = inb.get((b, v), 0) + w
        if s is not None:
            outb[(s, v)] = outb.get((s, v), 0) + a
    assert W <= max(fit_models.bound(moved), 1 if any(o != n for o, n in zip(cur_lists, new_lists)) else 0)
    if weight is None:   # unit weights: no rule can use fewer waves than the busiest receiver needs
        R = {}
        for _, recv, _, _ in moved:
            for b in recv:
                R[b] = R.get(b, 0) + 1
        assert W >= max([-(-r // B) for r in R.values()] + [0])


# ---- CPU -----------------------------------------------------------------------------------------------------------------

def test_symbols_are_exported_and_declared(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kassign.h")).read()
    for name, nargs in (("ka_ctx_set_wave_rule", 2), ("ka_ctx_wave_rule", 1)):
        assert hasattr(raw, name)
        res, args = _native.SYMBOLS[name]
        assert res is ctypes.c_int32 and len(args) == nargs
    assert "int32_t ka_ctx_set_wave_rule(ka_ctx* ctx, int32_t rule);" in header
    assert "int32_t ka_ctx_wave_rule(ka_ctx* ctx);" in header
    assert "KA_WAVE_GREEDY = 0," in header and "KA_WAVE_FIRST_FIT = 1" in header
    assert (_native.KA_WAVE_GREEDY, _native.KA_WAVE_FIRST_FIT) == (0, 1)


def test_without_a_context_is_no_device(native_lib):
    assert native_lib.ka_ctx_set_wave_rule(None, 1) == NO_DEVICE
    assert native_lib.ka_ctx_wave_rule(None) == NO_DEVICE


class _FakeRuleLib:
    def __init__(self):
        self.rule, self.calls = 0, []

    def ka_ctx_set_wave_rule(self, h, rule):
        self.calls.append(rule)
        if rule not in (0, 1):
            return BAD
        self.rule = rule
        return 0

    def ka_ctx_wave_rule(self, h):
        return self.rule


def test_set_wave_rule_marshals_its_argument():
    lib = _FakeRuleLib()
    s = util.fake_solver(lib)
    assert s.wave_rule == "greedy"
    s.set_wave_rule("first_fit")
    assert lib.calls == [1] and s.wave_rule == "first_fit"
    s.set_wave_rule("greedy")
    assert lib.calls == [1, 0] and s.wave_rule == "greedy"
    with pytest.raises(ValueError):
        s.set_wave_rule("best_fit")
    assert lib.calls == [1, 0]


def test_model_fills_the_hole_greedy_leaves():
    # row 1 pushes broker 3 into wave 2 with broker 2; greedy then keeps broker 3 out of wave 1, first fit puts row 2 there
    cur, new = [[1], [1], [1]], [[2], [2, 3], [3]]
    g_wave, g_summ, _ = _model(cur, new, 1, first_fit=False)
    f_wave, f_summ, st = _model(cur, new, 1)
    assert st == (0, 0, 0)
    assert g_wave.tolist() == [1, 2, 3] and f_wave.tolist() == [1, 2, 1]
    assert f_summ == [dict(rows=2, rows_moved=2, replicas_added=2, max_broker_in=1, max_broker_in_id=2),
                      dict(rows=1, rows_moved=1, replicas_added=2, max_broker_in=1, max_broker_in_id=2)]
    # the sender is one more bucket: the leader 1 sends once per wave, and the row led by 5 drops back into wave 1
    cur, new = [[1], [1], [5], [5]], [[2], [3], [4], [2]]
    f_wave, f_summ, _ = _model(cur, new, 1, send=([1, 5], 1))
    assert f_wave.tolist() == [1, 2, 1, 2]
    assert f_summ[0]["max_broker_out"] == 1 and f_summ[1]["max_broker_out_id"] == 1
    g_wave, _, _ = _model(cur, new, 1, send=([1, 5], 1), first_fit=False)
    assert g_wave.tolist() == [1, 2, 1, 2]


def test_model_hand_worked_weights():
    # a row heavier than B is alone in its bucket; zero weights fit anywhere, from wave 1
    wave, summ, _ = _model([[1]] * 5, [[2]] * 5, 3, weight=[5, 1, 4, 2, 0])
    assert wave.tolist() == [1, 2, 3, 2, 2]
    assert [s["max_broker_in"] for s in summ] == [5, 3, 4]
    wave, _, _ = _model([[1]] * 3, [[2]] * 3, 3, weight=[5, 0, 0])
    assert wave.tolist() == [1, 2, 2]
    # errors are the greedy rule's
    assert _model([[1], [1], [1]], [[2], [3, 3], [200]], 1)[2] == (BAD, 1, 3)
    assert _model([[1], [1]], [[2], [3]], 1, send=([2], 1))[2] == (BAD, 0, 1)


@pytest.mark.parametrize("seed", range(6))
def test_model_invariants(seed):
    rng = np.random.default_rng(seed)
    ids = np.arange(1, 13)
    cur_lists, new_lists = util.random_wave_case(rng, 300, 12)
    for B, weight in ((1, None), (4, None), (10 ** 6, None), (50, rng.integers(0, 40, 300)), (30, rng.integers(0, 80, 300))):
        for send in (None, (list(ids), 3 * B)):
            wave, summ, st = _model(cur_lists, new_lists, B, weight, ids, send)
            assert st == (0, 0, 0)
            check_first_fit(cur_lists, new_lists, wave, summ, B, weight, send)
            g_summ = _model(cur_lists, new_lists, B, weight, ids, send, first_fit=False)[1]
            assert sum(s["replicas_added"] for s in summ) == sum(s["replicas_added"] for s in g_summ)


@pytest.mark.parametrize("seed", range(4))
def test_model_equals_greedy_without_repeats(seed):
    """No broker receives two moved rows and no leader sends two: the two rules agree."""
    rng = np.random.default_rng(40 + seed)
    brokers = [int(x) for x in rng.permutation(np.arange(1, 400))]
    cur_lists, new_lists = [], []
    for g in range(60):
        leader = brokers.pop()
        recv = [brokers.pop() for _ in range(int(rng.integers(1, 4)))]
        cur_lists.append([leader])
        new_lists.append([leader] + recv if g % 2 else recv)
    cur_lists += [[5000], [5001, 5002]]
    new_lists += [[5000], [5002]]
    ids = sorted(set(b for x in new_lists for b in x))
    for B, weight in ((1, None), (3, rng.integers(1, 9, 62))):
        for send in (None, (sorted(set(x[0] for x in cur_lists)), 2)):
            f = _model(cur_lists, new_lists, B, weight, ids, send)
            g = _model(cur_lists, new_lists, B, weight, ids, send, first_fit=False)
            assert np.array_equal(f[0], g[0]) and f[1] == g[1]


# ---- GPU -----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("remove", [0.0, 0.02])
def test_solve_rows(native_lib, remove):
    cl = kab.synth.make_ragged_cluster(T=4000, N=400, max_partitions=128, seed=7, remove_frac=remove)
    s, out, out_len, S = util.solved(cl)
    Q = len(out_len)
    weight = np.random.default_rng(3).integers(0, 1 << 30, Q).astype(np.int64)
    mean = int(weight.mean())
    for B, w in ((1, None), (3, None), (INT64_MAX, None), (16 * mean, weight), (1, weight)):
        for C in (None, min(2 * B, INT64_MAX) if w is None else 16 * mean):
            wave, summ, st = util.check_plan(s, cl.rep_off, cl.cur, out, out_len, B, w, cl.all_broker_id, C)
            assert st.code == 0 and len(summ) > 0
            s.set_wave_rule("greedy")
            g_wave, g_summ, _ = s.plan_waves(cl.rep_off, cl.cur, out, out_len, B, weight=w,
                                              **({} if C is None else dict(max_broker_out=C, send_brokers=cl.all_broker_id)))
            assert int(summ["replicas_added"].sum()) == int(g_summ["replicas_added"].sum())


@pytest.mark.gpu
@pytest.mark.parametrize("table", ["smem_lut", "global_lut", "bsearch", "state_in_smem", "state_in_global"])
def test_lookup_modes_and_claim_state(native_lib, table):
    """The chain keeps a claim and a hint word per broker and sender (8 bytes): shared memory up to 25 600 of them."""
    N = dict(smem_lut=50, global_lut=50, bsearch=50, state_in_smem=25600, state_in_global=25601)[table]
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
    every = 3 if N <= 51 else 50
    new_lists = [[int(x) for x in rng.choice(hot if g % every == 0 else ids, int(rng.integers(1, 4)), replace=False)]
                 for g in range(Q)]
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    for B, w in ((1, None), (16, None), (500, rng.integers(0, 100, Q).astype(np.int64))):
        util.check_plan(s, rep_off, cur, out, out_len, B, w)
    # with a sender part: the send table is the brokers, then padded with ids no row names so that the words of brokers and
    # senders leave shared memory (fewer rows: the load table grows with the senders)
    for pad, q in ((0, Q), (25600, 3000)):
        send_ids = np.union1d(ids, 10 ** 8 + np.arange(pad)).astype(np.int32)
        rep_off, cur = util.cur_lists(cur_lists[:q])
        out, out_len = util.rows(new_lists[:q], 3)
        util.check_plan(s, rep_off, cur, out, out_len, 4, None, send_ids, 6)


@pytest.mark.gpu
def test_hand_built_rows(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))

    def run(cur_lists, new_lists, B, weight=None, stride=None):
        rep_off, cur = util.cur_lists(cur_lists)
        out, out_len = util.rows(new_lists, stride)
        return util.check_plan(s, rep_off, cur, out, out_len, B, None if weight is None else np.asarray(weight, dtype=np.int64))

    assert run([[1], [1], [1]], [[2], [2, 3], [3]], 1)[0].tolist() == [1, 2, 1]                 # the hole greedy leaves
    assert run([[1]] * 5, [[2]] * 5, 3, [5, 1, 4, 2, 0])[0].tolist() == [1, 2, 3, 2, 2]          # heavier, zero
    assert run([[3, 3], [99, 1], [], [100]], [[3, 5], [1, 6], [7, 8], []], 1)[0].tolist() == [1, 1, 1, 1]  # dup / dead / empty
    assert len(run([], [], 1)[1]) == 0                                                           # Q = 0
    wave, summ, _ = run([[1, 2]] * 50, [[2, 1]] * 50, 1)                                          # reorders only
    assert wave.tolist() == [1] * 50 and len(summ) == 1
    wave, summ, _ = run([[1]] * 5000, [[2]] * 5000, 1)                                            # fully serial, across chunks
    assert wave.tolist() == list(range(1, 5001)) and len(summ) == 5000
    eight = [[int(x) for x in 1 + (np.arange(8) + g) % 40] for g in range(3000)]                  # 8 receivers per row
    run([[]] * 3000, eight, 1)
    run([[]] * 3000, eight, 5, np.arange(3000) % 4)
    rng = np.random.default_rng(2)
    cur_lists, new_lists = util.random_wave_case(rng, 20000, 40, 8)
    for B in (1, 2, 9):
        wave, summ, _ = run(cur_lists, new_lists, B, stride=8)
        check_first_fit(cur_lists, new_lists, wave, [util.record_of(x, WAVE_SUMMARY_DTYPE.names) for x in summ], B)
        run(cur_lists, new_lists, B * 10, rng.integers(0, 30, 20000), stride=8)


def _documents(s, names, part_off, part_id, rep_off, cur, out, out_len, B, L, rollback, C=None):
    send = {} if C is None else dict(max_broker_out=C, send_brokers=s.broker_id)
    args = (names, part_off, part_id, rep_off, cur, out, out_len, B)
    if L is None:
        docs, wave, summ, st = s.plan_waves_json(*args, **send)
        backs, doc_wave = None, np.arange(1, len(docs) + 1)
    elif not rollback:
        docs, doc_wave, wave, summ, st = s.plan_wave_parts_json(*args, L, **send)
        backs = None
    else:
        docs, backs, doc_wave, wave, summ, st = s.plan_wave_parts_rollback_json(*args, L, **send)
    e_docs, e_backs, e_doc_wave, e_wave, e_summ, e_st = fit_models.wave_documents(
        names, part_off, part_id, rep_off, cur, out, out_len, s.broker_id, B, None, None if C is None else (list(s.broker_id), C), L,
        rollback)
    assert (st.code, st.a, st.b) == e_st
    assert np.array_equal(wave, e_wave) and list(doc_wave) == e_doc_wave
    dtype = WAVE_SUMMARY_DTYPE if C is None else WAVE_SEND_SUMMARY_DTYPE
    assert [util.record_of(x, dtype.names) for x in summ] == e_summ
    assert [bytes(x) for x in docs] == e_docs
    if rollback:
        assert [bytes(x) for x in backs] == e_backs
    return wave


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_documents_parts_and_rollback(native_lib, seed):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 31), 4))
    s.set_wave_rule("first_fit")
    rng = np.random.default_rng(300 + seed)
    names, part_off, part_id, rep_off, cur, out, out_len = util.ragged_wave_case(rng, 400, 30, shrink=0.1)
    for B, C in ((1, None), (3, None), (2, 4)):
        for L, rollback in ((None, False), (600, False), (10 ** 7, False), (600, True), (900, True)):
            _documents(s, names, part_off, part_id, rep_off, cur, out, out_len, B, L, rollback, C)


@pytest.mark.gpu
def test_broker_usage_of_a_first_fit_plan(native_lib):
    cl = kab.synth.make_ragged_cluster(T=3000, N=400, max_partitions=128, seed=21, remove_frac=0.02)
    s, out, out_len, _ = util.solved(cl)
    wave, _, st = util.check_plan(s, cl.rep_off, cl.cur, out, out_len, 1)
    assert st.code == 0
    usage, W, ust = s.broker_usage(cl.rep_off, cl.cur, out, out_len, wave, cl.all_broker_id)
    assert ust.code == 0 and W == int(wave.max())
    e, e_W, e_st = usage_models.broker_usage(cl.rep_off, cl.cur, out, out_len, wave, cl.all_broker_id)
    assert e_st == (0, 0, 0) and e_W == W
    assert [util.record_of(x, usage_models.FIELDS) for x in usage] == e


@pytest.mark.gpu
def test_the_rule_is_context_configuration(native_lib):
    cl = kab.synth.make_ragged_cluster(T=3000, N=400, max_partitions=128, seed=5, remove_frac=0.0)
    s, out, out_len, _ = util.solved(cl)
    assert s.wave_rule == "greedy"
    greedy = s.plan_waves(cl.rep_off, cl.cur, out, out_len, 1)
    fit = util.check_plan(s, cl.rep_off, cl.cur, out, out_len, 1)
    assert not np.array_equal(fit[0], greedy[0])
    s.reset()   # keeps the rule
    assert s.wave_rule == "first_fit"
    again = s.plan_waves(cl.rep_off, cl.cur, out, out_len, 1)
    assert np.array_equal(again[0], fit[0]) and np.array_equal(again[1], fit[1])
    s.set_wave_rule("greedy")   # back to exactly the earlier plan
    back = s.plan_waves(cl.rep_off, cl.cur, out, out_len, 1)
    assert np.array_equal(back[0], greedy[0]) and np.array_equal(back[1], greedy[1])
    assert s._L.ka_ctx_set_wave_rule(s._h, 2) == BAD and s._L.ka_ctx_set_wave_rule(s._h, -1) == BAD
    assert s.wave_rule == "greedy"


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
    s.set_wave_rule("first_fit")
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
    assert call(rep_off=bad_off)[0] == BAD and call(rep_off=rep_off + 1)[0] == BAD
    assert call(stride=9, new=np.full((1000, 9), -1, dtype=np.int32))[:2] == (LIMIT, 9)
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
    for rows, expect in (({700: [5, 5], 300: [1, 99]}, (BAD, 300, 99)), ({700: [1, 99], 300: [2, 6, 2]}, (BAD, 300, 2)),
                         ({999: [21]}, (BAD, 999, 21)), ({0: [3, 3]}, (BAD, 0, 3))):
        o, ln = out.copy(), out_len.copy()
        for g, x in rows.items():
            o[g, :] = -1
            o[g, :len(x)] = x
            ln[g] = len(x)
        assert call(new=o, new_len=ln) == expect
        assert fit_models.plan_waves(rep_off, cur, o, ln, s.broker_id, 2)[2] == expect
    assert call(Q=0)[0] == 0
    e_wave, e_summ, _ = fit_models.plan_waves(rep_off, cur, out, out_len, s.broker_id, 1)
    W = len(e_summ)
    assert W > 3
    few = np.zeros(3, dtype=WAVE_SUMMARY_DTYPE)
    rc, _, n = _raw(s, 1000, rep_off, cur, 3, out_len, out, None, 1, wave, few, 3)
    assert rc == 0 and n.value == W and [util.record_of(x, WAVE_SUMMARY_DTYPE.names) for x in few] == e_summ[:3]
    assert np.array_equal(wave, e_wave)
    # the sender row error of ka_plan_waves_send: a leader the send table lacks
    _, _, st = s.plan_waves(rep_off, cur, out, out_len, 2, max_broker_out=3, send_brokers=s.broker_id[1:])
    e = fit_models.plan_waves(rep_off, cur, out, out_len, s.broker_id, 2, send=(list(s.broker_id[1:]), 3))[2]
    assert (st.code, st.a, st.b) == e and e[0] == BAD and e[2] == 1


@pytest.mark.gpu
def test_load_table_limit(native_lib):
    """65 535 brokers and M rows all received by broker 2: Wb = M, so the 2^30-byte table holds 2 048 rows' waves, not 2 049."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 65536), 8))
    s.set_wave_rule("first_fit")
    for M, code in ((2048, 0), (2049, LIMIT)):
        rep_off, cur = util.cur_lists([[1]] * M)
        out, out_len = util.rows([[2]] * M)
        wave, summ, st = s.plan_waves(rep_off, cur, out, out_len, 1)
        assert st.code == code
        if code == 0:
            assert wave.tolist() == list(range(1, M + 1)) and len(summ) == M
        else:
            assert st.a == M and len(wave) == 0
    # a row error comes first
    rep_off, cur = util.cur_lists([[1]] * 2049)
    out, out_len = util.rows([[2]] * 2048 + [[3, 3]])
    assert s.plan_waves(rep_off, cur, out, out_len, 1)[2].code == BAD


@pytest.mark.gpu
def test_launches_are_fixed(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))
    rng = np.random.default_rng(9)
    counts = []
    for Q in (500, 20000):
        cur_lists, new_lists = util.random_wave_case(rng, Q, 40)
        rep_off, cur = util.cur_lists(cur_lists)
        out, out_len = util.rows(new_lists, 3)
        for rule in ("greedy", "first_fit"):
            s.set_wave_rule(rule)
            n0 = s.launch_count()
            rc, _, n = _raw(s, Q, rep_off, cur, 3, out_len, out, None, 1, np.zeros(Q, dtype=np.int32), None, 0)
            assert rc == 0 and n.value > 1
            counts.append(s.launch_count() - n0)
    assert counts[1] == counts[0] + 3 and counts[2:] == counts[:2]


@pytest.mark.gpu
def test_cpp_host_mirror(native_lib):
    """host/test_waves_first_fit.cpp: KafkaTopicAssigner::setWaveRule and planWaves under both rules."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_WAVES_FIRST_FIT_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
