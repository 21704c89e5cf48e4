"""ka_score_candidates: the batched ragged solve of ka_solve_candidates, summarised on the device per candidate (data moved and
broker balance). Every summary must equal, field for field, the numpy reference models.move_summary computed from ka_solve_candidates' rows;
statuses and (when asked for) rows must equal ka_solve_candidates' for the same call."""
import ctypes
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import MOVE_SUMMARY_DTYPE
from tests import models, util

FIELDS = MOVE_SUMMARY_DTYPE.names
INT64_MAX = np.iinfo(np.int64).max


# ---- CPU -----------------------------------------------------------------------------------------------------------------

def test_reference_on_a_hand_written_case():
    ids = np.array([1, 2, 3, 4, 6], dtype=np.int64)                     # broker 5 removed; 6 is left with nothing
    cur_lists = [[1, 2, 3], [2, 1], [5, 1], [3, 3], []]                 # unchanged, leader swap, removed broker, duplicate, empty
    new_lists = [[1, 2, 3], [1, 2], [4, 1], [3, 4], [2, 3]]
    rep_off = np.zeros(6, dtype=np.int64)
    np.cumsum([len(x) for x in cur_lists], out=rep_off[1:])
    cur = np.array([b for x in cur_lists for b in x], dtype=np.int32)
    out = np.full((5, 3), -1, dtype=np.int32)
    for g, x in enumerate(new_lists):
        out[g, :len(x)] = x
    out_len = np.array([len(x) for x in new_lists], dtype=np.int32)
    w = np.array([1, 10, 100, 1000, 10000], dtype=np.int64)
    s, rep, lead, inb = models.move_summary(out, out_len, rep_off, cur, ids, w)
    assert s == dict(rows_changed=4, rows_moved=3, leaders_changed=3, replicas_added=21100, replicas_dropped=100,
                     max_broker_in=10000, max_broker_in_id=2, max_broker_replicas=11001, min_broker_replicas=0,
                     max_broker_leaders=10000, min_broker_leaders=0)
    assert rep.tolist() == [111, 10011, 11001, 1100, 0]
    assert lead.tolist() == [11, 10000, 1000, 100, 0]
    assert inb.tolist() == [0, 10000, 10000, 1100, 0]
    s1, rep1, lead1, inb1 = models.move_summary(out, out_len, rep_off, cur, ids)
    assert s1 == dict(rows_changed=4, rows_moved=3, leaders_changed=3, replicas_added=4, replicas_dropped=1, max_broker_in=2,
                      max_broker_in_id=4, max_broker_replicas=3, min_broker_replicas=0, max_broker_leaders=2, min_broker_leaders=0)
    assert rep1.tolist() == [3, 3, 3, 2, 0] and lead1.tolist() == [2, 1, 1, 1, 0] and inb1.tolist() == [0, 1, 1, 2, 0]
    # nothing added: no receiving broker
    s2, _, _, _ = models.move_summary(out[:1], out_len[:1], rep_off[:2], cur, ids)
    assert s2["replicas_added"] == 0 and s2["max_broker_in"] == 0 and s2["max_broker_in_id"] == -1


def test_symbol_is_exported(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    assert hasattr(raw, "ka_score_candidates") and "ka_score_candidates" in _native.SYMBOLS
    assert ctypes.sizeof(_native.KaMoveSummary) == 11 * 8 and MOVE_SUMMARY_DTYPE.itemsize == 11 * 8


def test_without_a_context_is_no_device(native_lib):
    st = (kab.KaStatus * 3)()
    summary = np.zeros(3, dtype=MOVE_SUMMARY_DTYPE)
    summary["rows_changed"] = 7
    cand_off = np.array([0, 1, 2, 2], dtype=np.int32)
    ids = np.array([1, 2], dtype=np.int32)
    racks = np.zeros(2, dtype=np.int32)
    vp = ctypes.c_void_p
    rc = native_lib.ka_score_candidates(None, 3, cand_off.ctypes.data_as(vp), ids.ctypes.data_as(vp), racks.ctypes.data_as(vp), 0,
                                        None, None, None, None, None, -1, 1, None, summary.ctypes.data_as(vp), None, None, None,
                                        None, None, st)
    assert rc == _native.KA_ERR_NO_DEVICE
    assert [st[k].code for k in range(3)] == [_native.KA_ERR_NO_DEVICE] * 3
    assert [util.record_of(s, FIELDS) for s in summary] == [util.EMPTY_SUMMARY] * 3
    assert native_lib.ka_score_candidates(None, 1, None, None, None, 0, None, None, None, None, None, -1, 1, None,
                                          summary.ctypes.data_as(vp), None, None, None, None, None, None) == _native.KA_ERR_BAD_ARG
    assert native_lib.ka_score_candidates(None, 1, None, None, None, 0, None, None, None, None, None, -1, 1, None, None, None, None,
                                          None, None, None, st) == _native.KA_ERR_BAD_ARG   # summary is required


# ---- GPU -----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_ragged_clusters(native_lib, oracle, seed):
    rng = np.random.default_rng(seed)
    cl = kab.synth.make_ragged_cluster(T=80, N=40, R=5, max_partitions=64, seed=seed, remove_frac=0.1)
    tables = util.ragged_mixed_tables(rng, cl)
    n_ok = 0
    for desired_rf in (-1, 1, 2, 3):
        prob = util.Problem(*util.sparse_with_empty_topics(cl, rng, desired_rf > 0), desired_rf)
        Q = int(prob.part_off[-1])
        weight = rng.integers(0, 1 << 40, size=Q, dtype=np.int64)
        sts, _ = util.check_scores(prob, tables, weight, oracle if desired_rf in (-1, 2) else None)
        n_ok += sum(st[0] == 0 for st in sts)
        assert sts[-1][0] == _native.KA_ERR_RF_GT_BROKERS
        # no weights == weights of one
        s = kab.Solver(0)
        a, _ = s.score_ragged_candidates(tables, *prob.args(), out_stride=prob.S)
        b, _ = s.score_ragged_candidates(tables, *prob.args(), out_stride=prob.S, weight=np.ones(Q, dtype=np.int64))
        assert np.array_equal(a, b)
    assert n_ok >= 16, n_ok


@pytest.mark.gpu
def test_one_exception_per_candidate(native_lib, oracle):
    A = util.table(np.arange(1, 9, dtype=np.int32))
    B = util.table(np.arange(1, 3, dtype=np.int32))            # gamma: RF 3 > 2 brokers
    C = util.table(np.arange(1, 4, dtype=np.int32))            # polygenelubricants: hash index
    D = util.table(np.arange(1, 9, dtype=np.int32), 4)         # gamma: unassignable over two racks
    E = util.table(np.zeros(0, dtype=np.int32))                # no broker
    kinds = set()
    for tail in ("mismatch", "empty", None):
        prob = util.exception_problem(tail)
        sts, summary = util.check_scores(prob, [A, B, C, D, E, A], oracle=oracle)
        kinds |= {st[0] for st in sts}
        if tail is None:
            assert sts[0][0] == sts[5][0] == 0 and util.record_of(summary[0], FIELDS) == util.record_of(summary[5], FIELDS)
            assert summary[0]["rows_changed"] > 0
    assert kinds == {0, 1, 2, 3, 4, 5}


@pytest.mark.gpu
def test_c3_in_the_ragged_layout(native_lib):
    cl = kab.synth.make_config("c3", "mixed")
    rng = np.random.default_rng(3)
    ids = [np.sort(rng.choice(cl.broker_id, len(cl.broker_id) - 20, replace=False)) for _ in range(8)]
    tables = [(i, cl.rack_index[np.searchsorted(cl.broker_id, i)]) for i in ids]
    part_off, part_id, rep_off, cur = cl.ragged()
    prob = util.Problem(cl.topic_names, cl.topic_hash, part_off, part_id, rep_off, cur)
    weight = rng.integers(1, 1 << 30, size=int(part_off[-1]), dtype=np.int64)
    sts, summary = util.check_scores(prob, tables, weight, sequential=False)
    assert all(st[0] == 0 for st in sts) and np.all(summary["replicas_added"] > 0)


@pytest.mark.gpu
def test_million_partition_cluster_at_k32(native_lib):
    cl = kab.synth.make_ragged_cluster(T=240000, N=400, max_partitions=128, seed=11)
    assert cl.Q > 1_000_000
    rng = np.random.default_rng(32)
    tables = kab.synth.ragged_decommission_tables(cl, util.FRACS)
    tables += [(cl.broker_id[k], cl.rack_index[k]) for k in (np.sort(rng.choice(len(cl.broker_id), 392, replace=False))
                                                               for _ in range(32 - len(tables)))]
    prob = util.Problem.of(cl)
    s = kab.Solver(0)
    out, ln, sts = prob.batched(tables, s)
    weight = rng.integers(0, 1 << 36, size=cl.Q, dtype=np.int64)
    summary, st = s.score_ragged_candidates(tables, *prob.args(), weight=weight)
    assert [util.fields(x) for x in st] == sts and sum(x[0] == 0 for x in sts) >= 24
    for k, (ids, _) in enumerate(tables):
        if sts[k][0] == 0:
            e, _, _, _ = models.move_summary(out[k], ln[k], prob.rep_off, prob.cur, np.asarray(ids, dtype=np.int64), weight)
            assert util.record_of(summary[k], FIELDS) == e, k
        else:
            assert util.record_of(summary[k], FIELDS) == util.EMPTY_SUMMARY, k


@pytest.mark.gpu
def test_ctx_is_untouched(native_lib):
    cl = kab.synth.make_ragged_cluster(T=3000, N=120, R=6, seed=21)
    half = kab.synth.make_ragged_cluster(T=1500, N=120, R=6, seed=22)
    s, fresh = kab.Solver(0), kab.Solver(0)
    for x in (s, fresh):
        x.set_brokers(cl.broker_id, cl.rack_index)
        x.solve_ragged(*util.Problem.of(half).args(), 3)
    before = s.counters()
    util.check_scores(util.Problem.of(cl), kab.synth.ragged_decommission_tables(cl, (0.1, 0.3)), solver=s, sequential=False)
    assert np.array_equal(s.counters(), before) and np.array_equal(s.broker_id, cl.broker_id)
    a, al, ast = s.solve_ragged(*util.Problem.of(cl).args(), 3)
    b, bl, bst = fresh.solve_ragged(*util.Problem.of(cl).args(), 3)
    assert ast.code == bst.code == 0 and np.array_equal(a, b) and np.array_equal(al, bl)
    assert np.array_equal(s.counters(), fresh.counters())


@pytest.mark.gpu
def test_launches_do_not_depend_on_k(native_lib):
    cl = kab.synth.make_ragged_cluster(T=3000, N=120, R=6, seed=21)
    prob = util.Problem.of(cl)
    s = kab.Solver(0)
    counts = []
    for K in (1, 8):
        tables = kab.synth.ragged_decommission_tables(cl, np.linspace(0.0, 0.2, K))
        n0 = s.launch_count()
        prob.batched(tables, solver=s)
        n1 = s.launch_count()
        s.score_ragged_candidates(tables, *prob.args())
        counts.append((n1 - n0, s.launch_count() - n1))
    assert counts[0] == counts[1] and counts[0][1] == counts[0][0] + 2, counts


def _call(fn, s, prob, tables, st, K=None, out_stride=None, T=None, part_off=None, rep_off=None, weight=None, out_elems=None,
          summary=True):
    """ka_solve_candidates (fn == 'solve') or ka_score_candidates (fn == 'score', rows not asked for) through ctypes, with every
    argument overridable."""
    ids = np.concatenate([t[0] for t in tables]).astype(np.int32) if tables else np.zeros(1, dtype=np.int32)
    racks = np.concatenate([t[1] for t in tables]).astype(np.int32) if tables else np.zeros(1, dtype=np.int32)
    off = np.zeros(len(tables) + 1, dtype=np.int32)
    np.cumsum([len(t[0]) for t in tables], out=off[1:])
    part_off = prob.part_off if part_off is None else part_off
    rep_off = prob.rep_off if rep_off is None else rep_off
    S = prob.S if out_stride is None else out_stride
    vp = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    K = len(tables) if K is None else K
    T = len(prob.topic_hash) if T is None else T
    head = (s._h, K, vp(off), vp(ids), vp(racks), T, vp(prob.topic_hash), vp(part_off), vp(prob.part_id), vp(rep_off), vp(prob.cur),
            prob.desired_rf, S)
    if fn == "solve":
        out = np.zeros(out_elems or max(len(tables), 1) * max(int(prob.part_off[-1]), 1) * max(S, 1), dtype=np.int32)
        return s._L.ka_solve_candidates(*head, None, vp(out), st)
    summ = np.zeros(max(K, 1), dtype=MOVE_SUMMARY_DTYPE) if summary else None
    return s._L.ka_score_candidates(*head, vp(weight), vp(summ), None, None, None, None, None, st)


@pytest.mark.gpu
def test_arguments_and_limits(native_lib):
    cl = kab.synth.make_ragged_cluster(T=40, N=30, R=5, seed=5)
    prob = util.Problem.of(cl)
    Q = int(prob.part_off[-1])
    good = [(cl.broker_id, cl.rack_index)]
    s = kab.Solver(0)
    st, st2 = (kab.KaStatus * 200)(), (kab.KaStatus * 200)()

    def same(*a, **kw):
        """Both entry points give the same code and statuses; returns the code."""
        rc = _call("score", s, *a, st, **kw)
        kw.pop("weight", None)
        assert _call("solve", s, *a, st2, **kw) == rc, (rc, kw)
        assert [util.fields(st[k]) for k in range(len(a[1]))] == [util.fields(st2[k]) for k in range(len(a[1]))], kw
        return rc

    assert same(prob, []) == 0
    assert same(prob, good, T=0) == 0
    assert same(prob, good * 129) == _native.KA_ERR_LIMIT and st[128].code == _native.KA_ERR_LIMIT
    assert same(prob, good, out_stride=4) == _native.KA_ERR_LIMIT
    assert same(prob, good, out_stride=2) == _native.KA_ERR_BAD_ARG
    assert same(prob, good, out_stride=0) == _native.KA_ERR_BAD_ARG
    unsorted = [(cl.broker_id[::-1].copy(), cl.rack_index[::-1].copy())]
    assert same(prob, good + unsorted) == _native.KA_ERR_BAD_ARG
    bad_part = prob.part_off.copy()
    bad_part[5] = bad_part[6] + 1
    bad_rep = prob.rep_off.copy()
    bad_rep[7] = bad_rep[8] + 1
    neg = np.ones(Q, dtype=np.int64)
    neg[Q // 2] = -1
    for kw in (dict(part_off=bad_part), dict(rep_off=bad_rep), dict(part_off=prob.part_off + 1)):
        assert same(prob, good * 2, **kw) == _native.KA_ERR_BAD_ARG
        assert same(prob, good * 2, weight=neg, **kw) == _native.KA_ERR_BAD_ARG   # the solve's status comes first
    assert same(prob, good * 2, weight=neg, out_stride=4) == _native.KA_ERR_LIMIT
    # the new checks: a negative weight, 3 x the sum of the weights beyond INT64_MAX
    assert _call("score", s, prob, good * 2, st, weight=neg) == _native.KA_ERR_BAD_ARG and st[1].code == _native.KA_ERR_BAD_ARG
    edge = np.zeros(Q, dtype=np.int64)
    edge[0] = INT64_MAX // 3 - (Q - 1)
    edge[1:] = 1
    assert _call("score", s, prob, good, st, weight=edge) == 0
    edge[3] += 1
    assert _call("score", s, prob, good * 2, st, weight=edge) == _native.KA_ERR_LIMIT and st[1].code == _native.KA_ERR_LIMIT
    huge = np.full(Q, INT64_MAX // 2, dtype=np.int64)                            # the sum itself would wrap
    assert _call("score", s, prob, good, st, weight=huge) == _native.KA_ERR_LIMIT
    assert _call("score", s, prob, good, st, summary=False) == _native.KA_ERR_BAD_ARG and st[0].code == _native.KA_ERR_BAD_ARG
    assert _call("score", s, prob, good, None) == _native.KA_ERR_BAD_ARG
    # at the largest total weight the sums are still exact
    summary, sts = s.score_ragged_candidates(good, *prob.args(), weight=np.where(np.arange(Q) == 3, edge - 1, edge))
    out, ln, _ = prob.batched(good, s)
    e, _, _, _ = models.move_summary(out[0], ln[0], prob.rep_off, prob.cur, cl.broker_id.astype(np.int64),
                                     np.where(np.arange(Q) == 3, edge - 1, edge))
    assert sts[0].code == 0 and util.record_of(summary[0], FIELDS) == e
    # T == 0: zero summaries and per-broker entries
    summary, sts, rep, lead, inb = s.score_ragged_candidates(good * 2, prob.topic_hash[:0], prob.part_off[:1], None, prob.rep_off[:1],
                                                             prob.cur[:0], -1, out_stride=3, per_broker=True)
    assert [util.record_of(x, FIELDS) for x in summary] == [util.EMPTY_SUMMARY] * 2 and all(x.code == 0 for x in sts)
    assert all(len(a) == len(cl.broker_id) and not a.any() for a in rep + lead + inb)
    # K * ΣP at 2^31: refused before anything is written
    big_q = (1 << 31) // 128
    big = util.Problem(["t"], prob.topic_hash[:1], np.array([0, big_q], dtype=np.int64), None, np.zeros(big_q + 1, dtype=np.int64),
                       np.zeros(0, dtype=np.int32), 1, 1)
    assert same(big, good * 128, out_elems=1) == _native.KA_ERR_LIMIT


@pytest.mark.gpu
def test_cpp_host_mirror(native_lib):
    """host/test_candidate_scores.cpp: KafkaTopicAssigner::scoreTopicsCandidates against summaries of solveTopicsCandidates."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_SCORES_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
