"""ka_score_clusters: the fleet of ka_solve_clusters, summarised on the device per cluster (data moved and broker balance). Every
cluster's summary and per-broker sums must equal the numpy reference (models.move_summary) over that cluster's rows
from ka_solve_clusters, and what ka_score_candidates gives for the cluster alone with its one table; statuses and (when asked
for) rows must equal ka_solve_clusters' for the same call."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import MOVE_SUMMARY_DTYPE
from tests import models, util
from tests.util import MIN_HASH, Member

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = MOVE_SUMMARY_DTYPE.names
INT64_MAX = np.iinfo(np.int64).max


# ---- CPU -----------------------------------------------------------------------------------------------------------------

def test_symbol_is_exported(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    assert hasattr(raw, "ka_score_clusters") and "ka_score_clusters" in _native.SYMBOLS


def test_without_a_context_is_no_device(native_lib):
    st = (kab.KaStatus * 3)()
    summary = np.zeros(3, dtype=MOVE_SUMMARY_DTYPE)
    summary["rows_changed"] = 7
    cand_off = np.array([0, 1, 2, 2], dtype=np.int32)
    ids = np.array([1, 2], dtype=np.int32)
    racks = np.zeros(2, dtype=np.int32)
    topic_off = np.zeros(4, dtype=np.int32)
    vp = ctypes.c_void_p
    p = lambda a: a.ctypes.data_as(vp)  # noqa: E731
    L = native_lib
    rc = L.ka_score_clusters(None, 3, p(cand_off), p(ids), p(racks), p(topic_off), None, None, None, None, None, None, 1, None,
                             p(summary), None, None, None, None, None, st)
    assert rc == _native.KA_ERR_NO_DEVICE
    assert [st[k].code for k in range(3)] == [_native.KA_ERR_NO_DEVICE] * 3
    assert [util.record_of(s, FIELDS) for s in summary] == [util.EMPTY_SUMMARY] * 3
    assert L.ka_score_clusters(None, 1, None, None, None, None, None, None, None, None, None, None, 1, None, p(summary), None, None,
                               None, None, None, None) == _native.KA_ERR_BAD_ARG          # st is required
    assert L.ka_score_clusters(None, 1, None, None, None, None, None, None, None, None, None, None, 1, None, None, None, None, None,
                               None, None, st) == _native.KA_ERR_BAD_ARG                 # summary is required
    assert st[0].code == _native.KA_ERR_BAD_ARG


def test_starts_with_the_batched_prologue():
    """Like the other batched entry points, ka_score_clusters runs batch_args, which refuses rows wider than 3: kernel A's CAND
    instances only ever run SM 3."""
    src = open(os.path.join(ROOT, "kafka_assigner_b200", "csrc", "kassign.cu")).read()
    fn = re.search(r"int32_t ka_score_clusters\(.*?\n}\n", src, flags=re.S)
    assert fn, "ka_score_clusters moved: update this test"
    assert re.search(r"int rc = batch_args\(c, K, out_stride, st\);\s*if \(rc != KA_OK\) return rc;", fn.group(0))


# ---- GPU -----------------------------------------------------------------------------------------------------------------

def _weights(fleet, rng):
    return [rng.integers(0, 1 << 40, size=int(m.part_off[-1]) if len(m.part_off) else 0, dtype=np.int64) for m in fleet]


def _check_scores(fleet, weights=None, S=None, solver=None, single=True):
    """One score_clusters call (rows and per-broker sums asked for) against solve_clusters' statuses and rows, the numpy
    reference of each cluster's rows, and (single) score_ragged_candidates of each cluster alone with its one table. Returns
    the statuses and summaries."""
    S = S or util.fleet_stride(fleet)
    s = solver or kab.Solver(0)
    entries = [m.entry() for m in fleet]
    solved = s.solve_clusters(entries, out_stride=S)
    res = s.score_clusters(entries, out_stride=S, weights=weights, rows=True, per_broker=True)
    assert len(res) == len(fleet)
    sts = []
    for k, (m, (out, ln, st), (summ, sst, sc_out, sc_len, rep, lead, inb)) in enumerate(zip(fleet, solved, res)):
        assert util.fields(sst) == util.fields(st), (k, util.fields(sst), util.fields(st))
        sts.append(util.fields(st))
        ids = np.asarray(m.ids, dtype=np.int64)
        assert len(rep) == len(lead) == len(inb) == len(ids)
        if st.code != 0:
            assert util.record_of(summ, FIELDS) == util.EMPTY_SUMMARY, k
            assert not rep.any() and not lead.any() and not inb.any(), k
            continue
        assert np.array_equal(sc_out, out) and np.array_equal(sc_len, ln), k
        w = None if weights is None else weights[k]
        rep_off = np.asarray(m.rep_off, dtype=np.int64) if len(m.rep_off) else np.zeros(1, dtype=np.int64)
        e, e_rep, e_lead, e_in = models.move_summary(out, ln, rep_off, np.asarray(m.cur), ids, w)
        assert util.record_of(summ, FIELDS) == e, (k, util.record_of(summ, FIELDS), e)
        assert np.array_equal(rep, e_rep) and np.array_equal(lead, e_lead) and np.array_equal(inb, e_in), k
        if single:
            one, ost, *brk = kab.Solver(0).score_ragged_candidates([(m.ids, m.racks)], m.topic_hash, m.part_off, m.part_id, m.rep_off,
                                                                  m.cur, m.desired_rf, out_stride=S, weight=w, per_broker=True)
            assert util.fields(ost[0]) == util.fields(st) and util.record_of(one[0], FIELDS) == util.record_of(summ, FIELDS), k
            assert all(np.array_equal(a[0], b) for a, b in zip(brk, (rep, lead, inb))), k
    return sts, [r[0] for r in res]


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2])
def test_heterogeneous_fleet(native_lib, seed):
    rng = np.random.default_rng(seed)
    mk = kab.synth.make_ragged_cluster
    fleet = [
        Member.of(mk(T=60, N=40, R=5, max_partitions=64, seed=seed)),                                         # rack-aware, RF 1..3
        Member.of(mk(T=30, N=30, R=4, seed=seed + 10, rf_weights=(1.0,)), desired_rf=2),                       # grows to 2
        Member.of(mk(T=40, N=50, R=6, seed=seed + 20), desired_rf=1),                                          # shrinks to 1
        Member.of(mk(T=25, N=20, R=3, seed=seed + 30, rf_weights=(0.5, 0.5))),                                 # rows of 1 and 2
        Member.of(mk(T=50, N=30, R=5, seed=seed + 40, max_partitions=1)),                                      # 1 partition per topic
        Member.of(mk(T=12, N=60, R=6, seed=seed + 50, max_partitions=600, tail=0.4)),                          # topics of hundreds
        Member.of(mk(T=30, N=40, R=5, seed=seed + 60), table=util.table(np.arange(1, 41))),                    # no racks
        Member.of(mk(T=30, N=30, R=5, seed=seed + 70), table=util.table(1 + 2 * np.arange(20000), 500)),       # global id LUT
        Member.of(mk(T=30, N=30, R=5, seed=seed + 80), table=util.bsearch_table(30)),                          # binary search
        util.min_hash_cluster(util.table(np.arange(1, 7))),
        Member.of(mk(T=20, N=24, R=4, seed=seed + 90), desired_rf=3),
    ]
    fleet = [fleet[i] for i in rng.permutation(len(fleet))]
    s = kab.Solver(0)
    for weights in (_weights(fleet, rng), None):
        sts, summ = _check_scores(fleet, weights, solver=s)
        assert sum(st[0] == 0 for st in sts) >= 8, sts
        assert s.last_stage_plan()[6] == 7   # all three id lookup modes in one call
        assert sum(x["replicas_added"] > 0 for x in summ) >= 6


@pytest.mark.gpu
def test_exceptions_and_refusals_are_isolated(native_lib):
    ok = [Member.of(kab.synth.make_ragged_cluster(T=40, N=30, R=5, seed=s)) for s in (3, 4, 5)]
    rf3 = {11: [1, 2, 3], 12: [2, 3, 4], 13: [3, 4, 5]}
    fails = [
        Member.of_topics(util.table(np.arange(1, 9)), [("t", {0: [1, 2], 9: [3]})]),                      # RF mismatch
        Member.of_topics(util.table(np.arange(1, 9)), [("t", {0: [1, 2]}), ("none", {})]),                # no positive RF
        Member.of_topics(util.table(np.arange(1, 3)), [("gamma", rf3)]),                                  # RF 3 > 2 brokers
        Member.of_topics(util.table(np.arange(1, 9), 4), [("gamma", rf3)]),                               # two racks
        Member.of_topics(util.table(np.arange(1, 4)), [(MIN_HASH, {5: [1, 2, 3]})]),                       # hash index
        Member.of_topics(util.table(np.zeros(0)), [("alpha", {0: [1, 2]})]),                               # no broker at all
    ]
    bad_part = Member.of(kab.synth.make_ragged_cluster(T=20, N=30, R=5, seed=6))
    bad_part.part_off = bad_part.part_off.copy()
    bad_part.part_off[5] = bad_part.part_off[6] + 1
    bad_rep = Member.of(kab.synth.make_ragged_cluster(T=20, N=30, R=5, seed=7))
    bad_rep.rep_off = bad_rep.rep_off.copy()
    bad_rep.rep_off[7] = bad_rep.rep_off[8] + 1
    huge = Member.of(kab.synth.make_ragged_cluster(T=20, N=40, R=5, seed=8), table=util.table(np.arange(1, 40001), 100))
    fleet = [ok[0]] + fails[:3] + [bad_part, ok[1], bad_rep] + fails[3:] + [huge, ok[2]]
    rng = np.random.default_rng(9)
    sts, _ = _check_scores(fleet, _weights(fleet, rng), S=3, single=False)
    codes = [st[0] for st in sts]
    assert codes[0] == codes[5] == codes[-1] == 0
    assert set(codes) >= {1, 2, 3, 4, 5, _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT}, codes
    assert sts[-2][0] == _native.KA_ERR_LIMIT and sts[-2][4] == 40000
    two = [Member.of(kab.synth.make_ragged_cluster(T=20, N=20, R=4, seed=9, rf_weights=(0.5, 0.5)))]
    long_list = Member.of_topics(util.table(np.arange(1, 9)), [("t", {0: [1, 2, 3]})])                      # longer than the stride
    sts, _ = _check_scores(two + [long_list] + two, S=2)
    assert [st[0] for st in sts] == [0, _native.KA_ERR_BAD_ARG, 0]


@pytest.mark.gpu
def test_segment_edges(native_lib):
    mk = kab.synth.make_ragged_cluster
    rng = np.random.default_rng(17)
    # 128 tiny clusters of 1..40 rows: boundaries inside warps and CTAs
    tiny = []
    for k in range(128):
        P = int(rng.integers(1, 41))
        topics = [("t%d" % k, {p: [int(x) for x in rng.choice(np.arange(1, 13), 3, replace=False)] for p in range(P)})]
        tiny.append(Member.of_topics(util.table(np.arange(1, 13), 3), topics))
    sts, _ = _check_scores(tiny, _weights(tiny, rng), single=False)
    assert sum(st[0] == 0 for st in sts) >= 64   # random lists over 4 racks: some clusters are unassignable
    # clusters with no topics, or only empty topics under a desired RF, between non-empty ones
    empty = Member([np.arange(1, 5, dtype=np.int32), np.zeros(4, dtype=np.int32)], [], [], np.zeros(1, dtype=np.int64),
                   np.zeros(0, dtype=np.int32), np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.int32))
    no_rows = Member.of_topics(util.table(np.arange(1, 5)), [("e1", {}), ("e2", {})], desired_rf=2)
    one = Member.of(mk(T=300, N=60, R=6, seed=31))
    fleet = [empty, one, empty, no_rows, Member.of(mk(T=50, N=30, R=5, seed=32)), empty]
    sts, summ = _check_scores(fleet, _weights(fleet, rng))
    assert all(st[0] == 0 for st in sts) and [util.record_of(summ[k], FIELDS) for k in (0, 2, 3, 5)] == [util.EMPTY_SUMMARY] * 4
    sts, summ = _check_scores([empty, no_rows])                                  # nothing to solve at all
    assert all(st[0] == 0 for st in sts) and [util.record_of(x, FIELDS) for x in summ] == [util.EMPTY_SUMMARY] * 2
    # a cluster whose rows start exactly at a multiple of 256
    first = Member.of_topics(util.table(np.arange(1, 9), 1), [("a", {p: [1 + p % 8, 1 + (p + 3) % 8] for p in range(200)}),
                                                           ("b", {p: [1 + p % 7, 1 + (p + 2) % 7] for p in range(312)})])
    assert int(first.part_off[-1]) == 512
    mid = Member.of(mk(T=40, N=30, R=5, seed=33))
    sts, _ = _check_scores([first, mid, first], _weights([first, mid, first], rng))
    assert all(st[0] == 0 for st in sts)
    # current lists with duplicate ids and with brokers missing from the cluster's table
    dup = Member.of_topics(util.table(np.arange(1, 7), 2), [("d", {0: [3, 3], 1: [9, 1], 2: [2, 2], 3: [40, 41], 4: [1, 2]})])
    sts, summ = _check_scores([one, dup, first], _weights([one, dup, first], rng))
    assert sts[1][0] == 0 and summ[1]["replicas_dropped"] > 0 and summ[1]["replicas_added"] > 0


@pytest.mark.gpu
def test_weights(native_lib):
    mk = kab.synth.make_ragged_cluster
    fleet = [Member.of(mk(T=40, N=30, R=5, seed=s)) for s in (41, 42, 43)]
    entries = [m.entry() for m in fleet]
    sizes = [int(m.part_off[-1]) for m in fleet]
    Q = sum(sizes)
    s = kab.Solver(0)
    a = s.score_clusters(entries)
    b = s.score_clusters(entries, weights=[np.ones(n, dtype=np.int64) for n in sizes])
    assert [util.record_of(x[0], FIELDS) for x in a] == [util.record_of(x[0], FIELDS) for x in b] and all(x[1].code == 0 for x in a)

    def split(flat):
        return [flat[o:o + n] for o, n in zip(np.cumsum([0] + sizes[:-1]), sizes)]

    edge = np.ones(Q, dtype=np.int64)
    edge[0] = INT64_MAX // 3 - (Q - 1)
    res = s.score_clusters(entries, weights=split(edge))
    assert all(x[1].code == 0 for x in res)
    solved = s.solve_clusters(entries)
    e, _, _, _ = models.move_summary(solved[0][0], solved[0][1], fleet[0].rep_off, fleet[0].cur, fleet[0].ids.astype(np.int64),
                                     split(edge)[0])
    assert util.record_of(res[0][0], FIELDS) == e
    over = edge.copy()
    over[Q - 1] += 1                                                          # in the last cluster: the whole call is refused
    res = s.score_clusters(entries, weights=split(over))
    assert all(x[1].code == _native.KA_ERR_LIMIT for x in res) and all(util.record_of(x[0], FIELDS) == util.EMPTY_SUMMARY for x in res)
    neg = np.ones(Q, dtype=np.int64)
    neg[sizes[0] + 3] = -1
    res = s.score_clusters(entries, weights=split(neg), per_broker=True)
    assert all(x[1].code == _native.KA_ERR_BAD_ARG for x in res)
    assert all(not a.any() for x in res for a in x[2:])
    # a call refused as a whole by ka_solve_clusters' own checks reports that code, not the weights'
    cand_off, ids, racks, t_off, drf, th, p_off, pid, r_off, cur = kab.Solver.marshal_clusters(entries)
    st = (kab.KaStatus * 3)()
    summary = np.zeros(3, dtype=MOVE_SUMMARY_DTYPE)
    vp = lambda x: None if x is None else x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    bad_t = np.array([0, 30, 20, 120], dtype=np.int32)

    def call(topic_off=t_off, S=3, tables=(cand_off, ids, racks)):
        return s._L.ka_score_clusters(s._h, 3, *[vp(x) for x in tables], vp(topic_off), vp(drf), vp(th), vp(p_off), vp(pid), vp(r_off),
                                      vp(cur), S, vp(neg), vp(summary), None, None, None, None, None, st)

    assert call(topic_off=bad_t) == _native.KA_ERR_BAD_ARG
    assert call(S=4) == _native.KA_ERR_LIMIT and all(st[k].code == _native.KA_ERR_LIMIT for k in range(3))
    unsorted = (cand_off, np.ascontiguousarray(ids[::-1]), racks)
    assert call(tables=unsorted) == _native.KA_ERR_BAD_ARG and all(st[k].code == _native.KA_ERR_BAD_ARG for k in range(3))
    assert call() == _native.KA_ERR_BAD_ARG   # the same call with a valid layout: the negative weight


@pytest.mark.gpu
def test_launches_state_and_optional_outputs(native_lib):
    mk = kab.synth.make_ragged_cluster
    s = kab.Solver(0)
    for K in (1, 8, 128):
        fleet = [Member.of(mk(T=8 if K == 128 else 60, N=24, R=4, max_partitions=32, seed=500 + k)) for k in range(K)]
        entries = [m.entry() for m in fleet]
        n0 = s.launch_count()
        s.solve_clusters(entries, out_stride=3)
        n1 = s.launch_count()
        s.score_clusters(entries, out_stride=3)
        assert s.launch_count() - n1 == n1 - n0 + 2, (K, n1 - n0, s.launch_count() - n1)
    # no side effects: the Solver's own table and counters, and two identical calls agree
    cl = mk(T=2000, N=120, R=6, seed=61)
    s.set_brokers(cl.broker_id, cl.rack_index)
    s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    before = s.counters()
    fleet = [Member.of(mk(T=300, N=40 + 10 * k, R=5, seed=63 + k)) for k in range(4)]
    entries = [m.entry() for m in fleet]
    w = _weights(fleet, np.random.default_rng(5))
    full = s.score_clusters(entries, weights=w, rows=True, per_broker=True)
    again = s.score_clusters(entries, weights=w, rows=True, per_broker=True)
    assert np.array_equal(s.counters(), before) and np.array_equal(s.broker_id, cl.broker_id)
    for x, y in zip(full, again):
        assert util.record_of(x[0], FIELDS) == util.record_of(y[0], FIELDS) and util.fields(x[1]) == util.fields(y[1])
        assert all(np.array_equal(a, b) for a, b in zip(x[2:], y[2:]))
    # rows=False and per_broker=False give the summaries of the full call
    for kw in (dict(), dict(rows=True), dict(per_broker=True)):
        part = s.score_clusters(entries, weights=w, **kw)
        assert [util.record_of(x[0], FIELDS) for x in part] == [util.record_of(x[0], FIELDS) for x in full], kw
        assert len(part[0]) == 2 + 2 * bool(kw.get("rows")) + 3 * bool(kw.get("per_broker"))


@pytest.mark.gpu
def test_cpp_host_mirror(native_lib):
    """host/test_cluster_scores.cpp: KafkaTopicAssigner::scoreClusters against scoreTopicsCandidates with one table per cluster."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_CLUSTER_SCORES_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
