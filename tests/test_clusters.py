"""ka_solve_clusters: a fleet of independent ragged clusters, each against its own broker table, in one call. Cluster k must give
exactly what a fresh context with table k gives through ka_solve over the cluster's own topics (rows, out_len, status), and the
oracle's answer where the size allows."""
import ctypes
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from tests import util
from tests.util import MIN_HASH, Member

pytestmark = pytest.mark.gpu

def _check_fleet(fleet, oracle=None, solver=None, S=None):
    S = S or util.fleet_stride(fleet)
    s = solver or kab.Solver(0)
    res = s.solve_clusters([m.entry() for m in fleet], out_stride=S)
    assert len(res) == len(fleet)
    ref = kab.Solver(0)
    sts = []
    for k, (m, (out, ln, st)) in enumerate(zip(fleet, res)):
        e_out, e_len, e_st = m.sequential(ref, S)
        assert util.fields(st) == e_st, (k, util.fields(st), e_st)
        sts.append(e_st)
        if e_st[0] != 0:
            continue   # the rows of a failed cluster are unspecified
        assert np.array_equal(out, e_out) and np.array_equal(ln, e_len), k
        if oracle is not None:
            o_len, _, o_out, o_st = oracle.run(oracle.OracleContext(), m.names, m.part_off, m.part_id, m.rep_off, m.cur, m.ids,
                                               ["k%d" % r for r in m.racks], m.desired_rf, S, raise_on_error=False)
            assert o_st.code == 0, k
            assert np.array_equal(out, o_out) and np.array_equal(ln, o_len), k
    return sts


@pytest.mark.parametrize("seed", [1, 2])
def test_heterogeneous_fleet_matches_sequential_and_oracle(native_lib, oracle, seed):
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
    order = rng.permutation(len(fleet))
    fleet = [fleet[i] for i in order]
    s = kab.Solver(0)
    sts = _check_fleet(fleet, oracle, solver=s)
    assert sum(st[0] == 0 for st in sts) >= 8, sts
    assert s.last_stage_plan()[6] == 7   # all three id lookup modes in one call
    assert s.last_order_plan()[7] == len(fleet)


def test_exceptions_and_refusals_are_isolated(native_lib, oracle):
    ok = [Member.of(kab.synth.make_ragged_cluster(T=40, N=30, R=5, seed=s)) for s in (3, 4, 5)]
    rf3 = {11: [1, 2, 3], 12: [2, 3, 4], 13: [3, 4, 5]}
    fails = [
        Member.of_topics(util.table(np.arange(1, 9)), [("t", {0: [1, 2], 9: [3]})]),                      # RF mismatch (KTA:58-60)
        Member.of_topics(util.table(np.arange(1, 9)), [("t", {0: [1, 2]}), ("none", {})]),                # no positive RF (KTA:65-66)
        Member.of_topics(util.table(np.arange(1, 3)), [("gamma", rf3)]),                                  # RF 3 > 2 brokers (KTA:67-69)
        Member.of_topics(util.table(np.arange(1, 9), 4), [("gamma", rf3)]),                               # two racks (KAS:183-184)
        Member.of_topics(util.table(np.arange(1, 4)), [(MIN_HASH, {5: [1, 2, 3]})]),                       # 2^31 % 3 (KAS:190-192)
        Member.of_topics(util.table(np.zeros(0)), [("alpha", {0: [1, 2]})]),                               # no broker at all
    ]
    bad_part = Member.of(kab.synth.make_ragged_cluster(T=20, N=30, R=5, seed=6))
    bad_part.part_off = bad_part.part_off.copy()
    bad_part.part_off[5] = bad_part.part_off[6] + 1                                                        # topic 5 ends before it starts
    bad_rep = Member.of(kab.synth.make_ragged_cluster(T=20, N=30, R=5, seed=7))
    bad_rep.rep_off = bad_rep.rep_off.copy()
    bad_rep.rep_off[7] = bad_rep.rep_off[8] + 1                                                            # a list of negative size
    long_list = Member.of_topics(util.table(np.arange(1, 9)), [("t", {0: [1, 2, 3]})])                      # longer than the stride 2
    huge = Member.of(kab.synth.make_ragged_cluster(T=20, N=40, R=5, seed=8), table=util.table(np.arange(1, 40001), 100))  # level-plan limit
    fleet = [ok[0]] + fails[:3] + [bad_part, ok[1], bad_rep] + fails[3:] + [huge, ok[2]]
    sts = _check_fleet(fleet, oracle, S=3)   # (the malformed rep_off has a list longer than 3)
    codes = [st[0] for st in sts]
    assert codes[0] == codes[5] == codes[-1] == 0
    assert set(codes) >= {1, 2, 3, 4, 5, _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT}, codes
    assert sts[-2][0] == _native.KA_ERR_LIMIT and sts[-2][4] == 40000
    # the return code is the status of the lowest failing cluster; a stride below a cluster's lists fails that cluster alone
    s = kab.Solver(0)
    st = (kab.KaStatus * 3)()
    assert _call(s, [ok[0], fails[4], fails[2]], st) == _native.KA_ERR_HASH_INDEX
    assert st[0].code == 0 and st[1].code == _native.KA_ERR_HASH_INDEX and st[2].code == _native.KA_ERR_RF_GT_BROKERS
    two = [Member.of(kab.synth.make_ragged_cluster(T=20, N=20, R=4, seed=9, rf_weights=(0.5, 0.5)))]
    sts = _check_fleet(two + [long_list] + two, S=2)
    assert [st[0] for st in sts] == [0, _native.KA_ERR_BAD_ARG, 0]


def test_edges(native_lib):
    mk = kab.synth.make_ragged_cluster
    one = Member.of(mk(T=300, N=60, R=6, seed=31))
    _check_fleet([one])                                                       # K = 1 is ka_solve
    empty = Member([np.arange(1, 5, dtype=np.int32), np.zeros(4, dtype=np.int32)], [], [], np.zeros(1, dtype=np.int64),
                   np.zeros(0, dtype=np.int32), np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.int32))
    no_rows = Member.of_topics(util.table(np.arange(1, 5)), [("e1", {}), ("e2", {})], desired_rf=2)
    sts = _check_fleet([empty, one, empty, no_rows, Member.of(mk(T=50, N=30, R=5, seed=32)), empty])
    assert all(st[0] == 0 for st in sts), sts
    assert all(st[0] == 0 for st in _check_fleet([empty, empty]))            # nothing to solve at all
    tiny = [Member.of(mk(T=8, N=24, R=4, seed=100 + k, max_partitions=32)) for k in range(128)]
    sts = _check_fleet(tiny)                                                  # K = 128
    assert sum(st[0] == 0 for st in sts) >= 32
    skewed = [Member.of(mk(T=20000, N=200, R=10, seed=40))] + [Member.of(mk(T=30, N=20, R=4, seed=41 + k)) for k in range(7)]
    assert skewed[0].part_off[-1] > 10 * sum(int(m.part_off[-1]) for m in skewed[1:])
    _check_fleet(skewed)


def _call(s, fleet, st, K=None, S=None, topic_off=None, part_off=None, rep_off=None, desired=True, tables=None):
    """ka_solve_clusters through ctypes, with every argument overridable."""
    lay = list(kab.Solver.marshal_clusters([m.entry() for m in fleet]))
    if tables is not None:
        lay[:3] = kab.Solver._candidate_tables(tables)
    cand_off, ids, racks, t_off, drf, th, p_off, pid, r_off, cur = lay
    t_off = t_off if topic_off is None else topic_off
    p_off = p_off if part_off is None else part_off
    r_off = r_off if rep_off is None else rep_off
    S = util.fleet_stride(fleet) if S is None else S
    out = np.zeros(max(int(p_off[-1]), 1) * max(S, 1), dtype=np.int32)
    vp = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    return s._L.ka_solve_clusters(s._h, len(fleet) if K is None else K, vp(cand_off), vp(ids), vp(racks), vp(t_off),
                                  vp(drf) if desired else None, vp(th), vp(p_off), vp(pid), vp(r_off), vp(cur), S, None, vp(out), st)


def test_arguments_and_limits(native_lib):
    mk = kab.synth.make_ragged_cluster
    fleet = [Member.of(mk(T=20, N=30, R=5, seed=s)) for s in (51, 52, 53)]
    s = kab.Solver(0)
    st = (kab.KaStatus * 200)()

    def every(code, n=len(fleet)):
        return all(st[k].code == code for k in range(n))

    assert _call(s, fleet, st, K=0) == 0
    assert _call(s, fleet * 43, st) == _native.KA_ERR_LIMIT and every(_native.KA_ERR_LIMIT, 129)
    assert _call(s, fleet, st, S=4) == _native.KA_ERR_LIMIT and every(_native.KA_ERR_LIMIT)
    assert _call(s, fleet, st, S=0) == _native.KA_ERR_BAD_ARG and every(_native.KA_ERR_BAD_ARG)
    t_off = kab.Solver.marshal_clusters([m.entry() for m in fleet])[3]
    for bad in ([1, 20, 40, 60], [0, 30, 20, 60]):                            # not from 0, decreasing
        assert _call(s, fleet, st, topic_off=np.array(bad, dtype=np.int32)) == _native.KA_ERR_BAD_ARG and every(_native.KA_ERR_BAD_ARG)
    p_off = kab.Solver.marshal_clusters([m.entry() for m in fleet])[6].copy()
    p_off[t_off[1]] = p_off[t_off[2]] + 1                                     # cluster 1 starts after cluster 2
    assert _call(s, fleet, st, part_off=p_off) == _native.KA_ERR_BAD_ARG and every(_native.KA_ERR_BAD_ARG)
    r_off = kab.Solver.marshal_clusters([m.entry() for m in fleet])[8].copy()
    row2 = int(kab.Solver.marshal_clusters([m.entry() for m in fleet])[6][t_off[2]])
    r_off[row2] = -1                                                          # cluster 2's lists start before cluster 1's
    assert _call(s, fleet, st, rep_off=r_off) == _native.KA_ERR_BAD_ARG and every(_native.KA_ERR_BAD_ARG)
    unsorted = [(m.ids, m.racks) for m in fleet[:2]] + [(fleet[2].ids[::-1].copy(), fleet[2].racks[::-1].copy())]
    assert _call(s, fleet, st, tables=unsorted) == _native.KA_ERR_BAD_ARG and every(_native.KA_ERR_BAD_ARG)
    assert _call(s, fleet, None) == _native.KA_ERR_BAD_ARG
    # desired_rf == NULL: -1 for every cluster
    assert _call(s, fleet, st, desired=False) == 0 and every(0)


def test_ctx_state_and_launches(native_lib):
    mk = kab.synth.make_ragged_cluster
    cl = mk(T=2000, N=120, R=6, seed=61)
    half = mk(T=1000, N=120, R=6, seed=62)
    s, fresh = kab.Solver(0), kab.Solver(0)
    for x in (s, fresh):
        x.set_brokers(cl.broker_id, cl.rack_index)
        x.solve_ragged(half.topic_hash, half.part_off, half.part_id, half.rep_off, half.cur, -1, 3)   # counters in the Context
    before = s.counters()
    _check_fleet([Member.of(mk(T=300, N=40 + 10 * k, R=5, seed=63 + k)) for k in range(4)], solver=s)
    assert np.array_equal(s.counters(), before) and np.array_equal(s.broker_id, cl.broker_id)
    a, al, ast = s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    b, bl, bst = fresh.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    assert ast.code == bst.code == 0 and np.array_equal(a, b) and np.array_equal(al, bl)
    assert np.array_equal(s.counters(), fresh.counters())
    # the same total shape cut into 2 or 32 clusters: the same launches
    big = mk(T=3200, N=100, R=6, seed=64)
    counts = []
    for K in (2, 32):
        cut = np.linspace(0, big.T, K + 1).astype(int)
        fleet = []
        for k in range(K):
            a_, b_ = cut[k], cut[k + 1]
            r0, r1 = int(big.part_off[a_]), int(big.part_off[b_])
            fleet.append(Member((big.broker_id, big.rack_index), big.topic_names[a_:b_], big.topic_hash[a_:b_],
                                big.part_off[a_:b_ + 1] - r0, big.part_id[r0:r1], big.rep_off[r0:r1 + 1] - big.rep_off[r0],
                                big.cur[big.rep_off[r0]:big.rep_off[r1]]))
        n0 = s.launch_count()
        res = s.solve_clusters([m.entry() for m in fleet], out_stride=3)
        counts.append(s.launch_count() - n0)
        assert all(st.code == 0 for _, _, st in res)
        assert s.last_order_plan()[7] == K and s.last_stage_plan()[3] == K
    assert counts[0] == counts[1] > 0, counts


def test_cpp_host_mirror(native_lib):
    """host/test_clusters.cpp: KafkaTopicAssigner::solveClusters against one fresh assigner per cluster, exception texts."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_CLUSTERS_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
