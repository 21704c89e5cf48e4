"""ka_solve_clusters_json: a fleet of independent ragged clusters, each against its own broker table, with every cluster's
reassignment JSON built on the device in one call. Cluster k's text and status must equal what a fresh context with table k
gives through ka_solve_json over the cluster's own topics, and its text the oracle's where the size allows."""
import ctypes
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from tests import models, util
from tests.util import MIN_HASH, Member

pytestmark = pytest.mark.gpu


def _raw(s, fleet, cap=1 << 22, K=None, names=True, json=True, json_off=True, part_id=True, topic_off=None, tables=None):
    """ka_solve_clusters_json through ctypes, with every argument overridable: (rc, json_off, buffer, st)."""
    lay = list(kab.Solver.marshal_clusters([m.entry() for m in fleet]))
    if tables is not None:
        lay[:3] = kab.Solver._candidate_tables(tables)
    cand_off, ids, racks, t_off, drf, th, p_off, pid, r_off, cur = lay
    t_off = t_off if topic_off is None else topic_off
    nm, noff = kab.Solver.marshal_names([n for m in fleet for n in m.names])
    buf = np.zeros(max(cap, 1), dtype=np.uint8)
    off = np.full(max(len(fleet), 1) + 1, -7, dtype=np.int64)
    st = (kab.KaStatus * max(len(fleet), 1))()
    vp = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = s._L.ka_solve_clusters_json(s._h, len(fleet) if K is None else K, vp(cand_off), vp(ids), vp(racks), vp(t_off), vp(drf), vp(th),
                                     vp(p_off), vp(pid) if part_id else None, vp(r_off), vp(cur), vp(nm) if names else None,
                                     vp(noff) if names else None, vp(buf) if json else None, cap, vp(off) if json_off else None, st)
    return rc, off, buf, st


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
        util.min_hash_cluster(util.table(np.arange(1, 7))),                                                    # hashCode MIN_VALUE
        Member.of(mk(T=20, N=24, R=4, seed=seed + 90), desired_rf=3),
    ]
    fleet = [fleet[i] for i in rng.permutation(len(fleet))]
    s = kab.Solver(0)
    sts, texts = util.check_fleet(fleet, oracle, solver=s)
    assert sum(st[0] == 0 for st in sts) >= 8, sts
    assert s.last_stage_plan()[6] == 7   # all three id lookup modes in one call
    assert s.last_order_plan()[7] == len(fleet)


def test_exceptions_refusals_and_edges_are_isolated(native_lib, oracle):
    mk = kab.synth.make_ragged_cluster
    ok = [Member.of(mk(T=40, N=30, R=5, seed=s)) for s in (3, 4, 5)]
    rf3 = {11: [1, 2, 3], 12: [2, 3, 4], 13: [3, 4, 5]}
    fails = [
        Member.of_topics(util.table(np.arange(1, 9)), [("t", {0: [1, 2], 9: [3]})]),                      # RF mismatch (KTA:58-60)
        Member.of_topics(util.table(np.arange(1, 9)), [("t", {0: [1, 2]}), ("none", {})]),                # no positive RF (KTA:65-66)
        Member.of_topics(util.table(np.arange(1, 3)), [("gamma", rf3)]),                                  # RF 3 > 2 brokers (KTA:67-69)
        Member.of_topics(util.table(np.arange(1, 9), 4), [("gamma", rf3)]),                               # two racks (KAS:183-184)
        Member.of_topics(util.table(np.arange(1, 4)), [(MIN_HASH, {5: [1, 2, 3]})]),                       # 2^31 % 3 (KAS:190-192)
    ]
    wide = Member.of_topics(util.table(np.arange(1, 9)), [("w", {0: [1, 2, 3, 4], 1: [2, 3, 4, 5]})])       # width 4
    quoted = Member.of(mk(T=20, N=30, R=5, seed=9))
    quoted.names[4] = "a/b"                                                                                 # org.json escapes '/'
    empty = Member([np.arange(1, 5, dtype=np.int32), np.zeros(4, dtype=np.int32)], [], [], np.zeros(1, dtype=np.int64),
                   np.zeros(0, dtype=np.int32), np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.int32))
    no_rows = Member.of_topics(util.table(np.arange(1, 5)), [("e1", {}), ("e2", {})], desired_rf=2)
    fleet = [fails[0], empty, ok[0], fails[1], wide, no_rows, fails[2], ok[1], quoted, fails[3], empty, ok[2], fails[4]]
    sts, texts = util.check_fleet(fleet, oracle)
    codes = [st[0] for st in sts]
    assert codes == [1, 0, 0, 2, _native.KA_ERR_LIMIT, 0, 3, 0, _native.KA_ERR_BAD_ARG, 4, 0, 0, 5], codes
    assert sts[4][3] == 4 and sts[8][3] == ord("/")
    assert texts[1] == texts[5] == texts[10] == models.EMPTY_DOCUMENT.encode()
    # the failing clusters first and last, and a fleet where only the empty documents are left
    util.check_fleet([wide, ok[0], quoted])
    assert [st[0] for st in util.check_fleet([empty, quoted, no_rows])[0]] == [0, _native.KA_ERR_BAD_ARG, 0]
    assert [st[0] for st in util.check_fleet([empty, empty])[0]] == [0, 0]


def test_many_documents_per_block_and_fragments_per_document(native_lib):
    # one row per cluster: a 256-row block of the length and write passes spans 128 documents
    tiny = [Member.of_topics(util.table(np.arange(1, 4 + k % 5)), [("t%d" % k, {k: [1 + k % 3, 2 + k % 2]})], desired_rf=k % 3 - 1)
            for k in range(128)]
    sts, _ = util.check_fleet(tiny)
    assert sum(st[0] == 0 for st in sts) >= 80
    mk = kab.synth.make_ragged_cluster
    util.check_fleet([Member.of(mk(T=8, N=24, R=4, seed=100 + k, max_partitions=32)) for k in range(128)])   # 128 tiny clusters
    # clusters large enough that the fragments of 2^18 rows cut through a document
    big = [Member.of(mk(T=30000, N=400, max_partitions=128, seed=100 + k)) for k in range(3)]
    assert sum(int(m.part_off[-1]) for m in big) > 1 << 18
    assert all(st[0] == 0 for st in util.check_fleet([big[0], Member.of(mk(T=20, N=20, R=4, seed=74)), big[1], big[2]])[0])


def test_part_id_null_and_sparse(native_lib):
    mk = kab.synth.make_ragged_cluster
    fleet = [Member.of(mk(T=40, N=30, R=5, seed=80 + k)) for k in range(3)]
    s = kab.Solver(0)
    for m in fleet:   # the ordinal form: ka_solve_json with part_id NULL
        m.part_id = None
    rc, off, buf, st = _raw(s, fleet, part_id=False)
    ref = kab.Solver(0)
    assert rc == next((st[k].code for k in range(3) if st[k].code), 0)
    for k, m in enumerate(fleet):
        e_text, e_st = util.sequential_json(m, ref)
        assert util.fields(st[k]) == e_st and bytes(buf[off[k]:off[k + 1]]) == e_text


def test_buffer_size_and_arguments(native_lib):
    mk = kab.synth.make_ragged_cluster
    bad = Member.of_topics(util.table(np.arange(1, 3)), [("gamma", {0: [1, 2, 3]})])
    fleet = [Member.of(mk(T=20, N=30, R=5, seed=s)) for s in (51, 52)] + [bad]
    s = kab.Solver(0)
    rc, off, buf, st = _raw(s, fleet)
    assert rc == 3 and off[0] == 0 and [st[k].code for k in range(3)] == [0, 0, 3] and off[2] == off[3]
    need = int(off[-1])
    text = bytes(buf[:need])
    rc, off2, buf2, st2 = _raw(s, fleet, cap=need)
    assert rc == 3 and np.array_equal(off, off2) and bytes(buf2[:need]) == text
    rc, off2, _, st2 = _raw(s, fleet, cap=need - 1)
    assert rc == _native.KA_ERR_LIMIT and not off2.any()
    assert [util.fields(st2[k]) for k in range(3)] == [(_native.KA_ERR_LIMIT, -1, -1, need - 1, 0)] * 2 + [util.fields(st[2])]
    # the documented sufficient size is what Solver.solve_clusters_json allocates
    assert all(bytes(t) == bytes(buf[off[k]:off[k + 1]])
               for k, (t, _) in enumerate(s.solve_clusters_json([m.entry() for m in fleet], [m.names for m in fleet])))
    # K == 0, and the whole-call argument checks
    rc, off, _, _ = _raw(s, fleet, K=0)
    assert rc == 0 and off[0] == 0

    def every(st, code):
        return all(st[k].code == code for k in range(len(fleet)))

    for kw in (dict(names=False), dict(json=False), dict(topic_off=np.array([0, 30, 20, 41], dtype=np.int32)),
               dict(tables=[(m.ids, m.racks) for m in fleet[:2]] + [(bad.ids[::-1].copy(), bad.racks)])):
        rc, off, _, st = _raw(s, fleet, **kw)
        assert rc == _native.KA_ERR_BAD_ARG and every(st, rc) and not off.any(), kw
    rc, _, _, st = _raw(s, fleet, json_off=False)
    assert rc == _native.KA_ERR_BAD_ARG and every(st, rc)
    rc, _, _, st = _raw(s, fleet * 43)
    assert rc == _native.KA_ERR_LIMIT and all(st[k].code == rc for k in range(129))
    assert _raw(s, fleet, K=3)[0] == 3
    stn = None
    assert s._L.ka_solve_clusters_json(s._h, 1, None, None, None, None, None, None, None, None, None, None, None, None, None, 0, None,
                                       stn) == _native.KA_ERR_BAD_ARG


def test_ctx_state_and_launches(native_lib):
    mk = kab.synth.make_ragged_cluster
    cl = mk(T=2000, N=120, R=6, seed=61)
    half = mk(T=1000, N=120, R=6, seed=62)
    s, fresh = kab.Solver(0), kab.Solver(0)
    for x in (s, fresh):
        x.set_brokers(cl.broker_id, cl.rack_index)
        x.solve_ragged(half.topic_hash, half.part_off, half.part_id, half.rep_off, half.cur, -1, 3)   # counters in the Context
    before = s.counters()
    fleet = [Member.of(mk(T=300, N=40 + 10 * k, R=5, seed=63 + k)) for k in range(4)]
    util.check_fleet(fleet, solver=s)
    assert s.last_order_plan()[7] == len(fleet) and s.last_stage_plan()[3] == len(fleet)
    assert np.array_equal(s.counters(), before) and np.array_equal(s.broker_id, cl.broker_id)
    a, al, ast = s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    b, bl, bst = fresh.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    assert ast.code == bst.code == 0 and np.array_equal(a, b) and np.array_equal(al, bl)
    assert np.array_equal(s.counters(), fresh.counters())
    # the same total shape cut into 2 or 64 clusters: the same launches
    big = mk(T=3200, N=100, R=6, seed=64)
    counts = []
    for K in (2, 64):
        cut = np.linspace(0, big.T, K + 1).astype(int)
        fleet = []
        for k in range(K):
            a_, b_ = cut[k], cut[k + 1]
            r0, r1 = int(big.part_off[a_]), int(big.part_off[b_])
            fleet.append(Member((big.broker_id, big.rack_index), big.topic_names[a_:b_], big.topic_hash[a_:b_],
                                big.part_off[a_:b_ + 1] - r0, big.part_id[r0:r1], big.rep_off[r0:r1 + 1] - big.rep_off[r0],
                                big.cur[big.rep_off[r0]:big.rep_off[r1]]))
        n0 = s.launch_count()
        res = s.solve_clusters_json([m.entry() for m in fleet], [m.names for m in fleet])
        counts.append(s.launch_count() - n0)
        assert all(st.code == 0 for _, st in res)
        assert s.last_order_plan()[7] == K
    assert counts[0] == counts[1] > 0, counts


def test_cpp_host_mirror(native_lib):
    """host/test_clusters_json.cpp: KafkaTopicAssigner::solveClustersJson against one fresh assigner per cluster, exception
    texts, and the clusters that fall back to solveTopicsJson (names that need escapes, rows of 4 and 5)."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_CLUSTERS_JSON_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
