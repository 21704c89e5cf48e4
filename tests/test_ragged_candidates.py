"""ka_solve_candidates: one ragged (real-cluster-shaped) problem against K candidate broker tables in one call. Candidate k must
give exactly what a fresh context with table k gives through ka_solve (rows, out_len, status), and the oracle's answer where
the size allows."""
import ctypes
import os
import subprocess
from unittest import mock

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from tests import util

pytestmark = pytest.mark.gpu

@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_ragged_clusters_match_sequential_and_oracle(native_lib, oracle, seed):
    rng = np.random.default_rng(seed)
    cl = kab.synth.make_ragged_cluster(T=80, N=40, R=5, max_partitions=64, seed=seed, remove_frac=0.1)
    tables = util.ragged_mixed_tables(rng, cl)
    n_ok = 0
    for desired_rf in (-1, 1, 2, 3):
        # topics without partitions fail every run without a desired RF (KTA:65-66): only with one
        prob = util.Problem(*util.sparse_with_empty_topics(cl, rng, desired_rf > 0), desired_rf)
        assert desired_rf < 0 or np.any(np.diff(prob.part_off) == 0)
        sts = util.check_equal(prob, tables, oracle)
        n_ok += sum(st[0] == 0 for st in sts)
        assert sts[-1][0] == _native.KA_ERR_RF_GT_BROKERS
        if seed == 1 and desired_rf == -1:   # the same call with every counter column in global memory
            with mock.patch.dict(os.environ, {"KA_ORDER_GLOBAL_CTR": "1"}):
                util.check_equal(prob, tables, oracle)
    assert n_ok >= 16, n_ok


def test_one_exception_per_candidate(native_lib, oracle):
    A = util.table(np.arange(1, 9, dtype=np.int32))            # solves the three topics
    B = util.table(np.arange(1, 3, dtype=np.int32))            # gamma: RF 3 > 2 brokers (KTA:67-69)
    C = util.table(np.arange(1, 4, dtype=np.int32))            # polygenelubricants: 2^31 % 3 != 0 (KAS:190-192)
    D = util.table(np.arange(1, 9, dtype=np.int32), 4)         # gamma: RF 3 over two racks (KAS:183-184)
    E = util.table(np.zeros(0, dtype=np.int32))                # alpha: no broker at all
    tables = [A, B, C, D, E]
    kinds = {}
    for tail, first in (("mismatch", _native.KA_ERR_RF_MISMATCH), ("empty", _native.KA_ERR_RF_NOT_POSITIVE)):
        prob = util.exception_problem(tail)
        sts = util.check_equal(prob, tables, oracle)
        assert sts[0][:2] == (first, 3)
        assert sts[1][:2] == (_native.KA_ERR_RF_GT_BROKERS, 2) and sts[1][3] == 3
        assert sts[2][0] == _native.KA_ERR_HASH_INDEX and sts[2][1] == 1 and sts[2][3:] == (-2, 3)
        assert sts[3][:2] == (_native.KA_ERR_UNASSIGNABLE, 2) and sts[3][2] in (11, 12, 13)   # partition ids, not ordinals
        assert sts[4][:2] == (_native.KA_ERR_RF_GT_BROKERS, 0)
        if tail == "mismatch":
            assert sts[0][2:4] == (9, 1)                                                       # partition 9 of "delta"
        for st in sts:
            kinds[st[0]] = st
    assert set(kinds) == {1, 2, 3, 4, 5}
    # the return code is the status of the lowest failing candidate
    prob = util.exception_problem(None)
    st = (kab.KaStatus * 3)()
    assert _call(kab.Solver(0), prob, [A, C, B], st) == _native.KA_ERR_HASH_INDEX
    assert st[0].code == 0 and st[1].code == _native.KA_ERR_HASH_INDEX and st[2].code == _native.KA_ERR_RF_GT_BROKERS
    assert _call(kab.Solver(0), prob, [A, D, A], st) == _native.KA_ERR_UNASSIGNABLE


def _dense_rows(cl, tables):
    import torch
    d_hash = torch.from_numpy(np.ascontiguousarray(cl.topic_hash)).cuda()
    d_cur = torch.from_numpy(np.ascontiguousarray(cl.cur)).cuda()
    K = len(tables)
    out = torch.full((K, cl.T, cl.P, cl.RF), -7, dtype=torch.int32, device="cuda")
    ln = torch.full((K, cl.T, cl.P), -7, dtype=torch.int32, device="cuda")
    sts = kab.Solver(0).solve_dense_candidates_device(tables, cl.T, d_hash.data_ptr(), cl.P, cl.RF, d_cur.data_ptr(), -1, cl.RF,
                                                      ln.data_ptr(), out.data_ptr())
    return out.cpu().numpy().reshape(K, -1, cl.RF), ln.cpu().numpy().reshape(K, -1), [util.fields(st) for st in sts]


@pytest.mark.parametrize("key", ["c2", "c3"])
def test_baseline_configs_in_the_ragged_layout_match_the_dense_batch(native_lib, key):
    cl = kab.synth.make_config(key, "mixed")
    if key == "c2":
        tables = kab.synth.decommission_tables("c2", (0.0, 0.05, 0.1, 0.2))
    else:
        rng = np.random.default_rng(3)
        ids = [np.sort(rng.choice(cl.broker_id, len(cl.broker_id) - 20, replace=False)) for _ in range(8)]
        tables = [(i, cl.rack_index[np.searchsorted(cl.broker_id, i)]) for i in ids]
    part_off, part_id, rep_off, cur = cl.ragged()
    s = kab.Solver(0)
    out, ln, sts = s.solve_ragged_candidates(tables, cl.topic_hash, part_off, part_id, rep_off, cur, -1)
    d_out, d_ln, d_sts = _dense_rows(cl, tables)
    assert [util.fields(st) for st in sts] == d_sts and all(st[0] == 0 for st in d_sts)
    assert np.array_equal(out, d_out) and np.array_equal(ln, d_ln)
    if key == "c2":   # and the sequential single solves
        util.check_equal(util.Problem(cl.topic_names, cl.topic_hash, part_off, part_id, rep_off, cur), tables)


def test_million_partition_ragged_cluster_decommission_sweep(native_lib):
    cl = kab.synth.make_ragged_cluster(T=240000, N=400, max_partitions=128, seed=11)
    assert cl.Q > 1_000_000
    tables = kab.synth.ragged_decommission_tables(cl, util.FRACS)
    sts = util.check_equal(util.Problem.of(cl), tables)
    assert all(st[0] == 0 for st in sts[:6]), sts   # up to 30 % removed; beyond, some partition may find no rack left


def _call(s, prob, tables, st, K=None, out_stride=None, T=None, part_off=None, rep_off=None, out_elems=None):
    """ka_solve_candidates through ctypes, with every argument overridable."""
    ids = np.concatenate([t[0] for t in tables]).astype(np.int32) if tables else np.zeros(1, dtype=np.int32)
    racks = np.concatenate([t[1] for t in tables]).astype(np.int32) if tables else np.zeros(1, dtype=np.int32)
    off = np.zeros(len(tables) + 1, dtype=np.int32)
    np.cumsum([len(t[0]) for t in tables], out=off[1:])
    part_off = prob.part_off if part_off is None else part_off
    rep_off = prob.rep_off if rep_off is None else rep_off
    S = prob.S if out_stride is None else out_stride
    out = np.zeros(out_elems or max(len(tables), 1) * max(int(prob.part_off[-1]), 1) * max(S, 1), dtype=np.int32)
    vp = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    return s._L.ka_solve_candidates(s._h, len(tables) if K is None else K, vp(off), vp(ids), vp(racks),
                                    len(prob.topic_hash) if T is None else T, vp(prob.topic_hash), vp(part_off), vp(prob.part_id),
                                    vp(rep_off), vp(prob.cur), prob.desired_rf, S, None, vp(out), st)


def test_ctx_is_untouched(native_lib):
    cl = kab.synth.make_ragged_cluster(T=3000, N=120, R=6, seed=21)
    half = kab.synth.make_ragged_cluster(T=1500, N=120, R=6, seed=22)
    s, fresh = kab.Solver(0), kab.Solver(0)
    for x in (s, fresh):
        x.set_brokers(cl.broker_id, cl.rack_index)
        x.solve_ragged(*util.Problem.of(half).args(), 3)   # some counters in the Context
    before = s.counters()
    util.check_equal(util.Problem.of(cl), kab.synth.ragged_decommission_tables(cl, (0.1, 0.3)), solver=s)
    assert np.array_equal(s.counters(), before) and np.array_equal(s.broker_id, cl.broker_id)
    a, al, ast = s.solve_ragged(*util.Problem.of(cl).args(), 3)
    b, bl, bst = fresh.solve_ragged(*util.Problem.of(cl).args(), 3)
    assert ast.code == bst.code == 0 and np.array_equal(a, b) and np.array_equal(al, bl)
    assert np.array_equal(s.counters(), fresh.counters())


def test_launches_do_not_depend_on_k(native_lib):
    cl = kab.synth.make_ragged_cluster(T=3000, N=120, R=6, seed=21)
    prob = util.Problem.of(cl)
    s = kab.Solver(0)
    counts = []
    for K in (1, 8):
        n0 = s.launch_count()
        prob.batched(kab.synth.ragged_decommission_tables(cl, np.linspace(0.0, 0.2, K)), solver=s)
        counts.append(s.launch_count() - n0)
    assert counts[0] == counts[1] > 0, counts


def test_arguments_and_limits(native_lib):
    cl = kab.synth.make_ragged_cluster(T=40, N=30, R=5, seed=5)
    prob = util.Problem.of(cl)
    good = [(cl.broker_id, cl.rack_index)]
    s = kab.Solver(0)
    st = (kab.KaStatus * 200)()
    assert _call(s, prob, [], st) == 0
    assert _call(s, prob, good, st, T=0) == 0
    assert _call(s, prob, good * 129, st) == _native.KA_ERR_LIMIT and st[128].code == _native.KA_ERR_LIMIT
    assert _call(s, prob, good, st, out_stride=4) == _native.KA_ERR_LIMIT
    assert _call(s, prob, good, st, out_stride=2) == _native.KA_ERR_BAD_ARG   # lists of 3
    assert _call(s, prob, good, st, out_stride=0) == _native.KA_ERR_BAD_ARG
    two = kab.synth.make_ragged_cluster(T=40, N=30, R=5, seed=5, rf_weights=(0.5, 0.5))   # lists of 1 and 2
    p2 = util.Problem.of(two)
    assert p2.S == 2 and _call(s, p2, good, st) == 0
    p3 = util.Problem(p2.names, p2.topic_hash, p2.part_off, p2.part_id, p2.rep_off, p2.cur, 3, 2)
    assert _call(s, p3, good, st) == _native.KA_ERR_BAD_ARG                      # desired RF above the stride
    unsorted = [(cl.broker_id[::-1].copy(), cl.rack_index[::-1].copy())]
    assert _call(s, prob, good + unsorted, st) == _native.KA_ERR_BAD_ARG and st[0].code == st[1].code == _native.KA_ERR_BAD_ARG
    assert _call(s, prob, good, None) == _native.KA_ERR_BAD_ARG
    # malformed offsets: the status ka_solve reports, in every candidate
    ref = kab.Solver(0)
    ref.set_brokers(*good[0])
    bad_part = prob.part_off.copy()
    bad_part[5] = bad_part[6] + 1                                                # topic 5 ends before it starts
    bad_rep = prob.rep_off.copy()
    bad_rep[7] = bad_rep[8] + 1                                                  # a list of negative size
    shifted = prob.part_off + 1
    for kw in (dict(part_off=bad_part), dict(rep_off=bad_rep), dict(part_off=shifted)):
        p_off, r_off = kw.get("part_off", prob.part_off), kw.get("rep_off", prob.rep_off)
        _, _, rst = ref.solve_ragged(prob.topic_hash, p_off, prob.part_id, r_off, prob.cur, -1, 3, check=False)
        assert rst.code == _native.KA_ERR_BAD_ARG
        assert _call(s, prob, good * 2, st, **kw) == _native.KA_ERR_BAD_ARG
        assert util.fields(st[0]) == util.fields(st[1]) == util.fields(rst), kw
    # K * ΣP at 2^31: the call-wide level table's positions are 32-bit (refused before anything is written)
    Q = (1 << 31) // 128
    big = util.Problem(["t"], prob.topic_hash[:1], np.array([0, Q], dtype=np.int64), None, np.zeros(Q + 1, dtype=np.int64),
                       np.zeros(0, dtype=np.int32), 1, 1)
    assert _call(s, big, good * 128, st, out_elems=1) == _native.KA_ERR_LIMIT and st[127].code == _native.KA_ERR_LIMIT


def test_cpp_host_mirror(native_lib):
    """host/test_candidates.cpp: KafkaTopicAssigner::solveTopicsCandidates against fresh assigners, exception texts."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_CANDIDATES_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
