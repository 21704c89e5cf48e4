"""ka_solve_dense_candidates_device: one cluster against K candidate broker tables in one call. Candidate k must give exactly
what a fresh context with table k gives through ka_solve_dense_device (rows, out_len, status), and the oracle's answer where
the size allows."""
import ctypes
import os
from unittest import mock

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from tests import util

pytestmark = pytest.mark.gpu

DECOMMISSION_FRACS = (0.01, 0.02, 0.05, 0.10, 0.20, 0.30, 0.40, 0.50)


def _mixed_tables(rng, cl):
    old = cl.broker_id
    return [
        util.table(np.sort(rng.choice(old, len(old) - 3, replace=False)), 2),                  # capacity > 1, racks
        util.table(np.sort(rng.choice(old, len(old) - 5, replace=False))),                     # capacity > 1, no racks
        util.table(np.arange(1000, 1000 + 4000, dtype=np.int32), 40),                          # capacity 1, racks
        util.table(np.arange(900, 900 + 3000, dtype=np.int32)),                                # capacity 1, no racks
        util.table(1000 + 2 * np.arange(20000, dtype=np.int32), 500),                          # 20 000 brokers, global id LUT
    ]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_dense_clusters_match_sequential_and_oracle(native_lib, oracle, seed):
    rng = np.random.default_rng(seed)
    for RF, desired_rf in ((1, -1), (2, -1), (3, -1), (2, 3), (3, 2), (1, 2)):
        cl = kab.synth.make_cluster(T=40, P=16, RF=RF, N=24, R=4, seed=seed * 101 + RF, kind="mixed")
        prob = util.DenseProblem(cl.topic_hash, cl.cur, desired_rf)
        tables = _mixed_tables(rng, cl)
        util.check_dense_equal(prob, tables, oracle)
        if RF == 3 and desired_rf == -1:   # the same call with every counter column in global memory
            with mock.patch.dict(os.environ, {"KA_ORDER_GLOBAL_CTR": "1"}):
                util.check_dense_equal(prob, tables, oracle)


def test_baseline_c2_k4(native_lib, oracle):
    cl = kab.synth.make_config("c2", "mixed")
    tables = kab.synth.decommission_tables("c2", (0.0, 0.05, 0.1, 0.2))
    util.check_dense_equal(util.DenseProblem(cl.topic_hash, cl.cur), tables, oracle)


def test_baseline_c3_k8(native_lib):
    cl = kab.synth.make_config("c3", "mixed")
    rng = np.random.default_rng(3)
    tables = [(np.sort(rng.choice(cl.broker_id, len(cl.broker_id) - 20, replace=False)),) for _ in range(8)]
    tables = [(ids, cl.rack_index[np.searchsorted(cl.broker_id, ids)]) for (ids,) in tables]
    assert all(st[0] == 0 for st in util.check_dense_equal(util.DenseProblem(cl.topic_hash, cl.cur), tables))


def test_baseline_c5_decommission_sweep(native_lib):
    cl = kab.synth.make_config("c5", "mixed")
    tables = kab.synth.decommission_tables("c5", DECOMMISSION_FRACS)
    assert all(st[0] == 0 for st in util.check_dense_equal(util.DenseProblem(cl.topic_hash, cl.cur), tables))


def test_per_candidate_failures(native_lib):
    cl = kab.synth.make_cluster(T=30, P=12, RF=3, N=24, R=4, seed=77, kind="mixed")
    good = (cl.broker_id, cl.rack_index)
    too_small = util.table(cl.broker_id[:2], 1)                 # fewer brokers than RF
    two_racks = util.table(cl.broker_id, 12)                    # RF 3 over two racks
    tables = [good, too_small, good, two_racks, util.table(np.zeros(0, dtype=np.int32)), good]
    prob = util.DenseProblem(cl.topic_hash, cl.cur)
    sts = util.check_dense_equal(prob, tables)
    assert sts[1][0] == _native.KA_ERR_RF_GT_BROKERS and sts[3][0] == _native.KA_ERR_UNASSIGNABLE
    assert sts[0][0] == sts[2][0] == sts[5][0] == 0
    # return code: the status of the lowest failing candidate
    st = (kab.KaStatus * len(tables))()
    rc = _call(kab.Solver(0), prob, tables, st)
    assert rc == _native.KA_ERR_RF_GT_BROKERS


def _call(s, prob, tables, st, K=None, out_stride=None, T=None):
    import torch
    ids = np.concatenate([t[0] for t in tables]).astype(np.int32) if tables else np.zeros(1, dtype=np.int32)
    racks = np.concatenate([t[1] for t in tables]).astype(np.int32) if tables else np.zeros(1, dtype=np.int32)
    off = np.zeros(len(tables) + 1, dtype=np.int32)
    np.cumsum([len(t[0]) for t in tables], out=off[1:])
    S = out_stride or prob.S
    out = torch.empty((max(len(tables), 1), prob.T, prob.P, max(S, 1)), dtype=torch.int32, device="cuda")
    return s._L.ka_solve_dense_candidates_device(
        s._h, len(tables) if K is None else K, off.ctypes.data_as(ctypes.c_void_p), ids.ctypes.data_as(ctypes.c_void_p),
        racks.ctypes.data_as(ctypes.c_void_p), prob.T if T is None else T, ctypes.c_void_p(prob.d_hash.data_ptr()), prob.P, prob.RF,
        ctypes.c_void_p(prob.d_cur.data_ptr()), prob.desired_rf, S, None, ctypes.c_void_p(out.data_ptr()), None, st)


def test_ctx_is_untouched(native_lib):
    cl = kab.synth.make_config("c2", "mixed")
    half = kab.synth.make_cluster(**dict(kab.synth.CONFIGS["c2"], T=500), kind="mixed")
    s, fresh = kab.Solver(0), kab.Solver(0)
    for x in (s, fresh):
        x.set_brokers(cl.broker_id, cl.rack_index)
        x.solve_dense(half.topic_hash, half.cur)   # some counters in the Context
    before = s.counters()
    prob = util.DenseProblem(cl.topic_hash, cl.cur)
    prob.batched(kab.synth.decommission_tables("c2", (0.1, 0.3)), solver=s)
    assert np.array_equal(s.counters(), before) and np.array_equal(s.broker_id, cl.broker_id)
    a, al, ast = s.solve_dense(cl.topic_hash, cl.cur)
    b, bl, bst = fresh.solve_dense(cl.topic_hash, cl.cur)
    assert ast.code == bst.code == 0 and np.array_equal(a, b) and np.array_equal(al, bl)
    assert np.array_equal(s.counters(), fresh.counters())


def test_launches_do_not_depend_on_k(native_lib):
    cl = kab.synth.make_config("c2", "mixed")
    prob = util.DenseProblem(cl.topic_hash, cl.cur)
    s = kab.Solver(0)
    counts = []
    for K in (1, 8):
        n0 = s.launch_count()
        prob.batched(kab.synth.decommission_tables("c2", np.linspace(0.0, 0.2, K)), solver=s)
        counts.append(s.launch_count() - n0)
    assert counts[0] == counts[1] > 0, counts


def test_arguments(native_lib):
    cl = kab.synth.make_cluster(T=10, P=8, RF=3, N=12, R=4, seed=5, kind="mixed")
    prob = util.DenseProblem(cl.topic_hash, cl.cur)
    good = [(cl.broker_id, cl.rack_index)]
    s = kab.Solver(0)
    st = (kab.KaStatus * 200)()
    assert _call(s, prob, [], st) == 0
    assert _call(s, prob, good, st, T=0) == 0
    assert _call(s, prob, good * 129, st) == _native.KA_ERR_LIMIT and st[128].code == _native.KA_ERR_LIMIT
    assert _call(s, prob, good, st, out_stride=4) == _native.KA_ERR_LIMIT
    assert _call(s, prob, good, st, out_stride=2) == _native.KA_ERR_BAD_ARG
    unsorted = [(cl.broker_id[::-1].copy(), cl.rack_index[::-1].copy())]
    assert _call(s, prob, good + unsorted, st) == _native.KA_ERR_BAD_ARG and st[0].code == st[1].code == _native.KA_ERR_BAD_ARG
    assert _call(s, prob, good, None) == _native.KA_ERR_BAD_ARG
