"""Chain sub-blocks of large blocks: a dense single solve cuts every staged block of at least 1 024 topics into one chain
sub-block per 512 topics (at most 16 per block; never fewer than a smaller block would get), and launches each slot chain
behind the one before it on its stream.

Each case names the plan it must reach through ka_ctx_last_order_plan (field 6 = slot-chain launches of the call: two per
sub-block), then its rows must equal the oracle's and the Context counters the per-position histogram of the oracle's rows.
Plan tuples as in test_chain_variants: (rec_kind, levels, chain threads, ring_log2, gctr, loop shape, chain launches, K).
"""
import os
from unittest import mock

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from tests import models

pytestmark = pytest.mark.gpu

SINGLE, FULL = 2, 3


def _device_solve(s, cl):
    """ka_solve_dense_device on device copies of the cluster's inputs; returns (rows, lengths, status)."""
    import torch
    d_hash, d_cur = torch.from_numpy(cl.topic_hash).cuda(), torch.from_numpy(cl.cur).cuda()
    d_out = torch.full((cl.T, cl.P, cl.RF), -7, dtype=torch.int32, device="cuda")
    d_len = torch.full((cl.T, cl.P), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    st = s.solve_dense_device(cl.T, d_hash.data_ptr(), cl.P, cl.RF, d_cur.data_ptr(), -1, cl.RF, d_len.data_ptr(), d_out.data_ptr())
    torch.cuda.synchronize()
    return d_out.cpu().numpy().reshape(-1, cl.RF), d_len.cpu().numpy().reshape(-1), st


def test_c3_device_solve_cuts_large_blocks(native_lib, oracle):
    """BASELINE config 3 (10 000 topics x 128 partitions): 4 staged blocks of 2 500 topics, 4 chain sub-blocks each (2 before
    the large-block rule)."""
    cl = kab.synth.make_config("c3", "mixed")
    exp, exp_len, est = oracle.fast_run_dense(oracle.FastContext(), cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index)
    assert est.code == 0
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    out, out_len, st = _device_solve(s, cl)
    assert st.code == 0
    assert s.last_order_plan() == (3, 0, 128, 10, 0, FULL, 2 * 4 * 4, 0)
    assert np.array_equal(out, exp) and np.array_equal(out_len, exp_len)
    assert np.array_equal(s.counters(), models.histogram(cl.broker_id, exp, exp_len))


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_one_context_across_two_large_solves(native_lib, oracle, device):
    """Two pipelined solves of 4 096 topics (2 blocks of 2 048 topics, 4 sub-blocks each) through one Context: the second
    starts from the counters the first left, as the oracle's Context does."""
    s = kab.Solver(0)
    fctx = oracle.FastContext()
    total = None
    for i in range(2):
        cl = kab.synth.make_cluster(T=4096, P=64, RF=3, N=300, R=12, seed=0x5C0 + i, kind="mixed")
        exp, exp_len, est = oracle.fast_run_dense(fctx, cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index)
        assert est.code == 0
        if device:
            if i == 0:
                s.set_brokers(cl.broker_id, cl.rack_index)
            out, out_len, st = _device_solve(s, cl)
        else:
            out, out_len, st = s.solve_cluster(cl, check=False)
            out, out_len = out.reshape(-1, cl.RF), out_len.reshape(-1)
        assert st.code == 0, i
        assert s.last_order_plan() == (3, 0, 64, 10, 0, FULL, 2 * 2 * 4, 0), i
        assert np.array_equal(out, exp) and np.array_equal(out_len, exp_len), i
        h = models.histogram(cl.broker_id, exp, exp_len)
        total = h if total is None else total + h
        assert np.array_equal(s.counters(), total), i


LIMIT_CASES = [
    # one block of 8 192 topics: exactly 16 sub-blocks of 512; 12 000 topics would take 23: clipped to the limit
    dict(id="t8192", T=8192, P=16, env={}, plan=(3, 0, 32, 10, 0, 1, 32, 0)),
    dict(id="t12000", T=12000, P=16, env={}, plan=(3, 0, 32, 10, 0, 1, 32, 0)),
    # the override, above the limit, on a block too small for the large-block rule
    dict(id="override40", T=301, P=40, env={"KA_CHAIN_SUBBLOCKS": "40"}, plan=(3, 0, 64, 10, 0, SINGLE, 32, 0)),
]


@pytest.mark.parametrize("case", LIMIT_CASES, ids=[c["id"] for c in LIMIT_CASES])
def test_subblock_limit(native_lib, oracle, case):
    cl = kab.synth.make_cluster(T=case["T"], P=case["P"], RF=3, N=200, R=10, seed=0x5C10 + case["T"], kind="mixed")
    exp, exp_len, est = oracle.fast_run_dense(oracle.FastContext(), cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index)
    assert est.code == 0
    s = kab.Solver(0)
    with mock.patch.dict(os.environ, case["env"]):
        out, out_len, st = s.solve_cluster(cl, check=False)
    assert st.code == 0
    assert s.last_order_plan() == case["plan"]
    assert np.array_equal(out.reshape(-1, 3), exp) and np.array_equal(out_len.reshape(-1), exp_len)
    assert np.array_equal(s.counters(), models.histogram(cl.broker_id, exp, exp_len))
