"""CPU model of the round-2 leader-order design, checked against the structure-faithful oracle (no GPU needed).

The CUDA path replaces the reference's single pass over all partitions (KafkaAssignmentStrategy.java:217-237, one shared
`Context.counter`) by
  1. a per-topic CONFLICT-LEVEL schedule (partitions of one level share no broker; levels run in order, topics one after the other),
  2. records that list a row's brokers in the order the reference's rotated scan visits them (KAS:263-278, 188-200) plus the
     precomputed tie-breaks e_pq of the slot-1 scan, short rows padded with a dummy broker whose counters are "infinite",
  3. ONE CHAIN PER REPLICA SLOT: slot 0 only reads/bumps counter[.][0], slot 1 counter[.][1] (given the slot-0 winner), and
     counter[.][2] is a plain sum for rows of <= 3 replicas.
tests/models.py (build_records, slot_chains) restates exactly that in Python — the same record layout and decision rules as
kassign_stage.cuh / kassign_order.cuh — and this file asserts that it reproduces the oracle's ordered lists AND its final
Context, even when the partitions of a level are processed in a scrambled order and the whole slot-0 chain runs before the
slot-1 chain starts.
"""
import random

import pytest

import kafka_assigner_b200 as kab
from tests import models, util


def run_model(cl, sets, rng):
    N = cl.N
    c0, c1, c2 = [0] * N + [models.INF], [0] * N + [models.INF], [0] * (N + 1)
    out = models.slot_chains(cl, sets, rng, c0, c1, c2)
    return out, c0, c1, c2


@pytest.mark.parametrize("shape", [dict(T=30, P=24, RF=3, N=40, R=5), dict(T=12, P=90, RF=3, N=60, R=6),      # capacity 2 / 5: levels
                                   dict(T=40, P=16, RF=3, N=120, R=6), dict(T=25, P=20, RF=2, N=30, R=5),   # capacity 1; RF 2
                                   dict(T=50, P=9, RF=1, N=12, R=4), dict(T=10, P=8, RF=3, N=6, R=3, n_old=6)])
def test_level_schedule_and_per_slot_chains_reproduce_the_reference(oracle, shape):
    rng = random.Random(1234)
    ran = 0
    for kind in ("structured", "random", "mixed"):
        cl = kab.synth.make_cluster(seed=0x51D + shape["T"], kind=kind, **shape)
        octx = oracle.OracleContext()
        exp, exp_len, est = util.oracle_dense(oracle, cl, octx)
        if est.code != 0:
            continue
        exp = exp.reshape(cl.T, cl.P, -1)
        sets = [[[int(b) for b in exp[t, p, :exp_len[t * cl.P + p]]] for p in range(cl.P)] for t in range(cl.T)]
        out, c0, c1, c2 = run_model(cl, sets, rng)
        for t in range(cl.T):
            for p in range(cl.P):
                got = [int(cl.broker_id[i]) for i in out[t * cl.P + p]]
                assert got == sets[t][p], (shape, kind, t, p)
        for i, b in enumerate(cl.broker_id):
            assert (c0[i], c1[i], c2[i]) == tuple(octx.counter(int(b), s) for s in range(3)), (shape, kind, int(b))
        ran += 1
    assert ran >= 1, shape
