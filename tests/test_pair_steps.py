"""Pair steps of the capacity-1 slot chains: two topics decided per step from one snapshot of the counters.

With capacity 1 every real broker sits in at most one partition of a topic. So partition q of topic t+1 needs, for each of
its brokers b, counter[b][slot] as it stands after topic t: the snapshot S taken before topic t, plus one if b's HOLDER h
(the one partition of topic t that holds b) gave b the slot. h's decision depends only on h's record and S, so q can
recompute it. A step reads S once, decides topic t and topic t+1 (recomputing the holders' decisions), then adds the
winners' bumps; the dummy broker (index N) that pads short rows never has a holder.

This file restates that schedule in Python (records as tests/test_schedule_model.py builds them, steps cut at launch edges,
a single-topic step at the end of an odd launch) and asserts the oracle's rows and final Context. The CUDA chains do not
run pair steps: on the H100 a pair step costs about four one-topic levels (DESIGN.md §2 B, "Pair steps"), so they would be
slower. The model pins that the recompute is exact, for any later schedule that decides several topics from one snapshot.
"""
import random

import pytest

import kafka_assigner_b200 as kab
from tests import models, util


def holders_of(recs, N, P, t):
    """For each record of topic t >= 1: per broker field, the position of that broker in topic t-1, or None."""
    pos = {}
    for i in range(P):
        a, k, _ = recs[(t - 1) * P + i]
        for b in a:
            if b != N:
                assert b not in pos, "capacity 1: a broker sits in at most one partition of a topic"
                pos[b] = i
    return [[None if b == N else pos.get(b) for b in recs[t * P + i][0]] for i in range(P)]


def slot0_pick(a, x):
    L10, L20, L21 = x[1] < x[0], x[2] < x[0], x[2] < x[1]   # strict '<' in scan order: ties to the earlier position
    return 2 if (L21 if L10 else L20) else (1 if L10 and not L21 else 0)


def slot1_pick(op, oq, e, c):
    return oq if c[oq] < c[op] + e else op


def run_pair_model(cl, sets, launches, c0, c1, c2):
    """Both slot chains as pair steps over the topic ranges `launches` (each cut into (t, t+1) steps, a single step at the
    end of an odd range). Updates the counter lists in place; returns the ordered rows (broker indices)."""
    N, P = cl.N, cl.P
    recs = models.build_records(cl, sets)
    hold = {t: holders_of(recs, N, P, t) for t in range(1, cl.T)}
    mid, out = {}, {}

    def decide0(t, i, snap):
        a, k, e = recs[t * P + i]
        return slot0_pick(a, [snap[b] for b in a])

    def decide1(t, i, snap):
        op, oq, e, oA, k = mid[t * P + i]
        return slot1_pick(op, oq, e, snap)

    for t0, t1 in launches:
        for t in range(t0, t1, 2):
            pair = t + 1 < t1
            # ---- slot 0: read phase from one snapshot, then the adds
            S = list(c0)
            win = {}   # (topic, position) -> scan position of the slot-0 winner
            for i in range(P):
                win[(t, i)] = decide0(t, i, S)
            if pair:
                for i in range(P):
                    a, k, e = recs[(t + 1) * P + i]
                    x = []
                    for j, b in enumerate(a):
                        h = hold[t + 1][i][j]
                        bump = h is not None and recs[t * P + h][0][decide0(t, h, S)] == b
                        x.append(S[b] + int(bump))
                    win[(t + 1, i)] = slot0_pick(a, x)
            for (u, i), w in win.items():
                a, k, e = recs[u * P + i]
                if k > 0:                                    # the dummy is never bumped (models.slot_chains)
                    c0[a[w]] += 1
                p_, q_ = (1, 2) if w == 0 else ((0, 2) if w == 1 else (0, 1))
                mid[u * P + i] = (a[p_], a[q_], e[{(0, 1): 0, (0, 2): 1, (1, 2): 2}[(p_, q_)]], a[w], k)
        for t in range(t0, t1, 2):
            pair = t + 1 < t1
            # ---- slot 1: the same on counter[.][1], holders' records are their slot-1 records
            S = list(c1)
            pick = {}
            for i in range(P):
                op, oq, e, oA, k = mid[t * P + i]
                pick[(t, i)] = slot1_pick(op, oq, e, S)
            if pair:
                for i in range(P):
                    op, oq, e, oA, k = mid[(t + 1) * P + i]
                    a = recs[(t + 1) * P + i][0]
                    c = {}
                    for b in (op, oq):
                        h = None if b == N else hold[t + 1][i][a.index(b)]
                        c[b] = S[b] + int(h is not None and decide1(t, h, S) == b)
                    pick[(t + 1, i)] = oq if c[oq] < c[op] + e else op
            for (u, i), o1 in pick.items():
                op, oq, e, oA, k = mid[u * P + i]
                if k > 1:
                    c1[o1] += 1
                o2 = op if o1 == oq else oq
                if k > 2:
                    c2[o2] += 1
                out[u * P + i] = [oA, o1, o2][:k]
    return out


def _sets(oracle, cl, octx):
    exp, exp_len, est = util.oracle_dense(oracle, cl, octx)
    assert est.code == 0
    exp = exp.reshape(cl.T, cl.P, -1)
    return [[[int(b) for b in exp[t, p, :exp_len[t * cl.P + p]]] for p in range(cl.P)] for t in range(cl.T)]


def _cuts(T, rng):
    """Topic ranges of the chain launches: the whole run, or cut at random points (odd ranges included)."""
    if T < 3 or rng.random() < 0.3:
        return [(0, T)]
    cuts = sorted(rng.sample(range(1, T), min(T - 1, rng.randint(1, 3))))
    edges = [0] + cuts + [T]
    return list(zip(edges[:-1], edges[1:]))


# capacity 1 everywhere: N >= P * target RF
PAIR_SHAPES = [
    dict(T=9, P=5, RF=1, N=12, R=4),                    # RF 1, odd T
    dict(T=10, P=20, RF=2, N=45, R=5),                  # RF 2, even T
    dict(T=11, P=40, RF=3, N=130, R=6),                 # RF 3, odd T
    dict(T=8, P=30, RF=3, N=95, R=5, desired_rf=2),     # rows of 2: the dummy in slot 2
    dict(T=7, P=30, RF=3, N=95, R=5, desired_rf=1),     # rows of 1: slot 1 compares the dummy against itself
    dict(T=7, P=1, RF=3, N=5, R=3),                     # P 1
    dict(T=6, P=97, RF=3, N=300, R=10),
    dict(T=4, P=256, RF=3, N=800, R=20),                # P 256
    dict(T=5, P=256, RF=2, N=513, R=9),                 # tight: nearly every broker held in every topic
]


@pytest.mark.parametrize("shape", PAIR_SHAPES, ids=lambda s: "T%d-P%d-RF%d-N%d-d%d" % (s["T"], s["P"], s["RF"], s["N"], s.get("desired_rf", -1)))
def test_pair_steps_reproduce_the_reference(oracle, shape):
    shape = dict(shape)
    desired = shape.pop("desired_rf", -1)
    rng = random.Random(shape["T"] * 1000 + shape["P"])
    for kind in ("structured", "random", "mixed"):
        cl = kab.synth.make_cluster(seed=0x9A1 + shape["P"], kind=kind, **shape)
        cl.desired_rf = desired
        octx = oracle.OracleContext()
        sets = _sets(oracle, cl, octx)
        N = cl.N
        c0, c1, c2 = [0] * N + [models.INF], [0] * N + [models.INF], [0] * (N + 1)
        out = run_pair_model(cl, sets, _cuts(cl.T, rng), c0, c1, c2)
        for t in range(cl.T):
            for p in range(cl.P):
                assert [int(cl.broker_id[i]) for i in out[t * cl.P + p]] == sets[t][p], (shape, kind, t, p)
        for i, b in enumerate(cl.broker_id):
            assert (c0[i], c1[i], c2[i]) == tuple(octx.counter(int(b), s) for s in range(3)), (shape, kind, int(b))


def test_pair_steps_carry_one_context_across_runs(oracle):
    rng = random.Random(7)
    octx = oracle.OracleContext()
    first = kab.synth.make_cluster(T=9, P=60, RF=3, N=200, R=8, seed=31, kind="mixed")
    N = first.N
    c0, c1, c2 = [0] * N + [models.INF], [0] * N + [models.INF], [0] * (N + 1)
    for seed, T in ((31, 9), (32, 6)):
        cl = kab.synth.make_cluster(T=T, P=60, RF=3, N=200, R=8, seed=seed, kind="mixed")
        assert list(cl.broker_id) == list(first.broker_id)
        sets = _sets(oracle, cl, octx)
        out = run_pair_model(cl, sets, _cuts(cl.T, rng), c0, c1, c2)
        for t in range(cl.T):
            for p in range(cl.P):
                assert [int(cl.broker_id[i]) for i in out[t * cl.P + p]] == sets[t][p], (seed, t, p)
        for i, b in enumerate(cl.broker_id):
            assert (c0[i], c1[i], c2[i]) == tuple(octx.counter(int(b), s) for s in range(3)), (seed, int(b))

