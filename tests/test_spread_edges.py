"""The orphan spread of kernel A (KAS:133-186) on inputs that leave many replicas without a broker.

The spread places every orphan replica first-fit in the topic's rotated broker order, scanning 32 order positions per warp
step. These cases put the first feasible broker on every side of those windows: tables of 31 .. 2 049 brokers and one near
kernel A's shared-memory budget, rotations next to the wrap, racks that exclude whole windows, partitions that cannot be
placed, with no orphans placed until far into the order. Each case names the kernel A instantiation it must reach (load
bytes, levels, SM, batched), checked through ka_ctx_last_stage_plan; its rows, list lengths and full status must equal the
oracle's and, for single solves, the Context counters the oracle's rows give.
"""
import numpy as np
import pytest

import kafka_assigner_b200 as kab
from tests import models, util

pytestmark = pytest.mark.gpu

INT_MIN = -2**31


def _racks(N, R, contiguous=False):
    """Rack index of each of N brokers: R racks, interleaved (i % R) or in contiguous runs; R = None: no broker has a rack."""
    if R is None:
        return None
    return [i // -(-N // R) if contiguous else i % R for i in range(N)]


def _table(N, R, contiguous=False):
    ids = 1000 + np.arange(N, dtype=np.int32)
    rk = _racks(N, R, contiguous)
    return util.table(ids) if rk is None else (ids, kab.synth.rack_indices(ids, ["k%d" % r for r in rk]))


def _orphan_heavy(T, P, RF, ids, seed, keep=0.25):
    """Current lists [T, P, RF]: a quarter of the replicas on brokers of the table, the rest on ids outside it (orphans)."""
    rng = np.random.default_rng(seed)
    live = rng.choice(ids, size=(T, P, RF))
    dead = (int(ids[-1]) + 1 + rng.integers(0, 1000, size=(T, P, RF))).astype(np.int32)
    return np.where(rng.random((T, P, RF)) < keep, live, dead).astype(np.int32)


def _hashes(T, N, seed):
    """Topic hashes whose rotation i0 = (N - |h| % N) % N puts order position 0 at the first and last brokers, around every
    word edge and at random; one Integer.MIN_VALUE."""
    rng = np.random.default_rng(seed)
    i0s = [0, 1, N - 1, N - 2, 31 % N, 32 % N, 33 % N, (N - 32) % N, (N - 33) % N]
    h = [(N - i) % N for i in i0s] + list(rng.integers(-2**31 + 1, 2**31 - 1, size=max(T - len(i0s) - 1, 0)))
    h = (h + [INT_MIN])[:T]
    return np.array(h, dtype=np.int64).astype(np.int32)


def _check_single(oracle, s, th, cur, table, plan, desired=-1, S=None):
    ids, racks = table
    S = S or max(cur.shape[2], desired, 1)
    exp, exp_len, est = oracle.fast_run_dense(oracle.FastContext(), th, cur, ids, racks, desired, S)
    s.reset()
    s.set_brokers(ids, racks)
    out, ln, st = s.solve_dense(th, cur, desired, S, check=False)
    assert s.last_stage_plan()[:4] == plan, (s.last_stage_plan(), plan)
    assert util.fields(st) == util.fields(est), (util.fields(st), util.fields(est))
    if est.code == 0:
        assert np.array_equal(out.reshape(-1, S), exp)
        assert np.array_equal(ln.reshape(-1), exp_len)
        assert np.array_equal(s.counters(), models.histogram(ids, exp, exp_len))
    return util.fields(st)


# (N, R, contiguous racks): one window, window and 1 024-broker edges, many windows; racks that exclude whole windows; no racks
TABLES = [(31, 5, False), (32, 4, True), (33, 6, False), (1023, 10, False), (1024, 8, True), (1025, None, False),
          (2049, 7, False), (2049, 3, True)]


@pytest.mark.parametrize("N,R,contiguous", TABLES)
def test_capacity_one(native_lib, oracle, N, R, contiguous):
    """Capacity 1 (1-byte loads, no levels)."""
    table = _table(N, R, contiguous)
    T, RF = 24, 3
    P = max(1, N // RF)
    cur = _orphan_heavy(T, P, RF, table[0], seed=N)
    _check_single(oracle, kab.Solver(0), _hashes(T, N, N), cur, table, (1, 0, 3, 0))


@pytest.mark.parametrize("N,R,contiguous", TABLES)
def test_capacity_above_one(native_lib, oracle, N, R, contiguous):
    """Capacity 3 (levels): a broker stays feasible until its load reaches the capacity."""
    table = _table(N, R, contiguous)
    T, RF = 12, 3
    cur = _orphan_heavy(T, N, RF, table[0], seed=N + 1)
    _check_single(oracle, kab.Solver(0), _hashes(T, N, N + 1), cur, table, (1, 1, 3, 0))


def test_two_byte_loads(native_lib, oracle):
    """Capacity 273 on 33 brokers: 2-byte loads."""
    table = _table(33, 11)
    cur = _orphan_heavy(2, 3000, 3, table[0], seed=7)
    _check_single(oracle, kab.Solver(0), _hashes(2, 33, 7), cur, table, (2, 1, 3, 0))


@pytest.mark.parametrize("N", [33, 1025])
def test_rows_of_five(native_lib, oracle, N):
    """Rows of 5 (SM 8), and rows of 2 grown to 3 (short current lists)."""
    table = _table(N, 7)
    cur = _orphan_heavy(10, 200, 5, table[0], seed=N + 2)
    _check_single(oracle, kab.Solver(0), _hashes(10, N, N + 2), cur, table, (1, int(-(-200 * 5 // N) > 1), 8, 0))
    cur = _orphan_heavy(10, 200, 2, table[0], seed=N + 3)
    _check_single(oracle, kab.Solver(0), _hashes(10, N, N + 3), cur, table, (1, int(-(-200 * 3 // N) > 1), 3, 0), desired=3)


def test_near_budget(native_lib, oracle):
    """60 000 brokers (a global id LUT): one warp per CTA, 1 875 windows per scan."""
    N = 60000
    table = (1000 + 2 * np.arange(N, dtype=np.int32), np.arange(N, dtype=np.int32) % 9)
    cur = _orphan_heavy(6, 400, 3, table[0], seed=11)
    _check_single(oracle, kab.Solver(0), _hashes(6, N, 11), cur, table, (1, 0, 3, 0))


@pytest.mark.parametrize("N", [33, 1025, 2049])
def test_unassignable(native_lib, oracle, N):
    """Racks 0 (all brokers but two), 1 and 2: the first orphan partition takes the two single-broker racks, the next one
    falls short. Those two brokers are the table's last, so the shortfall shows only at the end of the scan."""
    ids = 1000 + np.arange(N, dtype=np.int32)
    racks = np.zeros(N, dtype=np.int32)
    racks[-2], racks[-1] = 1, 2
    cur = np.full((3, 8, 3), 10**6, dtype=np.int32)   # every replica an orphan
    st = _check_single(oracle, kab.Solver(0), np.array([5, 17, 3], dtype=np.int32), cur, (ids, racks), (1, 0, 3, 0))
    assert st[:3] == (4, 0, 1), st


def test_wrap_edges(native_lib, oracle):
    """All brokers but one rack full from the sticky fill: the only feasible brokers sit right before and after the wrap of
    each topic's rotated order."""
    N, R = 1025, 5
    table = _table(N, R)
    T, RF = 40, 1
    P = N // RF
    rng = np.random.default_rng(5)
    cur = np.empty((T, P, RF), dtype=np.int32)
    for t in range(T):
        cur[t, :, 0] = rng.permutation(table[0])[:P]
        cur[t, rng.integers(0, P, size=3), 0] = 10**6   # three orphans, a few free brokers
    _check_single(oracle, kab.Solver(0), _hashes(T, N, 5), cur, table, (1, 0, 3, 0))


def test_candidates_of_different_sizes(native_lib, oracle):
    """The batched instantiation (CAND) on candidate tables of 33, 1 025 and 2 049 brokers."""
    tables = [_table(33, 6), _table(1025, 8, True), _table(2049, None)]
    cur = _orphan_heavy(20, 10, 3, np.concatenate([t[0] for t in tables]), seed=21, keep=0.5)
    prob = util.DenseProblem(_hashes(20, 33, 21), cur)
    s = kab.Solver(0)
    util.check_dense_equal(prob, tables, oracle, solver=s)
    assert s.last_stage_plan()[:4] == (1, 0, 3, 3), s.last_stage_plan()


def test_clusters_of_different_sizes(native_lib):
    """The batched instantiation on a fleet of clusters of 31, 1 024 and 2 049 brokers, each against a fresh context."""
    fleet = []
    for k, (N, R, contiguous) in enumerate([(31, 5, False), (1024, 8, True), (2049, 7, False)]):
        table = _table(N, R, contiguous)
        T, P, RF = 8, max(1, N // 3), 3
        cur = _orphan_heavy(T, P, RF, table[0], seed=30 + k)
        part_off = np.arange(T + 1, dtype=np.int64) * P
        rep_off = np.arange(T * P + 1, dtype=np.int64) * RF
        part_id = np.tile(np.arange(P, dtype=np.int32), T)
        fleet.append(util.Member(table, ["t%d" % t for t in range(T)], _hashes(T, N, 30 + k), part_off, part_id, rep_off,
                                 cur.reshape(-1)))
    s = kab.Solver(0)
    res = s.solve_clusters([m.entry() for m in fleet], out_stride=3)
    assert s.last_stage_plan()[:4] == (1, 1, 3, 3), s.last_stage_plan()
    ref = kab.Solver(0)
    for k, (m, (out, ln, st)) in enumerate(zip(fleet, res)):
        e_out, e_len, e_st = m.sequential(ref, 3)
        assert util.fields(st) == e_st, (k, util.fields(st), e_st)
        if e_st[0] == 0:
            assert np.array_equal(out, e_out) and np.array_equal(ln, e_len), k
