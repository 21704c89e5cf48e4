"""ka_wave_broker_usage on the device: every field of every table entry, and W, must equal `usage_models` (the plain loop on small
cases, its numpy form on large ones) for plans of ka_plan_waves and ka_plan_waves_send, hand-made waves at the radix passes'
boundaries, tables of 0, 1 and 65535 brokers, one broker with more than 10^6 events, the 1.06 M-partition cluster, and every
refusal; the Context is untouched, the launches depend on bit lengths only, and the C++ mirror agrees with Solver.broker_usage."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from tests import usage_models, util

pytestmark = pytest.mark.gpu
BAD, LIMIT = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT
FIELDS = usage_models.FIELDS


def check(s, rep_off, cur, out, out_len, wave, ids, weight=None, base=None, cap=None, loop=False):
    """Solver.broker_usage against the model (the loop with `loop`, else its numpy form); returns the report."""
    usage, W, st = s.broker_usage(rep_off, cur, out, out_len, wave, ids, weight=weight, base=base, capacity=cap)
    assert (st.code, st.a, st.b) == (0, 0, 0), (st.code, st.a, st.b)
    if loop:
        e, e_W, e_st = usage_models.broker_usage(rep_off, cur, out, out_len, wave, ids, weight, base, cap)
        assert e_st == (0, 0, 0) and W == e_W
        assert [{f: int(x[f]) for f in FIELDS} for x in usage] == e
    else:
        e, e_W = usage_models.broker_usage_np(rep_off, cur, out, out_len, wave, ids, weight, base, cap)
        assert W == e_W
        for f in FIELDS:
            assert np.array_equal(usage[f], e[f]), (f, np.nonzero(usage[f] != e[f])[0][:10])
    return usage


@pytest.mark.parametrize("remove", [0.0, 0.03])
def test_plans_of_a_solved_cluster(native_lib, remove):
    cl = kab.synth.make_ragged_cluster(T=4000, N=400, max_partitions=128, seed=17, remove_frac=remove)
    s, out, out_len, S = util.solved(cl)
    Q = len(out_len)
    rng = np.random.default_rng(5)
    weight = rng.integers(0, 1 << 30, Q).astype(np.int64)
    ids = cl.all_broker_id
    n = len(ids)
    for B, w, send in ((1, None, None), (4, None, 2), (8 * int(weight.mean()), weight, None), (int(weight.mean()), weight, 3)):
        kw = {} if send is None else dict(max_broker_out=send * (1 if w is None else int(weight.mean())), send_brokers=ids)
        wave, summ, st = s.plan_waves(cl.rep_off, cl.cur, out, out_len, B, weight=w, **kw)
        assert st.code == 0 and len(summ) > 1
        usage = check(s, cl.rep_off, cl.cur, out, out_len, wave, ids, w)
        mean = int(usage["before"].mean())
        base = rng.integers(0, max(mean, 1), n).astype(np.int64)
        cap = (usage["peak"] + base - rng.integers(-2, 3, n)).astype(np.int64).clip(0)
        usage = check(s, cl.rep_off, cl.cur, out, out_len, wave, ids, w, base, cap)
        assert (usage["over_wave"] >= 0).any() and (usage["over_wave"] < 0).any()
        # the plan reordered: waves reversed
        W = int(wave.max())
        check(s, cl.rep_off, cl.cur, out, out_len, np.where(wave > 0, W + 1 - wave, 0), ids, w, base, cap)
    # the whole solve as one document
    one = check(s, cl.rep_off, cl.cur, out, out_len, (s.plan_waves(cl.rep_off, cl.cur, out, out_len, 1 << 40)[0] > 0).astype(np.int32), ids)
    assert (one["peak"] >= one["after"]).all()


@pytest.mark.parametrize("seed", range(6))
def test_small_cases_against_the_loop(native_lib, seed):
    rng = np.random.default_rng(40 + seed)
    N, Q = 16, int(rng.integers(1, 700))
    cur_l, new_l = util.random_wave_case(rng, Q, N)
    for g in range(Q):
        if cur_l[g] and rng.random() < 0.2:
            cur_l[g] = cur_l[g] + [cur_l[g][0], 99]   # a duplicate and an id outside the table
    rep_off, cur = util.cur_lists(cur_l)
    out, out_len = util.rows(new_l, 3)
    wave = rng.integers(0, 12, Q).astype(np.int32)
    ids = np.arange(1, N + 1, dtype=np.int32)
    s = kab.Solver(0)
    weight = rng.integers(0, 100, Q).astype(np.int64) if seed % 2 else None
    base = rng.integers(0, 50, N).astype(np.int64) if seed % 3 else None
    cap = rng.integers(0, 300, N).astype(np.int64) if seed != 1 else None
    check(s, rep_off, cur, out, out_len, wave, ids, weight, base, cap, loop=True)
    check(s, rep_off, cur, out, out_len, wave, ids, weight, base, cap)


@pytest.mark.parametrize("W", [1, 254, 255, 256, 65534, 65535, 65536, (1 << 24) - 1, 1 << 24, (1 << 31) - 1])
def test_waves_at_radix_boundaries(native_lib, W):
    """Waves up to W (W + 1 on the drops' side) across the 8-bit passes, rows on CTA edges, a table of 3 brokers."""
    rng = np.random.default_rng(W % 1000)
    s = kab.Solver(0)
    for Q in (255, 256, 257, 513):
        cur_l = [[1 + g % 3] for g in range(Q)]
        new_l = [[1 + (g + 1) % 3] if g % 4 else [1 + g % 3] for g in range(Q)]
        rep_off, cur = util.cur_lists(cur_l)
        out, out_len = util.rows(new_l)
        wave = rng.integers(0, W + 1, Q).astype(np.int32)
        wave[Q - 1] = W
        weight = rng.integers(1, 10, Q).astype(np.int64)
        usage = check(s, rep_off, cur, out, out_len, wave, [1, 2, 3], weight, cap=np.array([Q, Q // 2, Q], dtype=np.int64) * 2)
        assert (usage["peak_wave"] <= W).all()


@pytest.mark.parametrize("n_use", [0, 1, 2, 256, 257, 65535])
def test_table_sizes(native_lib, n_use):
    rng = np.random.default_rng(n_use)
    ids = np.sort(rng.choice(1 << 20, n_use, replace=False)).astype(np.int32) if n_use > 2 else np.arange(1, n_use + 1, dtype=np.int32)
    s = kab.Solver(0)
    Q = 20000
    pool = ids if n_use else np.array([7, 8, 9], dtype=np.int32)
    cur_l = [[int(x)] for x in rng.choice(pool, Q)]
    new_l = [[c[0]] if n_use == 0 else [int(rng.choice(ids))] for c in cur_l]
    rep_off, cur = util.cur_lists(cur_l)
    out, out_len = util.rows(new_l)
    wave = rng.integers(0, 300, Q).astype(np.int32)
    base = rng.integers(0, 5, n_use).astype(np.int64)
    usage = check(s, rep_off, cur, out, out_len, wave, ids, base=base, cap=base + 40)
    assert len(usage) == n_use


def test_one_broker_with_a_million_events(native_lib):
    """Broker 1 drains 1.1 M rows and broker 2 receives them, over 5000 waves: one segment of 1.1 M events each."""
    Q = 1_100_000
    rep_off = np.arange(Q + 1, dtype=np.int64)
    cur = np.ones(Q, dtype=np.int32)
    out, out_len = np.full((Q, 1), 2, dtype=np.int32), np.ones(Q, dtype=np.int32)
    wave = (1 + np.arange(Q) % 5000).astype(np.int32)
    rng = np.random.default_rng(1)
    weight = rng.integers(0, 1000, Q).astype(np.int64)
    s = kab.Solver(0)
    usage = check(s, rep_off, cur, out, out_len, wave, [1, 2, 3], weight, cap=np.array([10 ** 12, int(weight.sum()) // 3, 0]))
    assert usage["before"][0] == usage["peak"][0] == weight.sum() and usage["after"][0] == 0
    assert usage["after"][1] == weight.sum() and usage["over_wave"][1] > 0


def test_nothing_to_run(native_lib):
    s = kab.Solver(0)
    empty = np.zeros(0, dtype=np.int32)
    usage, W, st = s.broker_usage([0], empty, np.zeros((0, 2), dtype=np.int32), empty, empty, [3, 5], base=[4, 9], capacity=[5, 5])
    assert st.code == 0 and W == 0
    assert [list(x) for x in usage] == [[4, 4, 0, 4, -1], [9, 9, 0, 9, 0]]
    rep_off, cur = util.cur_lists([[1, 2], [3], [], [2, 2]])
    out, out_len = util.rows([[1, 2], [3], [], [2]])
    check(s, rep_off, cur, out, out_len, np.zeros(4, dtype=np.int32), [1, 2, 3], base=[1, 1, 1], cap=[2, 2, 2], loop=True)
    check(s, rep_off, cur, out, out_len, np.array([0, 3, 0, 0], dtype=np.int32), [1, 2, 3], loop=True)


def _raw(s, Q, rep_off, cur, stride, new_len, new, weight, wave, n_use, use_id, base, cap, usage, n=None):
    st = kab.KaStatus()
    n = ctypes.c_int32(-7) if n is None else n
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = s._L.ka_wave_broker_usage(s._h, Q, p(rep_off), p(cur), stride, p(new_len), p(new), p(weight), p(wave), n_use, p(use_id),
                                   p(base), p(cap), p(usage), ctypes.byref(n) if n is not False else None, ctypes.byref(st))
    return rc, st, n


def test_errors(native_lib):
    s = kab.Solver(0)
    rng = np.random.default_rng(4)
    Q = 1000
    cur_l, new_l = util.random_wave_case(rng, Q, 20)
    rep_off, cur = util.cur_lists(cur_l)
    out, out_len = util.rows(new_l, 3)
    wave = rng.integers(0, 9, Q).astype(np.int32)
    ids = np.arange(1, 21, dtype=np.int32)
    usage = np.zeros(20, dtype=kab.assigner.BROKER_USAGE_DTYPE)
    keys = ("s", "Q", "rep_off", "cur", "stride", "new_len", "new", "weight", "wave", "n_use", "use_id", "base", "cap", "usage")
    ok = (s, Q, rep_off, cur, 3, out_len, out, None, wave, 20, ids, None, None, usage)

    def call(n=None, **kw):
        a = dict(zip(keys, ok))
        a.update(kw)
        rc, st, n = _raw(*a.values(), n=n)
        assert rc == st.code
        if n is not False:
            assert n.value == (int(a["wave"].max()) if rc == 0 else 0)
        return rc, st.a, st.b

    assert call() == (0, 0, 0)
    neg = np.array([-1] + [0] * 19, dtype=np.int64)
    # argument errors, then limits, then the table's order, then signs, then rows, then the sums
    assert call(Q=-1)[0] == BAD and call(stride=0, n_use=70000)[0] == BAD and call(n_use=-1)[0] == BAD
    assert call(usage=None)[0] == BAD and call(n=False)[0] == BAD and call(wave=None)[0] == BAD and call(use_id=None)[0] == BAD
    assert call(rep_off=rep_off + 1)[0] == BAD and call(cur=None)[0] == BAD and call(new=None, n_use=70000)[0] == BAD
    assert call(stride=9, new=np.full((Q, 9), -1, dtype=np.int32), use_id=ids[::-1].copy())[:2] == (LIMIT, 9)
    many = np.arange(1, 65537, dtype=np.int32)
    assert call(n_use=65536, use_id=many, usage=np.zeros(65536, dtype=usage.dtype), weight=np.full(Q, -1))[:2] == (LIMIT, 65536)
    assert call(use_id=ids[::-1].copy(), base=neg)[0] == BAD
    dup = ids.copy()
    dup[5] = dup[4]
    assert call(use_id=dup)[0] == BAD
    w = np.ones(Q, dtype=np.int64)
    w[7] = -1
    bad_len = out_len.copy()
    bad_len[3] = 4
    assert call(weight=w, new_len=bad_len) == (BAD, 0, 0) and call(base=neg) == (BAD, 0, 0) and call(cap=neg) == (BAD, 0, 0)
    assert call(new_len=bad_len) == (BAD, 3, 0)
    bad_wave = wave.copy()
    bad_wave[[2, 600]] = -1
    assert call(wave=bad_wave, new_len=bad_len) == (BAD, 2, 0)
    big = np.full(Q, 1 << 60, dtype=np.int64)
    assert call(weight=big, new_len=bad_len)[:2] == (BAD, 3) and call(weight=big)[0] == LIMIT
    assert call(base=np.full(20, 1 << 59, dtype=np.int64))[0] == LIMIT
    # on the device: the lowest failing row, at its first failing position
    o, ln = out.copy(), out_len.copy()
    cases = {}
    for g, x in ((700, [5, 5]), (400, [1, 77]), (900, [88])):
        o[g, :] = -1
        o[g, :len(x)] = x
        ln[g] = len(x)
        cases[g] = x
    wv = wave.copy()
    wv[[400, 700, 900]] = [3, 1, 0]
    e = usage_models.broker_usage(rep_off, cur, o, ln, wv, ids)[2]
    assert e == (BAD, 400, 77) and call(new=o, new_len=ln, wave=wv) == e
    wv[400] = 0   # a row that does not run may name any broker; a new list naming one twice is refused anyway
    assert call(new=o, new_len=ln, wave=wv) == (BAD, 700, 5) == usage_models.broker_usage(rep_off, cur, o, ln, wv, ids)[2]
    wv[700], o[700, 1], ln[700] = 0, -1, 1
    assert call(new=o, new_len=ln, wave=wv)[0] == 0
    assert call(new=o, new_len=ln, wave=wv, n_use=0, use_id=None, usage=None)[0] == BAD   # every receiver is outside an empty table


def test_context_is_untouched_and_launches_depend_on_bit_lengths(native_lib):
    cl = kab.synth.make_ragged_cluster(T=3000, N=400, max_partitions=128, seed=21, remove_frac=0.02)
    s, out, out_len, _ = util.solved(cl)
    wave, _, _ = s.plan_waves(cl.rep_off, cl.cur, out, out_len, 2)
    before = (s.counters(), s.last_order_plan(), s.last_stage_plan())
    n0 = s.launch_count()
    usage, W, st = s.broker_usage(cl.rep_off, cl.cur, out, out_len, wave, cl.all_broker_id)
    assert st.code == 0 and W > 1
    passes = -(-(W + 1).bit_length() // 8) + -(-(len(cl.all_broker_id) - 1).bit_length() // 8)
    assert s.launch_count() - n0 == 2 + 3 * passes
    assert np.array_equal(s.counters(), before[0]) and (s.last_order_plan(), s.last_stage_plan()) == before[1:]
    args = (cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    again, again_len, _ = s.solve_ragged(*args)
    fresh = kab.Solver(0)
    fresh.set_brokers(cl.broker_id, cl.rack_index)
    fresh.solve_ragged(*args)
    f_out, f_len, _ = fresh.solve_ragged(*args)
    assert np.array_equal(again, f_out) and np.array_equal(again_len, f_len)

    def launches(Q, W, n_use):
        rep_off, cur = util.cur_lists([[1]] * Q)
        o, ln = util.rows([[2]] * Q)
        wv = np.full(Q, W, dtype=np.int32)
        n0 = s.launch_count()
        _, got, st = s.broker_usage(rep_off, cur, o, ln, wv, np.arange(2, n_use + 2, dtype=np.int32))
        assert st.code == 0 and got == (W if Q else 0)
        return s.launch_count() - n0

    assert launches(0, 0, 2) == launches(5000, 0, 300) == 2
    # one pass per 8 bits of W + 1, one per 8 bits of n_use - 1
    assert launches(10, 1, 1) == launches(300000, 254, 1) == 2 + 3
    assert launches(10, 255, 1) == launches(20, 3, 2) == launches(20, 254, 256) == 2 + 6
    assert launches(20, 3, 257) == 2 + 9
    assert launches(7, 70000, 65535) == 2 + 5 * 3


def test_the_million_partition_plan(native_lib):
    """The 1.06 M-partition cluster of wave_plan_times.py with its seeded weights, planned with a budget of 16 x the mean weight."""
    cl = kab.synth.make_ragged_cluster(T=240000, N=400, max_partitions=128, seed=11, remove_frac=0.02)
    s, out, out_len, _ = util.solved(cl)
    weight = np.random.default_rng(0x5EED).integers(1, 1 << 34, size=len(out_len), dtype=np.int64)
    wave, summ, st = s.plan_waves(cl.rep_off, cl.cur, out, out_len, 16 * int(weight.mean()), weight=weight)
    assert st.code == 0 and len(summ) > 100
    usage = check(s, cl.rep_off, cl.cur, out, out_len, wave, cl.all_broker_id, weight)
    assert (usage["peak"] > np.maximum(usage["before"], usage["after"])).any()


def test_cpp_host_mirror(native_lib):
    """host/test_broker_usage.cpp: brokerUsage equals its plain loop, and Solver.broker_usage on the inputs it wrote."""
    kab.build_mod.build_host()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "usage.txt")
        r = subprocess.run([kab.build_mod.HOST_BROKER_USAGE_TEST, path], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        assert r.stdout.strip().endswith("OK")
        lines = [np.array(x.split(), dtype=np.int64) for x in open(path).read().split("\n")]
    Q, stride, n, W = (int(x) for x in lines[0])
    rep_off, cur, out_len, new, weight, wave, ids, base, cap, rep = lines[1:11]
    usage, got_W, st = kab.Solver(0).broker_usage(rep_off, cur, new.reshape(Q, stride), out_len, wave, ids, weight=weight, base=base,
                                                  capacity=cap)
    assert st.code == 0 and got_W == W and np.array_equal(usage.view(np.int64).reshape(n, 5), rep.reshape(n, 5))
