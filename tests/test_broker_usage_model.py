"""ka_wave_broker_usage on the CPU: `usage_models.broker_usage` on hand-worked cases and against a brute force that rebuilds what
every broker holds in every wave from the rows' states; the numpy form of the model against the loop; the check order; the
declarations; and what Solver.broker_usage hands the C ABI and makes of what it gets back, through a fake library."""
import ctypes
import os

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import BROKER_USAGE_DTYPE
from tests import models, usage_models, util

BAD, LIMIT = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(cur, new, wave, stride=None):
    rep_off, flat = util.cur_lists(cur)
    out, out_len = util.rows(new, stride)
    return rep_off, flat, out, out_len, np.asarray(wave, dtype=np.int32)


def brute_force(cur, new, wave, ids, weight=None, base=None, cap=None):
    """What every table broker holds in every wave 0..W, from each row's state: before its wave it holds its current list,
    during it both lists, after it its new list (a row with wave 0 keeps its current list); `after` once every wave has run.
    A broker holds a row's copy once, however often a list names it."""
    W = max(list(wave) + [0])
    w = [1] * len(cur) if weight is None else [int(x) for x in weight]

    def held(g, v):
        if wave[g] == 0 or v < wave[g]:
            return set(cur[g])
        return set(cur[g]) | set(new[g]) if v == wave[g] else set(new[g])

    res = []
    for i, b in enumerate(ids):
        b0 = 0 if base is None else int(base[i])
        usage = [b0 + sum(w[g] for g in range(len(cur)) if b in held(g, v)) for v in range(W + 1)]
        after = b0 + sum(w[g] for g in range(len(cur)) if b in (set(new[g]) if wave[g] else set(cur[g])))
        peak = max(usage)
        over = -1 if cap is None else next((v for v, u in enumerate(usage) if u > int(cap[i])), -1)
        res.append(dict(before=usage[0], peak=peak, peak_wave=usage.index(peak), after=after, over_wave=over))
    return res


def test_worked_example():
    """Broker 3 holds 4 before the plan, 14 in waves 1 and 2 and 10 after: over a capacity of 12 in wave 1 only."""
    case = _case([[1, 2], [3]], [[3, 2], [1]], [1, 2])
    res, W, st = usage_models.broker_usage(*case, [1, 2, 3], weight=[10, 4], cap=[100, 100, 12])
    assert st == (0, 0, 0) and W == 2
    assert res[2] == dict(before=4, peak=14, peak_wave=1, after=10, over_wave=1)
    assert res[0] == dict(before=10, peak=10, peak_wave=0, after=4, over_wave=-1)   # broker 1 frees 10 after wave 1, gets 4 in 2
    assert res[1] == dict(before=10, peak=10, peak_wave=0, after=10, over_wave=-1)
    assert brute_force([[1, 2], [3]], [[3, 2], [1]], [1, 2], [1, 2, 3], [10, 4], cap=[100, 100, 12]) == res


@pytest.mark.parametrize("seed", range(30))
def test_model_against_brute_force(seed):
    rng = np.random.default_rng(seed)
    N = int(rng.integers(3, 12))
    Q = int(rng.integers(0, 40))
    cur, new = util.random_wave_case(rng, Q, N)
    for g in range(Q):   # a duplicate id in some current lists
        if cur[g] and rng.random() < 0.15:
            cur[g].append(cur[g][0])
    W = int(rng.integers(0, 6))
    wave = [int(rng.integers(0, W + 1)) for _ in range(Q)]
    ids = sorted(int(x) for x in rng.choice(np.arange(1, N + 3), int(rng.integers(0, N + 2)), replace=False))
    # every receiver of a run row in the table (else the row is refused)
    for g in range(Q):
        if wave[g] and any(b not in cur[g] and b not in ids for b in new[g]):
            wave[g] = 0
    weight = rng.integers(0, 9, Q) if seed % 2 else None
    base = rng.integers(0, 20, len(ids)) if seed % 3 else None
    cap = rng.integers(0, 30, len(ids)) if seed % 4 else None
    case = _case(cur, new, wave, 4)
    res, got_W, st = usage_models.broker_usage(*case, ids, weight, base, cap)
    assert st == (0, 0, 0) and got_W == max(wave + [0])
    assert res == brute_force(cur, new, wave, ids, weight, base, cap)
    fast, fW = usage_models.broker_usage_np(*case, ids, weight, base, cap)
    assert fW == got_W and [{f: int(fast[f][i]) for f in usage_models.FIELDS} for i in range(len(ids))] == res


def test_duplicate_and_unknown_ids_in_current_lists():
    # broker 5 is named twice in a current list: it holds one copy, drops one; broker 99 is in no table: not tracked
    case = _case([[5, 5, 99], [5]], [[6], [5, 6]], [1, 2])
    res, W, st = usage_models.broker_usage(*case, [5, 6], weight=[3, 2])
    assert st == (0, 0, 0) and W == 2
    assert res == [dict(before=5, peak=5, peak_wave=0, after=2, over_wave=-1),
                   dict(before=0, peak=5, peak_wave=2, after=5, over_wave=-1)]
    # a receiver outside the table refuses the row, in a row with a wave only; a new list naming a broker twice always
    assert usage_models.broker_usage(*_case([[1], [1]], [[1], [7]], [0, 3]), [1])[2] == (BAD, 1, 7)
    assert usage_models.broker_usage(*_case([[1], [1]], [[1], [7]], [0, 0]), [1])[2] == (0, 0, 0)
    assert usage_models.broker_usage(*_case([[1], [1], [2]], [[2, 2], [7], [3]], [0, 1, 1]), [1, 2, 3])[2] == (BAD, 0, 2)


def test_changed_rows_with_wave_zero_count_before_only():
    case = _case([[1, 2], [1]], [[3, 4], [2]], [0, 0])
    res, W, st = usage_models.broker_usage(*case, [1, 2, 3, 4])
    assert st == (0, 0, 0) and W == 0
    assert [r["before"] for r in res] == [2, 1, 0, 0] and all(r["peak"] == r["after"] == r["before"] for r in res)
    res, W, _ = usage_models.broker_usage(*_case([[1, 2], [1]], [[3, 4], [2]], [0, 4]), [1, 2, 3, 4], cap=[1, 1, 1, 1])
    assert W == 4 and res[1] == dict(before=1, peak=2, peak_wave=4, after=2, over_wave=4)
    assert res[0] == dict(before=2, peak=2, peak_wave=0, after=1, over_wave=0)


@pytest.mark.parametrize("seed", range(5))
def test_one_wave_plans(seed):
    """A whole solve as one document (wave = changed ? 1 : 0): every broker peaks at what it holds before + what it receives,
    and with no base ends at ka_move_summary's broker_replicas."""
    rng = np.random.default_rng(100 + seed)
    N, Q = 12, 60
    cur, new = util.random_wave_case(rng, Q, N)
    wave = [int(c != n) for c, n in zip(cur, new)]
    ids = np.arange(1, N + 1)
    weight = rng.integers(0, 50, Q).astype(np.int64)
    case = _case(cur, new, wave, 3)
    res, W, st = usage_models.broker_usage(*case, ids, weight)
    assert st == (0, 0, 0) and W == (1 if any(wave) else 0)
    _, rep, _, inb = models.move_summary(case[2], case[3], case[0], case[1], ids, weight)
    assert [r["after"] for r in res] == rep.tolist()
    assert [r["peak"] for r in res] == [r["before"] + int(x) for r, x in zip(res, inb)]


def test_check_order():
    case = _case([[1], [2]], [[2], [3]], [1, 1])
    ids = [1, 2, 3]
    ok = usage_models.host_checks(*case, ids)
    assert ok == (0, 0, 0)
    assert usage_models.host_checks(*case, ids, stride=9) == (LIMIT, 9, 0)
    assert usage_models.host_checks(*case, list(range(1, 65538))) == (LIMIT, 65537, 0)
    assert usage_models.host_checks(*case, [1, 3, 2], weight=[-1, 0]) == (BAD, 0, 0)   # order before signs
    for kw in (dict(weight=[1, -1]), dict(base=[0, -2, 0]), dict(cap=[0, 0, -1])):
        assert usage_models.host_checks(*case, ids, **kw) == (BAD, 0, 0)
    rep_off, cur, out, out_len, wave = case
    assert usage_models.host_checks(rep_off, cur, out, np.array([1, 2]), wave, ids) == (BAD, 1, 0)
    assert usage_models.host_checks(rep_off, cur, out, out_len, np.array([1, -1]), ids) == (BAD, 1, 0)
    assert usage_models.host_checks(rep_off, cur, out, np.array([1, 2]), np.array([-1, 0]), ids, weight=[-1, 0]) == (BAD, 0, 0)
    big = 2 ** 62
    assert usage_models.host_checks(*case, ids, weight=[big, 0]) == (LIMIT, 0, 0)        # 2 x 2^62 > INT64_MAX
    assert usage_models.host_checks(*case, ids, weight=[big // 4, big // 4]) == (0, 0, 0)
    assert usage_models.host_checks(*case, ids, base=[big, big, 0]) == (LIMIT, 0, 0)
    # the host checks come before the row checks
    bad_rows = _case([[1]], [[4, 4]], [1])
    assert usage_models.broker_usage(*bad_rows, [1, 4])[2] == (BAD, 0, 4)
    assert usage_models.broker_usage(*bad_rows, [1, 4], weight=[-1])[2] == (BAD, 0, 0)


# ---- the C ABI --------------------------------------------------------------------------------------------------------------

def test_symbol_is_exported_and_declared(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    header = open(os.path.join(ROOT, "include", "kassign.h")).read()
    assert hasattr(raw, "ka_wave_broker_usage")
    res, args = _native.SYMBOLS["ka_wave_broker_usage"]
    assert res is ctypes.c_int32 and len(args) == 16
    assert "int32_t ka_wave_broker_usage(ka_ctx* ctx," in header and "} ka_broker_usage;" in header
    assert ctypes.sizeof(_native.KaBrokerUsage) == 40 and BROKER_USAGE_DTYPE.itemsize == 40
    assert BROKER_USAGE_DTYPE.names == usage_models.FIELDS


def test_without_a_context_is_no_device(native_lib):
    L = native_lib
    st = kab.KaStatus()
    n = ctypes.c_int32(5)
    args = (None, 0, None, None, 1, None, None, None, None, 0, None, None, None, None, ctypes.byref(n))
    assert L.ka_wave_broker_usage(*args, ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE
    assert st.code == _native.KA_ERR_NO_DEVICE and n.value == 0
    assert L.ka_wave_broker_usage(*args, None) == BAD


class FakeUsageLib:
    """Stands in for libkassign.so's ka_wave_broker_usage: records what it is handed, writes field f of broker i as 10 i + f and
    W = 7, or refuses the call with `fail` = (code, a, b)."""

    def __init__(self, fail=None):
        self.fail, self.calls = fail, []

    def ka_wave_broker_usage(self, h, Q, rep_off, cur, stride, new_len, new_broker, weight, wave, n, use_id, base, cap, usage, n_waves,
                             st):
        r_off = util.view(rep_off, Q + 1, np.int64)
        self.calls.append(dict(Q=Q, stride=stride, rep_off=r_off, cur=util.view(cur, int(r_off[-1]), np.int32),
                               new_len=util.view(new_len, Q, np.int32), new=util.view(new_broker, Q * stride, np.int32),
                               weight=util.view(weight, Q, np.int64), wave=util.view(wave, Q, np.int32), n=n,
                               use_id=util.view(use_id, n, np.int32), base=util.view(base, n, np.int64), cap=util.view(cap, n, np.int64)))
        if self.fail:
            st._obj.code, st._obj.a, st._obj.b = self.fail
            n_waves._obj.value = 0
            return self.fail[0]
        if n:
            util.writable(usage, 5 * n, np.int64).reshape(n, 5)[:] = np.arange(n)[:, None] * 10 + np.arange(5)
        n_waves._obj.value = 7
        st._obj.code = 0
        return 0


def test_broker_usage_marshals_its_arguments():
    lib = FakeUsageLib()
    s = util.fake_solver(lib)
    rep_off, cur, out, out_len, wave = _case([[1], [2, 3], [4]], [[1, 2], [3], [4, 5, 6]], [1, 0, 2])
    use = [1, 2, 3, 4, 5, 6]
    usage, W, st = s.broker_usage(rep_off.astype(np.int32), cur.astype(np.int64), out, out_len, wave.astype(np.int64), use,
                                  weight=[5, 0, 7], base=np.arange(6), capacity=[9] * 6)
    assert st.code == 0 and W == 7 and len(lib.calls) == 1
    c = lib.calls[0]
    assert c["Q"] == 3 and c["stride"] == 3 and c["n"] == 6 and c["use_id"].tolist() == use
    assert np.array_equal(c["rep_off"], rep_off) and np.array_equal(c["cur"], cur) and np.array_equal(c["new"], out.reshape(-1))
    assert c["new_len"].tolist() == out_len.tolist() and c["wave"].tolist() == [1, 0, 2] and c["weight"].tolist() == [5, 0, 7]
    assert c["base"].tolist() == list(range(6)) and c["cap"].tolist() == [9] * 6
    assert usage.dtype == BROKER_USAGE_DTYPE and [list(x) for x in usage] == [[10 * i + f for f in range(5)] for i in range(6)]
    # the optional arrays go as NULL; no table is an empty report
    usage, W, st = s.broker_usage(rep_off, cur, out, out_len, wave, [])
    c = lib.calls[-1]
    assert c["weight"] is None and c["base"] is None and c["cap"] is None and c["n"] == 0 and len(usage) == 0 and W == 7
    with pytest.raises(AssertionError):
        s.broker_usage(rep_off, cur, out, out_len, wave[:2], use)
    with pytest.raises(AssertionError):
        s.broker_usage(rep_off, cur, out, out_len, wave, use, base=[1, 2])


@pytest.mark.parametrize("fail", [(BAD, 0, 0), (BAD, 2, 99), (LIMIT, 9, 0)])
def test_a_refused_call_gives_an_empty_report_and_its_status(fail):
    s = util.fake_solver(FakeUsageLib(fail))
    usage, W, st = s.broker_usage(*_case([[1]], [[2]], [1]), [1, 2])
    assert (st.code, st.a, st.b) == fail and len(usage) == 0 and W == 0
