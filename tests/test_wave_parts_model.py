"""ka_plan_waves_json_parts(_rollback) on the CPU: the greedy cut of `models.cut_parts`, over one side and over the paired
sides, against a brute force over every cut of random record lengths; the parts of `models.wave_documents` against its per-wave
documents; the declarations; and what Solver.plan_wave_parts_json hands the C ABI and makes of what it gets back, through a
fake library."""
import ctypes
import json
import os

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SEND_SUMMARY_DTYPE, WAVE_SUMMARY_DTYPE
from tests import models, util

BAD, LIMIT = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _size(lengths):
    return 29 + sum(lengths) + len(lengths) - 1


def _fits(sides, a, b, L):
    return all(_size(x[a:b]) <= L for x in sides)


def _brute(sides, L):
    """Every cut of the records into consecutive runs in which each run fits on every side and each run but the last could not
    take the next record on at least one side: the greedy cut, found without a greedy loop."""
    n = len(sides[0])
    found = []
    for mask in range(1 << max(n - 1, 0)):
        bounds = [0] + [i + 1 for i in range(n - 1) if mask >> i & 1] + [n]
        runs = list(zip(bounds, bounds[1:]))
        if all(_fits(sides, a, b, L) for a, b in runs) and not any(_fits(sides, a, b + 1, L) for a, b in runs[:-1]):
            found.append(runs)
    return found


@pytest.mark.parametrize("paired", [False, True])
@pytest.mark.parametrize("seed", range(6))
def test_cut_is_the_only_greedy_cut(seed, paired):
    rng = np.random.default_rng(seed)
    for _ in range(60):
        n = int(rng.integers(1, 11))
        fwd = [int(x) for x in rng.integers(40, 120, n)]
        if not paired:
            L = int(rng.integers(29 + max(fwd), 29 + sum(fwd) + n + 20))
            runs = models.cut_parts([fwd], L)
            assert _brute([fwd], L) == [runs], (fwd, L)
            assert all(_size(fwd[a:b]) <= L for a, b in runs)
            continue
        back = [int(x) for x in rng.integers(40, 120, n)]
        L = int(rng.integers(29 + max(fwd + back), 29 + max(sum(fwd), sum(back)) + n + 20))
        runs = models.cut_parts([fwd, back], L)
        assert _brute([fwd, back], L) == [runs], (fwd, back, L)
        # every part fits on both sides; a part and the next part's first record exceed L on at least one side
        assert all(_fits([fwd, back], a, b, L) for a, b in runs)
        assert not any(_fits([fwd, back], a, b + 1, L) for a, b in runs[:-1])
        # the same lengths on both sides: the one-sided cut
        assert models.cut_parts([fwd, fwd], L) == models.cut_parts([fwd], L)
        # a rollback side never longer than the forward side: the one-sided cut too
        shorter = [max(1, f - int(d)) for f, d in zip(fwd, rng.integers(0, 30, n))]
        assert models.cut_parts([fwd, shorter], L) == models.cut_parts([fwd], L)


@pytest.mark.parametrize("seed", range(4))
def test_parts_hold_every_wave_in_order_and_stay_within_the_limit(seed):
    rng = np.random.default_rng(10 + seed)
    case = (*util.ragged_wave_case(rng, 30, 12), np.arange(1, 13))
    for B, send in ((1, None), (3, None), (2, (list(range(1, 13)), 4)), (10 ** 6, None)):
        docs, _, doc_wave, wave, summ, st = models.wave_documents(*case, B, send=send)
        assert st == (0, 0, 0) and doc_wave == list(range(1, len(docs) + 1))
        smallest = util.smallest_limit(*case[:7], wave)
        for L in (smallest, smallest + 57, 700, 2000, max(len(d) for d in docs)):
            parts, _, part_wave, p_wave, p_summ, p_st = models.wave_documents(*case, B, send=send, L=L)
            assert p_st == (0, 0, 0) and np.array_equal(p_wave, wave) and p_summ == summ
            assert part_wave == sorted(part_wave) and set(part_wave) == set(range(1, len(docs) + 1))
            assert all(len(p) <= L for p in parts)
            for v, doc in enumerate(docs, 1):
                mine = [json.loads(p) for p, pv in zip(parts, part_wave) if pv == v]
                assert all(m["version"] == 1 and m["partitions"] for m in mine)
                # joined, a wave's parts are its records in order; a part and the next part's first record exceed L
                assert [r for m in mine for r in m["partitions"]] == json.loads(doc)["partitions"]
                for a, b in zip(mine, mine[1:]):
                    assert len(models.document([json.dumps(r, separators=(",", ":")) for r in a["partitions"] + b["partitions"][:1]])) > L
            assert len(parts) >= len(docs)


def test_exact_size_keeps_a_part_whole_and_one_byte_less_cuts_it():
    rng = np.random.default_rng(3)
    case = (*util.ragged_wave_case(rng, 30, 12), np.arange(1, 13))
    docs = models.wave_documents(*case, 10 ** 6)[0]
    assert len(docs) == 1
    whole = len(docs[0])
    parts, _, part_wave, _, _, _ = models.wave_documents(*case, 10 ** 6, L=whole)
    assert parts == docs and part_wave == [1]
    parts, _, part_wave, _, _, _ = models.wave_documents(*case, 10 ** 6, L=whole - 1)
    assert len(parts) == 2 and part_wave == [1, 1]
    assert len(parts[0]) <= whole - 1 and len(parts[0]) + len(parts[1]) - 29 + 1 == whole


def test_a_limit_above_every_wave_gives_the_wave_documents():
    rng = np.random.default_rng(4)
    case = (*util.ragged_wave_case(rng, 30, 12), np.arange(1, 13))
    for B in (1, 2, 5):
        docs, _, doc_wave, wave, summ, _ = models.wave_documents(*case, B)
        parts, _, part_wave, p_wave, p_summ, _ = models.wave_documents(*case, B, L=max(len(d) for d in docs))
        assert parts == docs and part_wave == doc_wave == list(range(1, len(docs) + 1)) and p_summ == summ


def test_over_long_rows_and_plan_errors():
    cur = [[1], [2], [3], [4]]
    new = [[5], [1, 2, 3], [6, 7, 8, 9], [3]]
    rep_off, cur_flat = util.cur_lists(cur)
    out, out_len = util.rows(new)
    case = (["abc"], np.array([0, 4]), None, rep_off, cur_flat, out, out_len, np.arange(1, 20))
    lens = [29 + len(models.record("abc", g, new[g])) for g in range(4)]
    # the lowest over-long row, with its one-record document's length
    assert models.wave_documents(*case, 10, L=max(lens) - 1)[5] == (LIMIT, 2, lens[2])
    assert models.wave_documents(*case, 10, L=min(lens) - 1)[5] == (LIMIT, 0, lens[0])
    assert models.wave_documents(*case, 10, L=max(lens))[5] == (0, 0, 0)
    # the plan's own errors come first
    bad = util.rows([[5, 5], [1], [1], [1]])
    assert models.wave_documents(*case[:5], *bad, case[7], 10, L=1)[5] == (BAD, 0, 5)
    # nothing changed: no part
    same = util.rows(cur)
    parts, _, part_wave = models.wave_documents(*case[:5], *same, case[7], 10, L=100)[:3]
    assert (parts, part_wave) == ([], [])


# ---- the C ABI --------------------------------------------------------------------------------------------------------------

def test_symbols_are_exported_and_declared(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    header = open(os.path.join(ROOT, "include", "kassign.h")).read()
    for name, n_args in (("ka_plan_waves_json_parts", 24), ("ka_plan_waves_send_json_parts", 28)):
        assert hasattr(raw, name)
        res, args = _native.SYMBOLS[name]
        assert res is ctypes.c_int32 and len(args) == n_args
        assert "int32_t %s(ka_ctx* ctx," % name in header


def test_without_a_context_is_no_device(native_lib):
    L = native_lib
    st = kab.KaStatus()
    n, d = ctypes.c_int32(5), ctypes.c_int32(6)
    args = (None, 0, None, None, None, None, 1, None, None, None, 1, None, None, None, 0, 100, None, None, ctypes.byref(d), None,
            ctypes.byref(n), None, 0)
    assert L.ka_plan_waves_json_parts(*args, ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE
    assert st.code == _native.KA_ERR_NO_DEVICE and n.value == 0 and d.value == 0
    assert L.ka_plan_waves_json_parts(*args, None) == BAD
    n.value, d.value = 5, 6
    send_args = args[:11] + (0, None, 1) + args[11:22] + (None, 0)
    assert L.ka_plan_waves_send_json_parts(*send_args, ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE
    assert n.value == 0 and d.value == 0


def test_plan_wave_parts_json_marshals_its_arguments():
    lib = util.FakeWaveLib(2)
    s = util.fake_solver(lib)
    names, part_off, part_id, rep_off, cur, out, out_len = util.wave_inputs()
    weight = np.array([5, 0, 7, 1], dtype=np.int64)
    parts, part_wave, wave, summ, st = s.plan_wave_parts_json(names, part_off, part_id, rep_off.astype(np.int32), cur.astype(np.int64),
                                                              out, out_len, 9, 1 << 20, weight=weight)
    assert st.code == 0 and len(lib.calls) == 1
    c = lib.calls[0]
    assert c["T"] == 3 and c["stride"] == 3 and c["B"] == 9 and c["cap"] == 4 and c["L"] == 1 << 20 and c["doc_wave"]
    assert c["part_off"].tolist() == part_off and c["part_id"].tolist() == part_id
    assert np.array_equal(c["rep_off"], rep_off) and np.array_equal(c["cur"], cur) and np.array_equal(c["weight"], weight)
    assert c["names"] == b"alphabc" and c["json_cap"] == models.json_bound(names, part_off, 3)
    assert [bytes(p) for p in parts] == [b"[%d]" % d for d in range(4)] and part_wave.tolist() == [1, 1, 2, 2]
    assert wave.tolist() == [1, 2, 1, 2] and [list(x) for x in summ] == [[v * 10 + f for f in range(5)] for v in range(2)]
    assert summ.dtype == WAVE_SUMMARY_DTYPE
    # a sender budget takes the _send form; a caller's buffer is used as given
    buf = np.zeros(64, dtype=np.uint8)
    parts, part_wave, _, summ, st = s.plan_wave_parts_json(names, part_off, None, rep_off, cur, out, out_len, 2, 1000, json_buf=buf,
                                                           max_broker_out=7, send_brokers=[1, 2, 3])
    c = lib.calls[-1]
    assert c["C"] == 7 and c["send_id"].tolist() == [1, 2, 3] and c["json_cap"] == 64 and c["L"] == 1000 and c["part_id"] is None
    assert summ.dtype == WAVE_SEND_SUMMARY_DTYPE and summ["max_broker_out"].tolist() == [5, 15]
    assert bytes(buf[:6]) == b"[0][1]" and parts[1].base is buf
    with pytest.raises(ValueError):
        s.plan_wave_parts_json(names, part_off, None, rep_off, cur, out, out_len, 2, 1000, max_broker_out=7)


@pytest.mark.parametrize("fail", [(BAD, 0, 0), (LIMIT, 2, 123), (LIMIT, 4000, 0)])
def test_a_refused_call_gives_empty_results_and_its_status(fail):
    s = util.fake_solver(util.FakeWaveLib(3, fail))
    names, part_off, part_id, rep_off, cur, out, out_len = util.wave_inputs()
    for send in ({}, dict(max_broker_out=7, send_brokers=[1, 2])):
        parts, part_wave, wave, summ, st = s.plan_wave_parts_json(names, part_off, part_id, rep_off, cur, out, out_len, 9, 0, **send)
        assert (st.code, st.a, st.b) == fail
        assert parts == [] and len(part_wave) == len(wave) == len(summ) == 0
