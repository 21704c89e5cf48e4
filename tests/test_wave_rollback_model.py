"""ka_plan_waves_json_parts_rollback on the CPU: the rollback documents of `models.wave_documents`; the record-length identity
of the two key orders; the declarations; and what Solver.plan_wave_parts_rollback_json hands the C ABI and makes of what it gets
back, through a fake library. The paired cut itself is tested beside the one-sided cut, in tests/test_wave_parts_model.py."""
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


@pytest.mark.parametrize("seed", range(20))
def test_record_lengths_differ_only_by_the_list(seed):
    """Both key orders print 39 bytes + name + partition digits + list: the forward and rollback records of the same partition
    differ only by the printed list, and each document frame is 29 bytes."""
    rng = np.random.default_rng(seed)
    name = "t" * int(rng.integers(0, 50))
    part = int(rng.integers(-2 ** 31, 2 ** 31))
    a = [int(x) for x in rng.integers(-2 ** 31, 2 ** 31, int(rng.integers(0, 5)))]
    b = [int(x) for x in rng.integers(-2 ** 31, 2 ** 31, int(rng.integers(0, 5)))]
    lst = lambda x: len(",".join(str(v) for v in x))  # noqa: E731
    fwd, back = models.record(name, part, a), models.current_record(name, part, b)
    assert len(fwd) == 39 + len(name) + len(str(part)) + lst(a)
    assert len(back) == 39 + len(name) + len(str(part)) + lst(b)
    assert len(models.document([])) == len(models.rollback_document([])) == 29
    assert json.loads(back) == {"topic": name, "partition": part, "replicas": b}
    assert list(json.loads(back)) == ["topic", "partition", "replicas"]


@pytest.mark.parametrize("seed", range(4))
def test_rollback_documents_hold_each_part_on_its_current_lists(seed):
    rng = np.random.default_rng(20 + seed)
    for shrink in (0.0, 1.0):
        case = (*util.ragged_wave_case(rng, 30, 12, shrink), np.arange(1, 13))
        names, part_off, part_id, rep_off, cur = case[:5]
        current = {}
        for t, name in enumerate(names):
            for g in range(int(part_off[t]), int(part_off[t + 1])):
                current[(name, int(part_id[g]))] = cur[int(rep_off[g]):int(rep_off[g + 1])].tolist()
        for B, send in ((1, None), (3, None), (2, (list(range(1, 13)), 4)), (10 ** 6, None)):
            parts, _, p_wave, e_wave, summ, st = models.wave_documents(*case, B, send=send, L=10 ** 9)
            for L in (700, 2000, 10 ** 9):
                r = models.wave_documents(*case, B, send=send, L=L, rollback=True)
                if r[5][0]:
                    continue
                fwd, back, part_wave, wave, r_summ, r_st = r
                assert r_st == (0, 0, 0) and np.array_equal(wave, e_wave) and r_summ == summ and len(fwd) == len(back)
                assert all(len(p) <= L for p in fwd + back)
                for f, b in zip(fwd, back):
                    fr, br = json.loads(f)["partitions"], json.loads(b)["partitions"]
                    assert json.loads(b)["version"] == 1
                    assert [(x["topic"], x["partition"]) for x in fr] == [(x["topic"], x["partition"]) for x in br]
                    assert all(x["replicas"] == current[(x["topic"], x["partition"])] for x in br)
                # joined, each wave's forward parts are its document, as in the one-sided cut
                for v in set(part_wave):
                    joined = [x for f, pv in zip(fwd, part_wave) if pv == v for x in json.loads(f)["partitions"]]
                    assert joined == json.loads(parts[v - 1])["partitions"]
                if L == 10 ** 9:
                    assert fwd == parts and part_wave == p_wave


def test_shorter_current_lists_give_the_one_sided_cut_and_longer_ones_more_parts():
    rng = np.random.default_rng(7)
    case = (*util.ragged_wave_case(rng, 40, 12, 1.0), np.arange(1, 13))
    B = 10 ** 6
    smallest = max(29 + len(models.record(n, 0, [12, 12, 12])) for n in case[0])
    more = []
    for L in (smallest + 100, 900, 3000):
        parts = models.wave_documents(*case, B, L=L)[0]
        fwd, back = models.wave_documents(*case, B, L=L, rollback=True)[:2]
        assert len(fwd) >= len(parts) and max(len(b) for b in back) <= L
        more.append(len(fwd) > len(parts))
    assert any(more)
    # swap the sides: new lists the current ones, current lists the shrunk ones, so no current list prints longer
    names, part_off, part_id, rep_off, cur, out, out_len, ids = case
    new_lists = [cur[int(rep_off[g]):int(rep_off[g + 1])].tolist() for g in range(len(out_len))]
    cur_lists = [out[g][:int(out_len[g])].tolist() for g in range(len(out_len))]
    r_off, c_flat = util.cur_lists(cur_lists)
    o, o_len = util.rows(new_lists, 3)
    swapped = (names, part_off, part_id, r_off, c_flat, o, o_len, ids)
    for L in (smallest + 100, 900, 3000):
        parts, _, part_wave, wave, summ, st = models.wave_documents(*swapped, B, L=L)
        fwd, back, r_wave, r_plan, r_summ, r_st = models.wave_documents(*swapped, B, L=L, rollback=True)
        assert (fwd, r_wave, r_summ, r_st) == (parts, part_wave, summ, st) and np.array_equal(r_plan, wave)


def test_over_long_rows_and_plan_errors():
    cur = [[1], [2, 3, 4, 5, 6, 7], [3], [4]]
    new = [[5], [1], [6, 7, 8], [3]]
    rep_off, cur_flat = util.cur_lists(cur)
    out, out_len = util.rows(new)
    case = (["abc"], np.array([0, 4]), None, rep_off, cur_flat, out, out_len, np.arange(1, 20))
    fwd = [29 + len(models.record("abc", g, new[g])) for g in range(4)]
    back = [29 + len(models.current_record("abc", g, cur[g])) for g in range(4)]
    lens = [max(f, b) for f, b in zip(fwd, back)]
    assert back[1] > fwd[1] and fwd[2] > back[2]
    # the lowest over-long row on either side, with the longer one-record document's length
    assert models.wave_documents(*case, 10, rollback=True, L=max(lens) - 1)[5] == (LIMIT, 1, lens[1])
    assert models.wave_documents(*case, 10, rollback=True, L=min(lens) - 1)[5] == (LIMIT, 0, lens[0])
    assert models.wave_documents(*case, 10, rollback=True, L=fwd[1])[5] == (LIMIT, 1, back[1])
    assert models.wave_documents(*case, 10, rollback=True, L=max(lens))[5] == (0, 0, 0)
    # the plan's own errors come first
    bad = util.rows([[5, 5], [1], [1], [1]])
    assert models.wave_documents(*case[:5], *bad, case[7], 10, L=1, rollback=True)[5] == (BAD, 0, 5)
    # nothing changed: no part
    same = util.rows(cur, 6)
    assert models.wave_documents(*case[:5], *same, case[7], 10, L=100, rollback=True)[:3] == ([], [], [])


# ---- the C ABI --------------------------------------------------------------------------------------------------------------

def test_symbols_are_exported_and_declared(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    header = open(os.path.join(ROOT, "include", "kassign.h")).read()
    for name, n_args in (("ka_plan_waves_json_parts_rollback", 27), ("ka_plan_waves_send_json_parts_rollback", 31)):
        assert hasattr(raw, name)
        res, args = _native.SYMBOLS[name]
        assert res is ctypes.c_int32 and len(args) == n_args
        assert "int32_t %s(ka_ctx* ctx," % name in header


def test_without_a_context_is_no_device(native_lib):
    L = native_lib
    st = kab.KaStatus()
    n, d = ctypes.c_int32(5), ctypes.c_int32(6)
    args = (None, 0, None, None, None, None, 1, None, None, None, 1, None, None, None, 0, 100, None, None, ctypes.byref(d), None, 0,
            None, None, ctypes.byref(n), None, 0)
    assert L.ka_plan_waves_json_parts_rollback(*args, ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE
    assert st.code == _native.KA_ERR_NO_DEVICE and n.value == 0 and d.value == 0
    assert L.ka_plan_waves_json_parts_rollback(*args, None) == BAD
    n.value, d.value = 5, 6
    send_args = args[:11] + (0, None, 1) + args[11:25] + (None, 0)
    assert L.ka_plan_waves_send_json_parts_rollback(*send_args, ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE
    assert n.value == 0 and d.value == 0


def test_plan_wave_parts_rollback_json_marshals_its_arguments():
    lib = util.FakeWaveLib(2)
    s = util.fake_solver(lib)
    names, part_off, part_id, rep_off, cur, out, out_len = util.wave_inputs()
    weight = np.array([5, 0, 7, 1], dtype=np.int64)
    parts, rollback, part_wave, wave, summ, st = s.plan_wave_parts_rollback_json(
        names, part_off, part_id, rep_off.astype(np.int32), cur.astype(np.int64), out, out_len, 9, 1 << 20, weight=weight)
    assert st.code == 0 and len(lib.calls) == 1
    c = lib.calls[0]
    assert c["T"] == 3 and c["stride"] == 3 and c["B"] == 9 and c["cap"] == 4 and c["L"] == 1 << 20 and c["doc_wave"]
    assert c["part_off"].tolist() == part_off and c["part_id"].tolist() == part_id
    assert np.array_equal(c["rep_off"], rep_off) and np.array_equal(c["cur"], cur) and np.array_equal(c["weight"], weight)
    assert c["names"] == b"alphabc" and c["json_cap"] == models.json_bound(names, part_off, 3)
    # the documented rollback bound: per row 79 + its topic's name, 12 per current broker
    assert c["back_cap"] == models.json_bound(names, part_off, 0) + 12 * len(cur)
    assert [bytes(p) for p in parts] == [b"[%d]" % d for d in range(4)] and part_wave.tolist() == [1, 1, 2, 2]
    assert [bytes(p) for p in rollback] == [b"(%d)" % d for d in range(4)]
    assert wave.tolist() == [1, 2, 1, 2] and [list(x) for x in summ] == [[v * 10 + f for f in range(5)] for v in range(2)]
    assert summ.dtype == WAVE_SUMMARY_DTYPE
    # a sender budget takes the _send form; a caller's buffers are used as given
    buf, back = np.zeros(64, dtype=np.uint8), np.zeros(40, dtype=np.uint8)
    parts, rollback, part_wave, _, summ, st = s.plan_wave_parts_rollback_json(
        names, part_off, None, rep_off, cur, out, out_len, 2, 1000, json_buf=buf, back_buf=back, max_broker_out=7, send_brokers=[1, 2, 3])
    c = lib.calls[-1]
    assert c["C"] == 7 and c["send_id"].tolist() == [1, 2, 3] and c["json_cap"] == 64 and c["back_cap"] == 40 and c["L"] == 1000
    assert c["part_id"] is None
    assert summ.dtype == WAVE_SEND_SUMMARY_DTYPE and summ["max_broker_out"].tolist() == [5, 15]
    assert bytes(buf[:6]) == b"[0][1]" and parts[1].base is buf
    assert bytes(back[:6]) == b"(0)(1)" and rollback[1].base is back
    with pytest.raises(ValueError):
        s.plan_wave_parts_rollback_json(names, part_off, None, rep_off, cur, out, out_len, 2, 1000, max_broker_out=7)


@pytest.mark.parametrize("fail", [(BAD, 0, 0), (LIMIT, 2, 123), (LIMIT, 4000, 0)])
def test_a_refused_call_gives_empty_results_and_its_status(fail):
    s = util.fake_solver(util.FakeWaveLib(3, fail))
    names, part_off, part_id, rep_off, cur, out, out_len = util.wave_inputs()
    for send in ({}, dict(max_broker_out=7, send_brokers=[1, 2])):
        parts, rollback, part_wave, wave, summ, st = s.plan_wave_parts_rollback_json(names, part_off, part_id, rep_off, cur, out,
                                                                                     out_len, 9, 0, **send)
        assert (st.code, st.a, st.b) == fail
        assert parts == [] and rollback == [] and len(part_wave) == len(wave) == len(summ) == 0
