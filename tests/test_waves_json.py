"""ka_plan_waves_json: one reassignment document per wave of a wave plan, built on the device. `models.wave_documents` prints
the waves of `models.plan_waves` record by record in the key order of the device emitter; every document, wave,
summary and W of the device must equal it byte for byte. The CPU tests pin the model and what Solver.plan_waves_json hands the
C ABI."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SUMMARY_DTYPE
from tests import models, util

BAD, LIMIT = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT
INT64_MAX = np.iinfo(np.int64).max


def _one_topic(Q, name="t"):
    return [name], np.array([0, Q], dtype=np.int64)


# ---- CPU -----------------------------------------------------------------------------------------------------------------

def test_symbol_is_exported_and_declared(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    assert hasattr(raw, "ka_plan_waves_json")
    res, args = _native.SYMBOLS["ka_plan_waves_json"]
    assert res is ctypes.c_int32 and len(args) == 21
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kassign.h")).read()
    assert "int32_t ka_plan_waves_json(ka_ctx* ctx, int32_t T," in header


def test_without_a_context_is_no_device(native_lib):
    L = native_lib
    st = kab.KaStatus()
    n = ctypes.c_int32(5)
    args = (None, 0, None, None, None, None, 1, None, None, None, 1, None, None, None, 0, None, None, ctypes.byref(n), None, 0)
    assert L.ka_plan_waves_json(*args, ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE
    assert st.code == _native.KA_ERR_NO_DEVICE and n.value == 0
    assert L.ka_plan_waves_json(*args, None) == BAD


def test_plan_waves_json_marshals_its_arguments():
    lib = util.FakeWaveLib(3)
    s = util.fake_solver(lib)
    out, out_len = util.rows([[1, 2], [3], [4, 5, 6], []])
    rep_off, cur = util.cur_lists([[1], [2, 3], [4], [7, 8]])
    weight = np.array([5, 0, 7, 1], dtype=np.int64)
    names = ["alpha", "", "bc"]
    part_off, part_id = [0, 3, 3, 4], [4, 9, -2, 0]
    docs, wave, summ, st = s.plan_waves_json(names, part_off, part_id, rep_off.astype(np.int32), cur.astype(np.int64), out, out_len, 9,
                                             weight=weight)
    assert st.code == 0 and len(lib.calls) == 1
    c = lib.calls[0]
    assert c["T"] == 3 and c["stride"] == 3 and c["B"] == 9 and c["cap"] == 4
    assert c["part_off"].tolist() == part_off and c["part_id"].tolist() == part_id
    assert np.array_equal(c["rep_off"], rep_off) and np.array_equal(c["cur"], cur)
    assert np.array_equal(c["new_len"], out_len) and np.array_equal(c["new_broker"], out.ravel())
    assert np.array_equal(c["weight"], weight)
    assert c["names"] == b"alphabc" and c["name_off"].tolist() == [0, 5, 5, 7]
    assert c["json_cap"] == models.json_bound(names, part_off, 3) == 3 * (79 + 36 + 5) + (79 + 36 + 2)
    assert [bytes(d) for d in docs] == [b"<0>", b"<1>", b"<2>"]
    assert wave.tolist() == [1, 2, 3, 1] and [list(x) for x in summ] == [[v * 10 + f for f in range(5)] for v in range(3)]
    buf = np.zeros(50, dtype=np.uint8)
    docs, _, _, _ = s.plan_waves_json(names, part_off, None, rep_off, cur, out, out_len, 1, json_buf=buf)
    assert lib.calls[-1]["weight"] is None and lib.calls[-1]["part_id"] is None and lib.calls[-1]["json_cap"] == 50
    assert bytes(buf[:9]) == b"<0><1><2>" and docs[1].base is buf


def test_model_hand_worked():
    cur = [[1, 2], [1, 2], [1], [2], [1, 2], [1, 2], [5], [1], [2]]
    new = [[1, 3], [3, 4], [3], [4], [2, 1], [1, 2], [4, 5], [3, 4], [3]]
    rep_off, cur_flat = util.cur_lists(cur)
    out, out_len = util.rows(new)
    docs, _, _, wave, summ, st = models.wave_documents(["a", "empty", "b.c"], [0, 4, 4, 9], [0, 1, 5, 7, 2, 3, 4, -6, 8], rep_off,
                                                       cur_flat, out, out_len, np.arange(1, 100), 2)
    assert st == (0, 0, 0) and wave.tolist() == [1, 1, 2, 1, 1, 0, 2, 2, 3]
    assert docs == [
        b'{"partitions":[{"partition":0,"replicas":[1,3],"topic":"a"},{"partition":1,"replicas":[3,4],"topic":"a"},'
        b'{"partition":7,"replicas":[4],"topic":"a"},{"partition":2,"replicas":[2,1],"topic":"b.c"}],"version":1}',
        b'{"partitions":[{"partition":5,"replicas":[3],"topic":"a"},{"partition":4,"replicas":[4,5],"topic":"b.c"},'
        b'{"partition":-6,"replicas":[3,4],"topic":"b.c"}],"version":1}',
        b'{"partitions":[{"partition":8,"replicas":[3],"topic":"b.c"}],"version":1}']
    # ordinals without part_id; nothing changed gives no document; a refused plan none either
    docs = models.wave_documents(["a", "b"], [0, 1, 3], None, *util.cur_lists([[1], [1], [1]]), *util.rows([[2], [1], [2]]), [1, 2], 1)[0]
    assert docs == [b'{"partitions":[{"partition":0,"replicas":[2],"topic":"a"}],"version":1}',
                    b'{"partitions":[{"partition":1,"replicas":[2],"topic":"b"}],"version":1}']
    assert models.wave_documents(["a"], [0, 1], None, *util.cur_lists([[1]]), *util.rows([[1]]), [1], 1)[0] == []
    assert models.wave_documents(["a"], [0, 1], None, *util.cur_lists([[1]]), *util.rows([[2, 2]]), [1, 2], 1)[::5] == (None, (BAD, 0, 2))


@pytest.mark.parametrize("seed", range(4))
def test_model_invariants(seed):
    """Every document parses, and the documents together hold every changed row exactly once, within the documented bound."""
    rng = np.random.default_rng(seed)
    T = 40
    sizes = rng.integers(0, 9, T)
    part_off = np.concatenate([[0], np.cumsum(sizes)])
    Q = int(part_off[-1])
    names = ["topic-%d" % t for t in range(T)]
    part_id = np.concatenate([np.sort(rng.choice(1000, n, replace=False)) for n in sizes]).astype(np.int32)
    cur_lists = [[int(x) for x in rng.choice(np.arange(1, 13), int(rng.integers(0, 4)), replace=False)] for _ in range(Q)]
    new_lists = [c if rng.random() < 0.3 else [int(x) for x in rng.choice(np.arange(1, 13), int(rng.integers(0, 4)), replace=False)]
                 for c in cur_lists]
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    topic_of = np.repeat(np.arange(T), sizes)
    for B, weight in ((1, None), (3, None), (40, rng.integers(0, 30, Q))):
        docs, _, _, wave, summ, st = models.wave_documents(names, part_off, part_id, rep_off, cur, out, out_len, np.arange(1, 13), B,
                                                           weight)
        assert st == (0, 0, 0) and len(docs) == len(summ)
        seen = []
        for v, doc in enumerate(docs):
            parsed = json.loads(doc)
            assert parsed["version"] == 1 and len(parsed["partitions"]) == summ[v]["rows"] > 0
            seen += [(r["topic"], r["partition"], tuple(r["replicas"])) for r in parsed["partitions"]]
        want = [(names[topic_of[g]], int(part_id[g]), tuple(new_lists[g])) for g in range(Q) if new_lists[g] != cur_lists[g]]
        assert sorted(seen) == sorted(want) and len(set(seen)) == len(seen)
        assert sum(len(d) for d in docs) <= models.json_bound(names, part_off, 3)


# ---- GPU -----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("remove", [0.0, 0.02, 0.2])
def test_solve_rows(native_lib, remove):
    cl = kab.synth.make_ragged_cluster(T=4000, N=400, max_partitions=128, seed=7, remove_frac=remove)
    s, out, out_len, S = util.solved(cl)
    Q = len(out_len)
    weight = np.random.default_rng(3).integers(0, 1 << 20, Q).astype(np.int64)
    sparse = (cl.part_id.astype(np.int64) * 7 - 50).astype(np.int32)   # sparse and negative ids
    for B, w, pid in ((1, None, cl.part_id), (3, None, None), (INT64_MAX, None, sparse), (int(weight.mean()), weight, sparse)):
        docs, _, _, _, summ, st = util.check_wave_documents(s, cl.topic_names, cl.part_off, pid, cl.rep_off, cl.cur, out, out_len, B,
                                                            weight=w)
        assert st.code == 0
        if B == INT64_MAX:   # a single wave
            assert len(docs) == 1
    assert len(docs) >= 10   # the weighted plan: tens of waves


@pytest.mark.gpu
def test_growing_rf_rows_of_4_to_8(native_lib):
    for drf, shape in ((5, dict(N=60, seed=16)), (8, dict(N=200, seed=19, max_partitions=64))):
        cl = kab.synth.make_ragged_cluster(T=600, R=6, rack_frac=0.0, desired_rf=drf, **shape)
        s, out, out_len, S = util.solved(cl, drf)
        assert S == drf and out_len.max() == drf
        for B in (1, 1000):
            util.check_wave_documents(s, cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, B)


@pytest.mark.gpu
def test_hand_built_rows(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))

    def run(names, part_off, part_id, cur_lists, new_lists, B, weight=None, stride=None):
        rep_off, cur = util.cur_lists(cur_lists)
        out, out_len = util.rows(new_lists, stride)
        docs, _, _, wave, summ, st = util.check_wave_documents(
            s, names, np.asarray(part_off, dtype=np.int64), None if part_id is None else np.asarray(part_id, dtype=np.int32), rep_off,
            cur, out, out_len, B, weight=None if weight is None else np.asarray(weight, dtype=np.int64))
        return docs, wave, summ, st

    # reorder only (changed without a receiver: wave 1), drops only, and topics without partitions at both ends and inside
    docs, wave, _, _ = run(["none", "a", "gap", "b", "end"], [0, 0, 2, 2, 4, 4], [3, 9, -1, 0],
                           [[1, 2], [3, 4], [1, 2, 3], [5]], [[2, 1], [3, 4], [1], [6]], 1)
    assert wave.tolist() == [1, 0, 1, 1] and len(docs) == 1
    assert bytes(docs[0]) == (b'{"partitions":[{"partition":3,"replicas":[2,1],"topic":"a"},{"partition":-1,"replicas":[1],"topic":"b"},'
                              b'{"partition":0,"replicas":[6],"topic":"b"}],"version":1}')
    # an empty new list, INT32 extremes of the partition id
    run(["x"], [0, 3], [-2 ** 31, 0, 2 ** 31 - 1], [[1], [2], [3]], [[], [7], [8, 9]], 1)
    # nothing changed: W = 0; and no rows at all
    docs, wave, summ, st = run(["x"], [0, 50], None, [[1, 2]] * 50, [[1, 2]] * 50, 1)
    assert st.code == 0 and docs == [] and not wave.any() and len(summ) == 0
    docs, _, _, st = run([], [0], None, [], [], 1)
    assert st.code == 0 and docs == []
    docs, _, _, st = run(["x", "y"], [0, 0, 0], None, [], [], 1)
    assert st.code == 0 and docs == []
    # 8 receivers per row, unit and weighted
    eight = [[int(x) for x in 1 + (np.arange(8) + g) % 40] for g in range(3000)]
    run(["e%d" % t for t in range(30)], np.arange(31) * 100, None, [[]] * 3000, eight, 1)
    run(["e%d" % t for t in range(30)], np.arange(31) * 100, None, [[]] * 3000, eight, 5, np.arange(3000) % 4)


@pytest.mark.gpu
@pytest.mark.parametrize("Q", [100, 127, 128, 129, 255, 256, 257, 2100, 70000])
def test_fully_serial_plans_cross_every_sort_pass(native_lib, Q):
    """Every row receives the same broker with B = 1: W = Q, one row per document. W on both sides of 128 and of 256 (one 8-bit
    pass or two), above 2 048, and above 65 536 (three passes)."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))
    T = 7
    part_off = (np.arange(T + 1) * Q) // T
    names = ["serial-%d" % t for t in range(T)]
    rep_off, cur = util.cur_lists([[1]] * Q)
    out, out_len = util.rows([[2]] * Q)
    docs, _, _, wave, _, st = util.check_wave_documents(s, names, part_off, None, rep_off, cur, out, out_len, 1)
    assert st.code == 0 and len(docs) == Q and wave.tolist() == list(range(1, Q + 1))


@pytest.mark.gpu
def test_scattered_waves_in_two_passes(native_lib):
    """A few hot brokers with B = 1: hundreds of waves whose rows are scattered over the whole input."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 61), 4))
    rng = np.random.default_rng(8)
    Q = 30000
    cur_lists = [[int(x) for x in rng.choice(np.arange(1, 41), 2, replace=False)] for _ in range(Q)]
    new_lists = [[c[0], int(rng.integers(41, 61))] if rng.random() < 0.4 else c for c in cur_lists]
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 2)
    part_off = np.concatenate([[0], np.sort(rng.choice(np.arange(1, Q), 499, replace=False)), [Q]])
    names = ["t.%d" % t for t in range(500)]
    docs = util.check_wave_documents(s, names, part_off, None, rep_off, cur, out, out_len, 1)[0]
    assert len(docs) > 256
    docs = util.check_wave_documents(s, names, part_off, None, rep_off, cur, out, out_len, 3)[0]
    assert 128 < len(docs) < 256


@pytest.mark.gpu
def test_long_names_take_the_direct_path(native_lib):
    """Names of about 400 bytes: the text of 256 rows exceeds the 64 KiB staging area, and those CTAs write straight to global
    memory; short names beside them keep other CTAs staged."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))
    rng = np.random.default_rng(9)
    T, Q = 40, 4000
    names = [("long-%02d-" % t) + "x" * int(rng.integers(380, 420)) if t % 4 else "s%d" % t for t in range(T)]
    part_off = np.arange(T + 1) * (Q // T)
    cur_lists = [[int(x) for x in rng.choice(np.arange(1, 31), 3, replace=False)] for _ in range(Q)]
    new_lists = [[c[0], c[1], int(rng.integers(31, 41))] if rng.random() < 0.8 else c for c in cur_lists]
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    for B in (1, 50, 10 ** 6):
        docs = util.check_wave_documents(s, names, part_off, None, rep_off, cur, out, out_len, B)[0]
    assert len(docs) == 1 and len(docs[0]) > 256 * 400


@pytest.mark.gpu
@pytest.mark.parametrize("table", ["smem_lut", "global_lut", "bsearch", "state_in_smem", "state_in_global"])
def test_lookup_modes_and_chain_state(native_lib, table):
    N = dict(smem_lut=50, global_lut=50, bsearch=50, state_in_smem=12800, state_in_global=12801)[table]
    if table == "global_lut":
        ids, racks = util.table(1 + 700 * np.arange(N), 5)
    elif table == "bsearch":
        ids, racks = util.bsearch_table(N)
    else:
        ids, racks = util.table(np.arange(1, N + 1), 8)
    s = kab.Solver(0)
    s.set_brokers(ids, racks)
    rng = np.random.default_rng(N)
    Q = 12000
    cur_lists = [[int(x) for x in rng.choice(ids, int(rng.integers(0, 4)), replace=False)] for _ in range(Q)]
    hot = ids[-5:]
    new_lists = [[int(x) for x in rng.choice(hot if g % 3 == 0 else ids, int(rng.integers(1, 4)), replace=False)] for g in range(Q)]
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    part_off = np.arange(61) * 200
    names = ["m%d" % t for t in range(60)]
    for B, w in ((1, None), (500, rng.integers(0, 100, Q).astype(np.int64))):
        util.check_wave_documents(s, names, part_off, None, rep_off, cur, out, out_len, B, weight=w)


@pytest.mark.gpu
def test_errors(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 21), 4))
    rng = np.random.default_rng(4)
    Q, T = 1000, 10
    cur_lists = [[int(x) for x in rng.choice(np.arange(1, 21), int(rng.integers(0, 4)), replace=False)] for _ in range(Q)]
    new_lists = [c if rng.random() < 0.3 else [int(x) for x in rng.choice(np.arange(1, 21), int(rng.integers(0, 4)), replace=False)]
                 for c in cur_lists]
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 3)
    topic_names = ["err-%d" % t for t in range(T)]
    names, name_off = kab.Solver.marshal_names(topic_names)
    part_off = np.arange(T + 1, dtype=np.int64) * 100
    cap = models.json_bound(topic_names, part_off, 3)
    js, doc_off = np.zeros(cap, dtype=np.uint8), np.zeros(Q + 1, dtype=np.int64)
    wave, summ = np.zeros(Q, dtype=np.int32), np.zeros(Q, dtype=WAVE_SUMMARY_DTYPE)
    keys = ("s", "T", "part_off", "part_id", "rep_off", "cur", "stride", "new_len", "new", "weight", "B", "names", "name_off", "js",
            "json_cap", "doc_off", "wave", "summary", "cap")
    ok = (s, T, part_off, None, rep_off, cur, 3, out_len, out, None, 2, names, name_off, js, cap, doc_off, wave, summ, Q)

    def call(n=None, **kw):
        a = dict(zip(keys, ok))
        a.update(kw)
        rc, st, n = util.raw_plan_waves_json(*a.values(), n=n)
        assert rc == st.code
        if n is not False:
            assert rc == 0 or n.value == 0
        return rc, st.a, st.b

    assert call()[0] == 0
    # what ka_plan_waves refuses, with its operands
    assert call(stride=0)[0] == BAD and call(n=False)[0] == BAD and call(cap=-1)[0] == BAD
    assert call(summary=None)[0] == BAD and call(B=0)[0] == BAD
    bad_off = rep_off.copy()
    bad_off[500] = bad_off[501] + 1
    assert call(rep_off=bad_off)[0] == BAD and call(rep_off=rep_off + 1)[0] == BAD
    assert call(stride=9, new=np.full((Q, 9), -1, dtype=np.int32))[:2] == (LIMIT, 9)
    long_len = out_len.copy()
    long_len[[700, 300]] = [4, -1]
    assert call(new_len=long_len)[:2] == (BAD, 300)
    neg = np.ones(Q, dtype=np.int64)
    neg[10] = -1
    assert call(weight=neg)[0] == BAD
    edge = np.ones(Q, dtype=np.int64)
    edge[0] = INT64_MAX // 8 - 999
    assert call(weight=edge)[0] == 0
    edge[1] += 1
    assert call(weight=edge)[0] == LIMIT
    # the layout, the names and the buffers; the plan's refusals come first
    assert call(T=-1)[0] == BAD and call(part_off=None)[0] == BAD and call(part_off=part_off + 1)[0] == BAD
    dented = part_off.copy()
    dented[4] = dented[3] - 1
    assert call(part_off=dented)[0] == BAD
    assert call(names=None)[0] == BAD and call(name_off=None)[0] == BAD and call(js=None)[0] == BAD
    assert call(json_cap=-1)[0] == BAD and call(doc_off=None)[0] == BAD
    assert call(stride=9, new=np.full((Q, 9), -1, dtype=np.int32), js=None)[:2] == (LIMIT, 9)
    for ch in (b'"', b"\\", b"/", b"\x1f"):
        odd = names.copy()
        odd[7] = ch[0]
        assert call(names=odd)[:2] == (BAD, ch[0])
        assert call(names=odd, new_len=long_len)[:2] == (BAD, 300)
    # on the device the plan's lowest failing row wins
    for rows, expect in (({700: [5, 5], 300: [1, 99]}, (BAD, 300, 99)), ({999: [21]}, (BAD, 999, 21)), ({0: [3, 3]}, (BAD, 0, 3))):
        o, ln = out.copy(), out_len.copy()
        for g, x in rows.items():
            o[g, :] = -1
            o[g, :len(x)] = x
            ln[g] = len(x)
        assert call(new=o, new_len=ln) == expect
        assert call(new=o, new_len=ln, json_cap=0) == expect
    # the text's exact size succeeds, one byte less is KA_ERR_LIMIT with a = json_cap; the bound always succeeds
    e_docs = models.wave_documents(topic_names, part_off, None, rep_off, cur, out, out_len, s.broker_id, 2)[0]
    size = sum(len(d) for d in e_docs)
    assert 0 < size <= cap
    assert call(json_cap=size - 1)[:2] == (LIMIT, size - 1) and call(json_cap=0)[:2] == (LIMIT, 0)
    js[:] = 0
    rc, _, n = util.raw_plan_waves_json(*ok[:14], size, *ok[15:])
    assert rc == 0 and n.value == len(e_docs) and bytes(js[:size]) == b"".join(e_docs) and not js[size:].any()
    assert doc_off[:n.value + 1].tolist() == np.concatenate([[0], np.cumsum([len(d) for d in e_docs])]).tolist()
    # Q == 0: no document, doc_off[0] = 0 when given
    doc_off[0] = 5
    assert call(T=0)[0] == 0 and doc_off[0] == 0
    assert call(T=0, doc_off=None, names=None, name_off=None, part_off=None)[0] == 0
    # a summary capacity below W, and no wave array: the documents all the same
    few = np.zeros(2, dtype=WAVE_SUMMARY_DTYPE)
    js[:] = 0
    rc, _, n = util.raw_plan_waves_json(*ok[:16], None, few, 2)
    assert rc == 0 and n.value == len(e_docs) > 2 and bytes(js[:size]) == b"".join(e_docs)
    assert [util.record_of(x, WAVE_SUMMARY_DTYPE.names) for x in few] == [util.record_of(x, WAVE_SUMMARY_DTYPE.names) for x in summ[:2]]


@pytest.mark.gpu
def test_context_is_untouched_and_launches_follow_the_bits_of_w(native_lib):
    import torch
    cl = kab.synth.make_ragged_cluster(T=3000, N=400, max_partitions=128, seed=21, remove_frac=0.02)
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    args = (cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    out, out_len, _ = s.solve_ragged(*args)
    # a dense solve left pending on its stream: its status is still there to collect after the call
    rng = np.random.default_rng(6)
    dT, dP = 50, 16
    d_hash_h = rng.integers(-2 ** 31 + 1, 2 ** 31 - 1, dT).astype(np.int32)
    d_cur_h = np.stack([rng.choice(cl.broker_id, 3, replace=False) for _ in range(dT * dP)]).astype(np.int32).reshape(dT, dP, 3)
    s2 = kab.Solver(0)
    s2.set_brokers(cl.broker_id, cl.rack_index)
    d_hash, d_cur = torch.as_tensor(d_hash_h, device="cuda"), torch.as_tensor(d_cur_h, device="cuda")
    d_out = torch.full((dT * dP, 3), -1, dtype=torch.int32, device="cuda")
    d_len = torch.zeros(dT * dP, dtype=torch.int32, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    s2.solve_dense_device(dT, d_hash.data_ptr(), dP, 3, d_cur.data_ptr(), -1, 3, d_len.data_ptr(), d_out.data_ptr(),
                          stream=stream.cuda_stream, sync=False)
    docs, _, _, st = s2.plan_waves_json(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, 2)
    assert st.code == 0 and len(docs) > 1
    assert s2.last_status().code == 0
    ref = kab.Solver(0)
    ref.set_brokers(cl.broker_id, cl.rack_index)
    ref_out, _, _ = ref.solve_dense(d_hash_h, d_cur_h, -1, 3)
    assert np.array_equal(d_out.cpu().numpy().reshape(ref_out.shape), ref_out) and np.array_equal(s2.counters(), ref.counters())

    before = (s.counters(), s.last_order_plan(), s.last_stage_plan())
    docs, _, _, st = s.plan_waves_json(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, 2)
    assert st.code == 0 and len(docs) > 1
    assert np.array_equal(s.counters(), before[0]) and (s.last_order_plan(), s.last_stage_plan()) == before[1:]
    again, again_len, _ = s.solve_ragged(*args)
    fresh = kab.Solver(0)
    fresh.set_brokers(cl.broker_id, cl.rack_index)
    fresh.solve_ragged(*args)
    f_out, f_len, _ = fresh.solve_ragged(*args)
    assert np.array_equal(again, f_out) and np.array_equal(again_len, f_len)

    # launches: the plan's 7, then 3 per radix pass (8 bits of W each) and the 3 text kernels; none of the latter when W = 0
    def launches(Q, same=False):
        names, part_off = _one_topic(Q)
        rep_off, cur = util.cur_lists([[1]] * Q)
        o, ln = util.rows([[1 if same else 2]] * Q)
        n0 = s.launch_count()
        docs, _, _, st = s.plan_waves_json(names, part_off, None, rep_off, cur, o, ln, 1)
        assert st.code == 0 and len(docs) == (0 if same else Q)
        return s.launch_count() - n0

    n0 = s.launch_count()
    s.plan_waves(cl.rep_off, cl.cur, out, out_len, 2)
    assert s.launch_count() - n0 == 7
    assert launches(100) == launches(120) == launches(255) == 7 + 3 + 3
    assert launches(256) == launches(3000) == 7 + 6 + 3
    assert launches(500, same=True) == 7


@pytest.mark.gpu
def test_cpp_host_mirror(native_lib):
    """host/test_waves_json.cpp: every document of KafkaTopicAssigner::planWavesJson equals newAssignmentJson of the same wave of
    planWaves, and names that need escapes give the host emitter's text."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_WAVES_JSON_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
