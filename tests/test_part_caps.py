"""The part caps (ka_ctx_set_part_caps): the most rows and the most data (weight x receivers) one part of a wave holds, beside the
byte limit of the four _parts entry points. CPU tests check the capped cut of tests/part_cap_models.py against a brute-force statement of the rule and
what Solver.set_part_caps hands the C ABI; GPU tests check every capped document, doc_off, doc_wave, wave and summary of the
device byte for byte against its capped wave documents, for the four entry points under both wave rules."""
import ctypes
import json
import os
import subprocess
import threading

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from tests import models, util
from tests import part_cap_models as pcm

BAD, NO_DEVICE = _native.KA_ERR_BAD_ARG, _native.KA_ERR_NO_DEVICE
ZNODE = 0xFFFFF   # ZooKeeper's default jute.maxbuffer


# ---- the model cut ---------------------------------------------------------------------------------------------------------

def _fits(sides, a, L, Lr, Lx, i, j):
    """Whether records i..j-1 make a part under the rule of include/kassign.h."""
    n = j - i
    if any(29 + sum(s[i:j]) + n - 1 > L for s in sides):
        return False
    if Lr is not None and n > Lr:
        return False
    return Lx is None or n == 1 or sum(a[i:j]) <= Lx


def _brute_cut(sides, a, L, Lr, Lx):
    """From each part's first record, the longest run that fits (every condition is monotone, so the longest is the greedy)."""
    runs, i, m = [], 0, len(sides[0])
    while i < m:
        j = max(j for j in range(i + 1, m + 1) if all(_fits(sides, a, L, Lr, Lx, i, k) for k in range(i + 1, j + 1)))
        runs.append((i, j))
        i = j
    return runs


@pytest.mark.parametrize("seed", range(4))
def test_model_cut_is_the_unique_greedy_cut(seed):
    rng = np.random.default_rng(seed)
    for _ in range(300):
        m = int(rng.integers(1, 14))
        sides = [rng.integers(40, 90, m).tolist() for _ in range(int(rng.integers(1, 3)))]
        a = (rng.integers(0, 4, m) * (rng.random(m) < 0.7)).tolist()   # reorder-only rows move nothing
        L = 29 + max(max(s) for s in sides) + int(rng.integers(0, 400))
        Lr = None if rng.random() < 0.3 else int(rng.integers(1, 6))
        Lx = None if rng.random() < 0.3 else int(rng.integers(1, 8))
        runs = pcm.cut_parts(sides, L, Lr, Lx, a)
        assert runs == _brute_cut(sides, a, L, Lr, Lx)
        assert runs[0][0] == 0 and runs[-1][1] == m and all(x[1] == y[0] for x, y in zip(runs, runs[1:]))
        for i, j in runs:   # every part within Lr and Lx, or a single row
            assert Lr is None or j - i <= Lr
            assert Lx is None or j - i == 1 or sum(a[i:j]) <= Lx
        for (i, _), (_, j) in zip(runs, runs[1:]):   # no two consecutive parts could be merged
            assert not _fits(sides, a, L, Lr, Lx, i, j)
        assert pcm.cut_parts(sides, L, a=a) == models.cut_parts(sides, L)   # no caps: the uncapped cut


def test_model_caps_off_gives_the_uncapped_documents():
    rng = np.random.default_rng(3)
    ids = np.arange(1, 21, dtype=np.int32)
    names, part_off, part_id, rep_off, cur, out, out_len = util.ragged_wave_case(rng, 40, 20)
    weight = rng.integers(0, 9, len(out_len)).astype(np.int64)
    for L, rollback in ((400, False), (900, True)):
        base = models.wave_documents(names, part_off, part_id, rep_off, cur, out, out_len, ids, 3, weight, None, L, rollback)
        args = (names, part_off, part_id, rep_off, cur, out, out_len, ids, 3, weight, None, L, rollback)
        assert pcm.wave_documents(*args)[:3] == base[:3]
        recs = pcm.wave_records(names, part_off, part_id, rep_off, cur, out, out_len, base[3], weight)
        docs, backs, doc_wave, _ = pcm.cut_documents(recs, L, rollback=rollback)   # the capped cut with no caps
        assert (docs, backs if rollback else None, doc_wave) == base[:3]
        capped = pcm.wave_documents(*args, Lr=2, Lx=5)
        assert b"".join(capped[0]) != b"".join(base[0]) and len(capped[0]) > len(base[0])
        assert np.array_equal(capped[3], base[3]) and capped[4] == base[4]


# ---- the Python mirror -------------------------------------------------------------------------------------------------------

class _CapsLib:
    """Stands in for ka_ctx_set_part_caps / ka_ctx_part_caps: records what they are handed, refuses a negative cap as the
    library does and keeps the caps otherwise."""

    def __init__(self):
        self.calls, self.caps = [], (0, 0)

    def ka_ctx_set_part_caps(self, h, rows, data):
        self.calls.append((rows, data))
        if rows < 0 or data < 0:
            return BAD
        self.caps = (rows, data)
        return 0

    def ka_ctx_part_caps(self, h, rows, data):
        rows._obj.value, data._obj.value = self.caps
        return 0


def test_set_part_caps_marshals_its_arguments():
    lib = _CapsLib()
    s = util.fake_solver(lib)
    assert s.part_caps() == (None, None)
    s.set_part_caps(max_rows=10000)
    s.set_part_caps(max_in=7)
    s.set_part_caps(12, 3)
    assert lib.calls == [(10000, 0), (0, 7), (12, 3)] and s.part_caps() == (12, 3)
    s.set_part_caps(0, None)
    assert lib.calls[-1] == (0, 0) and s.part_caps() == (None, None)
    s.set_part_caps(5, 6)
    for bad in (dict(max_rows=-1), dict(max_in=-2), dict(max_rows=3, max_in=-1)):
        with pytest.raises(ValueError):
            s.set_part_caps(**bad)
    assert lib.calls[-1] == (5, 6) and s.part_caps() == (5, 6)   # a refused cap never reaches the library


def test_abi_declares_the_part_caps(native_lib):
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kassign.h")).read()
    assert "int32_t ka_ctx_set_part_caps(ka_ctx* ctx, int64_t max_part_rows, int64_t max_part_in);" in header
    assert "int32_t ka_ctx_part_caps(ka_ctx* ctx, int64_t* max_part_rows, int64_t* max_part_in);" in header
    rows, data = ctypes.c_int64(-9), ctypes.c_int64(-9)
    assert native_lib.ka_ctx_set_part_caps(None, 1, 1) == NO_DEVICE
    assert native_lib.ka_ctx_part_caps(None, ctypes.byref(rows), ctypes.byref(data)) == NO_DEVICE
    assert rows.value == data.value == -9


# ---- the device --------------------------------------------------------------------------------------------------------------

ENTRIES = [(False, False), (True, False), (False, True), (True, True)]   # (sender budget, rollback)


def _solver(n=30, rule="greedy"):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, n + 1), 4))
    s.set_wave_rule(rule)
    return s


def _fit_documents(s, case, B, L, Lr, Lx, weight, send, rollback, json_buf):
    """Under the first-fit rule: the plan against fit_models.plan_waves (util.check_plan), then the documents of the call
    against the capped cut over that plan's waves, the records in input row order. Returns the shape of check_wave_documents."""
    names, part_off, part_id, rep_off, cur, out, out_len = case
    send_ids = list(np.asarray(s.broker_id))
    p_wave, p_summ, p_st = util.check_plan(s, rep_off, cur, out, out_len, B, weight, send_ids if send else None, 3 if send else None)
    assert p_st.code == 0
    kw = dict(max_broker_out=3, send_brokers=send_ids) if send else {}
    if rollback:
        got = s.plan_wave_parts_rollback_json(names, part_off, part_id, rep_off, cur, out, out_len, B, L, weight=weight, json_buf=json_buf,
                                              **kw)
    else:
        docs, doc_wave, wave, summ, st = s.plan_wave_parts_json(names, part_off, part_id, rep_off, cur, out, out_len, B, L, weight=weight,
                                                                json_buf=json_buf, **kw)
        got = (docs, None, doc_wave, wave, summ, st)
    assert got[5].code == 0 and np.array_equal(got[3], p_wave) and np.array_equal(got[4], p_summ)
    recs = pcm.wave_records(names, part_off, part_id, rep_off, cur, out, out_len, p_wave, weight)
    e_docs, e_backs, e_doc_wave, _ = pcm.cut_documents(recs, L, Lr, Lx, rollback)
    assert [bytes(d) for d in got[0]] == e_docs and got[2].tolist() == e_doc_wave
    if rollback:
        assert [bytes(d) for d in got[1]] == e_backs
    return got


def _check(s, case, B, L, Lr=None, Lx=None, weight=None, send=False, rollback=False):
    """check_wave_documents under the caps (set on s here; under the first-fit rule _fit_documents), and doc_off: the documents
    lie back to back from the buffer's start (the back buffer's too). Returns its result."""
    names, part_off, part_id, rep_off, cur, out, out_len = case
    s.set_part_caps(Lr, Lx)
    Lr, Lx = Lr or None, Lx or None   # 0 is no cap
    buf = np.zeros(models.json_bound(names, part_off, out.shape[1]) + 16, dtype=np.uint8)
    if s.wave_rule == "first_fit":
        got = _fit_documents(s, case, B, L, Lr, Lx, weight, send, rollback, buf)
    else:
        got = pcm.check_wave_documents(s, names, part_off, part_id, rep_off, cur, out, out_len, B, L, rollback=rollback, weight=weight,
                                        C=3 if send else None, json_buf=buf, Lr=Lr, Lx=Lx)
    assert got[5].code == 0
    text = b"".join(bytes(d) for d in got[0])
    assert bytes(buf[:len(text)]) == text
    if rollback:   # the rollback views lie back to back in their own buffer
        starts = [b.__array_interface__["data"][0] for b in got[1]]
        assert all(y - x == len(b) for x, y, b in zip(starts, starts[1:], got[1]))
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("rule", ["greedy", "first_fit"])
@pytest.mark.parametrize("send,rollback", ENTRIES)
def test_random_ragged_cases(native_lib, rule, send, rollback):
    s = _solver(rule=rule)
    rng = np.random.default_rng(7 + 2 * send + rollback)
    case = util.ragged_wave_case(rng, 250, 30, shrink=0.1 if rollback else 0.0)
    weight = rng.integers(0, 50, len(case[6])).astype(np.int64)
    for w in (None, weight):
        mean = 1 if w is None else max(int(w.mean()), 1)
        for B in (2, 10 ** 9):
            for Lr, Lx in ((3, None), (None, 2 * mean), (5, 3 * mean), (1, 1)):
                for L in (700, ZNODE):
                    got = _check(s, case, B, L, Lr, Lx, w, send, rollback)
                    assert Lr is None or all(len(json.loads(bytes(d))["partitions"]) <= Lr for d in got[0])


@pytest.mark.gpu
@pytest.mark.parametrize("send,rollback", ENTRIES)
def test_caps_off_and_cleared_match_a_fresh_context(native_lib, send, rollback):
    rng = np.random.default_rng(21)
    case = util.ragged_wave_case(rng, 200, 30)
    fresh, used = _solver(), _solver()
    for L in (600, ZNODE):
        ref = _check(fresh, case, 3, L, send=send, rollback=rollback)
        used.set_part_caps(2, 1)
        _check(used, case, 3, L, 2, 1, send=send, rollback=rollback)
        for Lr, Lx in ((None, None), (0, 0)):   # never set, and cleared
            got = _check(used, case, 3, L, Lr, Lx, send=send, rollback=rollback)
            assert [bytes(d) for d in got[0]] == [bytes(d) for d in ref[0]] and np.array_equal(got[2], ref[2])
            if rollback:
                assert [bytes(d) for d in got[1]] == [bytes(d) for d in ref[1]]


def _moved(case, weight=None):
    names, part_off, part_id, rep_off, cur, out, out_len = case
    return np.array([pcm.moved_data(rep_off, cur, out, out_len, weight, g) for g in range(len(out_len))])


def _part_rows(case, docs):
    """The rows of every part, through the partition ids in its records (one topic per part id here)."""
    names, part_off, part_id = case[:3]
    row_of = {(names[t], int(part_id[g])): g for t in range(len(names)) for g in range(int(part_off[t]), int(part_off[t + 1]))}
    return [[row_of[(r["topic"], r["partition"])] for r in json.loads(bytes(d))["partitions"]] for d in docs]


@pytest.mark.gpu
@pytest.mark.parametrize("send,rollback", ENTRIES)
def test_each_cap_as_the_binding_one(native_lib, send, rollback):
    s = _solver()
    rng = np.random.default_rng(33)
    case = util.ragged_wave_case(rng, 200, 30)
    wave = s.plan_waves(*case[3:7], 4)[0]
    changed = int((wave > 0).sum())
    # Lr = 1: one part per changed row
    assert len(_check(s, case, 4, ZNODE, Lr=1, send=send, rollback=rollback)[0]) == changed
    # Lx = 1 at unit weights: every moved row alone, the reorder-only rows (a = 0) join freely
    a = _moved(case)
    docs = _check(s, case, 4, ZNODE, Lx=1, send=send, rollback=rollback)[0]
    assert all(sum(a[g] > 0 for g in rows) <= 1 or len(rows) == 1 for rows in _part_rows(case, docs))
    assert len(docs) < changed and any(len(rows) > 1 for rows in _part_rows(case, docs))
    # weights with zeros, and rows heavier than Lx: those stand alone
    weight = rng.integers(0, 4, len(case[6])).astype(np.int64) * rng.integers(0, 2, len(case[6]))
    aw = _moved(case, weight)
    docs = _check(s, case, 4, ZNODE, Lx=3, weight=weight, send=send, rollback=rollback)[0]
    parts = _part_rows(case, docs)
    assert any(aw[g] > 3 for g in range(len(aw)) if wave[g])
    for rows in parts:
        assert len(rows) == 1 or sum(aw[g] for g in rows) <= 3
        assert all(len(rows) == 1 for g in rows if aw[g] > 3)
    # one wave where the byte limit, Lr and Lx each decide a different cut
    B = 10 ** 9
    cuts = [tuple(len(r) for r in _part_rows(case, _check(s, case, B, 2000, Lr, Lx, send=send, rollback=rollback)[0]))
            for Lr, Lx in ((None, None), (6, None), (None, 4), (6, 4))]
    assert len(set(cuts)) == 4


@pytest.mark.gpu
def test_parts_straddle_ctas_and_the_staging_limit(native_lib):
    s = _solver(40)
    rng = np.random.default_rng(9)
    T, Q = 40, 6000
    names = [("long-%02d-" % t) + "x" * int(rng.integers(380, 420)) if t % 4 else "s%d" % t for t in range(T)]
    part_off = np.arange(T + 1) * (Q // T)
    cur_l = [[int(x) for x in rng.choice(np.arange(1, 31), 3, replace=False)] for _ in range(Q)]
    new_l = [[c[0], c[1], int(rng.integers(31, 41))] if rng.random() < 0.8 else c[::-1] for c in cur_l]
    rep_off, cur = util.cur_lists(cur_l)
    out, out_len = util.rows(new_l, 3)
    case = (names, part_off, np.tile(np.arange(Q // T, dtype=np.int32), T), rep_off, cur, out, out_len)
    for B in (50, 10 ** 6):
        for Lr, Lx in ((300, None), (None, 250), (700, 200), (257, 255)):
            for rollback in (False, True):
                _check(s, case, B, ZNODE, Lr, Lx, rollback=rollback)


@pytest.mark.gpu
def test_one_wave_of_more_than_65536_parts_by_the_row_cap(native_lib):
    """Every row reordered only (wave 1), a limit that never binds and Lr = 1: 70 000 parts in one wave (17 doubling levels), with
    exactly the launches of the uncapped call."""
    s = _solver(10)
    Q = 70000
    names, part_off = ["w"], np.array([0, Q], dtype=np.int64)
    part_id = np.arange(Q, dtype=np.int32)
    rep_off, cur = util.cur_lists([[1, 2]] * Q)
    out, out_len = util.rows([[2, 1]] * Q)
    case = (names, part_off, part_id, rep_off, cur, out, out_len)
    counts = []
    for Lr in (None, 1):
        s.set_part_caps(Lr, None)
        n0 = s.launch_count()
        st = s.plan_wave_parts_json(names, part_off, part_id, rep_off, cur, out, out_len, 1, ZNODE)[4]
        assert st.code == 0
        counts.append(s.launch_count() - n0)
    assert counts[0] == counts[1]
    parts = _check(s, case, 1, ZNODE, Lr=1)[0]
    assert len(parts) == Q
    assert len(_check(s, case, 1, ZNODE, Lr=3, Lx=1)[0]) == -(-Q // 3)   # nothing moves: Lx never binds


@pytest.mark.gpu
def test_no_wave_and_no_rows(native_lib):
    s = _solver(10)
    s.set_part_caps(1, 1)
    rep_off, cur = util.cur_lists([[1, 2]] * 50)
    out, out_len = util.rows([[1, 2]] * 50)
    for names, part_off in ((["x"], [0, 50]), ([], [0]), (["x", "y"], [0, 0, 0])):
        Q = part_off[-1]
        args = (names, np.asarray(part_off), None, rep_off[:Q + 1], cur[:rep_off[Q]], out[:Q], out_len[:Q], 1, 100)
        parts, part_wave, wave, summ, st = s.plan_wave_parts_json(*args)
        assert st.code == 0 and parts == [] and len(part_wave) == 0 and not wave.any() and len(summ) == 0
        parts, backs, part_wave, wave, summ, st = s.plan_wave_parts_rollback_json(*args)
        assert st.code == 0 and parts == [] and backs == [] and len(part_wave) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("send,rollback", ENTRIES)
def test_launch_counts_do_not_change_with_the_caps(native_lib, send, rollback):
    s = _solver()
    for topics in (20, 400):   # the same on any Q
        names, part_off, part_id, rep_off, cur, out, out_len = util.ragged_wave_case(np.random.default_rng(topics), topics, 30)
        kw = dict(max_broker_out=3, send_brokers=s.broker_id) if send else {}
        for Lr, Lx in ((2, None), (None, 1), (4, 2)):
            got = []
            for caps in ((Lr, Lx), (None, None)):
                s.set_part_caps(*caps)
                n0 = s.launch_count()
                if rollback:
                    st = s.plan_wave_parts_rollback_json(names, part_off, part_id, rep_off, cur, out, out_len, 3, 800, **kw)[5]
                else:
                    st = s.plan_wave_parts_json(names, part_off, part_id, rep_off, cur, out, out_len, 3, 800, **kw)[4]
                assert st.code == 0
                got.append(s.launch_count() - n0)
            assert got[0] == got[1]


@pytest.mark.gpu
@pytest.mark.parametrize("remove", [0.0, 0.02])
def test_million_partition_cluster_with_a_unit_data_cap(native_lib, remove):
    cl = kab.synth.make_ragged_cluster(T=240000, N=400, max_partitions=128, seed=11, remove_frac=remove)
    s, out, out_len, S = util.solved(cl)
    B = len(out_len) if remove == 0.0 else 4000
    s.set_part_caps(None, 1)
    parts, _, part_wave, wave, _, st = pcm.check_wave_documents(s, cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out,
                                                                 out_len, B, ZNODE, Lx=1)
    assert st.code == 0
    a = np.array([pcm.moved_data(cl.rep_off, cl.cur, out, out_len, None, g) for g in range(len(out_len))])
    # every part within the limit, and within Lx = 1 unless it is one row: at most one moved row per part
    moved_parts = 0
    rows = np.nonzero(wave)[0]
    order = rows[np.argsort(wave[rows], kind="stable")]
    at = 0
    for p in parts:
        n = len(json.loads(bytes(p))["partitions"])
        assert len(p) <= ZNODE
        moved = int((a[order[at:at + n]] > 0).sum())
        assert n == 1 or moved <= 1
        moved_parts += moved > 0
        at += n
    assert at == len(order) and moved_parts == int((a[order] > 0).sum())


@pytest.mark.gpu
def test_caps_are_per_context_across_threads(native_lib):
    rng = np.random.default_rng(44)
    case = util.ragged_wave_case(rng, 300, 30)
    solvers = [_solver(), _solver()]
    caps = [(2, None), (None, 1)]
    errors = []

    def run(k):
        try:
            for _ in range(3):
                _check(solvers[k], case, 3, ZNODE, *caps[k])
                assert solvers[k].part_caps() == caps[k]
        except Exception as e:   # noqa: BLE001 - reported on the main thread
            errors.append(e)

    threads = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


@pytest.mark.gpu
def test_cpp_host_mirror(native_lib):
    """host/test_part_caps.cpp: KafkaTopicAssigner::setPartCaps on the device and host paths."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_PART_CAPS_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
