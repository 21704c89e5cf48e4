"""ka_plan_waves_json_parts and ka_plan_waves_send_json_parts on the GPU: every part, its wave, D, wave and the summaries of the
device must equal `models.wave_documents` byte for byte; with a limit above every wave the text and doc_off must be those of
ka_plan_waves(_send)_json."""
import ctypes
import json
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SEND_SUMMARY_DTYPE, WAVE_SUMMARY_DTYPE
from tests import models, util

pytestmark = pytest.mark.gpu
BAD, LIMIT = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT
ZNODE = 0xFFFFF   # ZooKeeper's default jute.maxbuffer


@pytest.mark.parametrize("seed", range(3))
def test_random_ragged_cases(native_lib, seed):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 31), 4))
    rng = np.random.default_rng(100 + seed)
    names, part_off, part_id, rep_off, cur, out, out_len = util.ragged_wave_case(rng, 300, 30)
    weight = rng.integers(0, 50, len(out_len)).astype(np.int64)
    for B, w, C in ((1, None, None), (4, None, None), (10 ** 9, None, None), (60, weight, None), (2, None, 3), (80, weight, 200)):
        wave = s.plan_waves(rep_off, cur, out, out_len, B, weight=w)[0]
        small = util.smallest_limit(names, part_off, part_id, rep_off, cur, out, out_len, wave)
        for L in (small, small + 1, 500, 3000, 70000, ZNODE):
            st = util.check_wave_documents(s, names, part_off, part_id, rep_off, cur, out, out_len, B, L, weight=w, C=C)[5]
            assert st.code == 0
        parts = util.check_wave_documents(s, names, part_off, part_id, rep_off, cur, out, out_len, B, small, weight=w, C=C)[0]
        assert len(parts) >= len(set(wave[wave > 0].tolist()))


@pytest.mark.parametrize("send", [False, True])
def test_a_limit_above_every_wave_gives_the_wave_documents(native_lib, send):
    cl = kab.synth.make_ragged_cluster(T=3000, N=200, max_partitions=64, seed=5, remove_frac=0.02)
    s, out, out_len, S = util.solved(cl)
    kw = dict(max_broker_out=5, send_brokers=cl.all_broker_id) if send else {}   # removed brokers still send
    for B in (2, 10 ** 9):
        docs, wave, summ, st = s.plan_waves_json(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, B, **kw)
        assert st.code == 0
        buf = np.zeros(models.json_bound(cl.topic_names, cl.part_off, S), dtype=np.uint8)
        parts, part_wave, p_wave, p_summ, st = s.plan_wave_parts_json(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out,
                                                                      out_len, B, max(len(d) for d in docs), json_buf=buf, **kw)
        assert st.code == 0 and part_wave.tolist() == list(range(1, len(docs) + 1))
        assert np.array_equal(p_wave, wave) and np.array_equal(p_summ, summ)
        assert [bytes(p) for p in parts] == [bytes(d) for d in docs]
        # doc_off: the parts lie back to back from the buffer's start
        text = b"".join(bytes(d) for d in docs)
        assert bytes(buf[:len(text)]) == text
        util.check_wave_documents(s, cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, B, 4096,
                                  C=5 if send else None, send_ids=cl.all_broker_id)


def test_parts_straddle_ctas_and_the_staging_limit(native_lib):
    """Names of about 400 bytes beside short ones: CTAs whose text exceeds the 64 KiB stage write straight to global memory, and
    parts start and end inside CTAs and across their boundaries."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))
    rng = np.random.default_rng(9)
    T, Q = 40, 6000
    names = [("long-%02d-" % t) + "x" * int(rng.integers(380, 420)) if t % 4 else "s%d" % t for t in range(T)]
    part_off = np.arange(T + 1) * (Q // T)
    cur_l = [[int(x) for x in rng.choice(np.arange(1, 31), 3, replace=False)] for _ in range(Q)]
    new_l = [[c[0], c[1], int(rng.integers(31, 41))] if rng.random() < 0.8 else c for c in cur_l]
    rep_off, cur = util.cur_lists(cur_l)
    out, out_len = util.rows(new_l, 3)
    for B in (50, 10 ** 6):
        for L in (1000, 5000, 64 * 1024, 200 * 1024, ZNODE):
            parts, _, _, _, _, st = util.check_wave_documents(s, names, part_off, None, rep_off, cur, out, out_len, B, L)
            assert st.code == 0
    assert len(parts) > 1


@pytest.mark.parametrize("weighted", [False, True])
def test_one_wave_of_more_than_65536_parts(native_lib, weighted):
    """Every row reordered only (wave 1) and the smallest L: one part per row, 70 000 parts in one wave (17 doubling levels)."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 11), 2))
    Q = 70000
    names, part_off = ["w"], np.array([0, Q], dtype=np.int64)
    part_id = np.full(Q, 7, dtype=np.int32)   # every record the same length
    rep_off, cur = util.cur_lists([[1, 2]] * Q)
    out, out_len = util.rows([[2, 1]] * Q)
    w = np.arange(Q, dtype=np.int64) % 5 if weighted else None
    L = 29 + len(models.record("w", 7, [2, 1]))
    n0 = s.launch_count()
    st = s.plan_wave_parts_json(names, part_off, part_id, rep_off, cur, out, out_len, 1, L, weight=w)[4]
    # launches: the plan's 7, one radix pass, 4, 2 x 17 - 1 doubling, the 3 text passes
    assert st.code == 0 and s.launch_count() - n0 == 7 + 3 + 4 + 33 + 3
    parts, _, part_wave, _, _, st = util.check_wave_documents(s, names, part_off, part_id, rep_off, cur, out, out_len, 1, L, weight=w)
    assert st.code == 0 and len(parts) == Q and set(part_wave.tolist()) == {1}
    parts = util.check_wave_documents(s, names, part_off, part_id, rep_off, cur, out, out_len, 1, 3 * L, weight=w)[0]
    assert Q // 4 <= len(parts) < Q // 2


def test_no_wave_and_no_rows(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 11), 2))
    rep_off, cur = util.cur_lists([[1, 2]] * 50)
    out, out_len = util.rows([[1, 2]] * 50)
    for names, part_off in ((["x"], [0, 50]), ([], [0]), (["x", "y"], [0, 0, 0])):
        Q = part_off[-1]
        parts, part_wave, wave, summ, st = s.plan_wave_parts_json(names, np.asarray(part_off), None, rep_off[:Q + 1], cur[:rep_off[Q]],
                                                                  out[:Q], out_len[:Q], 1, 100)
        assert st.code == 0 and parts == [] and len(part_wave) == 0 and not wave.any() and len(summ) == 0


def _raw(s, T, part_off, rep_off, cur, stride, new_len, new, B, names, name_off, js, json_cap, L, doc_off, doc_wave, n_docs=True,
         summary=None, cap=0):
    st = kab.KaStatus()
    n, d = ctypes.c_int32(-7), ctypes.c_int32(-7)
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = s._L.ka_plan_waves_json_parts(s._h, T, p(part_off), None, p(rep_off), p(cur), stride, p(new_len), p(new), None, B, p(names),
                                       p(name_off), p(js), json_cap, L, p(doc_off), p(doc_wave), ctypes.byref(d) if n_docs else None,
                                       None, ctypes.byref(n), p(summary), cap, ctypes.byref(st))
    assert rc == st.code
    if rc:
        assert n.value == 0 and (not n_docs or d.value == 0)
    return rc, st.a, st.b, d.value


def test_errors(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 21), 4))
    rng = np.random.default_rng(4)
    Q, T = 1000, 10
    cur_l = [[int(x) for x in rng.choice(np.arange(1, 21), int(rng.integers(1, 4)), replace=False)] for _ in range(Q)]
    new_l = [c if rng.random() < 0.3 else [int(x) for x in rng.choice(np.arange(1, 21), int(rng.integers(0, 4)), replace=False)]
             for c in cur_l]
    rep_off, cur = util.cur_lists(cur_l)
    out, out_len = util.rows(new_l, 3)
    topic_names = ["err-%d" % t for t in range(T)]
    names, name_off = kab.Solver.marshal_names(topic_names)
    part_off = np.arange(T + 1, dtype=np.int64) * 100
    cap = models.json_bound(topic_names, part_off, 3)
    js, doc_off, doc_wave = np.zeros(cap, dtype=np.uint8), np.zeros(Q + 1, dtype=np.int64), np.zeros(Q, dtype=np.int32)
    ok = dict(T=T, part_off=part_off, rep_off=rep_off, cur=cur, stride=3, new_len=out_len, new=out, B=2, names=names, name_off=name_off,
              js=js, json_cap=cap, L=ZNODE, doc_off=doc_off, doc_wave=doc_wave)

    def call(**kw):
        return _raw(s, **dict(ok, **kw))

    assert call()[0] == 0
    # L < 1 and the missing outputs, after every check of ka_plan_waves_json
    assert call(L=0)[0] == BAD and call(L=-5)[0] == BAD and call(doc_wave=None)[0] == BAD and call(n_docs=False)[0] == BAD
    assert call(L=0, stride=9, new=np.full((Q, 9), -1, dtype=np.int32))[:2] == (LIMIT, 9)
    assert call(L=0, js=None)[0] == BAD and call(L=0, B=0)[0] == BAD
    # Q == 0: nothing required, doc_off[0] = 0
    doc_off[0] = 5
    assert call(T=0, doc_wave=None, n_docs=False)[0] == 0 and doc_off[0] == 0
    # the lowest over-long changed row, with its one-record document's length; the plan's row errors come first
    lens = {}
    wave = s.plan_waves(rep_off, cur, out, out_len, 2)[0]
    for g in range(Q):
        if wave[g]:
            t = g // 100
            lens[g] = 29 + len(models.record(topic_names[t], g - 100 * t, new_l[g]))
    longest = max(lens.values())
    low = min(g for g, n in lens.items() if n == longest)
    assert call(L=longest - 1)[:3] == (LIMIT, low, longest)
    assert call(L=longest)[0] == 0
    assert call(L=1)[:3] == (LIMIT, min(lens), lens[min(lens)])
    o, ln = out.copy(), out_len.copy()
    o[999, :2], ln[999] = [4, 4], 2
    assert call(L=1, new=o, new_len=ln)[:3] == (BAD, 999, 4)
    # over-long rows come before json_cap; then a text above json_cap is KA_ERR_LIMIT with a = json_cap
    e_parts = models.wave_documents(topic_names, part_off, None, rep_off, cur, out, out_len, s.broker_id, 2, L=300)[0]
    size = sum(len(p) for p in e_parts)
    assert call(L=300, json_cap=size - 1)[:2] == (LIMIT, size - 1)
    assert call(L=longest - 1, json_cap=0)[:3] == (LIMIT, low, longest)
    js[:] = 0
    rc, _, _, D = call(L=300, json_cap=size)
    assert rc == 0 and D == len(e_parts) and bytes(js[:size]) == b"".join(e_parts) and not js[size:].any()
    assert doc_off[:D + 1].tolist() == np.concatenate([[0], np.cumsum([len(p) for p in e_parts])]).tolist()


@pytest.mark.parametrize("remove", [0.0, 0.02])
def test_million_partition_cluster_under_the_znode_limit(native_lib, remove):
    cl = kab.synth.make_ragged_cluster(T=240000, N=400, max_partitions=128, seed=11, remove_frac=remove)
    s, out, out_len, S = util.solved(cl)
    B = len(out_len) if remove == 0.0 else 4000   # everything in wave 1 (one solve's document under the limit), or waves
    parts, _, part_wave, _, _, st = util.check_wave_documents(s, cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out,
                                                              out_len, B, ZNODE)
    assert st.code == 0
    assert (part_wave == 1).sum() >= 25   # the reorder-only rows of wave 1 alone are about 25 MB
    for p in parts:
        assert len(p) <= ZNODE and json.loads(bytes(p))["version"] == 1


def test_cpp_host_mirror(native_lib):
    """host/test_wave_parts.cpp: KafkaTopicAssigner::planWaveParts against planWavesJson, on the device and host paths."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_WAVE_PARTS_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
