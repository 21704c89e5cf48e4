"""ka_plan_waves_json_parts_rollback and ka_plan_waves_send_json_parts_rollback on the GPU: every part, every rollback document,
D, part_wave, wave and the summaries of the device must equal `models.wave_documents` byte for byte; every rollback
document must name exactly its part's partitions, in order, on their current lists; where no current list prints longer than
its new list the results must be those of ka_plan_waves(_send)_json_parts."""
import ctypes
import json
import re
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


def _current(names, part_off, part_id, rep_off, cur):
    """(topic, partition) -> its current list."""
    got = {}
    for t, name in enumerate(names):
        for g in range(int(part_off[t]), int(part_off[t + 1])):
            p = int(part_id[g]) if part_id is not None else g - int(part_off[t])
            got[(name, p)] = cur[int(rep_off[g]):int(rep_off[g + 1])].tolist()
    return got


def _check_pairs(parts, rollback, current, L):
    """Every rollback document parses to its part's partitions, in order, on their current lists; both sides <= L."""
    for p, b in zip(parts, rollback):
        assert len(p) <= L and len(b) <= L
        fwd, back = json.loads(bytes(p)), json.loads(bytes(b))
        assert list(back) == ["version", "partitions"] and back["version"] == 1
        assert [(r["topic"], r["partition"]) for r in back["partitions"]] == [(r["topic"], r["partition"]) for r in fwd["partitions"]]
        assert all(r["replicas"] == current[(r["topic"], r["partition"])] for r in back["partitions"])


@pytest.mark.parametrize("seed", range(3))
def test_random_ragged_cases(native_lib, seed):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 31), 4))
    rng = np.random.default_rng(200 + seed)
    case = util.ragged_wave_case(rng, 300, 30, shrink=0.3)
    names, part_off, part_id, rep_off, cur, out, out_len = case
    current = _current(names, part_off, part_id, rep_off, cur)
    weight = rng.integers(0, 50, len(out_len)).astype(np.int64)
    for B, w, C in ((1, None, None), (4, None, None), (10 ** 9, None, None), (60, weight, None), (2, None, 3), (80, weight, 200)):
        wave = s.plan_waves(rep_off, cur, out, out_len, B, weight=w)[0]
        small = util.smallest_limit(*case, wave, rollback=True)
        for L in (small, small + 1, 500, 3000, 70000, ZNODE):
            parts, rollback, _, _, _, st = util.check_wave_documents(s, *case, B, L, True, weight=w, C=C)
            assert st.code == 0
            _check_pairs(parts, rollback, current, L)
        assert len(parts) >= len(set(wave[wave > 0].tolist()))


@pytest.mark.parametrize("send", [False, True])
def test_no_longer_current_lists_give_the_parts_call(native_lib, send):
    """The proposed lists of a solve that only adds brokers (desired RF 3 over RF <= 3 topics) never print shorter than the
    current lists when the ids have as many digits: the paired cut is the one-sided one, byte for byte."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(10, 50), 4))
    rng = np.random.default_rng(31)
    Q, T = 4000, 40
    names = ["same.%d" % t for t in range(T)]
    part_off = np.arange(T + 1, dtype=np.int64) * (Q // T)
    cur_l = [[int(x) for x in rng.choice(np.arange(10, 50), int(rng.integers(0, 3)), replace=False)] for _ in range(Q)]
    new_l = [c + [int(x) for x in rng.choice(np.setdiff1d(np.arange(10, 50), c), 3 - len(c), replace=False)] if rng.random() < 0.7
             else c for c in cur_l]
    rep_off, cur = util.cur_lists(cur_l)
    out, out_len = util.rows(new_l, 3)
    kw = dict(max_broker_out=6, send_brokers=list(range(10, 50))) if send else {}
    for B in (3, 40, 10 ** 6):
        for L in (200, 1000, 30000, ZNODE):
            parts, part_wave, wave, summ, st = s.plan_wave_parts_json(names, part_off, None, rep_off, cur, out, out_len, B, L, **kw)
            r_parts, rollback, r_part_wave, r_wave, r_summ, r_st = s.plan_wave_parts_rollback_json(names, part_off, None, rep_off, cur,
                                                                                                   out, out_len, B, L, **kw)
            assert st.code == r_st.code == 0
            assert [bytes(p) for p in r_parts] == [bytes(p) for p in parts] and np.array_equal(r_part_wave, part_wave)
            assert np.array_equal(r_wave, wave) and np.array_equal(r_summ, summ) and len(rollback) == len(parts)
            _check_pairs(r_parts, rollback, _current(names, part_off, None, rep_off, cur), L)


def test_a_replication_factor_reduction_takes_more_parts(native_lib):
    """desired_rf = 2 over a cluster with RF-3 topics: their rollback records are the longer side and force the cut."""
    cl = kab.synth.make_ragged_cluster(T=2000, N=120, max_partitions=48, seed=8, remove_frac=0.0)
    s, out, out_len, S = util.solved(cl, desired_rf=2)
    current = _current(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur)
    for L in (4000, 65536, ZNODE):
        parts, _, _, _, st = s.plan_wave_parts_json(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, 10 ** 9, L)
        assert st.code == 0
        r_parts, rollback, _, _, _, st = util.check_wave_documents(s, cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out,
                                                                   out_len, 10 ** 9, L, True)
        assert st.code == 0 and len(r_parts) >= len(parts) and (L > 4000 or len(r_parts) > len(parts))
        _check_pairs(r_parts, rollback, current, L)


@pytest.mark.parametrize("send", [False, True])
def test_a_limit_above_every_document_gives_the_wave_documents(native_lib, send):
    cl = kab.synth.make_ragged_cluster(T=3000, N=200, max_partitions=64, seed=5, remove_frac=0.02)
    s, out, out_len, S = util.solved(cl)
    kw = dict(max_broker_out=5, send_brokers=cl.all_broker_id) if send else {}   # removed brokers still send
    current = _current(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur)
    for B in (2, 10 ** 9):
        docs, wave, summ, st = s.plan_waves_json(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, B, **kw)
        assert st.code == 0
        L = 10 ** 9
        parts, rollback, part_wave, p_wave, p_summ, st = s.plan_wave_parts_rollback_json(cl.topic_names, cl.part_off, cl.part_id,
                                                                                         cl.rep_off, cl.cur, out, out_len, B, L, **kw)
        assert st.code == 0 and part_wave.tolist() == list(range(1, len(docs) + 1))
        assert np.array_equal(p_wave, wave) and np.array_equal(p_summ, summ)
        assert [bytes(p) for p in parts] == [bytes(d) for d in docs]
        _check_pairs(parts, rollback, current, L)
        util.check_wave_documents(s, cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, B, 4096, True,
                                  C=5 if send else None, send_ids=cl.all_broker_id)


def test_parts_straddle_ctas_and_the_staging_limit(native_lib):
    """Names of about 400 bytes beside short ones: CTAs whose text exceeds the 64 KiB stage write straight to global memory on
    both sides, and parts start and end inside CTAs and across their boundaries. Long current lists (6 brokers) make the
    rollback side the longer one for most rows."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))
    rng = np.random.default_rng(19)
    T, Q = 40, 6000
    names = [("long-%02d-" % t) + "x" * int(rng.integers(380, 420)) if t % 4 else "s%d" % t for t in range(T)]
    part_off = np.arange(T + 1) * (Q // T)
    cur_l = [[int(x) for x in rng.choice(np.arange(1, 31), int(rng.integers(1, 7)), replace=False)] for _ in range(Q)]
    new_l = [[c[0], int(rng.integers(31, 41))] if rng.random() < 0.8 else c[:3] for c in cur_l]
    rep_off, cur = util.cur_lists(cur_l)
    out, out_len = util.rows(new_l, 3)
    current = _current(names, part_off, None, rep_off, cur)
    for B in (50, 10 ** 6):
        for L in (1000, 5000, 64 * 1024, 200 * 1024, ZNODE):
            parts, rollback, _, _, _, st = util.check_wave_documents(s, names, part_off, None, rep_off, cur, out, out_len, B, L, True)
            assert st.code == 0
            _check_pairs(parts, rollback, current, L)
    assert len(parts) > 1


def test_launches_are_those_of_the_parts_call_and_three(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 31), 4))
    rng = np.random.default_rng(5)
    for T, B, L in ((300, 1, 500), (300, 10 ** 9, 3000), (40, 4, ZNODE), (600, 2, 300)):
        case = util.ragged_wave_case(rng, T, 30, shrink=0.3)
        wave = s.plan_waves(*case[3:7], B)[0]
        L = max(L, util.smallest_limit(*case, wave, rollback=True))
        n0 = s.launch_count()
        st = s.plan_wave_parts_json(*case, B, L)[4]
        n1 = s.launch_count()
        # the paired cut may make a wave's widest run of parts differ, not its row count: the doubling levels stay the same
        st2 = s.plan_wave_parts_rollback_json(*case, B, L)[5]
        assert st.code == st2.code == 0 and s.launch_count() - n1 == n1 - n0 + 3
    # no wave: the plan's launches only, as the _parts call
    rep_off, cur = util.cur_lists([[1, 2]] * 50)
    out, out_len = util.rows([[1, 2]] * 50)
    n0 = s.launch_count()
    s.plan_wave_parts_json(["x"], np.array([0, 50]), None, rep_off, cur, out, out_len, 1, 100)
    n1 = s.launch_count()
    r = s.plan_wave_parts_rollback_json(["x"], np.array([0, 50]), None, rep_off, cur, out, out_len, 1, 100)
    assert r[5].code == 0 and r[0] == r[1] == [] and s.launch_count() - n1 == n1 - n0


def _raw(s, T, part_off, rep_off, cur, stride, new_len, new, B, names, name_off, js, json_cap, L, doc_off, doc_wave, back, back_cap,
         back_off, n_docs=True):
    st = kab.KaStatus()
    n, d = ctypes.c_int32(-7), ctypes.c_int32(-7)
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = s._L.ka_plan_waves_json_parts_rollback(s._h, T, p(part_off), None, p(rep_off), p(cur), stride, p(new_len), p(new), None, B,
                                                p(names), p(name_off), p(js), json_cap, L, p(doc_off), p(doc_wave),
                                                ctypes.byref(d) if n_docs else None, p(back), back_cap, p(back_off), None,
                                                ctypes.byref(n), None, 0, ctypes.byref(st))
    assert rc == st.code
    if rc:
        assert n.value == 0 and (not n_docs or d.value == 0)
    return rc, st.a, st.b, d.value


def test_errors(native_lib):
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 21), 4))
    rng = np.random.default_rng(4)
    Q, T = 1000, 10
    cur_l = [[int(x) for x in rng.choice(np.arange(1, 21), int(rng.integers(1, 6)), replace=False)] for _ in range(Q)]
    new_l = [c[:3] if rng.random() < 0.3 else [int(x) for x in rng.choice(np.arange(1, 21), int(rng.integers(0, 4)), replace=False)]
             for c in cur_l]
    rep_off, cur = util.cur_lists(cur_l)
    out, out_len = util.rows(new_l, 3)
    topic_names = ["err-%d" % t for t in range(T)]
    names, name_off = kab.Solver.marshal_names(topic_names)
    part_off = np.arange(T + 1, dtype=np.int64) * 100
    cap = models.json_bound(topic_names, part_off, 3)
    back_bound = models.json_bound(topic_names, part_off, 0) + 12 * len(cur)
    js, doc_off, doc_wave = np.zeros(cap, dtype=np.uint8), np.zeros(Q + 1, dtype=np.int64), np.zeros(Q, dtype=np.int32)
    back, back_off = np.zeros(back_bound, dtype=np.uint8), np.zeros(Q + 1, dtype=np.int64)
    ok = dict(T=T, part_off=part_off, rep_off=rep_off, cur=cur, stride=3, new_len=out_len, new=out, B=2, names=names, name_off=name_off,
              js=js, json_cap=cap, L=ZNODE, doc_off=doc_off, doc_wave=doc_wave, back=back, back_cap=back_bound, back_off=back_off)

    def call(**kw):
        return _raw(s, **dict(ok, **kw))

    assert call()[0] == 0
    # back, back_cap and back_off after every check of ka_plan_waves_json_parts
    assert call(back=None)[0] == BAD and call(back_cap=-1)[0] == BAD and call(back_off=None)[0] == BAD
    assert call(back=None, L=0)[0] == BAD and call(back=None, doc_wave=None)[0] == BAD
    assert call(back=None, stride=9, new=np.full((Q, 9), -1, dtype=np.int32))[:2] == (LIMIT, 9)
    # Q == 0: back_off not required, back_off[0] = 0
    back_off[0] = 5
    assert call(T=0, doc_wave=None, n_docs=False, back_off=None)[0] == 0
    assert call(T=0, doc_wave=None, n_docs=False)[0] == 0 and back_off[0] == 0
    # the lowest over-long changed row on either side, with the longer length; the plan's row errors come first
    lens = {}
    wave = s.plan_waves(rep_off, cur, out, out_len, 2)[0]
    for g in range(Q):
        if wave[g]:
            t = g // 100
            lens[g] = 29 + max(len(models.record(topic_names[t], g - 100 * t, new_l[g])),
                               len(models.current_record(topic_names[t], g - 100 * t, cur_l[g])))
    longest = max(lens.values())
    low = min(g for g, n in lens.items() if n == longest)
    assert call(L=longest - 1)[:3] == (LIMIT, low, longest)
    assert call(L=longest)[0] == 0
    assert call(L=1)[:3] == (LIMIT, min(lens), lens[min(lens)])
    o, ln = out.copy(), out_len.copy()
    o[999, :2], ln[999] = [4, 4], 2
    assert call(L=1, new=o, new_len=ln)[:3] == (BAD, 999, 4)
    # over-long rows, then json_cap, then back_cap; each cap one byte short is refused and exact is taken
    e_parts, e_back = models.wave_documents(topic_names, part_off, None, rep_off, cur, out, out_len, s.broker_id, 2, L=400,
                                            rollback=True)[:2]
    size, bsize = sum(len(p) for p in e_parts), sum(len(p) for p in e_back)
    assert call(L=400, json_cap=size - 1)[:2] == (LIMIT, size - 1)
    assert call(L=400, json_cap=size - 1, back_cap=0)[:2] == (LIMIT, size - 1)
    assert call(L=400, back_cap=bsize - 1)[:2] == (LIMIT, bsize - 1)
    assert call(L=longest - 1, json_cap=0, back_cap=0)[:3] == (LIMIT, low, longest)
    js[:] = 0
    back[:] = 0
    rc, _, _, D = call(L=400, json_cap=size, back_cap=bsize)
    assert rc == 0 and D == len(e_parts) == len(e_back)
    assert bytes(js[:size]) == b"".join(e_parts) and not js[size:].any()
    assert bytes(back[:bsize]) == b"".join(e_back) and not back[bsize:].any()
    assert back_off[:D + 1].tolist() == np.concatenate([[0], np.cumsum([len(p) for p in e_back])]).tolist()


@pytest.mark.parametrize("remove", [0.0, 0.02])
def test_million_partition_cluster_under_the_znode_limit(native_lib, remove):
    cl = kab.synth.make_ragged_cluster(T=240000, N=400, max_partitions=128, seed=11, remove_frac=remove)
    s, out, out_len, S = util.solved(cl)
    B = len(out_len) if remove == 0.0 else 4000
    parts, rollback, part_wave, _, _, st = util.check_wave_documents(s, cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out,
                                                                     out_len, B, ZNODE, True)
    assert st.code == 0 and (part_wave == 1).sum() >= 25
    _check_pairs(parts, rollback, _current(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur), ZNODE)


def test_rollback_text_past_4_gib(native_lib):
    """68 000 rows in topics of names of about 64 KiB: the rollback text passes 2^32 bytes, so back_off and the text positions
    of the CTAs beyond it need their 64 bits. Three short-named topics at the end keep CTAs on the staged store path past 2^32.
    The expected documents are printed with placeholder names and cut by the real record lengths; the whole expected text is
    never built."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))
    rng = np.random.default_rng(15)
    lens = rng.integers(65000, 65537, 68)
    names = ["L%02d-" % t + "n" * (int(n) - 4) for t, n in enumerate(lens)] + ["s%d" % t for t in range(3)]
    part_off = np.concatenate([[0], np.cumsum([1000] * 68 + [800] * 3)]).astype(np.int64)
    Q = int(part_off[-1])
    g = np.arange(Q)
    rep_off, cur = util.cur_lists([[1, 2, 3]] * Q)   # every rollback record longer than its forward one
    out, out_len = util.rows([[1, 2, 3] if x % 50 == 0 else [1, 4 + x % 4] for x in g.tolist()], 3)
    B, L = 2, ZNODE
    ph = ["@%d@" % t for t in range(len(names))]
    real = [n.encode() for n in names]
    wave = models.plan_waves(rep_off, cur, out, out_len, s.broker_id, B)[0]
    recs = {}
    for t in range(len(names)):
        for r in range(int(part_off[t]), int(part_off[t + 1])):
            if wave[r]:
                f = models.record(ph[t], r - int(part_off[t]), out[r][:int(out_len[r])]).encode()
                b = models.current_record(ph[t], r - int(part_off[t]), cur[3 * r:3 * r + 3]).encode()
                grow = len(real[t]) - len(ph[t])
                recs.setdefault(int(wave[r]), []).append((f, b, len(f) + grow, len(b) + grow))
    topic = re.compile(rb'"topic":"@(\d+)@"')

    def expand(doc):
        return topic.sub(lambda m: b'"topic":"' + real[int(m.group(1))] + b'"', doc)

    e_back = []
    for v in sorted(recs):
        rs = recs[v]
        for a, b in models.cut_parts([[x[2] for x in rs], [x[3] for x in rs]], L):
            e_back.append((b'{"version":1,"partitions":[' + b",".join(x[1] for x in rs[a:b]) + b"]}", b - a))
    slab, name_off = kab.Solver.marshal_names(names)
    cap = models.json_bound(names, part_off, 3)
    back_cap = models.json_bound(names, part_off, 0) + 12 * len(cur)
    js, back = np.empty(cap, dtype=np.uint8), np.empty(back_cap, dtype=np.uint8)
    doc_off, doc_wave, back_off = np.zeros(Q + 1, dtype=np.int64), np.zeros(Q, dtype=np.int32), np.zeros(Q + 1, dtype=np.int64)
    rc, _, _, D = _raw(s, len(names), part_off, rep_off, cur, 3, out_len, out, B, slab, name_off, js, cap, L, doc_off, doc_wave, back,
                       back_cap, back_off)
    assert rc == 0 and D == len(e_back)
    assert back_off[D] > 1 << 32
    at = 0
    straddle = 0
    for d, (doc, rows) in enumerate(e_back):
        e = expand(doc)
        assert int(back_off[d]) == at, d
        assert back[at:at + len(e)].tobytes() == e, d
        # the forward part names the same rows
        fwd = js[int(doc_off[d]):int(doc_off[d + 1])].tobytes()
        assert fwd.count(b'{"partition":') == rows and len(fwd) <= L and len(e) <= L
        straddle += at < 1 << 32 < at + len(e)
        at += len(e)
    assert int(back_off[D]) == at and straddle == 1
    s.close()


def test_cpp_host_mirror(native_lib):
    """host/test_wave_rollback.cpp: KafkaTopicAssigner::planWavePartsRollback against kafkaReassignmentJson, on the device and
    host paths."""
    kab.build_mod.build_host()
    r = subprocess.run([kab.build_mod.HOST_WAVE_ROLLBACK_TEST], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
