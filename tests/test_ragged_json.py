"""ka_solve_json: the ragged solve + the reassignment JSON (KAG:169-186) built on the device, and the CLI that prints it.
Every text is compared byte for byte with text built on the host from the oracle's rows, in the predicted org.json key order
(SURVEY §3.4); every error with what ka_solve reports for the same input."""
import ctypes
import json
import random
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from tests import models, util


def _json(solver, names, th, part_off, part_id, rep_off, cur, desired, **kw):
    text, st = solver.solve_ragged_json(names, th, part_off, part_id, rep_off, cur, desired, check=False, **kw)
    return bytes(text).decode(), st


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_solve_json_without_a_context_is_no_device(native_lib):
    st = kab.KaStatus()
    nbytes = ctypes.c_int64(7)
    buf = ctypes.create_string_buffer(64)
    rc = native_lib.ka_solve_json(None, 0, None, None, None, None, None, -1, None, None, buf, 64, ctypes.byref(nbytes), ctypes.byref(st))
    assert rc == st.code == kab._native.KA_ERR_NO_DEVICE and nbytes.value == 0


def test_make_ragged_cluster_is_seeded_and_ragged():
    a = kab.synth.make_ragged_cluster(T=3000, N=60, R=6, seed=4, remove_frac=0.1)
    b = kab.synth.make_ragged_cluster(T=3000, N=60, R=6, seed=4, remove_frac=0.1)
    for f in ("part_off", "part_id", "rep_off", "cur", "broker_id", "rack_index"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    P, sizes = np.diff(a.part_off), np.diff(a.rep_off)
    assert P.min() == 1 and P.max() > 100 and np.median(P) < 10          # heavy tail of partition counts
    assert set(np.unique(sizes)) == {1, 2, 3}                            # RF 1..3
    assert any(r is None for r in a.rack_name) and any(r is not None for r in a.rack_name)
    assert a.N == 54 and len(a.all_broker_id) == 60 and np.all(np.diff(a.broker_id) > 0)
    for g in range(0, a.Q, 13):                                          # lists hold distinct brokers
        lst = a.cur[a.rep_off[g]:a.rep_off[g + 1]]
        assert len(set(lst.tolist())) == len(lst)
    assert not np.array_equal(kab.synth.make_ragged_cluster(T=3000, N=60, R=6, seed=5).cur[:500], a.cur[:500])


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _error_cases():
    """One case of every reference exception (KTA:58-60, 65-66, 67-69; KAS:183-184, 190-192)."""
    return [
        dict(topics=[("ok", {0: [1, 2]}), ("t", {3: [1, 2], 9: [1]})], brokers=[1, 2, 3], racks={}, desired_rf=-1),
        dict(topics=[("ok", {0: [1, 2]}), ("none", {})], brokers=[1, 2, 3], racks={}, desired_rf=-1),
        dict(topics=[("t", {-4: [1, 2, 3]})], brokers=[1, 2], racks={}, desired_rf=-1),
        dict(topics=[("t", {0: [1, 2], 7: [2, 1]})], brokers=[1, 2, 3], racks={1: "x", 2: "x", 3: "y"}, desired_rf=3),
        dict(topics=[("polygenelubricants", {5: [1, 2, 3]})], brokers=[1, 2, 3], racks={}, desired_rf=-1),
    ]


@pytest.mark.gpu
def test_random_ragged_cases_json_vs_oracle(native_lib, oracle):
    """~300 seeded cases: sparse and negative partition ids, topics without partitions, lists of 1..5 replicas, desired RF
    above and below the current one (the 4..8-wide chain builds text too), part_id given or NULL; and every error kind."""
    rng = random.Random(23)
    s, ref = kab.Solver(0), kab.Solver(0)
    cases = []
    for it in range(300):
        nb = rng.randint(1, 40)
        brokers = sorted(rng.sample(range(-5, 200), nb))
        racks = {b: "k%d" % rng.randrange(max(2, nb // 3)) for b in brokers if rng.random() < 0.7}
        universe = brokers + [1000, 1001, -77]
        topics = []
        for ti in range(rng.randint(1, 6)):
            rf = rng.randint(1, min(5, nb))
            ragged = rng.random() < 0.2
            lo = rng.choice([0, 0, -1000, -2**31])
            ids = sorted(rng.sample(range(lo, lo + rng.choice([80, 5000, 2**31 - 1])), rng.randint(0 if rng.random() < 0.08 else 1, 60)))
            if rng.random() < 0.3:
                ids = list(range(len(ids)))
            topics.append(("rt%d_%d" % (it, ti), {p: rng.sample(universe, min(rng.randint(0, 5) if ragged else rf, len(universe))) for p in ids}))
        cases.append(dict(topics=topics, brokers=brokers, racks=racks, desired_rf=rng.choice([-1, -1, -1, 1, 2, 3, 4, 5, 0])))
    cases += _error_cases()
    kinds, n_ok, n_wide = set(), 0, 0
    for it, case in enumerate(cases):
        names, part_off, part_id, rep_off, cur = util.flatten(case["topics"])
        brokers = sorted(case["brokers"])
        desired = case["desired_rf"]
        exp, est = util.oracle_text(oracle, names, part_off, part_id, rep_off, cur, brokers, [case["racks"].get(b) for b in brokers], desired)
        th = np.array([kab.java_string_hash(n) for n in names], dtype=np.int32)
        if all(np.array_equal(part_id[part_off[t]:part_off[t + 1]], np.arange(part_off[t + 1] - part_off[t])) for t in range(len(names))) \
                and it % 2:
            part_id = None                                               # the ordinal form
        for solver in (s, ref):
            solver.reset()
            solver.set_brokers_with_racks(brokers, case["racks"])
        text, st = _json(s, names, th, part_off, part_id, rep_off, cur, desired)
        _, _, rst = ref.solve_ragged(th, part_off, part_id, rep_off, cur, desired, util.row_width(rep_off, desired), check=False)
        assert util.fields(st) == util.fields(rst), (it, case)
        if exp is None:
            assert text == "" and (st.code, st.topic_index, st.partition, st.a, st.b) == (est.code, est.topic_index, est.partition, est.a, est.b), (it, case)
            kinds.add(st.code)
        else:
            assert st.code == 0 and text == exp, (it, case)
            assert np.array_equal(s.counters(), ref.counters()), it
            n_ok += 1
            n_wide += util.row_width(rep_off, desired) >= 4
    assert kinds == {1, 2, 3, 4, 5} and n_ok > 60 and n_wide > 20, (kinds, n_ok, n_wide)


def _fast_text(oracle, cl):
    out, ln, est = oracle.fast_run_dense(oracle.FastContext(), cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index)
    assert est.code == 0
    part_off, part_id, _, _ = cl.ragged()
    return models.solve_document(cl.topic_names, part_off, part_id, out, ln)


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["c2", "c3"])
def test_baseline_configs_through_the_ragged_entry(native_lib, oracle, key):
    """The dense BASELINE shapes fed as ragged input: the same text as ka_solve_dense_json and as the oracle's rows; config 3
    (1.28 M rows) is streamed in several fragments of a fixed row count (3 kernel launches each)."""
    cl = kab.synth.make_config(key, "mixed")
    part_off, part_id, rep_off, cur = cl.ragged()
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    text, st = _json(s, cl.topic_names, cl.topic_hash, part_off, part_id, rep_off, cur, -1)
    assert st.code == 0
    d = kab.Solver(0)
    d.set_brokers(cl.broker_id, cl.rack_index)
    dense, dst = d.solve_dense_json(cl.topic_names, cl.topic_hash, cl.cur)
    assert dst.code == 0 and text == bytes(dense).decode()
    assert text == _fast_text(oracle, cl)
    r = kab.Solver(0)
    r.set_brokers(cl.broker_id, cl.rack_index)
    r.solve_ragged(cl.topic_hash, part_off, part_id, rep_off, cur, -1, cl.RF)
    fragments = (s.launch_count() - r.launch_count()) // 3
    assert fragments == -(-(cl.T * cl.P) // (1 << 18))
    if key == "c3":
        assert fragments > 1
    assert np.array_equal(s.counters(), r.counters())


@pytest.mark.gpu
def test_million_partition_ragged_cluster(native_lib, oracle):
    cl = kab.synth.make_ragged_cluster(T=240000, N=400, max_partitions=128, seed=11, remove_frac=0.05)
    assert cl.Q > 1_000_000
    octx = oracle.OracleContext()
    exp, est = util.oracle_text(oracle, cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, cl.broker_id, cl.rack_name, -1, octx)
    assert est.code == 0
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    text, st = _json(s, cl.topic_names, cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1)
    assert st.code == 0 and text == exp
    r = kab.Solver(0)
    r.set_brokers(cl.broker_id, cl.rack_index)
    r.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    ctr = s.counters()
    assert np.array_equal(ctr, r.counters())
    for i, bid in enumerate(cl.broker_id):
        assert [ctr[i, k] for k in range(3)] == [octx.counter(int(bid), k) for k in range(3)], int(bid)


@pytest.mark.gpu
def test_edge_cases(native_lib, oracle):
    s = kab.Solver(0)
    s.set_brokers(np.arange(1, 7, dtype=np.int32), np.arange(6, dtype=np.int32))
    names = ["a", "b"]
    th = np.array([kab.java_string_hash(n) for n in names], dtype=np.int32)
    part_off, part_id, rep_off, cur = (np.array([0, 2, 3], dtype=np.int64), np.array([0, 4, 1], dtype=np.int32),
                                       np.array([0, 2, 4, 6], dtype=np.int64), np.array([1, 2, 2, 3, 4, 1], dtype=np.int32))
    # the empty run: no topics, or only topics without partitions under a desired RF
    assert _json(s, [], np.zeros(0, np.int32), np.zeros(1, np.int64), None, np.zeros(1, np.int64), np.zeros(0, np.int32), -1)[0] == models.EMPTY_DOCUMENT
    text, st = _json(s, names, th, np.zeros(3, np.int64), None, np.zeros(1, np.int64), np.zeros(0, np.int32), 2)
    assert st.code == 0 and text == models.EMPTY_DOCUMENT
    text, st = _json(s, names, th, np.zeros(3, np.int64), None, np.zeros(1, np.int64), np.zeros(0, np.int32), -1)
    assert (st.code, st.topic_index, text) == (2, 0, "")                  # KTA:65-66 without a desired RF
    # a name the device emitter would have to escape: refused before anything is solved
    s.reset()
    assert _json(s, names, th, part_off, part_id, rep_off, cur, -1)[1].code == 0
    before = s.counters()
    assert before.any()
    for bad in ('a"b', "a\\b", "a/b", "a\tb"):
        text, st = _json(s, [bad, "b"], th, part_off, part_id, rep_off, cur, -1)
        assert (st.code, text) == (kab._native.KA_ERR_BAD_ARG, ""), bad
        assert np.array_equal(s.counters(), before)
    # buffer sizes: exact fits, one byte short is KA_ERR_LIMIT with no text
    s.reset()
    exp, _ = _json(s, names, th, part_off, part_id, rep_off, cur, -1)
    for cap, code in ((len(exp), 0), (len(exp) - 1, kab._native.KA_ERR_LIMIT)):
        s.reset()
        buf = np.zeros(cap, dtype=np.uint8)
        text, st = _json(s, names, th, part_off, part_id, rep_off, cur, -1, json_buf=buf)
        assert st.code == code and text == (exp if code == 0 else "")
    buf = np.zeros(len(models.EMPTY_DOCUMENT) - 1, dtype=np.uint8)
    assert _json(s, [], np.zeros(0, np.int32), np.zeros(1, np.int64), None, np.zeros(1, np.int64), np.zeros(0, np.int32), -1,
                 json_buf=buf)[1].code == kab._native.KA_ERR_LIMIT


# ---- the CLI ------------------------------------------------------------------------------------------------------
def _snapshot(tmp_path, cl, topics, fname="cluster.json"):
    brokers = [dict(id=int(b), host="h%d" % b, port=9092, **({"rack": r} if r is not None else {}))
               for b, r in zip(cl.all_broker_id, cl.all_rack_name)]
    parts = [dict(topic=n, partition=p, replicas=r) for n, asg in topics for p, r in asg.items()]
    path = tmp_path / fname
    path.write_text(json.dumps(dict(brokers=brokers, topics=[n for n, _ in topics], partitions=parts)))
    return str(path)


def _cli_expected(oracle, cl, topics, live, desired):
    names, part_off, part_id, rep_off, cur = util.flatten(topics)
    racks = dict(zip(cl.all_broker_id.tolist(), cl.all_rack_name))
    new, st = util.oracle_text(oracle, names, part_off, part_id, rep_off, cur, live, [racks[b] for b in live], desired)
    assert st.code == 0
    current = ",".join('{"topic":%s,"partition":%d,"replicas":[%s]}' % (models.kafka_quote(n), p, ",".join(map(str, asg[p])))
                       for n, asg in topics for p in sorted(asg))
    return "CURRENT ASSIGNMENT:\n" + '{"version":1,"partitions":[' + current + ']}' + "\nNEW ASSIGNMENT:\n" + new + "\n"


@pytest.mark.gpu
def test_cli_prints_device_json_for_a_ragged_snapshot(native_lib, oracle, tmp_path):
    cli = kab.build_mod.build_host()
    cl = kab.synth.make_ragged_cluster(T=1800, N=60, R=6, max_partitions=16, seed=3)
    assert cl.Q >= 5000
    topics = cl.topics()
    snap = _snapshot(tmp_path, cl, topics)
    all_ids = cl.all_broker_id.tolist()
    gone = all_ids[5:8]
    for args, live, desired in (([], all_ids, -1),
                                (["--broker_hosts_to_remove", ",".join("h%d" % b for b in gone)], [b for b in all_ids if b not in gone], -1),
                                (["--desired_replication_factor", "2"], all_ids, 2),
                                (["--broker_hosts_to_remove", "h%d" % gone[0], "--desired_replication_factor", "3"], [b for b in all_ids if b != gone[0]], 3)):
        r = subprocess.run([cli, "--zk_string", "file:" + snap, "--mode", "PRINT_REASSIGNMENT"] + args, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and r.stderr == "", r.stderr
        assert r.stdout == _cli_expected(oracle, cl, topics, live, desired), args
    # a topic name org.json escapes goes through the host emitter, with the same text
    quoted = [('a"b', topics[0][1])] + topics[1:40]
    snap = _snapshot(tmp_path, cl, quoted, "quoted.json")
    r = subprocess.run([cli, "--zk_string", snap, "--mode", "PRINT_REASSIGNMENT"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout == _cli_expected(oracle, cl, quoted, all_ids, -1)
    assert '"topic":"a\\"b"' in r.stdout
