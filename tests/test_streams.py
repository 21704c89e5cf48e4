"""The stream contract of the device entry points, and Contexts used at the same time.

include/kassign.h promises that a device-pointer call reads its inputs and writes its outputs in the order of the caller's
stream, that without a status it is fully asynchronous, and that different Contexts may be in flight at once, from different
host threads. The host driver keeps that promise by forking its own streams off the caller's and joining them back; these
tests check it without any device-wide synchronisation between enqueue and read. Two helpers do the work:

- late inputs: the device inputs hold a decoy (a valid cluster of the same shape over the same broker table) until, on the
  caller's stream, a device sleep and then a copy of the real inputs run. A read ahead of the copy sees the decoy's valid ids:
  the rows come out wrong and nothing faults. The sleep must outlast the host's enqueue of the call, which is checked.
- early reader: the outputs hold -7; straight after an asynchronous call they are cloned on the same stream, and only that
  stream is synchronised. A clone ahead of the library's last write sees -7 or rows of the decoy.

Every result is compared with the oracle: rows, list lengths, the full status and every Context counter. Threads run a fixed
sequence of calls once; they check results, they do not wait for a failure.
"""
import os
import re
import threading
import time
from unittest import mock

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from tests import fit_models, models, usage_models, util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kafka_assigner_b200", "csrc")

LEGACY = "legacy"     # the legacy default stream, passed to the library as 0
SIDE = "side"         # a torch.cuda.Stream of its own


# ---- CPU: one place sets a kernel's shared-memory cap ---------------------------------------------------------------------

def test_shared_memory_cap_is_set_in_one_guarded_place():
    """cudaFuncSetAttribute changes a kernel's cap for every Context of the process. kassign.cu calls it in exactly one place,
    allow_smem_of, which holds a lock and only ever raises the cap; no header calls it."""
    for f in sorted(os.listdir(CSRC)):
        if f.endswith(".cuh"):
            assert "cudaFuncSetAttribute" not in open(os.path.join(CSRC, f)).read(), f
    cu = open(os.path.join(CSRC, "kassign.cu")).read()
    assert len(re.findall(r"\bcudaFuncSetAttribute\s*\(", cu)) == 1
    body = re.search(r"\ncudaError_t allow_smem_of\(const void\* kernel, size_t bytes\) \{\n(.*?)\n\}\n", cu, re.S)
    assert body, "allow_smem_of moved: update this test"
    body = body.group(1)
    assert "cudaFuncSetAttribute(" in body
    lock, check, call = (body.find(x) for x in ("std::lock_guard<std::mutex>", "if (bytes <= have) return cudaSuccess;",
                                                "cudaFuncSetAttribute("))
    assert 0 <= lock < check < call, "the cap is set outside the lock or without the raise-only check"
    assert "have = bytes;" in body[call:]


# ---- helpers ---------------------------------------------------------------------------------------------------------------

def _stream(kind):
    """(torch stream, the handle the library takes)."""
    import torch
    if kind == LEGACY:
        s = torch.cuda.default_stream()
        assert s.cuda_stream == 0
        return s, 0
    s = torch.cuda.Stream()
    return s, s.cuda_stream


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def late_inputs(stream, pairs):
    """On `stream`: a device sleep, then dst.copy_(src) for every (dst, src). Returns the sleep's (start, end) events."""
    import torch
    sleep = util.device_sleep(stream)
    with torch.cuda.stream(stream):
        for dst, src in pairs:
            dst.copy_(src, non_blocking=True)
    return sleep


def early_read(stream, *tensors):
    """Clones of `tensors` on `stream`, enqueued at once; waits for that stream only. Returns them as numpy arrays."""
    import torch
    with torch.cuda.stream(stream):
        got = [t.clone() for t in tensors]
    stream.synchronize()
    return [g.cpu().numpy() for g in got]


def decoy_of(cl):
    """A valid cluster of cl's shape over cl's broker table, with other topics and other current lists."""
    m = cl.meta
    d = kab.synth.make_cluster(T=m["T"], P=m["P"], RF=m["RF"], N=m["N"], R=m["R"], seed=m["seed"] ^ 0xDEC0, kind="random",
                               topic_prefix="decoy-")
    assert np.array_equal(d.broker_id, cl.broker_id) and np.array_equal(d.rack_index, cl.rack_index)
    assert not np.array_equal(d.cur, cl.cur)
    return d


def expected(oracle, cl, table=None):
    """(rows [Q, S], lengths [Q], status fields, counters [N, 8]) of the oracle on a fresh Context."""
    ids, racks = table or (cl.broker_id, cl.rack_index)
    out, ln, st = oracle.fast_run_dense(oracle.FastContext(), cl.topic_hash, cl.cur, ids, racks)
    return out, ln, util.fields(st), models.histogram(ids, out, ln) if st.code == 0 else None


def oracle_from(oracle, cl, ctr):
    """(rows, lengths, status fields, counters [N, 8]) of the oracle from the preloaded counters ctr [N, 8]."""
    octx = oracle.OracleContext()
    for i, b in enumerate(cl.broker_id):
        for s in range(models.SLOTS):
            octx.set_counter(int(b), s, int(ctr[i, s]))
    part_off, part_id, rep_off, cur = cl.ragged()
    ln, _, out, st = oracle.run(octx, cl.topic_names, part_off, part_id, rep_off, cur, cl.broker_id, cl.rack_name, -1, cl.RF,
                                raise_on_error=False)
    got = np.array([[octx.counter(int(b), s) for s in range(models.SLOTS)] for b in cl.broker_id], dtype=np.int64)
    return out, ln, util.fields(st), got


class DeviceProblem:
    """A dense cluster's inputs on the device, holding its decoy's until late_inputs copies the real ones in, and its outputs."""

    def __init__(self, cl):
        import torch
        self.cl, self.S = cl, cl.RF
        dec = decoy_of(cl)
        self.d_hash, self.d_cur = _dev(dec.topic_hash), _dev(dec.cur)
        self.real = [(self.d_hash, _dev(cl.topic_hash)), (self.d_cur, _dev(cl.cur))]
        self.d_out = torch.full((cl.T, cl.P, self.S), -7, dtype=torch.int32, device="cuda")
        self.d_len = torch.full((cl.T, cl.P), -7, dtype=torch.int32, device="cuda")

    def solve_args(self):
        cl = self.cl
        return (cl.T, self.d_hash.data_ptr(), cl.P, cl.RF, self.d_cur.data_ptr(), -1, self.S, self.d_len.data_ptr(),
                self.d_out.data_ptr())

    def stage_args(self):
        cl = self.cl
        return cl.T, self.d_hash.data_ptr(), cl.P, cl.RF, self.d_cur.data_ptr(), -1, self.S

    def warm(self, s, table=None):
        """One synchronous solve of the decoy, so that the Context's scratch is reserved at this shape (a reservation that
        frees a smaller buffer waits for the device), then a fresh Context: the timed call enqueues without waiting."""
        import torch
        s.reset()
        s.set_brokers(*(table or (self.cl.broker_id, self.cl.rack_index)))
        s.solve_dense_device(*self.solve_args())
        s.reset()
        self.d_out.fill_(-7)
        self.d_len.fill_(-7)
        torch.cuda.synchronize()


def check_rows(got_out, got_len, exp, cid):
    out, ln = exp[0], exp[1]
    got_out, got_len = got_out.reshape(len(ln), -1), got_len.reshape(-1)
    bad = np.nonzero(np.any(got_out != out, axis=1) | (got_len != ln))[0]
    unwritten = int(np.sum(np.any(got_out[bad] == -7, axis=1) | (got_len[bad] == -7)))
    assert len(bad) == 0, (cid, "%d of %d rows differ from the oracle, first %s" % (len(bad), len(ln), bad[:5].tolist()),
                           "rows still holding -7: %d" % unwritten)


# ---- dense device solves: late inputs, early reader ----------------------------------------------------------------------

# (id, make_cluster shape, environment, (rec_kind, levels, chain launches)) — ka_ctx_last_order_plan fields 0, 1 and 6
DENSE_CASES = [
    ("slots-one-block", dict(T=40, P=16, RF=3, N=100, R=10), {}, (3, 0, 2)),
    ("rows4", dict(T=30, P=16, RF=4, N=80, R=8), {}, (4, 0, 1)),
    ("rows6-fused", dict(T=20, P=16, RF=6, N=120, R=8), {}, (8, 0, 1)),
    ("levels", dict(T=60, P=64, RF=3, N=30, R=5), {}, (3, 1, 2)),
    # 2 pipelined blocks of 2 048 topics, 4 chain sub-blocks each (as in test_chain_subblocks)
    ("pipelined-t4096", dict(T=4096, P=64, RF=3, N=300, R=12), {}, (3, 0, 2 * 2 * 4)),
    # 3 pipelined blocks of 300 topics, 2 chain sub-blocks each
    ("pipelined-3-stages", dict(T=900, P=32, RF=3, N=200, R=10), {"KA_PIPELINE_STAGES": "3"}, (3, 0, 3 * 2 * 2)),
    # one block, one chain sub-block: the solve's only emit writes all 262 144 rows after the slot-1 chain ends, so a reader
    # that is not held behind the emit (the join into the caller's stream) reads rows that are still -7
    ("one-long-emit", dict(T=2048, P=128, RF=3, N=400, R=10), {"KA_PIPELINE_STAGES": "1", "KA_CHAIN_SUBBLOCKS": "1"}, (3, 0, 2)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [SIDE, LEGACY])
@pytest.mark.parametrize("case", DENSE_CASES, ids=[c[0] for c in DENSE_CASES])
def test_dense_device_solve_follows_the_stream(native_lib, oracle, case, kind):
    """ka_solve_dense_device without a status: inputs copied in behind a sleep on the caller's stream, outputs cloned on it
    straight after the call; then ka_last_status, the rows, lengths and every counter against the oracle."""
    cid, shape, env, plan = case
    cl = kab.synth.make_cluster(seed=0x57EA + shape["T"] + shape["RF"], kind="mixed", **shape)
    exp = expected(oracle, cl)
    assert exp[2][0] == 0
    p = DeviceProblem(cl)
    s = kab.Solver(0)
    stream, h = _stream(kind)
    with mock.patch.dict(os.environ, env):
        p.warm(s)
        sleep = late_inputs(stream, p.real)
        t0 = time.perf_counter()
        s.solve_dense_device(*p.solve_args(), stream=h, sync=False)
        t_call = time.perf_counter() - t0
        out, ln = early_read(stream, p.d_out, p.d_len)
    util.enqueued_behind(sleep, t_call)
    assert util.fields(s.last_status()) == exp[2]
    got_plan = s.last_order_plan()
    assert (got_plan[0], got_plan[1], got_plan[6]) == plan, (cid, got_plan)
    check_rows(out, ln, exp, cid)
    assert np.array_equal(s.counters(), exp[3]), cid


@pytest.mark.gpu
def test_dense_candidates_device_reads_late_inputs(native_lib, oracle):
    """ka_solve_dense_candidates_device (synchronous) on a side stream whose inputs arrive behind a sleep: every candidate's
    rows, lengths and status equal the oracle's on a fresh Context of its table."""
    import torch
    cl = kab.synth.make_config("c2", "mixed")
    tables = kab.synth.decommission_tables("c2", [0.0, 0.1, 0.3])
    exps = [expected(oracle, cl, t) for t in tables]
    p = DeviceProblem(cl)
    K = len(tables)
    d_out = torch.full((K, cl.T, cl.P, cl.RF), -7, dtype=torch.int32, device="cuda")
    d_len = torch.full((K, cl.T, cl.P), -7, dtype=torch.int32, device="cuda")
    s = kab.Solver(0)
    args = (tables, cl.T, p.d_hash.data_ptr(), cl.P, cl.RF, p.d_cur.data_ptr(), -1, cl.RF, d_len.data_ptr(), d_out.data_ptr())
    s.solve_dense_candidates_device(*args)          # reserves the batch's scratch at this shape
    d_out.fill_(-7)
    d_len.fill_(-7)
    torch.cuda.synchronize()
    stream, h = _stream(SIDE)
    sleep = late_inputs(stream, p.real)
    sts = s.solve_dense_candidates_device(*args, stream=h)
    print("device sleep %.1f ms" % sleep[0].elapsed_time(sleep[1]))
    out, ln = early_read(stream, d_out, d_len)
    for k, e in enumerate(exps):
        assert util.fields(sts[k]) == e[2], k
        check_rows(out[k], ln[k], e, ("candidate", k))


# ---- the staged path on one stream ------------------------------------------------------------------------------------------

def _staged_problem(seed, RF=3):
    cl = kab.synth.make_cluster(T=300, P=32, RF=RF, N=150, R=10, seed=seed, kind="mixed")
    rng = np.random.default_rng(seed)
    ctr = np.zeros((cl.N, models.SLOTS), dtype=np.int64)
    return cl, rng, ctr


@pytest.mark.gpu
def test_staged_slot_chains_on_one_stream(native_lib, oracle):
    """stage, import a counter column written behind the sleep, slot-0 chain, export, import, slot-1 chain, emit: all on one
    side stream, no host synchronisation until the exported columns and rows are cloned on it."""
    import torch
    cl, rng, ctr = _staged_problem(0x57A6)
    cols = rng.integers(0, 40, size=(cl.N, 2))
    ctr[:, :2] = cols
    exp_out, exp_ln, exp_st, exp_ctr = oracle_from(oracle, cl, ctr)
    assert exp_st[0] == 0
    p = DeviceProblem(cl)
    s = kab.Solver(0)
    p.warm(s)
    col = [torch.full((cl.N,), 10**6, dtype=torch.int32, device="cuda") for _ in range(2)]     # the decoy columns
    got = [torch.full((cl.N,), -7, dtype=torch.int32, device="cuda") for _ in range(3)]
    torch.cuda.synchronize()
    stream, h = _stream(SIDE)
    sleep = late_inputs(stream, p.real + [(col[r], _dev(cols[:, r].astype(np.int32))) for r in range(2)])
    t0 = time.perf_counter()
    s.stage_dense_device(*p.stage_args(), stream=h)
    assert s.staged_slot_chains() == 2
    for slot in (0, 1):
        s.import_counter_slot_device(slot, col[slot].data_ptr(), stream=h)
        s.order_slot_device(slot, stream=h)
        s.export_counter_slot_device(slot, got[slot].data_ptr(), stream=h)
    s.emit_device(p.d_len.data_ptr(), p.d_out.data_ptr(), stream=h, sync=False)
    s.export_counter_slot_device(2, got[2].data_ptr(), stream=h)
    t_call = time.perf_counter() - t0
    out, ln, c0, c1, c2 = early_read(stream, p.d_out, p.d_len, *got)
    util.enqueued_behind(sleep, t_call)
    assert util.fields(s.last_status()) == exp_st
    check_rows(out, ln, (exp_out, exp_ln), "staged-slots")
    for slot, c in enumerate((c0, c1, c2)):
        assert np.array_equal(c, exp_ctr[:, slot]), slot
    assert np.array_equal(s.counters(), exp_ctr)


@pytest.mark.gpu
def test_staged_slot_chains_back_to_back(native_lib, oracle):
    """order_slot_device(0) and (1) with nothing between them, then an asynchronous emit: the rows and counters of a fresh
    Context, cloned on the stream straight after the emit."""
    cl, _, _ = _staged_problem(0x57A7)
    exp = expected(oracle, cl)
    p = DeviceProblem(cl)
    s = kab.Solver(0)
    p.warm(s)
    stream, h = _stream(SIDE)
    sleep = late_inputs(stream, p.real)
    t0 = time.perf_counter()
    s.stage_dense_device(*p.stage_args(), stream=h)
    s.order_slot_device(0, stream=h)
    s.order_slot_device(1, stream=h)
    s.emit_device(p.d_len.data_ptr(), p.d_out.data_ptr(), stream=h, sync=False)
    t_call = time.perf_counter() - t0
    out, ln = early_read(stream, p.d_out, p.d_len)
    util.enqueued_behind(sleep, t_call)
    assert util.fields(s.last_status()) == exp[2]
    check_rows(out, ln, exp, "back-to-back")
    assert np.array_equal(s.counters(), exp[3])


@pytest.mark.gpu
@pytest.mark.parametrize("RF", [3, 4])
def test_staged_order_with_device_counters(native_lib, oracle, RF):
    """The whole counter table imported from a buffer written behind the sleep, stage, ka_order_device without a status
    (rows of 3: slot chains and emits on the library's streams; rows of 4: one fused chain), the table exported: rows and
    the exported table, cloned on the stream, equal the oracle's from the same counters."""
    import torch
    cl, rng, ctr = _staged_problem(0x57A8 + RF, RF)
    ctr[:] = rng.integers(0, 60, size=ctr.shape)
    exp_out, exp_ln, exp_st, exp_ctr = oracle_from(oracle, cl, ctr)
    assert exp_st[0] == 0
    p = DeviceProblem(cl)
    s = kab.Solver(0)
    p.warm(s)
    d_ctr = torch.full((cl.N, models.SLOTS), 10**6, dtype=torch.int32, device="cuda")
    d_exp = torch.full((cl.N, models.SLOTS), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    stream, h = _stream(SIDE)
    sleep = late_inputs(stream, p.real + [(d_ctr, _dev(ctr.astype(np.int32)))])
    t0 = time.perf_counter()
    s.import_counters_device(d_ctr.data_ptr(), stream=h)
    s.stage_dense_device(*p.stage_args(), stream=h)
    s.order_device(p.d_len.data_ptr(), p.d_out.data_ptr(), stream=h, sync=False)
    s.export_counters_device(d_exp.data_ptr(), stream=h)
    t_call = time.perf_counter() - t0
    out, ln, got_ctr = early_read(stream, p.d_out, p.d_len, d_exp)
    util.enqueued_behind(sleep, t_call)
    assert util.fields(s.last_status()) == exp_st
    assert s.last_order_plan()[0] == (3 if RF == 3 else 4)
    check_rows(out, ln, (exp_out, exp_ln), ("staged-order", RF))
    assert np.array_equal(got_ctr, exp_ctr)


# ---- two Contexts in flight on one stream --------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("failing_first", [True, False], ids=["failing-first", "failing-second"])
def test_two_contexts_in_flight_on_one_stream(native_lib, oracle, failing_first):
    """Two asynchronous solves on two Contexts, enqueued one after the other on one stream behind the sleep. One fails
    (replication factor above its 2-broker table): each ka_last_status reports its own status, and the other's rows and
    counters are the oracle's."""
    cl = kab.synth.make_cluster(T=200, P=32, RF=3, N=120, R=10, seed=0x57C0, kind="mixed")
    bad_cl = kab.synth.make_cluster(T=50, P=8, RF=3, N=30, R=5, seed=0x57C1, kind="mixed")
    bad_table = (bad_cl.broker_id[:2], bad_cl.rack_index[:2])
    exp, bad_exp = expected(oracle, cl), expected(oracle, bad_cl, bad_table)
    assert exp[2][0] == 0 and bad_exp[2][0] == _native.KA_ERR_RF_GT_BROKERS
    good, bad = DeviceProblem(cl), DeviceProblem(bad_cl)
    s_good, s_bad = kab.Solver(0), kab.Solver(0)
    good.warm(s_good)
    bad.warm(s_bad, bad_table)
    stream, h = _stream(SIDE)
    sleep = late_inputs(stream, good.real + bad.real)
    calls = [(s_bad, bad), (s_good, good)] if failing_first else [(s_good, good), (s_bad, bad)]
    t0 = time.perf_counter()
    for s, p in calls:
        s.solve_dense_device(*p.solve_args(), stream=h, sync=False)
    t_call = time.perf_counter() - t0
    out, ln = early_read(stream, good.d_out, good.d_len)
    util.enqueued_behind(sleep, t_call)
    assert util.fields(s_bad.last_status()) == bad_exp[2]
    assert util.fields(s_good.last_status()) == exp[2]
    check_rows(out, ln, exp, "good")
    assert np.array_equal(s_good.counters(), exp[3])


# ---- destroy right after an asynchronous call ----------------------------------------------------------------------------

@pytest.mark.gpu
def test_destroy_waits_for_the_pending_call(native_lib, oracle):
    """An asynchronous pipelined solve behind the sleep, Solver.close() at once, then the outputs read on the caller's stream:
    they are the oracle's rows (ka_ctx_destroy collected the pending call before freeing its buffers)."""
    cl = kab.synth.make_cluster(T=4096, P=64, RF=3, N=300, R=12, seed=0x57D0, kind="mixed")
    exp = expected(oracle, cl)
    p = DeviceProblem(cl)
    s = kab.Solver(0)
    p.warm(s)
    stream, h = _stream(SIDE)
    sleep = late_inputs(stream, p.real)
    t0 = time.perf_counter()
    s.solve_dense_device(*p.solve_args(), stream=h, sync=False)
    t_call = time.perf_counter() - t0
    s.close()
    out, ln = early_read(stream, p.d_out, p.d_len)
    util.enqueued_behind(sleep, t_call)
    check_rows(out, ln, exp, "destroy")


# ---- host threads, one Context each -----------------------------------------------------------------------------------------

# Per thread: a dense capacity-1 table (kernel A and the slot chains sized by N: a few hundred brokers, the middle, and both
# sides of the rows <= 3 band edge 25 023 / 25 024 of test_chain_edges) and a ragged table below kernel A's level-plan limit
# (its level instantiation and the wave chains sized by N as well).
THREAD_TABLES = [(300, 200), (4000, 1500), (25023, 6000), (25024, 15000)]
THREAD_B = 2
THREAD_ROUNDS = 2


def _thread_work(oracle, i, N_dense, N_ragged):
    """Inputs and CPU-computed expectations of thread i."""
    import torch
    cl = kab.synth.make_cluster(T=64, P=64, RF=3, N=N_dense, R=10, seed=0x5770 + i, kind="mixed")
    rc = kab.synth.make_ragged_cluster(T=250, N=N_ragged, R=10, seed=0x5780 + i, max_partitions=64, remove_frac=0.05)
    S = 3
    r_len, _, r_out, r_st = oracle.run(oracle.OracleContext(), rc.topic_names, rc.part_off, rc.part_id, rc.rep_off, rc.cur,
                                       rc.broker_id, rc.rack_name, -1, S, raise_on_error=False)
    assert r_st.code == 0
    ids = rc.broker_id
    waves = {}
    for rule, plan in (("greedy", models.plan_waves), ("first_fit", fit_models.plan_waves)):
        wave, summ, st = plan(rc.rep_off, rc.cur, r_out, r_len, ids, THREAD_B)
        assert st == (0, 0, 0)
        waves[rule] = (wave, summ)
    usage, W = usage_models.broker_usage_np(rc.rep_off, rc.cur, r_out, r_len, waves["greedy"][0], rc.all_broker_id)
    p = DeviceProblem(cl)
    for dst, src in p.real:          # no late inputs here: the threads read the real ones
        dst.copy_(src)
    return dict(cl=cl, dense=expected(oracle, cl), p=p, rc=rc, S=S, ragged=(r_out, r_len), waves=waves,
                usage=(usage, W), stream=torch.cuda.Stream())


def _thread_run(s, w, barrier, results, i):
    """The thread's fixed sequence of calls; every result is checked against w's expectations."""
    import torch
    try:
        cl, rc, p, S = w["cl"], w["rc"], w["p"], w["S"]
        stream, h = w["stream"], w["stream"].cuda_stream
        barrier.wait()
        for rnd in range(THREAD_ROUNDS):
            s.reset()
            s.set_brokers(cl.broker_id, cl.rack_index)
            st = s.solve_dense_device(*p.solve_args(), stream=h)
            assert util.fields(st) == w["dense"][2], ("dense", rnd, util.fields(st))
            out, ln = early_read(stream, p.d_out, p.d_len)
            check_rows(out, ln, w["dense"], ("dense", i, rnd))
            assert np.array_equal(s.counters(), w["dense"][3]), ("dense counters", i, rnd)
            s.reset()
            s.set_brokers(rc.broker_id, rc.rack_index)
            out, ln, st = s.solve_ragged(rc.topic_hash, rc.part_off, rc.part_id, rc.rep_off, rc.cur, -1, S, check=False)
            assert st.code == 0, ("ragged", i, rnd, util.fields(st))
            assert np.array_equal(out, w["ragged"][0]) and np.array_equal(ln, w["ragged"][1]), ("ragged", i, rnd)
            for rule in ("greedy", "first_fit"):
                s.set_wave_rule(rule)
                wave, summ, st = s.plan_waves(rc.rep_off, rc.cur, out, ln, THREAD_B)
                assert st.code == 0, (rule, i, rnd, util.fields(st))
                e_wave, e_summ = w["waves"][rule]
                assert np.array_equal(wave, e_wave), (rule, i, rnd)
                assert [util.record_of(x, kab.assigner.WAVE_SUMMARY_DTYPE.names) for x in summ] == e_summ, (rule, i, rnd)
            usage, W, st = s.broker_usage(rc.rep_off, rc.cur, out, ln, w["waves"]["greedy"][0], rc.all_broker_id)
            assert st.code == 0, ("usage", i, rnd, util.fields(st))
            e_usage, e_W = w["usage"]
            assert W == e_W
            for f, v in e_usage.items():
                assert np.array_equal(usage[f], v), ("usage", f, i, rnd)
        torch.cuda.synchronize()
        results[i] = "ok"
    except BaseException as e:       # reported by the main thread
        results[i] = e


@pytest.mark.gpu
def test_contexts_in_four_host_threads(native_lib, oracle):
    """Four host threads, each with its own Solver, stream and broker tables of its own sizes, run the same fixed sequence at
    the same time: a dense device solve, a host-buffer ragged solve, plan_waves under both rules and broker_usage, twice.
    Kernel A, the slot chains and the wave chains get a different dynamic shared-memory size in every thread; every result
    equals the one computed on the CPU beforehand."""
    import torch
    works = [_thread_work(oracle, i, nd, nr) for i, (nd, nr) in enumerate(THREAD_TABLES)]
    solvers = [kab.Solver(0) for _ in works]
    torch.cuda.synchronize()
    barrier = threading.Barrier(len(works))
    results = [None] * len(works)
    threads = [threading.Thread(target=_thread_run, args=(s, w, barrier, results, i)) for i, (s, w) in enumerate(zip(solvers, works))]
    t0 = time.perf_counter()
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    print("four threads: %.2f s" % (time.perf_counter() - t0))
    assert not any(t.is_alive() for t in threads), "a thread did not finish"
    for i, r in enumerate(results):
        if r != "ok":
            raise AssertionError("thread %d (tables %s)" % (i, THREAD_TABLES[i])) from r
