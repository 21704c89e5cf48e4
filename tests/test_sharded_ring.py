"""The topic-sharded solve on one GPU: W Contexts as concurrent ranks, each on its own stream, counters handed on in stream
order, checked against one oracle run over all topics.

multi.ring_solve_phases drives the staged per-slot API the same way on one H100 and on eight; only the interconnect differs.
Here every rank is a host thread with its own Solver (one Context) and its own non-blocking torch stream, and FakeDist stands
in for torch.distributed with NCCL's stream semantics rather than gloo's:

- send enqueues, on the sender's stream, a copy into a mailbox and then an event; recv blocks the host only until that send
  has been enqueued, makes the receiver's stream wait for the event and copies out on the receiver's stream;
- a collective joins every rank's stream into one reducing stream (events), reduces there, and joins back into every rank's
  stream before each rank copies the result in on its own stream;
- FakeDist never waits for a stream, an event or the device: those calls fail an assert inside it (no_host_waits);
- every mailbox starts out holding a decoy (valid counter values, not the ones sent), and a sender can sleep on the device
  ahead of its copy, so that a read which runs ahead of its hand-off gives wrong rows instead of a fault;
- every host wait has a timeout, and a rank that raises wakes every waiting rank (RankFailed).

So rank g's slot-0 chain runs while rank g-1's slot-1 chain and emit still run, as they do on eight GPUs. The GPU cases run
in one child process (util.run_child), which writes every rank's rows, counters, aborts and statuses to a directory; the
oracle's results are computed meanwhile and compared case by case. A CPU test pins FakeDist to the values the gloo backend
gives in tests/test_multi_gloo.py, so that a GPU failure points at the library rather than at the harness.
"""
import collections
import contextlib
import functools
import json
import os
import threading
import time
import traceback
from unittest import mock

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import multi
from tests import models, util

MIN_HASH = -2**31        # String.hashCode == Integer.MIN_VALUE (KAS:190-192): fails unless 2^31 % N == 0
WAIT_TIMEOUT = 60.0      # seconds any rank waits on another before the run fails
CHILD_TIMEOUT = 900      # seconds for every GPU case together: about 35 s of the module's 55 s on an H100 (DESIGN.md §6)


# ---- FakeDist: a stream-ordered, in-process torch.distributed ---------------------------------------------------------------

class RankFailed(RuntimeError):
    """Raised in a rank that waits on the others after one of them raised or a wait timed out."""


_local = threading.local()


def _dist_op(fn):
    """A FakeDist operation: while it runs in a thread, no_host_waits forbids that thread to wait for the device."""
    @functools.wraps(fn)
    def op(self, *a, **k):
        _local.in_dist = True
        try:
            return fn(self, *a, **k)
        finally:
            _local.in_dist = False
    return op


def _forbidden(what, orig):
    def call(*a, **k):
        assert not getattr(_local, "in_dist", False), "FakeDist must never wait for the device (%s)" % what
        return orig(*a, **k)
    return call


@contextlib.contextmanager
def no_host_waits():
    """torch.cuda.synchronize, Stream.synchronize and Event.synchronize fail an assert when a FakeDist operation calls them."""
    import torch
    with contextlib.ExitStack() as stack:
        for owner, name, what in ((torch.cuda, "synchronize", "device"), (torch.cuda.Stream, "synchronize", "stream"),
                                  (torch.cuda.Event, "synchronize", "event")):
            stack.enter_context(mock.patch.object(owner, name, _forbidden(what, getattr(owner, name))))
        yield


class FakeWorld:
    """W ranks in one process. Tensors live on the GPU (cuda) or on the CPU; on the CPU every operation completes at once.

    box_numel / dtype / depth: every ring mailbox (g -> g + 1) holds `depth` messages of up to box_numel elements, each
    starting out as a decoy of valid counter values (1..59). sleep_cycles: every send sleeps that long on the sender's stream
    ahead of its copy (the sleeps' events are kept in `sleeps`). Every host wait gives up after `timeout` seconds."""

    def __init__(self, world, cuda, box_numel, dtype=None, depth=4, timeout=WAIT_TIMEOUT, sleep_cycles=0, seed=0):
        import torch
        self.world, self.cuda, self.timeout, self.sleep_cycles = world, cuda, timeout, sleep_cycles
        self.cond = threading.Condition()
        self.failed = None
        self.sent = {}                          # (src, dst, seq) -> event after the copy into the mailbox (None on the CPU)
        self.seq = collections.Counter()        # (src, dst, "send" / "recv") -> messages so far
        self.colls = []                         # collectives in call order
        self.n_coll = [0] * world
        self.logs = [[] for _ in range(world)]  # every rank's operations, in order
        self.sleeps = []
        rng = np.random.default_rng(seed)
        dev, dtype = ("cuda" if cuda else "cpu"), (dtype or torch.int32)
        self.boxes = {(g, g + 1): [torch.from_numpy(rng.integers(1, 60, box_numel)).to(device=dev, dtype=dtype) for _ in range(depth)]
                      for g in range(world - 1)}
        self.reduce_stream = torch.cuda.Stream() if cuda else None

    def rank(self, g):
        return FakeDist(self, g)

    def fail(self, why):
        with self.cond:
            if self.failed is None:
                self.failed = why
            self.cond.notify_all()

    def wait(self, ready, what):
        """Blocks the host until ready() (checked under the lock), another rank fails, or the timeout."""
        deadline = time.monotonic() + self.timeout
        with self.cond:
            while not ready():
                if self.failed is not None:
                    raise RankFailed("waiting for %s: %s" % (what, self.failed))
                left = deadline - time.monotonic()
                if left <= 0:
                    err = TimeoutError("waited %.1f s for %s" % (self.timeout, what))
                    self.failed = repr(err)
                    self.cond.notify_all()
                    raise err
                self.cond.wait(left)

    def event(self):
        """An event recorded on the current stream (None on the CPU)."""
        import torch
        if not self.cuda:
            return None
        e = torch.cuda.Event()
        e.record()
        return e

    def combine(self, c):
        """A collective's result, computed on the reducing stream once every rank has joined it."""
        import torch
        ts = [c["inputs"][g][0] for g in range(self.world)]
        if c["kind"] == "barrier":
            return True
        if c["kind"] == "broadcast":
            return ts[c["src"]].clone()
        x = torch.stack(ts)
        return {"min": lambda: x.amin(0), "max": lambda: x.amax(0), "sum": lambda: x.sum(0, dtype=x.dtype)}[c["op"]]()

    def collective(self, g, tensor, kind, op=None, src=None):
        import torch
        with self.cond:
            k = self.n_coll[g]
            self.n_coll[g] += 1
            if k == len(self.colls):
                self.colls.append(dict(kind=kind, op=op, src=src, inputs={}, result=None, done=None))
            c = self.colls[k]
            assert (c["kind"], c["op"], c["src"]) == (kind, op, src), ("ranks disagree on collective %d" % k, c["kind"], kind)
            c["inputs"][g] = (tensor, self.event())
            if len(c["inputs"]) == self.world:
                if self.cuda:
                    with torch.cuda.stream(self.reduce_stream):
                        for _, e in c["inputs"].values():
                            self.reduce_stream.wait_event(e)
                        result = self.combine(c)
                        c["done"] = self.event()
                else:
                    result = self.combine(c)
                c["result"] = result
                self.cond.notify_all()
        self.wait(lambda: c["result"] is not None, "collective %d (%s) on rank %d" % (k, kind, g))
        if self.cuda:
            torch.cuda.current_stream().wait_event(c["done"])
        if tensor is not None:
            tensor.copy_(c["result"], non_blocking=True)


class FakeDist:
    """Rank g's view of a FakeWorld: what multi.ring_solve_phases and bench.Workload call on torch.distributed. No
    batch_isend_irecv, so multi._p2p takes its plain send / recv branch."""

    class ReduceOp:
        MIN, SUM, MAX = "min", "sum", "max"

    def __init__(self, w, g):
        self.w, self.rank, self.world = w, g, w.world

    def new_group(self, *a, **k):
        return ("group", id(self.w))

    @_dist_op
    def send(self, tensor, dst, group=None):
        import torch
        w, key = self.w, (self.rank, dst)
        w.logs[self.rank].append("send")
        seq = w.seq[key + ("send",)]
        w.seq[key + ("send",)] += 1
        box = w.boxes[key][seq].view(-1)[:tensor.numel()]
        if w.cuda and w.sleep_cycles:
            w.sleeps.append(util.device_sleep(torch.cuda.current_stream(), w.sleep_cycles))
        box.copy_(tensor.view(-1), non_blocking=True)
        ev = w.event()
        with w.cond:
            w.sent[key + (seq,)] = ev
            w.cond.notify_all()

    @_dist_op
    def recv(self, tensor, src, group=None):
        import torch
        w, key = self.w, (src, self.rank)
        w.logs[self.rank].append("recv")
        seq = w.seq[key + ("recv",)]
        w.seq[key + ("recv",)] += 1
        w.wait(lambda: key + (seq,) in w.sent, "send %d -> %d #%d" % (src, self.rank, seq))
        if w.cuda:
            torch.cuda.current_stream().wait_event(w.sent[key + (seq,)])
        tensor.view(-1).copy_(w.boxes[key][seq].view(-1)[:tensor.numel()], non_blocking=True)

    @_dist_op
    def broadcast(self, tensor, src, group=None):
        self.w.logs[self.rank].append("broadcast")
        self.w.collective(self.rank, tensor, "broadcast", src=src)

    @_dist_op
    def all_reduce(self, tensor, op=ReduceOp.SUM, group=None):
        self.w.logs[self.rank].append("all_reduce:" + op)
        self.w.collective(self.rank, tensor, "all_reduce", op=op)

    @_dist_op
    def barrier(self, group=None):
        self.w.logs[self.rank].append("barrier")
        self.w.collective(self.rank, None, "barrier")


def run_ranks(w, fn, streams=None):
    """fn(dist) in one host thread per rank, with streams[g] the current stream of rank g on the GPU. Returns what each rank
    returned or raised. A rank that raises wakes every waiting rank; a thread still running after the world's timeout fails
    the run."""
    import torch
    results = [None] * w.world

    def body(g):
        try:
            if w.cuda:
                with torch.cuda.stream(streams[g]):
                    results[g] = fn(w.rank(g))
            else:
                results[g] = fn(w.rank(g))
        except BaseException as e:       # reported to the caller
            results[g] = e
            w.fail("rank %d raised %r" % (g, e))

    threads = [threading.Thread(target=body, args=(g,), daemon=True) for g in range(w.world)]
    with no_host_waits():
        for t in threads:
            t.start()
        deadline = time.monotonic() + w.timeout + 30
        for t in threads:
            t.join(max(0.0, deadline - time.monotonic()))
        stuck = [g for g, t in enumerate(threads) if t.is_alive()]
        if stuck:
            w.fail("ranks %s did not finish" % stuck)
            for t in threads:
                t.join(5)
            raise AssertionError("ranks %s did not finish within %.0f s" % (stuck, w.timeout + 30))
    return results


# ---- CPU: FakeDist gives gloo's values ----------------------------------------------------------------------------------------

def _phase_pipeline(dist):
    """The two serial chains and one sum of test_multi_gloo.py::test_phase_pipeline_world3_gloo, through FakeDist."""
    import torch
    g = dist.rank
    state = {"a": 0, "b": 0, "c": 10 * (g + 1), "log": []}
    bufs = [torch.zeros(1, dtype=torch.int64), torch.zeros(1, dtype=torch.int64)]

    def mk(name, step):
        def run():
            state[name] = state[name] * 3 + step + g      # order-dependent: only the rank-ordered chain gives the right value
            state["log"].append("run_" + name)

        def export(t):
            t[0] = state[name]

        def import_(t):
            state[name] = int(t[0])
        return run, export, import_

    pa, pb = mk("a", 1), mk("b", 5)
    csum = torch.zeros(1, dtype=torch.int64)
    multi.ring_solve_phases(g, dist.world, lambda: state["log"].append("stage"),
                            lambda: [(pa[0], pa[1], pa[2], bufs[0]), (pb[0], pb[1], pb[2], bufs[1])], dist,
                            finish=lambda: state["log"].append("finish"),
                            final_sums=[(lambda t: t.__setitem__(0, state["c"]), lambda t: state.__setitem__("c_total", int(t[0])), csum)],
                            group=dist.new_group())
    assert state["log"] == ["stage", "run_a", "run_b", "finish"], state["log"]
    return state["a"], state["b"], state.get("c_total", state["c"])   # one rank: no final sum, its own value is the total


@pytest.mark.parametrize("W", range(1, 9))
def test_fake_dist_gives_gloo_values(W):
    """Two chains extended in rank order, broadcast from the last rank, and one all-reduced sum: every rank ends with the
    values the gloo run of test_multi_gloo.py gives (there for W = 3), and the ring's operations come in the order of
    multi.ring_solve_phases."""
    import torch
    w = FakeWorld(W, False, 1, dtype=torch.int64, timeout=10)
    got = run_ranks(w, _phase_pipeline)
    a = b = 0
    for g in range(W):
        a, b = a * 3 + 1 + g, b * 3 + 5 + g
    assert got == [(a, b, 10 * W * (W + 1) // 2)] * W
    for g in range(W):
        ring = (["recv"] if g > 0 else []) + (["send"] if g < W - 1 else [])
        tail = ["broadcast", "broadcast", "all_reduce:sum"] if W > 1 else []
        assert w.logs[g] == ring * 2 + tail, (g, w.logs[g])


def test_fake_dist_abort_wakes_every_rank():
    """Rank 2 of 5 raises in its first chain: ranks 3 and 4, blocked in recv, and ranks 0 and 1, blocked in the broadcast,
    all raise RankFailed, and every thread ends well inside the timeout."""
    import torch

    def ring(dist):
        buf = torch.zeros(1, dtype=torch.int64)

        def run():
            if dist.rank == 2:
                raise ValueError("rank 2 fails")
        multi.ring_solve_phases(dist.rank, dist.world, lambda: None, [(run, lambda t: None, lambda t: None, buf)], dist)
        return "done"

    w = FakeWorld(5, False, 1, dtype=torch.int64, timeout=10)
    t0 = time.monotonic()
    got = run_ranks(w, ring)
    assert time.monotonic() - t0 < 5
    assert isinstance(got[2], ValueError)
    assert all(isinstance(got[g], RankFailed) for g in (0, 1, 3, 4)), got


def test_fake_dist_wait_times_out():
    """A recv whose send never comes, and a barrier that one rank never reaches: the first wait to time out raises
    TimeoutError and wakes the other rank."""
    import torch

    def lonely(dist):
        t = torch.zeros(1, dtype=torch.int64)
        if dist.rank == 1:
            dist.recv(t, src=0)
        else:
            dist.barrier()

    w = FakeWorld(2, False, 1, dtype=torch.int64, timeout=0.5)
    t0 = time.monotonic()
    got = run_ranks(w, lonely)
    assert time.monotonic() - t0 < 5
    assert sorted(type(x).__name__ for x in got) == ["RankFailed", "TimeoutError"], got


# ---- the cases ---------------------------------------------------------------------------------------------------------------

Block = collections.namedtuple("Block", "t0 topic_hash cur desired_rf S")
# bench: run bench.Workload.device_step (the rows only); config: the BASELINE config whose blocks these are
Case = collections.namedtuple("Case", "W table runs fresh sleep bench config", defaults=(None,))


def _cluster(T, P, RF, N, R, seed, t_offset=0):
    return kab.synth.make_cluster(T=T, P=P, RF=RF, N=N, R=R, seed=seed, kind="mixed", t_offset=t_offset)


def _blocks(cl, W, desired_rf=-1, ids=None):
    """cl's topics sharded over W ranks (multi.shard_range); ids: new ascending ids for cl's brokers 1000, 1001, ..."""
    cur = cl.cur if ids is None else ids[cl.cur - 1000]
    S = max(cl.RF, desired_rf, 1)
    return [Block(t0, cl.topic_hash[t0:t1].copy(), np.ascontiguousarray(cur[t0:t1]), desired_rf, S)
            for t0, t1 in (multi.shard_range(cl.T, W, g) for g in range(W))]


def _ring(W, T, shape, seed, desired_rf=-1, runs=1, ids=None, fresh=False, sleep=False):
    """`runs` consecutive runs of T topics each (run k: topics k T .. (k + 1) T - 1) over one broker table."""
    cls = [_cluster(T, seed=seed, t_offset=k * T, **shape) for k in range(runs)]
    cl = cls[0]
    table = (cl.broker_id if ids is None else ids, cl.rack_index)
    return Case(W, table, [_blocks(c, W, desired_rf, ids) for c in cls], fresh, sleep, None)


def _mixed_rf(W, RFs, T_per, P, N, R, seed):
    """Rank g's block has rows of RFs[g]: one run whose topics differ in replication factor from block to block."""
    blocks = []
    for g, RF in enumerate(RFs):
        cl = _cluster(T_per, P, RF, N, R, seed, t_offset=g * T_per)
        blocks.append(Block(g * T_per, cl.topic_hash.copy(), cl.cur, -1, RF))
    return Case(W, (cl.broker_id, cl.rack_index), [blocks], False, False, None)


def _failing(kind, where, W=4, T_per=6):
    """Topics that fail on the ranks `where`, over one table: "hash" one topic hashed to Integer.MIN_VALUE in the middle of
    the block (2^31 % 15 != 0); "rf" every topic of the block has 3 replicas over a table of 2 brokers; "racks" every topic of
    the block has 3 replicas over a table of 2 racks. The other ranks' topics solve."""
    T = W * T_per
    if kind == "hash":
        cl = _cluster(T, 8, 3, 15, 5, 0xFA11)
        table, blocks = (cl.broker_id, cl.rack_index), _blocks(cl, W)
        for g in where:
            blocks[g].topic_hash[T_per // 2] = MIN_HASH
        return Case(W, table, [blocks], False, False, None)
    N, R = (3, 3) if kind == "rf" else (12, 4)
    ok, bad = _cluster(T, 4, 2, N, R, 0xFA12), _cluster(T, 4, 3, N, R, 0xFA12)
    table = util.table(ok.broker_id[:2]) if kind == "rf" else util.table(ok.broker_id, 6)
    blocks = _blocks(ok, W)
    for g in where:
        t0 = blocks[g].t0
        blocks[g] = Block(t0, bad.topic_hash[t0:t0 + T_per].copy(), bad.cur[t0:t0 + T_per], -1, 3)
    return Case(W, table, [blocks], False, False, None)


_CONFIG_BLOCKS = {}


def config_blocks(key, W):
    """W consecutive blocks of BASELINE config `key`, as bench.Workload makes them (block g: topics g T .. (g + 1) T - 1)."""
    if (key, W) not in _CONFIG_BLOCKS:
        T = kab.synth.CONFIGS[key]["T"]
        cls = [kab.synth.make_config(key, "mixed", t_offset=g * T) for g in range(W)]
        _CONFIG_BLOCKS[key, W] = ((cls[0].broker_id, cls[0].rack_index),
                                  [Block(g * T, c.topic_hash, c.cur, -1, c.RF) for g, c in enumerate(cls)])
    return _CONFIG_BLOCKS[key, W]


def _config(key, W, bench=False):
    table, blocks = config_blocks(key, W)
    return Case(W, table, [blocks], False, False, bench, key)


CAP1 = dict(P=16, RF=3, N=120, R=6)          # capacity 1: P x RF <= N
LEVELS = dict(P=40, RF=3, N=50, R=5)         # capacity 3: level plans
LUT_N = 1000
LUT_IDS = {"shared": 1000 + np.arange(LUT_N, dtype=np.int32),                               # id range 1 000: shared LUT
           "global": 1 + 37 * np.arange(LUT_N, dtype=np.int32),                             # range 36 964: global LUT
           "bsearch": np.append(np.arange(1, LUT_N, dtype=np.int32), np.int32(1 << 27))}    # range 2^27: binary search
LUT_MASK = {"shared": 1, "global": 2, "bsearch": 4}                                         # ka_ctx_last_stage_plan field 6
FAIL_WHERE = {"first": [0], "middle": [2], "last": [3], "two": [1, 3]}
CONFIG_CASES = ("c4shard-", "bench-")                                                       # ids of the BASELINE config cases

CASES = {}
for _W in (2, 3, 5, 8):
    CASES["ring-w%d-cap1" % _W] = functools.partial(_ring, _W, 30 * _W + 1, CAP1, 0x5A01)
    CASES["ring-w%d-levels" % _W] = functools.partial(_ring, _W, 30 * _W + 2, LEVELS, 0x5A02)
CASES.update({
    "rf1": functools.partial(_ring, 3, 61, dict(P=16, RF=1, N=40, R=4), 0x5B01),
    "rf2": functools.partial(_ring, 3, 61, dict(P=16, RF=2, N=40, R=4), 0x5B02),
    "grow-2to3": functools.partial(_ring, 3, 61, dict(P=16, RF=2, N=40, R=4), 0x5B03, 3),
    "shrink-3to1": functools.partial(_ring, 3, 61, dict(P=16, RF=3, N=40, R=4), 0x5B04, 1),
    "shrink-3to2": functools.partial(_ring, 4, 61, dict(P=30, RF=3, N=40, R=4), 0x5B05, 2),
    "mixed-rf-per-rank": functools.partial(_mixed_rf, 3, [3, 1, 2], 20, 16, 40, 4, 0x5B06),
    "rows4": functools.partial(_ring, 3, 40, dict(P=12, RF=4, N=60, R=6), 0x5C01),
    "rows5-levels": functools.partial(_ring, 4, 41, dict(P=16, RF=5, N=30, R=10), 0x5C02),
    "rows8": functools.partial(_ring, 3, 40, dict(P=12, RF=8, N=96, R=8), 0x5C03),
    "empty-w5-t3": functools.partial(_ring, 5, 3, CAP1, 0x5D01),
    "empty-w8-t5-rows4": functools.partial(_ring, 8, 5, dict(P=12, RF=4, N=60, R=6), 0x5D02),
    "w4-t5": functools.partial(_ring, 4, 5, LEVELS, 0x5D03),
    "subblocks-w3-t3073": functools.partial(_ring, 3, 3073, dict(P=4, RF=3, N=60, R=6), 0x5E01),
    "subblocks-w2-t2047": functools.partial(_ring, 2, 2047, dict(P=4, RF=3, N=60, R=6), 0x5E02),
    "two-runs-w3-levels": functools.partial(_ring, 3, 90, LEVELS, 0x5F01, runs=2),
    "two-runs-w5-cap1": functools.partial(_ring, 5, 151, CAP1, 0x5F02, runs=2),
    "two-runs-w3-rows4": functools.partial(_ring, 3, 60, dict(P=12, RF=4, N=60, R=6), 0x5F03, runs=2),
    "sleep-w4": functools.partial(_ring, 4, 200, dict(P=32, RF=3, N=200, R=10), 0x5001, runs=1, fresh=True, sleep=True),
    "sleep-w3-rows5": functools.partial(_ring, 3, 60, dict(P=8, RF=5, N=80, R=10), 0x5002, runs=1, fresh=True, sleep=True),
    "c4shard-w8": functools.partial(_config, "c4shard", 8),
    "bench-c2-w8": functools.partial(_config, "c2", 8, True),
    "bench-c4shard-w8": functools.partial(_config, "c4shard", 8, True),
})
for _m, _ids in LUT_IDS.items():
    CASES["lut-" + _m] = functools.partial(_ring, 4, 120, dict(P=32, RF=3, N=LUT_N, R=10), 0x5E10, ids=_ids)
for _k in ("hash", "rf", "racks"):
    for _where, _g in FAIL_WHERE.items():
        CASES["fail-%s-%s" % (_k, _where)] = functools.partial(_failing, _k, _g)


def case(cid):
    c = CASES[cid]()
    if c.sleep:   # the same blocks twice on fresh Contexts: the first run reserves every Context's scratch at this shape
        c = c._replace(runs=c.runs * 2)
    return c


def test_cases_fail_only_where_intended(oracle):
    """Every fail-* case: the blocks of the ranks named fail alone (on a fresh Context), the others solve, and the whole run
    fails first inside the lowest of those ranks. Every other case solves (the BASELINE configs are checked by bench.py)."""
    for cid in CASES:
        if cid.startswith(CONFIG_CASES):
            continue
        if not cid.startswith("fail-"):
            assert expected_of(oracle, cid)["abort"] is None, cid
            continue
        c, where = case(cid), FAIL_WHERE[cid.split("-")[2]]
        for g, blk in enumerate(c.runs[0]):
            assert (block_status(oracle, c.table, blk) is not None) == (g in where), (cid, g)
        first = expected_of(oracle, cid)["abort"][0]
        blk = c.runs[0][where[0]]
        assert blk.t0 <= first < blk.t0 + len(blk.topic_hash), cid


# ---- the oracle --------------------------------------------------------------------------------------------------------------

def block_status(oracle, table, blk):
    """(code, run-wide topic, partition, a, b) of the block alone on a fresh Context, or None when it solves."""
    if len(blk.topic_hash) == 0:
        return None
    _, _, st = oracle.fast_run_dense(oracle.FastContext(), blk.topic_hash, blk.cur, *table, blk.desired_rf, blk.S)
    return (st.code, blk.t0 + st.topic_index, st.partition, st.a, st.b) if st.code else None


_CONFIG_EXPECTED = {}


def expected_of(oracle, cid):
    """One oracle run over all topics, block after block through one Context: every run's rows per rank and the final
    counters, or the abort (index, status) of the first failing topic and every rank's own status. The run over a BASELINE
    config's blocks is computed once and shared by the cases on them (bench's ring installs no final Context: rows only)."""
    c = case(cid)
    if c.config is None:
        return oracle_run(oracle, c)
    if (c.config, c.W) not in _CONFIG_EXPECTED:
        _CONFIG_EXPECTED[c.config, c.W] = oracle_run(oracle, c)
    exp = _CONFIG_EXPECTED[c.config, c.W]
    return dict(exp, counters=None) if c.bench else exp


def oracle_run(oracle, c):
    ids, racks = c.table
    fctx, ctr, runs = oracle.FastContext(), np.zeros((len(ids), models.SLOTS), dtype=np.int64), []
    for blocks in c.runs:
        if c.fresh:
            fctx, ctr[:] = oracle.FastContext(), 0
        rows = []
        for blk in blocks:
            if len(blk.topic_hash) == 0:
                rows.append((np.zeros((0, blk.S), dtype=np.int32), np.zeros(0, dtype=np.int32)))
                continue
            out, ln, st = oracle.fast_run_dense(fctx, blk.topic_hash, blk.cur, ids, racks, blk.desired_rf, blk.S)
            if st.code:
                return dict(abort=(blk.t0 + st.topic_index, (st.code, blk.t0 + st.topic_index, st.partition, st.a, st.b)),
                            status=[block_status(oracle, c.table, b) for b in blocks])
            rows.append((out, ln))
            ctr += models.histogram(ids, out, ln)
        runs.append(rows)
    return dict(abort=None, runs=runs, counters=ctr)


# ---- the rank step (GPU, in the child) ---------------------------------------------------------------------------------------

def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Rank:
    """One rank: its Context (a Solver on the run's broker table), its own stream, the buffers its counters travel in, and
    its topic block of the current run on the device."""

    def __init__(self, table):
        import torch
        self.s = kab.Solver(0)
        self.s.set_brokers(*table)
        self.stream = torch.cuda.Stream()
        N = len(table[0])
        self.col = [torch.zeros(N, dtype=torch.int32, device="cuda") for _ in range(3)]   # slot 0, slot 1, the slot-2 sum
        self.table_buf = torch.zeros(N * models.SLOTS, dtype=torch.int32, device="cuda")
        self.before2 = torch.zeros(N, dtype=torch.int32, device="cuda")
        self.slots = self.status = None

    def load(self, blk, seed):
        """The block of the next run. Every buffer the rank receives into holds a decoy until its hand-off lands: valid
        counter values, not the ones sent, so that a library import which reads it ahead of the copy gives wrong rows."""
        import torch
        rng = np.random.default_rng(seed)
        for t in self.col + [self.table_buf]:
            t.copy_(_dev(rng.integers(1, 60, t.numel()).astype(np.int32)))
        self.blk = blk
        T, P, _ = blk.cur.shape
        self.s.set_topic_base(blk.t0)
        self.d_hash, self.d_cur = _dev(blk.topic_hash), _dev(blk.cur)
        self.d_out = torch.full((T, P, blk.S), -7, dtype=torch.int32, device="cuda")
        self.d_len = torch.full((T, P), -7, dtype=torch.int32, device="cuda")

    def step(self, dist, status=True):
        """bench.Workload.device_step's ring, plus what it leaves out: the ranks agree on the lowest failing topic, the last
        rank broadcasts its counter columns, and counter[.][2] is summed over the ranks."""
        import torch
        s, sp, blk = self.s, self.stream.cuda_stream, self.blk
        T, P, RF = blk.cur.shape
        dl, do = self.d_len.data_ptr(), self.d_out.data_ptr()
        self.slots = self.status = None

        def stage():
            s.export_counter_slot_device(2, self.before2.data_ptr(), sp)    # counter[.][2] as the run starts
            s.stage_dense_device(T, self.d_hash.data_ptr(), P, RF, self.d_cur.data_ptr(), blk.desired_rf, blk.S, stream=sp)

        def phases():   # after stage(): rows <= 3 -> two slot chains handed on separately; else one fused chain
            self.slots = s.staged_slot_chains()
            if self.slots == 2:
                return [(lambda r=r: s.order_slot_device(r, sp), lambda t, r=r: s.export_counter_slot_device(r, t.data_ptr(), sp),
                         lambda t, r=r: s.import_counter_slot_device(r, t.data_ptr(), sp), self.col[r]) for r in (0, 1)]
            return [(lambda: s.order_device(dl, do, stream=sp, sync=False), lambda t: s.export_counters_device(t.data_ptr(), sp),
                     lambda t: s.import_counters_device(t.data_ptr(), sp), self.table_buf)]

        def finish():
            if self.slots == 2:
                s.emit_device(dl, do, stream=sp, sync=False)

        def first_failure():
            st = s.last_status()
            self.status = util.fields(st)
            return st.topic_index if st.code != 0 else None

        multi.ring_solve_phases(dist.rank, dist.world, stage, phases, dist, finish=finish, final_broadcast=True,
                                final_sums=self.slot2_sum(), status=first_failure if status else None,
                                tensor_factory=lambda v: torch.tensor(v, dtype=torch.int64, device="cuda"))

    def slot2_sum(self):
        """Rows <= 3: no chain reads counter[.][2], so every rank bumps it for its own block only and the ranks add up what
        their blocks added. A generator, so that whether the block had slot chains is only asked at the end of the run."""
        if self.slots == 2:
            yield self.export_delta, self.add_total, self.col[2]

    def export_delta(self, t):
        """What this rank's block added to counter[.][2]: the column now minus the column at the start of the run."""
        self.s.export_counter_slot_device(2, t.data_ptr(), self.stream.cuda_stream)
        t.sub_(self.before2)

    def add_total(self, t):
        t.add_(self.before2)
        self.s.import_counter_slot_device(2, t.data_ptr(), self.stream.cuda_stream)


def run_ring(c, info, arrays):
    import torch
    ranks = [Rank(c.table) for _ in range(c.W)]
    N = len(c.table[0])
    for k, blocks in enumerate(c.runs):
        sleep = c.sleep and k == len(c.runs) - 1
        if c.fresh:
            for r in ranks:
                r.s.reset()
        for g, (r, blk) in enumerate(zip(ranks, blocks)):
            r.load(blk, (k, g))
        w = FakeWorld(c.W, True, N * models.SLOTS, seed=k + 1, sleep_cycles=util.SLEEP_CYCLES if sleep else 0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = run_ranks(w, lambda dist: ranks[dist.rank].step(dist, status=not sleep), [r.stream for r in ranks])
        t_enqueue = time.perf_counter() - t0
        torch.cuda.synchronize()
        run = dict(aborted=[], status=[r.status for r in ranks], logs=w.logs, enqueue_ms=1e3 * t_enqueue, sleep=sleep,
                   stage_plan=[r.s.last_stage_plan() for r in ranks], order_plan=[r.s.last_order_plan() for r in ranks])
        if sleep:
            run["sleep_ms"] = [a.elapsed_time(b) for a, b in w.sleeps]
        for g, (r, x) in enumerate(zip(ranks, got)):
            if isinstance(x, BaseException) and not isinstance(x, multi.RunAborted):
                raise AssertionError("rank %d of run %d raised" % (g, k)) from x
            run["aborted"].append(x.topic_index if isinstance(x, multi.RunAborted) else None)
            arrays["out_%d_%d" % (k, g)] = r.d_out.cpu().numpy().reshape(-1, r.blk.S)
            arrays["len_%d_%d" % (k, g)] = r.d_len.cpu().numpy().reshape(-1)
        info["runs"].append(run)
        if any(a is not None for a in run["aborted"]):
            break
    arrays["counters"] = np.stack([r.s.counters() for r in ranks])


def run_bench(c, info, arrays):
    """bench.Workload(...).device_step() of every rank, through FakeDist."""
    import torch
    import bench
    streams = [torch.cuda.Stream() for _ in range(c.W)]
    w = FakeWorld(c.W, True, len(c.table[0]) * models.SLOTS)
    wls = [bench.Workload(c.config, "mixed", g, c.W, 0, torch, kab, w.rank(g), streams[g]) for g in range(c.W)]
    for wl in wls:
        wl.d_out.fill_(-7)
        wl.d_len.fill_(-7)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    got = run_ranks(w, lambda dist: wls[dist.rank].device_step(), streams)
    t_enqueue = time.perf_counter() - t0
    torch.cuda.synchronize()
    for g, x in enumerate(got):
        if isinstance(x, BaseException):
            raise AssertionError("rank %d raised" % g) from x
    info["runs"].append(dict(aborted=[None] * c.W, status=[util.fields(wl.solver.last_status()) for wl in wls], logs=w.logs,
                             enqueue_ms=1e3 * t_enqueue))
    for g, wl in enumerate(wls):
        arrays["out_0_%d" % g] = wl.d_out.cpu().numpy().reshape(-1, wl.S)
        arrays["len_0_%d" % g] = wl.d_len.cpu().numpy().reshape(-1)


def run_cases(d):
    """The child: every GPU case in turn; rows, counters and a report (run details, errors, seconds) written to d."""
    import torch
    report = {}
    t_all = time.perf_counter()
    for cid in CASES:
        t0 = time.perf_counter()
        info, arrays = dict(runs=[], error=None), {}
        try:
            c = case(cid)
            t1 = time.perf_counter()
            (run_bench if c.bench else run_ring)(c, info, arrays)
            info["gpu_seconds"] = time.perf_counter() - t1
            np.savez(os.path.join(d, cid + ".npz"), **arrays)
        except Exception:
            info["error"] = traceback.format_exc()
            torch.cuda.synchronize()
        info["seconds"] = time.perf_counter() - t0
        report[cid] = info
        print("%-24s %6.2f s%s" % (cid, info["seconds"], "  FAILED" if info["error"] else ""), flush=True)
    print("all cases %.1f s" % (time.perf_counter() - t_all), flush=True)
    with open(os.path.join(d, "report.json"), "w") as f:
        json.dump(report, f)


_CHILD = r"""
import sys
from tests import test_sharded_ring
test_sharded_ring.run_cases(sys.argv[1])
"""


# ---- GPU: the checks ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def sharded(tmp_path_factory, native_lib, oracle):
    """(directory, oracle results, child report) of every case: the child runs them on the GPU while the oracle runs here."""
    d = tmp_path_factory.mktemp("sharded")
    exp, out, secs = util.run_child(_CHILD, d, CHILD_TIMEOUT, lambda: {cid: expected_of(oracle, cid) for cid in CASES},
                                    "the sharded runs")
    print("child and oracle %.1f s\n%s" % (secs, out))
    with open(d / "report.json") as f:
        return d, exp, json.load(f)


def check_rows(got_out, got_len, out, ln, what):
    bad = np.nonzero(np.any(got_out != out, axis=1) | (got_len != ln))[0]
    unwritten = int(np.sum(np.any(got_out[bad] == -7, axis=1) | (got_len[bad] == -7)))
    assert len(bad) == 0, (what, "%d of %d rows differ from the oracle, first %s" % (len(bad), len(ln), bad[:5].tolist()),
                           "rows still holding -7: %d" % unwritten)


def check_case(sharded, cid):
    """The rows and list lengths of every rank equal the oracle's run over all topics, every rank's final Context equals
    the oracle's; or, when a topic fails, every rank aborts with the run-wide index of the oracle's first failing topic and
    none installs counters from the dead run. Returns (report of the case, its arrays)."""
    d, exp_all, report = sharded
    info, exp = report[cid], exp_all[cid]
    assert info["error"] is None, info["error"]
    got = np.load(d / (cid + ".npz"))
    W = len(info["runs"][0]["aborted"])
    if exp["abort"] is not None:
        index, st = exp["abort"]
        run = info["runs"][0]
        assert run["aborted"] == [index] * W, (run["aborted"], index)
        for g in range(W):
            e = exp["status"][g]
            assert (tuple(run["status"][g]) == e) if e is not None else run["status"][g][0] == 0, (g, run["status"][g], e)
            assert run["logs"][g][-1] == "all_reduce:min" and "broadcast" not in run["logs"][g], (g, run["logs"][g])
        return info, got
    for k, rows in enumerate(exp["runs"]):
        assert info["runs"][k]["aborted"] == [None] * W
        for g, (out, ln) in enumerate(rows):
            check_rows(got["out_%d_%d" % (k, g)], got["len_%d_%d" % (k, g)], out, ln, (cid, "run", k, "rank", g))
    if exp["counters"] is not None:
        for g in range(W):
            bad = np.nonzero(np.any(got["counters"][g] != exp["counters"], axis=1))[0]
            assert len(bad) == 0, (cid, "rank", g, "counters of %d brokers differ, first %s" % (len(bad), bad[:5].tolist()))
    return info, got


def _ids(prefix):
    return [cid for cid in CASES if cid.startswith(prefix)]


@pytest.mark.gpu
@pytest.mark.parametrize("cid", _ids("ring-"))
def test_per_slot_ring(sharded, cid):
    """W = 2, 3, 5, 8 ranks, rows of 3, capacity 1 and level plans: slot-0 of rank g runs while slot-1 and the emit of rank g - 1
    still run."""
    info, _ = check_case(sharded, cid)
    assert all((p[0], p[1]) == (3, "levels" in cid) for p in info["runs"][0]["order_plan"])


@pytest.mark.gpu
@pytest.mark.parametrize("cid", ["rf1", "rf2", "grow-2to3", "shrink-3to1", "shrink-3to2", "mixed-rf-per-rank"])
def test_short_rows(sharded, cid):
    """Rows of 1 and 2 (slot chains padded with dummies), from current lists of that length and from a desired replication
    factor that grows or shrinks them, and blocks whose rows differ in length from rank to rank."""
    check_case(sharded, cid)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", ["rows4", "rows5-levels", "rows8"])
def test_fused_ring(sharded, cid):
    """Rows of 4, 5 and 8: one fused leader-order chain per rank, the whole counter table handed on and broadcast."""
    info, _ = check_case(sharded, cid)
    assert all((p[0], p[1]) == ((4 if cid == "rows4" else 8), "levels" in cid) for p in info["runs"][0]["order_plan"])


@pytest.mark.gpu
@pytest.mark.parametrize("cid", ["empty-w5-t3", "empty-w8-t5-rows4", "w4-t5"])
def test_empty_ranks(sharded, cid):
    """Fewer topics than ranks: the ranks without topics emit nothing and pass both columns (or the table) on unchanged,
    the last of them to every rank in the final broadcast; and W + 1 topics."""
    check_case(sharded, cid)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", _ids("subblocks-"))
def test_chain_subblocks(sharded, cid):
    """Blocks of 1 023, 1 024 and 1 025 topics: each slot chain of a staged block is cut into min(8, T / 128) sub-blocks."""
    info, _ = check_case(sharded, cid)
    c = case(cid)
    for g, blk in enumerate(c.runs[0]):
        assert info["runs"][0]["order_plan"][g][6] == 2 * min(8, len(blk.topic_hash) // 128), g


@pytest.mark.gpu
@pytest.mark.parametrize("cid", _ids("lut-"))
def test_lookup_modes(sharded, cid):
    """One broker table on every rank, each its own Context, in each broker-id lookup mode."""
    info, _ = check_case(sharded, cid)
    assert all(p[6] == LUT_MASK[cid[4:]] for p in info["runs"][0]["stage_plan"])


@pytest.mark.gpu
@pytest.mark.parametrize("cid", _ids("two-runs-"))
def test_two_runs(sharded, cid):
    """A second sharded run through the same Contexts starts from the first run's final Context on every rank: its rows and
    the final counters equal one oracle Context through both runs (counter[.][2] summed as deltas, not totals)."""
    info, _ = check_case(sharded, cid)
    assert len(info["runs"]) == 2


@pytest.mark.gpu
@pytest.mark.parametrize("cid", _ids("fail-"))
def test_failing_topic(sharded, cid):
    """A topic that fails (hash Integer.MIN_VALUE, RF above the brokers, RF above the racks) on the first, a middle or the last
    rank, or on two ranks: every rank raises RunAborted with the run-wide index of the oracle's first failing topic, every
    failing rank reports its own first failing topic with the run-wide index, and no rank takes part in a final broadcast."""
    check_case(sharded, cid)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", _ids("sleep-"))
def test_ring_behind_sender_sleeps(sharded, cid):
    """Every send sleeps on the sender's stream ahead of its copy, and every mailbox and every receive buffer holds a decoy
    until its copy lands (the warm-up run before this one solved the same blocks). The whole ring is enqueued well inside one
    sleep, so a FakeDist copy or a library import that reads a hand-off ahead of its copy reads a decoy."""
    info, _ = check_case(sharded, cid)
    run = info["runs"][-1]
    assert run["sleep"], [{k: v for k, v in r.items() if k != "logs"} for r in info["runs"]]
    assert len(run["sleep_ms"]) == (case(cid).W - 1) * (2 if "rows" not in cid else 1)
    print("shortest sender sleep %.1f ms, host enqueue of the whole ring %.3f ms" % (min(run["sleep_ms"]), run["enqueue_ms"]))
    assert run["enqueue_ms"] < min(run["sleep_ms"]) / 2, "the ring's enqueue outlasted half a sleep: an early read could go unseen"


@pytest.mark.gpu
def test_c4shard_w8(sharded):
    """The shape bench.py --gpus 8 runs: 8 blocks of 12 500 topics x 256 partitions, RF 3, 5 000 brokers (25.6 M rows)."""
    info, _ = check_case(sharded, "c4shard-w8")
    print("c4shard, 8 ranks: %.2f s on the GPU (all eight Contexts set up, one run, rows copied back)" % info["gpu_seconds"])
    assert all(p[6] == 2 * 8 for p in info["runs"][0]["order_plan"])


@pytest.mark.gpu
@pytest.mark.parametrize("cid", _ids("bench-"))
def test_bench_device_step(sharded, cid):
    """bench.Workload(...).device_step() of 8 ranks through FakeDist: the code a multi-GPU bench runs, row for row."""
    info, _ = check_case(sharded, cid)
    assert all(st[0] == 0 for st in info["runs"][0]["status"])


@pytest.mark.gpu
def test_emit_takes_null_rows_only_without_rows(native_lib, oracle):
    """ka_emit_device takes a NULL row pointer only when the staged block has no rows. A block without topics ends its
    staged solve with NULL rows and leaves the Context's counters alone; a block with rows refuses NULL rows with
    KA_ERR_BAD_ARG, stays staged, and then emits the oracle's rows into real ones."""
    import torch
    from kafka_assigner_b200 import _native
    cl = _cluster(40, 16, 3, 60, 6, 0x5E30)
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    none = torch.zeros(0, dtype=torch.int32, device="cuda")
    assert none.data_ptr() == 0
    s.stage_dense_device(0, none.data_ptr(), cl.P, cl.RF, none.data_ptr(), -1, cl.RF)
    assert s.staged_slot_chains() == 2
    for r in (0, 1):
        s.order_slot_device(r)
    assert s.emit_device(0, 0).code == 0
    assert not s.counters().any()

    d_hash, d_cur = _dev(cl.topic_hash), _dev(cl.cur)
    d_out = torch.full((cl.T, cl.P, cl.RF), -7, dtype=torch.int32, device="cuda")
    d_len = torch.full((cl.T, cl.P), -7, dtype=torch.int32, device="cuda")
    s.stage_dense_device(cl.T, d_hash.data_ptr(), cl.P, cl.RF, d_cur.data_ptr(), -1, cl.RF)
    for r in (0, 1):
        s.order_slot_device(r)
    assert s.emit_device(d_len.data_ptr(), 0).code == _native.KA_ERR_BAD_ARG
    assert s.staged_slot_chains() == 2
    assert s.emit_device(d_len.data_ptr(), d_out.data_ptr()).code == 0
    out, ln, st = oracle.fast_run_dense(oracle.FastContext(), cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index)
    assert st.code == 0
    check_rows(d_out.cpu().numpy().reshape(-1, cl.RF), d_len.cpu().numpy().reshape(-1), out, ln, "emit")
    assert np.array_equal(s.counters(), models.histogram(cl.broker_id, out, ln))
