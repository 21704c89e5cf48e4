"""One Context over its whole life: broker tables that change, brokers that leave and return, and host calls made while an
asynchronous call of the same Context is still queued on the caller's stream.

A Context's leader-preference counters are keyed by broker id and live as long as the assigner (KTA:19-23, KAS:289-301):
include/kassign.h promises that the counters of a broker that leaves the table come back when its id returns. Every test here
drives ONE library Context and ONE oracle Context through the same sequence of calls, and checks rows, statuses and every
counter of the current table after each step. Counters of ids outside the table are checked by bringing the ids back: a
"roll call" switches to a table of every id the run has seen, compares all their counters, and switches back.

The last part holds an asynchronous call behind a device sleep on a torch stream and makes one host call at once; the host
call must act as if the asynchronous call had finished (include/kassign.h: a host call sees every earlier call of the ctx).
"""
import os
from unittest import mock

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from oracle import py_oracle as po
from tests import models, util

SLOTS = models.SLOTS
INT_MAX = 0x7FFFFFFF


# ---- random inputs -------------------------------------------------------------------------------------------------------

def random_table(rng, pool, n=None):
    """A broker table drawn from `pool`: (ascending ids, rack names), a fifth of the brokers without a rack."""
    n = int(rng.integers(1, len(pool) + 1)) if n is None else n
    ids = np.sort(rng.choice(pool, n, replace=False)).astype(np.int32)
    R = int(rng.integers(1, 6))
    return ids, [None if rng.random() < 0.2 else "r%d" % (int(b) % R) for b in ids]


class Dense:
    """T topics of P partitions, every current list RF long over ids of `pool` (ids outside the table included)."""

    def __init__(self, rng, pool, tag, T=None, max_rf=3, rf=None, desired_rf=None):
        self.T = int(rng.integers(1, 5)) if T is None else T
        self.P = int(rng.integers(1, 13))
        self.RF = int(rng.integers(1, max_rf + 1)) if rf is None else rf
        self.cur = np.array([[rng.choice(pool, self.RF, replace=False) for _ in range(self.P)] for _ in range(self.T)],
                            dtype=np.int32).reshape(self.T, self.P, self.RF)
        if desired_rf is None:
            desired_rf = int(rng.integers(1, max_rf + 1)) if rng.random() < 0.3 else -1
        self.desired_rf = desired_rf
        self.names = ["%s-%d" % (tag, t) for t in range(self.T)]
        self.hash = np.array([kab.java_string_hash(n) for n in self.names], dtype=np.int32)
        self.S = max(self.RF, desired_rf, 1)
        self.part_off = np.arange(self.T + 1, dtype=np.int64) * self.P
        self.part_id = np.tile(np.arange(self.P, dtype=np.int32), self.T)
        self.rep_off = np.arange(self.T * self.P + 1, dtype=np.int64) * self.RF
        self.flat = np.ascontiguousarray(self.cur.reshape(-1))

    def ragged(self):
        return self.hash, self.part_off, self.part_id, self.rep_off, self.flat


# ---- CPU: the two oracles agree on sequences -----------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_oracles_agree_on_call_sequences(oracle, seed):
    """py_oracle.KafkaTopicAssigner and the C++ oracle through the same generate_assignment calls, a different broker set and
    rack map on each: ids that leave and return, disjoint sets, an empty set (the reference's exception), desired RF changing.
    After every call the rows and then every counter of every id seen so far; after an exception both start afresh."""
    rng = np.random.default_rng(0xC7A0 + seed)
    pool = np.arange(1, 31, dtype=np.int32)
    halves = (pool[:15], pool[15:])
    py, octx = po.KafkaTopicAssigner(), oracle.OracleContext()
    seen, errors, kinds = set(), 0, set()
    for step in range(60):
        pick = rng.random()
        if pick < 0.08:
            ids, racks = np.zeros(0, dtype=np.int32), []
            kinds.add("empty")
        elif pick < 0.35:
            ids, racks = random_table(rng, halves[step % 2])      # consecutive calls on disjoint sets
            kinds.add("disjoint")
        else:
            ids, racks = random_table(rng, pool)
        seen.update(int(b) for b in ids)
        prob = Dense(rng, pool, "seq%d-%d" % (seed, step), T=1, max_rf=4)
        cur = {p: [int(b) for b in prob.cur[0, p]] for p in range(prob.P)}
        rack_map = {int(b): r for b, r in zip(ids, racks) if r is not None}
        ln, _, out, st = oracle.run(octx, prob.names, prob.part_off, prob.part_id, prob.rep_off, prob.flat, ids, racks,
                                    prob.desired_rf, prob.S, raise_on_error=False)
        try:
            fin = py.generate_assignment(prob.names[0], cur, set(int(b) for b in ids), rack_map, prob.desired_rf)
        except po.JavaError as e:
            assert (st.code, st.partition, st.a) == (e.kind, e.partition, e.a), (step, e.message, st.message)
            errors += 1
            py = po.KafkaTopicAssigner()
            octx.reset()
            continue
        assert st.code == 0, (step, st.message)
        assert {p: [int(b) for b in out[p, :ln[p]]] for p in range(prob.P)} == fin, step
        for b in sorted(seen):
            for r in range(SLOTS):
                assert octx.counter(b, r) == py.context.counter.get(b, {}).get(r, 0), (step, b, r)
    assert errors > 0 and kinds == {"empty", "disjoint"}


# ---- the mirror: one library Context and one oracle Context ---------------------------------------------------------------

ENTRIES = ("solve", "solve_json", "dense", "dense_json", "device_sync", "device_async", "staged_order", "staged_slots")


class Mirror:
    """One Solver and one oracle Context, driven through the same calls; every method checks what it can see."""

    def __init__(self, oracle):
        self.ol, self.s, self.octx = oracle, kab.Solver(0), oracle.OracleContext()
        self.ids, self.racks = np.zeros(0, dtype=np.int32), []
        self.seen = set()
        self.last = None   # (problem, rows, lengths) of the last solve that passed
        self.errors = 0    # solves that ended in a reference exception

    def oracle_counters(self, ids):
        return np.array([[self.octx.counter(int(b), r) for r in range(SLOTS)] for b in ids], dtype=np.int32).reshape(-1, SLOTS)

    def check_counters(self, what=""):
        got = self.s.counters()
        exp = self.oracle_counters(self.ids)
        bad = np.nonzero(np.any(got != exp, axis=1))[0]
        assert len(bad) == 0, (what, "counters of %d ids differ, first" % len(bad),
                               [(int(self.ids[i]), got[i].tolist(), exp[i].tolist()) for i in bad[:3]])

    def set_table(self, ids, racks):
        ids = np.asarray(ids, dtype=np.int32)
        self.s.set_brokers(ids, kab.synth.rack_indices(ids, racks))
        self.ids, self.racks = ids, list(racks)
        self.seen.update(int(b) for b in ids)
        self.check_counters("table of %d" % len(ids))

    def roll_call(self):
        """Every id seen so far in one table (their counters, parked ones restored, against the oracle's), then back."""
        ids, racks = self.ids, self.racks
        every = np.array(sorted(self.seen), dtype=np.int32)
        self.set_table(every, [None] * len(every))
        self.set_table(ids, racks)

    def set_counters(self, ctr):
        self.s.set_counters(ctr)
        for i, b in enumerate(self.ids):
            for r in range(SLOTS):
                self.octx.set_counter(int(b), r, int(ctr[i, r]))
        self.check_counters("set_counters")

    def reset(self):
        self.s.reset()
        self.octx.reset()
        self.check_counters("reset")

    def device_round_trip(self, rng):
        """Export every counter to the device, check them, import them with some changed, and one column the same way."""
        import torch
        s, N = self.s, len(self.ids)
        buf = torch.full((max(N, 1), SLOTS), -7, dtype=torch.int32, device="cuda")
        s.export_counters_device(buf.data_ptr())
        assert np.array_equal(buf.cpu().numpy()[:N], self.oracle_counters(self.ids))
        new = buf.cpu().numpy()[:N] + rng.integers(0, 3, size=(N, SLOTS)).astype(np.int32)
        buf[:N] = torch.from_numpy(new).cuda()
        s.import_counters_device(buf.data_ptr())
        slot = int(rng.integers(0, SLOTS))
        col = torch.from_numpy(np.ascontiguousarray(new[:, slot] * 2 + 1) if N else np.zeros(1, dtype=np.int32)).cuda()
        s.import_counter_slot_device(slot, col.data_ptr())
        new[:, slot] = new[:, slot] * 2 + 1
        back = torch.full((max(N, 1),), -7, dtype=torch.int32, device="cuda")
        s.export_counter_slot_device(slot, back.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(back.cpu().numpy()[:N], new[:, slot])
        for i, b in enumerate(self.ids):
            for r in range(SLOTS):
                self.octx.set_counter(int(b), r, int(new[i, r]))
        self.check_counters("device round trip")

    def expected(self, prob):
        """The oracle's (rows [Q, S], lengths [Q], status) for prob, through the oracle Context."""
        ln, _, out, st = self.ol.run(self.octx, prob.names, prob.part_off, prob.part_id, prob.rep_off, prob.flat, self.ids,
                                     self.racks, prob.desired_rf, prob.S, raise_on_error=False)
        return out, ln, st

    def solve(self, prob, entry):
        """prob through the entry point `entry` and through the oracle: the same status; on success the same rows (or text)
        and counters. A reference exception leaves the counters undefined (include/kassign.h): both sides start afresh."""
        s = self.s
        got_out, got_ln, text, st = None, None, None, None
        if entry == "solve":
            got_out, got_ln, st = s.solve_ragged(*prob.ragged(), prob.desired_rf, prob.S, check=False)
        elif entry == "solve_json":
            text, st = s.solve_ragged_json(prob.names, *prob.ragged(), prob.desired_rf, check=False)
        elif entry == "dense":
            got_out, got_ln, st = s.solve_dense(prob.hash, prob.cur, prob.desired_rf, prob.S, check=False)
        elif entry == "dense_json":
            text, st = s.solve_dense_json(prob.names, prob.hash, prob.cur, prob.desired_rf, check=False)
        else:
            got_out, got_ln, st = self._device(prob, entry)
        out, ln, est = self.expected(prob)
        code = st if isinstance(st, int) else st.code
        if est.code != 0 or code != 0:
            assert code == est.code, (entry, code, est.code, est.message)
            if not isinstance(st, int):
                assert (st.topic_index, st.partition) == (est.topic_index, est.partition), (entry, est.message)
            s.reset()
            self.octx.reset()
            self.errors += 1
            return
        if text is not None:
            assert bytes(text).decode() == models.solve_document(prob.names, prob.part_off, prob.part_id, out, ln), entry
        else:
            got_out = got_out.reshape(len(ln), -1)
            assert np.array_equal(got_out, out) and np.array_equal(got_ln.reshape(-1), ln), entry
        self.last = (prob, out, ln)
        self.check_counters(entry)

    def _device(self, prob, entry):
        import torch
        s = self.s
        d_hash, d_cur = torch.from_numpy(prob.hash).cuda(), torch.from_numpy(prob.cur).cuda()
        d_out = torch.full((prob.T, prob.P, prob.S), -7, dtype=torch.int32, device="cuda")
        d_len = torch.full((prob.T, prob.P), -7, dtype=torch.int32, device="cuda")
        args = (prob.T, d_hash.data_ptr(), prob.P, prob.RF, d_cur.data_ptr(), prob.desired_rf, prob.S)
        if entry == "device_sync":
            st = s.solve_dense_device(*args, d_len.data_ptr(), d_out.data_ptr())
        elif entry == "device_async":
            s.solve_dense_device(*args, d_len.data_ptr(), d_out.data_ptr(), sync=False)
            st = s.last_status()
        else:
            try:
                s.stage_dense_device(*args)
            except kab.KassignError as e:
                return None, None, e.code
            if entry == "staged_slots" and s.staged_slot_chains() == 2:
                s.order_slot_device(0)
                s.order_slot_device(1)
                s.emit_device(d_len.data_ptr(), d_out.data_ptr(), sync=False)
            else:
                s.order_device(d_len.data_ptr(), d_out.data_ptr(), sync=False)
            st = s.last_status()
        return d_out.cpu().numpy(), d_len.cpu().numpy(), st

    def batched(self, rng, pool):
        """The batched calls, which include/kassign.h says leave the Context, its table and its parked counters alone; their
        own results are other modules' business. Then the current table's counters, unchanged."""
        s = self.s
        prob = Dense(rng, pool, "batch", max_rf=3)
        other = random_table(rng, pool)
        tables = [(self.ids, kab.synth.rack_indices(self.ids, self.racks)), (other[0], kab.synth.rack_indices(*other))]
        s.solve_ragged_candidates(tables, *prob.ragged(), prob.desired_rf)
        s.score_ragged_candidates(tables, *prob.ragged(), prob.desired_rf)
        fleet = [t + prob.ragged() + (prob.desired_rf,) for t in tables]
        s.solve_clusters(fleet)
        s.score_clusters(fleet)
        if self.last is not None:
            p, out, ln = self.last
            wave, _, st = s.plan_waves(p.rep_off, p.flat, out, ln, 2)
            s.plan_waves_json(p.names, p.part_off, p.part_id, p.rep_off, p.flat, out, ln, 2)
            if st.code == 0:
                use = np.unique(np.concatenate([p.flat, out[out >= 0]])).astype(np.int32)
                s.broker_usage(p.rep_off, p.flat, out, ln, wave, use)
        self.check_counters("batched calls")


def ranks(n, rng, lo=0, hi=40):
    return rng.integers(lo, hi, size=(n, SLOTS)).astype(np.int32)


# ---- parked counters, case by case --------------------------------------------------------------------------------------

POOL = np.arange(1, 41, dtype=np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["solve", "dense", "device_sync", "staged_slots"])
def test_leave_and_return(native_lib, oracle, entry):
    """Table A, then B (some of A's ids gone, new ones added), then C (some of A's ids back): rows and counters after each."""
    rng = np.random.default_rng(0x1EAF)
    m = Mirror(oracle)
    a = np.arange(1, 25)
    b = np.concatenate([a[8:], np.arange(25, 33)])
    c = np.concatenate([a[:12], np.arange(29, 37)])
    for k, ids in enumerate((a, b, c, a)):
        m.set_table(ids, ["r%d" % (i % 4) for i in ids])
        for j in range(2):
            m.solve(Dense(rng, POOL, "lr%d-%d" % (k, j), rf=3), entry)
    m.roll_call()


# KA_ORDER_GLOBAL_CTR=1 keeps the chains' counters in global memory rather than shared memory
@pytest.mark.gpu
@pytest.mark.parametrize("env", [{}, {"KA_ORDER_GLOBAL_CTR": "1"}], ids=["shared-ctr", "global-ctr"])
def test_lookup_modes_both_ways(native_lib, oracle, env):
    """Tables in each lookup mode, switched in both directions (shared LUT -> global LUT -> binary search -> shared LUT ->
    binary search -> global LUT -> shared LUT), the problems' current brokers among ids 1..60: the counters carry over each
    switch."""
    rng = np.random.default_rng(0x700C)
    m = Mirror(oracle)
    tables = {"smem": util.table(np.arange(1, 61), 5), "global-lut": util.table(1 + 2 * np.arange(20000, dtype=np.int32), 500),
              "bsearch": util.bsearch_table(20000)}
    mask = {"smem": 1, "global-lut": 2, "bsearch": 4}
    hot = np.arange(1, 61, dtype=np.int32)
    with mock.patch.dict(os.environ, env):
        for k, mode in enumerate(("smem", "global-lut", "bsearch", "smem", "bsearch", "global-lut", "smem")):
            ids, racks = tables[mode]
            m.set_table(ids, [None if r is None else "k%d" % r for r in racks.tolist()])
            prob = Dense(rng, hot, "lut%d" % k, T=3, rf=3)
            m.solve(prob, ("device_sync", "solve", "staged_slots")[k % 3])
            assert m.s.last_stage_plan()[6] == mask[mode], mode
    m.roll_call()
    assert m.errors == 0


@pytest.mark.gpu
def test_wide_rows_park_every_slot(native_lib, oracle):
    """Rows of 4..8 bump slots 3..7; those counters are parked with the rest and restored exactly, with rows of 3 solved
    in between."""
    rng = np.random.default_rng(0x81DE)
    m = Mirror(oracle)
    a, b = np.arange(1, 33), np.arange(9, 41)
    racks = lambda ids: ["r%d" % (i % 8) for i in ids]
    for k, (ids, rf, drf) in enumerate(((a, 4, 8), (b, 3, -1), (a, 3, 6), (b, 8, -1), (a, 3, -1), (b, 5, 7), (a, 3, 3))):
        m.set_table(ids, racks(ids))
        m.solve(Dense(rng, POOL, "wide%d" % k, T=2, rf=rf, max_rf=8, desired_rf=drf), ("solve", "dense", "device_sync")[k % 3])
    assert m.errors == 0 and np.any(m.s.counters()[:, 3:] != 0)
    m.roll_call()


@pytest.mark.gpu
def test_empty_and_refused_tables(native_lib, oracle):
    """A table of no brokers parks every counter (a solve on it is the reference's exception); the ids then return. A refused
    table (ids not ascending, a rack index out of range) changes neither the table nor any counter."""
    rng = np.random.default_rng(0xE777)
    m = Mirror(oracle)
    a = np.arange(1, 21)
    m.set_table(a, ["r%d" % (i % 3) for i in a])
    m.solve(Dense(rng, POOL, "e0", rf=3), "solve")
    before = m.s.counters()
    racks = kab.synth.rack_indices(a, m.racks)
    for ids, rk in ((a[::-1].copy(), racks), (a, np.where(np.arange(len(a)) == 3, -1, racks))):
        with pytest.raises(kab.KassignError):
            m.s.set_brokers(ids, rk)
        assert np.array_equal(m.s.counters(), before)
        m.solve(Dense(rng, a, "e1", rf=3), "device_sync")   # solves on the old table, from the old counters
        before = m.s.counters()
    saved = (m.ids, m.racks)
    m.set_table(np.zeros(0, dtype=np.int32), [])
    out, ln, st = m.s.solve_ragged(*Dense(rng, POOL, "e2", rf=2).ragged(), -1, 2, check=False)
    assert st.code == kab.assigner._native.KA_ERR_RF_GT_BROKERS
    m.set_table(*saved)
    m.solve(Dense(rng, POOL, "e3", rf=3), "dense")
    m.roll_call()


@pytest.mark.gpu
def test_zeroed_counters_return_as_zeros(native_lib, oracle):
    """set_counters zeroes some brokers' rows, then they leave: they are erased from the parked ones, not parked with their
    old values, and come back as zeros."""
    rng = np.random.default_rng(0x2E80)
    m = Mirror(oracle)
    a = np.arange(1, 31)
    m.set_table(a, ["r%d" % (i % 5) for i in a])
    m.solve(Dense(rng, POOL, "z0", rf=3), "solve")
    m.set_table(a[5:], ["r%d" % (i % 5) for i in a[5:]])    # ids 1..5 parked with nonzero counters
    m.set_table(a, ["r%d" % (i % 5) for i in a])            # and back
    ctr = m.s.counters()
    ctr[:10] = 0
    m.set_counters(ctr)
    m.set_table(a[10:], ["r%d" % (i % 5) for i in a[10:]])
    m.set_table(a, ["r%d" % (i % 5) for i in a])
    assert not np.any(m.s.counters()[:10])
    m.solve(Dense(rng, POOL, "z1", rf=3), "dense")


@pytest.mark.gpu
def test_reset_drops_parked_counters(native_lib, oracle):
    """reset() while counters are parked: a returning id comes back with zeros."""
    rng = np.random.default_rng(0x8E5E)
    m = Mirror(oracle)
    a = np.arange(1, 31)
    m.set_table(a, ["r%d" % (i % 5) for i in a])
    m.solve(Dense(rng, POOL, "r0", rf=3), "solve")
    m.set_table(a[:10], ["r%d" % (i % 5) for i in a[:10]])
    m.reset()
    m.set_table(a, ["r%d" % (i % 5) for i in a])
    assert not np.any(m.s.counters())
    m.solve(Dense(rng, POOL, "r1", rf=3), "device_sync")
    m.roll_call()


@pytest.mark.gpu
def test_counters_near_int_max_are_parked_exactly(native_lib, oracle):
    """Counters at and near INT_MAX (as in test_chain_edges.test_high_counters_with_short_rows), parked and restored bit
    for bit; a solve from them is the oracle's (every value a run reads stays below INT_MAX)."""
    rng = np.random.default_rng(0x7FFF)
    m = Mirror(oracle)
    a = np.arange(1, 31)
    m.set_table(a, ["r%d" % (i % 5) for i in a])
    ctr = (INT_MAX - 1000 + ranks(len(a), rng, 0, 200)).astype(np.int32)
    ctr[::7] = INT_MAX      # slots 3..7, which rows of at most 3 never read
    ctr[::7, :3] = INT_MAX - 500
    m.set_counters(ctr)
    m.set_table(a[10:], ["r%d" % (i % 5) for i in a[10:]])
    m.solve(Dense(rng, a[10:], "h0", rf=2), "solve")
    m.set_table(a, ["r%d" % (i % 5) for i in a])
    assert np.array_equal(m.s.counters()[:10], ctr[:10])
    m.solve(Dense(rng, a, "h1", rf=3), "staged_slots")
    m.roll_call()


@pytest.mark.gpu
def test_batched_calls_between_leave_and_return(native_lib, oracle):
    """Batched calls between a leave and a return leave the table and the parked counters alone: the returning ids'
    counters and the next solve are the oracle's."""
    rng = np.random.default_rng(0xBA7C)
    m = Mirror(oracle)
    a = np.arange(1, 31)
    m.set_table(a, ["r%d" % (i % 5) for i in a])
    m.solve(Dense(rng, POOL, "b0", rf=3), "solve")
    m.set_table(a[8:], ["r%d" % (i % 5) for i in a[8:]])
    m.solve(Dense(rng, POOL, "b1", rf=3), "dense")
    m.batched(rng, POOL)
    m.set_table(a, ["r%d" % (i % 5) for i in a])
    m.solve(Dense(rng, POOL, "b2", rf=3), "device_sync")
    m.roll_call()


# ---- random sequences ------------------------------------------------------------------------------------------------------

# ids 1..40 (a shared-memory LUT), 40 000 (a table holding it and a small id takes the global LUT) and 2^27 (binary search)
SEQ_POOL = np.concatenate([np.arange(1, 41), [40000, 1 << 27]]).astype(np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [11, 12, 13])
def test_random_sequences(native_lib, oracle, seed):
    """90 random steps per seed: a table change (now and then a roll call), a solve through a random entry point, set_counters,
    reset, a device export / import round trip, or the batched calls; every step checked against the oracle Context."""
    rng = np.random.default_rng(0x5E90 + seed)
    m = Mirror(oracle)
    m.set_table(*random_table(rng, SEQ_POOL))
    done = set()
    for step in range(90):
        pick = rng.random()
        if pick < 0.2:
            m.set_table(*random_table(rng, SEQ_POOL))
            done.add("table")
        elif pick < 0.25:
            m.roll_call()
        elif pick < 0.7:
            entry = ENTRIES[int(rng.integers(len(ENTRIES)))]
            m.solve(Dense(rng, SEQ_POOL, "s%d-%d" % (seed, step), max_rf=5 if rng.random() < 0.2 else 3), entry)
            done.add(entry)
        elif pick < 0.78:
            m.set_counters(ranks(len(m.ids), rng))
        elif pick < 0.82:
            m.reset()
        elif pick < 0.91:
            m.device_round_trip(rng)
            done.add("round trip")
        else:
            m.batched(rng, SEQ_POOL)
            done.add("batched")
    m.roll_call()
    assert len(done) >= 8, done


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [21, 22])
def test_front_ends_agree_on_call_sequences(native_lib, seed):
    """The Python KafkaTopicAssigner (its broker-table cache keyed by brokers and racks) against py_oracle's through the same
    generate_assignment calls, the broker set and rack map changing between them: the reference JUnit's calls."""
    rng = np.random.default_rng(0xF407 + seed)
    pool = np.arange(1, 31, dtype=np.int32)
    lib, ref = kab.KafkaTopicAssigner(0), po.KafkaTopicAssigner()
    ids, racks = random_table(rng, pool)
    for step in range(60):
        if rng.random() < 0.4:
            ids, racks = random_table(rng, pool) if rng.random() < 0.9 else (np.zeros(0, dtype=np.int32), [])
        elif rng.random() < 0.2:
            racks = [None if r is None else r + "x" for r in racks]   # the same brokers on other racks
        prob = Dense(rng, pool, "fe%d-%d" % (seed, step), T=1, max_rf=4)
        cur = {p: [int(b) for b in prob.cur[0, p]] for p in range(prob.P)}
        rack_map = {int(b): r for b, r in zip(ids, racks) if r is not None}
        brokers = set(int(b) for b in ids)
        try:
            exp = ref.generate_assignment(prob.names[0], cur, brokers, rack_map, prob.desired_rf)
        except po.JavaError:
            with pytest.raises((kab.IllegalStateException, kab.ArrayIndexOutOfBoundsException)):
                lib.generate_assignment(prob.names[0], cur, brokers, rack_map, prob.desired_rf)
            lib, ref = kab.KafkaTopicAssigner(0), po.KafkaTopicAssigner()
            continue
        assert lib.generate_assignment(prob.names[0], cur, brokers, rack_map, prob.desired_rf) == exp, step
        got = lib._solver.counters()
        for i, b in enumerate(lib._solver.broker_id):
            assert got[i].tolist() == [ref.context.counter.get(int(b), {}).get(r, 0) for r in range(SLOTS)], (step, int(b))


# ---- host calls behind asynchronous calls on the same Context ---------------------------------------------------------

# asynchronous calls that leave no status pending, then the controls, whose pending status every host call already collects
ASYNC = ["stage", "order_slot0", "order_slot1", "import", "export", "import_slot", "export_slot",
         "solve_device", "order_device", "emit"]
HOST = ["get_counters", "set_counters", "reset", "set_brokers", "solve_ragged", "solve_dense", "last_status"]
COL = 1   # the counter column of the one-slot import / export


@pytest.fixture(scope="module")
def behind(oracle):
    """The problem X the asynchronous calls solve, the other problem Y the host solves take, on one table of 40 brokers, and
    counters: C0 in the Context, C1 to import, C2 for set_counters. F and R: the counters and rows of X solved from C0."""
    X = kab.synth.make_cluster(T=6, P=16, RF=3, N=40, R=5, seed=0xB41D, kind="mixed")
    Y = kab.synth.make_cluster(T=3, P=8, RF=3, N=40, R=5, seed=0xB41E, kind="mixed", topic_prefix="other-")
    assert np.array_equal(X.broker_id, Y.broker_id) and np.array_equal(X.rack_index, Y.rack_index)
    rng = np.random.default_rng(0xB41D)
    N = len(X.broker_id)
    C0, C1, C2 = ranks(N, rng), ranks(N, rng, 50, 90), ranks(N, rng, 100, 140)
    R, F = from_counters(oracle, X, C0)[:2]
    return dict(X=X, Y=Y, C0=C0, C1=C1, C2=C2, F=F, R=R)


def from_counters(oracle, cl, ctr):
    """(rows [Q, RF], counters [N, 8] after, lengths) of the oracle solving cl from the preloaded counters ctr."""
    octx = oracle.OracleContext()
    for i, b in enumerate(cl.broker_id):
        for r in range(SLOTS):
            octx.set_counter(int(b), r, int(ctr[i, r]))
    part_off, part_id, rep_off, cur = cl.ragged()
    ln, _, out, st = oracle.run(octx, cl.topic_names, part_off, part_id, rep_off, cur, cl.broker_id, cl.rack_name, -1, cl.RF)
    after = np.array([[octx.counter(int(b), r) for r in range(SLOTS)] for b in cl.broker_id], dtype=np.int32)
    return out, after, ln


def after_async(call, b):
    """The Context's counters once the asynchronous call has run, from C0."""
    C0, F = b["C0"], b["F"]
    post = C0.copy()
    if call == "order_slot0":
        post[:, 0] = F[:, 0]
    elif call == "order_slot1":
        post[:, :2] = F[:, :2]
    elif call in ("emit", "solve_device", "order_device"):
        post = F.copy()
    elif call == "import":
        post = b["C1"].copy()
    elif call == "import_slot":
        post[:, COL] = b["C1"][:, COL]
    return post


@pytest.mark.gpu
@pytest.mark.parametrize("host", HOST)
@pytest.mark.parametrize("call", ASYNC)
def test_host_call_sees_async_call(native_lib, oracle, behind, call, host):
    """One asynchronous call held behind a device sleep on a non-blocking torch stream, then at once one host call of the same
    Context. The host call must act as if the asynchronous call had finished: the sleep has ended when it returns, a read
    sees what the asynchronous call wrote, a write does not reach what it read (an export carries C0, not what set_counters
    or set_brokers wrote after it), and a staged block then ordered gives the oracle's rows from the counters of that moment."""
    import time
    import torch
    b = behind
    X, Y, C0 = b["X"], b["Y"], b["C0"]
    N = len(X.broker_id)
    s = kab.Solver(0)
    s.set_brokers(X.broker_id, X.rack_index)
    d_hash, d_cur = torch.from_numpy(X.topic_hash).cuda(), torch.from_numpy(X.cur).cuda()
    d_out = torch.full((X.T, X.P, 3), -7, dtype=torch.int32, device="cuda")
    d_len = torch.full((X.T, X.P), -7, dtype=torch.int32, device="cuda")
    d_c1 = torch.from_numpy(b["C1"]).cuda()
    d_col = torch.from_numpy(np.ascontiguousarray(b["C1"][:, COL])).cuda()
    d_exp = torch.full((N, SLOTS), -7, dtype=torch.int32, device="cuda")
    d_exp_col = torch.full((N,), -7, dtype=torch.int32, device="cuda")
    stage_args = (X.T, d_hash.data_ptr(), X.P, X.RF, d_cur.data_ptr(), -1, 3)
    # scratch reserved at this shape (a reservation that frees a buffer waits for the device), then the Context at C0
    s.solve_dense_device(*stage_args, d_len.data_ptr(), d_out.data_ptr())
    s.solve_dense(Y.topic_hash, Y.cur)
    s.set_counters(C0)
    d_out.fill_(-7)
    d_len.fill_(-7)
    if call in ("order_slot0", "order_slot1", "order_device", "emit"):
        s.stage_dense_device(*stage_args)
        assert s.staged_slot_chains() == 2
        if call in ("order_slot1", "emit"):
            s.order_slot_device(0)
        if call == "emit":
            s.order_slot_device(1)
    torch.cuda.synchronize()

    stream = torch.cuda.Stream()
    h = stream.cuda_stream
    sleep = util.device_sleep(stream)
    t0 = time.perf_counter()
    if call == "stage":
        s.stage_dense_device(*stage_args, stream=h)
    elif call in ("order_slot0", "order_slot1"):
        s.order_slot_device(int(call[-1]), stream=h)
    elif call == "import":
        s.import_counters_device(d_c1.data_ptr(), stream=h)
    elif call == "export":
        s.export_counters_device(d_exp.data_ptr(), stream=h)
    elif call == "import_slot":
        s.import_counter_slot_device(COL, d_col.data_ptr(), stream=h)
    elif call == "export_slot":
        s.export_counter_slot_device(COL, d_exp_col.data_ptr(), stream=h)
    elif call == "solve_device":
        s.solve_dense_device(*stage_args, d_len.data_ptr(), d_out.data_ptr(), stream=h, sync=False)
    elif call == "order_device":
        s.order_device(d_len.data_ptr(), d_out.data_ptr(), stream=h, sync=False)
    else:
        s.emit_device(d_len.data_ptr(), d_out.data_ptr(), stream=h, sync=False)
    t_call = time.perf_counter() - t0

    post = after_async(call, b)
    now = None          # the counters the Context holds after the host call
    if host == "get_counters":
        got = s.counters()
        done = sleep[1].query()
        now = post
    elif host == "set_counters":
        s.set_counters(b["C2"])
        done = sleep[1].query()
        now = b["C2"]
    elif host == "reset":
        s.reset()
        done = sleep[1].query()
        now = np.zeros_like(C0)
    elif host == "set_brokers":
        # the same number of brokers: 8 of X's leave, 8 new ids come; no buffer is reallocated
        ids = np.concatenate([X.broker_id[8:], X.broker_id[-1] + 1 + np.arange(8)]).astype(np.int32)
        s.set_brokers(ids, np.arange(N, dtype=np.int32) % 5)
        done = sleep[1].query()
        torch.cuda.synchronize()
        s.set_brokers(X.broker_id, X.rack_index)   # X's ids return with what they held when they left
        now = post
    elif host in ("solve_ragged", "solve_dense"):
        if host == "solve_ragged":
            part_off, part_id, rep_off, cur = Y.ragged()
            y_out, y_len, st = s.solve_ragged(Y.topic_hash, part_off, part_id, rep_off, cur, -1, 3, check=False)
        else:
            y_out, y_len, st = s.solve_dense(Y.topic_hash, Y.cur, check=False)
        done = sleep[1].query()
        e_out, now, e_len = from_counters(oracle, Y, post)
        assert st.code == 0
        assert np.array_equal(y_out.reshape(-1, 3), e_out), ("the host solve did not start from the %s call's counters" % call,
                                                   differs(y_out.reshape(-1, 3), e_out))
        assert np.array_equal(y_len.reshape(-1), e_len)
    else:
        st = s.last_status()
        done = sleep[1].query()
        assert st.code == 0
        now = post
    torch.cuda.synchronize()
    util.enqueued_behind(sleep, t_call)
    if host == "get_counters":
        assert np.array_equal(got, post), ("get_counters did not see the %s call's counters" % call, differs(got, post))
    if call == "export":
        assert np.array_equal(d_exp.cpu().numpy(), C0), ("the export carried counters written after it", differs(d_exp.cpu().numpy(), C0))
    if call == "export_slot":
        got_col = d_exp_col.cpu().numpy()
        assert np.array_equal(got_col, C0[:, COL]), ("the export carried counters written after it", differs(got_col, C0[:, COL]))
    if call in ("solve_device", "order_device", "emit"):
        assert np.array_equal(d_out.cpu().numpy().reshape(-1, 3), b["R"])
    if call == "stage" and host not in ("solve_ragged", "solve_dense"):
        # the staged block, ordered now, from the counters of this moment
        st = s.order_device(d_len.data_ptr(), d_out.data_ptr())
        assert st.code == 0
        e_out, now, _ = from_counters(oracle, X, now)
        got_out = d_out.cpu().numpy().reshape(-1, 3)
        assert np.array_equal(got_out, e_out), ("the staged rows are not the oracle's", differs(got_out, e_out))
    final = s.counters()
    assert np.array_equal(final, now), ("the counters after %s are not what the calls in order leave" % host, differs(final, now))
    assert done, "%s returned before the %s call queued ahead of it had run" % (host, call)
    s.close()


def differs(got, exp):
    """How got differs from exp: the number of rows that differ and the first few, (row, got, expected)."""
    got, exp = got.reshape(len(exp), -1), exp.reshape(len(exp), -1)
    bad = np.nonzero(np.any(got != exp, axis=1))[0]
    return "%d of %d rows differ" % (len(bad), len(exp)), [(int(i), got[i].tolist(), exp[i].tolist()) for i in bad[:3]]
