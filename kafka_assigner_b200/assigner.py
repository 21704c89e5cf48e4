"""Host-side mirror of the reference's interface for the hot path, over the C ABI (include/kassign.h).

  KafkaTopicAssigner.generate_assignment(...)  <->  KafkaTopicAssigner.generateAssignment
                                                    (reference KafkaTopicAssigner.java:42-72)
  Solver.solve_cluster(...)                    <->  the per-topic loop with ONE shared assigner
                                                    (reference KafkaAssignmentGenerator.java:172-184)

Same names, argument meaning and error behaviour (message texts of KTA:58-60, 65-66, 67-69 and
KAS:183-184). All compute happens in libkassign.so's CUDA kernels; nothing here falls back to a CPU
solver — if the library or a GPU is missing, construction raises.
"""
import collections
import ctypes

import numpy as np

from . import _native
from ._native import KaBrokerUsage, KaMoveSummary, KaStatus, KaWaveSendSummary, KaWaveSummary

# numpy view of ka_move_summary (KaMoveSummary): one record per candidate
MOVE_SUMMARY_DTYPE = np.dtype([(name, np.int64) for name, _ in KaMoveSummary._fields_])
# numpy view of ka_wave_summary (KaWaveSummary): one record per wave of Solver.plan_waves
WAVE_SUMMARY_DTYPE = np.dtype([(name, np.int64) for name, _ in KaWaveSummary._fields_])
# ka_wave_summary followed by ka_wave_send_summary: one record per wave of a plan with a sender budget
WAVE_SEND_SUMMARY_DTYPE = np.dtype([(name, np.int64) for name, _ in KaWaveSummary._fields_ + KaWaveSendSummary._fields_])
_SEND_FIELDS = [name for name, _ in KaWaveSendSummary._fields_]
# numpy view of ka_broker_usage (KaBrokerUsage): one record per broker of Solver.broker_usage's usage table
BROKER_USAGE_DTYPE = np.dtype([(name, np.int64) for name, _ in KaBrokerUsage._fields_])


class IllegalStateException(Exception):
    """java.lang.IllegalStateException as thrown by Preconditions.checkState on the reference path."""


class ArrayIndexOutOfBoundsException(Exception):
    """java.lang.ArrayIndexOutOfBoundsException (topic.hashCode() == Integer.MIN_VALUE, KAS:190-192)."""


class KassignError(RuntimeError):
    """Library-side failure with no reference counterpart (bad argument, CUDA error, size limit)."""

    def __init__(self, code, msg=""):
        super().__init__("kassign error %d %s" % (code, msg))
        self.code = code


def java_string_hash(s: str) -> int:
    """String.hashCode of s (ka_java_string_hash). A name holding U+0000 is a ValueError: the C string would end there, and
    the topic would be solved with the hash of its prefix."""
    if "\0" in s:
        raise ValueError("topic name %r holds U+0000" % s)
    return _native.load().ka_java_string_hash(s.encode("utf-8"))


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _vp(x):
    """An optional device pointer or stream (an int, 0 for none) as a C ABI argument."""
    return ctypes.c_void_p(x) if x else None


def _check(rc, what=""):
    """Raise KassignError for a nonzero return code."""
    if rc:
        raise KassignError(rc, what)


def _statuses(K):
    """The KaStatus array of a batched call (never empty: the C ABI requires st) and the list of its first K, which share its
    memory and so read what the call wrote."""
    st = (KaStatus * max(K, 1))()
    return st, st[:K]


def _stride(longest, desired_rf):
    """The row stride when the caller gives none: max(longest current list, desired_rf, 1)."""
    return max(longest, desired_rf, 1)


def _json_size(rows, name_bytes, stride):
    """The sufficient buffer size kassign.h documents for one document: 64 + per row (50 + 12·stride + its topic's name
    length); name_bytes = Σ rows·name length over the topics."""
    return 64 + rows * (50 + 12 * stride) + name_bytes


def _send_part(max_broker_out, send_brokers):
    """The sender part of a wave plan as the _send entry points take it: None without a sender budget, else (n_send, send_id as
    contiguous int32, max_broker_out). send_brokers is required with a budget, and only with one."""
    if max_broker_out is None and send_brokers is None:
        return None
    if max_broker_out is None or send_brokers is None:
        raise ValueError("max_broker_out and send_brokers go together")
    send_id = np.ascontiguousarray(send_brokers, dtype=np.int32)
    return len(send_id), send_id, int(max_broker_out)


def _with_send(summary, send_summary):
    """summary [W] (WAVE_SUMMARY_DTYPE) and send_summary [W] (its ka_wave_send_summary fields) as one WAVE_SEND_SUMMARY_DTYPE
    array."""
    both = np.zeros(len(summary), dtype=WAVE_SEND_SUMMARY_DTYPE)
    for name in WAVE_SUMMARY_DTYPE.names:
        both[name] = summary[name]
    for j, name in enumerate(_SEND_FIELDS):
        both[name] = send_summary[:, j]
    return both


def _wave_json_size(rows, name_bytes, stride):
    """The sufficient buffer size kassign.h documents for the documents of a wave plan: per row 79 + 12·stride + its topic's
    name length (a record of _json_size, and a document's 29 bytes of header and trailer charged to every row)."""
    return rows * (79 + 12 * stride) + name_bytes


class _Ragged(collections.namedtuple("_Ragged", "topic_hash part_off part_id rep_off cur_broker Q")):
    """A ragged problem as the C ABI takes it: (topic_hash, part_off, part_id, rep_off, cur_broker) as contiguous arrays of
    their element types (part_id may be None), and Q = ΣP, its number of rows."""
    __slots__ = ()

    def stride(self, desired_rf):
        sizes = np.diff(self.rep_off)
        return _stride(int(sizes.max()) if len(sizes) else 0, desired_rf)

    def name_bytes(self, name_len):
        """Σ rows·name length, name_len holding one length per topic."""
        return int(np.dot(np.diff(self.part_off), name_len))

    def ptrs(self):
        return tuple(_ptr(a) for a in self[:5])


def _ragged(topic_hash, part_off, part_id, rep_off, cur_broker):
    part_off = np.ascontiguousarray(part_off, dtype=np.int64)
    return _Ragged(np.ascontiguousarray(topic_hash, dtype=np.int32), part_off,
                   None if part_id is None else np.ascontiguousarray(part_id, dtype=np.int32),
                   np.ascontiguousarray(rep_off, dtype=np.int64), np.ascontiguousarray(cur_broker, dtype=np.int32),
                   int(part_off[-1]) if len(part_off) else 0)


def raise_for_status(st: KaStatus, topic_names=None):
    """Re-throw a ka_status as the reference's exception with the identical message."""
    if st.code == 0:
        return
    topic = topic_names[st.topic_index] if (topic_names is not None and 0 <= st.topic_index < len(topic_names)) else "?"
    if st.code == _native.KA_ERR_RF_MISMATCH:
        raise IllegalStateException("Topic %s has partition %d with unexpected replication factor %d" % (topic, st.partition, st.a))
    if st.code == _native.KA_ERR_RF_NOT_POSITIVE:
        raise IllegalStateException("Topic %s does not have a positive replication factor!" % topic)
    if st.code == _native.KA_ERR_RF_GT_BROKERS:
        raise IllegalStateException("Topic %s has a higher replication factor (%d) than available brokers!" % (topic, st.a))
    if st.code == _native.KA_ERR_UNASSIGNABLE:
        raise IllegalStateException("Partition %d could not be fully assigned!" % st.partition)
    if st.code == _native.KA_ERR_HASH_INDEX:
        raise ArrayIndexOutOfBoundsException(str(st.a))
    raise KassignError(st.code, "(topic_index=%d partition=%d a=%d b=%d)" % (st.topic_index, st.partition, st.a, st.b))


class Solver:
    """One ka_ctx: one Context (KAS:360-369) plus device scratch. Batch-level API on flat arrays."""

    def __init__(self, device=0):
        self._L = _native.load()
        h = self._L.ka_ctx_create(int(device))
        if not h:
            raise KassignError(_native.KA_ERR_NO_DEVICE, "no usable CUDA device: kassign has no CPU fallback")
        self._h = ctypes.c_void_p(h)
        self.device = device
        self.N = 0
        self.broker_id = None

    def close(self):
        if getattr(self, "_h", None):
            self._L.ka_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- Context -------------------------------------------------------------------------------
    def reset(self):
        _check(self._L.ka_ctx_reset(self._h))

    def set_brokers(self, broker_id, rack_index):
        b = np.ascontiguousarray(broker_id, dtype=np.int32)
        r = np.ascontiguousarray(rack_index, dtype=np.int32)
        _check(self._L.ka_ctx_set_brokers(self._h, len(b), _ptr(b), _ptr(r)), "ka_ctx_set_brokers")
        self.N = len(b)
        self.broker_id = b

    def set_brokers_with_racks(self, brokers, rack_assignment):
        """brokers: iterable of ids (any order); rack_assignment: {id: rack string} (may lack entries)."""
        b = np.array(sorted(set(int(x) for x in brokers)), dtype=np.int32)
        names = [rack_assignment.get(int(x)) for x in b]
        arr = (ctypes.c_char_p * len(b))(*[(n.encode("utf-8") if n is not None else None) for n in names])
        racks = np.zeros(len(b), dtype=np.int32)
        _check(self._L.ka_rack_indices(len(b), _ptr(b), ctypes.cast(arr, ctypes.c_void_p), _ptr(racks)), "ka_rack_indices")
        self.set_brokers(b, racks)
        return b

    def counters(self):
        slots = self._L.ka_ctx_counter_slots(self._h)
        out = np.zeros((self.N, slots), dtype=np.int32)
        _check(self._L.ka_ctx_get_counters(self._h, _ptr(out)))
        return out

    def set_counters(self, ctr):
        c = np.ascontiguousarray(ctr, dtype=np.int32)
        assert c.shape == (self.N, self._L.ka_ctx_counter_slots(self._h))
        _check(self._L.ka_ctx_set_counters(self._h, _ptr(c)))

    def set_timing(self, on=True):
        self._L.ka_ctx_set_timing(self._h, 1 if on else 0)

    WAVE_RULES = {"greedy": _native.KA_WAVE_GREEDY, "first_fit": _native.KA_WAVE_FIRST_FIT}

    def set_wave_rule(self, rule):
        """The wave rule of every plan_waves / plan_waves_json / plan_wave_parts_json / plan_wave_parts_rollback_json call of this
        Solver (ka_ctx_set_wave_rule): "greedy" (the default: a broker's waves only move forward) or "first_fit" (each row in the
        earliest wave where its receivers and its leader still have room, which often needs fewer waves). reset() keeps it."""
        if rule not in self.WAVE_RULES:
            raise ValueError("wave rule must be one of %s, not %r" % (sorted(self.WAVE_RULES), rule))
        _check(self._L.ka_ctx_set_wave_rule(self._h, self.WAVE_RULES[rule]), "ka_ctx_set_wave_rule")

    @property
    def wave_rule(self):
        """The wave rule set_wave_rule chose: "greedy" or "first_fit"."""
        code = self._L.ka_ctx_wave_rule(self._h)
        _check(min(code, 0), "ka_ctx_wave_rule")
        return {v: k for k, v in self.WAVE_RULES.items()}[code]

    def set_part_caps(self, max_rows=None, max_in=None):
        """The part caps of every plan_wave_parts_json / plan_wave_parts_rollback_json call of this Solver
        (ka_ctx_set_part_caps): a part holds at most max_rows rows, and moves at most max_in of data (weight x the row's new
        replicas, summed over the part's rows) unless it is a single row. None (or 0) is no cap. The cut only gets finer: the
        plan, wave and the summaries stay those of the uncapped call. reset() keeps them. A negative cap raises ValueError and
        leaves the caps as they were."""
        rows, data = (0 if x is None else int(x) for x in (max_rows, max_in))
        if rows < 0 or data < 0:
            raise ValueError("part caps must be >= 0 (0 or None: no cap), not %r, %r" % (max_rows, max_in))
        _check(self._L.ka_ctx_set_part_caps(self._h, rows, data), "ka_ctx_set_part_caps")

    def part_caps(self):
        """(max_rows, max_in) as set_part_caps set them, None where there is no cap."""
        rows, data = ctypes.c_int64(0), ctypes.c_int64(0)
        _check(self._L.ka_ctx_part_caps(self._h, ctypes.byref(rows), ctypes.byref(data)), "ka_ctx_part_caps")
        return tuple(x.value or None for x in (rows, data))

    def last_timing(self):
        ms = np.zeros(8, dtype=np.float32)
        self._L.ka_ctx_last_timing(self._h, _ptr(ms))
        return dict(sticky_spread_ms=float(ms[0]), level_tables_ms=float(ms[1]), leader_order_ms=float(ms[2]),
                    h2d_ms=float(ms[3]), d2h_ms=float(ms[4]), total_ms=float(ms[5]), slot1_emit_ms=float(ms[6]), chains_wall_ms=float(ms[7]))

    def set_topic_base(self, topic_base):
        """Topic-sharded runs: index of this rank's first topic in the whole run (status reporting)."""
        _check(self._L.ka_ctx_set_topic_base(self._h, int(topic_base)))

    def launch_count(self):
        return int(self._L.ka_ctx_launch_count(self._h))

    def last_order_plan(self):
        """The leader-order plan of the last solve call (ka_ctx_last_order_plan): (rec_kind, levels, chain threads, ring_log2,
        gctr, loop shape [0 general, 1 warp1, 2 single, 3 full], chain launches, candidates K)."""
        plan = np.zeros(8, dtype=np.int32)
        _check(self._L.ka_ctx_last_order_plan(self._h, _ptr(plan)), "ka_ctx_last_order_plan")
        return tuple(int(x) for x in plan)

    def last_stage_plan(self):
        """The sticky/spread plan of the last solve call (ka_ctx_last_stage_plan): (load bytes, levels, SM, candidates K,
        warps per CTA, grid.x, lookup-mode mask [1 shared LUT, 2 global LUT, 4 binary search], kernel A launches)."""
        plan = np.zeros(8, dtype=np.int32)
        _check(self._L.ka_ctx_last_stage_plan(self._h, _ptr(plan)), "ka_ctx_last_stage_plan")
        return tuple(int(x) for x in plan)

    # -- solves --------------------------------------------------------------------------------
    def solve_dense(self, topic_hash, cur, desired_rf=-1, out_stride=None, out=None, out_len=None, check=True,
                    topic_names=None):
        """cur: int32 [T, P, RF] host array -> (out [T, P, out_stride], out_len [T, P], status)."""
        cur = np.ascontiguousarray(cur, dtype=np.int32)
        T, P, RF = cur.shape
        th = np.ascontiguousarray(topic_hash, dtype=np.int32)
        assert th.shape == (T,)
        if out_stride is None:
            out_stride = _stride(RF, desired_rf)
        if out is None:
            out = np.full((T, P, out_stride), -1, dtype=np.int32)
        if out_len is None:
            out_len = np.zeros((T, P), dtype=np.int32)
        st = KaStatus()
        self._L.ka_solve_dense(self._h, T, _ptr(th), P, RF, _ptr(cur), int(desired_rf), int(out_stride), _ptr(out_len),
                               _ptr(out), ctypes.byref(st))
        if check:
            raise_for_status(st, topic_names)
        return out, out_len, st

    @staticmethod
    def marshal_names(topic_names):
        """(concatenated UTF-8 bytes, offsets[T+1]) — the name slab ka_solve_dense_json takes."""
        enc = [n.encode("utf-8") for n in topic_names]
        name_off = np.zeros(len(enc) + 1, dtype=np.int64)
        name_off[1:] = np.cumsum([len(e) for e in enc])
        return np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8), name_off

    def solve_dense_json(self, topic_names, topic_hash, cur, desired_rf=-1, json_buf=None, check=True, names_slab=None):
        """Solve + emit the reassignment JSON on the device (KAG:169-186); returns (bytes-like view of the text, status).
        json_buf: optional writable uint8 numpy array (pinned memory for full PCIe speed); names_slab: marshal_names() result."""
        cur = np.ascontiguousarray(cur, dtype=np.int32)
        T, P, RF = cur.shape
        th = np.ascontiguousarray(topic_hash, dtype=np.int32)
        names, name_off = names_slab if names_slab is not None else self.marshal_names(topic_names)
        if json_buf is None:    # every topic has P rows
            json_buf = np.empty(_json_size(T * P, P * int(name_off[-1]), _stride(RF, desired_rf)), dtype=np.uint8)
        nbytes = ctypes.c_int64(0)
        st = KaStatus()
        self._L.ka_solve_dense_json(self._h, T, _ptr(th), P, RF, _ptr(cur), int(desired_rf), _ptr(names), _ptr(name_off),
                                    _ptr(json_buf), int(json_buf.size), ctypes.byref(nbytes), ctypes.byref(st))
        if check:
            raise_for_status(st, topic_names)
        return json_buf[:nbytes.value], st

    def solve_ragged(self, topic_hash, part_off, part_id, rep_off, cur_broker, desired_rf, out_stride, check=True,
                     topic_names=None):
        r = _ragged(topic_hash, part_off, part_id, rep_off, cur_broker)
        out = np.full((r.Q, out_stride), -1, dtype=np.int32)
        out_len = np.zeros(r.Q, dtype=np.int32)
        st = KaStatus()
        self._L.ka_solve(self._h, len(r.topic_hash), *r.ptrs(), int(desired_rf), int(out_stride), _ptr(out_len), _ptr(out),
                         ctypes.byref(st))
        if check:
            raise_for_status(st, topic_names)
        return out, out_len, st

    def solve_ragged_json(self, topic_names, topic_hash, part_off, part_id, rep_off, cur_broker, desired_rf, json_buf=None,
                          check=True):
        """ka_solve_json: the ragged solve of solve_ragged + the reassignment JSON built on the device (KAG:169-186);
        returns (bytes-like view of the text, status). json_buf: optional writable uint8 numpy array (pinned for full
        PCIe speed); by default one of the documented sufficient size."""
        r = _ragged(topic_hash, part_off, part_id, rep_off, cur_broker)
        names, name_off = self.marshal_names(topic_names)
        if json_buf is None:
            json_buf = np.empty(_json_size(r.Q, r.name_bytes(np.diff(name_off)), r.stride(desired_rf)), dtype=np.uint8)
        nbytes = ctypes.c_int64(0)
        st = KaStatus()
        self._L.ka_solve_json(self._h, len(r.topic_hash), *r.ptrs(), int(desired_rf), _ptr(names), _ptr(name_off), _ptr(json_buf),
                              int(json_buf.size), ctypes.byref(nbytes), ctypes.byref(st))
        if check:
            raise_for_status(st, topic_names)
        return json_buf[:nbytes.value], st

    def _synced(self, name, *args, stream, sync):
        """Call the device-pointer entry `name` on `stream`: with sync, return its KaStatus without raising; otherwise raise
        on its return code and return None."""
        st = KaStatus()
        rc = getattr(self._L, name)(self._h, *args, _vp(stream), ctypes.byref(st) if sync else None)
        if sync:
            return st
        _check(rc, name)

    def solve_dense_device(self, T, d_topic_hash, P, RF, d_cur, desired_rf, out_stride, d_out_len, d_out, stream=0,
                           sync=True):
        """Device-pointer form (ints from tensor.data_ptr()); returns KaStatus when sync else None."""
        return self._synced("ka_solve_dense_device", int(T), ctypes.c_void_p(d_topic_hash), int(P), int(RF), ctypes.c_void_p(d_cur),
                            int(desired_rf), int(out_stride), _vp(d_out_len), ctypes.c_void_p(d_out), stream=stream, sync=sync)

    def solve_dense_candidates_device(self, tables, T, d_topic_hash, P, RF, d_cur, desired_rf, out_stride, d_out_len, d_out,
                                      stream=0):
        """ka_solve_dense_candidates_device: the dense device solve against every broker table of `tables` (a list of
        (broker_id, rack_index) numpy pairs), each on a fresh Context; this Solver's own Context is untouched. Candidate k's
        rows are d_out[k] ([K, T, P, out_stride] on the device). Synchronous; returns the K KaStatus."""
        cand_off, broker_id, broker_rack = self._candidate_tables(tables)
        st, sts = _statuses(len(tables))
        self._L.ka_solve_dense_candidates_device(self._h, len(tables), _ptr(cand_off), _ptr(broker_id), _ptr(broker_rack), int(T),
                                                 ctypes.c_void_p(d_topic_hash), int(P), int(RF), ctypes.c_void_p(d_cur),
                                                 int(desired_rf), int(out_stride), _vp(d_out_len), ctypes.c_void_p(d_out),
                                                 _vp(stream), st)
        return sts

    @staticmethod
    def _candidate_tables(tables):
        """(cand_off, broker_id, broker_rack) of a list of (broker_id, rack_index) pairs: the candidate tables of the C ABI."""
        ids = [np.ascontiguousarray(b, dtype=np.int32) for b, _ in tables]
        racks = [np.ascontiguousarray(r, dtype=np.int32) for _, r in tables]
        assert all(len(b) == len(r) for b, r in zip(ids, racks))
        cand_off = np.zeros(len(tables) + 1, dtype=np.int32)
        np.cumsum([len(b) for b in ids], out=cand_off[1:])
        broker_id = np.concatenate(ids) if ids else np.zeros(0, dtype=np.int32)
        broker_rack = np.concatenate(racks) if racks else np.zeros(0, dtype=np.int32)
        return cand_off, broker_id, broker_rack

    def _candidates_call(self, tables, ragged, desired_rf, out_stride):
        """The start both ragged candidate calls share: (Q, the row stride, cand_off, the leading C ABI arguments ctx, K,
        tables, T, problem, desired_rf, stride) for the ragged problem `ragged` against every table of `tables`."""
        r = _ragged(*ragged)
        S = r.stride(desired_rf) if out_stride is None else out_stride
        cand_off, broker_id, broker_rack = self._candidate_tables(tables)
        return r.Q, S, cand_off, (self._h, len(tables), _ptr(cand_off), _ptr(broker_id), _ptr(broker_rack), len(r.topic_hash),
                                  *r.ptrs(), int(desired_rf), int(S))

    def solve_ragged_candidates(self, tables, topic_hash, part_off, part_id, rep_off, cur_broker, desired_rf, out_stride=None):
        """ka_solve_candidates: the ragged solve of solve_ragged against every broker table of `tables` (a list of
        (broker_id, rack_index) numpy pairs), each on a fresh Context; this Solver's own Context is untouched. out_stride
        defaults to max(longest current list, desired_rf, 1). Returns (out [K, ΣP, out_stride], out_len [K, ΣP], [KaStatus] * K);
        the rows of a failed candidate are unspecified."""
        K = len(tables)
        Q, S, _, args = self._candidates_call(tables, (topic_hash, part_off, part_id, rep_off, cur_broker), desired_rf, out_stride)
        out = np.full((K, Q, S), -1, dtype=np.int32)
        out_len = np.zeros((K, Q), dtype=np.int32)
        st, sts = _statuses(K)
        self._L.ka_solve_candidates(*args, _ptr(out_len), _ptr(out), st)
        return out, out_len, sts

    def score_ragged_candidates(self, tables, topic_hash, part_off, part_id, rep_off, cur_broker, desired_rf, out_stride=None,
                                weight=None, rows=False, per_broker=False):
        """ka_score_candidates: solve_ragged_candidates scored on the device. weight: [ΣP] int64 per row (e.g. partition bytes),
        None = 1 per row. Returns (summary, [KaStatus] * K), summary a numpy structured array [K] with the fields of
        ka_move_summary; then, with rows=True, (out [K, ΣP, out_stride], out_len [K, ΣP]) as solve_ragged_candidates returns
        them; then, with per_broker=True, (replicas, leaders, added): one int64 array per table, aligned with its broker ids."""
        K = len(tables)
        Q, S, cand_off, args = self._candidates_call(tables, (topic_hash, part_off, part_id, rep_off, cur_broker), desired_rf,
                                                     out_stride)
        weight = None if weight is None else np.ascontiguousarray(weight, dtype=np.int64)
        summary = np.zeros(K, dtype=MOVE_SUMMARY_DTYPE)
        out = np.full((K, Q, S), -1, dtype=np.int32) if rows else None
        out_len = np.zeros((K, Q), dtype=np.int32) if rows else None
        brk = [np.zeros(int(cand_off[-1]), dtype=np.int64) for _ in range(3)] if per_broker else [None] * 3
        st, sts = _statuses(K)
        self._L.ka_score_candidates(*args, _ptr(weight), _ptr(summary), *[_ptr(a) for a in brk], _ptr(out_len), _ptr(out), st)
        res = (summary, sts)
        if rows:
            res += (out, out_len)
        if per_broker:
            res += tuple([a[cand_off[k]:cand_off[k + 1]] for k in range(K)] for a in brk)
        return res

    @staticmethod
    def marshal_clusters(clusters):
        """The shared layout of ka_solve_clusters from a list of clusters, each (broker_id, rack_index, topic_hash, part_off,
        part_id, rep_off, cur_broker, desired_rf) with its own offsets from 0 (part_id may be None: 0..P-1 per topic). Returns
        (cand_off, broker_id, broker_rack, topic_off, desired_rf, topic_hash, part_off, part_id, rep_off, cur_broker)."""
        cand_off, broker_id, broker_rack = Solver._candidate_tables([(c[0], c[1]) for c in clusters])
        rg = [_ragged(*c[2:7]) for c in clusters]         # a cluster without topics may pass part_off = [0] or []
        topic_off = np.zeros(len(clusters) + 1, dtype=np.int32)
        np.cumsum([len(r.topic_hash) for r in rg], out=topic_off[1:])
        reps = [int(r.rep_off[r.Q]) if r.Q > 0 else 0 for r in rg]
        row0 = np.concatenate([[0], np.cumsum([r.Q for r in rg])]).astype(np.int64)
        rep0 = np.concatenate([[0], np.cumsum(reps)]).astype(np.int64)
        part_off = np.concatenate([[0]] + [r.part_off[1:len(r.topic_hash) + 1] + row0[k] for k, r in enumerate(rg)]).astype(np.int64)
        rep_off = np.concatenate([[0]] + [r.rep_off[1:r.Q + 1] + rep0[k] for k, r in enumerate(rg)]).astype(np.int64)
        none = np.zeros(0, dtype=np.int32)

        def ids(r):   # partition ids of a cluster (ordinals inside each topic when it has none)
            if r.part_id is not None:
                return r.part_id[:r.Q]
            return np.concatenate([none] + [np.arange(int(r.part_off[t + 1] - r.part_off[t]), dtype=np.int32)
                                            for t in range(len(r.topic_hash))])

        part_id = np.concatenate([none] + [ids(r) for r in rg])
        desired_rf = np.array([int(c[7]) for c in clusters], dtype=np.int32)
        return (cand_off, broker_id, broker_rack, topic_off, desired_rf, np.concatenate([none] + [r.topic_hash for r in rg]), part_off,
                part_id, rep_off, np.concatenate([none] + [r.cur_broker[:reps[k]] for k, r in enumerate(rg)]))

    def solve_clusters(self, clusters, out_stride=None):
        """ka_solve_clusters: every cluster of `clusters` solved against its own broker table, each on a fresh Context, in one
        device call; this Solver's own Context is untouched. Each entry is (broker_id, rack_index, topic_hash, part_off, part_id,
        rep_off, cur_broker, desired_rf), e.g. from synth.make_ragged_cluster. out_stride defaults to max(longest current list,
        largest desired_rf, 1) over the fleet. Returns one (out [P_k, out_stride], out_len [P_k], KaStatus) per cluster; the rows
        of a failed cluster are unspecified."""
        K = len(clusters)
        cand_off, broker_id, broker_rack, topic_off, drf, *fleet = self.marshal_clusters(clusters)
        fleet = _ragged(*fleet)
        if out_stride is None:
            out_stride = fleet.stride(int(drf.max()) if K else -1)
        out = np.full((fleet.Q, out_stride), -1, dtype=np.int32)
        out_len = np.zeros(fleet.Q, dtype=np.int32)
        st, sts = _statuses(K)
        self._L.ka_solve_clusters(self._h, K, _ptr(cand_off), _ptr(broker_id), _ptr(broker_rack), _ptr(topic_off), _ptr(drf),
                                  *fleet.ptrs(), int(out_stride), _ptr(out_len), _ptr(out), st)
        rows = fleet.part_off[topic_off]
        return [(out[rows[k]:rows[k + 1]], out_len[rows[k]:rows[k + 1]], sts[k]) for k in range(K)]

    def score_clusters(self, clusters, out_stride=None, weights=None, rows=False, per_broker=False):
        """ka_score_clusters: the fleet of solve_clusters scored on the device, one ka_move_summary per cluster. weights: None
        (1 per row) or one int64 array [P_k] per cluster, in the cluster's row order. Returns one tuple per cluster: (summary
        record, KaStatus); then, with rows=True, (out [P_k, out_stride], out_len [P_k]) as solve_clusters returns them; then,
        with per_broker=True, (replicas, leaders, added), int64 arrays aligned with the cluster's broker ids. A failed cluster
        has a zero summary (max_broker_in_id = -1) and zero per-broker sums; its rows are unspecified."""
        K = len(clusters)
        cand_off, broker_id, broker_rack, topic_off, drf, *fleet = self.marshal_clusters(clusters)
        fleet = _ragged(*fleet)
        if out_stride is None:
            out_stride = fleet.stride(int(drf.max()) if K else -1)
        weight = None
        if weights is not None:
            assert len(weights) == K
            weight = np.concatenate([np.zeros(0, dtype=np.int64)] + [np.asarray(w, dtype=np.int64) for w in weights])
            assert len(weight) == fleet.Q
        summary = np.zeros(K, dtype=MOVE_SUMMARY_DTYPE)
        out = np.full((fleet.Q, out_stride), -1, dtype=np.int32) if rows else None
        out_len = np.zeros(fleet.Q, dtype=np.int32) if rows else None
        brk = [np.zeros(int(cand_off[-1]), dtype=np.int64) for _ in range(3)] if per_broker else [None] * 3
        st, sts = _statuses(K)
        self._L.ka_score_clusters(self._h, K, _ptr(cand_off), _ptr(broker_id), _ptr(broker_rack), _ptr(topic_off), _ptr(drf),
                                  *fleet.ptrs(), int(out_stride), _ptr(weight), _ptr(summary), *[_ptr(a) for a in brk], _ptr(out_len),
                                  _ptr(out), st)
        row0 = fleet.part_off[topic_off]
        res = []
        for k in range(K):
            r = (summary[k], sts[k])
            if rows:
                r += (out[row0[k]:row0[k + 1]], out_len[row0[k]:row0[k + 1]])
            if per_broker:
                r += tuple(a[cand_off[k]:cand_off[k + 1]] for a in brk)
            res.append(r)
        return res

    def solve_clusters_json(self, clusters, topic_names, json_buf=None):
        """ka_solve_clusters_json: the fleet of solve_clusters, every cluster's reassignment JSON built on the device.
        topic_names: one list of names per cluster. json_buf: optional writable uint8 numpy array (pinned for full PCIe speed);
        by default one of the documented sufficient size. Returns one (bytes-like view of the cluster's text, KaStatus) per
        cluster; the text of a failed cluster is empty."""
        K = len(clusters)
        cand_off, broker_id, broker_rack, topic_off, drf, *fleet = self.marshal_clusters(clusters)
        fleet = _ragged(*fleet)
        names, name_off = self.marshal_names([n for names_k in topic_names for n in names_k])
        assert len(name_off) == len(fleet.topic_hash) + 1
        if json_buf is None:    # one document per cluster, each sized as solve_ragged_json sizes it
            name_len = np.diff(name_off)
            cap = 0
            for k, c in enumerate(clusters):
                r = _ragged(*c[2:7])
                cap += _json_size(r.Q, r.name_bytes(name_len[topic_off[k]:topic_off[k + 1]]), r.stride(int(drf[k])))
            json_buf = np.empty(max(cap, 1), dtype=np.uint8)
        json_off = np.zeros(K + 1, dtype=np.int64)
        st, sts = _statuses(K)
        self._L.ka_solve_clusters_json(self._h, K, _ptr(cand_off), _ptr(broker_id), _ptr(broker_rack), _ptr(topic_off), _ptr(drf),
                                       *fleet.ptrs(), _ptr(names), _ptr(name_off), _ptr(json_buf), int(json_buf.size), _ptr(json_off),
                                       st)
        return [(json_buf[json_off[k]:json_off[k + 1]], sts[k]) for k in range(K)]

    # The most summaries plan_waves asks for in its first call (40 bytes each): min(Q, this) covers W (never above Q) in one call
    # on any cluster of up to 64 k rows and, on larger ones, every plan of up to 64 k waves.
    WAVE_SUMMARY_CAP = 1 << 16

    def plan_waves(self, rep_off, cur_broker, out, out_len, max_broker_in, weight=None, max_broker_out=None, send_brokers=None):
        """ka_plan_waves: the proposed lists out [Q, stride] / out_len [Q] (e.g. solve_ragged's rows) against the current lists
        cur_broker[rep_off[g] .. rep_off[g + 1]), cut into waves in which no broker of this Solver's table receives more than
        max_broker_in (weight: [Q] int64 per row, None = 1 per row). Returns (wave [Q] int32, 0 for an unchanged row; summary, a
        numpy structured array [W] with the fields of ka_wave_summary; KaStatus). On an error wave and summary are empty. A plan
        of more than min(Q, WAVE_SUMMARY_CAP) waves takes a second call for the rest of the summaries. The waves follow this
        Solver's wave rule (set_wave_rule), as do those of every wave document call.
        max_broker_out: ka_plan_waves_send instead, which also caps what each row's leader (the first broker of its current
        list) sends per wave; send_brokers (required then: the ascending send table, e.g. every broker of the cluster before an
        exclusion) holds every such leader. The summary then has the fields of WAVE_SEND_SUMMARY_DTYPE."""
        out = np.ascontiguousarray(out, dtype=np.int32)
        Q = len(out)
        stride = out.shape[1] if out.ndim == 2 else 1
        out_len = np.ascontiguousarray(out_len, dtype=np.int32)
        rep_off = np.ascontiguousarray(rep_off, dtype=np.int64)
        cur_broker = np.ascontiguousarray(cur_broker, dtype=np.int32)
        weight = None if weight is None else np.ascontiguousarray(weight, dtype=np.int64)
        assert out_len.shape == (Q,) and rep_off.shape == (Q + 1,) and (weight is None or weight.shape == (Q,))
        send = _send_part(max_broker_out, send_brokers)
        wave = np.zeros(Q, dtype=np.int32)
        n_waves = ctypes.c_int32(0)
        st = KaStatus()
        cap = max(1, min(Q, self.WAVE_SUMMARY_CAP))
        while True:
            summary = np.zeros(cap, dtype=WAVE_SUMMARY_DTYPE)
            rows = (self._h, Q, _ptr(rep_off), _ptr(cur_broker), int(stride), _ptr(out_len), _ptr(out), _ptr(weight), int(max_broker_in))
            if send is None:
                self._L.ka_plan_waves(*rows, _ptr(wave), ctypes.byref(n_waves), _ptr(summary), cap, ctypes.byref(st))
            else:
                send_summary = np.zeros((cap, len(_SEND_FIELDS)), dtype=np.int64)
                self._L.ka_plan_waves_send(*rows, send[0], _ptr(send[1]), send[2], _ptr(wave), ctypes.byref(n_waves), _ptr(summary),
                                           _ptr(send_summary), cap, ctypes.byref(st))
            if st.code != 0:
                dtype = WAVE_SUMMARY_DTYPE if send is None else WAVE_SEND_SUMMARY_DTYPE
                return np.zeros(0, dtype=np.int32), np.zeros(0, dtype=dtype), st
            if n_waves.value <= cap:
                W = n_waves.value
                return wave, summary[:W] if send is None else _with_send(summary[:W], send_summary[:W]), st
            cap = n_waves.value

    def plan_waves_json(self, topic_names, part_off, part_id, rep_off, cur_broker, out, out_len, max_broker_in, weight=None,
                        json_buf=None, max_broker_out=None, send_brokers=None):
        """ka_plan_waves_json: plan_waves over the rows of the ragged layout part_off / part_id (None = 0..P-1 per topic), and
        every wave's reassignment JSON built on the device. json_buf: optional writable uint8 numpy array (pinned for full PCIe
        speed); by default one of the documented sufficient size. Returns (docs, wave, summary, KaStatus): docs a list of W
        bytes-like views of the buffer, docs[v] the document of wave v + 1; wave and summary as plan_waves returns them. On an
        error docs, wave and summary are empty. max_broker_out / send_brokers: ka_plan_waves_send_json, as in plan_waves."""
        docs, _, _, wave, summary, st = self._wave_documents(topic_names, part_off, part_id, rep_off, cur_broker, out, out_len,
                                                             max_broker_in, weight, json_buf, max_broker_out, send_brokers, None)
        return docs, wave, summary, st

    def plan_wave_parts_json(self, topic_names, part_off, part_id, rep_off, cur_broker, out, out_len, max_broker_in, max_doc_bytes,
                             weight=None, json_buf=None, max_broker_out=None, send_brokers=None):
        """ka_plan_waves_json_parts: plan_waves_json with every wave cut on the device into parts whose documents are at most
        max_doc_bytes bytes (1048575 fits ZooKeeper's default jute.maxbuffer). Returns (parts, part_wave, wave, summary,
        KaStatus): parts a list of D bytes-like views of the buffer in (wave, place in the wave) order, part_wave [D] int32 the
        wave (1..W) of each; the other arguments and results as plan_waves_json takes and returns them. On an error parts,
        part_wave, wave and summary are empty. With max_broker_in >= the sum of the weights every changed row is in wave 1: the
        whole reassignment under the limit."""
        parts, _, part_wave, wave, summary, st = self._wave_documents(topic_names, part_off, part_id, rep_off, cur_broker, out,
                                                                      out_len, max_broker_in, weight, json_buf, max_broker_out,
                                                                      send_brokers, int(max_doc_bytes))
        return parts, part_wave, wave, summary, st

    def plan_wave_parts_rollback_json(self, topic_names, part_off, part_id, rep_off, cur_broker, out, out_len, max_broker_in,
                                      max_doc_bytes, weight=None, json_buf=None, back_buf=None, max_broker_out=None, send_brokers=None):
        """ka_plan_waves_json_parts_rollback: plan_wave_parts_json with every part's rollback document, the document that puts
        exactly that part's partitions back on their current lists (cur_broker). A row joins a part only while both documents
        stay <= max_doc_bytes. back_buf: optional writable uint8 numpy array for the rollback text; by default one of the
        documented sufficient size. Returns (parts, rollback, part_wave, wave, summary, KaStatus): rollback[d] a bytes-like view
        of back_buf, the rollback document of parts[d]; the rest as plan_wave_parts_json returns them. On an error every result
        is empty."""
        return self._wave_documents(topic_names, part_off, part_id, rep_off, cur_broker, out, out_len, max_broker_in, weight,
                                    json_buf, max_broker_out, send_brokers, int(max_doc_bytes), True, back_buf)

    def _wave_documents(self, topic_names, part_off, part_id, rep_off, cur_broker, out, out_len, max_broker_in, weight, json_buf,
                        max_broker_out, send_brokers, max_doc_bytes, rollback=False, back_buf=None):
        """One call of the six wave document entry points: with max_doc_bytes None ka_plan_waves(_send)_json, else their
        _parts forms, and with rollback their _parts_rollback forms. Returns (docs, backs, doc_wave, wave, summary, KaStatus);
        doc_wave is 1..W without a limit, backs the rollback documents (None without rollback)."""
        out = np.ascontiguousarray(out, dtype=np.int32)
        Q = len(out)
        stride = out.shape[1] if out.ndim == 2 else 1
        out_len = np.ascontiguousarray(out_len, dtype=np.int32)
        r = _ragged(np.zeros(len(topic_names), dtype=np.int32), part_off, part_id, rep_off, cur_broker)
        weight = None if weight is None else np.ascontiguousarray(weight, dtype=np.int64)
        assert r.Q == Q and out_len.shape == (Q,) and r.rep_off.shape == (Q + 1,) and (weight is None or weight.shape == (Q,))
        names, name_off = self.marshal_names(topic_names)
        if json_buf is None:
            json_buf = np.empty(max(_wave_json_size(Q, r.name_bytes(np.diff(name_off)), stride), 1), dtype=np.uint8)
        if rollback and back_buf is None:   # per row 79 + its topic's name, 12 per current broker
            back_buf = np.empty(max(_wave_json_size(Q, r.name_bytes(np.diff(name_off)), 0) + 12 * len(r.cur_broker), 1), dtype=np.uint8)
        doc_off = np.zeros(Q + 1, dtype=np.int64)
        wave = np.zeros(Q, dtype=np.int32)
        n_waves = ctypes.c_int32(0)
        st = KaStatus()
        cap = max(1, Q)   # W never exceeds Q: one call, so the text is built once
        summary = np.zeros(cap, dtype=WAVE_SUMMARY_DTYPE)
        send = _send_part(max_broker_out, send_brokers)
        rows = (self._h, len(topic_names), _ptr(r.part_off), _ptr(r.part_id), _ptr(r.rep_off), _ptr(r.cur_broker), int(stride),
                _ptr(out_len), _ptr(out), _ptr(weight), int(max_broker_in))
        if max_doc_bytes is None:
            text = (_ptr(names), _ptr(name_off), _ptr(json_buf), int(json_buf.size), _ptr(doc_off), _ptr(wave), ctypes.byref(n_waves),
                    _ptr(summary))
            entry = self._L.ka_plan_waves_json if send is None else self._L.ka_plan_waves_send_json
        else:
            doc_wave = np.zeros(Q, dtype=np.int32)
            n_docs = ctypes.c_int32(0)
            back = ()
            if rollback:
                back_off = np.zeros(Q + 1, dtype=np.int64)
                back = (_ptr(back_buf), int(back_buf.size), _ptr(back_off))
            text = (_ptr(names), _ptr(name_off), _ptr(json_buf), int(json_buf.size), max_doc_bytes, _ptr(doc_off), _ptr(doc_wave),
                    ctypes.byref(n_docs), *back, _ptr(wave), ctypes.byref(n_waves), _ptr(summary))
            if rollback:
                entry = self._L.ka_plan_waves_json_parts_rollback if send is None else self._L.ka_plan_waves_send_json_parts_rollback
            else:
                entry = self._L.ka_plan_waves_json_parts if send is None else self._L.ka_plan_waves_send_json_parts
        if send is None:
            entry(*rows, *text, cap, ctypes.byref(st))
        else:
            send_summary = np.zeros((cap, len(_SEND_FIELDS)), dtype=np.int64)
            entry(*rows, send[0], _ptr(send[1]), send[2], *text, _ptr(send_summary), cap, ctypes.byref(st))
        if st.code != 0:
            dtype = WAVE_SUMMARY_DTYPE if send is None else WAVE_SEND_SUMMARY_DTYPE
            return [], [] if rollback else None, np.zeros(0, dtype=np.int32), np.zeros(0, dtype=np.int32), np.zeros(0, dtype=dtype), st
        W = n_waves.value
        summary = summary[:W] if send is None else _with_send(summary[:W], send_summary[:W])
        D, doc_wave = (W, np.arange(1, W + 1, dtype=np.int32)) if max_doc_bytes is None else (n_docs.value, doc_wave[:n_docs.value])
        backs = [back_buf[back_off[d]:back_off[d + 1]] for d in range(D)] if rollback else None
        return [json_buf[doc_off[d]:doc_off[d + 1]] for d in range(D)], backs, doc_wave, wave, summary, st

    def broker_usage(self, rep_off, cur_broker, out, out_len, wave, use_brokers, weight=None, base=None, capacity=None):
        """ka_wave_broker_usage: what every broker of use_brokers (strictly ascending ids, e.g. every broker of the cluster before
        an exclusion) holds across the wave plan `wave` [Q] (plan_waves' wave unchanged, or any waves >= 0) of the proposed lists
        out [Q, stride] / out_len [Q] against the current lists cur_broker[rep_off[g] .. rep_off[g + 1]). weight: [Q] int64 per
        row, None = 1 per row; base, capacity: int64 per broker of use_brokers, None = 0 / no capacity. Returns (usage, a numpy
        structured array [len(use_brokers)] with the fields of ka_broker_usage, aligned with use_brokers; W; KaStatus). On an
        error usage is empty and W = 0."""
        out = np.ascontiguousarray(out, dtype=np.int32)
        Q = len(out)
        stride = out.shape[1] if out.ndim == 2 else 1
        out_len = np.ascontiguousarray(out_len, dtype=np.int32)
        rep_off = np.ascontiguousarray(rep_off, dtype=np.int64)
        cur_broker = np.ascontiguousarray(cur_broker, dtype=np.int32)
        wave = np.ascontiguousarray(wave, dtype=np.int32)
        use_id = np.ascontiguousarray(use_brokers, dtype=np.int32)
        n = len(use_id)
        weight, base, capacity = (None if a is None else np.ascontiguousarray(a, dtype=np.int64) for a in (weight, base, capacity))
        assert out_len.shape == wave.shape == (Q,) and rep_off.shape == (Q + 1,) and (weight is None or weight.shape == (Q,))
        assert (base is None or base.shape == (n,)) and (capacity is None or capacity.shape == (n,))
        usage = np.zeros(n, dtype=BROKER_USAGE_DTYPE)
        n_waves = ctypes.c_int32(0)
        st = KaStatus()
        self._L.ka_wave_broker_usage(self._h, Q, _ptr(rep_off), _ptr(cur_broker), int(stride), _ptr(out_len), _ptr(out), _ptr(weight),
                                     _ptr(wave), n, _ptr(use_id), _ptr(base), _ptr(capacity), _ptr(usage), ctypes.byref(n_waves),
                                     ctypes.byref(st))
        if st.code != 0:
            return np.zeros(0, dtype=BROKER_USAGE_DTYPE), 0, st
        return usage, n_waves.value, st

    def stage_dense_device(self, T, d_topic_hash, P, RF, d_cur, desired_rf, out_stride, stream=0):
        """Context-free stage (KAS:65-200) of a topic block — shards across GPUs."""
        _check(self._L.ka_stage_dense_device(self._h, int(T), ctypes.c_void_p(d_topic_hash), int(P), int(RF), ctypes.c_void_p(d_cur),
                                             int(desired_rf), int(out_stride), _vp(stream)), "ka_stage_dense_device")

    def order_device(self, d_out_len, d_out, stream=0, sync=True):
        """Leader-order stage (KAS:202-239) of the staged block against this Context's counters."""
        return self._synced("ka_order_device", _vp(d_out_len), ctypes.c_void_p(d_out), stream=stream, sync=sync)

    def staged_slot_chains(self):
        """2 when the staged block is ordered by per-slot chains (rows <= 3), else 0."""
        return int(self._L.ka_staged_slot_chains(self._h))

    def order_slot_device(self, slot, stream=0):
        """Slot-0 / slot-1 leader-order chain of the staged block (reads and bumps only counter[.][slot])."""
        _check(self._L.ka_order_slot_device(self._h, int(slot), _vp(stream)), "ka_order_slot_device")

    def emit_device(self, d_out_len, d_out, stream=0, sync=True):
        return self._synced("ka_emit_device", _vp(d_out_len), ctypes.c_void_p(d_out), stream=stream, sync=sync)

    def export_counter_slot_device(self, slot, d_ptr, stream=0):
        _check(self._L.ka_ctx_export_counter_slot_device(self._h, int(slot), ctypes.c_void_p(d_ptr), _vp(stream)))

    def import_counter_slot_device(self, slot, d_ptr, stream=0):
        _check(self._L.ka_ctx_import_counter_slot_device(self._h, int(slot), ctypes.c_void_p(d_ptr), _vp(stream)))

    def last_status(self):
        st = KaStatus()
        self._L.ka_last_status(self._h, ctypes.byref(st))
        return st

    def export_counters_device(self, d_ptr, stream=0):
        _check(self._L.ka_ctx_export_counters_device(self._h, ctypes.c_void_p(d_ptr), _vp(stream)))

    def import_counters_device(self, d_ptr, stream=0):
        _check(self._L.ka_ctx_import_counters_device(self._h, ctypes.c_void_p(d_ptr), _vp(stream)))

    def solve_cluster(self, cluster, check=True):
        """The KAG:172-184 loop for a synth.Cluster: all topics in order through this Context."""
        self.set_brokers(cluster.broker_id, cluster.rack_index)
        return self.solve_dense(cluster.topic_hash, cluster.cur, cluster.desired_rf, check=check,
                                topic_names=cluster.topic_names)


class KafkaTopicAssigner:
    """Mirror of siftscience.kafka.tools.KafkaTopicAssigner (KafkaTopicAssigner.java:18-72).

    One instance owns one Context, exactly like the reference (KTA:19-23): leader-preference counters
    persist across generate_assignment calls on the same instance.
    """

    def __init__(self, device=0):
        self._solver = Solver(device)
        self._brokers_key = None

    def generate_assignment(self, topic, current_assignment, brokers, rack_assignment, desired_replication_factor):
        """generateAssignment(topic, currentAssignment, brokers, rackAssignment, desiredReplicationFactor).

        current_assignment: {partition: [broker ids, leader first]}; brokers: set of ids;
        rack_assignment: {broker id: rack string}; returns {partition: [broker ids, leader first]}
        (ascending partition order, like the reference's TreeMap).
        """
        if current_assignment is None:
            raise TypeError("currentAssignment is null")  # NullPointerException at KTA:51
        key = (tuple(sorted(set(int(b) for b in brokers))), tuple(sorted((int(k), v) for k, v in rack_assignment.items())))
        if key != self._brokers_key:
            self._solver.set_brokers_with_racks(brokers, rack_assignment)
            self._brokers_key = key
        parts = sorted(int(p) for p in current_assignment)
        lists = [list(current_assignment[p]) for p in parts]
        part_off = np.array([0, len(parts)], dtype=np.int64)
        rep_off = np.zeros(len(parts) + 1, dtype=np.int64)
        if parts:
            np.cumsum([len(l) for l in lists], out=rep_off[1:])
        cur = np.array([b for l in lists for b in l], dtype=np.int32)
        r = _ragged([java_string_hash(topic)], part_off, parts, rep_off, cur)
        out, out_len, _ = self._solver.solve_ragged(*r[:5], desired_replication_factor, r.stride(desired_replication_factor),
                                                    check=True, topic_names=[topic])
        return {p: [int(x) for x in out[i, :out_len[i]]] for i, p in enumerate(parts)}
