"""Host-side mirror of the reference's interface for the hot path, over the C ABI (include/kassign.h).

  KafkaTopicAssigner.generate_assignment(...)  <->  KafkaTopicAssigner.generateAssignment
                                                    (reference KafkaTopicAssigner.java:42-72)
  Solver.solve_cluster(...)                    <->  the per-topic loop with ONE shared assigner
                                                    (reference KafkaAssignmentGenerator.java:172-184)

Same names, argument meaning and error behaviour (message texts of KTA:58-60, 65-66, 67-69 and
KAS:183-184). All compute happens in libkassign.so's CUDA kernels; nothing here falls back to a CPU
solver — if the library or a GPU is missing, construction raises.
"""
import ctypes

import numpy as np

from . import _native
from ._native import KaMoveSummary, KaStatus

# numpy view of ka_move_summary (KaMoveSummary): one record per candidate
MOVE_SUMMARY_DTYPE = np.dtype([(name, np.int64) for name, _ in KaMoveSummary._fields_])


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
    return _native.load().ka_java_string_hash(s.encode("utf-8"))


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _ragged_arrays(topic_hash, part_off, part_id, rep_off, cur_broker):
    """The ragged layout as the C ABI takes it: (topic_hash, part_off, part_id, rep_off, cur_broker) as contiguous arrays of
    its element types; part_id may be None."""
    return (np.ascontiguousarray(topic_hash, dtype=np.int32), np.ascontiguousarray(part_off, dtype=np.int64),
            None if part_id is None else np.ascontiguousarray(part_id, dtype=np.int32),
            np.ascontiguousarray(rep_off, dtype=np.int64), np.ascontiguousarray(cur_broker, dtype=np.int32))


def _default_stride(rep_off, desired_rf):
    """The row stride of a ragged solve when the caller gives none: max(longest current list, desired_rf, 1)."""
    sizes = np.diff(rep_off)
    return max(int(sizes.max()) if len(sizes) else 0, desired_rf, 1)


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
        rc = self._L.ka_ctx_reset(self._h)
        if rc:
            raise KassignError(rc)

    def set_brokers(self, broker_id, rack_index):
        b = np.ascontiguousarray(broker_id, dtype=np.int32)
        r = np.ascontiguousarray(rack_index, dtype=np.int32)
        rc = self._L.ka_ctx_set_brokers(self._h, len(b), _ptr(b), _ptr(r))
        if rc:
            raise KassignError(rc, "ka_ctx_set_brokers")
        self.N = len(b)
        self.broker_id = b

    def set_brokers_with_racks(self, brokers, rack_assignment):
        """brokers: iterable of ids (any order); rack_assignment: {id: rack string} (may lack entries)."""
        b = np.array(sorted(set(int(x) for x in brokers)), dtype=np.int32)
        names = [rack_assignment.get(int(x)) for x in b]
        arr = (ctypes.c_char_p * len(b))(*[(n.encode("utf-8") if n is not None else None) for n in names])
        racks = np.zeros(len(b), dtype=np.int32)
        rc = self._L.ka_rack_indices(len(b), _ptr(b), ctypes.cast(arr, ctypes.c_void_p), _ptr(racks))
        if rc:
            raise KassignError(rc, "ka_rack_indices")
        self.set_brokers(b, racks)
        return b

    def counters(self):
        slots = self._L.ka_ctx_counter_slots(self._h)
        out = np.zeros((self.N, slots), dtype=np.int32)
        rc = self._L.ka_ctx_get_counters(self._h, _ptr(out))
        if rc:
            raise KassignError(rc)
        return out

    def set_counters(self, ctr):
        c = np.ascontiguousarray(ctr, dtype=np.int32)
        assert c.shape == (self.N, self._L.ka_ctx_counter_slots(self._h))
        rc = self._L.ka_ctx_set_counters(self._h, _ptr(c))
        if rc:
            raise KassignError(rc)

    def set_timing(self, on=True):
        self._L.ka_ctx_set_timing(self._h, 1 if on else 0)

    def last_timing(self):
        ms = np.zeros(8, dtype=np.float32)
        self._L.ka_ctx_last_timing(self._h, _ptr(ms))
        return dict(sticky_spread_ms=float(ms[0]), level_tables_ms=float(ms[1]), leader_order_ms=float(ms[2]),
                    h2d_ms=float(ms[3]), d2h_ms=float(ms[4]), total_ms=float(ms[5]), slot1_emit_ms=float(ms[6]), chains_wall_ms=float(ms[7]))

    def set_topic_base(self, topic_base):
        """Topic-sharded runs: index of this rank's first topic in the whole run (status reporting)."""
        rc = self._L.ka_ctx_set_topic_base(self._h, int(topic_base))
        if rc:
            raise KassignError(rc)

    def launch_count(self):
        return int(self._L.ka_ctx_launch_count(self._h))

    def last_order_plan(self):
        """The leader-order plan of the last solve call (ka_ctx_last_order_plan): (rec_kind, levels, chain threads, ring_log2,
        gctr, loop shape [0 general, 1 warp1, 2 single, 3 full], chain launches, candidates K)."""
        plan = np.zeros(8, dtype=np.int32)
        rc = self._L.ka_ctx_last_order_plan(self._h, _ptr(plan))
        if rc:
            raise KassignError(rc, "ka_ctx_last_order_plan")
        return tuple(int(x) for x in plan)

    def last_stage_plan(self):
        """The sticky/spread plan of the last solve call (ka_ctx_last_stage_plan): (load bytes, levels, SM, candidates K,
        warps per CTA, grid.x, lookup-mode mask [1 shared LUT, 2 global LUT, 4 binary search], kernel A launches)."""
        plan = np.zeros(8, dtype=np.int32)
        rc = self._L.ka_ctx_last_stage_plan(self._h, _ptr(plan))
        if rc:
            raise KassignError(rc, "ka_ctx_last_stage_plan")
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
            out_stride = max(RF, desired_rf if desired_rf >= 0 else RF, 1)
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
        S = max(RF, desired_rf, 1)
        cap = 64 + T * P * (50 + 12 * S) + int(P * name_off[-1])
        if json_buf is None:
            json_buf = np.empty(cap, dtype=np.uint8)
        nbytes = ctypes.c_int64(0)
        st = KaStatus()
        self._L.ka_solve_dense_json(self._h, T, _ptr(th), P, RF, _ptr(cur), int(desired_rf), _ptr(names), _ptr(name_off),
                                    _ptr(json_buf), int(json_buf.size), ctypes.byref(nbytes), ctypes.byref(st))
        if check:
            raise_for_status(st, topic_names)
        return json_buf[:nbytes.value], st

    def solve_ragged(self, topic_hash, part_off, part_id, rep_off, cur_broker, desired_rf, out_stride, check=True,
                     topic_names=None):
        th, part_off, part_id, rep_off, cur_broker = _ragged_arrays(topic_hash, part_off, part_id, rep_off, cur_broker)
        Q = int(part_off[-1]) if len(part_off) else 0
        out = np.full((Q, out_stride), -1, dtype=np.int32)
        out_len = np.zeros(Q, dtype=np.int32)
        st = KaStatus()
        self._L.ka_solve(self._h, len(th), _ptr(th), _ptr(part_off), _ptr(part_id), _ptr(rep_off), _ptr(cur_broker),
                         int(desired_rf), int(out_stride), _ptr(out_len), _ptr(out), ctypes.byref(st))
        if check:
            raise_for_status(st, topic_names)
        return out, out_len, st

    def solve_ragged_json(self, topic_names, topic_hash, part_off, part_id, rep_off, cur_broker, desired_rf, json_buf=None,
                          check=True):
        """ka_solve_json: the ragged solve of solve_ragged + the reassignment JSON built on the device (KAG:169-186);
        returns (bytes-like view of the text, status). json_buf: optional writable uint8 numpy array (pinned for full
        PCIe speed); by default one of the documented sufficient size."""
        th, part_off, part_id, rep_off, cur_broker = _ragged_arrays(topic_hash, part_off, part_id, rep_off, cur_broker)
        names, name_off = self.marshal_names(topic_names)
        if json_buf is None:
            S = _default_stride(rep_off, desired_rf)
            rows = np.diff(part_off)
            json_buf = np.empty(64 + int(part_off[-1]) * (50 + 12 * S) + int(np.dot(rows, np.diff(name_off))), dtype=np.uint8)
        nbytes = ctypes.c_int64(0)
        st = KaStatus()
        self._L.ka_solve_json(self._h, len(th), _ptr(th), _ptr(part_off), _ptr(part_id), _ptr(rep_off), _ptr(cur_broker),
                              int(desired_rf), _ptr(names), _ptr(name_off), _ptr(json_buf), int(json_buf.size),
                              ctypes.byref(nbytes), ctypes.byref(st))
        if check:
            raise_for_status(st, topic_names)
        return json_buf[:nbytes.value], st

    def solve_dense_device(self, T, d_topic_hash, P, RF, d_cur, desired_rf, out_stride, d_out_len, d_out, stream=0,
                           sync=True):
        """Device-pointer form (ints from tensor.data_ptr()); returns KaStatus when sync else None."""
        st = KaStatus()
        rc = self._L.ka_solve_dense_device(self._h, int(T), ctypes.c_void_p(d_topic_hash), int(P), int(RF),
                                           ctypes.c_void_p(d_cur), int(desired_rf), int(out_stride),
                                           ctypes.c_void_p(d_out_len) if d_out_len else None, ctypes.c_void_p(d_out),
                                           ctypes.c_void_p(stream) if stream else None,
                                           ctypes.byref(st) if sync else None)
        if not sync:
            if rc:
                raise KassignError(rc, "ka_solve_dense_device")
            return None
        return st

    def solve_dense_candidates_device(self, tables, T, d_topic_hash, P, RF, d_cur, desired_rf, out_stride, d_out_len, d_out,
                                      stream=0):
        """ka_solve_dense_candidates_device: the dense device solve against every broker table of `tables` (a list of
        (broker_id, rack_index) numpy pairs), each on a fresh Context; this Solver's own Context is untouched. Candidate k's
        rows are d_out[k] ([K, T, P, out_stride] on the device). Synchronous; returns the K KaStatus."""
        cand_off, broker_id, broker_rack = self._candidate_tables(tables)
        st = (KaStatus * max(len(tables), 1))()
        self._L.ka_solve_dense_candidates_device(self._h, len(tables), _ptr(cand_off), _ptr(broker_id), _ptr(broker_rack), int(T),
                                                 ctypes.c_void_p(d_topic_hash), int(P), int(RF), ctypes.c_void_p(d_cur),
                                                 int(desired_rf), int(out_stride),
                                                 ctypes.c_void_p(d_out_len) if d_out_len else None, ctypes.c_void_p(d_out),
                                                 ctypes.c_void_p(stream) if stream else None, st)
        return [st[k] for k in range(len(tables))]

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

    def solve_ragged_candidates(self, tables, topic_hash, part_off, part_id, rep_off, cur_broker, desired_rf, out_stride=None):
        """ka_solve_candidates: the ragged solve of solve_ragged against every broker table of `tables` (a list of
        (broker_id, rack_index) numpy pairs), each on a fresh Context; this Solver's own Context is untouched. out_stride
        defaults to max(longest current list, desired_rf, 1). Returns (out [K, ΣP, out_stride], out_len [K, ΣP], [KaStatus] * K);
        the rows of a failed candidate are unspecified."""
        th, part_off, part_id, rep_off, cur_broker = _ragged_arrays(topic_hash, part_off, part_id, rep_off, cur_broker)
        if out_stride is None:
            out_stride = _default_stride(rep_off, desired_rf)
        cand_off, broker_id, broker_rack = self._candidate_tables(tables)
        K = len(tables)
        Q = int(part_off[-1]) if len(part_off) else 0
        out = np.full((K, Q, out_stride), -1, dtype=np.int32)
        out_len = np.zeros((K, Q), dtype=np.int32)
        st = (KaStatus * max(K, 1))()
        self._L.ka_solve_candidates(self._h, K, _ptr(cand_off), _ptr(broker_id), _ptr(broker_rack), len(th), _ptr(th),
                                    _ptr(part_off), _ptr(part_id), _ptr(rep_off), _ptr(cur_broker), int(desired_rf),
                                    int(out_stride), _ptr(out_len), _ptr(out), st)
        return out, out_len, [st[k] for k in range(K)]

    def score_ragged_candidates(self, tables, topic_hash, part_off, part_id, rep_off, cur_broker, desired_rf, out_stride=None,
                                weight=None, rows=False, per_broker=False):
        """ka_score_candidates: solve_ragged_candidates scored on the device. weight: [ΣP] int64 per row (e.g. partition bytes),
        None = 1 per row. Returns (summary, [KaStatus] * K), summary a numpy structured array [K] with the fields of
        ka_move_summary; then, with rows=True, (out [K, ΣP, out_stride], out_len [K, ΣP]) as solve_ragged_candidates returns
        them; then, with per_broker=True, (replicas, leaders, added): one int64 array per table, aligned with its broker ids."""
        th, part_off, part_id, rep_off, cur_broker = _ragged_arrays(topic_hash, part_off, part_id, rep_off, cur_broker)
        weight = None if weight is None else np.ascontiguousarray(weight, dtype=np.int64)
        if out_stride is None:
            out_stride = _default_stride(rep_off, desired_rf)
        cand_off, broker_id, broker_rack = self._candidate_tables(tables)
        K = len(tables)
        Q = int(part_off[-1]) if len(part_off) else 0
        summary = np.zeros(K, dtype=MOVE_SUMMARY_DTYPE)
        out = np.full((K, Q, out_stride), -1, dtype=np.int32) if rows else None
        out_len = np.zeros((K, Q), dtype=np.int32) if rows else None
        brk = [np.zeros(int(cand_off[-1]), dtype=np.int64) for _ in range(3)] if per_broker else [None] * 3
        st = (KaStatus * max(K, 1))()
        self._L.ka_score_candidates(self._h, K, _ptr(cand_off), _ptr(broker_id), _ptr(broker_rack), len(th), _ptr(th),
                                    _ptr(part_off), _ptr(part_id), _ptr(rep_off), _ptr(cur_broker), int(desired_rf),
                                    int(out_stride), _ptr(weight), _ptr(summary), *[_ptr(a) for a in brk], _ptr(out_len),
                                    _ptr(out), st)
        res = (summary, [st[k] for k in range(K)])
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
        th = [np.ascontiguousarray(c[2], dtype=np.int32) for c in clusters]
        po = [np.ascontiguousarray(c[3], dtype=np.int64) for c in clusters]
        ro = [np.ascontiguousarray(c[5], dtype=np.int64) for c in clusters]
        cur = [np.ascontiguousarray(c[6], dtype=np.int32) for c in clusters]
        topic_off = np.zeros(len(clusters) + 1, dtype=np.int32)
        np.cumsum([len(h) for h in th], out=topic_off[1:])
        rows = [int(p[-1]) if len(p) > 1 else 0 for p in po]          # a cluster without topics may pass part_off = [0] or []
        reps = [int(r[rows[k]]) if rows[k] > 0 else 0 for k, r in enumerate(ro)]
        row0 = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
        rep0 = np.concatenate([[0], np.cumsum(reps)]).astype(np.int64)
        part_off = np.concatenate([[0]] + [p[1:len(h) + 1] + row0[k] for k, (p, h) in enumerate(zip(po, th))]).astype(np.int64)
        rep_off = np.concatenate([[0]] + [r[1:rows[k] + 1] + rep0[k] for k, r in enumerate(ro)]).astype(np.int64)
        none = np.zeros(0, dtype=np.int32)

        def ids(k):   # partition ids of cluster k (ordinals inside each topic when it has none)
            if clusters[k][4] is not None:
                return np.ascontiguousarray(clusters[k][4], dtype=np.int32)[:rows[k]]
            return np.concatenate([none] + [np.arange(int(po[k][t + 1] - po[k][t]), dtype=np.int32) for t in range(len(th[k]))])

        part_id = np.concatenate([none] + [ids(k) for k in range(len(clusters))])
        desired_rf = np.array([int(c[7]) for c in clusters], dtype=np.int32)
        return (cand_off, broker_id, broker_rack, topic_off, desired_rf, np.concatenate([none] + th), part_off, part_id, rep_off,
                np.concatenate([none] + [c[:reps[k]] for k, c in enumerate(cur)]))

    def solve_clusters(self, clusters, out_stride=None):
        """ka_solve_clusters: every cluster of `clusters` solved against its own broker table, each on a fresh Context, in one
        device call; this Solver's own Context is untouched. Each entry is (broker_id, rack_index, topic_hash, part_off, part_id,
        rep_off, cur_broker, desired_rf), e.g. from synth.make_ragged_cluster. out_stride defaults to max(longest current list,
        largest desired_rf, 1) over the fleet. Returns one (out [P_k, out_stride], out_len [P_k], KaStatus) per cluster; the rows
        of a failed cluster are unspecified."""
        K = len(clusters)
        cand_off, broker_id, broker_rack, topic_off, drf, th, part_off, part_id, rep_off, cur = self.marshal_clusters(clusters)
        if out_stride is None:
            out_stride = _default_stride(rep_off, int(drf.max()) if K else -1)
        Q = int(part_off[-1])
        out = np.full((Q, out_stride), -1, dtype=np.int32)
        out_len = np.zeros(Q, dtype=np.int32)
        st = (KaStatus * max(K, 1))()
        self._L.ka_solve_clusters(self._h, K, _ptr(cand_off), _ptr(broker_id), _ptr(broker_rack), _ptr(topic_off), _ptr(drf),
                                  _ptr(th), _ptr(part_off), _ptr(part_id), _ptr(rep_off), _ptr(cur), int(out_stride), _ptr(out_len),
                                  _ptr(out), st)
        rows = part_off[topic_off]
        return [(out[rows[k]:rows[k + 1]], out_len[rows[k]:rows[k + 1]], st[k]) for k in range(K)]

    def solve_clusters_json(self, clusters, topic_names, json_buf=None):
        """ka_solve_clusters_json: the fleet of solve_clusters, every cluster's reassignment JSON built on the device.
        topic_names: one list of names per cluster. json_buf: optional writable uint8 numpy array (pinned for full PCIe speed);
        by default one of the documented sufficient size. Returns one (bytes-like view of the cluster's text, KaStatus) per
        cluster; the text of a failed cluster is empty."""
        K = len(clusters)
        cand_off, broker_id, broker_rack, topic_off, drf, th, part_off, part_id, rep_off, cur = self.marshal_clusters(clusters)
        names, name_off = self.marshal_names([n for names_k in topic_names for n in names_k])
        assert len(name_off) == len(th) + 1
        if json_buf is None:
            rows, name_len, cap = np.diff(part_off), np.diff(name_off), 0
            for k in range(K):
                t0, t1 = int(topic_off[k]), int(topic_off[k + 1])
                S = _default_stride(rep_off[part_off[t0]:part_off[t1] + 1], int(drf[k]))
                cap += 64 + int(part_off[t1] - part_off[t0]) * (50 + 12 * S) + int(np.dot(rows[t0:t1], name_len[t0:t1]))
            json_buf = np.empty(max(cap, 1), dtype=np.uint8)
        json_off = np.zeros(K + 1, dtype=np.int64)
        st = (KaStatus * max(K, 1))()
        self._L.ka_solve_clusters_json(self._h, K, _ptr(cand_off), _ptr(broker_id), _ptr(broker_rack), _ptr(topic_off), _ptr(drf),
                                       _ptr(th), _ptr(part_off), _ptr(part_id), _ptr(rep_off), _ptr(cur), _ptr(names),
                                       _ptr(name_off), _ptr(json_buf), int(json_buf.size), _ptr(json_off), st)
        return [(json_buf[json_off[k]:json_off[k + 1]], st[k]) for k in range(K)]

    def stage_dense_device(self, T, d_topic_hash, P, RF, d_cur, desired_rf, out_stride, stream=0):
        """Context-free stage (KAS:65-200) of a topic block — shards across GPUs."""
        rc = self._L.ka_stage_dense_device(self._h, int(T), ctypes.c_void_p(d_topic_hash), int(P), int(RF),
                                           ctypes.c_void_p(d_cur), int(desired_rf), int(out_stride),
                                           ctypes.c_void_p(stream) if stream else None)
        if rc:
            raise KassignError(rc, "ka_stage_dense_device")

    def order_device(self, d_out_len, d_out, stream=0, sync=True):
        """Leader-order stage (KAS:202-239) of the staged block against this Context's counters."""
        st = KaStatus()
        rc = self._L.ka_order_device(self._h, ctypes.c_void_p(d_out_len) if d_out_len else None, ctypes.c_void_p(d_out),
                                     ctypes.c_void_p(stream) if stream else None, ctypes.byref(st) if sync else None)
        if not sync:
            if rc:
                raise KassignError(rc, "ka_order_device")
            return None
        return st

    def staged_slot_chains(self):
        """2 when the staged block is ordered by per-slot chains (rows <= 3), else 0."""
        return int(self._L.ka_staged_slot_chains(self._h))

    def order_slot_device(self, slot, stream=0):
        """Slot-0 / slot-1 leader-order chain of the staged block (reads and bumps only counter[.][slot])."""
        rc = self._L.ka_order_slot_device(self._h, int(slot), ctypes.c_void_p(stream) if stream else None)
        if rc:
            raise KassignError(rc, "ka_order_slot_device")

    def emit_device(self, d_out_len, d_out, stream=0, sync=True):
        st = KaStatus()
        rc = self._L.ka_emit_device(self._h, ctypes.c_void_p(d_out_len) if d_out_len else None, ctypes.c_void_p(d_out),
                                    ctypes.c_void_p(stream) if stream else None, ctypes.byref(st) if sync else None)
        if not sync:
            if rc:
                raise KassignError(rc, "ka_emit_device")
            return None
        return st

    def export_counter_slot_device(self, slot, d_ptr, stream=0):
        rc = self._L.ka_ctx_export_counter_slot_device(self._h, int(slot), ctypes.c_void_p(d_ptr), ctypes.c_void_p(stream) if stream else None)
        if rc:
            raise KassignError(rc)

    def import_counter_slot_device(self, slot, d_ptr, stream=0):
        rc = self._L.ka_ctx_import_counter_slot_device(self._h, int(slot), ctypes.c_void_p(d_ptr), ctypes.c_void_p(stream) if stream else None)
        if rc:
            raise KassignError(rc)

    def last_status(self):
        st = KaStatus()
        self._L.ka_last_status(self._h, ctypes.byref(st))
        return st

    def export_counters_device(self, d_ptr, stream=0):
        rc = self._L.ka_ctx_export_counters_device(self._h, ctypes.c_void_p(d_ptr), ctypes.c_void_p(stream) if stream else None)
        if rc:
            raise KassignError(rc)

    def import_counters_device(self, d_ptr, stream=0):
        rc = self._L.ka_ctx_import_counters_device(self._h, ctypes.c_void_p(d_ptr), ctypes.c_void_p(stream) if stream else None)
        if rc:
            raise KassignError(rc)

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
        maxlen = max([len(l) for l in lists], default=0)
        stride = max(1, maxlen, desired_replication_factor if desired_replication_factor >= 0 else 0)
        th = np.array([java_string_hash(topic)], dtype=np.int32)
        out, out_len, _ = self._solver.solve_ragged(th, part_off, np.array(parts, dtype=np.int32), rep_off, cur,
                                                    desired_replication_factor, stride, check=True, topic_names=[topic])
        return {p: [int(x) for x in out[i, :out_len[i]]] for i, p in enumerate(parts)}
