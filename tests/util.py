"""Shared helpers of the test suite, each written once: flatten {topic: {partition: [brokers]}} cases into the flat layout of
include/kassign.h and run them through the C++ oracle or the CUDA library; broker tables, problems, fleets and wave inputs;
the checks and fakes more than one test module uses. The plain-Python models live in tests/models.py."""
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SEND_SUMMARY_DTYPE, WAVE_SUMMARY_DTYPE
from tests import fit_models, models

HERE = os.path.dirname(os.path.abspath(__file__))
FRACS = (0.01, 0.02, 0.05, 0.10, 0.20, 0.30, 0.40, 0.50)
MIN_HASH = "polygenelubricants"   # String.hashCode == Integer.MIN_VALUE (KAS:190-192)


def load_golden():
    with open(os.path.join(HERE, "golden", "cases.json")) as f:
        cases = json.load(f)
    for c in cases:
        c["topics"] = [(n, {int(k): v for k, v in cur.items()}) for n, cur in c["topics"]]
        c["racks"] = {int(k): v for k, v in c["racks"].items()}
    return cases


def flatten(topics):
    """topics: [(name, {partition: [brokers]})] -> names, part_off, part_id, rep_off, cur (ascending partitions)."""
    names, part_off, part_id, rep_off, cur = [], [0], [], [0], []
    for name, asg in topics:
        names.append(name)
        for p in sorted(asg):
            part_id.append(p)
            cur.extend(asg[p])
            rep_off.append(len(cur))
        part_off.append(len(part_id))
    return (names, np.array(part_off, dtype=np.int64), np.array(part_id, dtype=np.int32),
            np.array(rep_off, dtype=np.int64), np.array(cur, dtype=np.int32))


def stride_for(topics, desired_rf):
    m = max([len(v) for _, a in topics for v in a.values()], default=0)
    return max(1, m, desired_rf if desired_rf >= 0 else 0)


def records_from_flat(names, part_off, part_id, out, out_len):
    recs = []
    for t, n in enumerate(names):
        for g in range(int(part_off[t]), int(part_off[t + 1])):
            recs.append([n, int(part_id[g]), [int(x) for x in out[g, :out_len[g]]]])
    return recs


def run_oracle_case(ol, case):
    names, part_off, part_id, rep_off, cur = flatten(case["topics"])
    brokers = sorted(case["brokers"])
    racks = [case["racks"].get(b) for b in brokers]
    stride = stride_for(case["topics"], case["desired_rf"])
    ln, pid, out, st = ol.run(ol.OracleContext(), names, part_off, part_id, rep_off, cur, brokers, racks,
                              case["desired_rf"], stride, raise_on_error=False)
    if st.code != 0:
        return {"error": {"kind": st.code, "message": st.message.decode(), "partition": st.partition, "a": st.a, "b": st.b},
                "topic_index": st.topic_index}
    return {"records": records_from_flat(names, part_off, pid, out, ln)}


def run_gpu_case(kab, case, solver=None):
    """Through the C ABI (ka_solve, ragged form). Returns records or the re-thrown reference exception."""
    names, part_off, part_id, rep_off, cur = flatten(case["topics"])
    s = solver or kab.Solver(0)
    s.set_brokers_with_racks(case["brokers"], case["racks"])
    stride = stride_for(case["topics"], case["desired_rf"])
    th = np.array([kab.java_string_hash(n) for n in names], dtype=np.int32)
    out, out_len, st = s.solve_ragged(th, part_off, part_id, rep_off, cur, case["desired_rf"], stride, check=False)
    if st.code != 0:
        try:
            kab.raise_for_status(st, names)
        except (kab.IllegalStateException, kab.ArrayIndexOutOfBoundsException) as e:
            return {"error": {"kind": st.code, "message": str(e), "partition": st.partition, "a": st.a, "b": st.b},
                    "topic_index": st.topic_index}
    return {"records": records_from_flat(names, part_off, part_id, out, out_len)}


def oracle_dense(ol, cl, ctx=None):
    """Run a synth.Cluster through the C++ oracle; returns (out [T*P, RF], out_len, status)."""
    part_off, part_id, rep_off, cur = cl.ragged()
    ln, _, out, st = ol.run(ctx or ol.OracleContext(), cl.topic_names, part_off, part_id, rep_off, cur, cl.broker_id,
                            cl.rack_name, cl.desired_rf, max(cl.RF, cl.desired_rf, 1), raise_on_error=False)
    return out, ln, st


def fields(st):
    """A KaStatus as a comparable tuple."""
    return (st.code, st.topic_index, st.partition, st.a, st.b)


def record_of(s, names):
    """The fields `names` of one structured-array summary as a dict of ints."""
    return {f: int(s[f]) for f in names}


EMPTY_SUMMARY = dict({f: 0 for f in kab.assigner.MOVE_SUMMARY_DTYPE.names}, max_broker_in_id=-1)   # a refused candidate's


def row_width(rep_off, desired_rf):
    """The narrowest row stride for these lists and desired RF."""
    sizes = np.diff(rep_off)
    return max(int(sizes.max()) if len(sizes) else 0, desired_rf, 1)


def run_child(code, d, timeout, meanwhile, what):
    """Runs the Python source `code` in a child process, from the repository root with the package importable and argv[1] = d,
    while the parent calls meanwhile(). A child that is not done `timeout` seconds after its start is killed and fails the test
    ("<what> did not finish"): device calls that never finished go away with the child, not the test session. Returns
    (meanwhile's result, the child's output, seconds from its start to its end)."""
    root = os.path.dirname(HERE)
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    flags = ["-s"] if sys.flags.no_user_site else []
    t0 = time.monotonic()
    child = subprocess.Popen([sys.executable] + flags + ["-c", code, str(d)], cwd=root, env=env, stdout=subprocess.PIPE,
                             stderr=subprocess.STDOUT, text=True)
    try:
        res = meanwhile()
        out, _ = child.communicate(timeout=max(1.0, timeout - (time.monotonic() - t0)))
    except subprocess.TimeoutExpired:
        pytest.fail("%s did not finish within %d s" % (what, timeout))
    finally:
        if child.poll() is None:
            child.kill()
            child.communicate()
    assert child.returncode == 0, out
    return res, out, time.monotonic() - t0


def has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


# ---- work held behind a device sleep -------------------------------------------------------------------------------------

# About 0.1 s at the H100's 1.98 GHz SM clock: far longer than the host's enqueue of any call the tests hold behind it.
SLEEP_CYCLES = 200_000_000


def device_sleep(stream, cycles=SLEEP_CYCLES):
    """A device sleep on `stream`, enqueued at once. Returns its (start, end) events."""
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        a.record()
        torch.cuda._sleep(cycles)
        b.record()
    return a, b


def enqueued_behind(sleep, t_call):
    """The call was enqueued (t_call seconds on the host) well inside the sleep ahead of its inputs."""
    ms = sleep[0].elapsed_time(sleep[1])
    print("device sleep %.1f ms, host enqueue %.3f ms" % (ms, 1e3 * t_call))
    assert 1e3 * t_call < ms / 2, ("the call's enqueue outlasted half the sleep: the test would not see an early read", t_call, ms)


# ---- fakes of the library ------------------------------------------------------------------------------------------------

def view(p, n, ctype):
    """A copy of the n elements of `ctype` at the C pointer p (None for a NULL pointer)."""
    if p is None:
        return None
    if n == 0:
        return np.zeros(0, dtype=ctype)
    return np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(np.ctypeslib.as_ctypes_type(ctype))), shape=(n,)).copy()


def writable(p, n, ctype):
    return np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(np.ctypeslib.as_ctypes_type(ctype))), shape=(n,))


def fake_solver(lib):
    s = object.__new__(kab.Solver)
    s._L = lib
    s._h = ctypes.c_void_p(1)
    return s


class FakeWaveLib:
    """Stands in for libkassign.so's eight wave entry points: records what each call is handed, plans W waves
    (wave[g] = 1 + g % W), writes recognisable summaries (field f of summary v: 10 v + f, the sender fields as f = 5, 6), at most
    `cap` of them, and writes document v of the per-wave calls as b"<v>"; the _parts calls write D = 2 W parts (2 W <= Q), part d
    as b"[d]" of wave 1 + d // 2, and the _parts_rollback calls part d's rollback document as b"(d)". With `fail` = (code, a, b)
    every call is refused with that status."""

    def __init__(self, W, fail=None):
        self.W, self.fail, self.calls = W, fail, []

    @staticmethod
    def _rows(Q, rep_off, cur, stride, new_len, new_broker, weight, B, wave):
        r_off = view(rep_off, Q + 1, np.int64)
        return dict(Q=Q, stride=stride, rep_off=r_off, cur=view(cur, int(r_off[-1]), np.int32), new_len=view(new_len, Q, np.int32),
                    new_broker=view(new_broker, Q * stride, np.int32), weight=view(weight, Q, np.int64), B=B, wave=wave is not None)

    @staticmethod
    def _write(buf, cap, offsets, Q, docs):
        text, off = writable(buf, cap, np.uint8), writable(offsets, Q + 1, np.int64)
        at = 0
        for d, doc in enumerate(docs):
            off[d] = at
            text[at:at + len(doc)] = np.frombuffer(doc, dtype=np.uint8)
            at += len(doc)
        off[len(docs)] = at

    def _docs(self, T, part_off, part_id, names, name_off, js, json_cap, doc_off, parts=None, back=None):
        """Writes the documents: the W per-wave ones, or with parts = (L, doc_wave, n_docs) the 2 W parts and with
        back = (back, back_cap, back_off) their rollback documents; nothing for a refused call. Returns Q and what the text
        arguments were."""
        p_off = view(part_off, T + 1, np.int64)
        Q = int(p_off[-1])
        n_off = view(name_off, T + 1, np.int64)
        text = dict(T=T, part_off=p_off, part_id=view(part_id, Q, np.int32), names=bytes(view(names, int(n_off[-1]), np.uint8)),
                    name_off=n_off, json_cap=json_cap)
        if parts is not None:
            text.update(L=parts[0], doc_wave=parts[1] is not None)
        if back is not None:
            text.update(back_cap=back[1])
        if self.fail:
            return Q, text
        if parts is None:
            self._write(js, json_cap, doc_off, Q, [b"<%d>" % v for v in range(self.W)])
            return Q, text
        D = 2 * self.W
        self._write(js, json_cap, doc_off, Q, [b"[%d]" % d for d in range(D)])
        if back is not None:
            self._write(*back, Q, [b"(%d)" % d for d in range(D)])
        writable(parts[1], Q, np.int32)[:D] = 1 + np.arange(D) // 2
        parts[2]._obj.value = D
        return Q, text

    def _call(self, Q, rows, text, send, cap):
        call = dict(self._rows(Q, *rows), **text)
        if send is not None:
            call.update(send_id=view(send[1], send[0], np.int32), C=send[2])
        self.calls.append(dict(call, cap=cap))

    def _fill(self, Q, wave, n_waves, summary, send_summary, cap, st, n_docs=None):
        if self.fail:
            st._obj.code, st._obj.a, st._obj.b = self.fail
            n_waves._obj.value = 0
            if n_docs is not None:
                n_docs._obj.value = 0
            return self.fail[0]
        if wave is not None and Q:
            writable(wave, Q, np.int32)[:] = 1 + np.arange(Q) % self.W
        n = min(cap, self.W)
        if cap:
            writable(summary, cap * 5, np.int64).reshape(cap, 5)[:n] = np.arange(n)[:, None] * 10 + np.arange(5)
            if send_summary is not None:
                writable(send_summary, cap * 2, np.int64).reshape(cap, 2)[:n] = np.arange(n)[:, None] * 10 + 5 + np.arange(2)
        n_waves._obj.value = self.W
        st._obj.code = 0
        return 0

    def ka_plan_waves(self, h, Q, rep_off, cur, stride, new_len, new_broker, weight, B, wave, n_waves, summary, cap, st):
        self._call(Q, (rep_off, cur, stride, new_len, new_broker, weight, B, wave), {}, None, cap)
        return self._fill(Q, wave, n_waves, summary, None, cap, st)

    def ka_plan_waves_send(self, h, Q, rep_off, cur, stride, new_len, new_broker, weight, B, n_send, send_id, C, wave, n_waves, summary,
                           send_summary, cap, st):
        self._call(Q, (rep_off, cur, stride, new_len, new_broker, weight, B, wave), {}, (n_send, send_id, C), cap)
        return self._fill(Q, wave, n_waves, summary, send_summary, cap, st)

    def ka_plan_waves_json(self, h, T, part_off, part_id, rep_off, cur, stride, new_len, new_broker, weight, B, names, name_off,
                           js, json_cap, doc_off, wave, n_waves, summary, cap, st):
        Q, text = self._docs(T, part_off, part_id, names, name_off, js, json_cap, doc_off)
        self._call(Q, (rep_off, cur, stride, new_len, new_broker, weight, B, wave), text, None, cap)
        return self._fill(Q, wave, n_waves, summary, None, cap, st)

    def ka_plan_waves_send_json(self, h, T, part_off, part_id, rep_off, cur, stride, new_len, new_broker, weight, B, n_send, send_id, C,
                                names, name_off, js, json_cap, doc_off, wave, n_waves, summary, send_summary, cap, st):
        Q, text = self._docs(T, part_off, part_id, names, name_off, js, json_cap, doc_off)
        self._call(Q, (rep_off, cur, stride, new_len, new_broker, weight, B, wave), text, (n_send, send_id, C), cap)
        return self._fill(Q, wave, n_waves, summary, send_summary, cap, st)

    def ka_plan_waves_json_parts(self, h, T, part_off, part_id, rep_off, cur, stride, new_len, new_broker, weight, B, names,
                                 name_off, js, json_cap, L, doc_off, doc_wave, n_docs, wave, n_waves, summary, cap, st):
        Q, text = self._docs(T, part_off, part_id, names, name_off, js, json_cap, doc_off, (L, doc_wave, n_docs))
        self._call(Q, (rep_off, cur, stride, new_len, new_broker, weight, B, wave), text, None, cap)
        return self._fill(Q, wave, n_waves, summary, None, cap, st, n_docs)

    def ka_plan_waves_send_json_parts(self, h, T, part_off, part_id, rep_off, cur, stride, new_len, new_broker, weight, B, n_send,
                                      send_id, C, names, name_off, js, json_cap, L, doc_off, doc_wave, n_docs, wave, n_waves,
                                      summary, send_summary, cap, st):
        Q, text = self._docs(T, part_off, part_id, names, name_off, js, json_cap, doc_off, (L, doc_wave, n_docs))
        self._call(Q, (rep_off, cur, stride, new_len, new_broker, weight, B, wave), text, (n_send, send_id, C), cap)
        return self._fill(Q, wave, n_waves, summary, send_summary, cap, st, n_docs)

    def ka_plan_waves_json_parts_rollback(self, h, T, part_off, part_id, rep_off, cur, stride, new_len, new_broker, weight, B, names,
                                          name_off, js, json_cap, L, doc_off, doc_wave, n_docs, back, back_cap, back_off, wave,
                                          n_waves, summary, cap, st):
        Q, text = self._docs(T, part_off, part_id, names, name_off, js, json_cap, doc_off, (L, doc_wave, n_docs),
                             (back, back_cap, back_off))
        self._call(Q, (rep_off, cur, stride, new_len, new_broker, weight, B, wave), text, None, cap)
        return self._fill(Q, wave, n_waves, summary, None, cap, st, n_docs)

    def ka_plan_waves_send_json_parts_rollback(self, h, T, part_off, part_id, rep_off, cur, stride, new_len, new_broker, weight, B,
                                               n_send, send_id, C, names, name_off, js, json_cap, L, doc_off, doc_wave, n_docs,
                                               back, back_cap, back_off, wave, n_waves, summary, send_summary, cap, st):
        Q, text = self._docs(T, part_off, part_id, names, name_off, js, json_cap, doc_off, (L, doc_wave, n_docs),
                             (back, back_cap, back_off))
        self._call(Q, (rep_off, cur, stride, new_len, new_broker, weight, B, wave), text, (n_send, send_id, C), cap)
        return self._fill(Q, wave, n_waves, summary, send_summary, cap, st, n_docs)


# ---- broker tables -------------------------------------------------------------------------------------------------------

def table(ids, racks_per=None):
    """(ids, rack_index): racks_per = brokers per rack (contiguous), or None: no broker has a rack."""
    ids = np.asarray(ids, dtype=np.int32)
    names = [None] * len(ids) if racks_per is None else ["k%d" % (i // racks_per) for i in range(len(ids))]
    return ids, kab.synth.rack_indices(ids, names)


def bsearch_table(N):
    """Brokers 1..N plus one id far away: an id range beyond the global LUT, so ids are looked up by binary search."""
    return table(np.concatenate([np.arange(1, N + 1), [1 << 27]]).astype(np.int32), 4)


def ragged_mixed_tables(rng, cl):
    """Candidate tables for a make_ragged_cluster: every capacity and lookup mode, and one without brokers (the last)."""
    live = cl.broker_id
    return [
        (cl.broker_id, cl.rack_index),                                                        # capacity > 1, the cluster's racks
        table(np.sort(rng.choice(live, len(live) - 4, replace=False))),                       # capacity > 1, no racks
        table(np.sort(rng.choice(live, len(live) - 6, replace=False)), 3),                    # capacity > 1, other racks
        table(np.arange(1, 1 + 4000, dtype=np.int32), 40),                                    # capacity 1, racks
        table(np.arange(1, 1 + 3000, dtype=np.int32)),                                        # capacity 1, no racks
        table(1 + 2 * np.arange(20000, dtype=np.int32), 500),                                 # 20 000 brokers, global id LUT
        table(np.zeros(0, dtype=np.int32)),                                                   # no broker
    ]


# ---- candidate problems --------------------------------------------------------------------------------------------------

class DenseProblem:
    """A dense problem on the device: topic hashes, current lists, and room for K candidates' rows."""

    def __init__(self, topic_hash, cur, desired_rf=-1, out_stride=None):
        import torch
        self.T, self.P, self.RF = cur.shape
        self.desired_rf = desired_rf
        self.S = out_stride or max(self.RF, desired_rf, 1)
        self.topic_hash, self.cur = topic_hash, cur
        self.d_hash = torch.from_numpy(np.ascontiguousarray(topic_hash, dtype=np.int32)).cuda()
        self.d_cur = torch.from_numpy(np.ascontiguousarray(cur, dtype=np.int32)).cuda()

    def sequential(self, tables):
        """The contract's reference: a fresh context per table, ka_ctx_set_brokers + ka_solve_dense_device."""
        import torch
        rows = []
        for ids, racks in tables:
            s = kab.Solver(0)
            s.set_brokers(ids, racks)
            out = torch.full((self.T, self.P, self.S), -7, dtype=torch.int32, device="cuda")
            ln = torch.full((self.T, self.P), -7, dtype=torch.int32, device="cuda")
            st = s.solve_dense_device(self.T, self.d_hash.data_ptr(), self.P, self.RF, self.d_cur.data_ptr(), self.desired_rf,
                                      self.S, ln.data_ptr(), out.data_ptr())
            rows.append((out.cpu().numpy(), ln.cpu().numpy(), fields(st)))
            s.close()
        return rows

    def batched(self, tables, solver=None):
        import torch
        K = len(tables)
        out = torch.full((K, self.T, self.P, self.S), -7, dtype=torch.int32, device="cuda")
        ln = torch.full((K, self.T, self.P), -7, dtype=torch.int32, device="cuda")
        s = solver or kab.Solver(0)
        sts = s.solve_dense_candidates_device(tables, self.T, self.d_hash.data_ptr(), self.P, self.RF, self.d_cur.data_ptr(),
                                              self.desired_rf, self.S, ln.data_ptr(), out.data_ptr())
        return out.cpu().numpy(), ln.cpu().numpy(), [fields(st) for st in sts]


def check_dense_equal(prob, tables, oracle=None, solver=None):
    """ka_solve_dense_candidates_device against a fresh context per table (and the oracle). Returns the statuses."""
    out, ln, sts = prob.batched(tables, solver)
    seq = prob.sequential(tables)
    for k, (e_out, e_len, e_st) in enumerate(seq):
        assert sts[k] == e_st, (k, sts[k], e_st)
        if e_st[0] != 0:
            continue   # the rows of a failed candidate are unspecified
        assert np.array_equal(out[k], e_out), k
        assert np.array_equal(ln[k], e_len), k
        if oracle is not None:
            ids, racks = tables[k]
            exp, exp_len, est = oracle.fast_run_dense(oracle.FastContext(), prob.topic_hash, prob.cur, ids, racks, prob.desired_rf,
                                                      prob.S)
            assert est.code == 0, k
            assert np.array_equal(out[k].reshape(-1, prob.S), exp), k
            assert np.array_equal(ln[k].reshape(-1), exp_len), k
    return sts


class Problem:
    """The ka_solve inputs of one run (host arrays)."""

    def __init__(self, names, topic_hash, part_off, part_id, rep_off, cur, desired_rf=-1, out_stride=None):
        self.names, self.topic_hash, self.part_off, self.part_id, self.rep_off, self.cur = names, topic_hash, part_off, part_id, rep_off, cur
        self.desired_rf = desired_rf
        self.S = out_stride or row_width(rep_off, desired_rf)

    @classmethod
    def of(cls, cl, desired_rf=-1):
        return cls(cl.topic_names, cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, desired_rf)

    def args(self):
        return self.topic_hash, self.part_off, self.part_id, self.rep_off, self.cur, self.desired_rf

    def sequential(self, tables):
        """The contract's reference: a fresh context per table, ka_ctx_set_brokers + ka_solve."""
        rows = []
        for ids, racks in tables:
            s = kab.Solver(0)
            s.set_brokers(ids, racks)
            out, ln, st = s.solve_ragged(*self.args(), self.S, check=False)
            rows.append((out, ln, fields(st)))
            s.close()
        return rows

    def batched(self, tables, solver=None):
        s = solver or kab.Solver(0)
        out, ln, sts = s.solve_ragged_candidates(tables, *self.args(), out_stride=self.S)
        return out, ln, [fields(st) for st in sts]


def check_equal(prob, tables, oracle=None, solver=None):
    """ka_solve_candidates against a fresh context per table (and the oracle). Returns the statuses."""
    out, ln, sts = prob.batched(tables, solver)
    seq = prob.sequential(tables)
    assert len(sts) == len(tables)
    for k, (e_out, e_len, e_st) in enumerate(seq):
        assert sts[k] == e_st, (k, sts[k], e_st)
        if e_st[0] != 0:
            continue   # the rows of a failed candidate are unspecified
        assert np.array_equal(out[k], e_out), k
        assert np.array_equal(ln[k], e_len), k
        if oracle is not None:
            ids, racks = tables[k]
            o_len, _, o_out, o_st = oracle.run(oracle.OracleContext(), prob.names, prob.part_off, prob.part_id, prob.rep_off, prob.cur,
                                               ids, ["k%d" % r for r in racks], prob.desired_rf, prob.S, raise_on_error=False)
            assert o_st.code == 0, k
            assert np.array_equal(out[k], o_out) and np.array_equal(ln[k], o_len), k
    return sts


def check_scores(prob, tables, weight=None, oracle=None, solver=None, sequential=True):
    """One ka_score_candidates call (rows and per-broker arrays asked for) against ka_solve_candidates' rows (checked against
    fresh single solves and the oracle when `sequential`) and the numpy reference. Returns the statuses and summaries."""
    s = solver or kab.Solver(0)
    if sequential:
        sts = check_equal(prob, tables, oracle, solver=s)
        out, ln, _ = prob.batched(tables, s)
    else:
        out, ln, sts = prob.batched(tables, s)
    summary, st, sc_out, sc_len, rep, lead, inb = s.score_ragged_candidates(tables, *prob.args(), out_stride=prob.S, weight=weight,
                                                                           rows=True, per_broker=True)
    assert [fields(x) for x in st] == sts
    names = kab.assigner.MOVE_SUMMARY_DTYPE.names
    w = np.ones(int(prob.part_off[-1]), dtype=np.int64) if weight is None else weight
    for k, (ids, _) in enumerate(tables):
        if sts[k][0] != 0:
            assert record_of(summary[k], names) == EMPTY_SUMMARY, k
            assert not rep[k].any() and not lead[k].any() and not inb[k].any(), k
            continue
        assert np.array_equal(sc_out[k], out[k]) and np.array_equal(sc_len[k], ln[k]), k
        e, e_rep, e_lead, e_in = models.move_summary(out[k], ln[k], prob.rep_off, prob.cur, np.asarray(ids, dtype=np.int64), weight)
        assert record_of(summary[k], names) == e, (k, record_of(summary[k], names), e)
        assert np.array_equal(rep[k], e_rep) and np.array_equal(lead[k], e_lead) and np.array_equal(inb[k], e_in), k
        # identities
        assert rep[k].sum() == int((w * ln[k]).sum()) and lead[k].sum() == int(w[ln[k] > 0].sum())
        assert inb[k].sum() == summary[k]["replicas_added"]
    return sts, summary


def sparse_with_empty_topics(cl, rng, empty):
    """cl's topics with sparse (ascending, gapped) partition ids and, with `empty`, a topic without partitions after every
    seventh one."""
    names, th, P, pid = [], [], [], []
    for t in range(cl.T):
        a, b = int(cl.part_off[t]), int(cl.part_off[t + 1])
        names.append(cl.topic_names[t])
        th.append(cl.topic_hash[t])
        P.append(b - a)
        pid.append(np.cumsum(rng.integers(1, 9, size=b - a)).astype(np.int32) - 1)
        if empty and t % 7 == 3:
            names.append("empty.%d" % t)
            th.append(kab.java_string_hash("empty.%d" % t))
            P.append(0)
            pid.append(np.zeros(0, dtype=np.int32))
    part_off = np.zeros(len(P) + 1, dtype=np.int64)
    np.cumsum(P, out=part_off[1:])
    return names, np.array(th, dtype=np.int32), part_off, np.concatenate(pid), cl.rep_off, cl.cur


def exception_problem(tail):
    """Three topics whose failure depends on the table, then `tail`: a list-size mismatch, or a topic without partitions."""
    topics = [("alpha", {3: [1, 2], 7: [2, 3], 8: [3, 4], 40: [4, 5], 41: [5, 6]}),
              ("polygenelubricants", {5: [1, 2], 6: [2, 1]}),       # String.hashCode == Integer.MIN_VALUE (KAS:190-192)
              ("gamma", {11: [1, 2, 3], 12: [2, 3, 4], 13: [3, 4, 5]})]
    if tail == "mismatch":
        topics.append(("delta", {0: [1, 2], 9: [3]}))
    elif tail == "empty":
        topics.append(("none", {}))
    names, part_off, part_id, rep_off, cur = flatten(topics)
    th = np.array([kab.java_string_hash(n) for n in names], dtype=np.int32)
    return Problem(names, th, part_off, part_id, rep_off, cur, -1, 3)


# ---- fleets --------------------------------------------------------------------------------------------------------------

class Member:
    """One cluster of a fleet: its table, its ka_solve inputs (offsets from 0) and its topic names."""

    def __init__(self, table, names, topic_hash, part_off, part_id, rep_off, cur, desired_rf=-1):
        self.ids, self.racks = table
        self.names = list(names)
        self.topic_hash = np.asarray(topic_hash, dtype=np.int32)
        self.part_off, self.part_id, self.rep_off, self.cur = part_off, part_id, rep_off, cur
        self.desired_rf = desired_rf

    @classmethod
    def of(cls, cl, table=None, desired_rf=-1):
        return cls(table or (cl.broker_id, cl.rack_index), cl.topic_names, cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off,
                   cl.cur, desired_rf)

    @classmethod
    def of_topics(cls, table, topics, desired_rf=-1):
        names, part_off, part_id, rep_off, cur = flatten(topics)
        return cls(table, names, [kab.java_string_hash(n) for n in names], part_off, part_id, rep_off, cur, desired_rf)

    def entry(self):
        return (self.ids, self.racks, self.topic_hash, self.part_off, self.part_id, self.rep_off, self.cur, self.desired_rf)

    def sequential(self, s, S):
        """The contract's reference: a fresh Context with this cluster's table, then ka_solve."""
        s.reset()
        s.set_brokers(self.ids, self.racks)
        out, ln, st = s.solve_ragged(self.topic_hash, self.part_off, self.part_id, self.rep_off, self.cur, self.desired_rf, S,
                                     check=False)
        return out, ln, fields(st)


def fleet_stride(fleet):
    """The narrowest row stride for every cluster of the fleet."""
    return max([row_width(m.rep_off, m.desired_rf) for m in fleet] + [1])


def min_hash_cluster(table):
    """Topics around one whose hashCode is Integer.MIN_VALUE, with lists of 2 (|hash| % 2 == 0: it solves)."""
    topics = [("a", {0: [1, 2], 1: [2, 3]}), (MIN_HASH, {3: [1, 2], 5: [2, 3], 6: [3, 1]}), ("z", {0: [3, 4]})]
    return Member.of_topics(table, topics)


def oracle_text(ol, names, part_off, part_id, rep_off, cur, brokers, rack_names, desired, ctx=None):
    """(text or None, oracle status) of one run through the C++ oracle."""
    pid = part_id if part_id is not None else np.concatenate(
        [np.arange(part_off[t + 1] - part_off[t], dtype=np.int32) for t in range(len(names))] + [np.zeros(0, np.int32)])
    ln, opid, out, st = ol.run(ctx or ol.OracleContext(), names, part_off, pid, rep_off, cur, brokers, rack_names, desired,
                               row_width(rep_off, desired), raise_on_error=False)
    return (None if st.code else models.solve_document(names, part_off, opid, out, ln)), st


def sequential_json(m, s):
    """The contract's reference: a fresh Context with this cluster's table, then ka_solve_json; a cluster wider than the batched
    chains' 3 is refused with its width instead."""
    width = row_width(m.rep_off, m.desired_rf)
    if width > 3:
        return b"", (_native.KA_ERR_LIMIT, -1, -1, width, 0)
    s.reset()
    s.set_brokers(m.ids, m.racks)
    text, st = s.solve_ragged_json(m.names, m.topic_hash, m.part_off, m.part_id, m.rep_off, m.cur, m.desired_rf, check=False)
    return bytes(text), fields(st)


def check_fleet(fleet, oracle=None, solver=None):
    """ka_solve_clusters_json: every cluster against its sequential ka_solve_json (and the oracle's text); the documents back to
    back in cluster order."""
    s = solver or kab.Solver(0)
    res = s.solve_clusters_json([m.entry() for m in fleet], [m.names for m in fleet])
    assert len(res) == len(fleet)
    ref = kab.Solver(0)
    sts, texts = [], []
    for k, (m, (text, st)) in enumerate(zip(fleet, res)):
        e_text, e_st = sequential_json(m, ref)
        assert fields(st) == e_st, (k, fields(st), e_st)
        assert bytes(text) == e_text, k
        sts.append(e_st)
        texts.append(bytes(text))
        if oracle is not None and e_st[0] == 0:
            exp, o_st = oracle_text(oracle, m.names, m.part_off, m.part_id, m.rep_off, m.cur, m.ids, ["k%d" % r for r in m.racks],
                                    m.desired_rf)
            assert o_st.code == 0 and bytes(text).decode() == exp, k
    # the documents back to back in cluster order, in one buffer (a failed cluster's range is empty)
    starts = [t.__array_interface__["data"][0] for t, _ in res if len(t)]
    assert all(b - a == len(t) for a, b, t in zip(starts, starts[1:], [t for t in texts if t]))
    return sts, texts


# ---- wave plans ----------------------------------------------------------------------------------------------------------

def rows(lists, stride=None):
    """(out [Q, stride], out_len [Q]) from a list of new lists; unused slots -1."""
    stride = stride or max([len(x) for x in lists] + [1])
    out = np.full((len(lists), stride), -1, dtype=np.int32)
    for g, x in enumerate(lists):
        out[g, :len(x)] = x
    return out, np.array([len(x) for x in lists], dtype=np.int32)


def cur_lists(lists):
    """(rep_off, cur) from a list of current lists."""
    rep_off = np.zeros(len(lists) + 1, dtype=np.int64)
    np.cumsum([len(x) for x in lists], out=rep_off[1:])
    return rep_off, np.array([b for x in lists for b in x], dtype=np.int32)


def random_wave_case(rng, Q, N, stride=3):
    """Q random (current, new) list pairs over brokers 1..N, 30 % of them unchanged."""
    cur, new = [], []
    for _ in range(Q):
        m = int(rng.integers(0, stride + 1))
        cur.append([int(x) for x in rng.choice(np.arange(1, N + 1), m, replace=False)])
        if rng.random() < 0.3:
            new.append(list(cur[-1]))
        else:
            n = int(rng.integers(0, stride + 1))
            new.append([int(x) for x in rng.choice(np.arange(1, N + 1), n, replace=False)])
    return cur, new


def ragged_wave_case(rng, T, N, shrink=0.0):
    """(names, part_off, part_id, rep_off, cur, out, out_len): T topics of 0..29 partitions (sparse ids below 5000, names of up to
    50 bytes) with the rows of random_wave_case over brokers 1..N; with probability `shrink` a row is a replication-factor
    reduction instead: a 3-broker current list onto its first one or two."""
    sizes = rng.integers(0, 30, T)
    part_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    Q = int(part_off[-1])
    names = ["ragged.%d.%s" % (t, "y" * int(rng.integers(0, 40))) for t in range(T)]
    part_id = np.concatenate([np.sort(rng.choice(5000, n, replace=False)) for n in sizes]).astype(np.int32)
    cur_l, new_l = random_wave_case(rng, Q, N)
    for g in range(Q if shrink else 0):
        if rng.random() < shrink:
            cur_l[g] = [int(x) for x in rng.choice(np.arange(1, N + 1), 3, replace=False)]
            new_l[g] = cur_l[g][:int(rng.integers(1, 3))]
    rep_off, cur = cur_lists(cur_l)
    out, out_len = rows(new_l, 3)
    return names, part_off, part_id, rep_off, cur, out, out_len


def wave_inputs():
    """(names, part_off, part_id, rep_off, cur, out, out_len): four rows in three topics, one empty, for the marshalling tests."""
    out, out_len = rows([[1, 2], [3], [4, 5, 6], []])
    rep_off, cur = cur_lists([[1], [2, 3], [4], [7, 8]])
    return ["alpha", "", "bc"], [0, 3, 3, 4], [4, 9, -2, 0], rep_off, cur, out, out_len


def smallest_limit(names, part_off, part_id, rep_off, cur, out, out_len, wave, rollback=False):
    """The smallest L that fits every changed row: its longest one-record document, on either side with rollback."""
    best = 0
    for t, name in enumerate(names):
        for g in range(int(part_off[t]), int(part_off[t + 1])):
            if wave[g]:
                p = int(part_id[g]) if part_id is not None else g - int(part_off[t])
                best = max(best, 29 + len(models.record(name, p, out[g][:int(out_len[g])]).encode()))
                if rollback:
                    best = max(best, 29 + len(models.current_record(name, p, cur[int(rep_off[g]):int(rep_off[g + 1])]).encode()))
    return best


def check_wave_documents(s, names, part_off, part_id, rep_off, cur, out, out_len, B, L=None, rollback=False, weight=None, C=None,
                         send_ids=None, json_buf=None):
    """plan_waves_json (L None), plan_wave_parts_json or, with rollback, plan_wave_parts_rollback_json against
    models.wave_documents and against plan_waves on the same inputs; with C a sender budget over send_ids (None: the Solver's
    table). Returns (docs, backs, doc_wave, wave, summary, status), the shape of models.wave_documents."""
    send_ids = list(np.asarray(s.broker_id if send_ids is None else send_ids))
    send = {} if C is None else dict(max_broker_out=C, send_brokers=send_ids)
    args = (names, part_off, part_id, rep_off, cur, out, out_len, B)
    if L is None:
        docs, wave, summ, st = s.plan_waves_json(*args, weight=weight, json_buf=json_buf, **send)
        got = (docs, None, np.arange(1, len(docs) + 1, dtype=np.int32), wave, summ, st)
    elif not rollback:
        docs, doc_wave, wave, summ, st = s.plan_wave_parts_json(*args, L, weight=weight, json_buf=json_buf, **send)
        got = (docs, None, doc_wave, wave, summ, st)
    else:
        got = s.plan_wave_parts_rollback_json(*args, L, weight=weight, json_buf=json_buf, **send)
    docs, backs, doc_wave, wave, summ, st = got
    e_docs, e_backs, e_doc_wave, e_wave, e_summ, e_st = models.wave_documents(
        names, part_off, part_id, rep_off, cur, out, out_len, s.broker_id, B, weight, None if C is None else (send_ids, C), L, rollback)
    assert (st.code, st.a, st.b) == e_st, ((st.code, st.a, st.b), e_st)
    p_wave, p_summ, p_st = s.plan_waves(rep_off, cur, out, out_len, B, weight=weight, **send)
    assert (p_st.code, p_st.a, p_st.b) == (e_st if e_st[0] != _native.KA_ERR_LIMIT else (0, 0, 0))
    if st.code == 0:
        dtype = WAVE_SUMMARY_DTYPE if C is None else WAVE_SEND_SUMMARY_DTYPE
        assert np.array_equal(wave, e_wave) and np.array_equal(wave, p_wave)
        assert [record_of(x, dtype.names) for x in summ] == e_summ and np.array_equal(summ, p_summ)
        assert doc_wave.tolist() == e_doc_wave and len(docs) == len(e_docs)
        for d, (x, e) in enumerate(zip(docs, e_docs)):
            assert bytes(x) == e, (d, bytes(x)[:200], e[:200])
        if rollback:
            assert len(backs) == len(e_backs)
            for d, (x, e) in enumerate(zip(backs, e_backs)):
                assert bytes(x) == e, (d, bytes(x)[:200], e[:200])
    else:
        assert docs == [] and backs in (None, []) and len(doc_wave) == len(wave) == len(summ) == 0
    return got


def summary_array(summ, dtype):
    """A model's summary dicts as a structured array of `dtype`."""
    return np.array([tuple(s[f] for f in dtype.names) for s in summ], dtype=dtype)


def check_plan(s, rep_off, cur, out, out_len, B, weight=None, send_ids=None, C=None, rule="first_fit"):
    """plan_waves under `rule` against its model (fit_models.plan_waves or models.plan_waves), every field; with C a sender
    budget over send_ids. Returns (wave, summary, status)."""
    s.set_wave_rule(rule)
    send = {} if C is None else dict(max_broker_out=C, send_brokers=send_ids)
    wave, summ, st = s.plan_waves(rep_off, cur, out, out_len, B, weight=weight, **send)
    plan = fit_models.plan_waves if rule == "first_fit" else models.plan_waves
    e_wave, e_summ, e_st = plan(rep_off, cur, out, out_len, s.broker_id, B, weight, None if C is None else (list(send_ids), C))
    assert (st.code, st.a, st.b) == e_st, ((st.code, st.a, st.b), e_st)
    if st.code == 0:
        assert np.array_equal(wave, e_wave), np.nonzero(wave != e_wave)[0][:10]
        names = (WAVE_SUMMARY_DTYPE if C is None else WAVE_SEND_SUMMARY_DTYPE).names
        assert [record_of(x, names) for x in summ] == e_summ
    return wave, summ, st


def solved(cl, desired_rf=-1):
    """A fresh Solver on the cluster's table and the rows ka_solve gives for it."""
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    S = max(int(np.diff(cl.rep_off).max()), desired_rf, 1)
    out, out_len, st = s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, desired_rf, S)
    assert st.code == 0
    return s, out, out_len, S


def raw_plan_waves_json(s, T, part_off, part_id, rep_off, cur, stride, new_len, new, weight, B, names, name_off, js, json_cap, doc_off,
                        wave, summary, cap, n=None):
    """ka_plan_waves_json through ctypes: (rc, status, W)."""
    st = kab.KaStatus()
    n = ctypes.c_int32(-7) if n is None else n
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = s._L.ka_plan_waves_json(s._h, T, p(part_off), p(part_id), p(rep_off), p(cur), stride, p(new_len), p(new), p(weight), B,
                                 p(names), p(name_off), p(js), json_cap, p(doc_off), p(wave),
                                 ctypes.byref(n) if n is not False else None, p(summary), cap, ctypes.byref(st))
    return rc, st, n
