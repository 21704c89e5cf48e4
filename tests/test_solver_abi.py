"""What the Python Solver hands the C ABI, without a device: the library is a fake object that records every argument and writes
recognisable rows, texts and statuses. Pins the arrays, the row stride, the JSON buffer size, K and the sliced results of the
single, JSON, candidate and score calls, generate_assignment's stride, and the return contract of the device-pointer calls."""

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import assigner
from tests import util

I32, I64 = np.int32, np.int64


def _ragged(th, part_off, part_id, rep_off, cur, T):
    p_off = util.view(part_off, T + 1, I64)
    Q = int(p_off[-1])
    r_off = util.view(rep_off, Q + 1, I64)
    return dict(T=T, topic_hash=util.view(th, T, I32), part_off=p_off, part_id=util.view(part_id, Q, I32), rep_off=r_off,
                cur=util.view(cur, int(r_off[-1]), I32)), Q


class _FakeLib:
    """Stands in for libkassign.so. Rows are 0, 1, 2, ... in order, list lengths (g % 4) per row, statuses code 3 for member 1
    (or `code` for a single call); `rc` is what every call returns."""

    def __init__(self, code=0, rc=0):
        self.code, self.rc, self.seen = code, rc, {}

    def _rows(self, out, out_len, n, S):
        if out is not None:
            util.writable(out, n * S, I32)[:] = np.arange(n * S, dtype=I32)
        if out_len is not None:
            util.writable(out_len, n, I32)[:] = np.arange(n, dtype=I32) % 4

    def _status(self, st):
        st._obj.code, st._obj.topic_index = self.code, 1

    def _statuses(self, st, K):
        for k in range(K):
            st[k].code, st[k].topic_index = (3 if k == 1 else 0), k

    def _text(self, json, cap, nbytes, doc=b"<doc>"):
        util.writable(json, cap, np.uint8)[:len(doc)] = np.frombuffer(doc, dtype=np.uint8)
        nbytes._obj.value = len(doc)

    def ka_solve_dense_json(self, h, T, th, P, RF, cur, drf, names, name_off, json, cap, nbytes, st):
        n_off = util.view(name_off, T + 1, I64)
        self.seen = dict(T=T, P=P, RF=RF, topic_hash=util.view(th, T, I32), cur=util.view(cur, T * P * RF, I32), desired_rf=drf,
                         name_off=n_off, names=bytes(util.view(names, int(n_off[-1]), np.uint8)), cap=cap)
        self._text(json, cap, nbytes)
        self._status(st)
        return self.rc

    def ka_solve(self, h, T, th, part_off, part_id, rep_off, cur, drf, S, out_len, out, st):
        self.seen, Q = _ragged(th, part_off, part_id, rep_off, cur, T)
        self.seen.update(desired_rf=drf, S=S)
        self._rows(out, out_len, Q, S)
        self._status(st)
        return self.rc

    def ka_solve_json(self, h, T, th, part_off, part_id, rep_off, cur, drf, names, name_off, json, cap, nbytes, st):
        self.seen, Q = _ragged(th, part_off, part_id, rep_off, cur, T)
        n_off = util.view(name_off, T + 1, I64)
        self.seen.update(desired_rf=drf, name_off=n_off, names=bytes(util.view(names, int(n_off[-1]), np.uint8)), cap=cap)
        self._text(json, cap, nbytes)
        self._status(st)
        return self.rc

    def _tables(self, K, cand_off, ids, racks):
        c_off = util.view(cand_off, K + 1, I32)
        return dict(K=K, cand_off=c_off, broker_id=util.view(ids, int(c_off[-1]), I32), broker_rack=util.view(racks, int(c_off[-1]), I32))

    def ka_solve_candidates(self, h, K, cand_off, ids, racks, T, th, part_off, part_id, rep_off, cur, drf, S, out_len, out, st):
        self.seen, Q = _ragged(th, part_off, part_id, rep_off, cur, T)
        self.seen.update(self._tables(K, cand_off, ids, racks), desired_rf=drf, S=S)
        self._rows(out, out_len, K * Q, S)
        self._statuses(st, K)
        return self.rc

    def ka_score_candidates(self, h, K, cand_off, ids, racks, T, th, part_off, part_id, rep_off, cur, drf, S, weight, summary,
                            b_rep, b_lead, b_in, out_len, out, st):
        self.seen, Q = _ragged(th, part_off, part_id, rep_off, cur, T)
        self.seen.update(self._tables(K, cand_off, ids, racks), desired_rf=drf, S=S, weight=util.view(weight, Q, I64),
                         per_broker=[b is not None for b in (b_rep, b_lead, b_in)], rows=out is not None)
        sm = util.writable(summary, K * len(assigner.MOVE_SUMMARY_DTYPE.names), I64).reshape(K, -1)
        sm[:, 0] = 100 + np.arange(K)                                            # rows_changed
        nb = int(self.seen["cand_off"][-1])
        for i, b in enumerate((b_rep, b_lead, b_in)):
            if b is not None:
                util.writable(b, nb, I64)[:] = 10 * (i + 1) + np.arange(nb)
        self._rows(out, out_len, K * Q, S)
        self._statuses(st, K)
        return self.rc

    def ka_rack_indices(self, n, ids, names, racks):
        self.brokers = util.view(ids, n, I32).tolist()
        util.writable(racks, n, I32)[:] = 0
        return 0

    def ka_ctx_set_brokers(self, h, n, ids, racks):
        return 0

    def ka_solve_dense_device(self, h, T, th, P, RF, cur, drf, S, out_len, out, stream, st):
        self.seen = dict(args=(T, th.value, P, RF, cur.value, drf, S, out_len and out_len.value, out.value,
                               stream and stream.value), st=st is not None)
        if st is not None:
            self._status(st)
        return self.rc

    def ka_order_device(self, h, out_len, out, stream, st):
        self.seen = dict(args=(out_len and out_len.value, out.value, stream and stream.value), st=st is not None)
        if st is not None:
            self._status(st)
        return self.rc

    ka_emit_device = ka_order_device

    def ka_ctx_set_topic_base(self, h, base):
        return self.rc


# two topics of a ragged cluster: lists of 2, 3 and 1 replicas, partition ids 4, 7, 0
RAGGED = ([11, 12], [0, 2, 3], [4, 7, 0], [0, 2, 5, 6], [1, 2, 2, 3, 1, 4])
TABLES = [(np.array([1, 2, 3], I32), np.array([0, 0, 1], I32)), (np.array([4], I32), np.array([0], I32)),
          (np.array([5, 6], I32), np.array([0, 1], I32))]


def _check_ragged(got):
    assert got["T"] == 2 and got["topic_hash"].tolist() == [11, 12]
    assert got["part_off"].tolist() == [0, 2, 3] and got["part_id"].tolist() == [4, 7, 0]
    assert got["rep_off"].tolist() == [0, 2, 5, 6] and got["cur"].tolist() == [1, 2, 2, 3, 1, 4]


def _check_tables(got):
    assert got["K"] == 3 and got["cand_off"].tolist() == [0, 3, 4, 6]
    assert got["broker_id"].tolist() == [1, 2, 3, 4, 5, 6] and got["broker_rack"].tolist() == [0, 0, 1, 0, 0, 1]


@pytest.mark.parametrize("desired_rf, S", [(-1, 2), (1, 2), (3, 3)])
def test_solve_dense_json_marshals_names_and_the_sufficient_buffer(desired_rf, S):
    s = util.fake_solver(_FakeLib())
    cur = np.arange(12).reshape(2, 3, 2)                                     # T = 2, P = 3, RF = 2 (int64: coerced to int32)
    text, st = s.solve_dense_json(["ab", "cde"], [5, 6], cur, desired_rf)
    got = s._L.seen
    assert (got["T"], got["P"], got["RF"], got["desired_rf"]) == (2, 3, 2, desired_rf)
    assert got["topic_hash"].tolist() == [5, 6] and got["cur"].tolist() == list(range(12))
    assert got["names"] == b"abcde" and got["name_off"].tolist() == [0, 2, 5]
    # the documented sufficient size: 64 + T·P rows of (50 + 12·S) + P × all name bytes
    assert got["cap"] == 64 + 6 * (50 + 12 * S) + 3 * 5
    assert bytes(text) == b"<doc>" and st.code == 0


def test_solve_dense_json_takes_a_buffer_and_a_name_slab():
    s = util.fake_solver(_FakeLib(code=kab._native.KA_ERR_RF_MISMATCH))
    buf = np.zeros(40, dtype=np.uint8)
    slab = kab.Solver.marshal_names(["x", "yz"])
    text, st = s.solve_dense_json(None, [5, 6], np.ones((2, 1, 1), I32), -1, json_buf=buf, check=False, names_slab=slab)
    assert s._L.seen["cap"] == 40 and s._L.seen["names"] == b"xyz" and bytes(buf[:5]) == b"<doc>"
    assert bytes(text) == b"<doc>" and st.code == kab._native.KA_ERR_RF_MISMATCH
    with pytest.raises(kab.IllegalStateException, match="Topic yz has partition"):
        s.solve_dense_json(["x", "yz"], [5, 6], np.ones((2, 1, 1), I32), -1, json_buf=buf)


@pytest.mark.parametrize("desired_rf, S", [(-1, 3), (2, 3), (4, 4)])
def test_solve_ragged_json_marshals_the_layout_and_the_sufficient_buffer(desired_rf, S):
    s = util.fake_solver(_FakeLib())
    text, st = s.solve_ragged_json(["alpha", "be"], *RAGGED, desired_rf)
    got = s._L.seen
    _check_ragged(got)
    assert got["desired_rf"] == desired_rf and got["names"] == b"alphabe" and got["name_off"].tolist() == [0, 5, 7]
    # 64 + ΣP rows of (50 + 12·S) + every row's own name length
    assert got["cap"] == 64 + 3 * (50 + 12 * S) + 2 * 5 + 1 * 2
    assert bytes(text) == b"<doc>" and st.code == 0


def test_solve_ragged_json_without_ids_or_topics():
    s = util.fake_solver(_FakeLib())
    s.solve_ragged_json([], [], [0], None, [0], [], -1)
    assert s._L.seen["part_id"] is None and s._L.seen["cap"] == 64
    buf = np.zeros(30, dtype=np.uint8)
    text, _ = s.solve_ragged_json(["alpha", "be"], *RAGGED, -1, json_buf=buf)
    assert s._L.seen["cap"] == 30 and bytes(text) == b"<doc>"


def test_solve_ragged_passes_the_stride_and_slices_nothing():
    s = util.fake_solver(_FakeLib())
    out, ln, st = s.solve_ragged(*RAGGED, -1, 4)
    _check_ragged(s._L.seen)
    assert s._L.seen["S"] == 4 and out.shape == (3, 4) and out[2].tolist() == [8, 9, 10, 11] and ln.tolist() == [0, 1, 2]


@pytest.mark.parametrize("desired_rf, out_stride, S", [(-1, None, 3), (4, None, 4), (-1, 2, 2)])
def test_solve_ragged_candidates_marshals_tables_and_slices_rows(desired_rf, out_stride, S):
    s = util.fake_solver(_FakeLib())
    out, ln, st = s.solve_ragged_candidates(TABLES, *RAGGED, desired_rf, out_stride)
    got = s._L.seen
    _check_ragged(got)
    _check_tables(got)
    assert got["desired_rf"] == desired_rf and got["S"] == S
    assert out.shape == (3, 3, S) and ln.shape == (3, 3)
    assert out[1, 0].tolist() == list(range(3 * S, 4 * S)) and ln[2].tolist() == [2, 3, 0]
    assert [x.code for x in st] == [0, 3, 0] and [x.topic_index for x in st] == [0, 1, 2]


def test_solve_ragged_candidates_without_tables():
    s = util.fake_solver(_FakeLib())
    out, ln, st = s.solve_ragged_candidates([], *RAGGED, -1)
    assert s._L.seen["K"] == 0 and s._L.seen["cand_off"].tolist() == [0]
    assert out.shape == (0, 3, 3) and ln.shape == (0, 3) and st == []


@pytest.mark.parametrize("rows, per_broker", [(False, False), (True, False), (False, True), (True, True)])
def test_score_ragged_candidates_marshals_and_returns_what_was_asked(rows, per_broker):
    s = util.fake_solver(_FakeLib())
    res = s.score_ragged_candidates(TABLES, *RAGGED, -1, weight=[5, 6, 7], rows=rows, per_broker=per_broker)
    got = s._L.seen
    _check_ragged(got)
    _check_tables(got)
    assert got["S"] == 3 and got["weight"].tolist() == [5, 6, 7]
    assert got["rows"] == rows and got["per_broker"] == [per_broker] * 3
    assert len(res) == 2 + 2 * rows + 3 * per_broker
    summary, st = res[:2]
    assert summary.dtype == assigner.MOVE_SUMMARY_DTYPE and summary["rows_changed"].tolist() == [100, 101, 102]
    assert [x.code for x in st] == [0, 3, 0]
    if rows:
        out, ln = res[2:4]
        assert out.shape == (3, 3, 3) and out[2, 2].tolist() == [24, 25, 26] and ln.shape == (3, 3)
    if per_broker:
        rep, lead, add = res[-3:]
        assert [a.tolist() for a in rep] == [[10, 11, 12], [13], [14, 15]]
        assert [a.tolist() for a in lead] == [[20, 21, 22], [23], [24, 25]]
        assert [a.tolist() for a in add] == [[30, 31, 32], [33], [34, 35]]


def test_score_ragged_candidates_default_weight_and_stride():
    s = util.fake_solver(_FakeLib())
    s.score_ragged_candidates(TABLES, *RAGGED, 4, out_stride=None)
    assert s._L.seen["weight"] is None and s._L.seen["S"] == 4
    s.score_ragged_candidates(TABLES, *RAGGED, -1, out_stride=2)
    assert s._L.seen["S"] == 2


@pytest.mark.parametrize("current, desired_rf, S", [({0: [1, 2], 3: [2, 3, 1]}, -1, 3), ({0: [1, 2], 3: [2, 3, 1]}, 4, 4),
                                                    ({0: [1], 1: [2]}, 2, 2), ({}, -1, 1)])
def test_generate_assignment_stride(monkeypatch, current, desired_rf, S):
    monkeypatch.setattr(assigner, "java_string_hash", lambda s: 77)
    kta = object.__new__(kab.KafkaTopicAssigner)
    kta._solver, kta._brokers_key = util.fake_solver(_FakeLib()), None
    res = kta.generate_assignment("t", current, {3, 1, 2}, {}, desired_rf)
    got = kta._solver._L.seen
    assert kta._solver._L.brokers == [1, 2, 3]
    assert got["S"] == S and got["desired_rf"] == desired_rf and got["topic_hash"].tolist() == [77]
    assert got["part_off"].tolist() == [0, len(current)] and got["part_id"].tolist() == sorted(current)
    assert got["cur"].tolist() == [b for p in sorted(current) for b in current[p]]
    assert res == {p: list(range(i * S, i * S + i % 4)) for i, p in enumerate(sorted(current))}


_DEVICE_CALLS = [
    ("solve_dense_device", (2, 0x100, 3, 2, 0x200, -1, 3, 0x300, 0x400), (2, 0x100, 3, 2, 0x200, -1, 3, 0x300, 0x400),
     (2, 0x100, 3, 2, 0x200, -1, 3, 0, 0x400), (2, 0x100, 3, 2, 0x200, -1, 3, None, 0x400)),
    ("order_device", (0x300, 0x400), (0x300, 0x400), (0, 0x400), (None, 0x400)),
    ("emit_device", (0x300, 0x400), (0x300, 0x400), (0, 0x400), (None, 0x400)),
]


@pytest.mark.parametrize("name, args, passed, args0, passed0", _DEVICE_CALLS)
def test_device_calls_sync_contract(name, args, passed, args0, passed0):
    s = util.fake_solver(_FakeLib(code=4, rc=-2))
    st = getattr(s, name)(*args, stream=0x500)                              # sync: the status, never a raise
    assert s._L.seen == dict(args=passed + (0x500,), st=True) and st.code == 4
    with pytest.raises(kab.KassignError) as e:                              # async: rc raises, no status
        getattr(s, name)(*args0, sync=False)
    assert e.value.code == -2 and s._L.seen == dict(args=passed0 + (None,), st=False)
    s._L.rc = 0
    assert getattr(s, name)(*args, sync=False) is None


def test_nonzero_rc_raises():
    s = util.fake_solver(_FakeLib(rc=-1))
    with pytest.raises(kab.KassignError) as e:
        s.set_topic_base(3)
    assert e.value.code == -1
    s._L.rc = 0
    s.set_topic_base(3)
