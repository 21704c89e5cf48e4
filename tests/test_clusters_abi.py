"""ka_solve_clusters without a device: the symbol is exported and declared, a NULL context is KA_ERR_NO_DEVICE for every cluster,
and Solver.solve_clusters lays a fleet out as the C ABI takes it (checked against a hand-built layout, the library call mocked)."""
import ctypes
import os

import numpy as np

import kafka_assigner_b200 as kab
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbol_is_exported_and_declared(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    assert hasattr(raw, "ka_solve_clusters") and "ka_solve_clusters" in kab._native.SYMBOLS
    with open(os.path.join(ROOT, "include", "kassign.h")) as f:
        assert "int32_t ka_solve_clusters(ka_ctx* ctx, int32_t K," in f.read()
    assert len(kab._native.SYMBOLS["ka_solve_clusters"][1]) == 16


def test_clusters_without_a_context_is_no_device(native_lib):
    st = (kab.KaStatus * 3)()
    cand_off = np.array([0, 1, 2, 2], dtype=np.int32)
    ids = np.array([1, 2], dtype=np.int32)
    racks = np.zeros(2, dtype=np.int32)
    topic_off = np.zeros(4, dtype=np.int32)
    vp = ctypes.c_void_p
    rc = native_lib.ka_solve_clusters(None, 3, cand_off.ctypes.data_as(vp), ids.ctypes.data_as(vp), racks.ctypes.data_as(vp),
                                      topic_off.ctypes.data_as(vp), None, None, None, None, None, None, 1, None, None, st)
    assert rc == kab._native.KA_ERR_NO_DEVICE
    assert [st[k].code for k in range(3)] == [kab._native.KA_ERR_NO_DEVICE] * 3
    assert native_lib.ka_solve_clusters(None, 1, None, None, None, None, None, None, None, None, None, None, 1, None, None,
                                        None) == kab._native.KA_ERR_BAD_ARG   # st is required


class _FakeLib:
    """Stands in for libkassign.so: records what ka_solve_clusters is handed and writes recognisable rows and statuses."""

    def __init__(self):
        self.seen = None

    def ka_solve_clusters(self, h, K, cand_off, ids, racks, topic_off, drf, th, part_off, part_id, rep_off, cur, S, out_len, out, st):
        c_off = util.view(cand_off, K + 1, np.int32)
        t_off = util.view(topic_off, K + 1, np.int32)
        T = int(t_off[-1])
        p_off = util.view(part_off, T + 1, np.int64)
        Q = int(p_off[-1])
        r_off = util.view(rep_off, Q + 1, np.int64)
        self.seen = dict(K=K, S=S, cand_off=c_off, broker_id=util.view(ids, int(c_off[-1]), np.int32),
                         broker_rack=util.view(racks, int(c_off[-1]), np.int32), topic_off=t_off, desired_rf=util.view(drf, K, np.int32),
                         topic_hash=util.view(th, T, np.int32), part_off=p_off, part_id=util.view(part_id, Q, np.int32), rep_off=r_off,
                         cur=util.view(cur, int(r_off[-1]), np.int32))
        rows = np.ctypeslib.as_array(ctypes.cast(out, ctypes.POINTER(ctypes.c_int32)), shape=(Q * S,))
        rows[:] = np.arange(Q * S, dtype=np.int32)
        lens = np.ctypeslib.as_array(ctypes.cast(out_len, ctypes.POINTER(ctypes.c_int32)), shape=(Q,))
        lens[:] = np.arange(Q, dtype=np.int32) % 4
        for k in range(K):
            st[k].code, st[k].topic_index = (3 if k == 1 else 0), k
        return 3


def test_solve_clusters_marshals_the_shared_layout():
    a = (np.array([1, 2, 3], np.int32), np.array([0, 0, 1], np.int32), np.array([11, 12], np.int32), np.array([0, 2, 3], np.int64),
         np.array([4, 7, 0], np.int32), np.array([0, 2, 4, 5], np.int64), np.array([1, 2, 2, 3, 1], np.int32), -1)
    empty = (np.array([9], np.int32), np.array([0], np.int32), np.zeros(0, np.int32), np.array([0], np.int64), None,
             np.array([0], np.int64), np.zeros(0, np.int32), 2)
    b = (np.array([5, 6], np.int32), np.array([0, 1], np.int32), np.array([21], np.int32), np.array([0, 2], np.int64), None,
         np.array([0, 3, 6], np.int64), np.array([5, 6, 7, 6, 5, 7], np.int32), 3)
    s = util.fake_solver(_FakeLib())
    res = s.solve_clusters([a, empty, b])
    got = s._L.seen
    # by hand: the three clusters one after the other, offsets continued from where the previous cluster ends
    assert got["K"] == 3 and got["S"] == 3                                # longest list 3, desired RF up to 3
    assert got["cand_off"].tolist() == [0, 3, 4, 6]
    assert got["broker_id"].tolist() == [1, 2, 3, 9, 5, 6] and got["broker_rack"].tolist() == [0, 0, 1, 0, 0, 1]
    assert got["topic_off"].tolist() == [0, 2, 2, 3]
    assert got["desired_rf"].tolist() == [-1, 2, 3]
    assert got["topic_hash"].tolist() == [11, 12, 21]
    assert got["part_off"].tolist() == [0, 2, 3, 5]
    assert got["part_id"].tolist() == [4, 7, 0, 0, 1]                    # cluster b without ids: ordinals
    assert got["rep_off"].tolist() == [0, 2, 4, 5, 8, 11]
    assert got["cur"].tolist() == [1, 2, 2, 3, 1, 5, 6, 7, 6, 5, 7]
    # rows come back per cluster, in place
    assert [r[0].shape for r in res] == [(3, 3), (0, 3), (2, 3)]
    assert res[2][0].tolist() == [[9, 10, 11], [12, 13, 14]] and res[2][1].tolist() == [3, 0]
    assert [r[2].code for r in res] == [0, 3, 0] and [r[2].topic_index for r in res] == [0, 1, 2]


def test_solve_clusters_takes_an_explicit_stride():
    c = (np.array([1, 2], np.int32), np.array([0, 1], np.int32), np.array([5], np.int32), np.array([0, 1], np.int64), None,
         np.array([0, 1], np.int64), np.array([2], np.int32), -1)
    s = util.fake_solver(_FakeLib())
    out, ln, st = s.solve_clusters([c, c], out_stride=2)[1]
    assert s._L.seen["S"] == 2 and out.shape == (1, 2)
    assert s._L.seen["part_off"].tolist() == [0, 1, 2] and s._L.seen["rep_off"].tolist() == [0, 1, 2]
