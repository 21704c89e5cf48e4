"""ka_solve_clusters_json without a device: the symbol is exported and declared, a NULL context is KA_ERR_NO_DEVICE for every
cluster, st is required, and Solver.solve_clusters_json lays a fleet and its names out as the C ABI takes them and slices the
documents back out (checked against a hand-built layout, the library call mocked)."""
import ctypes
import os

import numpy as np

import kafka_assigner_b200 as kab
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbol_is_exported_and_declared(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    assert hasattr(raw, "ka_solve_clusters_json") and "ka_solve_clusters_json" in kab._native.SYMBOLS
    with open(os.path.join(ROOT, "include", "kassign.h")) as f:
        assert "int32_t ka_solve_clusters_json(ka_ctx* ctx, int32_t K," in f.read()
    assert len(kab._native.SYMBOLS["ka_solve_clusters_json"][1]) == 18


def test_without_a_context_is_no_device(native_lib):
    st = (kab.KaStatus * 3)()
    cand_off = np.array([0, 1, 2, 2], dtype=np.int32)
    ids = np.array([1, 2], dtype=np.int32)
    racks = np.zeros(2, dtype=np.int32)
    topic_off = np.zeros(4, dtype=np.int32)
    json_off = np.full(4, 9, dtype=np.int64)
    buf = ctypes.create_string_buffer(64)
    vp = ctypes.c_void_p
    rc = native_lib.ka_solve_clusters_json(None, 3, cand_off.ctypes.data_as(vp), ids.ctypes.data_as(vp), racks.ctypes.data_as(vp),
                                           topic_off.ctypes.data_as(vp), None, None, None, None, None, None, None, None, buf, 64,
                                           json_off.ctypes.data_as(vp), st)
    assert rc == kab._native.KA_ERR_NO_DEVICE
    assert [st[k].code for k in range(3)] == [kab._native.KA_ERR_NO_DEVICE] * 3
    assert not json_off.any()
    assert native_lib.ka_solve_clusters_json(None, 1, None, None, None, None, None, None, None, None, None, None, None, None, buf, 64,
                                             json_off.ctypes.data_as(vp), None) == kab._native.KA_ERR_BAD_ARG   # st is required


class _FakeLib:
    """Stands in for libkassign.so: records what ka_solve_clusters_json is handed and writes one recognisable document per
    cluster (none for a failed one)."""

    def __init__(self):
        self.seen = None

    def ka_solve_clusters_json(self, h, K, cand_off, ids, racks, topic_off, drf, th, part_off, part_id, rep_off, cur, names, name_off,
                               json, json_cap, json_off, st):
        c_off = util.view(cand_off, K + 1, np.int32)
        t_off = util.view(topic_off, K + 1, np.int32)
        T = int(t_off[-1])
        p_off = util.view(part_off, T + 1, np.int64)
        Q = int(p_off[-1])
        r_off = util.view(rep_off, Q + 1, np.int64)
        n_off = util.view(name_off, T + 1, np.int64)
        self.seen = dict(K=K, cap=json_cap, cand_off=c_off, topic_off=t_off, desired_rf=util.view(drf, K, np.int32), topic_hash=util.view(th, T, np.int32),
                         part_off=p_off, part_id=util.view(part_id, Q, np.int32), rep_off=r_off, cur=util.view(cur, int(r_off[-1]), np.int32),
                         name_off=n_off, names=bytes(util.view(names, int(n_off[-1]), np.uint8)))
        buf = np.ctypeslib.as_array(ctypes.cast(json, ctypes.POINTER(ctypes.c_uint8)), shape=(json_cap,))
        offs = np.ctypeslib.as_array(ctypes.cast(json_off, ctypes.POINTER(ctypes.c_int64)), shape=(K + 1,))
        offs[0] = 0
        for k in range(K):
            doc = b"" if k == 1 else ("<doc %d>" % k).encode()
            buf[offs[k]:offs[k] + len(doc)] = np.frombuffer(doc, dtype=np.uint8)
            offs[k + 1] = offs[k] + len(doc)
            st[k].code, st[k].topic_index = (3 if k == 1 else 0), k
        return 3


def test_solve_clusters_json_marshals_the_layout_and_names():
    a = (np.array([1, 2, 3], np.int32), np.array([0, 0, 1], np.int32), np.array([11, 12], np.int32), np.array([0, 2, 3], np.int64),
         np.array([4, 7, 0], np.int32), np.array([0, 2, 4, 5], np.int64), np.array([1, 2, 2, 3, 1], np.int32), -1)
    empty = (np.array([9], np.int32), np.array([0], np.int32), np.zeros(0, np.int32), np.array([0], np.int64), None,
             np.array([0], np.int64), np.zeros(0, np.int32), 2)
    b = (np.array([5, 6], np.int32), np.array([0, 1], np.int32), np.array([21], np.int32), np.array([0, 2], np.int64), None,
         np.array([0, 3, 6], np.int64), np.array([5, 6, 7, 6, 5, 7], np.int32), 3)
    s = util.fake_solver(_FakeLib())
    res = s.solve_clusters_json([a, empty, b], [["alpha", "be"], [], ["c.d"]])
    got = s._L.seen
    assert got["K"] == 3
    assert got["cand_off"].tolist() == [0, 3, 4, 6] and got["topic_off"].tolist() == [0, 2, 2, 3]
    assert got["desired_rf"].tolist() == [-1, 2, 3] and got["topic_hash"].tolist() == [11, 12, 21]
    assert got["part_off"].tolist() == [0, 2, 3, 5] and got["part_id"].tolist() == [4, 7, 0, 0, 1]
    assert got["rep_off"].tolist() == [0, 2, 4, 5, 8, 11] and got["cur"].tolist() == [1, 2, 2, 3, 1, 5, 6, 7, 6, 5, 7]
    # one name slab over all topics, in input order
    assert got["names"] == b"alphabec.d" and got["name_off"].tolist() == [0, 5, 7, 10]
    # the documented sufficient size: per cluster 64 + per row (50 + 12 x its width + the row's name length)
    assert got["cap"] == (64 + 2 * (50 + 12 * 2 + 5) + 1 * (50 + 12 * 2 + 2)) + (64) + (64 + 2 * (50 + 12 * 3 + 3))
    assert [bytes(t) for t, _ in res] == [b"<doc 0>", b"", b"<doc 2>"]
    assert [st.code for _, st in res] == [0, 3, 0] and [st.topic_index for _, st in res] == [0, 1, 2]


def test_solve_clusters_json_takes_a_buffer():
    c = (np.array([1, 2], np.int32), np.array([0, 1], np.int32), np.array([5], np.int32), np.array([0, 1], np.int64), None,
         np.array([0, 1], np.int64), np.array([2], np.int32), -1)
    s = util.fake_solver(_FakeLib())
    buf = np.zeros(100, dtype=np.uint8)
    res = s.solve_clusters_json([c, c, c], [["x"], ["y"], ["z"]], json_buf=buf)
    assert s._L.seen["cap"] == 100 and bytes(buf[:7]) == b"<doc 0>"
    assert [bytes(t) for t, _ in res] == [b"<doc 0>", b"", b"<doc 2>"]
