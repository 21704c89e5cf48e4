"""Every cluster's reassignment JSON for a fleet of independent real-cluster-shaped (ragged) clusters, each with its own broker
table: (a) K sequential ka_solve_json calls against (b) one ka_solve_clusters_json call, with one ka_solve_clusters (rows only,
no text) beside them as the floor. All buffers on the host. The fleets of cluster_batch_times.py: K = 8 and K = 32
make_ragged_cluster clusters of 30 k topics each; a skewed fleet, one 240 k-topic cluster and 31 of 2 k topics; K = 128 tiny
clusters of 40 topics.

The contexts and buffers are made before the timed window. A sequential step is, per cluster, ka_ctx_reset (a fresh Context) +
ka_ctx_set_brokers + ka_solve_json; a batched step is one call over the fleet's layout, marshalled once beforehand. Every call is
synchronous and timed with the host clock, the L2 flushed (256 MiB written) before every step; the median of --steps steps after
--warmup warm-up steps. The statuses of the two JSON arms, and the text of every cluster, are checked equal first. Prints the
GPU, its power limit and SM clock, and a markdown table."""
import argparse
import ctypes
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

import kafka_assigner_b200 as kab  # noqa: E402
from tests.tools.cluster_batch_times import gpu_info  # noqa: E402


def _vp(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def measure(name, clusters, steps, warmup):
    """clusters: synth.RaggedCluster list, each solved against its own live table, rows of 3 replicas at most."""
    K = len(clusters)
    S = max(int(np.diff(c.rep_off).max()) for c in clusters)
    entries = [(c.broker_id, c.rack_index, c.topic_hash, c.part_off, c.part_id, c.rep_off, c.cur, -1) for c in clusters]
    cand_off, broker_id, broker_rack, topic_off, drf, th, part_off, part_id, rep_off, cur = kab.Solver.marshal_clusters(entries)
    names, name_off = kab.Solver.marshal_names([n for c in clusters for n in c.topic_names])
    Q = int(part_off[-1])
    # the documented sufficient sizes: per cluster for (a), their sum for (b)
    own = []
    for c in clusters:
        nm, noff = kab.Solver.marshal_names(c.topic_names)
        Sk = max(int(np.diff(c.rep_off).max()), 1)
        cap = 64 + c.Q * (50 + 12 * Sk) + int(np.dot(np.diff(c.part_off), np.diff(noff)))
        own.append(tuple(np.ascontiguousarray(a) for a in (c.broker_id, c.rack_index, c.topic_hash, c.part_off, c.part_id, c.rep_off,
                                                          c.cur, nm, noff)) + (np.empty(cap, dtype=np.uint8),))
    bat_json = np.empty(sum(o[-1].size for o in own), dtype=np.uint8)
    json_off = np.zeros(K + 1, dtype=np.int64)
    seq_bytes = [ctypes.c_int64(0) for _ in clusters]
    rows_out = np.empty((Q, S), dtype=np.int32)
    rows_len = np.empty(Q, dtype=np.int32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    solvers = [kab.Solver(0) for _ in clusters]
    batch = kab.Solver(0)
    L = batch._L
    seq_st, sts, row_st = (kab.KaStatus * K)(), (kab.KaStatus * K)(), (kab.KaStatus * K)()
    key = lambda st: (st.code, st.topic_index, st.partition, st.a, st.b)  # noqa: E731

    def sequential():
        for k, (s, (ids, racks, h, po, pid, ro, cr, nm, noff, buf)) in enumerate(zip(solvers, own)):
            assert L.ka_ctx_reset(s._h) == 0
            assert L.ka_ctx_set_brokers(s._h, len(ids), _vp(ids), _vp(racks)) == 0
            L.ka_solve_json(s._h, len(h), _vp(h), _vp(po), _vp(pid), _vp(ro), _vp(cr), -1, _vp(nm), _vp(noff), _vp(buf), buf.size,
                            ctypes.byref(seq_bytes[k]), ctypes.byref(seq_st[k]))

    def batched():
        L.ka_solve_clusters_json(batch._h, K, _vp(cand_off), _vp(broker_id), _vp(broker_rack), _vp(topic_off), _vp(drf), _vp(th),
                                 _vp(part_off), _vp(part_id), _vp(rep_off), _vp(cur), _vp(names), _vp(name_off), _vp(bat_json),
                                 bat_json.size, _vp(json_off), sts)

    def rows_only():
        L.ka_solve_clusters(batch._h, K, _vp(cand_off), _vp(broker_id), _vp(broker_rack), _vp(topic_off), _vp(drf), _vp(th),
                            _vp(part_off), _vp(part_id), _vp(rep_off), _vp(cur), S, _vp(rows_len), _vp(rows_out), row_st)

    def timed(fn):
        ms = []
        for i in range(warmup + steps):
            flush.fill_(i & 0xFF)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            t1 = time.perf_counter()
            if i >= warmup:
                ms.append((t1 - t0) * 1e3)
        return float(np.median(ms))

    sequential()
    batched()
    assert [key(sts[k]) for k in range(K)] == [key(seq_st[k]) for k in range(K)], name + ": statuses differ"
    for k in range(K):
        assert bytes(bat_json[json_off[k]:json_off[k + 1]]) == bytes(own[k][-1][:seq_bytes[k].value]), name + ": text differs"
    ok = sum(seq_st[k].code == 0 for k in range(K))
    t_seq, t_bat, t_rows = timed(sequential), timed(batched), timed(rows_only)
    print("| %s | %d | %d | %d | %.1f | %.2f | %.2f | %.2f | %.2fx |" % (name, K, Q, ok, json_off[-1] / 1e6, t_seq, t_bat, t_rows,
                                                                        t_seq / t_bat), flush=True)
    for s in solvers + [batch]:
        s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    mk = kab.synth.make_ragged_cluster
    print("GPU:", gpu_info())
    print("| fleet | K | partitions | clusters solved | text, MB | (a) K sequential ka_solve_json, ms "
          "| (b) one ka_solve_clusters_json, ms | ka_solve_clusters (rows only), ms | (a)/(b) |")
    print("|---|---|---|---|---|---|---|---|---|")
    for K in (8, 32):
        measure("%d x 30 k topics" % K, [mk(T=30000, N=400, max_partitions=128, seed=100 + k) for k in range(K)], args.steps,
                args.warmup)
    measure("skewed: 240 k + 31 x 2 k topics",
            [mk(T=240000, N=400, max_partitions=128, seed=11)] + [mk(T=2000, N=100, max_partitions=128, seed=200 + k) for k in range(31)],
            args.steps, args.warmup)
    measure("128 tiny clusters, 40 topics", [mk(T=40, N=24, R=4, max_partitions=32, seed=300 + k) for k in range(128)], args.steps,
            args.warmup)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
