"""Scoring every cluster of a fleet (data moved and broker balance per cluster) before its documents go out: what it costs to
get each cluster's ka_move_summary. The fleets of cluster_batch_times.py: K = 8 and K = 32 make_ragged_cluster clusters of 30 k
topics each; a skewed fleet, one 240 k-topic cluster and 31 of 2 k topics; K = 128 tiny clusters of 40 topics. A seeded random
weight per partition. Arms, all buffers on the host:

  (a) ka_solve_clusters (every cluster's rows and list lengths copied back) + the numpy summary of
      tests/models.py per cluster on the host; in brackets, the ka_solve_clusters call alone;
  (b) ka_score_clusters without rows (K summaries come back);
  (c) ka_score_clusters with rows (the summaries and the rows of (a)).

Every step is synchronous and timed with the host clock, the L2 flushed (256 MiB written) before it; the median of --steps
steps after --warmup warm-up steps. Before timing, the statuses, summaries and per-broker arrays of the three arms, and the rows
of (a) and (c), are checked equal. Prints the GPU, its power limit and SM clock, and a markdown table."""
import argparse
import ctypes
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

import kafka_assigner_b200 as kab  # noqa: E402
from kafka_assigner_b200.assigner import MOVE_SUMMARY_DTYPE  # noqa: E402
from tests import models  # noqa: E402
from tests.tools.cluster_batch_times import gpu_info  # noqa: E402


def _vp(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def measure(name, clusters, steps, warmup, seed):
    """clusters: synth.RaggedCluster list, each solved against its own live table, rows of 3 replicas at most."""
    K = len(clusters)
    S = max(int(np.diff(c.rep_off).max()) for c in clusters)
    entries = [(c.broker_id, c.rack_index, c.topic_hash, c.part_off, c.part_id, c.rep_off, c.cur, -1) for c in clusters]
    cand_off, broker_id, broker_rack, topic_off, drf, th, part_off, part_id, rep_off, cur = kab.Solver.marshal_clusters(entries)
    Q, nb = int(part_off[-1]), int(cand_off[-1])
    row0 = part_off[topic_off]
    weight = np.random.default_rng(seed).integers(1, 1 << 34, size=Q, dtype=np.int64)   # up to 16 GiB per partition
    out, out_c = np.empty((Q, S), dtype=np.int32), np.empty((Q, S), dtype=np.int32)
    out_len, len_c = np.empty(Q, dtype=np.int32), np.empty(Q, dtype=np.int32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    s = kab.Solver(0)
    L = s._L
    st_a, st_b, st_c = ((kab.KaStatus * K)() for _ in range(3))
    sum_a, sum_b, sum_c = (np.zeros(K, dtype=MOVE_SUMMARY_DTYPE) for _ in range(3))
    sum_a["max_broker_in_id"] = -1   # a failed cluster keeps the empty summary in (a) too
    brk_a, brk_b, brk_c = (np.zeros((3, nb), dtype=np.int64) for _ in range(3))
    key = lambda st: (st.code, st.topic_index, st.partition, st.a, st.b)  # noqa: E731
    head = (s._h, K, _vp(cand_off), _vp(broker_id), _vp(broker_rack), _vp(topic_off), _vp(drf), _vp(th), _vp(part_off), _vp(part_id),
            _vp(rep_off), _vp(cur), S)
    solve_ms = []

    def host_summary():
        t0 = time.perf_counter()
        L.ka_solve_clusters(*head, _vp(out_len), _vp(out), st_a)
        solve_ms.append((time.perf_counter() - t0) * 1e3)
        for k, c in enumerate(clusters):
            if st_a[k].code != 0:
                continue
            r0, r1 = row0[k], row0[k + 1]
            e, rep, lead, inb = models.move_summary(out[r0:r1], out_len[r0:r1], c.rep_off, c.cur, c.broker_id.astype(np.int64),
                                                    weight[r0:r1])
            for f, v in e.items():
                sum_a[k][f] = v
            for i, a in enumerate((rep, lead, inb)):
                brk_a[i, cand_off[k]:cand_off[k + 1]] = a

    def scored(summary, brk, st, rows):
        L.ka_score_clusters(*head, _vp(weight), _vp(summary), _vp(brk[0]), _vp(brk[1]), _vp(brk[2]), _vp(len_c) if rows else None,
                            _vp(out_c) if rows else None, st)

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

    host_summary()
    scored(sum_b, brk_b, st_b, False)
    scored(sum_c, brk_c, st_c, True)
    ok = [k for k in range(K) if st_a[k].code == 0]
    rows_ok = np.concatenate([np.arange(row0[k], row0[k + 1]) for k in ok]) if ok else np.zeros(0, dtype=np.int64)
    assert [key(x) for x in st_a] == [key(x) for x in st_b] == [key(x) for x in st_c], name + ": statuses differ"
    assert np.array_equal(sum_a, sum_b) and np.array_equal(sum_b, sum_c), name + ": summaries differ"
    assert np.array_equal(brk_a, brk_b) and np.array_equal(brk_b, brk_c), name + ": per-broker sums differ"
    assert np.array_equal(out[rows_ok], out_c[rows_ok]) and np.array_equal(out_len[rows_ok], len_c[rows_ok]), name + ": rows differ"
    t_a = timed(host_summary)
    t_solve = float(np.median(solve_ms[-steps:]))   # the ka_solve_clusters part of (a)'s timed steps
    t_b = timed(lambda: scored(sum_b, brk_b, st_b, False))
    t_c = timed(lambda: scored(sum_c, brk_c, st_c, True))
    print("| %s | %d | %d | %d | %.1f (%.2f) | %.2f | %.2f | %.1fx |" % (name, K, Q, len(ok), t_a, t_solve, t_b, t_c, t_a / t_b),
          flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    mk = kab.synth.make_ragged_cluster
    print("GPU:", gpu_info())
    print("| fleet | K | partitions | clusters solved | (a) ka_solve_clusters + numpy summary (solve alone), ms "
          "| (b) ka_score_clusters, no rows, ms | (c) ka_score_clusters + rows, ms | (a)/(b) |")
    print("|---|---|---|---|---|---|---|---|")
    for K in (8, 32):
        measure("%d x 30 k topics" % K, [mk(T=30000, N=400, max_partitions=128, seed=100 + k) for k in range(K)], args.steps,
                args.warmup, 0x5EED + K)
    measure("skewed: 240 k + 31 x 2 k topics",
            [mk(T=240000, N=400, max_partitions=128, seed=11)] + [mk(T=2000, N=100, max_partitions=128, seed=200 + k) for k in range(31)],
            args.steps, args.warmup, 0x5EED)
    measure("128 tiny clusters, 40 topics", [mk(T=40, N=24, R=4, max_partitions=32, seed=300 + k) for k in range(128)], args.steps,
            args.warmup, 0x5EED + 128)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
