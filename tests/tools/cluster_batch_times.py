"""A fleet of independent real-cluster-shaped (ragged) clusters, each with its own broker table: K sequential ka_solve calls
against one ka_solve_clusters call, all buffers on the host. Fleets: (a) K = 8 and K = 32 make_ragged_cluster clusters of
30 k topics each (different seeds); (b) a skewed fleet, one 240 k-topic cluster and 31 of 2 k topics; (c) K = 128 tiny clusters
of 40 topics (a few hundred partitions each).

The contexts are created before the timed window. A sequential step is, per cluster, ka_ctx_reset (a fresh Context) +
ka_ctx_set_brokers + ka_solve (what one run of the tool per cluster does); a batched step is one ka_solve_clusters over the
fleet's layout, marshalled once beforehand. Both are synchronous and timed with the host clock, the L2 flushed (256 MiB written)
before every step; the median of --steps steps after --warmup warm-up steps. The statuses of the two arms, and the rows of
every cluster that solved, are checked equal first. Prints the GPU, its power limit and SM clock, and a markdown table."""
import argparse
import ctypes
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

import kafka_assigner_b200 as kab  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name(0)


def _vp(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def measure(name, clusters, steps, warmup):
    """clusters: synth.RaggedCluster list, each solved against its own live table, rows of 3 replicas at most."""
    K = len(clusters)
    S = max(int(np.diff(c.rep_off).max()) for c in clusters)
    entries = [(c.broker_id, c.rack_index, c.topic_hash, c.part_off, c.part_id, c.rep_off, c.cur, -1) for c in clusters]
    lay = kab.Solver.marshal_clusters(entries)
    cand_off, broker_id, broker_rack, topic_off, drf, th, part_off, part_id, rep_off, cur = lay
    Q = int(part_off[-1])
    rows = part_off[topic_off]
    seq_out = np.empty((Q, S), dtype=np.int32)
    seq_len = np.empty(Q, dtype=np.int32)
    bat_out = np.empty((Q, S), dtype=np.int32)
    bat_len = np.empty(Q, dtype=np.int32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    solvers = [kab.Solver(0) for _ in clusters]
    batch = kab.Solver(0)
    L = batch._L
    seq_st = (kab.KaStatus * K)()
    sts = (kab.KaStatus * K)()
    key = lambda st: (st.code, st.topic_index, st.partition, st.a, st.b)  # noqa: E731
    # the sequential arm's own arrays, and where its rows land in the shared output
    own = [tuple(np.ascontiguousarray(a) for a in (c.broker_id, c.rack_index, c.topic_hash, c.part_off, c.part_id, c.rep_off, c.cur))
           for c in clusters]

    def sequential():
        for k, (s, (ids, racks, h, po, pid, ro, cr)) in enumerate(zip(solvers, own)):
            assert L.ka_ctx_reset(s._h) == 0
            assert L.ka_ctx_set_brokers(s._h, len(ids), _vp(ids), _vp(racks)) == 0
            L.ka_solve(s._h, len(h), _vp(h), _vp(po), _vp(pid), _vp(ro), _vp(cr), -1, S, _vp(seq_len[rows[k]:]),
                       _vp(seq_out[rows[k]:]), ctypes.byref(seq_st[k]))

    def batched():
        L.ka_solve_clusters(batch._h, K, _vp(cand_off), _vp(broker_id), _vp(broker_rack), _vp(topic_off), _vp(drf), _vp(th),
                            _vp(part_off), _vp(part_id), _vp(rep_off), _vp(cur), S, _vp(bat_len), _vp(bat_out), sts)

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
    ok = [k for k in range(K) if seq_st[k].code == 0]   # the rows of a failed cluster are unspecified
    assert [key(sts[k]) for k in range(K)] == [key(seq_st[k]) for k in range(K)], name + ": statuses differ"
    for k in ok:
        a, b = rows[k], rows[k + 1]
        assert np.array_equal(seq_out[a:b], bat_out[a:b]) and np.array_equal(seq_len[a:b], bat_len[a:b]), name + ": rows differ"
    sizes = np.diff(rows)
    t_seq, t_bat = timed(sequential), timed(batched)
    print("| %s | %d | %d | %d | %d | %.2f | %.2f | %.2fx |" % (name, K, Q, int(sizes.max()), len(ok), t_seq, t_bat, t_seq / t_bat),
          flush=True)
    for s in solvers + [batch]:
        s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    mk = kab.synth.make_ragged_cluster
    print("GPU:", gpu_info())
    print("| fleet | K | partitions | largest cluster | clusters solved | (a) K sequential ka_solve, ms | (b) one ka_solve_clusters, ms "
          "| (a)/(b) |")
    print("|---|---|---|---|---|---|---|---|")
    for K in (8, 32):
        measure("(a) %d x 30 k topics" % K, [mk(T=30000, N=400, max_partitions=128, seed=100 + k) for k in range(K)], args.steps,
                args.warmup)
    measure("(b) skewed: 240 k + 31 x 2 k topics",
            [mk(T=240000, N=400, max_partitions=128, seed=11)] + [mk(T=2000, N=100, max_partitions=128, seed=200 + k) for k in range(31)],
            args.steps, args.warmup)
    measure("(c) 128 tiny clusters, 40 topics", [mk(T=40, N=24, R=4, max_partitions=32, seed=300 + k) for k in range(128)], args.steps,
            args.warmup)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
