"""Choosing between candidate broker sets of one real-cluster-shaped (ragged) problem: what it costs to get each candidate's
movement and balance summary. Workload: the 240 k-topic make_ragged_cluster (1.06 M partitions) with K = 8 and 32 candidates
that each remove a different seeded random 2 % of the brokers, and a seeded random weight per partition. Arms, all buffers on
the host:

  (a) ka_solve_candidates (every candidate's rows and list lengths copied back) + the numpy summary of
      tests/models.py per candidate on the host;
  (b) ka_score_candidates without rows (K summaries come back);
  (c) ka_score_candidates with rows (the summaries and the rows of (a)).

Every step is synchronous and timed with the host clock, the L2 flushed (256 MiB written) before it; the median of --steps
steps after --warmup warm-up steps. Before timing, the statuses, summaries and per-broker arrays of the three arms, and the rows
of (a) and (c), are checked equal. Prints the GPU, its power limit and SM clock, and a markdown table."""
import argparse
import ctypes
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import kafka_assigner_b200 as kab  # noqa: E402
from kafka_assigner_b200.assigner import MOVE_SUMMARY_DTYPE  # noqa: E402
from tests import models  # noqa: E402
from tests.tools.ragged_candidate_times import gpu_info, random_tables  # noqa: E402


def _vp(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def measure(name, prob, tables, weight, steps, warmup):
    th, part_off, part_id, rep_off, cur = prob
    T, Q, K, S = len(th), int(part_off[-1]), len(tables), int(np.diff(rep_off).max())
    out = np.empty((K, Q, S), dtype=np.int32)
    out_len = np.empty((K, Q), dtype=np.int32)
    out_c = np.empty((K, Q, S), dtype=np.int32)
    len_c = np.empty((K, Q), dtype=np.int32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    s = kab.Solver(0)
    L = s._L
    tabs = [(np.ascontiguousarray(i, dtype=np.int32), np.ascontiguousarray(r, dtype=np.int32)) for i, r in tables]
    cand_off, broker_id, broker_rack = kab.Solver._candidate_tables(tabs)
    nb = int(cand_off[-1])
    st_a, st_b, st_c = ((kab.KaStatus * K)() for _ in range(3))
    sum_a, sum_b, sum_c = (np.zeros(K, dtype=MOVE_SUMMARY_DTYPE) for _ in range(3))
    brk_a, brk_b, brk_c = (np.zeros((3, nb), dtype=np.int64) for _ in range(3))
    key = lambda st: (st.code, st.topic_index, st.partition, st.a, st.b)  # noqa: E731
    head = lambda: (s._h, K, _vp(cand_off), _vp(broker_id), _vp(broker_rack), T, _vp(th), _vp(part_off), _vp(part_id),  # noqa: E731
                    _vp(rep_off), _vp(cur), -1, S)

    solve_ms = []

    def host_summary():
        t0 = time.perf_counter()
        L.ka_solve_candidates(*head(), _vp(out_len), _vp(out), st_a)
        solve_ms.append((time.perf_counter() - t0) * 1e3)
        for k, (ids, _) in enumerate(tabs):
            if st_a[k].code != 0:
                continue
            e, rep, lead, inb = models.move_summary(out[k], out_len[k], rep_off, cur, ids.astype(np.int64), weight)
            for f, v in e.items():
                sum_a[k][f] = v
            for i, a in enumerate((rep, lead, inb)):
                brk_a[i, cand_off[k]:cand_off[k + 1]] = a

    def scored(summary, brk, st, rows):
        L.ka_score_candidates(*head(), _vp(weight), _vp(summary), _vp(brk[0]), _vp(brk[1]), _vp(brk[2]),
                              _vp(len_c) if rows else None, _vp(out_c) if rows else None, st)

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
    assert [key(x) for x in st_a] == [key(x) for x in st_b] == [key(x) for x in st_c], name + ": statuses differ"
    assert np.array_equal(sum_a[ok], sum_b[ok]) and np.array_equal(sum_b, sum_c), name + ": summaries differ"
    assert np.array_equal(brk_a, brk_b) and np.array_equal(brk_b, brk_c), name + ": per-broker sums differ"
    assert np.array_equal(out[ok], out_c[ok]) and np.array_equal(out_len[ok], len_c[ok]), name + ": rows differ"
    t_a = timed(host_summary)
    t_solve = float(np.median(solve_ms[-steps:]))   # the ka_solve_candidates part of (a)'s timed steps
    t_b = timed(lambda: scored(sum_b, brk_b, st_b, False))
    t_c = timed(lambda: scored(sum_c, brk_c, st_c, True))
    print("| %s | %d | %d | %d | %.1f (%.1f) | %.1f | %.1f | %.2fx |" % (name, Q, K, len(ok), t_a, t_solve, t_b, t_c, t_a / t_b),
          flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    print("GPU:", gpu_info())
    print("| workload | partitions | K | candidates solved | (a) solve + numpy summary (solve alone), ms | (b) score, no rows, ms | "
          "(c) score + rows, ms | (a)/(b) |")
    print("|---|---|---|---|---|---|---|---|")
    rc = kab.synth.make_ragged_cluster(T=240000, N=400, max_partitions=128, seed=11)
    prob = (rc.topic_hash, rc.part_off, rc.part_id, rc.rep_off, rc.cur)
    weight = np.random.default_rng(0x5EED).integers(1, 1 << 34, size=rc.Q, dtype=np.int64)   # up to 16 GiB per partition
    for K in (8, 32):
        measure("ragged 240 k topics, random 2 %", prob, random_tables(rc.broker_id, rc.rack_index, K, 0.02, 0x5EED + K), weight,
                args.steps, args.warmup)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
