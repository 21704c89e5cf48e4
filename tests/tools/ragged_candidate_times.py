"""Candidate broker sets over one real-cluster-shaped (ragged) problem: K sequential ka_solve calls against one
ka_solve_candidates call, all buffers on the host. Workloads: the 240 k-topic make_ragged_cluster (1.06 M partitions) with the
eight removal fractions of ragged_decommission_tables (K = 8) and with K = 1, 8 and 32 candidates that each remove a different
seeded random 2 % of the brokers; BASELINE config 3 in the ragged layout with K = 8 such candidates.

The contexts are created before the timed window. A sequential step is, per candidate, ka_ctx_reset + ka_ctx_set_brokers +
ka_solve (what one run of the tool per broker set does); a batched step is one ka_solve_candidates. Both are synchronous and
timed with the host clock, the L2 flushed (256 MiB written) before every step; the median of --steps steps after --warmup
warm-up steps. The statuses of the two arms, and the rows of every candidate that solved, are checked equal first. Prints
the GPU, its power limit and SM clock, and a markdown table."""
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

FRACS = (0.01, 0.02, 0.05, 0.10, 0.20, 0.30, 0.40, 0.50)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name(0)


def random_tables(broker_id, rack_index, K, frac, seed):
    rng = np.random.default_rng(seed)
    n = len(broker_id) - int(round(frac * len(broker_id)))
    out = []
    for _ in range(K):
        keep = np.sort(rng.choice(len(broker_id), n, replace=False))
        out.append((broker_id[keep], rack_index[keep]))
    return out


def _vp(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def measure(name, prob, tables, steps, warmup):
    """prob = (topic_hash, part_off, part_id, rep_off, cur) host arrays, rows of 3 replicas at most."""
    th, part_off, part_id, rep_off, cur = prob
    T, Q, K, S = len(th), int(part_off[-1]), len(tables), int(np.diff(rep_off).max())
    seq_out = np.empty((K, Q, S), dtype=np.int32)
    seq_len = np.empty((K, Q), dtype=np.int32)
    bat_out = np.empty((K, Q, S), dtype=np.int32)
    bat_len = np.empty((K, Q), dtype=np.int32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    solvers = [kab.Solver(0) for _ in tables]
    batch = kab.Solver(0)
    L = batch._L
    tabs = [(np.ascontiguousarray(i, dtype=np.int32), np.ascontiguousarray(r, dtype=np.int32)) for i, r in tables]
    cand_off, broker_id, broker_rack = kab.Solver._candidate_tables(tabs)
    seq_st = (kab.KaStatus * K)()
    sts = (kab.KaStatus * K)()
    key = lambda st: (st.code, st.topic_index, st.partition, st.a, st.b)  # noqa: E731

    def sequential():
        for k, (s, (ids, racks)) in enumerate(zip(solvers, tabs)):
            assert L.ka_ctx_reset(s._h) == 0
            assert L.ka_ctx_set_brokers(s._h, len(ids), _vp(ids), _vp(racks)) == 0
            L.ka_solve(s._h, T, _vp(th), _vp(part_off), _vp(part_id), _vp(rep_off), _vp(cur), -1, S, _vp(seq_len[k]),
                       _vp(seq_out[k]), ctypes.byref(seq_st[k]))

    def batched():
        L.ka_solve_candidates(batch._h, K, _vp(cand_off), _vp(broker_id), _vp(broker_rack), T, _vp(th), _vp(part_off),
                              _vp(part_id), _vp(rep_off), _vp(cur), -1, S, _vp(bat_len), _vp(bat_out), sts)

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
    ok = [k for k in range(K) if seq_st[k].code == 0]   # the rows of a failed candidate are unspecified
    assert [key(sts[k]) for k in range(K)] == [key(seq_st[k]) for k in range(K)], name + ": statuses differ"
    assert np.array_equal(seq_out[ok], bat_out[ok]) and np.array_equal(seq_len[ok], bat_len[ok]), name + ": rows differ"
    t_seq, t_bat = timed(sequential), timed(batched)
    print("| %s | %d | %d | %d | %.2f | %.2f | %.2fx |" % (name, Q, K, len(ok), t_seq, t_bat, t_seq / t_bat), flush=True)
    for s in solvers + [batch]:
        s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    print("GPU:", gpu_info())
    print("| workload | partitions | K | candidates solved | (a) K sequential ka_solve, ms | (b) one ka_solve_candidates, ms | (a)/(b) |")
    print("|---|---|---|---|---|---|---|")
    rc = kab.synth.make_ragged_cluster(T=240000, N=400, max_partitions=128, seed=11)
    prob = (rc.topic_hash, rc.part_off, rc.part_id, rc.rep_off, rc.cur)
    measure("ragged 240 k topics, removal fractions", prob, kab.synth.ragged_decommission_tables(rc, FRACS), args.steps, args.warmup)
    for K in (1, 8, 32):
        measure("ragged 240 k topics, random 2 %", prob, random_tables(rc.broker_id, rc.rack_index, K, 0.02, 0x5EED + K), args.steps,
                args.warmup)
    del rc, prob
    c3 = kab.synth.make_config("c3", "mixed")
    part_off, part_id, rep_off, cur = c3.ragged()
    measure("c3 ragged layout, random 2 %", (c3.topic_hash, part_off, part_id, rep_off, cur),
            random_tables(c3.broker_id, c3.rack_index, 8, 0.02, 0x5EED + 8), args.steps, args.warmup)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
