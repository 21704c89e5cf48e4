"""Candidate broker sets over one cluster: K sequential ka_solve_dense_device calls (a fresh Context each) against one
ka_solve_dense_candidates_device call. Workloads: BASELINE config 5 with the eight removal fractions of decommission_sweep.py
(K = 8), and config 3 with K = 1, 8 and 32 candidates, each removing a different seeded random 2 % of the brokers.

Both arms run on the same stream, timed with CUDA events, the L2 flushed (256 MiB written) before every step; the median of
--steps steps after --warmup warm-up steps. The rows of the two arms are checked equal first. Prints the GPU, its power limit
and SM clock, a markdown table, and the replicas each candidate moves (computed here in torch)."""
import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

import kafka_assigner_b200 as kab  # noqa: E402

FRACS = (0.01, 0.02, 0.05, 0.10, 0.20, 0.30, 0.40, 0.50)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name(0)


def random_tables(cl, K, frac, seed):
    rng = np.random.default_rng(seed)
    n = len(cl.broker_id) - int(round(frac * len(cl.broker_id)))
    out = []
    for _ in range(K):
        keep = np.sort(rng.choice(len(cl.broker_id), n, replace=False))
        out.append((cl.broker_id[keep], cl.rack_index[keep]))
    return out


def measure(name, cl, tables, steps, warmup):
    T, P, RF, K = cl.T, cl.P, cl.RF, len(tables)
    stream = torch.cuda.current_stream()
    sp = stream.cuda_stream
    d_hash = torch.from_numpy(cl.topic_hash).cuda()
    d_cur = torch.from_numpy(cl.cur).cuda()
    seq_out = torch.empty((K, T, P, RF), dtype=torch.int32, device="cuda")
    bat_out = torch.empty((K, T, P, RF), dtype=torch.int32, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    solvers = []
    for ids, racks in tables:
        s = kab.Solver(0)
        s.set_brokers(ids, racks)
        solvers.append(s)
    batch = kab.Solver(0)

    def sequential():
        for k, s in enumerate(solvers):
            st = s.solve_dense_device(T, d_hash.data_ptr(), P, RF, d_cur.data_ptr(), -1, RF, 0, seq_out[k].data_ptr(), stream=sp)
            assert st.code == 0, (name, k, st.code)

    def batched():
        sts = batch.solve_dense_candidates_device(tables, T, d_hash.data_ptr(), P, RF, d_cur.data_ptr(), -1, RF, 0,
                                                  bat_out.data_ptr(), stream=sp)
        assert all(st.code == 0 for st in sts), (name, [st.code for st in sts])

    def timed(fn):
        ms = []
        for i in range(warmup + steps):
            for s in solvers:
                s.reset()   # a fresh Context for every sequential solve
            flush.fill_(i & 0xFF)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            b.synchronize()
            if i >= warmup:
                ms.append(a.elapsed_time(b))
        return float(np.median(ms))

    for s in solvers:
        s.reset()
    sequential()
    batched()
    torch.cuda.synchronize()
    assert torch.equal(seq_out, bat_out), name + ": batched rows differ from the sequential solves"
    t_seq, t_bat = timed(sequential), timed(batched)
    cur = d_cur.view(1, T, P, RF)
    moved = (~(bat_out.unsqueeze(-1) == cur.unsqueeze(-2)).any(-1)).sum(dim=(1, 2, 3)).tolist()
    print("| %s | %d | %.3f | %.3f | %.2fx | %s |" % (name, K, t_seq, t_bat, t_seq / t_bat, " ".join(str(m) for m in moved)),
          flush=True)
    for s in solvers + [batch]:
        s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    print("GPU:", gpu_info())
    print("| workload | K | (a) K sequential solves, ms | (b) one batched call, ms | (a)/(b) | replicas moved per candidate |")
    print("|---|---|---|---|---|---|")
    c5 = kab.synth.make_config("c5", "mixed")
    measure("c5, removal fractions", c5, kab.synth.decommission_tables("c5", FRACS), args.steps, args.warmup)
    del c5
    c3 = kab.synth.make_config("c3", "mixed")
    for K in (1, 8, 32):
        measure("c3, random 2 %", c3, random_tables(c3, K, 0.02, 0x5EED + K), args.steps, args.warmup)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
