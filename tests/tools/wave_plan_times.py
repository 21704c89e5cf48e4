"""Cutting a solve's reassignment into waves on the device (ka_plan_waves): what it costs, how many waves and how many rounds of
the chain a real cluster gives. The 1.06 M-partition make_ragged_cluster (T = 240 k topics, 10 % of the brokers joined empty),
with no broker removed and with 2 % removed, solved with ka_solve on a fresh Context; its rows (all buffers on the host) then
planned
  - with unit weights and a budget of 1 replica per broker per wave, and
  - with a seeded random weight per partition (up to 16 GiB) and a budget of 16 x the mean weight.

Two arms: ONE ka_plan_waves C call with a summary buffer of W entries, and Solver.plan_waves (which asks for min(Q, 64 k)
summaries, so here it also makes one C call; the tool checks that W fits). Every step is synchronous and timed with the host clock, the L2 flushed (256 MiB written) before it; the median of --steps
steps after --warmup warm-up steps. Before timing, every wave and summary is checked equal to models.plan_waves of
tests/models.py. The chain's rounds are counted from the records in the chain's own chunks (a record decides in round
1 + the latest round of the earlier records of its chunk that share a receiver with it). Prints the GPU, its power limit and SM
clock, and a markdown table."""
import argparse
import ctypes
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

import kafka_assigner_b200 as kab  # noqa: E402
from kafka_assigner_b200.assigner import WAVE_SUMMARY_DTYPE  # noqa: E402
from tests import models, util  # noqa: E402
from tests.tools.cluster_batch_times import gpu_info  # noqa: E402

CHUNK = 2048   # KA_WAVE_CHUNK of kassign_waves.cuh: records the chain decides together


def chain_rounds(rep_off, cur, out, out_len):
    """Rounds of the chain over the moved rows (rows with a receiver), in input order, chunk by chunk."""
    rounds, depth, last = 0, 0, {}
    k = 0
    for g in range(len(out_len)):
        old = set(cur[rep_off[g]:rep_off[g + 1]].tolist())
        recv = [b for b in out[g, :out_len[g]].tolist() if b not in old]
        if not recv:
            continue
        if k % CHUNK == 0:
            rounds += depth
            depth, last = 0, {}
        d = 1 + max(last.get(b, 0) for b in recv)
        for b in recv:
            last[b] = d
        depth = max(depth, d)
        k += 1
    return rounds + depth, k


def _vp(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def plan_once(s, rep_off, cur, out, out_len, B, w, wave, summary):
    """One ka_plan_waves call into `wave` and `summary` (its capacity: len(summary)); returns (rc, W)."""
    n, st = ctypes.c_int32(0), kab.KaStatus()
    rc = s._L.ka_plan_waves(s._h, len(out_len), _vp(rep_off), _vp(cur), out.shape[1], _vp(out_len), _vp(out), _vp(w), int(B), _vp(wave),
                            ctypes.byref(n), _vp(summary), len(summary), ctypes.byref(st))
    return rc, n.value


def measure(name, cl, steps, warmup, flush):
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    args = (cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)

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

    def solve():
        s.reset()
        return s.solve_ragged(*args)

    out, out_len, st = solve()
    assert st.code == 0
    t_solve = timed(solve)
    Q = len(out_len)
    weight = np.random.default_rng(0x5EED).integers(1, 1 << 34, size=Q, dtype=np.int64)
    rounds, moved = chain_rounds(cl.rep_off, cl.cur, out, out_len)
    for label, B, w in (("unit, B = 1", 1, None), ("weighted, B = 16 x mean", 16 * int(weight.mean()), weight)):
        wave, summ, st = s.plan_waves(cl.rep_off, cl.cur, out, out_len, B, weight=w)
        e_wave, e_summ, e_st = models.plan_waves(cl.rep_off, cl.cur, out, out_len, cl.broker_id, B, w)
        assert st.code == 0 and e_st[0] == 0, name + ": refused"
        assert np.array_equal(wave, e_wave) and [util.record_of(x, WAVE_SUMMARY_DTYPE.names) for x in summ] == e_summ, name + ": plan differs from the model"
        W = len(summ)
        assert W <= min(Q, s.WAVE_SUMMARY_CAP), name + ": Solver.plan_waves would make a second call"
        wave1, summ1 = np.zeros(Q, dtype=np.int32), np.zeros(W, dtype=WAVE_SUMMARY_DTYPE)
        assert plan_once(s, cl.rep_off, cl.cur, out, out_len, B, w, wave1, summ1) == (0, W), name + ": single call refused"
        assert np.array_equal(wave1, wave) and np.array_equal(summ1, summ), name + ": single call differs"
        t_call = timed(lambda: plan_once(s, cl.rep_off, cl.cur, out, out_len, B, w, wave1, summ1))
        t_solver = timed(lambda: s.plan_waves(cl.rep_off, cl.cur, out, out_len, B, weight=w))
        print("| %s | %s | %d | %d | %d | %d | %d | %.1f | %.2f | %.2f |" % (name, label, Q, int((wave > 0).sum()), moved, W, rounds,
                                                                           t_solve, t_call, t_solver), flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    mk = kab.synth.make_ragged_cluster
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print("GPU:", gpu_info())
    print("| cluster | budget | partitions | rows changed | rows moved | waves W | chain rounds | ka_solve, ms "
          "| ka_plan_waves, one C call, ms | Solver.plan_waves, ms |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for remove in (0.0, 0.02):
        cl = mk(T=240000, N=400, max_partitions=128, seed=11, remove_frac=remove)
        measure("240 k topics, %d %% removed" % round(100 * remove), cl, args.steps, args.warmup, flush)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
