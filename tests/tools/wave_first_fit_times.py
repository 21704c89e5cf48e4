"""The two wave rules on a real cluster: how many waves each needs and what each costs on the device. The 1.06 M-partition
make_ragged_cluster of wave_plan_times.py (T = 240 k topics, 10 % of the brokers joined empty), with no broker removed and with
2 % removed, solved with ka_solve; its rows planned under KA_WAVE_GREEDY and KA_WAVE_FIRST_FIT
  - with unit weights and a budget of 1 replica per broker per wave, and
  - with wave_plan_times.py's seeded weights (up to 16 GiB) and a budget of 16 x the mean weight.

Before timing, every wave and summary of each rule is checked equal to its model (models.plan_waves of tests/models.py,
fit_models.plan_waves of tests/fit_models.py),
and the documents call's waves equal the plan's. Reports W, the lower bound max_b ceil(received_b / B) (unit weights), the
first-fit bound Wb of include/kassign.h and its load table's bytes (Wb x N x 8), and the median time of --steps synchronous
calls after --warmup (the L2 flushed, 256 MiB written, before each) of ONE ka_plan_waves C call and of
Solver.plan_wave_parts_rollback_json (ka_plan_waves_json_parts_rollback, L = 1048575). Prints the GPU, its power limit and SM
clock before and after, and a markdown table."""
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
from tests import fit_models, models, util  # noqa: E402
from tests.tools.cluster_batch_times import gpu_info  # noqa: E402

ZNODE = 1048575


def _vp(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def receivers(rep_off, cur, out, out_len):
    """The receivers of every row with one (new-list brokers its current list lacks)."""
    res = []
    for g in range(len(out_len)):
        old = set(cur[rep_off[g]:rep_off[g + 1]].tolist())
        recv = [b for b in out[g, :out_len[g]].tolist() if b not in old]
        if recv:
            res.append(recv)
    return res


def bounds(recv, B):
    """(lower bound max_b ceil(R_b / B), Wb = min(M, 1 + max over rows of sum (R_b - 1)))."""
    R = {}
    for r in recv:
        for b in r:
            R[b] = R.get(b, 0) + 1
    worst = max(sum(R[b] - 1 for b in r) for r in recv)
    return max(-(-x // B) for x in R.values()), min(len(recv), 1 + worst)


def measure(name, cl, steps, warmup, flush):
    s, out, out_len, _ = util.solved(cl)
    Q = len(out_len)
    weight = np.random.default_rng(0x5EED).integers(1, 1 << 34, size=Q, dtype=np.int64)
    recv = receivers(cl.rep_off, cl.cur, out, out_len)
    names = ["t%d" % t for t in range(cl.T)]

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

    for label, B, w in (("unit, B = 1", 1, None), ("weighted, B = 16 x mean", 16 * int(weight.mean()), weight)):
        low, Wb = bounds(recv, 1)
        for rule in ("greedy", "first_fit"):
            s.set_wave_rule(rule)
            wave, summ, st = s.plan_waves(cl.rep_off, cl.cur, out, out_len, B, weight=w)
            model = fit_models.plan_waves if rule == "first_fit" else models.plan_waves
            e_wave, e_summ, e_st = model(cl.rep_off, cl.cur, out, out_len, cl.broker_id, B, w)
            assert st.code == 0 and e_st[0] == 0, name + ": refused"
            assert np.array_equal(wave, e_wave), name + " " + rule + ": waves differ from the model"
            assert [util.record_of(x, WAVE_SUMMARY_DTYPE.names) for x in summ] == e_summ, name + " " + rule + ": summaries differ"
            W = len(summ)
            wave1, summ1, n, kst = np.zeros(Q, dtype=np.int32), np.zeros(W, dtype=WAVE_SUMMARY_DTYPE), ctypes.c_int32(0), kab.KaStatus()

            def call():
                return s._L.ka_plan_waves(s._h, Q, _vp(cl.rep_off), _vp(cl.cur), out.shape[1], _vp(out_len), _vp(out), _vp(w), int(B),
                                          _vp(wave1), ctypes.byref(n), _vp(summ1), W, ctypes.byref(kst))
            assert call() == 0 and n.value == W and np.array_equal(wave1, wave), name + ": single call differs"

            def docs():
                return s.plan_wave_parts_rollback_json(names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, B, ZNODE,
                                                       weight=w)
            parts, _, part_wave, d_wave, _, dst = docs()
            assert dst.code == 0 and np.array_equal(d_wave, wave) and part_wave[-1] == W, name + ": documents differ"
            t_call, t_docs = timed(call), timed(docs)
            fit = rule == "first_fit"
            print("| %s | %s | %s | %d | %s | %s | %s | %.2f | %.1f | %d |" % (
                name, label, rule, W, low if w is None else "—", Wb if fit else "—",
                "%.1f MB" % (Wb * len(cl.broker_id) * 8 / 1e6) if fit else "—", t_call, t_docs, len(parts)), flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    mk = kab.synth.make_ragged_cluster
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print("GPU:", gpu_info())
    print("| cluster | budget | rule | waves W | lower bound | Wb | load table | ka_plan_waves, one C call, ms "
          "| plan_wave_parts_rollback_json, ms | parts |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for remove in (0.0, 0.02):
        cl = mk(T=240000, N=400, max_partitions=128, seed=11, remove_frac=remove)
        measure("240 k topics, %d %% removed" % round(100 * remove), cl, args.steps, args.warmup, flush)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
