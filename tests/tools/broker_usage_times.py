"""Every broker's disk usage across a wave plan on the device (ka_wave_broker_usage) against a numpy host build of the same
report. The 1.06 M-partition make_ragged_cluster of wave_plan_times.py (T = 240 k topics, 10 % of the brokers joined empty), with
no broker removed and with 2 % removed, solved with ka_solve on a fresh Context and planned with ka_plan_waves under the seeded
random weights (up to 16 GiB per partition) and a budget of 16 x the mean weight. The usage table is every broker of the cluster
before the exclusion.

Before timing, the device report is checked equal to usage_models.broker_usage_np. Each step is synchronous and timed with the
host clock, the L2 flushed (256 MiB written) before it; the median of --steps steps after --warmup warm-up steps. Prints the GPU,
its power limit and SM clock, a markdown table, and how many brokers peak above both their start and their end, and by how much."""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

import kafka_assigner_b200 as kab  # noqa: E402
from tests import usage_models, util  # noqa: E402
from tests.tools.cluster_batch_times import gpu_info  # noqa: E402


def measure(name, cl, steps, warmup, flush):
    s, out, out_len, _ = util.solved(cl)
    Q = len(out_len)
    weight = np.random.default_rng(0x5EED).integers(1, 1 << 34, size=Q, dtype=np.int64)
    wave, summ, st = s.plan_waves(cl.rep_off, cl.cur, out, out_len, 16 * int(weight.mean()), weight=weight)
    assert st.code == 0
    ids = cl.all_broker_id
    args = (cl.rep_off, cl.cur, out, out_len, wave, ids, weight)

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

    usage, W, st = s.broker_usage(*args)
    e, e_W = usage_models.broker_usage_np(*args)
    assert st.code == 0 and W == e_W, name + ": refused"
    assert all(np.array_equal(usage[f], e[f]) for f in usage_models.FIELDS), name + ": report differs from the model"
    n0 = s.launch_count()
    s.broker_usage(*args)
    launches = s.launch_count() - n0
    _, _, ev_idx, _ = usage_models.replica_events(*args[:6], weight)
    t_dev = timed(lambda: s.broker_usage(*args))
    t_host = timed(lambda: usage_models.broker_usage_np(*args))
    inside = usage["peak"] > np.maximum(usage["before"], usage["after"])
    excess = (usage["peak"] - np.maximum(usage["before"], usage["after"]))[inside]
    rel = excess / np.maximum(np.maximum(usage["before"], usage["after"])[inside], 1)
    print("| %s | %d | %d | %d | %d | %d | %.2f | %.1f |" % (name, Q, W, len(ids), len(ev_idx), launches, t_dev, t_host), flush=True)
    if inside.any():
        print("    %s: %d of %d brokers peak above both ends, by %.1f %% at the median and %.1f %% at most (of the larger end)"
              % (name, int(inside.sum()), len(ids), 100 * float(np.median(rel)), 100 * float(rel.max())), flush=True)
    else:
        print("    %s: no broker peaks above both ends" % name, flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    mk = kab.synth.make_ragged_cluster
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print("GPU:", gpu_info())
    print("| cluster | partitions | waves W | usage brokers | replica events | launches | ka_wave_broker_usage, ms "
          "| numpy host build, ms |")
    print("|---|---|---|---|---|---|---|---|")
    for remove in (0.0, 0.02):
        cl = mk(T=240000, N=400, max_partitions=128, seed=11, remove_frac=remove)
        measure("240 k topics, %d %% removed" % round(100 * remove), cl, args.steps, args.warmup, flush)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
