"""What a sender budget changes in a wave plan (ka_plan_waves_send), and what it costs. The 1.06 M-partition make_ragged_cluster of
wave_plan_times.py (T = 240 k topics), with no broker removed and with 2 % removed, solved with ka_solve on a fresh Context; its
rows (all buffers on the host) then planned with unit weights and B = 1, and with a seeded random weight per partition (up to
16 GiB) and B = 16 x the mean weight. The send table is every broker of the cluster before the exclusion.

For each: the largest per-wave sender load of ka_plan_waves's plan (computed here from its waves: what a receive budget alone
lets one leader send), then ka_plan_waves_send with C = B and C = 4 B: W, the chain's rounds (a record decides in round 1 + the
latest round of the earlier records of its chunk that share a receiver or its sender with it) and the time of one C call, with
ka_plan_waves's on the same rows beside it. Every plan is checked equal to its model (models.plan_waves,
without and with a sender) before it is timed. Each step is synchronous and timed with the host clock, the L2 flushed (256 MiB
written) before it; the median of --steps steps after --warmup. Prints the GPU, its power limit and SM clock, and a markdown
table."""
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


def moved_rows(rep_off, cur, out, out_len):
    """[(row, receivers, sender or None)] of the rows with a receiver, in input order."""
    res = []
    for g in range(len(out_len)):
        old = cur[rep_off[g]:rep_off[g + 1]].tolist()
        recv = [b for b in out[g, :out_len[g]].tolist() if b not in old]
        if recv:
            res.append((g, recv, old[0] if old else None))
    return res


def chain_rounds(moved, send):
    """Rounds of the chain over the moved rows, chunk by chunk; with `send` a record also conflicts through its sender."""
    rounds, depth, last = 0, 0, {}
    for k, (_, recv, s) in enumerate(moved):
        if k % CHUNK == 0:
            rounds += depth
            depth, last = 0, {}
        keys = [("in", b) for b in recv] + ([("out", s)] if send and s is not None else [])
        d = 1 + max(last.get(x, 0) for x in keys)
        for x in keys:
            last[x] = d
        depth = max(depth, d)
    return rounds + depth


def max_send(moved, wave, w):
    """The largest per-wave outgoing sum of one leader under the plan `wave`."""
    loads = {}
    for g, recv, s in moved:
        if s is not None:
            key = (int(wave[g]), s)
            loads[key] = loads.get(key, 0) + (1 if w is None else int(w[g])) * len(recv)
    return max(loads.values()) if loads else 0


def _vp(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def measure(name, cl, steps, warmup, flush):
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    out, out_len, st = s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    assert st.code == 0
    Q = len(out_len)
    send_id = np.ascontiguousarray(cl.all_broker_id, dtype=np.int32)
    weight = np.random.default_rng(0x5EED).integers(1, 1 << 34, size=Q, dtype=np.int64)
    moved = moved_rows(cl.rep_off, cl.cur, out, out_len)
    r_in, r_send = chain_rounds(moved, False), chain_rounds(moved, True)

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

    wave = np.zeros(Q, dtype=np.int32)
    summ = np.zeros(Q, dtype=WAVE_SUMMARY_DTYPE)
    ssum = np.zeros((Q, 2), dtype=np.int64)
    n, kst = ctypes.c_int32(0), kab.KaStatus()
    head = lambda B, w: (s._h, Q, _vp(cl.rep_off), _vp(cl.cur), 3, _vp(out_len), _vp(out), _vp(w), int(B))  # noqa: E731

    def plan(B, w):
        return s._L.ka_plan_waves(*head(B, w), _vp(wave), ctypes.byref(n), _vp(summ), Q, ctypes.byref(kst))

    def plan_send(B, C, w):
        return s._L.ka_plan_waves_send(*head(B, w), len(send_id), _vp(send_id), int(C), _vp(wave), ctypes.byref(n), _vp(summ),
                                       _vp(ssum), Q, ctypes.byref(kst))

    for label, B, w in (("unit, B = 1", 1, None), ("weighted, B = 16 x mean", 16 * int(weight.mean()), weight)):
        assert plan(B, w) == 0
        e_wave, e_summ, _ = models.plan_waves(cl.rep_off, cl.cur, out, out_len, cl.broker_id, B, w)
        assert np.array_equal(wave, e_wave) and [util.record_of(x, WAVE_SUMMARY_DTYPE.names) for x in summ[:n.value]] == e_summ, name + ": plan differs from the model"
        W0, open_send = n.value, max_send(moved, wave, w)
        t0 = timed(lambda: plan(B, w))
        for cm in (1, 4):
            C = cm * B
            assert plan_send(B, C, w) == 0
            e_wave, e_summ, _ = models.plan_waves(cl.rep_off, cl.cur, out, out_len, cl.broker_id, B, w, send=(send_id, C))
            got = [dict(util.record_of(x, WAVE_SUMMARY_DTYPE.names), max_broker_out=int(y[0]), max_broker_out_id=int(y[1])) for x, y in zip(summ[:n.value], ssum)]
            assert np.array_equal(wave, e_wave) and got == e_summ, name + ": send plan differs from the model"
            W, peak = n.value, max_send(moved, wave, w)
            t1 = timed(lambda: plan_send(B, C, w))
            print("| %s | %s | %d | %d | %d | %d | C = %d B | %d | %d | %d | %d | %.2f | %.2f |"
                  % (name, label, Q, len(moved), W0, open_send, cm, peak, W, r_in, r_send, t0, t1), flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    mk = kab.synth.make_ragged_cluster
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print("GPU:", gpu_info())
    print("| cluster | budget | partitions | rows moved | W, receive budget only | its largest leader send per wave | send budget "
          "| largest leader send per wave | W | chain rounds, receive only | chain rounds, with senders | ka_plan_waves, ms "
          "| ka_plan_waves_send, ms |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for remove in (0.0, 0.02):
        cl = mk(T=240000, N=400, max_partitions=128, seed=11, remove_frac=remove)
        measure("240 k topics, %d %% removed" % round(100 * remove), cl, args.steps, args.warmup, flush)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
