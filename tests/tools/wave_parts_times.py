"""Every wave document under a size limit, cut on the device (ka_plan_waves_json_parts): what the cut costs beside
ka_plan_waves_json on the cluster and plans of wave_json_times.py (the 1.06 M-partition make_ragged_cluster, no broker removed
and 2 % removed; unit weights with a budget of 1, and seeded random weights with a budget of 16 x the mean), at L = 1 048 575
(ZooKeeper's default jute.maxbuffer, so each part fits one znode) and at the smallest feasible L (the longest one-record
document: every part then holds as few rows as any cut can give).

Both arms start from the rows in host memory and end with every document's text in host memory (a pinned buffer of the
documented sufficient size): ONE ka_plan_waves_json C call, and ONE ka_plan_waves_json_parts C call. Every step is synchronous
and timed with the host clock, the L2 flushed (256 MiB written) before it; the median of --steps steps after --warmup warm-up
steps. Before timing, every document of both arms is checked equal, byte for byte, to the model, models.wave_documents without
and with the limit. Prints the GPU, its power limit and SM clock, and a markdown table."""
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
from tests.tools.wave_plan_times import _vp  # noqa: E402

ZNODE = 0xFFFFF


def measure(name, cl, steps, warmup, flush):
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    out, out_len, st = s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    assert st.code == 0
    Q, T = len(out_len), len(cl.topic_names)
    names, name_off = s.marshal_names(cl.topic_names)
    cap = models.json_bound(cl.topic_names, cl.part_off, 3)
    text = torch.empty(cap, dtype=torch.uint8).pin_memory().numpy()
    doc_off, doc_wave, wave = np.zeros(Q + 1, dtype=np.int64), np.zeros(Q, dtype=np.int32), np.zeros(Q, dtype=np.int32)
    weight = np.random.default_rng(0x5EED).integers(1, 1 << 34, size=Q, dtype=np.int64)

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
        case = (cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, cl.broker_id, B, w)
        e_docs, _, _, e_wave, _, e_st = models.wave_documents(*case)
        assert e_st[0] == 0, name + ": refused"
        W = len(e_docs)
        summ = np.zeros(W, dtype=WAVE_SUMMARY_DTYPE)
        rows = (s._h, T, _vp(cl.part_off), _vp(cl.part_id), _vp(cl.rep_off), _vp(cl.cur), 3, _vp(out_len), _vp(out), _vp(w), int(B),
                _vp(names), _vp(name_off), _vp(text), cap)

        def docs():
            n, st = ctypes.c_int32(0), kab.KaStatus()
            rc = s._L.ka_plan_waves_json(*rows, _vp(doc_off), _vp(wave), ctypes.byref(n), _vp(summ), W, ctypes.byref(st))
            return rc, n.value

        def parts(L):
            n, d, st = ctypes.c_int32(0), ctypes.c_int32(0), kab.KaStatus()
            rc = s._L.ka_plan_waves_json_parts(*rows, L, _vp(doc_off), _vp(doc_wave), ctypes.byref(d), _vp(wave), ctypes.byref(n),
                                               _vp(summ), W, ctypes.byref(st))
            return rc, n.value, d.value

        assert docs() == (0, W) and np.array_equal(wave, e_wave), name + ": device plan differs from the model"
        for v, e in enumerate(e_docs):
            assert bytes(text[doc_off[v]:doc_off[v + 1]]) == e, "%s: document %d differs from the model" % (name, v)
        t_docs = timed(docs)
        smallest = util.smallest_limit(*case[:7], e_wave)
        for L_label, L in (("1 048 575", ZNODE), ("smallest, %d" % smallest, smallest)):
            e_parts, _, e_part_wave = models.wave_documents(*case, L=L)[:3]
            D = len(e_parts)
            assert parts(L) == (0, W, D) and np.array_equal(wave, e_wave), name + ": device parts plan differs"
            assert doc_wave[:D].tolist() == e_part_wave, name + ": part waves differ from the model"
            for d, e in enumerate(e_parts):
                assert bytes(text[doc_off[d]:doc_off[d + 1]]) == e, "%s: part %d differs from the model" % (name, d)
            t_parts = timed(lambda: parts(L))
            print("| %s | %s | %s | %d | %d | %d | %d | %d | %.2f | %.2f |" % (
                name, label, L_label, W, int(doc_off[D]), D, max(len(p) for p in e_parts), e_part_wave.count(1), t_docs, t_parts),
                flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--topics", type=int, default=240000)
    args = ap.parse_args()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print("GPU:", gpu_info())
    print("| cluster | budget | L | waves W | text bytes | parts D | largest part, bytes | parts of wave 1 "
          "| ka_plan_waves_json, ms | ka_plan_waves_json_parts, ms |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for remove in (0.0, 0.02):
        cl = kab.synth.make_ragged_cluster(T=args.topics, N=400, max_partitions=128, seed=11, remove_frac=remove)
        measure("%d k topics, %d %% removed" % (args.topics // 1000, round(100 * remove)), cl, args.steps, args.warmup, flush)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
