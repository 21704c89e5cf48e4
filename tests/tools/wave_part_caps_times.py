"""What the part caps (ka_ctx_set_part_caps) cost: ka_plan_waves_json_parts and ka_plan_waves_json_parts_rollback with no caps, a
row cap Lr = 10 000, a data cap Lx (1 000 replicas on the unit plans, 1 000 x the mean weight on the weighted ones) and both,
on the cluster and plans of wave_parts_times.py (the 1.06 M-partition make_ragged_cluster, no broker removed and 2 % removed;
unit weights with a budget of 1, and seeded random weights with a budget of 16 x the mean) at L = 1 048 575.

Each arm is ONE C call from the rows in host memory to every document's text in host memory (pinned buffers of the documented
sufficient sizes), synchronous and timed with the host clock, the L2 flushed (256 MiB written) before it; the median of --steps
calls after --warmup warm-up calls. Before timing, every document, rollback document and part wave of both calls is checked
equal, byte for byte, to the model's cut (tests/part_cap_models.py over the records of models.record /
models.current_record). Prints the GPU, its power limit and SM clock, and a markdown table: D, the largest part's rows and
data (sum of a), and both times."""
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
from tests import models  # noqa: E402
from tests import part_cap_models as pcm  # noqa: E402
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
    back_cap = models.json_bound(cl.topic_names, cl.part_off, 0) + 12 * len(cl.cur)
    text = torch.empty(cap, dtype=torch.uint8).pin_memory().numpy()
    back = torch.empty(back_cap, dtype=torch.uint8).pin_memory().numpy()
    doc_off, back_off = np.zeros(Q + 1, dtype=np.int64), np.zeros(Q + 1, dtype=np.int64)
    doc_wave, wave = np.zeros(Q, dtype=np.int32), np.zeros(Q, dtype=np.int32)
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
        e_wave = models.plan_waves(cl.rep_off, cl.cur, out, out_len, cl.broker_id, B, w)[0]
        recs = pcm.wave_records(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out, out_len, e_wave, w)
        W = len(recs)
        summ = np.zeros(W, dtype=WAVE_SUMMARY_DTYPE)
        rows = (s._h, T, _vp(cl.part_off), _vp(cl.part_id), _vp(cl.rep_off), _vp(cl.cur), 3, _vp(out_len), _vp(out), _vp(w), int(B),
                _vp(names), _vp(name_off), _vp(text), cap, ZNODE, _vp(doc_off), _vp(doc_wave))

        def parts():
            n, d, st = ctypes.c_int32(0), ctypes.c_int32(0), kab.KaStatus()
            rc = s._L.ka_plan_waves_json_parts(*rows, ctypes.byref(d), _vp(wave), ctypes.byref(n), _vp(summ), W, ctypes.byref(st))
            return rc, n.value, d.value

        def rollback():
            n, d, st = ctypes.c_int32(0), ctypes.c_int32(0), kab.KaStatus()
            rc = s._L.ka_plan_waves_json_parts_rollback(*rows, ctypes.byref(d), _vp(back), back_cap, _vp(back_off), _vp(wave),
                                                         ctypes.byref(n), _vp(summ), W, ctypes.byref(st))
            return rc, n.value, d.value

        mean = 1 if w is None else int(w.mean())
        for caps_label, Lr, Lx in (("none", None, None), ("Lr = 10 000", 10000, None), ("Lx = 1 000 x %d" % mean, None, 1000 * mean),
                                   ("both", 10000, 1000 * mean)):
            s.set_part_caps(Lr, Lx)
            times = []
            for is_back, call in ((False, parts), (True, rollback)):
                e_docs, e_backs, e_doc_wave, sizes = pcm.cut_documents(recs, ZNODE, Lr, Lx, is_back)
                D = len(e_docs)
                assert call() == (0, W, D) and np.array_equal(wave, e_wave), "%s %s: device plan differs" % (name, caps_label)
                assert doc_wave[:D].tolist() == e_doc_wave, "%s %s: part waves differ from the model" % (name, caps_label)
                for d in range(D):
                    assert bytes(text[doc_off[d]:doc_off[d + 1]]) == e_docs[d], "%s %s: part %d differs" % (name, caps_label, d)
                    if is_back:
                        assert bytes(back[back_off[d]:back_off[d + 1]]) == e_backs[d], "%s %s: rollback %d differs" % (name, caps_label, d)
                times.append((D, max(r for r, _ in sizes), max(a for _, a in sizes), timed(call)))
            (D, rmax, amax, t_parts), (Db, rbmax, abmax, t_back) = times
            print("| %s | %s | %s | %d | %d | %d | %.2f | %d | %d | %d | %.2f |" % (
                name, label, caps_label, D, rmax, amax, t_parts, Db, rbmax, abmax, t_back), flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--topics", type=int, default=240000)
    args = ap.parse_args()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print("GPU:", gpu_info())
    print("| cluster | plan | caps | parts D | largest part, rows | largest part, data | ka_plan_waves_json_parts, ms "
          "| rollback D | largest, rows | largest, data | ka_plan_waves_json_parts_rollback, ms |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for remove in (0.0, 0.02):
        cl = kab.synth.make_ragged_cluster(T=args.topics, N=400, max_partitions=128, seed=11, remove_frac=remove)
        measure("%d k topics, %d %% removed" % (args.topics // 1000, round(100 * remove)), cl, args.steps, args.warmup, flush)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
