"""One reassignment document per wave, built on the device (ka_plan_waves_json): what it costs beside planning the waves and
building the same documents on the host. The 1.06 M-partition make_ragged_cluster of wave_plan_times.py (T = 240 k topics, 10 %
of the brokers joined empty), with no broker removed and with 2 % removed, solved with ka_solve; its rows (all buffers on the
host) then planned
  - with unit weights and a budget of 1 replica per broker per wave, and
  - with a seeded random weight per partition (up to 16 GiB) and a budget of 16 x the mean weight.

Two arms, both starting from the rows in host memory and ending with every document's text in host memory:
  - device: ONE ka_plan_waves_json C call into a pinned text buffer of the documented sufficient size;
  - host:   ONE ka_plan_waves C call, then `host_docs`: a straightforward numpy grouping (stable argsort of the changed rows by
            wave) and Python string formatting of every record. It is what a script around Solver.plan_waves would do, NOT a
            tuned emitter: a compiled one would be much faster.
Every step is synchronous and timed with the host clock, the L2 flushed (256 MiB written) before it; the median of --steps steps
after --warmup warm-up steps. Before timing, the documents of both arms are checked equal, byte for byte, to models.wave_documents
of tests/models.py. Prints the GPU, its power limit and SM clock, and a markdown table."""
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
from tests.tools.cluster_batch_times import gpu_info  # noqa: E402
from tests.tools.wave_plan_times import _vp, plan_once  # noqa: E402


def host_docs(names, part_off, part_id, out, out_len, wave, W):
    """The W documents from the planned waves, on the host: group the changed rows by wave with a stable sort, print each."""
    changed = np.nonzero(wave)[0]
    order = changed[np.argsort(wave[changed], kind="stable")]
    topic_of = np.searchsorted(part_off, order, side="right") - 1
    ends = np.cumsum(np.bincount(wave[changed], minlength=W + 1)[1:]).tolist()
    recs = [models.record(names[t], p, row[:n])
            for p, row, n, t in zip(part_id[order].tolist(), out[order].tolist(), out_len[order].tolist(), topic_of.tolist())]
    return [models.document(recs[a:b]).encode() for a, b in zip([0] + ends[:-1], ends)]


def measure(name, cl, steps, warmup, flush):
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    out, out_len, st = s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, 3)
    assert st.code == 0
    Q, T = len(out_len), len(cl.topic_names)
    names, name_off = s.marshal_names(cl.topic_names)
    cap = models.json_bound(cl.topic_names, cl.part_off, 3)
    text = torch.empty(cap, dtype=torch.uint8).pin_memory().numpy()
    doc_off, wave = np.zeros(Q + 1, dtype=np.int64), np.zeros(Q, dtype=np.int32)
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
        e_docs, _, _, e_wave, e_summ, e_st = models.wave_documents(cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, out,
                                                                   out_len, cl.broker_id, B, w)
        assert e_st[0] == 0, name + ": refused"
        W = len(e_docs)
        summ = np.zeros(W, dtype=WAVE_SUMMARY_DTYPE)

        def device():
            n, st = ctypes.c_int32(0), kab.KaStatus()
            rc = s._L.ka_plan_waves_json(s._h, T, _vp(cl.part_off), _vp(cl.part_id), _vp(cl.rep_off), _vp(cl.cur), 3, _vp(out_len),
                                         _vp(out), _vp(w), int(B), _vp(names), _vp(name_off), _vp(text), cap, _vp(doc_off), _vp(wave),
                                         ctypes.byref(n), _vp(summ), W, ctypes.byref(st))
            return rc, n.value

        def host():
            assert plan_once(s, cl.rep_off, cl.cur, out, out_len, B, w, wave, summ) == (0, W)
            return host_docs(cl.topic_names, cl.part_off, cl.part_id, out, out_len, wave, W)

        assert device() == (0, W) and np.array_equal(wave, e_wave), name + ": device plan differs from the model"
        for v, e in enumerate(e_docs):
            assert bytes(text[doc_off[v]:doc_off[v + 1]]) == e, "%s: document %d differs from the model" % (name, v)
        assert host() == e_docs, name + ": host documents differ from the model"
        t_plan = timed(lambda: plan_once(s, cl.rep_off, cl.cur, out, out_len, B, w, wave, summ))
        t_dev = timed(device)
        t_host = timed(host)
        print("| %s | %s | %d | %d | %d | %d | %.2f | %.2f | %.0f |" % (name, label, Q, int((e_wave > 0).sum()), W, int(doc_off[W]),
                                                                       t_plan, t_dev, t_host), flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--topics", type=int, default=240000)
    args = ap.parse_args()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print("GPU:", gpu_info())
    print("| cluster | budget | partitions | rows changed | waves W | text bytes | ka_plan_waves alone, ms "
          "| ka_plan_waves_json, one C call, ms | ka_plan_waves + numpy / Python documents on the host, ms |")
    print("|---|---|---|---|---|---|---|---|---|")
    for remove in (0.0, 0.02):
        cl = kab.synth.make_ragged_cluster(T=args.topics, N=400, max_partitions=128, seed=11, remove_frac=remove)
        measure("%d k topics, %d %% removed" % (args.topics // 1000, round(100 * remove)), cl, args.steps, args.warmup, flush)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
