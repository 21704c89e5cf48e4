"""Every part's rollback document, built on the device (ka_plan_waves_json_parts_rollback): what it costs beside
ka_plan_waves_json_parts on the cluster and plans of wave_parts_times.py (the 1.06 M-partition make_ragged_cluster, no broker
removed and 2 % removed; unit weights with a budget of 1, and seeded random weights with a budget of 16 x the mean), and on the
same cluster solved with desired_rf = 2, whose RF-3 topics shrink so that their rollback records are the longer side and drive
the cut. L = 1 048 575 (ZooKeeper's default jute.maxbuffer) and the smallest feasible L (the longest one-record document on
either side).

Three arms, each from the rows in host memory to every document's text in host memory (pinned buffers of the documented
sufficient sizes):
  parts      ONE ka_plan_waves_json_parts call: the forward documents only
  parts+host the same call, then the rollback documents built on the host with numpy and Python (group the changed rows by wave,
             count each part's records, print their current lists): what an operator has to do without the new call. These
             documents follow the forward-only cut, so some may exceed L.
  rollback   ONE ka_plan_waves_json_parts_rollback call
Every step is synchronous and timed with the host clock, the L2 flushed (256 MiB written) before it; the median of --steps steps
after --warmup warm-up steps (--host-steps for the host arm). Before timing, every document of every arm is checked equal, byte
for byte, to the model, models.wave_documents with the limit, one-sided and paired; the host arm's documents to the rollback
documents of the one-sided parts. Prints the GPU, its power limit and SM clock, and a markdown table."""
import argparse
import ctypes
import json
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


def rollback_of(cl, parts):
    """The rollback document of each forward part: its records' partitions on their current lists, in its order."""
    row = {(name, int(cl.part_id[g])): g for t, name in enumerate(cl.topic_names)
           for g in range(int(cl.part_off[t]), int(cl.part_off[t + 1]))}
    docs = []
    for p in parts:
        recs = []
        for r in json.loads(p)["partitions"]:
            g = row[(r["topic"], r["partition"])]
            recs.append(models.current_record(r["topic"], r["partition"], cl.cur[int(cl.rep_off[g]):int(cl.rep_off[g + 1])]))
        docs.append(models.rollback_document(recs).encode())
    return docs


def host_rollback(cl, wave, fwd_text, doc_off, D):
    """The rollback documents of the forward parts, built on the host: the changed rows grouped by wave (stable), each part's
    record count read from its text, and the current lists printed."""
    order = np.argsort(wave, kind="stable")
    order = order[wave[order] > 0]
    topic_of = np.repeat(np.arange(len(cl.topic_names)), np.diff(cl.part_off))
    counts = [bytes(fwd_text[doc_off[d]:doc_off[d + 1]]).count(b'{"partition":') for d in range(D)]
    names, rep_off, cur, part_id = cl.topic_names, cl.rep_off, cl.cur.tolist(), cl.part_id.tolist()
    docs, at = [], 0
    for n in counts:
        rows = order[at:at + n].tolist()
        at += n
        docs.append(('{"version":1,"partitions":[' + ",".join(
            '{"topic":"%s","partition":%d,"replicas":[%s]}' % (names[topic_of[g]], part_id[g], ",".join(map(str, cur[rep_off[g]:rep_off[g + 1]])))
            for g in rows) + "]}").encode())
    return docs


def measure(name, cl, desired_rf, steps, warmup, host_steps, flush):
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    S = 3
    out, out_len, st = s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, desired_rf, S)
    assert st.code == 0
    Q, T = len(out_len), len(cl.topic_names)
    names, name_off = s.marshal_names(cl.topic_names)
    cap = models.json_bound(cl.topic_names, cl.part_off, S)
    back_cap = models.json_bound(cl.topic_names, cl.part_off, 0) + 12 * len(cl.cur)
    text = torch.empty(cap, dtype=torch.uint8).pin_memory().numpy()
    back = torch.empty(back_cap, dtype=torch.uint8).pin_memory().numpy()
    doc_off, back_off = np.zeros(Q + 1, dtype=np.int64), np.zeros(Q + 1, dtype=np.int64)
    doc_wave, wave = np.zeros(Q, dtype=np.int32), np.zeros(Q, dtype=np.int32)
    weight = np.random.default_rng(0x5EED).integers(1, 1 << 34, size=Q, dtype=np.int64)

    def timed(fn, n_steps):
        ms = []
        for i in range(warmup + n_steps):
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
        _, _, _, e_wave, e_summ, e_st = models.wave_documents(*case)
        assert e_st[0] == 0, name + ": refused"
        W = len(e_summ)
        summ = np.zeros(W, dtype=WAVE_SUMMARY_DTYPE)
        rows = (s._h, T, _vp(cl.part_off), _vp(cl.part_id), _vp(cl.rep_off), _vp(cl.cur), S, _vp(out_len), _vp(out), _vp(w), int(B),
                _vp(names), _vp(name_off), _vp(text), cap)

        def parts(L):
            n, d, st = ctypes.c_int32(0), ctypes.c_int32(0), kab.KaStatus()
            rc = s._L.ka_plan_waves_json_parts(*rows, L, _vp(doc_off), _vp(doc_wave), ctypes.byref(d), _vp(wave), ctypes.byref(n),
                                               _vp(summ), W, ctypes.byref(st))
            return rc, n.value, d.value

        def parts_host(L):
            rc, _, D = parts(L)
            return host_rollback(cl, wave, text, doc_off, D)

        def rollback(L):
            n, d, st = ctypes.c_int32(0), ctypes.c_int32(0), kab.KaStatus()
            rc = s._L.ka_plan_waves_json_parts_rollback(*rows, L, _vp(doc_off), _vp(doc_wave), ctypes.byref(d), _vp(back), back_cap,
                                                        _vp(back_off), _vp(wave), ctypes.byref(n), _vp(summ), W, ctypes.byref(st))
            return rc, n.value, d.value

        smallest = util.smallest_limit(*case[:7], e_wave, rollback=True)
        for L_label, L in (("1 048 575", ZNODE), ("smallest, %d" % smallest, smallest)):
            e_fwd = models.wave_documents(*case, L=L)[0]
            e_one_back = rollback_of(cl, e_fwd)
            e_pair, e_pair_back = models.wave_documents(*case, L=L, rollback=True)[:2]
            D1, D2 = len(e_fwd), len(e_pair)
            # arm 1 and arm 2 against the model
            host = parts_host(L)
            assert np.array_equal(wave, e_wave), name + ": device plan differs from the model"
            assert all(bytes(text[doc_off[d]:doc_off[d + 1]]) == e for d, e in enumerate(e_fwd)), name + ": parts differ"
            assert host == e_one_back, name + ": host rollback documents differ from the model"
            over = sum(len(h) > L for h in host)
            # arm 3 against the model
            assert rollback(L) == (0, W, D2) and np.array_equal(wave, e_wave), name + ": device rollback plan differs"
            for d, (e, eb) in enumerate(zip(e_pair, e_pair_back)):
                assert bytes(text[doc_off[d]:doc_off[d + 1]]) == e, "%s: part %d differs from the model" % (name, d)
                assert bytes(back[back_off[d]:back_off[d + 1]]) == eb, "%s: rollback %d differs from the model" % (name, d)
            fwd_bytes, back_bytes = int(doc_off[D2]), int(back_off[D2])
            t_parts = timed(lambda: parts(L), steps)
            t_host = timed(lambda: parts_host(L), host_steps)
            t_back = timed(lambda: rollback(L), steps)
            print("| %s | %s | %s | %d | %d | %d | %d | %d | %d | %.2f | %.0f | %.2f |" % (
                name, label, L_label, W, D1, over, D2, fwd_bytes, back_bytes, t_parts, t_host, t_back), flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-steps", type=int, default=3)
    ap.add_argument("--topics", type=int, default=240000)
    ap.add_argument("--clusters", default="0,1,2", help="which of the three clusters (0 %% removed, 2 %% removed, desired RF 2)")
    args = ap.parse_args()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print("GPU:", gpu_info())
    print("| cluster | plan | L | waves W | parts D, forward-only cut | host rollback documents > L | parts D, paired cut "
          "| forward text bytes | rollback text bytes | parts, ms | parts + host rollback, ms | parts_rollback, ms |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|")
    for k in map(int, args.clusters.split(",")):
        remove, rf = ((0.0, -1), (0.02, -1), (0.0, 2))[k]
        cl = kab.synth.make_ragged_cluster(T=args.topics, N=400, max_partitions=128, seed=11, remove_frac=remove)
        measure("%d k topics, %d %% removed%s" % (args.topics // 1000, round(100 * remove), ", desired RF 2" if rf == 2 else ""), cl, rf,
                args.steps, args.warmup, args.host_steps, flush)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
