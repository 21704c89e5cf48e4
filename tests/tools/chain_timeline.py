"""Dev tool: the kernel timeline of one warmed dense device solve (c3 by default) under torch.profiler.

Writes, under --out: the Chrome trace of every traced solve (chain_timeline_<n>.pt.trace.json) and a text summary
(chain_timeline.txt). For each kernel-A, slot-0 chain, slot-1 chain and emit launch the summary gives its start and end
(us after the solve's first kernel), its gap to its predecessor on the same chain, the time it was ready (its stream
predecessor and its cross-stream dependency both done) and what else ran on the GPU when it started. Then per solve:
  tail      end of the solve's last kernel - end of its last slot-0 chain
  boundary  start of a slot-0 chain - end of the slot-0 chain before it inside one staged block (a negative gap: the
            launch overlapped its predecessor)
With --subblocks n1,n2,.. the solve is traced once per chain sub-block count (KA_CHAIN_SUBBLOCKS) as well, and the slot-0
chain's span (first start .. last end) is fitted against the number of sub-blocks: the slope is what one more sub-block
boundary costs on the slot-0 path, prologue and epilogue inside the kernels included.
Verifies the default solve's rows against the flat-array CPU solver."""
import argparse
import json
import os
import re
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import kafka_assigner_b200 as kab  # noqa: E402
from oracle import oracle_lib as ol  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="c3")
ap.add_argument("--kind", default="mixed")
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--subblocks", default="", help="comma-separated KA_CHAIN_SUBBLOCKS values traced besides the default")
ap.add_argument("--out", required=True, help="output directory (trace and summary)")
a = ap.parse_args()
os.makedirs(a.out, exist_ok=True)

cl = kab.synth.make_config(a.workload, a.kind)
s = kab.Solver(0)
s.set_brokers(cl.broker_id, cl.rack_index)
s.set_timing(True)   # as bench.py runs it: the timing events are recorded between the launches
stream = torch.cuda.Stream()
d_hash = torch.from_numpy(cl.topic_hash).cuda()
d_cur = torch.from_numpy(cl.cur).cuda()
d_out = torch.empty((cl.T, cl.P, cl.RF), dtype=torch.int32, device="cuda")
d_len = torch.empty((cl.T, cl.P), dtype=torch.int32, device="cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def step(i):
    s.reset()
    flush.fill_(i & 0xFF)
    torch.cuda.synchronize()
    st = s.solve_dense_device(cl.T, d_hash.data_ptr(), cl.P, cl.RF, d_cur.data_ptr(), -1, cl.RF, d_len.data_ptr(), d_out.data_ptr(),
                              stream=stream.cuda_stream)
    assert st.code == 0, st.code


def kind_of(name):
    m = re.search(r"ka_order_levels_kernel<(\d+)", name)
    if m:
        return {"0": "slot0", "1": "slot1"}.get(m.group(1))
    if "ka_emit3_kernel" in name:
        return "emit"
    if "ka_sticky_spread_kernel" in name:
        return "A"
    return None


def trace(label):
    for i in range(a.warmup):
        step(i)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(a.warmup)
        torch.cuda.synchronize()
    path = os.path.join(a.out, "chain_timeline_%s.pt.trace.json" % label)
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    ev = [e for e in ev if kind_of(e["name"]) is not None]
    ev.sort(key=lambda e: e["ts"])
    t0 = ev[0]["ts"]
    rows = [{"kind": kind_of(e["name"]), "start": e["ts"] - t0, "end": e["ts"] + e["dur"] - t0, "stream": e["args"].get("stream")} for e in ev]
    return rows, s.last_timing()


def analyse(rows):
    by = {k: [r for r in rows if r["kind"] == k] for k in ("A", "slot0", "slot1", "emit")}
    K = max(1, len(by["A"]))
    nsub = len(by["slot0"]) // K
    for k, lst in by.items():
        for j, r in enumerate(lst):
            r["j"] = j
            r["gap"] = r["start"] - lst[j - 1]["end"] if j > 0 else None
    # readiness: slot-0 j waits for slot-0 j-1 and for kernel A of its block; slot-1 j for slot-0 j, slot-1 j-1 and, when
    # the emits share its stream, emit j-1; emit j for slot-1 j; kernel A k for kernel A k-1 (its stream)
    for j, r in enumerate(by["slot0"]):
        deps = [by["A"][min(j // max(nsub, 1), K - 1)]["end"]] if by["A"] else []
        if j > 0:
            deps.append(by["slot0"][j - 1]["end"])
        r["ready"] = max(deps) if deps else r["start"]
    for j, r in enumerate(by["slot1"]):
        deps = [by["slot0"][j]["end"]] if j < len(by["slot0"]) else []
        if j > 0:
            deps.append(by["slot1"][j - 1]["end"])
            if j - 1 < len(by["emit"]) and by["emit"][j - 1]["stream"] == r["stream"]:
                deps.append(by["emit"][j - 1]["end"])
        r["ready"] = max(deps) if deps else r["start"]
    for j, r in enumerate(by["emit"]):
        r["ready"] = by["slot1"][j]["end"] if j < len(by["slot1"]) else r["start"]
    for j, r in enumerate(by["A"]):
        r["ready"] = by["A"][j - 1]["end"] if j > 0 else r["start"]
    for r in rows:
        r["busy"] = sorted({o["kind"] for o in rows if o is not r and o["start"] <= r["start"] < o["end"]})
    s0 = by["slot0"]
    bounds = [s0[j]["start"] - s0[j - 1]["end"] for j in range(1, len(s0)) if nsub > 0 and j % nsub != 0]
    xblock = [s0[j]["start"] - s0[j - 1]["end"] for j in range(1, len(s0)) if nsub > 0 and j % nsub == 0]
    end_all = max(r["end"] for r in rows)
    return {
        "K": K, "nsub": nsub, "by": by,
        "tail": end_all - s0[-1]["end"] if s0 else 0.0,
        "last": max(rows, key=lambda r: r["end"])["kind"],
        "bounds": bounds, "xblock": xblock,
        "slot0_span": s0[-1]["end"] - s0[0]["start"] if s0 else 0.0,
        "slot0_sum": sum(r["end"] - r["start"] for r in s0),
        "slot1_sum": sum(r["end"] - r["start"] for r in by["slot1"]),
        "emit_sum": sum(r["end"] - r["start"] for r in by["emit"]),
        "end": end_all,
        "late": [(r["kind"], r["j"], r["start"] - r["ready"], r["busy"]) for r in s0 + by["slot1"]
                 if r["start"] - r["ready"] > 2.0 and ("A" in r["busy"] or "emit" in r["busy"])],
    }


def fmt(v):
    return "%9.1f" % v if v is not None else "        -"


props = torch.cuda.get_device_properties(0)
lines = ["# %s (%s), %d topics x %d partitions RF=%d, %d brokers; one warmed solve_dense_device, timing on" % (
    a.workload, a.kind, cl.T, cl.P, cl.RF, cl.N)]
try:
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    lines.append("# GPU: %s" % q)
except Exception as e:  # noqa: BLE001
    lines.append("# GPU: %s (nvidia-smi: %s)" % (props.name, e))
lines.append("# times in us after the solve's first kernel; gap = start - end of the same chain's previous launch; "
             "wait = start - ready (stream predecessor and cross-stream dependency done)")

os.environ.pop("KA_CHAIN_SUBBLOCKS", None)
rows, tm = trace("default")
exp, exp_len, fst = ol.fast_run_dense(ol.FastContext(), cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index)
ok = fst.code == 0 and np.array_equal(d_out.cpu().numpy().reshape(-1, cl.RF), exp) and np.array_equal(d_len.cpu().numpy().reshape(-1), exp_len)
r = analyse(rows)
lines.append("")
lines.append("## default plan: %d staged blocks x %d chain sub-blocks; rows verified against the CPU solver: %s" % (r["K"], r["nsub"], ok))
lines.append("%-6s %3s %9s %9s %9s %9s %9s  %s" % ("kernel", "j", "start", "end", "dur", "gap", "wait", "running at start"))
for x in sorted(rows, key=lambda x: x["start"]):
    lines.append("%-6s %3d %s %s %s %s %s  %s" % (x["kind"], x["j"], fmt(x["start"]), fmt(x["end"]), fmt(x["end"] - x["start"]), fmt(x["gap"]),
                                                   fmt(x["start"] - x["ready"]), ",".join(x["busy"]) or "-"))
lines.append("")
lines.append("solve (first kernel start .. last kernel end): %.1f us; library total_ms: %.1f us" % (r["end"], tm["total_ms"] * 1e3))
lines.append("slot-0 chain: span %.1f us, kernels %.1f us; slot-1 chain kernels %.1f us; emit kernels %.1f us" % (
    r["slot0_span"], r["slot0_sum"], r["slot1_sum"], r["emit_sum"]))
lines.append("tail (last kernel end - last slot-0 end): %.1f us, last kernel: %s" % (r["tail"], r["last"]))
if r["bounds"]:
    lines.append("slot-0 boundaries inside a block: %d, gap min / median / max %.1f / %.1f / %.1f us" % (
        len(r["bounds"]), min(r["bounds"]), float(np.median(r["bounds"])), max(r["bounds"])))
if r["xblock"]:
    lines.append("slot-0 boundaries between blocks: %s us" % " ".join("%.1f" % v for v in r["xblock"]))
lines.append("chain launches that waited > 2 us past ready while kernel A or emit ran: %s" % (
    "; ".join("%s %d waited %.1f us (%s)" % (k, j, w, ",".join(b)) for k, j, w, b in r["late"]) or "none"))

spans = [(r["K"] * r["nsub"], r["slot0_span"], r["slot0_sum"], r["tail"], r["end"])]
for n in [int(v) for v in a.subblocks.split(",") if v]:
    os.environ["KA_CHAIN_SUBBLOCKS"] = str(n)
    rr = analyse(trace("sub%d" % n)[0])
    spans.append((rr["K"] * rr["nsub"], rr["slot0_span"], rr["slot0_sum"], rr["tail"], rr["end"]))
os.environ.pop("KA_CHAIN_SUBBLOCKS", None)
if len(spans) > 1:
    lines.append("")
    lines.append("## slot-0 chain against the number of sub-blocks per solve (KA_CHAIN_SUBBLOCKS per block)")
    lines.append("%6s %12s %12s %10s %12s" % ("subs", "slot0 span", "slot0 kern", "tail", "solve"))
    for n, sp, sm, tl, en in sorted(spans):
        lines.append("%6d %12.1f %12.1f %10.1f %12.1f" % (n, sp, sm, tl, en))
    x = np.array([v[0] for v in spans], dtype=float)
    if len(set(x)) > 1:
        slope = np.polyfit(x, np.array([v[1] for v in spans]), 1)[0]
        kslope = np.polyfit(x, np.array([v[2] for v in spans]), 1)[0]
        lines.append("cost of one more slot-0 boundary (least-squares slope of the span): %.2f us (of it inside the kernels: %.2f us)" % (slope, kslope))

text = "\n".join(lines) + "\n"
with open(os.path.join(a.out, "chain_timeline.txt"), "w") as f:
    f.write(text)
print(text)
