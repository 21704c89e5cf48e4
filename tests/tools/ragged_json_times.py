"""Dev tool: what building the reassignment JSON on the device buys on a real-cluster shape (synth.make_ragged_cluster).

Reports, on one instance: the median wall time of ka_solve (rows to host) and of ka_solve_json (text to host) after
warm-up, the size of the text, and the CLI's wall time split into snapshot parsing (PRINT_CURRENT_BROKERS: parse only),
printing the current assignment, and solve + print (PRINT_REASSIGNMENT minus PRINT_CURRENT_ASSIGNMENT, which includes
creating the CUDA context). Prints one JSON line; the card name and power limit are part of it."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

import kafka_assigner_b200 as kab  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--topics", type=int, default=240000)
ap.add_argument("--brokers", type=int, default=400)
ap.add_argument("--max-partitions", type=int, default=128)
ap.add_argument("--seed", type=int, default=11)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--cli-runs", type=int, default=3)
a = ap.parse_args()

cl = kab.synth.make_ragged_cluster(T=a.topics, N=a.brokers, max_partitions=a.max_partitions, seed=a.seed)
s = kab.Solver(0)
s.set_brokers(cl.broker_id, cl.rack_index)
S = max(int(np.diff(cl.rep_off).max()), 1)
cap = 64 + cl.Q * (50 + 12 * S) + int(np.dot(np.diff(cl.part_off), [len(n) for n in cl.topic_names]))
pinned = torch.empty(cap, dtype=torch.uint8).pin_memory().numpy()


def median_ms(fn):
    for _ in range(a.warmup):
        s.reset()
        fn()
    ts = []
    for _ in range(a.steps):
        s.reset()
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


rows_ms = median_ms(lambda: s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, S))
text_ms = median_ms(lambda: s.solve_ragged_json(cl.topic_names, cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1,
                                                json_buf=pinned))
s.reset()   # a fresh Context, like the CLI's
text, st = s.solve_ragged_json(cl.topic_names, cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, json_buf=pinned)
assert st.code == 0

cli = kab.build_mod.build_host()
with tempfile.TemporaryDirectory() as d:
    snap = os.path.join(d, "cluster.json")
    brokers = [dict(id=int(b), host="h%d" % b, port=9092, **({"rack": r} if r is not None else {}))
               for b, r in zip(cl.all_broker_id, cl.all_rack_name)]
    parts = [dict(topic=n, partition=p, replicas=r) for n, asg in cl.topics() for p, r in asg.items()]
    with open(snap, "w") as f:
        json.dump(dict(brokers=brokers, topics=cl.topic_names, partitions=parts), f)

    def cli_ms(mode):
        ts = []
        for _ in range(a.cli_runs):
            t0 = time.perf_counter()
            r = subprocess.run([cli, "--zk_string", "file:" + snap, "--mode", mode], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
            ts.append((time.perf_counter() - t0) * 1e3)
            assert r.returncode == 0, r.stderr[-500:]
        return float(np.median(ts)), r.stdout

    parse_ms, _ = cli_ms("PRINT_CURRENT_BROKERS")
    current_ms, _ = cli_ms("PRINT_CURRENT_ASSIGNMENT")
    reassign_ms, out = cli_ms("PRINT_REASSIGNMENT")
    assert out.endswith(b"NEW ASSIGNMENT:\n" + bytes(text) + b"\n")

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
except OSError:
    power = "?"
print(json.dumps(dict(
    card=torch.cuda.get_device_name(0), power_limit=power, topics=cl.T, partitions=cl.Q, brokers=cl.N, steps=a.steps, warmup=a.warmup,
    ka_solve_rows_to_host_ms=round(rows_ms, 2), ka_solve_json_text_to_host_ms=round(text_ms, 2), text_bytes=len(text),
    cli_runs=a.cli_runs, cli_parse_ms=round(parse_ms, 1), cli_parse_and_print_current_ms=round(current_ms, 1),
    cli_reassignment_ms=round(reassign_ms, 1), cli_solve_and_print_ms=round(reassign_ms - current_ms, 1))))
