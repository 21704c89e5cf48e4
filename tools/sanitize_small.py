"""Small end-to-end cases for compute-sanitizer (memcheck): dense + ragged + error + 8-slot rows + pipelined, a wave plan with its
rollback documents, the broker usage of that plan, a fleet's documents and a scored candidate batch. Every Solver is closed, so
that --leak-check full sees each Context's buffers freed."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kafka_assigner_b200 as kab  # noqa: E402

solvers = []


def solver():
    s = kab.Solver(0)
    solvers.append(s)
    return s


cl = kab.synth.make_cluster(T=12, P=19, RF=3, N=30, R=5, seed=5, kind="mixed")
out, out_len, st = solver().solve_cluster(cl)
assert st.code == 0
a = kab.KafkaTopicAssigner()
solvers.append(a._solver)
print(a.generate_assignment("test", {0: [10, 11], 1: [11, 12], 2: [12, 10], 3: [10, 12]}, {10, 11, 13}, {}, -1))
print(a.generate_assignment("wide", {p: [1 + (p + i) % 9 for i in range(6)] for p in range(7)}, set(range(1, 12)), {}, -1))
try:
    a.generate_assignment("t", {0: [1, 2], 1: [2, 1]}, {1, 2, 3}, {1: "x", 2: "x", 3: "y"}, 3)
except kab.IllegalStateException as e:
    print("expected:", e)
big = kab.synth.make_cluster(T=40, P=16, RF=3, N=2000, R=20, seed=4, kind="random")   # global-LUT-free, larger table
print(solver().solve_cluster(big)[2].code)
lv = kab.synth.make_cluster(T=30, P=90, RF=3, N=60, R=6, seed=9, kind="mixed")      # capacity 5: conflict levels, chunk table, window mode
print(solver().solve_cluster(lv)[2].code)
wide = kab.synth.make_cluster(T=40, P=160, RF=3, N=600, R=6, seed=10, kind="mixed")  # capacity 1, 160-wide topics: bounds-free chain loop
s = solver()
s.set_brokers(wide.broker_id, wide.rack_index)
text, st = s.solve_dense_json(wide.topic_names, wide.topic_hash, wide.cur)            # + the device-side JSON emitter
print(st.code, len(text))
rg = kab.synth.make_ragged_cluster(T=200, N=40, max_partitions=16, seed=6, remove_frac=0.05)
w = solver()
w.set_brokers(rg.broker_id, rg.rack_index)
S = max(int(np.diff(rg.rep_off).max()), 1)
new, new_len, st = w.solve_ragged(rg.topic_hash, rg.part_off, rg.part_id, rg.rep_off, rg.cur, -1, S)
assert st.code == 0
parts, rollback, part_wave, wave, summary, st = w.plan_wave_parts_rollback_json(rg.topic_names, rg.part_off, rg.part_id, rg.rep_off,
                                                                                 rg.cur, new, new_len, 2, 4096)
print(st.code, len(parts), len(rollback))
usage, W, st = w.broker_usage(rg.rep_off, rg.cur, new, new_len, wave, rg.all_broker_id)
print(st.code, W, len(usage))
fleet = [kab.synth.make_ragged_cluster(T=30, N=20, max_partitions=8, seed=11 + k) for k in range(3)]
docs = solver().solve_clusters_json([(f.broker_id, f.rack_index, f.topic_hash, f.part_off, f.part_id, f.rep_off, f.cur, -1)
                                     for f in fleet], [f.topic_names for f in fleet])   # the batch table image + the fleet segments
print([(st.code, len(text)) for text, st in docs])
tables = [(rg.broker_id, rg.rack_index), (rg.broker_id[::2], rg.rack_index[::2])]
summary, sts, rep, lead, added = w.score_ragged_candidates(tables, rg.topic_hash, rg.part_off, rg.part_id, rg.rep_off, rg.cur, -1,
                                                           weight=np.arange(rg.Q), per_broker=True)
print([st.code for st in sts], summary["rows_moved"].tolist(), [len(a) for a in rep])
for s in solvers:
    s.close()
print("sanitize cases done")
