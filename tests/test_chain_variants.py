"""Every instantiation of the leader-order chain kernel (ka_order_levels_kernel) against the oracle.

launch_order picks one instantiation per call from the solve's plan: the record kind (rows <= 3 as two slot chains, rows of 4
and rows of 5..8 as one fused chain), where the counters live (shared memory or global memory, GCTR), the ring size, the loop
shape (WARP1 window mode, SINGLE, FULL, or general over uniform levels or the chunk table) and CAND (a batched candidate solve).
Each case below names the plan it must reach, checked through ka_ctx_last_order_plan, so that a case cannot drift to another
variant when a heuristic changes; then its rows must equal the oracle's and, for single solves, the Context counters must
equal the per-position histogram of the oracle's rows.

Plan tuples: (rec_kind, levels, chain threads, ring_log2, gctr, loop shape, chain launches of the call, candidates K).
Counter bands (make_plan): rows <= 3 keep (N + 1) int32 per slot chain next to the ring, so ring_log2 is 10 up to N = 25 023,
9 up to 41 407, 8 up to 49 599, 7 up to 53 695, and the counters go to global memory beyond. Rows of 4 keep 4 int32 per
broker: ring_log2 9 / 8 / 7 up to N = 6 256 / 10 352 / 12 400; rows of 5..8 keep 8: up to 3 128 / 5 176 / 6 200. Kernel A's
level scratch caps level plans (capacity > 1, ragged) at about 18 600 brokers, so the shrunk-ring and natural-GCTR cells of
the slot chains are capacity-1 problems.
"""
import ctypes
import os
import re
from unittest import mock

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from tests import models, util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

GENERAL, WARP1, SINGLE, FULL = 0, 1, 2, 3
GCTR = {"KA_ORDER_GLOBAL_CTR": "1"}


def _case(cid, plan, env=None, **gen):
    return dict(id=cid, plan=plan, env=dict(env or {}), gen=gen)


def _threads(n):
    return {"KA_ORDER_THREADS": str(n)}


# ---- single dense solves (ka_solve_dense): gen = make_cluster arguments (+ desired_rf) -----------------------------------
SINGLE_CASES = [
    # rows <= 3, counters in shared memory, ring_log2 10
    _case("r10-warp1-uniform", (3, 0, 32, 10, 0, WARP1, 2, 0), T=40, P=24, RF=3, N=200, R=10),
    _case("r10-warp1-table", (3, 1, 32, 10, 0, WARP1, 2, 0), T=40, P=60, RF=3, N=70, R=7),
    _case("r10-single-p33", (3, 0, 64, 10, 0, SINGLE, 2, 0), T=30, P=33, RF=3, N=400, R=10),
    _case("r10-single-p100", (3, 0, 128, 10, 0, SINGLE, 2, 0), T=30, P=100, RF=3, N=400, R=10),
    _case("r10-single-p700", (3, 0, 704, 10, 0, SINGLE, 2, 0), T=12, P=700, RF=2, N=1500, R=10),
    _case("r10-full-p128", (3, 0, 128, 10, 0, FULL, 2, 0), T=30, P=128, RF=3, N=400, R=10),
    _case("r10-full-p1024", (3, 0, 1024, 10, 0, FULL, 2, 0), T=4, P=1024, RF=2, N=2100, R=10),
    _case("r10-general-uniform-p1025", (3, 0, 544, 10, 0, GENERAL, 2, 0), T=4, P=1025, RF=2, N=2100, R=10),
    _case("r10-general-uniform-p1500", (3, 0, 768, 10, 0, GENERAL, 2, 0), T=4, P=1500, RF=2, N=3100, R=10),
    _case("r10-general-table", (3, 1, 64, 10, 0, GENERAL, 2, 0), T=40, P=200, RF=3, N=250, R=10),
    _case("r10-general-table-wide", (3, 1, 512, 10, 0, GENERAL, 2, 0), T=12, P=2500, RF=3, N=3000, R=10),
    # ring edges: Q = 8 << ring_log2 records, and one past it
    _case("r10-q8192", (3, 0, 128, 10, 0, FULL, 2, 0), T=64, P=128, RF=3, N=400, R=10),
    _case("r10-q8193", (3, 0, 928, 10, 0, GENERAL, 2, 0), T=3, P=2731, RF=2, N=6000, R=10),
    # ring_log2 9 / 8 / 7 (capacity 1, global id LUT)
    _case("r9-warp1", (3, 0, 32, 9, 0, WARP1, 2, 0), T=6, P=24, RF=3, N=30000, R=10),
    _case("r9-single-p100", (3, 0, 128, 9, 0, SINGLE, 2, 0), T=6, P=100, RF=3, N=30000, R=10),
    _case("r9-full-p256", (3, 0, 256, 9, 0, FULL, 2, 0), T=6, P=256, RF=3, N=30000, R=10),
    _case("r9-general-p1025", (3, 0, 544, 9, 0, GENERAL, 2, 0), T=4, P=1025, RF=3, N=30000, R=10),
    _case("r8-warp1", (3, 0, 32, 8, 0, WARP1, 2, 0), T=6, P=24, RF=3, N=45000, R=10),
    _case("r8-single-p33", (3, 0, 64, 8, 0, SINGLE, 2, 0), T=6, P=33, RF=3, N=45000, R=10),
    _case("r8-full-p128", (3, 0, 128, 8, 0, FULL, 2, 0), T=6, P=128, RF=3, N=45000, R=10),
    _case("r8-general-p1500", (3, 0, 768, 8, 0, GENERAL, 2, 0), T=4, P=1500, RF=3, N=45000, R=10),
    _case("r7-warp1", (3, 0, 32, 7, 0, WARP1, 2, 0), T=6, P=24, RF=3, N=52000, R=10),
    _case("r7-single-p700", (3, 0, 704, 7, 0, SINGLE, 2, 0), T=4, P=700, RF=3, N=52000, R=10),      # ring stage 128 < P
    _case("r7-full-p896", (3, 0, 896, 7, 0, FULL, 2, 0), T=4, P=896, RF=3, N=52000, R=10),         # the 896-thread cap
    _case("r7-general-p1000", (3, 0, 896, 7, 0, GENERAL, 2, 0), T=4, P=1000, RF=3, N=52000, R=10),
    _case("r7-general-p1500", (3, 0, 768, 7, 0, GENERAL, 2, 0), T=4, P=1500, RF=3, N=52000, R=10),
    _case("r7-q1024", (3, 0, 128, 7, 0, FULL, 2, 0), T=8, P=128, RF=3, N=52000, R=10),
    _case("r7-q1025", (3, 0, 64, 7, 0, SINGLE, 2, 0), T=25, P=41, RF=3, N=52000, R=10),
    # counters beyond shared memory
    _case("gctr-warp1", (3, 0, 32, 10, 1, WARP1, 2, 0), T=6, P=24, RF=3, N=56000, R=10),
    _case("gctr-single-p700", (3, 0, 704, 10, 1, SINGLE, 2, 0), T=4, P=700, RF=3, N=56000, R=10),
    _case("gctr-full-p1024", (3, 0, 1024, 10, 1, FULL, 2, 0), T=4, P=1024, RF=3, N=56000, R=10),
    _case("gctr-general-p1025", (3, 0, 544, 10, 1, GENERAL, 2, 0), T=4, P=1025, RF=3, N=56000, R=10),
    # counters forced into global memory
    _case("fgctr-warp1-uniform", (3, 0, 32, 10, 1, WARP1, 2, 0), GCTR, T=40, P=24, RF=3, N=200, R=10),
    _case("fgctr-warp1-table", (3, 1, 32, 10, 1, WARP1, 2, 0), GCTR, T=40, P=60, RF=3, N=70, R=7),
    _case("fgctr-single-p100", (3, 0, 128, 10, 1, SINGLE, 2, 0), GCTR, T=30, P=100, RF=3, N=400, R=10),
    _case("fgctr-full-p128", (3, 0, 128, 10, 1, FULL, 2, 0), GCTR, T=30, P=128, RF=3, N=400, R=10),
    _case("fgctr-general-uniform-p1025", (3, 0, 544, 10, 1, GENERAL, 2, 0), GCTR, T=4, P=1025, RF=2, N=2100, R=10),
    _case("fgctr-general-table", (3, 1, 64, 10, 1, GENERAL, 2, 0), GCTR, T=40, P=200, RF=3, N=250, R=10),
    _case("fgctr-r9-single-p100", (3, 0, 128, 9, 1, SINGLE, 2, 0), GCTR, T=6, P=100, RF=3, N=30000, R=10),
    # KA_ORDER_THREADS
    _case("threads32-p100", (3, 0, 32, 10, 0, WARP1, 2, 0), _threads(32), T=30, P=100, RF=3, N=400, R=10),
    _case("threads64-p100", (3, 0, 64, 10, 0, GENERAL, 2, 0), _threads(64), T=30, P=100, RF=3, N=400, R=10),
    _case("threads100-p100", (3, 0, 96, 10, 0, GENERAL, 2, 0), _threads(100), T=30, P=100, RF=3, N=400, R=10),
    _case("threads100-table", (3, 1, 96, 10, 0, GENERAL, 2, 0), _threads(100), T=40, P=200, RF=3, N=250, R=10),
    _case("threads32-r7-p700", (3, 0, 32, 7, 0, WARP1, 2, 0), _threads(32), T=4, P=700, RF=3, N=52000, R=10),
    # KA_CHAIN_SUBBLOCKS on an odd topic count (sub-block edges fall mid-run); 301 topics cut in 2 by default
    _case("sub-default-uniform", (3, 0, 64, 10, 0, SINGLE, 4, 0), T=301, P=40, RF=3, N=200, R=10),
    _case("sub1-uniform", (3, 0, 64, 10, 0, SINGLE, 2, 0), {"KA_CHAIN_SUBBLOCKS": "1"}, T=301, P=40, RF=3, N=200, R=10),
    _case("sub3-uniform", (3, 0, 64, 10, 0, SINGLE, 6, 0), {"KA_CHAIN_SUBBLOCKS": "3"}, T=301, P=40, RF=3, N=200, R=10),
    _case("sub8-uniform", (3, 0, 64, 10, 0, SINGLE, 16, 0), {"KA_CHAIN_SUBBLOCKS": "8"}, T=301, P=40, RF=3, N=200, R=10),
    _case("sub1-table", (3, 1, 64, 10, 0, GENERAL, 2, 0), {"KA_CHAIN_SUBBLOCKS": "1"}, T=301, P=200, RF=3, N=250, R=10),
    _case("sub3-table", (3, 1, 64, 10, 0, GENERAL, 6, 0), {"KA_CHAIN_SUBBLOCKS": "3"}, T=301, P=200, RF=3, N=250, R=10),
    _case("sub8-table", (3, 1, 64, 10, 0, GENERAL, 16, 0), {"KA_CHAIN_SUBBLOCKS": "8"}, T=301, P=200, RF=3, N=250, R=10),
    _case("sub3-warp1-table", (3, 1, 32, 10, 0, WARP1, 6, 0), {"KA_CHAIN_SUBBLOCKS": "3"}, T=301, P=60, RF=3, N=70, R=7),
    # KA_PIPELINE_STAGES: topic super-chunks of an odd topic count, one chain pair per chunk
    _case("pipe2-table", (3, 1, 64, 10, 0, GENERAL, 4, 0), {"KA_PIPELINE_STAGES": "2"}, T=301, P=200, RF=3, N=250, R=10),
    _case("pipe5-table", (3, 1, 64, 10, 0, GENERAL, 10, 0), {"KA_PIPELINE_STAGES": "5"}, T=301, P=200, RF=3, N=250, R=10),
    _case("pipe8-table", (3, 1, 64, 10, 0, GENERAL, 16, 0), {"KA_PIPELINE_STAGES": "8"}, T=301, P=200, RF=3, N=250, R=10),
    _case("pipe5-uniform", (3, 0, 64, 10, 0, SINGLE, 10, 0), {"KA_PIPELINE_STAGES": "5"}, T=301, P=40, RF=3, N=200, R=10),
    # rows of 4: one fused chain
    _case("w4-r9-32", (4, 0, 32, 9, 0, GENERAL, 1, 0), T=20, P=24, RF=4, N=200, R=8),
    _case("w4-r9-wide", (4, 0, 224, 9, 0, GENERAL, 1, 0), T=10, P=200, RF=4, N=1000, R=8),
    _case("w4-r9-table", (4, 1, 128, 9, 0, GENERAL, 1, 0), T=20, P=600, RF=4, N=1000, R=8),
    _case("w4-r8-32", (4, 0, 32, 8, 0, GENERAL, 1, 0), T=6, P=24, RF=4, N=8000, R=8),
    _case("w4-r8-wide", (4, 0, 224, 8, 0, GENERAL, 1, 0), T=6, P=200, RF=4, N=8000, R=8),
    _case("w4-r7-32", (4, 0, 32, 7, 0, GENERAL, 1, 0), T=6, P=24, RF=4, N=12000, R=8),
    _case("w4-r7-wide", (4, 0, 512, 7, 0, GENERAL, 1, 0), T=6, P=500, RF=4, N=12000, R=8),
    _case("w4-r7-table", (4, 1, 512, 7, 0, GENERAL, 1, 0), T=3, P=3100, RF=4, N=12000, R=8),
    _case("w4-gctr-32", (4, 0, 32, 9, 1, GENERAL, 1, 0), T=6, P=24, RF=4, N=14000, R=8),
    _case("w4-gctr-wide", (4, 0, 224, 9, 1, GENERAL, 1, 0), T=6, P=200, RF=4, N=14000, R=8),
    _case("w4-gctr-table", (4, 1, 448, 9, 1, GENERAL, 1, 0), T=3, P=3600, RF=4, N=14000, R=8),
    _case("w4-fgctr-32", (4, 0, 32, 9, 1, GENERAL, 1, 0), GCTR, T=20, P=24, RF=4, N=200, R=8),
    _case("w4-fgctr-table", (4, 1, 128, 9, 1, GENERAL, 1, 0), GCTR, T=20, P=600, RF=4, N=1000, R=8),
    _case("w4-fgctr-threads32-table", (4, 1, 32, 9, 1, GENERAL, 1, 0), dict(GCTR, **_threads(32)), T=20, P=600, RF=4, N=1000, R=8),
    # rows of 5..8: one fused chain over 8 slots (RF 5 / 6, or RF 3 grown to 6)
    _case("w8-r9-32", (8, 0, 32, 9, 0, GENERAL, 1, 0), T=20, P=24, RF=6, N=300, R=6),
    _case("w8-r9-wide", (8, 0, 160, 9, 0, GENERAL, 1, 0), T=10, P=150, RF=6, N=1000, R=6),
    _case("w8-r9-table", (8, 1, 96, 9, 0, GENERAL, 1, 0), T=20, P=400, RF=6, N=1000, R=6),
    _case("w5-r9-wide", (8, 0, 64, 9, 0, GENERAL, 1, 0), T=20, P=40, RF=5, N=500, R=6),
    _case("w8-r8-32", (8, 0, 32, 8, 0, GENERAL, 1, 0), T=6, P=24, RF=6, N=4000, R=6),
    _case("w8-r8-wide-grow6", (8, 0, 224, 8, 0, GENERAL, 1, 0), T=6, P=200, RF=3, N=4000, R=6, desired_rf=6),
    _case("w8-r7-32", (8, 0, 32, 7, 0, GENERAL, 1, 0), T=6, P=24, RF=6, N=6000, R=6),
    _case("w8-r7-wide", (8, 0, 256, 7, 0, GENERAL, 1, 0), T=6, P=250, RF=6, N=6000, R=6),
    _case("w8-r7-table-grow6", (8, 1, 256, 7, 0, GENERAL, 1, 0), T=3, P=1200, RF=3, N=6000, R=6, desired_rf=6),
    _case("w8-gctr-32", (8, 0, 32, 9, 1, GENERAL, 1, 0), T=6, P=24, RF=6, N=7000, R=6),
    _case("w8-gctr-wide-grow6", (8, 0, 224, 9, 1, GENERAL, 1, 0), T=6, P=200, RF=3, N=7000, R=6, desired_rf=6),
    _case("w8-fgctr-32", (8, 0, 32, 9, 1, GENERAL, 1, 0), GCTR, T=20, P=24, RF=6, N=300, R=6),
    _case("w8-fgctr-table", (8, 1, 96, 9, 1, GENERAL, 1, 0), GCTR, T=20, P=400, RF=6, N=1000, R=6),
]

# ---- batched dense candidates (ka_solve_dense_candidates_device): the cluster's own table + tables = [(n, racks_per)], ids
# 1000 + i. All tables have capacity 1 where the largest is beyond kernel A's level scratch; small tables run under a big-N plan.
CAND_CASES = [
    _case("cand-r10-warp1", (3, 0, 32, 10, 0, WARP1, 2, 3), T=30, P=24, RF=3, N=200, R=10, tables=[(150, 15), (5000, 50)]),
    _case("cand-r10-warp1-table", (3, 1, 32, 10, 0, WARP1, 2, 2), T=30, P=40, RF=3, N=28, R=4, tables=[(70, 7)]),
    _case("cand-r10-single", (3, 0, 128, 10, 0, SINGLE, 2, 3), T=30, P=100, RF=3, N=400, R=10, tables=[(400, 40), (5000, 50)]),
    _case("cand-r10-full", (3, 0, 128, 10, 0, FULL, 2, 3), T=30, P=128, RF=3, N=400, R=10, tables=[(480, 32), (5000, 50)]),
    _case("cand-r10-general-uniform", (3, 0, 544, 10, 0, GENERAL, 2, 3), T=4, P=1025, RF=2, N=2100, R=10,
          tables=[(2600, 50), (20000, 500)]),
    _case("cand-r10-general-table", (3, 1, 64, 10, 0, GENERAL, 2, 3), T=30, P=40, RF=3, N=28, R=4, tables=[(26, 2), (3000, 30)]),
    _case("cand-r9-single", (3, 0, 128, 9, 0, SINGLE, 2, 3), T=6, P=100, RF=3, N=400, R=10, tables=[(400, 40), (30000, 500)]),
    _case("cand-r7-warp1", (3, 0, 32, 7, 0, WARP1, 2, 3), T=6, P=24, RF=3, N=200, R=10, tables=[(100, 10), (52000, 500)]),
    _case("cand-r7-single-p700", (3, 0, 704, 7, 0, SINGLE, 2, 3), T=4, P=700, RF=2, N=1500, R=10, tables=[(1800, 20), (52000, 500)]),
    _case("cand-r7-full-p896", (3, 0, 896, 7, 0, FULL, 2, 3), T=4, P=896, RF=2, N=1800, R=10, tables=[(2300, 32), (52000, 500)]),
    _case("cand-r7-general-p1025", (3, 0, 544, 7, 0, GENERAL, 2, 3), T=4, P=1025, RF=2, N=2100, R=10,
          tables=[(2600, 50), (52000, 500)]),
    _case("cand-gctr-warp1", (3, 0, 32, 10, 1, WARP1, 2, 3), T=6, P=24, RF=3, N=200, R=10, tables=[(100, 10), (56000, 500)]),
    _case("cand-gctr-single", (3, 0, 128, 10, 1, SINGLE, 2, 3), T=6, P=100, RF=3, N=400, R=10, tables=[(400, 40), (56000, 500)]),
    _case("cand-gctr-full", (3, 0, 128, 10, 1, FULL, 2, 3), T=6, P=128, RF=3, N=400, R=10, tables=[(480, 32), (56000, 500)]),
    _case("cand-gctr-general", (3, 0, 544, 10, 1, GENERAL, 2, 3), T=4, P=1025, RF=2, N=2100, R=10,
          tables=[(2600, 50), (56000, 500)]),
    _case("cand-fgctr-warp1", (3, 0, 32, 10, 1, WARP1, 2, 3), GCTR, T=30, P=24, RF=3, N=200, R=10, tables=[(150, 15), (5000, 50)]),
    _case("cand-fgctr-warp1-table", (3, 1, 32, 10, 1, WARP1, 2, 2), GCTR, T=30, P=40, RF=3, N=28, R=4, tables=[(70, 7)]),
    _case("cand-fgctr-single", (3, 0, 128, 10, 1, SINGLE, 2, 3), GCTR, T=30, P=100, RF=3, N=400, R=10,
          tables=[(400, 40), (5000, 50)]),
    _case("cand-fgctr-full", (3, 0, 128, 10, 1, FULL, 2, 3), GCTR, T=30, P=128, RF=3, N=400, R=10, tables=[(480, 32), (5000, 50)]),
    _case("cand-fgctr-general-uniform", (3, 0, 544, 10, 1, GENERAL, 2, 3), GCTR, T=4, P=1025, RF=2, N=2100, R=10,
          tables=[(2600, 50), (20000, 500)]),
    _case("cand-fgctr-general-table", (3, 1, 64, 10, 1, GENERAL, 2, 3), GCTR, T=30, P=40, RF=3, N=28, R=4,
          tables=[(26, 2), (3000, 30)]),
    _case("cand-sub3-table", (3, 1, 64, 10, 0, GENERAL, 6, 2), {"KA_CHAIN_SUBBLOCKS": "3"}, T=301, P=40, RF=3, N=28, R=4,
          tables=[(3000, 30)]),
]

# ---- batched ragged candidates (ka_solve_candidates): make_ragged_cluster(T=80, N=40, R=5, max_partitions=64) and tables
# [(n, racks_per, id step)], ids 1 + step * i
RAGGED_CAND_CASES = [
    _case("rcand-fgctr-threads32-warp1", (3, 1, 32, 10, 1, WARP1, 2, 4), dict(GCTR, **_threads(32)), seed=1,
          tables=[(36, 3, 1), (3000, 30, 1), (20000, 500, 2)]),
    _case("rcand-fgctr-threads128-table", (3, 1, 128, 10, 1, GENERAL, 2, 4), dict(GCTR, **_threads(128)), seed=2,
          tables=[(36, 3, 1), (3000, 30, 1), (20000, 500, 2)]),
    _case("rcand-warp1", (3, 1, 32, 10, 0, WARP1, 2, 3), seed=3, tables=[(36, 3, 1), (120, 6, 1)]),
]

# ---- one Context across variants: N = 3 000 brokers throughout, the counters carry from call to call ---------------------
SEQUENCE = [
    _case("seq-capacity1-single", (3, 0, 512, 10, 0, SINGLE, 2, 0), T=20, P=500, RF=3),
    _case("seq-capacity3-table", (3, 1, 512, 10, 0, GENERAL, 2, 0), T=10, P=2500, RF=3),
    _case("seq-capacity3-table-gctr", (3, 1, 512, 10, 1, GENERAL, 2, 0), GCTR, T=10, P=2500, RF=3),
    _case("seq-capacity3-threads32", (3, 1, 32, 10, 0, WARP1, 2, 0), _threads(32), T=10, P=2500, RF=3),
    _case("seq-capacity1-p1500", (3, 0, 768, 10, 0, GENERAL, 2, 0), T=4, P=1500, RF=2),
]
SEQUENCE_N, SEQUENCE_R = 3000, 10

# ---- broker tables in every id -> index lookup mode, in one batch ------------------------------------------------------
LUT_DENSE_PLAN = (3, 1, 32, 10, 0, WARP1, 2, 4)
LUT_RAGGED_PLAN = (3, 1, 32, 10, 0, WARP1, 2, 4)

ALL_PLANS = [c["plan"] for c in SINGLE_CASES + CAND_CASES + RAGGED_CAND_CASES + SEQUENCE] + [LUT_DENSE_PLAN, LUT_RAGGED_PLAN]


def _seed(cid):
    return 0xC4A1 + sum(ord(ch) * (i + 1) for i, ch in enumerate(cid))


# ---- CPU ------------------------------------------------------------------------------------------------------------------

def _dispatch_from_source():
    """(reachable (rec_kind, cand, gctr, shape) dispatches, {rec_kind: ring_log2 values}) read from kassign.cu: the
    instantiations launch_order can launch and make_plan's ring range."""
    src = open(os.path.join(ROOT, "kafka_assigner_b200", "csrc", "kassign.cu")).read()
    body = re.search(r"cudaError_t launch_order\(.*?\n}\n", src, flags=re.S).group(0)
    fused, slots = body.split("} else {", 1)
    pat = r"launch_order_t<KIND, MAXNT, (CAND|false), (true|false), (true|false), (true|false), (true|false)>"
    out = set()
    for part, kinds in ((fused, (4, 8)), (slots, (3,))):
        for cand, gctr, single, warp1, full in re.findall(pat, part):
            shape = WARP1 if warp1 == "true" else (FULL if full == "true" else (SINGLE if single == "true" else GENERAL))
            for kind in kinds:
                for c in ((0, 1) if cand == "CAND" else (0,)):
                    out.add((kind, c, int(gctr == "true"), shape))
    lg = re.search(r"const int lg_max = pl\.rec_kind == 3 \? (\d+) : (\d+), lg_min = (\d+);", src)
    assert lg, "make_plan's ring range moved: update this test"
    hi3, hi, lo = (int(x) for x in lg.groups())
    rings = {3: set(range(lo, hi3 + 1)), 4: set(range(lo, hi + 1)), 8: set(range(lo, hi + 1))}
    return out, rings


def test_case_table_names_every_dispatch_and_ring():
    reachable, rings = _dispatch_from_source()
    assert len(reachable) == 20, sorted(reachable)   # rows <= 3: 2 CAND x 2 GCTR x 4 shapes; rows of 4 / 5..8: 2 GCTR each
    named = {(p[0], int(p[7] > 0), p[4], p[5]) for p in ALL_PLANS}
    assert reachable - named == set(), "dispatches without a case: %s" % sorted(reachable - named)
    assert named <= reachable, "cases naming a dispatch launch_order cannot make: %s" % sorted(named - reachable)
    for kind, lgs in rings.items():
        # counters in shared memory at every ring size, and in global memory
        got = {p[3] for p in ALL_PLANS if p[0] == kind and not p[4]}
        assert lgs <= got, (kind, sorted(lgs - got))
        assert any(p[0] == kind and p[4] for p in ALL_PLANS), kind
    ids = [c["id"] for c in SINGLE_CASES + CAND_CASES + RAGGED_CAND_CASES + SEQUENCE]
    assert len(ids) == len(set(ids))


def test_last_order_plan_null_arguments(native_lib):
    plan = np.zeros(8, dtype=np.int32)
    assert native_lib.ka_ctx_last_order_plan(None, plan.ctypes.data_as(ctypes.c_void_p)) == _native.KA_ERR_BAD_ARG
    assert native_lib.ka_ctx_last_order_plan(None, None) == _native.KA_ERR_BAD_ARG
    assert not plan.any()


# ---- GPU ------------------------------------------------------------------------------------------------------------------

def _cluster(g, seed):
    cl = kab.synth.make_cluster(T=g["T"], P=g["P"], RF=g["RF"], N=g["N"], R=g["R"], seed=seed, kind="mixed")
    cl.desired_rf = g.get("desired_rf", -1)
    return cl


@pytest.mark.gpu
@pytest.mark.parametrize("case", SINGLE_CASES, ids=[c["id"] for c in SINGLE_CASES])
def test_single_solve_variant(native_lib, oracle, case):
    g = case["gen"]
    cl = _cluster(g, _seed(case["id"]))
    S = max(cl.RF, cl.desired_rf, 1)
    exp, exp_len, est = oracle.fast_run_dense(oracle.FastContext(), cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index,
                                              cl.desired_rf, S)
    assert est.code == 0
    s = kab.Solver(0)
    with mock.patch.dict(os.environ, case["env"]):
        out, out_len, st = s.solve_cluster(cl, check=False)
    assert s.last_order_plan() == case["plan"]
    assert st.code == 0, (st.code, st.topic_index, st.a, st.b)
    assert np.array_equal(out.reshape(-1, S), exp)
    assert np.array_equal(out_len.reshape(-1), exp_len)
    assert np.array_equal(s.counters(), models.histogram(cl.broker_id, exp, exp_len))


def _cand_tables(cl, g, base):
    tables = [(cl.broker_id, cl.rack_index)]
    for spec in g["tables"]:
        n, per, step = (tuple(spec) + (1,))[:3]
        tables.append(util.table(base + step * np.arange(n, dtype=np.int32), per))
    return tables


@pytest.mark.gpu
@pytest.mark.parametrize("case", CAND_CASES, ids=[c["id"] for c in CAND_CASES])
def test_dense_candidates_variant(native_lib, oracle, case):
    g = case["gen"]
    cl = _cluster(g, _seed(case["id"]))
    tables = _cand_tables(cl, g, 1000)
    s = kab.Solver(0)
    with mock.patch.dict(os.environ, case["env"]):
        sts = util.check_dense_equal(util.DenseProblem(cl.topic_hash, cl.cur), tables, oracle, solver=s)
    assert s.last_order_plan() == case["plan"]
    assert all(st[0] == 0 for st in sts), sts


@pytest.mark.gpu
@pytest.mark.parametrize("case", RAGGED_CAND_CASES, ids=[c["id"] for c in RAGGED_CAND_CASES])
def test_ragged_candidates_variant(native_lib, oracle, case):
    g = case["gen"]
    cl = kab.synth.make_ragged_cluster(T=80, N=40, R=5, max_partitions=64, seed=g["seed"], remove_frac=0.1)
    tables = _cand_tables(cl, g, 1)
    s = kab.Solver(0)
    with mock.patch.dict(os.environ, case["env"]):
        sts = util.check_equal(util.Problem.of(cl), tables, oracle, solver=s)
    assert s.last_order_plan() == case["plan"]
    assert all(st[0] == 0 for st in sts), sts


@pytest.mark.gpu
def test_one_context_across_variants(native_lib, oracle):
    """Counter hand-over between placements: shared-memory counters, then GCTR, then other shapes, on one Context."""
    s = kab.Solver(0)
    fctx = oracle.FastContext()
    ids = None
    total = None
    for i, case in enumerate(SEQUENCE):
        g = case["gen"]
        cl = kab.synth.make_cluster(T=g["T"], P=g["P"], RF=g["RF"], N=SEQUENCE_N, R=SEQUENCE_R, seed=0x5E0 + i, kind="mixed")
        if ids is None:
            ids = cl.broker_id
            total = np.zeros((len(ids), models.SLOTS), dtype=np.int64)
        assert np.array_equal(cl.broker_id, ids)
        exp, exp_len, est = oracle.fast_run_dense(fctx, cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index)
        assert est.code == 0
        with mock.patch.dict(os.environ, case["env"]):
            out, out_len, st = s.solve_cluster(cl, check=False)
        assert s.last_order_plan() == case["plan"], case["id"]
        assert st.code == 0, case["id"]
        assert np.array_equal(out.reshape(-1, cl.RF), exp), case["id"]
        assert np.array_equal(out_len.reshape(-1), exp_len), case["id"]
        total += models.histogram(ids, exp, exp_len)
        assert np.array_equal(s.counters(), total), case["id"]


@pytest.mark.gpu
def test_staged_entry_points_record_their_chains(native_lib, oracle):
    """ka_stage_dense_device starts a plan; ka_order_device, or the per-slot chains, add their launches to it."""
    import torch
    cl = kab.synth.make_cluster(T=30, P=100, RF=3, N=400, R=10, seed=77, kind="mixed")
    exp, exp_len, _ = oracle.fast_run_dense(oracle.FastContext(), cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index)
    d_hash, d_cur = torch.from_numpy(cl.topic_hash).cuda(), torch.from_numpy(cl.cur).cuda()
    for per_slot in (False, True):
        s = kab.Solver(0)
        s.set_brokers(cl.broker_id, cl.rack_index)
        d_out = torch.full((cl.T, cl.P, 3), -7, dtype=torch.int32, device="cuda")
        d_len = torch.full((cl.T, cl.P), -7, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        s.stage_dense_device(cl.T, d_hash.data_ptr(), cl.P, cl.RF, d_cur.data_ptr(), -1, 3)
        assert s.last_order_plan() == (0,) * 8
        if per_slot:
            s.order_slot_device(0)
            assert s.last_order_plan() == (3, 0, 128, 10, 0, SINGLE, 1, 0)
            s.order_slot_device(1)
            st = s.emit_device(d_len.data_ptr(), d_out.data_ptr())
        else:
            st = s.order_device(d_len.data_ptr(), d_out.data_ptr())
        assert st.code == 0
        assert s.last_order_plan() == (3, 0, 128, 10, 0, SINGLE, 2, 0)
        assert np.array_equal(d_out.cpu().numpy().reshape(-1, 3), exp) and np.array_equal(d_len.cpu().numpy().reshape(-1), exp_len)
    # a NULL plan pointer on a live context
    assert s._L.ka_ctx_last_order_plan(s._h, None) == _native.KA_ERR_BAD_ARG


def _lut_universe():
    """Broker ids for every lookup mode: 40 ids within a few hundred (shared-memory LUT), 10 within +-40 000 (global LUT),
    and ids near -2^31 and 2^31 (binary search); negative ids in all three."""
    rng = np.random.default_rng(31)
    small = rng.choice(np.arange(-300, 300), 40, replace=False)
    medium = rng.choice(np.arange(-40000, 40000), 10, replace=False)
    extreme = np.array([-2**31 + 1, -2**31 + 77, -2**31 + 5000, 2**31 - 1, 2**31 - 90, 2**31 - 4000])
    return np.unique(np.concatenate([small, medium, extreme])).astype(np.int32), np.sort(small).astype(np.int32)


def _lut_tables(universe, small):
    mid = universe[(universe > -40001) & (universe < 40001)]
    tables = [util.table(small, 5), util.table(mid), util.table(universe, 7), util.table(universe[universe < 0])]
    modes = []
    for ids, _ in tables:
        rng_ = int(ids[-1]) - int(ids[0]) + 1
        modes.append(0 if rng_ <= 32768 else (1 if rng_ <= 1 << 25 else 2))
    assert modes == [0, 1, 2, 2]
    return tables


@pytest.mark.gpu
def test_lookup_modes_in_one_batch(native_lib, oracle):
    """Candidate tables in the shared-memory LUT, global LUT and binary-search modes, alone and mixed in one batch, through
    the dense and ragged candidate solves and the candidate score (which looks the per-broker sums up by id)."""
    universe, small = _lut_universe()
    tables = _lut_tables(universe, small)
    # dense: make_cluster's brokers 1000 + i renamed to the universe's ids (ascending: rack order is kept)
    cl = kab.synth.make_cluster(T=30, P=30, RF=3, N=len(universe), R=6, seed=41, kind="mixed")
    cur = universe[cl.cur - 1000]
    prob = util.DenseProblem(cl.topic_hash, cur)
    for batch in ([tables[0]], [tables[1]], [tables[2]], tables):
        s = kab.Solver(0)
        sts = util.check_dense_equal(prob, batch, oracle, solver=s)
        assert all(st[0] == 0 for st in sts), sts
        if len(batch) == 4:
            assert s.last_order_plan() == LUT_DENSE_PLAN
    # ragged: brokers 1..N renamed
    rc = kab.synth.make_ragged_cluster(T=60, N=len(universe), R=6, max_partitions=40, seed=43)
    rprob = util.Problem(rc.topic_names, rc.topic_hash, rc.part_off, rc.part_id, rc.rep_off, universe[rc.cur - 1])
    for batch in ([tables[0]], [tables[1]], [tables[2]], tables):
        s = kab.Solver(0)
        sts, _ = util.check_scores(rprob, batch, oracle=oracle, solver=s)
        assert all(st[0] == 0 for st in sts), sts
        if len(batch) == 4:
            assert s.last_order_plan() == LUT_RAGGED_PLAN


@pytest.mark.gpu
def test_level_scratch_limit_is_a_clean_error(native_lib, oracle):
    """A ragged table beyond kernel A's level scratch (30 000 brokers) is refused with KA_ERR_LIMIT, b = N, by every ragged
    entry point, before anything runs."""
    cl = kab.synth.make_ragged_cluster(T=20, N=30000, R=10, max_partitions=32, seed=9)
    prob = util.Problem.of(cl)
    key = lambda st: (st.code, st.topic_index, st.partition, st.a, st.b)   # noqa: E731
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    _, _, st = s.solve_ragged(*prob.args(), prob.S, check=False)
    assert st.code == _native.KA_ERR_LIMIT and st.b == cl.N, key(st)
    assert s.last_order_plan() == (0,) * 8
    _, jst = s.solve_ragged_json(cl.topic_names, *prob.args(), check=False)
    assert key(jst) == key(st)
    _, _, csts = kab.Solver(0).solve_ragged_candidates([(cl.broker_id, cl.rack_index)] * 2, *prob.args(), out_stride=prob.S)
    assert [key(x) for x in csts] == [key(st)] * 2
    # the context still solves once the table fits
    small = [int(b) for b in cl.broker_id[:2000]]
    case = dict(topics=cl.topics(), brokers=small, racks={b: r for b, r in zip(small, cl.rack_name) if r is not None}, desired_rf=-1)
    assert util.run_gpu_case(kab, case, solver=s) == util.run_oracle_case(oracle, case)
