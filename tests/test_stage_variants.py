"""Every instantiation of the sticky/spread kernel (ka_sticky_spread_kernel, kernel A) against the oracle.

launch_stage_plan / launch_stage pick one instantiation per call from the solve's plan: the load width (1 or 2 bytes per
broker), LEVELS (the conflict-level pass, on when a topic may hold a broker twice or the input is ragged), SM (the row bound:
3, or 8 for rows of 4..8) and CAND (a batched candidate solve, rows <= 3 only). Inside the kernel, behaviour also changes with
the id lookup mode of the broker table, the staging path of the current lists, the record kind and the warps per CTA. Each
case below names the plan it must reach, checked through ka_ctx_last_stage_plan, so that a case cannot drift to another
variant when a heuristic changes; then its rows, list lengths and full status must equal the oracle's and, for single
solves, the Context counters must equal the per-position histogram of the oracle's rows.

Stage plan tuples: (load bytes, levels, SM, candidates K, warps per CTA, grid.x, lookup-mode mask, kernel A launches).
Lookup-mode mask: 1 shared-memory id LUT, 2 global LUT, 4 binary search. grid.x = PERSIST: the grid is capped by occupancy,
so that the topics outnumber grid.x x warps and the persistent topic loop runs (asserted as grid.x x warps < T); grid.x =
AUTO: one CTA per `warps` topics, ceil(T / warps). Warps per CTA = None: make_plan's count for the case's layout, computed by
models.stage_warps (the budget edges and deep-level cases pin it at 1, the small cases at 16).
"""
import ctypes
import os
import re

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from tests import models, util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERSIST = None
AUTO = -1
INT_MIN = -2**31


# ---- make_plan's kernel A arithmetic (kassign.cu, restated by models.stage_warps): the budget edges below are computed with it

def _lut_mode(ids):
    rng_ = int(ids[-1]) - int(ids[0]) + 1 if len(ids) else 0
    return 0 if rng_ <= 32768 else (1 if rng_ <= 1 << 25 else 2)


def _largest_p(N, S, rf, blob):
    """The largest P of a dense single solve (rf = S) that kernel A's layout holds for a table of N brokers."""
    def fits(P):
        cap = -(-P * rf // N)
        return models.stage_warps(N, blob, P, S, cap, cap > 1) > 0 and not (cap > 1 and P > 32767)
    lo, hi = 1, 32767
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid - 1)
    return lo


def _dense_cap(P, rf, n):
    """dense_capmax: the capacity of a table of n brokers, counted only when it can serve the target RF."""
    return -(-P * rf // n) if 0 < n and 0 <= rf <= n else 0


def _ragged_cap(part_off, rep_off, S, n):
    """ragged_capmax (desired_rf = -1): over the topics whose RF (first list's length) the table can serve."""
    cap = 0
    for t in range(len(part_off) - 1):
        a, b = int(part_off[t]), int(part_off[t + 1])
        if b > a:
            rf = int(rep_off[a + 1] - rep_off[a])
            if 0 < rf <= min(S, n):
                cap = max(cap, -(-(b - a) * rf // n))
    return cap


def _dense_warps(tables, P, rf, S):
    """make_plan's warps for a dense call over `tables` (its layout follows the largest table and blob)."""
    cap = max(_dense_cap(P, rf, len(t[0])) for t in tables)
    return models.stage_warps(max(len(t[0]) for t in tables), max(models.blob_bytes(t[0]) for t in tables), P, S, cap, cap > 1)


def _ragged_warps(tables, part_off, rep_off, S):
    cap = max(_ragged_cap(part_off, rep_off, S, len(t[0])) for t in tables)
    Pmax = int(np.diff(part_off).max())
    return models.stage_warps(max(len(t[0]) for t in tables), max(models.blob_bytes(t[0]) for t in tables), Pmax, S, cap, True)


# ---- broker tables and current lists ---------------------------------------------------------------------------------------

def _ext(ids, racks, mode):
    """The table (ids, racks) in lookup mode `mode`: one extra empty broker, in a rack of its own, far enough above the others
    to widen the id range past the shared-memory LUT (mode 1: global LUT) or the global LUT (mode 2: binary search)."""
    ids = np.asarray(ids, dtype=np.int32)
    racks = np.asarray(racks, dtype=np.int32)
    if mode == 0:
        return ids, racks
    far = int(ids[-1]) + 40000 if mode == 1 else 2**31 - 100
    out = np.append(ids, np.int32(far)).astype(np.int32), np.append(racks, racks.max() + 1).astype(np.int32)
    assert _lut_mode(out[0]) == mode
    return out


def _respace(ids, cur, mode):
    """The same brokers under new ids spaced so that the table is in lookup mode `mode` (1: global LUT, 2: binary search);
    cur follows. Capacities and racks are unchanged."""
    ids = np.asarray(ids, dtype=np.int64)
    if mode == 0:
        return ids.astype(np.int32), cur
    n = max(len(ids) - 1, 1)
    base, step = (1000, 40000 // n + 1) if mode == 1 else (-2**30, (1 << 26) // n + 1)
    new = base + step * np.arange(len(ids), dtype=np.int64)
    out = new[np.searchsorted(ids, cur)].astype(np.int32)
    assert np.array_equal(ids[np.searchsorted(ids, cur)], cur) and _lut_mode(new) == mode
    return new.astype(np.int32), out


def _dirty(cur, ids, seed):
    """cur with duplicate ids inside some lists (slot 1 := slot 0) and dead ids in others: below the table, and inside its id
    range but not a broker."""
    cur = cur.copy()
    flat = cur.reshape(-1, cur.shape[-1])
    rng = np.random.default_rng(seed)
    idset = set(int(x) for x in ids)
    inside = next(x for x in range(int(ids[0]) + 1, int(ids[-1])) if x not in idset) if len(ids) < int(ids[-1]) - int(ids[0]) + 1 \
        else int(ids[0]) - 1
    rows = rng.permutation(len(flat))
    n = len(flat) // 8
    flat[rows[:n], 1 % flat.shape[1]] = flat[rows[:n], 0]
    flat[rows[n:2 * n], -1] = int(ids[0]) - 5
    flat[rows[2 * n:3 * n], 0] = inside
    return cur


def _seed(cid):
    return 0x57A6 + sum(ord(ch) * (i + 1) for i, ch in enumerate(cid))


def _case(cid, plan, **gen):
    return dict(id=cid, plan=plan, gen=gen)


# ---- single dense solves: make_cluster(T, P, RF, N, R) in lookup mode `lut`; path: host (ka_solve_dense), device
# (ka_solve_dense_device), unaligned (the same with d_cur one int32 past a 16-byte boundary) --------------------------------
_DISPATCH = [
    # (id, (load, levels, SM), gen): capacity 1 / 2 / 256 with rows <= 3 and rows of 4..8
    ("u8-flat-sm3", (1, 0, 3), dict(T=40, P=24, RF=3, N=200, R=10)),
    ("u8-lv-sm3", (1, 1, 3), dict(T=40, P=60, RF=3, N=100, R=10)),
    ("u16-lv-sm3", (2, 1, 3), dict(T=6, P=600, RF=3, N=6, R=6, kind="structured")),
    ("u8-flat-sm8", (1, 0, 8), dict(T=20, P=24, RF=4, N=400, R=8)),
    ("u8-lv-sm8", (1, 1, 8), dict(T=20, P=40, RF=6, N=60, R=6)),
    ("u16-lv-sm8", (2, 1, 8), dict(T=4, P=600, RF=4, N=8, R=8, kind="structured")),
]

SINGLE_CASES = [
    _case("%s-lut%d" % (cid, lut), kind + (0, None, AUTO, 1 << lut, 1), lut=lut, **g) for cid, kind, g in _DISPATCH for lut in (0, 1, 2)
] + [
    # capacity 255 / 256: the u8 / u16 switch
    _case("cap255", (1, 1, 3, 0, None, AUTO, 1, 1), T=6, P=510, RF=3, N=6, R=3),
    _case("cap256", (2, 1, 3, 0, None, AUTO, 1, 1), T=6, P=511, RF=3, N=6, R=3),
    # staging: RF == S with P * RF % 4 != 0 (scalar), out_stride > RF, desired_rf growing and shrinking
    _case("scalar-p25", (1, 0, 3, 0, None, AUTO, 1, 1), T=30, P=25, RF=3, N=100, R=10),
    _case("scalar-lv-p25", (1, 1, 3, 0, None, AUTO, 2, 1), T=30, P=25, RF=3, N=20, R=10, lut=1),
    _case("stride3-rf2", (1, 0, 3, 0, None, AUTO, 1, 1), T=30, P=24, RF=2, N=50, R=10, out_stride=3),
    _case("stride8-rf3", (1, 1, 8, 0, None, AUTO, 1, 1), T=30, P=24, RF=3, N=40, R=10, out_stride=8),
    _case("grow-2-3", (1, 1, 3, 0, None, AUTO, 1, 1), T=30, P=24, RF=2, N=40, R=10, desired_rf=3),
    _case("shrink-3-2", (1, 1, 3, 0, None, AUTO, 1, 1), T=30, P=24, RF=3, N=40, R=10, desired_rf=2),
    _case("grow-3-6", (1, 1, 8, 0, None, AUTO, 1, 1), T=30, P=24, RF=3, N=60, R=6, desired_rf=6),
    _case("shrink-6-4", (1, 1, 8, 0, None, AUTO, 4, 1), T=30, P=24, RF=6, N=60, R=10, desired_rf=4, lut=2),
    # duplicate and dead ids in the current lists
    _case("dirty-sm3", (1, 1, 3, 0, None, AUTO, 2, 1), T=40, P=32, RF=3, N=60, R=10, lut=1, dirty=True),
    _case("dirty-sm8", (1, 1, 8, 0, None, AUTO, 4, 1), T=40, P=32, RF=4, N=60, R=8, lut=2, dirty=True),
    _case("dirty-flat", (1, 0, 3, 0, None, AUTO, 1, 1), T=40, P=32, RF=3, N=200, R=10, dirty=True),
    # topic sizes around the 32-lane window
    *[_case("p%d" % P, (1, int(-(-P * 3 // 8) > 1), 3, 0, None, AUTO, 1, 1), T=9, P=P, RF=3, N=8, R=8, kind="structured")
      for P in (1, 31, 32, 33, 64, 65, 96, 128)],
    # a middle warp count
    _case("warps-mid", (1, 1, 3, 0, None, AUTO, 1, 1), T=40, P=2000, RF=3, N=1000, R=1000, kind="structured"),
    # many more topics than grid.x x warps: the persistent topic loop
    _case("persist-flat", (1, 0, 3, 0, None, PERSIST, 1, 1), T=20000, P=8, RF=3, N=100, R=10),
    _case("persist-lv", (1, 1, 3, 0, None, PERSIST, 1, 1), T=20000, P=8, RF=3, N=12, R=12, kind="structured"),
    # device pointers: aligned source (int4 loads), and one int32 past a 16-byte boundary (scalar loads)
    _case("device-aligned", (1, 0, 3, 0, None, AUTO, 1, 1), T=30, P=24, RF=3, N=100, R=10, path="device"),
    _case("device-unaligned", (1, 0, 3, 0, None, AUTO, 1, 1), T=30, P=24, RF=3, N=100, R=10, path="unaligned"),
    _case("device-unaligned-lv", (1, 1, 3, 0, None, AUTO, 2, 1), T=30, P=24, RF=3, N=20, R=10, lut=1, path="unaligned"),
]

# ---- deep levels: N == RF == S, every partition shares every broker, so a topic of P partitions has P levels; P is the
# largest the layout holds (one warp per CTA) -----------------------------------------------------------------------------
DEEP_S = (1, 2, 3, 4, 6)

# ---- budget edges: (N, RF, R, lookup mode); the largest P solves with one warp, P + 1 is KA_ERR_LIMIT (a = P + 1, b = N) ---
EDGES = [(64, 3, 64, 0), (64, 4, 64, 2), (60000, 3, 10, 1)]

# ---- ragged solves (ka_solve): gen = make_ragged_cluster arguments, or dense= make_cluster arguments in the ragged layout -----
RAGGED_CASES = [
    _case("r-lut0", (1, 1, 3, 0, None, AUTO, 1, 1), rc=dict(T=80, N=40, R=5, max_partitions=64)),
    _case("r-lut1", (1, 1, 3, 0, None, AUTO, 2, 1), rc=dict(T=80, N=40, R=5, max_partitions=64), lut=1),
    _case("r-lut2", (1, 1, 3, 0, None, AUTO, 4, 1), rc=dict(T=80, N=40, R=5, max_partitions=64), lut=2),
    _case("r-sm8", (1, 1, 8, 0, None, AUTO, 1, 1), rc=dict(T=80, N=60, R=60, max_partitions=64, rf_weights=(1, 1, 2, 2, 2, 2))),
    _case("r-sm8-lut2", (1, 1, 8, 0, None, AUTO, 4, 1), rc=dict(T=80, N=60, R=60, max_partitions=64, rf_weights=(1, 1, 2, 2, 2, 2)),
          lut=2),
    _case("r-cap1", (1, 1, 3, 0, None, AUTO, 1, 1), dense=dict(T=20, P=24, RF=3, N=200, R=10)),
    _case("r-cap2", (1, 1, 3, 0, None, AUTO, 1, 1), dense=dict(T=20, P=60, RF=3, N=100, R=10)),
    _case("r-cap255", (1, 1, 3, 0, None, AUTO, 1, 1), dense=dict(T=3, P=510, RF=3, N=6, R=3)),
    _case("r-cap256", (2, 1, 3, 0, None, AUTO, 1, 1), dense=dict(T=3, P=511, RF=3, N=6, R=3)),
    _case("r-cap256-sm8", (2, 1, 8, 0, None, AUTO, 2, 1), dense=dict(T=3, P=600, RF=4, N=8, R=8, kind="structured"), lut=1),
    _case("r-dirty", (1, 1, 3, 0, None, AUTO, 2, 1), dense=dict(T=40, P=32, RF=3, N=60, R=10), lut=1, dirty=True),
]

# ---- batched dense candidates (ka_solve_dense_candidates_device): the cluster's table in every lookup mode (mask 7). The
# extra empty broker of the other modes lowers a capacity-255 problem's capacity, which may leave a partition unassignable
# there (own_only: only the cluster's own table must solve; every candidate still equals its sequential solve) ---------------
CAND_CASES = [
    _case("c-u8-flat", (1, 0, 3, 3, None, AUTO, 7, 1), T=30, P=24, RF=3, N=200, R=10),
    _case("c-cap2", (1, 1, 3, 3, None, AUTO, 7, 1), T=30, P=60, RF=3, N=100, R=10),
    _case("c-u8-lv", (1, 1, 3, 3, None, AUTO, 7, 1), T=30, P=40, RF=3, N=28, R=4),
    _case("c-cap255", (1, 1, 3, 3, None, AUTO, 7, 1), T=4, P=510, RF=3, N=6, R=6, kind="structured", own_only=True),
    _case("c-cap256", (2, 1, 3, 3, None, AUTO, 7, 1), T=4, P=511, RF=3, N=6, R=6, kind="structured", own_only=True),
    _case("c-stride3-rf2", (1, 1, 3, 3, None, AUTO, 7, 1), T=30, P=24, RF=2, N=20, R=10, out_stride=3),
    _case("c-dirty", (1, 1, 3, 3, None, AUTO, 7, 1), T=40, P=32, RF=3, N=60, R=10, dirty=True),
]

# ---- batched ragged candidates (ka_solve_candidates) ---------------------------------------------------------------------------
RCAND_CASES = [
    _case("rc-lv", (1, 1, 3, 3, None, AUTO, 7, 1), rc=dict(T=80, N=40, R=40, max_partitions=64)),
    _case("rc-cap1", (1, 1, 3, 3, None, AUTO, 7, 1), dense=dict(T=20, P=24, RF=3, N=200, R=10)),
    _case("rc-cap255", (1, 1, 3, 3, None, AUTO, 7, 1), dense=dict(T=3, P=510, RF=3, N=6, R=6, kind="structured"), own_only=True),
    _case("rc-cap256", (2, 1, 3, 3, None, AUTO, 7, 1), dense=dict(T=3, P=511, RF=3, N=6, R=6, kind="structured"), own_only=True),
]

# K = 128 candidates over 3 000 topics: grid.x drops to a CTA or two per candidate, so every warp loops over many topics
K128_PLAN = (1, 0, 3, 128, 16, PERSIST, 7, 1)

# the regression cases of the candidate capacity bound
AB_PLAN = (1, 0, 3, 2, 1, 4, 3, 1)
AB20K_PLAN = (1, 0, 3, 2, 6, 1, 3, 1)
P33000_PLAN = (1, 0, 3, 0, 1, 1, 1, 1)

ALL_PLANS = [c["plan"] for c in SINGLE_CASES + RAGGED_CASES + CAND_CASES + RCAND_CASES] + [K128_PLAN, AB_PLAN, AB20K_PLAN,
                                                                                               P33000_PLAN]


# ---- CPU ------------------------------------------------------------------------------------------------------------------

def _dispatch_from_source():
    """Reachable (load bytes, levels, SM, cand) instantiations of kernel A, read from kassign.cu: the launch_stage<...> calls of
    launch_stage_plan, the SM values of launch_stage, and the out_stride limit of the batched entry points."""
    src = open(os.path.join(ROOT, "kafka_assigner_b200", "csrc", "kassign.cu")).read()
    body = re.search(r"int launch_stage_plan\(.*?\n}\n", src, flags=re.S).group(0)
    kinds = re.findall(r"launch_stage<(\w+), (true|false), CAND>", body)
    assert kinds, "launch_stage_plan moved: update this test"
    ls = re.search(r"cudaError_t launch_stage\(.*?\n}\n", src, flags=re.S).group(0)
    sms = sorted(set(int(x) for x in re.findall(r"launch_stage_t<LoadT, LEVELS, (\d+), CAND>", ls)))
    assert sms == [3, 8], sms
    assert "p.S <= 3 ? launch_stage_t<LoadT, LEVELS, 3, CAND>" in ls
    # every batched entry point starts with the shared prologue, which refuses rows wider than 3: CAND only ever runs SM 3
    prologue = re.search(r"int batch_args\(.*?\n}\n", src, flags=re.S)
    assert prologue, "batch_args moved: update this test"
    assert "if (K > KA_MAX_CANDIDATES || out_stride > 3) return fail_members(st, K, KA_ERR_LIMIT);" in prologue.group(0)
    for entry in ("ka_solve_dense_candidates_device", "ka_solve_candidates", "ka_score_candidates", "ka_solve_clusters"):
        fn = re.search(r"int32_t %s\(.*?\n}\n" % entry, src, flags=re.S)
        assert fn, "%s moved: update this test" % entry
        assert re.search(r"int rc = batch_args\(c, K, out_stride, st\);\s*if \(rc != KA_OK\) return rc;", fn.group(0)), entry
    nbytes = {"uint8_t": 1, "uint16_t": 2, "uint32_t": 4}
    out = set()
    for load, lv in kinds:
        for sm in sms:
            for cand in ((0, 1) if sm == 3 else (0,)):
                out.add((nbytes[load], int(lv == "true"), sm, cand))
    return out


def test_case_table_names_every_dispatch():
    reachable = _dispatch_from_source()
    # u8 without levels (capacity <= 1), u8 / u16 with levels; x SM 3 / 8 single, SM 3 batched
    assert len(reachable) == 9, sorted(reachable)
    named = {(p[0], p[1], p[2], int(p[3] > 0)) for p in ALL_PLANS}
    assert reachable - named == set(), "dispatches without a case: %s" % sorted(reachable - named)
    assert named <= reachable, "cases naming a dispatch launch_stage_plan cannot make: %s" % sorted(named - reachable)
    # every single dispatch in every lookup mode; every batched dispatch with all three modes in one call
    single = {(p[0], p[1], p[2], p[6]) for p in ALL_PLANS if p[3] == 0}
    for load, lv, sm, cand in reachable:
        if cand:
            assert any(p[:3] == (load, lv, sm) and p[3] > 0 and p[6] == 7 for p in ALL_PLANS), (load, lv, sm)
        else:
            assert all((load, lv, sm, 1 << m) in single for m in range(3)), (load, lv, sm)
    ids = [c["id"] for c in SINGLE_CASES + RAGGED_CASES + CAND_CASES + RCAND_CASES]
    assert len(ids) == len(set(ids))


def test_named_dispatch_follows_make_plan():
    """The load width, levels and SM each dense single case names are what make_plan gives its layout, and the warp counts
    span 16 down to a middle value (the budget-edge and deep-level cases pin 1)."""
    warps = {}
    for c in SINGLE_CASES:
        g = c["gen"]
        cl = kab.synth.make_cluster(T=1, P=1, RF=g["RF"], N=g["N"], R=g["R"], seed=1)
        ids = _respace(cl.broker_id, cl.broker_id, g.get("lut", 0))[0]
        rf = g.get("desired_rf", -1)
        rf = rf if rf >= 0 else g["RF"]
        S = g.get("out_stride") or max(g["RF"], rf)
        cap = _dense_cap(g["P"], rf, len(ids))
        assert (1 if cap <= 255 else 2, int(cap > 1), 3 if S <= 3 else 8) == c["plan"][:3], c["id"]
        assert _lut_mode(ids) == c["plan"][6].bit_length() - 1, c["id"]
        warps[c["id"]] = _dense_warps([(ids,)], g["P"], rf, S)
    assert warps["u8-flat-sm3-lut0"] == 16 and 1 < warps["warps-mid"] < 16, warps
    assert all(w > 0 for w in warps.values()), warps


def test_regression_plans_follow_make_plan():
    """The plans the capacity-bound regression cases name: table B (fewer brokers than the RF) adds nothing to the bound."""
    A52, A20, B = (1000 + np.arange(52000),), (1000 + 2 * np.arange(20000),), (1000 + np.arange(2),)
    assert _dense_cap(1000, 3, 2) == 0 and _dense_cap(1000, 3, 52000) == 1
    assert _dense_warps([A52, B], 1000, 3, 3) == AB_PLAN[4]
    assert _dense_warps([A20, B], 1000, 3, 3) == AB20K_PLAN[4]
    assert _dense_warps([(np.array([7]),)], 33000, 2, 2) == P33000_PLAN[4]
    # the bound of the parent: B's 1 500 turns levels on, and neither layout fits
    assert models.stage_warps(52000, models.blob_bytes(A52[0]), 1000, 3, 1500, True) == 0
    assert models.stage_warps(20000, models.blob_bytes(A20[0]), 1000, 3, 1500, True) == 0
    # the ragged layout of A20 (levels, capacity 1) fits
    assert models.stage_warps(20000, models.blob_bytes(A20[0]), 1000, 3, 1, True) > 0


def test_last_stage_plan_null_arguments(native_lib):
    plan = np.zeros(8, dtype=np.int32)
    assert native_lib.ka_ctx_last_stage_plan(None, plan.ctypes.data_as(ctypes.c_void_p)) == _native.KA_ERR_BAD_ARG
    assert native_lib.ka_ctx_last_stage_plan(None, None) == _native.KA_ERR_BAD_ARG
    assert not plan.any()


# ---- Integer.MIN_VALUE topic hashes ------------------------------------------------------------------------------------------

def _py_hash(s):
    h = 0
    for ch in s:
        h = (31 * h + ord(ch)) & 0xFFFFFFFF
    return h - (1 << 32) if h & 0x80000000 else h


def _min_names(n, seed=0x3117):
    """Topic names whose String.hashCode is Integer.MIN_VALUE: "polygenelubricants", then seeded random prefixes completed by
    a 7-character suffix solved in base 31 (characters '0'..'N': hash(prefix + t) = hash(prefix) * 31^7 + hash(t) mod 2^32,
    and 31^7 > 2^32, so every residue has a suffix)."""
    rng = np.random.default_rng(seed)
    names = ["polygenelubricants"]
    while len(names) < n:
        prefix = "mv.%d." % int(rng.integers(0, 10**9))
        hp = _py_hash(prefix) & 0xFFFFFFFF
        y = (2**31 - hp * 31**7 - 48 * (31**7 - 1) // 30) % 2**32
        digits = []
        for _ in range(7):
            digits.append(y % 31)
            y //= 31
        names.append(prefix + "".join(chr(48 + d) for d in reversed(digits)))
    assert all(_py_hash(x) == INT_MIN for x in names)
    return names


MIN_N_DIVIDES = (2, 4, 16, 1024)
MIN_N_OTHER = (3, 6, 12)
MIN_RF = (1, 2, 3, 4, 6, 7, 8)
MIN_COMBOS = [(N, rf) for N in MIN_N_DIVIDES + MIN_N_OTHER for rf in MIN_RF if rf <= N]


def _min_cluster(N, rf, name, P=10, seed=0):
    """Three topics of P partitions and RF rf over N brokers, each in a rack of its own; the middle one is named `name`
    (hashCode == MIN_VALUE)."""
    cl = kab.synth.make_cluster(T=3, P=P, RF=rf, N=N, R=N, seed=0x4D1 + 7 * N + rf + seed, kind="mixed")
    cl.topic_names = [cl.topic_names[0], name, cl.topic_names[2]]
    cl.topic_hash = np.array([_py_hash(x) for x in cl.topic_names], dtype=np.int32)
    return cl


def _expected_min_status(N, rf):
    """(code, topic, partition, a, b) the reference throws for the MIN_VALUE topic (topic 1), or None when it solves."""
    if 2**31 % N:
        return (5, 1, -1, -(2**31 % N), N)                       # getNodeProcessingOrder of the orphan spread
    k = next((k for k in range(rf, 0, -1) if 2**31 % k), None)   # leader order: remaining-set sizes rf, rf - 1, ...
    return None if k is None else (5, 1, -1, -(2**31 % k), k)


def _oracle_ragged(oracle, names, part_off, part_id, rep_off, cur, ids, rack_names, desired_rf, S):
    ln, _, out, st = oracle.run(oracle.OracleContext(), names, part_off, part_id, rep_off, cur, ids, rack_names, desired_rf, S,
                                raise_on_error=False)
    return out, ln, (st.code, st.topic_index, st.partition, st.a, st.b)


def test_min_value_names(native_lib):
    names = _min_names(6)
    assert len(set(names)) == 6
    for n in names:
        assert kab.java_string_hash(n) == INT_MIN, n


def test_min_value_oracles_agree(oracle):
    """The fast oracle (hash passed in) and the structure-faithful oracle (hash of the name) agree on every MIN_VALUE case,
    and both give the status the reference's arithmetic predicts."""
    names = _min_names(4)
    for i, (N, rf) in enumerate(MIN_COMBOS):
        cl = _min_cluster(N, rf, names[i % len(names)])
        for S in sorted({rf, 3 if rf <= 3 else 8, 8}):
            f_out, f_len, fst = oracle.fast_run_dense(oracle.FastContext(), cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index,
                                                      -1, S)
            part_off, part_id, rep_off, cur = cl.ragged()
            o_out, o_len, ost = _oracle_ragged(oracle, cl.topic_names, part_off, part_id, rep_off, cur, cl.broker_id,
                                               cl.rack_name, -1, S)
            f = (fst.code, fst.topic_index, fst.partition, fst.a, fst.b)
            assert f == ost, (N, rf, S, f, ost)
            exp = _expected_min_status(N, rf)
            assert f == (exp or (0, -1, -1, 0, 0)), (N, rf, f)
            if exp is None:
                assert np.array_equal(f_out, o_out) and np.array_equal(f_len, o_len), (N, rf, S)
                # rotation 0: slot 0 scans the row in ascending id order
                assert np.all(f_len[cl.P:2 * cl.P] == rf)


# ---- GPU ------------------------------------------------------------------------------------------------------------------

def _check_plan(s, want, T, cid, warps=None):
    """The stage plan of s's last call is `want`; warps = make_plan's count where want names None."""
    got = s.last_stage_plan()
    want = list(want)
    if want[4] is None:
        want[4] = warps
    if want[5] is PERSIST:
        assert got[5] * got[4] < T, (cid, got)
        want[5] = got[5]
    elif want[5] == AUTO:
        want[5] = -(-T // want[4])
    assert got == tuple(want), (cid, got, tuple(want))


def _dense(g, seed):
    """(topic_hash, cur, table ids, table racks, desired_rf, S) of a dense case."""
    cl = kab.synth.make_cluster(T=g["T"], P=g["P"], RF=g["RF"], N=g["N"], R=g["R"], seed=seed, kind=g.get("kind", "mixed"))
    ids, cur = _respace(cl.broker_id, cl.cur, g.get("lut", 0))
    racks = cl.rack_index
    cur = _dirty(cur, ids, seed) if g.get("dirty") else cur
    desired = g.get("desired_rf", -1)
    S = g.get("out_stride") or max(g["RF"], desired, 1)
    return cl, cl.topic_hash, cur, ids, racks, desired, S


def _solve_dense(s, th, cur, desired, S, path):
    import torch
    T, P, RF = cur.shape
    if path == "host":
        out, ln, st = s.solve_dense(th, cur, desired, S, check=False)
        return out.reshape(-1, S), ln.reshape(-1), st
    d_hash = torch.from_numpy(np.ascontiguousarray(th, dtype=np.int32)).cuda()
    off = 1 if path == "unaligned" else 0
    buf = torch.zeros(cur.size + 4, dtype=torch.int32, device="cuda")
    buf[off:off + cur.size] = torch.from_numpy(np.ascontiguousarray(cur, dtype=np.int32).reshape(-1)).cuda()
    d_cur = buf[off:]
    assert (d_cur.data_ptr() % 16 == 0) == (off == 0)
    out = torch.full((T * P, S), -7, dtype=torch.int32, device="cuda")
    ln = torch.full((T * P,), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    st = s.solve_dense_device(T, d_hash.data_ptr(), P, RF, d_cur.data_ptr(), desired, S, ln.data_ptr(), out.data_ptr())
    return out.cpu().numpy(), ln.cpu().numpy(), st


def _check_single(oracle, s, th, cur, ids, racks, desired, S, path="host", cid=""):
    exp, exp_len, est = oracle.fast_run_dense(oracle.FastContext(), th, cur, ids, racks, desired, S)
    s.reset()   # a fresh Context: the counters must come from this solve alone
    s.set_brokers(ids, racks)
    out, ln, st = _solve_dense(s, th, cur, desired, S, path)
    assert util.fields(st) == util.fields(est), (cid, util.fields(st), util.fields(est))
    if est.code == 0:
        assert np.array_equal(out, exp), cid
        assert np.array_equal(ln, exp_len), cid
        assert np.array_equal(s.counters(), models.histogram(ids, exp, exp_len)), cid
    return util.fields(st)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SINGLE_CASES, ids=[c["id"] for c in SINGLE_CASES])
def test_single_solve_stage_variant(native_lib, oracle, case):
    g = case["gen"]
    cl, th, cur, ids, racks, desired, S = _dense(g, _seed(case["id"]))
    s = kab.Solver(0)
    st = _check_single(oracle, s, th, cur, ids, racks, desired, S, g.get("path", "host"), case["id"])
    assert st[0] == 0, st
    rf = desired if desired >= 0 else g["RF"]
    _check_plan(s, case["plan"], g["T"], case["id"], _dense_warps([(ids,)], g["P"], rf, S))


def _deep_p(S):
    return _largest_p(S, S, S, models.blob_bytes(np.arange(S)))


@pytest.mark.gpu
@pytest.mark.parametrize("S", DEEP_S)
def test_deep_levels(native_lib, oracle, S):
    """N == RF == S: every partition of a topic shares every broker, so each is a level of its own (P levels per topic, the
    16-bit level arrays and the 15-bit cursor near their ends), at the largest P the layout holds."""
    P = _deep_p(S)
    assert P > 8000
    cl = kab.synth.make_cluster(T=2, P=P, RF=S, N=S, R=S, seed=0xDEE + S, kind="mixed")
    s = kab.Solver(0)
    assert _check_single(oracle, s, cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index, -1, S, cid="deep%d" % S)[0] == 0
    _check_plan(s, (1 if P <= 255 else 2, 1, 3 if S <= 3 else 8, 0, 1, 2, 1, 1), 2, "deep%d" % S)


@pytest.mark.gpu
@pytest.mark.parametrize("edge", EDGES, ids=["N%d-RF%d-lut%d" % (e[0], e[1], e[3]) for e in EDGES])
def test_budget_edge(native_lib, oracle, edge):
    """The largest P kernel A's layout holds solves with one warp per CTA; one partition more is KA_ERR_LIMIT (a = P, b = N)
    before anything runs, with an all-zero stage plan."""
    N, RF, R, lut = edge
    cl0 = kab.synth.make_cluster(T=1, P=1, RF=RF, N=N, R=R, seed=1)
    ids, racks = _respace(cl0.broker_id, cl0.broker_id, lut)[0], cl0.rack_index
    P = _largest_p(len(ids), RF, RF, models.blob_bytes(ids))
    cap = -(-P * RF // len(ids))
    s = kab.Solver(0)
    for p, ok in ((P, True), (P + 1, False)):
        cl = kab.synth.make_cluster(T=2, P=p, RF=RF, N=N, R=R, seed=0xED6 + p, kind="structured")
        cur = _respace(cl.broker_id, cl.cur, lut)[1]
        st = _check_single(oracle, s, cl.topic_hash, cur, ids, racks, -1, RF, cid="edge P=%d" % p) if ok else \
            util.fields(s.solve_dense(cl.topic_hash, cur, -1, RF, check=False)[2])
        if ok:
            assert st[0] == 0, st
            _check_plan(s, (1 if cap <= 255 else 2, int(cap > 1), 3 if RF <= 3 else 8, 0, 1, 2, 1 << lut, 1), 2, "edge")
        else:
            assert st == (_native.KA_ERR_LIMIT, -1, -1, P + 1, len(ids)), st
            assert s.last_stage_plan() == (0,) * 8
            assert s.last_order_plan() == (0,) * 8


def _ragged_problem(case):
    """(names, hash, part_off, part_id, rep_off, cur, table ids, racks, rack names, S) of a ragged case."""
    g = case["gen"]
    seed = _seed(case["id"])
    if "rc" in g:
        cl = kab.synth.make_ragged_cluster(seed=seed, remove_frac=0.1, **g["rc"])
        names, th, part_off, part_id, rep_off, cur = cl.topic_names, cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur
        ids0, racks0 = cl.broker_id, cl.rack_index
    else:
        cl = kab.synth.make_cluster(seed=seed, **dict(dict(kind="mixed"), **g["dense"]))
        names, th = cl.topic_names, cl.topic_hash
        part_off, part_id, rep_off, cur = cl.ragged()
        ids0, racks0 = cl.broker_id, cl.rack_index
    if "rc" in g:   # its lists hold ids of removed brokers: widen the range with an extra empty broker instead
        ids, racks = _ext(ids0, racks0, g.get("lut", 0))
    else:
        (ids, cur), racks = _respace(ids0, cur, g.get("lut", 0)), racks0
    if g.get("dirty"):
        cur = _dirty(cur.reshape(-1, 1) if cur.ndim == 1 else cur, ids, seed).reshape(-1)
        # one duplicate inside a list: slot 1 := slot 0 of every eighth row of three or more
        sizes = np.diff(rep_off)
        rows = np.nonzero(sizes >= 3)[0][::8]
        cur = cur.copy()
        cur[rep_off[rows] + 1] = cur[rep_off[rows]]
    sizes = np.diff(rep_off)
    S = max(int(sizes.max()) if len(sizes) else 0, 1)
    return names, th, part_off, part_id, rep_off, cur, ids, racks, ["k%d" % r for r in racks], S


@pytest.mark.gpu
@pytest.mark.parametrize("case", RAGGED_CASES, ids=[c["id"] for c in RAGGED_CASES])
def test_ragged_stage_variant(native_lib, oracle, case):
    names, th, part_off, part_id, rep_off, cur, ids, racks, rnames, S = _ragged_problem(case)
    exp, exp_len, est = _oracle_ragged(oracle, names, part_off, part_id, rep_off, cur, ids, rnames, -1, S)
    s = kab.Solver(0)
    s.set_brokers(ids, racks)
    out, ln, st = s.solve_ragged(th, part_off, part_id, rep_off, cur, -1, S, check=False)
    assert util.fields(st) == est == (0, -1, -1, 0, 0), (util.fields(st), est)
    assert np.array_equal(out, exp) and np.array_equal(ln, exp_len)
    assert np.array_equal(s.counters(), models.histogram(ids, exp, exp_len))
    _check_plan(s, case["plan"], len(th), case["id"], _ragged_warps([(ids,)], part_off, rep_off, S))


def _lut_tables(ids, racks):
    return [_ext(ids, racks, m) for m in (0, 1, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CAND_CASES, ids=[c["id"] for c in CAND_CASES])
def test_dense_candidates_stage_variant(native_lib, oracle, case):
    g = case["gen"]
    cl, th, cur, ids, racks, desired, S = _dense(g, _seed(case["id"]))
    s = kab.Solver(0)
    tables = _lut_tables(ids, racks)
    sts = util.check_dense_equal(util.DenseProblem(th, cur, desired, S), tables, oracle, solver=s)
    assert all(st[0] == 0 for st in (sts[:1] if g.get("own_only") else sts)), sts
    rf = desired if desired >= 0 else g["RF"]
    _check_plan(s, case["plan"], g["T"], case["id"], _dense_warps(tables, g["P"], rf, S))


@pytest.mark.gpu
@pytest.mark.parametrize("case", RCAND_CASES, ids=[c["id"] for c in RCAND_CASES])
def test_ragged_candidates_stage_variant(native_lib, oracle, case):
    names, th, part_off, part_id, rep_off, cur, ids, racks, _, S = _ragged_problem(case)
    s = kab.Solver(0)
    prob = util.Problem(names, th, part_off, part_id, rep_off, cur, out_stride=S)
    tables = _lut_tables(ids, racks)
    sts = util.check_equal(prob, tables, oracle, solver=s)
    assert all(st[0] == 0 for st in (sts[:1] if case["gen"].get("own_only") else sts)), sts
    _check_plan(s, case["plan"], len(th), case["id"], _ragged_warps(tables, part_off, rep_off, S))


@pytest.mark.gpu
def test_candidates_k128_persistent_topics(native_lib, oracle):
    """K = 128 (the limit) over 3 000 topics: a CTA or two per candidate, each warp looping over many topics. Tables in all
    three lookup modes, some without the cluster's brokers, and one too small for the RF."""
    cl = kab.synth.make_cluster(T=3000, P=8, RF=3, N=60, R=6, seed=0x128, kind="mixed")
    rng = np.random.default_rng(128)
    tables = []
    for k in range(127):
        keep = np.sort(rng.choice(len(cl.broker_id), len(cl.broker_id) - k % 20, replace=False))
        tables.append(_ext(cl.broker_id[keep], cl.rack_index[keep], k % 3))
    tables.append(_ext(cl.broker_id[:2], cl.rack_index[:2], 0))
    s = kab.Solver(0)
    sts = util.check_dense_equal(util.DenseProblem(cl.topic_hash, cl.cur), tables, oracle, solver=s)
    assert all(st[0] == 0 for st in sts[:127]), sts
    assert sts[127] == (_native.KA_ERR_RF_GT_BROKERS, 0, -1, 3, 0)
    assert _dense_warps(tables, cl.P, 3, 3) == K128_PLAN[4]
    _check_plan(s, K128_PLAN, cl.T, "k128")


# ---- MIN_VALUE on the device ----------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_min_value_single_dense(native_lib, oracle):
    """The MIN_VALUE topic between two normal ones, hash passed directly: table sizes that divide 2^31 and ones that do not,
    rows of 1..8 (rows of <= 2 also under the record kinds of rows of 4 and 5..8)."""
    names = _min_names(4)
    s = kab.Solver(0)
    for i, (N, rf) in enumerate(MIN_COMBOS):
        cl = _min_cluster(N, rf, names[i % len(names)])
        for S in sorted({rf, 3 if rf <= 3 else 8, 4 if rf <= 4 else 8, 8}):
            st = _check_single(oracle, s, cl.topic_hash, cl.cur, cl.broker_id, cl.rack_index, -1, S, cid=(N, rf, S))
            assert st == (_expected_min_status(N, rf) or (0, -1, -1, 0, 0)), (N, rf, S, st)
            assert s.last_stage_plan()[2] == (3 if S <= 3 else 8)


@pytest.mark.gpu
def test_min_value_ragged(native_lib, oracle):
    """The same problems in the ragged layout (ka_solve), the hash taken from the name, against the structure-faithful oracle."""
    names = _min_names(4)
    s = kab.Solver(0)
    for i, (N, rf) in enumerate(MIN_COMBOS):
        cl = _min_cluster(N, rf, names[i % len(names)])
        part_off, part_id, rep_off, cur = cl.ragged()
        th = np.array([kab.java_string_hash(x) for x in cl.topic_names], dtype=np.int32)
        assert th[1] == INT_MIN
        exp, exp_len, est = _oracle_ragged(oracle, cl.topic_names, part_off, part_id, rep_off, cur, cl.broker_id, cl.rack_name,
                                           -1, rf)
        s.reset()
        s.set_brokers(cl.broker_id, cl.rack_index)
        out, ln, st = s.solve_ragged(th, part_off, part_id, rep_off, cur, -1, rf, check=False)
        assert util.fields(st) == est == (_expected_min_status(N, rf) or (0, -1, -1, 0, 0)), (N, rf, util.fields(st), est)
        if est[0] == 0:
            assert np.array_equal(out, exp) and np.array_equal(ln, exp_len), (N, rf)
            assert np.array_equal(s.counters(), models.histogram(cl.broker_id, exp, exp_len)), (N, rf)


@pytest.mark.gpu
def test_min_value_candidates(native_lib, oracle):
    """Batched: tables on which the MIN_VALUE topic solves (N divides 2^31, rows of 2), fails early (N does not) and fails late
    (rows of 3), in the dense and the ragged batch."""
    names = _min_names(3)
    for rf, sizes in ((2, (2, 4, 16, 1024, 3, 6, 12)), (3, (4, 16, 1024, 3, 6, 12, 2))):
        cl = _min_cluster(1024, rf, names[rf - 1], P=12)
        # every broker in a rack of its own: a table of n >= rf brokers never leaves a partition unassignable
        tables = [util.table(np.sort(np.random.default_rng(n).choice(cl.broker_id, n, replace=False))) for n in sizes]
        s = kab.Solver(0)
        sts = util.check_dense_equal(util.DenseProblem(cl.topic_hash, cl.cur), tables, oracle, solver=s)
        seen = set()
        for (ids, racks), st in zip(tables, sts):
            n = len(ids)
            _, _, est = oracle.fast_run_dense(oracle.FastContext(), cl.topic_hash, cl.cur, ids, racks)
            assert st == util.fields(est), (rf, n, st, util.fields(est))
            if st[0] in (0, _native.KA_ERR_HASH_INDEX):
                assert st == (_expected_min_status(n, rf) or (0, -1, -1, 0, 0)), (rf, n, st)
                seen.add("solve" if st[0] == 0 else ("early" if 2**31 % n else "late"))
        assert seen == ({"solve", "early"} if rf == 2 else {"early", "late"}), (rf, seen)
        assert s.last_stage_plan()[3] == len(tables)
        part_off, part_id, rep_off, cur = cl.ragged()
        prob = util.Problem(cl.topic_names, np.array([kab.java_string_hash(x) for x in cl.topic_names], dtype=np.int32), part_off,
                            part_id, rep_off, cur)
        assert util.check_equal(prob, tables, oracle) == sts


# ---- the dense capacity bound counts only tables that can serve the target RF ----------------------------------------------

def _ab_problem():
    cl = kab.synth.make_cluster(T=4, P=1000, RF=3, N=3000, R=10, seed=0xAB, kind="mixed")
    return cl


@pytest.mark.gpu
def test_small_table_does_not_change_the_dense_batch_plan(native_lib, oracle):
    """Table A (52 000 brokers, capacity 1) and table B (2 brokers, RF 3): B fails alone with KA_ERR_RF_GT_BROKERS, and A
    solves under A's own plan (no levels, 1-byte loads) instead of the level scratch B's bound would ask for."""
    cl = _ab_problem()
    A = util.table(1000 + np.arange(52000, dtype=np.int32), 500)
    B = util.table(cl.broker_id[:2], 1)
    s = kab.Solver(0)
    sts = util.check_dense_equal(util.DenseProblem(cl.topic_hash, cl.cur), [A, B], oracle, solver=s)
    assert sts == [(0, -1, -1, 0, 0), (_native.KA_ERR_RF_GT_BROKERS, 0, -1, 3, 0)], sts
    _check_plan(s, AB_PLAN, cl.T, "A+B")
    assert s.last_order_plan()[1] == 0


@pytest.mark.gpu
def test_dense_and_ragged_batches_agree_with_a_small_table(native_lib, oracle):
    """The same cluster and tables through the dense and the ragged candidate solves: identical statuses and rows. Table A
    has 20 000 brokers (global id LUT), which fits the ragged layout's level scratch but not levels with 2-byte loads."""
    cl = _ab_problem()
    A = util.table(1000 + 2 * np.arange(20000, dtype=np.int32), 500)
    B = util.table(cl.broker_id[:2], 1)
    s = kab.Solver(0)
    dprob = util.DenseProblem(cl.topic_hash, cl.cur)
    d_out, d_len, d_sts = dprob.batched([A, B], s)
    part_off, part_id, rep_off, cur = cl.ragged()
    rprob = util.Problem(cl.topic_names, cl.topic_hash, part_off, part_id, rep_off, cur)
    r_out, r_len, r_sts = rprob.batched([A, B])
    assert d_sts == r_sts == [(0, -1, -1, 0, 0), (_native.KA_ERR_RF_GT_BROKERS, 0, -1, 3, 0)], (d_sts, r_sts)
    assert np.array_equal(d_out[0].reshape(-1, 3), r_out[0]) and np.array_equal(d_len[0].reshape(-1), r_len[0])
    assert util.check_equal(rprob, [A, B], oracle) == r_sts
    assert util.check_dense_equal(dprob, [A, B], oracle) == d_sts
    _check_plan(s, AB20K_PLAN, cl.T, "A20k+B")


@pytest.mark.gpu
def test_rf_above_a_one_broker_table_is_the_reference_error(native_lib, oracle):
    """T = 1, P = 33 000, RF = 2 over one broker: the reference's "higher replication factor (2) than available brokers",
    not a level-layout limit (33 000 partitions exceed the 15-bit level cursors, but the table cannot serve RF 2 at all)."""
    cur = np.full((1, 33000, 2), 7, dtype=np.int32)
    ids, racks = np.array([7], dtype=np.int32), np.array([0], dtype=np.int32)
    th = np.array([kab.java_string_hash("big-topic")], dtype=np.int32)
    _, _, est = oracle.fast_run_dense(oracle.FastContext(), th, cur, ids, racks)
    s = kab.Solver(0)
    s.set_brokers(ids, racks)
    st = util.fields(s.solve_dense(th, cur, check=False)[2])
    assert st == (est.code, est.topic_index, est.partition, est.a, est.b) == (_native.KA_ERR_RF_GT_BROKERS, 0, -1, 2, 0), st
    _check_plan(s, P33000_PLAN, 1, "P33000")
