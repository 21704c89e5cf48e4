"""The leader-order chains at both sides of every shared-memory band edge, and from preloaded Context counters.

make_plan (kassign.cu) places the chain's counters next to its record ring in KA_ORDER_SMEM_BUDGET bytes of shared memory:
rows <= 3 keep (N + 1) int32 per slot chain (the dummy broker that pads short rows at index N), rows of 4 keep 4 N and rows of
5..8 keep 8 N. The ring shrinks from 2^10 (rows <= 3) or 2^9 records per stage down to 2^7 as N grows, and the counters move
to global memory (GCTR) beyond. At the top N of a band the counters and ring fill the budget to the byte, with the highest
broker's counter and the dummy in its last bytes; one broker more is the next band. order_plan below restates that half of
make_plan from the constants in the sources, and the CPU tests pin the edges it gives, so that a changed constant names its new
edges instead of leaving the GPU cases in the middle of a band.

Every GPU case runs once on each side of an edge, names the plan it must reach (ka_ctx_last_order_plan), and puts the top
broker (index N - 1) and the lowest one in every topic, with rows of 1 and 2 that pad with the dummy. Single solves start from
preloaded counters (ties and +-1 gaps between the top broker, the lowest broker and the rest), low, around 2^30 and up to
INT_MAX minus the run's rows; their rows, list lengths, status and every counter of every slot must equal the
structure-faithful oracle's. Level plans (every ragged entry point) cannot reach the bands of rows <= 3: kernel A's level
scratch refuses their tables first, and those pairs are checked for that documented KA_ERR_LIMIT.

The sentinel: the dummy's counter is INT_MAX, listed after every real broker of its row and never bumped, so that a real
counter at any value wins against it. The CPU test checks that with the slot-chain model and the oracle from counters
above 2^30 (where the former sentinel, 2^30 - 1, lost to the dummy).

Plan tuples: (rec_kind, levels, chain threads, ring_log2, gctr, loop shape, chain launches of the call, candidates K).
"""
import os
import random
import re

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from tests import models, util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kafka_assigner_b200", "csrc")
GENERAL, WARP1, SINGLE, FULL = 0, 1, 2, 3
LIMIT = _native.KA_ERR_LIMIT
INT_MAX = 2**31 - 1
SENTINEL_LOW = 0x3FFFFFFF - 2      # the lower end of the high counter range (the former dummy counter was 0x3FFFFFFF)


# ---- make_plan's order half, restated from the sources ----------------------------------------------------------------------

def _source_constants():
    cu = open(os.path.join(CSRC, "kassign.cu")).read()
    oh = open(os.path.join(CSRC, "kassign_order.cuh")).read()
    found = dict(
        budget=re.search(r"constexpr size_t KA_ORDER_SMEM_BUDGET = (\d+) \* 1024;", cu),
        stages=re.search(r"#define KA_RING_STAGES (\d+)", oh),
        lg=re.search(r"const int lg_max = pl\.rec_kind == 3 \? (\d+) : (\d+), lg_min = (\d+);", cu),
        max_nt=re.search(r"const int max_nt = pl\.rec_kind == 3 \? (\d+) : \(pl\.rec_kind == 4 \? (\d+) : (\d+)\);", cu),
        ring=re.search(r"return \(\(size_t\)KA_RING_STAGES << l\) \* pl\.rec_bytes \+ (\d+); \};", cu),
        dummy=re.search(r"if \(GCTR\) ctr8\[\(size_t\)N \* KA_MAX_SLOTS \+ KIND\] = (0x[0-9A-Fa-f]+); else ctr\[N\] = (0x[0-9A-Fa-f]+);", oh))
    missing = [k for k, v in found.items() if v is None]
    assert not missing, "make_plan or the chain kernel moved (%s): update this restatement" % missing
    lg_max3, lg_max, lg_min = (int(x) for x in found["lg"].groups())
    nt3, nt4, nt8 = (int(x) for x in found["max_nt"].groups())
    d0, d1 = (int(x, 16) for x in found["dummy"].groups())
    assert d0 == d1
    return dict(budget=int(found["budget"].group(1)) * 1024, stages=int(found["stages"].group(1)), ring_pad=int(found["ring"].group(1)),
                lg_max={3: lg_max3, 4: lg_max, 8: lg_max}, lg_min=lg_min, max_nt={3: nt3, 4: nt4, 8: nt8}, dummy=d0)


K = _source_constants()


def rec_kind(S):
    return 3 if S <= 3 else (4 if S == 4 else 8)


def _ctr_bytes(kind, N):
    return (max(N, 1) + 1) * 4 if kind == 3 else max(N, 1) * (8 if kind == 8 else 4) * 4


def _ring_bytes(kind, lg):
    return (K["stages"] << lg) * (16 if kind == 3 else 32) + K["ring_pad"]


def order_plan(N, S, Pmax, capmax, ragged):
    """make_plan's leader-order half: (rec_kind, ring_log2, gctr, chain threads) without the environment overrides."""
    kind = rec_kind(S)
    levels = capmax > 1 or ragged
    lg = K["lg_max"][kind]
    while lg > K["lg_min"] and _ctr_bytes(kind, N) + _ring_bytes(kind, lg) > K["budget"]:
        lg -= 1
    gctr = _ctr_bytes(kind, N) + _ring_bytes(kind, lg) > K["budget"]
    if gctr:
        lg = K["lg_max"][kind]
    max_nt = K["max_nt"][kind]
    width = min(Pmax, max(1, N // max(S, 1) // 2)) if levels else Pmax
    cuts = -(-max(width, 1) // max_nt)
    width = -(-max(width, 1) // cuts)
    nt = min(max_nt, -(-width // 32) * 32)
    nt = max(32, min(max_nt, nt // 32 * 32))
    nt = min(nt, (K["stages"] - 1) << lg)
    return kind, lg, int(gctr), nt


def band_edges(kind):
    """{ring_log2: the largest N whose counters sit in shared memory next to a ring of that size, "gctr": the first N whose
    counters go to global memory}, found by bisection over N on order_plan (the ring size only shrinks as N grows)."""
    S = {3: 3, 4: 4, 8: 8}[kind]
    edges = {}
    for lg in range(K["lg_max"][kind], K["lg_min"] - 1, -1):
        fits = lambda n: (lambda p: not p[2] and p[1] >= lg)(order_plan(n, S, 1, 1, False))   # noqa: E731
        if not fits(1):
            continue
        lo, hi = 1, 1 << 17
        while lo < hi:
            mid = (lo + hi + 1) // 2
            lo, hi = (mid, hi) if fits(mid) else (lo, mid - 1)
        edges[lg] = lo
    edges["gctr"] = edges[K["lg_min"]] + 1
    return edges


# The bands as they stand: rows <= 3 (16 B records, N + 1 counters per slot chain), rows of 4 (4 N), rows of 5..8 (8 N).
PINNED_EDGES = {3: {10: 25023, 9: 41407, 8: 49599, 7: 53695, "gctr": 53696},
                4: {9: 6256, 8: 10352, 7: 12400, "gctr": 12401},
                8: {9: 3128, 8: 5176, 7: 6200, "gctr": 6201}}
EDGES = {kind: band_edges(kind) for kind in (3, 4, 8)}


def _edge(kind, lg, side):
    """N at one side of a band edge: the top of the band of ring_log2 lg ("top"), or one past the top of the band above it
    ("bottom"; lg None: the first GCTR N)."""
    e = EDGES[kind]
    if lg is None:
        return e["gctr"]
    if side == "top":
        return e[lg]
    return e[lg + 1] + 1


# ---- cases ----------------------------------------------------------------------------------------------------------------
# Counter bases: the values preloaded around them (base - 1 .. base + 1) are low, straddle the former sentinel 2^30 - 1, or
# reach INT_MAX minus the run's rows.
LOW, SENT, TOP = "low", "sent", "top"


def _single(cid, plan, kind, lg, side, T, P, RF, desired=-1, base=LOW):
    return dict(id=cid, plan=plan, kind=kind, N=_edge(kind, lg, side), T=T, P=P, RF=RF, desired=desired, base=base)


# Single dense solves (ka_solve_dense), capacity 1 (no level pass). Q = T * P also sits on ring edges: Q = 8 << lg records and
# one more. Rows of 4 and of 5..8 run level widths of max_nt and max_nt + 1 (512 / 513, 256 / 257).
SINGLE_CASES = [
    # rows <= 3 (rows of 2: RF 2; rows of 1: desired RF 1); both slot chains, one launch each
    _single("r3-lg10-top-full", (3, 0, 1024, 10, 0, FULL, 2, 0), 3, 10, "top", T=4, P=1024, RF=2, base=SENT),
    _single("r3-lg10-top-warp1", (3, 0, 32, 10, 0, WARP1, 2, 0), 3, 10, "top", T=6, P=30, RF=2, desired=1, base=TOP),
    _single("r3-lg9-bottom-q4097", (3, 0, 256, 9, 0, SINGLE, 2, 0), 3, 9, "bottom", T=17, P=241, RF=2, desired=1, base=TOP),
    _single("r3-lg9-top-q4096", (3, 0, 256, 9, 0, FULL, 2, 0), 3, 9, "top", T=16, P=256, RF=2, base=LOW),
    _single("r3-lg8-bottom-q2049", (3, 0, 704, 8, 0, SINGLE, 2, 0), 3, 8, "bottom", T=3, P=683, RF=2, base=TOP),
    _single("r3-lg8-top-q2048", (3, 0, 256, 8, 0, FULL, 2, 0), 3, 8, "top", T=8, P=256, RF=2, desired=1, base=SENT),
    _single("r3-lg7-bottom-warp1", (3, 0, 32, 7, 0, WARP1, 2, 0), 3, 7, "bottom", T=4, P=24, RF=2, base=TOP),
    _single("r3-lg7-top-general", (3, 0, 896, 7, 0, GENERAL, 2, 0), 3, 7, "top", T=4, P=1000, RF=2, base=SENT),
    _single("r3-gctr-bottom-general", (3, 0, 768, 10, 1, GENERAL, 2, 0), 3, None, "bottom", T=4, P=1500, RF=2, desired=1, base=TOP),
    _single("r3-gctr-bottom-warp1", (3, 0, 32, 10, 1, WARP1, 2, 0), 3, None, "bottom", T=6, P=20, RF=2, base=SENT),
    # rows of 4: one fused chain
    _single("r4-lg9-top-q4096-w512", (4, 0, 512, 9, 0, GENERAL, 1, 0), 4, 9, "top", T=8, P=512, RF=4, base=SENT),
    _single("r4-lg9-q4097", (4, 0, 256, 9, 0, GENERAL, 1, 0), 4, 9, "top", T=17, P=241, RF=4, base=LOW),
    _single("r4-lg8-bottom-w513", (4, 0, 288, 8, 0, GENERAL, 1, 0), 4, 8, "bottom", T=4, P=513, RF=4, base=TOP),
    _single("r4-lg8-top-q2048", (4, 0, 512, 8, 0, GENERAL, 1, 0), 4, 8, "top", T=4, P=512, RF=4, base=LOW),
    _single("r4-lg8-q2049", (4, 0, 352, 8, 0, GENERAL, 1, 0), 4, 8, "bottom", T=3, P=683, RF=4, base=SENT),
    _single("r4-lg7-bottom-q1025", (4, 0, 224, 7, 0, GENERAL, 1, 0), 4, 7, "bottom", T=5, P=205, RF=4, base=SENT),
    _single("r4-lg7-top-q1024", (4, 0, 512, 7, 0, GENERAL, 1, 0), 4, 7, "top", T=2, P=512, RF=4, base=TOP),
    _single("r4-gctr-bottom-w513", (4, 0, 288, 9, 1, GENERAL, 1, 0), 4, None, "bottom", T=2, P=513, RF=4, base=SENT),
    # rows of 5..8: one fused chain over 8 slots
    _single("r8-lg9-top-q4096-w256", (8, 0, 256, 9, 0, GENERAL, 1, 0), 8, 9, "top", T=16, P=256, RF=6, base=SENT),
    _single("r8-lg9-q4097", (8, 0, 256, 9, 0, GENERAL, 1, 0), 8, 9, "top", T=17, P=241, RF=6, base=LOW),
    _single("r8-lg8-bottom-w257", (8, 0, 160, 8, 0, GENERAL, 1, 0), 8, 8, "bottom", T=8, P=257, RF=5, base=TOP),
    _single("r8-lg8-top-q2049", (8, 0, 256, 8, 0, GENERAL, 1, 0), 8, 8, "top", T=3, P=683, RF=5, base=LOW),
    _single("r8-lg8-q2048", (8, 0, 256, 8, 0, GENERAL, 1, 0), 8, 8, "top", T=8, P=256, RF=6, base=SENT),
    _single("r8-lg7-bottom-q1025", (8, 0, 224, 7, 0, GENERAL, 1, 0), 8, 7, "bottom", T=5, P=205, RF=8, base=SENT),
    _single("r8-lg7-top-q1024", (8, 0, 256, 7, 0, GENERAL, 1, 0), 8, 7, "top", T=4, P=256, RF=6, base=TOP),
    _single("r8-gctr-bottom-w257", (8, 0, 160, 9, 1, GENERAL, 1, 0), 8, None, "bottom", T=2, P=257, RF=6, base=SENT),
]

# Batched dense candidates (ka_solve_dense_candidates_device, rows <= 3 only): the edge table beside a small one that can
# still serve the problem at capacity 1; every table on a fresh Context.
CAND_CASES = [
    dict(id="cand-lg10-top", plan=(3, 0, 128, 10, 0, SINGLE, 2, 2), N=_edge(3, 10, "top"), P=100),
    dict(id="cand-lg9-bottom", plan=(3, 0, 128, 9, 0, FULL, 2, 2), N=_edge(3, 9, "bottom"), P=128),
    dict(id="cand-lg9-top", plan=(3, 0, 32, 9, 0, WARP1, 2, 2), N=_edge(3, 9, "top"), P=24),
    dict(id="cand-lg8-bottom", plan=(3, 0, 704, 8, 0, SINGLE, 2, 2), N=_edge(3, 8, "bottom"), P=700),
    dict(id="cand-lg8-top", plan=(3, 0, 1024, 8, 0, SINGLE, 2, 2), N=_edge(3, 8, "top"), P=1000),
    dict(id="cand-lg7-bottom", plan=(3, 0, 544, 7, 0, GENERAL, 2, 2), N=_edge(3, 7, "bottom"), P=1025),
    dict(id="cand-lg7-top", plan=(3, 0, 32, 7, 0, WARP1, 2, 2), N=_edge(3, 7, "top"), P=32),
    dict(id="cand-gctr-bottom", plan=(3, 0, 256, 10, 1, FULL, 2, 2), N=_edge(3, None, "bottom"), P=256),
]

# ka_solve (ragged, a level plan) at the edges of rows of 4 and of 5..8: RF per topic cycles through `rfs` (short rows in the
# wide records), topic sizes through `sizes`.
RAGGED_CASES = []
for _kind, _rfs, _lgs in ((4, (4, 2, 3, 1), (9, 8, 7)), (8, (6, 5, 8, 3, 1), (9, 8, 7))):
    for _lg in _lgs + (None,):
        for _side in (("top", "bottom") if _lg is not None else ("bottom",)):
            if _lg == K["lg_max"][_kind] and _side == "bottom":
                continue   # no band above the largest ring
            _N = _edge(_kind, _lg, _side)
            _kd, _lgp, _g, _nt = order_plan(_N, _kind, 300, 1, True)
            RAGGED_CASES.append(dict(id="ragged-r%d-%s-%s" % (_kind, "gctr" if _lg is None else "lg%d" % _lg, _side),
                                     plan=(_kind, 1, _nt, _lgp, _g, GENERAL, 1, 0), kind=_kind, N=_N, rfs=_rfs,
                                     sizes=(300, 1, 77, 150, 33), base=(SENT, TOP, LOW)[len(RAGGED_CASES) % 3]))

# Level-plan entry points at the edges of rows <= 3: beyond kernel A's level scratch, refused before anything runs.
R3_SIDES = [(lg, side) for lg in (10, 9, 8, 7) for side in ("top", "bottom") if not (lg == 10 and side == "bottom")] + [(None, "bottom")]

# Staged per-slot chains (ka_order_slot_device with counter-column export / import) at the top of the rows <= 3 bands.
STAGED_CASES = [dict(id="staged-lg7-top", plan=(3, 0, 704, 7, 0, SINGLE), N=_edge(3, 7, "top")),
                dict(id="staged-gctr-bottom", plan=(3, 0, 704, 10, 1, SINGLE), N=_edge(3, None, "bottom"))]
STAGED_T, STAGED_P = 4, 700

# Ragged rows of 1..3 (levels, chunk table) from counters in the high range, in the loop shapes a level plan takes.
HIGH_RAGGED = [dict(id="high-ragged-general-sent", plan=(3, 1, 96, 10, 0, GENERAL, 2, 0), env={}, base=SENT),
               dict(id="high-ragged-general-top", plan=(3, 1, 96, 10, 0, GENERAL, 2, 0), env={}, base=TOP),
               dict(id="high-ragged-warp1-top", plan=(3, 1, 32, 10, 0, WARP1, 2, 0), env={"KA_ORDER_THREADS": "32"}, base=TOP),
               dict(id="high-ragged-gctr-top", plan=(3, 1, 96, 10, 1, GENERAL, 2, 0), env={"KA_ORDER_GLOBAL_CTR": "1"}, base=TOP)]
HIGH_T, HIGH_N, HIGH_PMAX, HIGH_SEED = 80, 3000, 200, 5


def _seed(cid):
    return 0xED6E + sum(ord(ch) * (i + 1) for i, ch in enumerate(cid))


# ---- inputs ---------------------------------------------------------------------------------------------------------------

def _ids(N):
    return (1000 + np.arange(N)).astype(np.int32)


def _topic_lists(rng, N, sizes_rfs):
    """One list of current lists per topic, (P, RF) per topic: distinct brokers inside a topic (capacity 1, so the lists
    stay), and the lowest (index 0) and top (index N - 1) broker in every topic, at random rows."""
    out = []
    for P, RF in sizes_rfs:
        need = P * RF
        assert 2 <= need <= N
        pick = rng.choice(np.arange(1, N - 1), need - 2, replace=False)
        rows = rng.permutation(np.concatenate([[0, N - 1], pick]))
        out.append([[int(x) for x in rows[p * RF:(p + 1) * RF]] for p in range(P)])
    return out


def _names(cid, T):
    names = ["edge.%s.%04d" % (cid, t) for t in range(T)]
    return names, kab.synth.java_string_hash_ascii(names)


def _counters(rng, N, base, rows):
    """Preloaded counters [N, 8]: base - 1 .. base + 1 at random (ties and +-1 gaps), the top and the lowest broker tied below
    the rest in slot 0, the top one below the lowest one in slot 1. base LOW: 1; SENT: 2^30 - 1, so that the values straddle
    the former sentinel; TOP: INT_MAX - rows - 1, so that no counter of the run passes INT_MAX."""
    b = {LOW: 1, SENT: 0x3FFFFFFF, TOP: INT_MAX - rows - 1}[base]
    ctr = (b + rng.integers(-1, 2, size=(N, models.SLOTS))).astype(np.int64)
    ctr[[0, N - 1], 0] = b - 1
    ctr[N - 1, 1], ctr[0, 1] = b - 1, b
    assert ctr.max() + rows <= INT_MAX and (base == LOW or ctr.min() >= SENTINEL_LOW)
    return ctr.astype(np.int32)


def _oracle(oracle, ctr, ids, names, part_off, rep_off, cur, desired, S):
    """(out, out_len, status fields, counters [N, 8]) of the oracle from the preloaded counters ctr."""
    octx = oracle.OracleContext()
    for i, b in enumerate(ids):
        for s in range(models.SLOTS):
            octx.set_counter(int(b), s, int(ctr[i, s]))
    part_id = np.concatenate([np.arange(part_off[t + 1] - part_off[t], dtype=np.int32) for t in range(len(names))])
    ln, _, out, st = oracle.run(octx, names, part_off, part_id, rep_off, cur, ids, [None] * len(ids), desired, S, raise_on_error=False)
    got = np.array([[octx.counter(int(b), s) for s in range(models.SLOTS)] for b in ids], dtype=np.int32)
    return out, ln, (st.code, st.topic_index, st.partition, st.a, st.b), got


def _flat(lists):
    part_off = np.concatenate([[0], np.cumsum([len(t) for t in lists])]).astype(np.int64)
    rows = [r for t in lists for r in t]
    rep_off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    return part_off, rep_off, np.array([b for r in rows for b in r], dtype=np.int32)


# ---- CPU: the restatement and its edges -----------------------------------------------------------------------------------

def test_band_edges_of_the_sources():
    """order_plan over the constants in the sources gives the bands as they stand; a changed constant fails here with the
    new edges, so that the GPU cases (built from the computed edges) follow them."""
    assert K["budget"] == 226 * 1024 and K["stages"] == 8 and K["ring_pad"] == 256
    assert EDGES == PINNED_EDGES, "the chain's shared-memory bands moved: %s" % EDGES
    for kind, e in EDGES.items():
        for lg, top in e.items():
            if lg == "gctr":
                continue
            S = {3: 3, 4: 4, 8: 8}[kind]
            # at the top of a band the counters and the ring fill the budget to the byte (each band is 2^lg stages * 8 records
            # smaller than the one above, a multiple of the counter row); one broker more does not fit
            assert _ctr_bytes(kind, top) + _ring_bytes(kind, lg) == K["budget"], (kind, lg)
            assert order_plan(top, S, 1, 1, False)[1:3] == (lg, 0)
            assert order_plan(top + 1, S, 1, 1, False)[1:3] == ((lg - 1, 0) if lg > K["lg_min"] else (K["lg_max"][kind], 1))


@pytest.mark.parametrize("S", [1, 2, 3, 4, 5, 6, 7, 8])
def test_every_row_width_takes_its_kind_bands(S):
    kind = rec_kind(S)
    e = EDGES[kind]
    for lg in range(K["lg_min"], K["lg_max"][kind] + 1):
        if lg in e:
            assert order_plan(e[lg], S, 64, 1, False)[:3] == (kind, lg, 0), (S, lg)
    assert order_plan(e["gctr"], S, 64, 1, False)[:3] == (kind, K["lg_max"][kind], 1)
    assert order_plan(65535, S, 64, 1, False)[:3] == (kind, K["lg_max"][kind], 1)


def _case_plan(c):
    S = max(c["RF"], c["desired"], 1)
    rf = c["desired"] if c["desired"] >= 0 else c["RF"]
    cap = -(-c["P"] * rf // c["N"])
    return order_plan(c["N"], S, c["P"], cap, False), cap


def test_cases_name_the_plans_of_the_restatement():
    """Each GPU case's named plan (rec_kind, ring_log2, gctr, threads) is the restatement's for its shape, every case sits on
    a band or ring edge, and every (row kind, edge side) pair of the table has a single-solve case."""
    sides = set()
    for c in SINGLE_CASES:
        (kind, lg, gctr, nt), cap = _case_plan(c)
        assert cap == 1, c["id"]
        assert (c["plan"][0], c["plan"][3], c["plan"][4], c["plan"][2]) == (kind, lg, gctr, nt), c["id"]
        sides.add((kind, c["N"]))
    for kind, e in EDGES.items():
        tops = [e[lg] for lg in e if lg != "gctr"]
        assert {(kind, n) for n in tops + [n + 1 for n in tops]} <= sides, (kind, sorted(sides))
    # ring edges Q = 8 << lg and one more, for rows <= 3 at lg 9 and 8, for the wide rows at every lg
    for kind, lgs in ((3, (9, 8)), (4, (9, 8, 7)), (8, (9, 8, 7))):
        for lg in lgs:
            qs = {c["T"] * c["P"] for c in SINGLE_CASES if c["plan"][0] == kind and c["plan"][3] == lg and not c["plan"][4]}
            assert {8 << lg, (8 << lg) + 1} <= qs, (kind, lg, sorted(qs))
    # level widths max_nt and max_nt + 1 of the fused chains
    for kind in (4, 8):
        ps = {c["P"] for c in SINGLE_CASES if c["plan"][0] == kind}
        assert {K["max_nt"][kind], K["max_nt"][kind] + 1} <= ps, kind
    for c in CAND_CASES:
        S, P = 2, c["P"]
        kind, lg, gctr, nt = order_plan(c["N"], S, P, 1, False)
        assert (c["plan"][0], c["plan"][3], c["plan"][4], c["plan"][2]) == (kind, lg, gctr, nt), c["id"]
    assert {c["N"] for c in CAND_CASES} == {_edge(3, lg, side) for lg, side in R3_SIDES}
    for c in STAGED_CASES:
        assert order_plan(c["N"], 2, STAGED_P, 1, False) == (3, c["plan"][3], c["plan"][4], c["plan"][2]), c["id"]
    ids = [c["id"] for c in SINGLE_CASES + CAND_CASES + RAGGED_CASES + STAGED_CASES + HIGH_RAGGED]
    assert len(ids) == len(set(ids))


# ---- CPU: which entry point reaches which edge ----------------------------------------------------------------------------

def _level_plan_fits(N, S, Pmax):
    """Kernel A's layout for a level plan (every ragged entry point) over brokers 1000 .. 1000 + N - 1."""
    return models.stage_warps(N, models.blob_bytes(_ids(N)), Pmax, S, 1, True) > 0


def reachable(entry, kind, N, Pmax):
    """None when `entry` runs a table of N brokers at rows of `kind` (Pmax partitions in the largest topic, capacity 1), else
    the documented refusal: (code, a, b) of every status it reports (a = 0 / b = 0 where the refusal does not name them)."""
    S = {3: 3, 4: 4, 8: 8}[kind]
    if entry in ("dense_candidates", "ragged_candidates", "clusters", "staged_slots") and kind != 3:
        # the batched chains and the per-slot chains are the slot chains of rows <= 3: out_stride > 3 is refused for the
        # whole batched call; a staged block of wider rows has no per-slot chains (ka_staged_slot_chains() == 0)
        return (LIMIT, 0, 0) if entry != "staged_slots" else "no per-slot chains"
    if entry in ("ragged", "ragged_candidates", "clusters") and not _level_plan_fits(N, S, Pmax):
        return (LIMIT, Pmax, N)
    assert _level_plan_fits(N, S, Pmax) or models.stage_warps(N, models.blob_bytes(_ids(N)), Pmax, S, 1, False) > 0
    return None


ENTRIES = ("dense", "staged_slots", "dense_candidates", "ragged", "ragged_candidates", "clusters")


def test_reachability_of_every_edge():
    """Every (entry point, edge side) pair either runs or has its documented refusal. Single dense solves and the dense
    batched and staged paths (capacity 1: no level pass) reach every band of their rows; level plans are capped by kernel
    A's level scratch below the first band edge of rows <= 3, and reach every edge of the wider rows."""
    for kind, e in EDGES.items():
        for v in sorted(set(e.values()) | {x + 1 for x in e.values()}):
            for entry in ENTRIES:
                got = reachable(entry, kind, v, 300)
                if entry == "dense" or (entry in ("staged_slots", "dense_candidates") and kind == 3) or (entry == "ragged" and kind != 3):
                    assert got is None, (entry, kind, v, got)
                else:
                    assert got is not None, (entry, kind, v)
    # the level scratch's largest table at rows <= 3 lies below the first band edge, whatever the topic sizes
    largest = max(n for n in range(15000, EDGES[3][10] + 1, 16) if _level_plan_fits(n, 3, 1))
    assert largest < EDGES[3][10], largest
    # the level plans at the wide rows' edges run with room to spare for a 300-partition topic
    assert all(_level_plan_fits(e["gctr"], {4: 4, 8: 8}[kind], 300) for kind, e in EDGES.items() if kind != 3)


# ---- CPU: the dummy broker's sentinel -------------------------------------------------------------------------------------

def test_model_sentinel_is_the_kernels():
    """The slot-chain model pads with the counter the chain kernel writes for the dummy broker."""
    assert K["dummy"] == models.INF == INT_MAX


def _ragged_rows_1_to_3(seed, T=40, N=60, max_partitions=24):
    cl = kab.synth.make_ragged_cluster(T=T, N=N, R=6, max_partitions=max_partitions, seed=seed, rf_weights=(0.4, 0.4, 0.2))
    rf = np.diff(cl.rep_off)
    assert set(rf.tolist()) == {1, 2, 3}
    return cl


@pytest.mark.parametrize("base", [SENTINEL_LOW + 1, 0x3FFFFFFF, 0x40000000, "top"])
@pytest.mark.parametrize("seed", [3, 11])
def test_sentinel_never_beats_a_real_counter(oracle, base, seed):
    """Rows of 1, 2 and 3 mixed in one run (a ragged cluster, capacity > 1: levels), from counters in
    [2^30 - 3, INT_MAX - rows] with ties and +-1 gaps: the slot-chain model, which pads with the kernel's dummy, gives the
    oracle's rows and final Context. With the former sentinel (2^30 - 1) the dummy won slot 0 of a row of 1 or 2 whose real
    counters were above it, and a dummy bumped by rows of 1 wrapped past INT_MAX."""
    cl = _ragged_rows_1_to_3(seed)
    Q = cl.Q
    rng = np.random.default_rng(seed)
    b = INT_MAX - Q - 1 if base == "top" else base
    ctr = (b + rng.integers(-1, 2, size=(cl.N, 3))).astype(np.int64)
    ctr[[0, cl.N - 1], 0] = b - 1
    assert ctr.min() >= SENTINEL_LOW and ctr.max() + Q <= INT_MAX
    octx = oracle.OracleContext()
    for i, bid in enumerate(cl.broker_id):
        for s in range(3):
            octx.set_counter(int(bid), s, int(ctr[i, s]))
    S = 3
    ln, _, out, st = oracle.run(octx, cl.topic_names, cl.part_off, cl.part_id, cl.rep_off, cl.cur, cl.broker_id, cl.rack_name, -1, S)
    assert st.code == 0
    sets = [[[int(x) for x in out[g, :ln[g]]] for g in range(int(cl.part_off[t]), int(cl.part_off[t + 1]))] for t in range(cl.T)]
    assert {len(r) for t in sets for r in t} == {1, 2, 3}
    c0 = [int(x) for x in ctr[:, 0]] + [models.INF]
    c1 = [int(x) for x in ctr[:, 1]] + [models.INF]
    c2 = [int(x) for x in ctr[:, 2]] + [0]
    got = models.slot_chains(cl, sets, random.Random(seed), c0, c1, c2)
    for g in range(Q):
        assert cl.N not in got[g], (g, "the dummy broker won a slot")
        assert [int(cl.broker_id[i]) for i in got[g]] == [int(x) for x in out[g, :ln[g]]], g
    for i, bid in enumerate(cl.broker_id):
        assert (c0[i], c1[i], c2[i]) == tuple(octx.counter(int(bid), s) for s in range(3)), int(bid)


# ---- GPU ------------------------------------------------------------------------------------------------------------------

def _check_counters(s, exp_ctr, cid):
    got = s.counters()
    bad = np.argwhere(got != exp_ctr)
    assert not len(bad), (cid, [(int(i), int(r), int(got[i, r]), int(exp_ctr[i, r])) for i, r in bad[:8]])


@pytest.mark.gpu
@pytest.mark.parametrize("case", SINGLE_CASES, ids=[c["id"] for c in SINGLE_CASES])
def test_single_solve_at_band_edge(native_lib, oracle, case):
    c = case
    rng = np.random.default_rng(_seed(c["id"]))
    N, T, P, RF = c["N"], c["T"], c["P"], c["RF"]
    S = max(RF, c["desired"], 1)
    ids = _ids(N)
    lists = _topic_lists(rng, N, [(P, RF)] * T)
    cur = ids[np.array(lists, dtype=np.int64)]
    names, th = _names(c["id"], T)
    ctr = _counters(rng, N, c["base"], T * P)
    part_off, rep_off, flat = _flat([[[int(ids[b]) for b in r] for r in t] for t in lists])
    exp, exp_len, est, exp_ctr = _oracle(oracle, ctr, ids, names, part_off, rep_off, flat, c["desired"], S)
    assert est[0] == 0, est
    s = kab.Solver(0)
    s.set_brokers(*util.table(ids))
    s.set_counters(ctr)
    assert np.array_equal(s.counters(), ctr)   # ka_ctx_get_counters after ka_ctx_set_counters
    out, out_len, st = s.solve_dense(th, cur, c["desired"], S, check=False)
    assert s.last_order_plan() == c["plan"], (c["id"], s.last_order_plan())
    assert util.fields(st) == est, (c["id"], util.fields(st), est)
    assert np.array_equal(out.reshape(-1, S), exp), c["id"]
    assert np.array_equal(out_len.reshape(-1), exp_len), c["id"]
    _check_counters(s, exp_ctr, c["id"])


@pytest.mark.gpu
@pytest.mark.parametrize("case", CAND_CASES, ids=[c["id"] for c in CAND_CASES])
def test_dense_candidates_at_band_edge(native_lib, oracle, case):
    """The edge table as the largest of two, beside one that serves the problem at capacity 1: the call's one plan is the
    edge table's, and each candidate equals its own fresh-Context solve and the oracle."""
    c = case
    rng = np.random.default_rng(_seed(c["id"]))
    N, P, T, RF = c["N"], c["P"], 3, 2
    ids = _ids(N)
    lists = _topic_lists(rng, N, [(P, RF)] * T)
    cur = ids[np.array(lists, dtype=np.int64)]
    _, th = _names(c["id"], T)
    small = util.table(_ids(max(256, P * RF)))
    s = kab.Solver(0)
    sts = util.check_dense_equal(util.DenseProblem(th, cur), [small, util.table(ids)], oracle, solver=s)
    assert s.last_order_plan() == c["plan"], (c["id"], s.last_order_plan())
    assert all(x[0] == 0 for x in sts), sts


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [4, 8])
def test_wide_rows_are_refused_by_the_batched_calls(native_lib, kind):
    """Rows wider than 3 at the wide rows' edges: the batched calls refuse the stride for every member before anything runs
    (their chains are the slot chains of rows <= 3); single solves take them (above)."""
    rng = np.random.default_rng(kind)
    N, S = EDGES[kind][K["lg_min"]], kind
    ids = _ids(N)
    lists = _topic_lists(rng, N, [(20, S), (10, 1)])
    names, th = _names("wide%d" % kind, 2)
    part_off, rep_off, flat = _flat([[[int(ids[b]) for b in r] for r in t] for t in lists])
    pid = np.concatenate([np.arange(20), np.arange(10)]).astype(np.int32)
    tables = [util.table(_ids(300)), util.table(ids)]
    s = kab.Solver(0)
    _, _, sts = s.solve_ragged_candidates(tables, th, part_off, pid, rep_off, flat, -1)
    assert [util.fields(x) for x in sts] == [(LIMIT, -1, -1, 0, 0)] * 2
    assert s.last_order_plan() == (0,) * 8
    res = s.solve_clusters([(*tables[1], th, part_off, pid, rep_off, flat, -1)])
    assert [util.fields(x[2]) for x in res] == [(LIMIT, -1, -1, 0, 0)]
    import torch
    cur = torch.from_numpy(ids[np.array(lists[0], dtype=np.int64)].reshape(1, 20, S)).cuda()
    d_th = torch.from_numpy(th[:1].copy()).cuda()
    out = torch.zeros((2, 1, 20, S), dtype=torch.int32, device="cuda")
    sts = s.solve_dense_candidates_device(tables, 1, d_th.data_ptr(), 20, S, cur.data_ptr(), -1, S, 0, out.data_ptr())
    assert [util.fields(x) for x in sts] == [(LIMIT, -1, -1, 0, 0)] * 2


@pytest.mark.gpu
@pytest.mark.parametrize("case", RAGGED_CASES, ids=[c["id"] for c in RAGGED_CASES])
def test_ragged_solve_at_band_edge(native_lib, oracle, case):
    """ka_solve (a level plan) at the edges of rows of 4 and of 5..8, rows of every length up to the kind's, from preloaded
    counters."""
    c = case
    rng = np.random.default_rng(_seed(c["id"]))
    N = c["N"]
    T = 10
    shape = [(c["sizes"][t % len(c["sizes"])], c["rfs"][t % len(c["rfs"])]) for t in range(T)]
    S = max(rf for _, rf in shape)
    assert reachable("ragged", c["kind"], N, max(p for p, _ in shape)) is None
    ids = _ids(N)
    lists = _topic_lists(rng, N, shape)
    names, th = _names(c["id"], T)
    part_off, rep_off, flat = _flat([[[int(ids[b]) for b in r] for r in t] for t in lists])
    Q = int(part_off[-1])
    ctr = _counters(rng, N, c["base"], Q)
    exp, exp_len, est, exp_ctr = _oracle(oracle, ctr, ids, names, part_off, rep_off, flat, -1, S)
    assert est[0] == 0, est
    s = kab.Solver(0)
    s.set_brokers(*util.table(ids))
    s.set_counters(ctr)
    pid = np.concatenate([np.arange(p, dtype=np.int32) for p, _ in shape])
    out, out_len, st = s.solve_ragged(th, part_off, pid, rep_off, flat, -1, S, check=False)
    assert s.last_order_plan() == c["plan"], (c["id"], s.last_order_plan())
    assert util.fields(st) == est, (c["id"], util.fields(st), est)
    assert np.array_equal(out, exp) and np.array_equal(out_len, exp_len), c["id"]
    _check_counters(s, exp_ctr, c["id"])


def _r3_ragged(rng, N, cid):
    """A ragged problem of rows of 1..3 over brokers 1000 .. 1000 + N - 1, with the top and lowest broker in every topic."""
    shape = [(40, 2), (12, 1), (30, 3), (25, 2)]
    ids = _ids(N)
    lists = _topic_lists(rng, N, shape)
    names, th = _names(cid, len(shape))
    part_off, rep_off, flat = _flat([[[int(ids[b]) for b in r] for r in t] for t in lists])
    pid = np.concatenate([np.arange(p, dtype=np.int32) for p, _ in shape])
    return ids, names, th, part_off, pid, rep_off, flat, max(p for p, _ in shape)


@pytest.mark.gpu
@pytest.mark.parametrize("lg,side", R3_SIDES, ids=["%s-%s" % ("gctr" if lg is None else "lg%d" % lg, side) for lg, side in R3_SIDES])
def test_level_plans_refuse_the_bands_of_short_rows(native_lib, oracle, lg, side):
    """ka_solve, ka_solve_candidates and ka_solve_clusters at a rows <= 3 edge: kernel A's level scratch refuses the table
    (KA_ERR_LIMIT, a = the largest topic, b = N) before anything runs. ka_solve_candidates sizes one plan from its largest
    table, so every candidate reports it; ka_solve_clusters refuses only the clusters whose own plan fails, and the others
    still solve."""
    N = _edge(3, lg, side)
    rng = np.random.default_rng(N)
    ids, names, th, part_off, pid, rep_off, flat, Pmax = _r3_ragged(rng, N, "lvl%d" % N)
    want = (LIMIT, -1, -1, Pmax, N)
    assert reachable("ragged", 3, N, Pmax) == (LIMIT, Pmax, N)
    s = kab.Solver(0)
    s.set_brokers(*util.table(ids))
    _, _, st = s.solve_ragged(th, part_off, pid, rep_off, flat, -1, 3, check=False)
    assert util.fields(st) == want and s.last_order_plan() == (0,) * 8
    small = util.table(_ids(200))
    _, _, sts = s.solve_ragged_candidates([small, util.table(ids)], th, part_off, pid, rep_off, flat, -1)
    assert [util.fields(x) for x in sts] == [want] * 2
    # a fleet: a small cluster beside this edge's table and the next band's first
    N2 = N + 1
    ids2 = _ids(N2)
    lists2 = _topic_lists(rng, N2, [(Pmax, 2), (7, 3)])
    th2 = _names("lvl2-%d" % N2, 2)[1]
    po2, ro2, fl2 = _flat([[[int(ids2[b]) for b in r] for r in t] for t in lists2])
    pid2 = np.concatenate([np.arange(Pmax), np.arange(7)]).astype(np.int32)
    small_cl = util.Member.of(kab.synth.make_ragged_cluster(T=12, N=200, R=5, max_partitions=30, seed=N, remove_frac=0.05))
    fleet = [small_cl, util.Member(util.table(ids), names, th, part_off, pid, rep_off, flat),
             util.Member(util.table(ids2), ["a", "b"], th2, po2, pid2, ro2, fl2)]
    res = s.solve_clusters([m.entry() for m in fleet], out_stride=3)
    assert util.fields(res[1][2]) == want
    assert util.fields(res[2][2]) == (LIMIT, -1, -1, Pmax, N2)
    e_out, e_len, e_st = small_cl.sequential(kab.Solver(0), 3)
    assert util.fields(res[0][2]) == e_st and e_st[0] == 0
    assert np.array_equal(res[0][0], e_out) and np.array_equal(res[0][1], e_len)


@pytest.mark.gpu
@pytest.mark.parametrize("case", STAGED_CASES, ids=[c["id"] for c in STAGED_CASES])
def test_staged_slot_chains_at_band_edge(native_lib, oracle, case):
    """The staged per-slot path at the top of the rows <= 3 bands: ka_ctx_set_counters loads every slot, then each slot
    chain's column is replaced through ka_ctx_import_counter_slot_device before it runs and read back through
    ka_ctx_export_counter_slot_device after; rows and every counter equal the oracle's from the same counters."""
    import torch
    c = case
    rng = np.random.default_rng(_seed(c["id"]))
    N, T, P, RF = c["N"], STAGED_T, STAGED_P, 2
    ids = _ids(N)
    lists = _topic_lists(rng, N, [(P, RF)] * T)
    cur = ids[np.array(lists, dtype=np.int64)]
    names, th = _names(c["id"], T)
    set_ctr = _counters(rng, N, TOP, T * P)
    cols = _counters(rng, N, SENT, T * P)[:, :2]        # what the per-slot imports bring in, straddling 2^30
    ctr = set_ctr.copy()
    ctr[:, :2] = cols
    part_off, rep_off, flat = _flat([[[int(ids[b]) for b in r] for r in t] for t in lists])
    exp, exp_len, est, exp_ctr = _oracle(oracle, ctr, ids, names, part_off, rep_off, flat, -1, RF)
    assert est[0] == 0
    s = kab.Solver(0)
    s.set_brokers(*util.table(ids))
    s.set_counters(set_ctr)
    d_th, d_cur = torch.from_numpy(th).cuda(), torch.from_numpy(cur).cuda()
    d_out = torch.full((T, P, RF), -7, dtype=torch.int32, device="cuda")
    d_len = torch.full((T, P), -7, dtype=torch.int32, device="cuda")
    col = torch.zeros(N, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    s.stage_dense_device(T, d_th.data_ptr(), P, RF, d_cur.data_ptr(), -1, RF)
    assert s.staged_slot_chains() == 2
    for slot in (0, 1):
        col.copy_(torch.from_numpy(np.ascontiguousarray(cols[:, slot])))
        torch.cuda.synchronize()
        s.import_counter_slot_device(slot, col.data_ptr())
        s.order_slot_device(slot)
        assert s.last_order_plan() == c["plan"] + (slot + 1, 0), (c["id"], s.last_order_plan())
        col.fill_(-7)
        s.export_counter_slot_device(slot, col.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(col.cpu().numpy(), exp_ctr[:, slot]), (c["id"], slot)
    st = s.emit_device(d_len.data_ptr(), d_out.data_ptr())
    assert util.fields(st) == est
    assert np.array_equal(d_out.cpu().numpy().reshape(-1, RF), exp) and np.array_equal(d_len.cpu().numpy().reshape(-1), exp_len)
    _check_counters(s, exp_ctr, c["id"])


@pytest.mark.gpu
@pytest.mark.parametrize("case", HIGH_RAGGED, ids=[c["id"] for c in HIGH_RAGGED])
def test_high_counters_with_short_rows(native_lib, oracle, case):
    """Rows of 1, 2 and 3 in one run (the dummy pads rows of 1 and 2) from counters in the high range, in the loop shapes
    and counter placements a level plan takes: rows, status and every counter equal the oracle's."""
    from unittest import mock
    c = case
    rng = np.random.default_rng(_seed(c["id"]))
    cl = _ragged_rows_1_to_3(HIGH_SEED, T=HIGH_T, N=HIGH_N, max_partitions=HIGH_PMAX)
    ids = cl.broker_id
    S = 3
    ctr = _counters(rng, len(ids), c["base"], cl.Q)
    exp, exp_len, est, exp_ctr = _oracle(oracle, ctr, ids, cl.topic_names, cl.part_off, cl.rep_off, cl.cur, -1, S)
    assert est[0] == 0
    s = kab.Solver(0)
    s.set_brokers(*util.table(ids))
    s.set_counters(ctr)
    with mock.patch.dict(os.environ, c["env"]):
        out, out_len, st = s.solve_ragged(cl.topic_hash, cl.part_off, cl.part_id, cl.rep_off, cl.cur, -1, S, check=False)
    assert s.last_order_plan() == c["plan"], (c["id"], s.last_order_plan())
    assert util.fields(st) == est
    assert np.array_equal(out, exp) and np.array_equal(out_len, exp_len), c["id"]
    _check_counters(s, exp_ctr, c["id"])
