"""The second half of the reference path's contract: the exception of the first topic that throws (KAG:173 aborts there).
ka_status names the LOWEST failing topic in loop order and, inside it, the first failure in the reference's own evaluation
order (include/kassign.h). At scale that report crosses every piece of the pipelined solve: kernel A's per-topic status and
atomicMin (kassign_stage.cuh), the flags reset once for all topic blocks, block bounds that differ between host-buffer and
device entries, chain sub-blocks, JSON fragments streamed before the status is known, the asynchronous status, and the
staged per-slot calls' topic_base.

In kernel A a topic's failure depends on that topic alone (its lists, its hash, the table and desired_rf), so failing DONOR
topics, found with the oracle, are spliced into an otherwise solvable cluster at chosen topic indices: the run must fail at
its lowest donor with that donor's status. Donors go to the first and last topic of the run and of every topic block, and to
the first topic of a chain sub-block j > 0, under every block layout the dispatcher reaches; a small restatement of that
layout (pipeline_stages, the block bounds, chain_subblocks, sub_block in kassign.cu), pinned to the source below, says where
those topics are, and each GPU case checks through ka_ctx_last_order_plan that it reached the layout it names.

CPU: the donors, the hosts, the splice rule and the layout restatement. GPU: every dense single-solve entry point, the ragged
solves at JSON fragment edges, the staged per-slot calls, the CLI, and what a Context holds after a failure. Every status is
compared field by field (code, topic_index, partition, a, b) with the oracle's."""
import functools
import json
import os
import re
import subprocess
from unittest import mock

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from oracle import oracle_lib as ol
from tests import models, util

CSRC = os.path.join(os.path.dirname(util.HERE), "kafka_assigner_b200", "csrc")

P, RF, N = 48, 3, 48       # zero slack: P * RF == N * capacity (capacity 3)
INT_MIN = -2 ** 31
ENV_KEYS = ("KA_PIPELINE_STAGES", "KA_CHAIN_SUBBLOCKS")


# ---- the layout of a dense single solve, restated from kassign.cu ----------------------------------------------------------

def _source():
    return open(os.path.join(CSRC, "kassign.cu")).read()


def _constants():
    cu = _source()
    get = lambda pat: int(re.search(pat, cu).group(1))  # noqa: E731
    return dict(max_blocks=get(r"constexpr int KA_MAX_BLOCKS = (\d+);"),
                max_chain_blocks=get(r"constexpr int KA_MAX_CHAIN_BLOCKS = (\d+);"),
                sub_topics=get(r"constexpr int KA_CHAIN_SUB_TOPICS = (\d+);"),
                large_block=get(r"constexpr int KA_CHAIN_LARGE_BLOCK = (\d+);"),
                frag_rows=1 << get(r"constexpr int64_t KA_JSON_FRAG_ROWS = 1 << (\d+);"))


MAX_BLOCKS, MAX_CHAIN_BLOCKS, CHAIN_SUB_TOPICS, CHAIN_LARGE_BLOCK = 8, 16, 512, 1024
MAX_CHAIN_EVENTS = MAX_BLOCKS * MAX_CHAIN_BLOCKS     # chain sub-blocks per solve
JSON_FRAG_ROWS = 1 << 18


def _atoi(s):
    m = re.match(r"\s*([+-]?\d+)", s)
    return int(m.group(1)) if m else 0


def pipeline_stages(T, Q, env):
    """Topic blocks of a dense solve."""
    k = min(4, T // 2048) if Q >= 262144 else 1
    if "KA_PIPELINE_STAGES" in env:
        k = _atoi(env["KA_PIPELINE_STAGES"])
    return max(1, min(k, min(MAX_BLOCKS, max(T, 1))))


def bounds(T, K, host_io):
    """The K + 1 block bounds. host_io (an entry with host inputs or outputs): with K >= 3 the end blocks get half the weight
    of the inner ones (1:2:..:2:1)."""
    host_io = host_io and K >= 3
    wsum = 2 * (K - 1) if host_io else K

    def bound(k):
        if k <= 0:
            return 0
        if k >= K:
            return T
        return T * (2 * k - 1 if host_io else k) // wsum
    return [bound(k) for k in range(K + 1)]


def chain_subblocks(Tb, blocks_in_solve, overlapped, env):
    """Chain sub-blocks of a dense block of Tb topics with rows of 3."""
    if Tb < 2:
        return 1
    n = max(1, 8 // max(1, blocks_in_solve))
    n = min(n, max(1, Tb // 128))
    if overlapped and Tb >= CHAIN_LARGE_BLOCK:
        n = max(n, Tb // CHAIN_SUB_TOPICS)
    if "KA_CHAIN_SUBBLOCKS" in env:
        n = max(1, min(_atoi(env["KA_CHAIN_SUBBLOCKS"]), Tb))
    return min(n, MAX_CHAIN_BLOCKS)


def sub_block(Tb, j, nsub):
    """Topics [t0, t1) of sub-block j of a block."""
    return Tb * j // nsub, Tb * (j + 1) // nsub


class Layout:
    """Where the blocks and sub-blocks of a dense single solve of T topics of P partitions fall, for an entry with or without
    host buffers."""

    def __init__(self, T, env, host_io):
        self.T, self.env = T, env
        self.K = pipeline_stages(T, T * P, env)
        self.b = bounds(T, self.K, host_io)
        self.nsub = [chain_subblocks(self.b[k + 1] - self.b[k], self.K, True, env) for k in range(self.K)]
        assert sum(self.nsub) <= MAX_CHAIN_EVENTS

    def chain_launches(self):
        return 2 * sum(self.nsub)

    def positions(self):
        """{name: topic}: topic 0 and the last topic, the first and the last topic of every block, the first topic of
        sub-block 1 of the first and of the last block. One name per topic, the first that reaches it."""
        named = [("t0", 0), ("last", self.T - 1)]
        for k in range(self.K):
            named += [("b%dfirst" % k, self.b[k]), ("b%dlast" % k, self.b[k + 1] - 1)]
        for k in sorted({0, self.K - 1}):
            if self.nsub[k] > 1:
                named.append(("b%ds1first" % k, self.b[k] + sub_block(self.b[k + 1] - self.b[k], 1, self.nsub[k])[0]))
        out = {}
        for name, t in named:
            if t not in out.values():
                out[name] = t
        return out


# ---- donors: topics that fail alone, found with the oracle ------------------------------------------------------------------

def _table(kind):
    """The 48-broker tables: 'flat' without racks (every broker its own rack), 'racked' with racks i % 4 of 12 brokers each."""
    ids = (1000 + np.arange(N)).astype(np.int32)
    names = [None] * N if kind == "flat" else ["r%02d" % (i % 4) for i in range(N)]
    return ids, names, kab.synth.rack_indices(ids, names)


def _structured(t):
    """A topic whose lists keep every current replica on either table: consecutive ids, each broker three times."""
    return ((1000 + (t + 3 * np.arange(P)[:, None] + np.arange(RF)[None, :]) % N)).astype(np.int32)


def _dense_status(table, hashes, cur, ctx=None):
    ids, _, racks = _table(table)
    out, ln, st = ol.fast_run_dense(ctx or ol.FastContext(), np.asarray(hashes, dtype=np.int32), cur, ids, racks)
    return out, ln, (st.code, st.topic_index, st.partition, st.a, st.b)


class Donor:
    def __init__(self, name, table, topic, topic_hash, cur):
        self.name, self.table, self.topic, self.hash, self.cur = name, table, topic, int(topic_hash), cur


def _search(table, seed, want):
    """The first topic of a random zero-slack cluster on `table` for which want(status) holds."""
    cl = kab.synth.make_cluster(T=400, P=P, RF=RF, N=N, R=4, seed=seed, kind="random", rack_aware=table == "racked",
                                n_old=N, topic_prefix="donor-")
    for t in range(cl.T):
        _, _, st = _dense_status(table, cl.topic_hash[t:t + 1], cl.cur[t:t + 1])
        if want(st):
            return cl.topic_names[t], cl.topic_hash[t], cl.cur[t]
    raise AssertionError("no such donor")


def _cannot_serve():
    """Racks A, B, C, D (brokers i % 4 == 0..3). Partitions 0..35 keep one C and one D replica each, which fills both racks
    (12 brokers x capacity 3); partitions 36..47 hold only A and B replicas (their third one repeats the rack of the first),
    so each needs a third rack that has no room left: 12 partitions cannot be fully assigned, the first of them 36."""
    rk = lambda r, j: 1000 + 4 * j + r  # noqa: E731   broker j of rack r
    cur = np.zeros((P, RF), dtype=np.int32)
    for p in range(36):
        cur[p] = [rk(2, p % 12), rk(3, p % 12), rk(p % 2, p % 12)]
    for i in range(12):
        cur[36 + i] = [rk(0, 2 * (i % 6) + 1), rk(1, 2 * (i % 6)), rk(0, 2 * ((i + 1) % 6) + 1)]
    name = "donor.cannot-serve"
    return name, kab.synth.java_string_hash_ascii([name])[0], cur


@functools.lru_cache(maxsize=None)
def donors():
    """The dense donors by name (they also serve the ragged layout): UNASSIGNABLE on each table (on the racked one with its
    first failing partition inside the topic), HASH_INDEX (hashCode Integer.MIN_VALUE on 48 brokers: 2^31 % 48 != 0)."""
    d = {}
    d["unassignable-flat"] = Donor("unassignable-flat", "flat",
                                   *_search("flat", 0xD0401, lambda st: st[0] == 4 and 0 < st[2] < P - 1))
    d["unassignable-racked"] = Donor("unassignable-racked", "racked",
                                     *_search("racked", 0xD0402, lambda st: st[0] == 4 and 0 < st[2] < P - 8))
    d["cannot-serve"] = Donor("cannot-serve", "racked", *_cannot_serve())
    _, _, cur = _search("flat", 0xD0403, lambda st: st[0] == 0)
    d["hash-index"] = Donor("hash-index", "flat", util.MIN_HASH, INT_MIN, cur)
    return d


DENSE_DONORS = ("unassignable-flat", "cannot-serve", "hash-index", "unassignable-racked")


@functools.lru_cache(maxsize=None)
def alone(name):
    """The oracle's status of a donor solved alone."""
    dn = donors()[name]
    return _dense_status(dn.table, [dn.hash], dn.cur[None])[2]


# ---- hosts: clusters that solve, on each table --------------------------------------------------------------------------------

HOST_T = 6144


@functools.lru_cache(maxsize=None)
def host(table):
    """A mixed zero-slack cluster of HOST_T topics on `table` that solves: every topic that fails alone is replaced by a
    structured one. Smaller hosts are its prefixes."""
    cl = kab.synth.make_cluster(T=HOST_T, P=P, RF=RF, N=N, R=4, seed=0x4057 + (table == "racked"), kind="mixed",
                                rack_aware=table == "racked", n_old=N)
    for t in range(cl.T):
        if _dense_status(table, cl.topic_hash[t:t + 1], cl.cur[t:t + 1])[2][0] != 0:
            cl.cur[t] = _structured(t)
    return cl


def spliced(table, T, placed):
    """The host's first T topics with donors at chosen topics: placed = {topic: donor name}. (names, hashes, cur)."""
    h = host(table)
    names, th, cur = list(h.topic_names[:T]), h.topic_hash[:T].copy(), h.cur[:T].copy()
    for t, name in placed.items():
        dn = donors()[name]
        assert dn.table == table
        names[t], th[t], cur[t] = dn.topic if len(placed) == 1 else "%s.%d" % (dn.topic, t), dn.hash, dn.cur
        if dn.name == "hash-index":
            names[t] = util.MIN_HASH   # the name must keep its hash
    return names, th, cur


@functools.lru_cache(maxsize=None)
def expected(table, T, placed):
    """The oracle's status of a spliced cluster (placed: a tuple of (topic, donor name))."""
    _, th, cur = spliced(table, T, dict(placed))
    return _dense_status(table, th, cur)[2]


def splice_rule(placed):
    """The status a spliced run must report: its lowest donor's, at that donor's topic."""
    t, name = min(placed)
    code, _, part, a, b = alone(name)
    return code, t, part, a, b


# ---- the cases ----------------------------------------------------------------------------------------------------------------

LAYOUTS = [
    dict(id="K1", T=300, env={"KA_PIPELINE_STAGES": "1"}),
    dict(id="K2", T=600, env={"KA_PIPELINE_STAGES": "2"}),
    dict(id="K3", T=900, env={"KA_PIPELINE_STAGES": "3"}),
    dict(id="K5", T=1000, env={"KA_PIPELINE_STAGES": "5"}),
    dict(id="K8", T=1200, env={"KA_PIPELINE_STAGES": "8"}),
    # the default rule: Q >= 262 144 and T >= 4 096 gives 3 blocks of about 2 048 topics, each cut by the large-block rule
    dict(id="default", T=6144, env={}),
    dict(id="sub40", T=700, env={"KA_PIPELINE_STAGES": "2", "KA_CHAIN_SUBBLOCKS": "40"}),
    # 8 blocks of 16 sub-blocks: the 128 chain sub-blocks a solve can hold
    dict(id="cap128", T=1200, env={"KA_PIPELINE_STAGES": "8", "KA_CHAIN_SUBBLOCKS": "16"}),
]
# dense entry points: name -> uses host buffers (the block bounds of host_io)
ENTRIES = {"host": True, "device": False, "async": False, "json": True, "json-small": True}


def _dense_cases():
    cases = []
    for lay in LAYOUTS:
        for entry, host_io in ENTRIES.items():
            L = Layout(lay["T"], lay["env"], host_io)
            pos = L.positions()
            for i, (pname, t) in enumerate(pos.items()):
                name = DENSE_DONORS[i % len(DENSE_DONORS)]
                cases.append(dict(id="%s-%s-%s-%s" % (lay["id"], pname, name, entry), layout=lay, entry=entry,
                                  table=donors_table(name), placed=((t, name),)))
            if L.K >= 2:
                # two donors in different blocks: the later one's kind (hashCode, KAS:190) is evaluated before the earlier
                # one's (KAS:183) inside a topic, and still the lower topic wins
                t1, t2 = L.b[1] - 1, L.b[L.K - 1]
                cases.append(dict(id="%s-b0last+b%dfirst-two-donors-%s" % (lay["id"], L.K - 1, entry), layout=lay, entry=entry,
                                  table="flat", placed=((t1, "unassignable-flat"), (t2, "hash-index"))))
    return cases


def donors_table(name):
    return "racked" if name in ("cannot-serve", "unassignable-racked") else "flat"


DENSE_CASES = _dense_cases()


# ---- CPU: the layout restatement, pinned to the source -----------------------------------------------------------------------

def test_layout_constants_are_the_sources():
    assert _constants() == dict(max_blocks=MAX_BLOCKS, max_chain_blocks=MAX_CHAIN_BLOCKS, sub_topics=CHAIN_SUB_TOPICS,
                                large_block=CHAIN_LARGE_BLOCK, frag_rows=JSON_FRAG_ROWS)
    cu = _source()
    for line in ("constexpr int KA_MAX_CHAIN_EVENTS = KA_MAX_BLOCKS * KA_MAX_CHAIN_BLOCKS;",
                 # pipeline_stages
                 "int k = Q >= 262144 ? std::min(4, T / 2048) : 1;",
                 'if (const char* e = std::getenv("KA_PIPELINE_STAGES")) k = std::atoi(e);',
                 "return std::max(1, std::min(k, std::min(KA_MAX_BLOCKS, std::max(T, 1))));",
                 # run_solve's block bounds
                 "const int K = ragged ? 1 : pipeline_stages(T, (int64_t)T * sh.P);",
                 "const bool host_io = (io.h_cur != nullptr || io.h_out != nullptr) && K >= 3;",
                 "const int wsum = host_io ? 2 * (K - 1) : K;",
                 "auto bound = [&](int k) { return k <= 0 ? 0 : (k >= K ? T : (int)((int64_t)T * (host_io ? 2 * k - 1 : k) / wsum)); };",
                 # chain_subblocks
                 "if (d.d_part_off || d.pl.rec_kind != 3 || d.T < 2) return 1;",
                 "int n = std::max(1, 8 / std::max(1, blocks_in_solve));",
                 "n = std::min(n, std::max(1, d.T / 128));",
                 "if (overlapped && d.T >= KA_CHAIN_LARGE_BLOCK) n = std::max(n, d.T / KA_CHAIN_SUB_TOPICS);",
                 'if (const char* e = std::getenv("KA_CHAIN_SUBBLOCKS")) n = std::max(1, std::min(std::atoi(e), d.T));',
                 "return std::min(n, KA_MAX_CHAIN_BLOCKS);",
                 "const int nsub = chain_subblocks(d, blocks_in_solve, true);",
                 "if (e >= KA_MAX_BLOCKS || io.chains + nsub > KA_MAX_CHAIN_EVENTS) return KA_ERR_LIMIT;",
                 # sub_block
                 "b.t0 = (int)((int64_t)d.T * j / nsub);",
                 "b.t1 = (int)((int64_t)d.T * (j + 1) / nsub);",
                 # the staged per-slot calls cut the staged block as a one-block solve does, without overlap
                 "const int nsub = chain_subblocks(d, 1);"):
        assert line in cu, line


def test_layout_restatement_gives_the_plans_other_modules_pin():
    """The chain launches test_chain_subblocks pins, from the restatement."""
    def launches(T, Pt, env, host_io=False):
        K = pipeline_stages(T, T * Pt, env)
        b = bounds(T, K, host_io)
        return K, 2 * sum(chain_subblocks(b[k + 1] - b[k], K, True, env) for k in range(K))
    assert launches(10000, 128, {}) == (4, 32)                          # c3: 4 blocks of 2 500 topics, 4 sub-blocks each
    assert launches(4096, 64, {}) == (2, 16)
    assert launches(8192, 16, {}) == (1, 32) and launches(12000, 16, {}) == (1, 32)
    assert launches(301, 40, {"KA_CHAIN_SUBBLOCKS": "40"}) == (1, 32)
    assert launches(301, 200, {"KA_PIPELINE_STAGES": "5"}) == (5, 10)   # test_chain_variants pipe5-table
    # host buffers: 1:2:1 for three blocks, not thirds
    assert bounds(900, 3, True) == [0, 225, 675, 900] and bounds(900, 3, False) == [0, 300, 600, 900]
    assert bounds(900, 2, True) == bounds(900, 2, False) == [0, 450, 900]


def test_cases_reach_every_layout_they_name():
    """Each layout is what its id says: K blocks, blocks above 1 024 topics cut by the large-block rule, the override at 40,
    and the 128 sub-blocks of a full solve."""
    byid = {lay["id"]: lay for lay in LAYOUTS}
    for lid, K in (("K1", 1), ("K2", 2), ("K3", 3), ("K5", 5), ("K8", 8), ("default", 3), ("sub40", 2), ("cap128", 8)):
        for host_io in (False, True):
            assert Layout(byid[lid]["T"], byid[lid]["env"], host_io).K == K, lid
    d = Layout(6144, {}, False)
    assert d.b == [0, 2048, 4096, 6144] and d.nsub == [4, 4, 4]        # 8 // 3 == 2 sub-blocks before the large-block rule
    assert Layout(6144, {}, True).nsub == [3, 6, 3]
    assert Layout(700, byid["sub40"]["env"], False).nsub == [16, 16]
    assert Layout(1200, byid["cap128"]["env"], False).chain_launches() == 2 * MAX_CHAIN_EVENTS
    assert Layout(1200, byid["cap128"]["env"], True).chain_launches() == 2 * MAX_CHAIN_EVENTS
    # every block boundary is a position of some case, on both kinds of bounds
    for lay in LAYOUTS:
        for host_io in (False, True):
            L = Layout(lay["T"], lay["env"], host_io)
            pos = set(L.positions().values())
            assert all(L.b[k] in pos and L.b[k + 1] - 1 in pos for k in range(L.K)), lay["id"]


# ---- CPU: donors, hosts and the splice rule -----------------------------------------------------------------------------------

def test_donors_fail_alone():
    d = donors()
    st = {name: alone(name) for name in d}
    assert st["unassignable-flat"][0] == 4 and 0 < st["unassignable-flat"][2] < P - 1
    assert st["unassignable-racked"][0] == 4 and 0 < st["unassignable-racked"][2] < P - 1
    # several partitions cannot be served: the first one is neither the topic's first nor its last
    assert st["cannot-serve"] == (4, 0, 36, 0, 0)
    # Math.abs(Integer.MIN_VALUE) % 48 == -(2^31 % 48) == -32: index -32 into an array of 48
    assert kab.synth.java_string_hash_ascii([util.MIN_HASH])[0] == INT_MIN
    assert st["hash-index"] == (5, 0, -1, -32, 48)
    # the hash-index donor's lists solve under any other hash
    _, _, ok = _dense_status("flat", [12345], d["hash-index"].cur[None])
    assert ok[0] == 0
    # the same topic through the structure-faithful oracle (ragged form, rack names)
    for name, dn in d.items():
        ids, rack_names, _ = _table(dn.table)
        part_off = np.array([0, P], dtype=np.int64)
        rep_off = np.arange(P + 1, dtype=np.int64) * RF
        _, _, _, o = ol.run(ol.OracleContext(), [dn.topic], part_off, np.arange(P, dtype=np.int32), rep_off, dn.cur.reshape(-1),
                            ids, rack_names, -1, RF, raise_on_error=False)
        assert (o.code, o.topic_index, o.partition, o.a, o.b) == st[name], name


@pytest.mark.parametrize("table", ["flat", "racked"])
def test_hosts_solve(table):
    h = host(table)
    ids, _, racks = _table(table)
    assert np.array_equal(h.broker_id, ids) and np.array_equal(h.rack_index, racks)
    out, ln, st = _dense_status(table, h.topic_hash, h.cur)
    assert st[0] == 0
    moved = (out.reshape(h.T, P, RF) != h.cur).any(axis=(1, 2)).sum()
    assert moved > h.T // 10   # the hosts do real work: many topics get new lists


@pytest.mark.parametrize("case", [c for c in DENSE_CASES if c["entry"] in ("host", "device")],
                         ids=lambda c: c["id"].rsplit("-", 1)[0] + ("-hostbounds" if c["entry"] == "host" else "-devicebounds"))
def test_spliced_cluster_fails_at_its_lowest_donor(case):
    assert expected(case["table"], case["layout"]["T"], case["placed"]) == splice_rule(case["placed"])


# ---- GPU helpers --------------------------------------------------------------------------------------------------------------

class layout_env:
    """The process environment of a layout: its variables set, the other layout variables unset."""

    def __init__(self, env):
        self.env = env

    def __enter__(self):
        self.patch = mock.patch.dict(os.environ, self.env)
        self.patch.__enter__()
        for k in ENV_KEYS:
            if k not in self.env:
                os.environ.pop(k, None)

    def __exit__(self, *exc):
        return self.patch.__exit__(*exc)


@pytest.fixture(scope="module")
def solvers(native_lib):
    """One Solver per table, reset by every test that takes it."""
    out = {}
    for table in ("flat", "racked"):
        ids, _, racks = _table(table)
        s = kab.Solver(0)
        s.set_brokers(ids, racks)
        out[table] = s
    yield out
    for s in out.values():
        s.close()


def run_dense(s, entry, names, th, cur, json_cap=None):
    """One dense solve through `entry`; returns the status fields (and for the JSON entries checks *json_bytes == 0)."""
    import torch
    T = len(th)
    if entry == "host":
        _, _, st = s.solve_dense(th, cur, check=False)
        return util.fields(st)
    if entry in ("json", "json-small"):
        buf = np.empty(4096, dtype=np.uint8) if entry == "json-small" else None
        text, st = s.solve_dense_json(names, th, cur, json_buf=buf, check=False)
        assert len(text) == 0, "a failed JSON solve left %d bytes" % len(text)
        return util.fields(st)
    d_hash, d_cur = torch.from_numpy(np.ascontiguousarray(th)).cuda(), torch.from_numpy(np.ascontiguousarray(cur)).cuda()
    d_out = torch.full((T, P, RF), -7, dtype=torch.int32, device="cuda")
    d_len = torch.full((T, P), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    if entry == "device":
        st = s.solve_dense_device(T, d_hash.data_ptr(), P, RF, d_cur.data_ptr(), -1, RF, d_len.data_ptr(), d_out.data_ptr())
    else:
        assert s.solve_dense_device(T, d_hash.data_ptr(), P, RF, d_cur.data_ptr(), -1, RF, d_len.data_ptr(), d_out.data_ptr(),
                                    sync=False) is None
        st = s.last_status()
    torch.cuda.synchronize()
    return util.fields(st)


# ---- GPU: dense single solves -------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("case", DENSE_CASES, ids=[c["id"] for c in DENSE_CASES])
def test_dense_solve_reports_the_lowest_failing_topic(solvers, case):
    lay = case["layout"]
    s = solvers[case["table"]]
    s.reset()
    names, th, cur = spliced(case["table"], lay["T"], dict(case["placed"]))
    with layout_env(lay["env"]):
        got = run_dense(s, case["entry"], names, th, cur)
    assert s.last_order_plan()[6] == Layout(lay["T"], lay["env"], ENTRIES[case["entry"]]).chain_launches()
    assert got == expected(case["table"], lay["T"], case["placed"])


# ---- ragged solves: sparse negative partition ids, donors at the edges of a JSON fragment -------------------------------------

def _ragged_donors():
    """The ragged-only failures, on the flat table: an RF mismatch inside the topic (KTA:58-60; ordinals 17 and 30 are one
    replica short), a topic whose lists are all empty (KTA:65-66), and the flat UNASSIGNABLE donor. (lists, part_id)."""
    base = _structured(5)
    mism = [list(base[p]) if p not in (17, 30) else list(base[p][:2]) for p in range(P)]
    return {"rf-mismatch": mism, "rf-not-positive": [[] for _ in range(P)],
            "unassignable-flat": [list(x) for x in donors()["unassignable-flat"].cur]}


def _part_ids(t, n):
    """Sparse ascending partition ids of topic t, starting below zero."""
    return (-20 - (t % 7) + np.cumsum(2 + (np.arange(n) * 7 + t) % 5)).astype(np.int32)


RAGGED_T = 5560   # a 16-row topic, then host topics of 48 rows: rows 2^18 - 48 .. 2^18 + 48 are topics 5461 and 5462
RAGGED_POS = {"t0": 0, "frag0last": 5461, "frag1first": 5462, "last": RAGGED_T - 1}


@functools.lru_cache(maxsize=None)
def ragged_case(pos, donor):
    """(names, topic_hash, part_off, part_id, rep_off, cur) of the flat host as a ragged run with a donor at topic pos."""
    h = host("flat")
    lists, names, th = [], [], []
    for t in range(RAGGED_T):
        if t == pos:   # the name keeps its hash: the oracle hashes the names
            lists.append(_ragged_donors()[donor])
            names.append(donors()[donor].topic if donor in donors() else "ragged.%s" % donor)
            th.append(kab.synth.java_string_hash_ascii(names[-1:])[0])
            continue
        rows = _structured(t)[:16] if t == 0 else h.cur[t]
        lists.append([list(x) for x in rows])
        names.append(h.topic_names[t])
        th.append(h.topic_hash[t])
    sizes = [len(x) for x in lists]
    part_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    part_id = np.concatenate([_part_ids(t, n) for t, n in enumerate(sizes)])
    flat = [r for x in lists for r in x]
    rep_off = np.concatenate([[0], np.cumsum([len(r) for r in flat])]).astype(np.int64)
    cur = np.array([b for r in flat for b in r], dtype=np.int32)
    return names, np.array(th, dtype=np.int32), part_off, part_id, rep_off, cur


@functools.lru_cache(maxsize=None)
def ragged_expected(pos, donor):
    names, th, part_off, part_id, rep_off, cur = ragged_case(pos, donor)
    ids, rack_names, _ = _table("flat")
    _, _, _, st = ol.run(ol.OracleContext(), names, part_off, part_id, rep_off, cur, ids, rack_names, -1, RF, raise_on_error=False)
    return st.code, st.topic_index, st.partition, st.a, st.b


RAGGED_CASES = [(p, d) for p in RAGGED_POS for d in ("rf-mismatch", "rf-not-positive", "unassignable-flat")]


def test_ragged_layout_puts_the_donors_at_the_fragment_edges():
    for pname, pos in RAGGED_POS.items():
        _, _, part_off, part_id, _, _ = ragged_case(pos, "rf-mismatch")
        assert part_off[-1] > JSON_FRAG_ROWS
        if pname == "frag0last":
            assert part_off[pos + 1] == JSON_FRAG_ROWS
        if pname == "frag1first":
            assert part_off[pos] == JSON_FRAG_ROWS
        assert (part_id < 0).any() and all(np.all(np.diff(part_id[part_off[t]:part_off[t + 1]]) > 1) for t in (0, pos))


@pytest.mark.parametrize("pos,donor", RAGGED_CASES, ids=["%s-%s" % (p, d) for p, d in RAGGED_CASES])
def test_ragged_donors_fail_at_their_own_topic(pos, donor):
    """The splice rule in the ragged layout, with the partition mapped through part_id."""
    t = RAGGED_POS[pos]
    _, _, part_off, part_id, _, _ = ragged_case(t, donor)
    ordinal = {"rf-mismatch": 17, "rf-not-positive": None, "unassignable-flat": alone("unassignable-flat")[2]}[donor]
    part = -1 if ordinal is None else int(part_id[part_off[t] + ordinal])
    code, a = {"rf-mismatch": (1, 2), "rf-not-positive": (2, 0), "unassignable-flat": (4, 0)}[donor]
    assert ragged_expected(t, donor) == (code, t, part, a, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["solve", "json"])
@pytest.mark.parametrize("pos,donor", RAGGED_CASES, ids=["%s-%s" % (p, d) for p, d in RAGGED_CASES])
def test_ragged_solve_reports_the_failing_partition_id(solvers, pos, donor, entry):
    t = RAGGED_POS[pos]
    names, th, part_off, part_id, rep_off, cur = ragged_case(t, donor)
    s = solvers["flat"]
    s.reset()
    with layout_env({}):
        if entry == "solve":
            _, _, st = s.solve_ragged(th, part_off, part_id, rep_off, cur, -1, RF, check=False)
        else:
            text, st = s.solve_ragged_json(names, th, part_off, part_id, rep_off, cur, -1, check=False)
            assert len(text) == 0
    assert s.last_order_plan()[6] == 2    # one block, one chain sub-block
    assert util.fields(st) == ragged_expected(t, donor)


# RF_GT_BROKERS needs a table smaller than a list: two brokers, lists of one or two, a donor with lists of three
TINY_T = 40


def _tiny(pos):
    """TINY_T topics on brokers 1 and 2 (topic t: 24 partitions with lists of 1 + t % 2), the one at pos with lists of 3."""
    topics = []
    for t in range(TINY_T):
        if t == pos:
            topics.append(("tiny.donor", {-3 + 4 * p: [1 + p % 2, 2 - p % 2, 7] for p in range(5)}))
        else:
            topics.append(("tiny.%d" % t, {-9 + 3 * p: [1 + (p + t) % 2, 2 - (p + t) % 2][:1 + t % 2] for p in range(24)}))
    return topics


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["solve", "json"])
@pytest.mark.parametrize("pos", [0, TINY_T // 2, TINY_T - 1], ids=["t0", "middle", "last"])
def test_ragged_rf_above_the_table(native_lib, pos, entry):
    topics = _tiny(pos)
    case = dict(topics=topics, brokers=[1, 2], racks={}, desired_rf=-1)
    res = util.run_oracle_case(ol, case)
    exp = res["error"]
    assert (exp["kind"], res["topic_index"], exp["partition"], exp["a"], exp["b"]) == (3, pos, -1, 3, 0)
    names, part_off, part_id, rep_off, cur = util.flatten(topics)
    th = np.array([kab.java_string_hash(n) for n in names], dtype=np.int32)
    s = kab.Solver(0)
    s.set_brokers(np.array([1, 2], dtype=np.int32), np.array([0, 1], dtype=np.int32))
    if entry == "solve":
        _, _, st = s.solve_ragged(th, part_off, part_id, rep_off, cur, -1, 3, check=False)
    else:
        text, st = s.solve_ragged_json(names, th, part_off, part_id, rep_off, cur, -1, check=False)
        assert len(text) == 0
    assert util.fields(st) == (exp["kind"], res["topic_index"], exp["partition"], exp["a"], exp["b"])


# ---- GPU: the staged per-slot calls, reported from topic_base ------------------------------------------------------------------

STAGED_T, TOPIC_BASE = 900, 1000
STAGED_NSUB = chain_subblocks(STAGED_T, 1, False, {})
STAGED_POS = {"t0": 0, "s3first": sub_block(STAGED_T, 3, STAGED_NSUB)[0], "last": STAGED_T - 1}


@pytest.mark.gpu
@pytest.mark.parametrize("pos", list(STAGED_POS), ids=list(STAGED_POS))
@pytest.mark.parametrize("donor", ["unassignable-flat", "hash-index"])
def test_staged_slot_calls_report_from_topic_base(solvers, pos, donor):
    import torch
    t = STAGED_POS[pos]
    placed = ((t, donor),)
    _, th, cur = spliced("flat", STAGED_T, dict(placed))
    s = solvers["flat"]
    s.reset()
    d_hash, d_cur = torch.from_numpy(th).cuda(), torch.from_numpy(cur).cuda()
    d_out = torch.full((STAGED_T, P, RF), -7, dtype=torch.int32, device="cuda")
    d_len = torch.full((STAGED_T, P), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    s.set_topic_base(TOPIC_BASE)
    try:
        with layout_env({}):
            s.stage_dense_device(STAGED_T, d_hash.data_ptr(), P, RF, d_cur.data_ptr(), -1, RF)
            assert s.staged_slot_chains() == 2
            s.order_slot_device(0)
            s.order_slot_device(1)
            st = s.emit_device(d_len.data_ptr(), d_out.data_ptr())
    finally:
        s.set_topic_base(0)
    assert s.last_order_plan()[6] == 2 * STAGED_NSUB
    code, ti, part, a, b = expected("flat", STAGED_T, placed)
    assert util.fields(st) == (code, TOPIC_BASE + ti, part, a, b)


# ---- GPU: the CLI, through the C++ mirror --------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_cli_prints_the_exception_of_the_lowest_failing_topic(native_lib, tmp_path):
    cli = kab.build_mod.build_host()
    T, t = 300, 157
    names, th, cur = spliced("flat", T, {t: "unassignable-flat"})
    ids, _, _ = _table("flat")
    brokers = [dict(id=int(b), host="h%d" % b, port=9092) for b in ids]
    parts = [dict(topic=names[i], partition=p, replicas=[int(x) for x in cur[i, p]]) for i in range(T) for p in range(P)]
    path = tmp_path / "cluster.json"
    path.write_text(json.dumps(dict(brokers=brokers, topics=names, partitions=parts)))
    exp = expected("flat", T, ((t, "unassignable-flat"),))
    assert exp[:2] == (4, t)
    r = subprocess.run([cli, "--zk_string", str(path), "--mode", "PRINT_REASSIGNMENT", "--disable_rack_awareness"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "NEW ASSIGNMENT" not in r.stdout
    assert "java.lang.IllegalStateException: Partition %d could not be fully assigned!" % exp[2] in r.stderr, r.stderr[-2000:]


# ---- GPU: what a Context holds after a failure -------------------------------------------------------------------------------

AFTER = dict(T=900, env={"KA_PIPELINE_STAGES": "3"})


def _failing(t, T=AFTER["T"], donor="unassignable-flat"):
    return spliced("flat", T, {t: donor}), expected("flat", T, ((t, donor),))


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "device"])
def test_reset_after_a_failure_gives_the_oracles_rows_and_counters(solvers, entry):
    import torch
    s = solvers["flat"]
    s.reset()
    (names, th, cur), exp = _failing(700)
    h = host("flat")
    T = AFTER["T"]
    with layout_env(AFTER["env"]):
        assert run_dense(s, entry, names, th, cur) == exp
        s.reset()
        if entry == "host":
            out, ln, st = s.solve_dense(h.topic_hash[:T], h.cur[:T], check=False)
        else:
            d_hash, d_cur = torch.from_numpy(h.topic_hash[:T].copy()).cuda(), torch.from_numpy(h.cur[:T].copy()).cuda()
            d_out = torch.full((T, P, RF), -7, dtype=torch.int32, device="cuda")
            d_len = torch.full((T, P), -7, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            st = s.solve_dense_device(T, d_hash.data_ptr(), P, RF, d_cur.data_ptr(), -1, RF, d_len.data_ptr(), d_out.data_ptr())
            out, ln = d_out.cpu().numpy(), d_len.cpu().numpy()
    e_out, e_len, e_st = _dense_status("flat", h.topic_hash[:T], h.cur[:T])
    assert st.code == 0 == e_st[0]
    assert np.array_equal(out.reshape(-1, RF), e_out) and np.array_equal(ln.reshape(-1), e_len)
    assert np.array_equal(s.counters()[:, :RF], models.histogram(h.broker_id, e_out, e_len)[:, :RF])


@pytest.mark.gpu
def test_set_counters_after_a_failure_starts_the_next_solve_from_them(solvers):
    s = solvers["flat"]
    s.reset()
    (names, th, cur), exp = _failing(450)
    h = host("flat")
    T = AFTER["T"]
    with layout_env(AFTER["env"]):
        assert run_dense(s, "host", names, th, cur) == exp
        ctr = np.random.default_rng(0xC7).integers(0, 5000, size=s.counters().shape).astype(np.int32)
        s.set_counters(ctr)
        out, ln, st = s.solve_dense(h.topic_hash[:T], h.cur[:T], check=False)
    octx = ol.OracleContext()
    ids, rack_names, _ = _table("flat")
    for i, b in enumerate(ids):
        for r in range(ctr.shape[1]):
            octx.set_counter(int(b), r, int(ctr[i, r]))
    part_off, part_id, rep_off, flat = h.subset(0, T).ragged()
    o_len, _, o_out, o_st = ol.run(octx, h.topic_names[:T], part_off, part_id, rep_off, flat, ids, rack_names, -1, RF)
    assert st.code == 0 == o_st.code
    assert np.array_equal(out.reshape(-1, RF), o_out) and np.array_equal(ln.reshape(-1), o_len)
    got = s.counters()
    for i, b in enumerate(ids):
        for r in range(ctr.shape[1]):
            assert got[i, r] == octx.counter(int(b), r), (int(b), r)


@pytest.mark.gpu
def test_async_status_after_failures(solvers):
    """A failing asynchronous call, a good one (its status is OK), then a failing call with fewer topics at a higher index than
    the first failure: it reports its own topic, not one left from the larger call."""
    s = solvers["flat"]
    s.reset()
    h = host("flat")
    with layout_env({"KA_PIPELINE_STAGES": "8"}):
        (names, th, cur), exp = _failing(100, T=1200)
        assert run_dense(s, "async", names, th, cur) == exp and exp[1] == 100
        st = run_dense(s, "async", h.topic_names[:1200], h.topic_hash[:1200], h.cur[:1200])
        assert st == (0, -1, -1, 0, 0)
        assert util.fields(s.last_status()) == st
        (names, th, cur), exp = _failing(100, T=1200)
        assert run_dense(s, "async", names, th, cur) == exp
        (names, th, cur), exp = _failing(250, T=300, donor="hash-index")
        assert exp[:2] == (5, 250)
        assert run_dense(s, "async", names, th, cur) == exp
        (names, th, cur), exp = _failing(30, T=1200)
        assert run_dense(s, "device", names, th, cur) == exp
        (names, th, cur), exp = _failing(290, T=300)
        assert run_dense(s, "host", names, th, cur) == exp


@pytest.mark.gpu
@pytest.mark.parametrize("pos,donor", [("frag1first", "unassignable-flat"), ("last", "rf-mismatch")])
def test_json_leaves_the_counters_of_the_plain_solve(native_lib, pos, donor):
    """kassign.h: on any error *st is what ka_solve reports and the ctx counters afterwards equal those after ka_solve."""
    t = RAGGED_POS[pos]
    names, th, part_off, part_id, rep_off, cur = ragged_case(t, donor)
    ids, _, racks = _table("flat")
    got = []
    for entry in ("solve", "json"):
        s = kab.Solver(0)
        s.set_brokers(ids, racks)
        if entry == "solve":
            _, _, st = s.solve_ragged(th, part_off, part_id, rep_off, cur, -1, RF, check=False)
        else:
            text, st = s.solve_ragged_json(names, th, part_off, part_id, rep_off, cur, -1, check=False)
            assert len(text) == 0
        got.append((util.fields(st), s.counters()))
        s.close()
    assert got[0][0] == got[1][0] == ragged_expected(t, donor)
    assert np.array_equal(got[0][1], got[1][1])
