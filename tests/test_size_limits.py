"""The wave and text passes at their size limits, each checked exactly against the models the suite already has:

- the wave chain's claim-key reset after 2^21 rounds, in all four chain instances (state in shared or global memory, with or
  without a sender), on plans of about 2.1 M rows;
- the radix passes of the wave documents over tiles of more than 2 048 rows (more than 2 048 x 1 024 rows in a call);
- wave documents whose text passes 2^32 bytes (64-bit document offsets);
- the 32-bit fragment limit of ka_solve_json and ka_solve_clusters_json, on both sides.

`models.chain_rounds` restates the chain's round rule (kassign_waves.cuh). The device does not report its rounds, so this model is
the evidence that a plan reaches the reset. The plans that cross it run in a child process with a timeout: a chain that stopped
finishing would fail its test and go away with the process."""
import re

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SEND_SUMMARY_DTYPE, WAVE_SUMMARY_DTYPE
from tests import models, util
from tests.util import Member

LIMIT = _native.KA_ERR_LIMIT
CHUNK, RESET = models.WAVE_CHUNK, models.WAVE_RESET
UINT32_MAX = (1 << 32) - 1


# ---- CPU: the round model ------------------------------------------------------------------------------------------------

def _claims(records, senders=None):
    """The chain's mechanism, round by round (without the reset): every pending record of a chunk claims its brokers with the
    key (round, the earlier slot wins), and a record that holds all its claims decides. Claims stay across chunks."""
    rounds = np.zeros(len(records), dtype=np.int64)
    rows = [g for g, r in enumerate(records) if r]
    rnd = 0
    claim = {}
    for c0 in range(0, len(rows), CHUNK):
        pend = list(enumerate(rows[c0:c0 + CHUNK]))   # (slot, row)
        while pend:
            rnd += 1
            for slot, g in pend:
                for k in models.chain_keys(records, senders, g):
                    claim[k] = max(claim.get(k, (0, 0)), (rnd, -slot))
            won = {g for slot, g in pend if all(claim[k] == (rnd, -slot) for k in models.chain_keys(records, senders, g))}
            for g in won:
                rounds[g] = rnd
            pend = [(slot, g) for slot, g in pend if g not in won]
    return rounds


def test_a_fully_serial_chunk_takes_2048_rounds():
    rounds = models.chain_rounds([[7]] * (CHUNK + 3))
    assert rounds.tolist() == list(range(1, CHUNK + 4))
    # a sender alone makes records serial, as a shared receiver does
    rounds = models.chain_rounds([[100 + g] for g in range(CHUNK + 1)], [1] * (CHUNK + 1))
    assert rounds.tolist() == list(range(1, CHUNK + 2))
    # without a send table the sender is no link
    assert models.chain_rounds([[100 + g] for g in range(CHUNK + 1)]).tolist() == [1] * CHUNK + [2]


def test_a_chunk_of_independent_records_takes_one_round():
    rounds = models.chain_rounds([[g, g + 50000] for g in range(3 * CHUNK)])
    assert rounds.tolist() == [1] * CHUNK + [2] * CHUNK + [3] * CHUNK
    assert models.chain_rounds([[g] for g in range(10)], [None] * 10).tolist() == [1] * 10


def test_a_path_is_serial():
    L = CHUNK + 1
    records = [[1 + i % L, 1 + (i + 1) % L] for i in range(2 * CHUNK + 5)]
    assert models.chain_rounds(records).tolist() == list(range(1, 2 * CHUNK + 6))
    # two interleaved paths (record i receives i and i + 2) are two chains: half the rounds
    assert models.chain_rounds([[i, i + 2] for i in range(CHUNK)]).tolist() == [1 + i // 2 for i in range(CHUNK)]


def test_unchanged_and_receiverless_rows_are_not_records():
    cur_lists = [[1], [1, 2], [1, 2], [1, 2], [3], [], [4]]
    new_lists = [[2], [1, 2], [2, 1], [1], [2], [], [4, 2]]
    rcv, snd = models.wave_records(*util.cur_lists(cur_lists), *util.rows(new_lists))
    assert rcv == [[2], [], [], [], [2], [], [2]] and snd == [1, 1, 1, 1, 3, None, 4]
    assert models.chain_rounds(rcv).tolist() == [1, 0, 0, 0, 2, 0, 3]
    # rows that are no record take no slot of a chunk: 2 047 serial records, 500 other rows, then the chunk's last record
    cur_lists = [[1]] * (CHUNK - 1) + [[1, 2]] * 500 + [[1], [1]]
    new_lists = [[2]] * (CHUNK - 1) + [[2, 1] if g % 2 else [1, 2] for g in range(500)] + [[2], [2]]
    rcv, _ = models.wave_records(*util.cur_lists(cur_lists), *util.rows(new_lists))
    rounds = models.chain_rounds(rcv)
    assert rounds[CHUNK - 1:CHUNK + 499].tolist() == [0] * 500
    assert rounds[-2:].tolist() == [CHUNK, CHUNK + 1]


@pytest.mark.parametrize("seed", range(4))
def test_the_rule_is_the_claims_mechanism(seed):
    """chain_rounds' closed rule equals the rounds of the claim protocol it summarises, on random records with hot brokers."""
    rng = np.random.default_rng(seed)
    n = 2 * CHUNK + 300
    records = [[int(x) for x in rng.choice(np.arange(1, 400) if g % 5 else np.arange(1, 21), int(rng.integers(0, 4)), replace=False)]
               for g in range(n)]
    senders = [None if rng.random() < 0.2 else int(rng.integers(1, 60)) for _ in range(n)]
    for s in (None, senders):
        assert np.array_equal(models.chain_rounds(records, s), _claims(records, s))


# ---- GPU: plans that cross round 2^21, and their documents ---------------------------------------------------------------

def reset_input(send, seed=5):
    """A plan whose chain crosses round 2^21 in a chunk of mixed rows. A serial prefix costs 1 023 chunks of 2 048 rounds and
    1 987 more: without a sender, record i receives b_(i mod 2 053) and b_(i + 1 mod 2 053) (two records per broker, so little
    contention on a claim word); with one, every record is led by broker 1 and receives one of 2 049 brokers in turn. A row of
    the prefix weighs the budget, so its waves are 1, 2, 3, ... Then a tail of random rows on other brokers: four hot receivers
    (and, with a sender, four hot leaders), random weights, unchanged rows and rows without receivers. Its first records fill
    the prefix's last chunk; the next chunk starts 60 rounds before the reset and runs past it. Returns a dict of the inputs."""
    rng = np.random.default_rng(seed)
    n_pre = 1023 * CHUNK + CHUNK - 1 - 60
    i = np.arange(n_pre)
    if send:
        B, C, NB = 9, 5, 6400
        pre_cur = np.ones(n_pre, dtype=np.int32)
        pre_new = np.stack([np.ones(n_pre, dtype=np.int64), 2 + i % 2049, np.full(n_pre, -1)], axis=1)
        pre_len, pre_rep, first_free = np.full(n_pre, 2), 1, 2051
    else:
        B, C, NB = 7, None, 12800
        pre_cur = np.zeros(0, dtype=np.int32)
        pre_new = np.stack([1 + i % 2053, 1 + (i + 1) % 2053, np.full(n_pre, -1)], axis=1)
        pre_len, pre_rep, first_free = np.full(n_pre, 2), 0, 2054
    pool = np.arange(first_free, NB + 1)
    hot, leaders = pool[:4], pool[4:8]
    cur_lists, new_lists = [], []
    for g in range(40000):
        c = [int(x) for x in rng.choice(pool, int(rng.integers(0, 4)), replace=False)]
        if send and c and rng.random() < 0.3:
            c[0] = int(rng.choice(leaders[~np.isin(leaders, c)]))
        u = rng.random()
        if u < 0.2:
            new = list(c)                                   # unchanged
        elif u < 0.3:
            new = c[1:] + c[:1]                             # a reorder or a drop: no receiver
        else:
            new = c[:1]
            while len(new) < 1 + int(rng.integers(1, 3)):
                b = int(rng.choice(hot)) if len(new) == 1 and rng.random() < 0.5 else int(rng.choice(pool))
                if b not in new and b not in c:
                    new.append(b)
        cur_lists.append(c)
        new_lists.append(new)
    t_off, t_cur = util.cur_lists(cur_lists)
    t_out, t_len = util.rows(new_lists, 3)
    bound = C if send else B
    weight = np.concatenate([np.full(n_pre, bound), rng.integers(0, 2 * bound + 1, len(t_len))]).astype(np.int64)
    rep_off = np.concatenate([np.arange(n_pre + 1, dtype=np.int64) * pre_rep, n_pre * pre_rep + t_off[1:]])
    Q = len(weight)
    part_off = np.concatenate([[0], np.sort(rng.choice(np.arange(1, Q), 999, replace=False)), [Q]]).astype(np.int64)
    ids, racks = util.table(np.arange(1, NB + 1), 8)
    inp = dict(rep_off=rep_off, cur=np.concatenate([pre_cur, t_cur]).astype(np.int32),
               out=np.concatenate([pre_new, t_out]).astype(np.int32), out_len=np.concatenate([pre_len, t_len]).astype(np.int32),
               weight=weight, B=np.int64(B), part_off=part_off, names=np.array(["reset.%d" % t for t in range(1000)]),
               ids=ids, racks=racks)
    if send:   # N + n_send: 12 800 words of chain state in shared memory, 12 801 in global memory
        inp.update(C=np.int64(C), send_smem=np.arange(1, NB + 1, dtype=np.int32), send_global=np.arange(1, NB + 2, dtype=np.int32))
    else:
        gids, gracks = util.table(np.arange(1, NB + 2), 8)
        inp.update(ids_global=gids, racks_global=gracks)
    return inp


# Run in a child process (util.run_child): both plans (chain state in shared and in global memory) and the documents, written
# back to the directory given.
_CHILD = r"""
import sys
import time
import numpy as np
import kafka_assigner_b200 as kab
d = sys.argv[1]
a = dict(np.load(d + "/in.npz"))
send = "C" in a
rows = (a["rep_off"], a["cur"], a["out"], a["out_len"], int(a["B"]))
res = {}
for tag in ("smem", "global"):
    s = kab.Solver(0)
    s.set_brokers(a["ids_global"] if tag == "global" and not send else a["ids"], a["racks_global"] if tag == "global" and not send else a["racks"])
    kw = dict(max_broker_out=int(a["C"]), send_brokers=a["send_" + tag]) if send else {}
    t = time.perf_counter()
    wave, summ, st = s.plan_waves(*rows, weight=a["weight"], **kw)
    print("%s plan_waves %.2f s" % (tag, time.perf_counter() - t))
    res[tag + "_wave"], res[tag + "_summary"], res[tag + "_status"] = wave, summ, np.array([st.code, st.a, st.b])
    if tag == "smem":
        t = time.perf_counter()
        docs, wave, summ, st = s.plan_waves_json(list(a["names"]), a["part_off"], None, *rows, weight=a["weight"], **kw)
        print("plan_waves_json %.2f s" % (time.perf_counter() - t))
        base = docs[0].__array_interface__["data"][0] if docs else 0
        off = np.array([x.__array_interface__["data"][0] - base for x in docs] + [0], dtype=np.int64)
        off[-1] = off[-2] + len(docs[-1]) if docs else 0
        res.update(json_wave=wave, json_summary=summ, json_status=np.array([st.code, st.a, st.b]), json_off=off,
                   json_text=docs[0].base[:off[-1]] if docs else np.zeros(0, np.uint8))
np.savez(d + "/out.npz", **res)
"""
CHILD_TIMEOUT = 300   # seconds: about five times what the child takes on an H100


@pytest.fixture(scope="module", params=["receive", "send"])
def reset_plans(request, tmp_path_factory, native_lib):
    """The device's plans and documents for reset_input (from the child) with the models of the same input, each computed once:
    (input, device results, model docs, model waves, model summaries, chain rounds, records, senders)."""
    send = request.param == "send"
    d = tmp_path_factory.mktemp(request.param)
    inp = reset_input(send)
    np.savez(d / "in.npz", **inp)
    args = (inp["rep_off"], inp["cur"], inp["out"], inp["out_len"])

    def expected():   # the models, while the device plans
        records, senders = models.wave_records(*args)
        rounds = models.chain_rounds(records, senders if send else None)
        names, part_off = list(inp["names"]), inp["part_off"]
        if send:
            e_docs, _, _, e_wave, e_summ, e_st = models.wave_documents(names, part_off, None, *args, inp["ids"], int(inp["B"]),
                                                                       inp["weight"], send=(inp["send_smem"], int(inp["C"])))
        else:
            e_docs, _, _, e_wave, e_summ, e_st = models.wave_documents(names, part_off, None, *args, inp["ids"], int(inp["B"]),
                                                                       inp["weight"])
        assert e_st == (0, 0, 0)
        e_summ = util.summary_array(e_summ, WAVE_SEND_SUMMARY_DTYPE if send else WAVE_SUMMARY_DTYPE)
        return records, senders, rounds, e_docs, e_wave, e_summ

    (records, senders, rounds, e_docs, e_wave, e_summ), out, secs = util.run_child(_CHILD, d, CHILD_TIMEOUT, expected,
                                                                                   "the plans of " + request.param)
    print("%s: child and models %.1f s\n%s" % (request.param, secs, out))
    dev = dict(np.load(d / "out.npz"))
    return inp, dev, e_docs, e_wave, e_summ, rounds, records, senders if send else None


@pytest.mark.gpu
def test_plans_cross_round_2_21(reset_plans):
    """All four chain instances: every wave, W and summary field of both state placements equal the model, and the chain really
    crossed round 2^21 inside a chunk, with records of that chunk on both sides of the reset and brokers they share across it."""
    inp, dev, _, e_wave, e_summ, rounds, records, senders = reset_plans
    before, after, shared, later = models.crossing_chunk(records, senders, rounds)
    assert before >= 300 and after >= 300 and shared >= 4 and later >= 5, (before, after, shared, later)
    assert int(rounds.max()) > RESET
    W = len(e_summ)
    assert W > kab.Solver.WAVE_SUMMARY_CAP   # plan_waves makes its second call for the rest of the summaries
    for tag in ("smem", "global"):
        assert dev[tag + "_status"].tolist() == [0, 0, 0]
        assert np.array_equal(dev[tag + "_wave"], e_wave), (tag, np.nonzero(dev[tag + "_wave"] != e_wave)[0][:10])
        assert len(dev[tag + "_summary"]) == W
        for f in e_summ.dtype.names:
            assert np.array_equal(dev[tag + "_summary"][f], e_summ[f]), (tag, f)


@pytest.mark.gpu
def test_documents_of_more_than_2_21_rows(reset_plans):
    """ka_plan_waves_json / ka_plan_waves_send_json on the same plans: Q > 2 048 x 1 024, so every radix pass takes tiles of
    more than 2 048 rows, and W > 65 535, so there are three passes. Every document byte for byte."""
    inp, dev, e_docs, e_wave, e_summ, _, _, _ = reset_plans
    assert len(inp["out_len"]) > 2048 * 1024 and len(e_docs) > 65535
    assert dev["json_status"].tolist() == [0, 0, 0]
    assert np.array_equal(dev["json_wave"], e_wave) and np.array_equal(dev["json_summary"], dev["smem_summary"])
    e_off = np.concatenate([[0], np.cumsum([len(x) for x in e_docs])])
    assert np.array_equal(dev["json_off"], e_off)
    assert dev["json_text"].tobytes() == b"".join(e_docs)


def _compare_docs(docs, e_docs):
    assert len(docs) == len(e_docs)
    assert [len(d) for d in docs] == [len(e) for e in e_docs]
    assert b"".join(bytes(d) for d in docs) == b"".join(e_docs)


@pytest.mark.gpu
def test_scattered_documents_over_large_tiles(native_lib):
    """2.5 M rows, 40 % of them moving one replica to one of 20 brokers with B = 1: about 50 000 waves (two radix passes) whose
    rows are scattered over the whole input. Every tile of a pass (2 560 rows) holds many digit values, and the first pass
    drops the 60 % of unchanged rows."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 61), 4))
    rng = np.random.default_rng(14)
    Q = 2_500_000
    first = rng.integers(0, 40, Q)
    cur = np.stack([first, (first + rng.integers(1, 40, Q)) % 40], axis=1) + 1
    out = cur.copy()
    moved = rng.random(Q) < 0.4
    out[moved, 1] = rng.integers(41, 61, int(moved.sum()))
    out, out_len = out.astype(np.int32), np.full(Q, 2, dtype=np.int32)
    rep_off, cur = np.arange(Q + 1, dtype=np.int64) * 2, cur.astype(np.int32).ravel()
    part_off = np.concatenate([[0], np.sort(rng.choice(np.arange(1, Q), 1999, replace=False)), [Q]]).astype(np.int64)
    names = ["scatter-%d" % t for t in range(2000)]
    assert Q > 2048 * 1024
    docs, wave, summ, st = s.plan_waves_json(names, part_off, None, rep_off, cur, out, out_len, 1)
    e_docs, _, _, e_wave, e_summ, e_st = models.wave_documents(names, part_off, None, rep_off, cur, out, out_len, s.broker_id, 1)
    assert st.code == 0 and e_st == (0, 0, 0) and 256 <= len(e_docs) <= 65535
    assert np.array_equal(wave, e_wave)
    e_summ = util.summary_array(e_summ, WAVE_SUMMARY_DTYPE)
    assert all(np.array_equal(summ[f], e_summ[f]) for f in WAVE_SUMMARY_DTYPE.names)
    _compare_docs(docs, e_docs)


# ---- GPU: text at and past 4 GiB ---------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_wave_documents_past_4_gib(native_lib):
    """ka_plan_waves_json with 68 000 rows in topics of names of about 64 KiB: the text passes 2^32 bytes, so the document
    offsets and the text positions of the CTAs beyond it need their 64 bits. Three short-named topics at the end keep CTAs on
    the staged store path past 2^32. Every document is compared on its own, against the model's documents printed with
    placeholder names that are then replaced by the real ones; the whole expected text is never built."""
    s = kab.Solver(0)
    s.set_brokers(*util.table(np.arange(1, 41), 4))
    rng = np.random.default_rng(15)
    lens = rng.integers(65000, 65537, 68)
    names = ["L%02d-" % t + "n" * (int(n) - 4) for t, n in enumerate(lens)] + ["s%d" % t for t in range(3)]
    part_off = np.concatenate([[0], np.cumsum([1000] * 68 + [800] * 3)]).astype(np.int64)
    Q = int(part_off[-1])
    # every row moves one replica to one of four brokers, B = 2: about eight rows per wave; one row in 50 is unchanged
    g = np.arange(Q)
    cur_lists = [[1, 2]] * Q
    new_lists = [[1, 2] if x % 50 == 0 else [1, 3 + x % 4] for x in g.tolist()]
    rep_off, cur = util.cur_lists(cur_lists)
    out, out_len = util.rows(new_lists, 2)
    ph = ["@%d@" % t for t in range(len(names))]
    e_docs, _, _, e_wave, e_summ, e_st = models.wave_documents(ph, part_off, None, rep_off, cur, out, out_len, s.broker_id, 2)
    assert e_st == (0, 0, 0)
    real = [n.encode() for n in names]
    topic = re.compile(rb'"topic":"@(\d+)@"')

    def expand(doc):
        return topic.sub(lambda m: b'"topic":"' + real[int(m.group(1))] + b'"', doc)

    slab, name_off = kab.Solver.marshal_names(names)
    cap = models.json_bound(names, part_off, 2)
    js = np.empty(cap, dtype=np.uint8)
    doc_off, wave = np.zeros(Q + 1, dtype=np.int64), np.zeros(Q, dtype=np.int32)
    summ = np.zeros(Q, dtype=WAVE_SUMMARY_DTYPE)
    rc, st, n = util.raw_plan_waves_json(s, len(names), part_off, None, rep_off, cur, 2, out_len, out, None, 2, slab, name_off, js,
                                         cap, doc_off, wave, summ, Q)
    W = n.value
    assert rc == 0 and W == len(e_docs) and np.array_equal(wave, e_wave) and [util.record_of(x, WAVE_SUMMARY_DTYPE.names) for x in summ[:W]] == e_summ
    assert doc_off[W] > 1 << 32
    at = 0
    straddle = 0
    for v, doc in enumerate(e_docs):
        e = expand(doc)
        assert int(doc_off[v]) == at, v
        assert js[at:at + len(e)].tobytes() == e, v
        straddle += at < 1 << 32 < at + len(e)
        at += len(e)
    assert int(doc_off[W]) == at and straddle == 1
    s.close()


def _fragment_cluster(Q, T, L, seed):
    """Q rows in T topics with names of L bytes, lists of 3 replicas, 11-character partition and broker ids (below
    -999 999 999, ascending): every record prints at exactly the bound's 50 + 12 x 3 + L bytes."""
    rng = np.random.default_rng(seed)
    N = 400
    ids = (-2_100_000_000 + 1000 * np.arange(N)).astype(np.int32)
    a = rng.integers(0, N, Q)
    picks = np.stack([a, (a + 1 + rng.integers(0, N // 2 - 1, Q)) % N, (a + N // 2 + rng.integers(0, N // 2 - 1, Q)) % N], axis=1)
    names = ["f%03d-" % t + "q" * (L - 5) for t in range(T)]
    return dict(names=names, th=np.array([kab.java_string_hash(n) for n in names], dtype=np.int32),
                part_off=(np.arange(T + 1, dtype=np.int64) * Q) // T, part_id=(-2_000_000_000 + 3 * np.arange(Q)).astype(np.int32),
                rep_off=np.arange(Q + 1, dtype=np.int64) * 3, cur=ids[picks].astype(np.int32).ravel(), ids=ids,
                racks=["k%d" % (i // 4) for i in range(N)])


def _l0(Q, S=3):
    """The longest name a Q-row fragment (Q <= 2^18) of stride S accepts: 64 + Q (50 + 12 S + L0) <= UINT32_MAX."""
    L0 = (UINT32_MAX - 64) // Q - (50 + 12 * S)
    assert 64 + Q * (50 + 12 * S + L0) <= UINT32_MAX < 64 + Q * (50 + 12 * S + L0 + 1)
    return L0


@pytest.mark.gpu
def test_solve_json_at_the_fragment_limit(native_lib, oracle):
    """ka_solve_json with Q = 2^18 rows, one fragment, stride 3: names of L0 bytes solve and print the oracle's text, ending
    within Q + 64 bytes of 2^32; one name of L0 + 1 is refused with KA_ERR_LIMIT, a = L0 + 1, before anything is solved."""
    Q, T = 1 << 18, 64
    L0 = _l0(Q)
    c = _fragment_cluster(Q, T, L0, 16)
    s = kab.Solver(0)
    s.set_brokers(*util.table(c["ids"], 4))
    args = (c["part_off"], c["part_id"], c["rep_off"], c["cur"], -1)
    text, st = s.solve_ragged_json(c["names"], c["th"], *args, check=False)
    assert st.code == 0
    n = len(text)
    assert n == Q * (50 + 12 * 3 + L0) - 1 + 15 + 14 and 0 < (1 << 32) - n <= Q + 64
    octx = oracle.OracleContext()
    o_len, o_pid, o_out, o_st = oracle.run(octx, c["names"], *args[:4], c["ids"], c["racks"], -1, 3, raise_on_error=False)
    assert o_st.code == 0 and (o_len == 3).all()
    at = 15
    assert text[:at].tobytes() == b'{"partitions":['
    for t in range(T):   # record by record, one topic's slice at a time
        a, b = int(c["part_off"][t]), int(c["part_off"][t + 1])
        e = ("," if t else "") + models.solve_document([c["names"][t]], [0, b - a], o_pid[a:b], o_out[a:b], o_len[a:b])[15:-14]
        assert text[at:at + len(e)].tobytes() == e.encode(), t
        at += len(e)
    assert text[at:].tobytes() == b'],"version":1}'
    ctr = s.counters()
    assert [[int(ctr[i, k]) for k in range(3)] for i in range(len(c["ids"]))] == [[octx.counter(int(b), k) for k in range(3)] for b in c["ids"]]
    del text
    # one name a byte longer: refused before anything is solved
    names = list(c["names"])
    names[T // 2] += "q"
    th = c["th"].copy()
    th[T // 2] = kab.java_string_hash(names[T // 2])
    text, st = s.solve_ragged_json(names, th, *args, check=False)
    assert (st.code, st.a) == (LIMIT, L0 + 1) and len(text) == 0
    assert np.array_equal(s.counters(), ctr)
    s.close()


@pytest.mark.gpu
def test_solve_clusters_json_applies_the_limit_per_cluster(native_lib, oracle):
    """Three clusters; the middle one (4 096 rows, stride 3) has one name of its own L0 + 1 bytes: it alone is refused with
    KA_ERR_LIMIT, a = that length, and an empty range; the other two equal their own ka_solve_json texts and the oracle's."""
    Q = 4096
    L0 = _l0(Q)
    mk = kab.synth.make_ragged_cluster
    c = _fragment_cluster(Q, 32, 20, 17)
    c["names"][0] = "f000-" + "q" * (L0 + 1 - 5)
    c["th"][0] = kab.java_string_hash(c["names"][0])
    middle = Member(util.table(c["ids"], 4), c["names"], c["th"], c["part_off"], c["part_id"], c["rep_off"], c["cur"])
    fleet = [Member.of(mk(T=60, N=40, R=5, max_partitions=64, seed=31)), middle, Member.of(mk(T=40, N=30, R=4, seed=32))]
    sts, texts = util.check_fleet(fleet, oracle)
    assert sts[1] == (LIMIT, -1, -1, L0 + 1, 0) and texts[1] == b""
    assert sts[0][0] == sts[2][0] == 0 and texts[0] and texts[2]
