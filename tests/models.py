"""The plain-Python models the device is checked against, each written once: the move summary, the wave rule (with and
without a sender budget), the wave chain's claim rounds, the reassignment JSON printers, the wave documents and their greedy cut, the schedule model's records,
slot chains and the expected counter histogram, and kernel A's shared-memory budget.
Each restates a rule of include/kassign.h. This module imports numpy and the status codes only: it never loads the library
or the oracle, so CPU tests, GPU tests and tests/tools can all use it."""
import numpy as np

from kafka_assigner_b200 import _native

BAD = _native.KA_ERR_BAD_ARG
SLOTS = 8            # counter slots per broker (ka_ctx_counter_slots)
INF = 0x7FFFFFFF     # the counter of the slot chains' dummy broker (index N): INT_MAX, never bumped


# ---- the move summary ----------------------------------------------------------------------------------------------------

def move_summary(out, out_len, rep_off, cur, ids, weight=None):
    """(summary dict, replicas, leaders, added) of one candidate's rows out [Q, S] / out_len [Q] against the current lists
    cur[rep_off[g] .. rep_off[g + 1]), for the broker table `ids`. Position counts, as ka_move_summary defines them."""
    Q, S = out.shape
    m = np.diff(rep_off).astype(np.int64)
    n = out_len.astype(np.int64)
    w = np.ones(Q, dtype=np.int64) if weight is None else np.asarray(weight, dtype=np.int64)
    pos = np.arange(S)
    cmask, nmask = pos < m[:, None], pos < n[:, None]
    cb = np.zeros((Q, S), dtype=np.int64)
    cb[cmask] = cur[(rep_off[:-1, None] + pos)[cmask]]
    nb = np.where(nmask, out, 0).astype(np.int64)
    eq = nb[:, :, None] == cb[:, None, :]                       # [g, new position, current position]
    added_pos = nmask & ~(eq & cmask[:, None, :]).any(2)
    dropped_pos = cmask & ~(eq & nmask[:, :, None]).any(1)
    n_add, n_drop = added_pos.sum(1), dropped_pos.sum(1)
    changed = (n != m) | (nmask & cmask & (nb != cb)).any(1)
    leader = (m == 0) | (n == 0) | (nb[:, 0] != cb[:, 0])
    idx = np.searchsorted(ids, nb)
    assert np.all(ids[idx[nmask]] == nb[nmask]), "a row holds a broker outside the table"
    wq = np.broadcast_to(w[:, None], (Q, S))
    rep, lead, inb = (np.zeros(len(ids), dtype=np.int64) for _ in range(3))
    np.add.at(rep, idx[nmask], wq[nmask])
    np.add.at(lead, idx[n > 0, 0], w[n > 0])
    np.add.at(inb, idx[added_pos], wq[added_pos])
    s = dict(rows_changed=int(changed.sum()), rows_moved=int(((n_add + n_drop) > 0).sum()), leaders_changed=int(leader.sum()),
             replicas_added=int((w * n_add).sum()), replicas_dropped=int((w * n_drop).sum()))
    if len(ids):
        top = int(np.argmax(inb))   # the first maximum: the lowest id
        s.update(max_broker_in=int(inb[top]), max_broker_in_id=int(ids[top]) if inb[top] > 0 else -1,
                 max_broker_replicas=int(rep.max()), min_broker_replicas=int(rep.min()),
                 max_broker_leaders=int(lead.max()), min_broker_leaders=int(lead.min()))
    else:
        s.update(max_broker_in=0, max_broker_in_id=-1, max_broker_replicas=0, min_broker_replicas=0, max_broker_leaders=0,
                 min_broker_leaders=0)
    return s, rep, lead, inb


# ---- wave plans ----------------------------------------------------------------------------------------------------------

def plan_waves(rep_off, cur, out, out_len, ids, B, weight=None, send=None):
    """(wave [Q] int32, [summary dict per wave], (code, a, b)) of the wave rule, rows in input order.

    send=None is ka_plan_waves: no broker receives more than B per wave; the five ka_wave_summary fields. send=(send_ids, C) is
    ka_plan_waves_send: also no leader (the first broker of a row's current list) sends more than C per wave; the seven fields.
    The lowest failing row wins: a new list naming a broker twice or a receiver missing from the table `ids` (at its first such
    position), else, with a sender budget, a row with receivers whose leader is missing from `send_ids`: (KA_ERR_BAD_ARG, row,
    id), and no plan."""
    Q = len(out_len)
    table = set(int(x) for x in ids)
    senders, C = (None, None) if send is None else (set(int(x) for x in send[0]), send[1])
    opened, load, sopen, sload = {}, {}, {}, {}
    inb, outb = {}, {}                               # (wave, broker id) -> incoming / outgoing weight
    wave = np.zeros(Q, dtype=np.int32)
    recv_of = {}
    for g in range(Q):
        new = [int(x) for x in out[g][:int(out_len[g])]]
        old = [int(x) for x in cur[int(rep_off[g]):int(rep_off[g + 1])]]
        recv = []
        for j, b in enumerate(new):
            if b in new[:j] or (b not in old and b not in table):
                return None, None, (BAD, g, b)
            if b not in old:
                recv.append(b)
        if new == old:
            continue
        if not recv:
            wave[g] = 1
            continue
        s = old[0] if send is not None and old else None
        if s is not None and s not in senders:
            return None, None, (BAD, g, s)
        w = 1 if weight is None else int(weight[g])
        a = w * len(recv)
        v = max(opened.get(b, 1) if load.get(b, 0) == 0 or load.get(b, 0) + w <= B else opened.get(b, 1) + 1 for b in recv)
        if s is not None:
            o, x = sopen.get(s, 1), sload.get(s, 0)
            v = max(v, o if x == 0 or x + a <= C else o + 1)
        for b in recv:
            if v > opened.get(b, 1):
                opened[b], load[b] = v, w
            else:
                load[b] = load.get(b, 0) + w
            inb[(v, b)] = inb.get((v, b), 0) + w
        if s is not None:
            if v > sopen.get(s, 1):
                sopen[s], sload[s] = v, a
            else:
                sload[s] = sload.get(s, 0) + a
            outb[(v, s)] = outb.get((v, s), 0) + a
        wave[g] = v
        recv_of[g] = (len(recv), w)
    W = int(wave.max()) if Q else 0
    empty = dict(rows=0, rows_moved=0, replicas_added=0, max_broker_in=0, max_broker_in_id=-1)
    peaks = [(inb, "max_broker_in", "max_broker_in_id")]
    if send is not None:
        empty.update(max_broker_out=0, max_broker_out_id=-1)
        peaks.append((outb, "max_broker_out", "max_broker_out_id"))
    summ = [dict(empty) for _ in range(W)]
    for g in np.nonzero(wave)[0]:
        s = summ[wave[g] - 1]
        s["rows"] += 1
        if g in recv_of:
            n, w = recv_of[g]
            s["rows_moved"] += 1
            s["replicas_added"] += n * w
    for bins, peak, pid in peaks:
        for (v, b), x in sorted(bins.items()):
            s = summ[v - 1]
            if x > s[peak]:
                s[peak], s[pid] = x, b
    return wave, summ, (0, 0, 0)


# ---- the wave chain's rounds (both rules) ----------------------------------------------------------------------------------
# The device does not report its rounds, so these restatements of the round rule of kassign_waves.cuh are the evidence that a
# plan reaches the chain's claim reset.

WAVE_CHUNK = 2048            # KA_WAVE_CHUNK: records the chain decides together
WAVE_RESET = 1 << 21         # KA_WAVE_MAX_ROUND: the round at which the chain clears its claims and counts from 1 again


def wave_records(rep_off, cur, out, out_len):
    """(receivers, senders) per row: the new-list brokers its current list lacks, in list order, and the first broker of its
    current list (None when it is empty). A row with receivers is a record of the chain; the others are not."""
    rcv, snd = [], []
    for g in range(len(out_len)):
        old = cur[int(rep_off[g]):int(rep_off[g + 1])].tolist()
        rcv.append([b for b in out[g, :int(out_len[g])].tolist() if b not in old])
        snd.append(old[0] if old else None)
    return rcv, snd


def chain_keys(records, senders, g):
    """The chain's words a record claims: its receivers', and with a send table its sender's (a separate set of words)."""
    keys = [("r", b) for b in records[g]]
    if senders is not None and senders[g] is not None:
        keys.append(("s", senders[g]))
    return keys


def chain_rounds(records, senders=None):
    """The global round in which the chain decides every record (int64 per row, 0 for a row without receivers). records: the
    receivers of every row; senders (the send form): the sender of every row, or None. The records, in row order, are cut into
    chunks of 2 048. A record decides in round 1 + the latest round among the earlier records of its chunk that share a receiver
    with it, or its sender; a chunk takes as many rounds as its latest record, and the count runs on across chunks."""
    rounds = np.zeros(len(records), dtype=np.int64)
    base = top = n = 0
    last = {}
    for g, rcv in enumerate(records):
        if not rcv:
            continue
        if n == WAVE_CHUNK:
            base, top, n, last = base + top, 0, 0, {}
        keys = chain_keys(records, senders, g)
        r = 1 + max(last.get(k, 0) for k in keys)
        for k in keys:
            last[k] = r
        top = max(top, r)
        n += 1
        rounds[g] = base + r
    return rounds


def crossing_chunk(records, senders, rounds):
    """The chunk in which round 2^21 falls: (records decided before the reset, after it, keys (receivers or senders) with records
    on both sides, chunks after it). Fails unless exactly one chunk has records on both sides."""
    rows = np.nonzero(rounds)[0]
    chunk = np.arange(len(rows)) // WAVE_CHUNK
    starts = np.arange(0, len(rows), WAVE_CHUNK)
    lo, hi = np.minimum.reduceat(rounds[rows], starts), np.maximum.reduceat(rounds[rows], starts)
    mixed = np.nonzero((lo < WAVE_RESET) & (hi >= WAVE_RESET))[0]
    assert len(mixed) == 1, mixed
    c = int(mixed[0])
    mine = rows[chunk == c]
    before = rounds[mine] < WAVE_RESET
    sides = {}
    for g, b in zip(mine, before):
        for k in chain_keys(records, senders, g):
            sides.setdefault(k, set()).add(bool(b))
    shared = sum(len(v) == 2 for v in sides.values())
    return int(before.sum()), int((~before).sum()), shared, len(starts) - 1 - c


# ---- reassignment JSON ---------------------------------------------------------------------------------------------------
# The records of KafkaAssignmentGenerator.java:169-186 in the predicted org.json key order (SURVEY §3.4): "partition",
# "replicas", "topic" inside {"partitions":[...],"version":1}.

_SHORT = {"\b": "\\b", "\t": "\\t", "\n": "\\n", "\f": "\\f", "\r": "\\r", '"': '\\"', "\\": "\\\\"}


def _quote(name, wide):
    """org.json 20131018 JSONObject.quote() over the UTF-16 code units of `name`: '"' and '\\' escaped, '/' only right after
    '<', \\b \\t \\n \\f \\r short, every other unit below 0x20 (and with `wide` every unit in [0x80, 0xA0) or [0x2000, 0x2100))
    as \\u plus four lowercase hex digits; the rest kept. No escaped unit is a surrogate, so walking the code points of `name`
    visits the same units: a char above U+FFFF (two surrogates) is kept whole and is never the '<' before a '/'."""
    out, prev = [], ""
    for ch in name:
        c = ord(ch)
        if ch in _SHORT:
            out.append(_SHORT[ch])
        elif ch == "/":
            out.append("\\/" if prev == "<" else "/")
        elif c < 0x20 or (wide and (0x80 <= c < 0xA0 or 0x2000 <= c < 0x2100)):
            out.append("\\u%04x" % c)
        else:
            out.append(ch)
        prev = ch
    return '"' + "".join(out) + '"'


def quote(name):
    """org.json 20131018 JSONObject.quote() of a topic name (the records of the reassignment JSON): the ASCII escapes, and
    every char in [0x80, 0xA0) or [0x2000, 0x2100) as \\u%04x. U+007F and U+00A0 are kept; "" gives '""'."""
    return _quote(name, True)


def kafka_quote(name):
    """The quote of the CURRENT ASSIGNMENT and rollback records (Kafka's own encoder, not org.json): the ASCII escapes of quote
    only; every char above 0x7F is kept."""
    return _quote(name, False)


def device_refuses(name):
    """(char, a) of the first char of `name` the device emitters refuse (ka_json_name_refused), a its code point, or None:
    a char quote() rewrites, or '/' (quote() escapes it only after '<'; the device refuses every one)."""
    for ch in name:
        c = ord(ch)
        if c < 0x20 or ch in '"\\/' or 0x80 <= c < 0xA0 or 0x2000 <= c < 0x2100:
            return ch, c
    return None


def record(name, partition, replicas):
    return '{"partition":%d,"replicas":[%s],"topic":%s}' % (partition, ",".join(str(int(b)) for b in replicas), quote(name))


def document(records):
    """The document of these records (str)."""
    return '{"partitions":[' + ",".join(records) + '],"version":1}'


def current_record(name, partition, replicas):
    """The rollback record: the host's CURRENT ASSIGNMENT record (Kafka 0.10 ZkUtils.formatAsReassignmentJson key order) of a
    partition on its current list `replicas`, printed as given."""
    return '{"topic":%s,"partition":%d,"replicas":[%s]}' % (kafka_quote(name), partition, ",".join(str(int(b)) for b in replicas))


def rollback_document(records):
    """The rollback document of these current records (str)."""
    return '{"version":1,"partitions":[' + ",".join(records) + ']}'


EMPTY_DOCUMENT = document([])


def solve_document(names, part_off, part_id, out, out_len):
    """The text of ka_solve_json for the rows out [Q, S] / out_len [Q] of the topics `names` (partition ids part_id)."""
    return document(record(name, part_id[g], out[g, :out_len[g]]) for t, name in enumerate(names)
                    for g in range(int(part_off[t]), int(part_off[t + 1])))


def dense_document(cl, out, out_len):
    """The text of ka_solve_dense_json for the dense cluster cl's rows out [T * P, S] / out_len [T * P]."""
    return solve_document(cl.topic_names, np.arange(cl.T + 1) * cl.P, np.tile(np.arange(cl.P), cl.T), out.reshape(cl.T * cl.P, -1),
                          out_len.reshape(-1))


def json_bound(names, part_off, stride):
    """The sufficient json_cap of include/kassign.h for one document per wave."""
    return sum(int(part_off[t + 1] - part_off[t]) * (79 + 12 * stride + len(n.encode())) for t, n in enumerate(names))


def cut_parts(sides, L):
    """The greedy cut of ka_plan_waves_json_parts(_rollback) over one wave's records, in order: [(first, end)] runs. `sides`
    holds one list of record byte lengths, or two with the rollback records'. A part of n records is 29 + their bytes + (n - 1)
    long on each side; a record joins the current part while every side stays <= L."""
    runs, size = [], [0] * len(sides)
    for i, lens in enumerate(zip(*sides)):
        if runs and all(s + 1 + b <= L for s, b in zip(size, lens)):
            runs[-1] = (runs[-1][0], i + 1)
            size = [s + 1 + b for s, b in zip(size, lens)]
        else:
            runs.append((i, i + 1))
            size = [29 + b for b in lens]
    return runs


def wave_documents(topic_names, part_off, part_id, rep_off, cur, out, out_len, ids, B, weight=None, send=None, L=None,
                   rollback=False):
    """(docs [bytes], backs [bytes] or None, doc_wave, wave, summary, (code, a, b)) of the six wave document entry points, the
    shape Solver._wave_documents returns: the records of every wave of plan_waves in input row order (ordinals where part_id is
    None), one document per wave with L None (ka_plan_waves(_send)_json), else cut by cut_parts (their _parts forms), and with
    rollback backs[d] the current records of docs[d]'s rows (their _parts_rollback forms). A changed row whose one-record
    document on either side exceeds L, the lowest in input order, gives (KA_ERR_LIMIT, row, the longer length) and no docs."""
    wave, summ, st = plan_waves(rep_off, cur, out, out_len, ids, B, weight, send)
    if st[0] != 0:
        return None, None, None, wave, summ, st
    recs = [[] for _ in summ]
    for t, name in enumerate(topic_names):
        for g in range(int(part_off[t]), int(part_off[t + 1])):
            if wave[g]:
                p = int(part_id[g]) if part_id is not None else g - int(part_off[t])
                sides = [record(name, p, out[g][:int(out_len[g])])]
                if rollback:
                    sides.append(current_record(name, p, cur[int(rep_off[g]):int(rep_off[g + 1])]))
                longest = 29 + max(len(x.encode()) for x in sides)
                if L is not None and longest > L:
                    return None, None, None, wave, summ, (_native.KA_ERR_LIMIT, g, min(longest, 2 ** 31 - 1))
                recs[wave[g] - 1].append(sides)
    docs, backs, doc_wave = [], [] if rollback else None, []
    for v, rs in enumerate(recs, 1):
        runs = [(0, len(rs))] if L is None else cut_parts([[len(r[k].encode()) for r in rs] for k in range(len(rs[0]))], L)
        for a, b in runs:
            docs.append(document([r[0] for r in rs[a:b]]).encode())
            if rollback:
                backs.append(rollback_document([r[1] for r in rs[a:b]]).encode())
            doc_wave.append(v)
    return docs, backs, doc_wave, wave, summ, st


# ---- the leader-order schedule and the counters --------------------------------------------------------------------------

def java_abs_hash(h):
    return int(np.int64(abs(int(h))) if h != -2**31 else 2**31)


def build_records(cl, sets):
    """What kernel A emits for every row: ([a0, a1, a2] in slot-0 scan order with the dummy N for missing slots, len, e01, e02, e12).
    sets[t]: the rows of topic t (a dense cluster's P rows, or a ragged topic's)."""
    N = cl.N
    idx_of = {int(b): i for i, b in enumerate(cl.broker_id)}
    recs = []
    for t in range(cl.T):
        habs = java_abs_hash(cl.topic_hash[t])
        s2, s3 = habs % 2, habs % 3
        for row in sets[t]:
            ix = sorted(idx_of[int(b)] for b in row)                 # ascending index == ascending id (KAS:205-214)
            k = len(ix)
            a, e = [N, N, N], (0, 0, 0)
            if k == 1:
                a[0] = ix[0]
            elif k == 2:
                a[0], a[1] = ix[s2], ix[1 - s2]                       # |hash| % 2 == 1: the higher id is scanned first
            elif k == 3:
                i = [(3 - s3) % 3, (4 - s3) % 3, (5 - s3) % 3]        # list position at scan position 0, 1, 2
                a = [ix[i[0]], ix[i[1]], ix[i[2]]]
                e = tuple(s2 if i[x] < i[y] else 1 - s2 for x, y in ((0, 1), (0, 2), (1, 2)))
            recs.append((a, k, e))
    return recs


def i32(v):
    """v as a Java int (two's complement wrap)."""
    return (int(v) + 2**31) % 2**32 - 2**31


def conflict_levels(rows):
    """Conflict level of every record of one topic (kernel A's LEVELS pass)."""
    last, lv = {}, []
    for a, k, _ in rows:
        real = [b for b in a[:max(k, 0)]]
        lvl = 1 + max([last.get(b, 0) for b in real] or [0])
        for b in real:
            last[b] = lvl
        lv.append(lvl)
    return lv


def slot_chains(cl, sets, rng, c0, c1, c2):
    """The leader order of the CUDA path for rows of <= 3, as kassign_stage.cuh / kassign_order.cuh run it: the records of
    build_records in a level schedule (topic by topic, level by level, in a scrambled order inside a level), the whole slot-0
    chain first, then the slot-1 chain; slot 2 a plain sum. c0 / c1 / c2: counter[.][0 / 1 / 2] by broker index, each with
    the dummy's entry at index N (INF for c0 and c1); updated in place with int32 arithmetic, as the device adds. A row of k
    replicas bumps slot r only when r < k, so the dummy is never bumped. Returns {record: ordered broker indices}."""
    N = cl.N
    recs = build_records(cl, sets)
    order, g0 = [], 0
    for t in range(cl.T):
        rows = recs[g0:g0 + len(sets[t])]
        lv = conflict_levels(rows)
        for level in range(1, max(lv + [0]) + 1):
            members = [g0 + p for p in range(len(rows)) if lv[p] == level]
            used = [b for q in members for b in recs[q][0][:recs[q][1]]]
            assert len(used) == len(set(used)), "partitions of one level must not share a broker"
            rng.shuffle(members)
            order.extend(members)
        g0 += len(rows)
    assert sorted(order) == list(range(len(recs)))
    assert c0[N] == INF and c1[N] == INF
    # ---- slot-0 chain over ALL rows first (it never needs a slot-1 decision) ----
    mid = {}
    for q in order:
        a, k, e = recs[q]
        x = [c0[a[0]], c0[a[1]], c0[a[2]]]
        L10, L20, L21 = x[1] < x[0], x[2] < x[0], x[2] < x[1]       # strict '<' in scan order: ties to the earlier position
        is2 = L21 if L10 else L20
        is1 = L10 and not L21
        w = 2 if is2 else (1 if is1 else 0)
        if k > 0:
            c0[a[w]] = i32(c0[a[w]] + 1)
        p_, q_ = (1, 2) if w == 0 else ((0, 2) if w == 1 else (0, 1))
        mid[q] = (a[p_], a[q_], e[{(0, 1): 0, (0, 2): 1, (1, 2): 2}[(p_, q_)]], a[w], k)
    # ---- slot-1 chain ----
    out = {}
    for q in order:
        op, oq, e, oA, k = mid[q]
        pick = c1[oq] < i32(c1[op] + e)
        o1, o2 = (oq, op) if pick else (op, oq)
        if k > 1:
            c1[o1] = i32(c1[o1] + 1)
        if k > 2:
            c2[o2] = i32(c2[o2] + 1)                                 # slot 2: a plain sum (the emit kernel's atomicAdd)
        out[q] = [oA, o1, o2][:k]
    assert c0[N] == INF and c1[N] == INF
    return out


def histogram(ids, out, out_len):
    """counter[b][r] of a fresh Context after these rows: the number of rows with broker ids[b] at position r."""
    ids = np.asarray(ids)
    ctr = np.zeros((len(ids), SLOTS), dtype=np.int64)
    for r in range(out.shape[1]):
        sel = out_len > r
        idx = np.searchsorted(ids, out[sel, r])
        assert np.all(ids[idx] == out[sel, r])
        np.add.at(ctr[:, r], idx, 1)
    return ctr


# ---- kernel A's shared-memory budget (make_plan, kassign.cu) --------------------------------------------------------------

def a16(v):
    return (v + 15) & ~15


def blob_bytes(ids):
    """Bytes of the broker blob kernel A stages: rack indices, plus the id LUT when the id range fits shared memory."""
    n = len(ids)
    rng_ = int(ids[-1]) - int(ids[0]) + 1 if n else 0
    lut = a16(max(rng_, 1) * 2) if rng_ <= 32768 else 0
    return a16(max(n, 1) * 2) + lut


def stage_warps(N, blob, Pmax, S, capmax, levels):
    """Warps per CTA of make_plan, or 0 when the layout exceeds the 200 KB budget (KA_ERR_LIMIT, a = Pmax, b = N)."""
    lsz = 1 if capmax <= 255 else 2
    per_warp = a16(max(N, 1) * lsz) + a16(max(Pmax, 1) * S * 2) + a16(max(Pmax, 1))
    if levels:
        per_warp += a16(max(N, 1) * 4) + a16(max(N, 1) * 2) + 2 * a16((max(Pmax, 1) + 2) * 2)
    shared = 16 + blob
    if shared + per_warp > 200 * 1024:
        return 0
    return min(16, (200 * 1024 - shared) // per_warp)
