"""The plain-Python model of the first-fit wave rule (KA_WAVE_FIRST_FIT of include/kassign.h), its bound Wb on the waves, and
the documents built from its plan, beside the greedy rule's in tests/models.py. Like that module it imports numpy and the
status codes only, so CPU tests, GPU tests and tests/tools can all use it."""
import numpy as np

from kafka_assigner_b200 import _native
from tests import models


def plan_waves(rep_off, cur, out, out_len, ids, B, weight=None, send=None):
    """(wave [Q] int32, [summary dict per wave], (code, a, b)) of the first-fit rule, rows in input order, with the arguments and
    results of models.plan_waves (send=None: ka_plan_waves, send=(send_ids, C): ka_plan_waves_send) and its row errors.

    A row with receivers takes the smallest wave v >= 1 in which every receiver's bucket (b, v) is empty or stays within B with
    its weight w, and its sender's bucket (s, v) is empty or stays within C with a = w x receivers. A row of weight >= 1 starts
    its search at the largest hint of its buckets' rows, the lowest wave whose load is below the budget (every wave below it
    refuses such a row); tests check the result against a search from wave 1."""
    Q = len(out_len)
    table = set(int(x) for x in ids)
    senders, C = (None, None) if send is None else (set(int(x) for x in send[0]), send[1])
    bucket, hint = {}, {}                            # ("r" | "s", broker id, wave) -> load; ("r" | "s", broker id) -> hint
    wave = np.zeros(Q, dtype=np.int32)
    recv_of = {}
    for g in range(Q):
        new = [int(x) for x in out[g][:int(out_len[g])]]
        old = [int(x) for x in cur[int(rep_off[g]):int(rep_off[g + 1])]]
        recv = []
        for j, b in enumerate(new):
            if b in new[:j] or (b not in old and b not in table):
                return None, None, (models.BAD, g, b)
            if b not in old:
                recv.append(b)
        if new == old:
            continue
        if not recv:
            wave[g] = 1
            continue
        s = old[0] if send is not None and old else None
        if s is not None and s not in senders:
            return None, None, (models.BAD, g, s)
        w = 1 if weight is None else int(weight[g])
        places = [("r", b, w, B) for b in recv] + ([("s", s, w * len(recv), C)] if s is not None else [])
        v = max(hint.get((k, b), 1) for k, b, _, _ in places) if w > 0 else 1
        while not all(bucket.get((k, b, v), 0) == 0 or bucket[(k, b, v)] + x <= cap for k, b, x, cap in places):
            v += 1
        for k, b, x, cap in places:
            bucket[(k, b, v)] = bucket.get((k, b, v), 0) + x
            h = hint.get((k, b), 1)
            while bucket.get((k, b, h), 0) >= cap:
                h += 1
            hint[(k, b)] = h
        wave[g] = v
        recv_of[g] = (len(recv), w)
    W = int(wave.max()) if Q else 0
    empty = dict(rows=0, rows_moved=0, replicas_added=0, max_broker_in=0, max_broker_in_id=-1)
    peaks = [("r", "max_broker_in", "max_broker_in_id")]
    if send is not None:
        empty.update(max_broker_out=0, max_broker_out_id=-1)
        peaks.append(("s", "max_broker_out", "max_broker_out_id"))
    summ = [dict(empty) for _ in range(W)]
    for g in np.nonzero(wave)[0]:
        s = summ[wave[g] - 1]
        s["rows"] += 1
        if g in recv_of:
            n, w = recv_of[g]
            s["rows_moved"] += 1
            s["replicas_added"] += n * w
    for kind, peak, pid in peaks:
        for (k, b, v), x in sorted(bucket.items(), key=lambda e: (e[0][2], e[0][1])):
            s = summ[v - 1]
            if k == kind and x > s[peak]:
                s[peak], s[pid] = x, b
    return wave, summ, (0, 0, 0)


def moved(cur_lists, new_lists, weight, send):
    """[(row, receivers, w, sender or None)] of the rows with receivers (the chain's records), from the current and new lists."""
    res = []
    for g, (old, new) in enumerate(zip(cur_lists, new_lists)):
        recv = [b for b in new if b not in old]
        if old != new and recv:
            res.append((g, recv, 1 if weight is None else int(weight[g]), old[0] if send is not None and old else None))
    return res


def bound(moved):
    """Wb of include/kassign.h over the records of `moved`: min(M, 1 + max over moved rows of sum (R_b - 1) + (S_s - 1))."""
    R, S = {}, {}
    for _, recv, _, s in moved:
        for b in recv:
            R[b] = R.get(b, 0) + 1
        if s is not None:
            S[s] = S.get(s, 0) + 1
    if not moved:
        return 0
    worst = max(sum(R[b] - 1 for b in recv) + (S[s] - 1 if s is not None else 0) for _, recv, _, s in moved)
    return min(len(moved), 1 + worst)


def wave_documents(topic_names, part_off, part_id, rep_off, cur, out, out_len, ids, B, weight=None, send=None, L=None,
                   rollback=False):
    """models.wave_documents over the first-fit plan: (docs, backs, doc_wave, wave, summary, (code, a, b)) of the six wave
    document entry points under KA_WAVE_FIRST_FIT, with the same arguments, documents, cut and errors."""
    wave, summ, st = plan_waves(rep_off, cur, out, out_len, ids, B, weight, send)
    if st[0] != 0:
        return None, None, None, wave, summ, st
    recs = [[] for _ in summ]
    for t, name in enumerate(topic_names):
        for g in range(int(part_off[t]), int(part_off[t + 1])):
            if wave[g]:
                p = int(part_id[g]) if part_id is not None else g - int(part_off[t])
                sides = [models.record(name, p, out[g][:int(out_len[g])])]
                if rollback:
                    sides.append(models.current_record(name, p, cur[int(rep_off[g]):int(rep_off[g + 1])]))
                longest = 29 + max(len(x.encode()) for x in sides)
                if L is not None and longest > L:
                    return None, None, None, wave, summ, (_native.KA_ERR_LIMIT, g, min(longest, 2 ** 31 - 1))
                recs[wave[g] - 1].append(sides)
    docs, backs, doc_wave = [], [] if rollback else None, []
    for v, rs in enumerate(recs, 1):
        runs = [(0, len(rs))] if L is None else models.cut_parts([[len(r[k].encode()) for r in rs] for k in range(len(rs[0]))], L)
        for a, b in runs:
            docs.append(models.document([r[0] for r in rs[a:b]]).encode())
            if rollback:
                backs.append(models.rollback_document([r[1] for r in rs[a:b]]).encode())
            doc_wave.append(v)
    return docs, backs, doc_wave, wave, summ, st
