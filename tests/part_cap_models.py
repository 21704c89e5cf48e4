"""The model of the part caps (ka_ctx_set_part_caps), restated from include/kassign.h beside the uncapped models of
tests/models.py, which it builds on: every row's moved data a_g, the capped greedy cut, the capped wave documents, and the check
of one Solver call against them. Like tests/models.py it never loads the library itself (the check takes a Solver)."""
import numpy as np

from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SEND_SUMMARY_DTYPE, WAVE_SUMMARY_DTYPE
from tests import models


def moved_data(rep_off, cur, out, out_len, weight, g):
    """a_g: row g's weight (1 without weights) x its receivers, the new-list brokers its current list lacks; what
    ka_wave_summary.replicas_added adds for the row."""
    old = set(int(x) for x in cur[int(rep_off[g]):int(rep_off[g + 1])])
    w = 1 if weight is None else int(weight[g])
    return w * sum(int(b) not in old for b in out[g][:int(out_len[g])])


def cut_parts(sides, L, Lr=None, Lx=None, a=None):
    """models.cut_parts under the part caps (None: no cap): a record joins the current part while every side stays <= L, the
    part stays within Lr records, and the a of its records (a[i] per record) sum to at most Lx. With both caps None this is
    models.cut_parts."""
    runs, size, moved = [], [0] * len(sides), 0
    for i, lens in enumerate(zip(*sides)):
        ai = 0 if a is None else a[i]
        if (runs and all(s + 1 + b <= L for s, b in zip(size, lens)) and (Lr is None or i + 1 - runs[-1][0] <= Lr)
                and (Lx is None or moved + ai <= Lx)):
            runs[-1] = (runs[-1][0], i + 1)
            size = [s + 1 + b for s, b in zip(size, lens)]
            moved += ai
        else:
            runs.append((i, i + 1))
            size = [29 + b for b in lens]
            moved = ai
    return runs


def wave_records(names, part_off, part_id, rep_off, cur, out, out_len, wave, weight):
    """Per wave of `wave`: the (record, rollback record, a) of its rows, in input row order."""
    recs = [[] for _ in range(int(wave.max()) if len(wave) else 0)]
    for t, name in enumerate(names):
        for g in range(int(part_off[t]), int(part_off[t + 1])):
            if wave[g]:
                p = int(part_id[g]) if part_id is not None else g - int(part_off[t])
                recs[wave[g] - 1].append((models.record(name, p, out[g][:int(out_len[g])]),
                                          models.current_record(name, p, cur[int(rep_off[g]):int(rep_off[g + 1])]),
                                          moved_data(rep_off, cur, out, out_len, weight, g)))
    return recs


def cut_documents(recs, L, Lr=None, Lx=None, rollback=False):
    """(docs [bytes], backs [bytes], doc_wave, [(rows, data)] per part) of the capped cut of wave_records' records. A record
    whose one-record document on either side exceeds L is the caller's to refuse first."""
    docs, backs, doc_wave, sizes = [], [], [], []
    for v, rs in enumerate(recs, 1):
        sides = [[len(r[0].encode()) for r in rs]] + ([[len(r[1].encode()) for r in rs]] if rollback else [])
        for i, j in cut_parts(sides, L, Lr, Lx, [r[2] for r in rs]):
            docs.append(models.document([r[0] for r in rs[i:j]]).encode())
            backs.append(models.rollback_document([r[1] for r in rs[i:j]]).encode())
            doc_wave.append(v)
            sizes.append((j - i, sum(r[2] for r in rs[i:j])))
    return docs, backs, doc_wave, sizes


def wave_documents(names, part_off, part_id, rep_off, cur, out, out_len, ids, B, weight=None, send=None, L=None, rollback=False,
                   Lr=None, Lx=None):
    """models.wave_documents of the _parts forms (L given) under the part caps: (docs, backs or None, doc_wave, wave, summary,
    (code, a, b)). The plan is models.plan_waves (the greedy rule); the caps change no error."""
    e = models.wave_documents(names, part_off, part_id, rep_off, cur, out, out_len, ids, B, weight, send, L, rollback)
    if e[5][0] != 0 or (Lr is None and Lx is None):
        return e
    recs = wave_records(names, part_off, part_id, rep_off, cur, out, out_len, e[3], weight)
    docs, backs, doc_wave = cut_documents(recs, L, Lr, Lx, rollback)[:3]
    return docs, backs if rollback else None, doc_wave, e[3], e[4], e[5]


def check_wave_documents(s, names, part_off, part_id, rep_off, cur, out, out_len, B, L, rollback=False, weight=None, C=None,
                         send_ids=None, json_buf=None, Lr=None, Lx=None):
    """s.plan_wave_parts_json or, with rollback, s.plan_wave_parts_rollback_json (the Solver's caps set by the caller to Lr /
    Lx) against wave_documents and against s.plan_waves on the same inputs; with C a sender budget over send_ids (None: the
    Solver's table). Returns (docs, backs, doc_wave, wave, summary, status)."""
    send_ids = list(np.asarray(s.broker_id if send_ids is None else send_ids))
    send = {} if C is None else dict(max_broker_out=C, send_brokers=send_ids)
    args = (names, part_off, part_id, rep_off, cur, out, out_len, B)
    if rollback:
        got = s.plan_wave_parts_rollback_json(*args, L, weight=weight, json_buf=json_buf, **send)
    else:
        docs, doc_wave, wave, summ, st = s.plan_wave_parts_json(*args, L, weight=weight, json_buf=json_buf, **send)
        got = (docs, None, doc_wave, wave, summ, st)
    docs, backs, doc_wave, wave, summ, st = got
    e_docs, e_backs, e_doc_wave, e_wave, e_summ, e_st = wave_documents(
        names, part_off, part_id, rep_off, cur, out, out_len, s.broker_id, B, weight, None if C is None else (send_ids, C), L, rollback,
        Lr, Lx)
    assert (st.code, st.a, st.b) == e_st, ((st.code, st.a, st.b), e_st)
    p_wave, p_summ, p_st = s.plan_waves(rep_off, cur, out, out_len, B, weight=weight, **send)
    assert (p_st.code, p_st.a, p_st.b) == (e_st if e_st[0] != _native.KA_ERR_LIMIT else (0, 0, 0))
    if st.code == 0:
        fields = (WAVE_SUMMARY_DTYPE if C is None else WAVE_SEND_SUMMARY_DTYPE).names
        assert np.array_equal(wave, e_wave) and np.array_equal(wave, p_wave)
        assert [{f: int(x[f]) for f in fields} for x in summ] == e_summ and np.array_equal(summ, p_summ)
        assert doc_wave.tolist() == e_doc_wave and len(docs) == len(e_docs)
        for d, (x, e) in enumerate(zip(docs, e_docs)):
            assert bytes(x) == e, (d, bytes(x)[:200], e[:200])
        if rollback:
            assert [bytes(x) for x in backs] == e_backs
    return got
