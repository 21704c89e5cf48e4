"""The plain-Python model of ka_plan_waves(_send)_json_parts: every wave document of a wave plan cut into parts of at most L
bytes. It restates the rule of include/kassign.h over the wave rule and the record printer of tests/models.py. Like that
module it imports numpy and the status codes only, so CPU tests, GPU tests and tests/tools can all use it."""
from kafka_assigner_b200 import _native
from tests import models


def cut_parts(lengths, L):
    """The greedy cut of ka_plan_waves_json_parts over the byte lengths of one wave's records, in order: [(first, end)] runs.
    A part of n records is 29 + their bytes + (n - 1) long; a record joins the current part while it stays <= L."""
    runs, size = [], 0
    for i, b in enumerate(lengths):
        if runs and size + 1 + b <= L:
            runs[-1] = (runs[-1][0], i + 1)
            size += 1 + b
        else:
            runs.append((i, i + 1))
            size = 29 + b
    return runs


def wave_parts(topic_names, part_off, part_id, rep_off, cur, out, out_len, ids, B, L, weight=None, send=None):
    """(parts [bytes], part_wave, wave, summary, (code, a, b)) of ka_plan_waves(_send)_json_parts: the records of every wave of
    models.plan_waves, in input row order, cut by cut_parts. A changed row whose one-record document exceeds L, the lowest in
    input order, gives (KA_ERR_LIMIT, row, that length) and no parts."""
    wave, summ, st = models.plan_waves(rep_off, cur, out, out_len, ids, B, weight, send)
    if st[0] != 0:
        return None, None, wave, summ, st
    recs = [[] for _ in summ]
    for t, name in enumerate(topic_names):
        for g in range(int(part_off[t]), int(part_off[t + 1])):
            if wave[g]:
                p = int(part_id[g]) if part_id is not None else g - int(part_off[t])
                rec = models.record(name, p, out[g][:int(out_len[g])]).encode()
                if 29 + len(rec) > L:
                    return None, None, wave, summ, (_native.KA_ERR_LIMIT, g, min(29 + len(rec), 2 ** 31 - 1))
                recs[wave[g] - 1].append(rec)
    parts, part_wave = [], []
    for v, rs in enumerate(recs, 1):
        for a, b in cut_parts([len(r) for r in rs], L):
            parts.append(b'{"partitions":[' + b",".join(rs[a:b]) + b'],"version":1}')
            part_wave.append(v)
    return parts, part_wave, wave, summ, st
