"""The plain-Python model of ka_plan_waves(_send)_json_parts_rollback: every wave of a wave plan cut into parts whose document
and rollback document both stay within L bytes, and every part's rollback document. It restates the rule of include/kassign.h
over the wave rule and the record printer of tests/models.py. Like that module it imports numpy and the status codes only, so
CPU tests, GPU tests and tests/tools can all use it."""
from kafka_assigner_b200 import _native
from tests import models


def current_record(name, partition, replicas):
    """The rollback record: the host's CURRENT ASSIGNMENT record (Kafka 0.10 ZkUtils.formatAsReassignmentJson key order) of a
    partition on its current list `replicas`, printed as given."""
    return '{"topic":%s,"partition":%d,"replicas":[%s]}' % (models.quote(name), partition, ",".join(str(int(b)) for b in replicas))


def rollback_document(records):
    """The rollback document of these current records (str)."""
    return '{"version":1,"partitions":[' + ",".join(records) + ']}'


def cut_parts_paired(fwd_lengths, back_lengths, L):
    """The paired cut of ka_plan_waves_json_parts_rollback over the byte lengths of one wave's records and of their rollback
    records, in order: [(first, end)] runs. A record joins the current part while both its document and its rollback document
    (29 + their bytes + (n - 1) each) stay <= L."""
    runs, size, back = [], 0, 0
    for i, (b, r) in enumerate(zip(fwd_lengths, back_lengths)):
        if runs and size + 1 + b <= L and back + 1 + r <= L:
            runs[-1] = (runs[-1][0], i + 1)
            size, back = size + 1 + b, back + 1 + r
        else:
            runs.append((i, i + 1))
            size, back = 29 + b, 29 + r
    return runs


def wave_rollback_parts(topic_names, part_off, part_id, rep_off, cur, out, out_len, ids, B, L, weight=None, send=None):
    """(parts [bytes], rollback [bytes], part_wave, wave, summary, (code, a, b)) of ka_plan_waves(_send)_json_parts_rollback:
    the records of every wave of models.plan_waves, in input row order, cut by cut_parts_paired; rollback[d] holds the current
    records of parts[d]'s rows. A changed row whose one-record document on either side exceeds L, the lowest in input order,
    gives (KA_ERR_LIMIT, row, the longer length) and no parts."""
    wave, summ, st = models.plan_waves(rep_off, cur, out, out_len, ids, B, weight, send)
    if st[0] != 0:
        return None, None, None, wave, summ, st
    recs = [[] for _ in summ]
    for t, name in enumerate(topic_names):
        for g in range(int(part_off[t]), int(part_off[t + 1])):
            if wave[g]:
                p = int(part_id[g]) if part_id is not None else g - int(part_off[t])
                rec = models.record(name, p, out[g][:int(out_len[g])]).encode()
                back = current_record(name, p, cur[int(rep_off[g]):int(rep_off[g + 1])]).encode()
                if 29 + max(len(rec), len(back)) > L:
                    return None, None, None, wave, summ, (_native.KA_ERR_LIMIT, g, min(29 + max(len(rec), len(back)), 2 ** 31 - 1))
                recs[wave[g] - 1].append((rec, back))
    parts, rollback, part_wave = [], [], []
    for v, rs in enumerate(recs, 1):
        for a, b in cut_parts_paired([len(f) for f, _ in rs], [len(r) for _, r in rs], L):
            parts.append(models.document([f.decode() for f, _ in rs[a:b]]).encode())
            rollback.append(rollback_document([r.decode() for _, r in rs[a:b]]).encode())
            part_wave.append(v)
    return parts, rollback, part_wave, wave, summ, st
