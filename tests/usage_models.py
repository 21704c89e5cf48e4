"""The model of ka_wave_broker_usage: every broker's disk usage across a wave plan. `broker_usage` restates the rule and the check
order of include/kassign.h as a plain loop over the waves 0..W of every broker; `broker_usage_np` is the same rule over the
replica events in numpy, for plans whose W or size is too large for the loop (it takes inputs the checks pass). This module
imports numpy and the status codes only."""
import numpy as np

from kafka_assigner_b200 import _native

BAD, LIMIT = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT
INT64_MAX = 2 ** 63 - 1
FIELDS = ("before", "peak", "peak_wave", "after", "over_wave")


def _lists(rep_off, cur, out, out_len, g):
    return ([int(x) for x in cur[int(rep_off[g]):int(rep_off[g + 1])]], [int(x) for x in out[g][:int(out_len[g])]])


def host_checks(rep_off, cur, out, out_len, wave, use_id, weight=None, base=None, cap=None, stride=None):
    """(code, a, b) of the host-side checks after the argument errors, in their order, or (0, 0, 0)."""
    Q = len(out_len)
    stride = out.shape[1] if stride is None else stride
    n = len(use_id)
    if stride > 8:
        return LIMIT, stride, 0
    if n > 65535:
        return LIMIT, n, 0
    if any(int(use_id[i]) <= int(use_id[i - 1]) for i in range(1, n)):
        return BAD, 0, 0
    if any(int(x) < 0 for a in (weight, base, cap) if a is not None for x in a):
        return BAD, 0, 0
    for g in range(Q):
        if not 0 <= int(out_len[g]) <= stride or int(wave[g]) < 0:
            return BAD, g, 0
    total = sum(int(x) for x in base) if base is not None else 0
    for g in range(Q):
        total += (1 if weight is None else int(weight[g])) * (int(rep_off[g + 1] - rep_off[g]) + int(out_len[g]))
    if total > INT64_MAX or Q * stride + (int(rep_off[Q]) if Q else 0) > 2 ** 31 - 1:
        return LIMIT, 0, 0
    return 0, 0, 0


def broker_usage(rep_off, cur, out, out_len, wave, use_id, weight=None, base=None, cap=None):
    """([dict of the ka_broker_usage fields per table broker], W, (code, a, b)): the host checks, then the row checks (the lowest
    failing row: a new list naming a broker twice, or a receiver of a row with a wave that the table lacks, at its first such
    position), then the rule, one wave at a time."""
    st = host_checks(rep_off, cur, out, out_len, wave, use_id, weight, base, cap)
    if st[0]:
        return None, 0, st
    Q = len(out_len)
    table = [int(x) for x in use_id]
    for g in range(Q):
        old, new = _lists(rep_off, cur, out, out_len, g)
        for j, b in enumerate(new):
            if b in new[:j] or (int(wave[g]) > 0 and b not in old and b not in table):
                return None, 0, (BAD, g, b)
    W = max([int(v) for v in wave] + [0])
    res = []
    for i, b in enumerate(table):
        w_of = [1 if weight is None else int(weight[g]) for g in range(Q)]
        holds = [b in _lists(rep_off, cur, out, out_len, g)[0] for g in range(Q)]
        new_has = [b in _lists(rep_off, cur, out, out_len, g)[1] for g in range(Q)]
        receives = [new_has[g] and not holds[g] for g in range(Q)]
        drops = [holds[g] and not new_has[g] for g in range(Q)]
        before = (0 if base is None else int(base[i])) + sum(w_of[g] for g in range(Q) if holds[g])
        usage = []
        for v in range(W + 1):
            u = before
            u += sum(w_of[g] for g in range(Q) if 1 <= int(wave[g]) <= v and receives[g])
            u -= sum(w_of[g] for g in range(Q) if 1 <= int(wave[g]) < v and drops[g])
            usage.append(u)
        peak = max(usage)
        after = usage[W] - sum(w_of[g] for g in range(Q) if int(wave[g]) == W and W >= 1 and drops[g])
        over = -1
        if cap is not None:
            over = next((v for v in range(W + 1) if usage[v] > int(cap[i])), -1)
        res.append(dict(before=before, peak=peak, peak_wave=usage.index(peak), after=after, over_wave=over))
    return res, W, (0, 0, 0)


def replica_events(rep_off, cur, out, out_len, wave, use_id, weight=None):
    """(before [n] without the bases, idx, wave, w) of valid inputs: the rows' sums per table broker and their replica events,
    (index, wave, +w) per receiver and (index, wave + 1, -w) per distinct dropper of every row with a wave."""
    use_id = np.asarray(use_id, dtype=np.int64)
    n = len(use_id)
    Q = len(out_len)
    S = out.shape[1]
    m = np.diff(np.asarray(rep_off, dtype=np.int64))
    M = max(int(m.max()) if Q else 0, 1)
    w = np.ones(Q, dtype=np.int64) if weight is None else np.asarray(weight, dtype=np.int64)
    wv = np.asarray(wave, dtype=np.int64)
    cmask = np.arange(M) < m[:, None]
    cb = np.full((Q, M), -1, dtype=np.int64)
    cb[cmask] = np.asarray(cur, dtype=np.int64)[(np.asarray(rep_off[:-1], dtype=np.int64)[:, None] + np.arange(M))[cmask]]
    nmask = np.arange(S) < np.asarray(out_len)[:, None]
    nb = np.where(nmask, out, -1).astype(np.int64)
    held = ((nb[:, :, None] == cb[:, None, :]) & cmask[:, None, :]).any(2)
    recv = nmask & ~held
    earlier = np.tril(np.ones((M, M), dtype=bool), -1)                     # [i, h]: h < i
    first = cmask & ~((cb[:, :, None] == cb[:, None, :]) & earlier[None] & cmask[:, None, :]).any(2)
    kept = ((cb[:, :, None] == nb[:, None, :]) & nmask[:, None, :]).any(2)
    drop = first & ~kept

    def index(ids):
        at = np.searchsorted(use_id, ids)
        ok = at < n
        ok[ok] = use_id[at[ok]] == ids[ok]
        return np.where(ok, at, -1)

    ci, ni = index(cb), index(nb)
    before = np.zeros(n, dtype=np.int64)
    sel = first & (ci >= 0)
    np.add.at(before, ci[sel], np.broadcast_to(w[:, None], (Q, M))[sel])
    run = (wv > 0)[:, None]
    r = recv & run
    assert (ni[r] >= 0).all(), "a receiver outside the usage table"
    d = drop & run & (ci >= 0)
    idx = np.concatenate([ni[r], ci[d]])
    ev_wave = np.concatenate([np.broadcast_to(wv[:, None], (Q, S))[r], np.broadcast_to(wv[:, None] + 1, (Q, M))[d]])
    ev_w = np.concatenate([np.broadcast_to(w[:, None], (Q, S))[r], -np.broadcast_to(w[:, None], (Q, M))[d]])
    return before, idx, ev_wave, ev_w


def broker_usage_np(rep_off, cur, out, out_len, wave, use_id, weight=None, base=None, cap=None):
    """The report of broker_usage for inputs every check passes, over the sorted replica events: a structured-free dict of int64
    arrays [n] per field, and W."""
    n = len(use_id)
    W = int(np.max(wave)) if len(wave) else 0
    before, idx, ev_wave, ev_w = replica_events(rep_off, cur, out, out_len, wave, use_id, weight)
    if base is not None:
        before = before + np.asarray(base, dtype=np.int64)
    after = before.copy()
    np.add.at(after, idx, ev_w)
    order = np.lexsort((ev_wave, idx))
    idx, ev_wave, ev_w = idx[order], ev_wave[order], ev_w[order]
    cs = np.cumsum(ev_w)
    start = np.searchsorted(idx, np.arange(n))
    prior = np.where(start > 0, cs[np.maximum(start - 1, 0)] if len(cs) else 0, 0)
    val = before[idx] + cs - prior[idx]
    # usage(v) at the last event of every (broker, wave) pair with v <= W
    last = np.ones(len(idx), dtype=bool)
    last[:-1] = (idx[1:] != idx[:-1]) | (ev_wave[1:] != ev_wave[:-1])
    pt = last & (ev_wave <= W)
    p_idx, p_wave, p_val = idx[pt], ev_wave[pt], val[pt]
    peak, peak_wave = before.copy(), np.zeros(n, dtype=np.int64)
    o = np.lexsort((p_wave, -p_val, p_idx))                               # per broker: largest value, then lowest wave
    u, at = np.unique(p_idx[o], return_index=True)
    best_v, best_w = p_val[o][at], p_wave[o][at]
    higher = best_v > peak[u]
    peak[u[higher]], peak_wave[u[higher]] = best_v[higher], best_w[higher]
    over = np.full(n, -1, dtype=np.int64)
    if cap is not None:
        cap = np.asarray(cap, dtype=np.int64)
        over[before > cap] = 0
        hit = p_val > cap[p_idx]
        u, at = np.unique(p_idx[hit], return_index=True)                   # events are in wave order per broker
        still = over[u] < 0
        over[u[still]] = p_wave[hit][at][still]
    return dict(before=before, peak=peak, peak_wave=peak_wave, after=after, over_wave=over), W
