"""ka_plan_waves_json_parts on the CPU: the greedy cut of `part_models.cut_parts` / `part_models.wave_parts` against a brute force over
every cut of random record lengths and against the per-wave documents of `models.wave_docs`; the declarations; and what
Solver.plan_wave_parts_json hands the C ABI and makes of what it gets back, through a fake library."""
import ctypes
import json
import os

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from kafka_assigner_b200.assigner import WAVE_SEND_SUMMARY_DTYPE, WAVE_SUMMARY_DTYPE
from tests import models, part_models, util

BAD, LIMIT = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _size(lengths):
    return 29 + sum(lengths) + len(lengths) - 1


def _brute(lengths, L):
    """Every cut of the records into consecutive runs in which each run fits and each run but the last could not take the next
    record: the greedy cut, found without a greedy loop."""
    n = len(lengths)
    found = []
    for mask in range(1 << max(n - 1, 0)):
        bounds = [0] + [i + 1 for i in range(n - 1) if mask >> i & 1] + [n]
        runs = list(zip(bounds, bounds[1:]))
        if all(_size(lengths[a:b]) <= L for a, b in runs) and all(_size(lengths[a:b + 1]) > L for a, b in runs[:-1]):
            found.append(runs)
    return found


@pytest.mark.parametrize("seed", range(6))
def test_cut_is_the_only_greedy_cut(seed):
    rng = np.random.default_rng(seed)
    for _ in range(60):
        n = int(rng.integers(1, 11))
        lengths = [int(x) for x in rng.integers(40, 120, n)]
        L = int(rng.integers(29 + max(lengths), 29 + sum(lengths) + n + 20))
        runs = part_models.cut_parts(lengths, L)
        assert _brute(lengths, L) == [runs], (lengths, L)
        assert all(_size(lengths[a:b]) <= L for a, b in runs)


def _random_case(rng, T=30, N=12):
    sizes = rng.integers(0, 9, T)
    part_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    Q = int(part_off[-1])
    names = ["topic.%d-%s" % (t, "x" * int(rng.integers(0, 30))) for t in range(T)]
    part_id = np.concatenate([np.sort(rng.choice(1000, n, replace=False)) for n in sizes]).astype(np.int32)
    cur, new = util.random_wave_case(rng, Q, N)
    rep_off, cur_flat = util.cur_lists(cur)
    out, out_len = util.rows(new, 3)
    return names, part_off, part_id, rep_off, cur_flat, out, out_len, np.arange(1, N + 1)


@pytest.mark.parametrize("seed", range(4))
def test_parts_hold_every_wave_in_order_and_stay_within_the_limit(seed):
    rng = np.random.default_rng(10 + seed)
    case = _random_case(rng)
    for B, send in ((1, None), (3, None), (2, (list(range(1, 13)), 4)), (10 ** 6, None)):
        docs, wave, summ, st = models.wave_docs(*case, B, send=send)
        assert st == (0, 0, 0)
        smallest = max(len(models.document([r])) for d in docs for r in _records(d))
        for L in (smallest, smallest + 57, 700, 2000, max(len(d) for d in docs)):
            parts, part_wave, p_wave, p_summ, p_st = part_models.wave_parts(*case, B, L, send=send)
            assert p_st == (0, 0, 0) and np.array_equal(p_wave, wave) and p_summ == summ
            assert part_wave == sorted(part_wave) and set(part_wave) == set(range(1, len(docs) + 1))
            assert all(len(p) <= L for p in parts)
            for v, doc in enumerate(docs, 1):
                mine = [json.loads(p) for p, pv in zip(parts, part_wave) if pv == v]
                assert all(m["version"] == 1 and m["partitions"] for m in mine)
                # joined, a wave's parts are its records in order; a part and the next part's first record exceed L
                assert [r for m in mine for r in m["partitions"]] == json.loads(doc)["partitions"]
                for a, b in zip(mine, mine[1:]):
                    assert len(models.document([json.dumps(r, separators=(",", ":")) for r in a["partitions"] + b["partitions"][:1]])) > L
            assert len(parts) >= len(docs)


def _records(doc):
    return [json.dumps(r, separators=(",", ":")) for r in json.loads(doc)["partitions"]]


def test_exact_size_keeps_a_part_whole_and_one_byte_less_cuts_it():
    rng = np.random.default_rng(3)
    case = _random_case(rng)
    docs = models.wave_docs(*case, 10 ** 6)[0]
    assert len(docs) == 1
    whole = len(docs[0])
    parts, part_wave, _, _, _ = part_models.wave_parts(*case, 10 ** 6, whole)
    assert parts == docs and part_wave == [1]
    parts, part_wave, _, _, _ = part_models.wave_parts(*case, 10 ** 6, whole - 1)
    assert len(parts) == 2 and part_wave == [1, 1]
    assert len(parts[0]) <= whole - 1 and len(parts[0]) + len(parts[1]) - 29 + 1 == whole


def test_a_limit_above_every_wave_gives_the_wave_documents():
    rng = np.random.default_rng(4)
    case = _random_case(rng)
    for B in (1, 2, 5):
        docs, wave, summ, _ = models.wave_docs(*case, B)
        parts, part_wave, p_wave, p_summ, _ = part_models.wave_parts(*case, B, max(len(d) for d in docs))
        assert parts == docs and part_wave == list(range(1, len(docs) + 1)) and p_summ == summ


def test_over_long_rows_and_plan_errors():
    cur = [[1], [2], [3], [4]]
    new = [[5], [1, 2, 3], [6, 7, 8, 9], [3]]
    rep_off, cur_flat = util.cur_lists(cur)
    out, out_len = util.rows(new)
    case = (["abc"], np.array([0, 4]), None, rep_off, cur_flat, out, out_len, np.arange(1, 20))
    lens = [29 + len(models.record("abc", g, new[g])) for g in range(4)]
    # the lowest over-long row, with its one-record document's length
    assert part_models.wave_parts(*case, 10, max(lens) - 1)[4] == (LIMIT, 2, lens[2])
    assert part_models.wave_parts(*case, 10, min(lens) - 1)[4] == (LIMIT, 0, lens[0])
    assert part_models.wave_parts(*case, 10, max(lens))[4] == (0, 0, 0)
    # the plan's own errors come first
    bad = util.rows([[5, 5], [1], [1], [1]])
    assert part_models.wave_parts(*case[:5], *bad, case[7], 10, 1)[4] == (BAD, 0, 5)
    # nothing changed: no part
    same = util.rows(cur)
    assert part_models.wave_parts(*case[:5], *same, case[7], 10, 100)[:2] == ([], [])


# ---- the C ABI --------------------------------------------------------------------------------------------------------------

def test_symbols_are_exported_and_declared(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    header = open(os.path.join(ROOT, "include", "kassign.h")).read()
    for name, n_args in (("ka_plan_waves_json_parts", 24), ("ka_plan_waves_send_json_parts", 28)):
        assert hasattr(raw, name)
        res, args = _native.SYMBOLS[name]
        assert res is ctypes.c_int32 and len(args) == n_args
        assert "int32_t %s(ka_ctx* ctx," % name in header


def test_without_a_context_is_no_device(native_lib):
    L = native_lib
    st = kab.KaStatus()
    n, d = ctypes.c_int32(5), ctypes.c_int32(6)
    args = (None, 0, None, None, None, None, 1, None, None, None, 1, None, None, None, 0, 100, None, None, ctypes.byref(d), None,
            ctypes.byref(n), None, 0)
    assert L.ka_plan_waves_json_parts(*args, ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE
    assert st.code == _native.KA_ERR_NO_DEVICE and n.value == 0 and d.value == 0
    assert L.ka_plan_waves_json_parts(*args, None) == BAD
    n.value, d.value = 5, 6
    send_args = args[:11] + (0, None, 1) + args[11:22] + (None, 0)
    assert L.ka_plan_waves_send_json_parts(*send_args, ctypes.byref(st)) == _native.KA_ERR_NO_DEVICE
    assert n.value == 0 and d.value == 0


class FakePartsLib(util.FakeWaveLib):
    """FakeWaveLib with the two _parts entry points: records what each call is handed; writes D = 2 W parts (2 W <= Q), part d as b"[d]"
    of wave 1 + d // 2; or, with `fail` = (code, a, b), refuses the call with that status."""

    def __init__(self, W, fail=None):
        super().__init__(W)
        self.fail = fail

    def _parts(self, T, part_off, part_id, names, name_off, js, json_cap, L, doc_off, doc_wave, n_docs, st):
        Q, text = self._docs(T, part_off, part_id, names, name_off, js, json_cap, doc_off)
        text.update(L=L, doc_wave=doc_wave is not None)
        if self.fail:
            return Q, text, False
        D = 2 * self.W
        buf, off, dw = writable(js, json_cap), util.writable(doc_off, Q + 1, np.int64), util.writable(doc_wave, Q, np.int32)
        at = 0
        for d in range(D):
            p = b"[%d]" % d
            off[d] = at
            buf[at:at + len(p)] = np.frombuffer(p, dtype=np.uint8)
            at += len(p)
            dw[d] = 1 + d // 2
        off[D] = at
        n_docs._obj.value = D
        return Q, text, True

    def _refuse(self, st, n_waves, n_docs):
        st._obj.code, st._obj.a, st._obj.b = self.fail
        n_waves._obj.value = n_docs._obj.value = 0
        return self.fail[0]

    def ka_plan_waves_json_parts(self, h, T, part_off, part_id, rep_off, cur, stride, new_len, new_broker, weight, B, names,
                                 name_off, js, json_cap, L, doc_off, doc_wave, n_docs, wave, n_waves, summary, cap, st):
        Q, text, ok = self._parts(T, part_off, part_id, names, name_off, js, json_cap, L, doc_off, doc_wave, n_docs, st)
        self.calls.append(dict(self._rows(Q, rep_off, cur, stride, new_len, new_broker, weight, B, wave), **text, cap=cap))
        return self._fill(Q, wave, n_waves, summary, None, cap, st) if ok else self._refuse(st, n_waves, n_docs)

    def ka_plan_waves_send_json_parts(self, h, T, part_off, part_id, rep_off, cur, stride, new_len, new_broker, weight, B, n_send,
                                      send_id, C, names, name_off, js, json_cap, L, doc_off, doc_wave, n_docs, wave, n_waves,
                                      summary, send_summary, cap, st):
        Q, text, ok = self._parts(T, part_off, part_id, names, name_off, js, json_cap, L, doc_off, doc_wave, n_docs, st)
        self.calls.append(dict(self._rows(Q, rep_off, cur, stride, new_len, new_broker, weight, B, wave), **text,
                               send_id=util.view(send_id, n_send, np.int32), C=C, cap=cap))
        return self._fill(Q, wave, n_waves, summary, send_summary, cap, st) if ok else self._refuse(st, n_waves, n_docs)


def writable(p, n):
    return util.writable(p, n, np.uint8)


def _inputs():
    out, out_len = util.rows([[1, 2], [3], [4, 5, 6], []])
    rep_off, cur = util.cur_lists([[1], [2, 3], [4], [7, 8]])
    return ["alpha", "", "bc"], [0, 3, 3, 4], [4, 9, -2, 0], rep_off, cur, out, out_len


def test_plan_wave_parts_json_marshals_its_arguments():
    lib = FakePartsLib(2)
    s = util.fake_solver(lib)
    names, part_off, part_id, rep_off, cur, out, out_len = _inputs()
    weight = np.array([5, 0, 7, 1], dtype=np.int64)
    parts, part_wave, wave, summ, st = s.plan_wave_parts_json(names, part_off, part_id, rep_off.astype(np.int32), cur.astype(np.int64),
                                                              out, out_len, 9, 1 << 20, weight=weight)
    assert st.code == 0 and len(lib.calls) == 1
    c = lib.calls[0]
    assert c["T"] == 3 and c["stride"] == 3 and c["B"] == 9 and c["cap"] == 4 and c["L"] == 1 << 20 and c["doc_wave"]
    assert c["part_off"].tolist() == part_off and c["part_id"].tolist() == part_id
    assert np.array_equal(c["rep_off"], rep_off) and np.array_equal(c["cur"], cur) and np.array_equal(c["weight"], weight)
    assert c["names"] == b"alphabc" and c["json_cap"] == models.json_bound(names, part_off, 3)
    assert [bytes(p) for p in parts] == [b"[%d]" % d for d in range(4)] and part_wave.tolist() == [1, 1, 2, 2]
    assert wave.tolist() == [1, 2, 1, 2] and [list(x) for x in summ] == [[v * 10 + f for f in range(5)] for v in range(2)]
    assert summ.dtype == WAVE_SUMMARY_DTYPE
    # a sender budget takes the _send form; a caller's buffer is used as given
    buf = np.zeros(64, dtype=np.uint8)
    parts, part_wave, _, summ, st = s.plan_wave_parts_json(names, part_off, None, rep_off, cur, out, out_len, 2, 1000, json_buf=buf,
                                                           max_broker_out=7, send_brokers=[1, 2, 3])
    c = lib.calls[-1]
    assert c["C"] == 7 and c["send_id"].tolist() == [1, 2, 3] and c["json_cap"] == 64 and c["L"] == 1000 and c["part_id"] is None
    assert summ.dtype == WAVE_SEND_SUMMARY_DTYPE and summ["max_broker_out"].tolist() == [5, 15]
    assert bytes(buf[:6]) == b"[0][1]" and parts[1].base is buf
    with pytest.raises(ValueError):
        s.plan_wave_parts_json(names, part_off, None, rep_off, cur, out, out_len, 2, 1000, max_broker_out=7)


@pytest.mark.parametrize("fail", [(BAD, 0, 0), (LIMIT, 2, 123), (LIMIT, 4000, 0)])
def test_a_refused_call_gives_empty_results_and_its_status(fail):
    s = util.fake_solver(FakePartsLib(3, fail))
    names, part_off, part_id, rep_off, cur, out, out_len = _inputs()
    for send in ({}, dict(max_broker_out=7, send_brokers=[1, 2])):
        parts, part_wave, wave, summ, st = s.plan_wave_parts_json(names, part_off, part_id, rep_off, cur, out, out_len, 9, 0, **send)
        assert (st.code, st.a, st.b) == fail
        assert parts == [] and len(part_wave) == len(wave) == len(summ) == 0
