"""Topic names through every text path. The reference prints names with org.json 20131018's JSONObject.quote(), which rewrites
'"', '\\', '/' after '<', chars below 0x20 and those in [0x80, 0xA0) and [0x2000, 0x2100) of the name's UTF-16 code units. The
device emitters copy names verbatim, so they refuse every name with such a char (or a '/': ka_json_name_refused) and the
host emitters print it instead. One alphabet of names -- every ASCII byte, both org.json ranges at their edges, characters of
2, 3 and 4 UTF-8 bytes, the empty name -- goes through the nine device entry points, the CLI and the C++ mirror's host path;
every accepted text is compared byte for byte with models.quote over the oracle's rows, every refusal with models.device_refuses."""
import ctypes
import json
import subprocess

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from kafka_assigner_b200 import _native
from oracle import py_oracle as po
from tests import models, util

BAD, LIMIT = _native.KA_ERR_BAD_ARG, _native.KA_ERR_LIMIT

EDGES = ["\x7f", "\x80", "\x85", "\x9f", "\xa0", "\u1fff", "\u2000", "\u2013", "\u20ac", "\u20ff", "\u2100"]
WIDE = ["é", "日", "\uffff", "\U00010000", "\U0001F600", "\U0010FFFF"]
# every name of the alphabet: "t" + ch + "x" for every char, a few bare chars and runs, and the empty name
NAMES = list(dict.fromkeys(["t" + chr(c) + "x" for c in range(0x80)] + ["t" + ch + "x" for ch in EDGES + WIDE] +
                           ["é", "\U0001F600", "\u2013", "\x85", "/", "<", "a</b", "日\U0001F600é", ""]))
ACCEPTED = [n for n in NAMES if models.device_refuses(n) is None]
REFUSED = [n for n in NAMES if models.device_refuses(n) is not None]
IDS = np.arange(1, 7, dtype=np.int32)
RACKS = IDS % 3                                  # rack index per broker; the oracle's rack names are "k<index>"
PARTS = {0: [1, 2], 3: [2, 3], 7: [3, 1], 9: [4, 5], 12: [6, 1]}


def java_hash(names):
    """String.hashCode of every name, from the UTF-16 model (a name with a NUL has no ka_java_string_hash)."""
    return np.array([po.java_string_hash(n) for n in names], dtype=np.int32)


def problem(names):
    """(names, topic_hash, part_off, part_id, rep_off, cur): every name a topic on the lists of PARTS."""
    names, part_off, part_id, rep_off, cur = util.flatten([(n, PARTS) for n in names])
    return names, java_hash(names), part_off, part_id, rep_off, cur


def oracle_text(oracle, names, part_off, part_id, rep_off, cur, desired=-1):
    text, st = util.oracle_text(oracle, names, part_off, part_id, rep_off, cur, IDS, ["k%d" % r for r in RACKS], desired)
    assert st.code == 0
    return text


def solver():
    s = kab.Solver(0)
    s.set_brokers(IDS, RACKS)
    return s


def refused_status(st, name):
    assert (st.code, st.a) == (BAD, models.device_refuses(name)[1]), (name, util.fields(st))


# ---- CPU: the model, the rule, the hash -------------------------------------------------------------------------------

def test_quote_model_hand_worked():
    """Worked from org.json 20131018 JSONObject.quote: '/' only after '<'; \\b \\t \\n \\f \\r short; other units below 0x20
    and those in [0x80, 0xA0) and [0x2000, 0x2100) as \\u + 4 lowercase hex digits; U+007F, U+00A0, U+1FFF, U+2100 and
    non-BMP characters (two surrogates, outside both ranges) kept."""
    q = models.quote
    assert q("") == '""'
    assert q("a</b") == '"a<\\/b"' and q("a/b") == '"a/b"' and q("</") == '"<\\/"' and q("<\U0001F600/") == '"<\U0001F600/"'
    assert q('a"b\\c') == '"a\\"b\\\\c"'
    assert q("\b\t\n\f\r") == '"\\b\\t\\n\\f\\r"'
    assert q("\x00\x1f\x0b") == '"\\u0000\\u001f\\u000b"'
    assert q("\x7f") == '"\x7f"'
    assert q("\x80") == '"\\u0080"' and q("\x9f") == '"\\u009f"' and q("\xa0") == '"\xa0"'
    assert q("\u1fff") == '"\u1fff"' and q("\u2000") == '"\\u2000"' and q("\u2013") == '"\\u2013"'
    assert q("price\u20ac") == '"price\\u20ac"' and q("\u20ff") == '"\\u20ff"' and q("\u2100") == '"\u2100"'
    assert q("\U0001F600") == '"\U0001F600"' and q("eu\u2013west").encode() == b'"eu\\u2013west"'
    # the CURRENT ASSIGNMENT / rollback quote: the ASCII rewrites only
    k = models.kafka_quote
    assert k("a</b\t\"\\") == '"a<\\/b\\t\\"\\\\"' and k("\x80\u2013\u20ac") == '"\x80\u2013\u20ac"' and k("") == '""'


def test_device_rule_model_hand_worked():
    d = models.device_refuses
    assert d("ok.name-1_é日\U0001F600\x7f\xa0\u1fff\u2100") is None and d("") is None
    assert d("a/b") == ("/", 0x2F) and d("a<b") is None and d("x\x85\u2013") == ("\x85", 0x85)
    assert d("eu\u2013west") == ("\u2013", 0x2013) and d("t\x00x") == ("\x00", 0) and d('"') == ('"', 0x22)
    assert len(ACCEPTED) > 90 and len(REFUSED) > 40 and "" in ACCEPTED


def test_library_rule_equals_the_model_for_every_name(native_lib):
    """ka_json_name_refused, the rule of every _json entry point and of the C++ mirror, over each name's UTF-8 bytes."""
    for n in NAMES:
        b = n.encode()
        e = models.device_refuses(n)
        assert native_lib.ka_json_name_refused(b, len(b)) == (-1 if e is None else e[1]), n
    # only whole UTF-8 forms of the two ranges: a lead byte alone, or one followed by a byte outside them, passes
    for raw, exp in ((b"\xc2", -1), (b"\xc2\xa0", -1), (b"\xc2\x7f", -1), (b"\xe2\x80", -1), (b"\xe2\x84\x80", -1),
                     (b"\xe2\x83\xbf", 0x20FF), (b"a\xe2\x80\x80", 0x2000), (b"\xe2\x80\x2f", 0x2F), (b"a\x00b", 0)):
        assert native_lib.ka_json_name_refused(raw, len(raw)) == exp, raw
    assert native_lib.ka_json_name_refused(b"a/b", 1) == -1 and native_lib.ka_json_name_refused(None, 0) == -1


def test_hash_equals_the_utf16_model_for_every_name(native_lib):
    """String.hashCode over UTF-16 units: the hash that orders every topic's rows. A NUL would end the C string, so a name with
    one is refused rather than hashed as its prefix."""
    for n in NAMES:
        if "\0" in n:
            with pytest.raises(ValueError):
                kab.java_string_hash(n)
        else:
            assert kab.java_string_hash(n) == po.java_string_hash(n), n
    # a lone surrogate in its own 3-byte form (the CLI's reading of a lone \ud800 escape) hashes as that unit, as Java does
    assert native_lib.ka_java_string_hash(b"t\xed\xa0\x80x") == po.java_string_hash("t\ud800x")
    assert native_lib.ka_java_string_hash(b"\xed\xa0\xbd\xed\xb8\x80") == po.java_string_hash("\U0001F600")


# ---- CPU: the CLI's snapshot reader and its host emitters ---------------------------------------------------------------

@pytest.fixture(scope="module")
def cli(native_lib):
    return kab.build_mod.build_host()


def write_snapshot(path, names, ensure_ascii, racks=None):
    brokers = [dict(id=int(b), host="h%d" % b, port=9092, rack=(racks or {}).get(int(b), "k%d" % r)) for b, r in zip(IDS, RACKS)]
    parts = [dict(topic=n, partition=p, replicas=r) for n in names for p, r in sorted(PARTS.items())]
    path.write_bytes(json.dumps(dict(brokers=brokers, topics=names, partitions=parts), ensure_ascii=ensure_ascii).encode())
    return str(path)


def run_cli(cli, snap, mode):
    r = subprocess.run([cli, "--zk_string", "file:" + snap, "--mode", mode], capture_output=True, timeout=300)
    return r.returncode, r.stdout, r.stderr.decode(errors="replace")


def current_text(names):
    return '{"version":1,"partitions":[' + ",".join(models.current_record(n, p, r) for n in names for p, r in sorted(PARTS.items())) + ']}'


def test_cli_reads_both_snapshot_encodings_alike(cli, tmp_path):
    """json.dumps writes a character above U+FFFF as a surrogate pair with ensure_ascii, as raw UTF-8 without: both must read as
    the same name, so CURRENT ASSIGNMENT (Kafka's quote) is the same text, and the one the model prints."""
    names = [n for n in NAMES if "\0" not in n]
    outs = []
    for ea in (True, False):
        rc, out, err = run_cli(cli, write_snapshot(tmp_path / ("s%d.json" % ea), names, ea), "PRINT_CURRENT_ASSIGNMENT")
        assert rc == 0, err
        outs.append(out)
    assert outs[0] == outs[1] == ("CURRENT ASSIGNMENT:\n" + current_text(names) + "\n").encode()


def test_cli_broker_list_quotes_rack_names_as_org_json(cli, tmp_path):
    """PRINT_CURRENT_BROKERS prints free-form rack names through the org.json emitter."""
    alphabet = [n for n in NAMES if "\0" not in n]
    for k in range(0, len(alphabet), len(IDS)):
        racks = dict(zip(IDS.tolist(), alphabet[k:k + len(IDS)]))
        outs = []
        for ea in (True, False):
            rc, out, err = run_cli(cli, write_snapshot(tmp_path / ("b%d.json" % ea), [], ea, racks), "PRINT_CURRENT_BROKERS")
            assert rc == 0, err
            outs.append(out)
        exp = "[" + ",".join('{"rack":%s,"port":9092,"host":"h%d","id":%d}' % (models.quote(racks.get(int(b), "k%d" % r)), b, b)
                             for b, r in zip(IDS, RACKS)) + "]"
        assert outs[0] == outs[1] == ("CURRENT BROKERS:\n" + exp + "\n").encode(), k


def test_cli_refuses_a_topic_name_with_nul(cli, tmp_path):
    for ea in (True, False):
        rc, out, err = run_cli(cli, write_snapshot(tmp_path / "nul.json", ["ok", "t\0x"], ea), "PRINT_CURRENT_ASSIGNMENT")
        assert rc != 0 and out == b"" and "\\u0000" in err, err


def test_cli_keeps_a_lone_surrogate_in_its_3_byte_form(cli, tmp_path):
    snap = tmp_path / "lone.json"
    snap.write_text('{"brokers":[],"partitions":[{"topic":"t\\ud800x","partition":0,"replicas":[1]},'
                    '{"topic":"\\ud83d\\ude00\\ud800","partition":1,"replicas":[2]}]}')
    rc, out, err = run_cli(cli, str(snap), "PRINT_CURRENT_ASSIGNMENT")
    assert rc == 0, err
    assert out == (b'CURRENT ASSIGNMENT:\n{"version":1,"partitions":[{"topic":"t\xed\xa0\x80x","partition":0,"replicas":[1]},'
                   b'{"topic":"\xf0\x9f\x98\x80\xed\xa0\x80","partition":1,"replicas":[2]}]}\n')


# ---- GPU: the nine device entry points ------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_solve_json_and_dense_json_over_the_alphabet(native_lib, oracle):
    """ka_solve_json and ka_solve_dense_json: every accepted name in one call gives the oracle's rows in models.quote's text;
    every refused name gives KA_ERR_BAD_ARG with its code point, no text and untouched counters."""
    names, th, part_off, part_id, rep_off, cur = problem(ACCEPTED)
    exp = oracle_text(oracle, names, part_off, part_id, rep_off, cur)
    s, ref = solver(), solver()
    text, st = s.solve_ragged_json(names, th, part_off, part_id, rep_off, cur, -1, check=False)
    assert st.code == 0 and bytes(text).decode() == exp
    ref.solve_ragged(th, part_off, part_id, rep_off, cur, -1, 2)
    assert np.array_equal(s.counters(), ref.counters())
    # dense: every topic the partitions 0..4 of PARTS' lists
    dense_cur = np.array([[PARTS[p] for p in sorted(PARTS)]] * len(names), dtype=np.int32)
    d = solver()
    dtext, dst = d.solve_dense_json(names, th, dense_cur, check=False)
    d_off = np.arange(len(names) + 1, dtype=np.int64) * len(PARTS)
    d_id = np.tile(np.arange(len(PARTS), dtype=np.int32), len(names))
    assert dst.code == 0 and bytes(dtext).decode() == oracle_text(oracle, names, d_off, d_id, rep_off, cur)

    for bad in REFUSED:
        two = ["ok", bad]
        _, th2, po2, pi2, ro2, cu2 = problem(two)
        before, d_before = s.counters(), d.counters()
        text, st = s.solve_ragged_json(two, th2, po2, pi2, ro2, cu2, -1, check=False)
        refused_status(st, bad)
        assert len(text) == 0 and np.array_equal(s.counters(), before)
        dtext, dst = d.solve_dense_json(two, th2, dense_cur[:2], check=False)
        refused_status(dst, bad)
        assert len(dtext) == 0 and np.array_equal(d.counters(), d_before)


@pytest.mark.gpu
def test_clusters_json_one_cluster_per_name(native_lib, oracle):
    """ka_solve_clusters_json with one cluster per name of the alphabet: a refused cluster has its own status and no text, and
    every other cluster the oracle's text."""
    s = kab.Solver(0)
    for k0 in range(0, len(NAMES), 100):
        chunk = NAMES[k0:k0 + 100]
        fleet = [util.Member((IDS, RACKS), *problem([n])) for n in chunk]
        res = s.solve_clusters_json([m.entry() for m in fleet], [m.names for m in fleet])
        for m, n, (text, st) in zip(fleet, chunk, res):
            if models.device_refuses(n):
                refused_status(st, n)
                assert len(text) == 0
            else:
                assert st.code == 0 and bytes(text).decode() == oracle_text(oracle, m.names, m.part_off, m.part_id, m.rep_off, m.cur), n


def wave_case(names):
    """The ka_solve rows of `names` on a fresh table, as wave inputs: (names, part_off, part_id, rep_off, cur, out, out_len)."""
    names, th, part_off, part_id, rep_off, cur = problem(names)
    out, out_len, st = solver().solve_ragged(th, part_off, part_id, rep_off, cur, 2, 2)
    assert st.code == 0 and (out_len == 2).all()
    return names, part_off, part_id, rep_off, cur, out, out_len


FORMS = [dict(L=None), dict(L=None, C=2), dict(L=400), dict(L=400, C=2), dict(L=400, rollback=True), dict(L=400, rollback=True, C=2)]


@pytest.mark.gpu
@pytest.mark.parametrize("form", range(len(FORMS)))
def test_wave_documents_over_the_alphabet(native_lib, form):
    """The six ka_plan_waves*_json* forms: the accepted names give models.wave_documents' documents, parts and rollback
    documents; a refused name gives KA_ERR_BAD_ARG with its code point and no document."""
    kw = FORMS[form]
    s = solver()
    case = wave_case(ACCEPTED)
    docs = util.check_wave_documents(s, *case, 3, **kw)[0]
    assert len(docs) > 1
    L, rollback, C = kw.get("L"), kw.get("rollback", False), kw.get("C")
    send = {} if C is None else dict(max_broker_out=C, send_brokers=list(IDS))
    for bad in REFUSED:
        args = wave_case(["ok", bad]) + (3,)
        if L is None:
            got = s.plan_waves_json(*args, **send)
            assert got[0] == []
        elif not rollback:
            got = s.plan_wave_parts_json(*args, L, **send)
            assert got[0] == [] and len(got[1]) == 0
        else:
            got = s.plan_wave_parts_rollback_json(*args, L, **send)
            assert got[0] == [] and got[1] == []
        refused_status(got[-1], bad)


@pytest.mark.gpu
def test_refused_wave_call_writes_no_counts(native_lib):
    """On a refused name ka_plan_waves_json leaves *n_waves at 0 and ka_plan_waves_json_parts(_rollback) *n_docs at 0."""
    s = solver()
    names, part_off, part_id, rep_off, cur, out, out_len = wave_case(["ok", "eu\u2013west"])
    enc = np.frombuffer("".join(names).encode(), dtype=np.uint8)
    name_off = np.array([0, 2, 2 + len(names[1].encode())], dtype=np.int64)
    Q = len(out_len)
    js, back = np.zeros(4096, np.uint8), np.zeros(4096, np.uint8)
    doc_off, back_off, doc_wave, wave = (np.zeros(Q + 1, np.int64), np.zeros(Q + 1, np.int64), np.zeros(Q, np.int32),
                                         np.zeros(Q, np.int32))
    summary = np.zeros(Q, dtype=kab.assigner.WAVE_SUMMARY_DTYPE)
    rc, st, W = util.raw_plan_waves_json(s, 2, part_off, part_id, rep_off, cur, 2, out_len, out, None, 3, enc, name_off, js, js.size,
                                         doc_off, wave, summary, Q)
    assert rc == BAD and (st.code, st.a, W.value) == (BAD, 0x2013, 0)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    for rollback in (False, True):
        n_docs, n_waves, st = ctypes.c_int32(-7), ctypes.c_int32(-7), kab.KaStatus()
        head = (s._h, 2, p(part_off), p(part_id), p(rep_off), p(cur), 2, p(out_len), p(out), None, 3, p(enc), p(name_off), p(js),
                js.size, 400, p(doc_off), p(doc_wave), ctypes.byref(n_docs))
        tail = (p(wave), ctypes.byref(n_waves), p(summary), Q, ctypes.byref(st))
        if rollback:
            rc = s._L.ka_plan_waves_json_parts_rollback(*head, p(back), back.size, p(back_off), *tail)
        else:
            rc = s._L.ka_plan_waves_json_parts(*head, *tail)
        assert rc == BAD and (st.code, st.a, n_docs.value, n_waves.value) == (BAD, 0x2013, 0, 0), rollback


# ---- GPU: byte accounting where characters and bytes differ ----------------------------------------------------------------

MULTI = ["é", "日本", "\U0001F600", "mix-é日\U0001F600"]


@pytest.mark.gpu
def test_solve_json_buffer_fits_to_the_byte_with_multibyte_names(native_lib, oracle):
    names, th, part_off, part_id, rep_off, cur = problem(MULTI)
    exp = oracle_text(oracle, names, part_off, part_id, rep_off, cur).encode()
    assert len(exp) > len(exp.decode())
    s = solver()
    for cap, code in ((len(exp), 0), (len(exp) - 1, LIMIT)):
        s.reset()
        text, st = s.solve_ragged_json(names, th, part_off, part_id, rep_off, cur, -1, json_buf=np.zeros(cap, np.uint8), check=False)
        assert st.code == code and bytes(text) == (exp if code == 0 else b""), cap


@pytest.mark.gpu
def test_wave_buffers_and_cuts_count_bytes_with_multibyte_names(native_lib):
    """ka_plan_waves_json with json_cap exact and one short; the _parts forms with L at exactly one part's length (that part
    stays whole) and one byte less (the cut moves); the rollback text with back_cap exact and one short."""
    s = solver()
    case = wave_case(MULTI)
    docs = util.check_wave_documents(s, *case, 3)[0]
    total = sum(len(d) for d in docs)
    util.check_wave_documents(s, *case, 3, json_buf=np.zeros(total, np.uint8))
    st = s.plan_waves_json(*case, 3, json_buf=np.zeros(total - 1, np.uint8))[-1]
    assert st.code == LIMIT
    for rollback in (False, True):
        # one wave of every changed row (a budget above every row), one part under a limit above it: its longest side is L
        whole = util.check_wave_documents(s, *case, 100, L=100000, rollback=rollback)
        assert len(whole[0]) == 1
        longest = max(len(d) for d in whole[0] + (whole[1] or []))
        at = util.check_wave_documents(s, *case, 100, L=longest, rollback=rollback)
        below = util.check_wave_documents(s, *case, 100, L=longest - 1, rollback=rollback)
        assert len(at[0]) == 1 and len(below[0]) == 2, rollback
    docs, backs = util.check_wave_documents(s, *case, 3, L=300, rollback=True)[:2]
    assert len(docs) > 2 and any(len(bytes(b)) > len(bytes(b).decode()) for b in backs)
    back_total = sum(len(b) for b in backs)
    got = s.plan_wave_parts_rollback_json(*case, 3, 300, back_buf=np.zeros(back_total, np.uint8))
    assert got[-1].code == 0 and [bytes(b) for b in got[1]] == [bytes(b) for b in backs]
    got = s.plan_wave_parts_rollback_json(*case, 3, 300, back_buf=np.zeros(back_total - 1, np.uint8))
    assert got[-1].code == LIMIT and got[0] == []


# ---- GPU: the host emitters -----------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_cli_prints_org_json_text_for_every_name(native_lib, oracle, cli, tmp_path):
    """PRINT_REASSIGNMENT over the whole alphabet (the refused names through the host emitter), from a snapshot written with
    surrogate pairs and from one written in raw UTF-8: the same stdout, the model's CURRENT ASSIGNMENT and the oracle's rows
    in models.quote's text as NEW ASSIGNMENT."""
    names = [n for n in NAMES if "\0" not in n]
    _, _, part_off, part_id, rep_off, cur = problem(names)
    racks = dict(zip(IDS.tolist(), ["k%d" % r for r in RACKS]))
    exp = ("CURRENT ASSIGNMENT:\n" + current_text(names) + "\nNEW ASSIGNMENT:\n" +
           oracle_text(oracle, names, part_off, part_id, rep_off, cur) + "\n").encode()
    for ea in (True, False):
        rc, out, err = run_cli(cli, write_snapshot(tmp_path / ("r%d.json" % ea), names, ea, racks), "PRINT_REASSIGNMENT")
        assert rc == 0, err
        assert out == exp, ea
    # the accepted names alone: the device emitter's text
    _, _, part_off, part_id, rep_off, cur = problem(ACCEPTED)
    exp = ("CURRENT ASSIGNMENT:\n" + current_text(ACCEPTED) + "\nNEW ASSIGNMENT:\n" +
           oracle_text(oracle, ACCEPTED, part_off, part_id, rep_off, cur) + "\n").encode()
    for ea in (True, False):
        rc, out, err = run_cli(cli, write_snapshot(tmp_path / ("a%d.json" % ea), ACCEPTED, ea, racks), "PRINT_REASSIGNMENT")
        assert rc == 0 and out == exp, (ea, err)


@pytest.mark.gpu
def test_cpp_mirror_wave_documents_quote_every_refused_name(native_lib, tmp_path):
    """planWavesJson of the C++ mirror takes the host emitter for every refused name: each record prints models.quote."""
    kab.build_mod.build_host()
    lines = ["%s %s" % (n.encode().hex(), models.quote(n).encode().hex()) for n in REFUSED if "\0" not in n]
    path = tmp_path / "names.txt"
    path.write_text("\n".join(lines) + "\n")
    r = subprocess.run([kab.build_mod.HOST_WAVES_JSON_TEST, str(path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
