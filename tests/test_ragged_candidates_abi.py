"""ka_solve_candidates without a device: the symbol is exported, a NULL context is KA_ERR_NO_DEVICE for every candidate; and
synth.ragged_decommission_tables reproduces make_ragged_cluster's live sets."""
import ctypes

import numpy as np

import kafka_assigner_b200 as kab


def test_symbol_is_exported(native_lib):
    raw = ctypes.CDLL(kab.lib_path())
    assert hasattr(raw, "ka_solve_candidates") and "ka_solve_candidates" in kab._native.SYMBOLS


def test_ragged_candidates_without_a_context_is_no_device(native_lib):
    st = (kab.KaStatus * 3)()
    cand_off = np.array([0, 1, 2, 2], dtype=np.int32)
    ids = np.array([1, 2], dtype=np.int32)
    racks = np.zeros(2, dtype=np.int32)
    vp = ctypes.c_void_p
    rc = native_lib.ka_solve_candidates(None, 3, cand_off.ctypes.data_as(vp), ids.ctypes.data_as(vp), racks.ctypes.data_as(vp), 0,
                                        None, None, None, None, None, -1, 1, None, None, st)
    assert rc == kab._native.KA_ERR_NO_DEVICE
    assert [st[k].code for k in range(3)] == [kab._native.KA_ERR_NO_DEVICE] * 3
    assert native_lib.ka_solve_candidates(None, 1, None, None, None, 0, None, None, None, None, None, -1, 1, None, None,
                                          None) == kab._native.KA_ERR_BAD_ARG   # st is required


def test_ragged_decommission_tables_match_make_ragged_cluster():
    fracs = (0.0, 0.01, 0.05, 0.2, 0.5)
    kw = dict(T=50, N=300, R=7, seed=9, rack_frac=0.6)
    base = kab.synth.make_ragged_cluster(**kw)
    tables = kab.synth.ragged_decommission_tables(base, fracs)
    assert len(tables) == len(fracs)
    for f, (ids, racks) in zip(fracs, tables):
        cl = kab.synth.make_ragged_cluster(remove_frac=f, **kw)
        assert np.array_equal(ids, cl.broker_id) and np.array_equal(racks, cl.rack_index), f
        assert len(ids) == 300 - int(round(f * 300))
    # the same cluster regenerated with a removal: the tables depend only on the seed and the removal rule
    removed = kab.synth.make_ragged_cluster(remove_frac=0.3, **kw)
    for a, b in zip(kab.synth.ragged_decommission_tables(removed, fracs), tables):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
