"""ka_solve_dense_candidates_device without a device: a NULL context is KA_ERR_NO_DEVICE, reported for every candidate."""
import ctypes

import numpy as np
import pytest

import kafka_assigner_b200 as kab
from tests import util


@pytest.mark.skipif(util.has_gpu(), reason="only meaningful on a box without a GPU")
def test_candidates_without_a_context_is_no_device(native_lib):
    st = (kab.KaStatus * 2)()
    cand_off = np.array([0, 1, 2], dtype=np.int32)
    ids = np.array([1, 2], dtype=np.int32)
    racks = np.zeros(2, dtype=np.int32)
    vp = ctypes.c_void_p
    rc = native_lib.ka_solve_dense_candidates_device(None, 2, cand_off.ctypes.data_as(vp), ids.ctypes.data_as(vp),
                                                     racks.ctypes.data_as(vp), 0, None, 0, 1, None, -1, 1, None, None, None, st)
    assert rc == st[0].code == st[1].code == kab._native.KA_ERR_NO_DEVICE
