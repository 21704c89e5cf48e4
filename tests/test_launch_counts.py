"""The work every solve entry point enqueues, pinned: kernel launches per call at fixed shapes, and the per-phase timings
each entry point reports with timing on. A change to a launch count is a change of schedule (more or fewer kernels,
sub-blocks or JSON passes), so it has to be deliberate."""
import os
from unittest import mock

import pytest

import kafka_assigner_b200 as kab

pytestmark = pytest.mark.gpu

# launches of ONE call of each entry point on BASELINE config 2 (1000 topics x 64 partitions, RF 3, 100 brokers: capacity 2,
# so conflict levels and level tables; rows of 3, so per-slot chains cut into topic sub-blocks). Recorded by running this
# module as a script (`python -m tests.test_launch_counts` on a GPU) with the host code as it was before the solve entry points
# shared one driver; a deliberate schedule change re-records them the same way.
EXPECTED_LAUNCHES = {"ragged": 6, "dense_host": 24, "dense_host_pipelined3": 21, "dense_device": 24, "dense_json": 45,
                     "staged_order": 24, "staged_slots_emit": 18}


def _device_inputs(cl):
    import torch
    d = dict(hash=torch.from_numpy(cl.topic_hash).cuda(), cur=torch.from_numpy(cl.cur).cuda(),
             out=torch.empty((cl.T, cl.P, cl.RF), dtype=torch.int32, device="cuda"),
             len=torch.empty((cl.T, cl.P), dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    return d


def _ragged(s, cl):
    part_off, part_id, rep_off, cur = cl.ragged()
    return s.solve_ragged(cl.topic_hash, part_off, part_id, rep_off, cur, -1, cl.RF)[2].code


def _dense_host(s, cl):
    return s.solve_dense(cl.topic_hash, cl.cur)[2].code


def _dense_host_pipelined(s, cl):
    with mock.patch.dict(os.environ, {"KA_PIPELINE_STAGES": "3"}):
        return s.solve_dense(cl.topic_hash, cl.cur)[2].code


def _dense_device(s, cl):
    d = _device_inputs(cl)
    return s.solve_dense_device(cl.T, d["hash"].data_ptr(), cl.P, cl.RF, d["cur"].data_ptr(), -1, cl.RF, d["len"].data_ptr(),
                                d["out"].data_ptr()).code


def _dense_json(s, cl):
    return s.solve_dense_json(cl.topic_names, cl.topic_hash, cl.cur)[1].code


def _staged_order(s, cl):
    d = _device_inputs(cl)
    s.stage_dense_device(cl.T, d["hash"].data_ptr(), cl.P, cl.RF, d["cur"].data_ptr(), -1, cl.RF)
    return s.order_device(d["len"].data_ptr(), d["out"].data_ptr()).code


def _staged_slots_emit(s, cl):
    d = _device_inputs(cl)
    s.stage_dense_device(cl.T, d["hash"].data_ptr(), cl.P, cl.RF, d["cur"].data_ptr(), -1, cl.RF)
    assert s.staged_slot_chains() == 2
    s.order_slot_device(0)
    s.order_slot_device(1)
    return s.emit_device(d["len"].data_ptr(), d["out"].data_ptr()).code


ENTRY_POINTS = {"ragged": _ragged, "dense_host": _dense_host, "dense_host_pipelined3": _dense_host_pipelined,
                "dense_device": _dense_device, "dense_json": _dense_json, "staged_order": _staged_order,
                "staged_slots_emit": _staged_slots_emit}


def measure(name):
    """(launches of one call, last_timing()) of entry point `name` on a fresh, timed context."""
    cl = kab.synth.make_config("c2", "mixed")
    s = kab.Solver(0)
    s.set_brokers(cl.broker_id, cl.rack_index)
    s.set_timing(True)
    n0 = s.launch_count()
    assert ENTRY_POINTS[name](s, cl) == 0, name
    return s.launch_count() - n0, s.last_timing()


@pytest.mark.parametrize("name", sorted(ENTRY_POINTS))
def test_launches_and_timing_per_entry_point(native_lib, name):
    launches, tm = measure(name)
    assert launches == EXPECTED_LAUNCHES[name]
    assert tm["total_ms"] > 0 and tm["sticky_spread_ms"] > 0, tm


if __name__ == "__main__":
    print({name: measure(name)[0] for name in sorted(ENTRY_POINTS)})
