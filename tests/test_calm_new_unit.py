"""The calm loop's one-pod new gang (leanNew1 in csrc/hived_lean.inc) against the general loop, at each unit shape and
each hand-over.

The traces run on C3's tree (B200 leaves, halves of 4, nodes of 8, racks of 32 nodes), one VC of two racks per CTA,
and reach: a leaf unit below a bound half and below a bound node; a 4-GPU half directly under a bound node and below a
new node; an 8-GPU node unit directly under the bound rack (the unit at the view level); the first gang of a
preassigned cell (nothing above the unit bound: a hand-over); pods of 2 GPUs whose leaves are single units; a dirty
list longer than 32 nodes; and a result pool too small for the batch.  The comparison is test_calm_loop's: every
record, the pool, the state snapshot, the counters and the oracle's hash."""
import ctypes as C

import numpy as np
import pytest

from conftest import snapshot_bytes
from hivedscheduler_b200 import _cabi, config, trace
from test_calm_loop import PC_CALM, _check, _path_counters

ERR_CAPACITY = 102  # HIVED_ERR_CAPACITY (include/hived.h)
LEVELS = [("HALF", "B200", 4), ("NODE", "HALF", 2), ("RACK", "NODE", 32), ("POD", "RACK", 16)]


def _trace(name, ops, n_vcs=2):
    """ops: ("s", group, vc, leaf_num) / ("d", group, vc, leaf_num); every gang is one pod."""
    tb = trace.TraceBuilder(len(ops) + 16)
    for op, g, v, k in ops:
        if op == "s":
            tb.schedule(group=g, vc=v, priority=0, leaf_type=0, leaf_num=k, pod_num=1, first=True)
        else:
            tb.delete_allocated(g, k, 0, vc=v)
    ev, dec = tb.finish()
    cfg = config._synthetic(LEVELS, 1, "NODE", {"vc%d" % i: [("POD.RACK", 2)] for i in range(n_vcs)}, "n%04d")
    n_groups = 1 + max(g for _, g, _, _ in ops)
    return {"name": name, "config": cfg, "events": ev, "decision": dec, "n_groups": n_groups, "n_pods": tb.next_pod,
            "max_group_leaves": 64, "max_group_pods": 8}


def unit_shapes():
    """Per VC: the first gang of the preassigned rack (hand-over), then a leaf below the bound half, a half directly
    under the bound node, a node directly under the bound rack, a 2-GPU pod (leaf units), a half and a leaf in new
    nodes below the bound rack once the used nodes are full, then a churn of 1 / 2 / 4 / 8-GPU pods with releases."""
    ops, g = [], 0
    rng = trace.XorShift64Star(trace.seed_for(23))
    alive = [[], []]
    for v in range(2):
        for k in (1, 1, 4, 8, 2, 1, 1, 8, 4, 1, 2, 4, 8, 8, 1):
            ops.append(("s", g, v, k)); alive[v].append((g, k)); g += 1
    for _ in range(600):
        v = rng.below(2)
        if alive[v] and rng.below(100) < 45:
            og, ok = alive[v].pop(rng.below(len(alive[v])))
            ops.append(("d", og, v, ok))
        else:
            k = (1, 2, 4, 8)[rng.below(4)]
            ops.append(("s", g, v, k)); alive[v].append((g, k)); g += 1
    return _trace("unit-shapes", ops)


def long_dirty_list():
    """40 node gangs released one after the other leave 40 dirty view nodes before the next new gang (the general
    sort); then leaf and half gangs."""
    ops = [("s", g, 0, 8) for g in range(41)]
    ops += [("d", g, 0, 8) for g in range(1, 41)]
    ops += [("s", 41 + i, 0, (1, 4, 1, 8)[i % 4]) for i in range(20)]
    return _trace("long-dirty-list", ops, n_vcs=1)


@pytest.mark.parametrize("name", ["unit-shapes", "long-dirty-list"])
def test_calm_new_unit_matches_general_loop(simt_lib, oracle_lib, monkeypatch, name):
    t = {"unit-shapes": unit_shapes, "long-dirty-list": long_dirty_list}[name]()
    _check(simt_lib, oracle_lib, t, monkeypatch)


def _run_small_pool(lib, t, monkeypatch, calm, words):
    monkeypatch.setenv("HIVED_NO_CALM", "0" if calm else "1")
    monkeypatch.delenv("HIVED_NCTA", raising=False)
    bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
    try:
        bc.set_all_nodes_healthy()
        ev = np.ascontiguousarray(t["events"])
        res = np.zeros(len(ev), dtype=trace.RESULT_DT)
        pool = np.zeros(words, dtype=np.int32)
        rc = lib.hived_process_events(bc.ctx, ev.ctypes.data_as(C.POINTER(_cabi.Event)), len(ev), None, 0,
                                      res.ctypes.data_as(C.POINTER(_cabi.Result)),
                                      pool.ctypes.data_as(C.POINTER(C.c_int32)), words)
        return rc, res, pool, bc.stats(), snapshot_bytes(lib, bc.ctx), _path_counters(lib, bc.ctx)
    finally:
        bc.close()


def test_calm_new_unit_pool_too_small(simt_lib, monkeypatch):
    """A pool that runs out part-way: the records past that point carry HIVED_ERR_CAPACITY, the same in both loops."""
    t = unit_shapes()
    on = _run_small_pool(simt_lib, t, monkeypatch, True, 3 * 8 * 20)
    off = _run_small_pool(simt_lib, t, monkeypatch, False, 3 * 8 * 20)
    assert on[0] == off[0] != 0  # the call reports the exhausted pool
    assert (on[1]["error"] == ERR_CAPACITY).any()
    for i in range(len(on[1])):
        assert on[1][i].tobytes() == off[1][i].tobytes(), "event %d: %r != %r" % (i, on[1][i], off[1][i])
    assert on[2].tobytes() == off[2].tobytes()
    assert on[3] == off[3]
    assert on[4] == off[4]
    assert on[5][:PC_CALM] == off[5][:PC_CALM]
    assert on[5][PC_CALM] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["unit-shapes", "long-dirty-list"])
def test_calm_new_unit_matches_general_loop_gpu(cuda_lib, oracle_lib, monkeypatch, name):
    t = {"unit-shapes": unit_shapes, "long-dirty-list": long_dirty_list}[name]()
    _check(cuda_lib, oracle_lib, t, monkeypatch)
