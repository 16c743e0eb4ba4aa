"""The device program at the sizes it branches on, against the oracle: node widths of 2, 32 (as 2 x 16 and 4 x 8), 33
and 64 leaves, fan-outs of 32, 33 and 64 above the node, chains of 7 (AS == LEAN_LV), 8 and 15 levels, gangs of 31, 32
and 33 lean-lane units, gangs of exactly hived_options_t's max_group_leaves / max_group_pods and one more, the
one-launch-per-call and resident per-call paths at their pool window and capacity edges, and the pool compaction of a
VC-parallel batch past one 1024-wide tile of block sums.

Every shape test also reads hived_bench_path_counters and asserts the path the shape exists for (the bucketed view,
the lean lane, or the general code), so that a shape that silently takes another path fails instead of passing parity
on the wrong code.  The 1-lane emulation runs the lean lane for single-unit gangs only (units > HIVED_WARPSZ falls
back); the SIMT emulation and the GPU run it for up to 32 units.

Config limits: the device library rejects more than MAX_NODE_LEAVES (64) leaves below one cluster-view node, more than
MAX_FANOUT (64) children per cell and chains of more than MAXL - 1 (15) levels with HIVED_ERR_CAPACITY.  The oracle
accepts all three: they are documented limits of the device program's fixed-size frames, not a parity property.
"""
import ctypes as C
import json
import os
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest

import fuzz_api
from conftest import ORACLE_LIB, snapshot_bytes
from hivedscheduler_b200 import _cabi, trace
from hivedscheduler_b200.config import _synthetic, to_spec_text

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# hived_dev.h PC_*: which path the scheduling passes, commits and deletes took
PC_FAST_VIEW, PC_GENERAL_VIEW, PC_FAST_COMMIT, PC_GENERAL_COMMIT, PC_FAST_DELETE, PC_GENERAL_DELETE = 0, 1, 4, 5, 6, 7
HIVED_ERR_CAPACITY = 102
SERVE_POOL_WINDOW = 16384  # hived_core.h: pool words the resident per-call kernel returns in its slot


def path_counters(lib, ctx):
    f = lib.hived_bench_path_counters
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    out = (C.c_int64 * 16)()
    n = f(ctx, out)
    return [int(x) for x in out[:n]]


def _hooks(lib):
    for hook in (lib.hived_debug_view_hash, lib.hived_debug_bookkeeping_hash):
        hook.restype = C.c_uint64
        hook.argtypes = [C.c_void_p]
    return lib


# ---------------------------------------------------------------------------------------------------------------------
# shapes

def shape_config(node, above, n_top, vcs):
    """One chain with leaf type GPU.  node: fan-outs of the levels inside a node, bottom-up ((16, 2): a node of two
    16-leaf cells); above: fan-outs of the levels above the node, bottom-up; n_top: top-level cells.  Cell type "Lk" is
    chain level k (GPU is level 1).  vcs: {vc: [(level, count)]}.  Returns (config, {level: leaves per cell})."""
    fan = list(node) + list(above)
    top = len(fan) + 1
    names, leaves = {1: "GPU"}, {1: 1}
    levels = []
    for i, f in enumerate(fan):
        lv = i + 2
        names[lv] = "L%d" % lv
        leaves[lv] = leaves[lv - 1] * f
        levels.append((names[lv], names[lv - 1], f))
    vc_cells = {v: [(".".join(names[x] for x in range(top, lv - 1, -1)), n) for lv, n in cells] for v, cells in vcs.items()}
    return _synthetic(levels, n_top, names[len(node) + 1], vc_cells, "n%04d"), leaves


# expect: "fast"     the bucketed view places the gangs and the lean lane commits and deletes them;
#         "general"  the full view pass on the worker warps and the general commit (no bucketed view at all);
#         "nolean"   the bucketed view may place, but every commit and delete takes the general code;
#         "units"    gangs of more than one unit: the lean lane on 32-lane builds, the general code on the 1-lane one.
SHAPES = {
    # 32-leaf nodes: bucket 32 of BK_STRIDE, the full 32-bit free mask
    "node32-2x16": dict(node=(16, 2), above=(4,), n_top=4, vcs={"vc0": [(4, 2)], "vc1": [(3, 3)]},
                        gangs=[(1, 1), (2, 1), (4, 1), (32, 1), (2, 4), (1, 8)], expect="fast"),
    "node32-4x8": dict(node=(8, 4), above=(4,), n_top=4, vcs={"vc0": [(4, 2)], "vc1": [(3, 3)]},
                       gangs=[(1, 1), (8, 1), (32, 1), (4, 2), (16, 1), (8, 4)], expect="fast"),
    # wider than 32 leaves: the general view pass, findLeafCellsInNode with up to 64 leaves.  Pods of 1-3 leaves or a
    # whole node: the reference's leaf search enumerates k-subsets of a node's free leaves in order until one has the
    # optimal affinity, so a mid-sized pod on a fragmented 64-leaf node takes minutes or more on every implementation
    "node33-3x11": dict(node=(11, 3), above=(4,), n_top=4, vcs={"vc0": [(4, 2)], "vc1": [(3, 3)]},
                        gangs=[(1, 1), (2, 1), (3, 1), (33, 1), (1, 4), (2, 3)], expect="general"),
    "node64-4x16": dict(node=(16, 4), above=(4,), n_top=4, vcs={"vc0": [(4, 2)], "vc1": [(3, 3)]},
                        gangs=[(1, 1), (2, 1), (3, 1), (64, 1), (1, 8), (2, 4)], expect="general"),
    "node2": dict(node=(2,), above=(8, 4), n_top=2, vcs={"vc0": [(4, 1)], "vc1": [(3, 2)]},
                  gangs=[(1, 1), (2, 1), (2, 4), (1, 3), (2, 8)], expect="fast"),
    # fan-out above the node: 32 is the widest child mask of the bucketed view, 33 and 64 fill the mapping frames
    "fanout32": dict(node=(8,), above=(32,), n_top=2, vcs={"vc0": [(3, 1)], "vc1": [(2, 16)]},
                     gangs=[(1, 1), (8, 1), (8, 4), (4, 2), (8, 32)], expect="fast"),
    "fanout33": dict(node=(4,), above=(33,), n_top=3, vcs={"vc0": [(3, 1)], "vc1": [(2, 20)]},
                     gangs=[(1, 1), (4, 1), (4, 8), (2, 2), (4, 33)], expect="general"),
    "fanout64": dict(node=(4,), above=(64,), n_top=3, vcs={"vc0": [(3, 1)], "vc1": [(2, 40)]},
                     gangs=[(1, 1), (4, 1), (4, 16), (2, 2), (4, 64)], expect="general"),
    # chain depth: 7 levels is AS == LEAN_LV, one more turns the lean lane off, 15 is MAXL - 1
    "depth7": dict(node=(2, 2), above=(2, 2, 2, 2), n_top=2, vcs={"vc0": [(7, 1)], "vc1": [(5, 2)]},
                   gangs=[(1, 1), (2, 1), (4, 1), (2, 2), (4, 4)], expect="fast"),
    "depth8": dict(node=(2, 2), above=(2, 2, 2, 2, 2), n_top=2, vcs={"vc0": [(8, 1)], "vc1": [(6, 2)]},
                   gangs=[(1, 1), (2, 1), (4, 1), (2, 2), (4, 4)], expect="nolean"),
    "depth15": dict(node=(2, 2), above=(2, 1, 1, 2, 1, 1, 1, 1, 1, 2, 1, 1), n_top=4,
                    vcs={"vc0": [(15, 2)], "vc1": [(12, 1)]}, gangs=[(1, 1), (2, 1), (4, 1), (2, 2), (4, 4)],
                    expect="nolean"),
    # gangs of 31, 32 and 33 lean-lane units (one leaf each) on 32-leaf nodes
    "units31": dict(node=(16, 2), above=(4,), n_top=4, vcs={"vc0": [(4, 2)], "vc1": [(3, 3)]}, gangs=[(1, 31)],
                    expect="units"),
    "units32": dict(node=(16, 2), above=(4,), n_top=4, vcs={"vc0": [(4, 2)], "vc1": [(3, 3)]}, gangs=[(1, 32)],
                    expect="units"),
    "units33": dict(node=(16, 2), above=(4,), n_top=4, vcs={"vc0": [(4, 2)], "vc1": [(3, 3)]}, gangs=[(1, 33)],
                    expect="nolean"),
}


def shape_limits(shape):
    """(max_group_leaves, max_group_pods) that every gang of the shape fits."""
    return max(64, max(k * m for k, m in shape["gangs"])), max(16, max(m for _, m in shape["gangs"]))


def shape_trace(name, n_gangs=60, opp_rate=0.0, n_bad=2):
    """A batch trace on the shape: guaranteed gangs of the shape's sizes under a per-VC admission window (chunk 1, every
    node healthy: the VC-parallel regime on the GPU), then n_bad nodes go bad and come back halfway through chunk 2
    (opp_rate: the share of opportunistic gangs in chunk 2).  t["split"] is the first event of chunk 2."""
    sh = SHAPES[name]
    cfg, leaves = shape_config(sh["node"], sh["above"], sh["n_top"], sh["vcs"])
    vcs = sorted(sh["vcs"])
    limit = [int(0.75 * sum(leaves[lv] * n for lv, n in sh["vcs"][v])) for v in vcs]
    n_nodes = sh["n_top"] * int(np.prod(sh["above"]))
    rng = random.Random(zlib.crc32(name.encode()))
    tb = trace.TraceBuilder(64 * n_gangs)
    alive = [[] for _ in vcs]
    used = [0] * len(vcs)
    split, bad = None, []
    g = 0
    for i in range(n_gangs):
        if i == n_gangs // 2:
            split = tb.n
            bad = rng.sample(range(n_nodes), n_bad)
            for nd in bad:
                tb.node_health(nd, False)
        if i == 3 * n_gangs // 4:
            for nd in bad:
                tb.node_health(nd, True)
        k, m = sh["gangs"][rng.randrange(len(sh["gangs"]))]
        v = rng.randrange(len(vcs))
        opp = i >= n_gangs // 2 and rng.random() < opp_rate
        if not opp:
            while used[v] + k * m > limit[v] and alive[v]:
                og, ok, om = alive[v].pop(0)
                for j in range(om):
                    tb.delete_allocated(og, ok, j, vc=v)
                used[v] -= ok * om
        for j in range(m):
            tb.schedule(group=g, vc=v, priority=-1 if opp else 0, leaf_type=0, leaf_num=k, pod_num=m, first=(j == 0))
        if not opp:
            alive[v].append((g, k, m))
            used[v] += k * m
        g += 1
    ev, dec = tb.finish()
    lmax, pmax = shape_limits(sh)
    return {"name": name, "config": cfg, "events": ev, "decision": dec, "n_groups": g, "n_pods": tb.next_pod,
            "max_group_leaves": lmax, "max_group_pods": pmax, "split": split}


def pool_words(events):
    sched = events[events["type"] == _cabi.EV_SCHEDULE]["spec"]
    leaves = (sched["member_leaf_num"][:, 0].astype(np.int64) * sched["member_pod_num"][:, 0]).sum()
    return int(3 * leaves + 64 * len(events) + 4096)


def replay(lib, t):
    """The trace in its two chunks; everything a caller can observe, plus the path counters where the library has them."""
    _hooks(lib)
    bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
    bc.set_all_nodes_healthy()
    ev = t["events"]
    chunks = []
    for a, b in ((0, t["split"]), (t["split"], len(ev))):
        res, pool = bc.process(ev[a:b], pool_words(ev[a:b]))
        chunks.append((res.tobytes(), pool.tobytes()))
    out = {"chunks": chunks, "hash": bc.result_hash(), "stats": bc.stats(), "cells": snapshot_bytes(lib, bc.ctx),
           "views": int(lib.hived_debug_view_hash(bc.ctx)), "books": int(lib.hived_debug_bookkeeping_hash(bc.ctx)),
           "kinds": np.concatenate([np.frombuffer(r, dtype=trace.RESULT_DT)["kind"] for r, _ in chunks])}
    out["paths"] = path_counters(lib, bc.ctx) if hasattr(lib, "hived_bench_path_counters") else None
    bc.close()
    return out


def check_paths(name, pc, lanes):
    expect = SHAPES[name]["expect"]
    if expect == "units":
        expect = "fast" if lanes == 32 else "nolean"
    msg = "%s on a %d-lane build: path counters %r" % (name, lanes, pc)
    if expect == "fast":
        assert pc[PC_FAST_VIEW] > 0 and pc[PC_FAST_COMMIT] > 0 and pc[PC_FAST_DELETE] > 0, msg
    elif expect == "general":
        assert pc[PC_FAST_VIEW] == 0 and pc[PC_FAST_COMMIT] == 0 and pc[PC_FAST_DELETE] == 0, msg
        assert pc[PC_GENERAL_VIEW] > 0 and pc[PC_GENERAL_COMMIT] > 0, msg
    else:
        assert pc[PC_FAST_COMMIT] == 0 and pc[PC_FAST_DELETE] == 0 and pc[PC_GENERAL_COMMIT] > 0, msg
        if SHAPES[name]["expect"] == "nolean":
            assert pc[PC_FAST_VIEW] > 0, msg  # placed by the bucketed view, committed by the general code


def shape_trace_parity(lib, oracle_lib, name, lanes):
    t = shape_trace(name)
    a, b = replay(lib, t), replay(oracle_lib, t)
    for i, ((ra, pa), (rb, pb)) in enumerate(zip(a["chunks"], b["chunks"])):
        assert ra == rb, "%s chunk %d: results differ" % (name, i)
        assert pa == pb, "%s chunk %d: pool differs" % (name, i)
    for key in ("hash", "stats", "cells", "views", "books"):
        assert a[key] == b[key], "%s: %s differ" % (name, key)
    sched = t["events"]["type"] == _cabi.EV_SCHEDULE
    assert (a["kinds"][sched] == _cabi.KIND_BIND).sum() > sched.sum() // 3, name  # placements, not only waits
    check_paths(name, a["paths"], lanes)


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_shape_trace_emu(emu_lib, oracle_lib, name):
    shape_trace_parity(emu_lib, oracle_lib, name, 1)


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_shape_trace_simt(simt_lib, oracle_lib, name):
    shape_trace_parity(simt_lib, oracle_lib, name, 32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_shape_trace_cuda(cuda_lib, oracle_lib, name):
    shape_trace_parity(cuda_lib, oracle_lib, name, 32)


# ---- regression: the lean delete of a multi-unit gang while some node is bad

def lean_delete_with_bad_node(lib):
    """A gang of one 4-leaf pod on 32-leaf nodes (4 leaf units, committed by the lean lane once a first gang has bound
    the VC's preassigned cell), then an unrelated node goes bad, then the pod is deleted.  leanDeleteMulti compares the units' preassigned cells when any node is bad; its
    shuffle ran in the lanes of a unit only (`act && pre != hv_shfl(pre, 0)`), a warp collective without lanes 4-31 (the
    SIMT emulation hung on it, the shape traces' bad-node chunk found it)."""
    cfg, _ = shape_config((16, 2), (4,), 4, {"vc0": [(4, 2)], "vc1": [(3, 3)]})
    bc = trace.BatchContext(lib, cfg, 16, 64, 64, 16)
    bc.set_all_nodes_healthy()
    tb = trace.TraceBuilder(8)
    tb.schedule(group=2, vc=0, priority=0, leaf_type=0, leaf_num=1, pod_num=1)  # binds vc0's preassigned cell
    tb.schedule(group=0, vc=0, priority=0, leaf_type=0, leaf_num=4, pod_num=1)
    tb.node_health(15, False)
    tb.delete_allocated(0, 4, 0, vc=0)
    tb.schedule(group=1, vc=0, priority=0, leaf_type=0, leaf_num=4, pod_num=1)
    ev, _ = tb.finish()
    out = []
    for i in range(len(ev)):  # one call per event: the per-call path
        res, pool = bc.process(ev[i:i + 1], 4096)
        out.append((res.tobytes(), pool.tobytes()))
    out.append(snapshot_bytes(lib, bc.ctx))
    out.append(int(_hooks(lib).hived_debug_bookkeeping_hash(bc.ctx)))
    pc = path_counters(lib, bc.ctx) if hasattr(lib, "hived_bench_path_counters") else None
    bc.close()
    return out, pc


def test_lean_delete_with_bad_node_simt(simt_lib, oracle_lib):
    got, pc = lean_delete_with_bad_node(simt_lib)
    assert got == lean_delete_with_bad_node(oracle_lib)[0]
    assert pc[PC_FAST_COMMIT] >= 1 and pc[PC_FAST_DELETE] == 1, pc


@pytest.mark.gpu
def test_lean_delete_with_bad_node_cuda(cuda_lib, oracle_lib):
    got, pc = lean_delete_with_bad_node(cuda_lib)
    assert got == lean_delete_with_bad_node(oracle_lib)[0]
    assert pc[PC_FAST_COMMIT] >= 1 and pc[PC_FAST_DELETE] == 1, pc


# ---- the API fuzz on every shape

def shape_fixture(name):
    """The shape's cluster and 40 pod specs sized to it (its trace gangs, single leaves and whole nodes, 1-4 pods,
    a second member now and then, priorities -1..2, typed and untyped)."""
    sh = SHAPES[name]
    cfg, leaves = shape_config(sh["node"], sh["above"], sh["n_top"], sh["vcs"])
    lmax, pmax = shape_limits(sh)
    node_leaves = leaves[len(sh["node"]) + 1]
    # (the sizes of the trace only: see the comment above SHAPES' wide nodes on the cost of mid-sized pods)
    sizes = sorted({1, node_leaves} | {k for k, _ in sh["gangs"]})
    rng = random.Random(zlib.crc32(name.encode()) ^ 0x5eed)
    pss = {}
    for i in range(40):
        if i < len(sh["gangs"]):
            members = [{"leafCellNumber": sh["gangs"][i][0], "podNumber": sh["gangs"][i][1]}]
        else:
            members = [{"leafCellNumber": rng.choice(sizes), "podNumber": rng.choice([1, 1, 2, 3, 4])}]
            if rng.random() < 0.2:
                members.append({"leafCellNumber": rng.choice(sizes), "podNumber": rng.choice([1, 2])})
            while sum(m["leafCellNumber"] * m["podNumber"] for m in members) > lmax:
                members[0]["podNumber"] = 1
                members = members[:1]
        pss["spec%02d" % i] = {
            "affinityGroup": {"members": members, "name": "sg%d" % i}, "gangReleaseEnable": False,
            "ignoreK8sSuggestedNodes": rng.random() < 0.5, "lazyPreemptionEnable": rng.random() < 0.5,
            "leafCellNumber": members[0]["leafCellNumber"], "leafCellType": "GPU" if rng.random() < 0.7 else "",
            "pinnedCellId": "", "priority": rng.choice([-1, 0, 0, 1, 2]), "virtualCluster": rng.choice(sorted(sh["vcs"]))}
    return {"design_config": cfg, "pss": pss}, lmax, pmax


FUZZ_SEEDS = (1, 2, 3)


def shape_fuzz(lib, oracle_lib, name, filtering, monkeypatch, seeds=FUZZ_SEEDS):
    monkeypatch.setenv("FUZZ_FILTERING", "1" if filtering else "0")
    fx, lmax, pmax = shape_fixture(name)
    for seed in seeds:
        d = fuzz_api.run_seed(lib, oracle_lib, seed, 300, fx=fx, max_group_leaves=lmax, max_group_pods=pmax)
        assert d is None, "%s: %s" % (name, d)


# (the unit shapes are the 32-leaf cluster with one gang size; the oracle's leaf search over 64-leaf nodes takes over a
# minute per seed: that shape is covered by its trace)
FUZZ_SHAPES = sorted(n for n in SHAPES if not n.startswith("units") and n != "node64-4x16")


@pytest.mark.parametrize("filtering", [False, True], ids=["default", "filtering"])
@pytest.mark.parametrize("name", FUZZ_SHAPES)
def test_shape_fuzz_emu(emu_lib, oracle_lib, name, filtering, monkeypatch):
    shape_fuzz(emu_lib, oracle_lib, name, filtering, monkeypatch, seeds=FUZZ_SEEDS[:1])


@pytest.mark.gpu
@pytest.mark.parametrize("filtering", [False, True], ids=["default", "filtering"])
@pytest.mark.parametrize("name", FUZZ_SHAPES)
def test_shape_fuzz_cuda(cuda_lib, oracle_lib, name, filtering, monkeypatch):
    shape_fuzz(cuda_lib, oracle_lib, name, filtering, monkeypatch)


# ---- gangs of exactly max_group_leaves / max_group_pods, and one more

def _process_rc(lib, ctx, events, cap):
    """hived_process_events' return code, results and pool (no exception on a failing call)."""
    events = np.ascontiguousarray(events)
    res = np.zeros(len(events), dtype=trace.RESULT_DT)
    pool = np.zeros(max(cap, 1), dtype=np.int32)
    rc = lib.hived_process_events(ctx, events.ctypes.data_as(C.POINTER(_cabi.Event)), len(events), None, 0,
                                  res.ctypes.data_as(C.POINTER(_cabi.Result)), pool.ctypes.data_as(C.POINTER(C.c_int32)),
                                  cap)
    return rc, res, pool[:cap]


def group_capacity_answers(lib):
    """On the 32-leaf-node cluster with max_group_leaves = 64, max_group_pods = 8: the return code and results of a gang
    of exactly 64 leaves (2 x 32), exactly 8 pods (8 x 1), 65 leaves (13 x 5), 9 pods (9 x 1), one 64-leaf pod and one
    65-leaf pod, each alone in a fresh context."""
    cfg, _ = shape_config((16, 2), (4,), 4, {"vc0": [(4, 2)], "vc1": [(3, 3)]})
    out = []
    for k, m in ((32, 2), (1, 8), (13, 5), (1, 9), (64, 1), (65, 1)):
        bc = trace.BatchContext(lib, cfg, 64, 256, 64, 8)
        bc.set_all_nodes_healthy()
        tb = trace.TraceBuilder(16)
        for j in range(m):
            tb.schedule(group=1, vc=0, priority=0, leaf_type=0, leaf_num=k, pod_num=m, first=(j == 0))
        ev, _ = tb.finish()
        rc, res, pool = _process_rc(lib, bc.ctx, ev, 3 * k * m * m + 64)
        out.append((k, m, rc, res.tobytes() if rc == 0 else None, pool.tobytes() if rc == 0 else None))
        bc.close()
    return out


def _group_capacity(lib, oracle_lib):
    got, want = group_capacity_answers(lib), group_capacity_answers(oracle_lib)
    assert got == want
    # (64 x 1 is within the limits and waits: no 32-leaf node holds the pod)
    assert [rc for _, _, rc, _, _ in got] == [0, 0, HIVED_ERR_CAPACITY, HIVED_ERR_CAPACITY, 0, HIVED_ERR_CAPACITY]
    assert np.frombuffer(got[4][3], dtype=trace.RESULT_DT)["kind"][0] == _cabi.KIND_WAIT


def test_group_capacity_emu(emu_lib, oracle_lib):
    _group_capacity(emu_lib, oracle_lib)


def test_group_capacity_simt(simt_lib, oracle_lib):
    _group_capacity(simt_lib, oracle_lib)


@pytest.mark.gpu
def test_group_capacity_cuda(cuda_lib, oracle_lib):
    _group_capacity(cuda_lib, oracle_lib)


# ---- config limits: at the limit the device library creates and schedules, one past it hived_create refuses

LIMITS = {
    # name: (at the limit, one past it)
    "node-leaves": (dict(node=(16, 4), above=(2,), vcs={"vc0": [(4, 2)]}), dict(node=(13, 5), above=(2,), vcs={"vc0": [(4, 2)]})),
    "fan-out": (dict(node=(2,), above=(64,), vcs={"vc0": [(3, 2)]}), dict(node=(2,), above=(65,), vcs={"vc0": [(3, 2)]})),
    "levels": (dict(node=(2,), above=(2,) + (1,) * 12, vcs={"vc0": [(15, 2)]}),
               dict(node=(2,), above=(2,) + (1,) * 13, vcs={"vc0": [(16, 2)]})),
}


def _create(lib, cfg):
    opt = _cabi.Options(max_groups=64, max_pods=256, max_group_leaves=64, max_group_pods=8, device=0)
    ctx = C.c_void_p()
    rc = lib.hived_create(to_spec_text(cfg).encode(), C.byref(opt), C.byref(ctx))
    msg = (lib.hived_create_error() or b"").decode()
    if rc == 0:
        lib.hived_destroy(ctx)
    return rc, msg


def config_limit(lib, oracle_lib, name):
    at, over = LIMITS[name]
    cfg_over, _ = shape_config(over["node"], over["above"], 2, over["vcs"])
    rc, msg = _create(lib, cfg_over)
    assert rc == HIVED_ERR_CAPACITY and msg, (name, rc, msg)
    assert _create(oracle_lib, cfg_over)[0] == 0  # the oracle has no such limit
    cfg_at, leaves = shape_config(at["node"], at["above"], 2, at["vcs"])
    answers = []
    for lb in (lib, oracle_lib):
        bc = trace.BatchContext(lb, cfg_at, 64, 256, 64, 8)
        bc.set_all_nodes_healthy()
        tb = trace.TraceBuilder(8)
        node_leaves = leaves[len(at["node"]) + 1]
        tb.schedule(group=0, vc=0, priority=0, leaf_type=0, leaf_num=node_leaves, pod_num=1)
        tb.schedule(group=1, vc=0, priority=0, leaf_type=0, leaf_num=1, pod_num=2)
        tb.schedule(group=1, vc=0, priority=0, leaf_type=0, leaf_num=1, pod_num=2, first=False)
        tb.delete_allocated(0, node_leaves, 0, vc=0)
        ev, _ = tb.finish()
        res, pool = bc.process(ev, 4096)
        answers.append((res.tobytes(), pool.tobytes(), snapshot_bytes(lb, bc.ctx)))
        assert (res["kind"][:3] == _cabi.KIND_BIND).all(), name
        bc.close()
    assert answers[0] == answers[1], name


@pytest.mark.parametrize("name", sorted(LIMITS))
def test_config_limit_emu(emu_lib, oracle_lib, name):
    config_limit(emu_lib, oracle_lib, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(LIMITS))
def test_config_limit_cuda(cuda_lib, oracle_lib, name):
    config_limit(cuda_lib, oracle_lib, name)


# ---------------------------------------------------------------------------------------------------------------------
# per-call path edges (GPU): batches of <= 8 events go through bk_run_small — the resident kernel, or with
# HIVED_NO_RESIDENT=1 one launch per call with its own pinned stage — and 9 events through the batch path

def _window_cluster():
    """64-leaf nodes (4 x 16), 16 of them, all in one VC: a gang of 16 x 64 leaves fills the cluster."""
    return shape_config((16, 4), (4,), 4, {"vc0": [(4, 4)]})[0]


def _window_events(n_pods=8, extra_noop=False):
    """The first n_pods pods of a 16 x 64-leaf gang: every result carries the gang's 1024 leaves (3072 pool words), so
    8 of them need more than SERVE_POOL_WINDOW words; extra_noop appends a delete of an unknown group (a 9th event
    that emits nothing)."""
    tb = trace.TraceBuilder(16)
    for j in range(n_pods):
        tb.schedule(group=0, vc=0, priority=0, leaf_type=0, leaf_num=64, pod_num=16, first=(j == 0))
    if extra_noop:
        tb.delete_allocated(7, 64, 0, vc=0)
    return tb.finish()[0]


def window_answers(lib, events, caps):
    """For each pool capacity: (return code, results, pool) of the events in a fresh context."""
    out = []
    for cap in caps:
        bc = trace.BatchContext(lib, _window_cluster(), 16, 64, 1024, 16)
        bc.set_all_nodes_healthy()
        rc, res, pool = _process_rc(lib, bc.ctx, events, cap)
        out.append((rc, res.tobytes() if rc == 0 else None, pool.tobytes() if rc == 0 else None))
        bc.close()
    return out


def percall_checks(lib, oracle_lib, with_fuzz):
    """Returns a list of failures (empty: all good)."""
    bad = []
    ev8, ev9 = _window_events(), _window_events(extra_noop=True)
    used = 8 * 3 * 1024
    assert used > SERVE_POOL_WINDOW
    # 8 events (bk_run_small) and the same 8 plus a no-op (the batch path): same answers, pool above the window
    caps = [used, used - 1]
    a8, o8 = window_answers(lib, ev8, caps), window_answers(oracle_lib, ev8, caps)
    a9, o9 = window_answers(lib, ev9, caps), window_answers(oracle_lib, ev9, caps)
    if a8 != o8:
        bad.append("8 events: %r != oracle %r" % ([x[0] for x in a8], [x[0] for x in o8]))
    if a9 != o9:
        bad.append("9 events: %r != oracle %r" % ([x[0] for x in a9], [x[0] for x in o9]))
    if [x[0] for x in a8] != [0, HIVED_ERR_CAPACITY] or [x[0] for x in a9] != [0, HIVED_ERR_CAPACITY]:
        bad.append("capacity edge: %r / %r" % ([x[0] for x in a8], [x[0] for x in a9]))
    if a8[0][0] == 0 and a9[0][0] == 0:
        r8, r9 = np.frombuffer(a8[0][1], dtype=trace.RESULT_DT), np.frombuffer(a9[0][1], dtype=trace.RESULT_DT)
        if r8.tobytes() != r9[:8].tobytes() or a8[0][2] != a9[0][2]:
            bad.append("8 and 9 events answer differently")
        if int((r8["leaf_off"] + 3 * r8["n_leaves"]).max()) != used:
            bad.append("the 8 results do not use %d pool words" % used)
    # the small traces and (in the one-launch-per-call process) the API fuzz on a few shapes
    for t in (trace.trace_c1(), shape_trace("node64-4x16", n_gangs=40)):
        if "split" not in t:
            t["split"] = len(t["events"]) // 2
        ra, rb = replay(lib, t), replay(oracle_lib, t)
        if any(ra[k] != rb[k] for k in ("chunks", "hash", "stats", "cells", "views", "books")):
            bad.append("trace %s differs" % t["name"])
    if with_fuzz:
        for name in ("node32-2x16", "node33-3x11", "fanout64", "depth15"):
            fx, lmax, pmax = shape_fixture(name)
            for seed in (1, 2):
                d = fuzz_api.run_seed(lib, oracle_lib, seed, 300, fx=fx, max_group_leaves=lmax, max_group_pods=pmax)
                if d:
                    bad.append("%s: %s" % (name, d))
    return bad


@pytest.mark.gpu
def test_percall_resident_cuda(cuda_lib, oracle_lib):
    """The resident per-call kernel: its slot holds SERVE_POOL_WINDOW pool words, the rest comes by cudaMemcpy."""
    assert percall_checks(cuda_lib, oracle_lib, with_fuzz=False) == []


@pytest.mark.gpu
def test_percall_one_launch_cuda(oracle_lib):
    """HIVED_NO_RESIDENT=1 (a fresh process: the switch is read once per context's stream): every call of <= 8 events
    is one launch with the pinned stage of bk_run_small and its SMALL_POOL_WINDOW."""
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from hivedscheduler_b200 import _cabi\n"
            "import test_shape_limits as ts\n"
            "print(json.dumps(ts.percall_checks(_cabi.load_cuda_library(), _cabi.load_library(%r), True)))\n") % (
                ROOT, HERE, ORACLE_LIB)
    out = subprocess.check_output([sys.executable, "-c", code], env=dict(os.environ, HIVED_NO_RESIDENT="1"))
    assert json.loads(out.decode().strip().splitlines()[-1]) == []


# ---------------------------------------------------------------------------------------------------------------------
# pool compaction after a VC-parallel batch (GPU)

def _compaction_config():
    """16 VCs of one 64-leaf rack each (8 nodes x 8 leaves)."""
    return shape_config((4, 2), (8,), 16, {"vc%02d" % v: [(4, 1)] for v in range(16)})[0]


def compaction_events(n):
    """n SCHEDULE / DELETE events at one priority over 16 VCs: rounds of 16 gangs (one per VC, 1-3 pods of 1-4 leaves),
    each round deleting the gangs of four rounds before.  Group ids are reused per VC, never across VCs."""
    rounds = n // 16 + 8
    rng = np.random.default_rng(n)
    k = rng.choice(np.array([1, 2, 4], dtype=np.int32), size=(rounds, 16))
    m = rng.integers(1, 4, size=(rounds, 16), dtype=np.int32)
    slots = 8
    ev = np.zeros(rounds * 16 * 6, dtype=trace.EVENT_DT)
    pos = 0
    vc = np.arange(16, dtype=np.int32)
    for r in range(rounds):
        if r >= 4:
            old = r - 4
            for j in range(3):
                sel = m[old] > j
                cnt = int(sel.sum())
                e = ev[pos:pos + cnt]
                e["type"] = _cabi.EV_DELETE_ALLOCATED
                e["arg0"] = j
                e["suggested_off"] = -1
                e["spec"]["group"] = (old % slots) * 16 + vc[sel]
                e["spec"]["leaf_num"] = k[old][sel]
                e["spec"]["vc"] = vc[sel]
                pos += cnt
        for j in range(3):
            sel = m[r] > j
            cnt = int(sel.sum())
            e = ev[pos:pos + cnt]
            e["type"] = _cabi.EV_SCHEDULE
            e["phase"] = _cabi.PHASE_PREEMPTING
            e["suggested_off"] = -1
            s = e["spec"]
            s["group"] = (r % slots) * 16 + vc[sel]
            s["vc"] = vc[sel]
            s["pinned"] = -1
            s["leaf_type"] = 0
            s["leaf_num"] = k[r][sel]
            s["flags"] = _cabi.SPEC_IGNORE_SUGGESTED
            s["n_members"] = 1
            s["member_leaf_num"][:, 0] = k[r][sel]
            s["member_pod_num"][:, 0] = m[r][sel]
            pos += cnt
        if pos >= n:
            break
    out = np.zeros(n, dtype=trace.EVENT_DT)
    out.view(np.uint8)[:] = ev[:n].view(np.uint8)
    sched = out["type"] == _cabi.EV_SCHEDULE
    out["spec"]["pod"][sched] = np.arange(int(sched.sum()), dtype=np.int32)
    return out


def compaction_run(lib, n):
    """(results, pool, number of CTAs) of the batch in a fresh context."""
    ev = compaction_events(n)
    sched = ev["type"] == _cabi.EV_SCHEDULE
    bc = trace.BatchContext(lib, _compaction_config(), 16 * 8, int(sched.sum()) + 16, 64, 8)
    bc.set_all_nodes_healthy()
    cap = int(3 * (ev["spec"]["member_leaf_num"][sched, 0].astype(np.int64) * ev["spec"]["member_pod_num"][sched, 0]).sum()) + 4096
    res, pool = bc.process(ev, cap)
    f = lib.hived_bench_num_ctas
    f.restype = C.c_int
    f.argtypes = [C.c_void_p]
    ctas = f(bc.ctx)
    bc.close()
    return res, pool, ctas


def compaction_sequential(n, path):
    """The same batch with HIVED_NCTA=1 in a fresh process: the sequential path, no compaction; saved to path."""
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import numpy as np\n"
            "from hivedscheduler_b200 import _cabi\n"
            "import test_shape_limits as ts\n"
            "res, pool, ctas = ts.compaction_run(_cabi.load_cuda_library(), %d)\n"
            "assert ctas == 1, ctas\n"
            "np.savez(%r, res=res.view(np.int32), pool=pool)\n") % (ROOT, HERE, n, path)
    subprocess.check_call([sys.executable, "-c", code], env=dict(os.environ, HIVED_NCTA="1"))
    z = np.load(path)
    return z["res"].view(trace.RESULT_DT).reshape(-1), z["pool"]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [700, 1024, 1024 * 1024, 1024 * 1024 + 1025])
def test_pool_compaction_cuda(cuda_lib, n, tmp_path):
    """The canonical pool of a 16-CTA batch: every result's words at the exclusive prefix sum of the words before it in
    event order (3 per leaf of a bind, 2 per victim), this_off - leaf_off kept, and the pool word for word that of the
    sequential run.  At 1024 x 1024 results the 1024 block sums fill one tile and the grand total is the first entry
    of the second; at 1024 x 1024 + 1025 the second tile holds block sums too."""
    res, pool, ctas = compaction_run(cuda_lib, n)
    assert ctas == 16
    seq_res, seq_pool = compaction_sequential(n, str(tmp_path / "seq.npz"))
    bind = res["kind"] == _cabi.KIND_BIND
    pre = res["kind"] == _cabi.KIND_PREEMPT
    words = np.where(bind, 3 * res["n_leaves"], 0) + np.where(pre, 2 * res["n_victims"], 0)
    assert bind.sum() > n // 3 and not pre.any()
    excl = np.concatenate([[0], np.cumsum(words.astype(np.int64))[:-1]])
    assert (res["leaf_off"][bind] == excl[bind]).all()
    assert (res["victim_off"][pre] == excl[pre]).all()
    total = int(words.sum())
    for f in ("kind", "error", "wait_code", "node", "n_leaves", "this_n", "pod_index", "n_victims"):
        assert (res[f] == seq_res[f]).all(), f
    assert ((res["this_off"] - res["leaf_off"])[bind] == (seq_res["this_off"] - seq_res["leaf_off"])[bind]).all()
    assert (seq_res["leaf_off"][bind] == excl[bind]).all()
    assert (pool[:total] == seq_pool[:total]).all()
