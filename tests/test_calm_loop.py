"""The calm leader loop (csrc/hived_calm.inc) against the general one.

A batch the host judges calm (every node healthy, one guaranteed priority, only SCHEDULE / DELETE events) runs the
leader through the calm loop, which handles deletes, further pods of allocated gangs and new single-member gangs
itself and hands every other event to the unchanged general code.  HIVED_NO_CALM=1 makes the same library run every
batch through the general loop.  Every result record, the result pool, the cluster state and the counters must be the
same either way, and the result hash the oracle's.  The CPU tier runs the SIMT emulation (32-lane warps, one CTA per
group of VCs); a GPU-marked copy runs the CUDA library."""
import ctypes as C
from collections import deque

import pytest

from conftest import snapshot_bytes
from hivedscheduler_b200 import config, trace

# hived_dev.h PC_*: indices into hived_bench_path_counters
PC_COMMIT_GENERAL, PC_RELEASE_GENERAL, PC_MAP_GENERAL, PC_CALM, PC_CALM_FALLBACK = 5, 7, 9, 12, 13


def c3_slice(n_gangs=700):
    """C3's tree, gang mix and admission window at 90 % load, on 8 VCs of two racks each (one POD): a full C3 pass in
    miniature, one CTA per VC at 8 CTAs."""
    t = trace.trace_c3(n_gangs=n_gangs, n_vcs=8, vc_gpus=2 * 32 * 8)
    levels = [("HALF", "B200", 4), ("NODE", "HALF", 2), ("RACK", "NODE", 32), ("POD", "RACK", 16)]
    t["config"] = config._synthetic(levels, 1, "NODE", {"vc%d" % i: [("POD.RACK", 2)] for i in range(8)}, "n%04d")
    return t


def recycled_ids(n_gangs=700, n_ids=160):
    """C3's mix on 2 VCs where a released gang's id is taken by a later gang of the same VC within the batch."""
    rng = trace.XorShift64Star(trace.seed_for(11))
    tb = trace.TraceBuilder(4 * n_gangs)
    n_vcs, limit = 2, int(0.9 * (16 + 6) * 32 * 8)
    free = [deque(range(v, n_ids, n_vcs)) for v in range(n_vcs)]
    alive = [deque() for _ in range(n_vcs)]
    used = [0] * n_vcs
    for _ in range(n_gangs):
        pod_num, leaf_num = trace._gang_shape(rng.below(100))
        v = rng.below(n_vcs)
        while (used[v] + pod_num * leaf_num > limit or not free[v]) and alive[v]:
            og, opn, oln = alive[v].popleft()
            for j in range(opn):
                tb.delete_allocated(og, oln, j, vc=v)
            used[v] -= opn * oln
            free[v].append(og)
        g = free[v].popleft()
        for j in range(pod_num):
            tb.schedule(group=g, vc=v, priority=0, leaf_type=0, leaf_num=leaf_num, pod_num=pod_num, first=(j == 0))
        alive[v].append((g, pod_num, leaf_num))
        used[v] += pod_num * leaf_num
    ev, dec = tb.finish()
    return {"name": "recycled-ids", "config": config.config_c3(n_pods=4, n_vcs=2, racks_per_vc=6), "events": ev,
            "decision": dec, "n_groups": n_ids, "n_pods": tb.next_pod, "max_group_leaves": 64, "max_group_pods": 8}


TRACES = {
    "c3-slice": c3_slice,
    "multi-member": lambda: trace.trace_multi_member(n_gangs=300),
    "heterogeneous": lambda: trace.trace_heterogeneous(n_gangs=500),
    "recycled-ids": recycled_ids,
}


def _path_counters(lib, ctx):
    out = (C.c_int64 * 16)()
    n = lib.hived_bench_path_counters(ctx, out)
    return [int(x) for x in out[:n]]


def _run(lib, t, monkeypatch, calm, n_cta=None, chunks=2):
    monkeypatch.setenv("HIVED_NO_CALM", "0" if calm else "1")
    if n_cta is None:
        monkeypatch.delenv("HIVED_NCTA", raising=False)
    else:
        monkeypatch.setenv("HIVED_NCTA", str(n_cta))
    bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
    try:
        bc.set_all_nodes_healthy()
        ev = t["events"]
        bounds = [len(ev) * (i + 1) // chunks for i in range(chunks)]
        start, out = 0, []
        for b in bounds:
            res, pool = bc.process(ev[start:b], 3 * 64 * (b - start) + 4096)
            n = int((res["leaf_off"] + 3 * res["n_leaves"]).max()) if len(res) else 0
            out.append((res, pool[:n]))
            start = b
        return {"hash": bc.result_hash(), "out": out, "stats": bc.stats(), "snap": snapshot_bytes(lib, bc.ctx),
                "paths": _path_counters(lib, bc.ctx) if hasattr(lib, "hived_bench_path_counters") else None}
    finally:
        bc.close()


def _check(lib, oracle_lib, t, monkeypatch, n_cta=None):
    on = _run(lib, t, monkeypatch, True, n_cta)
    off = _run(lib, t, monkeypatch, False, n_cta)
    ref = _run(oracle_lib, t, monkeypatch, True, n_cta)
    assert on["hash"] == off["hash"] == ref["hash"]
    for (ra, pa), (rb, pb) in zip(on["out"], off["out"]):
        assert len(ra) == len(rb)
        for i in range(len(ra)):  # event by event: the first differing record is named
            assert ra[i].tobytes() == rb[i].tobytes(), "event %d: %r != %r" % (i, ra[i], rb[i])
        assert pa.tobytes() == pb.tobytes()
    assert on["stats"] == off["stats"]
    assert on["snap"] == off["snap"]
    assert on["paths"][:PC_CALM] == off["paths"][:PC_CALM]  # the same paths, whichever loop chose them
    assert on["paths"][PC_CALM] > 0
    assert off["paths"][PC_CALM] == off["paths"][PC_CALM_FALLBACK] == 0
    return on


def _check_c3(lib, oracle_lib, monkeypatch, n_cta):
    t = c3_slice()
    on = _check(lib, oracle_lib, t, monkeypatch, n_cta)
    p = on["paths"]
    # on C3 only the gangs that need the general mapping or commit, and their releases, leave the calm loop
    assert p[PC_CALM] + p[PC_CALM_FALLBACK] == len(t["events"])
    assert p[PC_CALM_FALLBACK] == p[PC_COMMIT_GENERAL] + p[PC_RELEASE_GENERAL]
    assert p[PC_MAP_GENERAL] <= p[PC_COMMIT_GENERAL]


@pytest.mark.parametrize("n_cta", [1, 8])
def test_calm_loop_matches_general_loop_on_c3(simt_lib, oracle_lib, monkeypatch, n_cta):
    _check_c3(simt_lib, oracle_lib, monkeypatch, n_cta)


@pytest.mark.parametrize("name", ["multi-member", "heterogeneous", "recycled-ids"])
def test_calm_loop_matches_general_loop(simt_lib, oracle_lib, monkeypatch, name):
    _check(simt_lib, oracle_lib, TRACES[name](), monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("n_cta", [1, 8])
def test_calm_loop_matches_general_loop_on_c3_gpu(cuda_lib, oracle_lib, monkeypatch, n_cta):
    _check_c3(cuda_lib, oracle_lib, monkeypatch, n_cta)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["multi-member", "heterogeneous", "recycled-ids"])
def test_calm_loop_matches_general_loop_gpu(cuda_lib, oracle_lib, monkeypatch, name):
    _check(cuda_lib, oracle_lib, TRACES[name](), monkeypatch)
