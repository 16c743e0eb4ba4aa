"""The host's per-batch decisions: which CTA owns each event, and whether the batch is calm (DESIGN.md §4).

A batch runs VC-parallel, one CTA per group of VCs, when it is calm and has at least 256 events.  Calm means every
node is healthy, one guaranteed priority is in use, there has been no recovery, and the batch has only SCHEDULE /
DELETE events.  A DELETE belongs to the VC its group was last scheduled under, and a group id that one batch uses
under two VCs makes the batch sequential.  Each case below is decided by one of these rules.  It ends with one large
batch, and asserts that batch's CTA count (hived_bench_num_ctas), whether its events ran through the calm leader loop
(path counters) and the oracle's result hash.

Batches of at most 8 events take the CUDA library's per-call path, which bypasses the batch staging, so the cases
with a per-call step check its bookkeeping only on the GPU.  The host builds stage those batches like any other."""
import ctypes as C

import numpy as np
import pytest

from hivedscheduler_b200 import trace
from test_calm_loop import PC_CALM, PC_CALM_FALLBACK, c3_slice

N_CTAS = 8  # the slice has 8 VCs: one CTA per VC
EXTRA_GROUPS = 8  # group ids past the trace's, for the cases' own gangs


def _steps(name, t):
    """The case's batches: (events, per-call?) in order; the last one is the batch the assertions are about."""
    ev = t["events"]
    g0 = t["n_groups"]  # a group id the trace never uses
    tb = trace.TraceBuilder(8)
    tb.next_pod = t["n_pods"]
    if name == "calm":
        return [(ev[:600], False)]
    if name == "two-vcs":  # g0 scheduled under VC 0, released, then scheduled under VC 1 in the same batch
        tb.schedule(group=g0, vc=0, priority=0, leaf_type=0, leaf_num=1, pod_num=1)
        tb.delete_allocated(g0, 1, 0)
        tb.schedule(group=g0, vc=1, priority=0, leaf_type=0, leaf_num=1, pod_num=1)
        return [(np.concatenate([ev[:600], tb.finish()[0]]), False)]
    if name == "per-call-delete":  # g0 scheduled per call under VC 3; the batch releases it and reuses its id under VC 5
        tb.schedule(group=g0, vc=3, priority=0, leaf_type=0, leaf_num=1, pod_num=1)
        call = tb.finish()[0]
        tb = trace.TraceBuilder(8)
        tb.next_pod = t["n_pods"] + 1
        tb.delete_allocated(g0, 1, 0)
        tb.schedule(group=g0, vc=5, priority=0, leaf_type=0, leaf_num=1, pod_num=1)
        return [(call, True), (np.concatenate([ev[:600], tb.finish()[0]]), False)]
    if name == "per-call-priority":  # a second guaranteed priority, used per call before the batch
        tb.schedule(group=g0, vc=2, priority=1, leaf_type=0, leaf_num=1, pod_num=1)
        return [(tb.finish()[0], True), (ev[:600], False)]
    if name == "unknown-delete":  # a DELETE of a group nobody scheduled, without a VC: it runs (as a no-op) on VC 0
        tb.delete_allocated(g0 + 1, 1, 0)
        return [(np.concatenate([ev[:300], tb.finish()[0], ev[300:600]]), False)]
    if name == "small":  # calm, but too small to split
        return [(ev[:200], False)]
    raise KeyError(name)


# case -> (CTAs of the last batch, whether it ran through the calm loop)
CASES = {
    "calm": (N_CTAS, True),
    "two-vcs": (1, False),
    "per-call-delete": (1, False),
    "per-call-priority": (1, False),
    "unknown-delete": (N_CTAS, True),
    "small": (1, True),
}


def _path_counters(lib, ctx):
    out = (C.c_int64 * 16)()
    n = lib.hived_bench_path_counters(ctx, out)
    return [int(x) for x in out[:n]]


def _run(lib, t, steps, measured):
    bc = trace.BatchContext(lib, t["config"], t["n_groups"] + EXTRA_GROUPS, t["n_pods"] + 4, t["max_group_leaves"],
                            t["max_group_pods"])
    try:
        bc.set_all_nodes_healthy()
        for i, (ev, per_call) in enumerate(steps):
            assert (len(ev) <= 8) == per_call
            last = i == len(steps) - 1
            before = _path_counters(lib, bc.ctx) if measured and last else None
            bc.process(ev, 3 * 64 * len(ev) + 4096)
        out = {"hash": bc.result_hash()}
        if measured:
            after = _path_counters(lib, bc.ctx)
            out["ctas"] = lib.hived_bench_num_ctas(bc.ctx)
            out["calm"] = after[PC_CALM] - before[PC_CALM]
            out["handed_over"] = after[PC_CALM_FALLBACK] - before[PC_CALM_FALLBACK]
        return out
    finally:
        bc.close()


def _check(lib, oracle_lib, monkeypatch, name):
    monkeypatch.delenv("HIVED_NCTA", raising=False)
    monkeypatch.delenv("HIVED_NO_CALM", raising=False)
    t = c3_slice()
    steps = _steps(name, t)
    got = _run(lib, t, steps, True)
    ref = _run(oracle_lib, t, steps, False)
    ctas, calm = CASES[name]
    n = len(steps[-1][0])
    assert got["ctas"] == ctas
    if calm:  # every event enters the calm loop, which runs most of them itself
        assert got["calm"] + got["handed_over"] == n
        assert got["calm"] > n // 2
    else:
        assert got["calm"] == got["handed_over"] == 0
    assert got["hash"] == ref["hash"]


@pytest.mark.parametrize("name", list(CASES))
def test_batch_routing(emu_mt_lib, oracle_lib, monkeypatch, name):
    _check(emu_mt_lib, oracle_lib, monkeypatch, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_batch_routing_gpu(cuda_lib, oracle_lib, monkeypatch, name):
    _check(cuda_lib, oracle_lib, monkeypatch, name)
