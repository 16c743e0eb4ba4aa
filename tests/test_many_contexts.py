"""The batches of several contexts in one call (hived_process_events_many, include/hived_multictx.h).

Every context of a joint call is compared with two runs of the same batch: the same library, one context at a time
through hived_process_events on a fresh context built the same way, and the oracle, also one context at a time.
Compared: rc, results and pool bytes, the running result hash, the work counters, the cell snapshots, the view-order and
bookkeeping hashes; against the same library also the path counters and the last error text.  The CPU tier runs the
thread emulation (every CTA of every context at the same time, tests/emu/hived_emu_mt_many.cpp), the SIMT emulation
(one grid of (max C) x k CTAs, tests/emu/hived_simt_many.cpp) and the 1-lane emulation (the contexts one after another);
the GPU tier the joint kernel, in one launch or in rounds when the contexts' CTAs do not fit on the device together."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, snapshot_bytes
from hivedscheduler_b200 import _cabi, config, dist, trace
from test_device_program_emu import small_c3, small_cluster

ERR_CAPACITY, ERR_BAD_SPEC = 102, 7  # HIVED_ERR_CAPACITY, HIVED_ERR_BAD_SPEC
N_PATH = 12                          # PC_COUNT (hived_dev.h)
SPARE = 8                            # group ids / pod ids beyond the trace's, for the per-call operations


def _hooks(lib):
    for name in ("hived_debug_view_hash", "hived_debug_bookkeeping_hash"):
        getattr(lib, name).restype = C.c_uint64
        getattr(lib, name).argtypes = [C.c_void_p]
    return lib


def workloads(short):
    """The six kinds of context of the mixed call (each with its own cluster)."""
    c5 = trace.trace_c5(n_steps=2, gangs_per_step=150 if short else 300, n_nodes=4 * 16 * 32, n_vcs=2,
                        vc_gpus=(16 + 6) * 32 * 8, config=small_cluster())
    return [small_c3(400 if short else 1500),                   # VC-parallel, 2 CTAs
            c5,                                                 # bad nodes: one CTA
            trace.trace_heterogeneous(n_gangs=300 if short else 1500),
            trace.trace_suggested_nodes(n_gangs=200 if short else 900),
            trace.trace_multi_member(n_gangs=150 if short else 600),
            trace.trace_bad_requests()]


def _ctx(lib, t):
    bc = trace.BatchContext(lib, t["config"], t["n_groups"] + SPARE, t["n_pods"] + 64 * SPARE, t["max_group_leaves"],
                            t["max_group_pods"])
    bc.set_all_nodes_healthy()
    return bc


def _single(bc, ev, words, sp=None):
    """hived_process_events, keeping the rc (BatchContext.process raises on one)."""
    ev = np.ascontiguousarray(ev)
    res = np.zeros(len(ev), dtype=trace.RESULT_DT)
    pool = np.zeros(max(int(words), 1), dtype=np.int32)
    spp, sw = None, 0
    if sp is not None and len(sp):
        sp = np.ascontiguousarray(sp, dtype=np.uint32)
        spp, sw = sp.ctypes.data_as(C.POINTER(C.c_uint32)), len(sp)
    rc = bc.lib.hived_process_events(bc.ctx, ev.ctypes.data_as(C.POINTER(_cabi.Event)), len(ev), spp, sw,
                                     res.ctypes.data_as(C.POINTER(_cabi.Result)),
                                     pool.ctypes.data_as(C.POINTER(C.c_int32)), int(words))
    return rc, res, pool


def _state(bc, same_lib):
    lib, ctx = bc.lib, bc.ctx
    s = (bc.result_hash(), bc.stats(), snapshot_bytes(lib, ctx), int(lib.hived_debug_view_hash(ctx)),
         int(lib.hived_debug_bookkeeping_hash(ctx)))
    if same_lib:
        pc = (C.c_int64 * 16)()
        lib.hived_bench_path_counters(ctx, pc)
        s += (list(pc)[:N_PATH], lib.hived_last_error(ctx))
    return s


class Trio:
    """One workload on three contexts: the joint one, the same library one context at a time, the oracle."""

    def __init__(self, lib, oracle, t):
        self.t = t
        self.joint, self.single, self.ref = _ctx(lib, t), _ctx(lib, t), _ctx(oracle, t)

    def each(self, fn):
        """A per-call operation (or a single-context batch) on all three contexts."""
        return [fn(bc) for bc in (self.joint, self.single, self.ref)]

    def check(self, got, ev, words, oracle=True):
        rc, res, pool = got
        for bc, same in ((self.single, True), (self.ref, False)):
            if not same and not oracle:
                continue
            want = _single(bc, ev, words, self.t.get("sugg_pool"))
            name = "%s vs %s" % (self.t["name"], "same library" if same else "oracle")
            assert rc == want[0], name
            assert res.tobytes() == want[1].tobytes(), name
            assert pool.tobytes() == want[2].tobytes(), name
            assert _state(self.joint, same) == _state(bc, same), name

    def close(self):
        for bc in (self.joint, self.single, self.ref):
            bc.close()


def _words(ev):
    return 3 * 64 * len(ev) + 4096


def joint_round(trios, chunks, words=None):
    got = trace.process_many([x.joint for x in trios], chunks, words or [_words(ev) for ev in chunks],
                             [x.t.get("sugg_pool") for x in trios])
    for x, ev, g, w in zip(trios, chunks, got, words or [_words(ev) for ev in chunks]):
        x.check(g, ev, w)
    return got


def _chunks(ev, parts):
    return [ev[len(ev) * i // parts:len(ev) * (i + 1) // parts] for i in range(parts)]


def _emu_many_lib(name, flags):
    """tests/emu/<name>.cpp: an emulation library with a joint launch of its own."""
    out = os.path.join(ROOT, "tests", "_build", "lib%s.so" % name)
    emu = os.path.join(ROOT, "tests", "emu")
    csrc = os.path.join(ROOT, "hivedscheduler_b200", "csrc")
    deps = [os.path.join(emu, f) for f in os.listdir(emu)] + [os.path.join(csrc, f) for f in os.listdir(csrc)
                                                             if f.endswith((".h", ".hpp", ".inc"))]
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++"] + flags + ["-std=c++17", "-fPIC", "-shared", "-o", out,
                                                 os.path.join(emu, name + ".cpp")])
    return _cabi.load_library(out)


@pytest.fixture(scope="module")
def emu_mt_many_lib():
    return _emu_many_lib("hived_emu_mt_many", ["-O2", "-pthread"])


@pytest.fixture(scope="module")
def simt_many_lib():
    return _emu_many_lib("hived_simt_many", ["-O1", "-g"])


@pytest.fixture(params=["emu_mt_many", "simt_many", "emu"])
def lib(request):
    return _hooks(request.getfixturevalue(request.param + "_lib"))


def _short(lib):
    return "simt" in lib._name or lib._name.endswith("libhived_emu.so")


# ---- CPU tier (thread and SIMT emulations) ------------------------------------------------------------------------------

def test_mixed_contexts_in_one_call(lib, oracle_lib):
    """Six different clusters in one call: VC-parallel, bad nodes, two chains, suggested-node sets, multi-member gangs,
    per-event user errors.  Two different clusters in one call also catch a joint build that reads another slot's
    state."""
    trios = [Trio(lib, _hooks(oracle_lib), t) for t in workloads(short=_short(lib))]
    got = joint_round(trios, [x.t["events"] for x in trios])
    assert [g[0] for g in got] == [0] * len(trios)
    if not lib._name.endswith("libhived_emu.so"):  # (the 1-lane emulation runs every batch on one CTA)
        assert lib.hived_bench_num_ctas(trios[0].joint.ctx) == 2  # small_c3 ran VC-parallel
    for x in trios:
        x.close()


def test_rounds_with_per_call_operations_in_between(lib, oracle_lib):
    """Three joint calls on the same contexts; in between, per-call schedule / delete / node health on one context and a
    single-context hived_process_events on another."""
    short = _short(lib)
    ts = workloads(short)
    trios = [Trio(lib, _hooks(oracle_lib), t) for t in (ts[0], ts[2], ts[4])]
    # b's batches 1 and 3 run alone between the joint calls, which take its batches 0, 2 and 4
    parts = [_chunks(trios[0].t["events"], 3), _chunks(trios[1].t["events"], 3), _chunks(trios[2].t["events"], 5)]
    a, b = trios[1], trios[2]
    spec = _cabi.PodSpec(pod=a.t["n_pods"], group=a.t["n_groups"], vc=0, priority=0, pinned=-1, leaf_type=0,
                         leaf_num=1, flags=_cabi.SPEC_IGNORE_SUGGESTED, n_members=1)
    spec.member_leaf_num[0], spec.member_pod_num[0] = 1, 1

    def schedule(bc):
        res, pool = _cabi.Result(), (C.c_int32 * 64)()
        rc = bc.lib.hived_schedule(bc.ctx, C.byref(spec), None, _cabi.PHASE_PREEMPTING, C.byref(res), pool, 64)
        return rc, bytes(res), bytes(pool)

    ops = [
        lambda: a.each(schedule),
        lambda: a.each(lambda bc: bc.lib.hived_set_node_health(bc.ctx, bc.n_nodes - 1, 0)),
        lambda: a.each(lambda bc: bc.lib.hived_delete_allocated_pod(bc.ctx, spec.group, 1, 0)),
    ]
    for r in range(3):
        joint_round(trios, [parts[0][r], parts[1][r], parts[2][2 * r]])
        outs = ops[r]()
        assert outs[0] == outs[1] == outs[2]
        if r < 2:
            alone = parts[2][2 * r + 1]
            got = b.each(lambda bc: _single(bc, alone, _words(alone)))
            assert got[0][0] == got[1][0] == got[2][0] == 0
            assert got[0][1].tobytes() == got[1][1].tobytes() == got[2][1].tobytes()
    for x in trios:
        x.close()


def test_one_context_is_byte_identical_to_process_events(lib, oracle_lib):
    t = small_c3(300)
    x = Trio(lib, _hooks(oracle_lib), t)
    for ev in _chunks(t["events"], 2):
        joint_round([x], [ev])
    x.close()


def test_empty_batch_in_the_list(lib, oracle_lib):
    ts = workloads(short=True)
    trios = [Trio(lib, _hooks(oracle_lib), t) for t in (ts[5], ts[2])]
    got = joint_round(trios, [trios[0].t["events"][:0], trios[1].t["events"]])
    assert got[0][0] == 0 and len(got[0][1]) == 0
    for x in trios:
        x.close()


def test_pool_one_word_short_fails_only_that_batch(lib, oracle_lib):
    ts = workloads(short=True)
    trios = [Trio(lib, _hooks(oracle_lib), t) for t in (ts[4], ts[2])]
    probe = _ctx(lib, ts[4])
    res, pool = probe.process(ts[4]["events"], _words(ts[4]["events"]))
    used = int(np.flatnonzero(pool).max()) + 1 if pool.any() else 0
    probe.close()
    words = [used - 1, _words(ts[2]["events"])]
    got = trace.process_many([x.joint for x in trios], [x.t["events"] for x in trios], words)
    assert got[0][0] == ERR_CAPACITY and got[1][0] == 0
    trios[0].check(got[0], ts[4]["events"], words[0], oracle=False)
    trios[1].check(got[1], ts[2]["events"], words[1])
    for x in trios:
        x.close()


def test_refused_lists_change_nothing(lib, oracle_lib):
    t = trace.trace_bad_requests()
    ctxs = [_ctx(lib, t) for _ in range(_cabi.HIVED_MANY_MAX + 1)]
    ev = t["events"]
    before = [_state(bc, False) for bc in ctxs]

    def call(bcs):
        arr = (_cabi.Batch * max(len(bcs), 1))()
        keep = []
        for i, bc in enumerate(bcs):
            res, pool = np.zeros(len(ev), dtype=trace.RESULT_DT), np.zeros(_words(ev), dtype=np.int32)
            keep.append((res, pool))
            arr[i].ctx = bc.ctx if bc is not None else None
            arr[i].events, arr[i].n = ev.ctypes.data_as(C.POINTER(_cabi.Event)), len(ev)
            arr[i].res, arr[i].pool = res.ctypes.data_as(C.POINTER(_cabi.Result)), pool.ctypes.data_as(C.POINTER(C.c_int32))
            arr[i].pool_cap = _words(ev)
        return _cabi.bind_many(lib).hived_process_events_many(arr, len(bcs))

    assert call([]) == ERR_BAD_SPEC
    assert call(ctxs) == ERR_BAD_SPEC                      # k = 17
    assert call([ctxs[0], ctxs[1], ctxs[0]]) == ERR_BAD_SPEC
    assert call([ctxs[0], None]) == ERR_BAD_SPEC
    # a context staged for a multi-GPU partition
    dist.bind_multigpu(lib)
    calm = trace.TraceBuilder(4)
    calm.schedule(group=1, vc=0, priority=0, leaf_type=0, leaf_num=1, pod_num=1)
    cev, _ = calm.finish()
    staged = _ctx(lib, t)
    assert lib.hived_mg_stage(staged.ctx, cev.ctypes.data_as(C.POINTER(_cabi.Event)), len(cev), 4096, 0, 1) == 0
    staged_before = _state(staged, False)
    assert call([ctxs[0], staged]) == ERR_BAD_SPEC
    assert _state(staged, False) == staged_before
    assert [_state(bc, False) for bc in ctxs] == before
    # and the same contexts still run a joint call normally
    assert call(ctxs[:3]) == 0
    for bc in ctxs + [staged]:
        bc.close()


# ---- GPU tier ---------------------------------------------------------------------------------------------------------

def c3_ctx_trace(n_vcs, n_gangs):
    """C3's gang mix on n_vcs VCs of a POD and a rack each (one CTA per VC)."""
    t = trace.trace_c3(n_gangs=n_gangs, n_vcs=n_vcs, vc_gpus=(16 + 1) * 32 * 8, config_number=3)
    t["config"] = config.config_c3(n_pods=n_vcs + 1, n_vcs=n_vcs, racks_per_vc=1)
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 4, 16])
def test_gpu_joint_calls(cuda_lib, oracle_lib, k):
    ts = workloads(short=False)
    trios = [Trio(_hooks(cuda_lib), _hooks(oracle_lib), ts[i % len(ts)]) for i in range(k)]
    for r in range(2):
        got = joint_round(trios, [_chunks(x.t["events"], 2)[r] for x in trios])
        assert all(g[0] == 0 for g in got)
    for x in trios:
        x.close()


@pytest.mark.gpu
def test_gpu_more_ctas_than_fit_run_in_rounds(cuda_lib, oracle_lib):
    """16 contexts of 16 VCs each: 256 CTAs, more than an H100 holds at once (one CTA per SM)."""
    t = c3_ctx_trace(16, 1500)
    x = Trio(_hooks(cuda_lib), _hooks(oracle_lib), t)  # its single-context and oracle runs stand for all 16
    joint = [x.joint] + [_ctx(x.joint.lib, t) for _ in range(15)]
    ev = t["events"]
    got = trace.process_many(joint, [ev] * 16, [_words(ev)] * 16)
    x.check(got[0], ev, _words(ev))
    for bc, g in zip(joint[1:], got[1:]):
        assert g[0] == 0 and g[1].tobytes() == got[0][1].tobytes() and g[2].tobytes() == got[0][2].tobytes()
        assert _state(bc, True) == _state(x.joint, True)
    assert all(cuda_lib.hived_bench_num_ctas(bc.ctx) == 16 for bc in joint)
    for bc in joint[1:]:
        bc.close()
    x.close()


@pytest.mark.gpu
def test_gpu_resident_per_call_kernels_around_a_joint_call(cuda_lib, oracle_lib):
    """A participant with a live resident per-call kernel before and after the joint call, and a context outside the
    list that owns the device's constant bank with a live resident kernel, which keeps answering correctly."""
    lib = _hooks(cuda_lib)
    ts = workloads(short=False)
    part, other = Trio(lib, _hooks(oracle_lib), ts[2]), Trio(lib, _hooks(oracle_lib), ts[4])
    mate = Trio(lib, _hooks(oracle_lib), ts[0])

    def spec_for(x, i):
        s = _cabi.PodSpec(pod=x.t["n_pods"] + i, group=x.t["n_groups"] + i, vc=0, priority=0, pinned=-1, leaf_type=-1,
                          leaf_num=1, flags=_cabi.SPEC_IGNORE_SUGGESTED, n_members=1)
        s.member_leaf_num[0], s.member_pod_num[0] = 1, 1
        return s

    def schedule(x, i):
        s = spec_for(x, i)

        def one(bc):
            res, pool = _cabi.Result(), (C.c_int32 * 64)()
            rc = bc.lib.hived_schedule(bc.ctx, C.byref(s), None, _cabi.PHASE_PREEMPTING, C.byref(res), pool, 64)
            return rc, bytes(res), bytes(pool)
        outs = x.each(one)
        assert outs[0] == outs[1] == outs[2]

    halves = [_chunks(x.t["events"], 2) for x in (part, mate)]
    for r in range(2):
        schedule(part, 2 * r)       # the participant's resident kernel is live ...
        schedule(other, 2 * r)      # ... and so is the constant bank owner's, which is not in the list
        joint_round([part, mate], [halves[0][r], halves[1][r]])
        schedule(part, 2 * r + 1)
        schedule(other, 2 * r + 1)
        assert _state(other.joint, True) == _state(other.single, True)
        assert _state(other.joint, False) == _state(other.ref, False)
    for x in (part, other, mate):
        x.close()
