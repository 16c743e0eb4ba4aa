"""Concurrent contexts (HIVED_OPT_CONCURRENT, include/hived.h "Threads"): the per-call path of each on a resident kernel
of its own, driven by its own thread at the same time as the other contexts of the process.

CPU tier: the flag changes nothing on the oracle and the emulations (API fuzz and a batch trace, with and without it),
and the Python layers carry it.  GPU tier: every answer compared with the oracle (the API fuzz compares results, every
cell, the view order and the bookkeeping after every call) — threads on contexts of their own, calls of two contexts
interleaved without turns, the per-device capacity and slot reuse, a concurrent context through batches, a joint call and
a state rewind while another one keeps answering, and the calls that still take turns."""
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

import fuzz_api
from conftest import ORACLE_LIB, ROOT
from hivedscheduler_b200 import _cabi, config, trace
from test_device_program_emu import small_c3
from test_many_contexts import _hooks, _single, _state, _words
from test_shape_limits import _process_rc, _window_cluster, _window_events

HERE = os.path.dirname(os.path.abspath(__file__))
FLAG = _cabi.OPT_CONCURRENT
ERR_CAPACITY = 102  # HIVED_ERR_CAPACITY


class Flagged:
    """A library whose hived_create adds `flags` to hived_options_t.flags; everything else is the library itself.  It
    gives fuzz_api.run_seed concurrent contexts: against the oracle (which ignores the flag), or against the same library
    without the flag."""

    def __init__(self, lib, flags):
        self._lib, self._flags = lib, flags

    def hived_create(self, spec, opt, out):
        opt._obj.flags |= self._flags
        return self._lib.hived_create(spec, opt, out)

    def __getattr__(self, name):
        return getattr(self._lib, name)


def _launches(lib):
    lib.hived_bench_kernel_launches.restype = C.c_int64
    lib.hived_bench_kernel_launches.argtypes = [C.c_void_p]
    return lib


def replay(lib, t, flags):
    """The trace through hived_process_events: its first 36 events in chunks of 1..8 (the per-call path on the GPU),
    then the rest in one batch.  Returns every chunk's (rc, results, pool) and the final state."""
    bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"],
                            flags=flags)
    try:
        bc.set_all_nodes_healthy()
        ev, out, at = t["events"], [], 0
        for size in [1, 2, 3, 4, 5, 6, 7, 8] + [len(t["events"])]:
            chunk = ev[at:at + size]
            if len(chunk) == 0:
                break
            rc, res, pool = _single(bc, chunk, _words(chunk))
            out.append((rc, res.tobytes(), pool.tobytes()))
            at += len(chunk)
        return out, _state(bc, hasattr(lib, "hived_bench_path_counters"))
    finally:
        bc.close()


# ---- CPU tier ---------------------------------------------------------------------------------------------------------

@pytest.fixture(params=["oracle", "emu", "simt"])
def any_lib(request):
    return _hooks(request.getfixturevalue(request.param + "_lib"))


def test_flag_changes_nothing_off_the_gpu(any_lib):
    """The oracle and the emulations accept the flag and ignore it: one batch trace and one API-fuzz seed give the same
    bytes with and without it."""
    t = small_c3(200)
    assert replay(any_lib, t, FLAG) == replay(any_lib, t, 0)
    assert fuzz_api.run_seed(Flagged(any_lib, FLAG), any_lib, 5, 120) is None


def test_python_layers_carry_the_flag(emu_lib, oracle_lib, monkeypatch):
    hdr = open(os.path.join(ROOT, "include", "hived.h")).read()
    assert "#define HIVED_OPT_CONCURRENT %d " % _cabi.OPT_CONCURRENT in hdr
    assert "#define HIVED_CONCURRENT_MAX %d " % _cabi.HIVED_CONCURRENT_MAX in hdr
    t = trace.trace_c1()
    bc = trace.BatchContext(emu_lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"],
                            flags=FLAG)
    assert bc.opt.flags == FLAG
    bc.close()
    bc = trace.BatchContext(emu_lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
    assert bc.opt.flags == 0
    bc.close()
    h = fuzz_api.alg.HivedAlgorithm(t["config"], lib=emu_lib, flags=FLAG)  # HivedAlgorithm(**options) forwards flags
    assert h._opt.flags == FLAG
    h.close()
    # the API fuzz's contexts get the flag through Flagged, on the flagged side only
    seen = []
    real = fuzz_api.alg.HivedAlgorithm

    class Recording(real):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            seen.append(int(self._opt.flags))

    monkeypatch.setattr(fuzz_api.alg, "HivedAlgorithm", Recording)
    assert fuzz_api.run_seed(Flagged(emu_lib, FLAG), oracle_lib, 1, 3) is None
    assert fuzz_api.run_seed(emu_lib, oracle_lib, 1, 3) is None
    assert seen == [FLAG, 0, 0, 0]


# ---- GPU tier ---------------------------------------------------------------------------------------------------------

def _fuzz_threads(cuda_lib, oracle_lib, jobs, n_ops):
    """jobs: [(seed, flags)], one thread each, all at once, each on contexts created with its flags (the CUDA side).
    Returns {seed: divergence or None}."""
    out = {}

    def work(seed, flags):
        try:
            out[seed] = fuzz_api.run_seed(Flagged(cuda_lib, flags), oracle_lib, seed, n_ops)
        except BaseException as e:  # noqa
            out[seed] = "exception: %r" % (e,)

    threads = [threading.Thread(target=work, args=job) for job in jobs]
    for th in threads:
        th.start()
    for th in threads:
        th.join(timeout=900)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 4, 16])
def test_gpu_threads_each_drive_a_concurrent_context(cuda_lib, oracle_lib, k):
    seeds = list(range(41, 41 + k))
    out = _fuzz_threads(cuda_lib, oracle_lib, [(s, FLAG) for s in seeds], 150)
    assert out == {s: None for s in seeds}


@pytest.mark.gpu
def test_gpu_concurrent_and_turn_taking_contexts_together(cuda_lib, oracle_lib):
    jobs = [(61, FLAG), (62, 0), (63, FLAG), (64, 0)]
    out = _fuzz_threads(cuda_lib, oracle_lib, jobs, 150)
    assert out == {s: None for s, _ in jobs}


@pytest.mark.gpu
def test_gpu_concurrent_path_matches_the_turn_taking_path(cuda_lib):
    """The same library with and without the flag, call by call (API fuzz), and on a batch trace in small chunks."""
    lib = _hooks(cuda_lib)
    assert fuzz_api.run_seed(Flagged(lib, FLAG), lib, 7, 200) is None
    t = small_c3(400)
    assert replay(lib, t, FLAG) == replay(lib, t, 0)


class PerCall:
    """Schedule + delete of one-pod gangs on one context, through hived_process_events(n = 1) and
    hived_delete_allocated_pod; every answer is kept."""

    def __init__(self, lib, t, flags=0):
        self.lib = lib
        self.bc = trace.BatchContext(lib, t["config"], 4096, 4096, t["max_group_leaves"], t["max_group_pods"], flags=flags)
        self.bc.set_all_nodes_healthy()
        self.n_vcs = lib.hived_num_vcs(self.bc.ctx)
        self.i = 0
        self.answers = []
        self.ev = np.zeros(1, dtype=trace.EVENT_DT)
        self.res = np.zeros(1, dtype=trace.RESULT_DT)
        self.pool = np.zeros(4096, dtype=np.int32)
        self.pending = None

    def schedule(self):
        g = self.i % 1024
        tb = trace.TraceBuilder(1)
        tb.schedule(group=g, vc=self.i % self.n_vcs, priority=0, leaf_type=0, leaf_num=8, pod_num=1)
        self.ev[:] = tb.finish()[0]
        self.ev["spec"]["pod"] = g
        self.i += 1
        rc = self.lib.hived_process_events(self.bc.ctx, self.ev.ctypes.data_as(C.POINTER(_cabi.Event)), 1, None, 0,
                                           self.res.ctypes.data_as(C.POINTER(_cabi.Result)),
                                           self.pool.ctypes.data_as(C.POINTER(C.c_int32)), len(self.pool))
        used = int(self.res["leaf_off"][0] + 3 * self.res["n_leaves"][0]) if rc == 0 and self.res["kind"][0] == 1 else 0
        self.answers.append((rc, self.res.tobytes(), self.pool[:used].tobytes()))
        self.pending = (g, int(self.res["pod_index"][0])) if rc == 0 and self.res["kind"][0] == 1 else None

    def delete(self):
        if self.pending is None:
            return
        g, pod_index = self.pending
        self.answers.append(("del", self.lib.hived_delete_allocated_pod(self.bc.ctx, g, 8, pod_index)))
        self.pending = None

    def calls(self):
        return len(self.answers)

    def close(self):
        self.bc.close()


@pytest.mark.gpu
def test_gpu_interleaved_calls_take_no_turns(cuda_lib, oracle_lib):
    """One thread, calls of two contexts interleaved A, B, A, B ... in a tight loop: concurrent contexts keep their
    resident kernels (far fewer launches than calls), ordinary ones take turns on the constant bank (a launch per call).
    Both answer like the oracle."""
    lib = _launches(cuda_lib)
    t = small_c3(10)
    for flags, rounds in ((FLAG, 600), (0, 600)):
        ctxs = [PerCall(lib, t, flags) for _ in range(2)]
        refs = [PerCall(oracle_lib, t) for _ in range(2)]
        before = [lib.hived_bench_kernel_launches(x.bc.ctx) for x in ctxs]
        for _ in range(rounds):
            for x in ctxs:
                x.schedule()
            for x in ctxs:
                x.delete()
        launches = [lib.hived_bench_kernel_launches(x.bc.ctx) - b for x, b in zip(ctxs, before)]
        for _ in range(rounds):
            for x in refs:
                x.schedule()
            for x in refs:
                x.delete()
        calls = [x.calls() for x in ctxs]
        assert sum(calls) >= 2000
        for x, r in zip(ctxs, refs):
            assert x.answers == r.answers
            assert _state(x.bc, False) == _state(r.bc, False)
        if flags:
            assert all(n <= 1 + c // 50 for n, c in zip(launches, calls)), (launches, calls)
        else:
            assert all(n >= 0.9 * c for n, c in zip(launches, calls)), (launches, calls)
        for x in ctxs + refs:
            x.close()


def _free_bytes():
    import torch
    return torch.cuda.mem_get_info(0)[0]


@pytest.mark.gpu
def test_gpu_capacity_and_slot_reuse(cuda_lib, oracle_lib):
    """16 concurrent contexts on device 0 all answer; the 17th hived_create fails with HIVED_ERR_CAPACITY, names the limit
    and leaves no device memory behind; a context created after one is destroyed takes the freed slot."""
    t = small_c3(10)
    ctxs = [PerCall(cuda_lib, t, FLAG) for _ in range(_cabi.HIVED_CONCURRENT_MAX)]
    refs = [PerCall(oracle_lib, t)]
    try:
        for _ in range(3):
            for x in ctxs + refs:
                x.schedule()
            for x in ctxs + refs:
                x.delete()
        assert all(x.answers == refs[0].answers for x in ctxs)
        big = t["config"]
        opt = _cabi.Options(max_groups=1 << 17, max_pods=1 << 17, max_group_leaves=64, max_group_pods=8, device=0,
                            flags=FLAG)
        ctx = C.c_void_p()
        _free_bytes()  # (the first query sets up torch's own state on the device)
        free0 = _free_bytes()
        rc = cuda_lib.hived_create(config.to_spec_text(big).encode(), C.byref(opt), C.byref(ctx))
        assert rc == ERR_CAPACITY and not ctx
        assert "HIVED_CONCURRENT_MAX" in cuda_lib.hived_create_error().decode()
        assert _free_bytes() >= free0 - (16 << 20)  # the failed context took ~100 MB while it was being built
        ctxs.pop(5).close()
        fresh = PerCall(cuda_lib, t, FLAG)
        ctxs.append(fresh)
        ref = PerCall(oracle_lib, t)
        refs.append(ref)
        for _ in range(3):
            for x in (fresh, ref):
                x.schedule()
                x.delete()
        assert fresh.answers == ref.answers
    finally:
        for x in ctxs + refs:
            x.close()


@pytest.mark.gpu
def test_gpu_concurrent_context_through_batches_joint_call_and_rewind(cuda_lib, oracle_lib):
    """A concurrent context goes through per-call operations, a VC-parallel batch, a joint call with an ordinary context
    and a state rewind, then per-call operations again, every step as the oracle; meanwhile a third (concurrent) context
    answers calls from another thread, like the oracle, throughout."""
    lib = _hooks(cuda_lib)
    lib.hived_bench_save_state.argtypes = lib.hived_bench_restore_state.argtypes = [C.c_void_p]
    t = small_c3(600)
    chunks = [t["events"][:300], t["events"][300:]]

    def ctx(lb, flags=0):
        bc = trace.BatchContext(lb, t["config"], t["n_groups"] + 64, t["n_pods"] + 64, t["max_group_leaves"],
                                t["max_group_pods"], flags=flags)
        bc.set_all_nodes_healthy()
        return bc

    x, xo, xs = ctx(lib, FLAG), ctx(oracle_lib), ctx(oracle_lib)  # xs: the oracle held at the saved state
    o, oo = ctx(lib), ctx(oracle_lib)
    stop, ready, worker_err, stamps = threading.Event(), threading.Event(), [], []

    def worker():
        w, wo = PerCall(lib, t, FLAG), PerCall(oracle_lib, t)
        deadline = time.time() + 300
        try:
            while not stop.is_set() and time.time() < deadline:
                for y in (w, wo):
                    y.schedule()
                    y.delete()
                if w.answers[-2:] != wo.answers[-2:]:
                    worker_err.append("call %d differs from the oracle" % w.calls())
                    return
                stamps.append(time.perf_counter())
                ready.set()
                if len(stamps) % 100 == 0:
                    # a pause now and then, as a real caller has: the resident kernel leaves after ~2 ms idle, and a
                    # device-wide synchronisation of the main thread (cudaFree when a batch buffer grows) waits for that
                    time.sleep(0.005)
        except BaseException as e:  # noqa
            worker_err.append(repr(e))
        finally:
            ready.set()
            w.close()
            wo.close()

    def per_call(bcs, k):
        """One pod scheduled and allocated (hived_process_events, n = 1), a node set bad and healthy again."""
        outs = []
        for bc in bcs:
            tb = trace.TraceBuilder(1)
            tb.schedule(group=t["n_groups"] + k, vc=k % 2, priority=0, leaf_type=0, leaf_num=8, pod_num=1)
            ev = tb.finish()[0]
            ev["spec"]["pod"] = t["n_pods"] + k
            rc, res, pool = _single(bc, ev, 256)
            node = (7 * k) % bc.n_nodes
            health = (bc.lib.hived_set_node_health(bc.ctx, node, 0), bc.lib.hived_set_node_health(bc.ctx, node, 1))
            outs.append((rc, res.tobytes(), pool.tobytes(), health))
        assert all(out == outs[-1] for out in outs)
        assert all(_state(bc, False) == _state(bcs[-1], False) for bc in bcs[:-1])

    th = threading.Thread(target=worker)
    th.start()
    try:
        assert ready.wait(timeout=300) and not worker_err
        t0 = time.perf_counter()
        for k in range(4):
            per_call([x, xo, xs], k)
        lib.hived_bench_save_state(x.ctx)
        got = _single(x, chunks[0], _words(chunks[0]))
        assert lib.hived_bench_num_ctas(x.ctx) == 2  # VC-parallel
        want = _single(xo, chunks[0], _words(chunks[0]))
        assert got[0] == want[0] == 0 and got[1].tobytes() == want[1].tobytes() and got[2].tobytes() == want[2].tobytes()
        assert _state(x, False) == _state(xo, False)
        both = trace.process_many([x, o], [chunks[1], chunks[0]], [_words(chunks[1]), _words(chunks[0])])
        for (rc, res, pool), ref, ev in ((both[0], xo, chunks[1]), (both[1], oo, chunks[0])):
            want = _single(ref, ev, _words(ev))
            assert rc == want[0] == 0 and res.tobytes() == want[1].tobytes() and pool.tobytes() == want[2].tobytes()
        assert _state(x, False) == _state(xo, False) and _state(o, False) == _state(oo, False)
        assert lib.hived_bench_restore_state(x.ctx) == 0
        assert _state(x, False) == _state(xs, False)
        for k in range(4, 8):
            per_call([x, xs], k)
        t1 = time.perf_counter()
        seen = len(stamps)
    finally:
        stop.set()
        th.join(timeout=600)
        for bc in (x, xo, xs, o, oo):
            bc.close()
    assert not th.is_alive()
    assert worker_err == []
    during = [s for s in stamps if t0 <= s <= t1]
    assert seen > 0 and len(during) > 0
    gaps = np.diff([t0] + during + [t1])
    assert gaps.max() < 5.0, "the third context stopped answering for %.1f s" % gaps.max()


def window_answers(lib, events, caps, flags):
    """test_shape_limits.window_answers for contexts created with `flags`."""
    out = []
    for cap in caps:
        bc = trace.BatchContext(lib, _window_cluster(), 16, 64, 1024, 16, flags=flags)
        bc.set_all_nodes_healthy()
        rc, res, pool = _process_rc(lib, bc.ctx, events, cap)
        out.append((rc, res.tobytes() if rc == 0 else None, pool.tobytes() if rc == 0 else None))
        bc.close()
    return out


def fallback_checks(lib, oracle_lib):
    """Pool above the resident slot's window (8 events, 24 576 words: the rest comes by an async copy), at the capacity
    edge; an API-fuzz seed and a batch trace against the oracle.  Returns a list of failures."""
    bad = []
    ev8 = _window_events()
    used = 8 * 3 * 1024
    caps = [used, used - 1]
    got, want = window_answers(lib, ev8, caps, FLAG), window_answers(oracle_lib, ev8, caps, 0)
    if got != want or [x[0] for x in got] != [0, ERR_CAPACITY]:
        bad.append("pool window: %r != oracle %r" % ([x[0] for x in got], [x[0] for x in want]))
    d = fuzz_api.run_seed(Flagged(lib, FLAG), oracle_lib, 9, 150)
    if d:
        bad.append(d)
    t = small_c3(300)
    ra, rb = replay(_hooks(lib), t, FLAG), replay(_hooks(oracle_lib), t, 0)
    if ra[0] != rb[0] or ra[1][:5] != rb[1][:5]:
        bad.append("batch trace differs")
    return bad


@pytest.mark.gpu
def test_gpu_pool_above_the_window(cuda_lib, oracle_lib):
    assert fallback_checks(cuda_lib, oracle_lib) == []


@pytest.mark.gpu
def test_gpu_no_resident_takes_turns(oracle_lib):
    """HIVED_NO_RESIDENT=1 (a fresh process, the switch is read at hived_create): a concurrent context's calls take
    turns with one launch each, and answer the same."""
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from hivedscheduler_b200 import _cabi\n"
            "import test_concurrent_contexts as tc\n"
            "print(json.dumps(tc.fallback_checks(_cabi.load_cuda_library(), _cabi.load_library(%r))))\n") % (
                ROOT, HERE, ORACLE_LIB)
    out = subprocess.check_output([sys.executable, "-c", code], env=dict(os.environ, HIVED_NO_RESIDENT="1"))
    assert json.loads(out.decode().strip().splitlines()[-1]) == []
