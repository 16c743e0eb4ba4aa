"""Concurrent contexts' batches (HIVED_OPT_CONCURRENT, include/hived.h "Threads"): a batch the per-call path does not take
runs on the context's own stream and CTAs, at the same time as other contexts' batches and calls, without a turn on the
library's device lock.

CPU tier: the co-residency seat ledger (hivedscheduler_b200/csrc/hived_seats.h) driven from many threads.  GPU tier:
every answer compared with the oracle run one context at a time (rc, results and pool bytes per batch; at the end the
result hash, work counters, cell snapshots, view-order and bookkeeping hashes), and hived_bench_turns shows that the
batches took no turn."""
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

from conftest import ORACLE_LIB, ROOT
from hivedscheduler_b200 import _cabi, frontend as fe_mod, trace
from test_concurrent_contexts import FLAG, PerCall
from test_device_program_emu import small_c3
from test_frontend import MAXG, MAXP, cluster, fe_answer, mirror_answers, workload
from test_many_contexts import SPARE, _ctx, _hooks, _single, _state, _words, c3_ctx_trace

HERE = os.path.dirname(os.path.abspath(__file__))
ERR_CAPACITY = 102  # HIVED_ERR_CAPACITY
ORACLE_C3_HASH = 0xe3becf53c2d32f79  # the oracle's result hash on the full-size C3 trace (bench.py's parity witness)


# ---- CPU tier ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cap,threads,seed", [(132, 24, 1), (7, 16, 2)])
def test_seat_ledger_under_many_threads(tmp_path, cap, threads, seed):
    """Random requests from many threads never hold more than the capacity and all complete; grants follow arrival
    order; a request larger than the device is refused."""
    exe = str(tmp_path / "seat_ledger_stress")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", "-o", exe,
                           os.path.join(HERE, "harness", "seat_ledger_stress.cpp")])
    out = subprocess.run([exe, str(cap), str(threads), "200", str(seed)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr


# ---- GPU tier ---------------------------------------------------------------------------------------------------------

def mixed_priority(t):
    """The trace with every seventh group at priority 1: two priorities in use, so every batch runs on one CTA."""
    t = dict(t)
    ev = t["events"].copy()
    sched = ev["type"] == 0
    ev["spec"]["priority"][sched] = np.where(ev["spec"]["group"][sched] % 7 == 0, 1, 0)
    t["events"], t["name"] = ev, t["name"] + "-mixed"
    return t


def _per_call(bc, t, k):
    """One pod scheduled (hived_process_events, n = 1) and a node set bad and healthy again: the per-call path."""
    tb = trace.TraceBuilder(1)
    tb.schedule(group=t["n_groups"] + k, vc=k % 2, priority=0, leaf_type=0, leaf_num=8, pod_num=1)
    ev = tb.finish()[0]
    ev["spec"]["pod"] = t["n_pods"] + k
    rc, res, pool = _single(bc, ev, 256)
    node = (7 * k) % bc.n_nodes
    health = (bc.lib.hived_set_node_health(bc.ctx, node, 0), bc.lib.hived_set_node_health(bc.ctx, node, 1))
    return rc, res.tobytes(), pool.tobytes(), health


def script(bc, t, sizes=(9, 64, 1000)):
    """Batches of the given sizes and then the rest of the trace, a per-call step after each; every answer kept."""
    ev, out, at = t["events"], [], 0
    for k, size in enumerate(list(sizes) + [len(ev)]):
        chunk = ev[at:at + size]
        if len(chunk) == 0:
            break
        rc, res, pool = _single(bc, chunk, _words(chunk))
        out.append(("batch", rc, res.tobytes(), pool.tobytes(), bc.lib.hived_bench_num_ctas(bc.ctx)
                    if hasattr(bc.lib, "hived_bench_num_ctas") else None))
        out.append(("per-call",) + _per_call(bc, t, k))
        at += len(chunk)
    return out


def answers(out):
    """script's answers without the CTA counts of its batches (the oracle runs everything on one)."""
    return [o[:-1] if o[0] == "batch" else o for o in out]


_oracle_cache = {}


def oracle_script(oracle_lib, t, sizes=(9, 64, 1000)):
    key = (t["name"], len(t["events"]), tuple(sizes))
    if key not in _oracle_cache:
        bc = _ctx(_hooks(oracle_lib), t)
        out = script(bc, t, sizes)
        _oracle_cache[key] = (answers(out), _state(bc, False))
        bc.close()
    return _oracle_cache[key]


def run_threads(fns, timeout=600):
    errs, out = [], [None] * len(fns)

    def work(i):
        try:
            out[i] = fns[i]()
        except BaseException as e:  # noqa
            errs.append(repr(e))

    th = [threading.Thread(target=work, args=(i,)) for i in range(len(fns))]
    for x in th:
        x.start()
    for x in th:
        x.join(timeout=timeout)
    assert not any(x.is_alive() for x in th), "a thread did not finish"
    assert errs == []
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 4, 16])
def test_gpu_threads_each_run_batches_on_a_concurrent_context(cuda_lib, oracle_lib, k):
    """k threads, each on its own concurrent context: half run a C3-shaped 8-VC trace (VC-parallel from 256 events on),
    half a mixed-priority one (one CTA).  Batches of 9, 64 and 1 000 events and then the rest, per-call steps in between,
    every answer as the oracle's, and not one turn on the device lock after hived_create."""
    lib = _hooks(cuda_lib)
    base = c3_ctx_trace(8, 1500)
    ts = [base, mixed_priority(base)]
    bcs = [trace.BatchContext(lib, ts[i % 2]["config"], ts[i % 2]["n_groups"] + SPARE, ts[i % 2]["n_pods"] + 64 * SPARE,
                              ts[i % 2]["max_group_leaves"], ts[i % 2]["max_group_pods"], flags=FLAG) for i in range(k)]
    for bc in bcs:
        bc.set_all_nodes_healthy()
    turns0 = [bc.turns() for bc in bcs]
    got = run_threads([lambda bc=bc, i=i: script(bc, ts[i % 2]) for i, bc in enumerate(bcs)])
    try:
        for i, (bc, out) in enumerate(zip(bcs, got)):
            want, state = oracle_script(oracle_lib, ts[i % 2])
            assert answers(out) == want, (i, ts[i % 2]["name"])
            assert _state(bc, False) == state
            ctas = [o[-1] for o in out if o[0] == "batch"]
            assert ctas[:3] == ([1, 1, 8] if i % 2 == 0 else [1, 1, 1]), ctas
        assert [bc.turns() for bc in bcs] == turns0
    finally:
        for bc in bcs:
            bc.close()


@pytest.mark.gpu
def test_gpu_small_batches_run_while_a_full_size_batch_is_in_flight(cuda_lib, oracle_lib):
    """Thread A runs one full-size C3 batch (100 000 gangs, VC-parallel); thread B's concurrent context completes at
    least 10 batches of 64 events while A's call is in flight."""
    lib = _hooks(cuda_lib)
    big = trace.trace_c3(n_gangs=100000)
    small = c3_ctx_trace(2, 20000)
    a = trace.BatchContext(lib, big["config"], big["n_groups"], big["n_pods"], big["max_group_leaves"],
                           big["max_group_pods"], flags=FLAG)
    a.set_all_nodes_healthy()
    b = trace.BatchContext(lib, small["config"], small["n_groups"] + SPARE, small["n_pods"] + 64 * SPARE,
                           small["max_group_leaves"], small["max_group_pods"], flags=FLAG)
    b.set_all_nodes_healthy()
    turns0 = (a.turns(), b.turns())
    started, a_done = threading.Event(), threading.Event()
    span, stamps, b_out = [], [], []

    def run_a():
        started.wait(60)
        ev = big["events"]
        t0 = time.perf_counter()
        got = _single(a, ev, trace.pool_words_for(big))
        span.extend([t0, time.perf_counter()])
        a_done.set()
        return got[0]

    def run_b():
        ev, at = small["events"], 0
        while at + 64 <= len(ev):
            chunk = ev[at:at + 64]
            rc, res, pool = _single(b, chunk, _words(chunk))
            b_out.append((rc, res.tobytes(), pool.tobytes()))
            stamps.append((time.perf_counter()))
            at += 64
            started.set()
            if a_done.is_set() and len(stamps) > 20:
                break
        started.set()
        return at

    rc_a, b_end = run_threads([run_a, run_b])
    try:
        assert rc_a == 0 and a.result_hash() == ORACLE_C3_HASH
        during = [s for s in stamps if span[0] < s < span[1]]
        assert len(during) >= 10, "B completed %d batches during A's %.2f s call" % (len(during), span[1] - span[0])
        ref = _ctx(_hooks(oracle_lib), small)
        ev = small["events"]
        for i, got in enumerate(b_out):
            want = _single(ref, ev[64 * i:64 * (i + 1)], _words(ev[64 * i:64 * (i + 1)]))
            assert got == (want[0], want[1].tobytes(), want[2].tobytes()), i
        assert _state(b, False) == _state(ref, False)
        ref.close()
        assert (a.turns(), b.turns()) == turns0
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_gpu_seat_pressure(cuda_lib, oracle_lib):
    """16 concurrent contexts of 16 VCs each run VC-parallel batches at once (256 CTAs against the seats left beside
    their resident kernels), while a turn-taking context runs a VC-parallel batch and two more contexts make a joint
    call.  Everything finishes, and everything answers as the oracle."""
    lib = _hooks(cuda_lib)
    t = c3_ctx_trace(16, 1500)
    ev = t["events"]
    conc = [trace.BatchContext(lib, t["config"], t["n_groups"] + SPARE, t["n_pods"] + 64 * SPARE, t["max_group_leaves"],
                               t["max_group_pods"], flags=FLAG) for _ in range(_cabi.HIVED_CONCURRENT_MAX)]
    plain = [_ctx(lib, t) for _ in range(3)]
    for bc in conc:
        bc.set_all_nodes_healthy()
    ref = _ctx(_hooks(oracle_lib), t)
    want = _single(ref, ev, _words(ev))
    want = (want[0], want[1].tobytes(), want[2].tobytes())
    turns0 = [bc.turns() for bc in conc]

    def one(bc):
        rc, res, pool = _single(bc, ev, _words(ev))
        return (rc, res.tobytes(), pool.tobytes()), lib.hived_bench_num_ctas(bc.ctx)

    def joint():
        got = trace.process_many(plain[1:], [ev, ev], [_words(ev)] * 2)
        return [((rc, res.tobytes(), pool.tobytes()), 16) for rc, res, pool in got]

    try:
        outs = run_threads([lambda bc=bc: one(bc) for bc in conc + plain[:1]] + [joint])
        outs = outs[:-1] + outs[-1]
        assert all(o == (want, 16) for o in outs)
        state = _state(ref, False)
        assert all(_state(bc, False) == state for bc in conc + plain)
        assert [bc.turns() for bc in conc] == turns0
    finally:
        for bc in conc + plain + [ref]:
            bc.close()


@pytest.mark.gpu
def test_gpu_buffers_grow_under_per_call_traffic(cuda_lib, oracle_lib):
    """Thread A keeps per-call requests coming on its concurrent context until B is done; thread B runs batches each
    larger than the last, so its staging must grow while A's resident kernel never goes idle.  B finishes; both answer
    as the oracle."""
    lib = _hooks(cuda_lib)
    tb_ = small_c3(4000)
    ev = tb_["events"]
    sizes, at = [], 0
    size = 9
    while at < len(ev):
        sizes.append(min(size, len(ev) - at))
        at += sizes[-1]
        size = int(size * 1.7) + 1
    a = PerCall(lib, small_c3(10), FLAG)
    b = trace.BatchContext(lib, tb_["config"], tb_["n_groups"], tb_["n_pods"], tb_["max_group_leaves"],
                           tb_["max_group_pods"], flags=FLAG)
    b.set_all_nodes_healthy()
    b_done = threading.Event()
    b_out = []

    def run_a():
        deadline = time.time() + 30
        while not b_done.is_set():
            if time.time() > deadline:
                raise AssertionError("B did not finish within 30 s of per-call traffic")
            a.schedule()
            a.delete()
        return a.calls()

    def run_b():
        try:
            at = 0
            for n in sizes:
                chunk = ev[at:at + n]
                rc, res, pool = _single(b, chunk, _words(chunk))
                b_out.append((rc, res.tobytes(), pool.tobytes()))
                at += n
        finally:
            b_done.set()

    try:
        calls, _ = run_threads([run_a, run_b])
        assert calls > 0 and len(b_out) == len(sizes)
        ref = _ctx(_hooks(oracle_lib), tb_)
        at = 0
        for n, got in zip(sizes, b_out):
            chunk = ev[at:at + n]
            want = _single(ref, chunk, _words(chunk))
            assert got == (want[0], want[1].tobytes(), want[2].tobytes()), n
            at += n
        assert _state(b, False) == _state(ref, False)
        ref.close()
        ra = PerCall(oracle_lib, small_c3(10))
        while ra.calls() < a.calls():
            ra.schedule()
            ra.delete()
        assert a.answers == ra.answers[:len(a.answers)]
        ra.close()
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_gpu_edges_of_a_concurrent_batch(cuda_lib, oracle_lib):
    """On a concurrent context: a pool one word short gives HIVED_ERR_CAPACITY for that batch alone; a batch with a
    suggested-node pool; a batch right after the context's own per-call operations, then a joint call and a state rewind.
    All as the oracle, with no turn taken outside the joint call and the rewind."""
    lib = _hooks(cuda_lib)
    lib.hived_bench_save_state.argtypes = lib.hived_bench_restore_state.argtypes = [C.c_void_p]
    ora = _hooks(oracle_lib)

    t = small_c3(600)
    ev, rest = t["events"][:400], t["events"][400:]

    def pair(flags=FLAG):
        out = [trace.BatchContext(lb, t["config"], t["n_groups"] + SPARE, t["n_pods"] + 64 * SPARE,
                                  t["max_group_leaves"], t["max_group_pods"], flags=flags if lb is lib else 0)
               for lb in (lib, ora)]
        for bc in out:
            bc.set_all_nodes_healthy()
        return out

    def same(got, want):
        assert got[0] == want[0] and got[1].tobytes() == want[1].tobytes() and got[2].tobytes() == want[2].tobytes()

    # a pool one word short gives HIVED_ERR_CAPACITY, and the next batch on the same context runs as usual.  Compared
    # with the oracle (rc, results, pool) and with the same library without the flag (also the state: after an event
    # that ran out of room the device program's work counters already count its placement, the oracle's do not)
    x, xo = pair()
    want = _single(xo, ev, _words(ev))
    used = int(max([r["leaf_off"] + 3 * r["n_leaves"] for r in want[1] if r["kind"] == 1] + [0]))
    x.close()
    xo.close()
    for words in (used - 1, used):
        x, xo = pair()
        xp, spare = pair(0)
        spare.close()
        turns0 = x.turns()
        for batch, cap in ((ev, words), (rest, _words(rest))):
            got, plain, want = _single(x, batch, cap), _single(xp, batch, cap), _single(xo, batch, cap)
            assert got[0] == plain[0] == want[0] == (ERR_CAPACITY if cap < used else 0)
            if got[0] == 0:
                same(got, plain)
                same(got, want)
            assert _state(x, True) == _state(xp, True)
        if words == used:
            assert _state(x, False) == _state(xo, False)
        assert x.turns() == turns0
        for bc in (x, xp, xo):
            bc.close()

    # a suggested-node pool
    ts = trace.trace_suggested_nodes(n_gangs=300)
    s, so = (trace.BatchContext(lb, ts["config"], ts["n_groups"], ts["n_pods"], ts["max_group_leaves"],
                                ts["max_group_pods"], flags=FLAG if lb is lib else 0) for lb in (lib, ora))
    for bc in (s, so):
        bc.set_all_nodes_healthy()
    turns0 = s.turns()
    same(*(_single(bc, ts["events"], _words(ts["events"]), ts["sugg_pool"]) for bc in (s, so)))
    assert _state(s, False) == _state(so, False) and s.turns() == turns0
    s.close()
    so.close()

    # per-call operations, a batch right after them, a joint call with an ordinary context, a rewind, a batch again
    x, xo = pair()
    xs = _ctx(ora, t)  # the oracle held at the saved state
    o, oo = _ctx(lib, t), _ctx(ora, t)
    try:
        for k in range(3):
            assert _per_call(x, t, k) == _per_call(xo, t, k) == _per_call(xs, t, k)
        turns0 = x.turns()
        lib.hived_bench_save_state(x.ctx)
        same(_single(x, ev, _words(ev)), _single(xo, ev, _words(ev)))
        assert lib.hived_bench_num_ctas(x.ctx) == 2 and x.turns() == turns0  # VC-parallel, no turn
        assert _state(x, False) == _state(xo, False)
        both = trace.process_many([x, o], [rest, ev], [_words(rest), _words(ev)])
        for got, ref, e in ((both[0], xo, rest), (both[1], oo, ev)):
            same(got, _single(ref, e, _words(e)))
        assert _state(x, False) == _state(xo, False) and _state(o, False) == _state(oo, False)
        assert lib.hived_bench_restore_state(x.ctx) == 0
        assert _state(x, False) == _state(xs, False)
        same(_single(x, ev, _words(ev)), _single(xs, ev, _words(ev)))
        assert _state(x, False) == _state(xs, False)
    finally:
        for bc in (x, xo, xs, o, oo):
            bc.close()


def no_resident_checks(lib, oracle_lib):
    """A concurrent context's batches under HIVED_NO_RESIDENT=1: each takes a turn, and the answers are the oracle's.
    Returns a list of failures."""
    lib, t = _hooks(lib), c3_ctx_trace(8, 600)
    bc = trace.BatchContext(lib, t["config"], t["n_groups"] + SPARE, t["n_pods"] + 64 * SPARE, t["max_group_leaves"],
                            t["max_group_pods"], flags=FLAG)
    bc.set_all_nodes_healthy()
    turns0 = bc.turns()
    out = script(bc, t)
    bad = []
    want, state = oracle_script(oracle_lib, t)
    if answers(out) != want or _state(bc, False) != state:
        bad.append("answers differ from the oracle")
    if bc.turns() < turns0 + 4:
        bad.append("batches took no turns: %d -> %d" % (turns0, bc.turns()))
    bc.close()
    return bad


@pytest.mark.gpu
def test_gpu_no_resident_batches_take_turns():
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from hivedscheduler_b200 import _cabi\n"
            "import test_concurrent_batches as tb\n"
            "print(json.dumps(tb.no_resident_checks(_cabi.load_cuda_library(), _cabi.load_library(%r))))\n") % (
                ROOT, HERE, ORACLE_LIB)
    out = subprocess.check_output([sys.executable, "-c", code], env=dict(os.environ, HIVED_NO_RESIDENT="1"))
    assert json.loads(out.decode().strip().splitlines()[-1]) == []


@pytest.mark.gpu
def test_gpu_two_front_ends_on_concurrent_contexts(cuda_lib, oracle_lib):
    """Two extender front ends (include/hived_frontend.h), each over its own concurrent context and driven by a thread of
    its own at the same time as the other: its queued filter calls drained into a batch of more than 8 events.  Every
    answer is the reference-shaped mirror's, and neither context takes a turn."""
    lib = cuda_lib
    pods = workload(60)
    want = mirror_answers(oracle_lib, pods)
    fes = []
    for _ in range(2):
        bc = trace.BatchContext(lib, cluster(), MAXG, MAXP, 64, 8, flags=FLAG)
        bc.set_all_nodes_healthy()
        fes.append((fe_mod.FrontEnd(lib, bc.ctx, MAXG, MAXP), bc, bc.turns()))

    def drive(f, bc):
        for uid, key, ann in pods:
            assert f.add_unbound_pod(uid, key, ann) == 0
        tickets = {uid: f.enqueue_filter(uid) for uid, _, _ in pods}
        assert f.drain() == 0  # the queued filter calls go out as one batch
        return {uid: fe_answer(f, lib, bc, f.take(tk)) for uid, tk in tickets.items()}, f.stats()

    try:
        outs = run_threads([lambda f=f, bc=bc: drive(f, bc) for f, bc, _ in fes])
        for (got, st), (f, bc, turns0) in zip(outs, fes):
            assert got == want
            assert st["largest_batch"] > 8
            assert bc.turns() == turns0
    finally:
        for f, bc, _ in fes:
            f.close()
            bc.close()
