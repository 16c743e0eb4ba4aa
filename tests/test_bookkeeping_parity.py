"""Parity of the state that decides FUTURE picks: the free, bad-free and per-VC doomed-bad lists in list order and the
vcFree / allVCFree / totalLeft / allVCDoomed counters (hived_debug_bookkeeping_hash, defined alike in the device
library and the oracle).  A mistake there shows in no result until it changes a later decision.

The reference's doomed-bad lists are slices that keep stale entries: releaseBadCell (hived_algorithm.go:1487-1500)
unbinds a doomed bad cell below a released bad preassigned cell without taking it off its VC's list, so a later
tryBindDoomedBadCell can grow the list past the VC's preassigned cells of that level.  The device program gives each
segment DM_STALE_SLACK entries of room for that (hived_topo.hpp).  Overflowing the slack (HIVED_ERR_CAPACITY) is not
tested: it needs 17 stale entries in one (VC, level) segment, and no API sequence found on the test clusters leaves
more than one — each stale entry needs a bad preassigned cell released above a doomed one, and the next
tryUnbindDoomedBadCell that meets a stale entry at the head of the list ends the run with the reference's nil
dereference (a platform error on both sides).
"""
import copy
import ctypes as C
import json
import os
import subprocess
import sys

import pytest

import fuzz_api
from conftest import snapshot_bytes
from hivedscheduler_b200 import algorithm as alg
from hivedscheduler_b200 import trace
from hivedscheduler_b200.config import new_config
from test_device_program_emu import small_c3, small_cluster

HERE = os.path.dirname(os.path.abspath(__file__))
SEED_2098_ENV = {"FUZZ_CLUSTER": "synthetic", "FUZZ_RENAME": "0.0", "FUZZ_FILTERING": "1"}


def _hooks(lib):
    for hook in (lib.hived_debug_view_hash, lib.hived_debug_bookkeeping_hash):
        hook.restype = C.c_uint64
        hook.argtypes = [C.c_void_p]
    return lib


def _bookkeeping(lib, ctx):
    return int(_hooks(lib).hived_debug_bookkeeping_hash(ctx))


# ---- seed 2098 of the API fuzz: the doomed-bad list of vcA at the RACK level outgrew its one preassigned cell

def _seed_2098(lib, oracle_lib, monkeypatch):
    for k, v in SEED_2098_ENV.items():
        monkeypatch.setenv(k, v)
    assert fuzz_api.run_seed(lib, oracle_lib, 2098, 300) is None


def test_seed_2098_emu(emu_lib, oracle_lib, monkeypatch):
    _seed_2098(emu_lib, oracle_lib, monkeypatch)


def test_seed_2098_simt(simt_lib, oracle_lib, monkeypatch):
    _seed_2098(simt_lib, oracle_lib, monkeypatch)


@pytest.mark.gpu
def test_seed_2098_cuda(cuda_lib, oracle_lib, monkeypatch):
    _seed_2098(cuda_lib, oracle_lib, monkeypatch)


# ---- the same divergence as an explicit call sequence (seed 2098 cut down to the 43 calls that still leave a stale
# entry in a doomed-bad list and then append behind it), replayed call by call on two implementations

def _doomed_list(oracle_lib, h, vc, level):
    f = oracle_lib.hived_oracle_doomed_bad_list
    f.restype = C.c_int32
    f.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    pre, stale = C.c_int32(), C.c_int32()
    n = f(h._ctx, vc.encode(), b"POD", level, C.byref(pre), C.byref(stale))
    return n, pre.value, stale.value


def _replay(libs):
    """Yields after every call: (call, [result per lib], [algorithm per lib])."""
    ops = json.load(open(os.path.join(HERE, "golden", "doomed_bad_stale_ops.json")))
    cfg = fuzz_api.synthetic_fixture()["design_config"]
    hs = [alg.HivedAlgorithm(new_config(copy.deepcopy(cfg)), lib=lib, max_groups=1024, max_pods=4096,
                             max_group_leaves=128, max_group_pods=16) for lib in libs]
    pods = [{} for _ in hs]  # uid -> ("allocated" | "preempting", pod)
    try:
        for n in hs[0].node_names:
            for h in hs:
                h.setHealthyNode(n)
        for op in ops:
            res = []
            for k, h in enumerate(hs):
                kind = op[0]
                if kind == "Schedule":
                    spec, uid, sugg, phase = op[1:]
                    pod = alg.Pod(name=uid, namespace="fz", uid=uid, annotations={alg.ANNOTATION_POD_SCHEDULING_SPEC: spec})
                    r = fuzz_api._call(lambda: fuzz_api._norm(h.Schedule(pod, sugg, phase)))
                    if r[0] == "ok" and r[1][0] == "bind":
                        bound = alg.new_binding_pod(pod, r[1][1])
                        r = (r, fuzz_api._call(lambda: h.AddAllocatedPod(bound)))
                        pods[k][uid] = ("allocated", bound)
                    elif r[0] == "ok" and r[1][0] == "preempt" and phase == alg.PREEMPTING_PHASE:
                        pods[k][uid] = ("preempting", pod)
                elif kind in ("DeleteAllocatedPod", "DeleteUnallocatedPod"):
                    want = "allocated" if kind == "DeleteAllocatedPod" else "preempting"
                    if pods[k].get(op[1], ("",))[0] != want:
                        r = ("skipped", None)
                    else:
                        pod = pods[k].pop(op[1])[1]
                        r = fuzz_api._call(lambda: getattr(h, kind)(pod))
                else:
                    r = fuzz_api._call(lambda: getattr(h, kind)(op[1]))
                res.append(r)
            yield op, res, hs
    finally:
        for h in hs:
            h.close()


def _scenario(lib, oracle_lib):
    _hooks(lib)
    _hooks(oracle_lib)
    longest, pre, stale = 0, 0, 0
    for i, (op, res, hs) in enumerate(_replay([lib, oracle_lib])):
        what = "call %d %s(%s)" % (i, op[0], op[2] if op[0] == "Schedule" else op[1])
        assert res[0] == res[1], what
        assert "platform" not in repr(res[1]), what
        assert snapshot_bytes(lib, hs[0]._ctx) == snapshot_bytes(oracle_lib, hs[1]._ctx), what
        assert lib.hived_debug_view_hash(hs[0]._ctx) == oracle_lib.hived_debug_view_hash(hs[1]._ctx), what
        assert lib.hived_debug_bookkeeping_hash(hs[0]._ctx) == oracle_lib.hived_debug_bookkeeping_hash(hs[1]._ctx), what
        n, pre, s = _doomed_list(oracle_lib, hs[1], "vcA", 4)
        longest, stale = max(longest, n), max(stale, s)
    # a stale entry was left in vcA's RACK-level list, and the list then outgrew the VC's one preassigned RACK cell
    assert stale >= 1 and pre == 1 and longest == 2, (stale, pre, longest)


def test_stale_doomed_entry_scenario_emu(emu_lib, oracle_lib):
    _scenario(emu_lib, oracle_lib)


def test_stale_doomed_entry_scenario_simt(simt_lib, oracle_lib):
    _scenario(simt_lib, oracle_lib)


@pytest.mark.gpu
def test_stale_doomed_entry_scenario_cuda(cuda_lib, oracle_lib):
    _scenario(cuda_lib, oracle_lib)


# ---- bookkeeping after every chunk of the batch traces test_gpu_parity replays

TRACES = ["C1", "C2", "C3-small", "multi-member", "heterogeneous", "suggested-nodes", "bad-requests", "C5-churn"]


def make_trace(name):
    if name == "C5-churn":
        return trace.trace_c5(n_steps=4, gangs_per_step=300, n_nodes=4 * 16 * 32, n_vcs=2, vc_gpus=(16 + 6) * 32 * 8,
                              config=small_cluster())
    return {"C1": trace.trace_c1, "C2": trace.trace_c2, "C3-small": small_c3, "multi-member": trace.trace_multi_member,
            "heterogeneous": trace.trace_heterogeneous, "suggested-nodes": trace.trace_suggested_nodes,
            "bad-requests": trace.trace_bad_requests}[name]()


def chunk_hashes(lib, t, chunks=4):
    """(result hash, bookkeeping hash) after every chunk of the trace."""
    bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
    bc.set_all_nodes_healthy()
    ev = t["events"]
    out, start = [], 0
    for i in range(chunks):
        end = len(ev) * (i + 1) // chunks
        bc.process(ev[start:end], 3 * 64 * (end - start) + 4096, t.get("sugg_pool"))
        out.append((bc.result_hash(), _bookkeeping(lib, bc.ctx)))
        start = end
    bc.close()
    return out


@pytest.mark.parametrize("name", TRACES)
def test_trace_bookkeeping_emu(emu_lib, oracle_lib, name):
    t = make_trace(name)
    assert chunk_hashes(emu_lib, t) == chunk_hashes(oracle_lib, t)


@pytest.mark.parametrize("name", TRACES)
def test_trace_bookkeeping_simt(simt_lib, oracle_lib, name):
    t = make_trace(name)
    assert chunk_hashes(simt_lib, t) == chunk_hashes(oracle_lib, t)


@pytest.mark.gpu
@pytest.mark.parametrize("ncta", ["1", "16"])
@pytest.mark.parametrize("name", TRACES)
def test_trace_bookkeeping_cuda(cuda_lib, oracle_lib, name, ncta):
    """On the GPU with HIVED_NCTA CTAs (a fresh process: the CTA count is fixed when the library starts): at 16 the VCs
    run in parallel and the chain-wide free lists are updated inside the ordered shared sections."""
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from hivedscheduler_b200 import _cabi\n"
            "import test_bookkeeping_parity as tb\n"
            "print(json.dumps(tb.chunk_hashes(_cabi.load_cuda_library(), tb.make_trace(%r))))\n") % (
                os.path.dirname(HERE), HERE, name)
    out = subprocess.check_output([sys.executable, "-c", code], env=dict(os.environ, HIVED_NCTA=ncta))
    got = [tuple(x) for x in json.loads(out.decode().strip().splitlines()[-1])]
    assert got == chunk_hashes(oracle_lib, make_trace(name))
