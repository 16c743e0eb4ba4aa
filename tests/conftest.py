import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ORACLE_LIB = os.path.join(ROOT, "oracle", "libhived_oracle.so")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def _build_oracle():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])


@pytest.fixture(scope="session")
def oracle_lib():
    """The CPU oracle behind the same C ABI (test infrastructure only)."""
    from hivedscheduler_b200 import _cabi
    _build_oracle()
    return _cabi.load_library(ORACLE_LIB)


@pytest.fixture(scope="session")
def cuda_lib():
    """The product library; GPU tests fail loudly if it is missing or no device is present."""
    from hivedscheduler_b200 import _cabi
    return _cabi.load_cuda_library()


EMU_LIB = os.path.join(ROOT, "tests", "_build", "libhived_emu.so")


@pytest.fixture(scope="session")
def emu_lib():
    """Host emulation of the DEVICE PROGRAM (1-thread CTA) — test-only, validates kernel logic on CPU."""
    from hivedscheduler_b200 import _cabi
    os.makedirs(os.path.dirname(EMU_LIB), exist_ok=True)
    src = os.path.join(ROOT, "tests", "emu", "hived_emu.cpp")
    deps = [src] + [os.path.join(ROOT, "hivedscheduler_b200", "csrc", f)
                    for f in os.listdir(os.path.join(ROOT, "hivedscheduler_b200", "csrc")) if f.endswith((".h", ".hpp", ".inc"))]
    if not os.path.exists(EMU_LIB) or any(os.path.getmtime(d) > os.path.getmtime(EMU_LIB) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-o", EMU_LIB, src])
    return _cabi.load_library(EMU_LIB)


@pytest.fixture(scope="session")
def emu_mt_lib():
    """The DEVICE PROGRAM on host threads (one 1-lane "CTA" per thread, tests/emu/hived_emu_mt.cpp) — test / bench only."""
    from hivedscheduler_b200 import _cabi
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    return _cabi.load_library(g.build_cpu_flat())


def run_trace(lib, t, n_events=None, chunks=1, device=0, snapshots=None):
    """Replay a trace on a library; returns (hash, results, pool, stats)."""
    import numpy as np
    from hivedscheduler_b200 import trace
    bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"],
                            device=device)
    bc.set_all_nodes_healthy()
    ev = t["events"] if n_events is None else t["events"][:n_events]
    bounds = [len(ev) * (i + 1) // chunks for i in range(chunks)]
    start, all_res = 0, []
    for b in bounds:
        res, pool = bc.process(ev[start:b], 3 * 64 * (b - start) + 4096, t.get("sugg_pool"))
        all_res.append((res, pool))
        start = b
    out = (bc.result_hash(), all_res, bc.stats())
    if snapshots is not None:
        snapshots.append(snapshot_bytes(lib, bc.ctx))
    bc.close()
    return out


def snapshot_bytes(lib, ctx):
    """Every cell's (priority, state, health, binding, split/pinned/in-free-list) — the raw material of
    GetClusterStatus (hived_algorithm.go:323-363) — as bytes, for cross-implementation comparison."""
    import ctypes as C
    from hivedscheduler_b200 import _cabi
    n_p, n_v = lib.hived_num_physical_cells(ctx), lib.hived_num_virtual_cells(ctx)
    ps, vs = (_cabi.CellStatus * n_p)(), (_cabi.CellStatus * n_v)()
    assert lib.hived_snapshot_physical(ctx, ps, n_p) == 0
    assert lib.hived_snapshot_virtual(ctx, vs, n_v) == 0
    return bytes(ps) + bytes(vs)


SIMT_LIB = os.path.join(ROOT, "tests", "_build", "libhived_simt.so")


@pytest.fixture(scope="session")
def simt_lib():
    """Functional SIMT emulation of the DEVICE PROGRAM with the kernel's real geometry (32-lane warps, leader + worker
    warps, one CTA per group of VCs; tests/emu/simt_rt.h) — test-only, covers the warp-level code and the ordered
    shared sections between CTAs on a box without a GPU."""
    from hivedscheduler_b200 import _cabi
    os.makedirs(os.path.dirname(SIMT_LIB), exist_ok=True)
    src = os.path.join(ROOT, "tests", "emu", "hived_simt.cpp")
    deps = [src, os.path.join(ROOT, "tests", "emu", "simt_rt.h")] + [
        os.path.join(ROOT, "hivedscheduler_b200", "csrc", f)
        for f in os.listdir(os.path.join(ROOT, "hivedscheduler_b200", "csrc")) if f.endswith((".h", ".hpp", ".inc"))]
    if not os.path.exists(SIMT_LIB) or any(os.path.getmtime(d) > os.path.getmtime(SIMT_LIB) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-o", SIMT_LIB, src])
    return _cabi.load_library(SIMT_LIB)
