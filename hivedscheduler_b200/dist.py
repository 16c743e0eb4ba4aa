"""One calm batch of events partitioned over several GPUs (SURVEY.md section 8 row e; include/hived_multigpu.h).

One process per GPU.  Every rank holds the whole cluster; rank r owns the virtual clusters v with v % world == r.
The device program does the work; this module is the protocol's host side: two collectives per round
(all_reduce(MIN) of the next event that may touch the cluster-wide state, broadcast of that state from the event's
owner) on torch.distributed — NCCL over NVLink on GPUs, gloo in the CPU tests (against the test-only emulation
library, whose "device" pointers are host pointers).  The rest is rank plumbing for bench.py."""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence, Tuple

from . import _cabi

DONE = 0x7FFFFFFF


def dist_env() -> Tuple[int, int, int]:
    """(rank, world_size, local_rank) from the torchrun environment (defaults: single process)."""
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")),
            int(os.environ.get("LOCAL_RANK", "0")))


def max_over_ranks(values: Sequence[float], device: str = "cpu") -> List[float]:
    """Element-wise MAX of per-rank timings (identity without an initialised process group)."""
    import torch
    import torch.distributed as dist
    t = torch.tensor(list(values), dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return [float(x) for x in t.tolist()]


def aggregate_throughput(units_per_rank: int, steps: int, seconds_max: float, world: int) -> float:
    """Whole-job throughput of `world` replicas: all units of all ranks over the slowest rank's time."""
    return world * units_per_rank * steps / seconds_max


def vc_owner(vc: int, n_partitions: int) -> int:
    """The partition (CTA inside a GPU, rank across GPUs) that owns a virtual cluster's events — the engine's rule."""
    return vc % n_partitions


def bind_multigpu(lib: C.CDLL) -> None:
    """Type the entry points of include/hived_multigpu.h on a library loaded with _cabi.load_library."""
    P = C.c_void_p
    lib.hived_mg_stage.restype = C.c_int
    lib.hived_mg_stage.argtypes = [P, C.POINTER(_cabi.Event), C.c_int32, C.c_int64, C.c_int32, C.c_int32]
    lib.hived_mg_reset.restype = C.c_int
    lib.hived_mg_reset.argtypes = [P]
    lib.hived_mg_run.restype = C.c_int
    lib.hived_mg_run.argtypes = [P, C.POINTER(C.c_int32)]
    lib.hived_mg_run_window.restype = C.c_int
    lib.hived_mg_run_window.argtypes = [P, C.c_int32, C.POINTER(C.c_int32)]
    lib.hived_mg_solo.restype = C.c_int
    lib.hived_mg_solo.argtypes = [P, C.c_int32]
    lib.hived_mg_shared_bytes.restype = C.c_int64
    lib.hived_mg_shared_bytes.argtypes = [P]
    lib.hived_mg_export_shared.restype = C.c_int
    lib.hived_mg_export_shared.argtypes = [P, C.c_void_p]
    lib.hived_mg_import_shared.restype = C.c_int
    lib.hived_mg_import_shared.argtypes = [P, C.c_void_p]
    lib.hived_mg_finish.restype = C.c_int
    lib.hived_mg_finish.argtypes = [P]
    lib.hived_bench_fetch_results.restype = C.c_int
    lib.hived_bench_fetch_results.argtypes = [P, C.POINTER(_cabi.Result), C.POINTER(C.c_int32), C.c_int64, C.POINTER(C.c_int64)]
    lib.hived_mg_chain_hash.restype = C.c_int
    lib.hived_mg_chain_hash.argtypes = [C.POINTER(_cabi.Event), C.c_int32, C.c_int32, C.POINTER(C.c_void_p),
                                        C.POINTER(C.c_void_p), C.c_uint64, C.POINTER(C.c_uint64)]


def _check(lib, ctx, rc: int, what: str) -> None:
    if rc != 0:
        msg = lib.hived_last_error(ctx)
        raise RuntimeError("%s failed: rc=%d %s" % (what, rc, msg.decode() if msg else ""))


def run_partitioned(lib: C.CDLL, ctx, events, n: int, pool_cap: int, rank: int, world: int, device: Optional[str] = None,
                    staged: bool = False, window: Optional[int] = None) -> dict:
    """Drive one partitioned batch on this rank (collective: every rank of the process group calls it with the same
    batch).  `device`: torch device of the exchange buffer ("cuda:k" for the product library; "cpu" for the
    emulation library under gloo).  Returns {"rounds": events run alone on the cluster, "solo_here": those this rank ran,
    "shared_bytes": bytes of one broadcast, "collective_s": host time inside the two collectives (waiting for the
    slowest rank included), "windows": horizon advances}.  `window`: events per horizon step (default
    HIVED_MG_WINDOW or 1024; 0 = no horizon, the first form of the protocol)."""
    import torch
    import torch.distributed as dist
    if not staged:
        _check(lib, ctx, lib.hived_mg_stage(ctx, events, n, pool_cap, rank, world), "hived_mg_stage")
    multi = world > 1
    dev = device or "cpu"
    nbytes = int(lib.hived_mg_shared_bytes(ctx))
    buf = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev) if multi else None
    # who owns an event: only the owner of the winning event needs to know, and it knows (its stop == the minimum);
    # the broadcast needs the owner's RANK on every rank: a second MIN over (stop == E ? rank : world)
    import time
    rounds = solo_here = windows = 0
    t_coll = 0.0
    stop = C.c_int32(0)
    if window is None:
        window = int(os.environ.get("HIVED_MG_WINDOW", "1024"))
    horizon = window if window > 0 else DONE
    while True:
        _check(lib, ctx, lib.hived_mg_run_window(ctx, min(horizon, DONE), C.byref(stop)), "hived_mg_run_window")
        mine = int(stop.value)
        tc = time.perf_counter()
        if multi:
            # one all_reduce: (event << 8 | rank) is monotone in the event and names the owner
            key = torch.tensor([mine * 256 + rank if mine != DONE else DONE * 256], dtype=torch.int64, device=dev)
            dist.all_reduce(key, op=dist.ReduceOp.MIN)
            k = int(key.item())
            e_min, owner = (DONE, -1) if k >= DONE * 256 else (k // 256, k % 256)
        else:
            e_min, owner = mine, 0
        t_coll += time.perf_counter() - tc
        if e_min == DONE:
            if horizon >= n:
                break
            horizon += window
            windows += 1
            continue
        rounds += 1
        if owner == rank:
            _check(lib, ctx, lib.hived_mg_solo(ctx, e_min), "hived_mg_solo")
            solo_here += 1
            if multi:
                lib.hived_mg_export_shared(ctx, C.c_void_p(buf.data_ptr()))
        if multi:
            tc = time.perf_counter()
            dist.broadcast(buf, src=owner)
            if dev != "cpu":
                torch.cuda.current_stream().synchronize()
            t_coll += time.perf_counter() - tc
            if owner != rank:
                lib.hived_mg_import_shared(ctx, C.c_void_p(buf.data_ptr()))
    _check(lib, ctx, lib.hived_mg_finish(ctx), "hived_mg_finish")
    return {"rounds": rounds, "solo_here": solo_here, "shared_bytes": nbytes, "collective_s": t_coll, "windows": windows,
            "window": window}


def chain_hash(lib: C.CDLL, events, n: int, world: int, results: Sequence, pools: Sequence, seed: int = 0xCBF29CE484222325) -> int:
    """Chain hash (include/hived_hash.h) of the merged results: results[r] / pools[r] = what rank r fetched."""
    res_p = (C.c_void_p * world)(*[C.cast(r, C.c_void_p) for r in results])
    pool_p = (C.c_void_p * world)(*[C.cast(p, C.c_void_p) for p in pools])
    out = C.c_uint64(0)
    rc = lib.hived_mg_chain_hash(events, n, world, res_p, pool_p, C.c_uint64(seed), C.byref(out))
    if rc != 0:
        raise RuntimeError("hived_mg_chain_hash failed: rc=%d" % rc)
    return int(out.value)


def fetch_results(lib: C.CDLL, ctx, n: int, pool_cap: int):
    """(results, pool, used words) of the batch just run on this rank: records of other ranks' events are all-zero."""
    import numpy as np
    from .trace import RESULT_DT
    res = np.zeros(max(n, 1), dtype=RESULT_DT)
    pool = np.zeros(max(pool_cap, 1), dtype=np.int32)
    used = C.c_int64(0)
    rc = lib.hived_bench_fetch_results(ctx, res.ctypes.data_as(C.POINTER(_cabi.Result)), pool.ctypes.data_as(C.POINTER(C.c_int32)),
                                       pool_cap, C.byref(used))
    _check(lib, ctx, rc, "hived_bench_fetch_results")
    return res[:n], pool, int(used.value)
