"""A calm batch partitioned over ranks (include/hived_multigpu.h) against the oracle's single run, event by event.

`world` contexts of one library in one process stand for the ranks; the two collectives of the protocol are done by
hand (min over the ranks' stop events; the owner's cluster-wide arrays copied to the others).  Each trace runs as one
batch or as three successive partitioned batches on the same contexts.  After every batch:

- every event's result record, DELETE_ALLOCATED included, merged by owner (a SCHEDULE by its VC, a DELETE by the VC its
  group was scheduled under, as dist.py routes them) and normalised — the record without its pool offsets, plus the
  pool words it names — equals the oracle's; the records of events a rank does not own are all-zero;
- every rank's bookkeeping hash (free lists, counters) equals the oracle's;
- on the rank that owns a VC: the snapshot records of the VC's virtual cells and of the physical cells bound into them,
  and the VC's view order (hived_debug_view_hash_vc), equal the oracle's.  Other VCs' cells and views are stale on a
  rank by design;
- the work counters summed over the ranks equal the oracle's, and the path counters summed over the ranks equal those
  of an ordinary run of the same library: every event is counted once, a stopped attempt not at all.

A batch that is not calm (suggested-node sets, node health, two priorities, a recovery, one group id under two VCs) is
refused by hived_mg_stage with HIVED_ERR_BAD_SPEC before anything runs, and leaves nothing behind that changes a later
calm batch."""
import ctypes as C

import numpy as np
import pytest

from hivedscheduler_b200 import _cabi, dist, trace
from test_device_program_emu import small_cluster

ERR_BAD_SPEC = 7           # HIVED_ERR_BAD_SPEC
EV_ADD_ALLOCATED = 17      # Core::EV_ADD_ALLOCATED (hived_core.h): the batch form of hived_add_allocated_pod
N_PATH = 12                # PC_COUNT (hived_dev.h)


def _hooks(lib):
    lib.hived_debug_bookkeeping_hash.restype = C.c_uint64
    lib.hived_debug_bookkeeping_hash.argtypes = [C.c_void_p]
    lib.hived_debug_view_hash_vc.restype = C.c_uint64
    lib.hived_debug_view_hash_vc.argtypes = [C.c_void_p, C.c_int32]
    return lib


# ---- traces (each calm: SCHEDULE / DELETE_ALLOCATED only, priority 0, every node healthy) ---------------------------

def fill_and_drain(cycles=2, gangs=300, reuse_ids=False):
    """small_cluster(): both VCs filled with `gangs` gangs (1x8, 2x8, 1x4, 1x1, alternating VCs), then every gang deleted
    pod by pod; the cycle repeats.  The last deletions of a cycle empty the VCs' preassigned cells.  reuse_ids: every
    cycle uses the same group ids, each under the other VC than in the cycle before (one cycle per batch)."""
    shapes = [(1, 8), (2, 8), (1, 4), (1, 1)]  # (pods, leaves)
    tb = trace.TraceBuilder(8 * gangs * cycles)
    for c in range(cycles):
        alive = []
        for i in range(gangs):
            g = i if reuse_ids else c * gangs + i
            v = (i + c) % 2 if reuse_ids else i % 2
            pods, leaves = shapes[i % 4]
            for j in range(pods):
                tb.schedule(group=g, vc=v, priority=0, leaf_type=0, leaf_num=leaves, pod_num=pods, first=(j == 0))
            alive.append((g, pods, leaves, v))
        for g, pods, leaves, v in alive:
            for j in range(pods):
                tb.delete_allocated(g, leaves, j, vc=v)
    ev, dec = tb.finish()
    return {"name": "fill-and-drain", "config": small_cluster(), "events": ev, "decision": dec,
            "n_groups": gangs * (1 if reuse_ids else cycles), "n_pods": tb.next_pod, "max_group_leaves": 64, "max_group_pods": 8}


def c3_emptying_racks(n_gangs=700, vc_gpus=2 * 32 * 8):
    """small_cluster() and C3's gang mix (1x1, 1x4, 1x8, 8x8), but a VC whose admission window is full lets ALL its gangs
    go, pod by pod: the deletions empty racks, and the VC's preassigned cells go back to the buddy free lists."""
    rng = trace.XorShift64Star(trace.seed_for(3))
    tb = trace.TraceBuilder(4 * n_gangs)
    alive, alive_gpus = [[], []], [0, 0]
    for g in range(n_gangs):
        pod_num, leaf_num = trace._gang_shape(rng.below(100))
        v = rng.below(2)
        if alive_gpus[v] + pod_num * leaf_num > vc_gpus:
            for og, opn, oln in alive[v]:
                for j in range(opn):
                    tb.delete_allocated(og, oln, j, vc=v)
            alive[v], alive_gpus[v] = [], 0
        for j in range(pod_num):
            tb.schedule(group=g, vc=v, priority=0, leaf_type=0, leaf_num=leaf_num, pod_num=pod_num, first=(j == 0))
        alive[v].append((g, pod_num, leaf_num))
        alive_gpus[v] += pod_num * leaf_num
    ev, dec = tb.finish()
    return {"name": "c3-emptying-racks", "config": small_cluster(), "events": ev, "decision": dec,
            "n_groups": n_gangs, "n_pods": tb.next_pod, "max_group_leaves": 64, "max_group_pods": 8}


TRACES = {
    "heterogeneous": lambda short: trace.trace_heterogeneous(n_gangs=400 if short else 1500),
    "fill-and-drain": lambda short: fill_and_drain(gangs=60 if short else 300),
    "multi-member": lambda short: trace.trace_multi_member(n_gangs=150 if short else 600),
    "c2": lambda short: trace.trace_c2(n_pods=600 if short else 2000),
    "c3-emptying-racks": lambda short: c3_emptying_racks(250 if short else 700),
}


def _reuse_trace(name, short, chunks):
    if name == "fill-and-drain" and chunks > 1:
        return fill_and_drain(cycles=chunks, gangs=60 if short else 300, reuse_ids=True)
    return TRACES[name](short)


# ---- the ranks -------------------------------------------------------------------------------------------------------

def _context(lib, t):
    bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
    bc.set_all_nodes_healthy()
    return bc


class Ranks:
    """`world` in-process contexts of one library, driven through the partition protocol batch after batch.
    alloc(nbytes) -> (keepalive, pointer) of the exchange buffer (device memory for the CUDA library)."""

    def __init__(self, lib, t, world, alloc=None):
        dist.bind_multigpu(lib)
        self.lib, self.world = _hooks(lib), world
        self.ranks = [_context(lib, t) for _ in range(world)]
        nbytes = int(lib.hived_mg_shared_bytes(self.ranks[0].ctx))
        if alloc is None:
            self._buf = np.zeros(nbytes, dtype=np.uint8)
            self.buf = self._buf.ctypes.data
        else:
            self._buf, self.buf = alloc(nbytes)
        self.group_vc = {}

    def stage(self, ev):
        ev = np.ascontiguousarray(ev)
        evp = ev.ctypes.data_as(C.POINTER(_cabi.Event))
        cap = 3 * 64 * len(ev) + 4096
        return [self.lib.hived_mg_stage(bc.ctx, evp, len(ev), cap, r, self.world) for r, bc in enumerate(self.ranks)], cap

    def run(self, ev, window=0):
        """One partitioned batch.  Returns ([(results, pool)] per rank, [(event, type)] of the events run alone, owner
        rank per event)."""
        lib = self.lib
        ev = np.ascontiguousarray(ev)
        n = len(ev)
        rcs, cap = self.stage(ev)
        assert rcs == [0] * self.world, [lib.hived_last_error(bc.ctx) for bc in self.ranks]
        solos = []
        horizon = window if window > 0 else dist.DONE
        while True:
            stops = []
            for bc in self.ranks:
                s = C.c_int32(0)
                assert lib.hived_mg_run_window(bc.ctx, min(horizon, dist.DONE), C.byref(s)) == 0, lib.hived_last_error(bc.ctx)
                stops.append(s.value)
            e = min(stops)
            if e == dist.DONE:
                if horizon >= n:
                    break
                horizon += window
                continue
            solos.append((e, int(ev["type"][e])))
            owner = stops.index(e)
            assert lib.hived_mg_solo(self.ranks[owner].ctx, e) == 0, lib.hived_last_error(self.ranks[owner].ctx)
            lib.hived_mg_export_shared(self.ranks[owner].ctx, C.c_void_p(self.buf))
            for r, bc in enumerate(self.ranks):
                if r != owner:
                    lib.hived_mg_import_shared(bc.ctx, C.c_void_p(self.buf))
        fetched = []
        for bc in self.ranks:
            assert lib.hived_mg_finish(bc.ctx) == 0, lib.hived_last_error(bc.ctx)
            res, pool, _ = dist.fetch_results(lib, bc.ctx, n, cap)
            fetched.append((res, pool))
        owners = np.zeros(n, dtype=np.int64)
        for i in range(n):  # the routing of hived_engine.hpp Engine::route
            g, v = int(ev["spec"]["group"][i]), int(ev["spec"]["vc"][i])
            if ev["type"][i] == _cabi.EV_SCHEDULE:
                self.group_vc[g] = v
            owners[i] = self.group_vc.get(g, max(v, 0)) % self.world
        return fetched, solos, owners

    def close(self):
        for bc in self.ranks:
            bc.close()


# ---- comparison --------------------------------------------------------------------------------------------------------

_OFFSETS = ("this_off", "leaf_off", "victim_off")


def _norm(rec, pool):
    """The record without its pool offsets, plus the pool words it names (leaf triples, this pod's triples, victims)."""
    fields = tuple(rec[f].tolist() for f in trace.RESULT_DT.names if f not in _OFFSETS)
    words = (pool[rec["leaf_off"]: rec["leaf_off"] + 3 * rec["n_leaves"]].tolist(),
             pool[rec["this_off"]: rec["this_off"] + 3 * rec["this_n"]].tolist(),
             pool[rec["victim_off"]: rec["victim_off"] + 2 * rec["n_victims"]].tolist())
    return fields, words


def _cells(lib, ctx):
    n_p, n_v = lib.hived_num_physical_cells(ctx), lib.hived_num_virtual_cells(ctx)
    ps, vs = (_cabi.CellStatus * n_p)(), (_cabi.CellStatus * n_v)()
    assert lib.hived_snapshot_physical(ctx, ps, n_p) == 0 and lib.hived_snapshot_virtual(ctx, vs, n_v) == 0
    return [bytes(x) for x in ps], [bytes(x) for x in vs], [x.peer for x in ps]


def _path_counters(lib, ctx):
    out = np.zeros(64, dtype=np.int64)
    lib.hived_bench_path_counters(ctx, out.ctypes.data_as(C.POINTER(C.c_int64)))
    return out[:N_PATH]


def _vc_of_virtual(oracle_lib, ctx, n_v):
    out = []
    for i in range(n_v):
        ci = _cabi.CellInfo()
        assert oracle_lib.hived_virtual_cell_info(ctx, i, C.byref(ci)) == 0
        out.append(ci.vc)
    return out


def _compare_batch(ranks, oracle_lib, obc, plain, ev, ores, opool, fetched, owners):
    lib, world = ranks.lib, ranks.world
    n = len(ev)
    # results, event by event
    for i in range(n):
        o = owners[i]
        rec, pool = fetched[o][0][i], fetched[o][1]
        got, want = _norm(rec, pool), _norm(ores[i], opool)
        assert got == want, "event %d (type %d, VC %d, group %d): partitioned %r, oracle %r" % (
            i, ev["type"][i], ev["spec"]["vc"][i], ev["spec"]["group"][i], got, want)
        for r in range(world):
            if r != o:
                assert not fetched[r][0][i].tobytes().strip(b"\0"), "rank %d wrote event %d of rank %d" % (r, i, o)
    # the state no result shows
    books = int(oracle_lib.hived_debug_bookkeeping_hash(obc.ctx))
    assert [int(lib.hived_debug_bookkeeping_hash(bc.ctx)) for bc in ranks.ranks] == [books] * world
    ops, ovs, opeer = _cells(oracle_lib, obc.ctx)
    vc_of = _vc_of_virtual(oracle_lib, obc.ctx, len(ovs))
    n_vcs = int(oracle_lib.hived_num_vcs(obc.ctx))
    for r, bc in enumerate(ranks.ranks):
        ps, vs, peer = _cells(lib, bc.ctx)
        own = {i for i, v in enumerate(vc_of) if v % world == r}
        bad_v = [i for i in sorted(own) if vs[i] != ovs[i]]
        assert not bad_v, "rank %d: virtual cells %s differ" % (r, bad_v[:8])
        bad_p = [i for i in range(len(ps)) if (opeer[i] in own or peer[i] in own) and ps[i] != ops[i]]
        assert not bad_p, "rank %d: physical cells %s differ" % (r, bad_p[:8])
        for v in range(n_vcs):
            if v % world == r:
                assert lib.hived_debug_view_hash_vc(bc.ctx, v) == oracle_lib.hived_debug_view_hash_vc(obc.ctx, v), \
                    "rank %d: view order of VC %d" % (r, v)
    # every event counted once
    total = {}
    for bc in ranks.ranks:
        for k, x in bc.stats().items():
            total[k] = total.get(k, 0) + x
    assert total == obc.stats()
    assert sum(_path_counters(lib, bc.ctx) for bc in ranks.ranks).tolist() == _path_counters(lib, plain.ctx).tolist()


def check_partitioned(lib, oracle_lib, t, world, chunks, window, alloc=None):
    """Run `t` in `chunks` partitioned batches over `world` ranks and compare after every batch.  Returns the solo
    events [(event index in its batch, type)] of all batches."""
    _hooks(oracle_lib)
    ranks = Ranks(lib, t, world, alloc)
    obc, plain = _context(oracle_lib, t), _context(lib, t)
    ev = t["events"]
    bounds = [len(ev) * (k + 1) // chunks for k in range(chunks)]
    start, solos = 0, []
    try:
        for b in bounds:
            batch = np.ascontiguousarray(ev[start:b])
            fetched, s, owners = ranks.run(batch, window)
            ores, opool = obc.process(batch, 3 * 64 * len(batch) + 4096)
            plain.process(batch, 3 * 64 * len(batch) + 4096)
            _compare_batch(ranks, oracle_lib, obc, plain, batch, ores, opool, fetched, owners)
            solos += s
            start = b
    finally:
        ranks.close()
        obc.close()
        plain.close()
    return solos


# ---- CPU tier: the thread emulation (one host thread per CTA) and the SIMT emulation ----------------------------------

MT_SHAPES = [(1, 1, 0), (2, 1, 0), (2, 3, 7), (4, 3, 64), (4, 1, 1)]  # (world, chunks, window)


@pytest.mark.parametrize("world,chunks,window", MT_SHAPES)
@pytest.mark.parametrize("name", sorted(TRACES))
def test_partitioned_mt_matches_oracle_event_by_event(emu_mt_lib, oracle_lib, name, world, chunks, window):
    t = _reuse_trace(name, False, chunks)
    solos = check_partitioned(emu_mt_lib, oracle_lib, t, world, chunks, window)
    assert solos  # the first gang of a VC binds a preassigned cell
    if name in ("fill-and-drain", "c3-emptying-racks"):
        # deletions that give a preassigned cell back run alone
        assert any(typ == _cabi.EV_DELETE_ALLOCATED for _, typ in solos)


@pytest.mark.parametrize("world,chunks,window", [(1, 1, 0), (2, 3, 1), (3, 1, 7), (3, 3, 64)])
@pytest.mark.parametrize("name", ["heterogeneous", "fill-and-drain", "c3-emptying-racks"])
def test_partitioned_simt_matches_oracle_event_by_event(simt_lib, oracle_lib, name, world, chunks, window):
    t = _reuse_trace(name, True, chunks)
    assert check_partitioned(simt_lib, oracle_lib, t, world, chunks, window)


def test_fill_and_drain_deletes_report_their_pod(emu_mt_lib, oracle_lib):
    """The deletion that empties a VC's preassigned cell stops and runs alone; it still reports the pod it removed
    (hived_delete_allocated_pod_ex's removed pod, which a shim uses to recycle pod ids)."""
    t = fill_and_drain()
    _hooks(oracle_lib)
    ranks = Ranks(emu_mt_lib, t, 2)
    obc = _context(oracle_lib, t)
    try:
        ev = np.ascontiguousarray(t["events"])
        fetched, solos, owners = ranks.run(ev)
        ores, _ = obc.process(ev, 3 * 64 * len(ev) + 4096)
        dels = [i for i, typ in solos if typ == _cabi.EV_DELETE_ALLOCATED]
        assert dels
        for i in dels:
            assert ores["pod_index"][i] >= 0
            assert fetched[owners[i]][0]["pod_index"][i] == ores["pod_index"][i], i
    finally:
        ranks.close()
        obc.close()


# ---- refusals ------------------------------------------------------------------------------------------------------------

def _not_calm(kind, first, second):
    """`second` (the next calm batch) made not calm in one way."""
    ev = np.ascontiguousarray(second).copy()
    sched = np.flatnonzero(ev["type"] == _cabi.EV_SCHEDULE)
    k = int(sched[len(sched) // 2])
    if kind == "suggested-nodes":
        ev["suggested_off"][k] = 0
        ev["spec"]["flags"][k] = 0
    elif kind == "node-health":
        ev["type"][k] = _cabi.EV_NODE_HEALTH
        ev["arg0"][k], ev["arg1"][k] = 3, 0
    elif kind == "two-priorities":
        ev["spec"]["priority"][k] = 1
    elif kind == "recovery":
        ev["type"][k] = EV_ADD_ALLOCATED
    elif kind == "group-under-two-vcs":
        # a gang of the first batch that the second one deletes, scheduled again under the other VC, then under its own
        first_groups = {int(g): int(v) for g, v, typ in zip(first["spec"]["group"], first["spec"]["vc"], first["type"])
                        if typ == _cabi.EV_SCHEDULE}
        g = next(int(x) for x, typ in zip(ev["spec"]["group"], ev["type"])
                 if typ == _cabi.EV_DELETE_ALLOCATED and int(x) in first_groups)
        v = first_groups[g]
        row = first[np.flatnonzero((first["type"] == _cabi.EV_SCHEDULE) & (first["spec"]["group"] == g))[0]].copy()
        a, b = row.copy(), row.copy()
        a["spec"]["vc"] = 1 - v
        ev = np.concatenate([np.array([a, b], dtype=trace.EVENT_DT), ev])
    return np.ascontiguousarray(ev)


@pytest.mark.parametrize("kind", ["suggested-nodes", "node-health", "two-priorities", "recovery", "group-under-two-vcs"])
def test_partition_refuses_a_batch_that_is_not_calm(emu_mt_lib, oracle_lib, kind):
    lib = _hooks(emu_mt_lib)
    dist.bind_multigpu(lib)
    _hooks(oracle_lib)
    t = trace.trace_heterogeneous(n_gangs=400)
    ev = t["events"]
    half = len(ev) // 2
    first, second = np.ascontiguousarray(ev[:half]), np.ascontiguousarray(ev[half:])
    ranks = Ranks(lib, t, 2)
    obc, plain = _context(oracle_lib, t), _context(lib, t)
    try:
        for batch, run_it in ((first, True), (_not_calm(kind, first, second), False), (second, True)):
            if not run_it:
                before = [(int(lib.hived_debug_bookkeeping_hash(bc.ctx)), _cells(lib, bc.ctx)[:2]) for bc in ranks.ranks]
                rcs, _ = ranks.stage(batch)
                assert rcs == [ERR_BAD_SPEC] * 2, [lib.hived_last_error(bc.ctx) for bc in ranks.ranks]
                assert all(b"multi-GPU partition" in lib.hived_last_error(bc.ctx) for bc in ranks.ranks)
                assert before == [(int(lib.hived_debug_bookkeeping_hash(bc.ctx)), _cells(lib, bc.ctx)[:2]) for bc in ranks.ranks]
                continue
            fetched, _, owners = ranks.run(batch)
            ores, opool = obc.process(batch, 3 * 64 * len(batch) + 4096)
            plain.process(batch, 3 * 64 * len(batch) + 4096)
            _compare_batch(ranks, oracle_lib, obc, plain, batch, ores, opool, fetched, owners)
    finally:
        ranks.close()
        obc.close()
        plain.close()


# ---- GPU tier: `world` contexts on one device, the exchange buffer in device memory -------------------------------------

def _device_alloc(nbytes):
    import torch
    b = torch.empty(max(nbytes, 16), dtype=torch.uint8, device="cuda")
    return b, b.data_ptr()


@pytest.mark.gpu
@pytest.mark.parametrize("world,chunks,window", [(2, 1, 0), (4, 3, 64)])
@pytest.mark.parametrize("name", sorted(TRACES))
def test_partitioned_cuda_matches_oracle_event_by_event(cuda_lib, oracle_lib, name, world, chunks, window):
    t = _reuse_trace(name, False, chunks)
    solos = check_partitioned(cuda_lib, oracle_lib, t, world, chunks, window, alloc=_device_alloc)
    assert solos
    if name in ("fill-and-drain", "c3-emptying-racks"):
        assert any(typ == _cabi.EV_DELETE_ALLOCATED for _, typ in solos)
