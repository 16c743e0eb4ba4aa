"""hived_clone (include/hived_clone.h): a new context that answers every later call exactly as its source would have.

Every case runs a prefix on a source context, clones it, runs the same suffix on both, and compares each with the
oracle run from scratch over prefix + suffix: rc, results and pool bytes, the running result hash, the work counters,
the cell snapshots, the view-order and bookkeeping hashes; source and clone (the same library) also by their path
counters.  The suffixes are chosen to meet what a rebuild by recovery would lose: the order of the cluster views and of
the free, bad-free and doomed-bad lists, erased groups that cells still name, lazy-preempted and preempting groups,
and the host state that decides how a batch runs (node health, recovery, priorities in use).  The CPU tier runs the
thread emulation and the SIMT emulation; the GPU tier the CUDA library with ordinary and concurrent contexts."""
import copy
import ctypes as C
import json
import os
import threading

import numpy as np
import pytest

import fuzz_api
from conftest import snapshot_bytes
from hivedscheduler_b200 import _cabi, dist, trace
from hivedscheduler_b200 import algorithm as alg
from hivedscheduler_b200.config import new_config
from test_calm_loop import PC_CALM, PC_CALM_FALLBACK, c3_slice
from test_many_contexts import _ctx, _hooks, _single, _words, workloads

HERE = os.path.dirname(os.path.abspath(__file__))
FLAG = _cabi.OPT_CONCURRENT
ERR_BAD_SPEC, ERR_CAPACITY = 7, 102  # HIVED_ERR_BAD_SPEC, HIVED_ERR_CAPACITY
N_PATH = 14                          # PC_COUNT (hived_dev.h)
# (source flags, clone flags): the pairings of ordinary and concurrent contexts
PAIRS = {"ordinary": (0, 0), "to-concurrent": (0, FLAG), "from-concurrent": (FLAG, 0), "concurrent": (FLAG, FLAG)}


def _paths(bc):
    out = (C.c_int64 * 16)()
    bc.lib.hived_bench_path_counters(bc.ctx, out)
    return list(out)[:N_PATH]


def _state(bc):
    """What a later call can show of a context: hash, counters, cells, view order, bookkeeping."""
    lib, ctx = bc.lib, bc.ctx
    return (bc.result_hash(), bc.stats(), snapshot_bytes(lib, ctx), int(lib.hived_debug_view_hash(ctx)),
            int(lib.hived_debug_bookkeeping_hash(ctx)))


def _lib_state(bc):
    """... and what only the same library shows: the path counters."""
    return _state(bc) + (_paths(bc),)


def _chunks(ev):
    """A suffix in several batches: small ones (the per-call path on the GPU), then the rest."""
    out, at = [], 0
    for size in (1, 3, 8, len(ev)):
        if at < len(ev):
            out.append(ev[at:at + size])
            at += size
    return out


def _run(bc, chunks, sugg):
    return [_single(bc, ev, _words(ev), sugg) for ev in chunks]


def _same(a, b):
    assert len(a) == len(b)
    for (rca, resa, poola), (rcb, resb, poolb) in zip(a, b):
        assert rca == rcb
        assert resa.tobytes() == resb.tobytes()
        assert poola.tobytes() == poolb.tobytes()


def _clone_traces(lib, oracle_lib, pair=(0, 0), of_clone=False, short=True):
    """Case 1 and 2 on every trace of the mixed workload: each equals the oracle, neither changes the other."""
    oracle = _hooks(oracle_lib)
    for t in workloads(short)[:5]:
        ev, sugg = t["events"], t.get("sugg_pool")
        cut = len(ev) // 2
        src = trace.BatchContext(lib, t["config"], t["n_groups"] + 8, t["n_pods"] + 512, t["max_group_leaves"],
                                 t["max_group_pods"], flags=pair[0])
        src.set_all_nodes_healthy()
        ref = _ctx(oracle, t)
        head = [ev[:cut // 2], ev[cut // 2:cut]]
        _same(_run(src, head, sugg), _run(ref, head, sugg))
        first = src.clone(flags=pair[1]) if of_clone else None
        clone = (first or src).clone(flags=pair[1])
        if first is not None:
            first.close()
        assert lib.hived_last_error(clone.ctx) == b""
        assert _lib_state(clone) == _lib_state(src), t["name"]
        tail = _chunks(ev[cut:])
        want = _run(ref, tail, sugg)
        before = _lib_state(src)
        _same(_run(clone, tail, sugg), want)
        assert _lib_state(src) == before, "%s: the clone's suffix changed the source" % t["name"]
        mid = _lib_state(clone)
        _same(_run(src, tail, sugg), want)
        assert _lib_state(clone) == mid, "%s: the source's suffix changed the clone" % t["name"]
        assert _state(src) == _state(ref) == _state(clone), t["name"]
        assert _paths(src) == _paths(clone), t["name"]
        for bc in (src, clone, ref):
            bc.close()


# ---- name-level runs: the API fuzz with clones taken along the way ---------------------------------------------------

class Sides:
    """HivedAlgorithm shims driven call by call in lock step: sides[0] the source, sides[1] the oracle, then clones.
    pods[k]: uid -> pod object of side k (a clone starts with its source's)."""

    def __init__(self, lib, oracle_lib, cfg, flags=0):
        self.hs = [alg.HivedAlgorithm(new_config(copy.deepcopy(cfg)), lib=x, max_groups=1024, max_pods=4096,
                                      max_group_leaves=128, max_group_pods=16, flags=flags)
                   for x in (lib, oracle_lib)]
        for x in (lib, oracle_lib):
            _hooks(x)
        self.pods = [{}, {}]
        self.clones = 0

    def clone(self, k, concurrent=False):
        self.hs.append(self.hs[k].clone(concurrent=concurrent))
        self.pods.append(dict(self.pods[k]))
        self.clones += 1

    def call(self, fn):
        """fn(h, pods) on every side; the answers must agree.  Returns side 0's."""
        out = [fuzz_api._call(lambda: fn(h, p)) for h, p in zip(self.hs, self.pods)]
        assert all(o == out[0] for o in out[1:]), out
        return out[0]

    def check(self):
        snaps = [snapshot_bytes(h._lib, h._ctx) for h in self.hs]
        assert all(s == snaps[0] for s in snaps[1:]), "cell states differ"
        for hook in ("hived_debug_view_hash", "hived_debug_bookkeeping_hash"):
            v = [int(getattr(h._lib, hook)(h._ctx)) for h in self.hs]
            assert all(x == v[0] for x in v[1:]), hook
        # the source and its clones (the same library): every group's record, `referenced` included, the shims' id
        # tables with their recycled ids and the kept pod objects, and the name-level inspect answer
        same = [self.hs[0]] + self.hs[2:]

        def groups(h):
            out = []
            for gid in range(len(h._groups.names)):
                gi = _cabi.GroupInfo()
                h._lib.hived_get_group(h._ctx, gid, C.byref(gi))
                out.append(bytes(gi))
            return out

        def shim(h):
            return (h._groups.ids, h._groups.names, h._groups.free, h._pods.ids, h._pods.names, h._pods.free,
                    sorted(h._pod_objs), h._rand.getstate(), h.GetAllAffinityGroups())

        g0, s0 = groups(same[0]), shim(same[0])
        for h in same[1:]:
            assert groups(h) == g0
            assert shim(h) == s0
        # against the oracle: the records' scheduling fields (`referenced` is the device's conservative answer, and the
        # preempting-pod count of a group that is not preempting is not part of the contract)
        o = self.hs[1]
        for gid in range(len(o._groups.names)):
            a, b = _cabi.GroupInfo(), _cabi.GroupInfo()
            self.hs[0]._lib.hived_get_group(self.hs[0]._ctx, gid, C.byref(a))
            o._lib.hived_get_group(o._ctx, gid, C.byref(b))
            assert (a.state, a.vc, a.priority, a.has_virtual) == (b.state, b.vc, b.priority, b.has_virtual)

    def close(self):
        for h in self.hs:
            h.close()


def _schedule(uid, spec_yaml, sugg, phase):
    def op(h, pods):
        pod = alg.Pod(name=uid, namespace="fz", uid=uid, annotations={alg.ANNOTATION_POD_SCHEDULING_SPEC: spec_yaml})
        r = fuzz_api._norm(h.Schedule(pod, sugg, phase))
        if r[0] == "bind":
            bound = alg.new_binding_pod(pod, r[1])
            h.AddAllocatedPod(bound)
            pods[uid] = ("allocated", bound)
        elif r[0] == "preempt" and phase == alg.PREEMPTING_PHASE:
            pods[uid] = ("preempting", pod)
        return r
    return op


def _delete(kind, uid):
    def op(h, pods):
        want = "allocated" if kind == "DeleteAllocatedPod" else "preempting"
        if pods.get(uid, ("",))[0] != want:
            return "skipped"
        return getattr(h, kind)(pods.pop(uid)[1])
    return op


def fuzz_with_clones(lib, oracle_lib, seed, n_ops, clone_at, concurrent=(False, False), flags=0):
    """tests/fuzz_api.py's operation stream for `seed` (the same random choices), on a source and the oracle; after
    operation clone_at[0] the source is cloned, after clone_at[1] that clone is cloned, and every side takes every later
    call.  Stops where the reference would panic (a platform error on every side)."""
    fx = fuzz_api.env_fixture()
    rng = random_for(seed)
    s = Sides(lib, oracle_lib, fx["design_config"], flags)
    try:
        nodes = list(s.hs[0].node_names)
        healthy = {n: True for n in nodes}
        for n in nodes:
            s.call(lambda h, p: h.setHealthyNode(n))
        spec_names = sorted(fx["pss"])
        allocated, preempting, serial = [], [], 0
        for step in range(n_ops):
            r = rng.random()
            if r < 0.55 or not allocated:
                name = rng.choice(spec_names)
                spec = copy.deepcopy(fx["pss"][name])
                if rng.random() < 0.5:
                    spec["affinityGroup"]["name"] = "%s-%d" % (spec["affinityGroup"]["name"], rng.randrange(6))
                serial += 1
                uid = "u%d" % serial
                sugg = nodes if rng.random() < 0.8 else [n for n in nodes if rng.random() < 0.7]
                res = s.call(_schedule(uid, alg.to_yaml(spec), sugg, alg.PREEMPTING_PHASE))
                if res[0] == "ok" and res[1][0] == "bind":
                    allocated.append(uid)
                elif res[0] == "ok" and res[1][0] == "preempt":
                    preempting.append(uid)
            elif r < 0.78:
                res = s.call(_delete("DeleteAllocatedPod", allocated.pop(rng.randrange(len(allocated)))))
            elif r < 0.85 and preempting:
                res = s.call(_delete("DeleteUnallocatedPod", preempting.pop(rng.randrange(len(preempting)))))
            else:
                n = rng.choice(nodes)
                healthy[n] = not healthy[n]
                res = s.call(lambda h, p: (h.setHealthyNode if healthy[n] else h.setBadNode)(n))
            if res[0] == "platform":
                break
            s.check()
            for i, at in enumerate(clone_at):
                if step == at:
                    s.clone(0 if i == 0 else len(s.hs) - 1, concurrent[i])
                    s.check()
        return s.clones
    finally:
        s.close()


def random_for(seed):
    import random
    return random.Random(seed)


def replay_stale_doomed(lib, oracle_lib, clone_at, concurrent=False):
    """The 43 calls of tests/golden/doomed_bad_stale_ops.json (a stale doomed-bad entry, then an append behind it) on
    the synthetic cluster, cloned after call clone_at."""
    ops = json.load(open(os.path.join(HERE, "golden", "doomed_bad_stale_ops.json")))
    s = Sides(lib, oracle_lib, fuzz_api.synthetic_fixture()["design_config"])
    try:
        for n in s.hs[0].node_names:
            s.call(lambda h, p: h.setHealthyNode(n))
        for i, op in enumerate(ops):
            kind = op[0]
            if kind == "Schedule":
                s.call(_schedule(op[2], op[1], op[3], op[4]))
            elif kind in ("DeleteAllocatedPod", "DeleteUnallocatedPod"):
                s.call(_delete(kind, op[1]))
            else:
                s.call(lambda h, p: getattr(h, kind)(op[1]))
            s.check()
            if i == clone_at:
                s.clone(0, concurrent)
                s.check()
        return s.clones
    finally:
        s.close()


# ---- the host state that decides how a batch runs ---------------------------------------------------------------------

def _recover_one(bc, group, pod, vc):
    """hived_schedule of a one-leaf gang, then hived_add_allocated_pod of its placement: a recovered pod."""
    spec = _cabi.PodSpec(pod=pod, group=group, vc=vc, priority=0, pinned=-1, leaf_type=0, leaf_num=1,
                         flags=_cabi.SPEC_IGNORE_SUGGESTED, n_members=1)
    spec.member_leaf_num[0], spec.member_pod_num[0] = 1, 1
    res, pool = _cabi.Result(), (C.c_int32 * 64)()
    assert bc.lib.hived_schedule(bc.ctx, C.byref(spec), None, _cabi.PHASE_PREEMPTING, C.byref(res), pool, 64) == 0
    assert res.kind == _cabi.KIND_BIND
    info = _cabi.BindInfo(node=pool[res.leaf_off], first_leaf=pool[res.leaf_off + 1], chain=res.chain, has_preassigned=1,
                          n_members=1, n_leaves=1)
    info.member_leaf_num[0], info.member_pod_num[0] = 1, 1
    leaves = (C.c_int32 * 3)(*pool[res.leaf_off:res.leaf_off + 3])
    assert bc.lib.hived_add_allocated_pod(bc.ctx, C.byref(spec), C.byref(info), leaves, 0) == 0


def _priority_one(bc, group, pod, vc):
    tb = trace.TraceBuilder(4)
    tb.next_pod = pod
    tb.schedule(group=group, vc=vc, priority=1, leaf_type=0, leaf_num=1, pod_num=1)
    assert _single(bc, tb.finish()[0], 4096)[0] == 0


# case -> (what happens before the clone, what happens after it on every context, (CTAs, calm) of the batch after that)
ROUTING = {
    "bad-node": (lambda bc, t: bc.lib.hived_set_node_health(bc.ctx, 5, 0), None, (1, False)),
    "bad-node-healed": (lambda bc, t: bc.lib.hived_set_node_health(bc.ctx, 5, 0),
                        lambda bc, t: bc.lib.hived_set_node_health(bc.ctx, 5, 1), (8, True)),
    "recovered-pod": (lambda bc, t: _recover_one(bc, t["n_groups"], t["n_pods"], 3), None, (1, False)),
    "second-priority": (lambda bc, t: _priority_one(bc, t["n_groups"], t["n_pods"], 2), None, (1, False)),
}


def _routing(lib, oracle_lib, monkeypatch, name, pair=(0, 0)):
    """Case 4: a clone runs its next batch in the source's regime: CTA count, calm loop, path counters."""
    monkeypatch.delenv("HIVED_NCTA", raising=False)
    monkeypatch.delenv("HIVED_NO_CALM", raising=False)
    before, after, (ctas, calm) = ROUTING[name]
    t = c3_slice()
    ev = t["events"]

    def make(x, flags):
        bc = trace.BatchContext(x, t["config"], t["n_groups"] + 8, t["n_pods"] + 8, t["max_group_leaves"],
                                t["max_group_pods"], flags=flags)
        bc.set_all_nodes_healthy()
        assert _single(bc, ev[:300], _words(ev[:300]))[0] == 0
        before(bc, t)
        return bc

    src, ref = make(lib, pair[0]), make(_hooks(oracle_lib), 0)
    clone = src.clone(flags=pair[1])
    for bc in (src, clone, ref):
        if after:
            after(bc, t)
    want = _single(ref, ev[300:900], _words(ev[300:900]))
    seen = []
    for bc in (src, clone):
        p0 = _paths(bc)
        _same([_single(bc, ev[300:900], _words(ev[300:900]))], [want])
        p1 = _paths(bc)
        seen.append((lib.hived_bench_num_ctas(bc.ctx), p1[PC_CALM] + p1[PC_CALM_FALLBACK] - p0[PC_CALM] - p0[PC_CALM_FALLBACK],
                     p1))
    assert seen[0] == seen[1]
    n_ctas, n_calm, _ = seen[0]
    if not lib._name.endswith("libhived_emu.so"):  # (the 1-lane emulation runs every batch on one CTA)
        assert n_ctas == ctas
    assert n_calm == (600 if calm else 0)
    assert _state(src) == _state(clone) == _state(ref)
    for bc in (src, clone, ref):
        bc.close()


# ---- CPU tier ---------------------------------------------------------------------------------------------------------

@pytest.fixture(params=["emu_mt", "simt"])
def lib(request):
    return _hooks(request.getfixturevalue(request.param + "_lib"))


def _short(lib):
    return "simt" in lib._name


def test_clone_continues_every_trace_like_its_source(lib, oracle_lib):
    _clone_traces(lib, oracle_lib, short=_short(lib))


def test_clone_of_a_clone(emu_mt_lib, oracle_lib):
    _clone_traces(_hooks(emu_mt_lib), oracle_lib, of_clone=True)


@pytest.mark.parametrize("seed", [16, 31, 775, 2385])
def test_clone_mid_api_fuzz(emu_lib, oracle_lib, seed):
    """API-fuzz seeds whose histories hold erased groups that cells still name (16, 31, 2385: ghost records), lazy
    preemption and preempting groups, recovered pods (every bind is followed by AddAllocatedPod) and a pod deleted
    through another pod's slot that the shim keeps (775).  A clone after call 100 and a clone of that clone after call
    200 take every later call with the source and the oracle, all compared after every call."""
    assert fuzz_with_clones(_hooks(emu_lib), oracle_lib, seed, 300, (100, 200)) == 2


def test_clone_mid_api_fuzz_simt(simt_lib, oracle_lib):
    assert fuzz_with_clones(_hooks(simt_lib), oracle_lib, 16, 200, (60, 120)) == 2


@pytest.mark.parametrize("at", [20, 34])
def test_clone_with_a_stale_doomed_bad_entry(lib, oracle_lib, at):
    assert replay_stale_doomed(lib, oracle_lib, at) == 1


@pytest.mark.parametrize("name", list(ROUTING))
def test_clone_runs_its_next_batch_in_the_sources_regime(emu_mt_lib, oracle_lib, monkeypatch, name):
    _routing(_hooks(emu_mt_lib), oracle_lib, monkeypatch, name)


def test_shim_clone_answers_by_name(emu_lib, oracle_lib):
    """HivedAlgorithm.clone: a gang scheduled on both shims gets the same placement, a group deleted on both frees the
    same id, and the shims' own tables are copies, not shared."""
    fx = fuzz_api.env_fixture()
    h = alg.HivedAlgorithm(new_config(copy.deepcopy(fx["design_config"])), lib=emu_lib, max_groups=64, max_pods=256,
                           max_group_leaves=128, max_group_pods=16)
    try:
        for n in h.node_names:
            h.setHealthyNode(n)
        spec = copy.deepcopy(fx["pss"][sorted(fx["pss"])[0]])
        pods = []
        for i in range(3):
            spec["affinityGroup"]["name"] = "g%d" % i
            pod = alg.Pod(name="p%d" % i, namespace="ns", uid="u%d" % i,
                          annotations={alg.ANNOTATION_POD_SCHEDULING_SPEC: alg.to_yaml(spec)})
            r = h.Schedule(pod, h.node_names, alg.PREEMPTING_PHASE)
            if r.pod_bind_info is not None:
                pods.append(alg.new_binding_pod(pod, r.pod_bind_info))
                h.AddAllocatedPod(pods[-1])
        assert pods
        c = h.clone()
        try:
            assert c._groups is not h._groups and c._pod_objs is not h._pod_objs
            for x in (h, c):
                x.DeleteAllocatedPod(pods[0])
            assert c._groups.free == h._groups.free and c._pods.free == h._pods.free and h._groups.free
            spec["affinityGroup"]["name"] = "g-new"
            pod = alg.Pod(name="q", namespace="ns", uid="q", annotations={alg.ANNOTATION_POD_SCHEDULING_SPEC: alg.to_yaml(spec)})
            a, b = (x.Schedule(pod, x.node_names, alg.PREEMPTING_PHASE) for x in (h, c))
            assert fuzz_api._norm(a) == fuzz_api._norm(b)
            assert h._groups.ids["g-new"] == c._groups.ids["g-new"]  # the recycled id, on both
            gname = alg.extract_pod_scheduling_spec(pods[1])["affinityGroup"]["name"]
            assert h.GetAffinityGroup(gname) == c.GetAffinityGroup(gname)
            # only the clone deletes: the source still has the group
            c.DeleteAllocatedPod(pods[1])
            assert h.GetAffinityGroup(gname)
            with pytest.raises(alg.WebServerError):
                c.GetAffinityGroup(gname)
        finally:
            c.close()
    finally:
        h.close()


def test_clone_refused_for_a_partition_staged_source(lib):
    t = trace.trace_bad_requests()
    bc = _ctx(lib, t)
    dist.bind_multigpu(lib)
    tb = trace.TraceBuilder(4)
    tb.schedule(group=1, vc=0, priority=0, leaf_type=0, leaf_num=1, pod_num=1)
    ev, _ = tb.finish()
    assert lib.hived_mg_stage(bc.ctx, ev.ctypes.data_as(C.POINTER(_cabi.Event)), len(ev), 4096, 0, 1) == 0
    before = _state(bc)
    out = C.c_void_p(1)
    assert _cabi.bind_clone(lib).hived_clone(bc.ctx, -1, 0, C.byref(out)) == ERR_BAD_SPEC
    assert not out.value
    assert b"multi-GPU partition" in lib.hived_create_error()
    assert _state(bc) == before
    bc.close()


# ---- GPU tier ---------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("pair", list(PAIRS))
def test_gpu_clone_continues_every_trace(cuda_lib, oracle_lib, pair):
    _clone_traces(_hooks(cuda_lib), oracle_lib, PAIRS[pair], short=False)


@pytest.mark.gpu
def test_gpu_clone_of_a_clone(cuda_lib, oracle_lib):
    _clone_traces(_hooks(cuda_lib), oracle_lib, (FLAG, 0), of_clone=True, short=False)


@pytest.mark.gpu
@pytest.mark.parametrize("pair", list(PAIRS))
@pytest.mark.parametrize("seed", [16, 2385])
def test_gpu_clone_mid_api_fuzz(cuda_lib, oracle_lib, seed, pair):
    src, dst = PAIRS[pair]
    assert fuzz_with_clones(_hooks(cuda_lib), oracle_lib, seed, 300, (100, 200), (bool(dst), not dst), flags=src) == 2


@pytest.mark.gpu
@pytest.mark.parametrize("pair", ["ordinary", "concurrent"])
def test_gpu_clone_with_a_stale_doomed_bad_entry(cuda_lib, oracle_lib, pair):
    assert replay_stale_doomed(_hooks(cuda_lib), oracle_lib, 34, concurrent=bool(PAIRS[pair][1])) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("pair", list(PAIRS))
@pytest.mark.parametrize("name", list(ROUTING))
def test_gpu_clone_runs_its_next_batch_in_the_sources_regime(cuda_lib, oracle_lib, monkeypatch, name, pair):
    _routing(_hooks(cuda_lib), oracle_lib, monkeypatch, name, PAIRS[pair])


@pytest.mark.gpu
def test_gpu_full_size_c3_clone_at_half(cuda_lib):
    """The BASELINE C3 trace (64k GPUs, 100k gangs): cloned at the checkpoint halfway through (about gang 50 000), the
    clone's later checkpoint hashes and final counters are the oracle's committed ones."""
    t = trace.trace_c3()
    golden = json.load(open(os.path.join(HERE, "golden", "trace_hashes.json")))["C3"]
    cps = golden["checkpoints"]
    half = len(cps) // 2
    gangs = np.cumsum(t["decision"])  # gangs decided up to and including each event
    assert 45000 <= gangs[cps[half - 1]["events"] - 1] <= 55000
    src = trace.BatchContext(cuda_lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
    src.set_all_nodes_healthy()
    start = 0
    for cp in cps[:half]:
        src.process(t["events"][start:cp["events"]], 3 * 64 * (cp["events"] - start) + 4096)
        start = cp["events"]
    assert "%016x" % src.result_hash() == cps[half - 1]["hash"]
    clone = src.clone()
    src.close()
    for cp in cps[half:]:
        chunk = t["events"][start:cp["events"]]
        res, _ = clone.process(chunk, 3 * 64 * len(chunk) + 4096)
        assert "%016x" % clone.result_hash() == cp["hash"], "diverged from the oracle before event %d" % cp["events"]
        assert int((res["kind"][chunk["type"] == _cabi.EV_SCHEDULE] == 1).sum()) == cp["binds"]
        start = cp["events"]
    assert cps[-1]["hash"] == "e3becf53c2d32f79"
    stats = clone.stats()
    for key in ("view_nodes_scanned", "leaves_committed", "free_cells_scanned", "pods_placed", "algorithmic_bytes"):
        assert stats[key] == golden["stats"][key]
    clone.close()


def _prefix_and_suffixes(k):
    """One C3-shaped cluster, a prefix, and k different suffixes (every one its own slice of a longer trace)."""
    from test_device_program_emu import small_c3
    t = small_c3(1500)
    ev = t["events"]
    cut = len(ev) // 4
    n = (len(ev) - cut) // k
    return t, ev[:cut], [ev[cut + i * n:cut + (i + 1) * n] for i in range(k)]


@pytest.mark.gpu
def test_gpu_joint_what_if(cuda_lib, oracle_lib):
    """Four clones of one source, each with its own suffix, in one hived_process_events_many call: each equals the
    oracle's run of prefix + its suffix, and the source is unchanged."""
    lib, oracle = _hooks(cuda_lib), _hooks(oracle_lib)
    t, head, tails = _prefix_and_suffixes(4)
    src = _ctx(lib, t)
    assert _single(src, head, _words(head))[0] == 0
    before = _lib_state(src)
    clones = [src.clone() for _ in tails]
    got = trace.process_many(clones, tails, [_words(x) for x in tails])
    for bc, tail, g in zip(clones, tails, got):
        ref = _ctx(oracle, t)
        assert _single(ref, head, _words(head))[0] == 0
        _same([g], [_single(ref, tail, _words(tail))])
        assert _state(bc) == _state(ref)
        ref.close()
        bc.close()
    assert _lib_state(src) == before
    src.close()


@pytest.mark.gpu
def test_gpu_concurrent_clones_on_their_own_threads(cuda_lib, oracle_lib):
    """Concurrent clones, each driven from a thread of its own through per-call batches and one large batch, while the
    concurrent source keeps serving per-call operations on the main thread.  Every context's answers equal its oracle
    run."""
    lib, oracle = _hooks(cuda_lib), _hooks(oracle_lib)
    t, head, tails = _prefix_and_suffixes(3)
    src = trace.BatchContext(lib, t["config"], t["n_groups"] + 8, t["n_pods"] + 512, t["max_group_leaves"],
                             t["max_group_pods"], flags=FLAG)
    src.set_all_nodes_healthy()
    assert _single(src, head, _words(head))[0] == 0
    clones = [src.clone(flags=FLAG) for _ in tails]
    got = [None] * len(tails)

    def drive(i):
        got[i] = _run(clones[i], _chunks(tails[i]), None)

    threads = [threading.Thread(target=drive, args=(i,)) for i in range(len(tails))]
    for th in threads:
        th.start()
    # the source, meanwhile: the first suffix one event per call
    mine = [_single(src, tails[0][i:i + 1], _words(tails[0][i:i + 1])) for i in range(64)]
    for th in threads:
        th.join()
    for i, tail in enumerate(tails):
        ref = _ctx(oracle, t)
        assert _single(ref, head, _words(head))[0] == 0
        _same(got[i], _run(ref, _chunks(tail), None))
        assert _state(clones[i]) == _state(ref)
        ref.close()
    ref = _ctx(oracle, t)
    assert _single(ref, head, _words(head))[0] == 0
    _same(mine, [_single(ref, tails[0][i:i + 1], _words(tails[0][i:i + 1])) for i in range(64)])
    assert _state(src) == _state(ref)
    for bc in clones + [src, ref]:
        bc.close()


@pytest.mark.gpu
def test_gpu_clone_on_a_second_device(cuda_lib, oracle_lib):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    lib, oracle = _hooks(cuda_lib), _hooks(oracle_lib)
    t, head, tails = _prefix_and_suffixes(1)
    src = _ctx(lib, t)
    assert _single(src, head, _words(head))[0] == 0
    for flags in (0, FLAG):
        clone = src.clone(device=1, flags=flags)
        ref = _ctx(oracle, t)
        assert _single(ref, head, _words(head))[0] == 0
        _same(_run(clone, _chunks(tails[0]), None), _run(ref, _chunks(tails[0]), None))
        assert _state(clone) == _state(ref)
        clone.close()
        ref.close()
    src.close()


@pytest.mark.gpu
def test_gpu_concurrent_clone_past_the_limit(cuda_lib, oracle_lib):
    """With every concurrent slot of the device taken, a concurrent clone gives HIVED_ERR_CAPACITY and creates nothing;
    an ordinary clone still works, and so do the existing contexts."""
    lib, oracle = _hooks(cuda_lib), _hooks(oracle_lib)
    t, head, tails = _prefix_and_suffixes(1)
    src = _ctx(lib, t)
    assert _single(src, head, _words(head))[0] == 0
    held = [trace.BatchContext(lib, t["config"], 16, 64, t["max_group_leaves"], t["max_group_pods"], flags=FLAG)
            for _ in range(_cabi.HIVED_CONCURRENT_MAX)]
    out = C.c_void_p(1)
    assert _cabi.bind_clone(lib).hived_clone(src.ctx, -1, FLAG, C.byref(out)) == ERR_CAPACITY
    assert not out.value
    assert b"HIVED_CONCURRENT_MAX" in lib.hived_create_error()
    clone = src.clone()
    ref = _ctx(oracle, t)
    assert _single(ref, head, _words(head))[0] == 0
    want = _run(ref, _chunks(tails[0]), None)
    for bc in (src, clone):
        _same(_run(bc, _chunks(tails[0]), None), want)
        assert _state(bc) == _state(ref)
    for bc in held:
        bc.set_all_nodes_healthy()
    for bc in held + [src, clone, ref]:
        bc.close()
