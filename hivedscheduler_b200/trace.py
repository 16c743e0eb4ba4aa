"""Seeded synthetic event traces of the benchmark configs (SURVEY.md section 8d) and the batch driver.

A trace is a numpy structured array with the exact memory layout of ``hived_event_t``
(include/hived.h); it is generated up-front on the host and replayed identically by every
implementation of the ABI (``hived_process_events``).  The generators are results-independent:
the admission window only uses gang sizes, so the same trace is valid for oracle and product.
"""
from __future__ import annotations

import ctypes as C
from collections import deque
from typing import Any, Dict, List, Tuple

import numpy as np

from . import _cabi
from .config import config_c1, config_c2, config_c3

_SPEC_DT = np.dtype([
    ("pod", "<i4"), ("group", "<i4"), ("vc", "<i4"), ("priority", "<i4"), ("pinned", "<i4"),
    ("leaf_type", "<i4"), ("leaf_num", "<i4"), ("flags", "<i4"), ("n_members", "<i4"),
    ("member_leaf_num", "<i4", (8,)), ("member_pod_num", "<i4", (8,))], align=True)
EVENT_DT = np.dtype([("type", "<i4"), ("phase", "<i4"), ("arg0", "<i4"), ("arg1", "<i4"),
                     ("suggested_off", "<i8"), ("spec", _SPEC_DT)], align=True)
assert EVENT_DT.itemsize == C.sizeof(_cabi.Event), (EVENT_DT.itemsize, C.sizeof(_cabi.Event))

RESULT_DT = np.dtype([
    ("kind", "<i4"), ("error", "<i4"), ("wait_code", "<i4"), ("wait_cell", "<i4"), ("chain", "<i4"),
    ("pod_index", "<i4"), ("node", "<i4"), ("this_off", "<i4"), ("this_n", "<i4"), ("n_members", "<i4"),
    ("member_leaf_num", "<i4", (8,)), ("member_pod_num", "<i4", (8,)), ("leaf_off", "<i4"),
    ("n_leaves", "<i4"), ("victim_off", "<i4"), ("n_victims", "<i4"), ("has_virtual", "<i4"),
    ("incomplete", "<i4")], align=True)
assert RESULT_DT.itemsize == C.sizeof(_cabi.Result)

MASK64 = (1 << 64) - 1


class XorShift64Star:
    """xorshift64* of SURVEY.md section 8d."""

    def __init__(self, seed: int):
        self.x = seed & MASK64
        if self.x == 0:
            self.x = 0x9E3779B97F4A7C15

    def next(self) -> int:
        x = self.x
        x ^= x >> 12
        x ^= (x << 25) & MASK64
        x ^= x >> 27
        self.x = x
        return (x * 0x2545F4914F6CDD1D) & MASK64

    def below(self, n: int) -> int:
        return self.next() % n


def seed_for(config_number: int) -> int:
    return 0x9E3779B97F4A7C15 ^ config_number


class TraceBuilder:
    def __init__(self, capacity: int):
        self.ev = np.zeros(capacity, dtype=EVENT_DT)
        self.n = 0
        self.decision = np.zeros(capacity, dtype=bool)  # True on the first pod of each gang
        self.next_pod = 0

    def _grow(self):
        if self.n == len(self.ev):
            grown = np.zeros(2 * len(self.ev), dtype=EVENT_DT)
            grown.view(np.uint8)[:self.ev.nbytes] = self.ev.view(np.uint8)
            self.ev = grown
            self.decision = np.concatenate([self.decision, np.zeros(len(self.decision), dtype=bool)])

    def schedule(self, group: int, vc: int, priority: int, leaf_type: int, leaf_num: int, pod_num: int,
                 phase: int = _cabi.PHASE_PREEMPTING, flags: int = _cabi.SPEC_IGNORE_SUGGESTED,
                 first: bool = True, members=None) -> int:
        """members: [(leaf_num, pod_num), ...] of the whole gang when it has several (the pod itself asks for
        ``leaf_num``); default: one member (leaf_num x pod_num)."""
        self._grow()
        e = self.ev[self.n]
        e["type"] = _cabi.EV_SCHEDULE
        e["phase"] = phase
        e["suggested_off"] = -1
        s = e["spec"]
        s["pod"] = self.next_pod
        s["group"] = group
        s["vc"] = vc
        s["priority"] = priority
        s["pinned"] = -1
        s["leaf_type"] = leaf_type
        s["leaf_num"] = leaf_num
        s["flags"] = flags
        if members is None:
            members = [(leaf_num, pod_num)]
        s["n_members"] = len(members)
        for i, (ln, pn) in enumerate(members):
            s["member_leaf_num"][i] = ln
            s["member_pod_num"][i] = pn
        self.decision[self.n] = first
        self.n += 1
        self.next_pod += 1
        return self.next_pod - 1

    def delete_allocated(self, group: int, leaf_num: int, pod_index: int, vc: int = -1):
        self._grow()
        e = self.ev[self.n]
        e["type"] = _cabi.EV_DELETE_ALLOCATED
        e["arg0"] = pod_index
        e["suggested_off"] = -1
        e["spec"]["group"] = group
        e["spec"]["leaf_num"] = leaf_num
        e["spec"]["vc"] = vc  # the pod's VC (from its annotation): routes the event to the CTA owning the VC
        self.n += 1

    def node_health(self, node: int, healthy: bool):
        self._grow()
        e = self.ev[self.n]
        e["type"] = _cabi.EV_NODE_HEALTH
        e["arg0"] = node
        e["arg1"] = 1 if healthy else 0
        e["suggested_off"] = -1
        self.n += 1

    def finish(self) -> Tuple[np.ndarray, np.ndarray]:
        # byte-wise copy: numpy's structured copy leaves the alignment padding uninitialised
        out = np.zeros(self.n, dtype=EVENT_DT)
        out.view(np.uint8)[:] = self.ev[:self.n].view(np.uint8)
        return out, self.decision[:self.n].copy()


def trace_c1() -> Dict[str, Any]:
    """C1: 4 single-GPU pods (own group each), priority 0, typed K80; SURVEY.md section 8c."""
    tb = TraceBuilder(8)
    for i in range(4):
        tb.schedule(group=i, vc=0, priority=0, leaf_type=0, leaf_num=1, pod_num=1)
    ev, dec = tb.finish()
    return {"name": "C1", "config": config_c1(), "events": ev, "decision": dec, "n_groups": 4, "n_pods": tb.next_pod,
            "max_group_leaves": 8, "max_group_pods": 8}


def trace_c2(n_pods: int = 10000) -> Dict[str, Any]:
    """C2: 10 000 one-GPU single-pod groups, group i -> vc(i mod 4), no deletions."""
    tb = TraceBuilder(n_pods)
    for i in range(n_pods):
        tb.schedule(group=i, vc=i % 4, priority=0, leaf_type=0, leaf_num=1, pod_num=1)
    ev, dec = tb.finish()
    return {"name": "C2", "config": config_c2(), "events": ev, "decision": dec, "n_groups": n_pods,
            "n_pods": tb.next_pod, "max_group_leaves": 8, "max_group_pods": 8}


def _gang_shape(r: int) -> Tuple[int, int]:
    """40 % 1x1, 25 % 1x4, 25 % 1x8, 10 % 8x8 -> (pod_num, leaf_num); r uniform in [0,100)."""
    if r < 40:
        return 1, 1
    if r < 65:
        return 1, 4
    if r < 90:
        return 1, 8
    return 8, 8


def trace_c3(n_gangs: int = 100000, n_vcs: int = 8, vc_gpus: int = 7168, load: float = 0.9,
             config_number: int = 3) -> Dict[str, Any]:
    """C3: 100 000 mixed gangs on the 64k-GPU tree with the per-VC admission window."""
    rng = XorShift64Star(seed_for(config_number))
    tb = TraceBuilder(4 * n_gangs)
    alive: List[deque] = [deque() for _ in range(n_vcs)]  # (group, pod_num, leaf_num)
    alive_gpus = [0] * n_vcs
    limit = int(load * vc_gpus)
    for g in range(n_gangs):
        pod_num, leaf_num = _gang_shape(rng.below(100))
        v = rng.below(n_vcs)
        size = pod_num * leaf_num
        while alive_gpus[v] + size > limit and alive[v]:
            og, opn, oln = alive[v].popleft()
            for j in range(opn):
                tb.delete_allocated(og, oln, j, vc=v)
            alive_gpus[v] -= opn * oln
        for j in range(pod_num):
            tb.schedule(group=g, vc=v, priority=0, leaf_type=0, leaf_num=leaf_num, pod_num=pod_num, first=(j == 0))
        alive[v].append((g, pod_num, leaf_num))
        alive_gpus[v] += size
    ev, dec = tb.finish()
    return {"name": "C%d" % config_number, "config": config_c3(), "events": ev, "decision": dec,
            "n_groups": n_gangs, "n_pods": tb.next_pod, "max_group_leaves": 64, "max_group_pods": 8}


def trace_multi_member(n_gangs: int = 1200, n_vcs: int = 2, vc_gpus: int = (16 + 6) * 32 * 8, load: float = 0.85,
                       config=None) -> Dict[str, Any]:
    """Gangs with several members (AffinityGroup.Members with different leafCellNumbers, api/types.go:90-99): e.g.
    1 x 8-GPU + 2 x 4-GPU + 3 x 1-GPU pods, scheduled pod by pod in a PRNG-shuffled member order, with the admission
    window of C3.  Not a BASELINE config: it covers the member bookkeeping (merged, sorted members; slot offsets) of
    the whole-gang commit / release paths, which the single-member C1-C5 traces do not."""
    rng = XorShift64Star(seed_for(7))
    shapes = [[(8, 1), (4, 2), (1, 3)], [(4, 1), (2, 2)], [(8, 2), (1, 1)], [(1, 2), (2, 1), (4, 1), (8, 1)], [(8, 8)],
              [(2, 3)], [(4, 2), (8, 4)]]
    tb = TraceBuilder(16 * n_gangs)
    alive: List[deque] = [deque() for _ in range(n_vcs)]
    alive_gpus = [0] * n_vcs
    limit = int(load * vc_gpus)
    for g in range(n_gangs):
        members = shapes[rng.below(len(shapes))]
        v = rng.below(n_vcs)
        size = sum(ln * pn for ln, pn in members)
        while alive_gpus[v] + size > limit and alive[v]:
            og, om = alive[v].popleft()
            for ln, pn in om:
                for j in range(pn):
                    tb.delete_allocated(og, ln, j, vc=v)
            alive_gpus[v] -= sum(ln * pn for ln, pn in om)
        # the spec lists the members in a shuffled order; pods arrive member by member in that order
        order = list(members)
        for i in range(len(order) - 1, 0, -1):
            j = rng.below(i + 1)
            order[i], order[j] = order[j], order[i]
        first = True
        for ln, pn in order:
            for _ in range(pn):
                tb.schedule(group=g, vc=v, priority=0, leaf_type=0, leaf_num=ln, pod_num=pn, first=first, members=order)
                first = False
        alive[v].append((g, members))
        alive_gpus[v] += size
    ev, dec = tb.finish()
    from .config import config_c3
    return {"name": "multi-member", "config": config if config is not None else config_c3(n_pods=4, n_vcs=2, racks_per_vc=6),
            "events": ev, "decision": dec, "n_groups": n_gangs, "n_pods": tb.next_pod, "max_group_leaves": 64,
            "max_group_pods": 16}


def config_heterogeneous() -> Dict[str, Any]:
    """Two chains (leaf types A and B, different depths and fan-outs), a pinned cell, VCs that own cells of both
    chains at different levels — the shape of the reference's own test cluster, sized for thousands of decisions."""
    from .config import new_config
    raw = {
        "physicalCluster": {
            "cellTypes": {
                "A-NODE": {"childCellType": "A", "childCellNumber": 4, "isNodeLevel": True},
                "A-RACK": {"childCellType": "A-NODE", "childCellNumber": 4},
                "B-NODE": {"childCellType": "B", "childCellNumber": 8, "isNodeLevel": True},
                "B-RACK": {"childCellType": "B-NODE", "childCellNumber": 2},
                "B-POD": {"childCellType": "B-RACK", "childCellNumber": 2},
            },
            "physicalCells": (
                [{"cellType": "A-RACK",
                  "cellChildren": [dict({"cellAddress": "a%d" % (4 * r + i)}, **({"pinnedCellId": "pin0"} if (r, i) == (0, 0) else {}))
                                   for i in range(4)]} for r in range(4)] +
                [{"cellType": "B-POD",
                  "cellChildren": [{"cellChildren": [{"cellAddress": "b%d" % (4 * p + 2 * r + i)} for i in range(2)]}
                                   for r in range(2)]} for p in range(3)]),
        },
        "virtualClusters": {
            "vc0": {"virtualCells": [{"cellType": "A-RACK", "cellNumber": 1}, {"cellType": "B-POD.B-RACK", "cellNumber": 3}],
                    "pinnedCells": [{"pinnedCellId": "pin0"}]},
            "vc1": {"virtualCells": [{"cellType": "A-RACK.A-NODE", "cellNumber": 5}, {"cellType": "B-POD", "cellNumber": 1}]},
        },
    }
    return new_config(raw)


def trace_heterogeneous(n_gangs: int = 1500) -> Dict[str, Any]:
    """Typed (A / B), untyped and pinned-cell requests of 1-8 GPUs over config_heterogeneous, in one ordered batch with
    deletions; some requests must wait (the wait results are part of the parity)."""
    rng = XorShift64Star(seed_for(8))
    tb = TraceBuilder(8 * n_gangs)
    alive: deque = deque()
    for g in range(n_gangs):
        v = rng.below(2)
        kind = rng.below(10)
        pinned = -1
        if kind < 4:
            leaf_type, leaf_num, pod_num = 0, [1, 2, 4, 4][rng.below(4)], 1 + rng.below(2)      # type A
        elif kind < 8:
            leaf_type, leaf_num, pod_num = 1, [1, 2, 4, 8][rng.below(4)], 1 + rng.below(2)      # type B
        elif kind == 8:
            leaf_type, leaf_num, pod_num = -1, 1 + rng.below(2), 1                               # any leaf cell type
        else:
            v, pinned, leaf_type, leaf_num, pod_num = 0, 0, -1, 1 + rng.below(2), 1             # vc0's pinned cell
        while len(alive) > 18:
            og, opn, oln, ov = alive.popleft()
            for j in range(opn):
                tb.delete_allocated(og, oln, j, vc=ov)
        for j in range(pod_num):
            tb.schedule(group=g, vc=v, priority=0, leaf_type=leaf_type, leaf_num=leaf_num, pod_num=pod_num, first=(j == 0))
            tb.ev[tb.n - 1]["spec"]["pinned"] = pinned
        alive.append((g, pod_num, leaf_num, v))
    ev, dec = tb.finish()
    return {"name": "heterogeneous", "config": config_heterogeneous(), "events": ev, "decision": dec, "n_groups": n_gangs,
            "n_pods": tb.next_pod, "max_group_leaves": 16, "max_group_pods": 8}


def trace_suggested_nodes(n_gangs: int = 900, n_sets: int = 6) -> Dict[str, Any]:
    """K8s suggested nodes in batch mode: most requests honour a suggested-node set (ignoreK8sSuggestedNodes = false,
    hived_algorithm.go:190-193) drawn from a few PRNG bitmaps that leave out ~15 % of the nodes; some nodes are bad.
    Covers the suggested / healthy sort keys, the non-suggested wait reasons and the backtracking mapping
    (cell_allocation.go:199-315) through hived_event_t.suggested_off."""
    from .config import config_c3
    cfg = config_c3(n_pods=4, n_vcs=2, racks_per_vc=6)
    n_nodes = 4 * 16 * 32
    words = (n_nodes + 31) // 32
    rng = XorShift64Star(seed_for(9))
    pool = np.zeros(n_sets * words, dtype=np.uint32)
    for k in range(n_sets):
        for node in range(n_nodes):
            if rng.below(100) >= 15:
                pool[k * words + (node >> 5)] |= np.uint32(1 << (node & 31))
    tb = TraceBuilder(8 * n_gangs)
    for _ in range(40):
        tb.node_health(rng.below(n_nodes), False)
    alive: List[deque] = [deque() for _ in range(2)]
    alive_gpus = [0, 0]
    limit = int(0.8 * (16 + 6) * 32 * 8)
    for g in range(n_gangs):
        pod_num, leaf_num = _gang_shape(rng.below(100))
        v = rng.below(2)
        size = pod_num * leaf_num
        while alive_gpus[v] + size > limit and alive[v]:
            og, opn, oln = alive[v].popleft()
            for j in range(opn):
                tb.delete_allocated(og, oln, j, vc=v)
            alive_gpus[v] -= opn * oln
        honour = rng.below(10) < 7
        off = rng.below(n_sets) * words
        phase = _cabi.PHASE_FILTERING if rng.below(2) else _cabi.PHASE_PREEMPTING
        for j in range(pod_num):
            tb.schedule(group=g, vc=v, priority=0, leaf_type=0, leaf_num=leaf_num, pod_num=pod_num, first=(j == 0),
                        flags=0 if honour else _cabi.SPEC_IGNORE_SUGGESTED, phase=phase)
            if honour:
                tb.ev[tb.n - 1]["suggested_off"] = off
        alive[v].append((g, pod_num, leaf_num))
        alive_gpus[v] += size
    ev, dec = tb.finish()
    return {"name": "suggested-nodes", "config": cfg, "events": ev, "decision": dec, "n_groups": n_gangs,
            "n_pods": tb.next_pod, "max_group_leaves": 64, "max_group_pods": 8, "sugg_pool": pool}


def trace_bad_requests() -> Dict[str, Any]:
    """Requests the reference answers with a 400 / a panic, interleaved with good ones in one batch (every event gets its
    own error code; a failing event leaves the state unchanged, pkg/internal/types.go:58-61): unknown VC, unknown /
    foreign leaf type, unknown pinned cell, opportunistic pod in a pinned cell, priority / leaf number out of range,
    a pod that is not a member of its own group, more pods than the member has, deletes of unknown groups and slots.
    (Ids or sizes beyond hived_options_t fail the whole call with HIVED_ERR_CAPACITY and are not part of this batch.)"""
    cfg = config_heterogeneous()
    tb = TraceBuilder(256)

    def bad(**over):
        tb.schedule(group=over.pop("group", 900), vc=over.pop("vc", 0), priority=over.pop("priority", 0),
                    leaf_type=over.pop("leaf_type", 0), leaf_num=over.pop("leaf_num", 1), pod_num=over.pop("pod_num", 1),
                    members=over.pop("members", None), first=True)
        e = tb.ev[tb.n - 1]
        for k, val in over.items():
            e["spec"][k] = val

    for rnd in range(3):
        g0 = 10 * rnd
        tb.schedule(group=g0, vc=0, priority=0, leaf_type=0, leaf_num=2, pod_num=2)          # good: pod 0 of a 2-pod gang
        bad(vc=-1)                                                                           # unknown VC
        bad(vc=7)
        bad(leaf_type=-2)                                                                    # unknown leaf type string
        bad(leaf_type=5)
        bad(pinned=-2)                                                                       # unknown pinned cell id
        bad(pinned=3)
        bad(vc=1, pinned=0)                                                                  # vc1 does not own pin0
        bad(pinned=0, priority=-1)                                                           # opportunistic in a pinned cell
        bad(priority=-2)
        bad(priority=1001)
        bad(leaf_num=0)
        bad(leaf_num=3, members=[(2, 1)])                                                    # pod not among the members
        bad(members=[(1, 0)])
        tb.schedule(group=g0, vc=0, priority=0, leaf_type=0, leaf_num=2, pod_num=2)          # good: pod 1
        tb.schedule(group=g0, vc=0, priority=0, leaf_type=0, leaf_num=2, pod_num=2)          # a third pod: too many
        tb.schedule(group=g0 + 1, vc=1, priority=0, leaf_type=1, leaf_num=8, pod_num=1)      # good, other chain
        tb.delete_allocated(777, 1, 0, vc=0)                                                 # unknown group: no-op
        tb.delete_allocated(g0, 2, 5, vc=0)                                                  # slot out of range
        tb.delete_allocated(g0, 3, 0, vc=0)                                                  # no member with 3 leaves
        tb.delete_allocated(g0, 2, 0, vc=0)
        tb.delete_allocated(g0, 2, 1, vc=0)                                                  # last pod: the gang is released
        tb.delete_allocated(g0, 2, 1, vc=0)                                                  # again: unknown by now
    ev, dec = tb.finish()
    return {"name": "bad-requests", "config": cfg, "events": ev, "decision": dec, "n_groups": 1000, "n_pods": tb.next_pod,
            "max_group_leaves": 16, "max_group_pods": 8}


def trace_c5(n_steps: int = 10, gangs_per_step: int = 2000, n_nodes: int = 8192, n_vcs: int = 8, vc_gpus: int = 7168,
             flip_fraction: float = 0.1, load: float = 0.9, config=None) -> Dict[str, Any]:
    """C5: churn — every step flips the health of 10 % PRNG-chosen nodes, then schedules 2000 gangs
    (C3 mix, admission window).  Gangs on nodes that went bad stay allocated (hived_algorithm.go:677-682)."""
    rng = XorShift64Star(seed_for(5))
    tb = TraceBuilder(8 * n_steps * gangs_per_step)
    healthy = [True] * n_nodes
    alive: List[deque] = [deque() for _ in range(n_vcs)]
    alive_gpus = [0] * n_vcs
    limit = int(load * vc_gpus)
    g = 0
    for _ in range(n_steps):
        for _k in range(int(flip_fraction * n_nodes)):
            node = rng.below(n_nodes)
            healthy[node] = not healthy[node]
            tb.node_health(node, healthy[node])
        for _k in range(gangs_per_step):
            pod_num, leaf_num = _gang_shape(rng.below(100))
            v = rng.below(n_vcs)
            size = pod_num * leaf_num
            while alive_gpus[v] + size > limit and alive[v]:
                og, opn, oln = alive[v].popleft()
                for j in range(opn):
                    tb.delete_allocated(og, oln, j, vc=v)
                alive_gpus[v] -= opn * oln
            for j in range(pod_num):
                tb.schedule(group=g, vc=v, priority=0, leaf_type=0, leaf_num=leaf_num, pod_num=pod_num, first=(j == 0))
            alive[v].append((g, pod_num, leaf_num))
            alive_gpus[v] += size
            g += 1
    ev, dec = tb.finish()
    return {"name": "C5", "config": config if config is not None else config_c3(), "events": ev, "decision": dec,
            "n_groups": g, "n_pods": tb.next_pod, "max_group_leaves": 64, "max_group_pods": 8}


def run_c4_interactive(lib, config, n_gangs: int, n_vcs: int, vc_gpus: int, total_gpus: int, load: float = 0.9,
                       max_groups: int = None, lazy_percent: int = 0):
    """C4: guaranteed (priority 0/1/2, lazyPreemptionEnable false) and opportunistic (-1) gangs interleaved by
    the PRNG.  The event stream depends on the decisions, so the harness plays kube-scheduler call by call
    (SURVEY.md section 8d): Filtering-phase Schedule; on a preempt result -> Preempting-phase Schedule ->
    delete every pod of every victim gang -> Filtering-phase Schedule again.  Returns (hash, decision log).
    lazy_percent > 0 (not a BASELINE config): that share of the guaranteed gangs sets lazyPreemptionEnable, so a
    higher-priority gang downgrades them to opportunistic instead of preempting them (hived_algorithm.go:944-965,
    1165-1222)."""
    rng = XorShift64Star(seed_for(4))
    lazy_rng = XorShift64Star(seed_for(14))
    bc = BatchContext(lib, config, max_groups or (n_gangs + 8), 8 * n_gangs + 64, 64, 8)
    bc.set_all_nodes_healthy()
    tb = TraceBuilder(4)
    pod_home = {}      # pod id -> (group, leaf_num, pod_index, vc)
    group_pods = {}    # group -> [pod ids]
    group_size = {}
    alive = [deque() for _ in range(n_vcs)]
    alive_gpus = [0] * n_vcs
    opp_alive, opp_gpus = deque(), 0
    log = []
    lazy_seen = set()

    def one(ev_builder):
        tb.n = 0
        ev_builder()
        res, pool = bc.process(tb.ev[:tb.n].copy(), 4096)
        return res[0], pool

    def delete_group(g, v):
        for pid in group_pods.pop(g, []):
            _, ln, pi, _ = pod_home.pop(pid)
            one(lambda: tb.delete_allocated(g, ln, pi, vc=v))

    for g in range(n_gangs):
        pod_num, leaf_num = _gang_shape(rng.below(100))
        v = rng.below(n_vcs)
        opportunistic = rng.below(2) == 1
        prio = -1 if opportunistic else rng.below(3)
        size = pod_num * leaf_num
        gang_flags = _cabi.SPEC_IGNORE_SUGGESTED
        if lazy_percent > 0 and not opportunistic and lazy_rng.below(100) < lazy_percent:
            gang_flags |= _cabi.SPEC_LAZY_PREEMPTION
        if opportunistic:
            while opp_gpus + size > int(load * total_gpus) and opp_alive:
                og, ov = opp_alive.popleft()
                if og in group_pods:
                    opp_gpus -= group_size[og]
                    delete_group(og, ov)
        else:
            while alive_gpus[v] + size > int(load * vc_gpus) and alive[v]:
                og = alive[v].popleft()
                if og in group_pods:
                    alive_gpus[v] -= group_size[og]
                    delete_group(og, v)
        bound = True
        for j in range(pod_num):
            def sched(phase):
                pid = tb.next_pod
                tb.schedule(group=g, vc=v, priority=prio, leaf_type=0, leaf_num=leaf_num, pod_num=pod_num, phase=phase,
                            flags=gang_flags, first=(j == 0))
                return pid
            holder = {}
            r, pool = one(lambda: holder.setdefault("pid", sched(_cabi.PHASE_FILTERING)))
            if r["kind"] == _cabi.KIND_PREEMPT:
                r, pool = one(lambda: holder.__setitem__("pid", sched(_cabi.PHASE_PREEMPTING)))
                victims = sorted({int(pool[r["victim_off"] + 2 * k]) for k in range(int(r["n_victims"]))})
                log.append((g, j, "preempt", tuple(victims)))
                for vg in sorted({pod_home[p][0] for p in victims if p in pod_home}):
                    vv = pod_home[group_pods[vg][0]][3]
                    if vg in group_size:
                        if vv >= 0 and vg in alive[vv]:
                            alive_gpus[vv] -= group_size[vg]
                        elif vv < 0:
                            opp_gpus -= group_size[vg]
                    delete_group(vg, vv if vv >= 0 else 0)
                r, pool = one(lambda: holder.__setitem__("pid", sched(_cabi.PHASE_FILTERING)))
            if r["kind"] == _cabi.KIND_BIND:
                pid = holder["pid"]
                pod_home[pid] = (g, leaf_num, int(r["pod_index"]), -1 if opportunistic else v)
                group_pods.setdefault(g, []).append(pid)
                log.append((g, j, "bind", int(r["node"]),
                            tuple(int(pool[r["this_off"] + 3 * k + 1]) for k in range(int(r["this_n"])))))
            else:
                log.append((g, j, "wait" if r["kind"] == _cabi.KIND_WAIT else "preempt-again", int(r["wait_code"])))
                bound = False
                break
        if bound and lazy_percent > 0 and not opportunistic:
            # which alive gangs of this VC have lost their virtual placement (were lazy-preempted) by now?
            gi = _cabi.GroupInfo()
            for og in alive[v]:
                if og in group_pods and og not in lazy_seen:
                    lib.hived_get_group(bc.ctx, og, C.byref(gi))
                    if gi.state != _cabi.GROUP_NONE and not gi.has_virtual:
                        lazy_seen.add(og)
        if bound:
            group_size[g] = size
            if opportunistic:
                opp_alive.append((g, v)); opp_gpus += size
            else:
                alive[v].append(g); alive_gpus[v] += size
        elif g in group_pods:
            delete_group(g, v)
    h = bc.result_hash()
    stats = bc.stats()
    stats["lazy_preempted_groups"] = len(lazy_seen)  # gangs observed without a virtual placement while alive
    bc.close()
    return h, log, stats


def run_c4_compiled(lib, config, n_gangs: int, n_vcs: int, vc_gpus: int, total_gpus: int, load: float = 0.9,
                    max_groups: int = None, batch_deletes: bool = True, player_path: str = None):
    """The closed loop of run_c4_interactive played by compiled code (tests/harness/c4_player.cpp; built by
    __graft_entry__.build_c4_player) — no interpreter between the calls; the deletions of one gang's pods travel as one
    batch of <= 8 events.  Returns (hash, decision log in run_c4_interactive's format, stats, timing dict)."""
    import os
    if player_path is None:
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        player_path = os.path.join(root, "tests", "_build", "libhived_c4player.so")
        if not os.path.exists(player_path):  # (normally built by __graft_entry__.build())
            import sys
            if root not in sys.path:
                sys.path.insert(0, root)
            import __graft_entry__ as ge
            ge.build_c4_player()
    player = C.CDLL(player_path)
    player.c4_play.restype = C.c_int
    bc = BatchContext(lib, config, max_groups or (n_gangs + 8), 8 * n_gangs + 64, 64, 8)
    bc.set_all_nodes_healthy()
    cap = 80 * n_gangs + 4096
    buf = np.zeros(cap, dtype=np.int32)
    words, calls, events, secs = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_double(0.0)
    rc = player.c4_play(C.cast(lib.hived_process_events, C.c_void_p), bc.ctx, C.c_int32(n_gangs), C.c_int32(n_vcs),
                        C.c_int32(vc_gpus), C.c_int32(total_gpus), C.c_double(load), C.c_int32(1 if batch_deletes else 0),
                        buf.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int64(cap), C.byref(words), C.byref(calls),
                        C.byref(events), C.byref(secs))
    if rc != 0:
        raise RuntimeError("c4_play failed (%d): %s" % (rc, (lib.hived_last_error(bc.ctx) or b"").decode()))
    log, i, w = [], 0, buf[:words.value].tolist()
    kinds = ("preempt", "bind", "wait", "preempt-again")
    while i < len(w):
        g, j, kind, n = w[i:i + 4]
        payload = w[i + 4:i + 4 + n]
        i += 4 + n
        if kind == 0:
            log.append((g, j, "preempt", tuple(payload)))
        elif kind == 1:
            log.append((g, j, "bind", payload[0], tuple(payload[1:])))
        else:
            log.append((g, j, kinds[kind], payload[0]))
    h = bc.result_hash()
    stats = bc.stats()
    stats["lazy_preempted_groups"] = 0
    bc.close()
    return h, log, stats, {"calls": calls.value, "events": events.value, "seconds": secs.value}


# ------------------------------------------------------------------------------------------------
# batch driver
# ------------------------------------------------------------------------------------------------

class BatchContext:
    """A raw ctx of include/hived.h for the batch path (bench.py, parity tests).  flags: hived_options_t.flags
    (_cabi.OPT_*)."""

    def __init__(self, lib, config: Dict[str, Any], max_groups: int, max_pods: int, max_group_leaves: int = 64,
                 max_group_pods: int = 8, device: int = 0, flags: int = 0):
        from .config import to_spec_text
        self.lib = lib
        self.opt = _cabi.Options(max_groups=max_groups, max_pods=max_pods, max_group_leaves=max_group_leaves,
                                 max_group_pods=max_group_pods, device=device, flags=flags)
        self.ctx = C.c_void_p()
        rc = lib.hived_create(to_spec_text(config).encode(), C.byref(self.opt), C.byref(self.ctx))
        if rc != 0:
            raise RuntimeError("hived_create failed (%d): %s" % (rc, (lib.hived_create_error() or b"").decode()))
        self.n_nodes = lib.hived_num_nodes(self.ctx)

    def clone(self, device: int = -1, flags: int = 0) -> "BatchContext":
        """hived_clone (include/hived_clone.h): a new BatchContext over an independent copy of this one's context."""
        out = C.c_void_p()
        rc = _cabi.bind_clone(self.lib).hived_clone(self.ctx, device, flags, C.byref(out))
        if rc != 0:
            raise RuntimeError("hived_clone failed (%d): %s" % (rc, (self.lib.hived_create_error() or b"").decode()))
        bc = BatchContext.__new__(BatchContext)
        bc.lib, bc.ctx, bc.n_nodes = self.lib, out, self.n_nodes
        bc.opt = _cabi.Options.from_buffer_copy(self.opt)
        bc.opt.device, bc.opt.flags = self.opt.device if device < 0 else device, flags
        return bc

    def set_all_nodes_healthy(self):
        """Healthy nodes arrive in ascending node id (= name) order (SURVEY.md Appendix A item 10)."""
        ev = np.zeros(self.n_nodes, dtype=EVENT_DT)
        ev["type"] = _cabi.EV_NODE_HEALTH
        ev["arg0"] = np.arange(self.n_nodes, dtype=np.int32)
        ev["arg1"] = 1
        ev["suggested_off"] = -1
        self.process(ev, pool_words=16)

    def process(self, events: np.ndarray, pool_words: int = None, sugg_pool: np.ndarray = None):
        """sugg_pool: uint32 words backing hived_event_t.suggested_off (node bitmaps), or None."""
        n = len(events)
        if pool_words is None:
            pool_words = 3 * 64 * n // 4 + 4096
        res = np.zeros(n, dtype=RESULT_DT)
        pool = np.zeros(pool_words, dtype=np.int32)
        events = np.ascontiguousarray(events)
        sp, sw = None, 0
        if sugg_pool is not None and len(sugg_pool):
            sugg_pool = np.ascontiguousarray(sugg_pool, dtype=np.uint32)
            sp, sw = sugg_pool.ctypes.data_as(C.POINTER(C.c_uint32)), len(sugg_pool)
        rc = self.lib.hived_process_events(
            self.ctx, events.ctypes.data_as(C.POINTER(_cabi.Event)), n, sp, sw,
            res.ctypes.data_as(C.POINTER(_cabi.Result)), pool.ctypes.data_as(C.POINTER(C.c_int32)), pool_words)
        if rc != 0:
            raise RuntimeError("hived_process_events failed (%d): %s" % (
                rc, (self.lib.hived_last_error(self.ctx) or b"").decode()))
        return res, pool

    def result_hash(self) -> int:
        return int(self.lib.hived_result_hash(self.ctx))

    def turns(self) -> int:
        """hived_bench_turns (include/hived_bench.h): this context's calls that took turns on the library's device lock."""
        fn = self.lib.hived_bench_turns
        fn.restype, fn.argtypes = C.c_int64, [C.c_void_p]
        return int(fn(self.ctx))

    def stats(self) -> Dict[str, int]:
        st = _cabi.Stats()
        self.lib.hived_get_stats(self.ctx, C.byref(st))
        return {f: getattr(st, f) for f, _ in _cabi.Stats._fields_}

    def close(self):
        if self.ctx:
            self.lib.hived_destroy(self.ctx)
            self.ctx = None


def process_many(batch_contexts: List[BatchContext], events_list: List[np.ndarray], pool_words_list: List[int],
                 sugg_pools: List[np.ndarray] = None):
    """The batches of several contexts of one library and device in one call (hived_process_events_many,
    include/hived_multictx.h).  Returns [(rc, results, pool)] in list order; each rc is what BatchContext.process's
    hived_process_events would have returned.  Raises if the call itself fails (a refused list, a failed launch)."""
    k = len(batch_contexts)
    lib = _cabi.bind_many(batch_contexts[0].lib)
    if sugg_pools is None:
        sugg_pools = [None] * k
    arr = (_cabi.Batch * max(k, 1))()
    keep = []
    for i, (bc, ev, words, sp) in enumerate(zip(batch_contexts, events_list, pool_words_list, sugg_pools)):
        ev = np.ascontiguousarray(ev)
        res = np.zeros(len(ev), dtype=RESULT_DT)
        pool = np.zeros(max(int(words), 1), dtype=np.int32)
        b = arr[i]
        b.ctx, b.n, b.pool_cap = bc.ctx, len(ev), int(words)
        b.events = ev.ctypes.data_as(C.POINTER(_cabi.Event))
        b.res = res.ctypes.data_as(C.POINTER(_cabi.Result))
        b.pool = pool.ctypes.data_as(C.POINTER(C.c_int32))
        if sp is not None and len(sp):
            sp = np.ascontiguousarray(sp, dtype=np.uint32)
            b.suggested_pool, b.suggested_words = sp.ctypes.data_as(C.POINTER(C.c_uint32)), len(sp)
        keep.append((ev, res, pool, sp))
    rc = lib.hived_process_events_many(arr, k)
    if rc != 0:
        raise RuntimeError("hived_process_events_many failed (%d)" % rc)
    return [(arr[i].rc, keep[i][1], keep[i][2]) for i in range(k)]


def pool_words_for(trace: Dict[str, Any]) -> int:
    """Upper bound of result-pool words: every SCHEDULE event may emit the whole gang placement."""
    ev = trace["events"]
    sched = ev[ev["type"] == _cabi.EV_SCHEDULE]["spec"]
    leaves = (sched["member_leaf_num"][:, 0].astype(np.int64) * sched["member_pod_num"][:, 0]).sum()
    return int(3 * leaves + 4096)
