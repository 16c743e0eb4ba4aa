"""Logic parity of the DEVICE PROGRAM (csrc/hived_core.h) against the oracle, executed on the host by
the test-only 1-thread emulation (tests/emu).  The real sm_90a build is covered by test_gpu_parity.py;
these tests let kernel-logic regressions show up in the CPU-only CI tier."""
import numpy as np
import pytest

from conftest import run_trace
from golden_scenario import Scenario
from hivedscheduler_b200 import config, trace


def test_emu_reproduces_reference_golden_vectors(emu_lib, oracle_lib):
    sc = Scenario(emu_lib)
    assert sc.run() == []
    so = Scenario(oracle_lib)
    assert so.run() == []
    assert sc.decisions == so.decisions  # full PodBindInfo / victims / wait-reason strings


@pytest.mark.parametrize("name", ["C1", "C2"])
def test_emu_matches_oracle_on_trace(emu_lib, oracle_lib, name):
    t = trace.trace_c1() if name == "C1" else trace.trace_c2(n_pods=3000)
    he, re_, se = run_trace(emu_lib, t)
    ho, ro, so = run_trace(oracle_lib, t)
    assert he == ho
    assert se == so  # identical work counters => identical algorithmic bytes
    for (a, pa), (b, pb) in zip(re_, ro):
        assert a.tobytes() == b.tobytes()


def small_c3(n_gangs=1500):
    """C3's shape (5 levels, mixed 1/4/8/64-GPU gangs, admission window) on 4 PODs / 2 VCs."""
    t = trace.trace_c3(n_gangs=n_gangs, n_vcs=2, vc_gpus=(16 + 6) * 32 * 8, config_number=3)
    t["config"] = config.config_c3(n_pods=4, n_vcs=2, racks_per_vc=6)
    return t


def test_emu_matches_oracle_on_small_c3(emu_lib, oracle_lib):
    t = small_c3()
    snaps = []
    he, re_, se = run_trace(emu_lib, t, chunks=3, snapshots=snaps)
    ho, ro, so = run_trace(oracle_lib, t, chunks=3, snapshots=snaps)
    assert he == ho
    assert se == so
    assert snaps[0] == snaps[1]  # every cell's priority / state / health / binding / free-list membership
    sched = t["events"]["type"] == 0
    assert (np.concatenate([r[0]["kind"] for r in re_])[sched] == 1).all()


def test_emu_matches_oracle_on_multi_member_gangs(emu_lib, oracle_lib):
    """Several members per gang, listed in shuffled order (members are merged and sorted, types.go:157-160)."""
    t = trace.trace_multi_member()
    snaps = []
    he, re_, se = run_trace(emu_lib, t, chunks=3, snapshots=snaps)
    ho, ro, so = run_trace(oracle_lib, t, chunks=3, snapshots=snaps)
    assert he == ho and se == so
    assert snaps[0] == snaps[1]
    for (a, pa), (b, pb) in zip(re_, ro):
        assert a.tobytes() == b.tobytes()
    kinds = np.concatenate([r[0]["kind"] for r in re_])[t["events"]["type"] == 0]
    assert (kinds == 1).all()


def test_emu_matches_oracle_on_heterogeneous_cluster(emu_lib, oracle_lib):
    """Two chains, a pinned cell, typed / untyped / pinned requests, waits and deletes in one batch."""
    t = trace.trace_heterogeneous()
    snaps = []
    he, re_, se = run_trace(emu_lib, t, chunks=2, snapshots=snaps)
    ho, ro, so = run_trace(oracle_lib, t, chunks=2, snapshots=snaps)
    assert he == ho and se == so
    assert snaps[0] == snaps[1]
    for (a, pa), (b, pb) in zip(re_, ro):
        assert a.tobytes() == b.tobytes()
    sched = t["events"]["type"] == 0
    kinds = np.concatenate([r[0]["kind"] for r in re_])[sched]
    errors = np.concatenate([r[0]["error"] for r in re_])[sched]
    assert (errors == 0).all() and (kinds == 1).sum() > 500 and (kinds == 0).sum() > 0  # binds and waits both occur


def test_emu_matches_oracle_with_suggested_node_sets(emu_lib, oracle_lib):
    """Suggested-node bitmaps through the batch interface, bad nodes, both scheduling phases."""
    t = trace.trace_suggested_nodes()
    snaps = []
    he, re_, se = run_trace(emu_lib, t, chunks=2, snapshots=snaps)
    ho, ro, so = run_trace(oracle_lib, t, chunks=2, snapshots=snaps)
    assert he == ho and se == so
    assert snaps[0] == snaps[1]
    for (a, pa), (b, pb) in zip(re_, ro):
        assert a.tobytes() == b.tobytes()
    sched = t["events"]["type"] == 0
    kinds = np.concatenate([r[0]["kind"] for r in re_])[sched]
    codes = np.concatenate([r[0]["wait_code"] for r in re_])[sched]
    assert (kinds == 1).sum() > 300
    assert len(np.unique(codes[kinds == 0])) >= 1  # some requests wait on bad / non-suggested nodes


def test_emu_matches_oracle_with_lazy_preemption(emu_lib, oracle_lib):
    """C4's call-by-call harness with lazyPreemptionEnable on half of the guaranteed gangs (lazy preemption,
    revert on a failed mapping, downgraded gangs being deleted / preempted later)."""
    # no admission window (load 3): the VCs fill up, higher priorities have to take cells from lower ones
    kw = dict(config=small_cluster(), n_gangs=4500, n_vcs=2, vc_gpus=(16 + 6) * 32 * 8, total_gpus=4 * 16 * 32 * 8,
              lazy_percent=50, load=3.0)
    he, le, se = trace.run_c4_interactive(emu_lib, **kw)
    ho, lo, so = trace.run_c4_interactive(oracle_lib, **kw)
    assert le == lo
    assert he == ho and se == so
    assert so["lazy_preempted_groups"] > 0  # lazy preemption really happens in this workload


def test_emu_matches_oracle_on_bad_requests(emu_lib, oracle_lib):
    """Requests the reference rejects (400s and panics), interleaved with good ones: per-event error codes, and the
    state after a failing event is the state before it."""
    t = trace.trace_bad_requests()
    snaps = []
    he, re_, se = run_trace(emu_lib, t, snapshots=snaps)
    ho, ro, so = run_trace(oracle_lib, t, snapshots=snaps)
    assert he == ho and se == so and snaps[0] == snaps[1]
    assert re_[0][0].tobytes() == ro[0][0].tobytes()
    errors = set(int(e) for e in re_[0][0]["error"])
    assert {0, 1, 2, 3, 4, 6, 7, 100} <= errors  # unknown VC / pinned / opp-in-pinned / leaf type / too many pods / bad spec / panic


@pytest.mark.parametrize("field,value", [("group", 5000), ("group", -1), ("pod", 10 ** 6), ("member_leaf_num", 64)])
def test_ids_beyond_the_capacities_fail_the_call(emu_lib, oracle_lib, field, value):
    """Interned ids / gang sizes beyond hived_options_t are a HIVED_ERR_CAPACITY for the whole call (102), on both."""
    t = trace.trace_bad_requests()
    tb = trace.TraceBuilder(4)
    tb.schedule(group=1, vc=0, priority=0, leaf_type=0, leaf_num=1, pod_num=1)
    if field == "member_leaf_num":
        tb.ev[0]["spec"]["member_leaf_num"][0] = value
        tb.ev[0]["spec"]["leaf_num"] = value
    else:
        tb.ev[0]["spec"][field] = value
    ev, _ = tb.finish()
    for lib in (emu_lib, oracle_lib):
        bc = trace.BatchContext(lib, t["config"], 1000, 64, 16, 8)
        bc.set_all_nodes_healthy()
        with pytest.raises(RuntimeError) as ei:
            bc.process(ev, 4096)
        assert "(102)" in str(ei.value)
        bc.close()


def test_emu_matches_oracle_on_reseeded_traces(emu_lib, oracle_lib):
    """Two more seeds of every trace family (tests/fuzz_parity.py runs as many as one likes)."""
    import fuzz_parity
    assert fuzz_parity.run_seeds(emu_lib, oracle_lib, 1001, 2, verbose=False) == 0


def small_cluster():
    return config.config_c3(n_pods=4, n_vcs=2, racks_per_vc=6)


def test_emu_matches_oracle_under_churn_c5(emu_lib, oracle_lib):
    """C5 shape at a size the oracle finishes in seconds: node health flips + gangs (rows a11, a18)."""
    t = trace.trace_c5(n_steps=4, gangs_per_step=300, n_nodes=4 * 16 * 32, n_vcs=2, vc_gpus=(16 + 6) * 32 * 8,
                       config=small_cluster())
    snaps = []
    he, re_, se = run_trace(emu_lib, t, chunks=2, snapshots=snaps)
    ho, ro, so = run_trace(oracle_lib, t, chunks=2, snapshots=snaps)
    assert he == ho and se == so
    assert snaps[0] == snaps[1]
    kinds = np.concatenate([r[0]["kind"] for r in re_])[t["events"]["type"] == 0]
    assert (kinds == 1).sum() > 500  # most gangs still bind around the bad nodes


def test_emu_matches_oracle_with_preemption_c4(emu_lib, oracle_lib):
    """C4 shape (guaranteed priorities 0/1/2 + opportunistic, kube-scheduler emulation) — rows a12, a19."""
    kw = dict(config=small_cluster(), n_gangs=2500, n_vcs=2, vc_gpus=(16 + 6) * 32 * 8, total_gpus=4 * 16 * 32 * 8)
    he, le, se = trace.run_c4_interactive(emu_lib, **kw)
    ho, lo, so = trace.run_c4_interactive(oracle_lib, **kw)
    assert le == lo
    assert he == ho and se == so
    assert any(x[2] == "preempt" for x in le), "the scenario is expected to exercise preemption"


def test_compiled_c4_player_equals_python_harness(emu_lib):
    """tests/harness/c4_player.cpp (the closed loop of C4 as compiled code, what bench.py times) issues exactly the
    calls of trace.run_c4_interactive: same parity hash, decision log and work counters — with the deletions of a
    gang's pods sent one by one and as one batch."""
    import __graft_entry__ as ge
    ge.build_c4_player()
    kw = dict(config=small_cluster(), n_gangs=3500, n_vcs=2, vc_gpus=(16 + 6) * 32 * 8, total_gpus=4 * 16 * 32 * 8)
    hp, lp, sp = trace.run_c4_interactive(emu_lib, **kw)
    assert any(x[2] == "preempt" for x in lp)
    for batch in (False, True):
        hc, lc, sc, tm = trace.run_c4_compiled(emu_lib, batch_deletes=batch, **kw)
        assert lc == lp
        assert hc == hp and sc == sp
        assert tm["events"] > sp["schedule_events"]  # the deletions
        assert (tm["calls"] < tm["events"]) == batch


@pytest.mark.parametrize("seed", [16, 31, 160, 553, 775, 2385])
def test_api_fuzz_seeds_with_recreated_group(emu_lib, oracle_lib, seed):
    """tests/fuzz_api.py: random calls of the 14-method API, results + every cell + every view order compared after every
    call.  Seeds 16 and 31 erase a group that is being preempted while its leaves still name it and create a new group
    under the same name (hived_algorithm.go:671-707 -> :1114-1145): the old object lives on as a ghost record
    (Core::ghostify) — the victims of a later preemption are ITS pods.  160 / 553: nil dereferences of the reference
    (allocatePreassignedCell of a nil cell, lazy preemption of an unbound virtual leaf) are platform errors on both
    sides.  775: a pod deleted through a slot that holds ANOTHER pod stays a possible victim (the shim keeps it).
    2385: DeleteAllocatedPod of a pod bound under an earlier incarnation of a name deletes the PREEMPTING group that
    carries the name now; its Reserved leaves keep naming the erased object, and a later Schedule that overlaps them
    cancels "its" preemption (hived_algorithm.go:731-742): a ghost reached through p_resv, erased by name
    (Core::eraseGroupByName); the shim keeps the id with the name while hived_get_group reports `referenced`."""
    import fuzz_api
    assert fuzz_api.run_seed(emu_lib, oracle_lib, seed, 300) is None


@pytest.mark.parametrize("seed", [7, 12, 29, 782, 1059])
def test_api_fuzz_with_filtering_phase_calls(emu_lib, oracle_lib, seed, monkeypatch):
    """The same fuzz with 40 % of the Schedule calls in the Filtering phase (FUZZ_FILTERING=1): binds that land on
    Reserved cells make the reference's incremental used-leaf counters drift from its leaf priorities (modelled exactly:
    noteDelta), and seed 7 reaches a Reserved cell without a reserving group — the reference dereferences the nil
    group when it cancels the overlapping preemptions (hived_algorithm.go:1116): a platform error on both sides.
    Seed 782 releases a preassigned cell that is already free, again and again: the reference's free list (a slice)
    holds the cell 16 times (hived_core.h fl_append: first-occurrence positions + a duplicate count per segment, bounded
    by FL_DUP_SLACK); seed 1059 deletes a group twice through a stale cell pointer."""
    import fuzz_api
    monkeypatch.setenv("FUZZ_FILTERING", "1")
    assert fuzz_api.run_seed(emu_lib, oracle_lib, seed, 300) is None


def test_group_id_stays_with_its_name_while_an_erased_object_is_referenced(emu_lib, oracle_lib, monkeypatch):
    """include/hived.h "Id lifetime": in API-fuzz seed 2385 a PREEMPTING group is deleted by DeleteAllocatedPod while its
    Reserved leaves keep naming it — hived_get_group then reports NONE with `referenced` = 1 on both implementations, the
    mirror keeps name <-> id (no other group can be handed that id), and the run stays divergence-free."""
    import ctypes as C
    import fuzz_api
    from hivedscheduler_b200 import _cabi
    from hivedscheduler_b200 import algorithm as alg
    seen = {"emu": [], "oracle": []}
    orig = alg.HivedAlgorithm._release_group_if_gone

    def spy(self, name, gid):
        gi = _cabi.GroupInfo()
        self._lib.hived_get_group(self._ctx, gid, C.byref(gi))
        side = "emu" if self._lib is emu_lib else "oracle"
        if gi.state == _cabi.GROUP_NONE and gi.referenced:
            seen[side].append((name, gid))
        orig(self, name, gid)
        if gi.state == _cabi.GROUP_NONE and gi.referenced:
            assert self._groups.ids.get(name) == gid  # still interned

    monkeypatch.setattr(alg.HivedAlgorithm, "_release_group_if_gone", spy)
    assert fuzz_api.run_seed(emu_lib, oracle_lib, 2385, 300) is None
    assert seen["oracle"], "the scenario no longer occurs in this seed"
    assert set(seen["oracle"]) <= set(seen["emu"])  # the device's answer is the conservative one


def test_batched_mapping_leaves_a_cell_with_a_stale_binding_to_the_general_path(emu_lib, oracle_lib, monkeypatch):
    """Synthetic-cluster fuzz seed 1087 (names always re-used, Filtering-phase calls): a leaf that kept its binding below
    an UNBOUND cell (a gang lazy-preempted on a bad node keeps its bindings, hived_algorithm.go:1332-1335).  The
    reference's mapping skips such a child — here: finds no usable leaf and waits — while the whole-placement mapping
    (mapPlacementBatched) used to hand it out as "the j-th child" and answered with a preemption."""
    import fuzz_api
    monkeypatch.setenv("FUZZ_CLUSTER", "synthetic")
    monkeypatch.setenv("FUZZ_RENAME", "0.0")
    monkeypatch.setenv("FUZZ_FILTERING", "1")
    assert fuzz_api.run_seed(emu_lib, oracle_lib, 1087, 300) is None


@pytest.mark.parametrize("seed,filtering", [(3, False), (11, True)])
def test_api_fuzz_on_the_synthetic_five_level_cluster(emu_lib, oracle_lib, seed, filtering, monkeypatch):
    """tests/fuzz_api.py with FUZZ_CLUSTER=synthetic: the same random API calls on a small forest in the shape of
    BASELINE's C3-C5 (GPU / HALF / NODE / RACK / POD, VCs with POD-, RACK- and NODE-level cells, generated pod specs with
    1-2 members): buddy splits and merges over three levels above the node, preemption, bad nodes, opportunistic pods."""
    import fuzz_api
    monkeypatch.setenv("FUZZ_CLUSTER", "synthetic")
    if filtering:
        monkeypatch.setenv("FUZZ_FILTERING", "1")
    assert fuzz_api.run_seed(emu_lib, oracle_lib, seed, 300) is None
