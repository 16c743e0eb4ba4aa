"""Parity tests proper: the CUDA path (libhived_cuda.so, through the C ABI) against the oracle on the
same seeded inputs, against the reference's golden vectors, and — at BASELINE size — against the
committed oracle checkpoints plus size-independent properties.  Bit-exact: all work is integer."""
import json
import os

import numpy as np
import pytest

from conftest import run_trace
from golden_scenario import Scenario
from hivedscheduler_b200 import _cabi, trace
from test_device_program_emu import small_c3

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def test_cuda_backend_is_the_one_loaded(cuda_lib):
    assert cuda_lib.hived_backend() == b"cuda-sm90a"


def test_cuda_reproduces_reference_golden_vectors(cuda_lib, oracle_lib):
    sc = Scenario(cuda_lib)
    assert sc.run() == []
    so = Scenario(oracle_lib)
    assert so.run() == []
    assert sc.decisions == so.decisions


@pytest.mark.parametrize("name", ["C1", "C2", "C3-small", "multi-member", "heterogeneous", "suggested-nodes", "bad-requests"])
def test_cuda_matches_oracle_on_trace(cuda_lib, oracle_lib, name):
    t = {"C1": trace.trace_c1, "C2": trace.trace_c2, "C3-small": small_c3, "multi-member": trace.trace_multi_member,
         "heterogeneous": trace.trace_heterogeneous, "suggested-nodes": trace.trace_suggested_nodes,
         "bad-requests": trace.trace_bad_requests}[name]()
    snaps = []
    hc, rc, sc = run_trace(cuda_lib, t, chunks=2, snapshots=snaps)
    ho, ro, so = run_trace(oracle_lib, t, chunks=2, snapshots=snaps)
    assert hc == ho
    assert sc == so
    assert snaps[0] == snaps[1]  # cell state after the trace, incl. the ancestors repaired after VC-parallel batches
    for (a, pa), (b, pb) in zip(rc, ro):
        assert a.tobytes() == b.tobytes()
        n = int((a["leaf_off"] + 3 * a["n_leaves"]).max()) if len(a) else 0
        assert pa[:n].tobytes() == pb[:n].tobytes()


def _replay_occupancy(t, results):
    """Size-independent properties of a bind-only trace: every GPU is held by at most one alive gang,
    a pod's GPUs sit on one node, and later pods of a gang repeat the gang's stored placement."""
    ev = t["events"]
    owner = {}
    placement = {}
    k = 0
    for res, pool in results:
        for i in range(len(res)):
            e = ev[k]
            k += 1
            g = int(e["spec"]["group"])
            if e["type"] == _cabi.EV_SCHEDULE:
                r = res[i]
                assert r["error"] == 0
                if r["kind"] != _cabi.KIND_BIND:
                    continue
                leaves = pool[r["leaf_off"]:r["leaf_off"] + 3 * r["n_leaves"]].reshape(-1, 3)
                mine = pool[r["this_off"]:r["this_off"] + 3 * r["this_n"]].reshape(-1, 3)
                assert (mine[:, 0] == r["node"]).all()
                key = [(int(a), int(b)) for a, b, _ in leaves]
                if g in placement:
                    assert placement[g][0] == key
                    placement[g][1] += 1
                else:
                    for gpu in key:
                        assert gpu not in owner, "GPU %r double-allocated" % (gpu,)
                        owner[gpu] = g
                    placement[g] = [key, 1]
            elif e["type"] == _cabi.EV_DELETE_ALLOCATED and g in placement:
                placement[g][1] -= 1
                if placement[g][1] == 0:
                    for gpu in placement[g][0]:
                        del owner[gpu]
                    del placement[g]
    return len(owner)


def test_cuda_full_size_c3_against_oracle_checkpoints(cuda_lib):
    """BASELINE size: 64k-GPU tree, 100k gangs.  The oracle needs ~20 minutes for this trace, so its
    parity hashes per chunk are committed in tests/golden/trace_hashes.json (make_trace_hashes.py)."""
    t = trace.trace_c3()
    golden = json.load(open(os.path.join(HERE, "golden", "trace_hashes.json")))["C3"]
    assert golden["n_events"] == len(t["events"])
    bc = trace.BatchContext(cuda_lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
    bc.set_all_nodes_healthy()
    start, results = 0, []
    for cp in golden["checkpoints"]:
        chunk = t["events"][start:cp["events"]]
        res, pool = bc.process(chunk, 3 * 64 * len(chunk) + 4096)
        sched = chunk["type"] == _cabi.EV_SCHEDULE
        assert "%016x" % bc.result_hash() == cp["hash"], "diverged from the oracle before event %d" % cp["events"]
        assert int((res["kind"][sched] == 1).sum()) == cp["binds"]
        results.append((res, pool))
        start = cp["events"]
    stats = bc.stats()
    for key in ("view_nodes_scanned", "leaves_committed", "free_cells_scanned", "pods_placed", "algorithmic_bytes"):
        assert stats[key] == golden["stats"][key]
    in_use = _replay_occupancy(t, results)
    assert 0 < in_use <= 8 * 7168
    bc.close()


def test_schedule_is_idempotent_without_commit(cuda_lib):
    """Schedule alone does not allocate (hived_algorithm.go:180-224): asking twice gives the same answer."""
    from hivedscheduler_b200 import algorithm as alg
    from hivedscheduler_b200.config import config_c1
    h = alg.HivedAlgorithm(config_c1(), lib=cuda_lib, max_groups=16, max_pods=16, max_group_leaves=8, max_group_pods=8)
    for n in h.node_names:
        h.setHealthyNode(n)
    pod = alg.Pod("p0", "ns")
    pod.annotations[alg.ANNOTATION_POD_SCHEDULING_SPEC] = alg.to_yaml(
        {"virtualCluster": "default", "priority": 0, "leafCellType": "K80", "leafCellNumber": 2})
    a = h.Schedule(pod, h.node_names, alg.FILTERING_PHASE).pod_bind_info
    b = h.Schedule(pod, h.node_names, alg.FILTERING_PHASE).pod_bind_info
    assert a == b and a["leafCellIsolation"] == [0, 1]
    h.close()


def test_cuda_matches_oracle_under_churn_c5(cuda_lib, oracle_lib):
    """C5 shape: node-health flips (single-CTA path: health events are global) — rows a11, a18."""
    from test_device_program_emu import small_cluster
    t = trace.trace_c5(n_steps=4, gangs_per_step=300, n_nodes=4 * 16 * 32, n_vcs=2, vc_gpus=(16 + 6) * 32 * 8,
                       config=small_cluster())
    hc, rc, sc = run_trace(cuda_lib, t, chunks=2)
    ho, ro, so = run_trace(oracle_lib, t, chunks=2)
    assert hc == ho and sc == so
    for (a, pa), (b, pb) in zip(rc, ro):
        assert a.tobytes() == b.tobytes()


def test_cuda_matches_oracle_with_preemption_c4(cuda_lib, oracle_lib):
    """C4 shape: priorities 0/1/2 + opportunistic pods, call-by-call kube-scheduler emulation — rows a12, a19."""
    from test_device_program_emu import small_cluster
    kw = dict(config=small_cluster(), n_gangs=1200, n_vcs=2, vc_gpus=(16 + 6) * 32 * 8, total_gpus=4 * 16 * 32 * 8)
    hc, lc, sc = trace.run_c4_interactive(cuda_lib, **kw)
    ho, lo, so = trace.run_c4_interactive(oracle_lib, **kw)
    assert lc == lo
    assert hc == ho and sc == so


def test_vc_parallel_equals_single_cta(cuda_lib):
    """The VC-parallel execution (one CTA per group of VCs) must give the bytes of the sequential one."""
    import subprocess, sys
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from hivedscheduler_b200 import _cabi, trace\n"
            "from conftest import run_trace\n"
            "from test_device_program_emu import small_c3\n"
            "import hashlib\n"
            "h, res, st = run_trace(_cabi.load_cuda_library(), small_c3(4000))\n"
            "m = hashlib.sha256()\n"
            "for r, p in res:\n"
            "    m.update(r.tobytes()); n = int((r['leaf_off'] + 3 * r['n_leaves']).max()); m.update(p[:n].tobytes())\n"
            "print('%%016x %%s %%s' %% (h, m.hexdigest(), sorted(st.items())))\n") % (os.path.dirname(HERE), HERE)
    outs = []
    for ncta in ("1", "2", "16"):
        env = dict(os.environ, HIVED_NCTA=ncta)
        outs.append(subprocess.check_output([sys.executable, "-c", code], env=env).decode().strip().splitlines()[-1])
    assert outs[0] == outs[1] == outs[2], outs


def test_cuda_matches_oracle_with_lazy_preemption(cuda_lib, oracle_lib):
    """C4's call-by-call harness, VCs left to fill up, lazyPreemptionEnable on half of the guaranteed gangs: lazy
    preemption, its revert on a failed mapping, and downgraded gangs being preempted later — rows a7, a19."""
    from test_device_program_emu import small_cluster
    kw = dict(config=small_cluster(), n_gangs=4500, n_vcs=2, vc_gpus=(16 + 6) * 32 * 8, total_gpus=4 * 16 * 32 * 8,
              lazy_percent=50, load=3.0)
    hc, lc, sc = trace.run_c4_interactive(cuda_lib, **kw)
    ho, lo, so = trace.run_c4_interactive(oracle_lib, **kw)
    assert lc == lo
    assert hc == ho and sc == so
    assert so["lazy_preempted_groups"] > 0


def test_cuda_full_size_c5_against_oracle_checkpoints(cuda_lib):
    """BASELINE config 5 at full size (64k GPUs, 10 % of the nodes flipping per step, 20 000 gangs): the oracle's parity
    hash after every tenth of the trace and its work counters are committed (tests/golden/make_trace_hashes.py C5)."""
    t = trace.trace_c5()
    golden = json.load(open(os.path.join(HERE, "golden", "trace_hashes.json")))["C5"]
    assert golden["n_events"] == len(t["events"])
    bc = trace.BatchContext(cuda_lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
    bc.set_all_nodes_healthy()
    start = 0
    for cp in golden["checkpoints"]:
        chunk = t["events"][start:cp["events"]]
        res, pool = bc.process(chunk, 3 * 64 * len(chunk) + 4096)
        sched = chunk["type"] == _cabi.EV_SCHEDULE
        assert "%016x" % bc.result_hash() == cp["hash"], "diverged from the oracle before event %d" % cp["events"]
        assert int((res["kind"][sched] == 1).sum()) == cp["binds"] and int((res["kind"][sched] == 0).sum()) == cp["waits"]
        start = cp["events"]
    assert bc.stats() == golden["stats"]
    bc.close()


def test_cuda_full_size_c4_against_oracle(cuda_lib):
    """BASELINE config 4 at full size (64k GPUs, 50 000 guaranteed + 50 000 opportunistic gangs with preemption), played
    call by call like kube-scheduler would: final parity hash, sha256 of the decision log and the work counters of the
    oracle's run are committed (tests/golden/make_trace_hashes.py C4, about an hour of oracle time)."""
    golden = json.load(open(os.path.join(HERE, "golden", "trace_hashes.json"))).get("C4")
    if golden is None:
        pytest.skip("tests/golden/trace_hashes.json has no C4 entry")
    sys_path = os.path.join(HERE, "golden")
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_trace_hashes", os.path.join(sys_path, "make_trace_hashes.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    h, log, stats = trace.run_c4_interactive(cuda_lib, **gen.c4_kwargs(golden["n_gangs"]))
    assert len(log) == golden["log_entries"]
    assert gen.log_digest(log) == golden["log_sha256"]
    assert "%016x" % h == golden["hash"]
    assert stats == golden["stats"]


@pytest.mark.parametrize("seed", [16, 31, 160, 553, 775, 2385, 3, 5, 8])
def test_cuda_api_fuzz_seeds(cuda_lib, oracle_lib, seed):
    """API-level fuzz (tests/fuzz_api.py) on the GPU through the per-call path: results, every cell and every view order
    after every call; 16 and 31 are the re-created-group seeds (ghost records), 160 / 553 nil dereferences of the
    reference (platform errors on both sides), 775 a pod deleted through another pod's slot, 2385 a PREEMPTING group
    deleted by DeleteAllocatedPod whose Reserved leaves keep naming it (a ghost reached through p_resv later; the id stays
    with the name while hived_get_group reports `referenced`)."""
    import fuzz_api
    assert fuzz_api.run_seed(cuda_lib, oracle_lib, seed, 300) is None


@pytest.mark.parametrize("seed", [7, 782, 1059])
def test_cuda_api_fuzz_with_filtering_phase_calls(cuda_lib, oracle_lib, seed, monkeypatch):
    """The Filtering-phase form of the fuzz on the GPU: 7 = a Reserved cell without a reserving group (platform error on
    both sides), 782 = a free-list segment holding one cell 16 times (hived_core.h fl_append), 1059 = a group deleted
    twice through a stale cell pointer."""
    import fuzz_api
    monkeypatch.setenv("FUZZ_FILTERING", "1")
    assert fuzz_api.run_seed(cuda_lib, oracle_lib, seed, 300) is None


def test_cuda_api_fuzz_on_the_synthetic_cluster(cuda_lib, oracle_lib, monkeypatch):
    """Synthetic-cluster fuzz seed 1087 on the GPU (a stale binding below an unbound cell: mapPlacementBatched hands the
    placement to the general mapping, which finds no usable leaf like the reference)."""
    import fuzz_api
    monkeypatch.setenv("FUZZ_CLUSTER", "synthetic")
    monkeypatch.setenv("FUZZ_RENAME", "0.0")
    monkeypatch.setenv("FUZZ_FILTERING", "1")
    assert fuzz_api.run_seed(cuda_lib, oracle_lib, 1087, 300) is None


def test_contexts_of_several_threads_take_turns_on_one_device(cuda_lib, oracle_lib):
    """Three host threads, each driving ITS OWN context through the per-call path (API fuzz vs the oracle, every cell
    compared after every call): the contexts share the device's constant bank (one Dev loaded at a time,
    hived_cuda.cu ensureDevLoaded) and each has a resident per-call kernel that the next owner must stop first."""
    import threading
    import fuzz_api
    out = {}

    def work(seed):
        try:
            out[seed] = fuzz_api.run_seed(cuda_lib, oracle_lib, seed, 150)
        except BaseException as e:  # noqa
            out[seed] = "exception: %r" % (e,)

    threads = [threading.Thread(target=work, args=(s,)) for s in (21, 22, 23)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    assert out == {21: None, 22: None, 23: None}


def test_cuda_full_size_c4_compiled_player(cuda_lib):
    """The same full-size C4 run driven by compiled code (tests/harness/c4_player.cpp: no interpreter between the calls,
    a gang's pod deletions as one batch): same hash, log and counters as the oracle's committed run."""
    golden = json.load(open(os.path.join(HERE, "golden", "trace_hashes.json"))).get("C4")
    if golden is None:
        pytest.skip("tests/golden/trace_hashes.json has no C4 entry")
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_trace_hashes", os.path.join(HERE, "golden", "make_trace_hashes.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    h, log, stats, tm = trace.run_c4_compiled(cuda_lib, **gen.c4_kwargs(golden["n_gangs"]))
    assert len(log) == golden["log_entries"]
    assert gen.log_digest(log) == golden["log_sha256"]
    assert "%016x" % h == golden["hash"]
    assert stats == golden["stats"]


def test_c_driver_through_the_abi(cuda_lib, tmp_path):
    """Schedule -> AddAllocatedPod -> DeleteAllocatedPod on the GPU from plain C (tests/c/test_cabi_gpu.c): the
    boundary as a cgo shim sees it, without Python in between."""
    import subprocess
    from hivedscheduler_b200.config import config_c1, to_spec_text
    root = os.path.dirname(HERE)
    csrc = os.path.join(root, "hivedscheduler_b200", "csrc")
    exe = str(tmp_path / "test_cabi_gpu")
    subprocess.check_call(["gcc", "-O1", "-std=c99", "-I", os.path.join(root, "include"), "-o", exe,
                           os.path.join(HERE, "c", "test_cabi_gpu.c"), "-L", csrc, "-lhived_cuda", "-Wl,-rpath," + csrc])
    spec = tmp_path / "c1.spec"
    spec.write_text(to_spec_text(config_c1()))
    out = subprocess.run([exe, str(spec)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "test_cabi_gpu: ok" in out.stdout


@pytest.mark.parametrize("world,window", [(1, 0), (2, 0), (4, 0), (8, 0), (2, 1024), (4, 256), (8, 1024)])
def test_vc_partition_over_ranks_matches_single_gpu_run(cuda_lib, world, window):
    """SURVEY.md section 8 row (e): the C3 cluster's 8 VCs partitioned over `world` ranks (here: `world` contexts on
    one GPU, the two collectives done by hand — the protocol of hivedscheduler_b200/dist.py without the process
    group); the chain hash over the merged results equals the hash of the ordinary single-context run.  window > 0: the
    horizon form (hived_mg_run_window), what dist.run_partitioned drives; several contexts of one process also take
    turns on the device's constant bank (ensureDevLoaded)."""
    import torch
    from test_multigpu_partition import simulate
    t = trace.trace_c3(n_gangs=6000)
    h1, _, _ = run_trace(cuda_lib, t)

    def alloc(nbytes):
        b = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        return b, b.data_ptr()

    h, rounds = simulate(cuda_lib, t, world, alloc=alloc, window=window)
    assert h == h1
    assert rounds >= 8


def test_frontend_batch_drain_on_gpu(cuda_lib, oracle_lib):
    """SURVEY.md section 8 row f4 on the GPU: queued filter calls and pod deletions answered from ONE
    hived_process_events batch give every pod the node and GPUs the reference-shaped mirror (one Schedule +
    AddAllocatedPod at a time, on the CPU checker) gives it; request bodies go through the ingest helpers (f1)."""
    import json as _json
    from hivedscheduler_b200 import frontend as fe_mod
    import test_frontend as tf
    bc = trace.BatchContext(cuda_lib, tf.cluster(), tf.MAXG, tf.MAXP, 64, 8)
    bc.set_all_nodes_healthy()
    f = fe_mod.FrontEnd(cuda_lib, bc.ctx, tf.MAXG, tf.MAXP)
    pods = tf.workload(120)
    deletes = {10: "uid-3", 25: "uid-7", 40: "uid-g4-1", 90: "uid-51"}
    want = tf.mirror_answers(oracle_lib, pods, deletes)
    names = [cuda_lib.hived_node_name(bc.ctx, i).decode() for i in range(bc.n_nodes)]
    body = _json.dumps(names).encode()  # kube-scheduler found every node feasible
    for uid, key, ann in pods:
        assert f.add_unbound_pod(uid, key, ann) == 0
    tickets = {}
    for k, (uid, key, ann) in enumerate(pods):
        tickets[uid] = f.enqueue_filter(uid, body)
        if k in deletes:
            f.delete_pod(deletes[k])
    assert f.drain() == 0
    got = {uid: tf.fe_answer(f, cuda_lib, bc, f.take(t)) for uid, t in tickets.items()}
    assert got == want
    st = f.stats()
    assert st["drains"] <= 1 + len(deletes) and st["events"] == len(pods) + len(deletes)
    # and one at a time (the per-call path of the engine) from a fresh scheduler: the same answers
    f.close()
    bc.close()
    bc = trace.BatchContext(cuda_lib, tf.cluster(), tf.MAXG, tf.MAXP, 64, 8)
    bc.set_all_nodes_healthy()
    f = fe_mod.FrontEnd(cuda_lib, bc.ctx, tf.MAXG, tf.MAXP)
    got = {}
    for k, (uid, key, ann) in enumerate(pods):
        f.add_unbound_pod(uid, key, ann)
        got[uid] = tf.fe_answer(f, cuda_lib, bc, f.filter(uid, body))
        if k in deletes:
            f.delete_pod(deletes[k])
    assert got == want
    f.close()
    bc.close()


def test_shared_section_protocol_litmus():
    """The message-passing protocol of the ordered shared sections (plain stores, fence, volatile progress word /
    spin, fence, plain loads through a warm L1) with the library's own primitives: tests/litmus/shared_enter_litmus.cu,
    compiled by build()."""
    import subprocess
    import __graft_entry__ as g
    exe = g.build_litmus()
    out = subprocess.run([exe, "20000", "4096"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "shared_enter_litmus: ok" in out.stdout
