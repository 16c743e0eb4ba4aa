"""K full-size C3 contexts on one GPU: their batches in one joint launch (hived_process_events_many,
include/hived_multictx.h) against the same K batches one after another through the single-context path.

Every context holds its own copy of the C3 state and gets the same trace (bench.py's flagship batch).  Two legs, each
alternating joint and sequential runs step by step, the state rewound (hived_bench_restore_state) between steps:
  kernel-only  staged batches; joint: hived_bench_run_staged_many, its CUDA-event time; sequential: hived_bench_run_staged
               per context, the sum of their CUDA-event times; L2 flushed before every launch;
  end-to-end   joint: one hived_process_events_many call; sequential: K hived_process_events calls; host clock.
K = 1 joint against K = 1 sequential is the price of the joint build's indexed state pointers (every fetch of a state
pointer is a constant load indexed by blockIdx.y, where the single-context kernel has a constant-bank operand).
Every context's parity hash must equal the oracle's.  Prints one JSON line.  Needs the GPU."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from hivedscheduler_b200 import _cabi, trace  # noqa: E402

ORACLE_C3_HASH = "e3becf53c2d32f79"  # the oracle on C3: bench.py's parity witness


def bind(lib):
    P = C.c_void_p
    for name, res, args in [
            ("hived_bench_save_state", C.c_int, [P]), ("hived_bench_restore_state", C.c_int, [P]),
            ("hived_bench_stage_events", C.c_int, [P, C.POINTER(_cabi.Event), C.c_int32, C.c_int64]),
            ("hived_bench_run_staged", C.c_int, [P]), ("hived_bench_run_staged_many", C.c_int, [C.POINTER(P), C.c_int32]),
            ("hived_bench_last_kernel_ms", C.c_double, [P]), ("hived_bench_flush_l2", C.c_int, [P]),
            ("hived_bench_set_result_hash", C.c_int, [P, C.c_int]), ("hived_bench_num_ctas", C.c_int, [P])]:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return _cabi.bind_many(lib)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8,16")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--gangs", type=int, default=100000)
    args = ap.parse_args()
    ks = [int(k) for k in args.ks.split(",")]
    name, power = card()
    lib = bind(_cabi.load_cuda_library())
    t = trace.trace_c3(n_gangs=args.gangs)
    ev = np.ascontiguousarray(t["events"])
    n, n_dec, words = len(ev), int(t["decision"].sum()), trace.pool_words_for(t)
    evp = ev.ctypes.data_as(C.POINTER(_cabi.Event))
    K = max(ks)
    bcs = []
    for _ in range(K):
        bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
        bc.set_all_nodes_healthy()
        lib.hived_bench_save_state(bc.ctx)
        bcs.append(bc)
    ctxs = [bc.ctx for bc in bcs]
    outs = [(np.zeros(n, dtype=trace.RESULT_DT), np.zeros(words, dtype=np.int32)) for _ in range(K)]
    batches = (_cabi.Batch * K)()
    for i, (res, pool) in enumerate(outs):
        b = batches[i]
        b.ctx, b.events, b.n, b.pool_cap = ctxs[i], evp, n, words
        b.res, b.pool = res.ctypes.data_as(C.POINTER(_cabi.Result)), pool.ctypes.data_as(C.POINTER(C.c_int32))

    def restore(k):
        for c in ctxs[:k]:
            lib.hived_bench_restore_state(c)

    # parity: every context through one joint call, the hash on
    restore(K)
    assert lib.hived_process_events_many(batches, K) == 0
    assert [batches[i].rc for i in range(K)] == [0] * K
    hashes = ["%016x" % bc.result_hash() for bc in bcs]
    assert hashes == [ORACLE_C3_HASH] * K, hashes
    n_ctas = lib.hived_bench_num_ctas(ctxs[0])

    # kernel-only leg
    for c in ctxs:
        assert lib.hived_bench_stage_events(c, evp, n, words) == 0
    carr = (C.c_void_p * K)(*ctxs)

    def joint_kernel(k):
        restore(k)
        lib.hived_bench_flush_l2(ctxs[0])
        assert lib.hived_bench_run_staged_many(carr, k) == 0
        return lib.hived_bench_last_kernel_ms(ctxs[0]) / 1e3

    def seq_kernel(k):
        restore(k)
        s = 0.0
        for c in ctxs[:k]:
            lib.hived_bench_flush_l2(c)
            assert lib.hived_bench_run_staged(c) == 0
            s += lib.hived_bench_last_kernel_ms(c) / 1e3
        return s

    # end-to-end leg (the running parity hash is off while timing, as in bench.py)
    for c in ctxs:
        lib.hived_bench_set_result_hash(c, 0)
    res0, pool0 = outs[0]

    def joint_e2e(k):
        restore(k)
        t0 = time.perf_counter()
        assert lib.hived_process_events_many(batches, k) == 0
        dt = time.perf_counter() - t0
        assert all(batches[i].rc == 0 for i in range(k))
        return dt

    def seq_e2e(k):
        restore(k)
        t0 = time.perf_counter()
        for c in ctxs[:k]:
            assert lib.hived_process_events(c, evp, n, None, 0, res0.ctypes.data_as(C.POINTER(_cabi.Result)),
                                            pool0.ctypes.data_as(C.POINTER(C.c_int32)), words) == 0
        return time.perf_counter() - t0

    rows = {}
    for k in ks:
        row = {}
        for leg, (jf, sf) in (("kernel", (joint_kernel, seq_kernel)), ("e2e", (joint_e2e, seq_e2e))):
            for _ in range(args.warmup):
                jf(k), sf(k)
            js, ss = [], []
            for _ in range(args.steps):  # alternating
                js.append(jf(k))
                ss.append(sf(k))
            row[leg] = {"joint_decisions_per_s": k * n_dec * args.steps / sum(js),
                        "sequential_decisions_per_s": k * n_dec * args.steps / sum(ss),
                        "joint_over_sequential": sum(ss) / sum(js),
                        "joint_s": [round(x, 5) for x in js], "sequential_s": [round(x, 5) for x in ss]}
        rows[str(k)] = row
    line = {"what": "K full-size C3 contexts, one joint launch vs one after another", "card": name, "power_limit": power,
            "decisions_per_context": n_dec, "ctas_per_context": n_ctas, "steps": args.steps, "warmup": args.warmup,
            "parity": {"result_hash": hashes[0], "all_contexts_match_oracle": True}, "by_k": rows}
    if "1" in rows:
        line["k1_joint_over_single_kernel_time"] = 1.0 / rows["1"]["kernel"]["joint_over_sequential"]
    print(json.dumps(line))
    for bc in bcs:
        bc.close()


if __name__ == "__main__":
    main()
