"""K threads, each with its own full-size C3 context and the same 100 000-gang trace (bench.py's flagship batch), each
thread running the whole trace as one hived_process_events call at the same time as the others.  Three ways, step by
step in alternation, every context rewound (hived_bench_restore_state) before every step:
  concurrent    contexts created with HIVED_OPT_CONCURRENT: each batch on its own stream and CTAs, no turn;
  taking turns  the same without the flag: the batches run one after another behind the library's device lock;
  joint         the K batches in one hived_process_events_many call from one thread (include/hived_multictx.h).
Decisions/s end to end: K x decisions per trace over the host-clock time from the common start to the last return.
Every context's parity hash must equal the oracle's, with and without the flag.  Prints one JSON line.  Needs the GPU.

    python profiles/micro/concurrent_batches.py [--ks 1,2,4,8,12,16] [--steps 2] [--warmup 1]
"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from hivedscheduler_b200 import _cabi, trace  # noqa: E402
from many_contexts import ORACLE_C3_HASH, bind, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8,12,16")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--gangs", type=int, default=100000)
    args = ap.parse_args()
    ks = [int(k) for k in args.ks.split(",")]
    K = max(ks)
    name, power = card()
    lib = bind(_cabi.load_cuda_library())
    t = trace.trace_c3(n_gangs=args.gangs)
    ev = np.ascontiguousarray(t["events"])
    n, n_dec, words = len(ev), int(t["decision"].sum()), trace.pool_words_for(t)
    evp = ev.ctypes.data_as(C.POINTER(_cabi.Event))

    def contexts(flags):
        out = []
        for _ in range(K):
            bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"],
                                    t["max_group_pods"], flags=flags)
            bc.set_all_nodes_healthy()
            lib.hived_bench_save_state(bc.ctx)
            out.append(bc)
        return out

    conc, plain = contexts(_cabi.OPT_CONCURRENT), contexts(0)
    bufs = [(np.zeros(n, dtype=trace.RESULT_DT), np.zeros(words, dtype=np.int32)) for _ in range(K)]
    batches = (_cabi.Batch * K)()
    for i, (res, pool) in enumerate(bufs):
        b = batches[i]
        b.ctx, b.events, b.n, b.pool_cap = plain[i].ctx, evp, n, words
        b.res, b.pool = res.ctypes.data_as(C.POINTER(_cabi.Result)), pool.ctypes.data_as(C.POINTER(C.c_int32))

    def threaded(bcs):
        """One thread per context, all released at once; seconds from the release to the last return."""
        k = len(bcs)
        go, done, rcs = threading.Barrier(k + 1), [0.0] * k, [None] * k

        def work(i):
            res, pool = bufs[i]
            go.wait()
            rcs[i] = lib.hived_process_events(bcs[i].ctx, evp, n, None, 0, res.ctypes.data_as(C.POINTER(_cabi.Result)),
                                              pool.ctypes.data_as(C.POINTER(C.c_int32)), words)
            done[i] = time.perf_counter()

        th = [threading.Thread(target=work, args=(i,)) for i in range(k)]
        for x in th:
            x.start()
        go.wait()
        t0 = time.perf_counter()
        for x in th:
            x.join()
        assert rcs == [0] * k, rcs
        return max(done) - t0

    def restore(bcs):
        for bc in bcs:
            lib.hived_bench_restore_state(bc.ctx)

    def run_conc(k):
        restore(conc[:k])
        return threaded(conc[:k])

    def run_turns(k):
        restore(plain[:k])
        return threaded(plain[:k])

    def run_joint(k):
        restore(plain[:k])
        t0 = time.perf_counter()
        assert lib.hived_process_events_many(batches, k) == 0
        dt = time.perf_counter() - t0
        assert all(batches[i].rc == 0 for i in range(k))
        return dt

    # parity: every context through the whole trace at once, the running hash on
    run_conc(K)
    run_turns(K)
    hashes = {"concurrent": ["%016x" % bc.result_hash() for bc in conc],
              "taking_turns": ["%016x" % bc.result_hash() for bc in plain]}
    ok = all(h == ORACLE_C3_HASH for hs in hashes.values() for h in hs)
    assert ok, hashes
    n_ctas = lib.hived_bench_num_ctas(conc[0].ctx)
    turns_before = [bc.turns() for bc in conc]
    for bc in conc + plain:  # the running parity hash is off while timing, as in bench.py
        lib.hived_bench_set_result_hash(bc.ctx, 0)

    ways = (("concurrent", run_conc), ("taking_turns", run_turns), ("joint", run_joint))
    rows = {}
    for k in ks:
        for _ in range(args.warmup):
            for _, fn in ways:
                fn(k)
        secs = {w: [] for w, _ in ways}
        for _ in range(args.steps):  # alternating
            for w, fn in ways:
                secs[w].append(fn(k))
        row = {w: {"decisions_per_s": k * n_dec * args.steps / sum(s), "s": [round(x, 5) for x in s]}
               for w, s in secs.items()}
        row["concurrent_over_turns"] = sum(secs["taking_turns"]) / sum(secs["concurrent"])
        row["concurrent_over_joint"] = sum(secs["joint"]) / sum(secs["concurrent"])
        rows[str(k)] = row
    # restores take turns (a rewind hook); the batches themselves did not
    batch_turns = [bc.turns() - b - (args.warmup + args.steps) * sum(1 for k in ks if k > i)
                   for i, (bc, b) in enumerate(zip(conc, turns_before))]
    line = {"what": "K threads, one full-size C3 context each, the whole trace per hived_process_events call: "
                    "concurrent contexts vs taking turns vs one joint call",
            "card": name, "power_limit": power, "decisions_per_context": n_dec, "ctas_per_context": n_ctas,
            "steps": args.steps, "warmup": args.warmup, "host_cpus": os.cpu_count(),
            "parity": {"result_hash": hashes["concurrent"][0], "all_contexts_match_oracle": ok,
                       "per_context": hashes},
            "turns_taken_by_concurrent_batches": sum(batch_turns), "by_k": rows}
    print(json.dumps(line))
    for bc in conc + plain:
        bc.close()


if __name__ == "__main__":
    main()
