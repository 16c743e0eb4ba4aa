"""What a clone of a live scheduler context costs (hived_clone, include/hived_clone.h), and what K what-if clones gain
from one joint launch.

The source is a full-size C3 context (bench.py's flagship cluster) after the trace's first 50 000 gangs.  Measured, host
clock around calls that end in a device synchronisation:
  create          hived_create of an empty C3 context and its node-health batch (what a clone replaces);
  clone           hived_clone on the source's device, ordinary and HIVED_OPT_CONCURRENT, and to a second device when
                  there is one;
  what-if         K = 1, 4, 16 clones, each running its own 2 000-gang slice of the rest of the trace: one
                  hived_process_events_many call (joint) against K hived_process_events calls one after another
                  (sequential), alternating; clone creation not included.  Every clone's joint results must equal its
                  sequential results.
Medians over --reps repetitions (and the minimum).  Prints one JSON line.  Needs the GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from hivedscheduler_b200 import _cabi, trace  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()
    name, power = [s.strip() for s in out[0].split(",")]
    return name, power, len(out)


def ms(xs):
    return {"median_ms": round(statistics.median(xs) * 1e3, 3), "min_ms": round(min(xs) * 1e3, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gangs", type=int, default=50000, help="gangs the source has run when it is cloned")
    ap.add_argument("--suffix", type=int, default=2000, help="gangs of each what-if clone's slice")
    ap.add_argument("--ks", default="1,4,16")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    ks = [int(k) for k in args.ks.split(",")]
    name, power, n_gpus = card()
    lib = _cabi.load_cuda_library()
    t = trace.trace_c3()
    ev = np.ascontiguousarray(t["events"])
    gang_at = np.cumsum(t["decision"])  # gangs decided up to and including each event

    def cut(g):
        return int(np.searchsorted(gang_at, g))  # first event after the first g gangs

    def make():
        bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
        bc.set_all_nodes_healthy()
        return bc

    create = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        bc = make()
        create.append(time.perf_counter() - t0)
        bc.close()
    src = make()
    head = ev[:cut(args.gangs)]
    src.process(head, 3 * 64 * len(head) + 4096)

    def clone_times(device, flags):
        out = []
        for _ in range(args.reps + 1):  # the first one warms up the device's allocator and streams
            t0 = time.perf_counter()
            c = src.clone(device=device, flags=flags)
            out.append(time.perf_counter() - t0)
            c.close()
        return ms(out[1:])

    result = {"metric": "clone_cost", "gpu": name, "power_limit": power, "source_gangs": args.gangs,
              "create_c3": ms(create),
              "clone_same_device": clone_times(-1, 0),
              "clone_same_device_concurrent": clone_times(-1, _cabi.OPT_CONCURRENT),
              "clone_second_device": clone_times(1, 0) if n_gpus > 1 else "one GPU",
              "clone_second_device_concurrent": clone_times(1, _cabi.OPT_CONCURRENT) if n_gpus > 1 else "one GPU"}

    at = cut(args.gangs)
    slices = []
    for i in range(max(ks)):
        lo, hi = cut(args.gangs + i * args.suffix), cut(args.gangs + (i + 1) * args.suffix)
        assert hi > lo and at <= lo, "the trace is too short for %d slices" % max(ks)
        slices.append(np.ascontiguousarray(ev[lo:hi]))
    words = [3 * 64 * len(s) + 4096 for s in slices]
    whatif = {}
    for k in ks:
        joint, seq = [], []
        for _ in range(args.reps + 1):
            clones = [src.clone() for _ in range(k)]
            t0 = time.perf_counter()
            got = trace.process_many(clones, slices[:k], words[:k])
            dt = time.perf_counter() - t0
            joint.append(dt)
            assert all(g[0] == 0 for g in got)
            for c in clones:
                c.close()
            clones = [src.clone() for _ in range(k)]
            t0 = time.perf_counter()
            alone = [c.process(s, w) for c, s, w in zip(clones, slices, words)]
            seq.append(time.perf_counter() - t0)
            for (_, res, pool), (res2, pool2) in zip(got, alone):
                assert res.tobytes() == res2.tobytes() and pool.tobytes() == pool2.tobytes()
            for c in clones:
                c.close()
        j, s = ms(joint[1:]), ms(seq[1:])
        whatif[str(k)] = {"joint": j, "sequential": s, "speedup": round(s["median_ms"] / j["median_ms"], 2)}
    result["whatif_suffix_gangs"] = args.suffix
    result["whatif"] = whatif
    src.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
