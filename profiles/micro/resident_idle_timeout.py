"""How long the resident per-call kernel (hived_serve_kernel) stays on the GPU without a request.

One call through hived_process_events(n = 1), an idle gap of d ms on the host, then a second call: the second call
needed a relaunch exactly when the kernel had already left (hived_bench_kernel_launches grows).  Prints, per gap, the
share of second calls that relaunched it, over `reps` tries.

    python profiles/micro/resident_idle_timeout.py [reps]
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from hivedscheduler_b200 import _cabi, trace  # noqa: E402

GAPS_MS = (0.5, 1, 1.5, 2, 2.5, 3, 4, 6, 10)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    lib = _cabi.load_cuda_library()
    bench.bind_bench_hooks(lib)
    t = trace.trace_c3(n_gangs=4000)
    bc = trace.BatchContext(lib, t["config"], t["n_groups"], t["n_pods"], t["max_group_leaves"], t["max_group_pods"])
    bc.set_all_nodes_healthy()
    ev, k = t["events"], 0

    def call():
        nonlocal k
        bc.process(ev[k:k + 1], 3 * 64 + 4096)
        k += 1

    call()
    share = {}
    for gap_ms in GAPS_MS:
        relaunched = 0
        for _ in range(reps):
            call()
            t0 = time.perf_counter()
            while time.perf_counter() - t0 < gap_ms / 1e3:
                pass
            n0 = lib.hived_bench_kernel_launches(bc.ctx)
            call()
            relaunched += lib.hived_bench_kernel_launches(bc.ctx) > n0
        share[str(gap_ms)] = relaunched / reps
    bc.close()
    print(json.dumps({"calls": k, "relaunch_share_by_idle_gap_ms": share}))


if __name__ == "__main__":
    main()
