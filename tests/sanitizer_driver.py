"""Driver for the compute-sanitizer runs: a short calm C3-shaped trace with `vcs` virtual
clusters (= CTAs of the VC-parallel launch) and a short C5-shaped churn trace (bad nodes: one CTA), replayed through
the C ABI on whatever library HIVED_CUDA_LIB / the default build provides; prints the result hashes.

    compute-sanitizer --tool memcheck  python tests/sanitizer_driver.py 8 1500
    compute-sanitizer --tool racecheck python tests/sanitizer_driver.py 16 1500
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from hivedscheduler_b200 import _cabi, config, trace  # noqa: E402
from conftest import run_trace  # noqa: E402


def calm_trace(vcs: int, gangs: int):
    if vcs == 8:
        return trace.trace_c3(n_gangs=gangs)
    racks = 4
    t = trace.trace_c3(n_gangs=gangs, n_vcs=vcs, vc_gpus=(16 + racks) * 32 * 8)
    t["config"] = config.config_c3(n_pods=vcs + (vcs * racks + 15) // 16, n_vcs=vcs, racks_per_vc=racks)
    return t


def main():
    vcs = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    gangs = int(sys.argv[2]) if len(sys.argv) > 2 else 1500
    lib = _cabi.load_library(os.environ["HIVED_ANY_LIB"]) if os.environ.get("HIVED_ANY_LIB") else _cabi.load_cuda_library()
    print("backend", lib.hived_backend().decode())
    t = calm_trace(vcs, gangs)
    h, _, st = run_trace(lib, t)
    print("calm vcs=%d gangs=%d events=%d hash=%016x binds=%d" % (vcs, gangs, len(t["events"]), h, st["bind_results"]))
    t5 = trace.trace_c5(n_steps=2, gangs_per_step=300)
    h5, _, st5 = run_trace(lib, t5)
    print("churn events=%d hash=%016x binds=%d" % (len(t5["events"]), h5, st5["bind_results"]))


if __name__ == "__main__":
    main()
