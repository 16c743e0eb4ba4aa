"""Driver of profiles/micro/concurrent_calls.c: writes the full-size C3 spec and builds the C program in a temporary
directory, runs it against the built libhived_cuda.so and prints its JSON line with the card's name and power limit
added.  Needs the GPU.

    python profiles/micro/concurrent_calls.py [--ks 1,2,4,8,16] [--calls 2000] [--reps 2]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from hivedscheduler_b200 import config  # noqa: E402

CSRC = os.path.join(ROOT, "hivedscheduler_b200", "csrc")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8,16")
    ap.add_argument("--calls", type=int, default=2000, help="rounds (schedule + delete) per thread and run")
    ap.add_argument("--reps", type=int, default=2, help="runs with and without the flag, alternating, per K")
    args = ap.parse_args()
    name, power = card()
    with tempfile.TemporaryDirectory(prefix="hived_concurrent_") as tmp:
        spec = os.path.join(tmp, "c3.spec")
        with open(spec, "w") as f:
            f.write(config.to_spec_text(config.config_c3()))
        exe = os.path.join(tmp, "concurrent_calls")
        subprocess.check_call(["gcc", "-O2", "-pthread", "-I", os.path.join(ROOT, "include"), "-o", exe,
                               os.path.join(ROOT, "profiles", "micro", "concurrent_calls.c"), "-L", CSRC, "-lhived_cuda",
                               "-Wl,-rpath," + CSRC])
        out = subprocess.run([exe, spec, args.ks, str(args.calls), str(args.reps)], capture_output=True, text=True)
    sys.stderr.write(out.stderr)
    line = json.loads(out.stdout.strip().splitlines()[-1])
    line.update({"card": name, "power_limit": power})
    print(json.dumps(line))
    return out.returncode


if __name__ == "__main__":
    sys.exit(main())
