#!/usr/bin/env python
"""SASS opcode summary of the built product library (cuobjdump -sass), per kernel.
usage: python profiles/scripts/sass_summary.py [path/to/libhived_cuda.so] > profiles/<round>_sass_summary.md"""
import collections
import re
import subprocess
import sys

lib = sys.argv[1] if len(sys.argv) > 1 else "hivedscheduler_b200/csrc/libhived_cuda.so"
txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
fn = None
ops = {}
ins = re.compile(r"^\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)")
for line in txt.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        fn = subprocess.run(["c++filt", "-p", m.group(1)], capture_output=True, text=True).stdout.strip()
        ops[fn] = collections.Counter()
        continue
    m = ins.match(line)
    if m and fn:
        ops[fn][m.group(1)] += 1
GROUPS = [
    ("local memory (spills / device stack)", ("LDL", "STL")),
    ("calls", ("CALL", "RET", "BRX", "JMX")),
    ("global loads", ("LDG", "LD.")),
    ("global stores", ("STG", "ST.")),
    ("shared loads / stores", ("LDS", "STS")),
    ("shared atomics", ("ATOMS",)),
    ("global atomics / reductions", ("ATOMG", "RED", "ATOM.")),
    ("async copies global->shared (LDGSTS)", ("LDGSTS",)),
    ("bulk / tensor copies (UBLKCP, UTMALDG)", ("UBLKCP", "UTMALDG", "UTMASTG")),
    ("barriers", ("BAR",)),
    ("warp votes / shuffles / match / redux", ("VOTE", "SHFL", "MATCH", "REDUX")),
    ("fences", ("MEMBAR", "FENCE", "ERRBAR", "CCTL")),
    ("branches", ("BRA", "BSSY", "BSYNC", "WARPSYNC", "EXIT")),
]
print("# SASS opcode summary of `%s` (sm_90a)\n" % lib.split("/")[-1])
print("Produced by `profiles/scripts/sass_summary.py` from `cuobjdump -sass`; counts are static instructions.\n")
for f, c in ops.items():
    total = sum(c.values())
    print("## `%s` — %d instructions (%.2f MB)\n" % (f.split("(")[0], total, total * 16 / 1e6))
    print("| class | count | opcodes |\n|---|---|---|")
    for name, pre in GROUPS:
        hit = {k: v for k, v in c.items() if any(k == p.rstrip(".") or k.startswith(p) for p in pre)}
        if hit:
            print("| %s | %d | %s |" % (name, sum(hit.values()), ", ".join("%s %d" % kv for kv in sorted(hit.items(), key=lambda kv: -kv[1])[:6])))
    print()
