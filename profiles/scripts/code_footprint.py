#!/usr/bin/env python
"""Static code footprint of the built product library: SASS bytes per kernel by source function, and the calm leader
loop's region by lean case.

usage: python profiles/scripts/code_footprint.py [path/to/libhived_cuda.so] [--kernel SUBSTR] [--top N]

Builds nothing and needs no GPU.  Extracts the cubin as `spill_summary.py` does and disassembles it with inline
information (`nvdisasm -gi`), so that an instruction of an inlined function is credited to that function and not to
the line it was inlined at.  Per kernel it prints:
  * its size, and the bytes by out-of-line (ABI-called) function;
  * the bytes by innermost source function (hived_core.h / hived_lean.inc / hived_runahead.inc / hived_calm.inc by
    enclosing member function, other files by file);
  * the calm region: the instructions of the kernel body whose inline stack passes through runLeaderCalm (the calm
    loop, leaderLoop<true>, and everything inlined into it).  The general program behind processEventCall and the other
    out-of-line functions are separate stretches of code and not part of it.  Its bytes by lean case — (a) a DELETE
    that is not the gang's last, (b) the last DELETE (leanDelete, eraseGroup), (c) a further pod (calmPodOfGang),
    (d) a new gang (calmNewGang), the per-event dispatch (calmEvent) and the loop around it — and the bytes of cold
    exits among them: instructions whose innermost calm-side source line hands the event over (`return false`,
    `return 0`) or panics.  That split is by source line and therefore approximate; the case totals are exact.
Sizes are static bytes (16 per instruction), not executions."""
import argparse
import collections
import glob
import os
import re
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from spill_summary import CSRC, FOLDED, demangle, enclosing, function_ranges, tool  # noqa: E402

INSN = re.compile(r"\s*/\*([0-9a-f]+)\*/\s+\S")
FRAME = re.compile(r'\s*//## File "([^"]+)", line (\d+)')
COLD = re.compile(r"\breturn (false|0)\b|\bpanic\(")
# the lean cases, by the outermost calm-side function on the inline stack
CASES = (("calmNewGang", "(d) new gang"), ("calmPodOfGang", "(c) further pod"), ("calmDelete", "(a) DELETE, not the last"))
LAST_DELETE = {"leanDelete", "leanDelete1", "eraseGroup"}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("lib", nargs="?", default=os.path.join(CSRC, "libhived_cuda.so"))
    ap.add_argument("--kernel", default="hived_events_kernel", help="report only kernels whose name contains this")
    ap.add_argument("--top", type=int, default=25, help="source functions listed per kernel")
    a = ap.parse_args()
    ranges = {f: function_ranges(f) for f in FOLDED}
    text = {}
    for f in FOLDED:
        with open(os.path.join(CSRC, f)) as fh:
            text[f] = fh.read().split("\n")
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run([tool("cuobjdump"), "-xelf", "all", os.path.abspath(a.lib)], cwd=tmp, check=True, capture_output=True)
        dis = ""
        for cb in sorted(glob.glob(os.path.join(tmp, "*.cubin"))):
            dis += subprocess.run([tool("nvdisasm"), "-gi", "-c", cb], capture_output=True, text=True, check=True).stdout

    def fn_of(fr):
        f, ln = fr
        return enclosing(ranges[f], ln) if f in ranges else "(%s)" % f

    kernels = collections.OrderedDict()
    kern = sub = None
    stack, pending = [], []
    for line in dis.split("\n"):
        m = re.match(r"\s*\.section\s+\.text\.(\S+?),", line)
        if m:
            kern, sub, stack, pending = m.group(1), None, [], []
            kernels.setdefault(kern, {"total": 0, "sub": collections.Counter(), "fn": collections.Counter(),
                                      "calm": collections.Counter(), "calm_cold": collections.Counter(),
                                      "calm_fn": collections.Counter()})
            continue
        m = re.match(r"\s*\.type\s+\$(\S+?)\$(\S+?),@function", line)
        if m and kern:
            sub = m.group(2)
            continue
        m = FRAME.match(line)
        if m:  # one frame per line, innermost first; the outermost has no "inlined at"
            pending.append((os.path.basename(m.group(1)), int(m.group(2))))
            if "inlined at" not in line:
                stack, pending = pending, []
            continue
        if kern is None or not INSN.match(line):
            continue
        k = kernels[kern]
        k["total"] += 16
        k["sub"][sub or "(kernel body)"] += 16
        k["fn"][fn_of(stack[0]) if stack else "(no line)"] += 16
        fns = [fn_of(fr) for fr in stack]  # innermost first
        if sub is not None or "runLeaderCalm" not in fns:
            continue
        case = "loop (leaderLoop<true>)"
        outer = fns[::-1]
        if "calmEvent" in outer:
            case = "dispatch (calmEvent)"
        for fn, name in CASES:
            if fn in outer:
                case = name
                if fn == "calmDelete" and LAST_DELETE & set(outer[outer.index(fn):]):
                    case = "(b) last DELETE (leanDelete, eraseGroup)"
                break
        k["calm"][case] += 16
        k["calm_fn"][(case, fns[0])] += 16
        # cold: the innermost frame in the calm / lean sources is a hand-over or panic line
        for fr in stack:
            if fr[0] in ("hived_calm.inc", "hived_lean.inc") or fr[0] == "hived_core.h" and fn_of(fr) == "emitBind":
                if COLD.search(text[fr[0]][fr[1] - 1]):
                    k["calm_cold"][case] += 16
                break
    names = demangle(list(kernels) + sorted({s for k in kernels.values() for s in k["sub"] if s[0] != "("}))
    print("# Code footprint of `%s`\n" % os.path.basename(a.lib))
    print("Produced by `profiles/scripts/code_footprint.py` from `nvdisasm -gi`; static bytes.\n")
    for kern, k in kernels.items():
        pretty = names.get(kern, kern).split("(")[0]
        if a.kernel not in pretty:
            continue
        print("## `%s` — %d B (%d instructions)\n" % (pretty, k["total"], k["total"] // 16))
        print("| out-of-line function | bytes |\n|---|---|")
        for s, b in k["sub"].most_common(a.top):
            print("| %s | %d |" % (names.get(s, s).split("(")[0] if s[0] != "(" else s, b))
        print("\n| innermost source function | bytes |\n|---|---|")
        for s, b in k["fn"].most_common(a.top):
            print("| %s | %d |" % (s, b))
        if k["calm"]:
            tot = sum(k["calm"].values())
            cold = sum(k["calm_cold"].values())
            print("\n### calm region: %d B, of which %d B on cold-exit lines\n" % (tot, cold))
            print("| case | bytes | cold-exit bytes |\n|---|---|---|")
            for case, b in sorted(k["calm"].items()):
                print("| %s | %d | %d |" % (case, b, k["calm_cold"][case]))
            print("\n| case: innermost source function | bytes |\n|---|---|")
            for (case, fn), b in k["calm_fn"].most_common(a.top):
                print("| %s: %s | %d |" % (case, fn, b))
        print()


if __name__ == "__main__":
    main()
