#!/usr/bin/env python
"""Local-memory traffic (LDL / STL: register spills and the device stack) of the built product library, per kernel.

usage: python profiles/scripts/spill_summary.py [path/to/libhived_cuda.so] [--top N]

Builds nothing and needs no GPU: extracts the cubin (`cuobjdump -xelf`), disassembles it with line information
(`nvdisasm -g`) and prints, per kernel, the register count and stack frame (`cuobjdump -res-usage`), its static LDL /
STL count, and the same count split by out-of-line (ABI-called) function, by the function of hived_core.h /
hived_lean.inc / hived_runahead.inc / hived_calm.inc whose line range holds the instruction's source line (other files:
by file), and by source line.  `ptxas -v`'s register line cannot show what setmaxnreg does (it prints the launch-time
count), this can.  Counts are static instructions, not executions."""
import argparse
import collections
import glob
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CSRC = os.path.join(ROOT, "hivedscheduler_b200", "csrc")
FOLDED = ("hived_core.h", "hived_lean.inc", "hived_runahead.inc", "hived_calm.inc")
# a member function's definition in struct Core (two spaces of indentation), template line or not
DEF = re.compile(r"^  (?:template\s*<.*>\s*)?HIVED_DEV(?:_NOINLINE)?\s+(?:static\s+)?[\w:<>,*&\s]*?\b(\w+)\s*\(")


def tool(name):
    for cand in (os.path.join("/usr/local/cuda/bin", name), name):
        if os.path.exists(cand) or "/" not in cand:
            return cand


def function_ranges(fname):
    """[(first line, last line, name)] of the member functions defined in csrc/<fname>, ascending.  A definition on one
    line ends there; any other ends before the next definition."""
    out = []
    with open(os.path.join(CSRC, fname)) as f:
        lines = f.read().split("\n")
    for i, line in enumerate(lines, 1):
        m = DEF.match(line)
        if m:
            first = i - 1 if i > 1 and lines[i - 2].lstrip().startswith("template") else i
            one_line = line.count("{") > 0 and line.count("{") == line.count("}")
            out.append([first, i if one_line else None, m.group(1)])
    for j, r in enumerate(out):
        if r[1] is None:
            r[1] = out[j + 1][0] - 1 if j + 1 < len(out) else len(lines)
    return out


def enclosing(ranges, line):
    for first, last, fn in ranges:
        if first <= line <= last:
            return fn
    return "(between functions)"


def demangle(names):
    if not names:
        return {}
    r = subprocess.run(["c++filt", "-p"], input="\n".join(names), capture_output=True, text=True, check=True)
    return dict(zip(names, r.stdout.split("\n")))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("lib", nargs="?", default=os.path.join(CSRC, "libhived_cuda.so"))
    ap.add_argument("--top", type=int, default=12, help="source lines listed per kernel")
    a = ap.parse_args()
    ranges = {f: function_ranges(f) for f in FOLDED}
    usage = {}
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run([tool("cuobjdump"), "-xelf", "all", os.path.abspath(a.lib)], cwd=tmp, check=True, capture_output=True)
        cubins = sorted(glob.glob(os.path.join(tmp, "*.cubin")))
        dis = ""
        for cb in cubins:
            dis += subprocess.run([tool("nvdisasm"), "-g", "-c", cb], capture_output=True, text=True, check=True).stdout
            res = subprocess.run([tool("cuobjdump"), "-res-usage", cb], capture_output=True, text=True, check=True).stdout
            for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", res):
                usage[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    # per kernel: counters keyed by (kind, key) -> [LDL, STL]
    kernels = collections.OrderedDict()
    kern = sub = None
    src_file, src_line = "?", 0
    for line in dis.split("\n"):
        m = re.match(r"\s*\.section\s+\.text\.(\S+?),", line)
        if m:
            kern, sub = m.group(1), None
            kernels.setdefault(kern, collections.defaultdict(lambda: [0, 0]))
            continue
        m = re.match(r"\s*\.type\s+\$(\S+?)\$(\S+?),@function", line)
        if m and kern:
            sub = m.group(2)
            continue
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)', line)
        if m:
            src_file, src_line = os.path.basename(m.group(1)), int(m.group(2))
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?(LDL|STL)\b", line)
        if not m or kern is None:
            continue
        i = 0 if m.group(1) == "LDL" else 1
        c = kernels[kern]
        c[("total", "")][i] += 1
        c[("sass", sub or "(kernel body)")][i] += 1
        fn = enclosing(ranges[src_file], src_line) if src_file in ranges else "(file)"
        c[("func", "%s: %s" % (src_file, fn))][i] += 1
        c[("line", "%s:%d" % (src_file, src_line))][i] += 1
    names = demangle(list(kernels) + sorted({k[1] for c in kernels.values() for k in c if k[0] == "sass"}))
    print("# Local-memory instructions (LDL / STL) of `%s`\n" % os.path.basename(a.lib))
    print("Produced by `profiles/scripts/spill_summary.py` from `nvdisasm -g`; static instruction counts.\n")
    for kern, c in kernels.items():
        reg, stack = usage.get(kern, ("?", "?"))
        ldl, stl = c[("total", "")]
        print("## `%s` — REG %s, stack frame %s B, LDL %d, STL %d\n" % (names.get(kern, kern).split("(")[0], reg, stack, ldl, stl))
        if ldl + stl == 0:
            continue
        for kind, title in (("sass", "out-of-line function"), ("func", "source function (file: enclosing function)"),
                            ("line", "source line")):
            rows = sorted(((k[1], v) for k, v in c.items() if k[0] == kind), key=lambda kv: -(kv[1][0] + kv[1][1]))
            if kind == "line":
                rows = rows[:a.top]
            print("| %s | LDL | STL |\n|---|---|---|" % title)
            for key, (l_, s_) in rows:
                shown = names.get(key, key).split("(")[0] if kind == "sass" and key[0] != "(" else key
                print("| %s | %d | %d |" % (shown, l_, s_))
            print()


if __name__ == "__main__":
    main()
