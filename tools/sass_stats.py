#!/usr/bin/env python
"""Per-kernel SASS opcode statistics of an object file / shared library (cuobjdump -sass).

    python tools/sass_stats.py dasp_pytorch_b200/libdasp_b200.so [--filter eq_] [--md]

Used to check, without a GPU, what the compiler made of a kernel (FFMA / FMUL / FADD counts, shuffles, shared-memory
and local-memory traffic, TMA bulk copies).
"""
import collections
import re
import subprocess
import sys

KEYS = ["FFMA2", "FMUL2", "FADD2", "FFMA", "FMUL", "FADD", "DFMA", "MUFU", "SHFL", "LDS", "STS", "LDG", "STG", "LDL", "STL",
        "UBLKCP", "SYNCS", "BAR", "IMAD", "MOV", "SEL", "BRA"]


def main():
    path = sys.argv[1]
    flt = None
    if "--filter" in sys.argv:
        flt = sys.argv[sys.argv.index("--filter") + 1]
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
    funcs = collections.OrderedDict()
    cur = None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m and cur:
            op = m.group(1).split(".")[0]
            funcs[cur][op] += 1
            funcs[cur]["_total"] += 1
    demangle = lambda n: subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
    md = "--md" in sys.argv
    if md:
        print("| kernel | total | " + " | ".join(KEYS) + " |")
        print("|---|---:|" + "---:|" * len(KEYS))
    for name, c in funcs.items():
        if flt and flt not in name:
            continue
        d = demangle(name)
        d = re.sub(r"\(anonymous namespace\)::", "", d)
        if d.endswith(")"):                      # drop the trailing parameter list (balanced parentheses from the end)
            depth = 0
            for i in range(len(d) - 1, -1, -1):
                depth += d[i] == ")"
                depth -= d[i] == "("
                if depth == 0:
                    d = d[:i]
                    break
        if md:
            print(f"| `{d}` | {c['_total']} | " + " | ".join(str(c[k]) for k in KEYS) + " |")
        else:
            print(d, c["_total"], {k: c[k] for k in KEYS if c[k]})


if __name__ == "__main__":
    main()
