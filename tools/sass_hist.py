"""Instruction histogram per kernel of libqd_b200.so (cuobjdump -sass): the static evidence that the
library is hand-written sm_90a code -- FMNMX.NAN (NaN-propagating float min/max), UBLKCP / SYNCS
(TMA bulk copies and their mbarriers), SHFL-based table search, 128-bit LDG/STG -- and how large each
kernel is.  Runs without a GPU.

    python tools/sass_hist.py [--out profiles/sass_r2.md]
"""
import argparse
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "quantized_distillation_b200", "libqd_b200.so")
KEYS = ["LDG.E.128", "STG.E.128", "LDG", "STG", "LDS", "STS", "UBLKCP", "SYNCS", "FMNMX", "SHFL", "VOTE", "BAR", "FFMA", "FMUL", "FADD",
        "FSETP", "FSEL", "MUFU", "FRND", "DADD", "F2F", "ATOM", "RED", "CALL", "BRA"]


def demangle(names):
    try:
        out = subprocess.run(["c++filt"] + names, capture_output=True, text=True, check=True).stdout.splitlines()
        return dict(zip(names, out))
    except Exception:
        return {n: n for n in names}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "sass_r2.md"))
    args = ap.parse_args()
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels, cur = collections.OrderedDict(), None
    ins = re.compile(r"^\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)")
    for line in sass.splitlines():
        if "Function :" in line:
            cur = line.split("Function :")[1].strip()
            kernels[cur] = collections.Counter()
            continue
        m = ins.match(line)
        if m and cur:
            kernels[cur][m.group(1)] += 1
    names = demangle(list(kernels))
    rows = []
    for k, c in kernels.items():
        total = sum(c.values())
        def cnt(prefix):
            return sum(v for op, v in c.items() if op == prefix or op.startswith(prefix + "."))
        wide_ld = sum(v for op, v in c.items() if op.startswith("LDG") and ".128" in op)
        wide_st = sum(v for op, v in c.items() if op.startswith("STG") and ".128" in op)
        rows.append((names[k], total, wide_ld, wide_st, [cnt(x) for x in KEYS[2:]]))
    with open(args.out, "w") as f:
        f.write("SASS instruction histogram of `libqd_b200.so` (static counts, `cuobjdump -sass`, sm_90a).\n"
                "`FMNMX` = `{min,max}.NaN.f32`, `UBLKCP`/`SYNCS` = TMA bulk copy + mbarrier, "
                "`SHFL` in the centroid kernels = lane-table search.\n\n")
        f.write("| kernel | instr | LDG.128 | STG.128 | " + " | ".join(KEYS[2:]) + " |\n|---|---|---|---|" + "---|" * len(KEYS[2:]) + "\n")
        for name, total, wl, ws, cs in rows:
            short = re.sub(r"\(.*", "", name).replace("void ", "")
            f.write(f"| `{short}` | {total} | {wl} | {ws} | " + " | ".join(str(x) for x in cs) + " |\n")
        tot = collections.Counter()
        for c in kernels.values():
            tot.update(c)
        f.write(f"\n{len(kernels)} kernels, {sum(tot.values())} instructions; library-wide: "
                + ", ".join(f"{k} {sum(v for op, v in tot.items() if op == k or op.startswith(k + '.'))}" for k in ("FMNMX", "UBLKCP", "SYNCS", "SHFL", "MUFU")) + ".\n")
    print("wrote", args.out, len(kernels), "kernels")


if __name__ == "__main__":
    sys.exit(main())
