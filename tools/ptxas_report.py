"""Registers, spills and static shared memory per kernel of libqd_b200.so as ptxas reports them (`-Xptxas -v`): compiles
the library's translation units into a scratch file (the in-tree library is not touched) and tabulates the log.  Runs
without a GPU.

    python tools/ptxas_report.py [--out profiles/ptxas_r2.md]
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def demangle(names):
    try:
        out = subprocess.run(["c++filt"] + names, capture_output=True, text=True, check=True).stdout.splitlines()
        return dict(zip(names, out))
    except Exception:
        return {n: n for n in names}


def short(sig):
    """`void qd::kernel<...>(args)` -> `qd::kernel<...>`"""
    sig = re.sub(r"^void ", "", sig)
    depth = 0
    for i, ch in enumerate(sig):
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0:
            return sig[:i]
    return sig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "ptxas_r2.md"))
    ap.add_argument("--log", default=None, help="parse an existing `nvcc -Xptxas -v` log instead of compiling")
    args = ap.parse_args()
    if args.log:
        log = open(args.log).read()
    else:
        from quantized_distillation_b200 import build as B
        with tempfile.TemporaryDirectory() as tmp:
            cmd = [B.nvcc()] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-o", os.path.join(tmp, "scratch.so")] + B.SOURCES
            res = subprocess.run(cmd, capture_output=True, text=True)
            if res.returncode != 0:
                raise SystemExit(res.stderr)
            log = res.stderr
    rows, cur = [], None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)' for 'sm_90a'", line)
        if m:
            cur = {"name": m.group(1), "stack": 0, "spill_st": 0, "spill_ld": 0, "regs": 0, "smem": 0, "barriers": 0}
            rows.append(cur)
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            cur["stack"], cur["spill_st"], cur["spill_ld"] = (int(v) for v in m.groups())
        m = re.search(r"Used (\d+) registers(?:, used (\d+) barriers)?(?:, (\d+) bytes smem)?", line)
        if m:
            cur["regs"], cur["barriers"], cur["smem"] = int(m.group(1)), int(m.group(2) or 0), int(m.group(3) or 0)
    names = demangle([r["name"] for r in rows])
    for r in rows:
        r["kernel"] = short(names[r["name"]])
    rows.sort(key=lambda r: r["kernel"])
    spilled = [r for r in rows if r["spill_st"] or r["spill_ld"]]
    with open(args.out, "w") as f:
        f.write("Registers / spills / static shared memory per kernel of `libqd_b200.so`, from `nvcc -Xptxas -v` "
                "(sm_90a, the library's own flags; `tools/ptxas_report.py`, no GPU needed).\n\n")
        f.write(f"{len(rows)} kernels; {len(spilled)} with register spills "
                f"(max {max([r['spill_st'] for r in rows] + [0])} B of spill stores); "
                f"max registers {max(r['regs'] for r in rows)}.\n\n")
        f.write("| kernel | registers | stack B | spill stores B | spill loads B | static smem B | barriers |\n|---|---|---|---|---|---|---|\n")
        for r in rows:
            f.write(f"| `{r['kernel']}` | {r['regs']} | {r['stack']} | {r['spill_st']} | {r['spill_ld']} | {r['smem']} | {r['barriers']} |\n")
    print(f"{len(rows)} kernels, {len(spilled)} with spills -> {args.out}")


if __name__ == "__main__":
    main()
