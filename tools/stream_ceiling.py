"""Copy ceiling of the headline's traffic: builds and runs tools/stream_ceiling.cu (copy kernels over the headline's
64 Mi floats in rows of 256, 16 B per element, under several row orders, plus the library's headline call in the same
process), records the card, and writes profiles/stream_ceiling.json and MEASURED_PEAKS.json (hbm_gbs = the best copy
variant's median, read by bench.py and tools/block_bench.py as the peak).

    python tools/stream_ceiling.py [--launches 200] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        res = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True)
    except FileNotFoundError:
        return "unknown (no nvidia-smi)"
    return res.stdout.strip().splitlines()[0] if res.returncode == 0 and res.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "stream_ceiling.json"))
    args = ap.parse_args()
    from quantized_distillation_b200 import build as B
    lib = B.build()
    libdir = os.path.dirname(lib)
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "stream_ceiling")
        cmd = [B.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
               "-I", os.path.join(libdir, "csrc"), "-o", exe, os.path.join(ROOT, "tools", "stream_ceiling.cu"),
               "-L" + libdir, "-lqd_b200", "-Xlinker", "-rpath=" + libdir]
        subprocess.run(cmd, check=True)
        before = card()
        res = subprocess.run([exe, str(args.launches), str(args.rounds)], capture_output=True, text=True)
        after = card()
    if res.returncode != 0:
        raise SystemExit(res.stderr)
    raw = json.loads(res.stdout)
    bytes_per_launch = raw["n"] * raw["bytes_per_elem"]
    table = {}
    for name, samples in raw["us"].items():
        gbs = [bytes_per_launch / (u * 1e-6) / 1e9 for u in samples]
        table[name] = {"us_median": round(statistics.median(samples), 2), "GBps_median": round(statistics.median(gbs), 1),
                       "GBps_min": round(min(gbs), 1), "GBps_max": round(max(gbs), 1), "us": samples}
    copies = {k: v for k, v in table.items() if not k.startswith("headline")}
    best = max(copies, key=lambda k: copies[k]["GBps_median"])
    out = {"card_before": before, "card_after": after, "launches": raw["launches"], "rounds": raw["rounds"], "sms": raw["sms"],
           "n": raw["n"], "row_floats": raw["row_floats"], "bytes_per_launch": bytes_per_launch, "best_copy": best, "variants": table}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    with open(os.path.join(ROOT, "MEASURED_PEAKS.json"), "w") as f:
        json.dump({"hbm_gbs": table[best]["GBps_median"], "source": f"tools/stream_ceiling.py {best}, {before}"}, f, indent=1)
    print(f"card: {before} -> {after}")
    for name, r in table.items():
        print(f"{name:40s} {r['us_median']:8.2f} us  {r['GBps_median']:7.1f} GB/s  [{r['GBps_min']:.1f} .. {r['GBps_max']:.1f}]")
    print("best copy:", best, "; wrote", args.out)


if __name__ == "__main__":
    main()
