"""Throughput of the built-in path choice per row length and op at 64 Mi floats: rows of 1280 .. 49152 floats
(warp two-pass and staged ring, DESIGN.md section 3), or with --small rows of 384 .. 1024 floats (warp path, and the
staged ring for the ragged min/max backward rows).

    python tools/block_bench.py [--out block_path.json] [--quick | --small]

Writes the JSON rows to --out (default: block_path.json in the current directory) and a Markdown table next to it.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from quantized_distillation_b200 import _native as N  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="block_path.json")
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--small", action="store_true", help="rows of 384 .. 1024 floats")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    lib, sp = N.lib(), N.stream_ptr(dev)
    peak = 3350.0                                   # H100 SXM data sheet, used without a measured peak
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peak = float(json.load(open(pk))["hbm_gbs"])
    n = 1 << 26
    x = torch.randn(n, device=dev) * 0.05
    g = torch.randn(n, device=dev)
    q, go = torch.empty_like(x), torch.empty_like(g)
    idx = torch.empty(n, dtype=torch.uint8, device=dev)
    pts4 = torch.linspace(0, 1, 4, device=dev)
    pts16 = torch.sort(torch.rand(16, device=dev))[0]

    def timed(fn, iters=8):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters * 1e-3

    if args.small:
        buckets, out = (384, 512, 768, 1024), args.out.replace(".json", "_small_rows.json")
    else:
        buckets = (1280, 1536, 2048) if args.quick else (1280, 2048, 3072, 4096, 6144, 8192, 12288, 16384, 24576, 32768, 49152)
        out = args.out
    rows = []
    for bucket in buckets:
        ws = N.workspace(n, bucket, dev)
        ops = {
            "uniform_fwd": (8, lambda: N.check(lib.qd_uniform_fwd(N.ptr(x), N.ptr(q), None, None, None, None, None, n, bucket, 16, None, 0.0, 0, 0, 0, N.ptr(ws), ws.numel(), sp))),
            "fused_ste": (16, lambda: N.check(lib.qd_uniform_fwd_bwd(N.ptr(x), N.ptr(g), N.ptr(q), N.ptr(go), n, bucket, 16, N.BWD_STE, N.ptr(ws), ws.numel(), sp))),
            "fused_minmax": (16, lambda: N.check(lib.qd_uniform_fwd_bwd(N.ptr(x), N.ptr(g), N.ptr(q), N.ptr(go), n, bucket, 16, N.BWD_MINMAX, N.ptr(ws), ws.numel(), sp))),
            "bwd_minmax": (12, lambda: N.check(lib.qd_uniform_bwd(N.ptr(x), N.ptr(g), N.ptr(go), n, bucket, 16, N.BWD_MINMAX, N.ptr(ws), ws.numel(), sp))),
            "nonuniform_K4_mid": (9, lambda: N.check(lib.qd_nonuniform_fwd(N.ptr(x), N.ptr(pts4), 4, N.RULE_MIDPOINT, N.ptr(q), N.ptr(idx), None, None, None, n, bucket, None, 0.0, N.ptr(ws), ws.numel(), sp))),
            "nonuniform_K16_near": (9, lambda: N.check(lib.qd_nonuniform_fwd(N.ptr(x), N.ptr(pts16), 16, N.RULE_NEAREST, N.ptr(q), N.ptr(idx), None, None, None, n, bucket, None, 0.0, N.ptr(ws), ws.numel(), sp))),
        }
        for oname, (bpe, fn) in ops.items():
            sec = timed(fn)
            gbs = n * bpe / sec / 1e9
            rows.append({"bucket": bucket, "op": oname, "us": round(sec * 1e6, 1), "GBps": round(gbs, 1),
                         "frac_measured_peak": round(gbs / peak, 3)})
        print(f"bucket {bucket:6d}: " + " | ".join(f"{r['op']} {r['us']:.0f}" for r in rows if r["bucket"] == bucket), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        json.dump({"n": n, "peak_GBps": peak, "rows": rows}, f, indent=1)
    with open(out.replace(".json", ".md"), "w") as f:
        f.write(f"64 Mi float32, levels 16; microseconds per launch (fraction of the measured HBM peak {peak:.0f} GB/s)\n\n")
        opn = list(dict.fromkeys(r["op"] for r in rows))
        f.write("| bucket | " + " | ".join(opn) + " |\n|---|" + "---|" * len(opn) + "\n")
        for b in buckets:
            cells = [next(f"{r['us']:.0f} ({r['frac_measured_peak']:.2f})" for r in rows if r["bucket"] == b and r["op"] == o) for o in opn]
            f.write(f"| {b} | " + " | ".join(cells) + " |\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
