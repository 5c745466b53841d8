"""Throughput of the block path (rows of 1025 .. 49152 floats) per row length, op and VARIANT:
warp-per-row two-pass, CTA-per-row TMA chunk ring with two rows in flight (staged2) or one (staged1).
The variants are forced through qd_debug_set_tuning; `auto` is the built-in choice.

    python tools/block_bench.py [--out gpurun_out/block_path.json] [--quick]
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
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "block_path.json"))
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--small", action="store_true", help="rows of 384 .. 1024 floats: warp path vs staged ring (tuning key 4)")
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

    def tune(key, value):
        N.check(lib.qd_debug_set_tuning(key, value))

    rows = []
    if args.small:
        return small_rows(args, lib, sp, dev, peak, n, x, g, q, go, idx, pts4, pts16, timed, tune)
    buckets = (1280, 1536, 2048) if args.quick else (1280, 2048, 3072, 4096, 6144, 8192, 12288, 16384, 24576, 32768, 49152)
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
        # variant -> (key 0 warp2_max, key 1 two_stage_max, key 2 threads per CTA)
        variants = {"auto": (-1, -1, -1)}
        if bucket <= 8192:
            variants["warp2"] = (1 << 20, -1, -1)
        for stages, threads in ((2, 64), (2, 128), (2, 256), (2, 512), (1, 256), (1, 512), (1, 1024)):
            if stages == 2 and bucket > 24576:
                continue
            if threads == 64 and bucket > 2048 or threads == 128 and bucket > 4096 or threads == 256 and bucket > 16384 or threads == 1024 and bucket < 8192:
                continue
            if stages == 1 and bucket < 4096:
                continue
            variants[f"s{stages}t{threads}"] = (0, (1 << 20) if stages == 2 else 0, threads)
        for vname, (t0, t1, t2) in variants.items():
            tune(0, t0)
            tune(1, t1)
            tune(2, t2)
            for oname, (bpe, fn) in ops.items():
                if vname == "warp2" and oname == "uniform_fwd" and bucket <= 2048:
                    continue          # the plain forward keeps rows <= 2048 in registers (warp path), not a block variant
                sec = timed(fn)
                gbs = n * bpe / sec / 1e9
                rows.append({"bucket": bucket, "variant": vname, "op": oname, "us": round(sec * 1e6, 1), "GBps": round(gbs, 1),
                             "frac_measured_peak": round(gbs / peak, 3)})
        tune(2, -1)
        tune(0, -1)
        tune(1, -1)
        print(f"bucket {bucket:6d}: " + " | ".join(
            f"{o} " + "/".join(f"{r['variant']}={r['us']:.0f}" for r in rows if r["bucket"] == bucket and r["op"] == o) for o in ops), flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"n": n, "peak_GBps": peak, "rows": rows}, f, indent=1)
    with open(args.out.replace(".json", ".md"), "w") as f:
        f.write(f"64 Mi float32, levels 16; microseconds per launch (fraction of the measured HBM peak {peak:.0f} GB/s)\n\n")
        opn = list(dict.fromkeys(r["op"] for r in rows))
        f.write("| bucket | variant | " + " | ".join(opn) + " |\n|---|---|" + "---|" * len(opn) + "\n")
        for b in buckets:
            for v in list(dict.fromkeys(r["variant"] for r in rows)):
                cells = []
                for o in opn:
                    m = [r for r in rows if r["bucket"] == b and r["variant"] == v and r["op"] == o]
                    cells.append(f"{m[0]['us']:.0f} ({m[0]['frac_measured_peak']:.2f})" if m else "-")
                if any(c != "-" for c in cells):
                    f.write(f"| {b} | {v} | " + " | ".join(cells) + " |\n")
    print("wrote", args.out)


def small_rows(args, lib, sp, dev, peak, n, x, g, q, go, idx, pts4, pts16, timed, tune):
    """Rows the warp path keeps in registers (R = 4: <= 512, R = 8: <= 1024) against the staged ring forced down to them."""
    rows = []
    for bucket in (384, 512, 768, 1024):
        ws = N.workspace(n, bucket, dev)
        ops = {
            "uniform_fwd": (8, lambda: N.check(lib.qd_uniform_fwd(N.ptr(x), N.ptr(q), None, None, None, None, None, n, bucket, 16, None, 0.0, 0, 0, 0, N.ptr(ws), ws.numel(), sp))),
            "fused_ste": (16, lambda: N.check(lib.qd_uniform_fwd_bwd(N.ptr(x), N.ptr(g), N.ptr(q), N.ptr(go), n, bucket, 16, N.BWD_STE, N.ptr(ws), ws.numel(), sp))),
            "fused_minmax": (16, lambda: N.check(lib.qd_uniform_fwd_bwd(N.ptr(x), N.ptr(g), N.ptr(q), N.ptr(go), n, bucket, 16, N.BWD_MINMAX, N.ptr(ws), ws.numel(), sp))),
            "bwd_minmax": (12, lambda: N.check(lib.qd_uniform_bwd(N.ptr(x), N.ptr(g), N.ptr(go), n, bucket, 16, N.BWD_MINMAX, N.ptr(ws), ws.numel(), sp))),
            "nonuniform_K4_mid": (9, lambda: N.check(lib.qd_nonuniform_fwd(N.ptr(x), N.ptr(pts4), 4, N.RULE_MIDPOINT, N.ptr(q), N.ptr(idx), None, None, None, n, bucket, None, 0.0, N.ptr(ws), ws.numel(), sp))),
            "nonuniform_K16_near": (9, lambda: N.check(lib.qd_nonuniform_fwd(N.ptr(x), N.ptr(pts16), 16, N.RULE_NEAREST, N.ptr(q), N.ptr(idx), None, None, None, n, bucket, None, 0.0, N.ptr(ws), ws.numel(), sp))),
        }
        for vname, key4 in (("warp", -1), ("staged_t64", 256)):
            tune(4, key4)
            for oname, (bpe, fn) in ops.items():
                sec = timed(fn)
                gbs = n * bpe / sec / 1e9
                rows.append({"bucket": bucket, "variant": vname, "op": oname, "us": round(sec * 1e6, 1), "frac_measured_peak": round(gbs / peak, 3)})
        tune(4, -1)
        print(f"bucket {bucket:5d}: " + " | ".join(f"{o} " + "/".join(f"{r['variant']}={r['us']:.0f}" for r in rows if r["bucket"] == bucket and r["op"] == o) for o in ops), flush=True)
    out = args.out.replace(".json", "_small_rows.json")
    json.dump({"rows": rows}, open(out, "w"), indent=1)
    with open(out.replace(".json", ".md"), "w") as f:
        opn = list(dict.fromkeys(r["op"] for r in rows))
        f.write("64 Mi float32, levels 16; microseconds per launch (fraction of the measured HBM peak)\n\n| bucket | variant | " + " | ".join(opn) + " |\n|---|---|" + "---|" * len(opn) + "\n")
        for b in (384, 512, 768, 1024):
            for v in ("warp", "staged_t64"):
                cells = [next(f"{r['us']:.0f} ({r['frac_measured_peak']:.2f})" for r in rows if r["bucket"] == b and r["variant"] == v and r["op"] == o) for o in opn]
                f.write(f"| {b} | {v} | " + " | ".join(cells) + " |\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
