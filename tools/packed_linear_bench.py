"""Times a fully-connected layer three ways, for choosing PackedLinear.CROSSOVER_ROWS:
  (a) qd_packed_linear on the packed codes,
  (b) decode (qd_unpack_dequant_*) into a scratch float32 weight, then F.linear -- PackedLinear above the crossover,
  (c) F.linear on a resident float32 weight -- an unpacked model.
Shapes: the student's 1600 -> 500, AlexNet's 9216 -> 4096 and 4096 -> 4096 heads, WRN's 1408 -> 10 classifier; batch
m in {1, 4, 16, 32, 64, 128, 1024} (the kernel only for m <= 64); 2, 4 and 8 bits, uniform and non-uniform, bucket 256.

Every variant cycles through enough distinct weight copies that its working set exceeds twice the 50 MB L2, so small-m
numbers are HBM numbers -- except where that would take more than 4096 copies: the packed WRN classifier (16 MB of
codes and scales at 2 bits, 31 MB at 4, 59 MB at 8), whose (a) and (b) cells are L2-resident.  A timed unit is one
CUDA graph of back-to-back calls over every copy (at least `launches` calls; host launch cost excluded: this compares
GPU time); rounds alternate (a), (b), (c) on the same inputs in the same process, and the table gives the median and
range of the per-call time over the rounds.  Rates use the bytes each variant must move (computed from the
shapes) against 3.35 TB/s.  The card name, power limit and SM clock are read in the same run.

    python -m tools.packed_linear_bench [--out profiles/packed_linear_bench.json] [--rounds 5] [--launches 20]"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SHAPES = [("student", 500, 1600), ("alexnet_fc6", 4096, 9216), ("alexnet_fc7", 4096, 4096), ("wrn_fc", 10, 1408)]
MS = [1, 4, 16, 32, 64, 128, 1024]
BITS = [2, 4, 8]
BUCKET = 256
HBM = 3.35e12
L2_BYTES = 50 << 20


def _copies(nbytes):
    return max(2, min(4096, math.ceil(2 * L2_BYTES / max(nbytes, 1))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "packed_linear_bench.json"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="one shape, m in {1, 16, 64}: a rehearsal of the script")
    args = ap.parse_args()

    import torch
    from quantized_distillation_b200 import _native as N
    from tools.packed_bench import card

    N.require_cuda()
    info = card()
    L = N.lib()
    shapes, ms = (SHAPES[:1], [1, 16, 64]) if args.quick else (SHAPES, MS)
    rows = []
    for name, O, K in shapes:
        n = O * K
        nb = N.geometry(n, BUCKET)[0]
        g = torch.Generator(device="cuda").manual_seed(0)
        for bits in BITS:
            for kind in ("uniform", "nonuniform"):
                levels = 1 << bits if kind == "uniform" else 0
                pts = None if kind == "uniform" else torch.sort(torch.rand(1 << bits, device="cuda", generator=g)).values
                kpts = 0 if pts is None else pts.numel()
                code_bytes = (n * bits + 7) // 8
                packed_bytes = code_bytes + 8 * nb
                cp = _copies(packed_bytes)
                codes = torch.randint(0, 256, (cp, code_bytes), dtype=torch.int32, device="cuda", generator=g).to(torch.uint8)
                alpha = torch.rand(cp, nb, device="cuda", generator=g) * 0.1
                beta = torch.randn(cp, nb, device="cuda", generator=g) * 0.05
                cf = _copies(4 * n)
                wf = torch.randn(cf, O, K, device="cuda", generator=g) * 0.05
                bias = torch.randn(O, device="cuda", generator=g)
                scratch = torch.empty(O, K, device="cuda")
                sp = lambda: N.stream_ptr()   # noqa: E731 - the capture stream

                def decode(c):
                    if pts is None:
                        N.check(L.qd_unpack_dequant_uniform(N.ptr(codes[c]), bits, N.ptr(alpha[c]), N.ptr(beta[c]), N.ptr(scratch), n,
                                                            BUCKET, levels, sp()))
                    else:
                        N.check(L.qd_unpack_dequant_nonuniform(N.ptr(codes[c]), bits, N.ptr(pts), kpts, N.ptr(alpha[c]), N.ptr(beta[c]),
                                                               N.ptr(scratch), n, BUCKET, sp()))

                for m in ms:
                    x = torch.randn(m, K, device="cuda", generator=g)
                    y = torch.empty(m, O, device="cuda")
                    variants = {}
                    if m <= N.PACKED_LINEAR_MAX_ROWS:
                        def run_a(c, x=x, y=y, m=m):
                            N.check(L.qd_packed_linear(N.ptr(x), m, K, O, N.ptr(codes[c]), bits, N.ptr(alpha[c]), N.ptr(beta[c]), N.ptr(pts),
                                                       kpts, levels, BUCKET, N.ptr(bias), N.ptr(y), sp()))
                        variants["a_packed_kernel"] = (run_a, cp, packed_bytes + 4 * (m * K + m * O + O))

                    def run_b(c, x=x, y=y):
                        decode(c)
                        torch.addmm(bias, x, scratch.T, out=y)     # F.linear's arithmetic, into a preallocated output
                    variants["b_decode_linear"] = (run_b, cp, packed_bytes + 8 * n + 4 * (m * K + m * O + O))

                    def run_c(c, x=x, y=y):
                        torch.addmm(bias, x, wf[c].T, out=y)
                    variants["c_resident_linear"] = (run_c, cf, 4 * n + 4 * (m * K + m * O + O))

                    graphs, launches = {}, {}
                    for key, (fn, ncopies, _) in variants.items():
                        fn(0)                                      # warm up: modules, cuBLAS heuristics
                        torch.cuda.synchronize()
                        launches[key] = max(args.launches, ncopies)   # every copy once per replay
                        gr = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(gr):
                            for i in range(launches[key]):
                                fn(i % ncopies)
                        graphs[key] = gr
                    times = {k: [] for k in graphs}
                    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                    for _ in range(args.rounds):
                        for key, gr in graphs.items():
                            gr.replay()                            # the copies the next replay reads are not all in L2
                            ev[0].record()
                            gr.replay()
                            ev[1].record()
                            torch.cuda.synchronize()
                            times[key].append(ev[0].elapsed_time(ev[1]) * 1e3 / launches[key])
                    for key, ts in times.items():
                        med = statistics.median(ts)
                        nbytes = variants[key][2]
                        rows.append({"shape": name, "out": O, "in": K, "m": m, "bits": bits, "kind": kind, "variant": key,
                                     "us_median": round(med, 2), "us_min": round(min(ts), 2), "us_max": round(max(ts), 2),
                                     "bytes": nbytes, "GBps": round(nbytes / med / 1e3, 1), "of_hbm": round(nbytes / med / 1e-6 / HBM, 3)})
                    del graphs
                    r = {row["variant"]: row["us_median"] for row in rows[-len(times):]}
                    print(f"{name:12s} m={m:5d} {bits}b {kind:10s} " + "  ".join(f"{k}={v:9.2f}us" for k, v in r.items()), flush=True)
                del codes, alpha, beta, wf, scratch
                torch.cuda.empty_cache()
    out = {"card": info, "bucket": BUCKET, "min_launches_per_graph": args.launches, "rounds": args.rounds, "rows": rows}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(info))
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
