"""Times a convolution four ways, for choosing PackedConv2d.CROSSOVER_MACS:
  (a) qd_packed_conv2d on the packed codes,
  (b) decode (qd_unpack_dequant_*) into a scratch float32 weight, then F.conv2d with TF32 on (torch's default, what the
      models here run with) -- PackedConv2d above the crossover,
  (c) the same with TF32 off,
  (d) F.conv2d on a resident float32 weight (TF32 on) -- an unpacked model.
Layers: every distinct convolution of the student and of WRN-16-22; batch N in {1, 2, 4, 8, 25, 32, 128}; 2, 4 and 8
bits, uniform and non-uniform, bucket 256.  Then a whole-model forward at batch 1 and 128 of the student and
WRN-16-22, attach_packed_-loaded against unpack_-loaded (4-bit codes, TF32 on).

A timed unit is one CUDA graph of back-to-back calls (host launch cost excluded: this compares GPU time) that cycles
through distinct weight copies, enough that the copies exceed twice the 50 MB L2, at most --max-copies of them (layers
whose copies stay under that, the student's and the small WRN layers' packed cells, run partly from L2).  Rounds
alternate the variants on the same inputs in the same process; the table gives the median and range of the per-call
time over the rounds.  Where even the FP32 data-sheet rate (67 TFLOP/s) would put (a) above the measured (b), (a) is
not timed: the kernel cannot win that cell, and timing it would cost minutes of GPU time per cell.  The card name,
power limit and SM clock are read in the same run.

    python -m tools.packed_conv_bench [--out profiles/packed_conv_bench.json] [--rounds 3] [--quick]"""
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

# (name, C, O, H, W, k, stride, padding)
STUDENT = [("student0", 3, 75, 32, 32, 5, 1, 2), ("student1", 75, 50, 32, 32, 5, 1, 2), ("student2", 50, 50, 16, 16, 5, 1, 2),
           ("student3", 50, 25, 16, 16, 5, 1, 2)]
WRN = [("wrn_stem", 3, 16, 32, 32, 3, 1, 1), ("wrn_l1_16_352", 16, 352, 32, 32, 3, 1, 1), ("wrn_l1_352_352", 352, 352, 32, 32, 3, 1, 1),
       ("wrn_l1_sc_16_352", 16, 352, 32, 32, 1, 1, 0), ("wrn_l2_352_704", 352, 704, 32, 32, 3, 1, 1),
       ("wrn_l2_704_s2", 704, 704, 32, 32, 3, 2, 1), ("wrn_l2_sc_s2", 352, 704, 32, 32, 1, 2, 0), ("wrn_l2_704_704", 704, 704, 16, 16, 3, 1, 1),
       ("wrn_l3_704_1408", 704, 1408, 16, 16, 3, 1, 1), ("wrn_l3_1408_s2", 1408, 1408, 16, 16, 3, 2, 1),
       ("wrn_l3_sc_s2", 704, 1408, 16, 16, 1, 2, 0), ("wrn_l3_1408_1408", 1408, 1408, 8, 8, 3, 1, 1)]
BATCHES = [1, 2, 4, 8, 25, 32, 128]
BITS = [2, 4, 8]
BUCKET = 256
FP32_PEAK = 67e12            # H100 SXM data sheet, dense FP32
L2_BYTES = 50 << 20


def _graph_time(torch, fns, rounds, launches):
    """{key: per-call microseconds over rounds} of graphs of `launches[key]` calls fns[key](i), rounds alternating."""
    graphs = {}
    for key, fn in fns.items():
        fn(0)                                      # warm up: modules, cuDNN heuristics
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(launches[key]):
                fn(i)
        graphs[key] = g
    times = {k: [] for k in graphs}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(rounds):
        for key, g in graphs.items():
            g.replay()                             # the copies the next replay reads are not all in L2
            ev[0].record()
            g.replay()
            ev[1].record()
            torch.cuda.synchronize()
            times[key].append(ev[0].elapsed_time(ev[1]) * 1e3 / launches[key])
    return times


def layers(args, torch, N, card_rows):
    import torch.nn.functional as F
    L = N.lib()
    shapes = (STUDENT[1:2] + WRN[1:2]) if args.quick else STUDENT + WRN
    batches = [1, 32] if args.quick else BATCHES
    rows = []
    for name, C, O, H, W, k, st, pd in shapes:
        K = C * k * k
        n = O * K
        nb = N.geometry(n, BUCKET)[0]
        Ho, Wo = (H + 2 * pd - k) // st + 1, (W + 2 * pd - k) // st + 1
        g = torch.Generator(device="cuda").manual_seed(0)
        for bits in BITS:
            for kind in ("uniform", "nonuniform"):
                levels = 1 << bits if kind == "uniform" else 0
                pts = None if kind == "uniform" else torch.sort(torch.rand(1 << bits, device="cuda", generator=g)).values
                kpts = 0 if pts is None else pts.numel()
                code_bytes = (n * bits + 7) // 8
                cp = max(2, min(args.max_copies, math.ceil(2 * L2_BYTES / (code_bytes + 8 * nb))))
                codes = torch.randint(0, 256, (cp, code_bytes), dtype=torch.int32, device="cuda", generator=g).to(torch.uint8)
                alpha = torch.rand(cp, nb, device="cuda", generator=g) * 0.1
                beta = torch.randn(cp, nb, device="cuda", generator=g) * 0.05
                cf = max(2, min(args.max_copies, math.ceil(2 * L2_BYTES / (4 * n))))
                wf = torch.randn(cf, O, C, k, k, device="cuda", generator=g) * 0.05
                bias = torch.randn(O, device="cuda", generator=g)

                def decode(c, scratch):
                    sp = N.stream_ptr()
                    if pts is None:
                        N.check(L.qd_unpack_dequant_uniform(N.ptr(codes[c]), bits, N.ptr(alpha[c]), N.ptr(beta[c]), N.ptr(scratch), n,
                                                            BUCKET, levels, sp))
                    else:
                        N.check(L.qd_unpack_dequant_nonuniform(N.ptr(codes[c]), bits, N.ptr(pts), kpts, N.ptr(alpha[c]), N.ptr(beta[c]),
                                                               N.ptr(scratch), n, BUCKET, sp))

                for nbatch in batches:
                    x = torch.randn(nbatch, C, H, W, device="cuda", generator=g)
                    y = torch.empty(nbatch, O, Ho, Wo, device="cuda")
                    macs = nbatch * Ho * Wo * O * K

                    def run_a(i, x=x, y=y, nbatch=nbatch):
                        c = i % cp
                        N.check(L.qd_packed_conv2d(N.ptr(x), nbatch, C, H, W, O, k, k, st, st, pd, pd, N.ptr(codes[c]), bits, N.ptr(alpha[c]),
                                                   N.ptr(beta[c]), N.ptr(pts), kpts, levels, BUCKET, N.ptr(bias), N.ptr(y), N.stream_ptr()))

                    def run_decode(i, x=x, tf32=True):
                        torch.backends.cudnn.allow_tf32 = tf32
                        scratch = torch.empty(O, C, k, k, device="cuda")   # freed after the call, as in PackedConv2d
                        decode(i % cp, scratch)
                        return F.conv2d(x, scratch, bias, st, pd)

                    def run_d(i, x=x):
                        torch.backends.cudnn.allow_tf32 = True
                        return F.conv2d(x, wf[i % cf], bias, st, pd)
                    fns = {"b_decode_tf32": run_decode, "c_decode_fp32": lambda i, x=x: run_decode(i, x, False), "d_resident_tf32": run_d}
                    launches = {"b_decode_tf32": max(args.launches, cp), "c_decode_fp32": max(args.launches, cp),
                                "d_resident_tf32": max(args.launches, cf)}
                    times = _graph_time(torch, fns, args.rounds, launches)
                    b_med = statistics.median(times["b_decode_tf32"])
                    a_floor_us = 2 * macs / FP32_PEAK * 1e6
                    if a_floor_us < b_med:
                        times.update(_graph_time(torch, {"a_packed_kernel": run_a}, args.rounds, {"a_packed_kernel": max(args.launches, cp)}))
                    torch.backends.cudnn.allow_tf32 = True
                    cell = {"shape": name, "C": C, "O": O, "H": H, "W": W, "k": k, "stride": st, "padding": pd, "batch": nbatch,
                            "bits": bits, "kind": kind, "macs": macs, "copies_packed": cp, "copies_float": cf}
                    for key, ts in sorted(times.items()):
                        med = statistics.median(ts)
                        cell[key] = {"us_median": round(med, 2), "us_min": round(min(ts), 2), "us_max": round(max(ts), 2)}
                        if key == "a_packed_kernel":
                            cell[key]["TFLOPs"] = round(2 * macs / med / 1e6, 2)
                            cell[key]["of_fp32_datasheet"] = round(2 * macs / med / 1e-6 / FP32_PEAK, 3)
                    if "a_packed_kernel" not in times:
                        cell["a_packed_kernel"] = {"skipped": f"67 TFLOP/s would take {a_floor_us:.1f} us > (b) {b_med:.1f} us"}
                    rows.append(cell)
                    print(f"{name:18s} N={nbatch:4d} {bits}b {kind:10s} MACs={macs:.3g} " +
                          "  ".join(f"{kk[0]}={v['us_median']:9.2f}" for kk, v in sorted(cell.items()) if isinstance(v, dict) and "us_median" in v),
                          flush=True)
                    del x, y
                del codes, alpha, beta, wf
                torch.cuda.empty_cache()
    return rows


def models(args, torch):
    """Whole-model forward, eval mode, attach_packed_ against unpack_, one CUDA graph per forward."""
    from quantized_distillation_b200 import codec
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet
    makes = {"student": lambda: cfm.ConvolForwardNet(**cfm.smallerModelSpec, useBatchNorm=True, useAffineTransformInBatchNorm=True).cuda(),
             "wrn_16_22": lambda: Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10).cuda()}
    out = []
    torch.backends.cudnn.allow_tf32 = True
    for name, make in makes.items():
        torch.manual_seed(0)
        pm = codec.pack_model(make(), 4, 256, quantize_first_and_last_layer=False, include_buffers=True)
        unpacked, attached = make().eval(), make().eval()
        codec.unpack_(pm, unpacked)
        torch.cuda.synchronize()
        mem0 = torch.cuda.memory_allocated()
        replaced = codec.attach_packed_(pm, attached)
        torch.cuda.synchronize()
        freed = mem0 - torch.cuda.memory_allocated()
        for nbatch in (1, 128):
            x = torch.randn(nbatch, 3, 32, 32, device="cuda")
            with torch.no_grad():
                times = _graph_time(torch, {"unpack_": lambda i: unpacked(x), "attach_packed_": lambda i: attached(x)}, args.rounds,
                                    {"unpack_": 5, "attach_packed_": 5})
            row = {"model": name, "batch": nbatch, "replaced_modules": len(replaced), "freed_bytes": freed}
            for key, ts in times.items():
                row[key] = {"us_median": round(statistics.median(ts), 1), "us_min": round(min(ts), 1), "us_max": round(max(ts), 1)}
            out.append(row)
            print(json.dumps(row), flush=True)
        del unpacked, attached, pm
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "packed_conv_bench.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--max-copies", type=int, default=256)
    ap.add_argument("--quick", action="store_true", help="two layers, batch 1 and 32: a rehearsal of the script")
    ap.add_argument("--no-models", action="store_true")
    ap.add_argument("--no-layers", action="store_true")
    args = ap.parse_args()

    import torch
    from quantized_distillation_b200 import _native as N
    from tools.packed_bench import card

    N.require_cuda()
    info = card()
    rows = [] if args.no_layers else layers(args, torch, N, info)
    whole = [] if args.no_models else models(args, torch)
    out = {"card": info, "card_after": card(), "bucket": BUCKET, "rounds": args.rounds, "max_copies": args.max_copies,
           "fp32_datasheet_flops": FP32_PEAK, "rows": rows, "models": whole}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(info))
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
