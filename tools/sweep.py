"""Per-op / per-size throughput table (BASELINE.json config 5: synthetic weight-tensor
sweep, uniform + non-uniform fwd/bwd, GB/s vs the H100 HBM roofline).

    python -m tools.sweep [--out gpurun_out/sweep.json] [--max-log2 28]

Each row: CUDA-event time per launch (inputs resident in HBM, 3 warm-ups, buffers
rotated so that consecutive launches never touch the same cache lines when the
tensor is smaller than L2), algorithmic bytes (SURVEY.md section 8d), GB/s and the
fraction of the HBM peak (measured copy peak when MEASURED_PEAKS.json is present,
the H100 SXM data sheet's 3.35 TB/s otherwise)."""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def run(dev=None, out_path=None, max_log2=28, min_log2=10, only=None):
    import torch
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    dev = dev or torch.device("cuda", torch.cuda.current_device())
    lib = N.lib()
    peak = 3350.0
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peak = float(json.load(open(pk))["hbm_gbs"])
    sp = N.stream_ptr(dev)
    rows = []
    L2_BYTES = 50 << 20

    def timeit(fn, nbuf, iters):
        for i in range(3):
            fn(i % nbuf)
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            fn(i % nbuf)
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) / iters * 1e-3

    for lg in range(min_log2, max_log2 + 1, 2):
        n = 1 << lg
        per_set = n * 4 * 4
        nbuf = max(1, min(8, (2 * L2_BYTES) // per_set + 1)) if per_set < 2 * L2_BYTES else 1
        iters = 200 if lg <= 20 else (50 if lg <= 24 else 10)
        gen = torch.Generator(device=dev).manual_seed(lg)
        xs = [torch.randn(n, generator=gen, device=dev) * 0.05 for _ in range(nbuf)]
        gs = [torch.randn(n, generator=gen, device=dev) for _ in range(nbuf)]
        qs = [torch.empty(n, device=dev) for _ in range(nbuf)]
        gos = [torch.empty(n, device=dev) for _ in range(nbuf)]
        idx = [torch.empty(n, dtype=torch.uint8, device=dev) for _ in range(nbuf)]
        pts4 = torch.linspace(0, 1, 4, device=dev)
        pts16 = torch.linspace(0, 1, 16, device=dev)
        pts8 = torch.linspace(0, 1, 8, device=dev)
        gp = torch.empty(16, device=dev)
        for bucket in (256, 0):
            ws = N.workspace(n, bucket, dev)
            rws, rlen, _ = N.geometry(n, bucket)
            alpha = torch.ones(rws, device=dev)
            beta = torch.zeros(rws, device=dev)
            ops = {
                "uniform_fwd": (8 if bucket else (12 if n > 49152 else 8), lambda i: N.check(lib.qd_uniform_fwd(
                    N.ptr(xs[i]), N.ptr(qs[i]), None, None, None, None, None, n, bucket, 16, None, 0.0, 0, 0, 0, N.ptr(ws), ws.numel(), sp))),
                "uniform_fwd_bwd_ste": (16 if bucket or n <= 49152 else 20, lambda i: N.check(lib.qd_uniform_fwd_bwd(
                    N.ptr(xs[i]), N.ptr(gs[i]), N.ptr(qs[i]), N.ptr(gos[i]), n, bucket, 16, N.BWD_STE, N.ptr(ws), ws.numel(), sp))),
                "uniform_fwd_bwd_truncated": (16 if bucket or n <= 49152 else 20, lambda i: N.check(lib.qd_uniform_fwd_bwd(
                    N.ptr(xs[i]), N.ptr(gs[i]), N.ptr(qs[i]), N.ptr(gos[i]), n, bucket, 16, N.BWD_TRUNCATED, N.ptr(ws), ws.numel(), sp))),
                "nonuniform_fwd_K4_midpoint_u8": (9 if bucket or n <= 49152 else 13, lambda i: N.check(lib.qd_nonuniform_fwd(
                    N.ptr(xs[i]), N.ptr(pts4), 4, N.RULE_MIDPOINT, N.ptr(qs[i]), N.ptr(idx[i]), None, None, None, n, bucket, None, 0.0,
                    N.ptr(ws), ws.numel(), sp))),
                "nonuniform_fwd_K16_nearest_u8": (9 if bucket or n <= 49152 else 13, lambda i: N.check(lib.qd_nonuniform_fwd(
                    N.ptr(xs[i]), N.ptr(pts16), 16, N.RULE_NEAREST, N.ptr(qs[i]), N.ptr(idx[i]), None, None, None, n, bucket, None, 0.0,
                    N.ptr(ws), ws.numel(), sp))),
                "nonuniform_fwd_K8_nearest_u8": (9 if bucket or n <= 49152 else 13, lambda i: N.check(lib.qd_nonuniform_fwd(
                    N.ptr(xs[i]), N.ptr(pts8), 8, N.RULE_NEAREST, N.ptr(qs[i]), N.ptr(idx[i]), None, None, None, n, bucket, None, 0.0,
                    N.ptr(ws), ws.numel(), sp))),
                "nonuniform_fwd_K16_midpoint_u8": (9 if bucket or n <= 49152 else 13, lambda i: N.check(lib.qd_nonuniform_fwd(
                    N.ptr(xs[i]), N.ptr(pts16), 16, N.RULE_MIDPOINT, N.ptr(qs[i]), N.ptr(idx[i]), None, None, None, n, bucket, None, 0.0,
                    N.ptr(ws), ws.numel(), sp))),
                "nonuniform_bwd_K4_u8": (5, lambda i: N.check(lib.qd_nonuniform_bwd(
                    N.ptr(gs[i]), N.ptr(idx[i]), None, N.ptr(alpha), 4, N.ptr(gp), n, bucket, N.ptr(ws), ws.numel(), sp))),
                "nonuniform_bwd_K16_u8": (5, lambda i: N.check(lib.qd_nonuniform_bwd(
                    N.ptr(gs[i]), N.ptr(idx[i]), None, N.ptr(alpha), 16, N.ptr(gp), n, bucket, N.ptr(ws), ws.numel(), sp))),
            }
            if bucket:
                # helper entry points (scaling alone, pre-scaled index search, packed codec)
                xh = [torch.empty(rws * rlen, device=dev) for _ in range(nbuf)]
                packed = torch.empty((n * 4 + 7) // 8, dtype=torch.uint8, device=dev)
                ops["scale_down"] = (8, lambda i: N.check(lib.qd_scale_down(
                    N.ptr(xs[i]), N.ptr(xh[i]), N.ptr(alpha), N.ptr(beta), None, None, n, bucket, None, 0.0, N.ptr(ws), ws.numel(), sp)))
                ops["inv_scale_down"] = (8, lambda i: N.check(lib.qd_inv_scale_down(
                    N.ptr(xh[i]), N.ptr(qs[i]), N.ptr(alpha), N.ptr(beta), None, n, bucket, sp)))
                ops["centroid_index_K4_u8"] = (5, lambda i: N.check(lib.qd_centroid_index(
                    N.ptr(xh[i]), N.ptr(pts4), 4, N.RULE_MIDPOINT, N.ptr(idx[i]), None, None, n, sp)))
                ops["pack_4bit"] = (1.5, lambda i: N.check(lib.qd_pack_indices(N.ptr(idx[i]), N.ptr(packed), n, 4, sp)))
                ops["unpack_dequant_uniform_4bit"] = (4.5, lambda i: N.check(lib.qd_unpack_dequant_uniform(
                    N.ptr(packed), 4, N.ptr(alpha), N.ptr(beta), N.ptr(qs[i]), n, bucket, 16, sp)))
                # write-only yardstick (torch's fill kernel, not ours): what a pure store stream reaches on this part
                ops["yardstick_fill_torch"] = (4, lambda i: qs[i].fill_(1.0))
                ops["yardstick_copy_torch"] = (8, lambda i: qs[i].copy_(xs[i]))
                packed2 = torch.empty((n * 2 + 7) // 8, dtype=torch.uint8, device=dev)
                ops["pack_2bit"] = (1.25, lambda i: N.check(lib.qd_pack_indices(N.ptr(idx[i]), N.ptr(packed2), n, 2, sp)))
                ops["unpack_dequant_nonuniform_4bit"] = (4.5, lambda i: N.check(lib.qd_unpack_dequant_nonuniform(
                    N.ptr(packed), 4, N.ptr(pts16), 16, N.ptr(alpha), N.ptr(beta), N.ptr(qs[i]), n, bucket, sp)))
                # Huffman codec on the 16 levels of the weight-like xs[0]: the stream is made once, outside the timed
                # loop, and the algorithmic bytes come from its actual length (+ one uint32 offset per chunk)
                hidx, ha, hb = torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(rws, device=dev), torch.empty(rws, device=dev)
                N.check(lib.qd_uniform_fwd(N.ptr(xs[0]), None, N.ptr(hidx), N.ptr(ha), N.ptr(hb), None, None, n, bucket, 16, None, 0.0,
                                           0, 0, 0, N.ptr(ws), ws.numel(), sp))
                hcounts = torch.bincount(hidx, minlength=256).cpu().numpy()
                hlen = codec.huffman_code_lengths(hcounts)
                htab = torch.from_numpy(codec.huffman_table(hlen)).to(dev)
                hchunks = -(-n // codec.HUFFMAN_CHUNK)
                hcap = -(-int(sum(int(hcounts[s_]) * l_ for s_, l_ in hlen.items())) // 32) + hchunks
                hwords = torch.empty(hcap, dtype=torch.int32, device=dev)
                hoffs = torch.empty(hchunks, dtype=torch.int32, device=dev)
                htot = torch.zeros(1, dtype=torch.int64, device=dev)
                N.check(lib.qd_huffman_encode(N.ptr(hidx), n, N.ptr(htab), N.ptr(hwords), hcap, N.ptr(hoffs), N.ptr(htot), sp))
                hn = int(htot.item())
                hstream = (hn + hchunks) * 4 / n          # stream + chunk index bytes per element
                ops["huffman_encode_16lvl"] = (2 + hstream, lambda i: N.check(lib.qd_huffman_encode(
                    N.ptr(hidx), n, N.ptr(htab), N.ptr(hwords), hcap, N.ptr(hoffs), N.ptr(htot), sp)))
                ops["huffman_decode_dequant_uniform_16lvl"] = (4 + hstream, lambda i: N.check(lib.qd_huffman_decode_dequant_uniform(
                    N.ptr(hwords), hn, N.ptr(hoffs), N.ptr(htab), N.ptr(ha), N.ptr(hb), N.ptr(qs[i]),
                    n, bucket, 16, sp)))
                ops["uniform_fwd_bwd_minmax"] = (16, lambda i: N.check(lib.qd_uniform_fwd_bwd(
                    N.ptr(xs[i]), N.ptr(gs[i]), N.ptr(qs[i]), N.ptr(gos[i]), n, bucket, 16, N.BWD_MINMAX, N.ptr(ws), ws.numel(), sp)))
                ops["uniform_bwd_minmax"] = (12, lambda i: N.check(lib.qd_uniform_bwd(
                    N.ptr(xs[i]), N.ptr(gs[i]), N.ptr(gos[i]), n, bucket, 16, N.BWD_MINMAX, N.ptr(ws), ws.numel(), sp)))
            for i in range(nbuf):
                idx[i].random_(0, 4)
            for name, (bpe, fn) in ops.items():
                if only and not any(k in name for k in only):
                    continue
                sec = timeit(fn, nbuf, iters)
                gbs = n * bpe / sec / 1e9
                rows.append({"op": name, "n": n, "bucket": bucket or None, "us": round(sec * 1e6, 2), "bytes_per_elem": bpe,
                             "GBps": round(gbs, 1), "frac_measured_peak": round(gbs / peak, 4), "frac_8000": round(gbs / 8000.0, 4)})
        del xs, gs, qs, gos, idx
        torch.cuda.empty_cache()
    out_path = out_path or os.path.join(ROOT, "gpurun_out", "sweep.json")
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump({"peak_GBps": peak, "rows": rows}, f, indent=1)
    md = out_path.replace(".json", ".md")
    with open(md, "w") as f:
        f.write(f"| op | n | bucket | us/launch | B/elt | GB/s | frac of measured {peak:.0f} | frac of 8000 |\n|---|---|---|---|---|---|---|---|\n")
        for r in rows:
            f.write(f"| {r['op']} | 2^{r['n'].bit_length() - 1} | {r['bucket']} | {r['us']} | {r['bytes_per_elem']} | {r['GBps']} | "
                    f"{r['frac_measured_peak']} | {r['frac_8000']} |\n")
    return out_path


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--max-log2", type=int, default=28)
    ap.add_argument("--min-log2", type=int, default=10)
    ap.add_argument("--only", default="", help="comma-separated substrings: time only the ops whose name contains one of them")
    a = ap.parse_args()
    print(run(out_path=a.out, max_log2=a.max_log2, min_log2=a.min_log2, only=[k for k in a.only.split(",") if k]))
