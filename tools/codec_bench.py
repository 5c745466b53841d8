"""Times the Huffman-coded model container on the WRN-16-22 student (reference config 3, 82.7 M parameters with
weight-like values, 2 bits, bucket 256, first and last layer float32): compress_model, save/load, decompress_, with the file's
size breakdown next to what get_size_quantized_model reports.  Writes JSON with the card name and power limit
read in the same run.

    python -m tools.codec_bench [--out profiles/codec_bench.json] [--reps 5]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return {"gpu": "unknown", "power_limit": f"unknown ({type(e).__name__})"}


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2]


def run(out_path, reps, numBits=2, bucket=256):
    import torch
    import quantized_distillation_b200.quantization as Q
    from quantized_distillation_b200 import codec
    from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet
    torch.manual_seed(0)
    model = Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10).cuda()
    params = list(model.parameters())
    with torch.no_grad():           # weight-like values (randn * 0.05): at the uniform initialisation all levels are equally likely
        for p in params:
            p.normal_(0, 0.05)
    cm = codec.compress_model(model, numBits, bucket_size=bucket, quantize_first_and_last_layer=False)
    t_compress = timed(lambda: codec.compress_model(model, numBits, bucket_size=bucket, quantize_first_and_last_layer=False), reps)
    fresh = Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10).cuda()
    t_decompress = timed(lambda: codec.decompress_(cm, fresh), reps)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "wrn.qdh")
        t0 = time.perf_counter()
        size = codec.save_compressed(cm, path)
        t_save = time.perf_counter() - t0
        t0 = time.perf_counter()
        back = codec.load_compressed(path, device="cuda")
        torch.cuda.synchronize()
        t_load = time.perf_counter() - t0
    qf = lambda t: Q.uniformQuantization(t, 2 ** numBits, bucket_size=bucket)   # noqa: E731
    ref_mb = codec.get_size_quantized_model(model, numBits, qf, bucket_size=bucket, quantizeFirstLastLayer=False)
    count_q = sum(p.numel() for p in params[1:-1])
    weights = sum(p.numel() for p in params)
    sb = back.size_breakdown()
    res = dict(card(), model="Wide_ResNet(16, 22)", parameters=weights, quantized_parameters=count_q, numBits=numBits, bucket=bucket,
               compress_model_s=round(t_compress, 4), decompress_s=round(t_decompress, 4), save_s=round(t_save, 4), load_s=round(t_load, 4),
               decompress_GBps_out=round(weights * 4 / t_decompress / 1e9, 1), file_bytes=size,
               get_size_quantized_model_MB=ref_mb, file_MB=size / 1e6, size_breakdown=sb,
               code_bits_per_weight=sb["code_bits"] / count_q,
               overhead_fraction=(sb["chunk_index_bytes"] + sb["padding_bits"] / 8 + sb["header_bytes"] + sb["alignment_bytes"]) / size,
               reps=reps, timing="median host wall time around the call, synchronised")
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)
    return res


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "codec_bench.json"))
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(run(a.out, a.reps), indent=1))
