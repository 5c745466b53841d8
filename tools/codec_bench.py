"""Times the Huffman-coded model container on the WRN-16-22 student (reference config 3, 82.7 M parameters with
weight-like values, 2 bits, bucket 256, first and last layer float32): compress_model, save, load_compressed to the
device, decompress_ (one whole-model decode launch) against the per-tensor decode loop it replaces and against the
whole-model decode call alone, with the file's size breakdown next to what get_size_quantized_model reports.  Writes
JSON with the card name and power limit read in the same run.

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
    # what decompress_ did before the whole-model launch: one per-tensor decode launch after the other
    outs = [p.data for p in fresh.parameters()]
    t_per_tensor = timed(lambda: [codec.decompress_tensor(cm, k, out=d) for k, d in enumerate(outs)], reps)
    # the whole-model call alone (descriptor copy + one kernel), CUDA events over repeated calls
    from quantized_distillation_b200 import _native as N
    dev = outs[0].device
    items = [(t, d) for t, d in zip(cm.tensors, outs) if t.quantized]
    args, keep = codec._decode_args(cm, items, dev, codec._mover(cm, dev))
    launches = 50
    for _ in range(5):
        N.check(N.lib().qd_huffman_decode_dequant_model(*args))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    kernel_ms = []
    for _ in range(reps):
        ev[0].record()
        for _ in range(launches):
            N.check(N.lib().qd_huffman_decode_dequant_model(*args))
        ev[1].record()
        torch.cuda.synchronize()
        kernel_ms.append(ev[0].elapsed_time(ev[1]) / launches)
    per_tensor_chunks = [-(-t.numel // codec.HUFFMAN_CHUNK) for t, _ in items]
    chunks = sum(per_tensor_chunks)
    ctas = sum(-(-c // 128) for c in per_tensor_chunks)          # 128 chunks (one per thread) per CTA
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "wrn.qdh")
        t0 = time.perf_counter()
        size = codec.save_compressed(cm, path)
        t_save = time.perf_counter() - t0
        t_load = timed(lambda: codec.load_compressed(path, device="cuda"), reps)     # file in the page cache after the first
        back = codec.load_compressed(path, device="cuda")
    qf = lambda t: Q.uniformQuantization(t, 2 ** numBits, bucket_size=bucket)   # noqa: E731
    ref_mb = codec.get_size_quantized_model(model, numBits, qf, bucket_size=bucket, quantizeFirstLastLayer=False)
    count_q = sum(p.numel() for p in params[1:-1])
    weights = sum(p.numel() for p in params)
    sb = back.size_breakdown()
    res = dict(card(), model="Wide_ResNet(16, 22)", parameters=weights, quantized_parameters=count_q, numBits=numBits, bucket=bucket,
               compress_model_s=round(t_compress, 4), decompress_s=round(t_decompress, 4),
               per_tensor_decode_loop_s=round(t_per_tensor, 4), loop_over_decompress=round(t_per_tensor / t_decompress, 2),
               model_decode_call_us=round(sorted(kernel_ms)[len(kernel_ms) // 2] * 1e3, 1), model_decode_calls_per_rep=launches,
               quantized_tensors=len(items), chunks=chunks, ctas=ctas,
               save_s=round(t_save, 4), load_to_device_s=round(t_load, 4),
               decompress_GBps_out=round(weights * 4 / t_decompress / 1e9, 1), file_bytes=size,
               get_size_quantized_model_MB=ref_mb, file_MB=size / 1e6, size_breakdown=sb,
               code_bits_per_weight=sb["code_bits"] / count_q,
               overhead_fraction=(sb["chunk_index_bytes"] + sb["padding_bits"] / 8 + sb["header_bytes"] + sb["alignment_bytes"]) / size,
               reps=reps, timing="median host wall time around the call, synchronised; model_decode_call_us: median over reps of "
                                 "CUDA events around model_decode_calls_per_rep back-to-back qd_huffman_decode_dequant_model calls")
    del keep
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
