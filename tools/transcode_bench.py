"""Times the container transcoders on WRN-16-22 (2 bits) and the student (4 bits), bucket 256, first and last layer
float32, weight-like values (randn * 0.05):
- qd_huffman_decode_packed_model (stream -> fixed-width codes) against qd_huffman_decode_dequant_model (stream -> float32)
  on the same file: CUDA events around back-to-back launches, the two calls alternating round by round;
- pack_compressed and compress_packed, host wall time around a synchronised call, next to decompress_ and compress_model.
Writes JSON with the card name and power limit read in the same run.

    python -m tools.transcode_bench [--out profiles/transcode_bench.json] [--rounds 7] [--launches 50]"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.codec_bench import card, timed  # noqa: E402


def _models():
    import torch
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet

    def wrn():
        return Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10).cuda()

    def student():
        return cfm.ConvolForwardNet(**cfm.smallerModelSpec, useBatchNorm=True, useAffineTransformInBatchNorm=True).cuda()
    torch.manual_seed(0)
    return [("Wide_ResNet(16, 22)", wrn, 2), ("student", student, 4)]


def _repack_args(codec, N, cm, dev):
    """Arguments of qd_huffman_decode_packed_model for every quantized tensor of the device-resident ``cm``, as
    pack_compressed builds them, and the tensors they point into."""
    import torch
    q = [t for t in cm.tensors if t.quantized]
    desc, keep = np.zeros(len(q), codec._REPACK_TENSOR), []
    for k, t in enumerate(q):
        limit = int(cm.levels) if cm.kind == "uniform" else t.points.numel()
        bits = codec.bits_for(limit)
        packed = torch.empty((t.numel * bits + 7) // 8, dtype=torch.uint8, device=dev)
        desc[k] = (N.ptr(t.words) if t.words.numel() else 0, N.ptr(t.chunk_offsets), N.ptr(packed), t.words.numel(), t.numel, bits, limit)
        keep.append(packed)
    ws = torch.empty(int(N.lib().qd_huffman_repack_model_workspace_bytes(len(q))), dtype=torch.uint8, device=dev)
    bad = torch.zeros(len(q), dtype=torch.int64, device=dev)
    keep += [desc, ws, bad]
    return (desc.ctypes.data, len(q), N.ptr(cm.table(dev)), N.ptr(bad), N.ptr(ws), ws.numel(), N.stream_ptr(dev)), keep


def _events(fn, launches):
    import torch
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(launches):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / launches * 1e3      # microseconds per call


def run_one(name, make, numBits, bucket, rounds, launches, reps):
    import torch
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    model = make()
    with torch.no_grad():
        for p in model.parameters():
            p.normal_(0, 0.05)
    kw = dict(bucket_size=bucket, quantize_first_and_last_layer=False)
    cm = codec.compress_model(model, numBits, **kw)
    pm = codec.pack_compressed(cm)
    dev = next(model.parameters()).device
    fresh = make()
    outs = [p.data for p in fresh.parameters()]
    items = [(t, d) for t, d in zip(cm.tensors, outs) if t.quantized]
    deq_args, keep_d = codec._decode_args(cm, items, dev, codec._mover(cm, dev))
    pk_args, keep_p = _repack_args(codec, N, cm, dev)
    calls = {"packed": lambda: N.check(N.lib().qd_huffman_decode_packed_model(*pk_args)),
             "dequant": lambda: N.check(N.lib().qd_huffman_decode_dequant_model(*deq_args))}
    for fn in calls.values():                              # warm up both shapes
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    us = {k: [] for k in calls}
    for r in range(rounds):                                # alternate which call goes first
        order = ("packed", "dequant") if r % 2 == 0 else ("dequant", "packed")
        for k in order:
            us[k].append(_events(calls[k], launches))
    stats = {k: dict(median_us=round(float(np.median(v)), 1), min_us=round(min(v), 1), max_us=round(max(v), 1)) for k, v in us.items()}
    q = [t for t in cm.tensors if t.quantized]
    n_q = sum(t.numel for t in q)
    res = dict(model=name, numBits=numBits, bucket=bucket, quantized_parameters=n_q, quantized_tensors=len(q),
               stream_bytes=sum(t.words.numel() * 4 for t in q), packed_bytes=sum(t.packed.numel() for t in pm.tensors if t.quantized),
               float_bytes=n_q * 4,
               decode_packed_model=stats["packed"], decode_dequant_model=stats["dequant"],
               packed_over_dequant=round(stats["packed"]["median_us"] / stats["dequant"]["median_us"], 3),
               pack_compressed_ms=round(timed(lambda: codec.pack_compressed(cm), reps) * 1e3, 2),
               compress_packed_ms=round(timed(lambda: codec.compress_packed(pm), reps) * 1e3, 2),
               decompress_ms=round(timed(lambda: codec.decompress_(cm, fresh), reps) * 1e3, 2),
               compress_model_ms=round(timed(lambda: codec.compress_model(model, numBits, **kw), reps) * 1e3, 2))
    del keep_d, keep_p
    return res


def run(out_path, rounds, launches, reps, bucket=256):
    res = dict(card(), results=[run_one(name, make, b, bucket, rounds, launches, reps) for name, make, b in _models()],
               timing=f"kernel: CUDA events around {launches} back-to-back launches of one call, {rounds} rounds alternating the two "
                      "calls' order, median / min / max over rounds; *_ms: median of host wall time around the call followed by "
                      f"torch.cuda.synchronize(), {reps} repetitions after one warm-up")
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)
    return res


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "transcode_bench.json"))
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(run(a.out, a.rounds, a.launches, a.reps), indent=1))
