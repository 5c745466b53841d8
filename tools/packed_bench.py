"""Times fixed-width storage.  (1) The fused quantize-and-pack encoder (qd_uniform_fwd_packed) against the level op
followed by qd_pack_indices at 2^26 floats, bucket 256, 2 and 4 bits.  (2) On WRN-16-22 (82.7 M parameters with
weight-like values, 2 bits, bucket 256, first and last layer float32): the whole-model unpack (qd_unpack_dequant_model)
against the per-tensor unpack loop and the whole-model Huffman decode (qd_huffman_decode_dequant_model) of the same
weights, then unpack_ and load_packed wall time.  Kernel times are CUDA events around back-to-back launches (median and
range over rounds); rates use the bytes each algorithm must move, computed from the shapes.  Writes JSON with the card
name, power limit and SM clock read in the same run.

    python -m tools.packed_bench [--out profiles/packed_bench.json] [--rounds 7] [--launches 50]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = (x.strip() for x in out.split(","))
        return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return {"gpu": "unknown", "power_limit": f"unknown ({type(e).__name__})"}


def events(fn, launches, rounds):
    """Per-launch microseconds of `fn` (median, min, max over rounds of `launches` back-to-back calls)."""
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    us = []
    for _ in range(rounds):
        ev[0].record()
        for _ in range(launches):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        us.append(ev[0].elapsed_time(ev[1]) * 1e3 / launches)
    return {"us_median": round(statistics.median(us), 2), "us_min": round(min(us), 2), "us_max": round(max(us), 2)}


def wall(fn, rounds):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return {"s_median": round(statistics.median(ts), 4), "s_min": round(min(ts), 4), "s_max": round(max(ts), 4)}


def with_rate(t, nbytes):
    t["bytes"] = int(nbytes)
    t["GBps_median"] = round(nbytes / (t["us_median"] * 1e-6) / 1e9, 1)
    return t


def encoder(launches, rounds, n=1 << 26, bucket=256):
    import torch
    from quantized_distillation_b200 import _native as N
    lib, sp = N.lib(), N.stream_ptr()
    x = torch.randn(n, generator=torch.Generator(device="cuda").manual_seed(0), device="cuda") * 0.05
    rows = N.geometry(n, bucket)[0]
    alpha, beta = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
    idx = torch.empty(n, dtype=torch.uint8, device="cuda")
    ws = torch.empty(int(lib.qd_packed_workspace_bytes(n, bucket)), dtype=torch.uint8, device="cuda")
    out = {}
    for bits, s in ((2, 4), (4, 16)):
        packed = torch.empty((n * bits + 7) // 8, dtype=torch.uint8, device="cuda")
        ref = torch.empty_like(packed)

        def fused():
            N.check(lib.qd_uniform_fwd_packed(N.ptr(x), N.ptr(packed), bits, N.ptr(alpha), N.ptr(beta), n, bucket, s, N.ptr(ws), ws.numel(), sp))

        def levels():
            N.check(lib.qd_uniform_fwd(N.ptr(x), None, N.ptr(idx), N.ptr(alpha), N.ptr(beta), None, None, n, bucket, s, None, 0.0, 0, 0, 0,
                                       N.ptr(ws), ws.numel(), sp))

        def pack():
            N.check(lib.qd_pack_indices(N.ptr(idx), N.ptr(ref), n, bits, sp))

        def two_step():
            levels()
            pack()
        two_step()
        fused()
        assert torch.equal(packed, ref), "fused encoder and levels + pack disagree"
        scales = 8 * rows
        out[f"{bits}bit"] = {
            "fused": with_rate(events(fused, launches, rounds), 4 * n + n * bits // 8 + scales),
            "levels_then_pack": with_rate(events(two_step, launches, rounds), 4 * n + n + scales + n + n * bits // 8),
            "levels_alone": with_rate(events(levels, launches, rounds), 4 * n + n + scales),
            "pack_alone": with_rate(events(pack, launches, rounds), n + n * bits // 8),
        }
        out[f"{bits}bit"]["fused_speedup"] = round(out[f"{bits}bit"]["levels_then_pack"]["us_median"] / out[f"{bits}bit"]["fused"]["us_median"], 2)
    return {"n": n, "bucket": bucket, "variants": out}


def model(launches, rounds, numBits=2, bucket=256):
    import torch
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet
    torch.manual_seed(0)
    make = lambda: Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10).cuda()   # noqa: E731
    net = make()
    with torch.no_grad():
        for p in net.parameters():
            p.normal_(0, 0.05)
    pm = codec.pack_model(net, numBits, bucket_size=bucket, quantize_first_and_last_layer=False, include_buffers=True)
    cm = codec.compress_model(net, numBits, bucket_size=bucket, quantize_first_and_last_layer=False)
    fresh = make()
    outs = [p.data for p in fresh.parameters()]
    dev = outs[0].device
    items = [(t, d) for t, d in zip(pm.tensors, outs) if t.quantized]
    args, keep = codec._decode_args(pm, items, dev, codec._mover(pm, dev))
    h_items = [(t, d) for t, d in zip(cm.tensors, outs) if t.quantized]
    h_args, h_keep = codec._decode_args(cm, h_items, dev, codec._mover(cm, dev))
    lib, sp, s = N.lib(), N.stream_ptr(), 2 ** numBits

    def per_tensor():
        for t, d in items:
            N.check(lib.qd_unpack_dequant_uniform(N.ptr(t.packed), t.bits, N.ptr(t.alpha), N.ptr(t.beta), N.ptr(d), t.numel, bucket, s, sp))

    n_q = sum(t.numel for t, _ in items)
    nbytes = sum(t.packed.numel() + 8 * t.alpha.numel() + 4 * t.numel for t, _ in items)
    res = {
        "quantized_tensors": len(items), "quantized_parameters": n_q,
        "model_unpack": with_rate(events(lambda: N.check(lib.qd_unpack_dequant_model(*args)), launches, rounds), nbytes),
        "per_tensor_unpack_loop": with_rate(events(per_tensor, launches, rounds), nbytes),
        "huffman_model_decode": events(lambda: N.check(lib.qd_huffman_decode_dequant_model(*h_args)), launches, rounds),
    }
    want = [d.clone() for _, d in items]
    N.check(lib.qd_unpack_dequant_model(*args))
    assert all(torch.equal(a, d) for a, (_, d) in zip(want, items)), "model unpack and Huffman decode disagree"
    del keep, h_keep
    res["unpack_"] = wall(lambda: codec.unpack_(pm, fresh), rounds)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "wrn.qdp")
        res["file_bytes"] = codec.save_packed(pm, path)
        res["load_packed_host"] = wall(lambda: codec.load_packed(path), rounds)         # file in the page cache after the first
        res["load_packed_cuda"] = wall(lambda: codec.load_packed(path, device="cuda"), rounds)
        back = codec.load_packed(path)
        res["unpack_from_host_file"] = wall(lambda: codec.unpack_(back, fresh), rounds)
    res["size_breakdown"] = pm.size_breakdown()
    res["huffman_size_breakdown"] = cm.size_breakdown()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "packed_bench.json"))
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--launches", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("packed_bench needs a CUDA device")
    before = card()
    res = {"card": before, "encoder": encoder(a.launches, a.rounds), "wrn_16_22_2bit_bucket256": model(a.launches, a.rounds)}
    res["card_after"] = card()
    res["timing"] = ("kernel rows: CUDA events around `launches` back-to-back calls, per-launch median / min / max over `rounds`; "
                     "s_* rows: host wall time around the call, synchronised")
    res["launches"], res["rounds"] = a.launches, a.rounds
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
