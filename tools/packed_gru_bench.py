"""Times the recurrent layers of the NMT model built with rnn_type GRU three ways, per step:
  (a) packed: PackedGRU (one qd_packed_gru_layer call, one fused cell launch per step) / PackedGRUCell,
  (b) nn.GRU / nn.GRUCell on resident float32 weights (cuDNN / cuBLAS, TF32 off: the setting is recorded),
  (c) decode + torch: the same packed modules forced onto their fallback (decode both weights, then torch's GRU).
Shapes: the encoder layer (I = H = 500) over T = 50 steps, and the decoder's input-feeding cells 1000 -> 500 and
500 -> 500; batch 1, 5, 30 and 64; weights at 2 bits, uniform, bucket 256.  Every matrix fits in the 50 MB L2, as it
does when a decoder steps through a sentence.  A timed unit is one CUDA graph of `launches` back-to-back calls (host
launch cost excluded); rounds alternate the three arms of one cell in the same process and the table gives the median
and range of the per-step time.  The floor of one launch is measured on a 1 x 8 -> 8 cell and a 1 x 8 -> 32
qd_packed_linear.  Then an NMT-shaped GRU model (two 50,000 x 500 embeddings, a two-layer bidirectional GRU encoder of
2 x 250, a StackedGRU decoder of nn.GRUCell 1000 -> 500 and 500 -> 500, a 1000 -> 500 attention Linear, a tied
generator) is loaded with attach_packed_(..., embeddings=True) and with gru=True as well, and the drops in allocated
device memory are recorded.  The card name, power limit and SM clock are read in the same run.

    python -m tools.packed_gru_bench [--out profiles/packed_gru_bench.json] [--rounds 5] [--launches 20] [--quick]"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

BATCHES = [1, 5, 30, 64]
STEPS = 50


def _packed_weight(codec, N, rows, cols, g, bits=2, bucket=256):
    import torch
    n = rows * cols
    nb = N.geometry(n, bucket)[0]
    return codec.PackedEntry("w", (rows, cols), bits=bits,
                             packed=torch.randint(0, 256, ((n * bits + 7) // 8,), dtype=torch.int32, device="cuda", generator=g).to(torch.uint8),
                             alpha=torch.rand(nb, device="cuda", generator=g) * 0.1 / cols ** 0.5,
                             beta=-torch.rand(nb, device="cuda", generator=g) * 0.05 / cols ** 0.5)


def _time(graphs, launches, rounds):
    import torch
    times = {k: [] for k in graphs}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(rounds):
        for key, gr in graphs.items():
            gr.replay()
            ev[0].record()
            gr.replay()
            ev[1].record()
            torch.cuda.synchronize()
            times[key].append(ev[0].elapsed_time(ev[1]) * 1e3 / launches)
    return times


def _graph(fn, launches):
    import torch
    fn()
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for _ in range(launches):
            fn()
    return gr


def _memory_drop(codec):
    import torch

    class NMT(torch.nn.Module):
        def __init__(self, v=50_000, d=500):
            super().__init__()
            self.src_emb = torch.nn.Embedding(v, d, padding_idx=1)
            self.tgt_emb = torch.nn.Embedding(v, d, padding_idx=1)
            self.encoder = torch.nn.GRU(d, d // 2, num_layers=2, bidirectional=True)
            self.cells = torch.nn.ModuleList([torch.nn.GRUCell(2 * d, d), torch.nn.GRUCell(d, d)])
            self.attn = torch.nn.Linear(2 * d, d, bias=False)
            self.generator = torch.nn.Linear(d, v)
            self.generator.weight = self.tgt_emb.weight

    torch.manual_seed(0)
    pm = codec.pack_model(NMT().cuda(), 2, 256, quantize_first_and_last_layer=True)
    out = {}
    for gru in (False, True):
        net = NMT().cuda()
        rec_bytes = 4 * sum(p.numel() for n, p in net.named_parameters() if n.startswith(("encoder", "cells")) and p.dim() == 2)
        gc.collect()
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        names = codec.attach_packed_(pm, net, embeddings=True, gru=gru)
        gc.collect()
        torch.cuda.synchronize()
        after = torch.cuda.memory_allocated()
        out["gru" if gru else "embeddings_only"] = {"replaced": names, "allocated_drop_MB": round((before - after) / 1e6, 2)}
        out["float32_recurrent_weights_MB"] = round(rec_bytes / 1e6, 2)
        del net
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "packed_gru_bench.json"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="batch 1 and 64 only, no memory model: a rehearsal of the script")
    args = ap.parse_args()

    import torch
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    from tools.packed_bench import card

    N.require_cuda()
    info = card()
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    batches = [1, 64] if args.quick else BATCHES
    shapes = [("encoder_layer_500x500", "layer", 500, 500), ("decoder_cell_1000x500", "cell", 1000, 500),
              ("decoder_cell_500x500", "cell", 500, 500)]
    with torch.no_grad():
        for name, what, I, H in shapes:
            e_ih, e_hh = _packed_weight(codec, N, 3 * H, I, g), _packed_weight(codec, N, 3 * H, H, g)
            b = (torch.randn(3 * H, device="cuda", generator=g) * 0.1, torch.randn(3 * H, device="cuda", generator=g) * 0.1)
            if what == "layer":
                packed = codec.PackedGRU([(e_ih, e_hh)], "uniform", 4, 256, biases=[b]).eval()
                slow = codec.PackedGRU([(e_ih, e_hh)], "uniform", 4, 256, biases=[b]).eval()
                ref = torch.nn.GRU(I, H).cuda().eval()
                w = packed.decoded_weights()
            else:
                packed = codec.PackedGRUCell(e_ih, e_hh, "uniform", 4, 256, *b)
                slow = codec.PackedGRUCell(e_ih, e_hh, "uniform", 4, 256, *b)
                ref = torch.nn.GRUCell(I, H).cuda()
                w = list(packed.decoded_weights()) + list(b)
            packed.CROSSOVER_ROWS = N.PACKED_GRU_MAX_ROWS          # always the kernel
            slow.CROSSOVER_ROWS = 0                                 # always the decode + torch fallback
            for p, v in zip(ref.parameters(), w):
                p.copy_(v)
            for B in batches:
                if what == "layer":
                    x = torch.randn(STEPS, B, I, device="cuda", generator=g)
                    arms = {"a_packed": lambda: packed(x), "b_resident_float32": lambda: ref(x), "c_decode_torch": lambda: slow(x)}
                    per = STEPS
                else:
                    x = torch.randn(B, I, device="cuda", generator=g)
                    hx = torch.randn(B, H, device="cuda", generator=g)
                    arms = {"a_packed": lambda: packed(x, hx), "b_resident_float32": lambda: ref(x, hx), "c_decode_torch": lambda: slow(x, hx)}
                    per = 1
                graphs = {}
                for k, fn in arms.items():
                    try:
                        graphs[k] = _graph(fn, args.launches)
                    except RuntimeError as e:             # an arm torch cannot capture is reported, not timed
                        print(f"{name} batch={B} {k}: not captured ({str(e)[:120]})", flush=True)
                        rows.append({"shape": name, "batch": B, "arm": k, "error": str(e)[:200]})
                        torch.cuda.synchronize()
                times = _time(graphs, args.launches, args.rounds)
                b_med = statistics.median(times["b_resident_float32"])
                for key, ts in times.items():
                    med = statistics.median(ts) / per
                    rows.append({"shape": name, "batch": B, "steps": per, "arm": key, "us_per_step_median": round(med, 2),
                                 "us_per_step_min": round(min(ts) / per, 2), "us_per_step_max": round(max(ts) / per, 2),
                                 "vs_resident": round(med * per / b_med, 3)})
                    print(f"{name:24s} batch={B:3d} {key:20s} {med:9.2f} us/step [{min(ts) / per:.2f}, {max(ts) / per:.2f}]  "
                          f"x{med * per / b_med:.3f} of (b)", flush=True)
                del graphs
        # the floor of one launch: the smallest cell, and qd_packed_linear at the same scale
        e_ih, e_hh = _packed_weight(codec, N, 24, 8, g), _packed_weight(codec, N, 24, 8, g)
        tiny = codec.PackedGRUCell(e_ih, e_hh, "uniform", 4, 256)
        tiny.CROSSOVER_ROWS = N.PACKED_GRU_MAX_ROWS
        lin = codec.PackedLinear(_packed_weight(codec, N, 32, 8, g), "uniform", 4, 256)
        x = torch.randn(1, 8, device="cuda")
        hx = torch.zeros(1, 8, device="cuda")
        graphs = {"cell_1x8_to_8": _graph(lambda: tiny(x, hx), args.launches), "linear_1x8_to_32": _graph(lambda: lin(x), args.launches)}
        floor = {k: round(statistics.median(v), 2) for k, v in _time(graphs, args.launches, args.rounds).items()}
        print("floor us per call:", json.dumps(floor), flush=True)
        del graphs
    gc.collect()
    torch.cuda.empty_cache()
    memory = None if args.quick else _memory_drop(codec)
    out = {"card": info, "tf32": False, "launches_per_graph": args.launches, "rounds": args.rounds, "rows": rows, "launch_floor_us": floor,
           "attach_memory": memory}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(info))
    print(json.dumps(memory))
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
