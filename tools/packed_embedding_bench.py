"""Times an embedding lookup two ways:
  (a) PackedEmbedding: qd_packed_embedding gathering rows straight from the packed codes,
  (b) F.embedding on a resident float32 table -- an unpacked model,
and gives (c), the rate of (a) over its algorithmic bytes: tokens*dim*(4 + bits/8) for the output and the codes, plus
8 bytes (alpha, beta) per bucket each gathered row touches.
Tables: the NMT default 50,000 x 500 and 10,000 x 256; 2, 4 and 8 bits, uniform and non-uniform; bucket 256 and None;
tokens 1, 64, 1,600 (64 sentences x 25), 16,384 and 262,144, uniformly random indices.

Every variant cycles through enough distinct table copies that its copies exceed twice the 50 MB L2, so that a call
rarely finds its rows left in L2 by the one before.  A timed unit is one CUDA graph of back-to-back calls over every
copy (at least `launches` calls; host launch cost excluded: this compares GPU time); rounds alternate every variant of
one (table, tokens) cell in the same process, and the table gives the median and range of the per-call time over the
rounds.  Then an NMT-shaped model (two 50,000 x 500 embeddings, two-layer LSTM encoder, LSTM decoder, generator tied
to the target embedding) is loaded with attach_packed_(..., embeddings=True) and the drop in allocated device memory
is recorded next to the float32 bytes of its tables.  The card name, power limit and SM clock are read in the same run.

    python -m tools.packed_embedding_bench [--out profiles/packed_embedding_bench.json] [--rounds 5] [--launches 20]"""
from __future__ import annotations

import argparse
import gc
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TABLES = [("nmt_50000x500", 50_000, 500), ("10000x256", 10_000, 256)]
TOKENS = [1, 64, 1600, 16_384, 262_144]
BITS = [2, 4, 8]
BUCKETS = [256, None]
L2_BYTES = 50 << 20


def _copies(nbytes):
    return max(2, min(4096, math.ceil(2 * L2_BYTES / max(nbytes, 1))))


def _touched_scale_bytes(idx, dim, n, bucket):
    """8 bytes (alpha, beta) per bucket each gathered row spans."""
    L = n if bucket is None or n < bucket else bucket
    first = idx * dim // L
    last = (idx * dim + dim - 1) // L
    return int(8 * (last - first + 1).sum())


def _time(graphs, launches, rounds):
    import torch
    times = {k: [] for k in graphs}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(rounds):
        for key, gr in graphs.items():
            gr.replay()                            # the copies the next replay reads are not all in L2
            ev[0].record()
            gr.replay()
            ev[1].record()
            torch.cuda.synchronize()
            times[key].append(ev[0].elapsed_time(ev[1]) * 1e3 / launches[key])
    return times


def _memory_drop(codec):
    import torch

    class NMT(torch.nn.Module):
        def __init__(self, v=50_000, d=500):
            super().__init__()
            self.src_emb = torch.nn.Embedding(v, d, padding_idx=1)
            self.tgt_emb = torch.nn.Embedding(v, d, padding_idx=1)
            self.encoder = torch.nn.LSTM(d, d, num_layers=2)
            self.decoder = torch.nn.LSTM(d, d, num_layers=2)
            self.generator = torch.nn.Linear(d, v)
            self.generator.weight = self.tgt_emb.weight

    torch.manual_seed(0)
    pm = codec.pack_model(NMT().cuda(), 2, 256, quantize_first_and_last_layer=True)
    net = NMT().cuda()
    table_bytes = 4 * (net.src_emb.weight.numel() + net.tgt_emb.weight.numel())
    params_bytes = 4 * sum(p.numel() for p in net.parameters())
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    names = codec.attach_packed_(pm, net, embeddings=True)
    gc.collect()
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    return {"replaced": names, "float32_params_MB": round(params_bytes / 1e6, 1), "float32_tables_MB": round(table_bytes / 1e6, 1),
            "allocated_drop_MB": round((before - after) / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "packed_embedding_bench.json"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="the small table, 2 bits, tokens {1, 1600}: a rehearsal of the script")
    args = ap.parse_args()

    import numpy as np
    import torch
    import torch.nn.functional as F
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    from tools.packed_bench import card

    N.require_cuda()
    info = card()
    tables, tokens, bits_list = (TABLES[1:], [1, 1600], [2]) if args.quick else (TABLES, TOKENS, BITS)
    rows = []
    for name, V, D in tables:
        n = V * D
        g = torch.Generator(device="cuda").manual_seed(0)
        cf = _copies(4 * n)
        wf = [torch.randn(V, D, device="cuda", generator=g) * 0.05 for _ in range(cf)]
        mods = {}                                  # (bits, kind, bucket) -> PackedEmbedding per copy
        for bits in bits_list:
            for kind in ("uniform", "nonuniform"):
                for bucket in BUCKETS:
                    nb = N.geometry(n, bucket or 0)[0]
                    cp = _copies((n * bits + 7) // 8 + 8 * nb)
                    pts = None if kind == "uniform" else torch.sort(torch.rand(1 << bits, device="cuda", generator=g)).values
                    mods[(bits, kind, bucket)] = [
                        codec.PackedEmbedding(codec.PackedEntry(
                            "w", (V, D), bits=bits, points=pts,
                            packed=torch.randint(0, 256, ((n * bits + 7) // 8,), dtype=torch.int32, device="cuda", generator=g).to(torch.uint8),
                            alpha=torch.rand(nb, device="cuda", generator=g) * 0.1, beta=torch.randn(nb, device="cuda", generator=g) * 0.05),
                            kind, 1 << bits, bucket) for _ in range(cp)]
        for t in tokens:
            idx = torch.randint(0, V, (t,), device="cuda", generator=g)
            idx_np = idx.cpu().numpy().astype(np.int64)
            variants = {"b_resident_embedding": (lambda c: F.embedding(idx, wf[c]), cf, 8 * t * D)}
            for (bits, kind, bucket), ms in mods.items():
                nbytes = t * D * (4 * 8 + bits) // 8 + _touched_scale_bytes(idx_np, D, n, bucket)
                variants[f"a_packed_{bits}b_{kind}_bucket{bucket}"] = (lambda c, ms=ms: ms[c](idx), len(ms), nbytes)
            graphs, launches = {}, {}
            with torch.no_grad():
                for key, (fn, ncopies, _) in variants.items():
                    fn(0)                                      # warm up
                    torch.cuda.synchronize()
                    launches[key] = max(args.launches, ncopies)   # every copy once per replay
                    gr = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(gr):
                        for i in range(launches[key]):
                            fn(i % ncopies)
                    graphs[key] = gr
            times = _time(graphs, launches, args.rounds)
            b_med = statistics.median(times["b_resident_embedding"])
            for key, ts in times.items():
                med = statistics.median(ts)
                nbytes = variants[key][2]
                rows.append({"table": name, "V": V, "D": D, "tokens": t, "variant": key, "us_median": round(med, 2),
                             "us_min": round(min(ts), 2), "us_max": round(max(ts), 2), "bytes": nbytes,
                             "GBps": round(nbytes / med / 1e3, 1), "vs_resident": round(med / b_med, 3)})
                print(f"{name:14s} tokens={t:7d} {key:40s} {med:10.2f} us [{min(ts):.2f}, {max(ts):.2f}]  "
                      f"{nbytes / med / 1e3:8.1f} GB/s  x{med / b_med:.3f} of (b)", flush=True)
            del graphs
        for ms in mods.values():
            for m in ms:
                assert m.invalid_index_count() == 0
        del wf, mods
        gc.collect()
        torch.cuda.empty_cache()
    memory = None if args.quick else _memory_drop(codec)
    out = {"card": info, "min_launches_per_graph": args.launches, "rounds": args.rounds, "rows": rows, "attach_memory": memory}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(info))
    print(json.dumps(memory))
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
