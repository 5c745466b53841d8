"""Generates tests/golden/warp_traversal_minmax.npz: SHA-256 digests of q and gout from the fused uniform forward +
min/max backward (qd_uniform_fwd_bwd, levels 16, bucket 256) on the register warp path, for row counts around the
persistent grid the warp path used before it got one warp per row (132 SMs x 3 CTAs x 8 warps = 3168 rows on an H100
SXM), a ragged last row and an unaligned view.  The inputs are a fixed integer hash of the element index, so they need
no stored arrays and no random-number stream.  Needs a GPU; the digests were taken with the library at the commit
before that change, and tests/test_gpu_warp_traversal.py checks that today's library still produces the same bytes:

    python tests/golden/make_golden_warp_traversal.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "warp_traversal_minmax.npz")

LEVELS, BUCKET = 16, 256
OLD_GRID_ROWS = 132 * 3 * 8
# (elements, offset of the view in floats, seed); offset 1 makes every row 4-byte aligned only (scalar mapping)
CASES = [(256, 0, 1), (100 * 256, 0, 2), ((OLD_GRID_ROWS - 1) * 256, 0, 3), (OLD_GRID_ROWS * 256, 0, 4),
         ((OLD_GRID_ROWS + 1) * 256, 0, 5), ((2 * OLD_GRID_ROWS - 1) * 256, 0, 6), ((2 * OLD_GRID_ROWS + 1) * 256, 0, 7),
         ((OLD_GRID_ROWS + 1) * 256 - 100, 0, 8), ((OLD_GRID_ROWS + 1) * 256, 1, 9), (1000 * 256 + 1, 1, 10)]


def inputs(n, seed):
    """x: weight-like values in (-0.1, 0.1) with a per-row scale, g in (-1, 1); splitmix64 of (index, seed)."""
    with np.errstate(over="ignore"):
        i = np.arange(2 * n, dtype=np.uint64) + np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15)
        z = i * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    u = ((z >> np.uint64(40)).astype(np.float64) / float(1 << 24)).astype(np.float32)   # [0, 1), 24 bits
    scale = (1.0 + (np.arange(n) // BUCKET) % 7).astype(np.float32) / np.float32(70.0)
    x = ((u[:n] - np.float32(0.5)) * scale).astype(np.float32)
    g = (u[n:] * np.float32(2.0) - np.float32(1.0)).astype(np.float32)
    return x, g


def run_fused_minmax(x_np, g_np, offset):
    """q and gout of qd_uniform_fwd_bwd (min/max backward) on views that start `offset` floats into their buffers."""
    import torch
    from quantized_distillation_b200 import _native as N
    n = x_np.size
    xb = torch.zeros(n + offset, device="cuda")
    gb = torch.zeros(n + offset, device="cuda")
    qb = torch.zeros(n + offset, device="cuda")
    ob = torch.zeros(n + offset, device="cuda")
    x, g, q, go = (t[offset:] for t in (xb, gb, qb, ob))
    x.copy_(torch.from_numpy(x_np))
    g.copy_(torch.from_numpy(g_np))
    ws = N.workspace(n, BUCKET, x.device)
    N.check(N.lib().qd_uniform_fwd_bwd(N.ptr(x), N.ptr(g), N.ptr(q), N.ptr(go), n, BUCKET, LEVELS, N.BWD_MINMAX, N.ptr(ws),
                                       ws.numel(), N.stream_ptr()))
    return q.cpu().numpy(), go.cpu().numpy()


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).digest(), dtype=np.uint8)


def main():
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    qs, gs = [], []
    for n, offset, seed in CASES:
        x, g = inputs(n, seed)
        q, go = run_fused_minmax(x, g, offset)
        qs.append(digest(q))
        gs.append(digest(go))
    np.savez_compressed(OUT, cases=np.array(CASES, dtype=np.int64), q_sha256=np.stack(qs), gout_sha256=np.stack(gs))
    print("wrote", OUT, len(CASES), "cases")


if __name__ == "__main__":
    main()
