"""Generates tests/golden/reference_nonfinite.npz: the UNMODIFIED reference (antspy/quantized_distillation,
mounted at /root/reference) run on non-uniform quantization inputs whose x_hat is NaN or infinite somewhere.
Companion of make_golden.py and make_golden_options.py; run in the build container only:

    python tests/golden/make_golden_nonfinite.py

What is executed, for every case:
  * quantization.nonUniformQuantization (direct path, nearest rule)                     (quant_functions.py:196-290)
  * quantization.nonUniformQuantization_variable(pre_process_tensors=True).forward, i.e. SearchSorted.query on the
    pre-processed tensor (midpoint rule)                                                 (:408-469, 509-573)

Inputs: bucketed tensors whose rows are, in a fixed mix, finite, hold a NaN, hold +inf, hold -inf, or hold -3e38 and
3e38 (finite values whose range overflows: alpha = +inf, and x_hat = inf/inf = NaN at the maximum); and one-row
tensors (bucket None) of each kind, large enough for the grid path of the kernels.  K in {3, 4, 5, 16, 33}; the
points are sorted, some with k_0 = 0 (0 * inf = NaN in q) and some below 0 or above 1.
"""
import os
import sys
import warnings

import numpy as np
import torch

REF = "/root/reference"
sys.path.insert(0, REF)
warnings.filterwarnings("ignore")
import quantization as Q  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_nonfinite.npz")
KINDS = ("finite", "nan", "posinf", "neginf", "overflow")
KS = (3, 4, 5, 16, 33)


def points(K, seed):
    rng = np.random.default_rng(seed)
    p = np.sort(rng.random(K) * 1.2 - 0.1).astype(np.float32)
    if K % 2 == 0:
        p[0] = 0.0
    return p


def poison(row, kind, rng):
    """Puts the non-finite (or overflowing) values of `kind` into `row` in place, at seeded positions."""
    if kind == "finite":
        return
    pos = rng.choice(row.size, size=min(3, row.size), replace=False)
    if kind == "nan":
        row[pos[0]] = np.nan
    elif kind == "posinf":
        row[pos[0]] = np.inf
    elif kind == "neginf":
        row[pos[0]] = -np.inf
    else:
        row[pos[0]], row[pos[1]] = np.float32(-3e38), np.float32(3e38)


def make_x(n, bucket, kinds, seed):
    """Values on a 1/64 grid (the fixture compresses well), then row r gets kinds[r % len(kinds)]."""
    rng = np.random.default_rng(seed)
    x = (rng.integers(-64, 65, n) / 64.0).astype(np.float32)
    row_len = n if bucket is None else bucket
    for r, start in enumerate(range(0, n, row_len)):
        poison(x[start:start + row_len], kinds[r % len(kinds)], rng)
    return x


def main():
    store, meta = {}, []
    ci = 0
    cases = []
    for K in KS:
        for b, n in ((256, 256 * 7 + 77), (3002, 3002 * 5 + 1001)):
            cases.append((K, b, n, ("finite", "nan", "posinf", "finite", "neginf", "overflow")))
    for K, kind in zip(KS, KINDS):                     # one row of 50,000 floats: the grid path of the kernels
        cases.append((K, None, 50000, (kind,)))
    for K, kind in zip(KS, KINDS[1:] + KINDS[:1]):     # and one row the warp path holds
        cases.append((K, None, 700, (kind,)))
    for K, b, n, kinds in cases:
        x = make_x(n, b, kinds, 500 + ci)
        pts = points(K, 900 + ci)
        xt, pt = torch.from_numpy(x.copy()), torch.from_numpy(pts.copy())
        q, idx, _ = Q.nonUniformQuantization(xt.clone(), pt, bucket_size=b)
        f = Q.nonUniformQuantization_variable(bucket_size=b, pre_process_tensors=True, tensor=xt.clone())
        qm = f.forward(None, pt)
        im = f.savedForBackward["indices"]
        key = f"c{ci}"
        store[key + "_x"] = x
        store[key + "_points"] = pts
        store[key + "_q_nearest"] = q.numpy().reshape(-1)
        store[key + "_idx_nearest"] = idx.numpy().reshape(-1).astype(np.uint8)
        store[key + "_q_midpoint"] = qm.numpy().reshape(-1)
        store[key + "_idx_midpoint"] = im.numpy().reshape(-1).astype(np.uint8)
        assert idx.max() < K and im.max() < K
        meta.append(("nonfinite", key, "+".join(kinds), n, -1 if b is None else b, K))
        ci += 1
    store["meta"] = np.array(["|".join(str(v) for v in m) for m in meta])
    np.savez_compressed(OUT, **store)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB;", len(meta), "cases; torch", torch.__version__, "numpy", np.__version__)


if __name__ == "__main__":
    main()
