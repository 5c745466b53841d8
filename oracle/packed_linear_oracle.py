"""CPU oracle of the fully-connected layer on fixed-width packed weights (qd_packed_linear) -- TEST INFRASTRUCTURE ONLY.

The weights are the packed codec's: the code of element e of the flattened [out_features, in_features] weight sits
in byte e*bits/8 at bit (e*bits)%8 (qd_pack_indices), and q_e = (unit[code] * alpha_b) + beta_b, each op rounded to
float32, with b = e // row_len of the bucket geometry (buckets run over the flattened tensor, so they straddle output
rows whenever in_features is not a multiple of the bucket) and unit[c] = c / (s - 1) (uniform, float32 division) or
points[c] (non-uniform).  The product is then taken in float64: y = x @ q.T + bias, the reference the float32 kernel is
held to within a summation-order tolerance.
"""
from __future__ import annotations

import numpy as np

from .quant_oracle import bucket_geometry

F32 = np.float32


def unpack_codes(packed, n: int, bits: int) -> np.ndarray:
    """Codes of elements 0 .. n-1 (int64) from the qd_pack_indices layout."""
    packed = np.asarray(packed, dtype=np.uint8)
    e = np.arange(n, dtype=np.int64)
    bit = e * bits
    return ((packed[bit >> 3].astype(np.int64) >> (bit & 7)) & ((1 << bits) - 1)).astype(np.int64)


def unit_table(levels=None, points=None) -> np.ndarray:
    """Value in [0, 1] of every code: c / (levels - 1) in float32 (uniform) or the points themselves."""
    if (levels is None) == (points is None):
        raise ValueError("give levels (uniform) or points (non-uniform)")
    if points is not None:
        return np.asarray(points, dtype=F32).reshape(-1)
    return (np.arange(levels, dtype=F32) / F32(levels - 1)).astype(F32)


def dequantize(codes, alpha, beta, bucket_size, levels=None, points=None) -> np.ndarray:
    """q (float32, flattened) of the codes: unit[code] * alpha_b + beta_b, two float32 roundings."""
    codes = np.asarray(codes, dtype=np.int64).reshape(-1)
    unit = unit_table(levels, points)
    if codes.size and codes.max() >= unit.size:
        raise ValueError("a code has no level / point")
    _, row_len, _ = bucket_geometry(codes.size, bucket_size)
    b = np.arange(codes.size, dtype=np.int64) // row_len
    a = np.asarray(alpha, dtype=F32)[b]
    be = np.asarray(beta, dtype=F32)[b]
    return ((unit[codes] * a).astype(F32) + be).astype(F32)


def packed_linear(x, packed, bits: int, alpha, beta, out_features: int, in_features: int, bucket_size, levels=None,
                  points=None, bias=None):
    """(y, magnitude): y = x @ q.T (+ bias) in float64 for x of shape [m, in_features], and sum_k |x_k q_k| per
    element (the scale of the float32 summation error)."""
    n = out_features * in_features
    q = dequantize(unpack_codes(packed, n, bits), alpha, beta, bucket_size, levels, points).astype(np.float64)
    w = q.reshape(out_features, in_features)
    x = np.asarray(x, dtype=F32).astype(np.float64).reshape(-1, in_features)
    y = x @ w.T
    if bias is not None:
        y = y + np.asarray(bias, dtype=F32).astype(np.float64)[None, :]
    return y, np.abs(x) @ np.abs(w).T


def tolerance(y, magnitude, in_features: int) -> np.ndarray:
    """Bound of a float32 fmaf sum of in_features terms (any fixed order) against the float64 value, plus the
    rounding of the result itself: K * 2^-23 * sum |x q| + 2^-23 * |y|."""
    eps = 2.0 ** -23
    return in_features * eps * np.asarray(magnitude) + eps * np.abs(np.asarray(y))
