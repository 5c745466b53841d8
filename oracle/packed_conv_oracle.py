"""CPU oracle of the convolution on fixed-width packed weights (qd_packed_conv2d) -- TEST INFRASTRUCTURE ONLY.

The weights are those of packed_linear_oracle: the codes of the flattened [O, C, kh, kw] weight unpacked from the
qd_pack_indices layout and dequantized per bucket of the flattened tensor (buckets straddle output channels whenever
C*kh*kw is not a multiple of the bucket), each op rounded to float32.  The convolution is then taken in float64: groups
1, dilation 1, zero padding on both sides, y[n, o, i, j] = sum_{c, r, s} xpad[n, c, i*sh + r, j*sw + s] * q[o, c, r, s]
(+ bias[o]), the reference the float32 kernel is held to within a summation-order tolerance.
"""
from __future__ import annotations

import numpy as np

from .packed_linear_oracle import dequantize, tolerance, unpack_codes  # noqa: F401 - tolerance is this oracle's too

F32 = np.float32


def output_size(size: int, kernel: int, stride: int, pad: int) -> int:
    """Output side of one dimension; ValueError when the kernel is larger than the padded input."""
    if size + 2 * pad < kernel:
        raise ValueError(f"a kernel of {kernel} does not fit an input of {size} padded by {pad} on each side")
    return (size + 2 * pad - kernel) // stride + 1


def conv2d_f64(x, w, stride=(1, 1), padding=(0, 0)):
    """(y, magnitude) of the float64 convolution of x [N, C, H, W] with w [O, C, kh, kw]: y and sum |x w| per output."""
    x = np.asarray(x, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    n, c, h, wd = x.shape
    o, c2, kh, kw = w.shape
    if c != c2:
        raise ValueError(f"input has {c} channels, the weight {c2}")
    (sh, sw), (ph, pw) = stride, padding
    ho, wo = output_size(h, kh, sh, ph), output_size(wd, kw, sw, pw)
    xp = np.pad(x, ((0, 0), (0, 0), (ph, ph), (pw, pw)))
    y = np.zeros((n, o, ho, wo))
    mag = np.zeros((n, o, ho, wo))
    for r in range(kh):
        for s in range(kw):
            patch = xp[:, :, r:r + sh * (ho - 1) + 1:sh, s:s + sw * (wo - 1) + 1:sw]      # [N, C, Ho, Wo]
            y += np.einsum("nchw,oc->nohw", patch, w[:, :, r, s])
            mag += np.einsum("nchw,oc->nohw", np.abs(patch), np.abs(w[:, :, r, s]))
    return y, mag


def packed_conv2d(x, packed, bits: int, alpha, beta, shape, bucket_size, stride=(1, 1), padding=(0, 0), levels=None,
                  points=None, bias=None):
    """(y, magnitude): the float64 convolution of x [N, C, H, W] with the decoded weight of ``shape`` (O, C, kh, kw)
    (+ bias), and sum |x q| per output (the scale of the float32 summation error)."""
    n = int(np.prod(shape))
    q = dequantize(unpack_codes(packed, n, bits), alpha, beta, bucket_size, levels, points).reshape(shape)
    y, mag = conv2d_f64(np.asarray(x, dtype=F32), q, stride, padding)
    if bias is not None:
        y = y + np.asarray(bias, dtype=F32).astype(np.float64)[None, :, None, None]
    return y, mag
