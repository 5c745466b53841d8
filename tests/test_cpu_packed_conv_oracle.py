"""The packed convolution oracle (oracle/packed_conv_oracle.py) against torch.nn.functional.conv2d in float64 on
hand-built codes: buckets straddling output channels, bucket None, stride 2, padding, non-square kernels, a kernel wider
than the input, and a kernel wider than the padded input (refused).  No GPU."""
import numpy as np
import pytest
import torch

from oracle import packed_conv_oracle as PC
from oracle import packed_linear_oracle as P


def _pack(codes, bits):
    out = np.zeros((len(codes) * bits + 7) // 8, np.uint8)
    for e, c in enumerate(codes):
        out[e * bits // 8] |= (int(c) << (e * bits % 8)) & 0xFF
    return out


def _direct_weight(codes, alpha, beta, bucket, unit, shape):
    """Element by element: q_e = fl(fl(unit[code_e] * alpha_b) + beta_b), b = e // row_len."""
    n = int(np.prod(shape))
    row_len = n if bucket is None or n < bucket else bucket
    q = np.zeros(n, np.float32)
    for e in range(n):
        b = e // row_len
        q[e] = np.float32(np.float32(unit[codes[e]] * alpha[b]) + beta[b])
    return q.reshape(shape)


CASES = [  # (N, C, H, W), (O, kh, kw), stride, padding, bucket
    ((2, 3, 8, 8), (5, 3, 3), (1, 1), (1, 1), 16),       # C*kh*kw = 27: buckets straddle output channels
    ((1, 4, 9, 7), (3, 3, 3), (2, 2), (1, 1), 256),      # stride 2, one bucket for the whole tensor
    ((2, 2, 6, 10), (4, 3, 5), (2, 1), (0, 2), 7),       # non-square kernel, stride (2, 1), padding (0, 2)
    ((1, 3, 5, 5), (2, 1, 1), (2, 2), (0, 0), None),     # 1x1 shortcut at stride 2, bucket None
    ((3, 1, 2, 3), (2, 5, 5), (1, 1), (2, 2), 4),        # kernel wider than the input, not than the padded input
    ((1, 1, 1, 1), (1, 1, 1), (1, 1), (0, 0), None),     # C = O = 1 on a 1x1 input
]


@pytest.mark.parametrize("bits,levels,points", [(1, 2, None), (2, 3, None), (4, 16, None), (8, 256, None), (2, None, [0.0, 0.2, 0.9])])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("with_bias", [False, True])
def test_oracle_matches_torch_conv2d_in_float64(bits, levels, points, case, with_bias):
    (n, c, h, w), (o, kh, kw), stride, padding, bucket = CASES[case]
    rng = np.random.default_rng(bits * 100 + case * 10 + with_bias)
    shape = (o, c, kh, kw)
    ne = o * c * kh * kw
    k = levels if points is None else len(points)
    codes = rng.integers(0, k, ne)
    rows = 1 if bucket is None or ne < bucket else -(-ne // bucket)
    alpha = rng.random(rows).astype(np.float32) + np.float32(0.5)
    beta = rng.standard_normal(rows).astype(np.float32)
    x = rng.standard_normal((n, c, h, w)).astype(np.float32)
    bias = rng.standard_normal(o).astype(np.float32) if with_bias else None
    packed = _pack(codes, bits)
    y, mag = PC.packed_conv2d(x, packed, bits, alpha, beta, shape, bucket, stride, padding, levels, points, bias)
    q = _direct_weight(codes, alpha, beta, bucket, P.unit_table(levels, points), shape)
    want = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(q).double(),
                                      None if bias is None else torch.from_numpy(bias).double(), stride, padding).numpy()
    assert y.shape == want.shape
    np.testing.assert_allclose(y, want, rtol=1e-12, atol=1e-12)
    mag_want = torch.nn.functional.conv2d(torch.from_numpy(np.abs(x)).double(), torch.from_numpy(np.abs(q)).double(), None, stride,
                                          padding).numpy()
    np.testing.assert_allclose(mag, mag_want, rtol=1e-12, atol=1e-12)
    assert np.all(P.tolerance(y, mag, c * kh * kw) >= 0)


def test_buckets_straddle_output_channels():
    """C*kh*kw = 3, bucket 2: weight (0, 2) and (1, 0) share bucket 1, so one scale pair spans two output channels."""
    codes = np.ones(6, np.int64)
    alpha = np.array([1, 10, 100], np.float32)
    beta = np.zeros(3, np.float32)
    x = np.zeros((3, 3, 1, 1), np.float32)             # three images, image i a one-hot on channel i
    for i in range(3):
        x[i, i, 0, 0] = 1
    y, _ = PC.packed_conv2d(x, _pack(codes, 1), 1, alpha, beta, (2, 3, 1, 1), 2, levels=2)
    assert y[:, :, 0, 0].T.tolist() == [[1, 1, 10], [10, 100, 100]]


def test_padding_taps_read_zero():
    """A 3x3 kernel of ones over a 2x2 input padded by 1: each output sums the input taps inside the image."""
    x = np.arange(1, 5, dtype=np.float32).reshape(1, 1, 2, 2)
    y, mag = PC.packed_conv2d(x, _pack(np.ones(9, np.int64), 1), 1, np.ones(1, np.float32), np.zeros(1, np.float32), (1, 1, 3, 3),
                              None, padding=(1, 1), levels=2)
    assert y.reshape(-1).tolist() == [10, 10, 10, 10]
    assert mag.reshape(-1).tolist() == [10, 10, 10, 10]


def test_kernel_wider_than_the_padded_input_is_refused():
    with pytest.raises(ValueError, match="does not fit"):
        PC.packed_conv2d(np.zeros((1, 1, 4, 2), np.float32), _pack(np.zeros(15, np.int64), 1), 1, np.ones(1, np.float32),
                         np.zeros(1, np.float32), (1, 1, 3, 5), None, padding=(0, 1), levels=2)
    assert PC.output_size(2, 5, 1, 2) == 2 and PC.output_size(4, 3, 2, 0) == 1
