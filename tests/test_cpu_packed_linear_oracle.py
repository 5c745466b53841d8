"""The packed fully-connected oracle (oracle/packed_linear_oracle.py) against a direct element-by-element restatement
on hand-built codes: the packed layout, the bucket of every weight (buckets straddling output rows, bucket None, a
short tensor) and the float64 product with and without bias.  No GPU."""
import numpy as np
import pytest

from oracle import packed_linear_oracle as P


def _pack(codes, bits):
    out = np.zeros((len(codes) * bits + 7) // 8, np.uint8)
    for e, c in enumerate(codes):
        out[e * bits // 8] |= (int(c) << (e * bits % 8)) & 0xFF
    return out


def _direct(codes, alpha, beta, bucket, unit, out_f, in_f, x, bias):
    n = out_f * in_f
    row_len = n if bucket is None or n < bucket else bucket
    w = np.zeros((out_f, in_f))
    for e in range(n):
        b = e // row_len
        q = np.float32(np.float32(unit[codes[e]] * alpha[b]) + beta[b])
        w[e // in_f, e % in_f] = float(q)
    y = np.zeros((x.shape[0], out_f))
    for i in range(x.shape[0]):
        for o in range(out_f):
            y[i, o] = sum(float(x[i, k]) * w[o, k] for k in range(in_f)) + (0.0 if bias is None else float(bias[o]))
    return y


def test_unpack_codes_reads_the_pack_layout():
    assert P.unpack_codes(np.array([0b10001101, 1], np.uint8), 9, 1).tolist() == [1, 0, 1, 1, 0, 0, 0, 1, 1]
    assert P.unpack_codes(np.array([0b011011], np.uint8), 3, 2).tolist() == [3, 2, 1]
    assert P.unpack_codes(np.array([0x5A, 0x0F], np.uint8), 3, 4).tolist() == [0xA, 0x5, 0xF]


def test_unit_table():
    assert P.unit_table(levels=3).tolist() == [0.0, 0.5, 1.0]
    assert P.unit_table(levels=4)[1] == np.float32(1) / np.float32(3)
    assert P.unit_table(points=[0.1, 0.7]).tolist() == [np.float32(0.1), np.float32(0.7)]
    with pytest.raises(ValueError):
        P.unit_table()


@pytest.mark.parametrize("bits,levels,points", [(1, 2, None), (2, 3, None), (4, 16, None), (8, 256, None), (2, None, [0.0, 0.2, 0.9]),
                                                (4, None, [0.5])])
@pytest.mark.parametrize("out_f,in_f,bucket", [(5, 7, 4), (3, 10, 8), (4, 6, None), (2, 3, 100), (6, 5, 5)])
@pytest.mark.parametrize("with_bias", [False, True])
def test_oracle_matches_a_direct_restatement(bits, levels, points, out_f, in_f, bucket, with_bias):
    rng = np.random.default_rng(bits * 100 + out_f * 10 + in_f)
    n = out_f * in_f
    k = levels if points is None else len(points)
    codes = rng.integers(0, k, n)
    rows = 1 if bucket is None or n < bucket else -(-n // bucket)
    alpha = rng.random(rows).astype(np.float32) + np.float32(0.5)
    beta = rng.standard_normal(rows).astype(np.float32)
    x = rng.standard_normal((3, in_f)).astype(np.float32)
    bias = rng.standard_normal(out_f).astype(np.float32) if with_bias else None
    packed = _pack(codes, bits)
    assert P.unpack_codes(packed, n, bits).tolist() == codes.tolist()
    unit = P.unit_table(levels, points)
    y, mag = P.packed_linear(x, packed, bits, alpha, beta, out_f, in_f, bucket, levels, points, bias)
    want = _direct(codes, alpha, beta, bucket, unit, out_f, in_f, x, bias)
    np.testing.assert_allclose(y, want, rtol=1e-12, atol=1e-12)
    assert np.all(P.tolerance(y, mag, in_f) >= 0)


def test_buckets_straddle_output_rows():
    """in_features 3, bucket 2: weight (0, 2) and (1, 0) share bucket 1, so one scale pair spans two output rows."""
    codes = np.array([1, 1, 1, 1, 1, 1])
    alpha = np.array([1, 10, 100], np.float32)
    beta = np.zeros(3, np.float32)
    q = P.dequantize(codes, alpha, beta, 2, levels=2)
    assert q.tolist() == [1, 1, 10, 10, 100, 100]
    y, _ = P.packed_linear(np.eye(3, dtype=np.float32), _pack(codes, 1), 1, alpha, beta, 2, 3, 2, levels=2)
    assert y.T.tolist() == [[1, 1, 10], [10, 100, 100]]
