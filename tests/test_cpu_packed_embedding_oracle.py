"""The packed embedding lookup restated in NumPy from the packed fully-connected oracle (oracle/packed_linear_oracle.py:
unpack_codes, unit_table, dequantize reshaped to [V, D] and indexed) and pinned against a bit-by-bit restatement on
hand-built codes: odd row widths whose rows start inside a byte, buckets straddling rows, bucket None, and non-uniform
points with duplicates.  No GPU."""
import numpy as np
import pytest

from oracle import packed_linear_oracle as P


def embedding_oracle(indices, packed, bits, alpha, beta, num_embeddings, dim, bucket_size, levels=None, points=None):
    """out[..., :] = row indices[...] of the decoded [num_embeddings, dim] weight (float32)."""
    n = num_embeddings * dim
    q = P.dequantize(P.unpack_codes(packed, n, bits), alpha, beta, bucket_size, levels, points).reshape(num_embeddings, dim)
    return q[np.asarray(indices, dtype=np.int64)]


def _pack(codes, bits):
    out = np.zeros((len(codes) * bits + 7) // 8, np.uint8)
    for e, c in enumerate(codes):
        out[e * bits // 8] |= (int(c) << (e * bits % 8)) & 0xFF
    return out


def _direct(indices, packed, bits, alpha, beta, dim, bucket, unit, n):
    """Element by element: the code's byte and bit offset, its bucket, two float32 roundings."""
    row_len = n if bucket is None or n < bucket else bucket
    out = np.zeros((len(indices), dim), np.float32)
    for i, r in enumerate(indices):
        for d in range(dim):
            e = int(r) * dim + d
            code = (int(packed[e * bits // 8]) >> (e * bits % 8)) & ((1 << bits) - 1)
            b = e // row_len
            out[i, d] = np.float32(np.float32(unit[code] * alpha[b]) + beta[b])
    return out


def test_rows_start_inside_a_byte():
    """dim 3 at 1 bit: row 1 starts at bit 3, row 2 at bit 6 and runs into the second byte."""
    codes = [1, 0, 1, 1, 1, 0, 0, 1, 1]
    packed = _pack(codes, 1)
    alpha, beta = np.array([2.0], np.float32), np.array([-1.0], np.float32)
    out = embedding_oracle([2, 0, 1, 2], packed, 1, alpha, beta, 3, 3, None, levels=2)
    assert out.tolist() == [[-1, 1, 1], [1, -1, 1], [1, 1, -1], [-1, 1, 1]]


def test_buckets_straddle_rows():
    """dim 3, bucket 2: element (0, 2) and (1, 0) share bucket 1, so one scale pair spans two rows."""
    codes = np.ones(6, np.int64)
    alpha = np.array([1, 10, 100], np.float32)
    out = embedding_oracle([1, 0], _pack(codes, 2), 2, alpha, np.zeros(3, np.float32), 2, 3, 2, levels=2)
    assert out.tolist() == [[10, 100, 100], [1, 1, 10]]


@pytest.mark.parametrize("bits,levels,points", [(1, 2, None), (2, 3, None), (2, 4, None), (4, 11, None), (8, 256, None),
                                                (2, None, [0.1, 0.1, 0.8]), (4, None, [0.0, 0.5, 0.5, 0.5, 1.0]),
                                                (1, None, [0.3]), (8, None, None)])
@pytest.mark.parametrize("num_embeddings,dim,bucket", [(7, 3, None), (5, 7, 4), (9, 5, 8), (4, 31, 100), (3, 1, 2), (6, 9, 9),
                                                       (11, 3, 5)])
def test_oracle_matches_a_direct_restatement(bits, levels, points, num_embeddings, dim, bucket):
    rng = np.random.default_rng(bits * 1000 + num_embeddings * 10 + dim)
    if bits == 8 and levels is None and points is None:        # 256 points, many repeated
        points = np.sort(rng.integers(0, 40, 256) / 40.0).astype(np.float32)
    n = num_embeddings * dim
    k = levels if points is None else len(points)
    codes = rng.integers(0, k, n)
    rows = 1 if bucket is None or n < bucket else -(-n // bucket)
    alpha = rng.random(rows).astype(np.float32) + np.float32(0.5)
    beta = rng.standard_normal(rows).astype(np.float32)
    packed = _pack(codes, bits)
    indices = np.concatenate([rng.integers(0, num_embeddings, 13), np.arange(num_embeddings)[::-1], [0, 0, num_embeddings - 1]])
    got = embedding_oracle(indices, packed, bits, alpha, beta, num_embeddings, dim, bucket, levels, points)
    want = _direct(indices, packed, bits, alpha, beta, dim, bucket, P.unit_table(levels, points), n)
    assert got.dtype == np.float32 and got.shape == (len(indices), dim)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_index_shapes_carry_through():
    codes = np.arange(12) % 4
    out = embedding_oracle(np.array([[0, 3], [2, 1]]), _pack(codes, 2), 2, np.ones(1, np.float32), np.zeros(1, np.float32), 4, 3,
                           None, levels=4)
    assert out.shape == (2, 2, 3)
    assert np.array_equal(out[1, 0], P.unit_table(levels=4)[[2, 3, 0]])        # row 2: elements 6, 7, 8
