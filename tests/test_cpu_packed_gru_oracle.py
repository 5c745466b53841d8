"""The packed GRU oracle (oracle/packed_gru_oracle.py) pinned against torch's CPU nn.GRUCell and nn.GRU in float64 on
decoded weights: gate order and both biases (b_hn inside r * (...)), reverse direction, bidirectional, multi-layer and
batch_first, sorted and unsorted packed sequences of lengths 1 .. T, h_n; and its one-step bound against a float32
restatement of the kernel's order.  No GPU."""
import numpy as np
import pytest
import torch

from oracle import packed_gru_oracle as O
from oracle import packed_linear_oracle as P


def _pack_bits(codes, bits):
    out = np.zeros((len(codes) * bits + 7) // 8, np.uint8)
    for e, c in enumerate(codes):
        out[e * bits // 8] |= (int(c) << (e * bits % 8)) & 0xFF
    return out


def _decoded(rng, rows, cols, bits=2, levels=4, bucket=7):
    """A weight decoded from random codes through the oracle (buckets straddling rows)."""
    n = rows * cols
    codes = rng.integers(0, levels, n)
    nb = 1 if bucket is None or n < bucket else -(-n // bucket)
    alpha = (rng.random(nb) * 0.6 + 0.2).astype(np.float32)
    beta = (-alpha / 2).astype(np.float32)
    w = O.decode_weight(_pack_bits(codes, bits), bits, alpha, beta, rows, cols, bucket, levels=levels)
    want = P.dequantize(codes, alpha, beta, bucket, levels=levels).reshape(rows, cols)
    assert np.array_equal(w.view(np.uint32), want.view(np.uint32))
    return w


def _weights(rng, I, H, num_layers, dirs, bias=True):
    out = []
    for k in range(num_layers * dirs):
        in_size = I if k < dirs else dirs * H
        w = [_decoded(rng, 3 * H, in_size), _decoded(rng, 3 * H, H, bits=4, levels=11, bucket=None)]
        w += [rng.standard_normal(3 * H) * 0.3, rng.standard_normal(3 * H) * 0.3] if bias else [None, None]
        out.append(w)
    return out


def _load(mod, weights):
    with torch.no_grad():
        for name, p in mod.named_parameters():
            kind, which, *rest = name.split("_")          # weight_ih_l0_reverse, bias_hh_l1, weight_ih (cell)
            k = 0
            if rest:
                k = int(rest[0][1:]) * (2 if mod.bidirectional else 1) + (len(rest) > 1)
            j = (0 if which == "ih" else 1) + (2 if kind == "bias" else 0)
            p.copy_(torch.from_numpy(np.asarray(weights[k][j], np.float64)))


@pytest.mark.parametrize("bias", [True, False])
def test_cell_gate_order_and_biases(bias):
    rng = np.random.default_rng(1)
    I, H, B = 5, 3, 4
    w = _weights(rng, I, H, 1, 1, bias)[0]
    cell = torch.nn.GRUCell(I, H, bias=bias).double()
    _load(cell, [w])
    x, h = rng.standard_normal((B, I)), rng.standard_normal((B, H))
    h1 = O.cell(x, h, *w)
    with torch.no_grad():
        th = cell(torch.from_numpy(x), torch.from_numpy(h))
    assert np.allclose(h1, th.numpy(), rtol=1e-12, atol=1e-13)
    # the gates really are r, z, n: a huge update gate keeps h; with z = 0 and r = 0, h' = tanh(gi_n) and b_hn is
    # dropped with the rest of gh_n (it sits inside r * (...))
    zero_w = (np.zeros((3 * H, I)), np.zeros((3 * H, H)))
    b_z = np.zeros(3 * H)
    b_z[H:2 * H] = 60.0
    assert np.allclose(O.cell(x, h, *zero_w, b_z, None), h, rtol=1e-12)
    b_ih, b_hh = np.zeros(3 * H), np.zeros(3 * H)
    b_ih[:H], b_ih[H:2 * H], b_ih[2 * H:] = -60.0, -60.0, 0.5
    b_hh[2 * H:] = 7.0
    assert np.allclose(O.cell(x, h, *zero_w, b_ih, b_hh), np.tanh(0.5), rtol=1e-12)


@pytest.mark.parametrize("num_layers,bidirectional,batch_first", [(1, False, False), (2, True, False), (3, False, True), (2, True, True)])
def test_padded_batch_against_nn_gru(num_layers, bidirectional, batch_first):
    rng = np.random.default_rng(num_layers * 10 + bidirectional)
    I, H, T, B = 6, 5, 7, 3
    dirs = 2 if bidirectional else 1
    w = _weights(rng, I, H, num_layers, dirs)
    gru = torch.nn.GRU(I, H, num_layers=num_layers, bidirectional=bidirectional, batch_first=batch_first).double()
    _load(gru, w)
    x = rng.standard_normal((T, B, I))
    h0 = rng.standard_normal((num_layers * dirs, B, H))
    xt = torch.from_numpy(x.transpose(1, 0, 2).copy() if batch_first else x)
    out_t, hn_t = gru(xt, torch.from_numpy(h0))
    if batch_first:
        out_t = out_t.transpose(0, 1)
    out, hn = O.gru(x.reshape(T * B, I), O.padded_batch_sizes(T, B), w, num_layers, bidirectional, h0)
    assert np.allclose(out.reshape(T, B, -1), out_t.detach().numpy(), rtol=1e-11, atol=1e-12)
    assert np.allclose(hn, hn_t.detach().numpy(), rtol=1e-11, atol=1e-12)


@pytest.mark.parametrize("reverse", [False, True])
def test_one_layer_each_direction_against_nn_gru(reverse):
    """O.layer in one direction is the matching half of a bidirectional nn.GRU, started from h0 or from zeros."""
    rng = np.random.default_rng(5 + reverse)
    I, H, T, B = 4, 6, 5, 2
    w = _weights(rng, I, H, 1, 2)
    gru = torch.nn.GRU(I, H, bidirectional=True).double()
    _load(gru, w)
    x = rng.standard_normal((T, B, I))
    for h0 in (None, rng.standard_normal((2, B, H))):
        out_t, hn_t = gru(torch.from_numpy(x), None if h0 is None else torch.from_numpy(h0))
        start = np.zeros((B, H)) if h0 is None else h0[int(reverse)]
        out, hn = O.layer(x.reshape(T * B, I), O.padded_batch_sizes(T, B), start, *w[int(reverse)], reverse=reverse)
        half = out_t.detach().numpy()[:, :, H * reverse:H * (reverse + 1)]
        assert np.allclose(out.reshape(T, B, H), half, rtol=1e-11, atol=1e-12)
        assert np.allclose(hn, hn_t.detach().numpy()[int(reverse)], rtol=1e-11, atol=1e-12)


@pytest.mark.parametrize("enforce_sorted", [True, False])
@pytest.mark.parametrize("bidirectional", [False, True])
def test_packed_sequences_against_nn_gru(enforce_sorted, bidirectional):
    rng = np.random.default_rng(7 + bidirectional)
    I, H, T, num_layers = 4, 3, 6, 2
    dirs = 2 if bidirectional else 1
    lengths = [T, 1, 3, T, 2, 5] if not enforce_sorted else [T, T, 5, 3, 2, 1]   # every length 1 .. T
    B = len(lengths)
    w = _weights(rng, I, H, num_layers, dirs)
    gru = torch.nn.GRU(I, H, num_layers=num_layers, bidirectional=bidirectional).double()
    _load(gru, w)
    x = rng.standard_normal((T, B, I))
    h0 = rng.standard_normal((num_layers * dirs, B, H))
    ps = torch.nn.utils.rnn.pack_padded_sequence(torch.from_numpy(x), torch.tensor(lengths), enforce_sorted=enforce_sorted)
    out_t, hn_t = gru(ps, torch.from_numpy(h0))
    # the oracle on the sorted sequences: its batch row i is the PackedSequence's sorted row i
    order = ps.sorted_indices.numpy() if ps.sorted_indices is not None else np.arange(B)
    data, bs = O.pack([x[:lengths[b], b] for b in order])
    assert np.array_equal(data, ps.data.numpy()) and bs == ps.batch_sizes.tolist()
    out, hn = O.gru(data, bs, w, num_layers, bidirectional, h0[:, order])
    assert np.allclose(out, out_t.data.detach().numpy(), rtol=1e-11, atol=1e-12)
    assert np.allclose(hn[:, np.argsort(order)], hn_t.detach().numpy(), rtol=1e-11, atol=1e-12)


def test_step_tolerance_covers_a_float32_step():
    """A float32 restatement of the kernel's order (gi and gh complete, then the adds and activations rounded one by
    one) stays inside step_tolerance of the float64 oracle."""
    rng = np.random.default_rng(3)
    I, H, B = 300, 200, 5
    w_ih, w_hh = _decoded(rng, 3 * H, I, bucket=256), _decoded(rng, 3 * H, H, bucket=100)
    b_ih, b_hh = (rng.standard_normal(3 * H) * 0.2).astype(np.float32), (rng.standard_normal(3 * H) * 0.2).astype(np.float32)
    x, h = (rng.standard_normal(s).astype(np.float32) for s in ((B, I), (B, H)))
    f32 = np.float32
    gi = ((x @ w_ih.T).astype(f32) + b_ih).astype(f32)
    gh = ((h @ w_hh.T).astype(f32) + b_hh).astype(f32)
    sig = lambda v: (f32(1) / (f32(1) + np.exp(-v).astype(f32))).astype(f32)  # noqa: E731
    (i_r, i_z, i_n), (h_r, h_z, h_n) = np.split(gi, 3, axis=-1), np.split(gh, 3, axis=-1)
    r, z = sig((i_r + h_r).astype(f32)), sig((i_z + h_z).astype(f32))
    n = np.tanh((i_n + (r * h_n).astype(f32)).astype(f32)).astype(f32)
    h1 = (n + (z * (h - n).astype(f32)).astype(f32)).astype(f32)
    assert np.all(np.abs(h1 - O.cell(x, h, w_ih, w_hh, b_ih, b_hh)) <= O.step_tolerance(x, h, w_ih, w_hh, b_ih, b_hh))
