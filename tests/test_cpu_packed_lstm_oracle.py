"""The packed LSTM oracle (oracle/packed_lstm_oracle.py) pinned against torch's CPU nn.LSTMCell and nn.LSTM in float64
on decoded weights: gate order and both biases, bidirectional, multi-layer and batch_first, sorted and unsorted packed
sequences of lengths 1 .. T, h_n and c_n.  No GPU."""
import numpy as np
import pytest
import torch

from oracle import packed_linear_oracle as P
from oracle import packed_lstm_oracle as O


def _pack_bits(codes, bits):
    out = np.zeros((len(codes) * bits + 7) // 8, np.uint8)
    for e, c in enumerate(codes):
        out[e * bits // 8] |= (int(c) << (e * bits % 8)) & 0xFF
    return out


def _decoded(rng, rows, cols, bits=2, levels=4, bucket=7):
    """A weight decoded from random codes through the oracle (buckets straddling rows), and its codes' inputs."""
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
        w = [_decoded(rng, 4 * H, in_size), _decoded(rng, 4 * H, H, bits=4, levels=11, bucket=None)]
        w += [rng.standard_normal(4 * H) * 0.3, rng.standard_normal(4 * H) * 0.3] if bias else [None, None]
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
    cell = torch.nn.LSTMCell(I, H, bias=bias).double()
    _load(cell, [w])
    x, h, c = rng.standard_normal((B, I)), rng.standard_normal((B, H)), rng.standard_normal((B, H))
    h1, c1 = O.cell(x, h, c, *w)
    with torch.no_grad():
        th, tc = cell(torch.from_numpy(x), (torch.from_numpy(h), torch.from_numpy(c)))
    assert np.allclose(h1, th.numpy(), rtol=1e-12, atol=1e-13) and np.allclose(c1, tc.numpy(), rtol=1e-12, atol=1e-13)
    # the gates really are i, f, g, o: a huge forget preactivation keeps c, a huge negative input gate drops g
    w2 = [a.copy() if a is not None else np.zeros(4 * H) for a in w]
    w2[2] = np.zeros(4 * H)
    w2[2][H:2 * H] = 60.0
    w2[2][:H] = -60.0
    _, c2 = O.cell(x, h, c, w2[0] * 0, w2[1] * 0, w2[2], None)
    assert np.allclose(c2, c, rtol=1e-12)


@pytest.mark.parametrize("num_layers,bidirectional,batch_first", [(1, False, False), (2, True, False), (3, False, True), (2, True, True)])
def test_padded_batch_against_nn_lstm(num_layers, bidirectional, batch_first):
    rng = np.random.default_rng(num_layers * 10 + bidirectional)
    I, H, T, B = 6, 5, 7, 3
    dirs = 2 if bidirectional else 1
    w = _weights(rng, I, H, num_layers, dirs)
    lstm = torch.nn.LSTM(I, H, num_layers=num_layers, bidirectional=bidirectional, batch_first=batch_first).double()
    _load(lstm, w)
    x = rng.standard_normal((T, B, I))
    h0, c0 = rng.standard_normal((num_layers * dirs, B, H)), rng.standard_normal((num_layers * dirs, B, H))
    xt = torch.from_numpy(x.transpose(1, 0, 2).copy() if batch_first else x)
    out_t, (hn_t, cn_t) = lstm(xt, (torch.from_numpy(h0), torch.from_numpy(c0)))
    if batch_first:
        out_t = out_t.transpose(0, 1)
    out, hn, cn = O.lstm(x.reshape(T * B, I), O.padded_batch_sizes(T, B), w, num_layers, bidirectional, (h0, c0))
    assert np.allclose(out.reshape(T, B, -1), out_t.detach().numpy(), rtol=1e-11, atol=1e-12)
    assert np.allclose(hn, hn_t.detach().numpy(), rtol=1e-11, atol=1e-12)
    assert np.allclose(cn, cn_t.detach().numpy(), rtol=1e-11, atol=1e-12)


@pytest.mark.parametrize("enforce_sorted", [True, False])
@pytest.mark.parametrize("bidirectional", [False, True])
def test_packed_sequences_against_nn_lstm(enforce_sorted, bidirectional):
    rng = np.random.default_rng(7 + bidirectional)
    I, H, T, num_layers = 4, 3, 6, 2
    dirs = 2 if bidirectional else 1
    lengths = [T, 1, 3, T, 2, 5] if not enforce_sorted else [T, T, 5, 3, 2, 1]   # every length 1 .. T
    B = len(lengths)
    w = _weights(rng, I, H, num_layers, dirs)
    lstm = torch.nn.LSTM(I, H, num_layers=num_layers, bidirectional=bidirectional).double()
    _load(lstm, w)
    x = rng.standard_normal((T, B, I))
    h0, c0 = rng.standard_normal((num_layers * dirs, B, H)), rng.standard_normal((num_layers * dirs, B, H))
    ps = torch.nn.utils.rnn.pack_padded_sequence(torch.from_numpy(x), torch.tensor(lengths), enforce_sorted=enforce_sorted)
    out_t, (hn_t, cn_t) = lstm(ps, (torch.from_numpy(h0), torch.from_numpy(c0)))
    # the oracle on the sorted sequences: its batch row i is the PackedSequence's sorted row i
    order = ps.sorted_indices.numpy() if ps.sorted_indices is not None else np.arange(B)
    data, bs = O.pack([x[:lengths[b], b] for b in order])
    assert np.array_equal(data, ps.data.numpy()) and bs == ps.batch_sizes.tolist()
    out, hn, cn = O.lstm(data, bs, w, num_layers, bidirectional, (h0[:, order], c0[:, order]))
    assert np.allclose(out, out_t.data.detach().numpy(), rtol=1e-11, atol=1e-12)
    inv = np.argsort(order)
    assert np.allclose(hn[:, inv], hn_t.detach().numpy(), rtol=1e-11, atol=1e-12)
    assert np.allclose(cn[:, inv], cn_t.detach().numpy(), rtol=1e-11, atol=1e-12)


def test_step_tolerance_covers_a_float32_step():
    """A float32 restatement of the kernel's order (sums, then the adds and activations rounded one by one) stays inside
    step_tolerance of the float64 oracle."""
    rng = np.random.default_rng(3)
    I, H, B = 300, 200, 5
    w_ih, w_hh = _decoded(rng, 4 * H, I, bucket=256), _decoded(rng, 4 * H, H, bucket=100)
    b_ih, b_hh = (rng.standard_normal(4 * H) * 0.2).astype(np.float32), (rng.standard_normal(4 * H) * 0.2).astype(np.float32)
    x, h, c = (rng.standard_normal(s).astype(np.float32) for s in ((B, I), (B, H), (B, H)))
    f32 = np.float32
    z = ((x @ w_ih.T).astype(f32) + b_ih).astype(f32)
    z = ((z + (h @ w_hh.T).astype(f32)).astype(f32) + b_hh).astype(f32)
    sig = lambda v: (f32(1) / (f32(1) + np.exp(-v).astype(f32))).astype(f32)  # noqa: E731
    i, f, g, o = np.split(z, 4, axis=-1)
    c1 = ((sig(f) * c).astype(f32) + (sig(i) * np.tanh(g)).astype(f32)).astype(f32)
    h1 = (sig(o) * np.tanh(c1)).astype(f32)
    h_ref, c_ref = O.cell(x, h, c, w_ih, w_hh, b_ih, b_hh)
    tol_h, tol_c = O.step_tolerance(x, h, c, w_ih, w_hh, b_ih, b_hh)
    assert np.all(np.abs(c1 - c_ref) <= tol_c) and np.all(np.abs(h1 - h_ref) <= tol_h)
