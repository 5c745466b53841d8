"""CPU oracle of the LSTM layers on fixed-width packed weights (qd_packed_lstm_cell, qd_packed_lstm_layer) -- TEST
INFRASTRUCTURE ONLY.

The weights are the packed codec's, decoded by packed_linear_oracle.dequantize into float32 [4H, I] and [4H, H]
matrices; everything after that is float64: the gates z = x W_ih^T + b_ih + h W_hh^T + b_hh in torch's order (i, f, g,
o), c' = sigmoid(f) c + sigmoid(i) tanh(g), h' = sigmoid(o) tanh(c').  A layer runs over a padded batch or a
PackedSequence's data (rows of step t at offset sum(batch_sizes[:t])) in either direction; a row's previous h and c are
its state at the previous step it was active in, else h0 / c0, and its h_n / c_n are its state after its last step.
step_tolerance bounds the float32 kernel's h' and c' against this for one step whose inputs are exact.
"""
from __future__ import annotations

import numpy as np

from .packed_linear_oracle import dequantize, unpack_codes

F64 = np.float64


def decode_weight(packed, bits: int, alpha, beta, rows: int, cols: int, bucket_size, levels=None, points=None) -> np.ndarray:
    """The float32 [rows, cols] matrix the packed codes decode to (qd_unpack_dequant_*)."""
    n = rows * cols
    return dequantize(unpack_codes(packed, n, bits), alpha, beta, bucket_size, levels, points).reshape(rows, cols)


def _sigmoid(z):
    return 1.0 / (1.0 + np.exp(-z))


def cell(x, h, c, w_ih, w_hh, b_ih=None, b_hh=None):
    """(h', c') of one LSTM step in float64 for rows x [m, I], h and c [m, H]."""
    x, h, c = (np.asarray(t, dtype=F64) for t in (x, h, c))
    z = x @ np.asarray(w_ih, F64).T + h @ np.asarray(w_hh, F64).T
    for b in (b_ih, b_hh):
        if b is not None:
            z = z + np.asarray(b, F64)
    i, f, g, o = np.split(z, 4, axis=-1)
    c1 = _sigmoid(f) * c + _sigmoid(i) * np.tanh(g)
    return _sigmoid(o) * np.tanh(c1), c1


def layer(data, batch_sizes, h0, c0, w_ih, w_hh, b_ih=None, b_hh=None, reverse=False):
    """(out [N, H], h_n [B, H], c_n [B, H]) of one layer and direction over PackedSequence data [N, I] with
    ``batch_sizes`` (a padded batch of T steps passes T equal entries)."""
    bs = [int(b) for b in batch_sizes]
    off = np.concatenate([[0], np.cumsum(bs)]).astype(np.int64)
    h, c = np.array(h0, dtype=F64), np.array(c0, dtype=F64)
    H = h.shape[1]
    data = np.asarray(data, dtype=F64)
    out = np.zeros((data.shape[0], H), F64)
    for t in (reversed(range(len(bs))) if reverse else range(len(bs))):
        m = bs[t]
        h[:m], c[:m] = cell(data[off[t]:off[t] + m], h[:m], c[:m], w_ih, w_hh, b_ih, b_hh)
        out[off[t]:off[t] + m] = h[:m]
    return out, h, c


def lstm(data, batch_sizes, weights, num_layers: int, bidirectional: bool, hx=None):
    """nn.LSTM over PackedSequence data (sorted: batch row i is the i-th longest sequence).  ``weights``: one (w_ih, w_hh,
    b_ih, b_hh) per layer and direction in nn.LSTM's order, biases may be None; hx = (h0, c0) of shape [L*D, B, H] or
    None.  Returns (out [N, D*H], h_n, c_n)."""
    dirs = 2 if bidirectional else 1
    B = int(batch_sizes[0])
    H = np.asarray(weights[0][1]).shape[1]
    h0, c0 = (np.zeros((num_layers * dirs, B, H)),) * 2 if hx is None else (np.asarray(hx[0], F64), np.asarray(hx[1], F64))
    h_n, c_n = np.zeros((num_layers * dirs, B, H)), np.zeros((num_layers * dirs, B, H))
    x = np.asarray(data, F64)
    for layer_i in range(num_layers):
        outs = []
        for d in range(dirs):
            k = layer_i * dirs + d
            o, h_n[k], c_n[k] = layer(x, batch_sizes, h0[k], c0[k], *weights[k], reverse=d == 1)
            outs.append(o)
        x = np.concatenate(outs, axis=1)
    return x, h_n, c_n


def padded_batch_sizes(steps: int, batch: int) -> list:
    return [batch] * steps


def pack(seqs):
    """(data, batch_sizes) of sequences [T_b, I] already sorted by decreasing length: PackedSequence's layout."""
    T = len(seqs[0])
    batch_sizes = [sum(len(s) > t for s in seqs) for t in range(T)]
    data = np.concatenate([np.stack([s[t] for s in seqs[:batch_sizes[t]]]) for t in range(T)])
    return data, batch_sizes


def step_tolerance(x, h, c, w_ih, w_hh, b_ih=None, b_hh=None):
    """(tol_h, tol_c): bounds of |h' - oracle| and |c' - oracle| for a float32 step whose inputs x, h, c are exact.
    Each gate's float32 sum of I + H products and two bias adds is off by at most (I + H + 4) * 2^-23 * m, m the sum of
    the magnitudes of its terms; sigmoid moves by at most a quarter of that, tanh by at most all of it, and each of
    expf, tanhf and the float32 ops of the update adds a few units of 2^-23 (IEEE expf and tanhf are within 2 ulp)."""
    eps = 2.0 ** -23
    x, h, c = (np.asarray(t, F64) for t in (x, h, c))
    mag = np.abs(x) @ np.abs(np.asarray(w_ih, F64)).T + np.abs(h) @ np.abs(np.asarray(w_hh, F64)).T
    for b in (b_ih, b_hh):
        if b is not None:
            mag = mag + np.abs(np.asarray(b, F64))
    dz = (x.shape[-1] + h.shape[-1] + 4) * eps * mag
    di, df, dg, do = np.split(dz, 4, axis=-1)
    dsig = 8 * eps
    tol_c = np.abs(c) * (0.25 * df + dsig) + (0.25 * di + dsig) + (dg + dsig) + 4 * eps * (np.abs(c) + 1)
    tol_h = (0.25 * do + dsig) + tol_c + 4 * eps
    return tol_h, tol_c
