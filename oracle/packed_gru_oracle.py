"""CPU oracle of the GRU layers on fixed-width packed weights (qd_packed_gru_cell, qd_packed_gru_layer) -- TEST
INFRASTRUCTURE ONLY.

The weights are the packed codec's, decoded by packed_linear_oracle.dequantize (packed_lstm_oracle.decode_weight) into
float32 [3H, I] and [3H, H] matrices; everything after that is float64, in torch's gate order (r, z, n):
gi = x W_ih^T + b_ih, gh = h W_hh^T + b_hh, r = sigmoid(gi_r + gh_r), z = sigmoid(gi_z + gh_z),
n = tanh(gi_n + r gh_n), h' = n + z (h - n).  A layer runs over a padded batch or a PackedSequence's data (rows of step t
at offset sum(batch_sizes[:t])) in either direction; a row's previous h is its state at the previous step it was active
in, else h0, and its h_n is its state after its last step.  step_tolerance bounds the float32 kernel's h' against this
for one step whose inputs are exact.
"""
from __future__ import annotations

import numpy as np

from .packed_lstm_oracle import decode_weight, pack, padded_batch_sizes  # noqa: F401  (the same decode and layouts)

F64 = np.float64


def _sigmoid(v):
    return 1.0 / (1.0 + np.exp(-v))


def _linear(x, w, b):
    y = np.asarray(x, F64) @ np.asarray(w, F64).T
    return y if b is None else y + np.asarray(b, F64)


def cell(x, h, w_ih, w_hh, b_ih=None, b_hh=None):
    """h' of one GRU step in float64 for rows x [m, I] and h [m, H]."""
    h = np.asarray(h, F64)
    gi, gh = _linear(x, w_ih, b_ih), _linear(h, w_hh, b_hh)
    i_r, i_z, i_n = np.split(gi, 3, axis=-1)
    h_r, h_z, h_n = np.split(gh, 3, axis=-1)
    r, z = _sigmoid(i_r + h_r), _sigmoid(i_z + h_z)
    n = np.tanh(i_n + r * h_n)
    return n + z * (h - n)


def layer(data, batch_sizes, h0, w_ih, w_hh, b_ih=None, b_hh=None, reverse=False):
    """(out [N, H], h_n [B, H]) of one layer and direction over PackedSequence data [N, I] with ``batch_sizes`` (a
    padded batch of T steps passes T equal entries)."""
    bs = [int(b) for b in batch_sizes]
    off = np.concatenate([[0], np.cumsum(bs)]).astype(np.int64)
    h = np.array(h0, dtype=F64)
    data = np.asarray(data, dtype=F64)
    out = np.zeros((data.shape[0], h.shape[1]), F64)
    for t in (reversed(range(len(bs))) if reverse else range(len(bs))):
        m = bs[t]
        h[:m] = cell(data[off[t]:off[t] + m], h[:m], w_ih, w_hh, b_ih, b_hh)
        out[off[t]:off[t] + m] = h[:m]
    return out, h


def gru(data, batch_sizes, weights, num_layers: int, bidirectional: bool, h0=None):
    """nn.GRU over PackedSequence data (sorted: batch row i is the i-th longest sequence).  ``weights``: one (w_ih, w_hh,
    b_ih, b_hh) per layer and direction in nn.GRU's order, biases may be None; h0 of shape [L*D, B, H] or None.
    Returns (out [N, D*H], h_n)."""
    dirs = 2 if bidirectional else 1
    B = int(batch_sizes[0])
    H = np.asarray(weights[0][1]).shape[1]
    h0 = np.zeros((num_layers * dirs, B, H)) if h0 is None else np.asarray(h0, F64)
    h_n = np.zeros((num_layers * dirs, B, H))
    x = np.asarray(data, F64)
    for layer_i in range(num_layers):
        outs = []
        for d in range(dirs):
            k = layer_i * dirs + d
            o, h_n[k] = layer(x, batch_sizes, h0[k], *weights[k], reverse=d == 1)
            outs.append(o)
        x = np.concatenate(outs, axis=1)
    return x, h_n


def step_tolerance(x, h, w_ih, w_hh, b_ih=None, b_hh=None):
    """Bound of |h' - oracle| for a float32 step whose inputs x and h are exact.  gi and gh are each a float32 sum of
    I (H) products and a bias add, off by at most (I + 2) * 2^-23 * m (H + 2 for gh), m the sum of the magnitudes of
    its terms.  sigmoid moves by at most a quarter of its argument's error and tanh by at most all of it; each of
    expf, tanhf and the float32 ops of the update adds a few units of 2^-23 (IEEE expf and tanhf are within 2 ulp)."""
    eps = 2.0 ** -23
    x, h = np.asarray(x, F64), np.asarray(h, F64)
    mi = np.abs(x) @ np.abs(np.asarray(w_ih, F64)).T + (0 if b_ih is None else np.abs(np.asarray(b_ih, F64)))
    mh = np.abs(h) @ np.abs(np.asarray(w_hh, F64)).T + (0 if b_hh is None else np.abs(np.asarray(b_hh, F64)))
    di, dh = (x.shape[-1] + 2) * eps * mi, (h.shape[-1] + 2) * eps * mh
    di_r, di_z, di_n = np.split(di, 3, axis=-1)
    dh_r, dh_z, dh_n = np.split(dh, 3, axis=-1)
    mi_n, mh_n = np.split(mi, 3, axis=-1)[2], np.split(mh, 3, axis=-1)[2]
    dsig = 8 * eps
    dr = 0.25 * (di_r + dh_r) + dsig
    dz = 0.25 * (di_z + dh_z) + dsig
    dn = di_n + dh_n + dr * mh_n + 4 * eps * (mi_n + mh_n) + dsig
    return dn + dz * (np.abs(h) + 1) + 4 * eps * (np.abs(h) + 1)
