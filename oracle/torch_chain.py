"""Torch-CPU restatement of the reference's op chain -- TEST / BASELINE ONLY.

The reference's CPU implementation of the hot path is a chain of stock torch
tensor ops (clone, min, max, sub_, div_, mul_, round_, div_, mul_, add_, ...;
SURVEY.md section 3.1).  The reference is not a dependency of this project, so this
module restates that chain, op for op and pass for pass, with the same torch
CPU kernels, so that ``bench.py --impl reference`` and the ``cpu_baseline`` leg
time the same memory passes the reference makes on the host cores
(``kind: "port"``).  The functions are device-agnostic like the reference's own code, so
tools/plan_bench.py can also time "the reference's stock-torch op chain on the same
GPU" next to the fused kernels.  It is also a second oracle, independent of the NumPy one,
and is pinned bit-for-bit against the golden vectors in
tests/test_oracle_golden.py::test_torch_chain_matches_golden.

Only tests/, __graft_entry__.smoke() and bench.py may import this file.
Citations: quantization/quant_functions.py (reference checkout).
"""
from __future__ import annotations

import numpy as np
import torch

_TOL = 1e-10  # quant_functions.py:40


class ChainState:
    __slots__ = ("alpha", "beta", "argmin", "argmax", "n", "shape", "rows_shape")


def _rows(t: torch.Tensor, bucket):
    """help_functions.py:67-94: flatten, pad the tail row with the last element
    (torch.cat copy, like the reference), view as rows."""
    if bucket is None:
        return t.view(-1)
    t = t.view(-1)
    n = t.numel()
    multiple, rest = divmod(n, bucket)
    if multiple != 0 and rest != 0:
        t = torch.cat([t, torch.ones(bucket - rest, device=t.device) * t[-1]])   # .cuda() in the reference (:84)
    return t.view(1, n) if multiple == 0 else t.view(-1, bucket)


def scale_down_(t: torch.Tensor, bucket) -> tuple[torch.Tensor, ChainState]:
    """quant_functions.py:76-107 on an already-cloned tensor."""
    st = ChainState()
    st.shape, st.n = t.size(), t.numel()
    t = _rows(t, bucket)
    dim = 0 if bucket is None else 1
    mn, st.argmin = t.min(dim=dim, keepdim=True)
    mx, st.argmax = t.max(dim=dim, keepdim=True)
    alpha = mx - mn
    alpha[alpha < _TOL] = 1
    st.alpha, st.beta, st.rows_shape = alpha, mn, t.size()
    t.sub_(mn.expand_as(t))
    t.div_(alpha.expand_as(t))
    return t, st


def inv_scale_down_(t: torch.Tensor, st: ChainState) -> torch.Tensor:
    """quant_functions.py:141-150."""
    t.mul_(st.alpha.expand_as(t))
    t.add_(st.beta.expand_as(t))
    t.add_(0)
    return t.view(-1)[0:st.n].view(st.shape)


def uniform_fwd(x: torch.Tensor, s: int, bucket):
    """quant_functions.py:155-194, deterministic rounding."""
    t, st = scale_down_(x.clone(), bucket)
    S = s - 1
    t.mul_(S)
    t.round_()
    t.div_(S)
    return inv_scale_down_(t, st), st


def uniform_bwd_minmax(x: torch.Tensor, g: torch.Tensor, s: int, bucket: int):
    """quant_functions.py:339-402 with the two shape bugs repaired (the sparse
    N x N product is replaced by the index_add_ it stands for)."""
    saved = x.clone()                                     # :309
    q, _ = uniform_fwd(saved, s, bucket)                  # :341
    qh, st = scale_down_(q.clone(), bucket)               # :350 (state now that of q)
    n = st.n
    qh = qh.view(-1)[0:n]
    rows = st.alpha.size(0)
    row_len = st.rows_shape[1]
    alpha = st.alpha.expand(rows, row_len).contiguous().view(-1)[0:n]
    beta = st.beta.expand(rows, row_len).contiguous().view(-1)[0:n]
    adder = torch.arange(0, row_len * rows, row_len, device=g.device).view(-1, 1)
    amax = (st.argmax + adder).view(-1)
    amin = (st.argmin + adder).view(-1)
    v = g.view(-1) * (qh - (saved.view(-1) - beta) / alpha)
    # M^T v of the reference (:380-400): per bucket r_b = sum_j v_j, +r_b at argmax', -r_b at argmin'
    vp = torch.zeros(rows * row_len, device=g.device)
    vp[0:n] = v
    r = vp.view(rows, row_len).sum(dim=1)
    corr = torch.zeros(n, device=g.device).index_add_(0, amax, r).index_add_(0, amin, -r)
    return (g.view(-1) + corr).view(g.size())


def nonuniform_fwd(x: torch.Tensor, points: torch.Tensor, bucket, rule="nearest"):
    """quant_functions.py:243-290: scale on torch, index search on host numpy."""
    t, st = scale_down_(x.clone(), bucket)
    v = t.view(-1).cpu().numpy()                           # device -> host like the reference (:255-258)
    k = points.cpu().numpy()
    if rule == "nearest":                                  # :267-273
        i = np.searchsorted(k, v, side="left").clip(max=k.size - 1)
        m = (i > 0) & ((i == len(k)) | (np.fabs(v - k[i - 1]) < np.fabs(v - k[i])))
        i = i - m
    else:                                                  # :531-573 closed form
        mid = k[:-1] + np.diff(k) / 2
        i = np.searchsorted(mid, v, side="right")
    out = torch.from_numpy(k[i]).view(*st.rows_shape).to(x.device)   # host -> device (:282-284)
    idx = torch.from_numpy(np.asarray(i)).long().to(x.device)
    q = inv_scale_down_(out, st)
    return q, idx.view(-1)[0:st.n].view(st.shape), st


def nonuniform_bwd_points(g: torch.Tensor, idx: torch.Tensor, st: ChainState, num_points: int, bucket):
    """quant_functions.py:471-506: clone, bucket, scale by alpha, K masked sums."""
    m = _rows(g.clone(), bucket)
    m = m * st.alpha.expand_as(m)
    m = m.view(-1)[0:g.numel()].view(g.size())
    out = torch.zeros(num_points, device=g.device)
    for k in range(num_points):
        out[k] = torch.masked_select(m, idx == k).sum()
    return out


class PreprocessedCentroids:
    """The pre-processed path of the differentiable-quantization loop, pass for pass
    (quant_functions.py:432-447 preprocess, :509-573 SearchSorted, :275-289 the tail of
    nonUniformQuantization): the scaled tensor is sorted ONCE on the host; each step costs a
    K-1 element searchsorted into the sorted copy, one or two N-element index fills in sorted
    order, a permutation scatter back to tensor order, a host gather of k[idx], the host->device
    copies of values and int64 indices, and the three-pass inverse scaling on the device."""

    def __init__(self, x: torch.Tensor, bucket):
        scaled, self.st = scale_down_(x.clone(), bucket)               # :433-437
        self.device = x.device
        host = scaled.view(-1).cpu().numpy().copy()                     # :440-445
        self.order = np.argsort(host)                                   # :520
        self.sorted = host[self.order]                                  # :521
        self.rank_of = np.argsort(self.order)                           # :522
        self.last_runs = None
        self.last_idx = None

    @staticmethod
    def _runs(cuts):
        """(end position in sorted order, centroid index) for every non-empty run (:535-543)."""
        runs, prev = [], 0
        for j, c in enumerate(cuts):
            if c != prev:
                runs.append((int(c), j))
                prev = c
        return runs

    @staticmethod
    def _fill(runs, n, K):
        out = np.zeros(n, dtype=int)                                    # :566-573
        start = 0
        for end, j in runs:
            out[start:end] = j
            start = end
        out[start:] = K - 1
        return out

    def query(self, k: np.ndarray) -> np.ndarray:
        mid = k[:-1] + np.diff(k) / 2                                   # :533
        runs = self._runs(np.searchsorted(self.sorted, mid))            # :534
        n, K = self.sorted.shape[0], len(k)
        if self.last_idx is None:                                       # :545-553
            self.last_idx = self._fill(runs, n, K)[self.rank_of]
        else:                                                           # :555-561 incremental update
            old, new = self._fill(self.last_runs, n, K), self._fill(runs, n, K)
            moved = new != old
            self.last_idx[self.order[moved]] = new[moved]
        self.last_runs = runs
        return self.last_idx

    def forward(self, points: torch.Tensor):
        k = points.detach().cpu().numpy()                               # :261
        idx = self.query(k)
        vals = torch.from_numpy(k[idx]).to(self.device)                 # :278-284
        idx_t = torch.from_numpy(idx).long().to(self.device)
        q = inv_scale_down_(vals.view(*self.st.rows_shape), self.st)    # :286-287
        return q, idx_t.view(-1)[0:self.st.n].view(self.st.shape)       # :288-289


def quantize_model_step(params, s: int, bucket):
    """The per-step choreography of cnn_models/conv_forward_model.py:236-247:
    one uniform_fwd per parameter tensor."""
    return [uniform_fwd(p, s, bucket)[0] for p in params]
