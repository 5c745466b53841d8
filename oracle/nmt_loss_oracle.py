"""CPU oracle of the fused NMT loss (qd_nmt_loss_fwd, qd_nmt_loss_bwd) -- TEST INFRASTRUCTURE ONLY.

A float64 NumPy restatement of the contract in include/qd_b200.h, for student logits z_s [R, V], an optional teacher
z_t [R, V], int64 targets y [R], padding_idx (-1: none) and w = weight_teacher_loss (the ABI takes it as float32, so
it is rounded to float32 first):
  lse_s = log sum_c exp(z_s)          (-inf for a row of -inf)
  lse_t = log sum_c exp(z_t)          (0 without a teacher)
  loss_i = lse_s - z_s[y]                                        without a teacher
         = (1-w)(lse_s - z_s[y]) + w sum_c p_t (z_t - lse_t - z_s + lse_s),  p_t = exp(z_t - lse_t)
           (a column with z_t = -inf adds 0; one with z_t finite and z_s = -inf adds +inf, even where p_t underflows)
  grad_i = g (exp(z_s - lse_s) - w p_t - (1-w)[c = y])           (w = 0 without a teacher)
Padding rows: loss 0, gradient 0, counted nowhere.  A target outside [0, V) that is not padding: loss and gradient NaN,
counted in n_invalid.  n_words counts the other rows, n_correct those whose first-occurrence argmax of z_s is y.
"""
from __future__ import annotations

import numpy as np

F64 = np.float64


def _lse(z):
    m = z.max(axis=1, initial=-np.inf)
    fin = np.isfinite(m)
    shift = np.where(fin, m, 0.0)[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.exp(z - shift).sum(axis=1)
        return np.where(fin, m + np.log(s), m)


def nmt_loss(logits, target, padding_idx=-1, teacher_logits=None, w=0.7, grad_loss=1.0):
    """dict(row_lse [R, 2], row_loss [R], loss, counts [n_words, n_correct, n_invalid], argmax [R], grad [R, V])."""
    zs = np.asarray(logits, F64)
    R, V = zs.shape
    y = np.asarray(target, np.int64).reshape(R)
    teacher = teacher_logits is not None
    w = float(np.float32(w)) if teacher else 0.0
    lse_s = _lse(zs)
    pad = (y == padding_idx) if padding_idx >= 0 else np.zeros(R, bool)
    invalid = ~pad & ((y < 0) | (y >= V))
    word = ~pad & ~invalid
    yc = np.where(word, y, 0)
    rows = np.arange(R)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        nll = lse_s - zs[rows, yc]
        ps = np.exp(zs - lse_s[:, None])
        grad = ps.copy()
        if teacher:
            zt = np.asarray(teacher_logits, F64)
            lse_t = _lse(zt)
            pt = np.exp(zt - lse_t[:, None])
            terms = np.where(np.isneginf(zt), 0.0,
                             np.where(np.isneginf(zs), np.inf, pt * (zt - lse_t[:, None] - zs + lse_s[:, None])))
            loss_rows = (1.0 - w) * nll + w * terms.sum(axis=1)
            grad -= w * pt
        else:
            lse_t = np.zeros(R)
            loss_rows = nll
        grad[rows[word], yc[word]] -= 1.0 - w
    loss_rows = np.where(pad, 0.0, np.where(invalid, np.nan, loss_rows))
    grad[pad] = 0.0
    grad[invalid] = np.nan
    argmax = zs.argmax(axis=1) if V > 0 and R > 0 else np.zeros(R, np.int64)
    counts = np.array([word.sum(), (word & (argmax == y)).sum(), invalid.sum()], np.int64)
    return dict(row_lse=np.stack([lse_s, lse_t], axis=1), row_loss=loss_rows, loss=float(loss_rows.sum()), counts=counts,
                argmax=argmax, grad=grad * float(np.float32(grad_loss)))
