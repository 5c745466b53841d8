"""CPU oracle of onmt's SRU recurrence (onmt/modules/SRU.py:71-347, sru_fwd / sru_bwd / sru_bi_fwd / sru_bi_bwd) and
of the native kernels qd_sru_fwd / qd_sru_bwd -- TEST INFRASTRUCTURE ONLY.

The reference kernels' forward and backward restated in float64 numpy, column by column as the kernels run them:
  g1 = sigmoid(u1 + bias1),  g2 = sigmoid(u2 + bias2),  c_t = (c_{t-1} - u0) g1 + u0  (c_{-1} = init),
  h_t = (act(c_t) mask_h - x') g2 + x',  x' = u3 (k = 4) or the layer input x (k = 3),
with bidirectional columns j >= d run backwards in time.  Layouts as include/qd_b200.h: u [len, batch, dir*d, k];
x, h, c, grad_h [len, batch, dir*d]; init, mask_h, grad_last [batch, dir*d]; bias [2*dir*d].

Every value also carries a first-order bound on the error of the float32 kernels' value, from the same expressions:
each float32 operation adds u |result| (u = 2^-24), expf and tanhf 2 ulp each (so sigmoid adds 8u |g|), a product
adds |a| err_b + |b| err_a + err_a err_b, and relu's branch (and the backward's c > 0 test) takes the whole jump when
|c| is within its bound of 0.  bounds() returns twice the propagated bound plus 2^-140 per step for subnormal
results: the propagation drops second-order terms.
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -140


class _V:
    """A float64 value with a bound on the float32 kernels' error of it."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v, self.e = np.asarray(v, np.float64), np.asarray(e, np.float64) + 0.0 * np.asarray(v, np.float64)

    def __add__(self, o):
        o = o if isinstance(o, _V) else _V(o)
        r = self.v + o.v
        return _V(r, self.e + o.e + U * np.abs(r))

    def __sub__(self, o):
        o = o if isinstance(o, _V) else _V(o)
        r = self.v - o.v
        return _V(r, self.e + o.e + U * np.abs(r))

    def __rsub__(self, o):
        return _V(o) - self

    def __mul__(self, o):
        o = o if isinstance(o, _V) else _V(o)
        r = self.v * o.v
        return _V(r, np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e + U * np.abs(r))


def _sigmoid(a):
    g = 1.0 / (1.0 + np.exp(-a.v))
    return _V(g, g * (1.0 - g) * a.e + 8 * U * g)


def _act(activation, c):
    if activation == 1:
        t = np.tanh(c.v)
        return _V(t, (1.0 - t * t) * c.e + 4 * U * np.abs(t))
    if activation == 2:
        return _V(np.maximum(c.v, 0.0), c.e)            # relu is 1-Lipschitz
    return c


def _time_order(a, d, bidirectional):
    """a [len, batch, dir*d, ...] with the columns j >= d reversed in time when bidirectional (an involution)."""
    a = np.array(a, np.float64, copy=True)
    if bidirectional:
        a[:, :, d:] = a[::-1, :, d:]
    return a


def sru(u, x, bias, d, bidirectional, activation, init=None, mask_h=None, grad_h=None, grad_last=None):
    """The recurrence and, given grad_h, its gradients.  Returns (values, bounds): dicts of h, c and, with grad_h,
    grad_u, grad_x (k = 3), grad_bias (summed over the batch) and grad_init."""
    u = np.asarray(u, np.float64)
    L, B, D, k = u.shape
    init = np.zeros((B, D)) if init is None else np.asarray(init, np.float64).reshape(B, D)
    mask = np.ones((B, D)) if mask_h is None else np.asarray(mask_h, np.float64).reshape(B, D)
    b1, b2 = np.asarray(bias, np.float64)[:D], np.asarray(bias, np.float64)[D:]
    uo = _time_order(u, d, bidirectional)
    xo = uo[..., 3] if k == 4 else _time_order(x, d, bidirectional)
    g1s, g2s, cs = [], [], []
    hv, he, cv, ce = (np.empty((L, B, D)) for _ in range(4))
    cur = _V(init)
    for t in range(L):
        g1, g2 = _sigmoid(_V(uo[t, ..., 1]) + _V(b1)), _sigmoid(_V(uo[t, ..., 2]) + _V(b2))
        u0, xv = _V(uo[t, ..., 0]), _V(xo[t])
        cur = (cur - u0) * g1 + u0
        h = (_act(activation, cur) * _V(mask) - xv) * g2 + xv
        g1s.append(g1), g2s.append(g2), cs.append(cur)
        hv[t], he[t], cv[t], ce[t] = h.v, h.e, cur.v, cur.e
    vals = {"h": _time_order(hv, d, bidirectional), "c": _time_order(cv, d, bidirectional)}
    errs = {"h": _time_order(he, d, bidirectional), "c": _time_order(ce, d, bidirectional)}
    if grad_h is not None:
        gho = _time_order(grad_h, d, bidirectional)
        gl = np.zeros((B, D)) if grad_last is None else np.asarray(grad_last, np.float64).reshape(B, D)
        gu, gue, gx, gxe = np.empty((L, B, D, k)), np.empty((L, B, D, k)), np.empty((L, B, D)), np.empty((L, B, D))
        cur, gb1, gb2 = _V(gl), _V(np.zeros((B, D))), _V(np.zeros((B, D)))
        for t in range(L - 1, -1, -1):
            g1, g2, c = g1s[t], g2s[t], cs[t]
            prev = cs[t - 1] if t > 0 else _V(init)
            gh, xv, u0 = _V(gho[t]), _V(xo[t]), _V(uo[t, ..., 0])
            cval = _act(activation, c)
            gxt = gh * (1 - g2)
            gg2 = gh * (cval * _V(mask) - xv) * (g2 * (1 - g2))
            gb2 = gb2 + gg2
            if activation == 1:
                tmp = g2 * (1 - cval * cval)
            elif activation == 2:
                pos = cval.v > 0
                tmp = _V(np.where(pos, g2.v, 0.0), np.where(np.abs(c.v) <= c.e, g2.v + g2.e, np.where(pos, g2.e, 0.0)))
            else:
                tmp = g2
            gc = gh * _V(mask) * tmp + cur
            gu0 = gc * (1 - g1)
            gg1 = gc * (prev - u0) * (g1 * (1 - g1))
            gb1 = gb1 + gg1
            cur = gc * g1
            gu[t, ..., 0], gu[t, ..., 1], gu[t, ..., 2] = gu0.v, gg1.v, gg2.v
            gue[t, ..., 0], gue[t, ..., 1], gue[t, ..., 2] = gu0.e, gg1.e, gg2.e
            if k == 4:
                gu[t, ..., 3], gue[t, ..., 3] = gxt.v, gxt.e
            gx[t], gxe[t] = gxt.v, gxt.e
        vals["grad_u"], errs["grad_u"] = _time_order(gu, d, bidirectional), _time_order(gue, d, bidirectional)
        if k == 3:
            vals["grad_x"], errs["grad_x"] = _time_order(gx, d, bidirectional), _time_order(gxe, d, bidirectional)
        vals["grad_init"], errs["grad_init"] = cur.v, cur.e
        # the batch sum of the per-(batch, column) partials, in b order
        parts = np.stack([gb1.v, gb2.v])                 # [2, B, D]
        perr = np.stack([gb1.e, gb2.e])
        vals["grad_bias"] = parts.sum(1).reshape(-1)
        errs["grad_bias"] = (perr.sum(1) + B * U * np.abs(parts).sum(1)).reshape(-1)
    return vals, errs


def bounds(errs, length):
    """The per-element bounds the tests allow: twice the propagated first-order bound plus 2^-140 per step."""
    return {k: 2.0 * e + TINY * (length + 2) for k, e in errs.items()}
