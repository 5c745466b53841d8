"""CPU oracle of onmt's Transformer sublayers (onmt/modules/MultiHeadedAttn.py:44-110, onmt/modules/UtilClass.py:24-46,
onmt/modules/Transformer.py:17-40, 43-66, 107-164) and of their fused cores (qd_mha_fwd / qd_mha_bwd,
qd_onmt_layernorm_fwd / _bwd) -- TEST INFRASTRUCTURE ONLY.

The reference's forward restated in float64 torch, gradients through autograd:
  per head: x = (q_h . k_h) / sqrt(dh), -inf where masked;  p = softmax over the keys, computed twice as the reference
  does (once for top_attn = head 0, once for the dropout path);  out = sum_s p'_s v_s, p' = p keep / (1 - p_drop)
  layer norm: z = x + residual;  (z - mean) / (std_unbiased + eps) * a_2 + b_2;  z itself when the width is 1
Module-level chains take a state_dict-like mapping of the reference's parameter names to arrays and return the
gradients under the same names.

core_bounds and layer_norm_bounds give the error bounds of the float32 kernels stated in include/qd_b200.h, propagated
to first order from the float64 values: a sum of k terms in the kernels' orders is within (ceil(k/32) + 6) u sum|terms|
(lane sums) or (k + 2) u sum|terms| (ordered sums), u = 2^-24, and each float32 operation may add 2^-149 more where its
result is subnormal.  The propagated bound is doubled, as in attention_oracle: first-order propagation through the
softmax and the normalisation drops second-order terms.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
TINY = 2.0 ** -149        # the spacing of float32 subnormals


def _t(x, grad=True):
    return torch.tensor(np.asarray(x, dtype=np.float64), dtype=torch.float64, requires_grad=grad)


def _core(q, k, v, heads, mask, keep, p):
    """out [B, Lq, D], top [B, Lq, Lk] of the reference's chain between the projections and the residual."""
    B, Lq, D = q.shape
    Lk = k.shape[1]
    dh = D // heads

    def shape(x):
        b, L, _ = x.shape
        return x.view(b, L, heads, dh).transpose(1, 2).contiguous().view(b * heads, L, dh)

    scaled = torch.bmm(shape(q), shape(k).transpose(1, 2)) / math.sqrt(dh)
    if mask is not None:
        m = torch.as_tensor(np.asarray(mask)).bool().unsqueeze(1).expand(B, heads, Lq, Lk)
        scaled = scaled.view(B, heads, Lq, Lk).masked_fill(m, -float("inf")).view(B * heads, Lq, Lk)
    top = torch.softmax(scaled, dim=-1).view(B, heads, Lq, Lk)[:, 0].contiguous()
    drop = torch.softmax(scaled, dim=-1)
    if keep is not None:
        drop = drop * torch.as_tensor(np.asarray(keep, np.float64)) * (1.0 / (1.0 - p))
    out = torch.bmm(drop, shape(v)).view(B, heads, Lq, dh).transpose(1, 2).contiguous().view(B, Lq, D)
    return out, top


def core(q, k, v, heads, mask=None, keep=None, p=0.0, grad_out=None, grad_top=None):
    """The fused core in float64: dict of out and top and, given upstream gradients (either may be None), grad_q,
    grad_k and grad_v."""
    q_, k_, v_ = _t(q), _t(k), _t(v)
    out, top = _core(q_, k_, v_, heads, mask, keep, p)
    o = {"out": out.detach().numpy(), "top": top.detach().numpy()}
    if grad_out is None and grad_top is None:
        return o
    loss = 0
    if grad_out is not None:
        loss = loss + (out * torch.tensor(np.asarray(grad_out, np.float64))).nansum()
    if grad_top is not None:
        loss = loss + (top * torch.tensor(np.asarray(grad_top, np.float64))).nansum()
    loss.backward()
    o.update(grad_q=q_.grad.numpy(), grad_k=k_.grad.numpy(), grad_v=v_.grad.numpy())
    return o


def _layer_norm(z, a, b, eps):
    if z.shape[1] == 1:
        return z
    mu = z.mean(dim=1, keepdim=True)
    sigma = z.std(dim=1, keepdim=True)
    return (z - mu) / (sigma + eps) * a + b


def layer_norm(x, a_2, b_2, eps=1e-3, residual=None, grad_y=None):
    """onmt's LayerNorm of x (+ residual) [rows, d] in float64: y and, given grad_y, grad_x (= grad_residual),
    grad_a_2 and grad_b_2 (zeros when d = 1: the reference leaves them without a gradient)."""
    x_, a_, b_ = _t(x), _t(a_2), _t(b_2)
    z = x_ if residual is None else x_ + _t(residual, False)
    y = _layer_norm(z, a_, b_, eps)
    o = {"y": y.detach().numpy()}
    if grad_y is not None:
        (y * torch.tensor(np.asarray(grad_y, np.float64))).sum().backward()
        z0 = np.zeros(np.shape(a_2))
        o.update(grad_x=x_.grad.numpy(), grad_a_2=z0 if a_.grad is None else a_.grad.numpy(),
                 grad_b_2=z0 if b_.grad is None else b_.grad.numpy())
    return o


def bottle_layer_norm(x, a_2, b_2, eps=1e-3, grad_y=None):
    """BottleLayerNorm: 2-D input as layer_norm, 3-D over its flattened rows."""
    x = np.asarray(x, np.float64)
    if x.ndim == 2:
        return layer_norm(x, a_2, b_2, eps, None, grad_y)
    B, L, d = x.shape
    o = layer_norm(x.reshape(B * L, d), a_2, b_2, eps, None, None if grad_y is None else np.reshape(grad_y, (B * L, d)))
    o["y"] = o["y"].reshape(B, L, d)
    if "grad_x" in o:
        o["grad_x"] = o["grad_x"].reshape(B, L, d)
    return o


# ---- the reference's modules as chains over named parameters ----------------------------------------------------------
def _mha(P, pre, key, value, query, heads, mask):
    lin = lambda x, n: x @ P[f"{pre}{n}.weight"].t()
    out, top = _core(lin(query, "linear_query"), lin(key, "linear_keys"), lin(value, "linear_values"), heads, mask,
                     None, 0.0)
    z = out + query
    B, L, d = z.shape
    ret = _layer_norm(z.reshape(B * L, d), P[f"{pre}layer_norm.a_2"], P[f"{pre}layer_norm.b_2"], 1e-3).view(B, L, d)
    return ret, top


def _ffn(P, pre, x):
    B, L, d = x.shape
    h = torch.relu(x.reshape(B * L, d) @ P[f"{pre}w_1.weight"].t() + P[f"{pre}w_1.bias"])
    o = (h @ P[f"{pre}w_2.weight"].t() + P[f"{pre}w_2.bias"]) + x.reshape(B * L, d)
    return _layer_norm(o, P[f"{pre}layer_norm.a_2"], P[f"{pre}layer_norm.b_2"], 1e-3).view(B, L, d)


def _run(params, inputs, fn, grads):
    """Runs fn(P, *inputs) in float64 with every parameter and float input a leaf; with upstream gradients of its
    outputs (NaN terms dropped), returns the gradients of the inputs (grad_<i>) and of the parameters by name."""
    P = {n: _t(v) for n, v in params.items() if np.asarray(v).dtype.kind == "f"}
    X = [_t(x) if x is not None and np.asarray(x).dtype.kind == "f" else x for x in inputs]
    outs = fn(P, *X)
    o = {f"out{i}": t.detach().numpy() for i, t in enumerate(outs)}
    if grads is not None:
        loss = sum((t * torch.tensor(np.asarray(g, np.float64))).nansum() for t, g in zip(outs, grads) if g is not None)
        loss.backward()
        for i, x in enumerate(X):
            if isinstance(x, torch.Tensor) and x.requires_grad:
                o[f"grad_in{i}"] = x.grad.numpy()
        for n, t in P.items():
            o[f"grad_{n}"] = np.zeros(t.shape) if t.grad is None else t.grad.numpy()
    return o


def multi_headed_attention(params, key, value, query, heads, mask=None, grads=None):
    """MultiHeadedAttention in eval mode: out0 = ret, out1 = top_attn."""
    return _run(params, [key, value, query], lambda P, k, v, q: _mha(P, "", k, v, q, heads, mask), grads)


def feed_forward(params, x, grads=None):
    """PositionwiseFeedForward in eval mode: out0."""
    return _run(params, [x], lambda P, x: (_ffn(P, "", x),), grads)


def encoder_layer(params, x, mask, heads, grads=None):
    """TransformerEncoderLayer(input, mask) in eval mode: out0."""
    return _run(params, [x], lambda P, x: (_ffn(P, "feed_forward.", _mha(P, "self_attn.", x, x, x, heads, mask)[0]),),
                grads)


def subsequent_mask(L):
    return np.triu(np.ones((1, L, L)), k=1).astype(np.uint8)


def decoder_layer(params, x, context, src_pad_mask, tgt_pad_mask, heads, grads=None):
    """TransformerDecoderLayer(input, context, src_pad_mask, tgt_pad_mask) in eval mode: out0 = output, out1 = the
    context attention's top_attn.  The self-attention mask is tgt_pad_mask + the subsequent mask > 0."""
    T = x.shape[1]
    dec_mask = (np.asarray(tgt_pad_mask, np.int64) + subsequent_mask(T)) > 0

    def fn(P, x, c):
        q, _ = _mha(P, "self_attn.", x, x, x, heads, dec_mask)
        mid, attn = _mha(P, "context_attn.", c, c, q, heads, src_pad_mask)
        return _ffn(P, "feed_forward.", mid), attn
    return _run(params, [x, context], fn, grads)


# ---- error bounds of the float32 kernels ------------------------------------------------------------------------------
def _heads(x, heads):
    """[B, L, D] -> [B, heads, L, dh]"""
    B, L, D = x.shape
    return np.asarray(x, np.float64).reshape(B, L, heads, D // heads).transpose(0, 2, 1, 3)


def _unheads(x):
    B, h, L, dh = x.shape
    return x.transpose(0, 2, 1, 3).reshape(B, L, h * dh)


def core_bounds(q, k, v, heads, mask=None, keep=None, p=0.0, grad_out=None, grad_top=None):
    """Per-element error bounds of the float32 kernels against core(): out, top and, given grad_out, grad_q, grad_k and
    grad_v.  Entries the reference gives as NaN (an all-masked row) get bound 0; compare them for NaN separately."""
    qh, kh, vh = _heads(q, heads), _heads(k, heads), _heads(v, heads)
    B, h, Lq, dh = qh.shape
    Lk = kh.shape[2]
    r = math.sqrt(dh)
    cH, cS = math.ceil(dh / 32) + 6, math.ceil(Lk / 32) + 6
    m = np.zeros((B, 1, Lq, Lk), bool) if mask is None else np.asarray(mask).astype(bool)[:, None]
    x = np.einsum("bhtj,bhsj->bhts", qh, kh) / r
    x = np.where(m, -np.inf, x)
    e_x = (cH + 2) * U * np.einsum("bhtj,bhsj->bhts", np.abs(qh), np.abs(kh)) / r
    e_x = np.where(m, 0.0, e_x)
    with np.errstate(invalid="ignore", divide="ignore"):
        xm = x.max(axis=3, keepdims=True)
        ex = np.exp(x - xm)
        P = ex / ex.sum(axis=3, keepdims=True)
        dx = np.where(m, 0.0, U * np.abs(x - xm))
    dead = ~np.isfinite(xm)                                       # all-masked rows: NaN in the reference
    P = np.where(dead, 0.0, P)
    dx = np.where(dead, 0.0, dx)
    e_p = P * (2 * e_x.max(axis=3, keepdims=True) + dx + (P * dx).sum(axis=3, keepdims=True) + (cS + 8) * U) + 8 * TINY
    kp = np.ones_like(P) if keep is None else np.asarray(keep, np.float64).reshape(B, h, Lq, Lk) / (1.0 - p)
    Pd = P * kp
    e_pd = kp * e_p + 2 * U * Pd
    av = np.abs(vh)
    e_out = np.einsum("bhts,bhsj->bhtj", e_pd, av) + (Lk + 2) * U * np.einsum("bhts,bhsj->bhtj", Pd, av) + (Lk + 2) * TINY
    b = {"out": 2 * _unheads(e_out), "top": 2 * e_p[:, 0]}
    if grad_out is None:
        return b
    go = _heads(grad_out, heads)
    gt = np.zeros((B, Lq, Lk)) if grad_top is None else np.asarray(grad_top, np.float64)
    gpd = np.einsum("bhtj,bhsj->bhts", go, vh)
    e_gpd = cH * U * np.einsum("bhtj,bhsj->bhts", np.abs(go), av) + (dh + 2) * TINY
    G = gpd * kp
    G[:, 0] += gt
    e_G = kp * e_gpd + 3 * U * (np.abs(gpd * kp) + np.abs(G))
    D = (P * G).sum(axis=3, keepdims=True)
    e_D = (e_p * np.abs(G) + P * e_G).sum(axis=3, keepdims=True) + cS * U * (P * np.abs(G)).sum(axis=3, keepdims=True)
    dS = P * (G - D) / r
    e_dS = (e_p * np.abs(G - D) + P * (e_G + e_D) + 3 * U * P * (np.abs(G) + np.abs(D))) / r + 2 * U * np.abs(dS) + 3 * TINY
    dS = np.where(m, 0.0, dS)
    e_dS = np.where(m | dead, 0.0, e_dS)
    ak, aq, ago = np.abs(kh), np.abs(qh), np.abs(go)
    e_gq = (np.einsum("bhts,bhsj->bhtj", e_dS, ak) + (Lk + 2) * U * np.einsum("bhts,bhsj->bhtj", np.abs(dS), ak)
            + (Lk + 2) * TINY)
    e_gk = (np.einsum("bhts,bhtj->bhsj", e_dS, aq) + (Lq + 2) * U * np.einsum("bhts,bhtj->bhsj", np.abs(dS), aq)
            + (Lq + 2) * TINY)
    e_gv = (np.einsum("bhts,bhtj->bhsj", e_pd, ago) + (Lq + 2) * U * np.einsum("bhts,bhtj->bhsj", Pd, ago)
            + (Lq + 2) * TINY)
    b.update(grad_q=2 * _unheads(e_gq), grad_k=2 * _unheads(e_gk), grad_v=2 * _unheads(e_gv))
    return b


def layer_norm_bounds(x, a_2, b_2, eps=1e-3, residual=None, grad_y=None):
    """Per-element error bounds of the float32 kernels against layer_norm(): y and, given grad_y, grad_x, grad_a_2 and
    grad_b_2.  Width 1 is exact (bound 0) but for the residual add."""
    x = np.asarray(x, np.float64)
    a, bb = np.asarray(a_2, np.float64), np.asarray(b_2, np.float64)
    z = x if residual is None else x + np.asarray(residual, np.float64)
    rows, d = z.shape
    e_z = np.zeros_like(z) if residual is None else U * np.abs(z)
    if d == 1:
        out = {"y": 2 * e_z}
        if grad_y is not None:
            out.update(grad_x=np.zeros_like(z), grad_a_2=np.zeros(1), grad_b_2=np.zeros(1))
        return out
    cd = math.ceil(d / 32) + 6
    az = np.abs(z)
    mu = z.mean(axis=1, keepdims=True)
    e_mu = U * np.abs(mu) + (cd + 1) * U * az.sum(axis=1, keepdims=True) / d + e_z.sum(axis=1, keepdims=True) / d
    c = z - mu
    e_c = e_z + e_mu + U * np.abs(c)
    ss = (c * c).sum(axis=1, keepdims=True)
    e_ss = (2 * np.abs(c) * e_c).sum(axis=1, keepdims=True) + (cd + 1) * U * ss
    var = ss / (d - 1)
    e_var = e_ss / (d - 1) + U * var
    s = np.sqrt(var)
    e_s = e_var / (2 * s) + U * s
    Dn = s + eps
    e_D = e_s + U * Dn
    xh = c / Dn
    e_xh = e_c / Dn + np.abs(c) * e_D / Dn ** 2 + U * np.abs(xh)
    y = xh * a + bb
    e_y = e_xh * np.abs(a) + U * np.abs(xh * a) + U * np.abs(y) + 3 * TINY
    out = {"y": 2 * e_y}
    if grad_y is None:
        return out
    dy = np.asarray(grad_y, np.float64)
    g = dy * a
    e_g = U * np.abs(g)
    mg = g.mean(axis=1, keepdims=True)
    e_mg = (cd + 1) * U * np.abs(g).sum(axis=1, keepdims=True) / d + e_g.sum(axis=1, keepdims=True) / d + U * np.abs(mg)
    sgc = (g * c).sum(axis=1, keepdims=True)
    e_sgc = (e_g * np.abs(c) + np.abs(g) * e_c).sum(axis=1, keepdims=True) + (cd + 1) * U * np.abs(g * c).sum(axis=1, keepdims=True)
    den = Dn ** 2 * (d - 1) * s
    kc = -sgc / den
    e_k = e_sgc / den + np.abs(kc) * (2 * e_D / Dn + e_s / s + 6 * U)
    t1 = (g - mg) / Dn
    e_1 = (e_g + e_mg + U * np.abs(g - mg)) / Dn + np.abs(g - mg) * e_D / Dn ** 2 + U * np.abs(t1)
    gx = t1 + kc * c
    e_gx = e_1 + e_k * np.abs(c) + np.abs(kc) * e_c + U * np.abs(kc * c) + U * np.abs(gx) + 4 * TINY
    ady = np.abs(dy)
    e_ga = (ady * e_xh).sum(axis=0) + (rows + 2) * U * (ady * np.abs(xh)).sum(axis=0) + (rows + 2) * TINY
    e_gb = (rows + 2) * U * ady.sum(axis=0)
    out.update(grad_x=2 * e_gx, grad_a_2=2 * e_ga, grad_b_2=2 * e_gb)
    return out
