"""CPU oracle of onmt's global attention for attn_type "mlp" (Bahdanau; onmt/modules/GlobalAttention.py:93-106,
108-188) and of its fused core (qd_attn_mlp_fwd, qd_attn_mlp_bwd) -- TEST INFRASTRUCTURE ONLY.

The reference's forward restated in float64 torch, gradients through autograd:
  score[n, t, s] = v . tanh(wq[n, t] + uh[n, s]),  wq = linear_query(input) (with bias), uh = linear_context(context)
  align = softmax over s;  c = sum_s align_s context[n, s];  concat = [c | input];  attn_h = linear_out(concat)
with its bias and no tanh.  The core is evaluated one batch entry at a time, so the [T, S, H] tanh of the largest
test shapes stays small; grad_v is summed over the entries.

mlp_core_bounds gives the error bounds of the float32 kernels stated in include/qd_b200.h, propagated to first order
and doubled, in the way attention_oracle.core_bounds does for "dot" and "general".
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .attention_oracle import TINY, U, _t

def mlp_core(wq, uh, v, inp, ctx, grad_align=None, grad_concat=None):
    """The fused "mlp" core in float64: dict of align [T, N, S], concat [T, N, 2H] and, given upstream gradients
    (either may be None), grad_wq, grad_uh ([N, S, H]), grad_v ([H]), grad_input (through the concat only) and
    grad_context ([N, S, H])."""
    wq, uh, inp, ctx = (np.asarray(a, np.float64) for a in (wq, uh, inp, ctx))
    v = np.asarray(v, np.float64).reshape(-1)
    Nb, T, H = wq.shape
    S = ctx.shape[1]
    grads = grad_align is not None or grad_concat is not None
    out = {"align": np.zeros((T, Nb, S)), "concat": np.zeros((T, Nb, 2 * H))}
    if grads:
        out.update(grad_wq=np.zeros_like(wq), grad_uh=np.zeros_like(uh), grad_v=np.zeros(H),
                   grad_input=np.zeros_like(inp), grad_context=np.zeros_like(ctx))
    for n in range(Nb):
        q_, u_, v_, i_, c_ = _t(wq[n]), _t(uh[n]), _t(v), _t(inp[n]), _t(ctx[n])
        e = torch.tanh(q_.unsqueeze(1) + u_.unsqueeze(0))                 # [T, S, H]
        align = torch.softmax(e @ v_, dim=1)                              # [T, S]
        concat = torch.cat([align @ c_, i_], 1)                           # [T, 2H]
        out["align"][:, n] = align.detach().numpy()
        out["concat"][:, n] = concat.detach().numpy()
        if not grads:
            continue
        loss = 0
        if grad_align is not None:
            loss = loss + (align * torch.tensor(np.asarray(grad_align, np.float64)[:, n])).sum()
        if grad_concat is not None:
            loss = loss + (concat * torch.tensor(np.asarray(grad_concat, np.float64)[:, n])).sum()
        loss.backward()
        out["grad_wq"][n], out["grad_uh"][n], out["grad_input"][n] = q_.grad.numpy(), u_.grad.numpy(), i_.grad.numpy()
        out["grad_context"][n] = c_.grad.numpy()
        out["grad_v"] += v_.grad.numpy()
    return out


def mlp_global_attention(input, context, w_ctx, w_q, b_q, v, w_out, b_out, grad_h=None, grad_align=None):
    """The reference's GlobalAttention.forward for attn_type "mlp" in float64, as the reference computes it (the
    [N, T, S, H] expansion): input [N, H] or [N, T, H], context [N, S, H]; w_ctx, w_q [H, H], b_q [H], v [1, H],
    w_out [H, 2H], b_out [H].  Returns attn_h, align and, with upstream gradients of both outputs, the gradients of
    input, context and every weight (grad_w_ctx, grad_w_q, grad_b_q, grad_v, grad_w_out, grad_b_out)."""
    i_, c_ = _t(input), _t(context)
    ws = {k: _t(a) for k, a in (("w_ctx", w_ctx), ("w_q", w_q), ("b_q", b_q), ("v", v), ("w_out", w_out),
                                ("b_out", b_out))}
    one_step = i_.dim() == 2
    x = i_.unsqueeze(1) if one_step else i_
    Nb, T, H = x.shape
    S = c_.shape[1]
    wq = (x @ ws["w_q"].t() + ws["b_q"]).unsqueeze(2).expand(Nb, T, S, H)
    uh = (c_ @ ws["w_ctx"].t()).unsqueeze(1).expand(Nb, T, S, H)
    score = (torch.tanh(wq + uh) @ ws["v"].t()).squeeze(3)
    align = torch.softmax(score, dim=2)
    attn_h = torch.cat([torch.bmm(align, c_), x], 2) @ ws["w_out"].t() + ws["b_out"]
    if one_step:
        attn_h, align = attn_h.squeeze(1), align.squeeze(1)
    else:
        attn_h, align = attn_h.transpose(0, 1), align.transpose(0, 1)
    out = {"attn_h": attn_h.detach().numpy(), "align": align.detach().numpy()}
    if grad_h is not None:
        loss = (attn_h * torch.tensor(grad_h)).sum() + (align * torch.tensor(grad_align)).sum()
        loss.backward()
        out.update(grad_input=i_.grad.numpy(), grad_context=c_.grad.numpy())
        out.update({f"grad_{k}": w.grad.numpy() for k, w in ws.items()})
    return out


def mlp_core_bounds(wq, uh, v, inp, ctx, grad_align=None, grad_concat=None):
    """Per-element error bounds of the float32 "mlp" kernels against mlp_core(): align, c (= concat[..., :H]; the
    input half is copied exactly) and, given grad_concat, grad_wq, grad_uh, grad_v and grad_context.  e = tanhf(fl(wq
    + uh)) is within 2 ulp (4u |e|) of tanh of its rounded argument, which is within u |wq + uh|."""
    wq, uh, ctx = (np.asarray(a, np.float64) for a in (wq, uh, ctx))
    v = np.asarray(v, np.float64).reshape(-1)
    av = np.abs(v)
    Nb, T, H = wq.shape
    S = ctx.shape[1]
    cH, cS = math.ceil(H / 32) + 6, math.ceil(S / 32) + 6
    chunks = -(-S // 8)
    grads = grad_concat is not None
    b = {"align": np.zeros((T, Nb, S)), "c": np.zeros((T, Nb, H))}
    if grads:
        gcs = np.asarray(grad_concat, np.float64)[:, :, :H]
        gas = None if grad_align is None else np.asarray(grad_align, np.float64)
        b.update(grad_wq=np.zeros((Nb, T, H)), grad_uh=np.zeros((Nb, S, H)), grad_context=np.zeros((Nb, S, H)))
        gv_err, gv_abs = np.zeros(H), np.zeros(H)
    for n in range(Nb):
        x = wq[n][:, None, :] + uh[n][None, :, :]                          # [T, S, H]
        e = np.tanh(x)
        de = 1 - e * e
        E_e = 4 * U * np.abs(e) + U * de * np.abs(x) + 2 * TINY
        score = e @ v
        e_score = cH * U * (np.abs(e) @ av) + E_e @ av + (H + 2) * TINY
        p = np.exp(score - score.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        dx = U * np.abs(score - score.max(1, keepdims=True))
        e_p = p * (2 * e_score.max(1, keepdims=True) + dx + (p * dx).sum(1, keepdims=True) + (cS + 8) * U) + 8 * TINY
        actx = np.abs(ctx[n])
        e_c = e_p @ actx + (S + 2) * U * (p @ actx) + (S + 2) * TINY
        b["align"][:, n], b["c"][:, n] = 2 * e_p, 2 * e_c
        if not grads:
            continue
        gc = gcs[:, n]                                                    # [T, H]
        ga_add = np.zeros_like(p) if gas is None else gas[:, n]
        ga = gc @ ctx[n].T + ga_add
        e_ga = cH * U * (np.abs(gc) @ actx.T + np.abs(ga_add)) + (H + 2) * TINY
        D = (p * ga).sum(1, keepdims=True)
        e_D = (e_p * np.abs(ga) + p * e_ga).sum(1, keepdims=True) + cS * U * (p * np.abs(ga)).sum(1, keepdims=True)
        gs = p * (ga - D)
        e_gs = e_p * np.abs(ga - D) + p * (e_ga + e_D) + 3 * U * p * (np.abs(ga) + np.abs(D)) + 3 * TINY
        ags = np.abs(gs)[:, :, None]
        d_abs = ags * av * de                                             # |terms| gs v (1 - e^2)
        e_d = (e_gs[:, :, None] * av * de + ags * av * (2 * np.abs(e) * E_e + U * e * e + 3 * U * de) + 3 * TINY)
        b["grad_wq"][n] = 2 * (e_d.sum(1) + (S + 2) * U * d_abs.sum(1) + (S + 2) * TINY)
        b["grad_uh"][n] = 2 * (e_d.sum(0) + (T + 2) * U * d_abs.sum(0) + (T + 2) * TINY)
        agc = np.abs(gc)
        b["grad_context"][n] = 2 * (e_p.T @ agc + (T + 2) * U * (p.T @ agc) + (T + 2) * TINY)
        gv_err += (e_gs[:, :, None] * np.abs(e) + ags * E_e + U * ags * np.abs(e) + TINY).sum((0, 1))
        gv_abs += (ags * np.abs(e)).sum((0, 1))
    if grads:
        k = 8 * T + Nb * chunks
        b["grad_v"] = 2 * (gv_err + (k + 2) * U * gv_abs + (k + 2) * TINY)
    return b
