"""CPU oracle of onmt's global attention (onmt/modules/GlobalAttention.py:108-188, "dot" and "general") and of its
fused core (qd_attn_fwd, qd_attn_bwd) -- TEST INFRASTRUCTURE ONLY.

The reference's forward restated in float64 torch, gradients through autograd:
  score[n, t, s] = q[n, t] . context[n, s]         q = linear_in(input) for "general", input for "dot"
  align = softmax over s;  c = sum_s align_s context[n, s];  concat = [c | input]
  attn_h = tanh(linear_out(concat))
Outputs in the reference's order: one step [N, H] / [N, S]; multi-step [T, N, H] / [T, N, S].

core_bounds gives the error bounds of the float32 kernels stated in include/qd_b200.h, propagated through the chain
from the float64 values: a sum of k terms in the kernels' orders is within (ceil(k/32) + 6) u sum|terms| (the lane
sums) or (k + 2) u sum|terms| (the ordered sums), u = 2^-24; each float32 operation may add 2^-149 more where its
result is subnormal.  The propagated bound is doubled: the first-order propagation through the softmax drops
second-order terms, which the peaked rows of random inputs at H >= 500 come close to.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
TINY = 2.0 ** -149        # the spacing of float32 subnormals


def _t(x):
    return torch.tensor(np.asarray(x, dtype=np.float64), dtype=torch.float64, requires_grad=True)


def _core(q, inp, ctx):
    """align [T, N, S], concat [T, N, 2H] of q, inp [N, T, H] and ctx [N, S, H] (float64 torch)."""
    align = torch.softmax(torch.bmm(q, ctx.transpose(1, 2)), dim=2)
    c = torch.bmm(align, ctx)
    return align.transpose(0, 1), torch.cat([c, inp], 2).transpose(0, 1)


def core(q, inp, ctx, grad_align=None, grad_concat=None):
    """The fused core in float64: dict of align, concat and, given upstream gradients (either may be None),
    grad_q, grad_input (through the concat only) and grad_context ([N, S, H])."""
    q_, i_, c_ = _t(q), _t(inp), _t(ctx)
    align, concat = _core(q_, i_, c_)
    out = {"align": align.detach().numpy(), "concat": concat.detach().numpy()}
    if grad_align is None and grad_concat is None:
        return out
    loss = 0
    if grad_align is not None:
        loss = loss + (align * torch.tensor(np.asarray(grad_align, np.float64))).sum()
    if grad_concat is not None:
        loss = loss + (concat * torch.tensor(np.asarray(grad_concat, np.float64))).sum()
    loss.backward()
    out.update(grad_q=q_.grad.numpy(), grad_input=i_.grad.numpy(), grad_context=c_.grad.numpy())
    return out


def global_attention(input, context, attn_type, w_in, w_out, grad_h=None, grad_align=None):
    """The reference's GlobalAttention.forward in float64: input [N, H] or [N, T, H], context [N, S, H] (the view the
    decoders pass), w_in [H, H] ("general" only), w_out [H, 2H].  Returns attn_h, align and, with upstream gradients of
    both outputs, the gradients of input, context, w_in and w_out."""
    i_, c_, wo = _t(input), _t(context), _t(w_out)
    wi = _t(w_in) if attn_type == "general" else None
    one_step = i_.dim() == 2
    x = i_.unsqueeze(1) if one_step else i_
    q = x @ wi.t() if attn_type == "general" else x
    align, concat = _core(q, x, c_)
    attn_h = torch.tanh(concat @ wo.t())
    if one_step:
        attn_h, align = attn_h.squeeze(0), align.squeeze(0)
    out = {"attn_h": attn_h.detach().numpy(), "align": align.detach().numpy()}
    if grad_h is not None:
        loss = (attn_h * torch.tensor(grad_h)).sum() + (align * torch.tensor(grad_align)).sum()
        loss.backward()
        out.update(grad_input=i_.grad.numpy(), grad_context=c_.grad.numpy(), grad_w_out=wo.grad.numpy())
        if wi is not None:
            out["grad_w_in"] = wi.grad.numpy()
    return out


def core_bounds(q, inp, ctx, grad_align=None, grad_concat=None):
    """Per-element error bounds of the float32 kernels against core(): align, c (= concat[..., :H]; the input half is
    copied exactly) and, given grad_concat, grad_q and grad_context."""
    q, ctx = np.asarray(q, np.float64), np.asarray(ctx, np.float64)
    Nb, T, H = q.shape
    S = ctx.shape[1]
    o = core(q, inp, ctx, grad_align, grad_concat)
    cH, cS = math.ceil(H / 32) + 6, math.ceil(S / 32) + 6
    p = o["align"].transpose(1, 0, 2)                                   # [N, T, S]
    actx = np.abs(ctx)
    e_score = cH * U * np.einsum("nth,nsh->nts", np.abs(q), actx)
    # x - m is rounded before the exponential: a relative error of u |x - m| in each term and in their sum
    x = np.einsum("nth,nsh->nts", q, ctx)
    dx = U * np.abs(x - x.max(axis=2, keepdims=True))
    e_p = p * (2 * e_score.max(axis=2, keepdims=True) + dx + (p * dx).sum(axis=2, keepdims=True) + (cS + 8) * U) + 8 * TINY
    e_c = np.einsum("nts,nsh->nth", e_p, actx) + (S + 2) * U * np.einsum("nts,nsh->nth", p, actx)
    e_c += (S + 2) * TINY
    b = {"align": 2 * e_p.transpose(1, 0, 2), "c": 2 * e_c.transpose(1, 0, 2)}
    if grad_concat is None:
        return b
    gc = np.asarray(grad_concat, np.float64).transpose(1, 0, 2)[:, :, :H]     # [N, T, H]
    ga_add = np.zeros_like(p) if grad_align is None else np.asarray(grad_align, np.float64).transpose(1, 0, 2)
    ga = np.einsum("nth,nsh->nts", gc, ctx) + ga_add
    e_ga = cH * U * (np.einsum("nth,nsh->nts", np.abs(gc), actx) + np.abs(ga_add)) + (H + 2) * TINY
    D = (p * ga).sum(axis=2, keepdims=True)
    e_D = (e_p * np.abs(ga) + p * e_ga).sum(axis=2, keepdims=True) + cS * U * (p * np.abs(ga)).sum(axis=2, keepdims=True)
    gs = p * (ga - D)
    e_gs = e_p * np.abs(ga - D) + p * (e_ga + e_D) + 3 * U * p * (np.abs(ga) + np.abs(D)) + 3 * TINY
    e_gq = (np.einsum("nts,nsh->nth", e_gs, actx) + (S + 2) * U * np.einsum("nts,nsh->nth", np.abs(gs), actx)
            + (S + 2) * TINY)
    aq = np.abs(q)
    e_gctx = (np.einsum("nts,nth->nsh", e_p, np.abs(gc)) + np.einsum("nts,nth->nsh", e_gs, aq)
              + (T + 3) * U * (np.einsum("nts,nth->nsh", p, np.abs(gc)) + np.einsum("nts,nth->nsh", np.abs(gs), aq))
              + 3 * (T + 1) * TINY)
    b.update(grad_q=2 * e_gq, grad_context=2 * e_gctx)
    return b
