"""onmt's Transformer sublayers (onmt/modules/MultiHeadedAttn.py, onmt/modules/UtilClass.py:24-46) with their cores in
fused kernels (qd_mha_fwd / qd_mha_bwd, qd_onmt_layernorm_fwd / _bwd).

The reference runs each attention sublayer as three transpose copies in and one out, a bmm, a division, a masked_fill
on an expanded mask, the softmax twice (once for top_attn, once for the dropout path), a bmm and a head-0 slice copy,
then its own LayerNorm as about seven elementwise and reduction kernels.  Here the Linears still run as modules (cuBLAS,
or PackedLinear after codec.attach_packed_); the attention core between them is one launch forward and two backward,
read and written in the projections' own [B, L, heads*dh] layout, and the residual add with the layer norm is one
launch forward and two backward.

    mha_core(q, k, v, heads, mask=None, keep=None, p=0.0) -> (out [B, Lq, D], top_attn [B, Lq, Lk])
    onmt_layer_norm(x, a_2, b_2, eps, residual=None) -> y
    MultiHeadedAttention(head_count, model_dim, p=0.1)
    LayerNorm(d_hid, eps=1e-3), BottleLayerNorm(d_hid, eps=1e-3)

There is no CPU implementation: CPU or non-float32 tensors raise ValueError.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from . import _native as N


def _as_bytes(m):
    """uint8 view of a bool or uint8 tensor, strides kept (a stride-0 expanded mask stays a view)."""
    return m.view(torch.uint8) if m.dtype == torch.bool else m


def _mask_args(mask):
    if mask is None:
        return None, 0, 0, 0
    return N.ptr(mask), mask.stride(0), mask.stride(1), mask.stride(2)


class _MhaCore(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, heads, mask, keep, scale):
        B, Lq, D = q.shape
        Lk = k.shape[1]
        dh = D // heads
        dev = q.device
        out = torch.empty(B, Lq, D, dtype=torch.float32, device=dev)
        probs = torch.empty(B, heads, Lq, Lk, dtype=torch.float32, device=dev)
        top = torch.empty(B, Lq, Lk, dtype=torch.float32, device=dev)
        mp, mb, mq, mk = _mask_args(mask)
        with torch.cuda.device(dev):
            N.check(N.lib().qd_mha_fwd(N.ptr(q), N.ptr(k), N.ptr(v), mp, mb, mq, mk, N.ptr(keep), scale, B, Lq, Lk,
                                       heads, dh, N.ptr(out), N.ptr(probs), N.ptr(top), N.stream_ptr(dev)))
        ctx.heads, ctx.scale, ctx.mask = heads, scale, mask
        ctx.save_for_backward(q, k, v, probs, keep)
        return out, top

    @staticmethod
    def backward(ctx, grad_out, grad_top):
        q, k, v, probs, keep = ctx.saved_tensors
        B, Lq, D = q.shape
        Lk = k.shape[1]
        heads = ctx.heads
        dev = q.device
        if grad_out is None:
            grad_out = torch.zeros(B, Lq, D, dtype=torch.float32, device=dev)
        grad_out = grad_out.contiguous()
        grad_top = None if grad_top is None else grad_top.contiguous()
        grad_q, grad_k, grad_v = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        mp, mb, mq, mk = _mask_args(ctx.mask)
        with torch.cuda.device(dev):
            ws = torch.empty(int(N.lib().qd_mha_workspace_bytes(B, heads, Lq, Lk)), dtype=torch.uint8, device=dev)
            N.check(N.lib().qd_mha_bwd(N.ptr(grad_out), N.ptr(grad_top), N.ptr(q), N.ptr(k), N.ptr(v), N.ptr(probs), mp,
                                       mb, mq, mk, N.ptr(keep), ctx.scale, B, Lq, Lk, heads, D // heads, N.ptr(grad_q),
                                       N.ptr(grad_k), N.ptr(grad_v), N.ptr(ws), ws.numel(), N.stream_ptr(dev)))
        return grad_q, grad_k, grad_v, None, None, None, None


def mha_core(q, k, v, heads, mask=None, keep=None, p=0.0):
    """(out, top_attn) of the attention core of onmt's MultiHeadedAttention for the projections q [B, Lq, D] and k, v
    [B, Lk, D], D = heads * dh, in their own layout.  mask: bool or uint8 [B, Lq, Lk] (any strides, nonzero = masked,
    so onmt's expanded padding masks are read in place) or None.  keep: uint8 or bool [B*heads, Lq, Lk], the dropout
    draw of the attention probabilities (1 = kept), scaled by 1/(1-p); None for no dropout.
    out: [B, Lq, D] = sum_s p' v_s per head, unshaped as the reference; top_attn: head 0's probabilities [B, Lq, Lk].
    Differentiable in q, k and v (through both outputs).  The backward saves q, k, v, the probabilities and keep."""
    N.require_cuda()
    N.check_float_cuda(q, "q", 3)
    N.check_float_cuda(k, "k", 3)
    N.check_float_cuda(v, "v", 3)
    if not isinstance(heads, int) or heads < 1:
        raise ValueError("heads must be a positive int")
    B, Lq, D = q.shape
    if k.shape != v.shape or k.shape[0] != B or k.shape[2] != D:
        raise ValueError(f"shapes do not match: q {tuple(q.shape)}, k {tuple(k.shape)}, v {tuple(v.shape)}")
    if D % heads != 0:
        raise ValueError(f"the width {D} is not divisible by heads = {heads}")
    Lk = k.shape[1]
    if B == 0 or Lq == 0 or Lk == 0 or D == 0:
        raise ValueError("q, k and v must not be empty")
    if k.device != q.device or v.device != q.device:
        raise ValueError("q, k and v must be on the same device")
    if mask is not None:
        if not isinstance(mask, torch.Tensor) or mask.dtype not in (torch.bool, torch.uint8) or mask.device != q.device:
            raise ValueError("mask must be a bool or uint8 tensor on the device of q")
        if tuple(mask.shape) != (B, Lq, Lk):
            raise ValueError(f"mask must be [B, Lq, Lk] = {(B, Lq, Lk)}, got {tuple(mask.shape)}")
        mask = _as_bytes(mask)
        if any(s < 0 for s in mask.stride()):
            mask = mask.contiguous()
    scale = 1.0
    if keep is not None:
        if not isinstance(keep, torch.Tensor) or keep.dtype not in (torch.bool, torch.uint8) or keep.device != q.device:
            raise ValueError("keep must be a bool or uint8 tensor on the device of q")
        if tuple(keep.shape) != (B * heads, Lq, Lk):
            raise ValueError(f"keep must be [B*heads, Lq, Lk] = {(B * heads, Lq, Lk)}, got {tuple(keep.shape)}")
        if not 0.0 <= p < 1.0:
            raise ValueError(f"dropout p must be in [0, 1) with a keep mask, got {p}")
        keep = _as_bytes(keep).contiguous()
        scale = 1.0 / (1.0 - p)
    return _MhaCore.apply(q.contiguous(), k.contiguous(), v.contiguous(), heads, mask, keep, scale)


class _LayerNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, a_2, b_2, eps, residual):
        rows, d = x.shape
        y = torch.empty_like(x)
        dev = x.device
        with torch.cuda.device(dev):
            N.check(N.lib().qd_onmt_layernorm_fwd(N.ptr(x), N.ptr(residual), N.ptr(a_2), N.ptr(b_2), rows, d, eps,
                                                  N.ptr(y), N.stream_ptr(dev)))
        ctx.eps, ctx.has_residual = eps, residual is not None
        ctx.save_for_backward(x, a_2, residual)
        return y

    @staticmethod
    def backward(ctx, grad_y):
        x, a_2, residual = ctx.saved_tensors
        rows, d = x.shape
        dev = x.device
        grad_y = grad_y.contiguous()
        grad_x = torch.empty_like(x)
        grad_a, grad_b = torch.empty_like(a_2), torch.empty_like(a_2)
        with torch.cuda.device(dev):
            ws = torch.empty(int(N.lib().qd_onmt_layernorm_workspace_bytes(rows, d)), dtype=torch.uint8, device=dev)
            N.check(N.lib().qd_onmt_layernorm_bwd(N.ptr(grad_y), N.ptr(x), N.ptr(residual), N.ptr(a_2), rows, d, ctx.eps,
                                                  N.ptr(grad_x), N.ptr(grad_a), N.ptr(grad_b),
                                                  N.ptr(ws) if ws.numel() else None, ws.numel(), N.stream_ptr(dev)))
        if d == 1:                      # the reference returns z unchanged: a_2 and b_2 take no part
            grad_a = grad_b = None
        return grad_x, grad_a, grad_b, None, (grad_x if ctx.has_residual else None)


def onmt_layer_norm(x, a_2, b_2, eps, residual=None):
    """onmt's LayerNorm of the rows of x [rows, d] with z = x + residual (residual: the same shape, or None):
    (z - mean) / (std + eps) * a_2 + b_2 with the unbiased std; z itself when d = 1.  Differentiable in x, a_2, b_2 and
    residual."""
    N.require_cuda()
    N.check_float_cuda(x, "x", 2)
    N.check_float_cuda(a_2, "a_2", 1)
    N.check_float_cuda(b_2, "b_2", 1)
    d = x.shape[1]
    if a_2.shape[0] != d or b_2.shape[0] != d:
        raise ValueError(f"a_2 {tuple(a_2.shape)} and b_2 {tuple(b_2.shape)} must have the width {d} of x")
    if residual is not None:
        N.check_float_cuda(residual, "residual", 2)
        if residual.shape != x.shape:
            raise ValueError(f"residual {tuple(residual.shape)} must have the shape of x {tuple(x.shape)}")
        residual = residual.contiguous()
    if any(t.device != x.device for t in (a_2, b_2) + (() if residual is None else (residual,))):
        raise ValueError("x, a_2, b_2 and residual must be on the same device")
    eps = float(eps)
    if not math.isfinite(eps):
        raise ValueError("eps must be finite")
    return _LayerNorm.apply(x.contiguous(), a_2.contiguous(), b_2.contiguous(), eps, residual)


class LayerNorm(nn.Module):
    """Drop-in replacement of onmt.modules.UtilClass.LayerNorm: parameters a_2 (ones) and b_2 (zeros), eps outside
    the unbiased std, input [rows, d] returned unchanged when d = 1.  forward also takes an optional residual that is
    added first, in the same launch."""

    def __init__(self, d_hid, eps=1e-3):
        super().__init__()
        self.eps = eps
        self.a_2 = nn.Parameter(torch.ones(d_hid), requires_grad=True)
        self.b_2 = nn.Parameter(torch.zeros(d_hid), requires_grad=True)

    def forward(self, z, residual=None):
        if not isinstance(z, torch.Tensor) or z.dim() != 2:
            raise ValueError("LayerNorm takes [rows, d] (BottleLayerNorm takes [B, L, d] too)")
        return onmt_layer_norm(z, self.a_2, self.b_2, self.eps, residual)


class BottleLayerNorm(LayerNorm):
    """Drop-in replacement of onmt.modules.BottleLayerNorm: 2-D input as LayerNorm, 3-D [B, L, d] over its B*L rows."""

    def forward(self, z, residual=None):
        if not isinstance(z, torch.Tensor) or z.dim() not in (2, 3):
            raise ValueError("BottleLayerNorm takes [rows, d] or [B, L, d]")
        if z.dim() == 2:
            return super().forward(z, residual)
        B, L, d = z.shape
        r = None if residual is None else residual.reshape(B * L, d)
        return onmt_layer_norm(z.reshape(B * L, d), self.a_2, self.b_2, self.eps, r).view(B, L, d)


class MultiHeadedAttention(nn.Module):
    """Drop-in replacement of onmt.modules.MultiHeadedAttention: the same constructor, submodules (linear_keys,
    linear_values, linear_query without bias, layer_norm with a_2 / b_2, dropout, res_dropout), so the same state_dict
    keys, and the same forward(key, value, query, mask=None) -> (ret, top_attn).  The Linears are called as modules, so
    codec.attach_packed_ may replace them by PackedLinear; res_dropout stays torch; the attention core and the residual
    add with the layer norm are native.  In training mode with p > 0 the keep mask of the attention dropout is drawn
    with torch on the weights' device.

    Refused: model_dim not divisible by head_count or by 8 (the reference's assertions): ValueError; inputs that are not
    float32 CUDA tensors: ValueError."""

    def __init__(self, head_count, model_dim, p=0.1):
        if model_dim % head_count != 0:
            raise ValueError(f"model_dim {model_dim} must be divisible by head_count {head_count}")
        if model_dim % 8 != 0:
            raise ValueError(f"model_dim {model_dim} must be divisible by 8")
        super().__init__()
        self.dim_per_head = model_dim // head_count
        self.model_dim = model_dim
        self.head_count = head_count
        self.linear_keys = nn.Linear(model_dim, head_count * self.dim_per_head, bias=False)
        self.linear_values = nn.Linear(model_dim, head_count * self.dim_per_head, bias=False)
        self.linear_query = nn.Linear(model_dim, head_count * self.dim_per_head, bias=False)
        self.layer_norm = BottleLayerNorm(model_dim)
        self.dropout = nn.Dropout(p)
        self.res_dropout = nn.Dropout(p)

    def forward(self, key, value, query, mask=None):
        for t, what in ((key, "key"), (value, "value"), (query, "query")):
            N.check_float_cuda(t, what, 3)
        B, Lk, d = key.shape
        if value.shape != key.shape or query.shape[0] != B or query.shape[2] != d or d != self.model_dim:
            raise ValueError(f"key {tuple(key.shape)}, value {tuple(value.shape)} and query {tuple(query.shape)} do not "
                             f"match model_dim {self.model_dim}")
        Lq = query.shape[1]
        kp, vp, qp = self.linear_keys(key), self.linear_values(value), self.linear_query(query)
        p = self.dropout.p
        keep = None
        if self.training and p > 0:
            keep = torch.rand(B * self.head_count, Lq, Lk, device=self.linear_query.weight.device) >= p
        out, top = mha_core(qp, kp, vp, self.head_count, mask, keep, p)
        ret = self.layer_norm(self.res_dropout(out), residual=query)
        return ret, top
