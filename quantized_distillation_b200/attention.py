"""onmt's global attention (onmt/modules/GlobalAttention.py), "dot" and "general", with its core in fused kernels
(qd_attn_fwd / qd_attn_bwd).

Every decoder step of the reference's NMT models calls GlobalAttention: linear_in, bmm, softmax, bmm, cat, linear_out
and tanh forward, and about as many kernels backward, each moving a few MB.  Here the two Linears still run as modules
(cuBLAS, or PackedLinear after codec.attach_packed_); the score, the softmax over the source, the weighted context and
the concatenation are one launch forward and two backward.  The context is read in the layout the decoders pass it,
the transpose of onmt's [S, N, H] memory bank, without a copy.

    attention_core(q, input, context, kind) -> (align [T, N, S], concat [T, N, 2H])
    GlobalAttention(dim, coverage=False, attn_type="dot")

There is no CPU implementation: CPU tensors raise ValueError.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _native as N

ATTN_DOT, ATTN_GENERAL = 0, 1       # QD_ATTN_DOT, QD_ATTN_GENERAL


def _usable_context(context):
    """context itself when the kernels can read it in place (unit stride along H, (n, s) rows that do not overlap),
    else a contiguous copy."""
    Nb, S, H = context.shape
    sN, sS, sH = context.stride()
    (lo, clo), (hi, chi) = sorted([(sS, S), (sN, Nb)])
    if sH == 1 and (clo <= 1 or lo >= H) and (chi <= 1 or hi >= (clo - 1) * lo + H):
        return context
    return context.contiguous()


class _AttentionCore(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, input, context, kind):
        Nb, T, H = input.shape
        S = context.shape[1]
        dev = input.device
        align = torch.empty(T, Nb, S, dtype=torch.float32, device=dev)
        concat = torch.empty(T, Nb, 2 * H, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            N.check(N.lib().qd_attn_fwd(kind, None if kind == ATTN_DOT else N.ptr(q), N.ptr(input), N.ptr(context),
                                        context.stride(0), context.stride(1), Nb, T, S, H, N.ptr(align), N.ptr(concat),
                                        N.stream_ptr(dev)))
        ctx.save_for_backward(q, context, align)
        return align, concat

    @staticmethod
    def backward(ctx, grad_align, grad_concat):
        q, context, align = ctx.saved_tensors
        Nb, T, H = q.shape
        S = context.shape[1]
        dev = q.device
        if grad_concat is None:
            grad_concat = torch.zeros(T, Nb, 2 * H, dtype=torch.float32, device=dev)
        grad_concat = grad_concat.contiguous()
        grad_align = None if grad_align is None else grad_align.contiguous()
        grad_q = torch.empty_like(q)
        grad_context = torch.empty_strided(context.shape, context.stride(), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            ws = torch.empty(int(N.lib().qd_attn_workspace_bytes(Nb * T, S)), dtype=torch.uint8, device=dev)
            N.check(N.lib().qd_attn_bwd(N.ptr(grad_concat), N.ptr(grad_align), N.ptr(align), N.ptr(q), N.ptr(context),
                                        context.stride(0), context.stride(1), Nb, T, S, H, N.ptr(grad_q),
                                        N.ptr(grad_context), N.ptr(ws) if ws.numel() else None, ws.numel(),
                                        N.stream_ptr(dev)))
        grad_input = grad_concat[:, :, H:].transpose(0, 1)
        return grad_q, grad_input, grad_context, None


def attention_core(q, input, context, kind):
    """(align, concat) of the attention core for queries q and decoder outputs input [N, T, H] (q is input for dot)
    against context [N, S, H] (any strides; the transposed view of a contiguous [S, N, H] is read in place).
    align: [T, N, S], the softmax over the source; concat: [T, N, 2H] = [sum_s align_s context_s | input].
    Differentiable in q, input and context.  The backward saves align, q and the context."""
    N.require_cuda()
    if kind not in (ATTN_DOT, ATTN_GENERAL):
        raise ValueError("kind must be ATTN_DOT or ATTN_GENERAL")
    N.check_float_cuda(input, "input", 3)
    N.check_float_cuda(context, "context", 3)
    N.check_float_cuda(q, "q", 3)
    if kind == ATTN_DOT and q is not input:
        raise ValueError("dot attention takes the input itself as its query")
    if q.shape != input.shape or context.shape[0] != input.shape[0] or context.shape[2] != input.shape[2]:
        raise ValueError(f"shapes do not match: q {tuple(q.shape)}, input {tuple(input.shape)}, context {tuple(context.shape)}")
    if q.device != input.device or context.device != input.device:
        raise ValueError("q, input and context must be on the same device")
    input = input.contiguous()
    q = input if kind == ATTN_DOT else q.contiguous()
    return _AttentionCore.apply(q, input, _usable_context(context), kind)


class GlobalAttention(nn.Module):
    """Drop-in replacement of onmt.modules.GlobalAttention for attn_type "dot" and "general": the same constructor,
    submodules (so the same state_dict keys: linear_in for "general", linear_out, linear_cover with coverage=True) and
    outputs, with the core in fused kernels.  linear_in and linear_out are called as modules, so codec.attach_packed_
    may replace them by PackedLinear.

    Refused, none of which the reference's NMT models use:
      - attn_type "mlp" (Bahdanau): NotImplementedError; any other unknown type: ValueError;
      - a coverage argument to forward: NotImplementedError (onmt's decoders pass none);
      - applyMask with a mask: NotImplementedError (nothing in the reference calls it);
      - inputs that are not float32 CUDA tensors: ValueError (there is no CPU implementation).
    """

    def __init__(self, dim, coverage=False, attn_type="dot"):
        super().__init__()
        if attn_type == "mlp":
            raise NotImplementedError("mlp (Bahdanau) attention is not implemented; use 'dot' or 'general'")
        if attn_type not in ("dot", "general"):
            raise ValueError("Please select a valid attention type.")
        self.dim = dim
        self.attn_type = attn_type
        if attn_type == "general":
            self.linear_in = nn.Linear(dim, dim, bias=False)
        self.linear_out = nn.Linear(dim * 2, dim, bias=False)
        self.mask = None
        if coverage:
            self.linear_cover = nn.Linear(1, dim, bias=False)

    def applyMask(self, mask):
        if mask is not None:
            raise NotImplementedError("masked attention is not implemented")
        self.mask = None

    def forward(self, input, context, coverage=None):
        """input: [N, H] (one step) or [N, T, H]; context: [N, S, H].  Returns (attn_h, align_vectors): [N, H] and
        [N, S] for one step, else contiguous [T, N, H] and [T, N, S], as the reference."""
        if coverage is not None:
            raise NotImplementedError("coverage attention is not implemented")
        N.check_float_cuda(context, "context", 3)
        if not isinstance(input, torch.Tensor) or input.dim() not in (2, 3):
            raise ValueError("input must be [N, H] or [N, T, H]")
        one_step = input.dim() == 2
        if one_step:
            input = input.unsqueeze(1)
        N.check_float_cuda(input, "input", 3)
        if input.shape[0] != context.shape[0] or input.shape[2] != self.dim or context.shape[2] != self.dim:
            raise ValueError(f"input {tuple(input.shape)} and context {tuple(context.shape)} do not match dim {self.dim}")
        input = input.contiguous()
        if self.attn_type == "general":
            align, concat = attention_core(self.linear_in(input), input, context, ATTN_GENERAL)
        else:
            align, concat = attention_core(input, input, context, ATTN_DOT)
        attn_h = torch.tanh(self.linear_out(concat))
        if one_step:
            return attn_h.squeeze(0), align.squeeze(0)
        return attn_h, align
