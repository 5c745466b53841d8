"""onmt's global attention (onmt/modules/GlobalAttention.py), "dot" and "general", with its core in fused kernels
(qd_attn_fwd / qd_attn_bwd).

Every decoder step of the reference's NMT models calls GlobalAttention: linear_in, bmm, softmax, bmm, cat, linear_out
and tanh forward, and about as many kernels backward, each moving a few MB.  Here the two Linears still run as modules
(cuBLAS, or PackedLinear after codec.attach_packed_); the score, the softmax over the source, the weighted context and
the concatenation are one launch forward and two backward.  The context is read in the layout the decoders pass it,
the transpose of onmt's [S, N, H] memory bank, without a copy.

    attention_core(q, input, context, kind) -> (align [T, N, S], concat [T, N, 2H])
    GlobalAttention(dim, coverage=False, attn_type="dot")

"mlp" (Bahdanau) attention has its own drop-in, since its submodules differ: the reference expands linear_query(h_t)
and linear_context(h_s) to [N, T, S, H], adds them, takes tanh and reduces with v, and autograd keeps that tensor for
the backward.  Here the score, softmax, weighted context and concatenation are one launch forward (qd_attn_mlp_fwd)
and three backward (qd_attn_mlp_bwd), which recompute tanh instead of storing it; only [T, N, S] is kept.

    mlp_attention_core(wq, uh, v, input, context) -> (align [T, N, S], concat [T, N, 2H])
    MLPGlobalAttention(dim, coverage=False, attn_type="mlp")
    make_global_attention(dim, coverage=False, attn_type="dot"): the module for any of the three types

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


class _MLPAttentionCore(torch.autograd.Function):
    @staticmethod
    def forward(ctx, wq, uh, v, input, context):
        Nb, T, H = input.shape
        S = context.shape[1]
        dev = input.device
        align = torch.empty(T, Nb, S, dtype=torch.float32, device=dev)
        concat = torch.empty(T, Nb, 2 * H, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            N.check(N.lib().qd_attn_mlp_fwd(N.ptr(wq), N.ptr(uh), uh.stride(0), uh.stride(1), N.ptr(v), N.ptr(input),
                                            N.ptr(context), context.stride(0), context.stride(1), Nb, T, S, H,
                                            N.ptr(align), N.ptr(concat), N.stream_ptr(dev)))
        ctx.save_for_backward(wq, uh, v, context, align)
        return align, concat

    @staticmethod
    def backward(ctx, grad_align, grad_concat):
        wq, uh, v, context, align = ctx.saved_tensors
        Nb, T, H = wq.shape
        S = context.shape[1]
        dev = wq.device
        if grad_concat is None:
            grad_concat = torch.zeros(T, Nb, 2 * H, dtype=torch.float32, device=dev)
        grad_concat = grad_concat.contiguous()
        grad_align = None if grad_align is None else grad_align.contiguous()
        grad_input = grad_concat[:, :, H:].transpose(0, 1)
        if Nb * T == 0:                        # no rows: the kernels do nothing, every gradient is zero
            return (torch.zeros_like(wq), torch.zeros_like(uh), torch.zeros_like(v), grad_input,
                    torch.zeros_like(context))
        grad_wq = torch.empty_like(wq)
        grad_uh = torch.empty_strided(uh.shape, uh.stride(), dtype=torch.float32, device=dev)
        grad_v = torch.empty_like(v)
        grad_context = torch.empty_strided(context.shape, context.stride(), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            ws = torch.empty(int(N.lib().qd_attn_mlp_workspace_bytes(Nb, T, S, H)), dtype=torch.uint8, device=dev)
            N.check(N.lib().qd_attn_mlp_bwd(N.ptr(grad_concat), N.ptr(grad_align), N.ptr(align), N.ptr(wq), N.ptr(uh),
                                            uh.stride(0), uh.stride(1), N.ptr(v), N.ptr(context), context.stride(0),
                                            context.stride(1), Nb, T, S, H, N.ptr(grad_wq), N.ptr(grad_uh),
                                            N.ptr(grad_v), N.ptr(grad_context), N.ptr(ws), ws.numel(),
                                            N.stream_ptr(dev)))
        return grad_wq, grad_uh, grad_v, grad_input, grad_context


def mlp_attention_core(wq, uh, v, input, context):
    """(align, concat) of the "mlp" attention core: wq = linear_query(input) and input [N, T, H], uh =
    linear_context(context) and context [N, S, H] (any strides; the transposed view of a contiguous [S, N, H] is read
    in place), v the H weights of onmt's v ([H] or [1, H]).  score[n, t, s] = sum_h v_h tanh(wq[n, t] + uh[n, s])[h];
    align: [T, N, S], the softmax over the source; concat: [T, N, 2H] = [sum_s align_s context_s | input].
    Differentiable in all five.  The backward saves wq, uh, v, the context and align, and recomputes tanh."""
    N.require_cuda()
    for t, what in ((wq, "wq"), (uh, "uh"), (input, "input"), (context, "context")):
        N.check_float_cuda(t, what, 3)
    N.check_float_cuda(v, "v")
    Nb, T, H = input.shape
    if (wq.shape != input.shape or context.shape[0] != Nb or context.shape[2] != H or uh.shape != context.shape
            or v.numel() != H or v.dim() not in (1, 2)):
        raise ValueError(f"shapes do not match: wq {tuple(wq.shape)}, uh {tuple(uh.shape)}, v {tuple(v.shape)}, "
                         f"input {tuple(input.shape)}, context {tuple(context.shape)}")
    if any(t.device != input.device for t in (wq, uh, v, context)):
        raise ValueError("wq, uh, v, input and context must be on the same device")
    return _MLPAttentionCore.apply(wq.contiguous(), _usable_context(uh), v.contiguous().view(H), input.contiguous(),
                                   _usable_context(context))


class MLPGlobalAttention(nn.Module):
    """Drop-in replacement of onmt.modules.GlobalAttention for attn_type "mlp" (Bahdanau): the same constructor,
    submodules (so the same state_dict keys: linear_context, linear_query with its bias, v, linear_out with its bias,
    linear_cover with coverage=True) and outputs, with the core in fused kernels.  linear_query, linear_context and
    linear_out are called as modules and v is read as a weight, so codec.attach_packed_ may replace any of the four by
    PackedLinear.  linear_context runs on the memory bank in the layout the decoders pass it (the transpose of
    [S, N, H]), so the reference's per-call copy of the bank is gone.

    Refused, as GlobalAttention refuses them: a coverage argument to forward and applyMask with a mask
    (NotImplementedError), inputs that are not float32 CUDA tensors and an attn_type other than "mlp" (ValueError).
    """

    def __init__(self, dim, coverage=False, attn_type="mlp"):
        super().__init__()
        if attn_type != "mlp":
            raise ValueError("MLPGlobalAttention is the 'mlp' attention type; use GlobalAttention for 'dot' and 'general'")
        self.dim = dim
        self.attn_type = attn_type
        self.linear_context = nn.Linear(dim, dim, bias=False)
        self.linear_query = nn.Linear(dim, dim, bias=True)
        self.v = nn.Linear(dim, 1, bias=False)
        self.linear_out = nn.Linear(dim * 2, dim, bias=True)
        self.mask = None
        if coverage:
            self.linear_cover = nn.Linear(1, dim, bias=False)

    def applyMask(self, mask):
        if mask is not None:
            raise NotImplementedError("masked attention is not implemented")
        self.mask = None

    def _v_weight(self):
        v = self.v
        return v.decoded_weight() if hasattr(v, "decoded_weight") else v.weight

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
        bank = context.transpose(0, 1)
        if bank.is_contiguous() and not context.is_contiguous():
            uh = self.linear_context(bank).transpose(0, 1)          # the decoders' [S, N, H] bank, as it lies
        else:
            uh = self.linear_context(context)
        align, concat = mlp_attention_core(self.linear_query(input), uh, self._v_weight(), input, context)
        attn_h = self.linear_out(concat)
        if one_step:
            return attn_h.squeeze(0), align.squeeze(0)
        return attn_h, align


def make_global_attention(dim, coverage=False, attn_type="dot"):
    """The drop-in for onmt.modules.GlobalAttention(dim, coverage, attn_type) of any type: GlobalAttention for "dot"
    and "general", MLPGlobalAttention for "mlp".  Bind onmt.modules.GlobalAttention to this when a model may use any of
    the three."""
    if attn_type == "mlp":
        return MLPGlobalAttention(dim, coverage=coverage, attn_type=attn_type)
    return GlobalAttention(dim, coverage=coverage, attn_type=attn_type)
