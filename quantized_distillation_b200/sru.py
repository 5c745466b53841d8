"""onmt's SRU layers (onmt/modules/SRU.py, "Training RNNs as Fast as CNNs") with the recurrence in native kernels
(qd_sru_fwd / qd_sru_bwd).

The reference runs the recurrence in four NVRTC kernels through cupy and pynvrtc, behind a legacy autograd Function
that current torch refuses to run.  Here the projection u = x.mm(weight) stays a GEMM; the recurrence over time is
one launch forward and two backward, bit-identical to the reference's kernels compiled without FMA contraction.

    sru_compute(u, x, bias, d, bidirectional, activation, init=None, mask_h=None) -> (h, last)
    SRUCell(n_in, n_out, dropout=0, rnn_dropout=0, bidirectional=False, use_tanh=1, use_relu=0)
    SRU(input_size, hidden_size, num_layers=2, dropout=0, rnn_dropout=0, bidirectional=False, use_tanh=1, use_relu=0)

Drop-in, before the model is built:  onmt.modules.SRU = quantized_distillation_b200.sru.SRU

There is no CPU implementation: CPU tensors raise ValueError.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _native as N

IDENTITY, TANH, RELU = 0, 1, 2      # QD_SRU_IDENTITY, QD_SRU_TANH, QD_SRU_RELU


class _SRUCompute(torch.autograd.Function):
    @staticmethod
    def forward(ctx, u, x, bias, init, mask_h, three_d, d, bidirectional, activation, length, batch, k):
        dir_ = 2 if bidirectional else 1
        size = (length, batch, d * dir_) if three_d else (batch, d * dir_)
        h = torch.empty(size, dtype=torch.float32, device=u.device)
        c = torch.empty(size, dtype=torch.float32, device=u.device)
        with torch.cuda.device(u.device):
            N.check(N.lib().qd_sru_fwd(N.ptr(u), N.ptr(x), N.ptr(bias), N.ptr(init), N.ptr(mask_h), length, batch, d, k,
                                       int(bidirectional), activation, N.ptr(h), N.ptr(c), N.stream_ptr(u.device)))
        ctx.save_for_backward(u, x, bias, init, mask_h, c)
        ctx.shape = (three_d, d, bidirectional, activation, length, batch, k)
        if not three_d:
            last = c
        elif bidirectional:
            last = torch.stack((c[-1, :, :d], c[0, :, d:]))        # directions x batch x d
        else:
            last = c[-1].clone()
        return h, last

    @staticmethod
    def backward(ctx, grad_h, grad_last):
        u, x, bias, init, mask_h, c = ctx.saved_tensors
        three_d, d, bidirectional, activation, length, batch, k = ctx.shape
        if three_d and bidirectional:
            grad_last = torch.cat((grad_last[0], grad_last[1]), 1)
        grad_h, grad_last = grad_h.contiguous(), grad_last.contiguous()
        dev = u.device
        grad_u = torch.empty_like(u)
        grad_x = torch.empty_like(x) if x is not None else None
        grad_bias = torch.empty_like(bias)
        grad_init = torch.empty_like(init) if init is not None else None
        with torch.cuda.device(dev):
            ws = torch.empty(int(N.lib().qd_sru_workspace_bytes(batch, d, int(bidirectional))), dtype=torch.uint8, device=dev)
            N.check(N.lib().qd_sru_bwd(N.ptr(u), N.ptr(x), N.ptr(bias), N.ptr(init), N.ptr(mask_h), N.ptr(c), N.ptr(grad_h),
                                       N.ptr(grad_last), length, batch, d, k, int(bidirectional), activation, N.ptr(grad_u),
                                       N.ptr(grad_x), N.ptr(grad_bias), N.ptr(grad_init), N.ptr(ws), ws.numel(),
                                       N.stream_ptr(dev)))
        return grad_u, grad_x, grad_bias, grad_init, None, None, None, None, None, None, None, None


def sru_compute(u, x, bias, d, bidirectional, activation, init=None, mask_h=None):
    """The SRU recurrence of one layer, as the reference's SRU_Compute(activation, d, bidirectional)(u, x, bias, init,
    mask_h).  x: the layer's input [len, batch, n_in] or [batch, n_in] (for k = 3 the highway term, read before
    rnn_dropout as the reference does); u = x_2d.mm(weight): [len*batch, dir*d*k], k = 3 or 4; bias [2*dir*d];
    init, mask_h: [batch, dir*d] or None (zeros, ones).  Returns h ([len, batch, dir*d] or [batch, dir*d]) and the
    reference's last cell state: c for 2-D input, stack((c[-1, :, :d], c[0, :, d:])) when bidirectional, else c[-1].
    Differentiable in u, x (k = 3), bias and init."""
    N.require_cuda()
    for t, what in ((u, "u"), (x, "x"), (bias, "bias")):
        N.check_float_cuda(t, what)
    if x.dim() not in (2, 3):
        raise ValueError("x must be [len, batch, n_in] or [batch, n_in]")
    if activation not in (IDENTITY, TANH, RELU):
        raise ValueError("activation must be 0 (identity), 1 (tanh) or 2 (relu)")
    dir_ = 2 if bidirectional else 1
    length = x.size(0) if x.dim() == 3 else 1
    batch = x.size(-2)
    if d < 1 or length < 1 or batch < 1:
        raise ValueError(f"d, len and batch must be >= 1 (d={d}, len={length}, batch={batch})")
    k = u.size(-1) // (d * dir_)
    if k not in (3, 4) or u.dim() != 2 or u.shape != (length * batch, dir_ * d * k):
        raise ValueError(f"u must be [len*batch, dir*d*k] with k 3 or 4: got {tuple(u.shape)} for len {length}, batch "
                         f"{batch}, d {d}, dir {dir_}")
    if k == 3 and x.size(-1) != dir_ * d:
        raise ValueError(f"with k = 3 the input width {x.size(-1)} must be dir*d = {dir_ * d}")
    if bias.shape != (2 * dir_ * d,):
        raise ValueError(f"bias must be [{2 * dir_ * d}], got {tuple(bias.shape)}")
    for t, what in ((init, "init"), (mask_h, "mask_h")):
        if t is not None:
            N.check_float_cuda(t, what)
            if t.numel() != batch * dir_ * d:
                raise ValueError(f"{what} must hold batch*dir*d = {batch * dir_ * d} values, got {tuple(t.shape)}")
    if any(t is not None and t.device != u.device for t in (x, bias, init, mask_h)):
        raise ValueError("u, x, bias, init and mask_h must be on the same device")
    return _SRUCompute.apply(u.contiguous(), x.contiguous() if k == 3 else None, bias.contiguous(),
                             None if init is None else init.contiguous().view(batch, dir_ * d),
                             None if mask_h is None else mask_h.contiguous().view(batch, dir_ * d),
                             x.dim() == 3, d, bool(bidirectional), activation, length, batch, k)


class SRUCell(nn.Module):
    """Drop-in replacement of the reference's SRUCell: the same arguments, parameters (weight [n_in, k*n_out*dir],
    k = 4 when n_in differs from the output width dir*n_out, else 3; bias [2*n_out*dir]), initialisation, dropout
    masks (drawn on the weight's device in the reference's order: the rnn_dropout mask on the input, then mask_h) and
    outputs.  input: [len, batch, n_in] or [batch, n_in]; c0: [batch, dir*n_out] or None (zeros)."""

    def __init__(self, n_in, n_out, dropout=0, rnn_dropout=0, bidirectional=False, use_tanh=1, use_relu=0):
        super().__init__()
        self.n_in = n_in
        self.n_out = n_out
        self.rnn_dropout = rnn_dropout
        self.dropout = dropout
        self.bidirectional = bidirectional
        self.activation_type = RELU if use_relu else (TANH if use_tanh else IDENTITY)
        out_size = n_out * 2 if bidirectional else n_out
        k = 4 if n_in != out_size else 3
        self.size_per_dir = n_out * k
        self.weight = nn.Parameter(torch.empty(n_in, self.size_per_dir * 2 if bidirectional else self.size_per_dir))
        self.bias = nn.Parameter(torch.empty(n_out * 4 if bidirectional else n_out * 2))
        self.init_weight()

    def init_weight(self):
        val_range = (3.0 / self.n_in) ** 0.5
        self.weight.data.uniform_(-val_range, val_range)
        self.bias.data.zero_()

    def set_bias(self, bias_val=0):
        n_out = self.n_out
        if self.bidirectional:
            self.bias.data[n_out * 2:].zero_().add_(bias_val)
        else:
            self.bias.data[n_out:].zero_().add_(bias_val)

    def forward(self, input, c0=None):
        if not isinstance(input, torch.Tensor) or input.dim() not in (2, 3):
            raise ValueError("input must be [len, batch, n_in] or [batch, n_in]")
        N.check_float_cuda(input, "input")
        N.check_float_cuda(self.weight, "weight")
        n_in, n_out = self.n_in, self.n_out
        batch = input.size(-2)
        if self.training and self.rnn_dropout > 0:
            mask = self.get_dropout_mask_((batch, n_in), self.rnn_dropout)
            x = input * mask.expand_as(input)
        else:
            x = input
        x_2d = x if x.dim() == 2 else x.contiguous().view(-1, n_in)
        u = x_2d.mm(self.weight)
        mask_h = None
        if self.training and self.dropout > 0:
            bidir = 2 if self.bidirectional else 1
            mask_h = self.get_dropout_mask_((batch, n_out * bidir), self.dropout)
        return sru_compute(u, input, self.bias, n_out, self.bidirectional, self.activation_type, init=c0, mask_h=mask_h)

    def get_dropout_mask_(self, size, p):
        return self.weight.data.new_empty(size).bernoulli_(1 - p).div_(1 - p)


class SRU(nn.Module):
    """Drop-in replacement of the reference's SRU (onmt.modules.SRU): the same arguments, layers (rnn_lst.{i}, so the
    same state_dict keys), dropout on every layer but the last, c0 handling and outputs.  input: [len, batch, n_in];
    c0: None (zeros), a tensor (depth, batch, dir*n_out), or the tuple RNNDecoderState wraps it in.  Returns the last
    layer's h and, with return_hidden, fh: the layers' last cell states stacked, (depth, batch, n_out), or
    concatenated when bidirectional, (depth*2, batch, n_out) in the order layer 0 forward, layer 0 backward, ... that
    onmt's _fix_enc_hidden expects.  The reference's check_sru_requirement has nothing left to check."""

    def __init__(self, input_size, hidden_size, num_layers=2, dropout=0, rnn_dropout=0, bidirectional=False,
                 use_tanh=1, use_relu=0):
        super().__init__()
        self.n_in = input_size
        self.n_out = hidden_size
        self.depth = num_layers
        self.dropout = dropout
        self.rnn_dropout = rnn_dropout
        self.rnn_lst = nn.ModuleList()
        self.bidirectional = bidirectional
        self.out_size = hidden_size * 2 if bidirectional else hidden_size
        for i in range(num_layers):
            self.rnn_lst.append(SRUCell(n_in=self.n_in if i == 0 else self.out_size, n_out=self.n_out,
                                        dropout=dropout if i + 1 != num_layers else 0, rnn_dropout=rnn_dropout,
                                        bidirectional=bidirectional, use_tanh=use_tanh, use_relu=use_relu))

    def set_bias(self, bias_val=0):
        for layer in self.rnn_lst:
            layer.set_bias(bias_val)

    def forward(self, input, c0=None, return_hidden=True):
        if not isinstance(input, torch.Tensor) or input.dim() != 3:
            raise ValueError("input must be [len, batch, n_in]")
        if c0 is None:
            c0 = [None] * self.depth
        else:
            if isinstance(c0, tuple):           # RNNDecoderState wraps hidden as a tuple
                c0 = c0[0]
            if not isinstance(c0, torch.Tensor) or c0.dim() != 3:
                raise ValueError("c0 must be (depth, batch, dir*hidden_size)")
            c0 = [h.squeeze(0) for h in c0.chunk(self.depth, 0)]
        prevx = input
        lstc = []
        for i, rnn in enumerate(self.rnn_lst):
            h, c = rnn(prevx, c0[i])
            prevx = h
            lstc.append(c)
        fh = torch.cat(lstc) if self.bidirectional else torch.stack(lstc)
        if return_hidden:
            return prevx, fh
        return prevx
