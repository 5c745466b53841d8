"""The loss of the NMT loop over the target vocabulary, computed by fused kernels (qd_nmt_loss_fwd / qd_nmt_loss_bwd).

The reference (onmt/Loss.py:97-120) runs the generator, Linear -> LogSoftmax, takes the summed NLL at the targets with
weight 0 at the padding index and, when distilling, adds 0.7 times the KL divergence to the teacher's softmax.  That
chain materialises several [rows, V] tensors per op, forward and backward, which is why onmt computes it in shards of 32
time steps.  Here the generator's Linear still runs in torch; everything after it is one pass over the logits forward
(the student's and the teacher's rows read once) and one backward (both read again, the gradient written once).

    nmt_loss(logits, target, padding_idx, teacher_logits=None, weight_teacher_loss=0.7) -> (loss, stats)
    NMTLossCompute(generator, tgt_vocab, use_distillation_loss=False, teacher_generator=None)

There is no CPU implementation: without a CUDA device the calls raise RuntimeError.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _native as N

PAD_WORD = "<blank>"            # onmt.IO.PAD_WORD
WEIGHT_TEACHER_LOSS = 0.7       # onmt/Loss.py:109


def _check(logits, target, teacher_logits, padding_idx, w):
    N.require_cuda()
    if not isinstance(logits, torch.Tensor) or not logits.is_cuda or logits.dtype != torch.float32 or logits.dim() != 2:
        raise ValueError("logits must be a 2-D float32 CUDA tensor [rows, V]")
    R, V = logits.shape
    if V < 1:
        raise ValueError("the vocabulary must have at least one entry")
    if not isinstance(target, torch.Tensor) or target.dtype != torch.int64 or target.dim() != 1 or target.numel() != R:
        raise ValueError(f"target must be an int64 tensor of {R} entries, one per row of logits")
    if target.device != logits.device:
        raise ValueError("target and logits must be on the same device")
    if teacher_logits is not None:
        if (not isinstance(teacher_logits, torch.Tensor) or teacher_logits.dtype != torch.float32
                or teacher_logits.shape != logits.shape or teacher_logits.device != logits.device):
            raise ValueError("teacher_logits must be a float32 tensor of the logits' shape and device")
    if not (isinstance(padding_idx, int) and -1 <= padding_idx < V):
        raise ValueError(f"padding_idx must be -1 (none) or in [0, {V})")
    if not (0.0 <= float(w) <= 1.0):
        raise ValueError("weight_teacher_loss must be in [0, 1]")


class _NMTLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, teacher_logits, padding_idx, w):
        R, V = logits.shape
        dev = logits.device
        logits, target = logits.contiguous(), target.contiguous()
        teacher_logits = None if teacher_logits is None else teacher_logits.detach().contiguous()
        row_lse = torch.empty(R, 2, dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        stats = torch.empty(3, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            ws = torch.empty(int(N.lib().qd_nmt_loss_workspace_bytes(R)), dtype=torch.uint8, device=dev)
            N.check(N.lib().qd_nmt_loss_fwd(N.ptr(logits), N.ptr(teacher_logits), N.ptr(target), R, V, padding_idx, w,
                                            N.ptr(row_lse), N.ptr(loss), N.ptr(stats), N.ptr(ws) if ws.numel() else None,
                                            ws.numel(), N.stream_ptr(dev)))
        ctx.save_for_backward(logits, teacher_logits, target, row_lse)
        ctx.padding_idx, ctx.w = padding_idx, w
        ctx.mark_non_differentiable(stats)
        return loss, stats

    @staticmethod
    def backward(ctx, grad_loss, _grad_stats):
        logits, teacher_logits, target, row_lse = ctx.saved_tensors
        R, V = logits.shape
        dev = logits.device
        g = grad_loss.to(device=dev, dtype=torch.float32).contiguous()
        grad = torch.empty_like(logits)
        with torch.cuda.device(dev):
            N.check(N.lib().qd_nmt_loss_bwd(N.ptr(logits), N.ptr(teacher_logits), N.ptr(target), N.ptr(row_lse), N.ptr(g), R, V,
                                            ctx.padding_idx, ctx.w, N.ptr(grad), N.stream_ptr(dev)))
        return grad, None, None, None, None


def nmt_loss(logits, target, padding_idx, teacher_logits=None, weight_teacher_loss=WEIGHT_TEACHER_LOSS):
    """(loss, stats) of the NMT loss over rows of generator logits (before the LogSoftmax).

    loss: float32 0-d tensor, the sum over non-padding rows of NLL(log_softmax(logits), target), or with teacher_logits of
    (1-w) NLL + w KL(softmax(teacher_logits) || softmax(logits)) -- the reference's size_average=False.  Differentiable
    in logits only: the teacher gets no gradient, as the reference detaches it.  stats: int64 CUDA tensor
    [n_words, n_correct, n_invalid]; a target outside [0, V) that is not padding_idx makes the loss NaN and is counted in
    n_invalid.  padding_idx -1 means no padding.  Everything stays on the device: no synchronisation."""
    _check(logits, target, teacher_logits, padding_idx, weight_teacher_loss)
    return _NMTLoss.apply(logits, target, teacher_logits, padding_idx, float(weight_teacher_loss))


class Statistics:
    """What onmt.Statistics.update reads from a loss call: the summed loss (before any division), the words and the
    correctly predicted words."""

    def __init__(self, loss=0.0, n_words=0, n_correct=0):
        self.loss, self.n_words, self.n_correct = loss, n_words, n_correct

    def update(self, stat):
        self.loss += stat.loss
        self.n_words += stat.n_words
        self.n_correct += stat.n_correct


def _generator_linear(gen, what):
    if not (isinstance(gen, nn.Sequential) and len(gen) == 2 and isinstance(gen[0], nn.Linear)
            and isinstance(gen[1], nn.LogSoftmax)):
        raise ValueError(f"the {what} must be Sequential(Linear, LogSoftmax); other generators (CopyGenerator) are not supported")
    return gen[0]


class NMTLossCompute(nn.Module):
    """Drop-in replacement of onmt.Loss.NMTLossCompute (onmt/Loss.py:22-55, 79-120) whose loss is nmt_loss: the
    generator's Linear runs in torch, the LogSoftmax, NLL, KL and their gradients in the fused kernels."""

    def __init__(self, generator, tgt_vocab, use_distillation_loss=False, teacher_generator=None):
        if use_distillation_loss is True and teacher_generator is None:
            raise ValueError("to use distillation loss you have to pass the teacher generator")
        super().__init__()
        _generator_linear(generator, "generator")
        if teacher_generator is not None:
            _generator_linear(teacher_generator, "teacher generator")
        self.generator = generator
        self.tgt_vocab = tgt_vocab
        self.padding_idx = tgt_vocab.stoi[PAD_WORD]
        self.copy_attn = False
        self.use_distillation_loss = use_distillation_loss
        self.teacher_generator = teacher_generator

    @staticmethod
    def bottle(v):
        return v.view(-1, v.size(2))

    def forward(self, batch, output, target, **kwargs):
        return self.compute_loss(batch, output, target, **kwargs)

    def compute_loss(self, batch, output, target, teacher_outputs=None, **kwargs):
        """(loss, stats) for the decoder output [T, B, H] and targets [T, B]; loss is the summed float32 0-d tensor.
        Reading stats synchronises once, as the reference's loss.data[0] does."""
        logits = self.generator[0](self.bottle(output))
        teacher_logits = None
        if self.use_distillation_loss:
            if teacher_outputs is None:
                raise ValueError("the distillation loss needs teacher_outputs")
            with torch.no_grad():
                teacher_logits = self.teacher_generator[0](self.bottle(teacher_outputs))
        loss, counts = nmt_loss(logits, target.reshape(-1), self.padding_idx, teacher_logits)
        host = torch.cat([loss.detach().double().view(1), counts.double()]).tolist()
        if host[3] > 0:
            raise ValueError(f"{int(host[3])} targets are outside the vocabulary [0, {logits.shape[1]})")
        return loss, Statistics(host[0], int(host[1]), int(host[2]))

    def sharded_compute_loss(self, batch, output, attns, cur_trunc, trunc_size, shard_size, teacher_outputs=None):
        """The reference's slicing (make_gen_state: targets cur_trunc+1 .. cur_trunc+trunc_size) and backward of
        loss / batch.batch_size, but over the whole range in one fused call: no logits of a shard are kept for a second
        pass, so there is nothing to gain from shards.  shard_size is accepted and ignored."""
        target = batch.tgt[cur_trunc + 1: cur_trunc + trunc_size]
        loss, stats = self.compute_loss(batch, output, target, teacher_outputs=teacher_outputs)
        loss.div(batch.batch_size).backward()
        return stats
