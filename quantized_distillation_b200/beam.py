"""Batched beam search for onmt-style translation models, one fused kernel per step (qd_beam_step).

The reference (onmt/Translator.py:90-193, onmt/Beam.py) keeps one Beam object per sentence: each step synchronises the
host 2K+1 times per sentence (EOS tests inside Python `if`s), runs one index_select + copy_ per sentence and decoder
state tensor, and one topk per sentence over K*V entries.  Here the B sentences' beams live on the device together:
one kernel call normalises the generator's logits, selects every sentence's K best and updates the finished counters,
one index_select per state tensor reorders the decoder, and done() is the loop's only device-to-host read per step.

    BatchBeam(batch, beam, n_best, bos, eos, pad, max_len, device)
    beam_search(model, src, src_lengths, beam_size=5, n_best=1, max_sent_length=100, *, bos, eos, pad, global_scorer=None)

There is no CPU implementation: without a CUDA device the calls raise RuntimeError.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _native as N


class BatchBeam:
    """The state of B onmt Beams (Beam.py:11-45) on the device, rows in onmt's beam-major order r = k*B + b.

    tokens[t] [max_len+1, K, B] are the nextYs (step 0: BOS for beam 0, PAD for the others), origins[t] and
    step_scores[t] [max_len, K, B] the prevKs and the scores after step t, attn[t] [max_len, K, B, S] the attention
    gathered by origin (Beam.attn).  Sentences keep advancing after they are done until the whole batch is done, as in
    translateBatch."""

    def __init__(self, batch, beam, n_best, bos, eos, pad, max_len, device):
        N.require_cuda()
        if not (isinstance(beam, int) and 1 <= beam <= N.BEAM_MAX):
            raise ValueError(f"beam must be an int in [1, {N.BEAM_MAX}]")
        if not (isinstance(batch, int) and batch >= 0):
            raise ValueError("batch must be an int >= 0")
        if not (isinstance(n_best, int) and n_best >= 1):
            raise ValueError("n_best must be an int >= 1")
        if not (isinstance(max_len, int) and max_len >= 1):
            raise ValueError("max_len must be an int >= 1")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise ValueError("BatchBeam lives on a CUDA device")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.B, self.K, self.n_best, self.eos, self.max_len, self.device = batch, beam, n_best, int(eos), max_len, dev
        K, B = beam, batch
        self.scores = torch.zeros(K * B, dtype=torch.float32, device=dev)
        self.tokens = torch.full((max_len + 1, K, B), pad, dtype=torch.int64, device=dev)
        self.tokens[0, 0] = bos
        self.origins = torch.zeros(max_len, K, B, dtype=torch.int64, device=dev)
        self.step_scores = torch.zeros(max_len, K, B, dtype=torch.float32, device=dev)
        self.flat_origin = torch.zeros(K * B, dtype=torch.int64, device=dev)
        self.n_finished = torch.zeros(B, dtype=torch.int32, device=dev)
        self.eos_top = torch.zeros(B, dtype=torch.uint8, device=dev)
        self.attn = None
        self.steps = 0
        with torch.cuda.device(dev):
            self._ws = torch.empty(max(int(N.lib().qd_beam_workspace_bytes(B, K)), 1), dtype=torch.uint8, device=dev)

    def current_tokens(self) -> torch.Tensor:
        """The tokens of the last step, [K*B] in row order: the decoder's next input (Beam.getCurrentState)."""
        return self.tokens[self.steps].view(-1)

    def advance(self, out: torch.Tensor, attn: torch.Tensor, normalized: bool) -> torch.Tensor:
        """Beam.advance for every sentence at once.  out: float32 [K*B, V] log-probabilities (normalized=True) or the
        generator Linear's logits (normalized=False: the kernel takes the log-softmax, with the NMT loss's lse).
        attn: [K*B, S], the decoder's attn["std"] of the step.  Returns flat_origin [K*B], the rows that reorder the
        decoder state: state.index_select(1, flat_origin)."""
        K, B = self.K, self.B
        if self.steps >= self.max_len:
            raise ValueError(f"the beam has already advanced max_len={self.max_len} steps")
        if (not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.dim() != 2 or out.shape[0] != K * B
                or out.device != self.device):
            raise ValueError(f"out must be a float32 tensor [{K * B}, V] on {self.device}")
        if not isinstance(attn, torch.Tensor) or attn.dim() != 2 or attn.shape[0] != K * B or attn.device != self.device:
            raise ValueError(f"attn must be a tensor [{K * B}, src_len] on {self.device}")
        if self.attn is None:
            self.attn = torch.zeros(self.max_len, K, B, attn.shape[1], dtype=attn.dtype, device=self.device)
        elif attn.shape[1] != self.attn.shape[3] or attn.dtype != self.attn.dtype:
            raise ValueError("attn must keep its src_len and dtype from step to step")
        out = out.contiguous()
        t = self.steps
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_beam_step(
                N.ptr(out), 0 if normalized else 1, B, K, out.shape[1], self.eos, int(t == 0), N.ptr(self.scores),
                N.ptr(self.tokens[t]), N.ptr(self.origins[t]), N.ptr(self.flat_origin), N.ptr(self.tokens[t + 1]),
                N.ptr(self.n_finished), N.ptr(self.eos_top), N.ptr(self._ws), self._ws.numel(), N.stream_ptr(self.device)))
        self.step_scores[t].view(-1).copy_(self.scores)
        torch.index_select(attn, 0, self.flat_origin, out=self.attn[t].view(K * B, -1))
        self.steps = t + 1
        return self.flat_origin

    def done(self) -> bool:
        """Beam.done for every sentence: EOS topped its beam and n_best entries finished.  One device-to-host read."""
        return bool(((self.eos_top != 0) & (self.n_finished >= self.n_best)).all())

    def finish(self):
        """(hyps, scores, attn) per sentence, what translateBatch returns without the gold scores: the n_best
        hypotheses as lists of int, the scores (floats) of every finished entry in sortFinished order, and each
        hypothesis's attention [len, src_len] (CPU tensors).  The histories are copied to the host once.

        sortFinished(minimum=n_best) is rebuilt exactly: finished entries in step order, then beam order, sorted by
        -score with Python's stable sort.  When fewer than n_best finished, the reference's loop (Beam.py:113-121)
        never advances its index, so it appends the top beam of the last step repeatedly; so does this."""
        T, K, B = self.steps, self.K, self.B
        tokens = self.tokens[:T + 1].cpu().tolist()
        origins = self.origins[:T].cpu().tolist()
        step_scores = self.step_scores[:T].cpu()
        attn = self.attn[:T].cpu() if T else None
        sc_list = step_scores.tolist()
        hyps, scores, attns = [], [], []
        for b in range(B):
            finished = [(sc_list[t - 1][i][b], t, i) for t in range(1, T + 1) for i in range(K) if tokens[t][i][b] == self.eos]
            while len(finished) < self.n_best:
                finished.append((sc_list[T - 1][0][b] if T else 0.0, T, 0))
            finished.sort(key=lambda a: -a[0])
            hs, ats = [], []
            for _, t, k in finished[:self.n_best]:
                hyp, rows = [], []
                for j in range(t - 1, -1, -1):
                    hyp.append(tokens[j + 1][k][b])
                    rows.append(attn[j, k, b])
                    k = origins[j][k][b]
                hs.append(hyp[::-1])
                ats.append(torch.stack(rows[::-1]) if rows else torch.zeros(0, 0))
            hyps.append(hs)
            scores.append([s for s, _, _ in finished])
            attns.append(ats)
        return hyps, scores, attns


def _generator_linear(gen):
    """The Linear of a Sequential(Linear or PackedLinear, LogSoftmax) generator."""
    from .codec import PackedLinear
    if not (isinstance(gen, nn.Sequential) and len(gen) == 2 and isinstance(gen[0], (nn.Linear, PackedLinear))
            and isinstance(gen[1], nn.LogSoftmax)):
        raise ValueError("the generator must be Sequential(Linear or PackedLinear, LogSoftmax); other generators "
                         "(CopyGenerator) are not supported")
    return gen[0]


@torch.no_grad()
def beam_search(model, src, src_lengths, beam_size=5, n_best=1, max_sent_length=100, *, bos, eos, pad, global_scorer=None):
    """Translator.translateBatch (onmt/Translator.py:90-193) without copy attention, global scorer or gold scores, for a
    model that follows onmt's protocol: model.encoder(src, lengths) -> (enc_states, context [S, B, H]);
    model.decoder.init_decoder_state(src, context, enc_states) -> a state with repeat_beam_size_times and `_all`
    tensors [a, K*B, d]; model.decoder(inp [1, K*B, 1], context, state) -> (out [1, K*B, H], state, attn with
    attn["std"] [1, K*B, S]); model.generator = Sequential(Linear or PackedLinear, LogSoftmax).  Each step runs the
    decoder, the generator's Linear and one qd_beam_step on the logits, then reorders every state tensor with one
    index_select.  Returns (hyps, scores, attn) per sentence, as BatchBeam.finish.  A global scorer (GNMT) is refused:
    the reference ships it commented out (Translator.py:112)."""
    if global_scorer is not None:
        raise ValueError("a global scorer is not supported")
    if getattr(model.decoder, "_copy", False) or getattr(model.decoder, "copy_attn", False):
        raise ValueError("copy attention (CopyGenerator) is not supported")
    linear = _generator_linear(model.generator)
    K = beam_size
    B = int(src.shape[1])
    enc_states, context = model.encoder(src, src_lengths)
    state = model.decoder.init_decoder_state(src, context, enc_states)
    context = context.repeat(1, K, 1)
    state.repeat_beam_size_times(K)
    beam = BatchBeam(B, K, n_best, bos, eos, pad, max_sent_length, context.device)
    for _ in range(max_sent_length):
        if beam.done():
            break
        inp = beam.current_tokens().view(1, -1, 1)
        dec_out, state, attn = model.decoder(inp, context, state)
        logits = linear(dec_out.squeeze(0))
        flat_origin = beam.advance(logits, attn["std"].squeeze(0), normalized=False)
        for e in state._all:
            e.copy_(e.index_select(1, flat_origin))
    return beam.finish()
