"""NumPy restatement of onmt's beam search (onmt/Beam.py, and the batch loop of Translator.translateBatch,
onmt/Translator.py:90-193), the checker of qd_beam_step, BatchBeam and beam_search.

Every sum is a float32 add, as the reference's `wordLk + scores` on float32 tensors.  The top K of a sentence's keys are
ordered by key descending with ties to the lower flat index k*V + j, NaN above every number (as torch.topk) and -0 equal
to +0; the reference leaves the order of exact ties unspecified, this is the rule the kernel follows.
"""
from __future__ import annotations

import numpy as np

EOS_ROW_KEY = np.float32(-1e20)      # Beam.py:75, beamLk[i] = -1e20 on a float32 tensor


def key_order(keys):
    """int64 image of float32 keys that orders them as the selection does: NaN above +inf, -0 equal to +0."""
    k = np.asarray(keys, np.float32)
    k = np.where(k == 0, np.float32(0), k)
    u = k.view(np.uint32).astype(np.int64)
    o = np.where(u & 0x80000000, (~u) & 0xFFFFFFFF, u | 0x80000000)
    return np.where(np.isnan(k), 0xFFFFFFFF, o)


def top_k(flat_keys, K):
    """Indices of the K best of a 1-D float32 key array: keys descending, ties to the lower index."""
    o = key_order(flat_keys)
    kth = np.partition(o, o.size - K)[o.size - K]
    cand = np.nonzero(o >= kth)[0]                       # every index tied with the K-th too, in index order
    return cand[np.argsort(-o[cand], kind="stable")][:K]


def keys(word_lk, scores, last_tokens, eos, first):
    """beamLk of Beam.advance (Beam.py:68-77) for one sentence: word_lk [K, V] float32 log-probabilities, scores and
    last_tokens [K].  The first step keeps row 0 alone, without its score; later steps add the scores and give every
    column of a row that ended on EOS the key -1e20."""
    if first:
        return np.asarray(word_lk[0], np.float32).copy()
    with np.errstate(invalid="ignore", over="ignore"):
        lk = (np.asarray(word_lk, np.float32) + np.asarray(scores, np.float32)[:, None]).astype(np.float32)
    lk[np.asarray(last_tokens) == eos] = EOS_ROW_KEY
    return lk


def log_probs(logits, lse):
    """lp = fl(x - lse) per row, the kernel's normalize=1 log-probabilities for row lse values given in float32."""
    with np.errstate(invalid="ignore", over="ignore"):            # an all -inf row: -inf - (-inf) is NaN, as on the GPU
        return (np.asarray(logits, np.float32) - np.asarray(lse, np.float32)[:, None]).astype(np.float32)


def beam_step(lp, B, K, eos, first, scores, last_tokens, n_finished, eos_top):
    """qd_beam_step on rows r = k*B + b of lp [K*B, V] (log-probabilities).  Returns (scores, origin, flat_origin,
    tokens, n_finished, eos_top) as new arrays."""
    lp = np.asarray(lp, np.float32)
    V = lp.shape[1]
    sc, orig, flat, tok = (np.zeros(K * B, np.float32), np.zeros(K * B, np.int64), np.zeros(K * B, np.int64),
                           np.zeros(K * B, np.int64))
    nf, et = np.array(n_finished, np.int32), np.array(eos_top, np.uint8)
    for b in range(B):
        rows = np.arange(K) * B + b
        lk = keys(lp[rows], np.asarray(scores)[rows], np.asarray(last_tokens)[rows], eos, first).reshape(-1)
        best = top_k(lk, K)
        sc[rows], orig[rows], tok[rows] = lk[best], best // V, best % V
        flat[rows] = orig[rows] * B + b
        nf[b] += int(np.sum(tok[rows] == eos))
        if tok[rows[0]] == eos:
            et[b] = 1
    return sc, orig, flat, tok, nf, et


class Beam:
    """onmt.Beam on NumPy arrays, without the global scorer (the reference ships it commented out)."""

    def __init__(self, size, n_best, bos, eos, pad):
        self.size, self.n_best, self._eos = size, n_best, eos
        self.scores = np.zeros(size, np.float32)
        self.prevKs = []
        self.nextYs = [np.full(size, pad, np.int64)]
        self.nextYs[0][0] = bos
        self.eosTop = False
        self.attn = []
        self.finished = []

    def advance(self, word_lk, attn_out):
        V = word_lk.shape[1]
        lk = keys(word_lk, self.scores, self.nextYs[-1], self._eos, not self.prevKs).reshape(-1)
        best = top_k(lk, self.size)
        self.scores = lk[best]
        prev = best // V
        self.prevKs.append(prev)
        self.nextYs.append(best - prev * V)
        self.attn.append(np.asarray(attn_out)[prev])
        for i in range(self.size):
            if self.nextYs[-1][i] == self._eos:
                self.finished.append((self.scores[i], len(self.nextYs) - 1, i))
        if self.nextYs[-1][0] == self._eos:
            self.eosTop = True

    def done(self):
        return self.eosTop and len(self.finished) >= self.n_best

    def sortFinished(self, minimum=None):
        if minimum is not None:
            i = 0
            # the reference never advances i: short of `minimum` finished, it appends the top beam again and again
            while len(self.finished) < minimum:
                self.finished.append((self.scores[i], len(self.nextYs) - 1, i))
        self.finished.sort(key=lambda a: -a[0])
        return [float(s) for s, _, _ in self.finished], [(t, k) for _, t, k in self.finished]

    def getHyp(self, timestep, k):
        hyp, attn = [], []
        for j in range(len(self.prevKs[:timestep]) - 1, -1, -1):
            hyp.append(int(self.nextYs[j + 1][k]))
            attn.append(self.attn[j][k])
            k = self.prevKs[j][k]
        return hyp[::-1], np.stack(attn[::-1])


def translate_batch(step, B, K, n_best, max_len, bos, eos, pad, beam_update=None):
    """The loop of Translator.translateBatch over per-sentence Beams.  step(inp) runs the decoder and generator on the
    tokens inp [K*B] (row k*B + b) and returns (lp [K*B, V] float32, attn [K*B, S]); beam_update(b, origins) is the
    decoder state's beam_update after sentence b advances.  Returns (hyps, scores, attn, beams): per sentence its n_best
    hypotheses (lists of int), the scores of all its finished entries and the hypotheses' attention [len, S]."""
    beams = [Beam(K, n_best, bos, eos, pad) for _ in range(B)]
    for _ in range(max_len):
        if all(b.done() for b in beams):
            break
        inp = np.stack([b.nextYs[-1] for b in beams]).T.reshape(-1) if B else np.zeros(0, np.int64)
        lp, attn = step(inp)
        lp = np.asarray(lp, np.float32).reshape(K, B, -1)
        attn = np.asarray(attn).reshape(K, B, -1)
        for j, b in enumerate(beams):
            b.advance(lp[:, j], attn[:, j])
            if beam_update is not None:
                beam_update(j, b.prevKs[-1])
    hyps, scores, attns = [], [], []
    for b in beams:
        sc, ks = b.sortFinished(minimum=n_best)
        hs, at = zip(*[b.getHyp(t, k) for t, k in ks[:n_best]])
        hyps.append(list(hs))
        scores.append(sc)
        attns.append(list(at))
    return hyps, scores, attns, beams
