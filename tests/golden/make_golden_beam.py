"""Generates tests/golden/reference_beam.npz: the reference's own onmt/Beam.py, loaded unmodified by file path (with a
stub onmt.IO for its three special-word names), driven as Translator.translateBatch drives it (onmt/Translator.py:
136-193): a batch of Beams advanced on the same step's [K*B, V] log-probabilities until all are done or the step limit
is reached, then sortFinished(minimum=n_best) and getHyp.

On torch 0.3, `bestScoresId / numWords` (Beam.py:91) divided a LongTensor by an int in integers; current torch divides in
floats, so while the Beams run an integer tensor divided by an int is floor division.

The inputs are not stored: draw(seed, step, attempt, ...) regenerates them from integers with basic float32 operations
only, so every machine gets the same bits.  A draw whose top K+1 keys of some sentence hold an exact tie is redrawn
(the reference's order there is unspecified); a case that cannot avoid one (every beam of a sentence ended on EOS) is
dropped for the next seed.

Run in the build container only:  python tests/golden/make_golden_beam.py
"""
import importlib.util
import os
import sys
import types

import numpy as np

REF_BEAM = "/root/reference/onmt/Beam.py"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_beam.npz")
PAD, BOS = 1, 2                     # the stub vocabulary's <blank> and <s>; its </s> is eos_of(V)

# (K, n_best, V, B, max_len, eos_scale): eos_scale < 1 makes EOS likelier; small V makes it frequent anyway
CASES = [
    (1, 1, 4, 3, 30, 1.0), (1, 2, 5, 2, 12, 0.5), (1, 3, 50, 2, 40, 0.3),
    (2, 1, 2, 3, 25, 1.0), (2, 2, 7, 2, 30, 0.6), (2, 3, 300, 3, 6, 1.0),
    (5, 1, 5, 2, 40, 1.0), (5, 1, 6, 4, 40, 0.8), (5, 2, 40, 3, 50, 0.4), (5, 3, 1000, 2, 8, 1.0), (5, 1, 997, 3, 60, 0.15),
    (8, 1, 8, 2, 40, 1.0), (8, 2, 30, 2, 50, 0.5), (8, 3, 600, 2, 7, 1.0),
    (16, 1, 16, 1, 40, 1.0), (16, 2, 17, 2, 40, 0.7), (16, 3, 200, 2, 50, 0.3), (16, 1, 1000, 1, 5, 1.0),
]
SRC_LEN = 5


def eos_of(V):
    return min(3, V - 1)


def draw(seed, step, attempt, rows, V, eos_scale):
    """(lp [rows, V], attn [rows, SRC_LEN]) float32 of one step: log-probability-like keys -|x| * 2 with x standard
    normal, EOS's column scaled by eos_scale instead."""
    rng = np.random.default_rng([seed, step, attempt])
    x = np.abs(rng.standard_normal((rows, V), dtype=np.float32))
    lp = x * np.float32(-2.0)
    lp[:, eos_of(V)] = x[:, eos_of(V)] * np.float32(-2.0 * eos_scale)
    return lp.astype(np.float32), rng.random((rows, SRC_LEN), dtype=np.float32)


def _load_beam():
    io = types.ModuleType("onmt.IO")
    io.PAD_WORD, io.BOS_WORD, io.EOS_WORD = "<blank>", "<s>", "</s>"
    onmt = types.ModuleType("onmt")
    onmt.IO = io
    sys.modules["onmt"], sys.modules["onmt.IO"] = onmt, io
    spec = importlib.util.spec_from_file_location("reference_onmt_beam", REF_BEAM)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.Beam


def _tied(torch, word_lk, beam, K):
    """Whether the top K+1 keys of Beam.advance (computed as it computes them) hold an exact tie."""
    if len(beam.prevKs) > 0:
        lk = word_lk + beam.scores.unsqueeze(1).expand_as(word_lk)
        for i in range(K):
            if beam.nextYs[-1][i] == beam._eos:
                lk[i] = -1e20
    else:
        lk = word_lk[0]
    top = torch.sort(lk.reshape(-1), descending=True)[0][:K + 1]
    return torch.unique(top).numel() < top.numel()


def run_case(torch, Beam, seed, K, n_best, V, B, max_len, eos_scale):
    vocab = types.SimpleNamespace(stoi={"<blank>": PAD, "<s>": BOS, "</s>": eos_of(V)})
    beams = [Beam(K, n_best=n_best, cuda=False, vocab=vocab) for _ in range(B)]
    attempts, scores, prev, done = [], [], [], []
    for i in range(max_len):
        if all(b.done() for b in beams):
            break
        for attempt in range(20):
            lp, attn = draw(seed, i, attempt, K * B, V, eos_scale)
            out = torch.from_numpy(lp).view(K, B, V)
            if not any(_tied(torch, out[:, j], b, K) for j, b in enumerate(beams)):
                break
        else:
            return None
        at = torch.from_numpy(attn).view(K, B, SRC_LEN)
        for j, b in enumerate(beams):
            b.advance(out[:, j], at[:, j])
        attempts.append(attempt)
        scores.append(np.stack([b.scores.numpy() for b in beams]))
        prev.append(np.stack([b.prevKs[-1].numpy() for b in beams]))
        done.append([b.done() for b in beams])
    T = len(attempts)
    rec = {"meta": np.array([seed, K, n_best, V, B, max_len, T], np.int64), "attempts": np.array(attempts, np.int8),
           "scores": np.array(scores, np.float32).reshape(T, B, K), "prev": np.array(prev, np.int16).reshape(T, B, K),
           "next": np.array([np.stack([b.nextYs[t].numpy() for b in beams]) for t in range(T + 1)], np.int16),
           "done": np.array(done, bool).reshape(T, B), "eos_scale": np.float32(eos_scale)}
    fin_s, fin_tk, hyp_tok, hyp_len, hyp_attn, n_fin = [], [], [], [], [], []
    for b in beams:
        sc, ks = b.sortFinished(minimum=n_best)
        n_fin.append(len(sc))
        fin_s += [float(s) for s in sc]
        fin_tk += [(int(t), int(k)) for t, k in ks]
        for t, k in ks[:n_best]:
            hyp, att = b.getHyp(t, k)
            hyp_len.append(len(hyp))
            hyp_tok += [int(h) for h in hyp]
            hyp_attn.append(att.numpy())
    rec.update({"n_finished": np.array(n_fin, np.int32), "fin_scores": np.array(fin_s, np.float32),
                "fin_tk": np.array(fin_tk, np.int32).reshape(-1, 2), "hyp_len": np.array(hyp_len, np.int32),
                "hyp_tok": np.array(hyp_tok, np.int16), "hyp_attn": np.concatenate(hyp_attn).astype(np.float32)})
    return rec


def main():
    import torch
    Beam = _load_beam()
    true_div = torch.Tensor.__truediv__

    def floor_div(self, other):                  # torch 0.3: LongTensor / int is integer division
        if not self.is_floating_point() and isinstance(other, int):
            return torch.div(self, other, rounding_mode="floor")
        return true_div(self, other)

    torch.Tensor.__truediv__ = floor_div
    out = {}
    try:
        for c, (K, n_best, V, B, max_len, eos_scale) in enumerate(CASES):
            seed = 1000 * c
            while True:
                rec = run_case(torch, Beam, seed, K, n_best, V, B, max_len, eos_scale)
                if rec is not None:
                    break
                seed += 1
            for key, val in rec.items():
                out[f"c{c}_{key}"] = val
            print(f"case {c}: K={K} n_best={n_best} V={V} B={B} steps={rec['meta'][-1]}/{max_len} "
                  f"ended on done={bool(rec['done'][-1].all()) if rec['meta'][-1] else False}")
    finally:
        torch.Tensor.__truediv__ = true_div
    np.savez_compressed(OUT, n_cases=np.int64(len(CASES)), **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
