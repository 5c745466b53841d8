"""Times onmt's beam search three ways, per step and end to end.

Per step, on the [K*B, V] generator logits of a decoder batch (rows r = k*B + b), each path also reorders the decoder
state of a 2-layer, 500-wide input-feeding LSTM (h and c [2, K*B, 500], input feed [1, K*B, 500]):
  (a) fused: BatchBeam.advance(normalized=False) -- one qd_beam_step (log-softmax, keys, top K, finished counters) and
      one index_select + copy_ per state tensor;
  (b) torch: the same work as a batched torch chain -- log_softmax, + scores, EOS rows to -1e20, view(B, K*V).topk(K),
      div/mod -- and the same reorder;
  (c) reference: onmt's loop (Translator.py:168-177, Beam.py:55-106) restated on current torch on the GPU -- the
      generator's LogSoftmax, then per sentence Beam.advance (its 2K+1 EOS tests read the device) and beam_update.
Shapes: B in {1, 8, 30, 64}, K in {1, 5, 10}, V in {10,004; 50,004}.  Each path advances the same beams step after step;
the table gives the median time per step between CUDA events, and for the fused path GB/s at 4 bytes per logit read
(the lse pass and the key pass each read the row; the second mostly from L2, so this counts one read).

End to end, sentences/s of translation on an NMT-shaped model (embeddings 500, 2 x 500 LSTM encoder, input-feeding
2 x 500 LSTM decoder with general attention, V = 50,004, source length 50, beam 5, n_best 1, 100 steps at most; random
weights, so sentences mostly run the full 100 steps): beam_search at batch 1 and 30, and the reference-style loop at
batch 1 -- what the drivers run -- with the model in float32 and attached packed (4 bits, bucket 256, embeddings and
recurrent layers).  The card name and power limit are read in the same run.

    python -m tools.beam_bench [--out profiles/beam_bench.json] [--iters 20] [--quick]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.nmt_loss_bench import _card  # noqa: E402

BATCHES = [1, 8, 30, 64]
BEAMS = [1, 5, 10]
VOCABS = [10_004, 50_004]
HIDDEN, LAYERS, SRC_LEN = 500, 2, 50
BOS, EOS, PAD = 2, 3, 1


class RefBeam:
    """onmt.Beam (Beam.py:11-106) on current torch, on the device, without the global scorer."""

    def __init__(self, K, n_best, device):
        import torch
        self.K, self.n_best = K, n_best
        self.scores = torch.zeros(K, device=device)
        self.prevKs, self.finished, self.attn, self.eosTop = [], [], [], False
        self.nextYs = [torch.full((K,), PAD, dtype=torch.long, device=device)]
        self.nextYs[0][0] = BOS

    def advance(self, word_lk, attn_out):
        import torch
        V = word_lk.size(1)
        if self.prevKs:
            lk = word_lk + self.scores.unsqueeze(1).expand_as(word_lk)
            for i in range(self.K):
                if self.nextYs[-1][i] == EOS:
                    lk[i] = -1e20
        else:
            lk = word_lk[0]
        best, ids = lk.reshape(-1).topk(self.K, 0, True, True)
        self.scores = best
        prev = torch.div(ids, V, rounding_mode="floor")
        self.prevKs.append(prev)
        self.nextYs.append(ids - prev * V)
        self.attn.append(attn_out.index_select(0, prev))
        for i in range(self.K):
            if self.nextYs[-1][i] == EOS:
                self.finished.append((self.scores[i], len(self.nextYs) - 1, i))
        if self.nextYs[-1][0] == EOS:
            self.eosTop = True

    def done(self):
        return self.eosTop and len(self.finished) >= self.n_best


def beam_update(state, j, positions, K):
    """onmt's DecoderState.beam_update (Models.py:443-449)."""
    for e in state:
        a, br, d = e.size()
        sent = e.view(a, K, br // K, d)[:, :, j]
        sent.copy_(sent.index_select(1, positions))


def _step_paths(B, K, V, iters):
    import torch
    import torch.nn.functional as F
    from quantized_distillation_b200.beam import BatchBeam
    g = torch.Generator(device="cuda").manual_seed(B * 100 + K + V)
    logits = torch.randn(K * B, V, generator=g, device="cuda") * 3
    attn = torch.rand(K * B, SRC_LEN, generator=g, device="cuda")
    state = [torch.randn(LAYERS, K * B, HIDDEN, device="cuda"), torch.randn(LAYERS, K * B, HIDDEN, device="cuda"),
             torch.randn(1, K * B, HIDDEN, device="cuda")]
    fb = BatchBeam(B, K, 1, BOS, EOS, PAD, iters + 3, "cuda")

    def fused():
        fo = fb.advance(logits, attn, normalized=False)
        for e in state:
            e.copy_(e.index_select(1, fo))

    t_scores = torch.zeros(K, B, 1, device="cuda")
    t_last = torch.full((K, B), BOS, dtype=torch.long, device="cuda")

    def chain():
        lk = F.log_softmax(logits, dim=-1).view(K, B, V) + t_scores
        lk = lk.masked_fill(t_last.eq(EOS).unsqueeze(2), -1e20)
        best, ids = lk.transpose(0, 1).reshape(B, K * V).topk(K, 1)
        origin = torch.div(ids, V, rounding_mode="floor")
        t_scores.copy_(best.t().unsqueeze(2))
        t_last.copy_((ids - origin * V).t())
        fo = (origin.t() * B + torch.arange(B, device="cuda")).reshape(-1)
        for e in state:
            e.copy_(e.index_select(1, fo))

    beams = [RefBeam(K, 1, "cuda") for _ in range(B)]

    def reference():
        out = F.log_softmax(logits, dim=-1).view(K, B, V)
        at = attn.view(K, B, -1)
        for j, b in enumerate(beams):
            b.advance(out[:, j], at[:, j])
            beam_update(state, j, b.prevKs[-1], K)

    return {"fused": fused, "torch": chain, "reference": reference}


def bench_steps(B, K, V, iters):
    import torch
    fns = _step_paths(B, K, V, iters)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    out = {"B": B, "K": K, "V": V}
    for name, fn in fns.items():
        n = iters if name != "reference" else max(3, iters // 4)
        for _ in range(3):
            fn()
        times = []
        for _ in range(n):
            ev[0].record()
            fn()
            ev[1].record()
            torch.cuda.synchronize()
            times.append(ev[0].elapsed_time(ev[1]) * 1e3)
        out[name] = {"us_median": statistics.median(times), "us_min": min(times), "us_max": max(times)}
    out["fused"]["GBps_at_4B_per_logit"] = 4 * K * B * V / (out["fused"]["us_median"] * 1e-6) / 1e9
    return out


# ---- end to end -------------------------------------------------------------------------------------------------
def _model(V, seed):
    import torch
    import torch.nn as nn
    import torch.nn.functional as F

    class State:
        def __init__(self, hidden, feed):
            self.hidden, self.input_feed = hidden, feed

        @property
        def _all(self):
            return self.hidden + (self.input_feed,)

        def repeat_beam_size_times(self, k):
            v = [e.repeat(1, k, 1) for e in self._all]
            self.hidden, self.input_feed = tuple(v[:-1]), v[-1]

    class Encoder(nn.Module):
        def __init__(self):
            super().__init__()
            self.embeddings = nn.Embedding(V, HIDDEN, padding_idx=PAD)
            self.rnn = nn.LSTM(HIDDEN, HIDDEN, LAYERS)

        def forward(self, src, lengths):
            out, hidden = self.rnn(self.embeddings(src))
            return hidden, out

    class Decoder(nn.Module):
        def __init__(self):
            super().__init__()
            self.embeddings = nn.Embedding(V, HIDDEN, padding_idx=PAD)
            self.cells = nn.ModuleList([nn.LSTMCell(2 * HIDDEN if i == 0 else HIDDEN, HIDDEN) for i in range(LAYERS)])
            self.linear_in = nn.Linear(HIDDEN, HIDDEN, bias=False)
            self.linear_out = nn.Linear(2 * HIDDEN, HIDDEN, bias=False)

        def init_decoder_state(self, src, context, enc_hidden):
            return State(enc_hidden, context.new_zeros(1, context.shape[1], HIDDEN))

        def forward(self, inp, context, state):
            h, c = state.hidden
            feed = state.input_feed.squeeze(0)
            x = torch.cat([self.embeddings(inp[0].squeeze(-1)), feed], 1)
            hs, cs = [], []
            for i, cell in enumerate(self.cells):
                hi, ci = cell(x, (h[i], c[i]))
                hs.append(hi), cs.append(ci)
                x = hi
            a = F.softmax(torch.bmm(context.transpose(0, 1), self.linear_in(x).unsqueeze(2)).squeeze(2), -1)
            ctx = torch.bmm(a.unsqueeze(1), context.transpose(0, 1)).squeeze(1)
            feed = torch.tanh(self.linear_out(torch.cat([ctx, x], 1)))
            state.hidden, state.input_feed = (torch.stack(hs), torch.stack(cs)), feed.unsqueeze(0)
            return feed.unsqueeze(0), state, {"std": a.unsqueeze(0)}

    class Model(nn.Module):
        def __init__(self):
            super().__init__()
            self.encoder, self.decoder = Encoder(), Decoder()
            self.generator = nn.Sequential(nn.Linear(HIDDEN, V), nn.LogSoftmax(dim=-1))

    torch.manual_seed(seed)
    return Model().cuda().eval()


def reference_translate(model, src, lengths, K, max_len):
    """Translator.translateBatch's loop with per-sentence Beams (restated on current torch)."""
    import torch
    B = src.shape[1]
    with torch.no_grad():
        enc, context = model.encoder(src, lengths)
        state = model.decoder.init_decoder_state(src, context, enc)
        context = context.repeat(1, K, 1)
        state.repeat_beam_size_times(K)
        beams = [RefBeam(K, 1, "cuda") for _ in range(B)]
        for _ in range(max_len):
            if all(b.done() for b in beams):
                break
            inp = torch.stack([b.nextYs[-1] for b in beams]).t().contiguous().view(1, -1, 1)
            dec, state, attn = model.decoder(inp, context, state)
            out = model.generator(dec.squeeze(0)).view(K, B, -1)
            at = attn["std"].squeeze(0).view(K, B, -1)
            for j, b in enumerate(beams):
                b.advance(out[:, j], at[:, j])
                beam_update(state._all, j, b.prevKs[-1], K)
    return beams


def bench_end_to_end(packed, sentences, V, K=5, max_len=100):
    import torch
    from quantized_distillation_b200 import codec
    from quantized_distillation_b200.beam import beam_search
    model = _model(V, 0)
    if packed:
        pm = codec.pack_model(model, 4, 256, quantize_first_and_last_layer=True)
        model = _model(V, 1)
        codec.attach_packed_(pm, model, embeddings=True, recurrent=True)
        model.eval()
    g = torch.Generator().manual_seed(7)
    src_all = torch.randint(4, V, (SRC_LEN, sentences), generator=g).cuda()
    lengths = torch.full((sentences,), SRC_LEN)
    res = {}
    for name, batch in (("fused_b1", 1), ("fused_b30", 30), ("reference_b1", 1)):
        n = sentences if batch > 1 else min(sentences, 6 if name == "reference_b1" else 12)
        runs = [(b0, min(n, b0 + batch)) for b0 in range(0, n, batch)]
        if name.startswith("fused"):
            fn = lambda a, b: beam_search(model, src_all[:, a:b], lengths[a:b], K, 1, max_len, bos=BOS, eos=EOS, pad=PAD)  # noqa: E731
        else:
            fn = lambda a, b: reference_translate(model, src_all[:, a:b], lengths[a:b], K, max_len)  # noqa: E731
        fn(*runs[0])                                   # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for a, b in runs:
            fn(a, b)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        res[name] = {"sentences": n, "seconds": dt, "sentences_per_s": n / dt}
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "beam_bench.json"))
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--sentences", type=int, default=60)
    ap.add_argument("--quick", action="store_true", help="small shapes, for a rehearsal")
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("beam_bench needs a CUDA device: there is nothing to time without one")
    card = _card()
    print(json.dumps(card))
    shapes = [(B, K, V) for V in VOCABS for K in BEAMS for B in BATCHES]
    V_e2e, sentences = 50_004, args.sentences
    if args.quick:
        shapes, V_e2e, sentences = [(2, 5, 1_004)], 1_004, 4
    steps = []
    print(f"{'B':>3} {'K':>3} {'V':>6} | {'fused us':>9} {'GB/s':>6} | {'torch us':>9} | {'ref us':>9} | fused vs torch, vs ref")
    with torch.no_grad():
        for B, K, V in shapes:
            r = bench_steps(B, K, V, args.iters)
            steps.append(r)
            f, t, ref = (r[n]["us_median"] for n in ("fused", "torch", "reference"))
            print(f"{B:3d} {K:3d} {V:6d} | {f:9.1f} {r['fused']['GBps_at_4B_per_logit']:6.0f} | {t:9.1f} | {ref:9.1f} | "
                  f"{t / f:.2f}x {ref / f:.2f}x", flush=True)
            torch.cuda.empty_cache()
    e2e = {}
    for packed in (False, True):
        e2e["packed" if packed else "float32"] = r = bench_end_to_end(packed, sentences, V_e2e)
        print(("packed " if packed else "float32") + " end to end: " +
              ", ".join(f"{k} {v['sentences_per_s']:.2f} sent/s ({v['sentences']} in {v['seconds']:.1f} s)" for k, v in r.items()),
              flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"card": card, "iters": args.iters, "steps": steps, "end_to_end": e2e}, f, indent=1)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
