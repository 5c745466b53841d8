""""mlp" (Bahdanau) global attention at the reference's NMT shapes: the drop-in MLPGlobalAttention (fused core) against
the reference's chain in stock torch ops (linear_query, linear_context on the contiguous copy of the bank, expand to
[N, T, S, H], add, tanh, v, softmax, bmm, cat, linear_out), forward + backward except the translation rows, and one
input-feed decoder pass (two LSTMCell layers of 500, embedding 500, then attention; T = 50) with each.

Per shape: the median per-call time between CUDA events over rounds, the two arms alternating within every round
after every shape has been warmed up; launches per call (torch.profiler, a separate run); the peak memory allocated
above the inputs; the fused forward's bytes per call from the byte model in DESIGN.md section 3.14 over its time, and
N*T*S*H per second of each arm.  Prints one JSON line per shape, with the card's name and power limit read in the same
run, and writes them to profiles/attention_mlp_bench.json (or --out).

    python tools/attention_mlp_bench.py [--rounds 7] [--iters 50]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from quantized_distillation_b200.attention import MLPGlobalAttention  # noqa: E402
from tools.attention_bench import DecoderStep, card, launches, peak_above  # noqa: E402


class TorchMLPAttention(nn.Module):
    """The reference's forward (onmt/modules/GlobalAttention.py:93-106, 108-188, "mlp") in stock torch ops."""

    def __init__(self, dim):
        super().__init__()
        self.linear_context = nn.Linear(dim, dim, bias=False)
        self.linear_query = nn.Linear(dim, dim, bias=True)
        self.v = nn.Linear(dim, 1, bias=False)
        self.linear_out = nn.Linear(2 * dim, dim, bias=True)

    def forward(self, input, context):
        one_step = input.dim() == 2
        if one_step:
            input = input.unsqueeze(1)
        Nb, T, H = input.shape
        S = context.shape[1]
        wq = self.linear_query(input.reshape(-1, H)).view(Nb, T, 1, H).expand(Nb, T, S, H)
        uh = self.linear_context(context.contiguous().view(-1, H)).view(Nb, 1, S, H).expand(Nb, T, S, H)
        score = self.v(torch.tanh(wq + uh).view(-1, H)).view(Nb, T, S)
        align = torch.softmax(score.view(Nb * T, S), 1).view(Nb, T, S)
        attn_h = self.linear_out(torch.cat([torch.bmm(align, context), input], 2).view(Nb * T, 2 * H)).view(Nb, T, H)
        if one_step:
            return attn_h.squeeze(1), align.squeeze(1)
        return attn_h.transpose(0, 1).contiguous(), align.transpose(0, 1).contiguous()


def fused_bytes(Nb, T, S, H):
    """The fused forward's HBM traffic: the context and uh slabs once per tile of 8 rows, wq, input and v read, align
    and concat written."""
    tiles = -(-T // 8)
    R = Nb * T
    return 4 * (2 * Nb * tiles * S * H + 2 * R * H + H + R * S + 2 * R * H)


def time_alternating(fns, rounds, iters):
    """Median per-call microseconds of each fn; within a round the fns run one after another, the first one changing
    from round to round."""
    times = [[] for _ in fns]
    for r in range(rounds):
        order = list(range(len(fns)))
        if r % 2:
            order.reverse()
        for i in order:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fns[i]()
            b.record()
            torch.cuda.synchronize()
            times[i].append(a.elapsed_time(b) * 1e3 / iters)
    return [sorted(t)[len(t) // 2] for t in times]


def attention_calls(Nb, T, S, H, backward):
    torch.manual_seed(0)
    fused = MLPGlobalAttention(H).cuda()
    ref = TorchMLPAttention(H).cuda()
    ref.load_state_dict(fused.state_dict(), strict=True)
    x = torch.randn(*((Nb, H) if T == 1 else (Nb, T, H)), device="cuda", requires_grad=backward)
    bank = torch.randn(S, Nb, H, device="cuda", requires_grad=backward)
    g = torch.randn(*((Nb, H) if T == 1 else (T, Nb, H)), device="cuda")
    calls = []
    for m in (fused, ref):
        def call(m=m):
            if backward:
                h, _ = m(x, bank.transpose(0, 1))
                h.backward(g)
            else:
                with torch.no_grad():
                    m(x, bank.transpose(0, 1))
        calls.append(call)
    return calls


def decoder_calls(Nb=64, T=50, S=50, H=500):
    torch.manual_seed(0)
    fused = DecoderStep(MLPGlobalAttention(H)).cuda()
    ref = DecoderStep(TorchMLPAttention(H)).cuda()
    ref.load_state_dict(fused.state_dict(), strict=True)
    emb = torch.randn(T, Nb, H, device="cuda", requires_grad=True)
    bank = torch.randn(S, Nb, H, device="cuda", requires_grad=True)
    hidden = (torch.zeros(2, Nb, H, device="cuda"), torch.zeros(2, Nb, H, device="cuda"))
    feed = torch.zeros(Nb, H, device="cuda")
    return [lambda m=m: m(emb, bank, hidden, feed).sum().backward() for m in (fused, ref)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "attention_mlp_bench.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attention_mlp_bench needs a CUDA device")
    name, power = card()
    shapes = [("input-feed training", 64, 1, S, H, True) for S in (20, 50) for H in (500, 550)]
    shapes += [("StdRNNDecoder", 64, 50, S, H, True) for S in (20, 50) for H in (500, 550)]
    shapes += [("translation, forward", 150, 1, S, H, False) for S in (20, 50) for H in (500, 550)]
    cases = [(call, Nb, T, S, H, bwd, attention_calls(Nb, T, S, H, bwd)) for call, Nb, T, S, H, bwd in shapes]
    for c in cases:                                   # warm every shape of both arms before any timing
        for fn in c[-1]:
            for _ in range(3):
                fn()
    torch.cuda.synchronize()
    rows = []
    for call, Nb, T, S, H, bwd, fns in cases:
        f_us, t_us = time_alternating(fns, args.rounds, args.iters)
        row = {"call": call, "N": Nb, "T": T, "S": S, "H": H, "backward": bwd, "fused_us": round(f_us, 2),
               "torch_us": round(t_us, 2), "speedup": round(t_us / f_us, 3)}
        nts = Nb * T * S * H
        row["fused_NTSH_per_s"], row["torch_NTSH_per_s"] = round(nts / f_us * 1e6), round(nts / t_us * 1e6)
        if not bwd:
            row["fused_bytes"] = fused_bytes(Nb, T, S, H)
            row["fused_GBps"] = round(row["fused_bytes"] / f_us / 1e3, 1)
        rows.append(row)
    for row, (_, Nb, T, S, H, bwd, fns) in zip(rows, cases):    # counted apart from the timing: tracing slows the host
        row["fused_launches"], row["torch_launches"] = launches(fns[0]), launches(fns[1])
        row["fused_peak_MB"], row["torch_peak_MB"] = (round(peak_above(f) / 2 ** 20, 1) for f in fns)
    dec = decoder_calls()
    for fn in dec:
        fn()
    torch.cuda.synchronize()
    f_us, t_us = time_alternating(dec, args.rounds, 3)
    rows.append({"decoder": "input-feed, 2 x LSTMCell(500), T = 50, fwd + bwd", "N": 64, "S": 50,
                 "fused_ms": round(f_us / 1e3, 3), "torch_ms": round(t_us / 1e3, 3), "speedup": round(t_us / f_us, 3)})
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            r.update(card=name, power_limit=power)
            print(json.dumps(r))
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
