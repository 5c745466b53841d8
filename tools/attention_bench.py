"""Global attention at the reference's NMT shapes: the drop-in GlobalAttention (fused core) against the reference's
chain restated in torch (linear_in, bmm, softmax, bmm, cat, linear_out, tanh), forward + backward, and one input-feed
decoder step (two LSTMCell layers of 500, embedding 500, then attention) over T = 50 steps with each.

Per shape: the median per-call time between CUDA events over rounds, launches per call (torch.profiler, a separate
run), and the peak memory allocated above the inputs.  Also the fused forward's bytes per call from the byte model
in DESIGN.md section 3.11 (context slab once per tile of 8 rows, q, input, align and concat once) over its time.
Prints one JSON line per shape, with the card's name and power limit, and writes them to profiles/attention_bench.json.

    python tools/attention_bench.py [--rounds 7] [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from quantized_distillation_b200.attention import GlobalAttention  # noqa: E402


class TorchAttention(nn.Module):
    """The reference's forward (onmt/modules/GlobalAttention.py:108-188, "general") in stock torch ops."""

    def __init__(self, dim):
        super().__init__()
        self.linear_in = nn.Linear(dim, dim, bias=False)
        self.linear_out = nn.Linear(2 * dim, dim, bias=False)

    def forward(self, input, context):
        one_step = input.dim() == 2
        if one_step:
            input = input.unsqueeze(1)
        Nb, T, H = input.shape
        S = context.shape[1]
        h_t = self.linear_in(input.reshape(Nb * T, H)).view(Nb, T, H)
        align = torch.softmax(torch.bmm(h_t, context.transpose(1, 2)).view(Nb * T, S), 1).view(Nb, T, S)
        c = torch.bmm(align, context)
        attn_h = torch.tanh(self.linear_out(torch.cat([c, input], 2).view(Nb * T, 2 * H)).view(Nb, T, H))
        if one_step:
            return attn_h.squeeze(1), align.squeeze(1)
        return attn_h.transpose(0, 1).contiguous(), align.transpose(0, 1).contiguous()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(), "unknown"
    return name, power


def fused_bytes(Nb, T, S, H):
    tiles = -(-T // 8)
    R = Nb * T
    return 4 * (Nb * tiles * S * H + 2 * R * H + R * S + 2 * R * H)


def time_call(fn, rounds, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / iters)
    return sorted(times)[len(times) // 2]


def launches(fn):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.name not in ("Memset",)
               and not e.name.startswith("Memcpy"))


def peak_above(fn):
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def attention_case(Nb, T, S, H, backward, rounds, iters):
    torch.manual_seed(0)
    fused = GlobalAttention(H, attn_type="general").cuda()
    ref = TorchAttention(H).cuda()
    ref.load_state_dict(fused.state_dict())
    x = torch.randn(*((Nb, H) if T == 1 else (Nb, T, H)), device="cuda", requires_grad=backward)
    bank = torch.randn(S, Nb, H, device="cuda", requires_grad=backward)
    g = torch.randn(*((Nb, H) if T == 1 else (T, Nb, H)), device="cuda")
    row = {"N": Nb, "T": T, "S": S, "H": H, "backward": backward}
    for name, m in (("fused", fused), ("torch", ref)):
        def call(m=m):
            if backward:
                h, _ = m(x, bank.transpose(0, 1))
                h.backward(g)
            else:
                with torch.no_grad():
                    m(x, bank.transpose(0, 1))
        row[f"{name}_us"] = round(time_call(call, rounds, iters), 2)
        row[f"{name}_launches"] = launches(call)
        row[f"{name}_peak_bytes"] = peak_above(call)
    row["speedup"] = round(row["torch_us"] / row["fused_us"], 3)
    if not backward:
        row["fused_bytes"] = fused_bytes(Nb, T, S, H)
        row["fused_GBps"] = round(row["fused_bytes"] / row["fused_us"] / 1e3, 1)
    return row


class DecoderStep(nn.Module):
    """onmt's InputFeedRNNDecoder loop (onmt/Models.py:316-345) at the reference's shape: input feeding, two
    LSTMCell layers, then attention."""

    def __init__(self, attn, E=500, H=500, layers=2):
        super().__init__()
        self.cells = nn.ModuleList([nn.LSTMCell(E + H if i == 0 else H, H) for i in range(layers)])
        self.attn = attn

    def forward(self, emb, context, hidden, feed):
        h, c = hidden
        outs = []
        for t in range(emb.shape[0]):
            x = torch.cat([emb[t], feed], 1)
            hs, cs = [], []
            for i, cell in enumerate(self.cells):
                hi, ci = cell(x, (h[i], c[i]))
                hs.append(hi), cs.append(ci)
                x = hi
            feed, _ = self.attn(x, context.transpose(0, 1))
            h, c = torch.stack(hs), torch.stack(cs)
            outs.append(feed)
        return torch.stack(outs)


def decoder_case(rounds, Nb=64, T=50, S=50, H=500):
    torch.manual_seed(0)
    fused = DecoderStep(GlobalAttention(H, attn_type="general")).cuda()
    ref = DecoderStep(TorchAttention(H)).cuda()
    ref.load_state_dict(fused.state_dict())
    emb = torch.randn(T, Nb, H, device="cuda", requires_grad=True)
    bank = torch.randn(S, Nb, H, device="cuda", requires_grad=True)
    hidden = (torch.zeros(2, Nb, H, device="cuda"), torch.zeros(2, Nb, H, device="cuda"))
    feed = torch.zeros(Nb, H, device="cuda")
    row = {"decoder": "input-feed, 2 x LSTMCell(500), T = 50, fwd + bwd", "N": Nb, "S": S}
    for name, m in (("fused", fused), ("torch", ref)):
        def call(m=m):
            m(emb, bank, hidden, feed).sum().backward()
        row[f"{name}_ms"] = round(time_call(call, rounds, 3) / 1e3, 3)
    row["speedup"] = round(row["torch_ms"] / row["fused_ms"], 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "attention_bench.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attention_bench needs a CUDA device")
    name, power = card()
    rows = []
    shapes = [(64, 1, S, H, True) for S in (20, 50) for H in (500, 550)]
    shapes += [(64, 50, S, H, True) for S in (20, 50) for H in (500, 550)]
    shapes += [(150, 1, S, H, False) for S in (20, 50) for H in (500, 550)]
    for Nb, T, S, H, bwd in shapes:
        rows.append(attention_case(Nb, T, S, H, bwd, args.rounds, args.iters))
    rows.append(decoder_case(args.rounds))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            r.update(card=name, power_limit=power)
            print(json.dumps(r))
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
