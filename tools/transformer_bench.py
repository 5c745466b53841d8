"""Fused Transformer sublayers (transformer.py: qd_mha_fwd / _bwd, qd_onmt_layernorm_fwd / _bwd) against the torch
chain of the reference (onmt/modules/MultiHeadedAttn.py, UtilClass.py LayerNorm, Transformer.py layers, restated
below), at B = 64, L in {20, 50, 100}, model_dim 512, 8 heads, hidden 2048, eval mode:

  - the attention core alone (projections in, [B, L, D] out), one MultiHeadedAttention-based encoder layer and one
    decoder layer (self-attention with padding plus subsequent masks, context attention, feed-forward);
  - forward, and forward plus backward.

Per case: CUDA-event medians over several rounds, kernel launches counted with torch.profiler in a separate run, the
peak memory above the inputs, and the byte model of the fused attention core kept below.  The card's name and power
limit are read in the same run.  Prints one JSON object; on a machine without a CUDA device it fails.

    python tools/transformer_bench.py [--rounds 7] [--iters 20] [--out profiles/transformer_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from quantized_distillation_b200.transformer import BottleLayerNorm, MultiHeadedAttention, mha_core  # noqa: E402


# ---- the reference's chain, restated in float32 torch -------------------------------------------------------------------
class TorchLayerNorm(nn.Module):
    def __init__(self, d, eps=1e-3):
        super().__init__()
        self.eps = eps
        self.a_2, self.b_2 = nn.Parameter(torch.ones(d)), nn.Parameter(torch.zeros(d))

    def forward(self, z, residual=None):
        shape = z.shape
        z = z.reshape(-1, shape[-1])
        if residual is not None:
            z = z + residual.reshape(-1, shape[-1])
        mu, sd = z.mean(1, keepdim=True), z.std(1, keepdim=True)
        return ((z - mu.expand_as(z)) / (sd.expand_as(z) + self.eps) * self.a_2 + self.b_2).view(shape)


def torch_core(q, k, v, heads, mask=None):
    B, Lq, D = q.shape
    Lk, dh = k.shape[1], D // heads
    sh = lambda x: x.view(B, -1, heads, dh).transpose(1, 2).contiguous().view(B * heads, -1, dh)
    s = torch.bmm(sh(q), sh(k).transpose(1, 2)) / dh ** 0.5
    if mask is not None:
        s = s.view(B, heads, Lq, Lk).masked_fill(mask.unsqueeze(1).expand(B, heads, Lq, Lk), -float("inf")).view(B * heads, Lq, Lk)
    top = torch.softmax(s, -1).view(B, heads, Lq, Lk)[:, 0].contiguous()
    out = torch.bmm(torch.softmax(s, -1), sh(v))
    return out.view(B, heads, Lq, dh).transpose(1, 2).contiguous().view(B, Lq, D), top


class TorchMHA(nn.Module):
    def __init__(self, heads, d, p=0.1):
        super().__init__()
        self.h = heads
        self.linear_keys, self.linear_values, self.linear_query = (nn.Linear(d, d, bias=False) for _ in range(3))
        self.layer_norm = TorchLayerNorm(d)
        self.dropout, self.res_dropout = nn.Dropout(p), nn.Dropout(p)

    def forward(self, key, value, query, mask=None):
        out, top = torch_core(self.linear_query(query), self.linear_keys(key), self.linear_values(value), self.h, mask)
        return self.layer_norm(self.res_dropout(out) + query), top


class FFN(nn.Module):
    def __init__(self, d, hidden, LN):
        super().__init__()
        self.w_1, self.w_2 = nn.Linear(d, hidden), nn.Linear(hidden, d)
        self.layer_norm, self.relu, self.dropout = LN(d), nn.ReLU(), nn.Dropout(0.1)

    def forward(self, x):
        B, L, d = x.shape
        o = self.dropout(self.w_2(self.relu(self.w_1(x.view(B * L, d)))))
        return self.layer_norm(o, residual=x.reshape(B * L, d)).view(B, L, d)


class EncLayer(nn.Module):
    def __init__(self, fused, d=512, heads=8, hidden=2048):
        super().__init__()
        self.self_attn = (MultiHeadedAttention if fused else TorchMHA)(heads, d, 0.1)
        self.feed_forward = FFN(d, hidden, BottleLayerNorm if fused else TorchLayerNorm)

    def forward(self, x, mask):
        return self.feed_forward(self.self_attn(x, x, x, mask=mask)[0])


class DecLayer(nn.Module):
    def __init__(self, fused, d=512, heads=8, hidden=2048):
        super().__init__()
        M = MultiHeadedAttention if fused else TorchMHA
        self.self_attn, self.context_attn = M(heads, d, 0.1), M(heads, d, 0.1)
        self.feed_forward = FFN(d, hidden, BottleLayerNorm if fused else TorchLayerNorm)

    def forward(self, x, ctx, src_mask, dec_mask):
        q, _ = self.self_attn(x, x, x, mask=dec_mask)
        mid, attn = self.context_attn(ctx, ctx, q, mask=src_mask)
        return self.feed_forward(mid), attn


# ---- measurement ----------------------------------------------------------------------------------------------------------
def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({type(e).__name__})"


def core_bytes(B, Lq, Lk, heads, D, backward):
    """HBM bytes the fused core must move at least: forward reads q, k, v and writes out, probs and top; the backward
    reads grad_out, q, k, v, probs and writes grad_q, grad_k, grad_v, with dS written and read back once."""
    f, P = 4, B * heads * Lq * Lk
    fwd = f * (B * Lq * D + 2 * B * Lk * D + B * Lq * D + P + B * Lq * Lk)
    bwd = f * (B * Lq * D + B * Lq * D + 2 * B * Lk * D + P + B * Lq * D + 2 * B * Lk * D + 2 * P)
    return fwd + (bwd if backward else 0)


def time_call(fn, rounds, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / iters)
    ts.sort()
    return ts[len(ts) // 2]


def launches(fn):
    fn()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
               and "Memset" not in e.name)


def peak_above(fn):
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def measure(fns, rounds, iters):
    """fns: {name: callable}; times alternate between the variants round by round."""
    out = {n: {"launches": launches(f), "peak_bytes": peak_above(f)} for n, f in fns.items()}
    per = {n: [] for n in fns}
    for _ in range(rounds):
        for n, f in fns.items():
            per[n].append(time_call(f, 1, iters))
    for n in fns:
        v = sorted(per[n])
        out[n]["ms_median"] = v[len(v) // 2]
    return out


def masks(B, L, g):
    lens = torch.randint(L // 2, L + 1, (B,), generator=g)
    lens[0] = L
    pad = (torch.arange(L)[None, :] >= lens[:, None]).cuda()
    src = pad.unsqueeze(1).expand(B, L, L)
    dec = src | torch.ones(L, L, dtype=torch.bool, device="cuda").triu(1)
    return src, dec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transformer_bench needs a CUDA device")
    B, D, H = 64, 512, 8
    res = {"card": card(), "B": B, "model_dim": D, "heads": H, "cases": []}
    g = torch.Generator().manual_seed(0)
    for L in (20, 50, 100):
        src_mask, dec_mask = masks(B, L, g)
        q, k, v = (torch.randn(B, L, D, device="cuda", requires_grad=True) for _ in range(3))
        go = torch.randn(B, L, D, device="cuda")

        def core_f(bw, fused):
            def f():
                out, top = (mha_core(q, k, v, H, src_mask) if fused else torch_core(q, k, v, H, src_mask))
                if bw:
                    torch.autograd.backward([out], [go])
            return f

        torch.manual_seed(1)
        enc_f, enc_t = EncLayer(True).cuda().eval(), EncLayer(False).cuda().eval()
        enc_t.load_state_dict(enc_f.state_dict())
        dec_f, dec_t = DecLayer(True).cuda().eval(), DecLayer(False).cuda().eval()
        dec_t.load_state_dict(dec_f.state_dict())
        x = torch.randn(B, L, D, device="cuda", requires_grad=True)
        ctx = torch.randn(B, L, D, device="cuda", requires_grad=True)

        def layer_f(m, bw, dec):
            def f():
                y = m(x, ctx, src_mask, dec_mask)[0] if dec else m(x, src_mask)
                if bw:
                    torch.autograd.backward([y], [go])
            return f

        with torch.no_grad():
            y1, y2 = enc_f(x, src_mask), enc_t(x, src_mask)
            diff = (y1 - y2).abs().max().item()
        for bw in (False, True):
            ctxm = torch.enable_grad() if bw else torch.no_grad()
            with ctxm:
                for what, fns in (("core", {"fused": core_f(bw, True), "torch": core_f(bw, False)}),
                                  ("encoder_layer", {"fused": layer_f(enc_f, bw, False), "torch": layer_f(enc_t, bw, False)}),
                                  ("decoder_layer", {"fused": layer_f(dec_f, bw, True), "torch": layer_f(dec_t, bw, True)})):
                    r = measure(fns, a.rounds, a.iters)
                    case = {"what": what, "L": L, "backward": bw, **{f"{n}_{k}": val for n, d in r.items() for k, val in d.items()}}
                    case["fused_over_torch"] = r["fused"]["ms_median"] / r["torch"]["ms_median"]
                    if what == "core":
                        nb = core_bytes(B, L, L, H, D, bw)
                        case["core_min_bytes"] = nb
                        case["core_GBps_at_fused_time"] = nb / (r["fused"]["ms_median"] * 1e-3) / 1e9
                    if what == "encoder_layer":
                        case["encoder_fwd_max_abs_diff"] = diff
                    res["cases"].append(case)
                    print(json.dumps(case), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"], "cases": len(res["cases"])}))


if __name__ == "__main__":
    main()
