"""Generates tests/golden/reference_transformer.npz: the reference's own onmt/modules/MultiHeadedAttn.py, UtilClass.py
and Transformer.py, loaded unmodified by file path with a stub onmt.Utils.aeq and stub onmt.Models.EncoderBase /
DecoderState, run in float64 on the CPU in eval mode as the Transformer encoder and decoder call them
(onmt/modules/Transformer.py:95-104, 246-264): the padding masks are the stride-0 expansions of words.eq(padding_idx),
the decoder's self-attention mask is tgt_pad_mask + the subsequent mask > 0.

Cases: MultiHeadedAttention (self and context attention, Lq != Lk, no mask, a padding mask, padding plus subsequent,
one all-masked row, dh = 1), BottleLayerNorm (2-D, 3-D, width 1), PositionwiseFeedForward, TransformerEncoderLayer
and TransformerDecoderLayer.  Per case: the inputs and masks, every parameter (float32 values, stored as float64),
the outputs and, for random upstream gradients of every output, the gradients of the inputs and of every parameter.
The loss is the nansum of output * gradient, so an all-masked row's NaN outputs take no upstream gradient.  The file
also stores the state_dict key lists of TransformerEncoderLayer and TransformerDecoderLayer at their default sizes.
It is written with fixed zip timestamps, so a rerun gives the same bytes.

Run with the path of a reference checkout:  python tests/golden/make_golden_transformer.py <reference checkout>
"""
import importlib.util
import io
import os
import sys
import types
import zipfile

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_transformer.npz")
PAD = 1

# (name, kind, sizes): mha (B, Lq, Lk, d, heads, mask kind), ln (shape), ffn (B, L, d, hidden),
# enc (B, L, d, heads, hidden), dec (B, T, S, d, heads, hidden).  mask kinds: 0 none, 1 key padding, 2 padding plus
# subsequent (self-attention), 3 key padding with one all-masked row
CASES = [
    ("mha_self_nomask", "mha", (2, 5, 5, 16, 4, 0)),
    ("mha_context_pad", "mha", (3, 4, 6, 16, 2, 1)),
    ("mha_self_pad_sub", "mha", (2, 6, 6, 8, 8, 2)),
    ("mha_all_masked_row", "mha", (2, 3, 4, 16, 4, 3)),
    ("mha_one_key", "mha", (2, 3, 1, 8, 1, 0)),
    ("ln_2d", "ln", (4, 5)),
    ("ln_3d", "ln", (2, 3, 7)),
    ("ln_width1_2d", "ln", (3, 1)),
    ("ln_width1_3d", "ln", (2, 3, 1)),
    ("ffn", "ffn", (2, 3, 16, 24)),
    ("enc", "enc", (3, 5, 16, 4, 32)),
    ("dec", "dec", (2, 4, 5, 16, 4, 32)),
]


def _load(ref):
    import torch.nn  # noqa: F401  (the reference modules import torch themselves)
    onmt = types.ModuleType("onmt")
    utils = types.ModuleType("onmt.Utils")

    def aeq(*args):
        assert all(a == args[0] for a in args[1:]), f"size mismatch {args}"
    utils.aeq = aeq
    models = types.ModuleType("onmt.Models")
    models.EncoderBase = type("EncoderBase", (torch.nn.Module,), {})
    models.DecoderState = type("DecoderState", (object,), {})
    modules = types.ModuleType("onmt.modules")
    onmt.Utils, onmt.Models, onmt.modules = utils, models, modules
    sys.modules.update({"onmt": onmt, "onmt.Utils": utils, "onmt.Models": models, "onmt.modules": modules})
    for name in ("UtilClass", "MultiHeadedAttn", "Transformer"):
        spec = importlib.util.spec_from_file_location(f"onmt.modules.{name}", os.path.join(ref, "onmt", "modules", f"{name}.py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[f"onmt.modules.{name}"] = mod
        spec.loader.exec_module(mod)
        setattr(modules, name, mod)
        for k, v in vars(mod).items():
            if isinstance(v, type) and v.__module__ == mod.__name__:
                setattr(modules, k, v)
    return modules


def _f32(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float32).astype(np.float64)


def _randomize(torch, m, rng):
    """Every parameter from float32 draws (layer-norm gains around 1); returns the state_dict's float entries."""
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("a_2"):
                p.copy_(torch.from_numpy(1 + _f32(rng, *p.shape, scale=0.2)))
            elif n.endswith("weight"):
                p.copy_(torch.from_numpy(_f32(rng, *p.shape, scale=p.shape[1] ** -0.5)))
            else:
                p.copy_(torch.from_numpy(_f32(rng, *p.shape, scale=0.2)))
    return {n: p.detach().numpy().copy() for n, p in m.named_parameters()}


def _words(rng, B, L):
    """token ids [B, L] with padding at the end of every entry but the first (which keeps all L)."""
    w = rng.integers(2, 50, size=(B, L))
    for b in range(1, B):
        n = int(rng.integers(1, L + 1))
        w[b, n:] = PAD
    return w


def _mask(torch, rng, B, Lq, Lk, kind):
    if kind == 0:
        return None, None
    words = torch.from_numpy(_words(rng, B, Lk))
    pad = words.eq(PAD).unsqueeze(1).expand(B, Lq, Lk)
    if kind == 2:
        sub = torch.from_numpy(np.triu(np.ones((1, Lq, Lk)), k=1).astype(np.uint8))
        pad = torch.gt(pad + sub.expand_as(pad), 0)
    if kind == 3:
        pad = pad.clone()
        pad[B - 1, Lq - 1, :] = True
    return pad, pad.numpy().astype(np.uint8)


def _backward(torch, outs, rng):
    grads = [_f32(rng, *o.shape) for o in outs]
    sum((o * torch.from_numpy(g)).nansum() for o, g in zip(outs, grads)).backward()
    return grads


def run_case(torch, M, i, name, kind, sz):
    rng = np.random.default_rng([11, i])
    out = {}
    if kind == "mha":
        B, Lq, Lk, d, h, mk = sz
        m = M.MultiHeadedAttention(h, d, p=0.1).double().eval()
        out.update({f"p_{n}": v for n, v in _randomize(torch, m, rng).items()})
        query = torch.tensor(_f32(rng, B, Lq, d), requires_grad=True)
        ctx = query if Lq == Lk and mk != 1 else torch.tensor(_f32(rng, B, Lk, d), requires_grad=True)
        mask, mask_np = _mask(torch, rng, B, Lq, Lk, mk)
        ret, top = m(ctx, ctx, query, mask=mask)
        gs = _backward(torch, [ret, top], rng)
        out.update(query=query.detach().numpy(), out0=ret.detach().numpy(), out1=top.detach().numpy(),
                   g0=gs[0], g1=gs[1], grad_in2=query.grad.numpy())
        if ctx is not query:
            out.update(context=ctx.detach().numpy(), grad_in0=ctx.grad.numpy())
        if mask_np is not None:
            out["mask"] = mask_np
    elif kind == "ln":
        d = sz[-1]
        m = M.BottleLayerNorm(d).double()
        out.update({f"p_{n}": v for n, v in _randomize(torch, m, rng).items()})
        x = torch.tensor(_f32(rng, *sz), requires_grad=True)
        y = m(x)
        gs = _backward(torch, [y], rng)
        out.update(x=x.detach().numpy(), out0=y.detach().numpy(), g0=gs[0], grad_in0=x.grad.numpy())
        for n, p in m.named_parameters():
            out[f"grad_{n}"] = np.zeros(p.shape) if p.grad is None else p.grad.numpy()
    elif kind == "ffn":
        B, L, d, hid = sz
        m = M.Transformer.PositionwiseFeedForward(d, hid, 0.1).double().eval()
        out.update({f"p_{n}": v for n, v in _randomize(torch, m, rng).items()})
        x = torch.tensor(_f32(rng, B, L, d), requires_grad=True)
        y = m(x)
        gs = _backward(torch, [y], rng)
        out.update(x=x.detach().numpy(), out0=y.detach().numpy(), g0=gs[0], grad_in0=x.grad.numpy())
    elif kind == "enc":
        B, L, d, h, hid = sz
        m = M.Transformer.TransformerEncoderLayer(d, 0.1, head_count=h, hidden_size=hid).double().eval()
        out.update({f"p_{n}": v for n, v in _randomize(torch, m, rng).items()})
        x = torch.tensor(_f32(rng, B, L, d), requires_grad=True)
        mask, mask_np = _mask(torch, rng, B, L, L, 1)
        y = m(x, mask)
        gs = _backward(torch, [y], rng)
        out.update(x=x.detach().numpy(), mask=mask_np, out0=y.detach().numpy(), g0=gs[0], grad_in0=x.grad.numpy())
    else:
        B, T, S, d, h, hid = sz
        m = M.Transformer.TransformerDecoderLayer(d, 0.1, head_count=h, hidden_size=hid).double().eval()
        out.update({f"p_{n}": v for n, v in _randomize(torch, m, rng).items()})
        x = torch.tensor(_f32(rng, B, T, d), requires_grad=True)
        c = torch.tensor(_f32(rng, B, S, d), requires_grad=True)
        src, src_np = _mask(torch, rng, B, T, S, 1)
        tgt, tgt_np = _mask(torch, rng, B, T, T, 1)
        y, attn = m(x, c, src, tgt)
        gs = _backward(torch, [y, attn], rng)
        out.update(x=x.detach().numpy(), context=c.detach().numpy(), src_pad_mask=src_np, tgt_pad_mask=tgt_np,
                   out0=y.detach().numpy(), out1=attn.detach().numpy(), g0=gs[0], g1=gs[1],
                   grad_in0=x.grad.numpy(), grad_in1=c.grad.numpy())
    if kind != "ln":
        for n, p in m.named_parameters():
            out[f"grad_{n}"] = np.zeros(p.shape) if p.grad is None else p.grad.numpy()
    return {f"{name}/{k}": v for k, v in out.items()}


def _write_npz(path, arrays):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(), zipfile.ZIP_DEFLATED)


def main(ref):
    import torch
    torch.manual_seed(0)
    M = _load(ref)
    out = {}
    for i, (name, kind, sz) in enumerate(CASES):
        out.update(run_case(torch, M, i, name, kind, sz))
    enc = M.Transformer.TransformerEncoderLayer(512, 0.1)
    dec = M.Transformer.TransformerDecoderLayer(512, 0.1)
    out["keys/encoder_layer"] = np.array(list(enc.state_dict().keys()))
    out["keys/decoder_layer"] = np.array(list(dec.state_dict().keys()))
    _write_npz(OUT, out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit("usage: python tests/golden/make_golden_transformer.py <reference checkout>")
    main(sys.argv[1])
