"""The fused Transformer sublayers (qd_mha_fwd / qd_mha_bwd, qd_onmt_layernorm_fwd / _bwd, transformer.py) on the GPU:
the kernels against the float64 oracle's bounds (oracle/mha_oracle.py) over sizes, mask kinds (including stride-0
expanded views and an all-masked row), dropout keep masks, grad_top and offset views, with NaN-sentinel guards around
every output; the drop-ins against the reference's own modules (tests/golden/reference_transformer.npz) after
load_state_dict(strict=True); train mode, batch invariance and run-to-run bits, graphs, streams, no host
synchronisation, memory, packed Linears, a transformer encoder-decoder training step against its torch-chain twin, and
every refusal.  The layer structure of onmt/modules/Transformer.py is restated here (the reference is not read)."""
import os
import types

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import mha_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "reference_transformer.npz")
NAN = float("nan")
GUARD = 3


@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native
    return _native


def _np(t):
    return t.detach().double().cpu().numpy()


def _view(x, offset=0):
    """x copied to the GPU, starting `offset` floats into a larger buffer."""
    x = torch.as_tensor(x, dtype=torch.float32)
    b = torch.randn(x.numel() + offset + 1)
    b[offset:offset + x.numel()] = x.reshape(-1)
    return b.cuda()[offset:offset + x.numel()].view(*x.shape)


class _Out:
    """A NaN-filled output view with GUARD NaN floats on each side (and an `offset` float misalignment)."""

    def __init__(self, shape, offset=0):
        n = int(np.prod(shape))
        self.buf = torch.full((n + 2 * GUARD + offset,), NAN, device="cuda")
        self.lo, self.n = GUARD + offset, n
        self.t = self.buf[self.lo:self.lo + n].view(*shape)

    def guards_kept(self):
        return bool(torch.isnan(self.buf[:self.lo]).all()) and bool(torch.isnan(self.buf[self.lo + self.n:]).all())


def _within(got, want, bound, what):
    g = _np(got)
    nan_w = np.isnan(want)
    assert np.array_equal(np.isnan(g), nan_w), f"{what}: NaN pattern differs from the reference's"
    err = np.abs(g[~nan_w] - want[~nan_w])
    b = bound[~nan_w]
    assert np.all(err <= b), f"{what}: max err {err.max():.3e}, worst err/bound {(err / b).max():.3f}"


def _mask(kind, B, Lq, Lk, g):
    """(device mask, numpy mask) of a kind: none, an expanded padding mask (stride 0 over queries), padding plus
    subsequent (materialised), padding with one all-masked row."""
    if kind == "none":
        return None, None
    lens = torch.randint(1, Lk + 1, (B,), generator=g)
    lens[0] = Lk
    pad = torch.arange(Lk)[None, :] >= lens[:, None]
    m = pad.cuda().unsqueeze(1).expand(B, Lq, Lk)
    if kind == "sub":
        m = m | torch.ones(Lq, Lk, dtype=torch.bool, device="cuda").triu(1)
    if kind == "dead":
        m = m.clone()
        m[B - 1, Lq - 1] = True
    return m, m.cpu().numpy()


def _mha_fwd(N, q, k, v, heads, mask, keep, p, off=0):
    B, Lq, D = q.shape
    Lk = k.shape[1]
    out, probs, top = _Out((B, Lq, D), off), _Out((B, heads, Lq, Lk), off), _Out((B, Lq, Lk), off)
    mm = None if mask is None else mask.view(torch.uint8)
    N.check(N.lib().qd_mha_fwd(N.ptr(q), N.ptr(k), N.ptr(v), N.ptr(mm), *(mm.stride() if mm is not None else (0, 0, 0)),
                               N.ptr(keep), 1.0 / (1.0 - p), B, Lq, Lk, heads, D // heads, N.ptr(out.t), N.ptr(probs.t),
                               N.ptr(top.t), N.stream_ptr()))
    return out, probs, top


def _mha_bwd(N, go, gt, q, k, v, probs, heads, mask, keep, p, off=0):
    B, Lq, D = q.shape
    Lk = k.shape[1]
    gq, gk, gv = _Out(q.shape, off), _Out(k.shape, off), _Out(v.shape, off)
    ws = torch.empty(int(N.lib().qd_mha_workspace_bytes(B, heads, Lq, Lk)), dtype=torch.uint8, device="cuda")
    mm = None if mask is None else mask.view(torch.uint8)
    N.check(N.lib().qd_mha_bwd(N.ptr(go), N.ptr(gt), N.ptr(q), N.ptr(k), N.ptr(v), N.ptr(probs), N.ptr(mm),
                               *(mm.stride() if mm is not None else (0, 0, 0)), N.ptr(keep), 1.0 / (1.0 - p), B, Lq, Lk,
                               heads, D // heads, N.ptr(gq.t), N.ptr(gk.t), N.ptr(gv.t), N.ptr(ws), ws.numel(),
                               N.stream_ptr()))
    return gq, gk, gv


def _check_mha(N, B, Lq, Lk, h, dh, mkind, with_keep, with_top, off, seed):
    g = torch.Generator().manual_seed(seed)
    D = h * dh
    qn, kn, vn = (torch.randn(B, L, D, generator=g) for L in (Lq, Lk, Lk))
    q, k, v = _view(qn, off), _view(kn, off), _view(vn, off)
    mask, mask_np = _mask(mkind, B, Lq, Lk, g)
    p = 0.25 if with_keep else 0.0
    keep = (torch.rand(B * h, Lq, Lk, generator=g) >= p).to(torch.uint8).cuda() if with_keep else None
    keep_np = None if keep is None else keep.cpu().numpy()
    out, probs, top = _mha_fwd(N, q, k, v, h, mask, keep, p, off)
    go = _view(torch.randn(B, Lq, D, generator=g), off)
    gt = _view(torch.randn(B, Lq, Lk, generator=g), off) if with_top else None
    gq, gk, gv = _mha_bwd(N, go, gt, q, k, v, probs.t, h, mask, keep, p, off)
    args = (qn.double().numpy(), kn.double().numpy(), vn.double().numpy(), h, mask_np, keep_np, p, _np(go),
            None if gt is None else _np(gt))
    o, b = O.core(*args), O.core_bounds(*args)
    _within(out.t, o["out"], b["out"], "out")
    _within(top.t, o["top"], b["top"], "top_attn")
    _within(gq.t, o["grad_q"], b["grad_q"], "grad_q")
    _within(gk.t, o["grad_k"], b["grad_k"], "grad_k")
    _within(gv.t, o["grad_v"], b["grad_v"], "grad_v")
    assert torch.equal(probs.t[:, 0].nan_to_num(7.0), top.t.nan_to_num(7.0)), "top_attn is head 0 of the probabilities"
    for o_ in (out, probs, top, gq, gk, gv):
        assert o_.guards_kept(), "a write outside an output view"


MHA_SHAPES = [  # B, Lq, Lk, h, dh
    (1, 1, 1, 1, 1), (3, 2, 31, 8, 3), (3, 32, 33, 1, 64), (1, 50, 257, 8, 65), (64, 33, 2, 8, 64),
    (3, 257, 50, 1, 128), (64, 31, 32, 8, 1), (1, 33, 1, 8, 128), (3, 50, 50, 8, 64), (64, 2, 257, 1, 3),
]
MASKS = ["none", "pad", "sub", "dead"]


@pytest.mark.parametrize("i", range(len(MHA_SHAPES)))
@pytest.mark.parametrize("mkind", MASKS)
def test_mha_kernels_match_oracle(N, i, mkind):
    B, Lq, Lk, h, dh = MHA_SHAPES[i]
    if mkind == "sub" and Lq != Lk:
        Lk = Lq
    _check_mha(N, B, Lq, Lk, h, dh, mkind, with_keep=(i % 2 == 1), with_top=(i % 3 != 2), off=i % 2, seed=i * 10 + len(mkind))


@pytest.mark.parametrize("with_keep,with_top,off", [(False, False, 0), (True, True, 1), (True, False, 3), (False, True, 2)])
def test_mha_keep_grad_top_and_offsets(N, with_keep, with_top, off):
    _check_mha(N, 3, 20, 37, 8, 64, "pad", with_keep, with_top, off, seed=off)


def _ln(N, x, r, a, b, eps, gy, off):
    rows, d = x.shape
    y, gx, ga, gb = _Out((rows, d), off), _Out((rows, d), off), _Out((d,), off), _Out((d,), off)
    N.check(N.lib().qd_onmt_layernorm_fwd(N.ptr(x), N.ptr(r), N.ptr(a), N.ptr(b), rows, d, eps, N.ptr(y.t), N.stream_ptr()))
    ws = torch.empty(max(int(N.lib().qd_onmt_layernorm_workspace_bytes(rows, d)), 4), dtype=torch.uint8, device="cuda")
    N.check(N.lib().qd_onmt_layernorm_bwd(N.ptr(gy), N.ptr(x), N.ptr(r), N.ptr(a), rows, d, eps, N.ptr(gx.t), N.ptr(ga.t),
                                          N.ptr(gb.t), N.ptr(ws), ws.numel(), N.stream_ptr()))
    return y, gx, ga, gb


@pytest.mark.parametrize("d", [1, 2, 3, 512, 550, 2048])
@pytest.mark.parametrize("rows,with_res,off", [(1, False, 0), (33, True, 1), (700, True, 0), (70, False, 3)])
def test_layer_norm_kernels_match_oracle(N, d, rows, with_res, off):
    g = torch.Generator().manual_seed(d * 7 + rows)
    xn, rn, gyn = (torch.randn(rows, d, generator=g) for _ in range(3))
    an, bn = 1 + 0.2 * torch.randn(d, generator=g), 0.2 * torch.randn(d, generator=g)
    x, r, gy, a, b = _view(xn, off), _view(rn, off) if with_res else None, _view(gyn, off), _view(an, off), _view(bn, off)
    y, gx, ga, gb = _ln(N, x, r, a, b, 1e-3, gy, off)
    args = (xn.double().numpy(), an.double().numpy(), bn.double().numpy(), 1e-3, rn.double().numpy() if with_res else None,
            gyn.double().numpy())
    o, bd = O.layer_norm(*args), O.layer_norm_bounds(*args)
    _within(y.t, o["y"], bd["y"], "y")
    _within(gx.t, o["grad_x"], bd["grad_x"], "grad_x")
    _within(ga.t, o["grad_a_2"], bd["grad_a_2"], "grad_a_2")
    _within(gb.t, o["grad_b_2"], bd["grad_b_2"], "grad_b_2")
    if d == 1:
        assert torch.equal(gx.t, gy) and not ga.t.any() and not gb.t.any()
    for o_ in (y, gx, ga, gb):
        assert o_.guards_kept(), "a write outside an output view"


# ---- the drop-ins against the reference's modules ----------------------------------------------------------------------
def _restated():
    """PositionwiseFeedForward, TransformerEncoderLayer and TransformerDecoderLayer of onmt/modules/Transformer.py
    restated over the drop-ins."""
    from quantized_distillation_b200.transformer import BottleLayerNorm, MultiHeadedAttention

    class FFN(nn.Module):
        def __init__(self, size, hidden_size, dropout=0.1):
            super().__init__()
            self.w_1, self.w_2 = nn.Linear(size, hidden_size), nn.Linear(hidden_size, size)
            self.layer_norm = BottleLayerNorm(size)
            self.dropout, self.relu = nn.Dropout(dropout), nn.ReLU()

        def forward(self, x):
            B, L, d = x.shape
            out = self.dropout(self.w_2(self.relu(self.w_1(x.view(B * L, d)))))
            return self.layer_norm(out, residual=x.reshape(B * L, d)).view(B, L, d)

    class Enc(nn.Module):
        def __init__(self, size, dropout, head_count=8, hidden_size=2048):
            super().__init__()
            self.self_attn = MultiHeadedAttention(head_count, size, p=dropout)
            self.feed_forward = FFN(size, hidden_size, dropout)

        def forward(self, input, mask):
            mid, _ = self.self_attn(input, input, input, mask=mask)
            return self.feed_forward(mid)

    class Dec(nn.Module):
        def __init__(self, size, dropout, head_count=8, hidden_size=2048, max_size=5000):
            super().__init__()
            self.self_attn = MultiHeadedAttention(head_count, size, p=dropout)
            self.context_attn = MultiHeadedAttention(head_count, size, p=dropout)
            self.feed_forward = FFN(size, hidden_size, dropout)
            self.register_buffer("mask", torch.triu(torch.ones(1, max_size, max_size, dtype=torch.uint8), 1))

        def forward(self, input, context, src_pad_mask, tgt_pad_mask):
            T = tgt_pad_mask.shape[1]
            dec_mask = torch.gt(tgt_pad_mask + self.mask[:, :T, :T].expand_as(tgt_pad_mask), 0)
            query, _ = self.self_attn(input, input, input, mask=dec_mask)
            mid, attn = self.context_attn(context, context, query, mask=src_pad_mask)
            return self.feed_forward(mid), attn

    return FFN, Enc, Dec


FIX = np.load(FIXTURE) if os.path.exists(FIXTURE) else None


def _case(name):
    return {k[len(name) + 1:]: FIX[k] for k in FIX.files if k.startswith(name + "/")}


def _sd(d):
    return {k[2:]: torch.from_numpy(v).float() for k, v in d.items() if k.startswith("p_")}


def _close(got, want, what, rel=2e-5):
    g = _np(got)
    assert np.array_equal(np.isnan(g), np.isnan(want)), f"{what}: NaN pattern"
    f = ~np.isnan(want)
    scale = np.abs(want[f]).max() + 1e-6 if f.any() else 1.0
    assert np.abs(g[f] - want[f]).max(initial=0) <= rel * scale, f"{what}: {np.abs(g[f] - want[f]).max():.3e} vs {scale:.3e}"


def _expanded(m):
    """onmt's padding mask, [B, 1, L] expanded to [B, Lq, L], from a stored [B, Lq, L] array."""
    t = torch.from_numpy(m.astype(bool)).cuda()
    return t[:, :1].expand(t.shape) if (m == m[:, :1]).all() else t


@pytest.mark.parametrize("name", ["mha_self_nomask", "mha_context_pad", "mha_self_pad_sub", "mha_all_masked_row", "mha_one_key"])
def test_multi_headed_attention_matches_reference(N, name):
    from quantized_distillation_b200.transformer import MultiHeadedAttention
    d = _case(name)
    sd = _sd(d)
    dm = d["query"].shape[2]
    heads = {"mha_self_nomask": 4, "mha_context_pad": 2, "mha_self_pad_sub": 8, "mha_all_masked_row": 4, "mha_one_key": 1}[name]
    m = MultiHeadedAttention(heads, dm).cuda().eval()
    m.load_state_dict(sd, strict=True)
    q = torch.from_numpy(d["query"]).float().cuda().requires_grad_(True)
    c = q if "context" not in d else torch.from_numpy(d["context"]).float().cuda().requires_grad_(True)
    mask = _expanded(d["mask"]) if "mask" in d else None
    ret, top = m(c, c, q, mask=mask)
    _close(ret, d["out0"], "ret")
    _close(top, d["out1"], "top_attn")
    ((ret * torch.from_numpy(d["g0"]).float().cuda()).nansum() + (top * torch.from_numpy(d["g1"]).float().cuda()).nansum()).backward()
    _close(q.grad, d["grad_in2"], "grad of query")
    if c is not q:
        _close(c.grad, d["grad_in0"], "grad of key/value")
    for n, p in m.named_parameters():
        _close(p.grad, d[f"grad_{n}"], n, rel=1e-4)


@pytest.mark.parametrize("name", ["ln_2d", "ln_3d", "ln_width1_2d", "ln_width1_3d"])
def test_bottle_layer_norm_matches_reference(N, name):
    from quantized_distillation_b200.transformer import BottleLayerNorm
    d = _case(name)
    m = BottleLayerNorm(d["x"].shape[-1]).cuda()
    m.load_state_dict(_sd(d), strict=True)
    x = torch.from_numpy(d["x"]).float().cuda().requires_grad_(True)
    y = m(x)
    _close(y, d["out0"], "y")
    (y * torch.from_numpy(d["g0"]).float().cuda()).sum().backward()
    _close(x.grad, d["grad_in0"], "grad_x")
    for n, p in m.named_parameters():
        _close(torch.zeros_like(p) if p.grad is None else p.grad, d[f"grad_{n}"], n, rel=1e-4)


def test_feed_forward_and_layers_match_reference(N):
    FFN, Enc, Dec = _restated()
    d = _case("ffn")
    m = FFN(16, 24).cuda().eval()
    m.load_state_dict(_sd(d), strict=True)
    x = torch.from_numpy(d["x"]).float().cuda().requires_grad_(True)
    y = m(x)
    _close(y, d["out0"], "ffn")
    (y * torch.from_numpy(d["g0"]).float().cuda()).sum().backward()
    _close(x.grad, d["grad_in0"], "ffn grad_x")

    d = _case("enc")
    m = Enc(16, 0.1, head_count=4, hidden_size=32).cuda().eval()
    m.load_state_dict(_sd(d), strict=True)
    x = torch.from_numpy(d["x"]).float().cuda().requires_grad_(True)
    y = m(x, _expanded(d["mask"]))
    _close(y, d["out0"], "encoder layer")
    (y * torch.from_numpy(d["g0"]).float().cuda()).sum().backward()
    _close(x.grad, d["grad_in0"], "encoder grad_x", 1e-4)
    for n, p in m.named_parameters():
        _close(p.grad, d[f"grad_{n}"], n, rel=1e-4)

    d = _case("dec")
    m = Dec(16, 0.1, head_count=4, hidden_size=32).cuda().eval()
    sd = _sd(d)
    sd["mask"] = m.mask
    m.load_state_dict(sd, strict=True)
    x = torch.from_numpy(d["x"]).float().cuda().requires_grad_(True)
    c = torch.from_numpy(d["context"]).float().cuda().requires_grad_(True)
    src = _expanded(d["src_pad_mask"])
    tgt = _expanded(d["tgt_pad_mask"]).to(torch.uint8)
    y, attn = m(x, c, src, tgt)
    _close(y, d["out0"], "decoder layer")
    _close(attn, d["out1"], "decoder attn")
    ((y * torch.from_numpy(d["g0"]).float().cuda()).sum() + (attn * torch.from_numpy(d["g1"]).float().cuda()).sum()).backward()
    _close(x.grad, d["grad_in0"], "decoder grad_x", 1e-4)
    _close(c.grad, d["grad_in1"], "decoder grad_context", 1e-4)
    for n, p in m.named_parameters():
        _close(p.grad, d[f"grad_{n}"], n, rel=1e-4)


def test_restated_layers_have_the_reference_keys(N):
    _, Enc, Dec = _restated()
    assert list(Enc(512, 0.1).state_dict().keys()) == [str(k) for k in FIX["keys/encoder_layer"]]
    assert list(Dec(512, 0.1).state_dict().keys()) == [str(k) for k in FIX["keys/decoder_layer"]]


# ---- train mode, determinism, graphs, memory ---------------------------------------------------------------------------
class _TorchMHA(nn.Module):
    """The reference's MultiHeadedAttention restated in float32 torch, its keep mask drawn as the drop-in draws it."""

    def __init__(self, heads, d, p):
        super().__init__()
        self.h, self.p = heads, p
        self.linear_keys, self.linear_values, self.linear_query = (nn.Linear(d, d, bias=False) for _ in range(3))
        self.layer_norm = nn.Module()
        self.layer_norm.a_2, self.layer_norm.b_2 = nn.Parameter(torch.ones(d)), nn.Parameter(torch.zeros(d))
        self.dropout, self.res_dropout = nn.Dropout(p), nn.Dropout(p)

    def forward(self, key, value, query, mask=None):
        B, Lk, d = key.shape
        Lq, h, dh = query.shape[1], self.h, d // self.h
        sh = lambda x: x.view(B, -1, h, dh).transpose(1, 2).contiguous().view(B * h, -1, dh)
        kp, vp, qp = sh(self.linear_keys(key)), sh(self.linear_values(value)), sh(self.linear_query(query))
        keep = torch.rand(B * h, Lq, Lk, device=key.device) >= self.p if self.training and self.p > 0 else None
        s = torch.bmm(qp, kp.transpose(1, 2)) / dh ** 0.5
        if mask is not None:
            s = s.view(B, h, Lq, Lk).masked_fill(mask.unsqueeze(1).bool(), -float("inf")).view(B * h, Lq, Lk)
        a = torch.softmax(s, -1)
        top = a.view(B, h, Lq, Lk)[:, 0].contiguous()
        if keep is not None:
            a = a * keep / (1 - self.p)
        out = torch.bmm(a, vp).view(B, h, Lq, dh).transpose(1, 2).contiguous().view(B, Lq, d)
        z = (self.res_dropout(out) + query).view(B * Lq, d)
        mu, sd = z.mean(1, keepdim=True), z.std(1, keepdim=True)
        return ((z - mu) / (sd + 1e-3) * self.layer_norm.a_2 + self.layer_norm.b_2).view(B, Lq, d), top


def test_train_mode_matches_torch_chain_with_the_same_keep_mask(N):
    from quantized_distillation_b200.transformer import MultiHeadedAttention
    torch.manual_seed(0)
    fused = MultiHeadedAttention(8, 64, p=0.2).cuda().train()
    ref = _TorchMHA(8, 64, 0.2).cuda().train()
    ref.load_state_dict(fused.state_dict(), strict=True)
    key = torch.randn(4, 13, 64, device="cuda")
    query = torch.randn(4, 9, 64, device="cuda")
    mask = (torch.rand(4, 1, 13, device="cuda") < 0.2).expand(4, 9, 13)
    res = []
    for m in (fused, ref):
        torch.cuda.manual_seed(5)
        q = query.clone().requires_grad_(True)
        ret, top = m(key, key, q, mask)
        (ret * ret).sum().backward()
        res.append((ret.detach(), top.detach(), q.grad, {n: p.grad.clone() for n, p in m.named_parameters()}))
    (r1, t1, g1, p1), (r2, t2, g2, p2) = res
    # two float32 chains in different orders; the layer norm's backward cancels, so gradients get a looser bar
    assert (r1 - r2).abs().max() <= 1e-4 * r2.abs().max() and (t1 - t2).abs().max() <= 1e-5
    assert (g1 - g2).abs().max() <= 1e-3 * g2.abs().max()
    for n in p2:
        assert (p1[n] - p2[n]).abs().max() <= 1e-3 * (p2[n].abs().max() + 1e-6), n


def test_row_bits_alone_and_in_a_batch_and_across_runs(N):
    from quantized_distillation_b200.transformer import mha_core, onmt_layer_norm
    torch.manual_seed(2)
    B, L, h, D = 64, 50, 8, 512
    q, k, v = (torch.randn(B, L, D, device="cuda") for _ in range(3))
    out, top = mha_core(q, k, v, h)
    out2, top2 = mha_core(q, k, v, h)
    assert torch.equal(out, out2) and torch.equal(top, top2)
    o1, t1 = mha_core(q[5:6], k[5:6], v[5:6], h)
    assert torch.equal(o1, out[5:6]) and torch.equal(t1, top[5:6])
    o3, _ = mha_core(q[:, 7:9], k, v, h)
    assert torch.equal(o3, out[:, 7:9])
    x, a, b = torch.randn(B * L, D, device="cuda"), torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    y = onmt_layer_norm(x, a, b, 1e-3)
    assert torch.equal(y, onmt_layer_norm(x, a, b, 1e-3)) and torch.equal(y[17:18], onmt_layer_norm(x[17:18], a, b, 1e-3))
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    grads = []
    for _ in range(2):
        o, t = mha_core(qg, kg, vg, h)
        grads.append(torch.autograd.grad((o * o).sum() + t.sum(), [qg, kg, vg]))
    assert all(torch.equal(a_, b_) for a_, b_ in zip(*grads))


def test_graph_replay_stream_and_no_sync(N):
    _, Enc, _ = _restated()
    torch.manual_seed(0)
    m = Enc(64, 0.1, head_count=8, hidden_size=128).cuda().eval()
    x = torch.randn(8, 20, 64, device="cuda", requires_grad=True)
    mask = (torch.rand(8, 1, 20, device="cuda") < 0.2).expand(8, 20, 20)

    def step():
        y = m(x, mask)
        (y * y).sum().backward()
        return y

    y0 = step().detach().clone()
    want = x.grad.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        x.grad = None
        step()
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(x.grad, want)
    torch.cuda.set_sync_debug_mode("error")
    try:
        x.grad = None
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        xs = x.detach().clone().requires_grad_(True)

        def grads():
            y = m(xs, mask)
            return (y,) + torch.autograd.grad((y * y).sum(), [xs])

        grads()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        static = grads()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(static[0], y0) and torch.equal(static[1], want)


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_peak_memory_at_most_the_torch_chain(N):
    from quantized_distillation_b200.transformer import MultiHeadedAttention
    torch.manual_seed(0)
    fused = MultiHeadedAttention(8, 512).cuda().train()
    ref = _TorchMHA(8, 512, 0.1).cuda().train()
    ref.load_state_dict(fused.state_dict())
    x = torch.randn(64, 50, 512, device="cuda", requires_grad=True)
    mask = (torch.rand(64, 1, 50, device="cuda") < 0.2).expand(64, 50, 50)

    def run(m):
        def f():
            ret, top = m(x, x, x, mask)
            (ret.sum() + top.sum()).backward()
        return f

    run(fused)(), run(ref)()
    pf, pr = _peak(run(fused)), _peak(run(ref))
    assert pf <= pr, (pf, pr)


# ---- packed Linears ----------------------------------------------------------------------------------------------------
def test_packed_linears(N):
    from quantized_distillation_b200 import codec
    _, Enc, _ = _restated()
    torch.manual_seed(1)
    holder, dense = nn.Module(), nn.Module()
    holder.layer = Enc(64, 0.1, head_count=8, hidden_size=128).cuda().eval()
    dense.layer = Enc(64, 0.1, head_count=8, hidden_size=128).cuda().eval()
    pm = codec.pack_model(holder, 4, 256, quantize_first_and_last_layer=True)
    codec.unpack_(pm, dense)
    codec.attach_packed_(pm, holder)
    for n in ("linear_keys", "linear_values", "linear_query"):
        assert isinstance(getattr(holder.layer.self_attn, n), codec.PackedLinear), n
    assert isinstance(holder.layer.feed_forward.w_1, codec.PackedLinear)
    assert isinstance(holder.layer.feed_forward.w_2, codec.PackedLinear)
    x = torch.randn(4, 11, 64, device="cuda")
    mask = torch.zeros(4, 11, 11, dtype=torch.bool, device="cuda")
    with torch.no_grad():
        y1, y2 = holder.layer(x, mask), dense.layer(x, mask)
    assert (y1 - y2).abs().max().item() <= 1e-4


# ---- end to end: a small transformer encoder-decoder, one training step against its torch-chain twin -----------------
V_M, D_M, PAD = 37, 64, 1


class _Model(nn.Module):
    def __init__(self, fused):
        super().__init__()
        _, Enc, Dec = _restated()
        self.src_emb = nn.Embedding(V_M, D_M, padding_idx=PAD)
        self.tgt_emb = nn.Embedding(V_M, D_M, padding_idx=PAD)
        self.word_padding_idx = PAD
        self.enc = nn.ModuleList([Enc(D_M, 0.1, head_count=8, hidden_size=128) for _ in range(2)])
        self.dec = nn.ModuleList([Dec(D_M, 0.1, head_count=8, hidden_size=128, max_size=64) for _ in range(2)])
        self.generator = nn.Sequential(nn.Linear(D_M, V_M), nn.LogSoftmax(dim=-1))
        if not fused:
            for layer in list(self.enc) + list(self.dec):
                for name in ("self_attn", "context_attn"):
                    if hasattr(layer, name):
                        setattr(layer, name, _TorchMHA(8, D_M, 0.1))
                layer.feed_forward.layer_norm = _TorchLN(D_M)

    def forward(self, src, tgt):
        """src [S, B], tgt [T, B] -> decoder output [T, B, D] (onmt's TransformerEncoder / Decoder order)."""
        sw, tw = src.t(), tgt.t()
        B, S = sw.shape
        T = tw.shape[1]
        x = self.src_emb(src).transpose(0, 1).contiguous()
        smask = sw.eq(PAD).unsqueeze(1).expand(B, S, S)
        for layer in self.enc:
            x = layer(x, smask)
        y = self.tgt_emb(tgt).transpose(0, 1).contiguous()
        src_pad = sw.eq(PAD).unsqueeze(1).expand(B, T, S)
        tgt_pad = tw.eq(PAD).unsqueeze(1).expand(B, T, T).to(torch.uint8)
        for layer in self.dec:
            y, attn = layer(y, x, src_pad, tgt_pad)
        return y.transpose(0, 1).contiguous(), attn


class _TorchLN(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.a_2, self.b_2 = nn.Parameter(torch.ones(d)), nn.Parameter(torch.zeros(d))

    def forward(self, z, residual=None):
        z = z if residual is None else z + residual
        mu, sd = z.mean(1, keepdim=True), z.std(1, keepdim=True)
        return (z - mu) / (sd + 1e-3) * self.a_2 + self.b_2


def test_training_step_with_loss_and_quantizer_matches_torch_chain(N):
    from quantized_distillation_b200.cnn_models.conv_forward_model import WeightQuantizer
    from quantized_distillation_b200.nmt_loss import NMTLossCompute
    torch.manual_seed(0)
    fused = _Model(True).cuda()
    ref = _Model(False).cuda()
    ref.load_state_dict(fused.state_dict(), strict=True)
    g = torch.Generator().manual_seed(1)
    src = torch.randint(4, V_M, (9, 5), generator=g)
    tgt = torch.randint(4, V_M, (8, 5), generator=g)
    for b, (ls, lt) in enumerate([(9, 8), (7, 8), (5, 6), (9, 3), (2, 5)]):
        src[ls:, b] = PAD
        tgt[lt:, b] = PAD
    src, tgt = src.cuda(), tgt.cuda()
    res = []
    for m in (fused, ref):
        m.train()
        wq = WeightQuantizer(m, 8, 256, backprop_quantization_style="truncated")
        wq.quantize_weights_model()
        torch.cuda.manual_seed(3)
        out, attn = m(src, tgt[:-1])
        loss, _ = NMTLossCompute(m.generator, types.SimpleNamespace(stoi={"<blank>": PAD})).compute_loss(None, out, tgt[1:])
        loss.backward()
        wq.restore_weights_model()
        wq.backward_quant_weights_model()
        res.append((loss.item(), out.detach(), {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}))
    (l1, o1, g1), (l2, o2, g2) = res
    assert abs(l1 - l2) <= 1e-5 * abs(l2)
    assert (o1 - o2).abs().max() <= 1e-4 * o2.abs().max()
    assert g1.keys() == g2.keys() and any("self_attn.linear_query" in k for k in g1)
    for k in g2:
        assert (g1[k] - g2[k]).abs().max() <= 2e-4 * (g2[k].abs().max() + 1e-6), k


# ---- refusals ----------------------------------------------------------------------------------------------------------
def test_c_abi_refusals(N):
    B, Lq, Lk, h, dh = 2, 3, 4, 2, 5
    D = h * dh
    q, k, v = torch.randn(B, Lq, D, device="cuda"), torch.randn(B, Lk, D, device="cuda"), torch.randn(B, Lk, D, device="cuda")
    out, probs, top = _Out((B, Lq, D)), _Out((B, h, Lq, Lk)), _Out((B, Lq, Lk))
    s = N.stream_ptr()
    L = N.lib()

    def fwd(**kw):
        a = dict(q=N.ptr(q), k=N.ptr(k), v=N.ptr(v), mask=None, sb=0, sq=0, sk=0, keep=None, scale=1.0, B=B, Lq=Lq, Lk=Lk,
                 h=h, dh=dh, out=N.ptr(out.t), probs=N.ptr(probs.t), top=N.ptr(top.t))
        a.update(kw)
        return L.qd_mha_fwd(*a.values(), s)

    assert fwd() == N.QD_OK
    for kw in ({"B": 0}, {"Lq": 0}, {"Lk": -1}, {"h": 0}, {"dh": 0}, {"q": None}, {"out": None}, {"top": None},
               {"q": N.ptr(q) + 2}, {"out": N.ptr(out.t) + 1}, {"out": N.ptr(q)}, {"probs": N.ptr(out.t)},
               {"mask": N.ptr(q), "sb": -1}, {"keep": N.ptr(k), "scale": float("inf")}, {"Lk": 1 << 62},
               {"q": N.ptr(q) + 2, "out": N.ptr(q)}, {"out": None, "probs": N.ptr(out.t) + 1}):
        out.buf.fill_(NAN)
        assert fwd(**kw) == N.QD_ERR_INVALID_ARG, kw
        assert torch.isnan(out.buf).all(), kw
    gq, gk, gv = _Out(q.shape), _Out(k.shape), _Out(v.shape)
    ws = torch.empty(int(L.qd_mha_workspace_bytes(B, h, Lq, Lk)), dtype=torch.uint8, device="cuda")
    assert int(L.qd_mha_workspace_bytes(0, h, Lq, Lk)) == 0

    def bwd(**kw):
        a = dict(go=N.ptr(q), gt=None, q=N.ptr(q), k=N.ptr(k), v=N.ptr(v), probs=N.ptr(probs.t), mask=None, sb=0, sq=0,
                 sk=0, keep=None, scale=1.0, B=B, Lq=Lq, Lk=Lk, h=h, dh=dh, gq=N.ptr(gq.t), gk=N.ptr(gk.t),
                 gv=N.ptr(gv.t), ws=N.ptr(ws), nws=ws.numel())
        a.update(kw)
        return L.qd_mha_bwd(*a.values(), s)

    assert bwd() == N.QD_OK
    for kw, rc in (({"ws": None}, N.QD_ERR_WORKSPACE), ({"nws": ws.numel() - 1}, N.QD_ERR_WORKSPACE),
                   ({"ws": N.ptr(ws) + 1}, N.QD_ERR_WORKSPACE), ({"go": None}, N.QD_ERR_INVALID_ARG),
                   ({"probs": None}, N.QD_ERR_INVALID_ARG), ({"gq": N.ptr(q)}, N.QD_ERR_INVALID_ARG),
                   ({"gk": N.ptr(gq.t)}, N.QD_ERR_INVALID_ARG), ({"ws": N.ptr(probs.t)}, N.QD_ERR_INVALID_ARG),
                   ({"gt": N.ptr(q) + 1}, N.QD_ERR_INVALID_ARG), ({"B": 0}, N.QD_ERR_INVALID_ARG),
                   ({"ws": None, "gq": N.ptr(q)}, N.QD_ERR_WORKSPACE), ({"ws": N.ptr(ws) + 1, "go": None}, N.QD_ERR_INVALID_ARG),
                   ({"nws": ws.numel() - 1, "gt": N.ptr(q) + 1}, N.QD_ERR_INVALID_ARG)):
        gq.buf.fill_(NAN)
        assert bwd(**kw) == rc, kw
        assert torch.isnan(gq.buf).all(), kw
    x, a2, b2 = torch.randn(5, 7, device="cuda"), torch.randn(7, device="cuda"), torch.randn(7, device="cuda")
    y, gx, ga, gb = _Out((5, 7)), _Out((5, 7)), _Out((7,)), _Out((7,))
    for args in ((N.ptr(x), None, N.ptr(a2), N.ptr(b2), 5, 0, 1e-3, N.ptr(y.t)),
                 (N.ptr(x), None, N.ptr(a2), N.ptr(b2), -1, 7, 1e-3, N.ptr(y.t)),
                 (N.ptr(x), None, N.ptr(a2), N.ptr(b2), 5, 7, float("nan"), N.ptr(y.t)),
                 (N.ptr(x), None, None, N.ptr(b2), 5, 7, 1e-3, N.ptr(y.t)),
                 (N.ptr(x), None, N.ptr(a2), N.ptr(b2), 5, 7, 1e-3, None),
                 (N.ptr(x), None, N.ptr(a2), N.ptr(b2), 5, 7, 1e-3, N.ptr(x)),
                 (N.ptr(x), N.ptr(y.t), N.ptr(a2), N.ptr(b2), 5, 7, 1e-3, N.ptr(y.t)),
                 (N.ptr(x) + 2, None, N.ptr(a2), N.ptr(b2), 5, 7, 1e-3, N.ptr(y.t))):
        y.buf.fill_(NAN)
        assert L.qd_onmt_layernorm_fwd(*args, s) == N.QD_ERR_INVALID_ARG, args
        assert torch.isnan(y.buf).all()
    need = int(L.qd_onmt_layernorm_workspace_bytes(5, 7))
    lws = torch.empty(need, dtype=torch.uint8, device="cuda")
    base = [N.ptr(x), N.ptr(x), None, N.ptr(a2), 5, 7, 1e-3, N.ptr(gx.t), N.ptr(ga.t), N.ptr(gb.t), N.ptr(lws), need]
    assert L.qd_onmt_layernorm_bwd(*base, s) == N.QD_OK
    for i, val, rc in ((10, None, N.QD_ERR_WORKSPACE), (11, need - 4, N.QD_ERR_WORKSPACE), (7, N.ptr(x), N.QD_ERR_INVALID_ARG),
                       (8, N.ptr(gx.t), N.QD_ERR_INVALID_ARG), (0, None, N.QD_ERR_INVALID_ARG), (9, None, N.QD_ERR_INVALID_ARG)):
        a = list(base)
        a[i] = val
        gx.buf.fill_(NAN)
        assert L.qd_onmt_layernorm_bwd(*a, s) == rc, (i, val)
        assert torch.isnan(gx.buf).all()
    # d = 1 needs no workspace: NULL is accepted, a misaligned pointer is not
    d1 = list(base)
    d1[5], d1[10], d1[11] = 1, None, 0
    assert L.qd_onmt_layernorm_bwd(*d1, s) == N.QD_OK
    d1[10] = N.ptr(lws) + 1
    assert L.qd_onmt_layernorm_bwd(*d1, s) == N.QD_ERR_WORKSPACE
    d1[10], d1[7] = None, N.ptr(x)
    assert L.qd_onmt_layernorm_bwd(*d1, s) == N.QD_ERR_INVALID_ARG


def test_python_refusals(N):
    from quantized_distillation_b200.transformer import (BottleLayerNorm, LayerNorm, MultiHeadedAttention, mha_core,
                                                        onmt_layer_norm)
    with pytest.raises(ValueError):
        MultiHeadedAttention(3, 64)
    with pytest.raises(ValueError):
        MultiHeadedAttention(2, 12)
    q = torch.randn(2, 3, 16, device="cuda")
    for bad in (q.cpu(), q.double(), q[0]):
        with pytest.raises(ValueError):
            mha_core(bad, q, q, 2)
    with pytest.raises(ValueError):
        mha_core(q, q, q, 3)
    with pytest.raises(ValueError):
        mha_core(q, q[:, :2], q, 2)
    with pytest.raises(ValueError):
        mha_core(q, q, q, 2, mask=torch.zeros(2, 3, 2, dtype=torch.bool, device="cuda"))
    with pytest.raises(ValueError):
        mha_core(q, q, q, 2, mask=torch.zeros(2, 3, 3, device="cuda"))
    with pytest.raises(ValueError):
        mha_core(q, q, q, 2, keep=torch.ones(2, 3, 3, dtype=torch.uint8, device="cuda"), p=0.1)
    with pytest.raises(ValueError):
        mha_core(q, q, q, 2, keep=torch.ones(4, 3, 3, dtype=torch.uint8, device="cuda"), p=1.0)
    m = MultiHeadedAttention(2, 16).cuda()
    with pytest.raises(ValueError):
        m(q.cpu(), q.cpu(), q.cpu())
    with pytest.raises(ValueError):
        m(torch.randn(2, 3, 8, device="cuda"), torch.randn(2, 3, 8, device="cuda"), torch.randn(2, 3, 8, device="cuda"))
    x, a = torch.randn(4, 16, device="cuda"), torch.ones(16, device="cuda")
    for args in ((x.cpu(), a, a), (x.double(), a, a), (x, a[:8], a), (x[0], a, a)):
        with pytest.raises(ValueError):
            onmt_layer_norm(*args, 1e-3)
    with pytest.raises(ValueError):
        onmt_layer_norm(x, a, a, float("inf"))
    with pytest.raises(ValueError):
        onmt_layer_norm(x, a, a, 1e-3, residual=x[:2])
    with pytest.raises(ValueError):
        LayerNorm(16).cuda()(q)
    with pytest.raises(ValueError):
        BottleLayerNorm(16).cuda()(torch.randn(1, 2, 3, 16, device="cuda"))
