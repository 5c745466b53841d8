"""The fused "mlp" (Bahdanau) global-attention core (qd_attn_mlp_fwd / qd_attn_mlp_bwd) and the drop-in
MLPGlobalAttention: the kernels against the float64 oracle (oracle/attention_mlp_oracle.py, mlp_core) within the error
bounds stated in include/qd_b200.h (mlp_core_bounds), at S from 1 to 1000 and H from 1 to 1000, rows from 0 to 3,200
and T in {1, 3, 50}, with the context and uh each as the decoders' transposed [S, N, H] view, as a contiguous [N, S, H]
and at an offset that is not 16-byte aligned, with grad_align given and absent, into NaN-filled outputs; the module
against the reference's own GlobalAttention(attn_type="mlp") (tests/golden/reference_attention_mlp.npz) after
load_state_dict(strict=True); determinism, CUDA graphs, streams, no synchronisation, memory against the torch chain,
packed Linears, a small onmt-protocol decoder through a training step with NMTLossCompute and WeightQuantizer and
through beam search against a twin holding the torch chain, make_global_attention, and every refusal."""
import os
import types

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import attention_mlp_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native
    return _native


def _buf(shape, g, offset=0, scale=1.0):
    """A float32 CUDA tensor of `shape` starting `offset` floats into its storage."""
    n = int(np.prod(shape))
    b = (torch.randn(n + offset, generator=g, dtype=torch.float32) * scale).cuda()
    return b[offset:].view(*shape)


def _slab(Nb, S, H, layout, g, scale=1.0):
    if layout == "nsh":
        return _buf((Nb, S, H), g, scale=scale)
    return _buf((S, Nb, H), g, 1 if layout == "offset" else 0, scale).transpose(0, 1)   # the decoders' transposed bank


def _inputs(Nb, T, S, H, layout, seed):
    g = torch.Generator().manual_seed(seed)
    off = 1 if layout == "offset" else 0
    wq, inp = _buf((Nb, T, H), g, off), _buf((Nb, T, H), g, off)
    v = _buf((H,), g, off, scale=2 * H ** -0.5)
    return wq, _slab(Nb, S, H, layout, g), v, inp, _slab(Nb, S, H, layout, g)


def _nan_like(t):
    return torch.empty_strided(t.shape, t.stride(), device="cuda").fill_(float("nan"))


def _fwd(N, wq, uh, v, inp, ctx):
    Nb, T, H = inp.shape
    S = ctx.shape[1]
    align = torch.full((T, Nb, S), float("nan"), device="cuda")
    concat = torch.full((T, Nb, 2 * H), float("nan"), device="cuda")
    N.check(N.lib().qd_attn_mlp_fwd(N.ptr(wq), N.ptr(uh), uh.stride(0), uh.stride(1), N.ptr(v), N.ptr(inp), N.ptr(ctx),
                                    ctx.stride(0), ctx.stride(1), Nb, T, S, H, N.ptr(align), N.ptr(concat), N.stream_ptr()))
    return align, concat


def _bwd(N, gc, ga, align, wq, uh, v, ctx):
    Nb, T, H = wq.shape
    S = ctx.shape[1]
    gwq, guh, gv, gctx = _nan_like(wq), _nan_like(uh), _nan_like(v), _nan_like(ctx)
    ws = torch.empty(max(int(N.lib().qd_attn_mlp_workspace_bytes(Nb, T, S, H)), 4), dtype=torch.uint8, device="cuda")
    N.check(N.lib().qd_attn_mlp_bwd(N.ptr(gc), N.ptr(ga), N.ptr(align), N.ptr(wq), N.ptr(uh), uh.stride(0), uh.stride(1),
                                    N.ptr(v), N.ptr(ctx), ctx.stride(0), ctx.stride(1), Nb, T, S, H, N.ptr(gwq), N.ptr(guh),
                                    N.ptr(gv), N.ptr(gctx), N.ptr(ws), ws.numel(), N.stream_ptr()))
    return gwq, guh, gv, gctx


def _np(t):
    return t.detach().double().cpu().numpy()


def _within(got, want, bound, what):
    err = np.abs(_np(got) - want)
    assert np.all(err <= bound), f"{what}: max err {err.max():.3e}, worst err/bound {(err / bound).max():.3f}"


def _check_core(N, Nb, T, S, H, layout, with_ga, seed=0):
    wq, uh, v, inp, ctx = _inputs(Nb, T, S, H, layout, seed)
    align, concat = _fwd(N, wq, uh, v, inp, ctx)
    g = torch.Generator().manual_seed(seed + 1)
    gc = torch.randn(T, Nb, 2 * H, generator=g).cuda()
    ga = torch.randn(T, Nb, S, generator=g).cuda() if with_ga else None
    gwq, guh, gv, gctx = _bwd(N, gc, ga, align, wq, uh, v, ctx)
    args = (_np(wq), _np(uh), _np(v), _np(inp), _np(ctx), None if ga is None else _np(ga), _np(gc))
    o, b = O.mlp_core(*args), O.mlp_core_bounds(*args)
    _within(align, o["align"], b["align"], "align")
    _within(concat[..., :H], o["concat"][..., :H], b["c"], "context vector")
    assert torch.equal(concat[..., H:], inp.transpose(0, 1)), "the input half of concat is a copy"
    _within(gwq, o["grad_wq"], b["grad_wq"], "grad_wq")
    _within(guh, o["grad_uh"], b["grad_uh"], "grad_uh")
    _within(gv, o["grad_v"], b["grad_v"], "grad_v")
    _within(gctx, o["grad_context"], b["grad_context"], "grad_context")


@pytest.mark.parametrize("S", [1, 2, 31, 32, 33, 255, 256, 257, 1000])
@pytest.mark.parametrize("H", [1, 3, 4, 500, 512, 550, 1000])
def test_core_matches_oracle_over_s_and_h(N, S, H):
    _check_core(N, 2, 1, S, H, "bank", with_ga=False, seed=S * 7 + H)


@pytest.mark.parametrize("layout", ["bank", "nsh", "offset"])
@pytest.mark.parametrize("with_ga", [False, True])
@pytest.mark.parametrize("Nb,T,S,H", [(1, 1, 5, 3), (5, 3, 33, 550), (64, 1, 50, 550), (64, 50, 50, 500), (7, 3, 257, 4)])
def test_core_matches_oracle_layouts_and_rows(N, Nb, T, S, H, layout, with_ga):
    _check_core(N, Nb, T, S, H, layout, with_ga, seed=Nb + T + S + H)


def test_uh_and_context_in_different_layouts(N):
    Nb, T, S, H = 4, 3, 9, 40
    wq, uh, v, inp, ctx = _inputs(Nb, T, S, H, "bank", 21)
    uh = uh.contiguous()                                            # a contiguous [N, S, H] beside the transposed bank
    align, concat = _fwd(N, wq, uh, v, inp, ctx)
    gc = torch.randn(T, Nb, 2 * H, device="cuda")
    gwq, guh, gv, gctx = _bwd(N, gc, None, align, wq, uh, v, ctx)
    args = (_np(wq), _np(uh), _np(v), _np(inp), _np(ctx), None, _np(gc))
    o, b = O.mlp_core(*args), O.mlp_core_bounds(*args)
    _within(align, o["align"], b["align"], "align")
    _within(guh, o["grad_uh"], b["grad_uh"], "grad_uh")
    _within(gctx, o["grad_context"], b["grad_context"], "grad_context")
    assert guh.stride() == uh.stride() and gctx.stride() == ctx.stride()


def test_zero_rows_is_a_no_op(N):
    ctx = torch.randn(2, 3, 4, device="cuda")
    for Nb, T in ((0, 5), (2, 0)):
        N.check(N.lib().qd_attn_mlp_fwd(None, N.ptr(ctx), 12, 4, None, None, N.ptr(ctx), 12, 4, Nb, T, 3, 4, None, None,
                                        N.stream_ptr()))
        N.check(N.lib().qd_attn_mlp_bwd(None, None, None, None, N.ptr(ctx), 12, 4, None, N.ptr(ctx), 12, 4, Nb, T, 3, 4,
                                        None, None, None, None, None, 0, N.stream_ptr()))
        assert int(N.lib().qd_attn_mlp_workspace_bytes(Nb, T, 3, 4)) == 0


@pytest.mark.parametrize("T", [1, 3])
def test_function_matches_oracle(N, T):
    from quantized_distillation_b200.attention import mlp_attention_core
    Nb, S, H = 6, 40, 550
    wq0, uh0, v0, inp0, ctx0 = _inputs(Nb, T, S, H, "bank", 5)
    wq, uh, inp = (t.detach().clone().requires_grad_(True) for t in (wq0, uh0, inp0))
    v = v0.detach().clone().view(1, H).requires_grad_(True)         # onmt's v.weight is [1, H]
    ctx = ctx0.detach().clone().requires_grad_(True)                # a contiguous [N, S, H] leaf
    align, concat = mlp_attention_core(wq, uh, v, inp, ctx)
    g = torch.Generator().manual_seed(9)
    gc, ga = torch.randn(T, Nb, 2 * H, generator=g).cuda(), torch.randn(T, Nb, S, generator=g).cuda()
    ((concat * gc).sum() + (align * ga).sum()).backward()
    args = (_np(wq0), _np(uh0), _np(v0), _np(inp0), _np(ctx0), _np(ga), _np(gc))
    o, b = O.mlp_core(*args), O.mlp_core_bounds(*args)
    _within(align, o["align"], b["align"], "align")
    _within(concat[..., :H], o["concat"][..., :H], b["c"], "c")
    _within(wq.grad, o["grad_wq"], b["grad_wq"], "grad_wq")
    _within(uh.grad, o["grad_uh"], b["grad_uh"], "grad_uh")
    _within(v.grad.view(H), o["grad_v"], b["grad_v"], "grad_v")
    _within(ctx.grad, o["grad_context"], b["grad_context"], "grad_context")
    assert torch.equal(inp.grad, gc[..., H:].transpose(0, 1))


# ---- the drop-in against the reference's own GlobalAttention(attn_type="mlp") ---------------------------------------
DATA = np.load(os.path.join(HERE, "golden", "reference_attention_mlp.npz"))
WEIGHTS = [("linear_context.weight", "w_ctx"), ("linear_query.weight", "w_q"), ("linear_query.bias", "b_q"),
           ("v.weight", "v"), ("linear_out.weight", "w_out"), ("linear_out.bias", "b_out")]


def _tol(want):
    return 2e-5 * (np.abs(want).max() + 1e-3)


@pytest.mark.parametrize("i", range(len(DATA["cases"])))
def test_drop_in_matches_reference(N, i):
    from quantized_distillation_b200.attention import MLPGlobalAttention
    Nb, T, S, H = DATA["cases"][i].tolist()
    d = {k[len(f"c{i}_"):]: DATA[k] for k in DATA.files if k.startswith(f"c{i}_")}
    m = MLPGlobalAttention(H).cuda()
    m.load_state_dict({k: torch.from_numpy(d[s]).float() for k, s in WEIGHTS}, strict=True)
    x = torch.from_numpy(d["input"]).float().cuda().requires_grad_(True)
    bank = torch.from_numpy(d["bank"]).float().cuda().requires_grad_(True)
    attn_h, align = m(x, bank.transpose(0, 1))
    assert attn_h.shape == d["attn_h"].shape and align.shape == d["align"].shape
    assert attn_h.is_contiguous() and align.is_contiguous()
    ((attn_h * torch.from_numpy(d["grad_h"]).float().cuda()).sum()
     + (align * torch.from_numpy(d["grad_align"]).float().cuda()).sum()).backward()
    params = dict(m.named_parameters())
    checks = [(attn_h, "attn_h"), (align, "align"), (x.grad, "grad_input"), (bank.grad, "grad_bank")]
    checks += [(params[k].grad, "grad_" + s) for k, s in WEIGHTS]
    for got, key in checks:
        assert np.abs(_np(got) - d[key]).max() <= _tol(d[key]), key


def test_state_dict_keys_are_the_references(N):
    from quantized_distillation_b200.attention import MLPGlobalAttention
    assert sorted(MLPGlobalAttention(8).state_dict()) == sorted(k for k, _ in WEIGHTS)
    assert sorted(MLPGlobalAttention(8, coverage=True).state_dict()) == sorted([k for k, _ in WEIGHTS] + ["linear_cover.weight"])
    m = MLPGlobalAttention(8)
    assert all(type(getattr(m, k)) is nn.Linear for k in ("linear_context", "linear_query", "v", "linear_out"))


# ---- determinism, graphs, streams, synchronisation, memory --------------------------------------------------------
def test_row_bits_alone_and_in_a_batch_and_across_runs(N):
    Nb, T, S, H = 40, 7, 50, 550
    wq, uh, v, inp, ctx = _inputs(Nb, T, S, H, "bank", 11)
    align, concat = _fwd(N, wq, uh, v, inp, ctx)
    for n in (0, 17, 39):
        a1, c1 = _fwd(N, wq[n:n + 1].clone(), uh[n:n + 1].clone(), v, inp[n:n + 1].clone(), ctx[n:n + 1].clone())
        assert torch.equal(a1[:, 0], align[:, n]) and torch.equal(c1[:, 0], concat[:, n])
        # one row of that batch entry alone (T = 1)
        a2, c2 = _fwd(N, wq[n:n + 1, 3:4].clone(), uh[n:n + 1], v, inp[n:n + 1, 3:4].clone(), ctx[n:n + 1])
        assert torch.equal(a2[0, 0], align[3, n]) and torch.equal(c2[0, 0], concat[3, n])
    gc = torch.randn(T, Nb, 2 * H, device="cuda")
    ga = torch.randn(T, Nb, S, device="cuda")
    r1, r2 = _bwd(N, gc, ga, align, wq, uh, v, ctx), _bwd(N, gc, ga, align, wq, uh, v, ctx)
    a3, c3 = _fwd(N, wq, uh, v, inp, ctx)
    assert torch.equal(a3, align) and torch.equal(c3, concat)
    assert all(torch.equal(x, y) for x, y in zip(r1, r2))          # grad_wq, grad_uh, grad_v, grad_context


def test_graph_replay_stream_and_no_sync(N):
    from quantized_distillation_b200.attention import MLPGlobalAttention
    torch.manual_seed(0)
    m = MLPGlobalAttention(500).cuda()
    x = torch.randn(64, 500, device="cuda", requires_grad=True)
    bank = torch.randn(50, 64, 500, device="cuda", requires_grad=True)

    def step():
        h, a = m(x, bank.transpose(0, 1))
        (h.sum() + (a * a).sum()).backward()
        return h, a

    h0, a0 = step()
    want = (h0.detach().clone(), a0.detach().clone(), x.grad.clone(), bank.grad.clone(), m.v.weight.grad.clone())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            x.grad = bank.grad = None
            m.zero_grad(set_to_none=True)
            step()
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(x.grad, want[2]) and torch.equal(bank.grad, want[3]) and torch.equal(m.v.weight.grad, want[4])
    torch.cuda.set_sync_debug_mode("error")
    try:
        x.grad = bank.grad = None
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # graph capture of the forward and backward into static outputs; the leaves are made on the side stream, since
    # autograd syncs a leaf's own stream with the capture, which the legacy default stream cannot join
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        xs, bs = x.detach().clone().requires_grad_(True), bank.detach().clone().requires_grad_(True)

        def grads():
            h, a = m(xs, bs.transpose(0, 1))
            return (h, a) + torch.autograd.grad(h.sum() + (a * a).sum(), [xs, bs])

        grads()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        static = grads()
    g.replay()
    torch.cuda.synchronize()
    for got, w in zip(static, want[:4]):
        assert torch.equal(got, w)


def _torch_mlp_chain(wq, uh, v, inp, ctx):
    """The reference's score in stock torch ops: expand to [N, T, S, H], add, tanh, reduce with v."""
    Nb, T, H = inp.shape
    S = ctx.shape[1]
    e = torch.tanh(wq.unsqueeze(2).expand(Nb, T, S, H) + uh.unsqueeze(1).expand(Nb, T, S, H))
    align = torch.softmax((e.reshape(-1, H) @ v.view(H, 1)).view(Nb, T, S), 2)
    concat = torch.cat([torch.bmm(align, ctx), inp], 2)
    return align.transpose(0, 1), concat.transpose(0, 1)


@pytest.mark.parametrize("T", [50, 1])
def test_memory_of_forward_and_backward_at_most_the_torch_chain(N, T):
    from quantized_distillation_b200.attention import mlp_attention_core
    Nb, S, H = 64, 50, 500
    peaks = []
    for fn in (mlp_attention_core, _torch_mlp_chain):
        wq = torch.randn(Nb, T, H, device="cuda", requires_grad=True)
        uh = torch.randn(S, Nb, H, device="cuda", requires_grad=True)
        v = torch.randn(H, device="cuda", requires_grad=True)
        inp = torch.randn(Nb, T, H, device="cuda", requires_grad=True)
        bank = torch.randn(S, Nb, H, device="cuda", requires_grad=True)
        gc = torch.randn(T, Nb, 2 * H, device="cuda")
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        align, concat = fn(wq, uh.transpose(0, 1), v, inp, bank.transpose(0, 1))
        (concat * gc).sum().backward()
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
        del wq, uh, v, inp, bank, gc, align, concat
    assert peaks[0] <= peaks[1], peaks


# ---- packed Linears ------------------------------------------------------------------------------------------------
def test_packed_linears(N):
    from quantized_distillation_b200 import codec
    from quantized_distillation_b200.attention import MLPGlobalAttention
    torch.manual_seed(1)
    holder = nn.Module()
    holder.attn = MLPGlobalAttention(64).cuda()
    pm = codec.pack_model(holder, 4, 256, quantize_first_and_last_layer=True)
    dense = nn.Module()
    dense.attn = MLPGlobalAttention(64).cuda()
    codec.unpack_(pm, dense)
    names = codec.attach_packed_(pm, holder)
    for k in ("linear_context", "linear_query", "v", "linear_out"):
        assert isinstance(getattr(holder.attn, k), codec.PackedLinear), (k, names)
    x, bank = torch.randn(16, 64, device="cuda"), torch.randn(9, 16, 64, device="cuda")
    with torch.no_grad():
        h1, a1 = holder.attn(x, bank.transpose(0, 1))
        h2, a2 = dense.attn(x, bank.transpose(0, 1))
    assert (h1 - h2).abs().max().item() <= 1e-5 and (a1 - a2).abs().max().item() <= 1e-5


# ---- end to end: an onmt-protocol input-feeding decoder, the drop-in against the torch chain -------------------------
E, H_M, V_M, LAYERS = 16, 32, 61, 2
BOS, EOS, PAD = 2, 3, 1


class _TorchMLPAttention(nn.Module):
    """The reference's "mlp" GlobalAttention restated in float32 torch (one step)."""

    def __init__(self, dim):
        super().__init__()
        self.linear_context = nn.Linear(dim, dim, bias=False)
        self.linear_query = nn.Linear(dim, dim, bias=True)
        self.v = nn.Linear(dim, 1, bias=False)
        self.linear_out = nn.Linear(2 * dim, dim, bias=True)

    def forward(self, input, context):
        e = torch.tanh(self.linear_query(input).unsqueeze(1) + self.linear_context(context))
        a = F.softmax(self.v(e).squeeze(2), -1)
        c = torch.bmm(a.unsqueeze(1), context).squeeze(1)
        return self.linear_out(torch.cat([c, input], 1)), a


class _State:
    def __init__(self, hidden, input_feed):
        self.hidden, self.input_feed = hidden, input_feed

    @property
    def _all(self):
        return self.hidden + (self.input_feed,)

    def repeat_beam_size_times(self, k):
        v = [e.repeat(1, k, 1) for e in self._all]
        self.hidden, self.input_feed = tuple(v[:-1]), v[-1]

    def beam_update(self, idx, positions, beam_size):
        for e in self._all:
            a, br, d = e.size()
            sent = e.view(a, beam_size, br // beam_size, d)[:, :, idx]
            sent.copy_(sent.index_select(1, positions))


class _Encoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.embeddings = nn.Embedding(V_M, E, padding_idx=PAD)
        self.rnn = nn.LSTM(E, H_M, LAYERS)

    def forward(self, src, lengths):
        packed = nn.utils.rnn.pack_padded_sequence(self.embeddings(src), lengths.tolist())
        out, hidden = self.rnn(packed)
        return hidden, nn.utils.rnn.pad_packed_sequence(out)[0]


class _Decoder(nn.Module):
    def __init__(self, fused):
        super().__init__()
        from quantized_distillation_b200.attention import make_global_attention
        self.embeddings = nn.Embedding(V_M, E, padding_idx=PAD)
        self.cells = nn.ModuleList([nn.LSTMCell(E + H_M if i == 0 else H_M, H_M) for i in range(LAYERS)])
        self.attn = make_global_attention(H_M, attn_type="mlp") if fused else _TorchMLPAttention(H_M)

    def init_decoder_state(self, src, context, enc_hidden):
        return _State(enc_hidden, context.new_zeros(1, context.shape[1], H_M))

    def forward(self, inp, context, state):
        h, c = state.hidden
        feed = state.input_feed.squeeze(0)
        outs, attns = [], []
        for t in range(inp.shape[0]):
            x = torch.cat([self.embeddings(inp[t].squeeze(-1)), feed], 1)
            hs, cs = [], []
            for i, cell in enumerate(self.cells):
                hi, ci = cell(x, (h[i], c[i]))
                hs.append(hi), cs.append(ci)
                x = hi
            feed, a = self.attn(x, context.transpose(0, 1))
            h, c = torch.stack(hs), torch.stack(cs)
            outs.append(feed), attns.append(a)
        state.hidden, state.input_feed = (h, c), feed.unsqueeze(0)
        return torch.stack(outs), state, {"std": torch.stack(attns)}


class _Model(nn.Module):
    def __init__(self, seed, fused):
        torch.manual_seed(seed)
        super().__init__()
        self.encoder, self.decoder = _Encoder(), _Decoder(fused)
        self.generator = nn.Sequential(nn.Linear(H_M, V_M), nn.LogSoftmax(dim=-1))
        with torch.no_grad():
            self.generator[0].bias[EOS] += 2.5
        self.cuda()


def _twins(seed):
    a, b = _Model(seed, True), _Model(seed, False)
    b.load_state_dict(a.state_dict(), strict=True)
    return a, b


def _src(seed, B=6, S=7):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.sort(torch.randint(1, S + 1, (B,), generator=g), descending=True)[0]
    lengths[0] = S
    src = torch.randint(4, V_M, (S, B), generator=g)
    for b, L in enumerate(lengths.tolist()):
        src[L:, b] = PAD
    return src.cuda(), lengths


def test_decoder_training_step_with_loss_and_quantizer_matches_torch_chain(N):
    from quantized_distillation_b200.cnn_models.conv_forward_model import WeightQuantizer
    from quantized_distillation_b200.nmt_loss import NMTLossCompute
    fused, ref = _twins(0)
    assert isinstance(fused.decoder.attn, __import__("quantized_distillation_b200.attention").attention.MLPGlobalAttention)
    src, lengths = _src(0)
    tgt = torch.randint(4, V_M, (10, src.shape[1]), generator=torch.Generator().manual_seed(1))
    tgt[8:, 3] = PAD
    tgt = tgt.cuda()
    res = []
    for m in (fused, ref):
        m.train()
        wq = WeightQuantizer(m, 8, 256, backprop_quantization_style="truncated")
        wq.quantize_weights_model()
        enc, context = m.encoder(src, lengths)
        state = m.decoder.init_decoder_state(src, context, enc)
        out, _, attn = m.decoder(tgt[:-1].unsqueeze(-1), context, state)
        loss, _ = NMTLossCompute(m.generator, types.SimpleNamespace(stoi={"<blank>": PAD})).compute_loss(None, out, tgt[1:])
        loss.backward()
        wq.restore_weights_model()
        wq.backward_quant_weights_model()
        res.append((loss.item(), out.detach(), attn["std"].detach(),
                    {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}))
    (l1, o1, a1, g1), (l2, o2, a2, g2) = res
    assert abs(l1 - l2) <= 1e-5 * abs(l2)
    assert (o1 - o2).abs().max().item() <= 1e-5 and (a1 - a2).abs().max().item() <= 1e-5
    assert g1.keys() == g2.keys() and "decoder.attn.v.weight" in g1
    for k in g2:
        assert (g1[k] - g2[k]).abs().max().item() <= 2e-4 * (g2[k].abs().max().item() + 1e-6), k


@pytest.mark.parametrize("K,n_best,max_len", [(5, 1, 12), (4, 3, 8)])
def test_beam_search_same_hypotheses_as_torch_chain(N, K, n_best, max_len):
    from quantized_distillation_b200.beam import beam_search
    fused, ref = _twins(3)
    fused.eval(), ref.eval()
    src, lengths = _src(K)
    got = beam_search(fused, src, lengths, K, n_best, max_len, bos=BOS, eos=EOS, pad=PAD)
    want = beam_search(ref, src, lengths, K, n_best, max_len, bos=BOS, eos=EOS, pad=PAD)
    assert got[0] == want[0]
    for gs, ws in zip(got[1], want[1]):
        assert np.allclose(np.array(gs, np.float64), np.array(ws, np.float64), rtol=1e-5, atol=1e-5)


def test_make_global_attention_picks_the_module(N):
    from quantized_distillation_b200.attention import GlobalAttention, MLPGlobalAttention, make_global_attention
    assert type(make_global_attention(8)) is GlobalAttention
    assert type(make_global_attention(8, attn_type="general")) is GlobalAttention
    assert make_global_attention(8, attn_type="general").attn_type == "general"
    m = make_global_attention(8, coverage=True, attn_type="mlp")
    assert type(m) is MLPGlobalAttention and hasattr(m, "linear_cover")
    with pytest.raises(ValueError):
        make_global_attention(8, attn_type="bahdanau")


# ---- refusals ------------------------------------------------------------------------------------------------------
def test_c_abi_refusals(N):
    Nb, T, S, H = 2, 3, 4, 5
    wq, uh, v, inp, ctx = _inputs(Nb, T, S, H, "nsh", 0)
    align = torch.full((T, Nb, S), float("nan"), device="cuda")
    concat = torch.full((T, Nb, 2 * H), float("nan"), device="cuda")
    st = N.stream_ptr()
    lib = N.lib()

    def fwd(wp=None, up=None, uN=S * H, uS=H, vp=None, ip=None, cp=None, sN=S * H, sS=H, n=Nb, t=T, s=S, h=H, ap=None,
            op=None):
        return lib.qd_attn_mlp_fwd(N.ptr(wq) if wp is None else wp, N.ptr(uh) if up is None else up, uN, uS,
                                   N.ptr(v) if vp is None else vp, N.ptr(inp) if ip is None else ip,
                                   N.ptr(ctx) if cp is None else cp, sN, sS, n, t, s, h,
                                   N.ptr(align) if ap is None else ap, N.ptr(concat) if op is None else op, st)

    bad = [dict(n=-1), dict(s=-1), dict(h=-1), dict(t=-1), dict(s=0), dict(h=0), dict(sN=-1), dict(uN=-1), dict(sS=2),
           dict(uS=2), dict(sN=H, sS=H), dict(uN=H, uS=H), dict(sS=1 << 62), dict(uS=1 << 62), dict(wp=0), dict(up=0),
           dict(vp=0), dict(ip=0), dict(cp=0), dict(ap=0), dict(op=0), dict(ap=N.ptr(align) + 2), dict(up=N.ptr(uh) + 1),
           dict(vp=N.ptr(v) + 2), dict(wp=N.ptr(wq) + 1), dict(ap=N.ptr(concat)), dict(op=N.ptr(inp)), dict(ap=N.ptr(ctx)),
           dict(ap=N.ptr(uh)), dict(op=N.ptr(wq)), dict(ap=N.ptr(v)), dict(ap=N.ptr(align) + 2, op=N.ptr(inp)),
           dict(ip=0, cp=N.ptr(ctx) + 1)]
    for kw in bad:
        assert fwd(**kw) == N.QD_ERR_INVALID_ARG, kw
        assert torch.isnan(align).all() and torch.isnan(concat).all(), kw        # nothing written
    assert fwd() == N.QD_OK
    gc = torch.randn(T, Nb, 2 * H, device="cuda")
    outs = [torch.full_like(wq, float("nan")), torch.full_like(uh, float("nan")), torch.full_like(v, float("nan")),
            torch.full_like(ctx, float("nan"))]
    need = int(lib.qd_attn_mlp_workspace_bytes(Nb, T, S, H))
    assert need == (Nb * T * S + Nb * ((S + 7) // 8) * H) * 4
    ws = torch.full((need // 4,), float("nan"), device="cuda")

    def bwd(gp=None, up=None, uS=H, vp=None, wp=None, wn=need, o0=None, o1=None, o2=None, o3=None, sS=H):
        o = [N.ptr(x) for x in outs]
        for i, p in enumerate((o0, o1, o2, o3)):
            if p is not None:
                o[i] = p
        return lib.qd_attn_mlp_bwd(N.ptr(gc) if gp is None else gp, None, N.ptr(align), N.ptr(wq),
                                   N.ptr(uh) if up is None else up, S * H, uS, N.ptr(v) if vp is None else vp, N.ptr(ctx),
                                   S * H, sS, Nb, T, S, H, *o, N.ptr(ws) if wp is None else wp, wn, st)

    def untouched():
        return all(torch.isnan(x).all() for x in outs) and torch.isnan(ws).all()

    assert bwd(wn=need - 1) == N.QD_ERR_WORKSPACE and untouched()
    assert bwd(wp=0) == N.QD_ERR_WORKSPACE and untouched()
    assert bwd(wp=N.ptr(ws) + 2) == N.QD_ERR_WORKSPACE and untouched()
    assert bwd(wp=0, o0=N.ptr(outs[3])) == N.QD_ERR_WORKSPACE and untouched()
    assert bwd(wn=need - 1, gp=0) == N.QD_ERR_INVALID_ARG and untouched()
    for kw in (dict(gp=0), dict(up=0), dict(vp=0), dict(o0=0), dict(o1=0), dict(o2=0), dict(o3=0), dict(o3=N.ptr(ctx)),
               dict(o1=N.ptr(uh)), dict(o2=N.ptr(v)), dict(o0=N.ptr(outs[3])), dict(o2=N.ptr(outs[0])),
               dict(wp=N.ptr(outs[0])), dict(sS=2), dict(uS=2), dict(o0=N.ptr(outs[0]) + 2), dict(o2=N.ptr(outs[2]) + 1),
               dict(up=N.ptr(uh) + 1)):
        assert bwd(**kw) == N.QD_ERR_INVALID_ARG, kw
        assert untouched(), kw
    assert bwd() == N.QD_OK
    torch.cuda.synchronize()
    assert not any(torch.isnan(x).any() for x in outs)
    assert int(lib.qd_attn_mlp_workspace_bytes(-1, T, S, H)) == 0 and int(lib.qd_attn_mlp_workspace_bytes(Nb, T, S, 0)) == 0


def test_python_refusals(N):
    from quantized_distillation_b200.attention import MLPGlobalAttention, mlp_attention_core
    with pytest.raises(ValueError):
        MLPGlobalAttention(8, attn_type="general")
    m = MLPGlobalAttention(8, coverage=True).cuda()
    x, ctx = torch.randn(2, 8, device="cuda"), torch.randn(2, 3, 8, device="cuda")
    with pytest.raises(NotImplementedError):
        m(x, ctx, coverage=torch.zeros(2, 3, device="cuda"))
    with pytest.raises(NotImplementedError):
        m.applyMask(torch.zeros(1, 2, 3, dtype=torch.uint8, device="cuda"))
    m.applyMask(None)
    with pytest.raises(ValueError):
        m(x.cpu(), ctx.cpu())
    with pytest.raises(ValueError):
        m(x.double(), ctx.double())
    with pytest.raises(ValueError):
        m(x, torch.randn(3, 3, 8, device="cuda"))
    h, a = m(x, ctx)
    assert h.shape == (2, 8) and a.shape == (2, 3)
    wq, uh, v, inp, c = _inputs(2, 1, 3, 8, "nsh", 0)
    with pytest.raises(ValueError):
        mlp_attention_core(wq, uh, v[:4], inp, c)
    with pytest.raises(ValueError):
        mlp_attention_core(wq.cpu(), uh, v, inp, c)
    with pytest.raises(ValueError):
        mlp_attention_core(wq, uh[:, :2], v, inp, c)
