"""The fused global-attention core (qd_attn_fwd / qd_attn_bwd) and the drop-in GlobalAttention: the kernels against the
float64 oracle (oracle/attention_oracle.py) within the error bounds stated in include/qd_b200.h, at S from 1 to 1000,
H from 1 to 1000 (550 and 3 with rows that are not 16-byte multiples), rows from 0 to 3,200 and T in {1, 3, 50}, with
the context as the decoders' transposed [S, N, H] view, as a contiguous [N, S, H] and at an offset that is not 16-byte
aligned, with grad_align given and absent; the module against the reference's own GlobalAttention
(tests/golden/reference_attention.npz) after load_state_dict(strict=True); determinism, CUDA graphs, streams, no
synchronisation, memory, packed Linears, a small onmt-protocol decoder against a twin holding the torch chain, and
every refusal."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import attention_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native
    return _native


def _buf(shape, g, offset=0):
    """A float32 CUDA tensor of `shape` starting `offset` floats into its storage."""
    n = int(np.prod(shape))
    b = torch.randn(n + offset, generator=g, dtype=torch.float32).cuda()
    return b[offset:].view(*shape)


def _inputs(Nb, T, S, H, layout, seed):
    g = torch.Generator().manual_seed(seed)
    off = 1 if layout == "offset" else 0
    q, inp = _buf((Nb, T, H), g, off), _buf((Nb, T, H), g, off)
    if layout == "nsh":
        ctx = _buf((Nb, S, H), g)
    else:
        ctx = _buf((S, Nb, H), g, off).transpose(0, 1)           # the decoders' context.transpose(0, 1)
    return q, inp, ctx


def _fwd(N, q, inp, ctx, kind=1):
    Nb, T, H = inp.shape
    S = ctx.shape[1]
    align = torch.full((T, Nb, S), float("nan"), device="cuda")
    concat = torch.full((T, Nb, 2 * H), float("nan"), device="cuda")
    N.check(N.lib().qd_attn_fwd(kind, None if kind == 0 else N.ptr(q), N.ptr(inp), N.ptr(ctx), ctx.stride(0), ctx.stride(1),
                                Nb, T, S, H, N.ptr(align), N.ptr(concat), N.stream_ptr()))
    return align, concat


def _bwd(N, gc, ga, align, q, ctx):
    Nb, T, H = q.shape
    S = ctx.shape[1]
    gq = torch.full_like(q, float("nan"))
    gctx = torch.empty_strided(ctx.shape, ctx.stride(), device="cuda").fill_(float("nan"))
    ws = torch.empty(max(int(N.lib().qd_attn_workspace_bytes(Nb * T, S)), 4), dtype=torch.uint8, device="cuda")
    N.check(N.lib().qd_attn_bwd(N.ptr(gc), N.ptr(ga), N.ptr(align), N.ptr(q), N.ptr(ctx), ctx.stride(0), ctx.stride(1), Nb, T, S,
                                H, N.ptr(gq), N.ptr(gctx), N.ptr(ws), ws.numel(), N.stream_ptr()))
    return gq, gctx


def _np(t):
    return t.detach().double().cpu().numpy()


def _within(got, want, bound, what):
    err = np.abs(_np(got) - want)
    assert np.all(err <= bound), f"{what}: max err {err.max():.3e}, worst err/bound {(err / bound).max():.3f}"


def _check_core(N, Nb, T, S, H, layout, with_ga, seed=0):
    q, inp, ctx = _inputs(Nb, T, S, H, layout, seed)
    align, concat = _fwd(N, q, inp, ctx)
    g = torch.Generator().manual_seed(seed + 1)
    gc = torch.randn(T, Nb, 2 * H, generator=g).cuda()
    ga = torch.randn(T, Nb, S, generator=g).cuda() if with_ga else None
    gq, gctx = _bwd(N, gc, ga, align, q, ctx)
    args = (_np(q), _np(inp), _np(ctx), None if ga is None else _np(ga), _np(gc))
    o, b = O.core(*args), O.core_bounds(*args)
    _within(align, o["align"], b["align"], "align")
    _within(concat[..., :H], o["concat"][..., :H], b["c"], "context vector")
    assert torch.equal(concat[..., H:], inp.transpose(0, 1)), "the input half of concat is a copy"
    _within(gq, o["grad_q"], b["grad_q"], "grad_q")
    _within(gctx, o["grad_context"], b["grad_context"], "grad_context")


@pytest.mark.parametrize("S", [1, 2, 31, 32, 33, 255, 256, 257, 1000])
@pytest.mark.parametrize("H", [1, 3, 4, 500, 512, 550, 1000])
def test_core_matches_oracle_over_s_and_h(N, S, H):
    _check_core(N, 3, 1, S, H, "bank", with_ga=False, seed=S * 7 + H)


@pytest.mark.parametrize("layout", ["bank", "nsh", "offset"])
@pytest.mark.parametrize("with_ga", [False, True])
@pytest.mark.parametrize("Nb,T,S,H", [(1, 1, 5, 3), (5, 3, 33, 550), (2, 50, 20, 500), (64, 1, 50, 550), (64, 50, 50, 500),
                                      (7, 3, 257, 4)])
def test_core_matches_oracle_layouts_and_rows(N, Nb, T, S, H, layout, with_ga):
    _check_core(N, Nb, T, S, H, layout, with_ga, seed=Nb + T + S + H)


def test_zero_rows_is_a_no_op(N):
    ctx = torch.randn(2, 3, 4, device="cuda")
    for Nb, T in ((0, 5), (2, 0)):
        N.check(N.lib().qd_attn_fwd(1, None, None, N.ptr(ctx), 12, 4, Nb, T, 3, 4, None, None, N.stream_ptr()))
        N.check(N.lib().qd_attn_bwd(None, None, None, None, N.ptr(ctx), 12, 4, Nb, T, 3, 4, None, None, None, 0, N.stream_ptr()))
    assert int(N.lib().qd_attn_workspace_bytes(0, 3)) == 0


@pytest.mark.parametrize("attn_type", ["dot", "general"])
@pytest.mark.parametrize("T", [1, 3])
def test_function_matches_oracle(N, attn_type, T):
    from quantized_distillation_b200.attention import ATTN_DOT, ATTN_GENERAL, attention_core
    Nb, S, H = 6, 40, 550
    q0, inp0, ctx0 = _inputs(Nb, T, S, H, "bank", 5)
    inp = inp0.clone().requires_grad_(True)
    ctx = ctx0.detach().clone().requires_grad_(True)      # a contiguous [N, S, H] leaf
    if attn_type == "dot":
        align, concat = attention_core(inp, inp, ctx, ATTN_DOT)
    else:
        q = q0.clone().requires_grad_(True)
        align, concat = attention_core(q, inp, ctx, ATTN_GENERAL)
    g = torch.Generator().manual_seed(9)
    gc, ga = torch.randn(T, Nb, 2 * H, generator=g).cuda(), torch.randn(T, Nb, S, generator=g).cuda()
    ((concat * gc).sum() + (align * ga).sum()).backward()
    qn = _np(inp0) if attn_type == "dot" else _np(q0)
    args = (qn, _np(inp0), _np(ctx0), _np(ga), _np(gc))
    o, b = O.core(*args), O.core_bounds(*args)
    _within(align, o["align"], b["align"], "align")
    _within(concat[..., :H], o["concat"][..., :H], b["c"], "c")
    _within(ctx.grad, o["grad_context"], b["grad_context"], "grad_context")
    if attn_type == "dot":
        _within(inp.grad, o["grad_q"] + o["grad_input"], b["grad_q"], "grad_input")
    else:
        _within(q.grad, o["grad_q"], b["grad_q"], "grad_q")
        assert torch.equal(inp.grad, gc[..., H:].transpose(0, 1))


# ---- the drop-in against the reference's own GlobalAttention --------------------------------------------------------
DATA = np.load(os.path.join(HERE, "golden", "reference_attention.npz"))


def _tol(want):
    return 2e-5 * (np.abs(want).max() + 1e-3)


@pytest.mark.parametrize("i", range(len(DATA["cases"])))
def test_drop_in_matches_reference(N, i):
    from quantized_distillation_b200.attention import GlobalAttention
    kind, Nb, T, S, H = DATA["cases"][i].tolist()
    attn_type = ["dot", "general"][kind]
    d = {k[len(f"c{i}_"):]: DATA[k] for k in DATA.files if k.startswith(f"c{i}_")}
    m = GlobalAttention(H, attn_type=attn_type).cuda()
    sd = {"linear_out.weight": torch.from_numpy(d["w_out"]).float()}
    if attn_type == "general":
        sd["linear_in.weight"] = torch.from_numpy(d["w_in"]).float()
    m.load_state_dict(sd, strict=True)
    x = torch.from_numpy(d["input"]).float().cuda().requires_grad_(True)
    bank = torch.from_numpy(d["bank"]).float().cuda().requires_grad_(True)
    attn_h, align = m(x, bank.transpose(0, 1))
    assert attn_h.shape == d["attn_h"].shape and align.shape == d["align"].shape
    assert attn_h.is_contiguous() and align.is_contiguous()
    ((attn_h * torch.from_numpy(d["grad_h"]).float().cuda()).sum()
     + (align * torch.from_numpy(d["grad_align"]).float().cuda()).sum()).backward()
    for got, key in ((attn_h, "attn_h"), (align, "align"), (x.grad, "grad_input"), (bank.grad, "grad_bank"),
                     (m.linear_out.weight.grad, "grad_w_out")) + (((m.linear_in.weight.grad, "grad_w_in"),)
                                                                   if attn_type == "general" else ()):
        assert np.abs(_np(got) - d[key]).max() <= _tol(d[key]), key


# ---- determinism, graphs, streams, synchronisation, memory --------------------------------------------------------
def test_row_bits_alone_and_in_a_batch_and_across_runs(N):
    Nb, T, S, H = 40, 7, 50, 550
    q, inp, ctx = _inputs(Nb, T, S, H, "bank", 11)
    align, concat = _fwd(N, q, inp, ctx)
    for n in (0, 17, 39):
        a1, c1 = _fwd(N, q[n:n + 1].clone(), inp[n:n + 1].clone(), ctx[n:n + 1].clone())
        assert torch.equal(a1[:, 0], align[:, n]) and torch.equal(c1[:, 0], concat[:, n])
        # one row of that batch entry alone (T = 1)
        a2, c2 = _fwd(N, q[n:n + 1, 3:4].clone(), inp[n:n + 1, 3:4].clone(), ctx[n:n + 1])
        assert torch.equal(a2[0, 0], align[3, n]) and torch.equal(c2[0, 0], concat[3, n])
    gc = torch.randn(T, Nb, 2 * H, device="cuda")
    ga = torch.randn(T, Nb, S, device="cuda")
    r1, r2 = _bwd(N, gc, ga, align, q, ctx), _bwd(N, gc, ga, align, q, ctx)
    a3, c3 = _fwd(N, q, inp, ctx)
    assert torch.equal(a3, align) and torch.equal(c3, concat)
    assert all(torch.equal(x, y) for x, y in zip(r1, r2))


def test_graph_replay_stream_and_no_sync(N):
    from quantized_distillation_b200.attention import GlobalAttention
    torch.manual_seed(0)
    m = GlobalAttention(500, attn_type="general").cuda()
    x = torch.randn(64, 500, device="cuda", requires_grad=True)
    bank = torch.randn(50, 64, 500, device="cuda", requires_grad=True)

    def step():
        h, a = m(x, bank.transpose(0, 1))
        (h.sum() + (a * a).sum()).backward()
        return h, a

    h0, a0 = step()
    want = (h0.detach().clone(), a0.detach().clone(), x.grad.clone(), bank.grad.clone(), m.linear_in.weight.grad.clone())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            x.grad = bank.grad = None
            m.zero_grad(set_to_none=True)
            step()
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(x.grad, want[2]) and torch.equal(bank.grad, want[3])
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
    assert torch.equal(static[0], want[0]) and torch.equal(static[1], want[1])
    assert torch.equal(static[2], want[2]) and torch.equal(static[3], want[3])


def test_memory_of_forward_and_backward(N):
    from quantized_distillation_b200.attention import ATTN_GENERAL, attention_core
    Nb, T, S, H = 64, 50, 50, 500
    q = torch.randn(Nb, T, H, device="cuda", requires_grad=True)
    inp = torch.randn(Nb, T, H, device="cuda", requires_grad=True)
    bank = torch.randn(S, Nb, H, device="cuda", requires_grad=True)
    gc = torch.randn(T, Nb, 2 * H, device="cuda")
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    align, concat = attention_core(q, inp, bank.transpose(0, 1), ATTN_GENERAL)
    (concat * gc).sum().backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    R, f = Nb * T, 4
    outputs = R * S * f + R * 2 * H * f                        # align, concat
    grads = 2 * R * H * f + S * Nb * H * f + R * 2 * H * f     # q, input, context; the product concat * gc
    workspace = R * S * f                                      # the backward's gs
    margin = 64 * (R + Nb * S) + (4 << 20)                     # allocator rounding, the sum's scalars
    assert peak <= outputs + grads + workspace + margin, (peak, outputs + grads + workspace + margin)


# ---- packed Linears ------------------------------------------------------------------------------------------------
def test_packed_linears(N):
    from quantized_distillation_b200 import codec
    from quantized_distillation_b200.attention import GlobalAttention
    torch.manual_seed(1)
    holder = nn.Module()
    holder.attn = GlobalAttention(64, attn_type="general").cuda()
    pm = codec.pack_model(holder, 4, 256, quantize_first_and_last_layer=True)
    dense = nn.Module()
    dense.attn = GlobalAttention(64, attn_type="general").cuda()
    codec.unpack_(pm, dense)
    names = codec.attach_packed_(pm, holder)
    assert isinstance(holder.attn.linear_in, codec.PackedLinear) and isinstance(holder.attn.linear_out, codec.PackedLinear), names
    x, bank = torch.randn(16, 64, device="cuda"), torch.randn(9, 16, 64, device="cuda")
    with torch.no_grad():
        h1, a1 = holder.attn(x, bank.transpose(0, 1))
        h2, a2 = dense.attn(x, bank.transpose(0, 1))
    assert (h1 - h2).abs().max().item() <= 1e-5 and (a1 - a2).abs().max().item() <= 1e-5


# ---- end to end: an onmt-protocol input-feeding decoder, the drop-in against the torch chain -------------------------
E, H_M, V_M, LAYERS = 16, 32, 61, 2
BOS, EOS, PAD = 2, 3, 1


class _TorchAttention(nn.Module):
    """The reference's "general" GlobalAttention restated in float32 torch."""

    def __init__(self, dim):
        super().__init__()
        self.linear_in = nn.Linear(dim, dim, bias=False)
        self.linear_out = nn.Linear(2 * dim, dim, bias=False)

    def forward(self, input, context):
        a = F.softmax(torch.bmm(context, self.linear_in(input).unsqueeze(2)).squeeze(2), -1)
        c = torch.bmm(a.unsqueeze(1), context).squeeze(1)
        return torch.tanh(self.linear_out(torch.cat([c, input], 1))), a


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
        from quantized_distillation_b200.attention import GlobalAttention
        self.embeddings = nn.Embedding(V_M, E, padding_idx=PAD)
        self.cells = nn.ModuleList([nn.LSTMCell(E + H_M if i == 0 else H_M, H_M) for i in range(LAYERS)])
        self.attn = GlobalAttention(H_M, attn_type="general") if fused else _TorchAttention(H_M)

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


def test_decoder_training_step_matches_torch_chain(N):
    fused, ref = _twins(0)
    src, lengths = _src(0)
    tgt = torch.randint(4, V_M, (9, src.shape[1], 1), generator=torch.Generator().manual_seed(1)).cuda()
    outs = []
    for m in (fused, ref):
        enc, context = m.encoder(src, lengths)
        state = m.decoder.init_decoder_state(src, context, enc)
        out, _, attn = m.decoder(tgt, context, state)
        loss = F.nll_loss(m.generator(out.view(-1, H_M)), tgt.view(-1), reduction="sum")
        loss.backward()
        outs.append((out.detach(), attn["std"].detach(), {k: p.grad.clone() for k, p in m.named_parameters()}))
    (o1, a1, g1), (o2, a2, g2) = outs
    assert (o1 - o2).abs().max().item() <= 1e-5 and (a1 - a2).abs().max().item() <= 1e-5
    for k in g2:
        scale = g2[k].abs().max().item() + 1e-6
        assert (g1[k] - g2[k]).abs().max().item() <= 1e-4 * scale, k


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


# ---- refusals ------------------------------------------------------------------------------------------------------
def test_c_abi_refusals(N):
    Nb, T, S, H = 2, 3, 4, 5
    q, inp, ctx = _inputs(Nb, T, S, H, "nsh", 0)
    align = torch.empty(T, Nb, S, device="cuda")
    concat = torch.empty(T, Nb, 2 * H, device="cuda")
    st = N.stream_ptr()
    lib = N.lib()

    def fwd(kind=1, qp=None, ip=None, cp=None, sN=S * H, sS=H, n=Nb, t=T, s=S, h=H, ap=None, op=None):
        return lib.qd_attn_fwd(kind, N.ptr(q) if qp is None else qp, N.ptr(inp) if ip is None else ip,
                               N.ptr(ctx) if cp is None else cp, sN, sS, n, t, s, h, N.ptr(align) if ap is None else ap,
                               N.ptr(concat) if op is None else op, st)

    assert fwd() == N.QD_OK
    bad = [dict(kind=2), dict(kind=-1), dict(kind=0), dict(n=-1), dict(s=-1), dict(h=-1), dict(t=-1), dict(s=0), dict(h=0),
           dict(sN=-1), dict(sS=2), dict(sN=H, sS=H), dict(sS=1 << 62), dict(ip=0), dict(cp=0), dict(ap=0), dict(op=0),
           dict(ap=N.ptr(align) + 2), dict(cp=N.ptr(ctx) + 1), dict(ap=N.ptr(concat)), dict(op=N.ptr(inp)),
           dict(ap=N.ptr(ctx)), dict(ap=N.ptr(align) + 2, op=N.ptr(inp)), dict(ip=0, cp=N.ptr(ctx) + 1)]
    for kw in bad:
        assert fwd(**kw) == N.QD_ERR_INVALID_ARG, kw
    gc = torch.randn(T, Nb, 2 * H, device="cuda")
    gq, gctx = torch.empty_like(q), torch.empty_like(ctx)
    need = int(lib.qd_attn_workspace_bytes(Nb * T, S))
    assert need == Nb * T * S * 4
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")

    def bwd(gp=None, wp=None, wn=need, gq_=None, gctx_=None, sS=H):
        return lib.qd_attn_bwd(N.ptr(gc) if gp is None else gp, None, N.ptr(align), N.ptr(q), N.ptr(ctx), S * H, sS, Nb, T, S, H,
                               N.ptr(gq) if gq_ is None else gq_, N.ptr(gctx) if gctx_ is None else gctx_,
                               N.ptr(ws) if wp is None else wp, wn, st)

    assert bwd() == N.QD_OK
    assert bwd(wn=need - 1) == N.QD_ERR_WORKSPACE
    assert bwd(wp=0) == N.QD_ERR_WORKSPACE
    assert bwd(wp=0, gq_=N.ptr(gctx)) == N.QD_ERR_WORKSPACE
    assert bwd(wn=need - 1, gp=0) == N.QD_ERR_INVALID_ARG
    for kw in (dict(gp=0), dict(gq_=0), dict(gctx_=N.ptr(ctx)), dict(gq_=N.ptr(gctx)), dict(wp=N.ptr(gq)), dict(sS=2),
               dict(gq_=N.ptr(gq) + 2)):
        assert bwd(**kw) == N.QD_ERR_INVALID_ARG, kw


def test_python_refusals(N):
    from quantized_distillation_b200.attention import GlobalAttention
    with pytest.raises(NotImplementedError):
        GlobalAttention(8, attn_type="mlp")
    with pytest.raises(ValueError):
        GlobalAttention(8, attn_type="bahdanau")
    m = GlobalAttention(8, attn_type="general", coverage=True).cuda()
    assert sorted(m.state_dict()) == ["linear_cover.weight", "linear_in.weight", "linear_out.weight"]
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
    assert sorted(GlobalAttention(8).state_dict()) == ["linear_out.weight"]
