"""The batched beam search: qd_beam_step against the NumPy oracle (oracle/beam_oracle.py) bit for bit, at K from 1 to
16, B in {0, 1, 7, 30, 64} and V in {K, K+1, 257, 10,004, 50,004}, on the first step and later ones, with rows that
ended on EOS, -inf columns, NaN and an all -inf row, a constructed key tie across the K-th place, and with normalize=1
against the lse of qd_nmt_loss_fwd; BatchBeam replaying the reference's own Beam (tests/golden/reference_beam.npz);
batching, streams, CUDA-graph replay, no synchronisation and every refusal; beam_search on a small onmt-protocol model
against the oracle's per-sentence translateBatch, in float32 and after attach_packed_."""
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import beam_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native
    return _native


def _lse(N, x):
    """Row lse_s of qd_nmt_loss_fwd on the logits x [R, V] (no padding, no teacher)."""
    R, V = x.shape
    row_lse = torch.empty(R, 2, device="cuda")
    loss, counts = torch.empty((), device="cuda"), torch.empty(3, dtype=torch.int64, device="cuda")
    ws = torch.empty(max(int(N.lib().qd_nmt_loss_workspace_bytes(R)), 16), dtype=torch.uint8, device="cuda")
    tg = torch.zeros(R, dtype=torch.int64, device="cuda")
    N.check(N.lib().qd_nmt_loss_fwd(N.ptr(x), None, N.ptr(tg), R, V, -1, 0.0, N.ptr(row_lse), N.ptr(loss), N.ptr(counts),
                                    N.ptr(ws), ws.numel(), N.stream_ptr()))
    return row_lse[:, 0].cpu().numpy()


class Step:
    """Device buffers of one qd_beam_step call."""

    def __init__(self, N, out, B, K, V, eos, scores, last, n_fin, eos_top):
        self.N, self.out, self.B, self.K, self.V, self.eos = N, out, B, K, V, eos
        d = "cuda"
        self.scores = torch.tensor(scores, dtype=torch.float32, device=d)
        self.last = torch.tensor(last, dtype=torch.int64, device=d)
        self.origin, self.flat, self.tokens = (torch.full((K * B,), -7, dtype=torch.int64, device=d) for _ in range(3))
        self.n_fin = torch.tensor(n_fin, dtype=torch.int32, device=d)
        self.eos_top = torch.tensor(eos_top, dtype=torch.uint8, device=d)
        self.ws = torch.empty(max(int(N.lib().qd_beam_workspace_bytes(B, K)), 16), dtype=torch.uint8, device=d)

    def __call__(self, normalize, first, stream=None):
        N = self.N
        return N.lib().qd_beam_step(N.ptr(self.out), normalize, self.B, self.K, self.V, self.eos, first, N.ptr(self.scores),
                                    N.ptr(self.last), N.ptr(self.origin), N.ptr(self.flat), N.ptr(self.tokens),
                                    N.ptr(self.n_fin), N.ptr(self.eos_top), N.ptr(self.ws), self.ws.numel(),
                                    stream if stream is not None else N.stream_ptr())

    def result(self):
        return tuple(t.cpu().numpy() for t in (self.scores, self.origin, self.flat, self.tokens, self.n_fin, self.eos_top))


def _same_float(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and \
        np.array_equal(a[~np.isnan(a)].view(np.uint32), b[~np.isnan(b)].view(np.uint32))


def _check(got, want):
    assert _same_float(got[0], want[0]), "scores"
    for g, w, name in zip(got[1:], want[1:], ("origin", "flat_origin", "tokens", "n_finished", "eos_top")):
        assert np.array_equal(g, w), name


def _inputs(B, K, V, seed, specials):
    g = np.random.default_rng(seed)
    x = (g.standard_normal((K * B, V)) * 3).astype(np.float32)
    eos = int(g.integers(0, V))
    last = g.integers(0, V, K * B)
    scores = (-np.abs(g.standard_normal(K * B)) * 5).astype(np.float32)
    if specials and K * B:
        x[:, g.integers(0, V, max(1, V // 50))] = -np.inf            # masked columns
        last[g.random(K * B) < 0.3] = eos                            # beams that ended on EOS
        if B > 1:
            last[np.arange(K) * B + 1] = eos                         # a sentence whose every beam ended on EOS
        r = int(g.integers(0, K * B))
        x[r] = -np.inf                                               # a row whose logits are all -inf
        r = int(g.integers(0, K * B))
        x[r, int(g.integers(0, V))] = np.nan                         # a NaN
        scores[int(g.integers(0, K * B))] = -np.inf
    n_fin = g.integers(0, 3, B).astype(np.int32)
    eos_top = (g.random(B) < 0.3).astype(np.uint8)
    return x, eos, last, scores, n_fin, eos_top


KS = [1, 2, 5, 8, 13, 16]
BS = [0, 1, 7, 30, 64]


@pytest.mark.parametrize("V", ["K", "K+1", 257, 10_004, 50_004])
@pytest.mark.parametrize("B", BS)
@pytest.mark.parametrize("K", KS)
def test_step_matches_oracle(N, K, B, V):
    V = {"K": K, "K+1": K + 1}.get(V, V)
    for specials in (False, True):
        x, eos, last, scores, n_fin, eos_top = _inputs(B, K, V, K * 1000 + B * 7 + V + specials, specials)
        xd = torch.from_numpy(x).cuda()
        lse = _lse(N, xd) if K * B else np.zeros(0, np.float32)
        for normalize in (0, 1):
            lp = O.log_probs(x, lse) if normalize else x
            for first in (1, 0):
                st = Step(N, xd, B, K, V, eos, scores, last, n_fin, eos_top)
                N.check(st(normalize, first))
                want = O.beam_step(lp, B, K, eos, bool(first), scores, last, n_fin, eos_top)
                _check(st.result(), want)


def test_key_tie_across_kth_place(N):
    """Two different logits whose keys round to the same float32 across the K-th place: the tie goes to the lower
    column, which a per-row selection by logit would already have dropped."""
    K, B, V = 2, 1, 16
    x = np.full((K * B, V), -10.0, np.float32)
    x[0, 1], x[0, 3], x[0, 7] = -0.1, -0.50001, -0.5
    scores = np.array([-1000.0, -1000.0], np.float32)
    assert x[0, 3] != x[0, 7] and np.float32(x[0, 3] + scores[0]) == np.float32(x[0, 7] + scores[0])
    st = Step(N, torch.from_numpy(x).cuda(), B, K, V, 15, scores, [0, 0], [0], [0])
    N.check(st(0, 0))
    got = st.result()
    assert got[3].tolist() == [1, 3] and got[1].tolist() == [0, 0]
    _check(got, O.beam_step(x, B, K, 15, False, scores, [0, 0], [0], [0]))


def test_lse_is_the_nmt_loss_lse(N):
    """normalize=1 subtracts exactly qd_nmt_loss_fwd's lse_s of the row, whatever the row's alignment: the first
    step's scores are fl(x - lse) of row 0 at the selected columns (every column when V <= 16)."""
    for V in (5, 16, 1025, 50_004):
        xd = torch.randn(1, V, device="cuda") * 4
        lp = O.log_probs(xd.cpu().numpy(), _lse(N, xd))[0]
        K = min(V, 16)
        for offset in (0, 1, 2, 3):
            big = torch.empty(K * V + offset, device="cuda")[offset:].view(K, V)
            big.copy_(xd.expand(K, V))
            st = Step(N, big, 1, K, V, 0, np.zeros(K, np.float32), np.zeros(K, np.int64), [0], [0])
            N.check(st(1, 1))
            idx = st.result()[3]
            assert np.array_equal(idx, O.top_k(lp, K)) and _same_float(st.result()[0], lp[idx])


def _gen():
    spec = importlib.util.spec_from_file_location("make_golden_beam", os.path.join(HERE, "golden", "make_golden_beam.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_batch_beam_replays_reference(N):
    from quantized_distillation_b200.beam import BatchBeam
    G = _gen()
    data = np.load(os.path.join(HERE, "golden", "reference_beam.npz"))
    for c in range(int(data["n_cases"])):
        r = {k[len(f"c{c}_"):]: data[k] for k in data.files if k.startswith(f"c{c}_")}
        seed, K, n_best, V, B, max_len, T = (int(v) for v in r["meta"])
        bb = BatchBeam(B, K, n_best, G.BOS, G.eos_of(V), G.PAD, max_len, "cuda")
        t = 0
        while t < max_len and not bb.done():
            lp, at = G.draw(seed, t, int(r["attempts"][t]), K * B, V, float(r["eos_scale"]))
            bb.advance(torch.from_numpy(lp).cuda(), torch.from_numpy(at).cuda(), normalized=True)
            t += 1
        assert t == T, c
        assert np.array_equal(bb.step_scores[:T].cpu().numpy().transpose(0, 2, 1).view(np.uint32), r["scores"].view(np.uint32)), c
        assert np.array_equal(bb.origins[:T].cpu().numpy().transpose(0, 2, 1), r["prev"]), c
        assert np.array_equal(bb.tokens[:T + 1].cpu().numpy().transpose(0, 2, 1), r["next"]), c
        hyps, scores, attn = bb.finish()
        ends = np.cumsum(r["n_finished"])[:-1]
        lens, tok, att = iter(r["hyp_len"].tolist()), 0, 0
        for j, fs in enumerate(np.split(r["fin_scores"], ends)):
            assert np.array_equal(np.array(scores[j], np.float32).view(np.uint32), fs.view(np.uint32)), (c, j)
            for n in range(n_best):
                L = next(lens)
                assert hyps[j][n] == r["hyp_tok"][tok:tok + L].tolist(), (c, j, n)
                assert np.array_equal(attn[j][n].numpy().view(np.uint32), r["hyp_attn"][att:att + L].view(np.uint32)), (c, j, n)
                tok, att = tok + L, att + L


def test_sentence_alone_in_batch_and_streams(N):
    K, V = 5, 10_004
    x, eos, last, scores, n_fin, eos_top = _inputs(7, K, V, 5, True)
    ref = {}
    for normalize in (0, 1):
        st = Step(N, torch.from_numpy(x).cuda(), 7, K, V, eos, scores, last, n_fin, eos_top)
        N.check(st(normalize, 0))
        ref[normalize] = st.result()
    for b in (0, 3, 6):
        rows = np.arange(K) * 7 + b
        for normalize in (0, 1):
            st = Step(N, torch.from_numpy(x[rows]).cuda(), 1, K, V, eos, scores[rows], last[rows], n_fin[b:b + 1], eos_top[b:b + 1])
            N.check(st(normalize, 0))
            got, want = st.result(), ref[normalize]
            assert _same_float(got[0], want[0][rows])
            assert np.array_equal(got[1], want[1][rows]) and np.array_equal(got[3], want[3][rows])
            assert np.array_equal(got[2], want[1][rows])                  # alone, flat_origin is the origin
            assert got[4][0] == want[4][b] and got[5][0] == want[5][b]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = Step(N, torch.from_numpy(x).cuda(), 7, K, V, eos, scores, last, n_fin, eos_top)
    c = Step(N, torch.from_numpy(x).cuda(), 7, K, V, eos, scores, last, n_fin, eos_top)
    torch.cuda.synchronize()
    N.check(a(1, 0, s1.cuda_stream))
    N.check(c(1, 0, s2.cuda_stream))
    torch.cuda.synchronize()
    _check(a.result(), ref[1])
    _check(c.result(), ref[1])


def test_graph_replay_and_no_sync(N):
    from quantized_distillation_b200.beam import BatchBeam
    K, B, V = 5, 30, 10_004
    x, eos, last, scores, n_fin, eos_top = _inputs(B, K, V, 9, True)
    xd = torch.from_numpy(x).cuda()
    eager = Step(N, xd, B, K, V, eos, scores, last, n_fin, eos_top)
    N.check(eager(1, 0))
    g_step = Step(N, xd, B, K, V, eos, scores, last, n_fin, eos_top)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            N.check(g_step(1, 0, side.cuda_stream))
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    torch.cuda.synchronize()
    _check(g_step.result(), eager.result())

    bb = BatchBeam(B, K, 2, 2, eos, 1, 4, "cuda")
    attn = torch.rand(K * B, 9, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for normalized in (False, True, False):
            bb.advance(xd, attn, normalized)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert bb.steps == 3


def test_c_abi_refusals(N):
    K, B, V = 4, 3, 50
    x, eos, last, scores, n_fin, eos_top = _inputs(B, K, V, 1, False)
    st = Step(N, torch.from_numpy(x).cuda(), B, K, V, eos, scores, last, n_fin, eos_top)
    lib, p = N.lib(), N.ptr
    need = int(lib.qd_beam_workspace_bytes(B, K))
    assert need == B * K * K * 8 and lib.qd_beam_workspace_bytes(0, K) == 0

    def call(**kw):
        a = dict(out=p(st.out), normalize=1, batch=B, beam=K, V=V, eos=eos, first=0, scores=p(st.scores), last=p(st.last),
                 origin=p(st.origin), flat=p(st.flat), tokens=p(st.tokens), n_fin=p(st.n_fin), eos_top=p(st.eos_top),
                 ws=p(st.ws), ws_bytes=need)
        a.update(kw)
        return lib.qd_beam_step(*a.values(), N.stream_ptr())

    before = st.result()
    bad = [dict(beam=0), dict(beam=17), dict(batch=-1), dict(V=K - 1), dict(eos=-1), dict(eos=V), dict(normalize=2),
           dict(out=None), dict(scores=None), dict(last=None), dict(origin=None), dict(flat=None), dict(tokens=None),
           dict(n_fin=None), dict(eos_top=None), dict(out=p(st.out) + 2), dict(scores=p(st.scores) + 2),
           dict(last=p(st.last) + 4), dict(origin=p(st.origin) + 4), dict(flat=p(st.flat) + 4), dict(tokens=p(st.tokens) + 4),
           dict(n_fin=p(st.n_fin) + 2), dict(tokens=p(st.origin)), dict(flat=p(st.tokens) + 8), dict(scores=p(st.out) + 64),
           dict(origin=p(st.last)), dict(ws=p(st.out)), dict(n_fin=p(st.scores)), dict(eos_top=p(st.n_fin) + 1),
           dict(ws=p(st.origin)), dict(batch=1 << 62), dict(out=p(st.out) + 2, ws=None), dict(scores=None, n_fin=p(st.n_fin) + 2),
           dict(last=p(st.last) + 4, tokens=p(st.origin))]
    for kw in bad:
        assert call(**kw) == N.QD_ERR_INVALID_ARG, kw
    # a batch past the workspace query's range (which then returns 0) still needs a workspace
    assert lib.qd_beam_workspace_bytes(1 << 53, 1) == 0
    for kw in (dict(ws=None), dict(ws_bytes=need - 1), dict(ws=p(st.ws) + 8), dict(ws=None, origin=p(st.last)),
               dict(ws=p(st.ws) + 8, flat=p(st.tokens)), dict(ws=None, batch=1 << 53, beam=1, V=1, eos=0)):
        assert call(**kw) == N.QD_ERR_WORKSPACE, kw
    torch.cuda.synchronize()
    for g, w in zip(st.result(), before):
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8))
    assert call(batch=0, out=None, scores=None, ws=None) == N.QD_OK
    assert call() == N.QD_OK


def test_python_refusals(N):
    from quantized_distillation_b200.beam import BatchBeam, beam_search, _generator_linear
    for kw in (dict(beam=0), dict(beam=17), dict(batch=-1), dict(n_best=0), dict(max_len=0), dict(device="cpu")):
        a = dict(batch=2, beam=3, n_best=1, bos=2, eos=3, pad=1, max_len=2, device="cuda")
        a.update(kw)
        with pytest.raises(ValueError):
            BatchBeam(**a)
    bb = BatchBeam(2, 3, 1, 2, 3, 1, 1, "cuda")
    at = torch.rand(6, 4, device="cuda")
    for out in (torch.randn(6, 10, device="cuda").double(), torch.randn(5, 10, device="cuda"), torch.randn(6, 10)):
        with pytest.raises(ValueError):
            bb.advance(out, at, True)
    with pytest.raises(ValueError):
        bb.advance(torch.randn(6, 2, device="cuda"), at, True)          # V < beam
    bb.advance(torch.randn(6, 10, device="cuda"), at, True)
    with pytest.raises(ValueError):
        bb.advance(torch.randn(6, 10, device="cuda"), at, True)          # past max_len
    for gen in (nn.Sequential(nn.Linear(4, 9), nn.Softmax(-1)), nn.Linear(4, 9), nn.Sequential(nn.Linear(4, 9))):
        with pytest.raises(ValueError):
            _generator_linear(gen)
    model = _Model(0)
    with pytest.raises(ValueError):
        beam_search(model, *_src(0), bos=2, eos=3, pad=1, global_scorer=object())
    model.decoder.copy_attn = True
    with pytest.raises(ValueError):
        beam_search(model, *_src(0), bos=2, eos=3, pad=1)


# ---- a small onmt-protocol model: embeddings, LSTM encoder, input-feeding decoder with general attention ----------
E, H, V_MODEL, LAYERS = 16, 32, 61, 2
BOS, EOS, PAD = 2, 3, 1


class _State:
    """onmt's RNNDecoderState (Models.py:452-500): hidden (h, c) [layers, N, H] and input_feed [1, N, H]."""

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
        self.embeddings = nn.Embedding(V_MODEL, E, padding_idx=PAD)
        self.rnn = nn.LSTM(E, H, LAYERS)

    def forward(self, src, lengths):
        packed = nn.utils.rnn.pack_padded_sequence(self.embeddings(src), lengths.tolist())
        out, hidden = self.rnn(packed)
        return hidden, nn.utils.rnn.pad_packed_sequence(out)[0]


class _Decoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.embeddings = nn.Embedding(V_MODEL, E, padding_idx=PAD)
        self.cells = nn.ModuleList([nn.LSTMCell(E + H if i == 0 else H, H) for i in range(LAYERS)])
        self.linear_in = nn.Linear(H, H, bias=False)
        self.linear_out = nn.Linear(2 * H, H, bias=False)

    def init_decoder_state(self, src, context, enc_hidden):
        return _State(enc_hidden, context.new_zeros(1, context.shape[1], H))

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
            # general global attention (onmt GlobalAttention, attn_type "general")
            score = torch.bmm(context.transpose(0, 1), self.linear_in(x).unsqueeze(2)).squeeze(2)       # [N, S]
            a = F.softmax(score, -1)
            ctx = torch.bmm(a.unsqueeze(1), context.transpose(0, 1)).squeeze(1)
            feed = torch.tanh(self.linear_out(torch.cat([ctx, x], 1)))
            h, c = torch.stack(hs), torch.stack(cs)
            outs.append(feed), attns.append(a)
        state.hidden, state.input_feed = (h, c), feed.unsqueeze(0)
        return torch.stack(outs), state, {"std": torch.stack(attns)}


class _Model(nn.Module):
    def __init__(self, seed):
        torch.manual_seed(seed)
        super().__init__()
        self.encoder, self.decoder = _Encoder(), _Decoder()
        self.generator = nn.Sequential(nn.Linear(H, V_MODEL), nn.LogSoftmax(dim=-1))
        with torch.no_grad():
            self.generator[0].bias[EOS] += 2.5            # EOS often enough that sentences finish
        self.cuda().eval()


def _src(seed, B=6, S=7):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.sort(torch.randint(1, S + 1, (B,), generator=g), descending=True)[0]
    lengths[0] = S
    src = torch.randint(4, V_MODEL, (S, B), generator=g)
    for b, L in enumerate(lengths.tolist()):
        src[L:, b] = PAD
    return src.cuda(), lengths


def _oracle_translate(N, model, src, lengths, K, n_best, max_len):
    """The oracle's per-sentence translateBatch on the same model: the decoder on the GPU, the Beams in NumPy, each
    sentence's beam_update after its advance."""
    B = src.shape[1]
    with torch.no_grad():
        enc, context = model.encoder(src, lengths)
        state = model.decoder.init_decoder_state(src, context, enc)
        context = context.repeat(1, K, 1)
        state.repeat_beam_size_times(K)

        def step(inp):
            nonlocal state
            x = torch.from_numpy(inp).cuda().view(1, -1, 1)
            out, state, attn = model.decoder(x, context, state)
            logits = model.generator[0](out.squeeze(0)).contiguous()
            return O.log_probs(logits.cpu().numpy(), _lse(N, logits)), attn["std"].squeeze(0).cpu().numpy()

        def update(j, positions):
            state.beam_update(j, torch.from_numpy(positions).cuda(), K)

        hyps, scores, attn, _ = O.translate_batch(step, B, K, n_best, max_len, BOS, EOS, PAD, update)
    return hyps, scores, attn


def _compare(got, want):
    for (gh, gs, ga), (wh, ws, wa) in zip(zip(*got), zip(*want)):
        assert gh == wh
        assert np.array_equal(np.array(gs, np.float32).view(np.uint32), np.array(ws, np.float32).view(np.uint32))
        for x, y in zip(ga, wa):
            assert np.array_equal(x.numpy().view(np.uint32), np.asarray(y, np.float32).view(np.uint32))


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("K,n_best,max_len", [(5, 1, 12), (1, 1, 10), (4, 3, 8), (16, 2, 9)])
def test_beam_search_matches_oracle_translate_batch(N, K, n_best, max_len, packed):
    from quantized_distillation_b200 import codec
    from quantized_distillation_b200.beam import beam_search
    model = _Model(0)
    if packed:
        pm = codec.pack_model(model, 4, 256, quantize_first_and_last_layer=True)
        model = _Model(1)
        names = codec.attach_packed_(pm, model, embeddings=True, recurrent=True)
        assert isinstance(model.generator[0], codec.PackedLinear) and isinstance(model.encoder.rnn, codec.PackedLSTM), names
        model.eval()
    src, lengths = _src(K)
    got = beam_search(model, src, lengths, K, n_best, max_len, bos=BOS, eos=EOS, pad=PAD)
    want = _oracle_translate(N, model, src, lengths, K, n_best, max_len)
    _compare(got, want)
    assert len(got[0]) == src.shape[1] and all(len(h) == n_best for h in got[0])
