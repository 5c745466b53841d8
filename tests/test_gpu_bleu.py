"""BLEU on the GPU: qd_bleu_stats and qd_bleu_fold against the oracle (oracle/bleu_oracle.py, itself pinned on the
reference's multi-bleu.perl by tests/golden/reference_bleu.json) on every fixture and on random corpora (N 0 .. 3,000,
lengths 0 .. 5,000 across the shared-memory staging limit, 0-4 references, offsets not starting at 0); the drop-in
get_bleu_moses returning the fixtures' perl bytes; BatchBeam.finish_on_device against finish() on the reference's Beam
replays and on random histories (K 1-16, n_best 1-16, the `minimum` quirk); bleu_model end to end on a small
onmt-protocol model against the oracle's score of beam_search's strings, float32 and attached packed; batching,
streams, graph replay, no synchronisation and the C ABI's refusals.

All histories here are NaN-free: Python's sort gives NaN scores no defined order, so finish() and the kernel's stated
NaN rule cannot be compared on them."""
import base64
import importlib.util
import json
import os
import random

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import bleu_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "reference_bleu.json")))["cases"]
STAGE_WORDS = 2048                                  # kStageWords of qd_bleu.cu: words staged per sentence


@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native
    return _native


def _d(s):
    return base64.b64decode(s)


class Corpus:
    """Hypotheses and references as int32 word ids in the C ABI's CSR layout, on the device.  hyps[s]: list of ids;
    refs[s]: list of id lists.  `lead` junk words precede each word array, so offsets start past 0."""

    def __init__(self, hyps, refs, lead=0, shuffle_refs=False, seed=0):
        g = random.Random(seed)
        hw, ho = [-5] * lead, [lead]
        for h in hyps:
            hw += h
            ho.append(len(hw))
        rw, ro, first, count = [-7] * lead, [lead], [0] * len(refs), []
        order = list(range(len(refs)))
        if shuffle_refs:
            g.shuffle(order)                    # a sentence's spans are consecutive, sentences in any order
        for s in order:
            first[s] = len(ro) - 1
            for r in refs[s]:
                rw += r
                ro.append(len(rw))
        count = [len(r) for r in refs]
        self.n = len(hyps)
        t = lambda v, dt: torch.tensor(v, dtype=dt, device="cuda")
        self.hw, self.ho, self.rw, self.ro = t(hw, torch.int32), t(ho, torch.int64), t(rw, torch.int32), t(ro, torch.int64)
        self.first, self.count = t(first, torch.int64), t(count, torch.int64)

    def stats(self, N, out=None, stream=None):
        out = out if out is not None else torch.full((self.n, 10), -3, dtype=torch.int64, device="cuda")
        N.check(N.lib().qd_bleu_stats(N.ptr(self.hw), self.hw.numel(), N.ptr(self.ho), self.n, N.ptr(self.rw),
                                      self.rw.numel(), N.ptr(self.ro), self.ro.numel() - 1, N.ptr(self.first),
                                      N.ptr(self.count), N.ptr(out), stream if stream is not None else N.stream_ptr()))
        return out


def _fold(N, stats):
    out = torch.full((10,), -3, dtype=torch.int64, device="cuda")
    N.check(N.lib().qd_bleu_fold(N.ptr(stats), stats.shape[0], N.ptr(out), N.stream_ptr()))
    return out.tolist()


def _fixture_words(c):
    table = {}
    ids = lambda ws: [table.setdefault(w, len(table)) for w in ws]
    refs = []
    for _, b in c["files"]:
        for s, line in enumerate(O.perl_lines(_d(b))):
            if s == len(refs):
                refs.append([])
            refs[s].append(O.perl_words(line, c["lowercase"]))
    hyps = [O.perl_words(line, c["lowercase"]) for line in O.perl_lines(_d(c["stdin"]))]
    refs += [[] for _ in range(len(hyps) - len(refs))]
    return [ids(h) for h in hyps], [[ids(r) for r in rs] for rs in refs[:len(hyps)]], hyps, refs


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_stats_match_oracle_on_fixtures(N, c):
    hyps, refs, hw, rw = _fixture_words(c)
    got = Corpus(hyps, refs, lead=3).stats(N)
    want = O.corpus_stats(hw, rw)
    assert got.cpu().tolist() == want
    assert _fold(N, got) == O.fold(want)
    from quantized_distillation_b200 import bleu
    assert bleu.multi_bleu(_d(c["stdin"]), [_d(b) for _, b in c["files"]], c["lowercase"]) == _d(c["stdout"])


def _random_corpus(seed, n, lengths, vocab=6, max_refs=4):
    g = random.Random(seed)
    hyps = [[g.randrange(vocab) for _ in range(lengths(g))] for _ in range(n)]
    refs = [[[g.randrange(vocab) for _ in range(lengths(g))] for _ in range(g.randint(0, max_refs))] for _ in range(n)]
    return hyps, refs


@pytest.mark.parametrize("n", [0, 1, 7, 3000])
def test_stats_random_corpora(N, n):
    for seed, (lead, vocab) in enumerate([(0, 3), (5, 8), (1, 40)]):
        hyps, refs = _random_corpus(seed * 100 + n, n, lambda g: g.choice([0, 1, 2, 3, 4, g.randint(0, 40)]), vocab)
        c = Corpus(hyps, refs, lead=lead, shuffle_refs=seed == 1, seed=seed)
        got = c.stats(N)
        want = O.corpus_stats(hyps, refs)
        assert got.cpu().tolist() == want
        assert _fold(N, got) == O.fold(want)


def test_stats_long_sentences_straddle_staging(N):
    """Sentences whose hypothesis plus references are just below, at and above the staged words, and up to 5,000."""
    g = random.Random(7)
    hyps, refs = [], []
    for L, ref_lens in [(0, [0]), (0, [5000]), (STAGE_WORDS, []), (STAGE_WORDS - 10, [10]), (STAGE_WORDS - 10, [11]),
                        (1000, [500, 548]), (1000, [500, 549]), (5000, [4990]), (3000, [100, 2000, 2999, 3001]),
                        (4999, [1]), (1, [4999])]:
        voc = g.choice([2, 5, 50])
        hyps.append([g.randrange(voc) for _ in range(L)])
        refs.append([[g.randrange(voc) for _ in range(r)] for r in ref_lens])
    hyps.append([9] * 3000)                                  # one token repeated
    refs.append([[9] * 1200, [9, 8] * 700])
    got = Corpus(hyps, refs, lead=11).stats(N)
    assert got.cpu().tolist() == O.corpus_stats(hyps, refs)


def test_drop_in_returns_fixture_bytes(N, tmp_path):
    from quantized_distillation_b200 import bleu
    for c in CASES:
        if not c["lowercase"]:
            continue
        if c["mode"] == "list":
            got = bleu.get_bleu_moses(c["hypotheses"], c["reference"])
        else:
            d = tmp_path / c["name"]
            d.mkdir()
            stem = str(d / "ref")
            for suffix, data in c["files"]:
                (d / ("ref" + suffix)).write_bytes(_d(data))
            (d / "hyp.txt").write_bytes(_d(c["stdin"]))
            got = bleu.get_bleu_moses(str(d / "hyp.txt"), stem, file_input=True)
        assert got == _d(c["stdout"]), c["name"]


def test_corpus_bleu_and_bleu_stats(N):
    from quantized_distillation_b200 import bleu
    c = next(c for c in CASES if c["name"] == "random_mixed_case_lc1")
    hyps, refs = c["hypotheses"], c["reference"]
    line = O.multi_bleu("\n".join(h for h in hyps).encode() + b"\n", ["".join(r + "\n" for r in refs).encode()], True)[0]
    assert line.startswith(b"BLEU = %.2f," % bleu.corpus_bleu(hyps, refs))
    with pytest.raises(ValueError):
        bleu.corpus_bleu(hyps[:-1], refs)
    # batches in any order, by sentence index, give the corpus totals
    R = bleu.References(refs)
    st = bleu.BleuStats(R)
    perm = list(range(len(hyps)))
    random.Random(3).shuffle(perm)
    for lo in range(0, len(perm), 37):
        idx = perm[lo:lo + 37]
        st.add([hyps[i] for i in idx], idx)
    whole = bleu.BleuStats(bleu.References(refs))
    whole.add(hyps)
    assert st.totals() == whole.totals()
    assert bleu.format_line(st.totals()) == line


# ---- determinism, streams, capture, refusals ---------------------------------------------------------------------

def test_sentence_alone_in_batch_streams_and_graph(N):
    hyps, refs = _random_corpus(11, 64, lambda g: g.randint(0, 60), 5)
    hyps[9] = [1, 2] * 1500                                   # one sentence past the staging limit
    c = Corpus(hyps, refs)
    ref = c.stats(N).cpu()
    for s in (0, 9, 31, 63):
        for pos, n in ((0, 1), (2, 3), (4, 5)):
            hs = [hyps[(s + k) % 64] for k in range(-pos, n - pos)]
            rs = [refs[(s + k) % 64] for k in range(-pos, n - pos)]
            assert Corpus(hs, rs, lead=pos).stats(N)[pos].cpu().equal(ref[s])
    s1 = torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    out = torch.full((64, 10), -3, dtype=torch.int64, device="cuda")
    c.stats(N, out, s1.cuda_stream)
    torch.cuda.current_stream().wait_stream(s1)
    assert out.cpu().equal(ref)
    g_out = torch.full((64, 10), -3, dtype=torch.int64, device="cuda")
    totals = torch.full((10,), -3, dtype=torch.int64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            c.stats(N, g_out, side.cuda_stream)
            N.check(N.lib().qd_bleu_fold(N.ptr(g_out), 64, N.ptr(totals), side.cuda_stream))
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    torch.cuda.synchronize()
    assert g_out.cpu().equal(ref) and totals.tolist() == ref.sum(0).tolist()
    torch.cuda.set_sync_debug_mode("error")
    try:
        c.stats(N, g_out)
        N.check(N.lib().qd_bleu_fold(N.ptr(g_out), 64, N.ptr(totals), N.stream_ptr()))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _fold(N, g_out) == ref.sum(0).tolist()


def test_bleu_c_abi_refusals(N):
    hyps, refs = _random_corpus(5, 6, lambda g: g.randint(0, 9), 4)
    c = Corpus(hyps, refs)
    out = torch.full((6, 10), -3, dtype=torch.int64, device="cuda")
    lib, p = N.lib(), N.ptr

    def call(**kw):
        a = dict(hw=p(c.hw), nhw=c.hw.numel(), ho=p(c.ho), n=6, rw=p(c.rw), nrw=c.rw.numel(), ro=p(c.ro), nr=c.ro.numel() - 1,
                 first=p(c.first), count=p(c.count), out=p(out))
        a.update(kw)
        return lib.qd_bleu_stats(*a.values(), N.stream_ptr())

    bad = [dict(n=-1), dict(nhw=-1), dict(nrw=-1), dict(nr=-1), dict(ho=None), dict(ro=None), dict(first=None),
           dict(count=None), dict(out=None), dict(hw=None), dict(rw=None), dict(hw=p(c.hw) + 2), dict(ho=p(c.ho) + 4),
           dict(out=p(out) + 4), dict(out=p(c.ho)), dict(out=p(c.hw)), dict(out=p(c.first) - 8), dict(n=1 << 62)]
    for kw in bad:
        assert call(**kw) == N.QD_ERR_INVALID_ARG, kw
    totals = torch.full((10,), -3, dtype=torch.int64, device="cuda")
    for kw in (dict(n=-1), dict(stats=None), dict(totals=None), dict(totals=p(out) + 8), dict(totals=p(totals) + 4)):
        a = dict(stats=p(out), n=6, totals=p(totals))
        a.update(kw)
        assert lib.qd_bleu_fold(*a.values(), N.stream_ptr()) == N.QD_ERR_INVALID_ARG, kw
    torch.cuda.synchronize()
    assert (out == -3).all() and (totals == -3).all()
    assert call(n=0, ho=None, out=None) == N.QD_OK
    assert call() == N.QD_OK
    assert out.cpu().tolist() == O.corpus_stats(hyps, refs)
    assert lib.qd_bleu_fold(None, 0, p(totals), N.stream_ptr()) == N.QD_OK
    assert totals.tolist() == [0] * 10
    # device spans out of range are read as empty, not followed: a clamped offset and a span past n_refs
    bad_ho = c.ho.clone()
    bad_ho[3] = 10 ** 9
    bad_first = c.first.clone()
    bad_first[1] = 10 ** 6
    o2 = torch.empty_like(out)
    N.check(lib.qd_bleu_stats(p(c.hw), c.hw.numel(), p(bad_ho), 6, p(c.rw), c.rw.numel(), p(c.ro), c.ro.numel() - 1,
                              p(bad_first), p(c.count), p(o2), N.stream_ptr()))
    assert o2[1, 1].item() == 9999
    assert o2[2, 0].item() == c.hw.numel() - c.ho[2].item() and o2[3, 0].item() == 0


# ---- the device finish -------------------------------------------------------------------------------------------

def _same_f32(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _compare_finish(bb):
    hyps, scores, attn = bb.finish()
    d = bb.finish_on_device()
    toks, lens, sc, arg = (t.cpu() for t in d)
    T = bb.steps
    for b in range(bb.B):
        assert _same_f32(sc[b].numpy(), scores[b][:bb.n_best]), b
        for j in range(bb.n_best):
            L = int(lens[b, j])
            assert L == len(hyps[b][j]) and toks[b, j, :L].tolist() == hyps[b][j], (b, j)
            assert (toks[b, j, L:] == -1).all() and (arg[b, j, L:] == -1).all()
            if L:
                assert arg[b, j, :L].tolist() == attn[b][j].max(1)[1].tolist(), (b, j)
    assert toks.shape == (bb.B, bb.n_best, T)


def _gen():
    spec = importlib.util.spec_from_file_location("make_golden_beam", os.path.join(HERE, "golden", "make_golden_beam.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_finish_on_device_replays_reference(N):
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
        _compare_finish(bb)


def _random_beam(K, B, n_best, T, S, eos_rate, seed, ties=False):
    from quantized_distillation_b200.beam import BatchBeam
    g = torch.Generator().manual_seed(seed)
    V, eos = 7, 3
    bb = BatchBeam(B, K, n_best, 2, eos, 1, max(T, 1), "cuda")
    tok = torch.randint(0, V, (T + 1, K, B), generator=g)
    tok[1:][torch.rand(T, K, B, generator=g) < eos_rate] = eos
    sc = -torch.rand(T, K, B, generator=g) * 10
    if ties:                                            # repeated scores, and -0.0 next to +0.0
        sc = (sc * 2).round() / 2
        sc[torch.rand(T, K, B, generator=g) < 0.2] = 0.0
        sc[torch.rand(T, K, B, generator=g) < 0.2] = -0.0
    at = torch.rand(T, K, B, S, generator=g)
    if ties:
        at = (at * 3).floor()
    bb.tokens[:T + 1] = tok.cuda()
    bb.origins[:T] = torch.randint(0, K, (T, K, B), generator=g).cuda()
    bb.step_scores[:T] = sc.cuda()
    if T:
        bb.attn = torch.zeros(max(T, 1), K, B, S, device="cuda")
        bb.attn[:T] = at.cuda()
    bb.steps = T
    return bb


@pytest.mark.parametrize("K", [1, 2, 5, 16])
def test_finish_on_device_random_histories(N, K):
    for i, (n_best, T, eos_rate, ties) in enumerate([(1, 6, 0.3, False), (3, 9, 0.05, False), (16, 7, 0.1, True),
                                                     (K, 12, 0.5, True), (2, 1, 0.0, False), (5, 0, 0.0, False),
                                                     (16, 40, 0.02, False), (1, 20, 0.9, True)]):
        B = [1, 3, 7, 30][i % 4]
        _compare_finish(_random_beam(K, B, n_best, T, 1 + 5 * i, eos_rate, 1000 * K + i, ties))


def test_finish_on_device_refusals_and_capture(N):
    from quantized_distillation_b200.beam import BatchBeam
    with pytest.raises(ValueError):
        BatchBeam(2, 3, 17, 2, 3, 1, 4, "cuda").finish_on_device()
    bb = _random_beam(5, 30, 2, 10, 9, 0.2, 5)
    want = [t.cpu() for t in bb.finish_on_device()]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        bb.finish_on_device()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    outs = [torch.full_like(w.cuda(), -9) for w in want]
    lib, p = N.lib(), N.ptr

    def call(stream, **kw):
        a = dict(tokens=p(bb.tokens), origins=p(bb.origins), scores=p(bb.step_scores), attn=p(bb.attn), T=10, B=30, K=5,
                 S=9, eos=bb.eos, n_best=2, ht=p(outs[0]), hl=p(outs[1]), hs=p(outs[2]), ha=p(outs[3]))
        a.update(kw)
        return lib.qd_beam_finish(*a.values(), stream)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            N.check(call(side.cuda_stream))
    torch.cuda.current_stream().wait_stream(side)
    for o in outs:
        o.fill_(-9)
    torch.cuda.synchronize()
    bad = [dict(K=0), dict(K=17), dict(n_best=0), dict(n_best=17), dict(B=-1), dict(T=-1), dict(S=-1), dict(S=0),
           dict(tokens=None), dict(origins=None), dict(scores=None), dict(attn=None), dict(ht=None), dict(hl=None),
           dict(hs=None), dict(ha=None), dict(ht=p(outs[0]) + 4), dict(hs=p(outs[2]) + 2), dict(ht=p(bb.tokens)),
           dict(ha=p(outs[0]) + 8), dict(hl=p(bb.origins) + 8)]
    for kw in bad:
        assert call(N.stream_ptr(), **kw) == N.QD_ERR_INVALID_ARG, kw
    torch.cuda.synchronize()
    assert all((o == -9).all() for o in outs)
    graph.replay()
    torch.cuda.synchronize()
    for o, w in zip(outs, want):
        assert o.cpu().view(torch.int32 if o.dtype == torch.float32 else o.dtype).equal(
            w.view(torch.int32 if w.dtype == torch.float32 else w.dtype))


# ---- end to end: a small onmt-protocol model (the shape of test_gpu_beam.py's) -----------------------------------
E, H, V_MODEL, LAYERS = 16, 32, 61, 2
UNK, PAD, BOS, EOS = 0, 1, 2, 3


class _State:
    def __init__(self, hidden, input_feed):
        self.hidden, self.input_feed = hidden, input_feed

    @property
    def _all(self):
        return self.hidden + (self.input_feed,)

    def repeat_beam_size_times(self, k):
        v = [e.repeat(1, k, 1) for e in self._all]
        self.hidden, self.input_feed = tuple(v[:-1]), v[-1]


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
            score = torch.bmm(context.transpose(0, 1), self.linear_in(x).unsqueeze(2)).squeeze(2)
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
            self.generator[0].weight *= 8                # sharper scores: hypotheses of more than one word
        self.cuda().eval()


SPECIALS = ["<unk>", "<blank>", "<s>", "</s>"]
TGT_ITOS = SPECIALS + [("W" if i % 3 == 0 else "w") + str(i % 23) for i in range(4, V_MODEL)]
SRC_ITOS = SPECIALS + ["s%d" % (i % 17) if i % 5 else "W%d" % (i % 23) for i in range(4, V_MODEL)]


def _src(seed, B, S):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.sort(torch.randint(1, S + 1, (B,), generator=g), descending=True)[0]
    lengths[0] = S
    src = torch.randint(4, V_MODEL, (S, B), generator=g)
    for b, L in enumerate(lengths.tolist()):
        src[L:, b] = PAD
    return src.cuda(), lengths


def _build_target_tokens(pred, src_col, attn, replace_unk, tgt_itos):
    """Translator.buildTargetTokens (Translator.py:43-60) without copy vocabularies."""
    tokens = []
    for tok in pred:
        tokens.append(tgt_itos[tok])
        if tokens[-1] == "</s>":
            tokens = tokens[:-1]
            break
    if replace_unk:
        for i in range(len(tokens)):
            if tokens[i] == tgt_itos[UNK]:
                tokens[i] = SRC_ITOS[src_col[int(attn[i].max(0)[1])]]
    return tokens


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("replace_unk", [True, False])
def test_bleu_model_matches_oracle_of_beam_search_strings(N, replace_unk, packed):
    from quantized_distillation_b200 import bleu, codec
    from quantized_distillation_b200.beam import beam_search
    model = _Model(0)
    if packed:
        pm = codec.pack_model(model, 4, 256, quantize_first_and_last_layer=True)
        model = _Model(1)
        codec.attach_packed_(pm, model, embeddings=True, recurrent=True)
        assert isinstance(model.generator[0], codec.PackedLinear)
        model.eval()
    batches = [_src(1, 6, 7), _src(2, 5, 9)]
    perm = [9, 6, 10, 7, 8]                              # the second batch's sentences, out of order
    indices = [list(range(6)), perm]
    searched = [beam_search(model, src, lengths, 5, 1, 12, bos=BOS, eos=EOS, pad=PAD) for src, lengths in batches]
    # buildTargetTokens compares words: give the model's most frequent token the UNK word, so replace_unk has work
    counts = np.bincount([t for hyps, _, _ in searched for h in hyps for t in h[0] if t != EOS], minlength=V_MODEL)
    tgt_itos = list(TGT_ITOS)
    tgt_itos[int(counts.argmax())] = tgt_itos[UNK]
    lines = [None] * 11
    for (src, _), idx, (hyps, _, attn) in zip(batches, indices, searched):
        for b, s in enumerate(idx):
            lines[s] = " ".join(_build_target_tokens(hyps[b][0], src[:, b].tolist(), attn[b][0], replace_unk, tgt_itos))
    assert counts.max() > 0 and (not any("<unk>" in ln.split() for ln in lines)) == replace_unk
    # references that share some n-grams with the hypotheses, so that every precision can be nonzero
    g = random.Random(4)
    refs = []
    for ln in lines:
        w = [x if g.random() < 0.7 else g.choice(TGT_ITOS[4:]) for x in ln.split()][:g.randint(0, 14)]
        refs.append(" ".join(w + [g.choice(SRC_ITOS[4:]) for _ in range(g.randint(0, 3))]))
    want = O.multi_bleu("".join(ln + "\n" for ln in lines).encode(), ["".join(r + "\n" for r in refs).encode()], True)[0]
    got = bleu.bleu_model(model, [(s, l, i) for (s, l), i in zip(batches, indices)], refs, src_vocab=SRC_ITOS,
                          tgt_vocab=tgt_itos, replace_unk=replace_unk, beam_size=5, max_sent_length=12, bos=BOS, eos=EOS,
                          pad=PAD, unk=UNK)
    assert got == want and got.startswith(b"BLEU = ")
    # the same through the string drop-in, and the default consecutive indices
    assert bleu.get_bleu_moses(lines, refs) == O.get_bleu_moses(lines, refs)
    got1 = bleu.bleu_model(model, [batches[0]], refs[:6], src_vocab=SRC_ITOS, tgt_vocab=tgt_itos, replace_unk=replace_unk,
                           beam_size=5, max_sent_length=12, bos=BOS, eos=EOS, pad=PAD, unk=UNK)
    assert got1 == O.multi_bleu("".join(ln + "\n" for ln in lines[:6]).encode(),
                                ["".join(r + "\n" for r in refs[:6]).encode()], True)[0]
