"""LSTM layers run from their packed codes: qd_packed_lstm_cell against its stated contract (preactivations from
qd_packed_linear plus float32 adds, activations carried in float64) and the float64 oracle over code widths, uniform and
non-uniform weights at different widths, buckets straddling gate rows, odd sizes up to the NMT shapes, every row tile
and unaligned strides; determinism (alone / in a batch, four streams, CUDA-graph replay of a whole PackedLSTM);
qd_packed_lstm_layer against step-by-step cells and the oracle; PackedLSTM / PackedLSTMCell against cuDNN on the decoded
weights and, above 64 rows, equal to unpack_ + torch; refusals at the C ABI and in the modules; and
attach_packed_(..., recurrent=True) on an NMT-shaped model (exact memory account), on the Huffman route and on the
recurrent modules it must leave to unpack_."""
import gc
import threading

import numpy as np
import pytest
import torch

from oracle import packed_lstm_oracle as O

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -23


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    return N, codec


class W:
    """One packed [rows, cols] weight on the device: random codes, scales, points; q as qd_unpack_dequant_* decodes it."""

    def __init__(self, N, rows, cols, bits, s, k, bucket, seed, shift=0):
        g = torch.Generator(device="cuda").manual_seed(seed)
        n = rows * cols
        self.rows, self.cols, self.bits, self.s, self.k, self.bucket = rows, cols, bits, s, k, bucket
        codes = torch.randint(0, s or k, (n,), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
        buf = torch.zeros((n * bits + 7) // 8 + shift, dtype=torch.uint8, device="cuda")
        self.packed = buf[shift:]
        N.check(N.lib().qd_pack_indices(N.ptr(codes), N.ptr(self.packed), n, bits, N.stream_ptr()))
        nb = N.geometry(n, bucket or 0)[0]
        scale = 1.0 / max(cols, 1) ** 0.5
        self.alpha = (torch.rand(nb, generator=g, device="cuda") + 0.5) * 2 * scale
        self.beta = -self.alpha / 2 + torch.randn(nb, generator=g, device="cuda") * 0.1 * scale
        self.points = None if k is None else torch.sort(torch.rand(k, generator=g, device="cuda")).values
        self.q = torch.empty(rows, cols, device="cuda")
        if k is None:
            N.check(N.lib().qd_unpack_dequant_uniform(N.ptr(self.packed), bits, N.ptr(self.alpha), N.ptr(self.beta), N.ptr(self.q), n,
                                                      bucket or 0, s, N.stream_ptr()))
        else:
            N.check(N.lib().qd_unpack_dequant_nonuniform(N.ptr(self.packed), bits, N.ptr(self.points), k, N.ptr(self.alpha),
                                                         N.ptr(self.beta), N.ptr(self.q), n, bucket or 0, N.stream_ptr()))
        from quantized_distillation_b200.codec import _PACKED_TENSOR
        self.desc = np.zeros(1, _PACKED_TENSOR)
        self.desc[0] = (self.packed.data_ptr(), self.alpha.data_ptr(), self.beta.data_ptr(),
                        0 if self.points is None else self.points.data_ptr(), 0, n, bits, 0 if k is None else k)

    def entry(self, codec, name="w"):
        return codec.PackedEntry(name, (self.rows, self.cols), bits=self.bits, packed=self.packed, alpha=self.alpha, beta=self.beta,
                                 points=self.points)

    def linear(self, N, x, bias=None):
        """qd_packed_linear(x, W, bias): the sum the cell's contract is stated in."""
        y = torch.empty(x.shape[0], self.rows, device="cuda")
        xc = x.contiguous()
        N.check(N.lib().qd_packed_linear(N.ptr(xc), xc.shape[0], self.cols, self.rows, N.ptr(self.packed), self.bits, N.ptr(self.alpha),
                                         N.ptr(self.beta), N.ptr(self.points), 0 if self.k is None else self.k, self.s or 0,
                                         self.bucket or 0, N.ptr(bias), N.ptr(y), N.stream_ptr()))
        return y


def _pair(N, I, H, bits_ih, bits_hh, uniform, bucket, seed, shift=0):
    if uniform:
        s = min(1 << bits_ih, 1 << bits_hh, 16)
        s = max(2, s - (seed % 2))                         # levels that do not fill the code width too
        return W(N, 4 * H, I, bits_ih, s, None, bucket, seed, shift), W(N, 4 * H, H, bits_hh, s, None, bucket, seed + 1, shift), s
    k_ih, k_hh = min(1 << bits_ih, 11), min(1 << bits_hh, 5 + seed % 3)
    return W(N, 4 * H, I, bits_ih, None, k_ih, bucket, seed, shift), W(N, 4 * H, H, bits_hh, None, k_hh, bucket, seed + 1, shift), 0


def _cell(N, x, h, c, w_ih, w_hh, levels, bucket, b_ih, b_hh, h_out=None, c_out=None, stream=None):
    m, H = h.shape[0], w_hh.cols
    h_out = torch.empty(m, H, device="cuda") if h_out is None else h_out
    c_out = torch.empty(m, H, device="cuda") if c_out is None else c_out
    rc = N.lib().qd_packed_lstm_cell(N.ptr(x), x.stride(0), N.ptr(h), h.stride(0), N.ptr(c), m, w_ih.cols, H, w_ih.desc.ctypes.data,
                                     w_hh.desc.ctypes.data, levels, bucket or 0, N.ptr(b_ih), N.ptr(b_hh), N.ptr(h_out), h_out.stride(0),
                                     N.ptr(c_out), stream if stream is not None else N.stream_ptr())
    N.check(rc)
    return h_out, c_out


def _contract(N, x, h, c, w_ih, w_hh, b_ih, b_hh):
    """(h', c', tol_h, tol_c): the preactivations recomputed in float32 as the contract states them, then the
    activations in float64, and a few-ulp bound of the kernel's float32 expf / tanhf / update ops against it."""
    z = w_ih.linear(N, x, b_ih) + w_hh.linear(N, h)
    if b_hh is not None:
        z = z + b_hh
    z = z.double()
    i, f, g, o = z.chunk(4, dim=1)
    si, sf, so, tg = torch.sigmoid(i), torch.sigmoid(f), torch.sigmoid(o), torch.tanh(g)
    c1 = sf * c.double() + si * tg
    h1 = so * torch.tanh(c1)
    tol_c = 10 * EPS * ((sf * c.double()).abs() + (si * tg).abs()) + 1e-38
    tol_h = 12 * EPS * h1.abs() + so * tol_c + 1e-38
    return h1, c1, tol_h, tol_c


def _inputs(m, I, H, seed, ldx=None, ldh=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    xb = torch.randn(m, ldx or I, generator=g, device="cuda")
    hb = torch.randn(m, ldh or H, generator=g, device="cuda") * 0.5
    return xb[:, :I], hb[:, :H], torch.randn(m, H, generator=g, device="cuda")


COMBOS = [(1, 2, True), (2, 2, True), (4, 8, True), (8, 4, True), (2, 4, False), (8, 1, False), (1, 1, False), (4, 4, False)]
SHAPES = [(1, 1), (3, 5), (33, 17), (129, 250), (1000, 500), (500, 500)]
ROWS = [1, 2, 3, 5, 8, 9, 64]


@pytest.mark.parametrize("bucket", [256, 100, 3, None], ids=lambda b: f"bucket{b}")
@pytest.mark.parametrize("bits_ih,bits_hh,uniform", COMBOS)
def test_cell_sweep_against_contract_and_oracle(env, bits_ih, bits_hh, uniform, bucket):
    N, _ = env
    for si, (I, H) in enumerate(SHAPES):
        seed = bits_ih * 100 + bits_hh * 10 + si + (bucket or 7)
        w_ih, w_hh, levels = _pair(N, I, H, bits_ih, bits_hh, uniform, bucket, seed)
        g = torch.Generator(device="cuda").manual_seed(seed)
        b_ih = torch.randn(4 * H, generator=g, device="cuda") * 0.2 if si % 2 == 0 else None
        b_hh = torch.randn(4 * H, generator=g, device="cuda") * 0.2 if si % 3 != 2 else None
        for m in ROWS:
            x, h, c = _inputs(m, I, H, seed + m)
            h1, c1 = _cell(N, x, h, c, w_ih, w_hh, levels, bucket, b_ih, b_hh)
            hr, cr, th, tc = _contract(N, x, h, c, w_ih, w_hh, b_ih, b_hh)
            assert torch.all((c1.double() - cr).abs() <= tc), (I, H, m, float((c1.double() - cr).abs().max()))
            assert torch.all((h1.double() - hr).abs() <= th), (I, H, m, float((h1.double() - hr).abs().max()))
            if m in (1, 64):
                args = [t.cpu().numpy() for t in (x, h, c, w_ih.q, w_hh.q)]
                bi, bh = (None if b is None else b.cpu().numpy() for b in (b_ih, b_hh))
                ho, co = O.cell(*args, bi, bh)
                tol_h, tol_c = O.step_tolerance(*args, bi, bh)
                assert np.all(np.abs(c1.cpu().numpy() - co) <= tol_c) and np.all(np.abs(h1.cpu().numpy() - ho) <= tol_h), (I, H, m)


@pytest.mark.parametrize("bits_ih,bits_hh,uniform", [(2, 2, True), (1, 4, False), (8, 8, True)])
@pytest.mark.parametrize("I,H", [(3, 5), (257, 129), (1000, 500)])
def test_unaligned_strides_and_codes(env, bits_ih, bits_hh, uniform, I, H):
    """Row strides past the rows (x, h, h_out), codes starting one byte past a word, c_out == c: the same bits as the
    contiguous, aligned call."""
    N, _ = env
    w_ih, w_hh, levels = _pair(N, I, H, bits_ih, bits_hh, uniform, 256, seed=I + H)
    s_ih, s_hh, _ = _pair(N, I, H, bits_ih, bits_hh, uniform, 256, seed=I + H, shift=1)
    b = torch.randn(4 * H, device="cuda")
    for m in (1, 7, 64):
        x, h, c = _inputs(m, I, H, m, ldx=I + 1, ldh=H + 3)
        want_h, want_c = _cell(N, x.contiguous(), h.contiguous(), c, w_ih, w_hh, levels, 256, b, b)
        out = torch.empty(m, H + 2, device="cuda")[:, :H]
        c_io = c.clone()
        got_h, got_c = _cell(N, x, h, c_io, s_ih, s_hh, levels, 256, b, b, h_out=out, c_out=c_io)
        assert torch.equal(got_h, want_h) and torch.equal(got_c, want_c) and got_c.data_ptr() == c_io.data_ptr()


def test_row_alone_and_in_batch_give_identical_bits(env):
    N, _ = env
    w_ih, w_hh, levels = _pair(N, 1000, 500, 2, 2, True, 256, seed=5)
    b = torch.randn(2000, device="cuda")
    x, h, c = _inputs(64, 1000, 500, 9)
    hb, cb = _cell(N, x, h, c, w_ih, w_hh, levels, 256, b, b)
    for i in (0, 1, 7, 8, 31, 63):
        for lo, hi in ((i, i + 1), (max(0, i - 3), min(64, i + 2))):
            hs, cs = _cell(N, x[lo:hi], h[lo:hi], c[lo:hi], w_ih, w_hh, levels, 256, b, b)
            assert torch.equal(hs[i - lo], hb[i]) and torch.equal(cs[i - lo], cb[i]), (i, lo, hi)


def test_four_streams_give_identical_bits(env):
    N, _ = env
    w_ih, w_hh, levels = _pair(N, 1000, 500, 4, 2, False, 100, seed=6)
    x, h, c = _inputs(30, 1000, 500, 3)
    ref = _cell(N, x, h, c, w_ih, w_hh, levels, 100, None, None)
    torch.cuda.synchronize()
    outs, errs = [None] * 4, []

    def work(i):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(5):
                    outs[i] = _cell(N, x, h, c, w_ih, w_hh, levels, 100, None, None, stream=st.cuda_stream)
            st.synchronize()
        except Exception as e:
            errs.append(e)
    threads = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errs, errs
    for o in outs:
        assert torch.equal(o[0], ref[0]) and torch.equal(o[1], ref[1])


# ------------------------------------------------------------------------------------------------ the layer
def _lstm_module(N, codec, I, H, num_layers, bidirectional, bits=2, s=4, bucket=256, seed=0, batch_first=False, bias=True):
    """(PackedLSTM, nn.LSTM on the decoded weights)."""
    dirs = 2 if bidirectional else 1
    pairs, biases, ref = [], [], torch.nn.LSTM(I, H, num_layers=num_layers, bidirectional=bidirectional, batch_first=batch_first,
                                                bias=bias).cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for k in range(num_layers * dirs):
            in_size = I if k < dirs else dirs * H
            w_ih = W(N, 4 * H, in_size, bits, s, None, bucket, seed + 2 * k)
            w_hh = W(N, 4 * H, H, bits, s, None, bucket, seed + 2 * k + 1)
            pairs.append((w_ih.entry(codec), w_hh.entry(codec)))
            sfx = f"_l{k // dirs}" + ("_reverse" if k % dirs else "")
            getattr(ref, "weight_ih" + sfx).copy_(w_ih.q)
            getattr(ref, "weight_hh" + sfx).copy_(w_hh.q)
            if bias:
                b = (torch.randn(4 * H, generator=g, device="cuda") * 0.2, torch.randn(4 * H, generator=g, device="cuda") * 0.2)
                getattr(ref, "bias_ih" + sfx).copy_(b[0])
                getattr(ref, "bias_hh" + sfx).copy_(b[1])
                biases.append(b)
    mod = codec.PackedLSTM(pairs, "uniform", s, bucket, num_layers=num_layers, batch_first=batch_first, bidirectional=bidirectional,
                           biases=biases if bias else None)
    mod.CROSSOVER_ROWS = N.PACKED_LSTM_MAX_ROWS                          # the kernel path up to its 64 rows
    return mod.eval(), ref.eval()


def _no_tf32():
    class _Ctx:
        def __enter__(self):
            self.old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

        def __exit__(self, *a):
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.old
    return _Ctx()


def _close(a, b, what):
    # float32 kernel against cuDNN float32 (TF32 off) on the same weights: summation orders differ, and the difference
    # is carried through every step; 2e-5 + 1e-4 relative holds for T <= 25 steps of width <= 500 with |h| <= 1
    assert torch.allclose(a, b, rtol=1e-4, atol=2e-5), (what, float((a - b).abs().max()))


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("lengths", [[6, 6, 6], [6, 5, 5, 3, 1], [1]])
def test_layer_against_stepped_cells_and_oracle(env, reverse, lengths):
    """qd_packed_lstm_layer over a PackedSequence equals, bit for bit, the cell stepped by hand with the kernel's own
    state (h from the previous active step or h0, c carried per row); each step is inside the oracle's step bound."""
    N, _ = env
    I, H = 37, 29
    w_ih, w_hh, levels = _pair(N, I, H, 2, 4, True, 100, seed=11)
    b_ih, b_hh = torch.randn(4 * H, device="cuda") * 0.3, torch.randn(4 * H, device="cuda") * 0.3
    bs = [sum(L > t for L in lengths) for t in range(lengths[0])]
    off = np.concatenate([[0], np.cumsum(bs)])
    B, total = bs[0], int(off[-1])
    data = torch.randn(total, I, device="cuda")
    h0, c0 = torch.randn(B, H, device="cuda") * 0.5, torch.randn(B, H, device="cuda")
    out = torch.empty(total, 2 * H, device="cuda")[:, H:]                  # the reverse half of a bidirectional output
    h_n, c_n = torch.empty(B, H, device="cuda"), torch.empty(B, H, device="cuda")
    bsa = np.asarray(bs, np.int64)
    N.check(N.lib().qd_packed_lstm_layer(N.ptr(data), I, bsa.ctypes.data, len(bs), int(reverse), I, H, w_ih.desc.ctypes.data,
                                         w_hh.desc.ctypes.data, levels, 100, N.ptr(b_ih), N.ptr(b_hh), N.ptr(h0), N.ptr(c0), N.ptr(out),
                                         2 * H, N.ptr(h_n), N.ptr(c_n), N.stream_ptr()))
    h, c = h0.clone(), c0.clone()
    for t in (reversed(range(len(bs))) if reverse else range(len(bs))):
        m = bs[t]
        x = data[off[t]:off[t] + m]
        h1, c1 = _cell(N, x, h[:m].contiguous(), c[:m].contiguous(), w_ih, w_hh, levels, 100, b_ih, b_hh)
        assert torch.equal(out[off[t]:off[t] + m], h1), t
        args = [a.cpu().numpy() for a in (x, h[:m], c[:m], w_ih.q, w_hh.q)]
        ho, co = O.cell(*args, b_ih.cpu().numpy(), b_hh.cpu().numpy())
        tol_h, tol_c = O.step_tolerance(*args, b_ih.cpu().numpy(), b_hh.cpu().numpy())
        assert np.all(np.abs(h1.cpu().numpy() - ho) <= tol_h) and np.all(np.abs(c1.cpu().numpy() - co) <= tol_c), t
        h[:m], c[:m] = h1, c1
    assert torch.equal(h_n, h) and torch.equal(c_n, c)


@pytest.mark.parametrize("num_layers,bidirectional,batch_first,with_hx", [(1, False, False, False), (2, True, False, True),
                                                                          (3, False, True, True), (2, True, True, False),
                                                                          (3, True, False, True)])
def test_module_padded_against_cudnn(env, num_layers, bidirectional, batch_first, with_hx):
    N, codec = env
    I, H, T, B = 40, 48, 25, 5
    mod, ref = _lstm_module(N, codec, I, H, num_layers, bidirectional, seed=num_layers * 7 + bidirectional, batch_first=batch_first)
    dirs = 2 if bidirectional else 1
    x = torch.randn(B, T, I, device="cuda") if batch_first else torch.randn(T, B, I, device="cuda")
    hx = (torch.randn(num_layers * dirs, B, H, device="cuda") * 0.5, torch.randn(num_layers * dirs, B, H, device="cuda")) if with_hx else None
    with torch.no_grad(), _no_tf32():
        out, (h_n, c_n) = mod(x, hx)
        want, (wh, wc) = ref(x, hx)
    assert out.shape == want.shape and h_n.shape == wh.shape and c_n.shape == wc.shape
    _close(out, want, "output"), _close(h_n, wh, "h_n"), _close(c_n, wc, "c_n")
    # the float64 oracle on the kernel's own decoded weights, run from the same start
    flat = [w.cpu().numpy() if w is not None else None for w in mod.decoded_weights()]
    weights = [flat[4 * k:4 * k + 4] for k in range(num_layers * dirs)]
    xs = (x.transpose(0, 1) if batch_first else x).cpu().numpy()
    h0 = hx[0].cpu().numpy() if hx else None
    o, hn, cn = O.lstm(xs.reshape(T * B, I), O.padded_batch_sizes(T, B), weights, num_layers, bidirectional,
                       None if hx is None else (h0, hx[1].cpu().numpy()))
    got = (out.transpose(0, 1) if batch_first else out).reshape(T * B, -1).cpu().numpy()
    assert np.allclose(got, o, rtol=1e-4, atol=2e-5) and np.allclose(h_n.cpu().numpy(), hn, rtol=1e-4, atol=2e-5)


def test_module_unbatched_and_packed_sequences(env):
    N, codec = env
    I, H, T = 24, 32, 9
    mod, ref = _lstm_module(N, codec, I, H, 2, True, bits=4, s=16, bucket=None, seed=3)
    with torch.no_grad(), _no_tf32():
        x = torch.randn(T, I, device="cuda")                                 # unbatched
        out, (h_n, c_n) = mod(x)
        want, (wh, wc) = ref(x)
        assert out.shape == want.shape == (T, 2 * H) and h_n.shape == wh.shape == (4, H)
        _close(out, want, "unbatched"), _close(c_n, wc, "unbatched c_n")
        lengths = [9, 2, 7, 1, 9, 4]
        xp = torch.randn(T, len(lengths), I, device="cuda")
        hx = (torch.randn(4, len(lengths), H, device="cuda"), torch.randn(4, len(lengths), H, device="cuda"))
        for enforce_sorted in (True, False):
            ls = sorted(lengths, reverse=True) if enforce_sorted else lengths
            ps = torch.nn.utils.rnn.pack_padded_sequence(xp, torch.tensor(ls), enforce_sorted=enforce_sorted)
            out, (h_n, c_n) = mod(ps, hx)
            want, (wh, wc) = ref(ps, hx)
            assert torch.equal(out.batch_sizes, want.batch_sizes)
            _close(out.data, want.data, "packed"), _close(h_n, wh, "packed h_n"), _close(c_n, wc, "packed c_n")
            # a sequence gives the same bits alone as inside the PackedSequence
            b = 2
            alone, (ah, ac) = mod(xp[:ls[b], b], (hx[0][:, b], hx[1][:, b]))
            padded, _ = torch.nn.utils.rnn.pad_packed_sequence(out)
            assert torch.equal(alone, padded[:ls[b], b]) and torch.equal(ah, h_n[:, b]) and torch.equal(ac, c_n[:, b])


def test_cell_module_against_nn_lstm_cell(env):
    N, codec = env
    I, H = 1000, 500
    w_ih, w_hh, levels = _pair(N, I, H, 2, 2, True, 256, seed=21)
    b_ih, b_hh = torch.randn(4 * H, device="cuda") * 0.1, torch.randn(4 * H, device="cuda") * 0.1
    cell = codec.PackedLSTMCell(w_ih.entry(codec), w_hh.entry(codec), "uniform", levels, 256, b_ih, b_hh)
    cell.CROSSOVER_ROWS = N.PACKED_LSTM_MAX_ROWS
    ref = torch.nn.LSTMCell(I, H).cuda()
    with torch.no_grad():
        ref.weight_ih.copy_(w_ih.q), ref.weight_hh.copy_(w_hh.q), ref.bias_ih.copy_(b_ih), ref.bias_hh.copy_(b_hh)
        assert all(torch.equal(a, b) for a, b in zip(cell.decoded_weights(), (w_ih.q, w_hh.q)))
        for B in (1, 5, 30, 64):
            x, h, c = _inputs(B, I, H, B)
            with _no_tf32():
                got, want = cell(x, (h, c)), ref(x, (h, c))
            _close(got[0], want[0], B), _close(got[1], want[1], B)
            assert torch.equal(got[0], _cell(N, x, h, c, w_ih, w_hh, levels, 256, b_ih, b_hh)[0])
        x = torch.randn(I, device="cuda")
        h1, c1 = cell(x)
        assert h1.shape == c1.shape == (H,)
        assert torch.equal(h1, cell(x[None], (torch.zeros(1, H, device="cuda"),) * 2)[0][0])
        x, h, c = _inputs(65, I, H, 65)                                       # above 64 rows: decode + torch, as unpack_ would
        got = cell(x, (h, c))
        want = ref(x, (h, c))
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_module_above_64_rows_equals_unpack_and_torch(env):
    N, codec = env
    mod, ref = _lstm_module(N, codec, 32, 40, 2, True, seed=8)
    ref.flatten_parameters()
    with torch.no_grad():
        for x in (torch.randn(7, 65, 32, device="cuda"),
                  torch.nn.utils.rnn.pack_padded_sequence(torch.randn(7, 70, 32, device="cuda"), torch.randint(1, 8, (70,)),
                                                          enforce_sorted=False)):
            out, (h_n, c_n) = mod(x)
            want, (wh, wc) = ref(x)
            o, w = (out.data, want.data) if isinstance(out, torch.nn.utils.rnn.PackedSequence) else (out, want)
            assert torch.equal(o, w) and torch.equal(h_n, wh) and torch.equal(c_n, wc)


def test_cuda_graph_replay_of_a_whole_forward(env):
    N, codec = env
    mod, _ = _lstm_module(N, codec, 64, 96, 2, True, seed=4)
    x = torch.randn(12, 5, 64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad():
        with torch.cuda.stream(side):
            ref, (rh, rc) = mod(x)
            ref, rh, rc = ref.clone(), rh.clone(), rc.clone()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out, (h_n, c_n) = mod(x)
    for _ in range(3):
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, ref) and torch.equal(h_n, rh) and torch.equal(c_n, rc)


# ------------------------------------------------------------------------------------------------ refusals
def test_c_abi_refusals(env):
    N, _ = env
    I, H, m = 6, 5, 3
    w_ih, w_hh, levels = _pair(N, I, H, 2, 2, True, 256, seed=1)
    _, w_bad, _ = _pair(N, I, I, 2, 2, True, 256, seed=1)                 # [4I, I]: not [4H, H]
    x, h, c = _inputs(m, I, H, 0)
    x, h = x.contiguous(), h.contiguous()
    ho, co = torch.empty(m, H, device="cuda"), torch.empty(m, H, device="cuda")
    pts = torch.rand(5, device="cuda")
    L = N.lib()

    def cell(**kw):
        a = dict(x=N.ptr(x), ldx=I, h=N.ptr(h), ldh=H, c=N.ptr(c), m=m, I=I, H=H, w_ih=w_ih.desc.ctypes.data, w_hh=w_hh.desc.ctypes.data,
                 levels=levels, bucket=256, b_ih=None, b_hh=None, h_out=N.ptr(ho), ldo=H, c_out=N.ptr(co))
        a.update(kw)
        return L.qd_packed_lstm_cell(*a.values(), N.stream_ptr())
    assert cell() == N.QD_OK and cell(c_out=N.ptr(c)) == N.QD_OK
    torch.cuda.synchronize()
    bad_bits = w_ih.desc.copy()
    bad_bits["bits"] = 3
    narrow = w_ih.desc.copy()
    narrow["points"], narrow["num_points"] = pts.data_ptr(), 5
    for bad in (dict(x=None), dict(h=None), dict(c=None), dict(h_out=None), dict(c_out=None), dict(w_ih=None), dict(w_hh=None),
                dict(m=0), dict(m=-1), dict(I=0), dict(H=0), dict(ldx=I - 1), dict(ldh=H - 1), dict(ldo=H - 1),
                dict(w_hh=w_bad.desc.ctypes.data), dict(w_ih=bad_bits.ctypes.data), dict(levels=5), dict(levels=1),
                dict(levels=0, w_ih=narrow.ctypes.data), dict(levels=0), dict(w_ih=narrow.ctypes.data), dict(bucket=-1),
                dict(h_out=N.ptr(x)), dict(h_out=N.ptr(h)), dict(h_out=N.ptr(c)), dict(c_out=N.ptr(c) + 4),
                dict(c_out=N.ptr(x))):
        assert cell(**bad) == N.QD_ERR_INVALID_ARG, bad
        assert L.qd_last_error().decode()
    assert cell(m=65) == N.QD_ERR_UNSUPPORTED and L.qd_last_error().decode()

    B = 3
    data = torch.randn(9, I, device="cuda")
    out = torch.empty(9, H, device="cuda")
    h0, c0 = torch.zeros(B, H, device="cuda"), torch.zeros(B, H, device="cuda")
    hn, cn = torch.empty(B, H, device="cuda"), torch.empty(B, H, device="cuda")

    def layer(bs, **kw):
        bsa = np.asarray(bs, np.int64)
        a = dict(x=N.ptr(data), ldx=I, sizes=bsa.ctypes.data, steps=len(bs), reverse=0, I=I, H=H, w_ih=w_ih.desc.ctypes.data,
                 w_hh=w_hh.desc.ctypes.data, levels=levels, bucket=256, b_ih=None, b_hh=None, h0=N.ptr(h0), c0=N.ptr(c0), out=N.ptr(out),
                 ldo=H, h_n=N.ptr(hn), c_n=N.ptr(cn))
        a.update(kw)
        return L.qd_packed_lstm_layer(*a.values(), N.stream_ptr())
    assert layer([3, 3, 3]) == N.QD_OK and layer([3, 2, 1], reverse=1) == N.QD_OK and layer([3, 3, 3], c_n=N.ptr(c0)) == N.QD_OK
    torch.cuda.synchronize()
    for bs, bad in (([3, 3, 3], dict(x=None)), ([3, 3, 3], dict(sizes=None)), ([3, 3, 3], dict(h0=None)), ([3, 3, 3], dict(c0=None)),
                    ([3, 3, 3], dict(out=None)), ([3, 3, 3], dict(h_n=None)), ([3, 3, 3], dict(c_n=None)), ([3], dict(steps=0)),
                    ([2, 3, 1], {}), ([3, 1, 2], {}), ([3, 0], {}), ([3, 3, 3], dict(ldx=I - 1)), ([3, 3, 3], dict(ldo=H - 1)),
                    ([3, 3, 3], dict(out=N.ptr(data))), ([3, 3, 3], dict(h_n=N.ptr(out))), ([3, 3, 3], dict(c_n=N.ptr(hn))),
                    ([3, 3, 3], dict(out=N.ptr(h0))), ([3, 3, 3], dict(levels=7))):
        assert layer(bs, **bad) == N.QD_ERR_INVALID_ARG, (bs, bad)
        assert L.qd_last_error().decode()
    data65 = torch.randn(65, I, device="cuda")
    assert layer([65], x=N.ptr(data65)) == N.QD_ERR_UNSUPPORTED and L.qd_last_error().decode()


def test_module_refusals(env):
    N, codec = env
    mod, _ = _lstm_module(N, codec, 8, 6, 2, False, seed=2)
    mod.dropout = 0.3
    x = torch.randn(4, 2, 8, device="cuda")
    with torch.no_grad():
        mod.train()
        with pytest.raises(RuntimeError, match="dropout"):
            mod(x)
        mod.eval()
        mod(x)
        for bad in (x.cpu(), x.double(), torch.randn(4, 2, 7, device="cuda"), torch.randn(2, 2, 2, 8, device="cuda")):
            with pytest.raises(ValueError):
                mod(bad)
        with pytest.raises(ValueError):
            mod(x, (torch.zeros(2, 3, 6, device="cuda"), torch.zeros(2, 3, 6, device="cuda")))
    with pytest.raises(RuntimeError, match="forward only"):
        mod(x.clone().requires_grad_())
    with pytest.raises(RuntimeError, match="float32"):
        mod.double()(x)
    w_ih, w_hh, levels = _pair(N, 8, 6, 2, 2, True, 256, seed=3)
    cell = codec.PackedLSTMCell(w_ih.entry(codec), w_hh.entry(codec), "uniform", levels, 256)
    with pytest.raises(ValueError):
        cell(torch.randn(3, 8))
    with pytest.raises(ValueError):
        cell(torch.randn(3, 9, device="cuda"))
    with pytest.raises(RuntimeError, match="forward only"):
        cell(torch.randn(3, 8, device="cuda", requires_grad=True))
    with pytest.raises(RuntimeError, match="float32"):
        codec.PackedLSTMCell(w_ih.entry(codec), w_hh.entry(codec), "uniform", levels, 256).half()(torch.randn(3, 8, device="cuda"))
    with pytest.raises(ValueError):
        codec.PackedLSTMCell(w_hh.entry(codec), w_ih.entry(codec), "uniform", levels, 256)     # [24, 6] ih then [24, 8] hh
    with pytest.raises(ValueError):
        cell(torch.randn(3, 8, device="cuda"), (torch.zeros(2, 6, device="cuda"), torch.zeros(2, 6, device="cuda")))


# ------------------------------------------------------------------------------------------------ attaching
class _NMT(torch.nn.Module):
    """The reference's NMT shape in small: embeddings with a padding index, an LSTM encoder fed a PackedSequence, a
    StackedLSTM-style decoder of nn.LSTMCell with input feeding, a global-attention nn.Linear and a generator tied to
    the target embedding."""

    def __init__(self, vs=900, vt=700, d=48, layers=2, bidirectional=False):
        super().__init__()
        self.bidirectional = bidirectional
        self.src_emb = torch.nn.Embedding(vs, d, padding_idx=1)
        self.tgt_emb = torch.nn.Embedding(vt, d, padding_idx=1)
        self.encoder = torch.nn.LSTM(d, d // 2 if bidirectional else d, num_layers=layers, bidirectional=bidirectional)
        self.cells = torch.nn.ModuleList([torch.nn.LSTMCell(2 * d if i == 0 else d, d) for i in range(layers)])
        self.attn = torch.nn.Linear(2 * d, d, bias=False)
        self.generator = torch.nn.Linear(d, vt)
        self.generator.weight = self.tgt_emb.weight

    def forward(self, src, lengths, tgt):
        ps = torch.nn.utils.rnn.pack_padded_sequence(self.src_emb(src), lengths, enforce_sorted=False)
        mem, (h, c) = self.encoder(ps)
        mem = torch.nn.utils.rnn.pad_packed_sequence(mem)[0].transpose(0, 1)                  # [B, S, d]
        if self.bidirectional:
            h = torch.cat([h[0::2], h[1::2]], 2)
            c = torch.cat([c[0::2], c[1::2]], 2)
        state = [(h[i], c[i]) for i in range(len(self.cells))]
        feed = torch.zeros_like(state[0][0])
        logits = []
        for y in self.tgt_emb(tgt):
            inp = torch.cat([y, feed], 1)
            for i, cell in enumerate(self.cells):
                state[i] = cell(inp, state[i])
                inp = state[i][0]
            ctx = torch.softmax(torch.bmm(mem, inp[:, :, None]), 1).transpose(1, 2).bmm(mem)[:, 0]
            feed = torch.tanh(self.attn(torch.cat([ctx, inp], 1)))
            logits.append(self.generator(feed))
        return torch.stack(logits)


def _nmt(seed, **kw):
    torch.manual_seed(seed)
    return _NMT(**kw).cuda()


def _blocks(ptrs):
    """{block start: size} of the caching allocator's allocated blocks that contain the given addresses."""
    sizes = {}
    for seg in torch.cuda.memory_snapshot():
        addr = seg["address"]
        for blk in seg["blocks"]:
            if blk["state"] == "active_allocated" and any(addr <= p < addr + blk["size"] for p in ptrs):
                sizes[addr] = blk["size"]
            addr += blk["size"]
    return sizes


def _batch(g, B=6, S=11, T=7):
    src = torch.randint(2, 900, (S, B), device="cuda", generator=g)
    lengths = torch.tensor([S, 4, 9, 1, S, 6][:B])
    for b, L in enumerate(lengths.tolist()):
        src[L:, b] = 1
    return src, lengths, torch.randint(2, 700, (T, B), device="cuda", generator=g)


@pytest.mark.parametrize("bidirectional", [False, True])
@pytest.mark.parametrize("kind", ["uniform", "nonuniform"])
def test_attach_nmt_model(env, kind, bidirectional):
    N, codec = env
    trained = _nmt(0, bidirectional=bidirectional)
    if kind == "uniform":
        pm = codec.pack_model(trained, 4, 256, quantize_first_and_last_layer=True)
    else:
        n_q = len(list(trained.parameters()))
        pts = [np.sort(np.random.default_rng(i).random(3 + i % 14)).astype(np.float32) for i in range(n_q)]
        pm = codec.pack_model(trained, points=pts, bucket_size=256, quantize_first_and_last_layer=True)
    ref = _nmt(1, bidirectional=bidirectional)
    codec.unpack_(pm, ref)
    fresh = _nmt(2, bidirectional=bidirectional)
    enc = fresh.encoder
    enc_ptrs = {p.data_ptr() for p in enc.parameters()}
    released = _blocks(enc_ptrs)
    assert len(released) == 1                                             # the LSTM's one flattened buffer, biases included
    cell_params = [p for cell in fresh.cells for p in cell.parameters()]
    released.update(_blocks({p.data_ptr() for p in cell_params} | {fresh.src_emb.weight.data_ptr(), fresh.tgt_emb.weight.data_ptr(),
                                                                      fresh.attn.weight.data_ptr()}))
    assert len(released) == 1 + len(cell_params) + 3
    n_bias = 2 * enc.num_layers * (2 if bidirectional else 1) + 2 * len(fresh.cells)
    bias_block = -(-4 * 4 * fresh.cells[0].hidden_size // 512) * 512                     # a copied bias's allocator block
    enc_bias_block = -(-4 * 4 * enc.hidden_size // 512) * 512
    new = 2 * 512 + 2 * enc.num_layers * (2 if bidirectional else 1) * enc_bias_block + 2 * len(fresh.cells) * bias_block
    del enc, cell_params
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    names = codec.attach_packed_(pm, fresh, embeddings=True, recurrent=True)
    gc.collect()
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    assert names == ["src_emb", "tgt_emb", "encoder", "cells.0", "cells.1", "attn", "generator"]
    assert type(fresh.encoder) is codec.PackedLSTM and all(type(c) is codec.PackedLSTMCell for c in fresh.cells)
    assert n_bias == sum(1 for n, _ in fresh.named_buffers() if n.endswith(".bias") and (n.startswith("encoder") or n.startswith("cells")))
    # every float32 LSTM / LSTMCell weight is gone: the encoder's flattened buffer, the cells' four tensors each, both
    # tables and the attention weight; each copied bias and each embedding's invalid-index counter is one new block
    assert before - after == sum(released.values()) - new, (before, after, sum(released.values()), new)
    assert not any(p.dim() == 2 and n.startswith(("encoder", "cells")) for n, p in fresh.named_parameters())
    got = dict(fresh.named_parameters())
    got.update({n: b for n, b in fresh.named_buffers()})
    for name, t in ref.named_parameters():                                # the biases as unpack_ wrote them
        if name.startswith("cells."):
            i, which = name.split(".")[1], name.split(".")[2]
            if which.startswith("bias"):
                assert torch.equal(got[f"cells.{i}.weights.{0 if which == 'bias_ih' else 1}.bias"], t.data), name
        elif name.startswith("encoder.bias"):
            _, which, lyr, *rev = name.split(".")[1].split("_")
            k = int(lyr[1:]) * (2 if bidirectional else 1) + bool(rev)
            assert torch.equal(got[f"encoder.cells.{k}.{0 if which == 'ih' else 1}.bias"], t.data), name
        elif name == "generator.bias":
            assert torch.equal(got["generator.bias"], t.data)
    for k, (ih, hh) in enumerate(fresh.encoder.cells):
        sfx = f"_l{k // (2 if bidirectional else 1)}" + ("_reverse" if bidirectional and k % 2 else "")
        assert torch.equal(ih.decoded(), getattr(ref.encoder, "weight_ih" + sfx).data)
        assert torch.equal(hh.decoded(), getattr(ref.encoder, "weight_hh" + sfx).data)
    for cell, rc in zip(fresh.cells, ref.cells):
        assert all(torch.equal(a, b) for a, b in zip(cell.decoded_weights(), (rc.weight_ih.data, rc.weight_hh.data)))
    g = torch.Generator(device="cuda").manual_seed(3)
    src, lengths, tgt = _batch(g)
    with torch.no_grad(), _no_tf32():
        out, want = fresh(src, lengths, tgt), ref(src, lengths, tgt)
    assert torch.allclose(out, want, rtol=1e-4, atol=1e-4 * float(want.abs().max())), float((out - want).abs().max())


class _Ineligible(torch.nn.Module):
    """Recurrent modules attach_packed_ must leave to unpack_ even with recurrent=True: a GRU, an LSTM subclass, an LSTM
    with a projection, two LSTMCells sharing a weight, and an LSTM whose first matrix the model keeps float32; one plain
    LSTM and one plain LSTMCell it replaces."""

    class Sub(torch.nn.LSTM):
        pass

    def __init__(self):
        super().__init__()
        self.first = torch.nn.LSTM(8, 8)                   # the model's first parameter: stored float32
        self.gru = torch.nn.GRU(8, 8)
        self.sub = _Ineligible.Sub(8, 8)
        self.proj = torch.nn.LSTM(8, 8, proj_size=4)
        self.shared_a = torch.nn.LSTMCell(8, 8)
        self.shared_b = torch.nn.LSTMCell(8, 8)
        self.shared_b.weight_hh = self.shared_a.weight_hh
        self.plain = torch.nn.LSTM(8, 8)
        self.plain_cell = torch.nn.LSTMCell(8, 8)
        self.last = torch.nn.Linear(8, 3)


def test_attach_leaves_ineligible_recurrent_modules_to_unpack(env):
    N, codec = env
    torch.manual_seed(0)
    pm = codec.pack_model(_Ineligible().cuda(), 4, 64, quantize_first_and_last_layer=False)
    torch.manual_seed(1)
    ref = _Ineligible().cuda()
    codec.unpack_(pm, ref)
    torch.manual_seed(2)
    fresh = _Ineligible().cuda()
    assert codec.attach_packed_(pm, fresh, recurrent=True) == ["plain", "plain_cell", "last"]
    assert type(fresh.first) is torch.nn.LSTM and type(fresh.gru) is torch.nn.GRU and type(fresh.sub) is _Ineligible.Sub
    assert type(fresh.proj) is torch.nn.LSTM and type(fresh.shared_a) is torch.nn.LSTMCell and type(fresh.shared_b) is torch.nn.LSTMCell
    assert fresh.shared_b.weight_hh is fresh.shared_a.weight_hh
    got = dict(fresh.named_parameters())
    got.update(dict(fresh.named_buffers()))                               # a replaced Linear holds its bias as a buffer
    for name, t in ref.named_parameters():
        if not name.startswith(("plain", "last.weight")):
            assert torch.equal(got[name].data, t.data), name
    x = torch.randn(5, 3, 8, device="cuda")
    with torch.no_grad(), _no_tf32():
        _close(fresh.plain(x)[0], ref.plain(x)[0], "plain")
        _close(fresh.plain_cell(x[0])[0], ref.plain_cell(x[0])[0], "plain_cell")
    torch.manual_seed(2)
    default = _Ineligible().cuda()
    assert codec.attach_packed_(pm, default, embeddings=True) == ["last"]  # without recurrent=True: nothing recurrent
    assert type(default.plain) is torch.nn.LSTM and torch.equal(default.plain.weight_ih_l0, ref.plain.weight_ih_l0)


def test_attach_huffman_route(env):
    """A Huffman-coded model transcoded to fixed-width codes and attached with recurrent=True holds the weights
    decompress_ writes, and computes the same logits within tolerance."""
    N, codec = env
    cm = codec.compress_model(_nmt(0), 4, bucket_size=256, quantize_first_and_last_layer=True)
    net = _nmt(2)
    assert codec.attach_packed_(codec.pack_compressed(cm), net, embeddings=True, recurrent=True) == \
        ["src_emb", "tgt_emb", "encoder", "cells.0", "cells.1", "attn", "generator"]
    ref = _nmt(1)
    codec.decompress_(cm, ref)
    assert torch.equal(net.encoder.cells[1][1].decoded(), ref.encoder.weight_hh_l1.data)
    assert torch.equal(net.cells[0].decoded_weights()[0], ref.cells[0].weight_ih.data)
    g = torch.Generator(device="cuda").manual_seed(4)
    src, lengths, tgt = _batch(g)
    with torch.no_grad(), _no_tf32():
        out, want = net(src, lengths, tgt), ref(src, lengths, tgt)
    assert torch.allclose(out, want, rtol=1e-4, atol=1e-4 * float(want.abs().max())), float((out - want).abs().max())
