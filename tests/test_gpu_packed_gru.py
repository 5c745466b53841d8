"""GRU layers run from their packed codes: qd_packed_gru_cell against its stated contract (gi and gh from
qd_packed_linear, the gate adds in float32, activations carried in float64) and the float64 oracle over code widths,
uniform and non-uniform weights at different widths, buckets straddling gate rows, odd sizes up to the NMT shapes,
every row tile and unaligned strides; determinism (alone / in a batch, four streams, CUDA-graph replay of a whole
PackedGRU); qd_packed_gru_layer against step-by-step cells and the oracle; PackedGRU / PackedGRUCell against cuDNN on
the decoded weights and, above 64 rows or CROSSOVER_ROWS, equal to unpack_ + torch; refusals at the C ABI and in the
modules; and attach_packed_(..., gru=True) on an NMT-shaped GRU model (exact memory account), on the Huffman route and
on the recurrent modules it must leave to unpack_."""
import gc
import threading

import numpy as np
import pytest
import torch

from oracle import packed_gru_oracle as O

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
        """qd_packed_linear(x, W, bias): the outputs the cell's contract is stated in."""
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
        return W(N, 3 * H, I, bits_ih, s, None, bucket, seed, shift), W(N, 3 * H, H, bits_hh, s, None, bucket, seed + 1, shift), s
    k_ih, k_hh = min(1 << bits_ih, 11), min(1 << bits_hh, 5 + seed % 3)
    return W(N, 3 * H, I, bits_ih, None, k_ih, bucket, seed, shift), W(N, 3 * H, H, bits_hh, None, k_hh, bucket, seed + 1, shift), 0


def _cell(N, x, h, w_ih, w_hh, levels, bucket, b_ih, b_hh, h_out=None, stream=None):
    m, H = h.shape[0], w_hh.cols
    h_out = torch.empty(m, H, device="cuda") if h_out is None else h_out
    rc = N.lib().qd_packed_gru_cell(N.ptr(x), x.stride(0), N.ptr(h), h.stride(0), m, w_ih.cols, H, w_ih.desc.ctypes.data,
                                    w_hh.desc.ctypes.data, levels, bucket or 0, N.ptr(b_ih), N.ptr(b_hh), N.ptr(h_out), h_out.stride(0),
                                    stream if stream is not None else N.stream_ptr())
    N.check(rc)
    return h_out


def _contract(N, x, h, w_ih, w_hh, b_ih, b_hh):
    """(h', tol): gi and gh from qd_packed_linear and the r / z gate adds in float32, as the contract states them, then
    the activations and the update in float64, and a few-ulp bound of the kernel's float32 expf / tanhf / update ops."""
    gi, gh = w_ih.linear(N, x, b_ih), w_hh.linear(N, h, b_hh)
    (i_r, i_z, i_n), (h_r, h_z, h_n) = gi.chunk(3, dim=1), gh.chunk(3, dim=1)
    r, z = torch.sigmoid((i_r + h_r).double()), torch.sigmoid((i_z + h_z).double())
    i_n, h_n, hd = i_n.double(), h_n.double(), h.double()
    pre = i_n + r * h_n
    n = torch.tanh(pre)
    h1 = n + z * (hd - n)
    dr = dz = 6 * EPS
    dn = h_n.abs() * dr + 2 * EPS * ((r * h_n).abs() + pre.abs()) + 3 * EPS * n.abs()
    tol = 2 * (dn + (hd - n).abs() * dz + 3 * EPS * ((hd - n).abs() + h1.abs())) + 1e-38
    return h1, tol


def _inputs(m, I, H, seed, ldx=None, ldh=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    xb = torch.randn(m, ldx or I, generator=g, device="cuda")
    hb = torch.randn(m, ldh or H, generator=g, device="cuda") * 0.5
    return xb[:, :I], hb[:, :H]


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
        b_ih = torch.randn(3 * H, generator=g, device="cuda") * 0.2 if si % 2 == 0 else None
        b_hh = torch.randn(3 * H, generator=g, device="cuda") * 0.2 if si % 3 != 2 else None
        for m in ROWS:
            x, h = _inputs(m, I, H, seed + m)
            h1 = _cell(N, x, h, w_ih, w_hh, levels, bucket, b_ih, b_hh)
            hr, th = _contract(N, x, h, w_ih, w_hh, b_ih, b_hh)
            assert torch.all((h1.double() - hr).abs() <= th), (I, H, m, float((h1.double() - hr).abs().max()))
            if m in (1, 64):
                args = [t.cpu().numpy() for t in (x, h, w_ih.q, w_hh.q)]
                bi, bh = (None if b is None else b.cpu().numpy() for b in (b_ih, b_hh))
                ho = O.cell(*args, bi, bh)
                assert np.all(np.abs(h1.cpu().numpy() - ho) <= O.step_tolerance(*args, bi, bh)), (I, H, m)


@pytest.mark.parametrize("bits_ih,bits_hh,uniform", [(2, 2, True), (1, 4, False), (8, 8, True)])
@pytest.mark.parametrize("I,H", [(3, 5), (257, 129), (1000, 500)])
def test_unaligned_strides_and_codes(env, bits_ih, bits_hh, uniform, I, H):
    """Row strides past the rows (x, h, h_out) and codes starting one byte past a word: the same bits as the
    contiguous, aligned call."""
    N, _ = env
    w_ih, w_hh, levels = _pair(N, I, H, bits_ih, bits_hh, uniform, 256, seed=I + H)
    s_ih, s_hh, _ = _pair(N, I, H, bits_ih, bits_hh, uniform, 256, seed=I + H, shift=1)
    b = torch.randn(3 * H, device="cuda")
    for m in (1, 7, 64):
        x, h = _inputs(m, I, H, m, ldx=I + 1, ldh=H + 3)
        want = _cell(N, x.contiguous(), h.contiguous(), w_ih, w_hh, levels, 256, b, b)
        out = torch.empty(m, H + 2, device="cuda")[:, :H]
        got = _cell(N, x, h, s_ih, s_hh, levels, 256, b, b, h_out=out)
        assert torch.equal(got, want)


def test_row_alone_and_in_batch_give_identical_bits(env):
    N, _ = env
    w_ih, w_hh, levels = _pair(N, 1000, 500, 2, 2, True, 256, seed=5)
    b = torch.randn(1500, device="cuda")
    x, h = _inputs(64, 1000, 500, 9)
    hb = _cell(N, x, h, w_ih, w_hh, levels, 256, b, b)
    for i in (0, 1, 7, 8, 31, 63):
        for lo, hi in ((i, i + 1), (max(0, i - 3), min(64, i + 2))):
            hs = _cell(N, x[lo:hi], h[lo:hi], w_ih, w_hh, levels, 256, b, b)
            assert torch.equal(hs[i - lo], hb[i]), (i, lo, hi)


def test_four_streams_give_identical_bits(env):
    N, _ = env
    w_ih, w_hh, levels = _pair(N, 1000, 500, 4, 2, False, 100, seed=6)
    x, h = _inputs(30, 1000, 500, 3)
    ref = _cell(N, x, h, w_ih, w_hh, levels, 100, None, None)
    torch.cuda.synchronize()
    outs, errs = [None] * 4, []

    def work(i):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(5):
                    outs[i] = _cell(N, x, h, w_ih, w_hh, levels, 100, None, None, stream=st.cuda_stream)
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
        assert torch.equal(o, ref)


# ------------------------------------------------------------------------------------------------ the layer
def _gru_module(N, codec, I, H, num_layers, bidirectional, bits=2, s=4, bucket=256, seed=0, batch_first=False, bias=True):
    """(PackedGRU on the kernel path, nn.GRU on the decoded weights)."""
    dirs = 2 if bidirectional else 1
    pairs, biases, ref = [], [], torch.nn.GRU(I, H, num_layers=num_layers, bidirectional=bidirectional, batch_first=batch_first,
                                               bias=bias).cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for k in range(num_layers * dirs):
            in_size = I if k < dirs else dirs * H
            w_ih = W(N, 3 * H, in_size, bits, s, None, bucket, seed + 2 * k)
            w_hh = W(N, 3 * H, H, bits, s, None, bucket, seed + 2 * k + 1)
            pairs.append((w_ih.entry(codec), w_hh.entry(codec)))
            sfx = f"_l{k // dirs}" + ("_reverse" if k % dirs else "")
            getattr(ref, "weight_ih" + sfx).copy_(w_ih.q)
            getattr(ref, "weight_hh" + sfx).copy_(w_hh.q)
            if bias:
                b = (torch.randn(3 * H, generator=g, device="cuda") * 0.2, torch.randn(3 * H, generator=g, device="cuda") * 0.2)
                getattr(ref, "bias_ih" + sfx).copy_(b[0])
                getattr(ref, "bias_hh" + sfx).copy_(b[1])
                biases.append(b)
    mod = codec.PackedGRU(pairs, "uniform", s, bucket, num_layers=num_layers, batch_first=batch_first, bidirectional=bidirectional,
                          biases=biases if bias else None)
    mod.CROSSOVER_ROWS = N.PACKED_GRU_MAX_ROWS                            # the kernel path up to its 64 rows
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
    """qd_packed_gru_layer over a PackedSequence equals, bit for bit, the cell stepped by hand with the kernel's own
    state (h from the previous active step or h0); each step is inside the oracle's step bound."""
    N, _ = env
    I, H = 37, 29
    w_ih, w_hh, levels = _pair(N, I, H, 2, 4, True, 100, seed=11)
    b_ih, b_hh = torch.randn(3 * H, device="cuda") * 0.3, torch.randn(3 * H, device="cuda") * 0.3
    bs = [sum(L > t for L in lengths) for t in range(lengths[0])]
    off = np.concatenate([[0], np.cumsum(bs)])
    B, total = bs[0], int(off[-1])
    data = torch.randn(total, I, device="cuda")
    h0 = torch.randn(B, H, device="cuda") * 0.5
    out = torch.empty(total, 2 * H, device="cuda")[:, H:]                  # the reverse half of a bidirectional output
    h_n = torch.empty(B, H, device="cuda")
    bsa = np.asarray(bs, np.int64)
    N.check(N.lib().qd_packed_gru_layer(N.ptr(data), I, bsa.ctypes.data, len(bs), int(reverse), I, H, w_ih.desc.ctypes.data,
                                        w_hh.desc.ctypes.data, levels, 100, N.ptr(b_ih), N.ptr(b_hh), N.ptr(h0), N.ptr(out), 2 * H,
                                        N.ptr(h_n), N.stream_ptr()))
    h = h0.clone()
    for t in (reversed(range(len(bs))) if reverse else range(len(bs))):
        m = bs[t]
        x = data[off[t]:off[t] + m]
        h1 = _cell(N, x, h[:m].contiguous(), w_ih, w_hh, levels, 100, b_ih, b_hh)
        assert torch.equal(out[off[t]:off[t] + m], h1), t
        args = [a.cpu().numpy() for a in (x, h[:m], w_ih.q, w_hh.q)]
        ho = O.cell(*args, b_ih.cpu().numpy(), b_hh.cpu().numpy())
        assert np.all(np.abs(h1.cpu().numpy() - ho) <= O.step_tolerance(*args, b_ih.cpu().numpy(), b_hh.cpu().numpy())), t
        h[:m] = h1
    assert torch.equal(h_n, h)


@pytest.mark.parametrize("num_layers,bidirectional,batch_first,with_hx", [(1, False, False, False), (2, True, False, True),
                                                                          (3, False, True, True), (2, True, True, False),
                                                                          (2, False, False, True)])
def test_module_padded_against_cudnn(env, num_layers, bidirectional, batch_first, with_hx):
    N, codec = env
    I, H, T, B = 40, 48, 25, 5
    mod, ref = _gru_module(N, codec, I, H, num_layers, bidirectional, seed=num_layers * 7 + bidirectional, batch_first=batch_first)
    dirs = 2 if bidirectional else 1
    x = torch.randn(B, T, I, device="cuda") if batch_first else torch.randn(T, B, I, device="cuda")
    hx = torch.randn(num_layers * dirs, B, H, device="cuda") * 0.5 if with_hx else None
    with torch.no_grad(), _no_tf32():
        out, h_n = mod(x, hx)
        want, wh = ref(x, hx)
    assert out.shape == want.shape and h_n.shape == wh.shape
    _close(out, want, "output"), _close(h_n, wh, "h_n")
    # the float64 oracle on the kernel's own decoded weights, run from the same start
    flat = [w.cpu().numpy() if w is not None else None for w in mod.decoded_weights()]
    weights = [flat[4 * k:4 * k + 4] for k in range(num_layers * dirs)]
    xs = (x.transpose(0, 1) if batch_first else x).cpu().numpy()
    o, hn = O.gru(xs.reshape(T * B, I), O.padded_batch_sizes(T, B), weights, num_layers, bidirectional,
                  None if hx is None else hx.cpu().numpy())
    got = (out.transpose(0, 1) if batch_first else out).reshape(T * B, -1).cpu().numpy()
    assert np.allclose(got, o, rtol=1e-4, atol=2e-5) and np.allclose(h_n.cpu().numpy(), hn, rtol=1e-4, atol=2e-5)


def test_module_unbatched_and_packed_sequences(env):
    N, codec = env
    I, H, T = 24, 32, 9
    mod, ref = _gru_module(N, codec, I, H, 2, True, bits=4, s=16, bucket=None, seed=3)
    with torch.no_grad(), _no_tf32():
        x = torch.randn(T, I, device="cuda")                                 # unbatched
        out, h_n = mod(x)
        want, wh = ref(x)
        assert out.shape == want.shape == (T, 2 * H) and h_n.shape == wh.shape == (4, H)
        _close(out, want, "unbatched"), _close(h_n, wh, "unbatched h_n")
        hx1 = torch.randn(4, H, device="cuda")
        _close(mod(x, hx1)[0], ref(x, hx1)[0], "unbatched with hx")
        lengths = [9, 2, 7, 1, 9, 4]
        xp = torch.randn(T, len(lengths), I, device="cuda")
        hx = torch.randn(4, len(lengths), H, device="cuda")
        for enforce_sorted in (True, False):
            ls = sorted(lengths, reverse=True) if enforce_sorted else lengths
            ps = torch.nn.utils.rnn.pack_padded_sequence(xp, torch.tensor(ls), enforce_sorted=enforce_sorted)
            for h_start in (None, hx):
                out, h_n = mod(ps, h_start)
                want, wh = ref(ps, h_start)
                assert torch.equal(out.batch_sizes, want.batch_sizes)
                _close(out.data, want.data, "packed"), _close(h_n, wh, "packed h_n")
            # a sequence gives the same bits alone as inside the PackedSequence
            b = 2
            alone, ah = mod(xp[:ls[b], b], hx[:, b])
            padded, _ = torch.nn.utils.rnn.pad_packed_sequence(out)
            assert torch.equal(alone, padded[:ls[b], b]) and torch.equal(ah, h_n[:, b])


def test_cell_module_against_nn_gru_cell(env):
    N, codec = env
    I, H = 1000, 500
    w_ih, w_hh, levels = _pair(N, I, H, 2, 2, True, 256, seed=21)
    b_ih, b_hh = torch.randn(3 * H, device="cuda") * 0.1, torch.randn(3 * H, device="cuda") * 0.1
    cell = codec.PackedGRUCell(w_ih.entry(codec), w_hh.entry(codec), "uniform", levels, 256, b_ih, b_hh)
    cell.CROSSOVER_ROWS = N.PACKED_GRU_MAX_ROWS
    ref = torch.nn.GRUCell(I, H).cuda()
    with torch.no_grad():
        ref.weight_ih.copy_(w_ih.q), ref.weight_hh.copy_(w_hh.q), ref.bias_ih.copy_(b_ih), ref.bias_hh.copy_(b_hh)
        assert all(torch.equal(a, b) for a, b in zip(cell.decoded_weights(), (w_ih.q, w_hh.q)))
        for B in (1, 5, 30, 64):
            x, h = _inputs(B, I, H, B)
            with _no_tf32():
                got, want = cell(x, h), ref(x, h)
            _close(got, want, B)
            assert torch.equal(got, _cell(N, x, h, w_ih, w_hh, levels, 256, b_ih, b_hh))
        x = torch.randn(I, device="cuda")
        h1 = cell(x)
        assert h1.shape == (H,)
        assert torch.equal(h1, cell(x[None], torch.zeros(1, H, device="cuda"))[0])
        x, h = _inputs(65, I, H, 65)                                          # above 64 rows: decode + torch, as unpack_ would
        assert torch.equal(cell(x, h), ref(x, h))


def test_above_crossover_equals_unpack_and_torch(env):
    """Above 64 rows, and with the default CROSSOVER_ROWS above it, the modules decode and call torch: the same bits
    as nn.GRU / nn.GRUCell on the decoded weights."""
    N, codec = env
    mod, ref = _gru_module(N, codec, 32, 40, 2, True, seed=8)
    ref.flatten_parameters()
    default = type(mod).CROSSOVER_ROWS
    with torch.no_grad():
        cases = [(torch.randn(7, 65, 32, device="cuda"), N.PACKED_GRU_MAX_ROWS),
                 (torch.nn.utils.rnn.pack_padded_sequence(torch.randn(7, 70, 32, device="cuda"), torch.randint(1, 8, (70,)),
                                                          enforce_sorted=False), N.PACKED_GRU_MAX_ROWS)]
        if default < N.PACKED_GRU_MAX_ROWS:
            cases.append((torch.randn(7, default + 1, 32, device="cuda"), default))
        for x, crossover in cases:
            mod.CROSSOVER_ROWS = crossover
            out, h_n = mod(x)
            want, wh = ref(x)
            o, w = (out.data, want.data) if isinstance(out, torch.nn.utils.rnn.PackedSequence) else (out, want)
            assert torch.equal(o, w) and torch.equal(h_n, wh)
        w_ih, w_hh, levels = _pair(N, 24, 16, 4, 4, True, 256, seed=9)
        cell = codec.PackedGRUCell(w_ih.entry(codec), w_hh.entry(codec), "uniform", levels, 256)
        rc = torch.nn.GRUCell(24, 16, bias=False).cuda()
        rc.weight_ih.copy_(w_ih.q), rc.weight_hh.copy_(w_hh.q)
        for B in sorted({cell.CROSSOVER_ROWS + 1, 65}):
            x, h = _inputs(B, 24, 16, B)
            assert torch.equal(cell(x, h), rc(x, h))


def test_cuda_graph_replay_of_a_whole_forward(env):
    N, codec = env
    mod, _ = _gru_module(N, codec, 64, 96, 2, True, seed=4)
    x = torch.randn(12, 5, 64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad():
        with torch.cuda.stream(side):
            ref, rh = mod(x)
            ref, rh = ref.clone(), rh.clone()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out, h_n = mod(x)
    for _ in range(3):
        out.zero_()
        h_n.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, ref) and torch.equal(h_n, rh)


# ------------------------------------------------------------------------------------------------ refusals
def test_c_abi_refusals(env):
    N, _ = env
    I, H, m = 6, 5, 3
    w_ih, w_hh, levels = _pair(N, I, H, 2, 2, True, 256, seed=1)
    _, w_bad, _ = _pair(N, I, I, 2, 2, True, 256, seed=1)                 # [3I, I]: not [3H, H]
    w_lstm = W(N, 4 * H, I, 2, levels, None, 256, seed=2)                  # an LSTM's [4H, I]
    x, h = _inputs(m, I, H, 0)
    x, h = x.contiguous(), h.contiguous()
    ho = torch.empty(m, H, device="cuda")
    pts = torch.rand(5, device="cuda")
    L = N.lib()

    def cell(**kw):
        a = dict(x=N.ptr(x), ldx=I, h=N.ptr(h), ldh=H, m=m, I=I, H=H, w_ih=w_ih.desc.ctypes.data, w_hh=w_hh.desc.ctypes.data,
                 levels=levels, bucket=256, b_ih=None, b_hh=None, h_out=N.ptr(ho), ldo=H)
        a.update(kw)
        return L.qd_packed_gru_cell(*a.values(), N.stream_ptr())
    assert cell() == N.QD_OK
    torch.cuda.synchronize()
    bad_bits = w_ih.desc.copy()
    bad_bits["bits"] = 3
    narrow = w_ih.desc.copy()
    narrow["points"], narrow["num_points"] = pts.data_ptr(), 5
    for bad in (dict(x=None), dict(h=None), dict(h_out=None), dict(w_ih=None), dict(w_hh=None),
                dict(m=0), dict(m=-1), dict(I=0), dict(H=0), dict(ldx=I - 1), dict(ldh=H - 1), dict(ldo=H - 1),
                dict(w_hh=w_bad.desc.ctypes.data), dict(w_ih=w_lstm.desc.ctypes.data), dict(w_ih=bad_bits.ctypes.data),
                dict(levels=5), dict(levels=1), dict(levels=0, w_ih=narrow.ctypes.data), dict(levels=0), dict(w_ih=narrow.ctypes.data),
                dict(bucket=-1), dict(h_out=N.ptr(x)), dict(h_out=N.ptr(h)), dict(h_out=N.ptr(h) + 4)):
        assert cell(**bad) == N.QD_ERR_INVALID_ARG, bad
        assert L.qd_last_error().decode()
    assert cell(m=65) == N.QD_ERR_UNSUPPORTED and L.qd_last_error().decode()

    B = 3
    data = torch.randn(9, I, device="cuda")
    out = torch.empty(9, H, device="cuda")
    h0 = torch.zeros(B, H, device="cuda")
    hn = torch.empty(B, H, device="cuda")

    def layer(bs, **kw):
        bsa = np.asarray(bs, np.int64)
        a = dict(x=N.ptr(data), ldx=I, sizes=bsa.ctypes.data, steps=len(bs), reverse=0, I=I, H=H, w_ih=w_ih.desc.ctypes.data,
                 w_hh=w_hh.desc.ctypes.data, levels=levels, bucket=256, b_ih=None, b_hh=None, h0=N.ptr(h0), out=N.ptr(out), ldo=H,
                 h_n=N.ptr(hn))
        a.update(kw)
        return L.qd_packed_gru_layer(*a.values(), N.stream_ptr())
    assert layer([3, 3, 3]) == N.QD_OK and layer([3, 2, 1], reverse=1) == N.QD_OK
    torch.cuda.synchronize()
    for bs, bad in (([3, 3, 3], dict(x=None)), ([3, 3, 3], dict(sizes=None)), ([3, 3, 3], dict(h0=None)), ([3, 3, 3], dict(out=None)),
                    ([3, 3, 3], dict(h_n=None)), ([3], dict(steps=0)), ([2, 3, 1], {}), ([3, 1, 2], {}), ([3, 0], {}),
                    ([3, 3, 3], dict(ldx=I - 1)), ([3, 3, 3], dict(ldo=H - 1)), ([3, 3, 3], dict(out=N.ptr(data))),
                    ([3, 3, 3], dict(h_n=N.ptr(out))), ([3, 3, 3], dict(h_n=N.ptr(h0))), ([3, 3, 3], dict(h_n=N.ptr(data))),
                    ([3, 3, 3], dict(out=N.ptr(h0))), ([3, 3, 3], dict(levels=7)), ([3, 3, 3], dict(w_hh=w_bad.desc.ctypes.data))):
        assert layer(bs, **bad) == N.QD_ERR_INVALID_ARG, (bs, bad)
        assert L.qd_last_error().decode()
    data65 = torch.randn(65, I, device="cuda")
    assert layer([65], x=N.ptr(data65)) == N.QD_ERR_UNSUPPORTED and L.qd_last_error().decode()


def test_module_refusals(env):
    N, codec = env
    mod, _ = _gru_module(N, codec, 8, 6, 2, False, seed=2)
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
        for bad_hx in (torch.zeros(2, 3, 6, device="cuda"), torch.zeros(2, 2, 6), torch.zeros(2, 2, 6, device="cuda").double()):
            with pytest.raises(ValueError):
                mod(x, bad_hx)
    with pytest.raises(RuntimeError, match="forward only"):
        mod(x.clone().requires_grad_())
    with pytest.raises(RuntimeError, match="float32"):
        mod.double()(x)
    w_ih, w_hh, levels = _pair(N, 8, 6, 2, 2, True, 256, seed=3)
    cell = codec.PackedGRUCell(w_ih.entry(codec), w_hh.entry(codec), "uniform", levels, 256)
    with pytest.raises(ValueError):
        cell(torch.randn(3, 8))
    with pytest.raises(ValueError):
        cell(torch.randn(3, 9, device="cuda"))
    with pytest.raises(RuntimeError, match="forward only"):
        cell(torch.randn(3, 8, device="cuda", requires_grad=True))
    with pytest.raises(RuntimeError, match="float32"):
        codec.PackedGRUCell(w_ih.entry(codec), w_hh.entry(codec), "uniform", levels, 256).half()(torch.randn(3, 8, device="cuda"))
    with pytest.raises(ValueError):
        codec.PackedGRUCell(w_hh.entry(codec), w_ih.entry(codec), "uniform", levels, 256)      # [18, 6] ih then [18, 8] hh
    lstm_ih = W(N, 24, 8, 2, levels, None, 256, seed=4)                                        # [4H, I]: an LSTM's, not 3H
    with pytest.raises(ValueError):
        codec.PackedGRUCell(lstm_ih.entry(codec), w_hh.entry(codec), "uniform", levels, 256)
    with pytest.raises(ValueError):
        cell(torch.randn(3, 8, device="cuda"), torch.zeros(2, 6, device="cuda"))


# ------------------------------------------------------------------------------------------------ attaching
class _NMT(torch.nn.Module):
    """The reference's NMT shape built with rnn_type GRU, in small by default: embeddings with a padding index, a
    bidirectional GRU encoder fed a PackedSequence, a StackedGRU-style decoder of nn.GRUCell with input feeding (2d -> d,
    then d -> d), a global-attention nn.Linear and a generator tied to the target embedding."""

    def __init__(self, vs=900, vt=700, d=48, layers=2):
        super().__init__()
        self.src_emb = torch.nn.Embedding(vs, d, padding_idx=1)
        self.tgt_emb = torch.nn.Embedding(vt, d, padding_idx=1)
        self.encoder = torch.nn.GRU(d, d // 2, num_layers=layers, bidirectional=True)
        self.cells = torch.nn.ModuleList([torch.nn.GRUCell(2 * d if i == 0 else d, d) for i in range(layers)])
        self.attn = torch.nn.Linear(2 * d, d, bias=False)
        self.generator = torch.nn.Linear(d, vt)
        self.generator.weight = self.tgt_emb.weight

    def forward(self, src, lengths, tgt):
        ps = torch.nn.utils.rnn.pack_padded_sequence(self.src_emb(src), lengths, enforce_sorted=False)
        mem, h = self.encoder(ps)
        mem = torch.nn.utils.rnn.pad_packed_sequence(mem)[0].transpose(0, 1)                  # [B, S, d]
        h = torch.cat([h[0::2], h[1::2]], 2)
        state = [h[i] for i in range(len(self.cells))]
        feed = torch.zeros_like(state[0])
        logits = []
        for y in self.tgt_emb(tgt):
            inp = torch.cat([y, feed], 1)
            for i, cell in enumerate(self.cells):
                state[i] = cell(inp, state[i])
                inp = state[i]
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


NAMES = ["src_emb", "tgt_emb", "encoder", "cells.0", "cells.1", "attn", "generator"]


def _logits_close(out, want):
    assert torch.allclose(out, want, rtol=1e-4, atol=1e-4 * float(want.abs().max())), float((out - want).abs().max())


@pytest.mark.parametrize("kind", ["uniform", "nonuniform"])
def test_attach_nmt_model(env, kind):
    N, codec = env
    trained = _nmt(0)
    if kind == "uniform":
        pm = codec.pack_model(trained, 4, 256, quantize_first_and_last_layer=True)
    else:
        n_q = len(list(trained.parameters()))
        pts = [np.sort(np.random.default_rng(i).random(3 + i % 14)).astype(np.float32) for i in range(n_q)]
        pm = codec.pack_model(trained, points=pts, bucket_size=256, quantize_first_and_last_layer=True)
    ref = _nmt(1)
    codec.unpack_(pm, ref)
    fresh = _nmt(2)
    enc = fresh.encoder
    released = _blocks({p.data_ptr() for p in enc.parameters()})
    assert len(released) == 1                                             # the GRU's one flattened buffer, biases included
    cell_params = [p for cell in fresh.cells for p in cell.parameters()]
    released.update(_blocks({p.data_ptr() for p in cell_params} | {fresh.src_emb.weight.data_ptr(), fresh.tgt_emb.weight.data_ptr(),
                                                                      fresh.attn.weight.data_ptr()}))
    assert len(released) == 1 + len(cell_params) + 3
    n_bias = 2 * enc.num_layers * 2 + 2 * len(fresh.cells)
    bias_block = -(-4 * 3 * fresh.cells[0].hidden_size // 512) * 512                     # a copied bias's allocator block
    enc_bias_block = -(-4 * 3 * enc.hidden_size // 512) * 512
    new = 2 * 512 + 2 * enc.num_layers * 2 * enc_bias_block + 2 * len(fresh.cells) * bias_block
    del enc, cell_params
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    names = codec.attach_packed_(pm, fresh, embeddings=True, gru=True)
    gc.collect()
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    assert names == NAMES
    assert type(fresh.encoder) is codec.PackedGRU and all(type(c) is codec.PackedGRUCell for c in fresh.cells)
    assert n_bias == sum(1 for n, _ in fresh.named_buffers() if n.endswith(".bias") and (n.startswith("encoder") or n.startswith("cells")))
    # every float32 GRU / GRUCell weight is gone: the encoder's flattened buffer, the cells' four tensors each, both
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
            k = int(lyr[1:]) * 2 + bool(rev)
            assert torch.equal(got[f"encoder.cells.{k}.{0 if which == 'ih' else 1}.bias"], t.data), name
        elif name == "generator.bias":
            assert torch.equal(got["generator.bias"], t.data)
    for k, (ih, hh) in enumerate(fresh.encoder.cells):
        sfx = f"_l{k // 2}" + ("_reverse" if k % 2 else "")
        assert torch.equal(ih.decoded(), getattr(ref.encoder, "weight_ih" + sfx).data)
        assert torch.equal(hh.decoded(), getattr(ref.encoder, "weight_hh" + sfx).data)
    for cell, rc in zip(fresh.cells, ref.cells):
        assert all(torch.equal(a, b) for a, b in zip(cell.decoded_weights(), (rc.weight_ih.data, rc.weight_hh.data)))
    g = torch.Generator(device="cuda").manual_seed(3)
    src, lengths, tgt = _batch(g)
    with torch.no_grad(), _no_tf32():
        want = ref(src, lengths, tgt)
        _logits_close(fresh(src, lengths, tgt), want)
        for m in (fresh.encoder, *fresh.cells):                          # and on the packed kernels
            m.CROSSOVER_ROWS = N.PACKED_GRU_MAX_ROWS
        _logits_close(fresh(src, lengths, tgt), want)


def test_attach_nmt_shapes(env):
    """The NMT widths: d = 500, so the first decoder cell is 1000 -> 500 and the encoder 2 x 250 per layer.  Another
    seed than the other tests; every recurrent module is replaced, no float32 recurrent matrix is left, and the logits
    match the unpack_-loaded model on both paths."""
    N, codec = env
    pm = codec.pack_model(_nmt(10, d=500), 2, 256, quantize_first_and_last_layer=True)
    ref = _nmt(11, d=500)
    codec.unpack_(pm, ref)
    fresh = _nmt(12, d=500)
    assert codec.attach_packed_(pm, fresh, embeddings=True, gru=True) == NAMES
    assert (fresh.cells[0].input_size, fresh.cells[0].hidden_size) == (1000, 500)
    assert not any(p.dim() == 2 for p in fresh.parameters())
    g = torch.Generator(device="cuda").manual_seed(13)
    src, lengths, tgt = _batch(g)
    with torch.no_grad(), _no_tf32():
        want = ref(src, lengths, tgt)
        _logits_close(fresh(src, lengths, tgt), want)
        for m in (fresh.encoder, *fresh.cells):
            m.CROSSOVER_ROWS = N.PACKED_GRU_MAX_ROWS
        _logits_close(fresh(src, lengths, tgt), want)


class _Ineligible(torch.nn.Module):
    """Recurrent modules attach_packed_ must leave to unpack_ even with gru=True: a GRU subclass, two GRUCells sharing a
    weight, a GRU whose first matrix the model keeps float32, and an LSTM (recurrent=False); one plain GRU and one plain
    GRUCell it replaces."""

    class Sub(torch.nn.GRU):
        pass

    def __init__(self):
        super().__init__()
        self.first = torch.nn.GRU(8, 8)                    # the model's first parameter: stored float32
        self.sub = _Ineligible.Sub(8, 8)
        self.shared_a = torch.nn.GRUCell(8, 8)
        self.shared_b = torch.nn.GRUCell(8, 8)
        self.shared_b.weight_ih = self.shared_a.weight_ih
        self.lstm = torch.nn.LSTM(8, 8)
        self.plain = torch.nn.GRU(8, 8, num_layers=2, bidirectional=True)
        self.plain_cell = torch.nn.GRUCell(8, 8, bias=False)
        self.last = torch.nn.Linear(8, 3)


def test_attach_leaves_ineligible_gru_modules_to_unpack(env):
    N, codec = env
    torch.manual_seed(0)
    pm = codec.pack_model(_Ineligible().cuda(), 4, 64, quantize_first_and_last_layer=False)
    torch.manual_seed(1)
    ref = _Ineligible().cuda()
    codec.unpack_(pm, ref)
    torch.manual_seed(2)
    fresh = _Ineligible().cuda()
    assert codec.attach_packed_(pm, fresh, gru=True) == ["plain", "plain_cell", "last"]
    assert type(fresh.first) is torch.nn.GRU and type(fresh.sub) is _Ineligible.Sub and type(fresh.lstm) is torch.nn.LSTM
    assert type(fresh.shared_a) is torch.nn.GRUCell and type(fresh.shared_b) is torch.nn.GRUCell
    assert fresh.shared_b.weight_ih is fresh.shared_a.weight_ih
    assert type(fresh.plain) is codec.PackedGRU and type(fresh.plain_cell) is codec.PackedGRUCell and not fresh.plain_cell.bias
    got = dict(fresh.named_parameters())
    got.update(dict(fresh.named_buffers()))                               # a replaced Linear holds its bias as a buffer
    for name, t in ref.named_parameters():
        if not name.startswith(("plain", "last.weight")):
            assert torch.equal(got[name].data, t.data), name
    x = torch.randn(5, 3, 8, device="cuda")
    with torch.no_grad(), _no_tf32():
        _close(fresh.plain(x)[0], ref.plain(x)[0], "plain")
        _close(fresh.plain_cell(x[0]), ref.plain_cell(x[0]), "plain_cell")
    torch.manual_seed(2)
    both = _Ineligible().cuda()
    assert codec.attach_packed_(pm, both, recurrent=True, gru=True) == ["lstm", "plain", "plain_cell", "last"]
    torch.manual_seed(2)
    default = _Ineligible().cuda()
    assert codec.attach_packed_(pm, default, embeddings=True, recurrent=True) == ["lstm", "last"]  # without gru=True: no GRU
    assert type(default.plain) is torch.nn.GRU and torch.equal(default.plain.weight_ih_l0, ref.plain.weight_ih_l0)
    assert type(default.plain_cell) is torch.nn.GRUCell and torch.equal(default.plain_cell.weight_hh, ref.plain_cell.weight_hh)


def test_attach_huffman_route(env):
    """A Huffman-coded model transcoded to fixed-width codes and attached with gru=True holds the weights decompress_
    writes, and computes the same logits within tolerance."""
    N, codec = env
    cm = codec.compress_model(_nmt(0), 4, bucket_size=256, quantize_first_and_last_layer=True)
    net = _nmt(2)
    assert codec.attach_packed_(codec.pack_compressed(cm), net, embeddings=True, gru=True) == NAMES
    ref = _nmt(1)
    codec.decompress_(cm, ref)
    assert torch.equal(net.encoder.cells[3][1].decoded(), ref.encoder.weight_hh_l1_reverse.data)
    assert torch.equal(net.cells[0].decoded_weights()[0], ref.cells[0].weight_ih.data)
    g = torch.Generator(device="cuda").manual_seed(4)
    src, lengths, tgt = _batch(g)
    with torch.no_grad(), _no_tf32():
        _logits_close(net(src, lengths, tgt), ref(src, lengths, tgt))
