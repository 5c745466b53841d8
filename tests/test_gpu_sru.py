"""The SRU recurrence (qd_sru_fwd / qd_sru_bwd) and the drop-in SRU / SRUCell: the kernels bit for bit against the
reference's own kernels built with -fmad=false (oracle/_ref/libsru_ref_nofma.so, built by oracle/sru_ref_build.py;
those tests skip when it is absent), and, with the default-contraction build, against the float64 oracle
(oracle/sru_oracle.py) within its bounds, over len {1, 2, 50, 200}, batch {1, 3, 64, 320}, d {1, 31, 250, 500, 550},
k 3 and 4, both directions, the three activations, mask_h and init on and off; the kernels against the reference
kernels' CPU fixture (tests/golden/reference_sru.npz); batch invariance, run-to-run bits, CUDA graphs, a side
stream, no synchronisation and NaN guards around offset views; the modules against a per-step torch-chain twin in
train and eval mode; an onmt-protocol SRU encoder-decoder trained one step and translated with beam search against
the same model on the twin; every refusal."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import sru_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
G = 5                               # NaN guard elements on each side of every output


@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native
    return _native


def _ref_lib(name):
    path = os.path.join(REF_DIR, name)
    if not os.path.exists(path):
        pytest.skip(f"{path} not built (oracle/sru_ref_build.py needs a reference checkout)")
    lib = C.CDLL(path)
    lib.sru_ref_fwd.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_int] * 4 + [C.c_void_p] * 2 + [C.c_int, C.c_void_p]
    lib.sru_ref_bwd.argtypes = [C.c_int] + [C.c_void_p] * 8 + [C.c_int] * 4 + [C.c_void_p] * 4 + [C.c_int, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def REF(N):
    return _ref_lib("libsru_ref_nofma.so")


@pytest.fixture(scope="module")
def REF_FMA(N):
    return _ref_lib("libsru_ref.so")


def _guarded(n, offset=0):
    """(buffer, view): n floats starting G + offset floats into a NaN buffer."""
    b = torch.full((n + 2 * G + offset,), float("nan"), device="cuda")
    return b, b[G + offset:G + offset + n]


def _in(shape, g, offset=0, scale=1.0):
    n = int(np.prod(shape))
    b = torch.randn(n + offset, generator=g, device="cuda") * scale
    return b[offset:].view(*shape)


class Case:
    def __init__(self, L, B, d, k, bi, act, mask, init, seed=0, offset=0):
        self.L, self.B, self.d, self.k, self.bi, self.act = L, B, d, k, int(bi), act
        self.D = d * (2 if bi else 1)
        g = torch.Generator(device="cuda").manual_seed(seed)
        D = self.D
        self.u = _in((L, B, D, k), g, offset)
        self.x = _in((L, B, D), g, offset) if k == 3 else None
        self.bias = _in((2 * D,), g, offset, 0.5)
        self.init = _in((B, D), g, offset) if init else None
        self.mask = ((torch.rand(B, D, generator=g, device="cuda") < 0.7).float() / 0.7) if mask else None
        self.gh = _in((L, B, D), g, offset)
        self.gl = _in((B, D), g, offset) if init else None
        self.offset = offset

    def fwd(self, N):
        n = self.L * self.B * self.D
        hb, h = _guarded(n, self.offset)
        cb, c = _guarded(n, self.offset)
        N.check(N.lib().qd_sru_fwd(N.ptr(self.u), N.ptr(self.x), N.ptr(self.bias), N.ptr(self.init), N.ptr(self.mask),
                                   self.L, self.B, self.d, self.k, self.bi, self.act, N.ptr(h), N.ptr(c), N.stream_ptr()))
        for b in (hb, cb):
            assert torch.isnan(b[:G + self.offset]).all() and torch.isnan(b[G + self.offset + n:]).all(), "guard written"
        return h.view(self.L, self.B, self.D), c.view(self.L, self.B, self.D)

    def bwd(self, N, c):
        n, nc = self.L * self.B * self.D, self.B * self.D
        bufs = [_guarded(n * self.k, self.offset), _guarded(n, self.offset) if self.k == 3 else (None, None),
                _guarded(2 * self.D, self.offset), _guarded(nc, self.offset)]
        (_, gu), (_, gx), (_, gb), (_, gi) = bufs
        ws = torch.empty(int(N.lib().qd_sru_workspace_bytes(self.B, self.d, self.bi)), dtype=torch.uint8, device="cuda")
        N.check(N.lib().qd_sru_bwd(N.ptr(self.u), N.ptr(self.x), N.ptr(self.bias), N.ptr(self.init), N.ptr(self.mask),
                                   N.ptr(c), N.ptr(self.gh), N.ptr(self.gl), self.L, self.B, self.d, self.k, self.bi,
                                   self.act, N.ptr(gu), N.ptr(gx), N.ptr(gb), N.ptr(gi), N.ptr(ws), ws.numel(),
                                   N.stream_ptr()))
        for (b, v) in bufs:
            if b is not None:
                off = G + self.offset
                assert torch.isnan(b[:off]).all() and torch.isnan(b[off + v.numel():]).all(), "guard written"
        return {"grad_u": gu.view(self.L, self.B, self.D, self.k), "grad_x": gx, "grad_bias": gb,
                "grad_init": gi.view(self.B, self.D), "partial": ws.view(torch.float32).view(2, self.B, self.D)}

    def ref(self, lib, N):
        zeros = torch.zeros(self.B, self.D, device="cuda")
        init = self.init if self.init is not None else zeros
        gl = self.gl if self.gl is not None else zeros
        n = self.L * self.B * self.D
        h, c = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
        assert lib.sru_ref_fwd(self.bi, N.ptr(self.u), N.ptr(self.x), N.ptr(self.bias), N.ptr(init), N.ptr(self.mask),
                               self.L, self.B, self.d, self.k, N.ptr(h), N.ptr(c), self.act, N.stream_ptr()) == 0
        gu = torch.empty(n * self.k, device="cuda")
        gx = torch.empty(n, device="cuda") if self.k == 3 else None
        gb, gi = torch.empty(2, self.B, self.D, device="cuda"), torch.empty(self.B, self.D, device="cuda")
        assert lib.sru_ref_bwd(self.bi, N.ptr(self.u), N.ptr(self.x), N.ptr(self.bias), N.ptr(init), N.ptr(self.mask),
                               N.ptr(c), N.ptr(self.gh), N.ptr(gl), self.L, self.B, self.d, self.k, N.ptr(gu), N.ptr(gx),
                               N.ptr(gb), N.ptr(gi), self.act, N.stream_ptr()) == 0
        return {"h": h.view(self.L, self.B, self.D), "c": c.view(self.L, self.B, self.D),
                "grad_u": gu.view(self.L, self.B, self.D, self.k), "grad_x": gx, "partial": gb, "grad_init": gi}

    def oracle(self):
        np_ = lambda t: None if t is None else t.double().cpu().numpy()  # noqa: E731
        vals, errs = O.sru(np_(self.u), np_(self.x), np_(self.bias), self.d, bool(self.bi), self.act, init=np_(self.init),
                           mask_h=np_(self.mask), grad_h=np_(self.gh), grad_last=np_(self.gl))
        return vals, O.bounds(errs, self.L)


def _same(a, b, what):
    assert a.shape == b.shape, what
    eq = (a.view(torch.int32) == b.view(torch.int32))
    assert bool(eq.all()), f"{what}: {int((~eq).sum())} of {eq.numel()} elements differ"


def _sequential_sum(partial):
    """grad_bias as the kernels sum it: over the batch in b order, float32."""
    p = partial.cpu().numpy()
    s = np.zeros(p.shape[0::2], np.float32)
    for b in range(p.shape[1]):
        s = s + p[:, b]
    return torch.from_numpy(s.reshape(-1))


def _within(got, want, bound, what):
    err = np.abs(got.double().cpu().numpy() - want)
    assert np.all(err <= bound), f"{what}: max err {err.max():.3e}, worst err/bound {(err / bound).max():.3f}"


# every (len, batch, d); the (k, direction, activation, mask, init) settings cycle over them, each shape running four
SHAPES = list(itertools.product([1, 2, 50, 200], [1, 3, 64, 320], [1, 31, 250, 500, 550]))
MAX_U = 1 << 26                     # floats of u per case: above it a shape runs only its first setting


def _settings(i):
    kb = [(4, 0), (3, 0), (4, 1), (3, 1)]
    return [(k, bi, (i + j) % 3, (i + j) % 2 == 0, (i + j // 2) % 2 == 1) for j, (k, bi) in enumerate(kb)]


@pytest.mark.parametrize("L,B,d", SHAPES)
def test_kernels_bit_identical_to_reference_kernels(N, REF, L, B, d):
    i = SHAPES.index((L, B, d))
    ran = 0
    for k, bi, act, mask, init in _settings(i):
        if L * B * d * (2 if bi else 1) * k > MAX_U and ran:
            continue
        cs = Case(L, B, d, k, bi, act, mask, init, seed=i)
        h, c = cs.fwd(N)
        got = cs.bwd(N, c)
        want = cs.ref(REF, N)
        tag = f"L={L} B={B} d={d} k={k} bi={bi} act={act} mask={mask} init={init}"
        _same(h, want["h"], "h " + tag)
        _same(c, want["c"], "c " + tag)
        _same(got["grad_u"], want["grad_u"], "grad_u " + tag)
        if k == 3:
            _same(got["grad_x"], want["grad_x"].view(-1), "grad_x " + tag)
        _same(got["grad_init"], want["grad_init"], "grad_init " + tag)
        _same(got["partial"], want["partial"], "bias partials " + tag)
        _same(got["grad_bias"].cpu(), _sequential_sum(want["partial"]), "grad_bias " + tag)
        ran += 1


ORACLE_SHAPES = [(1, 3, 31), (2, 1, 1), (2, 64, 31), (50, 3, 31), (50, 1, 250), (200, 3, 1), (50, 64, 1), (2, 320, 31)]


@pytest.mark.parametrize("L,B,d", ORACLE_SHAPES)
def test_kernels_and_default_fmad_reference_within_oracle_bounds(N, REF_FMA, L, B, d):
    i = ORACLE_SHAPES.index((L, B, d))
    for k, bi, act, mask, init in _settings(i):
        for offset in (0, 1):
            cs = Case(L, B, d, k, bi, act, mask, init, seed=100 + i, offset=offset)
            h, c = cs.fwd(N)
            got = dict(cs.bwd(N, c), h=h, c=c)
            fma = cs.ref(REF_FMA, N)
            fma["grad_bias"] = fma["partial"].double().sum(1).view(-1)
            vals, bnd = cs.oracle()
            tag = f" L={L} B={B} d={d} k={k} bi={bi} act={act} offset={offset}"
            for name in ("h", "c", "grad_u", "grad_init", "grad_bias") + (("grad_x",) if k == 3 else ()):
                want = vals[name].reshape(-1)
                _within(got[name].reshape(-1), want, bnd[name].reshape(-1), name + tag)
                _within(fma[name].reshape(-1), want, bnd[name].reshape(-1), "default-fmad reference " + name + tag)


def test_kernels_match_the_reference_cpu_fixture(N):
    data = np.load(os.path.join(HERE, "golden", "reference_sru.npz"))
    for i, (bi, k, act, mask, L, B, d, _, _) in enumerate(data["cases"].tolist()):
        f = {key[len(f"c{i}_"):]: data[key] for key in data.files if key.startswith(f"c{i}_")}
        cs = Case(L, B, d, k, bi, act, False, False)
        cuda = lambda a: torch.from_numpy(a).cuda()  # noqa: E731
        cs.u, cs.x, cs.bias = cuda(f["u"]), cuda(f["x"]) if "x" in f else None, cuda(f["bias"])
        cs.init, cs.gh, cs.gl = cuda(f["init"]), cuda(f["grad_h"]), cuda(f["grad_last"])
        cs.mask = cuda(f["mask_h"]) if "mask_h" in f else None
        h, c = cs.fwd(N)
        got = dict(cs.bwd(N, c), h=h, c=c)
        vals, bnd = cs.oracle()
        fixture = dict(f, grad_bias=f["grad_bias_partial"].astype(np.float64).sum(1).reshape(-1))
        for name in ("h", "c", "grad_u", "grad_init", "grad_bias") + (("grad_x",) if k == 3 else ()):
            _within(got[name].reshape(-1), vals[name].reshape(-1), bnd[name].reshape(-1), f"case {i} {name}")
            # kernel and fixture are both within the bound of the exact value: within twice of each other
            err = np.abs(got[name].double().cpu().numpy().reshape(-1) - fixture[name].reshape(-1))
            assert np.all(err <= 2 * bnd[name].reshape(-1)), f"case {i} {name} against the CPU-compiled reference"


# ---- bit properties ------------------------------------------------------------------------------------------------
def test_columns_alone_and_in_a_batch_and_across_runs(N):
    for k, bi in ((4, 1), (3, 0)):
        cs = Case(20, 64, 250, k, bi, 1, True, True, seed=7)
        h, c = cs.fwd(N)
        g = cs.bwd(N, c)
        for b in (0, 17, 63):
            one = Case(20, 1, 250, k, bi, 1, True, True)
            one.u, one.bias = cs.u[:, b:b + 1].contiguous(), cs.bias
            one.x = cs.x[:, b:b + 1].contiguous() if k == 3 else None
            one.init, one.mask, one.gh, one.gl = (t[..., b:b + 1, :].contiguous() for t in (cs.init, cs.mask, cs.gh, cs.gl))
            h1, c1 = one.fwd(N)
            g1 = one.bwd(N, c1)
            _same(h1[:, 0], h[:, b], "h alone")
            _same(g1["grad_u"][:, 0], g["grad_u"][:, b], "grad_u alone")
            _same(g1["grad_init"][0], g["grad_init"][b], "grad_init alone")
        h2, c2 = cs.fwd(N)
        g2 = cs.bwd(N, c2)
        _same(h2, h, "h run to run")
        for key in ("grad_u", "grad_bias", "grad_init"):
            _same(g2[key], g[key], key + " run to run")


def test_graph_replay_side_stream_and_no_sync(N):
    from quantized_distillation_b200.sru import SRU
    torch.manual_seed(0)
    m = SRU(500, 250, num_layers=2, bidirectional=True).cuda()
    x = torch.randn(50, 64, 500, device="cuda", requires_grad=True)
    c0 = torch.randn(2, 64, 500, device="cuda", requires_grad=True)

    def step():
        h, fh = m(x, c0)
        (h.sum() + (fh * fh).sum()).backward()
        return h, fh

    h0, f0 = step()
    want = (h0.detach().clone(), f0.detach().clone(), x.grad.clone(), c0.grad.clone(), m.rnn_lst[0].weight.grad.clone(),
            m.rnn_lst[1].bias.grad.clone())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        x.grad = c0.grad = None
        m.zero_grad(set_to_none=True)
        step()
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(x.grad, want[2]) and torch.equal(c0.grad, want[3]) and torch.equal(m.rnn_lst[1].bias.grad, want[5])
    torch.cuda.set_sync_debug_mode("error")
    try:
        x.grad = c0.grad = None
        m.zero_grad(set_to_none=True)
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        # the leaves are made on the side stream: autograd syncs a leaf's own stream with the capture, which the
        # legacy default stream of the module's parameters cannot join
        xs, cs = x.detach().clone().requires_grad_(True), c0.detach().clone().requires_grad_(True)

        def grads():
            h, fh = m(xs, cs)
            return (h, fh) + torch.autograd.grad(h.sum() + (fh * fh).sum(), [xs, cs])

        grads()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        static = grads()
    g.replay()
    torch.cuda.synchronize()
    for got, w in zip(static, want[:4]):
        assert torch.equal(got, w)


# ---- the modules against a per-step torch chain ----------------------------------------------------------------------
def _chain(u, x, bias, d, bi, act, init, mask_h):
    """The reference's recurrence in stock torch ops, one step at a time; x is [len, batch, n_in] or [batch, n_in]."""
    three_d = x.dim() == 3
    xx = x if three_d else x.unsqueeze(0)
    L, B = xx.shape[0], xx.shape[1]
    dir_ = 2 if bi else 1
    D = dir_ * d
    k = u.shape[-1] // D
    u4 = u.view(L, B, D, k)
    xh = u4[..., 3] if k == 4 else xx
    g1 = torch.sigmoid(u4[..., 1] + bias[:D])
    g2 = torch.sigmoid(u4[..., 2] + bias[D:])
    cur0 = init if init is not None else xx.new_zeros(B, D)
    parts = []
    for r in range(dir_):
        sl = slice(r * d, (r + 1) * d)
        cur, cs = cur0[:, sl], [None] * L
        for t in (range(L) if r == 0 else range(L - 1, -1, -1)):
            cur = (cur - u4[t, :, sl, 0]) * g1[t, :, sl] + u4[t, :, sl, 0]
            cs[t] = cur
        parts.append(torch.stack(cs))
    c = torch.cat(parts, 2)
    a = torch.tanh(c) if act == 1 else (torch.relu(c) if act == 2 else c)
    h = (a * (mask_h if mask_h is not None else 1.0) - xh) * g2 + xh
    if not three_d:
        return h[0], c[0]
    last = torch.stack((c[-1, :, :d], c[0, :, d:])) if bi else c[-1]
    return h, last


def _twin_cell_forward(self, input, c0=None):
    batch = input.size(-2)
    if self.training and self.rnn_dropout > 0:
        x = input * self.get_dropout_mask_((batch, self.n_in), self.rnn_dropout).expand_as(input)
    else:
        x = input
    u = (x if x.dim() == 2 else x.contiguous().view(-1, self.n_in)).mm(self.weight)
    mask_h = None
    if self.training and self.dropout > 0:
        mask_h = self.get_dropout_mask_((batch, self.n_out * (2 if self.bidirectional else 1)), self.dropout)
    return _chain(u, input, self.bias, self.n_out, self.bidirectional, self.activation_type, c0, mask_h)


def _twin(module):
    """module's twin: the same class and parameters, with every SRUCell running the torch chain."""
    from quantized_distillation_b200.sru import SRUCell
    import copy
    twin = copy.deepcopy(module)
    for m in twin.modules():
        if isinstance(m, SRUCell):
            m.forward = _twin_cell_forward.__get__(m)
    return twin


def _grads_close(a, b, what, rel=2e-5):
    scale = b.abs().max().item() + 1e-6
    assert (a - b).abs().max().item() <= rel * scale, f"{what}: {(a - b).abs().max().item():.3e} against scale {scale:.3e}"


@pytest.mark.parametrize("bi,use_tanh,use_relu,n_in", [(True, 1, 0, 48), (False, 1, 0, 32), (False, 0, 1, 40), (True, 0, 0, 64)])
@pytest.mark.parametrize("train", [True, False])
def test_module_matches_torch_chain(N, bi, use_tanh, use_relu, n_in, train):
    from quantized_distillation_b200.sru import SRU
    torch.manual_seed(5)
    m = SRU(n_in, 32, num_layers=3, dropout=0.3, rnn_dropout=0.2, bidirectional=bi, use_tanh=use_tanh,
            use_relu=use_relu).cuda()
    m.set_bias(-0.5)
    m.train(train)
    twin = _twin(m)
    x = torch.randn(9, 5, n_in, device="cuda")
    c0 = torch.randn(3, 5, 64 if bi else 32, device="cuda")
    outs = []
    for mod in (m, twin):
        xi, ci = x.clone().requires_grad_(True), c0.clone().requires_grad_(True)
        torch.cuda.manual_seed(11)
        h, fh = mod(xi, (ci,))
        ((h * h).sum() + fh.sum()).backward()
        outs.append((h.detach(), fh.detach(), xi.grad, ci.grad, {k: p.grad.clone() for k, p in mod.named_parameters()}))
    (h1, f1, gx1, gc1, gp1), (h2, f2, gx2, gc2, gp2) = outs
    assert f1.shape == ((6 if bi else 3), 5, 32)
    _grads_close(h1, h2, "h", 1e-5)
    _grads_close(f1, f2, "fh", 1e-5)
    _grads_close(gx1, gx2, "grad input")
    _grads_close(gc1, gc2, "grad c0")
    for k in gp2:
        _grads_close(gp1[k], gp2[k], k)


def test_state_dict_strict_loading_and_2d_input(N):
    from quantized_distillation_b200.sru import SRU, SRUCell
    m = SRU(20, 8, num_layers=2, bidirectional=True).cuda()
    assert sorted(m.state_dict()) == ["rnn_lst.0.bias", "rnn_lst.0.weight", "rnn_lst.1.bias", "rnn_lst.1.weight"]
    assert m.rnn_lst[0].weight.shape == (20, 4 * 8 * 2) and m.rnn_lst[1].weight.shape == (16, 3 * 8 * 2)
    assert m.rnn_lst[0].bias.shape == (32,)
    m2 = SRU(20, 8, num_layers=2, bidirectional=True).cuda()
    m2.load_state_dict(m.state_dict(), strict=True)
    m.eval(), m2.eval()
    x = torch.randn(4, 3, 20, device="cuda")
    assert torch.equal(m(x)[0], m2(x)[0]) and m(x, return_hidden=False).shape == (4, 3, 16)
    for bi, n_in in ((False, 8), (False, 5), (True, 16), (True, 7)):
        cell = SRUCell(n_in, 8, bidirectional=bi).cuda()
        twin = _twin(cell)
        x2 = torch.randn(6, n_in, device="cuda", requires_grad=True)
        c0 = torch.randn(6, 16 if bi else 8, device="cuda", requires_grad=True)
        h, c = cell(x2, c0)
        h_t, c_t = twin(x2, c0)
        _grads_close(h, h_t, "2-D h", 1e-5)
        _grads_close(c, c_t, "2-D c", 1e-5)
        ga = torch.autograd.grad((h * h).sum() + (c * c).sum(), [x2, c0, cell.weight])
        gb = torch.autograd.grad((h_t * h_t).sum() + (c_t * c_t).sum(), [x2, c0, twin.weight])
        for a, b in zip(ga, gb):
            _grads_close(a, b, "2-D grads")


# ---- end to end: an onmt-protocol SRU encoder-decoder --------------------------------------------------------------
E, H_M, V_M, LAYERS = 16, 32, 61, 2
BOS, EOS, PAD = 2, 3, 1


class _State:
    """onmt's RNNDecoderState for an SRU: hidden is a one-tensor tuple."""

    def __init__(self, hidden, B):
        self.hidden = (hidden,)
        self.input_feed = hidden.new_zeros(1, B, H_M)

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
    """onmt's RNNEncoder with rnn_type 'SRU': bidirectional, no packed sequences."""

    def __init__(self):
        super().__init__()
        from quantized_distillation_b200.sru import SRU
        self.embeddings = nn.Embedding(V_M, E, padding_idx=PAD)
        self.rnn = SRU(E, H_M // 2, num_layers=LAYERS, dropout=0.2, bidirectional=True)

    def forward(self, src, lengths=None):
        outputs, hidden_t = self.rnn(self.embeddings(src.squeeze(-1) if src.dim() == 3 else src))
        return hidden_t, outputs


class _Decoder(nn.Module):
    """onmt's StdRNNDecoder with rnn_type 'SRU' and "general" attention."""

    def __init__(self):
        super().__init__()
        from quantized_distillation_b200.attention import GlobalAttention
        from quantized_distillation_b200.sru import SRU
        self.embeddings = nn.Embedding(V_M, E, padding_idx=PAD)
        self.rnn = SRU(E, H_M, num_layers=LAYERS, dropout=0.2)
        self.attn = GlobalAttention(H_M, attn_type="general")

    def init_decoder_state(self, src, context, enc_hidden):
        h = torch.cat([enc_hidden[0:enc_hidden.size(0):2], enc_hidden[1:enc_hidden.size(0):2]], 2)
        return _State(h, context.shape[1])

    def forward(self, inp, context, state):
        emb = self.embeddings(inp.squeeze(-1))
        rnn_output, hidden = self.rnn(emb, state.hidden)
        attn_outputs, attn_scores = self.attn(rnn_output.transpose(0, 1).contiguous(), context.transpose(0, 1))
        state.hidden = (hidden,)
        return attn_outputs, state, {"std": attn_scores}


class _Model(nn.Module):
    def __init__(self, seed):
        torch.manual_seed(seed)
        super().__init__()
        self.encoder, self.decoder = _Encoder(), _Decoder()
        self.generator = nn.Sequential(nn.Linear(H_M, V_M), nn.LogSoftmax(dim=-1))
        with torch.no_grad():
            self.generator[0].bias[EOS] += 2.5
        self.cuda()


def _src(seed, B=6, S=7):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.full((B,), S)
    return torch.randint(4, V_M, (S, B), generator=g).cuda(), lengths


def test_training_step_with_loss_and_quantizer_matches_torch_chain(N):
    import types
    from quantized_distillation_b200.cnn_models.conv_forward_model import WeightQuantizer
    from quantized_distillation_b200.nmt_loss import NMTLossCompute
    fused = _Model(0)
    ref = _twin(fused)
    src, lengths = _src(0)
    tgt = torch.randint(4, V_M, (9, src.shape[1]), generator=torch.Generator().manual_seed(1)).cuda()
    res = []
    for m in (fused, ref):
        m.train()
        wq = WeightQuantizer(m, 8, 256, backprop_quantization_style="truncated")
        wq.quantize_weights_model()
        torch.cuda.manual_seed(3)
        enc, context = m.encoder(src, lengths)
        state = m.decoder.init_decoder_state(src, context, enc)
        out, _, attn = m.decoder(tgt[:-1].unsqueeze(-1), context, state)
        loss, stats = NMTLossCompute(m.generator, types.SimpleNamespace(stoi={"<blank>": PAD})).compute_loss(None, out, tgt[1:])
        loss.backward()
        wq.restore_weights_model()
        wq.backward_quant_weights_model()
        res.append((loss.item(), out.detach(), {k: p.grad.clone() for k, p in m.named_parameters()}))
    (l1, o1, g1), (l2, o2, g2) = res
    assert abs(l1 - l2) <= 1e-5 * abs(l2)
    _grads_close(o1, o2, "decoder output", 1e-5)
    for k in g2:
        _grads_close(g1[k], g2[k], k, 1e-4)
    assert any(k.startswith("encoder.rnn.rnn_lst") for k in g1) and g1["encoder.rnn.rnn_lst.0.weight"].abs().sum() > 0


@pytest.mark.parametrize("K,n_best,max_len", [(5, 1, 12), (4, 3, 8)])
def test_beam_search_same_hypotheses_as_torch_chain(N, K, n_best, max_len):
    from quantized_distillation_b200.beam import beam_search
    fused = _Model(3)
    ref = _twin(fused)
    fused.eval(), ref.eval()
    src, lengths = _src(K)
    got = beam_search(fused, src, lengths, K, n_best, max_len, bos=BOS, eos=EOS, pad=PAD)
    want = beam_search(ref, src, lengths, K, n_best, max_len, bos=BOS, eos=EOS, pad=PAD)
    assert got[0] == want[0]
    for gs, ws in zip(got[1], want[1]):
        assert np.allclose(np.array(gs, np.float64), np.array(ws, np.float64), rtol=1e-5, atol=1e-5)


# ---- refusals ------------------------------------------------------------------------------------------------------
def test_c_abi_refusals_leave_outputs_untouched(N):
    lib, st = N.lib(), N.stream_ptr()
    L, B, d = 3, 2, 4
    cs = Case(L, B, d, 4, 1, 1, True, True)
    cs3 = Case(L, B, d, 3, 1, 1, True, True)
    D, n = cs.D, L * B * cs.D
    h, c = torch.full((n,), float("nan"), device="cuda"), torch.full((n,), float("nan"), device="cuda")
    P = N.ptr

    def fwd(u=None, x=0, bias=None, ln=L, b=B, dd=d, k=4, bi=1, act=1, hp=None, cp=None):
        return lib.qd_sru_fwd(P(cs.u) if u is None else u, x or None, P(cs.bias) if bias is None else bias, P(cs.init),
                              P(cs.mask), ln, b, dd, k, bi, act, P(h) if hp is None else hp, P(c) if cp is None else cp, st)

    bad = [dict(k=3), dict(k=5), dict(k=2), dict(ln=0), dict(b=0), dict(dd=0), dict(ln=-1), dict(bi=2), dict(act=3),
           dict(act=-1), dict(x=P(cs3.x)), dict(u=0), dict(bias=0), dict(hp=0), dict(cp=0), dict(hp=P(h) + 2),
           dict(hp=P(cs.u)), dict(cp=P(h) + 4), dict(ln=1 << 62)]
    for kw in bad:
        assert fwd(**kw) == N.QD_ERR_INVALID_ARG, kw
    torch.cuda.synchronize()
    assert torch.isnan(h).all() and torch.isnan(c).all(), "a refused call wrote its outputs"
    assert lib.qd_sru_fwd(P(cs3.u), None, P(cs3.bias), None, None, L, B, d, 3, 1, 1, P(h), P(c), st) == N.QD_ERR_INVALID_ARG
    assert fwd() == N.QD_OK
    hh, cc = cs.fwd(N)
    assert torch.equal(h.view(L, B, D), hh) and torch.equal(c.view(L, B, D), cc)

    need = int(lib.qd_sru_workspace_bytes(B, d, 1))
    assert need == 2 * B * D * 4 and lib.qd_sru_workspace_bytes(0, d, 1) == 0
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    gu = torch.full((n * 4,), float("nan"), device="cuda")
    gb, gi = torch.full((2 * D,), float("nan"), device="cuda"), torch.full((B * D,), float("nan"), device="cuda")

    def bwd(k=4, x=0, gx=0, wp=None, wn=need, gup=None, ghp=None, gbp=None):
        return lib.qd_sru_bwd(P(cs.u), x or None, P(cs.bias), P(cs.init), P(cs.mask), P(c), P(cs.gh) if ghp is None else ghp,
                              P(cs.gl), L, B, d, k, 1, 1, P(gu) if gup is None else gup, gx or None,
                              P(gb) if gbp is None else gbp, P(gi), P(ws) if wp is None else wp, wn, st)

    assert bwd(wn=need - 1) == N.QD_ERR_WORKSPACE
    assert bwd(wp=0) == N.QD_ERR_WORKSPACE
    assert bwd(wp=P(ws) + 2) == N.QD_ERR_WORKSPACE
    for kw in (dict(k=3), dict(gx=P(gi)), dict(x=P(cs3.x)), dict(gup=0), dict(ghp=0), dict(gbp=0), dict(gup=P(c)),
               dict(gbp=P(gu) + 8), dict(wp=P(gu)), dict(gup=P(gu) + 2)):
        assert bwd(**kw) == N.QD_ERR_INVALID_ARG, kw
    torch.cuda.synchronize()
    assert torch.isnan(gu).all() and torch.isnan(gb).all() and torch.isnan(gi).all(), "a refused call wrote its outputs"
    assert bwd() == N.QD_OK


def test_python_refusals(N):
    from quantized_distillation_b200.sru import SRU, SRUCell, sru_compute
    m = SRU(8, 4).cuda()
    x = torch.randn(3, 2, 8, device="cuda")
    with pytest.raises(ValueError):
        m(x.cpu())
    with pytest.raises(ValueError):
        m(x.double())
    with pytest.raises(ValueError):
        m(x[0])
    with pytest.raises(ValueError):
        m(x, torch.zeros(2, 4, device="cuda"))
    with pytest.raises(ValueError):
        SRU(8, 4)(x.cpu())
    with pytest.raises(ValueError):
        SRUCell(8, 4).cuda()(torch.randn(3, 2, 2, 8, device="cuda"))
    u = torch.randn(6, 16, device="cuda")
    bias = torch.zeros(8, device="cuda")
    sru_compute(u, x, bias, 4, False, 1)
    for args in ((u, x, bias, 4, False, 3), (u[:, :12], x, bias, 4, False, 1), (u, x, bias[:6], 4, False, 1),
                 (u.cpu(), x.cpu(), bias.cpu(), 4, False, 1), (u, x, bias, 0, False, 1), (u, x.half(), bias, 4, False, 1)):
        with pytest.raises(ValueError):
            sru_compute(*args)
    with pytest.raises(ValueError):
        sru_compute(u, x, bias, 4, False, 1, init=torch.zeros(3, 4, device="cuda"))
