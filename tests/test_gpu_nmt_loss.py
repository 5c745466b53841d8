"""The fused NMT loss (qd_nmt_loss_fwd / qd_nmt_loss_bwd, nmt_loss, NMTLossCompute) against the float64 oracle at every
row-length class (1 to 50,004, around the 4-column group and the 256-thread CTA), 0 to 3,264 rows, teacher on and off,
padding none / 0 / 1 and offset views; against the float32 torch chain of the reference; through autograd with a
gradient other than 1; bit properties (a row alone and in a batch, two runs, CUDA graph replay); invalid targets;
refusals; the memory of forward + backward; and NMTLossCompute.sharded_compute_loss against the reference's sharded
torch path."""
import types

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import nmt_loss_oracle as O

pytestmark = pytest.mark.gpu

VS = [1, 2, 3, 4, 5, 1023, 1024, 1025, 4097, 10_004, 24_999, 50_004]
W = 0.7


@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native
    return _native


def _alloc(shape, offset, dtype=torch.float32):
    """A contiguous tensor of `shape` starting `offset` elements into a larger buffer (offset 1: no row 16-byte aligned
    when the row length is a multiple of 4)."""
    n = int(np.prod(shape))
    return torch.empty(n + offset, dtype=dtype, device="cuda")[offset:].view(shape)


def _inputs(R, V, teacher, padding_idx, offset, seed, masked=False):
    """masked: a masked vocabulary, -inf logits in both rows -- every thread's first group of four columns where the row
    is longer than one group per thread, a quarter of the other columns at random, a few columns -inf in the teacher
    alone -- with column V-1 always finite and the targets on finite student columns."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    zs = _alloc((R, V), offset)
    zs.copy_(torch.randn(R, V, generator=g, device="cuda") * 2)
    zt = None
    if teacher:
        zt = _alloc((R, V), offset)
        zt.copy_(torch.randn(R, V, generator=g, device="cuda") * 2)
    y = torch.randint(0, V, (R,), generator=g, device="cuda")
    if masked and R > 0:
        mask = torch.rand(R, V, generator=g, device="cuda") < 0.25
        if V > 4 * 256:
            mask[:, :4 * 256] = True
        mask[:, V - 1] = False
        zs.masked_fill_(mask, float("-inf"))
        if teacher:
            zt.masked_fill_(mask | ((torch.rand(R, V, generator=g, device="cuda") < 0.1) & (torch.arange(V, device="cuda") < V - 1)),
                            float("-inf"))
        finite = ~mask
        y = torch.where(finite.gather(1, y[:, None])[:, 0], y, torch.full_like(y, V - 1))
    if padding_idx >= 0 and R > 0:
        y[::5] = padding_idx
    return zs, zt, y


def _fwd(N, zs, zt, y, padding_idx, w=W):
    R, V = zs.shape
    row_lse = torch.full((R, 2), float("nan"), device="cuda")
    loss = torch.full((), float("nan"), device="cuda")
    counts = torch.full((3,), -1, dtype=torch.int64, device="cuda")
    ws = torch.empty(max(int(N.lib().qd_nmt_loss_workspace_bytes(R)), 1), dtype=torch.uint8, device="cuda")
    N.check(N.lib().qd_nmt_loss_fwd(N.ptr(zs), N.ptr(zt), N.ptr(y), R, V, padding_idx, w, N.ptr(row_lse), N.ptr(loss),
                                    N.ptr(counts), N.ptr(ws), ws.numel(), N.stream_ptr()))
    return row_lse, loss, counts


def _bwd(N, zs, zt, y, row_lse, g, padding_idx, w=W, offset=0):
    R, V = zs.shape
    grad = _alloc((R, V), offset)
    grad.fill_(float("nan"))
    gd = torch.tensor(g, dtype=torch.float32, device="cuda")
    N.check(N.lib().qd_nmt_loss_bwd(N.ptr(zs), N.ptr(zt), N.ptr(y), N.ptr(row_lse), N.ptr(gd), R, V, padding_idx, w, N.ptr(grad),
                                    N.stream_ptr()))
    return grad


def _lse_tol(lse_ref, zs):
    # 4 ulp of max(|lse|, |m|, 1): lse = m + log(S), and S sums float32 expf terms whose relative error (2 ulp each, and
    # the rounding of z - m) is an absolute error of log(S), so the bound scales with m and 1 as well as with lse
    m = np.abs(np.where(np.isfinite(zs), zs, 0.0)).max(axis=1, initial=0.0) if zs.size else np.zeros(len(lse_ref))
    return 4 * 2.0 ** -23 * np.maximum(np.maximum(np.abs(lse_ref), m), 1.0)


def _compare(N, R, V, teacher, padding_idx, offset, seed, g=1.0, chunk_elems=1 << 22, masked=False):
    zs, zt, y = _inputs(R, V, teacher, padding_idx, offset, seed, masked)
    row_lse, loss, counts = _fwd(N, zs, zt, y, padding_idx)
    grad = _bwd(N, zs, zt, y, row_lse, g, padding_idx, offset=offset)
    torch.cuda.synchronize()
    lse_h, grad_h, y_h = row_lse.cpu().numpy(), grad, y.cpu().numpy()
    ref_loss, ref_abs, ref_counts = 0.0, 0.0, np.zeros(3, np.int64)
    step = max(1, chunk_elems // V)
    for r0 in range(0, R, step):
        r1 = min(R, r0 + step)
        zs_c = zs[r0:r1].cpu().numpy()
        zt_c = None if zt is None else zt[r0:r1].cpu().numpy()
        o = O.nmt_loss(zs_c, y_h[r0:r1], padding_idx, zt_c, W, grad_loss=g)
        ref_loss += o["loss"]
        ref_abs += np.abs(o["row_loss"]).sum()
        ref_counts += o["counts"]
        tol = _lse_tol(o["row_lse"][:, 0], zs_c)
        assert np.all(np.abs(lse_h[r0:r1, 0] - o["row_lse"][:, 0]) <= tol), (R, V, r0)
        if teacher:
            tol_t = _lse_tol(o["row_lse"][:, 1], zt_c)
            assert np.all(np.abs(lse_h[r0:r1, 1] - o["row_lse"][:, 1]) <= tol_t), (R, V, r0)
        gc = grad_h[r0:r1].cpu().numpy().astype(np.float64)
        assert np.all(np.abs(gc - o["grad"]) <= 2e-6 * abs(g)), (R, V, r0, np.abs(gc - o["grad"]).max())
    assert list(counts.cpu().numpy()) == list(ref_counts), (R, V)
    got = float(loss.cpu())
    assert abs(got - ref_loss) <= 1e-5 * max(ref_abs, 1e-30) + 1e-30, (R, V, got, ref_loss)


@pytest.mark.parametrize("teacher", [False, True], ids=["plain", "teacher"])
@pytest.mark.parametrize("V", VS)
def test_against_oracle_small_batches(N, V, teacher):
    for R in (0, 1, 3, 64):
        for padding_idx in (-1, 0, 1):
            if padding_idx >= V:
                continue
            for offset in (0, 1):
                _compare(N, R, V, teacher, padding_idx, offset, seed=V * 7 + R + padding_idx)


@pytest.mark.parametrize("teacher", [False, True], ids=["plain", "teacher"])
@pytest.mark.parametrize("V", [1023, 4097, 10_004, 24_999, 50_004])
def test_against_oracle_training_batch(N, V, teacher):
    _compare(N, 3264, V, teacher, 1, offset=V % 2, seed=V)


@pytest.mark.parametrize("teacher", [False, True], ids=["plain", "teacher"])
@pytest.mark.parametrize("V", [3, 5, 1025, 4097, 50_004])
def test_against_oracle_masked_vocabulary(N, V, teacher):
    for R, padding_idx, offset in ((1, -1, 0), (3, 0, 1), (64, 1, 0), (64, 1, 1)):
        _compare(N, R, V, teacher, padding_idx, offset, seed=V + R, masked=True)


def test_teacher_term_against_student_minus_inf(N):
    """A finite teacher logit against a student -inf is +inf of KL, even where its exponential underflows in float32
    (gap 120 to the row maximum) or in float64 (gap 1000), and even when the thread's running teacher maximum grows by
    more than float64's exp range after it met the term; a teacher -inf against a student -inf adds 0."""
    V = 2048
    g = torch.Generator(device="cuda").manual_seed(4)
    zs = torch.randn(4, V, generator=g, device="cuda")
    zt = torch.randn(4, V, generator=g, device="cuda")
    zs[:, 7] = float("-inf")
    zt[0, 7] = -120.0                     # its group's other columns keep the running maximum near 0: expf underflows
    zt[1, 0:4] = -1000.0                  # columns 0-3, then 1024-1027: the same thread, running max -1000, then >= 0
    zs[1, 0] = float("-inf")
    zt[1, 1024] = 0.0
    zt[2, 7] = float("-inf")              # both -inf: adds 0
    y = torch.tensor([1, 2, 3, 4], device="cuda")
    for r, want_inf in ((0, True), (1, True), (2, False), (3, True)):
        lse, loss, _ = _fwd(N, zs[r:r + 1].contiguous(), zt[r:r + 1].contiguous(), y[r:r + 1], -1)
        o = O.nmt_loss(zs[r:r + 1].cpu().numpy(), y[r:r + 1].cpu().numpy(), -1, zt[r:r + 1].cpu().numpy(), W)
        got = loss.item()
        assert (got == float("inf")) == want_inf and (o["loss"] == np.inf) == want_inf, (r, got, o["loss"])
        if not want_inf:
            assert abs(got - o["loss"]) <= 1e-5 * abs(o["loss"])
        grad = _bwd(N, zs[r:r + 1].contiguous(), zt[r:r + 1].contiguous(), y[r:r + 1], lse, 1.0, -1)
        assert torch.isfinite(grad).all()


def _torch_chain(zs, zt, y, padding_idx, w=W):
    """The reference's compute_loss (onmt/Loss.py:97-120, 68-77) in float32 torch on the GPU: loss, gradient,
    [n_words, n_correct]."""
    zs = zs.detach().clone().requires_grad_(True)
    weight = torch.ones(zs.shape[1], device="cuda")
    weight[padding_idx] = 0
    scores = F.log_softmax(zs, dim=1)
    loss = F.nll_loss(scores, y, weight=weight, reduction="sum")
    if zt is not None:
        pt = F.log_softmax(zt, dim=1).exp().detach()
        kl = F.kl_div(scores, pt, reduction="none") * (y != padding_idx).float()[:, None]
        loss = (1 - w) * loss + w * kl.sum()
    loss.backward()
    non_padding = y.ne(padding_idx)
    n_correct = scores.max(1)[1].eq(y).masked_select(non_padding).sum()
    return loss.detach(), zs.grad, [int(non_padding.sum()), int(n_correct)], scores.detach()


@pytest.mark.parametrize("teacher", [False, True], ids=["plain", "teacher"])
@pytest.mark.parametrize("V", [10_004, 50_004])
def test_against_torch_chain(N, V, teacher):
    from quantized_distillation_b200.nmt_loss import nmt_loss
    R, pad = 3264, 1
    zs, zt, y = _inputs(R, V, teacher, pad, 0, seed=V + 1)
    # rows whose top two log-probs tie in float32 become padding, so the argmax is unambiguous on both sides
    top2 = F.log_softmax(zs, dim=1).topk(2, dim=1).values
    y[top2[:, 0] == top2[:, 1]] = pad
    ref_loss, ref_grad, ref_counts, _ = _torch_chain(zs, zt, y, pad)
    x = zs.detach().clone().requires_grad_(True)
    loss, stats = nmt_loss(x, y, pad, zt)
    loss.backward()
    assert stats.tolist() == ref_counts + [0]
    # the torch chain sums R x V float32 KL terms in float32: its own error, not the kernel's, sets this bound
    assert abs(loss.item() - ref_loss.item()) <= 1e-4 * abs(ref_loss.item())
    assert (x.grad - ref_grad).abs().max().item() <= 1e-5


def test_autograd_grad_output_not_one(N):
    from quantized_distillation_b200.nmt_loss import nmt_loss
    R, V, pad = 64, 1025, 0
    zs, zt, y = _inputs(R, V, True, pad, 0, seed=11)
    x = zs.detach().clone().requires_grad_(True)
    t = zt.detach().clone().requires_grad_(True)
    loss, stats = nmt_loss(x, y, pad, t)
    (loss.div(64) * 3).backward()
    assert t.grad is None and not stats.requires_grad
    o = O.nmt_loss(zs.cpu().numpy(), y.cpu().numpy(), pad, zt.cpu().numpy(), W, grad_loss=3 / 64)
    assert np.abs(x.grad.cpu().numpy() - o["grad"]).max() <= 2e-6 * 3 / 64
    # the same as the C ABI with g = float32(3/64) computed the way autograd does
    g = (torch.ones((), device="cuda") / 64 * 3).item()
    row_lse, _, _ = _fwd(N, zs, zt, y, pad)
    assert torch.equal(_bwd(N, zs, zt, y, row_lse, g, pad), x.grad)


def test_row_bits_alone_in_batch_and_across_runs(N):
    R, V, pad = 48, 10_007, 0          # odd V: the rows of the batch start at every 16-byte phase
    zs, zt, y = _inputs(R, V, True, pad, 0, seed=5)
    lse, loss, counts = _fwd(N, zs, zt, y, pad)
    grad = _bwd(N, zs, zt, y, lse, 0.25, pad)
    lse2, loss2, counts2 = _fwd(N, zs, zt, y, pad)
    assert torch.equal(lse, lse2) and torch.equal(loss.view(1).view(torch.int32), loss2.view(1).view(torch.int32))
    assert torch.equal(counts, counts2) and torch.equal(grad, _bwd(N, zs, zt, y, lse2, 0.25, pad))
    for i in (1, 2, 3, 17, 47):
        if y[i].item() == pad:
            continue
        for offset in (0, 1, 2, 3):
            one_s, one_t = _alloc((1, V), offset), _alloc((1, V), offset)
            one_s.copy_(zs[i:i + 1]), one_t.copy_(zt[i:i + 1])
            l1, loss1, _ = _fwd(N, one_s, one_t, y[i:i + 1], pad)
            assert torch.equal(l1[0], lse[i]), (i, offset)
            assert torch.equal(_bwd(N, one_s, one_t, y[i:i + 1], l1, 0.25, pad, offset=3 - offset)[0], grad[i]), (i, offset)
            # the row's float64 partial rounded once: the same value whatever the alignment
            if offset == 0:
                ref = loss1
            assert torch.equal(loss1, ref)


def test_graph_replay_matches_eager(N):
    R, V, pad = 200, 24_999, 1
    zs, zt, y = _inputs(R, V, True, pad, 1, seed=8)
    lse_e, loss_e, counts_e = _fwd(N, zs, zt, y, pad)
    grad_e = _bwd(N, zs, zt, y, lse_e, 0.5, pad)
    row_lse = torch.zeros(R, 2, device="cuda")
    loss = torch.zeros((), device="cuda")
    counts = torch.zeros(3, dtype=torch.int64, device="cuda")
    ws = torch.empty(int(N.lib().qd_nmt_loss_workspace_bytes(R)), dtype=torch.uint8, device="cuda")
    gd = torch.tensor(0.5, device="cuda")
    grad = torch.zeros(R, V, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            st = s.cuda_stream
            N.check(N.lib().qd_nmt_loss_fwd(N.ptr(zs), N.ptr(zt), N.ptr(y), R, V, pad, W, N.ptr(row_lse), N.ptr(loss), N.ptr(counts),
                                            N.ptr(ws), ws.numel(), st))
            N.check(N.lib().qd_nmt_loss_bwd(N.ptr(zs), N.ptr(zt), N.ptr(y), N.ptr(row_lse), N.ptr(gd), R, V, pad, W, N.ptr(grad), st))
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        grad.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(row_lse, lse_e) and torch.equal(counts, counts_e) and torch.equal(grad, grad_e)
        assert torch.equal(loss.view(1).view(torch.int32), loss_e.view(1).view(torch.int32))


def test_invalid_targets_nan_and_counted(N):
    from quantized_distillation_b200.nmt_loss import NMTLossCompute, nmt_loss
    R, V, pad = 8, 1000, 0
    zs, zt, y = _inputs(R, V, True, -1, 0, seed=3)
    y[:] = torch.tensor([5, -1, V, 0, V + 7, 9, -100, 999], device="cuda")
    lse, loss, counts = _fwd(N, zs, zt, y, pad)
    grad = _bwd(N, zs, zt, y, lse, 1.0, pad)
    torch.cuda.synchronize()
    assert torch.isnan(loss).item() and counts[2].item() == 4 and counts[0].item() == 3
    bad = torch.tensor([1, 2, 4, 6], device="cuda")
    assert torch.isnan(grad[bad]).all() and not grad[3].any() and torch.isfinite(grad[[0, 5, 7]]).all()
    # the Python layer reports them; NMTLossCompute refuses before any backward
    _, stats = nmt_loss(zs, y, pad, zt)
    assert stats[2].item() == 4
    gen = nn.Sequential(nn.Linear(6, V), nn.LogSoftmax(dim=-1)).cuda()
    lc = NMTLossCompute(gen, types.SimpleNamespace(stoi={"<blank>": pad}))
    out = torch.randn(2, 4, 6, device="cuda", requires_grad=True)
    with pytest.raises(ValueError, match="outside the vocabulary"):
        lc.compute_loss(None, out, y.view(2, 4))


def test_c_abi_refusals(N):
    R, V = 4, 10
    zs, zt, y = _inputs(R, V, True, -1, 0, seed=1)
    row_lse = torch.empty(R, 2, device="cuda")
    loss = torch.empty((), device="cuda")
    counts = torch.empty(3, dtype=torch.int64, device="cuda")
    ws = torch.empty(int(N.lib().qd_nmt_loss_workspace_bytes(R)), dtype=torch.uint8, device="cuda")
    L = N.lib()

    def fwd(**kw):
        a = dict(zs=N.ptr(zs), zt=N.ptr(zt), y=N.ptr(y), R=R, V=V, pad=1, w=W, lse=N.ptr(row_lse), loss=N.ptr(loss),
                 counts=N.ptr(counts), ws=N.ptr(ws), wsb=ws.numel())
        a.update(kw)
        return L.qd_nmt_loss_fwd(*a.values(), N.stream_ptr())
    assert fwd() == N.QD_OK and fwd(zt=None) == N.QD_OK and fwd(R=0, zs=None, y=None, lse=None, ws=None, wsb=0) == N.QD_OK
    for bad in (dict(zs=None), dict(y=None), dict(lse=None), dict(loss=None), dict(counts=None), dict(R=-1), dict(V=0),
                dict(pad=-2), dict(pad=V), dict(w=-0.1), dict(w=1.5), dict(w=float("nan")), dict(counts=N.ptr(counts) + 4),
                dict(zs=N.ptr(zs) + 2), dict(lse=N.ptr(zs)), dict(loss=N.ptr(zt) + 4), dict(counts=N.ptr(y)),
                dict(lse=N.ptr(ws)), dict(R=1 << 62, V=1 << 10), dict(zs=N.ptr(zs) + 2, lse=N.ptr(zs)),
                dict(loss=None, counts=N.ptr(counts) + 4), dict(counts=N.ptr(counts) + 4, ws=None)):
        assert fwd(**bad) == N.QD_ERR_INVALID_ARG, bad
        assert L.qd_last_error().decode()
    for bad in (dict(ws=None), dict(wsb=ws.numel() - 1), dict(ws=N.ptr(ws) + 8), dict(ws=None, lse=N.ptr(zs)),
                dict(ws=N.ptr(ws) + 8, counts=N.ptr(y))):
        assert fwd(**bad) == N.QD_ERR_WORKSPACE, bad
    # rows = 0 needs no workspace and takes any pointer for it
    assert fwd(R=0, zs=None, y=None, lse=None, ws=N.ptr(ws) + 1, wsb=0) == N.QD_OK
    torch.cuda.synchronize()
    gd = torch.ones((), device="cuda")
    grad = torch.empty(R, V, device="cuda")

    def bwd(**kw):
        a = dict(zs=N.ptr(zs), zt=N.ptr(zt), y=N.ptr(y), lse=N.ptr(row_lse), g=N.ptr(gd), R=R, V=V, pad=1, w=W, out=N.ptr(grad))
        a.update(kw)
        return L.qd_nmt_loss_bwd(*a.values(), N.stream_ptr())
    assert bwd() == N.QD_OK and bwd(R=0, zs=None, y=None) == N.QD_OK
    for bad in (dict(zs=None), dict(y=None), dict(lse=None), dict(g=None), dict(out=None), dict(V=0), dict(pad=V),
                dict(w=2.0), dict(out=N.ptr(zs)), dict(out=N.ptr(zt) + 4), dict(out=N.ptr(grad) + 2),
                dict(out=N.ptr(zs) + 2), dict(g=None, lse=N.ptr(row_lse) + 2)):
        assert bwd(**bad) == N.QD_ERR_INVALID_ARG, bad
    torch.cuda.synchronize()


def test_python_refusals(N):
    from quantized_distillation_b200.nmt_loss import NMTLossCompute, nmt_loss
    zs = torch.randn(4, 10, device="cuda")
    y = torch.randint(0, 10, (4,), device="cuda")
    for args, kw in (((zs.cpu(), y, 0), {}), ((zs.double(), y, 0), {}), ((zs.view(-1), y, 0), {}),
                     ((zs, y.int(), 0), {}), ((zs, y[:3], 0), {}), ((zs, y.cpu(), 0), {}), ((zs, y, 10), {}), ((zs, y, -2), {}),
                     ((zs, y, 0), dict(teacher_logits=zs[:, :9])), ((zs, y, 0), dict(teacher_logits=zs.half())),
                     ((zs, y, 0), dict(teacher_logits=zs, weight_teacher_loss=1.1))):
        with pytest.raises(ValueError):
            nmt_loss(*args, **kw)
    vocab = types.SimpleNamespace(stoi={"<blank>": 1})
    gen = nn.Sequential(nn.Linear(4, 10), nn.LogSoftmax(dim=-1))
    for bad in (nn.Linear(4, 10), nn.Sequential(nn.Linear(4, 10), nn.Softmax(dim=-1)),
                nn.Sequential(nn.Linear(4, 10), nn.LogSoftmax(dim=-1), nn.Dropout())):
        with pytest.raises(ValueError):
            NMTLossCompute(bad, vocab)
    with pytest.raises(ValueError):
        NMTLossCompute(gen, vocab, use_distillation_loss=True)


def test_memory_is_gradient_plus_rows(N):
    from quantized_distillation_b200.nmt_loss import nmt_loss
    R, V, pad = 3264, 24_004, 1
    zs, zt, y = _inputs(R, V, True, pad, 0, seed=2)
    x = zs.detach().requires_grad_(True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    loss, stats = nmt_loss(x, y, pad, zt)
    loss.div(64).backward()
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    assert extra <= R * V * 4 + 64 * R + 16384, extra


def _reference_sharded(generator, teacher_generator, batch, output, teacher_outputs, padding_idx, shard_size):
    """onmt's sharded_compute_loss (onmt/Loss.py:40-55, 97-120, 122-195) on current torch: the decoder output detached
    into a leaf, split into shards, one loss and backward per shard, then one backward into the decoder."""
    V = generator[0].out_features
    weight = torch.ones(V, device="cuda")
    weight[padding_idx] = 0
    target = batch.tgt[1:]
    leaf = output.detach().requires_grad_(True)
    loss_sum, n_words, n_correct = 0.0, 0, 0
    for out_s, tgt_s, t_s in zip(torch.split(leaf, shard_size), torch.split(target, shard_size), torch.split(teacher_outputs, shard_size)):
        scores = generator(out_s.reshape(-1, out_s.size(2)))
        tgt = tgt_s.reshape(-1)
        loss = F.nll_loss(scores, tgt, weight=weight, reduction="sum")
        pt = teacher_generator(t_s.reshape(-1, t_s.size(2))).exp().detach()
        kl = F.kl_div(scores, pt, reduction="none") * tgt.ne(padding_idx).float()[:, None]
        loss = (1 - W) * loss + W * kl.sum()
        loss.div(batch.batch_size).backward()
        non_padding = tgt.ne(padding_idx)
        loss_sum += loss.item()
        n_words += int(non_padding.sum())
        n_correct += int(scores.max(1)[1].eq(tgt).masked_select(non_padding).sum())
    torch.autograd.backward([output], [leaf.grad])
    return loss_sum, n_words, n_correct


def test_sharded_compute_loss_matches_reference(N):
    from quantized_distillation_b200.nmt_loss import NMTLossCompute
    torch.manual_seed(0)
    T, B, H, V, pad = 11, 8, 32, 1003, 1
    vocab = types.SimpleNamespace(stoi={"<blank>": pad})
    decoder = nn.Linear(H, H).cuda()
    gen = nn.Sequential(nn.Linear(H, V), nn.LogSoftmax(dim=-1)).cuda()
    tgen = nn.Sequential(nn.Linear(H, V), nn.LogSoftmax(dim=-1)).cuda()
    x = torch.randn(T, B, H, device="cuda")
    teacher_outputs = torch.randn(T, B, H, device="cuda")
    tgt = torch.randint(0, V, (T + 1, B), device="cuda")
    tgt[-3:, ::2] = pad                                        # shorter sentences padded at the end
    batch = types.SimpleNamespace(tgt=tgt, batch_size=B)
    params = list(decoder.parameters()) + list(gen.parameters())

    output = torch.tanh(decoder(x))
    ref = _reference_sharded(gen, tgen, batch, output, teacher_outputs, pad, 4)
    ref_grads = [p.grad.clone() for p in params]
    for p in params:
        p.grad = None
    lc = NMTLossCompute(gen, vocab, use_distillation_loss=True, teacher_generator=tgen)
    stats = lc.sharded_compute_loss(batch, torch.tanh(decoder(x)), {}, 0, T + 1, 4, teacher_outputs=teacher_outputs)
    assert (stats.n_words, stats.n_correct) == ref[1:]
    assert stats.loss == pytest.approx(ref[0], rel=1e-5)
    for p, r in zip(params, ref_grads):
        assert (p.grad - r).abs().max().item() <= 1e-5 * max(r.abs().max().item(), 1e-3)
    assert all(p.grad is None for p in tgen.parameters())
