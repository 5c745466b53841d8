"""Data-parallel differentiable quantization on the GPU.

* The split centroid backward of ``CentroidPlan`` (``backward_partial_`` then ``finish_``; C ABI
  ``qd_plan_nonuniform_bwd_partial`` / ``_finish``) against ``backward_``: bit for bit at scale 1, and on data whose
  sums are exact, a table reduced over W simulated ranks equals one process given the rank-average gradient.
* ``optimize_quantization_points`` on a ``FlatDataParallel``-wrapped student, two processes sharing ONE GPU over gloo:
  the ranks agree bit for bit, the points match a single process on the global batch, and mismatching point counts
  raise ``ValueError`` on every rank.  The mixed mode of ``train_model`` runs one mixed epoch under the wrapper.
* With two or more GPUs: NCCL, the step captured in a CUDA graph with its all-reduce, against eager steps.
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from oracle import quant_oracle as O

pytestmark = pytest.mark.gpu

F32 = np.float32


@pytest.fixture(scope="module")
def CP():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200.plan import CentroidPlan
    return CentroidPlan


def _point_sets(rng, count):
    """K = 1..32, some with a duplicated point, some with the end points 0 and 1."""
    pts = []
    for i in range(count):
        k = 1 + i % 32
        p = np.sort(rng.random(k)).astype(F32)
        if k >= 2 and i % 5 == 1:
            p[k // 2] = p[k // 2 - 1]
        if k >= 2 and i % 7 == 3:
            p[0], p[-1] = 0, 1
        pts.append(p)
    return pts


def _plan(CP, xs, pts, bucket):
    src = [torch.from_numpy(x).cuda() for x in xs]
    dst = [torch.empty_like(s) for s in src]
    plan = CP(src, dst, [torch.from_numpy(p).cuda() for p in pts], bucket)
    plan.forward_()
    return plan


def _sums(plan):
    return torch.full((len(plan.sources), plan.MAX_POINTS), float("nan"), dtype=torch.float64, device=plan.device)


def _sizes(rng, count, bucket):
    """Tensor sizes that put rows across the 1024-element gradient tiles and tensors across gradient blocks."""
    base = [1, 3, 100, 1023, 1024, 1025, 2053, 7 * (bucket or 1000) + 5, 65_543]
    if count <= len(base):
        return base[:count]
    return base + [int(v) for v in rng.integers(1, 5000, count - len(base))]


@pytest.mark.parametrize("bucket", [256, 1000])
@pytest.mark.parametrize("count", [1, 9, 58, 601])
def test_partial_then_finish_equals_backward(CP, count, bucket):
    """``backward_partial_`` + ``finish_(sums, 1)`` gives ``backward_``'s gradient bit for bit at K = 1..32 with
    duplicate points; the table holds the float64 sums (their float32 cast IS the gradient) and zeros past K."""
    rng = np.random.default_rng(11_000 + count + bucket)
    xs = [(rng.standard_normal(n) * 0.05).astype(F32) for n in _sizes(rng, count, bucket)]
    pts = [np.sort(rng.random(17)).astype(F32)] if count == 1 else _point_sets(rng, count)
    plan = _plan(CP, xs, pts, bucket)
    grads = [torch.from_numpy(rng.standard_normal(x.size).astype(F32)).cuda() for x in xs]
    ref = [t.clone() for t in plan.backward_(grads)]
    plan._gp_flat.fill_(float("nan"))
    sums = _sums(plan)
    plan.backward_partial_(grads, sums)
    assert bool(torch.isnan(plan._gp_flat).all()), "backward_partial_ wrote grad_points"
    got = plan.finish_(sums, 1.0)
    for i, p in enumerate(pts):
        what = f"count={count} b={bucket} tensor {i} (K={p.size})"
        assert torch.equal(got[i].view(torch.int32), ref[i].view(torch.int32)), what
        assert torch.equal(sums[i, :p.size].float().view(torch.int32), ref[i].view(torch.int32)), what
        assert bool((sums[i, p.size:] == 0).all()), f"{what}: table not zero past K"
    plan.close()


def test_partial_with_multi_tile_blocks(CP):
    """Enough tiles that each gradient block spans several tiles (5.1 M elements: 2 tiles per block)."""
    rng = np.random.default_rng(11_500)
    xs = [(rng.standard_normal(n) * 0.05).astype(F32) for n in (5, 1000, 2_000_003, 3_100_000)]
    pts = [np.sort(rng.random(k)).astype(F32) for k in (32, 1, 4, 17)]
    plan = _plan(CP, xs, pts, 256)
    grads = [torch.from_numpy(rng.standard_normal(x.size).astype(F32)).cuda() for x in xs]
    ref = [t.clone() for t in plan.backward_(grads)]
    sums = _sums(plan)
    got = plan.finish_(plan.backward_partial_(grads, sums), 1.0)
    for i in range(len(xs)):
        assert torch.equal(got[i].view(torch.int32), ref[i].view(torch.int32)), i
    plan.close()


def _exact_rows(rng, n, bucket):
    """Every row holds 0 and 2^-e (e = row % 4), everything else in between: alpha = 2^-e exactly."""
    rows, rl, _ = O.bucket_geometry(n, bucket)
    scale = np.repeat(np.ldexp(F32(1), -(np.arange(rows) % 4)).astype(F32), rl)[:n]
    x = rng.random(n, dtype=F32) * scale
    starts = np.arange(rows, dtype=np.int64) * rl
    x[starts] = 0
    second = starts[starts + 1 < np.minimum(starts + rl, n)] + 1
    x[second] = scale[second]
    return x


@pytest.mark.parametrize("world", [2, 4, 8])
def test_reduced_table_equals_rank_average_on_exact_data(CP, world):
    """alpha = 2^-e and integer gradients: every sum is exact.  W per-rank tables summed in float64 (what the
    all-reduce does) and finished with scale 1/W equal one process given the rank average of the gradients."""
    rng = np.random.default_rng(12_000 + world)
    sizes = [1, 3, 1023, 1025, 2053, 65_543, 300_001]
    xs = [_exact_rows(rng, n, 256) for n in sizes]
    pts = [np.sort(rng.random(k)).astype(F32) for k in (32, 1, 4, 16, 8, 3, 17)]
    plan = _plan(CP, xs, pts, 256)
    per_rank = [[rng.integers(-4, 5, n).astype(F32) * world for n in sizes] for _ in range(world)]
    total = _sums(plan).zero_()
    for gs in per_rank:
        s = _sums(plan)
        plan.backward_partial_([torch.from_numpy(g).cuda() for g in gs], s)
        total += s
    got = [t.clone() for t in plan.finish_(total, 1.0 / world)]
    avg = [(sum(r[i].astype(np.float64) for r in per_rank) / world).astype(F32) for i in range(len(sizes))]
    ref = plan.backward_([torch.from_numpy(a).cuda() for a in avg])
    for i in range(len(sizes)):
        assert torch.equal(got[i].view(torch.int32), ref[i].view(torch.int32)), (i, got[i], ref[i])
    plan.close()


def test_split_backward_refusals(CP):
    rng = np.random.default_rng(13_000)
    xs = [(rng.standard_normal(n) * 0.05).astype(F32) for n in (100, 300)]
    plan = _plan(CP, xs, _point_sets(rng, 2), 256)
    grads = [torch.zeros(x.size, device="cuda") for x in xs]
    for bad in (torch.zeros((2, 32), dtype=torch.float32, device="cuda"),     # float32
                torch.zeros((3, 32), dtype=torch.float64, device="cuda"),     # wrong shape
                torch.zeros((32, 2), dtype=torch.float64, device="cuda").t(),  # not contiguous
                torch.zeros((2, 32), dtype=torch.float64)):                   # host memory
        with pytest.raises(ValueError):
            plan.backward_partial_(grads, bad)
        with pytest.raises(ValueError):
            plan.finish_(bad, 1.0)
    with pytest.raises(ValueError):
        plan.backward_partial_(grads[:1], _sums(plan))
    plan.close()


def test_split_backward_in_cuda_graph(CP):
    """Partial, a device-side stand-in for the all-reduce and finish replay inside one CUDA graph."""
    rng = np.random.default_rng(14_000)
    xs = [(rng.standard_normal(n) * 0.05).astype(F32) for n in (100, 5000, 70_000)]
    pts = _point_sets(rng, 3)
    plan = _plan(CP, xs, pts, 256)
    grads = [torch.from_numpy(rng.standard_normal(x.size).astype(F32)).cuda() for x in xs]
    sums = _sums(plan)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        plan.finish_(plan.backward_partial_(grads, sums), 0.5)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan.backward_partial_(grads, sums)
        sums.mul_(2.0)
        plan.finish_(sums, 0.5)
    for g in grads:
        g.copy_(torch.randn_like(g))
    plan._gp_flat.zero_()
    graph.replay()
    torch.cuda.synchronize()
    got = [t.clone() for t in plan.grad_points]
    ref = plan.backward_(grads)
    for i in range(3):
        assert torch.equal(got[i].view(torch.int32), ref[i].view(torch.int32)), i
    plan.close()


# ==================================================================================== several processes
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _student(batch_norm=False):
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    spec = dict(cfm.smallerModelSpec)
    spec["spec_dropout_rates"] = []                  # no per-rank randomness: the run can be compared with one process
    return cfm.ConvolForwardNet(**spec, useBatchNorm=batch_norm, useAffineTransformInBatchNorm=batch_norm)


OQP = dict(initial_learning_rate=1e-3, epochs_to_train=1, print_every=1, numPointsPerTensor=4, bucket_size=256,
           verbose=False, evaluate=False)


def _run_dp(model, local, assign, **kw):
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    sd, pts, info = cfm.optimize_quantization_points(model, local, local, assignBitsAutomatically=assign, **{**OQP, **kw})
    return ({k: v.detach().cpu().clone() for k, v in sd.items()}, [p.detach().cpu().clone() for p in pts], info)


def _logits(sd, batch_norm):
    torch.manual_seed(0)
    net = _student(batch_norm).cuda()
    net.load_state_dict(sd)
    net.eval()
    x = torch.randn(8, 3, 32, 32, generator=torch.Generator().manual_seed(5)).cuda()
    with torch.no_grad():
        return net(x).cpu()


def _gloo_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK="0")
    torch.cuda.set_device(0)                                         # both ranks share the one GPU
    torch.backends.cudnn.allow_tf32 = False                          # compared with one process: IEEE float32 convolutions
    import torch.distributed as dist
    from quantized_distillation_b200 import distributed as D
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    from quantized_distillation_b200.cnn_models import help_fun as hf
    dist.init_process_group("gloo")
    try:
        batches = hf.synthetic_cifar_loader(6, 8, seed=7, pin=False)
        local = D.shard_batches(batches, rank, world)
        out = {}
        for assign in (False, True):
            torch.manual_seed(1234 + rank)                           # the wrapper broadcasts rank 0's weights
            # 0.25 MB buckets: the gradient-norm passes of assignBitsAutomatically must not reduce from the hooks
            model = D.FlatDataParallel(_student().cuda(), bucket_mb=0.25 if assign else 32.0)
            out[f"plain-{assign}"] = _run_dp(model, local, assign)
        torch.manual_seed(99)
        model = D.FlatDataParallel(_student(batch_norm=True).cuda())
        sd, pts, info = _run_dp(model, local, False, evaluate=True)
        out["bn"] = (sd, pts, info)
        out["bn-logits"] = _logits(sd, True)
        # a per-tensor fallback (more than 32 points): float32 gradients averaged by one all-reduce
        torch.manual_seed(3)
        out["fallback"] = _run_dp(D.FlatDataParallel(_student().cuda()), local, False, numPointsPerTensor=40,
                                  max_steps=3)
        # ranks that disagree on the point counts: the same ValueError everywhere, before anything is launched
        try:
            _run_dp(D.FlatDataParallel(_student().cuda()), local, False, numPointsPerTensor=4 + rank)
            out["mismatch"] = None
        except ValueError as e:
            out["mismatch"] = str(e)
        # mixed mode of train_model: one quantized-distillation epoch, one differentiable epoch, one more epoch
        torch.manual_seed(5)
        model = D.FlatDataParallel(_student(batch_norm=True).cuda())
        cfm.train_model(model, local[:3], local[:3], quantizeWeights=True, numBits=2, bucket_size=256, epochs_to_train=2,
                        mix_with_differentiable_quantization=True, print_every=1, verbose=False, evaluate=False)
        out["mixed"] = [p.detach().cpu().clone() for p in model.parameters()]
        ret[rank] = out
    finally:
        dist.destroy_process_group()


@pytest.fixture(scope="module")
def gloo_runs():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    world = 2
    with mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_gloo_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
        return [ret[r] for r in range(world)]


def _same(a, b):
    if isinstance(a, dict):
        return list(a) == list(b) and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, torch.Tensor):
        return a.dtype == b.dtype and a.shape == b.shape and bool((a.view(-1).view(torch.uint8) == b.view(-1).view(torch.uint8)).all())
    return a == b


@pytest.mark.parametrize("assign", [False, True])
def test_gloo_ranks_agree_and_match_one_process(gloo_runs, assign, monkeypatch):
    """Two gloo ranks on the halves of every global batch: points and state dicts bit-identical across ranks, and
    close to one process that saw the whole batches."""
    from quantized_distillation_b200.cnn_models import help_fun as hf
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    r0, r1 = (r[f"plain-{assign}"] for r in gloo_runs)
    assert _same(r0[0], r1[0]) and _same(r0[1], r1[1])
    assert r0[2]["multi_tensor_plan"] and r0[2]["data_parallel_world"] == 2
    assert not any(k.startswith("module.") for k in r0[0])
    torch.manual_seed(1234)
    single = _student().cuda()
    batches = hf.synthetic_cifar_loader(6, 8, seed=7, pin=False)
    sd, pts, _ = _run_dp(single, batches, assign)
    assert [p.numel() for p in pts] == [p.numel() for p in r0[1]]
    torch.manual_seed(1234)
    start = _run_dp(_student().cuda(), batches, assign, epochs_to_train=0)[1]
    # the per-rank losses differ from the global one in float32 rounding and cuDNN's summation order, which the
    # cancelling centroid sums amplify (with TF32 convolutions by several per cent, so both runs use IEEE float32
    # ones).  The data-parallel run must follow the single process's trajectory to 5 %, and much closer than a
    # process that saw only rank 0's halves (what every rank would learn without the reduction).
    moved = max(float((a - b).abs().max()) for a, b in zip(pts, start))
    err = max(float((a - b).abs().max()) for a, b in zip(pts, r0[1]))
    assert moved > 1e-4, "the points did not move"
    assert err <= 0.05 * moved, (err, moved)
    torch.manual_seed(1234)
    from quantized_distillation_b200 import distributed as D
    half = _run_dp(_student().cuda(), D.shard_batches(batches, 0, 2), assign)[1]
    if [p.numel() for p in half] == [p.numel() for p in pts]:
        local_err = max(float((a - b).abs().max()) for a, b in zip(pts, half))
        assert err <= 0.2 * local_err, (err, local_err)


def test_gloo_batch_norm_buffers_and_logits_agree(gloo_runs):
    """The quantized copy's batch-norm statistics come from rank 0 on every rank, so the returned state dicts and
    the logits of a network loaded from them are bit-identical; the evaluated accuracy is one number."""
    r0, r1 = (r["bn"] for r in gloo_runs)
    assert any("running_mean" in k for k in r0[0])
    assert _same(r0[0], r1[0]) and _same(r0[1], r1[1])
    assert r0[2]["predictionAccuracy"] == r1[2]["predictionAccuracy"]
    assert _same(gloo_runs[0]["bn-logits"], gloo_runs[1]["bn-logits"])


def test_gloo_per_tensor_fallback_agrees(gloo_runs):
    r0, r1 = (r["fallback"] for r in gloo_runs)
    assert not r0[2]["multi_tensor_plan"]
    assert _same(r0[0], r1[0]) and _same(r0[1], r1[1])


def test_gloo_point_count_mismatch_raises_on_every_rank(gloo_runs):
    for r in gloo_runs:
        assert r["mismatch"] is not None and "different numbers of points" in r["mismatch"]


def test_gloo_mixed_mode_ranks_agree(gloo_runs):
    assert _same(gloo_runs[0]["mixed"], gloo_runs[1]["mixed"])


def _nccl_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    from quantized_distillation_b200 import distributed as D
    from quantized_distillation_b200.cnn_models import help_fun as hf
    w, r, device = D.init_distributed(backend="nccl")
    import torch.distributed as dist
    torch.backends.cudnn.deterministic = True                        # eager and captured runs are compared bit for bit
    try:
        batches = hf.synthetic_cifar_loader(8, 16, seed=7, pin=False)
        local = D.shard_batches(batches, r, w)
        out = {}
        for graph in (False, True):
            torch.manual_seed(1234)
            model = D.FlatDataParallel(_student(batch_norm=True).to(device))
            out[graph] = _run_dp(model, local, False, cuda_graph_step=graph)
        ret[rank] = out
    finally:
        dist.destroy_process_group()


def test_nccl_captured_step_matches_eager():
    """Two GPUs, NCCL: the whole step captured in a CUDA graph, all-reduce included, ends on the same points and
    state dict as eager steps, bit for bit, on both ranks."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip(f"needs 2 GPUs for NCCL ranks, {torch.cuda.device_count() if torch.cuda.is_available() else 0} visible")
    world = 2
    with mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_nccl_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
        runs = [ret[r] for r in range(world)]
    for out in runs:
        assert out[True][2]["cuda_graph_step"] and not out[False][2]["cuda_graph_step"]
        assert _same(out[True][0], out[False][0]) and _same(out[True][1], out[False][1])
    assert _same(runs[0][True][0], runs[1][True][0]) and _same(runs[0][True][1], runs[1][True][1])
