"""GPU tests of the multi-tensor plans (plan.py, csrc/qd_plans.cu, csrc/qd_plan.cuh) against the oracle.

The training loops call the plans, not the per-tensor ops: ``QuantizationPlan`` (save-and-quantize, gradient
fix-up, fused SGD step) and ``CentroidPlan`` (forward and centroid gradient of the differentiable-quantization
loop).  The plans have their own kernels and their own dispatch, so every case below is checked against the
oracle (``oracle/quant_oracle.py``, ``oracle/c_oracle.py`` for large tensors), never only against the per-tensor
CUDA op: a bug shared by both CUDA paths must not cancel out.

The inputs sweep what the plans dispatch on:
* row length: the register kernel's R (2 up to 256 floats, 4 up to 512, 8 up to 1024, from the plan's LONGEST row),
  full and ragged rows, the per-tensor block fallback (1025 .. 49152), the grid fallback (> 49152), bucket None with
  short tensors (warp path, one row per tensor) and with long ones (the long-row plan);
* alignment: contiguous views at float offsets 0..3 into one flat buffer, mixed inside one plan, with the gradients
  aligned differently from the parameters (the kernels pick the 128-bit or the scalar lane map per row);
* tensor count: 1, 256, 257 and ~600 (above 256 the row search reads the table from global memory and the gradient
  pointers travel through a device table instead of the kernel parameters);
* levels per tensor: 2 .. 65536 (above 256 the exact quantization path);
* the fused SGD step's options: momentum 0 / 0.9, Nesterov, weight decay, a learning rate that changes.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import c_oracle as CO
from oracle import quant_oracle as O

pytestmark = pytest.mark.gpu

F32 = np.float32
LEVELS = [2, 3, 4, 16, 255, 256, 257, 1024, 65536]
# R = 2 (<= 256), R = 4 (257 .. 512), R = 8 (513 .. 1024), per-tensor block path (1025 .. 49152), grid path (> 49152)
WARP_BUCKETS = [64, 100, 128, 200, 256, 300, 384, 500, 512, 513, 700, 1000, 1024]
FALLBACK_BUCKETS = [1025, 2048, 3002, 49152, 49153, 100_000]
CHUNK = 16384                                   # chunk of the long-row plan (qd_plan.cuh kPlanChunk)


@pytest.fixture(scope="module")
def P():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import quantized_distillation_b200.quantization as Q
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import plan
    return SimpleNamespace(Q=Q, N=N, QuantizationPlan=plan.QuantizationPlan, CentroidPlan=plan.CentroidPlan)


# ----------------------------------------------------------------------- helpers
def bits(a):
    a = np.ascontiguousarray(np.asarray(a))
    return a.view(np.uint32) if a.dtype == np.float32 else a


def host(t):
    return t.detach().cpu().numpy().reshape(-1) if isinstance(t, torch.Tensor) else np.asarray(t).reshape(-1)


def assert_same(a, b, what=""):
    a, b = host(a), host(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not np.array_equal(bits(a), bits(b)):
        bad = np.nonzero(bits(a) != bits(b))[0]
        raise AssertionError(f"{what}: {bad.size} mismatches, first at {bad[:5]}: {a[bad[:5]]} vs {b[bad[:5]]}")


def assert_minmax_gradient(out, g, ref, argmax, argmin, abs_sum, r, what=""):
    """a5 parity bar.  Untouched elements are bit-identical to g.  At the two positions of bucket b the only freedom is
    the ORDER of the sum r_b = sum_j v_j (float64 in the oracle, float32 groups + float64 in the kernel):
    |out - ref| <= 1e-6 * sum_j |v_j| + one float32 ulp of r_b (its rounding) + one ulp of the result (the final add)."""
    out, g, ref = (np.asarray(host(a), dtype=F32) for a in (out, g, ref))
    pos = np.concatenate([np.asarray(argmax), np.asarray(argmin)]).astype(np.int64)
    rows = np.concatenate([np.arange(len(argmax)), np.arange(len(argmin))])
    touched = np.zeros(out.size, bool)
    touched[pos] = True
    assert np.array_equal(out[~touched].view(np.uint32), g[~touched].view(np.uint32)), f"{what}: element outside argmin'/argmax' changed"
    ulp = 2.0 ** -23
    tol = 1e-6 * abs_sum[rows] + ulp * np.abs(r[rows]) + ulp * np.maximum(np.abs(ref[pos]), np.abs(g[pos])) + 1e-37
    err = np.abs(out[pos].astype(np.float64) - ref[pos].astype(np.float64))
    bad = np.nonzero(err > tol)[0]
    assert bad.size == 0, f"{what}: {bad.size} positions off, worst {err[bad].max():.3e} vs tol {tol[bad][err[bad].argmax()]:.3e}"


def place(arrays, offsets):
    """Contiguous CUDA views into ONE flat float32 buffer; view i starts offsets[i] floats past a 256-byte boundary,
    so offsets 1..3 give rows that are not 16-byte aligned."""
    starts, pos = [], 0
    for a, off in zip(arrays, offsets):
        pos = -(-pos // 64) * 64 + int(off)
        starts.append(pos)
        pos += a.size
    flat = np.zeros(max(pos, 1), F32)
    for a, s in zip(arrays, starts):
        flat[s:s + a.size] = np.asarray(a, F32).reshape(-1)
    buf = torch.from_numpy(flat).cuda()
    views = [buf[s:s + a.size] for a, s in zip(arrays, starts)]
    for v, off in zip(views, offsets):
        assert v.is_contiguous() and v.data_ptr() % 16 == 4 * (int(off) % 4)
    return views


def mixed(count, shift=0):
    return [(i + shift) % 4 for i in range(count)]


def levels_for(count):
    return [LEVELS[i % len(LEVELS)] for i in range(count)]


def row_len(n, bucket):
    return O.bucket_geometry(n, bucket)[1]


def edge_sizes(bucket):
    """1, 3, 127, 128, 129, bucket - 1, bucket, bucket + 1, k * bucket + r and tensors shorter than the bucket."""
    if bucket is None:
        return [1, 3, 127, 128, 129, 255, 256, 257, 511, 512, 513, 700, 1000, 1023, 1024]
    b = bucket
    return [1, 3, 127, 128, 129, b - 1, b, b + 1, 3 * b + 5, 2 * b + b // 2, max(b // 2 - 1, 2), 4 * b]


def uniform_inputs(rng, sizes, scale=0.7):
    """Gaussian tensors (|x| > 1 in places, for the truncated fix-up) plus a constant tensor (alpha -> 1) and one with
    tied extremes (first-occurrence argmin / argmax)."""
    xs = [(rng.standard_normal(n) * scale).astype(F32) for n in sizes]
    if len(xs) > 2:
        xs[-2] = np.full(xs[-2].size, 0.25, F32)
        xs[-1] = (np.round(xs[-1] * 4) / 4 + 0.0).astype(F32)      # + 0.0: no -0.0, whose sign a min may keep or drop
    return xs


def snapshot(ts):
    return [t.detach().clone() for t in ts]


def assert_untouched(ts, before, what):
    torch.cuda.synchronize()
    for i, (t, b) in enumerate(zip(ts, before)):
        assert torch.equal(t.view(torch.int32), b.view(torch.int32)), f"{what}: tensor {i} changed"


# =============================================================================== 1. uniform plan
def check_uniform_plan(P, xs, levels, bucket, poffs, goff_sets, rng, what):
    """quantize_ / save_and_quantize_ / restore_master and both fix-ups of one plan against the oracle."""
    count = len(xs)
    params = place(xs, poffs)
    plan = P.QuantizationPlan(params, levels, bucket)
    refs = [O.uniform_fwd(x, lv, bucket)[0] for x, lv in zip(xs, levels)]
    plan.save_master()
    plan.quantize_()
    for i in range(count):
        assert_same(params[i], refs[i], f"{what} quantize_ tensor {i} (n={xs[i].size} levels={levels[i]})")
    plan.restore_master()
    for i in range(count):
        assert_same(params[i], xs[i], f"{what} restore_master tensor {i}")
    master = plan.save_and_quantize_()
    for i in range(count):
        assert_same(params[i], refs[i], f"{what} save_and_quantize_ q tensor {i} (n={xs[i].size} levels={levels[i]})")
        assert_same(master[i], xs[i], f"{what} save_and_quantize_ master tensor {i}")
    plan.restore_master()
    for i in range(count):
        assert_same(params[i], xs[i], f"{what} restore_master after save tensor {i}")

    for goffs in goff_sets:
        gs = [rng.standard_normal(x.size).astype(F32) for x in xs]
        grads = place(gs, goffs)
        plan.backward_(grads, "truncated")
        for i in range(count):
            assert_same(grads[i], O.uniform_bwd_truncated(xs[i], gs[i]), f"{what} truncated tensor {i} goff={goffs[i]}")

        grads = place(gs, goffs)
        longest = max(row_len(x.size, bucket) for x in xs)
        if bucket is None or longest > 49152:          # min/max needs a bucket, and rows the staged path can hold
            before = snapshot(grads)
            with pytest.raises(NotImplementedError):
                plan.backward_(grads, "complicated")
            assert_untouched(grads, before, f"{what} refused min/max backward")
            continue
        # The per-tensor op on the same memory layout must give the same bits.  The order in which a warp adds up
        # r_b follows its lane map, and the lane map follows the alignment of x and g, so the op runs on the plan's
        # own views (in place, like the plan); uniformQuantization_variable, which copies x and g to fresh aligned
        # tensors, is compared where the plan's views are aligned too.  Rows of 513 .. 1023 floats are the exception:
        # there the per-tensor op runs min/max on the staged ring instead of the register kernel (qd_quant.cu
        # run_rows), another summation order, so only the oracle's bar applies to them.
        expect = place(gs, goffs)
        for i in range(count):
            ws = P.N.workspace(xs[i].size, bucket, params[i].device)
            P.N.check(P.N.lib().qd_uniform_bwd(P.N.ptr(params[i]), P.N.ptr(expect[i]), P.N.ptr(expect[i]), xs[i].size, bucket,
                                               levels[i], P.N.BWD_MINMAX, P.N.ptr(ws), ws.numel(), P.N.stream_ptr()))
        aligned = all(p % 4 == 0 for p in poffs) and all(g % 4 == 0 for g in goffs)
        if aligned:
            api = []
            for i in range(count):
                f = P.Q.uniformQuantization_variable(levels[i], bucket_size=bucket)
                f.forward(params[i])
                api.append(f.backward(grads[i].clone()))
        plan.backward_(grads, "complicated")
        for i in range(count):
            ref, info = O.uniform_bwd_minmax(xs[i], gs[i], levels[i], bucket)
            assert_minmax_gradient(grads[i], gs[i], ref, info["argmax"], info["argmin"], info["abs_sum"], info["r"],
                                   f"{what} min/max tensor {i} (n={xs[i].size} levels={levels[i]} goff={goffs[i]})")
            if 512 < row_len(xs[i].size, bucket) < 1024:
                continue
            assert torch.equal(grads[i].view(torch.int32), expect[i].view(torch.int32)), \
                f"{what} min/max tensor {i} goff={goffs[i]}: plan and per-tensor op differ"
            if aligned:
                assert torch.equal(grads[i].view(torch.int32), api[i].reshape(-1).view(torch.int32)), \
                    f"{what} min/max tensor {i}: plan and uniformQuantization_variable differ"
    plan.close()
    return params


@pytest.mark.parametrize("bucket", WARP_BUCKETS + FALLBACK_BUCKETS + [None])
def test_uniform_plan_matches_oracle(P, bucket):
    """Every geometry class, per-tensor levels 2..65536, mixed float offsets: q and the master bit for bit, the truncated
    fix-up bit for bit, the min/max fix-up inside the a5 bar and bit-identical to the per-tensor op -- or, where the
    plan cannot do min/max (bucket None, rows over 49152 floats), a refusal that leaves every gradient untouched."""
    rng = np.random.default_rng(1000 + (bucket or 0))
    sizes = edge_sizes(bucket)
    xs = uniform_inputs(rng, sizes)
    count = len(xs)
    lv = levels_for(count)
    # unaligned parameters with unaligned, aligned and differently unaligned gradients; then aligned parameters
    check_uniform_plan(P, xs, lv, bucket, mixed(count), [mixed(count), [0] * count, mixed(count, 1)], rng, f"b={bucket} mixed")
    check_uniform_plan(P, xs, lv, bucket, [0] * count, [[0] * count, mixed(count, 1)], rng, f"b={bucket} aligned")


def many_sizes(rng, bucket, count):
    pool = edge_sizes(bucket)
    return [int(rng.choice(pool)) for _ in range(count)]


@pytest.mark.parametrize("bucket", [100, 300, 1000, 2048, None])
def test_uniform_plan_many_tensors(P, bucket):
    """256 tensors (the shared-memory row table and the by-value gradient table exactly full), 257 and ~600 (row table
    in global memory, gradient pointers through the device table) against the oracle, and one probe tensor that must
    give the same bits alone and at the end of the large plans."""
    rng = np.random.default_rng(2000 + (bucket or 0))
    probe = (rng.standard_normal(3 * (bucket or 300) + 7) * 0.7).astype(F32) if bucket else \
        (rng.standard_normal(1000) * 0.7).astype(F32)
    probe_g = rng.standard_normal(probe.size).astype(F32)
    got = {}
    for count in (1, 256, 257, 601):
        xs = uniform_inputs(rng, many_sizes(rng, bucket, count - 1)) + [probe] if count > 1 else [probe]
        lv = levels_for(count)
        lv[-1] = 16
        poffs, goffs = mixed(count, 1), mixed(count, 3)
        poffs[-1], goffs[-1] = 1, 3                     # the probe sits at the same offsets in every plan
        params = check_uniform_plan(P, xs, lv, bucket, poffs, [goffs], rng, f"b={bucket} count={count}")
        plan = P.QuantizationPlan(params, lv, bucket)
        gs = [rng.standard_normal(x.size).astype(F32) for x in xs[:-1]] + [probe_g]
        plan.save_and_quantize_()
        q = params[-1].clone()
        plan.restore_master()
        res = [q]
        for style in ("truncated", "complicated"):
            grads = place(gs, goffs)
            if style == "complicated" and bucket is None:
                continue
            plan.backward_(grads, style)
            res.append(grads[-1].clone())
        got[count] = res
        plan.close()
    for count in (256, 257, 601):
        for a, b in zip(got[1], got[count]):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"b={bucket}: the probe changes in a plan of {count}"


# =============================================================================== 2. fused optimizer step
OPT_SETS = [(0.0, False, 0.0), (0.0, False, 5e-4), (0.9, False, 0.0), (0.9, False, 5e-4), (0.9, True, 0.0), (0.9, True, 5e-4)]
LRS = [0.05, 0.05, 0.02, 0.02, 0.02]             # the learning rate changes at step 3


def run_fused(P, xs, levels, bucket, style, poffs, goffs, momentum, nesterov, wd, rng, what, clamp_start=True):
    """fused_step_ against torch.optim.SGD(foreach=True) on full-precision copies, preceded by the fix-up:
    the oracle's for truncated, the plan's own backward_ for complicated (section 1 anchors it to the oracle; the
    reference plan's views have the fused kernel's alignment, so both take the same lane map and summation order).
    For truncated, the training loop clamps the weights to [-1, 1] before the first step (clamp_start); without that
    clamp the first fused step's fix-up meets weights with |w| > 1 and must zero their gradients."""
    count = len(xs)
    live = place(xs, poffs)
    if style == "truncated" and clamp_start:
        for t in live:
            t.clamp_(-1, 1)
    ref_w = [torch.nn.Parameter(t.clone()) for t in live]
    ref_view = place([host(t) for t in live], poffs)
    ref_plan = P.QuantizationPlan(ref_view, levels, bucket) if style == "complicated" else None
    opt = torch.optim.SGD(ref_w, lr=LRS[0], momentum=momentum, nesterov=nesterov, weight_decay=wd, foreach=True)
    plan = P.QuantizationPlan(live, levels, bucket)
    plan.save_and_quantize_()
    for i in range(count):
        assert_same(live[i], O.uniform_fwd(host(ref_w[i]), levels[i], bucket)[0], f"{what} initial q tensor {i}")
    for step, lr in enumerate(LRS):
        gs = [rng.standard_normal(x.size).astype(F32) for x in xs]
        if style == "none":
            rg = [torch.from_numpy(g).cuda() for g in gs]
        elif style == "truncated":
            rg = [torch.from_numpy(O.uniform_bwd_truncated(host(p), g)).cuda() for p, g in zip(ref_w, gs)]
        else:
            for v, p in zip(ref_view, ref_w):
                v.copy_(p.data)
            rg = place(gs, goffs)
            ref_plan.backward_(rg, "complicated")
            rg = [g.clone() for g in rg]
        for p, g in zip(ref_w, rg):
            p.grad = g
        for grp in opt.param_groups:
            grp["lr"] = lr
        opt.step()
        if style == "truncated":
            with torch.no_grad():
                for p in ref_w:
                    p.clamp_(-1, 1)
        plan.fused_step_(place(gs, goffs), style, lr, momentum, wd, nesterov)
        for i, p in enumerate(ref_w):
            w = f"{what} step {step} tensor {i} (n={xs[i].size})"
            assert torch.equal(plan._master[i].view(-1), p.data.view(-1)), f"{w}: master"
            buf = opt.state[p].get("momentum_buffer")
            if momentum == 0.0:
                assert buf is None and not bool(plan.momentum_buffers[i].any()), f"{w}: momentum buffer written"
            else:
                assert bool((plan.momentum_buffers[i].view(-1) == buf.view(-1)).all()), f"{w}: momentum"
            assert_same(live[i], O.uniform_fwd(host(p), levels[i], bucket)[0], f"{w}: quantized")
    plan.close()
    if ref_plan is not None:
        ref_plan.close()


LAYOUTS = {"aligned": (0, 0), "unaligned": (1, 2), "params_aligned": (0, 1), "grads_aligned": (1, 0)}


def layout(name, count):
    p, g = LAYOUTS[name]
    return ([0] * count if p == 0 else mixed(count, p)), ([0] * count if g == 0 else mixed(count, g))


@pytest.mark.parametrize("style", ["none", "truncated", "complicated"])
@pytest.mark.parametrize("lay", list(LAYOUTS))
@pytest.mark.parametrize("bucket", [64, 100, 256, 300, 512])
def test_fused_step_matches_torch_sgd(P, bucket, lay, style):
    """R = 2 and 4, full and ragged rows, 11 tensors, every momentum / Nesterov / weight-decay combination torch
    accepts, five steps with the learning rate changed at step 3."""
    rng = np.random.default_rng(3000 + bucket)
    b = bucket
    sizes = [1, 3, 127, 129, b - 1, b, b + 1, 3 * b + 5, b // 2, 2 * b + 7, 5]
    xs = [(rng.standard_normal(n) * 0.6).astype(F32) for n in sizes]
    lv = levels_for(len(xs))
    poffs, goffs = layout(lay, len(xs))
    for clamp_start in ((True, False) if style == "truncated" else (True,)):
        for momentum, nesterov, wd in OPT_SETS:
            run_fused(P, xs, lv, bucket, style, poffs, goffs, momentum, nesterov, wd, rng,
                      f"b={bucket} {lay} {style} clamp_start={clamp_start} mu={momentum} nesterov={nesterov} wd={wd}",
                      clamp_start)


@pytest.mark.parametrize("style", ["none", "truncated", "complicated"])
@pytest.mark.parametrize("count", [256, 300])
@pytest.mark.parametrize("bucket", [256, 512])
def test_fused_step_many_tensors(P, bucket, count, style):
    """256 tensors (row table in shared memory and gradient pointers by value, both exactly full) and ~300 (row
    table in global memory, gradient pointers through the plan's device table)."""
    rng = np.random.default_rng(4000 + bucket + count)
    sizes = many_sizes(rng, bucket, count)
    xs = [(rng.standard_normal(n) * 0.6).astype(F32) for n in sizes]
    run_fused(P, xs, levels_for(len(xs)), bucket, style, mixed(len(xs)), mixed(len(xs), 2), 0.9, True, 5e-4, rng,
              f"b={bucket} {count} tensors {style}")


def test_fused_step_refusals_leave_state_untouched(P):
    rng = np.random.default_rng(5000)
    xs = [(rng.standard_normal(n) * 0.6).astype(F32) for n in (300, 77, 512, 5)]
    gs = [rng.standard_normal(x.size).astype(F32) for x in xs]

    def state(plan, live):
        return snapshot(plan._master) + snapshot(plan.momentum_buffers) + snapshot(live)

    # bucket None with tensors of at most 512 floats: none / truncated run (one row per tensor), min/max is refused
    live = place(xs, mixed(len(xs), 1))
    plan = P.QuantizationPlan(live, levels_for(len(xs)), None)
    plan.save_and_quantize_()
    plan.fused_step_(place(gs, mixed(len(xs))), "truncated", 0.05, 0.9, 5e-4, True)
    for i in range(len(xs)):
        assert_same(live[i], O.uniform_fwd(host(plan._master[i]), levels_for(len(xs))[i], None)[0], f"bucket None fused q {i}")
    before = state(plan, live)
    with pytest.raises(NotImplementedError):
        plan.fused_step_(place(gs, mixed(len(xs))), "complicated", 0.05, 0.9, 5e-4, True)
    assert_untouched(plan._master + plan.momentum_buffers + live, before, "min/max with bucket None")
    with pytest.raises(ValueError):
        plan.fused_step_(place(gs, mixed(len(xs))), "none", 0.05, 0.0, 5e-4, True)
    assert_untouched(plan._master + plan.momentum_buffers + live, before, "Nesterov without momentum")
    plan.close()

    # a row of more than 512 floats
    live = place(xs + [np.ones(513, F32)], [0] * (len(xs) + 1))
    plan = P.QuantizationPlan(live, 16, 1024)
    plan.save_and_quantize_()
    before = snapshot(plan._master) + snapshot(live)
    with pytest.raises(NotImplementedError):
        plan.fused_step_(place(gs + [np.ones(513, F32)], [0] * (len(xs) + 1)), "none", 0.05, 0.9, 5e-4, True)
    assert_untouched(plan._master + live, before, "rows over 512 floats")
    assert not bool(plan._momentum_flat.any())
    plan.close()


# =============================================================================== 3. centroid plan
def point_sets(rng, count):
    """K = 1..32 across the four table classes (<= 4, 8, 16, 32), some with a duplicated point, some with the
    end points 0 and 1 exactly."""
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


def make_centroid_plan(P, xs, pts, bucket, soffs, doffs):
    src = place(xs, soffs)
    dst = place([np.zeros_like(x) for x in xs], doffs)
    pd = [torch.from_numpy(p).cuda() for p in pts]
    return P.CentroidPlan(src, dst, pd, bucket), dst


def nu_magnitude(g, idx, alpha, K, bucket):
    """sum_{i: idx_i = k} |fl32(g_i * alpha_row(i))| per centroid."""
    n = g.size
    a = np.repeat(np.asarray(alpha, F32), row_len(n, bucket))[:n]
    v = np.abs((g.reshape(-1) * a).astype(F32).astype(np.float64))
    return np.bincount(np.asarray(idx).reshape(-1), weights=v, minlength=K)[:K]


@pytest.mark.parametrize("count", [1, "edges", 256, 257, 601])
@pytest.mark.parametrize("bucket", [64, 100, 256, 300, 512, 700, 1024, None])
def test_centroid_plan_matches_oracle(P, bucket, count):
    """q, idx, alpha and beta bit for bit against the midpoint-rule oracle; the centroid gradient of random g inside
    the bound of its accumulation: every float32 lane column adds at most 16 * 1024 / 32 = 512 products before the
    float64 flush, so per centroid |err| <= 512 * 2^-24 * sum_{idx=k} |g * alpha| + 2^-24 * |ref_k|."""
    rng = np.random.default_rng(6000 + (bucket or 0) + (0 if count == "edges" else count))
    if count == 1:                                  # one tensor: several full rows and a ragged one, 17 points, one doubled
        xs = [(rng.standard_normal(3 * bucket + 5 if bucket else 1000) * 0.05).astype(F32)]
        pts = [np.sort(rng.random(17)).astype(F32)]
        pts[0][8] = pts[0][7]
    else:
        sizes = edge_sizes(bucket) if count == "edges" else many_sizes(rng, bucket, count)
        xs = uniform_inputs(rng, sizes, 0.05)
        pts = point_sets(rng, len(xs))
    plan, dst = make_centroid_plan(P, xs, pts, bucket, mixed(len(xs)), mixed(len(xs), 2))
    plan.forward_()
    gs = [rng.standard_normal(x.size).astype(F32) for x in xs]
    first = [t.clone() for t in plan.backward_(place(gs, mixed(len(xs), 1)))]
    again = [t.clone() for t in plan.backward_(place(gs, mixed(len(xs), 1)))]
    for i, (x, p, g) in enumerate(zip(xs, pts, gs)):
        what = f"b={bucket} count={count} tensor {i} (n={x.size} K={p.size})"
        q, idx, st = O.nonuniform_fwd(x, p, bucket, rule="midpoint")
        assert_same(dst[i], q, f"{what} q")
        assert_same(host(plan.indices[i]).astype(np.int64), idx, f"{what} idx")
        assert_same(plan.alpha[i], st["alpha"], f"{what} alpha")
        assert_same(plan.beta[i], st["beta"], f"{what} beta")
        ref = O.nonuniform_bwd_points(g, idx, st["alpha"], p.size, bucket)
        got = host(first[i]).astype(np.float64)
        tol = 512 * 2.0 ** -24 * nu_magnitude(g, idx, st["alpha"], p.size, bucket) + 2.0 ** -24 * np.abs(ref)
        assert np.all(np.abs(got - ref) <= tol), (what, got, ref)
        assert torch.equal(first[i].view(torch.int32), again[i].view(torch.int32)), f"{what}: gradient not deterministic"
    plan.close()


def exact_rows(rng, n, bucket):
    """Every row holds 0 and 2^-e (e = row % 4), everything else in between: alpha = 2^-e exactly."""
    rows, rl, _ = O.bucket_geometry(n, bucket)
    scale = np.repeat(np.ldexp(F32(1), -(np.arange(rows) % 4)).astype(F32), rl)[:n]
    x = rng.random(n, dtype=F32) * scale
    starts = np.arange(rows, dtype=np.int64) * rl
    x[starts] = 0
    second = starts[starts + 1 < np.minimum(starts + rl, n)] + 1
    x[second] = scale[second]
    return x


def plan_block_tiles(sizes):
    tiles = sum(-(-n // 1024) for n in sizes)                    # gradient tiles of 1024 elements
    return int(min(16, max(1, -(-tiles // 4736))))              # qd_plan_nonuniform_create


@pytest.mark.parametrize("sizes,bucket,block_tiles", [
    ([1_000_003], 256, 1),
    ([1, 3, 1023, 1024, 1025, 2053, 65_543, 931_000], 256, 1),
    ([1, 3, 1023, 1024, 1025, 2053, 65_543, 931_000], 100, 1),
    ([5_000_000], 100, 2),
    ([5, 1000, 2_000_003, 3_000_000], 256, 2),
    ([5, 1000, 2_000_003, 3_000_000], 100, 2),
    ([72_900_001, 5000, 3, 1000], 256, 16),
], ids=["1M-one-b256", "1M-b256", "1M-b100", "5M-one-b100", "5M-b256", "5M-b100", "73M-b256"])
def test_centroid_plan_gradient_exact_sums(P, sizes, bucket, block_tiles):
    """Data whose every sum is exact in float32: alpha = 2^-e, g small integers.  The gradient must then equal the C
    oracle BIT FOR BIT, which catches a dropped or doubled element or a wrong alpha row.  The sizes put the plan's
    gradient blocks at 1, 2 and 16 tiles; at 16 the float32 columns are flushed inside the tile loop."""
    assert plan_block_tiles(sizes) == block_tiles
    rng = np.random.default_rng(7000 + sum(sizes) % 1000 + bucket)
    xs = [exact_rows(rng, n, bucket) for n in sizes]
    pts = [np.sort(rng.random(k)).astype(F32) for k in (32, 1, 4, 16, 8, 32, 3, 17)[:len(sizes)]]
    plan, dst = make_centroid_plan(P, xs, pts, bucket, mixed(len(xs)), mixed(len(xs), 1))
    plan.forward_()
    gs = [rng.integers(-4, 5, n, dtype=np.int8).astype(F32) for n in sizes]
    grads = place(gs, [0, 1, 0, 2, 0, 3, 0, 1][:len(sizes)])
    first = [t.clone() for t in plan.backward_(grads)]
    again = [t.clone() for t in plan.backward_(grads)]
    for i, (x, p, g) in enumerate(zip(xs, pts, gs)):
        what = f"{sizes} b={bucket} tensor {i} (n={x.size} K={p.size})"
        q, idx, st = CO.nonuniform_fwd(x, p, bucket, rule="midpoint")
        assert torch.equal(dst[i].view(torch.int32), torch.from_numpy(q).cuda().view(torch.int32)), f"{what} q"
        assert torch.equal(plan.indices[i].reshape(-1).long(), torch.from_numpy(idx).cuda()), f"{what} idx"
        assert_same(plan.alpha[i], st["alpha"], f"{what} alpha")
        ref = CO.nonuniform_bwd_points(g, idx, st["alpha"], p.size, bucket)
        assert_same(first[i], ref.astype(F32), f"{what} exact gradient")
        assert torch.equal(first[i].view(torch.int32), again[i].view(torch.int32)), f"{what}: gradient not deterministic"
        del q, idx
    plan.close()
    del plan, dst, grads
    torch.cuda.empty_cache()


# =============================================================================== 4. long-row plan
@pytest.mark.parametrize("count", [1, 256, 257, 601])
def test_long_row_plan_matches_oracle(P, count):
    """bucket None with tensors beyond 1024 floats: the long-row plan (chunks of 16384 floats), tensors at float
    offsets 1..3 with lengths straddling chunk edges; save_and_quantize_, quantize_ and the truncated fix-up bit for
    bit against the oracle; min/max refused with every gradient untouched."""
    rng = np.random.default_rng(8000 + count)
    longs = [CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 5]
    if count == 1:
        sizes = [3 * CHUNK + 5]
    else:
        pool = longs + [1, 3, 1000, 1025, 2 * CHUNK]
        sizes = longs + [int(rng.choice(pool)) for _ in range(count - len(longs))]
    xs = uniform_inputs(rng, sizes) if count > 1 else [(rng.standard_normal(sizes[0]) * 0.7).astype(F32)]
    lv = levels_for(count)
    offs = [1 + i % 3 for i in range(count)]
    params = place(xs, offs)
    plan = P.QuantizationPlan(params, lv, None)
    refs = [CO.uniform_fwd(x, l, None)[0] for x, l in zip(xs, lv)]
    master = plan.save_and_quantize_()
    for i in range(count):
        assert_same(params[i], refs[i], f"long count={count} save_and_quantize_ q tensor {i} (n={xs[i].size} levels={lv[i]})")
        assert_same(master[i], xs[i], f"long count={count} master tensor {i}")
    plan.restore_master()
    plan.quantize_()
    for i in range(count):
        assert_same(params[i], refs[i], f"long count={count} quantize_ tensor {i}")
    plan.restore_master()
    gs = [rng.standard_normal(x.size).astype(F32) for x in xs]
    grads = place(gs, [1 + (i + 1) % 3 for i in range(count)])
    plan.backward_(grads, "truncated")
    for i in range(count):
        assert_same(grads[i], O.uniform_bwd_truncated(xs[i], gs[i]), f"long count={count} truncated tensor {i}")
    before = snapshot(grads)
    with pytest.raises(NotImplementedError):
        plan.backward_(grads, "complicated")
    assert_untouched(grads, before, f"long count={count} refused min/max")
    plan.close()
