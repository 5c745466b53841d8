"""The register warp path gives every row its own warp (one CTA per 8 rows).  These tests cover that row -> warp
mapping where it can go wrong: row counts on each side of the old persistent grid (SMs x 3 CTAs x 8 warps), fewer rows
than that grid, a single row, a ragged last row (n % 256 != 0) and unaligned views, for the uniform forward, the
straight-through and truncated gradients and the min/max backward.  The fused min/max results on rows of 256 floats
must also be the very bytes the persistent-grid kernel produced (tests/golden/make_golden_warp_traversal.py)."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import quant_oracle as O
from test_gpu_parity import assert_minmax_gradient, assert_same

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_golden_warp_traversal", os.path.join(HERE, "golden", "make_golden_warp_traversal.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)


@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native as N
    return N


def old_grid_rows(N):
    import ctypes
    sms = ctypes.c_int(0)
    N.check(N.lib().qd_device_info(ctypes.byref(sms), None, None))
    return sms.value * 3 * 8


def views(n, offset):
    bufs = [torch.zeros(n + offset, device="cuda") for _ in range(4)]
    return [b[offset:] for b in bufs]


def cases(N):
    w = old_grid_rows(N)
    rows = (1, 5, 100, w - 1, w, w + 1, 2 * w - 1, 2 * w + 1)
    out = [(r * 256, 0) for r in rows]
    out += [((w + 1) * 256 - 100, 0), (3 * 256 + 7, 0), ((w - 1) * 256, 1), ((2 * w + 1) * 256 - 3, 2)]
    return out


@pytest.mark.parametrize("s", [4, 16])
def test_warp_rows_match_oracle(N, s):
    lib, sp = N.lib(), N.stream_ptr()
    for i, (n, offset) in enumerate(cases(N)):
        x_np, g_np = G.inputs(n, 100 + i)
        what = f"n={n} offset={offset} s={s}"
        x, g, q, go = views(n, offset)
        x.copy_(torch.from_numpy(x_np))
        g.copy_(torch.from_numpy(g_np))
        ws = N.workspace(n, 256, x.device)
        i8 = torch.full((n,), 255, dtype=torch.uint8, device="cuda")

        q_ref, idx_ref, _ = O.uniform_fwd(x_np, s, 256)
        N.check(lib.qd_uniform_fwd(N.ptr(x), N.ptr(q), N.ptr(i8), None, None, None, None, n, 256, s, None, 0.0, 0, 0, 0,
                                   N.ptr(ws), ws.numel(), sp))
        assert_same(q.cpu().numpy(), q_ref, "forward q " + what)
        assert_same(i8.cpu().numpy().astype(np.int64), idx_ref, "forward idx " + what)

        for mode, ref in ((N.BWD_STE, g_np), (N.BWD_TRUNCATED, O.uniform_bwd_truncated(x_np, g_np))):
            q.fill_(float("nan"))
            go.fill_(float("nan"))
            N.check(lib.qd_uniform_fwd_bwd(N.ptr(x), N.ptr(g), N.ptr(q), N.ptr(go), n, 256, s, mode, N.ptr(ws), ws.numel(), sp))
            assert_same(q.cpu().numpy(), q_ref, f"mode {mode} q " + what)
            assert_same(go.cpu().numpy(), ref, f"mode {mode} gout " + what)

        q.fill_(float("nan"))
        go.fill_(float("nan"))
        N.check(lib.qd_uniform_fwd_bwd(N.ptr(x), N.ptr(g), N.ptr(q), N.ptr(go), n, 256, s, N.BWD_MINMAX, N.ptr(ws), ws.numel(), sp))
        assert_same(q.cpu().numpy(), q_ref, "min/max q " + what)
        ref, info = O.uniform_bwd_minmax(x_np, g_np, s, 256)
        assert_minmax_gradient(go.cpu().numpy(), g_np, ref, info["argmax"], info["argmin"], info["abs_sum"], info["r"], "min/max gout " + what)


def test_fused_minmax_bytes_match_persistent_grid_kernel(N):
    golden = np.load(os.path.join(HERE, "golden", "warp_traversal_minmax.npz"))
    assert [tuple(c) for c in golden["cases"].tolist()] == G.CASES
    for (n, offset, seed), q_sha, g_sha in zip(G.CASES, golden["q_sha256"], golden["gout_sha256"]):
        x, g = G.inputs(n, seed)
        q, go = G.run_fused_minmax(x, g, offset)
        assert np.array_equal(G.digest(q), q_sha), f"q bytes differ: n={n} offset={offset}"
        assert np.array_equal(G.digest(go), g_sha), f"gout bytes differ: n={n} offset={offset}"
