"""Every kernel the per-tensor uniform ops can dispatch to, against the oracle.

run_rows / launch_block / launch_staged / with_row_regs (csrc/qd_quant.cu, csrc/qd_launch.h) pick a kernel from the op,
the backward mode, whether q is written, the row length L and the alignment of every pointer.  This file walks L through
BOUNDARIES, one value on each side of every threshold, and at each L runs

  * qd_uniform_fwd (q, idx_u8, alpha, beta, argmin, argmax) for s in {2, 16, 256}, plain, with max_element and with a
    device mean, and with stochastic rounding;
  * qd_uniform_fwd_bwd and qd_uniform_bwd in the straight-through, truncated and min/max modes;
  * qd_scale_down (with and without xhat) and qd_inv_scale_down (with and without a device mean);

on views of x, g, q, gout and idx_u8 at offsets chosen independently of each other, and with q aliasing x and gout
aliasing g.  Everything is bit for bit against oracle/quant_oracle.py (the C oracle above ORACLE_C_ABOVE elements),
except the min/max gradient, which has the a5 bar of tests/test_gpu_parity.py.  Every output buffer starts out holding a
NaN sentinel, and the guard elements around every view must still hold it afterwards.

The host-buffer entry points, the grid path's workspace contract and a hypothesis sweep of the fused op sit at the end;
test_boundary_list_tracks_the_dispatch_thresholds runs without a GPU and fails when a threshold in the sources moves
without this list."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st

from oracle import c_oracle as CO
from oracle import quant_oracle as O
from test_gpu_parity import assert_minmax_gradient, assert_same

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
gpu = pytest.mark.gpu

# Row lengths L (floats); None is bucket_size=None, one row spanning the tensor.
BOUNDARIES = [
    1, 2, 3, 4, 5, 7,       # rows shorter than one float4: the scalar warp kernel (rows_vectorizable needs L % 4 == 0)
    100,                    # ragged R = 2 row
    255, 256, 257,          # with_row_regs: R = 2 up to 256 (256 = the full, unpredicated variant)
    384,                    # ragged R = 4 row
    511, 512, 513,          # with_row_regs: R = 4 up to 512; ragged_minmax (run_rows) from 513
    768, 1000,              # ragged R = 8 rows; min/max on the staged ring (ragged_minmax)
    1023, 1024, 1025,       # ragged_minmax below 1024; the warp path ends at 1024 (run_rows)
    2047, 2048, 2049,       # launch_staged: 64 threads below 2048; kWarp2MinmaxMaxRow; kWarpTwoPassMaxRow
    3072, 3073,             # kTwoStageMaxRow: two rows in flight per CTA up to here
    4096, 4097,             # 2 * kWarpTwoPassMaxRow: scale / stats / stochastic leave the warp two-pass kernel
    12288, 12289,           # launch_staged: 256 threads up to 12288
    24576, 24577,           # launch_staged: 512 threads up to 24576, 1024 above
    49151, 49152, 49153,    # QD_MAX_STAGED_BUCKET: the grid path above, and min/max is refused
    65536, 100000,          # grid rows of several 16384-float chunks (kGridChunk), whole and ragged
    None,                   # grid path; min/max is refused
]

ORACLE_C_ABOVE = 4 << 20        # the NumPy oracle is slow beyond this; the C restatement takes over
MAX_FLOATS = 16 << 20           # no tensor above 64 MiB: the GPUs are shared
PAD = 8                         # guard elements after every view (and up to 3 before it)
SENT = 0x7FBADBAD               # NaN payload that no kernel writes
SENT8 = 0xAB
MODES = ("ste", "truncated", "minmax")


# ----------------------------------------------------------------------------------------------- no GPU needed
def _constant(text, name):
    m = re.search(rf"constexpr\s+int\s+{name}\s*=\s*(\d+)\s*;", text)
    assert m, f"{name} not found"
    return int(m.group(1))


def test_boundary_list_tracks_the_dispatch_thresholds():
    """Each dispatch threshold of the sources, and one past it, is in BOUNDARIES: a pull request that moves a threshold
    without moving these tests fails here, on any machine."""
    csrc = os.path.join(ROOT, "quantized_distillation_b200", "csrc")
    read = lambda *p: open(os.path.join(*p)).read()  # noqa: E731
    staged, block, quant = read(csrc, "qd_staged_path.cuh"), read(csrc, "qd_block_path.cuh"), read(csrc, "qd_quant.cu")
    m = re.search(r"#define\s+QD_MAX_STAGED_BUCKET\s+(\d+)", read(ROOT, "include", "qd_b200.h"))
    assert m
    two_pass = _constant(block, "kWarpTwoPassMaxRow")
    limits = {"kTwoStageMaxRow": _constant(staged, "kTwoStageMaxRow"), "kWarpTwoPassMaxRow": two_pass,
              "2 * kWarpTwoPassMaxRow": 2 * two_pass, "kWarp2MinmaxMaxRow": _constant(block, "kWarp2MinmaxMaxRow"),
              "QD_MAX_STAGED_BUCKET": int(m.group(1))}
    # the CTA-size steps of launch_staged are literals
    body = quant[quant.index("static int launch_staged("):]
    body = body[:body.index("\n}\n")]
    for v in re.findall(r"L <= (\d+)\)", body):
        limits[f"launch_staged L <= {v}"] = int(v)
    assert len(limits) >= 7, limits
    for what, v in limits.items():
        assert v in BOUNDARIES and v + 1 in BOUNDARIES, f"{what} = {v}: add {v} and {v + 1} to BOUNDARIES"


# ----------------------------------------------------------------------------------------------- helpers
@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native as N
    return N


def sm_count(N):
    sms = ctypes.c_int(0)
    N.check(N.lib().qd_device_info(ctypes.byref(sms), None, None))
    return sms.value


def ring_resident_ctas(N, L):
    """Upper bound of the staged-ring CTAs resident at once for rows of L floats (launch_staged's shape; 2048 threads,
    32 CTAs and 228 KB of shared memory per SM)."""
    stages, threads = (2, 64 if L < 2048 else 128) if L <= 3072 else (1, 256 if L <= 12288 else 512 if L <= 24576 else 1024)
    smem = stages * (-(-L // 32) * 32) * 4
    return sm_count(N) * min(32, 2048 // threads, (228 << 10) // (smem + 1024))


def shapes(N, L):
    """Tensor sizes n = rows * L + tail for tail in {0, 1, 3, L - 1}.  One size per L has many rows: on the staged ring
    more than twice the resident CTAs, so every CTA takes rows of both alignments (odd L) into the same ring slots."""
    if L is None:
        return [1, 7, 1000, 16384, 49152, 49153, 1_000_003, 3_000_017]
    tails = sorted({t for t in (0, 1, 3, L - 1) if t < L})
    if L > 49152:
        big_rows = 40                                        # grid path: 3 .. 40 rows
    elif L > 1024 or 512 < L < 1024:
        big_rows = min(2 * ring_resident_ctas(N, L) + 3, MAX_FLOATS // L - 1)
    else:
        big_rows = max(3, (1 << 20) // L)
    small_rows = 3
    big_tail = 3 if 3 in tails else tails[-1]
    out = [big_rows * L + big_tail] + [small_rows * L + t for t in tails if t != big_tail]
    return out


def make_inputs(n, seed):
    """x with |x| > 1 present (truncation fires) and, on half the elements, values on a 1/256 grid (ties at the row
    extremes and at the quantization levels); g standard normal.  No -0.0: which zero a kernel's min / max reduction
    returns for a row whose extreme is a tie of -0.0 and +0.0 is not pinned (DESIGN.md section 4)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n) * 0.6
    x = (np.where(rng.random(n) < 0.5, np.round(x * 256) / 256, x) + 0.0).astype(np.float32)
    g = rng.standard_normal(n).astype(np.float32)
    return x, g


def oracle_fwd(x, s, bucket, mean=None, max_element=False):
    """(q, idx, alpha, beta, argmin, argmax) of O.uniform_fwd on O.pre_ops(x, mean, max_element); the C restatement
    above ORACLE_C_ABOVE elements (it takes pre-processed input, and the mean is added back in float32 as O does)."""
    if x.size <= ORACLE_C_ABOVE:
        q, idx, stt = O.uniform_fwd(x, s, bucket, subtract_mean=mean is not None, max_element=max_element, mean=mean)
        return q.reshape(-1), idx.reshape(-1), stt
    flat, m = O.pre_ops(x, mean is not None, max_element, mean)
    q, idx, stt = CO.uniform_fwd(flat, s, bucket)
    if mean is not None or max_element is not False:
        q = (q + m).astype(np.float32)
    return q, idx, stt


def oracle_minmax(x, g, s, bucket, q_ref):
    """(gout, argmax' positions, argmin' positions, sum |v_j| per row, r_b per row)."""
    if x.size <= ORACLE_C_ABOVE:
        ref, info = O.uniform_bwd_minmax(x, g, s, bucket)
        return ref.reshape(-1), info["argmax"], info["argmin"], info["abs_sum"], info["r"]
    ref, abs_sum, r = CO.uniform_bwd_minmax_ex(x, g, s, bucket)
    rows, row_len, padded = O.bucket_geometry(x.size, bucket)
    qp = np.concatenate([q_ref, np.full(padded - x.size, q_ref[-1], np.float32)]).reshape(rows, row_len)
    base = np.arange(rows, dtype=np.int64) * row_len
    return ref, base + qp.argmax(1), base + qp.argmin(1), abs_sum, r


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def same_bits(got, want, what):
    """Bit equality of two device tensors (float32 compared as int32: NaN sentinels count as mismatches)."""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    a, b = (got.view(torch.int32), want.view(torch.int32)) if got.dtype == torch.float32 else (got, want)
    if not torch.equal(a, b):
        bad = torch.nonzero(a != b).view(-1)
        raise AssertionError(f"{what}: {bad.numel()} mismatches, first at {bad[:5].tolist()}: "
                             f"{got[bad[:5]].tolist()} vs {want[bad[:5]].tolist()}")


def check_minmax(go, g, ref, pos_max, pos_min, abs_sum, r, what):
    """The a5 bar (assert_minmax_gradient) with the full-tensor part on the device: nothing outside argmax' / argmin'
    changes, and the two positions of each row are inside the summation-order tolerance of the oracle."""
    pmax, pmin = cuda(pos_max), cuda(pos_min)
    changed = go.view(torch.int32) != g.view(torch.int32)
    changed[pmax] = False
    changed[pmin] = False
    if bool(changed.any()):
        bad = torch.nonzero(changed).view(-1)[:5].tolist()
        raise AssertionError(f"{what}: element outside argmin'/argmax' changed at {bad}")
    pos = torch.cat([pmax, pmin])
    rows = len(pos_max)
    assert_minmax_gradient(go[pos].cpu().numpy(), g[pos].cpu().numpy(), ref[pos].cpu().numpy(), np.arange(rows),
                           rows + np.arange(rows), abs_sum, r, what)


def offset_sets(seed):
    """(x, g, q, gout, idx_u8) offsets, in floats (idx_u8 in bytes): all aligned, all at k = 1..3, each pointer alone at 1,
    x aligned with the rest not and the reverse, and four seeded random assignments."""
    out = [(0, 0, 0, 0, 0)] + [(k,) * 5 for k in (1, 2, 3)]
    out += [tuple(int(i == j) for j in range(5)) for i in range(5)]
    out += [(0, 1, 3, 2, 1), (2, 0, 0, 0, 0)]
    rng = np.random.default_rng(seed)
    out += [tuple(int(v) for v in rng.integers(0, 4, 5)) for _ in range(4)]
    return out


class Views:
    """Sentinel-filled buffers with PAD guard elements, and views of n elements at chosen offsets into them."""

    def __init__(self, n, padded=None):
        self.n = n
        self.bufs = {k: torch.empty(n + PAD, dtype=torch.float32, device="cuda") for k in ("x", "g", "q", "go")}
        self.bufs["i8"] = torch.empty(n + PAD, dtype=torch.uint8, device="cuda")
        self.bufs["xh"] = torch.empty((padded or n) + PAD, dtype=torch.float32, device="cuda")
        self.used = {}

    def reset(self):
        for k, b in self.bufs.items():
            (b.fill_(SENT8) if b.dtype == torch.uint8 else b.view(torch.int32).fill_(SENT))
        self.used = {}

    def view(self, key, off, length=None):
        length = self.n if length is None else length
        self.used[key] = (off, length)
        return self.bufs[key][off:off + length]

    def check_guards(self, what):
        for k, b in self.bufs.items():
            off, length = self.used.get(k, (0, 0))
            s = SENT8 if b.dtype == torch.uint8 else SENT
            raw = b if b.dtype == torch.uint8 else b.view(torch.int32)
            for part, name in ((raw[:off], "before"), (raw[off + length:], "after")):
                if part.numel() and not bool((part == s).all()):
                    raise AssertionError(f"{what}: {k} written {name} its view")


def fresh(shape, dtype):
    """A device tensor holding the sentinel (NaN payload SENT, byte SENT8, or -7 for int64)."""
    t = torch.empty(shape, dtype=dtype, device="cuda")
    if dtype == torch.float32:
        t.view(torch.int32).fill_(SENT)
    else:
        t.fill_(SENT8 if dtype == torch.uint8 else -7)
    return t


def bucket_arg(L):
    return 0 if L is None else L


def minmax_refused(N, n, bucket):
    """True where the min/max backward is refused: bucket None (or 0), or rows beyond QD_MAX_STAGED_BUCKET floats."""
    return not bucket or N.geometry(n, bucket)[1] > N.MAX_STAGED_BUCKET


# ----------------------------------------------------------------------------------------------- forward, every L
@gpu
@pytest.mark.parametrize("L", BOUNDARIES, ids=str)
def test_forward_every_branch(N, L):
    """qd_uniform_fwd: q, idx_u8, alpha, beta, argmin, argmax bit for bit, s in {2, 16, 256}, at every offset set and
    with q aliasing x; the same with max_element, a device mean, and both."""
    lib, sp, b = N.lib(), N.stream_ptr(), bucket_arg(L)
    mean_val = np.float32(0.1875)
    mean_d = cuda(np.array([mean_val], np.float32))
    for si, n in enumerate(shapes(N, L)):
        x, _ = make_inputs(n, 1000 + si)
        xd = cuda(x)
        rows = N.geometry(n, b)[0]
        ws = N.workspace(n, b, xd.device)
        V = Views(n)
        variants = [(s, None, False) for s in (2, 16, 256)] + [(16, None, 0.75), (16, mean_val, False), (256, mean_val, 0.5)]
        for s, mean, me in variants:
            q, idx, stt = oracle_fwd(x, s, L, mean, me)
            qr, ir = cuda(q), cuda(idx.astype(np.uint8))
            refs = [cuda(stt[k]) for k in ("alpha", "beta", "argmin", "argmax")]
            cases = [(o, False) for o in offset_sets(si)] + [((0,) * 5, True), ((1, 0, 1, 0, 1), True), ((3, 0, 3, 0, 2), True)]
            for (ox, _, oq, _, oi), alias in cases:
                what = f"fwd n={n} L={L} s={s} mean={mean} max_element={me} offsets x={ox} q={oq} idx={oi} q is x={alias}"
                V.reset()
                xv = V.view("x", ox)
                xv.copy_(xd)
                qv = xv if alias else V.view("q", oq)
                iv = V.view("i8", oi)
                outs = [fresh(rows, torch.float32), fresh(rows, torch.float32), fresh(rows, torch.int64), fresh(rows, torch.int64)]
                N.check(lib.qd_uniform_fwd(N.ptr(xv), N.ptr(qv), N.ptr(iv), *[N.ptr(t) for t in outs], n, b, s,
                                           None if mean is None else N.ptr(mean_d), 0.0 if me is False else me, 0, 0, 0,
                                           N.ptr(ws), ws.numel(), sp))
                same_bits(qv, qr, what + " q")
                same_bits(iv, ir, what + " idx_u8")
                for t, r_, k in zip(outs, refs, ("alpha", "beta", "argmin", "argmax")):
                    same_bits(t, r_, f"{what} {k}")
                V.check_guards(what)


# ----------------------------------------------------------------------------------------------- backward, every L
@gpu
@pytest.mark.parametrize("L", BOUNDARIES, ids=str)
def test_fused_and_backward_every_branch(N, L):
    """qd_uniform_fwd_bwd and qd_uniform_bwd in the three modes at every offset set: q bit for bit, the straight-through
    and truncated gradients bit for bit, the min/max gradient inside the a5 bar and changing the same elements fused and
    alone.  With q aliasing x, gout aliasing g, or both, every output has the bits of the call without aliasing.  Where
    min/max is refused the call returns QD_ERR_UNSUPPORTED and leaves q and gout as they were."""
    lib, sp, b = N.lib(), N.stream_ptr(), bucket_arg(L)
    mode_of = {"ste": N.BWD_STE, "truncated": N.BWD_TRUNCATED, "minmax": N.BWD_MINMAX}
    for si, n in enumerate(shapes(N, L)):
        s = (2, 16, 256)[si % 3]
        x, g = make_inputs(n, 2000 + si)
        xd, gd = cuda(x), cuda(g)
        ws = N.workspace(n, b, xd.device)
        q, _, _ = oracle_fwd(x, s, L)
        qr = cuda(q)
        trunc = cuda(O.uniform_bwd_truncated(x, g))
        refused = minmax_refused(N, n, L)
        mm = None if refused else oracle_minmax(x, g, s, L, q)
        mmr = None if mm is None else cuda(mm[0])
        W = Views(n)
        cases = [(o, False, False) for o in offset_sets(3000 + si)]
        cases += [(o, aq, ag) for o in ((0,) * 5, (1, 2, 1, 2, 0), (0, 3, 0, 3, 0)) for aq, ag in ((1, 0), (0, 1), (1, 1))]
        for mode in MODES:
            for (ox, og, oq, ogo, _), aq, ag in cases:
                oq, ogo = (ox if aq else oq), (og if ag else ogo)
                what = f"{mode} n={n} L={L} s={s} offsets x={ox} g={og} q={oq} gout={ogo} q is x={bool(aq)} gout is g={bool(ag)}"
                results = []
                for fused in (True, False):
                    for alias in ((False, True) if (aq or ag) else (False,)):
                        W.reset()
                        xv, gv = W.view("x", ox), W.view("g", og)
                        xv.copy_(xd)
                        gv.copy_(gd)
                        qv = xv if (alias and aq) else W.view("q", oq)
                        gov = gv if (alias and ag) else W.view("go", ogo)
                        tag = f"{what} {'fused' if fused else 'alone'}{' aliased' if alias else ''}"
                        if fused:
                            rc = lib.qd_uniform_fwd_bwd(N.ptr(xv), N.ptr(gv), N.ptr(qv), N.ptr(gov), n, b, s, mode_of[mode],
                                                        N.ptr(ws), ws.numel(), sp)
                        else:
                            rc = lib.qd_uniform_bwd(N.ptr(xv), N.ptr(gv), N.ptr(gov), n, b, s, mode_of[mode], N.ptr(ws),
                                                    ws.numel(), sp)
                        if mode == "minmax" and refused:
                            assert rc == N.QD_ERR_UNSUPPORTED, (tag, rc)
                            torch.cuda.synchronize()
                            same_bits(qv, xd if (alias and aq) else fresh(n, torch.float32), tag + " q")
                            same_bits(gov, gd if (alias and ag) else fresh(n, torch.float32), tag + " gout")
                            W.check_guards(tag)
                            continue
                        N.check(rc)
                        if fused:
                            same_bits(qv, qr, tag + " q")
                        if mode == "ste":
                            same_bits(gov, gd, tag + " gout")
                        elif mode == "truncated":
                            same_bits(gov, trunc, tag + " gout")
                        else:
                            check_minmax(gov, gd, mmr, mm[1], mm[2], mm[3], mm[4], tag + " gout")
                        W.check_guards(tag)
                        results.append((fused, alias, qv.clone() if fused else None, gov.clone()))
                if mode == "minmax" and results:
                    # fused and alone may sum r_b in different orders, but they change the same elements
                    masks = [(r_[3] != gd) for r_ in results]
                    for m_ in masks[1:]:
                        assert torch.equal(m_, masks[0]), what + ": fused and stand-alone min/max change different elements"
                for fused in (True, False):
                    same = [r_ for r_ in results if r_[0] == fused]
                    for r_ in same[1:]:                       # aliased call: the bits of the call without aliasing
                        if fused:
                            same_bits(r_[2], same[0][2], what + " aliased q")
                        same_bits(r_[3], same[0][3], what + f" aliased gout ({'fused' if fused else 'alone'})")


# ----------------------------------------------------------------------------------------------- scale, every L
@gpu
@pytest.mark.parametrize("L", BOUNDARIES, ids=str)
def test_scale_down_and_inverse_every_branch(N, L):
    """qd_scale_down: xhat (padded layout), alpha, beta, argmin, argmax bit for bit; the stats-only call (xhat NULL)
    returns the same state.  qd_inv_scale_down on an arbitrary y, with and without a device mean.  x / xhat and y / out
    at independent offsets."""
    lib, sp, b = N.lib(), N.stream_ptr(), bucket_arg(L)
    mean_val = np.float32(-0.3125)
    mean_d = cuda(np.array([mean_val], np.float32))
    for si, n in enumerate(shapes(N, L)):
        x, _ = make_inputs(n, 4000 + si)
        rows, row_len, padded = N.geometry(n, b)
        xd = cuda(x)
        ws = N.workspace(n, b, xd.device)
        xh, stt = O.scale_down(x, L)
        xhr = cuda(xh.reshape(-1))
        refs = [cuda(stt[k]) for k in ("alpha", "beta", "argmin", "argmax")]
        rng = np.random.default_rng(5000 + si)
        y = rng.random(padded).astype(np.float32).reshape(rows, row_len)
        ya = (y * stt["alpha"][:, None]).astype(np.float32)
        inv_plain = (ya + stt["beta"][:, None]).astype(np.float32).reshape(-1)[:n]
        inv_mean = (inv_plain + mean_val).astype(np.float32)
        yd, inv_plain, inv_mean = cuda(y.reshape(-1)), cuda(inv_plain), cuda(inv_mean)
        V = Views(n, padded)
        yb = torch.empty(padded + PAD, device="cuda")
        for ox, oy, oxh, oout, _ in offset_sets(6000 + si):
            what = f"scale n={n} L={L} offsets x={ox} xhat={oxh} y={oy} out={oout}"
            for stats_only in (False, True):
                V.reset()
                xv = V.view("x", ox)
                xv.copy_(xd)
                xhv = None if stats_only else V.view("xh", oxh, padded)
                outs = [fresh(rows, torch.float32), fresh(rows, torch.float32), fresh(rows, torch.int64), fresh(rows, torch.int64)]
                N.check(lib.qd_scale_down(N.ptr(xv), N.ptr(xhv), *[N.ptr(t) for t in outs], n, b, None, 0.0, N.ptr(ws),
                                          ws.numel(), sp))
                if not stats_only:
                    same_bits(xhv, xhr, what + " xhat")
                for t, r_, k in zip(outs, refs, ("alpha", "beta", "argmin", "argmax")):
                    same_bits(t, r_, f"{what} {k}{' stats only' if stats_only else ''}")
                V.check_guards(what)
            for mean, ref in ((None, inv_plain), (mean_d, inv_mean)):
                V.reset()
                yv = yb[oy:oy + padded]
                yv.copy_(yd)
                outv = V.view("q", oout)
                N.check(lib.qd_inv_scale_down(N.ptr(yv), N.ptr(outv), N.ptr(refs[0]), N.ptr(refs[1]), N.ptr(mean), n, b, sp))
                same_bits(outv, ref, f"{what} inverse mean={mean is not None}")
                V.check_guards(what + " inverse")


# ----------------------------------------------------------------------------------------------- stochastic, every L
@gpu
@pytest.mark.parametrize("L", BOUNDARIES, ids=str)
def test_stochastic_every_branch(N, L):
    """Stochastic rounding, with the checks of test_stochastic_rounding_every_path: alpha / beta bit for bit, the level
    is floor(x_hat * S) or one above and never above the top, q is the oracle's chain given the up / down decisions;
    where the tensor is large enough, E[up | frac] = frac within 4 sigma and another seed or offset redraws.  The draw
    belongs to the element, so views at other offsets give the same levels."""
    lib, sp, b, s = N.lib(), N.stream_ptr(), bucket_arg(L), 4
    for si, n in enumerate(shapes(N, L)):
        x, _ = make_inputs(n, 7000 + si)
        rows = N.geometry(n, b)[0]
        xd = cuda(x)
        ws = N.workspace(n, b, xd.device)
        xh, stt = O.scale_down(x, L)
        S = np.float32(s - 1)
        prob = (S * xh).astype(np.float32).reshape(-1)[:n]
        lo = np.floor(prob)
        frac = (prob - lo).astype(np.float32)
        V = Views(n)

        def draw(ox, oq, oi, seed=1234, offset=0):
            V.reset()
            xv = V.view("x", ox)
            xv.copy_(xd)
            qv, iv = V.view("q", oq), V.view("i8", oi)
            alpha, beta = fresh(rows, torch.float32), fresh(rows, torch.float32)
            N.check(lib.qd_uniform_fwd(N.ptr(xv), N.ptr(qv), N.ptr(iv), N.ptr(alpha), N.ptr(beta), None, None, n, b, s, None,
                                       0.0, 1, seed, offset, N.ptr(ws), ws.numel(), sp))
            V.check_guards(f"stochastic n={n} L={L}")
            return qv.clone(), iv.clone(), alpha, beta

        q, lv, alpha, beta = draw(0, 0, 0)
        what = f"stochastic n={n} L={L}"
        assert_same(alpha.cpu().numpy(), stt["alpha"], what + " alpha")
        assert_same(beta.cpu().numpy(), stt["beta"], what + " beta")
        lvh = lv.cpu().numpy().astype(np.float32)
        up = lvh == lo + 1
        assert np.all(up | (lvh == lo)), what + ": level is neither floor nor floor + 1"
        assert not np.any(up & (frac == 0) & (lo == s - 1)), what + ": rounded up past the top level"
        u = np.full(xh.size, 2.0, np.float32)
        u[:n][up] = 0.0
        qref, _ = O.uniform_fwd_stochastic(x, s, L, u)
        assert_same(q.cpu().numpy(), qref.reshape(-1), what + " q")
        for k in range(10):
            m = (frac >= k / 10) & (frac < (k + 1) / 10)
            cnt = int(m.sum())
            if cnt < 1000:
                continue
            p = frac[m].astype(np.float64)
            sigma = np.sqrt((p * (1 - p)).sum()) / cnt
            assert abs(up[m].mean() - p.mean()) < 4 * sigma + 2.0 ** -24, (what, k, up[m].mean(), p.mean(), sigma)
        for ox, oq, oi in ((1, 1, 1), (0, 3, 2), (2, 0, 0)):
            q2, lv2, _, _ = draw(ox, oq, oi)
            same_bits(lv2, lv, f"{what} levels at offsets x={ox} q={oq} idx={oi}")
            same_bits(q2, q, f"{what} q at offsets x={ox} q={oq} idx={oi}")
        live = cuda((frac > 0.1) & (frac < 0.9))               # elements whose level the draw decides
        if int(live.sum()) >= 20000:
            for other in (draw(0, 0, 0, seed=1235)[1], draw(0, 0, 0, offset=1 << 20)[1]):
                differ = (other != lv)[live].float().mean().item()
                assert differ > 0.05, (what + ": another seed / offset draws the same levels", differ)


# ----------------------------------------------------------------------------------------------- grid workspace
@gpu
@pytest.mark.parametrize("n, bucket", [(3_000_017, 0), (40 * 65536 + 3, 65536), (7 * 100000 + 99999, 100000), (49153, 0)])
def test_grid_path_workspace_contract(N, n, bucket):
    """Rows beyond QD_MAX_STAGED_BUCKET floats use the caller's workspace: exactly qd_workspace_bytes(n, bucket) works
    for every op; one byte less, or NULL, returns QD_ERR_WORKSPACE before anything is written."""
    lib, sp = N.lib(), N.stream_ptr()
    L = None if bucket == 0 else bucket
    x, g = make_inputs(n, 8000 + n % 1000)
    xd, gd = cuda(x), cuda(g)
    rows, _, padded = N.geometry(n, bucket)
    need = int(lib.qd_workspace_bytes(n, bucket))
    assert need > 0
    q_ref, idx_ref, stt = oracle_fwd(x, 16, L)
    xh_ref, _ = O.scale_down(x, L)
    trunc = O.uniform_bwd_truncated(x, g)
    for size, label in ((need, "exact"), (need - 1, "one byte short"), (None, "NULL")):
        buf = torch.empty(need, dtype=torch.uint8, device="cuda")
        wp, wb = (None, 0) if size is None else (N.ptr(buf), size)
        q, go, xh, i8 = fresh(n, torch.float32), fresh(n, torch.float32), fresh(padded, torch.float32), fresh(n, torch.uint8)
        per_row = [fresh(rows, torch.float32), fresh(rows, torch.float32), fresh(rows, torch.int64), fresh(rows, torch.int64)]
        keep = [t.clone() for t in (q, go, xh, i8, *per_row)]
        calls = {
            "fwd": lambda: lib.qd_uniform_fwd(N.ptr(xd), N.ptr(q), N.ptr(i8), *[N.ptr(t) for t in per_row], n, bucket, 16, None,
                                              0.0, 0, 0, 0, wp, wb, sp),
            "stochastic": lambda: lib.qd_uniform_fwd(N.ptr(xd), N.ptr(q), None, None, None, None, None, n, bucket, 16, None, 0.0,
                                                     1, 5, 0, wp, wb, sp),
            "fwd_bwd truncated": lambda: lib.qd_uniform_fwd_bwd(N.ptr(xd), N.ptr(gd), N.ptr(q), N.ptr(go), n, bucket, 16,
                                                                N.BWD_TRUNCATED, wp, wb, sp),
            "bwd truncated": lambda: lib.qd_uniform_bwd(N.ptr(xd), N.ptr(gd), N.ptr(go), n, bucket, 16, N.BWD_TRUNCATED, wp, wb, sp),
            "scale_down": lambda: lib.qd_scale_down(N.ptr(xd), N.ptr(xh), *[N.ptr(t) for t in per_row], n, bucket, None, 0.0, wp,
                                                    wb, sp),
            "stats": lambda: lib.qd_scale_down(N.ptr(xd), None, *[N.ptr(t) for t in per_row], n, bucket, None, 0.0, wp, wb, sp),
        }
        for name, call in calls.items():
            rc = call()
            what = f"{name} n={n} bucket={bucket} workspace {label}"
            if size == need:
                N.check(rc)
                continue
            assert rc == N.QD_ERR_WORKSPACE, (what, rc)
            torch.cuda.synchronize()
            for t, k in zip((q, go, xh, i8, *per_row), keep):
                same_bits(t, k, what + ": an output was written")
        if size == need:
            # the last calls left: q / idx from "fwd_bwd truncated" and "fwd", xhat and the state from "scale_down"
            same_bits(q, cuda(q_ref), "q with the exact workspace")
            same_bits(i8, cuda(idx_ref.astype(np.uint8)), "idx with the exact workspace")
            same_bits(go, cuda(trunc), "truncated gout with the exact workspace")
            same_bits(xh, cuda(xh_ref.reshape(-1)), "xhat with the exact workspace")
            for t, k in zip(per_row, ("alpha", "beta", "argmin", "argmax")):
                same_bits(t, cuda(stt[k]), k + " with the exact workspace")


# ----------------------------------------------------------------------------------------------- host entry points
HOST_CASES = [
    # (n, bucket, pinned): the route it takes
    (1_000_003, 1000, True),        # pinned, <= 8 Mi elements: one launch on the host pointers
    (3_000_001, 256, True),
    (9_000_017, 1000, True),        # pinned, > 8 Mi: chunked pipeline
    (2_097_017, 1000, False),       # pageable (always chunked); the last chunk (17 elements) is shorter than a bucket
    (3_000_001, 65536, False),      # buckets beyond QD_MAX_STAGED_BUCKET in the chunked pipeline
    (9_000_001, 50000, True),
    (3_000_001, 0, False),          # bucket None larger than a chunk: the whole tensor staged on the device
    (3_000_001, 0, True),
    (300_001, 0, True),             # bucket None within a chunk, pinned: one launch
]


@gpu
@pytest.mark.parametrize("n, bucket, pinned", HOST_CASES)
def test_host_entry_points(N, n, bucket, pinned):
    """qd_uniform_fwd_host and qd_uniform_fwd_bwd_host in the three modes, with |x| > 1 present: bit for bit the resident
    call, and for the forward and the truncated gradient also the oracle.  Where the resident call refuses min/max
    (bucket None, rows beyond QD_MAX_STAGED_BUCKET), the host call refuses too and leaves q and gout as they were."""
    lib, sp, dev = N.lib(), N.stream_ptr(), torch.cuda.current_device()
    L = None if bucket == 0 else bucket
    x, g = make_inputs(n, 9000 + n % 997)
    host = (lambda a: torch.from_numpy(a).pin_memory()) if pinned else (lambda a: torch.from_numpy(a.copy()))
    hx, hg = host(x), host(g)
    q_ref, _, _ = oracle_fwd(x, 16, L)
    q_ref_t = torch.from_numpy(q_ref)
    xd, gd = hx.cuda(), hg.cuda()
    ws = N.workspace(n, bucket, xd.device)
    hq = host(np.zeros(n, np.float32))
    hq.view(torch.int32).fill_(SENT)
    N.check(lib.qd_uniform_fwd_host(N.ptr(hx), N.ptr(hq), n, bucket, 16, dev))
    assert torch.equal(hq.view(torch.int32), q_ref_t.view(torch.int32)), f"host fwd n={n} bucket={bucket} pinned={pinned}"
    for mode in (N.BWD_STE, N.BWD_TRUNCATED, N.BWD_MINMAX):
        what = f"host fwd_bwd mode={mode} n={n} bucket={bucket} pinned={pinned}"
        hq.view(torch.int32).fill_(SENT)
        hgo = host(np.zeros(n, np.float32))
        hgo.view(torch.int32).fill_(SENT)
        qd, god = torch.empty_like(xd), torch.empty_like(gd)
        rc_dev = lib.qd_uniform_fwd_bwd(N.ptr(xd), N.ptr(gd), N.ptr(qd), N.ptr(god), n, bucket, 16, mode, N.ptr(ws), ws.numel(), sp)
        rc = lib.qd_uniform_fwd_bwd_host(N.ptr(hx), N.ptr(hg), N.ptr(hq), N.ptr(hgo), n, bucket, 16, mode, dev)
        assert rc == rc_dev, (what, rc, rc_dev)
        if rc != N.QD_OK:
            assert rc == N.QD_ERR_UNSUPPORTED and mode == N.BWD_MINMAX and minmax_refused(N, n, bucket), (what, rc)
            assert bool((hq.view(torch.int32) == SENT).all()) and bool((hgo.view(torch.int32) == SENT).all()), what + ": written"
            continue
        assert torch.equal(hq.view(torch.int32), qd.cpu().view(torch.int32)), what + " q vs resident"
        assert torch.equal(hgo.view(torch.int32), god.cpu().view(torch.int32)), what + " gout vs resident"
        assert torch.equal(hq.view(torch.int32), q_ref_t.view(torch.int32)), what + " q vs oracle"
        if mode == N.BWD_STE:
            assert torch.equal(hgo.view(torch.int32), hg.view(torch.int32)), what + " gout"
        if mode == N.BWD_TRUNCATED:
            want = torch.from_numpy(O.uniform_bwd_truncated(x, g))
            assert bool((want != torch.from_numpy(g)).any()), "no |x| > 1: the truncated check would be vacuous"
            assert torch.equal(hgo.view(torch.int32), want.view(torch.int32)), what + " gout vs oracle"


# ----------------------------------------------------------------------------------------------- randomised
def _near_boundaries():
    return sorted({b + d for b in BOUNDARIES if b is not None for d in (-2, -1, 0, 1, 2) if 1 <= b + d <= 120000})


@gpu
@settings(max_examples=150, deadline=None, derandomize=True)
@given(n=st.integers(1, 120000),
       bucket=st.one_of(st.sampled_from(_near_boundaries()), st.none(), st.integers(1, 1024), st.integers(1025, 60000)),
       mode=st.sampled_from(MODES), s=st.sampled_from([2, 3, 16, 255, 256]), seed=st.integers(0, 2 ** 20),
       offs=st.tuples(*[st.integers(0, 3)] * 4), alias_q=st.booleans(), alias_g=st.booleans())
def test_fused_random(N, n, bucket, mode, s, seed, offs, alias_q, alias_g):
    """qd_uniform_fwd_bwd at random sizes and buckets (near every boundary, or anywhere), modes, level counts, four
    independent offsets and both aliasing flags, against the C oracle."""
    lib, sp = N.lib(), N.stream_ptr()
    b = bucket_arg(bucket)
    x, g = make_inputs(n, seed)
    xd, gd = cuda(x), cuda(g)
    ws = N.workspace(n, b, xd.device)
    ox, og, oq, ogo = offs
    oq, ogo = (ox if alias_q else oq), (og if alias_g else ogo)
    V = Views(n)
    V.reset()
    xv, gv = V.view("x", ox), V.view("g", og)
    xv.copy_(xd)
    gv.copy_(gd)
    qv = xv if alias_q else V.view("q", oq)
    gov = gv if alias_g else V.view("go", ogo)
    m = {"ste": N.BWD_STE, "truncated": N.BWD_TRUNCATED, "minmax": N.BWD_MINMAX}[mode]
    what = f"n={n} bucket={bucket} {mode} s={s} offsets={offs} q is x={alias_q} gout is g={alias_g}"
    rc = lib.qd_uniform_fwd_bwd(N.ptr(xv), N.ptr(gv), N.ptr(qv), N.ptr(gov), n, b, s, m, N.ptr(ws), ws.numel(), sp)
    if mode == "minmax" and minmax_refused(N, n, b):
        assert rc == N.QD_ERR_UNSUPPORTED, (what, rc)
        torch.cuda.synchronize()
        if alias_q:
            same_bits(qv, xd, what + " q")
        else:
            assert bool((qv.view(torch.int32) == SENT).all()), what + ": q written"
        if alias_g:
            same_bits(gov, gd, what + " gout")
        else:
            assert bool((gov.view(torch.int32) == SENT).all()), what + ": gout written"
        V.check_guards(what)
        return
    N.check(rc)
    qc, _, _ = CO.uniform_fwd(x, s, bucket)
    same_bits(qv, cuda(qc), what + " q")
    if mode == "ste":
        same_bits(gov, gd, what + " gout")
    elif mode == "truncated":
        same_bits(gov, cuda(O.uniform_bwd_truncated(x, g)), what + " gout")
    else:
        ref, abs_sum, r = CO.uniform_bwd_minmax_ex(x, g, s, b)
        rows, row_len, padded = O.bucket_geometry(n, bucket)
        qp = np.concatenate([qc, np.full(padded - n, qc[-1], np.float32)]).reshape(rows, row_len)
        base = np.arange(rows, dtype=np.int64) * row_len
        check_minmax(gov, gd, cuda(ref), base + qp.argmax(1), base + qp.argmin(1), abs_sum, r, what + " gout")
    V.check_guards(what)
