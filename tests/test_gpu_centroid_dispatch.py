"""Every kernel the per-tensor centroid (non-uniform) ops can dispatch to, against the oracle and the reference.

qd_nonuniform_fwd picks a kernel from the row length L (warp path up to 1024 floats, staged ring up to
QD_MAX_STAGED_BUCKET, grid path above), the centroid-table class of K (warp path: 4 / 8 / 16 / 32 in the lanes, 64 and
256 in shared memory; staged ring: 4 / 8 / 16 / 32 / 256), the alignment of every pointer, the outputs asked for and
the pre-ops (device mean, max_element).  This file walks L through BOUNDARIES and K through K_BOUNDARIES, one value on
each side of every table class, and runs

  * qd_nonuniform_fwd with both rules, five output sets, four pre-op settings, views of x / q / idx_u8 at independent
    offsets and q aliasing x, bit for bit against oracle/quant_oracle.py (the C oracle above ORACLE_C_ABOVE elements);
  * rows that push x_hat's division onto its IEEE fallback, at every path and position;
  * rows holding NaN, +inf, -inf or an overflowing range, pinned on the reference's own outputs
    (tests/golden/reference_nonfinite.npz), and the 48 pre-op cases of reference_vectors_options.npz;
  * qd_nonuniform_bwd in each of its tile / row modes, sweep counts and past its grid cap, with exact-sum data bit for
    bit, and its workspace contract;
  * qd_centroid_index, qd_index_histogram and qd_nonuniform_fwd_packed at their alignment and length edges.

Every output starts out holding a NaN sentinel, and the guard elements around every view must still hold it afterwards.
test_k_boundaries_track_the_table_classes runs without a GPU and fails when a table class or a backward constant in
the sources moves without this file."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import c_oracle as CO
from oracle import quant_oracle as O
from test_gpu_parity import assert_same
from test_gpu_uniform_dispatch import (BOUNDARIES, MAX_FLOATS, ORACLE_C_ABOVE, SENT, SENT8, Views, bucket_arg, cuda, fresh,
                                       offset_sets, same_bits, shapes)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "quantized_distillation_b200", "csrc")
gpu = pytest.mark.gpu
F32 = np.float32

# Both sides of every centroid-table class bound (warp path, staged ring, qd_centroid_index), and the ends 1 and 256.
K_BOUNDARIES = [1, 2, 3, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 255, 256]
LANE_REPS, SMEM_REPS = (3, 8, 16, 32), (33, 64, 65, 256)
RULES = ("nearest", "midpoint")

# qd_nonuniform_bwd (csrc/qd_points_grad.cuh, csrc/qd_quant.cu): K is swept in groups of PG_SWEEP, a warp item is a
# tile of PG_TILE elements, the float32 columns are flushed every PG_FLUSH_EVERY tiles, the grid stops at PG_MAX_CTAS
# CTAs of PG_WARPS warps.  BWD_BIG_N is past the grid cap, so warps take several tiles; the in-loop flush would need
# PG_FLUSH_EVERY tiles per warp, PG_FLUSH_N elements, which is over the 64 MiB tensor limit (DESIGN.md section 4).
PG_SWEEP, PG_TILE, PG_FLUSH_EVERY, PG_WARPS, PG_MAX_CTAS = 32, 1024, 16, 8, 132 * 8
BWD_BIG_N = 9_000_017
PG_FLUSH_N = PG_MAX_CTAS * PG_WARPS * PG_TILE * PG_FLUSH_EVERY


# ----------------------------------------------------------------------------------------------- no GPU needed
def _constant(text, name):
    m = re.search(rf"constexpr\s+(?:size_t|int)\s+{name}\s*=\s*([\d\s*]+);", text)
    assert m, f"{name} not found"
    return int(eval(m.group(1)))  # noqa: S307 - a literal product such as 132 * 8


def _body(text, start):
    body = text[text.index(start):]
    return body[:body.index("\n}\n")]


def test_k_boundaries_track_the_table_classes():
    """Each centroid-table class bound of qd_nonuniform_fwd, the staged ring's sweep, the grid path's chunk fast path and
    centroid_index_kernel, and one past it, is in K_BOUNDARIES; and the backward's sizes are the ones this file computes its cases from."""
    read = lambda *p: open(os.path.join(*p)).read()  # noqa: E731
    quant, staged, pg = read(CSRC, "qd_quant.cu"), read(CSRC, "qd_staged_path.cuh"), read(CSRC, "qd_points_grad.cuh")
    classes = {}
    fwd = _body(quant, 'extern "C" int qd_nonuniform_fwd(')
    classes["qd_nonuniform_fwd"] = [int(v) for v in re.findall(r"num_points <= (\d+)\) return launch_warp", fwd)]
    sweep = staged[staged.index("const int K = P.num_points;"):]
    sweep = sweep[:sweep.index("\n        }\n")]
    classes["staged sweep"] = [int(v) for v in re.findall(r"K <= (\d+)\) sweep", sweep)]
    kern = _body(quant, "centroid_index_kernel(")
    classes["centroid_index_kernel"] = [int(v) for v in re.findall(r"K <= (\d+)\) centroid_index_body", kern)]
    grid = read(CSRC, "qd_grid_path.cuh")
    classes["grid chunk fast path"] = [int(v) for v in re.findall(r"K <= (\d+)\) nonuniform_chunk<", grid)]
    for what, bounds in classes.items():
        assert len(bounds) >= 4, (what, bounds)
        for v in bounds + [256]:
            assert v in K_BOUNDARIES and (v == 256 or v + 1 in K_BOUNDARIES), f"{what}: class bound {v}: add {v} and {v + 1}"
    assert 1 in K_BOUNDARIES
    assert _constant(pg, "kPgSweep") == PG_SWEEP and _constant(pg, "kPgTile") == PG_TILE
    assert _constant(pg, "kPgFlushEvery") == PG_FLUSH_EVERY and _constant(pg, "kPgThreads") == 32 * PG_WARPS
    assert _constant(quant, "kPointsGradMaxCtas") == PG_MAX_CTAS
    # the backward cases below: one, two and eight sweeps, past the grid cap, inside the tensor limit
    assert 1 <= PG_SWEEP < 33 and 64 <= 2 * PG_SWEEP < 65 and -(-256 // PG_SWEEP) == 8
    assert PG_MAX_CTAS * PG_WARPS * PG_TILE < BWD_BIG_N <= MAX_FLOATS
    assert PG_FLUSH_N > MAX_FLOATS, "the in-loop flush is now reachable: add a case for it"


def pinned_points(K, seed):
    """Sorted points with duplicates and values below 0 and above 1, so some thresholds fall outside x_hat's range."""
    rng = np.random.default_rng(seed)
    p = np.sort(rng.random(K) * 1.4 - 0.2).astype(F32)
    if K >= 3:
        p[K // 2] = p[K // 2 - 1]
    if K >= 5:
        p[1] = p[0]
    return np.sort(p)


def test_nonfinite_fixture_pins_the_oracles():
    """The NumPy and C oracles give the reference's idx and q on rows holding NaN, +inf, -inf or an overflowing range
    (NaN x_hat -> K-1 under both rules); any two NaNs count as equal."""
    data = np.load(os.path.join(HERE, "golden", "reference_nonfinite.npz"))
    cases = [str(m).split("|") for m in data["meta"]]
    assert len(cases) == 20
    kinds = set()
    for _, key, kind, n, b, K in cases:
        kinds.update(kind.split("+"))
        b = None if int(b) < 0 else int(b)
        x, pts = data[key + "_x"], data[key + "_points"]
        for rule in RULES:
            want_i, want_q = data[f"{key}_idx_{rule}"].astype(np.int64), data[f"{key}_q_{rule}"]
            with np.errstate(all="ignore"):
                q, idx, _ = O.nonuniform_fwd(x, pts, b, rule=rule)
                qc, ic, _ = CO.nonuniform_fwd(x, pts, b, rule=rule)
            assert_same(idx.reshape(-1), want_i, f"{key} {kind} {rule} oracle idx")
            assert_same(q.reshape(-1), want_q, f"{key} {kind} {rule} oracle q")
            assert_same(ic, want_i, f"{key} {kind} {rule} C oracle idx")
            assert_same(qc, want_q, f"{key} {kind} {rule} C oracle q")
        if kind != "finite":                    # not vacuous: the reference sends NaN x_hat to K-1
            assert (data[key + "_idx_nearest"] == int(K) - 1).any() and (data[key + "_idx_midpoint"] == int(K) - 1).any(), key
    assert kinds == {"finite", "nan", "posinf", "neginf", "overflow"}


# ----------------------------------------------------------------------------------------------- helpers
@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native as N
    return N


def rule_of(N, rule):
    return N.RULE_NEAREST if rule == "nearest" else N.RULE_MIDPOINT


def centroid_inputs(n, seed):
    """x standard normal, half of it on a 1/256 grid (ties with the points and the thresholds); no -0.0."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n) * 0.6
    return (np.where(rng.random(n) < 0.5, np.round(x * 256) / 256, x) + 0.0).astype(F32)


def oracle_nu(x, pts, L, rule, mean=None, max_element=False):
    """(q, idx int64, alpha, beta) of O.nonuniform_fwd on O.pre_ops(x, mean, max_element); the C restatement above
    ORACLE_C_ABOVE elements (it takes pre-processed input; the mean is added back in float32 as O does)."""
    pre = mean is not None or max_element is not False
    if x.size <= ORACLE_C_ABOVE:
        with np.errstate(all="ignore"):
            q, idx, st = O.nonuniform_fwd(x, pts, L, rule=rule, subtract_mean=mean is not None, max_element=max_element, mean=mean)
        return q.reshape(-1), idx.reshape(-1), st["alpha"], st["beta"]
    flat, m = O.pre_ops(x, mean is not None, max_element, mean)
    q, idx, st = CO.nonuniform_fwd(flat, pts, L, rule=rule)
    if pre:
        q = (q + m).astype(F32)
    rows, row_len, _ = O.bucket_geometry(flat.size, L)
    beta = np.concatenate([flat, np.full(rows * row_len - flat.size, flat[-1], F32)]).reshape(rows, row_len).min(axis=1)
    return q, idx, st["alpha"], beta


# output sets of qd_nonuniform_fwd: (q, idx_u8, idx_i64, alpha/beta)
# (q, idx_u8, idx_i64, alpha/beta).  Without idx_i64 and without a pre-op, full aligned 16384-float chunks of a grid row
# take the chunk fast path (nonuniform_chunk); with idx_i64 they take the generic loop.
OUTSETS = {"q": (1, 0, 0, 0), "idx_u8": (0, 1, 0, 0), "idx_i64": (0, 0, 1, 0), "all": (1, 1, 1, 1), "all but alpha/beta": (1, 1, 1, 0),
           "q and idx_u8": (1, 1, 0, 1)}
FAST_OUTSETS = ("q and idx_u8", "q", "idx_u8")


class Fwd:
    """One qd_nonuniform_fwd call on sentinel-filled views, checked against the oracle's arrays."""

    def __init__(self, N, n, L):
        self.N, self.n, self.b = N, n, bucket_arg(L)
        self.rows = N.geometry(n, self.b)[0]
        self.V = Views(n)
        # int64 indices only where they fit the 64 MiB tensor limit; above it the idx_i64 sets write idx_u8 instead
        self.i64 = torch.empty(n, dtype=torch.int64, device="cuda") if n <= MAX_FLOATS // 2 else None
        self.ws = N.workspace(n, self.b, torch.device("cuda"))

    def run(self, xd, ptsd, K, rule, ref, offs, outset="all", alias=False, mean_d=None, me=0.0, what=""):
        N, V = self.N, self.V
        ox, oq, oi = offs
        wq, w8, w64, wab = OUTSETS[outset]
        if alias:
            wq = 1
        if w64 and self.i64 is None:
            w64, w8 = 0, 1
        V.reset()
        if self.i64 is not None:
            self.i64.fill_(-7)
        xv = V.view("x", ox)
        xv.copy_(xd)
        qv = xv if alias else (V.view("q", oq) if wq else None)
        iv = V.view("i8", oi) if w8 else None
        i64 = self.i64 if w64 else None
        alpha, beta = (fresh(self.rows, torch.float32), fresh(self.rows, torch.float32)) if wab else (None, None)
        what = f"{what} K={K} {rule} out={outset} offsets x={ox} q={oq} idx={oi} q is x={alias}"
        N.check(N.lib().qd_nonuniform_fwd(N.ptr(xv), N.ptr(ptsd), K, rule_of(N, rule), N.ptr(qv), N.ptr(iv), N.ptr(i64),
                                          N.ptr(alpha), N.ptr(beta), self.n, self.b, N.ptr(mean_d), me, N.ptr(self.ws),
                                          self.ws.numel(), N.stream_ptr()))
        qr, ir8, ir64, ar, br = ref
        if wq:
            same_bits(qv, qr, what + " q")
        if w8:
            same_bits(iv, ir8, what + " idx_u8")
        if w64:
            same_bits(self.i64, ir64, what + " idx_i64")
        elif self.i64 is not None:
            assert bool((self.i64 == -7).all()), what + ": idx_i64 written though not asked for"
        if wab:
            same_bits(alpha, ar, what + " alpha")
            same_bits(beta, br, what + " beta")
        V.check_guards(what)


def dev_ref(q, idx, alpha, beta, K):
    i64 = cuda(idx.astype(np.int64)) if idx.size <= MAX_FLOATS // 2 else None
    return cuda(q), cuda(idx.astype(np.uint8)), i64, cuda(alpha), cuda(beta)


def sweep_shapes(N, L):
    """Sizes of the K sweep: a few rows and a ragged tail; for bucket None one size per path (warp, staged, grid)."""
    if L is None:
        return [7, 1000, 3 * 16384 + 77]
    s = shapes(N, L)
    return [s[1] if len(s) > 1 else s[0]]


# ----------------------------------------------------------------------------------------------- forward, every L
@gpu
@pytest.mark.parametrize("L", BOUNDARIES, ids=str)
def test_forward_every_k_class(N, L):
    """Both rules at every K of K_BOUNDARIES, all outputs, aligned and at one unaligned offset set, and once with q
    aliasing x; aligned without idx_i64 too (the grid path's chunk fast path)."""
    for si, n in enumerate(sweep_shapes(N, L)):
        x = centroid_inputs(n, 100 + si)
        xd = cuda(x)
        F = Fwd(N, n, L)
        for ki, K in enumerate(K_BOUNDARIES):
            pts = pinned_points(K, 10 * K + si)
            ptsd = cuda(pts)
            for rule in RULES:
                ref = dev_ref(*oracle_nu(x, pts, L, rule), K)
                what = f"sweep n={n} L={L}"
                F.run(xd, ptsd, K, rule, ref, (0, 0, 0), what=what)
                F.run(xd, ptsd, K, rule, ref, (0, 0, 0), "q and idx_u8", what=what)
                F.run(xd, ptsd, K, rule, ref, (1, 3, 1), what=what)
                if (ki + (rule == "midpoint")) % 3 == 0:
                    F.run(xd, ptsd, K, rule, ref, (1, 0, 2), alias=True, what=what)


@gpu
@pytest.mark.parametrize("L", BOUNDARIES, ids=str)
def test_forward_offsets_outputs_and_pre_ops(N, L):
    """At every size of the uniform suite's shapes: one K in the lanes and one in shared memory, both rules, no pre-op,
    max_element, a device mean and both; every offset set with the output sets in turn, every output set aligned and
    unaligned, and q aliasing x at aligned and unaligned x."""
    mean_val = F32(0.1875)
    mean_d = cuda(np.array([mean_val], F32))
    for si, n in enumerate(shapes(N, L)):
        x = centroid_inputs(n, 200 + si)
        xd = cuda(x)
        F = Fwd(N, n, L)
        for K, rule in ((LANE_REPS[si % 4], RULES[si % 2]), (SMEM_REPS[si % 4], RULES[(si + 1) % 2])):
            pts = pinned_points(K, 300 + K)
            ptsd = cuda(pts)
            for pi, (mean, me) in enumerate(((None, False), (None, 0.75), (mean_val, False), (mean_val, 0.5))):
                ref = dev_ref(*oracle_nu(x, pts, L, rule, mean, me), K)
                what = f"n={n} L={L} mean={mean} max_element={me}"
                md, mev = (None if mean is None else mean_d), (0.0 if me is False else me)
                names = list(OUTSETS)
                cases = [(o, names[(i + pi) % len(names)], False) for i, (o) in enumerate(offset_sets(si))]
                cases += [(o, name, False) for name in names for o in ((0, 0, 0, 0, 0), (1, 1, 1, 1, 1), (0, 1, 1, 1, 3))]
                cases += [((0,) * 5, "all", True), ((1, 0, 1, 0, 1), "idx_u8", True), ((3, 0, 3, 0, 2), "all", True)]
                for (ox, _, oq, _, oi), outset, alias in cases:
                    F.run(xd, ptsd, K, rule, ref, (ox, oq, oi), outset, alias, md, mev, what)


# ----------------------------------------------------------------------------------------------- degenerate rows
DEGENERATE_PTS = [np.array([0.0, 1e-30, 0.5, 1.0], F32),
                  np.sort(np.concatenate([[0.0, 1e-30, 1e-12], np.linspace(0.01, 1.0, 62)]).astype(F32))]


def degenerate_patterns():
    """The rows of test_gpu_parity.test_nonuniform_tiny_and_degenerate_rows, and a constant row."""
    return [np.array([0.0, 1e-38, 1e-30, 1e-12, 0.5, 1.0, 3e-39, 1e-20], F32),
            np.array([0.0, 3e38, 1e10, 1.0], F32),
            np.array([1.0, 1.0 + 1e-7], F32),
            np.array([-2.5], F32),
            (np.arange(256) * 1e-42).astype(F32),
            np.array([0.125], F32)]


def degenerate_tensor(L, seed):
    """Rows of length L (bucket None: 3 * 16384 + 77 floats, one row of four grid chunks); row r is either a
    degenerate pattern tiled, or a [0, 1] row holding one element at a tiny distance above its minimum 0 -- at a
    position that moves between a vector group (5), the middle, the last ring chunk (L - 6) and the scalar tail
    (L - 1); for bucket None also in a later 16384-float chunk."""
    rng = np.random.default_rng(seed)
    rl = 3 * 16384 + 77 if L is None else L
    rows = []
    pats = degenerate_patterns()
    for r in range(2 * len(pats) if L is not None else 1):
        if r % 2 == 0 and L is not None:
            p = pats[(r // 2) % len(pats)]
            rows.append(np.tile(p, -(-rl // p.size))[:rl])
            continue
        row = rng.random(rl).astype(F32)
        row[rng.integers(0, rl)] = 0.0
        tiny = (1e-38, 3e-39, 1e-42)[r % 3]
        for pos in ({5, rl // 2, max(rl - 6, 0), rl - 1} | ({2 * 16384 + 5} if L is None else set())):
            row[pos] = tiny
        rows.append(row)
    return np.concatenate(rows)[: (len(rows) * rl - (3 if L is not None and L % 4 else 0))]


@gpu
@pytest.mark.parametrize("L", [256, 1000, 1025, 3002, 12289, 49152, None], ids=str)
def test_degenerate_rows_every_path(N, L):
    """x_hat's division leaves the hoisted-reciprocal domain (tiny distances, huge / tiny alpha, constant rows,
    denormals): the warp path's row vote, the staged ring's per-group decision, the grid path's chunk fast path (aligned,
    no idx_i64) and generic loop, and the scalar tails all fall back to the IEEE division; bit for bit with both rules,
    aligned and at x offset 1 (unaligned staged rows)."""
    tensors = [degenerate_tensor(L, 400)] if L is not None else [degenerate_tensor(L, 400 + i) for i in range(3)]
    if L is None:                                                   # every degenerate pattern as the one grid row
        rl = 3 * 16384 + 77
        tensors += [np.tile(p, -(-rl // p.size))[:rl] for p in degenerate_patterns()]
    for ti, x in enumerate(tensors):
        xd = cuda(x)
        F = Fwd(N, x.size, L)
        for pts in DEGENERATE_PTS:
            ptsd = cuda(pts)
            for rule in RULES:
                ref = dev_ref(*oracle_nu(x, pts, L, rule), pts.size)
                what = f"degenerate tensor {ti} n={x.size} L={L}"
                for offs in ((0, 0, 0), (1, 1, 1), (2, 0, 3)):
                    F.run(xd, ptsd, pts.size, rule, ref, offs, what=what)
                for outset in FAST_OUTSETS:
                    F.run(xd, ptsd, pts.size, rule, ref, (0, 0, 0), outset, what=what)


# ----------------------------------------------------------------------------------------------- non-finite rows
@pytest.fixture(scope="module")
def nonfinite():
    data = np.load(os.path.join(HERE, "golden", "reference_nonfinite.npz"))
    cases = []
    for m in data["meta"]:
        _, key, kind, n, b, K = str(m).split("|")
        cases.append(dict(key=key, kind=kind, n=int(n), bucket=None if int(b) < 0 else int(b), K=int(K)))
    return data, cases


def same_nan(got, want, what):
    """Bit equality with any two NaNs equal (assert_same's rule), on host copies."""
    assert_same(got.cpu().numpy(), np.asarray(want), what)


@gpu
def test_nonfinite_rows_match_the_reference(N, nonfinite):
    """Rows with NaN, +inf, -inf and an overflowing range on all three paths (bucket 256: warp; 3002: staged ring; None
    at 50,000 floats: grid, chunk fast path and generic loop; None at 700: warp), with both rules, aligned and
    unaligned: idx and q are the reference's,
    NaN x_hat getting K-1.  Then qd_centroid_index on the oracle's x_hat (itself pinned on the reference): the same
    indices, unit_out = points[idx]."""
    data, cases = nonfinite
    lib, sp = N.lib(), N.stream_ptr()
    for c in cases:
        k, K, b, n = c["key"], c["K"], bucket_arg(c["bucket"]), c["n"]
        x, pts = data[k + "_x"], data[k + "_points"]
        xd, ptsd = cuda(x), cuda(pts)
        rows = N.geometry(n, b)[0]
        ws = N.workspace(n, b, xd.device)
        buf = torch.empty(n + 4, device="cuda")
        with np.errstate(all="ignore"):
            xh, _ = O.scale_down(x, c["bucket"])
        xhd = cuda(xh.reshape(-1)[:n])
        for rule in RULES:
            want_i, want_q = data[f"{k}_idx_{rule}"].astype(np.int64), data[f"{k}_q_{rule}"]
            # with idx_i64: the grid path's generic loop; without it (and aligned): its chunk fast path
            for off, with_i64 in ((0, True), (1, True), (0, False), (1, False)):
                what = f"{k} {c['kind']} n={n} bucket={c['bucket']} K={K} {rule} offset {off} idx_i64={with_i64}"
                xv = buf[off:off + n]
                xv.copy_(xd)
                q, i8, i64 = fresh(n, torch.float32), fresh(n, torch.uint8), fresh(n, torch.int64)
                alpha, beta = fresh(rows, torch.float32), fresh(rows, torch.float32)
                N.check(lib.qd_nonuniform_fwd(N.ptr(xv), N.ptr(ptsd), K, rule_of(N, rule), N.ptr(q), N.ptr(i8),
                                              N.ptr(i64) if with_i64 else None, N.ptr(alpha), N.ptr(beta), n, b, None, 0.0,
                                              N.ptr(ws), ws.numel(), sp))
                if with_i64:
                    same_nan(i64, want_i, what + " idx_i64")
                same_nan(i8, want_i.astype(np.uint8), what + " idx_u8")
                same_nan(q, want_q, what + " q")
                if off == 0:
                    ci8, ci64, unit = fresh(n, torch.uint8), fresh(n, torch.int64), fresh(n, torch.float32)
                    N.check(lib.qd_centroid_index(N.ptr(xhd), N.ptr(ptsd), K, rule_of(N, rule), N.ptr(ci8), N.ptr(ci64),
                                                  N.ptr(unit), n, sp))
                    same_nan(ci64, want_i, what + " qd_centroid_index idx_i64")
                    same_nan(ci8, want_i.astype(np.uint8), what + " qd_centroid_index idx_u8")
                    same_nan(unit, pts[want_i], what + " qd_centroid_index unit_out")


@gpu
def test_nonfinite_rows_in_centroid_plans(N, nonfinite):
    """The centroid plans share the lane search: the fixture's tensors that fit a plan (K <= 32, rows of at most 1024
    floats) in one plan per bucket, each at its own float offset, give the reference's midpoint-rule idx and q."""
    from quantized_distillation_b200.plan import CentroidPlan
    data, cases = nonfinite
    for bucket in (256, None):
        sel = [c for c in cases if c["bucket"] == bucket and c["K"] <= 32 and (bucket is not None or c["n"] <= 1024)]
        assert len(sel) >= 3, bucket
        bufs = [torch.empty(c["n"] + 3, device="cuda") for c in sel]
        src = [b_[i % 4:i % 4 + c["n"]] for i, (b_, c) in enumerate(zip(bufs, sel))]
        for t, c in zip(src, sel):
            t.copy_(cuda(data[c["key"] + "_x"]))
        dst = [fresh(c["n"], torch.float32) for c in sel]
        plan = CentroidPlan(src, dst, [cuda(data[c["key"] + "_points"]) for c in sel], bucket)
        plan.forward_()
        for i, c in enumerate(sel):
            what = f"plan bucket={bucket} {c['key']} {c['kind']} K={c['K']}"
            same_nan(plan.indices[i].reshape(-1).long(), data[c["key"] + "_idx_midpoint"].astype(np.int64), what + " idx")
            same_nan(dst[i], data[c["key"] + "_q_midpoint"], what + " q")
        plan.close()


# ----------------------------------------------------------------------------------------------- pre-op reference cases
@gpu
def test_pre_ops_reference_cases(N, golden_options):
    """The reference's nonUniformQuantization with subtract_mean / max_element (48 cases): through the C ABI with the
    reference's own mean as the device mean, idx and q bit for bit; through nonUniformQuantization(subtract_mean=...,
    max_element=...), the mean within the summation-order tolerance and q / idx bit for bit against the oracle given
    the mean the op used."""
    import quantized_distillation_b200.quantization as Q
    data, cases = golden_options
    cases = cases["pre_nonuniform"]
    assert len(cases) == 48
    lib, sp = N.lib(), N.stream_ptr()
    for c in cases:
        k, b = c["key"], c["bucket"]
        x, pts = data[k + "_x"], data[k + "_points"]
        ref_mean = data[k + "_mean"][0]
        n, K = x.size, pts.size
        what = f"{k} n={n} bucket={b} K={K} subtract_mean={c['subtract_mean']} max_element={c['max_element']}"
        xd, ptsd = cuda(x), cuda(pts)
        q, i64 = fresh(n, torch.float32), fresh(n, torch.int64)
        ws = N.workspace(n, bucket_arg(b), xd.device)
        mean_d = cuda(np.array([ref_mean], F32)) if c["subtract_mean"] else None
        me = 0.0 if c["max_element"] is False else c["max_element"]
        N.check(lib.qd_nonuniform_fwd(N.ptr(xd), N.ptr(ptsd), K, N.RULE_NEAREST, N.ptr(q), None, N.ptr(i64), None, None, n,
                                      bucket_arg(b), N.ptr(mean_d), me, N.ptr(ws), ws.numel(), sp))
        same_bits(i64, cuda(data[k + "_idx"].reshape(-1).astype(np.int64)), what + " C ABI idx")
        same_bits(q, cuda(data[k + "_q"].reshape(-1)), what + " C ABI q")
        qp, ip, sf = Q.nonUniformQuantization(cuda(x), ptsd, bucket_size=b, subtract_mean=c["subtract_mean"],
                                              max_element=c["max_element"])
        used = F32(float(sf.mean_tensor)) if c["subtract_mean"] else None
        if c["subtract_mean"]:
            x64 = x.astype(np.float64)
            assert abs(float(used) - float(ref_mean)) <= 1e-6 * np.abs(x64).mean() + 1e-30, (what, float(used), float(ref_mean))
        with np.errstate(all="ignore"):
            qo, io, _ = O.nonuniform_fwd(x, pts, b, rule="nearest", subtract_mean=c["subtract_mean"], max_element=c["max_element"],
                                         mean=used)
        same_bits(qp.reshape(-1), cuda(qo.reshape(-1)), what + " nonUniformQuantization q")
        same_bits(ip.reshape(-1), cuda(io.reshape(-1)), what + " nonUniformQuantization idx")


# ----------------------------------------------------------------------------------------------- backward
def bwd_call(N, g, i8, i64, alpha, K, out, n, b, ws, wsb):
    return N.lib().qd_nonuniform_bwd(N.ptr(g), N.ptr(i8), N.ptr(i64), N.ptr(alpha), K, N.ptr(out), n, b, N.ptr(ws) if ws is not None else None,
                                     wsb, N.stream_ptr())


BWD_CASES = [
    # (n, L, K, idx dtype, g offset, idx offset): the branch it reaches
    (40 * 1024, 256, 32, "u8", 0, 0),            # vectorized tile mode: full tiles, rows change inside a tile
    (40 * 1024 + 700, 256, 33, "u8", 0, 0),      # ... and a last partial tile (scalar), two sweeps
    (40 * 1024, 1024, 65, "u8", 0, 0),           # vectorized, one row per tile, three sweeps
    (40 * 1024 + 3, 128, 256, "u8", 1, 0),       # scalar tile mode: g off 16 bytes; eight sweeps
    (40 * 1024, 256, 64, "u8", 0, 1),            # scalar tile mode: idx off 4 bytes
    (40 * 1024, 256, 17, "i64", 0, 0),           # scalar tile mode: int64 idx
    (30_001, 100, 1, "u8", 0, 0),                # row mode (L % 128 != 0), one point
    (30_001, 257, 33, "i64", 1, 1),              # row mode, int64, unaligned
    (30_001, 1000, 64, "u8", 3, 2),
    (30_001, 3002, 256, "u8", 0, 0),             # row mode, rows of several tiles
    (100_003, None, 65, "u8", 0, 0),             # bucket None: one row, tile mode
    (100_003, None, 256, "i64", 2, 0),
    (BWD_BIG_N, 256, 65, "u8", 0, 0),            # past the grid cap: warps take several tiles
    (BWD_BIG_N, None, 256, "u8", 0, 0),
    (BWD_BIG_N, 1000, 32, "u8", 1, 1),           # row mode past the cap
]


def bwd_data(rng, n, L, K, exact):
    rows = O.bucket_geometry(n, L)[0]
    if exact:
        alpha = np.ldexp(F32(1), -(np.arange(rows) % 4)).astype(F32)
        g = rng.integers(-4, 5, n, dtype=np.int8).astype(F32)
    else:
        alpha = (rng.random(rows) * 3 + 0.01).astype(F32)
        g = rng.standard_normal(n).astype(F32)
    idx = rng.integers(0, K, n, dtype=np.int64)
    return g, idx, alpha


@gpu
@pytest.mark.parametrize("n, L, K, kind, og, oi", BWD_CASES, ids=lambda v: str(v))
def test_backward_every_branch(N, n, L, K, kind, og, oi):
    """Exact-sum data (alpha = 2^-e, integer g) bit for bit against the C oracle and run to run; random data inside the
    per-column bound of test_gpu_plans.py (each float32 column adds at most 512 products before its float64 flush).
    Where the tensor fits, u8 and int64 indices give the same bits on the exact-sum data (random sums may differ in the
    last bit: the two tile modes add a lane's column in another order); indices >= K add nothing."""
    b = bucket_arg(L)
    ws = torch.empty(int(N.lib().qd_workspace_bytes(n, b)), dtype=torch.uint8, device="cuda")
    for exact in (True, False):
        rng = np.random.default_rng(n % 1000 + K + (7 if exact else 0))
        g, idx, alpha = bwd_data(rng, n, L, K, exact)
        gb = torch.empty(n + 4, device="cuda")
        gv = gb[og:og + n]
        gv.copy_(cuda(g))
        ad = cuda(alpha)
        # ~2% of the indices out of range: K .. 255 in u8; in int64 a third each of those values, 2^32 + k (which a
        # 32-bit compare would take for the valid index k) and negative values.  They must add nothing.
        extra = (rng.random(n) < 0.02) if K < 256 else np.zeros(n, bool)
        idx_run = np.where(extra, rng.integers(K, 256, n), idx) if K < 256 else idx
        third = rng.integers(0, 3, n)
        idx_run64 = np.where(extra & (third == 1), (1 << 32) + idx, np.where(extra & (third == 2), -1 - idx, idx_run))
        g_in = np.where(extra, F32(0), g).astype(F32)
        idx = np.where(extra, 0, idx)
        ref = CO.nonuniform_bwd_points(g_in, idx, alpha, K, L)
        what = f"bwd n={n} L={L} K={K} {kind} g+{og} idx+{oi} {'exact' if exact else 'random'}"
        outs = []
        kinds = [kind] + (["i64" if kind == "u8" else "u8"] if n * 8 <= MAX_FLOATS * 4 and K <= 256 else [])
        for kk in kinds:
            if kk == "u8":
                ib = torch.empty(n + 8, dtype=torch.uint8, device="cuda")
                iv = ib[oi:oi + n]
                iv.copy_(cuda(idx_run.astype(np.uint8)))
                args = (iv, None)
            else:
                ib = torch.empty(n + 2, dtype=torch.int64, device="cuda")
                iv = ib[oi:oi + n] if oi else ib[:n]
                iv.copy_(cuda(idx_run64.astype(np.int64)))
                args = (None, iv)
            for rep in range(2):
                out = fresh(K, torch.float32)
                N.check(bwd_call(N, gv, *args, ad, K, out, n, b, ws, ws.numel()))
                outs.append(out)
            same_bits(outs[-1], outs[-2], f"{what} idx {kk}: run to run")
        if exact:   # random sums: the vector and scalar tile modes add a lane's column in another order
            for o in outs[1:]:
                same_bits(o, outs[0], what + ": u8 and int64 indices")
        got = outs[0].cpu().numpy().astype(np.float64)
        if exact:
            assert_same(outs[0].cpu().numpy(), ref.astype(F32), what)
        else:
            a = np.repeat(alpha, O.bucket_geometry(n, L)[1])[:n]
            mag = np.bincount(idx, weights=np.abs((g_in * a).astype(F32)).astype(np.float64), minlength=K)[:K]
            tol = 512 * 2.0 ** -24 * mag + 2.0 ** -24 * np.abs(ref)
            assert np.all(np.abs(got - ref) <= tol), (what, got, ref)


@gpu
@pytest.mark.parametrize("n, bucket", [(1000, 256), (40 * 1024 + 3, 100), (3_000_017, 0), (40 * 65536 + 3, 65536)])
def test_backward_workspace_contract(N, n, bucket):
    """Exactly qd_workspace_bytes(n, bucket) works; one byte less, or NULL, returns QD_ERR_WORKSPACE and leaves
    grad_points as it was."""
    L = None if bucket == 0 else bucket
    rng = np.random.default_rng(n % 991)
    K = 33
    g, idx, alpha = bwd_data(rng, n, L, K, True)
    gd, i8, ad = cuda(g), cuda(idx.astype(np.uint8)), cuda(alpha)
    need = int(N.lib().qd_workspace_bytes(n, bucket))
    assert need > 0
    buf = torch.empty(need, dtype=torch.uint8, device="cuda")
    for size, label in ((need, "exact"), (need - 1, "one byte short"), (None, "NULL")):
        out = fresh(K, torch.float32)
        rc = bwd_call(N, gd, i8, None, ad, K, out, n, bucket, None if size is None else buf, 0 if size is None else size)
        what = f"bwd n={n} bucket={bucket} workspace {label}"
        if size == need:
            N.check(rc)
            assert_same(out.cpu().numpy(), CO.nonuniform_bwd_points(g, idx, alpha, K, L).astype(F32), what)
        else:
            assert rc == N.QD_ERR_WORKSPACE, (what, rc)
            torch.cuda.synchronize()
            assert bool((out.view(torch.int32) == SENT).all()), what + ": grad_points written"


# ----------------------------------------------------------------------------------------------- qd_centroid_index
def special_xhat(n, pts, seed):
    """x_hat with NaN, +-inf, -0.0, values outside [0, 1], the points and their midpoints themselves."""
    rng = np.random.default_rng(seed)
    v = (rng.random(n) * 1.6 - 0.3).astype(F32)
    specials = np.concatenate([[np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0, -1e-30, 2.0], pts, O.midpoints(pts)]).astype(F32)
    pick = rng.random(n) < 0.3
    v[pick] = specials[rng.integers(0, specials.size, int(pick.sum()))]
    return v


@gpu
@pytest.mark.parametrize("K", K_BOUNDARIES)
def test_centroid_index_every_branch(N, K):
    """qd_centroid_index at both rules: n = 1..7, n % 4 tails and n above one grid-stride pass; xhat, unit_out and
    idx_u8 each offset alone; each output alone and all three; x_hat holding NaN, +-inf, -0.0 and values outside
    [0, 1]; against O.nonuniform_index_* and points[idx]."""
    lib, sp = N.lib(), N.stream_ptr()
    pts = pinned_points(K, 500 + K)
    ptsd = cuda(pts)
    sizes = [1, 2, 3, 4, 5, 6, 7, 1000, 1001, 1002, 1003] + ([2_000_003] if K in (1, 5, 32, 33, 256) else [])
    for n in sizes:
        xh = special_xhat(n, pts, n + K)
        xhd = cuda(xh)
        xb = torch.empty(n + 8, device="cuda")
        ub = torch.empty(n + 8, device="cuda")
        ib = torch.empty(n + 8, dtype=torch.uint8, device="cuda")
        for rule in RULES:
            fn = O.nonuniform_index_nearest if rule == "nearest" else O.nonuniform_index_midpoint
            want = fn(xh, pts).reshape(-1)
            assert want.max() < K
            w64, w8, wu = cuda(want), cuda(want.astype(np.uint8)), cuda(pts[want])
            for (ox, ou, oi) in ((0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 3), (3, 2, 1)):
                for outs in ("all", "idx_u8", "idx_i64", "unit_out"):
                    if (ox, ou, oi) != (0, 0, 0) and outs != "all" and n > 1003:
                        continue
                    what = f"centroid_index K={K} {rule} n={n} offsets xhat={ox} unit={ou} idx={oi} out={outs}"
                    xb.view(torch.int32).fill_(SENT)
                    ub.view(torch.int32).fill_(SENT)
                    ib.fill_(SENT8)
                    xv = xb[ox:ox + n]
                    xv.copy_(xhd)
                    uv, iv = ub[ou:ou + n], ib[oi:oi + n]
                    i64 = fresh(n, torch.int64)
                    a8 = iv if outs in ("all", "idx_u8") else None
                    a64 = i64 if outs in ("all", "idx_i64") else None
                    au = uv if outs in ("all", "unit_out") else None
                    N.check(lib.qd_centroid_index(N.ptr(xv), N.ptr(ptsd), K, rule_of(N, rule), N.ptr(a8), N.ptr(a64), N.ptr(au), n, sp))
                    if a8 is not None:
                        same_bits(iv, w8, what + " idx_u8")
                    if a64 is not None:
                        same_bits(i64, w64, what + " idx_i64")
                    else:
                        assert bool((i64 == -7).all()), what + ": idx_i64 written"
                    if au is not None:
                        same_bits(uv, wu, what + " unit_out")
                    for buf, off, s in ((ub, ou if au is not None else 0, SENT), (ib, oi if a8 is not None else 0, SENT8)):
                        raw = buf.view(torch.int32) if buf.dtype == torch.float32 else buf
                        used = n if (buf is ub and au is not None) or (buf is ib and a8 is not None) else 0
                        keep = torch.cat([raw[:off], raw[off + used:]])
                        assert bool((keep == s).all()), what + ": written outside its view"


# ----------------------------------------------------------------------------------------------- qd_index_histogram
@gpu
@pytest.mark.parametrize("num_bins", [1, 2, 255, 256])
def test_index_histogram_every_branch(N, num_bins):
    """Counts exact against np.bincount at byte offsets 0..15, n < 16, n % 16 tails and sizes past one grid pass;
    values >= num_bins are present and dropped; counts accumulate onto nonzero starting values."""
    lib, sp = N.lib(), N.stream_ptr()
    rng = np.random.default_rng(num_bins)
    for n in (1, 2, 3, 7, 15, 16, 17, 31, 1000, 1024 + 9, 4_000_037):
        vals = rng.integers(0, 256, n).astype(np.uint8)
        if num_bins < 256:                              # mostly in range, a few at and above num_bins
            vals = np.where(rng.random(n) < 0.9, vals % num_bins, vals).astype(np.uint8)
        want_add = np.bincount(vals[vals < num_bins], minlength=num_bins)[:num_bins].astype(np.int64)
        vd = cuda(vals)
        buf = torch.empty(n + 32, dtype=torch.uint8, device="cuda")
        for off in (range(16) if n < 5000 else (0, 1, 4, 15)):
            buf.fill_(SENT8)
            v = buf[off:off + n]
            v.copy_(vd)
            start = rng.integers(0, 1000, num_bins).astype(np.int64)
            counts = cuda(start)
            N.check(lib.qd_index_histogram(N.ptr(v), n, num_bins, N.ptr(counts), sp))
            same_bits(counts, cuda(start + want_add), f"histogram n={n} bins={num_bins} offset {off}")


# ----------------------------------------------------------------------------------------------- packed forward
PACK_L = [L for L in BOUNDARIES if L is not None and L <= 1024] + [1025, None]


def bits_for(K):
    return 1 if K <= 2 else 2 if K <= 4 else 4 if K <= 16 else 8


@gpu
@pytest.mark.parametrize("L", PACK_L, ids=str)
def test_nonuniform_fwd_packed_every_branch(N, L):
    """qd_nonuniform_fwd_packed at every K class boundary and every allowed width, x at offsets 0..3 and the packed
    stream at byte offsets 0..3 (in-register path and fallback): the bytes are qd_nonuniform_fwd(idx_u8) followed by
    qd_pack_indices, alpha / beta its alpha / beta; every narrower width is refused with nothing written."""
    lib, sp, b = N.lib(), N.stream_ptr(), bucket_arg(L)
    n = 3 * 1000 + 5 if L is None else 3 * L + (3 if L > 3 else 0)
    rows = N.geometry(n, b)[0]
    x = centroid_inputs(n, 600 + n)
    xd = cuda(x)
    xb = torch.empty(n + 4, device="cuda")
    pw = torch.empty(int(lib.qd_packed_workspace_bytes(n, b)), dtype=torch.uint8, device="cuda")
    ws = N.workspace(n, b, xd.device)
    for ki, K in enumerate(K_BOUNDARIES):
        rule = RULES[ki % 2]
        pts = pinned_points(K, 700 + K)
        ptsd = cuda(pts)
        i8 = torch.empty(n, dtype=torch.uint8, device="cuda")
        a_ref, b_ref = fresh(rows, torch.float32), fresh(rows, torch.float32)
        N.check(lib.qd_nonuniform_fwd(N.ptr(xd), N.ptr(ptsd), K, rule_of(N, rule), None, N.ptr(i8), None, N.ptr(a_ref), N.ptr(b_ref),
                                      n, b, None, 0.0, N.ptr(ws), ws.numel(), sp))
        for bits in (1, 2, 4, 8):
            nbytes = (n * bits + 7) // 8
            pb = torch.empty(nbytes + 8, dtype=torch.uint8, device="cuda")
            if bits < bits_for(K):
                pb.fill_(SENT8)
                alpha, beta = fresh(rows, torch.float32), fresh(rows, torch.float32)
                rc = lib.qd_nonuniform_fwd_packed(N.ptr(xd), N.ptr(ptsd), K, rule_of(N, rule), N.ptr(pb), bits, N.ptr(alpha),
                                                  N.ptr(beta), n, b, N.ptr(pw), pw.numel(), sp)
                assert rc == N.QD_ERR_INVALID_ARG, (K, bits, rc)
                torch.cuda.synchronize()
                assert bool((pb == SENT8).all()) and bool((alpha.view(torch.int32) == SENT).all()), (K, bits, "written")
                continue
            want = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
            N.check(lib.qd_pack_indices(N.ptr(i8), N.ptr(want), n, bits, sp))
            for ox, op in ((0, 0), (1, 0), (2, 0), (3, 0), (0, 1), (0, 2), (0, 3), (1, 2)):
                what = f"packed L={L} n={n} K={K} {rule} bits={bits} x+{ox} packed+{op}"
                xv = xb[ox:ox + n]
                xv.copy_(xd)
                pb.fill_(SENT8)
                alpha, beta = fresh(rows, torch.float32), fresh(rows, torch.float32)
                N.check(lib.qd_nonuniform_fwd_packed(N.ptr(xv), N.ptr(ptsd), K, rule_of(N, rule), N.ptr(pb[op:]), bits, N.ptr(alpha),
                                                     N.ptr(beta), n, b, N.ptr(pw), pw.numel(), sp))
                same_bits(pb[op:op + nbytes], want, what + " bytes")
                assert bool((pb[:op] == SENT8).all()) and bool((pb[op + nbytes:] == SENT8).all()), what + ": written outside"
                same_bits(alpha, a_ref, what + " alpha")
                same_bits(beta, b_ref, what + " beta")
