"""CPU oracle for the fake-quantization hot path -- TEST INFRASTRUCTURE ONLY.

This file is a NumPy restatement of the per-tensor arithmetic of the reference
(antspy/quantized_distillation, ``quantization/quant_functions.py`` and
``quantization/help_functions.py``).  It is the *checker* for the CUDA path:
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline
legs may import it.  Nothing under ``quantized_distillation_b200/`` imports it,
and the product path raises when the CUDA extension is missing instead of
falling back to this code.

Pinning: the reference holds no tests or golden vectors for this path
(SURVEY.md section 4), so the oracle is pinned against the reference *itself*:
``tests/golden/make_golden.py`` imports ``/root/reference/quantization``
unmodified, runs it on seeded inputs and stores input/output pairs under
``tests/golden/`` (``make_golden_options.py`` does the same for ``subtract_mean``,
``max_element`` and stochastic rounding with the reference's own ``torch.rand``
draws); ``tests/test_oracle_golden.py`` checks every function below
bit-for-bit (tolerance only where the reference itself sums in a different
order) against those fixtures.

Every function computes in float32 with one IEEE rounding per reference torch
op (no fused multiply-add), which is what the chain of in-place torch ops in
the reference does.

Citations are ``path:line`` relative to the reference checkout.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
TOL_DIFF_ZERO = F32(1e-10)  # quantization/quant_functions.py:40


# --------------------------------------------------------------------------
# a1: bucket geometry (quantization/help_functions.py:67-94)
# --------------------------------------------------------------------------
def bucket_geometry(n: int, bucket_size):
    """Returns (num_buckets, row_len, padded_len) of the bucketed view.

    * ``bucket_size`` None -> one row holding the whole tensor
      (quant_functions.py:79-80, 85-87).
    * n < bucket_size     -> one row of n elements, no padding
      (help_functions.py:87-90).
    * otherwise           -> ceil(n / b) rows of b; the tail row is padded with
      copies of the LAST element (help_functions.py:75-76, 80-86).
    """
    if n <= 0:
        raise ValueError("empty tensor")
    if bucket_size is None:
        return 1, n, n
    if bucket_size <= 0:
        raise ValueError("bucket size must be positive")
    multiple, rest = divmod(n, bucket_size)
    if multiple == 0:
        return 1, n, n
    rows = multiple + (1 if rest else 0)
    return rows, bucket_size, rows * bucket_size


def bucketed(x: np.ndarray, bucket_size) -> np.ndarray:
    """Materialises the padded (rows, row_len) view used by the reference."""
    flat = np.asarray(x, dtype=F32).reshape(-1)
    rows, row_len, padded = bucket_geometry(flat.size, bucket_size)
    if padded != flat.size:
        flat = np.concatenate([flat, np.full(padded - flat.size, flat[-1], dtype=F32)])
    return flat.reshape(rows, row_len)


# --------------------------------------------------------------------------
# a2 / a3: linear scaling and its inverse (quant_functions.py:56-107, 131-152)
# --------------------------------------------------------------------------
def pre_ops(x: np.ndarray, subtract_mean=False, max_element=False, mean=None):
    """Optional global mean subtraction and clamp (quant_functions.py:66-74).  ``mean`` overrides the
    computed mean: the reference's is a float32 torch reduction whose last bit depends on the summation
    order, so everything AFTER the mean is pinned bit for bit by handing the reference's own value in
    (tests/test_oracle_golden.py), and the mean itself within a summation-order tolerance."""
    flat = np.asarray(x, dtype=F32).reshape(-1).copy()
    if subtract_mean:
        mean = F32(flat.mean(dtype=np.float64)) if mean is None else F32(mean)   # order-dependent in the reference
        flat = flat - mean
    else:
        mean = F32(0)
    if max_element is not False:
        m = F32(max_element)
        flat = np.minimum(np.maximum(flat, -m), m)
    return flat, mean


def bucket_stats(rows: np.ndarray):
    """beta=min, alpha=max-min (tiny -> 1), first-occurrence argmin/argmax per
    row (quant_functions.py:84-104)."""
    beta = rows.min(axis=1)
    mx = rows.max(axis=1)
    argmin = rows.argmin(axis=1).astype(np.int64)
    argmax = rows.argmax(axis=1).astype(np.int64)
    alpha = (mx - beta).astype(F32)
    alpha = np.where(alpha < TOL_DIFF_ZERO, F32(1), alpha).astype(F32)
    return alpha, beta.astype(F32), argmin, argmax


def scale_down(x, bucket_size, subtract_mean=False, max_element=False, mean=None):
    """x_hat = (x - beta) / alpha: subtract, then true division
    (quant_functions.py:106-107).  Returns the padded (rows, row_len) array and
    the per-row state the reference keeps on the ScalingFunction object."""
    flat, mean = pre_ops(x, subtract_mean, max_element, mean)
    rows = bucketed(flat, bucket_size)
    alpha, beta, argmin, argmax = bucket_stats(rows)
    xh = ((rows - beta[:, None]).astype(F32) / alpha[:, None]).astype(F32)
    return xh, dict(alpha=alpha, beta=beta, argmin=argmin, argmax=argmax, mean=mean,
                    n=flat.size, shape=np.shape(x))


def inv_scale_down(y_rows: np.ndarray, st) -> np.ndarray:
    """y*alpha, +beta, +mean, drop padding (quant_functions.py:141-150)."""
    y = (np.asarray(y_rows, dtype=F32) * st["alpha"][:, None]).astype(F32)
    y = (y + st["beta"][:, None]).astype(F32)
    y = (y + st["mean"]).astype(F32)
    return y.reshape(-1)[: st["n"]].reshape(st["shape"])


# --------------------------------------------------------------------------
# a4: uniform quantization (quant_functions.py:155-194)
# --------------------------------------------------------------------------
def uniform_levels(xh: np.ndarray, s: int) -> np.ndarray:
    """idx = rint(x_hat * (s-1)), round-half-even (quant_functions.py:172,189-190)."""
    S = F32(s - 1)
    return np.rint((xh * S).astype(F32)).astype(F32)


def uniform_fwd(x, s: int, bucket_size, subtract_mean=False, max_element=False, mean=None):
    """Returns (q, idx, state).  q = ((idx/S)*alpha + beta) (+mean), each op
    rounded to float32 (quant_functions.py:189-193, 142-148)."""
    xh, st = scale_down(x, bucket_size, subtract_mean, max_element, mean)
    S = F32(s - 1)
    lvl = uniform_levels(xh, s)
    q = inv_scale_down((lvl / S).astype(F32), st)
    idx = lvl.reshape(-1)[: st["n"]].astype(np.int64).reshape(st["shape"])
    return q, idx, st


def uniform_fwd_stochastic(x, s: int, bucket_size, u: np.ndarray, subtract_mean=False, max_element=False, mean=None):
    """Stochastic rounding given the uniform draws ``u`` (padded layout):
    floor(x_hat*S)/S + [u <= frac]/S (quant_functions.py:179-187)."""
    xh, st = scale_down(x, bucket_size, subtract_mean, max_element, mean)
    S = F32(s - 1)
    prob = (S * xh).astype(F32)
    fl = np.floor(prob).astype(F32)
    prob = (prob - fl).astype(F32)
    y = (fl / S).astype(F32)
    bump = ((u.reshape(xh.shape) <= prob).astype(F32) * F32(1) / S).astype(F32)
    y = (y + bump).astype(F32)
    return inv_scale_down(y, st), st


# --------------------------------------------------------------------------
# a10: absmax / absnorm scaling -- INTENDED semantics, PARITY UNPINNED.
# quant_functions.py:109-127, 144-146 cannot execute (`tensor.max(p=2)`, `norm_scaling.view` stored as a bound
# method), so the reference yields no output to pin this against; what follows restates what the lines intend
# with the two slips repaired, and only checks that the CUDA extension computes exactly that.
# --------------------------------------------------------------------------
def abs_scale_down(x, bucket_size, kind, norm=None):
    """sign, |x| / norm per (padded) bucket; norm = max (absmax) or L2 over the padded bucket (absnorm, float64
    accumulation rounded once); norm < 1e-10 -> 1.  `norm` overrides the computed scale (for exact checks of what
    follows it when the float64 sum order differs in the last bit)."""
    flat = np.asarray(x, dtype=F32).reshape(-1)
    rows = bucketed(flat, bucket_size)
    sign = np.sign(rows).astype(F32)
    v = np.abs(rows)
    if norm is None:
        if kind == "absmax":
            norm = v.max(axis=1)
        else:
            norm = np.sqrt((v.astype(np.float64) ** 2).sum(axis=1)).astype(F32)
        norm = np.where(norm < TOL_DIFF_ZERO, F32(1), norm).astype(F32)
    norm = np.asarray(norm, dtype=F32).reshape(-1)
    xh = (v / norm[:, None]).astype(F32)
    return xh, sign, norm, flat.size


def uniform_fwd_abs(x, s: int, bucket_size, kind, norm=None):
    """q = ((rint(x_hat*S)/S) * norm) * sign, one float32 rounding per op (:189-191, :145-146)."""
    xh, sign, norm, n = abs_scale_down(x, bucket_size, kind, norm)
    S = F32(s - 1)
    lvl = np.rint((xh * S).astype(F32)).astype(F32)
    q = (((lvl / S).astype(F32) * norm[:, None]).astype(F32) * sign).astype(F32)
    return q.reshape(-1)[:n].reshape(np.shape(x)), lvl.reshape(-1)[:n].astype(np.int64), norm


# --------------------------------------------------------------------------
# a5: backward of uniformQuantization_variable (quant_functions.py:319-406)
# --------------------------------------------------------------------------
def uniform_bwd_minmax(x, g, s: int, bucket_size):
    """The 'complicated' gradient, read literally from the reference with its
    two shape bugs repaired (SURVEY.md section 8 row a5):

    * the quantized tensor q is re-scaled with the SAME ScalingFunction object
      (quant_functions.py:350), which overwrites alpha/beta/argmin/argmax with
      those of q (lines 353-363 then read the overwritten fields);
    * v_j = g_j * (q_hat_j - (x_j - beta')/alpha')          (line 400)
    * out = g + M^T v, M[j, argmax'(bucket j)] = +1, M[j, argmin'(bucket j)] = -1
      (lines 380-400), i.e. r_b = sum_{j in b} v_j is added at argmax'_b and
      subtracted at argmin'_b.

    Padding rows never contribute: all per-element vectors are cut to the
    original length before the product (lines 351, 358-374).  Accumulated in
    float64 here; the reference sums in float32 in torch.mm order, so parity on
    r_b is by tolerance.
    """
    if bucket_size is None:
        raise NotImplementedError("reference refuses bucket_size None (quant_functions.py:332-334)")
    q, _, st = uniform_fwd(x, s, bucket_size)
    n = st["n"]
    qh, st2 = scale_down(q, bucket_size)               # line 350: overwrites the state
    rows, row_len = qh.shape
    a2 = np.repeat(st2["alpha"], row_len)[:n]
    b2 = np.repeat(st2["beta"], row_len)[:n]
    xf = np.asarray(x, dtype=F32).reshape(-1)
    gf = np.asarray(g, dtype=F32).reshape(-1)
    xs = ((xf - b2).astype(F32) / a2).astype(F32)
    v = (gf * (qh.reshape(-1)[:n] - xs).astype(F32)).astype(F32)
    out = gf.astype(np.float64).copy()
    owner = np.arange(n) // row_len
    r = np.zeros(rows, dtype=np.float64)
    np.add.at(r, owner, v.astype(np.float64))
    abs_sum = np.zeros(rows, dtype=np.float64)          # scale of the summation-order tolerance, per bucket
    np.add.at(abs_sum, owner, np.abs(v.astype(np.float64)))
    base = np.arange(rows, dtype=np.int64) * row_len
    amax = base + st2["argmax"]
    amin = base + st2["argmin"]
    corr = np.zeros(n, dtype=np.float64)
    np.add.at(corr, amax, r)
    np.add.at(corr, amin, -r)
    out = (gf.astype(np.float64) + corr.astype(F32).astype(np.float64)).astype(F32)
    return out.reshape(np.shape(g)), dict(r=r, abs_sum=abs_sum, row_len=row_len, argmax=amax, argmin=amin,
                                          alpha2=st2["alpha"], beta2=st2["beta"])


def uniform_bwd_truncated(w, g):
    """'truncated' style: grad[|w| > 1] = 0 (cnn_models/conv_forward_model.py:263-264)."""
    out = np.asarray(g, dtype=F32).copy()
    out[np.abs(np.asarray(w, dtype=F32)) > 1] = 0
    return out


# --------------------------------------------------------------------------
# a6 / a7: non-uniform quantization (quant_functions.py:196-290, 509-573)
# --------------------------------------------------------------------------
def midpoints(points: np.ndarray) -> np.ndarray:
    """m_j = k_j + (k_{j+1} - k_j)/2 in float32 (quant_functions.py:533)."""
    k = np.asarray(points, dtype=F32)
    return (k[:-1] + (np.diff(k) / F32(2)).astype(F32)).astype(F32)


def nonuniform_index_midpoint(xh: np.ndarray, points: np.ndarray) -> np.ndarray:
    """SearchSorted.query closed form: idx = #{ j : m_j <= x_hat }
    (quant_functions.py:531-573)."""
    m = midpoints(points)
    return np.searchsorted(m, xh.reshape(-1), side="right").astype(np.int64).reshape(xh.shape)


def nonuniform_index_nearest(xh: np.ndarray, points: np.ndarray) -> np.ndarray:
    """Direct path: searchsorted-left, clip, step left when strictly closer
    (ties stay right) (quant_functions.py:267-273)."""
    k = np.asarray(points, dtype=F32)
    v = xh.reshape(-1)
    i = np.searchsorted(k, v, side="left").clip(max=k.size - 1)
    left = np.fabs(v - k[np.maximum(i - 1, 0)])
    right = np.fabs(v - k[i])
    step = (i > 0) & (left < right)
    return (i - step).astype(np.int64).reshape(xh.shape)


def nonuniform_fwd(x, points, bucket_size, rule="nearest", subtract_mean=False, max_element=False, mean=None):
    """Returns (q, idx, state); q = k[idx]*alpha + beta (+ mean) (quant_functions.py:278-289)."""
    xh, st = scale_down(x, bucket_size, subtract_mean, max_element, mean)
    k = np.asarray(points, dtype=F32)
    idx = nonuniform_index_nearest(xh, k) if rule == "nearest" else nonuniform_index_midpoint(xh, k)
    q = inv_scale_down(k[idx], st)
    idx = idx.reshape(-1)[: st["n"]].reshape(st["shape"])
    return q, idx, st


def dequantize_levels(idx, alpha, beta, bucket_size, s=None, points=None) -> np.ndarray:
    """q of stored levels: unit * alpha + beta of the element's bucket, one float32 rounding per op, where unit is
    idx / (s-1) (uniform, quant_functions.py:191) or points[idx] (non-uniform, :278-289), then the inverse scaling's
    mul_ and add_ (:142-143).  Any bucket, ragged last row included; no mean is added (the stored models have
    none), so a -0.0 stays -0.0.  The flat float32 array of idx.size elements."""
    i = np.asarray(idx).reshape(-1).astype(np.int64)
    _, row_len, _ = bucket_geometry(i.size, bucket_size)
    if points is None:
        unit = (i.astype(F32) / F32(s - 1)).astype(F32)
    else:
        unit = np.asarray(points, dtype=F32).reshape(-1)[i]
    row = np.arange(i.size, dtype=np.int64) // row_len
    a = np.asarray(alpha, dtype=F32).reshape(-1)[row]
    b = np.asarray(beta, dtype=F32).reshape(-1)[row]
    return ((unit * a).astype(F32) + b).astype(F32)


# --------------------------------------------------------------------------
# a8: gradient w.r.t. the centroids (quant_functions.py:471-506)
# --------------------------------------------------------------------------
def nonuniform_bwd_points(g, idx, alpha, num_points: int, bucket_size):
    """grad_points[k] = sum_{i: idx_i = k} fl32(g_i * alpha_bucket(i)).  The
    product is rounded to float32 like the reference's in-place multiply
    (line 495); the sum is exact here (float64), float32 masked sums there
    (line 503) -> tolerance parity."""
    gf = np.asarray(g, dtype=F32).reshape(-1)
    n = gf.size
    _, row_len, _ = bucket_geometry(n, bucket_size)
    a = np.repeat(np.asarray(alpha, dtype=F32).reshape(-1), row_len)[:n]
    v = (gf * a).astype(F32).astype(np.float64)
    out = np.bincount(np.asarray(idx).reshape(-1), weights=v, minlength=num_points)
    return out[:num_points]


# --------------------------------------------------------------------------
# a9: centroid initialisation (help_functions.py:140-154)
# --------------------------------------------------------------------------
def initialize_points(x, bucket_size, num_points: int) -> np.ndarray:
    xh, st = scale_down(x, bucket_size)
    v = xh.reshape(-1)[: st["n"]]
    return np.percentile(v, np.linspace(0, 100, num=num_points)).astype(F32)


# --------------------------------------------------------------------------
# next rows: Huffman statistics (help_functions.py:157-232)
# --------------------------------------------------------------------------
def huffman_mean_bit_length(counts) -> float:
    """Mean code length of a Huffman code over the index histogram.  The mean
    length is independent of tie-breaking, so a plain heap suffices
    (help_functions.py:157-172, 228-230)."""
    import heapq
    counts = [int(c) for c in counts if c > 0]
    total = sum(counts)
    if len(counts) == 1:
        return 0.0  # the reference assigns the empty code to a single symbol
    heap = list(counts)
    heapq.heapify(heap)
    acc = 0
    while len(heap) > 1:
        a = heapq.heappop(heap)
        b = heapq.heappop(heap)
        acc += a + b
        heapq.heappush(heap, a + b)
    return acc / total
