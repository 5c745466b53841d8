"""H100 implementation of the reference's ``quantization.quant_functions``.

Same public names, argument meaning, return values and error behaviour as
``quantization/quant_functions.py`` of antspy/quantized_distillation (cited as
file:line below), but every op is ONE fused sm_90a kernel behind the C ABI of
``include/qd_b200.h`` instead of a chain of ~12 torch launches (uniform) or a
device->numpy->device round trip (non-uniform).

Tensors may live on a CUDA device (results stay there, work is enqueued on
torch's current stream, no host synchronisation) or on the host (the op still
runs on the GPU: the tensor is staged through the device and the result comes
back as a CPU tensor).  There is no CPU implementation: without a CUDA device
every call raises RuntimeError.
"""
from __future__ import annotations

import numbers

import torch

from .. import _native as N

# Row a10 of the scope table.  'absmax' / 'absnorm' scaling cannot execute in the reference
# (quant_functions.py:119-126: `tensor.max(p=2)`, a bound method stored as the scale), so there is nothing to be
# bit-identical TO.  The kernels implement what the lines evidently intend (csrc/qd_abs_path.cuh) as an
# extension with "parity: unpinned"; it stays refused unless the caller opts in explicitly.
ALLOW_UNPINNED_SCALING = False
_ABS_KIND = {"absmax": N.SCALE_ABSMAX, "absnorm": N.SCALE_ABSNORM}

__all__ = ("ScalingFunction", "uniformQuantization", "nonUniformQuantization", "uniformQuantization_variable",
           "nonUniformQuantization_variable", "SearchSorted")


# --------------------------------------------------------------------------- helpers
def _bucket_arg(bucket_size) -> int:
    return 0 if bucket_size is None else int(bucket_size)


def _check_tensor(t: torch.Tensor, name="tensor") -> None:
    if not torch.is_tensor(t):
        raise TypeError(f"{name} must be a torch tensor")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32 (got {t.dtype}); the quantization kernels are float32 like the reference")
    if t.numel() == 0:
        raise ValueError(f"{name} is empty")


def _to_device(t: torch.Tensor) -> torch.Tensor:
    """Contiguous CUDA view/copy of ``t`` (the reference flattens with .view(-1),
    i.e. also requires contiguity, help_functions.py:72)."""
    N.require_cuda()
    if not t.is_cuda:
        t = t.cuda(non_blocking=True)
    return t if t.is_contiguous() else t.contiguous()


def _max_element_arg(max_element) -> float:
    return 0.0 if max_element is False or max_element is None else float(max_element)


def _mean_tensor(x: torch.Tensor, subtract_mean: bool):
    """0-dim device tensor holding the mean (no host sync), or None."""
    return x.mean().reshape(1) if subtract_mean else None


class ScalingFunction(object):
    """Scale a tensor to [0, 1] bucket by bucket and back
    (reference: quant_functions.py:7-152).  Keeps the same public fields, which
    other reference code reads (help_functions.py:148-149, 216;
    quant_functions.py:351-363, 467)."""

    def __init__(self, type_scaling, max_element, subtract_mean, bucket_size, modify_in_place=False):
        type_scaling = type_scaling.lower()
        if type_scaling not in ("linear", "absmax", "absnorm"):                          # :22-25
            raise ValueError('Incorrect parameter: type of scaling must be "linear", "absMax" or "absNorm"')
        if bucket_size is not None and (not isinstance(bucket_size, int) or bucket_size <= 0):   # :27-29
            raise ValueError("Bucket size must be an integer and strictly positive. "
                             "Pass None if you want to avoid using buckets")
        if max_element is True or (max_element is not False and not isinstance(max_element, numbers.Number)):  # :31-33
            raise ValueError("maxElementAllowed must be a number")
        if type_scaling != "linear" and not ALLOW_UNPINNED_SCALING:
            # absmax / absnorm cannot execute in the reference (tensor.max(p=2) is invalid and
            # norm_scaling is bound to a method, quant_functions.py:119-126); no parity target exists.
            raise NotImplementedError("'absmax'/'absnorm' scaling is broken in the reference (quant_functions.py:119-126) "
                                      "and used by no experiment; the intended semantics exist here as an extension WITHOUT "
                                      "a parity target: set quantization.quant_functions.ALLOW_UNPINNED_SCALING = True to use it")
        self.type_scaling = type_scaling
        self.max_element = max_element
        self.subtract_mean = subtract_mean
        self.bucket_size = bucket_size
        self.modify_in_place = modify_in_place
        self.tol_diff_zero = 1e-10

        self.mean_tensor = None
        self.original_tensor_size = None
        self.original_tensor_length = None
        self.expected_tensor_size = None
        self.alpha = None
        self.beta = None
        self.idx_min_rows = None
        self.idx_max_rows = None
        self.norm_scaling = None
        self.tensor_sign = None
        self._mean_dev = None      # 1-element device tensor or None
        self._was_cpu = False

    # ---- internal: allocate the per-row state for a tensor of n elements ----
    def _prepare(self, x: torch.Tensor, want_arg=True):
        n = x.numel()
        rows, row_len, padded = N.geometry(n, _bucket_arg(self.bucket_size))
        dev = x.device
        stat_shape = (rows, 1) if self.bucket_size is not None else (1,)
        ab = torch.empty((2,) + stat_shape, dtype=torch.float32, device=dev)       # one allocation for alpha and beta
        self.alpha, self.beta = ab[0], ab[1]
        if want_arg:
            mm = torch.empty((2,) + stat_shape, dtype=torch.int64, device=dev)
            self.idx_min_rows, self.idx_max_rows = mm[0], mm[1]
        self.original_tensor_length = n
        self.expected_tensor_size = torch.Size((rows, row_len)) if self.bucket_size is not None else torch.Size((n,))
        self._mean_dev = _mean_tensor(x, self.subtract_mean)
        self.mean_tensor = self._mean_dev[0] if self._mean_dev is not None else 0      # :66-70
        return rows, row_len, padded

    def _finish(self):
        if self._was_cpu:
            for name in ("alpha", "beta", "idx_min_rows", "idx_max_rows"):
                v = getattr(self, name)
                if v is not None:
                    setattr(self, name, v.cpu())
            if self._mean_dev is not None:
                self.mean_tensor = self._mean_dev[0].cpu()

    def _scale_down_abs(self, tensor):
        """absmax / absnorm (extension, parity unpinned): |x| / norm per bucket, sign kept aside (:109-127)."""
        self._was_cpu = not tensor.is_cuda
        self.original_tensor_size = tensor.size()
        x = _to_device(tensor)
        n = x.numel()
        b = _bucket_arg(self.bucket_size)
        rows, row_len, padded = N.geometry(n, b)
        self.original_tensor_length = n
        self.expected_tensor_size = torch.Size((rows, row_len)) if self.bucket_size is not None else torch.Size((n,))
        self._mean_dev = _mean_tensor(x, self.subtract_mean)
        self.mean_tensor = self._mean_dev[0] if self._mean_dev is not None else 0
        out = torch.empty(padded, dtype=torch.float32, device=x.device)
        sign = torch.empty(padded, dtype=torch.float32, device=x.device)
        norm = torch.empty((rows, 1) if self.bucket_size is not None else (1,), dtype=torch.float32, device=x.device)
        N.check(N.lib().qd_scale_down_abs(N.ptr(x), N.ptr(out), N.ptr(sign), N.ptr(norm), n, b, _ABS_KIND[self.type_scaling],
                                          N.ptr(self._mean_dev), _max_element_arg(self.max_element), N.stream_ptr(x.device)))
        self.norm_scaling, self.tensor_sign = norm, sign.view(self.expected_tensor_size)
        out = out.view(self.expected_tensor_size)
        if self._was_cpu:
            out, self.norm_scaling, self.tensor_sign = out.cpu(), norm.cpu(), self.tensor_sign.cpu()
            if self._mean_dev is not None:
                self.mean_tensor = self._mean_dev[0].cpu()
        return out

    def scale_down(self, tensor):
        """(x - beta)/alpha per bucket; returns the (rows, bucket) tensor, padded
        with copies of the last element like the reference (:56-129)."""
        _check_tensor(tensor)
        if self.type_scaling != "linear":
            return self._scale_down_abs(tensor)
        self._was_cpu = not tensor.is_cuda
        self.original_tensor_size = tensor.size()
        x = _to_device(tensor)
        rows, row_len, padded = self._prepare(x)
        reuse = self.modify_in_place and padded == x.numel() and not self._was_cpu
        out = x.view(-1) if reuse else torch.empty(padded, dtype=torch.float32, device=x.device)
        ws = N.workspace(x.numel(), _bucket_arg(self.bucket_size), x.device)
        N.check(N.lib().qd_scale_down(N.ptr(x), N.ptr(out), N.ptr(self.alpha), N.ptr(self.beta), N.ptr(self.idx_min_rows),
                                      N.ptr(self.idx_max_rows), x.numel(), _bucket_arg(self.bucket_size),
                                      N.ptr(self._mean_dev), _max_element_arg(self.max_element), N.ptr(ws), ws.numel(),
                                      N.stream_ptr(x.device)))
        out = out.view(self.expected_tensor_size)
        if self._was_cpu:
            out = out.cpu()
            if self.modify_in_place and padded == tensor.numel():
                tensor.view(-1).copy_(out.view(-1))
                out = tensor.view(self.expected_tensor_size)
        self._finish()
        return out

    def inv_scale_down(self, tensor):
        """y*alpha + beta (+ mean), padding dropped, original shape restored (:131-152)."""
        _check_tensor(tensor)
        if self.type_scaling != "linear":
            if self.norm_scaling is None or self.tensor_sign is None:
                raise ValueError("scale_down must be called before inv_scale_down")
            if tensor.size() != self.expected_tensor_size:
                raise ValueError("The tensor passed has not the expected size.")
            was_cpu = not tensor.is_cuda
            y = _to_device(tensor)
            n = self.original_tensor_length
            out = torch.empty(n, dtype=torch.float32, device=y.device)
            mean_dev = self._mean_dev.to(y.device) if self._mean_dev is not None else None
            N.check(N.lib().qd_inv_scale_down_abs(N.ptr(y), N.ptr(self.tensor_sign.to(y.device).contiguous()),
                                                  N.ptr(self.norm_scaling.to(y.device)), N.ptr(mean_dev), N.ptr(out), n,
                                                  _bucket_arg(self.bucket_size), N.stream_ptr(y.device)))
            out = out.view(self.original_tensor_size)
            return out.cpu() if was_cpu else out
        if self.alpha is None:
            raise ValueError("scale_down must be called before inv_scale_down")
        if tensor.size() != self.expected_tensor_size:                                   # :138-139
            raise ValueError("The tensor passed has not the expected size.")
        was_cpu = not tensor.is_cuda
        y = _to_device(tensor)
        n = self.original_tensor_length
        alpha, beta = self.alpha.to(y.device), self.beta.to(y.device)
        reuse = self.modify_in_place and not was_cpu and y.numel() == n
        out = y.view(-1) if reuse else torch.empty(n, dtype=torch.float32, device=y.device)
        mean_dev = self._mean_dev.to(y.device) if self._mean_dev is not None else None
        N.check(N.lib().qd_inv_scale_down(N.ptr(y), N.ptr(out), N.ptr(alpha), N.ptr(beta), N.ptr(mean_dev), n,
                                          _bucket_arg(self.bucket_size), N.stream_ptr(y.device)))
        out = out.view(self.original_tensor_size)
        return out.cpu() if was_cpu else out


# --------------------------------------------------------------------------- uniform
def uniformQuantization(tensor, s, type_of_scaling="linear", stochastic_rounding=False, max_element=False,
                        subtract_mean=False, bucket_size=None, modify_in_place=False):
    """Uniform quantization with ``s`` levels (reference: quant_functions.py:155-194).
    Returns ``(quantized tensor, ScalingFunction)``.  One fused kernel: bucket
    min/max, scale, round, de-scale -- 8 bytes of HBM traffic per element."""
    _check_tensor(tensor)
    if modify_in_place and not tensor.is_contiguous():
        raise ValueError("modify_in_place needs a contiguous tensor (the reference's .view(-1) has the same requirement)")
    scaling_function = ScalingFunction(type_of_scaling, max_element, subtract_mean, bucket_size, modify_in_place=True)
    fast = N.fast()
    if (fast is not None and tensor.is_cuda and tensor.is_contiguous() and scaling_function.type_scaling == "linear"
            and not stochastic_rounding and max_element is False and not subtract_mean):
        # compiled front door: allocation, stream lookup and the C-ABI call happen in C++ (same kernel, same bits)
        sf = scaling_function
        n = tensor.numel()
        q, sf.alpha, sf.beta, sf.idx_min_rows, sf.idx_max_rows = fast.uniform_fwd(tensor, int(s), _bucket_arg(bucket_size),
                                                                                   bool(modify_in_place))
        sf.original_tensor_size = tensor.size()
        sf.original_tensor_length = n
        sf.expected_tensor_size = torch.Size((sf.alpha.size(0), bucket_size if n >= bucket_size else n)) if bucket_size is not None \
            else torch.Size((n,))
        sf.mean_tensor = 0
        return q, sf
    was_cpu = not tensor.is_cuda
    x = _to_device(tensor)
    scaling_function._was_cpu = was_cpu
    scaling_function.original_tensor_size = tensor.size()
    if scaling_function.type_scaling != "linear":        # a10 extension (parity unpinned): one fused kernel as well
        if stochastic_rounding:
            raise NotImplementedError("stochastic rounding is not offered with absmax / absnorm scaling")
        sf = scaling_function
        n, b = x.numel(), _bucket_arg(bucket_size)
        rows, row_len, _ = N.geometry(n, b)
        sf.original_tensor_length = n
        sf.expected_tensor_size = torch.Size((rows, row_len)) if bucket_size is not None else torch.Size((n,))
        sf._mean_dev = _mean_tensor(x, subtract_mean)
        sf.mean_tensor = sf._mean_dev[0] if sf._mean_dev is not None else 0
        sf.norm_scaling = torch.empty((rows, 1) if bucket_size is not None else (1,), dtype=torch.float32, device=x.device)
        in_place = modify_in_place and not was_cpu and x.data_ptr() == tensor.data_ptr()
        q = x if in_place else torch.empty_like(x)
        N.check(N.lib().qd_uniform_fwd_abs(N.ptr(x), N.ptr(q), None, N.ptr(sf.norm_scaling), n, b, int(s), _ABS_KIND[sf.type_scaling],
                                           N.ptr(sf._mean_dev), _max_element_arg(max_element), N.stream_ptr(x.device)))
        q = q.view(tensor.size())
        if was_cpu:
            q, sf.norm_scaling = q.cpu(), sf.norm_scaling.cpu()
            if modify_in_place:
                tensor.copy_(q)
                q = tensor
        return q, sf
    scaling_function._prepare(x)
    in_place = modify_in_place and not was_cpu and x.data_ptr() == tensor.data_ptr()
    q = x if in_place else torch.empty_like(x)
    b = _bucket_arg(bucket_size)
    ws = N.workspace(x.numel(), b, x.device) if N.needs_workspace(x.numel(), b) else None     # grid path only
    seed = offset = 0
    if stochastic_rounding:
        # one Philox stream per call, keyed from torch's default (host) generator so that
        # torch.manual_seed controls it (the reference draws torch.rand on the host, :185)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    rc = N.lib().qd_uniform_fwd(x.data_ptr(), q.data_ptr(), None, scaling_function.alpha.data_ptr(),
                                scaling_function.beta.data_ptr(), scaling_function.idx_min_rows.data_ptr(),
                                scaling_function.idx_max_rows.data_ptr(), x.numel(), b, int(s),
                                N.ptr(scaling_function._mean_dev), _max_element_arg(max_element),
                                1 if stochastic_rounding else 0, seed, offset, N.ptr(ws), ws.numel() if ws is not None else 0,
                                N.stream_ptr(x.device))
    if rc:
        N.check(rc)
    q = q.view(tensor.size())
    if was_cpu:
        q = q.cpu()
        if modify_in_place:
            tensor.copy_(q)
            q = tensor
    scaling_function._finish()
    return q, scaling_function


class uniformQuantization_variable(object):
    """Forward/backward pair of the uniform op, called instance-style by the
    training loop (``f.forward(p.data)`` / ``f.backward(p.grad.data)``,
    cnn_models/conv_forward_model.py:245, 266; reference: quant_functions.py:293-406).

    ``backward`` is the reference's hand-written gradient through the bucket
    min/max: with q the quantized tensor re-scaled by its own bucket extremes,
    ``r_b = sum_j g_j (q_hat_j - x_hat_j)`` is added to the gradient at the
    bucket's argmax and subtracted at its argmin.  (As written the reference
    code does not execute for more than one bucket -- two broadcasting bugs,
    SURVEY.md section 8 row a5 -- this is the same formula, per bucket.)"""

    def __init__(self, s, type_of_scaling="linear", stochastic_rounding=False, max_element=False, subtract_mean=False,
                 modify_in_place=False, bucket_size=None):
        self.s = s
        self.typeOfScaling = type_of_scaling
        self.stochasticRounding = stochastic_rounding
        self.maxElementAllowed = max_element
        self.subtractMean = subtract_mean
        self.modifyInPlace = modify_in_place
        self.bucket_size = bucket_size
        self.saved_for_backward = None

    def forward(self, input):
        self.saved_for_backward = {"input": input.clone()}                                # :308-309
        return uniformQuantization(input, s=self.s, type_of_scaling=self.typeOfScaling,
                                   stochastic_rounding=self.stochasticRounding, max_element=self.maxElementAllowed,
                                   subtract_mean=self.subtractMean, modify_in_place=self.modifyInPlace,
                                   bucket_size=self.bucket_size)[0]

    def backward(self, grad_output):
        if self.typeOfScaling != "linear":                                               # :326-327
            raise ValueError("Linear scaling is necessary to backpropagate")
        if self.subtractMean is True:                                                    # :329-330
            raise NotImplementedError("The backprop function assumes subtractMean to be False for now")
        if self.bucket_size is None:                                                     # :332-334
            raise NotImplementedError("Right now the code does not work with bucket_size None. Not hard to modify though")
        if self.saved_for_backward is None:                                              # :336-337
            raise ValueError("Need to have called .forward() to be able to call .backward()")
        if self.maxElementAllowed is not False or self.stochasticRounding:
            # the reference re-quantizes the saved input with these options inside backward (:341-347);
            # the backward kernel takes neither, so refuse instead of returning a different gradient
            raise NotImplementedError("backward with max_element / stochastic_rounding is not implemented "
                                      "(the reference re-runs the forward with them, quant_functions.py:341-347)")
        _check_tensor(grad_output, "grad_output")
        was_cpu = not grad_output.is_cuda
        x = _to_device(self.saved_for_backward["input"])
        g = _to_device(grad_output)
        if g.numel() != x.numel():
            raise ValueError("grad_output does not match the saved input")
        fast = N.fast()
        if fast is not None and not was_cpu:
            out = fast.uniform_bwd(x, g, int(self.s), int(self.bucket_size), N.BWD_MINMAX)
            self.saved_for_backward = None                                               # :404-405
            return out.view(grad_output.size())
        out = torch.empty_like(g)
        ws = N.workspace(x.numel(), self.bucket_size, x.device)
        N.check(N.lib().qd_uniform_bwd(N.ptr(x), N.ptr(g), N.ptr(out), x.numel(), int(self.bucket_size), int(self.s),
                                       N.BWD_MINMAX, N.ptr(ws), ws.numel(), N.stream_ptr(x.device)))
        self.saved_for_backward = None                                                   # :404-405
        out = out.view(grad_output.size())
        return out.cpu() if was_cpu else out


# --------------------------------------------------------------------------- non-uniform
class SearchSorted(object):
    """Stand-in for the reference's sorted-search accelerator
    (quant_functions.py:509-573).  The reference sorts the scaled tensor once and
    keeps 4x its size in permutations so that each query is a numpy searchsorted
    over the midpoints; on the GPU the same indices, ``#{ j : m_j <= x_hat }``,
    cost K-1 compares per element in registers, so nothing is sorted or cached
    beyond the scaled tensor itself."""

    def __init__(self, tensor, use_k_optimization=True):
        self.scaled = _to_device(tensor if torch.is_tensor(tensor) else torch.as_tensor(tensor)).view(-1)
        self.use_k_optimization = use_k_optimization

    def query(self, k, out_unit=None):
        pts = _points_tensor(k, self.scaled.device)
        idx = torch.empty(self.scaled.numel(), dtype=torch.int64, device=self.scaled.device)
        N.check(N.lib().qd_centroid_index(N.ptr(self.scaled), N.ptr(pts), pts.numel(), N.RULE_MIDPOINT, None, N.ptr(idx),
                                          N.ptr(out_unit), self.scaled.numel(), N.stream_ptr(self.scaled.device)))
        return idx


def _points_tensor(points, device) -> torch.Tensor:
    if isinstance(points, list):                                                         # :238-239
        points = torch.tensor(points, dtype=torch.float32)
    if not torch.is_tensor(points):
        points = torch.as_tensor(points, dtype=torch.float32)
    points = points.detach().to(device=device, dtype=torch.float32).contiguous()
    if points.dim() != 1 or points.numel() < 1:
        raise ValueError("listQuantizationPoints must be a non-empty 1-D list/tensor")
    if points.numel() > 256:
        raise ValueError("at most 256 quantization points are supported")
    return points


def nonUniformQuantization(tensor, listQuantizationPoints, max_element=False, subtract_mean=False, modify_in_place=False,
                           bucket_size=None, pre_processed_values=False, search_sorted_obj=None, scaling_function=None,
                           tensors_info=None, index_dtype=torch.int64):
    """Quantize to the nearest of the given points after bucket scaling
    (reference: quant_functions.py:196-290).  Returns
    ``(quantized tensor, indices, ScalingFunction)``.

    Direct path (``pre_processed_values=False``): nearest-point rule of the
    reference's numpy code (:267-273, ties go right).  Pre-processed path: the
    midpoint rule of ``SearchSorted.query`` (:531-573).  The two differ in about
    one element per million at K=16, so both are implemented.
    ``index_dtype=torch.uint8`` is an extension that cuts index traffic 8x."""
    if pre_processed_values is True and (search_sorted_obj is None or scaling_function is None or tensors_info is None):
        raise ValueError("If values are preprocessed, all pre processed arguments need to be passed")      # :230-231
    if pre_processed_values is False and not (search_sorted_obj is None and scaling_function is None
                                              and tensors_info is None):
        raise ValueError("pre processing is False but you are passing some pre processing values. "
                         "This is probably not what you wanted to do, so to avoid bugs an error is raised")  # :233-236
    if index_dtype not in (torch.int64, torch.uint8):
        raise ValueError("index_dtype must be torch.int64 or torch.uint8")

    if pre_processed_values:
        # scaled values live in search_sorted_obj; indices by the midpoint rule, values = k[idx]
        dev = search_sorted_obj.scaled.device
        unit = torch.empty(search_sorted_obj.scaled.numel(), dtype=torch.float32, device=dev)
        idx = search_sorted_obj.query(listQuantizationPoints, out_unit=unit)
        sf = scaling_function
        saved_mip, sf.modify_in_place = sf.modify_in_place, True
        try:
            moved = not sf.alpha.is_cuda
            if moved:
                sf.alpha, sf.beta = sf.alpha.to(dev), sf.beta.to(dev)
            q = sf.inv_scale_down(unit.view(sf.expected_tensor_size))                     # :286-287
        finally:
            sf.modify_in_place = saved_mip
        idx = idx[: sf.original_tensor_length].view(sf.original_tensor_size)             # :288-289
        if index_dtype == torch.uint8:
            idx = idx.to(torch.uint8)
        if tensors_info is not None and tensors_info[1] is False:
            q, idx = q.cpu(), idx.cpu()
        return q, idx, sf

    _check_tensor(tensor)
    was_cpu = not tensor.is_cuda
    x = _to_device(tensor)
    pts = _points_tensor(listQuantizationPoints, x.device)
    sf = ScalingFunction("linear", max_element, subtract_mean, bucket_size, modify_in_place=True)   # :248-250
    sf._was_cpu = was_cpu
    sf.original_tensor_size = tensor.size()
    sf._prepare(x, want_arg=False)
    in_place = modify_in_place and not was_cpu and x.data_ptr() == tensor.data_ptr()
    q = x if in_place else torch.empty_like(x)
    idx = torch.empty(x.numel(), dtype=index_dtype, device=x.device)
    b = _bucket_arg(bucket_size)
    ws = N.workspace(x.numel(), b, x.device)
    N.check(N.lib().qd_nonuniform_fwd(N.ptr(x), N.ptr(pts), pts.numel(), N.RULE_NEAREST, N.ptr(q),
                                      N.ptr(idx) if index_dtype == torch.uint8 else None,
                                      N.ptr(idx) if index_dtype == torch.int64 else None,
                                      N.ptr(sf.alpha), N.ptr(sf.beta), x.numel(), b, N.ptr(sf._mean_dev),
                                      _max_element_arg(max_element), N.ptr(ws), ws.numel(), N.stream_ptr(x.device)))
    q = q.view(tensor.size())
    idx = idx.view(tensor.size())
    if was_cpu:
        q, idx = q.cpu(), idx.cpu()
        if modify_in_place:
            tensor.copy_(q)
            q = tensor
    sf._finish()
    return q, idx, sf


class nonUniformQuantization_variable(object):
    """Differentiable-centroid quantization of one fixed tensor (reference:
    quant_functions.py:408-506), called instance-style by
    ``optimize_quantization_points`` (cnn_models/conv_forward_model.py:507-545):
    ``forward(None, points)`` re-quantizes the tensor with the current points,
    ``backward(g)`` returns ``(g, dLoss/dpoints)``.

    With ``pre_process_tensors=True`` the reference caches the scaled tensor,
    its argsort and the inverse permutation; here only the tensor is kept and
    each forward is one fused kernel (scale, midpoint search, de-scale, uint8
    indices): 9 bytes per element, no host round trip."""

    def __init__(self, max_element=False, subtract_mean=False, modify_in_place=False, bucket_size=None,
                 pre_process_tensors=False, tensor=None):
        if pre_process_tensors is True and (tensor is None):                             # :413-414
            raise ValueError("To pre-process tensors you need to pass the tensor and the scaling function options")
        self.maxElementAllowed = max_element
        self.subtractMean = subtract_mean
        self.modifyInPlace = modify_in_place
        self.bucket_size = bucket_size
        self.savedForBackward = None
        self.pre_process_tensors = pre_process_tensors
        self._search_sorted_obj = None
        self.tensors_info = None
        self.scaling_function = None
        self._tensor = None
        self._was_cpu = False
        if self.pre_process_tensors:
            self.preprocess(tensor)

    def preprocess(self, tensor):
        _check_tensor(tensor)
        self._was_cpu = not tensor.is_cuda
        x = _to_device(tensor)
        self._tensor = x if self.modifyInPlace else x.clone()                             # :433-434
        sf = ScalingFunction("linear", self.maxElementAllowed, self.subtractMean, self.bucket_size, modify_in_place=True)
        sf._was_cpu = False
        sf.original_tensor_size = tensor.size()
        sf._prepare(self._tensor, want_arg=False)
        self.scaling_function = sf
        self.tensors_info = (tensor.type(), tensor.is_cuda)                               # :446
        self._search_sorted_obj = None                                                    # built lazily, see the property

    @property
    def search_sorted_obj(self):
        """The reference builds a SearchSorted over the scaled tensor at :445.  forward()
        here never needs it (the fused kernel re-derives the scaling), so it is only
        materialised if a caller asks for it, e.g. to drive nonUniformQuantization's
        pre-processed path by hand (:218-227)."""
        if self._search_sorted_obj is None and self._tensor is not None:
            sf = ScalingFunction("linear", self.maxElementAllowed, self.subtractMean, self.bucket_size, False)
            self._search_sorted_obj = SearchSorted(sf.scale_down(self._tensor).view(-1))
        return self._search_sorted_obj

    def _fused_forward(self, x, points, rule, sf, out=None):
        pts = _points_tensor(points, x.device)
        if out is not None:
            if not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == x.numel()):
                raise ValueError("out must be a contiguous float32 CUDA tensor with as many elements as the input")
            q = out
        else:
            q = torch.empty_like(x)
        idx = torch.empty(x.numel(), dtype=torch.uint8, device=x.device)
        b = _bucket_arg(self.bucket_size)
        ws = N.workspace(x.numel(), b, x.device)
        N.check(N.lib().qd_nonuniform_fwd(N.ptr(x), N.ptr(pts), pts.numel(), rule, N.ptr(q), N.ptr(idx), None,
                                          N.ptr(sf.alpha), N.ptr(sf.beta), x.numel(), b, N.ptr(sf._mean_dev),
                                          _max_element_arg(self.maxElementAllowed), N.ptr(ws), ws.numel(),
                                          N.stream_ptr(x.device)))
        return q, idx

    def forward(self, inputTensor, listQuantizationPoints, out=None):
        """``out`` (extension): write the quantized tensor straight into an existing
        tensor, e.g. the live parameter, instead of allocating a new one."""
        if listQuantizationPoints.dim() != 1:                                            # :451-452
            raise ValueError("listPoints must be a 1-D tensor")
        numPoints = listQuantizationPoints.size()[0]
        if self.pre_process_tensors:
            x, sf, rule, was_cpu = self._tensor, self.scaling_function, N.RULE_MIDPOINT, self._was_cpu
            shape = sf.original_tensor_size
        else:
            _check_tensor(inputTensor)
            was_cpu = not inputTensor.is_cuda
            x = _to_device(inputTensor)
            sf = ScalingFunction("linear", self.maxElementAllowed, self.subtractMean, self.bucket_size, True)
            sf.original_tensor_size = inputTensor.size()
            sf._prepare(x, want_arg=False)
            rule, shape = N.RULE_NEAREST, inputTensor.size()
        q, idx = self._fused_forward(x, listQuantizationPoints, rule, sf, out=out)
        self.savedForBackward = {"indices": idx.view(shape), "numPoints": numPoints, "scalingFactor": sf.alpha}   # :467-468
        q = q.view(shape)
        return q.cpu() if was_cpu else q

    def backward(self, grad_output):
        grad_inputTensor = grad_output                                                    # :473 (same object: STE)
        if self.savedForBackward is None:                                                 # :478-479
            raise ValueError("Need savedIndices to be able to call backward()")
        _check_tensor(grad_output, "grad_output")
        idx = self.savedForBackward["indices"]
        K = self.savedForBackward["numPoints"]
        alpha = self.savedForBackward["scalingFactor"]
        g = _to_device(grad_output)
        if g.numel() != idx.numel():
            raise ValueError("grad_output does not match the quantized tensor")
        idx, alpha = idx.to(g.device), alpha.to(g.device)
        out = torch.empty(K, dtype=torch.float32, device=g.device)
        b = _bucket_arg(self.bucket_size)
        ws = N.workspace(g.numel(), b, g.device)
        N.check(N.lib().qd_nonuniform_bwd(N.ptr(g), N.ptr(idx) if idx.dtype == torch.uint8 else None,
                                          N.ptr(idx) if idx.dtype == torch.int64 else None, N.ptr(alpha), K, N.ptr(out),
                                          g.numel(), b, N.ptr(ws), ws.numel(), N.stream_ptr(g.device)))
        self.savedIndices = None                                                          # :505
        if not grad_output.is_cuda:
            out = out.cpu()
        return grad_inputTensor, out
