"""Multi-tensor quantization plan: ONE kernel launch quantizes every parameter
tensor of a model (SURVEY.md section 8 f1).

The reference walks ``model.parameters()`` and calls ``uniformQuantization`` per
tensor (cnn_models/conv_forward_model.py:236-247), keeps the full-precision
weights alive through ``model.state_dict()`` and copies them back with
``load_state_dict`` (:286, :302).  Here the full-precision master copy lives in
one flat shadow buffer, the live parameters are quantized IN PLACE (so DDP's
parameter references stay valid), and save / quantize / restore / gradient
fix-up are each a single launch regardless of the number of tensors.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _native as N

_STYLE = {"none": N.BWD_STE, None: N.BWD_STE, "truncated": N.BWD_TRUNCATED, "complicated": N.BWD_MINMAX}


class QuantizationPlan:
    def __init__(self, params, levels, bucket_size=None):
        N.require_cuda()
        self.params = [p.data if isinstance(p, torch.nn.Parameter) else p for p in params]
        if not self.params:
            raise ValueError("no tensors to quantize")
        for p in self.params:
            if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
                raise ValueError("plan tensors must be contiguous float32 CUDA tensors")
        self.device = self.params[0].device
        self.bucket_size = bucket_size
        count = len(self.params)
        self.levels = [int(levels)] * count if isinstance(levels, int) else [int(v) for v in levels]
        if len(self.levels) != count:
            raise ValueError("one level count per tensor expected")
        self._ptrs = (C.c_void_p * count)(*[p.data_ptr() for p in self.params])
        self._n = (C.c_int64 * count)(*[p.numel() for p in self.params])
        self._lv = (C.c_int32 * count)(*self.levels)
        self._handle = C.c_void_p()
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_create(C.byref(self._handle), count, self._ptrs, self._ptrs, self._n, self._lv,
                                           0 if bucket_size is None else int(bucket_size)))
        total = sum(p.numel() for p in self.params)
        # every tensor's shadow starts on a 256-byte boundary so its rows can use 128-bit accesses
        padded = sum(-(-p.numel() // 64) * 64 for p in self.params)
        self._master_flat = torch.empty(padded, dtype=torch.float32, device=self.device)
        self._master, off = [], 0
        for p in self.params:
            self._master.append(self._master_flat[off:off + p.numel()].view(p.shape))
            off += -(-p.numel() // 64) * 64
        self.numel = total
        self._momentum_flat = None
        self.momentum_buffers = None
        self._shadow_ptrs = (C.c_void_p * count)(*[m.data_ptr() for m in self._master])
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_set_shadow(self._handle, self._shadow_ptrs))

    # -- full-precision master copy ------------------------------------------------
    def save_master(self):
        """master <- params (replaces ``model_state_dict = model.state_dict()``, :286)."""
        torch._foreach_copy_(self._master, self.params)
        return self._master

    def restore_master(self):
        """params <- master (replaces ``model.load_state_dict(model_state_dict)``, :302)."""
        torch._foreach_copy_(self.params, self._master)

    # -- quantization -----------------------------------------------------------------
    def quantize_(self):
        """params <- uniformQuantization(params), every tensor, one launch (:236-247)."""
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_uniform_fwd(self._handle, N.stream_ptr(self.device)))

    def save_and_quantize_(self):
        """master <- params and params <- uniformQuantization(params) in ONE pass over the
        weights (12 bytes per element instead of 8 + 8)."""
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_uniform_fwd_save(self._handle, N.stream_ptr(self.device)))
        return self._master

    def backward_(self, grads, style):
        """grads <- gradient fix-up of the chosen backprop_quantization_style, in place,
        evaluated at the CURRENT (full-precision, i.e. restored) params (:249-266)."""
        mode = _STYLE[style]
        if mode == N.BWD_STE:
            return
        if len(grads) != len(self.params):
            raise ValueError("one gradient per tensor expected")
        for g, p in zip(grads, self.params):
            if not (g.is_cuda and g.dtype == torch.float32 and g.is_contiguous() and g.numel() == p.numel()):
                raise ValueError("gradients must be contiguous float32 CUDA tensors matching the params")
        gp = (C.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_uniform_bwd(self._handle, gp, mode, N.stream_ptr(self.device)))

    def fused_step_(self, grads, style, lr, momentum=0.0, weight_decay=0.0, nesterov=False):
        """End of step i and start of step i+1 in ONE pass over the model (24 B/elt): gradient fix-up of
        ``style`` at the master weights, ``torch.optim.SGD`` update of master + momentum buffer, and the
        live parameters re-quantized from the updated master (:302-317, :286-287).  Needs rows of at
        most 512 elements (NotImplementedError otherwise)."""
        if len(grads) != len(self.params):
            raise ValueError("one gradient per tensor expected")
        for g, p in zip(grads, self.params):
            if not (g.is_cuda and g.dtype == torch.float32 and g.is_contiguous() and g.numel() == p.numel()):
                raise ValueError("gradients must be contiguous float32 CUDA tensors matching the params")
        if self._momentum_flat is None:
            self._momentum_flat = torch.zeros_like(self._master_flat)
            self.momentum_buffers, off = [], 0
            for p in self.params:
                self.momentum_buffers.append(self._momentum_flat[off:off + p.numel()].view(p.shape))
                off += -(-p.numel() // 64) * 64
            mp = (C.c_void_p * len(self.params))(*[m.data_ptr() for m in self.momentum_buffers])
            with torch.cuda.device(self.device):
                N.check(N.lib().qd_plan_set_momentum(self._handle, mp))
        gp = (C.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_sgd_step(self._handle, gp, _STYLE[style], float(lr), float(momentum), float(weight_decay),
                                             1 if nesterov else 0, N.stream_ptr(self.device)))

    def close(self):
        if self._handle:
            N.lib().qd_plan_destroy(self._handle)
            self._handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CentroidPlan:
    """Multi-tensor plan of the differentiable-quantization loop
    (cnn_models/conv_forward_model.py:501-551): ``forward_()`` re-quantizes every tensor with its
    own current points in ONE launch (quantized values straight into the live parameters, uint8
    indices and per-row scales kept for the backward), ``backward_(grads)`` returns every tensor's
    centroid gradient from TWO launches -- instead of three launches per tensor per step.

    ``sources`` are the fixed full-precision tensors (the loop never changes them), ``targets`` the
    live parameters of the quantized copy of the model, ``points`` the per-tensor 1-D point
    tensors; the optimizer must update those IN PLACE (their addresses are in the plan).
    Raises ``NotImplementedError`` for more than 32 points or rows longer than 1024 elements:
    callers fall back to the per-tensor ops."""

    MAX_POINTS = 32

    def __init__(self, sources, targets, points, bucket_size=None):
        N.require_cuda()
        count = len(sources)
        if count == 0 or len(targets) != count or len(points) != count:
            raise ValueError("one source, target and point tensor per quantized tensor expected")
        for t in list(sources) + list(targets) + list(points):
            if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
                raise ValueError("plan tensors must be contiguous float32 CUDA tensors")
        self.device = sources[0].device
        self.sources, self.targets, self.points = list(sources), list(targets), list(points)
        self.bucket_size = bucket_size
        b = 0 if bucket_size is None else int(bucket_size)
        geo = [N.geometry(s.numel(), b) for s in sources]
        pad = lambda n, g: -(-n // g) * g
        self._idx_flat = torch.empty(sum(pad(s.numel(), 256) for s in sources), dtype=torch.uint8, device=self.device)
        self._scale_flat = torch.empty(2 * sum(pad(rows, 64) for rows, _, _ in geo), dtype=torch.float32, device=self.device)
        self._gp_flat = torch.zeros(count * self.MAX_POINTS, dtype=torch.float32, device=self.device)
        self.indices, self.alpha, self.beta, self.grad_points = [], [], [], []
        io = so = 0
        for i, (s, (rows, _, _)) in enumerate(zip(sources, geo)):
            self.indices.append(self._idx_flat[io:io + s.numel()].view(s.shape))
            io += pad(s.numel(), 256)
            self.alpha.append(self._scale_flat[so:so + rows])
            so += pad(rows, 64)
            self.beta.append(self._scale_flat[so:so + rows])
            so += pad(rows, 64)
            self.grad_points.append(self._gp_flat[i * self.MAX_POINTS:i * self.MAX_POINTS + points[i].numel()])
        arr = lambda ts: (C.c_void_p * count)(*[t.data_ptr() for t in ts])
        self._n = (C.c_int64 * count)(*[s.numel() for s in sources])
        self._k = (C.c_int32 * count)(*[p.numel() for p in points])
        self._handle = C.c_void_p()
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_nonuniform_create(C.byref(self._handle), count, arr(sources), arr(targets), arr(self.indices),
                                                      arr(self.alpha), arr(self.beta), arr(points), arr(self.grad_points),
                                                      self._n, self._k, b))

    def forward_(self):
        """targets <- nonUniformQuantization(sources, points) for every tensor, one launch (:525-532)."""
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_nonuniform_fwd(self._handle, N.stream_ptr(self.device)))

    def _grad_ptrs(self, grads):
        if len(grads) != len(self.sources):
            raise ValueError("one gradient per tensor expected")
        for g, s in zip(grads, self.sources):
            if not (g.is_cuda and g.dtype == torch.float32 and g.is_contiguous() and g.numel() == s.numel()):
                raise ValueError("gradients must be contiguous float32 CUDA tensors matching the tensors")
        return (C.c_void_p * len(grads))(*[g.data_ptr() for g in grads])

    def _check_sums(self, sums):
        if not (sums.is_cuda and sums.device == self.device and sums.dtype == torch.float64 and sums.is_contiguous()
                and tuple(sums.shape) == (len(self.sources), self.MAX_POINTS)):
            raise ValueError(f"sums must be a contiguous float64 CUDA tensor of shape ({len(self.sources)}, {self.MAX_POINTS}) "
                             "on the plan's device")

    def backward_(self, grads):
        """Every tensor's dLoss/dpoints from dLoss/d(quantized tensor) (:539-545); returns views of one
        flat buffer, overwritten by the next call."""
        gp = self._grad_ptrs(grads)
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_nonuniform_bwd(self._handle, gp, N.stream_ptr(self.device)))
        return self.grad_points

    def backward_partial_(self, grads, sums):
        """``backward_`` up to its last rounding: writes every tensor's float64 centroid-gradient sums into
        ``sums`` (float64, shape ``(tensors, 32)``, zeros past each tensor's point count) and leaves
        ``grad_points`` alone.  Data-parallel training reduces ``sums`` across ranks, then calls ``finish_``."""
        gp = self._grad_ptrs(grads)
        self._check_sums(sums)
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_nonuniform_bwd_partial(self._handle, gp, N.ptr(sums), N.stream_ptr(self.device)))
        return sums

    def finish_(self, sums, scale=1.0):
        """``grad_points[t][k] = float32(sums[t][k] * scale)``; returns ``grad_points``.  ``backward_partial_``
        followed by ``finish_(sums, 1.0)`` gives ``backward_``'s result bit for bit."""
        self._check_sums(sums)
        with torch.cuda.device(self.device):
            N.check(N.lib().qd_plan_nonuniform_bwd_finish(self._handle, N.ptr(sums), float(scale), N.stream_ptr(self.device)))
        return self.grad_points

    def close(self):
        if self._handle:
            N.lib().qd_plan_nonuniform_destroy(self._handle)
            self._handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
