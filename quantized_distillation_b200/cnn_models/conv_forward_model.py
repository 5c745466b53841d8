"""CIFAR conv-net and the two training loops that call the quantization hot path
on every step (reference: cnn_models/conv_forward_model.py):

* ``train_model(quantizeWeights=True)`` -- quantized distillation (:165-393);
  ``train_model_quantized`` is the alias BASELINE.json's north_star names.
* ``optimize_quantization_points`` -- differentiable quantization of the
  centroids (:395-592).

Same keyword arguments and return values as the reference.  What changes is the
per-step choreography around the model forward/backward: the reference saves
``state_dict()``, rebinds every ``p.data`` to a freshly quantized tensor (about
12 launches per tensor) and copies the weights back with ``load_state_dict``;
here a :class:`QuantizationPlan` snapshots, quantizes IN PLACE and restores all
tensors with one launch each, which also keeps ``DistributedDataParallel``'s
parameter references valid.  Unlike the reference (:369-374) exceptions are not
swallowed.
"""
from __future__ import annotations

import contextlib
import copy
import time
import warnings

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F
import torch.optim as optim

from .. import quantization
from ..plan import CentroidPlan, QuantizationPlan
from . import help_fun as cnn_hf

# paper specifications (reference :30-40): teacher ~5.3 M parameters, student ~1 M
teacherModelSpec = {"spec_conv_layers": [(76, 3, 3), (76, 3, 3), (126, 3, 3), (126, 3, 3), (148, 3, 3), (148, 3, 3),
                                         (148, 3, 3), (148, 3, 3)],
                    "spec_max_pooling": [(1, 2, 2), (3, 2, 2), (7, 2, 2)],
                    "spec_dropout_rates": [(1, 0.2), (3, 0.3), (7, 0.35), (8, 0.4), (9, 0.4)],
                    "spec_linear": [1200, 1200], "width": 32, "height": 32}
smallerModelSpec = {"spec_conv_layers": [(75, 5, 5), (50, 5, 5), (50, 5, 5), (25, 5, 5)],
                    "spec_max_pooling": [(1, 2, 2), (3, 2, 2)],
                    "spec_dropout_rates": [(1, 0.2), (3, 0.3), (4, 0.4)],
                    "spec_linear": [500], "width": 32, "height": 32}


class ConvolForwardNet(nn.Module):
    """Stack of same-padded conv layers with max-pooling / dropout inserted at given
    positions, then linear layers and a 10-way output layer, ReLU everywhere
    (reference :42-163).

    The output layer is registered BEFORE the layer lists on purpose: that is the
    reference's registration order (:124-132), so ``parameters()[0]`` is
    ``out_layer.weight`` and ``quantize_first_and_last_layer=False`` skips the
    same two tensors as in the reference."""

    def __init__(self, width, height, spec_conv_layers, spec_max_pooling, spec_linear, spec_dropout_rates,
                 useBatchNorm=False, useAffineTransformInBatchNorm=False):
        super().__init__()
        self.width, self.height = width, height
        self.useBatchNorm = useBatchNorm
        convs, norms, pools, drops, linears = [], [], [], [], []
        channels = 3
        for filters, kh, kw in spec_conv_layers:
            conv = nn.Conv2d(channels, filters, kernel_size=(kh, kw), padding=((kh - 1) // 2, (kw - 1) // 2))
            nn.init.xavier_uniform_(conv.weight, nn.init.calculate_gain("conv2d"))
            convs.append(conv)
            norms.append(nn.BatchNorm2d(filters, affine=useAffineTransformInBatchNorm))
            channels = filters
        self.max_pooling_positions = [pos for pos, _, _ in spec_max_pooling]
        pools = [nn.MaxPool2d((kh, kw)) for _, kh, kw in spec_max_pooling]
        self.dropout_positions = [pos for pos, _ in spec_dropout_rates]
        drops = [nn.Dropout2d(rate) if pos < len(convs) else nn.Dropout(rate) for pos, rate in spec_dropout_rates]
        features = channels * width * height // 2 ** (2 * len(pools))
        for units in spec_linear:
            lin = nn.Linear(features, units)
            nn.init.xavier_uniform_(lin.weight, nn.init.calculate_gain("linear"))
            linears.append(lin)
            norms.append(nn.BatchNorm1d(units, affine=useAffineTransformInBatchNorm))
            features = units
        self.out_layer = nn.Linear(features, 10)
        nn.init.xavier_uniform_(self.out_layer.weight, nn.init.calculate_gain("linear"))
        self.conv_layers = nn.ModuleList(convs)
        self.max_pooling_layers = nn.ModuleList(pools)
        self.dropout_layers = nn.ModuleList(drops)
        self.linear_layers = nn.ModuleList(linears)
        self.batchNormalizationLayers = nn.ModuleList(norms)
        self.num_conv_layers = len(convs)
        self.total_num_layers = len(convs) + len(linears)

    def forward(self, x):
        for i in range(self.total_num_layers):
            if i < self.num_conv_layers:
                x = F.relu(self.conv_layers[i](x))
            else:
                if i == self.num_conv_layers:
                    x = x.view(x.size(0), -1)
                x = F.relu(self.linear_layers[i - self.num_conv_layers](x))
            if self.useBatchNorm:
                x = self.batchNormalizationLayers[i](x)
            if i in self.max_pooling_positions:
                x = self.max_pooling_layers[self.max_pooling_positions.index(i)](x)
            if i in self.dropout_positions:
                x = self.dropout_layers[self.dropout_positions.index(i)](x)
        return F.relu(self.out_layer(x))


# ------------------------------------------------------------------------------------------
# data parallelism and CUDA-graph capture of a whole step, shared by both training loops
# ------------------------------------------------------------------------------------------
def _data_parallel_module(model):
    """The wrapped network when ``model`` is a :class:`FlatDataParallel` or stock DDP wrapper, else None."""
    from ..distributed import FlatDataParallel
    if isinstance(model, (FlatDataParallel, nn.parallel.DistributedDataParallel)):
        return model.module
    return None


class _RankGroup:
    """The collectives of the data-parallel training loops, on the wrapper's process group.  Without an
    initialised process group (a wrapper built in a single process) every call is the identity."""

    def __init__(self, wrapper):
        self.group = getattr(wrapper, "process_group", None)
        self.active = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(self.group) if self.active else 1
        self.nccl = self.active and dist.get_backend(self.group) == "nccl"
        self.src = (0 if self.group is None else dist.get_global_rank(self.group, 0)) if self.active else 0

    def average(self, tensors):
        """Rank average of a list of float32 tensors with ONE all-reduce; returns views of the reduced buffer."""
        if not self.active:
            return tensors
        flat = torch.cat([t.reshape(-1) for t in tensors])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group)
        flat.mul_(1.0 / self.world)
        return [v.view(t.shape) for v, t in zip(flat.split([t.numel() for t in tensors]), tensors)]

    def check_point_counts(self, counts, device):
        """Raises ValueError on every rank unless all ranks quantize the same tensors with the same point
        counts (all-reduce MIN of (c, -c): min and max of every count at once)."""
        if not self.active:
            return
        n = torch.tensor([len(counts), -len(counts)], dtype=torch.int64, device=device)
        dist.all_reduce(n, op=dist.ReduceOp.MIN, group=self.group)
        lo, hi = n.tolist()
        if lo != -hi:
            raise ValueError(f"ranks quantize different numbers of tensors ({lo} to {-hi})")
        c = torch.tensor([int(k) for k in counts], dtype=torch.int64, device=device)
        both = torch.cat([c, -c])
        dist.all_reduce(both, op=dist.ReduceOp.MIN, group=self.group)
        lo, hi = both[:len(counts)].tolist(), [-v for v in both[len(counts):].tolist()]
        bad = [i for i, (a, b) in enumerate(zip(lo, hi)) if a != b]
        if bad:
            i = bad[0]
            raise ValueError(f"ranks chose different numbers of points for {len(bad)} tensor(s); tensor {i}: "
                             f"{lo[i]} to {hi[i]} points")

    def broadcast_buffers(self, model):
        if self.active:
            for b in model.buffers():
                dist.broadcast(b.data, self.src, group=self.group)

    def mean(self, value, device):
        if not self.active:
            return value
        t = torch.tensor([value], dtype=torch.float64, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return float(t.item()) / self.world


def _step_capturable(model, ranks, device):
    """The one rule for capturing a whole step in a CUDA graph (``ranks``: None for an unwrapped model).  Not data
    parallel (no wrapper, or no process group): always.  Data parallel: only on NCCL behind FlatDataParallel,
    whose collectives are stream-ordered device work; stock DDP (host-side reducer hooks) and gloo run eagerly."""
    from ..distributed import FlatDataParallel
    return device.type == "cuda" and (ranks is None or not ranks.active
                                      or (ranks.nccl and isinstance(model, FlatDataParallel)))


def _side_stream(device):
    """A CUDA stream, and a context that runs work on it after the current stream's work, then makes the
    current stream wait for it."""
    stream = torch.cuda.Stream(device)

    @contextlib.contextmanager
    def on_side():
        stream.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(stream):
            yield
        torch.cuda.current_stream(device).wait_stream(stream)
    return stream, on_side


def _capture(fn, device, stream=None, thread_local=False, what="the training step"):
    """``(graph, fn())`` with ``fn`` captured on ``stream``, or None after a warning when capture fails.  A step
    that holds an NCCL collective needs ``thread_local``: the NCCL watchdog thread may call CUDA meanwhile."""
    try:
        torch.cuda.synchronize(device)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream, capture_error_mode="thread_local" if thread_local else "global"):
            out = fn()
        return graph, out
    except Exception as e:                                   # pragma: no cover - depends on driver / torch build
        warnings.warn(f"CUDA graph capture of {what} failed, running eagerly: {e}")
        with contextlib.suppress(Exception):
            torch.cuda.synchronize(device)
        return None


class _CapturedStep:
    """Runs a loop's ``step(batch, idx_minibatch, epoch) -> (loss, asked, total)``, eagerly or as a CUDA graph.

    Enabled, the first three steps run eagerly on the side stream the capture uses (warm pools and workspaces);
    the fourth is captured, and every batch of the captured shapes is then copied into static buffers and
    replayed.  A batch of another shape runs eagerly and the graph is kept.  With a process group every rank
    must have captured, or all stay eager; after a failed capture the run stays eager.  ``invalidate()`` (the
    graph holds the learning rate) makes the next step capture again.  ``captured``: every rank agreed once."""

    def __init__(self, step, optimizer, device, enabled, ranks=None, static_grads=False):
        self.step, self.optimizer, self.device, self.enabled = step, optimizer, device, enabled
        self.ranks = ranks if ranks is not None and ranks.active else None
        self.static_grads = static_grads          # FlatDataParallel's gradient views: allocated once, address-stable
        self.stream, self.on_side = _side_stream(device) if enabled else (None, None)
        self.steps, self.captured = 0, False
        self.invalidate()

    def invalidate(self):
        self.graph = self.x = self.y = self.out = None

    def _try_capture(self, batch):
        x, y = batch
        self.x = torch.empty(x.shape, dtype=x.dtype, device=self.device).copy_(x, non_blocking=True)
        self.y = torch.empty(y.shape, dtype=y.dtype, device=self.device).copy_(y, non_blocking=True)
        if not self.static_grads:
            self.optimizer.zero_grad(set_to_none=True)     # gradients are re-created inside the graph's pool
        got = _capture(lambda: self.step((self.x, self.y), 1, 0), self.device, self.stream,
                       thread_local=self.ranks is not None)
        ok = got is not None
        if self.ranks is not None:                          # a replayed collective needs every peer to replay it
            flag = torch.tensor([int(ok)], dtype=torch.int32, device=self.device)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.ranks.group)
            ok = bool(flag.item())
        if ok:
            self.graph, self.out = got
            self.captured = True
        else:
            self.invalidate()
            self.enabled = False

    def run(self, batch, idx_minibatch, epoch):
        if self.enabled and self.graph is None and self.steps >= 3:
            self._try_capture(batch)
        self.steps += 1
        if self.graph is not None and batch[0].shape == self.x.shape and batch[1].shape == self.y.shape:
            self.x.copy_(batch[0], non_blocking=True)
            self.y.copy_(batch[1], non_blocking=True)
            self.graph.replay()
            return self.out
        if not self.enabled:
            return self.step(batch, idx_minibatch, epoch)
        with self.on_side():
            return self.step(batch, idx_minibatch, epoch)


def _set_learning_rate(optimizers, lr, runner):
    """Sets ``lr`` in every parameter group; a change invalidates the captured step, which holds the old rate."""
    for opt in optimizers:
        for group in opt.param_groups:
            if group["lr"] != lr:
                runner.invalidate()
            group["lr"] = lr


# ------------------------------------------------------------------------------------------
# quantized distillation
# ------------------------------------------------------------------------------------------
def _selected_parameters(model, quantize_first_and_last_layer):
    params = list(model.parameters())
    if quantize_first_and_last_layer is False:
        params = params[1:-1]                                             # reference :237-239
    return params


def _uniform_levels(quantizationFunctionToUse, numBits):
    name = quantizationFunctionToUse.lower()
    if name == "uniformAbsMaxScaling".lower():
        return 2 ** (numBits - 1), "absmax"                               # reference :206-208 (broken scaling there)
    if name == "uniformLinearScaling".lower():
        return 2 ** numBits, "linear"                                     # reference :209-211
    raise ValueError("The specified quantization function is not present")


class WeightQuantizer:
    """``quantize_weights_model`` / ``backward_quant_weights_model`` of the reference
    (closures at :235-266) lifted to an object that owns the multi-tensor plan."""

    def __init__(self, model, numBits, bucket_size, quantizationFunctionToUse="uniformLinearScaling",
                 backprop_quantization_style="none", quantize_first_and_last_layer=True, *, stochastic_rounding=False,
                 max_element=False, subtract_mean=False):
        style = "none" if backprop_quantization_style is None else backprop_quantization_style.lower()
        if style not in ("none", "truncated", "complicated"):
            raise ValueError("The specified backprop_quantization_style not recognized")
        self.style = style
        self.s, self.scaling = _uniform_levels(quantizationFunctionToUse, numBits)
        self.bucket_size = bucket_size
        self.params = _selected_parameters(model, quantize_first_and_last_layer)
        # the options only the NMT loop passes (translation_models/model.py:162-164, 198-204: stochasticRounding,
        # maxElementAllowedForQuantization, subtractMeanInQuantization); the multi-tensor plan is the plain
        # deterministic op, so any of them selects the per-tensor fused kernel, which implements all three
        self.options = {"stochastic_rounding": bool(stochastic_rounding), "max_element": max_element,
                        "subtract_mean": bool(subtract_mean)}
        extra = self.options["stochastic_rounding"] or max_element is not False or self.options["subtract_mean"]
        if extra and self.scaling == "linear":
            if style == "complicated":
                # reference: backward raises for subtract_mean (quant_functions.py:329-330) and re-runs its forward with
                # max_element / stochastic rounding (:341-347), which the backward kernel does not take
                raise NotImplementedError("backprop_quantization_style 'complicated' is not available together with "
                                          "stochastic_rounding / max_element / subtract_mean")
            self.plan = None
            self._master = [torch.empty_like(p.data) for p in self.params]
            return
        if self.scaling != "linear":
            # 'uniformAbsMaxScaling' (:206-208) cannot execute in the reference; the intended semantics are an opt-in
            # extension without a parity target (quantization.quant_functions.ALLOW_UNPINNED_SCALING), per tensor
            if not quantization.quant_functions.ALLOW_UNPINNED_SCALING:
                raise NotImplementedError("absmax scaling does not execute in the reference (quant_functions.py:119-126); "
                                          "set quantization.quant_functions.ALLOW_UNPINNED_SCALING = True for the extension")
            if style == "complicated":
                raise ValueError("Linear scaling is necessary to backpropagate")              # quant_functions.py:326-327
            self.plan = None
            self._master = [torch.empty_like(p.data) for p in self.params]
            return
        self.plan = QuantizationPlan(self.params, self.s, bucket_size)

    def quantize_weights_model(self, save=True):
        """fp32 weights -> shadow buffer, then every tensor quantized in place."""
        if self.style == "truncated":
            torch._foreach_clamp_min_([p.data for p in self.params], -1.0)   # p.data.clamp_(-1, 1), reference :240-241
            torch._foreach_clamp_max_([p.data for p in self.params], 1.0)
        if self.plan is None:                                  # NMT-loop options / absmax extension: one fused launch per tensor
            if save:
                torch._foreach_copy_(self._master, [p.data for p in self.params])
            for p in self.params:
                quantization.uniformQuantization(p.data, self.s, type_of_scaling=self.scaling, bucket_size=self.bucket_size,
                                                 modify_in_place=True, **self.options)
            return
        if save:
            self.plan.save_and_quantize_()          # shadow copy + in-place quantization, one launch
        else:
            self.plan.quantize_()

    def restore_weights_model(self):
        if self.plan is None:
            torch._foreach_copy_([p.data for p in self.params], self._master)
            return
        self.plan.restore_master()

    def backward_quant_weights_model(self):
        if self.style == "none":
            return
        if self.plan is None:                                                 # 'truncated' is scaling-agnostic (:263-264)
            for p in self.params:
                p.grad.data.masked_fill_(p.data.abs() > 1, 0.0)
            return
        grads = []
        for p in self.params:
            if p.grad is None:
                raise ValueError("backward_quant_weights_model needs gradients on every quantized parameter")
            grads.append(p.grad.data if p.grad.is_contiguous() else p.grad.data.contiguous())
        self.plan.backward_(grads, self.style)
        for p, g in zip(self.params, grads):
            if g.data_ptr() != p.grad.data_ptr():
                p.grad.data.copy_(g)


def quantize_weights_model(model, numBits, bucket_size=None, quantize_first_and_last_layer=True):
    """One-shot post-training quantization of a model's weights, in place
    (what the drivers do tensor by tensor, cifar10_test.py:312-317)."""
    WeightQuantizer(model, numBits, bucket_size, quantize_first_and_last_layer=quantize_first_and_last_layer) \
        .quantize_weights_model(save=False)
    return model


def train_model(model, train_loader, test_loader, initial_learning_rate=0.001, use_nesterov=True,
                initial_momentum=0.9, weight_decayL2=0.00022, epochs_to_train=100, print_every=500,
                learning_rate_style="generic", use_distillation_loss=False, teacher_model=None,
                quantizeWeights=False, numBits=8, grad_clipping_threshold=False, start_epoch=0,
                bucket_size=None, quantizationFunctionToUse="uniformLinearScaling",
                backprop_quantization_style="none", estimate_quant_grad_every=1, add_gradient_noise=False,
                ask_teacher_strategy=("always", None), quantize_first_and_last_layer=True,
                mix_with_differentiable_quantization=False, *, max_steps=None, verbose=True, evaluate=True,
                step_hook=None, cuda_graph_step=False, fused_optimizer_step=False):
    """SGD training with optional distillation loss and optional per-step weight
    quantization (reference :165-393; same positional/keyword arguments, the
    keyword-only ones after ``*`` are additions).

    ``cuda_graph_step=True`` (``ask_teacher_strategy`` 'always', ``estimate_quant_grad_every`` 1, no gradient
    noise; data parallel only on NCCL behind ``FlatDataParallel``): after three eager steps the whole step --
    save+quantize, student/teacher forward, backward, all-reduce, restore, gradient fix-up, SGD update -- is
    captured once in a CUDA graph and replayed (:class:`_CapturedStep`); each step then costs one H2D copy of
    the batch and one graph launch.  Same arithmetic, same kernels; the graph is re-captured when the learning
    rate changes.  ``informationDict["cuda_graph_step"]``: every rank captured the step at least once.

    ``fused_optimizer_step=True`` (quantized training, bucket of at most 512, no gradient noise /
    clipping): restore, gradient fix-up, the SGD update and the NEXT step's save-and-quantize become
    one kernel over the quantized tensors (``QuantizationPlan.fused_step_``, 24 instead of 52 bytes
    per weight); the live parameters then always hold the quantized weights and the full-precision
    ones live in the plan's master buffer.  Same arithmetic as ``torch.optim.SGD`` + the unfused ops."""
    if use_distillation_loss is True and teacher_model is None:
        raise ValueError("To compute distillation loss you have to pass the teacher model")
    if teacher_model is not None:
        teacher_model.eval()
    learning_rate_style = learning_rate_style.lower()
    lr_scheduler = cnn_hf.LearningRateScheduler(initial_learning_rate, learning_rate_style)
    new_learning_rate = initial_learning_rate
    optimizer = optim.SGD(model.parameters(), lr=initial_learning_rate, nesterov=use_nesterov, momentum=initial_momentum,
                          weight_decay=weight_decayL2)
    start_time = time.time()
    pred_accuracy_epochs, percentages_asked_teacher, losses_epochs = [], [], []
    informationDict = {}
    last_loss_saved = float("inf")
    steps_since_estimate = 1
    batches_per_epoch = len(train_loader)
    quantizer = None
    if quantizeWeights:
        quantizer = WeightQuantizer(model, numBits, bucket_size, quantizationFunctionToUse, backprop_quantization_style,
                                    quantize_first_and_last_layer)
    if print_every > batches_per_epoch:
        print_every = max(batches_per_epoch // 2, 1)
    total_steps = 0
    stop = False
    epoch = start_epoch
    device = cnn_hf._device_of(model)
    state = {"since": steps_since_estimate}
    # data parallelism: FlatDataParallel exposes reduce_gradients(); DDP reduces inside backward
    reduce_gradients = getattr(model, "reduce_gradients", None)

    fused = bool(fused_optimizer_step and quantizer is not None and device.type == "cuda" and estimate_quant_grad_every == 1
                 and not add_gradient_noise and grad_clipping_threshold is False
                 and bucket_size is not None and bucket_size <= 512 and quantizer.plan is not None)
    rest_optimizer = None
    if fused:
        chosen = {id(p) for p in quantizer.params}
        rest = [p for p in model.parameters() if id(p) not in chosen]      # e.g. first / last layer left unquantized
        if rest:
            rest_optimizer = optim.SGD(rest, lr=initial_learning_rate, nesterov=use_nesterov, momentum=initial_momentum,
                                       weight_decay=weight_decayL2)
        state["lr"] = initial_learning_rate
        quantizer.quantize_weights_model()                                 # master <- weights, live <- quantized, once

    def fused_step(data, idx_minibatch=1, epoch=0):
        """The same step with the tail fused: live parameters are already quantized on entry."""
        model.zero_grad(set_to_none=False)
        loss, c_teach, c_total = cnn_hf.forward_and_backward(
            model, data, idx_minibatch, epoch, use_distillation_loss=use_distillation_loss, teacher_model=teacher_model,
            ask_teacher_strategy=ask_teacher_strategy, return_more_info=True, return_tensor=True)
        if reduce_gradients is not None:
            reduce_gradients()
        grads = []
        for p in quantizer.params:
            if p.grad is None:
                raise ValueError("every quantized parameter needs a gradient")
            if not p.grad.is_contiguous():
                p.grad = p.grad.contiguous()
            grads.append(p.grad.data)
        quantizer.plan.fused_step_(grads, quantizer.style, state["lr"], initial_momentum, weight_decayL2, use_nesterov)
        if rest_optimizer is not None:
            rest_optimizer.step()
        return loss, c_teach, c_total

    def one_step(data, idx_minibatch=1, epoch=0):
        """One training step of the reference loop (:280-322) on one batch."""
        if fused:
            return fused_step(data, idx_minibatch, epoch)
        quantize_now = quantizer is not None and state["since"] >= estimate_quant_grad_every
        if quantize_now:
            quantizer.quantize_weights_model()                            # :286-287
        model.zero_grad(set_to_none=False)
        loss, c_teach, c_total = cnn_hf.forward_and_backward(
            model, data, idx_minibatch, epoch, use_distillation_loss=use_distillation_loss, teacher_model=teacher_model,
            ask_teacher_strategy=ask_teacher_strategy, return_more_info=True, return_tensor=True)
        if reduce_gradients is not None:
            reduce_gradients()                                            # ONE all-reduce of the flat gradient buffer
        if quantize_now:
            quantizer.restore_weights_model()                             # :302
        if add_gradient_noise and not quantizeWeights:
            cnn_hf.add_gradient_noise(model, idx_minibatch, epoch, batches_per_epoch)
        if grad_clipping_threshold is not False:
            for p in model.parameters():
                if p.grad is not None:
                    p.grad.clamp_(-grad_clipping_threshold, grad_clipping_threshold)
        if quantize_now:
            quantizer.backward_quant_weights_model()                      # :315
        optimizer.step()
        if state["since"] >= estimate_quant_grad_every:
            state["since"] = 0
        state["since"] += 1
        return loss, c_teach, c_total

    strategy_name = (ask_teacher_strategy[0] if isinstance(ask_teacher_strategy, tuple) else ask_teacher_strategy).lower()
    ranks = _RankGroup(model) if _data_parallel_module(model) is not None else None
    runner = _CapturedStep(one_step, optimizer, device, static_grads=reduce_gradients is not None, ranks=ranks, enabled=bool(
        cuda_graph_step and estimate_quant_grad_every == 1 and not add_gradient_noise and strategy_name == "always"
        and _step_capturable(model, ranks, device)))
    try:
        for epoch in range(start_epoch, epochs_to_train + start_epoch):
            model.train()
            running = torch.zeros((), device=cnn_hf._device_of(model))
            asked, seen = 0, 0
            for idx_minibatch, data in enumerate(train_loader, start=1):
                loss, c_teach, c_total = runner.run(data, idx_minibatch, epoch)
                asked += c_teach
                seen += c_total
                running += loss
                total_steps += 1
                if step_hook is not None:
                    step_hook(total_steps, loss)
                if idx_minibatch % print_every == 0:
                    last_loss_saved = float(running.item()) / print_every
                    running.zero_()
                    if verbose:
                        msg = "Time Elapsed: {:.1f}s, [Start Epoch: {}, Epoch: {}, Minibatch: {}], loss: {:3f}".format(
                            time.time() - start_time, start_epoch + 1, epoch + 1, idx_minibatch, last_loss_saved)
                        if pred_accuracy_epochs:
                            msg += " Last prediction accuracy: {:2f}%".format(pred_accuracy_epochs[-1] * 100)
                        print(msg)
                if max_steps is not None and total_steps >= max_steps:
                    stop = True
                    break
            percentages_asked_teacher.append(asked / seen if seen else 0)
            losses_epochs.append(last_loss_saved)
            if evaluate:
                pred_accuracy_epochs.append(cnn_hf.evaluateModel(model, test_loader, fastEvaluation=False))
                if verbose:
                    print(" === Epoch: {} - prediction accuracy {:2f}% === ".format(epoch + 1, pred_accuracy_epochs[-1] * 100))
            if stop:
                break
            if mix_with_differentiable_quantization and epoch != start_epoch + epochs_to_train - 1:
                # the differentiable step works on a copy and hands back its state dict (reference :342-353)
                quantized_state_dict = optimize_quantization_points(
                    model, train_loader, test_loader, new_learning_rate, initial_momentum=initial_momentum,
                    epochs_to_train=1, print_every=print_every, use_nesterov=use_nesterov,
                    learning_rate_style=learning_rate_style, numPointsPerTensor=2 ** numBits,
                    assignBitsAutomatically=True, bucket_size=bucket_size, use_distillation_loss=True,
                    initialize_method="quantiles", quantize_first_and_last_layer=quantize_first_and_last_layer,
                    verbose=verbose, evaluate=evaluate, max_steps=max_steps)[0]
                inner = _data_parallel_module(model)                       # wrapped: unprefixed keys of the network
                (model if inner is None else inner).load_state_dict(quantized_state_dict)
                if fused:
                    quantizer.quantize_weights_model()                     # master <- the loaded weights, live <- quantized
                losses_epochs.append(last_loss_saved)
                if evaluate:
                    pred_accuracy_epochs.append(cnn_hf.evaluateModel(model, test_loader, fastEvaluation=False))
            error = 1 - pred_accuracy_epochs[-1] if pred_accuracy_epochs else 1.0
            new_learning_rate, stop_training = lr_scheduler.update_learning_rate(epoch, error)
            if stop_training is True:
                break
            _set_learning_rate([opt for opt in (optimizer, rest_optimizer) if opt is not None], new_learning_rate, runner)
            state["lr"] = new_learning_rate
    except KeyboardInterrupt:
        informationDict["errorFlag"] = False
        informationDict["numEpochsTrained"] = epoch - start_epoch
    else:
        informationDict["errorFlag"] = False
        informationDict["numEpochsTrained"] = epoch + 1 - start_epoch
    if quantizer is not None and not fused:                                # (fused: the live weights already are)
        quantizer.quantize_weights_model(save=False)                       # final weights are returned quantized (:384-385)
    informationDict["fused_optimizer_step"] = fused
    informationDict["cuda_graph_step"] = runner.captured
    if mix_with_differentiable_quantization:
        informationDict["numEpochsTrained"] *= 2
    informationDict["percentages_asked_teacher"] = percentages_asked_teacher
    informationDict["predictionAccuracy"] = pred_accuracy_epochs
    informationDict["lossSaved"] = losses_epochs
    informationDict["numStepsTrained"] = total_steps
    return model, informationDict


def train_model_quantized(model, train_loader, test_loader, numBits=8, bucket_size=None, **kwargs):
    """``train_model(..., quantizeWeights=True)``: the entry point BASELINE.json's
    north_star names (the reference spells it through the ``quantizeWeights`` flag)."""
    return train_model(model, train_loader, test_loader, quantizeWeights=True, numBits=numBits, bucket_size=bucket_size,
                       **kwargs)


# ------------------------------------------------------------------------------------------
# differentiable quantization
# ------------------------------------------------------------------------------------------
def _capture_point_graphs(quantize_all, point_gradients, device):
    """Captures the two per-step launch sequences of the differentiable-quantization loop.
    Returns (forward_graph, backward_graph, gradient tensors), or None when capture fails."""
    _, on_side = _side_stream(device)
    with on_side():                                          # warm the capture stream's workspace / caches
        quantize_all()
        point_gradients()
    fwd = _capture(quantize_all, device, what="the quantization step")
    bwd = fwd and _capture(point_gradients, device, what="the quantization step")
    return (fwd[0], bwd[0], bwd[1]) if bwd else None


def optimize_quantization_points(modelToQuantize, train_loader, test_loader, initial_learning_rate=1e-5,
                                 initial_momentum=0.9, epochs_to_train=30, print_every=500, use_nesterov=True,
                                 learning_rate_style="generic", numPointsPerTensor=16, assignBitsAutomatically=False,
                                 bucket_size=None, use_distillation_loss=True, initialize_method="quantiles",
                                 quantize_first_and_last_layer=True, *, max_steps=None, verbose=True, evaluate=True,
                                 step_hook=None, use_cuda_graphs=True, cuda_graph_step=False, use_plan=True):
    """Learn the quantization points of every tensor by SGD on the loss of the
    quantized network, the unquantized network acting as teacher (reference
    :395-592).  Returns ``(quantizedModel.state_dict(), pointsPerTensor, informationDict)``.

    Data parallel: pass the :class:`FlatDataParallel` or DDP wrapper (one process per GPU, each with its
    shard of every batch).  The quantized copy is built from the wrapped network and is not wrapped; per
    step the ranks reduce only the centroid gradients, as float64 sums with ONE all-reduce of a
    ``(tensors x 32)`` table, and round them to float32 once, so points, quantized weights and the
    returned (unprefixed) state dict are bit-identical on every rank.  ``assignBitsAutomatically`` uses the
    rank-averaged gradients; the point counts are checked to agree across ranks (``ValueError`` otherwise).
    Batch-norm buffers of the quantized copy are broadcast from rank 0 before each evaluation and before
    returning, and the evaluated accuracy is the mean over ranks.  ``cuda_graph_step=True`` captures the
    step with its collective on NCCL with ``FlatDataParallel``; stock DDP and gloo run eagerly."""
    dp_net = _data_parallel_module(modelToQuantize)
    dp = dp_net is not None
    ranks = _RankGroup(modelToQuantize) if dp else None
    net = dp_net if dp else modelToQuantize          # the network itself: teacher and source of the quantized copy
    numTensorsNetwork = sum(1 for _ in modelToQuantize.parameters())
    initialize_method = initialize_method.lower()
    if initialize_method not in ("quantiles", "uniform"):
        raise ValueError("The initialization method must be either quantiles or uniform")
    if isinstance(numPointsPerTensor, int):
        numPointsPerTensor = [numPointsPerTensor] * numTensorsNetwork
    if len(numPointsPerTensor) != numTensorsNetwork:
        raise ValueError("numPointsPerTensor must be equal to the number of tensor in the network")
    if quantize_first_and_last_layer is False:
        numPointsPerTensor = numPointsPerTensor[1:-1]
    device = cnn_hf._device_of(modelToQuantize)
    scalingFunction = quantization.ScalingFunction("linear", False, False, bucket_size, False)     # :420

    if assignBitsAutomatically:                                             # :424-448
        num_to_estimate_grad = 5
        modelToQuantize.zero_grad()
        with (modelToQuantize.no_sync() if dp else contextlib.nullcontext()):     # data parallel: accumulate locally
            for idx_minibatch, batch in enumerate(train_loader, start=1):
                cnn_hf.forward_and_backward(modelToQuantize, batch, idx_batch=idx_minibatch, epoch=0,
                                            use_distillation_loss=False, return_tensor=True)
                if idx_minibatch >= num_to_estimate_grad:
                    break
        # ||grad / num||_2 of every selected tensor: one multi-tensor launch, one device->host copy
        sel_grads = [p.grad for p in _selected_parameters(modelToQuantize, quantize_first_and_last_layer)]
        if dp:
            sel_grads = ranks.average(sel_grads)          # every rank takes the norms of the same averaged gradients
        norms = (quantization.help_functions.gradient_norms(sel_grads) / num_to_estimate_grad).tolist()
        modelToQuantize.zero_grad()
        numPointsPerTensor = quantization.help_functions.assign_bits_automatically(norms, numPointsPerTensor,
                                                                                   input_is_point=True)
    if dp:
        ranks.check_point_counts(numPointsPerTensor, device)     # before anything is sized by the counts

    selected = _selected_parameters(modelToQuantize, quantize_first_and_last_layer)
    pointsPerTensor = []
    # every tensor's points are a row of ONE (tensors x width) table padded with +inf, so that the
    # per-step re-sort of all lists (:550-551) is one torch.sort instead of one per tensor
    width = max(int(num) for num in numPointsPerTensor)
    points_table = torch.full((len(selected), width), float("inf"), dtype=torch.float32, device=device)
    for row, (p, num) in enumerate(zip(selected, numPointsPerTensor)):       # :451-482
        if initialize_method == "quantiles":
            init = quantization.help_functions.initialize_quantization_points(p.data, scalingFunction, num)
        else:
            init = torch.tensor([x / (num - 1) for x in range(num)], dtype=torch.float32, device=device)
        points_table[row, :num] = init.to(device)
        init = points_table[row, :num].detach().requires_grad_(True)         # leaf tensor sharing the table's storage
        init.grad = torch.zeros_like(init)
        pointsPerTensor.append(init)

    options = {"momentum": initial_momentum, "nesterov": use_nesterov} if initial_momentum != 0 else {}
    optimizer = optim.SGD(pointsPerTensor, lr=initial_learning_rate, **options)
    lr_scheduler = cnn_hf.LearningRateScheduler(initial_learning_rate, learning_rate_style)
    start_time = time.time()
    pred_accuracy_epochs, losses_epochs = [], []
    last_loss_saved = float("inf")
    batches_per_epoch = len(train_loader)
    if print_every > batches_per_epoch:
        print_every = max(batches_per_epoch // 2, 1)

    modelToQuantize.eval()
    quantizedModel = copy.deepcopy(net)                                       # :497-498
    q_selected = _selected_parameters(quantizedModel, quantize_first_and_last_layer)
    quantizationFunctions = [quantization.nonUniformQuantization_variable(
        max_element=False, subtract_mean=False, modify_in_place=False, bucket_size=bucket_size,
        pre_process_tensors=True, tensor=p.data) for p in q_selected]         # :501-511

    # Multi-tensor plan: ONE launch quantizes every tensor with its current points, TWO produce every
    # centroid gradient (3 launches per step instead of 3 per tensor).  More than 32 points per tensor
    # or rows longer than 1024 elements: per-tensor ops (NotImplementedError from the plan).
    plan = None
    if use_plan and device.type == "cuda":
        try:
            plan = CentroidPlan([fun._tensor for fun in quantizationFunctions], [p.data for p in q_selected],
                                [pts.data for pts in pointsPerTensor], bucket_size)
        except NotImplementedError:
            plan = None
    # data parallel: the float64 centroid-gradient sums of every tensor, reduced in place across ranks each step
    sums = torch.zeros((len(q_selected), CentroidPlan.MAX_POINTS), dtype=torch.float64, device=device) \
        if (dp and plan is not None) else None

    def quantize_all():                                                       # :525-532
        if plan is not None:
            plan.forward_()
            return
        for fun, p_q, pts in zip(quantizationFunctions, q_selected, pointsPerTensor):
            fun.forward(None, pts.data, out=p_q.data)

    def point_gradients():                                                    # :539-545
        if plan is not None:
            q_grads = [p_q.grad.data if p_q.grad.is_contiguous() else p_q.grad.data.contiguous() for p_q in q_selected]
            if sums is not None:              # global-batch gradient = rank average; rounded to float32 once, after the sum
                plan.backward_partial_(q_grads, sums)
                if ranks.active:
                    dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=ranks.group)
                return plan.finish_(sums, 1.0 / ranks.world)
            return plan.backward_(q_grads)
        return [fun.backward(p_q.grad.data)[1] for fun, p_q in zip(quantizationFunctions, q_selected)]

    # Without the plan the per-step quantization work is 3 small launches per tensor (22-60 tensors),
    # launch bound: after two eager steps the forward and the backward sequences are each captured
    # into a CUDA graph and replayed with one call per step.
    graphs = None
    graph_after = 2 if (use_cuda_graphs and plan is None and device.type == "cuda" and not cuda_graph_step) else None

    def one_step(data, idx_minibatch=1, epoch=0):
        """One step of the reference loop (:518-551)."""
        nonlocal graphs, graph_after
        quantizedModel.zero_grad(set_to_none=False)
        optimizer.zero_grad(set_to_none=False)
        if graphs is None and graph_after is not None and total_steps >= graph_after:
            graphs = _capture_point_graphs(quantize_all, point_gradients, device)
            if graphs is None:
                graph_after = None                                        # capture unavailable: stay eager
        if graphs:
            graphs[0].replay()
        else:
            quantize_all()
        loss = cnn_hf.forward_and_backward(quantizedModel, data, idx_minibatch, epoch,
                                           use_distillation_loss=use_distillation_loss, teacher_model=net,
                                           return_tensor=True)
        if graphs:
            graphs[1].replay()
            grads = graphs[2]
        else:
            grads = point_gradients()
        if dp and plan is None:                   # per-tensor fallback: its float32 gradients, ONE all-reduce (average)
            grads = ranks.average(grads)
        for pts, gp in zip(pointsPerTensor, grads):
            pts.grad = gp
        optimizer.step()
        points_table.copy_(torch.sort(points_table, dim=1)[0])            # :550-551, every list at once, in place
        return loss, 0, 0

    runner = _CapturedStep(one_step, optimizer, device, ranks=ranks,
                           enabled=bool(cuda_graph_step and _step_capturable(modelToQuantize, ranks, device)))

    total_steps, epoch, stop = 0, 0, False
    for epoch in range(epochs_to_train):
        quantizedModel.train()
        running = torch.zeros((), device=device)
        for idx_minibatch, data in enumerate(train_loader, start=1):
            loss = runner.run(data, idx_minibatch, epoch)[0]
            running += loss
            total_steps += 1
            if step_hook is not None:
                step_hook(total_steps, loss)
            if idx_minibatch % print_every == 0:
                last_loss_saved = float(running.item()) / print_every
                running.zero_()
                if verbose:
                    print("Time Elapsed: {:.1f}s, [Epoch: {}, Minibatch: {}], loss: {:3f}".format(
                        time.time() - start_time, epoch + 1, idx_minibatch, last_loss_saved))
            if max_steps is not None and total_steps >= max_steps:
                stop = True
                break
        losses_epochs.append(last_loss_saved)
        if evaluate:
            if dp:
                ranks.broadcast_buffers(quantizedModel)                    # every rank evaluates rank 0's statistics
            accuracy = cnn_hf.evaluateModel(quantizedModel, test_loader, fastEvaluation=False)
            # data parallel: one accuracy for all ranks, so that they take the same learning-rate decisions
            pred_accuracy_epochs.append(ranks.mean(accuracy, device) if dp else accuracy)
            if verbose:
                print(" === Epoch: {} - prediction accuracy {:2f}% === ".format(epoch + 1, pred_accuracy_epochs[-1] * 100))
        if stop:
            break
        error = 1 - pred_accuracy_epochs[-1] if pred_accuracy_epochs else 1.0
        new_learning_rate, stop_training = lr_scheduler.update_learning_rate(epoch, error)
        if stop_training is True:
            break
        _set_learning_rate([optimizer], new_learning_rate, runner)
    informationDict = {"predictionAccuracy": pred_accuracy_epochs, "numEpochsTrained": epoch + 1,
                       "lossSaved": losses_epochs, "numStepsTrained": total_steps,
                       "cuda_graph_step": runner.captured, "cuda_graph_quantization": bool(graphs),
                       "multi_tensor_plan": plan is not None}
    if dp:
        informationDict["data_parallel_world"] = ranks.world
        ranks.broadcast_buffers(quantizedModel)                            # one state dict on every rank
    # the state dict also carries the batch-norm running statistics of the quantized model (:579-592)
    return quantizedModel.state_dict(), pointsPerTensor, informationDict
