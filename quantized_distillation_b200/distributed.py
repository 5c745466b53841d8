"""Data-parallel plumbing: one process per GPU, NCCL gradient all-reduce over NVLink /
NVSwitch (SURVEY.md section 8e).

Two wrappers:

* :class:`FlatDataParallel` (default of ``wrap_data_parallel``) -- every gradient is a view into
  ONE flat float32 buffer (mirrors ``QuantizationPlan._master_flat``), the step issues ONE
  all-reduce on it, and nothing in it is host-driven (no reducer hooks, no bucket bookkeeping),
  so the whole training step -- quantize, forward/backward, all-reduce, restore, gradient
  fix-up, SGD -- can be captured in one CUDA graph and replayed (NCCL collectives are
  capturable).  This is what makes the 1 -> 8 GPU curve of the launch-bound student scale.
* ``wrap_ddp`` -- stock ``DistributedDataParallel`` (bucketed all-reduce overlapped with the
  backward, eager only); kept for comparison and for models whose backward is long enough to
  hide the collective.

The reference's multi-GPU story is single-process ``nn.DataParallel``
(cifar10_wideResNet.py:68-69, 97, 117); the quantization op itself needs no
collective -- every rank quantizes its full replica, and because the kernels are
deterministic the replicas stay bit-identical.  The only collective in a step is
DDP's bucketed gradient all-reduce, overlapped with backward.  The gradient
fix-up kernels run after it, on the already reduced gradients, like the reference
runs them on its single reduced copy (conv_forward_model.py:315)."""
from __future__ import annotations

import contextlib
import os
from collections import OrderedDict

import torch
import torch.distributed as dist


def env_world():
    return int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))


def init_distributed(backend=None):
    """Initialises the default process group from the torchrun environment.
    Returns (world, rank, device)."""
    world, rank, local_rank = env_world()
    use_cuda = torch.cuda.is_available()
    if use_cuda:
        torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank) if use_cuda else torch.device("cpu")
    if world > 1 and not dist.is_initialized():
        backend = backend or ("nccl" if use_cuda else "gloo")
        kwargs = {"device_id": device} if backend == "nccl" else {}
        dist.init_process_group(backend, **kwargs)
    return world, rank, device


def wrap_ddp(model, device):
    """DDP wrapper.  Parameters are only ever modified IN PLACE by the quantization
    plan, so the parameter objects DDP registered its hooks on stay the live ones."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return model
    from torch.nn.parallel import DistributedDataParallel as DDP
    if device.type == "cuda":
        return DDP(model, device_ids=[device.index], output_device=device.index, broadcast_buffers=True,
                   gradient_as_bucket_view=True)
    return DDP(model)


class FlatDataParallel(torch.nn.Module):
    """Replicated module whose gradients live in one flat buffer reduced by one collective per BUCKET.

    ``p.grad`` of every trainable parameter is a view of ``flat_grad`` (each tensor starts on a
    256-byte boundary, so the plan's 128-bit gradient fix-up kernels apply).  Autograd accumulates
    in place into an existing ``.grad``, ``zero_grad`` is one memset.  The buffer is cut into
    contiguous buckets of about ``bucket_mb`` (one bucket when the model is smaller: the 4 MB
    student).  With several buckets, each bucket's all-reduce (AVG on NCCL; SUM then scale on gloo)
    is issued on a communication stream as soon as the last gradient of the bucket has been
    accumulated (post-accumulate-grad hooks), so it overlaps the rest of the backward pass;
    ``reduce_gradients()`` issues whatever is still pending and joins the stream.  All of it is
    stream-ordered device work, so the whole training step -- collectives included -- can still be
    captured in ONE CUDA graph (the side stream forks from and joins the capturing stream).
    Parameters and buffers are broadcast from rank 0 once at construction; batch-norm statistics
    stay replica-local afterwards (the reference's ``nn.DataParallel`` keeps only replica 0's,
    cifar10_wideResNet.py:68-69)."""

    def __init__(self, module, process_group=None, bucket_mb=32.0):
        super().__init__()
        self.module = module
        self.process_group = process_group
        self.world = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
        params = [p for p in module.parameters() if p.requires_grad]
        if not params:
            raise ValueError("module has no trainable parameters")
        if self.world > 1:
            with torch.no_grad():
                for t in list(module.parameters()) + list(module.buffers()):
                    dist.broadcast(t.data, 0, group=process_group)
        device, dtype = params[0].device, params[0].dtype
        pad = lambda n: -(-n // 64) * 64                                  # 256-byte granules
        self.flat_grad = torch.zeros(sum(pad(p.numel()) for p in params), dtype=dtype, device=device)
        off, spans = 0, []
        for p in params:
            if p.device != device or p.dtype != dtype or not p.is_contiguous():
                raise ValueError("FlatDataParallel needs contiguous parameters of one dtype on one device")
            p.grad = self.flat_grad[off:off + p.numel()].view(p.shape)
            spans.append((off, off + pad(p.numel())))
            off += pad(p.numel())
        self._params = params
        self._paused = False
        self._nccl = self.world > 1 and dist.get_backend(process_group) == "nccl"
        # buckets: contiguous runs of parameters, in registration order, of >= bucket_mb each
        limit = int(bucket_mb * (1 << 20) / self.flat_grad.element_size())
        self._buckets, start, members = [], 0, []
        for i, (lo, hi) in enumerate(spans):
            members.append(i)
            if hi - start >= limit or i == len(spans) - 1:
                self._buckets.append({"lo": start, "hi": hi, "members": members, "pending": len(members), "sent": False})
                start, members = hi, []
        self._bucket_of = {}
        for b, bucket in enumerate(self._buckets):
            for i in bucket["members"]:
                self._bucket_of[i] = b
        # several buckets: each one is reduced from the backward pass as soon as it is complete (on a side stream on CUDA)
        self._early = self.world > 1 and len(self._buckets) > 1
        self._comm_stream = torch.cuda.Stream(device) if (self._early and device.type == "cuda") else None
        if self._early:
            for i, p in enumerate(params):
                p.register_post_accumulate_grad_hook(self._make_hook(i))

    # ---- bucketed, overlapped reduction ---------------------------------------------------------
    def _make_hook(self, index):
        def hook(_param):
            if self._paused:
                return
            bucket = self._buckets[self._bucket_of[index]]
            bucket["pending"] -= 1
            if bucket["pending"] == 0 and not bucket["sent"]:
                self._send(bucket)
        return hook

    def _all_reduce(self, view):
        if self._nccl:
            dist.all_reduce(view, op=dist.ReduceOp.AVG, group=self.process_group)
        else:
            dist.all_reduce(view, op=dist.ReduceOp.SUM, group=self.process_group)
            view.mul_(1.0 / self.world)

    def _send(self, bucket):
        bucket["sent"] = True
        view = self.flat_grad[bucket["lo"]:bucket["hi"]]
        if self._comm_stream is None:
            self._all_reduce(view)
            return
        self._comm_stream.wait_stream(torch.cuda.current_stream(self.flat_grad.device))   # the bucket's gradients are complete
        with torch.cuda.stream(self._comm_stream):
            self._all_reduce(view)

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def zero_grad(self, set_to_none: bool = False):
        """One memset; the views stay bound whatever ``set_to_none`` says (a ``None`` gradient
        would make autograd allocate a fresh tensor outside the flat buffer)."""
        self.flat_grad.zero_()
        for bucket in self._buckets:
            bucket["pending"], bucket["sent"] = len(bucket["members"]), False

    @contextlib.contextmanager
    def no_sync(self):
        """Backward passes inside the block accumulate into the flat buffer without any reduction, like
        DDP's ``no_sync()``; the caller reduces what it needs afterwards.  Every bucket is re-armed on exit."""
        self._paused = True
        try:
            yield
        finally:
            self._paused = False
            for bucket in self._buckets:
                bucket["pending"], bucket["sent"] = len(bucket["members"]), False

    def views_intact(self) -> bool:
        """True while every ``p.grad`` still aliases the flat buffer (an optimizer's
        ``zero_grad(set_to_none=True)`` would break that)."""
        lo = self.flat_grad.data_ptr()
        hi = lo + self.flat_grad.numel() * self.flat_grad.element_size()
        return all(p.grad is not None and lo <= p.grad.data_ptr() < hi for p in self._params)

    def reduce_gradients(self):
        """Average of the flat gradient over the replicas.  Buckets whose all-reduce was already issued from
        the backward pass are only waited for; the others (single-bucket models, parameters that took no
        part in the backward pass) are reduced now.  The call closes the step: every bucket is re-armed for
        the next backward pass, so a loop that clears gradients through its optimizer instead of this
        wrapper's ``zero_grad()`` still reduces every step.  (One backward pass per reduction: a second
        one before this call would accumulate into buckets that are already averaged.)"""
        if self.world == 1:
            return
        for bucket in self._buckets:
            if not bucket["sent"]:
                self._send(bucket)
        if self._comm_stream is not None:
            torch.cuda.current_stream(self.flat_grad.device).wait_stream(self._comm_stream)
        for bucket in self._buckets:
            bucket["pending"], bucket["sent"] = len(bucket["members"]), False


def wrap_data_parallel(model, device=None, flat=True, bucket_mb=32.0):
    """Data-parallel wrapper of the training harness: :class:`FlatDataParallel` (graph-capturable,
    one all-reduce per ``bucket_mb`` of gradients) or stock DDP (``flat=False``).  Single process: the model itself."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return model
    if flat:
        return FlatDataParallel(model, bucket_mb=bucket_mb)
    return wrap_ddp(model, device if device is not None else next(model.parameters()).device)


def shard_batches(batches, rank, world):
    """Batch-dimension partitioning of a list of (inputs, labels): rank r gets the
    r-th contiguous slice of every global batch (the reference's DataParallel
    scatter, cifar10_wideResNet.py:142)."""
    if world == 1:
        return batches
    out = []
    for x, y in batches:
        if x.size(0) % world != 0:
            raise ValueError("Batch size: {} must be a multiple of the number of gpus: {}".format(x.size(0), world))
        per = x.size(0) // world
        out.append((x[rank * per:(rank + 1) * per], y[rank * per:(rank + 1) * per]))
    return out


def convert_state_dict_to_data_parallel(state_dict):
    """Adds the ``module.`` prefix a (Distributed)DataParallel wrapper expects, to every key
    (reference: helpers/functions.py:179-189)."""
    return OrderedDict(("module." + k, v) for k, v in state_dict.items())


def convert_state_dict_from_data_parallel(state_dict):
    """Strips the ``module.`` prefix; a key without it raises ``ValueError`` like the reference
    (helpers/functions.py:191-205)."""
    out = OrderedDict()
    for k, v in state_dict.items():
        if not k.startswith("module."):
            raise ValueError("The state_dict passed was not saved by a data parallel instance")
        out[k[len("module."):]] = v
    return out


def gpu_numa_cpus(device_index: int):
    """(numa node, set of CPU ids) the GPU is attached to, read from sysfs, or None when the platform does
    not say.  Pinned host buffers that a rank streams to its GPU should be allocated and first touched by a
    thread running on these CPUs: with 4-8 ranks per box, staging through the other socket's memory halves
    the host-side bandwidth of every rank."""
    try:
        pr = torch.cuda.get_device_properties(device_index)
        bdf = f"{pr.pci_domain_id:04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0"
        node = int(open(f"/sys/bus/pci/devices/{bdf}/numa_node").read().strip())
        if node < 0:
            return None
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            lo, _, hi = part.partition("-")
            cpus.update(range(int(lo), int(hi or lo) + 1))
        return node, cpus
    except Exception:
        return None


class numa_local:
    """Context manager: pins the calling thread to the CPUs of the GPU's NUMA node (intersected with the
    CPUs the process may use) for the duration of the block, e.g. while pinned buffers are allocated and
    first touched; restores the previous affinity on exit.  No-op when sysfs has no answer."""

    def __init__(self, device_index: int):
        self.info = gpu_numa_cpus(device_index)
        self.prev = None
        self.applied = None

    def __enter__(self):
        try:
            if self.info is not None:
                self.prev = os.sched_getaffinity(0)
                local = self.info[1] & self.prev
                if local:
                    os.sched_setaffinity(0, local)
                    self.applied = {"numa_node": self.info[0], "cpus": len(local)}
        except Exception:
            self.applied = None
        return self

    def __exit__(self, *exc):
        if self.prev is not None:
            try:
                os.sched_setaffinity(0, self.prev)
            except Exception:
                pass
        return False


def max_over_ranks(value: float, device) -> float:
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
