"""The data-parallel path of ``optimize_quantization_points`` engages only for a wrapped model: an unwrapped model
with no process group runs the single-process code and calls no collective (``torch.distributed`` mocked)."""
import pytest
import torch
import torch.distributed as dist

from quantized_distillation_b200 import distributed as D
from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
from quantized_distillation_b200.cnn_models import help_fun as hf


class _Reached(Exception):
    """Raised where the loop would build its per-tensor quantization functions (past every setup collective)."""


def _student():
    spec = dict(cfm.smallerModelSpec)
    spec["spec_dropout_rates"] = []
    return cfm.ConvolForwardNet(**spec, useBatchNorm=False)


@pytest.fixture
def collectives(monkeypatch):
    calls = []

    def recorder(name):
        def call(*args, **kwargs):
            calls.append(name)
            raise AssertionError(f"torch.distributed.{name} called")
        return call
    for name in ("all_reduce", "broadcast", "all_gather", "reduce", "barrier", "get_world_size", "get_backend",
                 "get_global_rank"):
        monkeypatch.setattr(dist, name, recorder(name))

    def stop(*a, **k):
        raise _Reached()
    monkeypatch.setattr(cfm.quantization, "nonUniformQuantization_variable", stop)
    # the gradient norms of assignBitsAutomatically run on the GPU; here every tensor gets the same norm
    monkeypatch.setattr(cfm.quantization.help_functions, "gradient_norms", lambda ts: torch.ones(len(ts)))
    return calls


@pytest.mark.parametrize("assign", [False, True])
def test_unwrapped_model_calls_no_collective(collectives, assign):
    torch.manual_seed(0)
    model = _student()
    batches = hf.synthetic_cifar_loader(5, 4, seed=1, pin=False)
    with pytest.raises(_Reached):
        cfm.optimize_quantization_points(model, batches, batches, numPointsPerTensor=4, bucket_size=256,
                                         assignBitsAutomatically=assign, initialize_method="uniform", verbose=False)
    assert collectives == []


def test_wrapper_detection():
    model = _student()
    assert cfm._data_parallel_module(model) is None
    wrapped = D.FlatDataParallel(model)                  # no process group: world 1
    assert cfm._data_parallel_module(wrapped) is model


def test_wrapper_without_process_group_calls_no_collective(collectives):
    """A wrapper built in a single process takes the data-parallel path with every collective the identity."""
    if dist.is_initialized():
        pytest.skip("a process group is initialised in this process")
    torch.manual_seed(0)
    wrapped = D.FlatDataParallel(_student())
    batches = hf.synthetic_cifar_loader(5, 4, seed=1, pin=False)
    with pytest.raises(_Reached):
        cfm.optimize_quantization_points(wrapped, batches, batches, numPointsPerTensor=4, bucket_size=256,
                                         assignBitsAutomatically=True, initialize_method="uniform", verbose=False)
    assert collectives == []


def test_flat_wrapper_no_sync_issues_no_reduction(monkeypatch):
    """``FlatDataParallel.no_sync()``: the bucket hooks issue nothing inside the block and are re-armed after it."""
    torch.manual_seed(0)
    wrapped = D.FlatDataParallel(_student(), bucket_mb=0.25)
    sent = []
    monkeypatch.setattr(wrapped, "_send", lambda bucket: sent.append(bucket))
    wrapped._early = True                               # as with several ranks: reductions from the hooks
    for i, p in enumerate(wrapped._params):
        p.register_post_accumulate_grad_hook(wrapped._make_hook(i))
    x, y = hf.synthetic_cifar_loader(1, 4, seed=1, pin=False)[0]
    with wrapped.no_sync():
        for _ in range(2):
            torch.nn.functional.cross_entropy(wrapped(x), y).backward()
    assert sent == []
    assert all(b["sent"] is False and b["pending"] == len(b["members"]) for b in wrapped._buckets)
    torch.nn.functional.cross_entropy(wrapped(x), y).backward()
    assert len(sent) == len(wrapped._buckets)
