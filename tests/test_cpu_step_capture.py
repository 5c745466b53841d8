"""The CUDA-graph step runner of both training loops (``_CapturedStep``) on the CPU.  Its only CUDA calls, the
capture helper ``_capture`` and the side stream ``_side_stream``, are replaced by fakes that record where each step
ran: eagerly, on the side stream, under capture or as a replay."""
import contextlib
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from quantized_distillation_b200 import distributed as D
from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
from quantized_distillation_b200.cnn_models import help_fun as hf
from test_harness_cpu import _cpu_only_children, _free_port, student

CPU = torch.device("cpu")


class _Fakes:
    """``where`` is what the runner is doing; ``fail`` makes every capture fail after running the step, as a
    capture that raises at its end does.  A fake graph's replay runs the step again and writes its tensor outputs
    into the captured ones, as a real replay writes into the graph's static outputs."""

    def __init__(self, fail=False):
        self.fail, self.where, self.log = fail, "eager", []
        self.streams = self.captures = self.replays = 0

    def side_stream(self, device):
        self.streams += 1

        @contextlib.contextmanager
        def on_side():
            self.where = "side"
            yield
            self.where = "eager"
        return None, on_side

    def capture(self, fn, device, stream=None, thread_local=False, what=""):
        self.captures += 1
        self.where = "capture"
        out = fn()
        self.where = "eager"
        return None if self.fail else (_FakeGraph(self, fn, out), out)

    def step(self, batch, idx_minibatch, epoch):
        """A step function that records where it ran and returns (loss, asked, total) of its batch."""
        self.log.append(self.where)
        return batch[0].sum(), 0, batch[0].shape[0]


class _FakeGraph:
    def __init__(self, fakes, fn, out):
        self.fakes, self.fn, self.out = fakes, fn, out

    def replay(self):
        self.fakes.replays += 1
        self.fakes.where = "replay"
        for o, n in zip(self.out, self.fn()):
            if isinstance(o, torch.Tensor):
                o.copy_(n)
        self.fakes.where = "eager"


class _Optimizer:
    def __init__(self, lr=0.1):
        self.param_groups = [{"lr": lr}, {"lr": lr}]
        self.cleared = []

    def zero_grad(self, set_to_none=False):
        self.cleared.append(set_to_none)


@pytest.fixture
def fakes(monkeypatch):
    f = _Fakes()
    monkeypatch.setattr(cfm, "_capture", f.capture)
    monkeypatch.setattr(cfm, "_side_stream", f.side_stream)
    return f


def _batches(n, rows=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(rows, 3, generator=g), torch.zeros(rows, dtype=torch.int64)) for _ in range(n)]


def _run(runner, batches, epoch=0):
    return [runner.run(b, i, epoch) for i, b in enumerate(batches, start=1)]


def test_three_eager_steps_then_one_capture_then_replays(fakes):
    opt = _Optimizer()
    runner = cfm._CapturedStep(fakes.step, opt, CPU, enabled=True)
    for i, (x, y) in enumerate(_batches(7), start=1):
        loss, asked, total = runner.run((x, y), i, 0)    # a replay's loss is the graph's static output
        assert torch.equal(loss, x.sum()) and (asked, total) == (0, 4)
    assert fakes.log == ["side"] * 3 + ["capture"] + ["replay"] * 4
    assert fakes.captures == 1 and fakes.streams == 1 and runner.captured
    assert opt.cleared == [True]                     # gradients set to None once, right before the capture


def test_static_gradients_are_not_cleared(fakes):
    opt = _Optimizer()
    _run(cfm._CapturedStep(fakes.step, opt, CPU, enabled=True, static_grads=True), _batches(5))
    assert fakes.captures == 1 and opt.cleared == []


def test_disabled_runner_calls_the_step(fakes):
    runner = cfm._CapturedStep(fakes.step, _Optimizer(), CPU, enabled=False)
    _run(runner, _batches(6))
    assert fakes.log == ["eager"] * 6
    assert fakes.streams == 0 and fakes.captures == 0 and not runner.captured


def test_failed_capture_leaves_the_run_eager(fakes):
    fakes.fail = True
    runner = cfm._CapturedStep(fakes.step, _Optimizer(), CPU, enabled=True)
    outs = _run(runner, _batches(7))
    assert fakes.log == ["side"] * 3 + ["capture"] + ["eager"] * 4   # the capture's batch runs eagerly too
    assert fakes.captures == 1 and fakes.replays == 0 and not runner.captured
    assert torch.equal(outs[3][0], _batches(7)[3][0].sum())


def test_learning_rate_change_recaptures_once(fakes):
    opt = _Optimizer(lr=0.1)
    runner = cfm._CapturedStep(fakes.step, opt, CPU, enabled=True)
    _run(runner, _batches(5))
    cfm._set_learning_rate([opt], 0.1, runner)        # unchanged: the graph stays
    _run(runner, _batches(2, seed=1))
    assert fakes.captures == 1
    cfm._set_learning_rate([opt, _Optimizer(0.1)], 0.05, runner)
    assert all(g["lr"] == 0.05 for g in opt.param_groups)
    fakes.log.clear()
    _run(runner, _batches(4, seed=2))
    assert fakes.log == ["capture"] + ["replay"] * 4 and fakes.captures == 2 and runner.captured


def test_captured_stays_true_after_a_failed_recapture(fakes):
    opt = _Optimizer()
    runner = cfm._CapturedStep(fakes.step, opt, CPU, enabled=True)
    _run(runner, _batches(5))
    fakes.fail = True
    cfm._set_learning_rate([opt], 0.01, runner)
    fakes.log.clear()
    _run(runner, _batches(3))
    assert fakes.log == ["capture", "eager", "eager", "eager"] and runner.captured


def test_batch_of_another_shape_runs_eagerly_and_keeps_the_graph(fakes):
    runner = cfm._CapturedStep(fakes.step, _Optimizer(), CPU, enabled=True)
    _run(runner, _batches(5))
    fakes.log.clear()
    short = _batches(1, rows=3)[0]
    loss = runner.run(short, 6, 0)[0]
    _run(runner, _batches(2, seed=3))
    assert fakes.log == ["side", "replay", "replay"] and fakes.captures == 1
    assert torch.equal(loss, short[0].sum())


def test_train_model_reports_the_capture(monkeypatch):
    """``informationDict["cuda_graph_step"]`` is always set, and True when the step was captured at least once;
    a learning-rate change between epochs re-captures.  On the CPU the rule refuses capture; with the rule and the
    CUDA parts faked, the loop drives the runner."""
    data = hf.synthetic_cifar_loader(5, 4, pin=False)
    kw = dict(epochs_to_train=2, print_every=5, verbose=False, evaluate=False, cuda_graph_step=True)
    torch.manual_seed(0)
    assert cfm.train_model(student(), data, data, **kw)[1]["cuda_graph_step"] is False
    f = _Fakes()
    monkeypatch.setattr(cfm, "_capture", f.capture)
    monkeypatch.setattr(cfm, "_side_stream", f.side_stream)
    monkeypatch.setattr(cfm, "_step_capturable", lambda model, ranks, device: True)
    # 'cifar100' drops the rate after epoch 61: the second epoch captures again
    info = cfm.train_model(student(), data, data, learning_rate_style="cifar100", start_epoch=61, **kw)[1]
    assert info["cuda_graph_step"] is True and info["numStepsTrained"] == 10
    assert f.captures == 2 and f.replays == 2 + 5
    f.fail, f.captures = True, 0
    assert cfm.train_model(student(), data, data, **kw)[1]["cuda_graph_step"] is False and f.captures == 1


def test_capture_rule_single_process():
    model = student()
    cuda = torch.device("cuda")
    assert cfm._step_capturable(model, None, cuda) and not cfm._step_capturable(model, None, CPU)
    if not dist.is_initialized():                    # a wrapper without a process group is not data parallel
        wrapped = D.FlatDataParallel(model)
        assert cfm._step_capturable(wrapped, cfm._RankGroup(wrapped), cuda)


def _gloo_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    D.init_distributed(backend="gloo")
    try:
        group = dist.new_group(list(range(world)))     # not the default group: the agreement must use the wrapper's
        wrapper = D.FlatDataParallel(torch.nn.Linear(3, 2), process_group=group)
        ranks = cfm._RankGroup(wrapper)
        ddp = D.wrap_ddp(torch.nn.Linear(3, 2), CPU)
        cuda = torch.device("cuda")
        out = {"capturable": (cfm._step_capturable(wrapper, ranks, cuda),
                              cfm._step_capturable(ddp, cfm._RankGroup(ddp), cuda))}
        groups, all_reduce = [], dist.all_reduce

        def spy(tensor, op=dist.ReduceOp.SUM, group=None, async_op=False):
            groups.append(group)
            return all_reduce(tensor, op=op, group=group, async_op=async_op)
        dist.all_reduce = spy
        for failing in (None, 1):
            fakes = _Fakes(fail=rank == failing)
            cfm._capture, cfm._side_stream = fakes.capture, fakes.side_stream
            runner = cfm._CapturedStep(fakes.step, None, CPU, enabled=True, ranks=ranks, static_grads=True)
            _run(runner, _batches(6))
            out[failing] = (fakes.log, runner.captured)
        dist.all_reduce = all_reduce
        out["groups"] = [g is group for g in groups]
        ret[rank] = out
    finally:
        dist.destroy_process_group()


def test_ranks_agree_on_the_capture_gloo_world2():
    """Two gloo ranks: the capture flag is all-reduced once per capture on the wrapper's process group, both ranks
    replay when both captured, and both run eagerly when one rank's capture fails.  A gloo FlatDataParallel and a
    stock DDP wrapper are never captured."""
    world = 2
    with mp.Manager() as mgr:
        ret = mgr.dict()
        with _cpu_only_children():
            mp.spawn(_gloo_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
        runs = [ret[r] for r in range(world)]
    for out in runs:
        assert out["capturable"] == (False, False)
        assert out[None] == (["side"] * 3 + ["capture"] + ["replay"] * 3, True)
        assert out[1] == (["side"] * 3 + ["capture"] + ["eager"] * 3, False)
        assert out["groups"] == [True, True]
