"""Gradient accumulation without a GPU: grad_accumulation_dtype validation, and hvd.GraphedStep's eager micro-step loop
(CPU inputs: no graph) stepping the optimizer once per backward_passes_per_step calls and refusing a changed k."""
import copy

import pytest
import torch


@pytest.fixture
def hvd(native_built):
    import horovod_b200.torch as hvd
    hvd.init()
    yield hvd
    hvd.shutdown()


def _model():
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Tanh(), torch.nn.Linear(5, 2))


@pytest.mark.parametrize("bad", [torch.float16, torch.bfloat16, torch.float64, 'float32', 32])
def test_bad_grad_accumulation_dtype_raises(hvd, bad):
    m = _model()
    with pytest.raises(ValueError, match='grad_accumulation_dtype'):
        hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters(),
                                 backward_passes_per_step=2, grad_accumulation_dtype=bad)
    with pytest.raises(ValueError, match='grad_accumulation_dtype'):
        hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters(),
                                 shard_optimizer_state=True, grad_accumulation_dtype=bad)


def test_grad_accumulation_dtype_not_with_adasum(hvd):
    m = _model()
    with pytest.raises(ValueError, match='Adasum'):
        hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters(),
                                 op=hvd.Adasum, grad_accumulation_dtype=torch.float32)


def _batches(n):
    g = torch.Generator().manual_seed(1)
    return [(torch.randn(4, 6, generator=g), torch.randn(4, 2, generator=g)) for _ in range(n)]


@pytest.mark.parametrize("k", [1, 2, 3, 4])
@pytest.mark.parametrize("acc", [None, torch.float32])
def test_graphed_step_eager_loop_steps_once_per_k_calls(hvd, k, acc):
    """CPU inputs: GraphedStep runs its eager loop.  The optimizer steps after every k-th call and matches the reference
    idiom (zero_grad, k backward passes of loss / k, step); every call returns its own micro-batch's loss.  fp32
    parameters are not affected by grad_accumulation_dtype."""
    m = _model()
    ref = copy.deepcopy(m)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9),
                                   named_parameters=m.named_parameters(), backward_passes_per_step=k,
                                   grad_accumulation_dtype=acc)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.1, momentum=0.9)
    fn = lambda x, y: torch.nn.functional.mse_loss(m(x), y) / k  # noqa: E731
    data = _batches(2 * k + 1)
    step = hvd.GraphedStep(fn, opt, data[0])
    assert not step.captured and step.fallback_reason == 'inputs are not CUDA tensors'
    steps = []
    orig = opt.step
    opt.step = lambda *a, **kw: (steps.append(len(steps)), orig(*a, **kw))[1]
    for i, (x, y) in enumerate(data[:2 * k]):
        with torch.no_grad():
            expect = float(fn(x, y))
        assert float(step(x, y).detach()) == expect
        assert len(steps) == (i + 1) // k
    for s in range(2):
        ropt.zero_grad()
        for x, y in data[s * k:(s + 1) * k]:
            (torch.nn.functional.mse_loss(ref(x), y) / k).backward()
        ropt.step()
    for a, b in zip(m.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-7)


def test_graphed_step_refuses_changed_k(hvd):
    m = _model()
    opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters(),
                                   backward_passes_per_step=2)
    data = _batches(2)
    step = hvd.GraphedStep(lambda x, y: torch.nn.functional.mse_loss(m(x), y), opt, data[0])
    step(*data[0])
    opt.set_backward_passes_per_step(4)
    with pytest.raises(RuntimeError, match='backward_passes_per_step'):
        step(*data[1])
