"""hvd.GraphedStep with max_grad_norm without a GPU: its eager loop on CPU tensors equals torch's clipping loop exactly,
and the arguments it cannot honour are refused when the step is built."""
import copy
import math

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


def _batches(n):
    g = torch.Generator().manual_seed(1)
    return [(torch.randn(4, 6, generator=g), torch.randn(4, 2, generator=g)) for _ in range(n)]


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("norm_type", [2.0, math.inf])
def test_graphed_step_eager_clip_equals_torch_loop(hvd, k, norm_type):
    m = _model()
    ref = copy.deepcopy(m)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9),
                                   named_parameters=m.named_parameters(), backward_passes_per_step=k)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.1, momentum=0.9)
    fn = lambda x, y: torch.nn.functional.mse_loss(m(x), y) / k  # noqa: E731
    data = _batches(3 * k)
    step = hvd.GraphedStep(fn, opt, data[0], max_grad_norm=0.1, norm_type=norm_type)
    assert not step.captured
    for x, y in data:
        step(x, y)
    for s in range(3):
        ropt.zero_grad()
        for x, y in data[s * k:(s + 1) * k]:
            (torch.nn.functional.mse_loss(ref(x), y) / k).backward()
        assert float(torch.nn.utils.clip_grad_norm_(ref.parameters(), 0.1, norm_type)) > 0.1
        ropt.step()
    for a, b in zip(m.parameters(), ref.parameters()):
        assert torch.equal(a, b)


def test_graphed_step_rejections(hvd):
    m = _model()
    x = _batches(1)[0]
    fn = lambda x, y: torch.nn.functional.mse_loss(m(x), y)  # noqa: E731
    adasum = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters(),
                                      op=hvd.Adasum)
    with pytest.raises(ValueError, match='Adasum'):
        hvd.GraphedStep(fn, adasum, x, max_grad_norm=1.0)
    with pytest.raises(ValueError, match='Adasum'):
        hvd.GraphedStep(fn, adasum, x, scaler=torch.amp.GradScaler('cpu'))
    opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters())
    for bad in (1.0, 0.0, -math.inf):
        with pytest.raises(ValueError, match='norm_type'):
            hvd.GraphedStep(fn, opt, x, max_grad_norm=1.0, norm_type=bad)
    with pytest.raises(ValueError, match='CUDA'):
        hvd.GraphedStep(fn, opt, x, scaler=torch.amp.GradScaler('cpu'))
    with pytest.raises(ValueError, match='DistributedOptimizer'):
        hvd.GraphedStep(fn, torch.optim.SGD(m.parameters(), lr=0.1), x, max_grad_norm=1.0)
