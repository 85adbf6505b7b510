"""The classes hvd.DistributedOptimizer builds, without a GPU: the returned optimizer is an instance of its wrapper class
and of the wrapped optimizer's class, a subclass of it works, hvd.GraphedStep and broadcast_optimizer_state tell the
optimizers apart by type, and the Adasum optimizer checks its parameter names like the other two."""
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


def _loss(m, i):
    g = torch.Generator().manual_seed(i)
    return torch.nn.functional.mse_loss(m(torch.randn(4, 6, generator=g)), torch.randn(4, 2, generator=g))


def _adasum(m, named_parameters=None):
    """The Adasum optimizer as hvd.DistributedOptimizer builds it on more than one rank (on one rank it returns the
    unsharded optimizer)."""
    from horovod_b200.torch.compression import Compression
    from horovod_b200.torch.optimizer import _DistributedAdasumOptimizer
    sgd = torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9)
    cls = type('SGD', (_DistributedAdasumOptimizer, torch.optim.SGD), {})
    return cls(sgd.param_groups, m.named_parameters() if named_parameters is None else named_parameters,
               Compression.none)


def test_returned_optimizer_is_an_instance_of_both_classes(hvd):
    from horovod_b200.torch.optimizer import _DistributedAdasumOptimizer, _DistributedOptimizer, _DistributedOptimizerBase
    from horovod_b200.torch.sharded_optimizer import _ShardedDistributedOptimizer
    m = _model()
    opt = hvd.DistributedOptimizer(torch.optim.Adam(m.parameters(), lr=0.1), named_parameters=m.named_parameters())
    assert isinstance(opt, _DistributedOptimizer) and isinstance(opt, _DistributedOptimizerBase)
    assert isinstance(opt, torch.optim.Adam) and type(opt).__name__ == 'Adam'
    assert issubclass(_ShardedDistributedOptimizer, _DistributedOptimizerBase)
    ada = _adasum(_model())
    assert isinstance(ada, _DistributedAdasumOptimizer) and isinstance(ada, torch.optim.SGD)
    assert not isinstance(ada, _DistributedOptimizerBase)
    assert not hasattr(ada, 'clip_grad_norm_') and not hasattr(ada, 'ema_parameters')


def test_subclass_of_returned_class_steps_saves_and_loads(hvd):
    """A subclass's zero_grad(), step(), state_dict() and load_state_dict() reach the wrapper and the wrapped SGD, and it
    steps like torch's SGD (one rank: the averaged gradient is the gradient)."""
    from horovod_b200.torch.compression import Compression
    cls = type(hvd.DistributedOptimizer(torch.optim.SGD(_model().parameters(), lr=0.1)))
    calls = []

    class Counting(cls):
        def step(self, closure=None):
            calls.append('step')
            return super().step(closure)

    m = _model()
    ref = copy.deepcopy(m)
    opt = Counting(torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9).param_groups, m.named_parameters(),
                   Compression.none)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.1, momentum=0.9)
    for i in range(3):
        for mm, oo in ((m, opt), (ref, ropt)):
            oo.zero_grad()
            _loss(mm, i).backward()
            oo.step()
    assert calls == ['step'] * 3
    for a, b in zip(m.parameters(), ref.parameters()):
        assert torch.equal(a, b)
    sd = opt.state_dict()
    assert all(torch.equal(sd['state'][i]['momentum_buffer'], ropt.state[p]['momentum_buffer'])
               for i, p in enumerate(ref.parameters()))
    # a checkpoint of another run: both continue from it alike
    for p in ropt.state:
        ropt.state[p]['momentum_buffer'].mul_(0.5)
    opt.load_state_dict(copy.deepcopy(ropt.state_dict()))
    for mm, oo in ((m, opt), (ref, ropt)):
        oo.zero_grad()
        _loss(mm, 3).backward()
        oo.step()
    for a, b in zip(m.parameters(), ref.parameters()):
        assert torch.equal(a, b)


@pytest.mark.parametrize("adasum", [False, True], ids=['allreduce', 'adasum'])
def test_broadcast_optimizer_state_takes_the_wrapped_step(hvd, adasum):
    """A fresh optimizer's state is created by the wrapped optimizer's own step, which leaves the weights alone."""
    m = _model()
    opt = _adasum(m) if adasum else hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9),
                                                             named_parameters=m.named_parameters())
    before = [p.detach().clone() for p in m.parameters()]
    hvd.broadcast_optimizer_state(opt, root_rank=0)
    for p, b in zip(m.parameters(), before):
        assert torch.equal(p, b) and p.grad is None
        assert torch.equal(opt.state[p]['momentum_buffer'], torch.zeros_like(p))


def test_graphed_step_tells_the_optimizers_apart_by_type(hvd):
    m = _model()
    x = (torch.randn(4, 6), torch.randn(4, 2))
    fn = lambda x, y: torch.nn.functional.mse_loss(m(x), y)  # noqa: E731
    ada = _adasum(m)
    with pytest.raises(ValueError, match='Adasum'):
        hvd.GraphedStep(fn, ada, x, max_grad_norm=1.0)
    with pytest.raises(ValueError, match='Adasum'):
        hvd.GraphedStep(fn, ada, x, scaler=torch.amp.GradScaler('cpu'))
    assert hvd.GraphedStep(fn, ada, x).fallback_reason == 'inputs are not CUDA tensors'
    with pytest.raises(ValueError, match='DistributedOptimizer'):
        hvd.GraphedStep(fn, torch.optim.SGD(m.parameters(), lr=0.1), x, scaler=torch.amp.GradScaler('cpu'))


def test_adasum_checks_parameter_names(hvd):
    m = _model()
    ps = list(m.parameters())
    with pytest.raises(ValueError, match='unique'):
        _adasum(m, [('w', p) for p in ps])
    with pytest.raises(ValueError, match='tuples'):
        _adasum(m, [['w%d' % i, p] for i, p in enumerate(ps)])
    with pytest.raises(ValueError, match='not named'):
        _adasum(m, list(m.named_parameters())[1:])
