"""hvd.Lars.step (plain torch, CPU) against an independent fp64 implementation of the LARS update, its exclusion rule,
its state_dict round trip and hyper-parameter checks, and the ResNet-50 example with --optimizer lars."""
import copy
import math

import pytest
import torch

from horovod_b200.torch.lamb import Lamb
from horovod_b200.torch.lars import Lars
from test_examples import _hvdrun


def _ref_step(w, g, v, lr, mom, wd, tc, eps, adapt):
    """One LARS step in fp64 on flat lists of Python floats; returns the new w, v and the trust ratio."""
    d = [x + wd * y for x, y in zip(g, w)]
    wn, gn = math.sqrt(sum(x * x for x in w)), math.sqrt(sum(x * x for x in g))
    r = tc * wn / (gn + wd * wn + eps) if adapt and wn > 0 and gn > 0 else 1.0
    v = [mom * a + lr * r * x for a, x in zip(v, d)]
    return [x - a for x, a in zip(w, v)], v, r


def _model():
    torch.manual_seed(0)
    ps = {'decayed': torch.randn(7, 5), 'eps': torch.randn(4, 3), 'plain': torch.randn(6), 'adapted': torch.randn(3, 4),
          'zero': torch.zeros(9), 'still': torch.randn(4), 'nomom': torch.randn(5)}
    return {k: torch.nn.Parameter(v) for k, v in ps.items()}


GROUPS = [  # (parameter names, group options)
    (['decayed'], dict(weight_decay=0.1)),
    (['eps'], dict(weight_decay=0.01, eps=0.5, trust_coefficient=0.02)),
    (['plain'], dict(weight_decay=0.0)),                          # r = 1: no adaptation without weight decay
    (['adapted'], dict(weight_decay=0.0, always_adapt=True)),
    (['zero'], dict(weight_decay=0.01)),                          # ||w|| = 0 on the first step: r = 1
    (['still'], dict(weight_decay=0.0, always_adapt=True)),       # zero gradient: ||g|| = 0, r = 1
    (['nomom'], dict(weight_decay=0.05, momentum=0.0)),
]
LR, MOM, TC = 0.5, 0.9, 0.001


def _opt(ps):
    return Lars([dict(params=[ps[n] for n in names], **kw) for names, kw in GROUPS], lr=LR, momentum=MOM,
                trust_coefficient=TC)


def _grads(step, ps):
    gen = torch.Generator().manual_seed(step)
    out = {k: torch.randn(p.shape, generator=gen) for k, p in ps.items()}
    out['still'].zero_()
    return out


def test_lars_step_matches_fp64_reference():
    ps = _model()
    opt = _opt(ps)
    ref = {k: dict(w=p.detach().double().reshape(-1).tolist(), v=[0.0] * p.numel()) for k, p in ps.items()}
    hp = {n: kw for names, kw in GROUPS for n in names}
    ratios = {k: [] for k in ps}
    for step in range(1, 11):
        if step == 6:
            for g in opt.param_groups:
                g['lr'] = LR / 2  # a schedule: the rate enters the momentum, earlier steps keep theirs
        grads = _grads(step, ps)
        for k, p in ps.items():
            p.grad = grads[k].clone()
            h = hp[k]
            wd = h.get('weight_decay', 0.0)
            adapt = wd != 0.0 or h.get('always_adapt', False)
            s = ref[k]
            s['w'], s['v'], r = _ref_step(s['w'], grads[k].double().reshape(-1).tolist(), s['v'], LR if step < 6 else LR / 2,
                                          h.get('momentum', MOM), wd, h.get('trust_coefficient', TC), h.get('eps', 0.0),
                                          adapt)
            ratios[k].append(r)
        opt.step()
        for k, p in ps.items():
            want = torch.tensor(ref[k]['w'], dtype=torch.float64).reshape(p.shape)
            torch.testing.assert_close(p.detach().double(), want, rtol=1e-5, atol=1e-6,
                                       msg=lambda m: '%s step %d: %s' % (k, step, m))
            buf = opt.state[p]['momentum_buffer']
            assert buf.dtype == torch.float32 and 'step' not in opt.state[p]
            torch.testing.assert_close(buf.double().reshape(-1), torch.tensor(ref[k]['v'], dtype=torch.float64),
                                       rtol=1e-5, atol=1e-7)
    # every branch of r was taken: adapted ratios differ from 1, the others are exactly 1
    assert all(abs(r - 1.0) > 1e-3 for k in ('decayed', 'eps', 'adapted', 'nomom') for r in ratios[k])
    assert ratios['plain'] == [1.0] * 10 and ratios['still'] == [1.0] * 10 and ratios['zero'][0] == 1.0
    assert ratios['zero'][1] != 1.0
    assert torch.equal(ps['still'].detach(), _model()['still'])


def test_lars_exclusion_rule_is_lambs():
    assert Lars.adapts is Lamb.adapts
    for wd, always, want in ((0.0, False, False), (0.0, True, True), (1e-4, False, True)):
        assert Lars.adapts({'weight_decay': wd, 'always_adapt': always}) is want


def test_lars_excluded_group_is_momentum_sgd_with_lr_inside():
    """weight_decay == 0 without always_adapt: v = m v + lr g, w -= v."""
    p = torch.nn.Parameter(torch.randn(10))
    w0 = p.detach().double()
    opt = Lars([p], lr=0.1, momentum=0.9)
    v = torch.zeros_like(w0)
    for step in range(3):
        g = torch.randn(10, generator=torch.Generator().manual_seed(step))
        p.grad = g.clone()
        opt.step()
        v = 0.9 * v + 0.1 * g.double()
        w0 = w0 - v
        torch.testing.assert_close(p.detach().double(), w0, rtol=1e-6, atol=1e-7)


def test_lars_state_dict_round_trip():
    ps = _model()
    opt = _opt(ps)
    for step in range(1, 4):
        for k, g in _grads(step, ps).items():
            ps[k].grad = g
        opt.step()
    twin_ps = {k: torch.nn.Parameter(p.detach().clone()) for k, p in ps.items()}
    twin = _opt(twin_ps)
    twin.load_state_dict(copy.deepcopy(opt.state_dict()))
    for step in range(4, 7):
        for k, g in _grads(step, ps).items():
            ps[k].grad = g
            twin_ps[k].grad = g.clone()
        opt.step()
        twin.step()
    for k in ps:
        assert torch.equal(ps[k], twin_ps[k])


def test_lars_bf16_parameters_keep_fp32_momentum():
    """load_state_dict casts the momentum to the parameter's dtype; step() brings it back to fp32."""
    p = torch.nn.Parameter(torch.randn(16).to(torch.bfloat16))
    opt = Lars([p], lr=0.1, weight_decay=0.01)
    p.grad = torch.randn(16).to(torch.bfloat16)
    opt.step()
    assert opt.state[p]['momentum_buffer'].dtype == torch.float32
    opt.load_state_dict(opt.state_dict())
    assert opt.state[p]['momentum_buffer'].dtype == torch.bfloat16
    opt.step()
    assert opt.state[p]['momentum_buffer'].dtype == torch.float32


def test_lars_closure_returns_loss():
    p = torch.nn.Parameter(torch.ones(3))
    opt = Lars([p], lr=0.1)

    def closure():
        opt.zero_grad()
        loss = (p * p).sum()
        loss.backward()
        return loss
    assert float(opt.step(closure).detach()) == 3.0
    assert not torch.equal(p.detach(), torch.ones(3))


def test_lars_rejects_sparse_gradients():
    p = torch.nn.Parameter(torch.ones(4))
    opt = Lars([p], lr=0.1)
    p.grad = torch.ones(4).to_sparse()
    with pytest.raises(RuntimeError, match='sparse'):
        opt.step()


@pytest.mark.parametrize("kw", [dict(lr=-1e-3), dict(momentum=-0.1), dict(momentum=1.0), dict(weight_decay=-0.01),
                                dict(trust_coefficient=0.0), dict(trust_coefficient=-1.0), dict(eps=-1.0)])
def test_lars_rejects_invalid_hyper_parameters(kw):
    with pytest.raises(ValueError):
        Lars([torch.nn.Parameter(torch.zeros(2))], **dict(dict(lr=0.1), **kw))


def test_lars_is_an_optimizer_but_not_sgd():
    import horovod_b200.torch as hvd
    opt = Lars([torch.nn.Parameter(torch.zeros(2))], lr=0.1)
    assert hvd.Lars is Lars and isinstance(opt, torch.optim.Optimizer) and not isinstance(opt, torch.optim.SGD)


def test_imagenet_example_with_lars(native_built):
    rc, out = _hvdrun(2, 'examples/pytorch_imagenet_resnet50_synthetic.py', '--no-cuda', '--model', 'tiny',
                      '--optimizer', 'lars', '--epochs', '1', '--steps-per-epoch', '3', '--batch-size', '4',
                      '--image-size', '32')
    assert rc == 0 and 'TRAINING DONE' in out and 'finite loss: True' in out, out[-3000:]


def test_lars_needs_a_learning_rate():
    p = torch.nn.Parameter(torch.zeros(2))
    with pytest.raises(ValueError):
        Lars([p])
    assert Lars([{'params': [p], 'lr': 0.1}]).param_groups[0]['lr'] == 0.1
