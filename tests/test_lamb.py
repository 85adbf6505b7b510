"""hvd.Lamb.step (plain torch, CPU) against an independent fp64 implementation of the LAMB update, its state_dict round
trip and its hyper-parameter checks."""
import copy
import math

import pytest
import torch

from horovod_b200.torch.lamb import Lamb


def _ref_step(w, g, m, v, t, lr, b1, b2, eps, wd, bias_correction, adapt):
    """One LAMB step in fp64 on flat lists of Python floats; returns the new w, m, v and the trust ratio."""
    m = [b1 * a + (1 - b1) * x for a, x in zip(m, g)]
    v = [b2 * a + (1 - b2) * x * x for a, x in zip(v, g)]
    c1, c2 = (1 - b1 ** t, 1 - b2 ** t) if bias_correction else (1.0, 1.0)
    u = [(a / c1) / (math.sqrt(b / c2) + eps) + wd * x for a, b, x in zip(m, v, w)]
    wn, un = math.sqrt(sum(x * x for x in w)), math.sqrt(sum(x * x for x in u))
    r = wn / un if adapt and wn > 0 and un > 0 else 1.0
    return [x - lr * r * y for x, y in zip(w, u)], m, v, r


def _model():
    torch.manual_seed(0)
    ps = {'decayed': torch.randn(7, 5), 'plain': torch.randn(6), 'adapted': torch.randn(3, 4),
          'zero': torch.zeros(9), 'still': torch.randn(4)}
    return {k: torch.nn.Parameter(v) for k, v in ps.items()}


GROUPS = [  # (parameter names, group options)
    (['decayed'], dict(weight_decay=0.1)),
    (['plain'], dict(weight_decay=0.0)),                          # r = 1: no adaptation without weight decay
    (['adapted'], dict(weight_decay=0.0, always_adapt=True)),
    (['zero'], dict(weight_decay=0.01)),                          # ||w|| = 0 on the first step: r = 1
    (['still'], dict(weight_decay=0.0, always_adapt=True)),       # zero gradient and wd = 0: ||u|| = 0, r = 1
]


def _opt(ps, bias_correction):
    return Lamb([dict(params=[ps[n] for n in names], **kw) for names, kw in GROUPS], lr=0.02, betas=(0.9, 0.99), eps=1e-6,
                bias_correction=bias_correction)


def _grads(step, ps):
    gen = torch.Generator().manual_seed(step)
    out = {k: torch.randn(p.shape, generator=gen) for k, p in ps.items()}
    out['still'].zero_()
    return out


@pytest.mark.parametrize("bias_correction", [True, False])
def test_lamb_step_matches_fp64_reference(bias_correction):
    ps = _model()
    opt = _opt(ps, bias_correction)
    ref = {k: dict(w=p.detach().double().reshape(-1).tolist(), m=[0.0] * p.numel(), v=[0.0] * p.numel())
           for k, p in ps.items()}
    hp = {n: kw for names, kw in GROUPS for n in names}
    ratios = {k: [] for k in ps}
    for step in range(1, 11):
        grads = _grads(step, ps)
        for k, p in ps.items():
            p.grad = grads[k].clone()
            wd = hp[k].get('weight_decay', 0.0)
            adapt = wd != 0.0 or hp[k].get('always_adapt', False)
            s = ref[k]
            s['w'], s['m'], s['v'], r = _ref_step(s['w'], grads[k].double().reshape(-1).tolist(), s['m'], s['v'], step,
                                                  0.02, 0.9, 0.99, 1e-6, wd, bias_correction, adapt)
            ratios[k].append(r)
        opt.step()
        for k, p in ps.items():
            want = torch.tensor(ref[k]['w'], dtype=torch.float64).reshape(p.shape)
            torch.testing.assert_close(p.detach().double(), want, rtol=1e-5, atol=1e-6, msg=lambda m: '%s step %d: %s' % (k, step, m))
            st = opt.state[p]
            assert st['exp_avg'].dtype == torch.float32 and float(st['step']) == step
            torch.testing.assert_close(st['exp_avg'].double().reshape(-1), torch.tensor(ref[k]['m'], dtype=torch.float64),
                                       rtol=1e-5, atol=1e-7)
    # every branch of r was taken: adapted ratios differ from 1, the others are exactly 1
    assert all(abs(r - 1.0) > 1e-3 for r in ratios['decayed'] + ratios['adapted'])
    assert ratios['plain'] == [1.0] * 10 and ratios['still'] == [1.0] * 10 and ratios['zero'][0] == 1.0
    assert ratios['zero'][1] != 1.0
    assert torch.equal(ps['still'].detach(), _model()['still'])


def test_lamb_state_dict_round_trip():
    ps = _model()
    opt = _opt(ps, True)
    for step in range(1, 4):
        for k, g in _grads(step, ps).items():
            ps[k].grad = g
        opt.step()
    twin_ps = {k: torch.nn.Parameter(p.detach().clone()) for k, p in ps.items()}
    twin = _opt(twin_ps, True)
    twin.load_state_dict(copy.deepcopy(opt.state_dict()))
    for step in range(4, 7):
        for k, g in _grads(step, ps).items():
            ps[k].grad = g
            twin_ps[k].grad = g.clone()
        opt.step()
        twin.step()
    for k in ps:
        assert torch.equal(ps[k], twin_ps[k])


def test_lamb_bf16_parameters_keep_fp32_moments():
    """load_state_dict casts the moments to the parameter's dtype; step() brings them back to fp32."""
    p = torch.nn.Parameter(torch.randn(16).to(torch.bfloat16))
    opt = Lamb([p], lr=0.01, weight_decay=0.01)
    p.grad = torch.randn(16).to(torch.bfloat16)
    opt.step()
    assert opt.state[p]['exp_avg'].dtype == torch.float32
    opt.load_state_dict(opt.state_dict())
    assert opt.state[p]['exp_avg'].dtype == torch.bfloat16
    opt.step()
    assert opt.state[p]['exp_avg'].dtype == torch.float32 and opt.state[p]['exp_avg_sq'].dtype == torch.float32


def test_lamb_closure_returns_loss():
    p = torch.nn.Parameter(torch.ones(3))
    opt = Lamb([p], lr=0.1)

    def closure():
        opt.zero_grad()
        loss = (p * p).sum()
        loss.backward()
        return loss
    assert float(opt.step(closure).detach()) == 3.0
    assert not torch.equal(p.detach(), torch.ones(3))


@pytest.mark.parametrize("kw", [dict(lr=-1e-3), dict(eps=-1.0), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)),
                                dict(betas=(-0.1, 0.999)), dict(weight_decay=-0.01)])
def test_lamb_rejects_invalid_hyper_parameters(kw):
    with pytest.raises(ValueError):
        Lamb([torch.nn.Parameter(torch.zeros(2))], **kw)


def test_lamb_is_exported():
    import horovod_b200.torch as hvd
    assert hvd.Lamb is Lamb
