"""The fp32 weight EMA of the fused and sharded (ZeRO-1) optimizers (`hvd.DistributedOptimizer(..., ema_decay=d)`):
the kernels' EMA epilogue against an fp64 model of its fp32 arithmetic, the optimizer against torch's optimizers with
an fp64 EMA, GradScaler / clipping / GraphedStep / checkpoints / ema_parameters(), and the sharded EMA on 4 simulated
ranks against the unsharded one."""
import contextlib
import copy

import pytest
import torch

from conftest import run_parallel
from optim_cases import (LOW, LOW_IDS, PAIR_IDS, PAIRS, COUNTS, Slot, hvd, make_optimizer, mlp, mlp_loss, ngpu,  # noqa: F401
                         same, ulp)
from sim_ranks import FakeSet, NormConvNet, batch, reduced_grads, ref_step, sharded_team, team  # noqa: F401

pytestmark = pytest.mark.gpu

KINDS = ['sgd', 'adam', 'lamb', 'lars']
DECAY = 0.75


# ---- kernels ------------------------------------------------------------------------------------------------------------
def _cases(pdt, gdt, master, offset, seed=0):
    """One table entry per COUNTS size, each tensor at element `offset` of its own buffer (offset 1: unaligned views)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    out = []
    for n in COUNTS:
        w = torch.randn(n, device='cuda', generator=g) * 0.5
        sdt = torch.float32 if master or pdt == torch.float32 else pdt
        c = {'p': Slot((n,), pdt, offset, w.to(pdt)),
             'g': Slot((n,), gdt, offset, (torch.randn(n, device='cuda', generator=g) * 0.1).to(gdt)),
             'm': Slot((n,), torch.float32, offset, torch.randn(n, device='cuda', generator=g) * 0.01),
             'v': Slot((n,), torch.float32, offset, torch.rand(n, device='cuda', generator=g) * 0.01),
             's': Slot((n,), sdt, offset, (torch.randn(n, device='cuda', generator=g) * 0.01).to(sdt)),
             'e': Slot((n,), torch.float32, offset, torch.randn(n, device='cuda', generator=g))}
        if master:
            c['w'] = Slot((n,), torch.float32, offset, w)
        out.append(c)
    return out


def _launch(kind, cases, master, ema=None, start=False):
    """One fused update of `kind` over the cases (with the EMA of every case when `ema` is a decay)."""
    from horovod_b200 import ops
    L = lambda k: [c[k].t for c in cases]  # noqa: E731
    kw = dict(master_params=L('w') if master else None)
    if ema is not None:
        kw.update(ema_params=L('e'), ema_decay=ema, ema_start=start)
    if kind == 'sgd':
        ops.fused_sgd_step(L('p'), L('g'), L('s'), 0.1, 0.9, 0.1, 1e-2, nesterov=True, **kw)
    elif kind == 'adam':
        ops.fused_adam_step(L('p'), L('g'), L('m'), L('v'), 1e-2, weight_decay=0.01, step=3, **kw)
    elif kind == 'lamb':
        ops.fused_lamb_step(L('p'), L('g'), L('m'), L('v'), 1e-2, 0.9, 0.999, 1e-6, 0.01, 3, **kw)
    else:
        ops.fused_lars_step(L('p'), L('g'), L('m'), 0.5, 0.9, 1e-4, 1e-3, 0.0, **kw)


def _x(c, master):
    """The value the EMA averages: the updated master, or the value stored into the parameter."""
    return (c['w'].t if master else c['p'].t).double()


def _ema_model(e, x, decay):
    """fp64 model of e = fmaf(w, x - e, e) in fp32 with w = float32(1 - decay): x - e and w are exact fp32 values, their
    product is exact in fp64, and the one rounding of fmaf is that of the fp64 sum except at a double-rounding tie."""
    w = torch.tensor(1.0 - decay, dtype=torch.float64).float().double()
    d = (x.float() - e.float()).double()
    return (w * d + e.double()).float()


def _params(kinds_pairs):
    out = []
    for kind in KINDS:
        for (pdt, gdt), pid in zip(PAIRS, PAIR_IDS):
            for master in ([False, True] if pdt != torch.float32 else [False]):
                out.append(pytest.param(kind, pdt, gdt, master, id='%s-%s%s' % (kind, pid, '-master' if master else '')))
    return out


@pytest.mark.parametrize("offset", [0, 1], ids=['aligned', 'offset1'])
@pytest.mark.parametrize("kind,pdt,gdt,master", _params(KINDS))
def test_kernel_ema_against_fp64_model(hvd, kind, pdt, gdt, master, offset):
    """Two updates with the EMA against the same two without: the parameter, the states and the master are bit-identical;
    the first update (start) stores e = x bit for bit; the second is the fp64 model of fmaf(w, x - e, e); nothing
    outside the views is written."""
    a, b = _cases(pdt, gdt, master, offset), _cases(pdt, gdt, master, offset)
    _launch(kind, a, master)
    _launch(kind, b, master, ema=DECAY, start=True)
    for ca, cb in zip(a, b):
        for k in ca:
            if k != 'e':
                assert same(ca[k].t, cb[k].t), (k, ca[k].t.numel())
        assert same(cb['e'].t, _x(cb, master).float()), 'the EMA begins at the updated fp32 value'
    prev = [c['e'].t.clone() for c in b]
    _launch(kind, a, master)
    _launch(kind, b, master, ema=DECAY)
    for ca, cb, e0 in zip(a, b, prev):
        for k in ca:
            if k != 'e':
                assert same(ca[k].t, cb[k].t), (k, ca[k].t.numel())
        model = _ema_model(e0, _x(cb, master), DECAY)
        err = (cb['e'].t.double() - model.double()).abs()
        assert bool((err <= ulp(model.double(), torch.float32)).all()), 'one fp32 rounding of the fp64 model'
        assert (err == 0).float().mean() > 0.99
        assert all(c.intact() for c in cb.values())


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dt", LOW, ids=LOW_IDS)
def test_master_ema_equals_fp32_twin(hvd, kind, dt):
    """With masters the update and the EMA run on the master with the fp32 arithmetic: three steps of a bf16 / fp16 run
    give the EMA of the fp32-parameter run on the same values, bit for bit."""
    low = _cases(dt, dt, True, 0, seed=3)
    f32 = _cases(torch.float32, torch.float32 if dt == torch.float16 else torch.bfloat16, False, 0, seed=3)
    for cl, cf in zip(low, f32):
        cf['p'].t.copy_(cl['w'].t)
        cf['g'].t.copy_(cl['g'].t.float())
        cf['s'].t.copy_(cl['s'].t)
        for k in ('m', 'v', 'e'):
            cf[k].t.copy_(cl[k].t)
    for i in range(3):
        _launch(kind, low, True, ema=DECAY, start=i == 0)
        _launch(kind, f32, False, ema=DECAY, start=i == 0)
    for cl, cf in zip(low, f32):
        assert same(cl['w'].t, cf['p'].t)
        assert same(cl['e'].t, cf['e'].t)


@pytest.mark.parametrize("kind", KINDS)
def test_ema_adds_no_launch_and_no_host_sync(hvd, kind):
    from horovod_b200 import ops
    counts = []
    for ema in (None, DECAY):
        cases = _cases(torch.bfloat16, torch.bfloat16, True, 0)
        torch.cuda.synchronize()
        before = ops.kernel_launches()
        torch.cuda.set_sync_debug_mode('error')
        try:
            _launch(kind, cases, True, ema=ema, start=True)
        finally:
            torch.cuda.set_sync_debug_mode('default')
        counts.append(ops.kernel_launches() - before)
    assert counts[0] == counts[1] == (1 if kind in ('sgd', 'adam') else 3)


def test_kernel_ema_argument_errors(hvd):
    from horovod_b200 import ops
    c = _cases(torch.float32, torch.float32, False, 0)[:2]
    p, g, s = [x['p'].t for x in c], [x['g'].t for x in c], [x['s'].t for x in c]
    e = [x['e'].t for x in c]
    for bad in ([e[0]], [e[0].half(), e[1]], [e[0], torch.zeros(4, device='cuda')], [e[0], e[1].cpu()],
                [e[0], torch.zeros(2 * e[1].numel(), device='cuda')[::2]]):
        with pytest.raises(RuntimeError):
            ops.fused_sgd_step(p, g, s, 0.1, 0.9, ema_params=bad, ema_decay=0.5)
    for d in (None, -0.1, 1.5):
        with pytest.raises(ValueError):
            ops.fused_sgd_step(p, g, s, 0.1, 0.9, ema_params=e, ema_decay=d)


# ---- the optimizer at world size 1 ----------------------------------------------------------------------------------------
def _opt(hvd, kind, m, dt, **kw):
    return hvd.DistributedOptimizer(make_optimizer(hvd, kind, m.parameters()), named_parameters=m.named_parameters(),
                                    master_weights=dt != torch.float32, **kw)


def _ema_of(opt, m):
    return [opt.state[p]['ema_param'] for p in m.parameters()]


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=['f32', 'bf16-master'])
@pytest.mark.parametrize("kind", ['sgd', 'adamw', 'lamb', 'lars'])
def test_optimizer_ema_against_torch_and_fp64_ema(hvd, kind, dt):
    """20 steps with a decay change after step 10: the fused EMA follows the same torch optimizer (hvd.Lamb / hvd.Lars
    eager steps) on fp32 weights fed the same gradients, followed by an fp64 EMA of its weights.  The gap is the fp32
    rounding of the two trajectories (and, with bf16, the bf16 rounding of the forward that made the gradients, which
    both sides share)."""
    m = mlp(dt)
    opt = _opt(hvd, kind, m, dt, ema_decay=0.9)
    ref = mlp(torch.float32)
    with torch.no_grad():
        for a, b in zip(ref.parameters(), m.parameters()):
            a.copy_(b.float())
    ref_opt = make_optimizer(hvd, kind, ref.parameters())
    ema64 = None
    decay = 0.9
    for step in range(20):
        if step == 10:
            decay = 0.6
            for g in opt.param_groups:
                g['ema_decay'] = decay
        opt.zero_grad()
        mlp_loss(m, step, dt).backward()
        opt.synchronize()
        for a, b in zip(ref.parameters(), m.parameters()):
            a.grad = b.grad.float().clone()
        with opt.skip_synchronize():
            opt.step()
        ref_opt.step()
        x = [p.detach().double() for p in ref.parameters()]
        ema64 = x if ema64 is None else [e + (1 - decay) * (xi - e) for e, xi in zip(ema64, x)]
    tol = dict(rtol=1e-4, atol=1e-5) if dt == torch.float32 else dict(rtol=2e-3, atol=2e-4)
    for e, r in zip(_ema_of(opt, m), ema64):
        assert e.dtype == torch.float32
        torch.testing.assert_close(e.double(), r, **tol)


def test_sgd_ema_against_averaged_model(hvd):
    """fp32 SGD with momentum: the fused EMA against torch's AveragedModel + get_ema_multi_avg_fn on torch's SGD, within
    1e-5 relative / 1e-6 absolute (fp32 rounding of two trajectories of 20 steps)."""
    from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn
    m = mlp(torch.float32)
    opt = _opt(hvd, 'sgd', m, torch.float32, ema_decay=0.9)
    ref = copy.deepcopy(m)
    ref_opt = make_optimizer(hvd, 'sgd', ref.parameters())
    avg = AveragedModel(ref, multi_avg_fn=get_ema_multi_avg_fn(0.9))
    for step in range(20):
        if step == 10:
            avg.multi_avg_fn = get_ema_multi_avg_fn(0.6)
            for g in opt.param_groups:
                g['ema_decay'] = 0.6
        opt.zero_grad()
        mlp_loss(m, step, torch.float32).backward()
        opt.synchronize()
        for a, b in zip(ref.parameters(), m.parameters()):
            a.grad = b.grad.clone()
        with opt.skip_synchronize():
            opt.step()
        ref_opt.step()
        avg.update_parameters(ref)
    for e, r in zip(_ema_of(opt, m), avg.module.parameters()):
        torch.testing.assert_close(e, r.detach(), rtol=1e-5, atol=1e-6)


def test_optimizer_ema_off_and_on_state(hvd):
    """EMA off leaves no 'ema_param'; EMA on adds no launch to a step and leaves the parameters and the other state
    bit-identical to the run without it."""
    from horovod_b200 import ops
    runs = []
    for ema in (None, 0.99):
        m = mlp(torch.bfloat16)
        opt = _opt(hvd, 'adamw', m, torch.bfloat16, ema_decay=ema)
        launches = []
        for step in range(3):
            opt.zero_grad()
            mlp_loss(m, step, torch.bfloat16).backward()
            opt.synchronize()
            torch.cuda.synchronize()
            before = ops.kernel_launches()
            with opt.skip_synchronize():
                opt.step()
            launches.append(ops.kernel_launches() - before)
        runs.append((m, opt, launches))
    (m0, o0, l0), (m1, o1, l1) = runs
    assert l0 == l1
    for a, b in zip(m0.parameters(), m1.parameters()):
        assert same(a.detach(), b.detach())
        assert 'ema_param' not in o0.state[a] and 'ema_param' in o1.state[b]
        for key in o0.state[a]:
            if torch.is_tensor(o0.state[a][key]) and o0.state[a][key].is_cuda:
                assert same(o0.state[a][key], o1.state[b][key]), key


def test_parameter_without_gradient_does_not_advance(hvd):
    m = mlp(torch.float32)
    opt = _opt(hvd, 'sgd', m, torch.float32, ema_decay=0.5, zero_copy=False)
    ps = list(m.parameters())
    opt.zero_grad()
    mlp_loss(m, 0, torch.float32).backward()
    opt.step()
    e0 = [e.clone() for e in _ema_of(opt, m)]
    opt.zero_grad()
    mlp_loss(m, 1, torch.float32).backward()
    opt.synchronize()
    ps[0].grad = None
    with opt.skip_synchronize():
        opt.step()
    assert same(opt.state[ps[0]]['ema_param'], e0[0]), 'no gradient: no update, no EMA step'
    assert not same(opt.state[ps[1]]['ema_param'], e0[1])


def test_grad_scaler_skip_and_clipping(hvd):
    """A GradScaler and clip_grad_norm_: a step the scaler skips leaves the EMA bit for bit; a clipped step moves it to
    fmaf(w, x - e, e) with x the clipped update's parameter."""
    m = mlp(torch.float32)
    opt = _opt(hvd, 'adamw', m, torch.float32, ema_decay=DECAY)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 8)
    for step in range(4):
        opt.zero_grad()
        scaler.scale(mlp_loss(m, step, torch.float32)).backward()
        opt.synchronize()
        if step == 2:
            next(m.parameters()).grad.view(-1)[0] = float('inf')
        scaler.unscale_(opt)
        opt.clip_grad_norm_(1e-3)
        e0 = [e.clone() for e in _ema_of(opt, m)] if step else None
        with opt.skip_synchronize():
            scaler.step(opt)
        scaler.update()
        if step == 2:
            assert all(same(a, b) for a, b in zip(_ema_of(opt, m), e0)), 'a skipped step does not advance the EMA'
        elif step:
            for p, e, prev in zip(m.parameters(), _ema_of(opt, m), e0):
                model = _ema_model(prev, p.detach().double(), DECAY)
                assert bool(((e.double() - model.double()).abs() <= ulp(model.double(), torch.float32)).all())


def _graphed_run(hvd, kind, dt, acc, k, graphed, steps=3):
    m = mlp(dt)
    opt = _opt(hvd, kind, m, dt, ema_decay=0.9, fused=True, backward_passes_per_step=k,
               grad_accumulation_dtype=torch.float32 if acc else None)
    gen = torch.Generator(device='cuda').manual_seed(2)
    xs = [torch.randn(16, 24, device='cuda', generator=gen).to(dt) for _ in range(steps * k)]
    fn = lambda x: m(x).float().square().mean() / k  # noqa: E731
    if graphed:
        step = hvd.GraphedStep(fn, opt, (xs[0],))
        assert step.captured, step.fallback_reason
        for x in xs:
            step(x)
    else:
        for i, x in enumerate(xs):
            if i % k == 0:
                opt.zero_grad(set_to_none=False)
            fn(x).backward()
            if i % k == k - 1:
                opt.step()
    torch.cuda.synchronize()
    return m, opt


@pytest.mark.parametrize("case", [('sgd', torch.float32, False, 1), ('lars', torch.float32, False, 1),
                                  ('adamw', torch.bfloat16, True, 4), ('lamb', torch.bfloat16, True, 4)],
                         ids=['sgd-k1', 'lars-k1', 'adamw-bf16-acc32-k4', 'lamb-bf16-acc32-k4'])
def test_graphed_step_equals_eager_loop(hvd, monkeypatch, case):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    kind, dt, acc, k = case
    (a, oa), (b, ob) = [_graphed_run(hvd, kind, dt, acc, k, graphed) for graphed in (False, True)]
    for p, q in zip(a.parameters(), b.parameters()):
        assert same(p.detach(), q.detach())
        assert same(oa.state[p]['ema_param'], ob.state[q]['ema_param'])


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=['f32', 'bf16-master'])
def test_ema_parameters_block(hvd, dt):
    """Inside: every parameter is its EMA rounded to its dtype, in its own storage, and model.state_dict() is the EMA
    model; step() raises.  On exit: parameters, masters, moments and EMA are bit-identical to their values on entry."""
    m = mlp(dt)
    opt = _opt(hvd, 'adamw', m, dt, ema_decay=0.5)
    for step in range(3):
        opt.zero_grad()
        mlp_loss(m, step, dt).backward()
        opt.step()
    ps = list(m.parameters())
    before = [p.detach().clone() for p in ps]
    state = [{k: v.clone() for k, v in opt.state[p].items() if torch.is_tensor(v)} for p in ps]
    ptrs = [p.data_ptr() for p in ps]
    assert not all(same(p.detach(), opt.state[p]['ema_param'].to(dt)) for p in ps)
    with opt.ema_parameters():
        for p in ps:
            assert same(p.detach(), opt.state[p]['ema_param'].to(dt))
        assert [p.data_ptr() for p in ps] == ptrs
        sd = m.state_dict()
        assert all(same(sd[name], opt.state[p]['ema_param'].to(dt)) for name, p in m.named_parameters())
        with pytest.raises(RuntimeError):
            opt.step()
    for p, b, st in zip(ps, before, state):
        assert same(p.detach(), b)
        for k, v in st.items():
            assert same(opt.state[p][k], v), k


def test_checkpoint_round_trip_keeps_fp32_ema(hvd):
    """bf16 parameters: the checkpoint's fp32 EMA comes back as fp32 bit for bit, and both runs continue alike."""
    import io
    m = mlp(torch.bfloat16)
    opt = _opt(hvd, 'sgd', m, torch.bfloat16, ema_decay=0.99)
    for step in range(3):
        opt.zero_grad()
        mlp_loss(m, step, torch.bfloat16).backward()
        opt.step()
    buf = io.BytesIO()
    torch.save(opt.state_dict(), buf)
    m2 = copy.deepcopy(m)
    opt2 = _opt(hvd, 'sgd', m2, torch.bfloat16, ema_decay=0.99)
    opt2.load_state_dict(torch.load(io.BytesIO(buf.getvalue())))
    for p, q in zip(m.parameters(), m2.parameters()):
        assert opt2.state[q]['ema_param'].dtype == torch.float32
        assert same(opt.state[p]['ema_param'], opt2.state[q]['ema_param'])
    for mm, oo in ((m, opt), (m2, opt2)):
        oo.zero_grad()
        mlp_loss(mm, 3, torch.bfloat16).backward()
        oo.step()
    for p, q in zip(m.parameters(), m2.parameters()):
        assert same(opt.state[p]['ema_param'], opt2.state[q]['ema_param'])


def test_broadcast_optimizer_state_does_not_start_the_ema(hvd):
    m = mlp(torch.float32)
    opt = _opt(hvd, 'adamw', m, torch.float32, ema_decay=0.5)
    hvd.broadcast_optimizer_state(opt, root_rank=0)
    assert not any('ema_param' in opt.state[p] for p in m.parameters())


def test_argument_and_plan_errors(hvd):
    m = mlp(torch.float32)
    for d in (-0.01, 1.01, 'x', True, float('nan')):
        with pytest.raises(ValueError):
            _opt(hvd, 'sgd', m, torch.float32, ema_decay=d)
    with pytest.raises(ValueError):
        _opt(hvd, 'sgd', m, torch.float32, ema_decay=0.9, op=hvd.Adasum)
    with pytest.raises(ValueError):
        hvd.DistributedOptimizer(torch.optim.RMSprop(m.parameters()), named_parameters=m.named_parameters(), ema_decay=0.9)
    for opt in (torch.optim.SGD(m.parameters(), lr=0.1, maximize=True), torch.optim.Adam(m.parameters(), amsgrad=True)):
        with pytest.raises(ValueError):
            hvd.DistributedOptimizer(opt, named_parameters=m.named_parameters(), ema_decay=0.9)
    for d in (0.0, 1.0):
        assert _opt(hvd, 'sgd', mlp(torch.float32), torch.float32, ema_decay=d)._fused
    # a plan that cannot be fused at step time: CPU parameters
    cpu = torch.nn.Linear(4, 4)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(cpu.parameters(), lr=0.1), named_parameters=cpu.named_parameters(),
                                   ema_decay=0.9)
    cpu(torch.randn(2, 4)).sum().backward()
    with pytest.raises(RuntimeError):
        opt.step()
    # a scheduled decay out of range
    m = mlp(torch.float32)
    opt = _opt(hvd, 'sgd', m, torch.float32, ema_decay=0.9)
    opt.param_groups[0]['ema_decay'] = 2.0
    mlp_loss(m, 0, torch.float32).backward()
    with pytest.raises(ValueError):
        opt.step()
    with pytest.raises(RuntimeError):
        with _opt(hvd, 'sgd', mlp(torch.float32), torch.float32).ema_parameters():
            pass


# ---- 4 simulated ranks ---------------------------------------------------------------------------------------------------
def _make(kind):
    def make(m):
        decay = [p for p in m.parameters() if p.dim() > 1]
        rest = [p for p in m.parameters() if p.dim() <= 1]
        groups = [{'params': decay}, {'params': rest, 'weight_decay': 0.0}]
        if kind == 'sgd':
            return torch.optim.SGD(groups, lr=0.05, momentum=0.9, weight_decay=1e-3)
        if kind == 'adamw':
            return torch.optim.AdamW(groups, lr=1e-2, weight_decay=0.01)
        if kind == 'lamb':
            return hvd_module().Lamb(groups, lr=1e-2, weight_decay=0.01)
        return hvd_module().Lars(groups, lr=0.5, momentum=0.9, weight_decay=1e-3, trust_coefficient=0.02)
    return make


def hvd_module():
    import horovod_b200.torch as h
    return h


def _team_step(team, models, opts, step, dt):
    for r in range(team.n):
        opts[r].zero_grad()
        x, y = batch(step, r, dt)
        torch.nn.functional.cross_entropy(models[r](x), y).backward()
    for o in opts:
        o.synchronize()
    team.flush()
    grads = reduced_grads(opts, list(models[0].parameters()))

    def step_rank(r):
        with opts[r].skip_synchronize():
            opts[r].step()
    team.run(step_rank)
    return grads


def _check(models, opts, ref, ref_opt, what):
    sd = opts[0].state_dict()
    for r in range(len(models)):
        for (name, a), b in zip(models[r].named_parameters(), ref.parameters()):
            assert same(a.detach(), b.detach()), (what, name, r)
    for i, b in enumerate(_in_group_order(ref_opt)):  # the checkpoint's parameter index
        assert same(sd['state'][i]['ema_param'].cuda(), ref_opt.state[b]['ema_param']), (what, i)
    return sd


def _in_group_order(opt):
    return [p for g in opt.param_groups for p in g['params']]


def _ema_launch(x, e, decay, start):
    """The unsharded EMA epilogue alone: an SGD launch with lr 0 leaves x as it is and moves e toward it."""
    from horovod_b200 import ops
    ops.fused_sgd_step([x.clone()], [torch.zeros_like(x)], [], 0.0, ema_params=[e], ema_decay=decay, ema_start=start)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=['f32', 'bf16-master'])
@pytest.mark.parametrize("kind", ['sgd', 'adamw', 'lamb', 'lars'])
def test_sharded_ema_equals_unsharded(hvd, team, kind, dt):
    """After every step the gathered sharded EMA of every parameter equals, bit for bit, the unsharded EMA epilogue fed
    that parameter's sharded trajectory (the master with master weights); the EMA shard is 1/N of the bucket.  SGD and
    AdamW also equal a world-size-1 optimizer fed the reduced gradients bit for bit; LAMB's and LARS's trust-ratio norms
    are summed over the ranks in another order, so their trajectories agree to the tolerance of the sharded LAMB / LARS
    tests.  Then checkpoints sharded -> unsharded -> sharded carry the EMA exactly and continue alike."""
    torch.manual_seed(0)
    base = NormConvNet().cuda().to(dt)
    master = dt != torch.float32
    kw = dict(ema_decay=0.8, master_weights=master)
    exact = kind in ('sgd', 'adamw')
    tol = dict(rtol=1e-5, atol=1e-6) if dt == torch.float32 else dict(rtol=1e-2, atol=1e-3)
    models, opts = sharded_team(hvd, team, base, _make(kind), dt, min_buckets=2, straddle=not exact, **kw)
    for b in opts[0]._buckets:
        assert b['state']['ema_param'].numel() == b['shard'] == b['numel'] // team.n
    ref = copy.deepcopy(base)
    ref_opt = hvd.DistributedOptimizer(_make(kind)(ref), named_parameters=ref.named_parameters(), zero_copy=False, **kw)
    group_of = [gi for gi, g in enumerate(opts[0].param_groups) for _ in g['params']]
    mirror = None
    for step in range(4):
        if step == 2:
            for o in opts + [ref_opt]:
                o.param_groups[0]['ema_decay'] = 0.5
        ref_step(ref, ref_opt, _team_step(team, models, opts, step, dt))
        sd = opts[0].state_dict()
        xs = [sd['state'][i]['master_param'].cuda() if master else p.detach().float()
              for i, p in enumerate(_in_group_order(opts[0]))]
        if mirror is None:
            mirror = [torch.empty_like(x) for x in xs]
        for x, e, gi in zip(xs, mirror, group_of):
            _ema_launch(x, e, opts[0].param_groups[gi]['ema_decay'], step == 0)
        for i, e in enumerate(mirror):
            assert same(sd['state'][i]['ema_param'].cuda(), e), ('step %d' % step, i)
        if exact:
            _check(models, opts, ref, ref_opt, 'step %d' % step)
        else:
            for i, b in enumerate(_in_group_order(ref_opt)):
                torch.testing.assert_close(sd['state'][i]['ema_param'].cuda(), ref_opt.state[b]['ema_param'], **tol)
    # sharded -> unsharded: the EMA comes back exactly
    un = copy.deepcopy(models[0])
    un_opt = hvd.DistributedOptimizer(_make(kind)(un), named_parameters=un.named_parameters(), zero_copy=False, **kw)
    un_opt.load_state_dict(copy.deepcopy(sd))
    for i, p in enumerate(_in_group_order(un_opt)):
        assert un_opt.state[p]['ema_param'].dtype == torch.float32
        assert same(un_opt.state[p]['ema_param'], sd['state'][i]['ema_param'].cuda())
    # unsharded -> sharded: a fresh team loads the unsharded checkpoint and continues like the unsharded optimizer
    models2, opts2 = sharded_team(hvd, team, un, _make(kind), dt, **kw)
    for o in opts2:
        o.load_state_dict(un_opt.state_dict())
    ref_step(un, un_opt, _team_step(team, models2, opts2, 4, dt))
    sd2 = opts2[0].state_dict()
    for i, p in enumerate(_in_group_order(un_opt)):
        if exact:
            assert same(sd2['state'][i]['ema_param'].cuda(), un_opt.state[p]['ema_param']), i
        else:
            torch.testing.assert_close(sd2['state'][i]['ema_param'].cuda(), un_opt.state[p]['ema_param'], **tol)


def test_sharded_ema_parameters(hvd, team):
    """ema_parameters() on every rank: each holds the whole EMA model (rounded to bf16) and, after the block, its exact
    parameters, masters and EMA again; step() inside raises."""
    torch.manual_seed(0)
    dt = torch.bfloat16
    base = NormConvNet().cuda().to(dt)
    models, opts = sharded_team(hvd, team, base, _make('adamw'), dt, min_buckets=2, ema_decay=0.5, master_weights=True)
    for step in range(3):
        _team_step(team, models, opts, step, dt)
    sd = opts[0].state_dict()
    before = [[p.detach().clone() for p in m.parameters()] for m in models]
    shards = [[{k: v.clone() for k, v in b['state'].items()} for b in o._buckets] for o in opts]
    with contextlib.ExitStack() as stack:
        for o in opts:
            stack.enter_context(o.ema_parameters())
        team.flush()
        for o in opts:
            for i, p in enumerate(_in_group_order(o)):
                assert same(p.detach(), sd['state'][i]['ema_param'].cuda().to(dt))
        with pytest.raises(RuntimeError):
            opts[0].step()
    team.flush()
    for m, b in zip(models, before):
        assert all(same(p.detach(), q) for p, q in zip(m.parameters(), b))
    for o, st in zip(opts, shards):
        for bk, s in zip(o._buckets, st):
            assert all(same(bk['state'][k], v) for k, v in s.items())


@pytest.mark.skipif(ngpu() < 2, reason="needs >= 2 GPUs")
def test_sharded_ema_across_ranks(native_built):
    n = 2 if ngpu() < 4 else 4
    rc, out = run_parallel("ema_worker.py", np=n, timeout=420)
    assert "EMA OK" in out, out[-4000:]
