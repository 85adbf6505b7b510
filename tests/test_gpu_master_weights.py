"""fp32 master weights for bf16 / fp16 parameters (`master_params` of the fused kernels, `master_weights=True` of
hvd.DistributedOptimizer, unsharded and sharded).

* The master kernels against the existing fp32-parameter kernels, bit for bit: the master update is the fp32 update.
* The reconcile rule: parameter elements written from outside the optimizer restart their masters, the others keep them.
* The capability: a bf16 update below half an ulp is kept, and a bf16 AdamW model tracks fp32 AdamW.
* The optimizer at world size 1 (closure, frozen parameters, hvd.GraphedStep, checkpoints, errors) and on 4 simulated
  ranks of the sharded (ZeRO-1) optimizer against a world-size-1 master-weights optimizer fed the reduced gradient.
"""
import copy
import io
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import run_parallel
from optim_cases import COUNTS, LOW, LOW_IDS, Slot, adam_ref_kernel, bits, hvd, ngpu, same  # noqa: F401  (hvd: fixture)
from sim_ranks import batch, reduced_grads, ref_step, sharded_team, team  # noqa: F401  (team: fixture)

pytestmark = pytest.mark.gpu

# (param, grad, state) storage offsets in elements; the master and the state share the last one
OFFSETS = [(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (2, 0, 0), (0, 2, 2), (3, 3, 3), (0, 3, 0), (3, 0, 2)]
SGD_HP = [dict(lr=0.05, momentum=0.9, dampening=0.5, weight_decay=1e-2, grad_scale=0.25),
          dict(lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-2),
          dict(lr=0.05, weight_decay=1e-2), dict(lr=0.05)]
ADAM_HP = [dict(lr=1e-2, weight_decay=1e-2, adamw=True), dict(lr=1e-2, weight_decay=1e-2, adamw=False, eps=1e-3),
           dict(lr=1e-3, weight_decay=0.0, adamw=True, beta1=0.8, beta2=0.99, grad_scale=0.5)]


# ---- the kernels against the fp32-parameter kernels ------------------------------------------------------------------
def _case(shape, pdt, seed, offsets=(0, 0, 0), memory_format=torch.contiguous_format, sgd=False):
    """Master-mode slots (param pdt, grad pdt, fp32 master and state) with p == round(master): no reconcile."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    po, go, so = offsets
    rnd = lambda s: torch.randn(shape, device='cuda', generator=g) * s  # noqa: E731
    master = rnd(0.1)
    sl = {'w': Slot(shape, torch.float32, so, master, memory_format), 'p': Slot(shape, pdt, po, master.to(pdt), memory_format),
          'g': Slot(shape, pdt, go, rnd(1.0), memory_format)}
    if sgd:
        sl['buf'] = Slot(shape, torch.float32, so + 1, rnd(0.5), memory_format)
    else:
        sl['m'] = Slot(shape, torch.float32, so + 1, rnd(0.1), memory_format)
        sl['v'] = Slot(shape, torch.float32, so + 2, rnd(0.1).square(), memory_format)
    return sl


def _ref_grad(g):
    """The gradient the fp32-parameter kernel reads: bf16 as it is (the fp32 / bf16 instantiation), fp16 upcast to fp32
    (exact)."""
    return g if g.dtype == torch.bfloat16 else g.float()


def _kernel_vs_fp32(cases, pdt, sgd, expect_master=None, **hp):
    """One master launch over `cases` and one fp32-parameter launch over copies; masters, states and parameters must be
    bit-identical. expect_master: the masters the update starts from (default: the current ones)."""
    from horovod_b200 import ops
    start = expect_master or [c['w'].t.clone() for c in cases]
    ref_p = [s.clone() for s in start]
    ref_g = [_ref_grad(c['g'].t).clone() for c in cases]
    keys = ('buf',) if sgd else ('m', 'v')
    ref_s = {k: [c[k].t.clone() for c in cases] for k in keys}
    before_g = [c['g'].t.clone() for c in cases]
    gsd = hp.pop('grad_scale_dev', None)
    if sgd:
        mom = [c['buf'].t for c in cases] if hp.get('momentum', 0.0) else []
        ops.fused_sgd_step([c['p'].t for c in cases], [c['g'].t for c in cases], mom, grad_scale_dev=gsd,
                           master_params=[c['w'].t for c in cases], **hp)
        ops.fused_sgd_step(ref_p, ref_g, ref_s['buf'] if mom else [], grad_scale_dev=gsd, **hp)
    else:
        hp = dict(hp)
        ops.fused_adam_step([c['p'].t for c in cases], [c['g'].t for c in cases], [c['m'].t for c in cases],
                            [c['v'].t for c in cases], grad_scale_dev=gsd, master_params=[c['w'].t for c in cases], **hp)
        ops.fused_adam_step(ref_p, ref_g, ref_s['m'], ref_s['v'], grad_scale_dev=gsd, **hp)
    torch.cuda.synchronize()
    for i, c in enumerate(cases):
        assert same(c['w'].t, ref_p[i]), (i, 'master')
        assert same(c['p'].t, ref_p[i].to(pdt)), (i, 'param is not the rounded master')
        for k in keys:
            assert same(c[k].t, ref_s[k][i]), (i, k)
        assert same(c['g'].t, before_g[i]), (i, 'grad written')
        for k, s in c.items():
            assert s.intact(), (i, 'wrote outside ' + k)


@pytest.mark.parametrize("pdt", LOW, ids=LOW_IDS)
@pytest.mark.parametrize("count", COUNTS)
def test_master_kernels_equal_fp32_kernels(hvd, pdt, count):
    c = [_case((count,), pdt, seed=count, sgd=True)]
    _kernel_vs_fp32(c, pdt, True, first_step=True, **SGD_HP[0])
    for hp in SGD_HP:
        _kernel_vs_fp32(c, pdt, True, **hp)
    c = [_case((count,), pdt, seed=count + 1)]
    for step, hp in enumerate(ADAM_HP, 1):
        _kernel_vs_fp32(c, pdt, False, step=step, **hp)


@pytest.mark.parametrize("pdt", LOW, ids=LOW_IDS)
@pytest.mark.parametrize("offsets", OFFSETS, ids=['p%dg%ds%d' % o for o in OFFSETS])
def test_master_kernels_unaligned_views(hvd, pdt, offsets):
    for count in (5, 4097):
        _kernel_vs_fp32([_case((count,), pdt, seed=count, offsets=offsets, sgd=True)], pdt, True, **SGD_HP[1])
        _kernel_vs_fp32([_case((count,), pdt, seed=count, offsets=offsets)], pdt, False, step=4, **ADAM_HP[0])


@pytest.mark.parametrize("pdt", LOW, ids=LOW_IDS)
def test_master_kernels_many_tensors_channels_last_and_device_scale(hvd, pdt):
    rng = np.random.default_rng(5)
    sizes = [1, 2, 3, 4, 5, 7, 8, 4095, 4096, 4097, 1 << 20] + [int(x) for x in rng.integers(1, 70000, size=190)]
    offs = [(i % 4, (i // 4) % 4, (i // 16) % 4) for i in range(len(sizes))]
    before = hvd.runtime_stats()['kernel_launches']
    sgd = [_case((n,), pdt, seed=i, offsets=o, sgd=True) for i, (n, o) in enumerate(zip(sizes, offs))]
    _kernel_vs_fp32(sgd, pdt, True, **SGD_HP[0])
    adam = [_case((n,), pdt, seed=i, offsets=o) for i, (n, o) in enumerate(zip(sizes, offs))]
    _kernel_vs_fp32(adam, pdt, False, step=7, **ADAM_HP[1])
    assert hvd.runtime_stats()['kernel_launches'] - before == 4  # one master and one fp32 launch each
    cl = torch.channels_last
    for i, shape in enumerate([(64, 32, 3, 3), (7, 5, 3, 3), (8, 3, 1, 1)]):
        c = _case(shape, pdt, seed=i, offsets=(i, 0, i), memory_format=cl, sgd=True)
        assert c['p'].t.is_contiguous(memory_format=cl) and c['w'].t.stride() == c['p'].t.stride()
        _kernel_vs_fp32([c], pdt, True, **SGD_HP[1])
        _kernel_vs_fp32([_case(shape, pdt, seed=i, memory_format=cl)], pdt, False, step=2, **ADAM_HP[0])
    coef = torch.tensor([0.37], device='cuda')
    _kernel_vs_fp32([_case((4097,), pdt, seed=9, sgd=True)], pdt, True, grad_scale_dev=coef, **SGD_HP[0])
    _kernel_vs_fp32([_case((4097,), pdt, seed=9)], pdt, False, step=3, grad_scale_dev=coef, **ADAM_HP[2])


# ---- reconcile ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pdt", LOW, ids=LOW_IDS)
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_reconcile_restarts_exactly_the_overwritten_elements(hvd, pdt, kind):
    sgd = kind == 'sgd'
    hp = dict(SGD_HP[1]) if sgd else dict(step=2, **ADAM_HP[0])
    cases = [_case((n,), pdt, seed=n, offsets=(n % 4, 0, 1), sgd=sgd) for n in (5, 4097, 70001)]
    _kernel_vs_fp32(cases, pdt, sgd, **dict(hp, first_step=True) if sgd else hp)
    # the masters now carry sub-ulp information: p == round(master), master != p in most elements
    assert any(not torch.equal(c['w'].t, c['p'].t.float()) for c in cases)
    g = torch.Generator(device='cuda').manual_seed(3)
    expect = []
    for i, c in enumerate(cases):
        w, p = c['w'].t, c['p'].t
        if i == 0:
            idx = torch.arange(p.numel(), device='cuda')  # the whole tensor
        else:
            idx = torch.randperm(p.numel(), device='cuda', generator=g)[:p.numel() // 7]
        new = (p[idx].float() + 4.0).to(pdt)  # |p| < 1: every element changes
        assert not (bits(new) == bits(p[idx])).any()
        p[idx] = new
        e = w.clone()
        e[idx] = new.float()
        expect.append(e)
    if not sgd:
        hp['step'] = 3
    _kernel_vs_fp32(cases, pdt, sgd, expect_master=expect, **hp)
    # a zero-filled master takes the parameter's value
    for c in cases:
        c['w'].t.zero_()
    _kernel_vs_fp32(cases, pdt, sgd, expect_master=[c['p'].t.float() for c in cases], **hp)


def _mlp(dtype, seed=0):
    torch.manual_seed(seed)
    m = torch.nn.Sequential(torch.nn.Linear(24, 48), torch.nn.LayerNorm(48), torch.nn.ReLU(), torch.nn.Linear(48, 10))
    return m.cuda().to(dtype)


def _mlp_loss(m, step, dtype):
    g = torch.Generator(device='cuda').manual_seed(500 + step)
    x = torch.randn(16, 24, device='cuda', generator=g).to(dtype)
    return m(x).float().square().mean()


def test_reconcile_after_load_state_dict_and_broadcast_parameters(hvd):
    """Whole tensors written by model.load_state_dict and hvd.broadcast_parameters (world size 1), and single elements
    edited in place: exactly those restart from the new values; every other master stays bit for bit."""
    dt = torch.bfloat16
    m = _mlp(dt)
    opt = hvd.DistributedOptimizer(torch.optim.AdamW(m.parameters(), lr=1e-2), named_parameters=m.named_parameters(),
                                   master_weights=True)
    for step in range(3):
        opt.zero_grad()
        _mlp_loss(m, step, dt).backward()
        opt.step()
    other = _mlp(dt, seed=7)
    sd = m.state_dict()
    sd['0.weight'] = other[0].weight.detach().clone()
    m.load_state_dict(sd)
    hvd.broadcast_parameters({'3.bias': m[3].bias}, root_rank=0)  # at world size 1 the value stays; so must the master
    with torch.no_grad():
        m[3].weight[0, :5] = 0.5
    masters = {p: opt.state[p]['master_param'].clone() for p in m.parameters()}
    # a reloaded element that happens to equal its old rounded master is indistinguishable from an untouched one: by the
    # rule it keeps the master (for random weights a handful of the 1152 elements)
    w, new = masters[m[0].weight], m[0].weight.detach()
    masters[m[0].weight] = torch.where(bits(w.to(dt)) == bits(new), w, new.float())
    masters[m[3].weight][0, :5] = 0.5
    # oracle: an fp32 twin starting from those masters, the same gradients and state, the fp32 kernel
    twin = copy.deepcopy(m).float()
    with torch.no_grad():
        for q, p in zip(twin.parameters(), m.parameters()):
            q.copy_(masters[p])
    topt = hvd.DistributedOptimizer(torch.optim.AdamW(twin.parameters(), lr=1e-2), named_parameters=twin.named_parameters(),
                                    fused=True)
    # (deep copies: a loaded 'step' tensor would otherwise be shared with, and advanced by, both optimizers)
    topt.load_state_dict(copy.deepcopy({'state': {i: {k: v for k, v in opt.state[p].items() if k != 'master_param'}
                                                  for i, p in enumerate(m.parameters())},
                                        'param_groups': opt.state_dict()['param_groups']}))
    opt.zero_grad()
    _mlp_loss(m, 3, dt).backward()
    for q, p in zip(twin.parameters(), m.parameters()):
        q.grad = p.grad.float()
    opt.step()
    topt.step()
    torch.cuda.synchronize()
    for (name, p), q in zip(m.named_parameters(), twin.parameters()):
        assert same(opt.state[p]['master_param'], q.detach()), name
        assert same(p.detach(), q.detach().to(dt)), name


# ---- the capability ----------------------------------------------------------------------------------------------------
def test_bf16_update_below_half_an_ulp(hvd):
    """A bf16 weight of 1.0 and SGD steps of 1e-3 (half an ulp of bf16 below 1.0 is 2^-9): without masters the weight
    stalls at 1.0, with masters it follows fp32 and reads bf16(fp32 reference)."""
    lr = 1e-3
    out = {}
    for master in (False, True):
        w = torch.nn.Parameter(torch.ones(4096, device='cuda', dtype=torch.bfloat16))
        opt = hvd.DistributedOptimizer(torch.optim.SGD([w], lr=lr), named_parameters=[('w', w)], fused=True,
                                       master_weights=master)
        for _ in range(50):
            opt.zero_grad()
            w.float().sum().backward()  # gradient 1
            opt.step()
        out[master] = (w.detach().clone(), opt.state[w].get('master_param'))
    assert torch.all(out[False][0] == 1.0)
    ref = torch.ones(4096, device='cuda')
    for _ in range(50):
        ref = ref - torch.tensor(lr, dtype=torch.float32)
    assert float(ref[0]) < 0.96
    assert same(out[True][1], ref) and same(out[True][0], ref.to(torch.bfloat16))


def test_bf16_adamw_masters_track_fp32_adamw(hvd):
    """A small bf16 model, 20 AdamW steps on fixed gradients. Every step, the masters and moments agree with the float64
    model of the fused kernel (adam_ref_kernel, which test_gpu_fused_optimizer checks against torch.optim) within 1e-6 of
    its error scale. Over the 20 steps the masters follow torch's fp32 AdamW on the same gradients, up to the kernel's
    fp32 hyper-parameters (torch forms the betas' powers and bias corrections in float64): within 1e-6 of |p0| plus 1e-4
    of lr per step, while the bf16 parameters without masters would lose most of these updates."""
    dt, lr, wd, steps = torch.bfloat16, 1e-3, 0.05, 20
    m = _mlp(dt)
    ref = [torch.nn.Parameter(p.detach().float().clone()) for p in m.parameters()]
    p0 = [q.detach().abs().clone() for q in ref]
    opt = hvd.DistributedOptimizer(torch.optim.AdamW(m.parameters(), lr=lr, weight_decay=wd),
                                   named_parameters=m.named_parameters(), master_weights=True)
    ropt = torch.optim.AdamW(ref, lr=lr, weight_decay=wd, foreach=False)
    g = torch.Generator(device='cuda').manual_seed(1)
    grads = [torch.randn(p.shape, device='cuda', generator=g).to(dt) for p in m.parameters()]
    for step in range(1, steps + 1):
        before = {}
        for p in m.parameters():
            st = opt.state[p]
            before[p] = (p.detach().double(), torch.zeros_like(p, dtype=torch.float64), torch.zeros_like(p, dtype=torch.float64)) \
                if step == 1 else (st['master_param'].double(), st['exp_avg'].double(), st['exp_avg_sq'].double())
        opt.zero_grad()
        (sum((p.float() * gr.float()).sum() for p, gr in zip(m.parameters(), grads))).backward()  # p.grad == gr
        opt.step()
        for q, gr in zip(ref, grads):
            q.grad = gr.float()
        ropt.step()
        for (name, p), q, gr, a0 in zip(m.named_parameters(), ref, grads, p0):
            assert torch.equal(p.grad, gr)
            st = opt.state[p]
            w = st['master_param']
            p_, m_, v_ = before[p]
            pr, mr, vr, ps, ms, vs = adam_ref_kernel(p_, gr.double(), m_, v_, lr=lr, weight_decay=wd, step=step)
            for got, want, scale, what in ((w, pr, ps, 'master'), (st['exp_avg'], mr, ms, 'exp_avg'),
                                           (st['exp_avg_sq'], vr, vs, 'exp_avg_sq')):
                err = (got.double() - want).abs()
                assert bool((err <= 1e-6 * scale).all()), (name, step, what, float((err / scale).max()))
            err = (w - q.detach()).abs()
            assert bool((err <= step * (1e-6 * a0 + 1e-4 * lr)).all()), (name, step, float(err.max()))
            assert same(p.detach(), w.to(dt)), name


# ---- the optimizer at world size 1 -------------------------------------------------------------------------------------
def _twin_steps(hvd, make, dtype, steps, frozen_until=0, closure_at=()):
    """A master-weights model and an fp32 twin (the master kernel's oracle: fp32 parameters, fp32 kernel) fed the same
    gradients; `late` (the last Linear) stays frozen before step `frozen_until`. Returns both models and optimizers."""
    m = _mlp(dtype)
    twin = copy.deepcopy(m).float()
    for x in (m, twin):
        x[3].requires_grad_(frozen_until == 0)
    opt = hvd.DistributedOptimizer(make(m), named_parameters=m.named_parameters(), master_weights=True)
    topt = hvd.DistributedOptimizer(make(twin), named_parameters=twin.named_parameters(), fused=True)
    for step in range(steps):
        if step == frozen_until and step:
            for x in (m, twin):
                x[3].requires_grad_(True)
        opt.zero_grad(set_to_none=True)
        topt.zero_grad(set_to_none=True)
        loss = _mlp_loss(m, step, dtype)
        loss.backward()
        for q, p in zip(twin.parameters(), m.parameters()):
            q.grad = None if p.grad is None else p.grad.float()
        if step in closure_at:
            assert opt.step(lambda: loss) is loss
        else:
            assert opt.step() is None
        topt.step()
        torch.cuda.synchronize()
        for (name, p), q in zip(m.named_parameters(), twin.parameters()):
            if p.requires_grad and p in opt.state:
                assert same(opt.state[p]['master_param'], q.detach()), (name, step)
            assert same(p.detach(), q.detach().to(dtype)), (name, step)
    return m, opt, twin, topt


def _adamw(m):
    return torch.optim.AdamW(m.parameters(), lr=1e-2, weight_decay=0.05)


def _sgd(m):
    return torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-3)


@pytest.mark.parametrize("pdt", LOW, ids=LOW_IDS)
@pytest.mark.parametrize("kind", ["adamw", "sgd"])
def test_optimizer_follows_fp32_twin(hvd, pdt, kind):
    """Masters equal an fp32 model trained by the fused fp32 kernel on the same gradients, bit for bit, through a
    step(closure) and, with AdamW, a Linear frozen for the first 3 steps (its own step count). (The fp32 twin cannot
    follow a frozen Linear with SGD: without masters, partially initialised momentum takes torch's own update.)"""
    make = _adamw if kind == 'adamw' else _sgd
    m, opt, _, _ = _twin_steps(hvd, make, pdt, 6, frozen_until=3 if kind == 'adamw' else 0, closure_at=(1, 4))
    w = m[3].weight
    assert opt.state[w]['master_param'].dtype == torch.float32 and opt.state[w]['master_param'].stride() == w.stride()
    if kind == 'adamw':
        assert int(opt.state[w]['step']) == 3 and int(opt.state[m[0].weight]['step']) == 6
    else:
        assert opt.state[w]['momentum_buffer'].dtype == torch.float32


@pytest.mark.parametrize("pdt", LOW, ids=LOW_IDS)
def test_sgd_parameter_joining_later_starts_its_momentum(hvd, pdt):
    """SGD with momentum and masters: a Linear frozen for 3 steps gets a fresh fp32 momentum buffer (the first-step rule)
    while the others continue theirs, in the fused update: against the master kernel run by hand."""
    from horovod_b200 import ops
    m = _mlp(pdt)
    m[3].requires_grad_(False)
    opt = hvd.DistributedOptimizer(_sgd(m), named_parameters=m.named_parameters(), master_weights=True)
    for step in range(5):
        if step == 3:
            m[3].requires_grad_(True)
        opt.zero_grad(set_to_none=True)
        _mlp_loss(m, step, pdt).backward()
        if step == 3:
            late = list(m[3].parameters())
            p0 = [p.detach().clone() for p in late]
            g0 = [p.grad.clone() for p in late]
        opt.step()
        if step == 3:
            ps = [x.clone() for x in p0]
            ws, bufs = [x.float() for x in p0], [torch.zeros_like(x, dtype=torch.float32) for x in p0]
            ops.fused_sgd_step(ps, g0, bufs, 0.05, 0.9, weight_decay=1e-3, first_step=True, master_params=ws)
            for p, q, w, b in zip(late, ps, ws, bufs):
                assert same(p.detach(), q) and same(opt.state[p]['master_param'], w)
                assert same(opt.state[p]['momentum_buffer'], b)


def test_graphed_step_equals_eager(hvd, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    dt = torch.bfloat16
    runs = []
    for graphed in (False, True):
        m = _mlp(dt)
        opt = hvd.DistributedOptimizer(_adamw(m), named_parameters=m.named_parameters(), master_weights=True)
        g = torch.Generator(device='cuda').manual_seed(2)
        xs = [torch.randn(16, 24, device='cuda', generator=g).to(dt) for _ in range(6)]
        fn = lambda x: m(x).float().square().mean()  # noqa: E731
        if graphed:
            # the warm-up iterations run forward + backward only; the optimizer starts with the first replay
            step = hvd.GraphedStep(fn, opt, (xs[0],))
            assert step.captured, step.fallback_reason
            for x in xs:
                step(x)
        else:
            for x in xs:
                opt.zero_grad(set_to_none=False)
                fn(x).backward()
                opt.step()
        torch.cuda.synchronize()
        runs.append((m, opt))
    (a, oa), (b, ob) = runs
    for (name, p), q in zip(a.named_parameters(), b.parameters()):
        assert same(p.detach(), q.detach()), name
        assert same(oa.state[p]['master_param'], ob.state[q]['master_param']), name


@pytest.mark.parametrize("kind", ["adamw", "sgd"])
def test_checkpoint_round_trip_is_bit_exact(hvd, monkeypatch, kind):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    dt = torch.bfloat16
    make = _adamw if kind == 'adamw' else _sgd

    def fresh():
        m = _mlp(dt)
        return m, hvd.DistributedOptimizer(make(m), named_parameters=m.named_parameters(), master_weights=True)

    def train(m, o, steps):
        for s in steps:
            o.zero_grad()
            _mlp_loss(m, s, dt).backward()
            o.step()

    ma, oa = fresh()
    train(ma, oa, range(6))
    mb, ob = fresh()
    train(mb, ob, range(3))
    f = io.BytesIO()
    torch.save({'model': mb.state_dict(), 'opt': ob.state_dict()}, f)
    f.seek(0)
    ck = torch.load(f)
    assert all(st['master_param'].dtype == torch.float32 for st in ck['opt']['state'].values())
    mc, oc = fresh()
    mc.load_state_dict(ck['model'])
    oc.load_state_dict(ck['opt'])
    for p in mc.parameters():
        assert oc.state[p]['master_param'].dtype == torch.float32
        if kind == 'sgd':
            assert oc.state[p]['momentum_buffer'].dtype == torch.float32
    train(mc, oc, range(3, 6))
    for (name, a), c in zip(ma.named_parameters(), mc.parameters()):
        assert same(a.detach(), c.detach()), name
        for key, t in oa.state[a].items():
            if torch.is_tensor(t) and t.dim() > 0:
                assert same(t, oc.state[c][key]), (name, key)


def test_checkpoint_without_masters_loads(hvd):
    """A checkpoint of a bf16 model trained without masters: the masters start from the parameters."""
    dt = torch.bfloat16
    m = _mlp(dt)
    o = hvd.DistributedOptimizer(_adamw(m), named_parameters=m.named_parameters(), fused=True)
    for s in range(2):
        o.zero_grad()
        _mlp_loss(m, s, dt).backward()
        o.step()
    sd = o.state_dict()
    assert not any('master_param' in st for st in sd['state'].values())
    m2 = copy.deepcopy(m)
    o2 = hvd.DistributedOptimizer(_adamw(m2), named_parameters=m2.named_parameters(), master_weights=True)
    o2.load_state_dict(copy.deepcopy(sd))  # deep copies: see test_reconcile_after_load_state_dict_and_broadcast_parameters
    # oracle: the fp32 kernel on the upcast parameters with the loaded state
    twin = copy.deepcopy(m).float()
    t2 = hvd.DistributedOptimizer(_adamw(twin), named_parameters=twin.named_parameters(), fused=True)
    t2.load_state_dict(copy.deepcopy(sd))
    o2.zero_grad()
    _mlp_loss(m2, 2, dt).backward()
    for q, p in zip(twin.parameters(), m2.parameters()):
        q.grad = p.grad.float()
    o2.step()
    t2.step()
    for (name, p), q in zip(m2.named_parameters(), twin.parameters()):
        assert same(o2.state[p]['master_param'], q.detach()), name


def test_rejections(hvd):
    m = _mlp(torch.bfloat16)
    named = list(m.named_parameters())
    with pytest.raises(ValueError):
        hvd.DistributedOptimizer(_adamw(m), named_parameters=named, master_weights=True, op=hvd.Adasum)
    with pytest.raises(ValueError):
        hvd.DistributedOptimizer(torch.optim.AdamW(m.parameters(), amsgrad=True), named_parameters=named, master_weights=True)
    with pytest.raises(ValueError):
        hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1, maximize=True), named_parameters=named,
                                 master_weights=True)
    with pytest.raises(ValueError):
        hvd.DistributedOptimizer(torch.optim.RMSprop(m.parameters()), named_parameters=named, master_weights=True)
    # a step the fused kernels cannot take raises instead of falling back to torch's update
    cpu = torch.nn.Linear(4, 4).to(torch.bfloat16)
    opt = hvd.DistributedOptimizer(_adamw(cpu), named_parameters=cpu.named_parameters(), master_weights=True)
    cpu(torch.randn(2, 4, dtype=torch.bfloat16)).float().sum().backward()
    w0 = cpu.weight.detach().clone()
    with pytest.raises(RuntimeError, match='CUDA'):
        opt.step()
    assert torch.equal(cpu.weight.detach(), w0)


def test_kernel_rejects_bad_master_arguments(hvd):
    from horovod_b200 import ops
    z = lambda n=64, dt=torch.float32: torch.zeros(n, device='cuda', dtype=dt)  # noqa: E731
    pb, gb = z(dt=torch.bfloat16), z(dt=torch.bfloat16)

    def rejects(fn, *a, **kw):
        before = hvd.runtime_stats()['kernel_launches']
        with pytest.raises(RuntimeError):
            fn(*a, **kw)
        torch.cuda.synchronize()
        assert hvd.runtime_stats()['kernel_launches'] == before

    rejects(ops.fused_adam_step, [z()], [z()], [z()], [z()], lr=1e-3, master_params=[z()])          # fp32 params
    rejects(ops.fused_adam_step, [pb], [gb], [z()], [z()], lr=1e-3, master_params=[z(dt=torch.float16)])  # master dtype
    rejects(ops.fused_adam_step, [pb], [gb], [z()], [z()], lr=1e-3, master_params=[z(65)])          # master numel
    rejects(ops.fused_adam_step, [pb], [gb], [z()], [z()], lr=1e-3, master_params=[z(), z()])       # list length
    rejects(ops.fused_adam_step, [pb], [z()], [z()], [z()], lr=1e-3, master_params=[z()])           # fp32 grads
    rejects(ops.fused_adam_step, [pb], [gb], [z()], [z()], lr=1e-3, master_params=[torch.zeros(64)])  # on the host
    w = torch.zeros(4, 8, 3, 3, device='cuda', dtype=torch.bfloat16).to(memory_format=torch.channels_last)
    rejects(ops.fused_adam_step, [w], [torch.zeros_like(w)], [torch.zeros_like(w, dtype=torch.float32)],
            [torch.zeros_like(w, dtype=torch.float32)], lr=1e-3, master_params=[torch.zeros(4, 8, 3, 3, device='cuda')])
    rejects(ops.fused_sgd_step, [pb], [gb], [z(dt=torch.bfloat16)], lr=0.1, momentum=0.9, master_params=[z()])  # bf16 momentum
    rejects(ops.fused_sgd_step, [pb], [gb], [], lr=0.1, master_params=[z(32)])
    rejects(ops.fused_sgd_step, [z()], [z()], [], lr=0.1, master_params=[z()])


# ---- sharded (ZeRO-1) on 4 simulated ranks -----------------------------------------------------------------------------
class _ConvNet(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3)
        self.fc = torch.nn.Linear(8 * 6 * 6, 10)
        self.head = torch.nn.Linear(10, 10)  # its own param group in the SGD-without-momentum case

    def forward(self, x):
        return self.head(self.fc(torch.relu(self.conv(x)).flatten(1)))


def _make(kind, m):
    if kind == 'adamw':
        return torch.optim.AdamW(m.parameters(), lr=1e-2, weight_decay=0.05)
    # SGD with momentum, and a plain-SGD param group (no momentum: masters are its only state)
    return torch.optim.SGD([{'params': list(m.conv.parameters()) + list(m.fc.parameters())},
                            {'params': m.head.parameters(), 'momentum': 0.0, 'nesterov': False}], lr=0.05, momentum=0.9,
                           nesterov=True,
                           weight_decay=1e-4)


def _sharded_team(hvd, team, base, kind, dt):
    models, opts = sharded_team(hvd, team, base, lambda m: _make(kind, m), dt, min_buckets=3, master_weights=True)
    assert all('master_param' in b['state'] for b in opts[0]._buckets)
    return models, opts


def _reference(hvd, kind, model):
    """The oracle of the sharded runs: a world-size-1 master-weights optimizer (plain tensors, no gradient buckets)."""
    return hvd.DistributedOptimizer(_make(kind, model), named_parameters=model.named_parameters(), master_weights=True,
                                    zero_copy=False)


def _check_against(models, opts, ref, ref_opt, what):
    sd = opts[0].state_dict()
    for r in range(len(models)):
        for (name, a), b in zip(models[r].named_parameters(), ref.parameters()):
            assert same(a.detach(), b.detach()), (what, name, r)
    for i, (name, b) in enumerate(ref.named_parameters()):
        for key, t in ref_opt.state[b].items():
            if torch.is_tensor(t) and t.dim() > 0:
                assert same(sd['state'][i][key].cuda(), t), (what, name, key)
    return sd


@pytest.mark.parametrize("dt", LOW, ids=LOW_IDS)
@pytest.mark.parametrize("kind", ["adamw", "sgd"])
def test_sharded_masters_on_simulated_ranks(hvd, team, dt, kind):
    """After every step the gathered masters and moments and the allgathered parameters equal, bit for bit, a world-size-1
    master-weights optimizer fed the reduced gradient; then a sharded -> unsharded -> sharded checkpoint round trip."""
    n = team.n
    torch.manual_seed(0)
    base = _ConvNet().cuda().to(dtype=dt, memory_format=torch.channels_last)
    models, opts = _sharded_team(hvd, team, base, kind, dt)
    ref = copy.deepcopy(base)
    ref_opt = _reference(hvd, kind, ref)

    def step_all(models, opts, step):
        for r in range(n):
            opts[r].zero_grad()
            x, y = batch(step, r, dt)
            torch.nn.functional.cross_entropy(models[r](x), y).backward()
        for o in opts:
            o.synchronize()
        team.flush()
        grads = reduced_grads(opts, list(models[0].parameters()))
        for o in opts:
            with o.skip_synchronize():
                o.step()
        team.flush()
        return grads

    for step in range(4):
        ref_step(ref, ref_opt, step_all(models, opts, step))
        sd = _check_against(models, opts, ref, ref_opt, 'step %d' % step)
    if kind == 'sgd':
        # the plain-SGD group's bucket holds masters only; they are saved
        head = [i for i, (name, _) in enumerate(ref.named_parameters()) if name.startswith('head')]
        assert all(set(sd['state'][i]) == {'master_param'} for i in head)
    # sharded -> unsharded: a fresh world-size-1 optimizer loads the gathered checkpoint and continues like ref
    ref2 = copy.deepcopy(base)
    ref2.load_state_dict(ref.state_dict())
    ref2_opt = _reference(hvd, kind, ref2)
    ref2_opt.load_state_dict(copy.deepcopy(sd))
    # unsharded -> sharded: a fresh simulated team loads the world-size-1 checkpoint
    models2, opts2 = _sharded_team(hvd, team, ref2, kind, dt)
    usd = ref_opt.state_dict()
    for o in opts2:
        o.load_state_dict(usd)
    grads = step_all(models2, opts2, 4)
    ref_step(ref, ref_opt, grads)
    for p, g in zip(ref2.parameters(), grads):
        p.grad = g.clone()
    ref2_opt.step()
    _check_against(models2, opts2, ref, ref_opt, 'after unsharded -> sharded')
    for (name, a), b in zip(ref2.named_parameters(), ref.parameters()):
        assert same(a.detach(), b.detach()), name
        assert same(ref2_opt.state[a]['master_param'], ref_opt.state[b]['master_param']), name


def test_sharded_masters_with_grad_scaler_and_clipping(hvd, team):
    """fp16 model + AdamW + master weights + ShardedGradScaler + clip_grad_norm_ on 4 simulated ranks; in step 2 an inf in
    rank 0's local gradient makes every rank skip. The masters and parameters equal, bit for bit, a world-size-1
    master-weights optimizer fed the unscaled reduced gradient with the same clip coefficient."""
    n, dt = team.n, torch.float16
    torch.manual_seed(0)
    base = _ConvNet().cuda().to(dtype=dt, memory_format=torch.channels_last)
    models, opts = _sharded_team(hvd, team, base, 'adamw', dt)
    scalers = [hvd.ShardedGradScaler('cuda', init_scale=256.0) for _ in range(n)]
    ref = copy.deepcopy(base)
    ref_opt = _reference(hvd, 'adamw', ref)
    for step in range(5):
        for r in range(n):
            opts[r].zero_grad()
            x, y = batch(step, r, dt)
            scalers[r].scale(torch.nn.functional.cross_entropy(models[r](x), y)).backward()
        if step == 2:
            opts[0]._buckets[0]['gflat'][0] = math.inf
        before = [s.get_scale() for s in scalers]
        norms = team.run(lambda r: (scalers[r].unscale_(opts[r]), opts[r].clip_grad_norm_(0.5))[1])
        grads = reduced_grads(opts, list(models[0].parameters()))  # unscaled in place by unscale_
        coef = opts[0]._clip_coef.clone()
        team.run(lambda r: (scalers[r].step(opts[r]), scalers[r].update()))
        if step == 2:
            assert all(s.get_scale() == before[0] / 2 for s in scalers)
        else:
            assert all(torch.equal(x, norms[0]) for x in norms)
            ref_opt.zero_grad()
            for p, g in zip(ref.parameters(), grads):
                p.grad = g.clone()
            # the clip coefficient reaches the sharded update through grad_scale_dev; give the reference the same factor
            with torch.no_grad():
                from horovod_b200.torch.optimizer import _master_param
                for p in ref.parameters():
                    _master_param(ref_opt, p)
            _fused_with_coef(ref_opt, coef)
        _check_against(models, opts, ref, ref_opt, 'step %d' % step)


def _fused_with_coef(opt, coef):
    """The world-size-1 reference update with a device-side gradient factor: one fused AdamW launch per step count."""
    from horovod_b200 import ops
    group = opt.param_groups[0]
    ps = [p for p in group['params']]
    for p in ps:
        st = opt.state[p]
        if 'exp_avg' not in st:
            st['step'] = torch.tensor(0.0)
            st['exp_avg'] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
            st['exp_avg_sq'] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
        st['step'] += 1
    b1, b2 = group['betas']
    ops.fused_adam_step(ps, [p.grad for p in ps], [opt.state[p]['exp_avg'] for p in ps], [opt.state[p]['exp_avg_sq'] for p in ps],
                        group['lr'], b1, b2, group['eps'], group['weight_decay'], int(opt.state[ps[0]]['step']), 1.0, True,
                        grad_scale_dev=coef.reshape(1), master_params=[opt.state[p]['master_param'] for p in ps])


# ---- compute-sanitizer, real ranks -------------------------------------------------------------------------------------
_SANITIZER_TARGET = r'''
import torch
from horovod_b200 import ops
torch.cuda.set_device(0)
for dt in (torch.bfloat16, torch.float16):
    for n in (1, 3, 5, 4095, 4097):
        for off in (0, 1, 3):
            mk = lambda d: torch.randn(n + off + 3, device='cuda').to(d)[off:off + n]
            p, g, w, b = mk(dt), mk(dt), mk(torch.float32), mk(torch.float32)
            ops.fused_sgd_step([p], [g], [b], 0.1, 0.9, master_params=[w])
            ops.fused_adam_step([p], [g], [mk(torch.float32)], [mk(torch.float32).abs()], 1e-3, step=2, master_params=[w])
torch.cuda.synchronize()
print('MASTER SANITIZER OK')
'''


@pytest.mark.skipif(os.environ.get('HVD_RUN_COMPUTE_SANITIZER', '0') != '1',
                    reason='opt-in (HVD_RUN_COMPUTE_SANITIZER=1): memcheck instruments every kernel of the process')
def test_master_kernels_under_compute_sanitizer_memcheck():
    cs = shutil.which('compute-sanitizer') or '/usr/local/cuda/bin/compute-sanitizer'
    if not os.path.exists(cs):
        pytest.skip('compute-sanitizer not installed')
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([cs, '--tool', 'memcheck', '--error-exitcode', '77', sys.executable, '-c', _SANITIZER_TARGET],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, env=dict(os.environ, PYTHONPATH=repo))
    out = p.stdout.decode(errors='replace')
    assert p.returncode == 0 and 'MASTER SANITIZER OK' in out and 'ERROR SUMMARY: 0 errors' in out, out[-5000:]


@pytest.mark.skipif(ngpu() < 2, reason="needs >= 2 GPUs")
def test_master_weights_across_ranks(native_built):
    n = 2 if ngpu() < 4 else 4
    rc, out = run_parallel("master_weights_worker.py", np=n, timeout=420)
    assert "MASTER WEIGHTS OK" in out, out[-4000:]
