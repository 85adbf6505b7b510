"""Fused LARS: the sm_90a kernels (ops.fused_lars_step, ops.lars_norms / ops.lars_apply) against an fp64 reference,
the master-weight variants against the fp32-parameter kernels bit for bit, DistributedOptimizer(hvd.Lars(...), fused=True)
against Lars.step at world size 1 (and under hvd.GraphedStep), and the sharded (ZeRO-1) LARS update on 4 simulated ranks
against unsharded fused LARS; with >= 2 GPUs, across real ranks."""
import copy
import io
import math

import pytest
import torch

from conftest import run_parallel
from optim_cases import (LOW, LOW_IDS, PAIR_IDS, PAIRS, SIZES, Slot, cat, f32, hvd, lars_ref, mlp, mlp_loss,  # noqa: F401
                         ngpu, same, two_phase, ulp)
from sim_ranks import FakeSet, NormConvNet, batch, reduced_grads, ref_step, sharded_team, step_all, team  # noqa: F401

pytestmark = pytest.mark.gpu

HP = [dict(lr=0.5, momentum=0.9, weight_decay=1e-4, trust_coefficient=1e-3, eps=0.0),
      dict(lr=0.1, momentum=0.9, weight_decay=0.0, trust_coefficient=1e-3, eps=0.0, adapt=False, grad_scale=0.5),
      dict(lr=1.0, momentum=0.0, weight_decay=5e-3, trust_coefficient=0.02, eps=1e-3),
      dict(lr=0.2, momentum=0.8, weight_decay=0.0, trust_coefficient=0.01, eps=1e-5, adapt=True)]
U = 2.0 ** -24
# Rounding points of the kernel.  Each sum of squares: the scaled gradient is rounded once (2u on its square), then 16
# fmas per thread, a 5-level shuffle tree and 8 warps in order in fp32 (a sum of k non-negative terms is off by less than
# k u relative), the CTA partials added in fp64 and rounded to fp32 once more (u).  The norms are square roots (half the
# relative error, plus u each), r = tc * wn / (fma(wd, wn, gn) + eps) takes 4 more roundings and lr * r one: so the
# per-tensor rate lr * r is off by at most NORM_RTOL relative.
NORM_RTOL = (16 + 5 + 8 + 2 + 1) * U + 8 * U
# Per element: d = fma(wd, w, g * s) is 2 roundings relative to |g s| + |wd w|, the product with lr * r one, the momentum
# fma one relative to |m v| + |lr r d|, and w - v one of the result.
ELEM_RTOL = 4 * U


def _case(shape, pdt, gdt, seed, offsets=(0, 0, 0), memory_format=torch.contiguous_format, master=False):
    g = torch.Generator(device='cuda').manual_seed(seed)
    po, go, so = offsets
    rnd = lambda s: torch.randn(shape, device='cuda', generator=g) * s  # noqa: E731
    w = rnd(0.1)
    c = {'p': Slot(shape, pdt, po, w.to(pdt), memory_format), 'g': Slot(shape, gdt, go, rnd(1.0), memory_format),
         'v': Slot(shape, torch.float32, so, rnd(0.01), memory_format)}
    if master:
        c['w'] = Slot(shape, torch.float32, so + 1, w, memory_format)
    return c


def _run_and_check(cases, hp):
    from horovod_b200 import ops
    pdt = cases[0]['p'].t.dtype
    want = lars_ref(cases, **hp)
    g_before = [c['g'].t.clone() for c in cases]
    ops.fused_lars_step([c['p'].t for c in cases], [c['g'].t for c in cases], [c['v'].t for c in cases], **hp)
    torch.cuda.synchronize()
    e = {k: cat([x[k] for x in want]) for k in want[0]}
    got = {k: cat([c[k].t.double() for c in cases]) for k in ('p', 'v')}
    tol_v = e['scale_v'] * (NORM_RTOL + ELEM_RTOL)
    err_v = (got['v'] - e['v']).abs()
    assert not bool((err_v > tol_v).any()), ('momentum', int((err_v > tol_v).sum()))
    tol = tol_v + ulp(e['w'], torch.float32)
    if pdt != torch.float32:
        tol = tol + ulp(e['w'], pdt)  # then rounded to nearest in the parameter dtype
    err = (got['p'] - e['w']).abs()
    bad = err > tol
    assert not bool(bad.any()), (int(bad.sum()), float((err - tol).max()))
    for i, c in enumerate(cases):
        assert same(c['g'].t, g_before[i]), (i, 'grad written')
        for k, s in c.items():
            assert s.intact(), (i, 'wrote outside ' + k)


@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("hp", range(len(HP)))
def test_kernel_matches_fp64(hvd, pair, hp):
    """All sizes and ~200 small tensors in one launch, a channels_last tensor, a zero parameter (||w|| = 0 on the first
    step) and a zero gradient (||g|| = 0): a 10-step trajectory for the first hyper-parameter set, 2 steps for the
    others (each step checked from the state the kernel left)."""
    pdt, gdt = pair
    sizes = SIZES + [int(x) for x in torch.randint(1, 3000, (200,), generator=torch.Generator().manual_seed(hp))]
    cases = [_case((n,), pdt, gdt, seed=i) for i, n in enumerate(sizes)]
    cases.append(_case((8, 6, 5, 3), pdt, gdt, seed=999, memory_format=torch.channels_last))
    cases[1]['p'].t.zero_()
    for step in range(1, 11 if hp == 0 else 3):
        for i, c in enumerate(cases):
            c['g'].t.copy_(torch.randn(c['g'].t.shape, device='cuda', generator=torch.Generator(device='cuda').manual_seed(1000 * step + i)))
        cases[2]['g'].t.zero_()
        _run_and_check(cases, HP[hp])


@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("offsets", [(1, 0, 0), (0, 1, 0), (0, 0, 1), (2, 3, 1), (3, 2, 3)])
def test_kernel_unaligned_views(hvd, pair, offsets):
    pdt, gdt = pair
    cases = [_case((n,), pdt, gdt, seed=i, offsets=offsets) for i, n in enumerate(SIZES)]
    _run_and_check(cases, HP[0])


@pytest.mark.parametrize("pdt", LOW, ids=LOW_IDS)
def test_master_kernels_equal_fp32_kernels(hvd, pdt):
    """Masters, momentum and norms bit-identical to the fp32-parameter kernels started from the masters; parameters the
    rounded masters.  Some parameter elements are overwritten first: those masters restart from the parameter."""
    hp = dict(lr=0.5, momentum=0.9, weight_decay=1e-3, trust_coefficient=0.01, eps=1e-6)
    shapes = [(n,) for n in SIZES] + [(8, 6, 5, 3)] + [(n,) for n in range(1, 200, 7)]
    fmt = lambda s: torch.channels_last if len(s) == 4 else torch.contiguous_format  # noqa: E731
    cases = [_case(s, pdt, pdt, seed=i, offsets=(i % 4, (i + 1) % 4, (i + 2) % 4), master=True, memory_format=fmt(s))
             for i, s in enumerate(shapes)]
    gsd = torch.tensor([0.75], device='cuda')
    for c in cases[:3]:
        c['p'].t.reshape(-1)[::2] = 0.125  # an outside write: these elements restart from the parameter
    start = []
    for c in cases:
        kept = c['w'].t.to(pdt).view(torch.int16) == c['p'].t.view(torch.int16)
        start.append(torch.where(kept, c['w'].t, c['p'].t.float()))
    ref = [{'p': Slot(s.shape, torch.float32, 0, s, fmt(s.shape)),
            'g': Slot(s.shape, torch.bfloat16 if pdt == torch.bfloat16 else torch.float32, 0, c['g'].t, fmt(s.shape)),
            'v': Slot(s.shape, torch.float32, 0, c['v'].t, fmt(s.shape))}
           for c, s in zip(cases, start)]
    g_before = [c['g'].t.clone() for c in cases]
    for _ in range(3):
        norms = two_phase('lars', cases, True, gsd=gsd, **hp)
        ref_norms = two_phase('lars', ref, False, gsd=gsd, **hp)
        torch.cuda.synchronize()
        assert same(norms, ref_norms)
    for i, (c, r) in enumerate(zip(cases, ref)):
        assert same(c['w'].t, r['p'].t), (i, 'master')
        assert same(c['p'].t, r['p'].t.to(pdt)), (i, 'param is not the rounded master')
        assert same(c['v'].t, r['v'].t), (i, 'momentum')
        assert same(c['g'].t, g_before[i])
        for k, s in c.items():
            assert s.intact(), (i, 'wrote outside ' + k)


def test_deterministic_no_host_sync_and_fixed_launch_count(hvd):
    from horovod_b200 import ops
    for n in (5, 200):
        cases = [_case(((1 << 20) + 3 if i == 0 else 1000 + i,), torch.float32, torch.float32, seed=i) for i in range(n)]
        snap = [{k: s.t.clone() for k, s in c.items()} for c in cases]
        results = []
        for _ in range(2):
            for c, s in zip(cases, snap):
                for k in c:
                    c[k].t.copy_(s[k])
            torch.cuda.synchronize()
            before = ops.kernel_launches()
            torch.cuda.set_sync_debug_mode('error')
            try:
                ops.fused_lars_step([c['p'].t for c in cases], [c['g'].t for c in cases], [c['v'].t for c in cases],
                                    0.5, 0.9, 1e-4, 1e-3, 0.0, grad_scale_dev=torch.ones(1, device='cuda'))
            finally:
                torch.cuda.set_sync_debug_mode('default')
            assert ops.kernel_launches() - before == 3, 'partials, norms, update: independent of the tensor count'
            torch.cuda.synchronize()
            results.append([c[k].t.clone() for c in cases for k in ('p', 'v')])
        assert all(same(a, b) for a, b in zip(*results))


@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
def test_grad_scale_dev(hvd, pair):
    """A device factor of 1 is bit-identical to none; a factor k equals gradients scaled by k (k = 4: exact in every
    gradient dtype), in the norms and in the update alike: a factor that reached one phase only would differ."""
    pdt, gdt = pair
    from horovod_b200 import ops

    def run(gscale=1.0, phased=False, **kw):
        cases = [_case((n,), pdt, gdt, seed=i) for i, n in enumerate([1, 4097, 1 << 16])]
        for c in cases:
            c['g'].t.mul_(gscale)
        for _ in range(3):
            if phased:
                two_phase('lars', cases, False, gsd=kw.get('grad_scale_dev'), **HP[0])
            else:
                ops.fused_lars_step([c['p'].t for c in cases], [c['g'].t for c in cases], [c['v'].t for c in cases],
                                    0.5, 0.9, 1e-4, 1e-3, 0.0, **kw)
        return [c[k].t for c in cases for k in ('p', 'v')]

    four = torch.tensor([4.0], device='cuda')
    plain, one = run(), run(grad_scale_dev=torch.ones(1, device='cuda'))
    scaled, dev, host = run(gscale=4.0), run(grad_scale_dev=four), run(grad_scale=4.0)
    phases = run(phased=True, grad_scale_dev=four)
    assert all(same(a, b) for a, b in zip(plain, one))
    assert all(same(a, b) and same(a, c) and same(a, d) for a, b, c, d in zip(scaled, dev, host, phases))
    assert not all(same(a, b) for a, b in zip(plain, scaled))


def test_rejects_bad_arguments(hvd):
    from horovod_b200 import ops
    z = lambda n=64, dt=torch.float32: torch.zeros(n, device='cuda', dtype=dt)  # noqa: E731
    pb, gb = z(dt=torch.bfloat16), z(dt=torch.bfloat16)
    hp = (0.5, 0.9, 1e-4, 1e-3, 0.0)

    def rejects(fn, *a, **kw):
        p0 = [t.clone() for t in a[0]]
        torch.cuda.synchronize()
        before = hvd.runtime_stats()['kernel_launches']
        with pytest.raises(RuntimeError):
            fn(*a, **kw)
        torch.cuda.synchronize()
        assert hvd.runtime_stats()['kernel_launches'] == before
        assert all(torch.equal(x, y) for x, y in zip(a[0], p0))

    ones = [torch.ones(64, device='cuda')]
    rejects(ops.fused_lars_step, ones, [z()], [z(), z()], *hp)                               # list sizes
    rejects(ops.fused_lars_step, ones, [z(), z()], [z()], *hp)
    rejects(ops.fused_lars_step, ones, [z()], [z(dt=torch.bfloat16)], *hp)                    # momentum dtype
    rejects(ops.fused_lars_step, [pb], [gb], [pb.clone()], *hp)                              # bf16 momentum
    rejects(ops.fused_lars_step, ones, [z()], [z(64).as_strided((32,), (2,))], *hp)           # momentum size / strides
    rejects(ops.fused_lars_step, ones, [z(65)], [z()], *hp)                                   # grad size
    rejects(ops.fused_lars_step, ones, [torch.zeros(64)], [z()], *hp)                         # grad on the host
    rejects(ops.fused_lars_step, ones, [z(dt=torch.float16)], [z()], *hp)                     # no f32 / fp16 kernel
    rejects(ops.fused_lars_step, ones, [z()], [z()], *hp, master_params=[z()])                # masters for fp32 params
    rejects(ops.fused_lars_step, [pb], [gb], [z()], *hp, master_params=[z(dt=torch.float16)])
    rejects(ops.fused_lars_step, [pb], [z()], [z()], *hp, master_params=[z()])                # fp32 grads with masters
    rejects(ops.fused_lars_step, [pb], [gb], [z()], *hp, master_params=[z(), z()])            # master count
    rejects(ops.fused_lars_step, ones, [z()], [z()], *hp, grad_scale_dev=torch.ones(2, device='cuda'))
    rejects(ops.fused_lars_step, ones, [z()], [z()], *hp, grad_scale_dev=torch.ones(1))
    rejects(ops.fused_lars_step, [torch.ones(64, device='cuda', dtype=torch.float64)], [z()], [z()], *hp)
    for bad_out, slots in ((torch.zeros(2), None), (z(2, torch.float64), None), (z(4)[::2], None), (z(1), None),
                           (z(4), [2]), (z(4), [-1])):
        rejects(ops.lars_norms, ones, [z()], [z()], bad_out, slots=slots)
        rejects(ops.lars_apply, ones, [z()], [z()], *hp, bad_out, slots=slots)
    rejects(ops.lars_norms, ones * 2, [z(), z()], [z(), z()], z(8), slots=[1, 1])
    rejects(ops.lars_apply, ones * 2, [z(), z()], [z(), z()], *hp, z(8), slots=[1, 1])
    rejects(ops.lars_norms, ones, [z()], [z()], z(8), slots=[0, 1])
    rejects(ops.lars_apply, ones, [z()], [z()], *hp, z(8), grad_scale_dev=torch.ones(3, device='cuda'))


# ---- DistributedOptimizer at world size 1 -------------------------------------------------------------------------------
def _lars(hvd, m):
    """ResNet-style groups: weight decay (and so a trust ratio) on the matrices, none on biases and the norm layer; the
    always_adapt group covers the other branch."""
    decay = [p for n, p in m.named_parameters() if n.endswith('weight') and p.dim() == 2]
    ln = list(m[2].parameters())
    rest = [p for p in m.parameters() if all(p is not q for q in decay + ln)]
    return hvd.Lars([{'params': decay, 'weight_decay': 1e-3}, {'params': rest}, {'params': ln, 'always_adapt': True}],
                    lr=0.5, momentum=0.9, trust_coefficient=0.02)


def test_fused_optimizer_follows_lars_step(hvd):
    """fused=True against Lars.step over 10 steps: broadcast_optimizer_state first, the last Linear frozen for 3 steps,
    step(closure) twice, a learning-rate change at step 5."""
    dt = torch.float32
    m = mlp(dt)
    twin = copy.deepcopy(m)
    for x in (m, twin):
        x[3].requires_grad_(False)
    opt = hvd.DistributedOptimizer(_lars(hvd, m), named_parameters=m.named_parameters(), fused=True)
    ref = _lars(hvd, twin)
    for o in (opt, ref):
        hvd.broadcast_optimizer_state(o, root_rank=0)
    launches = []
    for step in range(10):
        if step == 3:
            for x in (m, twin):
                x[3].requires_grad_(True)
        if step == 5:
            for o in (opt, ref):
                for g in o.param_groups:
                    g['lr'] = 0.2
        opt.zero_grad(set_to_none=True)
        ref.zero_grad(set_to_none=True)
        loss = mlp_loss(m, step, dt)
        loss.backward()
        mlp_loss(twin, step, dt).backward()
        before = hvd.runtime_stats()['kernel_launches']
        if step in (2, 6):
            assert opt.step(lambda: loss) is loss
        else:
            assert opt.step() is None
        launches.append(hvd.runtime_stats()['kernel_launches'] - before)
        ref.step()
        for (name, p), q in zip(m.named_parameters(), twin.parameters()):
            torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6, msg=lambda s: '%s step %d: %s' % (name, step, s))
    # three launches per (group, dtype) and nothing else: the fused kernels ran, not Lars.step
    assert launches[5] >= 9, launches
    assert all(opt.state[p]['momentum_buffer'].dtype == torch.float32 for p in m.parameters())


def test_graphed_step_replays_equal_eager_fused_steps(hvd, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    for dt, master in ((torch.float32, False), (torch.bfloat16, True)):
        runs = []
        for graphed in (False, True):
            m = mlp(dt)
            opt = hvd.DistributedOptimizer(_lars(hvd, m), named_parameters=m.named_parameters(), fused=True,
                                           master_weights=master)
            g = torch.Generator(device='cuda').manual_seed(2)
            xs = [torch.randn(16, 24, device='cuda', generator=g).to(dt) for _ in range(6)]
            fn = lambda x: m(x).float().square().mean()  # noqa: E731
            if graphed:
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
            assert same(p.detach(), q.detach()), (dt, name)
            assert same(oa.state[p]['momentum_buffer'], ob.state[q]['momentum_buffer']), (dt, name)


def test_checkpoint_round_trip_is_bit_exact(hvd, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    dt = torch.bfloat16

    def fresh():
        m = mlp(dt)
        return m, hvd.DistributedOptimizer(_lars(hvd, m), named_parameters=m.named_parameters(), fused=True)

    def train(m, o, steps):
        for s in steps:
            o.zero_grad()
            mlp_loss(m, s, dt).backward()
            o.step()

    ma, oa = fresh()
    train(ma, oa, range(6))
    mb, ob = fresh()
    train(mb, ob, range(3))
    f = io.BytesIO()
    torch.save({'model': mb.state_dict(), 'opt': ob.state_dict()}, f)
    f.seek(0)
    ck = torch.load(f)
    mc, oc = fresh()
    mc.load_state_dict(ck['model'])
    oc.load_state_dict(ck['opt'])
    assert all(oc.state[p]['momentum_buffer'].dtype == torch.float32 for p in mc.parameters())  # not cast to bf16
    train(mc, oc, range(3, 6))
    for (name, a), c in zip(ma.named_parameters(), mc.parameters()):
        assert same(a.detach(), c.detach()), name
        assert same(oa.state[a]['momentum_buffer'], oc.state[c]['momentum_buffer']), name


def test_bf16_master_weights_follow_fp32_twin(hvd):
    """A bf16 model with master_weights=True and an fp32 twin on the fused fp32 kernels, fed the same gradients: the
    masters equal the twin's parameters bit for bit, the parameters are the rounded masters."""
    dt = torch.bfloat16
    m = mlp(dt)
    twin = copy.deepcopy(m).float()
    opt = hvd.DistributedOptimizer(_lars(hvd, m), named_parameters=m.named_parameters(), master_weights=True)
    topt = hvd.DistributedOptimizer(_lars(hvd, twin), named_parameters=twin.named_parameters(), fused=True)
    for step in range(6):
        opt.zero_grad(set_to_none=True)
        topt.zero_grad(set_to_none=True)
        mlp_loss(m, step, dt).backward()
        for q, p in zip(twin.parameters(), m.parameters()):
            q.grad = p.grad.float()
        opt.step()
        topt.step()
        for (name, p), q in zip(m.named_parameters(), twin.parameters()):
            assert same(opt.state[p]['master_param'], q.detach()), (name, step)
            assert same(p.detach(), q.detach().to(dt)), (name, step)
            assert same(opt.state[p]['momentum_buffer'], topt.state[q]['momentum_buffer']), (name, step)


def test_unfusable_plan_falls_back_or_raises(hvd):
    """A CPU model: fused=True falls back to Lars.step; master_weights=True raises instead."""
    cpu = torch.nn.Linear(4, 4)
    twin = copy.deepcopy(cpu)
    opt = hvd.DistributedOptimizer(hvd.Lars(cpu.parameters(), lr=0.1, weight_decay=0.01),
                                   named_parameters=cpu.named_parameters(), fused=True)
    ref = hvd.Lars(twin.parameters(), lr=0.1, weight_decay=0.01)
    x = torch.randn(2, 4)
    for mod, o in ((cpu, opt), (twin, ref)):
        mod(x).sum().backward()
        o.step()
    assert torch.equal(cpu.weight, twin.weight)
    half = torch.nn.Linear(4, 4).to(torch.bfloat16)
    mo = hvd.DistributedOptimizer(hvd.Lars(half.parameters(), lr=0.1), named_parameters=half.named_parameters(),
                                  master_weights=True)
    half(torch.randn(2, 4, dtype=torch.bfloat16)).float().sum().backward()
    with pytest.raises(RuntimeError, match='CUDA'):
        mo.step()


# ---- sharded (ZeRO-1) on 4 simulated ranks -----------------------------------------------------------------------------
def _make(hvd, m):
    decay = [m.conv.weight, m.fc.weight, m.head.weight]
    return hvd.Lars([{'params': decay, 'weight_decay': 5e-3},
                     {'params': [p for p in m.parameters() if all(p is not q for q in decay)], 'weight_decay': 0.0}],
                    lr=1.0, momentum=0.9, trust_coefficient=0.02)


@pytest.mark.parametrize("dt,master", [(torch.float32, False), (torch.bfloat16, True)], ids=['fp32', 'bf16-masters'])
def test_sharded_lars_on_simulated_ranks(hvd, team, dt, master):
    """Sharded LARS against unsharded fused LARS on the reduced gradients over 5 steps, then a sharded -> unsharded and an
    unsharded -> sharded checkpoint that both continue like the reference."""
    torch.manual_seed(0)
    base = NormConvNet().cuda().to(dtype=dt, memory_format=torch.channels_last)
    models, opts = sharded_team(hvd, team, base, lambda m: _make(hvd, m), dt, straddle=True, master_weights=master)
    ref = copy.deepcopy(base)
    ref_opt = hvd.DistributedOptimizer(_make(hvd, ref), named_parameters=ref.named_parameters(), fused=True,
                                       master_weights=master, zero_copy=False)
    tol = dict(rtol=1e-5, atol=1e-6) if dt == torch.float32 else dict(rtol=1e-2, atol=1e-3)

    def check(models, what):
        for (name, a), b in zip(models[0].named_parameters(), ref.parameters()):
            torch.testing.assert_close(a.float(), b.float(), **tol, msg=lambda s: '%s %s: %s' % (what, name, s))

    for step in range(5):
        grads, _ = step_all(team, models, opts, step, dt)
        ref_step(ref, ref_opt, grads)
        check(models, 'step %d' % step)
    sd = opts[0].state_dict()
    want = {'momentum_buffer'} | ({'master_param'} if master else set())
    assert len(sd['state']) == len(list(base.parameters())) and all(set(st) == want for st in sd['state'].values())
    # sharded -> unsharded
    un = copy.deepcopy(models[0])
    un_opt = hvd.DistributedOptimizer(_make(hvd, un), named_parameters=un.named_parameters(), fused=True,
                                      master_weights=master, zero_copy=False)
    un_opt.load_state_dict(copy.deepcopy(sd))
    # unsharded -> sharded
    models2, opts2 = sharded_team(hvd, team, copy.deepcopy(ref), lambda m: _make(hvd, m), dt, straddle=True,
                                  master_weights=master)
    usd = ref_opt.state_dict()
    for o in opts2:
        o.load_state_dict(usd)
    assert len(opts2[0].state_dict()['state']) == len(sd['state'])  # loaded momentum is state before any step
    grads, _ = step_all(team, models2, opts2, 5, dt)
    ref_step(ref, ref_opt, grads)
    ref_step(un, un_opt, grads)
    check(models2, 'unsharded -> sharded')
    for (name, a), b in zip(un.named_parameters(), models2[0].parameters()):
        torch.testing.assert_close(a.float(), b.float(), **tol, msg=lambda s: 'sharded -> unsharded %s: %s' % (name, s))


def test_sharded_lars_with_clipping(hvd, team):
    """opt.clip_grad_norm_ on the simulated ranks: its coefficient reaches both LARS phases through grad_scale_dev."""
    dt = torch.float32
    torch.manual_seed(0)
    base = NormConvNet().cuda().to(memory_format=torch.channels_last)
    models, opts = sharded_team(hvd, team, base, lambda m: _make(hvd, m), dt, straddle=True)
    ref = copy.deepcopy(base)
    ref_opt = hvd.DistributedOptimizer(_make(hvd, ref), named_parameters=ref.named_parameters(), fused=True, zero_copy=False)
    for step in range(4):
        grads, coef = step_all(team, models, opts, step, dt, clip=0.05)
        assert float(coef) < 1.0
        ref_step(ref, ref_opt, grads, coef, kind='lars')
        for (name, a), b in zip(models[0].named_parameters(), ref.parameters()):
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6, msg=lambda s: 'step %d %s: %s' % (step, name, s))


def test_sharded_lars_with_grad_scaler(hvd, team):
    """fp16 model with masters + ShardedGradScaler: the unscaled shards feed LARS; in step 1 an inf on rank 0 makes
    every rank skip alike."""
    n, dt = team.n, torch.float16
    torch.manual_seed(0)
    base = NormConvNet().cuda().to(dtype=dt, memory_format=torch.channels_last)
    models, opts = sharded_team(hvd, team, base, lambda m: _make(hvd, m), dt, straddle=True, master_weights=True)
    scalers = [hvd.ShardedGradScaler('cuda', init_scale=256.0) for _ in range(n)]
    ref = copy.deepcopy(base)
    ref_opt = hvd.DistributedOptimizer(_make(hvd, ref), named_parameters=ref.named_parameters(), master_weights=True,
                                       zero_copy=False)
    for step in range(4):
        for r in range(n):
            opts[r].zero_grad()
            x, y = batch(step, r, dt)
            scalers[r].scale(torch.nn.functional.cross_entropy(models[r](x), y)).backward()
        if step == 1:
            opts[0]._buckets[0]['gflat'][0] = math.inf
        before = [s.get_scale() for s in scalers]
        params_before = [p.detach().clone() for p in models[0].parameters()]
        team.run(lambda r: scalers[r].unscale_(opts[r]))
        grads = reduced_grads(opts, list(models[0].parameters()))
        team.run(lambda r: (scalers[r].step(opts[r]), scalers[r].update()))
        if step == 1:
            assert all(s.get_scale() == before[0] / 2 for s in scalers)
            assert all(same(a.detach(), b) for a, b in zip(models[0].parameters(), params_before))
        else:
            ref_step(ref, ref_opt, grads)
        for r in range(n):
            for (name, a), b in zip(models[r].named_parameters(), ref.parameters()):
                torch.testing.assert_close(a.float(), b.float(), rtol=1e-2, atol=1e-3, msg=lambda s: '%s: %s' % (name, s))


def test_trust_norms_buffer_only_for_lamb_and_lars(hvd, team):
    """The sharded optimizer allocates the padded norms buffer for Lamb and Lars only."""
    torch.manual_seed(0)
    base = NormConvNet().cuda()
    models, opts = sharded_team(hvd, team, base, lambda m: _make(hvd, m), torch.float32, straddle=True)
    assert opts[0]._trust_norms is not None and opts[0]._trust_norms.numel() % (32 * team.n) == 0
    assert opts[0]._trust_norms.numel() >= 2 * len(list(base.parameters()))
    for make in (lambda ps: hvd.Lamb(ps), lambda ps: torch.optim.SGD(ps, lr=0.1, momentum=0.9),
                 lambda ps: torch.optim.AdamW(ps)):
        m = copy.deepcopy(base)
        o = hvd.DistributedOptimizer(make(m.parameters()), named_parameters=m.named_parameters(),
                                     shard_optimizer_state=True, process_set=FakeSet(team.n, 0))
        assert (o._trust_norms is not None) == isinstance(o, hvd.Lamb)


@pytest.mark.skipif(ngpu() < 2, reason="needs >= 2 GPUs")
def test_sharded_lars_across_ranks(native_built):
    n = 2 if ngpu() < 4 else 4
    rc, out = run_parallel("lars_worker.py", np=n, timeout=420)
    assert "LARS OK" in out, out[-4000:]
