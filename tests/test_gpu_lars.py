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
from test_gpu_lamb import LOW, LOW_IDS, PAIR_IDS, PAIRS, SIZES, Slot, _cat, _ConvNet, _f32, _ngpu, _same, _ulp
from test_gpu_sharded_clip import _FakeSet, _SimTeam

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


def _ops():
    from horovod_b200 import ops
    return ops


@pytest.fixture(scope="module")
def hvd():
    import horovod_b200.torch as hvd
    hvd.init()
    torch.cuda.set_device(0)
    yield hvd
    hvd.shutdown()


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


def _ref(cases, lr, momentum, weight_decay, trust_coefficient, eps, adapt=True, grad_scale=1.0):
    """fp64 LARS from the values the kernel reads (parameter and gradient in their dtypes, fp32 momentum) and the
    hyper-parameters as the kernel holds them (fp32).  'scale_v' bounds the magnitudes that fp32 rounding errors are
    relative to."""
    lr, mom, wd, tc, eps = _f32(lr), _f32(momentum), _f32(weight_decay), _f32(trust_coefficient), _f32(eps)
    out = []
    for c in cases:
        w, g = c['p'].t.double(), c['g'].t.double() * _f32(grad_scale)
        vo = c['v'].t.double()
        wn, gn = float(w.norm()), float(g.norm())
        r = tc * wn / (gn + wd * wn + eps) if adapt and wn > 0 and gn > 0 else 1.0
        d = g + wd * w
        v = mom * vo + lr * r * d
        scale_v = mom * vo.abs() + lr * r * (g.abs() + (wd * w).abs())
        out.append({'w': w - v, 'v': v, 'scale_v': scale_v})
    return out


def _run_and_check(cases, hp):
    ops = _ops()
    pdt = cases[0]['p'].t.dtype
    want = _ref(cases, **hp)
    g_before = [c['g'].t.clone() for c in cases]
    ops.fused_lars_step([c['p'].t for c in cases], [c['g'].t for c in cases], [c['v'].t for c in cases], **hp)
    torch.cuda.synchronize()
    e = {k: _cat([x[k] for x in want]) for k in want[0]}
    got = {k: _cat([c[k].t.double() for c in cases]) for k in ('p', 'v')}
    tol_v = e['scale_v'] * (NORM_RTOL + ELEM_RTOL)
    err_v = (got['v'] - e['v']).abs()
    assert not bool((err_v > tol_v).any()), ('momentum', int((err_v > tol_v).sum()))
    tol = tol_v + _ulp(e['w'], torch.float32)
    if pdt != torch.float32:
        tol = tol + _ulp(e['w'], pdt)  # then rounded to nearest in the parameter dtype
    err = (got['p'] - e['w']).abs()
    bad = err > tol
    assert not bool(bad.any()), (int(bad.sum()), float((err - tol).max()))
    for i, c in enumerate(cases):
        assert _same(c['g'].t, g_before[i]), (i, 'grad written')
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


def _two_phase(cases, master, slots=None, out=None, gsd=None, **hp):
    """lars_norms then lars_apply over `cases`; returns the norms buffer."""
    ops = _ops()
    lists = [[c[k].t for c in cases] for k in ('p', 'g', 'v')]
    ws = [c['w'].t for c in cases] if master else None
    out = torch.zeros(2 * len(cases), device='cuda') if out is None else out
    ops.lars_norms(*lists, out, slots=slots, grad_scale_dev=gsd, master_params=ws)
    ops.lars_apply(*lists, hp['lr'], hp['momentum'], hp['weight_decay'], hp['trust_coefficient'], hp['eps'], out,
                   slots=slots, grad_scale_dev=gsd, master_params=ws)
    return out


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
        same = c['w'].t.to(pdt).view(torch.int16) == c['p'].t.view(torch.int16)
        start.append(torch.where(same, c['w'].t, c['p'].t.float()))
    ref = [{'p': Slot(s.shape, torch.float32, 0, s, fmt(s.shape)),
            'g': Slot(s.shape, torch.bfloat16 if pdt == torch.bfloat16 else torch.float32, 0, c['g'].t, fmt(s.shape)),
            'v': Slot(s.shape, torch.float32, 0, c['v'].t, fmt(s.shape))}
           for c, s in zip(cases, start)]
    g_before = [c['g'].t.clone() for c in cases]
    for _ in range(3):
        norms = _two_phase(cases, True, gsd=gsd, **hp)
        ref_norms = _two_phase(ref, False, gsd=gsd, **hp)
        torch.cuda.synchronize()
        assert _same(norms, ref_norms)
    for i, (c, r) in enumerate(zip(cases, ref)):
        assert _same(c['w'].t, r['p'].t), (i, 'master')
        assert _same(c['p'].t, r['p'].t.to(pdt)), (i, 'param is not the rounded master')
        assert _same(c['v'].t, r['v'].t), (i, 'momentum')
        assert _same(c['g'].t, g_before[i])
        for k, s in c.items():
            assert s.intact(), (i, 'wrote outside ' + k)


def test_deterministic_no_host_sync_and_fixed_launch_count(hvd):
    ops = _ops()
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
        assert all(_same(a, b) for a, b in zip(*results))


@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
def test_grad_scale_dev(hvd, pair):
    """A device factor of 1 is bit-identical to none; a factor k equals gradients scaled by k (k = 4: exact in every
    gradient dtype), in the norms and in the update alike: a factor that reached one phase only would differ."""
    pdt, gdt = pair
    ops = _ops()

    def run(gscale=1.0, two_phase=False, **kw):
        cases = [_case((n,), pdt, gdt, seed=i) for i, n in enumerate([1, 4097, 1 << 16])]
        for c in cases:
            c['g'].t.mul_(gscale)
        for _ in range(3):
            if two_phase:
                _two_phase(cases, False, gsd=kw.get('grad_scale_dev'), **HP[0])
            else:
                ops.fused_lars_step([c['p'].t for c in cases], [c['g'].t for c in cases], [c['v'].t for c in cases],
                                    0.5, 0.9, 1e-4, 1e-3, 0.0, **kw)
        return [c[k].t for c in cases for k in ('p', 'v')]

    four = torch.tensor([4.0], device='cuda')
    plain, one = run(), run(grad_scale_dev=torch.ones(1, device='cuda'))
    scaled, dev, host = run(gscale=4.0), run(grad_scale_dev=four), run(grad_scale=4.0)
    phases = run(two_phase=True, grad_scale_dev=four)
    assert all(_same(a, b) for a, b in zip(plain, one))
    assert all(_same(a, b) and _same(a, c) and _same(a, d) for a, b, c, d in zip(scaled, dev, host, phases))
    assert not all(_same(a, b) for a, b in zip(plain, scaled))


def test_rejects_bad_arguments(hvd):
    ops = _ops()
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
def _mlp(dtype, seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(24, 48), torch.nn.GELU(), torch.nn.LayerNorm(48),
                               torch.nn.Linear(48, 8)).cuda().to(dtype)


def _loss(m, step, dtype):
    g = torch.Generator(device='cuda').manual_seed(step)
    x = torch.randn(16, 24, device='cuda', generator=g).to(dtype)
    return m(x).float().square().mean()


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
    m = _mlp(dt)
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
        loss = _loss(m, step, dt)
        loss.backward()
        _loss(twin, step, dt).backward()
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
            m = _mlp(dt)
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
            assert _same(p.detach(), q.detach()), (dt, name)
            assert _same(oa.state[p]['momentum_buffer'], ob.state[q]['momentum_buffer']), (dt, name)


def test_checkpoint_round_trip_is_bit_exact(hvd, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    dt = torch.bfloat16

    def fresh():
        m = _mlp(dt)
        return m, hvd.DistributedOptimizer(_lars(hvd, m), named_parameters=m.named_parameters(), fused=True)

    def train(m, o, steps):
        for s in steps:
            o.zero_grad()
            _loss(m, s, dt).backward()
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
        assert _same(a.detach(), c.detach()), name
        assert _same(oa.state[a]['momentum_buffer'], oc.state[c]['momentum_buffer']), name


def test_bf16_master_weights_follow_fp32_twin(hvd):
    """A bf16 model with master_weights=True and an fp32 twin on the fused fp32 kernels, fed the same gradients: the
    masters equal the twin's parameters bit for bit, the parameters are the rounded masters."""
    dt = torch.bfloat16
    m = _mlp(dt)
    twin = copy.deepcopy(m).float()
    opt = hvd.DistributedOptimizer(_lars(hvd, m), named_parameters=m.named_parameters(), master_weights=True)
    topt = hvd.DistributedOptimizer(_lars(hvd, twin), named_parameters=twin.named_parameters(), fused=True)
    for step in range(6):
        opt.zero_grad(set_to_none=True)
        topt.zero_grad(set_to_none=True)
        _loss(m, step, dt).backward()
        for q, p in zip(twin.parameters(), m.parameters()):
            q.grad = p.grad.float()
        opt.step()
        topt.step()
        for (name, p), q in zip(m.named_parameters(), twin.parameters()):
            assert _same(opt.state[p]['master_param'], q.detach()), (name, step)
            assert _same(p.detach(), q.detach().to(dt)), (name, step)
            assert _same(opt.state[p]['momentum_buffer'], topt.state[q]['momentum_buffer']), (name, step)


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
@pytest.fixture
def team(hvd, monkeypatch):
    from horovod_b200.torch import mpi_ops
    t = _SimTeam(4)
    monkeypatch.setattr(mpi_ops, 'symm_empty', lambda numel, dtype, device, process_set: torch.empty(numel, dtype=dtype, device=device))
    monkeypatch.setattr(mpi_ops, 'symm_available', lambda process_set: True)
    monkeypatch.setattr(mpi_ops, 'cross_size', lambda: 1)
    monkeypatch.setattr(mpi_ops, 'captured_reducescatter_', t.reducescatter)
    monkeypatch.setattr(mpi_ops, 'captured_allgather_', t.allgather)
    monkeypatch.setattr(mpi_ops, 'captured_allreduce_', t.allreduce)
    t.opts = []

    def state_allgather(tensor, name, process_set):
        _, _, bi, key = name.split('.', 3)
        return torch.cat([o._buckets[int(bi)]['state'][key] for o in t.opts])
    monkeypatch.setattr(mpi_ops, 'allgather', state_allgather)
    return t


def _batch(step, r, dt):
    g = torch.Generator(device='cuda').manual_seed(100 * step + r)
    return torch.randn(5, 3, 8, 8, device='cuda', generator=g).to(dt), torch.randint(0, 10, (5,), device='cuda', generator=g)


def _make(hvd, m):
    decay = [m.conv.weight, m.fc.weight, m.head.weight]
    return hvd.Lars([{'params': decay, 'weight_decay': 5e-3},
                     {'params': [p for p in m.parameters() if all(p is not q for q in decay)], 'weight_decay': 0.0}],
                    lr=1.0, momentum=0.9, trust_coefficient=0.02)


def _sharded_team(hvd, team, base, dt, master):
    n = team.n
    models = [copy.deepcopy(base) for _ in range(n)]
    opts = [hvd.DistributedOptimizer(_make(hvd, m), named_parameters=m.named_parameters(), shard_optimizer_state=True,
                                     master_weights=master, process_set=_FakeSet(n, r), bucket_cap_mb=0.01 * dt.itemsize / 4)
            for r, m in enumerate(models)]
    team.opts = opts
    # at least one parameter is cut between two ranks' shards, so its norms must cross ranks
    straddle = 0
    for b in opts[0]._buckets:
        for _, off, numel in b['members']:
            straddle += off // b['shard'] != (off + numel - 1) // b['shard']
    assert straddle > 0
    return models, opts


def _reduced_grads(opts, params):
    from horovod_b200.torch.grad_buckets import full_from_shards
    out = {}
    for bi, b in enumerate(opts[0]._buckets):
        full = torch.cat([o._buckets[bi]['gshard'] for o in opts])
        for p, g in zip(b['params'], full_from_shards(b, [full], [p.shape for p in b['params']], [p.stride() for p in b['params']])):
            out[p] = g
    return [out[p] for p in params]


def _step_all(team, models, opts, step, dt, clip=None):
    n = team.n
    for r in range(n):
        opts[r].zero_grad()
        x, y = _batch(step, r, dt)
        torch.nn.functional.cross_entropy(models[r](x), y).backward()
    coef = None
    if clip is not None:
        team.run(lambda r: opts[r].clip_grad_norm_(clip))
        coef = opts[0]._clip_coef.clone()
    else:
        for o in opts:
            o.synchronize()
        team.flush()
    grads = _reduced_grads(opts, list(models[0].parameters()))
    mark = len(team.log)

    def step_rank(r):
        with opts[r].skip_synchronize():
            opts[r].step()
    team.run(step_rank)  # in lockstep: lars_apply must see the allreduced norms
    assert team.count('ar', mark) == n, 'one norms allreduce per rank and step'
    for r in range(1, n):
        for a, b in zip(models[r].parameters(), models[0].parameters()):
            assert _same(a.detach(), b.detach()), 'ranks differ after the allgather'
    return grads, coef


def _ref_step(ref, ref_opt, grads, coef=None):
    ref_opt.zero_grad()
    for p, g in zip(ref.parameters(), grads):
        p.grad = g.clone()
    if coef is None:
        ref_opt.step()
        return
    # the clip coefficient reaches the sharded update on the device; the reference gets it the same way
    from horovod_b200.torch.optimizer import _fused_plan
    from horovod_b200 import ops
    with torch.no_grad():
        for group, ps, gs in _fused_plan(ref_opt):
            st = [ref_opt.state[p] for p in ps]
            for s, p in zip(st, ps):
                if 'momentum_buffer' not in s:
                    s['momentum_buffer'] = torch.zeros_like(p, dtype=torch.float32)
            ops.fused_lars_step(ps, gs, [s['momentum_buffer'] for s in st], group['lr'], group['momentum'],
                                group['weight_decay'], group['trust_coefficient'], group['eps'], ref_opt.adapts(group),
                                grad_scale_dev=coef.reshape(1))


@pytest.mark.parametrize("dt,master", [(torch.float32, False), (torch.bfloat16, True)], ids=['fp32', 'bf16-masters'])
def test_sharded_lars_on_simulated_ranks(hvd, team, dt, master):
    """Sharded LARS against unsharded fused LARS on the reduced gradients over 5 steps, then a sharded -> unsharded and an
    unsharded -> sharded checkpoint that both continue like the reference."""
    torch.manual_seed(0)
    base = _ConvNet().cuda().to(dtype=dt, memory_format=torch.channels_last)
    models, opts = _sharded_team(hvd, team, base, dt, master)
    ref = copy.deepcopy(base)
    ref_opt = hvd.DistributedOptimizer(_make(hvd, ref), named_parameters=ref.named_parameters(), fused=True,
                                       master_weights=master, zero_copy=False)
    tol = dict(rtol=1e-5, atol=1e-6) if dt == torch.float32 else dict(rtol=1e-2, atol=1e-3)

    def check(models, what):
        for (name, a), b in zip(models[0].named_parameters(), ref.parameters()):
            torch.testing.assert_close(a.float(), b.float(), **tol, msg=lambda s: '%s %s: %s' % (what, name, s))

    for step in range(5):
        grads, _ = _step_all(team, models, opts, step, dt)
        _ref_step(ref, ref_opt, grads)
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
    models2, opts2 = _sharded_team(hvd, team, copy.deepcopy(ref), dt, master)
    usd = ref_opt.state_dict()
    for o in opts2:
        o.load_state_dict(usd)
    assert len(opts2[0].state_dict()['state']) == len(sd['state'])  # loaded momentum is state before any step
    grads, _ = _step_all(team, models2, opts2, 5, dt)
    _ref_step(ref, ref_opt, grads)
    _ref_step(un, un_opt, grads)
    check(models2, 'unsharded -> sharded')
    for (name, a), b in zip(un.named_parameters(), models2[0].parameters()):
        torch.testing.assert_close(a.float(), b.float(), **tol, msg=lambda s: 'sharded -> unsharded %s: %s' % (name, s))


def test_sharded_lars_with_clipping(hvd, team):
    """opt.clip_grad_norm_ on the simulated ranks: its coefficient reaches both LARS phases through grad_scale_dev."""
    dt = torch.float32
    torch.manual_seed(0)
    base = _ConvNet().cuda().to(memory_format=torch.channels_last)
    models, opts = _sharded_team(hvd, team, base, dt, False)
    ref = copy.deepcopy(base)
    ref_opt = hvd.DistributedOptimizer(_make(hvd, ref), named_parameters=ref.named_parameters(), fused=True, zero_copy=False)
    for step in range(4):
        grads, coef = _step_all(team, models, opts, step, dt, clip=0.05)
        assert float(coef) < 1.0
        _ref_step(ref, ref_opt, grads, coef)
        for (name, a), b in zip(models[0].named_parameters(), ref.parameters()):
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6, msg=lambda s: 'step %d %s: %s' % (step, name, s))


def test_sharded_lars_with_grad_scaler(hvd, team):
    """fp16 model with masters + ShardedGradScaler: the unscaled shards feed LARS; in step 1 an inf on rank 0 makes
    every rank skip alike."""
    n, dt = team.n, torch.float16
    torch.manual_seed(0)
    base = _ConvNet().cuda().to(dtype=dt, memory_format=torch.channels_last)
    models, opts = _sharded_team(hvd, team, base, dt, True)
    scalers = [hvd.ShardedGradScaler('cuda', init_scale=256.0) for _ in range(n)]
    ref = copy.deepcopy(base)
    ref_opt = hvd.DistributedOptimizer(_make(hvd, ref), named_parameters=ref.named_parameters(), master_weights=True,
                                       zero_copy=False)
    for step in range(4):
        for r in range(n):
            opts[r].zero_grad()
            x, y = _batch(step, r, dt)
            scalers[r].scale(torch.nn.functional.cross_entropy(models[r](x), y)).backward()
        if step == 1:
            opts[0]._buckets[0]['gflat'][0] = math.inf
        before = [s.get_scale() for s in scalers]
        params_before = [p.detach().clone() for p in models[0].parameters()]
        team.run(lambda r: scalers[r].unscale_(opts[r]))
        grads = _reduced_grads(opts, list(models[0].parameters()))
        team.run(lambda r: (scalers[r].step(opts[r]), scalers[r].update()))
        if step == 1:
            assert all(s.get_scale() == before[0] / 2 for s in scalers)
            assert all(_same(a.detach(), b) for a, b in zip(models[0].parameters(), params_before))
        else:
            _ref_step(ref, ref_opt, grads)
        for r in range(n):
            for (name, a), b in zip(models[r].named_parameters(), ref.parameters()):
                torch.testing.assert_close(a.float(), b.float(), rtol=1e-2, atol=1e-3, msg=lambda s: '%s: %s' % (name, s))


def test_trust_norms_buffer_only_for_lamb_and_lars(hvd, team):
    """The sharded optimizer allocates the padded norms buffer for Lamb and Lars only."""
    torch.manual_seed(0)
    base = _ConvNet().cuda()
    models, opts = _sharded_team(hvd, team, base, torch.float32, False)
    assert opts[0]._trust_norms is not None and opts[0]._trust_norms.numel() % (32 * team.n) == 0
    assert opts[0]._trust_norms.numel() >= 2 * len(list(base.parameters()))
    for make in (lambda ps: hvd.Lamb(ps), lambda ps: torch.optim.SGD(ps, lr=0.1, momentum=0.9),
                 lambda ps: torch.optim.AdamW(ps)):
        m = copy.deepcopy(base)
        o = hvd.DistributedOptimizer(make(m.parameters()), named_parameters=m.named_parameters(),
                                     shard_optimizer_state=True, process_set=_FakeSet(team.n, 0))
        assert (o._trust_norms is not None) == isinstance(o, hvd.Lamb)


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_sharded_lars_across_ranks(native_built):
    n = 2 if _ngpu() < 4 else 4
    rc, out = run_parallel("lars_worker.py", np=n, timeout=420)
    assert "LARS OK" in out, out[-4000:]
