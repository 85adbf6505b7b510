"""Fused LAMB: the sm_90a kernels (ops.fused_lamb_step, ops.lamb_norms / ops.lamb_apply) against an fp64 reference,
the master-weight variants against the fp32-parameter kernels bit for bit, DistributedOptimizer(hvd.Lamb(...), fused=True)
against Lamb.step at world size 1, and the sharded (ZeRO-1) LAMB update on 4 simulated ranks against unsharded fused
LAMB; with >= 2 GPUs, across real ranks."""
import copy
import io
import math

import numpy as np
import pytest
import torch

from conftest import run_parallel
from test_gpu_sharded_clip import _FakeSet, _SimTeam

pytestmark = pytest.mark.gpu

PAIRS = [(torch.float32, torch.float32), (torch.float32, torch.bfloat16), (torch.bfloat16, torch.bfloat16),
         (torch.float16, torch.float16)]
PAIR_IDS = ['f32', 'f32-bf16g', 'bf16', 'fp16']
LOW = [torch.bfloat16, torch.float16]
LOW_IDS = ['bf16', 'fp16']
SIZES = [1, 3, 4095, 4096, 4097, (1 << 20) + 3]
HP = [dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.01),
      dict(lr=2e-3, beta1=0.8, beta2=0.99, eps=1e-3, weight_decay=0.1, bias_correction=False),
      dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.0, adapt=False, grad_scale=0.5),
      dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, adapt=True)]
# Depth of the fp32 sums of squares in the kernel: 16 fmas per thread, a 5-level shuffle tree, 8 warps in order (the
# per-CTA partials are then added in fp64).  A sum of k non-negative fp32 terms has a relative error below k * 2^-24.
NORM_RTOL = (16 + 5 + 8) * 2.0 ** -24


def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.fixture(scope="module")
def hvd():
    import horovod_b200.torch as hvd
    hvd.init()
    torch.cuda.set_device(0)
    yield hvd
    hvd.shutdown()


def _ops():
    from horovod_b200 import ops
    return ops


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(_bits(a), _bits(b))


class Slot:
    """A tensor at element `offset` of a larger buffer; the slack around it must come back unchanged."""

    def __init__(self, shape, dtype, offset, fill, memory_format=torch.contiguous_format, slack=67):
        numel = int(np.prod(shape))
        self.buf = torch.randn(offset + numel + slack, device='cuda').to(dtype)
        strides = torch.empty(shape, memory_format=memory_format).stride() if len(shape) == 4 else torch.empty(shape).stride()
        self.t = self.buf.as_strided(shape, strides, offset)
        self.t.copy_(fill)
        self.lo, self.hi = offset, offset + numel
        self.slack = self._slack().clone()

    def _slack(self):
        b = _bits(self.buf)
        return torch.cat([b[:self.lo], b[self.hi:]])

    def intact(self):
        return torch.equal(self._slack(), self.slack)


def _case(shape, pdt, gdt, seed, offsets=(0, 0, 0), memory_format=torch.contiguous_format, master=False):
    g = torch.Generator(device='cuda').manual_seed(seed)
    po, go, so = offsets
    rnd = lambda s: torch.randn(shape, device='cuda', generator=g) * s  # noqa: E731
    w = rnd(0.1)
    c = {'p': Slot(shape, pdt, po, w.to(pdt), memory_format), 'g': Slot(shape, gdt, go, rnd(1.0), memory_format),
         'm': Slot(shape, torch.float32, so, rnd(0.1), memory_format),
         'v': Slot(shape, torch.float32, so + 1, rnd(0.1).square(), memory_format)}
    if master:
        c['w'] = Slot(shape, torch.float32, so + 2, w, memory_format)
    return c


def _f32(x):
    return float(np.float32(x))


def _ref(cases, lr, beta1, beta2, eps, weight_decay, step, bias_correction=True, adapt=True, grad_scale=1.0):
    """fp64 LAMB from the values the kernel reads (parameter and gradient in their dtypes, fp32 moments) and the
    hyper-parameters as the kernel holds them (fp32).  'scale_*' bound the magnitudes that fp32 rounding errors are
    relative to."""
    out = []
    b1, b2, lr, eps, wd = _f32(beta1), _f32(beta2), _f32(lr), _f32(eps), _f32(weight_decay)
    # as the binding forms them (and fused Adam's): 1 - (beta^step rounded to fp32), in fp32
    c1, c2 = (float(np.float32(1) - np.float32(beta1 ** step)), float(np.float32(1) - np.float32(beta2 ** step))) \
        if bias_correction else (1.0, 1.0)
    for c in cases:
        w, g = c['p'].t.double(), c['g'].t.double() * _f32(grad_scale)
        mo, vo = c['m'].t.double(), c['v'].t.double()
        m = b1 * mo + _f32(1 - b1) * g
        v = b2 * vo + _f32(1 - b2) * g * g
        adam = (m / c1) / ((v / c2).sqrt() + eps)
        u = adam + wd * w
        wn, un = float(w.norm()), float(u.norm())
        r = wn / un if adapt and wn > 0 and un > 0 else 1.0
        scale_m = (b1 * mo).abs() + (_f32(1 - b1) * g).abs()  # >= |m|: m's rounding errors are relative to this
        scale_u = (scale_m / c1) / ((v / c2).sqrt() + eps) + (wd * w).abs()
        out.append({'w': w - lr * r * u, 'm': m, 'v': v, 'scale_m': scale_m, 'scale_u': lr * r * scale_u})
    return out


def _ulp(x, dtype):
    """The spacing of `dtype` at |x| (fp64 tensor), subnormals included."""
    mant, emin = {torch.bfloat16: (7, -126), torch.float16: (10, -14), torch.float32: (23, -126)}[dtype]
    e = torch.floor(torch.log2(x.abs().clamp(min=2.0 ** emin))).clamp(min=emin)
    return torch.pow(2.0, e - mant)


def _cat(ts):
    return torch.cat([t.reshape(-1) for t in ts])


def _run_and_check(cases, hp, step):
    ops = _ops()
    pdt = cases[0]['p'].t.dtype
    hp = dict(hp)
    want = _ref(cases, step=step, **hp)
    g_before = [c['g'].t.clone() for c in cases]
    ops.fused_lamb_step([c['p'].t for c in cases], [c['g'].t for c in cases], [c['m'].t for c in cases],
                        [c['v'].t for c in cases], step=step, **hp)
    torch.cuda.synchronize()
    e = {k: _cat([x[k] for x in want]) for k in want[0]}
    got = {k: _cat([c[k].t.double() for c in cases]) for k in ('p', 'm', 'v')}
    # the moments: two or three fp32 roundings of non-cancelling terms (v) or of terms bounded by scale_m (m)
    assert bool(((got['m'] - e['m']).abs() <= 4 * 2.0 ** -24 * e['scale_m']).all())
    assert bool(((got['v'] - e['v']).abs() <= 4 * 2.0 ** -24 * e['v']).all())
    err = (got['p'] - e['w']).abs()
    # the fp32 result: r is off by at most NORM_RTOL (plus the norms' share of u's own error), u by a few fp32 roundings
    # of its terms, and the result is rounded once
    tol = e['scale_u'] * (NORM_RTOL + 32 * 2.0 ** -24) + _ulp(e['w'], torch.float32)
    if pdt != torch.float32:
        # then rounded to nearest in the parameter dtype: one ulp of it (the fp32 bound only matters where w - lr r u
        # cancels to far below |w|)
        tol = tol + _ulp(e['w'], pdt)
    bad = err > tol
    assert not bool(bad.any()), (int(bad.sum()), float((err - tol).max()))
    for i, c in enumerate(cases):
        assert _same(c['g'].t, g_before[i]), (i, 'grad written')
        for k, s in c.items():
            assert s.intact(), (i, 'wrote outside ' + k)


@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("hp", range(len(HP)))
def test_kernel_matches_fp64(hvd, pair, hp):
    """All sizes and ~200 small tensors in one launch, a channels_last tensor; a 10-step trajectory for the first
    hyper-parameter set, 2 steps for the others (each step checked from the state the kernel left)."""
    pdt, gdt = pair
    sizes = SIZES + [int(x) for x in torch.randint(1, 3000, (200,), generator=torch.Generator().manual_seed(hp))]
    cases = [_case((n,), pdt, gdt, seed=i) for i, n in enumerate(sizes)]
    cases.append(_case((8, 6, 5, 3), pdt, gdt, seed=999, memory_format=torch.channels_last))
    for step in range(1, 11 if hp == 0 else 3):
        for i, c in enumerate(cases):
            c['g'].t.copy_(torch.randn(c['g'].t.shape, device='cuda', generator=torch.Generator(device='cuda').manual_seed(1000 * step + i)))
        _run_and_check(cases, HP[hp], step)


@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("offsets", [(1, 0, 0), (0, 1, 0), (0, 0, 1), (2, 3, 1), (3, 2, 3)])
def test_kernel_unaligned_views(hvd, pair, offsets):
    pdt, gdt = pair
    cases = [_case((n,), pdt, gdt, seed=i, offsets=offsets) for i, n in enumerate(SIZES)]
    _run_and_check(cases, HP[0], 3)


def _two_phase(cases, master, slots=None, out=None, gsd=None, **hp):
    """lamb_norms then lamb_apply over `cases`; returns the norms buffer."""
    ops = _ops()
    lists = [[c[k].t for c in cases] for k in ('p', 'g', 'm', 'v')]
    ws = [c['w'].t for c in cases] if master else None
    out = torch.zeros(2 * len(cases), device='cuda') if out is None else out
    ops.lamb_norms(*lists, hp['beta1'], hp['beta2'], hp['eps'], hp['weight_decay'], hp['step'], out, slots=slots,
                   grad_scale_dev=gsd, master_params=ws)
    ops.lamb_apply(*lists, hp['lr'], hp['beta1'], hp['beta2'], hp['eps'], hp['weight_decay'], hp['step'], out, slots=slots,
                   master_params=ws)
    return out


@pytest.mark.parametrize("pdt", LOW, ids=LOW_IDS)
def test_master_kernels_equal_fp32_kernels(hvd, pdt):
    """Masters, moments and norms bit-identical to the fp32-parameter kernel started from the masters; parameters the
    rounded masters.  Some parameter elements are overwritten first: those masters restart from the parameter."""
    hp = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.01, step=4)
    shapes = [(n,) for n in SIZES] + [(8, 6, 5, 3)] + [(n,) for n in range(1, 200, 7)]
    cases = [_case(s, pdt, pdt, seed=i, offsets=(i % 4, (i + 1) % 4, (i + 2) % 4), master=True,
                   memory_format=torch.channels_last if len(s) == 4 else torch.contiguous_format) for i, s in enumerate(shapes)]
    gsd = torch.tensor([0.75], device='cuda')
    for c in cases[:3]:
        c['p'].t.reshape(-1)[::2] = 0.125  # an outside write: these elements restart from the parameter
    start = []
    for c in cases:
        same = c['w'].t.to(pdt).view(torch.int16) == c['p'].t.view(torch.int16)
        start.append(torch.where(same, c['w'].t, c['p'].t.float()))
    ref = [{'p': Slot(s.shape, torch.float32, 0, s, torch.channels_last if s.dim() == 4 else torch.contiguous_format),
            'g': Slot(s.shape, torch.bfloat16 if pdt == torch.bfloat16 else torch.float32, 0, c['g'].t,
                      torch.channels_last if s.dim() == 4 else torch.contiguous_format),
            'm': Slot(s.shape, torch.float32, 0, c['m'].t, torch.channels_last if s.dim() == 4 else torch.contiguous_format),
            'v': Slot(s.shape, torch.float32, 0, c['v'].t, torch.channels_last if s.dim() == 4 else torch.contiguous_format)}
           for c, s in zip(cases, start)]
    g_before = [c['g'].t.clone() for c in cases]
    norms = _two_phase(cases, True, gsd=gsd, **hp)
    ref_norms = _two_phase(ref, False, gsd=gsd, **hp)
    torch.cuda.synchronize()
    assert _same(norms, ref_norms)
    for i, (c, r) in enumerate(zip(cases, ref)):
        assert _same(c['w'].t, r['p'].t), (i, 'master')
        assert _same(c['p'].t, r['p'].t.to(pdt)), (i, 'param is not the rounded master')
        assert _same(c['m'].t, r['m'].t) and _same(c['v'].t, r['v'].t), (i, 'moments')
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
                ops.fused_lamb_step([c['p'].t for c in cases], [c['g'].t for c in cases], [c['m'].t for c in cases],
                                    [c['v'].t for c in cases], 1e-2, 0.9, 0.999, 1e-6, 0.01, 3,
                                    grad_scale_dev=torch.ones(1, device='cuda'))
            finally:
                torch.cuda.set_sync_debug_mode('default')
            assert ops.kernel_launches() - before == 3, 'moments + partials, norms, update: independent of the tensor count'
            torch.cuda.synchronize()
            results.append([c[k].t.clone() for c in cases for k in ('p', 'm', 'v')])
        assert all(_same(a, b) for a, b in zip(*results))


@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
def test_grad_scale_dev(hvd, pair):
    """A device factor of 1 is bit-identical to none; a factor k equals gradients scaled by k (k = 4: exact in every
    gradient dtype, fp16 subnormals included, where 1/4 would not be)."""
    pdt, gdt = pair
    ops = _ops()

    def run(gscale=1.0, **kw):
        cases = [_case((n,), pdt, gdt, seed=i) for i, n in enumerate([1, 4097, 1 << 16])]
        for c in cases:
            c['g'].t.mul_(gscale)
        for step in (1, 2, 3):
            ops.fused_lamb_step([c['p'].t for c in cases], [c['g'].t for c in cases], [c['m'].t for c in cases],
                                [c['v'].t for c in cases], 1e-2, 0.9, 0.999, 1e-6, 0.01, step, **kw)
        return [c[k].t for c in cases for k in ('p', 'm', 'v')]

    plain, one = run(), run(grad_scale_dev=torch.ones(1, device='cuda'))
    scaled, dev = run(gscale=4.0), run(grad_scale_dev=torch.tensor([4.0], device='cuda'))
    host = run(grad_scale=4.0)
    assert all(_same(a, b) for a, b in zip(plain, one))
    assert all(_same(a, b) and _same(a, c) for a, b, c in zip(scaled, dev, host))
    assert not all(_same(a, b) for a, b in zip(plain, scaled))


def test_rejects_bad_arguments(hvd):
    ops = _ops()
    z = lambda n=64, dt=torch.float32: torch.zeros(n, device='cuda', dtype=dt)  # noqa: E731
    pb, gb = z(dt=torch.bfloat16), z(dt=torch.bfloat16)
    hp = (1e-3, 0.9, 0.999, 1e-6, 0.01)

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
    rejects(ops.fused_lamb_step, ones, [z()], [z()], [z(), z()], *hp, 1)                     # list sizes
    rejects(ops.fused_lamb_step, ones, [z()], [z()], [z()], *hp, 0)                           # step 0
    rejects(ops.fused_lamb_step, ones, [z()], [z(dt=torch.bfloat16)], [z()], *hp, 1)           # moment dtype
    rejects(ops.fused_lamb_step, ones, [z(65)], [z()], [z()], *hp, 1)                         # grad size
    rejects(ops.fused_lamb_step, ones, [torch.zeros(64)], [z()], [z()], *hp, 1)               # grad on the host
    rejects(ops.fused_lamb_step, ones, [z()], [z()], [z()], *hp, 1, master_params=[z()])      # masters for fp32 params
    rejects(ops.fused_lamb_step, [pb], [gb], [z()], [z()], *hp, 1, master_params=[z(dt=torch.float16)])
    rejects(ops.fused_lamb_step, [pb], [z()], [z()], [z()], *hp, 1, master_params=[z()])      # fp32 grads with masters
    rejects(ops.fused_lamb_step, ones, [z()], [z()], [z()], *hp, 1, grad_scale_dev=torch.ones(2, device='cuda'))
    rejects(ops.fused_lamb_step, [torch.ones(64, device='cuda', dtype=torch.float64)], [z()], [z()], [z()], *hp, 1)
    b1, b2, eps, wd = 0.9, 0.999, 1e-6, 0.01
    for bad_out, slots in ((torch.zeros(2), None), (z(2, torch.float64), None), (z(4)[::2], None), (z(1), None),
                           (z(4), [2]), (z(4), [-1])):
        rejects(ops.lamb_norms, ones, [z()], [z()], [z()], b1, b2, eps, wd, 1, bad_out, slots=slots)
        rejects(ops.lamb_apply, ones, [z()], [z()], [z()], 1e-3, b1, b2, eps, wd, 1, bad_out, slots=slots)
    rejects(ops.lamb_norms, ones * 2, [z(), z()], [z(), z()], [z(), z()], b1, b2, eps, wd, 1, z(8), slots=[1, 1])
    rejects(ops.lamb_norms, ones, [z()], [z()], [z()], b1, b2, eps, wd, 1, z(8), slots=[0, 1])


# ---- DistributedOptimizer at world size 1 -------------------------------------------------------------------------------
def _mlp(dtype, seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(24, 48), torch.nn.GELU(), torch.nn.LayerNorm(48),
                               torch.nn.Linear(48, 8)).cuda().to(dtype)


def _loss(m, step, dtype):
    g = torch.Generator(device='cuda').manual_seed(step)
    x = torch.randn(16, 24, device='cuda', generator=g).to(dtype)
    return m(x).float().square().mean()


def _lamb(hvd, m):
    """BERT-style groups: weight decay on the matrices, none (so no trust ratio) on biases and LayerNorm; the always_adapt
    group covers the other branch."""
    decay = [p for n, p in m.named_parameters() if n.endswith('weight') and p.dim() == 2]
    ln = list(m[2].parameters())
    rest = [p for p in m.parameters() if all(p is not q for q in decay + ln)]
    return hvd.Lamb([{'params': decay, 'weight_decay': 0.01}, {'params': rest}, {'params': ln, 'always_adapt': True}],
                    lr=1e-2, eps=1e-6)


def test_fused_optimizer_follows_lamb_step(hvd):
    """fused=True against Lamb.step over 10 steps: broadcast_optimizer_state first, the last Linear frozen for 3 steps
    (its own step count), step(closure) twice."""
    dt = torch.float32
    m = _mlp(dt)
    twin = copy.deepcopy(m)
    for x in (m, twin):
        x[3].requires_grad_(False)  # before the optimizer is built: it gets no gradient bucket, so no zero gradient
    opt = hvd.DistributedOptimizer(_lamb(hvd, m), named_parameters=m.named_parameters(), fused=True)
    ref = _lamb(hvd, twin)
    for o in (opt, ref):
        hvd.broadcast_optimizer_state(o, root_rank=0)
    launches = []
    for step in range(10):
        if step == 3:
            for x in (m, twin):
                x[3].requires_grad_(True)
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
    assert int(opt.state[m[3].weight]['step']) == 7 and int(opt.state[m[0].weight]['step']) == 11
    # step 5: three launches per group and step count (two counts in two groups, one in the LayerNorm group), so the
    # fused kernels ran and not Lamb.step
    assert launches[5] >= 15, launches
    assert all(opt.state[p]['exp_avg'].dtype == torch.float32 for p in m.parameters())


def test_checkpoint_round_trip_is_bit_exact(hvd, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    dt = torch.bfloat16

    def fresh():
        m = _mlp(dt)
        return m, hvd.DistributedOptimizer(_lamb(hvd, m), named_parameters=m.named_parameters(), fused=True)

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
    assert all(oc.state[p]['exp_avg'].dtype == torch.float32 for p in mc.parameters())  # not cast to bf16
    train(mc, oc, range(3, 6))
    for (name, a), c in zip(ma.named_parameters(), mc.parameters()):
        assert _same(a.detach(), c.detach()), name
        for key in ('exp_avg', 'exp_avg_sq'):
            assert _same(oa.state[a][key], oc.state[c][key]), (name, key)


def test_bf16_master_weights_follow_fp32_twin(hvd):
    """A bf16 model with master_weights=True and an fp32 twin on the fused fp32 kernel, fed the same gradients: the
    masters equal the twin's parameters bit for bit, the parameters are the rounded masters."""
    dt = torch.bfloat16
    m = _mlp(dt)
    twin = copy.deepcopy(m).float()
    opt = hvd.DistributedOptimizer(_lamb(hvd, m), named_parameters=m.named_parameters(), master_weights=True)
    topt = hvd.DistributedOptimizer(_lamb(hvd, twin), named_parameters=twin.named_parameters(), fused=True)
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


def test_unfusable_plan_falls_back_or_raises(hvd):
    """A CPU model: fused=True falls back to Lamb.step; master_weights=True raises instead."""
    cpu = torch.nn.Linear(4, 4)
    twin = copy.deepcopy(cpu)
    opt = hvd.DistributedOptimizer(hvd.Lamb(cpu.parameters(), weight_decay=0.01), named_parameters=cpu.named_parameters(),
                                   fused=True)
    ref = hvd.Lamb(twin.parameters(), weight_decay=0.01)
    x = torch.randn(2, 4)
    for mod, o in ((cpu, opt), (twin, ref)):
        mod(x).sum().backward()
        o.step()
    assert torch.equal(cpu.weight, twin.weight)
    half = torch.nn.Linear(4, 4).to(torch.bfloat16)
    mo = hvd.DistributedOptimizer(hvd.Lamb(half.parameters()), named_parameters=half.named_parameters(), master_weights=True)
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


class _ConvNet(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3)
        self.fc = torch.nn.Linear(8 * 6 * 6, 10)
        self.norm = torch.nn.LayerNorm(10)
        self.head = torch.nn.Linear(10, 10)

    def forward(self, x):
        return self.head(self.norm(self.fc(torch.relu(self.conv(x)).flatten(1))))


def _batch(step, r, dt):
    g = torch.Generator(device='cuda').manual_seed(100 * step + r)
    return torch.randn(5, 3, 8, 8, device='cuda', generator=g).to(dt), torch.randint(0, 10, (5,), device='cuda', generator=g)


def _make(hvd, m):
    decay = [m.conv.weight, m.fc.weight, m.head.weight]
    return hvd.Lamb([{'params': decay, 'weight_decay': 0.05}, {'params': [p for p in m.parameters() if all(p is not q for q in decay)]}],
                    lr=1e-2, eps=1e-6)


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
    team.run(step_rank)  # in lockstep: lamb_apply must see the allreduced norms
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
                if 'exp_avg' not in s:
                    s['step'] = torch.tensor(0.0)
                    s['exp_avg'] = torch.zeros_like(p, dtype=torch.float32)
                    s['exp_avg_sq'] = torch.zeros_like(p, dtype=torch.float32)
                s['step'] += 1
            b1, b2 = group['betas']
            ops.fused_lamb_step(ps, gs, [s['exp_avg'] for s in st], [s['exp_avg_sq'] for s in st], group['lr'], b1, b2,
                                group['eps'], group['weight_decay'], int(st[0]['step']), group['bias_correction'],
                                ref_opt.adapts(group), grad_scale_dev=coef.reshape(1))


@pytest.mark.parametrize("dt,master", [(torch.float32, False), (torch.bfloat16, True)], ids=['fp32', 'bf16-masters'])
def test_sharded_lamb_on_simulated_ranks(hvd, team, dt, master):
    """Sharded LAMB against unsharded fused LAMB on the reduced gradients over 5 steps, then a sharded -> unsharded and an
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
    assert all(set(st) >= {'exp_avg', 'exp_avg_sq', 'step'} and (('master_param' in st) == master) for st in sd['state'].values())
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
    grads, _ = _step_all(team, models2, opts2, 5, dt)
    _ref_step(ref, ref_opt, grads)
    _ref_step(un, un_opt, grads)
    check(models2, 'unsharded -> sharded')
    for (name, a), b in zip(un.named_parameters(), models2[0].parameters()):
        torch.testing.assert_close(a.float(), b.float(), **tol, msg=lambda s: 'sharded -> unsharded %s: %s' % (name, s))


def test_sharded_lamb_with_clipping(hvd, team):
    """opt.clip_grad_norm_ on the simulated ranks: its coefficient reaches LAMB's first phase through grad_scale_dev."""
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


def test_sharded_lamb_with_grad_scaler(hvd, team):
    """fp16 model with masters + ShardedGradScaler: the unscaled shards feed LAMB; in step 1 an inf on rank 0 makes
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
        team.run(lambda r: scalers[r].unscale_(opts[r]))
        grads = _reduced_grads(opts, list(models[0].parameters()))
        team.run(lambda r: (scalers[r].step(opts[r]), scalers[r].update()))
        if step == 1:
            assert all(s.get_scale() == before[0] / 2 for s in scalers)
        else:
            _ref_step(ref, ref_opt, grads)
        for r in range(n):
            for (name, a), b in zip(models[r].named_parameters(), ref.parameters()):
                torch.testing.assert_close(a.float(), b.float(), rtol=1e-2, atol=1e-3, msg=lambda s: '%s: %s' % (name, s))


def test_trust_norms_buffer_only_for_lamb(hvd, team):
    """The sharded optimizer allocates the padded norms buffer for Lamb only."""
    torch.manual_seed(0)
    base = _ConvNet().cuda()
    models, opts = _sharded_team(hvd, team, base, torch.float32, False)
    assert opts[0]._trust_norms is not None and opts[0]._trust_norms.numel() % (32 * team.n) == 0
    m = copy.deepcopy(base)
    o = hvd.DistributedOptimizer(torch.optim.AdamW(m.parameters()), named_parameters=m.named_parameters(),
                                 shard_optimizer_state=True, process_set=_FakeSet(team.n, 0))
    assert o._trust_norms is None


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_sharded_lamb_across_ranks(native_built):
    n = 2 if _ngpu() < 4 else 4
    rc, out = run_parallel("lamb_worker.py", np=n, timeout=420)
    assert "LAMB OK" in out, out[-4000:]
