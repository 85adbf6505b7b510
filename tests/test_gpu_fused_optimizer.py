"""The fused SGD / Adam(W) kernels (csrc/kernels/optim_kernels.cu) against a float64 reference of the same update.

The reference mirrors the kernels' storage contract: parameters are rounded to their dtype after every step, Adam moments
are fp32, SGD momentum is stored in the parameter dtype, and hyper-parameters reach the kernel as fp32 (the bias
corrections are computed in double on the host and passed as fp32). Besides the value it returns an error scale per
element: the same expression evaluated on the magnitudes of its terms, so a tolerance relative to it stays meaningful
where terms cancel.

Tolerances: fp32 parameters and fp32 moments within 1e-6 of that scale per step (1e-5 over a 10-step trajectory);
bf16 / fp16 parameters and momentum within one ulp of their dtype, each step starting from the kernel's own previous
state. Every tensor lives inside a larger buffer whose slack must come back unchanged.
"""
import io
import itertools

import numpy as np
import pytest
import torch

from optim_cases import COUNTS, PAIRS, Slot, adam_ref, adam_ref_kernel, f32, hvd, ulp  # noqa: F401  (hvd: fixture)

# ---------------------------------------------------------------------------------------------------------------------
# float64 reference


def sgd_ref(p, g, buf, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, grad_scale=1.0,
            first_step=False):
    """One SGD step on float64 tensors. Returns (p, buf, p_scale, buf_scale); buf is None without momentum. As in torch,
    the first momentum step stores buf = d without dampening."""
    d = g * grad_scale
    ds = d.abs()
    if weight_decay != 0:
        d = d + weight_decay * p
        ds = ds + abs(weight_decay) * p.abs()
    bs = None
    if momentum != 0:
        if first_step:
            buf, bs = d, ds
        else:
            buf, bs = momentum * buf + (1 - dampening) * d, abs(momentum) * buf.abs() + abs(1 - dampening) * ds
        if nesterov:
            d, ds = d + momentum * buf, ds + abs(momentum) * bs
        else:
            d, ds = buf, bs
    return p - lr * d, buf, p.abs() + abs(lr) * ds, bs


def sgd_ref_kernel(p, g, buf, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, grad_scale=1.0,
                   first_step=False):
    """sgd_ref with the hyper-parameters the kernel receives (fp32)."""
    return sgd_ref(p, g, buf, f32(lr), f32(momentum), f32(dampening), f32(weight_decay), nesterov, f32(grad_scale),
                   first_step)


def test_reference_matches_torch_optim_in_float64():
    """The reference itself, on the CPU: 10 steps against torch.optim in float64, every hyper-parameter path."""
    torch.manual_seed(0)
    n = 257
    p0 = torch.randn(n, dtype=torch.float64)
    grads = [torch.randn(n, dtype=torch.float64) for _ in range(10)]

    def run_torch(opt_cls, **kw):
        p = torch.nn.Parameter(p0.clone())
        opt = opt_cls([p], foreach=False, **kw)
        for g in grads:
            p.grad = g.clone()
            opt.step()
        return p.detach(), opt.state[p]

    sgd_cases = [dict(lr=0.05), dict(lr=0.05, momentum=0.9), dict(lr=0.05, momentum=0.9, dampening=0.5),
                 dict(lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-2), dict(lr=0.05, weight_decay=1e-2)]
    for kw in sgd_cases:
        want, st = run_torch(torch.optim.SGD, **kw)
        p, buf = p0.clone(), None
        for i, g in enumerate(grads):
            p, buf, _, _ = sgd_ref(p, g, buf, first_step=i == 0, **kw)
        torch.testing.assert_close(p, want, rtol=1e-12, atol=1e-12, msg=lambda m: f'SGD {kw}: {m}')
        if kw.get('momentum'):
            torch.testing.assert_close(buf, st['momentum_buffer'], rtol=1e-12, atol=1e-12)
    # grad_scale is the kernel's folded gradient post-division: the same as scaling every gradient
    p, buf = p0.clone(), None
    q, qbuf = p0.clone(), None
    for i, g in enumerate(grads):
        p, buf, _, _ = sgd_ref(p, g, buf, 0.05, 0.9, first_step=i == 0, grad_scale=0.25)
        q, qbuf, _, _ = sgd_ref(q, g * 0.25, qbuf, 0.05, 0.9, first_step=i == 0)
    torch.testing.assert_close(p, q, rtol=1e-15, atol=1e-15)

    for opt_cls, adamw in ((torch.optim.Adam, False), (torch.optim.AdamW, True)):
        for kw in (dict(lr=1e-2), dict(lr=1e-2, weight_decay=1e-2), dict(lr=1e-3, eps=1e-3, weight_decay=0.1, betas=(0.8, 0.99))):
            want, st = run_torch(opt_cls, **kw)
            kw = dict(kw)
            wd = kw.pop('weight_decay', 1e-2 if adamw else 0.0)  # AdamW's default decay is 1e-2
            b1, b2 = kw.pop('betas', (0.9, 0.999))
            p, m, v = p0.clone(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
            for i, g in enumerate(grads):
                p, m, v, _, _, _ = adam_ref(p, g, m, v, beta1=b1, beta2=b2, weight_decay=wd, step=i + 1, adamw=adamw, **kw)
            torch.testing.assert_close(p, want, rtol=1e-12, atol=1e-12, msg=lambda msg: f'{opt_cls.__name__} {kw}: {msg}')
            torch.testing.assert_close(m, st['exp_avg'], rtol=1e-12, atol=1e-12)
            torch.testing.assert_close(v, st['exp_avg_sq'], rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------------------------------------------------------------
# helpers for the kernel tests

def check(name, got, ref, scale, dtype, rtol=1e-6):
    """got (kernel, any dtype) against ref (float64). fp32: |got - ref| <= rtol * scale. bf16 / fp16: within one ulp of
    the reference rounded to the dtype, plus the fp32 arithmetic error of the kernel before its final rounding."""
    got, ref, scale = got.double().flatten(), ref.flatten(), scale.flatten()
    if dtype == torch.float32:
        allowed = rtol * scale
        want = ref
    else:
        want = ref.to(dtype).double()
        allowed = ulp(want, dtype) + rtol * scale
    err = (got - want).abs()
    bad = ~(err <= allowed)  # NaN counts as bad
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError(f'{name}: {int(bad.sum())}/{got.numel()} elements off, first at {i}: got {got[i].item()!r} '
                             f'want {want[i].item()!r} (err {err[i].item():.3e} > {allowed[i].item():.3e})')


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _make(shape, pdt, gdt, seed, offsets=(0, 0, 0), memory_format=torch.contiguous_format, sgd=False):
    """Param / grad / state slots for one tensor: p ~ 0.1 N(0, 1), g ~ N(0, 1), state from earlier steps."""
    g = _gen(seed)
    po, go, so = offsets
    n = int(np.prod(shape)) if len(shape) else 1
    rnd = lambda scale: (torch.randn(n, device='cuda', generator=g, dtype=torch.float64) * scale).reshape(shape)  # noqa: E731
    slots = {'p': Slot(shape, pdt, po, rnd(0.1), memory_format), 'g': Slot(shape, gdt, go, rnd(1.0), memory_format)}
    if sgd:
        slots['buf'] = Slot(shape, pdt, so, rnd(0.5), memory_format)
    else:
        slots['m'] = Slot(shape, torch.float32, so, rnd(0.1), memory_format)
        slots['v'] = Slot(shape, torch.float32, so + 1, rnd(0.1).square(), memory_format)
    return slots


def _intact(name, slots):
    for k, s in slots.items():
        assert s.intact(), f'{name}: the kernel wrote outside {k}'


def run_sgd(tensors, pdt, **hp):
    """One fused SGD call over `tensors` (lists of slot dicts) and the reference check of every tensor."""
    from horovod_b200 import ops
    has_mom = hp.get('momentum', 0.0) != 0.0
    before = [{k: s.t.double().clone() for k, s in sl.items()} for sl in tensors]
    ops.fused_sgd_step([sl['p'].t for sl in tensors], [sl['g'].t for sl in tensors],
                       [sl['buf'].t for sl in tensors] if has_mom else [], **hp)
    torch.cuda.synchronize()
    for i, (sl, b) in enumerate(zip(tensors, before)):
        p, buf, ps, bs = sgd_ref_kernel(b['p'], b['g'], b['buf'] if has_mom else None, **hp)
        check(f'sgd[{i}] param {hp}', sl['p'].t, p, ps, pdt)
        if has_mom:
            check(f'sgd[{i}] momentum {hp}', sl['buf'].t, buf, bs, pdt)
        elif 'buf' in sl:
            assert torch.equal(sl['buf'].t.double(), b['buf']), 'momentum buffer written without momentum'
        _intact(f'sgd[{i}] {hp}', sl)


def run_adam(tensors, pdt, **hp):
    from horovod_b200 import ops
    before = [{k: s.t.double().clone() for k, s in sl.items()} for sl in tensors]
    ops.fused_adam_step([sl['p'].t for sl in tensors], [sl['g'].t for sl in tensors], [sl['m'].t for sl in tensors],
                        [sl['v'].t for sl in tensors], **hp)
    torch.cuda.synchronize()
    for i, (sl, b) in enumerate(zip(tensors, before)):
        p, m, v, ps, ms, vs = adam_ref_kernel(b['p'], b['g'], b['m'], b['v'], **hp)
        check(f'adam[{i}] param {hp}', sl['p'].t, p, ps, pdt)
        check(f'adam[{i}] exp_avg {hp}', sl['m'].t, m, ms, torch.float32)
        check(f'adam[{i}] exp_avg_sq {hp}', sl['v'].t, v, vs, torch.float32)
        _intact(f'adam[{i}] {hp}', sl)


DTYPE_IDS = ['fp32-fp32', 'fp32-bf16', 'bf16-bf16', 'fp16-fp16']

SGD_HP = dict(lr=0.05, momentum=0.9, dampening=0.5, weight_decay=1e-2, grad_scale=0.25)
ADAM_HP = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2)

# ---------------------------------------------------------------------------------------------------------------------
# the kernel matrix


@pytest.mark.gpu
@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("dtypes", PAIRS, ids=DTYPE_IDS)
def test_sgd_dtypes_and_counts(hvd, dtypes, count):
    pdt, gdt = dtypes
    t = [_make((count,), pdt, gdt, seed=count, sgd=True)]
    run_sgd(t, pdt, first_step=True, **SGD_HP)  # buf = d
    run_sgd(t, pdt, nesterov=True, **dict(SGD_HP, dampening=0.0))
    run_sgd(t, pdt, **SGD_HP)


@pytest.mark.gpu
@pytest.mark.parametrize("adamw", [True, False], ids=['adamw', 'adam'])
@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("dtypes", PAIRS, ids=DTYPE_IDS)
def test_adam_dtypes_and_counts(hvd, dtypes, count, adamw):
    pdt, gdt = dtypes
    t = [_make((count,), pdt, gdt, seed=count + 7)]
    for step in (1, 2, 3):
        run_adam(t, pdt, step=step, adamw=adamw, **ADAM_HP)


# (param, grad, state) storage offsets in elements: 16 B vectors are unusable for the shifted tensors only
OFFSETS = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (2, 0, 0), (0, 2, 2), (3, 3, 3), (0, 3, 0), (3, 0, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("offsets", OFFSETS, ids=[f'p{a}g{b}s{c}' for a, b, c in OFFSETS])
@pytest.mark.parametrize("dtypes", PAIRS, ids=DTYPE_IDS)
def test_unaligned_views(hvd, dtypes, offsets):
    pdt, gdt = dtypes
    for count in (5, 4097):
        run_sgd([_make((count,), pdt, gdt, seed=count, offsets=offsets, sgd=True)], pdt, **SGD_HP)
        run_adam([_make((count,), pdt, gdt, seed=count, offsets=offsets)], pdt, step=4, **ADAM_HP)


def _many_sizes():
    """~200 sizes from 0 to 2^20 elements: most CTAs of grid.y (sized for the largest tensor) exit at once."""
    rng = np.random.default_rng(5)
    sizes = [0, 1, 2, 3, 4, 5, 7, 8, 4095, 4096, 4097, 1 << 20]
    sizes += [int(x) for x in rng.integers(1, 70000, size=180)]
    sizes += [int(x) for x in rng.integers(0, 4, size=8)]
    return sizes


@pytest.mark.gpu
@pytest.mark.parametrize("dtypes", PAIRS, ids=DTYPE_IDS)
def test_many_tensors_in_one_launch(hvd, dtypes):
    pdt, gdt = dtypes
    sizes = _many_sizes()
    offs = [(i % 4, (i // 4) % 4, (i // 16) % 4) for i in range(len(sizes))]
    before = hvd.runtime_stats()['kernel_launches']
    run_sgd([_make((n,), pdt, gdt, seed=i, offsets=o, sgd=True) for i, (n, o) in enumerate(zip(sizes, offs))], pdt,
            nesterov=True, **dict(SGD_HP, dampening=0.0))
    run_adam([_make((n,), pdt, gdt, seed=i, offsets=o) for i, (n, o) in enumerate(zip(sizes, offs))], pdt, step=7,
             adamw=False, **ADAM_HP)
    assert hvd.runtime_stats()['kernel_launches'] - before == 2


@pytest.mark.gpu
@pytest.mark.parametrize("dtypes", PAIRS, ids=DTYPE_IDS)
def test_channels_last(hvd, dtypes):
    pdt, gdt = dtypes
    cl = torch.channels_last
    shapes = [(64, 32, 3, 3), (7, 5, 3, 3), (8, 3, 1, 1)]
    for i, shape in enumerate(shapes):
        sl = _make(shape, pdt, gdt, seed=i, offsets=(i, 0, 0), memory_format=cl, sgd=True)
        assert sl['p'].t.is_contiguous(memory_format=cl) and sl['g'].t.stride() == sl['p'].t.stride()
        assert i == 2 or not sl['p'].t.is_contiguous()
        run_sgd([sl], pdt, **SGD_HP)
        run_adam([_make(shape, pdt, gdt, seed=i, memory_format=cl)], pdt, step=2, **ADAM_HP)


@pytest.mark.gpu
@pytest.mark.parametrize("pdt", [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
def test_sgd_hyperparameters(hvd, pdt):
    for mom, damp, nest, wd, first, gs in itertools.product((0.0, 0.9), (0.0, 0.5), (False, True), (0.0, 1e-2),
                                                           (False, True), (1.0, 0.25)):
        run_sgd([_make((4097,), pdt, pdt, seed=3, sgd=True)], pdt, lr=0.05, momentum=mom, dampening=damp, nesterov=nest,
                weight_decay=wd, first_step=first, grad_scale=gs)


@pytest.mark.gpu
@pytest.mark.parametrize("pdt", [torch.float32, torch.bfloat16, torch.float16], ids=['fp32', 'bf16', 'fp16'])
def test_adam_hyperparameters(hvd, pdt):
    for adamw, eps, step, wd, gs in itertools.product((False, True), (1e-8, 1e-3), (1, 1000), (0.0, 1e-2), (1.0, 0.25)):
        run_adam([_make((4097,), pdt, pdt, seed=4)], pdt, lr=1e-2, eps=eps, step=step, weight_decay=wd, adamw=adamw,
                 grad_scale=gs)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sgd", "adam", "adamw"])
def test_fp32_trajectory(hvd, kind):
    """10 steps of the kernel against 10 steps of the reference (parameters and moments stored as fp32 in between)."""
    from horovod_b200 import ops
    n = (1 << 16) + 5
    sl = _make((n,), torch.float32, torch.float32, seed=11, offsets=(1, 2, 3), sgd=kind == 'sgd')
    ref = {k: s.t.double().clone() for k, s in sl.items()}
    if kind == 'sgd':
        ref['buf'] = None
    worst = torch.zeros(n, dtype=torch.float64, device='cuda')
    for step in range(1, 11):
        g = torch.randn(n, device='cuda', generator=_gen(step))
        sl['g'].t.copy_(g)
        if kind == 'sgd':
            hp = dict(lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-2)
            ops.fused_sgd_step([sl['p'].t], [sl['g'].t], [sl['buf'].t], first_step=step == 1, **hp)
            p, buf, ps, _ = sgd_ref_kernel(ref['p'], g.double(), ref['buf'], first_step=step == 1, **hp)
            ref.update(p=p.float().double(), buf=buf.float().double())
        else:
            hp = dict(ADAM_HP, adamw=kind == 'adamw', step=step)
            ops.fused_adam_step([sl['p'].t], [sl['g'].t], [sl['m'].t], [sl['v'].t], **hp)
            p, m, v, ps, _, _ = adam_ref_kernel(ref['p'], g.double(), ref['m'], ref['v'], **hp)
            ref.update(p=p.float().double(), m=m.float().double(), v=v.float().double())
        worst = torch.maximum(worst, ps)
    torch.cuda.synchronize()
    check(f'{kind} after 10 steps', sl['p'].t, ref['p'], worst, torch.float32, rtol=1e-5)
    _intact(kind, sl)


# ---------------------------------------------------------------------------------------------------------------------
# rejected on the host, before anything is staged or launched


def _rejects(hvd, fn, *args, **kw):
    before = hvd.runtime_stats()['kernel_launches']
    with pytest.raises(RuntimeError):
        fn(*args, **kw)
    torch.cuda.synchronize()
    assert hvd.runtime_stats()['kernel_launches'] == before


@pytest.mark.gpu
def test_adam_rejects_bad_arguments(hvd):
    from horovod_b200 import ops
    adam = ops.fused_adam_step
    z = lambda n=64, dt=torch.float32, **kw: torch.zeros(n, device='cuda', dtype=dt, **kw)  # noqa: E731
    p, g = z(), z()
    p0 = p.clone()
    _rejects(hvd, adam, [p], [g], [z(dt=torch.bfloat16)], [z()], lr=1e-3)         # bf16 exp_avg
    _rejects(hvd, adam, [p], [g], [z()], [z(dt=torch.float16)], lr=1e-3)          # fp16 exp_avg_sq
    _rejects(hvd, adam, [p], [z(65)], [z()], [z()], lr=1e-3)                      # grad larger than its param
    _rejects(hvd, adam, [p], [z(63)], [z()], [z()], lr=1e-3)                      # grad smaller than its param
    _rejects(hvd, adam, [p], [g], [z(65)], [z()], lr=1e-3)                        # state numel
    _rejects(hvd, adam, [p], [g.view(8, 8)], [z()], [z()], lr=1e-3)               # same numel, other size
    _rejects(hvd, adam, [p], [g], [z()], [z()], lr=1e-3, step=0)                  # c1 = 0
    _rejects(hvd, adam, [p], [g], [z()], [z()], lr=1e-3, step=-3)
    _rejects(hvd, adam, [p, z()], [g], [z(), z()], [z(), z()], lr=1e-3)           # list lengths
    _rejects(hvd, adam, [p, z()], [g, z()], [z()], [z(), z()], lr=1e-3)
    _rejects(hvd, adam, [p, z()], [g, z()], [z(), z()], [z()], lr=1e-3)
    _rejects(hvd, adam, [p, z(dt=torch.bfloat16)], [g, z(dt=torch.bfloat16)], [z(), z()], [z(), z()], lr=1e-3)  # params
    _rejects(hvd, adam, [p, z()], [g, z(dt=torch.bfloat16)], [z(), z()], [z(), z()], lr=1e-3)  # mixed grad dtypes
    _rejects(hvd, adam, [p], [torch.zeros(64)], [z()], [z()], lr=1e-3)            # grad on the host
    _rejects(hvd, adam, [p], [g], [torch.zeros(64)], [z()], lr=1e-3)              # state on the host
    _rejects(hvd, adam, [p], [z(dt=torch.float16)], [z()], [z()], lr=1e-3)        # no fp32-param / fp16-grad kernel
    w = torch.zeros(4, 8, 3, 3, device='cuda').to(memory_format=torch.channels_last)
    _rejects(hvd, adam, [w], [torch.zeros_like(w)], [torch.zeros(4, 8, 3, 3, device='cuda')], [torch.zeros_like(w)],
             lr=1e-3)                                                             # state strides differ from the param's
    _rejects(hvd, adam, [w], [torch.zeros(4, 8, 3, 3, device='cuda')], [torch.zeros_like(w)], [torch.zeros_like(w)],
             lr=1e-3)                                                             # grad strides
    assert torch.equal(p, p0)
    adam([], [], [], [], lr=1e-3)  # an empty list is a no-op


@pytest.mark.gpu
def test_sgd_rejects_bad_arguments(hvd):
    from horovod_b200 import ops
    sgd = ops.fused_sgd_step
    z = lambda n=64, dt=torch.float32: torch.zeros(n, device='cuda', dtype=dt)  # noqa: E731
    pb, gb = z(dt=torch.bfloat16), z(dt=torch.bfloat16)
    _rejects(hvd, sgd, [pb], [gb], [z()], lr=0.1, momentum=0.9)                  # momentum dtype != param dtype
    _rejects(hvd, sgd, [pb], [gb], [z(65, torch.bfloat16)], lr=0.1, momentum=0.9)  # momentum numel
    _rejects(hvd, sgd, [pb], [z(65, torch.bfloat16)], [], lr=0.1)                 # grad larger than its param
    _rejects(hvd, sgd, [pb, z(dt=torch.bfloat16)], [gb, z(dt=torch.bfloat16)], [z(dt=torch.bfloat16)], lr=0.1,
             momentum=0.9)                                                        # momentum list too short
    _rejects(hvd, sgd, [pb, z(dt=torch.bfloat16)], [gb], [], lr=0.1)              # grads list too short
    _rejects(hvd, sgd, [z(), pb], [z(), gb], [], lr=0.1)                          # mixed param dtypes
    _rejects(hvd, sgd, [z(), z()], [z(), gb], [], lr=0.1)                         # mixed grad dtypes
    _rejects(hvd, sgd, [z()], [torch.zeros(64)], [], lr=0.1)                      # grad on the host
    _rejects(hvd, sgd, [z()], [z()], [torch.zeros(64)], lr=0.1, momentum=0.9)     # momentum on the host
    w = torch.zeros(4, 8, 3, 3, device='cuda').to(memory_format=torch.channels_last)
    _rejects(hvd, sgd, [w], [torch.zeros_like(w)], [torch.zeros(4, 8, 3, 3, device='cuda')], lr=0.1, momentum=0.9)
    _rejects(hvd, sgd, [w], [torch.zeros(4, 8, 3, 3, device='cuda')], [], lr=0.1)


# ---------------------------------------------------------------------------------------------------------------------
# end to end at world size 1: hvd.DistributedOptimizer(..., fused=True)


class _Net(torch.nn.Module):
    """A Linear layer, a channels_last Conv2d and a LayerNorm; `late` joins the forward only when asked."""

    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3, padding=1)
        self.norm = torch.nn.LayerNorm(8)
        self.fc = torch.nn.Linear(8, 5)
        self.late = torch.nn.Linear(8, 5)

    def forward(self, x, use_late=True):
        y = self.norm(self.conv(x).mean((2, 3)))
        return self.fc(y) + self.late(y) if use_late else self.fc(y)


def _net(dtype):
    torch.manual_seed(0)
    return _Net().cuda().to(dtype=dtype, memory_format=torch.channels_last)


def _loss(model, step, dtype, use_late=True):
    g = _gen(1000 + step)
    x = torch.randn(6, 3, 5, 5, device='cuda', generator=g).to(dtype).contiguous(memory_format=torch.channels_last)
    return model(x, use_late).float().square().mean()


def _adamw(model):
    return torch.optim.AdamW(model.parameters(), lr=1e-2, weight_decay=0.05)


def _sgd(model):
    return torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-3)


def _dist(hvd, opt, model):
    return hvd.DistributedOptimizer(opt, named_parameters=model.named_parameters(), fused=True)


def _fused_adam_step_checked(opt, model, dtype, step_count, adamw=True, weight_decay=0.05):
    """opt.step() and, for every parameter, the reference Adam(W) step fed with the same inputs: fp32 moments with the
    parameter's strides afterwards, step count `step_count`."""
    before = {}
    for p in model.parameters():
        st = opt.state[p]
        before[p] = (p.detach().double().clone(), st['exp_avg'].double().clone(), st['exp_avg_sq'].double().clone())
    opt.step()
    torch.cuda.synchronize()
    for name, p in model.named_parameters():
        st = opt.state[p]
        assert st['exp_avg'].dtype == torch.float32 and st['exp_avg_sq'].dtype == torch.float32, name
        assert st['exp_avg'].stride() == p.stride() and st['exp_avg_sq'].stride() == p.stride(), name
        assert int(st['step']) == step_count, (name, float(st['step']), step_count)
        p0, m0, v0 = before[p]
        pr, mr, vr, ps, ms, vs = adam_ref_kernel(p0, p.grad.double(), m0, v0, lr=1e-2, weight_decay=weight_decay,
                                                 step=step_count, adamw=adamw)
        check(f'{name} step {step_count}', p, pr, ps, dtype)
        check(f'{name} exp_avg step {step_count}', st['exp_avg'], mr, ms, torch.float32)
        check(f'{name} exp_avg_sq step {step_count}', st['exp_avg_sq'], vr, vs, torch.float32)


DT3 = [torch.float32, torch.bfloat16, torch.float16]
DT3_IDS = ['fp32', 'bf16', 'fp16']


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DT3, ids=DT3_IDS)
def test_after_broadcast_optimizer_state(hvd, dtype):
    """broadcast_optimizer_state initialises the state with torch's own zero-gradient step (moments in the parameter
    dtype, step 1); the fused steps that follow use fp32 moments with the parameter's layout and count on from 1."""
    model = _net(dtype)
    opt = _dist(hvd, _adamw(model), model)
    hvd.broadcast_optimizer_state(opt, root_rank=0)
    assert all(int(opt.state[p]['step']) == 1 for p in model.parameters())
    for step in range(5):
        opt.zero_grad()
        _loss(model, step, dtype).backward()
        _fused_adam_step_checked(opt, model, dtype, step + 2)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
def test_step_closure_then_fused_steps(hvd, dtype):
    """step(closure) runs torch's own update (state in the parameter dtype); the fused steps after it normalise the
    state and match the reference. (Not fp16: torch's own fp16 Adam step flushes eps=1e-8 to zero and divides by
    zero wherever v underflows.)"""
    model = _net(dtype)
    opt = _dist(hvd, _adamw(model), model)
    opt.zero_grad()
    loss = _loss(model, 0, dtype)
    loss.backward()
    assert opt.step(lambda: loss) is loss
    for step in range(1, 4):
        opt.zero_grad()
        _loss(model, step, dtype).backward()
        _fused_adam_step_checked(opt, model, dtype, step + 1)


@pytest.mark.gpu
def test_fp16_model_with_adam(hvd):
    """fp16 parameters with Adam (L2 weight decay) and fused=True: fp32 moments, every step matches the reference."""
    model = _net(torch.float16)
    opt = _dist(hvd, torch.optim.Adam(model.parameters(), lr=1e-2, weight_decay=1e-3), model)
    for step in range(4):
        opt.zero_grad()
        _loss(model, step, torch.float16).backward()
        if step == 0:
            before = hvd.runtime_stats()['kernel_launches']
            opt.step()  # creates the state
            assert hvd.runtime_stats()['kernel_launches'] > before
            continue
        _fused_adam_step_checked(opt, model, torch.float16, step + 1, adamw=False, weight_decay=1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize("kind", ["adamw", "sgd"])
def test_checkpoint_round_trip_is_bit_exact(hvd, monkeypatch, dtype, kind):
    """3 steps, state_dict() through torch.save / torch.load into a fresh model and optimizer, 3 more steps: bit-identical
    to 6 uninterrupted steps (bf16 AdamW keeps its fp32 moments through load_state_dict)."""
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    make = _adamw if kind == 'adamw' else _sgd

    def train(model, opt, steps):
        for step in steps:
            opt.zero_grad()
            _loss(model, step, dtype).backward()
            opt.step()

    ma = _net(dtype)
    oa = _dist(hvd, make(ma), ma)
    train(ma, oa, range(6))

    mb = _net(dtype)
    ob = _dist(hvd, make(mb), mb)
    train(mb, ob, range(3))
    f = io.BytesIO()
    torch.save({'model': mb.state_dict(), 'opt': ob.state_dict()}, f)
    f.seek(0)
    ck = torch.load(f)
    mc = _net(dtype)
    mc.load_state_dict(ck['model'])
    oc = _dist(hvd, make(mc), mc)
    oc.load_state_dict(ck['opt'])
    if kind == 'adamw':
        for p in mc.parameters():
            assert oc.state[p]['exp_avg'].dtype == torch.float32 and oc.state[p]['exp_avg_sq'].dtype == torch.float32
    train(mc, oc, range(3, 6))
    for (name, a), c in zip(ma.named_parameters(), mc.parameters()):
        assert torch.equal(a, c), name
        for key, t in oa.state[a].items():
            if torch.is_tensor(t) and t.dim() > 0:
                assert torch.equal(t, oc.state[c][key]), (name, key)


@pytest.mark.gpu
def test_parameter_trained_from_step_3_has_its_own_step_count(hvd):
    """A parameter that gets its first gradient at step 3 (frozen until then, so zero_grad(set_to_none=True) leaves it
    without one) starts with step 1's bias corrections while the others are at step 4; torch.optim.AdamW keeps one
    count per parameter too."""
    model, ref = _net(torch.float32), _net(torch.float32)
    for m in (model, ref):
        m.late.requires_grad_(False)
    opt = _dist(hvd, _adamw(model), model)
    ropt = _adamw(ref)
    for step in range(6):
        if step == 3:
            for m in (model, ref):
                m.late.requires_grad_(True)
        for m, o in ((model, opt), (ref, ropt)):
            o.zero_grad(set_to_none=True)
            _loss(m, step, torch.float32).backward()
            o.step()
        if step == 2:
            assert model.late.weight.grad is None and model.late.weight not in opt.state
    assert int(opt.state[model.late.weight]['step']) == 3 and int(opt.state[model.fc.weight]['step']) == 6
    for (name, a), b in zip(model.named_parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6, msg=lambda m: f'{name}: {m}')


@pytest.mark.gpu
def test_mixed_step_counts_after_load(hvd):
    """A checkpoint whose parameters have different step counts: each parameter keeps its own bias corrections."""
    model = _net(torch.float32)
    opt = _dist(hvd, _adamw(model), model)
    opt.zero_grad()
    _loss(model, 0, torch.float32).backward()
    opt.step()
    sd = opt.state_dict()
    for i, st in enumerate(sd['state'].values()):
        st['step'] = torch.tensor(float(1 + 5 * (i % 3)))
    opt.load_state_dict(sd)
    counts = {p: int(opt.state[p]['step']) for p in model.parameters()}
    assert len(set(counts.values())) == 3
    opt.zero_grad()
    _loss(model, 1, torch.float32).backward()
    before = {p: (p.detach().double().clone(), opt.state[p]['exp_avg'].double().clone(),
                  opt.state[p]['exp_avg_sq'].double().clone()) for p in model.parameters()}
    opt.step()
    torch.cuda.synchronize()
    for name, p in model.named_parameters():
        p0, m0, v0 = before[p]
        pr, _, _, ps, _, _ = adam_ref_kernel(p0, p.grad.double(), m0, v0, lr=1e-2, weight_decay=0.05, step=counts[p] + 1)
        check(name, p, pr, ps, torch.float32)
