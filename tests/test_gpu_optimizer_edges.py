"""The fused SGD / Adam / LAMB / LARS / Adafactor kernels on the inputs their other tests never feed them: all-zero
tensors and the degenerate trust-ratio and clamp branches, one inf / -inf / NaN in a gradient or in the device gradient
scale, non-finite parameters, state and EMA, the extremes of the storage dtype (fp16 overflow, subnormals, fp32 moments
that overflow), fp32 masters around non-finite values, and Adafactor past 2^31 elements.

Every case runs the public `ops.*` entry points and checks against the float64 references of `optim_cases`:
* non-finite positions exactly: isnan and isinf (with sign) of the parameter, every state tensor, the master and the EMA
  equal those of the reference rounded to the stored dtype, element for element;
* finite elements within the tolerances of each optimizer's own test module;
* containment: the clean entries of a launch that also holds the poisoned one are bit-identical to the same launch
  without it (and, for the element-wise SGD / Adam, every other element of the poisoned tensor too).  LAMB and LARS also
  split the poisoned tensor over two calls whose pieces share a norm slot, the sharded layout.  Adafactor does not:
  fused_adafactor_step takes whole parameters and has no norm slots, so there is no split layout to test.
"""
import math

import numpy as np
import pytest
import torch

import test_gpu_adafactor as ada_t
import test_gpu_lamb as lamb_t
import test_gpu_lars as lars_t
from optim_cases import (LOW, LOW_IDS, PAIR_IDS, PAIRS, Slot, adafactor_ref, adam_ref, adam_ref_kernel, bits, f32, hvd,  # noqa: F401
                         lamb_ref, lars_ref, same, ulp)
from test_gpu_fused_optimizer import ADAM_HP, SGD_HP, _make, sgd_ref, sgd_ref_kernel

INF, NAN = float('inf'), float('nan')
U = 2.0 ** -24
LAMB_HP = dict(lamb_t.HP[0], step=2)
LARS_HP = lars_t.HP[0]  # eps = 0: the guard alone keeps r finite
ADA_HP = dict(ada_t.HP[2], step=2)
ADAM_STEP = 3
KINDS = ['sgd', 'adam', 'lamb', 'lars', 'adafactor']


def _positions(n):
    """Element 0, the interior of a 4-element vector and the scalar tail (for n = 4097: element 4096)."""
    return sorted({0, min(n - 1, 2050), n - 1})


# ---- checks ------------------------------------------------------------------------------------------------------------
def _masks(t):
    return torch.isnan(t), torch.isposinf(t), torch.isneginf(t)


def verify(name, got, want, allowed, stored=None):
    """got (the kernel's tensor) against want (float64): the NaN / +inf / -inf masks equal those of want rounded to
    `stored` (default got's dtype) element for element, and |got - want| <= allowed where both are finite."""
    got64 = got.double().flatten()
    want, allowed = want.flatten(), allowed.flatten()
    ref = want.to(stored or got.dtype).double()
    for what, a, b in zip(('NaN', '+inf', '-inf'), _masks(got64), _masks(ref)):
        if not torch.equal(a, b):
            i = int((a != b).nonzero()[0])
            raise AssertionError(f'{name}: {what} mask differs at {int((a != b).sum())} elements, first at {i}: got '
                                 f'{got64[i].item()!r}, want {want[i].item()!r}')
    fin = torch.isfinite(ref)
    err = (got64[fin] - want[fin]).abs()
    bad = ~(err <= allowed[fin])
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError(f'{name}: {int(bad.sum())} finite elements off, first: got {got64[fin][i].item()!r} want '
                             f'{want[fin][i].item()!r} (err {err[i].item():.3e} > {allowed[fin][i].item():.3e})')


def _elem_tol(want, scale, dtype, rtol=1e-6):
    """test_gpu_fused_optimizer.check's bound: rtol * scale, plus one ulp of the reference rounded to a 16-bit dtype (the
    reference it compares against is then that rounded value)."""
    if dtype == torch.float32:
        return want, rtol * scale
    w = want.to(dtype).double()
    return torch.where(torch.isfinite(w), w, want), ulp(w, dtype) + rtol * scale


class _Snap:
    def __init__(self, t):
        self.t = t.clone()


def _snapshot(cases):
    return [{k: _Snap(s.t) for k, s in c.items()} for c in cases]


def _intact(name, cases):
    for i, c in enumerate(cases):
        for k, s in c.items():
            assert s.intact(), f'{name}[{i}]: wrote outside {k}'


# ---- the five optimizers behind one interface ---------------------------------------------------------------------------
def _make_case(kind, shape, pdt, gdt, seed):
    if kind in ('sgd', 'adam'):
        return _make(shape, pdt, gdt, seed, sgd=kind == 'sgd')
    if kind == 'lamb':
        return lamb_t._case(shape, pdt, gdt, seed)
    if kind == 'lars':
        return lars_t._case(shape, pdt, gdt, seed)
    return ada_t._case(shape, pdt, gdt, seed, warm=True)


def _shapes(kind):
    return [(4097,), (3,)] + ([(33, 31)] if kind == 'adafactor' else [])


def _run(kind, cases, gsd=None, hp=None, ema=None, slots=None, **kw):
    """One step of `kind` over `cases` through its public entry point.  `slots`: LAMB / LARS as their two phases, with
    `cases` a list of calls (lists of cases) that all add into one norms buffer with these slots per call, the layout of
    the ranks' shards.  `ema`: (list of fp32 EMA tensors, decay, start)."""
    from horovod_b200 import ops
    get = lambda k: [c[k].t for c in cases]  # noqa: E731
    if ema is not None:
        kw.update(ema_params=ema[0], ema_decay=ema[1], ema_start=ema[2])
    if slots is None and 'w' in cases[0]:
        kw['master_params'] = get('w')
    if kind == 'sgd':
        ops.fused_sgd_step(get('p'), get('g'), get('buf'), **dict(hp or SGD_HP), grad_scale_dev=gsd, **kw)
    elif kind == 'adam':
        ops.fused_adam_step(get('p'), get('g'), get('m'), get('v'), step=ADAM_STEP, **dict(hp or ADAM_HP),
                            grad_scale_dev=gsd, **kw)
    elif kind == 'lamb':
        hp = dict(hp or LAMB_HP)
        if slots is None:
            ops.fused_lamb_step(get('p'), get('g'), get('m'), get('v'), grad_scale_dev=gsd, **hp, **kw)
        else:
            calls = [[[c[k].t for c in call] for k in ('p', 'g', 'm', 'v')] for call in cases]
            moments = hp['beta1'], hp['beta2'], hp['eps'], hp['weight_decay'], hp['step']
            norms = torch.zeros(2 * (max(max(s) for s in slots) + 1), device='cuda')
            for lists, sl in zip(calls, slots):
                ops.lamb_norms(*lists, *moments, norms, slots=sl, grad_scale_dev=gsd)
            for lists, sl in zip(calls, slots):
                ops.lamb_apply(*lists, hp['lr'], *moments, norms, slots=sl, **kw)
    elif kind == 'lars':
        hp = dict(hp or LARS_HP)
        if slots is None:
            ops.fused_lars_step(get('p'), get('g'), get('v'), grad_scale_dev=gsd, **hp, **kw)
        else:
            calls = [[[c[k].t for c in call] for k in ('p', 'g', 'v')] for call in cases]
            norms = torch.zeros(2 * (max(max(s) for s in slots) + 1), device='cuda')
            for lists, sl in zip(calls, slots):
                ops.lars_norms(*lists, norms, slots=sl, grad_scale_dev=gsd)
            for lists, sl in zip(calls, slots):
                ops.lars_apply(*lists, hp['lr'], hp['momentum'], hp['weight_decay'], hp['trust_coefficient'], hp['eps'],
                               norms, slots=sl, grad_scale_dev=gsd, **kw)
    else:
        hp = dict(hp or ADA_HP)
        ops.fused_adafactor_step(*ada_t._lists(cases), grad_scale_dev=gsd, **hp, **kw)
    torch.cuda.synchronize()


def _expect(kind, before, gscale=1.0, hp=None, **ref_kw):
    """Per case: {state key: (want, allowed)} in float64 from the references, with the bounds of the optimizer's own
    tests.  `gscale` is the device gradient scale the kernel multiplies in; `ref_kw` goes to the LAMB / LARS / Adafactor
    reference (its fp32 rounding options)."""
    out = []
    if kind == 'sgd':
        hp = dict(hp or SGD_HP)
        hp['grad_scale'] = hp.get('grad_scale', 1.0) * gscale
        for c in before:
            pdt = c['p'].t.dtype
            p, buf, ps, bs = sgd_ref_kernel(c['p'].t.double(), c['g'].t.double(), c['buf'].t.double(), **hp)
            out.append({'p': _elem_tol(p, ps, pdt), 'buf': _elem_tol(buf, bs, c['buf'].t.dtype)})
    elif kind == 'adam':
        hp = dict(hp or ADAM_HP)
        hp['grad_scale'] = hp.get('grad_scale', 1.0) * gscale
        for c in before:
            p, m, v, ps, ms, vs = adam_ref_kernel(c['p'].t.double(), c['g'].t.double(), c['m'].t.double(),
                                                  c['v'].t.double(), step=ADAM_STEP, **hp)
            out.append({'p': _elem_tol(p, ps, c['p'].t.dtype), 'm': _elem_tol(m, ms, torch.float32),
                        'v': _elem_tol(v, vs, torch.float32)})
    elif kind == 'lamb':
        hp = dict(hp or LAMB_HP)
        for c, e in zip(before, lamb_ref(before, grad_scale=hp.pop('grad_scale', 1.0) * gscale, **hp, **ref_kw)):
            pdt = c['p'].t.dtype
            tol = e['scale_u'] * (lamb_t.NORM_RTOL + 32 * U) + ulp(e['w'], torch.float32)
            if pdt != torch.float32:
                tol = tol + ulp(e['w'], pdt)
            out.append({'p': (e['w'], tol), 'm': (e['m'], 4 * U * e['scale_m']), 'v': (e['v'], 4 * U * e['v'].abs())})
    elif kind == 'lars':
        hp = dict(hp or LARS_HP)
        for c, e in zip(before, lars_ref(before, grad_scale=hp.pop('grad_scale', 1.0) * gscale, **hp, **ref_kw)):
            pdt = c['p'].t.dtype
            tol_v = e['scale_v'] * (lars_t.NORM_RTOL + lars_t.ELEM_RTOL)
            tol = tol_v + ulp(e['w'], torch.float32)
            if pdt != torch.float32:
                tol = tol + ulp(e['w'], pdt)
            out.append({'p': (e['w'], tol), 'v': (e['v'], tol_v)})
    else:
        hp = dict(hp or ADA_HP)
        gs = hp.pop('grad_scale', 1.0) * gscale
        for c in before:
            pdt, shape = c['p'].t.dtype, tuple(c['p'].t.shape)
            e = adafactor_ref(c, grad_scale=gs, **hp, **ref_kw)
            tol = e['scale'] * ada_t._tol_rel(shape) + e['p'].abs() * 2 * U + ulp(e['p'], torch.float32)
            if pdt != torch.float32:
                tol = tol + ulp(e['p'], pdt)
            d = {'p': (e['p'], tol)}
            for k in ('r', 'c', 'v'):
                if k in e:
                    rtol = ((shape[-1] / 32 + 80) if k == 'r' else 80) * U
                    d[k] = (e[k], rtol * e[k].abs() + 1e-38)
            out.append(d)
    return out


def _verify_all(name, kind, cases, before, gscale=1.0, hp=None, **ref_kw):
    for i, (c, e) in enumerate(zip(cases, _expect(kind, before, gscale, hp, **ref_kw))):
        for k, (want, allowed) in e.items():
            verify(f'{name}[{i}].{k}', c[k].t, want, allowed)
        assert same(c['g'].t, before[i]['g'].t), f'{name}[{i}]: gradient written'
    _intact(name, cases)


def _state_keys(c):
    return [k for k in c if k != 'g']


def _assert_same_state(name, a, b, skip=None):
    """Every state tensor of cases a and b bit for bit; `skip`: (flat index) allowed to differ in a[0]... b[0]."""
    for i, (ca, cb) in enumerate(zip(a, b)):
        for k in _state_keys(ca):
            x, y = bits(ca[k].t).flatten(), bits(cb[k].t).flatten()
            if skip is not None and i == 0:
                keep = torch.ones_like(x, dtype=torch.bool)
                keep[skip] = False
                x, y = x[keep], y[keep]
            assert torch.equal(x, y), f'{name}[{i}].{k}: changed bits'


def _fresh(kind, pdt, gdt, shape, clean=3):
    """The poisoned candidate (entry 0) and `clean` clean entries of other shapes."""
    others = [(4096,), (5,), (7, 9) if kind == 'adafactor' else (1,)][:clean]
    return [_make_case(kind, shape, pdt, gdt, seed=1)] + [_make_case(kind, s, pdt, gdt, seed=10 + j)
                                                           for j, s in enumerate(others)]


def _poison_and_check(kind, pair, shape, poison, name):
    """Runs [poisoned entry + clean entries], checks it against the references, and checks containment against the
    clean entries alone (and for SGD / Adam against the unpoisoned entry); `poison(cases)` edits entry 0 in place and
    returns the flat index it poisoned (or None for the whole tensor)."""
    pdt, gdt = pair
    cases = _fresh(kind, pdt, gdt, shape)
    at = poison(cases)
    before = _snapshot(cases)
    _run(kind, cases)
    _verify_all(name, kind, cases, before)
    clean = _fresh(kind, pdt, gdt, shape)[1:]
    _run(kind, clean)
    _assert_same_state(name + ' (clean entries)', cases[1:], clean)
    if kind in ('sgd', 'adam') and at is not None:
        unpoisoned = _fresh(kind, pdt, gdt, shape, clean=0)
        _run(kind, unpoisoned)
        _assert_same_state(name + ' (other elements)', cases[:1], unpoisoned, skip=at)
    if kind in ('lamb', 'lars') and len(shape) == 1 and shape[0] > 1:
        # the sharded layout: entry 0 split over two calls (two ranks' shards) whose pieces share slot 0, the first next
        # to the clean entries
        split = _fresh(kind, pdt, gdt, shape)
        poison(split)
        whole = split[0]
        h = shape[0] // 2 + 1
        halves = [{k: _View(s.t[:h]) for k, s in whole.items()}, {k: _View(s.t[h:]) for k, s in whole.items()}]
        _run(kind, [[halves[0]] + split[1:], [halves[1]]], slots=[[0, 1, 2, 3], [0]])
        for k, (want, allowed) in _expect(kind, before[:1])[0].items():
            verify(f'{name} split.{k}', whole[k].t, want, allowed)
        _assert_same_state(name + ' split (clean entries)', split[1:], clean)


class _View:
    """A view with the Slot interface (its guard is the parent Slot's)."""

    def __init__(self, t):
        self.t = t

    def intact(self):
        return True


# ---- 1. zero tensors and degenerate norms -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
def test_zero_tensors_and_degenerate_norms(hvd, pair):
    """LAMB with w = 0, with u = 0 (g = m = v = 0, wd = 0) and both: r = 1.  LARS with w = 0, g = 0 and both at eps = 0:
    r = 1 and no NaN.  Adafactor with an all-zero gradient from zero state (mean row_var = 0: the eps1 clamp), a zero
    row and a zero column, R = 1 and C = 1, and w = 0 (alpha = eps2 * rho).  Adam with g = 0 at step 1, and with eps = 0
    as well (0 / 0: NaN, as torch).  SGD with lr = 0 (parameter bits unchanged) and momentum with a zero gradient."""
    pdt, gdt = pair
    for shape in [(4097,), (3,)]:
        # LAMB
        for zero, hp in (('w', LAMB_HP), ('u', dict(LAMB_HP, weight_decay=0.0)), ('wu', dict(LAMB_HP, weight_decay=0.0))):
            cases = [lamb_t._case(shape, pdt, gdt, seed=3), lamb_t._case((4096,), pdt, gdt, seed=4)]
            if 'w' in zero:
                cases[0]['p'].t.zero_()
            if 'u' in zero:
                for k in ('g', 'm', 'v'):
                    cases[0][k].t.zero_()
            before = _snapshot(cases)
            _run('lamb', cases, hp=hp)
            _verify_all(f'lamb zero {zero} {shape}', 'lamb', cases, before, hp=hp)
            if zero == 'u':
                assert same(cases[0]['p'].t, before[0]['p'].t), 'lamb: u = 0 moved the parameter'
        # LARS
        for zero in ('w', 'g', 'wg'):
            cases = [lars_t._case(shape, pdt, gdt, seed=5), lars_t._case((4096,), pdt, gdt, seed=6)]
            if 'w' in zero:
                cases[0]['p'].t.zero_()
            if 'g' in zero:
                cases[0]['g'].t.zero_()
            before = _snapshot(cases)
            _run('lars', cases)
            _verify_all(f'lars zero {zero} {shape}', 'lars', cases, before)
            assert all(bool(torch.isfinite(c[k].t).all()) for c in cases for k in ('p', 'v')), f'lars zero {zero}: NaN'
        # Adam
        for eps in (1e-8, 0.0):
            hp = dict(ADAM_HP, eps=eps)
            cases = [_make(shape, pdt, gdt, seed=7), _make((4096,), pdt, gdt, seed=8)]
            for k in ('g', 'm', 'v'):
                cases[0][k].t.zero_()
            before = _snapshot(cases)
            from horovod_b200 import ops
            ops.fused_adam_step([c['p'].t for c in cases], [c['g'].t for c in cases], [c['m'].t for c in cases],
                                [c['v'].t for c in cases], step=1, **hp)
            torch.cuda.synchronize()
            for i, (c, b) in enumerate(zip(cases, before)):
                p, m, v, ps, ms, vs = adam_ref_kernel(b['p'].t.double(), b['g'].t.double(), b['m'].t.double(),
                                                      b['v'].t.double(), step=1, **hp)
                verify(f'adam zero eps={eps} [{i}].p', c['p'].t, *_elem_tol(p, ps, pdt))
                verify(f'adam zero eps={eps} [{i}].m', c['m'].t, *_elem_tol(m, ms, torch.float32))
                verify(f'adam zero eps={eps} [{i}].v', c['v'].t, *_elem_tol(v, vs, torch.float32))
            assert bool(torch.isnan(cases[0]['p'].t).all()) == (eps == 0.0)
        # SGD
        for hp in (dict(SGD_HP, lr=0.0), SGD_HP):
            cases = [_make(shape, pdt, gdt, seed=9, sgd=True), _make((4096,), pdt, gdt, seed=10, sgd=True)]
            cases[0]['g'].t.zero_()
            before = _snapshot(cases)
            _run('sgd', cases, hp=hp)
            _verify_all(f'sgd zero lr={hp["lr"]} {shape}', 'sgd', cases, before, hp=hp)
            if hp['lr'] == 0.0:
                assert all(same(c['p'].t, b['p'].t) for c, b in zip(cases, before)), 'sgd: lr = 0 changed parameter bits'
    # Adafactor
    for what, shape in (('zero grad', (33, 31)), ('zero row+col', (33, 31)), ('R=1', (1, 37)), ('C=1', (37, 1)),
                        ('w=0', (33, 31)), ('w=0', (4097,))):
        cases = [ada_t._case(shape, pdt, gdt, seed=11), ada_t._case((7, 9), pdt, gdt, seed=12)]
        g = cases[0]['g'].t
        if what == 'zero grad':
            g.zero_()
        elif what == 'zero row+col':
            g[5].zero_()
            g[:, 17].zero_()
        elif what == 'w=0':
            cases[0]['p'].t.zero_()
        before = _snapshot(cases)
        _run('adafactor', cases, hp=dict(ADA_HP, step=1))  # from zero state: row_var of a zero gradient is 0
        _verify_all(f'adafactor {what} {shape}', 'adafactor', cases, before, hp=dict(ADA_HP, step=1))


# ---- 2. one inf, -inf or NaN in a gradient, or in the device gradient scale ---------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("kind", KINDS)
def test_nonfinite_gradient(hvd, kind, pair):
    """One inf, -inf or NaN at element 0, inside a vector and in the scalar tail, next to clean entries; then the whole
    launch with grad_scale_dev = inf, NaN and 0.  SGD / Adam: only that element goes non-finite.  LAMB: u = NaN there,
    so ||u|| is NaN, r = 1 and only that element is NaN; LARS: ||g|| = inf gives r = 0 (NaN gives r = 1);  Adafactor:
    the element's row and column factors, and with them v, follow torch's clamps."""
    pdt, gdt = pair
    for shape in _shapes(kind):
        n = int(np.prod(shape))
        for at in _positions(n):
            for val in (INF, -INF, NAN):
                def poison(cases, at=at, val=val):
                    cases[0]['g'].t.view(-1)[at] = val
                    return at
                _poison_and_check(kind, pair, shape, poison, f'{kind} {shape} g[{at}]={val}')
    for gsv in (INF, NAN, 0.0):
        cases = _fresh(kind, pdt, gdt, (4097,))
        before = _snapshot(cases)
        _run(kind, cases, gsd=torch.tensor([gsv], device='cuda'))
        _verify_all(f'{kind} grad_scale_dev={gsv}', kind, cases, before, gscale=gsv)


# ---- 3. non-finite parameters, state and EMA ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("kind", KINDS)
def test_nonfinite_param_and_state(hvd, kind, pair):
    """A NaN, inf or -inf already stored in the parameter or in one state tensor (momentum, exp_avg / exp_avg_sq, an
    Adafactor factor or variance), at each position; then a NaN / inf in the EMA with ema_decay on (kept) and with
    ema_start (cleared)."""
    pdt, gdt = pair
    for shape in _shapes(kind):
        n = int(np.prod(shape))
        proto = _make_case(kind, shape, pdt, gdt, seed=1)
        for key in _state_keys(proto):
            m = proto[key].t.numel()
            for at in sorted({0, m // 2, m - 1}):
                for val in (INF, -INF, NAN):
                    def poison(cases, key=key, at=at, val=val):
                        cases[0][key].t.view(-1)[at] = val
                        return at if key not in ('r', 'c') else None
                    _poison_and_check(kind, pair, shape, poison, f'{kind} {shape} {key}[{at}]={val}')
    # the EMA: e = fmaf(1 - decay, x - e, e) with x the stored parameter; with start, e = x
    decay = 0.9
    for start in (False, True):
        cases = _fresh(kind, pdt, gdt, (4097,))
        emas = [torch.randn(c['p'].t.shape, device='cuda') for c in cases]
        for e in emas:
            e.view(-1)[0], e.view(-1)[-1] = NAN, -INF
        e0 = [e.clone() for e in emas]
        _run(kind, cases, ema=(emas, decay, start))
        w = f32(1 - decay)
        for i, (c, e, old) in enumerate(zip(cases, emas, e0)):
            x = c['p'].t.double()
            if start:
                assert same(e, c['p'].t.float()), f'{kind} ema start [{i}]: e is not the stored parameter'
                continue
            want = old.double() + w * (x - old.double())
            allowed = 4 * U * (old.double().abs() + w * (x - old.double()).abs()) + ulp(want, torch.float32)
            verify(f'{kind} ema [{i}]', e, want, allowed)


# ---- 4. extremes of the storage dtype -----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_fp16_parameters_crossing_65504(hvd):
    """fp16 parameters whose SGD or Adam update crosses 65504: inf exactly where the reference rounds to inf."""
    from horovod_b200 import ops
    n = 4097
    sign = torch.tensor([1.0, -1.0], device='cuda').repeat(n // 2 + 1)[:n]
    # SGD, lr = 1: p - g with p = +-64992 and |g| from 0 to 2000
    p0 = (64992 * sign).to(torch.float16)
    g0 = (-sign * torch.linspace(0, 2000, n, device='cuda')).to(torch.float16)
    p, g, buf = p0.clone(), g0.clone(), torch.zeros_like(p0)
    hp = dict(lr=1.0, momentum=0.0, dampening=0.0, weight_decay=0.0, grad_scale=1.0)
    ops.fused_sgd_step([p], [g], [], **hp)
    want, _, ps, _ = sgd_ref_kernel(p0.double(), g0.double(), None, **hp)
    verify('sgd fp16 65504', p, *_elem_tol(want, ps, torch.float16))
    assert bool(torch.isinf(p).any()) and bool(torch.isfinite(p).any())
    # Adam at step 1 moves every element by about lr: from +-65472 by 64 either way
    p0 = (65472 * sign).to(torch.float16)
    g0 = torch.randn(n, device='cuda', generator=torch.Generator(device='cuda').manual_seed(3)).to(torch.float16)
    p, m, v = p0.clone(), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
    hp = dict(lr=64.0, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0)
    ops.fused_adam_step([p], [g0], [m], [v], step=1, **hp)
    want, _, _, ps, _, _ = adam_ref_kernel(p0.double(), g0.double(), torch.zeros(n, dtype=torch.float64, device='cuda'),
                                           torch.zeros(n, dtype=torch.float64, device='cuda'), step=1, **hp)
    verify('adam fp16 65504', p, *_elem_tol(want, ps, torch.float16))
    assert bool(torch.isinf(p).any()) and bool(torch.isfinite(p).any())


_MIN_SUB = {torch.float32: 2.0 ** -149, torch.bfloat16: 2.0 ** -133, torch.float16: 2.0 ** -24}


@pytest.mark.gpu
@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
def test_subnormals_are_kept(hvd, pair):
    """Subnormal parameters and gradients (the build has no flush to zero): SGD with lr = 1/4 on multiples of the
    smallest subnormal, where every result is exact, so the kernel must match the reference bit for bit; Adam with
    lr = 0 leaves subnormal parameters unchanged."""
    from horovod_b200 import ops
    pdt, gdt = pair
    n = 4097
    gen = torch.Generator(device='cuda').manual_seed(4)
    # |k| < 100 smallest subnormals of the parameter dtype, and gradients of 4 j of them: p - g / 4 is exact
    kp = torch.randint(-100, 100, (n,), device='cuda', generator=gen).double()
    kg = torch.randint(-25, 25, (n,), device='cuda', generator=gen).double()
    p0 = (kp * _MIN_SUB[pdt]).to(pdt)
    g0 = (4 * kg * _MIN_SUB[gdt]).to(gdt)
    assert bool((p0.double() == kp * _MIN_SUB[pdt]).all()) and bool((g0.double() == 4 * kg * _MIN_SUB[gdt]).all())
    p = p0.clone()
    hp = dict(lr=0.25, momentum=0.0, dampening=0.0, weight_decay=0.0, grad_scale=1.0)
    ops.fused_sgd_step([p], [g0], [], **hp)
    torch.cuda.synchronize()
    want = (p0.double() - 0.25 * g0.double()).to(pdt)
    assert bool((want.double() == p0.double() - 0.25 * g0.double()).all()), 'the reference is not exact'
    assert same(p, want), f'sgd subnormals: {int((bits(p) != bits(want)).sum())} elements differ'
    p = p0.clone()
    m, v = torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
    ops.fused_adam_step([p], [g0], [m], [v], lr=0.0, step=1, weight_decay=0.0)
    torch.cuda.synchronize()
    assert same(p, p0), 'adam lr = 0: subnormal parameters changed'
    mw = (1 - f32(0.9)) * g0.double()
    verify('adam subnormal m', m, mw, ulp(mw, torch.float32))
    assert bool((m != 0).sum() >= (g0 != 0).sum() // 2), 'exp_avg of subnormal gradients flushed to zero'


@pytest.mark.gpu
def test_fp32_moments_overflow(hvd):
    """fp32 Adam with gradients of 1e19..1e20 and exp_avg_sq near the fp32 maximum: (1 - b2) d d and the v update
    overflow to inf in fp32, where a float64 reference would not.  So this reference rounds to fp32 wherever the kernel
    stores fp32 state and follows the kernel's operation order, v = fmaf(b2, v, ((1 - b2) d) d), m = fmaf(b1, m,
    (1 - b1) d): an inf v gives a zero step, never a NaN."""
    from horovod_b200 import ops
    n = 4097
    gen = torch.Generator(device='cuda').manual_seed(5)
    sgn = torch.randint(0, 2, (n,), device='cuda', generator=gen).double() * 2 - 1
    d = (sgn * 10 ** (19 + torch.rand(n, device='cuda', generator=gen, dtype=torch.float64))).float()
    v0 = torch.where(torch.arange(n, device='cuda') % 3 == 0, torch.full((n,), 3.4e38, device='cuda'),
                     torch.rand(n, device='cuda', generator=gen))
    m0 = torch.randn(n, device='cuda', generator=gen) * 1e18
    p0 = torch.randn(n, device='cuda', generator=gen)
    hp = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0)
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    ops.fused_adam_step([p], [d], [m], [v], step=ADAM_STEP, **hp)
    torch.cuda.synchronize()
    f = lambda x: x.float().double()  # noqa: E731  (round to fp32)
    b1, b2 = f32(0.9), f32(0.999)
    dd = d.double()
    m_want = f(b1 * m0.double() + f(f32(1 - b1) * dd))
    v_want = f(b2 * v0.double() + f(f(f32(1 - b2) * dd) * dd))
    verify('adam v overflow', v, v_want, 2 * U * v_want.abs())
    verify('adam m', m, m_want, 2 * U * (b1 * m0.double().abs() + (f32(1 - b1) * dd).abs()))
    assert bool(torch.isinf(v).any()) and bool(torch.isfinite(v).any())
    c1, c2 = f32(1 - f32(0.9 ** ADAM_STEP)), f32(1 - f32(0.999 ** ADAM_STEP))
    denom = v_want.sqrt() / c2 ** 0.5 + f32(1e-8)
    step = f32(1e-2) / c1 * m_want / denom
    want = p0.double() - step
    verify('adam p', p, want, 1e-6 * (p0.double().abs() + step.abs()))
    assert bool(torch.isfinite(p).all())


_OVERFLOW_REF = {'lamb': dict(fp32_moments=True), 'lars': dict(fp32_norms=True), 'adafactor': dict(fp32_squares=True)}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ['lamb', 'lars', 'adafactor'])
def test_fp32_norm_and_factor_overflow(hvd, kind):
    """fp32 LAMB / LARS / Adafactor with gradients of 2e19..1e20, whose squares pass the fp32 maximum: one tensor of such
    gradients, one with a single such element, next to a clean tensor.  LARS: sum g^2 overflows, ||g|| = inf, r = 0 and
    the step keeps only the momentum.  Adafactor: g^2 is inf, so the variance or the row / column factors (and with them
    the mean of row_var) are inf or NaN where torch's lerp and clamps make them so.  LAMB squares (1 - b2) g, which stays
    finite, so its exp_avg_sq starts near the fp32 maximum instead and overflows in the v update, and v / c2 overflows
    for v above c2 times the fp32 maximum: there u = m / inf = 0 plus the decay term.  The references round to fp32 where the kernel does and follow its operation order there."""
    pdt = torch.float32
    shapes = [(4097,), (4097,), (4096,)] + ([(33, 31), (33, 31)] if kind == 'adafactor' else [])
    clean_at = 2

    def make():
        cases = [_make_case(kind, s, pdt, pdt, seed=20 + j) for j, s in enumerate(shapes)]
        gen = torch.Generator(device='cuda').manual_seed(21)
        for j, c in enumerate(cases):
            if j == clean_at:
                continue
            g = c['g'].t.view(-1)
            n = g.numel()
            sgn = torch.randint(0, 2, (n,), device='cuda', generator=gen).float() * 2 - 1
            huge = sgn * 10 ** (19.31 + 0.69 * torch.rand(n, device='cuda', generator=gen))
            if j in (1, 3):  # a single huge element
                at = 2050 if n > 2050 else 5 * 31 + 17
                g[at] = huge[at]
            else:
                g.copy_(huge)
            if kind == 'lamb':
                c['v'].t.view(-1)[::3] = 3.4e38
        return cases

    cases = make()
    before = _snapshot(cases)
    _run(kind, cases)
    _verify_all(f'{kind} overflow', kind, cases, before, **_OVERFLOW_REF[kind])
    if kind != 'lars':
        nonfinite = [not bool(torch.isfinite(c[k].t).all()) for c in cases for k in _state_keys(c)]
        assert any(nonfinite), f'{kind}: no state overflowed'
    else:
        v_want = f32(LARS_HP['momentum']) * before[0]['v'].t.double()
        verify('lars overflow r = 0', cases[0]['v'].t, v_want, 4 * U * v_want.abs())
    clean = [_make_case(kind, shapes[clean_at], pdt, pdt, seed=20 + clean_at)]
    _run(kind, clean)
    _assert_same_state(f'{kind} overflow (clean entry)', [cases[clean_at]], clean)


# ---- 5. masters with non-finite and overflowing values ------------------------------------------------------------------
def _master_case(pdt, n, seed, kind):
    gen = torch.Generator(device='cuda').manual_seed(seed)
    w = torch.randn(n, device='cuda', generator=gen) * 0.1
    c = {'p': Slot((n,), pdt, 1, w.to(pdt)), 'g': Slot((n,), pdt, 2, torch.randn(n, device='cuda', generator=gen)),
         'w': Slot((n,), torch.float32, 3, w)}
    if kind == 'sgd':
        c['buf'] = Slot((n,), torch.float32, 0, torch.randn(n, device='cuda', generator=gen) * 0.5)
    else:
        c['m'] = Slot((n,), torch.float32, 0, torch.randn(n, device='cuda', generator=gen) * 0.1)
        c['v'] = Slot((n,), torch.float32, 0, (torch.randn(n, device='cuda', generator=gen) * 0.1).square())
    return c


def _master_expect(kind, before, pdt):
    """The master update is the fp32-parameter update started from the reconciled master: the master where the
    parameter's bits are those of round(master), else the parameter."""
    start = []
    for b in before:
        kept = bits(b['w'].t.to(pdt)) == bits(b['p'].t)
        start.append(torch.where(kept, b['w'].t, b['p'].t.float()))
    fp32 = [{**{k: _Snap(s.t.float() if k == 'g' else s.t) for k, s in b.items() if k not in ('p', 'w')},
             'p': _Snap(st)} for b, st in zip(before, start)]
    return _expect(kind, fp32)


@pytest.mark.gpu
@pytest.mark.parametrize("pdt", LOW, ids=LOW_IDS)
@pytest.mark.parametrize("kind", ['sgd', 'adam'])
def test_master_nonfinite_and_overflow(hvd, kind, pdt):
    """kMaster: an fp16 master above 65504 keeps its fp32 value while the parameter holds inf, and the next step continues
    from the master; a NaN written into the parameter restarts the master to NaN in exactly that element, and the NaN
    master keeps its bits over two more steps (which a restart would too: the GPU returns the canonical NaN from any NaN
    operand, so this pins the stored bits, not the reconcile rule); a zero of the other sign written into the parameter
    restarts a master that rounds to zero, the case that shows the reconcile compares bits, not values."""
    n = 4097
    cases = [_master_case(pdt, n, 1, kind), _master_case(pdt, 4096, 2, kind)]
    c = cases[0]
    p, w, g = c['p'].t, c['w'].t, c['g'].t
    big = 65530.0 if pdt == torch.float16 else 3.4e38
    w[0], p[0], g[0] = big, big, 0.0  # round(65530) in fp16 is inf: the parameter holds inf, the master 65530
    w[1], p[1], g[1] = big, big, 1e4 if kind == 'sgd' else 1.0  # SGD: back below 65504
    p[2] = NAN  # an outside write
    w[3], p[3], g[3] = 1e-45, -0.0, 0.0  # round(1e-45) is +0: the parameter's -0 is an outside write
    w[4], p[4], g[4] = -1e-45, -0.0, 0.0  # round(-1e-45) is -0: the master is kept
    w[5] = -w[5]  # an outside write to a finite value (round(w) != p)
    if kind == 'sgd':
        c['buf'].t[:8] = 0.0
    else:
        c['m'].t[:8], c['v'].t[:8] = 0.0, 0.0
    if pdt == torch.float16:
        assert bool(torch.isinf(p[:2]).all()) and float(w[0]) == 65530.0
    hp = None
    clean = [_master_case(pdt, 4096, 2, kind)]
    for step in range(3):
        before = _snapshot(cases)
        _run(kind, cases, hp=hp)
        for i, (cc, e) in enumerate(zip(cases, _master_expect(kind, before, pdt))):
            # the master and its fp32 state, within their bounds plus half the fp32 subnormal spacing: values that round
            # into the subnormal range (w[4] and its momentum) carry that absolute error
            want, allowed = e['p']
            verify(f'{kind} master step {step} [{i}].w', cc['w'].t, want, allowed + 2.0 ** -150, stored=torch.float32)
            assert same(cc['p'].t, cc['w'].t.to(pdt)), f'{kind} master step {step} [{i}]: param is not the rounded master'
            for k in e:
                if k != 'p':
                    verify(f'{kind} master step {step} [{i}].{k}', cc[k].t, e[k][0], e[k][1] + 2.0 ** -150)
        _intact(f'{kind} master step {step}', cases)
        if step == 0:
            assert math.isnan(float(w[2])), 'the NaN parameter did not restart its master'
            assert float(w[3]) == 0.0 and math.copysign(1.0, float(w[3])) < 0, 'the -0 parameter did not restart its master'
            assert float(w[4]) < 0, 'a kept master restarted'
            if pdt == torch.float16:
                assert 65504.0 < float(w[0]) < 65530.0, 'the fp16 master above 65504 did not continue from its value'
                assert math.isfinite(float(p[1])) or kind != 'sgd', 'the master crossing back below 65504 is still inf'
            nan_bits = int(bits(w)[2])
        else:
            assert int(bits(w)[2]) == nan_bits, f'step {step}: the NaN master changed bits'
        _run(kind, clean, hp=hp)
        _assert_same_state(f'{kind} master step {step} clean', cases[1:], clean)


# ---- 6. the references against torch.optim on the edge inputs, on the CPU ----------------------------------------------
def _edge_inputs(n):
    """Parameter and gradient vectors of the cases above, in float64 on the CPU: zeros, an inf / -inf / NaN gradient,
    a NaN / inf parameter."""
    torch.manual_seed(0)
    p, g = torch.randn(n, dtype=torch.float64), torch.randn(n, dtype=torch.float64)
    out = [('zero grad', p, torch.zeros(n, dtype=torch.float64)), ('zero param', torch.zeros(n, dtype=torch.float64), g),
           ('zero both', torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64))]
    for val in (INF, -INF, NAN):
        bad = g.clone()
        bad[n // 2] = val
        out.append((f'g={val}', p, bad))
        badp = p.clone()
        badp[1] = val
        out.append((f'p={val}', badp, g))
    return out


def _same_values(name, got, want):
    for what, a, b in zip(('NaN', '+inf', '-inf'), _masks(got), _masks(want)):
        assert torch.equal(a, b), f'{name}: {what} masks differ'
    fin = torch.isfinite(want)
    torch.testing.assert_close(got[fin], want[fin], rtol=1e-12, atol=1e-300, msg=lambda m: f'{name}: {m}')


def test_references_match_torch_optim_on_edge_inputs():
    """sgd_ref, adam_ref and adafactor_ref against torch.optim.SGD / Adam / AdamW / Adafactor in float64 on the CPU, on
    zero, inf, -inf and NaN gradients and parameters: the same values and the same NaN / inf masks, so the masks the
    GPU cases pin are torch's and not only the kernels'."""
    for name, p0, g0 in _edge_inputs(37):
        def torch_step(opt_cls, p_init, g, steps=1, **kw):
            p = torch.nn.Parameter(p_init.clone())
            opt = opt_cls([p], **kw)
            for _ in range(steps):
                p.grad = g.clone()
                opt.step()
            return p.detach(), opt.state[p]

        for kw in (dict(lr=0.05), dict(lr=0.0), dict(lr=0.05, momentum=0.9, dampening=0.5, weight_decay=1e-2)):
            want, st = torch_step(torch.optim.SGD, p0, g0, steps=2, foreach=False, **kw)
            p, buf = p0.clone(), None
            for i in range(2):
                p, buf, _, _ = sgd_ref(p, g0, buf, first_step=i == 0, **kw)
            _same_values(f'SGD {kw} {name}', p, want)
            if kw.get('momentum'):
                _same_values(f'SGD {kw} {name} momentum', buf, st['momentum_buffer'])
        for opt_cls, adamw in ((torch.optim.Adam, False), (torch.optim.AdamW, True)):
            for eps in (1e-8, 0.0):
                want, st = torch_step(opt_cls, p0, g0, foreach=False, lr=1e-2, eps=eps, weight_decay=1e-2)
                p, m, v, _, _, _ = adam_ref(p0.clone(), g0, torch.zeros_like(p0), torch.zeros_like(p0), 1e-2, eps=eps,
                                            weight_decay=1e-2, step=1, adamw=adamw)
                _same_values(f'{opt_cls.__name__} eps={eps} {name}', p, want)
                _same_values(f'{opt_cls.__name__} eps={eps} {name} exp_avg', m, st['exp_avg'])
                _same_values(f'{opt_cls.__name__} eps={eps} {name} exp_avg_sq', v, st['exp_avg_sq'])
        # Adafactor with hyper-parameters that fp32 holds exactly, so the reference's fp32 rounding changes nothing
        hp = dict(lr=2.0 ** -7, beta2_decay=-1.0, eps1=2.0 ** -20, eps2=2.0 ** -10, d=1.0, weight_decay=0.5)
        for shape in ((37,), (37, 1), (5, 7)):
            n = int(np.prod(shape))
            pp, gg = p0[:n].reshape(shape), g0[:n].reshape(shape)
            want, st = torch_step(torch.optim.Adafactor, pp, gg, foreach=False, lr=hp['lr'],
                                  beta2_decay=hp['beta2_decay'], eps=(hp['eps1'], hp['eps2']), d=hp['d'],
                                  weight_decay=hp['weight_decay'])
            c = {'p': _Snap(pp), 'g': _Snap(gg)}
            if len(shape) >= 2:
                c['r'], c['c'] = _Snap(torch.zeros(shape[0], 1, dtype=torch.float64)), \
                    _Snap(torch.zeros(1, shape[1], dtype=torch.float64))
            else:
                c['v'] = _Snap(torch.zeros(shape, dtype=torch.float64))
            e = adafactor_ref(c, step=1, **hp)
            _same_values(f'Adafactor {shape} {name}', e['p'], want)
            for k, tk in (('r', 'row_var'), ('c', 'col_var'), ('v', 'variance')):
                if k in e:
                    _same_values(f'Adafactor {shape} {name} {tk}', e[k], st[tk])


# ---- 7. Adafactor past 2^31 elements ------------------------------------------------------------------------------------
GiB = 1 << 30
B31 = 1 << 31
CHUNK = 1 << 26


@pytest.fixture
def room(hvd):
    """room(nbytes): skips the test unless the device has nbytes + 2 GiB free; frees the cached memory afterwards."""
    import gc

    def need(nbytes):
        free, _ = torch.cuda.mem_get_info()
        if free < nbytes + 2 * GiB:
            pytest.skip(f'needs {nbytes / GiB:.1f} GiB + 2 GiB free device memory, {free / GiB:.1f} GiB free')
    yield need
    gc.collect()
    torch.cuda.empty_cache()


def _chunks(n):
    return [(a, min(a + CHUNK, n)) for a in range(0, n, CHUNK)]


def _fill(t, seed, scale):
    for k, (a, b) in enumerate(_chunks(t.numel())):
        g = torch.Generator(device='cuda').manual_seed(1000 * seed + k)
        t[a:b].copy_(torch.randn(b - a, device='cuda', generator=g) * scale)


def _windows(n):
    """The head, both sides of element 2^31, the tail and 4096 seeded random indices."""
    parts = [torch.arange(0, 8192), torch.arange(B31 - 8192, B31 + 8192), torch.arange(n - 8192, n),
             torch.randint(0, n, (4096,), generator=torch.Generator().manual_seed(5))]
    idx = torch.cat(parts).unique()
    return idx[idx < n].cuda()


def _take(flat, idx):
    out = torch.empty(idx.numel(), dtype=flat.dtype, device=flat.device)
    for a, b in _chunks(flat.numel()):
        m = (idx >= a) & (idx < b)
        if bool(m.any()):
            out[m] = flat[a:b][idx[m] - a]
    return out


def _large_adafactor(shape, master):
    """One Adafactor step (from zero state, step 1, so alpha uses rho = lr) on a bf16 parameter of `shape`, then the
    factors in full and the parameter at the windows against float64 computed on the device in chunks."""
    from horovod_b200 import ops
    hp = dict(ADA_HP, step=1)
    n = int(np.prod(shape))
    p = torch.empty(n, dtype=torch.bfloat16, device='cuda')
    g = torch.empty(n, dtype=torch.bfloat16, device='cuda')
    _fill(p, 1, 0.1)
    _fill(g, 2, 1.0)
    idx = _windows(n)
    x_p, x_g = _take(p, idx).double(), _take(g, idx).double()
    w = None
    if master:
        w = torch.empty(n, dtype=torch.float32, device='cuda')
        for a, b in _chunks(n):
            w[a:b].copy_(p[a:b])  # the rounded master equals the parameter: nothing restarts
    f2 = len(shape) == 2
    R, C = shape if f2 else (n, 1)
    rv = torch.zeros(R, 1, device='cuda') if f2 else None
    cv = torch.zeros(1, C, device='cuda') if f2 else None
    var = None if f2 else torch.zeros(n, device='cuda')
    # float64 statistics of the inputs, in chunks of rows (2-D) or elements (1-D)
    beta_w = f32(1.0 ** hp['beta2_decay'])
    e1, e1sq = f32(hp['eps1']), f32(hp['eps1'] ** 2)
    wn2 = sum(float(p[a:b].double().square().sum()) for a, b in _chunks(n))
    g2 = g.view(R, C) if f2 else None
    if f2:
        rows_per = max(1, CHUNK // C)
        row_mean = torch.cat([g2[a:a + rows_per].double().square().mean(-1, keepdim=True) for a in range(0, R, rows_per)])
        col_sum = sum(g2[a:a + rows_per].double().square().sum(0, keepdim=True) for a in range(0, R, rows_per))
        r_want, c_want = beta_w * row_mean, beta_w * col_sum / R
        rmean = max(float(r_want.mean()), e1)
        u2 = sum(float((g2[a:a + rows_per].double().square() /
                        (r_want[a:a + rows_per] * c_want / rmean).clamp(min=e1sq)).sum()) for a in range(0, R, rows_per))
    else:
        u2 = sum(float((g[a:b].double().square() / (beta_w * g[a:b].double().square()).clamp(min=e1sq)).sum())
                 for a, b in _chunks(n))
    ops.fused_adafactor_step([p.view(shape)], [g.view(shape)], [rv], [cv], [var], master_params=[w.view(shape)] if master else None,
                             **hp)
    torch.cuda.synchronize()
    if f2:
        tol_r = (C / 32 + 80) * U
        verify('row_var', rv, r_want, tol_r * r_want.abs() + 1e-38)
        verify('col_var', cv, c_want, 80 * U * c_want.abs() + 1e-38)
        ri, ci = idx // C, idx % C
        v = r_want.view(-1)[ri] * c_want.view(-1)[ci] / rmean
    else:
        for a, b in _chunks(n):  # the variance in full, chunk by chunk
            want_v = beta_w * g[a:b].double().square()
            verify(f'variance[{a}:{b}]', var[a:b], want_v, 80 * U * want_v.abs() + 1e-38)
        v = beta_w * x_g.square()
    rho = f32(min(hp['lr'], 1.0))
    alpha = max(f32(hp['eps2']), (wn2 / n) ** 0.5) * rho
    denom = max(1.0, (u2 / n) ** 0.5 / f32(hp['d']))
    u = x_g * v.clamp(min=e1sq).rsqrt()
    want = x_p * f32(1 - hp['lr'] * hp['weight_decay']) - alpha / denom * u
    tol = (alpha / denom * u).abs() * ada_t._tol_rel(shape) + want.abs() * 2 * U + ulp(want, torch.float32)
    if master:
        verify('master', _take(w, idx), want, tol)
        assert same(_take(p, idx), _take(w, idx).to(torch.bfloat16)), 'param is not the rounded master'
    else:
        verify('param', _take(p, idx), want, tol + ulp(want, torch.bfloat16))
    assert same(_take(g, idx), x_g.to(torch.bfloat16)), 'gradient written'


@pytest.mark.gpu
@pytest.mark.parametrize("master", [False, True], ids=['plain', 'master'])
def test_large_adafactor_factored_bf16(room, master):
    """Needs 9 GiB (17 GiB with masters).  A bf16 parameter and gradient of [2^16 + 1, 2^15 + 3] (2^31 + 229379
    elements) with fp32 factors: the factors in full and the parameter (or master) at the windows, within the bounds of
    test_gpu_adafactor."""
    room((17 if master else 9) * GiB)
    _large_adafactor(((1 << 16) + 1, (1 << 15) + 3), master)


@pytest.mark.gpu
def test_large_adafactor_vector_bf16(room):
    """Needs 17 GiB.  A 1-D bf16 parameter of 2^31 + 4099 elements with its fp32 variance: the variance in full and the
    parameter at the windows, within the bounds of test_gpu_adafactor."""
    room(17 * GiB)
    _large_adafactor((B31 + 4099,), False)


@pytest.mark.gpu
def test_adafactor_rejects_2_pow_32_elements(hvd):
    """The kernels' element offsets are 32-bit: a parameter of 2^32 elements (an expanded view, no memory) raises
    RuntimeError naming the limit before anything is launched."""
    from horovod_b200 import ops
    p = torch.zeros(1, dtype=torch.bfloat16, device='cuda').expand(1 << 32)
    with pytest.raises(RuntimeError, match=r'2\^32 - 1'):
        ops.fused_adafactor_step([p], [p], [None], [None], [torch.zeros(1, device='cuda').expand(1 << 32)], lr=1e-2,
                                 beta2_decay=-0.8, eps1=None, eps2=1e-3, d=1.0, weight_decay=0.0, step=1)


@pytest.mark.gpu
@pytest.mark.parametrize("shapes, limit", [
    ([(1, B31 + 1)], r'2\^31 - 1 are supported in each dim'),
    ([(B31 + 1, 1)], r'2\^31 - 1 are supported in each dim'),
    ([(1, 1, B31)], r'2\^31 - 1 are supported in each dim'),
    ([(1, B31 - 1), (1, B31 + 1)], r'params\[1\] has size 2147483649'),
], ids=['[1, 2^31+1]', '[2^31+1, 1]', '[1, 1, 2^31]', 'next to [1, 2^31-1]'])
def test_adafactor_rejects_factored_dims_past_2_pow_31(hvd, shapes, limit):
    """A factored parameter's geometry holds int32 sizes and strides: one with a dim of 2^31 or more (expanded views, no
    memory) raises RuntimeError naming the limit before anything is launched, also next to a parameter within it."""
    from horovod_b200 import ops
    z = lambda shape, dt: torch.zeros(1, dtype=dt, device='cuda').expand(shape)  # noqa: E731
    ps = [z(s, torch.bfloat16) for s in shapes]
    rows = [z(s[:-1] + (1,), torch.float32) if len(s) >= 2 else None for s in shapes]
    cols = [z(s[:-2] + (1, s[-1]), torch.float32) if len(s) >= 2 else None for s in shapes]
    var = [z(s, torch.float32) if len(s) < 2 else None for s in shapes]
    with pytest.raises(RuntimeError, match=limit):
        ops.fused_adafactor_step(ps, ps, rows, cols, var, lr=1e-2, beta2_decay=-0.8, eps1=None, eps2=1e-3, d=1.0,
                                 weight_decay=0.0, step=1)
