"""The optimizer, gradient, SyncBatchNorm and sharded-collective kernels at sizes their other tests never reach.

* More than 65535 parameters in one fused SGD / Adam / LAMB / LARS call.  The kernels select the table entry with
  gridDim.y, which CUDA caps at 65535, so the binding launches a longer table in pieces: every result against the
  float64 reference and, bit for bit, against the same parameters updated in separate calls.
* Past 2^31 elements (and 2^32 bytes): the offsets where 32-bit index arithmetic (an int product, an unsigned cast, a
  grid dimension sized from a count) would go wrong.  Each test states the device memory it needs in its docstring and
  is skipped, with that number in the reason, when the device has less free memory than that plus 2 GiB.  No float64
  copy of a multi-GB tensor is made: element-wise results are checked against the float64 reference at fixed windows
  (the head, both sides of element 2^31, the fp32 element at byte offset 2^32, the tail and 4096 seeded random
  indices), reductions against float64 sums computed on the device in chunks of 2^26 elements.  Tolerances are those of
  the operation's own tests.  Gathers from a large tensor go through views of one chunk each (`_take`).
"""
import gc
import time

import numpy as np
import pytest
import torch

import test_gpu_lamb as lamb_t
import test_gpu_lars as lars_t
from optim_cases import adam_ref_kernel, f32, hvd, same, ulp  # noqa: F401  (hvd: fixture)
from test_gpu_fused_optimizer import ADAM_HP, SGD_HP, check, sgd_ref_kernel
from test_gpu_sync_batch_norm import EPS, _check

pytestmark = pytest.mark.gpu

GiB = 1 << 30


@pytest.fixture
def room(hvd):
    """room(nbytes): skips the test unless the device has nbytes + 2 GiB free; frees the cached memory afterwards."""
    def need(nbytes):
        free, _ = torch.cuda.mem_get_info()
        if free < nbytes + 2 * GiB:
            pytest.skip(f'needs {nbytes / GiB:.1f} GiB + 2 GiB free device memory, {free / GiB:.1f} GiB free')
    yield need
    gc.collect()
    torch.cuda.empty_cache()


# ---- more than 65535 parameters in one call ---------------------------------------------------------------------------
N_MANY = 70000  # non-empty parameters in one call
EMPTY_AT = (0, 30000, 65535, 65536, N_MANY)  # empty parameters inserted before these non-empty ones
SPLIT_AT = 60000  # the same update in two calls of at most 65535 non-empty parameters: [:SPLIT_AT], [SPLIT_AT:]


class _Part:
    """A parameter's view of a flat buffer, with the Slot interface the LAMB / LARS checks read.  The guard elements
    between the views are checked on the flat buffer."""

    def __init__(self, t):
        self.t = t

    def intact(self):
        return True


def _many_layout():
    """Sizes 1..7 (seeded) plus the empty ones, and each parameter's offset in a flat buffer that keeps one guard
    element after every parameter.  Returns (sizes, offsets, total, mask of the parameters' elements)."""
    sizes = torch.randint(1, 8, (N_MANY,), generator=torch.Generator().manual_seed(7)).tolist()
    for i in sorted(EMPTY_AT, reverse=True):
        sizes.insert(i, 0)
    offs = np.cumsum([0] + [n + 1 for n in sizes])
    total = int(offs[-1])
    inside = torch.ones(total, dtype=torch.bool)
    inside[torch.as_tensor(offs[1:] - 1)] = False
    return sizes, offs[:-1].tolist(), total, inside.cuda()


def _flat(total, scale, seed, square=False):
    x = torch.randn(total, device='cuda', generator=torch.Generator(device='cuda').manual_seed(seed)) * scale
    return x.square() if square else x


def _views(flat, sizes, offs):
    return {k: [v[o:o + n] for o, n in zip(offs, sizes)] for k, v in flat.items()}


def _copy(flat):
    return {k: v.clone() for k, v in flat.items()}


def _same_flat(a, b, what):
    for k in a:
        assert same(a[k], b[k]), f'{what}: {k} differs'


def _split(lists, slots=None):
    """The parameter lists (and slots) of the two separate calls."""
    heads = ({k: v[:SPLIT_AT] for k, v in lists.items()}, None if slots is None else slots[:SPLIT_AT])
    tails = ({k: v[SPLIT_AT:] for k, v in lists.items()}, None if slots is None else slots[SPLIT_AT:])
    assert sum(1 for t in heads[0]['p'] if t.numel()) <= 65535 and sum(1 for t in tails[0]['p'] if t.numel()) <= 65535
    return heads, tails


@pytest.mark.parametrize("kind", ['sgd', 'adam'])
def test_many_params_sgd_adam(hvd, kind):
    """fused_sgd_step (momentum, not the first step) and fused_adam_step over 70,000 fp32 parameters of 1..7 elements and
    5 empty ones: against the float64 reference of every element, the guards between them untouched, and bit for bit
    the same update made in two calls of at most 65535 parameters."""
    from horovod_b200 import ops
    sizes, offs, total, inside = _many_layout()
    if kind == 'sgd':
        f = {'p': _flat(total, 0.1, 1), 'g': _flat(total, 1.0, 2), 'buf': _flat(total, 0.5, 3)}
        run = lambda ls: ops.fused_sgd_step(ls['p'], ls['g'], ls['buf'], **SGD_HP)  # noqa: E731
    else:
        f = {'p': _flat(total, 0.1, 1), 'g': _flat(total, 1.0, 2), 'm': _flat(total, 0.1, 3),
             'v': _flat(total, 0.1, 4, square=True)}
        run = lambda ls: ops.fused_adam_step(ls['p'], ls['g'], ls['m'], ls['v'], step=3, **ADAM_HP)  # noqa: E731
    start = _copy(f)
    run(_views(f, sizes, offs))
    torch.cuda.synchronize()
    x = {k: v.double() for k, v in start.items()}
    if kind == 'sgd':
        p, buf, ps, bs = sgd_ref_kernel(x['p'], x['g'], x['buf'], **SGD_HP)
        want = {'p': (p, ps), 'buf': (buf, bs)}
    else:
        p, m, v, ps, ms, vs = adam_ref_kernel(x['p'], x['g'], x['m'], x['v'], step=3, **ADAM_HP)
        want = {'p': (p, ps), 'm': (m, ms), 'v': (v, vs)}
    for k, (ref, scale) in want.items():
        check(f'{kind} {k}', f[k][inside], ref[inside], scale[inside], torch.float32)
    for k in f:
        assert same(f[k][~inside], start[k][~inside]), f'{kind}: a guard element of {k} was written'
    pieces = _copy(start)
    for ls, _ in _split(_views(pieces, sizes, offs)):
        run(ls)
    torch.cuda.synchronize()
    _same_flat(f, pieces, f'{kind}: one call against two')


@pytest.mark.parametrize("kind", ['lamb', 'lars'])
def test_many_params_lamb_lars(hvd, kind):
    """fused_lamb_step / fused_lars_step over 70,000 fp32 parameters of 1..7 elements and 5 empty ones against the float64
    reference with the bounds of their own tests; the two phases (lamb_norms / lamb_apply, lars_norms / lars_apply)
    with permuted slots in one call each, and in two calls each, bit for bit the same parameters, state and norms."""
    from horovod_b200 import ops
    sizes, offs, total, inside = _many_layout()
    f = {'p': _flat(total, 0.1, 1), 'g': _flat(total, 1.0, 2)}
    if kind == 'lamb':
        f.update(m=_flat(total, 0.1, 3), v=_flat(total, 0.1, 4, square=True))
        hp, step = lamb_t.HP[0], 2
        moments = hp['beta1'], hp['beta2'], hp['eps'], hp['weight_decay'], step

        def norms(ls, out, slots):
            ops.lamb_norms(ls['p'], ls['g'], ls['m'], ls['v'], *moments, out, slots=slots)

        def apply(ls, out, slots):
            ops.lamb_apply(ls['p'], ls['g'], ls['m'], ls['v'], hp['lr'], *moments, out, slots=slots)
    else:
        f.update(v=_flat(total, 0.01, 3))
        hp = lars_t.HP[0]

        def norms(ls, out, slots):
            ops.lars_norms(ls['p'], ls['g'], ls['v'], out, slots=slots)

        def apply(ls, out, slots):
            ops.lars_apply(ls['p'], ls['g'], ls['v'], hp['lr'], hp['momentum'], hp['weight_decay'],
                           hp['trust_coefficient'], hp['eps'], out, slots=slots)
    start = _copy(f)
    lists = _views(f, sizes, offs)
    cases = [{k: _Part(lists[k][i]) for k in lists} for i in range(len(sizes))]
    if kind == 'lamb':
        lamb_t._run_and_check(cases, hp, step)
    else:
        lars_t._run_and_check(cases, hp)
    for k in f:
        assert same(f[k][~inside], start[k][~inside]), f'{kind}: a guard element of {k} was written'
    slots = list(reversed(range(len(sizes))))
    phased, phased_norms = _copy(start), torch.zeros(2 * len(sizes), device='cuda')
    ls = _views(phased, sizes, offs)
    norms(ls, phased_norms, slots)
    apply(ls, phased_norms, slots)
    pieces, pieces_norms = _copy(start), torch.zeros(2 * len(sizes), device='cuda')
    parts = _split(_views(pieces, sizes, offs), slots)
    for ls, sl in parts:
        norms(ls, pieces_norms, sl)
    for ls, sl in parts:
        apply(ls, pieces_norms, sl)
    torch.cuda.synchronize()
    _same_flat(f, phased, f'{kind}: the fused step against its two phases')
    _same_flat(f, pieces, f'{kind}: one call per phase against two')
    assert same(phased_norms, pieces_norms), f'{kind}: norms of one call against two'


def test_many_params_distributed_sgd(hvd):
    """DistributedOptimizer(torch.optim.SGD(...), fused=True) at world size 1 with one param group of 70,000 parameters
    against torch.optim.SGD, two steps (the first creates the momentum buffers).  The reduction at world size 1 is the
    identity and is skipped: what runs is the fused update of the whole group."""
    from horovod_b200 import ops
    sizes = [n for n in _many_layout()[0] if n]
    p0 = _flat(sum(sizes), 0.1, 1).split(sizes)
    ps = [torch.nn.Parameter(t.clone()) for t in p0]
    qs = [torch.nn.Parameter(t.clone()) for t in p0]
    hp = dict(lr=0.05, momentum=0.9, weight_decay=1e-3)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(ps, **hp), named_parameters=[(f'p{i}', p) for i, p in enumerate(ps)],
                                   fused=True)
    ref = torch.optim.SGD(qs, **hp)
    for step in range(2):
        for p, q, g in zip(ps, qs, _flat(sum(sizes), 1.0, 10 + step).split(sizes)):
            p.grad, q.grad = g.clone(), g.clone()
        before = ops.kernel_launches()
        with opt.skip_synchronize():
            opt.step()
        assert ops.kernel_launches() > before, 'the fused update did not run'
        ref.step()
    torch.cuda.synchronize()
    torch.testing.assert_close(torch.cat([p.detach() for p in ps]), torch.cat([q.detach() for q in qs]), rtol=1e-5, atol=1e-6)
    bufs = [opt.state[p]['momentum_buffer'] for p in ps]
    torch.testing.assert_close(torch.cat(bufs), torch.cat([ref.state[q]['momentum_buffer'] for q in qs]), rtol=1e-5, atol=1e-6)



# ---- past 2^31 elements ----------------------------------------------------------------------------------------------
B31 = 1 << 31
N_BIG = B31 + 4099  # the last vector of 4 elements is partial
CHUNK = 1 << 26  # elements per float64 reference chunk, per seeded fill and per gather


def _chunks(n):
    return [(a, min(a + CHUNK, n)) for a in range(0, n, CHUNK)]


def _chunk(seed, k, length, dtype, scale=1.0):
    """Chunk k of a seeded fill: the same values every time it is asked for."""
    g = torch.Generator(device='cuda').manual_seed(1000 * seed + k)
    return (torch.randn(length, device='cuda', generator=g) * scale).to(dtype)


def _fill(t, seed, scale=1.0):
    """Fills a 1-D tensor in place on the device, chunk by chunk (see _chunk)."""
    for k, (a, b) in enumerate(_chunks(t.numel())):
        t[a:b].copy_(_chunk(seed, k, b - a, t.dtype, scale))


def _windows(n, fp32_state=False):
    """The elements checked against the float64 reference: the head, both sides of element 2^31, the fp32 element at
    byte offset 2^32, the tail and 4096 seeded random indices (sorted, on the device)."""
    parts = [torch.arange(0, 8192), torch.arange(B31 - 8192, B31 + 8192), torch.arange(n - 8192, n),
             torch.randint(0, n, (4096,), generator=torch.Generator().manual_seed(5))]
    if fp32_state:
        parts.append(torch.tensor([1 << 30]))
    idx = torch.cat(parts).unique()
    return idx[idx < n].cuda()  # the window past 2^31 is longer than the tail beyond it


def _take(t, idx):
    """t.reshape(-1)[idx], gathered through views of one chunk each, so no gather indexes a tensor of 2^31 elements."""
    flat, out = t.reshape(-1), torch.empty(idx.numel(), dtype=t.dtype, device=t.device)
    assert bool(((idx >= 0) & (idx < flat.numel())).all()), 'window index out of range'
    for a, b in _chunks(flat.numel()):
        m = (idx >= a) & (idx < b)
        if bool(m.any()):
            out[m] = flat[a:b][idx[m] - a]
    return out


def _sumsq(t):
    """sum(t^2) in float64, chunk by chunk on the device."""
    return sum(float(t[a:b].double().square().sum()) for a, b in _chunks(t.numel()))


def _amax(t):
    return max(float(t[a:b].double().abs().max()) for a, b in _chunks(t.numel()))


def _views_of(bufs, offset, n):
    """Each buffer's view of n elements at `offset`, and a copy of the elements outside it."""
    views = {k: b[offset:offset + n] for k, b in bufs.items()}
    outside = {k: torch.cat([b[:offset], b[offset + n:]]).clone() for k, b in bufs.items()}
    return views, outside


def _outside_intact(bufs, outside, offset, n, what):
    for k, b in bufs.items():
        assert same(torch.cat([b[:offset], b[offset + n:]]), outside[k]), f'{what}: wrote outside {k}'


@pytest.mark.parametrize("offset", [0, 1], ids=['aligned', 'unaligned'])
def test_large_sgd_bf16(room, offset):
    """Needs 13 GiB.  fused_sgd_step with momentum on a bf16 parameter of 2^31 + 4099 elements (bf16 momentum, bf16
    gradient) and two small ones in the same call: the big one against the float64 SGD reference at the windows, the
    small ones in full, within the bounds of test_gpu_fused_optimizer.  `unaligned`: views 1 element into buffers one
    element longer, so the scalar path crosses 2^31 as well."""
    from horovod_b200 import ops
    room(13 * GiB)
    n = N_BIG
    kinds = (('p', 0.1), ('g', 1.0), ('buf', 0.5))
    bufs = {k: torch.empty(n + 1, dtype=torch.bfloat16, device='cuda') for k, _ in kinds}
    for seed, (k, scale) in enumerate(kinds):
        _fill(bufs[k], seed, scale)
    big, outside = _views_of(bufs, offset, n)
    small = [{k: _chunk(10 + i, j, m, torch.bfloat16, s) for j, (k, s) in enumerate(kinds)} for i, m in enumerate((3, 4097))]
    idx = _windows(n)
    before = [{k: _take(v, idx).double() for k, v in big.items()}] + [{k: v.double() for k, v in s.items()} for s in small]
    tensors = [big] + small
    ops.fused_sgd_step([t['p'] for t in tensors], [t['g'] for t in tensors], [t['buf'] for t in tensors], **SGD_HP)
    torch.cuda.synchronize()
    for i, (t, x) in enumerate(zip(tensors, before)):
        p, buf, ps, bs = sgd_ref_kernel(x['p'], x['g'], x['buf'], **SGD_HP)
        got = (_take(t['p'], idx), _take(t['buf'], idx)) if i == 0 else (t['p'], t['buf'])
        check(f'sgd[{i}] param', got[0], p, ps, torch.bfloat16)
        check(f'sgd[{i}] momentum', got[1], buf, bs, torch.bfloat16)
    assert same(_take(big['g'], idx), before[0]['g'].to(torch.bfloat16)), 'gradient written'
    _outside_intact(bufs, outside, offset, n, 'sgd')


@pytest.mark.parametrize("offset", [0, 1], ids=['aligned', 'unaligned'])
def test_large_lars_norms_and_apply_bf16(room, offset):
    """Needs 17 GiB.  lars_norms then lars_apply on a bf16 parameter and gradient of 2^31 + 4099 elements with an fp32
    momentum buffer, plus a small tensor: both sums of squares against float64 sums taken in chunks, within
    test_gpu_lars' NORM_RTOL (the CTA partials are added in fp64, so the bound does not grow with the length), then the
    update at the windows against the float64 LARS step with those norms, within test_gpu_lars' element bounds.  (LAMB's
    norms kernel is the same CTA tree, but its two fp32 moments would take the same size past 25 GiB.)"""
    from horovod_b200 import ops
    room(17 * GiB)
    n = N_BIG
    bufs = {'p': torch.empty(n + 1, dtype=torch.bfloat16, device='cuda'),
            'g': torch.empty(n + 1, dtype=torch.bfloat16, device='cuda'),
            'v': torch.empty(n + 1, dtype=torch.float32, device='cuda')}
    for seed, (k, scale) in enumerate((('p', 0.1), ('g', 1.0), ('v', 0.01))):
        _fill(bufs[k], seed, scale)
    big, outside = _views_of(bufs, offset, n)
    small = {'p': _chunk(20, 0, 777, torch.bfloat16, 0.1), 'g': _chunk(21, 0, 777, torch.bfloat16),
             'v': _chunk(22, 0, 777, torch.float32, 0.01)}
    hp = lars_t.HP[0]
    lr, mom, wd, tc, eps = (f32(hp[k]) for k in ('lr', 'momentum', 'weight_decay', 'trust_coefficient', 'eps'))
    idx = _windows(n, fp32_state=True)
    x = {k: _take(v, idx).double() for k, v in big.items()}
    want_norms = [_sumsq(big['p']), _sumsq(big['g']), _sumsq(small['p']), _sumsq(small['g'])]
    norms = torch.zeros(4, device='cuda')
    lists = [[t[k] for t in (big, small)] for k in ('p', 'g', 'v')]
    ops.lars_norms(*lists, norms)
    for j, (a, b) in enumerate(zip(norms.tolist(), want_norms)):
        assert abs(a - b) <= lars_t.NORM_RTOL * b, ('sum of squares', j, a, b)
    ops.lars_apply(*lists, hp['lr'], hp['momentum'], hp['weight_decay'], hp['trust_coefficient'], hp['eps'], norms)
    torch.cuda.synchronize()
    wn, gn = want_norms[0] ** 0.5, want_norms[1] ** 0.5
    r = tc * wn / (gn + wd * wn + eps)
    v = mom * x['v'] + lr * r * (x['g'] + wd * x['p'])
    scale_v = mom * x['v'].abs() + lr * r * (x['g'].abs() + (wd * x['p']).abs())
    tol_v = scale_v * (lars_t.NORM_RTOL + lars_t.ELEM_RTOL)
    err_v = (_take(big['v'], idx).double() - v).abs()
    assert not bool((err_v > tol_v).any()), ('momentum', int((err_v > tol_v).sum()))
    w = x['p'] - v
    tol = tol_v + ulp(w, torch.float32) + ulp(w, torch.bfloat16)
    err = (_take(big['p'], idx).double() - w).abs()
    assert not bool((err > tol).any()), ('param', int((err > tol).sum()), float((err - tol).max()))
    assert same(_take(big['g'], idx), x['g'].to(torch.bfloat16)), 'gradient written'
    _outside_intact(bufs, outside, offset, n, 'lars')


@pytest.mark.parametrize("offset", [0, 1], ids=['aligned', 'unaligned'])
def test_large_grad_accumulate_bf16(room, offset):
    """Needs 13 GiB.  grad_accumulate_ 'first', 'add', 'last' on a bf16 gradient of 2^31 + 4099 elements with an fp32
    accumulator: every element bit for bit the same torch ops in fp32, checked chunk by chunk on the device from the
    seeded gradients regenerated there."""
    from horovod_b200 import ops
    room(13 * GiB)
    n = N_BIG
    bufs = {'g': torch.empty(n + 1, dtype=torch.bfloat16, device='cuda'),
            'acc': torch.full((n + 1,), float('nan'), device='cuda')}
    _fill(bufs['g'], 0)
    views, outside = _views_of(bufs, offset, n)
    g, acc = views['g'], views['acc']
    grad = lambda seed, k, a, b: _chunk(seed, k, b - a, torch.bfloat16)  # noqa: E731
    _fill(g, 1)
    ops.grad_accumulate_([g], [acc], 'first')
    torch.cuda.synchronize()
    for k, (a, b) in enumerate(_chunks(n)):
        assert same(acc[a:b], grad(1, k, a, b).float()), ('first: accumulator', a)
        assert not bool(g[a:b].view(torch.int16).any()), ('first: gradient not zeroed', a)
    _fill(g, 2)
    ops.grad_accumulate_([g], [acc], 'add')
    torch.cuda.synchronize()
    for k, (a, b) in enumerate(_chunks(n)):
        assert same(acc[a:b], grad(1, k, a, b).float() + grad(2, k, a, b).float()), ('add: accumulator', a)
        assert not bool(g[a:b].view(torch.int16).any()), ('add: gradient not zeroed', a)
    _fill(g, 3)
    ops.grad_accumulate_([g], [acc], 'last')
    torch.cuda.synchronize()
    for k, (a, b) in enumerate(_chunks(n)):
        s = grad(1, k, a, b).float() + grad(2, k, a, b).float()
        assert same(acc[a:b], s), ('last: accumulator written', a)
        assert same(g[a:b], (s + grad(3, k, a, b).float()).to(torch.bfloat16)), ('last: gradient', a)
    _outside_intact(bufs, outside, offset, n, 'grad_accumulate_')


@pytest.mark.parametrize("offset", [0, 1], ids=['aligned', 'unaligned'])
def test_large_grad_shard_stats_bf16(room, offset):
    """Needs 5 GiB.  grad_shard_stats on a bf16 gradient of 2^31 + 4099 elements plus a small one: the sum of squares
    (within test_gpu_sharded_clip's 1e-6: the CTA partials are added in fp64, so it does not grow with the length) and
    the inf-norm (exact) against float64 chunk by chunk; an inf at element 2^31, and in another call at the last element,
    sets the non-finite flag; the in-place unscale at the windows bit for bit."""
    from horovod_b200 import ops
    room(5 * GiB)
    n = N_BIG
    bufs = {'g': torch.empty(n + 1, dtype=torch.bfloat16, device='cuda')}
    _fill(bufs['g'], 0, 3.0)
    views, outside = _views_of(bufs, offset, n)
    big = views['g']
    small = _chunk(1, 0, 1000, torch.bfloat16, 3.0)
    sum_sq, max_abs = _sumsq(big) + _sumsq(small), max(_amax(big), _amax(small))
    for norm_type in (2.0, float('inf')):
        out = torch.zeros(2, device='cuda')
        ops.grad_shard_stats([big, small], out, norm_type=norm_type)
        o = out.tolist()
        if norm_type == 2.0:
            assert abs(o[0] - sum_sq) <= 1e-6 * sum_sq, (o[0], sum_sq)
        else:
            assert o[0] == max_abs, (o[0], max_abs)
        assert o[1] == 0.0
    for where in (B31, n - 1):
        keep = big[where].clone()
        big[where] = float('inf')
        out = torch.zeros(2, device='cuda')
        ops.grad_shard_stats([big, small], out)
        assert out.tolist() == [float('inf'), 1.0], (where, out.tolist())
        big[where] = keep
    idx = _windows(n)
    s = torch.tensor([0.3719], device='cuda')
    expect = (_take(big, idx).float() * s).to(torch.bfloat16)
    out = torch.zeros(2, device='cuda')
    ops.grad_shard_stats([big, small], out, inv_scale=s)
    torch.cuda.synchronize()
    assert same(_take(big, idx), expect), 'in-place unscale'
    ref = _sumsq(big) + _sumsq(small)
    assert abs(float(out[0]) - ref) <= 1e-6 * ref and float(out[1]) == 0.0
    _outside_intact(bufs, outside, offset, n, 'grad_shard_stats')


def _bn_pieces(layout, ts):
    """The channels of rows [M, C] or planes [N, C, L] tensors in float64 chunks: (None, [rows, C] chunks) for rows,
    (c, 1-D chunks of one plane) for planes."""
    if layout == 'rows':
        step = CHUNK // ts[0].shape[1]
        for r0 in range(0, ts[0].shape[0], step):
            yield None, [t[r0:r0 + step].double() for t in ts]
    else:
        for i in range(ts[0].shape[0]):
            for c in range(ts[0].shape[1]):
                for a, b in _chunks(ts[0].shape[2]):
                    yield c, [t[i, c, a:b].double() for t in ts]


def _bn_sum(layout, f, ts, mean):
    """Per channel, the float64 sum of f(chunks of ts..., the channel's mean)."""
    acc = torch.zeros(ts[0].shape[1], dtype=torch.float64, device='cuda')
    for c, xs in _bn_pieces(layout, ts):
        if c is None:
            acc += f(*xs, mean.view(1, -1)).sum(0)
        else:
            acc[c] += f(*xs, mean[c]).sum()
    return acc


# rows: C = 7 is not a multiple of any vector width; planes: (n * C + c) * L passes 2^31 from plane (1, 0) on
BN_SHAPES = {'rows': (-(-N_BIG // 7), 7), 'planes': (2, 3, -(-N_BIG // 6))}


@pytest.mark.parametrize("layout", list(BN_SHAPES))
def test_large_sync_batch_norm_bf16(room, layout):
    """Needs 14 GiB.  The SyncBatchNorm kernels on a bf16 input of more than 2^31 elements, rows [M, 7] or planes
    [2, 3, L]: the slot's (count, mean, M2) and sync_bn_combine's mean / invstd against float64 statistics taken in chunks,
    y and, in a separate allocation, dx at the windows, and the backward sums; all within the bounds of
    test_gpu_sync_batch_norm's test_kernels_against_fp64."""
    from horovod_b200 import ops
    room(14 * GiB)
    shape = BN_SHAPES[layout]
    c = shape[1]
    x = torch.empty(shape, dtype=torch.bfloat16, device='cuda')
    _fill(x.view(-1), 0, 2.0)
    x.view(-1).add_(0.5)
    n = x.numel() // c
    zero = torch.zeros(c, dtype=torch.float64, device='cuda')
    mean = _bn_sum(layout, lambda v, m: v, [x], zero) / n
    var = _bn_sum(layout, lambda v, m: (v - m) ** 2, [x], mean) / n
    invstd, spread = 1.0 / torch.sqrt(var + EPS), var.sqrt()
    w = (torch.rand(c, generator=torch.Generator().manual_seed(1), dtype=torch.float64) + 0.5).float().cuda()
    b = torch.randn(c, generator=torch.Generator().manual_seed(2), dtype=torch.float64).float().cuda()
    per = ops.sync_bn_slot_doubles(c)
    slot = torch.full((per,), -7.0, dtype=torch.float64, device='cuda')
    ops.sync_bn_stats(x, slot)
    m, istd, cnt = ops.sync_bn_combine(slot.view(1, per), c, EPS, 0.1)
    torch.cuda.synchronize()
    assert float(slot[0]) == n and float(cnt[0]) == f32(n)  # the combined count is float32: n > 2^24 rounds
    top = float((mean.abs() + spread).max())
    torch.testing.assert_close(slot[1::3][:c], mean, rtol=0, atol=1e-6 * top)
    torch.testing.assert_close(slot[2::3][:c] / n, var, rtol=1e-4, atol=1e-6 * top ** 2 * 1e-3)
    torch.testing.assert_close(m.double(), mean, rtol=1e-5, atol=1e-6 * float(spread.max()))
    torch.testing.assert_close(istd.double(), invstd, rtol=1e-5, atol=0)
    idx = _windows(x.numel())
    ch = idx % c if layout == 'rows' else (idx // shape[2]) % c
    xd = _take(x, idx).double()
    wd, bd, md, sd = w.double()[ch], b.double()[ch], mean[ch], invstd[ch]
    y = ops.sync_bn_elemt(x, m, istd, w, b)
    scale_y = (xd.abs() + md.abs()) * sd * wd.abs() + bd.abs()
    _check(_take(y, idx), (xd - md) * sd * wd + bd, scale_y, torch.bfloat16, 'y')
    del y
    dy = torch.empty_like(x)
    _fill(dy.view(-1), 1)
    sums = torch.empty(2 * c, dtype=torch.float64, device='cuda')
    ops.sync_bn_backward_reduce(dy, x, m, istd, w, sums, False, False)
    dx = ops.sync_bn_backward_elemt(dy, x, m, istd, w, sums, cnt)
    torch.cuda.synchronize()
    sdy = _bn_sum(layout, lambda g, v, mu: g, [dy, x], mean)
    sdyx = _bn_sum(layout, lambda g, v, mu: g * (v - mu), [dy, x], mean)
    _check(sums[0::2], sdy, _bn_sum(layout, lambda g, v, mu: g.abs(), [dy, x], mean), torch.float32, 'sum_dy')
    _check(sums[1::2], sdyx, _bn_sum(layout, lambda g, v, mu: g.abs() * (v.abs() + mu.abs()), [dy, x], mean),
           torch.float32, 'sum_dy_xmu')
    dyd = _take(dy, idx).double()
    k = (invstd ** 2 * sdyx / n)[ch]
    want = (dyd - sdy[ch] / n - (xd - md) * k) * sd * wd
    scale_dx = (dyd.abs() + sdy.abs()[ch] / n + (xd.abs() + md.abs()) * k.abs()) * (sd * wd.abs())
    _check(_take(dx, idx), want, scale_dx, torch.bfloat16, 'dx')


def test_large_inplace_reducescatter_allgather_bf16(room):
    """Needs 9 GiB.  The in-place reduce-scatter and allgather kernels on 2 simulated ranks, each holding a bf16 tensor
    of 2^31 + 4112 elements (the nearest multiple of the 16 bytes per rank the kernels need), so rank 1's shard starts
    past byte 2^31 and ends past byte 2^32: the reduced shards at the windows against the float64 sum within
    test_gpu_sharded's bound, every byte outside a rank's own shard untouched, then the allgather byte for byte."""
    from horovod_b200.ops import sim
    room(9 * GiB)
    n = B31 + 4112
    h = n // 2
    seeds = (30, 31)
    ts = [torch.empty(n, dtype=torch.bfloat16, device='cuda') for _ in seeds]
    for t, s in zip(ts, seeds):
        _fill(t, s)
    idx = _windows(n)
    want = (_take(ts[0], idx).double() + _take(ts[1], idx).double()).to(torch.bfloat16).double()
    sim.inplace_reducescatter(ts, op=sim.SUM, ctas=8)
    torch.cuda.synchronize()
    reduced = torch.where(idx < h, _take(ts[0], idx), _take(ts[1], idx))
    torch.testing.assert_close(reduced.double(), want, rtol=2e-2, atol=2e-2)
    for r, (t, s) in enumerate(zip(ts, seeds)):
        lo, hi = r * h, (r + 1) * h
        for k, (a, b) in enumerate(_chunks(n)):
            x, got = _chunk(s, k, b - a, torch.bfloat16), t[a:b]
            keep = torch.ones(b - a, dtype=torch.bool, device='cuda')
            keep[max(lo, a) - a:max(min(hi, b) - a, 0)] = False
            assert same(got[keep], x[keep]), ('reduce-scatter wrote outside the own shard', r, a)
    sim.inplace_allgather(ts, ctas=8)
    torch.cuda.synchronize()
    for t in ts:
        assert same(_take(t, idx), reduced), 'allgather at the windows'
    for a, b in _chunks(n):
        assert same(ts[0][a:b], ts[1][a:b]), ('allgather: the ranks differ', a)


# ---- expert-parallel dispatch (moe_kernels.cu) and the captured alltoall past 2^31 --------------------------------------

def _peak(what, t0):
    """Prints the wall time since t0 and the peak device memory of the test, for the record."""
    torch.cuda.synchronize()
    print(f'\n{what}: {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / GiB:.1f} GiB')


def _seeded_ints(t, seed, high):
    """Fills a 1-D integer tensor in place with seeded values in [0, high), chunk by chunk."""
    for k, (a, b) in enumerate(_chunks(t.numel())):
        g = torch.Generator(device='cuda').manual_seed(1000 * seed + k)
        t[a:b].copy_(torch.randint(0, high, (b - a,), device='cuda', generator=g, dtype=t.dtype))


def test_large_moe_permute_bf16(room):
    """Needs 30 GiB.  moe_permute at the binding's limit: T k = 2^31 - 16 assignments (k = 16, int32 ids over E = 8
    experts, n = 4 ranks) of bf16 rows of h = 3 (6 bytes, the element path), so the send buffer passes 2^31 elements
    and 2^33 bytes.  The counts against bincount in chunks, the splits, and for every chunk and expert that the positions
    of that expert's assignments, ascending, are exactly base_e, base_e + 1, ... (the stable argsort, checked without a
    global sort); send[pos[a]] == x[a // k] at the windows.  Prints the call's time: the last route CTA scans the 2^20
    tiles serially per expert."""
    from horovod_b200 import ops
    room(30 * GiB)
    torch.cuda.reset_peak_memory_stats()
    t_start = time.perf_counter()
    k, E, n, h = 16, 8, 4, 3
    A = B31 - 16
    T = A // k
    ids = torch.empty(A, dtype=torch.int32, device='cuda')
    _seeded_ints(ids, 40, E)
    x = torch.empty(T * h, dtype=torch.bfloat16, device='cuda')
    _fill(x, 41)
    x = x.view(T, h)
    send = torch.empty(A, h, dtype=torch.bfloat16, device='cuda')
    counts = torch.full((E,), -5, dtype=torch.int64, device='cuda')
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pos, splits = ops.moe_permute(x, ids.view(T, k), E, n, send, counts)
    torch.cuda.synchronize()
    print(f'\nmoe_permute of {A} assignments: {time.perf_counter() - t0:.2f} s')
    want = sum(torch.bincount(ids[a:b], minlength=E) for a, b in _chunks(A))
    assert torch.equal(counts, want), (counts.tolist(), want.tolist())
    assert splits.tolist() == want.view(n, -1).sum(1).tolist()
    base = torch.cumsum(want, 0) - want
    flat = pos.view(-1)
    seen = [0] * E
    for a, b in _chunks(A):
        chunk_ids, chunk_pos = ids[a:b], flat[a:b]
        for e in range(E):
            got = chunk_pos[chunk_ids == e].long()
            start = int(base[e]) + seen[e]
            assert torch.equal(got, torch.arange(start, start + got.numel(), device='cuda')), ('stable order', a, e)
            seen[e] += got.numel()
    assert seen == want.tolist()
    idx = _windows(A)
    p = _take(flat, idx).long()
    for c in range(h):
        assert same(_take(send, p * h + c), _take(x, (idx // k) * h + c)), ('send rows', c)
    assert int(p.max()) * h > (1 << 32), 'the windows reach a send row past element 2^32'
    _peak('test_large_moe_permute_bf16', t_start)


def _rows_at(t, rows):
    """t[rows] for a 2-D tensor of more than 2^31 elements, one row view at a time."""
    return torch.stack([t[r] for r in rows.tolist()])


@pytest.mark.parametrize("h", [1 << 15, (1 << 15) + 3], ids=['vector', 'element'])
def test_large_moe_scatter_gather_regroup_bf16(room, h):
    """Needs 30 GiB.  T = 2^16 + 1 bf16 tokens of h = 2^15 (16 B rows, the vector path) or 2^15 + 3 (the element path),
    k = 2 over 4 experts: x passes 2^31 elements and the send buffer 2^32.  Checked at the tokens whose rows straddle
    element 2^31, whose send rows lie past element 2^32, the last token and 64 random ones:
    - moe_permute's copy: send[pos[t, j]] == x[t];
    - the weighted gather, bit-exact to the fp32 model and within the float64 bound;
    - the scaled scatter, bit-exact, and its gate-gradient dot within dot_bound;
    - the regroup with counts [4, 8] at sampled rows against a host-computed row map, and its reverse as the exact
      inverse, chunk by chunk."""
    from horovod_b200 import ops
    from test_gpu_moe_dispatch import dot_bound, ref_gather
    from test_gpu_moe_edges import check_value, gather64, same_bits
    room(30 * GiB)
    torch.cuda.reset_peak_memory_stats()
    t_start = time.perf_counter()
    T, k, E = (1 << 16) + 1, 2, 4
    R = T * k
    x = torch.empty(T * h, dtype=torch.bfloat16, device='cuda')
    _fill(x, 50)
    x = x.view(T, h)
    ids = torch.randint(0, E, (T, k), device='cuda', generator=torch.Generator(device='cuda').manual_seed(51))
    send = torch.empty(R, h, dtype=torch.bfloat16, device='cuda')
    pos, _ = ops.moe_permute(x, ids, E, 1, send, torch.empty(E, dtype=torch.int64, device='cuda'))
    gates = torch.rand(T, k, device='cuda', generator=torch.Generator(device='cuda').manual_seed(52))
    y = ops.moe_gather(send, pos, gates)
    dst = torch.zeros(R, h, dtype=torch.bfloat16, device='cuda')
    gg = ops.moe_scatter(x, pos, dst, gates, send)
    torch.cuda.synchronize()
    far = ((pos.long() + 1) * h > (1 << 32)).any(1).nonzero().flatten()  # a send row reaching past element 2^32
    assert far.numel() > 0
    toks = torch.cat([torch.arange(B31 // h - 1, B31 // h + 2, device='cuda'), far, torch.tensor([T - 1], device='cuda'),
                      torch.randint(0, T, (64,), device='cuda', generator=torch.Generator(device='cuda').manual_seed(53))])
    toks = toks[toks < T].unique()
    xt, pt, gt = _rows_at(x, toks), pos[toks], gates[toks]
    rows = [_rows_at(send, pt[:, j]) for j in range(k)]
    for j in range(k):
        assert same(rows[j], xt), ('send rows', j)
    local = torch.cat(rows)  # the k send rows of each token, as a small src with pos = j * len(toks) + i
    lpos = torch.stack([torch.arange(len(toks), device='cuda') + j * len(toks) for j in range(k)], 1).to(torch.int32)
    yt = _rows_at(y, toks)
    assert same_bits(yt, ref_gather(local, lpos, gt, torch.bfloat16)), 'gather bits'
    w64, bound = gather64(local, lpos, gt)
    check_value(yt, w64, bound, 'gather value')
    for j in range(k):
        assert same(_rows_at(dst, pt[:, j]), (gt[:, j:j + 1] * xt.float()).to(torch.bfloat16)), ('scatter', j)
        exact = (xt.double() * rows[j].double()).sum(-1)
        assert bool(((gg[toks, j].double() - exact).abs() <= dot_bound(xt, rows[j])).all()), ('gate gradient', j)
    del y, dst, gg
    gc.collect()
    torch.cuda.empty_cache()
    # regroup: 4 source ranks x 8 local experts, 5 rows short of R, some segments empty
    g = torch.Generator().manual_seed(54)
    wts = torch.rand(32, generator=g) * (torch.rand(32, generator=g) > 0.25)
    c = (wts / wts.sum() * (R - 5)).floor().long()
    c[int(wts.argmax())] += R - 5 - int(c.sum())
    counts = c.view(4, 8)
    total = int(counts.sum())
    out, offsets = ops.moe_regroup(send, counts.cuda())
    torch.cuda.synchronize()
    cl = counts.tolist()
    src_start, at = {}, 0
    for p in range(4):
        for e in range(8):
            src_start[(p, e)], at = at, at + cl[p][e]
    row_map, ends = [], []
    for e in range(8):
        for p in range(4):
            row_map += range(src_start[(p, e)], src_start[(p, e)] + cl[p][e])
        ends.append(len(row_map))
    assert offsets.tolist() == ends
    sample = torch.cat([torch.arange(0, 16), torch.arange(B31 // h - 2, B31 // h + 3), torch.arange((1 << 32) // h - 2, R),
                        torch.randint(0, R, (128,), generator=g)]).unique()
    sample = sample[sample < R]
    inside = sample[sample < total]
    assert same(_rows_at(out, inside.cuda()), _rows_at(send, torch.tensor([row_map[r] for r in inside.tolist()]).cuda()))
    assert not bool(out[total:].view(torch.int16).any()), 'tail not zeroed'
    back = torch.full_like(send, 3.0)
    ret = ops.moe_regroup_reverse(out, counts.cuda(), back)
    torch.cuda.synchronize()
    assert ret.tolist() == counts.sum(1).tolist()
    flat_b, flat_s = back.view(-1), send.view(-1)
    for a, b in _chunks(total * h):
        assert same(flat_b[a:b], flat_s[a:b]), ('reverse is not the inverse', a)
    assert bool((back[total:] == 3.0).all()), 'reverse wrote past the total'
    _peak(f'test_large_moe_scatter_gather_regroup_bf16[{h}]', t_start)


def _seeded_bytes(seed, k, length):
    g = torch.Generator(device='cuda').manual_seed(1000 * seed + k)
    return torch.randint(0, 256, (length,), dtype=torch.uint8, device='cuda', generator=g)


@pytest.mark.parametrize("R,row", [(530000, 4098), (265000, 8192)], ids=['bytes', 'vector'])
def test_large_captured_alltoall(room, R, row):
    """Needs 10 GiB.  The captured alltoall on 2 simulated ranks whose inputs are each just over 2^31 bytes: R rows of
    4098 bytes (unaligned rows, the byte path) or of 8192 bytes (the 16 B vector path), splits [[R - 1000, 1000],
    [R - 500, 500]], so rank 0's output passes byte 2^32 and both source offsets rank 1 reads are past 2^31.  The output
    byte for byte against the inputs, chunk by chunk on the device, the guard rows after it untouched, and the inputs
    unchanged against their seeded fill."""
    from horovod_b200.ops import sim
    room(10 * GiB)
    torch.cuda.reset_peak_memory_stats()
    t_start = time.perf_counter()
    assert R * row > B31
    M = [[R - 1000, 1000], [R - 500, 500]]
    ins = [torch.empty(R, row, dtype=torch.uint8, device='cuda') for _ in range(2)]
    for r, t in enumerate(ins):
        for i, (a, b) in enumerate(_chunks(t.numel())):
            t.view(-1)[a:b] = _seeded_bytes(60 + r, i, b - a)
    recv_rows = [M[0][q] + M[1][q] for q in range(2)]
    outs = [torch.full((recv_rows[q] + 3, row), 0x5A, dtype=torch.uint8, device='cuda') for q in range(2)]
    assert recv_rows[0] * row > (1 << 32)
    splits = [torch.tensor(m, dtype=torch.int64, device='cuda') for m in M]
    recv = [torch.full((2,), -7, dtype=torch.int64, device='cuda') for _ in range(2)]
    status = [torch.full((1,), -7, dtype=torch.int32, device='cuda') for _ in range(2)]
    sim.captured_alltoall(ins, splits, outs, recv, status, ctas=8)
    torch.cuda.synchronize()
    assert [int(s) for s in status] == [0, 0]
    assert recv[0].tolist() == [M[0][0], M[1][0]] and recv[1].tolist() == [M[0][1], M[1][1]]
    # (output q, its first row, sender p, the sender's first row, rows)
    pieces = [(0, 0, 0, 0, M[0][0]), (0, M[0][0], 1, 0, M[1][0]), (1, 0, 0, M[0][0], M[0][1]),
              (1, M[0][1], 1, M[1][0], M[1][1])]
    for q, o0, p, i0, n in pieces:
        dst, src = outs[q].view(-1)[o0 * row:(o0 + n) * row], ins[p].view(-1)[i0 * row:(i0 + n) * row]
        for a, b in _chunks(n * row):
            assert torch.equal(dst[a:b], src[a:b]), ('output', q, p, a)
    assert (M[0][0] * row > B31) and (M[1][0] * row > B31)
    for q in range(2):
        assert bool((outs[q][recv_rows[q]:] == 0x5A).all()), ('guard rows', q)
    for r, t in enumerate(ins):
        for i, (a, b) in enumerate(_chunks(t.numel())):
            assert torch.equal(t.view(-1)[a:b], _seeded_bytes(60 + r, i, b - a)), ('input written', r, a)
    _peak(f'test_large_captured_alltoall[{row}]', t_start)
