"""hvd.SyncBatchNorm's native path: the sm_90a kernels against a float64 model of SyncBatchNorm over the concatenated
batch, the statistics exchange on simulated ranks with the real collective kernels, the module (with capturable
stand-ins for the collectives) eagerly and in hvd.GraphedStep, and a real multi-GPU run when there are two GPUs."""
import zlib

import pytest
import torch

EPS = 1e-5


# ---- float64 reference ---------------------------------------------------------------------------------------------
def _ref_forward(xs, weight, bias, rm, rv, momentum, eps=EPS):
    """SyncBatchNorm over per-rank batches `xs` in float64: per-rank (count, mean, M2), merged in rank order (Chan)."""
    n, mean, m2 = 0.0, None, None
    for x in xs:
        x = x.double()
        c = x.size(1)
        flat = x.transpose(0, 1).reshape(c, -1)
        nb = flat.size(1)
        if nb == 0:
            continue
        mb = flat.mean(1)
        qb = ((flat - mb[:, None]) ** 2).sum(1)
        if mean is None:
            n, mean, m2 = float(nb), mb, qb
        else:
            nab = n + nb
            d = mb - mean
            mean = mean + d * (nb / nab)
            m2 = m2 + qb + d * d * (n * nb / nab)
            n = nab
    var = m2 / n
    invstd = 1.0 / torch.sqrt(var + eps)
    new_rm = new_rv = None
    if rm is not None:
        unbiased = var * n / (n - 1) if n > 1 else var
        new_rm = (1 - momentum) * rm.double() + momentum * mean
        new_rv = (1 - momentum) * rv.double() + momentum * unbiased
    shape = lambda x: [1, -1] + [1] * (x.dim() - 2)  # noqa: E731
    ys = []
    for x in xs:
        y = (x.double() - mean.view(shape(x))) * invstd.view(shape(x))
        if weight is not None:
            y = y * weight.double().view(shape(x)) + bias.double().view(shape(x))
        ys.append(y)
    return ys, mean, var, invstd, n, new_rm, new_rv


def _ref_backward(xs, dys, weight, mean, invstd, n):
    """dx per rank, the summed (sum dy, sum dy * (x - mean)), and per-rank local (grad_weight, grad_bias)."""
    shape = lambda x: [1, -1] + [1] * (x.dim() - 2)  # noqa: E731
    dims = lambda x: [0] + list(range(2, x.dim()))  # noqa: E731
    sdy = sum(dy.double().sum(dims(dy)) for dy in dys)
    sdyx = sum((dy.double() * (x.double() - mean.view(shape(x)))).sum(dims(x)) for x, dy in zip(xs, dys))
    w = weight.double() if weight is not None else torch.ones_like(mean)
    dxs, local = [], []
    for x, dy in zip(xs, dys):
        xmu = x.double() - mean.view(shape(x))
        dx = (dy.double() - (sdy / n).view(shape(x)) - xmu * (invstd ** 2 * sdyx / n).view(shape(x))) \
            * (invstd * w).view(shape(x))
        dxs.append(dx)
        lb = dy.double().sum(dims(x))
        local.append(((dy.double() * xmu).sum(dims(x)) * invstd, lb))
    return dxs, sdy, sdyx, local


def test_reference_matches_torch_batchnorm_on_the_concatenated_batch():
    """The float64 model (rank-order Chan merge of per-rank statistics) is BatchNorm over the concatenation."""
    g = torch.Generator().manual_seed(0)
    c = 5
    xs = [torch.randn(b, c, 3, 4, generator=g, dtype=torch.float64) * 3 + 7 for b in (1, 4, 2)]
    dys = [torch.randn(x.shape, generator=g, dtype=torch.float64) for x in xs]
    w = torch.rand(c, generator=g, dtype=torch.float64) + 0.5
    b = torch.randn(c, generator=g, dtype=torch.float64)
    rm, rv = torch.randn(c, generator=g, dtype=torch.float64), torch.rand(c, generator=g, dtype=torch.float64) + 1
    ys, mean, var, invstd, n, new_rm, new_rv = _ref_forward(xs, w, b, rm, rv, 0.3)
    dxs, sdy, sdyx, local = _ref_backward(xs, dys, w, mean, invstd, n)

    bn = torch.nn.BatchNorm2d(c, momentum=0.3).double()
    with torch.no_grad():
        bn.weight.copy_(w)
        bn.bias.copy_(b)
        bn.running_mean.copy_(rm)
        bn.running_var.copy_(rv)
    x = torch.cat(xs).requires_grad_()
    y = bn(x)
    y.backward(torch.cat(dys))
    tol = dict(rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(torch.cat(ys), y.detach(), **tol)
    torch.testing.assert_close(mean, x.detach().mean((0, 2, 3)), **tol)
    torch.testing.assert_close(var, x.detach().var((0, 2, 3), unbiased=False), **tol)
    torch.testing.assert_close(new_rm, bn.running_mean, **tol)
    torch.testing.assert_close(new_rv, bn.running_var, **tol)
    torch.testing.assert_close(torch.cat(dxs), x.grad, **tol)
    torch.testing.assert_close(sum(l[0] for l in local), bn.weight.grad, **tol)
    torch.testing.assert_close(sum(l[1] for l in local), bn.bias.grad, **tol)


# ---- helpers for the GPU tests -------------------------------------------------------------------------------------
def _make(shape, layout, dtype, offset, shift, gen, device='cuda'):
    """A tensor of `shape` in `layout` whose storage starts `offset` elements into its allocation."""
    x = torch.randn(shape, generator=gen, dtype=torch.float64) + shift
    if layout == 'cl4':
        perm = (0, 2, 3, 1)
    elif layout == 'cl5':
        perm = (0, 2, 3, 4, 1)
    else:
        perm = tuple(range(len(shape)))
    xp = x.permute(*perm).contiguous().to(dtype)
    buf = torch.empty(xp.numel() + offset, dtype=dtype, device=device)
    buf[offset:].copy_(xp.reshape(-1))
    inv = [perm.index(i) for i in range(len(shape))]
    return buf[offset:].view(xp.shape).permute(*inv)


def _ulp(t):
    """One unit in the last place of every element of t (in t's dtype), as float64."""
    t = t.abs()
    nxt = torch.nextafter(t.float(), torch.full_like(t.float(), float('inf'))) if t.dtype == torch.float32 else None
    if nxt is not None:
        return (nxt.double() - t.double())
    finfo = torch.finfo(t.dtype)
    e = torch.floor(torch.log2(torch.clamp(t.double(), min=finfo.smallest_normal)))
    return torch.pow(2.0, e) * finfo.eps


def _check(out, ref, scale, dtype, what):
    outd = out.double()
    tol = 1e-5 * scale
    if dtype != torch.float32:
        tol = tol + _ulp(ref.to(dtype))
    bad = (outd - ref).abs() > tol
    assert not bad.any(), '%s: %d elements off, worst %.3g (tol %.3g)' % (
        what, int(bad.sum()), float(((outd - ref).abs() - tol).max()), float(tol.max() if torch.is_tensor(tol) else tol))


def _guarded(n, dtype, fill, device='cuda'):
    """A view of n elements inside a buffer with 64 sentinel elements on each side; returns (view, buffer)."""
    buf = torch.full((n + 128,), fill, dtype=dtype, device=device)
    return buf[64:64 + n], buf


def _slack_ok(buf, n, fill):
    return bool((buf[:64] == fill).all()) and bool((buf[64 + n:] == fill).all())


CASES = []
for _dt in (torch.float32, torch.bfloat16, torch.float16):
    for _wdt in ('f32', 'same'):
        CASES.append(('cl4', (32, 64, 7, 7), _dt, _wdt, 0, 0.0))
for _lay, _shape in (('cl4', (4, {}, 5, 3)), ('cl5', (3, {}, 2, 3, 4)), ('nchw', (4, {}, 5, 3)), ('nc', (37, {})),
                     ('ncl', (5, {}, 19))):
    for _c in (1, 3, 8, 257):
        CASES.append((_lay, tuple(_c if s == {} else s for s in _shape), torch.bfloat16, 'f32', 0, 0.0))
for _lay, _shape in (('cl4', (6, 8, 5, 3)), ('nchw', (6, 8, 4, 4)), ('nc', (29, 257))):
    for _off in (1, 2, 3):
        for _dt in (torch.float32, torch.bfloat16):
            CASES.append((_lay, _shape, _dt, 'same', _off, 0.0))
CASES += [
    ('cl4', (32, 64, 112, 112), torch.bfloat16, 'f32', 0, 0.0),
    ('cl4', (32, 256, 56, 56), torch.bfloat16, 'f32', 0, 0.0),
    ('cl4', (32, 2048, 7, 7), torch.bfloat16, 'f32', 0, 0.0),
    ('cl4', (32, 2048, 1, 1), torch.bfloat16, 'f32', 0, 0.0),
    ('nchw', (32, 64, 56, 56), torch.float32, 'f32', 0, 0.0),
    ('nchw', (8, 3, 112, 112), torch.float16, 'same', 0, 0.0),
    ('cl4', (16, 64, 14, 14), torch.float32, 'f32', 0, 1000.0),
    ('cl4', (16, 64, 14, 14), torch.bfloat16, 'f32', 0, 300.0),
    ('nchw', (16, 8, 28, 28), torch.float32, 'f32', 0, 1000.0),
    ('nc', (4096, 8), torch.float32, 'f32', 0, 5000.0),
]


def _case_id(c):
    return '%s-%s-%s-w%s-off%d%s' % (c[0], 'x'.join(map(str, c[1])), str(c[2]).split('.')[-1], c[3], c[4],
                                     '-shift%g' % c[5] if c[5] else '')


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
def test_kernels_against_fp64(case):
    from horovod_b200 import ops
    layout, shape, dtype, wkind, offset, shift = case
    gen = torch.Generator().manual_seed(zlib.crc32(_case_id(case).encode()))
    x = _make(shape, layout, dtype, offset, shift, gen)
    dy = _make(shape, layout, dtype, offset, 0.0, gen)
    assert x.stride() == dy.stride()
    c = shape[1]
    wdt = torch.float32 if wkind == 'f32' else dtype
    w = (torch.rand(c, generator=gen, dtype=torch.float64) + 0.5).to(wdt).cuda()
    b = torch.randn(c, generator=gen, dtype=torch.float64).to(wdt).cuda()
    rm0 = torch.randn(c, generator=gen, dtype=torch.float64).to(wdt)
    rv0 = (torch.rand(c, generator=gen, dtype=torch.float64) + 0.5).to(wdt)

    ys, mean, var, invstd, n, new_rm, new_rv = _ref_forward([x.cpu()], w.cpu(), b.cpu(), rm0, rv0, 0.1)
    dxs, sdy, sdyx, local = _ref_backward([x.cpu()], [dy.cpu()], w.cpu(), mean, invstd, n)

    def run():
        per = ops.sync_bn_slot_doubles(c)
        slot, sbuf = _guarded(per, torch.float64, -7.0)
        ops.sync_bn_stats(x, slot)
        rm, rmb = _guarded(c, wdt, -3.0)
        rv, rvb = _guarded(c, wdt, -3.0)
        rm.copy_(rm0)
        rv.copy_(rv0)
        m, istd, cnt = ops.sync_bn_combine(slot.view(1, per), c, EPS, 0.1, rm, rv)
        y = ops.sync_bn_elemt(x, m, istd, w, b)
        sums, ubuf = _guarded(2 * c, torch.float64, -5.0)
        gw, gb = ops.sync_bn_backward_reduce(dy, x, m, istd, w, sums, True, True)
        dx = ops.sync_bn_backward_elemt(dy, x, m, istd, w, sums, cnt)
        torch.cuda.synchronize()
        assert _slack_ok(sbuf, per, -7.0) and _slack_ok(rmb, c, -3.0) and _slack_ok(rvb, c, -3.0) \
            and _slack_ok(ubuf, 2 * c, -5.0), 'a kernel wrote outside its output'
        assert y.stride() == x.stride() and dx.stride() == x.stride() and y.dtype == dtype and dx.dtype == dtype
        return dict(slot=slot.clone(), m=m, istd=istd, cnt=cnt, rm=rm.clone(), rv=rv.clone(), y=y, sums=sums.clone(),
                    gw=gw, gb=gb, dx=dx)

    r1, r2 = run(), run()
    for k in r1:
        assert torch.equal(r1[k].reshape(-1).view(torch.uint8), r2[k].reshape(-1).view(torch.uint8)), 'not reproducible: ' + k
    r = {k: v.cpu() for k, v in r1.items()}
    assert float(r['cnt'][0]) == n and float(r['slot'][0]) == n
    spread = var.sqrt()
    torch.testing.assert_close(r['slot'][1::3][:c], mean, rtol=0, atol=1e-6 * float((mean.abs() + spread).max()))
    torch.testing.assert_close(r['slot'][2::3][:c] / n, var, rtol=1e-4, atol=1e-6 * float((mean.abs() + spread).max()) ** 2 * 1e-3)
    torch.testing.assert_close(r['m'].double(), mean, rtol=1e-5, atol=1e-6 * float(spread.max()))
    torch.testing.assert_close(r['istd'].double(), invstd, rtol=1e-5, atol=0)
    _check(r['rm'], new_rm, rm0.double().abs() + mean.abs() + 1, wdt, 'running_mean')
    _check(r['rv'], new_rv, rv0.double().abs() + var + 1, wdt, 'running_var')

    shp = [1, -1] + [1] * (x.dim() - 2)
    xd = x.cpu().double()
    wd = w.cpu().double().view(shp)
    scale_y = ((xd.abs() + mean.abs().view(shp)) * invstd.view(shp) * wd.abs() + b.cpu().double().abs().view(shp))
    _check(r['y'], ys[0], scale_y, dtype, 'y')
    dims = [0] + list(range(2, x.dim()))
    dyd = dy.cpu().double()
    sum_abs_dy = dyd.abs().sum(dims)
    sum_abs_dyx = (dyd.abs() * (xd.abs() + mean.abs().view(shp))).sum(dims)
    _check(r['sums'][0::2], sdy, sum_abs_dy, torch.float32, 'sum_dy')
    _check(r['sums'][1::2], sdyx, sum_abs_dyx, torch.float32, 'sum_dy_xmu')
    _check(r['gb'], local[0][1], sum_abs_dy, wdt, 'grad_bias')
    _check(r['gw'], local[0][0], sum_abs_dyx * invstd, wdt, 'grad_weight')
    k = invstd ** 2 * sdyx / n
    scale_dx = (dyd.abs() + (sdy.abs() / n).view(shp) + (xd.abs() + mean.abs().view(shp)) * k.abs().view(shp)) \
        * (invstd.view(shp) * wd.abs())
    _check(r['dx'], dxs[0], scale_dx, dtype, 'dx')


@pytest.mark.gpu
@pytest.mark.parametrize('need_w,need_b', [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize('affine', [True, False])
def test_affine_and_needs_grad(affine, need_w, need_b):
    from horovod_b200 import ops
    gen = torch.Generator().manual_seed(3)
    x = _make((8, 16, 5, 5), 'cl4', torch.bfloat16, 0, 2.0, gen)
    dy = _make((8, 16, 5, 5), 'cl4', torch.bfloat16, 0, 0.0, gen)
    w = torch.rand(16, device='cuda') + 0.5 if affine else None
    b = torch.randn(16, device='cuda') if affine else None
    per = ops.sync_bn_slot_doubles(16)
    slot = torch.empty(per, dtype=torch.float64, device='cuda')
    ops.sync_bn_stats(x, slot)
    m, istd, cnt = ops.sync_bn_combine(slot.view(1, per), 16, EPS)
    y = ops.sync_bn_elemt(x, m, istd, w, b)
    sums = torch.empty(32, dtype=torch.float64, device='cuda')
    gw, gb = ops.sync_bn_backward_reduce(dy, x, m, istd, w, sums, need_w, need_b)
    dx = ops.sync_bn_backward_elemt(dy, x, m, istd, w, sums, cnt)
    ref = torch.nn.functional.batch_norm(x.double(), None, None, w.double() if affine else None,
                                         b.double() if affine else None, True, 0.0, EPS)
    assert (y.double() - ref).abs().max() < 0.05
    assert (gw is not None) == need_w and (gb is not None) == need_b
    xr = x.double().requires_grad_()
    wr = w.double().requires_grad_() if affine else None
    torch.nn.functional.batch_norm(xr, None, None, wr, b.double() if affine else None, True, 0.0, EPS).backward(dy.double())
    assert (dx.double() - xr.grad).abs().max() < 0.05 * float(xr.grad.abs().max())
    if need_w:
        torch.testing.assert_close(gw.double(), wr.grad if affine else (dy.double() * (x.double() - m.double().view(1, -1, 1, 1))).sum((0, 2, 3)) * istd.double(),
                                   rtol=1e-3, atol=1e-3)
    if need_b:
        torch.testing.assert_close(gb.double(), dy.double().sum((0, 2, 3)), rtol=1e-3, atol=1e-3)


@pytest.mark.gpu
def test_bad_arguments_are_rejected_before_launch():
    from horovod_b200 import ops
    x = torch.randn(4, 8, 3, 3, device='cuda')
    slot = torch.empty(ops.sync_bn_slot_doubles(8), dtype=torch.float64, device='cuda')
    with pytest.raises(RuntimeError, match='slot'):
        ops.sync_bn_stats(x, slot[:10])
    with pytest.raises(RuntimeError, match='channels-last'):
        ops.sync_bn_stats(x.transpose(2, 3), slot)
    with pytest.raises(RuntimeError, match='float32, bfloat16 or float16'):
        ops.sync_bn_stats(x.double(), slot)
    ops.sync_bn_stats(x, slot)
    m, istd, cnt = ops.sync_bn_combine(slot.view(1, -1), 8, EPS)
    with pytest.raises(RuntimeError, match='weight'):
        ops.sync_bn_elemt(x, m, istd, torch.ones(7, device='cuda'))
    with pytest.raises(RuntimeError, match='grad_output'):
        ops.sync_bn_backward_elemt(x.contiguous(memory_format=torch.channels_last), x, m, istd, None,
                                   torch.zeros(16, dtype=torch.float64, device='cuda'), cnt)


# ---- the exchange on simulated ranks --------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('nranks', [2, 4, 8])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_protocol_on_simulated_ranks(nranks, dtype):
    """Stats -> in-place allgather of the slots -> combine; backward reduce -> in-place allreduce -> elemt, with the real
    collective kernels on N simulated ranks: everything that the ranks share is bit-identical on every rank."""
    from horovod_b200 import ops
    from horovod_b200.ops import sim
    gen = torch.Generator().manual_seed(nranks)
    c = 24
    batches = [1] + [2 + 3 * r for r in range(1, nranks)]
    xs = [_make((bs, c, 6, 5), 'cl4', dtype, 0, 4.0, gen) for bs in batches]
    dys = [_make((bs, c, 6, 5), 'cl4', dtype, 0, 0.0, gen) for bs in batches]
    w = torch.rand(c, device='cuda') + 0.5
    b = torch.randn(c, device='cuda')
    rm0, rv0 = torch.randn(c), torch.rand(c) + 0.5
    per = ops.sync_bn_slot_doubles(c)
    regions = [torch.full((nranks * per,), float('nan'), dtype=torch.float64, device='cuda') for _ in range(nranks)]
    for r in range(nranks):
        ops.sync_bn_stats(xs[r], regions[r].view(nranks, per)[r])
    torch.cuda.synchronize()
    sim.inplace_allgather(regions)
    outs = []
    for r in range(nranks):
        rm, rv = rm0.cuda(), rv0.cuda()
        m, istd, cnt = ops.sync_bn_combine(regions[r].view(nranks, per), c, EPS, 0.1, rm, rv)
        outs.append((m, istd, cnt, rm, rv, ops.sync_bn_elemt(xs[r], m, istd, w, b)))
    sums = [torch.empty(2 * c, dtype=torch.float64, device='cuda') for _ in range(nranks)]
    for r in range(nranks):
        ops.sync_bn_backward_reduce(dys[r], xs[r], outs[r][0], outs[r][1], w, sums[r], True, True)
    torch.cuda.synchronize()
    sim.inplace_allreduce(sums, op=sim.SUM)
    dxs = [ops.sync_bn_backward_elemt(dys[r], xs[r], outs[r][0], outs[r][1], w, sums[r], outs[r][2]) for r in range(nranks)]
    torch.cuda.synchronize()
    for r in range(1, nranks):
        for k in range(5):
            assert torch.equal(outs[r][k], outs[0][k]), 'rank %d differs in %s' % (r, ['mean', 'invstd', 'count', 'rm', 'rv'][k])
        assert torch.equal(sums[r], sums[0]), 'rank %d differs in the reduced sums' % r

    ys, mean, var, invstd, n, new_rm, new_rv = _ref_forward([x.cpu() for x in xs], w.cpu(), b.cpu(), rm0, rv0, 0.1)
    rdx, sdy, sdyx, _ = _ref_backward([x.cpu() for x in xs], [d.cpu() for d in dys], w.cpu(), mean, invstd, n)
    assert float(outs[0][2][0]) == n
    torch.testing.assert_close(outs[0][0].cpu().double(), mean, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(outs[0][1].cpu().double(), invstd, rtol=1e-5, atol=0)
    torch.testing.assert_close(outs[0][3].cpu().double(), new_rm, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(outs[0][4].cpu().double(), new_rv, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(sums[0].cpu()[0::2], sdy, rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(sums[0].cpu()[1::2], sdyx, rtol=1e-4, atol=1e-3)
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    for r in range(nranks):
        torch.testing.assert_close(outs[r][5].cpu().double(), ys[r], rtol=tol, atol=tol * 10)
        torch.testing.assert_close(dxs[r].cpu().double(), rdx[r], rtol=tol, atol=tol * 10)


# ---- the module on one GPU, the peer a replica ----------------------------------------------------------------------
@pytest.fixture
def replica_world(monkeypatch):
    """SyncBatchNorm on 'two ranks' whose peer is a replica of this one: the slot allgather copies slot 0 to slot 1 and
    the sum allreduce doubles.  Both stand-ins are capturable torch ops on the current stream."""
    import horovod_b200.torch as hvd
    import horovod_b200.torch.sync_batch_norm as sbn
    hvd.init()
    torch.cuda.set_device(0)
    regions = {}

    def registered(nbytes, device):
        if regions.get(device) is None or regions[device].numel() < nbytes:
            assert not torch.cuda.is_current_stream_capturing()
            regions[device] = torch.zeros(max(nbytes, 4096), dtype=torch.uint8, device=device)
        return regions[device]

    def allgather(buf):
        half = buf.numel() // 2
        buf[half:].copy_(buf[:half])

    monkeypatch.setattr(sbn, '_native_world', lambda: (2, 0))
    monkeypatch.setattr(sbn, '_registered', registered)
    monkeypatch.setattr(sbn, '_allgather_slots', allgather)
    monkeypatch.setattr(sbn, '_allreduce_sums', lambda buf: buf.mul_(2))
    yield hvd
    hvd.shutdown()


def _twin_bn(c, momentum, dtype=torch.float32, affine=True):
    import horovod_b200.torch as hvd
    torch.manual_seed(0)
    ref = torch.nn.BatchNorm2d(c, momentum=momentum, affine=affine).cuda()
    if affine:
        with torch.no_grad():
            ref.weight.uniform_(0.5, 1.5)
            ref.bias.normal_()
    sync = hvd.SyncBatchNorm(c, momentum=momentum, affine=affine).cuda()
    sync.load_state_dict(ref.state_dict())
    return ref.to(dtype), sync.to(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize('momentum', [0.1, None])
def test_module_matches_batchnorm_on_the_doubled_batch(replica_world, momentum):
    ref, sync = _twin_bn(12, momentum)
    for step in range(3):
        x = (torch.randn(6, 12, 7, 5, device='cuda') * 2 + 3).contiguous(memory_format=torch.channels_last)
        xs = x.clone().requires_grad_()
        xr = x.clone().requires_grad_()
        dy = torch.randn_like(x)
        y = sync(xs)
        assert y.is_contiguous(memory_format=torch.channels_last)
        y.backward(dy)
        yr = ref(torch.cat([xr, xr]))
        yr.backward(torch.cat([dy, dy]))
        torch.testing.assert_close(y, yr[:6], rtol=1e-5, atol=1e-5)
        # xr feeds both halves of the doubled batch, so its gradient is twice one replica's dx; the local parameter
        # gradients are half of those over the doubled batch
        torch.testing.assert_close(xs.grad * 2, xr.grad, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(sync.weight.grad * 2, ref.weight.grad, rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(sync.bias.grad * 2, ref.bias.grad, rtol=1e-4, atol=1e-4)
        sync.weight.grad = sync.bias.grad = ref.weight.grad = ref.bias.grad = None
        torch.testing.assert_close(sync.running_mean, ref.running_mean, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(sync.running_var, ref.running_var, rtol=1e-5, atol=1e-6)
        assert int(sync.num_batches_tracked) == step + 1
    sync.eval()
    ref.eval()
    x = torch.randn(3, 12, 4, 4, device='cuda')
    torch.testing.assert_close(sync(x), ref(x))


def _conv_net(hvd):
    torch.manual_seed(1)
    net = torch.nn.Sequential(
        torch.nn.Conv2d(3, 16, 3, padding=1, bias=False), torch.nn.BatchNorm2d(16), torch.nn.ReLU(),
        torch.nn.Conv2d(16, 32, 3, padding=1, bias=False), torch.nn.BatchNorm2d(32, momentum=None), torch.nn.ReLU(),
        torch.nn.AdaptiveAvgPool2d(1), torch.nn.Flatten(), torch.nn.Linear(32, 5))
    net = hvd.SyncBatchNorm.convert_sync_batchnorm(net)
    return net.cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)


@pytest.mark.gpu
def test_convert_channels_last_bf16_net_without_host_sync(replica_world):
    hvd = replica_world
    plain = torch.nn.Sequential(torch.nn.Conv2d(3, 4, 1), torch.nn.BatchNorm2d(4, momentum=0.2)).cuda()
    plain[1].running_mean.fill_(0.5)
    conv = hvd.SyncBatchNorm.convert_sync_batchnorm(plain)
    assert isinstance(conv[1], hvd.SyncBatchNorm) and conv[1].momentum == 0.2
    assert torch.equal(conv[1].running_mean, torch.full((4,), 0.5, device='cuda'))
    net = _conv_net(hvd)
    assert sum(isinstance(m, hvd.SyncBatchNorm) for m in net.modules()) == 2
    x = torch.randn(8, 3, 12, 12, device='cuda').to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    net(x)  # sizes the registered region
    torch.cuda.synchronize()
    acts = []
    hook = net[1].register_forward_hook(lambda m, i, o: acts.append(o))
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = net(x)
        out.float().sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
        hook.remove()
    assert acts[0].is_contiguous(memory_format=torch.channels_last) and acts[0].dtype == torch.bfloat16
    assert torch.isfinite(out.float()).all()


@pytest.mark.gpu
def test_graphed_step_replays_bit_identical_to_eager(replica_world, monkeypatch):
    hvd = replica_world
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    xs = [torch.randn(8, 3, 12, 12, device='cuda').to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
          for _ in range(5)]
    ys = [torch.randint(0, 5, (8,), device='cuda') for _ in range(5)]

    def make():
        net = _conv_net(hvd)
        opt = hvd.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9),
                                       named_parameters=net.named_parameters(), fused=True)
        return net, opt

    def state(net):
        return [t.detach().clone() for t in list(net.parameters()) + list(net.buffers())]

    loss_fn = lambda net: (lambda x, y: torch.nn.functional.cross_entropy(net(x).float(), y))  # noqa: E731
    ge, oe = make()
    eager = hvd.GraphedStep(loss_fn(ge), oe, (xs[0], ys[0]), enabled=False)
    gg, og = make()
    graphed = hvd.GraphedStep(loss_fn(gg), og, (xs[0], ys[0]), warmup_iters=2)
    assert graphed.captured, graphed.fallback_reason
    # the warm-up ran forward passes that moved the BN buffers: start both from the same state
    with torch.no_grad():
        for a, b in zip(list(gg.parameters()) + list(gg.buffers()), list(ge.parameters()) + list(ge.buffers())):
            a.copy_(b)
    for x, y in zip(xs, ys):
        eager(x, y)
        graphed(x, y)
    torch.cuda.synchronize()
    assert graphed.replays == 5
    for a, b in zip(state(gg), state(ge)):
        assert torch.equal(a, b)
    assert int(gg[4].num_batches_tracked) == 5


# ---- real ranks -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_sync_bn_on_real_ranks():
    if torch.cuda.device_count() < 2:
        pytest.skip('needs at least 2 GPUs')
    from conftest import run_parallel
    n = min(torch.cuda.device_count(), 4)
    rc, out = run_parallel('sync_bn_worker.py', np=n, timeout=600)
    assert 'sync_bn_worker ok' in out, out[-3000:]
