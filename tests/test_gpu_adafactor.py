"""Fused Adafactor: the sm_90a kernels (ops.fused_adafactor_step) against an fp64 model of torch.optim.Adafactor's
update, the master-weight and EMA variants bit for bit against the plain kernels, determinism (run to run, per tensor,
CUDA graph replay, no host sync), and DistributedOptimizer(torch.optim.Adafactor(...), fused=True) against
torch.optim.Adafactor at world size 1, with masters, EMA, clipping, GradScaler, hvd.GraphedStep and checkpoints."""
import copy
import io

import pytest
import torch

from conftest import run_parallel
from optim_cases import (LOW, LOW_IDS, PAIR_IDS, PAIRS, SIZES, Slot, adafactor_ref, cat, f32, hvd, mlp,  # noqa: F401
                         mlp_loss, ngpu, same, ulp)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
HP = [dict(lr=1e-2, beta2_decay=-0.8, eps1=None, eps2=1e-3, d=1.0, weight_decay=0.0),
      dict(lr=0.05, beta2_decay=-0.5, eps1=1e-30, eps2=1e-3, d=0.5, weight_decay=0.1, grad_scale=0.5),
      dict(lr=1e-2, beta2_decay=-0.8, eps1=1e-3, eps2=1e-2, d=1.0, weight_decay=0.01)]
# 2-D and 3-D shapes around the warp (32 columns), the 64-row column chunk and the 4096-element tile, R or C of 1, and a
# channels_last 4-D tensor (its [batch, R, C] view has no single batch stride)
SHAPES = [(), (1, 5), (7, 1), (1, 1), (33, 31), (64, 65), (65, 64), (129, 4097), (3, 65, 70), (2, 3, 4, 5)]


def _fmt(shape):
    return torch.channels_last if len(shape) == 4 else torch.contiguous_format


def _case(shape, pdt, gdt, seed, offset=0, master=False, warm=False):
    """Parameter, gradient and state in guarded buffers; `warm`: positive state as a long run leaves it."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    rnd = lambda: torch.randn(shape, device='cuda', generator=g) * 0.1  # noqa: E731
    w = rnd()
    fmt = _fmt(shape)
    c = {'p': Slot(shape, pdt, offset, w.to(pdt), fmt), 'g': Slot(shape, gdt, offset + 1, rnd() * 10, fmt)}
    fill = (lambda s: torch.rand(s, device='cuda', generator=g) * 1e-2 + 1e-4) if warm else \
        (lambda s: torch.zeros(s, device='cuda'))
    if len(shape) >= 2:
        rs, cs = list(shape), list(shape)
        rs[-1], cs[-2] = 1, 1
        c['r'] = Slot(tuple(rs), torch.float32, offset + 2, fill(rs))
        c['c'] = Slot(tuple(cs), torch.float32, offset + 3, fill(cs))
    else:
        c['v'] = Slot(shape, torch.float32, offset + 2, fill(shape))
    if master:
        c['w'] = Slot(shape, torch.float32, offset + 1, w, fmt)
    return c


def _lists(cases):
    get = lambda c, k: c[k].t if k in c else None  # noqa: E731
    return ([c['p'].t for c in cases], [c['g'].t for c in cases], [get(c, 'r') for c in cases],
            [get(c, 'c') for c in cases], [get(c, 'v') for c in cases])


def _run(cases, hp, step, master=False, **kw):
    from horovod_b200 import ops
    hp = dict(hp)
    gs = hp.pop('grad_scale', 1.0)
    ops.fused_adafactor_step(*_lists(cases), step=step, grad_scale=gs,
                             master_params=[c['w'].t for c in cases] if master else None, **hp, **kw)


def _tol_rel(shape):
    """Relative error bound of the update alpha / denom * u.  v: a row sum of C squares in fp32 (C / 32 fmas per lane and a
    5-level tree), a column sum of 64-row chunks in fp32 added in fp64, the row mean in fp64, lerps (3 roundings each),
    the product and quotient (2): relative error below (C / 32 + 64 + 16) u; u = g * rsqrt(v) halves it and adds 3 u
    (scaling, the approximate rsqrt's 2 ulp).  alpha and denom: sums of squares as in LAMB (32 u), square roots, 6 more
    roundings.  Twice everything for the squares of u in ||u||."""
    C = shape[-1] if len(shape) >= 2 else 1
    e_u = ((C / 32 + 64 + 16) / 2 + 3) * U
    return 2 * e_u + 2 * (32 + 8) * U + e_u


def _check(cases, hp, step, before):
    pdt = cases[0]['p'].t.dtype
    for i, (c, b) in enumerate(zip(cases, before)):
        want = adafactor_ref(b, step=step, **hp)
        got = c['p'].t.double()
        tol = want['scale'] * _tol_rel(c['p'].t.shape) + want['p'].abs() * 2 * U + ulp(want['p'], torch.float32)
        if pdt != torch.float32:
            tol = tol + ulp(want['p'], pdt)
        err = (got - want['p']).abs()
        assert not bool((err > tol).any()), (i, tuple(c['p'].t.shape), float((err - tol).max()))
        for k in ('r', 'c', 'v'):
            if k in want:
                w = want[k]
                assert torch.allclose(c[k].t.double(), w, rtol=(c['p'].t.shape[-1] / 32 + 80) * U if k == 'r' else 80 * U,
                                      atol=1e-38), (i, k)
        for k, s in c.items():
            assert s.intact(), (i, 'wrote outside ' + k)


def _snapshot(cases):
    return [{k: type('S', (), {'t': s.t.clone()})() for k, s in c.items()} for c in cases]


@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("hp", range(len(HP)))
@pytest.mark.parametrize("step", [1, 1000])
def test_kernel_matches_fp64(hvd, pair, hp, step):
    """Vectors of every SIZES length, 0-dim, 2-D, 3-D and channels_last 4-D parameters in one launch; at step 1000 from a
    warm state (rho = 1 / sqrt(t) below lr), at step 1 from zeros; an explicit and a default eps1."""
    pdt, gdt = pair
    shapes = [(n,) for n in SIZES] + SHAPES
    cases = [_case(s, pdt, gdt, seed=i, warm=step > 1) for i, s in enumerate(shapes)]
    before = _snapshot(cases)
    _run(cases, HP[hp], step)
    torch.cuda.synchronize()
    _check(cases, HP[hp], step, before)


@pytest.mark.parametrize("pair", PAIRS, ids=PAIR_IDS)
@pytest.mark.parametrize("offset", [1, 2, 3])
def test_kernel_unaligned_views(hvd, pair, offset):
    pdt, gdt = pair
    cases = [_case(s, pdt, gdt, seed=i, offset=offset, warm=True) for i, s in enumerate([(4097,), (33, 31), (2, 3, 4, 5)])]
    before = _snapshot(cases)
    _run(cases, HP[1], 7)
    torch.cuda.synchronize()
    _check(cases, HP[1], 7, before)


def test_grad_scale_dev(hvd):
    """A device factor of 1 is bit-identical to none; a factor of 4 equals gradients scaled by 4, in every phase."""
    def run(gscale=1.0, **kw):
        cases = [_case(s, torch.float32, torch.float32, seed=i, warm=True) for i, s in enumerate([(4097,), (65, 70)])]
        for c in cases:
            c['g'].t.mul_(gscale)
        _run(cases, HP[0], 3, **kw)
        return [s.t for c in cases for k, s in c.items() if k != 'g']
    plain, one = run(), run(grad_scale_dev=torch.ones(1, device='cuda'))
    scaled, dev = run(gscale=4.0), run(grad_scale_dev=torch.tensor([4.0], device='cuda'))
    assert all(same(a, b) for a, b in zip(plain, one))
    assert all(same(a, b) for a, b in zip(scaled, dev))
    assert not all(same(a, b) for a, b in zip(plain, scaled))


@pytest.mark.parametrize("pdt", LOW, ids=LOW_IDS)
def test_master_kernels_equal_fp32_kernels(hvd, pdt):
    """With masters and an explicit eps1: masters and state bit-identical to the fp32-parameter kernels started from the
    masters; parameters are the rounded masters."""
    shapes = [(4097,), (1,), (33, 31), (3, 65, 70), (2, 3, 4, 5)]
    cases = [_case(s, pdt, pdt, seed=i, master=True, warm=True) for i, s in enumerate(shapes)]
    ref = []
    for c in cases:
        r = {'p': Slot(c['w'].t.shape, torch.float32, 0, c['w'].t, _fmt(c['w'].t.shape)),
             'g': Slot(c['g'].t.shape, torch.float32, 0, c['g'].t.float(), _fmt(c['g'].t.shape))}
        for k in ('r', 'c', 'v'):
            if k in c:
                r[k] = Slot(c[k].t.shape, torch.float32, 0, c[k].t)
        ref.append(r)
    hp = dict(HP[2])
    for step in (1, 2, 3):
        _run(cases, hp, step, master=True)
        _run(ref, hp, step)
    torch.cuda.synchronize()
    for i, (c, r) in enumerate(zip(cases, ref)):
        assert same(c['w'].t, r['p'].t), (i, 'master')
        assert same(c['p'].t, r['p'].t.to(pdt)), (i, 'param is not the rounded master')
        for k in ('r', 'c', 'v'):
            if k in c:
                assert same(c[k].t, r[k].t), (i, k)


@pytest.mark.parametrize("master", [False, True], ids=['plain', 'master'])
def test_ema_epilogue_changes_nothing_else(hvd, master):
    from horovod_b200 import ops
    pdt = torch.bfloat16 if master else torch.float32
    shapes = [(4097,), (33, 31), (2, 3, 4, 5)]
    runs = []
    for ema in (False, True):
        cases = [_case(s, pdt, pdt, seed=i, master=master, warm=True) for i, s in enumerate(shapes)]
        emas = [torch.empty_like(c['p'].t, dtype=torch.float32) for c in cases]
        for step in (1, 2):
            kw = dict(ema_params=emas, ema_decay=0.9, ema_start=step == 1) if ema else {}
            ops.fused_adafactor_step(*_lists(cases), step=step, master_params=[c['w'].t for c in cases] if master else None,
                                     **HP[2], **kw)
        runs.append((cases, emas))
    (a, _), (b, emas) = runs
    for ca, cb in zip(a, b):
        for k in ca:
            assert same(ca[k].t, cb[k].t), k
    # the EMA of the two updates: e = x1, then e += (1 - d) * (x2 - x1), with x the master or the stored parameter
    assert all(bool(torch.isfinite(e).all()) for e in emas)


def test_determinism_per_tensor_graph_and_no_sync(hvd):
    from horovod_b200 import ops
    shapes = [((1 << 20) + 3,), (3,), (), (300, 130), (3, 65, 70), (2, 3, 4, 5), (4097, 1)]

    def fresh():
        return [_case(s, torch.float32, torch.float32, seed=i, warm=True) for i, s in enumerate(shapes)]

    def state(cases):
        return [s.t.clone() for c in cases for s in c.values()]

    a, b = fresh(), fresh()
    torch.cuda.set_sync_debug_mode('error')
    try:
        _run(a, HP[1], 5)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    _run(b, HP[1], 5)
    assert all(same(x, y) for x, y in zip(state(a), state(b))), 'two runs differ'
    one = fresh()
    for c in one:
        _run([c], HP[1], 5)
    assert all(same(x, y) for x, y in zip(state(a), state(one))), 'a tensor depends on its neighbours'
    g = fresh()
    lists = _lists(g)
    gsd = torch.ones(1, device='cuda')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm up the allocator outside the capture
        snap = state(g)
        ops.fused_adafactor_step(*lists, step=5, grad_scale_dev=gsd, **{k: v for k, v in HP[1].items() if k != 'grad_scale'},
                                 grad_scale=0.5)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.fused_adafactor_step(*lists, step=5, grad_scale_dev=gsd, **{k: v for k, v in HP[1].items() if k != 'grad_scale'},
                                 grad_scale=0.5)
    for t, v in zip([s_.t for c in g for s_ in c.values()], snap):
        t.copy_(v)
    graph.replay()
    torch.cuda.synchronize()
    assert all(same(x, y) for x, y in zip(state(a), state(g))), 'graph replay differs from the eager call'


def test_rejects_bad_arguments(hvd):
    from horovod_b200 import ops
    c = [_case((5,), torch.float32, torch.float32, 0), _case((4, 6), torch.float32, torch.float32, 1)]
    p, g, r, col, v = _lists(c)
    hp = dict(lr=1e-2, beta2_decay=-0.8, eps1=None, eps2=1e-3, d=1.0, weight_decay=0.0, step=1)
    snap = [t.clone() for t in p]
    bad = [((p, g, r[:1], col, v), 'list sizes'),
           ((p, [g[0], g[1].double()], r, col, v), 'grads'),
           ((p, g, [None, None], col, v), 'missing'),
           ((p, g, r, [None, torch.zeros(1, 5, device='cuda')], v), 'size'),
           ((p, g, [torch.zeros(5, device='cuda'), r[1]], col, v), 'given'),
           ((p, g, r, col, [v[0], torch.zeros(4, 6, device='cuda')]), 'given'),
           ((p, g, r, [None, torch.zeros(1, 12, device='cuda')[:, ::2]], v), 'contiguous'),
           ((p, g, r, col, [v[0].double(), None]), 'variances'),
           (([p[0], torch.zeros(1, 1, 1, 1, 2, 3, device='cuda')], [g[0], torch.zeros(1, 1, 1, 1, 2, 3, device='cuda')],
             [None, torch.zeros(1, 1, 1, 1, 2, 1, device='cuda')], [None, torch.zeros(1, 1, 1, 1, 1, 3, device='cuda')],
             [v[0], None]), 'dims')]
    for args, match in bad:
        with pytest.raises(RuntimeError, match=match):
            ops.fused_adafactor_step(*args, **hp)
    with pytest.raises(RuntimeError, match='CUDA'):
        ops.fused_adafactor_step([p[0].cpu()], [g[0].cpu()], [None], [None], [v[0].cpu()], **hp)
    torch.cuda.synchronize()
    assert all(same(a, b) for a, b in zip(p, snap)), 'a rejected call wrote a parameter'


# ---- DistributedOptimizer at world size 1 -----------------------------------------------------------------------------------
class ConvNet(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3, padding=1)
        self.conv2 = torch.nn.Conv2d(8, 8, 3, padding=1)
        self.fc = torch.nn.Linear(8, 4)

    def forward(self, x):
        return self.fc(torch.relu(self.conv2(torch.relu(self.conv(x)))).mean((2, 3)))


def _adafactor(params, **kw):
    return torch.optim.Adafactor(params, lr=kw.pop('lr', 1e-2), weight_decay=kw.pop('weight_decay', 1e-2), **kw)


def _conv_batch(step):
    g = torch.Generator(device='cuda').manual_seed(step)
    return torch.randn(4, 3, 8, 8, device='cuda', generator=g).contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("model", ['mlp', 'conv'])
def test_fused_optimizer_follows_torch_adafactor(hvd, model, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    torch.manual_seed(0)
    m = mlp(torch.float32) if model == 'mlp' else ConvNet().cuda().to(memory_format=torch.channels_last)
    ref = copy.deepcopy(m)
    opt = hvd.DistributedOptimizer(_adafactor(m.parameters()), named_parameters=m.named_parameters(), fused=True)
    ropt = _adafactor(ref.parameters())
    loss = (lambda mod, s: mlp_loss(mod, s, torch.float32)) if model == 'mlp' else \
        (lambda mod, s: mod(_conv_batch(s)).square().mean())
    peak = 0
    for s in range(20):
        for mod, o in ((m, opt), (ref, ropt)):
            o.zero_grad()
            loss(mod, s).backward()
        for p, q in zip(m.parameters(), ref.parameters()):
            q.grad.copy_(p.grad)  # the same gradients: only the updates differ
        opt.synchronize()
        torch.cuda.synchronize()
        resident = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        with opt.skip_synchronize():
            opt.step()
        torch.cuda.synchronize()
        peak = max(peak, torch.cuda.max_memory_allocated() - resident) if s else 0  # step 1 creates the state
        ropt.step()
    n = sum(p.numel() for p in m.parameters())
    # scratch: 2 norm floats and one table entry (~150 B) per tensor, column partials and CTA partials (<= numel / 64
    # and numel / 4096 floats), each rounded to the allocator's 512 B blocks
    bound = 512 * (4 + 2 * len(list(m.parameters()))) + 4 * n // 32
    assert peak <= bound, (peak, bound)
    for (name, p), q in zip(m.named_parameters(), ref.parameters()):
        assert torch.allclose(p, q, rtol=1e-4, atol=1e-6), (name, float((p - q).abs().max()))
        st, rst = opt.state[p], ropt.state[q]
        assert float(st['step']) == float(rst['step']) == 20
        for k in ('row_var', 'col_var', 'variance'):
            assert (k in st) == (k in rst), k
            if k in st:
                assert st[k].shape == rst[k].shape and torch.allclose(st[k], rst[k], rtol=1e-4, atol=1e-12), (name, k)


def test_bf16_master_weights_follow_fp32_twin(hvd):
    dt = torch.bfloat16
    m = mlp(dt)
    twin = copy.deepcopy(m).float()
    opt = hvd.DistributedOptimizer(_adafactor(m.parameters(), eps=(1e-30, 1e-3)), named_parameters=m.named_parameters(),
                                   master_weights=True)
    topt = hvd.DistributedOptimizer(_adafactor(twin.parameters(), eps=(1e-30, 1e-3)),
                                    named_parameters=twin.named_parameters(), fused=True)
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


def test_ema_clipping_and_grad_scaler(hvd):
    """ema_decay with a mid-run change against an fp64 EMA of the parameters; clip_grad_norm_ and a GradScaler-skipped
    step (an inf gradient): the skipped step leaves parameters, state and EMA untouched."""
    torch.manual_seed(0)
    m = mlp(torch.float32)
    opt = hvd.DistributedOptimizer(_adafactor(m.parameters()), named_parameters=m.named_parameters(), ema_decay=0.9)
    scaler = torch.amp.GradScaler('cuda', init_scale=128.0)
    ema = None
    for s in range(8):
        if s == 4:
            opt.param_groups[0]['ema_decay'] = 0.5
        opt.zero_grad()
        scaler.scale(mlp_loss(m, s, torch.float32)).backward()
        opt.synchronize()
        if s == 5:
            next(m.parameters()).grad.view(-1)[0] = float('inf')
        scaler.unscale_(opt)
        opt.clip_grad_norm_(0.1)
        snap = [p.detach().clone() for p in m.parameters()]
        with opt.skip_synchronize():
            scaler.step(opt)
        scaler.update()
        if s == 5:
            assert all(same(a, p.detach()) for a, p in zip(snap, m.parameters())), 'skipped step wrote a parameter'
            continue
        d = 0.9 if s < 4 else 0.5
        x = [p.detach().double() for p in m.parameters()]
        ema = x if ema is None else [e + (1 - d) * (xi - e) for e, xi in zip(ema, x)]
    for p, e in zip(m.parameters(), ema):
        assert torch.allclose(opt.state[p]['ema_param'].double(), e, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("k", [1, 4])
def test_graphed_step_replays_equal_eager_fused_steps(hvd, monkeypatch, k):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    dt = torch.bfloat16 if k == 4 else torch.float32
    runs = []
    for graphed in (False, True):
        m = mlp(dt)
        opt = hvd.DistributedOptimizer(_adafactor(m.parameters()), named_parameters=m.named_parameters(), fused=True,
                                       backward_passes_per_step=k,
                                       grad_accumulation_dtype=torch.float32 if k > 1 else None)
        g = torch.Generator(device='cuda').manual_seed(2)
        xs = [torch.randn(16, 24, device='cuda', generator=g).to(dt) for _ in range(6 * k)]
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
        runs.append((m, opt))
    (a, oa), (b, ob) = runs
    for (name, p), q in zip(a.named_parameters(), b.parameters()):
        assert same(p.detach(), q.detach()), name


def test_checkpoints_both_ways_with_torch_adafactor(hvd):
    dt = torch.float32
    m = mlp(dt)
    opt = hvd.DistributedOptimizer(_adafactor(m.parameters()), named_parameters=m.named_parameters(), fused=True)
    for s in range(3):
        opt.zero_grad()
        mlp_loss(m, s, dt).backward()
        opt.step()
    f = io.BytesIO()
    torch.save({'model': m.state_dict(), 'opt': opt.state_dict()}, f)
    f.seek(0)
    ck = torch.load(f)
    t = mlp(dt)
    t.load_state_dict(ck['model'])
    topt = _adafactor(t.parameters())
    topt.load_state_dict(ck['opt'])  # fused -> torch
    for s in range(3, 5):
        topt.zero_grad()
        mlp_loss(t, s, dt).backward()
        topt.step()
    f = io.BytesIO()
    torch.save({'model': t.state_dict(), 'opt': topt.state_dict()}, f)
    f.seek(0)
    ck = torch.load(f)
    b = mlp(dt)
    b.load_state_dict(ck['model'])
    bopt = hvd.DistributedOptimizer(_adafactor(b.parameters()), named_parameters=b.named_parameters(), fused=True)
    bopt.load_state_dict(ck['opt'])  # torch -> fused
    for s in range(5, 7):
        bopt.zero_grad()
        mlp_loss(b, s, dt).backward()
        bopt.step()
    for p in b.parameters():
        assert float(bopt.state[p]['step']) == 7
        assert torch.isfinite(p).all()


def test_broadcast_optimizer_state_then_fused_step(hvd):
    dt = torch.bfloat16
    m = mlp(dt)
    opt = hvd.DistributedOptimizer(_adafactor(m.parameters()), named_parameters=m.named_parameters(), fused=True)
    hvd.broadcast_optimizer_state(opt, root_rank=0)
    opt.zero_grad()
    mlp_loss(m, 0, dt).backward()
    opt.step()
    for p in m.parameters():
        st = opt.state[p]
        assert all(st[k].dtype == torch.float32 for k in ('row_var', 'col_var', 'variance') if k in st)
        assert torch.isfinite(p).all()


def test_optimizer_argument_errors(hvd):
    m = mlp(torch.float32)
    with pytest.raises(ValueError, match='maximize'):
        hvd.DistributedOptimizer(_adafactor(m.parameters(), maximize=True), named_parameters=m.named_parameters(),
                                 master_weights=True)
    with pytest.raises(ValueError, match='Adasum'):
        hvd.DistributedOptimizer(_adafactor(m.parameters()), named_parameters=m.named_parameters(), ema_decay=0.9,
                                 op=hvd.Adasum)
    p = torch.nn.Parameter(torch.zeros(1, 1, 1, 1, 2, 3, device='cuda'))
    opt = hvd.DistributedOptimizer(_adafactor([p]), fused=True, ema_decay=0.9)
    p.grad = torch.ones_like(p)
    with pytest.raises(RuntimeError, match='dims'):
        opt.step()
    from horovod_b200.torch.sharded_optimizer import _ShardedDistributedOptimizer
    cls = type('Adafactor', (_ShardedDistributedOptimizer, torch.optim.Adafactor), {})
    with pytest.raises(ValueError, match='Adafactor'):
        cls(_adafactor(m.parameters()).param_groups, list(m.named_parameters()), hvd.Compression.none)


@pytest.mark.skipif(ngpu() < 2, reason="needs >= 2 GPUs")
def test_fused_adafactor_across_ranks(native_built):
    rc, out = run_parallel("adafactor_worker.py", np=2, timeout=420)
    assert "adafactor_worker OK" in out, out[-4000:]
