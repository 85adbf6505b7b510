"""Global-norm gradient clipping and AMP loss scaling in hvd.GraphedStep: the statistics kernel on ragged per-parameter
gradient lists against fp64, the unsharded optimizer's clip_grad_norm_ against torch.nn.utils.clip_grad_norm_ and
torch's optimizers, GraphedStep with max_grad_norm (and a GradScaler) against the eager loop bit for bit at world size
1, and the sharded (ZeRO-1) optimizer with ShardedGradScaler and clipping in GraphedStep on 4 simulated ranks."""
import copy
import math

import pytest
import torch

from conftest import run_parallel
from optim_cases import Slot, hvd, make_optimizer, mlp, ngpu, same  # noqa: F401  (hvd: fixture)
from sim_ranks import ConvNet, gteam, micro_batch, sharded_team, zero_copy_buckets  # noqa: F401  (gteam: fixture)

pytestmark = pytest.mark.gpu


# ---- the statistics kernel on per-parameter gradients ---------------------------------------------------------------------
RAGGED = [1, 3, 4095, 4096, 4097, 12289, 31 * 1024 * 1024 + 5, 1024, 77]


def _ragged(dtype, seed):
    """Sizes from 1 element to 31 M plus 60 small ones, each at its own unaligned element offset of a larger buffer."""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    sizes = RAGGED + [int(x) for x in torch.randint(1, 3000, (60,), generator=torch.Generator().manual_seed(seed))]
    return [Slot((n,), dtype, i % 5, torch.randn(n, device='cuda', generator=gen) * (1 + i % 7), slack=3)
            for i, n in enumerate(sizes)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=['fp32', 'bf16', 'fp16'])
def test_stats_kernel_on_ragged_gradients(hvd, dtype):
    from horovod_b200 import ops
    slots = _ragged(dtype, 3)
    views = [s.t for s in slots]
    want_sq = sum(float(v.double().square().sum()) for v in views)
    want_max = max(float(v.double().abs().max()) for v in views)
    for norm_type, want in ((2.0, want_sq), (math.inf, want_max)):
        outs = []
        for _ in range(2):
            out = torch.zeros(2, device='cuda')
            before = ops.kernel_launches()
            torch.cuda.set_sync_debug_mode('error')
            try:
                ops.grad_shard_stats(views, out, norm_type=norm_type)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            assert ops.kernel_launches() - before == 1, 'one launch per gradient dtype'
            outs.append(out)
        assert same(outs[0], outs[1]), 'the same input gives the same bits'
        assert abs(float(outs[0][0]) - want) <= 1e-5 * want, (norm_type, float(outs[0][0]), want)
        assert float(outs[0][1]) == 0.0
    # in-place unscale of a mixed-dtype list: one launch per dtype, the statistics of the stored values
    mixed = views[:5] + [s.t for s in _ragged(torch.float32 if dtype != torch.float32 else torch.bfloat16, 4)[:5]]
    inv = torch.full((1,), 0.25, device='cuda')
    want = [(v.float() * 0.25).to(v.dtype) for v in mixed]
    out = torch.zeros(2, device='cuda')
    before = ops.kernel_launches()
    ops.grad_shard_stats(mixed, out, inv_scale=inv)
    assert ops.kernel_launches() - before == 2
    assert all(same(v, w) for v, w in zip(mixed, want))
    ref = sum(float(w.double().square().sum()) for w in want)
    assert abs(float(out[0]) - ref) <= 1e-5 * ref
    for s in slots:
        assert same(s._slack(), s.slack), 'the kernel wrote outside a tensor'


def test_stats_kernel_flags_non_finite_in_a_large_tensor(hvd):
    from horovod_b200 import ops
    g = [torch.ones(n, device='cuda') for n in (5, 31 * 1024 * 1024, 4097)]
    g[1][-1] = float('nan')
    out = torch.zeros(2, device='cuda')
    ops.grad_shard_stats(g, out)
    assert float(out[1]) == 1.0 and math.isnan(float(out[0]))


# ---- the unsharded optimizer's clip_grad_norm_ ------------------------------------------------------------------------------
def _xs(n, dt, seed=2):
    gen = torch.Generator(device='cuda').manual_seed(seed)
    return [torch.randn(16, 24, device='cuda', generator=gen).to(dt) for _ in range(n)]


KINDS = ['sgd', 'adamw', 'lamb', 'lars']


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=['fp32', 'bf16-masters'])
@pytest.mark.parametrize("buckets", [False, True], ids=['per-param', 'buckets'])
def test_unsharded_clip_matches_torch(hvd, monkeypatch, kind, dt, buckets):
    """The norm against fp64, and the parameters after several clipped steps against torch's clip + torch's optimizer
    on an fp32 copy fed the same gradients."""
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    if buckets:
        zero_copy_buckets(monkeypatch)
    m = mlp(dt)
    ref = copy.deepcopy(m).float()
    opt = hvd.DistributedOptimizer(make_optimizer(hvd, kind, m.parameters()), named_parameters=m.named_parameters(), fused=True,
                                   master_weights=dt != torch.float32)
    assert bool(opt._buckets) == buckets
    ropt = make_optimizer(hvd, kind, ref.parameters())
    tol = dict(rtol=1e-5, atol=1e-6) if dt == torch.float32 else dict(rtol=1e-2, atol=2e-3)
    for i, x in enumerate(_xs(5, dt)):
        opt.zero_grad()
        m(x).float().square().mean().backward()
        grads = [p.grad.detach().double() for p in m.parameters()]
        want = math.sqrt(sum(float(g.square().sum()) for g in grads))
        max_norm = want * (0.3 if i % 2 == 0 else 3.0)
        norm = opt.clip_grad_norm_(max_norm)
        assert norm.dim() == 0 and norm.dtype == torch.float32 and norm.is_cuda
        assert abs(float(norm) - want) <= 1e-5 * want
        opt.step()
        for p, q in zip(ref.parameters(), m.parameters()):
            p.grad = q.grad.detach().float().clone()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
        ropt.step()
        for (name, a), b in zip(m.named_parameters(), ref.parameters()):
            torch.testing.assert_close(a.detach().float(), b.detach(), **tol, msg=lambda s: '%s step %d: %s' % (name, i, s))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=['fp32', 'bf16-masters'])
def test_clip_below_max_norm_is_bit_identical_to_no_clip(hvd, monkeypatch, kind, dt):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    runs = []
    for clip in (False, True):
        m = mlp(dt)
        opt = hvd.DistributedOptimizer(make_optimizer(hvd, kind, m.parameters()), named_parameters=m.named_parameters(),
                                       fused=True, master_weights=dt != torch.float32)
        for x in _xs(3, dt):
            opt.zero_grad()
            m(x).float().square().mean().backward()
            if clip:
                assert float(opt.clip_grad_norm_(1e9)) < 1e9
            opt.step()
        runs.append(m)
    for a, b in zip(*[r.parameters() for r in runs]):
        assert same(a.detach(), b.detach())


def test_unfused_clip_scales_grad_in_place(hvd):
    m = mlp(torch.float32)
    ref = copy.deepcopy(m)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9),
                                   named_parameters=m.named_parameters(), fused=False)
    x = _xs(1, torch.float32)[0]
    m(x).square().mean().backward()
    ref(x).square().mean().backward()
    norm = opt.clip_grad_norm_(0.01)
    want = torch.nn.utils.clip_grad_norm_(ref.parameters(), 0.01)
    torch.testing.assert_close(norm, want, rtol=1e-6, atol=0)
    assert float(norm) > 0.01
    for p, q in zip(m.parameters(), ref.parameters()):
        torch.testing.assert_close(p.grad, q.grad, rtol=1e-6, atol=1e-9)
    assert opt._clip_coef is None
    opt.step()


def test_clip_rejects_sparse_and_bad_norm_type(hvd):
    emb = torch.nn.Embedding(10, 4, sparse=True).cuda()
    opt = hvd.DistributedOptimizer(torch.optim.SGD(emb.parameters(), lr=0.1), named_parameters=emb.named_parameters())
    with pytest.raises(ValueError, match='norm_type'):
        opt.clip_grad_norm_(1.0, norm_type=1.0)
    emb(torch.tensor([1, 2], device='cuda')).sum().backward()
    with pytest.raises(ValueError, match='sparse'):
        opt.clip_grad_norm_(1.0)


# ---- GraphedStep against the eager loop at world size 1 -------------------------------------------------------------------
CASES = [('sgd', torch.float32, False), ('adamw', torch.float32, False), ('lamb', torch.float32, False),
         ('lars', torch.float32, False), ('sgd', torch.bfloat16, True), ('adamw', torch.bfloat16, True),
         ('lamb', torch.bfloat16, True), ('lars', torch.bfloat16, True)]
CASE_IDS = ['sgd', 'adamw', 'lamb', 'lars', 'sgd-bf16', 'adamw-bf16', 'lamb-bf16', 'lars-bf16']
MAX_NORM = 0.02  # below the model's gradient norm: every step clips


def _opt(hvd, kind, m, dt, k, acc):
    return hvd.DistributedOptimizer(make_optimizer(hvd, kind, m.parameters()), named_parameters=m.named_parameters(), fused=True,
                                    master_weights=dt != torch.float32, backward_passes_per_step=k,
                                    grad_accumulation_dtype=torch.float32 if acc and k > 1 else None)


def _clip_run(hvd, kind, dt, acc, k, mode, steps=3):
    """mode 'eager': the documented loop; 'graphed': GraphedStep(max_grad_norm); 'disabled': its eager fallback."""
    m = mlp(dt)
    opt = _opt(hvd, kind, m, dt, k, acc)
    xs = _xs(steps * k, dt)
    fn = lambda x: m(x).float().square().mean() / k  # noqa: E731
    norms = []
    orig = opt.clip_grad_norm_
    opt.clip_grad_norm_ = lambda *a, **kw: norms.append(orig(*a, **kw).clone()) or norms[-1]
    if mode == 'eager':
        for i, x in enumerate(xs):
            if i % k == 0:
                opt.zero_grad(set_to_none=False)
            fn(x).backward()
            if i % k == k - 1:
                opt.synchronize()
                opt.clip_grad_norm_(MAX_NORM)
                with opt.skip_synchronize():
                    opt.step()
    else:
        step = hvd.GraphedStep(fn, opt, (xs[0],), enabled=mode == 'graphed', max_grad_norm=MAX_NORM)
        assert step.captured == (mode == 'graphed'), step.fallback_reason
        for x in xs:
            step(x)
    torch.cuda.synchronize()
    assert len(norms) == steps and all(float(n) > MAX_NORM for n in norms)
    return m, opt, norms


@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_graphed_clip_equals_eager_loop(hvd, monkeypatch, k, case):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    kind, dt, acc = case
    runs = [_clip_run(hvd, kind, dt, acc, k, mode) for mode in ('eager', 'graphed', 'disabled')]
    (a, oa, na) = runs[0]
    for b, ob, nb in runs[1:]:
        assert all(same(x, y) for x, y in zip(na, nb))
        for (name, p), q in zip(a.named_parameters(), b.parameters()):
            assert same(p.detach(), q.detach()), name
            for key in oa.state[p]:
                if torch.is_tensor(oa.state[p][key]) and oa.state[p][key].is_cuda:
                    assert same(oa.state[p][key], ob.state[q][key]), (name, key)


def test_graphed_clip_does_not_sync_with_the_host(hvd, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    m = mlp(torch.float32)
    opt = _opt(hvd, 'adamw', m, torch.float32, 1, False)
    xs = _xs(3, torch.float32)
    step = hvd.GraphedStep(lambda x: m(x).square().mean(), opt, (xs[0],), max_grad_norm=MAX_NORM)
    assert step.captured, step.fallback_reason
    step(xs[0])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for x in xs[1:]:
            step(x)
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ---- fp16 autocast + GradScaler ----------------------------------------------------------------------------------------------
def _amp_run(hvd, kind, graphed, overflow_step=1, steps=4):
    m = mlp(torch.float32)
    opt = _opt(hvd, kind, m, torch.float32, 1, False)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 12)
    xs = _xs(steps, torch.float32)
    xs[overflow_step] = xs[overflow_step] * 1e5  # beyond fp16's range in the autocast matmul: inf gradients

    def fn(x):
        with torch.autocast('cuda', dtype=torch.float16):
            return m(x).float().square().mean()
    record = []
    if graphed:
        step = hvd.GraphedStep(fn, opt, (xs[0],), max_grad_norm=MAX_NORM, scaler=scaler)
        assert step.captured, step.fallback_reason
    for i, x in enumerate(xs):
        before = [p.detach().clone() for p in m.parameters()]
        if graphed:
            loss = step(x).detach().clone()
        else:
            opt.zero_grad()
            loss = fn(x)
            scaler.scale(loss).backward()
            opt.synchronize()
            scaler.unscale_(opt)
            opt.clip_grad_norm_(MAX_NORM)
            with opt.skip_synchronize():
                scaler.step(opt)
            scaler.update()
        torch.cuda.synchronize()
        record.append((loss, scaler.get_scale(), [p.detach().clone() for p in m.parameters()], before,
                       {k: v.clone() for k, v in opt.state[next(iter(m.parameters()))].items() if torch.is_tensor(v)}))
        if graphed:
            assert opt._clip_coef is None and not opt._reduced, 'a skipped step left its clip state behind'
    return record


@pytest.mark.parametrize("kind", KINDS)
def test_graphed_grad_scaler_equals_eager(hvd, monkeypatch, kind):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    eager, graphed = _amp_run(hvd, kind, False), _amp_run(hvd, kind, True)
    for i, (e, g) in enumerate(zip(eager, graphed)):
        assert same(e[0], g[0]) and e[1] == g[1], i
        assert all(same(a, b) for a, b in zip(e[2], g[2])), i
        assert e[4].keys() == g[4].keys() and all(same(e[4][k], g[4][k]) for k in e[4]), i
    skipped = graphed[1]
    assert skipped[1] == graphed[0][1] / 2, 'the scale backs off on the overflowing step'
    assert all(same(a, b) for a, b in zip(skipped[2], skipped[3])), 'the skipped step leaves the parameters alone'
    assert graphed[1][4].keys() == graphed[0][4].keys() and all(same(graphed[0][4][k], graphed[1][4][k]) for k in graphed[0][4])
    assert not all(same(a, b) for a, b in zip(graphed[2][2], graphed[2][3])), 'the step after it updates'


# ---- sharded (ZeRO-1) on 4 simulated ranks -----------------------------------------------------------------------------------
def _sharded_run(hvd, team, kind, k, graphed, steps=3):
    n = team.n
    torch.manual_seed(0)
    base = ConvNet().cuda().to(memory_format=torch.channels_last)
    models, opts = sharded_team(hvd, team, base, lambda m: make_optimizer(hvd, kind, m.parameters()), min_buckets=2,
                                backward_passes_per_step=k)
    scalers = [hvd.ShardedGradScaler('cuda', init_scale=256.0) for _ in range(n)]
    fns = [lambda x, y, m=m: torch.nn.functional.cross_entropy(m(x), y) / k for m in models]
    norms = [[] for _ in range(n)]
    for r, o in enumerate(opts):
        orig = o.clip_grad_norm_
        o.clip_grad_norm_ = lambda *a, orig=orig, r=r, **kw: norms[r].append(orig(*a, **kw).clone()) or norms[r][-1]
    if graphed:
        gsteps = [hvd.GraphedStep(fns[r], opts[r], micro_batch(0, 0, r, torch.float32), max_grad_norm=0.05, scaler=scalers[r])
                  for r in range(n)]
        assert all(g.captured and g.comm_in_graph for g in gsteps), gsteps[0].fallback_reason
        for r, o in enumerate(opts):  # the captured reduce-scatters run once every rank replayed its last graph
            orig = o.synchronize
            o.synchronize = lambda *a, orig=orig, **kw: (team.before_step(), orig(*a, **kw))[1]
    for step in range(steps):
        if graphed:
            for j in range(k - 1):
                for r in range(n):
                    gsteps[r](*micro_batch(step, j, r, torch.float32))
            team.run(lambda r: gsteps[r](*micro_batch(step, k - 1, r, torch.float32)))
        else:
            for r in range(n):
                opts[r].zero_grad()
                for j in range(k):
                    scalers[r].scale(fns[r](*micro_batch(step, j, r, torch.float32))).backward()
            team.flush()

            def update(r):
                opts[r].synchronize()
                scalers[r].unscale_(opts[r])
                opts[r].clip_grad_norm_(0.05)
                with opts[r].skip_synchronize():
                    scalers[r].step(opts[r])
                scalers[r].update()
            team.run(update)
        for r in range(1, n):
            assert same(norms[r][-1], norms[0][-1]), 'the norm differs between ranks'
            for a, b in zip(models[r].parameters(), models[0].parameters()):
                assert same(a.detach(), b.detach()), 'ranks differ'
    return models[0], norms[0]


@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("kind", ['adamw', 'lars'])
def test_sharded_graphed_clip_and_scaler_on_simulated_ranks(hvd, gteam, kind, k):
    a, na = _sharded_run(hvd, gteam, kind, k, graphed=False)
    b, nb = _sharded_run(hvd, gteam, kind, k, graphed=True)
    assert len(na) == len(nb) == 3 and all(float(x) > 0.05 for x in na)
    assert all(same(x, y) for x, y in zip(na, nb))
    for p, q in zip(a.parameters(), b.parameters()):
        assert same(p.detach(), q.detach())


# ---- across real ranks ---------------------------------------------------------------------------------------------------
@pytest.mark.skipif(ngpu() < 2, reason="needs >= 2 GPUs")
def test_graphed_clip_across_ranks(native_built):
    n = 2 if ngpu() < 4 else 4
    rc, out = run_parallel("graphed_clip_worker.py", np=n, timeout=420)
    assert "GRAPHED CLIP OK" in out, out[-4000:]
