"""Gradient accumulation in fp32 and in hvd.GraphedStep: the grad_accumulate_ kernel against the same torch ops in fp32
bit for bit, its single rounding against the 16-bit sum, GraphedStep with backward_passes_per_step = k against the eager
loop of k micro-steps at world size 1, the sharded (ZeRO-1) optimizer with k = 4 on 4 simulated ranks against the
unsharded fused update, and GraphedStep with k = 4 and the collectives captured in its last graph on 4 simulated ranks
(capturable stand-ins), unsharded and sharded, against the eager loop; with >= 2 GPUs, across real ranks."""
import copy
import math

import pytest
import torch

from conftest import run_parallel
from optim_cases import LOW, LOW_IDS, Slot, hvd, make_optimizer, mlp, ngpu, same  # noqa: F401  (hvd: fixture)
from sim_ranks import (ConvNet, gteam, micro_batch, reduced_grads, ref_step, sharded_team, team,  # noqa: F401
                       zero_copy_buckets)

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 3, 4, 4093, (1 << 24) + 3]


def _match(a, b):
    """Bit-identical where neither is NaN, NaN at the same places (NaN payloads are not compared)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and same(torch.where(na, 0, a), torch.where(nb, 0, b))


# ---- the kernel ---------------------------------------------------------------------------------------------------------
def _table(dtype, seed, offsets):
    """The sizes above plus 40 small tensors, gradients and accumulators at their own element offsets of guarded buffers."""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    sizes = SIZES + [int(x) for x in torch.randint(1, 600, (40,), generator=torch.Generator().manual_seed(seed))]
    go, ao = offsets
    grads = [Slot((n,), dtype, (go + i) % 4 if go < 0 else go, torch.randn(n, device='cuda', generator=gen) * 8, slack=5)
             for i, n in enumerate(sizes)]
    accs = [Slot((n,), torch.float32, (ao + i) % 4 if ao < 0 else ao, torch.randn(n, device='cuda', generator=gen) * 1000, slack=5)
            for i, n in enumerate(sizes)]
    return grads, accs


@pytest.mark.parametrize("dtype", LOW, ids=LOW_IDS)
@pytest.mark.parametrize("offsets", [(0, 0), (1, 0), (0, 3), (2, 1), (-1, -2)], ids=['aligned', 'g+1', 'acc+3', 'g+2-acc+1', 'mixed'])
def test_kernel_modes_match_torch_fp32(hvd, dtype, offsets):
    from horovod_b200 import ops
    grads, accs = _table(dtype, 3, offsets)
    g0, a0 = [s.t.clone() for s in grads], [s.t.clone() for s in accs]
    ops.grad_accumulate_([s.t for s in grads], [s.t for s in accs], 'first')
    for i, (g, a) in enumerate(zip(grads, accs)):
        assert same(a.t, g0[i].float()) and not bool(g.t.ne(0).any()) and not bool(g.t.signbit().any()), ('first', i)
    # add: a fresh gradient into the accumulator the 'first' fold left
    gen = torch.Generator(device='cuda').manual_seed(5)
    for g in grads:
        g.t.copy_(torch.randn(g.t.shape, device='cuda', generator=gen) * 3)
    g1, a1 = [s.t.clone() for s in grads], [s.t.clone() for s in accs]
    ops.grad_accumulate_([s.t for s in grads], [s.t for s in accs], 'add')
    for i, (g, a) in enumerate(zip(grads, accs)):
        assert same(a.t, a1[i] + g1[i].float()) and not bool(g.t.ne(0).any()), ('add', i)
    for g in grads:
        g.t.copy_(torch.randn(g.t.shape, device='cuda', generator=gen))
    g2, a2 = [s.t.clone() for s in grads], [s.t.clone() for s in accs]
    ops.grad_accumulate_([s.t for s in grads], [s.t for s in accs], 'last')
    for i, (g, a) in enumerate(zip(grads, accs)):
        assert same(g.t, (a2[i] + g2[i].float()).to(dtype)), ('last', i)
        assert same(a.t, a2[i]), ('last wrote the accumulator', i)
    for s in grads + accs:
        assert s.intact(), 'wrote outside a tensor'


@pytest.mark.parametrize("dtype", LOW, ids=LOW_IDS)
def test_kernel_propagates_inf_nan_and_overflows_fp16_only_at_last(hvd, dtype):
    from horovod_b200 import ops
    big = 6.0e4 if dtype == torch.float16 else 3.0e38
    g = torch.tensor([math.inf, -math.inf, math.nan, 1.0, big, -big, 2.0, 0.0] * 3, device='cuda').to(dtype)
    acc = torch.zeros(g.numel(), device='cuda')
    ops.grad_accumulate_([g.clone()], [acc], 'first')
    for mode in ('add', 'add'):
        ops.grad_accumulate_([g.clone()], [acc], mode)
    want = g.float() * 3
    assert _match(acc, want)  # fp32 holds 3 * 6e4 (fp16) and 9e38 overflows fp32 only for bf16's largest values
    if dtype == torch.float16:
        assert bool(torch.isfinite(acc[4::8]).all())
    out = g.clone()
    ops.grad_accumulate_([out], [acc], 'last')
    assert _match(out, (want + g.float()).to(dtype))
    assert bool(torch.isinf(out[4::8]).all()) and bool(torch.isnan(out[2::8]).all())


def test_fp32_accumulation_rounds_once(hvd):
    """16 bf16 micro-gradients whose magnitudes fall from 1 to 2^-12 (every element keeps its sign, so nothing cancels):
    the fp32 path is within 1 bf16 ulp of the fp64 sum everywhere; summing in bf16, as autograd does into a bf16 p.grad,
    loses the small contributions and is off by more."""
    from horovod_b200 import ops
    n = 1 << 16
    gen = torch.Generator(device='cuda').manual_seed(11)
    sign = torch.where(torch.rand(n, device='cuda', generator=gen) < 0.5, -1.0, 1.0)
    micro = [(sign * (0.5 + torch.rand(n, device='cuda', generator=gen)) * 2.0 ** -(12 * j / 15)).to(torch.bfloat16)
             for j in range(16)]
    exact = torch.stack([m.double() for m in micro]).sum(0)
    acc, g = torch.empty(n, device='cuda'), torch.empty(n, device='cuda', dtype=torch.bfloat16)
    for j, m in enumerate(micro):
        g.copy_(m)
        ops.grad_accumulate_([g], [acc], 'first' if j == 0 else 'last' if j == 15 else 'add')
    half = torch.zeros(n, device='cuda', dtype=torch.bfloat16)
    for m in micro:
        half += m
    ulp = torch.ldexp(torch.ones_like(exact), torch.frexp(exact.abs()).exponent - 8)
    err32, err16 = (g.double() - exact).abs(), (half.double() - exact).abs()
    assert bool((err32 <= ulp).all()), float((err32 / ulp).max())
    assert float((err16 / ulp).max()) > 1.0


def test_kernel_one_launch_no_sync_and_capturable(hvd):
    from horovod_b200 import ops
    grads, accs = _table(torch.bfloat16, 9, (1, 2))
    gs, as_ = [s.t for s in grads], [s.t for s in accs]
    snap = [t.clone() for t in gs + as_]
    torch.cuda.synchronize()
    before = ops.kernel_launches()
    torch.cuda.set_sync_debug_mode('error')
    try:
        ops.grad_accumulate_(gs, as_, 'add')
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert ops.kernel_launches() - before == 1
    eager = [t.clone() for t in gs + as_]
    for t, s in zip(gs + as_, snap):
        t.copy_(s)
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph):
            ops.grad_accumulate_(gs, as_, 'add')
    torch.cuda.current_stream().wait_stream(side)
    for t, s in zip(gs + as_, snap):
        t.copy_(s)
    graph.replay()
    torch.cuda.synchronize()
    assert all(same(a, b) for a, b in zip(gs + as_, eager))


def test_kernel_rejects_bad_arguments(hvd):
    from horovod_b200 import ops
    g, a = torch.zeros(64, device='cuda', dtype=torch.bfloat16), torch.zeros(64, device='cuda')
    with pytest.raises(ValueError):
        ops.grad_accumulate_([g], [a], 'middle')
    with pytest.raises(ValueError):
        ops.grad_accumulate_([g], [], 'add')
    for gg, aa in ((torch.zeros(64, device='cuda'), a), (g, a.to(torch.float16)), (g, torch.zeros(65, device='cuda')),
                   (g, torch.zeros(128, device='cuda')[::2]), (g.cpu(), a), (g, a.cpu())):
        with pytest.raises(RuntimeError):
            ops.grad_accumulate_([gg], [aa], 'add')


# ---- GraphedStep at world size 1 ----------------------------------------------------------------------------------------
CASES = [('sgd', torch.float32, False), ('adamw', torch.float32, False), ('lamb', torch.float32, False),
         ('lars', torch.float32, False), ('adamw', torch.bfloat16, False), ('adamw', torch.bfloat16, True),
         ('lars', torch.bfloat16, False), ('lars', torch.bfloat16, True)]
CASE_IDS = ['sgd', 'adamw', 'lamb', 'lars', 'adamw-bf16', 'adamw-bf16-acc32', 'lars-bf16', 'lars-bf16-acc32']


def _run(hvd, kind, dt, acc, k, graphed, buckets=False, steps=3, monkeypatch=None):
    if buckets:  # zero-copy buckets at world size 1
        zero_copy_buckets(monkeypatch)
    m = mlp(dt)
    opt = hvd.DistributedOptimizer(make_optimizer(hvd, kind, m.parameters()), named_parameters=m.named_parameters(), fused=True,
                                   master_weights=dt != torch.float32, backward_passes_per_step=k,
                                   grad_accumulation_dtype=torch.float32 if acc else None)
    assert bool(opt._buckets) == buckets
    gen = torch.Generator(device='cuda').manual_seed(2)
    xs = [torch.randn(16, 24, device='cuda', generator=gen).to(dt) for _ in range(steps * k)]
    fn = lambda x: m(x).float().square().mean() / k  # noqa: E731
    losses = []
    if graphed:
        step = hvd.GraphedStep(fn, opt, (xs[0],))
        assert step.captured, step.fallback_reason
        assert k == 1 or len(step.graphs) == min(k, 3)
        for x in xs:
            losses.append(step(x).detach().clone())
        assert step.replays == len(xs)
    else:
        for i, x in enumerate(xs):
            if i % k == 0:
                opt.zero_grad(set_to_none=False)
            loss = fn(x)
            loss.backward()
            losses.append(loss.detach().clone())
            if i % k == k - 1:
                opt.step()
    torch.cuda.synchronize()
    return m, opt, losses


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_graphed_step_equals_eager_loop(hvd, monkeypatch, k, case):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    kind, dt, acc = case
    (a, oa, la), (b, ob, lb) = [_run(hvd, kind, dt, acc, k, graphed) for graphed in (False, True)]
    assert all(same(x, y) for x, y in zip(la, lb)), 'every call returns its own micro-batch loss'
    for (name, p), q in zip(a.named_parameters(), b.parameters()):
        assert same(p.detach(), q.detach()), name
        sa, sb = oa.state[p], ob.state[q]
        assert sa.keys() == sb.keys()
        for key in sa:
            if torch.is_tensor(sa[key]) and sa[key].is_cuda:
                assert same(sa[key], sb[key]), (name, key)
        if 'step' in sa:
            assert float(sa['step']) == float(sb['step']) == 3, 'one optimizer step per k calls'
    assert bool(ob._param_accs) == acc


@pytest.mark.parametrize("k", [2, 4])
@pytest.mark.parametrize("acc", [False, True], ids=['bf16-sum', 'acc32'])
def test_graphed_step_equals_eager_loop_with_buckets(hvd, monkeypatch, k, acc):
    """The zero-copy bucket path: one fold per bucket and micro-step in the hooks, against the folds of the graphs."""
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    (a, oa, la), (b, ob, lb) = [_run(hvd, 'lars', torch.bfloat16, acc, k, graphed, buckets=True, monkeypatch=monkeypatch)
                                for graphed in (False, True)]
    assert all(same(x, y) for x, y in zip(la, lb))
    for (name, p), q in zip(a.named_parameters(), b.parameters()):
        assert same(p.detach(), q.detach()), name
        assert same(oa.state[p]['momentum_buffer'], ob.state[q]['momentum_buffer']), name
    assert all((bk['acc'] is not None) == acc for bk in ob._buckets)


def test_fp32_accumulation_differs_from_bf16_sum(hvd, monkeypatch):
    """The two accumulation paths see different gradients after k = 4 (else the feature would be moot), and the fp32
    one is the bf16 rounding of the fp32 sum of the micro-batch gradients."""
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    m16, _, _ = _run(hvd, 'lars', torch.bfloat16, False, 4, True, steps=2)
    m32, _, _ = _run(hvd, 'lars', torch.bfloat16, True, 4, True, steps=2)
    assert not all(same(p.detach(), q.detach()) for p, q in zip(m16.parameters(), m32.parameters()))


def test_k1_with_fp32_accumulation_is_the_default(hvd, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    (a, oa, la), (b, ob, lb) = [_run(hvd, 'adamw', torch.bfloat16, acc, 1, True) for acc in (False, True)]
    assert not ob._param_accs
    assert all(same(x, y) for x, y in zip(la, lb))
    for p, q in zip(a.parameters(), b.parameters()):
        assert same(p.detach(), q.detach())


def test_changed_k_raises(hvd):
    m = mlp(torch.float32)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters(),
                                   backward_passes_per_step=2)
    x = torch.randn(16, 24, device='cuda')
    step = hvd.GraphedStep(lambda x: m(x).square().mean(), opt, (x,))
    assert step.captured, step.fallback_reason
    step(x)
    opt.set_backward_passes_per_step(3)
    with pytest.raises(RuntimeError, match='backward_passes_per_step'):
        step(x)


# ---- sharded (ZeRO-1) on 4 simulated ranks ------------------------------------------------------------------------------
K = 4


def _backward_all(team, models, opts, step, dt, scalers=None):
    """K micro-batches on every rank: each rank reduce-scatters each bucket once, after its last micro-step."""
    mark = len(team.log)
    for r in range(team.n):
        opts[r].zero_grad()
        mine = len(team.log)
        for j in range(K):
            x, y = micro_batch(step, j, r, dt)
            loss = torch.nn.functional.cross_entropy(models[r](x), y) / K
            (scalers[r].scale(loss) if scalers else loss).backward()
            if j < K - 1:
                assert team.count('rs', mine) == 0, 'a reduce-scatter before the last micro-step'
    assert team.count('rs', mark) == team.n * len(opts[0]._buckets), 'one reduce-scatter per bucket, rank and step'


@pytest.mark.parametrize("kind", ['sgd', 'adamw', 'lamb', 'lars'])
@pytest.mark.parametrize("dt,master,acc", [(torch.float32, False, False), (torch.bfloat16, True, True)],
                         ids=['fp32', 'bf16-masters-acc32'])
def test_sharded_accumulation_on_simulated_ranks(hvd, team, monkeypatch, kind, dt, master, acc):
    """k = 4: the gradients each rank reduces are bit for bit its own micro-batch sum, computed by an unwrapped copy of
    its model (in fp32 and rounded once with the accumulator, in the model dtype without), the sharded update equals
    unsharded fused on the reduced gradients, and every rank ends with the same parameters."""
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    torch.manual_seed(0)
    base = ConvNet().cuda().to(dtype=dt, memory_format=torch.channels_last)
    models, opts = sharded_team(hvd, team, base, lambda m: make_optimizer(hvd, kind, m.parameters()), dt, min_buckets=2,
                                master_weights=master, backward_passes_per_step=K,
                                grad_accumulation_dtype=torch.float32 if acc else None)
    ref = copy.deepcopy(base)
    ref_opt = hvd.DistributedOptimizer(make_optimizer(hvd, kind, ref.parameters()), named_parameters=ref.named_parameters(),
                                       fused=True, master_weights=master, zero_copy=False)
    tol = dict(rtol=1e-5, atol=1e-6) if dt == torch.float32 else dict(rtol=1e-2, atol=1e-3)
    for step in range(3):
        # what every rank must contribute: its micro-batch gradients summed in fp32 (rounded once) or in the model dtype
        want = []
        for r in range(team.n):
            twin = copy.deepcopy(models[r])
            sums = [torch.zeros_like(p, dtype=torch.float32 if acc else dt) for p in twin.parameters()]
            for j in range(K):
                twin.zero_grad(set_to_none=True)
                x, y = micro_batch(step, j, r, dt)
                (torch.nn.functional.cross_entropy(twin(x), y) / K).backward()
                for s, p in zip(sums, twin.parameters()):
                    s += p.grad.to(s.dtype)
            want.append([s.to(dt) for s in sums])
        _backward_all(team, models, opts, step, dt)
        for r in range(team.n):  # before the reduction ran: the rank's own rounded sum sits in its gradient buckets
            for p, w in zip(models[r].parameters(), want[r]):
                assert same(p.grad, w), (step, r)
        for o in opts:
            o.synchronize()
        team.flush()
        grads = reduced_grads(opts, list(models[0].parameters()))

        def step_rank(r):
            with opts[r].skip_synchronize():
                opts[r].step()
        team.run(step_rank)
        ref_step(ref, ref_opt, grads)
        for r in range(1, team.n):
            for a, b in zip(models[r].parameters(), models[0].parameters()):
                assert same(a.detach(), b.detach()), 'ranks differ after the allgather'
        for (name, a), b in zip(models[0].named_parameters(), ref.parameters()):
            torch.testing.assert_close(a.float(), b.float(), **tol, msg=lambda s: 'step %d %s: %s' % (step, name, s))


def test_sharded_accumulation_with_clip_and_scaler(hvd, team):
    """fp16 with masters and the fp32 accumulator, ShardedGradScaler and clip_grad_norm_ with k = 4: one unscale, one
    norm and one coefficient per optimizer step; in step 1 an accumulator that is finite in fp32 but overflows fp16 at
    the 'last' fold on rank 0 makes every rank skip and halves every scale."""
    n, dt = team.n, torch.float16
    torch.manual_seed(0)
    base = ConvNet().cuda().to(dtype=dt, memory_format=torch.channels_last)
    models, opts = sharded_team(hvd, team, base, lambda m: make_optimizer(hvd, 'lars', m.parameters()), dt, min_buckets=2,
                                master_weights=True, backward_passes_per_step=K, grad_accumulation_dtype=torch.float32)
    scalers = [hvd.ShardedGradScaler('cuda', init_scale=256.0) for _ in range(n)]
    for step in range(3):
        before = [s.get_scale() for s in scalers]
        params_before = [p.detach().clone() for p in models[0].parameters()]
        if step == 1:
            # rank 0, before its last micro-step: an fp32 partial sum beyond fp16's range
            for r in range(n):
                opts[r].zero_grad()
            for j in range(K):
                for r in range(n):
                    if j == K - 1 and r == 0:
                        b0 = opts[0]._buckets[0]
                        b0['acc'][0] = 1.0e5
                        assert bool(torch.isfinite(b0['acc']).all())
                    x, y = micro_batch(step, j, r, dt)
                    scalers[r].scale(torch.nn.functional.cross_entropy(models[r](x), y) / K).backward()
        else:
            _backward_all(team, models, opts, step, dt, scalers)
        mark = len(team.log)
        team.run(lambda r: scalers[r].unscale_(opts[r]))
        norms = team.run(lambda r: opts[r].clip_grad_norm_(0.05))
        assert team.count('rs', mark) == 0, 'the gradients were reduced once, after the last micro-step'
        assert all(same(x, norms[0]) for x in norms)
        team.run(lambda r: (scalers[r].step(opts[r]), scalers[r].update()))
        if step == 1:
            assert all(s.get_scale() == before[0] / 2 for s in scalers)
            assert all(same(a.detach(), b) for a, b in zip(models[0].parameters(), params_before))
        else:
            assert all(s.get_scale() == before[0] for s in scalers)
            assert float(norms[0]) > 0.05 and not all(same(a.detach(), b) for a, b in zip(models[0].parameters(), params_before))
        for r in range(1, n):
            for a, b in zip(models[r].parameters(), models[0].parameters()):
                assert same(a.detach(), b.detach())


# ---- GraphedStep on 4 simulated ranks, unsharded and sharded -----------------------------------------------------------
def _team_run(hvd, team, kind, base, dt, shard, graphed, steps=3):
    n = team.n
    master = dt != torch.float32
    models, opts = sharded_team(hvd, team, base, lambda m: make_optimizer(hvd, kind, m.parameters()), dt, min_buckets=2,
                                shard_optimizer_state=shard, fused=True, master_weights=master, backward_passes_per_step=K,
                                grad_accumulation_dtype=torch.float32 if master else None)
    assert all(bool(o._buckets) for o in opts)
    nb = len(opts[0]._buckets)
    grad_kind = 'rs' if shard else 'ars'
    losses = [[] for _ in range(n)]
    fns = [lambda x, y, m=m: torch.nn.functional.cross_entropy(m(x), y) / K for m in models]
    if graphed:
        gsteps = []
        for r in range(n):
            gsteps.append(hvd.GraphedStep(fns[r], opts[r], micro_batch(0, 0, r, dt)))
            assert gsteps[r].captured and gsteps[r].comm_in_graph and len(gsteps[r].graphs) == 3, gsteps[r].fallback_reason
        # one collective per bucket, all of them recorded by the comm capture of the last graph
        assert all(len(c) == nb and all(x[0] == grad_kind and x[4] for x in c) for c in team.captured)
        for r in range(n):
            orig = opts[r].step
            opts[r].step = lambda *a, orig=orig, **kw: (team.before_step(), orig(*a, **kw))[1]
    for step in range(steps):
        mark = len(team.log)
        if graphed:
            for j in range(K - 1):
                for r in range(n):
                    losses[r].append(gsteps[r](*micro_batch(step, j, r, dt)).detach().clone())
            assert team.count(grad_kind, mark) == team.count('ran-' + grad_kind, mark) == 0
            runs = team.graph_runs
            out = team.run(lambda r: gsteps[r](*micro_batch(step, K - 1, r, dt)).detach().clone())
            for r in range(n):
                losses[r].append(out[r])
            assert team.graph_runs == runs + 1
            assert team.count('ran-' + grad_kind, mark) == n * nb and team.count(grad_kind, mark) == 0
        else:
            for r in range(n):
                opts[r].zero_grad(set_to_none=False)
                for j in range(K):
                    loss = fns[r](*micro_batch(step, j, r, dt))
                    loss.backward()
                    losses[r].append(loss.detach().clone())
            assert team.count(grad_kind, mark) == n * nb, 'one collective per bucket, rank and step'
            team.flush()

            def step_rank(r):
                with opts[r].skip_synchronize():
                    opts[r].step()
            for o in opts:
                o.synchronize()
            team.run(step_rank)
        for r in range(1, n):
            for a, b in zip(models[r].parameters(), models[0].parameters()):
                assert same(a.detach(), b.detach()), 'ranks differ'
    return models, opts, losses


@pytest.mark.parametrize("kind", ['sgd', 'adamw', 'lamb', 'lars'])
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=['fp32', 'bf16-masters-acc32'])
def test_graphed_step_on_simulated_ranks(hvd, gteam, kind, dt):
    """k = 4 on 4 simulated ranks, unsharded (bucket allreduce) and sharded (reduce-scatter): GraphedStep with the
    collectives captured in its last graph equals the eager loop bit for bit (parameters, losses, optimizer state); each
    bucket's collective is recorded once per rank, by the last graph, and runs once per optimizer step; every rank ends
    with the same parameters, and the sharded run follows the unsharded one."""
    torch.manual_seed(0)
    base = ConvNet().cuda().to(dtype=dt, memory_format=torch.channels_last)
    finals = {}
    for shard in (False, True):
        runs = []
        for graphed in (False, True):
            gteam.captured = [[] for _ in range(gteam.n)]
            runs.append(_team_run(hvd, gteam, kind, base, dt, shard, graphed))
        (me, oe, le), (mg, og, lg) = runs
        for r in range(gteam.n):
            assert all(same(a, b) for a, b in zip(le[r], lg[r])), (shard, r, 'losses')
            for (name, a), b in zip(me[r].named_parameters(), mg[r].parameters()):
                assert same(a.detach(), b.detach()), (shard, r, name)
        if shard:
            for be, bg in zip(oe[0]._buckets, og[0]._buckets):
                for key in be['state']:
                    assert same(be['state'][key], bg['state'][key]), key
                if dt != torch.float32:
                    assert bg['acc'] is not None
        else:
            for pe, pg in zip(me[0].parameters(), mg[0].parameters()):
                for key, t in oe[0].state[pe].items():
                    if torch.is_tensor(t) and t.is_cuda:
                        assert same(t, og[0].state[pg][key]), key
            assert all((b['acc'] is not None) == (dt != torch.float32) for b in og[0]._buckets)
        finals[shard] = mg[0]
    tol = dict(rtol=1e-5, atol=1e-6) if dt == torch.float32 else dict(rtol=1e-2, atol=1e-3)
    for (name, a), b in zip(finals[False].named_parameters(), finals[True].parameters()):
        torch.testing.assert_close(a.float(), b.float(), **tol, msg=lambda s: 'sharded vs unsharded %s: %s' % (name, s))


# ---- real ranks ----------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(ngpu() < 2, reason="needs >= 2 GPUs")
def test_grad_accumulation_across_ranks(hvd):
    n = 2 if ngpu() < 4 else 4
    rc, out = run_parallel("grad_accumulation_worker.py", np=n, timeout=420)
    assert "GRAD ACCUMULATION OK" in out, out[-4000:]
