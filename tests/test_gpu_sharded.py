"""Sharded optimizer state (ZeRO-1) on the GPU: the in-place reduce-scatter / allgather kernels with N simulated ranks on
one GPU (csrc/common/sim_api.cc), the reduce-scatter -> fused Adam on shards -> allgather chain against allreduce + full
Adam, world size 1, and (with >= 2 GPUs) the sharded DistributedOptimizer across real ranks."""
import pytest
import torch

from conftest import run_parallel
from optim_cases import hvd, ngpu  # noqa: F401  (hvd: fixture)
from sim_ranks import ConvNetWithUnused, batch, sharded_team, team  # noqa: F401  (team: fixture)

pytestmark = pytest.mark.gpu


# shard element counts: a multiple of 8 (16 B in every dtype) but not of the 4 KiB row or the 32 KiB chunk
SHARDS = [8, 24008, 40008]


def _inputs(n, shard, dtype, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    if dtype.is_floating_point:
        return [torch.randn(n * shard, device='cuda', generator=g).to(dtype) for _ in range(n)]
    return [torch.randint(-50, 50, (n * shard,), device='cuda', generator=g).to(dtype) for _ in range(n)]


RS_DTYPES = [torch.float32, torch.bfloat16, torch.float16, torch.int32, torch.float64, torch.int64]
SUM, MIN, MAX = 1, 3, 4
RS_CASES = ([pytest.param(d, SUM, id='dtype%d' % i) for i, d in enumerate(RS_DTYPES)] +
            [pytest.param(d, op, id='dtype%d-%s' % (i, name)) for op, name in ((MIN, 'min'), (MAX, 'max'))
             for i, d in enumerate(RS_DTYPES)])


@pytest.mark.parametrize("n", [2, 3, 4, 5, 6, 8])
@pytest.mark.parametrize("dtype,op", RS_CASES)
def test_sim_reducescatter(hvd, n, dtype, op):
    from horovod_b200.ops import sim
    repeats = 3
    # integers: SUM / MIN / MAX; floats: AVERAGE as SUM with scale (and a scaled MIN / MAX)
    scale = 1.0 if not dtype.is_floating_point else 1.0 / n
    for shard in SHARDS:
        ts = _inputs(n, shard, dtype, seed=shard + n)
        before = [t.clone() for t in ts]
        sim.inplace_reducescatter(ts, op=op, ctas=8, scale=scale, repeats=repeats)
        torch.cuda.synchronize()
        for r in range(n):
            lo, hi = r * shard, (r + 1) * shard
            # each repeat re-reduces: rank r's own shard already holds the previous result, the peers' shards do not
            if op == SUM:
                others = sum(before[q][lo:hi].double() for q in range(n) if q != r)
                ref = before[r][lo:hi].double()
                for _ in range(repeats):
                    ref = ((ref + others) * scale).to(dtype).double()
            else:
                # MIN / MAX select one input, then scale in the fp32 (fp64 for fp64) accumulator and round: exact
                pick = (lambda a, b: torch.minimum(a, b)) if op == MIN else (lambda a, b: torch.maximum(a, b))
                others = before[(r + 1) % n][lo:hi]
                for q in range(n):
                    if q != r:
                        others = pick(others, before[q][lo:hi])
                acc = torch.float64 if dtype == torch.float64 else torch.float32
                ref = before[r][lo:hi]
                for _ in range(repeats):
                    ref = pick(ref, others)
                    if dtype.is_floating_point:
                        ref = (ref.double() * float(torch.tensor(scale, dtype=acc))).to(acc).to(dtype)
                ref = ref.double()
            if not dtype.is_floating_point or op != SUM:
                assert torch.equal(ts[r][lo:hi].double(), ref)
            else:
                tol = {torch.float32: 1e-5, torch.float64: 1e-12}.get(dtype, 2e-2)
                torch.testing.assert_close(ts[r][lo:hi].double(), ref, rtol=tol, atol=tol)
            # nothing outside the own shard was written (catches stray peer stores)
            assert torch.equal(ts[r][:lo], before[r][:lo]) and torch.equal(ts[r][hi:], before[r][hi:])


@pytest.mark.parametrize("n", [2, 3, 4, 5, 6, 8])
def test_sim_allgather_is_byte_exact(hvd, n):
    from horovod_b200.ops import sim
    for shard_bytes in (16, 96032, 1 << 20):
        ts = [torch.randint(0, 256, (n * shard_bytes,), device='cuda', dtype=torch.uint8) for _ in range(n)]
        ref = torch.cat([ts[r][r * shard_bytes:(r + 1) * shard_bytes] for r in range(n)])
        sim.inplace_allgather(ts, ctas=8, repeats=2)
        torch.cuda.synchronize()
        for r in range(n):
            assert torch.equal(ts[r], ref)


def test_sim_rejects_sizes_not_divisible_by_ranks(hvd):
    from horovod_b200.ops import sim
    ts = [torch.zeros(4 * 8 + 4, device='cuda') for _ in range(4)]  # 144 B is not a multiple of 16 * 4
    with pytest.raises(RuntimeError):
        sim.inplace_reducescatter(ts, op=sim.SUM)
    with pytest.raises(RuntimeError):
        sim.inplace_allgather(ts)


def test_sim_sharded_adam_chain_matches_allreduce_and_full_adam(hvd):
    """reduce-scatter -> fused AdamW on each rank's shard -> allgather == allreduce -> AdamW on everything."""
    from horovod_b200.ops import sim
    from horovod_b200.torch import mpi_ops
    native = mpi_ops._native()
    n, shard = 4, 24008
    torch.manual_seed(0)
    p0 = torch.randn(n * shard, device='cuda')
    params = [p0.clone() for _ in range(n)]
    states = [(torch.zeros(shard, device='cuda'), torch.zeros(shard, device='cuda')) for _ in range(n)]
    ref_p = p0.clone()
    ref_m, ref_v = torch.zeros_like(ref_p), torch.zeros_like(ref_p)
    hp = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01)
    for step in range(1, 4):
        grads = [torch.randn(n * shard, device='cuda') for _ in range(n)]
        avg = torch.stack(grads).sum(0) / n
        native.fused_adam_step([ref_p], [avg], [ref_m], [ref_v], hp['lr'], hp['beta1'], hp['beta2'], hp['eps'],
                               hp['weight_decay'], step, 1.0, True)
        sim.inplace_reducescatter(grads, op=sim.SUM, scale=1.0 / n)
        for r in range(n):
            sl = slice(r * shard, (r + 1) * shard)
            native.fused_adam_step([params[r][sl]], [grads[r][sl]], [states[r][0]], [states[r][1]], hp['lr'], hp['beta1'],
                                   hp['beta2'], hp['eps'], hp['weight_decay'], step, 1.0, True)
        torch.cuda.synchronize()
        sim.inplace_allgather(params)
        torch.cuda.synchronize()
    for r in range(n):
        torch.testing.assert_close(params[r], ref_p, rtol=1e-5, atol=1e-6)
        assert torch.equal(params[r], params[0])
    # the sharded result also matches torch's own AdamW on the averaged gradients
    t = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([t], lr=hp['lr'], betas=(hp['beta1'], hp['beta2']), eps=hp['eps'], weight_decay=hp['weight_decay'])
    torch.manual_seed(0)
    torch.randn(n * shard, device='cuda')
    for _ in range(3):
        t.grad = torch.stack([torch.randn(n * shard, device='cuda') for _ in range(n)]).sum(0) / n
        opt.step()
    torch.testing.assert_close(params[0], t.detach(), rtol=1e-4, atol=1e-5)


def test_world_size_1_returns_the_existing_optimizer(hvd):
    from horovod_b200.torch.sharded_optimizer import _ShardedDistributedOptimizer
    torch.manual_seed(1)
    model = torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 8)).cuda()
    ref = torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 8)).cuda()
    ref.load_state_dict(model.state_dict())
    opt = hvd.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-2), named_parameters=model.named_parameters(),
                                   fused=True, shard_optimizer_state=True)
    assert not isinstance(opt, _ShardedDistributedOptimizer) and hasattr(opt, '_fused')
    ropt = torch.optim.AdamW(ref.parameters(), lr=1e-2)
    for i in range(5):
        x = torch.randn(16, 32, device='cuda')
        for m, o in ((model, opt), (ref, ropt)):
            o.zero_grad()
            m(x).square().mean().backward()
            o.step()
    for a, b in zip(model.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("kind", ["adamw", "sgd", "adamw-fp16"])
def test_sharded_optimizer_on_simulated_ranks(hvd, team, kind):
    """The sharded DistributedOptimizer itself (buckets, hooks, launch order, missing gradients, fused shard update,
    synchronize() followed by step()) on 4 simulated ranks, against plain torch on averaged gradients. The fp16 model
    is compared with an fp32 reference model, so only to fp16 accuracy; the ranks must still agree bit for bit."""
    import copy
    import warnings
    from horovod_b200.torch.sharded_optimizer import _ShardedDistributedOptimizer
    n = team.n
    dt = torch.float16 if kind == 'adamw-fp16' else torch.float32
    tol = dict(rtol=1e-4, atol=1e-5) if dt == torch.float32 else dict(rtol=2e-2, atol=2e-3)
    torch.manual_seed(0)
    base = ConvNetWithUnused().cuda().to(dtype=dt, memory_format=torch.channels_last)

    def make(m):
        if kind.startswith('adamw'):
            return torch.optim.AdamW(m.parameters(), lr=1e-2, weight_decay=0.05)
        return torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-4)

    models, opts = sharded_team(hvd, team, base, make, dt, min_buckets=3)
    assert all(isinstance(o, _ShardedDistributedOptimizer) for o in opts)
    assert models[0].conv.weight.is_contiguous(memory_format=torch.channels_last)
    ref = copy.deepcopy(base).float()
    ref_opt = make(ref)

    for step in range(6):
        use = lambda r: not (step == 2 or (step == 4 and r == 0))  # noqa: E731  unused on every rank / on rank 0 only
        grads = [torch.zeros_like(p) for p in ref.parameters()]
        for r in range(n):
            x, y = batch(step, r)
            ref.zero_grad()
            torch.nn.functional.cross_entropy(ref(x, use(r)), y).backward()
            for g, p in zip(grads, ref.parameters()):
                if p.grad is not None:
                    g += p.grad
        for g, p in zip(grads, ref.parameters()):
            p.grad = g / n
        ref_opt.step()

        for r in range(n):
            opts[r].zero_grad()
            x, y = batch(step, r)
            torch.nn.functional.cross_entropy(models[r](x.to(dt), use(r)), y).backward()
        if step == 1:
            with pytest.raises(AssertionError):
                opts[0].zero_grad()  # reduce-scatters may be in flight
        for o in opts:
            o.synchronize()
        team.flush()
        for o in opts:
            if step % 2:
                with warnings.catch_warnings(record=True) as w:
                    warnings.simplefilter('always')
                    o.step()  # after synchronize(): must not reduce a second time
                assert any('skip_synchronize' in str(x.message) for x in w)
            else:
                with o.skip_synchronize():
                    o.step()
        team.flush()
        for r in range(n):
            for (name, a), b in zip(models[r].named_parameters(), ref.parameters()):
                torch.testing.assert_close(a.float(), b, **tol, msg=lambda m: '%s step %d rank %d: %s' % (name, step, r, m))
                assert torch.equal(a, dict(models[0].named_parameters())[name])
    assert models[0].conv.weight.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.skipif(ngpu() < 2, reason="needs >= 2 GPUs")
def test_sharded_optimizer_across_ranks(native_built):
    n = 2 if ngpu() < 4 else (4 if ngpu() < 8 else 8)
    rc, out = run_parallel("sharded_optimizer_worker.py", np=n, timeout=420)
    assert "SHARDED OK" in out, out[-4000:]
