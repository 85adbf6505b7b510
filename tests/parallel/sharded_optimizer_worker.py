"""Sharded optimizer state (ZeRO-1) on >= 2 GPUs (run under hvdrun):

1. hvd.captured_reducescatter_ / hvd.captured_allgather_ on registered tensors against closed forms.
2. 10-step trajectories of AdamW and SGD-nesterov: sharded == unsharded fused=True == plain torch on averaged gradients;
   parameters bit-identical across ranks; optimizer-state bytes per rank == the padded 1/N.
3. backward_passes_per_step=2, and a parameter unused in a step (no hang, its gradient counts as zeros).
4. state_dict() round trips sharded <-> unsharded and training continues; broadcast_parameters +
   broadcast_optimizer_state.
5. hvd.GraphedStep: the reduce-scatters are graph nodes (comm_in_graph) and the trajectory follows the eager one.
"""
import copy

import torch

import horovod_b200.torch as hvd
from horovod_b200.torch.sharded_optimizer import _ShardedDistributedOptimizer

hvd.init()
rank, size = hvd.rank(), hvd.size()
torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank())


def check_captured_collectives():
    shard = (1 << 16) + 8
    for dtype in (torch.float32, torch.bfloat16):
        buf = hvd.symm_empty(size * shard, dtype=dtype)
        buf.copy_(torch.arange(size * shard, device=dev).remainder(97).to(dtype) + rank)
        before = buf.clone()
        view = hvd.captured_reducescatter_(buf, op=hvd.Average)
        torch.cuda.synchronize()
        lo, hi = rank * shard, (rank + 1) * shard
        assert view.data_ptr() == buf[lo:hi].data_ptr() and view.numel() == shard
        exp = (torch.arange(lo, hi, device=dev).remainder(97).double() + (size - 1) / 2.0)
        assert torch.allclose(view.double(), exp, rtol=1e-2 if dtype == torch.bfloat16 else 1e-6), dtype
        assert torch.equal(buf[:lo], before[:lo]) and torch.equal(buf[hi:], before[hi:])
        buf[lo:hi].fill_(float(rank + 1))
        hvd.captured_allgather_(buf)
        torch.cuda.synchronize()
        exp = torch.arange(size, device=dev).repeat_interleave(shard).to(dtype) + 1
        assert torch.equal(buf, exp), dtype
    try:
        hvd.captured_reducescatter_(hvd.symm_empty(size * 16 + 4, dtype=torch.float32))
        raise SystemExit('captured_reducescatter_ accepted a size that does not split into 16 B shards')
    except hvd.HorovodInternalError:
        pass
    print('[ok] captured reduce-scatter / allgather', flush=True)


class Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(48, 96)
        self.b = torch.nn.Linear(96, 10)
        self.unused = torch.nn.Linear(5, 10)  # only in the forward when asked

    def forward(self, x, use_all=True):
        y = self.b(torch.relu(self.a(x)))
        if use_all:
            y = y + self.unused(x[:, :5])
        return y


def _batch(step, k=0):
    g = torch.Generator(device=dev).manual_seed(1000 * step + 10 * rank + k)
    return torch.randn(32, 48, device=dev, generator=g), torch.randint(0, 10, (32,), device=dev, generator=g)


def _make(kind, base):
    m = copy.deepcopy(base)
    if kind == 'adamw':
        opt = torch.optim.AdamW(m.parameters(), lr=1e-2, weight_decay=0.05)
    else:
        opt = torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-4)
    return m, opt


def _train(m, opt, steps, start=0, use_all=lambda s: True, passes=1, plain=False):
    for s in range(start, start + steps):
        opt.zero_grad()
        for k in range(passes):
            x, y = _batch(s, k)
            torch.nn.functional.cross_entropy(m(x, use_all(s)), y).backward()
        if plain:  # plain torch on averaged gradients
            for name, p in m.named_parameters():
                if p.grad is None:
                    p.grad = torch.zeros_like(p)
                p.grad.copy_(hvd.allreduce(p.grad, op=hvd.Average, name='plain.' + name))
        opt.step()
    torch.cuda.synchronize()


def _same_across_ranks(m):
    for p in m.parameters():
        g = hvd.allgather(p.detach().reshape(1, -1))
        assert all(torch.equal(g[0], g[r]) for r in range(size)), 'parameters differ across ranks'


def _close(m1, m2, tol=1e-4):
    for (n1, a), b in zip(m1.named_parameters(), m2.parameters()):
        assert torch.allclose(a, b, rtol=tol, atol=tol), (n1, (a - b).abs().max().item())


def check_trajectories():
    for kind in ('adamw', 'sgd'):
        torch.manual_seed(0)
        base = Net().to(dev)
        ms, os_ = _make(kind, base)
        sharded = hvd.DistributedOptimizer(os_, named_parameters=ms.named_parameters(), shard_optimizer_state=True)
        assert isinstance(sharded, _ShardedDistributedOptimizer)
        mu, ou = _make(kind, base)
        unsharded = hvd.DistributedOptimizer(ou, named_parameters=mu.named_parameters(), fused=True)
        mp, op = _make(kind, base)
        _train(ms, sharded, 10)
        _train(mu, unsharded, 10)
        _train(mp, op, 10, plain=True)
        _close(ms, mu)
        _close(ms, mp)
        _same_across_ranks(ms)
        # optimizer state: this rank's padded shard of every bucket only
        per = 2 if kind == 'adamw' else 1
        state_bytes = sum(t.numel() * t.element_size() for b in sharded._buckets for t in b['state'].values())
        padded = sum(b['numel'] * 4 for b in sharded._buckets)  # fp32 parameters and fp32 state
        expected = per * padded // size
        assert state_bytes == expected, (state_bytes, expected)
        assert len(sharded.state) == 0
    print('[ok] trajectories (AdamW, SGD-nesterov), bit-identical parameters, 1/N state', flush=True)


def check_accumulation_and_unused():
    torch.manual_seed(1)
    base = Net().to(dev)
    ms, os_ = _make('adamw', base)
    sharded = hvd.DistributedOptimizer(os_, named_parameters=ms.named_parameters(), shard_optimizer_state=True,
                                       backward_passes_per_step=2)
    mp, op = _make('adamw', base)
    _train(ms, sharded, 4, passes=2)
    _train(mp, op, 4, passes=2, plain=True)
    _close(ms, mp)
    # a parameter unused in some steps, on every rank or on one rank only
    torch.manual_seed(2)
    base = Net().to(dev)
    ms, os_ = _make('sgd', base)
    sharded = hvd.DistributedOptimizer(os_, named_parameters=ms.named_parameters(), shard_optimizer_state=True)
    mp, op = _make('sgd', base)
    use = lambda s: not (s % 2 == 1 or (s == 2 and rank == 0))  # noqa: E731
    _train(ms, sharded, 6, use_all=use)
    _train(mp, op, 6, use_all=use, plain=True)
    _close(ms, mp)
    _same_across_ranks(ms)
    print('[ok] backward_passes_per_step=2, unused parameters', flush=True)


def check_synchronize_then_step():
    """The explicit synchronize() idiom: step() afterwards (with or without skip_synchronize) must not reduce again."""
    torch.manual_seed(5)
    base = Net().to(dev)
    ms, os_ = _make('adamw', base)
    sharded = hvd.DistributedOptimizer(os_, named_parameters=ms.named_parameters(), shard_optimizer_state=True)
    mp, op = _make('adamw', base)
    for s in range(4):
        sharded.zero_grad()
        x, y = _batch(s)
        torch.nn.functional.cross_entropy(ms(x), y).backward()
        if s == 0:
            try:
                sharded.zero_grad()
                raise SystemExit('zero_grad() between backward and step() was accepted')
            except AssertionError:
                pass
        sharded.synchronize()
        if s % 2:
            sharded.step()  # warns, does not reduce a second time
        else:
            with sharded.skip_synchronize():
                sharded.step()
    _train(mp, op, 4, plain=True)
    _close(ms, mp)
    _same_across_ranks(ms)
    print('[ok] synchronize() then step()', flush=True)


def check_checkpoints():
    torch.manual_seed(3)
    base = Net().to(dev)
    ms, os_ = _make('adamw', base)
    sharded = hvd.DistributedOptimizer(os_, named_parameters=ms.named_parameters(), shard_optimizer_state=True)
    mu, ou = _make('adamw', base)
    unsharded = hvd.DistributedOptimizer(ou, named_parameters=mu.named_parameters(), fused=True)
    _train(ms, sharded, 3)
    _train(mu, unsharded, 3)
    sd_s, sd_u = sharded.state_dict(), unsharded.state_dict()
    assert sorted(sd_s['state']) == sorted(sd_u['state'])
    for i, st in sd_s['state'].items():
        assert all(not v.is_cuda for v in st.values())
        for k in ('exp_avg', 'exp_avg_sq'):
            assert torch.allclose(st[k], sd_u['state'][i][k].cpu(), rtol=1e-5, atol=1e-6), (i, k)
        assert float(st['step']) == float(sd_u['state'][i]['step'])
    # sharded -> unsharded and unsharded -> sharded: both continue exactly like an uninterrupted run
    m2, o2 = _make('adamw', base)
    m2.load_state_dict(ms.state_dict())
    u2 = hvd.DistributedOptimizer(o2, named_parameters=m2.named_parameters(), fused=True)
    u2.load_state_dict(sd_s)
    m3, o3 = _make('adamw', base)
    m3.load_state_dict(mu.state_dict())
    s3 = hvd.DistributedOptimizer(o3, named_parameters=m3.named_parameters(), shard_optimizer_state=True)
    s3.load_state_dict(sd_u)
    _train(ms, sharded, 3, start=3)
    _train(m2, u2, 3, start=3)
    _train(m3, s3, 3, start=3)
    _close(ms, m2)
    _close(ms, m3)
    # broadcast_parameters + broadcast_optimizer_state: rank 0's weights, hyper-parameters and step counts everywhere
    torch.manual_seed(10 + rank)
    m4 = Net().to(dev)
    o4 = torch.optim.AdamW(m4.parameters(), lr=1e-3 * (rank + 1))
    s4 = hvd.DistributedOptimizer(o4, named_parameters=m4.named_parameters(), shard_optimizer_state=True)
    hvd.broadcast_parameters(m4.state_dict(), root_rank=0)
    hvd.broadcast_optimizer_state(s4, root_rank=0)
    assert s4.param_groups[0]['lr'] == 1e-3
    _same_across_ranks(m4)
    _train(m4, s4, 2)
    _same_across_ranks(m4)
    print('[ok] state_dict sharded <-> unsharded, broadcast_optimizer_state', flush=True)


def check_graphed_step():
    torch.manual_seed(4)
    base = Net().to(dev)
    me, oe = _make('adamw', base)
    eager = hvd.DistributedOptimizer(oe, named_parameters=me.named_parameters(), shard_optimizer_state=True)
    mg, og = _make('adamw', base)
    graphed = hvd.DistributedOptimizer(og, named_parameters=mg.named_parameters(), shard_optimizer_state=True)
    x0, y0 = _batch(0)
    step = hvd.GraphedStep(lambda x, y: torch.nn.functional.cross_entropy(mg(x), y), graphed, (x0, y0))
    assert step.captured and step.comm_in_graph, step.fallback_reason
    for s in range(6):
        x, y = _batch(s)
        step(x, y)
    _train(me, eager, 6)
    _close(mg, me)
    _same_across_ranks(mg)
    print('[ok] GraphedStep with the reduce-scatters inside the graph', flush=True)


check_captured_collectives()
check_trajectories()
check_accumulation_and_unused()
check_synchronize_then_step()
check_checkpoints()
check_graphed_step()
hvd.shutdown()
print('SHARDED OK', flush=True)
