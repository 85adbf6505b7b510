"""Global-norm clipping and AMP loss scaling in hvd.GraphedStep on >= 2 GPUs (run under hvdrun), for SGD, AdamW, hvd.Lamb
and hvd.Lars, the unsharded optimizer (zero-copy buckets, allreduce) and the sharded one (reduce-scatter), k = 1 and
k = 4, with the collectives in the graph:

1. GraphedStep(max_grad_norm=0.05, scaler=...) follows the eager loop (synchronize, unscale_, clip_grad_norm_,
   skip_synchronize + step, update).  Sharded, both issue the same kernels and agree bit for bit; unsharded, the eager
   bucket allreduce goes through the engine and the captured one is `captured_allreduce_`, so they are compared to a
   tolerance.
2. The clipped norm and the parameters are the same bits on every rank.
"""
import copy

import torch

import horovod_b200.torch as hvd

hvd.init()
rank, size = hvd.rank(), hvd.size()
torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank())
MAX_NORM = 0.05


def batch(step, r):
    g = torch.Generator(device=dev).manual_seed(1000 * step + r)
    return torch.randn(8, 48, device=dev, generator=g), torch.randint(0, 10, (8,), device=dev, generator=g)


def same_on_all_ranks(t):
    return all(torch.equal(x, t) for x in hvd.allgather(t.detach().reshape(1, -1).float()).unbind(0))


def make(m, shard, kind, k):
    ps = m.parameters()
    opt = {'sgd': lambda: torch.optim.SGD(ps, lr=0.05, momentum=0.9, weight_decay=1e-4),
           'adamw': lambda: torch.optim.AdamW(ps, lr=1e-2, weight_decay=0.01),
           'lamb': lambda: hvd.Lamb(ps, lr=1e-2, weight_decay=0.01),
           'lars': lambda: hvd.Lars(ps, lr=1.0, momentum=0.9, weight_decay=1e-3, trust_coefficient=0.01)}[kind]()
    return hvd.DistributedOptimizer(opt, named_parameters=m.named_parameters(), fused=True, shard_optimizer_state=shard,
                                    bucket_cap_mb=0.01, backward_passes_per_step=k)


def scaler_for(shard):
    return (hvd.ShardedGradScaler if shard else torch.amp.GradScaler)('cuda', init_scale=256.0)


def loss_fn(m, k):
    return lambda x, y: torch.nn.functional.cross_entropy(m(x).float(), y) / k


def eager(m, o, scaler, k, steps):
    norms = []
    for i in range(steps * k):
        if i % k == 0:
            o.zero_grad()
        scaler.scale(loss_fn(m, k)(*batch(i, rank))).backward()
        if i % k == k - 1:
            o.synchronize()
            scaler.unscale_(o)
            norms.append(o.clip_grad_norm_(MAX_NORM).clone())
            with o.skip_synchronize():
                scaler.step(o)
            scaler.update()
    torch.cuda.synchronize()
    return norms


torch.backends.cudnn.deterministic = True
for kind in ('sgd', 'adamw', 'lamb', 'lars'):
    torch.manual_seed(0)
    base = torch.nn.Sequential(torch.nn.Linear(48, 96), torch.nn.ReLU(), torch.nn.Linear(96, 10)).to(dev)
    hvd.broadcast_parameters(base.state_dict(), root_rank=0)
    for shard in (False, True):
        for k in (1, 4):
            mg, me = copy.deepcopy(base), copy.deepcopy(base)
            og, oe = make(mg, shard, kind, k), make(me, shard, kind, k)
            sg = scaler_for(shard)
            norms = []
            orig = og.clip_grad_norm_
            og.clip_grad_norm_ = lambda *a, **kw: norms.append(orig(*a, **kw).clone()) or norms[-1]
            gstep = hvd.GraphedStep(loss_fn(mg, k), og, batch(0, rank), max_grad_norm=MAX_NORM, scaler=sg)
            assert gstep.captured and gstep.comm_in_graph, (gstep.fallback_reason, gstep.comm_in_graph)
            for i in range(3 * k):
                gstep(*batch(i, rank))
            torch.cuda.synchronize()
            want = eager(me, oe, scaler_for(shard), k, 3)
            assert len(norms) == len(want) == 3 and all(float(n) > MAX_NORM for n in norms)
            for n, w in zip(norms, want):
                assert same_on_all_ranks(n) and same_on_all_ranks(w)
                torch.testing.assert_close(n, w, rtol=1e-5, atol=0)
            for a, b in zip(mg.parameters(), me.parameters()):
                assert same_on_all_ranks(a) and same_on_all_ranks(b)
                if shard:
                    assert torch.equal(a.detach().view(torch.uint8), b.detach().view(torch.uint8))
                else:
                    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
            print('[ok] %s %s k=%d GraphedStep clip + scaler' % (kind, 'sharded' if shard else 'unsharded', k), flush=True)

hvd.barrier()
if rank == 0:
    print('GRAPHED CLIP OK', flush=True)
