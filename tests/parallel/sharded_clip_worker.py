"""Gradient clipping and AMP loss scaling with sharded optimizer state on >= 2 GPUs (run under hvdrun):

1. 6-step AdamW trajectories with opt.clip_grad_norm_ (2-norm and inf-norm, the clip active on even steps): the sharded
   optimizer follows the unsharded DistributedOptimizer with synchronize() + torch.nn.utils.clip_grad_norm_; the returned
   norm has the same bits on every rank and matches torch's; parameters are bit-identical across ranks.
2. hvd.ShardedGradScaler with an fp16 model: an inf in rank 0's local gradient only makes every rank skip the step and
   back off the scale alike; the other steps update.
"""
import copy
import math

import torch

import horovod_b200.torch as hvd

hvd.init()
rank, size = hvd.rank(), hvd.size()
torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank())


def batch(step, r):
    g = torch.Generator(device=dev).manual_seed(1000 * step + r)
    return torch.randn(8, 48, device=dev, generator=g), torch.randint(0, 10, (8,), device=dev, generator=g)


def same_on_all_ranks(t):
    return all(torch.equal(x, t) for x in hvd.allgather(t.detach().reshape(1, -1).float()).unbind(0))


def check_clip(norm_type):
    torch.manual_seed(0)
    base = torch.nn.Sequential(torch.nn.Linear(48, 96), torch.nn.ReLU(), torch.nn.Linear(96, 10)).to(dev)
    hvd.broadcast_parameters(base.state_dict(), root_rank=0)
    ms, ops = [], []
    for shard in (True, False):
        m = copy.deepcopy(base)
        ops.append(hvd.DistributedOptimizer(torch.optim.AdamW(m.parameters(), lr=1e-2, weight_decay=0.05),
                                            named_parameters=m.named_parameters(), fused=True, shard_optimizer_state=shard,
                                            bucket_cap_mb=0.01))
        ms.append(m)
    for step in range(6):
        x, y = batch(step, rank)
        norms = []
        for i, (m, o) in enumerate(zip(ms, ops)):
            o.zero_grad()
            torch.nn.functional.cross_entropy(m(x), y).backward()
            if i == 0:
                # the same max_norm on every rank: half or twice the unsharded run's norm of this step, computed below
                continue
            o.synchronize()
            norm = torch.nn.utils.get_total_norm([p.grad for p in m.parameters()], norm_type)
            max_norm = float(norm) * (0.5 if step % 2 == 0 else 2.0)
            torch.nn.utils.clip_grad_norm_(m.parameters(), max_norm, norm_type)
            with o.skip_synchronize():
                o.step()
            norms.append(norm)
        got = ops[0].clip_grad_norm_(max_norm, norm_type=norm_type)
        ops[0].step()
        torch.cuda.synchronize()
        assert same_on_all_ranks(got), 'norm differs between ranks'
        assert abs(float(got) - float(norms[0])) <= 1e-5 * float(norms[0]), (step, float(got), float(norms[0]))
        for a, b in zip(ms[0].parameters(), ms[1].parameters()):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
            assert same_on_all_ranks(a)
    print('[ok] clip_grad_norm_ norm_type=%s' % norm_type, flush=True)


def poison(g):
    """An inf in one element of rank 0's local gradient, before the hook that launches its reduce-scatter."""
    g = g.clone()
    g.view(-1)[-1] = math.inf
    return g


def check_scaler():
    torch.manual_seed(1)
    m = torch.nn.Sequential(torch.nn.Linear(48, 96), torch.nn.ReLU(), torch.nn.Linear(96, 10)).to(dev).half()
    hvd.broadcast_parameters(m.state_dict(), root_rank=0)
    opt = hvd.DistributedOptimizer(torch.optim.AdamW(m.parameters(), lr=1e-3), named_parameters=m.named_parameters(),
                                   shard_optimizer_state=True, bucket_cap_mb=0.01)
    scaler = hvd.ShardedGradScaler('cuda', init_scale=256.0)
    for step in range(4):
        x, y = batch(step, rank)
        opt.zero_grad()
        before = [p.detach().clone() for p in m.parameters()]
        hook = m[0].weight.register_hook(poison) if step == 1 and rank == 0 else None
        scaler.scale(torch.nn.functional.cross_entropy(m(x.half()), y)).backward()
        if hook is not None:
            hook.remove()
        scaler.unscale_(opt)
        opt.clip_grad_norm_(5.0)
        scaler.step(opt)
        scaler.update()
        torch.cuda.synchronize()
        scale = torch.tensor([scaler.get_scale()], device=dev)
        assert same_on_all_ranks(scale), 'scales differ between ranks'
        changed = any(not torch.equal(a, b) for a, b in zip(before, m.parameters()))
        assert changed == (step != 1), (step, changed)
        assert scaler.get_scale() == (128.0 if step >= 1 else 256.0), scaler.get_scale()
        for p in m.parameters():
            assert same_on_all_ranks(p)
    print('[ok] ShardedGradScaler', flush=True)


check_clip(2.0)
check_clip(math.inf)
check_scaler()
hvd.barrier()
if rank == 0:
    print('SHARDED CLIP OK', flush=True)
hvd.shutdown()
