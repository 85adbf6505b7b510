"""Gradient accumulation (backward_passes_per_step = 4) on >= 2 GPUs (run under hvdrun), for SGD, AdamW, hvd.Lamb and
hvd.Lars, the unsharded optimizer (zero-copy buckets, allreduce) and the sharded one (reduce-scatter), with a bf16 model,
master weights and the fp32 accumulator, and with an fp32 model:

1. hvd.GraphedStep captures its three graphs with the collectives in the last one (comm_in_graph) and follows the eager
   loop of 4 micro-steps per optimizer step; every rank ends with the same parameters.  Sharded, the eager and the
   captured step issue the same reduce-scatter kernel with the same arguments, so they agree bit for bit.  Unsharded,
   the eager bucket allreduce goes through the engine and the captured one is `captured_allreduce_` with its own CTA
   count, so they are compared to a tolerance.
2. The sharded optimizer follows the unsharded one.
"""
import copy

import torch

import horovod_b200.torch as hvd

hvd.init()
rank, size = hvd.rank(), hvd.size()
torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank())
K = 4


def batch(step, r, dt):
    g = torch.Generator(device=dev).manual_seed(1000 * step + r)
    return torch.randn(8, 48, device=dev, generator=g).to(dt), torch.randint(0, 10, (8,), device=dev, generator=g)


def same_on_all_ranks(t):
    return all(torch.equal(x, t) for x in hvd.allgather(t.detach().reshape(1, -1).float()).unbind(0))


def make(m, shard, dt, kind):
    ps = m.parameters()
    opt = {'sgd': lambda: torch.optim.SGD(ps, lr=0.05, momentum=0.9, weight_decay=1e-4),
           'adamw': lambda: torch.optim.AdamW(ps, lr=1e-2, weight_decay=0.01),
           'lamb': lambda: hvd.Lamb(ps, lr=1e-2, weight_decay=0.01),
           'lars': lambda: hvd.Lars(ps, lr=1.0, momentum=0.9, weight_decay=1e-3, trust_coefficient=0.01)}[kind]()
    return hvd.DistributedOptimizer(opt, named_parameters=m.named_parameters(), master_weights=dt != torch.float32,
                                    fused=True, shard_optimizer_state=shard, bucket_cap_mb=0.01,
                                    backward_passes_per_step=K,
                                    grad_accumulation_dtype=torch.float32 if dt != torch.float32 else None)


def loss_fn(m):
    return lambda x, y: torch.nn.functional.cross_entropy(m(x).float(), y) / K


def eager(m, o, micro_steps, dt):
    for i in micro_steps:
        if i % K == 0:
            o.zero_grad()
        loss_fn(m)(*batch(i, rank, dt)).backward()
        if i % K == K - 1:
            o.step()
    torch.cuda.synchronize()


torch.backends.cudnn.deterministic = True
for kind, dt in [(k, d) for k in ('sgd', 'adamw', 'lamb', 'lars') for d in (torch.bfloat16, torch.float32)]:
    torch.manual_seed(0)
    base = torch.nn.Sequential(torch.nn.Linear(48, 96), torch.nn.ReLU(), torch.nn.Linear(96, 10)).to(dev, dt)
    hvd.broadcast_parameters(base.state_dict(), root_rank=0)
    tol = dict(rtol=1e-2, atol=1e-3) if dt != torch.float32 else dict(rtol=1e-5, atol=1e-6)
    finals = []
    for shard in (False, True):
        mg, me = copy.deepcopy(base), copy.deepcopy(base)
        og, oe = make(mg, shard, dt, kind), make(me, shard, dt, kind)
        gstep = hvd.GraphedStep(loss_fn(mg), og, batch(0, rank, dt))
        assert gstep.captured and gstep.comm_in_graph and len(gstep.graphs) == 3, (gstep.fallback_reason, gstep.comm_in_graph)
        for i in range(4 * K):
            gstep(*batch(i, rank, dt))
        torch.cuda.synchronize()
        eager(me, oe, range(4 * K), dt)
        for a, b in zip(mg.parameters(), me.parameters()):
            assert same_on_all_ranks(a) and same_on_all_ranks(b)
            if shard:
                assert torch.equal(a.detach().reshape(-1).view(torch.uint8), b.detach().reshape(-1).view(torch.uint8))
            else:
                torch.testing.assert_close(a.float(), b.float(), **tol)
        finals.append(me)
        print('[ok] %s %s %s GraphedStep k=%d comm_in_graph' % (kind, dt, 'sharded' if shard else 'unsharded', K), flush=True)
    for a, b in zip(finals[0].parameters(), finals[1].parameters()):
        torch.testing.assert_close(a.float(), b.float(), **tol)
    print('[ok] %s %s sharded follows unsharded' % (kind, dt), flush=True)

hvd.barrier()
if rank == 0:
    print('GRAD ACCUMULATION OK', flush=True)
hvd.shutdown()
