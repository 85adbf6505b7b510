"""Sharded (ZeRO-1) LARS on >= 2 GPUs (run under hvdrun):

1. A bf16 model with master weights, 6 LARS steps: the sharded optimizer follows the unsharded one (allreduce) to
   bf16 accuracy; parameters are bit-identical across ranks, and the small buckets cut parameters between ranks.
2. hvd.GraphedStep with the reduce-scatters inside the graph (comm_in_graph): the trajectory follows the eager sharded one.
3. Checkpoint: the sharded state_dict() loads into an unsharded optimizer and back into a sharded one; the sharded
   runs continue alike.
"""
import copy

import torch

import horovod_b200.torch as hvd

hvd.init()
rank, size = hvd.rank(), hvd.size()
torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank())
DT = torch.bfloat16


def batch(step, r):
    g = torch.Generator(device=dev).manual_seed(1000 * step + r)
    return torch.randn(8, 48, device=dev, generator=g).to(DT), torch.randint(0, 10, (8,), device=dev, generator=g)


def same_on_all_ranks(t):
    return all(torch.equal(x, t) for x in hvd.allgather(t.detach().reshape(1, -1).float()).unbind(0))


def make(m, shard):
    decay = [p for p in m.parameters() if p.dim() == 2]
    rest = [p for p in m.parameters() if p.dim() != 2]
    opt = hvd.Lars([{'params': decay, 'weight_decay': 1e-3}, {'params': rest, 'weight_decay': 0.0}], lr=2.0,
                   momentum=0.9, trust_coefficient=0.01)
    return hvd.DistributedOptimizer(opt, named_parameters=m.named_parameters(), master_weights=True,
                                    shard_optimizer_state=shard, bucket_cap_mb=0.01)


def loss_fn(m):
    return lambda x, y: torch.nn.functional.cross_entropy(m(x).float(), y)


def train(m, o, steps):
    for step in steps:
        x, y = batch(step, rank)
        o.zero_grad()
        loss_fn(m)(x, y).backward()
        o.step()
    torch.cuda.synchronize()


torch.manual_seed(0)
base = torch.nn.Sequential(torch.nn.Linear(48, 96), torch.nn.ReLU(), torch.nn.Linear(96, 10)).to(dev, DT)
hvd.broadcast_parameters(base.state_dict(), root_rank=0)

# 1. trajectory
ms = [copy.deepcopy(base) for _ in range(2)]
opts = [make(ms[0], True), make(ms[1], False)]
assert any(off // b['shard'] != (off + n - 1) // b['shard'] for b in opts[0]._buckets for _, off, n in b['members'])
for step in range(6):
    for m, o in zip(ms, opts):
        train(m, o, [step])
    for a, b in zip(ms[0].parameters(), ms[1].parameters()):
        assert same_on_all_ranks(a)
        torch.testing.assert_close(a.float(), b.float(), rtol=1e-2, atol=1e-3)
print('[ok] sharded trajectory', flush=True)

# 2. GraphedStep with the collectives in the graph against eager sharded steps
mg, me = copy.deepcopy(base), copy.deepcopy(base)
og, oe = make(mg, True), make(me, True)
x0, y0 = batch(0, rank)
gstep = hvd.GraphedStep(loss_fn(mg), og, (x0, y0))
assert gstep.captured and gstep.comm_in_graph, (gstep.fallback_reason, gstep.comm_in_graph)
for step in range(6):
    gstep(*batch(step, rank))
train(me, oe, range(6))
for a, b in zip(mg.parameters(), me.parameters()):
    assert same_on_all_ranks(a)
    torch.testing.assert_close(a.float(), b.float(), rtol=1e-2, atol=1e-3)
print('[ok] GraphedStep comm_in_graph', flush=True)

# 3. checkpoint: sharded -> unsharded -> sharded
sd = opts[0].state_dict()
m2 = copy.deepcopy(ms[0])
o2 = make(m2, False)
o2.load_state_dict(sd)
m3 = copy.deepcopy(ms[0])
o3 = make(m3, True)
o3.load_state_dict(o2.state_dict())
train(ms[0], opts[0], [6])
train(m3, o3, [6])
for a, b in zip(ms[0].parameters(), m3.parameters()):
    assert torch.equal(a, b)
print('[ok] checkpoint', flush=True)

hvd.barrier()
if rank == 0:
    print('LARS OK', flush=True)
hvd.shutdown()
