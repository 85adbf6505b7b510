"""Sharded (ZeRO-1) weight EMA on >= 2 GPUs (run under hvdrun):

1. A bf16 model with master weights and ema_decay, 6 AdamW steps sharded and unsharded (allreduce): the gathered
   sharded EMA follows the unsharded one to fp32 accuracy, and the parameters are bit-identical across ranks.
2. ema_parameters(): every rank holds the same whole EMA model inside the block, and its exact parameters after it.
3. Checkpoint: the sharded state_dict() (with the fp32 EMA) loads into an unsharded optimizer and back into a sharded
   one; the sharded runs continue alike.
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
    opt = torch.optim.AdamW(m.parameters(), lr=1e-2, weight_decay=0.01)
    return hvd.DistributedOptimizer(opt, named_parameters=m.named_parameters(), master_weights=True, ema_decay=0.8,
                                    shard_optimizer_state=shard, bucket_cap_mb=0.01)


def train(m, o, steps):
    for step in steps:
        x, y = batch(step, rank)
        o.zero_grad()
        torch.nn.functional.cross_entropy(m(x).float(), y).backward()
        o.step()
    torch.cuda.synchronize()


torch.manual_seed(0)
base = torch.nn.Sequential(torch.nn.Linear(48, 96), torch.nn.ReLU(), torch.nn.Linear(96, 10)).to(dev, DT)
hvd.broadcast_parameters(base.state_dict(), root_rank=0)

# 1. trajectory
ms = [copy.deepcopy(base) for _ in range(2)]
opts = [make(ms[0], True), make(ms[1], False)]
for step in range(6):
    for m, o in zip(ms, opts):
        train(m, o, [step])
    for a in ms[0].parameters():
        assert same_on_all_ranks(a)
sd = opts[0].state_dict()
for i, p in enumerate(ms[1].parameters()):
    torch.testing.assert_close(sd['state'][i]['ema_param'].to(dev), opts[1].state[p]['ema_param'], rtol=1e-2, atol=1e-3)
print('[ok] sharded EMA', flush=True)

# 2. ema_parameters
before = [p.detach().clone() for p in ms[0].parameters()]
with opts[0].ema_parameters():
    for i, p in enumerate(ms[0].parameters()):
        assert same_on_all_ranks(p)
        assert torch.equal(p.detach(), sd['state'][i]['ema_param'].to(dev).to(DT))
for p, b in zip(ms[0].parameters(), before):
    assert torch.equal(p.detach(), b)
print('[ok] ema_parameters', flush=True)

# 3. checkpoint: sharded -> unsharded -> sharded
m2 = copy.deepcopy(ms[0])
o2 = make(m2, False)
o2.load_state_dict(sd)
m3 = copy.deepcopy(ms[0])
o3 = make(m3, True)
o3.load_state_dict(o2.state_dict())
train(ms[0], opts[0], [6])
train(m3, o3, [6])
sd0, sd3 = opts[0].state_dict(), o3.state_dict()
for i, (a, b) in enumerate(zip(ms[0].parameters(), m3.parameters())):
    assert torch.equal(a, b)
    assert torch.equal(sd0['state'][i]['ema_param'], sd3['state'][i]['ema_param'])
print('[ok] checkpoint', flush=True)

hvd.barrier()
if rank == 0:
    print('EMA OK', flush=True)
hvd.shutdown()
