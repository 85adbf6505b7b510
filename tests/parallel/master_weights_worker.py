"""fp32 master weights with sharded optimizer state on >= 2 GPUs (run under hvdrun):

1. A bf16 model, 6 AdamW steps with `master_weights=True`: the sharded optimizer follows the unsharded one (allreduce)
   to fp32 accuracy in its masters; parameters are bit-identical across ranks.
2. Checkpoint: the sharded state_dict() (masters gathered as fp32) loads into an unsharded master-weights optimizer and
   back into a sharded one; both continue alike.
3. broadcast_parameters from rank 0 after training started: every rank's masters restart from the broadcast values, so
   the ranks stay bit-identical.
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
    return hvd.DistributedOptimizer(torch.optim.AdamW(m.parameters(), lr=1e-3, weight_decay=0.05),
                                    named_parameters=m.named_parameters(), master_weights=True,
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
    w = opts[1].state[p]['master_param']
    assert sd['state'][i]['master_param'].dtype == torch.float32
    torch.testing.assert_close(sd['state'][i]['master_param'].to(dev), w, rtol=1e-4, atol=1e-5)
print('[ok] sharded trajectory', flush=True)

# 2. checkpoint: sharded -> unsharded -> sharded
m2 = copy.deepcopy(ms[0])
o2 = make(m2, False)
o2.load_state_dict(sd)
for i, p in enumerate(m2.parameters()):
    assert torch.equal(o2.state[p]['master_param'].cpu(), sd['state'][i]['master_param'])
m3 = copy.deepcopy(ms[0])
o3 = make(m3, True)
o3.load_state_dict(o2.state_dict())
sd3 = o3.state_dict()
for i in sd['state']:
    for key, t in sd['state'][i].items():
        assert torch.equal(sd3['state'][i][key], t), (i, key)
train(ms[0], opts[0], [6])
train(m3, o3, [6])
for a, b in zip(ms[0].parameters(), m3.parameters()):
    assert torch.equal(a, b)
print('[ok] checkpoint', flush=True)

# 3. broadcast_parameters after training started
with torch.no_grad():
    for p in ms[0].parameters():
        p.add_(0.25 * (rank + 1))  # every rank different ...
hvd.broadcast_parameters(ms[0].state_dict(), root_rank=0)  # ... until rank 0's values arrive
train(ms[0], opts[0], [7, 8])
for a in ms[0].parameters():
    assert same_on_all_ranks(a)
for b in opts[0]._buckets:
    assert same_on_all_ranks(b['pflat'])
print('[ok] broadcast_parameters', flush=True)

hvd.barrier()
if rank == 0:
    print('MASTER WEIGHTS OK', flush=True)
hvd.shutdown()
