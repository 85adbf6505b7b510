"""Fused Adafactor on >= 2 GPUs (run under hvdrun; waits for a multi-GPU run): an fp32 MLP trained 6 steps with
DistributedOptimizer(torch.optim.Adafactor(...), fused=True) on per-rank batches.  The parameters are bit-identical on
every rank and equal a world-size-1 fused run on the averaged gradients (computed here on every rank)."""
import copy

import torch

import horovod_b200.torch as hvd
from horovod_b200 import ops

hvd.init()
rank, size = hvd.rank(), hvd.size()
torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank())


def batch(step, r):
    g = torch.Generator(device=dev).manual_seed(1000 * step + r)
    return torch.randn(8, 24, device=dev, generator=g)


torch.manual_seed(0)
m = torch.nn.Sequential(torch.nn.Linear(24, 48), torch.nn.GELU(), torch.nn.Linear(48, 8)).to(dev)
ref = copy.deepcopy(m)
opt = hvd.DistributedOptimizer(torch.optim.Adafactor(m.parameters(), lr=1e-2, weight_decay=1e-2),
                               named_parameters=m.named_parameters(), fused=True)
state = {}
for step in range(6):
    opt.zero_grad()
    m(batch(step, rank)).square().mean().backward()
    opt.step()
    # the world-size-1 run: every rank's gradient, averaged in fp64 order-independently, then the fused kernel
    grads = []
    for r in range(size):
        ref.zero_grad()
        ref(batch(step, r)).square().mean().backward()
        grads.append([p.grad.double().clone() for p in ref.parameters()])
    avg = [sum(g[i] for g in grads).div(size).float() for i in range(len(grads[0]))]
    ps = list(ref.parameters())
    for p in ps:
        st = state.setdefault(p, {'step': 0})
        st['step'] += 1
        if p.dim() >= 2:
            st.setdefault('row_var', torch.zeros(p.shape[0], 1, device=dev))
            st.setdefault('col_var', torch.zeros(1, p.shape[1], device=dev))
        else:
            st.setdefault('variance', torch.zeros_like(p))
    with torch.no_grad():
        ops.fused_adafactor_step(ps, avg, [state[p].get('row_var') for p in ps], [state[p].get('col_var') for p in ps],
                                 [state[p].get('variance') for p in ps], 1e-2, -0.8, None, 1e-3, 1.0, 1e-2, step + 1)
for (name, p), q in zip(m.named_parameters(), ref.parameters()):
    gathered = hvd.allgather(p.detach().reshape(1, -1))
    assert all(torch.equal(x, gathered[0]) for x in gathered), name
    assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), (name, float((p - q).abs().max()))
print('adafactor_worker OK rank', rank)
