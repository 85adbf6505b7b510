"""hvd.ExpertDispatcher on >= 2 GPUs (run under hvdrun):

1. eager dispatch, combine and backward with a bf16 layer of 2 experts per rank: expert_in byte for byte equal to a
   reference built from hvd.alltoall(splits=...) and torch indexing, y and grad_x bit for bit equal to the fp32 model;
2. dispatch and combine captured into a torch.cuda.graph, replayed with new router outputs written on the device;
3. an overflow (every token to expert 0 on a dispatcher of small capacity): every rank reports ALLTOALL_RECV_OVERFLOW
   with zero outputs, and the next call works.
"""
import torch

import horovod_b200.torch as hvd
from horovod_b200.torch.mpi_ops import ALLTOALL_RECV_OVERFLOW

hvd.init()
rank, size = hvd.rank(), hvd.size()
torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank())
E, K, H, MAX_T = 2 * size, 2, 40, 128
EL = E // size


def inputs(seed, T):
    g = torch.Generator(device=dev).manual_seed(1000 * seed + rank)
    x = torch.randn(T, H, device=dev, generator=g).to(torch.bfloat16)
    idx = torch.randint(0, E, (T, K), device=dev, generator=g)
    gates = torch.rand(T, K, device=dev, generator=g)
    return x, idx, gates


def reference_expert_in(x, idx):
    flat = idx.flatten()
    order = torch.argsort(flat, stable=True)
    rows = x.repeat_interleave(K, 0)[order]
    counts = torch.bincount(flat, minlength=E)
    recv, _ = hvd.alltoall(rows, splits=counts.view(size, EL).sum(1).cpu())
    rc, _ = hvd.alltoall(counts.view(size, EL).contiguous(), splits=torch.ones(size, dtype=torch.int64))
    rc = rc.tolist()
    seg, at = {}, 0
    for p in range(size):
        for e in range(EL):
            seg[(p, e)] = recv[at:at + rc[p][e]]
            at += rc[p][e]
    return torch.cat([seg[(p, e)] for e in range(EL) for p in range(size)])


def fp32_model(x, gates):
    """y of experts that double their rows, and grad_x for grad_y = 1, as the kernels compute them."""
    y = gx = None
    for j in range(K):
        term = gates[:, j:j + 1] * (x * 2).float()
        y = term if y is None else y + term
        go = (gates[:, j:j + 1] * torch.ones_like(x, dtype=torch.float32)).to(torch.bfloat16)
        t2 = (go * 2).float()
        gx = t2 if gx is None else gx + t2
    return y.to(torch.bfloat16), gx.to(torch.bfloat16)


def check_eager(disp):
    for it in range(3):
        x, idx, gates = inputs(it, 64 + 8 * rank + it)
        x.requires_grad_()
        expert_in, offsets, handle = disp.dispatch(x, idx)
        ref = reference_expert_in(x.detach(), idx)
        assert int(handle.status) == 0, int(handle.status)
        n = ref.shape[0]
        assert torch.equal(expert_in[:n].view(torch.uint8), ref.view(torch.uint8)), ('expert_in', it)
        assert not bool(expert_in[n:].view(torch.uint8).any()) and int(offsets[-1]) == n
        y = disp.combine(expert_in * 2, gates, handle)
        (gx,) = torch.autograd.grad(y, (x,), torch.ones_like(y))
        ry, rgx = fp32_model(x.detach(), gates)
        assert torch.equal(y.view(torch.uint8), ry.view(torch.uint8)), ('y', it)
        assert torch.equal(gx.view(torch.uint8), rgx.view(torch.uint8)), ('grad_x', it)
    print('[ok] eager', flush=True)


def check_graph(disp):
    x, idx, gates = inputs(10, MAX_T)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        expert_in, offsets, handle = disp.dispatch(x, idx)  # warm-up
        disp.combine(expert_in * 2, gates, handle)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        expert_in, offsets, handle = disp.dispatch(x, idx)
        y = disp.combine(expert_in * 2, gates, handle)
    for it in range(3):
        nx, nidx, ngates = inputs(20 + it, MAX_T)
        x.copy_(nx)
        idx.copy_(nidx)
        gates.copy_(ngates)
        graph.replay()
        ry, _ = fp32_model(x, gates)
        assert int(handle.status) == 0
        assert torch.equal(y.view(torch.uint8), ry.view(torch.uint8)), ('replay', it)
    print('[ok] graph', flush=True)


def check_overflow():
    small = hvd.ExpertDispatcher(E, H, torch.bfloat16, MAX_T, K, 64)
    x, idx, gates = inputs(30, 64)
    expert_in, offsets, handle = small.dispatch(x, torch.zeros_like(idx))
    y = small.combine(expert_in * 2, gates, handle)
    statuses = hvd.allgather(handle.status.cpu()).tolist()
    assert statuses == [ALLTOALL_RECV_OVERFLOW] * size, statuses
    assert not bool(expert_in.view(torch.uint8).any()) and not bool(y.view(torch.uint8).any())
    x, idx, gates = inputs(31, 8)
    expert_in, offsets, handle = small.dispatch(x, idx)
    assert int(handle.status) == 0 and int(offsets[-1]) == reference_expert_in(x, idx).shape[0]
    print('[ok] overflow', flush=True)


disp = hvd.ExpertDispatcher(E, H, torch.bfloat16, MAX_T, K, MAX_T * K * size)
check_eager(disp)
check_graph(disp)
check_overflow()
hvd.barrier()
if rank == 0:
    print('MOE WORKER OK', flush=True)
hvd.shutdown()
