#!/usr/bin/env python
"""Host-memory allgather / broadcast / reducescatter / alltoall: this runtime's CPU data plane next to torch.distributed's Gloo
backend (the reference's CPU ops run on Gloo or MPI) on the same tensors.

    hvdrun -np 4 python bench/cpu_collective_sweep.py --out cpu_collectives_np4_vs_gloo.json
    HVD_TEST_FAKE_HOSTS=2 hvdrun -np 4 python bench/cpu_collective_sweep.py        # ranks presented as 2 hosts: TCP between them

`bytes` is the size of the RESULT on one rank (allgather: N x input; reducescatter: input / N).  Wall-clock timing, `iters`
back-to-back calls after warm-up between barriers, max over ranks, best of 3 rounds.  Both arms allocate the result of
allgather / reducescatter / alltoall inside the timed call (hvd returns a new tensor; the reference's ops allocate their output
through the framework too), so first-touch page faults of large results are on both sides.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import horovod_b200.torch as hvd  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument('--sizes', default=','.join(str(1 << s) for s in (12, 16, 20, 24, 26)))
p.add_argument('--ops', default='allgather,broadcast,reducescatter,alltoall')
p.add_argument('--out', default=None)
args = p.parse_args()

_fake = int(os.environ.get('HVD_TEST_FAKE_HOSTS', '0'))
if _fake > 1:
    _r, _n = int(os.environ['HOROVOD_RANK']), int(os.environ['HOROVOD_SIZE'])
    _L = _n // _fake
    os.environ.update(HOROVOD_HOSTNAME='fakehost%d' % (_r // _L), HOROVOD_LOCAL_RANK=str(_r % _L), HOROVOD_LOCAL_SIZE=str(_L),
                      HOROVOD_CROSS_RANK=str(_r // _L), HOROVOD_CROSS_SIZE=str(_fake))
hvd.init()
rank, size = hvd.rank(), hvd.size()
if rank == 0:
    print(hvd.control_plane_info(), flush=True)
torch.set_num_threads(max(1, (os.cpu_count() or 4) // size))
dist.init_process_group('gloo', rank=rank, world_size=size,
                        init_method='tcp://127.0.0.1:%d' % (int(os.environ.get('HVD_BENCH_GLOO_PORT', '29612'))))


def timed(fn, nbytes):
    iters = 200 if nbytes <= (1 << 16) else 40 if nbytes <= (1 << 22) else 10
    for _ in range(3):
        fn()
    best = float('inf')
    for _ in range(3):
        hvd.barrier()
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        dt = (time.perf_counter() - t0) / iters
        best = min(best, hvd.allreduce(torch.tensor([dt], dtype=torch.float64), op=hvd.Max, name='ccs.max').item())
    return best


def case(op, nbytes):
    """-> (hvd callable, gloo callable, check callable)"""
    n = nbytes // 4
    if op == 'allgather':
        per = max(1, n // size)
        x = torch.full((per,), float(rank))
        exp = torch.cat([torch.full((per,), float(r)) for r in range(size)])
        return (lambda: hvd.allgather(x, name='ccs.ag.%d' % nbytes), lambda: dist.all_gather(list(torch.empty(per * size).chunk(size)), x),
                lambda: torch.equal(hvd.allgather(x, name='ccs.ag.chk.%d' % nbytes), exp))
    if op == 'broadcast':
        x = torch.full((n,), float(rank))
        return (lambda: hvd.broadcast_(x, 0, name='ccs.bc.%d' % nbytes), lambda: dist.broadcast(x, 0),
                lambda: bool(torch.all(hvd.broadcast(torch.full((n,), float(rank)), size - 1, name='ccs.bc.chk.%d' % nbytes) == size - 1)))
    if op == 'reducescatter':
        per = max(1, n)
        x = torch.full((per * size,), float(rank + 1))
        return (lambda: hvd.reducescatter(x, op=hvd.Sum, name='ccs.rs.%d' % nbytes), lambda: gloo_rs(torch.empty(per), x),
                lambda: bool(torch.all(hvd.reducescatter(x, op=hvd.Sum, name='ccs.rs.chk.%d' % nbytes) == size * (size + 1) / 2)))
    if op == 'alltoall':
        per = max(1, n // size)
        x = torch.full((per * size,), float(rank))
        exp = torch.cat([torch.full((per,), float(r)) for r in range(size)])
        return (lambda: hvd.alltoall(x, name='ccs.a2a.%d' % nbytes), lambda: gloo_a2a(torch.empty(per * size), x, per),
                lambda: torch.equal(hvd.alltoall(x, name='ccs.a2a.chk.%d' % nbytes), exp))
    raise ValueError(op)


def gloo_rs(out, x):
    # Gloo has no reduce_scatter: what a Gloo-based runtime does is allreduce + slice
    y = x.clone()
    dist.all_reduce(y)
    out.copy_(y.chunk(size)[rank])


def gloo_a2a(out, x, per):
    # Gloo has no all_to_all on CPU tensors in every build: gather-based fallback identical in bytes moved per rank
    try:
        dist.all_to_all_single(out, x)
    except Exception:  # noqa: BLE001
        outs = [torch.empty(per * size) for _ in range(size)]
        dist.all_gather(outs, x)
        out.copy_(torch.cat([o[rank * per:(rank + 1) * per] for o in outs]))


rows = []
for op in args.ops.split(','):
    for nbytes in [int(s) for s in args.sizes.split(',')]:
        f_hvd, f_gloo, check = case(op, nbytes)
        assert check(), (op, nbytes)
        t_hvd = timed(f_hvd, nbytes)
        t_gloo = timed(f_gloo, nbytes)
        row = {'op': op, 'bytes': nbytes, 'hvd_us': t_hvd * 1e6, 'gloo_us': t_gloo * 1e6, 'speedup': t_gloo / t_hvd}
        rows.append(row)
        if rank == 0:
            print(json.dumps(row), flush=True)
if rank == 0 and args.out:
    with open(args.out, 'w') as f:
        json.dump({'n_ranks': size, 'dtype': 'fp32', 'fake_hosts': _fake, 'timing': 'host wall clock, max over ranks, best of 3 rounds',
                   'note': 'gloo reducescatter = all_reduce + slice (Gloo has no reduce_scatter); alltoall falls back to all_gather + slice if unsupported',
                   'rows': rows}, f, indent=1)
hvd.shutdown()
