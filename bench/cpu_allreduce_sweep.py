#!/usr/bin/env python
"""Host-memory allreduce: this runtime's CPU data plane (shared-memory / TCP ring, `csrc/ops/cpu_ops.cc`) next to
torch.distributed's Gloo backend (the reference's CPU data plane is Gloo as well) on the same tensors.

    hvdrun -np 4 python bench/cpu_allreduce_sweep.py --out cpu_allreduce_np4.json

Wall-clock timing (there is no device): `iters` back-to-back calls after warm-up between barriers, max over ranks.
busBW = 2 (N-1)/N * bytes / time.
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
p.add_argument('--sizes', default=','.join(str(1 << s) for s in (10, 14, 18, 20, 22, 24, 26)))
p.add_argument('--out', default=None)
p.add_argument('--no-gloo', action='store_true')
args = p.parse_args()

_fake = int(os.environ.get('HVD_TEST_FAKE_HOSTS', '0'))
if _fake > 1:   # present the ranks of this box as several hosts (multi-host code paths: two-level control / data planes)
    _r, _n = int(os.environ['HOROVOD_RANK']), int(os.environ['HOROVOD_SIZE'])
    _L = _n // _fake
    os.environ.update(HOROVOD_HOSTNAME='fakehost%d' % (_r // _L), HOROVOD_LOCAL_RANK=str(_r % _L), HOROVOD_LOCAL_SIZE=str(_L),
                      HOROVOD_CROSS_RANK=str(_r // _L), HOROVOD_CROSS_SIZE=str(_fake))
hvd.init()
rank, size = hvd.rank(), hvd.size()
if rank == 0:
    print(hvd.control_plane_info(), flush=True)
torch.set_num_threads(max(1, (os.cpu_count() or 4) // size))
if not args.no_gloo:
    dist.init_process_group('gloo', rank=rank, world_size=size,
                            init_method='tcp://127.0.0.1:%d' % (int(os.environ.get('HVD_BENCH_GLOO_PORT', '29611'))))


def timed(fn, nbytes):
    iters = 200 if nbytes <= (1 << 16) else 40 if nbytes <= (1 << 22) else 10
    for _ in range(3):
        fn()
    best = float('inf')
    for _ in range(3):                      # best of 3 rounds: the host clock sees every scheduling hiccup of a shared box
        hvd.barrier()
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        dt = (time.perf_counter() - t0) / iters
        best = min(best, hvd.allreduce(torch.tensor([dt], dtype=torch.float64), op=hvd.Max, name='cpu_sweep.max').item())
    return best


rows = []
for nbytes in [int(s) for s in args.sizes.split(',')]:
    n = nbytes // 4
    x = torch.full((n,), float(rank + 1))
    expect = float(size * (size + 1) // 2)
    out = hvd.allreduce(x, op=hvd.Sum, name='cpu_sweep.check.%d' % nbytes)
    assert torch.all(out == expect)
    t_hvd = timed(lambda: hvd.allreduce_(x, op=hvd.Sum, name='cpu_sweep.%d' % nbytes), nbytes)
    row = {'bytes': nbytes, 'hvd_us': t_hvd * 1e6, 'hvd_busbw_GBps': 2 * (size - 1) / size * nbytes / t_hvd / 1e9}
    if not args.no_gloo:
        y = torch.full((n,), float(rank + 1))
        t_gloo = timed(lambda: dist.all_reduce(y), nbytes)
        row.update(gloo_us=t_gloo * 1e6, gloo_busbw_GBps=2 * (size - 1) / size * nbytes / t_gloo / 1e9, speedup=t_gloo / t_hvd)
    rows.append(row)
    if rank == 0:
        print(json.dumps(row), flush=True)

if rank == 0 and args.out:
    with open(args.out, 'w') as f:
        json.dump({'n_ranks': size, 'dtype': 'fp32', 'timing': 'host wall clock, max over ranks, best of 3 rounds', 'rows': rows}, f, indent=1)
hvd.shutdown()
