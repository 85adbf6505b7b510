#!/usr/bin/env python
"""Host path of a blocking small collective, split with the runtime's own probes (`hvd.metrics()['latency']`: queue = enqueue ->
negotiation start, negotiate = negotiation, execute = data path, total = enqueue -> completion callback).

    hvdrun -np 4 python bench/host_latency.py --out host_latency_np4.json
    HVD_TEST_FAKE_HOSTS=2 hvdrun -np 4 python bench/host_latency.py          # 2 "hosts": two-level control plane, TCP between them

Cases: a cached allreduce (same name every call), an allreduce under a NEW name every call (coordinator round), allgather,
alltoall without and with explicit splits, a cached allreduce inside a 2-rank process set.  CPU tensors of 1 KiB: what is timed is
the engine and the control plane, which are the same for GPU tensors.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument('--iters', type=int, default=2000)
p.add_argument('--out', default=None)
args = p.parse_args()
_fake = int(os.environ.get('HVD_TEST_FAKE_HOSTS', '0'))
if _fake > 1:
    _r, _n = int(os.environ['HOROVOD_RANK']), int(os.environ['HOROVOD_SIZE'])
    _L = _n // _fake
    os.environ.update(HOROVOD_HOSTNAME='fakehost%d' % (_r // _L), HOROVOD_LOCAL_RANK=str(_r % _L), HOROVOD_LOCAL_SIZE=str(_L),
                      HOROVOD_CROSS_RANK=str(_r // _L), HOROVOD_CROSS_SIZE=str(_fake))
import horovod_b200.torch as hvd  # noqa: E402

hvd.init()
rank, size = hvd.rank(), hvd.size()
x = torch.ones(256)
xs = torch.ones(8 * size)
splits = torch.tensor([8] * size, dtype=torch.int32)
ps = hvd.add_process_set([0, 1]) if size > 2 else None
cases = [('allreduce, cached name', lambda: hvd.allreduce_(x, name='lat.cached'), True),
         ('allreduce, new name every call', lambda: hvd.allreduce(x), True),
         ('allgather, cached name', lambda: hvd.allgather(x, name='lat.ag'), True),
         ('alltoall, uniform (no splits)', lambda: hvd.alltoall(xs, name='lat.a2a'), True),
         ('alltoall, explicit splits', lambda: hvd.alltoall(xs, splits=splits, name='lat.a2as'), True)]
if ps is not None:
    cases.append(('allreduce, cached, 2-rank process set', lambda: hvd.allreduce_(x, name='lat.ps', process_set=ps), ps.included()))


def probes():
    m = hvd.metrics()['latency']
    return {k: m[k] for k in m}


rows = []
for label, fn, mine in cases:
    if mine:
        for _ in range(200):
            fn()
    hvd.barrier()
    before = probes()
    t0 = time.perf_counter()
    if mine:
        for _ in range(args.iters):
            fn()
    dt = (time.perf_counter() - t0) / args.iters * 1e6
    after = probes()
    hvd.barrier()
    row = {'case': label, 'us_per_call': round(dt, 1)}
    for part in ('queue', 'negotiate', 'execute', 'total'):
        n = after[part + '_samples'] - before[part + '_samples']
        row[part + '_us'] = round((after[part + '_ns'] - before[part + '_ns']) / max(n, 1) / 1000.0, 1)
    rows.append(row)
    if rank == 0:
        print(json.dumps(row), flush=True)
if rank == 0 and args.out:
    with open(args.out, 'w') as f:
        json.dump({'n_ranks': size, 'fake_hosts': _fake, 'control_plane': hvd.control_plane_info(), 'tensor_bytes': 1024,
                   'timing': 'host wall clock on rank 0 over %d blocking calls; parts from hvd.metrics()' % args.iters, 'rows': rows}, f, indent=1)
hvd.shutdown()
