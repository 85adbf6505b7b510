#!/usr/bin/env python
"""Bandwidth sweep of the non-allreduce collectives: allgather, broadcast, alltoall, reducescatter.

    torchrun --nproc-per-node 8 bench/collective_sweep.py --out collectives8.json

Every op is timed on the device (CUDA events around `iters` back-to-back calls after warm-up, max over ranks) through
`horovod_b200.torch`, and — with `--nccl` — next to the same op issued through torch.distributed's NCCL backend on the same
tensors (what the reference's NCCL ops boil down to).  Results are value-checked before a number is reported.
algBW = bytes a rank ends up holding (allgather / alltoall / broadcast) or contributes (reducescatter) per second;
busBW uses the nccl-tests factors: (N-1)/N for allgather / reducescatter / alltoall, 1 for broadcast.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import horovod_b200.torch as hvd  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument('--ops', default='allgather,broadcast,alltoall,reducescatter')
p.add_argument('--sizes', default=','.join(str(1 << s) for s in (12, 16, 20, 24, 27)), help='total bytes of the RESULT per rank')
p.add_argument('--device', default='cuda')
p.add_argument('--nccl', action='store_true', help='also time torch.distributed (NCCL) on the same tensors')
p.add_argument('--tag', default='')
p.add_argument('--out', default=None)
args = p.parse_args()

hvd.init()
rank, size = hvd.rank(), hvd.size()
cuda = args.device == 'cuda'
if cuda:
    torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank()) if cuda else torch.device('cpu')
pg = None
if args.nccl and cuda and size > 1:
    # torch.distributed NCCL next to the hvd runtime, bootstrapped through the c10d store hvd.init() already uses (torchrun's
    # agent store) — never a second TCP server
    import torch.distributed as dist
    from horovod_b200.common.basics import _EmbeddedRendezvous
    if _EmbeddedRendezvous.stores:
        from datetime import timedelta
        dist.init_process_group('nccl', store=dist.PrefixStore('collective_sweep', _EmbeddedRendezvous.stores[-1]), rank=rank,
                                world_size=size, device_id=dev, timeout=timedelta(seconds=60))
        pg = dist
    elif rank == 0:
        print('no c10d store (not launched by torchrun): NCCL arm skipped', flush=True)


def timed(fn, iters):
    for _ in range(3):
        fn()
    hvd.barrier()
    if cuda:
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
    else:
        import time
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        ms = (time.perf_counter() - t0) * 1e3 / iters
    return hvd.allreduce(torch.tensor([ms], dtype=torch.float64), op=hvd.Max, name='cs.ms').item()


results = {}
for op in args.ops.split(','):
    rows = []
    for total in [int(s) for s in args.sizes.split(',')]:
        per = max(1, total // size // 4)  # fp32 elements per rank-sized piece
        iters = max(5, min(100, int(2e8 // max(per * size * 4, 1 << 16))))
        factor = 1.0 if op == 'broadcast' else (size - 1) / size
        nbytes = per * size * 4
        if op == 'allgather':
            x = torch.full((per,), float(rank), device=dev)
            out = hvd.allgather(x, name='cs.ag.%d' % total)
            assert out.numel() == per * size and float(out[-1]) == size - 1 and float(out[0]) == 0
            ours = timed(lambda: hvd.allgather(x, name='cs.ag.%d' % total), iters)
            ref = None
            if pg:
                o = torch.empty(per * size, device=dev)
                ref = timed(lambda: pg.all_gather_into_tensor(o, x), iters)
        elif op == 'broadcast':
            x = torch.full((per * size,), float(rank), device=dev)
            hvd.broadcast_(x, root_rank=0, name='cs.bc.%d' % total)
            assert float(x[-1]) == 0
            ours = timed(lambda: hvd.broadcast_(x, root_rank=0, name='cs.bc.%d' % total), iters)
            ref = timed(lambda: pg.broadcast(x, 0), iters) if pg else None
        elif op == 'alltoall':
            x = torch.full((per * size,), float(rank), device=dev)
            out = hvd.alltoall(x, name='cs.a2a.%d' % total)
            assert float(out[0]) == 0 and float(out[-1]) == size - 1
            ours = timed(lambda: hvd.alltoall(x, name='cs.a2a.%d' % total), iters)
            ref = None
            if pg:
                o = torch.empty_like(x)
                ref = timed(lambda: pg.all_to_all_single(o, x), iters)
        elif op == 'reducescatter':
            x = torch.ones(per * size, device=dev)
            out = hvd.reducescatter(x, op=hvd.Sum, name='cs.rs.%d' % total)
            assert out.numel() == per and float(out[0]) == size
            ours = timed(lambda: hvd.reducescatter(x, op=hvd.Sum, name='cs.rs.%d' % total), iters)
            ref = None
            if pg:
                o = torch.empty(per, device=dev)
                ref = timed(lambda: pg.reduce_scatter_tensor(o, x), iters)
        else:
            raise SystemExit('unknown op ' + op)
        row = {'bytes': nbytes, 'us': round(ours * 1e3, 2), 'busbw_gbs': round(nbytes * factor / (ours / 1e3) / 1e9, 2)}
        if ref is not None:
            row.update(nccl_us=round(ref * 1e3, 2), nccl_busbw_gbs=round(nbytes * factor / (ref / 1e3) / 1e9, 2))
        rows.append(row)
    results[op] = rows
    if rank == 0:
        print('== %s%s  [%s]' % (op, ' ' + args.tag if args.tag else '', hvd.gpu_backend_info() if cuda else 'cpu'), flush=True)
        for r in rows:
            extra = '   torch.distributed/NCCL %10.2f us  bus %8.2f GB/s' % (r['nccl_us'], r['nccl_busbw_gbs']) if 'nccl_us' in r else ''
            print('  %12d B  %10.2f us  bus %8.2f GB/s%s' % (r['bytes'], r['us'], r['busbw_gbs'], extra), flush=True)
if rank == 0 and args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    json.dump({'n_gpus': size, 'tag': args.tag, 'results': results},
              open(args.out, 'w'), indent=1)
if pg:
    pg.destroy_process_group()
hvd.shutdown()
