"""Micro-benchmark of hvd.captured_alltoall, the alltoall whose splits only the device reads.

(a) One GPU, N = 2, 4, 8 simulated ranks (`horovod_b200.ops.sim`): the captured-alltoall kernel next to sim.alltoallv,
    the engine's planned exchange (pack into the symmetric buffer, flag barrier, pull; planned on the host from host
    splits), on the same rows.  Cases: a mixture-of-experts dispatch of 4096 tokens x top-2 = 8192 rows of 4096 bf16 per
    rank, routed by random expert ids drawn on the device, and an exchange of 4 KiB per rank (64 rows of 64 B).
    Simulated peers are buffers in the same HBM: these numbers describe the count phase, the barriers and the local copy
    rate, not NVLink.  Columns, all from CUDA events:
      captured_graph_us  captured alltoall, per call, from replays of one CUDA graph of --iters calls of every rank (no
                         host work between calls)
      captured_call_us   captured alltoall, one call at a time, each waited for by the host
      planned_call_us    sim.alltoallv, one call at a time: host plan, table upload, launch and wait

(b) >= 2 GPUs (`--multi`, under hvdrun -np N): 4 KiB to 256 MiB per rank, uniform splits, max over ranks of
      captured_alltoall, hvd.alltoall(splits=<device tensor>) (its .cpu() of the splits and negotiation included) and
      torch.distributed.all_to_all_single on NCCL.

The GPU name and power limit are read in the same run.

    python bench/captured_alltoall_micro.py [--iters 20] [--out result.jsonl]
    hvdrun -np 8 python bench/captured_alltoall_micro.py --multi [--out result.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def _gpu_info(device=0):
    name = torch.cuda.get_device_name(device)
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(device), '--query-gpu=power.limit', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'unknown'


def _events_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def moe_splits(n, rows, gen):
    """Rows per destination rank of `rows` tokens routed to random experts, one expert group per rank (device)."""
    expert = torch.randint(0, n, (rows,), device='cuda', generator=gen)
    return torch.bincount(expert, minlength=n).to(torch.int64)


def simulated(iters):
    from horovod_b200.ops import sim
    cases = [('moe 4096 tok x top-2, 4096 bf16', 8192, (4096,), torch.bfloat16, True),
             ('4 KiB per rank', 64, (32,), torch.bfloat16, False)]
    results = []
    for n in (2, 4, 8):
        ctas = min(64, 256 // n)  # every simulated rank's CTAs must be resident at once
        for what, rows, row, dtype, moe in cases:
            gen = torch.Generator(device='cuda').manual_seed(n)
            splits = [moe_splits(n, rows, gen) if moe else torch.full((n,), rows // n, dtype=torch.int64, device='cuda')
                      for _ in range(n)]
            M = [s.tolist() for s in splits]
            cap = max(sum(M[p][q] for p in range(n)) for q in range(n))
            ins = [torch.randn(rows, *row, device='cuda', generator=gen).to(dtype) for _ in range(n)]
            outs = [torch.empty(cap, *row, dtype=dtype, device='cuda') for _ in range(n)]
            outs_ref = [[torch.empty(sum(M[p][q] for p in range(n)), *row, dtype=dtype, device='cuda')] for q in range(n)]
            recv = [torch.empty(n, dtype=torch.int64, device='cuda') for _ in range(n)]
            status = [torch.empty(1, dtype=torch.int32, device='cuda') for _ in range(n)]
            row_bytes = ins[0][0].numel() * ins[0].element_size()
            send_bytes = rows * row_bytes
            buf = max(1 << 20, send_bytes)  # one launch of the planned exchange
            captured = lambda streams=None: sim.captured_alltoall(ins, splits, outs, recv, status, ctas=ctas, streams=streams)  # noqa: E731
            planned = lambda: sim.alltoallv([[x] for x in ins], outs_ref, [M], cap=buf, ctas=ctas)  # noqa: E731
            captured()
            planned()
            torch.cuda.synchronize()
            assert all(int(s) == 0 for s in status)
            for q in range(n):  # both arms moved the same bytes
                k = outs_ref[q][0].shape[0]
                assert torch.equal(outs[q][:k].view(torch.uint8), outs_ref[q][0].view(torch.uint8)), (n, what, q)
            r = dict(part='a', n=n, case=what, rows_per_rank=rows, row_bytes=row_bytes, bytes_per_rank=send_bytes, ctas=ctas,
                     captured_call_us=_events_ms(captured, iters) * 1e3,
                     planned_call_us=_events_ms(planned, iters) * 1e3)
            # last: the graph keeps using this rank count's simulated team, which a larger planned exchange would replace
            streams = [torch.cuda.Stream() for _ in range(n)]
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                cur = torch.cuda.current_stream()
                for s in streams:
                    s.wait_stream(cur)
                for _ in range(iters):
                    captured(streams)
                for s in streams:
                    cur.wait_stream(s)
            g.replay()
            r['captured_graph_us'] = _events_ms(g.replay, 5) * 1e3 / iters
            torch.cuda.synchronize()
            del g
            r['captured_graph_GBps_per_rank'] = send_bytes / (r['captured_graph_us'] * 1e-6) / 1e9
            results.append(r)
            print('N=%d %-34s %9d B/rank  captured in graph %8.1f us  captured call %8.1f us  planned call %8.1f us'
                  % (n, what, send_bytes, r['captured_graph_us'], r['captured_call_us'], r['planned_call_us']), flush=True)
    return results


def multi(iters):
    import torch.distributed as dist
    import horovod_b200.torch as hvd
    hvd.init()
    rank, n = hvd.rank(), hvd.size()
    torch.cuda.set_device(hvd.local_rank())
    port = int(hvd.broadcast_object(29500 + os.getpid() % 1000 if rank == 0 else 0, root_rank=0))
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=n)
    results = []
    row = 1024  # 1 KiB rows of uint8
    for per_rank in [4 << 10, 64 << 10, 1 << 20, 16 << 20, 256 << 20]:
        rows = max(n, per_rank // row) // n * n
        buf = hvd.symm_empty((rows, row), dtype=torch.uint8)
        buf.copy_(torch.randint(0, 256, (rows, row), dtype=torch.uint8, device='cuda'))
        splits = torch.full((n,), rows // n, dtype=torch.int64, device='cuda')
        out = torch.empty(rows, row, dtype=torch.uint8, device='cuda')
        arms = {
            'captured_alltoall': lambda: hvd.captured_alltoall(buf, splits, rows),
            'hvd_alltoall_device_splits': lambda: hvd.alltoall(buf, splits=splits),
            'nccl_all_to_all_single': lambda: dist.all_to_all_single(out, buf, [rows // n] * n, [rows // n] * n),
        }
        r = dict(part='b', n=n, bytes_per_rank=rows * row)
        for name, fn in arms.items():
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            hvd.barrier()
            us = torch.tensor([_events_ms(fn, iters) * 1e3], dtype=torch.float64)
            r[name + '_us'] = float(hvd.allreduce(us, op=hvd.Max))
        results.append(r)
        if rank == 0:
            print(json.dumps(r), flush=True)
    dist.destroy_process_group()
    hvd.shutdown()
    return results if rank == 0 else []


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--multi', action='store_true', help='part (b): run under hvdrun on >= 2 GPUs')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('captured_alltoall_micro needs a CUDA GPU')
    name, power = _gpu_info()
    print('GPU: %s, power limit %s' % (name, power), flush=True)
    results = multi(a.iters) if a.multi else simulated(a.iters)
    for r in results:
        r.update(gpu=name, power_limit=power)
    if a.out and results:
        with open(a.out, 'w') as f:
            for r in results:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
