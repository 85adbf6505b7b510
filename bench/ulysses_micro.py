"""Micro-benchmark of hvd.UlyssesExchange, the sequence <-> head exchange of Ulysses sequence parallelism.

(a) One GPU, N = 2, 4, 8 simulated ranks (`horovod_b200.ops.sim`), seq_to_heads of
      gpt2-medium  fused QKV [B=4, S/N, 3, H=16, D=64] bf16 (seq_dim 1, head_dim 3), S = 8192
      7b-long      [B=1, S/N, H=32, D=128] bf16 (seq_dim 1, head_dim 2), S = 32768
    in two arms, each replayed from one CUDA graph of --iters exchanges of every rank:
      fused   the Ulysses kernel: stage, own block straight to the output, pull the peers' blocks
      torch   permute(...).contiguous() into rank-major order, sim.captured_alltoall with uniform splits, permute back
    The outputs of both arms are compared byte for byte before timing.  Columns: us per exchange (all N ranks), and the
    HBM bytes each arm moves by count over that time (per rank and tensor T: fused T read + T written by the stage,
    (N-1)/N T read + written by the pull, so 2 + 2 (N-1) / N T; torch 2 T for each permute and 2 T for the alltoall), against
    the 3.35 TB/s of the H100 SXM data sheet.  Simulated peers are buffers in the same HBM: this is the local copy
    rate, not NVLink.

(b) >= 2 GPUs (`--multi`, under hvdrun -np N): the same shapes per rank, max over ranks of UlyssesExchange.seq_to_heads,
    hvd.alltoall with the permutes, and torch.distributed.all_to_all_single on NCCL with the permutes.

The GPU name and power limit are read in the same run.

    python bench/ulysses_micro.py [--iters 10] [--out result.jsonl]
    hvdrun -np 8 python bench/ulysses_micro.py --multi [--out result.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# name: (per-rank shape for N ranks, seq_dim, head_dim, heads)
SHAPES = {'gpt2-medium': (lambda n: (4, 8192 // n, 3, 16, 64), 1, 3),
          '7b-long': (lambda n: (1, 32768 // n, 32, 128), 1, 2)}


def _gpu_info(device=0):
    name = torch.cuda.get_device_name(device)
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(device), '--query-gpu=power.limit', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'unknown'


def rank_major(x, n, head_dim):
    """[..., H, ...] -> the view [N, ..., H/N, ...]: block q is what goes to rank q."""
    s = list(x.shape)
    return x.view(*s[:head_dim], n, s[head_dim] // n, *s[head_dim + 1:]).movedim(head_dim, 0)


def from_sender_major(y, seq_dim):
    """[N, ..., S/N, ..., H/N, ...] (sender p's block p) -> [..., S, ..., H/N, ...] contiguous."""
    v = y.movedim(0, seq_dim)  # [..., N, S/N, ...]
    s = list(v.shape)
    return v.reshape(*s[:seq_dim], s[seq_dim] * s[seq_dim + 1], *s[seq_dim + 2:])


def _graph_ms(body, iters, replays):
    """ms per iteration of body(), captured `iters` times into one graph and replayed `replays` times."""
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            body()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / (replays * iters)


def simulated(args):
    from horovod_b200.ops import sim
    name, power = _gpu_info()
    rows = []
    for shape_name, (make, seq, head) in SHAPES.items():
        for n in (2, 4, 8):
            shape = make(n)
            ctas = max(8, 128 // n)
            gen = torch.Generator(device='cuda').manual_seed(0)
            xs = [torch.randn(shape, device='cuda', generator=gen).to(torch.bfloat16) for _ in range(n)]
            nbytes = xs[0].numel() * xs[0].element_size()
            staging = [torch.empty(nbytes, dtype=torch.uint8, device='cuda') for _ in range(n)]
            status = [torch.zeros(1, dtype=torch.int32, device='cuda') for _ in range(n)]
            out_s = list(shape)
            out_s[seq] *= n
            out_s[head] //= n
            fused = [torch.empty(out_s, dtype=torch.bfloat16, device='cuda') for _ in range(n)]
            splits = [torch.ones(n, dtype=torch.int64, device='cuda') for _ in range(n)]
            recv = [torch.empty(n, dtype=torch.int64, device='cuda') for _ in range(n)]
            a2a_status = [torch.empty(1, dtype=torch.int32, device='cuda') for _ in range(n)]
            blocks = [rank_major(x, n, head).contiguous() for x in xs]
            got = [torch.empty_like(b) for b in blocks]
            torch_out = [None] * n
            streams = [torch.cuda.Stream() for _ in range(n)]
            # warm-up without streams: creates the simulated team of this N
            sim.ulysses_exchange(xs, fused, seq, head, sim.SEQ_TO_HEADS, status, staging=staging, ctas=ctas)
            sim.captured_alltoall(blocks, splits, got, recv, a2a_status, ctas=ctas)

            def fused_arm():
                cur = torch.cuda.current_stream()
                for s in streams:
                    s.wait_stream(cur)
                sim.ulysses_exchange(xs, fused, seq, head, sim.SEQ_TO_HEADS, status, staging=staging, ctas=ctas, streams=streams)
                for s in streams:
                    cur.wait_stream(s)

            def torch_arm():
                cur = torch.cuda.current_stream()
                for s in streams:
                    s.wait_stream(cur)
                for r in range(n):
                    with torch.cuda.stream(streams[r]):
                        blocks[r].copy_(rank_major(xs[r], n, head))
                sim.captured_alltoall(blocks, splits, got, recv, a2a_status, ctas=ctas, streams=streams)
                for r in range(n):
                    with torch.cuda.stream(streams[r]):
                        torch_out[r] = from_sender_major(got[r], seq)
                for s in streams:
                    cur.wait_stream(s)

            fused_arm()
            torch_arm()
            torch.cuda.synchronize()
            for r in range(n):
                assert torch.equal(fused[r].view(torch.int16), torch_out[r].view(torch.int16)), (shape_name, n, r)
            assert all(int(s) == 0 for s in status) and all(int(s) == 0 for s in a2a_status)
            fused_ms = _graph_ms(fused_arm, args.iters, args.replays)
            torch_ms = _graph_ms(torch_arm, args.iters, args.replays)
            row = {'shape': shape_name, 'nranks': n, 'per_rank_shape': list(shape), 'per_rank_mib': nbytes / 2 ** 20,
                   'ctas': ctas, 'fused_us': fused_ms * 1e3, 'torch_us': torch_ms * 1e3,
                   'fused_hbm_tb_s': (2 + 2 * (n - 1) / n) * n * nbytes / (fused_ms * 1e-3) / 1e12,
                   'torch_hbm_tb_s': 6 * n * nbytes / (torch_ms * 1e-3) / 1e12,
                   'fused_over_torch': fused_ms / torch_ms, 'gpu': name, 'power_limit': power}
            row['fused_share_of_3_35'] = row['fused_hbm_tb_s'] * 1e12 / HBM_BYTES_PER_S
            rows.append(row)
            print(json.dumps(row), flush=True)
            del xs, staging, fused, blocks, got, torch_out
            torch.cuda.empty_cache()
    return rows


def multi(args):
    import torch.distributed as dist
    import horovod_b200.torch as hvd
    hvd.init()
    torch.cuda.set_device(hvd.local_rank())
    n, rank = hvd.size(), hvd.rank()
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', '29533')
    dist.init_process_group('nccl', rank=rank, world_size=n)
    name, power = _gpu_info(hvd.local_rank())
    rows = []
    for shape_name, (make, seq, head) in SHAPES.items():
        shape = make(n)
        x = torch.randn(shape, device='cuda').to(torch.bfloat16)
        ex = hvd.UlyssesExchange(x.numel(), torch.bfloat16)

        def fused():
            return ex.seq_to_heads(x, seq, head)

        def horovod():
            recv = hvd.alltoall(rank_major(x, n, head).contiguous())
            return from_sender_major(recv, seq)

        def nccl():
            send = rank_major(x, n, head).contiguous()
            recv = torch.empty_like(send)
            dist.all_to_all_single(recv, send)
            return from_sender_major(recv, seq)

        ref = fused()
        for arm in (horovod, nccl):
            assert torch.equal(arm().view(torch.int16), ref.view(torch.int16)), arm.__name__
        row = {'shape': shape_name, 'nranks': n, 'per_rank_shape': list(shape), 'gpu': name, 'power_limit': power}
        for arm in (fused, horovod, nccl):
            for _ in range(3):
                arm()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                arm()
            e1.record()
            e1.synchronize()
            t = torch.tensor([e0.elapsed_time(e1) / args.iters * 1e3])
            row[arm.__name__ + '_us'] = float(hvd.allreduce(t, op=hvd.Max))
        if rank == 0:
            rows.append(row)
            print(json.dumps(row), flush=True)
    hvd.shutdown()
    return rows


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--iters', type=int, default=10)
    p.add_argument('--replays', type=int, default=5)
    p.add_argument('--multi', action='store_true')
    p.add_argument('--out')
    args = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit('ulysses_micro: needs a GPU')
    rows = multi(args) if args.multi else simulated(args)
    if args.out and rows:
        with open(args.out, 'w') as f:
            for r in rows:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
