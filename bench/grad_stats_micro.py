"""One-GPU micro-benchmark of the sharded optimizer's gradient statistics pass.

Times `horovod_b200.ops.grad_shard_stats` (one kernel per dtype: in-place unscale + sum of squares + inf/NaN flag in
one read pass) against what torch's GradScaler + clip_grad_norm_ would run on the same tensors,
`torch._foreach_norm` + `torch._amp_foreach_non_finite_check_and_unscale_`, with CUDA events and the two arms
alternated.  torch's unscale kernel has no bf16 version (GradScaler cannot unscale bf16 gradients), so for bf16 the
torch arm unscales with `torch._foreach_mul_` and takes the inf / NaN verdict from the norms instead.  The tensors are
the owned gradient shards of a rank: ResNet-50 (25.6 M parameters) and BERT-large (335 M) split into 32 MB buckets,
each cut into 8 or 2 shards.  Prints one JSON line per case with µs per call, the
arm's own HBM traffic in GB/s, and the share of the H100 SXM's 3.35 TB/s data-sheet bandwidth reached for the bytes
the job needs at least (read and write every element once), plus the GPU name and power limit read in the same run.

    python bench/grad_stats_micro.py [--rounds 15] [--iters 20] [--out result.jsonl]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from horovod_b200 import ops  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
MODELS = {'resnet50': 25_557_032, 'bert-large': 335_141_888}
BUCKET_BYTES = 32 * 1024 * 1024


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'unknown'


def _shards(params, nranks, dtype):
    item = torch.empty(0, dtype=dtype).element_size()
    per_bucket = BUCKET_BYTES // item
    sizes, left = [], params
    while left > 0:
        b = min(left, per_bucket)
        sizes.append((b + nranks - 1) // nranks)
        left -= b
    g = torch.Generator(device='cuda').manual_seed(0)
    return [torch.randn(n, device='cuda', generator=g).to(dtype) for n in sizes]


def _time(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3 / iters  # µs per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=15)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('grad_stats_micro needs a GPU')
    gpu, power = _gpu_info()
    lines = []
    for model, params in MODELS.items():
        for nranks in (8, 2):
            for dtype in (torch.float32, torch.bfloat16):
                shards = _shards(params, nranks, dtype)
                nbytes = sum(t.numel() * t.element_size() for t in shards)
                out = torch.zeros(2, device='cuda')
                one = torch.ones(1, device='cuda')  # inv_scale 1: every call rewrites the same values
                found = torch.zeros(1, device='cuda')

                def ours():
                    out.zero_()
                    ops.grad_shard_stats(shards, out, inv_scale=one)

                def torch_arm():
                    torch._foreach_norm(shards)
                    torch._amp_foreach_non_finite_check_and_unscale_(shards, found, one)

                def torch_arm_bf16():
                    norms = torch._foreach_norm(shards)
                    torch._foreach_mul_(shards, one.reshape(()))
                    found.copy_(torch.stack(norms).isfinite().all().logical_not())

                if dtype == torch.bfloat16:
                    torch_arm = torch_arm_bf16  # noqa: F811

                for fn in (ours, torch_arm):
                    _time(fn, 3)  # warm-up
                t_ours, t_torch = [], []
                for _ in range(args.rounds):
                    t_ours.append(_time(ours, args.iters))
                    t_torch.append(_time(torch_arm, args.iters))
                res = {'model': model, 'nranks': nranks, 'dtype': str(dtype).replace('torch.', ''), 'tensors': len(shards),
                       'shard_mb': round(nbytes / 2 ** 20, 2), 'gpu': gpu, 'power_limit': power,
                       'torch_arm': torch_arm.__name__}
                # own traffic: ours reads + writes once; torch reads for the norm, then reads + writes to unscale
                for arm, ts, traffic in (('stats_kernel', t_ours, 2 * nbytes), ('torch_foreach', t_torch, 3 * nbytes)):
                    us = statistics.median(ts)
                    res[arm] = {'us': round(us, 2), 'us_min': round(min(ts), 2), 'gbps': round(traffic / us / 1e3, 1),
                                'share_of_3.35TBps': round(2 * nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)}
                res['speedup'] = round(res['torch_foreach']['us'] / res['stats_kernel']['us'], 2)
                print(json.dumps(res), flush=True)
                lines.append(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            for r in lines:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
