"""One-GPU micro-benchmark of the AdamW update with fp32 master weights for a bf16 model.

The parameters have the shapes of BERT-large (horovod_b200.models.bert_large(), 335 M parameters in about 400 tensors),
stored as bf16 with bf16 gradients.  Three arms, timed with CUDA events and alternated round by round:

  (a) bf16   today's fused AdamW on the bf16 parameters: one `fused_adam_step` launch, fp32 moments;
  (b) master the same launch with `master_params`: the update runs on fp32 masters, the parameters get them rounded;
  (c) torch  what a user writes without this feature: `_foreach_copy_` of the bf16 gradients into fp32 gradient
             buffers, `torch.optim.AdamW(fused=True)` over the fp32 masters, `_foreach_copy_` of the masters into the
             bf16 parameters.

Prints one JSON line per arm with ms per step (median over rounds), the arm's bytes per parameter from the byte model
below, the achieved bytes/s and its share of the H100 SXM's 3.35 TB/s data-sheet bandwidth, plus the GPU name and
power limit read in the same run.

    python bench/master_weights_micro.py [--rounds 11] [--iters 20] [--out result.jsonl]
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

from horovod_b200 import models, ops  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# HBM bytes each arm has to move per parameter element (reads + writes; fp32 = 4 B, bf16 = 2 B)
BYTES = {
    'bf16': 2 + 2 + 4 + 4 + (2 + 4 + 4),            # read p, g, m, v; write p, m, v
    'master': 2 + 2 + 4 + 4 + 4 + (2 + 4 + 4 + 4),  # + read and write the fp32 master (reconcile reads p)
    'torch': (2 + 4) + (4 * 4 + 3 * 4) + (4 + 2),   # copy g in; fused AdamW reads w, g, m, v, writes w, m, v; copy p out
}


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'unknown'


def _shapes():
    with torch.device('meta'):
        return [tuple(p.shape) for p in models.bert_large().parameters()]


def _arms(shapes, lr=1e-4, wd=0.01):
    g = torch.Generator(device='cuda').manual_seed(0)
    rnd = lambda s, scale: torch.randn(s, device='cuda', generator=g) * scale  # noqa: E731
    masters = [rnd(s, 0.02) for s in shapes]
    params = [w.to(torch.bfloat16) for w in masters]
    grads = [rnd(s, 1e-3).to(torch.bfloat16) for s in shapes]
    zeros = lambda: [torch.zeros(s, device='cuda') for s in shapes]  # noqa: E731
    ma, va, mb, vb = zeros(), zeros(), zeros(), zeros()
    pb = [p.clone() for p in params]
    wb = [w.clone() for w in masters]

    def bf16():
        ops.fused_adam_step(params, grads, ma, va, lr, weight_decay=wd, step=10)

    def master():
        ops.fused_adam_step(pb, grads, mb, vb, lr, weight_decay=wd, step=10, master_params=wb)

    wc = [torch.nn.Parameter(w.clone()) for w in masters]
    pc = [p.clone() for p in params]
    for w in wc:
        w.grad = torch.zeros_like(w)
    opt = torch.optim.AdamW(wc, lr=lr, weight_decay=wd, fused=True)
    gc_ = [w.grad for w in wc]

    def torch_arm():
        torch._foreach_copy_(gc_, grads)
        opt.step()
        torch._foreach_copy_(pc, [w.detach() for w in wc])

    return {'bf16': bf16, 'master': master, 'torch': torch_arm}


def _time(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument('--rounds', type=int, default=11)
    p.add_argument('--iters', type=int, default=20)
    p.add_argument('--out', default=None, help='also append the JSON lines to this file')
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA GPU')
    torch.cuda.set_device(0)
    gpu, power = _gpu_info()
    shapes = _shapes()
    numel = sum(int(torch.Size(s).numel()) for s in shapes)
    arms = _arms(shapes)
    for fn in arms.values():  # warm-up: module loads, torch's fused kernels, the caching allocator
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for r in range(args.rounds):
        order = list(arms) if r % 2 == 0 else list(reversed(arms))
        for k in order:
            times[k].append(_time(arms[k], args.iters))
    lines = []
    for k, ts in times.items():
        ms = statistics.median(ts)
        rate = BYTES[k] * numel / (ms * 1e-3)
        lines.append({'arm': k, 'model': 'bert-large', 'tensors': len(shapes), 'params': numel, 'ms_per_step': round(ms, 3),
                      'ms_min': round(min(ts), 3), 'ms_max': round(max(ts), 3), 'bytes_per_param': BYTES[k],
                      'achieved_GBps': round(rate / 1e9, 1), 'share_of_3.35TBps': round(rate / HBM_BYTES_PER_S, 3),
                      'rounds': args.rounds, 'iters': args.iters, 'gpu': gpu, 'power_limit': power})
    for line in lines:
        print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, 'a') as f:
            for line in lines:
                f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()
