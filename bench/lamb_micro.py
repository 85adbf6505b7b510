"""One-GPU micro-benchmark of the fused LAMB step against hvd.Lamb.step, the eager per-parameter update.

The parameters have the shapes of BERT-large (horovod_b200.models.bert_large(), 335 M parameters in about 400 tensors),
whose usual pre-training optimizer is LAMB.  Two configurations, each with two arms timed with CUDA events and
alternated round by round:

  fp32         fused   `ops.fused_lamb_step` on fp32 parameters and gradients (three launches);
               eager   `hvd.Lamb.step()` on the same kind of tensors (about a dozen small kernels per parameter);
  bf16-master  fused   the same call on bf16 parameters and gradients with fp32 `master_params`;
               eager   `hvd.Lamb.step()` on the bf16 parameters (fp32 moments, no masters).

Prints one JSON line per arm with ms per step (median over rounds), and for the fused arms the bytes per parameter of
the byte model below, the achieved bytes/s and its share of the H100 SXM's 3.35 TB/s data-sheet bandwidth, plus the GPU
name and power limit read in the same run.

    python bench/lamb_micro.py [--rounds 11] [--iters 10] [--out result.jsonl]
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
from horovod_b200.torch.lamb import Lamb  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# HBM bytes the fused kernels move per parameter element (fp32 = 4 B, bf16 = 2 B); the norm partials are negligible.
#   stage 1 reads p, g, m, v (and the master) and writes m, v; stage 2 reads p, m, v (and the master) and writes p
#   (and the master)
BYTES = {
    'fp32': (4 + 4 + 4 + 4) + (4 + 4) + (4 + 4 + 4) + 4,
    'bf16-master': (2 + 2 + 4 + 4 + 4) + (4 + 4) + (2 + 4 + 4 + 4) + (2 + 4),
}
LR, BETAS, EPS, WD = 1e-3, (0.9, 0.999), 1e-6, 0.01


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


def _arms(shapes, config):
    g = torch.Generator(device='cuda').manual_seed(0)
    rnd = lambda s, scale: torch.randn(s, device='cuda', generator=g) * scale  # noqa: E731
    dt = torch.float32 if config == 'fp32' else torch.bfloat16
    masters = [rnd(s, 0.02) for s in shapes]
    grads = [rnd(s, 1e-3).to(dt) for s in shapes]
    zeros = lambda: [torch.zeros(s, device='cuda') for s in shapes]  # noqa: E731
    params, m, v = [w.to(dt) for w in masters], zeros(), zeros()
    ws = [w.clone() for w in masters] if config != 'fp32' else None

    def fused():
        ops.fused_lamb_step(params, grads, m, v, LR, BETAS[0], BETAS[1], EPS, WD, 10, master_params=ws)

    eager_params = [torch.nn.Parameter(w.to(dt)) for w in masters]
    for p, gr in zip(eager_params, grads):
        p.grad = gr.clone()
    opt = Lamb(eager_params, lr=LR, betas=BETAS, eps=EPS, weight_decay=WD)
    return {'fused': fused, 'eager': opt.step}


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
    p.add_argument('--iters', type=int, default=10)
    p.add_argument('--out', default=None, help='also append the JSON lines to this file')
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA GPU')
    torch.cuda.set_device(0)
    gpu, power = _gpu_info()
    shapes = _shapes()
    numel = sum(int(torch.Size(s).numel()) for s in shapes)
    lines = []
    for config in ('fp32', 'bf16-master'):
        arms = _arms(shapes, config)
        for fn in arms.values():  # warm-up: module loads, the caching allocator
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for r in range(args.rounds):
            for k in (list(arms) if r % 2 == 0 else list(reversed(arms))):
                times[k].append(_time(arms[k], args.iters))
        for k, ts in times.items():
            ms = statistics.median(ts)
            line = {'config': config, 'arm': k, 'model': 'bert-large', 'tensors': len(shapes), 'params': numel,
                    'ms_per_step': round(ms, 3), 'ms_min': round(min(ts), 3), 'ms_max': round(max(ts), 3)}
            if k == 'fused':
                rate = BYTES[config] * numel / (ms * 1e-3)
                line.update({'bytes_per_param': BYTES[config], 'achieved_GBps': round(rate / 1e9, 1),
                             'share_of_3.35TBps': round(rate / HBM_BYTES_PER_S, 3)})
            line.update({'rounds': args.rounds, 'iters': args.iters, 'gpu': gpu, 'power_limit': power})
            lines.append(line)
            print(json.dumps(line), flush=True)
        del arms
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'a') as f:
            for line in lines:
                f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()
