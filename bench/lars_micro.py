"""One-GPU micro-benchmark of the fused LARS step against hvd.Lars.step, the eager per-parameter update, and against the
fused momentum-SGD step that bench.py's ResNet-50 runs today.

The parameters have the shapes of ResNet-50 (horovod_b200.models.resnet50(), 161 tensors, 25.6 M parameters), whose
large-batch optimizer is LARS.  Two configurations, each with three arms timed with CUDA events and alternated round by
round:

  fp32         lars    `ops.fused_lars_step` on fp32 parameters and gradients (three launches);
               eager   `hvd.Lars.step()` on the same kind of tensors (several small kernels per parameter);
               sgd     `ops.fused_sgd_step` with momentum and weight decay (one launch): what LARS adds over it is the
                       cost of the trust ratios;
  bf16-master  the same three on bf16 parameters and gradients, the fused arms with fp32 `master_params` (the eager arm
               has fp32 momentum and no masters).

Prints one JSON line per arm with ms per step (median over rounds, min and max), and for the fused arms the bytes per
parameter of the byte model below, the achieved bytes/s and its share of the H100 SXM's 3.35 TB/s data-sheet bandwidth,
plus the GPU name and power limit read in the same run.

    python bench/lars_micro.py [--rounds 11] [--iters 20] [--out result.jsonl]
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
from horovod_b200.torch.lars import Lars  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# HBM bytes the fused kernels move per parameter element (fp32 = 4 B, bf16 = 2 B); the norm partials are negligible.
#   LARS: the norms stage reads p, g (and the master); the update reads p, g, v (and the master) and writes p, v (and the
#   master).  SGD: one pass that reads p, g, v (and the master) and writes p, v (and the master).
BYTES = {
    ('fp32', 'lars'): (4 + 4) + (4 + 4 + 4) + (4 + 4),
    ('fp32', 'sgd'): (4 + 4 + 4) + (4 + 4),
    ('bf16-master', 'lars'): (2 + 2 + 4) + (2 + 2 + 4 + 4) + (2 + 4 + 4),
    ('bf16-master', 'sgd'): (2 + 2 + 4 + 4) + (2 + 4 + 4),
}
LR, MOM, WD, TC = 2.0, 0.9, 5e-5, 0.001


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
        return [tuple(p.shape) for p in models.resnet50().parameters()]


def _arms(shapes, config):
    g = torch.Generator(device='cuda').manual_seed(0)
    rnd = lambda s, scale: torch.randn(s, device='cuda', generator=g) * scale  # noqa: E731
    dt = torch.float32 if config == 'fp32' else torch.bfloat16
    masters = [rnd(s, 0.02) for s in shapes]
    grads = [rnd(s, 1e-3).to(dt) for s in shapes]
    zeros = lambda: [torch.zeros(s, device='cuda') for s in shapes]  # noqa: E731
    ws = [w.clone() for w in masters] if config != 'fp32' else None
    lars_p, lars_v = [w.to(dt) for w in masters], zeros()
    sgd_p, sgd_v = [w.to(dt) for w in masters], zeros() if ws else [torch.zeros(s, device='cuda', dtype=dt) for s in shapes]
    sgd_w = [w.clone() for w in masters] if ws else None

    def lars():
        ops.fused_lars_step(lars_p, grads, lars_v, LR, MOM, WD, TC, 0.0, master_params=ws)

    def sgd():
        ops.fused_sgd_step(sgd_p, grads, sgd_v, LR, MOM, weight_decay=WD, master_params=sgd_w)

    eager_params = [torch.nn.Parameter(w.to(dt)) for w in masters]
    for p, gr in zip(eager_params, grads):
        p.grad = gr.clone()
    opt = Lars(eager_params, lr=LR, momentum=MOM, weight_decay=WD, trust_coefficient=TC)
    return {'lars': lars, 'eager': opt.step, 'sgd': sgd}


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
            line = {'config': config, 'arm': k, 'model': 'resnet50', 'tensors': len(shapes), 'params': numel,
                    'ms_per_step': round(ms, 4), 'ms_min': round(min(ts), 4), 'ms_max': round(max(ts), 4)}
            if (config, k) in BYTES:
                rate = BYTES[(config, k)] * numel / (ms * 1e-3)
                line.update({'bytes_per_param': BYTES[(config, k)], 'achieved_GBps': round(rate / 1e9, 1),
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
