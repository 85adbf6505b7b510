"""One-GPU micro-benchmark of the weight EMA (`hvd.DistributedOptimizer(..., ema_decay=d)`): the EMA written by the fused
update kernel against a user-kept fp32 EMA updated by a separate `torch._foreach_lerp_` pass.

Three arms per configuration, timed with CUDA events and alternated round by round:

  fused    the fused update without EMA (what a step costs today);
  ema      the same launch with `ema_params`: the kernel's epilogue reads and writes the fp32 EMA;
  lerp     the fused update, then `torch._foreach_lerp_(emas, params, 1 - d)` on user-kept fp32 EMAs (for bf16 the
           parameters are first cast to fp32 with `torch._foreach_copy_` into a scratch list, as a user-side fp32 EMA
           of a bf16 model must).

Configurations, with the parameter shapes of the models this project benchmarks:

  resnet50-sgd-fp32         ResNet-50 (161 tensors, 25.6 M parameters), SGD with momentum, fp32 parameters;
  resnet50-sgd-bf16-master  the same on bf16 parameters and gradients with fp32 master weights;
  bert-large-adamw-bf16-master  BERT-large (pre-training heads), AdamW, bf16 parameters with fp32 master weights.

Prints one JSON line per arm with ms per step (median over rounds, min and max), the bytes per parameter of the byte
model below, the achieved bytes/s, and the GPU name and power limit read in the same run.

    python bench/ema_micro.py [--rounds 11] [--iters 20] [--out result.jsonl]
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

DECAY = 0.9999
# HBM bytes per parameter element (fp32 = 4 B, bf16 = 2 B).  SGD: reads p, g, v (and the master), writes p, v (and the
# master).  AdamW: reads p, g, m, v and the master, writes p, m, v and the master.  The EMA epilogue adds one fp32 read
# and one fp32 write (8 B).  The lerp pass reads the EMA and the parameter (fp32: 4 B; bf16: the fp32 copy, made by a cast
# pass that reads 2 B and writes 4 B) and writes the EMA.
UPDATE_BYTES = {
    'resnet50-sgd-fp32': (4 + 4 + 4) + (4 + 4),
    'resnet50-sgd-bf16-master': (2 + 2 + 4 + 4) + (2 + 4 + 4),
    'bert-large-adamw-bf16-master': (2 + 2 + 4 + 4 + 4) + (2 + 4 + 4 + 4),
}
EMA_BYTES = 8
LERP_BYTES = {'fp32': 4 + 4 + 4, 'bf16': (2 + 4) + (4 + 4 + 4)}


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'unknown'


def _shapes(model):
    with torch.device('meta'):
        m = models.resnet50() if model == 'resnet50' else models.bert_large()
        return [tuple(p.shape) for p in m.parameters()]


def _arms(shapes, config):
    g = torch.Generator(device='cuda').manual_seed(0)
    rnd = lambda s, scale: torch.randn(s, device='cuda', generator=g) * scale  # noqa: E731
    low = config.endswith('bf16-master')
    dt = torch.bfloat16 if low else torch.float32
    init = [rnd(s, 0.02) for s in shapes]
    grads = [rnd(s, 1e-3).to(dt) for s in shapes]
    sgd = config.startswith('resnet50')

    def one_arm():
        """Parameters, state and masters of one arm, and its fused update (with or without EMA)."""
        ps = [w.to(dt) for w in init]
        ws = [w.clone() for w in init] if low else None
        if sgd:
            mom = [torch.zeros(s, device='cuda', dtype=torch.float32 if low else dt) for s in shapes]
            return ps, lambda **kw: ops.fused_sgd_step(ps, grads, mom, 0.1, 0.9, weight_decay=5e-5, master_params=ws, **kw)
        m = [torch.zeros(s, device='cuda') for s in shapes]
        v = [torch.zeros(s, device='cuda') for s in shapes]
        return ps, lambda **kw: ops.fused_adam_step(ps, grads, m, v, 1e-4, weight_decay=0.01, step=10, master_params=ws,
                                                    **kw)

    _, fused = one_arm()
    _, ema_update = one_arm()
    ema = [w.clone() for w in init]
    lerp_params, lerp_update = one_arm()
    lerp_ema = [w.clone() for w in init]
    scratch = [torch.empty(s, device='cuda') for s in shapes] if low else None

    def ema_arm():
        ema_update(ema_params=ema, ema_decay=DECAY)

    def lerp_arm():
        lerp_update()
        src = lerp_params
        if scratch is not None:
            torch._foreach_copy_(scratch, lerp_params)
            src = scratch
        torch._foreach_lerp_(lerp_ema, src, 1.0 - DECAY)

    return {'fused': fused, 'ema': ema_arm, 'lerp': lerp_arm}


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
    lines = []
    for config in UPDATE_BYTES:
        shapes = _shapes(config.split('-')[0] if config.startswith('resnet50') else 'bert')
        numel = sum(int(torch.Size(s).numel()) for s in shapes)
        arms = _arms(shapes, config)
        for fn in arms.values():  # warm-up: module loads, the caching allocator
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for r in range(args.rounds):
            for k in (list(arms) if r % 2 == 0 else list(reversed(arms))):
                times[k].append(_time(arms[k], args.iters))
        lerp = LERP_BYTES['bf16' if config.endswith('bf16-master') else 'fp32']
        model_bytes = {'fused': UPDATE_BYTES[config], 'ema': UPDATE_BYTES[config] + EMA_BYTES,
                       'lerp': UPDATE_BYTES[config] + lerp}
        for k, ts in times.items():
            ms = statistics.median(ts)
            rate = model_bytes[k] * numel / (ms * 1e-3)
            line = {'config': config, 'arm': k, 'tensors': len(shapes), 'params': numel, 'ms_per_step': round(ms, 4),
                    'ms_min': round(min(ts), 4), 'ms_max': round(max(ts), 4), 'bytes_per_param': model_bytes[k],
                    'achieved_GBps': round(rate / 1e9, 1), 'rounds': args.rounds, 'iters': args.iters, 'gpu': gpu,
                    'power_limit': power}
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
