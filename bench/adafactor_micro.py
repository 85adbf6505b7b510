"""One-GPU micro-benchmark of the fused Adafactor update (`ops.fused_adafactor_step`, what
`hvd.DistributedOptimizer(torch.optim.Adafactor(...), fused=True)` runs) against torch.optim.Adafactor.

Three arms per configuration, timed with CUDA events and alternated round by round:

  fused     ops.fused_adafactor_step over the whole model (five launches plus the table upload);
  foreach   torch.optim.Adafactor(foreach=True).step();
  single    torch.optim.Adafactor(foreach=False).step().

Configurations, with the parameter shapes of the transformer models this project benchmarks: BERT-large and
GPT-2-medium, each with fp32 parameters and with bf16 parameters and fp32 master weights (the torch arms have no
masters: they step the bf16 parameters with bf16 state).

Prints one JSON line per arm: ms per step (median over rounds, min and max), host synchronisations per step (counted with
torch.cuda.set_sync_debug_mode('warn')), the extra peak memory of one step over the resident state, for the fused arm
the bytes per parameter of the byte model below and the share of 3.35 TB/s (H100 SXM HBM3) it reaches, and the GPU
name, power limit and max SM clock read in the same run.

    python bench/adafactor_micro.py [--rounds 11] [--iters 10] [--out result.jsonl]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from horovod_b200 import models, ops  # noqa: E402

PEAK_BPS = 3.35e12
# HBM bytes per parameter element of the fused step.  fp32: the stats launch reads g twice (row sums, column partials),
# the norms launch reads w and g, the update reads w and g and writes w: 7 x 4 B.  bf16 with masters: g twice (2 x 2 B),
# then w (2 B), g (2 B) and the master (4 B), then w, g and the master read and the master and w written (14 B).  The
# factors, the variance of vectors and the scratch are O(R + C) per matrix and left out.
FUSED_BYTES = {'fp32': 7 * 4, 'bf16-master': 4 + 8 + 14}
CONFIGS = [('bert-large', 'fp32'), ('bert-large', 'bf16-master'), ('gpt2-medium', 'fp32'), ('gpt2-medium', 'bf16-master')]


def _gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    power, clock = (out.split(', ') + ['unknown', 'unknown'])[:2] if out else ('unknown', 'unknown')
    return torch.cuda.get_device_name(0), power, clock


def _shapes(model):
    with torch.device('meta'):
        m = models.bert_large() if model == 'bert-large' else models.gpt2_medium()
        return [tuple(p.shape) for p in m.parameters()]


def _arms(shapes, prec):
    g = torch.Generator(device='cuda').manual_seed(0)
    dt = torch.bfloat16 if prec == 'bf16-master' else torch.float32
    rnd = lambda s, scale: (torch.randn(s, device='cuda', generator=g) * scale)  # noqa: E731
    init = [rnd(s, 0.02) for s in shapes]
    grads = [rnd(s, 1e-3).to(dt) for s in shapes]
    ps = [x.to(dt) for x in init]
    masters = [x.clone() for x in init] if dt != torch.float32 else None
    rows = [torch.zeros(s[:-1] + (1,), device='cuda') if len(s) >= 2 else None for s in shapes]
    cols = [torch.zeros(s[:-2] + (1, s[-1]), device='cuda') if len(s) >= 2 else None for s in shapes]
    var = [torch.zeros(s, device='cuda') if len(s) < 2 else None for s in shapes]
    step = [0]

    def fused():
        step[0] += 1
        ops.fused_adafactor_step(ps, grads, rows, cols, var, 1e-2, -0.8, None, 1e-3, 1.0, 0.0, step[0],
                                 master_params=masters)

    arms = {'fused': fused}
    for name, foreach in (('foreach', True), ('single', False)):
        tp = [torch.nn.Parameter(x.to(dt)) for x in init]
        for p, gr in zip(tp, grads):
            p.grad = gr
        opt = torch.optim.Adafactor(tp, lr=1e-2, foreach=foreach)
        arms[name] = opt.step
    return arms


def _time(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def _syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    return sum('synchroniz' in str(x.message) for x in w)


def _extra_peak(fn):
    torch.cuda.synchronize()
    resident = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - resident


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument('--rounds', type=int, default=11)
    p.add_argument('--iters', type=int, default=10)
    p.add_argument('--out', default=None, help='also append the JSON lines to this file')
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA GPU')
    torch.cuda.set_device(0)
    gpu, power, clock = _gpu_info()
    lines = []
    for model, prec in CONFIGS:
        shapes = _shapes(model)
        numel = sum(int(torch.Size(s).numel()) for s in shapes)
        arms = _arms(shapes, prec)
        for fn in arms.values():  # warm-up: module loads, the caching allocator, the state of the torch arms
            for _ in range(2):
                fn()
        syncs = {k: _syncs(fn) for k, fn in arms.items()}
        peaks = {k: _extra_peak(fn) for k, fn in arms.items()}
        times = {k: [] for k in arms}
        for r in range(args.rounds):
            for k in (list(arms) if r % 2 == 0 else list(reversed(arms))):
                times[k].append(_time(arms[k], args.iters))
        for k, ts in times.items():
            ms = statistics.median(ts)
            line = {'config': '%s-%s' % (model, prec), 'arm': k, 'tensors': len(shapes), 'params': numel,
                    'ms_per_step': round(ms, 3), 'ms_min': round(min(ts), 3), 'ms_max': round(max(ts), 3),
                    'host_syncs_per_step': syncs[k], 'extra_peak_MB': round(peaks[k] / 2 ** 20, 1),
                    'rounds': args.rounds, 'iters': args.iters, 'gpu': gpu, 'power_limit': power, 'max_sm_clock': clock}
            if k == 'fused':
                rate = FUSED_BYTES[prec] * numel / (ms * 1e-3)
                line.update(bytes_per_param=FUSED_BYTES[prec], achieved_GBps=round(rate / 1e9, 1),
                            share_of_hbm_peak=round(rate / PEAK_BPS, 3))
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
