"""One-GPU micro-benchmark of gradient accumulation.

(a) `ops.grad_accumulate_` against the torch ops that do the same job, on the bf16 gradient buckets that
    hvd.DistributedOptimizer lays out (32 MB cap, 128 B aligned members) for ResNet-50 (horovod_b200.models.resnet50())
    and BERT-large (horovod_b200.models.bert_large()).  Per mode, both arms over every bucket:

      first   kernel: one launch             torch: acc.copy_(g); g.zero_()      per bucket
      add     kernel: one launch             torch: acc.add_(g); g.zero_()       per bucket
      last    kernel: one launch             torch: g.copy_(acc + g)             per bucket

    Byte model (HBM bytes per element, bf16 g = 2 B, fp32 acc = 4 B): first reads g and writes acc and g (8), add
    reads g and acc and writes acc and g (12), last reads g and acc and writes g (8).

(b) ResNet-50 at batch 64 per micro-batch, bf16 autocast, channels_last, hvd.Lars through hvd.DistributedOptimizer
    (fused), for backward_passes_per_step k = 1, 2, 4, 8: time per image of hvd.GraphedStep (k calls per optimizer
    step) against the eager loop of examples/pytorch_imagenet_resnet50_synthetic.py (zero_grad, k forward/backward
    passes, step).  One process, so the reductions are the identity.

Every arm is timed with CUDA events, arms alternated round by round; one JSON line per arm with the median over
rounds (min and max too), the GPU name and its power limit read in the same run.

    python bench/grad_accumulation_micro.py [--rounds 11] [--iters 20] [--train-rounds 9] [--train-steps 4] [--skip-train] [--out f.jsonl]
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
import torch.nn.functional as F  # noqa: E402

from horovod_b200 import models, ops  # noqa: E402
from horovod_b200.torch.grad_buckets import shard_layout  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BYTES = {'first': 8, 'add': 12, 'last': 8}
CAP = 32 * 1024 * 1024


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'unknown'


def _bucket_numels(make):
    """Element counts of the zero-copy buckets of DistributedOptimizer for the model's parameters in bf16."""
    with torch.device('meta'):
        params = [(p.numel(), torch.bfloat16) for p in make().parameters() if p.requires_grad]
    return [b['numel'] for b in shard_layout([params], 1, CAP)]


def _time(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def _alternate(arms, rounds, iters):
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for r in range(rounds):
        for k in (list(arms) if r % 2 == 0 else list(reversed(arms))):
            times[k].append(_time(arms[k], iters))
    return times


def bench_kernel(args, gpu, power):
    lines = []
    for model, make in (('resnet50', models.resnet50), ('bert-large', models.bert_large)):
        numels = _bucket_numels(make)
        total = sum(numels)
        gen = torch.Generator(device='cuda').manual_seed(0)
        grads = [(torch.randn(n, device='cuda', generator=gen) * 1e-3).to(torch.bfloat16) for n in numels]
        accs = [torch.zeros(n, device='cuda') for n in numels]
        torch_ops = {
            'first': lambda: [(a.copy_(g), g.zero_()) for g, a in zip(grads, accs)],
            'add': lambda: [(a.add_(g), g.zero_()) for g, a in zip(grads, accs)],
            'last': lambda: [g.copy_(a + g) for g, a in zip(grads, accs)],
        }
        for mode in ('first', 'add', 'last'):
            arms = {'kernel': lambda mode=mode: ops.grad_accumulate_(grads, accs, mode), 'torch': torch_ops[mode]}
            times = _alternate(arms, args.rounds, args.iters)
            for arm, ts in times.items():
                ms = statistics.median(ts)
                rate = BYTES[mode] * total / (ms * 1e-3)
                line = {'bench': 'grad_accumulate', 'model': model, 'buckets': len(numels), 'elements': total,
                        'mode': mode, 'arm': arm, 'ms': round(ms, 4), 'ms_min': round(min(ts), 4),
                        'ms_max': round(max(ts), 4), 'bytes_per_element': BYTES[mode],
                        'achieved_GBps': round(rate / 1e9, 1), 'share_of_3.35TBps': round(rate / HBM_BYTES_PER_S, 3),
                        'rounds': args.rounds, 'iters': args.iters, 'gpu': gpu, 'power_limit': power}
                lines.append(line)
                print(json.dumps(line), flush=True)
        del grads, accs
        torch.cuda.empty_cache()
    return lines


def bench_train(args, gpu, power):
    import horovod_b200.torch as hvd
    hvd.init()
    torch.backends.cudnn.benchmark = True
    batch = 64
    lines = []
    for k in (1, 2, 4, 8):
        def build():
            torch.manual_seed(0)
            model = models.resnet50().cuda().to(memory_format=torch.channels_last)
            decay = [q for q in model.parameters() if q.dim() > 1]
            no_decay = [q for q in model.parameters() if q.dim() <= 1]
            opt = hvd.Lars([{'params': decay, 'weight_decay': 5e-5}, {'params': no_decay, 'weight_decay': 0.0}],
                           lr=0.1, momentum=0.9)
            opt = hvd.DistributedOptimizer(opt, named_parameters=model.named_parameters(), fused=True,
                                           backward_passes_per_step=k)

            def loss_fn(x, y):
                with torch.autocast('cuda', dtype=torch.bfloat16):
                    return F.cross_entropy(model(x), y) / k
            return opt, loss_fn

        gen = torch.Generator(device='cuda').manual_seed(1)
        xs = [torch.randn(batch, 3, 224, 224, device='cuda', generator=gen).contiguous(memory_format=torch.channels_last)
              for _ in range(k)]
        ys = [torch.randint(0, 1000, (batch,), device='cuda', generator=gen) for _ in range(k)]
        eager_opt, eager_loss = build()

        def eager():
            eager_opt.zero_grad()
            for x, y in zip(xs, ys):
                eager_loss(x, y).backward()
            eager_opt.step()

        graph_opt, graph_loss = build()
        graphed_step = hvd.GraphedStep(graph_loss, graph_opt, (xs[0], ys[0]))
        if not graphed_step.captured:
            raise SystemExit('GraphedStep did not capture: %s' % graphed_step.fallback_reason)

        def graphed():
            for x, y in zip(xs, ys):
                graphed_step(x, y)

        times = _alternate({'graphed': graphed, 'eager': eager}, args.train_rounds, args.train_steps)
        for arm, ts in times.items():
            ms = statistics.median(ts)
            line = {'bench': 'resnet50_train', 'k': k, 'batch_per_micro_step': batch, 'arm': arm,
                    'ms_per_step': round(ms, 3), 'us_per_image': round(ms * 1e3 / (k * batch), 2),
                    'ms_min': round(min(ts), 3), 'ms_max': round(max(ts), 3), 'rounds': args.train_rounds,
                    'steps_per_round': args.train_steps, 'gpu': gpu, 'power_limit': power}
            lines.append(line)
            print(json.dumps(line), flush=True)
        del graphed_step, graph_opt, graph_loss, eager_opt, eager_loss, xs, ys
        torch.cuda.empty_cache()
    hvd.shutdown()
    return lines


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument('--rounds', type=int, default=11)
    p.add_argument('--iters', type=int, default=20)
    p.add_argument('--train-rounds', type=int, default=9)
    p.add_argument('--train-steps', type=int, default=4, help='optimizer steps per round of (b)')
    p.add_argument('--skip-train', action='store_true')
    p.add_argument('--out', default=None, help='also append the JSON lines to this file')
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA GPU')
    torch.cuda.set_device(0)
    gpu, power = _gpu_info()
    lines = bench_kernel(args, gpu, power)
    if not args.skip_train:
        lines += bench_train(args, gpu, power)
    if args.out:
        with open(args.out, 'a') as f:
            for line in lines:
                f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()
