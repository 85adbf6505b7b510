"""One-GPU measurement of global-norm gradient clipping on the unsharded optimizer and inside hvd.GraphedStep.

(a) The clip itself on the per-parameter gradients of ResNet-50 (161 tensors, 25.6 M elements) and BERT-large (302
    tensors, 336 M elements, one 31 M-element embedding), fp32 and bf16: the fused path of
    `optimizer.clip_grad_norm_` (one `grad_shard_stats` pass that reads every gradient once, then the coefficient
    min(max_norm / (norm + 1e-6), 1) on the device, which the fused update applies) against
    `torch.nn.utils.clip_grad_norm_` (foreach norm, then foreach mul: two reads and one write).  max_norm is large, so
    torch's multiply by 1 leaves the gradients unchanged from call to call.  Reports µs per call, the bytes each arm moves
    and their share of the H100 SXM's 3.35 TB/s data-sheet bandwidth.
(b) The BERT-large training step (seq 512, batch 8, bf16 autocast, fused AdamW) at world size 1: hvd.GraphedStep
    without clipping, hvd.GraphedStep(max_grad_norm=1.0), and the eager loop with torch's clip_grad_norm_.

CUDA events, warm-up, the arms alternated within every round, medians over the rounds; the GPU's name and power limit
are read in the same run.  Prints one JSON line per case.

    python bench/graphed_clip_micro.py [--rounds 11] [--iters 20] [--steps 10] [--out result.jsonl]
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

HBM_BYTES_PER_S = 3.35e12


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'unknown'


def _model(name):
    from horovod_b200 import models
    return models.resnet50() if name == 'resnet50' else models.bert_large()


def _elapsed_us(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3 / iters


def _alternate(arms, rounds, iters, warmup=3):
    for fn in arms.values():
        _elapsed_us(fn, warmup)
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(_elapsed_us(fn, iters))
    return times


def clip_cases(args, gpu, power):
    from horovod_b200 import ops
    for name in ('resnet50', 'bert-large'):
        shapes = [p.shape for p in _model(name).parameters()]
        for dtype in (torch.float32, torch.bfloat16):
            gen = torch.Generator(device='cuda').manual_seed(0)
            grads = [torch.randn(s, device='cuda', generator=gen).to(dtype) for s in shapes]
            nbytes = sum(g.numel() * g.element_size() for g in grads)
            stats = torch.zeros(2, device='cuda')
            max_norm = 1e30

            def fused():
                stats.zero_()
                ops.grad_shard_stats(grads, stats)
                torch.clamp(max_norm / (stats[0].sqrt() + 1e-6), max=1.0)

            def torch_clip():
                total = torch.nn.utils.get_total_norm(grads)
                torch._foreach_mul_(grads, torch.clamp(max_norm / (total + 1e-6), max=1.0))

            times = _alternate({'fused_clip': fused, 'torch_clip': torch_clip}, args.rounds, args.iters)
            res = {'case': 'clip', 'model': name, 'dtype': str(dtype).replace('torch.', ''), 'tensors': len(grads),
                   'grad_mb': round(nbytes / 2 ** 20, 1), 'gpu': gpu, 'power_limit': power}
            for arm, traffic in (('fused_clip', nbytes), ('torch_clip', 3 * nbytes)):
                us = statistics.median(times[arm])
                res[arm] = {'us': round(us, 1), 'us_min': round(min(times[arm]), 1), 'bytes_mb': round(traffic / 2 ** 20, 1),
                            'share_of_3.35TBps': round(traffic / (us * 1e-6) / HBM_BYTES_PER_S, 3)}
            res['speedup'] = round(res['torch_clip']['us'] / res['fused_clip']['us'], 2)
            yield res
            del grads


def bert_step_case(args, gpu, power):
    import horovod_b200.torch as hvd
    bs, seq = 8, 512
    gen = torch.Generator(device='cuda').manual_seed(0)
    ids = torch.randint(0, 30522, (bs, seq), device='cuda', generator=gen)
    labels = torch.where(torch.rand(bs, seq, device='cuda', generator=gen) < 0.15, ids, torch.full_like(ids, -100))
    nsp = torch.randint(0, 2, (bs,), device='cuda', generator=gen)
    batch = (ids, labels, nsp)
    arms = {}
    for arm in ('graphed', 'graphed_clip', 'eager_torch_clip'):
        torch.manual_seed(0)
        model = _model('bert-large').cuda()
        opt = hvd.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01),
                                       named_parameters=model.named_parameters(), fused=True)

        def fwd(*b, model=model):
            with torch.autocast('cuda', dtype=torch.bfloat16):
                return model(b[0], labels=b[1], next_sentence_label=b[2])
        if arm == 'eager_torch_clip':
            def step(model=model, opt=opt, fwd=fwd):
                opt.zero_grad()
                fwd(*batch).backward()
                opt.synchronize()
                torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0)
                with opt.skip_synchronize():
                    opt.step()
        else:
            g = hvd.GraphedStep(fwd, opt, batch, max_grad_norm=1.0 if arm == 'graphed_clip' else None)
            if not g.captured:
                raise SystemExit('GraphedStep did not capture: %s' % g.fallback_reason)
            step = (lambda g=g: g(*batch))
        arms[arm] = step
    times = _alternate(arms, args.rounds, args.steps)
    res = {'case': 'bert-large step', 'seq': seq, 'batch': bs, 'optimizer': 'AdamW (fused)', 'autocast': 'bf16',
           'gpu': gpu, 'power_limit': power}
    for arm, ts in times.items():
        res[arm] = {'ms': round(statistics.median(ts) / 1e3, 3), 'ms_min': round(min(ts) / 1e3, 3)}
    res['clip_cost_pct_of_graphed_step'] = round(100 * (res['graphed_clip']['ms'] / res['graphed']['ms'] - 1), 2)
    yield res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=11)
    ap.add_argument('--iters', type=int, default=20, help='clip calls per timed window')
    ap.add_argument('--steps', type=int, default=10, help='BERT-large steps per timed window')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('graphed_clip_micro needs a GPU')
    import horovod_b200.torch as hvd
    hvd.init()
    torch.cuda.set_device(0)
    gpu, power = _gpu_info()
    lines = []
    for gen in (clip_cases, bert_step_case):
        for res in gen(args, gpu, power):
            print(json.dumps(res), flush=True)
            lines.append(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            for r in lines:
                f.write(json.dumps(r) + '\n')
    hvd.shutdown()


if __name__ == '__main__':
    main()
