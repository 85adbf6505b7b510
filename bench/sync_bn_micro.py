"""One-GPU micro-benchmark of hvd.SyncBatchNorm's local kernels.

For every BatchNorm layer shape of `models.resnet50()` at batch 64, 224x224, channels-last bf16 (collected with
forward hooks), times the native path's local work -- forward: sync_bn_stats + sync_bn_combine + sync_bn_elemt;
backward: sync_bn_backward_reduce + sync_bn_backward_elemt -- against what the torch path of SyncBatchNorm runs on one
rank for the same layer: the `.contiguous()` copies of the input and of grad_output to NCHW, `batch_norm_stats`,
`batch_norm_gather_stats_with_counts` and `batch_norm_elemt`; `batch_norm_backward_reduce` and
`batch_norm_backward_elemt`.  The collectives are not part of either arm.  CUDA events, the two arms alternated per
round, the median over rounds.  The outputs of both arms are compared before timing.

Bytes are what the job needs at least: x read twice and y written in the forward, dy and x read twice and dx written
in the backward (8 passes over a bf16 activation); GB/s and the share of the H100 SXM's 3.35 TB/s data-sheet HBM
bandwidth follow from them.  The GPU name and power limit are read in the same run.

    python bench/sync_bn_micro.py [--batch 64] [--rounds 11] [--iters 10] [--out result.jsonl]
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
EPS = 1e-5


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'unknown'


def bn_shapes(batch):
    """(N, C, H, W) of every BatchNorm input of ResNet-50, with how often each occurs."""
    from horovod_b200.models.resnet import resnet50
    model = resnet50().to(memory_format=torch.channels_last)
    shapes = {}
    hooks = [m.register_forward_hook(lambda m, i, o: shapes.__setitem__(tuple(i[0].shape), shapes.get(tuple(i[0].shape), 0) + 1))
             for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    with torch.no_grad():
        model.eval()(torch.zeros(1, 3, 224, 224).contiguous(memory_format=torch.channels_last))
    for h in hooks:
        h.remove()
    return [((batch,) + s[1:], k) for s, k in sorted(shapes.items(), key=lambda kv: -kv[0][1] * kv[0][2] * kv[0][3])]


def native_arm(x, dy, w, b):
    c = x.size(1)
    per = ops.sync_bn_slot_doubles(c)
    slot = torch.empty(per, dtype=torch.float64, device='cuda')
    sums = torch.empty(2 * c, dtype=torch.float64, device='cuda')

    def run():
        ops.sync_bn_stats(x, slot)
        mean, invstd, count = ops.sync_bn_combine(slot.view(1, per), c, EPS)
        y = ops.sync_bn_elemt(x, mean, invstd, w, b)
        ops.sync_bn_backward_reduce(dy, x, mean, invstd, w, sums, True, True)
        dx = ops.sync_bn_backward_elemt(dy, x, mean, invstd, w, sums, count)
        return y, dx
    return run


def torch_arm(x, dy, w, b):
    def run():
        xc = x.contiguous()
        mean, invstd = torch.batch_norm_stats(xc, EPS)
        count = torch.full((1, 1), xc.numel() // xc.size(1), dtype=xc.dtype, device='cuda')
        mean, invstd = torch.batch_norm_gather_stats_with_counts(xc, mean.unsqueeze(0), invstd.unsqueeze(0), None, None,
                                                                 0.1, EPS, count.view(-1))
        y = torch.batch_norm_elemt(xc, w, b, mean, invstd, EPS)
        dyc = dy.contiguous()
        sum_dy, sum_dy_xmu, _, _ = torch.batch_norm_backward_reduce(dyc, xc, mean, invstd, w, True, True, True)
        dx = torch.batch_norm_backward_elemt(dyc, xc, mean, invstd, w, sum_dy, sum_dy_xmu, count.view(-1).to(torch.int32))
        return y, dx
    return run


def _time(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3 / iters  # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--rounds', type=int, default=11)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('sync_bn_micro: needs a CUDA GPU')
    name, power = _gpu_info()
    lines, tot_native, tot_torch = [], 0.0, 0.0
    for shape, count in bn_shapes(a.batch):
        g = torch.Generator(device='cuda').manual_seed(0)
        x = torch.randn(shape, device='cuda', generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        dy = torch.randn(shape, device='cuda', generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        w = torch.rand(shape[1], device='cuda', generator=g) + 0.5
        b = torch.randn(shape[1], device='cuda', generator=g)
        arms = {'native': native_arm(x, dy, w, b), 'torch': torch_arm(x, dy, w, b)}
        yn, dxn = arms['native']()
        yt, dxt = arms['torch']()
        dy_err = float((yn.float() - yt.float()).abs().max())
        dx_err = float((dxn.float() - dxt.float()).abs().max()) / max(float(dxt.float().abs().max()), 1e-30)
        assert dy_err < 0.1 and dx_err < 0.05, (shape, dy_err, dx_err)
        assert yn.is_contiguous(memory_format=torch.channels_last)
        for fn in arms.values():
            _time(fn, 3)
        times = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                times[k].append(_time(fn, a.iters))
        med = {k: statistics.median(v) for k, v in times.items()}
        nbytes = 8 * x.numel() * x.element_size()
        line = dict(shape=list(shape), layers=count, bytes=nbytes, native_us=round(med['native'], 2),
                    torch_us=round(med['torch'], 2), speedup=round(med['torch'] / med['native'], 3),
                    native_gbps=round(nbytes / med['native'] / 1e3, 1), torch_gbps=round(nbytes / med['torch'] / 1e3, 1),
                    native_hbm_share=round(nbytes / (med['native'] * 1e-6) / HBM_BYTES_PER_S, 3),
                    max_abs_y_diff=dy_err, max_rel_dx_diff=dx_err, gpu=name, power_limit=power)
        tot_native += count * med['native']
        tot_torch += count * med['torch']
        lines.append(line)
        print(json.dumps(line), flush=True)
    summary = dict(model='resnet50', batch=a.batch, dtype='bf16', layout='channels_last', layers=sum(l['layers'] for l in lines),
                   native_us_per_step=round(tot_native, 1), torch_us_per_step=round(tot_torch, 1),
                   speedup=round(tot_torch / tot_native, 3), gpu=name, power_limit=power)
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            for l in lines + [summary]:
                f.write(json.dumps(l) + '\n')


if __name__ == '__main__':
    main()
