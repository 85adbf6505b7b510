"""Memory and step time of sharded vs unsharded optimizer state (ZeRO-1), per rank.

    torchrun --nproc_per_node 8 bench/sharded_optimizer.py --model bert-large
    hvdrun -np 2 python bench/sharded_optimizer.py --model gpt2-medium
    hvdrun -np 8 python bench/sharded_optimizer.py --model bert-large --master-weights

Builds the model from horovod_b200.models, wraps AdamW in hvd.DistributedOptimizer and trains with bf16 autocast,
alternating `shard_optimizer_state=True` and the unsharded `fused=True` optimizer (fresh model and optimizer each time)
in one run, so both see the same GPUs, clocks and neighbours; with one rank both configurations are the unsharded one.  Prints one JSON line per rank and configuration:
optimizer-state bytes, torch.cuda.max_memory_allocated (above what was allocated before the run) and the device-timed step time (CUDA events around >= 30 steps
after warm-up), plus the GPU name and power limit read in the same run.

--master-weights trains a bf16 model (no autocast) with fp32 master weights (`master_weights=True`) instead, so the
optimizer-state bytes include the masters: 12 B per parameter unsharded, 12 / N B per rank sharded.

Parameters and gradients in registered symmetric memory are VMM allocations made by this library, not by PyTorch's
caching allocator: max_memory_allocated does not count them (in either configuration; the unsharded optimizer keeps its
gradient buckets there too, the sharded one also its parameters).  The optimizer-state bytes are counted directly.
"""
import argparse
import gc
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import horovod_b200.torch as hvd  # noqa: E402
from horovod_b200 import models  # noqa: E402


def _gpu_info(device):
    name = torch.cuda.get_device_name(device)
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(device), '--query-gpu=power.limit', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'unknown'


def _model(name, bs, seq, device, dtype):
    if name == 'bert-large':
        model = models.bert_large().to(device, dtype)
        g = torch.Generator(device=device).manual_seed(hvd.rank())
        ids = torch.randint(0, 30522, (bs, seq), device=device, generator=g)
        labels = torch.where(torch.rand(bs, seq, device=device, generator=g) < 0.15, ids, torch.full_like(ids, -100))
        nsp = torch.randint(0, 2, (bs,), device=device, generator=g)
        return model, lambda: model(ids, labels=labels, next_sentence_label=nsp)
    model = models.gpt2_medium().to(device, dtype)
    g = torch.Generator(device=device).manual_seed(hvd.rank())
    ids = torch.randint(0, 50257, (bs, seq), device=device, generator=g)
    return model, lambda: model(ids, labels=ids)


def _state_bytes(opt):
    if hasattr(opt, '_buckets') and opt._buckets and 'pshard' in opt._buckets[0]:  # sharded: per-bucket shard state
        return sum(t.numel() * t.element_size() for b in opt._buckets for t in b['state'].values())
    return sum(v.numel() * v.element_size() for st in opt.state.values() for v in st.values() if torch.is_tensor(v) and v.is_cuda)


def run(args, sharded, device):
    torch.manual_seed(0)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(device)
    base = torch.cuda.memory_allocated(device)  # whatever earlier runs left behind is not this run's
    model, loss_fn = _model(args.model, args.batch_size, args.seq_len, device,
                            torch.bfloat16 if args.master_weights else torch.float32)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01)
    opt = hvd.DistributedOptimizer(opt, named_parameters=model.named_parameters(), fused=True, shard_optimizer_state=sharded,
                                   master_weights=args.master_weights)

    def step():
        opt.zero_grad()
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=not args.master_weights):
            loss = loss_fn()
        loss.backward()
        opt.step()
        return loss

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    res = {'config': ('sharded' if sharded else 'unsharded fused') + (' + bf16 master weights' if args.master_weights else ''),
           'optimizer_state_bytes': _state_bytes(opt),
           'max_memory_allocated': torch.cuda.max_memory_allocated(device) - base, 'step_ms': round(ms, 3),
           'loss': float(loss)}
    del opt, model, loss_fn
    gc.collect()  # the gradient hooks tie model and optimizer into reference cycles
    torch.cuda.empty_cache()
    return res


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument('--model', default='bert-large', choices=['bert-large', 'gpt2-medium'])
    p.add_argument('--batch-size', type=int, default=None, help='per GPU (default 8 bert-large, 4 gpt2-medium)')
    p.add_argument('--seq-len', type=int, default=None, help='default 512 bert-large, 1024 gpt2-medium')
    p.add_argument('--steps', type=int, default=30)
    p.add_argument('--warmup', type=int, default=5)
    p.add_argument('--rounds', type=int, default=2, help='sharded / unsharded alternations')
    p.add_argument('--master-weights', action='store_true', help='bf16 model with fp32 master weights instead of autocast')
    args = p.parse_args()
    if args.steps < 30:
        p.error('--steps must be >= 30')
    args.batch_size = args.batch_size or (8 if args.model == 'bert-large' else 4)
    args.seq_len = args.seq_len or (512 if args.model == 'bert-large' else 1024)
    hvd.init()
    if not torch.cuda.is_available():
        raise SystemExit('needs CUDA GPUs')
    torch.cuda.set_device(hvd.local_rank())
    device = torch.device('cuda', hvd.local_rank())
    gpu, power = _gpu_info(hvd.local_rank())
    for _ in range(args.rounds):
        for sharded in (True, False):
            res = run(args, sharded, device)
            res.update({'rank': hvd.rank(), 'size': hvd.size(), 'model': args.model, 'batch_size': args.batch_size,
                        'seq_len': args.seq_len, 'steps': args.steps, 'gpu': gpu, 'power_limit': power,
                        'note': 'max_memory_allocated excludes registered (symmetric) parameter / gradient memory'})
            print(json.dumps(res), flush=True)
    hvd.shutdown()


if __name__ == '__main__':
    main()
