"""ImageNet-style training program (synthetic data) with everything a long job needs: rank-0 checkpoints and resume by
broadcast, LR warm-up scaled by the number of ranks, gradient accumulation (`backward_passes_per_step`), optional fp16 /
bf16 gradient compression, metric averaging, pinned side-stream input prefetch, and (on GPUs) the CUDA-graph step.
`--optimizer lars` trains with LARS (hvd.Lars, the large-batch optimizer of the MLPerf ResNet-50 reference) instead of
momentum SGD, with BatchNorm and bias parameters excluded from weight decay and trust ratio.

    hvdrun -np 8 python examples/pytorch_imagenet_resnet50_synthetic.py --epochs 3 --checkpoint-format /tmp/ckpt-{epoch}.pt
    hvdrun -np 2 python examples/pytorch_imagenet_resnet50_synthetic.py --no-cuda --model tiny --steps-per-epoch 4 --batch-size 8

Role parity: horovod/examples/pytorch/pytorch_imagenet_resnet50.py (checkpoint / resume pattern :147-154,189-199,280-286).
"""
import argparse
import math
import os

import torch
import torch.nn.functional as F

import horovod_b200.torch as hvd
from horovod_b200 import models
from horovod_b200.data import DevicePrefetcher
from horovod_b200.torch.callbacks import MetricAverage

p = argparse.ArgumentParser()
p.add_argument('--model', default='resnet50', choices=['resnet50', 'tiny'])
p.add_argument('--epochs', type=int, default=3)
p.add_argument('--steps-per-epoch', type=int, default=20)
p.add_argument('--batch-size', type=int, default=32)
p.add_argument('--batches-per-allreduce', type=int, default=1)
p.add_argument('--base-lr', type=float, default=0.0125)
p.add_argument('--warmup-epochs', type=float, default=1.0)
p.add_argument('--momentum', type=float, default=0.9)
p.add_argument('--wd', type=float, default=5e-5)
p.add_argument('--optimizer', default='sgd', choices=['sgd', 'lars'])
p.add_argument('--compression', default='none', choices=['none', 'fp16', 'bf16'])
p.add_argument('--checkpoint-format', default='')
p.add_argument('--no-cuda', action='store_true')
p.add_argument('--no-graph', action='store_true')
p.add_argument('--image-size', type=int, default=224)
args = p.parse_args()

hvd.init()
cuda = not args.no_cuda and torch.cuda.is_available()
if cuda:
    torch.cuda.set_device(hvd.local_rank())
    torch.backends.cudnn.benchmark = True
dev = torch.device('cuda', hvd.local_rank()) if cuda else torch.device('cpu')
torch.manual_seed(1234)
verbose = hvd.rank() == 0

if args.model == 'resnet50':
    model = models.resnet50()
else:
    model = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, stride=4), torch.nn.BatchNorm2d(8), torch.nn.ReLU(),
                                torch.nn.AdaptiveAvgPool2d(1), torch.nn.Flatten(), torch.nn.Linear(8, 1000))
model = model.to(dev)
if cuda:
    model = model.to(memory_format=torch.channels_last)

# ---- resume: rank 0 looks for the newest checkpoint, everyone learns the epoch by broadcast ---------------------------
resume_epoch = 0
if args.checkpoint_format and hvd.rank() == 0:
    for e in range(args.epochs, 0, -1):
        if os.path.exists(args.checkpoint_format.format(epoch=e)):
            resume_epoch = e
            break
resume_epoch = int(hvd.broadcast(torch.tensor(resume_epoch), root_rank=0, name='resume_epoch').item())

lr_scaler = args.batches_per_allreduce * hvd.size()
if args.optimizer == 'lars':
    # BatchNorm weights and biases and every bias (the 1-D parameters) get no weight decay and so no trust ratio
    decay = [q for q in model.parameters() if q.dim() > 1]
    no_decay = [q for q in model.parameters() if q.dim() <= 1]
    opt = hvd.Lars([{'params': decay, 'weight_decay': args.wd}, {'params': no_decay, 'weight_decay': 0.0}],
                   lr=args.base_lr * lr_scaler, momentum=args.momentum)
else:
    opt = torch.optim.SGD(model.parameters(), lr=args.base_lr * lr_scaler, momentum=args.momentum, weight_decay=args.wd)
compression = {'none': hvd.Compression.none, 'fp16': hvd.Compression.fp16, 'bf16': hvd.Compression.bf16}[args.compression]
opt = hvd.DistributedOptimizer(opt, named_parameters=model.named_parameters(), compression=compression,
                               backward_passes_per_step=args.batches_per_allreduce, op=hvd.Average,
                               gradient_predivide_factor=1.0, fused=cuda)
if resume_epoch > 0 and hvd.rank() == 0:
    ckpt = torch.load(args.checkpoint_format.format(epoch=resume_epoch), map_location=dev)
    model.load_state_dict(ckpt['model'])
    opt.load_state_dict(ckpt['optimizer'])
hvd.broadcast_parameters(model.state_dict(), root_rank=0)
hvd.broadcast_optimizer_state(opt, root_rank=0)


def adjust_lr(epoch, step):
    """Linear warm-up from base_lr to base_lr * size over the first epochs, then 10x decays at 30 / 60 / 80."""
    e = epoch + step / args.steps_per_epoch
    if e < args.warmup_epochs:
        factor = 1.0 / hvd.size() * (e * (hvd.size() - 1) / args.warmup_epochs + 1)
    else:
        factor = 10 ** -sum(e >= m for m in (30, 60, 80))
    for g in opt.param_groups:
        g['lr'] = args.base_lr * hvd.size() * args.batches_per_allreduce * factor


class Synthetic:
    """`steps` pinned host batches (a real job would put its DataLoader here, sharded with a DistributedSampler)."""

    def __init__(self, steps, seed):
        self.steps, self.seed = steps, seed

    def __len__(self):
        return self.steps

    def __iter__(self):
        g = torch.Generator().manual_seed(self.seed)
        for _ in range(self.steps):
            x = torch.randn(args.batch_size, 3, args.image_size, args.image_size, generator=g)
            y = torch.randint(0, 1000, (args.batch_size,), generator=g)
            yield (x.pin_memory(), y.pin_memory()) if cuda else (x, y)


def loss_fn(x, y):
    """The loss of one micro-batch, divided by the number of micro-batches per optimizer step."""
    if cuda:
        x = x.contiguous(memory_format=torch.channels_last)
    with torch.autocast('cuda', dtype=torch.bfloat16, enabled=cuda):
        return F.cross_entropy(model(x), y) / args.batches_per_allreduce


# GraphedStep: one call per micro-batch; the optimizer steps after every batches_per_allreduce-th call
use_graph = cuda and not args.no_graph and args.compression == 'none'
step_fn = None
average = MetricAverage(device=dev if cuda else None)
for epoch in range(resume_epoch, args.epochs):
    model.train()
    total, count = 0.0, 0
    loader = Synthetic(args.steps_per_epoch * args.batches_per_allreduce, seed=1000 * epoch + hvd.rank())
    it = iter(DevicePrefetcher(loader, device=dev))
    for step in range(args.steps_per_epoch):
        adjust_lr(epoch, step)
        if use_graph:
            for _ in range(args.batches_per_allreduce):
                x, y = next(it)
                if step_fn is None:
                    step_fn = hvd.GraphedStep(loss_fn, opt, (x, y))
                    if verbose:
                        print('GraphedStep: captured %s, comm_in_graph %s, backward_passes_per_step %d%s'
                              % (step_fn.captured, step_fn.comm_in_graph, step_fn.k,
                                 '' if step_fn.captured else ' (%s)' % step_fn.fallback_reason), flush=True)
                loss = step_fn(x, y)
        else:
            opt.zero_grad()
            for _ in range(args.batches_per_allreduce):
                x, y = next(it)
                loss = loss_fn(x, y)
                loss.backward()
            opt.step()
        total += float(loss.detach())
        count += 1
    logs = average({'loss': total / max(count, 1), 'lr': opt.param_groups[0]['lr']})
    if verbose:
        print('epoch %d: loss %.4f  lr %.5f' % (epoch + 1, logs['loss'], logs['lr']), flush=True)
    if args.checkpoint_format and hvd.rank() == 0:
        torch.save({'model': model.state_dict(), 'optimizer': opt.state_dict(), 'epoch': epoch + 1}, args.checkpoint_format.format(epoch=epoch + 1))
hvd.barrier()
if verbose:
    print('TRAINING DONE (resumed from epoch %d, finite loss: %s)' % (resume_epoch, math.isfinite(logs['loss'])), flush=True)
hvd.shutdown()
