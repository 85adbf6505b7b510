"""ResNet-50 synthetic training with the whole forward+backward replayed as one CUDA graph (hvd.GraphedStep).

    bin/hvdrun -np 8 python examples/pytorch_graphed_step.py --batch-size 64 [--max-grad-norm 1.0] [--fp16]

--max-grad-norm clips the global gradient norm before every update; --fp16 trains under fp16 autocast with a
torch.amp.GradScaler (bf16 autocast without one otherwise).
"""
import argparse
import time

import torch
import torch.nn.functional as F

import horovod_b200.torch as hvd
from horovod_b200 import models

p = argparse.ArgumentParser()
p.add_argument('--batch-size', type=int, default=64)
p.add_argument('--steps', type=int, default=50)
p.add_argument('--eager', action='store_true')
p.add_argument('--max-grad-norm', type=float, default=None)
p.add_argument('--fp16', action='store_true')
args = p.parse_args()

hvd.init()
torch.cuda.set_device(hvd.local_rank())
torch.backends.cudnn.benchmark = True
model = models.resnet50().cuda().to(memory_format=torch.channels_last)
opt = hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.01 * hvd.size(), momentum=0.9),
                               named_parameters=model.named_parameters(), fused=True)
hvd.broadcast_parameters(model.state_dict(), root_rank=0)
hvd.broadcast_optimizer_state(opt, root_rank=0)
x = torch.randn(args.batch_size, 3, 224, 224, device='cuda').contiguous(memory_format=torch.channels_last)
y = torch.randint(0, 1000, (args.batch_size,), device='cuda')


def loss_fn(x, y):
    with torch.autocast('cuda', dtype=torch.float16 if args.fp16 else torch.bfloat16):
        return F.cross_entropy(model(x), y)


scaler = torch.amp.GradScaler('cuda') if args.fp16 else None
step = hvd.GraphedStep(loss_fn, opt, (x, y), enabled=not args.eager, max_grad_norm=args.max_grad_norm, scaler=scaler)
if hvd.rank() == 0:
    print('CUDA graph captured:', step.captured, step.fallback_reason or '')
for _ in range(5):
    step(x, y)
torch.cuda.synchronize()
t0 = time.time()
for _ in range(args.steps):
    loss = step(x, y)
torch.cuda.synchronize()
dt = time.time() - t0
if hvd.rank() == 0:
    print('%.1f img/s on %d GPU(s), loss %.3f' % (args.batch_size * hvd.size() * args.steps / dt, hvd.size(), loss.item()))
hvd.shutdown()
