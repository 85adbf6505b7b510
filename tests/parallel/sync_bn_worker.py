"""hvd.SyncBatchNorm's native path on >= 2 GPUs (run under hvdrun):

1. A channels-last bf16 conv net converted with convert_sync_batchnorm, unequal per-rank batches: output, input
   gradient and running stats follow torch BatchNorm (fp32) on the allgathered batch, and stay channels-last.
2. hvd.GraphedStep with the gradient allreduces in the graph (comm_in_graph), once with shard_optimizer_state=True:
   SyncBatchNorm's collectives (their own barrier channel) run beside the gradient buckets' ones; after 4 steps the
   parameters and buffers are bit-identical on every rank.
"""
import torch

import horovod_b200.torch as hvd

hvd.init()
rank, size = hvd.rank(), hvd.size()
torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank())
torch.backends.cudnn.deterministic = True


def net():
    torch.manual_seed(0)
    m = torch.nn.Sequential(
        torch.nn.Conv2d(3, 16, 3, padding=1, bias=False), torch.nn.BatchNorm2d(16), torch.nn.ReLU(),
        torch.nn.Conv2d(16, 24, 3, padding=1, bias=False), torch.nn.BatchNorm2d(24), torch.nn.ReLU(),
        torch.nn.AdaptiveAvgPool2d(1), torch.nn.Flatten(), torch.nn.Linear(24, 5))
    return m


def same_on_all_ranks(t):
    return all(torch.equal(x, t) for x in hvd.allgather(t.detach().reshape(1, -1).float()).unbind(0))


# 1. forward / backward against torch BatchNorm on the allgathered batch
bs = 2 + 3 * rank
g = torch.Generator(device=dev).manual_seed(rank)
x = torch.randn(bs, 16, 9, 9, device=dev, generator=g).mul(2).add(1).to(torch.bfloat16)
x = x.contiguous(memory_format=torch.channels_last)
dy = torch.randn(x.shape, device=dev, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
sbn = hvd.SyncBatchNorm(16).to(dev)
xs = x.clone().requires_grad_()
y = sbn(xs)
assert y.is_contiguous(memory_format=torch.channels_last) and y.dtype == torch.bfloat16
y.backward(dy)
xa = hvd.allgather(x.float().contiguous())
dya = hvd.allgather(dy.float().contiguous())
ref = torch.nn.BatchNorm2d(16).to(dev)
xr = xa.clone().requires_grad_()
yr = ref(xr)
yr.backward(dya)
lo = sum(2 + 3 * r for r in range(rank))
torch.testing.assert_close(y.float(), yr[lo:lo + bs].detach(), rtol=2e-2, atol=2e-2)
torch.testing.assert_close(xs.grad.float(), xr.grad[lo:lo + bs], rtol=5e-2, atol=5e-2)
torch.testing.assert_close(sbn.running_mean, ref.running_mean, rtol=1e-4, atol=1e-4)
torch.testing.assert_close(sbn.running_var, ref.running_var, rtol=1e-4, atol=1e-4)
assert same_on_all_ranks(sbn.running_mean) and same_on_all_ranks(sbn.running_var)

# 2. GraphedStep with the collectives in the graph
for shard in (False, True):
    m = hvd.SyncBatchNorm.convert_sync_batchnorm(net()).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9),
                                   named_parameters=m.named_parameters(), fused=True, shard_optimizer_state=shard)
    hvd.broadcast_parameters(m.state_dict(), root_rank=0)
    gx = torch.Generator(device=dev).manual_seed(100 + rank)
    xs = [torch.randn(4 + rank, 3, 10, 10, device=dev, generator=gx).to(torch.bfloat16)
          .contiguous(memory_format=torch.channels_last) for _ in range(4)]
    ys = [torch.randint(0, 5, (4 + rank,), device=dev, generator=gx) for _ in range(4)]
    step = hvd.GraphedStep(lambda a, b: torch.nn.functional.cross_entropy(m(a).float(), b), opt, (xs[0], ys[0]))
    assert step.captured and step.comm_in_graph, (step.fallback_reason, step.comm_in_graph)
    for a, b in zip(xs, ys):
        loss = step(a, b)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    for t in list(m.parameters()) + list(m.buffers()):
        assert same_on_all_ranks(t), 'shard=%s: a parameter or buffer differs across ranks' % shard

hvd.shutdown()
print('sync_bn_worker ok (rank %d of %d)' % (rank, size))
