"""SyncBatchNorm: batch statistics computed over the whole (global) batch.

Native path (CUDA input of fp32 / bf16 / fp16 in training, more than one rank on one NVLink domain): per layer four
launches on the current stream in the forward -- this rank's count / mean / M2 per channel into its slot of a
registered buffer, a captured allgather of the slots, a rank-order combine (which also updates the running stats on
the device), the normalization -- and three in the backward.  No negotiation, no host synchronisation, the input's
layout (channels-last or contiguous) is kept, so a model with SyncBatchNorm can be one hvd.GraphedStep replay.

Otherwise (CPU, one rank, eval, the NCCL backend, several hosts, elastic, fp64): the forward allgathers per-rank
(count, mean, invstd) and combines them with torch.batch_norm_gather_stats_with_counts; the backward allreduces sum_dy
and sum_dy_xmu.  API parity: horovod/torch/sync_batch_norm.py."""
import torch
import torch.nn.functional as F
from torch.autograd.function import Function
from torch.nn.modules.batchnorm import _BatchNorm

from horovod_b200 import ops
from horovod_b200.torch.mpi_ops import (Sum, _native, allgather_async, allreduce_async, global_process_set, local_size,
                                        rank, size, symm_available, symm_empty, synchronize)

_NATIVE_DTYPES = (torch.float32, torch.bfloat16, torch.float16)
_SYNC_BN_CHANNEL = 4  # kSyncBnChannel: barrier flags of their own, apart from the gradient buckets' (p2p_kernels.h)


class SyncBatchNorm(_BatchNorm):
    """Applies synchronous batch normalization (convert a model with SyncBatchNorm.convert_sync_batchnorm(model)):
    identical to torch.nn.BatchNormNd in eval mode and at size() == 1."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True):
        super().__init__(num_features, eps, momentum, affine, track_running_stats)

    def _check_input_dim(self, input):
        if input.dim() < 2:
            raise ValueError('expected at least 2D input (got {}D input)'.format(input.dim()))

    def _run_bn(self, input, factor):
        return F.batch_norm(input, self.running_mean, self.running_var, self.weight, self.bias,
                            self.training or not self.track_running_stats, factor, self.eps)

    @torch.jit.unused
    def _maybe_run_sync_bn(self, input, factor):
        if size() == 1:
            return self._run_bn(input, factor)
        return _SyncBatchNorm.apply(input, self.weight, self.bias, self.running_mean, self.running_var, self.eps, factor)

    @classmethod
    def convert_sync_batchnorm(cls, module):
        """Returns `module` with every torch BatchNorm layer (any `_BatchNorm`) replaced by a SyncBatchNorm that shares
        its affine parameters and buffers, so dtype, device and values are kept (as torch.nn.SyncBatchNorm's method)."""
        out = module
        if isinstance(module, _BatchNorm):
            out = cls(module.num_features, module.eps, module.momentum, module.affine, module.track_running_stats)
            if module.affine:
                with torch.no_grad():
                    out.weight = module.weight
                    out.bias = module.bias
            out.running_mean = module.running_mean
            out.running_var = module.running_var
            out.num_batches_tracked = module.num_batches_tracked
            out.training = module.training
            if hasattr(module, 'qconfig'):
                out.qconfig = module.qconfig
        for name, child in module.named_children():
            out.add_module(name, cls.convert_sync_batchnorm(child))
        return out

    def _native_ok(self, input):
        if not (input.is_cuda and input.dtype in _NATIVE_DTYPES and (self.training or not self.track_running_stats)):
            return False
        for t in (self.weight, self.bias, self.running_mean, self.running_var):
            if t is not None and (t.dtype not in (torch.float32, input.dtype) or t.device != input.device):
                return False
        return True

    def forward(self, input):
        self._check_input_dim(input)
        world = _native_world() if self._native_ok(input) else None
        if world is not None:
            return self._native_forward(input, *world)
        # exponential averaging factor as in torch.nn.modules.batchnorm._BatchNorm.forward: momentum=None means a cumulative
        # moving average over the batches seen so far
        factor = 0.0 if self.momentum is None else self.momentum
        if self.training and self.track_running_stats:
            self.num_batches_tracked = self.num_batches_tracked + 1
            if self.momentum is None:
                factor = 1.0 / float(self.num_batches_tracked)
        if not self.training and self.track_running_stats:
            return self._run_bn(input, factor)
        if not input.is_cuda and size() > 1:
            return _SyncBatchNormCPU.apply(input, self.weight, self.bias, self.running_mean, self.running_var, self.eps, factor)
        return self._maybe_run_sync_bn(input, factor)

    def _native_forward(self, input, nranks, my_rank):
        nbt = None
        if self.training and self.track_running_stats:
            self.num_batches_tracked.add_(1)  # in place: a captured graph keeps counting on replay
            if self.momentum is None:
                nbt = self.num_batches_tracked  # the kernel reads 1 / num_batches_tracked on the device
        momentum = 0.0 if self.momentum is None else self.momentum
        rm, rv = (self.running_mean, self.running_var) if self.track_running_stats else (None, None)
        return _SyncBatchNormNative.apply(input, self.weight, self.bias, rm, rv, nbt, self.eps, momentum, nranks, my_rank)


class _SyncBatchNorm(Function):
    @staticmethod
    def forward(self, input, weight, bias, running_mean, running_var, eps, momentum):
        input = input.contiguous()
        size_ = input.numel() // input.size(1)
        count = torch.tensor([size_], device=input.device, dtype=torch.float32)
        mean, invstd = torch.batch_norm_stats(input, eps)
        count_handle = allgather_async(count.unsqueeze(0), name='sync_batch_norm.count')
        mean_handle = allgather_async(mean.unsqueeze(0), name='sync_batch_norm.mean')
        invstd_handle = allgather_async(invstd.unsqueeze(0), name='sync_batch_norm.invstd')
        count_all = synchronize(count_handle)
        mean_all = synchronize(mean_handle)
        invstd_all = synchronize(invstd_handle)
        counts = count_all.view(-1).float()
        mean, invstd = torch.batch_norm_gather_stats_with_counts(input, mean_all, invstd_all, running_mean, running_var,
                                                                 momentum, eps, counts)
        self.save_for_backward(input, weight, mean, invstd, count_all)
        return torch.batch_norm_elemt(input, weight, bias, mean, invstd, eps)

    @staticmethod
    def backward(self, grad_output):
        grad_output = grad_output.contiguous()
        saved_input, weight, mean, invstd, count_all = self.saved_tensors
        need_input_grad, need_weight_grad, need_bias_grad = self.needs_input_grad[0:3]
        sum_dy, sum_dy_xmu, grad_weight, grad_bias = torch.batch_norm_backward_reduce(
            grad_output, saved_input, mean, invstd, weight, need_input_grad, need_weight_grad, need_bias_grad)
        if need_input_grad:
            sum_dy_handle = allreduce_async(sum_dy, op=Sum, name='sync_batch_norm.sum_dy')
            sum_dy_xmu_handle = allreduce_async(sum_dy_xmu, op=Sum, name='sync_batch_norm.sum_dy_xmu')
            sum_dy = synchronize(sum_dy_handle)
            sum_dy_xmu = synchronize(sum_dy_xmu_handle)
            counts = count_all.view(-1).to(torch.int32)
            grad_input = torch.batch_norm_backward_elemt(grad_output, saved_input, mean, invstd, weight, sum_dy,
                                                         sum_dy_xmu, counts)
        else:
            grad_input = None
        if weight is None or not need_weight_grad:
            grad_weight = None
        if weight is None or not need_bias_grad:
            grad_bias = None
        return grad_input, grad_weight, grad_bias, None, None, None, None, None, None


class _SyncBatchNormCPU(Function):
    """Host fallback (the ATen batch_norm_stats kernels are CUDA-only): same math with plain tensor ops."""

    @staticmethod
    def forward(ctx, input, weight, bias, running_mean, running_var, eps, momentum):
        dims = [0] + list(range(2, input.dim()))
        n_local = input.numel() // input.size(1)
        local_sum = input.sum(dims)
        local_sqsum = (input * input).sum(dims)
        stats = torch.cat([local_sum, local_sqsum, torch.tensor([float(n_local)], dtype=input.dtype)])
        stats = synchronize(allreduce_async(stats, op=Sum, name='sync_batch_norm.cpu_stats'))
        c = input.size(1)
        n = stats[-1]
        mean = stats[:c] / n
        var = stats[c:2 * c] / n - mean * mean
        invstd = torch.rsqrt(var + eps)
        if running_mean is not None:
            running_mean.mul_(1 - momentum).add_(momentum * mean)
            unbiased = var * n / (n - 1) if float(n) > 1 else var  # a single sample has no unbiased estimate
            running_var.mul_(1 - momentum).add_(momentum * unbiased)
        shape = [1, c] + [1] * (input.dim() - 2)
        xhat = (input - mean.view(shape)) * invstd.view(shape)
        ctx.save_for_backward(xhat, weight, invstd, n)
        out = xhat
        if weight is not None:
            out = out * weight.view(shape)
        if bias is not None:
            out = out + bias.view(shape)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        xhat, weight, invstd, n = ctx.saved_tensors
        c = xhat.size(1)
        dims = [0] + list(range(2, xhat.dim()))
        shape = [1, c] + [1] * (xhat.dim() - 2)
        grad_bias = grad_output.sum(dims)
        grad_weight = (grad_output * xhat).sum(dims)
        both = synchronize(allreduce_async(torch.cat([grad_bias, grad_weight]), op=Sum, name='sync_batch_norm.cpu_bwd'))
        sum_dy, sum_dy_xhat = both[:c], both[c:]
        g = grad_output * (weight.view(shape) if weight is not None else 1.0)
        w = weight if weight is not None else torch.ones(c, dtype=xhat.dtype)
        grad_input = (g - (w * sum_dy / n).view(shape) - xhat * (w * sum_dy_xhat / n).view(shape)) * invstd.view(shape)
        return grad_input, grad_weight if weight is not None else None, grad_bias, None, None, None, None


# ---- native path -----------------------------------------------------------------------------------------------------
# One registered region per device (global process set) serves every SyncBatchNorm layer: the forward uses its first
# nranks * slot bytes (rank r's slot at r * slot), the backward its first 16 * C bytes.  Reusing it is safe by stream
# order alone:
#  * a captured collective completes on a rank only after every peer made its last access to that rank's region
#    (docs/kernels.md), so when a layer's stats kernel overwrites this rank's slot no peer still reads the previous one;
#  * each layer's combine (or backward elemt) reads the region before the next layer's stats (or backward reduce) kernel,
#    later on the same stream, writes it;
#  * a peer's next collective can store into this rank's copy only after its barrier A, which this rank passes only
#    after its previous combine.
# The region grows to the largest C seen, on the first training forward that needs more room: every rank runs the same
# forward, so the collective allocations match.  Outgrown regions are kept alive, as a captured graph may refer to them.
_regions = {}
_outgrown = []


def _native_world():
    """(size, rank) when the native path can run: more than one rank, all on this host, registered memory available;
    else None."""
    n = size()
    if n is None or n <= 1 or local_size() != n or not symm_available():
        return None
    return n, rank()


def _registered(nbytes, device):
    """A registered uint8 region of at least `nbytes` on `device`, shared by every layer."""
    buf = _regions.get(device)
    if buf is None or buf.numel() < nbytes:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('hvd.SyncBatchNorm: the registered statistics buffer would have to grow to %d bytes during '
                               'CUDA graph capture; run the step eagerly once before capturing it' % nbytes)
        if buf is not None:
            _outgrown.append(buf)
        size_ = 4096
        while size_ < nbytes:
            size_ *= 2
        buf = symm_empty(size_, dtype=torch.uint8, device=device)
        _regions[device] = buf
    return buf


def _allgather_slots(buf):
    """Every rank's contiguous 1/N of `buf` (a registered uint8 view) into every peer's copy, on the current stream."""
    _native().captured_allgather_(buf, global_process_set.process_set_id, 0, channel=_SYNC_BN_CHANNEL)


def _allreduce_sums(buf):
    """In-place sum of a registered float64 view over the ranks, on the current stream."""
    _native().captured_allreduce_(buf, int(Sum), 1.0, 1.0, global_process_set.process_set_id, 0, channel=_SYNC_BN_CHANNEL)


def _kernel_view(x):
    """x when the kernels read it in place (channels innermost, or contiguous), else a contiguous copy."""
    if x.is_contiguous():
        return x
    expect = 1
    for k in [1] + list(range(x.dim() - 1, 1, -1)) + [0]:
        if x.size(k) != 1 and x.stride(k) != expect:
            return x.contiguous()
        expect *= x.size(k)
    return x


class _SyncBatchNormNative(Function):
    @staticmethod
    def forward(ctx, input, weight, bias, running_mean, running_var, num_batches_tracked, eps, momentum, nranks, my_rank):
        x = _kernel_view(input)
        c = x.size(1)
        per = ops.sync_bn_slot_doubles(c)
        region = _registered(nranks * per * 8, x.device)
        gathered = region[:nranks * per * 8]
        slots = gathered.view(torch.float64).view(nranks, per)
        ops.sync_bn_stats(x, slots[my_rank])
        _allgather_slots(gathered)
        mean, invstd, count = ops.sync_bn_combine(slots, c, eps, momentum, running_mean, running_var, num_batches_tracked)
        y = ops.sync_bn_elemt(x, mean, invstd, weight, bias)
        ctx.save_for_backward(x, weight, mean, invstd, count)
        return y

    @staticmethod
    def backward(ctx, grad_output):
        x, weight, mean, invstd, count = ctx.saved_tensors
        need_input, need_weight, need_bias = ctx.needs_input_grad[0:3]
        dy = grad_output if grad_output.stride() == x.stride() else torch.empty_like(x).copy_(grad_output)
        c = x.size(1)
        sums = _registered(16 * c, x.device)[:16 * c].view(torch.float64)
        grad_weight, grad_bias = ops.sync_bn_backward_reduce(dy, x, mean, invstd, weight, sums,
                                                             need_weight and weight is not None, need_bias)
        grad_input = None
        if need_input:
            _allreduce_sums(sums)
            grad_input = ops.sync_bn_backward_elemt(dy, x, mean, invstd, weight, sums, count)
        return grad_input, grad_weight, grad_bias, None, None, None, None, None, None, None
