"""PyTorch collective API: named asynchronous allreduce / allgather / broadcast /
alltoall / reducescatter (+ grouped, in-place and autograd-aware variants),
join, barrier, poll/synchronize.

API parity: horovod/torch/mpi_ops.py.  (The module keeps the reference's
historical file name so user code that imports `horovod.torch.mpi_ops` ports
by changing only the package name; nothing here is MPI.)  Native calls go to
csrc/torch/binding.cc (`_hvd_torch`).  GPU collectives complete through CUDA
events chained into the caller's stream, so `synchronize()` does not block the
host on the GPU.
"""
import os

import torch

from horovod_b200.common.basics import HorovodBasics, lib_dir
from horovod_b200.common.exceptions import HorovodInternalError
from horovod_b200.common.process_sets import ProcessSet, global_process_set, _setup as _setup_process_sets
from horovod_b200.common.process_sets import add_process_set, remove_process_set  # noqa: F401  (reference: importable from here)
from horovod_b200.common.util import (resolve_op, num_rank_is_power_2, gpu_available,  # noqa: F401
                                      get_average_backwards_compatibility_fun)
from horovod_b200.torch.compression import Compression  # noqa: F401

_basics = HorovodBasics()
_lib = None


def _native():
    """Loads the pybind11 binding (building it on first use if missing)."""
    global _lib
    if _lib is None:
        import importlib.util
        _basics.lib  # load libhvd_core.so first (RTLD_GLOBAL) so the binding resolves against it
        path = os.path.join(lib_dir(), "_hvd_torch.so")
        if not os.path.exists(path):
            from horovod_b200 import build
            build.build_torch()
        spec = importlib.util.spec_from_file_location("_hvd_torch", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _lib = mod
    return _lib


# reduce ops (values follow csrc/common/common.h ReduceOp)
Average = 0
Sum = 1
Adasum = 2
Min = 3
Max = 4
Product = 5

# handle -> (tensors kept alive, output)
_handle_map = {}


def init(*args, **kwargs):
    """Initialises Horovod. Accepts `process_sets=[ProcessSet, ...]` (static registration) or "dynamic"."""
    global _handle_map
    _handle_map = {}
    # before the native runtime spawns its cycle thread (threads inherit the affinity of their creator)
    from horovod_b200.common.basics import _resolve_topology
    from horovod_b200.common.util import bind_to_gpu_numa
    try:
        _lr = _resolve_topology()[2]
        if torch.cuda.is_available():
            bind_to_gpu_numa((_lr if _lr and _lr > 0 else 0) % max(1, torch.cuda.device_count()))
    except Exception:  # noqa: BLE001
        pass
    _basics.init(*args, **kwargs)
    _native()
    _setup_process_sets(_basics)


def shutdown():
    """Shuts the runtime down and forgets outstanding handles."""
    _basics.shutdown()
    if _lib is not None:
        _lib.reset()
    _handle_map.clear()


is_initialized = _basics.is_initialized
start_timeline = _basics.start_timeline
stop_timeline = _basics.stop_timeline
size = _basics.size
local_size = _basics.local_size
cross_size = _basics.cross_size
rank = _basics.rank
local_rank = _basics.local_rank
cross_rank = _basics.cross_rank
is_homogeneous = _basics.is_homogeneous
mpi_threads_supported = _basics.mpi_threads_supported
mpi_enabled = _basics.mpi_enabled
mpi_built = _basics.mpi_built
gloo_enabled = _basics.gloo_enabled
gloo_built = _basics.gloo_built
nccl_built = _basics.nccl_built
ddl_built = _basics.ddl_built
ccl_built = _basics.ccl_built
cuda_built = _basics.cuda_built
rocm_built = _basics.rocm_built
p2p_built = _basics.p2p_built
gpu_topology = _basics.gpu_topology
gpu_backend_info = _basics.gpu_backend_info
runtime_stats = _basics.runtime_stats


def handle_average_backwards_compatibility(op, average):
    """op / deprecated `average=` -> the effective reduce op (reference torch/mpi_ops.py:80-84)."""
    return resolve_op(op, average, Average, Sum)

metrics = _basics.metrics
control_plane_info = _basics.control_plane_info
tunable_params = _basics.tunable_params


def _is_dense(tensor):
    """Contiguous in ANY memory format (row-major, channels_last, ...): the storage is one gap-free block, so an
    elementwise collective can treat it as a flat buffer (every rank holds the same layout)."""
    if tensor.is_contiguous():
        return True
    if tensor.dim() == 4 and tensor.is_contiguous(memory_format=torch.channels_last):
        return True
    if tensor.dim() == 5 and tensor.is_contiguous(memory_format=torch.channels_last_3d):
        return True
    return False


def _check_contiguous(tensor, what='tensor', allow_any_dense_format=False):
    if allow_any_dense_format and _is_dense(tensor):
        return
    if not tensor.is_contiguous():
        raise ValueError(f'Horovod: {what} must be contiguous; call .contiguous() first.')


def _wrap_native(fn, *args):
    try:
        return fn(*args)
    except RuntimeError as e:
        raise HorovodInternalError(e)


# ---------------------------------------------------------------------------
# allreduce

def _adasum_checks(tensor, process_set):
    if process_set.process_set_id != 0:
        raise NotImplementedError('Adasum does not support non-global process sets yet.')
    if not num_rank_is_power_2(size()):
        raise NotImplementedError('Running Adasum with non-power of 2 ranks is not supported yet.')
    if tensor.dtype not in (torch.float16, torch.bfloat16, torch.float32, torch.float64):
        raise ValueError('Adasum supports only floating point tensors.')


def _allreduce_async(tensor, output, name, op, prescale_factor, postscale_factor, process_set):
    _check_contiguous(tensor, allow_any_dense_format=True)
    if output is not tensor and output.stride() != tensor.stride():
        raise ValueError('Horovod: allreduce output must have the same memory layout as the input')
    if op == Adasum:
        _adasum_checks(tensor, process_set)
    if op == Average and not tensor.is_floating_point():
        # integer average: native sum, floor-divide afterwards (reference mpi_ops_v2.cc:62-68)
        handle = _wrap_native(_native().allreduce_async, tensor, output, name or '', Sum, prescale_factor, postscale_factor,
                              process_set.process_set_id)
        _handle_map[handle] = (tensor, output, ('intdiv', process_set.size()))
        return handle
    handle = _wrap_native(_native().allreduce_async, tensor, output, name or '', op, prescale_factor, postscale_factor,
                          process_set.process_set_id)
    _handle_map[handle] = (tensor, output, None)
    return handle


def _differentiate(*tensors):
    """False when no input can receive a gradient: the synchronous collectives then skip the autograd.Function wrapper (its
    `apply` costs more host time than the whole engine path of a small blocking collective)."""
    if not torch.is_grad_enabled():
        return False
    for t in tensors:
        if t.requires_grad:
            return True
    return False


def allreduce_async(tensor, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0,
                    process_set=global_process_set):
    """Asynchronous averaging/summing allreduce; returns a handle for poll()/synchronize(). The input is not modified."""
    op = resolve_op(op, average, Average, Sum)
    output = torch.empty_like(tensor)  # preserves channels_last etc.
    return _allreduce_async(tensor, output, name, op, prescale_factor, postscale_factor, process_set)


class HorovodAllreduce(torch.autograd.Function):
    """Differentiable allreduce: the gradient of an allreduce is the same allreduce of the gradient."""

    @staticmethod
    def forward(ctx, tensor, average, name, op, prescale_factor, postscale_factor, process_set):
        ctx.average = average
        ctx.op = op
        ctx.prescale_factor = prescale_factor
        ctx.postscale_factor = postscale_factor
        ctx.process_set = process_set
        handle = allreduce_async(tensor, average, name, op, prescale_factor, postscale_factor, process_set)
        return synchronize(handle)

    @staticmethod
    def backward(ctx, grad_output):
        return allreduce(grad_output.contiguous(), average=ctx.average, op=ctx.op, prescale_factor=ctx.prescale_factor,
                         postscale_factor=ctx.postscale_factor, process_set=ctx.process_set), None, None, None, None, None, None


def allreduce(tensor, average=None, name=None, compression=None, op=None, prescale_factor=1.0, postscale_factor=1.0,
              process_set=global_process_set):
    """Synchronous, differentiable allreduce (default op: Average). Optional wire `compression`."""
    from horovod_b200.torch.compression import Compression
    compression = compression or Compression.none
    tensor_compressed, ctx = compression.compress(tensor)
    if _differentiate(tensor_compressed):
        summed = HorovodAllreduce.apply(tensor_compressed, average, name, op, prescale_factor, postscale_factor, process_set)
    else:
        summed = synchronize(allreduce_async(tensor_compressed, average, name, op, prescale_factor, postscale_factor, process_set))
    return compression.decompress(summed, ctx)


def allreduce_async_(tensor, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0,
                     process_set=global_process_set):
    """In-place asynchronous allreduce."""
    op = resolve_op(op, average, Average, Sum)
    return _allreduce_async(tensor, tensor, name, op, prescale_factor, postscale_factor, process_set)


def allreduce_(tensor, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0,
               process_set=global_process_set):
    """In-place synchronous allreduce; returns `tensor`."""
    handle = allreduce_async_(tensor, average, name, op, prescale_factor, postscale_factor, process_set)
    return synchronize(handle)


# ---- grouped ----------------------------------------------------------------

def _grouped_allreduce_async(tensors, outputs, name, op, prescale_factor, postscale_factor, process_set):
    for t in tensors:
        _check_contiguous(t, allow_any_dense_format=True)
    if op == Adasum:
        for t in tensors:
            _adasum_checks(t, process_set)
    intdiv = None
    native_op = op
    if op == Average and not all(t.is_floating_point() for t in tensors):
        native_op = Sum
        intdiv = ('intdiv', process_set.size())
    handle = _wrap_native(_native().grouped_allreduce_async, list(tensors), list(outputs), name or '', native_op,
                          prescale_factor, postscale_factor, process_set.process_set_id)
    _handle_map[handle] = (tuple(tensors), tuple(outputs), intdiv)
    return handle


def grouped_allreduce_async(tensors, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0,
                            process_set=global_process_set):
    """Allreduce of a list of tensors negotiated and fused as one unit."""
    op = resolve_op(op, average, Average, Sum)
    outputs = [torch.empty_like(t) for t in tensors]
    return _grouped_allreduce_async(tensors, outputs, name, op, prescale_factor, postscale_factor, process_set)


class HorovodGroupedAllreduce(torch.autograd.Function):
    @staticmethod
    def forward(ctx, average, name, op, prescale_factor, postscale_factor, process_set, *tensors):
        ctx.average = average
        ctx.op = op
        ctx.prescale_factor = prescale_factor
        ctx.postscale_factor = postscale_factor
        ctx.process_set = process_set
        handle = grouped_allreduce_async(list(tensors), average, name, op, prescale_factor, postscale_factor, process_set)
        return tuple(synchronize(handle))

    @staticmethod
    def backward(ctx, *grad_output):
        grads = grouped_allreduce([g.contiguous() for g in grad_output], average=ctx.average, op=ctx.op,
                                  prescale_factor=ctx.prescale_factor, postscale_factor=ctx.postscale_factor,
                                  process_set=ctx.process_set)
        return (None, None, None, None, None, None, *grads)


def grouped_allreduce(tensors, average=None, name=None, compression=None, op=None, prescale_factor=1.0,
                      postscale_factor=1.0, process_set=global_process_set):
    """Synchronous, differentiable allreduce of a list of tensors as ONE fused group (one kernel launch)."""
    from horovod_b200.torch.compression import Compression
    compression = compression or Compression.none
    compressed, ctxs = zip(*[compression.compress(t) for t in tensors])
    if _differentiate(*compressed):
        summed = HorovodGroupedAllreduce.apply(average, name, op, prescale_factor, postscale_factor, process_set, *compressed)
    else:
        summed = synchronize(grouped_allreduce_async(list(compressed), average, name, op, prescale_factor, postscale_factor, process_set))
    return [compression.decompress(t, c) for t, c in zip(summed, ctxs)]


def grouped_allreduce_async_(tensors, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0,
                             process_set=global_process_set):
    """In-place asynchronous grouped allreduce; returns one handle for the group."""
    op = resolve_op(op, average, Average, Sum)
    return _grouped_allreduce_async(tensors, tensors, name, op, prescale_factor, postscale_factor, process_set)


def grouped_allreduce_(tensors, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0,
                       process_set=global_process_set):
    """In-place synchronous grouped allreduce; returns the list of tensors."""
    handle = grouped_allreduce_async_(tensors, average, name, op, prescale_factor, postscale_factor, process_set)
    return synchronize(handle)


def sparse_allreduce_async(tensor, name, op, process_set=global_process_set):
    """Sparse gradient exchange: allgather indices and values, rebuild (reference mpi_ops.py:567-588)."""
    t = tensor.coalesce() if tensor.is_sparse else tensor.to_sparse().coalesce()
    indices_handle = allgather_async(t._indices().transpose(0, 1).contiguous(), name=f'{name}.indices', process_set=process_set)
    values_handle = allgather_async(t._values().contiguous(), name=f'{name}.values', process_set=process_set)

    def handle():
        indices = synchronize(indices_handle)
        values = synchronize(values_handle)
        values = (values / process_set.size()) if op == Average else values
        if indices.dim() == 0 or values.dim() == 0:
            return t.new_empty(t.shape).to_sparse() if not t.is_sparse else t
        return torch.sparse_coo_tensor(indices.transpose(0, 1), values, t.shape).coalesce()

    return handle


# ---------------------------------------------------------------------------
# allgather

def allgather_async(tensor, name=None, process_set=global_process_set):
    """Concatenates the tensors of all ranks along dim 0 (dim 0 may differ between ranks)."""
    _check_contiguous(tensor)
    if tensor.dim() == 0:
        tensor = tensor.reshape(1)
    output = tensor.new_empty(0)
    handle = _wrap_native(_native().allgather_async, tensor, output, name or '', process_set.process_set_id)
    _handle_map[handle] = (tensor, output, None)
    return handle


class HorovodAllgather(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tensor, name, process_set):
        ctx.dim = tensor.shape[0] if tensor.dim() > 0 else 1
        ctx.process_set = process_set
        handle = allgather_async(tensor, name, process_set)
        return synchronize(handle)

    @staticmethod
    def backward(ctx, grad_output):
        # every rank holds the full gradient: average them, then keep the rows this rank contributed
        grad_reduced = allreduce(grad_output.contiguous(), op=Average, process_set=ctx.process_set)
        dim_t = torch.tensor([ctx.dim], dtype=torch.int64)
        dims = allgather(dim_t, process_set=ctx.process_set).view(ctx.process_set.size())
        r = ctx.process_set.rank()
        offset = int(dims.narrow(0, 0, r).sum().item()) if r != 0 else 0
        return grad_reduced.narrow(0, offset, ctx.dim), None, None


def allgather(tensor, name=None, process_set=global_process_set):
    """Synchronous, differentiable allgather along dim 0 (dim 0 may differ between ranks)."""
    if not _differentiate(tensor):
        return synchronize(allgather_async(tensor, name, process_set))
    return HorovodAllgather.apply(tensor, name, process_set)


def grouped_allgather_async(tensors, name=None, process_set=global_process_set):
    """Asynchronous grouped allgather; synchronize() returns the list of outputs."""
    tensors = [t.reshape(1) if t.dim() == 0 else t for t in tensors]
    for t in tensors:
        _check_contiguous(t)
    outputs = [t.new_empty(0) for t in tensors]
    handle = _wrap_native(_native().grouped_allgather_async, list(tensors), outputs, name or '', process_set.process_set_id)
    _handle_map[handle] = (tuple(tensors), tuple(outputs), None)
    return handle


class HorovodGroupedAllgather(torch.autograd.Function):
    @staticmethod
    def forward(ctx, name, process_set, *tensors):
        ctx.dims = [t.shape[0] if t.dim() > 0 else 1 for t in tensors]
        ctx.process_set = process_set
        handle = grouped_allgather_async(list(tensors), name, process_set)
        return tuple(synchronize(handle))

    @staticmethod
    def backward(ctx, *grad_output):
        reduced = grouped_allreduce([g.contiguous() for g in grad_output], op=Average, process_set=ctx.process_set)
        dim_t = torch.tensor(ctx.dims, dtype=torch.int64).reshape(1, -1)
        dims = allgather(dim_t, process_set=ctx.process_set)  # [size, ntensors]
        r = ctx.process_set.rank()
        grads = []
        for i, g in enumerate(reduced):
            offset = int(dims[:r, i].sum().item()) if r != 0 else 0
            grads.append(g.narrow(0, offset, ctx.dims[i]))
        return (None, None, *grads)


def grouped_allgather(tensors, name=None, process_set=global_process_set):
    """Synchronous, differentiable allgather of a list of tensors negotiated as one group."""
    if not _differentiate(*tensors):
        return list(synchronize(grouped_allgather_async(list(tensors), name, process_set)))
    return list(HorovodGroupedAllgather.apply(name, process_set, *tensors))


# ---------------------------------------------------------------------------
# broadcast

def _broadcast_async(tensor, output, root_rank, name, process_set):
    _check_contiguous(tensor, allow_any_dense_format=True)
    handle = _wrap_native(_native().broadcast_async, tensor, output, root_rank, name or '', process_set.process_set_id)
    _handle_map[handle] = (tensor, output, None)
    return handle


def broadcast_async(tensor, root_rank, name=None, process_set=global_process_set):
    """`root_rank` is a GLOBAL rank, also inside a process set."""
    output = torch.empty_like(tensor)
    return _broadcast_async(tensor, output, root_rank, name, process_set)


class HorovodBroadcast(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tensor, root_rank, name, process_set):
        ctx.root_rank = root_rank
        ctx.process_set = process_set
        handle = broadcast_async(tensor, root_rank, name, process_set)
        return synchronize(handle)

    @staticmethod
    def backward(ctx, grad_output):
        grad_reduced = allreduce(grad_output.contiguous(), op=Average, process_set=ctx.process_set)
        if rank() != ctx.root_rank:
            grad_reduced = grad_reduced * 0
        return grad_reduced, None, None, None


def broadcast(tensor, root_rank, name=None, process_set=global_process_set):
    """Synchronous, differentiable broadcast of root_rank's tensor; the input is not modified."""
    if not _differentiate(tensor):
        return synchronize(broadcast_async(tensor, root_rank, name, process_set))
    return HorovodBroadcast.apply(tensor, root_rank, name, process_set)


def broadcast_async_(tensor, root_rank, name=None, process_set=global_process_set):
    """In-place asynchronous broadcast; returns a handle."""
    return _broadcast_async(tensor, tensor, root_rank, name, process_set)


def broadcast_(tensor, root_rank, name=None, process_set=global_process_set):
    """In-place synchronous broadcast; returns `tensor`."""
    handle = broadcast_async_(tensor, root_rank, name, process_set)
    return synchronize(handle)


# ---------------------------------------------------------------------------
# alltoall

def alltoall_async(tensor, splits=None, name=None, process_set=global_process_set):
    """Scatters dim-0 slices to every rank and gathers what they send. Returns (output, received_splits) on sync
    when `splits` was given, else output."""
    _check_contiguous(tensor)
    if splits is None:
        splits_t = torch.empty(0, dtype=torch.int32)
    else:
        splits_t = splits if isinstance(splits, torch.Tensor) else torch.tensor(splits, dtype=torch.int32)
        if splits_t.is_floating_point() or splits_t.dtype == torch.bool or splits_t.dim() != 1:
            raise ValueError('alltoall: splits must be a 1-D integer tensor or a list of ints, got %s with %d dim(s)'
                             % (splits_t.dtype, splits_t.dim()))
    output = tensor.new_empty(0)
    recv_splits = torch.empty(0, dtype=torch.int32, device=splits_t.device if splits is not None else 'cpu')
    handle = _wrap_native(_native().alltoall_async, tensor, splits_t, output, recv_splits, name or '', process_set.process_set_id)
    _handle_map[handle] = (tensor, (output, recv_splits) if splits is not None else output, ('alltoall', recv_splits))
    return handle


class HorovodAlltoall(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tensor, splits, name, process_set):
        handle = alltoall_async(tensor, splits, name, process_set)
        result = synchronize(handle)
        ctx.process_set = process_set
        if splits is None:
            ctx.recvsplits = None
            return result
        output, recv_splits = result
        ctx.recvsplits = recv_splits
        ctx.mark_non_differentiable(recv_splits)
        return output, recv_splits

    @staticmethod
    def backward(ctx, grad_output, *dead):
        if ctx.recvsplits is None:
            return alltoall(grad_output.contiguous(), None, process_set=ctx.process_set), None, None, None
        grad_wrt_tensor, _ = alltoall(grad_output.contiguous(), splits=ctx.recvsplits, process_set=ctx.process_set)
        return grad_wrt_tensor, None, None, None


def alltoall(tensor, splits=None, name=None, process_set=global_process_set):
    """Synchronous, differentiable alltoall; with `splits` returns (output, received_splits)."""
    if not _differentiate(tensor):
        return synchronize(alltoall_async(tensor, splits, name, process_set))
    return HorovodAlltoall.apply(tensor, splits, name, process_set)


# ---------------------------------------------------------------------------
# reducescatter

def reducescatter_async(tensor, name=None, op=Average, process_set=global_process_set, prescale_factor=1.0,
                        postscale_factor=1.0):
    """Reduces across ranks and leaves rank r with its dim-0 slice (the first dim0 % size ranks get one extra row)."""
    _check_contiguous(tensor)
    if op not in (Average, Sum, Min, Max, Product):
        raise ValueError('reducescatter supports only Average, Sum, Min, Max and Product')
    output = tensor.new_empty(0)
    handle = _wrap_native(_native().reducescatter_async, tensor, output, name or '', op, prescale_factor, postscale_factor,
                          process_set.process_set_id)
    _handle_map[handle] = (tensor, output, None)
    return handle


class HorovodReducescatter(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tensor, name, op, process_set, prescale_factor, postscale_factor):
        ctx.op = op
        ctx.process_set = process_set
        ctx.prescale_factor = prescale_factor
        ctx.postscale_factor = postscale_factor
        handle = reducescatter_async(tensor, name, op, process_set, prescale_factor, postscale_factor)
        return synchronize(handle)

    @staticmethod
    def backward(ctx, grad_output):
        if ctx.op == Sum:
            grad_output = grad_output * ctx.process_set.size()
        if ctx.prescale_factor != 1.0:
            grad_output = grad_output * ctx.prescale_factor
        if ctx.postscale_factor != 1.0:
            grad_output = grad_output * ctx.postscale_factor
        return allgather(grad_output.contiguous(), process_set=ctx.process_set), None, None, None, None, None


def reducescatter(tensor, name=None, compression=None, op=Average, process_set=global_process_set, prescale_factor=1.0,
                  postscale_factor=1.0):
    """Synchronous, differentiable reducescatter: reduces over ranks, rank r keeps the r-th slice of dim 0."""
    from horovod_b200.torch.compression import Compression
    compression = compression or Compression.none
    tensor_compressed, ctx = compression.compress(tensor)
    if _differentiate(tensor_compressed):
        reduced = HorovodReducescatter.apply(tensor_compressed, name, op, process_set, prescale_factor, postscale_factor)
    else:
        reduced = synchronize(reducescatter_async(tensor_compressed, name, op, process_set, prescale_factor, postscale_factor))
    return compression.decompress(reduced, ctx)


def grouped_reducescatter_async(tensors, name=None, op=Average, process_set=global_process_set, prescale_factor=1.0,
                                postscale_factor=1.0):
    """Asynchronous grouped reducescatter; synchronize() returns the list of shards."""
    for t in tensors:
        _check_contiguous(t)
    outputs = [t.new_empty(0) for t in tensors]
    handle = _wrap_native(_native().grouped_reducescatter_async, list(tensors), outputs, name or '', op, prescale_factor,
                          postscale_factor, process_set.process_set_id)
    _handle_map[handle] = (tuple(tensors), tuple(outputs), None)
    return handle


class HorovodGroupedReducescatter(torch.autograd.Function):
    @staticmethod
    def forward(ctx, name, op, process_set, prescale_factor, postscale_factor, *tensors):
        ctx.op = op
        ctx.process_set = process_set
        ctx.prescale_factor = prescale_factor
        ctx.postscale_factor = postscale_factor
        handle = grouped_reducescatter_async(list(tensors), name, op, process_set, prescale_factor, postscale_factor)
        return tuple(synchronize(handle))

    @staticmethod
    def backward(ctx, *grad_output):
        scale = (ctx.process_set.size() if ctx.op == Sum else 1.0) * ctx.prescale_factor * ctx.postscale_factor
        grads = [g * scale if scale != 1.0 else g for g in grad_output]
        gathered = grouped_allgather([g.contiguous() for g in grads], process_set=ctx.process_set)
        return (None, None, None, None, None, *gathered)


def grouped_reducescatter(tensors, name=None, compression=None, op=Average, process_set=global_process_set,
                          prescale_factor=1.0, postscale_factor=1.0):
    """Synchronous, differentiable reducescatter of a list of tensors as one group."""
    from horovod_b200.torch.compression import Compression
    compression = compression or Compression.none
    compressed, ctxs = zip(*[compression.compress(t) for t in tensors])
    if _differentiate(*compressed):
        reduced = HorovodGroupedReducescatter.apply(name, op, process_set, prescale_factor, postscale_factor, *compressed)
    else:
        reduced = synchronize(grouped_reducescatter_async(list(compressed), name, op, process_set, prescale_factor, postscale_factor))
    return [compression.decompress(t, c) for t, c in zip(reduced, ctxs)]


# ---------------------------------------------------------------------------
# completion

def poll(handle):
    """True once the collective finished and the output is valid."""
    if callable(handle):
        return True
    return _native().poll(handle)


def synchronize(handle):
    """Waits for an asynchronous collective and returns its output (GPU: the current stream is made to wait)."""
    if callable(handle):  # sparse_allreduce_async
        return handle()
    if handle not in _handle_map:
        return None
    try:
        _native().wait_and_clear(handle)
    except RuntimeError as e:
        _handle_map.pop(handle, None)
        raise HorovodInternalError(e)
    _, output, post = _handle_map.pop(handle)
    if post is not None and post[0] == 'intdiv':
        outs = output if isinstance(output, tuple) else (output,)
        for o in outs:
            if not o.is_floating_point():
                o.copy_(torch.div(o, post[1], rounding_mode='floor'))
            else:
                o.div_(post[1])
    if isinstance(output, tuple) and post is None:
        return list(output)
    return output


def join(device=-1) -> int:
    """Signals that this rank has no more data; blocks until every rank joined. Returns the last rank to join.

    While waiting, the rank contributes zeros to allreduces issued by the others."""
    if device == -1 and torch.cuda.is_available() and is_initialized():
        try:
            device = torch.cuda.current_device()
        except Exception:
            device = -1
    handle = _wrap_native(_native().join, device, 0)
    try:
        return _native().wait_and_clear(handle)
    except RuntimeError as e:
        raise HorovodInternalError(e)


def barrier(process_set=global_process_set):
    """Blocks until every rank of the process set reached the barrier."""
    handle = _wrap_native(_native().barrier, process_set.process_set_id)
    try:
        _native().wait_and_clear(handle)
    except RuntimeError as e:
        raise HorovodInternalError(e)


# ---------------------------------------------------------------------------
# registered symmetric memory (new: no equivalent in the reference)

def symm_empty(shape, dtype=torch.float32, device=None, process_set=global_process_set):
    """COLLECTIVE. Returns an uninitialised CUDA tensor that lives in peer-mapped ("symmetric") memory of the process
    set. In-place allreduces on it (or on a view of it that every rank takes identically) skip the fusion-buffer
    pack/unpack and run the zero-copy NVLink kernel (`multimem` in-switch reduction where available).

    Every member of the process set must call this with the same size. The memory is released by hvd.shutdown();
    do not use the tensor afterwards."""
    if isinstance(shape, int):
        shape = (shape,)
    numel = 1
    for s in shape:
        numel *= int(s)
    itemsize = torch.empty(0, dtype=dtype).element_size()
    nbytes = max(16, (numel * itemsize + 15) // 16 * 16)
    if device is None:
        device = torch.cuda.current_device()
    dev_index = device.index if isinstance(device, torch.device) else int(device)
    try:
        raw = _native().symm_empty(nbytes, dev_index, process_set.process_set_id)
    except RuntimeError as e:
        raise HorovodInternalError(e)
    return raw[:numel * itemsize].view(dtype).view(*shape)


def captured_allreduce_(tensor, op=Average, prescale_factor=1.0, postscale_factor=1.0, process_set=global_process_set, max_ctas=0):
    """In-place allreduce of a tensor allocated with `hvd.symm_empty` (or a view of one taken identically on every rank),
    issued as ONE kernel on the CURRENT CUDA stream — no handle, no negotiation, no host synchronisation — so it can be
    captured into a CUDA graph (`torch.cuda.graph`) together with the compute that produces and consumes the tensor.

    Contract: every rank of the process set issues the same sequence of captured collectives (same tensors, same order);
    the kernel's own cross-GPU flag barrier is the only synchronisation.  `hvd.GraphedStep` uses this to make a whole
    data-parallel training step (forward, backward, gradient allreduce overlapped with backward) one graph launch.
    Ops: Average / Sum / Min / Max / Product.  Returns the tensor."""
    if op == Adasum:
        raise NotImplementedError('captured_allreduce_ does not support op=Adasum')
    try:
        _native().captured_allreduce_(tensor, int(op), float(prescale_factor), float(postscale_factor),
                                      process_set.process_set_id, int(max_ctas))
    except (RuntimeError, ValueError) as e:
        raise HorovodInternalError(e)
    return tensor


def _shard_view(tensor, process_set):
    n = process_set.size() or 1
    flat = tensor.view(-1)
    shard = flat.numel() // n
    r = process_set.rank() if n > 1 else 0
    return flat[r * shard:(r + 1) * shard]


def captured_reducescatter_(tensor, op=Average, prescale_factor=1.0, postscale_factor=1.0, process_set=global_process_set,
                            max_ctas=0):
    """In-place reduce-scatter of a contiguous tensor allocated with `hvd.symm_empty` (or a view of one taken identically on
    every rank), issued like `captured_allreduce_`: ONE kernel on the current CUDA stream, no handle, no negotiation, so
    it can be captured into a CUDA graph.  Every rank issues the same sequence of captured collectives.

    Rank r owns the contiguous slice [r*S, (r+1)*S) of the tensor, S = numel / set size; the byte size must be a multiple
    of 16 * set size.  Only that slice of rank r's tensor receives the reduction; the rest of the tensor is left as it
    was.  Ops: Average / Sum / Min / Max / Product.  Returns the view of this rank's reduced shard."""
    if op == Adasum:
        raise NotImplementedError('captured_reducescatter_ does not support op=Adasum')
    try:
        _native().captured_reducescatter_(tensor, int(op), float(prescale_factor), float(postscale_factor),
                                          process_set.process_set_id, int(max_ctas))
    except (RuntimeError, ValueError) as e:
        raise HorovodInternalError(e)
    return _shard_view(tensor, process_set)


def captured_allgather_(tensor, process_set=global_process_set, max_ctas=0):
    """In-place allgather of a contiguous registered tensor (the counterpart of `captured_reducescatter_`, same launch
    contract): every rank's contiguous 1/N slice of its own tensor is copied into that slice of every peer's tensor.
    The byte size must be a multiple of 16 * set size.  Returns the tensor."""
    try:
        _native().captured_allgather_(tensor, process_set.process_set_id, int(max_ctas))
    except (RuntimeError, ValueError) as e:
        raise HorovodInternalError(e)
    return tensor


# status codes of captured_alltoall (kern::AlltoallStatus)
ALLTOALL_OK, ALLTOALL_NEGATIVE_SPLIT, ALLTOALL_SEND_OVERFLOW, ALLTOALL_RECV_OVERFLOW, ALLTOALL_ROW_BYTES_MISMATCH, \
    ALLTOALL_ABORTED = range(6)


def captured_alltoall(tensor, splits, capacity, process_set=global_process_set, max_ctas=0):
    """Alltoall of the rows of `tensor` whose split vector exists only on the device, issued like `captured_allreduce_`:
    ONE kernel on the current CUDA stream, no handle, no negotiation, no host synchronisation, so it can be captured
    into a CUDA graph (the dispatch / combine of expert parallelism with router-computed row counts).

    tensor: a contiguous CUDA tensor [S, *row] in registered memory (`hvd.symm_empty`, or a view of one) of any dtype.
    The first splits[0] rows go to rank 0, the next splits[1] to rank 1, and so on.  The rows are read in place by the
    receivers: do not overwrite them before the call (stream order takes care of that).
    splits: int32 or int64 CUDA tensor [N] on the same device, N = process set size; only the device reads it.
    capacity: rows of the output.

    Returns (output, recv_splits, status), allocated on the current stream: output [capacity, *row] holds the rows from
    rank 0, then those from rank 1, ...; rows past the total received are not written.  recv_splits: int64 [N], the rows
    each rank sent here.  status: int32 [1], the same on every rank: 0 on success, else the first of
    ALLTOALL_NEGATIVE_SPLIT (1), ALLTOALL_SEND_OVERFLOW (2: some rank's splits sum to more than its S),
    ALLTOALL_RECV_OVERFLOW (3: some rank would receive more than its capacity) and ALLTOALL_ROW_BYTES_MISMATCH (4) that
    applies; then no rank copies any row, recv_splits still holds what was sent, and the next call works normally.
    ALLTOALL_ABORTED (5): a peer never arrived (the team was aborted or timed out).

    Contract: every rank of the process set issues the same sequence of captured collectives with the same `max_ctas`
    (0: the engine's CTA count), and a rank's captured_alltoall calls run in one stream order.  Argument errors the host
    can see raise HorovodInternalError, as does a process set for which `symm_available` is False."""
    if not symm_available(process_set):
        raise HorovodInternalError('captured_alltoall needs a peer-mapped process set of more than one rank (hvd.symm_available)')
    try:
        return tuple(_native().captured_alltoall(tensor, splits, int(capacity), process_set.process_set_id, int(max_ctas)))
    except (RuntimeError, ValueError, TypeError) as e:
        raise HorovodInternalError(e)


def symm_available(process_set=global_process_set):
    """True when the zero-copy path can be used: CUDA, more than one rank, everything on one NVLink domain."""
    return torch.cuda.is_available() and is_initialized() and process_set.size() is not None and process_set.size() > 1 \
        and os.environ.get('HVD_GPU_BACKEND', 'p2p') == 'p2p' and os.environ.get('HOROVOD_ELASTIC') != '1'
