"""Framework bridge: every non-PyTorch front end (numpy, TensorFlow, Keras, MXNet) reaches the native runtime through
the one pybind module (`lib/_hvd_torch.so`) by viewing its tensors as ``torch.Tensor`` — DLPack for device tensors,
the buffer protocol for host arrays — instead of compiling one C++ adapter per framework.

The reference builds a separate native extension per framework (tensorflow/mpi_ops.cc ~1900 lines, mxnet/mpi_ops.cc +
adapter.cc/tensor_util.cc ~1300 lines, torch/mpi_ops_v2.cc ~1200 lines), each re-implementing the same
Tensor/OpContext/ReadyEvent adapters (common/common.h:265-330).  On an H100 every framework that matters exports
DLPack capsules that alias its device memory, so one adapter is enough: the kernels read and write the framework's own
HBM allocation, and stream ordering is handled by the framework's DLPack stream contract (the producer stream is
synchronised with the consumer's current stream when the capsule is imported).
"""
import torch

from horovod_b200.torch import mpi_ops as _ops


class TensorBridge:
    """Converts between a framework's tensor type and torch tensors.  Subclasses override the two converters."""

    name = 'torch'

    def to_torch(self, x):
        return x

    def from_torch(self, t, like=None):
        return t


class BridgedOps:
    """The collective API over an arbitrary `TensorBridge`.  Handles are the torch front end's integer handles;
    `synchronize` converts the result back to the framework type."""

    Average, Sum, Adasum, Min, Max, Product = _ops.Average, _ops.Sum, _ops.Adasum, _ops.Min, _ops.Max, _ops.Product

    def __init__(self, bridge):
        self.bridge = bridge
        self._likes = {}

    # ---- helpers -------------------------------------------------------------------------------------------------
    def _in(self, x):
        t = self.bridge.to_torch(x)
        return t if t.is_contiguous() else t.contiguous()

    def _track(self, handle, like):
        self._likes[handle] = like
        return handle

    def synchronize(self, handle):
        """Waits for an asynchronous op and returns its result as a framework tensor (list for grouped ops)."""
        like = self._likes.pop(handle, None)
        out = _ops.synchronize(handle)
        if isinstance(out, (list, tuple)):
            if len(out) == 2 and isinstance(out[0], torch.Tensor) and isinstance(out[1], torch.Tensor) and \
                    isinstance(like, tuple) and like and like[0] == 'alltoall':
                return self.bridge.from_torch(out[0], like[1]), self.bridge.from_torch(out[1], None)
            likes = like if isinstance(like, (list, tuple)) else [like] * len(out)
            return [self.bridge.from_torch(o, l) for o, l in zip(out, likes)]
        return self.bridge.from_torch(out, like)

    def poll(self, handle):
        """True once the asynchronous op behind `handle` has finished."""
        return _ops.poll(handle)

    # ---- allreduce -----------------------------------------------------------------------------------------------
    def allreduce_async(self, tensor, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0,
                        process_set=_ops.global_process_set):
        """Asynchronous allreduce (default op: Average); returns a handle."""
        return self._track(_ops.allreduce_async(self._in(tensor), average, name, op, prescale_factor, postscale_factor,
                                                process_set), tensor)

    def allreduce(self, tensor, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0,
                  process_set=_ops.global_process_set):
        """Allreduce (default op: Average) of a framework tensor; the input is not modified."""
        return self.synchronize(self.allreduce_async(tensor, average, name, op, prescale_factor, postscale_factor,
                                                     process_set))

    def grouped_allreduce_async(self, tensors, average=None, name=None, op=None, prescale_factor=1.0,
                                postscale_factor=1.0, process_set=_ops.global_process_set):
        """Asynchronous allreduce of a list of tensors as one fused group; returns a handle."""
        return self._track(_ops.grouped_allreduce_async([self._in(t) for t in tensors], average, name, op, prescale_factor,
                                                        postscale_factor, process_set), list(tensors))

    def grouped_allreduce(self, tensors, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0,
                          process_set=_ops.global_process_set):
        """Allreduce of a list of tensors as one fused group."""
        return self.synchronize(self.grouped_allreduce_async(tensors, average, name, op, prescale_factor,
                                                             postscale_factor, process_set))

    # ---- allgather / broadcast / alltoall / reducescatter --------------------------------------------------------
    def allgather_async(self, tensor, name=None, process_set=_ops.global_process_set):
        """Asynchronous allgather along dim 0; returns a handle."""
        return self._track(_ops.allgather_async(self._in(tensor), name, process_set), tensor)

    def allgather(self, tensor, name=None, process_set=_ops.global_process_set):
        """Concatenates the tensors of all ranks along dim 0 (dim 0 may differ between ranks)."""
        return self.synchronize(self.allgather_async(tensor, name, process_set))

    def grouped_allgather(self, tensors, name=None, process_set=_ops.global_process_set):
        """Allgather of a list of tensors negotiated as one group."""
        h = self._track(_ops.grouped_allgather_async([self._in(t) for t in tensors], name, process_set), list(tensors))
        return self.synchronize(h)

    def broadcast_async(self, tensor, root_rank, name=None, process_set=_ops.global_process_set):
        """Asynchronous broadcast of root_rank's tensor; returns a handle."""
        return self._track(_ops.broadcast_async(self._in(tensor), root_rank, name, process_set), tensor)

    def broadcast(self, tensor, root_rank, name=None, process_set=_ops.global_process_set):
        """Returns root_rank's tensor on every rank."""
        return self.synchronize(self.broadcast_async(tensor, root_rank, name, process_set))

    def alltoall_async(self, tensor, splits=None, name=None, process_set=_ops.global_process_set):
        """Asynchronous alltoall; returns a handle."""
        if splits is not None and not isinstance(splits, (list, tuple, torch.Tensor)):
            splits = self.bridge.to_torch(splits).to(torch.int32).cpu()
        return self._track(_ops.alltoall_async(self._in(tensor), splits, name, process_set),
                           ('alltoall', tensor) if splits is not None else tensor)

    def alltoall(self, tensor, splits=None, name=None, process_set=_ops.global_process_set):
        """Scatters dim-0 slices to all ranks and gathers theirs; with `splits` returns (output, received_splits)."""
        return self.synchronize(self.alltoall_async(tensor, splits, name, process_set))

    def reducescatter_async(self, tensor, name=None, op=_ops.Average, process_set=_ops.global_process_set,
                            prescale_factor=1.0, postscale_factor=1.0):
        """Asynchronous reducescatter; returns a handle."""
        return self._track(_ops.reducescatter_async(self._in(tensor), name, op, process_set, prescale_factor,
                                                    postscale_factor), tensor)

    def reducescatter(self, tensor, name=None, op=_ops.Average, process_set=_ops.global_process_set, prescale_factor=1.0,
                      postscale_factor=1.0):
        """Reduces over ranks; rank r keeps the r-th slice of dim 0."""
        return self.synchronize(self.reducescatter_async(tensor, name, op, process_set, prescale_factor, postscale_factor))

    def grouped_reducescatter(self, tensors, name=None, op=_ops.Average, process_set=_ops.global_process_set,
                              prescale_factor=1.0, postscale_factor=1.0):
        """Reducescatter of a list of tensors as one group."""
        h = self._track(_ops.grouped_reducescatter_async([self._in(t) for t in tensors], name, op, process_set,
                                                         prescale_factor, postscale_factor), list(tensors))
        return self.synchronize(h)

    # ---- python objects ------------------------------------------------------------------------------------------
    @staticmethod
    def broadcast_object(obj, root_rank=0, name=None, process_set=_ops.global_process_set):
        """Broadcasts an arbitrary picklable object from root_rank."""
        from horovod_b200.torch.functions import broadcast_object
        return broadcast_object(obj, root_rank, name, process_set)

    @staticmethod
    def allgather_object(obj, name=None, process_set=_ops.global_process_set):
        """Returns [object of rank 0, object of rank 1, ...] on every rank."""
        from horovod_b200.torch.functions import allgather_object
        return allgather_object(obj, name, process_set)

    def export(self, namespace):
        """Publishes the op set and the process/topology queries into a front end module's globals."""
        for k in ('allreduce', 'allreduce_async', 'grouped_allreduce', 'grouped_allreduce_async', 'allgather',
                  'allgather_async', 'grouped_allgather', 'broadcast', 'broadcast_async', 'alltoall', 'alltoall_async',
                  'reducescatter', 'reducescatter_async', 'grouped_reducescatter', 'synchronize', 'poll',
                  'broadcast_object', 'allgather_object'):
            namespace[k] = getattr(self, k)
        for k in ('init', 'shutdown', 'is_initialized', 'start_timeline', 'stop_timeline', 'size', 'local_size',
                  'cross_size', 'rank', 'local_rank', 'cross_rank', 'is_homogeneous', 'mpi_threads_supported',
                  'mpi_enabled', 'mpi_built', 'gloo_enabled', 'gloo_built', 'nccl_built', 'ddl_built', 'ccl_built',
                  'cuda_built', 'rocm_built', 'p2p_built', 'gpu_topology', 'gpu_backend_info', 'runtime_stats', 'metrics', 'control_plane_info',
                  'tunable_params', 'join', 'barrier', 'Average', 'Sum', 'Adasum', 'Min', 'Max', 'Product',
                  'global_process_set'):
            namespace[k] = getattr(_ops, k)
        from horovod_b200.common.process_sets import ProcessSet, add_process_set, remove_process_set
        namespace.update(ProcessSet=ProcessSet, add_process_set=add_process_set, remove_process_set=remove_process_set)
