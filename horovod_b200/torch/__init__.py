"""`import horovod_b200.torch as hvd` — PyTorch front end (API parity: horovod/torch/__init__.py)."""
from horovod_b200.common.exceptions import HorovodInternalError, HostsUpdatedInterrupt  # noqa: F401
from horovod_b200.common.util import check_extension  # noqa: F401  (the native library is loaded, and reported missing, on first use)
from horovod_b200.common.process_sets import (ProcessSet, global_process_set, add_process_set,  # noqa: F401
                                              remove_process_set)
from horovod_b200.torch.compression import Compression  # noqa: F401
from horovod_b200.torch.mpi_ops import (  # noqa: F401
    init, shutdown, is_initialized, start_timeline, stop_timeline,
    size, local_size, cross_size, rank, local_rank, cross_rank, is_homogeneous,
    mpi_threads_supported, mpi_enabled, mpi_built, gloo_enabled, gloo_built, nccl_built, ddl_built, ccl_built,
    cuda_built, rocm_built, p2p_built, gpu_topology, gpu_backend_info, runtime_stats, metrics, control_plane_info, tunable_params,
    allreduce, allreduce_async, allreduce_, allreduce_async_,
    grouped_allreduce, grouped_allreduce_async, grouped_allreduce_, grouped_allreduce_async_,
    sparse_allreduce_async,
    allgather, allgather_async, grouped_allgather, grouped_allgather_async,
    broadcast, broadcast_async, broadcast_, broadcast_async_,
    alltoall, alltoall_async,
    reducescatter, reducescatter_async, grouped_reducescatter, grouped_reducescatter_async,
    join, barrier, poll, synchronize, symm_empty, symm_available, captured_allreduce_,
    captured_reducescatter_, captured_allgather_, captured_alltoall,
    Average, Sum, Adasum, Min, Max, Product)
from horovod_b200.torch.functions import (broadcast_parameters, broadcast_optimizer_state, broadcast_object,  # noqa: F401
                                          allgather_object)
from horovod_b200.torch.lamb import Lamb  # noqa: F401
from horovod_b200.torch.lars import Lars  # noqa: F401
from horovod_b200.torch.optimizer import DistributedOptimizer  # noqa: F401
from horovod_b200.torch.sharded_optimizer import ShardedGradScaler  # noqa: F401
from horovod_b200.torch.sync_batch_norm import SyncBatchNorm  # noqa: F401
from horovod_b200.torch.graph import GraphedStep  # noqa: F401
from horovod_b200.torch.moe import ExpertDispatcher  # noqa: F401
from horovod_b200.torch.sequence_parallel import UlyssesExchange  # noqa: F401
from horovod_b200.torch import elastic  # noqa: F401
