"""ctypes binding of the native runtime's C ABI + bootstrap logic.

Role parity: horovod/common/basics.py (HorovodBasics). The reference hands MPI
communicators or Gloo env to C++; here `init()` resolves rank/size from the
launcher's environment (hvdrun's HOROVOD_*, torchrun's RANK/WORLD_SIZE/..., or
single process) and finds/starts the HTTP rendezvous the C++ transport
bootstraps from.
"""
import atexit
import ctypes
import os
import socket
import threading

_LIB = None
_LIB_LOCK = threading.Lock()


def lib_dir():
    return os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "lib")


def load_library():
    """Loads (building on first use if missing) lib/libhvd_core.so."""
    global _LIB
    with _LIB_LOCK:
        if _LIB is not None:
            return _LIB
        path = os.path.join(lib_dir(), "libhvd_core.so")
        if not os.path.exists(path):
            from horovod_b200 import build
            build.build_core()
        lib = ctypes.CDLL(path, mode=ctypes.RTLD_GLOBAL)
        lib.hvd_last_error.restype = ctypes.c_char_p
        lib.hvd_init.argtypes = [ctypes.c_int] * 6 + [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p,
                                                      ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int), ctypes.c_int]
        lib.hvd_add_process_set.argtypes = [ctypes.POINTER(ctypes.c_int), ctypes.c_int]
        lib.hvd_process_set_ids.argtypes = [ctypes.POINTER(ctypes.c_int)]
        lib.hvd_process_set_ranks.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
        lib.hvd_start_timeline.argtypes = [ctypes.c_char_p, ctypes.c_int]
        lib.hvd_topology_string.argtypes = [ctypes.c_char_p, ctypes.c_int]
        lib.hvd_gpu_backend_string.argtypes = [ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
        lib.hvd_stat.restype = ctypes.c_ulonglong
        lib.hvd_stat.argtypes = [ctypes.c_int]
        lib.hvd_param.restype = ctypes.c_longlong
        lib.hvd_param.argtypes = [ctypes.c_int]
        _LIB = lib
        return lib


def _env_int(*names, default=None):
    for n in names:
        v = os.environ.get(n)
        if v is not None and v != '':
            return int(v)
    return default


class _EmbeddedRendezvous:
    """Rank 0 hosts the HTTP KV store in-process when no launcher-provided one exists (torchrun / manual env)."""
    server = None
    port = None
    stores = []


def _resolve_topology():
    """(rank, size, local_rank, local_size, cross_rank, cross_size). local_size -1 => let the runtime derive it."""
    rank = _env_int('HOROVOD_RANK', 'RANK', 'OMPI_COMM_WORLD_RANK', 'PMI_RANK', default=0)
    size = _env_int('HOROVOD_SIZE', 'WORLD_SIZE', 'OMPI_COMM_WORLD_SIZE', 'PMI_SIZE', default=1)
    local_rank = _env_int('HOROVOD_LOCAL_RANK', 'LOCAL_RANK', 'OMPI_COMM_WORLD_LOCAL_RANK', default=None)
    local_size = _env_int('HOROVOD_LOCAL_SIZE', 'LOCAL_WORLD_SIZE', 'OMPI_COMM_WORLD_LOCAL_SIZE', default=None)
    cross_rank = _env_int('HOROVOD_CROSS_RANK', 'GROUP_RANK', default=None)
    cross_size = _env_int('HOROVOD_CROSS_SIZE', default=None)
    if local_rank is None or local_size is None:
        if size == 1:
            local_rank, local_size, cross_rank, cross_size = 0, 1, 0, 1
        else:
            local_rank, local_size = (local_rank or 0), -1
    if cross_rank is None:
        cross_rank = rank // local_size if local_size and local_size > 0 else 0
    if cross_size is None:
        cross_size = (size + local_size - 1) // local_size if local_size and local_size > 0 else 1
    return rank, size, local_rank, local_size, cross_rank, cross_size


def _resolve_rendezvous(rank, size):
    """Returns (addr, port) of the HTTP KV store, starting one on rank 0 if the launcher gave none."""
    addr = os.environ.get('HOROVOD_GLOO_RENDEZVOUS_ADDR')
    port = _env_int('HOROVOD_GLOO_RENDEZVOUS_PORT', default=None)
    if addr and port:
        return addr, port
    if size == 1:
        return '', 0
    master_addr = os.environ.get('MASTER_ADDR', '127.0.0.1')
    master_port = _env_int('MASTER_PORT', default=None)
    if master_port is None:
        raise RuntimeError("hvd.init(): size > 1 but neither HOROVOD_GLOO_RENDEZVOUS_ADDR/PORT (hvdrun) nor "
                           "MASTER_ADDR/MASTER_PORT (torchrun) are set")
    # Exchange the KV server's port through the c10d TCPStore at MASTER_ADDR:MASTER_PORT. Under torchrun the
    # agent already hosts that store; with a hand-made environment rank 0 hosts it.
    from datetime import timedelta
    from torch.distributed import TCPStore
    agent_store = os.environ.get('TORCHELASTIC_USE_AGENT_STORE', '') == 'True'
    store = TCPStore(master_addr, master_port, size, is_master=(rank == 0 and not agent_store),
                     timeout=timedelta(seconds=_env_int('HOROVOD_GLOO_TIMEOUT_SECONDS', default=120)), wait_for_workers=False)
    _EmbeddedRendezvous.stores.append(store)  # rank 0 may host the store: it must outlive this function
    key = 'hvd_b200/rendezvous/%s' % os.environ.get('TORCHELASTIC_RUN_ID', 'default')
    if rank == 0:
        if _EmbeddedRendezvous.server is None:
            from horovod_b200.runner.http.http_server import RendezvousServer
            _EmbeddedRendezvous.server = RendezvousServer()
            _EmbeddedRendezvous.port = _EmbeddedRendezvous.server.start_server()
        store.set(key, str(_EmbeddedRendezvous.port))
        return master_addr if master_addr not in ('', 'localhost') else '127.0.0.1', _EmbeddedRendezvous.port
    port = int(store.get(key).decode())
    return master_addr, port


class HorovodBasics(object):
    """Wrapper class for the basic Horovod API."""

    def __init__(self):
        self._init_count = 0
        self._lib = None

    @property
    def lib(self):
        if self._lib is None:
            self._lib = load_library()
        return self._lib

    def _check(self, rc):
        if rc < 0:
            raise ValueError(self.lib.hvd_last_error().decode())
        return rc

    def init(self, comm=None, process_sets=None):
        """Initialises the runtime. `comm` accepts a list of global ranks (an mpi4py communicator is not supported:
        there is no MPI in this build). `process_sets`: list of ProcessSet objects / rank lists registered statically,
        or the string "dynamic" to enable add_process_set()/remove_process_set() at runtime (always enabled here)."""
        if self.is_initialized():
            if self.lib.hvd_is_running():
                return
            self.lib.hvd_shutdown()  # the loop ended on its own (peer shutdown / failure): start from scratch
        if comm is not None and not isinstance(comm, (list, tuple)):
            raise ValueError("hvd.init(comm=...) only accepts a list of ranks in this build (no MPI).")
        rank, size, local_rank, local_size, cross_rank, cross_size = _resolve_topology()
        scope = 'mesh.%s.%d' % (os.environ.get('HOROVOD_RENDEZVOUS_EPOCH', '0'), self._init_count)
        addr, port = _resolve_rendezvous(rank, size)
        if comm:
            # a job over a subset of the launched ranks (reference basics.py:51-148 with a rank list): the members
            # rendezvous under a scope derived from the list, are renumbered 0..len-1 in list order, and the native
            # runtime derives local / cross ranks from the hostnames it exchanges
            members = [int(r) for r in comm]
            if len(set(members)) != len(members) or any(r < 0 or r >= size for r in members):
                raise ValueError('hvd.init(comm=%r): ranks must be distinct and within [0, %d)' % (list(comm), size))
            if rank not in members:
                raise ValueError('hvd.init(comm=%r) called on rank %d, which is not part of that communicator' % (list(comm), rank))
            import hashlib
            scope += '.c' + hashlib.sha1(','.join(map(str, members)).encode()).hexdigest()[:10]
            rank, size = members.index(rank), len(members)
            if size == 1:
                local_rank, local_size, cross_rank, cross_size = 0, 1, 0, 1
            else:
                local_rank = local_size = cross_rank = cross_size = -1

        if os.environ.get('HOROVOD_ELASTIC') == '1' and addr:
            # elastic: the driver assigns rank/size for this rendezvous round (reference gloo_context.cc:168-214)
            from horovod_b200.runner.http.http_client import read_data_from_kvstore
            host = os.environ.get('HOROVOD_HOSTNAME', socket.gethostname())
            lrank = os.environ.get('HOROVOD_LOCAL_RANK', '0')
            etimeout = float(os.environ.get('HOROVOD_ELASTIC_TIMEOUT', '600'))
            reply = read_data_from_kvstore(addr, port, 'rank_and_size', f'{host}:{lrank}', timeout=etimeout,
                                           request_timeout=etimeout).decode()
            vals = [int(v) for v in reply.split(',')]
            if vals[0] < 0:
                raise RuntimeError("This worker was removed from the job by the elastic driver")
            rank, size, local_rank, local_size, cross_rank, cross_size = vals[:6]
            rnd = vals[6] if len(vals) > 6 else self._init_count
            scope = 'mesh.elastic.%d' % rnd
            os.environ['HOROVOD_RANK'] = str(rank)
            os.environ['HOROVOD_SIZE'] = str(size)
            os.environ['HOROVOD_LOCAL_RANK'] = str(local_rank)
            os.environ['HOROVOD_LOCAL_SIZE'] = str(local_size)
            os.environ['HOROVOD_CROSS_RANK'] = str(cross_rank)
            os.environ['HOROVOD_CROSS_SIZE'] = str(cross_size)

        sets = []
        if process_sets and process_sets != 'dynamic':
            for ps in process_sets:
                ranks = list(ps.ranks) if hasattr(ps, 'ranks') else list(ps)
                sets.append(sorted(int(r) for r in ranks))
        flat = [r for s in sets for r in s]
        sizes = [len(s) for s in sets]
        flat_arr = (ctypes.c_int * max(1, len(flat)))(*flat)
        size_arr = (ctypes.c_int * max(1, len(sizes)))(*sizes)
        rc = self.lib.hvd_init(rank, size, local_rank, local_size, cross_rank, cross_size, addr.encode(), port,
                               scope.encode(), flat_arr, size_arr, len(sizes))
        if rc != 0:
            raise RuntimeError(self.lib.hvd_last_error().decode())
        self._init_count += 1
        atexit.register(self.shutdown)
        if process_sets and process_sets != 'dynamic':
            for i, ps in enumerate(process_sets):
                if hasattr(ps, '_attach'):
                    ps._attach(i + 1)

    def shutdown(self):
        """Stops the background thread; pending collectives fail with HorovodInternalError. Safe to call twice."""
        if self._lib is not None:
            self.lib.hvd_shutdown()

    def is_initialized(self):
        """True between a successful init() and shutdown()."""
        return self._lib is not None and bool(self.lib.hvd_is_initialized())

    def _need_init(self, v):
        if v == -1:
            raise ValueError('Horovod has not been initialized; use hvd.init().')
        return v

    def size(self):
        """Number of ranks in the job."""
        return self._need_init(self.lib.hvd_size())

    def local_size(self):
        """Number of ranks on this host."""
        return self._need_init(self.lib.hvd_local_size())

    def cross_size(self):
        """Number of hosts that have a rank with my local_rank."""
        return self._need_init(self.lib.hvd_cross_size())

    def rank(self):
        """This process's rank in [0, size)."""
        return self._need_init(self.lib.hvd_rank())

    def local_rank(self):
        """Rank among the processes of this host; the usual CUDA device index."""
        return self._need_init(self.lib.hvd_local_rank())

    def cross_rank(self):
        """Index of my host among the hosts that have a rank with my local_rank."""
        return self._need_init(self.lib.hvd_cross_rank())

    def is_homogeneous(self):
        """True when every host runs the same number of ranks."""
        return bool(self.lib.hvd_is_homogeneous())

    # ---- capability queries -------------------------------------------------
    def mpi_threads_supported(self):
        """Always False: there is no MPI in this runtime."""
        return False

    def mpi_enabled(self):
        """Always False: the control plane is the native TCP/shm mesh."""
        return bool(self.lib.hvd_mpi_enabled())

    def mpi_built(self):
        """Always False (kept for API compatibility)."""
        return bool(self.lib.hvd_mpi_built())

    def gloo_enabled(self):
        """True: the native TCP/shm mesh plays the role Gloo plays in the reference."""
        return bool(self.lib.hvd_gloo_enabled())

    def gloo_built(self):
        """True (see gloo_enabled)."""
        return bool(self.lib.hvd_gloo_built())

    def nccl_built(self):
        """True: the NCCL baseline data path is compiled in (libnccl is dlopen'ed on first use)."""
        return int(self.lib.hvd_nccl_built())

    def ddl_built(self):
        """Always False."""
        return bool(self.lib.hvd_ddl_built())

    def ccl_built(self):
        """Always False."""
        return bool(self.lib.hvd_ccl_built())

    def cuda_built(self):
        """True when the native library was built with the sm_90a kernels."""
        return bool(self.lib.hvd_cuda_built())

    def rocm_built(self):
        """Always False."""
        return bool(self.lib.hvd_rocm_built())

    def p2p_built(self):
        """True: the sm_90a NVLink peer-to-peer kernels are compiled in (new capability)."""
        return bool(self.lib.hvd_p2p_built())

    # ---- timeline -------------------------------------------------------------
    def start_timeline(self, file_path, mark_cycles=False):
        """Starts writing a Chrome-tracing timeline to `file_path` (rank 0 writes); `mark_cycles` adds cycle markers."""
        self._check(self.lib.hvd_start_timeline(str(file_path).encode(), 1 if mark_cycles else 0))

    def stop_timeline(self):
        """Stops the timeline started with start_timeline() / HOROVOD_TIMELINE."""
        self._check(self.lib.hvd_stop_timeline())

    # ---- process sets -----------------------------------------------------------
    def _add_process_set_impl(self, ranks):
        arr = (ctypes.c_int * len(ranks))(*[int(r) for r in ranks])
        return self._check(self.lib.hvd_add_process_set(arr, len(ranks)))

    def _remove_process_set_impl(self, process_set_id):
        return self._check(self.lib.hvd_remove_process_set(int(process_set_id)))

    def _process_set_rank(self, process_set_id):
        return self._check(self.lib.hvd_process_set_rank(int(process_set_id)))

    def _process_set_size(self, process_set_id):
        return self._check(self.lib.hvd_process_set_size(int(process_set_id)))

    def _process_set_included(self, process_set_id):
        return bool(self._check(self.lib.hvd_process_set_included(int(process_set_id))))

    def _get_process_set_ids_and_ranks(self):
        """{id: ranks} of the registered process sets. The table can change between the calls below: when any rank
        shuts down, every rank's background loop exits and drops its sets, possibly while this rank is still inside
        hvd.init(). A set that is gone by the time it is queried is left out instead of failing init()."""
        n = self.lib.hvd_number_of_process_sets()
        ids = (ctypes.c_int * max(1, n))()
        self.lib.hvd_process_set_ids(ids)
        out = {}
        for i in range(n):
            sz = self.lib.hvd_process_set_size(ids[i])
            if sz < 0:
                continue
            ranks = (ctypes.c_int * max(1, sz, self.lib.hvd_size()))()
            sz = self.lib.hvd_process_set_ranks(ids[i], ranks)
            if sz < 0:
                continue
            out[ids[i]] = [ranks[j] for j in range(sz)]
        return out

    # ---- introspection (new) ------------------------------------------------------
    def gpu_topology(self):
        """Human-readable result of the GPU / NVLink topology discovery done in init()."""
        buf = ctypes.create_string_buffer(2048)
        self.lib.hvd_topology_string(buf, 2048)
        return buf.value.decode()

    def gpu_backend_info(self, process_set_id=0):
        """Which GPU data path a process set uses (p2p / nccl / host-staged / hierarchical, symmetric-memory kind, buffer size)."""
        buf = ctypes.create_string_buffer(1024)
        self.lib.hvd_gpu_backend_string(process_set_id, buf, 1024)
        return buf.value.decode()

    def control_plane_info(self, process_set_id=0):
        """What negotiation and host-tensor collectives of a process set run on (shared memory / two-level / TCP)."""
        buf = ctypes.create_string_buffer(512)
        self.lib.hvd_control_plane_string(int(getattr(process_set_id, 'process_set_id', process_set_id)), buf, 512)
        return buf.value.decode()

    def runtime_stats(self):
        """Counters of the background thread: cycles, idle cycles, responses executed, kernels launched."""
        return {'cycles': int(self.lib.hvd_stat(0)), 'idle_cycles': int(self.lib.hvd_stat(1)),
                'responses': int(self.lib.hvd_stat(2)), 'kernel_launches': int(self.lib.hvd_stat(3)),
                'captured_collectives': int(self.lib.hvd_stat(4)), 'ipc_zero_copy_allreduces': int(self.lib.hvd_stat(5))}

    def metrics(self):
        """Monotonic counters of this rank since init(): {'allreduce': {'responses', 'tensors', 'bytes', 'on_gpu', 'errors'}, ...}
        per collective type (a fused response counts once in 'responses' and once per tensor in 'tensors'), plus the
        'runtime' block of `runtime_stats()`.  Cheap (a few atomic loads); see horovod_b200.utils.metrics for exporters."""
        lib = self.lib
        lib.hvd_metric.restype = ctypes.c_ulonglong
        fields = ('responses', 'tensors', 'bytes', 'on_gpu', 'errors')
        out = {}
        buf = ctypes.create_string_buffer(64)
        for ty in range(12):
            if lib.hvd_metric_type_name(ty, buf, 64) != 0:
                continue
            vals = {f: int(lib.hvd_metric(ty, i)) for i, f in enumerate(fields)}
            if any(vals.values()):
                out[buf.value.decode().lower()] = vals
        out['runtime'] = self.runtime_stats()
        # host-path latency probes, monotonic like every other counter (so `utils.metrics.Interval` can diff them): total
        # nanoseconds and sample counts per stage — queue = enqueue -> its cycle starts, negotiate, execute = descriptor
        # staging + launch + events + callbacks, total = enqueue -> completion callback; mean = ns / samples
        lat = {}
        for i, name in enumerate(('queue', 'negotiate', 'execute', 'total')):
            lat[name + '_ns'] = int(lib.hvd_stat(10 + i))
            lat[name + '_samples'] = int(lib.hvd_stat(20 + i))
        out['latency'] = lat
        lib.hvd_host_path_count.restype = ctypes.c_ulonglong
        out['host_paths'] = {name: int(lib.hvd_host_path_count(i)) for i, name in enumerate(('shared_memory', 'two_level', 'base_transport'))}
        return out

    def tunable_params(self):
        """Current values of the autotuned parameters (fusion threshold, cycle time, kernel crossovers, CTA count)."""
        names = ['fusion_threshold_bytes', 'cycle_time_us', 'cache_enabled', 'oneshot_max_bytes', 'nvls_min_bytes',
                 'comm_ctas', 'autotune_active']
        return {n: int(self.lib.hvd_param(i)) for i, n in enumerate(names)}
