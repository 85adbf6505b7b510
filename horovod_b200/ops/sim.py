"""ctypes front end of `csrc/common/sim_api.cc`: run the P2P kernels with N simulated ranks on ONE GPU.

Every "rank" is a set of plain device tensors plus a kernel of its own on its own stream; the cross-"GPU" flag
protocol, chunk ownership and descriptor walking are exactly what runs across NVLink — only the address mapping differs.
All functions take lists indexed [rank][tensor] of CUDA tensors and return the average milliseconds per repeat where that
makes sense.  A non-zero native return code raises RuntimeError (-3 = a barrier of the simulation timed out, -4 = the
ranks' launch plans disagree and nothing was launched, -5 = no plan fits the buffer size `cap`).

reducescatter / allgatherv / broadcast / alltoallv run the launch plans of the engine's ops (csrc/ops/collective_plan.h)
for every simulated rank, check that the plans agree and only then launch them.  `cap` is the symmetric buffer size one
launch may use: small caps force the windowed multi-launch paths.
"""
import ctypes
import math

import torch

DTYPE_CODE = {torch.uint8: 0, torch.int8: 1, torch.int16: 3, torch.int32: 4, torch.int64: 5, torch.float16: 6, torch.float32: 7,
              torch.float64: 8, torch.bool: 9, torch.bfloat16: 10}
ONESHOT, TWOSHOT, NVLS = 0, 1, 2
AVERAGE, SUM, ADASUM, MIN, MAX, PRODUCT = 0, 1, 2, 3, 4, 5
_lib = None


def lib():
    global _lib
    if _lib is None:
        from horovod_b200.common.basics import load_library
        L = load_library()
        u64p, i64p, f32p = ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_float)
        L.hvd_sim_allreduce.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, i64p, u64p, u64p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_int, f32p]
        L.hvd_sim_allgather.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int64, u64p, u64p, ctypes.c_int]
        L.hvd_sim_adasum.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, i64p, u64p, u64p, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                     ctypes.c_double]
        L.hvd_sim_inplace.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int64, u64p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                      ctypes.c_double, ctypes.c_int, f32p]
        L.hvd_sim_inplace_reducescatter.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int64, u64p, ctypes.c_int, ctypes.c_int,
                                                    ctypes.c_int, ctypes.c_double, ctypes.c_int]
        L.hvd_sim_inplace_allgather.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int64, u64p, ctypes.c_int, ctypes.c_int]
        plan = [ctypes.c_int, ctypes.c_int, ctypes.c_int, i64p, i64p]
        L.hvd_sim_reducescatter.argtypes = plan + [u64p, u64p, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double,
                                                   ctypes.c_int64, ctypes.c_int]
        L.hvd_sim_allgatherv.argtypes = plan + [ctypes.c_int, u64p, u64p, ctypes.c_int64, ctypes.c_int]
        L.hvd_sim_broadcast.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, i64p, ctypes.c_int, u64p, u64p, ctypes.c_int64,
                                        ctypes.c_int]
        L.hvd_sim_alltoallv.argtypes = plan + [ctypes.c_int, u64p, u64p, ctypes.c_int64, ctypes.c_int]
        L.hvd_sim_captured_alltoall.argtypes = [ctypes.c_int, ctypes.c_int, u64p, i64p, i64p, u64p, ctypes.c_int, u64p, i64p, u64p,
                                                u64p, ctypes.c_int, u64p]
        L.hvd_sim_ulysses_exchange.argtypes = [ctypes.c_int, ctypes.c_int, u64p, u64p, u64p, i64p, i64p, i64p, ctypes.c_int,
                                               ctypes.c_int, u64p, ctypes.c_int, u64p]
        _lib = L
    return _lib


def _check(rc, what):
    if rc != 0:
        why = {-3: ' (simulated barrier timed out)', -4: ' (the ranks\' launch plans disagree)', -5: ' (no plan fits the buffer)'}
        raise RuntimeError('%s failed with code %d%s' % (what, rc, why.get(rc, '')))


def _ptrs(rows):
    flat = [t.data_ptr() for row in rows for t in row]
    return (ctypes.c_uint64 * len(flat))(*flat)


def allreduce(ins, outs, op=SUM, variant=TWOSHOT, ctas=8, wire_dtype=None, prescale=1.0, postscale=1.0, repeats=1, device=0):
    """ins/outs: [nranks][ntensors] (outs may alias ins).  wire_dtype: on-the-wire dtype for fp32 tensors (fused cast)."""
    n, t = len(ins), len(ins[0])
    dtype = ins[0][0].dtype
    counts = (ctypes.c_int64 * t)(*[x.numel() for x in ins[0]])
    ms = ctypes.c_float(0)
    _check(lib().hvd_sim_allreduce(n, device, t, counts, _ptrs(ins), _ptrs(outs), DTYPE_CODE[dtype], DTYPE_CODE[wire_dtype or dtype], op,
                                   variant, ctas, prescale, postscale, repeats, ctypes.byref(ms)), 'sim allreduce')
    return ms.value / max(repeats, 1)


def inplace_allreduce(tensors, op=SUM, ctas=8, scale=1.0, repeats=1, device=0):
    """tensors: one tensor per simulated rank, reduced in place by the zero-copy kernel (P2P two-shot variant)."""
    n = len(tensors)
    ptrs = (ctypes.c_uint64 * n)(*[t.data_ptr() for t in tensors])
    ms = ctypes.c_float(0)
    nbytes = tensors[0].numel() * tensors[0].element_size()
    _check(lib().hvd_sim_inplace(n, device, nbytes, ptrs, DTYPE_CODE[tensors[0].dtype], op, ctas, scale, repeats, ctypes.byref(ms)),
           'sim in-place allreduce')
    return ms.value / max(repeats, 1)


def inplace_reducescatter(tensors, op=SUM, ctas=8, scale=1.0, repeats=1, device=0):
    """tensors: one tensor per simulated rank; rank r's contiguous 1/n slice of its own tensor receives the reduction
    (scaled by `scale`), nothing else is written.  The byte size must be a multiple of 16 * n."""
    n = len(tensors)
    ptrs = (ctypes.c_uint64 * n)(*[t.data_ptr() for t in tensors])
    nbytes = tensors[0].numel() * tensors[0].element_size()
    _check(lib().hvd_sim_inplace_reducescatter(n, device, nbytes, ptrs, DTYPE_CODE[tensors[0].dtype], op, ctas, scale, repeats),
           'sim in-place reduce-scatter')


def inplace_allgather(tensors, ctas=8, repeats=1, device=0):
    """tensors: one tensor per simulated rank; rank r's contiguous 1/n slice of its own tensor is copied into every other
    rank's tensor.  The byte size must be a multiple of 16 * n."""
    n = len(tensors)
    ptrs = (ctypes.c_uint64 * n)(*[t.data_ptr() for t in tensors])
    nbytes = tensors[0].numel() * tensors[0].element_size()
    _check(lib().hvd_sim_inplace_allgather(n, device, nbytes, ptrs, ctas, repeats), 'sim in-place allgather')


def allgather(ins, outs, ctas=8, device=0):
    """ins[r]: rank r's contribution (all the same byte size); outs[r]: nranks * that size."""
    n = len(ins)
    nbytes = ins[0].numel() * ins[0].element_size()
    ip = (ctypes.c_uint64 * n)(*[t.data_ptr() for t in ins])
    op = (ctypes.c_uint64 * n)(*[t.data_ptr() for t in outs])
    _check(lib().hvd_sim_allgather(n, device, nbytes, ip, op, ctas), 'sim allgather')


def adasum(ins, outs, ctas=8, prescale=1.0, postscale=1.0, device=0):
    n, t = len(ins), len(ins[0])
    counts = (ctypes.c_int64 * t)(*[x.numel() for x in ins[0]])
    _check(lib().hvd_sim_adasum(n, device, t, counts, _ptrs(ins), _ptrs(outs), DTYPE_CODE[ins[0][0].dtype], ctas, prescale, postscale),
           'sim adasum')


def _i64(vals):
    vals = [int(v) for v in vals]
    return (ctypes.c_int64 * max(len(vals), 1))(*vals)


def _row(t):
    r = 1
    for d in t.shape[1:]:
        r *= d
    return r


def reducescatter(ins, outs, op=SUM, prescale=1.0, postscale=1.0, cap=1 << 20, ctas=8, device=0):
    """ins[r][t]: rank r's whole tensor t (the same shape on every rank); outs[r][t]: rank r's block of the result, dim 0
    split as the engine splits it (the first dim0 % n ranks get one extra row).  One-shot reduce, rank order 0 .. n-1."""
    n, t = len(ins), len(ins[0])
    x = ins[0]
    _check(lib().hvd_sim_reducescatter(n, device, t, _i64(a.shape[0] for a in x), _i64(_row(a) for a in x), _ptrs(ins), _ptrs(outs),
                                       DTYPE_CODE[x[0].dtype], op, prescale, postscale, cap, ctas), 'sim reducescatter')


def allgatherv(ins, outs, cap=1 << 20, ctas=8, device=0):
    """ins[r][t]: rank r's contribution to tensor t (first dims may differ per rank, may be 0); outs[r][t]: the
    concatenation along dim 0 in rank order."""
    n, t = len(ins), len(ins[0])
    dims = [ins[r][i].shape[0] for i in range(t) for r in range(n)]
    _check(lib().hvd_sim_allgatherv(n, device, t, _i64(dims), _i64(_row(a) for a in ins[0]), DTYPE_CODE[ins[0][0].dtype], _ptrs(ins),
                                    _ptrs(outs), cap, ctas), 'sim allgatherv')


def broadcast(ins, outs, root, cap=1 << 20, ctas=8, device=0):
    """ins[r][t] / outs[r][t]: every rank's tensors (the same byte sizes); outs[root][t] is ins[root][t] for an in-place
    broadcast.  Only the root's inputs are read."""
    n, t = len(ins), len(ins[0])
    nbytes = [a.numel() * a.element_size() for a in ins[0]]
    _check(lib().hvd_sim_broadcast(n, device, t, _i64(nbytes), root, _ptrs(ins), _ptrs(outs), cap, ctas), 'sim broadcast')


def alltoallv(ins, outs, splits, cap=1 << 20, ctas=8, device=0):
    """splits[t][p][q]: rows of tensor t that rank p sends to rank q (rank p's ins[p][t] holds them in q order); outs[q][t]
    receives them in p order."""
    n, t = len(ins), len(ins[0])
    flat = [splits[i][p][q] for i in range(t) for p in range(n) for q in range(n)]
    _check(lib().hvd_sim_alltoallv(n, device, t, _i64(flat), _i64(_row(a) for a in ins[0]), DTYPE_CODE[ins[0][0].dtype], _ptrs(ins),
                                   _ptrs(outs), cap, ctas), 'sim alltoallv')


def captured_alltoall(ins, splits, outs, recv_splits, status, ctas=8, streams=None, device=0):
    """The kernel of hvd.captured_alltoall on N simulated ranks, every argument a list indexed by rank: ins[r] [S_r, *row]
    (contiguous), splits[r] int32 / int64 [N] on the device, outs[r] [capacity_r, *row], recv_splits[r] int64 [N],
    status[r] int32 [1].  Rows and row bytes come from each rank's own tensors, so ranks may disagree on them.

    streams=None runs the N kernels and waits for them.  With streams (N torch.cuda.Stream) rank r's kernel is only
    launched on streams[r], after whatever that stream already holds, so a caller can order it after device work of its
    own or capture all N ranks into one CUDA graph.  That needs one earlier call with streams=None for this N, which
    creates the simulated team the kernels keep using."""
    n = len(ins)
    if len({s.dtype for s in splits}) != 1:
        raise ValueError('sim captured alltoall: every rank\'s splits need the same dtype')
    u64 = lambda vals: (ctypes.c_uint64 * n)(*vals)  # noqa: E731
    rc = lib().hvd_sim_captured_alltoall(
        n, device, u64(t.data_ptr() for t in ins), _i64(t.shape[0] for t in ins), _i64(_row(t) * t.element_size() for t in ins),
        u64(s.data_ptr() for s in splits), int(splits[0].dtype == torch.int64), u64(t.data_ptr() for t in outs),
        _i64(t.shape[0] for t in outs), u64(t.data_ptr() for t in recv_splits), u64(t.data_ptr() for t in status), ctas,
        None if streams is None else u64(s.cuda_stream for s in streams))
    _check(rc, 'sim captured alltoall')


SEQ_TO_HEADS, HEADS_TO_SEQ = 0, 1


def ulysses_view(shape, seq_dim, head_dim):
    """[A, D1, M, D2, R] of a tensor of `shape` whose named dims are seq_dim and head_dim (D1 the first of them)."""
    lo, hi = min(seq_dim, head_dim), max(seq_dim, head_dim)
    return [math.prod(shape[:lo]), shape[lo], math.prod(shape[lo + 1:hi]), shape[hi], math.prod(shape[hi + 1:])]


def ulysses_exchange(ins, outs, seq_dim, head_dim, direction, status, staging=None, ctas=8, streams=None, device=0):
    """The kernel of hvd.UlyssesExchange on N simulated ranks, every argument a list indexed by rank: ins[r] contiguous,
    outs[r] with the same bytes (contiguous), status[r] int32 [1] (keeps the first non-zero code).  direction
    SEQ_TO_HEADS splits head_dim into N blocks and concatenates the ranks' blocks along seq_dim; HEADS_TO_SEQ splits
    seq_dim and concatenates along head_dim.  The view [A, D1, M, D2, R] and the element size come from each rank's own
    input, so ranks may disagree on them.  staging[r]: rank r's staging buffer (any contiguous CUDA tensor of at least
    the input's bytes); None allocates one per rank for this call, which a captured graph must not rely on.

    streams as in captured_alltoall: with streams, rank r's kernel is only launched on streams[r]."""
    n = len(ins)
    if staging is None:
        staging = [torch.empty(max(t.numel() * t.element_size(), 1), dtype=torch.uint8, device=t.device) for t in ins]
    u64 = lambda vals: (ctypes.c_uint64 * n)(*vals)  # noqa: E731
    dims = [d for t in ins for d in ulysses_view(list(t.shape), seq_dim, head_dim)]
    rc = lib().hvd_sim_ulysses_exchange(
        n, device, u64(t.data_ptr() for t in ins), u64(t.data_ptr() for t in outs), u64(t.data_ptr() for t in staging),
        _i64(t.numel() * t.element_size() for t in staging), _i64(dims), _i64(t.element_size() for t in ins), int(direction),
        int(head_dim < seq_dim), u64(t.data_ptr() for t in status), ctas, None if streams is None else u64(s.cuda_stream for s in streams))
    _check(rc, 'sim ulysses exchange')
