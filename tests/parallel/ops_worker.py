"""Distributed op tests, run under `hvdrun -np N` (CPU: native TCP/shm ops; --device cuda: NVLink P2P kernels).

Case matrix modelled on the reference's test/parallel/test_torch.py: every op x dtype x dims, value-checked against
closed forms; in-place / async+fusion / pre-postscale / grouped / process sets / error paths / autograd / join /
barrier / duplicate names / reinit.  Each rank runs every check; a failing assert exits non-zero which makes the
launcher kill the job.
"""
import argparse
import itertools
import sys
import time
import traceback

import torch

import horovod_b200.torch as hvd
from horovod_b200.common.exceptions import HorovodInternalError

p = argparse.ArgumentParser()
p.add_argument('--device', default='cpu')
p.add_argument('--only', default='')
p.add_argument('--skip', default='')
args = p.parse_args()

import os
FAKE_HOSTS = int(os.environ.get('HVD_TEST_FAKE_HOSTS', '0'))
if FAKE_HOSTS > 1:
    # pretend the ranks of this box live on FAKE_HOSTS machines: the control plane drops to TCP, set-wide peer mapping is
    # refused and GPU allreduce takes the hierarchical path (intra-"host" kernels + cross-"host" CPU transport)
    _r, _n = int(os.environ['HOROVOD_RANK']), int(os.environ['HOROVOD_SIZE'])
    _L = _n // FAKE_HOSTS
    os.environ.update(HOROVOD_HOSTNAME='fakehost%d' % (_r // _L), HOROVOD_LOCAL_RANK=str(_r % _L), HOROVOD_LOCAL_SIZE=str(_L),
                      HOROVOD_CROSS_RANK=str(_r // _L), HOROVOD_CROSS_SIZE=str(FAKE_HOSTS))

hvd.init()
rank, size = hvd.rank(), hvd.size()
DEV_INDEX = rank if FAKE_HOSTS > 1 else hvd.local_rank()
if args.device == 'cuda':
    torch.cuda.set_device(DEV_INDEX)
DEV = torch.device('cuda', DEV_INDEX) if args.device == 'cuda' else torch.device('cpu')

FLOATS = [torch.float32, torch.float64, torch.float16, torch.bfloat16]
INTS = [torch.int32, torch.int64, torch.uint8, torch.int8, torch.int16]
DIMS = [1, 2, 3]


def tol(dtype):
    if dtype in (torch.float16, torch.bfloat16):
        return dict(rtol=2e-2, atol=2e-2)
    if dtype.is_floating_point:
        return dict(rtol=1e-5, atol=1e-5)
    return dict(rtol=0, atol=0)


def rand(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    if dtype.is_floating_point:
        return torch.rand(shape, generator=g).mul(4).sub(2).to(dtype).to(DEV)
    return torch.randint(0, 5, shape, generator=g).to(dtype).to(DEV)


def check(name):
    def deco(fn):
        fn._check_name = name
        CHECKS.append(fn)
        return fn
    return deco


CHECKS = []


@check('rank_size')
def _():
    assert 0 <= rank < size
    assert hvd.local_size() >= 1 and hvd.cross_size() >= 1
    assert hvd.local_rank() < hvd.local_size()
    assert hvd.is_initialized()


@check('fake_hosts_topology')
def _():
    if FAKE_HOSTS <= 1:
        return
    L = size // FAKE_HOSTS
    assert hvd.local_size() == L and hvd.cross_size() == FAKE_HOSTS
    assert hvd.local_rank() == rank % L and hvd.cross_rank() == rank // L
    assert hvd.is_homogeneous()
    # negotiation: shm among the ranks of a "host", host leaders over TCP (unless the test forces the TCP control plane)
    info = hvd.control_plane_info()
    if os.environ.get('HVD_CONTROL_PLANE') != 'tcp' and L > 1:
        assert 'two-level' in info and '%d ranks of this host' % L in info and '%d host leaders' % FAKE_HOSTS in info, info
    # a process set made of the ranks of ONE host negotiates and moves host tensors through that host's shared memory (own
    # channel + data slots); a set that spans hosts stays on the sockets
    if os.environ.get('HVD_CONTROL_PLANE') != 'tcp' and L > 1 and args.device == 'cpu':
        host_sets = [hvd.add_process_set(list(range(h * L, (h + 1) * L))) for h in range(FAKE_HOSTS)]
        spanning = hvd.add_process_set(list(range(0, size, L)))                # the first rank of every host
        mine = host_sets[rank // L]
        assert 'shared memory channel' in hvd.control_plane_info(mine), hvd.control_plane_info(mine)
        for step in range(3):                                                   # uncached, then cached
            out = hvd.allreduce(torch.full([1000], float(rank + 1)), op=hvd.Sum, name='hostset.ar', process_set=mine)
            assert float(out[0]) == float(sum(r + 1 for r in range((rank // L) * L, (rank // L + 1) * L))), out[:3]
        big = hvd.allreduce(torch.arange(300000, dtype=torch.float32) % 7 + rank, op=hvd.Sum, name='hostset.big', process_set=mine)
        members = list(range((rank // L) * L, (rank // L + 1) * L))
        assert torch.equal(big, (torch.arange(300000, dtype=torch.float32) % 7) * L + float(sum(members)))
        g = hvd.allgather(torch.full([rank % L + 1, 2], float(rank)), name='hostset.ag', process_set=mine)
        assert g.shape[0] == sum(range(1, L + 1)) and float(g[0, 0]) == float(members[0])
        if spanning.included():
            assert 'shared memory channel' not in hvd.control_plane_info(spanning)
            s2 = hvd.allreduce(torch.ones(5), op=hvd.Sum, name='spanning.ar', process_set=spanning)
            assert float(s2[0]) == float(FAKE_HOSTS)
        hvd.barrier()
        for ps in host_sets + [spanning]:
            hvd.remove_process_set(ps)


@check('hierarchical_allreduce')
def _():
    # big enough for several reduce-scatter / allgather windows when HVD_SYMM_BUFFER_BYTES is small; fused odd sizes
    for dtype in (torch.float32, torch.bfloat16, torch.int32):
        tensors = [rand([n], dtype, 77 + rank * 13 + i) for i, n in enumerate([1, 1000003, 17, 262144])]
        hs = [hvd.allreduce_async(t, op=hvd.Sum, name=f'hier.{dtype}.{i}') for i, t in enumerate(tensors)]
        outs = [hvd.synchronize(h) for h in hs]
        for i, n in enumerate([1, 1000003, 17, 262144]):
            ref = sum(rand([n], dtype, 77 + r * 13 + i).double() for r in range(size)).to(dtype)
            if dtype.is_floating_point:
                # two-level sums round twice in the tensor's dtype (intra-host, then cross-host): 2 ulp of bf16 at |x| <= 16
                t = dict(rtol=2e-2, atol=8e-2) if dtype == torch.bfloat16 else tol(dtype)
                torch.testing.assert_close(outs[i], ref, **t)
            else:
                assert torch.equal(outs[i], ref)
    x = torch.full((5, 3), float(rank + 1), device=DEV)
    avg = hvd.allreduce(x, op=hvd.Average, name='hier.avg', prescale_factor=2.0)
    torch.testing.assert_close(avg, torch.full((5, 3), 2.0 * (size + 1) / 2, device=DEV))
    mx = hvd.allreduce(x, op=hvd.Max, name='hier.max')
    assert torch.equal(mx, torch.full((5, 3), float(size), device=DEV))
    if args.device == 'cuda' and FAKE_HOSTS > 1 and size // FAKE_HOSTS >= 2:
        assert 'hierarchical' in hvd.gpu_backend_info(), hvd.gpu_backend_info()


@check('allreduce_sum_avg')
def _():
    for dtype, dim in itertools.product(FLOATS + INTS, DIMS):
        shape = [17] * dim
        mine = rand(shape, dtype, 1234 + rank)
        everyone = [rand(shape, dtype, 1234 + r) for r in range(size)]
        summed = hvd.allreduce(mine, op=hvd.Sum, name=f'ar.sum.{dtype}.{dim}')
        ref = torch.stack([e.double() if dtype.is_floating_point else e.long() for e in everyone]).sum(0).to(dtype)
        torch.testing.assert_close(summed, ref, **tol(dtype)) if dtype.is_floating_point else None
        if not dtype.is_floating_point:
            assert torch.equal(summed, ref), (dtype, dim)
        assert torch.equal(mine, everyone[rank]), 'out-of-place allreduce modified its input'
        avg = hvd.allreduce(mine, name=f'ar.avg.{dtype}.{dim}')  # default op = Average
        if dtype.is_floating_point:
            torch.testing.assert_close(avg.double(), ref.double() / size, **tol(dtype))
        else:
            assert torch.equal(avg, torch.div(ref, size, rounding_mode='floor')), (dtype, avg, ref)


@check('allreduce_inplace_prepost')
def _():
    for dtype in [torch.float32, torch.float64, torch.bfloat16]:
        t = rand([17, 17], dtype, 7 + rank)
        everyone = [rand([17, 17], dtype, 7 + r) for r in range(size)]
        out = hvd.allreduce_(t, op=hvd.Sum, prescale_factor=0.5, postscale_factor=3.0)
        assert out.data_ptr() == t.data_ptr()
        ref = torch.stack([(e.double() * 0.5) for e in everyone]).sum(0) * 3.0
        torch.testing.assert_close(t.double(), ref, **tol(dtype))


@check('allreduce_min_max_product')
def _():
    for dtype in [torch.float32, torch.int32]:
        mine = rand([33], dtype, 99 + rank) + 1
        everyone = torch.stack([rand([33], dtype, 99 + r) + 1 for r in range(size)])
        assert torch.equal(hvd.allreduce(mine, op=hvd.Min), everyone.min(0).values)
        assert torch.equal(hvd.allreduce(mine, op=hvd.Max), everyone.max(0).values)
        torch.testing.assert_close(hvd.allreduce(mine, op=hvd.Product), everyone.prod(0).to(dtype), **tol(torch.float32))


@check('allreduce_async_fused')
def _():
    """Many tensors in flight: they get fused; poll() must observe 'not done' at least once."""
    for rep in range(3):
        tensors = [rand([17] * (1 + i % 3), torch.float32, 31 * i + rank) for i in range(40)]
        handles = [hvd.allreduce_async(t, op=hvd.Sum, name=f'fused.{i}') for i, t in enumerate(tensors)]
        not_done = sum(0 if hvd.poll(h) else 1 for h in handles)
        outs = [hvd.synchronize(h) for h in handles]
        for i, o in enumerate(outs):
            ref = torch.stack([rand([17] * (1 + i % 3), torch.float32, 31 * i + r) for r in range(size)]).sum(0)
            torch.testing.assert_close(o, ref, **tol(torch.float32))
    stats = hvd.runtime_stats()
    assert stats['responses'] > 0


@check('allreduce_mixed_dtype_fusion')
def _():
    """fp32 / fp16 / int interleaved: the look-ahead planner still fuses same-dtype neighbours."""
    dts = [torch.float32, torch.float16, torch.int32]
    tensors = [rand([100], dts[i % 3], 5 * i + rank) for i in range(30)]
    handles = [hvd.allreduce_async(t, op=hvd.Sum, name=f'mixed.{i}') for i, t in enumerate(tensors)]
    for i, h in enumerate(handles):
        o = hvd.synchronize(h)
        ref = torch.stack([rand([100], dts[i % 3], 5 * i + r).double() for r in range(size)]).sum(0)
        torch.testing.assert_close(o.double(), ref, **tol(dts[i % 3]))


@check('grouped_allreduce')
def _():
    ts = [rand([10 + i], torch.float32, 200 + i + rank) for i in range(5)]
    outs = hvd.grouped_allreduce(ts, op=hvd.Sum, name='grp')
    for i, o in enumerate(outs):
        ref = torch.stack([rand([10 + i], torch.float32, 200 + i + r) for r in range(size)]).sum(0)
        torch.testing.assert_close(o, ref, **tol(torch.float32))
    ts2 = [t.clone() for t in ts]
    hvd.grouped_allreduce_(ts2, op=hvd.Average, name='grp_inplace')
    for i, o in enumerate(ts2):
        ref = torch.stack([rand([10 + i], torch.float32, 200 + i + r) for r in range(size)]).sum(0) / size
        torch.testing.assert_close(o, ref, **tol(torch.float32))


@check('allgather')
def _():
    for dtype, dim in itertools.product([torch.float32, torch.int64, torch.uint8, torch.bfloat16], DIMS):
        t = torch.full([17] * dim, rank, dtype=dtype, device=DEV)
        g = hvd.allgather(t)
        assert list(g.shape) == [17 * size] + [17] * (dim - 1)
        for r in range(size):
            assert (g[r * 17:(r + 1) * 17] == r).all()
    # variable first dimension
    sizes = [((r + 1) * 3) % 7 + 1 for r in range(size)]
    t = torch.full([sizes[rank], 5], float(rank), device=DEV)
    g = hvd.allgather(t, name='ag.var')
    assert g.shape[0] == sum(sizes)
    off = 0
    for r in range(size):
        assert (g[off:off + sizes[r]] == r).all()
        off += sizes[r]
    # scalar -> vector of size
    s = hvd.allgather(torch.tensor(float(rank), device=DEV))
    assert s.tolist() == [float(r) for r in range(size)]
    # grouped
    outs = hvd.grouped_allgather([torch.full([2], float(rank), device=DEV), torch.full([rank + 1, 2], float(rank), device=DEV)])
    assert outs[0].shape[0] == 2 * size and outs[1].shape[0] == size * (size + 1) // 2


@check('broadcast')
def _():
    for dtype, dim, root in itertools.product([torch.float32, torch.int32, torch.float16], DIMS, range(size)):
        t = torch.full([17] * dim, rank, dtype=dtype, device=DEV)
        out = hvd.broadcast(t, root)
        assert (out == root).all()
        assert (t == rank).all()
        t2 = t.clone()
        hvd.broadcast_(t2, root)
        assert (t2 == root).all()


@check('alltoall')
def _():
    for dtype in [torch.float32, torch.int64]:
        # equal splits
        t = torch.arange(size * 3, device=DEV).to(dtype) + 1000 * rank
        out = hvd.alltoall(t)
        exp = torch.cat([torch.arange(rank * 3, rank * 3 + 3).to(dtype) + 1000 * r for r in range(size)]).to(DEV)
        assert torch.equal(out, exp)
        # no explicit splits but a different dim 0 on every rank (rank r sends r + 1 rows to each destination): the
        # uniform-splits shortcut must NOT apply, the split matrix is exchanged
        t = torch.full((size * (rank + 1), 2), float(rank), device=DEV).to(dtype)
        out = hvd.alltoall(t, name='a2a.implicit.ragged.%s' % dtype)
        assert out.shape[0] == sum(r + 1 for r in range(size)), out.shape
        off = 0
        for r in range(size):
            assert (out[off:off + r + 1] == r).all(), (r, out)
            off += r + 1
        # one rank passes explicit (uniform) splits, the others none: same result as all-implicit
        t = torch.arange(size * 2, device=DEV).to(dtype) + 100 * rank
        out = hvd.alltoall(t, splits=[2] * size, name='a2a.mixed.%s' % dtype)[0] if rank == 0 else hvd.alltoall(t, name='a2a.mixed.%s' % dtype)
        exp = torch.cat([torch.arange(rank * 2, rank * 2 + 2).to(dtype) + 100 * r for r in range(size)]).to(DEV)
        assert torch.equal(out, exp), (out, exp)
        # uneven splits: rank r sends (d + 1) rows to destination d
        splits = torch.tensor([d + 1 for d in range(size)], dtype=torch.int32)
        rows = int(splits.sum())
        t = (torch.arange(rows, device=DEV).to(dtype) + 1000 * rank).reshape(rows, 1).repeat(1, 2).contiguous()
        out, rsplits = hvd.alltoall(t, splits=splits)
        assert rsplits.tolist() == [rank + 1] * size, rsplits
        assert out.shape == (size * (rank + 1), 2)
        start = sum(d + 1 for d in range(rank))
        for r in range(size):
            blk = out[r * (rank + 1):(r + 1) * (rank + 1), 0]
            assert torch.equal(blk, (torch.arange(start, start + rank + 1).to(dtype) + 1000 * r).to(DEV))


@check('reducescatter')
def _():
    for dtype, dim in itertools.product([torch.float32, torch.float64, torch.int32], DIMS):
        rows = size * 4 + (1 if size > 1 else 0)  # first rank gets one extra row
        shape = [rows] + [5] * (dim - 1)
        mine = rand(shape, dtype, 50 + rank)
        total = torch.stack([rand(shape, dtype, 50 + r).double() for r in range(size)]).sum(0)
        counts = [rows // size + (1 if r < rows % size else 0) for r in range(size)]
        off = sum(counts[:rank])
        out = hvd.reducescatter(mine, op=hvd.Sum)
        assert out.shape[0] == counts[rank]
        torch.testing.assert_close(out.double(), total[off:off + counts[rank]], **tol(dtype))
        if dtype.is_floating_point:
            avg = hvd.reducescatter(mine, op=hvd.Average)
            torch.testing.assert_close(avg.double(), total[off:off + counts[rank]] / size, **tol(dtype))
    outs = hvd.grouped_reducescatter([rand([size * 2, 3], torch.float32, 60 + rank), rand([size, 2], torch.float32, 70 + rank)], op=hvd.Sum)
    assert outs[0].shape == (2, 3) and outs[1].shape == (1, 2)


@check('fused_other_collectives')
def _():
    """Allgather / reducescatter / broadcast responses negotiated in one cycle are fused (one launch on GPUs): many small
    async ops with ragged sizes, values checked, and fewer responses than tensors in the engine's metrics
    (reference: controller.cc:915-918 reducescatter, :1003-1086 allgather fusion)."""
    m0 = hvd.metrics()
    K = 12
    # allgather: tensor k has (rank + k) % 3 + 1 rows of k + 1 columns
    ag_in = [torch.full([(rank + k) % 3 + 1, k + 1], float(rank * 100 + k), device=DEV) for k in range(K)]
    hs = [hvd.allgather_async(t, name='fo.ag.%d' % k) for k, t in enumerate(ag_in)]
    outs = [hvd.synchronize(h) for h in hs]
    for k, g in enumerate(outs):
        off = 0
        for r in range(size):
            n = (r + k) % 3 + 1
            assert g.shape[1] == k + 1 and (g[off:off + n] == r * 100 + k).all(), (k, r, g)
            off += n
        assert g.shape[0] == off
    # reducescatter: ragged first dims (not multiples of size)
    rs_in = [rand([size * 2 + k % 3, k % 4 + 1], torch.float32, 900 + 17 * k + rank) for k in range(K)]
    hs = [hvd.reducescatter_async(t, op=hvd.Sum, name='fo.rs.%d' % k) for k, t in enumerate(rs_in)]
    outs = [hvd.synchronize(h) for h in hs]
    for k, out in enumerate(outs):
        rows = size * 2 + k % 3
        total = torch.stack([rand([rows, k % 4 + 1], torch.float32, 900 + 17 * k + r).double() for r in range(size)]).sum(0)
        counts = [rows // size + (1 if r < rows % size else 0) for r in range(size)]
        off = sum(counts[:rank])
        torch.testing.assert_close(out.double(), total[off:off + counts[rank]], rtol=1e-5, atol=1e-5)
    # broadcast: two roots interleaved, mixed dtypes, odd byte counts
    bc = []
    for k in range(K):
        dt = [torch.float32, torch.uint8, torch.int64][k % 3]
        bc.append(torch.full([k * 3 + 1], rank + 1, dtype=dt, device=DEV))
    hs = [hvd.broadcast_async_(t, root_rank=k % min(size, 2), name='fo.bc.%d' % k) for k, t in enumerate(bc)]
    for h in hs:
        hvd.synchronize(h)
    for k, t in enumerate(bc):
        assert (t == k % min(size, 2) + 1).all(), (k, t)
    m1 = hvd.metrics()
    for op in ('allgather', 'reducescatter', 'broadcast'):
        tensors = m1[op]['tensors'] - m0.get(op, {}).get('tensors', 0)
        responses = m1[op]['responses'] - m0.get(op, {}).get('responses', 0)
        assert tensors == K, (op, tensors)
        if os.environ.get('HOROVOD_FUSION_THRESHOLD', '') != '0':
            assert responses < tensors, (op, responses, tensors)


@check('large_allreduce')
def _():
    """Large fused responses of ordinary tensors (GPU: the three-phase kernel, several segments of the symmetric buffer):
    exact integer-valued sums so every element can be checked."""
    big = (5 << 20) if args.device == 'cuda' else (1 << 18)
    for dtype in (torch.float32, torch.bfloat16):
        sizes = [big + 3, 1001, big // 2 + 17, 7, big]
        ts = [(torch.arange(n, device=DEV) % 13 + rank).to(dtype) for n in sizes]
        hs = [hvd.allreduce_async_(t, op=hvd.Sum, name='large.%s.%d' % (dtype, i)) for i, t in enumerate(ts)]
        for h in hs:
            hvd.synchronize(h)
        for n, t in zip(sizes, ts):
            exp = ((torch.arange(n, device=DEV) % 13) * size + sum(range(size))).to(dtype)
            assert torch.equal(t, exp), (dtype, n, t[:5], exp[:5], int((t != exp).sum()))
    # one large tensor, averaged, not in place
    x = torch.full([3 * big + 5], float(rank + 1), device=DEV)
    y = hvd.allreduce(x, op=hvd.Average, name='large.avg')
    assert torch.allclose(y, torch.full_like(y, (size + 1) / 2.0)) and float(x[0]) == rank + 1


@check('wire_dtype_env')
def _():
    """HVD_WIRE_DTYPE=bf16|fp16: fp32 tensors travel as 16-bit values (cast fused into the pack / unpack phases of the
    allreduce kernel, fp32 accumulation).  Values within 16-bit tolerance; on GPUs with the knob set the result must differ
    from the exact fp32 sum somewhere (i.e. the compression really happened)."""
    ts = [rand([n], torch.float32, 400 + rank * 7 + i) for i, n in enumerate([100003, 17, 65536])]
    hs = [hvd.allreduce_async(t, op=hvd.Sum, name='wire.%d' % i) for i, t in enumerate(ts)]
    outs = [hvd.synchronize(h) for h in hs]
    exact = True
    for i, n in enumerate([100003, 17, 65536]):
        ref = sum(rand([n], torch.float32, 400 + r * 7 + i).double() for r in range(size)).float()
        torch.testing.assert_close(outs[i], ref, rtol=2e-2, atol=2e-2 * size)
        exact = exact and bool(torch.allclose(outs[i], ref, rtol=1e-6, atol=1e-6))
    if args.device == 'cuda' and size > 1 and os.environ.get('HVD_WIRE_DTYPE', 'none') in ('bf16', 'fp16') and \
            os.environ.get('HVD_GPU_BACKEND', 'p2p') == 'p2p':
        assert not exact, 'HVD_WIRE_DTYPE is set but the sums are exact to fp32 precision'


@check('autograd')
def _():
    # allreduce: grad of sum-allreduce is sum-allreduce of ones
    x = torch.ones(5, device=DEV, requires_grad=True)
    y = hvd.allreduce(x, op=hvd.Sum)
    y.sum().backward()
    assert torch.allclose(x.grad, torch.full((5,), float(size), device=DEV))
    # allgather
    x = torch.ones(rank + 1, 3, device=DEV, requires_grad=True)
    g = hvd.allgather(x)
    (g * (torch.arange(g.shape[0], device=DEV).float().unsqueeze(1))).sum().backward()
    off = sum(r + 1 for r in range(rank))
    exp = torch.arange(off, off + rank + 1, device=DEV).float().unsqueeze(1).expand(-1, 3)
    assert torch.allclose(x.grad, exp), (x.grad, exp)
    # broadcast
    x = torch.ones(4, device=DEV, requires_grad=True)
    b = hvd.broadcast(x, 0)
    b.sum().backward()
    assert torch.allclose(x.grad, torch.full((4,), 1.0 if rank == 0 else 0.0, device=DEV))
    # alltoall
    x = torch.ones(size * 2, device=DEV, requires_grad=True)
    a = hvd.alltoall(x)
    (a * (rank + 1)).sum().backward()
    exp = torch.cat([torch.full((2,), float(r + 1)) for r in range(size)]).to(DEV)
    assert torch.allclose(x.grad, exp)
    # reducescatter (Sum): grad = allgather(grad * size)
    x = torch.ones(size * 2, 2, device=DEV, requires_grad=True)
    r_ = hvd.reducescatter(x, op=hvd.Sum)
    r_.sum().backward()
    assert torch.allclose(x.grad, torch.full((size * 2, 2), float(size), device=DEV))


@check('process_sets')
def _():
    if size < 2:
        return
    evens = hvd.add_process_set([r for r in range(size) if r % 2 == 0])
    odds = hvd.add_process_set([r for r in range(size) if r % 2 == 1])
    mine = evens if rank % 2 == 0 else odds
    assert mine.included() and mine.size() == len(mine.ranks)
    assert mine.rank() == mine.ranks.index(rank)
    t = torch.full((8,), float(rank), device=DEV)
    out = hvd.allreduce(t, op=hvd.Sum, process_set=mine)
    assert torch.allclose(out, torch.full((8,), float(sum(mine.ranks)), device=DEV))
    g = hvd.allgather(torch.full((1,), float(rank), device=DEV), process_set=mine)
    assert g.tolist() == [float(r) for r in mine.ranks]
    # broadcast root is a GLOBAL rank
    root = mine.ranks[-1]
    b = hvd.broadcast(torch.full((3,), float(rank), device=DEV), root, process_set=mine)
    assert (b == root).all()
    other = odds if rank % 2 == 0 else evens
    try:
        hvd.allreduce(t, process_set=other)
        raise AssertionError('allreduce on a foreign process set must fail')
    except (ValueError, HorovodInternalError):
        pass
    # the global set still works while subsets exist
    out = hvd.allreduce(t, op=hvd.Sum)
    assert torch.allclose(out, torch.full((8,), float(sum(range(size))), device=DEV))
    assert hvd.remove_process_set(odds) and hvd.remove_process_set(evens)
    assert odds.process_set_id is None


@check('errors')
def _():
    if size < 2:
        return
    # mismatched shapes
    try:
        hvd.allreduce(torch.ones(rank + 1, device=DEV), name='err.shape')
        raise AssertionError('shape mismatch must raise')
    except HorovodInternalError as e:
        assert 'shape' in str(e).lower(), e
    # mismatched dtypes
    try:
        hvd.allreduce(torch.ones(3, device=DEV, dtype=torch.float32 if rank % 2 == 0 else torch.float64), name='err.dtype')
        raise AssertionError('dtype mismatch must raise')
    except HorovodInternalError as e:
        assert 'type' in str(e).lower(), e
    # broadcast root mismatch
    try:
        hvd.broadcast(torch.ones(3, device=DEV), root_rank=rank, name='err.root')
        raise AssertionError('root mismatch must raise')
    except HorovodInternalError as e:
        assert 'root' in str(e).lower(), e
    # allgather trailing-dim mismatch
    try:
        hvd.allgather(torch.ones(2, rank + 2, device=DEV), name='err.ag')
        raise AssertionError('allgather dim mismatch must raise')
    except HorovodInternalError:
        pass
    # duplicate in-flight name.  A name is in flight until its response starts executing, which cannot happen before EVERY rank
    # submitted it: rank 0 submits late, so on the other ranks the second submission deterministically meets the first.
    t = torch.ones(1 << 18, device=DEV)
    if rank == 0:
        time.sleep(1.0)
        hvd.synchronize(hvd.allreduce_async(t, name='dup'))
    else:
        h = hvd.allreduce_async(t, name='dup')
        try:
            hvd.allreduce_async(t, name='dup')
            raise AssertionError('a second in-flight submission of the same name must be rejected')
        except (ValueError, HorovodInternalError) as e:
            assert 'dup' in str(e), e
        hvd.synchronize(h)
    # the library stays usable after errors
    assert torch.allclose(hvd.allreduce(torch.ones(2, device=DEV), op=hvd.Sum), torch.full((2,), float(size), device=DEV))


@check('cache_invalidation')
def _():
    """Same name, then a different shape under the same name: the cached response must be invalidated everywhere."""
    for step in range(3):
        out = hvd.allreduce(torch.ones(8, device=DEV), op=hvd.Sum, name='cache.t')
        assert torch.allclose(out, torch.full((8,), float(size), device=DEV))
    out = hvd.allreduce(torch.ones(12, device=DEV), op=hvd.Sum, name='cache.t')
    assert out.shape[0] == 12 and torch.allclose(out, torch.full((12,), float(size), device=DEV))
    out = hvd.allreduce(torch.ones(12, device=DEV, dtype=torch.float64), op=hvd.Sum, name='cache.t')
    assert out.dtype == torch.float64


@check('barrier_join')
def _():
    hvd.barrier()
    if size < 2:
        assert hvd.join() == 0
        return
    # ranks do a different number of steps; joined ranks contribute zeros; Average divides by the full size
    steps = rank + 1
    for s in range(steps):
        out = hvd.allreduce(torch.ones(4, device=DEV), name=f'join.{s}')
        active = sum(1 for r in range(size) if r + 1 > s)
        assert torch.allclose(out, torch.full((4,), active / size, device=DEV)), (s, out)
    last = hvd.join()
    assert last == size - 1, last
    hvd.barrier()


@check('objects_and_state')
def _():
    obj = hvd.broadcast_object({'a': rank, 'b': [1, 2, 3]}, root_rank=0)
    assert obj == {'a': 0, 'b': [1, 2, 3]}
    objs = hvd.allgather_object({'rank': rank})
    assert [o['rank'] for o in objs] == list(range(size))
    model = torch.nn.Linear(4, 3).to(DEV)
    with torch.no_grad():
        for p_ in model.parameters():
            p_.fill_(float(rank))
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)
    for p_ in model.parameters():
        assert (p_ == 0).all()
    for cls, kw in [(torch.optim.SGD, dict(lr=0.1 * (rank + 1), momentum=0.9)), (torch.optim.Adam, dict(lr=0.01 * (rank + 1))),
                    (torch.optim.AdamW, dict(lr=0.02 * (rank + 1))), (torch.optim.RMSprop, dict(lr=0.03 * (rank + 1)))]:
        opt = cls(model.parameters(), **kw)
        model(torch.randn(2, 4, device=DEV)).sum().backward()
        opt.step()
        hvd.broadcast_optimizer_state(opt, root_rank=0)
        lr0 = hvd.broadcast_object(opt.param_groups[0]['lr'], 0)
        assert abs(opt.param_groups[0]['lr'] - lr0) < 1e-12
        for st in opt.state.values():
            for k, v in st.items():
                if torch.is_tensor(v) and v.dim() > 0:
                    ref = hvd.broadcast(v.contiguous(), 0)
                    assert torch.allclose(v, ref)


@check('graphed_step')
def _():
    # hvd.GraphedStep on every rank: replayed forward/backward, reduction of all gradients in step(); the trajectory must
    # equal single-process training on the concatenated global batch
    if args.device != 'cuda':
        return
    def make():
        torch.manual_seed(11)
        return torch.nn.Sequential(torch.nn.Linear(16, 64), torch.nn.GELU(), torch.nn.Linear(64, 8)).to(DEV)
    model, ref_model = make(), make()
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)
    ref_model.load_state_dict(model.state_dict())
    for fused in (True,):
        opt = hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9),
                                       named_parameters=model.named_parameters(), fused=fused)
        ref_opt = torch.optim.SGD(ref_model.parameters(), lr=0.05, momentum=0.9)
        data = lambda step, r: (torch.randn(8, 16, generator=torch.Generator().manual_seed(50 * step + r)).to(DEV),
                                torch.randn(8, 8, generator=torch.Generator().manual_seed(70 * step + r)).to(DEV))
        gs = hvd.GraphedStep(lambda x, y: torch.nn.functional.mse_loss(model(x), y), opt, data(0, rank))
        assert gs.captured, gs.fallback_reason
        for step in range(5):
            gs(*data(step, rank))
            ref_opt.zero_grad()
            (sum(torch.nn.functional.mse_loss(ref_model(*data(step, r)[:1]), data(step, r)[1]) for r in range(size)) / size).backward()
            ref_opt.step()
        for a, b in zip(model.parameters(), ref_model.parameters()):
            torch.testing.assert_close(a, b, rtol=2e-4, atol=2e-5)


@check('optimizer')
def _():
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 4)).to(DEV)
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)
    ref_model = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 4)).to(DEV)
    ref_model.load_state_dict(model.state_dict())
    opt = hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9),
                                   named_parameters=model.named_parameters())
    ref_opt = torch.optim.SGD(ref_model.parameters(), lr=0.1, momentum=0.9)
    for step in range(4):
        # every rank sees different data; the reference model sees the whole global batch
        xs = [torch.randn(4, 8, generator=torch.Generator().manual_seed(100 * step + r)).to(DEV) for r in range(size)]
        ys = [torch.randn(4, 4, generator=torch.Generator().manual_seed(900 * step + r)).to(DEV) for r in range(size)]
        opt.zero_grad()
        torch.nn.functional.mse_loss(model(xs[rank]), ys[rank]).backward()
        opt.step()
        ref_opt.zero_grad()
        (sum(torch.nn.functional.mse_loss(ref_model(x), y) for x, y in zip(xs, ys)) / size).backward()
        ref_opt.step()
    for a, b in zip(model.parameters(), ref_model.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
    # gradient clipping pattern: synchronize() + skip_synchronize()
    opt.zero_grad()
    model(torch.randn(2, 8, device=DEV)).sum().backward()
    opt.synchronize()
    torch.nn.utils.clip_grad_norm_(model.parameters(), 0.1)
    with opt.skip_synchronize():
        opt.step()
    # backward_passes_per_step=2 with groups
    model2 = torch.nn.Linear(8, 2).to(DEV)
    hvd.broadcast_parameters(model2.state_dict(), 0)
    opt2 = hvd.DistributedOptimizer(torch.optim.SGD(model2.parameters(), lr=0.1), named_parameters=model2.named_parameters(),
                                    backward_passes_per_step=2, groups=1, compression=hvd.Compression.fp16)
    for _ in range(2):
        opt2.zero_grad()
        model2(torch.ones(1, 8, device=DEV) * (rank + 1)).sum().backward()
        model2(torch.ones(1, 8, device=DEV)).sum().backward()
        opt2.step()
    w = hvd.allgather(model2.weight.detach().reshape(1, -1).contiguous())
    for r in range(size):
        assert torch.allclose(w[r], w[0], atol=1e-3), 'weights diverged across ranks'
    # zero_grad race guard
    opt.zero_grad()
    model(torch.randn(2, 8, device=DEV)).sum().backward()
    try:
        opt.zero_grad()
        raise RuntimeError('zero_grad between backward and step must assert')
    except AssertionError:
        pass
    opt.step()
    # duplicate names are rejected
    try:
        hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.1),
                                 named_parameters=[('a', p_) for p_ in model.parameters()])
        raise RuntimeError('duplicate names must raise')
    except ValueError:
        pass


@check('force_allreduce')
def _():
    """A parameter whose gradient is not produced on some ranks is still reduced (zeros) so ranks stay in lock-step."""
    class Two(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.a = torch.nn.Linear(4, 1)
            self.b = torch.nn.Linear(4, 1)

        def forward(self, x, use_b):
            return self.b(x) if use_b else self.a(x)

    m = Two().to(DEV)
    hvd.broadcast_parameters(m.state_dict(), 0)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters())
    opt.zero_grad()
    m(torch.ones(2, 4, device=DEV), use_b=(rank % 2 == 1)).sum().backward()
    opt.step()
    w = hvd.allgather(torch.cat([p_.detach().reshape(-1) for p_ in m.parameters()]).reshape(1, -1).contiguous())
    for r in range(size):
        assert torch.allclose(w[r], w[0]), 'ranks diverged'


@check('sync_batch_norm')
def _():
    torch.manual_seed(1)
    bn = hvd.SyncBatchNorm(3).to(DEV)
    ref = torch.nn.BatchNorm1d(3).to(DEV)
    xs = [torch.randn(4, 3, generator=torch.Generator().manual_seed(r)).to(DEV) for r in range(size)]
    x = xs[rank].clone().requires_grad_(True)
    y = bn(x)
    full = torch.cat(xs).clone().requires_grad_(True)
    yr = ref(full)
    torch.testing.assert_close(y, yr[rank * 4:(rank + 1) * 4], rtol=1e-4, atol=1e-4)
    (y * (rank + 1)).sum().backward()
    w = torch.cat([torch.full((4, 3), float(r + 1)) for r in range(size)]).to(DEV)
    (yr * w).sum().backward()
    torch.testing.assert_close(x.grad, full.grad[rank * 4:(rank + 1) * 4], rtol=1e-3, atol=1e-4)
    torch.testing.assert_close(bn.running_mean, ref.running_mean, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(bn.running_var, ref.running_var, rtol=1e-4, atol=1e-5)
    assert int(bn.num_batches_tracked) == 1
    # momentum=None = cumulative moving average (torch.nn.BatchNorm semantics), two steps
    bn2, ref2 = hvd.SyncBatchNorm(3, momentum=None).to(DEV), torch.nn.BatchNorm1d(3, momentum=None).to(DEV)
    for it in range(2):
        xs2 = [torch.randn(4, 3, generator=torch.Generator().manual_seed(10 * it + r)).to(DEV) for r in range(size)]
        bn2(xs2[rank])
        ref2(torch.cat(xs2))
    torch.testing.assert_close(bn2.running_mean, ref2.running_mean, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(bn2.running_var, ref2.running_var, rtol=1e-4, atol=1e-5)
    assert int(bn2.num_batches_tracked) == 2
    # eval mode uses the running statistics and needs no communication; wrong input rank is rejected like in torch
    bn.eval()
    ref.eval()
    torch.testing.assert_close(bn(xs[rank]), ref(xs[rank]), rtol=1e-4, atol=1e-5)
    try:
        hvd.SyncBatchNorm(3).to(DEV)(torch.randn(3, device=DEV))
        raise AssertionError('1-D input accepted')
    except ValueError:
        pass


@check('adasum')
def _():
    if size & (size - 1):
        return
    # parallel vectors -> average; orthogonal vectors -> sum (reference test_adasum_pytorch.py)
    for dtype in [torch.float32, torch.float64] + ([torch.bfloat16, torch.float16] if DEV.type == 'cuda' else []):
        same = torch.arange(1, 65, device=DEV).to(dtype)
        out = hvd.allreduce(same.clone(), op=hvd.Adasum, name=f'adasum.par.{dtype}')
        torch.testing.assert_close(out, same, rtol=1e-2 if dtype.itemsize == 2 else 1e-4, atol=1e-4)
        ortho = torch.zeros(size * 8, device=DEV, dtype=dtype)
        ortho[rank * 8:(rank + 1) * 8] = rank + 1.0
        out = hvd.allreduce(ortho, op=hvd.Adasum, name=f'adasum.orth.{dtype}')
        exp = torch.cat([torch.full((8,), r + 1.0) for r in range(size)]).to(DEV).to(dtype)
        torch.testing.assert_close(out, exp, rtol=1e-2 if dtype.itemsize == 2 else 1e-4, atol=1e-4)
    # fused (several tensors in flight): per-tensor coefficients
    hs = [hvd.allreduce_async(torch.full((16,), float(i + 1), device=DEV), op=hvd.Adasum, name=f'adasum.f.{i}') for i in range(4)]
    for i, h in enumerate(hs):
        torch.testing.assert_close(hvd.synchronize(h), torch.full((16,), float(i + 1), device=DEV), rtol=1e-4, atol=1e-4)


@check('adasum_stability')
def _():
    # every rank holds a multiple of the same direction, with magnitudes (a) near the smallest normal number of the dtype and
    # (b) spread geometrically from tiny to sqrt(max): the dot products / norms must not underflow or overflow, and Adasum of
    # parallel vectors is their average (reference test_adasum_pytorch.py::test_stability, ::test_stability_2)
    if size & (size - 1):
        return
    import math
    import numpy as np
    dtypes = [(torch.float32, np.float32)]  # like the reference: fp32 (+ fp16 on GPUs); the accumulators are fp64
    if DEV.type == 'cuda':
        dtypes.append((torch.float16, np.float16))
    for tdt, ndt in dtypes:
        rng = np.random.RandomState(2)
        N = 1024
        tiny, big = float(np.finfo(ndt).tiny), math.sqrt(float(np.finfo(ndt).max))
        a1 = rng.normal(0, tiny, (N, 1))
        r1 = rng.normal(0, 1, (size, 1))
        a2 = rng.normal(0, 1, (N, 1))
        r2 = np.array([big ** ((i + 1) / size) * tiny ** ((size - i - 1) / size) for i in range(size)]).reshape(size, 1)
        rng.shuffle(r2)
        for tag, a, rr in (('tiny', a1, r1), ('spread', a2, r2)):
            q = np.dot(a, rr.T).astype(ndt).astype(np.float64)
            t = torch.from_numpy(q[:, rank].astype(ndt)).to(DEV)
            hvd.allreduce_(t, op=hvd.Adasum, name=f'adasum.stab.{tag}.{tdt}')
            expected = q.sum(axis=1) / size
            got = t.double().cpu().numpy()
            denom = np.linalg.norm(expected)
            ratio = np.linalg.norm(expected - got) / denom if denom > 0 else np.linalg.norm(got)
            limit = {np.float16: 1e-2, np.float32: 1e-4, np.float64: 1e-8}[ndt]
            assert ratio < limit, (tag, tdt, ratio)


@check('adasum_whole_model')
def _():
    # graph-mode Adasum optimizer (one wrapped-optimizer step for the whole model, then all deltas) == per-parameter hooks
    if size & (size - 1):
        return
    def make():
        torch.manual_seed(5)
        return torch.nn.Sequential(torch.nn.Linear(6, 12), torch.nn.Tanh(), torch.nn.Linear(12, 3)).to(DEV)
    ma, mb = make(), make()
    oa = hvd.DistributedOptimizer(torch.optim.SGD(ma.parameters(), lr=0.1, momentum=0.9), named_parameters=ma.named_parameters(), op=hvd.Adasum)
    ob = hvd.DistributedOptimizer(torch.optim.SGD(mb.parameters(), lr=0.1, momentum=0.9), named_parameters=mb.named_parameters(), op=hvd.Adasum)
    ob._graph_mode = True
    for step in range(3):
        x = torch.randn(5, 6, generator=torch.Generator().manual_seed(10 * step + rank)).to(DEV)
        y = torch.randn(5, 3, generator=torch.Generator().manual_seed(77 * step + rank)).to(DEV)
        for m, o in ((ma, oa), (mb, ob)):
            o.zero_grad()
            torch.nn.functional.mse_loss(m(x), y).backward()
            o.step()
    for a, b in zip(ma.parameters(), mb.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


@check('symm_zero_copy')
def _():
    """Registered symmetric tensors: in-place allreduce through the zero-copy kernel (and the packed path when small)."""
    if DEV.type != 'cuda' or size < 2 or not hvd.symm_available():
        return
    total = float(sum(range(1, size + 1)))
    for dtype in [torch.float32, torch.bfloat16]:
        t = hvd.symm_empty((1 << 20) + 24, dtype=dtype)          # > one-shot threshold -> zero-copy kernel
        for rep in range(3):
            t.fill_(rank + 1)
            hvd.allreduce_(t, op=hvd.Sum, name=f'zc.{dtype}')
            assert torch.allclose(t.float(), torch.full_like(t, total).float()), (dtype, rep, t[:4], t[-4:])
        t.fill_(rank + 1)
        hvd.allreduce_(t, op=hvd.Average, name=f'zc.avg.{dtype}', prescale_factor=2.0, postscale_factor=0.5)
        assert torch.allclose(t.float(), torch.full_like(t, total / size).float(), rtol=1e-2), t[:4]
        v = t[4096:4096 + (1 << 19)]                                # a view at an offset inside the region
        v.fill_(float(rank))
        hvd.allreduce_(v, op=hvd.Sum, name=f'zc.view.{dtype}')
        assert torch.allclose(v.float(), torch.full_like(v, float(sum(range(size)))).float())
        small = hvd.symm_empty(1000, dtype=dtype)                   # small: goes through the packed one-shot kernel
        small.fill_(1.0)
        hvd.allreduce_(small, op=hvd.Sum, name=f'zc.small.{dtype}')
        assert torch.allclose(small.float(), torch.full_like(small, float(size)).float())
    # min / max in place (no multicast for those)
    t = hvd.symm_empty(1 << 19, dtype=torch.float32)
    t.fill_(float(rank))
    hvd.allreduce_(t, op=hvd.Max, name='zc.max')
    assert (t == size - 1).all()
    # bucketed optimizer == plain optimizer
    torch.manual_seed(3)
    m1 = torch.nn.Sequential(torch.nn.Linear(256, 512), torch.nn.ReLU(), torch.nn.Linear(512, 512)).to(DEV)
    m2 = torch.nn.Sequential(torch.nn.Linear(256, 512), torch.nn.ReLU(), torch.nn.Linear(512, 512)).to(DEV)
    hvd.broadcast_parameters(m1.state_dict(), 0)
    m2.load_state_dict(m1.state_dict())
    o1 = hvd.DistributedOptimizer(torch.optim.SGD(m1.parameters(), lr=0.05, momentum=0.9), named_parameters=m1.named_parameters(),
                                  zero_copy=True, fused=True, bucket_cap_mb=0.6)
    o2 = hvd.DistributedOptimizer(torch.optim.SGD(m2.parameters(), lr=0.05, momentum=0.9),
                                  named_parameters=[('b.' + k, v) for k, v in m2.named_parameters()], zero_copy=False)
    assert o1._zero_copy and len(o1._buckets) >= 2 and not o2._zero_copy
    for step in range(4):
        x = torch.randn(16, 256, generator=torch.Generator().manual_seed(10 * step + rank)).to(DEV)
        for m, o in ((m1, o1), (m2, o2)):
            o.zero_grad()
            m(x).square().mean().backward()
            o.step()
    for a, b in zip(m1.parameters(), m2.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


@check('timeline')
def _():
    import json, os, tempfile
    path = os.path.join(tempfile.gettempdir(), f'hvd_timeline_{os.getppid()}.json')
    hvd.start_timeline(path, mark_cycles=True)
    for i in range(5):
        hvd.allreduce(torch.ones(64, device=DEV), name=f'tl.{i % 2}')
    time.sleep(0.05)
    hvd.stop_timeline()
    hvd.barrier()
    time.sleep(0.2)
    if rank == 0:
        text = open(path).read()
        assert 'NEGOTIATE_ALLREDUCE' in text and 'ALLREDUCE' in text and 'CYCLE_START' in text, text[:500]
        json.loads(text)
        os.remove(path)


@check('reinit')
def _():
    for _ in range(2):
        hvd.shutdown()
        assert not hvd.is_initialized()
        hvd.init()
        assert hvd.rank() == rank and hvd.size() == size
        out = hvd.allreduce(torch.ones(3, device=DEV), op=hvd.Sum)
        assert torch.allclose(out, torch.full((3,), float(size), device=DEV))


failed = []
only = set(args.only.split(',')) if args.only else None
skip = set(args.skip.split(',')) if args.skip else set()
for fn in CHECKS:
    if (only and fn._check_name not in only) or fn._check_name in skip:
        continue
    t0 = time.time()
    try:
        fn()
        if DEV.type == 'cuda':
            torch.cuda.synchronize()
        if rank == 0:
            print(f'[ok] {fn._check_name} ({time.time() - t0:.2f}s)', flush=True)
    except Exception:
        failed.append(fn._check_name)
        print(f'[FAIL] rank {rank} {fn._check_name}\n{traceback.format_exc()}', flush=True)
        break
hvd.shutdown()
if failed:
    sys.exit(1)
if rank == 0:
    print('ALL OK', flush=True)
