"""Reducescatter, allgatherv, broadcast and alltoallv on N simulated ranks on one GPU, through the launch plans the engine
runs (`horovod_b200.ops.sim`: every rank's plan from csrc/ops/collective_plan.cc, the cross-rank agreement check, then
the real kernels and flag protocol on N streams).

Reducescatter is the one-shot reduce into separate out-descriptors, modelled as in test_gpu_collective_numerics.py
(whose helpers this file imports):  out = T(A(sum_r W(A(x_r * prescale)) * postscale)), combined in rank order.  Floats
are held to that file's accumulation bound; integers, MIN and MAX must match exactly, and every rank's block must carry
the same bits as the matching rows of a one-shot allreduce of the same inputs.  Allgatherv, broadcast and alltoallv move
bytes, so their outputs must equal torch.cat / indexing of the inputs byte for byte.

Every case writes into views of larger buffers filled with a sentinel, at byte offsets 0 and 1..15 (16 B vector and
byte paths), checks that the sentinel around each output and every input are untouched, and runs three times (ping-pong
buffer slots, barrier epochs).  Small buffer sizes (`cap`) force the windowed multi-launch paths.

Not covered here: the broadcast root's multicast store and reducescatter's multimem reduce; the simulated team has no
multicast object.  tests/test_gpu_multi.py covers them on real multi-GPU teams.
"""
import numpy as np
import pytest
import torch

from test_gpu_collective_numerics import (MAX, MIN, ONESHOT, PROD, SUM, as_bits, check_float, inject_nonfinite, make,
                                          narrowing, reference)

pytestmark = pytest.mark.gpu

AVG = 'avg'  # AVERAGE as the engine runs it: SUM with postscale / n
SENTINEL = 0xA5
PAD = 48  # sentinel bytes after every output view
REPEATS = 3
CTAS = [1, 3, 8, 32]
RS_DTYPES = [torch.float32, torch.bfloat16, torch.float16, torch.float64, torch.int32, torch.int64, torch.uint8]


@pytest.fixture(scope='module')
def sim():
    from horovod_b200.ops import sim
    return sim


def place(x, shift):
    """A copy of x as a view at byte offset `shift` (a multiple of its element size) of a sentinel-filled uint8 buffer."""
    nbytes = x.numel() * x.element_size()
    base = torch.full((shift + nbytes + PAD,), SENTINEL, dtype=torch.uint8, device='cuda')
    v = base[shift:shift + nbytes].view(x.dtype).view(x.shape)
    v.copy_(x)
    return base, v


def guarded_empty(shape, dtype, shift):
    return place(torch.zeros(shape, dtype=dtype, device='cuda'), shift)


def sentinel_intact(base, shift, nbytes, what):
    b = base.cpu()
    assert (b[:shift] == SENTINEL).all() and (b[shift + nbytes:] == SENTINEL).all(), 'bytes around %s changed' % what


def shift_for(dtype, k):
    """Byte offsets 0 and 1..15 where the element size allows it."""
    return (k * dtype.itemsize) % 16


def bytes_of(t):
    return t.contiguous().view(torch.uint8).view(-1) if t.numel() else torch.empty(0, dtype=torch.uint8, device=t.device)


# ---------------------------------------------------------------------------------------------------------------------
# reducescatter

def rs_rows(d0, n):
    return [d0 // n + (1 if q < d0 % n else 0) for q in range(n)]


def rs_case(sim, n, dtype, op, shapes, ctas, cap, pre, seed, nonfinite=False):
    """Runs reducescatter of tensors `shapes` (dim0, row) and checks every rank's block against the model and, bit for
    bit, against a one-shot allreduce of the same inputs."""
    kop, post = (SUM, 1.0 / n) if op == AVG else (op, 1.0)
    flat = make(n, [d0 * row for d0, row in shapes], dtype, kop, seed)
    if nonfinite and dtype.is_floating_point:
        big = max(range(len(shapes)), key=lambda i: shapes[i][0] * shapes[i][1])
        inject_nonfinite(flat, big)
    keep = [[x.clone() for x in row] for row in flat]
    ins, in_bases, outs, out_bases = [], [], [], []
    for r in range(n):
        irow, ibase, orow, obase = [], [], [], []
        for i, (d0, row) in enumerate(shapes):
            b, v = place(flat[r][i].view(d0, row), shift_for(dtype, i + r))
            irow.append(v)
            ibase.append(b)
            b, v = guarded_empty((rs_rows(d0, n)[r], row), dtype, shift_for(dtype, i + 2 * r + 1))
            orow.append(v)
            obase.append(b)
        ins.append(irow), in_bases.append(ibase), outs.append(orow), out_bases.append(obase)
    what = 'reducescatter n=%d %s op %s ctas=%d cap=%d' % (n, dtype, op, ctas, cap)
    # the first repeats reduce other data (stale bytes in a buffer slot cannot pass for the result), the last the inputs
    other = make(n, [d0 * row for d0, row in shapes], dtype, kop, seed + 1)
    for rep in range(REPEATS):
        for r in range(n):
            for i in range(len(shapes)):
                ins[r][i].view(-1).copy_(flat[r][i] if rep == REPEATS - 1 else other[r][i])
        sim.reducescatter(ins, outs, op=kop, prescale=pre, postscale=post, cap=cap, ctas=ctas)
    torch.cuda.synchronize()
    # the same inputs through a one-shot allreduce: each rank's block must be those rows, bit for bit
    ar = [[torch.empty_like(x) for x in row] for row in keep]
    sim.allreduce(keep, ar, op=kop, variant=ONESHOT, ctas=8, prescale=pre, postscale=post)
    torch.cuda.synchronize()
    for i, (d0, row) in enumerate(shapes):
        ref, bound, exact = reference(keep, i, ONESHOT, kop, dtype, dtype, pre, post)
        rows = rs_rows(d0, n)
        for q in range(n):
            lo, hi = sum(rows[:q]) * row, sum(rows[:q + 1]) * row
            o = outs[q][i].reshape(-1)
            w = '%s tensor %d (%d x %d) rank %d' % (what, i, d0, row, q)
            assert torch.equal(as_bits(o), as_bits(ar[q][i][lo:hi])), w + ': differs from the one-shot allreduce rows'
            if not exact:
                check_float(o, ref[lo:hi], bound[lo:hi], narrowing(ONESHOT, dtype, dtype), w)
            elif dtype.is_floating_point:
                keepm = ~torch.stack([x[i].isnan().cpu() for x in keep]).any(0)[lo:hi]
                assert torch.equal(o.cpu().double()[keepm], torch.as_tensor(ref[lo:hi]).double()[keepm]), w
            else:
                assert np.array_equal(o.cpu().numpy(), ref[lo:hi]), w
    for r in range(n):
        for i in range(len(shapes)):
            sentinel_intact(out_bases[r][i], shift_for(dtype, i + 2 * r + 1), outs[r][i].numel() * dtype.itemsize,
                            '%s output %d rank %d' % (what, i, r))
            assert torch.equal(bytes_of(ins[r][i]), bytes_of(keep[r][i])), '%s: input %d of rank %d changed' % (what, i, r)
            sentinel_intact(in_bases[r][i], shift_for(dtype, i + r), ins[r][i].numel() * dtype.itemsize, 'input')


def rs_shapes(n):
    """First dims 1, n-1 (ranks without rows), n and k*n + r, rows of 1, 3, 5 and 1000 elements."""
    dims = [1, n - 1, n, 3 * n + n // 2 + 1]
    return [(d0, row) for row in (1, 3, 5, 1000) for d0 in dims]


@pytest.mark.parametrize('op', [SUM, AVG, MIN, MAX, PROD])
@pytest.mark.parametrize('dtype', RS_DTYPES)
@pytest.mark.parametrize('n', [2, 3, 5, 8])
def test_reducescatter_matches_model(sim, n, dtype, op):
    pre = 0.5 if op != PROD else 1.0 if not dtype.is_floating_point else 0.75
    ctas = CTAS[(n + RS_DTYPES.index(dtype)) % 4]
    rs_case(sim, n, dtype, op, rs_shapes(n), ctas, 1 << 20, pre, seed=n * 31 + RS_DTYPES.index(dtype),
            nonfinite=op in (SUM, MIN, MAX))


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.int64])
@pytest.mark.parametrize('n', [3, 8])
def test_reducescatter_larger_than_the_buffer(sim, n, dtype):
    """A tensor whose blocks exceed the buffer (element windows over several launches) next to small tensors that share
    the launches' regions, with a buffer of 4 and 12 KiB."""
    for cap, ctas in ((4096, 3), (12288, 32)):
        shapes = [(5, 3), (7 * n + 2, 1000), (1, 1), (2 * n + 1, 5), (n - 1, 1000)]
        rs_case(sim, n, dtype, SUM, shapes, ctas, cap, 0.5, seed=cap + n)


def test_reducescatter_many_tensors_one_response(sim):
    n = 5
    shapes = [(d0, row) for d0, row in zip([1, 4, 5, 17, 0, 9, 2, 33, 6, 11] * 10, [1, 3, 5, 7, 2, 1000, 1, 3, 64, 9] * 10)]
    rs_case(sim, n, torch.float32, AVG, shapes, 8, 1 << 20, 0.5, seed=3)
    rs_case(sim, n, torch.bfloat16, SUM, shapes, 32, 65536, 1.0, seed=4)  # the same response over several launches


# ---------------------------------------------------------------------------------------------------------------------
# allgatherv, broadcast, alltoallv: exact bytes

EX_DTYPES = [torch.uint8, torch.int16, torch.float32, torch.float64]


def random_bytes(shape, dtype, g):
    nbytes = int(np.prod(shape)) * dtype.itemsize
    return torch.randint(0, 256, (nbytes,), dtype=torch.uint8, generator=g).cuda().view(dtype).view(shape)


def refill(rows, g):
    """New random bytes in every tensor, in place: each repeat of a case moves different data, so that bytes left over
    from an earlier call (a stale buffer slot, a missed tail) cannot pass for the right ones."""
    for row in rows:
        for t in row:
            t.copy_(random_bytes(t.shape, t.dtype, g))


def views(shapes, dtype, salt):
    """shapes[r][i] -> (tensors, bases, shifts): every tensor a view at byte offset 0..15 of a sentinel-guarded buffer."""
    ts, bs, ss = [], [], []
    for r, row in enumerate(shapes):
        trow, brow, srow = [], [], []
        for i, shape in enumerate(row):
            sh = shift_for(dtype, 3 * i + 5 * r + salt)
            b, v = guarded_empty(shape, dtype, sh)
            trow.append(v), brow.append(b), srow.append(sh)
        ts.append(trow), bs.append(brow), ss.append(srow)
    return ts, bs, ss


def check_guards(tensors, bases, shifts, what):
    for r, row in enumerate(tensors):
        for i, t in enumerate(row):
            sentinel_intact(bases[r][i], shifts[r][i], t.numel() * t.element_size(), '%s tensor %d rank %d' % (what, i, r))


def check_outputs(outs, bases, shifts, refs, what):
    for r, row in enumerate(outs):
        for i, o in enumerate(row):
            assert torch.equal(bytes_of(o), bytes_of(refs[r][i])), '%s: output %d of rank %d' % (what, i, r)
    check_guards(outs, bases, shifts, what + ' output')


def check_inputs(ins, keep, bases, shifts, what, skip=()):
    for r, row in enumerate(ins):
        for i, x in enumerate(row):
            if (r, i) not in skip:
                assert torch.equal(bytes_of(x), bytes_of(keep[r][i])), '%s: input %d of rank %d changed' % (what, i, r)
    check_guards(ins, bases, shifts, what + ' input')


# kXChunk of exchange_kernels.cu: chunk c of the symmetric buffer belongs to CTA c % grid, and the grid of a launch is
# ceil(buffer bytes used / 32 KiB) CTAs at most.  With an 8 KiB buffer every launch is one chunk and one working CTA (the
# windowed paths); with 512 KiB a fused launch spans up to 16 chunks, so tensors start in the middle of chunks, span
# several, and end in an odd tail whose chunk belongs to another CTA than their first chunk.
CHUNK = 32768
CAPS = [8192, 1 << 19]


def ag_case(sim, n, dtype, ctas, cap):
    g = torch.Generator().manual_seed(n * 100 + ctas + cap)
    esz = dtype.itemsize
    # per tensor: (row, every rank's first dim); odd byte counts, ranks that contribute nothing, blocks over several chunks
    # with tails, one tensor over `cap`
    rows = [1, 13, 1, 1, 3, 7, 1]
    dims = [[1 if r % 2 else 0 for r in range(n)],
            [r % 3 for r in range(n)],
            [(16 * 40 + 7) if r != 1 else 0 for r in range(n)],
            [2 * CHUNK // esz + 3 + 5 * r for r in range(n)],
            [cap // (3 * esz) + 5 * r for r in range(n)],             # blocks larger than the buffer
            [0] * n,
            [13 + r for r in range(n)]]
    ins, ibases, ishifts = views([[(dims[i][r], rows[i]) for i in range(len(rows))] for r in range(n)], dtype, 0)
    outs, obases, oshifts = views([[(sum(dims[i]), rows[i]) for i in range(len(rows))] for _ in range(n)], dtype, 1)
    for rep in range(REPEATS):
        refill(ins, g)
        keep = [[x.clone() for x in row] for row in ins]
        sim.allgatherv(ins, outs, cap=cap, ctas=ctas)
        torch.cuda.synchronize()
        what = 'allgatherv n=%d %s ctas=%d cap=%d repeat %d' % (n, dtype, ctas, cap, rep)
        ref = [torch.cat([keep[r][i] for r in range(n)]) for i in range(len(rows))]
        check_outputs(outs, obases, oshifts, [ref] * n, what)
        check_inputs(ins, keep, ibases, ishifts, what)


def bc_case(sim, n, root, inplace, ctas, cap):
    g = torch.Generator().manual_seed(n * 10 + root + cap)
    sizes = [1, 13, 16 * 300 + 7, 0, 2 * CHUNK + 7, 3 * cap + 5, 16, 5 * CHUNK + 9, 2 * cap]
    ins, ibases, ishifts = views([[(s,) for s in sizes] for _ in range(n)], torch.uint8, 0)
    outs, obases, oshifts = views([[(s,) for s in sizes] for _ in range(n)], torch.uint8, 1)
    if inplace:
        outs[root], obases[root], oshifts[root] = ins[root], ibases[root], ishifts[root]
    for rep in range(REPEATS):
        refill(ins, g)  # every rank's input differs: only the root's may be read
        keep = [[x.clone() for x in row] for row in ins]
        sim.broadcast(ins, outs, root, cap=cap, ctas=ctas)
        torch.cuda.synchronize()
        what = 'broadcast n=%d root %d %s ctas=%d cap=%d repeat %d' % (n, root, 'in place' if inplace else 'out of place', ctas,
                                                                       cap, rep)
        check_outputs(outs, obases, oshifts, [keep[root]] * n, what)
        check_inputs(ins, keep, ibases, ishifts, what, skip={(root, i) for i in range(len(sizes))} if inplace else ())


def a2a_case(sim, n, dtype, ctas, cap):
    g = torch.Generator().manual_seed(n * 7 + ctas + cap)
    esz = dtype.itemsize
    rs = np.random.default_rng(n * 1000 + ctas + esz + cap)
    rows = [1, 5, 3]
    splits = []
    for i, row in enumerate(rows):
        hi = max(2, (2 * cap) // (n * row * esz)) if i == 1 else 40  # tensor 1: blocks larger than cap / n
        S = rs.integers(0, hi, size=(n, n))
        S[rs.integers(0, n), :] = 0  # a rank that sends nothing
        S[:, rs.integers(0, n)] = 0  # a rank that receives nothing
        S[rs.random((n, n)) < 0.2] = 0
        splits.append(S.tolist())
    ins, ibases, ishifts = views([[(sum(splits[i][p]), rows[i]) for i in range(len(rows))] for p in range(n)], dtype, 0)
    outs, obases, oshifts = views([[(sum(splits[i][p][q] for p in range(n)), rows[i]) for i in range(len(rows))]
                                   for q in range(n)], dtype, 1)
    for rep in range(REPEATS):
        refill(ins, g)
        keep = [[x.clone() for x in row] for row in ins]
        sim.alltoallv(ins, outs, splits, cap=cap, ctas=ctas)
        torch.cuda.synchronize()
        refs = []
        for q in range(n):
            row_refs = []
            for i in range(len(rows)):
                parts = []
                for p in range(n):
                    start = sum(splits[i][p][:q])
                    parts.append(keep[p][i][start:start + splits[i][p][q]])
                row_refs.append(torch.cat(parts))
            refs.append(row_refs)
        what = 'alltoallv n=%d %s ctas=%d cap=%d repeat %d' % (n, dtype, ctas, cap, rep)
        check_outputs(outs, obases, oshifts, refs, what)
        check_inputs(ins, keep, ibases, ishifts, what)


NS = [2, 3, 5, 8]


@pytest.mark.parametrize('cap', CAPS)
@pytest.mark.parametrize('ctas', CTAS)
@pytest.mark.parametrize('dtype', EX_DTYPES)
@pytest.mark.parametrize('n', NS)
def test_allgatherv_exact(sim, n, dtype, ctas, cap):
    ag_case(sim, n, dtype, ctas, cap)


@pytest.mark.parametrize('cap', CAPS)
@pytest.mark.parametrize('n', NS)
def test_broadcast_every_root_exact(sim, n, cap):
    for root in range(n):
        for inplace in (False, True):
            bc_case(sim, n, root, inplace, CTAS[(root + 2 * inplace) % 4], cap)


@pytest.mark.parametrize('cap', CAPS)
@pytest.mark.parametrize('ctas', CTAS)
@pytest.mark.parametrize('dtype', EX_DTYPES)
@pytest.mark.parametrize('n', NS)
def test_alltoallv_exact(sim, n, dtype, ctas, cap):
    a2a_case(sim, n, dtype, ctas, cap)


def test_buffer_without_a_plan_launches_nothing(sim):
    """1000 B split 8 ways leaves no 128 B region per rank: no plan, and the simulation refuses before any launch.  A
    4 KiB buffer (512 B per rank) works."""
    n = 8
    ins = [[torch.ones(8, 4, device='cuda')] for _ in range(n)]
    outs = [[torch.empty(1, 4, device='cuda')] for _ in range(n)]
    with pytest.raises(RuntimeError, match='-5'):
        sim.reducescatter(ins, outs, cap=1000)
    sim.reducescatter(ins, outs, cap=4096)
    torch.cuda.synchronize()
    assert all(torch.equal(o[0], torch.full((1, 4), float(n), device='cuda')) for o in outs)
