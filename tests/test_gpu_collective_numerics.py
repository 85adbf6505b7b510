"""Numerics of the collective kernels against a high-precision model of each variant's data path, on N simulated ranks
on one GPU (`horovod_b200.ops.sim`: N buffers, N concurrently running kernels, the real cross-GPU flag protocol).

The model (W = round to the wire dtype, T = round to the tensor dtype, A = the accumulator: fp32 for 16 / 32-bit floats,
fp64 for fp64, int32 for 8 / 16 / 32-bit integers, int64 for int64):

    pack (every fused variant)   w_r = W(A(x_r * prescale))     integers: trunc(double(x_r) * prescale), wrapped
    one-shot                     T(A(sum_r w_r * postscale))
    two-shot                     T(W(A(sum_r w_r * postscale)))  (the owner rounds to the wire before broadcasting)
    zero-copy in-place           W(A(sum_r x_r * scale))

Floats are compared with the accumulation bound |out - ref| <= (n-1) u_A sum_r |w_r| |postscale| (plus one rounding of
the product by a postscale != 1 and one ulp of every narrowing cast after the accumulation), never a flat tolerance;
integers, MIN and MAX exactly.  Every rank must also hold the same bits as rank 0, and the variants the same bits as each
other: data-parallel replicas must not drift apart.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ONESHOT, TWOSHOT, INPLACE = 0, 1, 'inplace'
SUM, MIN, MAX, PROD = 1, 3, 4, 5
FLOATS = [torch.float32, torch.float64, torch.bfloat16, torch.float16]
INTS = [torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64]
# mantissa bits (with the implicit one) and the smallest normal exponent: one ulp of a value of that dtype
FMT = {torch.float16: (11, -14), torch.bfloat16: (8, -126), torch.float32: (24, -126), torch.float64: (53, -1022)}
BITS_VIEW = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
LD = np.longdouble
LD_EPS = float(np.finfo(LD).eps)


@pytest.fixture(scope='module')
def sim():
    from horovod_b200.ops import sim
    return sim


def acc_dtype(wire):
    if wire.is_floating_point:
        return torch.float64 if wire == torch.float64 else torch.float32
    return torch.int64 if wire == torch.int64 else torch.int32


def kernel_scale(s, acc):
    """The scale as the kernel applies it: fp32 for an fp32 accumulator, double otherwise."""
    return float(np.float32(s)) if acc == torch.float32 else float(s)


def ulp(x, dtype):
    p, emin = FMT[dtype]
    x = np.abs(np.asarray(x, dtype=np.float64))
    _, e = np.frexp(x)
    e = np.where(x == 0, emin, np.maximum(e.astype(np.int64) - 1, emin))
    return np.ldexp(1.0, e - (p - 1)).astype(LD)


def to_ld(t):
    return t.detach().double().cpu().numpy().astype(LD)


def as_bits(t):
    return t.view(BITS_VIEW[t.element_size()])


def pack_float(x, pre, wire):
    """w = W(A(x * prescale)) for a float tensor x (any device), as float64 on the CPU (exact)."""
    acc = acc_dtype(wire)
    return (x.double().cpu() * kernel_scale(pre, acc)).to(acc).to(wire).double()


def pack_int(x, pre, wire):
    """w = wrap_W(trunc(double(x) * prescale)) (or x when prescale == 1), as numpy int64."""
    v = x.cpu().numpy().astype(np.int64)
    if pre != 1.0:
        v = np.trunc(x.cpu().numpy().astype(np.float64) * pre).astype(np.int64)
    return v.astype(torch.empty(0, dtype=wire).numpy().dtype).astype(np.int64)


def narrowing(variant, dtype, wire):
    """Casts after the accumulation that can round (each costs one ulp in the bound)."""
    acc = acc_dtype(wire)
    chain = [wire, dtype] if variant == TWOSHOT else [wire] if variant == INPLACE else [dtype]
    out, prev = [], acc
    for d in chain:
        if FMT[d][0] < FMT[prev][0]:
            out.append(d)
        prev = d
    return out


def float_sum_ref(ws, post, acc, errs=None):
    """ws: the n combined values (longdouble arrays), errs: a bound on the error each already carries (or None).
    Returns (ref, bound) of A(sum * post), without the ulps of later narrowing casts."""
    n = len(ws)
    u = 2.0 ** -24 if acc == torch.float32 else 2.0 ** -53
    s = kernel_scale(post, acc)
    errs = errs or [np.zeros_like(ws[0])] * n
    total = sum(ws)
    mag = sum(np.abs(w) + e for w, e in zip(ws, errs))
    ref = total * LD(s)
    bound = abs(s) * (sum(errs) + LD(1.01 * (n - 1) * u + (n + 1) * LD_EPS) * mag)
    if s != 1.0:
        bound += LD(u) * (np.abs(ref) + bound)
    return ref, bound


def float_prod_ref(ws, post, acc, errs=None):
    n = len(ws)
    u = 2.0 ** -24 if acc == torch.float32 else 2.0 ** -53
    s = kernel_scale(post, acc)
    errs = errs or [np.zeros_like(ws[0])] * n
    ref, hi, lo = LD(1), LD(1), LD(1)
    for w, e in zip(ws, errs):
        ref, hi, lo = ref * w, hi * (np.abs(w) + e), lo * np.abs(w)
    bound = abs(s) * ((hi - lo) + LD(1.01 * (n - 1) * u + (n + 1) * LD_EPS) * hi)
    ref = ref * LD(s)
    if s != 1.0:
        bound += LD(u) * (np.abs(ref) + bound)
    return ref, bound


def minmax_exact(ws, op, post, variant, dtype, wire):
    """MIN / MAX: the result is one of the packed values, so the whole rounding chain is replayed exactly (float64 CPU
    tensors in, float64 out).  Positions with a NaN input are left to the rank-agreement checks."""
    st = torch.stack(ws)
    m = st.min(0).values if op == MIN else st.max(0).values
    acc = acc_dtype(wire)
    m = (m * kernel_scale(post, acc)).to(acc)
    for d in ([wire, dtype] if variant == TWOSHOT else [wire] if variant == INPLACE else [dtype]):
        m = m.to(d)
    return m.double()


def int_ref(ws, op, post, dtype, wire):
    """Exact integer model on numpy int64, wrapping where the kernel's accumulator / wire / tensor dtype wraps."""
    acc = np.int64 if wire == torch.int64 else np.int32
    r = ws[0].astype(acc)
    for w in ws[1:]:
        w = w.astype(acc)
        with np.errstate(over='ignore'):
            r = (r + w if op == SUM else r * w if op == PROD else np.minimum(r, w) if op == MIN else np.maximum(r, w)).astype(acc)
    if post != 1.0:
        r = np.trunc(r.astype(np.float64) * post).astype(np.int64).astype(acc)
    np_w = torch.empty(0, dtype=wire).numpy().dtype
    np_t = torch.empty(0, dtype=dtype).numpy().dtype
    return r.astype(np_w).astype(np_t)


def check_float(out, ref, bound, narrow, what):
    """out: CUDA tensor; ref / bound: longdouble arrays.  Non-finite positions must agree with the reference exactly."""
    o = to_ld(out)
    nan_o, nan_r = np.isnan(o), np.isnan(ref)
    assert np.array_equal(nan_o, nan_r), '%s: NaN at %s, reference NaN at %s' % (what, np.flatnonzero(nan_o)[:8], np.flatnonzero(nan_r)[:8])
    inf_o, inf_r = np.isinf(o), np.isinf(ref)
    assert np.array_equal(inf_o, inf_r), '%s: inf at %s, reference inf at %s' % (what, np.flatnonzero(inf_o)[:8], np.flatnonzero(inf_r)[:8])
    assert np.array_equal(o[inf_o], ref[inf_r]), what
    f = np.isfinite(ref)
    b = bound[f].copy()
    for d in narrow:
        b += ulp(np.maximum(np.abs(o[f]), np.abs(ref[f])), d)
    err = np.abs(o[f] - ref[f])
    bad = np.flatnonzero(err > b)
    assert bad.size == 0, '%s: %d of %d elements outside the bound, e.g. index %d: out %r ref %r |err| %r > %r' % (
        what, bad.size, f.sum(), bad[0], float(o[f][bad[0]]), float(ref[f][bad[0]]), float(err[bad[0]]), float(b[bad[0]]))


def run(sim, variant, ins, outs, op, ctas, wire=None, pre=1.0, post=1.0):
    if variant == INPLACE:
        assert pre == 1.0
        sim.inplace_allreduce([row[0] for row in ins], op=op, ctas=ctas, scale=post)
    else:
        sim.allreduce(ins, outs, op=op, variant=variant, ctas=ctas, wire_dtype=wire, prescale=pre, postscale=post)
    torch.cuda.synchronize()
    return ins if variant == INPLACE else outs


def make(n, sizes, dtype, op, seed):
    g = torch.Generator().manual_seed(seed)
    rows = []
    for _ in range(n):
        row = []
        for s in sizes:
            if dtype.is_floating_point:
                x = torch.randn(s, generator=g, dtype=torch.float64)
                x = 1 + 0.05 * x if op == PROD else x
            elif op == PROD:
                x = torch.randint(0 if dtype == torch.uint8 else -3, 4, (s,), generator=g)
            else:
                info = torch.iinfo(dtype)
                lo, hi = (info.min, info.max) if dtype.itemsize <= 2 else (-(1 << 20), 1 << 20)
                x = torch.randint(lo, hi + 1, (s,), generator=g, dtype=torch.int64)
            row.append(x.to(dtype).cuda())
        rows.append(row)
    return rows


def reference(ins, i, variant, op, dtype, wire, pre, post, errs=None):
    """(ref, bound, exact) of tensor i."""
    n = len(ins)
    if not dtype.is_floating_point:
        return int_ref([pack_int(ins[r][i], pre, wire) for r in range(n)], op, post, dtype, wire), None, True
    ws = [pack_float(ins[r][i], pre, wire) for r in range(n)]
    if op in (MIN, MAX):
        return minmax_exact(ws, op, post, variant, dtype, wire), None, True
    fn = float_sum_ref if op == SUM else float_prod_ref
    ref, bound = fn([w.numpy().astype(LD) for w in ws], post, acc_dtype(wire), errs)
    return ref, bound, False


def check_against_reference(outs, ins, variant, op, dtype, wire, pre, post, what, ranks=None):
    n = len(ins)
    for i in range(len(ins[0])):
        ref, bound, exact = reference(ins, i, variant, op, dtype, wire, pre, post)
        for r in (ranks if ranks is not None else range(n)):
            o = outs[r][i]
            if not exact:
                check_float(o, ref, bound, narrowing(variant, dtype, wire), '%s tensor %d rank %d' % (what, i, r))
            elif dtype.is_floating_point:
                keep = ~torch.stack([x[i].isnan().cpu() for x in ins]).any(0)
                assert torch.equal(o.cpu().double()[keep], ref[keep]), '%s tensor %d rank %d' % (what, i, r)
            else:
                assert np.array_equal(o.cpu().numpy(), ref), '%s tensor %d rank %d' % (what, i, r)


def assert_ranks_agree(outs, what):
    for r in range(1, len(outs)):
        for i, (a, b) in enumerate(zip(outs[0], outs[r])):
            if not torch.equal(as_bits(a), as_bits(b)):
                d = torch.nonzero(as_bits(a) != as_bits(b)).flatten()
                pytest.fail('%s tensor %d: rank %d differs from rank 0 in %d of %d elements (first at %d: %r vs %r)' % (
                    what, i, r, d.numel(), a.numel(), int(d[0]), a[d[0]].item(), b[d[0]].item()))


# ---------------------------------------------------------------------------------------------------------------------
# A. every rank holds the same bits, non-finite inputs included

NONFINITE_AT = (3, 5, 7, 11, 13)


def inject_nonfinite(ins, i):
    """+inf on rank 1; -inf on rank 0 against +inf on rank n-1 (NaN); NaN on the last rank; NaN on rank 0; +inf
    everywhere."""
    n = len(ins)
    ins[1][i][3] = float('inf')
    ins[0][i][5], ins[n - 1][i][5] = float('-inf'), float('inf')
    ins[n - 1][i][7] = float('nan')
    ins[0][i][11] = float('nan')
    for r in range(n):
        ins[r][i][13] = float('inf')


@pytest.mark.parametrize('op', [SUM, MIN, MAX, PROD])
@pytest.mark.parametrize('dtype', FLOATS)
@pytest.mark.parametrize('variant', [ONESHOT, TWOSHOT, INPLACE])
@pytest.mark.parametrize('n', [2, 3, 4, 6, 8])
def test_ranks_agree_bitwise(sim, n, variant, dtype, op):
    sizes = [81928] if variant == INPLACE else [1, 4099, 70001]
    ins = make(n, sizes, dtype, op, seed=n * 100 + op)
    inject_nonfinite(ins, len(sizes) - 1)
    keep = [[x.clone() for x in row] for row in ins]
    outs = [[torch.empty_like(x) for x in row] for row in ins]
    post = 1.0 / n if op == SUM else 1.0
    res = run(sim, variant, ins, outs, op, ctas=8, post=post)
    assert_ranks_agree(res, 'variant %s n=%d %s op %d' % (variant, n, dtype, op))
    if op == SUM:  # the non-finite pattern (AMP's overflow check reads it) is the reference's
        i = len(sizes) - 1
        ref, _, _ = reference(keep, i, variant, op, dtype, dtype, 1.0, post)
        o = to_ld(res[0][i])
        assert np.array_equal(np.isnan(o), np.isnan(ref)) and np.array_equal(np.isinf(o), np.isinf(ref))
        assert np.array_equal(o[np.isinf(o)], ref[np.isinf(ref)])
        assert [int(x) for x in np.flatnonzero(~np.isfinite(o))] == [3, 5, 7, 11, 13]


# ---------------------------------------------------------------------------------------------------------------------
# B. the variants agree: with the wire dtype equal to the tensor dtype, the same sum in the same (rank) order

@pytest.mark.parametrize('dtype', FLOATS)
@pytest.mark.parametrize('n', [2, 3, 5, 8])
def test_variants_agree_bitwise(sim, n, dtype):
    count = 3 * 8192 + 40  # several chunks per CTA, a multiple of 16 B in every dtype
    base = make(n, [count], dtype, SUM, seed=7 + n)
    results = {}
    for variant in (ONESHOT, TWOSHOT, INPLACE):
        ins = [[x.clone() for x in row] for row in base]
        outs = [[torch.empty_like(x) for x in row] for row in ins]
        results[variant] = run(sim, variant, ins, outs, SUM, ctas=8, post=1.0 / n)
    for variant in (TWOSHOT, INPLACE):
        for r in range(n):
            a, b = as_bits(results[ONESHOT][r][0]), as_bits(results[variant][r][0])
            assert torch.equal(a, b), 'variant %s rank %d differs from one-shot in %d elements' % (variant, r, int((a != b).sum()))


# ---------------------------------------------------------------------------------------------------------------------
# C. accuracy against the model, fused allreduce

C_SIZES = [1, 17, 4099, 40001]


@pytest.mark.parametrize('scales', [(1.0, 1.0), (0.5, 'n'), ('n', 0.5)], ids=['pre1-post1', 'pre0.5-post1/n', 'pre1/n-post0.5'])
@pytest.mark.parametrize('op', [SUM, MIN, MAX, PROD])
@pytest.mark.parametrize('dtype', INTS + FLOATS)
@pytest.mark.parametrize('variant', [ONESHOT, TWOSHOT])
@pytest.mark.parametrize('n', [2, 3, 5, 8])
def test_allreduce_matches_model(sim, n, variant, dtype, op, scales):
    pre, post = [1.0 / n if s == 'n' else s for s in scales]
    ins = make(n, C_SIZES, dtype, op, seed=n + 10 * op)
    outs = [[torch.empty_like(x) for x in row] for row in ins]
    run(sim, variant, ins, outs, op, ctas=8, pre=pre, post=post)
    check_against_reference(outs, ins, variant, op, dtype, dtype, pre, post, 'variant %d' % variant)


@pytest.mark.parametrize('op', [SUM, MAX])
@pytest.mark.parametrize('wire', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('variant', [ONESHOT, TWOSHOT])
@pytest.mark.parametrize('n', [2, 3, 5, 8])
def test_wire_compression_matches_model(sim, n, variant, wire, op):
    """fp32 tensors, 16-bit wire: one-shot keeps the fp32 sum, two-shot rounds it to the wire."""
    ins = make(n, C_SIZES, torch.float32, op, seed=n)
    outs = [[torch.empty_like(x) for x in row] for row in ins]
    run(sim, variant, ins, outs, op, ctas=8, wire=wire, pre=0.5, post=1.0 / n)
    check_against_reference(outs, ins, variant, op, torch.float32, wire, 0.5, 1.0 / n, 'variant %d' % variant)
    assert_ranks_agree(outs, 'wire %s' % wire)


# ---------------------------------------------------------------------------------------------------------------------
# D. integer edges: wrap-around, and int64 values no double can hold

@pytest.mark.parametrize('variant', [ONESHOT, TWOSHOT, INPLACE])
@pytest.mark.parametrize('n', [2, 3, 5, 8])
def test_integer_wrap_and_int64_exact(sim, n, variant):
    cases = [(torch.int8, 100), (torch.uint8, 200), (torch.int16, 30000), (torch.int32, (1 << 31) - 5),
             (torch.int64, (1 << 53) + 1), (torch.int64, (1 << 62) + 3)]
    for dtype, v in cases:
        if variant == INPLACE and dtype not in (torch.int32, torch.int64):
            continue
        count = 4096 + 4  # past the 4 KiB row in every dtype; 16 B multiples for the in-place kernel's int32 / int64
        rows = []
        for r in range(n):
            x = torch.full((count,), v, dtype=torch.int64)
            x[1::2] = v - 2 * r - 1   # odd offsets below 2^53 apart: lost by any path through double
            rows.append([x.to(dtype).cuda()])
        keep = [[x.clone() for x in row] for row in rows]
        outs = [[torch.empty_like(x) for x in row] for row in rows]
        res = run(sim, variant, rows, outs, SUM, ctas=4)
        ref = int_ref([x[0].cpu().numpy().astype(np.int64) for x in keep], SUM, 1.0, dtype, dtype)
        for r in range(n):
            assert np.array_equal(res[r][0].cpu().numpy(), ref), (dtype, v, r)


# ---------------------------------------------------------------------------------------------------------------------
# E. where an fp16 wire overflows

def test_fp16_wire_overflow_is_where_the_model_puts_it(sim):
    n = 8
    big = [[torch.full((4099,), 7e4, device='cuda') + torch.arange(4099, device='cuda') * 1e-3] for _ in range(n)]
    for variant in (ONESHOT, TWOSHOT):
        outs = [[torch.empty_like(x) for x in row] for row in big]
        run(sim, variant, big, outs, SUM, ctas=8, wire=torch.float16)
        assert torch.isinf(outs[0][0]).all(), 'values above 65504 must overflow when packed to fp16'
        # prescale 1/n is applied before the cast (7e4 / 8 fits) and postscale 0.5 before two-shot's owner rounds the
        # sum to the wire (the 7e4 mean itself would not fit)
        run(sim, variant, big, outs, SUM, ctas=8, wire=torch.float16, pre=1.0 / n, post=0.5)
        assert torch.isfinite(outs[0][0]).all()
        check_against_reference(outs, big, variant, SUM, torch.float32, torch.float16, 1.0 / n, 0.5, 'prescaled')
    mid = [[torch.full((4099,), 3e4, device='cuda')] for _ in range(n)]  # fits fp16, the sum (2.4e5) does not
    outs = [[torch.empty_like(x) for x in row] for row in mid]
    run(sim, ONESHOT, mid, outs, SUM, ctas=8, wire=torch.float16)
    assert torch.isfinite(outs[0][0]).all(), 'one-shot stores the fp32 sum'
    check_against_reference(outs, mid, ONESHOT, SUM, torch.float32, torch.float16, 1.0, 1.0, 'one-shot 3e4')
    run(sim, TWOSHOT, mid, outs, SUM, ctas=8, wire=torch.float16)
    assert torch.isinf(outs[0][0]).all(), 'two-shot rounds the sum to the fp16 wire before broadcasting it'


# ---------------------------------------------------------------------------------------------------------------------
# F. shapes inside one fused response

def boundary_counts(width):
    """Element counts at the kernel's byte boundaries: the 16 B vector, the 128 B descriptor alignment, the 4 KiB row,
    the 8 / 16 / 32 KiB trips and chunk sizes, +- one element."""
    out = []
    for b in (16, 128, 4096, 8192, 16384, 32768, 65536):
        c = b // width
        out += [c - 1, c, c + 1]
    return [c for c in out if c > 0]


GUARD = 64  # elements of sentinel on both sides of every output view


def guarded(shape_count, dtype, offset, fill):
    base = torch.full((shape_count + 2 * GUARD + 3,), fill, dtype=dtype, device='cuda')
    return base, base[GUARD + offset:GUARD + offset + shape_count]


@pytest.mark.parametrize('ctas', [1, 3, 8, 32])
@pytest.mark.parametrize('variant', [ONESHOT, TWOSHOT])
@pytest.mark.parametrize('dtype', [torch.uint8, torch.float16, torch.float32, torch.float64])
def test_shapes_in_one_response(sim, dtype, variant, ctas):
    n = 4
    counts = boundary_counts(dtype.itemsize)
    counts = counts[:3] + [0] + counts[3:] + [0, 5]  # empty tensors between non-empty ones and before the last one
    op = SUM
    ins = make(n, counts, dtype, op, seed=ctas)
    # tensors 1, 4, 7, ...: views at element offsets 1..3 of a larger buffer (no 16 B alignment, scalar paths)
    for r in range(n):
        for i in range(1, len(counts), 3):
            buf = torch.zeros(counts[i] + 32, dtype=dtype, device='cuda')
            k = 1 + i % 3
            buf[k:k + counts[i]] = ins[r][i]
            ins[r][i] = buf[k:k + counts[i]]
    keep = [[x.clone() for x in row] for row in ins]
    bases, outs = [], []
    for r in range(n):
        b_row, o_row = [], []
        for i, c in enumerate(counts):
            if i % 4 == 2:  # output aliases the input
                b_row.append(None)
                o_row.append(ins[r][i])
            else:
                b, o = guarded(c, dtype, i % 4, 77)
                b_row.append(b)
                o_row.append(o)
        bases.append(b_row)
        outs.append(o_row)
    post = 1.0 if dtype == torch.uint8 else 0.5
    run(sim, variant, ins, outs, op, ctas=ctas, post=post)
    check_against_reference(outs, keep, variant, op, dtype, dtype, 1.0, post, 'ctas=%d' % ctas)
    assert_ranks_agree(outs, 'shapes')
    for r in range(n):
        for i, (b, c) in enumerate(zip(bases[r], counts)):
            if b is None:
                continue
            k = GUARD + i % 4
            assert (b[:k] == 77).all() and (b[k + c:] == 77).all(), 'bytes outside output view %d of rank %d changed' % (i, r)
        for i in range(1, len(counts), 3):  # the bytes around an input view are never written
            buf = ins[r][i]._base
            if buf is not None and i % 4 != 2:
                k = 1 + i % 3
                assert (buf[:k] == 0).all() and (buf[k + counts[i]:] == 0).all()


@pytest.mark.parametrize('variant', [ONESHOT, TWOSHOT])
def test_many_tensors_one_response(sim, variant):
    n = 4
    sizes = [1, 3, 7, 64, 333, 4097, 0, 12, 1025, 2] * 32 + [100003]  # 321 tensors
    ins = make(n, sizes, torch.float32, SUM, seed=5)
    outs = [[torch.empty_like(x) for x in row] for row in ins]
    run(sim, variant, ins, outs, SUM, ctas=16, post=0.25)
    check_against_reference(outs, ins, variant, SUM, torch.float32, torch.float32, 1.0, 0.25, 'many tensors', ranks=[0, n - 1])
    assert_ranks_agree(outs, 'many tensors')


def test_tiny_response_leaves_ctas_idle(sim):
    """Fewer chunks than CTAs: the idle CTAs still take part in every barrier."""
    for n, ctas in ((2, 32), (4, 32), (8, 16)):
        ins = make(n, [5], torch.float32, SUM, seed=n)
        outs = [[torch.empty_like(x) for x in row] for row in ins]
        for variant in (ONESHOT, TWOSHOT):
            run(sim, variant, ins, outs, SUM, ctas=ctas)
            check_against_reference(outs, ins, variant, SUM, torch.float32, torch.float32, 1.0, 1.0, 'tiny')


# ---------------------------------------------------------------------------------------------------------------------
# G. zero-copy in-place allreduce

G_BYTES = [16, 4096 - 16, 4096 + 16, 3 * 32768 + 4096 + 48, 1 << 20]


@pytest.mark.parametrize('op', [SUM, MIN, MAX, PROD])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16, torch.float64, torch.int32, torch.int64])
@pytest.mark.parametrize('n', [2, 3, 4, 5, 6, 7, 8])
def test_inplace_allreduce_matches_model(sim, n, dtype, op):
    scale = 1.0 / n if op in (SUM, MIN, MAX) else 1.0
    for nbytes in G_BYTES:
        count = nbytes // dtype.itemsize
        ins = make(n, [count], dtype, op, seed=nbytes + n)
        keep = [[x.clone() for x in row] for row in ins]
        run(sim, INPLACE, ins, None, op, ctas=8, post=scale)
        check_against_reference(ins, keep, INPLACE, op, dtype, dtype, 1.0, scale, '%d B' % nbytes)
        assert_ranks_agree(ins, 'in-place %d B' % nbytes)
    # repeats: every launch re-reduces the previous result, which every rank holds
    count = G_BYTES[3] // dtype.itemsize
    ins = make(n, [count], dtype, op, seed=n)
    if op == PROD and dtype.is_floating_point:  # three launches raise the product to the n^2-th power: stay near 1
        for row in ins:
            row[0].copy_(1 + (row[0].double() - 1) / 50)
    xs = [row[0].clone() for row in ins]
    sim.inplace_allreduce([row[0] for row in ins], op=op, ctas=8, scale=scale, repeats=3)
    torch.cuda.synchronize()
    if not dtype.is_floating_point:
        ref = [x.cpu().numpy().astype(np.int64) for x in xs]
        for _ in range(3):
            ref = [int_ref(ref, op, scale, dtype, dtype).astype(np.int64)] * n
        assert np.array_equal(ins[0][0].cpu().numpy(), ref[0])
    elif op in (MIN, MAX):
        ref = [x.double().cpu() for x in xs]
        for _ in range(3):
            ref = [minmax_exact(ref, op, scale, INPLACE, dtype, dtype)] * n
        assert torch.equal(ins[0][0].cpu().double(), ref[0])
    else:
        ws, errs = [to_ld(x) for x in xs], None
        fn = float_sum_ref if op == SUM else float_prod_ref
        for _ in range(3):
            ref, bound = fn(ws, scale, acc_dtype(dtype), errs)
            bound = bound + (ulp(np.abs(ref) + bound, dtype) if FMT[dtype][0] < FMT[acc_dtype(dtype)][0] else 0)
            ws, errs = [ref] * n, [bound] * n
        check_float(ins[0][0], ref, bound, [], 'repeats=3')
    assert_ranks_agree(ins, 'in-place repeats')


def test_inplace_rejects_sizes_not_multiple_of_16_bytes(sim):
    n = 2
    ts = [torch.zeros(5, device='cuda') for _ in range(n)]  # 20 B
    with pytest.raises(RuntimeError):
        sim.inplace_allreduce(ts)
    ins = make(n, [4099], torch.float32, SUM, seed=1)
    outs = [[torch.empty_like(x) for x in row] for row in ins]
    with pytest.raises(RuntimeError):  # the fused kernel has variants 0 (one-shot), 1 (two-shot) and 2 (NVLS) only
        sim.allreduce(ins, outs, op=SUM, variant=3, ctas=8)
    # the rejected calls leave the simulated ranks in step: the next collectives through their buffers still add up
    for variant in (ONESHOT, TWOSHOT):
        run(sim, variant, ins, outs, SUM, ctas=8)
        check_against_reference(outs, ins, variant, SUM, torch.float32, torch.float32, 1.0, 1.0, 'after a rejected call')


# ---------------------------------------------------------------------------------------------------------------------
# H. Adasum

def adasum_oracle(vs, seg, nt):
    """fp64 pairwise adaptive sum in the VHDD tree order, per tensor; vs: one fp64 vector per rank (all tensors
    concatenated), seg: the tensor index of every element.  Coefficient 1 where a norm is below sqrt(DBL_MIN)."""
    if len(vs) == 1:
        return vs[0]
    h = len(vs) // 2
    a, b = adasum_oracle(vs[:h], seg, nt), adasum_oracle(vs[h:], seg, nt)

    def segsum(x):
        return torch.zeros(nt, dtype=torch.float64, device=x.device).index_add_(0, seg, x)
    dot, na, nb = segsum(a * b), segsum(a * a), segsum(b * b)
    tiny = 1.4916681462400413e-154
    ac = torch.where(na >= tiny, 1 - dot / (2 * na), torch.ones_like(na))
    bc = torch.where(nb >= tiny, 1 - dot / (2 * nb), torch.ones_like(nb))
    return ac[seg] * a + bc[seg] * b


def adasum_inputs(n, sizes, dtype, seed, zero_on=()):
    g = torch.Generator().manual_seed(seed)
    ins = [[torch.randn(s, generator=g).to(dtype).cuda() for s in sizes] for _ in range(n)]
    for i, ranks in zero_on:
        for r in ranks:
            ins[r][i].zero_()
    return ins


def adasum_check(ins, outs, pre, post, dtype):
    """Normwise per tensor, against the oracle applied to exactly the fp32 values the kernel packs.

    Bound: each of the L = log2(n) levels rounds the fp32 coefficients (1 u) and the combine a*ac + b*bc (2 u) with
    |ac|, |bc| of order 1 for these inputs, so a level adds at most ~4 u of the norms it combines, all of which are at most
    sum_r |w_r|; the first-order propagation of an earlier level's error through the coefficients is of the same size.
    8 L u sum_r |w_r| covers both with margin; the fp32 postscale product adds 2 u, a 16-bit output one ulp per element."""
    n, nt = len(ins), len(ins[0])
    u = 2.0 ** -24
    L = max(1, (n - 1).bit_length())
    sizes = [x.numel() for x in ins[0]]
    seg = torch.repeat_interleave(torch.arange(nt, device='cuda'), torch.tensor(sizes, device='cuda'))
    ws = [torch.cat([(x.float() * np.float32(pre)).double() for x in row]) for row in ins]
    ref = adasum_oracle(ws, seg, nt) * float(np.float32(post))

    def segnorm(x):
        return torch.zeros(nt, dtype=torch.float64, device='cuda').index_add_(0, seg, x * x).sqrt()
    scale = sum(segnorm(w) for w in ws) * abs(post)
    for r in range(n):
        o = torch.cat([x.double() for x in outs[r]])
        assert torch.isfinite(o).all()
        bound = (8 * L + 2) * u * scale
        if dtype != torch.float32:
            bound = bound + segnorm(torch.from_numpy(ulp(o.abs().cpu().numpy(), dtype).astype(np.float64)).cuda())
        err = segnorm(o - ref)
        bad = torch.nonzero(err > bound).flatten()
        assert bad.numel() == 0, 'rank %d: tensor %d (%d elements) error %g > bound %g' % (
            r, int(bad[0]), sizes[int(bad[0])], float(err[bad[0]]), float(bound[bad[0]]))
    return ref


def run_adasum(sim, monkeypatch, persistent, ins, ctas, pre, post):
    monkeypatch.setenv('HVD_ADASUM_PERSISTENT', '1' if persistent else '0')
    outs = [[torch.empty_like(x) for x in row] for row in ins]
    sim.adasum(ins, outs, ctas=ctas, prescale=pre, postscale=post)
    torch.cuda.synchronize()
    return outs


# 1..7-element tensors between large ones: boundaries inside a 4 KiB row and inside a CTA's slice; tensor 2 is zero on
# some ranks, tensor 6 on every rank (the sqrt(DBL_MIN) branch, coefficient 1)
H_SIZES = [40000, 3, 1500, 1, 7, 70001, 2049, 5, 2, 12345, 6, 4]
H_ZERO = ((2, (0,)), (6, 'all'))


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize('ctas', [1, 3, 8, 16])
@pytest.mark.parametrize('n', [2, 4, 8])
def test_adasum_matches_oracle(sim, monkeypatch, n, ctas, dtype):
    zero = [(i, range(n) if r == 'all' else [q for q in r] + ([n - 1] if n > 2 else [])) for i, r in H_ZERO]
    ins = adasum_inputs(n, H_SIZES, dtype, seed=n * ctas, zero_on=zero)
    pre, post = 0.5, 1.0 / n
    p1 = run_adasum(sim, monkeypatch, True, ins, ctas, pre, post)
    ref = adasum_check(ins, p1, pre, post, dtype)
    assert_ranks_agree(p1, 'persistent adasum')
    p2 = run_adasum(sim, monkeypatch, True, ins, ctas, pre, post)
    for r in range(n):  # fixed reduction orders: bit-reproducible
        for a, b in zip(p1[r], p2[r]):
            assert torch.equal(as_bits(a), as_bits(b))
    m = run_adasum(sim, monkeypatch, False, ins, ctas, pre, post)
    adasum_check(ins, m, pre, post, dtype)
    assert_ranks_agree(m, 'multi-launch adasum')
    assert all(bool((x == 0).all()) for row in p1 for x in row[6:7]) and all(bool((x == 0).all()) for row in m for x in row[6:7])
    del ref


@pytest.mark.parametrize('persistent', [True, False])
def test_adasum_many_tensors_and_limit(sim, monkeypatch, persistent):
    n = 4
    sizes = [1, 5, 64, 333, 7, 1025, 2, 4096, 3, 17] * 100  # 1000 tensors
    ins = adasum_inputs(n, sizes, torch.float32, seed=1, zero_on=((4, (1,)), (7, range(n))))
    outs = run_adasum(sim, monkeypatch, persistent, ins, 8, 1.0, 1.0)
    adasum_check(ins, outs, 1.0, 1.0, torch.float32)
    assert_ranks_agree(outs, 'adasum 1000 tensors')
    over = adasum_inputs(2, [3] * 1251, torch.float32, seed=2)
    with pytest.raises(RuntimeError):
        run_adasum(sim, monkeypatch, persistent, over, 8, 1.0, 1.0)
