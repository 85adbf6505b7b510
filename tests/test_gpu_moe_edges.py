"""hvd.ExpertDispatcher's kernels on inputs test_gpu_moe_dispatch never uses: non-finite values, signed zeros,
subnormals, fp16 overflow, bf16 / fp16 gates through the whole chain, top-k = 16, route tile edges, ids that a 32-bit
cast would corrupt, empty ranks and a capacity exactly at the received total.

Every gather / scatter case checks three things:
- bits: against the documented fp32 model (test_gpu_moe_dispatch.ref_gather: j ascending, each product rounded, one
  final rounding), NaN compared by mask and the sign of zero compared;
- value: against float64, within k 2^-24 sum |g v| plus one ulp of the output dtype (the gate gradient within
  test_gpu_moe_dispatch.dot_bound); where the float64 value rounded to the output dtype is not finite, the same inf /
  NaN;
- containment: every element no special value feeds is bit-identical to the same call on clean inputs.
No input lets only an intermediate partial sum overflow, where the answer depends on the order of the sum.
"""
import pytest
import torch

from optim_cases import ulp
from test_gpu_moe_dispatch import (OK, RECV_OVERFLOW, SimMoE, _bytes, _expert_fn, _permute, check_permute,
                                   check_sim, dot_bound, one_rank, ops, ref_gather, sim)  # noqa: F401  (fixtures)

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
GATES = ['fp32', 'same']
NAN, INF = float('nan'), float('inf')
# per row dtype: the non-finite, zero, subnormal and extreme values planted in rows
ROW_SPECIALS = {torch.float32: [INF, -INF, NAN, 0.0, -0.0, 1e-40, -3e-42, 1e7],
                torch.bfloat16: [INF, -INF, NAN, 0.0, -0.0, 1e-39, -4e-40, 1e7],
                torch.float16: [INF, -INF, NAN, 0.0, -0.0, 6e-8, -1.2e-7, 65504.0]}
GATE_SPECIALS = {torch.float32: [0.0, -0.0, NAN, INF, -INF, 1e30],
                 torch.bfloat16: [0.0, -0.0, NAN, INF, -INF, 1e30],
                 torch.float16: [0.0, -0.0, NAN, INF, -INF, 65504.0]}  # 1e30 is inf in fp16


# ---- float64 references and comparisons (pinned against torch on the CPU below) ---------------------------------------

def gather64(src, pos, gates=None):
    """(y, bound): y[t] = sum over the in-range j of gates[t, j] * src[pos[t, j]] in float64 (+0 with none in range), and
    k 2^-24 sum |g v| + k 2^-150, the error bound of the fp32 sum of rounded products (an underflowing product is off
    by up to 2^-150, half the least fp32 subnormal)."""
    rows, k = src.shape[0], pos.shape[1]
    y = torch.zeros(pos.shape[0], src.shape[1], dtype=torch.float64, device=src.device)
    mag = torch.zeros_like(y)
    for j in range(k):
        p = pos[:, j].long()
        inside = ((p >= 0) & (p < rows)).view(-1, 1)
        v = src[p.clamp(0, max(rows - 1, 0))].double()
        term = v if gates is None else gates[:, j:j + 1].double() * v
        term = torch.where(inside, term, torch.zeros((), dtype=torch.float64, device=src.device))
        y, mag = y + term, mag + term.abs()
    return y, k * 2.0 ** -24 * mag + k * 2.0 ** -150


def nan_bits(t):
    """The bits of t with every NaN replaced by one NaN, so NaNs compare by mask and not by payload."""
    t = torch.where(torch.isnan(t), torch.full_like(t, NAN), t)
    return t.contiguous().view({2: torch.int16, 4: torch.int32}[t.element_size()])


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(nan_bits(a), nan_bits(b))


def check_value(got, want64, bound, what):
    """got (any float dtype) against the float64 value: where want64 rounded to got's dtype is finite, within bound plus
    one ulp; elsewhere the same inf or NaN."""
    rounded = want64.to(got.dtype)
    fin = torch.isfinite(rounded)
    g = got.double()
    assert torch.equal(torch.isnan(g), torch.isnan(rounded.double())), (what, 'NaN mask')
    assert torch.equal(g[~fin & ~torch.isnan(g)], rounded.double()[~fin & ~torch.isnan(g)]), (what, 'inf')
    err = (g[fin] - want64[fin]).abs()
    tol = bound[fin] + ulp(want64[fin], got.dtype)
    assert bool((err <= tol).all()), (what, float((err - tol).max()))


def test_references_against_torch_cpu():
    """gather64, same_bits, ulp and check_value against plain torch on the CPU, on the edge values of this file."""
    g = torch.Generator().manual_seed(0)
    src = torch.tensor([[1.0, -0.0, INF], [2.5, NAN, -3.0], [1e30, 0.0, 5e-324]], dtype=torch.float64)
    pos = torch.tensor([[0, 2], [1, -1], [-1, 3], [2, 0]], dtype=torch.int32)
    gates = torch.randn(4, 2, generator=g, dtype=torch.float64)
    y, bound = gather64(src, pos, gates)
    want = torch.stack([gates[0, 0] * src[0] + gates[0, 1] * src[2], gates[1, 0] * src[1], torch.zeros(3, dtype=torch.float64),
                        gates[3, 0] * src[2] + gates[3, 1] * src[0]])
    torch.testing.assert_close(y, want, equal_nan=True, rtol=0, atol=0)
    assert torch.equal(torch.signbit(y[2]), torch.zeros(3, dtype=torch.bool)), 'the empty sum is +0'
    assert bound[2].tolist() == [2 * 2.0 ** -150] * 3
    y1, _ = gather64(src, pos)
    torch.testing.assert_close(y1[0], src[0] + src[2], equal_nan=True, rtol=0, atol=0)
    # the fp32 model of test_gpu_moe_dispatch is within the bound of the float64 sum where every position is in range
    s32 = torch.randn(50, 7, generator=g)
    p32 = torch.randint(0, 50, (30, 5), generator=g, dtype=torch.int32)
    g32 = torch.rand(30, 5, generator=g)
    w64, b64 = gather64(s32, p32, g32)
    check_value(ref_gather(s32, p32, g32, torch.float32), w64, b64, 'fp32 model')
    with pytest.raises(AssertionError):
        check_value(ref_gather(s32, p32, g32, torch.float32) * (1 + 2 ** -20), w64, b64, 'fp32 model, perturbed')
    # NaNs compare by mask whatever their payload; the sign of zero counts
    a = torch.tensor([0x7e00, 0x7e01, 0xfe00 - 0x10000, -0x8000, 0, 0x7c00], dtype=torch.int16).view(torch.float16)
    b = torch.tensor([0x7e00, 0x7e00, 0x7e00, -0x8000, 0, 0x7c00], dtype=torch.int16).view(torch.float16)
    assert same_bits(a, b) and not torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert not same_bits(torch.tensor([0.0]), torch.tensor([-0.0]))
    # ulp: the spacing of each dtype, subnormal at zero
    x = torch.tensor([1.0, 3.0, 0.0, 65504.0], dtype=torch.float64)
    for dt, want in ((torch.float32, [2.0 ** -23, 2.0 ** -22, 2.0 ** -149, 2.0 ** -8]),
                     (torch.bfloat16, [2.0 ** -7, 2.0 ** -6, 2.0 ** -133, 2.0 ** 8]),
                     (torch.float16, [2.0 ** -10, 2.0 ** -9, 2.0 ** -24, 32.0])):
        assert ulp(x, dt).tolist() == want, dt
    # check_value: the float64 value rounded to inf must be inf; one NaN too many fails
    check_value(torch.tensor([INF, -65504.0], dtype=torch.float16), torch.tensor([65520.0, -65519.0], dtype=torch.float64),
                torch.zeros(2, dtype=torch.float64), 'fp16 overflow')
    with pytest.raises(AssertionError):
        check_value(torch.tensor([NAN], dtype=torch.float16), torch.tensor([1.0], dtype=torch.float64),
                    torch.zeros(1, dtype=torch.float64), 'NaN')


# ---- gather and scaled scatter on special values -----------------------------------------------------------------------

def _plant(t, values, frac, seed):
    """A copy of t with a seeded fraction `frac` of its elements replaced by `values` (cycled)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    out = t.clone().view(-1)
    at = (torch.rand(out.numel(), device='cuda', generator=g) < frac).nonzero().flatten()
    vals = torch.tensor(values, dtype=torch.float64).to(t.dtype).cuda()
    out[at] = vals[torch.arange(at.numel(), device='cuda') % len(values)]
    return out.view_as(t)


def _changed(a, b):
    return nan_bits(a) != nan_bits(b)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('gate', GATES)
@pytest.mark.parametrize('h', [72, 67])
def test_gather_special_values(ops, dtype, gate, h):
    """Rows with +-inf, NaN, +-0, subnormals and large values, gates of +-0, NaN, +-inf and 1e30 (65504 in fp16): the
    weighted gather and the unit-gate gather.  h = 72: 16 B rows on the vector path; h = 67: the element path."""
    T, k, rows = 400, 4, 1200
    gd = torch.float32 if gate == 'fp32' else dtype
    g = torch.Generator(device='cuda').manual_seed(h)
    clean_src = torch.randn(rows, h, device='cuda', generator=g).to(dtype)
    pos = torch.stack([torch.randperm(rows, device='cuda', generator=g)[:T] for _ in range(k)], 1).to(torch.int32)
    clean_g = torch.rand(T, k, device='cuda', generator=g).to(gd)
    src = _plant(clean_src, ROW_SPECIALS[dtype], 0.01, seed=1)
    gates = _plant(clean_g, GATE_SPECIALS[gd], 0.05, seed=2)
    for gt, cgt in ((gates, clean_g), (None, None)):
        y = ops.moe_gather(src, pos, gt)
        y_clean = ops.moe_gather(clean_src, pos, cgt)
        assert same_bits(y, ref_gather(src, pos, gt, dtype)), 'bits'
        want, bound = gather64(src, pos, gt)
        check_value(y, want, bound, ('value', gt is not None))
        fed = torch.zeros(T, h, dtype=torch.bool, device='cuda')
        for j in range(k):
            p = pos[:, j].long()
            fed |= _changed(src[p], clean_src[p])
            if gt is not None:
                fed |= _changed(gt[:, j:j + 1], cgt[:, j:j + 1]).expand(T, h)
        assert bool(fed.any()) and not bool(fed.all())
        assert same_bits(y[~fed], y_clean[~fed]), 'containment'


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('gate', GATES)
@pytest.mark.parametrize('h', [72, 67])
def test_scaled_scatter_special_values(ops, dtype, gate, h):
    """The combine backward's scaled scatter with the gate-gradient dot, special values in grad_y, the gates and the
    dot rows: dst rows bit for bit round(g * grad_y), the gate gradient against float64 within dot_bound."""
    T, k = 300, 3
    rows = T * k + 7
    gd = torch.float32 if gate == 'fp32' else dtype
    g = torch.Generator(device='cuda').manual_seed(100 + h)
    pos = torch.randperm(rows, device='cuda', generator=g)[:T * k].view(T, k).to(torch.int32)  # every row written once
    clean_gy = torch.randn(T, h, device='cuda', generator=g).to(dtype)
    clean_r = torch.randn(rows, h, device='cuda', generator=g).to(dtype)
    clean_g = torch.rand(T, k, device='cuda', generator=g).to(gd)
    gy = _plant(clean_gy, ROW_SPECIALS[dtype], 0.005, seed=3)
    dot_rows = _plant(clean_r, ROW_SPECIALS[dtype], 0.003, seed=4)
    gates = _plant(clean_g, GATE_SPECIALS[gd], 0.05, seed=5)
    dst = torch.full((rows, h), 3.0, dtype=dtype, device='cuda')
    dst_clean = dst.clone()
    gg = ops.moe_scatter(gy, pos, dst, gates, dot_rows)
    gg_clean = ops.moe_scatter(clean_gy, pos, dst_clean, clean_g, clean_r)
    fed_g = torch.zeros(T, k, dtype=torch.bool, device='cuda')
    for j in range(k):
        p = pos[:, j].long()
        got = dst[p]
        assert same_bits(got, (gates[:, j:j + 1].float() * gy.float()).to(dtype)), ('bits', j)
        want = gates[:, j:j + 1].double() * gy.double()
        check_value(got, want, 2.0 ** -24 * want.abs(), ('value', j))
        fed = _changed(gy, clean_gy) | _changed(gates[:, j:j + 1], clean_g[:, j:j + 1]).expand(T, h)
        assert same_bits(got[~fed], dst_clean[p][~fed]), ('containment', j)
        exact = (gy.double() * dot_rows[p].double()).sum(-1)
        bound = dot_bound(gy, dot_rows[p])
        if gd != torch.float32:  # rounded once more, to the gates' dtype
            bound = bound + exact.abs().nan_to_num(0, 0, 0) * torch.finfo(gd).eps
        check_value(gg[:, j], exact, bound, ('gate gradient', j))
        fed_g[:, j] = (_changed(gy, clean_gy) | _changed(dot_rows[p], clean_r[p])).any(1)
    assert bool(fed_g.any()) and not bool(fed_g.all())
    assert same_bits(gg[~fed_g], gg_clean[~fed_g]), 'gate gradient containment'
    untouched = torch.ones(rows, dtype=torch.bool, device='cuda')
    untouched[pos.flatten().long()] = False
    assert bool((dst[untouched] == 3.0).all()), 'wrote a row no position names'


@pytest.mark.gpu
@pytest.mark.parametrize('gate', GATES)
def test_fp16_overflow_threshold(ops, gate):
    """fp16 rows whose fp32 sum lands just below 65520 (rounds to 65504) and exactly at it (rounds to inf), both signs;
    the fp32 sums are exact, so the model, float64 and the kernel agree bit for bit."""
    src = torch.tensor([32768.0, 32752.0, 15.5, 1.0], dtype=torch.float16, device='cuda').view(4, 1).repeat(1, 9)
    src = torch.cat([src, -src])
    pos = torch.tensor([[1, 1, 2], [0, 1, -1], [5, 5, 6], [4, 5, 99], [1, 1, 3], [0, 1, 3]], dtype=torch.int32, device='cuda')
    gd = torch.float32 if gate == 'fp32' else torch.float16
    gates = torch.ones(6, 3, dtype=gd, device='cuda')
    gates[4:, 2] = 0.5  # 32752 + 32752 + 0.5 = 65504.5 (unit gates: 65505); 32768 + 0.5 + 32752 = 65520.5 (65521)
    # the model on the rows in range: positions out of range point at an appended zero row (no sum here is zero)
    padded = torch.cat([src, torch.zeros(1, 9, dtype=torch.float16, device='cuda')])
    inside = torch.where((pos >= 0) & (pos < 8), pos, torch.full_like(pos, 8))
    for gt in (gates, None):
        y = ops.moe_gather(src, pos, gt)
        assert same_bits(y, ref_gather(padded, inside, gt, torch.float16)), 'bits'
        assert y[:, 0].double().tolist() == [65504.0, INF, -65504.0, -INF, 65504.0, INF], (gt is None, y[:, 0].tolist())
        w64, bound = gather64(src, pos, gt)
        check_value(y, w64, bound, 'fp16 threshold')


@pytest.mark.gpu
def test_gate_gradient_dot_overflow(ops):
    """fp32 gate-gradient dots where every product overflows (+-inf) and where none does (a sum close to the fp32
    maximum), against float64."""
    h, T = 64, 4
    gy = torch.full((T, h), 1.5e19, device='cuda')
    r = torch.empty(T, h, device='cuda')
    r[0], r[1], r[2], r[3] = 3e19, -3e19, 2e17, -2e17  # products 4.5e38 (inf) | 3e36, summed to 1.92e38 (finite)
    pos = torch.arange(T, dtype=torch.int32, device='cuda').view(T, 1)
    dst = torch.zeros(T, h, device='cuda')
    gg = ops.moe_scatter(gy, pos, dst, torch.ones(T, 1, device='cuda'), r)
    exact = (gy.double() * r.double()).sum(-1)
    assert gg[:, 0].tolist()[:2] == [INF, -INF]
    assert all(abs(v) < 3.4e38 and v == v for v in gg[2:, 0].tolist())
    check_value(gg[:, 0], exact, dot_bound(gy, r), 'dot')


# ---- signed zeros --------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('h', [8, 13])
def test_gather_signed_zeros(ops, dtype, h):
    """A single -0 term stays -0 (also -1 * +0 and a -0 term next to positions out of range); a token none of whose
    positions is in [0, src_rows) gets +0, the empty sum torch gives, with and without gates."""
    src = torch.zeros(4, h, dtype=dtype, device='cuda')
    src[1] = -0.0
    src[2] = torch.arange(h, dtype=torch.float64).to(dtype)
    pos = torch.tensor([[1, -1, 4], [0, 4, 7], [-1, -1, -1], [4, 5, 1 << 30], [-1, 1, -1], [2, 2, -5]], dtype=torch.int32,
                       device='cuda')
    gates = torch.tensor([[1.0, 1, 1], [-1.0, 1, 1], [1.0, 1, 1], [2.0, 1, 1], [0.5, 3, 1], [0.0, -0.0, 1]], device='cuda')
    for gt in (gates, gates.to(dtype) if dtype != torch.float32 else None, None):
        y = ops.moe_gather(src, pos, gt)
        neg = torch.signbit(y.float())
        assert bool(neg[0].all()) and bool(neg[4].all()), 'a single -0 term'
        if gt is not None:
            assert bool(neg[1].all()), '-1 * +0'
        for t in (2, 3):
            assert bool((y[t] == 0).all()) and not bool(neg[t].any()), ('the empty sum is +0', t, gt is None)
        want, bound = gather64(src, pos, gt)
        check_value(y, want, bound, 'signed zeros')
        assert torch.equal(torch.signbit(y.float())[2:4], torch.signbit(want)[2:4])
        if gt is not None:
            assert torch.equal(torch.signbit(y[5].float()), torch.signbit((0.0 * src[2].float()) + (-0.0 * src[2].float())))


# ---- route edges ---------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('T,k', [(2047, 1), (2048, 1), (2049, 1), (128, 16), (683, 3), (4097, 1)])
def test_route_tile_edges(ops, T, k):
    """T k at, below and above one route tile (2048 assignments), and one assignment into a second partial tile."""
    g = torch.Generator(device='cuda').manual_seed(T)
    x = torch.randn(T, 6, device='cuda', generator=g).to(torch.bfloat16)
    for E, n in ((8, 4), (1024, 8), (1, 1)):
        idx = torch.randint(0, E, (T, k), device='cuda', generator=g).to(torch.int32 if k % 2 else torch.int64)
        check_permute(ops, x, idx, E, n, (T, k, E))


@pytest.mark.gpu
def test_route_bad_ids_at_tile_edges_and_wide_values(ops):
    """A bad id at assignment 0 and in the last, partial tile; ids that a 32-bit cast would turn into valid or other
    values: int32 INT32_MIN / INT32_MAX, int64 2^31, 2^32 + 1 and 2^40.  Each gives splits of -1, counts of 0 and pos -1
    at that assignment; the next call is correct."""
    T, k, E, n = 4097, 1, 8, 4
    x = torch.randn(T, 6, device='cuda').to(torch.bfloat16)
    cases = [(torch.int64, 0, E), (torch.int64, T - 1, -1), (torch.int32, 0, -2 ** 31), (torch.int32, T - 1, 2 ** 31 - 1),
             (torch.int32, 2048, -2 ** 31), (torch.int64, 5, 2 ** 31), (torch.int64, T - 1, 2 ** 32 + 1),
             (torch.int64, 2048, 2 ** 32), (torch.int64, 77, 2 ** 40), (torch.int64, 0, -2 ** 63)]
    for dt, at, bad in cases:
        idx = torch.randint(0, E, (T, k), device='cuda').to(dt)
        idx.view(-1)[at] = bad
        _, counts, pos, splits = _permute(ops, x, idx, E, n)
        assert splits.tolist() == [-1] * n, (dt, at, bad)
        assert counts.tolist() == [0] * E, (dt, at, bad)
        assert int(pos.view(-1)[at]) == -1, (dt, at, bad)
        check_permute(ops, x, idx.view(-1).clamp(0, E - 1).view(T, k), E, n, ('after', bad))


@pytest.mark.gpu
@pytest.mark.parametrize('dt', [torch.int32, torch.int64])
def test_route_one_expert_top16(ops, dt):
    """E = 1 with k = 16: every slot of every token names the same expert, so pos is the identity."""
    x = torch.randn(301, 5, device='cuda').to(torch.float16)
    idx = torch.zeros(301, 16, dtype=dt, device='cuda')
    _, _, pos, _ = check_permute(ops, x, idx, 1, 1, 'E = 1')
    assert torch.equal(pos.view(-1), torch.arange(301 * 16, dtype=torch.int32, device='cuda'))


# ---- the simulated-rank chain at the limits ---------------------------------------------------------------------------

def _run_sim(m, xs, ids, gates, gys, gate_dtype):
    gates = [g.to(gate_dtype) for g in gates]
    got, ref = m.run(xs, ids, gates, gys), m.reference(xs, ids, gates, gys)
    if gate_dtype != torch.float32:  # the gate gradient is rounded once more, to the gates' dtype
        ref['dot_tol'] = [t + ref['grad_gates'][r].abs() * torch.finfo(gate_dtype).eps for r, t in enumerate(ref['dot_tol'])]
    return got, ref


def _received(ids, E, n):
    """Rows each rank receives."""
    el = E // n
    return [sum(int(((i >= q * el) & (i < (q + 1) * el)).sum()) for i in ids) for q in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize('n,E,k,dtype,gate', [
    (8, 1024, 16, torch.bfloat16, torch.float32),  # 128 local experts
    (8, 8, 16, torch.bfloat16, torch.bfloat16),  # one expert per rank: the in-place regroup, duplicate experts per token
    (2, 8, 16, torch.float16, torch.float16),
    (4, 64, 5, torch.float16, torch.float16),
    (4, 16, 3, torch.bfloat16, torch.bfloat16),
    (2, 2, 1, torch.float32, torch.float32)])
def test_sim_chain_at_the_limits(sim, ops, n, E, k, dtype, gate):
    tokens = [37 + 53 * r for r in range(n)]
    m = SimMoE(sim, ops, n, E, k, 24, tokens, capacity=sum(tokens) * k, dtype=dtype)
    xs, ids, gates, gys = m.inputs(n + k)
    got, ref = _run_sim(m, xs, ids, gates, gys, gate)
    check_sim(m, got, ref, (n, E, k, dtype))


@pytest.mark.gpu
@pytest.mark.parametrize('n', [2, 4, 8])
def test_sim_chain_every_rank_empty(sim, ops, n):
    """Every rank with T = 0: every split, count and output empty, status OK."""
    m = SimMoE(sim, ops, n, 2 * n, 2, 16, [0] * n, capacity=4)
    m.max_rows = 1  # the send and return buffers keep one row
    m.send = [torch.zeros(1, m.h, dtype=m.dtype, device='cuda') for _ in range(n)]
    xs, ids, gates, gys = m.inputs(0)
    got = m.run(xs, ids, gates, gys)
    check_sim(m, got, m.reference(xs, ids, gates, gys), 'empty')
    for r in range(n):
        assert got['y'][r].shape == (0, m.h) and got['grad_gates'][r].shape == (0, 2)
        assert got['offsets'][r].tolist() == [0, 0] and not bool(_bytes(got['expert_in'][r]).any())


@pytest.mark.gpu
@pytest.mark.parametrize('n', [2, 4, 8])
def test_sim_chain_capacity_at_the_received_total(sim, ops, n):
    """Capacity equal to the busiest rank's received total: OK with a zero-length tail there.  One less:
    RECV_OVERFLOW on every rank, every output zero, and the next call correct."""
    tokens, E, k = [150 + 31 * r for r in range(n)], 4 * n, 3
    probe = SimMoE(sim, ops, n, E, k, 20, tokens, capacity=1)
    xs, ids, gates, gys = probe.inputs(7)
    for i in ids:  # rank 0 the busiest by a margin, so that the rows fit under busiest - 1 once spread out
        i[:40, 0] = 0
    busiest = max(_received(ids, E, n))
    assert sum(_received(ids, E, n)) <= n * (busiest - 1)
    m = SimMoE(sim, ops, n, E, k, 20, tokens, capacity=busiest)
    check_sim(m, m.run(xs, ids, gates, gys), m.reference(xs, ids, gates, gys), 'capacity at the total')
    m = SimMoE(sim, ops, n, E, k, 20, tokens, capacity=busiest - 1)
    got = m.run(xs, ids, gates, gys)
    torch.cuda.synchronize()
    assert [int(s) for s in got['status']] == [RECV_OVERFLOW] * n
    assert [int(s) for s in got['status2']] == [RECV_OVERFLOW] * n
    for r in range(n):
        for key in ('expert_in', 'offsets', 'y', 'grad_gates', 'grad_x'):
            assert not bool(_bytes(got[key][r]).any()), (r, key)
    ids = [i.clone() for i in ids]  # the same tokens, with ids moved from the busiest ranks to the least busy one
    el = E // n
    for _ in range(sum(tokens) * k):
        rec = _received(ids, E, n)
        if max(rec) <= busiest - 1:
            break
        q, r = rec.index(max(rec)), rec.index(min(rec))
        i = next(i for i in ids if bool(((i >= q * el) & (i < (q + 1) * el)).any()))
        at = ((i >= q * el) & (i < (q + 1) * el)).view(-1).nonzero()[0, 0]
        i.view(-1)[at] = r * el
    assert max(_received(ids, E, n)) <= busiest - 1
    check_sim(m, m.run(xs, ids, gates, gys), m.reference(xs, ids, gates, gys), 'next call')


@pytest.mark.gpu
@pytest.mark.parametrize('n', [2, 4, 8])
@pytest.mark.parametrize('bad', [NAN, INF], ids=['nan', 'inf'])
def test_sim_chain_containment(sim, ops, n, bad):
    """One NaN (or inf) in one token's row on rank 1: y, grad_x and grad_gates of every other token on every rank are
    bit-identical to the clean run, and the affected token's NaN / inf masks are those of float64."""
    tokens, E, k, h = [120] * n, 4 * n, 4, 32
    m = SimMoE(sim, ops, n, E, k, h, tokens, capacity=sum(tokens) * k)
    xs, ids, gates, gys = m.inputs(11)
    clean = m.run(xs, ids, gates, gys)
    clean = {key: [t.clone() for t in clean[key]] for key in ('y', 'grad_x', 'grad_gates')}
    t0, i0 = 57, 9
    xs = [x.clone() for x in xs]
    xs[1][t0, i0] = bad
    got = m.run(xs, ids, gates, gys)
    torch.cuda.synchronize()
    assert [int(s) for s in got['status']] == [OK] * n
    for r in range(n):
        keep = torch.ones(tokens[r], dtype=torch.bool, device='cuda')
        if r == 1:
            keep[t0] = False
        for key in ('y', 'grad_x', 'grad_gates'):
            assert same_bits(got[key][r][keep], clean[key][r][keep]), (r, key)
        assert same_bits(got['grad_x'][r], clean['grad_x'][r]), (r, 'grad_x does not read x')
    # the affected token against float64 over the stored expert outputs
    e = ids[1][t0]
    outs = torch.stack([(xs[1][t0] * m.w[e[j]]).double() for j in range(k)])  # [k, h]
    y64 = (gates[1][t0].double().view(k, 1) * outs).sum(0)
    gg64 = (gys[1][t0].double().view(1, h) * outs).sum(1)
    for got_t, want in ((got['y'][1][t0], y64), (got['grad_gates'][1][t0], gg64)):
        w = want.to(got_t.dtype)
        assert torch.equal(torch.isnan(got_t), torch.isnan(w)) and torch.equal(torch.isinf(got_t), torch.isinf(w))
        assert torch.equal(got_t[torch.isinf(w)], w[torch.isinf(w)])
        assert bool((~torch.isfinite(w)).any())


# ---- the public object, one rank holding every expert -----------------------------------------------------------------

def _dense64(x, gates, w, idx):
    xr, gr, wr = (t.detach().double().requires_grad_() for t in (x, gates, w))
    return xr, gr, wr, sum(gr[:, j:j + 1] * (xr * wr[idx[:, j]]) for j in range(idx.shape[1]))


def _close(got, want, dtype, what):
    rtol = 1e-5 if dtype == torch.float32 else 2e-2
    torch.testing.assert_close(got.double(), want.detach(), rtol=rtol, atol=rtol * max(1.0, float(want.detach().abs().max())) if
                               want.numel() else 0, msg=what)


@pytest.mark.gpu
@pytest.mark.parametrize('E', [8, 1])
def test_public_top16_fp16_gates(one_rank, E):
    """k = 16 with fp16 rows and fp16 gates, against the float64 autograd reference.  E = 1: one expert per rank, so
    the regroups run in place and every slot of a token names the same expert."""
    hvd = one_rank
    T, h, k, dt = 200, 24, 16, torch.float16
    disp = hvd.ExpertDispatcher(E, h, dt, max_tokens=T, top_k=k, capacity=T * k)
    g = torch.Generator(device='cuda').manual_seed(1)
    w = (torch.rand(E, h, device='cuda', generator=g) + 0.5).to(dt).requires_grad_()
    x = torch.randn(T, h, device='cuda', generator=g).to(dt).requires_grad_()
    idx = torch.randint(0, E, (T, k), device='cuda', generator=g)
    gates = (torch.rand(T, k, device='cuda', generator=g) / k).to(dt).requires_grad_()
    gy = torch.randn(T, h, device='cuda', generator=g).to(dt)
    expert_in, offsets, handle = disp.dispatch(x, idx)
    y = disp.combine(_expert_fn(w, expert_in, offsets), gates, handle)
    assert y.dtype == dt and int(handle.status) == OK
    gx, gg = torch.autograd.grad(y, (x, gates), gy)  # (w's gradient is torch's fp16 index backward, not ours)
    assert gg.dtype == dt
    xr, gr, wr, yr = _dense64(x, gates, w, idx)
    rx, rg = torch.autograd.grad(yr, (xr, gr), gy.double())
    _close(y, yr, dt, 'y')
    _close(gx, rx, dt, 'grad_x')
    _close(gg, rg, dt, 'grad_gates')


@pytest.mark.gpu
def test_public_gates_without_grad_and_outputs_without_grad(one_rank):
    """Gates that do not require grad (no gate-gradient dot rows are passed), and expert_out built under no_grad (no
    backward exchange runs), each against the float64 autograd reference."""
    hvd = one_rank
    T, h, E, k = 150, 16, 4, 2
    disp = hvd.ExpertDispatcher(E, h, torch.float32, max_tokens=T, top_k=k, capacity=T * k)
    g = torch.Generator(device='cuda').manual_seed(2)
    w = (torch.rand(E, h, device='cuda', generator=g) + 0.5).requires_grad_()
    x = torch.randn(T, h, device='cuda', generator=g).requires_grad_()
    idx = torch.randint(0, E, (T, k), device='cuda', generator=g)
    gates = torch.rand(T, k, device='cuda', generator=g)
    gy = torch.randn(T, h, device='cuda', generator=g)
    expert_in, offsets, handle = disp.dispatch(x, idx)
    y = disp.combine(_expert_fn(w, expert_in, offsets), gates, handle)
    gx, gw = torch.autograd.grad(y, (x, w), gy)
    xr, gr, wr, yr = _dense64(x, gates, w, idx)
    rx, rw = torch.autograd.grad(yr, (xr, wr), gy.double())
    _close(y, yr, torch.float32, 'y')
    _close(gx, rx, torch.float32, 'grad_x')
    _close(gw, rw, torch.float32, 'grad_w')
    gates.requires_grad_()
    expert_in, offsets, handle = disp.dispatch(x, idx)
    with torch.no_grad():
        expert_out = _expert_fn(w, expert_in, offsets)
    y = disp.combine(expert_out, gates, handle)
    (gg,) = torch.autograd.grad(y, (gates,), gy)
    _, gr, _, yr = _dense64(x, gates, w, idx)
    (rg,) = torch.autograd.grad(yr, (gr,), gy.double())
    _close(gg, rg, torch.float32, 'grad_gates')


@pytest.mark.gpu
def test_public_changing_tokens_and_two_layers(one_rank):
    """T that changes between calls, including 0, and one dispatcher serving two layers in one backward pass."""
    hvd = one_rank
    h, E, k, maxT = 20, 4, 3, 300
    disp = hvd.ExpertDispatcher(E, h, torch.float32, max_tokens=maxT, top_k=k, capacity=maxT * k)
    g = torch.Generator(device='cuda').manual_seed(3)
    w1 = (torch.rand(E, h, device='cuda', generator=g) + 0.5).requires_grad_()
    w2 = (torch.rand(E, h, device='cuda', generator=g) + 0.5).requires_grad_()
    for T in (300, 0, 17, 0, 256):
        x = torch.randn(T, h, device='cuda', generator=g).requires_grad_()
        i1, i2 = (torch.randint(0, E, (T, k), device='cuda', generator=g) for _ in range(2))
        g1, g2 = (torch.rand(T, k, device='cuda', generator=g).requires_grad_() for _ in range(2))
        gy = torch.randn(T, h, device='cuda', generator=g)
        a, off, hd = disp.dispatch(x, i1)
        y1 = disp.combine(_expert_fn(w1, a, off), g1, hd)
        b, off2, hd2 = disp.dispatch(y1, i2)
        y2 = disp.combine(_expert_fn(w2, b, off2), g2, hd2)
        assert y2.shape == (T, h) and int(hd.status) == OK and int(hd2.status) == OK
        grads = torch.autograd.grad(y2, (x, g1, g2, w1, w2), gy)
        xr, g1r, w1r, y1r = _dense64(x, g1, w1, i1)
        g2r, w2r = g2.detach().double().requires_grad_(), w2.detach().double().requires_grad_()
        y2r = sum(g2r[:, j:j + 1] * (y1r * w2r[i2[:, j]]) for j in range(k))
        refs = torch.autograd.grad(y2r, (xr, g1r, g2r, w1r, w2r), gy.double())
        _close(y2, y2r, torch.float32, ('y', T))
        for name, got, want in zip(('x', 'g1', 'g2', 'w1', 'w2'), grads, refs):
            _close(got, want, torch.float32, (name, T))
