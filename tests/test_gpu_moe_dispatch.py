"""hvd.ExpertDispatcher: expert-parallel dispatch and combine around the captured alltoall.

- The kernels alone (`ops.moe_permute`, `moe_scatter`, `moe_gather`, `moe_regroup`, `moe_regroup_reverse`) against
  torch references: the permute byte-exact against a stable argsort, the regroup byte-exact in both directions, the
  gather and the scaled scatter bit-exact against an fp32 torch model in j order, the gate gradient within a bound
  derived from sum |grad_y * v|, and every output bit-identical across runs and CTA counts.
- The whole exchange on N = 2, 4, 8 simulated ranks (`ops.sim.captured_alltoall` for the three exchanges), forward and
  backward with per-rank diagonal linear experts, against a single-process dense reference over every rank's tokens;
  the overflow and bad-id statuses; all ranks captured into one CUDA graph and replayed with new router outputs.
- The public object with a stand-in exchange (one rank holds every expert, so the exchange is the identity): end to end
  against a dense torch MoE, inside hvd.GraphedStep, and every host-side argument error.
- On several GPUs, tests/parallel/moe_worker.py runs the dispatcher on real ranks.
"""
import pytest
import torch

from conftest import run_parallel

pytestmark = pytest.mark.gpu

OK, NEGATIVE, RECV_OVERFLOW = 0, 1, 3
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


@pytest.fixture(scope='module')
def ops():
    from horovod_b200 import ops
    return ops


def _bytes(t):
    return t.contiguous().view(-1).view(torch.uint8) if t.numel() else torch.empty(0, dtype=torch.uint8, device=t.device)


def _rows(T, h, dtype, seed, offset=0):
    """[T, h] random rows; offset > 0 makes a contiguous view that starts `offset` elements into its storage."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    base = torch.randn(T * h + offset, device='cuda', generator=g).to(dtype)
    return base[offset:].view(T, h)


def _ids(T, k, E, seed, dtype=torch.int64, skew=False):
    g = torch.Generator(device='cuda').manual_seed(seed)
    if skew:
        return torch.full((T, k), E - 1, dtype=dtype, device='cuda')
    return torch.randint(0, E, (T, k), device='cuda', generator=g).to(dtype)


# ---- torch references -----------------------------------------------------------------------------------------------

def ref_permute(x, idx, E, n):
    """(send rows, pos [T, k], counts [E], splits [n]) of the stable argsort of the expert ids."""
    T, k = idx.shape
    flat = idx.flatten().long()
    order = torch.argsort(flat, stable=True)
    pos = torch.empty(T * k, dtype=torch.int32, device='cuda')
    pos[order] = torch.arange(T * k, dtype=torch.int32, device='cuda')
    counts = torch.bincount(flat, minlength=E)
    send = x.repeat_interleave(k, 0)[order] if T else x[:0]
    return send, pos.view(T, k), counts, counts.view(n, -1).sum(1).to(torch.int32)


def ref_gather(src, pos, gates, dtype):
    """The fp32 model: each product rounded, added in j order starting from term 0, rounded once."""
    acc = None
    for j in range(pos.shape[1]):
        v = src[pos[:, j].long()].float()
        term = v if gates is None else gates[:, j:j + 1].float() * v
        acc = term if acc is None else acc + term
    return acc.to(dtype)


def ref_regroup(src, counts):
    """Source-major rows (p, then e) -> expert-major rows (e, then p), with the group ends."""
    n, el = counts.shape
    c = counts.tolist()
    seg, at = {}, 0
    for p in range(n):
        for e in range(el):
            seg[(p, e)] = src[at:at + c[p][e]]
            at += c[p][e]
    out = torch.cat([seg[(p, e)] for e in range(el) for p in range(n)])
    ends = torch.tensor([sum(c[p][e2] for e2 in range(e + 1) for p in range(n)) for e in range(el)], dtype=torch.int32)
    return out, ends


def dot_bound(gy, v):
    """|fp32 dot - exact| <= (h / 32 + 6) u sum |gy * v|: a per-lane sum of h / 32 terms, then five butterfly levels."""
    h = gy.shape[-1]
    return (h / 32 + 6) * 2.0 ** -24 * (gy.double() * v.double()).abs().sum(-1) + 1e-30


# ---- the kernels alone ----------------------------------------------------------------------------------------------

def _permute(ops, x, idx, E, n, ctas=0, spare=3):
    T, k = idx.shape
    send = torch.full((T * k + spare, x.shape[1]), 7, dtype=x.dtype, device='cuda')
    counts = torch.full((E,), -5, dtype=torch.int64, device='cuda')
    pos, splits = ops.moe_permute(x, idx, E, n, send, counts, ctas=ctas)
    return send, counts, pos, splits


def check_permute(ops, x, idx, E, n, what):
    T, k = idx.shape
    send, counts, pos, splits = _permute(ops, x, idx, E, n)
    rsend, rpos, rcounts, rsplits = ref_permute(x, idx, E, n)
    assert torch.equal(pos, rpos), what
    assert torch.equal(counts, rcounts), what
    assert torch.equal(splits, rsplits), what
    assert torch.equal(_bytes(send[:T * k]), _bytes(rsend)), (what, 'send rows differ')
    assert bool((send[T * k:] == 7).all()), (what, 'wrote past the assignments')
    return send, counts, pos, splits


@pytest.mark.parametrize('E,n', [(1, 1), (8, 1), (8, 2), (8, 8), (64, 4), (256, 8), (1024, 2), (1024, 8)])
def test_permute_experts_and_ranks(ops, E, n):
    for k in (1, 2, 4, 8):
        for T in (0, 1, 4097, 16384):
            x = _rows(T, 8, torch.bfloat16, seed=T + k)
            idx = _ids(T, k, E, seed=E + n + k + T, dtype=torch.int32 if k % 2 else torch.int64)
            check_permute(ops, x, idx, E, n, (E, n, k, T))


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('h_bytes', [2, 6, 16 * 1024 + 2])
def test_permute_dtypes_row_sizes_and_unaligned_views(ops, dtype, h_bytes):
    size = torch.empty(0, dtype=dtype).element_size()
    if h_bytes % size:
        pytest.skip('row size not a multiple of the element size')
    h = h_bytes // size
    for offset in (0, 1, 3):
        x = _rows(300, h, dtype, seed=h + offset, offset=offset)
        check_permute(ops, x, _ids(300, 4, 64, seed=h), 64, 4, (dtype, h, offset))


def test_permute_skewed_router_and_bad_ids(ops):
    x = _rows(4097, 24, torch.float16, seed=1)
    check_permute(ops, x, _ids(4097, 2, 8, seed=0, skew=True), 8, 4, 'skewed')
    for bad in (-1, 8, 1 << 40):
        idx = _ids(4097, 2, 8, seed=2)
        idx[4000, 1] = bad
        _, counts, pos, splits = _permute(ops, x, idx, 8, 4)
        assert splits.tolist() == [-1] * 4, bad
        assert counts.tolist() == [0] * 8
        assert int(pos[4000, 1]) == -1
    check_permute(ops, x, _ids(4097, 2, 8, seed=3), 8, 4, 'after bad ids')


def _random_counts(n, el, max_rows, seed, zero_frac=0.3):
    g = torch.Generator(device='cuda').manual_seed(seed)
    c = torch.randint(0, max_rows + 1, (n, el), device='cuda', generator=g)
    return c * (torch.rand((n, el), device='cuda', generator=g) >= zero_frac)


@pytest.mark.parametrize('n,el', [(1, 1), (2, 1), (2, 4), (4, 16), (8, 128), (1, 1024)])
@pytest.mark.parametrize('dtype,h', [(torch.bfloat16, 1), (torch.float16, 3), (torch.float32, 64), (torch.bfloat16, 8193)])
def test_regroup_both_directions(ops, n, el, dtype, h):
    max_rows = max(1, 2000 // (n * el)) if h < 8000 else 2
    counts = _random_counts(n, el, max_rows, seed=n * el + h).to(torch.int64)
    total = int(counts.sum())
    cap = total + 5
    src = _rows(cap, h, dtype, seed=h)
    out, offsets = ops.moe_regroup(src, counts)
    ref, ends = ref_regroup(src[:total], counts)
    assert torch.equal(_bytes(out[:total]), _bytes(ref))
    assert bool((_bytes(out[total:]) == 0).all()), 'tail not zeroed'
    assert offsets.cpu().tolist() == ends.tolist()
    back = torch.full_like(src, 3)
    ret = ops.moe_regroup_reverse(out, counts, back)
    assert torch.equal(_bytes(back[:total]), _bytes(src[:total])), 'reverse is not the inverse'
    assert bool((back[total:] == 3).all()), 'reverse wrote past the total'
    assert ret.tolist() == counts.sum(1).tolist()
    if el == 1:  # in place: the same rows, only the tail written
        inplace = src.clone()
        _, off1 = ops.moe_regroup(inplace, counts, out=inplace)
        assert torch.equal(_bytes(inplace), _bytes(out)) and torch.equal(off1, offsets)
    status = torch.full((1,), RECV_OVERFLOW, dtype=torch.int32, device='cuda')
    dead, dead_off = ops.moe_regroup(src, counts, status)
    assert not bool(_bytes(dead).any()) and not bool(dead_off.any())
    assert not bool(ops.moe_regroup_reverse(out, counts, back, status).any())


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('gate_fp32', [True, False])
@pytest.mark.parametrize('h', [1, 3, 4096, 8193])
def test_gather_and_scatter_bit_exact(ops, dtype, gate_fp32, h):
    T, k, rows = 1000 if h < 8000 else 64, 4, 3000 if h < 8000 else 300
    g = torch.Generator(device='cuda').manual_seed(h)
    src = _rows(rows, h, dtype, seed=h + 1)
    pos = torch.stack([torch.randperm(rows, device='cuda', generator=g)[:T] for _ in range(k)], 1).to(torch.int32)
    gates = torch.rand(T, k, device='cuda', generator=g).to(torch.float32 if gate_fp32 else dtype)
    assert torch.equal(_bytes(ops.moe_gather(src, pos, gates)), _bytes(ref_gather(src, pos, gates, dtype)))
    assert torch.equal(_bytes(ops.moe_gather(src, pos)), _bytes(ref_gather(src, pos, None, dtype)))
    # scaled scatter: a permutation of the rows of the first slot, so every row is written once
    gy = _rows(T, h, dtype, seed=h + 2)
    perm = pos[:, :1].contiguous()
    dst = torch.zeros(rows, h, dtype=dtype, device='cuda')
    grad_gates = ops.moe_scatter(gy, perm, dst, gates[:, :1].contiguous(), src)
    ref = (gates[:, :1].float() * gy.float()).to(dtype)
    assert torch.equal(_bytes(dst[perm[:, 0].long()]), _bytes(ref))
    exact = (gy.double() * src[perm[:, 0].long()].double()).sum(-1)
    err = (grad_gates[:, 0].double() - exact).abs()
    tol = dot_bound(gy, src[perm[:, 0].long()])
    if not gate_fp32:  # rounded to the gates' dtype
        tol = tol + exact.abs() * torch.finfo(dtype).eps
    assert bool((err <= tol).all()), float((err / tol).max())


def test_deterministic_across_runs_and_cta_counts(ops):
    T, k, E, n, h = 16384, 8, 256, 8, 200
    x = _rows(T, h, torch.bfloat16, seed=5)
    idx = _ids(T, k, E, seed=6)
    gates = torch.rand(T, k, device='cuda')
    results = []
    for ctas in (1, 3, 17, 0, 0):
        send, counts, pos, splits = _permute(ops, x, idx, E, n, ctas=ctas)
        y = ops.moe_gather(send, pos, gates, ctas=ctas)
        dst = torch.zeros_like(send)
        gg = ops.moe_scatter(x, pos, dst, gates, send, ctas=ctas)
        c = _random_counts(n, E // n, 40, seed=1).to(torch.int64)
        rg, off = ops.moe_regroup(send, c, ctas=ctas)
        back = torch.zeros_like(send)
        ret = ops.moe_regroup_reverse(rg, c, back, ctas=ctas)
        results.append([send, counts, pos, splits, y, dst, gg, rg, off, back, ret])
    for other in results[1:]:
        for a, b in zip(results[0], other):
            assert torch.equal(_bytes(a), _bytes(b))


def test_status_zeroes_gather_and_gate_gradients(ops):
    src = _rows(50, 16, torch.float32, seed=1)
    pos = torch.arange(40, dtype=torch.int32, device='cuda').view(20, 2)
    gates = torch.rand(20, 2, device='cuda')
    status = torch.full((1,), NEGATIVE, dtype=torch.int32, device='cuda')
    y = ops.moe_gather(src, pos, gates, status)
    assert not bool(_bytes(y).any())
    dst = torch.full_like(src, 2.0)
    gg = ops.moe_scatter(src[:20], pos, dst, gates, src, status)
    assert not bool(_bytes(gg).any()) and bool((dst == 2.0).all())


# ---- the whole exchange on simulated ranks --------------------------------------------------------------------------

class SimMoE:
    """N simulated ranks, each with T_r tokens, top-k ids over E experts, gates and one diagonal linear expert per local
    expert (y = x * w[e], row by row, so that its bits do not depend on how rows are batched).  Kernels run step-major:
    every rank's step, then the next; the exchanges are ops.sim.captured_alltoall."""

    def __init__(self, sim, ops, n, E, k, h, tokens, capacity, dtype=torch.bfloat16, seed=0):
        self.sim, self.ops, self.n, self.E, self.k, self.h = sim, ops, n, E, k, h
        self.el, self.cap, self.dtype, self.tokens = E // n, capacity, dtype, tokens
        self.max_rows = max(tokens) * k
        g = torch.Generator(device='cuda').manual_seed(seed)
        self.w = (torch.rand(E, h, device='cuda', generator=g) + 0.5).to(dtype)  # expert e's diagonal
        self.send = [torch.zeros(self.max_rows, h, dtype=dtype, device='cuda') for _ in range(n)]
        self.ret = [torch.zeros(capacity, h, dtype=dtype, device='cuda') for _ in range(n)]
        self.counts = [torch.zeros(E, dtype=torch.int64, device='cuda') for _ in range(n)]
        self.count_splits = [torch.full((n,), self.el, dtype=torch.int32, device='cuda') for _ in range(n)]

    def exchange(self, ins, splits, cap, streams=None):
        like = ins[0]
        outs = [torch.empty(cap, *like.shape[1:], dtype=like.dtype, device='cuda') for _ in range(self.n)]
        recv = [torch.empty(self.n, dtype=torch.int64, device='cuda') for _ in range(self.n)]
        status = [torch.empty(1, dtype=torch.int32, device='cuda') for _ in range(self.n)]
        self.sim.captured_alltoall(ins, splits, outs, recv, status, ctas=4, streams=streams)
        return outs, status

    def expert_rows(self, rows, offsets, r):
        """Local expert e of rank r on its group of rows (found on the device), zero past the total."""
        eid = torch.searchsorted(offsets.long(), torch.arange(rows.shape[0], device='cuda'), right=True)
        w = torch.cat([self.w[r * self.el:(r + 1) * self.el], torch.zeros(1, self.h, dtype=self.dtype, device='cuda')])
        return rows * w[eid]

    def run(self, xs, ids, gates, gys, streams=None):
        n, ops = self.n, self.ops
        ctx = (lambda r: torch.cuda.stream(streams[r])) if streams else (lambda r: torch.cuda.stream(torch.cuda.current_stream()))
        out = {}
        # ---- dispatch ----
        pos, splits = [None] * n, [None] * n
        for r in range(n):
            with ctx(r):
                pos[r], splits[r] = ops.moe_permute(xs[r], ids[r], self.E, n, self.send[r], self.counts[r])
        rc, _ = self.exchange(self.counts, self.count_splits, self.E, streams)
        rc = [c.view(n, self.el) for c in rc]
        recv, status = self.exchange(self.send, splits, self.cap, streams)
        expert_in, offsets, expert_out = [None] * n, [None] * n, [None] * n
        for r in range(n):
            with ctx(r):
                expert_in[r], offsets[r] = ops.moe_regroup(recv[r], rc[r], status[r])
                expert_out[r] = self.expert_rows(expert_in[r], offsets[r], r)
        # ---- combine ----
        ret_splits = [None] * n
        for r in range(n):
            with ctx(r):
                ret_splits[r] = ops.moe_regroup_reverse(expert_out[r], rc[r], self.ret[r], status[r])
        back, _ = self.exchange(self.ret, ret_splits, self.max_rows, streams)
        ys, grad_gates = [None] * n, [None] * n
        for r in range(n):
            with ctx(r):
                ys[r] = ops.moe_gather(back[r], pos[r], gates[r], status[r])
        # ---- combine backward ----
        for r in range(n):
            with ctx(r):
                grad_gates[r] = ops.moe_scatter(gys[r], pos[r], self.send[r], gates[r], back[r], status[r])
        recv2, status2 = self.exchange(self.send, splits, self.cap, streams)
        grad_in = [None] * n
        for r in range(n):
            with ctx(r):
                grad_out, _ = ops.moe_regroup(recv2[r], rc[r], status[r])
                grad_in[r] = self.expert_rows(grad_out, offsets[r], r)
                out.setdefault('grad_w', []).append((grad_out, expert_in[r], offsets[r]))
        # ---- dispatch backward ----
        ret2 = [None] * n
        for r in range(n):
            with ctx(r):
                ret2[r] = ops.moe_regroup_reverse(grad_in[r], rc[r], self.ret[r], status[r])
        back2, _ = self.exchange(self.ret, ret2, self.max_rows, streams)
        grad_x = [None] * n
        for r in range(n):
            with ctx(r):
                grad_x[r] = ops.moe_gather(back2[r], pos[r], None, status[r])
        out.update(expert_in=expert_in, offsets=offsets, y=ys, grad_gates=grad_gates, grad_x=grad_x, status=status,
                   status2=status2)
        return out

    def inputs(self, seed, bad_rank=None):
        g = torch.Generator(device='cuda').manual_seed(seed)
        xs = [torch.randn(t, self.h, device='cuda', generator=g).to(self.dtype) for t in self.tokens]
        ids = [torch.randint(0, self.E, (t, self.k), device='cuda', generator=g) for t in self.tokens]
        if bad_rank is not None:
            ids[bad_rank][0, 0] = self.E
        gates = [torch.rand(t, self.k, device='cuda', generator=g) for t in self.tokens]
        gys = [torch.randn(t, self.h, device='cuda', generator=g).to(self.dtype) for t in self.tokens]
        return xs, ids, gates, gys

    def reference(self, xs, ids, gates, gys):
        """Dense, over every rank's tokens: expert_in per rank (torch indexing), y, grad_x, grad_gates (fp64) and each
        expert's weight gradient (fp64)."""
        n, el, dt = self.n, self.el, self.dtype
        ref = {'expert_in': [], 'y': [], 'grad_x': [], 'grad_gates': [], 'grad_w': torch.zeros(self.E, self.h, dtype=torch.float64,
                                                                                              device='cuda')}
        for q in range(n):
            parts = []
            for e in range(q * el, (q + 1) * el):
                for p in range(n):
                    flat = ids[p].flatten()
                    a = (flat == e).nonzero().flatten()  # ascending assignment order
                    parts.append(xs[p][a // self.k])
            ref['expert_in'].append(torch.cat(parts))
        for p in range(n):
            e = ids[p]
            out_j = [(xs[p] * self.w[e[:, j]]) for j in range(self.k)]
            y = None
            for j in range(self.k):
                term = gates[p][:, j:j + 1].float() * out_j[j].float()
                y = term if y is None else y + term
            ref['y'].append(y.to(dt))
            gx = None
            for j in range(self.k):
                go = (gates[p][:, j:j + 1].float() * gys[p].float()).to(dt)
                term = (go * self.w[e[:, j]]).float()
                gx = term if gx is None else gx + term
                ref['grad_w'].index_add_(0, e[:, j], go.double() * xs[p].double())
            ref['grad_x'].append(gx.to(dt))
            ref['grad_gates'].append(torch.stack([(gys[p].double() * o.double()).sum(-1) for o in out_j], 1))
            ref.setdefault('dot_tol', []).append(torch.stack([dot_bound(gys[p], o) for o in out_j], 1))
        return ref


def check_sim(m, got, ref, what):
    torch.cuda.synchronize()
    for r in range(m.n):
        assert int(got['status'][r]) == OK, (what, r)
        total = ref['expert_in'][r].shape[0]
        assert torch.equal(_bytes(got['expert_in'][r][:total]), _bytes(ref['expert_in'][r])), (what, r, 'expert_in')
        assert not bool(_bytes(got['expert_in'][r][total:]).any()), (what, r, 'tail')
        assert int(got['offsets'][r][-1]) == total
        assert torch.equal(_bytes(got['y'][r]), _bytes(ref['y'][r])), (what, r, 'y')
        assert torch.equal(_bytes(got['grad_x'][r]), _bytes(ref['grad_x'][r])), (what, r, 'grad_x')
        err = (got['grad_gates'][r].double() - ref['grad_gates'][r]).abs()
        assert bool((err <= ref['dot_tol'][r]).all()), (what, r, 'grad_gates')
    # expert weight gradients: sum over each group of grad_out * expert_in, in fp64, against the dense reference
    for r, (go, xin, off) in enumerate(got['grad_w']):
        ends = off.long().tolist()
        for e in range(m.el):
            lo = ends[e - 1] if e else 0
            gw = (go[lo:ends[e]].double() * xin[lo:ends[e]].double()).sum(0)
            torch.testing.assert_close(gw, ref['grad_w'][r * m.el + e], rtol=1e-9, atol=1e-9)


@pytest.fixture(scope='module')
def sim():
    from horovod_b200.ops import sim
    return sim


@pytest.mark.parametrize('n,E,k', [(2, 8, 2), (4, 64, 8), (8, 8, 1), (8, 256, 4)])
def test_sim_ranks_forward_backward(sim, ops, n, E, k):
    tokens = [300 + 97 * r for r in range(n)]
    tokens[n - 1] = 0  # a rank without tokens
    m = SimMoE(sim, ops, n, E, k, 40, tokens, capacity=sum(tokens) * k)
    for seed in range(2):
        xs, ids, gates, gys = m.inputs(seed)
        check_sim(m, m.run(xs, ids, gates, gys), m.reference(xs, ids, gates, gys), (n, E, k, seed))


@pytest.mark.parametrize('n', [2, 4])
@pytest.mark.parametrize('failure', ['overflow', 'bad id'])
def test_sim_ranks_failure_status(sim, ops, n, failure):
    tokens = [100] * n  # about 200 rows per rank for a uniform router
    m = SimMoE(sim, ops, n, 4 * n, 2, 24, tokens, capacity=300)
    xs, ids, gates, gys = m.inputs(1, bad_rank=1 if failure == 'bad id' else None)
    if failure == 'overflow':
        for r in range(n):
            ids[r].zero_()  # rank 0 receives 200 n rows, over its capacity of 300
    got = m.run(xs, ids, gates, gys)
    torch.cuda.synchronize()
    code = RECV_OVERFLOW if failure == 'overflow' else NEGATIVE
    assert [int(s) for s in got['status']] == [code] * n
    assert [int(s) for s in got['status2']] == [code] * n  # the backward exchange moved nothing either
    for r in range(n):
        for key in ('expert_in', 'offsets', 'y', 'grad_gates', 'grad_x'):
            assert not bool(_bytes(got[key][r]).any()), (failure, r, key)
    xs, ids, gates, gys = m.inputs(2)
    check_sim(m, m.run(xs, ids, gates, gys), m.reference(xs, ids, gates, gys), (failure, 'next call'))


@pytest.mark.parametrize('n', [2, 4, 8])
def test_sim_ranks_in_one_cuda_graph(sim, ops, n):
    tokens = [256] * n
    m = SimMoE(sim, ops, n, 2 * n, 2, 32, tokens, capacity=256 * n * 2)
    xs, ids, gates, gys = m.inputs(0)
    m.run(xs, ids, gates, gys)  # warm-up: the simulated team, the ticket arrays
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(n)]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cur = torch.cuda.current_stream()
        for s in streams:
            s.wait_stream(cur)
        got = m.run(xs, ids, gates, gys, streams=streams)
        for s in streams:
            cur.wait_stream(s)
    gen = torch.Generator(device='cuda').manual_seed(9)
    for it in range(4):
        for r in range(n):  # new router outputs and activations, written on the device
            ids[r].copy_(torch.randint(0, m.E, ids[r].shape, device='cuda', generator=gen))
            gates[r].copy_(torch.rand(gates[r].shape, device='cuda', generator=gen))
            xs[r].copy_(torch.randn(xs[r].shape, device='cuda', generator=gen).to(m.dtype))
        torch.cuda.set_sync_debug_mode('error')
        try:
            graph.replay()
        finally:
            torch.cuda.set_sync_debug_mode('default')
        check_sim(m, got, m.reference(xs, ids, gates, gys), ('replay', it))


# ---- the public object, one rank holding every expert ---------------------------------------------------------------

@pytest.fixture
def one_rank(monkeypatch):
    """hvd.ExpertDispatcher on one rank: registered buffers are plain tensors and the exchange is the identity (rank 0
    sends its rows to itself), with the kernel's statuses; all stand-ins are capturable torch ops."""
    import horovod_b200.torch as hvd
    import horovod_b200.torch.moe as moe
    hvd.init()
    torch.cuda.set_device(0)

    def alltoall(tensor, splits, capacity, process_set, max_ctas):
        out = torch.zeros(capacity, *tensor.shape[1:], dtype=tensor.dtype, device=tensor.device)
        m = min(capacity, tensor.shape[0])
        total = splits.long().sum()
        keep = (torch.arange(m, device=tensor.device) < total).view(-1, *[1] * (tensor.dim() - 1))
        out[:m].copy_(torch.where(keep, tensor[:m], torch.zeros((), dtype=tensor.dtype, device=tensor.device)))
        status = torch.where((splits < 0).any(), NEGATIVE, torch.where(total > capacity, RECV_OVERFLOW, OK))
        return out, splits.long(), status.to(torch.int32).view(1)

    monkeypatch.setattr(moe, '_symm_empty', lambda shape, dtype, device, ps: torch.zeros(shape, dtype=dtype, device=device))
    monkeypatch.setattr(moe, '_alltoall', alltoall)
    yield hvd
    hvd.shutdown()


def _expert_fn(w, expert_in, offsets):
    """Diagonal linear experts, each row's expert found on the device (no host sync)."""
    eid = torch.searchsorted(offsets.long(), torch.arange(expert_in.shape[0], device='cuda'), right=True)
    wz = torch.cat([w, torch.zeros(1, w.shape[1], dtype=w.dtype, device='cuda')])
    return expert_in * wz[eid]


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_public_object_matches_dense_moe(one_rank, dtype):
    hvd = one_rank
    T, h, E, k = 333, 48, 8, 2
    disp = hvd.ExpertDispatcher(E, h, dtype, max_tokens=400, top_k=k, capacity=800)
    g = torch.Generator(device='cuda').manual_seed(0)
    w = (torch.rand(E, h, device='cuda', generator=g) + 0.5).to(dtype).requires_grad_()
    for step in range(2):
        x = torch.randn(T, h, device='cuda', generator=g).to(dtype).requires_grad_()
        idx = torch.randint(0, E, (T, k), device='cuda', generator=g)
        gates = torch.rand(T, k, device='cuda', generator=g).requires_grad_()
        gy = torch.randn(T, h, device='cuda', generator=g).to(dtype)
        expert_in, offsets, handle = disp.dispatch(x, idx)
        assert int(handle.status) == OK and int(offsets[-1]) == T * k
        y = disp.combine(_expert_fn(w, expert_in, offsets), gates, handle)
        gx, gg, gw = torch.autograd.grad(y, (x, gates, w), gy)
        # dense reference: every token through its k experts
        xr, gr, wr = x.detach().double().requires_grad_(), gates.detach().double().requires_grad_(), w.detach().double().requires_grad_()
        yr = sum(gr[:, j:j + 1] * (xr * wr[idx[:, j]]) for j in range(k))
        rx, rg, rw = torch.autograd.grad(yr, (xr, gr, wr), gy.double())
        tol = dict(rtol=1e-5, atol=1e-5) if dtype == torch.float32 else dict(rtol=2e-2, atol=2e-2)
        torch.testing.assert_close(y.double(), yr.detach(), **tol)
        torch.testing.assert_close(gx.double(), rx, **tol)
        # the gate gradient is a dot with the expert outputs as stored (rounded to dtype), so compare against that
        rg_stored = torch.stack([(gy.double() * (x * w[idx[:, j]]).detach().double()).sum(-1) for j in range(k)], 1)
        torch.testing.assert_close(gg.double(), rg_stored, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(gw.double(), rw, rtol=tol['rtol'], atol=tol['atol'] * T)


def test_public_object_in_graphed_step(one_rank, monkeypatch):
    hvd = one_rank
    T, h, E, k = 256, 32, 4, 2

    def make():
        torch.manual_seed(3)
        net = torch.nn.ModuleDict({'router': torch.nn.Linear(h, E), 'head': torch.nn.Linear(h, 3)}).cuda()
        net.w = torch.nn.Parameter(torch.rand(E, h, device='cuda') + 0.5)
        disp = hvd.ExpertDispatcher(E, h, torch.float32, max_tokens=T, top_k=k, capacity=T * k)
        opt = hvd.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.05), named_parameters=net.named_parameters(),
                                       fused=True)

        def loss_fn(x, y):
            logits = net['router'](x)
            gates, idx = torch.topk(torch.softmax(logits, -1), k, dim=-1)
            expert_in, offsets, handle = disp.dispatch(x, idx)
            out = disp.combine(_expert_fn(net.w, expert_in, offsets), gates.contiguous(), handle)
            return torch.nn.functional.cross_entropy(net['head'](out), y)
        return net, opt, loss_fn

    g = torch.Generator(device='cuda').manual_seed(4)
    xs = [torch.randn(T, h, device='cuda', generator=g) for _ in range(4)]
    ys = [torch.randint(0, 3, (T,), device='cuda', generator=g) for _ in range(4)]
    ne, oe, fe = make()
    eager = hvd.GraphedStep(fe, oe, (xs[0], ys[0]), enabled=False)
    ng, og, fg = make()
    graphed = hvd.GraphedStep(fg, og, (xs[0], ys[0]), warmup_iters=2)
    assert graphed.captured, graphed.fallback_reason
    with torch.no_grad():
        for a, b in zip(ng.parameters(), ne.parameters()):
            a.copy_(b)
    for x, y in zip(xs, ys):
        eager(x, y)
        graphed(x, y)
    torch.cuda.synchronize()
    assert graphed.replays == 4
    for a, b in zip(ng.parameters(), ne.parameters()):
        assert torch.equal(a, b)


def test_public_object_failure_and_next_call(one_rank):
    hvd = one_rank
    disp = hvd.ExpertDispatcher(4, 16, torch.float32, max_tokens=100, top_k=2, capacity=50)
    x = torch.randn(100, 16, device='cuda', requires_grad=True)
    gates = torch.rand(100, 2, device='cuda', requires_grad=True)
    for idx, code in ((torch.zeros(100, 2, dtype=torch.int64, device='cuda'), RECV_OVERFLOW),
                      (torch.full((100, 2), 4, dtype=torch.int64, device='cuda'), NEGATIVE)):
        expert_in, offsets, handle = disp.dispatch(x, idx)
        y = disp.combine(expert_in * 2, gates, handle)
        gx, gg = torch.autograd.grad(y, (x, gates), torch.ones_like(y))
        assert int(handle.status) == code
        for t in (expert_in, offsets, y, gx, gg):
            assert not bool(_bytes(t.detach()).any())
    idx = torch.randint(0, 4, (20, 2), device='cuda')
    expert_in, offsets, handle = disp.dispatch(x[:20], idx)
    assert int(handle.status) == OK and int(offsets[-1]) == 40


def test_argument_errors(one_rank, monkeypatch):
    hvd = one_rank
    import horovod_b200.torch.moe as moe
    E = hvd.HorovodInternalError
    ctor = [((8, 16, torch.float64, 10, 2, 20), 'dtype'), ((0, 16, torch.float32, 10, 2, 20), 'num_experts'),
            ((1025, 16, torch.float32, 10, 2, 20), 'num_experts'), ((8, 16, torch.float32, 10, 17, 20), 'top_k'),
            ((8, 16, torch.float32, 10, 0, 20), 'top_k'), ((8, 0, torch.float32, 10, 2, 20), 'hidden'),
            ((8, 16, torch.float32, 2 ** 30, 4, 20), '2\\^31'), ((8, 16.0, torch.float32, 10, 2, 20), 'must be an int')]
    for args, msg in ctor:
        with pytest.raises(E, match=msg):
            hvd.ExpertDispatcher(*args)
    disp = hvd.ExpertDispatcher(8, 16, torch.float32, 10, 2, 20)
    x = torch.zeros(10, 16, device='cuda')
    idx = torch.zeros(10, 2, dtype=torch.int64, device='cuda')
    bad = [((x.cpu(), idx), 'CUDA tensor'), ((x[:, :8], idx), 'shape'), ((x.double(), idx), 'must be'),
           ((torch.zeros(11, 16, device='cuda'), torch.zeros(11, 2, dtype=torch.int64, device='cuda')), 'max_tokens'),
           ((torch.zeros(16, 10, device='cuda').t(), idx), 'contiguous'), ((x, idx[:, :1]), 'shape'),
           ((x, idx.float()), 'int32 or'), ((x, idx.cpu()), 'CUDA tensor'), ((x[0], idx), '2-D')]
    for args, msg in bad:
        with pytest.raises(E, match=msg):
            disp.dispatch(*args)
    expert_in, offsets, handle = disp.dispatch(x, idx)
    gates = torch.ones(10, 2, device='cuda')
    for args, msg in [((expert_in[:5], gates, handle), 'shape'), ((expert_in, gates[:5], handle), 'shape'),
                      ((expert_in, gates.double(), handle), 'must be'), ((expert_in, gates, None), 'handle'),
                      ((expert_in.half(), gates, handle), 'must be')]:
        with pytest.raises(E, match=msg):
            disp.combine(*args)
    with pytest.raises(E, match='multiple'):
        monkeypatch.setattr(hvd.global_process_set, 'size', lambda: 3)
        hvd.ExpertDispatcher(8, 16, torch.float32, 10, 2, 20)
    monkeypatch.undo()
    # a set without a peer-mapped team
    with pytest.raises(E, match='symm_available'):
        moe._symm_empty((4, 4), torch.float32, torch.device('cuda', 0), hvd.global_process_set)


# ---- real ranks -----------------------------------------------------------------------------------------------------

def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_ngpu() < 2, reason='needs >= 2 GPUs')
def test_real_ranks(native_built):
    n = 2 if _ngpu() < 4 else (4 if _ngpu() < 8 else 8)
    rc, out = run_parallel('moe_worker.py', np=n, timeout=600)
    assert 'MOE WORKER OK' in out, out[-4000:]
