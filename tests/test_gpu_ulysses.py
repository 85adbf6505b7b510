"""hvd.UlyssesExchange: the Ulysses exchange between sequence shards and head shards.

- The kernel on N = 2, 3, 4, 8 simulated ranks (`ops.sim.ulysses_exchange`), byte for byte against torch chunk / cat,
  for both directions, four layouts, three dtypes, run lengths from 2 B to several KiB, unaligned input views, empty
  tensors and more than 2^31 bytes per rank; inputs unchanged, guard bytes around the outputs untouched, and the round
  trip exact.
- A shape mismatch: status 4 and zero outputs on every rank, and the next call works.
- 100 back-to-back calls without a host sync, and all ranks captured into one CUDA graph.
- The public object on N = 2, 4, 8 simulated ranks (one thread per rank, the exchange routed into the simulation): a
  causal attention block forward and backward against the same block on the whole sequence.
- The public object inside hvd.GraphedStep on one rank with a capturable stand-in exchange, and every argument error.
- On several GPUs, tests/parallel/ulysses_worker.py runs the exchange on real ranks.
"""
import copy
import threading

import pytest
import torch
import torch.nn.functional as F

from conftest import run_parallel
from sim_ranks import FakeSet

pytestmark = pytest.mark.gpu

MISMATCH = 4
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
S2H, H2S = 0, 1
# (shape with S = seq shard and H = heads, seq_dim, head_dim)
LAYOUTS = {'BSHD': (lambda B, S, H, D: (B, S, H, D), 1, 2), 'SBHD': (lambda B, S, H, D: (S, B, H, D), 0, 2),
           'BS3HD': (lambda B, S, H, D: (B, S, 3, H, D), 1, 3), 'BHSD': (lambda B, S, H, D: (B, H, S, D), 2, 1)}


@pytest.fixture(scope='module')
def sim():
    from horovod_b200.ops import sim
    return sim


def _u8(t):
    return t.contiguous().view(-1).view(torch.uint8) if t.numel() else torch.empty(0, dtype=torch.uint8, device=t.device)


def ref(xs, seq, head, direction):
    """The contract, with torch chunk / cat."""
    n = len(xs)
    split, cat = (head, seq) if direction == S2H else (seq, head)
    return [torch.cat([x.chunk(n, split)[me] if x.shape[split] else x for x in xs], dim=cat) for me in range(n)]


def out_shape(shape, seq, head, direction, n):
    s = list(shape)
    split, cat = (head, seq) if direction == S2H else (seq, head)
    s[split] //= n
    s[cat] *= n
    return s


def _rand(shape, dtype, seed, offset=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    numel = 1
    for d in shape:
        numel *= d
    base = torch.randn(numel + offset, device='cuda', generator=g).to(dtype)
    return base[offset:].view(shape)


GUARD = 4096


def exchange(sim, xs, seq, head, direction, ctas=8, check=True):
    """One simulated exchange with guard bytes around every output; checks the guards and that the inputs are unchanged.
    Returns (outputs, statuses)."""
    n = len(xs)
    before = [x.clone() for x in xs]
    outs, bufs = [], []
    for x in xs:
        nb = x.numel() * x.element_size()
        buf = torch.full((nb + 2 * GUARD,), 0xAB, dtype=torch.uint8, device='cuda')
        bufs.append(buf)
        outs.append(buf[GUARD:GUARD + nb].view(x.dtype).view(out_shape(x.shape, seq, head, direction, n)))
    status = [torch.zeros(1, dtype=torch.int32, device='cuda') for _ in range(n)]
    sim.ulysses_exchange(xs, outs, seq, head, direction, status, ctas=ctas)
    if check:
        for r in range(n):
            assert bool((bufs[r][:GUARD] == 0xAB).all()) and bool((bufs[r][-GUARD:] == 0xAB).all()), ('guard', r)
            assert torch.equal(_u8(xs[r]), _u8(before[r])), ('input changed', r)
    return outs, [int(s) for s in status]


def check_both_ways(sim, xs, seq, head, what, ctas=8):
    ys, st = exchange(sim, xs, seq, head, S2H, ctas)
    assert st == [0] * len(xs), (what, st)
    for r, (a, b) in enumerate(zip(ys, ref(xs, seq, head, S2H))):
        assert torch.equal(_u8(a), _u8(b)), (what, 'seq_to_heads', r)
    back, st = exchange(sim, ys, seq, head, H2S, ctas)
    assert st == [0] * len(xs), (what, st)
    for r, (a, b, x) in enumerate(zip(back, ref(ys, seq, head, H2S), xs)):
        assert torch.equal(_u8(a), _u8(b)), (what, 'heads_to_seq', r)
        assert torch.equal(_u8(a), _u8(x)), (what, 'round trip', r)


@pytest.mark.parametrize('n', [2, 3, 4, 8])
@pytest.mark.parametrize('layout', list(LAYOUTS))
@pytest.mark.parametrize('dtype', DTYPES)
def test_byte_exact_layouts(sim, n, layout, dtype):
    make, seq, head = LAYOUTS[layout]
    xs = [_rand(make(2, 5, 2 * n, 3), dtype, 10 * n + r) for r in range(n)]  # runs of 2 * 3 elements: not 16 B multiples
    check_both_ways(sim, xs, seq, head, (n, layout, dtype))


@pytest.mark.parametrize('n', [2, 4])
@pytest.mark.parametrize('dtype,H,D', [(torch.float16, 4, 1), (torch.bfloat16, 4, 3), (torch.float32, 4, 5),
                                       (torch.float16, 8, 64), (torch.float32, 8, 1500), (torch.float32, 4, 2048)])
def test_run_lengths(sim, n, dtype, H, D):
    """Runs of (H / n) * D elements from 2 B to 8 KiB, and head first runs of 7 * D elements up to 56 KiB (several
    8 KiB pieces per run); totals past 32 KiB."""
    xs = [_rand((3, 7, H, D), dtype, r) for r in range(n)]
    check_both_ways(sim, xs, 1, 2, (n, dtype, H, D))
    check_both_ways(sim, [x.transpose(1, 2).contiguous() for x in xs], 2, 1, (n, dtype, H, D, 'head first'))


@pytest.mark.parametrize('offset', [1, 3])
def test_unaligned_input_view(sim, offset):
    n = 4
    for dtype in (torch.float16, torch.float32):
        xs = [_rand((2, 9, 8, 16), dtype, r, offset=offset) for r in range(n)]
        check_both_ways(sim, xs, 1, 2, (dtype, offset))


def test_zero_size(sim):
    for n in (2, 4):
        xs = [torch.empty(2, 0, 2 * n, 8, device='cuda') for _ in range(n)]
        for direction in (S2H, H2S):
            outs, st = exchange(sim, xs, 1, 2, direction)
            assert st == [0] * n and all(o.numel() == 0 for o in outs)
    # the team still works after the empty exchanges (every rank met both barriers)
    check_both_ways(sim, [_rand((2, 4, 8, 8), torch.float32, r) for r in range(4)], 1, 2, 'after empty')


def test_more_than_2_31_bytes_per_rank(sim):
    n, shape = 2, (1, 2 ** 15 + 1, 16, 2048)  # 2^31 + 2^16 bytes of bf16 per rank
    xs = [torch.empty(shape, dtype=torch.bfloat16, device='cuda') for _ in range(n)]
    for r, x in enumerate(xs):
        # every element distinct modulo 2^16 within a row, different per rank, and cheap to make
        x.view(-1).view(torch.int16).copy_(torch.arange(x.numel(), device='cuda', dtype=torch.int32).to(torch.int16) + 7 * r)
    outs, st = exchange(sim, xs, 1, 2, S2H, ctas=64, check=False)
    assert st == [0] * n
    for me in range(n):
        for p in range(n):
            got = outs[me][:, p * shape[1]:(p + 1) * shape[1]]
            assert torch.equal(got.view(torch.int16), xs[p][:, :, me * 8:(me + 1) * 8].view(torch.int16)), (me, p)
    del outs
    torch.cuda.empty_cache()


def test_shape_mismatch_then_next_call(sim):
    n = 4
    xs = [_rand((2, 6 if r == 1 else 5, 8, 4), torch.float32, r) for r in range(n)]
    outs = [torch.full(out_shape(x.shape, 1, 2, S2H, n), float('nan'), device='cuda') for x in xs]
    status = [torch.zeros(1, dtype=torch.int32, device='cuda') for _ in range(n)]
    sim.ulysses_exchange(xs, outs, 1, 2, S2H, status)
    assert [int(s) for s in status] == [MISMATCH] * n
    assert all(not bool(_u8(o).any()) for o in outs)
    # the status keeps the first non-zero code across a later good call
    xs = [_rand((2, 5, 8, 4), torch.float32, 10 + r) for r in range(n)]
    sim.ulysses_exchange(xs, [torch.empty(out_shape(x.shape, 1, 2, S2H, n), device='cuda') for x in xs], 1, 2, S2H, status)
    assert [int(s) for s in status] == [MISMATCH] * n
    check_both_ways(sim, xs, 1, 2, 'next call')


def test_back_to_back_without_sync(sim):
    n, shape = 4, (2, 64, 8, 32)
    xs = [torch.zeros(shape, dtype=torch.bfloat16, device='cuda') for _ in range(n)]
    staging = [torch.empty(xs[0].numel() * 2, dtype=torch.uint8, device='cuda') for _ in range(n)]
    status = [torch.zeros(1, dtype=torch.int32, device='cuda') for _ in range(n)]
    sim.ulysses_exchange(xs, [torch.empty(out_shape(shape, 1, 2, S2H, n), dtype=xs[0].dtype, device='cuda') for _ in xs],
                         1, 2, S2H, status, staging=staging)  # creates the simulated team
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(n)]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    seen, outs = [], []
    for it in range(100):
        ins = []
        for r in range(n):
            with torch.cuda.stream(streams[r]):  # new input written on the rank's stream, right before its exchange
                xs[r].copy_(torch.full(shape, float(it % 64 + r), dtype=torch.bfloat16, device='cuda')
                            + torch.arange(shape[2], device='cuda').view(1, 1, -1, 1).to(torch.bfloat16))
                ins.append(xs[r].clone())
        o = [torch.empty(out_shape(shape, 1, 2, S2H, n), dtype=xs[0].dtype, device='cuda') for _ in range(n)]
        sim.ulysses_exchange(xs, o, 1, 2, S2H, status, staging=staging, streams=streams)
        seen.append(ins)
        outs.append(o)
    torch.cuda.synchronize()
    assert [int(s) for s in status] == [0] * n
    for it in range(100):
        for r, (a, b) in enumerate(zip(outs[it], ref(seen[it], 1, 2, S2H))):
            assert torch.equal(_u8(a), _u8(b)), (it, r)


@pytest.mark.parametrize('n', [2, 4, 8])
def test_all_ranks_in_one_cuda_graph(sim, n):
    shape = (2, 16, 3, 2 * n, 24)
    xs = [_rand(shape, torch.bfloat16, r) for r in range(n)]
    staging = [torch.empty(xs[0].numel() * 2, dtype=torch.uint8, device='cuda') for _ in range(n)]
    status = [torch.zeros(1, dtype=torch.int32, device='cuda') for _ in range(n)]
    ys = [torch.empty(out_shape(shape, 1, 3, S2H, n), dtype=torch.bfloat16, device='cuda') for _ in range(n)]
    back = [torch.empty(shape, dtype=torch.bfloat16, device='cuda') for _ in range(n)]
    sim.ulysses_exchange(xs, ys, 1, 3, S2H, status, staging=staging)  # warm-up: the simulated team
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(n)]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cur = torch.cuda.current_stream()
        for s in streams:
            s.wait_stream(cur)
        sim.ulysses_exchange(xs, ys, 1, 3, S2H, status, staging=staging, streams=streams)
        sim.ulysses_exchange(ys, back, 1, 3, H2S, status, staging=staging, streams=streams)
        for s in streams:
            cur.wait_stream(s)
    gen = torch.Generator(device='cuda').manual_seed(5)
    for it in range(3):
        for x in xs:
            x.copy_(torch.randn(shape, device='cuda', generator=gen).to(torch.bfloat16))
        graph.replay()
        torch.cuda.synchronize()
        assert [int(s) for s in status] == [0] * n
        for r, (a, b) in enumerate(zip(ys, ref(xs, 1, 3, S2H))):
            assert torch.equal(_u8(a), _u8(b)), ('replay', it, r)
        for r in range(n):
            assert torch.equal(_u8(back[r]), _u8(xs[r])), ('replay round trip', it, r)


# ---- the public object on simulated ranks ------------------------------------------------------------------------------

class SimUlysses:
    """The exchanges of N simulated ranks, one thread each: every rank's call waits until all N ranks issued theirs, then
    one ops.sim.ulysses_exchange runs them on the real kernel and each rank gets its own output (a lockstep queue like
    tests/sim_ranks.py:SimTeam)."""

    def __init__(self, sim, n):
        self.sim, self.n, self.calls, self.outs, self.count = sim, n, [None] * n, [None] * n, 0
        self.barrier = threading.Barrier(n, action=self._run)

    def exchange(self, tensor, staging, status, seq_dim, head_dim, direction, process_set, max_ctas):
        self.calls[process_set.rank()] = (tensor, staging, status, seq_dim, head_dim, direction)
        self.barrier.wait(timeout=120)
        return self.outs[process_set.rank()]

    def _run(self):
        torch.cuda.synchronize()
        c = self.calls
        assert len({x[3:] for x in c}) == 1, 'ranks issued different exchanges'
        seq, head, direction = c[0][3:]
        outs = [torch.empty(out_shape(x[0].shape, seq, head, direction, self.n), dtype=x[0].dtype, device='cuda') for x in c]
        self.sim.ulysses_exchange([x[0] for x in c], outs, seq, head, direction, [x[2] for x in c],
                                  staging=[x[1] for x in c], ctas=4)
        self.outs, self.count = outs, self.count + 1

    def run(self, fn):
        res, errs = [None] * self.n, []

        def body(r):
            try:
                with torch.autograd.set_multithreading_enabled(False):  # each rank's backward on its own thread
                    res[r] = fn(r)
            except BaseException as e:  # noqa: B036  re-raised below
                errs.append(e)
                self.barrier.abort()
        ths = [threading.Thread(target=body, args=(r,)) for r in range(self.n)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        if errs:
            raise errs[0]
        torch.cuda.synchronize()
        return res


class Attention(torch.nn.Module):
    """A causal self-attention block with fused QKV; forward(x, ex) runs it sequence-parallel through ex."""

    def __init__(self, h, H, D):
        super().__init__()
        self.H, self.D = H, D
        self.qkv = torch.nn.Linear(h, 3 * H * D)
        self.proj = torch.nn.Linear(H * D, h)

    def forward(self, x, ex=None):
        B, S = x.shape[:2]
        qkv = self.qkv(x).view(B, S, 3, self.H, self.D)
        if ex is not None:
            qkv = ex.seq_to_heads(qkv, 1, 3)
        q, k, v = (t.transpose(1, 2) for t in qkv.unbind(2))
        o = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).contiguous()
        if ex is not None:
            o = ex.heads_to_seq(o, 1, 2)
        return self.proj(o.reshape(B, o.shape[1], self.H * self.D))


@pytest.fixture
def hvd_one(monkeypatch):
    import horovod_b200.torch as hvd
    import horovod_b200.torch.sequence_parallel as sp
    hvd.init()
    torch.cuda.set_device(0)
    monkeypatch.setattr(sp, '_symm_empty', lambda numel, dtype, device, ps: torch.zeros(numel, dtype=dtype, device=device))
    yield hvd, sp
    hvd.shutdown()


# fp32: the same math on every token and head, only the attention of each head split off: 1e-4.  bf16: the QKV and
# output projections round differently per shard shape: 2e-2.
TOL = {torch.float32: dict(rtol=1e-4, atol=1e-4), torch.bfloat16: dict(rtol=2e-2, atol=2e-2)}


@pytest.mark.parametrize('n', [2, 4, 8])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_attention_block_on_simulated_ranks(sim, hvd_one, monkeypatch, n, dtype):
    hvd, sp = hvd_one
    team = SimUlysses(sim, n)
    monkeypatch.setattr(sp, '_exchange', team.exchange)
    B, S, h, H, D = 2, 64, 48, 16, 8
    torch.manual_seed(0)
    dense = Attention(h, H, D).cuda().to(dtype)
    blocks = [copy.deepcopy(dense) for _ in range(n)]
    exs = [hvd.UlyssesExchange(B * S * 3 * H * D // n, dtype, process_set=FakeSet(n, r)) for r in range(n)]
    g = torch.Generator(device='cuda').manual_seed(1)
    x = torch.randn(B, S, h, device='cuda', generator=g).to(dtype)
    gy = torch.randn(B, S, h, device='cuda', generator=g).to(dtype)
    xs = [t.contiguous().requires_grad_() for t in x.chunk(n, 1)]

    def rank(r):
        y = blocks[r](xs[r], exs[r])
        (y * gy.chunk(n, 1)[r]).sum().backward()
        return y.detach()
    ys = team.run(rank)
    assert team.count == 4, team.count  # two exchanges forward, two backward
    assert all(int(ex.status) == 0 for ex in exs)
    xd = x.clone().requires_grad_()
    yd = dense(xd)
    (yd * gy).sum().backward()
    tol = TOL[dtype]
    torch.testing.assert_close(torch.cat(ys, 1).float(), yd.detach().float(), **tol)
    for r in range(n):
        torch.testing.assert_close(xs[r].grad.float(), xd.grad.chunk(n, 1)[r].float(), **tol)
    for name, p in dense.named_parameters():
        summed = sum(dict(b.named_parameters())[name].grad.float() for b in blocks)
        torch.testing.assert_close(summed, p.grad.float(), rtol=tol['rtol'], atol=tol['atol'] * n, msg=name)


# ---- the public object on one rank ------------------------------------------------------------------------------------

def _identity_exchange(tensor, staging, status, seq_dim, head_dim, direction, process_set, max_ctas):
    """The exchange of a one-rank set (a copy), with the kernel's sticky status: capturable torch ops."""
    out = tensor.clone()
    status.copy_(torch.where(status != 0, status, torch.zeros_like(status)))
    return out


def test_public_object_in_graphed_step(hvd_one, monkeypatch):
    hvd, sp = hvd_one
    monkeypatch.setattr(sp, '_exchange', _identity_exchange)
    B, S, h, H, D = 2, 32, 32, 4, 8

    def make():
        torch.manual_seed(3)
        net = torch.nn.ModuleDict({'attn': Attention(h, H, D), 'head': torch.nn.Linear(h, 5)}).cuda()
        ex = hvd.UlyssesExchange(B * S * 3 * H * D, torch.float32)
        opt = hvd.DistributedOptimizer(torch.optim.SGD(net.parameters(), lr=0.05), named_parameters=net.named_parameters(),
                                       fused=True)

        def loss_fn(x, y):
            ex.status.zero_()
            out = net['attn'](x, ex)
            return F.cross_entropy(net['head'](out).flatten(0, 1), y.flatten())
        return net, opt, loss_fn, ex

    g = torch.Generator(device='cuda').manual_seed(4)
    xs = [torch.randn(B, S, h, device='cuda', generator=g) for _ in range(4)]
    ys = [torch.randint(0, 5, (B, S), device='cuda', generator=g) for _ in range(4)]
    ne, oe, fe, exe = make()
    eager = hvd.GraphedStep(fe, oe, (xs[0], ys[0]), enabled=False)
    ng, og, fg, exg = make()
    graphed = hvd.GraphedStep(fg, og, (xs[0], ys[0]), warmup_iters=2)
    assert graphed.captured, graphed.fallback_reason
    with torch.no_grad():
        for a, b in zip(ng.parameters(), ne.parameters()):
            a.copy_(b)
    for x, y in zip(xs, ys):
        exe.status.fill_(MISMATCH)  # the step's own reset clears it, eager and replayed alike
        exg.status.fill_(MISMATCH)
        eager(x, y)
        graphed(x, y)
    torch.cuda.synchronize()
    assert graphed.replays == 4
    assert int(exe.status) == int(exg.status) == 0
    for a, b in zip(ng.parameters(), ne.parameters()):
        assert torch.equal(a, b)


def test_argument_errors(hvd_one, monkeypatch):
    hvd, sp = hvd_one
    E = hvd.HorovodInternalError
    for args, msg in [((0, torch.float32), 'max_numel'), ((16, torch.float64), 'dtype'), ((16.0, torch.float32), 'must be an int'),
                      ((16, torch.float32, hvd.global_process_set, -1), 'max_ctas')]:
        with pytest.raises(E, match=msg):
            hvd.UlyssesExchange(*args)
    monkeypatch.setattr(hvd.global_process_set, 'size', lambda: 2)
    ex = hvd.UlyssesExchange(1000, torch.float32)
    x = torch.zeros(2, 4, 6, 5, device='cuda')
    bad = [((x.cpu(), 1, 2), 'CUDA tensor'), ((x.double(), 1, 2), 'must be torch.float32'),
           ((x.transpose(1, 2), 2, 1), 'contiguous'), ((torch.zeros(2, 4, 6, 50, device='cuda'), 1, 2), 'max_numel'),
           ((x, 4, 2), 'seq_dim'), ((x, 1, -5), 'head_dim'), ((x, 1, 1), 'differ'), ((x, 1.0, 2), 'seq_dim'),
           ((torch.zeros(2, 4, 5, 5, device='cuda'), 1, 2), 'multiple')]
    for args, msg in bad:
        with pytest.raises(E, match=msg):
            ex.seq_to_heads(*args)
    with pytest.raises(E, match='multiple'):
        ex.heads_to_seq(torch.zeros(2, 5, 6, 5, device='cuda'), 1, 2)
    monkeypatch.undo()
    if torch.cuda.device_count() > 1:
        with pytest.raises(E, match='CUDA tensor on'):
            ex.seq_to_heads(torch.zeros(2, 4, 6, 5, device='cuda:1'), 1, 2)
    # a set without a peer-mapped team
    with pytest.raises(E, match='symm_available'):
        sp._symm_empty(4, torch.float32, torch.device('cuda', 0), hvd.global_process_set)
    # the binding's own checks, before anything is launched
    nat = hvd.mpi_ops._native()
    st = torch.zeros(1, dtype=torch.int32, device='cuda')
    stg = torch.zeros(4096, dtype=torch.uint8, device='cuda')
    call = dict(tensor=x, staging=stg, status=st, seq_dim=1, head_dim=2, direction=0, nranks=2, process_set_id=0, max_ctas=0)
    for change, msg in [(dict(tensor=x.cpu()), 'CUDA tensor expected'), (dict(tensor=x.transpose(1, 2)), 'contiguous'),
                        (dict(direction=2), 'direction'), (dict(nranks=9), 'nranks'), (dict(seq_dim=2), 'distinct'),
                        (dict(head_dim=4), 'distinct'), (dict(nranks=4), 'multiple of 4'),
                        (dict(staging=stg.cpu()), 'staging must be'), (dict(staging=stg[:100]), 'staging buffer'),
                        (dict(status=st.long()), 'status'), (dict(status=torch.zeros(2, dtype=torch.int32, device='cuda')), 'status'),
                        (dict(), 'sized for 2 ranks')]:
        with pytest.raises((RuntimeError, ValueError), match=msg):
            nat.captured_ulysses_exchange(**dict(call, **change))
    with pytest.raises((RuntimeError, ValueError), match='at least 2 ranks'):
        nat.captured_ulysses_exchange(**dict(call, nranks=1))


# ---- real ranks -----------------------------------------------------------------------------------------------------

def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_ngpu() < 2, reason='needs >= 2 GPUs')
def test_real_ranks(native_built):
    n = 2 if _ngpu() < 4 else (4 if _ngpu() < 8 else 8)
    rc, out = run_parallel('ulysses_worker.py', np=n, timeout=900)
    assert 'ULYSSES WORKER OK' in out, out[-4000:]
