"""hvd.captured_alltoall: the alltoall whose split vectors only the device reads, one kernel per rank.

On N simulated ranks on one GPU (`horovod_b200.ops.sim.captured_alltoall`: the real kernel, count region and flag
barriers on N streams), against a reference built with torch indexing:
- byte-exact outputs for N = 2, 3, 4, 8 and row sizes of 1, 2, 6, 16 and 4098 bytes over seeded random split matrices,
  with ranks that send or receive nothing, one rank that receives everything, totals past the 32 KiB chunk and one
  exchange of 256 MiB per rank; output rows past the received total keep their guard bytes, inputs are unchanged and
  recv_splits is exact;
- every status code, produced by device-side splits: the same code on every rank, no output byte written, and a valid
  call right after that succeeds;
- 100 calls with no host synchronisation in between, each with new device-generated splits and new inputs written on the
  ranks' streams (barrier B and the reuse of the count region);
- all N ranks captured into one CUDA graph, replayed with splits rewritten on the device, no host sync during replay;
- the host-side argument checks of the binding, the engine and the Python function.

On several GPUs, tests/parallel/captured_alltoall_worker.py compares the call, eager and captured, with hvd.alltoall.
"""
import pytest
import torch

from conftest import run_parallel
from optim_cases import hvd  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

GUARD = 0x5A
CTAS = 8
CHUNK = 32768
OK, NEGATIVE, SEND_OVERFLOW, RECV_OVERFLOW, ROW_BYTES = 0, 1, 2, 3, 4
# (dtype, row shape): row sizes of 1, 2, 6, 16 and 4098 bytes
ROWS = [(torch.uint8, ()), (torch.bfloat16, ()), (torch.float16, (3,)), (torch.float32, (4,)), (torch.int16, (2049,))]
ROW_IDS = ['1B', '2B', '6B', '16B', '4098B']


@pytest.fixture(scope='module')
def sim():
    from horovod_b200.ops import sim
    return sim


def _bytes(t):
    return t.contiguous().view(-1).view(torch.uint8) if t.numel() else torch.empty(0, dtype=torch.uint8, device=t.device)


def _random_input(rows, dtype, row, gen):
    raw = torch.randint(0, 256, (rows * _numel(row) * torch.empty(0, dtype=dtype).element_size(),), dtype=torch.uint8,
                        device='cuda', generator=gen)
    return raw.view(dtype).view(rows, *row)


def _numel(row):
    n = 1
    for d in row:
        n *= d
    return n


class Case:
    """Every simulated rank's input [S_p, *row], splits (device), guard-filled output [capacity_q, *row], recv_splits and
    status, for the split matrix M (M[p][q] = rows p sends to q)."""

    def __init__(self, M, dtype, row, slack_in=3, slack_out=5, seed=0, split_dtype=torch.int64, caps=None):
        n = len(M)
        gen = torch.Generator(device='cuda').manual_seed(seed)
        self.M, self.n = M, n
        self.ins = [_random_input(sum(M[p]) + slack_in, dtype, row, gen) for p in range(n)]
        self.before = [x.clone() for x in self.ins]
        caps = caps or [sum(M[p][q] for p in range(n)) + slack_out for q in range(n)]
        self.outs = [torch.empty(caps[q], *row, dtype=dtype, device='cuda') for q in range(n)]
        for o in self.outs:
            _bytes(o).fill_(GUARD)
        self.splits = [torch.tensor(M[p], dtype=split_dtype, device='cuda') for p in range(n)]
        self.recv = [torch.full((n,), -7, dtype=torch.int64, device='cuda') for _ in range(n)]
        self.status = [torch.full((1,), -7, dtype=torch.int32, device='cuda') for _ in range(n)]

    def run(self, sim, ctas=CTAS, streams=None):
        sim.captured_alltoall(self.ins, self.splits, self.outs, self.recv, self.status, ctas=ctas, streams=streams)


def reference(ins, M, q):
    """What rank q receives: rank p's rows [sum M[p][:q], + M[p][q]) for p in rank order."""
    parts = []
    for p in range(len(M)):
        off = sum(M[p][:q])
        parts.append(ins[p][off:off + M[p][q]])
    return torch.cat(parts)


def check_exact(c, ins=None, M=None, outs=None, recv=None, status=None, what=''):
    ins, M = ins or c.ins, M or c.M
    outs, recv, status = outs or c.outs, recv or c.recv, status or c.status
    torch.cuda.synchronize()
    for q in range(c.n):
        assert int(status[q]) == OK, (what, q, int(status[q]))
        ref = reference(ins, M, q)
        got = outs[q][:ref.shape[0]]
        assert torch.equal(_bytes(got), _bytes(ref)), (what, 'rank', q, 'received wrong bytes')
        assert bool((_bytes(outs[q][ref.shape[0]:]) == GUARD).all()), (what, 'rank', q, 'wrote past the received rows')
        assert recv[q].tolist() == [M[p][q] for p in range(c.n)], (what, q, recv[q].tolist())


def inputs_unchanged(c):
    for p in range(c.n):
        assert torch.equal(_bytes(c.ins[p]), _bytes(c.before[p])), ('input of rank', p, 'changed')


def random_matrix(n, max_rows, seed, zero_frac=0.25):
    """Seeded random split matrix, drawn on the device, with about zero_frac of the entries zero."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    m = torch.randint(0, max_rows + 1, (n, n), device='cuda', generator=g)
    m = m * (torch.rand((n, n), device='cuda', generator=g) >= zero_frac)
    return m.tolist()


# ---- byte-exact results ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize('n', [2, 3, 4, 8])
@pytest.mark.parametrize('spec', ROWS, ids=ROW_IDS)
def test_random_matrices_byte_exact(sim, n, spec):
    dtype, row = spec
    row_bytes = _numel(row) * torch.empty(0, dtype=dtype).element_size()
    # per receiver about 3 chunks on average, so that most totals cross the chunk size
    max_rows = max(2, 6 * CHUNK // (row_bytes * n))
    for seed in range(3):
        M = random_matrix(n, max_rows, 1000 * n + 10 * row_bytes + seed)
        M[n - 1][seed % n] = max(M[n - 1][seed % n], CHUNK // row_bytes + 1)  # at least one total past the chunk size
        c = Case(M, dtype, row, seed=seed, split_dtype=torch.int64 if seed % 2 == 0 else torch.int32)
        c.run(sim)
        check_exact(c, what=(n, row_bytes, seed))
        inputs_unchanged(c)


@pytest.mark.parametrize('n', [2, 3, 8])
@pytest.mark.parametrize('spec', [ROWS[0], ROWS[3], ROWS[4]], ids=['1B', '16B', '4098B'])
def test_edge_matrices(sim, n, spec):
    dtype, row = spec
    big = 3 * CHUNK // (_numel(row) * torch.empty(0, dtype=dtype).element_size()) + 7
    cases = {
        'all zero': [[0] * n for _ in range(n)],
        'rank 0 sends nothing, rank n-1 receives nothing': [[0] * n] + [[(p + q) % 5 + 1 if q < n - 1 else 0 for q in range(n)]
                                                                         for p in range(1, n)],
        'rank 1 receives everything': [[big if q == 1 else 0 for q in range(n)] for p in range(n)],
        'only self': [[big if q == p else 0 for q in range(n)] for p in range(n)],
    }
    for i, (what, M) in enumerate(cases.items()):
        c = Case(M, dtype, row, seed=i)
        c.run(sim, ctas=3)
        check_exact(c, what=(n, what))
        inputs_unchanged(c)


def test_256_mib_per_rank(sim):
    """Two ranks exchanging 256 MiB each: 32768 rows of 4096 bf16 per rank, uneven splits, default grid of 32 CTAs."""
    n, rows = 2, 32768
    M = [[12345, rows - 12345], [rows - 777, 777]]
    c = Case(M, torch.bfloat16, (4096,), slack_in=0, slack_out=1, seed=3)
    assert all(x.numel() * x.element_size() >= 256 << 20 for x in c.ins)
    c.run(sim, ctas=32)
    check_exact(c, what='256 MiB')
    inputs_unchanged(c)


# ---- status codes ---------------------------------------------------------------------------------------------------

def _device_splits(n, rows, bad_rank=None, bad_col=0, value=None, add=0):
    """Every rank's splits made on the device: rows // n each, one entry of `bad_rank` set to `value` or raised by `add`."""
    out = []
    for p in range(n):
        s = torch.full((n,), rows // n, dtype=torch.int64, device='cuda')
        if p == bad_rank:
            if value is not None:
                s[bad_col] = value
            s[bad_col] += add
        out.append(s)
    return out


@pytest.mark.parametrize('n', [2, 3, 4])
@pytest.mark.parametrize('code', [NEGATIVE, SEND_OVERFLOW, RECV_OVERFLOW, ROW_BYTES])
def test_status_codes(sim, n, code):
    rows = 8 * n
    dtype, row = torch.float32, (4,)
    base = [[rows // n] * n for _ in range(n)]
    c = Case(base, dtype, row, slack_in=0, slack_out=0, seed=code)
    if code == NEGATIVE:
        c.splits = _device_splits(n, rows, bad_rank=n - 1, bad_col=0, value=-1)
    elif code == SEND_OVERFLOW:
        c.splits = _device_splits(n, rows, bad_rank=1, bad_col=n - 1, add=1)  # rank 1 sends S + 1 rows
    elif code == RECV_OVERFLOW:
        c.splits = _device_splits(n, rows, bad_rank=0, bad_col=0, add=0)
        c.splits[0][1] -= 1
        c.splits[0][0] += 1  # rank 0 receives capacity + 1 rows (rank 0 still sends exactly S)
    else:
        c.ins[1] = _random_input(rows, dtype, (5,), torch.Generator(device='cuda').manual_seed(9))
        c.outs[1] = torch.empty(rows, 5, dtype=dtype, device='cuda')
        _bytes(c.outs[1]).fill_(GUARD)
    sent = [s.tolist() for s in c.splits]
    c.before = [x.clone() for x in c.ins]
    c.run(sim)
    torch.cuda.synchronize()
    assert [int(s) for s in c.status] == [code] * n, ([int(s) for s in c.status], code)
    for q in range(n):
        assert bool((_bytes(c.outs[q]) == GUARD).all()), ('rank', q, 'wrote output bytes under status', code)
        assert c.recv[q].tolist() == [sent[p][q] for p in range(n)], ('recv_splits of rank', q)
    inputs_unchanged(c)
    # the next call works normally
    ok = Case(base, dtype, row, seed=code + 10)
    ok.run(sim)
    check_exact(ok, what=('after status', code))


# ---- back to back ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('n', [3, 4])
def test_100_calls_without_host_sync(sim, n):
    calls, max_rows, row = 100, 40, (24,)  # 48 B bf16 rows: 16 B vectors and byte tails
    S = cap = n * max_rows
    gen = torch.Generator(device='cuda').manual_seed(n)
    splits = torch.randint(0, max_rows + 1, (calls, n, n), device='cuda', generator=gen)  # [call][p][q]
    src = torch.randn(calls, n, S, *row, device='cuda', generator=gen).to(torch.bfloat16)
    ins = [torch.empty(S, *row, dtype=torch.bfloat16, device='cuda') for _ in range(n)]
    outs = [[torch.full((cap, *row), 0, dtype=torch.bfloat16, device='cuda') for _ in range(n)] for _ in range(calls)]
    for per in outs:
        for o in per:
            _bytes(o).fill_(GUARD)
    recv = [[torch.empty(n, dtype=torch.int64, device='cuda') for _ in range(n)] for _ in range(calls)]
    status = [[torch.empty(1, dtype=torch.int32, device='cuda') for _ in range(n)] for _ in range(calls)]
    warm = Case([[1] * n for _ in range(n)], torch.bfloat16, row)
    warm.run(sim)  # creates the simulated team of this rank count
    streams = [torch.cuda.Stream() for _ in range(n)]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    for k in range(calls):
        for r in range(n):
            with torch.cuda.stream(streams[r]):
                ins[r].copy_(src[k, r])  # rank r's next input, written as soon as its previous call returned
        sim.captured_alltoall(ins, [splits[k, r] for r in range(n)], outs[k], recv[k], status[k], ctas=4, streams=streams)
    for s in streams:
        torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    M_all = splits.tolist()
    for k in range(calls):
        c = Case.__new__(Case)
        c.n = n
        check_exact(c, ins=[src[k, r] for r in range(n)], M=M_all[k], outs=outs[k], recv=recv[k], status=status[k], what=('call', k))


# ---- CUDA graph -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('n', [2, 4, 8])
def test_all_ranks_in_one_cuda_graph(sim, n):
    max_rows, row = 300, (8,)  # 32 B fp32 rows
    S = cap = n * max_rows
    gen = torch.Generator(device='cuda').manual_seed(100 + n)
    ins = [torch.empty(S, *row, device='cuda') for _ in range(n)]
    src = [torch.empty(S, *row, device='cuda') for _ in range(n)]
    splits = [torch.zeros(n, dtype=torch.int32, device='cuda') for _ in range(n)]
    outs = [torch.empty(cap, *row, device='cuda') for _ in range(n)]
    recv = [torch.empty(n, dtype=torch.int64, device='cuda') for _ in range(n)]
    status = [torch.empty(1, dtype=torch.int32, device='cuda') for _ in range(n)]
    sim.captured_alltoall(ins, splits, outs, recv, status, ctas=CTAS)  # warm-up: creates the simulated team
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(n)]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cur = torch.cuda.current_stream()
        for r in range(n):
            streams[r].wait_stream(cur)
            with torch.cuda.stream(streams[r]):
                ins[r].copy_(src[r])  # the producer of rank r's rows, inside the graph
        sim.captured_alltoall(ins, splits, outs, recv, status, ctas=CTAS, streams=streams)
        for r in range(n):
            cur.wait_stream(streams[r])
    for it in range(12):
        for r in range(n):
            splits[r].copy_(torch.randint(0, max_rows + 1, (n,), device='cuda', generator=gen))
            src[r].copy_(torch.randn(S, *row, device='cuda', generator=gen))
            _bytes(outs[r]).fill_(GUARD)
        torch.cuda.set_sync_debug_mode('error')
        try:
            g.replay()
        finally:
            torch.cuda.set_sync_debug_mode('default')
        M = [s.tolist() for s in splits]
        c = Case.__new__(Case)
        c.n = n
        check_exact(c, ins=src, M=M, outs=outs, recv=recv, status=status, what=('replay', it))


# ---- host-side argument errors --------------------------------------------------------------------------------------

def test_argument_errors(hvd, monkeypatch):
    from horovod_b200.torch import mpi_ops
    x = torch.zeros(16, 4, device='cuda')
    sp = torch.zeros(1, dtype=torch.int64, device='cuda')
    # a set of one rank has no peer-mapped team
    with pytest.raises(hvd.HorovodInternalError, match='symm_available'):
        hvd.captured_alltoall(x, sp, 16)
    monkeypatch.setattr(mpi_ops, 'symm_available', lambda process_set: True)  # past the Python check, into the binding
    bad = [
        ((x.cpu(), sp, 16), 'CUDA tensor expected'),
        ((torch.zeros((), device='cuda'), sp, 16), 'at least one dimension'),
        ((x.t(), sp, 16), 'must be contiguous'),
        ((x, sp.cpu(), 16), 'splits must be on the tensor'),
        ((x, sp.float(), 16), 'int32 or int64'),
        ((x, sp.view(1, 1), 16), 'contiguous 1-D'),
        ((x, torch.zeros(4, dtype=torch.int64, device='cuda')[::2], 16), 'contiguous 1-D'),
        ((x, sp, -1), 'capacity must be >= 0'),
        ((x, torch.zeros(2, dtype=torch.int64, device='cuda'), 16), 'splits has 2 entries'),
        ((x, sp, 16), 'at least 2 ranks'),
    ]
    for args, msg in bad:
        with pytest.raises(hvd.HorovodInternalError, match=msg):
            hvd.captured_alltoall(*args)


# ---- real ranks -----------------------------------------------------------------------------------------------------

def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_real_ranks_match_alltoall(native_built):
    n = 2 if _ngpu() < 4 else (4 if _ngpu() < 8 else 8)
    rc, out = run_parallel("captured_alltoall_worker.py", np=n, timeout=420)
    assert "CAPTURED ALLTOALL OK" in out, out[-4000:]
