"""Launch plans of allreduce, reducescatter, allgather(v), broadcast and alltoall(v) (csrc/ops/collective_plan.{h,cc}) on
the host, no GPU needed.

`hvd_plan_collective` plans every rank of a simulated team with fake tensor addresses (never dereferenced), runs the
cross-rank agreement check (`CheckPlans`: same launches and grids on every rank, buffer bounds and alignment, every
receive inside a send of its peer, the reducescatter region layout, exact coverage of every output) and returns each
byte range the plans move.  This file decodes those ranges and compares them with where the bytes must come from,
computed here independently of the planner: the row split of reducescatter (the first dim0 % n ranks get one extra row),
allgather displacements, alltoall send / receive displacements, and the broadcast root.

`hvd_plan_allreduce` returns one rank's allreduce plan, which must match tests/golden/allreduce_plans.json field for field:
the launches the engine made before the plan was a host function.
"""
import ctypes
import json
import os

import numpy as np
import pytest

RS, AG, BC, A2A = 0, 1, 2, 3
ESZ_DTYPE = {1: 0, 2: 6, 4: 7, 8: 8}  # element size -> a dtype code of that size (uint8, fp16, fp32, fp64)
SUM = 1
IN, OUT = 1, 2
_lib = None


def lib():
    global _lib
    if _lib is None:
        from horovod_b200.common.basics import load_library
        L = load_library()
        i64p, u64p = ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_uint64)
        L.hvd_plan_collective.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, i64p, i64p, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_int, u64p, u64p, ctypes.c_int64, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                          i64p, ctypes.c_int64, ctypes.c_char_p, ctypes.c_int]
        L.hvd_plan_collective.restype = ctypes.c_int64
        L.hvd_plan_allreduce.argtypes = [ctypes.c_int, ctypes.c_int, i64p, u64p, u64p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_double, ctypes.c_double, ctypes.c_char_p, ctypes.c_int64, ctypes.c_int,
                                         ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int64, i64p, ctypes.c_int64, i64p,
                                         ctypes.c_int64, ctypes.c_char_p, ctypes.c_int]
        L.hvd_plan_allreduce.restype = ctypes.c_int64
        _lib = L
    return _lib


def addr(io, rank, t, off=0):
    """Fake address of byte `off` of tensor t of `rank` (io: IN / OUT): the fields decode back exactly."""
    return ((io * 16 + rank + 1) << 48) | (t << 36) | off


def decode(a):
    a = np.asarray(a, dtype=np.int64)
    top = a >> 48
    return top // 16, top % 16 - 1, (a >> 36) & 0xFFF, a & ((1 << 36) - 1)


class Config:
    """One collective: kind, n ranks, per-tensor sizes, element size, cap, ctas, broadcast root / in-place flag."""

    def __init__(self, kind, n, dims, rows, esz, cap, ctas, root=-1, inplace=False):
        self.kind, self.n, self.dims, self.rows, self.esz = kind, n, dims, rows, esz
        self.cap, self.ctas, self.root, self.inplace = cap, ctas, root, inplace
        self.T = len(rows)

    # --- sizes in bytes, computed here from the definitions of the ops -------------------------------------------------
    def rs_rows(self, t):
        d0 = self.dims[t]
        return [d0 // self.n + (1 if q < d0 % self.n else 0) for q in range(self.n)]

    def in_bytes(self, r, t):
        row = self.rows[t] * self.esz
        if self.kind == RS:
            return self.dims[t] * row
        if self.kind == AG:
            return self.dims[t][r] * row
        if self.kind == BC:
            return self.dims[t]
        return sum(self.dims[t][r]) * row

    def out_bytes(self, r, t):
        row = self.rows[t] * self.esz
        if self.kind == RS:
            return self.rs_rows(t)[r] * row
        if self.kind == AG:
            return sum(self.dims[t]) * row
        if self.kind == BC:
            return 0 if (r == self.root and self.inplace) else self.dims[t]
        return sum(self.dims[t][p][r] for p in range(self.n)) * row

    def source(self, R, t, P):
        """(first output byte of rank R's tensor t that comes from rank P, its byte offset in P's input, bytes)."""
        row = self.rows[t] * self.esz
        if self.kind == RS:
            rows = self.rs_rows(t)
            return 0, sum(rows[:R]) * row, rows[R] * row
        if self.kind == AG:
            return sum(self.dims[t][:P]) * row, 0, self.dims[t][P] * row
        if self.kind == BC:
            return 0, 0, (self.dims[t] if P == self.root else 0)
        S = self.dims[t]
        return sum(S[p][R] for p in range(P)) * row, sum(S[P][:R]) * row, S[P][R] * row

    # --- the native call -----------------------------------------------------------------------------------------------
    def flat_dims(self):
        if self.kind in (RS, BC):
            return list(self.dims)
        if self.kind == AG:
            return [d for per in self.dims for d in per]
        return [d for S in self.dims for row in S for d in row]

    def plan(self, max_rows=1 << 18):
        n, T = self.n, self.T
        ins = [addr(IN, r, t) for r in range(n) for t in range(T)]
        outs = [addr(IN if (self.kind == BC and r == self.root and self.inplace) else OUT, r, t) for r in range(n) for t in range(T)]
        fd = self.flat_dims()
        dims = (ctypes.c_int64 * max(len(fd), 1))(*fd)
        rows = (ctypes.c_int64 * max(T, 1))(*self.rows)
        ip = (ctypes.c_uint64 * len(ins))(*ins)
        op = (ctypes.c_uint64 * len(outs))(*outs)
        nl = ctypes.c_int(-1)
        buf = np.zeros((max_rows, 6), dtype=np.int64)
        err = ctypes.create_string_buffer(512)
        m = lib().hvd_plan_collective(self.kind, n, T, dims, rows, ESZ_DTYPE[self.esz], SUM, self.root, ip, op, self.cap, self.ctas,
                                      ctypes.byref(nl), buf.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), max_rows, err, 512)
        return m, nl.value, buf[:max(m, 0)], err.value.decode()

    def __repr__(self):
        return 'Config(kind=%d, n=%d, T=%d, esz=%d, cap=%d, ctas=%d, root=%d, inplace=%s, rows=%s, dims=%s)' % (
            self.kind, self.n, self.T, self.esz, self.cap, self.ctas, self.root, self.inplace, self.rows[:8], str(self.dims)[:300])


def tile(starts, sizes, total, what):
    """Sorted ranges [starts[i], starts[i] + sizes[i]) must cover [0, total) exactly once."""
    if total == 0:
        assert starts.size == 0, what + ': bytes written into an empty output'
        return
    assert starts.size > 0, what + ': output never written'
    o = np.argsort(starts, kind='stable')
    s, z = starts[o], sizes[o]
    assert s[0] == 0, '%s: first written byte is %d' % (what, s[0])
    gaps = np.flatnonzero(s[1:] != s[:-1] + z[:-1])
    assert gaps.size == 0, '%s: range ending at %d followed by one at %d' % (what, s[gaps[0]] + z[gaps[0]], s[gaps[0] + 1])
    assert s[-1] + z[-1] == total, '%s: written up to %d of %d bytes' % (what, s[-1] + z[-1], total)


def verify(cfg):
    m, nlaunch, rows, err = cfg.plan()
    assert m >= 0, '%r: native plan failed (%d): %s' % (cfg, m, err)
    kind, rank, dst, src_rank, src, nbytes = rows.T
    assert (nbytes > 0).all(), '%r: empty range' % cfg
    assert nlaunch >= 0
    # packed input ranges lie inside the packing rank's own input (broadcast: only the root packs)
    pk = kind == 1
    io, r_, t_, off = decode(src[pk])
    assert (io == IN).all() and (r_ == rank[pk]).all(), cfg
    if cfg.kind == BC:
        assert (rank[pk] == cfg.root).all(), '%r: a rank other than the root packs' % cfg
    inb = np.array([[cfg.in_bytes(r, t) for t in range(cfg.T)] for r in range(cfg.n)], dtype=np.int64)
    assert (off + nbytes[pk] <= inb[r_, t_]).all(), '%r: a send reads past its input' % cfg
    # received ranges: decode both ends and compare with the independent source map
    rc = kind == 0
    dio, dr, dt, doff = decode(dst[rc])
    sio, sr, st, soff = decode(src[rc])
    b = nbytes[rc]
    assert (dio == OUT).all() and (dr == rank[rc]).all() and (sr == src_rank[rc]).all(), cfg
    assert (sio == IN).all() and (st == dt).all(), '%r: bytes of another tensor' % cfg
    n, T = cfg.n, cfg.T
    first = np.zeros((n, T, n), dtype=np.int64)
    sbase = np.zeros((n, T, n), dtype=np.int64)
    size = np.zeros((n, T, n), dtype=np.int64)
    for R in range(n):
        for t in range(T):
            for P in range(n):
                first[R, t, P], sbase[R, t, P], size[R, t, P] = cfg.source(R, t, P)
    lo = first[dr, dt, sr]
    assert (doff >= lo).all() and (doff + b <= lo + size[dr, dt, sr]).all(), '%r: bytes from the wrong rank' % cfg
    bad = np.flatnonzero(soff != sbase[dr, dt, sr] + (doff - lo))
    assert bad.size == 0, '%r: output byte %d of rank %d tensor %d reads byte %d of rank %d, expected %d' % (
        cfg, doff[bad[0]], dr[bad[0]], dt[bad[0]], soff[bad[0]], sr[bad[0]], sbase[dr, dt, sr][bad[0]] + doff[bad[0]] - lo[bad[0]])
    # coverage: reducescatter outputs once from every rank (one-shot reduce), the others once in all
    for R in range(n):
        for t in range(T):
            sel = (dr == R) & (dt == t)
            total = cfg.out_bytes(R, t)
            if cfg.kind == RS:
                for P in range(n):
                    s2 = sel & (sr == P)
                    tile(doff[s2], b[s2], total, '%r rank %d tensor %d from %d' % (cfg, R, t, P))
            else:
                tile(doff[sel], b[sel], total, '%r rank %d tensor %d' % (cfg, R, t))
    return nlaunch


def random_config(rng, i):
    kind = i % 4
    n = int(rng.integers(2, 9))
    esz = int(rng.choice([1, 2, 4, 8]))
    cap = 4096 * int(rng.choice([1, 1, 2, 3, 5, 16, 64]))
    ctas = int(rng.choice([1, 3, 8, 32, 128]))
    big = rng.random() < 0.03
    T = int(rng.integers(100, 201)) if big else int(rng.integers(1, 7))
    rows = [int(rng.integers(1, 8)) for _ in range(T)]

    def d0(t, spread=3.0):
        # 0, tiny, or up to `spread` times what fits the buffer
        u = rng.random()
        if u < 0.2:
            return 0
        if u < 0.5 or big:
            return int(rng.integers(1, 20))
        return int(rng.integers(0, int(spread * cap / (rows[t] * esz)) + 2))

    if kind == RS:
        dims = [d0(t) for t in range(T)]
    elif kind == AG:
        dims = [[d0(t, 1.5) for _ in range(n)] for t in range(T)]
    elif kind == BC:
        dims = [d0(t) * rows[t] * esz + int(rng.integers(0, 16)) * (rng.random() < 0.5) for t in range(T)]
    else:
        dims = []
        for t in range(T):
            S = [[d0(t, 1.0 / n * 3) for _ in range(n)] for _ in range(n)]
            if rng.random() < 0.3:
                z = int(rng.integers(0, n))
                for q in range(n):
                    S[z][q] = 0  # a rank that sends nothing
            if rng.random() < 0.3:
                z = int(rng.integers(0, n))
                for p in range(n):
                    S[p][z] = 0  # a rank that receives nothing
            dims.append(S)
    return Config(kind, n, dims, rows, esz, cap, ctas, root=i % n if kind == BC else -1, inplace=bool(rng.random() < 0.5))


def test_random_plans_agree_and_move_the_right_bytes():
    rng = np.random.default_rng(20261016)
    launches = {k: [] for k in (RS, AG, BC, A2A)}
    for i in range(3000):
        cfg = random_config(rng, i)
        launches[cfg.kind].append(verify(cfg))
    # the sweep reached the windowed / multi-launch paths of every op
    for k, v in launches.items():
        assert max(v) >= 3, (k, max(v))


@pytest.mark.parametrize('n', range(2, 9))
def test_broadcast_every_root(n):
    for root in range(n):
        for inplace in (False, True):
            for cap in (4096, 8192):
                cfg = Config(BC, n, [1, 13, 16 * 300 + 7, 0, 3 * cap + 5, 16], [1] * 6, 1, cap, 8, root=root, inplace=inplace)
                assert verify(cfg) >= 4


def test_windowed_paths():
    cap = 4096
    # allgather: a block of 2.5 caps runs alone in 3 windows, between two fused segments
    cfg = Config(AG, 4, [[5, 5, 5, 5], [0, 2 * cap + cap // 2, 1, 0], [7, 0, 0, 9]], [1, 1, 1], 1, cap, 8)
    assert verify(cfg) == 5
    # alltoall: blocks larger than cap / n take several launches, zeros in the split matrix included
    S = [[0, 3000, 0], [1, 0, 2], [0, 0, 0]]
    cfg = Config(A2A, 3, [S], [1], 1, cap, 8)
    assert verify(cfg) == 3  # win = 4096 / 3 rounded down to 16 = 1360 B; ceil(3000 / 1360) = 3
    # broadcast: 3 caps + 5 bytes
    assert verify(Config(BC, 2, [3 * cap + 5], [1], 1, cap, 8, root=1)) == 4
    # reducescatter: a tensor of several regions per destination, then small ones sharing the last launch
    assert verify(Config(RS, 4, [4 * 3000 + 3, 1, 3, 4], [1, 5, 1, 1000], 4, cap, 8)) >= 12


@pytest.mark.parametrize('kind,n,cap,dims', [
    (RS, 8, 1000, [64]),       # 1000 / 8 rounded down to 128 B: no region at all
    (RS, 5, 512, [5]),
    (A2A, 8, 100, [[[1] * 8] * 8]),  # 100 / 8 rounded down to 16 B: no window
    (AG, 2, 15, [[1, 1]]),
    (BC, 2, 8, [4]),
])
def test_no_plan_for_a_buffer_too_small(kind, n, cap, dims):
    """A buffer that leaves no room is an error, not an endless loop or a silently skipped tensor."""
    cfg = Config(kind, n, dims, [1] * len(dims), 4, cap, 8, root=0 if kind == BC else -1)
    m, _, _, err = cfg.plan()
    assert m == -5 and 'bytes' in err, (m, err)


def test_nothing_to_move_is_no_launch():
    for kind, dims in ((RS, [0]), (AG, [[0, 0, 0]]), (BC, [0]), (A2A, [[[0] * 3] * 3])):
        assert verify(Config(kind, 3, dims, [2], 4, 4096, 8, root=0 if kind == BC else -1)) == 0


@pytest.mark.parametrize('L', [2, 3, 4, 8])
def test_hierarchical_windows(L):
    """The two intra-host halves of the hierarchical allreduce: the reducescatter of the fusion buffer (L blocks of B bytes,
    B a multiple of 128) into the shard, and the allgather of the shard back into every block, in windows of the buffer."""
    for esz in (2, 4):
        for B in (128, 128 * 37, 3 * 4096 + 5 * 128):
            for cap in (128 * L, 4096, 3 * 4096, 1 << 20):
                region = cap // L // 128 * 128
                assert verify(Config(RS, L, [L * B // esz], [1], esz, cap, 128)) == -(-B // region)
                window = cap // 16 * 16
                assert verify(Config(AG, L, [[B] * L], [1], 1, cap, 128)) == -(-B // window)


# --- allreduce ---------------------------------------------------------------------------------------------------------
LAUNCH_FIELDS = ('reduce', 'variant', 'ctas', 'total_bytes', 'reduce_lo', 'reduce_hi', 'dtype', 'wire_dtype', 'op', 'prescale',
                 'postscale', 'inline', 'nout', 'oneshot_nvls', 'ndesc')


def plan_allreduce(c, max_launches=1024, max_descs=4096):
    """One rank's allreduce plan for a golden case's inputs, as one dict per launch with the golden's fields."""
    T = len(c['counts'])
    launches = np.zeros((max_launches, len(LAUNCH_FIELDS)), dtype=np.int64)
    descs = np.zeros((max_descs, 4), dtype=np.int64)
    err = ctypes.create_string_buffer(512)
    m = lib().hvd_plan_allreduce(
        c['n'], T, (ctypes.c_int64 * T)(*c['counts']), (ctypes.c_uint64 * T)(*c['ins']), (ctypes.c_uint64 * T)(*c['outs']),
        c['dtype'], c['wire'], c['op'], c['prescale'], c['postscale'], c['variant'].encode(), c['oneshot_max_bytes'],
        c['multicast'], c['nvls_min_bytes'], c['cap'], c['comm_ctas'], c['large_msg_ctas'],
        launches.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), max_launches,
        descs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), max_descs, err, 512)
    assert m >= 0, (m, err.value.decode())
    out, d = [], 0
    for row in launches[:m]:
        f = dict(zip(LAUNCH_FIELDS, (int(v) for v in row)))
        f['prescale'], f['postscale'] = (float(v) for v in row[9:11].view(np.float64))
        f['descs'] = descs[d:d + f['ndesc']].tolist()
        d += f['ndesc']
        out.append(f)
    return out


def test_allreduce_plans_match_the_golden():
    """Segments, variant, grid, arguments, inline or staged descriptors and every descriptor of each launch, over n = 2 / 4 / 8,
    fp32 / bf16 / fp16 / int32 and an fp32 -> bf16 wire, SUM / AVERAGE / MIN, every HVD_ALLREDUCE_VARIANT, with and without
    multicast, both sides of both crossovers, the four CtasFor bands, buffers that split pieces, zero-count pieces and more
    pieces than kInlineDescs."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'allreduce_plans.json')) as f:
        golden = json.load(f)
    assert len(golden['cases']) > 100
    for case in golden['cases']:
        c = dict(zip(golden['inputs'], case))
        launches = [dict(zip(golden['launch'], l)) for l in case[len(golden['inputs'])]]
        got = plan_allreduce(c)
        what = {k: v for k, v in c.items() if k not in ('ins', 'outs')}
        assert len(got) == len(launches), (what, len(got), len(launches))
        for k, (g, want) in enumerate(zip(got, launches)):
            assert g['reduce'] == 1 and g['ndesc'] == len(want['descs']), (what, k, g)
            for field, v in want.items():
                assert g[field] == v, (what, k, field, g[field], v)


def test_allreduce_needs_128_bytes_of_buffer():
    c = dict(n=2, counts=[64], ins=[1 << 32], outs=[1 << 33], dtype=7, wire=7, op=SUM, prescale=1.0, postscale=1.0, variant='auto',
             oneshot_max_bytes=0, multicast=0, nvls_min_bytes=0, cap=127, comm_ctas=8, large_msg_ctas=8)
    with pytest.raises(AssertionError, match='-5.*bytes'):
        plan_allreduce(c)
    assert len(plan_allreduce(dict(c, cap=128))) == 2
