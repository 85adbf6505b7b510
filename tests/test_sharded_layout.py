"""Layout of the sharded optimizer state (ZeRO-1) on the CPU: bucket padding, shard ranges, shard-to-parameter slices
and the round trip between a full per-parameter state and N shards."""
import pytest
import torch

from horovod_b200.torch.grad_buckets import full_from_shards, shard_from_full, shard_layout, shard_range, shard_slices

GROUPS = [[(1000, torch.float32), (7, torch.float32), (33, torch.bfloat16), (40000, torch.float32), (1, torch.bfloat16)],
          [(5, torch.float32), (129, torch.float16)]]


@pytest.mark.parametrize("n", [2, 4, 8])
def test_buckets_are_padded_and_aligned(n):
    buckets = shard_layout(GROUPS, n, cap_bytes=64 * 1024)
    assert {(b['group'], b['dtype']) for b in buckets} == {(0, torch.float32), (0, torch.bfloat16), (1, torch.float32), (1, torch.float16)}
    seen = set()
    for b in buckets:
        item = torch.empty(0, dtype=b['dtype']).element_size()
        assert (b['numel'] * item) % (n * 128) == 0
        assert b['shard'] * n == b['numel'] and (b['shard'] * item) % 128 == 0
        end = 0
        for i, off, numel in b['members']:
            assert GROUPS[b['group']][i] == (numel, b['dtype'])
            assert (off * item) % 128 == 0 and off >= end
            end = off + numel
            seen.add((b['group'], i))
        assert end <= b['numel']
    assert seen == {(g, i) for g in range(len(GROUPS)) for i in range(len(GROUPS[g]))}


def test_bucket_cap_and_reverse_order():
    buckets = shard_layout([[(1024, torch.float32)] * 4], 2, cap_bytes=2 * 4096)
    assert [[m[0] for m in b['members']] for b in buckets] == [[3, 2], [1, 0]]
    big = shard_layout([[(10, torch.float32), (100000, torch.float32)]], 2, cap_bytes=4096)
    assert [[m[0] for m in b['members']] for b in big] == [[1], [0]]


@pytest.mark.parametrize("n", [2, 4, 8])
def test_shard_ranges_and_slices_cover_every_element_once(n):
    for b in shard_layout(GROUPS, n, cap_bytes=64 * 1024):
        ranges = [shard_range(b, r) for r in range(n)]
        assert ranges[0][0] == 0 and ranges[-1][1] == b['numel']
        assert all(ranges[r][1] == ranges[r + 1][0] for r in range(n - 1))
        covered = {k: torch.zeros(numel, dtype=torch.int32) for k, (_, _, numel) in enumerate(b['members'])}
        for r in range(n):
            lo, hi = ranges[r]
            for k, plo, phi, slo in shard_slices(b, r):
                _, off, numel = b['members'][k]
                assert 0 <= plo < phi <= numel and 0 <= slo and slo + phi - plo <= hi - lo
                assert lo + slo == off + plo  # the shard element and the bucket element are the same
                covered[k][plo:phi] += 1
        assert all(bool((c == 1).all()) for c in covered.values())


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("kind", ["adam", "sgd"])
def test_state_round_trip(n, kind):
    torch.manual_seed(n)
    shapes = [(10, 100), (7,), (3, 11), (200, 200), (1,)]
    params = [torch.nn.Parameter(torch.randn(s)) for s in shapes]
    opt = torch.optim.Adam(params, lr=0.1) if kind == "adam" else torch.optim.SGD(params, lr=0.1, momentum=0.9)
    for _ in range(2):
        for p in params:
            p.grad = torch.randn_like(p)
        opt.step()
    keys = ['exp_avg', 'exp_avg_sq'] if kind == "adam" else ['momentum_buffer']
    buckets = shard_layout([[(p.numel(), p.dtype) for p in params]], n, cap_bytes=16 * 1024)
    for b in buckets:
        ps = [params[i] for i, _, _ in b['members']]
        for key in keys:
            full = [opt.state[p][key] for p in ps]
            shards = [shard_from_full(b, r, full) for r in range(n)]
            assert all(s.numel() == b['shard'] for s in shards)
            back = full_from_shards(b, shards, [p.shape for p in ps])
            for t, ref in zip(back, full):
                assert torch.equal(t, ref)
            # padding is zero and a missing state is zeros
            assert float(sum(s.abs().sum() for s in shards)) == pytest.approx(float(sum(t.abs().sum() for t in full)), rel=1e-5)
            none = [shard_from_full(b, r, [None] * len(ps)) for r in range(n)]
            assert all(float(s.abs().sum()) == 0.0 for s in none)


@pytest.mark.parametrize("n", [2, 4])
def test_state_round_trip_keeps_memory_format(n):
    """A channels_last parameter lies in the bucket in memory order: its state round-trips with the same strides."""
    w = torch.randn(6, 5, 3, 3).contiguous(memory_format=torch.channels_last)
    b = shard_layout([[(w.numel(), w.dtype), (7, w.dtype)]], n, cap_bytes=1 << 20)[0]
    full = [w if i == 0 else torch.arange(7.0) for i, _, _ in b['members']]
    strides = [w.stride() if i == 0 else (1,) for i, _, _ in b['members']]
    shapes = [w.shape if i == 0 else (7,) for i, _, _ in b['members']]
    shards = [shard_from_full(b, r, full, strides) for r in range(n)]
    flat = torch.cat(shards)
    k = [i for i, _, _ in b['members']].index(0)
    off = b['members'][k][1]
    assert torch.equal(flat[off:off + w.numel()], w.as_strided((w.numel(),), (1,)))  # memory order, not logical order
    back = full_from_shards(b, shards, shapes, strides)
    assert torch.equal(back[k], w) and back[k].is_contiguous(memory_format=torch.channels_last)


def test_factory_rejects_unsupported_configurations_before_any_collective():
    """Argument checks of shard_optimizer_state=True that need no GPU: an optimizer other than SGD / Adam / AdamW."""
    from horovod_b200.torch.sharded_optimizer import _ShardedDistributedOptimizer
    from horovod_b200.torch.compression import Compression
    p = torch.nn.Parameter(torch.randn(4))
    base = torch.optim.RMSprop([p], lr=0.1)
    cls = type('RMSprop', (_ShardedDistributedOptimizer, torch.optim.RMSprop), {})
    with pytest.raises(ValueError, match='SGD, Adam and AdamW'):
        cls(base.param_groups, None, Compression.none)
    adam = torch.optim.Adam([p], lr=0.1, amsgrad=True)
    cls = type('Adam', (_ShardedDistributedOptimizer, torch.optim.Adam), {})
    with pytest.raises(ValueError, match='amsgrad'):
        cls(adam.param_groups, None, Compression.none)
    sgd = torch.optim.SGD([p], lr=0.1)
    cls = type('SGD', (_ShardedDistributedOptimizer, torch.optim.SGD), {})
    from horovod_b200.torch.mpi_ops import Max
    with pytest.raises(ValueError, match='Average or op=Sum'):
        cls(sgd.param_groups, None, Compression.none, op=Max)
    with pytest.raises(ValueError, match='compression'):
        cls(sgd.param_groups, None, Compression.fp16)
    with pytest.raises(ValueError, match='dense CUDA'):
        cls(sgd.param_groups, None, Compression.none)  # a CPU parameter
    with pytest.raises(ValueError, match='unique'):
        cls(sgd.param_groups, [('w', p), ('w', p)], Compression.none)
