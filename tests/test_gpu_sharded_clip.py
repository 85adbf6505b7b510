"""Global-norm gradient clipping and AMP loss scaling for sharded optimizer state: the one-pass gradient statistics kernel
against an fp64 reference, the fused updates' device-side gradient scale, and opt.clip_grad_norm_ / hvd.ShardedGradScaler
on 4 simulated ranks (csrc/common/sim_api.cc) against plain torch on averaged gradients; with >= 2 GPUs, across real
ranks."""
import copy
import math
import warnings

import pytest
import torch

from conftest import run_parallel
from optim_cases import SIZES, hvd, ngpu  # noqa: F401  (hvd: fixture)
from sim_ranks import ConvNetWithUnused, batch, reduced_grads, sharded_team, team  # noqa: F401  (team: fixture)

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.bfloat16, torch.float16]


# ---- the statistics kernel ---------------------------------------------------------------------------------------------
def _views(dtype, seed, offset):
    """Views at element offset `offset` of slightly larger buffers: the sizes above plus ~200 small tensors in one table."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    sizes = SIZES + [int(x) for x in torch.randint(1, 3000, (200,), generator=torch.Generator().manual_seed(seed))]
    bufs = [(torch.randn(n + offset + 5, device='cuda', generator=g) * 3).to(dtype) for n in sizes]
    return bufs, [b[offset:offset + n] for b, n in zip(bufs, sizes)]


def _ref(views):
    v = torch.cat([x.double().reshape(-1) for x in views])
    return float(v.square().sum()), float(v.abs().max()), float(not bool(torch.isfinite(v).all()))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_stats_kernel_matches_fp64(hvd, dtype, offset):
    from horovod_b200 import ops
    bufs, views = _views(dtype, 7 + offset, offset)
    sum_sq, max_abs, flag = _ref(views)
    for norm_type in (2.0, math.inf):
        outs = []
        for _ in range(2):
            out = torch.zeros(2, device='cuda')
            ops.grad_shard_stats(views, out, norm_type=norm_type)
            outs.append(out.cpu())
        assert torch.equal(outs[0], outs[1]), 'not deterministic'
        if norm_type == 2.0:
            assert abs(float(outs[0][0]) - sum_sq) <= 1e-6 * sum_sq, (float(outs[0][0]), sum_sq)
        else:
            assert float(outs[0][0]) == max_abs
        assert float(outs[0][1]) == flag == 0.0
    # in-place unscale: every element becomes (g.float() * s) rounded to its dtype, the slack stays as it was
    s = torch.tensor([0.3719], device='cuda')
    before = [b.clone() for b in bufs]
    expect = [(v.float() * s).to(dtype) for v in views]
    out = torch.zeros(2, device='cuda')
    ops.grad_shard_stats(views, out, inv_scale=s)
    for b, b0, v, e in zip(bufs, before, views, expect):
        assert torch.equal(v, e)
        assert torch.equal(b[:offset], b0[:offset]) and torch.equal(b[offset + v.numel():], b0[offset + v.numel():])
    ref = _ref(expect)[0]
    assert abs(float(out[0]) - ref) <= 1e-6 * ref and float(out[1]) == 0.0


@pytest.mark.parametrize("dtype", DTYPES)
def test_stats_kernel_flags_inf_and_nan(hvd, dtype):
    from horovod_b200 import ops
    for bad in (math.inf, -math.inf, math.nan):
        for where in (0, -1):
            for k in (0, 5, len(SIZES) - 1):  # the first, a middle (4097) and the largest tensor of the table
                _, views = _views(dtype, 3, 1)
                views[k].reshape(-1)[where] = bad
                for norm_type in (2.0, math.inf):
                    for inv in (None, torch.tensor([0.5], device='cuda')):
                        out = torch.zeros(2, device='cuda')
                        ops.grad_shard_stats(views, out, inv_scale=inv, norm_type=norm_type)
                        o = out.cpu()
                        assert float(o[1]) == 1.0, (bad, where, k, norm_type)
                        if math.isnan(bad):
                            assert math.isnan(float(o[0]))
                        else:
                            assert float(o[0]) == math.inf


def test_stats_kernel_accumulates_over_dtypes(hvd):
    """Several launches (one per dtype) accumulate into one output; an empty list or empty tensors change nothing."""
    from horovod_b200 import ops
    views = []
    for i, dt in enumerate(DTYPES):
        views += _views(dt, 11 + i, i)[1][:20]
    out = torch.zeros(2, device='cuda')
    ops.grad_shard_stats(views + [torch.empty(0, device='cuda')], out)
    ref = _ref(views)[0]
    assert abs(float(out[0]) - ref) <= 1e-6 * ref and float(out[1]) == 0.0
    mx = torch.zeros(2, device='cuda')
    ops.grad_shard_stats(views, mx, norm_type='inf')
    assert float(mx[0]) == _ref(views)[1]
    same = out.clone()
    ops.grad_shard_stats([], same)
    assert torch.equal(same, out)


def test_stats_kernel_rejects_bad_arguments(hvd):
    from horovod_b200 import ops
    g = [torch.randn(100, device='cuda')]
    out = torch.zeros(2, device='cuda')
    with pytest.raises(ValueError):
        ops.grad_shard_stats(g, out, norm_type=1.0)
    for bad_out in (torch.zeros(1, device='cuda'), torch.zeros(2, device='cuda', dtype=torch.float64), torch.zeros(2)):
        with pytest.raises(RuntimeError):
            ops.grad_shard_stats(g, bad_out)
    for bad_inv in (torch.ones(1, device='cuda', dtype=torch.float16), torch.ones(1), torch.ones(2, device='cuda')):
        with pytest.raises(RuntimeError):
            ops.grad_shard_stats(g, out, inv_scale=bad_inv)
    with pytest.raises(RuntimeError):
        ops.grad_shard_stats([torch.ones(10, device='cuda', dtype=torch.float64)], out)


# ---- the fused updates' device-side gradient scale ----------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["sgd", "adamw"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_fused_update_grad_scale_dev_is_bit_identical(hvd, kind, dtype):
    from horovod_b200 import ops
    torch.manual_seed(5)
    sizes = [1, 4097, 1 << 16]
    p0 = [torch.randn(n, device='cuda').to(dtype) for n in sizes]
    g = [torch.randn(n, device='cuda').to(dtype) for n in sizes]
    factor = 0.3719

    def run(grad_scale, **kw):
        p = [x.clone() for x in p0]
        if kind == 'sgd':
            m = [torch.zeros_like(x) for x in p]
            for step in range(3):
                ops.fused_sgd_step(p, g, m, 0.1, momentum=0.9, weight_decay=1e-3, nesterov=True, grad_scale=grad_scale,
                                   first_step=step == 0, **kw)
            return p + m
        m = [torch.zeros_like(x, dtype=torch.float32) for x in p]
        v = [torch.zeros_like(x, dtype=torch.float32) for x in p]
        for step in range(1, 4):
            ops.fused_adam_step(p, g, m, v, 1e-2, weight_decay=0.05, step=step, grad_scale=grad_scale, **kw)
        return p + m + v

    host = run(factor)
    dev = run(1.0, grad_scale_dev=torch.tensor(factor, device='cuda'))
    both = run(2.0, grad_scale_dev=torch.tensor([factor / 2], device='cuda'))  # 2 * (factor / 2) is exact
    plain, none = run(1.0), run(1.0, grad_scale_dev=None)
    for a, b, c in zip(host, dev, both):
        assert torch.equal(a, b) and torch.equal(a, c)
    for a, b in zip(plain, none):
        assert torch.equal(a, b)
    assert not all(torch.equal(a, b) for a, b in zip(host, plain))


def test_fused_update_rejects_bad_grad_scale_dev(hvd):
    from horovod_b200 import ops
    p, g = [torch.zeros(8, device='cuda')], [torch.ones(8, device='cuda')]
    m, v = [torch.zeros(8, device='cuda')], [torch.zeros(8, device='cuda')]
    for bad in (torch.ones(1, device='cuda', dtype=torch.float64), torch.ones(1), torch.ones(2, device='cuda'),
                torch.ones(0, device='cuda')):
        with pytest.raises(RuntimeError):
            ops.fused_sgd_step(p, g, [], 0.1, grad_scale_dev=bad)
        with pytest.raises(RuntimeError):
            ops.fused_adam_step(p, g, m, v, 0.1, grad_scale_dev=bad)
    assert torch.equal(p[0], torch.zeros(8, device='cuda'))


# ---- simulated ranks ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["adamw", "sgd"])
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("norm_type", [2.0, math.inf])
def test_clip_grad_norm_on_simulated_ranks(hvd, team, kind, dt, norm_type):
    """opt.clip_grad_norm_ on 4 simulated ranks against torch.nn.utils.clip_grad_norm_ on averaged gradients, with the
    clip active on even steps only; in step 2 no rank uses one layer, so clip_grad_norm_ itself reduces those buckets."""
    n = team.n
    torch.manual_seed(0)
    base = ConvNetWithUnused().cuda()

    def make(m):
        if kind == 'adamw':
            # eps well above the smallest gradients: Adam then feels the clip coefficient, and a gradient element near
            # zero whose sign differs between the bf16 run and the fp32 reference moves its parameter by << lr
            return torch.optim.AdamW(m.parameters(), lr=1e-2, eps=1e-3, weight_decay=0.05)
        return torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-4)

    models, opts = sharded_team(hvd, team, copy.deepcopy(base).to(dtype=dt, memory_format=torch.channels_last), make, dt,
                                min_buckets=3)
    ref = copy.deepcopy(base).to(memory_format=torch.channels_last)
    ref_opt = make(ref)
    tol = dict(rtol=1e-4, atol=1e-5) if dt == torch.float32 else dict(rtol=5e-2, atol=1e-2)
    for step in range(8):
        use = step != 2
        grads = [torch.zeros_like(p) for p in ref.parameters()]
        for r in range(n):
            x, y = batch(step, r)
            ref.zero_grad()
            torch.nn.functional.cross_entropy(ref(x, use), y).backward()
            for g, p in zip(grads, ref.parameters()):
                if p.grad is not None:
                    g += p.grad
        for g, p in zip(grads, ref.parameters()):
            p.grad = g / n
        unclipped = float(torch.nn.utils.get_total_norm([p.grad for p in ref.parameters()], norm_type))
        max_norm = unclipped * (0.5 if step % 2 == 0 else 2.0)
        torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm, norm_type)
        ref_opt.step()

        for r in range(n):
            opts[r].zero_grad()
            x, y = batch(step, r)
            torch.nn.functional.cross_entropy(models[r](x.to(dt), use), y).backward()
        if step == 1:
            with pytest.raises(AssertionError):
                opts[0].zero_grad()  # reduce-scatters may be in flight
        mark = len(team.log)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter('always')
            norms = team.run(lambda r: opts[r].clip_grad_norm_(max_norm, norm_type=norm_type))
            assert team.count('ar', mark) == n and team.count('ag', mark) == 0
            # step 2: the buckets from the unused layer's on were not launched by hooks, clip_grad_norm_ reduces them
            assert (team.count('rs', mark) > 0) == (step == 2)
            reduced = [g.float() for g in reduced_grads(opts, list(models[0].parameters()))]
            mark = len(team.log)
            team.run(lambda r: opts[r].step())
            assert team.count('rs', mark) == 0, 'step() reduced a second time'
            assert team.count('ag', mark) == n * len(opts[0]._buckets)
        assert not [x for x in w if 'horovod_b200' in x.filename], [str(x.message) for x in w]
        # the norm: 0-dim fp32, the same bits on every rank, torch's on the averaged gradients the update saw
        assert norms[0].dim() == 0 and norms[0].dtype == torch.float32 and norms[0].is_cuda
        assert all(torch.equal(t, norms[0]) for t in norms)
        want = float(torch.nn.utils.get_total_norm(reduced, norm_type))
        assert abs(float(norms[0]) - want) <= 1e-5 * want, (step, float(norms[0]), want)
        if dt == torch.float32:
            assert abs(float(norms[0]) - unclipped) <= 1e-4 * unclipped
        for r in range(n):
            for (name, a), b in zip(models[r].named_parameters(), ref.parameters()):
                torch.testing.assert_close(a.float(), b, **tol, msg=lambda m: '%s step %d rank %d: %s' % (name, step, r, m))
                assert torch.equal(a, dict(models[0].named_parameters())[name])


def test_clip_grad_norm_rejections(hvd, team):
    torch.manual_seed(0)
    base = ConvNetWithUnused().cuda()
    models, opts = sharded_team(hvd, team, copy.deepcopy(base).to(memory_format=torch.channels_last),
                                lambda m: torch.optim.AdamW(m.parameters(), lr=1e-2), min_buckets=3)
    for bad in (1.0, 0.0, 3.0, -math.inf):
        with pytest.raises(ValueError):
            opts[0].clip_grad_norm_(1.0, norm_type=bad)
    for r in range(team.n):
        x, y = batch(0, r)
        torch.nn.functional.cross_entropy(models[r](x), y).backward()
    with pytest.raises(AssertionError):
        opts[0].zero_grad()  # between backward and clip: the reduce-scatters may still read the gradients
    team.run(lambda r: opts[r].clip_grad_norm_(1.0))
    team.run(lambda r: opts[r].step())


def test_sharded_grad_scaler_on_simulated_ranks(hvd, team):
    """fp16 model + AdamW + ShardedGradScaler on 4 simulated ranks.  In step 2 only rank 0's LOCAL gradient holds an inf,
    at a position rank 2 owns: every rank must skip and back off alike.  The other steps follow torch.amp.GradScaler on
    averaged gradients; unscale_ + clip_grad_norm_ + step cost one stats pass and one stats allreduce per rank."""
    from horovod_b200.ops import kernel_launches
    from horovod_b200.torch.grad_buckets import shard_range, shard_slices
    n = team.n
    torch.manual_seed(0)
    base = ConvNetWithUnused().cuda()

    def make(m):
        return torch.optim.AdamW(m.parameters(), lr=1e-2, eps=1e-3, weight_decay=0.05)  # eps: see the clip test

    models, opts = sharded_team(hvd, team, copy.deepcopy(base).to(dtype=torch.float16, memory_format=torch.channels_last),
                                make, torch.float16, min_buckets=3)
    scalers = [hvd.ShardedGradScaler('cuda', init_scale=256.0) for _ in range(n)]
    ref = copy.deepcopy(base).to(memory_format=torch.channels_last)
    ref_opt = make(ref)
    ref_scaler = torch.amp.GradScaler('cuda', init_scale=256.0)
    tol = dict(rtol=2e-2, atol=2e-3)
    # the poisoned element: the first parameter element inside rank 2's shard of bucket 0
    b0 = opts[0]._buckets[0]
    k, plo, _, slo = shard_slices(b0, 2)[0]
    pos = shard_range(b0, 2)[0] + slo
    pname = {id(p): name for name, p in models[0].named_parameters()}[id(b0['params'][k])]
    for step in range(6):
        grads = [torch.zeros_like(p) for p in ref.parameters()]
        for r in range(n):
            x, y = batch(step, r)
            ref.zero_grad()
            ref_scaler.scale(torch.nn.functional.cross_entropy(ref(x), y)).backward()
            for g, p in zip(grads, ref.parameters()):
                g += p.grad
        for g, (name, p) in zip(grads, ref.named_parameters()):
            p.grad = g / n
            if step == 2 and name == pname:
                p.grad.as_strided((p.numel(),), (1,), p.grad.storage_offset())[plo] = math.inf  # bucket order
        ref_scaler.unscale_(ref_opt)
        max_norm = 1.0 if step == 2 else 0.5 * float(torch.nn.utils.get_total_norm([p.grad for p in ref.parameters()]))
        torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
        ref_scaler.step(ref_opt)
        ref_scaler.update()

        for r in range(n):
            opts[r].zero_grad()
            x, y = batch(step, r)
            scalers[r].scale(torch.nn.functional.cross_entropy(models[r](x.half()), y)).backward()
        if step == 2:
            opts[0]._buckets[0]['gflat'][pos] = math.inf  # rank 0's local gradient; the reduce-scatter is still queued
        mark, launches = len(team.log), kernel_launches()
        sim0 = team.sim_launches

        def body(r):
            scalers[r].unscale_(opts[r])
            norm = opts[r].clip_grad_norm_(max_norm)
            scalers[r].step(opts[r])
            scalers[r].update()
            return norm
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter('always')
            team.run(body)
        assert not [x for x in w if 'horovod_b200' in x.filename], [str(x.message) for x in w]
        assert team.count('rs', mark) == 0 and team.count('ar', mark) == n
        own = kernel_launches() - launches - (team.sim_launches - sim0)
        assert own == (n if step == 2 else 2 * n), (step, own)  # stats (+ fused update unless skipped), per rank
        scales = [s.get_scale() for s in scalers]
        assert len(set(scales)) == 1 and scales[0] == ref_scaler.get_scale(), (step, scales, ref_scaler.get_scale())
        if step == 2:
            assert scales[0] == 128.0
        for r in range(n):
            for (name, a), b in zip(models[r].named_parameters(), ref.parameters()):
                torch.testing.assert_close(a.float(), b, **tol, msg=lambda m: '%s step %d rank %d: %s' % (name, step, r, m))
                assert torch.equal(a, dict(models[0].named_parameters())[name])


def test_sharded_grad_scaler_defers_to_torch_for_other_optimizers(hvd):
    torch.manual_seed(3)
    base = torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 8)).cuda()
    runs = []
    for cls in (torch.amp.GradScaler, hvd.ShardedGradScaler):
        m = copy.deepcopy(base)
        opt = torch.optim.AdamW(m.parameters(), lr=1e-2)
        scaler = cls('cuda', init_scale=1024.0)
        for i in range(5):
            g = torch.Generator(device='cuda').manual_seed(i)
            x = torch.randn(16, 32, device='cuda', generator=g)
            opt.zero_grad()
            with torch.autocast('cuda', dtype=torch.float16):
                loss = m(x).float().square().mean()
            scaler.scale(loss).backward()
            if i == 2:
                m[0].weight.grad[0, 0] = math.inf
            scaler.unscale_(opt)
            torch.nn.utils.clip_grad_norm_(m.parameters(), 0.5)
            scaler.step(opt)
            scaler.update()
        runs.append(([p.detach().clone() for p in m.parameters()], scaler.get_scale()))
    assert runs[0][1] == runs[1][1] == 512.0
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))


@pytest.mark.skipif(ngpu() < 2, reason="needs >= 2 GPUs")
def test_sharded_clip_across_ranks(native_built):
    n = 2 if ngpu() < 4 else 4
    rc, out = run_parallel("sharded_clip_worker.py", np=n, timeout=420)
    assert "SHARDED CLIP OK" in out, out[-4000:]
