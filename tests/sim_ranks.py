"""Simulated ranks for the GPU optimizer tests: N ranks of hvd.DistributedOptimizer in one process on one GPU, whose
collectives run on the real kernels as simulated launches over the N ranks' buffers (csrc/common/sim_api.cc), and the
models, batches and steps the sharded (ZeRO-1) tests drive them with.  A test module imports the fixtures `team` and
`gteam` by name, together with `hvd` from optim_cases; the asserts here carry their own messages, as pytest rewrites
asserts in test modules only."""
import copy
import threading

import pytest
import torch

from optim_cases import same


class FakeSet:
    """Process set of one simulated rank."""
    process_set_id = 0

    def __init__(self, n, r):
        self.n, self.r = n, r

    def size(self):
        return self.n

    def rank(self):
        return self.r

    def included(self):
        return True


class SimTeam:
    """N simulated ranks of the sharded optimizer in one process.  Every rank's captured collectives are queued and run by
    the real kernels as one simulated launch over the N ranks' buffers: by flush(), or, while run() drives the ranks in
    one thread each, as soon as every rank issued its next collective (a barrier, as the kernels' flags are on real
    GPUs), so that what a rank does after a collective sees its result.  `log` keeps (kind, rank) of every call,
    `sim_launches` counts the kernels the simulated launches took, and `opts` are the ranks' optimizers (for the
    gather of state_dict())."""

    def __init__(self, n):
        from horovod_b200.torch import mpi_ops
        self.n, self.queues, self.mpi_ops, self.log = n, [[] for _ in range(n)], mpi_ops, []
        self.opts = []
        self.lockstep = False
        self.sim_launches = 0
        self._barrier = threading.Barrier(n, action=self.flush)

    def _issue(self, r, kind, tensor, arg):
        self.queues[r].append((kind, tensor, arg))
        self.log.append((kind, r))
        if self.lockstep:
            self._barrier.wait(timeout=120)

    def reducescatter(self, tensor, op, prescale_factor, postscale_factor, process_set, max_ctas=0):
        scale = prescale_factor * postscale_factor / (self.n if op == self.mpi_ops.Average else 1)
        self._issue(process_set.r, 'rs', tensor, scale)

    def allgather(self, tensor, process_set, max_ctas=0):
        self._issue(process_set.r, 'ag', tensor, 1.0)

    def allreduce(self, tensor, op=1, prescale_factor=1.0, postscale_factor=1.0, process_set=None, max_ctas=0):
        assert prescale_factor == postscale_factor == 1.0 and op in (self.mpi_ops.Sum, self.mpi_ops.Max), \
            ('an allreduce other than an unscaled Sum or Max', op, prescale_factor, postscale_factor)
        self._issue(process_set.r, 'ar', tensor, op)
        return tensor

    def _launch(self, kind, ts, arg):
        from horovod_b200.ops import sim
        if kind == 'rs':
            sim.inplace_reducescatter(ts, op=sim.SUM, scale=arg)
        elif kind == 'ag':
            sim.inplace_allgather(ts)
        elif kind == 'ars':
            sim.inplace_allreduce(ts, op=sim.SUM, scale=arg)
        else:
            sim.inplace_allreduce(ts, op=sim.SUM if arg == self.mpi_ops.Sum else sim.MAX)

    def flush(self):
        from horovod_b200.ops import kernel_launches
        torch.cuda.synchronize()
        before = kernel_launches()
        assert len({len(q) for q in self.queues}) == 1, 'ranks issued different numbers of collectives'
        for calls in zip(*self.queues):
            assert len({(c[0], c[1].numel(), c[1].dtype, c[2]) for c in calls}) == 1, 'ranks issued different collectives'
            self._launch(calls[0][0], [c[1] for c in calls], calls[0][2])
        torch.cuda.synchronize()
        self.sim_launches += kernel_launches() - before
        self.queues = [[] for _ in range(self.n)]

    def run(self, fn):
        """fn(rank) on every rank at once, one thread per rank; returns the results in rank order."""
        self.flush()
        self.lockstep = True
        res, errs = [None] * self.n, []

        def body(r):
            try:
                res[r] = fn(r)
            except BaseException as e:  # noqa: B036  re-raised below
                errs.append(e)
                self._barrier.abort()
        ths = [threading.Thread(target=body, args=(r,)) for r in range(self.n)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        self.lockstep = False
        self._barrier.reset()
        if errs:
            raise errs[0]
        torch.cuda.synchronize()
        return res

    def count(self, kind, since):
        return sum(1 for k, _ in self.log[since:] if k == kind)


class GraphTeam(SimTeam):
    """SimTeam with capturable stand-ins.  A collective issued while a CUDA graph is being captured records, inside the
    graph, a copy of its tensor into a staging tensor of its own; after every rank replayed its graph, reduce_captured()
    runs the recorded collectives on the ranks' staging copies with the same simulation kernels as flush() and copies
    the results back into the tensors, which is what the in-place kernel would have left there.  Eager collectives are
    queued as in SimTeam; the gradient allreduce (op Average / Sum with scale factors) is supported as well."""

    def __init__(self, n):
        super().__init__(n)
        self.captured = [[] for _ in range(n)]  # per rank: [kind, tensor, staging, arg, issued from the comm capture]
        self.graph_runs = 0
        self._graph_barrier = threading.Barrier(n, action=self.reduce_captured)

    def _issue(self, r, kind, tensor, arg):
        if not torch.cuda.is_current_stream_capturing():
            return super()._issue(r, kind, tensor, arg)
        staging = torch.empty_like(tensor)
        staging.copy_(tensor)
        self.captured[r].append((kind, tensor, staging, arg, self.opts[r]._graph_capture is not None))
        self.log.append(('captured-' + kind, r))

    def allreduce(self, tensor, op=1, prescale_factor=1.0, postscale_factor=1.0, process_set=None, max_ctas=0):
        if op == self.mpi_ops.Average or (op == self.mpi_ops.Sum and (prescale_factor != 1.0 or postscale_factor != 1.0)):
            scale = prescale_factor * postscale_factor / (self.n if op == self.mpi_ops.Average else 1)
            self._issue(process_set.r, 'ars', tensor, scale)
            return tensor
        return super().allreduce(tensor, op, prescale_factor, postscale_factor, process_set)

    def allreduce_async_(self, tensor, name=None, op=0, prescale_factor=1.0, postscale_factor=1.0, process_set=None):
        """The unsharded optimizer's eager bucket allreduce; synchronize() of its handle is a no-op."""
        self.allreduce(tensor, op, prescale_factor, postscale_factor, process_set)
        return ('sim', name)

    def reduce_captured(self):
        torch.cuda.synchronize()
        assert len({len(c) for c in self.captured}) == 1, 'ranks captured different numbers of collectives'
        for calls in zip(*self.captured):
            assert len({(c[0], c[1].numel(), c[1].dtype, c[3]) for c in calls}) == 1, 'ranks captured different collectives'
            self._launch(calls[0][0], [c[2] for c in calls], calls[0][3])
            for c in calls:
                c[1].copy_(c[2])
            self.log.extend(('ran-' + calls[0][0], r) for r in range(self.n))
        torch.cuda.synchronize()
        self.graph_runs += 1

    def before_step(self):
        """Called by every rank's optimizer.step() after its last replay: the captured collectives run once all ranks
        are there."""
        self._graph_barrier.wait(timeout=120)


def zero_copy_buckets(monkeypatch):
    """Zero-copy gradient buckets without registered memory: flat gradient buffers in plain device memory."""
    from horovod_b200.torch import mpi_ops
    monkeypatch.setattr(mpi_ops, 'symm_available', lambda process_set: True)
    monkeypatch.setattr(mpi_ops, 'symm_empty', lambda numel, dtype, device, process_set: torch.empty(numel, dtype=dtype, device=device))


def _stand_in(monkeypatch, t):
    """Routes the optimizers' collectives, and the gather of the sharded state in state_dict(), to the team `t`."""
    from horovod_b200.torch import mpi_ops
    zero_copy_buckets(monkeypatch)
    monkeypatch.setattr(mpi_ops, 'cross_size', lambda: 1)
    monkeypatch.setattr(mpi_ops, 'captured_reducescatter_', t.reducescatter)
    monkeypatch.setattr(mpi_ops, 'captured_allgather_', t.allgather)
    monkeypatch.setattr(mpi_ops, 'captured_allreduce_', t.allreduce)

    def state_allgather(tensor, name, process_set):
        # state_dict()'s gather of one state key of one bucket: the shards of every simulated rank in rank order
        _, _, bi, key = name.split('.', 3)
        return torch.cat([o._buckets[int(bi)]['state'][key] for o in t.opts])
    monkeypatch.setattr(mpi_ops, 'allgather', state_allgather)
    return t


@pytest.fixture
def team(hvd, monkeypatch):
    return _stand_in(monkeypatch, SimTeam(4))


@pytest.fixture
def gteam(hvd, monkeypatch):
    from horovod_b200.torch import optimizer
    t = _stand_in(monkeypatch, GraphTeam(4))
    monkeypatch.setattr(optimizer, 'allreduce_async_', t.allreduce_async_)
    monkeypatch.setattr(optimizer, 'synchronize', lambda handle: None)
    # the ranks' agreement on the capture is a real allreduce over the process set: every simulated rank captures here
    monkeypatch.setattr(hvd.GraphedStep, '_agree_across_ranks', lambda self: None)
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    return t


def sharded_team(hvd, team, base, make, dt=torch.float32, min_buckets=1, straddle=False, **kw):
    """A copy of `base` per simulated rank and its DistributedOptimizer over make(model), sharded unless `kw` says
    shard_optimizer_state=False, with buckets small enough that the model fills at least `min_buckets` of them.
    straddle: require a parameter cut between two ranks' shards, so that its norms must cross ranks.  `kw` goes to
    DistributedOptimizer.  The optimizers become team.opts; returns (models, opts)."""
    n = team.n
    models = [copy.deepcopy(base) for _ in range(n)]
    kw = dict(dict(shard_optimizer_state=True), **kw)
    opts = [hvd.DistributedOptimizer(make(m), named_parameters=m.named_parameters(), process_set=FakeSet(n, r),
                                     bucket_cap_mb=0.01 * dt.itemsize / 4, **kw) for r, m in enumerate(models)]
    team.opts = opts
    assert len(opts[0]._buckets) >= min_buckets, ('too few buckets', len(opts[0]._buckets), min_buckets)
    if straddle:
        cut = 0
        for b in opts[0]._buckets:
            for _, off, numel in b['members']:
                cut += off // b['shard'] != (off + numel - 1) // b['shard']
        assert cut > 0, "no parameter is cut between two ranks' shards"
    return models, opts


def reduced_grads(opts, params):
    """Every parameter's reduced gradient, with its strides, assembled from the owners' gradient shards (what the sharded
    update reads)."""
    from horovod_b200.torch.grad_buckets import full_from_shards
    out = {}
    for bi, b in enumerate(opts[0]._buckets):
        full = torch.cat([o._buckets[bi]['gshard'] for o in opts])
        for p, g in zip(b['params'], full_from_shards(b, [full], [p.shape for p in b['params']], [p.stride() for p in b['params']])):
            out[p] = g
    return [out[p] for p in params]


# ---- models and batches -------------------------------------------------------------------------------------------------
class ConvNet(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3)
        self.fc = torch.nn.Linear(8 * 6 * 6, 10)

    def forward(self, x):
        return self.fc(torch.relu(self.conv(x)).flatten(1))


class ConvNetWithUnused(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3)
        self.fc = torch.nn.Linear(8 * 6 * 6, 10)
        self.unused = torch.nn.Linear(4, 10)  # only in the forward when asked

    def forward(self, x, use_all=True):
        y = self.fc(torch.relu(self.conv(x)).flatten(1))
        return y + self.unused(x[:, 0, 0, :4]) if use_all else y


class NormConvNet(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3)
        self.fc = torch.nn.Linear(8 * 6 * 6, 10)
        self.norm = torch.nn.LayerNorm(10)
        self.head = torch.nn.Linear(10, 10)

    def forward(self, x):
        return self.head(self.norm(self.fc(torch.relu(self.conv(x)).flatten(1))))


def batch(step, r, dt=torch.float32):
    g = torch.Generator(device='cuda').manual_seed(100 * step + r)
    return torch.randn(5, 3, 8, 8, device='cuda', generator=g).to(dt), torch.randint(0, 10, (5,), device='cuda', generator=g)


def micro_batch(step, micro, r, dt):
    g = torch.Generator(device='cuda').manual_seed(1000 * step + 10 * micro + r)
    return torch.randn(5, 3, 8, 8, device='cuda', generator=g).to(dt), torch.randint(0, 10, (5,), device='cuda', generator=g)


# ---- one LAMB / LARS step on the simulated ranks and its reference ------------------------------------------------------
def step_all(team, models, opts, step, dt, clip=None):
    """Backward on every rank, then clip_grad_norm_(clip) or synchronize(), then step() in lockstep.  Returns the reduced
    gradients the update read and the clip coefficient (None without clip)."""
    n = team.n
    for r in range(n):
        opts[r].zero_grad()
        x, y = batch(step, r, dt)
        torch.nn.functional.cross_entropy(models[r](x), y).backward()
    coef = None
    if clip is not None:
        team.run(lambda r: opts[r].clip_grad_norm_(clip))
        coef = opts[0]._clip_coef.clone()
    else:
        for o in opts:
            o.synchronize()
        team.flush()
    grads = reduced_grads(opts, list(models[0].parameters()))
    mark = len(team.log)

    def step_rank(r):
        with opts[r].skip_synchronize():
            opts[r].step()
    team.run(step_rank)  # in lockstep: the apply phase must see the allreduced norms
    assert team.count('ar', mark) == n, 'one norms allreduce per rank and step'
    for r in range(1, n):
        for a, b in zip(models[r].parameters(), models[0].parameters()):
            assert same(a.detach(), b.detach()), 'ranks differ after the allgather'
    return grads, coef


def ref_step(ref, ref_opt, grads, coef=None, kind=None):
    """The unsharded reference's step on `grads`; with a clip coefficient, the fused LAMB or LARS update (`kind`) with the
    coefficient as its device-side gradient scale."""
    ref_opt.zero_grad()
    for p, g in zip(ref.parameters(), grads):
        p.grad = g.clone()
    if coef is None:
        ref_opt.step()
        return
    # the clip coefficient reaches the sharded update on the device; the reference gets it the same way
    from horovod_b200 import ops
    from horovod_b200.torch.optimizer import _fused_plan
    with torch.no_grad():
        for group, ps, gs in _fused_plan(ref_opt):
            st = [ref_opt.state[p] for p in ps]
            if kind == 'lamb':
                for s, p in zip(st, ps):
                    if 'exp_avg' not in s:
                        s['step'] = torch.tensor(0.0)
                        s['exp_avg'] = torch.zeros_like(p, dtype=torch.float32)
                        s['exp_avg_sq'] = torch.zeros_like(p, dtype=torch.float32)
                    s['step'] += 1
                b1, b2 = group['betas']
                ops.fused_lamb_step(ps, gs, [s['exp_avg'] for s in st], [s['exp_avg_sq'] for s in st], group['lr'], b1, b2,
                                    group['eps'], group['weight_decay'], int(st[0]['step']), group['bias_correction'],
                                    ref_opt.adapts(group), grad_scale_dev=coef.reshape(1))
            else:
                assert kind == 'lars', ('ref_step with a clip coefficient needs kind lamb or lars', kind)
                for s, p in zip(st, ps):
                    if 'momentum_buffer' not in s:
                        s['momentum_buffer'] = torch.zeros_like(p, dtype=torch.float32)
                ops.fused_lars_step(ps, gs, [s['momentum_buffer'] for s in st], group['lr'], group['momentum'],
                                    group['weight_decay'], group['trust_coefficient'], group['eps'], ref_opt.adapts(group),
                                    grad_scale_dev=coef.reshape(1))
