"""Sharded optimizer state (ZeRO stage 1) for `hvd.DistributedOptimizer(..., shard_optimizer_state=True)`.

Parameters and gradients of every (param group, dtype) live in flat buckets of registered symmetric memory, padded so
that each bucket splits into N equal, 128 B aligned, contiguous shards.  Rank r owns shard r of every bucket and keeps
optimizer state for that shard only.  A step is

    reduce-scatter the gradient bucket   (hvd.captured_reducescatter_, launched as soon as the bucket is ready)
    update the own shard                 (one fused SGD / Adam(W) kernel per param group and dtype)
    allgather the parameter bucket       (hvd.captured_allgather_)

which moves the same NVLink bytes as the allreduce it replaces, while the update does 1/N of the work and the state
takes 1/N of the memory.  The allgather runs after the update and does not overlap backward.

LAMB (hvd.Lamb) and LARS (hvd.Lars) need the norms of whole parameters, which the shards cut at arbitrary elements:
their update is split into lamb_norms / lars_norms over the owned pieces, one allreduce of a small registered buffer of
per-parameter sums of squares, and lamb_apply / lars_apply, so every rank computes each trust ratio from the same bits.

Global-norm clipping (`clip_grad_norm_`) and AMP loss scaling (`ShardedGradScaler`) read only the owned shards: one
statistics kernel per gradient dtype and one scalar allreduce give every rank the same norm and the same inf / NaN
verdict, and the clip coefficient reaches the update on the device.

With `master_weights=True` every bf16 / fp16 bucket also keeps an fp32 master copy of its owned shard ('master_param'),
which the fused kernel updates and rounds into the parameter shard before the allgather.

With `ema_decay=d` every bucket keeps an fp32 exponential moving average of its owned shard ('ema_param', 1/N of the
parameters per rank, plus padding), written by the same fused launch that updates the shard (the apply phase for
LAMB / LARS), and a flag saying whether it has begun; every member of a bucket begins at the bucket's first update.
state_dict() gathers it per parameter like the moments.  `ema_parameters()` is COLLECTIVE: each rank writes its rounded
EMA shard into its parameter shard and the parameter buckets are allgathered, on entry and again, with the stashed
own shards, on exit.

With `backward_passes_per_step=k > 1` and `grad_accumulation_dtype=torch.float32` every bf16 / fp16 gradient bucket has an
fp32 accumulator of its full size: when a bucket has received a backward pass's gradients it is folded into the
accumulator and zeroed (grad_accumulate_ 'first' / 'add'), and after the k-th pass the sum rounded once is written back
('last') right before the bucket's reduce-scatter, on the same stream.
"""
import warnings

import torch

from horovod_b200.common.process_sets import global_process_set
from horovod_b200.torch import mpi_ops
from horovod_b200.torch.compression import Compression
from horovod_b200.torch.grad_buckets import (ALIGN, adopt_grad, adopt_missing_grads, check_named_parameters, fold_last,
                                             full_from_shards, grad_bucket, shard_from_full, shard_layout, shard_range,
                                             shard_slices)
from horovod_b200.torch.mpi_ops import Average, Sum
from horovod_b200.torch.optimizer import (_COUNTS_STEPS, _STATE_KEYS, _DistributedOptimizerBase, _fused_update,
                                          _optimizer_kind, _state_dtype, _state_keys)


class _ShardedDistributedOptimizer(_DistributedOptimizerBase):
    """Wraps SGD / Adam / AdamW / Lamb / Lars so that every rank keeps optimizer state for 1/N of the parameters (ZeRO
    stage 1).
    Built by `hvd.DistributedOptimizer(opt, shard_optimizer_state=True)`; the dynamic class derives from this one and from
    the wrapped optimizer's class."""

    _norm_type_error = 'clip_grad_norm_ with sharded optimizer state supports norm_type 2 and inf, got %r'

    def __init__(self, params, named_parameters, compression, backward_passes_per_step=1, op=Average,
                 gradient_predivide_factor=1.0, groups=None, sparse_as_dense=False, process_set=global_process_set,
                 bucket_cap_mb=32, master_weights=False, grad_accumulation_dtype=None, ema_decay=None):
        super().__init__(params, process_set, op, gradient_predivide_factor, backward_passes_per_step,
                         grad_accumulation_dtype, ema_decay)
        kind = _optimizer_kind(self)
        if kind is None:
            raise ValueError('shard_optimizer_state supports SGD, Adam and AdamW, and hvd.Lamb and hvd.Lars, only, not %s'
                             % type(self).__name__)
        if kind == 'adafactor':
            raise ValueError('shard_optimizer_state does not support torch.optim.Adafactor: its factored state is already '
                             'O(R + C) per matrix, so sharding would save only master weights, and the row / column '
                             'factors would need an allreduce of partial row and column sums')
        for g in self.param_groups:
            if g.get('maximize', False) or (kind == 'adam' and g.get('amsgrad', False)):
                raise ValueError('shard_optimizer_state does not support maximize=True or amsgrad=True')
        if op not in (Average, Sum):
            raise ValueError('shard_optimizer_state supports op=Average or op=Sum only')
        if compression is not Compression.none or groups is not None or sparse_as_dense:
            raise ValueError('shard_optimizer_state does not support compression, groups or sparse_as_dense')
        check_named_parameters(self, named_parameters)
        trainable = [[p for p in g['params'] if p.requires_grad] for g in self.param_groups]
        for ps in trainable:
            for p in ps:
                if not (p.is_cuda and mpi_ops._is_dense(p) and p.dtype in (torch.float32, torch.bfloat16, torch.float16)):
                    raise ValueError('shard_optimizer_state needs dense CUDA fp32 / bf16 / fp16 parameters')
        if not (process_set.included() and mpi_ops.symm_available(process_set) and mpi_ops.cross_size() == 1):
            raise ValueError('shard_optimizer_state needs registered symmetric memory (P2P backend, one host, not elastic)')

        self._kind = kind
        self._nranks, self._rank = process_set.size(), process_set.rank()
        _, hi_pri = torch.cuda.Stream.priority_range()
        device = trainable[0][0].device if any(trainable) else torch.device('cuda', torch.cuda.current_device())
        self._comm = torch.cuda.Stream(device=device, priority=hi_pri)

        self._buckets = shard_layout([[(p.numel(), p.dtype) for p in ps] for ps in trainable], self._nranks,
                                     int(bucket_cap_mb * 1024 * 1024))
        self._p_to_bucket = {}
        with torch.no_grad():
            for bi, b in enumerate(self._buckets):
                ps = [trainable[b['group']][i] for i, _, _ in b['members']]
                pflat = mpi_ops.symm_empty(b['numel'], dtype=b['dtype'], device=device, process_set=process_set)
                pflat.zero_()
                grad_bucket(b, ps, device, process_set)
                b.update({'pflat': pflat, 'index': bi, 'step': 0, 'mom_init': False, 'pending': 0, 'ready': False})
                for p, (_, off, numel) in zip(ps, b['members']):
                    # keep the parameter's memory format (channels_last stays channels_last)
                    pview = pflat[off:off + numel].as_strided(p.size(), p.stride())
                    pview.copy_(p.data)
                    p.data = pview
                    self._p_to_bucket[p] = b
                lo, hi = shard_range(b, self._rank)
                b['pshard'], b['gshard'] = pflat[lo:hi], b['gflat'][lo:hi]
                master = master_weights and b['dtype'] != torch.float32
                b['state'] = {key: torch.zeros(b['shard'], dtype=_state_dtype(kind, b['dtype'], master), device=device)
                              for key in _state_keys(kind, self.param_groups[b['group']])}
                if master:
                    # fp32 master copy of the owned shard of a bf16 / fp16 bucket: optimizer state, sharded like the moments
                    b['state']['master_param'] = b['pshard'].float()
                if self.param_groups[b['group']].get('ema_decay') is not None:
                    # fp32 EMA of the owned shard: written whole by the bucket's first update ('ema_started')
                    b['state']['ema_param'] = torch.zeros(b['shard'], dtype=torch.float32, device=device)
                b['stepped'] = False
                b['ema_started'] = False
        # cross-rank gradient statistics: [sum of squares or max |g|, non-finite] in registered memory, padded so that the
        # in-place allreduce can split it across the ranks
        self._stats = mpi_ops.symm_empty(ALIGN // 4 * self._nranks, dtype=torch.float32, device=device,
                                         process_set=process_set)
        self._stats.zero_()
        self._trust_norms = None
        if kind in ('lamb', 'lars'):
            # the whole-parameter sums of squares of LAMB (w, u) or LARS (w, g) that their trust ratios need, in slot =
            # the parameter's index in param_groups order: every rank adds the pieces of its own shards and one allreduce
            # sums them.  Padded like _stats.
            self._slot = {p: i for i, p in enumerate(p for g in self.param_groups for p in g['params'])}
            unit = ALIGN // 4 * self._nranks
            self._trust_norms = mpi_ops.symm_empty((2 * len(self._slot) + unit - 1) // unit * unit, dtype=torch.float32,
                                                   device=device, process_set=process_set)
        self._delay = {p: backward_passes_per_step for p in self._p_to_bucket}
        self._seen = set()  # parameters whose gradient hook fired since the last synchronize()
        self._reset_launch_order()
        self._hooks = [p.register_post_accumulate_grad_hook(self._make_hook(p)) for p in self._p_to_bucket]

    # ---- launch order ---------------------------------------------------------------------------------------------------
    def _reset_launch_order(self):
        self._next = 0
        for b in self._buckets:
            b['pending'], b['ready'] = len(b['params']), False
        self._reset_folds()

    def _comm_stream(self):
        return self._graph_capture['comm'] if self._graph_capture is not None else self._comm

    def _mark_ready(self, bucket):
        """A bucket's reduce-scatter is launched once the bucket and every lower-numbered bucket are ready: all ranks issue
        the same sequence without negotiating, and buckets that complete in order still overlap backward."""
        bucket['ready'] = True
        while self._next < len(self._buckets) and self._buckets[self._next]['ready']:
            b = self._buckets[self._next]
            fold_last(b, self._graph_capture is not None)
            comm = self._comm_stream()
            comm.wait_stream(torch.cuda.current_stream())
            pre, post = self._scales()
            with torch.cuda.stream(comm):
                mpi_ops.captured_reducescatter_(b['gflat'], op=self.op, prescale_factor=pre, postscale_factor=post,
                                                process_set=self.process_set)
            self._next += 1

    def _make_hook(self, p):
        def hook(*ignore):
            if self._graph_mode and self._graph_capture is None:
                return  # GraphedStep warm-up / replay: the reductions are issued by the capture or by step()
            bucket = self._p_to_bucket[p]
            adopt_grad(p, bucket['views'][p], densify=False)
            if self._graph_capture is not None:
                bucket['pending'] -= 1
                if bucket['pending'] == 0:
                    self._mark_ready(bucket)
                return
            more = self._count_backward_pass(p)
            self._seen.add(p)
            self._fold_arrived(bucket, more > 0)
            if more == 0:
                bucket['pending'] -= 1
                if bucket['pending'] == 0:
                    self._mark_ready(bucket)
        return hook

    # ---- public API -------------------------------------------------------------------------------------------------------
    def synchronize(self):
        """Reduce-scatters every gradient bucket whose hook has not launched it yet (missing gradients count as zeros) and
        makes the current stream wait for all of them.  Afterwards only THIS rank's shard of each gradient bucket holds the
        reduced gradient; the rest of p.grad keeps this rank's local values, so ranks see different p.grad.  Anything that
        reads the whole p.grad and decides per rank is therefore unsupported with sharded optimizer state: gradient
        clipping on the full gradient, and torch.amp.GradScaler (its inf check would skip step() on some ranks only):
        use optimizer.clip_grad_norm_() and hvd.ShardedGradScaler instead.
        A step() after an explicit synchronize() does not reduce again."""
        self._reduce_pending()
        self._synchronized = True

    def _reduce_pending(self):
        if not (self._graph_mode and self._graph_comm_captured):
            for b in self._buckets[self._next:]:
                adopt_missing_grads(b, self._seen, densify=False)
            for b in self._buckets[self._next:]:
                self._mark_ready(b)
            torch.cuda.current_stream().wait_stream(self._comm)
        self._reset_launch_order()
        self._delay = dict.fromkeys(self._delay, self.backward_passes_per_step)
        self._seen.clear()

    def _reduce_once(self):
        if self._graph_capture is not None:
            raise RuntimeError('clip_grad_norm_ and ShardedGradScaler work in eager mode only, not inside hvd.GraphedStep')
        super()._reduce_once()

    def _start_afresh(self):
        self._drop_iteration_state()  # also after a synchronize() no step() followed: the new gradients need reducing

    def _shard_stats(self, norm_type, inv_scale=None):
        """[sum of squares (norm_type 2) or max |g| (inf), non-finite flag] of the reduced gradients over all ranks'
        owned shards, as a new 2-element fp32 tensor: one stats kernel per gradient dtype on this rank's shards (scaling
        them in place by inv_scale first, if given), then one allreduce of the small stats buffer.  No host sync."""
        from horovod_b200 import ops
        self._stats.zero_()
        ops.grad_shard_stats([b['gshard'] for b in self._buckets], self._stats, inv_scale=inv_scale, norm_type=norm_type)
        mpi_ops.captured_allreduce_(self._stats, op=Sum if norm_type == 2.0 else mpi_ops.Max, process_set=self.process_set)
        return self._stats[:2].clone()

    def _unscale_and_check(self, inv_scale, found_inf):
        """ShardedGradScaler._unscale_grads_: unscales the owned shards in place (fp16 included) and sets found_inf to
        the global non-finite flag, so that every rank skips or takes the step alike."""
        self._reduce_once()
        stats = self._shard_stats(2.0, inv_scale=inv_scale.float())
        found_inf.copy_(stats[1].clamp(max=1.0).reshape(found_inf.shape))
        self._stats_cache = stats
        return found_inf

    def _grad_norm(self, norm_type):
        if norm_type == 2.0 and self._stats_cache is not None:
            stats = self._stats_cache  # ShardedGradScaler.unscale_ computed them in its pass over the same gradients
        else:
            stats = self._shard_stats(norm_type)
        return (stats[0].sqrt() if norm_type == 2.0 else stats[0].clone()), None

    def _update_shards(self, coef=None):
        """One fused kernel per param group and dtype over this rank's shards.  coef: the clip coefficient on the
        device, or None."""
        by_group = {}
        for b in self._buckets:
            by_group.setdefault((b['group'], b['dtype'], b['ema_started']), []).append(b)
        with torch.no_grad():
            if self._kind in ('lamb', 'lars'):
                self._update_shards_trust(by_group, coef)
                return
            for (gi, _, ema_started), bs in by_group.items():
                group = self.param_groups[gi]
                keys = _state_keys(self._kind, group)
                # every bucket of a (group, dtype) has a master or none has, and an EMA or none has
                masters = [b['state']['master_param'] for b in bs] if 'master_param' in bs[0]['state'] else []
                emas = [b['state']['ema_param'] for b in bs] if 'ema_param' in bs[0]['state'] else []
                if self._kind in _COUNTS_STEPS:
                    for b in bs:
                        b['step'] += 1
                _fused_update(self, self._kind, group, [b['pshard'] for b in bs], [b['gshard'] for b in bs],
                              [[b['state'][key] for b in bs] for key in keys], masters, step=bs[0]['step'],
                              first_step=bool(keys) and not bs[0]['mom_init'], coef=coef, emas=emas,
                              ema_start=not ema_started)
                for b in bs:
                    b['mom_init'] = b['mom_init'] or (self._kind == 'sgd' and bool(keys))
                    b['stepped'] = True
                    b['ema_started'] = bool(emas)

    def _update_shards_trust(self, by_group, coef):
        """The trust ratios of LAMB and LARS need the norms of whole parameters, which the shards cut at arbitrary
        elements.  One table entry per parameter piece in this rank's shards, in the slot of its parameter: the norms
        phase per (group, dtype) adds the pieces' sums of squares into the registered norms buffer, one allreduce sums
        them over the ranks, and the apply phase per (group, dtype) updates the pieces with the same r on every rank.
        The clip coefficient reaches the phases that read the gradient.  Padding is not touched."""
        keys = _STATE_KEYS[self._kind]
        calls = []
        for (gi, _, ema_started), bs in by_group.items():
            lists, masters, slots, emas = tuple([] for _ in range(2 + len(keys))), [], [], []
            for b in bs:
                st = b['state']
                b['step'] += 1
                b['stepped'] = True
                b['ema_started'] = 'ema_param' in st
                if self._kind == 'lars':
                    b['mom_init'] = True  # LARS momentum: state_dict() gathers it from now on
                for k, plo, phi, slo in shard_slices(b, self._rank):
                    cut = slice(slo, slo + phi - plo)
                    for out, t in zip(lists, (b['pshard'], b['gshard']) + tuple(st[key] for key in keys)):
                        out.append(t[cut])
                    if 'master_param' in st:
                        masters.append(st['master_param'][cut])
                    if 'ema_param' in st:
                        emas.append(st['ema_param'][cut])
                    slots.append(self._slot[b['params'][k]])
            calls.append((self.param_groups[gi], bs[0]['step'], lists, masters, slots, emas, not ema_started))
        norms = self._trust_norms
        norms.zero_()
        for group, step, lists, masters, slots, _, _ in calls:
            _fused_update(self, self._kind, group, lists[0], lists[1], list(lists[2:]), masters, step=step, coef=coef,
                          phase='norms', norms=norms, slots=slots)
        mpi_ops.captured_allreduce_(norms, op=Sum, process_set=self.process_set)
        for group, step, lists, masters, slots, emas, ema_start in calls:
            _fused_update(self, self._kind, group, lists[0], lists[1], list(lists[2:]), masters, step=step, coef=coef,
                          phase='apply', norms=norms, slots=slots, emas=emas, ema_start=ema_start)

    def _allgather_params(self):
        comm = self._comm
        comm.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(comm):
            for b in self._buckets:
                mpi_ops.captured_allgather_(b['pflat'], process_set=self.process_set)
        torch.cuda.current_stream().wait_stream(comm)

    def step(self, closure=None):
        self._check_not_in_ema()
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        if self._should_synchronize and not self._reduced:
            if self._synchronized:
                # a reduce-scatter is not idempotent: running it again would mix the reduced shard with the peers' local
                # gradients, so the reduction done by synchronize() is used as it is
                warnings.warn('optimizer.step() called without optimizer.skip_synchronize() context after '
                              'optimizer.synchronize(); the gradients are not reduced a second time.')
            else:
                self.synchronize()
        coef = self._clip_coef
        self._drop_iteration_state()
        self._update_shards(coef)
        self._allgather_params()
        return loss

    _params_written = _allgather_params  # ema_parameters() wrote the owned shards

    def _ema_pairs(self):
        return [(b['pshard'], b['state']['ema_param']) for b in self._buckets if b['ema_started']]

    def zero_grad(self, set_to_none=True):
        """Zeroes the gradient buckets in place: p.grad stays a view of registered memory (set_to_none is ignored)."""
        if self._next > 0 or self._seen:
            # a launched reduce-scatter may still be reading this rank's gradients for a peer
            raise AssertionError('optimizer.zero_grad() was called after loss.backward() but before optimizer.step() or '
                                 'optimizer.synchronize(). This is prohibited as it can cause a race condition.')
        self._drop_iteration_state()  # an iteration whose step() was skipped leaves nothing behind
        for b in self._buckets:
            b['gflat'].zero_()
            for p in b['params']:
                if p.grad is None:
                    p.grad = b['views'][p]

    # ---- hvd.GraphedStep -----------------------------------------------------------------------------------------------
    def _new_graph_capture(self):
        """The reduce-scatters become graph nodes, on a stream like the eager one."""
        self._reset_launch_order()
        return {'comm': torch.cuda.Stream(device=self._comm.device, priority=self._comm.priority)}

    def _launch_remaining(self):
        for b in self._buckets[self._next:]:
            self._mark_ready(b)
        self._reset_launch_order()

    # ---- checkpoints ------------------------------------------------------------------------------------------------------
    def state_dict(self):
        """COLLECTIVE.  Gathers the shards bucket by bucket and returns the wrapped optimizer's own format with per-parameter
        state tensors on the CPU, so the checkpoint loads into a sharded or an unsharded DistributedOptimizer alike."""
        sd = torch.optim.Optimizer.state_dict(self)
        index = {id(p): i for i, p in enumerate(p for g in self.param_groups for p in g['params'])}
        state = {}
        for b in self._buckets:
            # which state has begun (the same on every rank); an SGD / LARS bucket may hold masters or an EMA only
            started = ((b['step'] > 0) if self._kind in _COUNTS_STEPS else
                       (b['mom_init'] or ('master_param' in b['state'] and b['stepped'])))
            keys = [key for key in b['state'] if (b['ema_started'] if key == 'ema_param' else started)]
            if not keys:
                continue
            gathered = {}
            for key in keys:
                shard = b['state'][key]
                full = mpi_ops.allgather(shard, name='sharded_opt.state.%d.%s' % (b['index'], key), process_set=self.process_set)
                gathered[key] = full_from_shards(b, [full], [p.shape for p in b['params']], [p.stride() for p in b['params']])
            for k, p in enumerate(b['params']):
                st = {key: vals[k].detach().cpu().clone() for key, vals in gathered.items()}
                if self._kind in _COUNTS_STEPS and started:
                    st['step'] = torch.tensor(float(b['step']))
                state[index[id(p)]] = st
        sd['state'] = state
        return sd

    def load_state_dict(self, state_dict):
        """Accepts the format of state_dict() from a sharded or an unsharded optimizer and keeps this rank's slice only.
        Does not communicate."""
        self._check_not_in_ema(loading=True)
        groups = state_dict['param_groups']
        if len(groups) != len(self.param_groups) or any(len(a['params']) != len(b['params']) for a, b in zip(groups, self.param_groups)):
            raise ValueError('loaded state dict does not match the optimizer\'s parameter groups')
        for mine, saved in zip(self.param_groups, groups):
            for k, v in saved.items():
                if k != 'params':
                    mine[k] = v
        ids = {}
        for saved, mine in zip(groups, self.param_groups):
            for i, p in zip(saved['params'], mine['params']):
                ids[p] = i
        saved_state = state_dict['state']
        with torch.no_grad():
            for b in self._buckets:
                per = [saved_state.get(ids[p], saved_state.get(str(ids[p]), {})) for p in b['params']]
                for key, shard in b['state'].items():
                    full = [st.get(key) for st in per]
                    if key == 'ema_param':
                        # the bucket's EMA begins once for all members: members without a saved EMA (an unsharded
                        # optimizer had no gradient for them yet) continue from their parameter's current value
                        b['ema_started'] = any(t is not None for t in full)
                        if b['ema_started']:
                            full = [p.detach().float() if t is None else t for t, p in zip(full, b['params'])]
                    shard.copy_(shard_from_full(b, self._rank, [None if t is None else t.detach() for t in full],
                                                [p.stride() for p in b['params']], dtype=shard.dtype, device='cpu'))
                    if key == 'momentum_buffer':
                        b['mom_init'] = any(t is not None for t in full)
                    if key == 'master_param':
                        # members without a saved master get zeros, which the kernel replaces by the parameter's value
                        b['stepped'] = any(t is not None for t in full)
                steps = [float(st['step']) for st in per if 'step' in st]
                b['step'] = int(max(steps)) if steps else 0
        self._reset_launch_order()
        self._delay = dict.fromkeys(self._delay, self.backward_passes_per_step)
        self._seen.clear()

    def _broadcast_state(self, root_rank):
        """hvd.broadcast_optimizer_state for sharded state: every shard has a single owner, so only the hyper-parameters
        and the per-bucket step counts travel.  The moments of a shard cannot come from the root, so every rank must
        already hold the same step counts (a fresh start, or load_state_dict() on every rank): if they differ, e.g. after
        loading a checkpoint on the root only, every rank raises ValueError instead of resuming with zero moments."""
        from horovod_b200.torch.functions import allgather_object, broadcast_object
        mine = {'steps': [b['step'] for b in self._buckets], 'mom_init': [b['mom_init'] for b in self._buckets],
                'ema_started': [b['ema_started'] for b in self._buckets]}
        meta = dict(mine, param_groups=[{k: v for k, v in g.items() if k != 'params'} for g in self.param_groups])
        meta = broadcast_object(meta, root_rank, 'sharded_opt.meta', self.process_set)
        same = mine == {k: meta[k] for k in mine}
        if not all(allgather_object(same, 'sharded_opt.same', self.process_set)):
            raise ValueError('broadcast_optimizer_state: the sharded optimizer state differs between ranks (was the '
                             'checkpoint loaded on the root rank only?); call load_state_dict() on every rank')
        for g, saved in zip(self.param_groups, meta['param_groups']):
            g.update(saved)
        for b, s, m in zip(self._buckets, meta['steps'], meta['mom_init']):
            b['step'], b['mom_init'] = s, m


class ShardedGradScaler(torch.amp.GradScaler):
    """torch.amp.GradScaler for `hvd.DistributedOptimizer(..., shard_optimizer_state=True)`; any other optimizer gets
    torch's behaviour unchanged.

    With sharded optimizer state only this rank's shard of each gradient bucket is reduced, so torch's per-rank inf / NaN
    check would let ranks disagree and skip step() on some of them only.  Here unscale_ reduces the pending gradients,
    unscales the owned shards in place (fp16 gradients included) in the same pass that checks them, and allreduces the
    verdict, so every rank sees the same found_inf: step() is taken or skipped, and the scale backed off, alike on all
    ranks.  The pass also yields the 2-norm, which a following optimizer.clip_grad_norm_(max_norm) reuses:

        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        opt.clip_grad_norm_(1.0)
        scaler.step(opt)
        scaler.update()
    """

    def _unscale_grads_(self, optimizer, inv_scale, found_inf, allow_fp16):
        if not isinstance(optimizer, _ShardedDistributedOptimizer):
            return super()._unscale_grads_(optimizer, inv_scale, found_inf, allow_fp16)
        return {found_inf.device: optimizer._unscale_and_check(inv_scale, found_inf)}
