"""DistributedOptimizer: wraps any torch optimizer so that gradients are
allreduced (averaged) across ranks while the backward pass is still running.

API parity: horovod/torch/optimizer.py (DistributedOptimizer factory,
_DistributedOptimizer, _DistributedAdasumOptimizer).  Mechanism differences:
hooks use `register_post_accumulate_grad_hook` (fires right after AccumulateGrad
with no autograd-graph surgery), completion is event-chained (no host sync per
tensor), and `fused=True` replaces the wrapped SGD/Adam(W) math by one
multi-tensor sm_90a kernel (csrc/kernels/optim_kernels.cu).
"""
import math
import numbers
import os
import warnings
from contextlib import contextmanager

import torch

from horovod_b200.common.exceptions import HorovodInternalError
from horovod_b200.common.process_sets import global_process_set
from horovod_b200.common.util import split_list
from horovod_b200.torch import mpi_ops
from horovod_b200.torch.compression import Compression
from horovod_b200.torch.grad_buckets import (adopt_grad, adopt_missing_grads, bucket_acc, check_grad_accumulation_dtype,
                                             check_named_parameters, find_duplicates, fold, fold_last, grad_bucket,
                                             reset_folds, shard_layout)
from horovod_b200.torch.lamb import Lamb
from horovod_b200.torch.lars import Lars
from horovod_b200.torch.mpi_ops import (Adasum, Average, Sum, allreduce_async_, grouped_allreduce_async_, rank, size,
                                        synchronize)


class _DistributedOptimizerBase(torch.optim.Optimizer):
    """What the two optimizers that reduce gradients share: the unsharded _DistributedOptimizer and the sharded (ZeRO-1)
    _ShardedDistributedOptimizer.  hvd.DistributedOptimizer() builds a class that derives from one of them and from the
    wrapped optimizer's class, so super() in this class reaches the wrapped optimizer.

    A subclass sets `_buckets` (its gradient buckets) and `_delay` (parameter -> backward passes of the step still to
    come), and supplies
      _reduce_pending()      reduce the gradients that are still pending (for clip_grad_norm_),
      _grad_norm(norm_type)  (norm of the reduced gradients or None without any, the gradients clip_grad_norm_ scales in
                             place or None when the fused update applies the coefficient),
      _ema_pairs()           [(parameter or owned shard, its fp32 EMA)] of every EMA that has begun,
      _new_graph_capture()   the state of a hvd.GraphedStep capture ({'comm': side stream, ...}), or None when the
                             reductions cannot be captured,
      _launch_remaining()    while capturing: launch the reductions that no hook launched."""

    _norm_type_error = 'clip_grad_norm_ supports norm_type 2 and inf, got %r'

    def __init__(self, params, process_set, op, gradient_predivide_factor, backward_passes_per_step,
                 grad_accumulation_dtype, ema_decay):
        super().__init__(params)
        self.process_set = process_set
        self.op = op
        self.gradient_predivide_factor = gradient_predivide_factor
        self.backward_passes_per_step = backward_passes_per_step
        # fp32 accumulators of bf16 / fp16 gradients over the backward passes of one step (allocated on first use, not
        # optimizer state)
        self._acc_fp32 = check_grad_accumulation_dtype(grad_accumulation_dtype)
        # fp32 exponential moving average of every trainable parameter, kept as optimizer state ('ema_param') and written
        # by the fused update kernels only: ema_decay implies fused, like master_weights.  The decay goes into every param
        # group as group['ema_decay'], read at every step like 'lr'.
        check_ema_decay(ema_decay)
        self._ema = ema_decay is not None
        self._ema_active = False  # inside ema_parameters()
        if self._ema:
            self.defaults['ema_decay'] = float(ema_decay)  # add_param_group() takes it from here
            for g in self.param_groups:
                g['ema_decay'] = float(ema_decay)
        self._graph_mode = False  # set by hvd.GraphedStep: backward runs as a CUDA graph replay, hooks do not fire
        self._graph_capture = None  # while hvd.GraphedStep captures: _new_graph_capture()
        self._graph_comm_captured = False  # the captured graph contains the gradient reductions (nothing left for step())
        self._should_synchronize = True  # False inside skip_synchronize()
        self._synchronized = False  # set by a user's synchronize()
        self._reduced = False       # set by clip_grad_norm_ / ShardedGradScaler: step() does not reduce again, silently
        self._clip_coef = None      # 0-dim fp32 device tensor from clip_grad_norm_, applied by the next fused step()
        self._stats_cache = None    # [sum of squares, non-finite] of the unscaled gradients from hvd.ShardedGradScaler

    # ---- one iteration ---------------------------------------------------------------------------------------------------
    @contextmanager
    def skip_synchronize(self):
        """Use after an explicit optimizer.synchronize() (e.g. gradient clipping) so that step() does not synchronize
        again."""
        self._should_synchronize = False
        try:
            yield
        finally:
            self._should_synchronize = True

    def _drop_iteration_state(self):
        self._synchronized = self._reduced = False
        self._clip_coef = self._stats_cache = None

    def _start_afresh(self):
        """A new backward pass or zero_grad() after an iteration whose step() was skipped (e.g. GradScaler found inf)
        leaves nothing of that iteration behind."""
        if self._reduced or self._clip_coef is not None:
            self._drop_iteration_state()

    def _count_backward_pass(self, p):
        """The top of p's gradient hook in eager mode: counts one of the step's backward passes and returns how many are
        still to come (0: p's gradient is complete)."""
        self._start_afresh()
        if self._delay[p] <= 0:
            raise AssertionError('Gradients were computed more than backward_passes_per_step times before call to step(). '
                                 'Increase backward_passes_per_step to accumulate gradients locally.')
        self._delay[p] -= 1
        return self._delay[p]

    def set_backward_passes_per_step(self, passes):
        self.backward_passes_per_step = passes
        self._delay = dict.fromkeys(self._delay, passes)
        self._reset_folds()

    def _scales(self):
        """(prescale, postscale) of a gradient reduction: op=Average splits the averaging into pre- and post-division
        around the sum (reference optimizer.py:197-204)."""
        if self.op == Average:
            return 1.0 / self.gradient_predivide_factor, self.gradient_predivide_factor
        return 1.0, 1.0

    def _hvd_super_step(self, closure=None):
        """The wrapped optimizer's own step(), without any reduction."""
        return super().step(closure)

    # ---- gradient accumulation in fp32 (grad_accumulation_dtype=torch.float32) -------------------------------------------
    def _accumulates(self, grad):
        """True when `grad` (a bucket's 'gflat' or a parameter's gradient) is summed over the backward passes in fp32."""
        return (self._acc_fp32 and self.backward_passes_per_step > 1 and grad is not None and grad.is_cuda
                and not grad.is_sparse and grad.dtype in (torch.bfloat16, torch.float16))

    def _fold_arrived(self, bucket, more):
        """The hook of one of the bucket's gradients.  Once the bucket has this backward pass's gradients and `more`
        passes of the step are to come, they are folded into the fp32 accumulator and zeroed ('first', then 'add')."""
        if not self._accumulates(bucket['gflat']):
            return
        bucket['arrived'] += 1
        if bucket['arrived'] == len(bucket['params']):
            bucket['arrived'] = 0
            if more:
                fold([bucket['gflat']], [bucket_acc(bucket)], 'add' if bucket['folds'] else 'first')
                bucket['folds'] += 1

    def _reset_folds(self):
        reset_folds(self._buckets)

    def _accumulator_pairs(self, with_buckets=True):
        """(16-bit gradients, fp32 accumulators) of every accumulating bucket, allocated now if needed."""
        bs = [b for b in self._buckets if with_buckets and self._accumulates(b['gflat'])]
        return [b['gflat'] for b in bs], [bucket_acc(b) for b in bs]

    def _prepare_accumulators(self):
        """hvd.GraphedStep, before capture: the accumulators must exist outside the graphs' memory pool."""
        self._accumulator_pairs()

    def _graph_fold(self, mode, with_buckets=True):
        """hvd.GraphedStep, while capturing: one fold of every accumulator after the captured backward pass."""
        fold(*self._accumulator_pairs(with_buckets), mode)

    def _mark_fold_last(self, capturing):
        """hvd.GraphedStep begins (capturing) or ends the capture of a step's last graph."""
        for b in self._buckets:
            b['fold_last'] = capturing and self._accumulates(b['gflat'])

    # ---- gradient reductions as CUDA-graph nodes (hvd.GraphedStep) -------------------------------------------------------
    def _begin_graph_capture(self):
        """Called by hvd.GraphedStep right after stream capture began (on the capturing stream): the gradient reductions
        become nodes of the graph, unless HVD_GRAPH_COMM=0 or the subclass cannot capture them.  Returns whether they do."""
        self._graph_comm_captured = False
        if os.environ.get('HVD_GRAPH_COMM', '1') == '0':
            return False
        self._graph_capture = self._new_graph_capture()
        if self._graph_capture is None:
            return False
        self._mark_fold_last(True)  # with backward_passes_per_step > 1 this is the step's last graph
        return True

    def _end_graph_capture(self):
        """Before stream capture ends: the reductions no hook launched are launched now, then the capturing stream joins
        the communication stream."""
        cap = self._graph_capture
        if cap is None:
            return
        self._launch_remaining()
        torch.cuda.current_stream().wait_stream(cap['comm'])
        self._graph_capture = None
        self._mark_fold_last(False)
        self._graph_comm_captured = True

    # ---- global-norm gradient clipping -----------------------------------------------------------------------------------
    def _reduce_once(self):
        """Reduces what is still pending unless this iteration's gradients are reduced already; the following step()
        neither reduces again nor warns."""
        if not (self._synchronized or self._reduced):
            self._reduce_pending()
            self._reduced = True

    def clip_grad_norm_(self, max_norm, norm_type=2.0, error_if_nonfinite=False):
        """Global-norm gradient clipping, the counterpart of torch.nn.utils.clip_grad_norm_(model.parameters(), ...):
        call it after backward (and after GradScaler.unscale_ or ShardedGradScaler.unscale_, if used) and before step().

        Reduces the gradients that are still pending, as synchronize() does (the following step() neither reduces again
        nor warns), and returns the norm of the reduced gradients as a 0-dim fp32 tensor on their device, with the same
        bits on every rank.  On CUDA the norm is one statistics kernel per gradient dtype, without a host
        synchronisation; with sharded optimizer state it is computed from the ranks' owned shards with one scalar
        allreduce.  When step() runs the fused update (always with sharded state), the clip coefficient
        min(max_norm / (norm + 1e-6), 1) stays on the device and scales the gradient inside that update, and p.grad is
        not rescaled; otherwise p.grad is scaled in place, as torch does.  norm_type is 2 or inf; sparse gradients raise
        ValueError.  error_if_nonfinite=True synchronises with the host, as torch's does."""
        norm_type = float(norm_type)
        if norm_type not in (2.0, math.inf):
            raise ValueError(self._norm_type_error % norm_type)
        self._reduce_once()
        total, grads = self._grad_norm(norm_type)
        if total is None:
            return torch.zeros((), dtype=torch.float32)
        if self._clip_coef is not None:
            total = total * self._clip_coef  # clipping twice: the norm of the gradient as the first clip left it
        if error_if_nonfinite and bool(torch.logical_or(total.isnan(), total.isinf())):
            raise RuntimeError('The total norm of order %s for gradients from `parameters` is non-finite, so it cannot be '
                               'clipped. To disable this error and scale the gradients by the non-finite norm anyway, set '
                               '`error_if_nonfinite=False`' % norm_type)
        coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
        if grads is None:
            self._clip_coef = coef if self._clip_coef is None else self._clip_coef * coef
        else:
            torch._foreach_mul_(grads, coef)
        return total

    # ---- the weight EMA (ema_decay) --------------------------------------------------------------------------------------
    def _check_not_in_ema(self, loading=False):
        if not self._ema_active:
            return
        if loading:
            raise RuntimeError('load_state_dict() inside ema_parameters(): the block restores the parameters on exit')
        raise RuntimeError('optimizer.step() inside ema_parameters(): the parameters hold the EMA there, and the update '
                           'would start from it')

    def _params_written(self):
        """ema_parameters() wrote the tensors of _ema_pairs(); whole parameters need nothing more."""

    @contextmanager
    def ema_parameters(self):
        """Evaluates with the EMA (optimizer built with ema_decay): inside the block every parameter that has an EMA holds
        it, rounded to the parameter's dtype and written in place (storage and addresses stay, so a captured
        hvd.GraphedStep remains valid; model.state_dict() taken inside is the EMA model, sharing the parameters' storage,
        so save or clone it inside).  On exit the parameters get their exact previous values back; masters, moments and
        the EMA are not touched.  Parameters the optimizer has not updated yet have no EMA and keep their values, and
        buffers such as BatchNorm running statistics are never averaged.  step() inside the block raises RuntimeError.
        The stash costs one copy of the parameters in their own dtype.

        With sharded optimizer state the block is COLLECTIVE: every rank must enter and leave it together.  Each rank
        stashes its own parameter shards, writes its EMA shards into them and allgathers the parameter buckets, so every
        rank holds the whole EMA model; on exit the stashed shards are written back and allgathered again.  Buckets whose
        EMA has not begun keep their values."""
        if not self._ema:
            raise RuntimeError('ema_parameters() needs an optimizer built with ema_decay')
        self._check_not_in_ema()
        pairs = self._ema_pairs()
        with torch.no_grad():
            stash = [t.clone() for t, _ in pairs]
            for t, e in pairs:
                t.copy_(e)
            self._params_written()
        self._ema_active = True
        try:
            yield
        finally:
            self._ema_active = False
            with torch.no_grad():
                for (t, _), s in zip(pairs, stash):
                    t.copy_(s)
                self._params_written()


class _DistributedOptimizer(_DistributedOptimizerBase):
    def __init__(self, params, named_parameters, compression, backward_passes_per_step=1, op=Average,
                 gradient_predivide_factor=1.0, groups=None, sparse_as_dense=False, process_set=global_process_set,
                 fused=False, zero_copy=None, bucket_cap_mb=32, bucket_wire_dtype=None, master_weights=False,
                 grad_accumulation_dtype=None, ema_decay=None):
        super().__init__(params, process_set, op, gradient_predivide_factor, backward_passes_per_step,
                         grad_accumulation_dtype, ema_decay)
        self._compression = compression
        # fp32 accumulators of the parameters outside the buckets (the buckets' are bucket['acc'])
        self._param_accs = {}
        self._acc_open = set()  # parameters outside the buckets folded this step whose 'last' fold is still to come
        # fp32 master copies of bf16 / fp16 parameters, kept as optimizer state ('master_param') and updated by the fused
        # kernels only: master_weights implies fused, and step() never hands those parameters to torch's own update
        self._master_weights = bool(master_weights)
        fused = fused or self._master_weights or self._ema
        # opt-in: fp32 gradient buckets travel as bf16 / fp16 (a registered shadow bucket of half the bytes is what the
        # zero-copy kernel reduces; the switch accumulates in fp32).  Not validated on hardware yet (docs/roadmap.md B3).
        if bucket_wire_dtype is None:
            bucket_wire_dtype = {'bf16': torch.bfloat16, 'fp16': torch.float16}.get(os.environ.get('HVD_BUCKET_WIRE_DTYPE', ''))
        self._bucket_wire_dtype = bucket_wire_dtype

        named_parameters = check_named_parameters(self, named_parameters)
        self._parameter_names = {v: k for k, v in sorted(named_parameters)}
        self._delay = {v: self.backward_passes_per_step for _, v in sorted(named_parameters)}
        self.sparse_as_dense = sparse_as_dense
        self._fused = fused

        self._handles = {}
        self._grad_accs = []
        self._requires_update = set()

        self._num_groups = None
        self._groups = None
        if groups is not None:
            if not (isinstance(groups, list) or groups > 0):
                raise ValueError('groups should be a non-negative integer or a list of list of torch.Tensor.')
            if isinstance(groups, list):
                grouped_parameter_ids = set()
                for l in groups:
                    for p in l:
                        if not isinstance(p, torch.Tensor):
                            raise ValueError('groups must consist of torch.Tensor.')
                        if id(p) in grouped_parameter_ids:
                            raise ValueError('A parameter can only appear once in groups.')
                        grouped_parameter_ids.add(id(p))
                self._groups = groups
            else:
                self._num_groups = groups
        self._p_to_group = {}
        self._group_counts = {}
        self._group_handles = {}
        self._buckets = []
        self._p_to_bucket = {}
        self._zero_copy = False
        if zero_copy is None:
            zero_copy = os.environ.get('HVD_ZERO_COPY', '1') != '0'
        if (zero_copy and groups is None and compression is Compression.none and op in (Average, Sum) and not sparse_as_dense
                and self.process_set.included() and mpi_ops.symm_available(self.process_set)):
            self._setup_buckets(int(bucket_cap_mb * 1024 * 1024))

        if self.process_set.included() and (size() > 1 or True):
            self._register_hooks()

    # -- reference API ----------------------------------------------------------
    def load_state_dict(self, state_dict):
        self._check_not_in_ema(loading=True)
        self._handles = {}
        self._synchronized = False
        self._should_synchronize = True
        self._delay = dict.fromkeys(self._delay, self.backward_passes_per_step)
        self._reset_folds()
        decays = [g.get('ema_decay') for g in self.param_groups]
        super().load_state_dict(state_dict)
        for g, d in zip(self.param_groups, decays):
            if d is not None:
                g.setdefault('ema_decay', d)  # a checkpoint taken without an EMA does not switch it off
        if self._fused and _optimizer_kind(self):
            self._keep_fp32_moments(state_dict)

    def _keep_fp32_moments(self, state_dict):
        """torch casts every loaded floating state tensor to its parameter's dtype. The fused kernels keep fp32 state for
        bf16 / fp16 parameters (_state_dtype), and with master weights the fp32 master copy, and with ema_decay the fp32
        EMA, so take the checkpoint's fp32 values back: a checkpoint round-trips exactly instead of losing their low
        bits."""
        kind = _optimizer_kind(self)
        saved = [i for g in state_dict['param_groups'] for i in g['params']]
        params = [p for g in self.param_groups for p in g['params']]
        for pid, p in zip(saved, params):
            st = state_dict['state'].get(pid, {})
            keys = _STATE_KEYS[kind] if _state_dtype(kind, p.dtype, self._master_weights) == torch.float32 else ()
            for key in keys + (('master_param',) if self._master_weights else ()) + (('ema_param',) if self._ema else ()):
                t = st.get(key)
                if torch.is_tensor(t) and t.dtype == torch.float32 and p.dtype != torch.float32 and key in self.state[p]:
                    if key in ('row_var', 'col_var'):  # Adafactor's factors: their own shapes, contiguous
                        self.state[p][key] = t.to(p.device, torch.float32, copy=True).contiguous()
                    else:
                        self.state[p][key] = _state_like(p, t, torch.float32)

    @staticmethod
    def find_duplicates(lst):
        return find_duplicates(lst)

    def _register_hooks(self):
        if self._groups is not None:
            p_list = []
            # identify how many gradients each group expects
            for i, group in enumerate(self._groups):
                for p in group:
                    self._p_to_group[p] = group
                    p_list.append(p)
                self._group_counts[id(group)] = 0
            for param_group in self.param_groups:
                for p in param_group['params']:
                    if p.requires_grad and p not in self._p_to_group:
                        self._p_to_group[p] = [p]
                        self._group_counts[id(self._p_to_group[p])] = 0
        elif self._num_groups:
            p_list = []
            for param_group in self.param_groups:
                for p in param_group['params']:
                    if p.requires_grad:
                        p_list.append(p)
            # rank-consistent grouping: order by name everywhere
            p_list = sorted(p_list, key=lambda p: self._parameter_names.get(p))
            self._groups = [list(g) for g in split_list(p_list, self._num_groups)]
            for group in self._groups:
                for p in group:
                    self._p_to_group[p] = group
                self._group_counts[id(group)] = 0

        for param_group in self.param_groups:
            for p in param_group['params']:
                if p.requires_grad:
                    self._requires_update.add(p)
                    self._grad_accs.append(p.register_post_accumulate_grad_hook(self._make_hook(p)))

    # ---- zero-copy gradient buckets (new here: the reference allreduces per-parameter tensors through a fusion buffer) ----
    def _setup_buckets(self, cap_bytes):
        """Lays the gradients of all dense CUDA parameters out in a few flat buffers of registered symmetric memory
        (p.grad becomes a view, like DDP's gradient_as_bucket_view). A bucket is allreduced IN PLACE as one tensor by the
        zero-copy NVLink kernel as soon as its last gradient is accumulated: no per-tensor negotiation, no pack/unpack.
        The layout is the sharded optimizer's for one rank, with all parameters as one group."""
        params = [p for g in self.param_groups for p in g['params']
                  if p.requires_grad and p.is_cuda and mpi_ops._is_dense(p) and p.dtype in (torch.float32, torch.bfloat16, torch.float16)]
        try:
            for layout in shard_layout([[(p.numel(), p.dtype) for p in params]], 1, cap_bytes):
                members = [params[i] for i, _, _ in layout['members']]
                bucket = grad_bucket(layout, members, members[0].device, self.process_set)
                bucket.update({'pending': len(members), 'name': 'bucket.%d' % len(self._buckets), 'handle': None,
                               'shadow': None, 'shadow_views': None})
                self._buckets.append(bucket)
                if self._bucket_wire_dtype is not None and layout['dtype'] == torch.float32:
                    shadow = mpi_ops.symm_empty(layout['numel'], dtype=self._bucket_wire_dtype, device=members[0].device,
                                                process_set=self.process_set)
                    shadow.zero_()
                    bucket['shadow'] = shadow
                    bucket['shadow_views'] = {p: shadow[off:off + numel].as_strided(p.size(), p.stride())
                                              for p, (_, off, numel) in zip(members, layout['members'])}
                for p in members:
                    self._p_to_bucket[p] = bucket
            self._zero_copy = True
        except HorovodInternalError as e:
            warnings.warn('zero-copy gradient buckets unavailable (%s); using the fused pack/unpack path' % e)
            for b in self._buckets:
                for p in b['params']:
                    p.grad = None
            self._buckets, self._p_to_bucket, self._zero_copy = [], {}, False

    def _launch_bucket(self, bucket):
        """Allreduces the bucket in place: with allreduce_async_ on the caller's stream, or, while hvd.GraphedStep
        captures, as a captured_allreduce_ node forked onto the side stream (so it overlaps the rest of backward)."""
        cap = self._graph_capture
        fold_last(bucket, cap is not None)  # on the caller's stream, so it precedes the allreduce
        prescale_factor, postscale_factor = self._scales()
        if cap is not None:
            cap['comm'].wait_stream(torch.cuda.current_stream())  # fork: everything recorded so far (this bucket's gradients) precedes it
        with torch.cuda.stream(cap['comm'] if cap is not None else None):
            wire = bucket['gflat']
            if bucket['shadow'] is not None:
                wire = bucket['shadow']
                wire.copy_(bucket['gflat'])  # one cast kernel fp32 -> wire dtype
            if cap is None:
                bucket['handle'] = allreduce_async_(wire, name=bucket['name'], op=self.op, prescale_factor=prescale_factor,
                                                    postscale_factor=postscale_factor, process_set=self.process_set)
                bucket['pending'] = len(bucket['params'])
                return
            # the last bucket in registration order holds the first layers' gradients: backward is over when it is ready
            tail = cap['tail'] or bucket is self._buckets[-1]
            mpi_ops.captured_allreduce_(wire, op=self.op, prescale_factor=prescale_factor, postscale_factor=postscale_factor,
                                        process_set=self.process_set, max_ctas=cap['tail_ctas'] if tail else cap['ctas'])
        cap['launched'].add(id(bucket))

    def _allreduce_grad_async(self, p):
        if p.grad is None:
            # gradient was not computed on this rank but the peers will reduce it: contribute zeros
            p.grad = torch.zeros_like(p.data)
        name = self._parameter_names.get(p)
        tensor = p.grad
        if tensor.is_sparse:
            if self.sparse_as_dense:
                tensor = tensor.to_dense()
                p.grad = tensor
            else:
                return mpi_ops.sparse_allreduce_async(tensor, name=name, op=self.op, process_set=self.process_set), None
        tensor_compressed, ctx = self._compression.compress(tensor)
        prescale_factor, postscale_factor = self._scales()
        handle = allreduce_async_(tensor_compressed, name=name, op=self.op, prescale_factor=prescale_factor,
                                  postscale_factor=postscale_factor, process_set=self.process_set)
        return handle, ctx

    def _grouped_allreduce_grad_async(self, ps):
        name = self._parameter_names.get(ps[0])
        for p in ps:
            if p.grad is None:
                p.grad = torch.zeros_like(p.data)
        tensors_compressed, ctxs = zip(*[self._compression.compress(p.grad) for p in ps])
        prescale_factor, postscale_factor = self._scales()
        handle = grouped_allreduce_async_(list(tensors_compressed), name=name, op=self.op, prescale_factor=prescale_factor,
                                          postscale_factor=postscale_factor, process_set=self.process_set)
        return handle, ctxs

    def _launch_group(self, group):
        handle, ctxs = self._grouped_allreduce_grad_async(group)
        self._group_handles[handle] = (group, ctxs)
        for gp in group:
            self._handles[gp] = (handle, None)
        self._group_counts[id(group)] = 0

    def _make_hook(self, p):
        def hook(*ignore):
            if self._graph_mode:
                # hooks only run during warm-up and capture; while capturing, the last gradient of a bucket records the
                # bucket's allreduce INTO the graph (on a forked side stream, so it overlaps the rest of backward)
                if self._graph_capture is not None:
                    self._graph_hook(p)
                return
            assert not p.grad.requires_grad
            more = self._count_backward_pass(p)
            handle, ctx = None, None
            bucket = self._p_to_bucket.get(p)
            if bucket is not None:
                adopt_grad(p, bucket['views'][p], densify=True)
                self._handles[p] = ('bucket', None)
                self._fold_arrived(bucket, more > 0)
                if more == 0:
                    bucket['pending'] -= 1
                    if bucket['pending'] == 0:
                        self._launch_bucket(bucket)
                return
            if self._accumulates(p.grad):
                if more > 0:
                    self._fold_param(p, 'add' if p in self._acc_open else 'first')
                elif p in self._acc_open:
                    self._fold_param(p, 'last')
            if more == 0:
                if self._groups is not None:
                    group = self._p_to_group[p]
                    self._group_counts[id(group)] += 1
                    if self._group_counts[id(group)] == len(group):
                        self._launch_group(group)
                        return
                else:
                    handle, ctx = self._allreduce_grad_async(p)
            self._handles[p] = (handle, ctx)
        return hook

    # ---- gradient accumulation in fp32 of the parameters outside the buckets (the base class has the buckets') -----------
    def _param_acc(self, p):
        acc = self._param_accs.get(p)
        if acc is None or acc.shape != p.grad.shape or acc.stride() != p.grad.stride():
            acc = self._param_accs[p] = (torch.empty_like(p.grad, dtype=torch.float32) if acc is None
                                         else _state_like(p.grad, acc, torch.float32))
        return acc

    def _fold_param(self, p, mode):
        fold([p.grad], [self._param_acc(p)], mode)
        if mode == 'last':
            self._acc_open.discard(p)
        else:
            self._acc_open.add(p)

    def _finish_param_folds(self):
        """step() before every backward pass of the step arrived: parameters whose 'last' fold is missing get it now."""
        for p in list(self._acc_open):
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            self._fold_param(p, 'last')

    def _reset_folds(self):
        self._acc_open.clear()
        super()._reset_folds()

    def _accumulator_pairs(self, with_buckets=True):
        """(16-bit gradients, fp32 accumulators) of every accumulating bucket and parameter, allocated now if needed."""
        grads, accs = super()._accumulator_pairs(with_buckets)
        for group in self.param_groups:
            for p in group['params']:
                if p.requires_grad and p not in self._p_to_bucket and self._accumulates(p.grad):
                    grads.append(p.grad)
                    accs.append(self._param_acc(p))
        return grads, accs

    # ---- gradient allreduce as CUDA-graph nodes (hvd.GraphedStep) --------------------------------------------------------
    def _new_graph_capture(self):
        """The whole gradient reduction can live inside the captured step when every trainable parameter sits in a
        registered zero-copy bucket and the reduction is one the in-place kernel implements.  With
        backward_passes_per_step > 1 the reduction is part of the step's last graph only.  Whether it can depends on the
        model and the constructor arguments only, so every rank answers the same."""
        if not (self._zero_copy and self._buckets and self.op in (Average, Sum)):
            return None
        if not self.process_set.included() or self.process_set.size() <= 1:
            return None
        if not all(p in self._p_to_bucket for p in self._requires_update):
            return None
        lo_pri, hi_pri = torch.cuda.Stream.priority_range() if hasattr(torch.cuda.Stream, 'priority_range') else (0, -1)
        return {'comm': torch.cuda.Stream(priority=hi_pri), 'launched': set(),
                # few CTAs while backward still needs the SMs, all of them for the tail bucket(s) that nothing overlaps any more
                # (without NVLS — teams of 2 — the P2P two-shot kernel needs more CTAs to keep up with backward)
                'ctas': int(os.environ.get('HVD_GRAPH_COMM_CTAS', '16' if '+mc' in mpi_ops.gpu_backend_info() and self.process_set.size() >= 4 else '32')),
                'tail_ctas': int(os.environ.get('HVD_GRAPH_COMM_TAIL_CTAS', '128')), 'tail': False,
                'pending': {id(b): len(b['params']) for b in self._buckets}}

    def _graph_hook(self, p):
        bucket = self._p_to_bucket.get(p)
        if bucket is None:
            return
        cap = self._graph_capture
        cap['pending'][id(bucket)] -= 1
        if cap['pending'][id(bucket)] == 0:
            self._launch_bucket(bucket)

    def _launch_remaining(self):
        """Buckets whose last hook never fired (parameters unused by the step) are reduced now."""
        cap = self._graph_capture
        cap['tail'] = True
        for bucket in self._buckets:
            if id(bucket) not in cap['launched']:
                self._launch_bucket(bucket)

    def _restore_shadows(self):
        """Reduced values of wire-dtype shadow buckets -> the fp32 gradients that p.grad points at."""
        for bucket in self._buckets:
            if bucket.get('shadow') is not None and bucket.get('shadow_fresh'):
                bucket['gflat'].copy_(bucket['shadow'])
                bucket['shadow_fresh'] = False

    def _grad_for_update(self, p):
        """The tensor the fused optimizer kernel should read as p's gradient (the wire-dtype shadow when it is fresh)."""
        bucket = self._p_to_bucket.get(p)
        if bucket is not None and bucket.get('shadow') is not None and bucket.get('shadow_fresh'):
            return bucket['shadow_views'][p]
        return p.grad

    def synchronize(self, _defer_shadow_copy=False):
        """Waits for every outstanding gradient allreduce (enqueueing the ones whose hook never fired so that all
        ranks stay in lock-step) and writes the reduced gradients back."""
        if not self.process_set.included():
            self._synchronized = True
            return
        if self._graph_mode and self.process_set.size() == 1 and self.op in (Average, Sum):
            self._synchronized = True  # one rank: the reduction is the identity (prescale * postscale == 1)
            return
        if self._graph_mode and self._graph_comm_captured:
            # the replayed graph already reduced every bucket (captured_allreduce_ nodes): nothing to negotiate or launch
            for bucket in self._buckets:
                if bucket.get('shadow') is not None:
                    bucket['shadow_fresh'] = True
            if not _defer_shadow_copy:
                self._restore_shadows()
            self._synchronized = True
            return
        if self._zero_copy:
            for bucket in self._buckets:
                if bucket['handle'] is None:
                    # some gradient of this bucket was not produced on this rank (or accumulation is incomplete): reduce what
                    # is there so that all ranks stay in lock-step (missing gradients are zeros)
                    adopt_missing_grads(bucket, self._handles, densify=True)
                    self._launch_bucket(bucket)
            reset_folds(self._buckets)
            for bucket in self._buckets:
                synchronize(bucket['handle'])
                bucket['handle'] = None
                if bucket.get('shadow') is not None:
                    bucket['shadow_fresh'] = True
                for p in bucket['params']:
                    self._delay[p] = self.backward_passes_per_step
                    self._handles.pop(p, None)
        if self._zero_copy and not _defer_shadow_copy:
            self._restore_shadows()  # callers of synchronize() (gradient clipping, ...) read p.grad
        self._finish_param_folds()
        pending = [p for p in self._requires_update if p not in self._handles and p not in self._p_to_bucket]
        pending += [p for p, (h, _) in self._handles.items() if h is None]
        if self._groups is not None:
            launched = set()
            for p in pending:
                group = self._p_to_group[p]
                if id(group) not in launched:
                    launched.add(id(group))
                    self._launch_group(group)
        else:
            for p in pending:
                self._handles[p] = self._allreduce_grad_async(p)

        waited = set()
        for p, (handle, ctx) in self._handles.items():
            if handle in self._group_handles:
                if handle in waited:
                    continue
                waited.add(handle)
                group, ctxs = self._group_handles[handle]
                outputs = synchronize(handle)
                for gp, out, c in zip(group, outputs, ctxs):
                    self._delay[gp] = self.backward_passes_per_step
                    if out is not gp.grad:
                        gp.grad.set_(self._compression.decompress(out, c))
                continue
            output = synchronize(handle)
            self._delay[p] = self.backward_passes_per_step
            if p.grad.is_sparse:
                aggregated = self._compression.decompress(output, ctx)
                if not aggregated.is_sparse:
                    aggregated = aggregated.to_sparse()
                p.grad = aggregated
            elif output is not None and output is not p.grad:
                p.grad.set_(self._compression.decompress(output, ctx))
        self._handles.clear()
        self._group_handles.clear()
        self._synchronized = True

    def _reduce_pending(self):
        self.synchronize(_defer_shadow_copy=self._fused)

    def _grads_to_clip(self):
        """The gradients the next update reads, with a fresh wire-dtype shadow in place of its fp32 bucket: each zero-copy
        bucket as one flat tensor (its padding stays zero), every other parameter's gradient on its own."""
        grads = [b['shadow'] if b.get('shadow') is not None and b.get('shadow_fresh') else b['gflat'] for b in self._buckets]
        grads += [p.grad for g in self.param_groups for p in g['params'] if p.grad is not None and p not in self._p_to_bucket]
        if any(g.is_sparse for g in grads):
            raise ValueError('clip_grad_norm_ does not support sparse gradients')
        return grads

    def _grad_norm(self, norm_type):
        """All ranks hold the same reduced gradients, so no further collective is needed."""
        fused = self._master_weights or (self._fused and _fused_plan(self) is not None)
        if not fused:
            self._restore_shadows()
        grads = self._grads_to_clip()
        if not grads:
            return None, None
        if grads[0].is_cuda:
            from horovod_b200 import ops
            stats = torch.zeros(2, dtype=torch.float32, device=grads[0].device)
            ops.grad_shard_stats(grads, stats, norm_type=norm_type)
            total = stats[0].sqrt() if norm_type == 2.0 else stats[0].clone()
        else:  # CPU tensors: torch's norm
            total = torch.nn.utils.get_total_norm(grads, norm_type)
        return total, None if fused else grads

    def step(self, closure=None):
        self._check_not_in_ema()
        if self._should_synchronize and not self._reduced:
            if self._synchronized:
                warnings.warn("optimizer.step() called without optimizer.skip_synchronize() context after "
                              "optimizer.synchronize(). This can cause training slowdown. You may want to consider "
                              "using optimizer.skip_synchronize() context if you use optimizer.synchronize() in your "
                              "code.")
            self.synchronize(_defer_shadow_copy=self._fused and closure is None)
        coef = self._clip_coef
        self._drop_iteration_state()
        if self._master_weights or self._ema or (self._fused and closure is None):
            # the masters and the EMA live in the fused kernels only: evaluate the closure, then the fused update (or an
            # error)
            loss = None
            if closure is not None:
                with torch.enable_grad():
                    loss = closure()
            if _fused_step(self, coef):  # always True with masters or EMA: it raises when the update cannot be fused
                for bucket in self._buckets:
                    bucket['shadow_fresh'] = False
                return loss
        self._restore_shadows()
        if coef is not None:  # clip_grad_norm_ expected the fused update, which could not run
            torch._foreach_mul_(self._grads_to_clip(), coef)
        return super().step(closure)

    def _ema_pairs(self):
        return [(p.detach(), self.state[p]['ema_param']) for g in self.param_groups for p in g['params']
                if 'ema_param' in self.state.get(p, {})]

    def zero_grad(self, *args, **kwargs):
        if self._handles:
            raise AssertionError("optimizer.zero_grad() was called after loss.backward() but before optimizer.step() or "
                                 "optimizer.synchronize(). This is prohibited as it can cause a race condition.")
        self._start_afresh()
        if self._zero_copy:
            # bucketed gradients must stay views of the registered buffers: zero them in place (one memset per bucket)
            for bucket in self._buckets:
                bucket['gflat'].zero_()
            for group in self.param_groups:
                for p in group['params']:
                    if p not in self._p_to_bucket and p.grad is not None:
                        if self._graph_mode:
                            p.grad.zero_()  # addresses baked into the captured graph must stay valid
                        else:
                            p.grad = None
            return None
        if self._graph_mode:
            kwargs['set_to_none'] = False
            args = ()
        return super().zero_grad(*args, **kwargs)


def _optimizer_kind(opt):
    """Which fused update serves `opt`: 'sgd', 'adam' (Adam and AdamW), 'lamb' (hvd.Lamb), 'lars' (hvd.Lars),
    'adafactor' (torch.optim.Adafactor), or None."""
    kinds = ((torch.optim.SGD, 'sgd'), ((torch.optim.Adam, torch.optim.AdamW), 'adam'), (Lamb, 'lamb'), (Lars, 'lars'),
             (torch.optim.Adafactor, 'adafactor'))
    return next((kind for cls, kind in kinds if isinstance(opt, cls)), None)


# The state the fused kernels keep per parameter (per owned shard with sharded state), in the order the kernels take it.
# Every state tensor is fp32 except SGD momentum without master weights (_state_dtype).  Adam, LAMB and Adafactor also
# count steps.  Adafactor keeps row_var / col_var (torch's factor shapes) for a parameter of dim >= 2, else variance.
_STATE_KEYS = {'sgd': ('momentum_buffer',), 'adam': ('exp_avg', 'exp_avg_sq'), 'lamb': ('exp_avg', 'exp_avg_sq'),
               'lars': ('momentum_buffer',), 'adafactor': ('row_var', 'col_var', 'variance')}
_COUNTS_STEPS = ('adam', 'lamb', 'adafactor')
# the most dims of a parameter the fused Adafactor takes: the two factored dims and three batch dims
_ADAFACTOR_MAX_DIMS = 5


def _state_keys(kind, group):
    return () if kind == 'sgd' and group.get('momentum', 0.0) == 0.0 else _STATE_KEYS[kind]


def _state_dtype(kind, dtype, master):
    return dtype if kind == 'sgd' and not master else torch.float32


def check_ema_decay(decay):
    """ema_decay is None (no EMA) or a number d with 0 <= d <= 1, the range torch's get_ema_multi_avg_fn accepts."""
    if decay is not None and not (isinstance(decay, numbers.Real) and not isinstance(decay, bool) and 0.0 <= decay <= 1.0):
        raise ValueError('ema_decay must be None or a number in [0, 1], got %r' % (decay,))


def ema_weight(group):
    """The kernels' EMA weight 1 - d for the group's current decay d, checked (a schedule may have changed it)."""
    d = group['ema_decay']
    if torch.is_tensor(d):
        d = d.item()
    check_ema_decay(d)
    return 1.0 - float(d)


def _fused_update(opt, kind, group, ps, grads, states, masters, step=0, first_step=False, coef=None, phase=None,
                  norms=None, slots=None, emas=(), ema_start=False):
    """The native fused update of `kind` for params `ps` of `group` (hyper-parameters read now, so LR schedulers work),
    with one list per state key and fp32 masters ([]: none).  coef: a device factor on the gradient (clip coefficient).
    LAMB / LARS: both phases (phase None), or phase 'norms' / 'apply' on `norms` / `slots` to allreduce in between.
    emas: the fp32 EMA of every param (empty: none), written by the update launch with group['ema_decay'], and begun
    there with ema_start."""
    native = mpi_ops._native()
    lr, wd = float(group['lr']), float(group.get('weight_decay', 0.0))
    ema = (list(emas), ema_weight(group), bool(ema_start)) if emas else ([], 0.0, False)
    if kind == 'sgd':
        native.fused_sgd_step(ps, grads, states[0] if states else [], lr, float(group.get('momentum', 0.0)),
                              float(group.get('dampening', 0.0)), wd, bool(group.get('nesterov', False)), 1.0,
                              first_step, coef, masters, *ema)
    elif kind == 'adam':
        b1, b2 = group['betas']
        adamw = isinstance(opt, torch.optim.AdamW) or bool(group.get('decoupled_weight_decay', False))
        native.fused_adam_step(ps, grads, *states, lr, float(b1), float(b2), float(group['eps']), wd, step, 1.0, adamw,
                               coef, masters, *ema)
    elif kind == 'lamb':
        b1, b2 = group['betas']
        hp = (float(b1), float(b2), float(group['eps']), wd, step, bool(group['bias_correction']))
        if phase is None:
            native.fused_lamb_step(ps, grads, *states, lr, *hp, Lamb.adapts(group), 1.0, coef, masters, *ema)
        elif phase == 'norms':
            native.lamb_norms(ps, grads, *states, *hp, 1.0, coef, masters, norms, slots)
        else:
            native.lamb_apply(ps, grads, *states, lr, *hp, Lamb.adapts(group), masters, norms, slots, *ema)
    elif kind == 'adafactor':
        eps1, eps2 = group['eps']
        eps1 = torch.finfo(ps[0].dtype).eps if eps1 is None else float(eps1)  # resolved per launch, as torch does
        native.fused_adafactor_step(ps, grads, *states, lr, float(group['beta2_decay']), eps1, float(eps2),
                                    float(group['d']), wd, step, 1.0, coef, masters, *ema)
    else:
        hp = (lr, float(group['momentum']), wd, float(group['trust_coefficient']), float(group['eps']), Lars.adapts(group),
              1.0, coef, masters)
        if phase is None:
            native.fused_lars_step(ps, grads, *states, *hp, *ema)
        elif phase == 'norms':
            native.lars_norms(ps, grads, *states, 1.0, coef, masters, norms, slots)
        else:
            native.lars_apply(ps, grads, *states, *hp, norms, slots, *ema)


def _fused_plan(opt, why=None):
    """Pure eligibility pass of the fused optimizer step: returns the launch plan [(group, params, grads)] or None.
    Nothing is mutated here, so a `None` leaves the wrapped optimizer's own step() as a clean fallback; the reason is
    appended to the list `why`, if given."""
    def no(reason):
        if why is not None:
            why.append(reason)
        return None

    master = getattr(opt, '_master_weights', False)
    kind = _optimizer_kind(opt)
    if kind is None:
        return no('the optimizer is %s, not SGD, Adam or AdamW, hvd.Lamb or hvd.Lars, or torch.optim.Adafactor'
                  % type(opt).__name__)
    grad_of = getattr(opt, '_grad_for_update', lambda q: q.grad)
    plan = []
    for group in opt.param_groups:
        params = [p for p in group['params'] if p.grad is not None]
        if not params:
            continue
        if group.get('maximize', False) or (kind == 'adam' and group.get('amsgrad', False)):
            return no('maximize=True or amsgrad=True')
        if not all(p.is_cuda and not p.grad.is_sparse and mpi_ops._is_dense(p) and p.grad.stride() == p.stride() for p in params):
            return no('a parameter is not a dense CUDA tensor, its gradient is sparse, or its strides differ from the gradient\'s')
        if kind == 'adafactor' and any(p.dim() > _ADAFACTOR_MAX_DIMS for p in params):
            return no('a parameter has more than %d dims, the most the fused Adafactor factors' % _ADAFACTOR_MAX_DIMS)
        by_dtype = {}
        for p in params:
            by_dtype.setdefault((p.dtype, grad_of(p).dtype), []).append(p)
        if any(pd == torch.float32 and gd == torch.float16 for pd, gd in by_dtype):
            return no('fp16 gradients of fp32 parameters')  # no fp32-parameter / fp16-gradient kernel
        if master and any(pd != torch.float32 and gd != pd for pd, gd in by_dtype):
            return no('bf16 / fp16 parameters with gradients of another dtype')  # master kernels: (bf16, bf16), (fp16, fp16)
        for ps in by_dtype.values():
            if kind == 'sgd' and group.get('momentum', 0.0) != 0.0 and not master:
                have = [opt.state[p].get('momentum_buffer') is not None for p in ps]
                if any(have) and not all(have):
                    return None  # partially initialised momentum (parameters added later): let torch handle it
            plan.append((group, ps, [grad_of(p) for p in ps]))
    return plan


def _master_param(opt, p):
    """p's fp32 master copy with p's strides, created from p on first use (a checkpoint's or a stray layout is
    normalised). A master that p's value no longer matches is reconciled by the kernel itself."""
    st = opt.state[p]
    w = st.get('master_param')
    if w is None:
        w = st['master_param'] = _state_like(p, p.detach(), torch.float32)
    elif w.dtype != torch.float32 or w.stride() != p.stride() or w.device != p.device:
        w = st['master_param'] = _state_like(p, w, torch.float32)
    return w


def _ema_param(opt, p):
    """p's fp32 EMA with p's strides and whether it starts now (it does not exist yet: the update writes it whole)."""
    st = opt.state[p]
    e = st.get('ema_param')
    if e is None:
        st['ema_param'] = torch.empty_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
        return st['ema_param'], True
    if e.dtype != torch.float32 or e.stride() != p.stride() or e.device != p.device:
        e = st['ema_param'] = _state_like(p, e, torch.float32)
    return e, False


def _param_state(opt, kind, p, keys, master):
    """p's state `keys` for the fused kernel and whether it starts now: zeros, or in the kernel's dtype and p's strides
    (torch's step and load_state_dict leave p's dtype or a checkpoint's layout).  The step count becomes a tensor."""
    st = opt.state[p]
    dtype = _state_dtype(kind, p.dtype, master)
    fresh = bool(keys) and st.get(keys[0]) is None
    if kind in _COUNTS_STEPS:
        step = 0.0 if fresh else st['step']
        st['step'] = step if torch.is_tensor(step) else torch.tensor(float(step))
    out = []
    for key in keys:
        t = st.get(key)
        if t is None:
            t = st[key] = torch.zeros_like(p, dtype=dtype, memory_format=torch.preserve_format)
        elif t.dtype != dtype or t.stride() != p.stride():
            t = st[key] = _state_like(p, t, dtype)
        out.append(t)
    return out, fresh


def _adafactor_state(opt, p):
    """p's Adafactor state for the fused kernel as [row_var], [col_var], [variance] (None where p has none) and whether it
    starts now: zeros in torch's shapes, or fp32 (torch's own step keeps it in the gradient dtype) with the layout the
    kernel takes -- contiguous factors, a variance with p's strides."""
    st = opt.state[p]
    fresh = st.get('row_var') is None and st.get('variance') is None
    if p.dim() >= 2:
        for key, dim in (('row_var', -1), ('col_var', -2)):
            shape = list(p.shape)
            shape[dim] = 1
            t = st.get(key)
            if t is None:
                st[key] = torch.zeros(shape, dtype=torch.float32, device=p.device)
            elif t.dtype != torch.float32 or not t.is_contiguous() or t.device != p.device:
                if list(t.shape) != shape:
                    raise RuntimeError('optimizer state %s of shape %s does not fit a parameter of shape %s'
                                       % (key, tuple(t.shape), tuple(p.shape)))
                st[key] = t.to(device=p.device, dtype=torch.float32, memory_format=torch.contiguous_format)
        return [st['row_var'], st['col_var'], None], fresh
    t = st.get('variance')
    if t is None:
        t = st['variance'] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
    elif t.dtype != torch.float32 or t.stride() != p.stride():
        t = st['variance'] = _state_like(p, t, torch.float32)
    return [None, None, t], fresh


def _fused_step(opt, coef=None):
    """One multi-tensor kernel for the whole model when the wrapped optimizer is SGD or Adam/AdamW on CUDA, three for
    Lamb and Lars (their trust ratios need whole-tensor norms before the update). With master weights a plan that cannot
    be fused raises RuntimeError instead of returning False, and so does one with an EMA.  coef: the clip coefficient on the
    device, or None."""
    use_master = getattr(opt, '_master_weights', False)
    use_ema = getattr(opt, '_ema', False)
    why = []
    plan = _fused_plan(opt, why)
    if plan is None:
        if use_master:
            raise RuntimeError('master_weights: the fused optimizer update cannot run (%s), and torch\'s own update would '
                               'bypass the fp32 master weights' % (why[0] if why else 'not eligible'))
        if use_ema:
            raise RuntimeError('ema_decay: the fused optimizer update cannot run (%s), and torch\'s own update would not '
                               'update the EMA' % (why[0] if why else 'not eligible'))
        return False
    kind = _optimizer_kind(opt)
    for group, _, _ in plan:
        if use_ema and group.get('ema_decay') is not None:
            ema_weight(group)  # a scheduled decay out of range raises before any state is created
    with torch.no_grad():
        for group, ps, grads in plan:
            master = use_master and ps[0].dtype != torch.float32
            masters = [_master_param(opt, p) for p in ps] if master else []
            keys = _state_keys(kind, group)
            if kind == 'adafactor':
                per_param, fresh = zip(*[_adafactor_state(opt, p) for p in ps])
                for p, f in zip(ps, fresh):
                    step = 0.0 if f else opt.state[p]['step']
                    opt.state[p]['step'] = step if torch.is_tensor(step) else torch.tensor(float(step))
            else:
                per_param, fresh = zip(*[_param_state(opt, kind, p, keys, master) for p in ps])
            states = [[st[k] for st in per_param] for k in range(len(keys))]
            emas, ema_new = zip(*[_ema_param(opt, p) for p in ps]) if use_ema and group.get('ema_decay') is not None \
                else ([], [False] * len(ps))
            # one launch per (step count, momentum start, EMA start), normally one: Adam's and LAMB's bias corrections
            # follow each parameter's own count (a parameter without a gradient does not advance, a checkpoint may mix
            # counts); with masters an SGD parameter that joins later starts its momentum while the others continue, and
            # so does the EMA of a parameter whose first gradient comes later
            counts = [0] * len(ps)
            if kind in _COUNTS_STEPS:
                steps = [opt.state[p]['step'] for p in ps]
                # one host-side call for the whole group instead of a tensor op per parameter (BERT-large: ~400 of them)
                cpu_steps = [t for t in steps if not t.is_cuda]
                if cpu_steps:
                    torch._foreach_add_(cpu_steps, 1)
                for t in steps:
                    if t.is_cuda:
                        t.add_(1)
                counts = torch.stack(cpu_steps).tolist() if len(cpu_steps) == len(steps) else [t.item() for t in steps]
            parts = {}
            for i, (c, f, e) in enumerate(zip(counts, fresh, ema_new)):
                parts.setdefault((int(c), kind == 'sgd' and f, e), []).append(i)
            for (step, first, ema_start), idx in parts.items():
                pick = lambda xs: [xs[i] for i in idx] if xs else xs  # noqa: E731
                _fused_update(opt, kind, group, pick(ps), pick(grads), [pick(s) for s in states], pick(masters),
                              step=step, first_step=first, coef=coef, emas=pick(emas), ema_start=ema_start)
    return True


def _state_like(p, t, dtype):
    """A copy of optimizer state `t` in `dtype` with exactly p's strides, so the fused kernels can index it like p."""
    if t.shape != p.shape:
        raise RuntimeError('optimizer state of shape %s does not fit a parameter of shape %s' % (tuple(t.shape), tuple(p.shape)))
    out = torch.empty_like(p, dtype=dtype, memory_format=torch.preserve_format)
    out.copy_(t)
    return out


class _DistributedAdasumOptimizer(torch.optim.Optimizer):
    """Adasum works on parameter *deltas*: each parameter's hook runs the wrapped optimizer on that parameter only,
    allreduces delta = p_new - p_start with op=Adasum and step() applies start + adasum(delta).
    (reference horovod/torch/optimizer.py:345-513)"""

    def __init__(self, params, named_parameters, compression, backward_passes_per_step=1):
        super().__init__(params)
        self._compression = compression
        named_parameters = check_named_parameters(self, named_parameters)
        self._parameter_names = {v: k for k, v in sorted(named_parameters)}
        self.backward_passes_per_step = backward_passes_per_step
        self._delay = {v: self.backward_passes_per_step for _, v in sorted(named_parameters)}
        self._handles = {}
        self._grad_accs = []
        self._requires_update = set()
        self._synchronized = False
        self._should_synchronize = True
        self._starting_models = {p: torch.zeros_like(p, requires_grad=False) for _, p in named_parameters}
        self._graph_mode = False  # hvd.GraphedStep: hooks are silent, step() runs the whole-model variant below
        self._register_hooks()

    def set_backward_passes_per_step(self, passes):
        self.backward_passes_per_step = passes
        self._delay = dict.fromkeys(self._delay, passes)

    def _register_hooks(self):
        for param_group in self.param_groups:
            for p in param_group['params']:
                if p.requires_grad:
                    self._requires_update.add(p)
                    self._grad_accs.append(p.register_post_accumulate_grad_hook(self._make_hook(p)))

    def _allreduce_grad_async(self, p):
        # run the wrapped optimizer on this parameter alone
        name = self._parameter_names.get(p)
        if p.grad is None:
            p.grad = torch.zeros_like(p.data)
        stashed_params = []
        for group in self.param_groups:
            stashed_params.append(group['params'])
            if any(p is v for v in group['params']):
                group['params'] = [p]
            else:
                group['params'] = []
        start = self._starting_models[p]
        start.data.copy_(p)
        super().step()
        p.data.sub_(start)  # p now holds the local delta
        tensor_compressed, ctx = self._compression.compress(p.data)
        handle = allreduce_async_(tensor_compressed, name=name, op=Adasum)
        for stashed, group in zip(stashed_params, self.param_groups):
            group['params'] = stashed
        return handle, ctx

    def _make_hook(self, p):
        def hook(*ignore):
            if self._graph_mode:
                return
            if p in self._handles and self._handles[p][0] is not None:
                if self._delay[p] <= 0:
                    raise AssertionError(
                        "Gradients were computed more than backward_passes_per_step times before call to step(). "
                        "Increase backward_passes_per_step to accumulate gradients locally.")
            assert not p.grad.requires_grad
            assert self._delay[p] > 0
            handle, ctx = None, None
            self._delay[p] -= 1
            if self._delay[p] == 0:
                handle, ctx = self._allreduce_grad_async(p)
            self._handles[p] = (handle, ctx)
        return hook

    def _whole_model_step(self):
        """Same math as the per-parameter hooks, issued once for the whole model (graph mode: backward was a CUDA graph
        replay, so there is nothing to overlap with): stash, ONE wrapped-optimizer step over all parameters, delta =
        new - start, Adasum-allreduce every delta (the engine fuses them up to the fusion threshold), start + result."""
        ps = sorted(self._requires_update, key=lambda p: self._parameter_names.get(p))
        for p in ps:
            if p.grad is None:
                p.grad = torch.zeros_like(p.data)
        starts = [self._starting_models[p] for p in ps]
        datas = [p.data for p in ps]
        with torch.no_grad():
            torch._foreach_copy_(starts, datas)
            super().step()
            torch._foreach_sub_(datas, starts)
            handles = []
            for p in ps:
                comp, ctx = self._compression.compress(p.data)
                handles.append((allreduce_async_(comp, name=self._parameter_names.get(p), op=Adasum), ctx, p))
            for h, ctx, p in handles:
                delta = self._compression.decompress(synchronize(h), ctx)
                if delta is not p.data:
                    p.data.copy_(delta)
            torch._foreach_add_(starts, datas)
            torch._foreach_copy_(datas, starts)

    def synchronize(self):
        pass

    @contextmanager
    def skip_synchronize(self):
        raise AssertionError("Skipping synchronization is not supported when using Adasum optimizer.")

    def step(self, closure=None):
        loss = None
        if closure is not None:
            loss = closure()
        if self._graph_mode:
            self._whole_model_step()
            return loss
        missing_p = self._requires_update - set(self._handles.keys())
        for p in missing_p:
            self._delay[p] = 0
            handle, ctx = self._allreduce_grad_async(p)
            self._handles[p] = (handle, ctx)
        for p, (handle, ctx) in self._handles.items():
            if handle is None:
                handle, ctx = self._allreduce_grad_async(p)
                self._handles[p] = (handle, ctx)
        for p, (handle, ctx) in self._handles.items():
            delta = synchronize(handle)
            delta = self._compression.decompress(delta, ctx)
            start = self._starting_models[p]
            start.data.add_(delta.data)
            p.data.copy_(start)
            self._delay[p] = self.backward_passes_per_step
        self._handles.clear()
        return loss

    def zero_grad(self, *args, **kwargs):
        if self._handles:
            raise AssertionError("optimizer.zero_grad() was called after loss.backward() but before optimizer.step() or "
                                 "optimizer.synchronize(). This is prohibited as it can cause a race condition.")
        return super().zero_grad(*args, **kwargs)


def DistributedOptimizer(optimizer, named_parameters=None, compression=Compression.none, backward_passes_per_step=1,
                         op=Average, gradient_predivide_factor=1.0, num_groups=0, groups=None, sparse_as_dense=False,
                         process_set=global_process_set, fused=False, zero_copy=None, bucket_cap_mb=32, bucket_wire_dtype=None,
                         shard_optimizer_state=False, master_weights=False, grad_accumulation_dtype=None, ema_decay=None):
    """Wraps `optimizer` so gradients are combined across ranks before the parameter update.

    Arguments follow the reference (horovod/torch/optimizer.py:516-608). `fused=True` (new) runs the SGD /
    Adam(W) update as one multi-tensor CUDA kernel, and hvd.Lamb, hvd.Lars and torch.optim.Adafactor in a few.

    torch.optim.Adafactor (fused): torch's update and state keys (step, row_var [..., R, 1] and col_var [..., 1, C] for
    a parameter of dim >= 2, at most 5 dims, else variance), so checkpoints load both ways, with three differences: the
    state is fp32 for every parameter dtype (torch keeps the gradient dtype); for bf16 / fp16 parameters without
    masters the decay and the update are one fp32 expression rounded once (torch rounds twice); and maximize=True stays
    on torch's own step.  No host synchronisation and no model-sized temporary.  Not with shard_optimizer_state.

    `shard_optimizer_state=True` (new, ZeRO stage 1) keeps the optimizer state of 1/N of the parameters on each of the N
    ranks: gradients are reduce-scattered, each rank updates its shard with the fused kernel and the parameters are
    allgathered (see horovod_b200/torch/sharded_optimizer.py).  SGD / Adam / AdamW / Lamb / Lars with op Average or Sum
    on one host; raises ValueError otherwise.  The sharded update always runs the fused kernel, whatever `fused` says.  With one
    rank it is the ordinary optimizer.

    `master_weights=True` (new) gives every bf16 / fp16 trainable parameter an fp32 master copy, held as optimizer state
    ('master_param', sharded like the moments with shard_optimizer_state): the update runs in fp32 on the master and the
    parameter receives it rounded to nearest-even, so updates smaller than half an ulp of the parameter are not lost.
    SGD momentum is then fp32 as well.  fp32 parameters are unaffected.  Implies fused=True; SGD / Adam / AdamW / Lamb /
    Lars / Adafactor only, without maximize, amsgrad or op=Adasum (ValueError).  A parameter written from outside the optimizer
    (load_state_dict, broadcast_parameters, an in-place edit) is picked up by the next step: where it no longer equals
    its rounded master, the master restarts from it.

    `grad_accumulation_dtype=torch.float32` (new; default None) sums the bf16 / fp16 gradients of the
    `backward_passes_per_step` backward passes of one step in fp32: after each pass the gradient is folded into an fp32
    accumulator and zeroed, and after the last pass it holds the sum rounded once, which is what is reduced and applied.
    Between passes p.grad holds the current pass's gradient only.  fp32 gradients and backward_passes_per_step == 1 are
    unaffected.  The accumulators (one flat buffer per zero-copy bucket, else one per parameter) are allocated on first
    use and are not optimizer state: checkpoints are taken between steps.  Not with op=Adasum (ValueError).

    `ema_decay=d` (new; default None) keeps an fp32 exponential moving average of every trainable parameter as optimizer
    state ('ema_param', sharded like the moments with shard_optimizer_state), written by the same fused kernel launch
    that updates the parameter: e = x at a parameter's first update, then e = fmaf(w, x - e, e) in fp32 with
    w = float32(1 - d), where x is the fp32 master with master_weights, else the value stored into the parameter.  The
    EMA advances only in a step that updates the parameter (not in a step the GradScaler skips, nor for a parameter
    without a gradient in an unsharded step); a clipped step advances it toward the clipped update.  d is stored as
    group['ema_decay'] and read at every step like 'lr', so a schedule (warm-up) may change it; 0 <= d <= 1, else
    ValueError.  `with optimizer.ema_parameters(): ...` evaluates the EMA model.  Buffers (BatchNorm running statistics)
    are not averaged.  Implies fused=True; SGD / Adam / AdamW / Lamb / Lars / Adafactor only, without maximize, amsgrad or op=Adasum
    (ValueError); a step whose update cannot be fused raises RuntimeError."""
    check_grad_accumulation_dtype(grad_accumulation_dtype)
    check_ema_decay(ema_decay)
    if grad_accumulation_dtype is not None and op == Adasum:
        raise ValueError('grad_accumulation_dtype is not supported with op=Adasum')
    for what, on in (('master_weights', master_weights), ('ema_decay', ema_decay is not None)):
        if not on:
            continue
        if op == Adasum:
            raise ValueError('%s is not supported with op=Adasum' % what)
        if _optimizer_kind(optimizer) is None:
            raise ValueError('%s supports SGD, Adam and AdamW, hvd.Lamb and hvd.Lars, and torch.optim.Adafactor, only, '
                             'not %s' % (what, type(optimizer).__name__))
        for g in optimizer.param_groups:
            if g.get('maximize', False) or g.get('amsgrad', False):
                raise ValueError('%s does not support maximize=True or amsgrad=True' % what)
        fused = True
    if gradient_predivide_factor != 1.0:
        if rocm_built_safe():
            raise ValueError('gradient_predivide_factor not supported yet with ROCm')
        if op != Average:
            raise ValueError('gradient_predivide_factor not supported with op != Average')
    if num_groups != 0:
        warnings.warn('Parameter `num_groups` has been replaced by `groups` and will be removed', DeprecationWarning)
        if groups is None:
            groups = num_groups
    if shard_optimizer_state and (process_set.size() or 1) > 1:
        if bucket_wire_dtype is not None or zero_copy is False:
            raise ValueError('shard_optimizer_state keeps its buckets in registered memory in the parameter dtype: '
                             'bucket_wire_dtype and zero_copy=False are not supported')
        from horovod_b200.torch.sharded_optimizer import _ShardedDistributedOptimizer
        cls = type(optimizer.__class__.__name__, (_ShardedDistributedOptimizer, optimizer.__class__), {})
        return cls(optimizer.param_groups, named_parameters, compression, backward_passes_per_step, op,
                   gradient_predivide_factor, groups, sparse_as_dense, process_set, bucket_cap_mb, master_weights,
                   grad_accumulation_dtype, ema_decay)
    if op != Adasum or size() == 1:
        cls = type(optimizer.__class__.__name__, (_DistributedOptimizer, optimizer.__class__), {})
        return cls(optimizer.param_groups, named_parameters, compression, backward_passes_per_step, op,
                   gradient_predivide_factor, groups, sparse_as_dense, process_set, fused, zero_copy, bucket_cap_mb, bucket_wire_dtype,
                   master_weights, grad_accumulation_dtype, ema_decay)
    if process_set != global_process_set:
        raise NotImplementedError("Adasum does not support non-global process sets yet.")
    cls = type(optimizer.__class__.__name__, (_DistributedAdasumOptimizer, optimizer.__class__), {})
    return cls(optimizer.param_groups, named_parameters, compression, backward_passes_per_step)


def rocm_built_safe():
    try:
        return mpi_ops.rocm_built()
    except Exception:
        return False
