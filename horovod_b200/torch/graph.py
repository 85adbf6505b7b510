"""CUDA-graph training step: forward + backward captured once, replayed every step; gradients are reduced and the
(fused) optimizer applied right after the replay.

Why (nothing like it exists in the reference): a ResNet-50 / BERT step in eager PyTorch issues 1–3 thousand
kernel launches, and a GPU such as the H100 can finish them faster than one Python thread issues them — the step
time then is the host's launch time.  Replaying the step as ONE graph launch removes that bound.
On several GPUs the gradient allreduce is PART of the graph: while the step is being captured, the hook of the last
gradient of every zero-copy bucket records that bucket's `hvd.captured_allreduce_` kernel (multimem / P2P in-place
reduction on peer-mapped memory, flag barrier inside the kernel) on a forked high-priority stream, so on replay the
reduction of bucket k overlaps the backward pass of the layers below it, and a whole data-parallel step — forward,
backward, every collective — is ONE launch with no negotiation round and no host work.  `optimizer.step()` after the
replay only applies the (fused) update.  If some trainable parameter is not in a registered bucket (sparse gradients,
`zero_copy=False`, compression, `groups`) the reductions stay outside the graph and `step()` issues them as before.

    step = hvd.GraphedStep(lambda x, y: F.cross_entropy(model(x), y), optimizer, (x0, y0))
    for x, y in loader:
        loss = step(x, y)          # copies x, y into the static inputs, replays, allreduces, applies the update

Gradient accumulation: with `backward_passes_per_step=k > 1` every call is one micro-batch (divide the loss by k inside
`step_fn`, as in the eager idiom) and `optimizer.step()` runs after every k-th call only.  Up to three graphs share one
memory pool and the static inputs: the first micro-step's (zero_grad + forward/backward), the middle ones' (k >= 3) and
the last one's, which also holds the gradient collectives where they can be captured.  With
`grad_accumulation_dtype=torch.float32` each graph ends with its fold of the bf16 / fp16 gradients into the fp32
accumulators (in the last graph, each bucket's fold precedes its collective).  k is fixed when the step is built.
As with k = 1, a call returns the static loss tensor of the graph it replayed, which that graph's next replay
overwrites; the middle graph serves micro-steps 2 … k-1, so `.clone()` (or `.item()`) a loss that must outlive the
next call.

Gradient clipping and AMP loss scaling: `max_grad_norm=` clips the global norm (`norm_type` 2 or inf) of the reduced
gradients before each optimizer step, and `scaler=` (a torch.amp.GradScaler, or hvd.ShardedGradScaler with sharded
optimizer state) scales the loss that every captured backward pass differentiates.  The update itself stays outside
the graph; after the last backward pass of a step the call runs the documented sequence

    optimizer.synchronize()                       # with a scaler: unscale_ reads the reduced gradients
    scaler.unscale_(optimizer)                    # with a scaler
    optimizer.clip_grad_norm_(max_grad_norm)      # with max_grad_norm: one statistics pass, no host sync
    with optimizer.skip_synchronize():
        scaler.step(optimizer)                    # or optimizer.step()
    scaler.update()                               # with a scaler

The graph reads the scale from the scaler's device tensor, which update() rewrites in place, so every replay uses the
current scale; the returned loss is the unscaled one.  scaler.step() reads the inf / NaN verdict on the host, as torch
does: one host synchronisation per step with a scaler, none with clipping alone.  A step the scaler skips leaves no
clip coefficient or gradient statistics behind.  Not with op=Adasum, whose optimizer reduces parameter deltas rather
than gradients (ValueError).

Constraints (those of CUDA graphs): fixed input shapes/dtypes, no host synchronisation or data-dependent control flow
inside `step_fn`, `optimizer.zero_grad()` is part of the graph (do not call it yourself).  If capture fails the object
falls back to the eager step and says so in `.captured` / `.fallback_reason`.
"""
import math
import warnings

import torch

from horovod_b200.torch.mpi_ops import Adasum
from horovod_b200.torch.optimizer import _DistributedAdasumOptimizer, _DistributedOptimizerBase


class GraphedStep:
    """Training step whose forward + backward are one CUDA graph replay; `step(*inputs)` returns the (static) loss tensor.
    `.captured` tells whether the graph is in use, `.fallback_reason` why not.  `max_grad_norm` / `norm_type`: clip the
    global gradient norm before every optimizer step; `scaler`: AMP loss scaling (see the module docstring)."""

    def __init__(self, step_fn, optimizer, example_inputs, warmup_iters=3, enabled=True, max_grad_norm=None,
                 norm_type=2.0, scaler=None):
        self._check_clip_and_scaler(optimizer, max_grad_norm, norm_type, scaler)
        self.step_fn, self.optimizer = step_fn, optimizer
        self.max_grad_norm, self.norm_type, self.scaler = max_grad_norm, float(norm_type), scaler
        self.captured, self.fallback_reason = False, None
        self.graph, self.static_loss = None, None
        # backward_passes_per_step when built; k > 1: one graph and static loss per phase, replayed first, middle..., last
        self.k = int(getattr(optimizer, 'backward_passes_per_step', 1) or 1)
        self.graphs, self.static_losses = None, None
        self.micro_step = 0  # micro-batches of the current optimizer step already run
        self.comm_in_graph = False  # True: the gradient allreduces are kernel nodes of the captured graph
        self.static_inputs = tuple(example_inputs)
        self.replays = 0
        if not enabled:
            self.fallback_reason = 'disabled'
        elif not (torch.cuda.is_available() and all(t.is_cuda for t in example_inputs)):
            self.fallback_reason = 'inputs are not CUDA tensors'
        elif not isinstance(optimizer, (_DistributedOptimizerBase, _DistributedAdasumOptimizer)):
            self.fallback_reason = 'optimizer is not an hvd.DistributedOptimizer'
        else:
            try:
                self._capture(warmup_iters)
            except Exception as e:  # noqa: BLE001 - any capture failure must leave a working eager step behind
                self._abandon(e)
            self._agree_across_ranks()

    @staticmethod
    def _check_clip_and_scaler(optimizer, max_grad_norm, norm_type, scaler):
        if float(norm_type) not in (2.0, math.inf):
            raise ValueError('hvd.GraphedStep: norm_type must be 2 or inf, got %r' % (norm_type,))
        if max_grad_norm is None and scaler is None:
            return
        if isinstance(optimizer, _DistributedAdasumOptimizer) or (isinstance(optimizer, _DistributedOptimizerBase)
                                                                   and optimizer.op == Adasum):
            raise ValueError('hvd.GraphedStep: max_grad_norm and scaler are not supported with op=Adasum, whose optimizer '
                             'reduces parameter deltas, not gradients')
        if not isinstance(optimizer, _DistributedOptimizerBase):
            raise ValueError('hvd.GraphedStep: max_grad_norm and scaler need an hvd.DistributedOptimizer')
        if scaler is not None and not all(p.is_cuda for g in optimizer.param_groups for p in g['params']):
            raise ValueError('hvd.GraphedStep: scaler needs an optimizer of CUDA parameters')

    # ------------------------------------------------------------------------------------------------------------------
    def _backward(self, loss):
        (loss if self.scaler is None else self.scaler.scale(loss)).backward()

    def _fwd_bwd(self, zero_grad=True):
        if zero_grad:
            self.optimizer.zero_grad(set_to_none=False)
        loss = self.step_fn(*self.static_inputs)
        self._backward(loss)
        return loss

    def _capture(self, warmup_iters):
        opt = self.optimizer
        reduces = isinstance(opt, _DistributedOptimizerBase)  # the Adasum optimizer reduces in step() only
        opt._graph_mode = True
        self.static_inputs = tuple(t.detach().clone(memory_format=torch.preserve_format) for t in self.static_inputs)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup_iters)):  # cuDNN/cuBLAS autotuning, lazy allocations, gradient tensors
                self._fwd_bwd()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        missing = [p for g in opt.param_groups for p in g['params'] if p.requires_grad and p.grad is None]
        for p in missing:  # parameters unused by step_fn still need a static gradient for the optimizer
            p.grad = torch.zeros_like(p, memory_format=torch.preserve_format)
        if self.k > 1:
            self._capture_phases()
            return
        self.graph = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(self.graph):
                # multi-GPU: the gradient buckets' allreduce kernels become nodes of this graph (forked onto a side stream
                # as soon as a bucket's last gradient is recorded, joined before the capture ends)
                self.comm_in_graph = reduces and opt._begin_graph_capture()
                self.static_loss = self._fwd_bwd()
                if self.comm_in_graph:
                    opt._end_graph_capture()
        finally:
            if reduces:
                opt._graph_capture = None
        torch.cuda.synchronize()
        self.captured = True

    def _capture_phases(self):
        """k > 1: the first, middle (k >= 3) and last micro-steps as graphs of one memory pool.  Only the last one
        records the gradient collectives (as the one graph of k == 1 does) and the fp32 accumulation's 'last' folds."""
        opt = self.optimizer
        reduces = isinstance(opt, _DistributedOptimizerBase)
        if reduces:
            opt._prepare_accumulators()
        pool = torch.cuda.graph_pool_handle()
        phases = ('first', 'add', 'last') if self.k >= 3 else ('first', 'last')
        self.graphs, self.static_losses = {}, {}
        for phase in phases:
            graph = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(graph, pool=pool):
                    comm = phase == 'last' and reduces and opt._begin_graph_capture()
                    loss = self._fwd_bwd(zero_grad=phase == 'first')
                    if reduces:  # with comm, each bucket's fold precedes its collective
                        opt._graph_fold(phase, with_buckets=not comm)
                    if comm:
                        opt._end_graph_capture()
            finally:
                if reduces:
                    opt._graph_capture = None
            self.graphs[phase], self.static_losses[phase] = graph, loss
            self.comm_in_graph = self.comm_in_graph or comm
        self.graph, self.static_loss = self.graphs['last'], self.static_losses['last']
        torch.cuda.synchronize()
        self.captured = True

    def _agree_across_ranks(self):
        """A graph with the allreduce kernels inside only works if EVERY rank replays the same graph: if capture failed (or
        chose a different communication mode) anywhere, every rank drops to the eager step."""
        ps = getattr(self.optimizer, 'process_set', None)
        if ps is None or not ps.included() or (ps.size() or 1) <= 1:
            return
        from horovod_b200.torch import mpi_ops
        mine = torch.tensor([1.0 if self.captured else 0.0, 1.0 if self.comm_in_graph else 0.0], dtype=torch.float32)
        lo = mpi_ops.allreduce(mine, op=mpi_ops.Min, name='graphed_step.agree.min', process_set=ps)
        hi = mpi_ops.allreduce(mine, op=mpi_ops.Max, name='graphed_step.agree.max', process_set=ps)
        if self.captured and (lo[0] != hi[0] or lo[1] != hi[1]):
            self._abandon(RuntimeError('CUDA graph capture did not succeed identically on every rank'))

    def _abandon(self, exc):
        self.captured, self.graph, self.comm_in_graph = False, None, False
        self.graphs = self.static_losses = None
        self.optimizer._graph_mode = False
        if isinstance(self.optimizer, _DistributedOptimizerBase):
            self.optimizer._graph_comm_captured = False
        self.fallback_reason = '%s: %s' % (type(exc).__name__, str(exc).splitlines()[0] if str(exc) else '')
        try:
            torch.cuda.synchronize()
        except Exception:  # noqa: BLE001
            pass
        warnings.warn('hvd.GraphedStep: CUDA graph capture failed (%s); running the eager step' % self.fallback_reason)

    # ------------------------------------------------------------------------------------------------------------------
    def __call__(self, *inputs):
        k = int(getattr(self.optimizer, 'backward_passes_per_step', 1) or 1)
        if k != self.k:
            raise RuntimeError('hvd.GraphedStep was built for backward_passes_per_step=%d, the optimizer now has %d: build '
                               'a new GraphedStep after set_backward_passes_per_step()' % (self.k, k))
        if self.k > 1:
            return self._micro_step(inputs)
        if not self.captured:
            self.optimizer.zero_grad()
            loss = self.step_fn(*inputs)
            self._backward(loss)
            self._update()
            return loss
        for dst, src in zip(self.static_inputs, inputs):
            if dst is not src:
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        self.replays += 1
        self._update()
        return self.static_loss

    def _update(self):
        """The optimizer step after the last backward pass of a step, with unscaling and clipping where asked for."""
        opt = self.optimizer
        if self.scaler is None and self.max_grad_norm is None:
            opt.step()
            return
        if self.scaler is not None:
            opt.synchronize()
            self.scaler.unscale_(opt)
        if self.max_grad_norm is not None:
            opt.clip_grad_norm_(self.max_grad_norm, self.norm_type)
        with opt.skip_synchronize():
            if self.scaler is not None:
                self.scaler.step(opt)
            else:
                opt.step()
        if self.scaler is not None:
            self.scaler.update()
        # a step the scaler skipped must not leave its clip coefficient or statistics to the next one: on replay neither
        # a gradient hook nor zero_grad() (a node of the graph) runs Python that would drop them
        opt._drop_iteration_state()

    def _micro_step(self, inputs):
        """One micro-batch of k: the optimizer steps after the k-th.  Returns this micro-batch's loss."""
        first, last = self.micro_step == 0, self.micro_step == self.k - 1
        if not self.captured:
            if first:
                self.optimizer.zero_grad()
            loss = self.step_fn(*inputs)
            self._backward(loss)
        else:
            for dst, src in zip(self.static_inputs, inputs):
                if dst is not src:
                    dst.copy_(src, non_blocking=True)
            phase = 'first' if first else 'last' if last else 'add'
            self.graphs[phase].replay()
            self.replays += 1
            loss = self.static_losses[phase]
        self.micro_step = 0 if last else self.micro_step + 1
        if last:
            self._update()
        return loss
