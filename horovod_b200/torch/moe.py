"""Expert-parallel dispatch and combine for mixture-of-experts layers (hvd.ExpertDispatcher).

Each rank of a process set of N ranks holds num_experts / N experts.  `dispatch` sends every token's row to the ranks
of its top-k experts and hands each rank its received rows grouped by local expert; `combine` sends the expert outputs
back and sums them per token, weighted by the gates.  Both are differentiable, and every step runs on the current CUDA
stream with no host synchronisation, so a training step containing the layer can be one hvd.GraphedStep replay.

Per rank, the forward dispatch is four launches and two exchanges: moe_permute (the stable order of the [T, k]
assignments by expert, the per-expert counts and per-rank splits, and the copy of each token's row to its k rows of
the registered send buffer), the captured alltoall of the counts, the captured alltoall of the rows, and moe_regroup
(rows grouped by source rank to rows grouped by local expert).  The forward combine is moe_regroup_reverse into the
registered return buffer, the captured alltoall back to the senders and moe_gather (the weighted sum per token).  The
backwards run the same kernels in reverse.  The data movement is in horovod_b200/csrc/kernels/moe_kernels.cu, the
exchanges are hvd.captured_alltoall's kernel.
"""
import torch
from torch.autograd.function import Function

from horovod_b200 import ops
from horovod_b200.common.exceptions import HorovodInternalError
from horovod_b200.torch.mpi_ops import captured_alltoall, global_process_set, symm_available, symm_empty

_DTYPES = (torch.float32, torch.bfloat16, torch.float16)
_MAX_EXPERTS, _MAX_TOP_K = 1024, 16  # kern::kMoeMaxExperts, kern::kMoeMaxTopK
_INT32_MAX, _INT64_MAX = 2 ** 31 - 1, 2 ** 63 - 1


def _symm_empty(shape, dtype, device, process_set):
    """A registered tensor of the dispatcher (collective)."""
    if not symm_available(process_set):
        raise HorovodInternalError('ExpertDispatcher needs a peer-mapped process set of more than one rank '
                                   '(hvd.symm_available)')
    return symm_empty(shape, dtype=dtype, device=device, process_set=process_set)


def _alltoall(tensor, splits, capacity, process_set, max_ctas):
    """Every exchange of the dispatcher: hvd.captured_alltoall on the current stream, barrier channel 5."""
    return captured_alltoall(tensor, splits, capacity, process_set=process_set, max_ctas=max_ctas)


class DispatchHandle:
    """What `combine` and the backwards need from one `dispatch`: pos (int32 [T, k], the send-buffer row of each
    assignment), splits (int32 [N], the rows sent to each rank), recv_counts (int64 [N, E_local], the rows received from
    each rank for each local expert) and status (int32 [1], the exchange's verdict, the same on every rank).  None of
    them is a view of registered memory."""

    def __init__(self, dispatcher, tokens, pos, splits, recv_counts, status):
        self.dispatcher, self.tokens = dispatcher, tokens
        self.pos, self.splits, self.recv_counts, self.status = pos, splits, recv_counts, status


class ExpertDispatcher:
    """Dispatch and combine of an expert-parallel mixture-of-experts layer.  COLLECTIVE: every rank of `process_set`
    builds it with the same arguments.

        disp = hvd.ExpertDispatcher(num_experts, hidden, dtype, max_tokens, top_k, capacity)
        expert_in, offsets, handle = disp.dispatch(x, expert_idx)    # differentiable in x
        y = disp.combine(expert_out, gates, handle)                  # differentiable in expert_out and gates

    With N ranks, E_local = num_experts / N (it must divide exactly): global expert e lives on rank e // E_local as local
    expert e % E_local.

    dispatch(x, expert_idx): x [T, hidden] of `dtype` on this device, T <= max_tokens (T = 0 is allowed);
    expert_idx int32 / int64 [T, top_k] with values in [0, num_experts).  Returns expert_in [capacity, hidden], the
    received rows grouped by local expert, then by source rank, then in the sender's order (within a rank, assignment
    t * top_k + j ascending), zero past the received total; offsets, int32 [E_local], the end row of each group
    (torch._grouped_mm's `offs`); and the handle for `combine`.

    combine(expert_out, gates, handle): expert_out [capacity, hidden] of `dtype` in expert_in's layout; gates
    [T, top_k], fp32 or `dtype`.  Returns y [T, hidden] of `dtype`, y[t] = sum_j gates[t, j] * (the expert output of
    token t's slot j), computed in fp32 with j ascending and rounded once.  The gate gradient is an fp32 dot per slot.
    Every result is bit-identical from run to run; no reduction uses floating-point atomics.

    Failure: handle.status (int32 [1] on the device) is the same on every rank: ALLTOALL_RECV_OVERFLOW (3) when some
    rank would receive more than `capacity` rows, ALLTOALL_NEGATIVE_SPLIT (1) when an expert id is out of range.  Then
    every later exchange of that dispatch moves no rows, expert_in, offsets, y and every gradient are zeros, and the
    next call works normally.  Nothing raises on the device path; argument errors the host can see raise
    HorovodInternalError before anything is launched.

    Memory: the registered (hvd.symm_empty) buffers are allocated once, here: the send buffer of max_tokens * top_k
    rows, the return buffer of `capacity` rows and an int64 [N, E_local] counts buffer.  Registered memory is only
    released by hvd.shutdown().  One dispatcher can serve every MoE layer with the same hidden size and dtype: each
    exchange ends every peer's read of these buffers before it returns, so the next write, later in stream order, is
    safe.

    Contract (as for the other captured collectives): every rank issues dispatch, combine and their backwards in the
    same order with the same `max_ctas` (autograd does this on its own).  The exchanges run on barrier channel 5, like
    hvd.captured_alltoall, so they can run next to hvd.GraphedStep's gradient allreduces.

    Training an MoE model: the expert parameters differ from rank to rank, so keep them out of DistributedOptimizer and
    give them to a local optimizer.  DistributedOptimizer's default op=Average divides the dense gradients by N; divide
    the expert gradients by N too (for example with a hook, or a learning rate N times smaller) to optimise the same
    objective."""

    def __init__(self, num_experts, hidden, dtype, max_tokens, top_k, capacity, process_set=global_process_set,
                 max_ctas=0):
        for name, v in (('num_experts', num_experts), ('hidden', hidden), ('max_tokens', max_tokens), ('top_k', top_k),
                        ('capacity', capacity), ('max_ctas', max_ctas)):
            if not isinstance(v, int) or isinstance(v, bool):
                raise HorovodInternalError('ExpertDispatcher: %s must be an int, got %r' % (name, v))
        if dtype not in _DTYPES:
            raise HorovodInternalError('ExpertDispatcher: dtype must be float32, bfloat16 or float16, got %s' % (dtype,))
        if not 1 <= num_experts <= _MAX_EXPERTS:
            raise HorovodInternalError('ExpertDispatcher: num_experts must be in [1, %d], got %d' % (_MAX_EXPERTS, num_experts))
        if not 1 <= top_k <= _MAX_TOP_K:
            raise HorovodInternalError('ExpertDispatcher: top_k must be in [1, %d], got %d' % (_MAX_TOP_K, top_k))
        if hidden < 1 or max_tokens < 1 or capacity < 1 or max_ctas < 0:
            raise HorovodInternalError('ExpertDispatcher: hidden, max_tokens and capacity must be >= 1 and max_ctas >= 0')
        n = process_set.size()
        if n is None:
            raise HorovodInternalError('ExpertDispatcher: horovod is not initialized, or this rank is not in the process set')
        if num_experts % n != 0:
            raise HorovodInternalError('ExpertDispatcher: num_experts (%d) must be a multiple of the process set size (%d)'
                                       % (num_experts, n))
        itemsize = torch.empty(0, dtype=dtype).element_size()
        rows = max(max_tokens * top_k, capacity)
        if rows > _INT32_MAX or rows * hidden * itemsize > _INT64_MAX:
            raise HorovodInternalError('ExpertDispatcher: max_tokens * top_k and capacity must be below 2^31 rows, and '
                                       'every buffer below 2^63 bytes')
        self.num_experts, self.hidden, self.dtype = num_experts, hidden, dtype
        self.max_tokens, self.top_k, self.capacity = max_tokens, top_k, capacity
        self.process_set, self.max_ctas = process_set, max_ctas
        self.nranks, self.experts_per_rank = n, num_experts // n
        self.device = torch.device('cuda', torch.cuda.current_device())
        self._send = _symm_empty((max_tokens * top_k, hidden), dtype, self.device, process_set)
        self._ret = _symm_empty((capacity, hidden), dtype, self.device, process_set)
        self._counts = _symm_empty((n, self.experts_per_rank), torch.int64, self.device, process_set)
        self._count_splits = torch.full((n,), self.experts_per_rank, dtype=torch.int32, device=self.device)

    def _check(self, what, t, shape, dtypes):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != self.device:
            raise HorovodInternalError('ExpertDispatcher: %s must be a CUDA tensor on %s' % (what, self.device))
        if tuple(t.shape) != tuple(shape):
            raise HorovodInternalError('ExpertDispatcher: %s must have shape %s, got %s' % (what, list(shape), list(t.shape)))
        if t.dtype not in dtypes:
            raise HorovodInternalError('ExpertDispatcher: %s must be %s, got %s' % (what, ' or '.join(map(str, dtypes)), t.dtype))
        if not t.is_contiguous():
            raise HorovodInternalError('ExpertDispatcher: %s must be contiguous' % what)

    def dispatch(self, x, expert_idx):
        """Returns (expert_in, offsets, handle); see the class docstring."""
        if not isinstance(x, torch.Tensor) or x.dim() != 2:
            raise HorovodInternalError('ExpertDispatcher: x must be a 2-D tensor [tokens, hidden]')
        t = x.shape[0]
        if t > self.max_tokens:
            raise HorovodInternalError('ExpertDispatcher: %d tokens exceed max_tokens (%d)' % (t, self.max_tokens))
        self._check('x', x, (t, self.hidden), (self.dtype,))
        self._check('expert_idx', expert_idx, (t, self.top_k), (torch.int32, torch.int64))
        expert_in, offsets, pos, splits, recv_counts, status = _Dispatch.apply(x, expert_idx, self)
        return expert_in, offsets, DispatchHandle(self, t, pos, splits, recv_counts, status)

    def combine(self, expert_out, gates, handle):
        """Returns y [T, hidden]; see the class docstring."""
        if not isinstance(handle, DispatchHandle) or handle.dispatcher is not self:
            raise HorovodInternalError('ExpertDispatcher: handle must come from this dispatcher\'s dispatch')
        self._check('expert_out', expert_out, (self.capacity, self.hidden), (self.dtype,))
        self._check('gates', gates, (handle.tokens, self.top_k), tuple({torch.float32, self.dtype}))
        return _Combine.apply(expert_out, gates, handle.pos, handle.splits, handle.recv_counts, handle.status, self)

    # ---- the steps, shared by the forwards and the backwards ----
    def _exchange(self, tensor, splits, capacity):
        out, _, status = _alltoall(tensor, splits, capacity, self.process_set, self.max_ctas)
        return out, status

    def _to_experts(self, received, recv_counts, status):
        """Rows grouped by source rank -> grouped by local expert, zero tail; (rows, offsets)."""
        return ops.moe_regroup(received, recv_counts, status, out=received if self.experts_per_rank == 1 else None,
                               ctas=self.max_ctas)

    def _back_to_senders(self, expert_rows, recv_counts, status):
        """Rows grouped by local expert -> the senders, lined up with their send buffers' rows."""
        ret_splits = ops.moe_regroup_reverse(expert_rows, recv_counts, self._ret, status, ctas=self.max_ctas)
        out, _ = self._exchange(self._ret, ret_splits, self._send.shape[0])
        return out


class _Dispatch(Function):
    @staticmethod
    def forward(ctx, x, expert_idx, d):
        pos, splits = ops.moe_permute(x, expert_idx, d.num_experts, d.nranks, d._send, d._counts.view(-1), ctas=d.max_ctas)
        recv_counts, _ = d._exchange(d._counts.view(-1), d._count_splits, d.num_experts)
        recv_counts = recv_counts.view(d.nranks, d.experts_per_rank)
        received, status = d._exchange(d._send, splits, d.capacity)
        expert_in, offsets = d._to_experts(received, recv_counts, status)
        ctx.save_for_backward(pos, recv_counts, status)
        ctx.d = d
        ctx.mark_non_differentiable(offsets, pos, splits, recv_counts, status)
        return expert_in, offsets, pos, splits, recv_counts, status

    @staticmethod
    def backward(ctx, grad_expert_in, *_):
        if grad_expert_in is None:
            return None, None, None
        pos, recv_counts, status = ctx.saved_tensors
        d = ctx.d
        back = d._back_to_senders(grad_expert_in.contiguous(), recv_counts, status)
        return ops.moe_gather(back, pos, status=status, ctas=d.max_ctas), None, None


class _Combine(Function):
    @staticmethod
    def forward(ctx, expert_out, gates, pos, splits, recv_counts, status, d):
        back = d._back_to_senders(expert_out, recv_counts, status)
        y = ops.moe_gather(back, pos, gates, status, ctas=d.max_ctas)
        ctx.save_for_backward(back, gates, pos, splits, recv_counts, status)
        ctx.d = d
        return y

    @staticmethod
    def backward(ctx, grad_y):
        back, gates, pos, splits, recv_counts, status = ctx.saved_tensors
        d = ctx.d
        # gates[t, j] * grad_y[t] straight into the send buffer, and the gate gradient against the returned rows
        grad_gates = ops.moe_scatter(grad_y.contiguous(), pos, d._send, gates,
                                     back if ctx.needs_input_grad[1] else None, status, ctas=d.max_ctas)
        grad_expert_out = None
        if ctx.needs_input_grad[0]:
            # the forward splits: after a failed dispatch this exchange fails the same way and moves no rows
            received, _ = d._exchange(d._send, splits, d.capacity)
            grad_expert_out, _ = d._to_experts(received, recv_counts, status)
        return grad_expert_out, grad_gates, None, None, None, None, None
