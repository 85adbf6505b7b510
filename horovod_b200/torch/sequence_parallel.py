"""Ulysses sequence parallelism (hvd.UlyssesExchange): the exchange between sequence shards and head shards around the
attention of a model whose sequence is sharded over the ranks of a process set.

Each exchange is one sm_90a kernel (horovod_b200/csrc/kernels/ulysses_kernels.cu) on the current CUDA stream, with no
host synchronisation and no negotiation, so a training step containing it can be one hvd.GraphedStep replay.  The
kernel stages this rank's input into a registered buffer, writes its own block straight into the output and pulls
the peers' blocks from their staging buffers over NVLink, with the change of layout folded into the copies: no
permute().contiguous() before or after.
"""
import torch
from torch.autograd.function import Function

from horovod_b200.common.exceptions import HorovodInternalError
from horovod_b200.torch.mpi_ops import _native, global_process_set, symm_available, symm_empty

_DTYPES = (torch.float32, torch.bfloat16, torch.float16)
SEQ_TO_HEADS, HEADS_TO_SEQ = 0, 1  # kern::UlyssesDirection


def _symm_empty(numel, dtype, device, process_set):
    """The registered staging buffer (collective)."""
    if not symm_available(process_set):
        raise HorovodInternalError('UlyssesExchange needs a peer-mapped process set of more than one rank '
                                   '(hvd.symm_available)')
    return symm_empty(numel, dtype=dtype, device=device, process_set=process_set)


def _exchange(tensor, staging, status, seq_dim, head_dim, direction, process_set, max_ctas):
    """Every launch of UlyssesExchange: the kernel on the current stream, barrier channel 5.  Returns the output."""
    try:
        return _native().captured_ulysses_exchange(tensor, staging, status, seq_dim, head_dim, direction, process_set.size(),
                                                   process_set.process_set_id, max_ctas)
    except (RuntimeError, ValueError, TypeError) as e:
        raise HorovodInternalError(e)


class UlyssesExchange:
    """Sequence shards <-> head shards for Ulysses sequence parallelism.  COLLECTIVE: every rank of `process_set`
    builds it with the same arguments.

        ex = hvd.UlyssesExchange(max_numel, dtype)
        y = ex.seq_to_heads(x, seq_dim, head_dim)    # differentiable
        x = ex.heads_to_seq(y, seq_dim, head_dim)    # differentiable, the inverse

    With N ranks, rank `me` and x_p the argument of rank p (a contiguous CUDA tensor of `dtype` with at most
    `max_numel` elements; seq_dim and head_dim two distinct dims, in either order):

    - seq_to_heads(x) needs x.shape[head_dim] % N == 0 and returns
      torch.cat([x_p.chunk(N, head_dim)[me] for p in range(N)], dim=seq_dim): from this rank's sequence shard with all
      heads to the whole sequence with H / N heads.
    - heads_to_seq(y) needs y.shape[seq_dim] % N == 0 and returns
      torch.cat([y_p.chunk(N, seq_dim)[me] for p in range(N)], dim=head_dim).

    Each is the other's inverse and the other's backward.  The outputs are byte copies of the inputs, allocated on the
    current stream; nothing saved for backward is a view of registered memory.  A fused QKV tensor [B, S/N, 3, H, D]
    (seq_dim=1, head_dim=3) goes through in one call; GQA takes two (q, then k and v stacked).

    A sequence-parallel attention block, with the tokens and positions of rank r being its S/N slice of the sequence
    and the weights replicated:

        qkv = self.qkv(x).view(B, S // N, 3, H, D)                     # this rank's tokens, every head
        q, k, v = ex.seq_to_heads(qkv, 1, 3).unbind(2)                 # [B, S, H/N, D]: every token, H/N heads
        o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=True)
        o = ex.heads_to_seq(o.transpose(1, 2).contiguous(), 1, 2)      # [B, S/N, H, D]: this rank's tokens again
        out = self.proj(o.reshape(B, S // N, H * D))

    Wrap the optimizer in hvd.DistributedOptimizer over the same process set: it averages the replicated weights'
    gradients exactly as for data parallelism (each rank's gradient covers its own tokens).

    Failure: `status` (int32 [1] on the device) keeps the first non-zero code since the last `status.zero_()`, the same
    on every rank: ALLTOALL_ROW_BYTES_MISMATCH (4) when the ranks' shapes differ (that call pulls nothing and its
    output is zeros; the next call works), ALLTOALL_ABORTED (5) when a peer never arrived.  Check it once per step
    instead of synchronising after every call; the reset can be captured into a graph.  Argument errors the host can
    see raise HorovodInternalError before anything is launched.

    Memory: one registered (hvd.symm_empty) staging buffer of max_numel elements, allocated here and released only by
    hvd.shutdown().  One object can serve every layer: each exchange ends every peer's read of the buffer before it
    returns.

    Contract (as for the other captured collectives): every rank issues the same exchanges in the same order with the
    same `max_ctas` (autograd does this on its own for the backwards).  The exchanges run on barrier channel 5 and share
    its count region with hvd.captured_alltoall and hvd.ExpertDispatcher, so a process set's calls of the three must
    be issued in one stream order."""

    def __init__(self, max_numel, dtype, process_set=global_process_set, max_ctas=0):
        for name, v in (('max_numel', max_numel), ('max_ctas', max_ctas)):
            if not isinstance(v, int) or isinstance(v, bool):
                raise HorovodInternalError('UlyssesExchange: %s must be an int, got %r' % (name, v))
        if dtype not in _DTYPES:
            raise HorovodInternalError('UlyssesExchange: dtype must be float32, bfloat16 or float16, got %s' % (dtype,))
        if max_numel < 1 or max_ctas < 0:
            raise HorovodInternalError('UlyssesExchange: max_numel must be >= 1 and max_ctas >= 0')
        n = process_set.size()
        if n is None:
            raise HorovodInternalError('UlyssesExchange: horovod is not initialized, or this rank is not in the process set')
        self.max_numel, self.dtype, self.process_set, self.max_ctas, self.nranks = max_numel, dtype, process_set, max_ctas, n
        self.device = torch.device('cuda', torch.cuda.current_device())
        self._staging = _symm_empty(max_numel, dtype, self.device, process_set)
        self.status = torch.zeros(1, dtype=torch.int32, device=self.device)

    def _dims(self, x, seq_dim, head_dim, split):
        if not isinstance(x, torch.Tensor) or not x.is_cuda or x.device != self.device:
            raise HorovodInternalError('UlyssesExchange: the input must be a CUDA tensor on %s' % (self.device,))
        if x.dtype != self.dtype:
            raise HorovodInternalError('UlyssesExchange: the input must be %s, got %s' % (self.dtype, x.dtype))
        if not x.is_contiguous():
            raise HorovodInternalError('UlyssesExchange: the input must be contiguous')
        if x.numel() > self.max_numel:
            raise HorovodInternalError('UlyssesExchange: %d elements exceed max_numel (%d)' % (x.numel(), self.max_numel))
        nd = x.dim()
        dims = []
        for name, d in (('seq_dim', seq_dim), ('head_dim', head_dim)):
            if not isinstance(d, int) or isinstance(d, bool) or not -nd <= d < nd:
                raise HorovodInternalError('UlyssesExchange: %s must be a dim of a %d-D tensor, got %r' % (name, nd, d))
            dims.append(d % nd)
        if dims[0] == dims[1]:
            raise HorovodInternalError('UlyssesExchange: seq_dim and head_dim must differ, both are %d' % dims[0])
        d = dims[1] if split == 'head' else dims[0]
        if x.shape[d] % self.nranks:
            raise HorovodInternalError('UlyssesExchange: the %s dim (%d, size %d) must be a multiple of the process set '
                                       'size (%d)' % (split, d, x.shape[d], self.nranks))
        return dims

    def seq_to_heads(self, x, seq_dim, head_dim):
        """Sequence shard, every head -> every token, this rank's heads; see the class docstring."""
        s, h = self._dims(x, seq_dim, head_dim, 'head')
        return _Exchange.apply(x, self, s, h, SEQ_TO_HEADS)

    def heads_to_seq(self, y, seq_dim, head_dim):
        """Every token, this rank's heads -> sequence shard, every head; see the class docstring."""
        s, h = self._dims(y, seq_dim, head_dim, 'seq')
        return _Exchange.apply(y, self, s, h, HEADS_TO_SEQ)

    def _launch(self, x, seq_dim, head_dim, direction):
        return _exchange(x, self._staging, self.status, seq_dim, head_dim, direction, self.process_set, self.max_ctas)


class _Exchange(Function):
    @staticmethod
    def forward(ctx, x, ex, seq_dim, head_dim, direction):
        ctx.ex, ctx.dims, ctx.direction = ex, (seq_dim, head_dim), direction
        return ex._launch(x, seq_dim, head_dim, direction)

    @staticmethod
    def backward(ctx, grad):
        back = HEADS_TO_SEQ if ctx.direction == SEQ_TO_HEADS else SEQ_TO_HEADS
        return ctx.ex._launch(grad.contiguous(), *ctx.dims, back), None, None, None, None
