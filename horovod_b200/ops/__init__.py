"""Python access to the native sm_90a operations that are not collectives of the `hvd.*` API:

* `fused_sgd_step`, `fused_adam_step` — multi-tensor optimizer kernels (`csrc/kernels/optim_kernels.cu`);
* `fused_lamb_step`, and its two phases `lamb_norms` / `lamb_apply` — multi-tensor LAMB with per-tensor trust ratios
  (same file);
* `fused_lars_step`, and its two phases `lars_norms` / `lars_apply` — multi-tensor LARS on LAMB's table and norms
  layout (same file);
* `fused_adafactor_step` — multi-tensor torch.optim.Adafactor with factored second moments (same file);
* `grad_shard_stats` — one-pass gradient norm statistics, non-finite check and optional in-place unscale (same file);
* `grad_accumulate_` — folds bf16 / fp16 gradients into fp32 accumulators for gradient accumulation (same file);
* `sync_bn_stats`, `sync_bn_combine`, `sync_bn_elemt`, `sync_bn_backward_reduce`, `sync_bn_backward_elemt` — the
  kernels of hvd.SyncBatchNorm's native path (`csrc/kernels/sync_bn_kernels.cu`);
* `moe_permute`, `moe_scatter`, `moe_gather`, `moe_regroup`, `moe_regroup_reverse` — the local data movement of
  hvd.ExpertDispatcher (`csrc/kernels/moe_kernels.cu`);
* `symm_empty`, `symm_available` — registered symmetric memory for the zero-copy allreduce path;
* `sim` — the single-GPU simulation harness (N ranks = N concurrently running kernels on one device) used by the
  numerics tests, `bench/kernel_micro.py` and the ncu captures;
* `kernel_launches()` — how many kernels of this library were launched by this process (bench.py's `gpu_launches`).
"""
import torch

from horovod_b200.ops import sim  # noqa: F401


def _native():
    from horovod_b200.torch.mpi_ops import _native as n
    return n()


def _ema(ema_params, ema_decay, ema_start):
    """The native EMA arguments: (fp32 EMA tensors, weight 1 - decay, start).  No EMA: ([], 0.0, False)."""
    if not ema_params:
        return [], 0.0, False
    if ema_decay is None or not 0.0 <= float(ema_decay) <= 1.0:
        raise ValueError('ema_decay must be in [0, 1] with ema_params, got %r' % (ema_decay,))
    return list(ema_params), 1.0 - float(ema_decay), bool(ema_start)


def fused_sgd_step(params, grads, momentum_buffers, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False,
                   grad_scale=1.0, first_step=False, grad_scale_dev=None, master_params=None, ema_params=None, ema_decay=None,
                   ema_start=False):
    """One launch per 65535 non-empty parameters (fp32 / bf16 / fp16 parameters, fp32 or matching gradients).
    `grad_scale_dev`: an optional 1-element fp32 tensor on the parameters' device; the gradients are multiplied by
    grad_scale * grad_scale_dev[0], read by the kernel, so no host synchronisation is needed.

    `master_params`: optional fp32 master copies of bf16 / fp16 parameters (gradients of the parameters' dtype), one per
    parameter with its sizes and strides; momentum buffers are then fp32 too. The update runs on the master and the
    parameter receives it rounded to nearest-even. Where a parameter no longer equals its rounded master (it was
    written from outside, or the master is zero-filled), the master first restarts from the parameter.

    `ema_params`: optional fp32 exponential moving averages, one per parameter with its sizes and strides, updated in the
    same launch after the parameter: e = fmaf(1 - ema_decay, x - e, e) in fp32, with x the updated master if there is
    one, else the value stored into the parameter.  `ema_start=True` begins them: e = x, without reading e.

    A call with more than 65535 non-empty parameters (the grid limit of one launch) stages its table in pieces through a
    fixed host-to-device ring, and filling that ring may wait for the stream: such a call can synchronise with the host
    and cannot be captured into a CUDA graph.  The same holds for fused_adam_step, fused_lamb_step, fused_lars_step and
    their phases."""
    return _native().fused_sgd_step(list(params), list(grads), list(momentum_buffers), float(lr), float(momentum), float(dampening),
                                    float(weight_decay), bool(nesterov), float(grad_scale), bool(first_step), grad_scale_dev,
                                    list(master_params or []), *_ema(ema_params, ema_decay, ema_start))


def fused_adam_step(params, grads, exp_avgs, exp_avg_sqs, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, step=1,
                    grad_scale=1.0, adamw=True, grad_scale_dev=None, master_params=None, ema_params=None, ema_decay=None,
                    ema_start=False):
    """One launch of Adam / AdamW per 65535 non-empty parameters (fp32 / bf16 / fp16 parameters, fp32 or matching
    gradients, fp32 state with the parameters' sizes and strides; `step` is the 1-based step count). Mismatched
    lists, dtypes, sizes, strides or devices raise RuntimeError before anything is launched. `grad_scale_dev`,
    `master_params` and the EMA arguments as in fused_sgd_step."""
    return _native().fused_adam_step(list(params), list(grads), list(exp_avgs), list(exp_avg_sqs), float(lr), float(beta1), float(beta2),
                                     float(eps), float(weight_decay), int(step), float(grad_scale), bool(adamw), grad_scale_dev,
                                     list(master_params or []), *_ema(ema_params, ema_decay, ema_start))


def fused_lamb_step(params, grads, exp_avgs, exp_avg_sqs, lr, beta1, beta2, eps, weight_decay, step, bias_correction=True,
                    adapt=True, grad_scale=1.0, grad_scale_dev=None, master_params=None, ema_params=None, ema_decay=None,
                    ema_start=False):
    """One LAMB step in three launches per 65535 non-empty parameters (moments and per-CTA norm partials, the
    per-tensor norms, the update), with the argument rules of fused_adam_step. For each parameter w (1-based `step`):

        g = grad * grad_scale [* grad_scale_dev[0]];  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2
        u = (m / c1) / (sqrt(v / c2) + eps) + weight_decay * w      (c1 = 1 - b1^step, c2 = 1 - b2^step; 1 without bias_correction)
        w -= lr * r * u,   r = ||w|| / ||u|| if adapt and both norms are > 0, else 1

    The EMA arguments are those of fused_sgd_step; the update launch writes the EMA.
    Deterministic: the same input gives the same bits on every call. Up to 65535 non-empty parameters nothing is
    synchronised with the host (see fused_sgd_step)."""
    return _native().fused_lamb_step(list(params), list(grads), list(exp_avgs), list(exp_avg_sqs), float(lr), float(beta1),
                                     float(beta2), float(eps), float(weight_decay), int(step), bool(bias_correction),
                                     bool(adapt), float(grad_scale), grad_scale_dev, list(master_params or []),
                                     *_ema(ema_params, ema_decay, ema_start))


def lamb_norms(params, grads, exp_avgs, exp_avg_sqs, beta1, beta2, eps, weight_decay, step, out, slots=None,
               bias_correction=True, grad_scale=1.0, grad_scale_dev=None, master_params=None):
    """First phase of fused_lamb_step, for parameters split into pieces (e.g. over the ranks' shards): updates the
    moments and ADDS each piece's sum of w^2 and of u^2 into out[2 * slot] and out[2 * slot + 1]. `out` is a contiguous
    float32 tensor on the parameters' device that the caller zeroes; `slots` (default 0, 1, ...) gives each piece the
    slot of the tensor it belongs to, so that pieces of one tensor add up, at most once per call. Two launches."""
    n = len(params)
    return _native().lamb_norms(list(params), list(grads), list(exp_avgs), list(exp_avg_sqs), float(beta1), float(beta2),
                                float(eps), float(weight_decay), int(step), bool(bias_correction), float(grad_scale),
                                grad_scale_dev, list(master_params or []), out,
                                list(range(n)) if slots is None else [int(s) for s in slots])


def lamb_apply(params, grads, exp_avgs, exp_avg_sqs, lr, beta1, beta2, eps, weight_decay, step, norms, slots=None,
               bias_correction=True, adapt=True, master_params=None, ema_params=None, ema_decay=None, ema_start=False):
    """Second phase: w -= lr * r * u, with u recomputed from the moments of lamb_norms and r from the whole-tensor sums of
    squares in `norms` (e.g. after adding up every rank's pieces). `grads` are checked as in lamb_norms but not read.
    One launch, which also updates the EMA (arguments as in fused_sgd_step)."""
    n = len(params)
    return _native().lamb_apply(list(params), list(grads), list(exp_avgs), list(exp_avg_sqs), float(lr), float(beta1),
                                float(beta2), float(eps), float(weight_decay), int(step), bool(bias_correction),
                                bool(adapt), list(master_params or []), norms,
                                list(range(n)) if slots is None else [int(s) for s in slots],
                                *_ema(ema_params, ema_decay, ema_start))


def fused_lars_step(params, grads, momentum_buffers, lr, momentum=0.9, weight_decay=0.0, trust_coefficient=0.001, eps=0.0,
                    adapt=True, grad_scale=1.0, grad_scale_dev=None, master_params=None, ema_params=None, ema_decay=None,
                    ema_start=False):
    """One LARS step in three launches per 65535 non-empty parameters (per-CTA norm partials, the per-tensor norms,
    the update), with the argument rules of fused_adam_step; the momentum buffers are fp32. For each parameter w:

        g = grad * grad_scale [* grad_scale_dev[0]];  d = g + weight_decay * w
        r = trust_coefficient * ||w|| / (||g|| + weight_decay * ||w|| + eps) if adapt and both norms are > 0, else 1
        v = momentum * v + lr * r * d;  w -= v

    The EMA arguments are those of fused_sgd_step; the update launch writes the EMA.
    Deterministic: the same input gives the same bits on every call. Up to 65535 non-empty parameters nothing is
    synchronised with the host (see fused_sgd_step)."""
    return _native().fused_lars_step(list(params), list(grads), list(momentum_buffers), float(lr), float(momentum),
                                     float(weight_decay), float(trust_coefficient), float(eps), bool(adapt),
                                     float(grad_scale), grad_scale_dev, list(master_params or []),
                                     *_ema(ema_params, ema_decay, ema_start))


def lars_norms(params, grads, momentum_buffers, out, slots=None, grad_scale=1.0, grad_scale_dev=None, master_params=None):
    """First phase of fused_lars_step, for parameters split into pieces (e.g. over the ranks' shards): ADDS each piece's
    sum of w^2 and of g^2 (g scaled as in fused_lars_step) into out[2 * slot] and out[2 * slot + 1], with lamb_norms'
    rules for `out` and `slots`. The momentum buffers are checked as in lars_apply but not read. Two launches."""
    n = len(params)
    return _native().lars_norms(list(params), list(grads), list(momentum_buffers), float(grad_scale), grad_scale_dev,
                                list(master_params or []), out, list(range(n)) if slots is None else [int(s) for s in slots])


def lars_apply(params, grads, momentum_buffers, lr, momentum, weight_decay, trust_coefficient, eps, norms, slots=None,
               adapt=True, grad_scale=1.0, grad_scale_dev=None, master_params=None, ema_params=None, ema_decay=None,
               ema_start=False):
    """Second phase: the momentum and parameter update of fused_lars_step, with r from the whole-tensor sums of squares
    in `norms` (e.g. after adding up every rank's pieces). Reads the gradient again: pass the grad_scale /
    grad_scale_dev of lars_norms. One launch, which also updates the EMA (arguments as in fused_sgd_step)."""
    n = len(params)
    return _native().lars_apply(list(params), list(grads), list(momentum_buffers), float(lr), float(momentum),
                                float(weight_decay), float(trust_coefficient), float(eps), bool(adapt), float(grad_scale),
                                grad_scale_dev, list(master_params or []), norms,
                                list(range(n)) if slots is None else [int(s) for s in slots],
                                *_ema(ema_params, ema_decay, ema_start))


def fused_adafactor_step(params, grads, row_vars, col_vars, variances, lr, beta2_decay, eps1, eps2, d, weight_decay, step,
                         grad_scale=1.0, grad_scale_dev=None, master_params=None, ema_params=None, ema_decay=None,
                         ema_start=False):
    """One torch.optim.Adafactor step for the whole parameter list in five launches (row sums and column partials of g^2,
    the factors, per-CTA norm partials, the per-tensor norms, the update), with the argument rules of fused_adam_step.
    Parameters of dim >= 2 (at most 5) keep fp32 factors over their last two dims, row_vars[i] of shape [..., R, 1] and
    col_vars[i] of shape [..., 1, C] (contiguous), and None in variances[i]; parameters of dim <= 1 keep an fp32
    variances[i] with their sizes and strides, and None in the factor lists.  Any dense layout.  For each parameter w
    (1-based `step` t):

        g = grad * grad_scale [* grad_scale_dev[0]];  beta_w = t^beta2_decay;  rho = min(lr, 1 / sqrt(t))
        alpha = max(eps2, ||w|| / sqrt(numel)) * rho                     (w before the decay)
        dim >= 2: row_var = lerp(row_var, mean_c g^2, beta_w);  col_var = lerp(col_var, mean_r g^2, beta_w)
                  v = row_var * col_var / max(mean_r row_var, eps1)
        dim <= 1: variance = lerp(variance, g^2, beta_w);  v = variance
        u = g * rsqrt(max(v, eps1^2));  denom = max(1, ||u|| / (sqrt(numel) * d))
        w = w * (1 - lr * weight_decay) - (alpha / denom) * u             (one fp32 expression, rounded once)

    The max of the two clamps of v keeps a NaN (torch's clamp), the max in alpha and denom drops one (Python's max(eps2,
    nan) and max(1, nan), as torch evaluates them): a NaN gradient element makes its row's and column's v NaN, and with
    them the mean of row_var and so every v of that matrix, exactly where torch.optim.Adafactor gives NaN.

    `eps1=None` is torch.finfo(params' dtype).eps, as torch resolves it.  `master_params` and the EMA arguments as in
    fused_sgd_step.  Scratch comes from torch's caching allocator on the current stream; nothing is synchronised with the
    host, so the call can be captured into a CUDA graph.  Deterministic: the same input gives the same bits on every
    call, and a parameter's result does not depend on the other parameters of the call.  At most 65535 non-empty
    parameters per call (one launch's grid); each parameter must have fewer than 2^32 elements (the kernels' element
    offsets are 32-bit), and a factored one sizes and strides below 2^31 in every dim.  A call past any of these limits
    raises RuntimeError before anything is launched."""
    params = list(params)
    if eps1 is None:
        eps1 = torch.finfo(params[0].dtype).eps if params else 0.0
    return _native().fused_adafactor_step(params, list(grads), list(row_vars), list(col_vars), list(variances), float(lr),
                                          float(beta2_decay), float(eps1), float(eps2), float(d), float(weight_decay),
                                          int(step), float(grad_scale), grad_scale_dev, list(master_params or []),
                                          *_ema(ema_params, ema_decay, ema_start))


def grad_shard_stats(tensors, out, inv_scale=None, norm_type=2.0):
    """Statistics of a list of gradients (fp32 / bf16 / fp16, any mix) in one read pass per dtype, accumulated into
    `out`, a float32 CUDA tensor of at least 2 elements that the caller zeroes first:

    * out[0] += the sum of squares of all elements (norm_type=2), or out[0] = max(out[0], max |element|) (norm_type=inf);
    * out[1] = 1 if any element is inf or NaN (else left as it was).

    With `inv_scale` (a 1-element fp32 tensor on out's device) every element is first multiplied by inv_scale[0] in
    place and rounded to its dtype; the statistics are those of the stored result. fp16 is allowed. The result is
    deterministic: the same input gives the same bits on every call. Nothing is synchronised with the host."""
    norm_type = float(norm_type)
    if norm_type not in (2.0, float('inf')):
        raise ValueError('grad_shard_stats: norm_type must be 2 or inf, got %r' % norm_type)
    by_dtype = {}
    for t in tensors:
        by_dtype.setdefault(t.dtype, []).append(t)
    for ts in by_dtype.values():
        _native().grad_shard_stats(ts, out, inv_scale, norm_type != 2.0)
    return out


_ACC_MODES = {'first': 0, 'add': 1, 'last': 2}


def grad_accumulate_(grads, accs, mode):
    """Gradient accumulation in fp32 for bf16 / fp16 gradients.  grads[i] (bf16 or fp16) and accs[i] (float32, same
    shape and strides) are folded element by element, in place:

    * mode 'first': accs[i] = grads[i] in fp32, then grads[i] = 0;
    * mode 'add':   accs[i] += grads[i] in fp32, then grads[i] = 0;
    * mode 'last':  grads[i] = accs[i] + grads[i], computed in fp32 and rounded to nearest-even once (accs[i] is not
      written).

    So k micro-batch gradients summed as first, add, ..., add, last are rounded once instead of k times, and the results
    are bit-identical to the same torch ops in fp32.  inf and NaN propagate (an fp16 sum above 65504 becomes inf).  One
    launch per gradient dtype and 160 tensors, on the current stream, with no host synchronisation: the call can be
    captured into a CUDA graph."""
    if mode not in _ACC_MODES:
        raise ValueError("grad_accumulate_: mode must be 'first', 'add' or 'last', got %r" % (mode,))
    grads, accs = list(grads), list(accs)
    if len(grads) != len(accs):
        raise ValueError('grad_accumulate_: %d gradients but %d accumulators' % (len(grads), len(accs)))
    by_dtype = {}
    for g, a in zip(grads, accs):
        gs, as_ = by_dtype.setdefault(g.dtype, ([], []))
        gs.append(g)
        as_.append(a)
    for gs, as_ in by_dtype.values():
        _native().grad_accumulate(gs, as_, _ACC_MODES[mode])
    return grads


def sync_bn_slot_doubles(num_features):
    """float64 elements of one rank's slot in sync_bn_stats' layout: 3 per channel, padded to 16 bytes, so that N slots
    in a row make a region of a multiple of 16 * N bytes (what the in-place allgather needs)."""
    return (3 * int(num_features) + 1) // 2 * 2


def sync_bn_stats(x, slot):
    """This rank's statistics of x for SyncBatchNorm, one launch: for every channel c (dim 1), slot[3c : 3c+3] =
    (count, mean, M2) in float64.  x is float32 / bfloat16 / float16, channels-last (channels innermost, which includes
    [N, C] and spatial size 1) or contiguous; `slot` is a contiguous float64 CUDA tensor of at least 3C elements.
    Welford per thread, Chan across CTAs, combined in fp64 in a fixed order: the same input gives the same bits."""
    _native().sync_bn_stats(x, slot)
    return slot


def sync_bn_combine(slots, num_features, eps, momentum=0.1, running_mean=None, running_var=None, num_batches_tracked=None):
    """Merges the rows of `slots` ([nranks, >= 3C] float64, one sync_bn_stats slot per rank) in rank order in fp64 and
    returns (mean, invstd, count): float32 tensors of C, C and 1 elements.  Where running stats are given they are
    updated as torch does (rv with the unbiased variance, none for a count of 1), with factor `momentum`, or
    1 / num_batches_tracked[0] read on the device when `num_batches_tracked` is given.  One launch."""
    return _native().sync_bn_combine(slots, int(num_features), float(eps), float(momentum), running_mean, running_var,
                                     num_batches_tracked)


def sync_bn_elemt(x, mean, invstd, weight=None, bias=None):
    """y = (x - mean) * invstd * weight + bias per channel, in x's dtype and layout.  weight / bias: float32 or x's
    dtype, or None.  One launch."""
    return _native().sync_bn_elemt(x, mean, invstd, weight, bias)


def sync_bn_backward_reduce(grad_output, x, mean, invstd, weight, sums, need_weight_grad=True, need_bias_grad=True):
    """sums[2c] = sum dy and sums[2c+1] = sum dy * (x - mean) over this rank's batch (float64, `sums` has >= 2C
    elements), to be summed over the ranks; returns this rank's (grad_weight, grad_bias) in the weight's dtype, None
    where not asked for.  grad_output must have x's sizes and strides.  One launch, deterministic."""
    return _native().sync_bn_backward_reduce(grad_output, x, mean, invstd, weight, sums, bool(need_weight_grad),
                                             bool(need_bias_grad))


def sync_bn_backward_elemt(grad_output, x, mean, invstd, weight, sums, count):
    """dx = (dy - sum_dy / n - (x - mean) * invstd^2 * sum_dy_xmu / n) * invstd * weight, with the summed `sums` of
    sync_bn_backward_reduce and n = count[0] of sync_bn_combine.  One launch."""
    return _native().sync_bn_backward_elemt(grad_output, x, mean, invstd, weight, sums, count)


def moe_permute(x, expert_idx, num_experts, nranks, send, counts, ctas=0):
    """The dispatch's first step, in three launches: the stable order of the [T, k] assignments by expert (expert
    ascending, then t * k + j ascending: torch.argsort(expert_idx.flatten(), stable=True)) and the copy of x[t] to the
    send rows of its k assignments.  x [T, hidden] and send [R >= T * k, hidden]: contiguous, one dtype (fp32 / bf16 /
    fp16).  expert_idx: int32 / int64 [T, k], 1 <= k <= 16.  counts: int64 [num_experts], receives this rank's count per
    expert.  Returns (pos, splits): pos int32 [T, k], the send row of each assignment; splits int32 [nranks], the rows
    for each rank's num_experts / nranks experts.  An id outside [0, num_experts) makes every split -1 and every count
    0.  Nothing is synchronised with the host; the same input gives the same bits on every call."""
    return tuple(_native().moe_permute(x, expert_idx, send, counts, int(num_experts), int(nranks), int(ctas)))


def moe_scatter(src, pos, dst, gates=None, dot_rows=None, status=None, ctas=0):
    """dst[pos[t, j]] = src[t] for every t < T and j < k (the bytes as they are), or with `gates` ([T, k], fp32 or src's
    dtype) round(gates[t, j] * src[t]) computed in fp32.  With `dot_rows` (rows like dst) also returns grad_gates [T, k]
    in the gates' dtype: grad_gates[t, j] = the fp32 dot of src[t] and dot_rows[pos[t, j]], summed in an order that
    depends on the row length only.  Positions outside dst's rows are skipped.  A non-zero status[0] (int32 on the
    device) writes no row and zero gate gradients.  One launch; returns grad_gates or None."""
    return _native().moe_scatter(src, pos, dst, gates, dot_rows, status, int(ctas))


def moe_gather(src, pos, gates=None, status=None, ctas=0):
    """y[t] = sum over j ascending of gates[t, j] * src[pos[t, j]], in fp32 (each product rounded, then added), rounded
    once to src's dtype; without gates a plain fp32 sum in j order.  Positions outside src's rows add nothing; a non-zero
    status[0] gives y = 0.  One launch; returns y [T, hidden]."""
    return _native().moe_gather(src, pos, gates, status, int(ctas))


def moe_regroup(src, counts, status=None, out=None, ctas=0):
    """Received rows grouped by source rank (rank 0's rows for local experts 0, 1, ..., then rank 1's, ...) to rows
    grouped by local expert, then source rank, keeping the senders' order.  counts: int64 [nranks, experts_per_rank],
    counts[p, e] the rows from rank p for local expert e.  Rows of `out` (default: new, like src) past the total are
    zeroed; all of them when status[0] is non-zero.  out may be src itself with one expert per rank (the order is the
    same; only the tail is written).  One launch; returns (out, offsets), offsets int32 [experts_per_rank] the end row of
    each group (torch._grouped_mm's `offs`)."""
    if out is None:
        out = torch.empty_like(src)
    return out, _native().moe_regroup(src, counts, status, out, False, int(ctas))


def moe_regroup_reverse(src, counts, out, status=None, ctas=0):
    """The inverse of moe_regroup: rows grouped by local expert back to source-rank order, into `out` (rows like src;
    only the rows below the total are written).  One launch; returns the return splits, int32 [nranks]: the rows of
    each source rank, all zero when status[0] is non-zero."""
    return _native().moe_regroup(src, counts, status, out, True, int(ctas))


def symm_empty(*args, **kwargs):
    """Collective: a tensor in registered symmetric memory (see horovod_b200.torch.symm_empty)."""
    from horovod_b200.torch.mpi_ops import symm_empty as f
    return f(*args, **kwargs)


def symm_available(*args, **kwargs):
    """True when registered symmetric memory can be allocated for the process set."""
    from horovod_b200.torch.mpi_ops import symm_available as f
    return f(*args, **kwargs)


def kernel_launches():
    """Number of kernels of this library launched by this process so far."""
    from horovod_b200.torch.mpi_ops import runtime_stats
    return int(runtime_stats()['kernel_launches'])
