"""Python access to the native sm_90a operations that are not collectives of the `hvd.*` API:

* `fused_sgd_step`, `fused_adam_step` — multi-tensor optimizer kernels (`csrc/kernels/optim_kernels.cu`);
* `grad_shard_stats` — one-pass gradient norm statistics, non-finite check and optional in-place unscale (same file);
* `symm_empty`, `symm_available` — registered symmetric memory for the zero-copy allreduce path;
* `sim` — the single-GPU simulation harness (N ranks = N concurrently running kernels on one device) used by the
  numerics tests, `bench/kernel_micro.py` and the ncu captures;
* `kernel_launches()` — how many kernels of this library were launched by this process (bench.py's `gpu_launches`).
"""
from horovod_b200.ops import sim  # noqa: F401


def _native():
    from horovod_b200.torch.mpi_ops import _native as n
    return n()


def fused_sgd_step(params, grads, momentum_buffers, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False,
                   grad_scale=1.0, first_step=False, grad_scale_dev=None, master_params=None):
    """One launch for the whole parameter list (fp32 / bf16 / fp16 parameters, fp32 or matching gradients).
    `grad_scale_dev`: an optional 1-element fp32 tensor on the parameters' device; the gradients are multiplied by
    grad_scale * grad_scale_dev[0], read by the kernel, so no host synchronisation is needed.

    `master_params`: optional fp32 master copies of bf16 / fp16 parameters (gradients of the parameters' dtype), one per
    parameter with its sizes and strides; momentum buffers are then fp32 too. The update runs on the master and the
    parameter receives it rounded to nearest-even. Where a parameter no longer equals its rounded master (it was
    written from outside, or the master is zero-filled), the master first restarts from the parameter."""
    return _native().fused_sgd_step(list(params), list(grads), list(momentum_buffers), float(lr), float(momentum), float(dampening),
                                    float(weight_decay), bool(nesterov), float(grad_scale), bool(first_step), grad_scale_dev,
                                    list(master_params or []))


def fused_adam_step(params, grads, exp_avgs, exp_avg_sqs, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, step=1,
                    grad_scale=1.0, adamw=True, grad_scale_dev=None, master_params=None):
    """One launch of Adam / AdamW for the whole parameter list (fp32 / bf16 / fp16 parameters, fp32 or matching
    gradients, fp32 state with the parameters' sizes and strides; `step` is the 1-based step count). Mismatched
    lists, dtypes, sizes, strides or devices raise RuntimeError before anything is launched. `grad_scale_dev` and
    `master_params` as in fused_sgd_step."""
    return _native().fused_adam_step(list(params), list(grads), list(exp_avgs), list(exp_avg_sqs), float(lr), float(beta1), float(beta2),
                                     float(eps), float(weight_decay), int(step), float(grad_scale), bool(adamw), grad_scale_dev,
                                     list(master_params or []))


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
