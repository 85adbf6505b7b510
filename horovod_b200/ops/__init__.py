"""Python access to the native sm_90a operations that are not collectives of the `hvd.*` API:

* `fused_sgd_step`, `fused_adam_step` — multi-tensor optimizer kernels (`csrc/kernels/optim_kernels.cu`);
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
                   grad_scale=1.0, first_step=False):
    """One launch for the whole parameter list (fp32 / bf16 / fp16 parameters, fp32 or matching gradients)."""
    return _native().fused_sgd_step(list(params), list(grads), list(momentum_buffers), float(lr), float(momentum), float(dampening),
                                    float(weight_decay), bool(nesterov), float(grad_scale), bool(first_step))


def fused_adam_step(params, grads, exp_avgs, exp_avg_sqs, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, step=1,
                    grad_scale=1.0, adamw=True):
    """One launch of Adam / AdamW for the whole parameter list (fp32 / bf16 / fp16 parameters, fp32 or matching
    gradients, fp32 state with the parameters' sizes and strides; `step` is the 1-based step count). Mismatched
    lists, dtypes, sizes, strides or devices raise RuntimeError before anything is launched."""
    return _native().fused_adam_step(list(params), list(grads), list(exp_avgs), list(exp_avg_sqs), float(lr), float(beta1), float(beta2),
                                     float(eps), float(weight_decay), int(step), float(grad_scale), bool(adamw))


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
