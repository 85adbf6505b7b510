"""Gradient buckets of hvd.DistributedOptimizer, shared by the zero-copy path (optimizer.py, one in-place allreduce per
bucket) and the sharded path (sharded_optimizer.py, ZeRO-1: one reduce-scatter per bucket).

A bucket is a plain dict.  shard_layout() gives its layout ('group', 'dtype', 'members', 'numel', 'shard');
grad_bucket() adds a flat gradient buffer of registered memory ('gflat') of which every member's p.grad is a view
('params', 'views'), and the fp32 accumulation state ('acc', 'arrived', 'folds', 'fold_last').  Each optimizer adds the
keys of its own launch policy.  The functions here work on a bucket alone; what also reads the optimizer's settings
(its op, scales and accumulation) is a method of _DistributedOptimizerBase in optimizer.py.
"""
import torch

from horovod_b200.torch import mpi_ops

ALIGN = 128  # bytes: every parameter and every shard starts at a multiple of this


def _itemsize(dtype):
    return torch.empty(0, dtype=dtype).element_size()


# ---- layout ---------------------------------------------------------------------------------------------------------------
def shard_layout(groups, nranks, cap_bytes):
    """Pure layout of the gradient buckets (with nranks == 1: the zero-copy buckets).

    groups: one list per param group of (numel, dtype) of its trainable parameters, in registration order.
    Returns a list of buckets, each a dict with
      'group'    index of the param group,
      'dtype'    the parameters' dtype,
      'members'  [(index of the parameter in `groups[group]`, element offset in the bucket, numel)],
      'numel'    padded element count (its byte size is a multiple of nranks * 128),
      'shard'    elements per rank (numel // nranks).
    Parameters are taken in reverse order inside a group (gradients become ready roughly in that order), split by dtype,
    packed at 128 B alignment and cut into buckets of at most `cap_bytes` (a larger parameter gets a bucket of its own)."""
    buckets = []
    for gi, params in enumerate(groups):
        by_dtype = {}
        for i in reversed(range(len(params))):
            numel, dtype = params[i]
            by_dtype.setdefault(dtype, []).append((i, numel))
        for dtype, members in by_dtype.items():
            item = _itemsize(dtype)
            cur, cur_bytes = [], 0
            layouts = []
            for i, numel in members:
                nbytes = (numel * item + ALIGN - 1) // ALIGN * ALIGN
                if cur and cur_bytes + nbytes > cap_bytes:
                    layouts.append((cur, cur_bytes))
                    cur, cur_bytes = [], 0
                cur.append((i, cur_bytes // item, numel))
                cur_bytes += nbytes
            if cur:
                layouts.append((cur, cur_bytes))
            unit = nranks * ALIGN
            for mem, nbytes in layouts:
                padded = (nbytes + unit - 1) // unit * unit
                numel = padded // item
                buckets.append({'group': gi, 'dtype': dtype, 'members': mem, 'numel': numel, 'shard': numel // nranks})
    return buckets


def shard_range(bucket, rank):
    """Elements [lo, hi) of the bucket that `rank` owns."""
    return rank * bucket['shard'], (rank + 1) * bucket['shard']


def shard_slices(bucket, rank):
    """The parameter pieces inside `rank`'s shard: [(member position, first element in the parameter, last + 1,
    first element in the shard)]."""
    lo, hi = shard_range(bucket, rank)
    out = []
    for k, (_, off, numel) in enumerate(bucket['members']):
        a, b = max(lo, off), min(hi, off + numel)
        if a < b:
            out.append((k, a - off, b - off, a - lo))
    return out


def _memory_order(t, stride):
    """The elements of `t` in the memory order of a dense tensor of its shape with strides `stride` (None: row-major)."""
    if stride is None:
        return t.reshape(-1)
    x = torch.empty_strided(t.shape, stride, dtype=t.dtype, device=t.device)
    x.copy_(t)
    return x.as_strided((x.numel(),), (1,))


def shard_from_full(bucket, rank, full, strides=None, dtype=torch.float32, device=None):
    """This rank's shard of one state tensor.  full[k]: the state of member k (its parameter's shape) or None (zeros);
    strides[k]: the parameter's strides, i.e. the order in which its elements lie in the bucket (None: row-major).
    Padding is zero."""
    out = torch.zeros(bucket['shard'], dtype=dtype, device=device)
    for k, plo, phi, slo in shard_slices(bucket, rank):
        t = full[k]
        if t is not None:
            out[slo:slo + phi - plo].copy_(_memory_order(t, strides[k] if strides else None)[plo:phi])
    return out


def full_from_shards(bucket, shards, shapes, strides=None):
    """Inverse of shard_from_full: the N shards of a state tensor (in rank order) -> one tensor per member, shaped
    `shapes[k]` with strides `strides[k]` (None: row-major)."""
    flat = torch.cat([s.reshape(-1) for s in shards])
    out = []
    for k, (_, off, numel) in enumerate(bucket['members']):
        seg = flat[off:off + numel]
        out.append(seg.reshape(shapes[k]) if not strides else seg.as_strided(shapes[k], strides[k]))
    return out


# ---- the gradient buffer and p.grad ---------------------------------------------------------------------------------------
def grad_bucket(bucket, params, device, process_set):
    """Gives the layout `bucket` a zeroed flat gradient buffer of registered symmetric memory, 'gflat', and makes
    params[k], its k-th member, point p.grad at its view 'views'[p] (with p's strides, so channels_last stays
    channels_last; a gradient that exists already is copied in).  Returns the bucket."""
    gflat = mpi_ops.symm_empty(bucket['numel'], dtype=bucket['dtype'], device=device, process_set=process_set)
    gflat.zero_()
    bucket.update({'gflat': gflat, 'params': params, 'views': {}, 'acc': None, 'arrived': 0, 'folds': 0,
                   'fold_last': False})
    for p, (_, off, numel) in zip(params, bucket['members']):
        view = gflat[off:off + numel].as_strided(p.size(), p.stride())
        if p.grad is not None:
            view.copy_(p.grad)
        p.grad = view
        bucket['views'][p] = view
    return bucket


def adopt_grad(p, view, densify):
    """model.zero_grad() (set_to_none=True is torch's default) or `p.grad = None` dropped the bucket view and autograd
    allocated a fresh gradient: move it into the registered bucket and re-point p.grad, so the reference idiom keeps
    working (one extra copy for that parameter; optimizer.zero_grad() avoids it).  densify: a sparse gradient is made
    dense first (the zero-copy path); without it a sparse gradient raises, as the sharded path takes dense ones only."""
    if (densify and p.grad.is_sparse) or p.grad.data_ptr() != view.data_ptr():
        view.copy_(p.grad.to_dense() if p.grad.is_sparse else p.grad)
        p.grad = view


def adopt_missing_grads(bucket, seen, densify):
    """A bucket is reduced although some hook never fired: parameters whose gradient is None (dropped by
    model.zero_grad() and not produced this step) contribute zeros, unless their hook fired (`seen`), and get their
    bucket view back; fresh gradient tensors move into the bucket."""
    for p in bucket['params']:
        view = bucket['views'][p]
        if p.grad is None:
            if p not in seen:
                view.zero_()
            p.grad = view
        else:
            adopt_grad(p, view, densify)


# ---- gradient accumulation in fp32 (grad_accumulation_dtype=torch.float32) ------------------------------------------------
def check_grad_accumulation_dtype(dtype):
    """grad_accumulation_dtype: None (gradients accumulate in their own dtype) or torch.float32; True for the latter."""
    if dtype is None:
        return False
    if dtype is torch.float32:
        return True
    raise ValueError('grad_accumulation_dtype must be None or torch.float32, got %r' % (dtype,))


def fold(grads, accs, mode):
    from horovod_b200 import ops
    with torch.no_grad():
        ops.grad_accumulate_(grads, accs, mode)


def bucket_acc(bucket):
    if bucket['acc'] is None:  # plain device memory: the accumulator never travels
        bucket['acc'] = torch.empty(bucket['numel'], dtype=torch.float32, device=bucket['gflat'].device)
    return bucket['acc']


def fold_last(bucket, capturing):
    """Right before the bucket's collective, on the stream that issues it: the sum over the step's backward passes,
    rounded once, is what is reduced.  While hvd.GraphedStep captures the step's last graph, 'fold_last' marks the
    accumulating buckets (the hooks fold nothing during a capture)."""
    if bucket['folds'] or (capturing and bucket['fold_last']):
        fold([bucket['gflat']], [bucket_acc(bucket)], 'last')
        bucket['folds'] = 0


def reset_folds(buckets):
    for b in buckets:
        b['arrived'] = b['folds'] = 0


# ---- arguments shared by the optimizers -----------------------------------------------------------------------------------
def find_duplicates(lst):
    seen = set()
    dups = set()
    for el in lst:
        if el in seen:
            dups.add(el)
        seen.add(el)
    return dups


def check_named_parameters(opt, named_parameters):
    """The (name, parameter) pairs of every parameter of `opt`: `named_parameters` after checking it (tuples, unique
    names, no parameter left out), or generated names when it is None."""
    if named_parameters is not None:
        named_parameters = list(named_parameters)
    else:
        named_parameters = [(f'allreduce.noname.{i}.{j}', v)
                            for i, param_group in enumerate(opt.param_groups)
                            for j, v in enumerate(param_group['params'])]
    # make sure that named_parameters are tuples
    if any([not isinstance(p, tuple) for p in named_parameters]):
        raise ValueError('named_parameters should be a sequence of tuples (name, parameter), usually produced by '
                         'model.named_parameters().')
    dups = find_duplicates([k for k, _ in named_parameters])
    if len(dups) > 0:
        raise ValueError('Parameter names in named_parameters must be unique. Found duplicates: %s' % ', '.join(dups))
    all_param_ids = {id(v) for param_group in opt.param_groups for v in param_group['params']}
    named_param_ids = {id(v) for k, v in named_parameters}
    unnamed_param_ids = all_param_ids - named_param_ids
    if len(unnamed_param_ids):
        raise ValueError('named_parameters was specified, but one or more model parameters were not named. Python '
                         'object ids: %s' % ', '.join(str(id) for id in unnamed_param_ids))
    return named_parameters

