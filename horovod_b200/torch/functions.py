"""State synchronisation helpers: broadcast_parameters / broadcast_optimizer_state /
broadcast_object / allgather_object (API parity: horovod/torch/functions.py)."""
import io
import pickle

import torch

try:
    import cloudpickle
except ImportError:  # pragma: no cover
    cloudpickle = pickle

from horovod_b200.common.process_sets import global_process_set
from horovod_b200.torch.mpi_ops import (allgather, broadcast_, broadcast_async_, rank, size, synchronize)
from horovod_b200.torch.optimizer import _DistributedAdasumOptimizer, _DistributedOptimizerBase


def broadcast_parameters(params, root_rank, process_set=global_process_set):
    """Broadcasts `model.state_dict()`, `model.named_parameters()` or a list of (name, tensor) from root_rank."""
    if isinstance(params, dict):
        params = sorted(params.items())
    elif isinstance(params, list):
        params = [p if isinstance(p, tuple) else (None, p) for p in params]
    else:
        params = list(params)
        if params and not isinstance(params[0], tuple):
            raise ValueError('invalid params of type: %s' % type(params))
    handles = []
    for name, p in params:
        if p is None or not isinstance(p, torch.Tensor):
            continue
        t = p.data if isinstance(p, torch.nn.Parameter) else p
        if not t.is_contiguous():
            # broadcast a contiguous copy and write it back
            c = t.contiguous()
            handles.append((broadcast_async_(c, root_rank, 'broadcast.param.' + str(name), process_set), t, c))
        else:
            handles.append((broadcast_async_(t, root_rank, 'broadcast.param.' + str(name), process_set), None, None))
    for h, dst, src in handles:
        synchronize(h)
        if dst is not None:
            dst.copy_(src)


def broadcast_object(obj, root_rank=0, name=None, process_set=global_process_set):
    """Serialises `obj` on root_rank and returns it on every rank."""
    name = name or type(obj).__name__
    if rank() == root_rank:
        b = io.BytesIO()
        cloudpickle.dump(obj, b)
        t = torch.tensor(bytearray(b.getvalue()), dtype=torch.uint8)
        sz = torch.tensor([t.shape[0]], dtype=torch.int64)
        broadcast_(sz, root_rank, name + '.sz', process_set)
    else:
        sz = torch.zeros(1, dtype=torch.int64)
        broadcast_(sz, root_rank, name + '.sz', process_set)
        t = torch.empty(int(sz.item()), dtype=torch.uint8)
    broadcast_(t, root_rank, name + '.t', process_set)
    if rank() != root_rank:
        obj = cloudpickle.loads(t.numpy().tobytes())
    return obj


def allgather_object(obj, name=None, process_set=global_process_set):
    """Returns [obj of rank 0, obj of rank 1, ...] on every rank."""
    name = name or type(obj).__name__
    b = io.BytesIO()
    cloudpickle.dump(obj, b)
    t = torch.tensor(bytearray(b.getvalue()), dtype=torch.uint8)
    sizes = allgather(torch.tensor([t.shape[0]], dtype=torch.int64), name=name + '.sz', process_set=process_set)
    gathered = allgather(t, name=name + '.t', process_set=process_set)
    out, off = [], 0
    for s in sizes.tolist():
        out.append(cloudpickle.loads(gathered[off:off + s].numpy().tobytes()))
        off += s
    return out


def broadcast_optimizer_state(optimizer, root_rank, model=None, process_set=global_process_set):
    """Broadcasts optimizer state (tensors by collective, scalars/hyper-parameters as one pickled object)."""
    if isinstance(optimizer, torch.optim.LBFGS):
        raise ValueError('cannot broadcast torch.optim.LBFGS state')
    from horovod_b200.torch.sharded_optimizer import _ShardedDistributedOptimizer
    if isinstance(optimizer, _ShardedDistributedOptimizer):
        # every shard of the state has one owner: only hyper-parameters and step counts travel, no zero-gradient step
        optimizer._broadcast_state(root_rank)
        return
    state_dict = optimizer.state_dict()
    # Newly created optimizers have no state: materialise it with a zero-gradient step so every rank has the same keys
    created = []
    if len(state_dict['state']) == 0:
        for group in optimizer.param_groups:
            for p in group['params']:
                if p.requires_grad and p.grad is None:
                    p.grad = torch.zeros_like(p.data)
                    created.append(p)
        # a zero-grad step must not move the weights: snapshot and restore
        saved = [[p.data.clone() for p in g['params']] for g in optimizer.param_groups]
        if isinstance(optimizer, _DistributedOptimizerBase):  # the wrapped optimizer's own step, without a reduction
            optimizer._hvd_super_step()
        elif isinstance(optimizer, _DistributedAdasumOptimizer):
            super(_DistributedAdasumOptimizer, optimizer).step()
        else:
            optimizer.step()
        for g, ps in zip(optimizer.param_groups, saved):
            for p, s in zip(g['params'], ps):
                p.data.copy_(s)
        for p in created:
            p.grad = None  # leave no artificial gradients behind
        state_dict = optimizer.state_dict()
    if len(state_dict['state']) == 0:
        # stateless optimizer (plain SGD): only hyper-parameters travel
        pg = broadcast_object(state_dict['param_groups'], root_rank, 'opt.param_groups', process_set)
        if rank() != root_rank:
            state_dict['param_groups'] = pg
            optimizer.load_state_dict(state_dict)
        return

    scalars = {}
    tensors = []
    for pid, pstate in sorted(state_dict['state'].items(), key=lambda kv: str(kv[0])):
        for key, value in sorted(pstate.items()):
            if torch.is_tensor(value) and value.numel() > 0 and value.dim() > 0:
                tensors.append((f'opt.state.{pid}.{key}', value))
            else:
                scalars[(pid, key)] = value.item() if torch.is_tensor(value) and value.numel() == 1 else value
    meta = broadcast_object({'param_groups': state_dict['param_groups'], 'scalars': scalars}, root_rank, 'opt.meta', process_set)
    handles = []
    for name, t in tensors:
        c = t if t.is_contiguous() else t.contiguous()
        handles.append((broadcast_async_(c, root_rank, name, process_set), t, c))
    for h, dst, src in handles:
        synchronize(h)
        if dst is not src:
            dst.copy_(src)
    if rank() != root_rank:
        for (pid, key), value in meta['scalars'].items():
            cur = state_dict['state'][pid].get(key)
            if torch.is_tensor(cur):
                state_dict['state'][pid][key] = torch.as_tensor(value, dtype=cur.dtype, device=cur.device).reshape(cur.shape)
            else:
                state_dict['state'][pid][key] = value
        state_dict['param_groups'] = meta['param_groups']
        optimizer.load_state_dict(state_dict)
