"""LARS (You, Gitman, Ginsburg, "Large Batch Training of Convolutional Networks"), the optimizer of large-batch ResNet-50
training and of the MLPerf ResNet-50 reference; torch has none.

`Lars.step` is plain torch and runs anywhere: it is the readable definition of the update and what
`hvd.DistributedOptimizer(Lars(...))` runs without `fused=True`.  With `fused=True`, `master_weights=True` or
`shard_optimizer_state=True` the same update runs as the multi-tensor sm_90a kernels of `horovod_b200.ops.fused_lars_step`.
"""
import torch
from torch.optim.optimizer import required

from horovod_b200.torch.lamb import Lamb


class Lars(torch.optim.Optimizer):
    """For each parameter tensor w with gradient g:

        d = g + weight_decay * w
        r = trust_coefficient * ||w|| / (||g|| + weight_decay * ||w|| + eps)  if ||w|| > 0 and ||g|| > 0, else 1
        v = momentum * v + lr * r * d                                         norms over the whole tensor
        w = w - v

    The learning rate sits inside the momentum, as in Algorithm 1 of the paper and the MLPerf implementation; torch's
    SGD instead keeps v = momentum * v + d and steps w -= lr * v, which differs from this whenever lr changes during
    training.  A param group with weight_decay == 0 takes r = 1 unless always_adapt=True (the "exclude BatchNorm and
    bias" convention, the same rule as Lamb.adapts), so those parameters follow plain momentum SGD at rate lr.  No
    Nesterov.  The momentum buffer 'momentum_buffer' is fp32 for every parameter dtype and starts at zero, momentum=0
    included.  `lr` has no default: give it here or in every param group."""

    def __init__(self, params, lr=required, momentum=0.9, weight_decay=0.0, trust_coefficient=0.001, eps=0.0,
                 always_adapt=False):
        if lr is not required and not 0.0 <= lr:
            raise ValueError('Invalid learning rate: {}'.format(lr))
        if not 0.0 <= momentum < 1.0:
            raise ValueError('Invalid momentum value: {}'.format(momentum))
        if not 0.0 <= weight_decay:
            raise ValueError('Invalid weight_decay value: {}'.format(weight_decay))
        if not 0.0 < trust_coefficient:
            raise ValueError('Invalid trust_coefficient value: {}'.format(trust_coefficient))
        if not 0.0 <= eps:
            raise ValueError('Invalid epsilon value: {}'.format(eps))
        defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay, trust_coefficient=trust_coefficient, eps=eps,
                        always_adapt=always_adapt)
        super().__init__(params, defaults)

    adapts = staticmethod(Lamb.adapts)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            lr, mom, wd = group['lr'], group['momentum'], group['weight_decay']
            tc, eps = group['trust_coefficient'], group['eps']
            for p in group['params']:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError('Lars does not support sparse gradients')
                st = self.state[p]
                buf = st.get('momentum_buffer')
                if buf is None:
                    buf = st['momentum_buffer'] = torch.zeros_like(p, dtype=torch.float32,
                                                                   memory_format=torch.preserve_format)
                elif buf.dtype != torch.float32:  # load_state_dict casts state to the parameter's dtype
                    buf = st['momentum_buffer'] = buf.float()
                g, w = p.grad.float(), p.float()
                d = g.add(w, alpha=wd) if wd != 0.0 else g
                buf.mul_(mom)
                if self.adapts(group):
                    wn, gn = w.norm(), g.norm()
                    r = torch.where((wn > 0) & (gn > 0), tc * wn / (gn + wd * wn + eps), torch.ones_like(wn))
                    buf.add_(d * (lr * r))
                else:
                    buf.add_(d, alpha=lr)
                p.copy_(w.sub_(buf))
        return loss
