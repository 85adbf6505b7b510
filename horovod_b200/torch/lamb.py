"""LAMB (You et al., "Large Batch Optimization for Deep Learning: Training BERT in 76 minutes"), the optimizer of
large-batch transformer pre-training; torch has none.

`Lamb.step` is plain torch and runs anywhere: it is the readable definition of the update and what
`hvd.DistributedOptimizer(Lamb(...))` runs without `fused=True`.  With `fused=True`, `master_weights=True` or
`shard_optimizer_state=True` the same update runs as the multi-tensor sm_90a kernels of `horovod_b200.ops.fused_lamb_step`.
"""
import torch


class Lamb(torch.optim.Optimizer):
    """For each parameter tensor w at 1-based step t:

        g = grad
        m = b1 m + (1 - b1) g
        v = b2 v + (1 - b2) g^2
        u = (m / c1) / (sqrt(v / c2) + eps) + weight_decay * w     c1 = 1 - b1^t, c2 = 1 - b2^t (1 without bias_correction)
        r = ||w|| / ||u||  if both norms are > 0, else 1           norms over the whole tensor
        w = w - lr * r * u

    A param group with weight_decay == 0 takes r = 1 unless always_adapt=True (so biases and LayerNorm weights follow
    Adam), as apex FusedLAMB(use_nvlamb=False) and timm's Lamb do.  No gradient clipping of its own: use
    torch.nn.utils.clip_grad_norm_, or opt.clip_grad_norm_ with sharded optimizer state.  The moments 'exp_avg' and
    'exp_avg_sq' are fp32 for every parameter dtype; 'step' is a float CPU tensor, as in torch's Adam."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, bias_correction=True,
                 always_adapt=False):
        if not 0.0 <= lr:
            raise ValueError('Invalid learning rate: {}'.format(lr))
        if not 0.0 <= eps:
            raise ValueError('Invalid epsilon value: {}'.format(eps))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError('Invalid beta parameter at index 0: {}'.format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError('Invalid beta parameter at index 1: {}'.format(betas[1]))
        if not 0.0 <= weight_decay:
            raise ValueError('Invalid weight_decay value: {}'.format(weight_decay))
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, bias_correction=bias_correction,
                        always_adapt=always_adapt)
        super().__init__(params, defaults)

    @staticmethod
    def adapts(group):
        """Whether the trust ratio applies to the parameters of `group`."""
        return group['weight_decay'] != 0.0 or bool(group['always_adapt'])

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            b1, b2 = group['betas']
            lr, eps, wd = group['lr'], group['eps'], group['weight_decay']
            for p in group['params']:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError('Lamb does not support sparse gradients')
                st = self.state[p]
                if 'exp_avg' not in st:
                    st['step'] = torch.tensor(0.0)
                    st['exp_avg'] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
                    st['exp_avg_sq'] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
                for key in ('exp_avg', 'exp_avg_sq'):
                    if st[key].dtype != torch.float32:  # load_state_dict casts state to the parameter's dtype
                        st[key] = st[key].float()
                if not torch.is_tensor(st['step']):
                    st['step'] = torch.tensor(float(st['step']))
                st['step'] += 1
                t = float(st['step'])
                c1, c2 = (1.0 - b1 ** t, 1.0 - b2 ** t) if group['bias_correction'] else (1.0, 1.0)
                m, v = st['exp_avg'], st['exp_avg_sq']
                g, w = p.grad.float(), p.float()
                m.mul_(b1).add_(g, alpha=1.0 - b1)
                v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
                u = (m / c1) / ((v / c2).sqrt() + eps)
                if wd != 0.0:
                    u.add_(w, alpha=wd)
                if self.adapts(group):
                    wn, un = w.norm(), u.norm()
                    r = torch.where((wn > 0) & (un > 0), wn / un, torch.ones_like(wn))
                    u.mul_(r)
                p.copy_(w.add_(u, alpha=-lr))
        return loss
