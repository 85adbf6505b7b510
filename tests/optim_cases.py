"""Helpers shared by the GPU optimizer tests: the `hvd` fixture, guarded buffers, bit-level comparisons, the float64
reference of the fused Adam update and the kernel cases and models that several test modules build.  A test module
imports the `hvd` fixture by name; the asserts here carry their own messages, as pytest rewrites asserts in test
modules only."""
import numpy as np
import pytest
import torch

PAIRS = [(torch.float32, torch.float32), (torch.float32, torch.bfloat16), (torch.bfloat16, torch.bfloat16),
         (torch.float16, torch.float16)]
PAIR_IDS = ['f32', 'f32-bf16g', 'bf16', 'fp16']
LOW = [torch.bfloat16, torch.float16]
LOW_IDS = ['bf16', 'fp16']
SIZES = [1, 3, 4095, 4096, 4097, (1 << 20) + 3]
# around the 4-element vector, the 4096-element block (256 threads x 4 elements x 4 iterations) and a large tail
COUNTS = [1, 3, 4, 5, 4095, 4096, 4097, 3 * 4096 + 1, (1 << 20) + 3]


def ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.fixture(scope="module")
def hvd():
    import horovod_b200.torch as hvd
    hvd.init()
    torch.cuda.set_device(0)
    yield hvd
    hvd.shutdown()


def bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def same(a, b):
    """Bit-identical (NaN-safe, -0 != +0)."""
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(bits(a), bits(b))


def f32(x):
    return float(np.float32(x))


def cat(ts):
    return torch.cat([t.reshape(-1) for t in ts])


_MANT_EMIN = {torch.bfloat16: (7, -126), torch.float16: (10, -14), torch.float32: (23, -126)}


def ulp(x, dtype):
    """The spacing of `dtype` at |x| (float64 tensor), subnormals included."""
    mant, emin = _MANT_EMIN[dtype]
    _, e = torch.frexp(x.abs())  # |x| = f * 2^e, f in [0.5, 1); frexp(0) has e = 0, zero has the subnormal spacing
    e = torch.where(x == 0, torch.full_like(e, emin + 1), e)
    return torch.ldexp(torch.ones_like(x), torch.clamp(e - 1, min=emin) - mant)


class Slot:
    """A tensor of `shape` / `dtype` placed at element `offset` of a larger buffer; the slack is random bits that must
    survive the kernel (catches vector stores running past a tail or before a head)."""

    def __init__(self, shape, dtype, offset, fill, memory_format=torch.contiguous_format, slack=67):
        numel = int(np.prod(shape))
        self.buf = torch.randn(offset + numel + slack, device='cuda').to(dtype)
        strides = torch.empty(shape, memory_format=memory_format).stride() if len(shape) == 4 else torch.empty(shape).stride()
        self.t = self.buf.as_strided(shape, strides, offset)
        self.t.copy_(fill)
        self.lo, self.hi = offset, offset + numel
        self.slack = self._slack().clone()

    def _slack(self):
        b = bits(self.buf)
        return torch.cat([b[:self.lo], b[self.hi:]])

    def intact(self):
        return torch.equal(self._slack(), self.slack)


# ---- the float64 reference of the fused Adam(W) update ------------------------------------------------------------------
def adam_ref(p, g, m, v, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, step=1, adamw=True, grad_scale=1.0,
             bias=None):
    """One Adam (L2 weight decay) or AdamW (decoupled) step on float64 tensors, with `step` the parameter's 1-based step
    count; eps is added after sqrt(v) / sqrt(1 - beta2^step). `bias` overrides the two bias corrections. Returns
    (p, m, v, p_scale, m_scale, v_scale)."""
    c1, c2 = bias if bias is not None else (1 - beta1 ** step, 1 - beta2 ** step)
    d = g * grad_scale
    ds = d.abs()
    if adamw:
        p = p * (1 - lr * weight_decay)
    elif weight_decay != 0:
        d = d + weight_decay * p
        ds = ds + abs(weight_decay) * p.abs()
    m_new = beta1 * m + (1 - beta1) * d
    ms = beta1 * m.abs() + (1 - beta1) * ds
    v_new = beta2 * v + (1 - beta2) * d * d
    vs = beta2 * v + (1 - beta2) * ds * ds
    denom = v_new.sqrt() / c2 ** 0.5 + eps
    return p - (lr / c1) * m_new / denom, m_new, v_new, p.abs() + (lr / c1) * ms / denom, ms, vs


def adam_ref_kernel(p, g, m, v, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, step=1, adamw=True, grad_scale=1.0):
    """adam_ref with the hyper-parameters the kernel receives: fp32 values, bias corrections 1 - (float)beta^step."""
    bias = (f32(1.0 - f32(beta1 ** step)), f32(1.0 - f32(beta2 ** step)))
    return adam_ref(p, g, m, v, f32(lr), f32(beta1), f32(beta2), f32(eps), f32(weight_decay), step, adamw,
                    f32(grad_scale), bias)


# ---- LAMB / LARS kernel cases -------------------------------------------------------------------------------------------
def two_phase(kind, cases, master, gsd=None, **hp):
    """lamb_norms then lamb_apply (kind 'lamb') or lars_norms then lars_apply ('lars') over `cases`; returns the norms
    buffer."""
    from horovod_b200 import ops
    ws = [c['w'].t for c in cases] if master else None
    out = torch.zeros(2 * len(cases), device='cuda')
    if kind == 'lamb':
        lists = [[c[k].t for c in cases] for k in ('p', 'g', 'm', 'v')]
        moments = hp['beta1'], hp['beta2'], hp['eps'], hp['weight_decay'], hp['step']
        ops.lamb_norms(*lists, *moments, out, grad_scale_dev=gsd, master_params=ws)
        ops.lamb_apply(*lists, hp['lr'], *moments, out, master_params=ws)
    else:
        lists = [[c[k].t for c in cases] for k in ('p', 'g', 'v')]
        ops.lars_norms(*lists, out, grad_scale_dev=gsd, master_params=ws)
        ops.lars_apply(*lists, hp['lr'], hp['momentum'], hp['weight_decay'], hp['trust_coefficient'], hp['eps'], out,
                       grad_scale_dev=gsd, master_params=ws)
    return out


# ---- world size 1 -------------------------------------------------------------------------------------------------------
def mlp(dtype, seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(24, 48), torch.nn.GELU(), torch.nn.LayerNorm(48),
                               torch.nn.Linear(48, 8)).cuda().to(dtype)


def mlp_loss(m, step, dtype):
    g = torch.Generator(device='cuda').manual_seed(step)
    x = torch.randn(16, 24, device='cuda', generator=g).to(dtype)
    return m(x).float().square().mean()


def make_optimizer(hvd, kind, params):
    """The optimizer of one kind ('sgd', 'adamw', 'lamb' or 'lars') that the accumulation and clipping tests train with."""
    if kind == 'sgd':
        return torch.optim.SGD(params, lr=0.05, momentum=0.9, weight_decay=1e-4)
    if kind == 'adamw':
        return torch.optim.AdamW(params, lr=1e-2, weight_decay=0.01)
    if kind == 'lamb':
        return hvd.Lamb(params, lr=1e-2, weight_decay=0.01)
    return hvd.Lars(params, lr=0.5, momentum=0.9, weight_decay=1e-3, trust_coefficient=0.02)
