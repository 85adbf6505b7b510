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


# ---- the float64 references of the fused LAMB, LARS and Adafactor updates --------------------------------------------
def lamb_ref(cases, lr, beta1, beta2, eps, weight_decay, step, bias_correction=True, adapt=True, grad_scale=1.0,
             fp32_moments=False):
    """fp64 LAMB from the values the kernel reads (parameter and gradient in their dtypes, fp32 moments) and the
    hyper-parameters as the kernel holds them (fp32).  'scale_*' bound the magnitudes that fp32 rounding errors are
    relative to.  `fp32_moments`: m, v and v / c2 rounded to fp32 in the kernel's operation order, m = fmaf(b1, m,
    (1 - b1) g), v = fmaf(b2, v, ((1 - b2) g) g) and sqrt(v / c2), for values that overflow fp32 where float64 would
    not."""
    out = []
    b1, b2, lr, eps, wd = f32(beta1), f32(beta2), f32(lr), f32(eps), f32(weight_decay)
    # as the binding forms them (and fused Adam's): 1 - (beta^step rounded to fp32), in fp32
    c1, c2 = (float(np.float32(1) - np.float32(beta1 ** step)), float(np.float32(1) - np.float32(beta2 ** step))) \
        if bias_correction else (1.0, 1.0)
    for c in cases:
        w, g = c['p'].t.double(), c['g'].t.double() * f32(grad_scale)
        mo, vo = c['m'].t.double(), c['v'].t.double()
        if fp32_moments:
            f = lambda x: x.float().double()  # noqa: E731
            m = f(b1 * mo + f(f32(1 - b1) * g))
            v = f(b2 * vo + f(f(f32(1 - b2) * g) * g))
            vc = f(v / c2)
        else:
            m = b1 * mo + f32(1 - b1) * g
            v = b2 * vo + f32(1 - b2) * g * g
            vc = v / c2
        adam = (m / c1) / (vc.sqrt() + eps)
        u = adam + wd * w
        wn, un = float(w.norm()), float(u.norm())
        r = wn / un if adapt and wn > 0 and un > 0 else 1.0
        scale_m = (b1 * mo).abs() + (f32(1 - b1) * g).abs()  # >= |m|: m's rounding errors are relative to this
        scale_u = (scale_m / c1) / (vc.sqrt() + eps) + (wd * w).abs()
        out.append({'w': w - lr * r * u, 'm': m, 'v': v, 'scale_m': scale_m, 'scale_u': lr * r * scale_u})
    return out


def lars_ref(cases, lr, momentum, weight_decay, trust_coefficient, eps, adapt=True, grad_scale=1.0, fp32_norms=False):
    """fp64 LARS from the values the kernel reads (parameter and gradient in their dtypes, fp32 momentum) and the
    hyper-parameters as the kernel holds them (fp32).  'scale_v' bounds the magnitudes that fp32 rounding errors are
    relative to.  `fp32_norms`: the sums of squares rounded to fp32, as the kernel stores them, so one past the fp32
    maximum is inf (||g|| = inf gives r = 0)."""
    lr, mom, wd, tc, eps = f32(lr), f32(momentum), f32(weight_decay), f32(trust_coefficient), f32(eps)
    out = []
    for c in cases:
        w, g = c['p'].t.double(), c['g'].t.double() * f32(grad_scale)
        vo = c['v'].t.double()
        wn, gn = float(w.norm()), float(g.norm())
        if fp32_norms:
            wn, gn = (float(torch.tensor(x * x, dtype=torch.float64).float()) ** 0.5 for x in (wn, gn))
        r = tc * wn / (gn + wd * wn + eps) if adapt and wn > 0 and gn > 0 else 1.0
        d = g + wd * w
        v = mom * vo + lr * r * d
        scale_v = mom * vo.abs() + lr * r * (g.abs() + (wd * w).abs())
        out.append({'w': w - v, 'v': v, 'scale_v': scale_v})
    return out


def adafactor_ref(c, lr, beta2_decay, eps1, eps2, d, weight_decay, step, grad_scale=1.0, fp32_squares=False):
    """fp64 Adafactor from the values the kernel reads, with its fp32 hyper-parameters.  Returns the new parameter, its
    state, and the magnitude |alpha / denom * u| (the update) that the rounding errors are relative to.
    `fp32_squares`: g^2 rounded to fp32 as the kernel squares the scaled gradient, so a square past the fp32 maximum
    is inf."""
    pdt = c['p'].t.dtype
    eps1 = torch.finfo(pdt).eps if eps1 is None else eps1
    beta_w, rho = f32(step ** beta2_decay), f32(min(lr, 1 / step ** 0.5))
    e1, e1sq, e2, dd, decay = f32(eps1), f32(eps1 * eps1), f32(eps2), f32(d), f32(1 - lr * weight_decay)
    w, g = c['p'].t.double(), c['g'].t.double() * f32(grad_scale)
    # torch's two-sided lerp, as torch.optim.Adafactor and the kernel use it: lerp(0, inf, 1) is NaN, not inf
    lerp = lambda a, b: torch.lerp(a, b, beta_w)  # noqa: E731
    sq = (g * g).float().double() if fp32_squares else g * g
    out = {}
    if w.dim() >= 2:
        r = lerp(c['r'].t.double(), sq.mean(-1, keepdim=True))
        col = lerp(c['c'].t.double(), sq.mean(-2, keepdim=True))
        v = r * col / r.mean(-2, keepdim=True).clamp(min=e1)
        out.update(r=r, c=col)
    else:
        v = out['v'] = lerp(c['v'].t.double(), sq)
    u = g * v.clamp(min=e1sq).rsqrt()
    n = max(w.numel(), 1)
    alpha = max(e2, float(w.norm()) / n ** 0.5) * rho
    denom = max(1.0, float(u.norm()) / (n ** 0.5 * dd))
    out['p'] = w * decay - alpha / denom * u
    out['scale'] = (alpha / denom * u).abs()
    return out


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
