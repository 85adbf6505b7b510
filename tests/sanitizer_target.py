"""Small workload for compute-sanitizer: every kernel family once, on 2 and 4 simulated ranks, with ragged sizes."""
import ctypes

import torch

from horovod_b200.common.basics import load_library

lib = load_library()
lib.hvd_sim_allreduce.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int64),
                                  ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64), ctypes.c_int, ctypes.c_int,
                                  ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_int,
                                  ctypes.POINTER(ctypes.c_float)]
lib.hvd_sim_inplace.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.POINTER(ctypes.c_uint64), ctypes.c_int,
                                ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
lib.hvd_sim_allgather.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.POINTER(ctypes.c_uint64),
                                  ctypes.POINTER(ctypes.c_uint64), ctypes.c_int]
lib.hvd_sim_adasum.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int64),
                               ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64), ctypes.c_int, ctypes.c_int,
                               ctypes.c_double, ctypes.c_double]
FP32, BF16 = 7, 10
for n in (2, 4):
    sizes = [1, 333, 4099]
    for dt, tdt in ((FP32, torch.float32), (BF16, torch.bfloat16)):
        ins = [[torch.ones(s, device='cuda', dtype=tdt) for s in sizes] for _ in range(n)]
        outs = [[torch.empty_like(t) for t in r] for r in ins]
        counts = (ctypes.c_int64 * 3)(*sizes)
        ip = (ctypes.c_uint64 * (n * 3))(*[t.data_ptr() for r in ins for t in r])
        op = (ctypes.c_uint64 * (n * 3))(*[t.data_ptr() for r in outs for t in r])
        ms = ctypes.c_float(0)
        for variant in (0, 1):
            assert lib.hvd_sim_allreduce(n, 0, 3, counts, ip, op, dt, dt, 1, variant, 4, 1.0, 1.0, 1, ctypes.byref(ms)) == 0
            assert all(float(o[-1]) == n for o in outs[0])
        assert lib.hvd_sim_adasum(n, 0, 3, counts, ip, op, dt, 4, 1.0, 1.0) == 0
        assert abs(float(outs[0][2][-1]) - 1.0) < 1e-2  # identical vectors: adasum is the identity
    ts = [torch.ones(8192 + 4, device='cuda') for _ in range(n)]
    ptrs = (ctypes.c_uint64 * n)(*[t.data_ptr() for t in ts])
    ms = ctypes.c_float(0)
    assert lib.hvd_sim_inplace(n, 0, ts[0].numel() * 4, ptrs, FP32, 1, 4, 1.0, 1, ctypes.byref(ms)) == 0
    assert float(ts[0][-1]) == n
    src = [torch.full((1000,), float(r), device='cuda') for r in range(n)]
    dst = [torch.empty(1000 * n, device='cuda') for _ in range(n)]
    sp = (ctypes.c_uint64 * n)(*[t.data_ptr() for t in src])
    dp = (ctypes.c_uint64 * n)(*[t.data_ptr() for t in dst])
    rc = lib.hvd_sim_allgather(n, 0, 4000, sp, dp, 4)
    assert rc == 0, rc
    for r in range(n):
        got = dst[r].view(n, 1000)
        exp = torch.arange(n, device='cuda', dtype=torch.float32).view(n, 1).expand(n, 1000)
        assert torch.equal(got, exp), ('allgather mismatch', n, r, got[:, 0].tolist(), got[:, -1].tolist(),
                                       int((got != exp).sum()))

# fused SGD / Adam(W): every dtype pair, sizes around the 4-element vector and the 4096-element block, views at storage
# offsets 0-3 (unaligned params, grads and state), one launch over all of them. Each tensor is a view of an exactly
# sized buffer, so a store past a tail or before a head is an out-of-bounds access memcheck reports.
from horovod_b200 import ops  # noqa: E402


def _view(n, dtype, off):
    return torch.zeros(off + n, device='cuda', dtype=dtype)[off:]


sizes = [0, 1, 3, 4, 5, 4095, 4096, 4097, 3 * 4096 + 1]
for pdt, gdt in ((torch.float32, torch.float32), (torch.float32, torch.bfloat16), (torch.bfloat16, torch.bfloat16),
                 (torch.float16, torch.float16)):
    offs = [(i % 4, (i + 1) % 4, (i + 2) % 4) for i in range(len(sizes))]
    ps = [_view(n, pdt, a).fill_(1) for n, (a, _, _) in zip(sizes, offs)]
    gs = [_view(n, gdt, b).fill_(1) for n, (_, b, _) in zip(sizes, offs)]
    bufs = [_view(n, pdt, c) for n, (_, _, c) in zip(sizes, offs)]
    ms = [_view(n, torch.float32, c) for n, (_, _, c) in zip(sizes, offs)]
    vs = [_view(n, torch.float32, (c + 1) % 4) for n, (_, _, c) in zip(sizes, offs)]
    ops.fused_sgd_step(ps, gs, bufs, lr=0.5, momentum=0.9, nesterov=True, first_step=True)
    ops.fused_sgd_step(ps, gs, bufs, lr=0.5, momentum=0.9, weight_decay=0.1)
    ops.fused_adam_step(ps, gs, ms, vs, lr=1e-2, weight_decay=0.1, step=1, adamw=True)
    ops.fused_adam_step(ps, gs, ms, vs, lr=1e-2, weight_decay=0.1, step=2, adamw=False)
    torch.cuda.synchronize()
    assert all(float(p[-1]) < 0.5 for p in ps if p.numel()), [float(p[-1]) for p in ps if p.numel()]
torch.cuda.synchronize()
print('SANITIZER TARGET OK')
