"""Micro-benchmark of hvd.ExpertDispatcher's kernels: expert-parallel dispatch and combine on one GPU.

N = 2, 4, 8 simulated ranks (`horovod_b200.ops.sim`) run the whole layer, step by step for every rank, with identity
experts (expert_out = expert_in): dispatch (permute, counts exchange, rows exchange, regroup), combine (regroup-reverse,
exchange, gather) and both backwards (scaled scatter with the gate-gradient dot, exchange, regroup; regroup-reverse,
exchange, gather-sum).  All ranks of one step are captured into one CUDA graph, replayed --iters times and timed with
CUDA events.  The torch-op arm does the same exchanges with torch ops around them: a stable argsort and index_select
into the send buffer, index_add_ for the combine and the dispatch backward, index_select and a product for the combine
backward.  Both arms' y, grad_x and grad_gates are compared before anything is timed.

Per kernel (rank 0's data, CUDA events over --iters launches): time, bytes moved (computed from the shapes below) and
the achieved rate against the H100 SXM's 3.35 TB/s HBM3; and the regroup's share (both directions, forward and
backward) of the summed kernel time of one rank.  Simulated peers share one GPU's HBM: these numbers do not describe
NVLink, and the exchange times here are local copies.

Sizes (per rank): Mixtral-like, T = 4096 tokens, hidden 4096 bf16, E = 8, k = 2; fine-grained, T = 4096, hidden
2048 bf16, E = 64, k = 8.  Capacity: twice the mean received rows.  The GPU name and power limit are read in the same
run.

    python bench/moe_dispatch_micro.py [--iters 20] [--out result.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SIZES = {'mixtral': dict(T=4096, h=4096, E=8, k=2), 'fine-grained': dict(T=4096, h=2048, E=64, k=8)}


def _gpu_info(device=0):
    name = torch.cuda.get_device_name(device)
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(device), '--query-gpu=power.limit', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'unknown'


def _events_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


class World:
    """N simulated ranks' inputs, buffers and the two arms, every step issued for every rank before the next."""

    def __init__(self, sim, ops, n, T, h, E, k, dtype=torch.bfloat16):
        self.sim, self.ops, self.n, self.T, self.h, self.E, self.k, self.el = sim, ops, n, T, h, E, k, E // n
        self.A, self.cap, self.dtype = T * k, 2 * T * k, dtype
        g = torch.Generator(device='cuda').manual_seed(n)
        self.x = [torch.randn(T, h, device='cuda', generator=g).to(dtype) for _ in range(n)]
        self.idx = [torch.randint(0, E, (T, k), device='cuda', generator=g) for _ in range(n)]
        self.gates = [torch.rand(T, k, device='cuda', generator=g) for _ in range(n)]
        self.gy = [torch.randn(T, h, device='cuda', generator=g).to(dtype) for _ in range(n)]
        self.send = [torch.zeros(self.A, h, dtype=dtype, device='cuda') for _ in range(n)]
        self.ret = [torch.zeros(self.cap, h, dtype=dtype, device='cuda') for _ in range(n)]
        self.counts = [torch.zeros(E, dtype=torch.int64, device='cuda') for _ in range(n)]
        self.count_splits = [torch.full((n,), self.el, dtype=torch.int32, device='cuda') for _ in range(n)]
        self.streams = [torch.cuda.Stream() for _ in range(n)]

    def exchange(self, ins, splits, cap, streams):
        outs = [torch.empty(cap, *ins[0].shape[1:], dtype=ins[0].dtype, device='cuda') for _ in range(self.n)]
        recv = [torch.empty(self.n, dtype=torch.int64, device='cuda') for _ in range(self.n)]
        status = [torch.empty(1, dtype=torch.int32, device='cuda') for _ in range(self.n)]
        self.sim.captured_alltoall(ins, splits, outs, recv, status, ctas=32, streams=streams)
        return outs, recv, status

    def each(self, streams, fn):
        out = []
        for r in range(self.n):
            if streams:
                with torch.cuda.stream(streams[r]):
                    out.append(fn(r))
            else:
                out.append(fn(r))
        return out

    def kernels(self, streams=None):
        ops, n = self.ops, self.n
        ps = self.each(streams, lambda r: ops.moe_permute(self.x[r], self.idx[r], self.E, n, self.send[r], self.counts[r]))
        rc, _, _ = self.exchange(self.counts, self.count_splits, self.E, streams)
        rc = [c.view(n, self.el) for c in rc]
        recv, _, st = self.exchange(self.send, [p[1] for p in ps], self.cap, streams)
        ein = self.each(streams, lambda r: ops.moe_regroup(recv[r], rc[r], st[r])[0])
        ret = self.each(streams, lambda r: ops.moe_regroup_reverse(ein[r], rc[r], self.ret[r], st[r]))
        back, _, _ = self.exchange(self.ret, ret, self.A, streams)
        y = self.each(streams, lambda r: ops.moe_gather(back[r], ps[r][0], self.gates[r], st[r]))
        gg = self.each(streams, lambda r: ops.moe_scatter(self.gy[r], ps[r][0], self.send[r], self.gates[r], back[r], st[r]))
        recv2, _, _ = self.exchange(self.send, [p[1] for p in ps], self.cap, streams)
        gout = self.each(streams, lambda r: ops.moe_regroup(recv2[r], rc[r], st[r])[0])
        ret2 = self.each(streams, lambda r: ops.moe_regroup_reverse(gout[r], rc[r], self.ret[r], st[r]))
        back2, _, _ = self.exchange(self.ret, ret2, self.A, streams)
        gx = self.each(streams, lambda r: ops.moe_gather(back2[r], ps[r][0], None, st[r]))
        return y, gx, gg

    def torch_ops(self, streams=None):
        n, k, T = self.n, self.k, self.T

        def permute(r):
            flat = self.idx[r].flatten()
            order = torch.argsort(flat, stable=True)
            tok = order // k
            torch.index_select(self.x[r], 0, tok, out=self.send[r])
            counts = torch.zeros(self.E, dtype=torch.int64, device='cuda').index_add_(0, flat, torch.ones_like(flat))
            return tok, self.gates[r].flatten()[order], counts.view(n, self.el).sum(1), order
        ps = self.each(streams, permute)
        recv, rs, _ = self.exchange(self.send, [p[2] for p in ps], self.cap, streams)
        # identity experts: the received rows go back as they are
        self.each(streams, lambda r: self.ret[r].copy_(recv[r]))
        back, _, _ = self.exchange(self.ret, rs, self.A, streams)

        def combine(r):
            tok, g = ps[r][:2]
            return torch.zeros(T, self.h, device='cuda').index_add_(0, tok, g[:, None] * back[r].float()).to(self.dtype)
        y = self.each(streams, combine)

        def combine_bwd(r):
            tok, g = ps[r][:2]
            rows = self.gy[r].index_select(0, tok)
            self.send[r].copy_((g[:, None] * rows.float()).to(self.dtype))
            return (rows.float() * back[r].float()).sum(-1)
        ggs = self.each(streams, combine_bwd)
        recv2, rs2, _ = self.exchange(self.send, [p[2] for p in ps], self.cap, streams)
        self.each(streams, lambda r: self.ret[r].copy_(recv2[r]))
        back2, _, _ = self.exchange(self.ret, rs2, self.A, streams)
        gx = self.each(streams, lambda r: torch.zeros(T, self.h, device='cuda').index_add_(0, ps[r][0], back2[r].float())
                       .to(self.dtype))
        def gate_grads(r):  # back in [T, k] order
            gg = torch.empty_like(ggs[r])
            gg[ps[r][3]] = ggs[r]
            return gg.view(T, k)
        gg = self.each(streams, gate_grads)
        return y, gx, gg

    def graph(self, fn):
        fn()  # warm-up, and the simulated team
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            cur = torch.cuda.current_stream()
            for s in self.streams:
                s.wait_stream(cur)
            out = fn(self.streams)
            for s in self.streams:
                cur.wait_stream(s)
        return g, out


def kernel_times(w, iters):
    """Rank 0's kernels one at a time: (name, ms, bytes)."""
    ops, h, k, T, A = w.ops, w.h, w.k, w.T, w.A
    s = torch.empty(0, dtype=w.dtype).element_size()
    rb = h * s
    pos, splits = ops.moe_permute(w.x[0], w.idx[0], w.E, w.n, w.send[0], w.counts[0])
    counts = torch.stack([c.view(w.n, w.el)[0] for c in w.counts])  # what rank 0 receives
    R = int(counts.sum())
    recv = torch.randn(w.cap, h, device='cuda').to(w.dtype)
    ein, _ = ops.moe_regroup(recv, counts)
    back = torch.randn(A, h, device='cuda').to(w.dtype)
    out = []
    out.append(('permute', _events_ms(lambda: ops.moe_permute(w.x[0], w.idx[0], w.E, w.n, w.send[0], w.counts[0]), iters),
                T * rb + A * rb + A * 12))
    out.append(('regroup', _events_ms(lambda: ops.moe_regroup(recv, counts, out=ein), iters), R * rb + w.cap * rb))
    out.append(('regroup_reverse', _events_ms(lambda: ops.moe_regroup_reverse(ein, counts, w.ret[0]), iters), 2 * R * rb))
    out.append(('gather_combine', _events_ms(lambda: ops.moe_gather(back, pos, w.gates[0]), iters), A * rb + T * rb + A * 8))
    out.append(('gather_sum', _events_ms(lambda: ops.moe_gather(back, pos), iters), A * rb + T * rb + A * 4))
    out.append(('scatter_scaled_dot', _events_ms(lambda: ops.moe_scatter(w.gy[0], pos, w.send[0], w.gates[0], back), iters),
                T * rb + 2 * A * rb + A * 12))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    ap.add_argument('--ranks', default='2,4,8')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('moe_dispatch_micro: needs a CUDA GPU')
    from horovod_b200 import ops
    from horovod_b200.ops import sim
    name, power = _gpu_info()
    rows = []
    for size, shape in SIZES.items():
        for n in [int(v) for v in args.ranks.split(',')]:
            w = World(sim, ops, n, **shape)
            gk, (yk, gxk, ggk) = w.graph(w.kernels)
            gt, (yt, gxt, ggt) = w.graph(w.torch_ops)
            gk.replay()
            gt.replay()
            torch.cuda.synchronize()
            for r in range(n):  # same results before timing: the torch arm sums in another order
                torch.testing.assert_close(yk[r].float(), yt[r].float(), rtol=2e-2, atol=2e-2)
                torch.testing.assert_close(gxk[r].float(), gxt[r].float(), rtol=2e-2, atol=2e-2)
                torch.testing.assert_close(ggk[r].float(), ggt[r].float(), rtol=1e-3, atol=1e-2)
            kern_ms = _events_ms(gk.replay, args.iters)
            torch_ms = _events_ms(gt.replay, args.iters)
            per = kernel_times(w, args.iters)
            total = sum(ms for _, ms, _ in per) + sum(ms for nm, ms, _ in per if nm.startswith('regroup'))
            regroup = 2 * sum(ms for nm, ms, _ in per if nm.startswith('regroup'))
            row = {'size': size, 'nranks': n, **shape, 'gpu': name, 'power_limit': power,
                   'graph_fwd_bwd_all_ranks_us': kern_ms * 1e3, 'torch_ops_graph_fwd_bwd_all_ranks_us': torch_ms * 1e3,
                   'kernels': {nm: {'us': ms * 1e3, 'bytes': b, 'tb_per_s': b / (ms * 1e-3) / 1e12,
                                    'of_hbm_peak': b / (ms * 1e-3) / HBM_BYTES_PER_S} for nm, ms, b in per},
                   'regroup_share_of_rank_kernel_time': regroup / total}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del w, gk, gt
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'w') as f:
            for r in rows:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
