"""hvd.captured_alltoall on >= 2 GPUs (run under hvdrun):

1. eager calls on registered inputs with device-generated splits, bf16 rows of 66 B (byte path) and fp32 rows of 1 KiB
   (16 B vectors): output and recv_splits byte for byte equal to hvd.alltoall(splits=...) of the same rows;
2. the call captured into a torch.cuda.graph together with the producer of the rows, replayed with new splits and rows
   written on the device: every replay equal to hvd.alltoall;
3. an overflow (rank 0 sends one row more than rank 1's capacity): every rank reports the same status, and the next call
   works;
4. an unregistered input and a splits tensor of the wrong length raise HorovodInternalError.
"""
import torch

import horovod_b200.torch as hvd
from horovod_b200.torch.mpi_ops import ALLTOALL_RECV_OVERFLOW

hvd.init()
rank, size = hvd.rank(), hvd.size()
torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank())
MAX_ROWS = 50


def device_splits(seed):
    g = torch.Generator(device=dev).manual_seed(1000 * seed + rank)
    return torch.randint(0, MAX_ROWS + 1, (size,), device=dev, generator=g)


def fill_rows(buf, seed):
    g = torch.Generator(device=dev).manual_seed(7919 * seed + rank)
    buf.copy_(torch.randn(buf.shape, device=dev, generator=g).to(buf.dtype))


def expect(buf, splits, out, recv, status, what):
    total_sent = int(splits.sum())
    ref, ref_splits = hvd.alltoall(buf[:total_sent].clone(), splits=splits)
    assert int(status) == 0, (what, int(status))
    assert recv.tolist() == ref_splits.tolist(), (what, recv.tolist(), ref_splits.tolist())
    got = out[:ref.shape[0]]
    assert torch.equal(got.contiguous().view(torch.uint8), ref.contiguous().view(torch.uint8)), (what, 'bytes differ')


def check_eager():
    for dtype, row in ((torch.bfloat16, (33,)), (torch.float32, (256,))):
        S = cap = MAX_ROWS * size
        buf = hvd.symm_empty((S, *row), dtype=dtype)
        for it in range(3):
            fill_rows(buf, it)
            splits = device_splits(it).to(torch.int32 if it % 2 else torch.int64)
            out, recv, status = hvd.captured_alltoall(buf, splits, cap)
            expect(buf, splits, out, recv, status, ('eager', dtype, it))
    print('[ok] eager', flush=True)


def check_graph():
    row = (128,)
    S = cap = MAX_ROWS * size
    buf = hvd.symm_empty((S, *row), dtype=torch.bfloat16)
    src = torch.zeros(S, *row, device=dev, dtype=torch.bfloat16)
    splits = torch.zeros(size, dtype=torch.int64, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up outside capture (same sequence on every rank)
        buf.copy_(src)
        hvd.captured_alltoall(buf, splits, cap)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        buf.copy_(src)
        out, recv, status = hvd.captured_alltoall(buf, splits, cap)
    for it in range(10):
        splits.copy_(device_splits(100 + it))
        fill_rows(src, 100 + it)
        g.replay()
        torch.cuda.synchronize()
        expect(src, splits, out, recv, status, ('graph replay', it))
    print('[ok] graph', flush=True)


def check_overflow():
    row = (16,)
    cap = 4 * size
    buf = hvd.symm_empty((cap, *row), dtype=torch.float32)
    fill_rows(buf, 5)
    splits = torch.full((size,), 4, dtype=torch.int64, device=dev)
    if rank == 0:
        splits[1] += 1  # rank 1 would receive cap + 1 rows (rank 0 has one spare row to send: S = cap)
        splits[0] -= 1
    out, recv, status = hvd.captured_alltoall(buf, splits, cap)
    codes = hvd.allgather(status.clone()).tolist()
    assert codes == [ALLTOALL_RECV_OVERFLOW] * size, codes
    splits.fill_(4)
    out, recv, status = hvd.captured_alltoall(buf, splits, cap)
    expect(buf, splits, out, recv, status, 'after overflow')
    print('[ok] overflow', flush=True)


def check_errors():
    x = torch.zeros(64, 4, device=dev)
    for args in ((x, torch.zeros(size, dtype=torch.int64, device=dev), 64),
                 (hvd.symm_empty((64, 4)), torch.zeros(size + 1, dtype=torch.int64, device=dev), 64)):
        try:
            hvd.captured_alltoall(*args)
            raise SystemExit('captured_alltoall accepted %s' % ('an unregistered tensor' if args[0] is x else 'wrong splits'))
        except hvd.HorovodInternalError:
            pass
    print('[ok] errors', flush=True)


check_eager()
check_graph()
check_overflow()
check_errors()
hvd.barrier()
if rank == 0:
    print('CAPTURED ALLTOALL OK', flush=True)
hvd.shutdown()
