"""hvd.UlyssesExchange on >= 2 GPUs (run under hvdrun):

1. eager seq_to_heads / heads_to_seq of fp32, bf16 and fp16 tensors in the layouts [B, S, H, D], [B, S, 3, H, D] and
   [B, H, S, D], byte for byte equal to hvd.alltoall with torch permutes, and the round trip exact;
2. both exchanges captured into a torch.cuda.graph, replayed with new inputs written on the device;
3. a shape mismatch (rank 1 sends a longer shard): ALLTOALL_ROW_BYTES_MISMATCH on every rank, zero outputs, and the
   next call works;
4. a 2-layer GPT-2-style model trained for 3 steps with its sequence sharded over the ranks (hvd.DistributedOptimizer
   averages the replicated weights' gradients) against the same model trained on the whole sequence on every rank.
"""
import copy

import torch
import torch.nn.functional as F

import horovod_b200.torch as hvd
from horovod_b200.torch.mpi_ops import ALLTOALL_ROW_BYTES_MISMATCH

hvd.init()
rank, size = hvd.rank(), hvd.size()
torch.cuda.set_device(hvd.local_rank())
dev = torch.device('cuda', hvd.local_rank())


def reference(x, seq, head, to_heads):
    """The exchange through hvd.alltoall: permute into rank-major blocks, exchange, permute back."""
    split, cat = (head, seq) if to_heads else (seq, head)
    s = list(x.shape)
    blocks = x.view(*s[:split], size, s[split] // size, *s[split + 1:]).movedim(split, 0).contiguous()
    recv = hvd.alltoall(blocks)
    v = recv.movedim(0, cat)
    t = list(v.shape)
    return v.reshape(*t[:cat], t[cat] * t[cat + 1], *t[cat + 2:])


def check_eager():
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        ex = hvd.UlyssesExchange(1 << 16, dtype)
        for shape, seq, head in (((2, 7, 2 * size, 5), 1, 2), ((2, 6, 3, size, 8), 1, 3), ((2, 2 * size, 9, 4), 2, 1)):
            g = torch.Generator(device=dev).manual_seed(100 * rank + len(shape))
            x = torch.randn(shape, device=dev, generator=g).to(dtype)
            y = ex.seq_to_heads(x, seq, head)
            assert torch.equal(y.view(-1).view(torch.uint8), reference(x, seq, head, True).view(-1).view(torch.uint8)), (dtype, shape)
            back = ex.heads_to_seq(y, seq, head)
            assert torch.equal(back.view(-1).view(torch.uint8), reference(y, seq, head, False).view(-1).view(torch.uint8))
            assert torch.equal(back.view(-1).view(torch.uint8), x.view(-1).view(torch.uint8))
        assert int(ex.status) == 0
    print('[ok] eager', flush=True)


def check_graph():
    ex = hvd.UlyssesExchange(1 << 16, torch.bfloat16)
    x = torch.randn(2, 16, 3, 2 * size, 8, device=dev).to(torch.bfloat16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ex.heads_to_seq(ex.seq_to_heads(x, 1, 3), 1, 3)  # warm-up
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = ex.seq_to_heads(x, 1, 3)
        back = ex.heads_to_seq(y, 1, 3)
    for it in range(3):
        x.copy_(torch.randn(x.shape, device=dev).to(torch.bfloat16))
        graph.replay()
        assert torch.equal(y.view(torch.int16), reference(x, 1, 3, True).view(torch.int16)), ('replay', it)
        assert torch.equal(back.view(torch.int16), x.view(torch.int16)), ('replay round trip', it)
    assert int(ex.status) == 0
    print('[ok] graph', flush=True)


def check_mismatch():
    ex = hvd.UlyssesExchange(1 << 12, torch.float32)
    x = torch.randn(2, 5 + (rank == 1), 2 * size, 4, device=dev)
    y = ex.seq_to_heads(x, 1, 2)
    statuses = hvd.allgather(ex.status.cpu()).tolist()
    assert statuses == [ALLTOALL_ROW_BYTES_MISMATCH] * size, statuses
    assert not bool(y.view(torch.uint8).any())
    ex.status.zero_()
    x = torch.randn(2, 5, 2 * size, 4, device=dev)
    assert torch.equal(ex.seq_to_heads(x, 1, 2), reference(x, 1, 2, True)) and int(ex.status) == 0
    print('[ok] mismatch', flush=True)


class Block(torch.nn.Module):
    def __init__(self, h, H):
        super().__init__()
        self.H, self.D = H, h // H
        self.ln1, self.ln2 = torch.nn.LayerNorm(h), torch.nn.LayerNorm(h)
        self.qkv, self.proj = torch.nn.Linear(h, 3 * h), torch.nn.Linear(h, h)
        self.fc, self.out = torch.nn.Linear(h, 4 * h), torch.nn.Linear(4 * h, h)

    def forward(self, x, ex):
        B, S, h = x.shape
        qkv = self.qkv(self.ln1(x)).view(B, S, 3, self.H, self.D)
        if ex is not None:
            qkv = ex.seq_to_heads(qkv, 1, 3)
        q, k, v = (t.transpose(1, 2) for t in qkv.unbind(2))
        o = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).contiguous()
        if ex is not None:
            o = ex.heads_to_seq(o, 1, 2)
        x = x + self.proj(o.reshape(B, S, h))
        return x + self.out(F.gelu(self.fc(self.ln2(x))))


class GPT(torch.nn.Module):
    def __init__(self, vocab=97, h=64, H=2 * 8, S=128):
        super().__init__()
        self.wte, self.wpe = torch.nn.Embedding(vocab, h), torch.nn.Embedding(S, h)
        self.blocks = torch.nn.ModuleList([Block(h, H) for _ in range(2)])
        self.head = torch.nn.Linear(h, vocab)

    def forward(self, tokens, positions, ex=None):
        x = self.wte(tokens) + self.wpe(positions)
        for b in self.blocks:
            x = b(x, ex)
        return self.head(x)


def check_training():
    torch.manual_seed(0)
    B, S, vocab = 2, 128, 97
    full = GPT().to(dev)
    sharded = copy.deepcopy(full)
    ex = hvd.UlyssesExchange(B * S * 3 * 64 // size, torch.float32)
    opt_full = torch.optim.SGD(full.parameters(), lr=0.1)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(sharded.parameters(), lr=0.1), named_parameters=sharded.named_parameters())
    lo, hi = rank * S // size, (rank + 1) * S // size
    for step in range(3):
        g = torch.Generator(device=dev).manual_seed(step)  # the same batch on every rank
        tokens = torch.randint(0, vocab, (B, S + 1), device=dev, generator=g)
        pos = torch.arange(S, device=dev).expand(B, S)
        opt_full.zero_grad()
        F.cross_entropy(full(tokens[:, :-1], pos).flatten(0, 1), tokens[:, 1:].flatten()).backward()
        opt_full.step()
        opt.zero_grad()
        logits = sharded(tokens[:, lo:hi].contiguous(), pos[:, lo:hi].contiguous(), ex)
        # the mean over this rank's tokens; DistributedOptimizer's average over the ranks makes it the whole batch's mean
        F.cross_entropy(logits.flatten(0, 1), tokens[:, lo + 1:hi + 1].flatten()).backward()
        opt.step()
    assert int(ex.status) == 0
    for (name, a), b in zip(sharded.named_parameters(), full.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5, msg=name)
    print('[ok] training', flush=True)


check_eager()
check_graph()
check_mismatch()
check_training()
hvd.barrier()
if rank == 0:
    print('ULYSSES WORKER OK', flush=True)
hvd.shutdown()
