"""Pinned-memory, side-stream host→device prefetcher for the training input pipeline.

The reference leaves host→device staging to the framework's DataLoader (its synthetic benchmarks create the batch on
the device once: examples/pytorch/pytorch_synthetic_benchmark.py:79-86).  A ResNet-50 step takes tens of milliseconds, so a
38 MB batch copied synchronously from pageable memory is a visible bubble.  ``DevicePrefetcher`` wraps any iterable of
(nested) CPU tensors: batch *i+1* is copied into a ring of pinned staging buffers and sent over a dedicated copy
stream while batch *i* is being consumed; the consumer stream only waits on an event.
"""
import torch


def _map(obj, fn):
    if isinstance(obj, torch.Tensor):
        return fn(obj)
    if isinstance(obj, (list, tuple)):
        return type(obj)(_map(o, fn) for o in obj)
    if isinstance(obj, dict):
        return {k: _map(v, fn) for k, v in obj.items()}
    return obj


class DevicePrefetcher:
    """Iterates `loader`, delivering batches already on `device`: copies run `depth` batches ahead on a side stream from
    (reused) pinned staging buffers; `h2d_bytes` counts what was copied."""

    def __init__(self, loader, device=None, depth=2, channels_last=False):
        self.loader = loader
        self.device = torch.device(device if device is not None else
                                   (f'cuda:{torch.cuda.current_device()}' if torch.cuda.is_available() else 'cpu'))
        self.depth = max(1, int(depth))
        self.channels_last = channels_last
        self._cuda = self.device.type == 'cuda'
        self._stream = torch.cuda.Stream(self.device) if self._cuda else None
        self._pinned = {}  # (slot, leaf index) -> pinned staging tensor
        self._slot_event = {}  # slot -> event of the last copy issued from that slot's staging buffers
        self.h2d_bytes = 0

    def __len__(self):
        return len(self.loader)

    def _stage(self, slot, batch):
        leaf = [0]

        def send(t):
            i = leaf[0]
            leaf[0] += 1
            if not self._cuda:
                return t
            if t.is_cuda:
                return t
            self.h2d_bytes += t.numel() * t.element_size()
            src = t
            if not t.is_pinned():
                key = (slot, i)
                buf = self._pinned.get(key)
                if buf is None or buf.shape != t.shape or buf.dtype != t.dtype:
                    buf = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
                    self._pinned[key] = buf
                buf.copy_(t)
                src = buf
            out = src.to(self.device, non_blocking=True)
            if self.channels_last and out.dim() == 4:
                out = out.contiguous(memory_format=torch.channels_last)
            return out

        if not self._cuda:
            return _map(batch, send), None
        prev = self._slot_event.get(slot)
        if prev is not None:
            prev.synchronize()  # the DMA that last read this slot's pinned buffers must be done before we overwrite them
        with torch.cuda.stream(self._stream):
            out = _map(batch, send)
            ev = torch.cuda.Event()
            ev.record(self._stream)
        self._slot_event[slot] = ev
        return out, ev

    def __iter__(self):
        it = iter(self.loader)
        ring = []
        slot = 0
        # depth+1 pinned slots rotate; _stage() host-waits on the slot's previous copy event before overwriting it
        try:
            while len(ring) < self.depth:
                ring.append(self._stage(slot % (self.depth + 1), next(it)))
                slot += 1
        except StopIteration:
            it = None
        while ring:
            batch, ev = ring.pop(0)
            if ev is not None:
                torch.cuda.current_stream(self.device).wait_event(ev)
                _map(batch, lambda t: (t.record_stream(torch.cuda.current_stream(self.device)), t)[1] if t.is_cuda else t)
            if it is not None:
                try:
                    ring.append(self._stage(slot % (self.depth + 1), next(it)))
                    slot += 1
                except StopIteration:
                    it = None
            yield batch
