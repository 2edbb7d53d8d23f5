"""Step arena: bump allocation of the train step's activations and gradients out of a few large, persistent device
chunks.

Why: one train step allocates ~10 GB of short-lived tensors whose sizes change every step (the re-linked graph has a
different edge count each time), which makes the torch caching allocator fall back to cudaMalloc / cudaFree storms
(measured: the same step taking 31 ms or 70 ms).  With 80 GB of HBM per GPU the simple answer is an explicit arena:
`begin()` at the start of `GCBF.train_step`, every internal buffer is a view into a chunk, nothing is freed, the next
`begin()` rewinds.  Tensors handed back to the caller are cloned out of the arena first.
"""
import math

import torch

_ALIGN = 256
_CHUNK_BYTES = 1 << 30
_ITEMSIZE = {}


class StepArena:
    def __init__(self):
        self.device = None
        self.chunks = []          # uint8 tensors
        self.cur = 0
        self.off = 0
        self.active = False
        self.high_water = 0
        self._views = {}
        self.epoch = 0            # bumped by begin(): lets per-step pools (ops.amax_slot) notice the rewind

    def begin(self, device):
        if self.device != device:
            self.chunks, self.device, self._views = [], device, {}
        self.cur, self.off, self.active = 0, 0, True
        self.epoch += 1

    def end(self):
        self.active = False
        used = sum(c.numel() for c in self.chunks[:self.cur]) + self.off
        self.high_water = max(self.high_water, used)

    def _typed(self, ci: int, dtype) -> torch.Tensor:
        """dtype view of chunk `ci` (cached: one view per chunk and dtype)."""
        key = (ci, dtype)
        v = self._views.get(key)
        if v is None:
            v = self._views[key] = self.chunks[ci].view(dtype)
        return v

    def alloc(self, shape, dtype) -> torch.Tensor:
        n = 1
        for d in shape:
            n *= d
        if n == 0:
            return torch.empty(shape, device=self.device, dtype=dtype)
        itemsize = _ITEMSIZE.get(dtype)
        if itemsize is None:
            itemsize = _ITEMSIZE[dtype] = torch.empty(0, dtype=dtype).element_size()
        nbytes = n * itemsize
        need = (nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
        while True:
            if self.cur >= len(self.chunks):
                size = max(_CHUNK_BYTES, int(need * 1.25) // _ALIGN * _ALIGN + _ALIGN)
                self.chunks.append(torch.empty(size, device=self.device, dtype=torch.uint8))
            if self.off + need <= self.chunks[self.cur].numel():
                break
            self.cur += 1
            self.off = 0
        # one as_strided on the cached typed view of the chunk (contiguous strides computed here)
        strides, acc = [], 1
        for d in reversed(shape):
            strides.append(acc)
            acc *= d
        strides.reverse()
        out = self._typed(self.cur, dtype).as_strided(shape, strides, self.off // itemsize)
        self.off += need
        return out


ARENA = StepArena()


def empty(*shape, device, dtype=torch.float32) -> torch.Tensor:
    if len(shape) == 1 and isinstance(shape[0], (tuple, list, torch.Size)):
        shape = tuple(shape[0])
    if ARENA.active and torch.device(device) == ARENA.device:
        return ARENA.alloc(shape, dtype)
    return torch.empty(shape, device=device, dtype=dtype)


def zeros(*shape, device, dtype=torch.float32) -> torch.Tensor:
    t = empty(*shape, device=device, dtype=dtype)
    if ARENA.active and torch.device(device) == ARENA.device:
        t.zero_()
        return t
    return torch.zeros(t.shape, device=device, dtype=dtype) if t.numel() else t
