"""Environment-parallel (data-parallel) plumbing for GCBF.train_step -- SURVEY section 8e.

Graphs of a batch are independent (block-diagonal collation), so the B graphs are partitioned contiguously over the
ranks; weights, Adam state and the spectral-norm u/v buffers are replicated and stay bit-identical because every rank
applies the same all-reduced gradient.  Per step there are exactly three exchanges, all via torch.distributed (NCCL on
GPUs over NVLink/NVSwitch, gloo in the CPU tests):
  1. all-reduce of the 16 loss partial sums (fp64)   -> global counts for the masked means (gcbf.py:172,184,208,212)
  2. all-gather of h_dot (M floats per rank, unequal shards allowed: sizes travel over a gloo companion group) + all-reduce
     of one int64 pair count   -> the M x M `acc/derivative` (gcbf.py:209) over the GLOBAL agent count
  3. ONE all-reduce (sum) of the flat fp32 gradient bucket of both nets (24.46 M floats)   -> clip + Adam (gcbf.py:220-226)
The data-parallel vectorised Trainer adds host-side exchanges at evaluation only (broadcast of the episode seeds, gather of the
per-episode results), on the same gloo companion group.
"""
from typing import List, Optional, Tuple

import numpy as np
import torch


def shard_range(num_items: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous, balanced partition of `num_items` graphs: rank r owns [start, stop)."""
    base, rem = divmod(num_items, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


class Reducer:
    """Thin wrapper over a process group; a no-op for a single process."""

    def __init__(self, group=None):
        import torch.distributed as dist
        self.dist = dist
        self.group = group
        self.active = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if self.active else 1
        self.rank = dist.get_rank(group) if self.active else 0
        self._hg = None

    def sum_(self, t: torch.Tensor) -> torch.Tensor:
        if self.world > 1:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM, group=self.group)
        return t

    def max_(self, t: torch.Tensor) -> torch.Tensor:
        if self.world > 1:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX, group=self.group)
        return t

    def _host_group(self):
        """Process group for host-side metadata (per-rank sizes): the group itself when it is a CPU (gloo) group, else a gloo
        companion created once (collectively: every rank builds its Reducer at the same point of the first train step)."""
        if self._hg is None:
            backend = self.dist.get_backend(self.group)
            if 'gloo' in str(backend):
                self._hg = self.group if self.group is not None else self.dist.group.WORLD
            else:
                ranks = self.dist.get_process_group_ranks(self.group) if self.group is not None else None
                self._hg = self.dist.new_group(ranks=ranks, backend='gloo')
        return self._hg

    def sizes(self, n_local: int) -> List[int]:
        """Every rank's `n_local`, in rank order, exchanged on the host (no device sync).  Shards are NOT assumed equal:
        shard_range hands out B // world or B // world + 1 graphs, and GCBF.update de-duplicates its windows per rank."""
        if self.world == 1:
            return [int(n_local)]
        mine = torch.tensor([int(n_local)], dtype=torch.int64)
        out = [torch.zeros(1, dtype=torch.int64) for _ in range(self.world)]
        self.dist.all_gather(out, mine, group=self._host_group())
        return [int(x.item()) for x in out]

    def gather_cat(self, t: torch.Tensor, sizes: Optional[List[int]] = None) -> torch.Tensor:
        """Concatenation of the per-rank vectors, in rank order.  `sizes` (from `sizes()`) allows unequal lengths: the
        vectors travel padded to the longest one and the padding is dropped again."""
        if self.world == 1:
            return t
        t = t.contiguous()
        if sizes is None or len(set(sizes)) == 1:
            out = torch.empty(self.world * t.numel(), device=t.device, dtype=t.dtype)
            self.dist.all_gather_into_tensor(out, t, group=self.group)
            return out
        cap = max(sizes)
        padded = torch.zeros(cap, device=t.device, dtype=t.dtype)
        padded[:t.numel()] = t
        out = torch.empty(self.world, cap, device=t.device, dtype=t.dtype)
        self.dist.all_gather_into_tensor(out.view(-1), padded, group=self.group)
        return torch.cat([out[r, :n] for r, n in enumerate(sizes)])

    # ---- host arrays (the vectorised Trainer's sharded evaluation), over the gloo companion group ---------------------------
    def broadcast_host(self, a: np.ndarray) -> np.ndarray:
        """Rank 0's array on every rank; every rank passes an array of the same shape and dtype."""
        if self.world == 1:
            return a
        t = torch.from_numpy(np.array(a, copy=True))
        self.dist.broadcast(t, group_src=0, group=self._host_group())
        return t.numpy()

    def gather_rows(self, a: np.ndarray, sizes: Optional[List[int]] = None) -> np.ndarray:
        """Concatenation along axis 0 of every rank's array, in rank order.  Row counts may differ (`sizes`, from `sizes()`, or
        exchanged here); the trailing shape and the dtype must be the same on every rank."""
        if self.world == 1:
            return a
        sizes = self.sizes(a.shape[0]) if sizes is None else sizes
        padded = np.zeros((max(sizes),) + a.shape[1:], dtype=a.dtype)
        padded[:a.shape[0]] = a
        mine = torch.from_numpy(padded)
        out = [torch.empty_like(mine) for _ in range(self.world)]
        self.dist.all_gather(out, mine, group=self._host_group())
        return np.concatenate([o.numpy()[:n] for o, n in zip(out, sizes)])
