"""Multi-GPU inference for the AERO forward: batch sharding, one process per GPU.

Clips never interact in the forward (per-sample normalisation `aero.py:462-464`, per-sample GroupNorm, eval-mode
BatchNorm), so GPU g takes clips [g*B/G, (g+1)*B/G) and NO data-path collective is needed (SURVEY.md section 8e).
`torch.distributed` (NCCL on GPUs, gloo in the CPU tests) is used only to gather results when the caller wants
the whole batch on every rank, and for timing reductions.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def shard_range(n_items, rank, world):
    """Contiguous, balanced split: the first (n_items % world) ranks get one extra clip."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def reduce_max(value, device=None):
    """Max over ranks of a python float (used for max-over-ranks device timings)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


def average_over_ranks(value, count):
    """reference src/ddp/distrib.py:43-55 ``average([value], count)``: the mean of `value` over ranks, each weighted by its
    `count` (a rank with count 0 adds nothing; 0.0 when every count is 0).  Every rank must call it.  Reduces in fp64, on
    the current CUDA device under NCCL and on the CPU otherwise."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else None
    t = torch.tensor([float(value) * count, float(count)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t[0] / t[1]) if t[1] else 0.0


class ShardedAero:
    """Runs `model` on this rank's shard of a global batch; optionally all-gathers the waveforms."""

    def __init__(self, model, rank=None, world=None):
        self.model = model
        inited = dist.is_available() and dist.is_initialized()
        self.rank = rank if rank is not None else (dist.get_rank() if inited else 0)
        self.world = world if world is not None else (dist.get_world_size() if inited else 1)

    def local_slice(self, global_batch):
        return shard_range(global_batch, self.rank, self.world)

    @torch.no_grad()
    def forward(self, mix_global, gather=False):
        """mix_global: [B, C, L] (every rank holds, or can index, the global batch).  Returns this rank's
        outputs, or the whole batch on every rank when `gather` is set."""
        lo, hi = self.local_slice(mix_global.shape[0])
        dev = next(self.model.parameters()).device
        out = self.model(mix_global[lo:hi].to(dev))
        if not gather or self.world == 1:
            return out
        counts = [shard_range(mix_global.shape[0], r, self.world) for r in range(self.world)]
        width = max(h - l for l, h in counts)
        pad = out.new_zeros(width, *out.shape[1:])
        pad[: hi - lo] = out
        parts = [torch.empty_like(pad) for _ in range(self.world)]
        dist.all_gather(parts, pad)
        return torch.cat([p[: h - l] for p, (l, h) in zip(parts, counts)], 0)
