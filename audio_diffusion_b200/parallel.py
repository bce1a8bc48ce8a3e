"""Multi-GPU plumbing for batched sampling (SURVEY §8e): one process per GPU, ONE broadcast of the weights at init,
no per-step collective; every rank draws the full-batch noise stream from the same seed and keeps its rows, so the
result is independent of the number of shards."""
from __future__ import annotations

from typing import Iterable, Sequence

import torch


def broadcast_parameters(params: Iterable[torch.Tensor], src: int = 0) -> None:
    """Single collective: flatten -> broadcast -> scatter back (NCCL on GPUs, gloo in the CPU tests)."""
    import torch.distributed as dist
    params = list(params)
    flat = torch.cat([p.data.reshape(-1) for p in params])
    dist.broadcast(flat, src=src)
    off = 0
    with torch.no_grad():
        for p in params:
            p.copy_(flat[off:off + p.numel()].view_as(p))   # in place on the parameter: its version changes -> weights re-packed
            off += p.numel()


def shard_rows(n: int, rank: int, world: int) -> slice:
    if n % world:
        raise ValueError(f"global batch {n} is not divisible by world size {world}")
    per = n // world
    return slice(rank * per, (rank + 1) * per)


def shard_noise(global_shape: Sequence[int], generator: torch.Generator, rank: int, world: int, device) -> torch.Tensor:
    """Rows [rank*B/world, (rank+1)*B/world) of torch.randn(global_shape, generator) — the reference's own draw
    (pipeline_audio_diffusion.py:120-130) made once for the GLOBAL batch."""
    full = torch.randn(tuple(global_shape), generator=generator, device=device)
    return full[shard_rows(global_shape[0], rank, world)].contiguous()


def allreduce_mean_(flat: torch.Tensor) -> torch.Tensor:
    """Data-parallel training (scripts/train_unet.py:181,259 — accelerate's DDP): ONE all-reduce of the flat gradient
    buffer (113.67 M fp32 for the reference U-Net; NCCL over NVLink on GPUs, gloo in the CPU tests), then the mean.
    No-op without an initialised process group or with a single rank."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return flat
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    flat.div_(dist.get_world_size())
    return flat
