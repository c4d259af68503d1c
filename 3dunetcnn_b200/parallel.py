"""Batch-sharded data parallelism: one process per GPU, gradients averaged with one NCCL all-reduce over
NVLink/NVSwitch.  Replaces the reference's single-process ``torch.nn.DataParallel`` branch
(/root/reference/unet3d/models/build.py:18-20); GroupNorm and Dice are per-sample so the forward needs no exchange.
"""
from __future__ import annotations

import os
from typing import Iterable, List

import torch
import torch.distributed as dist


def init_process_group_from_env(backend: str | None = None) -> tuple[int, int, int]:
    """Returns (rank, world_size, local_rank); initialises torch.distributed when WORLD_SIZE > 1."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


class GradAllReduce:
    """Flat-bucket gradient averaging.  ``params`` are flattened into one contiguous fp32 buffer per call so the
    exchange is a single collective (96 MB at base_width 32: ~0.3 ms on NVSwitch, SURVEY.md 8e)."""

    def __init__(self, params: Iterable[torch.nn.Parameter], group=None, model=None):
        self.params: List[torch.nn.Parameter] = [p for p in params if p.requires_grad]
        self.group = group
        self.flat = None
        self.model = model       # a UNet3D in flat-gradient mode: its bucket IS the exchange buffer (no copies)

    def _reduce_mean(self, flat: torch.Tensor, world: int) -> None:
        if dist.get_backend(self.group) == "nccl":
            dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=self.group)     # sum and 1/world in the collective
        else:
            dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group)
            flat.mul_(1.0 / world)

    def broadcast_parameters(self, src: int = 0) -> None:
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(self.group) == 1:
            return
        for p in self.params:
            dist.broadcast(p.data, src=src, group=self.group)

    def __call__(self) -> None:
        if not (dist.is_available() and dist.is_initialized()):
            return
        world = dist.get_world_size(self.group)
        if world == 1:
            return
        bucket = self.model.flat_gradient_bucket() if self.model is not None else None
        if bucket is not None:
            lo, hi = bucket.data_ptr(), bucket.data_ptr() + bucket.numel() * 4
            if all(p.grad is not None and lo <= p.grad.data_ptr() < hi for p in self.params):
                self._reduce_mean(bucket, world)                              # gradients already live in the bucket
                return
        grads = [p.grad for p in self.params if p.grad is not None]
        if not grads:
            return
        total = sum(g.numel() for g in grads)
        if self.flat is None or self.flat.numel() != total or self.flat.device != grads[0].device:
            self.flat = torch.empty(total, dtype=torch.float32, device=grads[0].device)
        views = []
        off = 0
        for g in grads:
            v = self.flat[off:off + g.numel()].view_as(g)
            views.append(v)
            off += g.numel()
        torch._foreach_copy_(views, grads)
        self._reduce_mean(self.flat, world)
        torch._foreach_copy_(grads, views)


def shard_batch(n_items: int, rank: int, world: int) -> range:
    """Contiguous shard of ``n_items`` independent volumes for ``rank`` (weak scaling: equal shards)."""
    per = n_items // world
    rem = n_items % world
    start = rank * per + min(rank, rem)
    return range(start, start + per + (1 if rank < rem else 0))
