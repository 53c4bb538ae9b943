"""Multi-GPU plumbing of the training step (SURVEY 8e): the reference trains data-parallel over pids under
PyTorch-Lightning DDP -- rank r owns `np.array_split(pids, world)[r]` (datasets/samplers/distributed_pids_sampler.py:71),
losses are computed on the local P x K batch only, and ONE gradient all-reduce (mean) over all parameters follows
the backward.  The H100 trunk produces every parameter gradient at the end of its single backward call, so there
is nothing to overlap bucket by bucket: the gradients are packed into a few large flat fp32 buckets and reduced
with torch.distributed (NCCL on GPUs; gloo in the CPU tests).  Wrapping the module in torch DDP works too (its hooks
fire on the same `.grad`s); this helper is the dependency-free form.
"""
from __future__ import annotations

from typing import Iterable, List, Optional

import numpy as np
import torch
import torch.distributed as dist


def shard_pids(pids, world_size: int, rank: int) -> np.ndarray:
    """distributed_pids_sampler.py:66-72: contiguous, near-equal split of the (already shuffled) pid list."""
    return np.array_split(np.asarray(pids), world_size)[rank]


def allreduce_gradients(params: Iterable[torch.nn.Parameter], group=None, bucket_bytes: int = 256 << 20,
                        average: bool = True) -> int:
    """In-place mean (or sum) of `.grad` over the process group, through flat fp32 buckets.  Parameters whose
    gradient is None on this rank contribute zeros (DDP's find_unused_parameters semantics are NOT provided: the set
    of parameters with gradients must be the same on every rank, as it is for the CTL step).  Returns the number of
    collectives issued."""
    if not dist.is_available() or not dist.is_initialized():
        return 0
    world = dist.get_world_size(group)
    if world == 1:
        return 0
    grads: List[torch.Tensor] = [p.grad for p in params if p.grad is not None]
    if not grads:
        return 0
    calls = 0
    start = 0
    while start < len(grads):
        size, end = 0, start
        while end < len(grads) and (end == start or size + grads[end].numel() * 4 <= bucket_bytes):
            size += grads[end].numel() * 4
            end += 1
        bucket = grads[start:end]
        flat = torch.cat([g.detach().reshape(-1).float() for g in bucket])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        if average:
            flat.div_(world)
        off = 0
        for g in bucket:
            n = g.numel()
            g.copy_(flat[off:off + n].view_as(g))
            off += n
        calls += 1
        start = end
    return calls


class GradientReducer:
    """Mean all-reduce of every parameter gradient through ONE persistent flat fp32 buffer, with no copy-back: after
    the backward the gradients are packed by a single multi-tensor copy, the flat buffer is reduced in place (NCCL
    ReduceOp.AVG; SUM + divide on backends without AVG) and each `p.grad` is re-pointed at its slice of the buffer, which
    is what the fused optimizers (solver/build.py) then read.  One collective of ~26.6 M floats per step
    (distributed_pids_sampler.py:61-71 + PL DDP in the reference, utils/misc.py:101-119).

    The trunk's backward is one captured CUDA graph that delivers all gradients at once, so there is no per-layer
    bucket to overlap with; the reduction itself runs at NVLink speed (106 MB)."""

    def __init__(self, params: Iterable[torch.nn.Parameter], group=None):
        self.params = [p for p in params if p.requires_grad]
        self.group = group
        self.flat: Optional[torch.Tensor] = None
        self.views: List[torch.Tensor] = []

    def _ensure(self, grads):
        total = sum(g.numel() for g in grads)
        if self.flat is None or self.flat.numel() != total or self.flat.device != grads[0].device:
            self.flat = torch.empty(total, dtype=torch.float32, device=grads[0].device)
            self.views, off = [], 0
            for g in grads:
                self.views.append(self.flat[off:off + g.numel()].view_as(g))
                off += g.numel()

    def allreduce_mean(self) -> int:
        if not dist.is_available() or not dist.is_initialized():
            return 0
        world = dist.get_world_size(self.group)
        if world == 1:
            return 0
        owners = [p for p in self.params if p.grad is not None]
        grads = [p.grad for p in owners]
        if not grads:
            return 0
        self._ensure(grads)
        fresh = [(v, g) for v, g in zip(self.views, grads) if g.data_ptr() != v.data_ptr()]
        if fresh:
            torch._foreach_copy_([v for v, _ in fresh], [g.detach().float() if g.dtype != torch.float32 else g.detach() for _, g in fresh])
        backend = dist.get_backend(self.group)
        if backend == "nccl":
            dist.all_reduce(self.flat, op=dist.ReduceOp.AVG, group=self.group)
        else:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group)
            self.flat.div_(world)
        for p, v in zip(owners, self.views):
            p.grad = v
        return 1
