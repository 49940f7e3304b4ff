"""Data-parallel plumbing over torch.distributed (NCCL on GPUs / gloo in CPU tests).

Replaces the Horovod calls on the hot path (CLIP-ViP/src/utils/distributed.py, run_pretrain.py:226-232,344-353):
one process per GPU, rank-major differentiable all-gather of the embeddings, bucketed gradient averaging.
"""
from __future__ import annotations

import os
from typing import Iterable, Optional

import torch
import torch.distributed as dist


def init_from_env(backend: Optional[str] = None) -> tuple:
    """torchrun-style initialisation (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_*).  Returns (rank, local_rank, world)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend)
    return rank, local, world


def world_size(group=None) -> int:
    return dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1


class _AllGather(torch.autograd.Function):
    """hvd.allgather semantics (run_pretrain.py:344-345): forward = rank-major concat along dim 0.
    Backward = the local slice of the incoming gradient times `grad_scale` (default: world size), which equals
    all_reduce(SUM)+slice of LF-VILA's SyncFunction (LF-VILA/src/utils/dist.py:35-41) whenever every rank
    back-propagates the same loss of the same gathered tensors — the case on this path — without a collective."""

    @staticmethod
    def forward(ctx, t, group, grad_scale):
        world = world_size(group)
        ctx.meta = (dist.get_rank(group) if world > 1 else 0, t.shape[0], float(world if grad_scale is None else grad_scale))
        if world == 1:
            return t.clone()
        out = torch.empty((world * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(out, t.contiguous(), group=group)
        return out

    @staticmethod
    def backward(ctx, grad):
        rank, b, scale = ctx.meta
        return grad[rank * b:(rank + 1) * b] * scale, None, None


def allgather(t: torch.Tensor, group=None, grad_scale: Optional[float] = None) -> torch.Tensor:
    return _AllGather.apply(t, group, grad_scale)


def average_gradients(params: Iterable[torch.nn.Parameter], group=None, bucket_bytes: int = 256 << 20) -> None:
    """hvd.DistributedOptimizer's gradient averaging (run_pretrain.py:226-228,379): flat fp32 buckets, one
    all-reduce each (NVLS in-switch reduction when NCCL selects it), divided by the world size."""
    world = world_size(group)
    if world == 1:
        return
    bucket, size = [], 0
    def flush():
        nonlocal bucket, size
        if not bucket:
            return
        flat = torch.cat([g.reshape(-1) for g in bucket])
        dist.all_reduce(flat, group=group)
        flat.div_(world)
        off = 0
        for g in bucket:
            g.copy_(flat[off:off + g.numel()].view_as(g))
            off += g.numel()
        bucket, size = [], 0
    for p in params:
        if p.grad is None:
            continue
        bucket.append(p.grad)
        size += p.grad.numel() * p.grad.element_size()
        if size >= bucket_bytes:
            flush()
    flush()


class OverlappedGradAverager:
    """`model.clipmodel.grad_ready_hook = OverlappedGradAverager()` averages parameter gradients across ranks WHILE
    backward is still running: every finished gradient group arrives as one flat fp32 buffer and is all-reduced
    (ReduceOp.AVG) asynchronously on NCCL's stream; `finish()` (called at the end of the model's backward) makes
    the compute stream wait for the outstanding collectives.  Equivalent to hvd.DistributedOptimizer's backward
    hooks + synchronize() (run_pretrain.py:226-228,379)."""

    def __init__(self, group=None, comm_dtype=None):
        """comm_dtype=torch.bfloat16 halves the bytes on the wire (and the time NCCL's CTAs compete with the backward GEMMs):
        each bucket is cast to bf16, averaged, and written back into the fp32 gradient buffer.  The reference's own
        all-reduce runs on fp16 gradients (apex O2 model gradients, run_pretrain.py:234-236); the default keeps fp32."""
        self.group = group
        self.comm_dtype = comm_dtype
        self.pending = []

    def __call__(self, flat: torch.Tensor) -> None:
        if world_size(self.group) == 1:
            return
        if self.comm_dtype is not None and self.comm_dtype != flat.dtype:
            buf = flat.to(self.comm_dtype)
            work = dist.all_reduce(buf, op=dist.ReduceOp.AVG, group=self.group, async_op=True)
            self.pending.append((work, buf, flat))
        else:
            self.pending.append((dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=self.group, async_op=True), None, None))

    def finish(self) -> None:
        for work, buf, flat in self.pending:
            work.wait()
            if buf is not None:
                flat.copy_(buf)
        self.pending = []
