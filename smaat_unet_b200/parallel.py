"""Multi-GPU plumbing for the batch-sharded path (one process per GPU, torch.distributed).

The eval forward has NO data-path collective (samples are independent: BN running stats, CBAM
pools per sample -- SURVEY 8e): ranks own disjoint slices of the batch and a full copy of the
16 MB of weights.  torch.distributed (NCCL on GPUs, gloo in the CPU tests) is used only for
rendezvous, barriers and the max-over-ranks timing reduction.  The one real exchange step of
the SmaAt-UNet path -- the training gradient all-reduce -- goes through `allreduce_flat_`.
"""
from __future__ import annotations

import contextlib
import os

import numpy as np
import torch
import torch.distributed as dist


def env_rank_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def init_from_env(backend=None, device=None):
    """Initialise the default process group from torchrun's env (no-op for world size 1). Returns (rank, world, local)."""
    rank, world, local = env_rank_world()
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        backend = backend or ("nccl" if torch.cuda.is_available() else "gloo")
        kw = {"device_id": device} if (backend == "nccl" and device is not None) else {}
        dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    return rank, world, local


@contextlib.contextmanager
def process_group_from_env():
    """A command's process group under torchrun: with ``WORLD_SIZE`` > 1, each process takes the GPU of its ``LOCAL_RANK``
    and joins an NCCL group that is destroyed when the block ends.  Without torchrun's env (or with a group already
    initialised by the caller) nothing is set up or torn down.  Yields (rank, world, local)."""
    rank, world, local = env_rank_world()
    owned = world > 1 and not dist.is_initialized()
    if owned:
        torch.cuda.set_device(local)
        init_from_env("nccl", torch.device("cuda", local))
    try:
        yield rank, world, local
    finally:
        if owned:
            dist.destroy_process_group()


def rank_world():
    """(rank, world size) of the default process group; (0, 1) without one."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def _comm_device(device):
    """Where a collective's tensor lives: the rank's GPU for NCCL, the host for gloo."""
    if dist.get_backend() == "nccl":
        return device if device is not None else torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def allreduce_sum(values, device=None):
    """Elementwise sum over the ranks of a vector of host numbers, as float64 (exact for counts below 2**53).  Without a
    process group the values come back as they are."""
    v = np.asarray(values, dtype=np.float64)
    if rank_world()[1] == 1:
        return v
    t = torch.from_numpy(v.copy()).to(_comm_device(device))
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t.cpu().numpy()


def broadcast_from_rank0(obj, device=None):
    """Rank 0's ``obj`` (any picklable value) on every rank; ``obj`` itself without a process group."""
    if rank_world()[1] == 1:
        return obj
    box = [obj]
    dist.broadcast_object_list(box, src=0, device=_comm_device(device))
    return box[0]


def broadcast_tensors_(tensors, device=None):
    """Overwrite ``tensors`` (same device on every rank) with rank 0's values in place: one broadcast per dtype."""
    if rank_world()[1] == 1:
        return
    by_dtype = {}
    for t in tensors:
        by_dtype.setdefault(t.dtype, []).append(t)
    with torch.no_grad():
        for group in by_dtype.values():
            flat = torch.cat([t.reshape(-1) for t in group]).to(_comm_device(device))
            dist.broadcast(flat, src=0)
            off = 0
            for t in group:
                t.copy_(flat[off:off + t.numel()].view_as(t))
                off += t.numel()


def shard_range(n_items: int, rank: int, world: int):
    """Contiguous, balanced [lo, hi) slice of n_items for this rank (first n % world ranks get one extra)."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def barrier(device=None):
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        if device is not None and device.type == "cuda":
            dist.barrier(device_ids=[device.index])
        else:
            dist.barrier()
    if device is not None and device.type == "cuda":
        torch.cuda.synchronize(device)


def reduce_max(value: float, device=None) -> float:
    """max over ranks of a host scalar (timings are reported as the slowest rank's)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([value], dtype=torch.float64, device=device if device is not None else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def allreduce_flat_(tensors, average=True):
    """One all-reduce of a flat bucket holding all `tensors` (training gradients: 4 033 537 fp32 = 16 MB for
    SmaAt-UNet, a single bucket -- SURVEY 5).  In place; returns the number of elements reduced."""
    tensors = [t for t in tensors if t is not None]
    if not tensors:
        return 0
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return sum(t.numel() for t in tensors)
    flat = torch.cat([t.reshape(-1) for t in tensors])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    if average:
        flat /= dist.get_world_size()
    off = 0
    for t in tensors:
        n = t.numel()
        t.copy_(flat[off:off + n].view_as(t))
        off += n
    return off
