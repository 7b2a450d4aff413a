"""Batch sharding of reference frames over GPUs (SURVEY.md §8e).

Every reference frame (batch element) is an independent unit — all reductions of
the sweep are over channels, views and planes *within* a frame — so the path
shards by frame with NO data-path collective.  ``torch.distributed`` (NCCL over
NVLink between GPUs, gloo in the CPU tests) is used only for the barrier around
the timed region, the MAX-reduce of the elapsed time and, optionally, gathering
results for a global check.
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist


def shard_range(total: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, balanced split of ``total`` frames: the first ``total % world``
    ranks take one extra frame."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError(f"bad rank/world {rank}/{world}")
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_tuple(tup: dict, rank: int, world: int) -> dict:
    """Slices every batched tensor of a frame tuple to this rank's frames."""
    B = tup["src_feats"].shape[0]
    lo, hi = shard_range(B, rank, world)
    out = {}
    for k, v in tup.items():
        if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == B and k not in ("min_depth", "max_depth"):
            out[k] = v[lo:hi]
        else:
            out[k] = v
    return out


def init_distributed(backend: str | None = None) -> tuple[int, int, int]:
    """(rank, world, local_rank) from the torchrun environment; initialises the
    process group when WORLD_SIZE > 1."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend)
    return rank, world, local


def bind_to_gpu_numa(local: int) -> list[int] | None:
    """Pins this process to the CPUs NVML reports as local to GPU ``local`` (its NUMA node), so
    that pinned staging buffers allocated afterwards are node-local and the cudaMemcpyAsync calls
    of every rank do not cross the socket interconnect.  Returns the CPU list, or None when NVML
    / affinity is unavailable (nothing is changed then).  Call before allocating pinned memory."""
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(local)
        ncpu = os.cpu_count() or 1
        words = pynvml.nvmlDeviceGetCpuAffinity(h, (ncpu + 63) // 64)
        cpus = [64 * wi + b for wi, word in enumerate(words) for b in range(64) if (int(word) >> b) & 1]
        allowed = os.sched_getaffinity(0)
        cpus = [c for c in cpus if c in allowed]
        if not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return cpus
    except Exception:
        return None


def barrier() -> None:
    if dist.is_initialized():
        dist.barrier()


def max_over_ranks(value: float, device=None) -> float:
    """MAX all-reduce of a scalar (the per-rank elapsed time)."""
    if not dist.is_initialized():
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64,
                     device=device if device is not None else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def sum_over_ranks(value: float, device=None) -> float:
    if not dist.is_initialized():
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64,
                     device=device if device is not None else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


def gather_frames(local: torch.Tensor) -> torch.Tensor:
    """Concatenates per-rank frame results along dim 0 (equal shards assumed);
    off the timed path, for global parity checks."""
    if not dist.is_initialized():
        return local
    outs = [torch.empty_like(local) for _ in range(dist.get_world_size())]
    dist.all_gather(outs, local.contiguous())
    return torch.cat(outs, 0)
