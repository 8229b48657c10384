"""Multi-GPU plumbing of the hot path (SURVEY.md section 8e): one process per GPU, torch.distributed.

The exchange steps are tiny and latency-bound, so they are kept to the minimum the algorithm needs:

* VAE training: contigs are sharded by rows (``shard_rows``); every optimiser step all-reduces the packed
  gradient arena ONCE (``allreduce_mean_``) between ``vk_vae_grad_step`` and ``vk_vae_dadapt_step``; all
  ranks take the same number of steps per epoch (``agree_min``); BatchNorm batch statistics stay per GPU
  and the running statistics are averaged once before ``encode`` / ``save`` (``average_running_stats_``).
* encode: independent per shard.
* clustering: independent per shard ("bins are split per sample"); no collective.

The helpers are backend-agnostic so that the host logic is covered by world_size-2 gloo tests on CPU
(tests/test_parallel_cpu.py); on GPUs the backend is NCCL over NVLink.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def shard_rows(n: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous row range [lo, hi) of ``rank``: sizes differ by at most one, earlier ranks get the extra."""
    if not (0 <= rank < world):
        raise ValueError(f"rank {rank} outside world of {world}")
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def allreduce_mean_(t: torch.Tensor, group=None) -> torch.Tensor:
    """In-place mean over the group: one collective.  NCCL averages in the collective itself;
    gloo (CPU tests) has no AVG, so it sums and scales."""
    if dist.get_backend(group) == "nccl":
        dist.all_reduce(t, op=dist.ReduceOp.AVG, group=group)
    else:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
        t.div_(dist.get_world_size(group))
    return t


def agree_min(value: int, group=None, device="cpu") -> int:
    """The smallest ``value`` over the group (every rank must take the same number of steps)."""
    t = torch.tensor([int(value)], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
    return int(t.item())


def average_running_stats_(norms, group=None) -> None:
    """Average BatchNorm running_mean / running_var of the given modules over the group."""
    for bn in norms:
        allreduce_mean_(bn.running_mean, group)
        allreduce_mean_(bn.running_var, group)


def gather_rows(local: torch.Tensor, group=None) -> torch.Tensor:
    """Concatenate row shards of possibly different lengths (all-gather of padded shards)."""
    world = dist.get_world_size(group)
    n = torch.tensor([local.shape[0]], dtype=torch.int64, device=local.device)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    sizes = [int(s.item()) for s in sizes]
    m = max(sizes)
    pad = torch.zeros((m,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad, group=group)
    return torch.cat([p[:s] for p, s in zip(parts, sizes)], 0)
