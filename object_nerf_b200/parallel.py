"""Ray-sharded multi-GPU inference: rays are independent units (no cross-ray operation anywhere on the path),
so each rank renders a contiguous tile of the frame and the tiles are gathered with one collective
(SURVEY.md §8e).  One process per GPU, torch.distributed (NCCL on GPUs; gloo in the CPU tests of the
sharding logic)."""
from __future__ import annotations

from typing import Callable, Dict, Sequence

import torch
import torch.distributed as dist


def shard_bounds(n_rays: int, world_size: int, rank: int):
    """Contiguous, balanced partition: the first (n_rays % world_size) ranks get one extra ray."""
    base, rem = divmod(n_rays, world_size)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def tile_bounds(n_rays: int, group=None):
    """The rows this rank renders: all of them without a group, its shard_bounds with one."""
    if group is None:
        return 0, n_rays
    return shard_bounds(n_rays, dist.get_world_size(group), dist.get_rank(group))


def gather_tiles(local: torch.Tensor, n_rays: int, group=None) -> torch.Tensor:
    """All-gather ragged row tiles (shard_bounds order) into the full (n_rays, ...) tensor on every rank."""
    world = dist.get_world_size(group)
    sizes = [shard_bounds(n_rays, world, r) for r in range(world)]
    longest = max(b - a for a, b in sizes)
    padded = local
    if local.shape[0] < longest:
        pad = torch.zeros((longest - local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        padded = torch.cat([local, pad], 0)
    out = [torch.empty_like(padded) for _ in range(world)]
    dist.all_gather(out, padded.contiguous(), group=group)
    return torch.cat([o[: b - a] for o, (a, b) in zip(out, sizes)], 0)


def gather_tile_maps(maps: Dict[str, torch.Tensor], n_rays: int, group=None) -> Dict[str, torch.Tensor]:
    """gather_tiles of every tensor of `maps`; without a group, `maps` as they are (a new dict)."""
    if group is None:
        return dict(maps)
    return {k: gather_tiles(v, n_rays, group) for k, v in maps.items()}


def render_sharded(render_fn: Callable[[torch.Tensor, Dict[str, torch.Tensor]], Dict[str, torch.Tensor]],
                   rays: torch.Tensor, per_ray: Dict[str, torch.Tensor], keys: Sequence[str], group=None):
    """render_fn(rays_tile, per_ray_tile) -> result dict (e.g. a closure over render_rays / render_rays_multi);
    every rank holds the full `rays`; returns {key: full (N, ...) tensor} gathered on all ranks."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n = rays.shape[0]
    a, b = shard_bounds(n, world, rank)
    res = render_fn(rays[a:b], {k: v[a:b] for k, v in per_ray.items()})
    return {k: gather_tiles(res[k], n, group) for k in keys}
