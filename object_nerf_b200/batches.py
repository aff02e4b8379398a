"""Training batches drawn on the device (GenericDataset.__getitem__ through DataLoader(shuffle=True) in the reference,
datasets/generic_dataset.py:475-490 and train.py:121-129).

`RaySampler` uploads a training dataset's ray buffers once (or, with `from_frames`, draws from a frames.FrameSet and
rebuilds each row from its pixel: onerf_draw_frames_dstep, the same batches bit for bit).  Each `next()` is one kernel
(onerf_draw_batch_dstep) that draws the batch of the sampler's device step counter into fixed output buffers and
advances the counter.  It reads
nothing back to the host, so `next()` + `training.train_step` + `Adam(capturable=True)` capture in one CUDA graph, and
each replay trains on the next batch.

What a batch holds matches the reference: every epoch is a fresh shuffle of all R rays cut into batches of B, and every
drawn ray takes its instance-specific fields (instance_mask, instance_mask_weight, instance_ids, pass_through_mask) from
one instance column drawn uniformly from [0, I).  Under DDP every rank shuffles with the same permutation and takes a
disjoint stride of it (DistributedSampler).  Two differences are deliberate:
  - the draws come from the library's Philox (a keyed Feistel permutation per epoch, include/onerf_ext.h), not from
    torch's generator: the distribution is the reference's, the bits are not;
  - an epoch has P = floor(R / (B * W)) full batches (W ranks).  The reference ends each epoch with one partial batch
    (drop_last=False); a captured graph needs a fixed batch size.  Each epoch is a new permutation, so every ray has the
    same chance of being among the R - P*B*W rays an epoch leaves out.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch

from . import _lib, engine

__all__ = ["RaySampler"]

DATASET_KEYS = {"all_rays": "rays", "all_rgbs": "rgbs", "all_depths": "depths", "all_valid_masks": "valid_mask",
                "all_instance_masks": "instance_mask", "all_instance_masks_weight": "instance_mask_weight",
                "all_instance_ids": "instance_ids", "all_pass_through_masks": "pass_through_mask"}
COLUMN_KEYS = ("instance_mask", "instance_mask_weight", "instance_ids", "pass_through_mask")
MAX_RAYS = 1 << 40


def _column_fields(t: torch.Tensor, n: int, name: str):
    if t.dim() == 1:
        t = t.reshape(n, 1)
    if t.dim() != 2:
        raise ValueError(f"{name} must be (R,) or (R, I), got shape {tuple(t.shape)}")
    return t


def _group_rank(rank, world_size, group):
    """(rank, world_size), taken from `group` when one is given."""
    if group is None:
        return rank, world_size
    import torch.distributed as dist
    g_rank, g_world = dist.get_rank(group), dist.get_world_size(group)
    if (rank, world_size) not in ((0, 1), (g_rank, g_world)):
        raise ValueError(f"RaySampler: rank {rank} / world_size {world_size} disagree with the group's "
                         f"{g_rank} / {g_world}")
    return g_rank, g_world


def _check_batch(R, batch_size, rank, world_size):
    B, W = int(batch_size), int(world_size)
    if B < 1 or W < 1 or not 0 <= rank < W:
        raise ValueError(f"RaySampler: bad batch_size {B}, world_size {W} or rank {rank}")
    if R < B * W:
        raise ValueError(f"RaySampler: {R} rays hold no full batch of {B} rays on each of {W} ranks")
    if R >= MAX_RAYS:
        raise ValueError(f"RaySampler: {R} rays; at most 2^40 - 1 are supported")


class RaySampler:
    """Device-resident training batches of a GenericDataset's ray buffers.

    tensors     dict keyed by GenericDataset's attribute names: all_rays (R,8), all_rgbs (R,3), all_depths (R,),
                all_valid_masks (R,), all_instance_masks, all_instance_masks_weight, all_instance_ids and
                all_pass_through_masks (R,I) or (R,) for I = 1, and optionally all_frame_indices (R,).  Uploaded once:
                masks as uint8 (non-zero -> 1), float fields as float32, ids as int64.
    seed        Philox seed of the permutations and column draws; None draws one from torch's generator.  With `group`,
                rank 0's seed is broadcast once here, so every rank shares the permutation.
    rank, world_size  this rank's stride of every epoch; taken from `group` when one is given.

    `next()` returns the batch as a dict of device tensors with the reference's collated keys and shapes (the tensors
    are fixed buffers, overwritten by the next call)."""

    def __init__(self, tensors: Dict[str, torch.Tensor], batch_size: int = 2048, device="cuda", seed=None,
                 rank: int = 0, world_size: int = 1, group=None):
        missing = [k for k in DATASET_KEYS if k not in tensors]
        if missing:
            raise ValueError(f"RaySampler: missing dataset buffers {missing}")
        rank, world_size = _group_rank(rank, world_size, group)
        rays = tensors["all_rays"].reshape(-1, 8)
        R = rays.shape[0]
        src = {"rays": rays}
        for k, name in DATASET_KEYS.items():
            t = tensors[k]
            if t.shape[0] != R:
                raise ValueError(f"RaySampler: {k} has {t.shape[0]} rows, all_rays has {R}")
            if name in COLUMN_KEYS:
                src[name] = _column_fields(t, R, k)
            elif name != "rays":
                src[name] = t.reshape(R, 3) if name == "rgbs" else t.reshape(R)
        if tensors.get("all_frame_indices") is not None:
            if tensors["all_frame_indices"].shape[0] != R:
                raise ValueError(f"RaySampler: all_frame_indices has {tensors['all_frame_indices'].shape[0]} rows, "
                                 f"all_rays has {R}")
            src["frame_idx"] = tensors["all_frame_indices"].reshape(R)
        I = src["instance_mask"].shape[1]
        if any(src[k].shape[1] != I for k in COLUMN_KEYS):
            raise ValueError("RaySampler: the per-instance buffers differ in their number of instance columns: "
                             + ", ".join(f"{k} {src[k].shape[1]}" for k in COLUMN_KEYS))
        if I < 1:
            raise ValueError("RaySampler: the dataset has no instance column (I = 0)")
        _check_batch(R, batch_size, rank, world_size)

        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self._setup(dev, R, I, batch_size, rank, world_size, seed, group)

        def up(t, kind):
            t = t.to(dev)
            if kind == "mask":
                return (t != 0).to(torch.uint8).contiguous()
            return t.to(torch.float32 if kind == "float" else torch.int64).contiguous()

        kinds = {"rays": "float", "rgbs": "float", "depths": "float", "valid_mask": "mask", "frame_idx": "int",
                 "instance_mask": "mask", "instance_mask_weight": "float", "instance_ids": "int",
                 "pass_through_mask": "mask"}
        self.buffers = {k: up(t, kinds[k]) for k, t in src.items()}
        d = self._args.data
        d.n_rays, d.n_instances = R, I
        for k in kinds:
            setattr(d, k, self.buffers[k].data_ptr() if k in self.buffers else None)

    def _setup(self, dev, R, I, batch_size, rank, world_size, seed, group):
        """Counters, seed and the fixed output buffers; the dataset part of the argument block is the caller's."""
        B, W = int(batch_size), int(world_size)
        self.device, self.batch_size, self.rank, self.world_size = dev, B, int(rank), W
        self.n_rays, self.n_instances = R, I
        self.batches_per_epoch = R // (B * W)
        self.frames = None

        if seed is None:
            seed = engine.new_seed()
        if group is not None:
            import torch.distributed as dist
            on_dev = dist.get_backend(group) == "nccl"
            t = torch.tensor([int(seed)], dtype=torch.int64, device=dev if on_dev else "cpu")
            dist.broadcast(t, group_src=0, group=group)
            seed = int(t.item())
        self.seed = int(seed) & (2 ** 64 - 1)

        f = lambda *shape, dtype: torch.empty(*shape, dtype=dtype, device=dev)
        self._out = {"rays": f(B, 8, dtype=torch.float32), "rgbs": f(B, 3, dtype=torch.float32),
                     "depths": f(B, dtype=torch.float32), "valid_mask": f(B, dtype=torch.uint8),
                     "frame_idx": f(B, dtype=torch.int64), "instance_mask": f(B, dtype=torch.uint8),
                     "instance_mask_weight": f(B, dtype=torch.float32), "instance_ids": f(B, dtype=torch.int64),
                     "pass_through_mask": f(B, dtype=torch.uint8)}
        self._step = torch.zeros(1, dtype=torch.int64, device=dev)
        # the reference's collated shapes; masks as bool views of the uint8 buffers the kernel writes
        o = self._out
        self._batch = {"rays": o["rays"], "rgbs": o["rgbs"], "depths": o["depths"],
                       "valid_mask": o["valid_mask"].view(torch.bool), "frame_idx": o["frame_idx"],
                       "instance_mask": o["instance_mask"].view(torch.bool).view(B, 1),
                       "instance_mask_weight": o["instance_mask_weight"].view(B, 1),
                       "instance_ids": o["instance_ids"].view(B, 1),
                       "pass_through_mask": o["pass_through_mask"].view(torch.bool).view(B, 1)}
        a = _lib.BatchArgs()
        a.batch, a.rank, a.world, a.seed = B, self.rank, W, self.seed
        for k, t in o.items():
            setattr(a, k, t.data_ptr())
        self._args = a

    @classmethod
    def from_dataset(cls, dataset, **kw) -> "RaySampler":
        """A sampler over a GenericDataset's training buffers (or any object with its all_* attributes)."""
        names = list(DATASET_KEYS) + ["all_frame_indices"]
        return cls({k: getattr(dataset, k) for k in names if getattr(dataset, k, None) is not None}, **kw)

    @classmethod
    def from_frames(cls, frame_set, batch_size: int = 2048, device=None, seed=None, rank: int = 0,
                    world_size: int = 1, group=None) -> "RaySampler":
        """A sampler over a frames.FrameSet: the same batches as RaySampler(frame_set.expand(), ...) with the same
        seed, bit for bit, each row rebuilt from the frame store on the device (onerf_draw_frames_dstep) instead of
        read from per-ray buffers.  device: the frame set's (the default); another one is refused."""
        rank, world_size = _group_rank(rank, world_size, group)
        _check_batch(frame_set.n_rays, batch_size, rank, world_size)
        if device is not None and torch.device(device) not in (frame_set.device, torch.device(frame_set.device.type)):
            raise ValueError(f"RaySampler.from_frames: the frame set lives on {frame_set.device}, not {device}")
        self = cls.__new__(cls)
        self._setup(frame_set.device, frame_set.n_rays, frame_set.n_instances, batch_size, rank, world_size, seed,
                    group)
        self.frames, self.buffers = frame_set, {}
        return self

    def next(self) -> Dict[str, torch.Tensor]:
        """Draw the batch of the device step counter and advance the counter by one (kernels only: capturable)."""
        if self.frames is None:
            _lib.call("onerf_draw_batch_dstep", self.device, C.byref(self._args), self._step.data_ptr())
        else:
            _lib.call("onerf_draw_frames_dstep", self.device, C.byref(self.frames.args), C.byref(self._args),
                      self._step.data_ptr())
        return dict(self._batch)

    @property
    def step(self) -> int:
        """The counter: batches drawn so far (synchronises; meant for epoch-boundary hooks)."""
        return int(self._step.item())

    @property
    def epoch(self) -> int:
        return self.step // self.batches_per_epoch

    def set_step(self, k: int) -> None:
        """Set the counter (eagerly), e.g. to resume at batch k."""
        self._step.fill_(int(k))
