"""Embedding modules with the reference's names / buffers (reference models/embedding_helper.py).

`Embedding` is a marker for plain positional encoding; `EmbeddingVoxel` owns the sparse voxel grid
(feature table + dense index map + metadata buffers, same state_dict keys as the reference) and builds
it from a point cloud at construction time (cold path).  The per-sample encoding itself runs inside the
fused CUDA kernels; calling these modules directly uses the stand-alone encode kernel.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from . import engine


class Embedding(nn.Module):
    """[x, sin(2^k x), cos(2^k x)]_k, reference :40-74.  Supported: in_channels=3 with 10 or 4 octaves."""

    def __init__(self, in_channels, N_freqs, logscale=True):
        super().__init__()
        if not logscale:
            raise RuntimeError("only log-scale frequency bands are built")
        self.N_freqs, self.in_channels = N_freqs, in_channels
        self.out_channels = in_channels * (2 * N_freqs + 1)

    def forward(self, x):
        """(..., 3) CUDA -> (..., 63) for PE10 (positions) or (..., 27) for PE4 (directions).  The output remembers its
        source (`_onerf_src` = (points (B,3), self)), so that ObjectNeRF.forward / forward_instance on it run the fused
        kernel on the points / directions."""
        if self.in_channels == 3 and self.N_freqs in (10, 4) and x.is_cuda:
            pts = x.reshape(-1, 3)
            if self.N_freqs == 10:
                out = engine.encode(pts, None)[0]
            else:
                out = engine.dir_encode(pts)
            out = out.reshape(*x.shape[:-1], self.out_channels)
            out._onerf_src = (pts, self)
            return out
        raise NotImplementedError("stand-alone Embedding.forward is built for in_channels=3 with 10 (positions) or 4 "
                                  "(directions) octaves, on CUDA tensors")


class EmbeddingVoxel(nn.Module):
    def __init__(self, channels, N_freqs, max_voxels, dataset_extra_config, points=None):
        super().__init__()
        if (channels, N_freqs) != (24, 6):
            raise RuntimeError("object_nerf_b200 kernels are built for 24 voxel channels with PE 6")
        self.channels = channels
        self.instance_ftr_C = 8
        self.embedding_space_ftr = nn.Embedding(max_voxels, channels)
        self.conf = dataset_extra_config
        self.set_pointclouds(dataset_extra_config, points)

    # ---- cold path: grid construction (reference :86-200) ----
    def set_pointclouds(self, conf, points=None):
        if points is None:
            import open3d as o3d  # only needed to read the .ply the dataset config names
            points = np.asarray(o3d.io.read_point_cloud(conf["pcd_path"]).points)
        scale = conf["scale_factor"]
        pts = torch.from_numpy((np.asarray(points) - np.array(conf["scene_center"])) / scale).float()
        vsize = torch.scalar_tensor(conf["voxel_size"] / scale)
        lo, hi = pts.min(0)[0], pts.max(0)[0]
        self.register_buffer("voxel_size", vsize)
        self.register_buffer("bounds", torch.stack([lo, hi]))
        self.register_buffer("voxel_offset", -lo)
        shape = [int(((hi[i] - lo[i]) / vsize).int().item()) + 3 for i in range(3)]
        self.register_buffer("voxel_shape", torch.tensor(shape))
        self.register_buffer("voxel_count", torch.scalar_tensor(int(np.prod(shape))))
        occ = torch.zeros(shape, dtype=torch.bool)
        q = ((pts + self.voxel_offset) / vsize).round().long()
        ok = ((q >= 0) & (q < torch.tensor(shape))).all(1)
        q = q[ok]
        occ[q[:, 0], q[:, 1], q[:, 2]] = True
        # mark the neighbourhood of every occupied cell (box dilation)
        k = int(conf["neighbor_marks"])
        occ = F.max_pool3d(occ[None, None].float(), kernel_size=k, stride=1, padding=(k - 1) // 2)[0, 0] > 0
        self.register_buffer("voxel_occupancy", occ)
        self.generate_voxel_idx_map()

    def generate_voxel_idx_map(self):
        occ = self.voxel_occupancy
        cells = torch.nonzero(occ)
        if cells.shape[0] > self.embedding_space_ftr.num_embeddings:
            raise RuntimeError("more occupied voxels than N_max_voxels")
        idx = torch.full(tuple(occ.shape), -1, dtype=torch.long, device=occ.device)
        idx[cells[:, 0], cells[:, 1], cells[:, 2]] = torch.arange(cells.shape[0], device=occ.device)
        self.register_buffer("voxel_idx_map", idx)

    def grid_buffers(self) -> engine.GridBuffers:
        return engine.GridBuffers.from_module(self)

    def forward(self, xyz):
        """(B,3) -> (scene input (B,271), object voxel input (B,104)), reference :325-329.  The returned tensors remember
        the positions and grid they were encoded from, so that ObjectNeRF.forward(..., sigma_only=True) on them (the
        mesh-extraction call pattern, tools/extract_mesh.py:83-109) runs the fused encode + MLP kernel on the positions."""
        pts = xyz.reshape(-1, 3)
        scene, obj = engine.encode(pts, engine.GridBuffers.from_module(self))
        scene._onerf_src = obj._onerf_src = (pts, self)
        return scene, obj

    # ---- cold path at epoch boundaries: grid maintenance (reference :202-302, called from train.py:140-145) ----
    def _occupied(self):
        idx_occu = torch.nonzero(self.voxel_occupancy)
        voxel_xyz = idx_occu.float() * self.voxel_size - self.voxel_offset
        return idx_occu, voxel_xyz

    def self_pruning_empty_voxels(self, model, max_alpha_th=0.5, precision=None, _rand=None, _sigma_fn=None, *,
                                  seed=None, group=None):
        """Reference :202-245: drop every occupied voxel whose largest alpha over 16^3 jittered samples
        (`1 - exp(-relu(sigma))`, scene branch of `model`) stays below max_alpha_th: occupancy -> False, index map -> -1.
        Returns the number of voxels dropped (one host read).  Table rows are not renumbered.

        The pass runs on the device in two library calls (include/onerf_ext.h): onerf_prune_measure generates every
        voxel's samples and reduces them to the voxel's largest alpha (bf16: one fused tensor-core launch that evaluates
        only the layers sigma needs; fp32: the FFMA field chunk by chunk), onerf_prune_apply clears the cells below the
        threshold.  The density is the scene branch's, as `self.forward` + `model(..., sigma_only=True)` intend
        (upstream's call at :223 passes a tensor to `forward(inputs: dict)`).
          precision  arithmetic of the density (None = the library default).
          seed       Philox seed of the jitter (None: engine.new_seed(), so torch.manual_seed makes a run reproducible).
                     The jitter has torch.rand_like's distribution, not its bits.
          group      torch.distributed process group: rank 0's seed is broadcast, rank r measures the voxels
                     parallel.shard_bounds(K, W, r), the maxima are all-gathered and every rank applies the same mask,
                     so the grids stay identical across ranks.  A grouped train_step still wants sync_replicas after it
                     (training.py: any grid change).
          _rand      list of U[0,1) tensors, one (32 * 4096, 3) block per 32-voxel chunk: the jitter instead of Philox
                     (tests).
          _sigma_fn  xyz -> sigma: the reference's host loop over 32-voxel chunks with this density (CPU tests of the
                     grid logic)."""
        if _sigma_fn is None:
            return self._prune_on_device(model, max_alpha_th, precision, _rand, seed, group)
        if group is not None:
            raise ValueError("group= needs the device pass: _sigma_fn runs the host loop on one process")
        idx_occu, voxel_xyz = self._occupied()
        n_occu = voxel_xyz.shape[0]
        n_per_voxel, per_batch = 16 ** 3, 32
        empty = []
        for k, i in enumerate(range(0, n_occu, per_batch)):
            centres = voxel_xyz[i:i + per_batch]
            samples = centres[:, None, :].expand(-1, n_per_voxel, -1).reshape(-1, 3).clone()
            r = _rand[k][:samples.shape[0]].to(samples) if _rand is not None else torch.rand_like(samples)
            samples += r * self.voxel_size - self.voxel_size / 2
            sigmas = _sigma_fn(samples).reshape(-1)
            alphas = 1 - torch.exp(-torch.relu(sigmas))
            empty.append(alphas.view(-1, n_per_voxel).max(-1)[0] < max_alpha_th)
        empty_mask = torch.cat(empty, 0) if empty else torch.zeros(0, dtype=torch.bool, device=voxel_xyz.device)
        idx_empty = idx_occu[empty_mask, :]
        self.voxel_occupancy[idx_empty[:, 0], idx_empty[:, 1], idx_empty[:, 2]] = False
        self.voxel_idx_map[idx_empty[:, 0], idx_empty[:, 1], idx_empty[:, 2]] = -1
        return int(idx_empty.shape[0])

    def _prune_on_device(self, model, max_alpha_th, precision, _rand, seed, group):
        from . import _lib, parallel
        occ = self.voxel_occupancy
        cells = torch.nonzero(occ).contiguous()        # (CPU nonzero returns a column-major result)
        n_cells = cells.shape[0]
        if n_cells == 0:
            return 0
        dev = occ.device
        jitter = None
        if _rand is not None:
            # block i holds chunk i's rows: concatenated, row k * 4096 + s is sample s of voxel k
            per = 32 * _lib.PRUNE_SAMPLES
            blocks = [r[:min(per, (n_cells - i * 32) * _lib.PRUNE_SAMPLES)] for i, r in enumerate(_rand[:(n_cells + 31) // 32])]
            jitter = torch.cat(blocks).to(device=dev, dtype=torch.float32).contiguous()
            if jitter.shape != (n_cells * _lib.PRUNE_SAMPLES, 3):
                raise ValueError(f"_rand holds {jitter.shape[0]} jitter rows for {n_cells} voxels x 4096 samples")
            seed = 0
        elif seed is None:
            seed = engine.new_seed()
        if group is not None and jitter is None:
            import torch.distributed as dist
            t = torch.tensor([seed], dtype=torch.int64, device=dev)
            dist.broadcast(t, group_src=0, group=group)
            seed = int(t.item())
        begin, end = parallel.tile_bounds(n_cells, group)
        max_alpha = torch.zeros(end - begin, dtype=torch.float32, device=dev)
        grid = self.grid_buffers()
        packed = engine.packed_for(model, True)
        prec = engine.PRECISIONS[precision or engine.default_precision()]
        ws = torch.empty(_lib.load().onerf_prune_workspace_bytes(prec), dtype=torch.uint8, device=dev)
        a = _lib.PruneArgs()
        a.grid, a.packed, a.precision = C.pointer(grid.c), packed.data_ptr(), prec
        a.cells, a.n_cells, a.cell_begin, a.cell_end = _lib.ptr(cells), n_cells, begin, end
        a.jitter, a.seed = _lib.ptr(jitter), seed
        a.max_alpha_out = _lib.ptr(max_alpha)
        a.workspace, a.workspace_bytes = (ws.data_ptr() if ws.numel() else None), ws.numel()
        _lib.call("onerf_prune_measure", dev, C.byref(a))
        if group is not None:
            max_alpha = parallel.gather_tiles(max_alpha, n_cells, group)
        n_pruned = torch.zeros(1, dtype=torch.int64, device=dev)
        _lib.call("onerf_prune_apply", dev, _lib.ptr(cells), n_cells, _lib.ptr(max_alpha), float(max_alpha_th), occ.shape[1],
                  occ.shape[2], _lib.ptr(occ), _lib.ptr(self.voxel_idx_map), n_pruned.data_ptr())
        # the library wrote the buffers in place: count it as an in-place change (training._grid_stamp)
        torch.autograd.graph.increment_version(occ)
        torch.autograd.graph.increment_version(self.voxel_idx_map)
        return int(n_pruned.item())

    def voxel_subdivision(self, _features_fn=None):
        """Reference :247-302: halve the voxel size.  Every occupied voxel spawns its 8 children
        (itertools.product([0, 1], repeat=3) order), whose features are the trilinear samples of the OLD grid at the
        child positions (raw features, no positional encoding: `onerf_voxel_features`); occupancy / index map are
        rebuilt at twice the resolution and the children's rows written into the feature table.  More children than
        table rows raises RuntimeError with every buffer and the table unchanged."""
        idx_occu, voxel_xyz = self._occupied()
        dev = voxel_xyz.device
        target = self.voxel_size / 2
        new_xyz = []
        for cx in (0, 1):
            for cy in (0, 1):
                for cz in (0, 1):
                    new_xyz.append(voxel_xyz + torch.tensor([cx, cy, cz], device=dev) * target)
        new_xyz = torch.cat(new_xyz, 0)
        new_coord = ((new_xyz + self.voxel_offset) / target).round().long()
        features_fn = _features_fn or (lambda pts: engine.voxel_features(pts, self.grid_buffers()))
        with torch.no_grad():
            new_ftrs = features_fn(new_xyz)
        occ = torch.zeros([2 * int(v) for v in self.voxel_shape], dtype=torch.bool, device=dev)
        occ[new_coord[:, 0], new_coord[:, 1], new_coord[:, 2]] = True
        # refuse before touching any buffer: a failed call leaves the old grid whole (the index map matches the shape)
        if int(occ.sum()) > self.embedding_space_ftr.num_embeddings:
            raise RuntimeError("more occupied voxels than N_max_voxels")
        self.voxel_size = target
        self.voxel_shape *= 2
        self.voxel_occupancy = occ
        self.voxel_count = self.voxel_shape[0] * self.voxel_shape[1] * self.voxel_shape[2]
        self.generate_voxel_idx_map()
        with torch.no_grad():
            assign = self.voxel_idx_map[new_coord[:, 0], new_coord[:, 1], new_coord[:, 2]]
            self.embedding_space_ftr.weight[assign] = new_ftrs.to(self.embedding_space_ftr.weight.dtype)
        return int(torch.nonzero(self.voxel_occupancy).shape[0])
