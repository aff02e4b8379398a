"""Parameter container with the reference's ObjectNeRF attribute names / state_dict keys
(reference models/nerf_model.py:18-95), so checkpoints and optimizers are interchangeable.

It holds weights only.  The arithmetic lives in the CUDA library: render_rays() packs these
parameters (engine.packed_for) and runs the fused kernels.
"""
from __future__ import annotations

import torch
from torch import nn


def _cfg(cfg, key, default=None):
    try:
        return cfg[key]
    except (KeyError, TypeError):
        return getattr(cfg, key, default)


def _act_linear(k, n, act):
    return nn.Sequential(nn.Linear(k, n), act)


class ObjectNeRF(nn.Module):
    def __init__(self, model_config):
        super().__init__()
        self.model_config = model_config
        self.use_voxel_embedding = bool(_cfg(model_config, "use_voxel_embedding", True))
        D, W = _cfg(model_config, "D"), _cfg(model_config, "W")
        skips = list(_cfg(model_config, "skips"))
        inst_D, inst_W = _cfg(model_config, "inst_D"), _cfg(model_config, "inst_W")
        inst_skips = list(_cfg(model_config, "inst_skips"))
        nfx, nfd = _cfg(model_config, "N_freq_xyz"), _cfg(model_config, "N_freq_dir")
        if (D, W, skips, inst_D, inst_W, inst_skips, nfx, nfd) != (8, 256, [4], 4, 128, [2], 10, 4):
            raise RuntimeError("object_nerf_b200 kernels are built for the default architecture only "
                               "(D=8, W=256, skips=[4], inst_D=4, inst_W=128, inst_skips=[2], PE 10/4)")
        self.D, self.W, self.skips = D, W, skips
        self.inst_D, self.inst_W, self.inst_skips = inst_D, inst_W, inst_skips
        self.N_freq_xyz, self.N_freq_dir = nfx, nfd
        vox_scene = vox_obj = 0
        if self.use_voxel_embedding:
            self.N_freq_voxel = _cfg(model_config, "N_freq_voxel")
            self.N_scn_voxel_size = _cfg(model_config, "N_scn_voxel_size", 0)
            n_obj_vox = _cfg(model_config, "N_obj_voxel_size", 0)
            if (self.N_freq_voxel, self.N_scn_voxel_size, n_obj_vox) != (6, 16, 8):
                raise RuntimeError("object_nerf_b200 kernels are built for 16+8 voxel channels with PE 6")
            vox_scene = self.N_scn_voxel_size * (1 + 2 * self.N_freq_voxel)
            vox_obj = n_obj_vox * (1 + 2 * self.N_freq_voxel)
        n_code = _cfg(model_config, "N_obj_code_length")
        if n_code != 64:
            raise RuntimeError("object_nerf_b200 kernels are built for 64-long object codes")
        self.in_channels_xyz = 3 * (1 + 2 * nfx) + vox_scene
        self.in_channels_dir = 3 * (1 + 2 * nfd)
        self.inst_channel_in = self.in_channels_xyz + n_code + vox_obj
        self.activation = nn.LeakyReLU(inplace=True)
        act = self.activation
        # creation order below fixes the state_dict key order and the RNG consumption of default init
        for i in range(D):
            k = self.in_channels_xyz if i == 0 else (W + self.in_channels_xyz if i in skips else W)
            setattr(self, f"xyz_encoding_{i+1}", _act_linear(k, W, act))
        self.xyz_encoding_final = nn.Linear(W, W)
        self.sigma = nn.Linear(W, 1)
        self.rgb = nn.Sequential(nn.Linear(W // 2, 3), nn.Sigmoid())
        self.dir_encoding = _act_linear(W + self.in_channels_dir, W // 2, act)
        for i in range(inst_D):
            k = self.inst_channel_in if i == 0 else (inst_W + self.inst_channel_in if i in inst_skips else inst_W)
            setattr(self, f"instance_encoding_{i+1}", _act_linear(k, inst_W, act))
        self.instance_encoding_final = nn.Sequential(nn.Linear(inst_W, inst_W))
        self.instance_sigma = nn.Linear(inst_W, 1)
        self.inst_dir_encoding = _act_linear(inst_W + self.in_channels_dir, inst_W // 2, act)
        self.inst_rgb = nn.Sequential(nn.Linear(inst_W // 2, 3), nn.Sigmoid())

    def _source(self, inputs, key):
        """(points, module) an embedding module of this package attached to inputs[key], or None."""
        t = inputs.get(key) if isinstance(inputs, dict) else None
        return getattr(t, "_onerf_src", None), t

    def _query(self, inputs, sigma_only, obj_code):
        """Reference :97-152 on inputs made by this package's embeddings: the positions (and directions) they were encoded
        from run through the fused encode + MLP kernel.  Returns the branch's (..., 4) field (rgb, raw sigma)."""
        from . import engine, field_query, rendering
        (src, emb) = self._source(inputs, "emb_xyz")
        if src is None:
            raise NotImplementedError(
                "ObjectNeRF is a weight container: the MLP runs fused with the encoding.  forward / forward_instance take "
                "inputs produced by this package's EmbeddingVoxel(xyz) / Embedding(3, 10)(xyz) and Embedding(3, 4)(dirs) "
                "(they carry their positions); arbitrary pre-embedded features are not supported.")
        pts, emb_mod = src
        grid_module = emb_mod if rendering._is_voxel(emb_mod) else None
        if (grid_module is not None) != self.use_voxel_embedding:
            raise ValueError("emb_xyz was encoded for the other model kind (voxel / plain PE) than this ObjectNeRF's")
        dirs = None
        if not sigma_only:
            dsrc, _ = self._source(inputs, "emb_dir")
            if inputs.get("emb_dir") is None:
                raise ValueError("sigma_only=False needs inputs['emb_dir'] (the reference would fail in torch.cat)")
            if dsrc is None or getattr(dsrc[1], "N_freqs", None) != 4:
                raise NotImplementedError("emb_dir must be produced by this package's Embedding(3, 4)(dirs)")
            dirs = dsrc[0]
            if dirs.shape[0] != pts.shape[0]:
                raise ValueError(f"emb_dir holds {dirs.shape[0]} directions for {pts.shape[0]} points")
        fi = obj_code is not None
        codes = None
        if fi:
            codes = obj_code.reshape(1, -1).expand(pts.shape[0], -1) if obj_code.dim() == 1 else obj_code
            if codes.shape != (pts.shape[0], 64):
                raise ValueError(f"obj_code must be (64,) or ({pts.shape[0]}, 64); got {tuple(obj_code.shape)}")
        if torch.is_grad_enabled() and (pts.requires_grad or (dirs is not None and dirs.requires_grad)):
            raise ValueError("positions and directions get no gradient here: detach them (the field backward stops at "
                             "the encoding, as render_rays' does)")
        table = field_query.table_of(grid_module)
        grad = rendering._needs_grad(self, codes, table)
        shape = emb.shape[:-1]
        n = pts.shape[0]
        if not grad and sigma_only and n > 0 and (not fi or bool((codes == codes[:1]).all())):
            # the density-only route of mesh extraction and pruning, one code for every point
            sigma = rendering.query_sigma(self, emb_mod, pts, obj_code=codes[0] if fi else None)
            return torch.cat([torch.zeros(sigma.shape[0], 3, device=sigma.device), sigma[:, None]], 1).reshape(*shape, 4)
        rays = torch.zeros(n, 8, dtype=torch.float32, device=pts.device)
        if dirs is not None:
            rays[:, 3:6] = dirs.detach()
        z = torch.zeros(n, 1, dtype=torch.float32, device=pts.device)
        xyz = pts.detach().float().reshape(n, 1, 3).contiguous()
        prec = engine.train_precision(None)
        if grad:
            reached = (field_query.OBJECT_SIGMA if sigma_only else field_query.OBJECT) if fi else (
                field_query.SCENE_SIGMA if sigma_only else field_query.SCENE)
            scene, obj = field_query.field_eval(self, grid_module, rays, z, xyz, codes, fi, prec, reached)
        else:
            packed = engine.packed_for(self, grid_module is not None)
            grid = engine.GridBuffers.from_module(grid_module) if grid_module is not None else None
            scene, obj = engine.field(rays, z, packed, grid, codes=codes.contiguous() if fi else None, want_scene=not fi,
                                      want_object=fi, precision=prec, xyz=xyz)
        return (obj if fi else scene).reshape(*shape, 4)

    def forward(self, inputs, sigma_only=False):
        """Reference :97-121: {"sigma" (..., 1)[, "rgb" (..., 3)]} of the scene branch at the points emb_xyz was encoded
        from (and, without sigma_only, the directions of emb_dir).  Differentiable under grad (field_query)."""
        f = self._query(inputs, sigma_only, None)
        return {"sigma": f[..., 3:]} if sigma_only else {"sigma": f[..., 3:], "rgb": f[..., :3]}

    def forward_instance(self, inputs, sigma_only=False):
        """Reference :123-152: {"inst_sigma"[, "inst_rgb"]} of the object branch, inputs["obj_code"] (B,64) one code per
        point (any rows) or (64,)."""
        f = self._query(inputs, sigma_only, inputs["obj_code"])
        return {"inst_sigma": f[..., 3:]} if sigma_only else {"inst_sigma": f[..., 3:], "inst_rgb": f[..., :3]}
