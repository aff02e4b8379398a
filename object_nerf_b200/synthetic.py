"""Deterministic synthetic scenes (weights, voxel grid, codes, rays) and the module containers built from them, shared by
bench.py, __graft_entry__.smoke(), the tests and the golden-fixture generator (there are no datasets or checkpoints
offline: SURVEY.md §8d).

Everything is derived from numpy PCG64 seeds (stable across numpy versions and machines), so the
build container (where tools/make_golden.py runs the real reference) and the GPU box (which has no
/root/reference) regenerate bit-identical inputs; fixtures under tests/golden/ hold only outputs.

Sizes follow config/default_conf.yml:7-36 of the reference (D=8, W=256, skip 4; inst_D=4,
inst_W=128, skip 2; PE 10/4/6; 16+8 voxel channels; 64-long object codes).
"""
from __future__ import annotations

import math

import numpy as np
import torch

N_CODE = 64
N_VOX_CH = 24
N_OBJ_CH = 8


def layer_dims(use_voxel: bool = True):
    """(name, fan_in, fan_out) for every Linear of one ObjectNeRF; Appendix B of SURVEY.md."""
    xyz_in = 63 + (208 if use_voxel else 0)
    obj_in = xyz_in + (104 if use_voxel else 0) + N_CODE
    dims = []
    for i in range(8):
        k = xyz_in if i == 0 else (256 + xyz_in if i == 4 else 256)
        dims.append((f"scene.l{i}", k, 256))
    dims += [("scene.sigma", 256, 1), ("scene.final", 256, 256), ("scene.dir", 256 + 27, 128),
             ("scene.rgb", 128, 3)]
    for i in range(4):
        k = obj_in if i == 0 else (128 + obj_in if i == 2 else 128)
        dims.append((f"obj.l{i}", k, 128))
    dims += [("obj.sigma", 128, 1), ("obj.final", 128, 128), ("obj.dir", 128 + 27, 64), ("obj.rgb", 64, 3)]
    return dims


def make_weights(seed: int, use_voxel: bool = True, sigma_gain: float = 1.0, sigma_bias: float = 0.0,
                 rgb_gain: float = 1.0):
    """nn.Linear-style init U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for W and b, in a fixed layer order.
    sigma_gain / sigma_bias sharpen the density heads so that weights / PDFs are not degenerate
    (random init gives sigma ~ 0, i.e. a transparent scene); rgb_gain scales the colour heads (random init gives a flat
    grey: sigmoid of ~0 everywhere, on which any two renderers agree trivially)."""
    rng = np.random.default_rng(seed)
    w = {}
    for name, k, n in layer_dims(use_voxel):
        bound = 1.0 / math.sqrt(k)
        W = rng.uniform(-bound, bound, size=(n, k)).astype(np.float32)
        b = rng.uniform(-bound, bound, size=(n,)).astype(np.float32)
        if name.endswith(".sigma"):
            W = (W * sigma_gain).astype(np.float32)
            b = (b * sigma_gain + sigma_bias).astype(np.float32)
        if name.endswith(".rgb") and rgb_gain != 1.0:
            W = (W * rgb_gain).astype(np.float32)
            b = (b * rgb_gain).astype(np.float32)
        w[name] = (torch.from_numpy(W), torch.from_numpy(b))
    return w


def make_grid(seed: int, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05, n_rows=None,
              feat_scale=1.0):
    """A sparse voxel grid in the layout the reference's EmbeddingVoxel keeps
    (models/embedding_helper.py:107-133,189-200): idx_map -1 = empty, rows numbered in raster order of
    the occupied cells, table rows ~ N(0,1) like nn.Embedding init.  Returns a dict of tensors."""
    rng = np.random.default_rng(seed)
    occ = rng.random(shape) < occupancy
    n_occ = int(occ.sum())
    idx = -np.ones(shape, dtype=np.int64)
    idx[occ] = np.arange(n_occ)
    n_rows = n_rows or (n_occ + 1)
    table = (rng.standard_normal((n_rows, N_VOX_CH)) * feat_scale).astype(np.float32)
    ext = np.array(shape, dtype=np.float64) * voxel_size
    # the volume is centred on the origin: offset = -min corner
    offset = (0.5 * ext - voxel_size).astype(np.float32)
    return {
        "offset": torch.from_numpy(offset),
        "voxel_size": torch.tensor(voxel_size, dtype=torch.float32),
        "shape": torch.tensor(shape, dtype=torch.int64),
        "idx_map": torch.from_numpy(idx),
        "table": torch.from_numpy(table),
    }


def make_codes(seed: int, n_objs: int = 64):
    rng = np.random.default_rng(seed)
    return torch.from_numpy(rng.standard_normal((n_objs, N_CODE)).astype(np.float32))


def pinhole_rays(h: int, w: int, near: float = 0.15, far: float = 3.0, cam_pos=(-1.6, 0.1, 0.15),
                 look_at=(0.0, 0.0, 0.0), fov_x_deg: float = 60.0, pixel_index=None):
    """(N,8) rays [o, d(unit), near, far] of a pinhole camera (datasets/ray_utils.py:5-51 of the
    reference: no +0.5 pixel offset, unit-norm directions).  pixel_index: optional flat pixel ids."""
    focal = 0.5 * w / math.tan(0.5 * math.radians(fov_x_deg))
    ids = np.arange(h * w) if pixel_index is None else np.asarray(pixel_index)
    i = (ids % w).astype(np.float64)
    j = (ids // w).astype(np.float64)
    dirs = np.stack([(i - w / 2) / focal, -(j - h / 2) / focal, -np.ones_like(i)], -1)
    cam = np.asarray(cam_pos, dtype=np.float64)
    fwd = np.asarray(look_at, dtype=np.float64) - cam
    fwd /= np.linalg.norm(fwd)
    up = np.array([0.0, 0.0, 1.0])
    right = np.cross(fwd, up)
    right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    R = np.stack([right, up, -fwd], 1)  # camera axes (x right, y up, z back) in world
    d = dirs @ R.T
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    o = np.broadcast_to(cam, d.shape)
    nf = np.broadcast_to(np.array([near, far]), (d.shape[0], 2))
    return torch.from_numpy(np.concatenate([o, d, nf], -1).astype(np.float32))


def random_rays(seed: int, n: int, h: int = 480, w: int = 640, **kw):
    rng = np.random.default_rng(seed)
    return pinhole_rays(h, w, pixel_index=rng.integers(0, h * w, size=n), **kw)


def random_buffers(seed: int, n: int, s_coarse: int, n_importance: int):
    """The random draws the reference makes inside render_rays, pre-drawn so both sides see the same
    numbers: jitter U[0,1) (rendering.py:276), u U[0,1) (:40), gaussian sigma noise (:156,187)."""
    rng = np.random.default_rng(seed)
    s_fine = s_coarse + n_importance
    f = lambda a: torch.from_numpy(a.astype(np.float32))
    return {
        "jitter": f(rng.random((n, s_coarse))),
        "u": f(rng.random((n, n_importance))),
        "noise_scene_coarse": f(rng.standard_normal((n, s_coarse))),
        "noise_obj_coarse": f(rng.standard_normal((n, s_coarse))),
        "noise_scene_fine": f(rng.standard_normal((n, s_fine))),
        "noise_obj_fine": f(rng.standard_normal((n, s_fine))),
    }


# ------------------------------------------------------------------------------------------------
# parameter containers built from the synthetic scenes
# ------------------------------------------------------------------------------------------------
REF_NAMES = {  # weight-dict layout -> reference attribute names (models/nerf_model.py:41-58,77-95)
    **{f"scene.l{i}": f"xyz_encoding_{i+1}.0" for i in range(8)},
    "scene.final": "xyz_encoding_final", "scene.sigma": "sigma", "scene.dir": "dir_encoding.0",
    "scene.rgb": "rgb.0",
    **{f"obj.l{i}": f"instance_encoding_{i+1}.0" for i in range(4)},
    "obj.final": "instance_encoding_final.0", "obj.sigma": "instance_sigma",
    "obj.dir": "inst_dir_encoding.0", "obj.rgb": "inst_rgb.0",
}


class Cfg(dict):
    __getattr__ = dict.__getitem__


def model_config(use_voxel=True):
    """config/default_conf.yml:7-36 of the reference."""
    return Cfg(use_voxel_embedding=use_voxel, N_freq_xyz=10, N_freq_dir=4, N_freq_voxel=6, D=8, W=256,
               skips=[4], N_scn_voxel_size=16, inst_D=4, inst_W=128, inst_skips=[2], N_obj_voxel_size=8,
               N_max_objs=64, N_obj_code_length=64, N_max_voxels=800000)


def make_model(w, use_voxel, device):
    from .nerf_model import ObjectNeRF
    m = ObjectNeRF(model_config(use_voxel))
    sd = {}
    for k, (W, b) in w.items():
        sd[REF_NAMES[k] + ".weight"] = W
        sd[REF_NAMES[k] + ".bias"] = b
    m.load_state_dict(sd, strict=True)
    return m.to(device).eval()


class GridModule(torch.nn.Module):
    """Stands in for EmbeddingVoxel with an injected grid: the same buffers / parameter the kernels read."""

    def __init__(self, g):
        super().__init__()
        self.embedding_space_ftr = torch.nn.Embedding.from_pretrained(g["table"].clone(), freeze=False)
        self.register_buffer("voxel_idx_map", g["idx_map"].clone())
        self.register_buffer("voxel_offset", g["offset"].clone())
        self.register_buffer("voxel_size", g["voxel_size"].clone())
        self.register_buffer("voxel_shape", g["shape"].clone())


def make_embedding(g):
    """An EmbeddingVoxel holding grid `g` (make_grid) with occupancy = idx_map >= 0 (the state the reference's grid has
    after construction, here without a point cloud), so that grid maintenance can run on it."""
    from .embedding_helper import EmbeddingVoxel
    emb = EmbeddingVoxel.__new__(EmbeddingVoxel)
    torch.nn.Module.__init__(emb)
    emb.channels, emb.instance_ftr_C = N_VOX_CH, 8
    emb.embedding_space_ftr = torch.nn.Embedding.from_pretrained(g["table"].clone(), freeze=False)
    emb.register_buffer("voxel_size", g["voxel_size"].clone())
    emb.register_buffer("voxel_offset", g["offset"].clone())
    emb.register_buffer("voxel_shape", g["shape"].clone())
    emb.register_buffer("voxel_count", torch.scalar_tensor(int(g["idx_map"].numel())))
    emb.register_buffer("voxel_occupancy", g["idx_map"] >= 0)
    emb.register_buffer("voxel_idx_map", g["idx_map"].clone())
    return emb


def make_code_library(table):
    from .code_library import CodeLibrary
    lib = CodeLibrary(model_config())
    with torch.no_grad():
        lib.embedding_instance.weight.copy_(table)
    return lib
