"""Cases of the field-query fixtures (tests/golden/field_query_*.npz): point queries of ObjectNeRF.forward /
forward_instance and single passes of inference_model, with fixed cotangents.  The same definitions drive
tools/make_field_query_golden.py (the reference's own modules, CPU), the CPU oracle tests and the GPU tests; inputs are
regenerated from seeds, the fixtures hold the reference's outputs and gradient summaries (cases.sample_indices)."""
from __future__ import annotations

import numpy as np
import torch

from . import cases, synth

POINT_CASES = {
    "point_voxel": dict(use_voxel=True, n=200, seed=300),
    "point_plain": dict(use_voxel=False, n=200, seed=301),
}

INFER_CASES = {
    # training-mode pass: injected sigma noise, occlusion mask with pass-through, both branches
    "infer_noise_mask": dict(forward_instance=True, noise_std=1.0, is_eval=False, frustum_bound_th=0.025,
                             pass_through=True, zero_last_delta=False, seed=310),
    # scene branch only, noise, last delta 0
    "infer_no_instance": dict(forward_instance=False, noise_std=1.0, is_eval=False, frustum_bound_th=0.0,
                              pass_through=False, zero_last_delta=True, seed=311),
    # eval mode: no noise, the occlusion mask is not applied
    "infer_eval": dict(forward_instance=True, noise_std=0.0, is_eval=True, frustum_bound_th=0.025,
                       pass_through=True, zero_last_delta=False, seed=312),
}
INFER_RAYS, INFER_SAMPLES = 24, 32
MAP_KEYS = ("opacity", "rgb", "depth", "rgb_instance", "depth_instance", "opacity_instance")


def build_point_case(c):
    """Points inside the grid, up to 10 % of its extent outside, and exactly on voxel corners; unit directions; codes
    from 7 distinct rows; cotangents of (sigma, rgb, inst_sigma, inst_rgb)."""
    s, n = c["seed"], c["n"]
    w = synth.make_weights(s, c["use_voxel"], 8.0, 1.0)
    grid = synth.make_grid(**cases.GRID_KW)
    gen = torch.Generator().manual_seed(s)
    vs = float(grid["voxel_size"])
    ext = grid["shape"].float() * vs
    pts = torch.rand(n, 3, generator=gen) * ext * 1.2 - 0.1 * ext - grid["offset"]
    k = n // 5
    pts[:k] = torch.randint(0, 20, (k, 3), generator=gen).float() * vs - grid["offset"]
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=1)
    codes = synth.make_codes(s + 1)[torch.randint(0, 7, (n,), generator=gen)]
    cot = {"sigma": torch.rand(n, 1, generator=gen) + 0.5, "rgb": torch.rand(n, 3, generator=gen) + 0.5,
           "inst_sigma": torch.rand(n, 1, generator=gen) + 0.5, "inst_rgb": torch.rand(n, 3, generator=gen) + 0.5}
    return dict(weights=w, grid=grid, pts=pts, dirs=dirs, codes=codes, cot=cot)


def build_infer_case(c):
    """One pass of 24 rays x 32 ascending depths; xyz = o + d z (fp32, the reference's broadcasted mul + add); per-ray
    codes; injected N(0,1) noise for both branches; cotangents of every map."""
    s, n, S = c["seed"], INFER_RAYS, INFER_SAMPLES
    w = synth.make_weights(s, True, 8.0, 1.0)
    grid = synth.make_grid(**cases.GRID_KW)
    rays = synth.random_rays(s + 1, n)
    rng = np.random.default_rng(s + 2)
    t = np.sort(rng.random((n, S)), axis=1).astype(np.float32)
    near, far = rays[:, 6:7], rays[:, 7:8]
    z = near + (far - near) * torch.from_numpy(t)
    xyz = rays[:, None, 0:3] + rays[:, None, 3:6] * z[:, :, None]
    codes = synth.make_codes(s + 3)[torch.from_numpy(rng.integers(0, 7, n))]
    ptm = torch.from_numpy(rng.random((n, 1)) < 0.5) if c["pass_through"] else None
    f = lambda *shape: torch.from_numpy(rng.standard_normal(shape).astype(np.float32))
    noise = {"noise_scene": f(n, S), "noise_obj": f(n, S)}
    cot = {k: torch.from_numpy(rng.random((n, 3) if k.startswith("rgb") else (n,)).astype(np.float32)) + 0.5
           for k in MAP_KEYS}
    return dict(weights=w, grid=grid, rays=rays, z=z, xyz=xyz, codes=codes, pass_through_mask=ptm, noise=noise, cot=cot)


def grad_summary(named):
    """{name|norm, name|sum, name|samples} of every gradient in `named` ((name, grad) pairs; None skipped)."""
    fix = {}
    for name, g in named:
        if g is None:
            continue
        g = g.reshape(-1)
        fix[name + "|norm"] = g.norm()
        fix[name + "|sum"] = g.sum()
        fix[name + "|samples"] = g[cases.sample_indices(name, g.numel())]
    return fix
