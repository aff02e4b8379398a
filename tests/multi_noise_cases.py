"""Cases of render_rays_multi with sigma noise, perturbed importance sampling and 10-column (box-clipped) ray sets.  The
same dicts drive tools/make_golden.py (the reference's own render_rays_multi with injected draws; fixtures
tests/golden/multi_<name>.npz), the CPU oracle test and the GPU tests.  Kept apart from cases.MULTI_CASES, which
parametrizes the noise-free tests.

clip maps a set index to how its (near_box, far_box) columns are made from the set's per-ray near / far:
  inside    a random sub-interval of [near, far] (misses, near = far = 0, get the empty interval (0, 0))
  swallow   (near - 0.1, far + 0.1): every fine sample of the ray becomes far + 0.1, a missed ray's zeros included
  empty     near_box >= far_box (equal for half the rays): nothing is clipped
  far_zero  far_box = 0, near_box in {-3, -0.5}; 40 % of the rays get negative depths (near, far) -> (-far, -near), so
            their last fine depth becomes 0 and the fine pass mutes them
same_rays: set j takes set i's origins and directions (near / far stay its own) and set i's clip, so that two sets of
one object tie at far_box with identical fields there.
"""
from __future__ import annotations

import numpy as np
import torch

from . import cases

_B = dict(n_rays=32, n_samples=32, n_importance=32, white_back=False, boxes=False, perturb=0.0, noise_std=0.0, clip={},
          same_rays={})

NOISE_CLIP_CASES = {
    # noise in both passes, removed-object boxes on the scene set
    "noise_both": dict(_B, obj_ids=[0, 4], boxes=True, noise_std=1.0, seed=230),
    # perturb > 0 with injected u, white background, K != S
    "perturb_u": dict(_B, obj_ids=[0, 6], n_importance=48, white_back=True, perturb=1.0, seed=231),
    # 8- and 10-column sets mixed, noise and perturb together
    "mixed_clip": dict(_B, obj_ids=[0, 4, 6], perturb=1.0, noise_std=0.5, clip={1: "inside"}, seed=232),
    "clip_swallow": dict(_B, obj_ids=[0, 4], noise_std=1.0, clip={1: "swallow"}, seed=233),
    "clip_empty": dict(_B, obj_ids=[0, 4, 6], clip={1: "empty", 2: "inside"}, seed=234),
    "clip_far_zero": dict(_B, obj_ids=[0, 4], perturb=1.0, noise_std=1.0, clip={1: "far_zero"}, seed=235),
    # one object in two sets with the same rays and clip: fine samples tie at far_box inside a set and across the sets
    "dup_tied": dict(_B, obj_ids=[0, 4, 4], boxes=True, perturb=1.0, noise_std=1.0, clip={1: "inside", 2: "inside"},
                     same_rays={2: 1}, seed=236),
}


def _clip_columns(kind, rays, rng):
    n = rays.shape[0]
    near, far = rays[:, 6].clone(), rays[:, 7].clone()
    if kind == "inside":
        a = torch.from_numpy(rng.uniform(0.05, 0.5, n).astype(np.float32))
        b = torch.from_numpy(rng.uniform(0.55, 0.95, n).astype(np.float32))
        return near + a * (far - near), near + b * (far - near), rays
    if kind == "swallow":
        return near - 0.1, far + 0.1, rays
    if kind == "empty":
        lo = near + 0.5 * (far - near)
        hi = torch.where(torch.arange(n) % 2 == 0, lo, lo - 0.2)
        return lo, hi, rays
    if kind == "far_zero":
        neg = torch.from_numpy(rng.random(n) < 0.4)
        rays = rays.clone()
        rays[neg, 6], rays[neg, 7] = -far[neg], -near[neg]
        nb = torch.from_numpy(np.where(rng.random(n) < 0.5, -3.0, -0.5).astype(np.float32))
        return nb, torch.zeros(n), rays
    raise ValueError(kind)


def build_noise_clip_case(c):
    """cases.build_multi_case's scene, models and sets, then the clip columns, the shared rays and the injected draws:
    u (a list, one (N, K) per set), noise_coarse (N, n_sets * S) and noise_fine (N, n_sets * (S + K)), drawn whatever
    perturb and noise_std are (the reference draws its randn_like noise even at noise_std = 0)."""
    inp = cases.build_multi_case(c)
    rng = np.random.default_rng(c["seed"] + 50)
    rays_list = inp["rays_list"]
    for j, i in c["same_rays"].items():
        rays_list[j] = rays_list[j].clone()
        rays_list[j][:, 0:6] = rays_list[i][:, 0:6]
    clips = {}
    for i, kind in sorted(c["clip"].items()):
        if c["same_rays"].get(i) in clips:
            clips[i] = clips[c["same_rays"][i]]
            continue
        nb, fb, rays_list[i] = _clip_columns(kind, rays_list[i], rng)
        clips[i] = torch.stack([nb, fb], 1).float()
    inp["rays_list"] = [torch.cat([r, clips[i]], 1).contiguous() if i in clips else r for i, r in enumerate(rays_list)]
    n, s, k, no = c["n_rays"], c["n_samples"], c["n_importance"], len(c["obj_ids"])
    g = torch.Generator().manual_seed(c["seed"] + 60)
    inp["rand"] = {"u": [torch.rand(n, k, generator=g) for _ in range(no)],
                   "noise_coarse": torch.randn(n, no * s, generator=g),
                   "noise_fine": torch.randn(n, no * (s + k), generator=g)}
    return inp
