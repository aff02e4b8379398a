"""Training-step (gradient) case of the plain positional-encoding model (the reference's use_voxel_embedding: false):
GRAD_CASE of tests/cases.py on the plain model with its own seed.  Drives tools/make_golden.py (fixture
grad_train_step_plain), the CPU oracle test and the GPU tests of plain-PE training.  Inputs are regenerated from seeds
the same way cases.build_grad_case does for the voxel case."""
from __future__ import annotations

import numpy as np
import torch

from . import cases, synth

GRAD_CASE_PLAIN = dict(cases.GRAD_CASE, use_voxel=False, seed=310)


def build_grad_case_plain(n_rays=None):
    """n_rays=None: the fixture's case; other sizes reuse its seeds on more rays."""
    c = GRAD_CASE_PLAIN if n_rays is None else dict(GRAD_CASE_PLAIN, n_rays=n_rays)
    inp = cases.build_render_case(c)
    n = c["n_rays"]
    rng = np.random.default_rng(c["seed"] + 9)
    ids = rng.choice([4, 6], size=n)
    inp["instance_ids"] = torch.from_numpy(ids).view(n, 1)
    inp["code_table"] = synth.make_codes(c["seed"] + 2)
    inp["batch"] = {
        "rgbs": torch.from_numpy(rng.random((n, 3)).astype(np.float32)),
        "depths": torch.from_numpy(rng.uniform(0.3, 2.5, size=n).astype(np.float32)),
        "valid_mask": torch.from_numpy(rng.random(n) < 0.9),
        "instance_mask": torch.from_numpy(rng.random(n) < 0.5),
        "instance_mask_weight": torch.from_numpy(np.where(rng.random(n) < 0.5, 1.0, 0.05).astype(np.float32)),
    }
    return inp
