"""Training the plain positional-encoding model (the reference's use_voxel_embedding: false), CPU side: the oracle's
backward against the reference's own (fixture grad_train_step_plain, written by tools/make_golden.py), and the sizes of
the one-X-atom training workspace."""
import os

import pytest
import torch

from oracle import onerf_oracle as O
from tests import cases, grad_plain, helpers


def test_plain_training_step_gradients_match_reference(golden):
    """Oracle autograd (torch CPU) vs the reference's backward through render_rays + TotalLoss on the plain model."""
    g = golden("grad_train_step_plain")
    assert not any(k.startswith("voxel|") for k in g)
    c = grad_plain.GRAD_CASE_PLAIN
    inp = grad_plain.build_grad_case_plain()
    assert inp["grid"] is None
    leaves = {}

    def leaf(name, t):
        t = t.clone().requires_grad_(True)
        leaves[name] = t
        return t

    weights = {typ: {k: (leaf(f"{typ}.{helpers.REF_NAMES[k]}.weight", W), leaf(f"{typ}.{helpers.REF_NAMES[k]}.bias", b))
                     for k, (W, b) in w.items()} for typ, w in inp["weights"].items()}
    code_table = leaf("codes", inp["code_table"])
    codes = code_table[inp["instance_ids"].view(-1)]
    out = O.render_rays(weights, None, inp["rays"], codes, n_samples=c["n_samples"], perturb=c["perturb"],
                        noise_std=c["noise_std"], n_importance=c["n_importance"], frustum_bound_th=c["frustum_bound_th"],
                        pass_through_mask=inp["pass_through_mask"], is_eval=False, rand=inp["rand"])
    loss = cases.total_loss(out, inp["batch"])
    assert abs(loss.item() - g["loss"].item()) <= 1e-5 * abs(g["loss"].item())
    loss.backward()
    assert {k.split("|")[0] for k in g if k != "loss"} == set(leaves)
    assert len(leaves) == 81      # 2 x 40 nn.Linear tensors + the code table
    for name, t in leaves.items():
        gr = t.grad.reshape(-1)
        ref_norm = g[name + "|norm"].item()
        assert abs(gr.norm().item() - ref_norm) <= 1e-4 * max(ref_norm, 1e-6), name
        idx = cases.sample_indices(name, gr.numel())
        assert torch.allclose(gr[idx], g[name + "|samples"], rtol=1e-3, atol=1e-5 * max(ref_norm, 1e-6)), name


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


@pytest.mark.parametrize("n_rays, n_samples, n_importance", [(1, 2, 0), (40, 64, 64), (2048, 64, 64), (333, 40, 24)])
def test_plain_training_workspace_is_the_one_x_atom_layout(lib, n_rays, n_samples, n_importance):
    """onerf_field_train_bytes / onerf_train_workspace_bytes for use_voxel = 0 match a TrainLayout with one X atom
    (tests/helpers.py mirrors layout.h), and are smaller than the voxel model's."""
    for B in (n_rays * n_samples, n_rays * (n_samples + n_importance)):
        plain, voxel = lib.onerf_field_train_bytes(0, B), lib.onerf_field_train_bytes(1, B)
        assert plain == helpers.train_layout(False, B)["total"]
        assert voxel == helpers.train_layout(True, B)["total"]
        assert voxel - plain == 5 * helpers.train_layout(False, B)["n_tiles"] * helpers.ATOM_BYTES
    # the training workspace (train_ws.h): both passes' field workspaces, then buffers that do not depend on the model
    # except the kernel-layout gradient buffer
    up = lambda x: (x + 1023) // 1024 * 1024
    Bc, Bf = n_rays * n_samples, n_rays * (n_samples + n_importance)

    def ws(use_voxel):
        return (up(lib.onerf_field_train_bytes(use_voxel, Bc)) + (up(lib.onerf_field_train_bytes(use_voxel, Bf)) if n_importance else 0)
                + 2 * up(Bc * 16) + 6 * up(Bf * 16) + up(n_rays * 448 * 4) + up(n_rays * 27 * 4)
                + up(lib.onerf_grad_buffer_floats(use_voxel) * 4))

    plain, voxel = lib.onerf_train_workspace_bytes(0, n_rays, n_samples, n_importance), \
        lib.onerf_train_workspace_bytes(1, n_rays, n_samples, n_importance)
    assert plain == ws(0) and voxel == ws(1)
    assert plain < voxel
