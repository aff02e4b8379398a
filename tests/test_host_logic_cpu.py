"""CPU tests of the host-side logic: drop-in aliasing and signatures, weight-layout bookkeeping, box folding,
and the N > 1 sharding / gather path on a world_size-2 gloo group."""
import inspect
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import cases

def test_dropin_aliases_and_surface():
    from object_nerf_b200 import dropin
    saved = {k: sys.modules.get(k) for k in list(dropin.ALIASES) + ["models", "render_tools"]}
    try:
        dropin.install()
        from models.rendering import render_rays, sample_pdf, inference_model  # noqa: F401
        from models.nerf_model import ObjectNeRF  # noqa: F401
        from models.embedding_helper import Embedding, EmbeddingVoxel  # noqa: F401
        from models.code_library import CodeLibrary  # noqa: F401
        from render_tools.multi_rendering import render_rays_multi  # noqa: F401
        from models.losses import get_loss, TotalLoss  # noqa: F401
        import object_nerf_b200.rendering as R
        assert render_rays is R.render_rays
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


# the reference's signatures (models/rendering.py:233-250, :64-83, :11-17; render_tools/multi_rendering.py:160-175)
REF_SIGS = {
    "render_rays": ["models", "embeddings", "rays", "N_samples", "use_disp", "perturb", "noise_std", "N_importance",
                    "chunk", "white_back", "forward_instance", "embedding_instance", "frustum_bound_th",
                    "pass_through_mask", "rays_in_bbox"],
    "inference_model": ["results", "model", "embeddings", "typ", "xyz", "rays_d", "z_vals", "chunk", "noise_std",
                        "white_back", "is_eval", "use_zero_as_last_delta", "forward_instance", "embedding_instance",
                        "frustum_bound_th", "pass_through_mask", "rays_in_bbox"],
    "sample_pdf": ["bins", "weights", "N_importance", "det", "eps"],
    "render_rays_multi": ["models", "embeddings", "code_library", "rays_list", "obj_instance_ids", "N_samples",
                          "use_disp", "perturb", "noise_std", "N_importance", "chunk", "white_back",
                          "background_skip_bbox"],
}
# the reference's literal default values of those parameters (same source lines)
REF_DEFAULTS = {
    "render_rays": {"N_samples": 64, "use_disp": False, "perturb": 0, "noise_std": 1, "N_importance": 0,
                    "white_back": False, "forward_instance": True, "embedding_instance": None, "frustum_bound_th": 0,
                    "pass_through_mask": None, "rays_in_bbox": False},
    "inference_model": {"is_eval": False, "use_zero_as_last_delta": False, "forward_instance": True,
                        "embedding_instance": None, "frustum_bound_th": 0, "pass_through_mask": None,
                        "rays_in_bbox": False},
    "sample_pdf": {"det": False, "eps": 1e-05},
    "render_rays_multi": {"N_samples": 64, "use_disp": False, "perturb": 0, "noise_std": 0, "N_importance": 0,
                          "white_back": False, "background_skip_bbox": None},
}


def test_signatures_match_reference():
    from object_nerf_b200 import multi_rendering, rendering
    ours = {"render_rays": rendering.render_rays, "inference_model": rendering.inference_model,
            "sample_pdf": rendering.sample_pdf, "render_rays_multi": multi_rendering.render_rays_multi}
    for name, want in REF_SIGS.items():
        params = list(inspect.signature(ours[name]).parameters)
        assert params[: len(want)] == want, (name, params)
    for name, defaults in REF_DEFAULTS.items():
        params = inspect.signature(ours[name]).parameters
        for arg, want in defaults.items():
            assert params[arg].default == want, (name, arg, params[arg].default, want)


def test_state_dict_keys_match_reference_names():
    from object_nerf_b200 import CodeLibrary, ObjectNeRF
    from tests import helpers
    m = ObjectNeRF(helpers.model_config(True))
    keys = set(m.state_dict())
    want = {f"{n}.{p}" for n in helpers.REF_NAMES.values() for p in ("weight", "bias")}
    assert keys == want
    assert sum(p.numel() for p in m.parameters()) == 891208           # SURVEY.md appendix B
    assert sum(p.numel() for p in ObjectNeRF(helpers.model_config(False)).parameters()) == 704840
    assert list(CodeLibrary(helpers.model_config()).state_dict()) == ["embedding_instance.weight"]


def test_unsupported_architecture_is_a_hard_error():
    from object_nerf_b200 import ObjectNeRF
    from tests import helpers
    cfg = helpers.model_config(True)
    cfg["W"] = 128
    with pytest.raises(RuntimeError):
        ObjectNeRF(cfg)


def test_box_folding_matches_oracle_convention():
    from object_nerf_b200.multi_rendering import boxes_to_tensor
    inp = cases.build_multi_case(cases.MULTI_CASES["edit_dup"])

    class Box:
        pass
    boxes = {}
    for k, b in enumerate(inp["boxes"]):
        h = Box()
        h.scale_factor, h.pose_avg, h.axis_align_mat, h.bbox_bounds = (b["scale_factor"], b["pose_avg"],
                                                                       b["axis_align_mat"], b["bbox_bounds"])
        boxes[k] = h
    t = boxes_to_tensor(boxes, "cpu")
    assert t.shape == (2, 18)
    for row, b in zip(t, inp["boxes"]):
        A, tt, lo, hi = cases.box_affine(b)
        assert torch.allclose(row[:9].view(3, 3), A) and torch.allclose(row[9:12], tt)
        assert torch.allclose(row[12:15], lo) and torch.allclose(row[15:18], hi)


def test_embedding_voxel_grid_builder_matches_reference_buffers():
    """Cold path: EmbeddingVoxel.set_pointclouds builds the same buffers as the reference's (fixture written by
    tools/make_golden.py from the reference's constructor on the same synthetic cloud)."""
    path = os.path.join(os.path.dirname(__file__), "golden", "gridbuild.npz")
    if not os.path.exists(path):
        pytest.skip("fixture not generated")
    from object_nerf_b200 import EmbeddingVoxel
    g = np.load(path)
    conf = dict(pcd_path="synthetic", scene_center=[2.0, 2.0, 0.0], scale_factor=2.0, voxel_size=0.1, neighbor_marks=3)
    pts = np.random.default_rng(0).uniform([0, 0, -1], [4, 4, 1], size=(20000, 3))
    emb = EmbeddingVoxel(24, 6, 50000, conf, points=pts)
    assert emb.voxel_shape.tolist() == g["voxel_shape"].tolist()
    assert torch.equal(emb.voxel_idx_map, torch.from_numpy(g["voxel_idx_map"]))
    assert torch.allclose(emb.voxel_offset, torch.from_numpy(g["voxel_offset"]))
    assert torch.allclose(emb.voxel_size, torch.from_numpy(g["voxel_size"]))


def _worker(rank, world, port, n):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from object_nerf_b200 import parallel
    rays = torch.arange(n * 8, dtype=torch.float32).view(n, 8)
    per_ray = {"codes": torch.arange(n * 4, dtype=torch.float32).view(n, 4)}

    def fake_render(r, pr):   # stands in for render_rays: any per-ray function
        return {"rgb": r[:, :3] * 2 + pr["codes"][:, :3], "depth": r[:, 6] + 1}

    out = parallel.render_sharded(fake_render, rays, per_ray, ["rgb", "depth"])
    full = fake_render(rays, per_ray)
    assert torch.equal(out["rgb"], full["rgb"]) and torch.equal(out["depth"], full["depth"])
    dist.destroy_process_group()


@pytest.mark.parametrize("n", [10, 7])
def test_ray_sharded_gather_world2_gloo(n):
    from object_nerf_b200 import parallel
    assert [parallel.shard_bounds(7, 2, r) for r in range(2)] == [(0, 4), (4, 7)]
    port = 29500 + os.getpid() % 1000 + n
    mp.spawn(_worker, args=(2, port, n), nprocs=2, join=True)


# ------------------------------------------------------------------------------------------------
# voxel grid maintenance (SURVEY section 8f row 4): the grid surgery of our EmbeddingVoxel against the reference's,
# with the two device queries (raw trilinear features, density) supplied by the CPU oracle
# ------------------------------------------------------------------------------------------------
def _maint_embedding():
    from object_nerf_b200.embedding_helper import EmbeddingVoxel
    from tests import cases
    inp, c = cases.build_maint_case(), cases.MAINT_CASE
    emb = EmbeddingVoxel(24, 6, c["max_voxels"], c["extra"], points=inp["points"])
    with torch.no_grad():
        emb.embedding_space_ftr.weight.copy_(inp["table"])
    return emb, inp


def _oracle_grid(emb):
    from oracle import onerf_oracle as O
    return O.VoxelGrid(emb.voxel_offset, emb.voxel_size, emb.voxel_shape.tolist(), emb.voxel_idx_map,
                       emb.embedding_space_ftr.weight.detach().clone())


def _assert_grid_state(emb, gold, prefix):
    n = int(torch.nonzero(emb.voxel_occupancy).shape[0])
    assert torch.equal(emb.voxel_size, gold[prefix + "voxel_size"])
    assert torch.equal(emb.voxel_shape, gold[prefix + "voxel_shape"])
    assert torch.equal(emb.voxel_occupancy, gold[prefix + "voxel_occupancy"].bool())
    assert torch.equal(emb.voxel_idx_map, gold[prefix + "voxel_idx_map"])
    assert torch.equal(emb.embedding_space_ftr.weight.detach()[:n], gold[prefix + "table_rows"])


def test_voxel_subdivision_matches_reference_golden(golden):
    from oracle import onerf_oracle as O
    emb, _ = _maint_embedding()
    gold = golden("maint_subdivision")
    _assert_grid_state(emb, gold, "before|")                       # the constructor agrees with the reference first
    old = _oracle_grid(emb)
    n_after = emb.voxel_subdivision(_features_fn=lambda pts: O.voxel_features(pts, old))
    assert n_after == 8 * int(gold["before|table_rows"].shape[0])
    _assert_grid_state(emb, gold, "subdiv|")


def test_self_pruning_matches_reference_golden(golden):
    from oracle import onerf_oracle as O
    from tests import cases
    emb, inp = _maint_embedding()
    gold = golden("maint_pruning")
    grid = _oracle_grid(emb)
    n_occu = int(gold["n_before"])
    sigma = lambda pts: O.field_eval(inp["weights"], grid, pts, torch.zeros_like(pts), None, want_object=False)["sigma"]
    n_pruned = emb.self_pruning_empty_voxels(None, max_alpha_th=cases.MAINT_CASE["max_alpha_th"],
                                             _rand=cases.maint_rand((n_occu + 31) // 32), _sigma_fn=sigma)
    assert 0 < n_pruned < n_occu                                   # the case prunes some voxels and keeps others
    assert torch.equal(emb.voxel_occupancy, gold["pruned|voxel_occupancy"].bool())
    assert torch.equal(emb.voxel_idx_map, gold["pruned|voxel_idx_map"])
