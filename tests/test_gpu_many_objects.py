"""render_rays_multi with many ray sets (pytest -m gpu): the rank-merge joint sort for n_obj * samples > 4096 and the box
culling of object ray sets in the one-call entry.

- beyond the old 4096-sample cap: against the CPU oracle, with the tolerances of the existing multi-path parity tests;
- the merge path's order is exactly torch.sort(stable=True) over the concatenation, and for T <= 4096 it is bit-identical
  to the bitonic kernel;
- culling: the one-call route (culled) is bit-identical to the staged route (every ray evaluated), also when no ray, every
  ray or one ray hits a box; the culled call captures in a CUDA graph and repeats bit for bit.
"""
import numpy as np
import pytest
import torch

from oracle import onerf_oracle as O
from tests import cases, helpers

pytestmark = pytest.mark.gpu
DEV = "cuda"
PRECISIONS = ["fp32", "bf16"]


def _case(n_rays, obj_ids, n_samples, n_importance, seed, hits=None):
    """cases.build_multi_case with optional per-set hit patterns: hits[k] is None (the builder's 30 % misses), "none",
    "all" or "one" for object set k."""
    c = dict(n_rays=n_rays, n_samples=n_samples, n_importance=n_importance, obj_ids=obj_ids, white_back=False, boxes=True,
             seed=seed)
    inp = cases.build_multi_case(c)
    rng = np.random.default_rng(seed + 77)
    for k, h in enumerate(hits or []):
        if h is None or obj_ids[k] == 0:
            continue
        r = inp["rays_list"][k]
        near = torch.from_numpy(rng.uniform(0.4, 1.2, size=n_rays).astype(np.float32))
        far = near + torch.from_numpy(rng.uniform(0.2, 0.9, size=n_rays).astype(np.float32))
        hit = torch.zeros(n_rays, dtype=torch.bool)
        if h == "all":
            hit[:] = True
        elif h == "one":
            hit[n_rays // 2] = True
        near[~hit], far[~hit] = 0, 0
        r[:, 6], r[:, 7] = near, far
    return c, inp


def _boxes(inp):
    class Box:  # the attributes of BBoxRayHelper that the box mask reads
        pass
    out = {}
    for k, b in enumerate(inp["boxes"]):
        h = Box()
        h.scale_factor, h.pose_avg = b["scale_factor"], b["pose_avg"]
        h.axis_align_mat, h.bbox_bounds = b["axis_align_mat"], b["bbox_bounds"]
        out[k] = h
    return out


def _setup(inp):
    from object_nerf_b200 import Embedding
    models = {"coarse": helpers.make_model(inp["weights"]["coarse"], True, DEV),
              "fine": helpers.make_model(inp["weights"]["fine"], True, DEV)}
    emb = {"xyz": helpers.GridModule(inp["grid"]).to(DEV), "dir": Embedding(3, 4)}
    return models, emb, helpers.CodeLib(inp["code_table"]).to(DEV)


def _render(c, inp, precision, staged=False, setup=None):
    from object_nerf_b200.multi_rendering import render_rays_multi
    models, emb, lib = setup or _setup(inp)
    with torch.no_grad():
        return render_rays_multi(models, emb, lib, [r.to(DEV) for r in inp["rays_list"]], c["obj_ids"],
                                 N_samples=c["n_samples"], N_importance=c["n_importance"], white_back=c["white_back"],
                                 background_skip_bbox=_boxes(inp), precision=precision, _staged=staged)


def _equal(a, b):
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


# 1 scene set + 24 object sets (ids 4 / 6 / 5 duplicated) at 64 + 128: T = 4 800 in the fine pass
MANY_IDS = [0] + [4, 6, 5] * 8


@pytest.mark.parametrize("precision", PRECISIONS)
def test_beyond_the_old_cap_matches_oracle(precision):
    c, inp = _case(37, MANY_IDS, 64, 128, seed=610)
    assert len(MANY_IDS) * (64 + 128) > 4096
    out = _render(c, inp, precision)
    with torch.no_grad():
        want = O.render_rays_multi(inp["weights"], O.VoxelGrid(inp["grid"]["offset"], inp["grid"]["voxel_size"],
                                                               inp["grid"]["shape"].tolist(), inp["grid"]["idx_map"],
                                                               inp["grid"]["table"]),
                                   inp["code_table"], inp["rays_list"], c["obj_ids"], n_samples=64, n_importance=128,
                                   skip_boxes=[cases.box_affine(b) for b in inp["boxes"]])
    assert set(out) == set(want)
    gz = want["z_vals_coarse"]
    assert (out["z_vals_coarse"].cpu() - gz).abs().max().item() <= 1e-6
    untied = torch.ones_like(gz, dtype=torch.bool)   # tied depths: the oracle's tie order is torch's, see test_gpu_parity
    untied[:, 1:] &= gz[:, 1:] != gz[:, :-1]
    untied[:, :-1] &= gz[:, :-1] != gz[:, 1:]
    assert torch.equal(out["obj_ids_coarse"].cpu()[untied], want["obj_ids_coarse"][untied])
    tol = 2e-4 if precision == "fp32" else 3e-2
    ztol = {"coarse": 1e-6, "fine": 1e-4 if precision == "fp32" else 5e-2}
    for k in want:
        a, b = out[k].cpu(), want[k]
        if k.startswith("weights"):
            # 25 overlapping sets put samples of different sets within the depth tolerance of each other; such a pair
            # may sort either way against the oracle, so per-position weights are compared away from near ties (and
            # not for bf16 fine depths, which move by up to 5e-2 with the bf16 coarse weights; opacity covers their sum)
            p = k.split("_")[1]
            if p == "fine" and precision == "bf16":
                continue
            zw = want["z_vals_" + p]
            apart = torch.ones_like(zw, dtype=torch.bool)
            apart[:, 1:] &= (zw[:, 1:] - zw[:, :-1]).abs() > 2 * ztol[p]
            apart[:, :-1] &= (zw[:, 1:] - zw[:, :-1]).abs() > 2 * ztol[p]
            assert apart.float().mean() > 0.2   # (missed rays tie at z = 0 in every set)
            err = (a - b)[apart].abs()
            if p == "coarse":
                assert err.max().item() <= tol, k
            else:   # a fine depth 1e-4 off moves its delta, and at high density its weight by a few 1e-3
                assert (err > tol).float().mean().item() <= 1e-2 and err.max().item() <= 1e-2, k
        elif k.startswith(("rgb", "opacity", "depth")):
            t = tol if not k.startswith("depth") else max(tol, 5e-2 if precision == "bf16" else tol)
            err = (a - b).abs()
            if k.endswith("coarse") or precision == "bf16":
                assert err.max().item() <= t, k
            else:   # fp32 fine: the importance samples sit on sample_pdf's knife edge (test_gpu_parity.close_but) for a
                    # few rays, and 25 sets x 192 samples give it many chances; those rays are off by up to a few 1e-3
                assert err.max().item() <= 5e-3, k
        elif k == "z_vals_fine":   # fp32: the same knife edge moves a few importance samples
            err = (a - b).abs()
            t = 1e-4 if precision == "fp32" else 5e-2
            assert (err > t).float().mean().item() <= 3e-2 and err.max().item() <= max(t, 1e-2), k


def _composite_inputs(n_obj, n, s, seed):
    """Random sets with ties across sets, all-zero (muted) rays and descending sets."""
    g = torch.Generator().manual_seed(seed)
    z = torch.sort(torch.randint(0, 3 * s, (n_obj, n, s), generator=g).float() / 8 + 0.5, dim=2).values
    z[:, ::5] = 0.0                                       # muted rays
    if n_obj > 1:
        z[n_obj // 2, 1::3] = z[n_obj // 2, 1::3].flip(1)  # near > far: descending depths
    z[0, 2::7] = torch.rand(z[0, 2::7].shape, generator=g)  # unsorted set
    field = torch.rand(n_obj, n, s, 4, generator=g)
    field[..., 3] = field[..., 3] * 4 - 0.5
    return z.to(DEV).contiguous(), field.to(DEV).contiguous()


COMPOSITE_SHAPES = [(1, 37, 64), (3, 29, 2), (5, 101, 48), (2, 64, 2048), (24, 33, 192), (41, 19, 128)]


@pytest.mark.parametrize("n_obj,n,s", COMPOSITE_SHAPES)
def test_merge_path_order_is_the_stable_sort(n_obj, n, s):
    from object_nerf_b200 import engine
    z, field = _composite_inputs(n_obj, n, s, seed=n_obj * 1000 + s)
    out = engine.composite_multi(z, field, want_ids=True, want_unsorted=True, merge=True)
    cat = z.permute(1, 0, 2).reshape(n, n_obj * s)
    perm = torch.sort(cat.cpu(), dim=1, stable=True).indices.to(DEV)
    assert torch.equal(out["z_vals"], cat.gather(1, perm))
    assert torch.equal(out["obj_ids"], (perm // s).float())
    w_cat = out["weights_unsorted"].permute(1, 0, 2).reshape(n, n_obj * s)
    assert torch.equal(w_cat.gather(1, perm), out["weights"])
    # compositing in that order (float64 restatement of multi_rendering.py:125-150, last delta 0)
    zs = out["z_vals"].double()
    f = field.permute(1, 0, 2, 3).reshape(n, n_obj * s, 4).double().gather(1, perm[..., None].expand(-1, -1, 4))
    delta = torch.cat([zs[:, 1:] - zs[:, :-1], torch.zeros_like(zs[:, :1])], 1)
    alpha = 1 - torch.exp(-delta * f[..., 3].clamp(min=0))
    t = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], 1), 1)[:, :-1]
    w = alpha * t
    assert (out["weights"].double() - w).abs().max().item() < 1e-4
    assert (out["rgb"].double() - (w[..., None] * f[..., :3]).sum(1)).abs().max().item() < 1e-4
    if n_obj * s > 4096:   # the default entry takes the merge path on its own
        again = engine.composite_multi(z, field, want_ids=True, want_unsorted=True)
        _equal(again, out)


@pytest.mark.parametrize("n_obj,n,s", [x for x in COMPOSITE_SHAPES if x[0] * x[2] <= 4096])
@pytest.mark.parametrize("white_back", [False, True])
def test_merge_path_is_bit_identical_to_the_bitonic_kernel(n_obj, n, s, white_back):
    from object_nerf_b200 import engine
    z, field = _composite_inputs(n_obj, n, s, seed=7 + n_obj + s)
    a = engine.composite_multi(z, field, white_back, want_ids=True, want_unsorted=True, merge=True)
    b = engine.composite_multi(z, field, white_back, want_ids=True, want_unsorted=True)
    _equal(a, b)


def test_old_entry_still_refuses_above_4096():
    from object_nerf_b200 import _lib
    z, field = _composite_inputs(3, 4, 2048, seed=3)
    t = torch.empty(4, 3 * 2048, device=DEV)
    v = torch.empty(4, device=DEV)
    rgb = torch.empty(4, 3, device=DEV)
    rc = _lib.load().onerf_composite_multi(_lib.ctx(z.device), z.data_ptr(), field.data_ptr(), 4, 3, 2048, 0, t.data_ptr(),
                                           t.data_ptr(), None, None, v.data_ptr(), rgb.data_ptr(), v.data_ptr(),
                                           _lib.stream())
    assert rc == -2   # ONERF_ERR_UNSUPPORTED
    assert b"4096" in _lib.load().onerf_last_error()


CULL_CASES = {
    # hit pattern per object set; N not a multiple of 128 rays or samples
    "mixed": (300, [0, 4, 6, 4], 64, 64, [None, "none", "all", "one"]),
    "no_hits": (129, [0, 4, 4], 64, 64, [None, "none", "none"]),
    "objects_only": (77, [4, 6], 32, 32, ["one", None]),
    "beyond_cap": (53, MANY_IDS, 64, 128, None),
}


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(CULL_CASES))
def test_culled_one_call_is_bit_identical_to_staged_route(name, precision):
    n, ids, s, si, hits = CULL_CASES[name]
    c, inp = _case(n, ids, s, si, seed=640 + len(ids), hits=hits)
    setup = _setup(inp)
    one = _render(c, inp, precision, setup=setup)
    staged = _render(c, inp, precision, staged=True, setup=setup)
    _equal(one, staged)
    again = _render(c, inp, precision, setup=setup)   # repeatability
    _equal(one, again)


def test_culled_one_call_captures_in_a_cuda_graph():
    from object_nerf_b200 import engine
    from object_nerf_b200.multi_rendering import _render_multi_one_call, boxes_to_tensor
    from object_nerf_b200.rendering import _grid_of
    n, ids, s, si, hits = CULL_CASES["mixed"]
    c, inp = _case(n, ids, s, si, seed=650, hits=hits)
    models, emb, lib = _setup(inp)
    grid = _grid_of(emb["xyz"])
    code_table = engine._f32(lib.embedding_instance.weight.detach())
    boxes = boxes_to_tensor(_boxes(inp), torch.device(DEV))
    rays = [r.to(DEV).contiguous() for r in inp["rays_list"]]
    run = lambda: _render_multi_one_call(models, grid, code_table, rays, ids, s, False, 0.0, si, False, boxes, "bf16")
    with torch.no_grad():
        eager = run()
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            run()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                out = run()
        torch.cuda.current_stream().wait_stream(side)
        for v in out.values():
            v.zero_()
        g.replay()
        torch.cuda.synchronize()
    _equal(out, eager)
