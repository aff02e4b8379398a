"""Differentiable field queries at given points (ObjectNeRF.forward / forward_instance on embedded points, Embedding(3, 4)
on directions, inference_model under autograd) against the float64 autograd of the oracle's ObjectNeRF, and against
render_rays' own training route."""
import pytest
import torch

from object_nerf_b200 import Embedding, inference_model, render_rays, synthetic as S
from oracle import onerf_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _setup(use_voxel, n=3000, seed=0):
    w = S.make_weights(11 + seed, use_voxel, 8.0, 1.0)
    model = S.make_model(w, use_voxel, DEV).train()
    g = S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05)
    emb = S.make_embedding(g).to(DEV) if use_voxel else Embedding(3, 10)
    gen = torch.Generator().manual_seed(seed)
    ext = g["shape"].double() * float(g["voxel_size"])
    # inside the grid, up to half a voxel outside, and exactly on voxel corners (edges of the trilinear cells)
    u = torch.rand(n, 3, generator=gen, dtype=torch.float64) * 1.1 - 0.05
    pts = (u * ext - g["offset"].double()).float()
    pts[: n // 10] = (torch.randint(0, 20, (n // 10, 3), generator=gen).double() * float(g["voxel_size"])
                      - g["offset"].double()).float()
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=1)
    codes = S.make_codes(7)[torch.randint(0, 64, (n,), generator=gen)]
    return w, model, g, emb, pts, dirs, codes


def _oracle(model, g, use_voxel, pts, dirs, codes, branch, sigma_only, cot):
    """float64 reference outputs and gradients of sum(out * cot) (CPU autograd of the oracle's MLP)."""
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in model.state_dict().items()}
    w = {k: (sd[v + ".weight"], sd[v + ".bias"]) for k, v in S.REF_NAMES.items()}
    table = g["table"].double().requires_grad_(True)
    grid = O.VoxelGrid(g["offset"].double(), g["voxel_size"].double(), g["shape"].tolist(), g["idx_map"], table) \
        if use_voxel else None
    c = codes.double().requires_grad_(True)
    out = O.field_eval(w, grid, pts.double(), dirs.double(), c, want_scene=branch == "scene",
                       want_object=branch == "object")
    sig, rgb = (out["sigma"], out["rgb"]) if branch == "scene" else (out["inst_sigma"], out["inst_rgb"])
    f = sig[:, None] if sigma_only else torch.cat([rgb, sig[:, None]], 1)
    (f * cot.double()).sum().backward()
    grads = {k: v.grad for k, v in sd.items()}
    return f.detach(), grads, (table.grad if use_voxel else None), c.grad


def _rel(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / b.double().norm().clamp_min(1e-30)).item()


def _close(got, want, precision, fp32_tol=5e-3):
    """fp32: relative norm error <= fp32_tol (the kernels encode in fp32: sin / cos of 2^9 x carry up to 2^9 ulp of x, the
    oracle encodes in float64).  bf16: the gate of the tensor-core training tests (test_gpu_train_tc.py): norm within 5 %
    and cosine >= 0.995."""
    g, w = got.double().cpu().reshape(-1), want.double().cpu().reshape(-1)
    if precision == "fp32":
        return _rel(g, w) <= fp32_tol
    cos = (g @ w / (g.norm() * w.norm() + 1e-30)).item()
    return 0.95 <= (g.norm() / w.norm().clamp_min(1e-30)).item() <= 1.05 and cos >= 0.995


def _cotangent(n, width, seed):
    """loss-like weights in [0.5, 1.5): a gradient summed over many points, as a training loss gives"""
    return torch.rand(n, width, generator=torch.Generator().manual_seed(seed)) + 0.5


@pytest.mark.parametrize("precision,out_tol", [("fp32", 2e-4), ("bf16", 3e-2)])
@pytest.mark.parametrize("use_voxel", [True, False])
@pytest.mark.parametrize("branch,sigma_only", [("scene", False), ("object", False), ("scene", True), ("object", True)])
def test_point_query_matches_float64_autograd(monkeypatch, precision, out_tol, use_voxel, branch, sigma_only):
    monkeypatch.setenv("ONERF_PRECISION", precision)
    w, model, g, emb, pts, dirs, codes = _setup(use_voxel)
    n = pts.shape[0]
    cot = _cotangent(n, 1 if sigma_only else 4, 3)
    ref_f, ref_g, ref_table, ref_codes = _oracle(model, g, use_voxel, pts, dirs, codes, branch, sigma_only, cot)
    e = emb(pts.to(DEV))
    inputs = {"emb_xyz": e[0] if use_voxel else e, "emb_dir": Embedding(3, 4)(dirs.to(DEV))}
    code_dev = codes.to(DEV).requires_grad_(True)
    if branch == "object":
        if use_voxel:
            inputs["obj_voxel"] = e[1]
        inputs["obj_code"] = code_dev
        out = model.forward_instance(inputs, sigma_only=sigma_only)
        sig, rgb = out["inst_sigma"], out.get("inst_rgb")
    else:
        out = model.forward(inputs, sigma_only=sigma_only)
        sig, rgb = out["sigma"], out.get("rgb")
    f = sig if sigma_only else torch.cat([rgb, sig], 1)
    assert f.shape == ref_f.shape
    err = (f.detach().cpu().double() - ref_f).abs().max().item()
    assert err <= out_tol * max(1.0, ref_f.abs().max().item()), err
    (f * cot.to(DEV)).sum().backward()
    got = dict(model.named_parameters())
    for k, rg in ref_g.items():
        p = got[k]
        reached = rg is not None and rg.abs().sum() > 0
        if not reached:
            # the reference's graph does not reach this tensor: None, not zeros (Adam treats them differently)
            assert p.grad is None, k
            continue
        assert p.grad is not None, k
        assert _close(p.grad, rg, precision), (k, _rel(p.grad, rg))
    if use_voxel:
        tg = emb.embedding_space_ftr.weight.grad
        # 1e-2: a point on a voxel corner can fall in a neighbouring cell in fp32 position arithmetic than in float64,
        # sending its share of the gradient to that cell's rows
        assert _close(tg, ref_table, precision, fp32_tol=1e-2), _rel(tg, ref_table)
    if branch == "object":
        assert _close(code_dev.grad, ref_codes, precision), _rel(code_dev.grad, ref_codes)
    else:
        assert code_dev.grad is None


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_inference_model_matches_render_rays_training(precision):
    """inference_model under grad on render_rays' own coarse depths (N_importance = 0) gives RenderRaysFn's maps bit for
    bit and its gradients up to atomic summation order; with positions given explicitly as o + d z, the explicit-position
    dump and encoding backward agree within rounding of the positions."""
    w = S.make_weights(21, True, 8.0, 1.0)
    g = S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05)
    rays = S.random_rays(104, 200).to(DEV)
    codes0 = S.make_codes(105)[torch.arange(200) % 7].to(DEV)

    def run(route):
        model = S.make_model(w, True, DEV).train()
        emb = S.make_embedding(g).to(DEV)
        codes = codes0.clone().requires_grad_(True)
        embs = {"xyz": emb, "dir": Embedding(3, 4)}
        if route == "render":
            res = render_rays({"coarse": model}, embs, rays, N_samples=64, perturb=0, noise_std=0, N_importance=0,
                              embedding_instance=codes, precision=precision)
        else:
            with torch.no_grad():
                z = render_rays({"coarse": model}, embs, rays, N_samples=64, perturb=0, noise_std=0,
                                N_importance=0, embedding_instance=codes0, precision=precision)["z_vals_coarse"]
            res = {}
            xyz = rays[:, None, 0:3] + rays[:, None, 3:6] * z[:, :, None]
            inference_model(res, model, embs, "coarse", xyz, rays[:, 3:6], z, chunk=1024, noise_std=0,
                            white_back=False, embedding_instance=codes, precision=precision,
                            _rays=rays if route == "rays" else None)
        gen = torch.Generator(device=DEV).manual_seed(9)
        loss = sum((res[k] * torch.randn(res[k].shape, device=DEV, generator=gen)).sum()
                   for k in ("rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_instance_coarse",
                             "depth_instance_coarse", "opacity_instance_coarse"))
        loss.backward()
        grads = {k: p.grad for k, p in model.named_parameters()}
        grads["table"] = emb.embedding_space_ftr.weight.grad
        grads["codes"] = codes.grad
        return res, grads

    ref, ref_g = run("render")
    got, got_g = run("rays")
    for k in ("rgb_coarse", "depth_coarse", "opacity_coarse", "weights_coarse", "rgb_instance_coarse"):
        assert torch.equal(got[k], ref[k]), k
    for k, v in ref_g.items():
        assert _rel(got_g[k], v) <= 1e-5, (k, _rel(got_g[k], v))
    xg, x_g = run("xyz")
    for k in ("rgb_coarse", "depth_coarse", "rgb_instance_coarse"):
        assert (xg[k] - ref[k]).abs().max().item() <= (2e-4 if precision == "fp32" else 3e-2), k
    for k, v in ref_g.items():
        assert _rel(x_g[k], v) <= (1e-3 if precision == "fp32" else 3e-2), (k, _rel(x_g[k], v))


def test_point_query_tiles_of_one_sample_rays(monkeypatch):
    """S = 1: every 128-sample tile spans 128 rays; a batch that is not a multiple of 128 and bigger than a chunk."""
    from object_nerf_b200 import field_query
    old = field_query.CHUNK_SAMPLES
    field_query.CHUNK_SAMPLES = 1000
    try:
        w, model, g, emb, pts, dirs, codes = _setup(True, n=2777, seed=1)
        monkeypatch.setenv("ONERF_PRECISION", "bf16")
        cot = _cotangent(pts.shape[0], 4, 4)
        ref_f, ref_g, ref_table, ref_codes = _oracle(model, g, True, pts, dirs, codes, "object", False, cot)
        e = emb(pts.to(DEV))
        code_dev = codes.to(DEV).requires_grad_(True)
        out = model.forward_instance({"emb_xyz": e[0], "obj_voxel": e[1], "emb_dir": Embedding(3, 4)(dirs.to(DEV)),
                                      "obj_code": code_dev})
        f = torch.cat([out["inst_rgb"], out["inst_sigma"]], 1)
        (f * cot.to(DEV)).sum().backward()
        assert _close(code_dev.grad, ref_codes, "bf16"), _rel(code_dev.grad, ref_codes)
        assert _close(emb.embedding_space_ftr.weight.grad, ref_table, "bf16")
        for k, p in model.named_parameters():
            if k.startswith(("instance_", "inst_")):
                assert _close(p.grad, ref_g[k], "bf16"), k
    finally:
        field_query.CHUNK_SAMPLES = old


def test_dir_embedding_and_refusals():
    d = torch.nn.functional.normalize(torch.randn(100, 3, generator=torch.Generator().manual_seed(0)), dim=1)
    pe = Embedding(3, 4)(d.to(DEV))
    assert pe.shape == (100, 27)
    assert (pe.cpu() - O.posenc(d, 4)).abs().max().item() <= 1e-6
    d2 = Embedding(3, 4)(d.to(DEV).reshape(100, 1, 3))
    assert d2.shape == (100, 1, 27)
    w, model, g, emb, pts, dirs, codes = _setup(True, n=64)
    e = emb(pts.to(DEV))
    p = pts.to(DEV).requires_grad_(True)
    e2 = emb(p)
    with pytest.raises(ValueError):
        model.forward({"emb_xyz": e2[0], "emb_dir": Embedding(3, 4)(dirs.to(DEV))})
    with pytest.raises(ValueError):
        model.forward({"emb_xyz": e[0]})
