"""GPU parity tests (pytest -m gpu).  Every CUDA stage and the full reference call
surface are compared with (a) the CPU oracle on the same seeded inputs and (b) the committed golden
fixtures produced by the real reference (tests/golden/, tools/make_golden.py).

Tolerances (fp32 arithmetic, different summation association / libm than torch CPU):
  depths (z)                     1e-6 abs
  fp32 field kernel outputs      2e-5 abs on rgb / sigma*1e-5 rel
  rendered maps, fp32 precision  5e-5 abs
  rendered maps, bf16 tensor-core precision: PSNR vs reference >= 45 dB and max abs err <= 3e-2
"""
import numpy as np
import pytest
import torch

from oracle import onerf_oracle as O
from tests import cases, helpers, synth

pytestmark = pytest.mark.gpu
DEV = "cuda"

PRECISIONS = ["fp32", "bf16"]


def grid_obj(g):
    return O.VoxelGrid(g["offset"], g["voxel_size"], g["shape"].tolist(), g["idx_map"], g["table"])


def close(a, b, tol, name):
    a = a.detach().cpu()
    assert a.shape == b.shape, (name, a.shape, b.shape)
    err = (a - b).abs().max().item() if a.numel() else 0.0
    assert err <= tol, f"{name}: max abs err {err:.3e} > {tol:.1e}"


def close_but(a, b, tol, name, max_outlier_frac, outlier_tol):
    """Like close(), but a small fraction of elements may differ by up to outlier_tol.  Used where the
    reference itself sits on a knife edge: in sample_pdf the u = 1 sample lands in bin M or M-1 depending on
    whether the fp32 cdf ends at 1.0 or one ulp above (models/rendering.py:42-56), which depends on the
    summation order of the normaliser and is not even stable across CPU ISAs."""
    a = a.detach().cpu()
    assert a.shape == b.shape, (name, a.shape, b.shape)
    err = (a - b).abs()
    bad = (err > tol).float().mean().item()
    assert bad <= max_outlier_frac, f"{name}: {bad:.4f} of elements differ by more than {tol:.1e}"
    assert err.max().item() <= outlier_tol, f"{name}: max abs err {err.max().item():.3e} > {outlier_tol:.1e}"


def test_sample_pdf_matches_golden(golden):
    from object_nerf_b200 import rendering
    g = golden("stage_sample_pdf")
    si = cases.stage_inputs()
    det = rendering.sample_pdf(si["pdf_bins"].to(DEV), si["pdf_weights"].to(DEV), 64, det=True)
    rnd = rendering.sample_pdf(si["pdf_bins"].to(DEV), si["pdf_weights"].to(DEV), 64, det=False,
                               _u=si["pdf_u"].to(DEV))
    close_but(det, g["det"], 2e-5, "sample_pdf det", 0.01, 0.1)
    close_but(rnd, g["rnd"], 2e-5, "sample_pdf rnd", 0.01, 0.1)


def test_encode_matches_golden(golden):
    from object_nerf_b200 import engine
    si = cases.stage_inputs()
    pe = engine.encode(si["posenc_x"].to(DEV), None)[0]
    close(pe, golden("stage_posenc")["pe10"], 2e-6, "pe10")
    g = synth.make_grid(**cases.GRID_KW)
    gm = helpers.GridModule(g).to(DEV)
    s, o = engine.encode(si["voxel_xyz"].to(DEV), engine.GridBuffers.from_module(gm))
    gold = golden("stage_voxel")
    # sin/cos of 2^5 * f: an ulp of f is amplified 32x
    close(s, gold["scene_in"], 2e-5, "voxel scene_in")
    close(o, gold["obj_in"], 2e-5, "voxel obj_in")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("use_voxel", [True, False])
def test_field_matches_oracle(precision, use_voxel):
    """Fused encode + two-branch MLP on a ragged batch (not a multiple of the tile)."""
    from object_nerf_b200 import engine
    n, s = 19, 40
    w = synth.make_weights(21, use_voxel, sigma_gain=8.0, sigma_bias=1.0)
    g = synth.make_grid(**cases.GRID_KW) if use_voxel else None
    rays = synth.random_rays(22, n)
    z = O.stratified_z(rays, s)
    codes = synth.make_codes(23)[torch.arange(n) % 7]
    xyz = (rays[:, None, 0:3] + rays[:, None, 3:6] * z[:, :, None]).reshape(-1, 3)
    dirs = rays[:, None, 3:6].expand(n, s, 3).reshape(-1, 3)
    cds = codes[:, None, :].expand(n, s, 64).reshape(n * s, 64)
    ref = O.field_eval(w, grid_obj(g) if g else None, xyz, dirs, cds)
    model = helpers.make_model(w, use_voxel, DEV)
    packed = engine.packed_for(model, use_voxel)
    gb = engine.GridBuffers.from_module(helpers.GridModule(g).to(DEV)) if g else None
    so, oo = engine.field(rays.to(DEV), z.to(DEV), packed, gb, codes=codes.to(DEV), precision=precision)
    so, oo = so.cpu().view(-1, 4), oo.cpu().view(-1, 4)
    rgb_tol, sig_tol = (2e-5, 2e-4) if precision == "fp32" else (2e-2, 0.35)
    close(so[:, :3], ref["rgb"], rgb_tol, "scene rgb")
    close(oo[:, :3], ref["inst_rgb"], rgb_tol, "obj rgb")
    close(so[:, 3], ref["sigma"], sig_tol, "scene sigma")
    close(oo[:, 3], ref["inst_sigma"], sig_tol, "obj sigma")


def _run_render_case(c, precision):
    from object_nerf_b200 import Embedding, render_rays
    inp = cases.build_render_case(c)
    uv = c["use_voxel"]
    models = {"coarse": helpers.make_model(inp["weights"]["coarse"], uv, DEV)}
    if c["n_importance"] > 0:
        models["fine"] = helpers.make_model(inp["weights"]["fine"], uv, DEV)
    emb = helpers.GridModule(inp["grid"]).to(DEV) if uv else Embedding(3, 10)
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    ptm = inp["pass_through_mask"].to(DEV) if inp["pass_through_mask"] is not None else None
    with torch.no_grad():
        return render_rays(models, {"xyz": emb, "dir": Embedding(3, 4)}, inp["rays"].to(DEV),
                           N_samples=c["n_samples"], use_disp=c["use_disp"], perturb=c["perturb"],
                           noise_std=c["noise_std"], N_importance=c["n_importance"], chunk=32768,
                           white_back=c["white_back"], forward_instance=c["forward_instance"],
                           embedding_instance=inp["codes"].to(DEV), frustum_bound_th=c["frustum_bound_th"],
                           pass_through_mask=ptm, rays_in_bbox=c["rays_in_bbox"], is_eval=c["is_eval"],
                           precision=precision, _rand=rand)



def _plan_for_case(c, precision):
    """The same case through the ONE-CALL C entry point onerf_render_rays_fwd (engine.RenderPlan)."""
    from object_nerf_b200 import engine
    from object_nerf_b200.rendering import _grid_of, _is_voxel
    from object_nerf_b200 import Embedding
    inp = cases.build_render_case(c)
    uv = c["use_voxel"]
    models = {"coarse": helpers.make_model(inp["weights"]["coarse"], uv, DEV)}
    if c["n_importance"] > 0:
        models["fine"] = helpers.make_model(inp["weights"]["fine"], uv, DEV)
    emb = helpers.GridModule(inp["grid"]).to(DEV) if uv else Embedding(3, 10)
    assert _is_voxel(emb) == uv
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    ptm = inp["pass_through_mask"].to(DEV) if inp["pass_through_mask"] is not None else None
    return engine.RenderPlan(
        inp["rays"].to(DEV), engine.packed_for(models["coarse"], uv),
        engine.packed_for(models["fine"], uv) if c["n_importance"] > 0 else None, _grid_of(emb),
        codes=inp["codes"].to(DEV), n_samples=c["n_samples"], n_importance=c["n_importance"], use_disp=c["use_disp"],
        perturb=c["perturb"], noise_std=c["noise_std"], white_back=c["white_back"],
        forward_instance=c["forward_instance"], is_eval=c["is_eval"], rays_in_bbox=c["rays_in_bbox"],
        frustum_bound_th=c["frustum_bound_th"], pass_through_mask=ptm, precision=precision, rand=rand), models, emb


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(cases.RENDER_CASES))
def test_one_call_render_entry_is_bit_identical_to_the_staged_path(name, precision):
    """onerf_render_rays_fwd (one C call, what a non-Python host binds) runs the same kernels in the same order as the
    Python-orchestrated render_rays(): every output map must be bit-identical."""
    c = cases.RENDER_CASES[name]
    staged = _run_render_case(c, precision)
    plan, _models, _emb = _plan_for_case(c, precision)
    fused = plan.run()
    torch.cuda.synchronize()
    assert set(fused) == set(staged)
    for k in staged:
        assert torch.equal(fused[k], staged[k]), k


def test_one_call_render_entry_is_cuda_graph_capturable():
    """SURVEY section 8b: no host reads of device data, no allocation on the hot path -> the whole forward captures into a
    CUDA graph; replays reproduce the eager result bit for bit."""
    c = cases.RENDER_CASES["eval_voxel"]
    plan, _models, _emb = _plan_for_case(c, "bf16")
    eager = {k: v.clone() for k, v in plan.run().items()}
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        plan.run()                                   # warm-up on the capture stream
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            out = plan.run()
    torch.cuda.current_stream().wait_stream(side)
    for _ in range(2):
        for v in out.values():
            v.zero_()
        g.replay()
        torch.cuda.synchronize()
        for k in eager:
            assert torch.equal(out[k], eager[k]), k

@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(cases.RENDER_CASES))
def test_render_rays_matches_reference_golden(golden, name, precision):
    c = cases.RENDER_CASES[name]
    gold = golden("render_" + name)
    out = _run_render_case(c, precision)
    assert set(out) == set(gold), (sorted(out), sorted(gold))
    for k, v in out.items():
        assert v.is_cuda and v.dtype == torch.float32 and tuple(v.shape) == tuple(gold[k].shape), k
    close(out["z_vals_coarse"], gold["z_vals_coarse"], 1e-6, "z_vals_coarse")
    train = c["perturb"] > 0
    masked = (not c["is_eval"]) and c["frustum_bound_th"] > 0
    if precision == "fp32":
        # jittered fine samples can sit ~1e-4 apart, so an ulp of z is a 1e-3 relative error of that
        # delta; with |sigma| up to ~1e2 the fp32 weights agree to a few 1e-4.  With random u the inverse
        # CDF divides by pdf mass as small as 1e-5, which amplifies the same ulps in z_vals_fine.
        for k in gold:
            tol = 5e-4 if k.startswith("weights") else (1e-3 if (train and k == "z_vals_fine") else 2e-4)
            close(out[k], gold[k], tol, k)
    else:
        for k in gold:
            inst = "instance" in k
            if masked and inst:
                # the occlusion mask (depth_scene + th < z, models/rendering.py:192-202) is a hard threshold:
                # a bf16-sized change of the scene depth flips single samples in or out for a few rays
                close_but(out[k], gold[k], 3e-2 if not k.startswith("depth") else 5e-2, k, 0.15, 0.6)
            elif k.startswith(("rgb", "opacity")):
                close(out[k], gold[k], 3e-2, k)
                assert helpers.psnr(out[k].cpu(), gold[k]) >= 45.0, (k, helpers.psnr(out[k].cpu(), gold[k]))
            elif k.startswith("depth"):
                close(out[k], gold[k], 5e-2, k)
            elif k.startswith("weights"):
                close(out[k], gold[k], 3e-2, k)


def _run_multi_case(c, precision, staged=False):
    from object_nerf_b200 import Embedding
    from object_nerf_b200.multi_rendering import render_rays_multi
    inp = cases.build_multi_case(c)
    models = {"coarse": helpers.make_model(inp["weights"]["coarse"], True, DEV),
              "fine": helpers.make_model(inp["weights"]["fine"], True, DEV)}
    emb = helpers.GridModule(inp["grid"]).to(DEV)
    boxes = None
    if inp["boxes"]:
        class Box:  # the attributes of BBoxRayHelper that the box mask reads
            pass
        boxes = {}
        for k, b in enumerate(inp["boxes"]):
            h = Box()
            h.scale_factor, h.pose_avg = b["scale_factor"], b["pose_avg"]
            h.axis_align_mat, h.bbox_bounds = b["axis_align_mat"], b["bbox_bounds"]
            boxes[k] = h
    return render_rays_multi(models, {"xyz": emb, "dir": Embedding(3, 4)}, helpers.CodeLib(inp["code_table"]).to(DEV),
                             [r.to(DEV) for r in inp["rays_list"]], c["obj_ids"], N_samples=c["n_samples"],
                             N_importance=c["n_importance"], white_back=c["white_back"],
                             background_skip_bbox=boxes, precision=precision, _staged=staged)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(cases.MULTI_CASES))
def test_render_multi_one_call_is_bit_identical_to_staged_route(name, precision):
    """onerf_render_multi_fwd (the whole render_rays_multi forward in one C call) against the same kernels driven stage by
    stage from Python."""
    c = cases.MULTI_CASES[name]
    one, staged = _run_multi_case(c, precision), _run_multi_case(c, precision, staged=True)
    assert set(one) == set(staged)
    for k in one:
        assert torch.equal(one[k], staged[k]), k


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(cases.MULTI_CASES))
def test_render_rays_multi_matches_reference_golden(golden, name, precision):
    c = cases.MULTI_CASES[name]
    gold = golden("multi_" + name)
    out = _run_multi_case(c, precision)
    assert set(out) == set(gold), (sorted(out), sorted(gold))
    close(out["z_vals_coarse"], gold["z_vals_coarse"], 1e-6, "z_vals_coarse")
    # object tags are only defined up to the order of tied depths (torch.sort is not stable; whole ray sets
    # tie at z = 0 when an object's bbox is missed, and those samples are muted: SURVEY.md appendix A.11)
    gz = gold["z_vals_coarse"]
    untied = torch.ones_like(gz, dtype=torch.bool)
    untied[:, 1:] &= gz[:, 1:] != gz[:, :-1]
    untied[:, :-1] &= gz[:, :-1] != gz[:, 1:]
    assert untied.float().mean() > 0.5
    assert torch.equal(out["obj_ids_coarse"].cpu()[untied], gold["obj_ids_coarse"][untied])
    tol = 2e-4 if precision == "fp32" else 3e-2
    for k in gold:
        if k.startswith(("rgb", "opacity", "weights", "depth")):
            close(out[k], gold[k], tol if not k.startswith("depth") else max(tol, 5e-2 if precision == "bf16" else tol), k)
        elif k.startswith("z_vals"):
            close(out[k], gold[k], 1e-4 if precision == "fp32" else 5e-2, k)


def test_composite_backward_matches_oracle_autograd():
    from object_nerf_b200 import engine
    rng = np.random.default_rng(41)
    n, s = 29, 96
    rays = synth.random_rays(42, n)
    z = O.merge_sorted(O.stratified_z(rays, 48), O.stratified_z(rays, 48) + 0.013)
    f = lambda *sh: torch.from_numpy(rng.standard_normal(sh).astype(np.float32))
    sigma, isigma = (f(n, s) * 5).requires_grad_(True), (f(n, s) * 5).requires_grad_(True)
    rgb, irgb = torch.sigmoid(f(n, s, 3)).requires_grad_(True), torch.sigmoid(f(n, s, 3)).requires_grad_(True)
    ns, no = f(n, s), f(n, s)
    ptm = torch.from_numpy(rng.random((n, 1)) < 0.5)
    ref = {}
    O.composite_pass(ref, "x", sigma, rgb, isigma, irgb, z, noise_std=1.0, is_eval=False, frustum_bound_th=0.05,
                     pass_through_mask=ptm, noise_scene=ns, noise_obj=no)
    names = ["rgb", "depth", "opacity", "rgb_instance", "depth_instance", "opacity_instance"]
    gout = {k: f(*ref[f"{k}_x"].shape) for k in names}
    loss = sum((ref[f"{k}_x"] * gout[k]).sum() for k in names)
    loss.backward()
    scene = torch.cat([rgb, sigma[..., None]], -1).detach().contiguous().to(DEV)
    obj = torch.cat([irgb, isigma[..., None]], -1).detach().contiguous().to(DEV)
    dscene, dobj = engine.composite_bwd(z.to(DEV), scene, obj, ref["depth_x"].detach().to(DEV),
                                        {k: v.to(DEV) for k, v in gout.items()}, noise_std=1.0, frustum_bound_th=0.05,
                                        pass_through_mask=ptm.to(DEV), noise_scene=ns.to(DEV), noise_obj=no.to(DEV))
    for got, want_rgb, want_sigma, nm in ((dscene, rgb.grad, sigma.grad, "scene"), (dobj, irgb.grad, isigma.grad, "obj")):
        got = got.cpu()
        scale = max(1.0, want_sigma.abs().max().item())
        close(got[..., :3], want_rgb, 1e-5 * max(1.0, want_rgb.abs().max().item()), nm + " d_rgb")
        close(got[..., 3], want_sigma, 2e-4 * scale, nm + " d_sigma")


def test_gemm_kernel_all_modes():
    import ctypes as C
    from object_nerf_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(5)
    for (M, N, K, ta) in ((70, 50, 33, 0), (3, 128, 5000, 1), (256, 271, 9000, 1), (200, 64, 1, 0), (1, 256, 4097, 1)):
        A = torch.from_numpy(rng.standard_normal((K, M) if ta else (M, K)).astype(np.float32)).to(DEV)
        Bm = torch.from_numpy(rng.standard_normal((K, N)).astype(np.float32)).to(DEV)
        Cm = torch.ones(M, N, device=DEV)
        want = (A.double().t() if ta else A.double()) @ Bm.double()
        for acc in (0, 1):
            Cm.fill_(1.0)
            _lib.check(lib.onerf_gemm(_lib.ctx(torch.device(DEV, 0)), A.data_ptr(), A.shape[1], ta, Bm.data_ptr(), N,
                                      Cm.data_ptr(), N, M, N, K, acc, _lib.stream()))
            ref = want + (1.0 if acc else 0.0)
            err = (Cm.double() - ref).abs().max().item()
            assert err <= 1e-4 * max(1.0, ref.abs().max().item()), (M, N, K, ta, acc, err)


def test_inference_model_call_surface(golden):
    """inference_model() with explicit xyz / rays_d, as the reference signature has it."""
    from object_nerf_b200 import Embedding, inference_model
    c = cases.RENDER_CASES["cfg1_voxel"]
    gold = golden("render_cfg1_voxel")
    inp = cases.build_render_case(c)
    model = helpers.make_model(inp["weights"]["coarse"], True, DEV)
    emb = helpers.GridModule(inp["grid"]).to(DEV)
    rays = inp["rays"]
    z = O.stratified_z(rays, 64)
    xyz = rays[:, None, 0:3] + rays[:, None, 3:6] * z[:, :, None]
    res = {}
    with torch.no_grad():
        inference_model(res, model, {"xyz": emb, "dir": Embedding(3, 4)}, "coarse", xyz.to(DEV),
                        rays[:, None, 3:6].to(DEV), z.to(DEV), 32768, 0.0, False, forward_instance=False,
                        embedding_instance=None, precision="fp32")
    for k in ("weights_coarse", "rgb_coarse", "depth_coarse", "opacity_coarse"):
        close(res[k], gold[k], 5e-5, k)


def test_training_step_gradients_match_reference_golden(golden):
    """config 3 in miniature: render_rays (train mode) -> TotalLoss -> backward on the CUDA kernels, compared with
    the REFERENCE's own backward (fixture written by tools/make_golden.py: loss, per-tensor norm + sampled entries)."""
    from object_nerf_b200 import CodeLibrary, Embedding, render_rays
    g = golden("grad_train_step")
    c = cases.GRAD_CASE
    inp = cases.build_grad_case()
    models = {k: helpers.make_model(w, True, DEV).train() for k, w in inp["weights"].items()}
    emb = helpers.GridModule(inp["grid"]).to(DEV)
    lib = helpers.CodeLib(inp["code_table"]).to(DEV)
    codes = lib.embedding_instance(inp["instance_ids"].view(-1).to(DEV))
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    out = render_rays(models, {"xyz": emb, "dir": Embedding(3, 4)}, inp["rays"].to(DEV), N_samples=c["n_samples"],
                      perturb=c["perturb"], noise_std=c["noise_std"], N_importance=c["n_importance"],
                      embedding_instance=codes, frustum_bound_th=c["frustum_bound_th"],
                      pass_through_mask=inp["pass_through_mask"].to(DEV), is_eval=False, precision="fp32", _rand=rand)
    batch = {k: v.to(DEV) for k, v in inp["batch"].items()}
    loss = cases.total_loss(out, batch)
    assert abs(loss.item() - g["loss"].item()) <= 2e-4 * abs(g["loss"].item()), (loss.item(), g["loss"].item())
    loss.backward()
    named = [(f"{typ}.{k}", p) for typ, m in models.items() for k, p in m.named_parameters()]
    named += [("codes", lib.embedding_instance.weight), ("voxel", emb.embedding_space_ftr.weight)]
    for name, p in named:
        assert p.grad is not None, name
        gr = p.grad.detach().cpu().reshape(-1)
        ref_norm = g[name + "|norm"].item()
        assert abs(gr.norm().item() - ref_norm) <= 2e-3 * max(ref_norm, 1e-7), (name, gr.norm().item(), ref_norm)
        idx = cases.sample_indices(name, gr.numel())
        err = (gr[idx] - g[name + "|samples"]).abs().max().item()
        # per-entry: within 1 % of the tensor's RMS entry (fp32 accumulation order differs from torch's)
        rms = max(ref_norm, 1e-7) / max(1.0, gr.numel() ** 0.5)
        assert err <= 1e-2 * rms + 1e-8, (name, err, rms)
    nz = torch.nonzero(emb.embedding_space_ftr.weight.grad.abs().sum(1)).view(-1).cpu()
    assert torch.equal(nz, g["voxel|nonzero_rows"])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_query_sigma_matches_oracle(precision):
    """SURVEY section 8f row 4: dense density queries (mesh extraction, voxel pruning) through the fused kernel."""
    from object_nerf_b200 import query_sigma
    c = cases.RENDER_CASES["eval_voxel"]
    inp = cases.build_render_case(c)
    model = helpers.make_model(inp["weights"]["fine"], True, DEV)
    emb = helpers.GridModule(inp["grid"]).to(DEV)
    g = torch.Generator().manual_seed(5)
    lo = -inp["grid"]["offset"]
    hi = lo + inp["grid"]["voxel_size"] * inp["grid"]["shape"].float()
    xyz = lo + (hi - lo) * torch.rand(3000, 3, generator=g)            # inside the grid, some in empty voxels
    xyz[:50] = xyz[:50] + 100.0                                          # far outside: zero voxel features
    code = inp["codes"][0]
    w, grid = inp["weights"]["fine"], grid_obj(inp["grid"])
    dirs = torch.zeros(xyz.shape[0], 3)
    want = O.field_eval(w, grid, xyz, dirs, code[None, :].expand(xyz.shape[0], -1))
    if precision == "bf16":   # the mesh-extraction call pattern (tools/extract_mesh.py:83-109) routes to the same kernel
        from object_nerf_b200 import EmbeddingVoxel
        e_s, e_o = EmbeddingVoxel.forward(emb, xyz.to(DEV))
        via_fwd = model.forward({"emb_xyz": e_s, "obj_voxel": e_o}, sigma_only=True)["sigma"][:, 0]
        via_inst = model.forward_instance({"emb_xyz": e_s, "obj_voxel": e_o, "obj_code": code.to(DEV)[None].expand(xyz.shape[0], -1)},
                                          sigma_only=True)["inst_sigma"][:, 0]
        assert torch.equal(via_fwd, query_sigma(model, emb, xyz.to(DEV)))
        assert torch.equal(via_inst, query_sigma(model, emb, xyz.to(DEV), obj_code=code.to(DEV)))
    got_s = query_sigma(model, emb, xyz.to(DEV), precision=precision).cpu()
    got_o = query_sigma(model, emb, xyz.to(DEV), obj_code=code.to(DEV), chunk=1024, precision=precision).cpu()
    tol = 2e-4 if precision == "fp32" else 3e-2
    for got, k in ((got_s, "sigma"), (got_o, "inst_sigma")):
        ref = want[k]
        assert ((got - ref).abs() <= tol * (1 + ref.abs())).all(), (k, (got - ref).abs().max().item())
