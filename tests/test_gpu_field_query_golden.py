"""Field queries on the GPU against fixtures made from the reference's own modules (tests/golden/field_query_*.npz),
inference_model under grad against render_rays' training route in every configuration of the fixtures, and the
explicit-position encoding backwards against their o + d z entries."""
import ctypes as C

import pytest
import torch

from object_nerf_b200 import Embedding, inference_model, render_rays, synthetic as S
from tests import cases, field_query_cases as FQ, test_gpu_train_stages as TS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OUT_TOL = {"fp32": 2e-4, "bf16": 3e-2}


def _grads_match(fix, name, grad, precision):
    """fp32: norm and sampled entries within 5e-3 of the norm (1e-2 for the voxel table: a point on a voxel corner can fall
    in a neighbouring cell in fp32 arithmetic than in the reference's); bf16: the gate of test_gpu_train_tc.py, norm
    within 5 % and cosine of the sampled entries >= 0.995."""
    g = grad.reshape(-1).double().cpu()
    want_n = fix[name + "|norm"].double().item()
    s = g[cases.sample_indices(name, g.numel())]
    w = fix[name + "|samples"].double()
    if precision == "fp32":
        tol = 1e-2 if name == "voxel" else 5e-3
        return abs(g.norm().item() - want_n) <= tol * want_n and (s - w).abs().max().item() <= tol * want_n
    cos = (s @ w / (s.norm() * w.norm() + 1e-30)).item()
    # the voxel table's gradient is sparse: most of its 256 sampled entries are zero and a handful carry the cosine,
    # a noisier statistic than the whole-tensor cosine of that gate (its whole-tensor norm is held to the same 5 %)
    return 0.95 <= g.norm().item() / want_n <= 1.05 and cos >= (0.98 if name == "voxel" else 0.995)


def _psnr(a, b):
    return (-10 * torch.log10(((a.double().cpu() - b.double()) ** 2).mean().clamp_min(1e-30))).item()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(FQ.POINT_CASES))
def test_point_queries_match_reference_fixture(golden, monkeypatch, name, precision):
    monkeypatch.setenv("ONERF_PRECISION", precision)
    c = FQ.POINT_CASES[name]
    inp = FQ.build_point_case(c)
    fix = golden(f"field_query_{name}")
    model = S.make_model(inp["weights"], c["use_voxel"], DEV).train()
    emb = S.make_embedding(inp["grid"]).to(DEV) if c["use_voxel"] else Embedding(3, 10)
    codes = inp["codes"].to(DEV).requires_grad_(True)
    e = emb(inp["pts"].to(DEV))
    ex, ov = (e[0], e[1]) if c["use_voxel"] else (e, None)
    ed = Embedding(3, 4)(inp["dirs"].to(DEV))
    o = model.forward({"emb_xyz": ex, "emb_dir": ed})
    oi = model.forward_instance({"emb_xyz": ex, "emb_dir": ed, "obj_voxel": ov, "obj_code": codes})
    out = {"sigma": o["sigma"], "rgb": o["rgb"], "inst_sigma": oi["inst_sigma"], "inst_rgb": oi["inst_rgb"]}
    for k, v in out.items():
        assert v.shape == fix[k].shape, k
        err = (v.detach().cpu() - fix[k]).abs().max().item()
        assert err <= OUT_TOL[precision] * max(1.0, fix[k].abs().max().item()), (k, err)
        if precision == "bf16" and k.endswith("rgb"):
            assert _psnr(v.detach(), fix[k]) >= 45, k
    sum((out[k] * inp["cot"][k].to(DEV)).sum() for k in out).backward()
    for k, p in model.named_parameters():
        assert _grads_match(fix, k, p.grad, precision), k
    assert _grads_match(fix, "obj_code", codes.grad, precision)
    if c["use_voxel"]:
        tg = emb.embedding_space_ftr.weight.grad
        assert _grads_match(fix, "voxel", tg, precision)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(FQ.INFER_CASES))
def test_inference_model_matches_reference_fixture(golden, name, precision):
    c = FQ.INFER_CASES[name]
    inp = FQ.build_infer_case(c)
    fix = golden(f"field_query_{name}")
    model = S.make_model(inp["weights"], True, DEV).train()
    emb = S.make_embedding(inp["grid"]).to(DEV)
    codes = inp["codes"].to(DEV).requires_grad_(True)
    ptm = inp["pass_through_mask"].to(DEV) if inp["pass_through_mask"] is not None else None
    rand = {"noise_scene_coarse": inp["noise"]["noise_scene"].to(DEV), "noise_obj_coarse": inp["noise"]["noise_obj"].to(DEV)}
    res = {}
    inference_model(res, model, {"xyz": emb, "dir": Embedding(3, 4)}, "coarse", inp["xyz"].to(DEV),
                    inp["rays"][:, None, 3:6].to(DEV), inp["z"].to(DEV), 1024, c["noise_std"], False,
                    is_eval=c["is_eval"], use_zero_as_last_delta=c["zero_last_delta"],
                    forward_instance=c["forward_instance"], embedding_instance=codes,
                    frustum_bound_th=c["frustum_bound_th"], pass_through_mask=ptm, precision=precision, _rand=rand)
    keys = [k for k in FQ.MAP_KEYS if f"{k}_coarse" in fix]
    assert sorted(k for k in FQ.MAP_KEYS if f"{k}_coarse" in res) == sorted(keys)
    assert not res["weights_coarse"].requires_grad and not res["z_vals_coarse"].requires_grad
    for k in keys + ["weights"]:
        err = (res[f"{k}_coarse"].detach().cpu() - fix[f"{k}_coarse"]).abs().max().item()
        assert err <= OUT_TOL[precision], (k, err)
    sum((res[f"{k}_coarse"] * inp["cot"][k].to(DEV)).sum() for k in keys).backward()
    for k, p in model.named_parameters():
        if k + "|norm" in fix:
            assert _grads_match(fix, k, p.grad, precision), k
        else:
            assert p.grad is None, k      # the object branch when forward_instance is off
    assert _grads_match(fix, "voxel", emb.embedding_space_ftr.weight.grad, precision)
    if c["forward_instance"]:
        assert _grads_match(fix, "obj_code", codes.grad, precision)
    else:
        assert codes.grad is None


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(FQ.INFER_CASES))
def test_inference_model_matches_render_rays_in_every_configuration(name, precision):
    """render_rays (RenderRaysFn) at N_importance = 0 and inference_model under grad on its depths and rays, with the same
    injected noise, pass_through_mask, frustum_bound_th, eval flag, last delta and forward_instance: the same maps bit
    for bit, the same gradients up to atomic summation order."""
    c = FQ.INFER_CASES[name]
    w = S.make_weights(c["seed"], True, 8.0, 1.0)
    g = S.make_grid(**cases.GRID_KW)
    n, s = 96, 48
    rays = S.random_rays(c["seed"] + 7, n).to(DEV)
    gen = torch.Generator().manual_seed(c["seed"])
    codes0 = S.make_codes(3)[torch.randint(0, 7, (n,), generator=gen)].to(DEV)
    ptm = (torch.rand(n, 1, generator=gen) < 0.5).to(DEV) if c["pass_through"] else None
    noise = {"noise_scene_coarse": torch.randn(n, s, generator=gen).to(DEV),
             "noise_obj_coarse": torch.randn(n, s, generator=gen).to(DEV)}
    kw = dict(noise_std=c["noise_std"], is_eval=c["is_eval"], use_zero_as_last_delta=c["zero_last_delta"],
              forward_instance=c["forward_instance"], frustum_bound_th=c["frustum_bound_th"], pass_through_mask=ptm,
              precision=precision, _rand=noise)
    fi = c["forward_instance"]

    def run(route):
        model = S.make_model(w, True, DEV).train()
        emb = S.make_embedding(g).to(DEV)
        codes = codes0.clone().requires_grad_(True)
        embs = {"xyz": emb, "dir": Embedding(3, 4)}
        if route == "render":
            res = render_rays({"coarse": model}, embs, rays, N_samples=s, perturb=0, N_importance=0,
                              embedding_instance=codes, **kw)
        else:
            with torch.no_grad():
                z = render_rays({"coarse": model}, embs, rays, N_samples=s, perturb=0, N_importance=0,
                                embedding_instance=codes0, **kw)["z_vals_coarse"]
            res = {}
            inference_model(res, model, embs, "coarse", None, rays[:, 3:6], z, 1024, white_back=False,
                            embedding_instance=codes, _rays=rays, **kw)
        keys = [k for k in FQ.MAP_KEYS if f"{k}_coarse" in res]
        gg = torch.Generator(device=DEV).manual_seed(9)
        sum((res[f"{k}_coarse"] * (torch.rand(res[f"{k}_coarse"].shape, device=DEV, generator=gg) + 0.5)).sum()
            for k in keys).backward()
        grads = {k: p.grad for k, p in model.named_parameters()}
        grads["table"], grads["codes"] = emb.embedding_space_ftr.weight.grad, codes.grad
        return res, grads

    ref, ref_g = run("render")
    got, got_g = run("inference_model")
    assert sorted(got) == sorted(ref)
    for k in ref:
        assert torch.equal(got[k], ref[k]), k
    for k, v in ref_g.items():
        if not fi and (k.startswith(("instance_", "inst_")) or k == "codes"):
            assert got_g[k] is None, k
            continue
        rel = ((got_g[k] - v).norm() / v.norm().clamp_min(1e-30)).item()
        assert rel <= 1e-5, (k, rel)


def test_bwd_dx_at_explicit_positions_equals_rays_entry():
    """onerf_bwd_dx_xyz fed positions o + d z formed as the kernel forms them (one rounding of the exact product and sum)
    equals onerf_bwd_dx on rays + z within the matched gate of test_gpu_train_stages.py (atomic order)."""
    L = TS._lib()
    for n_rays, S_, want_object in ((1, 1, 1), (37, 61, 1), (300, 1, 1), (37, 61, 0)):
        w, g, rays, z, rays_d, z_d, packed, grid, ws, T = TS._dx_inputs(n_rays, S_, want_object, seed=11 + S_)
        B, n_tiles = n_rays * S_, T["n_tiles"]
        gen = torch.Generator(device=DEV).manual_seed(5)
        dz = {}
        for nm, slot, _, width in TS.DX_LAYERS:
            m = torch.randn(n_tiles * 128, 64 * T["dz_atoms"][slot], device=DEV, generator=gen)
            TS.helpers.write_atoms(ws, T["dz_off"][slot], m)
            dz[nm] = TS.bf(m[:B, :width]).double().cpu()
        xyz = (rays_d[:, None, 3:6].double() * z_d[:, :, None].double() + rays_d[:, None, 0:3].double()).float()
        xyz = xyz.reshape(-1, 3).contiguous()
        n_rows = g["table"].shape[0]
        prefill = torch.randn(n_rows, 24, device=DEV, generator=gen)
        a, b = prefill.clone(), prefill.clone()
        L.check(L.load().onerf_bwd_dx(TS._ctx(), want_object, packed.data_ptr(), ws.data_ptr(), rays_d.data_ptr(),
                                      z_d.data_ptr(), n_rays, S_, C.byref(grid.c), a.data_ptr(), L.stream()))
        L.check(L.load().onerf_bwd_dx_xyz(TS._ctx(), want_object, packed.data_ptr(), ws.data_ptr(), xyz.data_ptr(), B,
                                          C.byref(grid.c), b.data_ptr(), L.stream()))
        torch.cuda.synchronize()
        X = TS.helpers.from_atoms(ws, T["act_off"][0], n_tiles, 6)[:B].double().cpu()
        p = TS.grid_coords(rays, z, g["offset"], g["voxel_size"], fused=True)
        w_abs = {k: (v[0].to(torch.bfloat16).double().abs(), v[1]) for k, v in w.items()}
        bound = TS.table_grad_matched(TS.dx_from_dz({k: v.abs() for k, v in dz.items()}, w_abs, want_object),
                                      X.abs() + 2 ** -6, p, g["idx_map"], n_rows, want_object, bound=True)
        tol = 2e-4 * (bound + prefill.double().abs().cpu()) + 1e-6
        diff = (a.double() - b.double()).abs().cpu()
        assert (diff <= tol).all(), (n_rays, S_, diff.max().item())
        assert (a - prefill).abs().max() > 0


def test_encode_bwd_at_explicit_positions_equals_rays_entry():
    """onerf_encode_bwd_xyz with positions o + d z by multiply-then-add (the fp32 path's expression) equals
    onerf_encode_bwd on rays + z, chunked at sample0 = 0 and > 0, within the same gate."""
    L = TS._lib()
    n_rays, S_ = 37, 61
    w, g, rays, z, rays_d, z_d, packed, grid, ws, T = TS._dx_inputs(n_rays, S_, 1, seed=5)
    B = n_rays * S_
    X = TS.helpers.from_atoms(ws, T["act_off"][0], T["n_tiles"], 6)[:B].contiguous()
    gen = torch.Generator(device=DEV).manual_seed(3)
    dX = torch.randn(B, 384, device=DEV, generator=gen)
    xyz = (rays_d[:, None, 0:3] + rays_d[:, None, 3:6] * z_d[:, :, None]).reshape(-1, 3).contiguous()
    n_rows = g["table"].shape[0]
    prefill = torch.randn(n_rows, 24, device=DEV, generator=gen)
    a, b = prefill.clone(), prefill.clone()
    for s0, s1 in ((0, 1000), (1000, B)):
        L.check(L.load().onerf_encode_bwd(TS._ctx(), C.byref(grid.c), rays_d.data_ptr(), z_d.data_ptr(), n_rays, S_,
                                          X[s0:].data_ptr(), dX[s0:].data_ptr(), 384, s0, s1 - s0, a.data_ptr(), L.stream()))
        L.check(L.load().onerf_encode_bwd_xyz(TS._ctx(), C.byref(grid.c), xyz.data_ptr(), X[s0:].data_ptr(),
                                              dX[s0:].data_ptr(), 384, s0, s1 - s0, b.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    p = TS.grid_coords(rays, z, g["offset"], g["voxel_size"], fused=False)
    bound = TS.table_grad_matched(dX.double().cpu().abs(), X.double().cpu().abs() + 2 ** -6, p, g["idx_map"], n_rows, 1,
                                  bound=True)
    tol = 2e-4 * (bound + prefill.double().abs().cpu()) + 1e-6
    diff = (a.double() - b.double()).abs().cpu()
    assert (diff <= tol).all(), diff.max().item()
