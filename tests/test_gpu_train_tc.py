"""Tensor-core training path (SURVEY.md §8 row a14) through the C ABI: stage kernels against plain PyTorch fp32
references of the same op, and the whole step against the reference's own backward (fixture) and the fp32 path."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import cases, helpers, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

GEMM_OF_DZ = ["S0", "S1", "S2", "S3", "S4", "S5", "S6", "S7", "SFIN", "SDIR", "O0", "O1", "O2", "O3", "OFIN", "ODIR"]
GEMM_N = dict(S0=256, S1=256, S2=256, S3=256, S4=256, S5=256, S6=256, S7=256, SFIN=256, SDIR=128,
              O0=128, O1=128, O2=128, O3=128, OFIN=128, ODIR=64)
GEMM_K = dict(S0=288, S1=256, S2=256, S3=256, S4=544, S5=256, S6=256, S7=256, SFIN=256, SDIR=256,
              O0=384, O1=128, O2=512, O3=128, OFIN=128, ODIR=128)
GEMM_ORDER = ["S0", "S1", "S2", "S3", "S4", "S5", "S6", "S7", "SFIN", "SDIR", "O0", "O1", "O2", "O3", "OFIN", "ODIR"]


def grad_layout():
    off, w_off, b_off = 0, {}, {}
    for g in GEMM_ORDER:
        w_off[g] = off
        off += GEMM_N[g] * GEMM_K[g]
        b_off[g] = off
        off += GEMM_N[g]
        off = (off + 3) // 4 * 4
    heads = {}
    for name, n in (("sigma_w", 256), ("sigma_b", 1), ("rgb_w", 384), ("rgb_b", 3), ("osigma_w", 128), ("osigma_b", 1),
                    ("orgb_w", 192), ("orgb_b", 3)):
        heads[name] = off
        off += (n + 3) // 4 * 4
    return w_off, b_off, heads, off


def _lib():
    from object_nerf_b200 import _lib
    return _lib


def test_wgrad_kernel_matches_torch_matmul():
    """dW_l = dZ_l^T In_l over all samples with MN-major wgmma operands, on random bf16 operand tiles."""
    L = _lib()
    lib = L.load()
    n_samples = 128 * 37          # 37 tiles: 74 stages, not a multiple of anything convenient
    T = helpers.train_layout(True, n_samples)
    ws = helpers.aligned_u8(T["total"], DEV, fill=0)
    g = torch.Generator(device=DEV).manual_seed(0)
    acts = [torch.randn(n_samples, 64 * a, device=DEV, generator=g) for a in T["act_atoms"]]
    dzs = [torch.randn(n_samples, 64 * a, device=DEV, generator=g) for a in T["dz_atoms"]]
    for i, m in enumerate(acts):
        helpers.write_atoms(ws, T["act_off"][i], m)
    for i, m in enumerate(dzs):
        helpers.write_atoms(ws, T["dz_off"][i], m)
    w_off, b_off, heads, total = grad_layout()
    assert lib.onerf_grad_buffer_floats(1) == total
    grad = torch.zeros(total, device=DEV)
    L.check(lib.onerf_bwd_wgrad(L.ctx(torch.device(DEV)), 1, 1, ws.data_ptr(), n_samples, grad.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    bf = lambda t: t.to(torch.bfloat16).float()
    X = bf(acts[0])
    inputs = {  # kernel-K order
        "S0": X[:, :288], "S4": torch.cat([X[:, :288], bf(acts[4])], 1), "O0": X[:, :384],
        "O2": torch.cat([X[:, :384], bf(acts[12])], 1),
        "SFIN": bf(acts[8]), "SDIR": bf(acts[9]), "O1": bf(acts[11]), "O3": bf(acts[13]), "OFIN": bf(acts[14]),
        "ODIR": bf(acts[15]),
    }
    for l in (1, 2, 3, 5, 6, 7):
        inputs[f"S{l}"] = bf(acts[l])
    for d, gname in enumerate(GEMM_OF_DZ):
        dz = bf(dzs[d])[:, :GEMM_N[gname]]
        want = dz.t().double() @ inputs[gname].double()
        got = grad[w_off[gname]:w_off[gname] + GEMM_N[gname] * GEMM_K[gname]].view(GEMM_N[gname], GEMM_K[gname]).double()
        if gname in ("S0", "S4"):      # columns 271..287 belong to zero-weight padding: not part of the contract
            pass
        err = (got - want).abs().max().item()
        scale = want.abs().max().item()
        assert err <= 2e-3 * scale, (gname, err, scale)


def _small_scene(n_rays=96, S=64):
    c = dict(cases.RENDER_CASES["eval_voxel"], n_rays=n_rays)
    inp = cases.build_render_case(c)
    return inp


def _run_field(inp, S, precision, train=False, activations=False):
    from object_nerf_b200 import engine
    model = helpers.make_model(inp["weights"]["coarse"], True, DEV)
    emb = helpers.GridModule(inp["grid"]).to(DEV)
    rays = inp["rays"].to(DEV)
    n = rays.shape[0]
    z = engine.sample_coarse(rays, S)
    packed = engine.packed_for(model, True)
    grid = engine.GridBuffers.from_module(emb)
    codes = inp["codes"].to(DEV)
    return model, emb, rays, z, packed, grid, codes, n


def test_training_forward_dump_matches_fp32_activations():
    """The bf16 forward's training dump (activation tiles, X tiles, sign masks) against the fp32 kernel's activation dump."""
    from object_nerf_b200 import engine
    L = _lib()
    inp = _small_scene()
    S = 64
    model, emb, rays, z, packed, grid, codes, n = _run_field(inp, S, "bf16")
    B = n * S
    T = helpers.train_layout(True, B)
    ws = helpers.aligned_u8(T["total"], DEV, fill=0)
    a = L.FieldArgs()
    scene = torch.empty(n, S, 4, device=DEV)
    obj = torch.empty(n, S, 4, device=DEV)
    rc = torch.empty(n, 448, device=DEV)
    a.rays, a.z, a.z_stride, a.codes = rays.data_ptr(), z.data_ptr(), S, codes.data_ptr()
    a.n_rays, a.n_samples = n, S
    a.grid = C.pointer(grid.c)
    a.packed = packed.data_ptr()
    a.want_scene, a.want_object, a.precision = 1, 1, L.PREC_BF16
    a.scene_out, a.obj_out, a.out_stride, a.ray_const = scene.data_ptr(), obj.data_ptr(), S, rc.data_ptr()
    a.train_ws = ws.data_ptr()
    L.check(L.load().onerf_field_fwd(L.ctx(torch.device(DEV)), C.byref(a), L.stream()))
    # same result as the plain bf16 forward
    scene2, obj2 = engine.field(rays, z, packed, grid, codes=codes, precision="bf16")
    torch.cuda.synchronize()
    assert torch.equal(scene, scene2) and torch.equal(obj, obj2)
    # fp32 activations
    widths = [384] + [256] * 8 + [256, 128] + [128] * 4 + [128, 64]
    acts = [torch.empty(B, w, device=DEV) for w in widths]
    ptrs = (C.c_void_p * 17)(*[t.data_ptr() for t in acts])
    engine.field(rays, z, packed, grid, codes=codes, precision="fp32", activations=ptrs)
    torch.cuda.synchronize()
    masks = helpers.read_masks(ws, T)
    for slot in range(17):
        got = helpers.from_atoms(ws, T["act_off"][slot], T["n_tiles"], T["act_atoms"][slot])[:B, :widths[slot]]
        want = acts[slot]
        tol = 2e-2 + 2e-2 * want.abs()
        bad = ((got - want).abs() > tol).float().mean().item()
        assert bad < 2e-3, (slot, bad, (got - want).abs().max().item())
    # sign masks of the activated layers (compare where the fp32 value is clearly away from zero)
    word0 = {**{s: (s - 1) * 8 for s in range(1, 9)}, 10: 64, **{s: 68 + (s - 11) * 4 for s in range(11, 15)}, 16: 84}
    for slot, w0 in word0.items():
        Wd = widths[slot]
        nbits = 16 if Wd == 64 else 32
        bits = torch.stack([(masks[:, w0 + w, :] >> j) & 1 for w in range(Wd // nbits) for j in range(nbits)], -1)  # (T,128,Wd)
        bits = bits.reshape(-1, Wd)[:B]
        want = acts[slot] > 0
        clear = acts[slot].abs() > 2e-2
        agree = ((bits == 1) == want)[clear].float().mean().item()
        assert agree > 0.999, (slot, agree)


def _torch_chain(acts_bf, w, dA_s, dA_o):
    """fp32 reference of the input-gradient chain: dZ of every GEMM layer from the dumped (bf16) activations."""
    lk = lambda h: torch.where(h > 0, 1.0, 0.01)
    W = {k: (v[0].to(DEV), v[1].to(DEV)) for k, v in w.items()}
    dz = {}
    dz["SDIR"] = (dA_s[:, :3] @ W["scene.rgb"][0]) * lk(acts_bf[10])
    dz["SFIN"] = dz["SDIR"] @ W["scene.dir"][0][:, :256]
    d = (dz["SFIN"] @ W["scene.final"][0] + dA_s[:, 3:4] * W["scene.sigma"][0]) * lk(acts_bf[8])
    dz["S7"] = d
    for l in range(7, 0, -1):
        Wl = W[f"scene.l{l}"][0]
        if l == 4:
            Wl = Wl[:, 271:]
        d = (dz[f"S{l}"] @ Wl) * lk(acts_bf[l])
        dz[f"S{l-1}"] = d
    dz["ODIR"] = (dA_o[:, :3] @ W["obj.rgb"][0]) * lk(acts_bf[16])
    dz["OFIN"] = dz["ODIR"] @ W["obj.dir"][0][:, :128]
    dz["O3"] = (dz["OFIN"] @ W["obj.final"][0] + dA_o[:, 3:4] * W["obj.sigma"][0]) * lk(acts_bf[14])
    dz["O2"] = (dz["O3"] @ W["obj.l3"][0]) * lk(acts_bf[13])
    dz["O1"] = (dz["O2"] @ W["obj.l2"][0][:, 439:]) * lk(acts_bf[12])
    dz["O0"] = (dz["O1"] @ W["obj.l1"][0]) * lk(acts_bf[11])
    return dz


def test_bwd_chain_matches_torch_reference():
    from object_nerf_b200 import engine
    L = _lib()
    inp = _small_scene(n_rays=70)     # 70 x 64 = 4480 samples = 35 tiles
    S = 64
    model, emb, rays, z, packed, grid, codes, n = _run_field(inp, S, "bf16")
    B = n * S
    T = helpers.train_layout(True, B)
    ws = helpers.aligned_u8(T["total"], DEV, fill=0)
    a = L.FieldArgs()
    scene = torch.empty(n, S, 4, device=DEV); obj = torch.empty(n, S, 4, device=DEV); rc = torch.empty(n, 448, device=DEV)
    a.rays, a.z, a.z_stride, a.codes = rays.data_ptr(), z.data_ptr(), S, codes.data_ptr()
    a.n_rays, a.n_samples = n, S
    a.grid = C.pointer(grid.c); a.packed = packed.data_ptr()
    a.want_scene, a.want_object, a.precision = 1, 1, L.PREC_BF16
    a.scene_out, a.obj_out, a.out_stride, a.ray_const = scene.data_ptr(), obj.data_ptr(), S, rc.data_ptr()
    a.train_ws = ws.data_ptr()
    ctx = L.ctx(torch.device(DEV))
    L.check(L.load().onerf_field_fwd(ctx, C.byref(a), L.stream()))
    g = torch.Generator(device=DEV).manual_seed(1)
    dA_s = torch.randn(B, 4, device=DEV, generator=g)
    dA_o = torch.randn(B, 4, device=DEV, generator=g)
    L.check(L.load().onerf_bwd_chain(ctx, 1, 1, packed.data_ptr(), ws.data_ptr(), B, dA_s.data_ptr(), dA_o.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    widths = [384] + [256] * 8 + [256, 128] + [128] * 4 + [128, 64]
    acts = [helpers.from_atoms(ws, T["act_off"][s], T["n_tiles"], T["act_atoms"][s])[:B, :widths[s]] for s in range(17)]
    want = _torch_chain(acts, inp["weights"]["coarse"], dA_s, dA_o)
    for d, gname in enumerate(GEMM_OF_DZ):
        got = helpers.from_atoms(ws, T["dz_off"][d], T["n_tiles"], T["dz_atoms"][d])[:B, :GEMM_N[gname]]
        ref = want[gname]
        scale = ref.abs().mean().item() + 1e-12
        err = (got - ref).abs()
        # bf16 operands at every layer: compare in units of the layer's mean magnitude
        assert err.mean().item() <= 2e-2 * scale, (gname, err.mean().item(), scale)
        assert (err > 0.25 * scale + 0.05 * ref.abs()).float().mean().item() < 5e-3, (gname, err.max().item(), scale)


def _train_step(precision, inp, c, rand):
    from object_nerf_b200 import Embedding, render_rays
    models = {k: helpers.make_model(w, True, DEV).train() for k, w in inp["weights"].items()}
    emb = helpers.GridModule(inp["grid"]).to(DEV)
    lib = helpers.CodeLib(inp["code_table"]).to(DEV)
    codes = lib.embedding_instance(inp["instance_ids"].view(-1).to(DEV))
    out = render_rays(models, {"xyz": emb, "dir": Embedding(3, 4)}, inp["rays"].to(DEV), N_samples=c["n_samples"],
                      perturb=c["perturb"], noise_std=c["noise_std"], N_importance=c["n_importance"],
                      embedding_instance=codes, frustum_bound_th=c["frustum_bound_th"],
                      pass_through_mask=inp["pass_through_mask"].to(DEV), is_eval=False, precision=precision, _rand=rand)
    batch = {k: v.to(DEV) for k, v in inp["batch"].items()}
    loss = cases.total_loss(out, batch)
    loss.backward()
    named = [(f"{typ}.{k}", p) for typ, m in models.items() for k, p in m.named_parameters()]
    named += [("codes", lib.embedding_instance.weight), ("voxel", emb.embedding_space_ftr.weight)]
    return loss, named


def test_training_step_bf16_gradients_match_reference_golden(golden):
    """config 3 in miniature on the tensor cores: loss and gradients against the REFERENCE's own backward (fixture).
    Tolerances for bf16 operands / fp32 accumulation: loss 2 %, per-tensor norm 5 %, direction (cosine) >= 0.995."""
    g = golden("grad_train_step")
    c = cases.GRAD_CASE
    inp = cases.build_grad_case()
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    loss, named = _train_step("bf16", inp, c, rand)
    assert abs(loss.item() - g["loss"].item()) <= 2e-2 * abs(g["loss"].item()), (loss.item(), g["loss"].item())
    loss32, named32 = _train_step("fp32", inp, c, rand)
    report = []
    for (name, p), (_, p32) in zip(named, named32):
        assert p.grad is not None, name
        gr, g32 = p.grad.detach().reshape(-1).double(), p32.grad.detach().reshape(-1).double()
        ref_norm = g[name + "|norm"].item()
        cos = (gr @ g32 / (gr.norm() * g32.norm() + 1e-30)).item()
        report.append((name, gr.norm().item() / max(ref_norm, 1e-12), cos))
    bad = [r for r in report if not (0.95 <= r[1] <= 1.05 and r[2] >= 0.995)]
    assert not bad, bad


@pytest.mark.parametrize("n_rays", [2048])
def test_training_step_bf16_vs_fp32_at_batch_size(n_rays):
    """2048 rays (config/default_conf.yml:40) of the bench scene: tensor-core gradients against the fp32 path."""
    c = dict(cases.GRAD_CASE, n_rays=n_rays)
    inp = cases.build_grad_case(n_rays=n_rays)
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    loss, named = _train_step("bf16", inp, c, rand)
    loss32, named32 = _train_step("fp32", inp, c, rand)
    assert abs(loss.item() - loss32.item()) <= 2e-2 * abs(loss32.item())
    bad = []
    for (name, p), (_, p32) in zip(named, named32):
        gr, g32 = p.grad.detach().reshape(-1).double(), p32.grad.detach().reshape(-1).double()
        ratio = (gr.norm() / (g32.norm() + 1e-30)).item()
        cos = (gr @ g32 / (gr.norm() * g32.norm() + 1e-30)).item()
        if not (0.95 <= ratio <= 1.05 and cos >= 0.995):
            bad.append((name, ratio, cos))
    assert not bad, bad
