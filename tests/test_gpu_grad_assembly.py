"""How the tensor-core backward turns its kernel-layout buffers into the gradients the optimizer reads, entry by entry
against float64 (the restatement and the gate of tests/test_grad_assembly_cpu.py):
  - onerf_unpack_grads, both layouts, bit-exact: every reference entry is its prefill plus its one kernel entry;
  - onerf_render_rays_fwd + onerf_render_rays_bwd in bf16: every one of the 40 tensors of each pass and d_codes against
    the float64 assembly of the operands the kernels read back from the training workspace, the voxel-table gradient
    against the matched float64 reference of tests/test_train_stages_cpu.py;
  - training.train_step (onerf_train_step, then onerf_code_scatter_add) into prefilled .grad tensors: the same gates on
    both models, the code table's .grad by instance id (repeated and out-of-range ids), the voxel-table gradient;
  - onerf_code_gather / onerf_code_scatter_add, including ids outside the table."""
import ctypes as C

import pytest
import torch

from tests import cases, grad_plain, helpers
from tests.test_field_stages_cpu import GEMMS, N_OUT, REF, dims
from tests.test_gpu_train_stages import _grad_offsets
from tests.test_grad_assembly_cpu import (NAMES, OBJ, PRODUCERS, U, assemble, gate_constants, gate_share, prefill_adds,
                                         train_ws)
from tests.test_train_stages_cpu import dx_from_dz, grid_coords, table_grad_matched

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HEADS = {"scene.sigma": ("sigma_w", "sigma_b"), "scene.rgb": ("rgb_w", "rgb_b"), "obj.sigma": ("osigma_w", "osigma_b"),
         "obj.rgb": ("orgb_w", "orgb_b")}


def _lib():
    from object_nerf_b200 import _lib
    return _lib


def _ctx():
    return _lib().ctx(torch.device(DEV))


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


# ------------------------------------------------------------------------------------------------
# a. onerf_unpack_grads
# ------------------------------------------------------------------------------------------------
def expected_sources(use_voxel):
    """Per reference tensor, the kernel-buffer index each entry takes (-1: none, the hoisted direction and code columns),
    from the reference model's input definitions: the X-fed layers read [scene input | pad] at kernel column 0 and the
    object voxel block at kernel column 272, skip layers their hidden input after X, the dir layers leave the direction
    columns to the per-ray sums."""
    from object_nerf_b200 import synthetic
    xin, ovx, KX, KO = dims(use_voxel)
    oin = xin + ovx + 64
    Kd, w_off, b_off, heads, _ = _grad_offsets(use_voxel)
    shapes = {n: (o, i) for n, i, o in synthetic.layer_dims(bool(use_voxel))}
    ref_cols = {"scene.l0": [(0, 0, xin)], "scene.l4": [(0, 0, xin), (xin, KX, 256)],
                "obj.l0": [(0, 0, xin), (xin, 272, ovx)], "obj.l2": [(0, 0, xin), (xin, 272, ovx), (oin, KO, 128)],
                "scene.dir": [(0, 0, 256)], "obj.dir": [(0, 0, 128)]}
    src = {}
    for g in GEMMS:
        name = REF[g]
        n_out, n_in = shapes[name]
        K = Kd[g]
        idx = torch.full((n_out, n_in), -1, dtype=torch.long)
        rows = torch.arange(n_out)[:, None] * K + w_off[g]
        for ref0, k0, n in ref_cols.get(name, [(0, 0, n_in)]):
            idx[:, ref0:ref0 + n] = rows + torch.arange(k0, k0 + n)[None, :]
        src[name] = (idx, torch.arange(n_out) + b_off[g])
    for name, (hw, hb) in HEADS.items():
        n_out, n_in = shapes[name]
        src[name] = (heads[hw] + torch.arange(n_out * n_in).view(n_out, n_in), heads[hb] + torch.arange(n_out))
    return src


def _ref_tensors(use_voxel, gen, integer):
    from object_nerf_b200 import synthetic
    out = []
    for _, n_in, n_out in synthetic.layer_dims(bool(use_voxel)):
        for shape in ((n_out, n_in), (n_out,)):
            t = torch.randn(shape, device=DEV, generator=gen)
            out.append(torch.round(t * 2 ** 20) if integer else t)
    return out[0::2], out[1::2]


def test_unpack_grads_both_layouts_bit_exact():
    """Kernel buffer gk[i] = i + 1 (distinct, exact in fp32), reference tensors prefilled at random: each entry must be
    prefill + gk[its one kernel entry], entries fed by no kernel column (direction and code columns) keep their prefill
    bit for bit, and no padding column of the kernel layout is read.  Plain, voxel, plain in one context: the job
    tables are built once per context and layout."""
    L = _lib()
    lib = L.load()
    gen = torch.Generator(device=DEV).manual_seed(0)
    for use_voxel in (0, 1, 0):
        total = lib.onerf_grad_buffer_floats(use_voxel)
        gk = torch.arange(1, total + 1, dtype=torch.float32, device=DEV)
        for integer in (True, False):
            dW, db = _ref_tensors(use_voxel, gen, integer)
            pW, pb = [t.clone() for t in dW], [t.clone() for t in db]
            L.check(lib.onerf_unpack_grads(_ctx(), use_voxel, gk.data_ptr(), _ptrs(dW), _ptrs(db), L.stream()))
            torch.cuda.synchronize()
            src = expected_sources(use_voxel)
            seen = torch.zeros(total, dtype=torch.long)
            for i, name in enumerate(NAMES):
                for got, pre, idx in ((dW[i], pW[i], src[name][0]), (db[i], pb[i], src[name][1])):
                    idx = idx.to(DEV)
                    add = torch.where(idx >= 0, gk[idx.clamp(min=0)], torch.zeros_like(got))
                    want = torch.where(idx >= 0, pre + add, pre)       # one fp32 rounding, as the kernel's +=
                    assert torch.equal(got, want), (use_voxel, integer, name, (got != want).nonzero()[:4].tolist())
                    if integer:      # the sum is exact: recover which kernel entry arrived
                        arrived = (got - pre).long()
                        assert torch.equal(arrived, torch.where(idx >= 0, idx + 1, torch.zeros_like(idx))), name
                        seen += torch.bincount(idx[idx >= 0].cpu(), minlength=total)
            if integer:
                assert seen.max().item() == 1            # no kernel entry reaches two reference entries
                assert torch.equal(seen == 0, unread_kernel_entries(use_voxel, total))


def unread_kernel_entries(use_voxel, total):
    """The kernel-buffer entries no reference entry takes, stated as the complement of what the layers read: the kernel
    columns of the X-fed GEMMs that lie outside the layer's reference input (the scene layers: past the scene input; the
    object layers: past the scene input and outside the object voxel block at 272), and the gaps that align every block
    to 4 floats."""
    xin, ovx, KX, KO = dims(use_voxel)
    Kd, w_off, b_off, heads, off = _grad_offsets(use_voxel)
    unread = torch.ones(total, dtype=torch.bool)
    for g in GEMMS:
        K, N = Kd[g], N_OUT[g]
        cols = torch.ones(K, dtype=torch.bool)
        if g in ("S0", "S4"):
            cols[xin:KX] = False
        elif g in ("O0", "O2"):
            cols[xin:KO] = False
            cols[272:272 + ovx] = True
        unread[w_off[g]:w_off[g] + N * K] = ~cols.repeat(N)
        unread[b_off[g]:b_off[g] + N] = False
    for name, n in (("sigma_w", 256), ("sigma_b", 1), ("rgb_w", 384), ("rgb_b", 3), ("osigma_w", 128), ("osigma_b", 1),
                    ("orgb_w", 192), ("orgb_b", 3)):
        unread[heads[name]:heads[name] + n] = False
    return unread


# ------------------------------------------------------------------------------------------------
# b. onerf_render_rays_fwd + onerf_render_rays_bwd, bf16
# ------------------------------------------------------------------------------------------------
ASSEMBLY_CASES = {
    "voxel_1x2": dict(use_voxel=1, obj=1, R=1, S=2, Si=0, d_codes=True),      # the smallest shape render_rays takes
    "voxel_37x61_fine": dict(use_voxel=1, obj=1, R=37, S=61, Si=32, d_codes=True),
    "plain_37x61": dict(use_voxel=0, obj=1, R=37, S=61, Si=0, d_codes=True),
    "voxel_scene_only_13x200": dict(use_voxel=1, obj=0, R=13, S=200, Si=0, d_codes=True),
    "plain_13x200_fine_no_dcodes": dict(use_voxel=0, obj=1, R=13, S=200, Si=16, d_codes=False),
    "plain_scene_only_37x61_fine": dict(use_voxel=0, obj=0, R=37, S=61, Si=32, d_codes=True),
    "voxel_bench_2048x64_64": dict(use_voxel=1, obj=1, R=2048, S=64, Si=64, d_codes=True),
}


def _read_pass(ws, off, use_voxel, B):
    T = helpers.train_layout(bool(use_voxel), B)
    widths = [384 if use_voxel else 64] + [256] * 9 + [128] * 6 + [64]
    acts = [helpers.from_atoms(ws, off + T["act_off"][s], T["n_tiles"], T["act_atoms"][s])[:B, :widths[s]].double()
            for s in range(17)]
    dz = [helpers.from_atoms(ws, off + T["dz_off"][d], T["n_tiles"], T["dz_atoms"][d])[:B, :N_OUT[g]].double()
          for d, g in enumerate(GEMMS)]
    return acts, dz


def _f32_at(ws, off, n):
    return ws[off:off + 4 * n].view(torch.float32)


def _head_grads(dscene, dobj, scene, obj, B):
    """dA = d(rgb_pre, sigma) per sample from the field gradients and fields (onerf_head_bwd, bit-identical to fp32
    torch in tests/test_gpu_fp32_backward.py)."""
    L = _lib()
    dA = []
    for d, f in ((dscene, scene), (dobj, obj)):
        a = torch.zeros(B, 4, device=DEV)
        if d is not None:
            L.check(L.load().onerf_head_bwd(_ctx(), d.data_ptr(), f.data_ptr(), a.data_ptr(), B, L.stream()))
        dA.append(a)
    torch.cuda.synchronize()
    return dA[0].double(), dA[1].double()


def check_pass(ws, Wo, typ, uv, fi, R, Sp, dA, lin, got, pre, codes, label, shares):
    """Gate every entry of the 40 tensors of one pass (got = after the call, pre = before) against the float64 assembly
    of the operands the pass left in the training workspace; -> (d_codes, its bound, the pass's X and dZ) for the
    checks that sum over passes."""
    B = R * Sp
    acts, dz = _read_pass(ws, Wo["tl_" + typ], uv, B)
    pe = _f32_at(ws, Wo["pe"], R * 27).view(R, 27).double()
    codes64 = codes.double() if fi else torch.zeros(R, 64, dtype=torch.float64, device=DEV)
    ops = dict(acts=acts, dz=dz, dA_s=dA[0], dA_o=dA[1], pe=pe, codes=codes64)
    w = {n: (lin[i][0].detach().float(), lin[i][1].detach().float()) for i, n in enumerate(NAMES)}
    val, bnd, prod, (dc, dcb) = assemble(ops, w, uv, fi, Sp)
    cst, adds = gate_constants(B, R, Sp), prefill_adds(R)
    for i, name in enumerate(NAMES):
        for j in range(2):
            share = gate_share(got[i][j], pre[i][j], val[name][j], bnd[name][j], prod[name][j], cst, adds)
            worst = share.max().item()
            key = f"{typ}.{name}.{'W' if j == 0 else 'b'}"
            shares[key] = max(shares.get(key, 0.0), worst)
            assert worst <= 1.0, (label, key, worst, (share > 1).nonzero()[:4].tolist())
            if name in OBJ and not fi:
                assert torch.equal(got[i][j], pre[i][j]), key
    return dc, dcb, acts[0], dz


def table_grad_want(passes, w_by_pass, rays, g, fi):
    """Matched float64 voxel-table gradient summed over the passes (dX of the four X-fed layers on the bf16 weights,
    the PE chain rule on the dumped sin / cos, the trilinear scatter on the fp32 positions), and its bound."""
    n_rows = g["table"].shape[0]
    want = torch.zeros(n_rows, 24, dtype=torch.float64)
    bound = torch.zeros_like(want)
    for (X, dz, z), w in zip(passes, w_by_pass):
        dzd = {gm: dz[GEMMS.index(gm)].cpu() for gm in ("S0", "S4", "O0", "O2")}
        w_bf = {k: (v[0].detach().float().cpu().to(torch.bfloat16).double(), None) for k, v in w.items()}
        w_abs = {k: (v[0].abs(), None) for k, v in w_bf.items()}
        p = grid_coords(rays.cpu(), z.cpu(), g["offset"], g["voxel_size"], fused=True)
        Xc = X.cpu()
        want += table_grad_matched(dx_from_dz(dzd, w_bf, fi), Xc, p, g["idx_map"], n_rows, fi)
        bound += table_grad_matched(dx_from_dz({k: v.abs() for k, v in dzd.items()}, w_abs, fi), Xc.abs() + 2 ** -6, p,
                                    g["idx_map"], n_rows, fi, bound=True)
    return want, bound


def check_table_grad(got, prefill, want, bound, label, shares):
    """The gate of tests/test_gpu_train_stages.py::test_bwd_dx_matches_float64_references: 2e-4 (bound + |prefill|)."""
    err = ((got.double() - prefill.double()).cpu() - want).abs()
    tol = 2e-4 * (bound + prefill.double().abs().cpu()) + 1e-6
    shares["voxel_table"] = (err / tol).max().item()
    assert (err <= tol).all(), (label, shares["voxel_table"])


def _report(label, shares):
    print(f"\n{label}: worst share of its gate per tensor (1 = at the gate)")
    for k in sorted(shares, key=lambda k: -shares[k]):
        print(f"  {k:28s} {shares[k]:.3e}")


@pytest.mark.parametrize("case", list(ASSEMBLY_CASES))
def test_render_rays_bwd_tensors_match_float64_assembly(case):
    from object_nerf_b200 import engine
    c = ASSEMBLY_CASES[case]
    L = _lib()
    lib = L.load()
    uv, fi, R, S, Si = c["use_voxel"], c["obj"], c["R"], c["S"], c["Si"]
    inp = cases.build_render_case(dict(cases.RENDER_CASES["eval_voxel" if uv else "eval_plain"], n_rays=R,
                                       n_samples=S, n_importance=Si))
    typs = ["coarse"] + (["fine"] if Si else [])
    models = {t: helpers.make_model(inp["weights"][t], bool(uv), DEV) for t in typs}
    packed = {t: engine.packed_for(models[t], bool(uv)) for t in typs}
    grid = engine.GridBuffers.from_module(helpers.GridModule(inp["grid"]).to(DEV)) if uv else None
    rays, codes = inp["rays"].to(DEV), inp["codes"].to(DEV).contiguous()
    nbytes = lib.onerf_train_workspace_bytes_prec(L.PREC_BF16, uv, R, S, Si)
    Wo = train_ws(uv, R, S, Si)
    assert nbytes == Wo["total"]
    ws = helpers.aligned_u8(nbytes, DEV, fill=0)
    plan = engine.RenderPlan(rays, packed["coarse"], packed.get("fine"), grid, codes=codes, n_samples=S, n_importance=Si,
                             forward_instance=bool(fi), precision="bf16", train_ws=ws)
    out = plan.run()
    gen = torch.Generator(device=DEV).manual_seed(R + S)
    keys = ["rgb", "depth", "opacity"] + (["rgb_instance", "depth_instance", "opacity_instance"] if fi else [])
    gmaps = {t: {k: torch.randn(out[f"{k}_{t}"].shape, device=DEV, generator=gen) for k in keys} for t in typs}
    b = L.RenderBwdArgs()
    keep = []
    lin = {t: [(w.detach().float().contiguous(), bb) for w, bb in engine.model_linears(models[t])] for t in typs}
    pre, grads, shares = {}, {}, {}
    for t in typs:
        mg = getattr(b, t)
        for k, v in gmaps[t].items():
            setattr(mg, k, v.data_ptr())
        pre[t] = [(torch.randn(w.shape, device=DEV, generator=gen), torch.randn(bb.shape, device=DEV, generator=gen))
                  for w, bb in lin[t]]
        grads[t] = [(a.clone(), bb.clone()) for a, bb in pre[t]]
        Wp, dWp, dbp = _ptrs([w for w, _ in lin[t]]), _ptrs([a for a, _ in grads[t]]), _ptrs([bb for _, bb in grads[t]])
        keep += [Wp, dWp, dbp]
        setattr(b, "W_" + t, Wp)
        setattr(b, "dW_" + t, dWp)
        setattr(b, "db_" + t, dbp)
    dc_pre = torch.randn(R, 64, device=DEV, generator=gen)
    d_codes = dc_pre.clone() if c["d_codes"] else None
    b.d_codes = d_codes.data_ptr() if d_codes is not None else None
    tg_pre = torch.randn(inp["grid"]["table"].shape, device=DEV, generator=gen) if uv else None
    table_grad = tg_pre.clone() if uv else None
    b.table_grad = table_grad.data_ptr() if uv else None
    L.check(lib.onerf_render_rays_bwd(_ctx(), C.byref(plan.args), C.byref(b), L.stream()))
    torch.cuda.synchronize()
    dc_want = torch.zeros(R, 64, dtype=torch.float64, device=DEV)
    dc_bound = torch.zeros_like(dc_want)
    passes = []
    for t in typs:
        Sp = S + (Si if t == "fine" else 0)
        B = R * Sp
        if t == "coarse":       # the coarse pass runs last: its head gradients are still in the workspace
            dA = (_f32_at(ws, Wo["dA_s"], B * 4).view(B, 4).double(), _f32_at(ws, Wo["dA_o"], B * 4).view(B, 4).double())
        else:                   # the fine pass's were overwritten: recompute them from its fields
            scene = _f32_at(ws, Wo["scene_f"], B * 4).view(R, Sp, 4)
            obj = _f32_at(ws, Wo["obj_f"], B * 4).view(R, Sp, 4) if fi else None
            dscene, dobj = engine.composite_bwd(out["z_vals_fine"], scene, obj, out["depth_fine"], gmaps["fine"])
            dA = _head_grads(dscene, dobj, scene, obj, B)
        dc, dcb, X, dz = check_pass(ws, Wo, t, uv, fi, R, Sp, dA, lin[t], grads[t], pre[t], codes, case, shares)
        dc_want += dc
        dc_bound += dcb
        passes.append((X, dz, out["z_vals_" + t]))
    # d_codes: both passes add into it (fine, then coarse), each through two onerf_gemm calls
    if d_codes is not None:
        Smax = S + Si
        cd = gate_constants(R * Smax, R, Smax)
        cd[PRODUCERS.index("d_codes")] *= 2
        share = gate_share(d_codes, dc_pre, dc_want, dc_bound, torch.full((R, 64), PRODUCERS.index("d_codes")), cd,
                           prefill_adds(R, passes=len(typs)))
        shares["d_codes"] = share.max().item()
        assert share.max().item() <= 1.0, (case, share.max().item())
        if not fi:
            assert torch.equal(d_codes, dc_pre)
    if uv:
        want, bound = table_grad_want(passes, [dict(zip(NAMES, lin[t])) for t in typs], inp["rays"], inp["grid"], fi)
        check_table_grad(table_grad, tg_pre, want, bound, case, shares)
    _report(case, shares)


# ------------------------------------------------------------------------------------------------
# c. training.train_step into prefilled .grad tensors
# ------------------------------------------------------------------------------------------------
STEP_CASES = {"voxel": (True, None), "plain": (False, None), "voxel_2048": (True, 2048)}


@pytest.mark.parametrize("case", list(STEP_CASES))
def test_train_step_grads_match_float64_assembly(case):
    """onerf_train_step through training.train_step, every .grad prefilled: the 80 tensors of both models under the same
    gates (the fine pass's field gradients survive in TrainWs::dscene / dobj, so only its dA is recomputed; the coarse
    pass's dA is still in the workspace), d_codes, the code table's .grad = prefill + the scatter of d_codes by
    instance id with ids drawn from three rows plus ids below 0 and past the table (clamped to rows 0 and n_codes - 1,
    the rows the gather read), and the voxel-table gradient."""
    from object_nerf_b200 import Embedding, engine, training
    uv, n_rays = STEP_CASES[case]
    L = _lib()
    inp = cases.build_grad_case(n_rays=n_rays) if uv else grad_plain.build_grad_case_plain()
    c = cases.GRAD_CASE if uv else grad_plain.GRAD_CASE_PLAIN
    R = inp["rays"].shape[0]
    S, Si = c["n_samples"], c["n_importance"]
    models = {k: helpers.make_model(w, uv, DEV).train() for k, w in inp["weights"].items()}
    emb = helpers.GridModule(inp["grid"]).to(DEV) if uv else Embedding(3, 10)
    lib = helpers.CodeLib(inp["code_table"]).to(DEV)
    n_codes = lib.embedding_instance.weight.shape[0]
    gen = torch.Generator(device=DEV).manual_seed(R)
    ids = torch.tensor([4, 6, 9], device=DEV)[torch.randint(0, 3, (R,), device=DEV, generator=gen)]
    ids[:3] = torch.tensor([-3, n_codes, n_codes + 1000], device=DEV)
    batch = {k: v.to(DEV) for k, v in inp["batch"].items()}
    batch["rays"], batch["instance_ids"] = inp["rays"].to(DEV), ids
    typs = ["coarse"] + (["fine"] if Si else [])
    trained = [p for t in typs for w, bb in engine.model_linears(models[t]) for p in (w, bb)]
    trained += [lib.embedding_instance.weight] + ([emb.embedding_space_ftr.weight] if uv else [])
    for p in trained:
        p.grad = torch.randn(p.shape, device=DEV, generator=gen)
    pre = [p.grad.clone() for p in trained]
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    training.train_step(models, {"xyz": emb, "dir": Embedding(3, 4)}, lib, batch, cases.LOSS_CONF, N_samples=S,
                        perturb=c["perturb"], noise_std=c["noise_std"], N_importance=Si,
                        frustum_bound_th=c["frustum_bound_th"], pass_through_mask=inp["pass_through_mask"].to(DEV),
                        is_eval=False, precision="bf16", _rand=rand)
    torch.cuda.synchronize()
    (plan,) = training._plans[models["coarse"]].values()
    ws = plan.ws
    Wo = train_ws(uv, R, S, Si)
    assert ws.numel() >= Wo["step_total"]
    maps = plan.render.maps
    shares, passes, k = {}, [], 0
    dc_want = torch.zeros(R, 64, dtype=torch.float64, device=DEV)
    dc_bound = torch.zeros_like(dc_want)
    for t in typs:
        lin = engine.model_linears(models[t])
        got = [(lin[i][0].grad, lin[i][1].grad) for i in range(20)]
        pr = [(pre[k + 2 * i], pre[k + 2 * i + 1]) for i in range(20)]
        k += 40
        Sp = S + (Si if t == "fine" else 0)
        B = R * Sp
        if t == "coarse":
            dA = (_f32_at(ws, Wo["dA_s"], B * 4).view(B, 4).double(), _f32_at(ws, Wo["dA_o"], B * 4).view(B, 4).double())
        else:
            scene = _f32_at(ws, Wo["scene_f"], B * 4).view(R, Sp, 4)
            obj = _f32_at(ws, Wo["obj_f"], B * 4).view(R, Sp, 4)
            dA = _head_grads(_f32_at(ws, Wo["dscene"], B * 4), _f32_at(ws, Wo["dobj"], B * 4), scene, obj, B)
        dc, dcb, X, dz = check_pass(ws, Wo, t, uv, 1, R, Sp, dA, lin, got, pr, plan.codes, case, shares)
        dc_want += dc
        dc_bound += dcb
        passes.append((X, dz, maps[t]["z_vals"]))
    # d_codes (zeroed by the step, both passes add into it), then its scatter into the code table's .grad
    cd = gate_constants(R * (S + Si), R, S + Si)
    cd[PRODUCERS.index("d_codes")] *= 2
    share = gate_share(plan.d_codes, None, dc_want, dc_bound, torch.full((R, 64), PRODUCERS.index("d_codes")), cd)
    shares["d_codes"] = share.max().item()
    assert share.max().item() <= 1.0, (case, shares["d_codes"])
    rows = ids.clamp(0, n_codes - 1)
    assert torch.equal(plan.codes, lib.embedding_instance.weight.detach()[rows])
    cg, cpre = lib.embedding_instance.weight.grad, pre[k]
    want = cpre.double().index_add(0, rows, plan.d_codes.double())
    bound = cpre.double().abs().index_add(0, rows, plan.d_codes.double().abs())
    m = torch.bincount(rows, minlength=n_codes).double()[:, None]
    err = (cg.double() - want).abs()
    shares["code_table"] = (err / torch.where(bound > 0, (m + 1) * U * bound, torch.ones_like(bound))).max().item()
    assert (err <= (m + 1) * U * bound).all(), (case, shares["code_table"])
    assert m[0].item() >= 1 and m[n_codes - 1].item() >= 2     # the clamped ids landed on rows 0 and n_codes - 1
    untouched = m[:, 0] == 0
    assert torch.equal(cg[untouched], cpre[untouched])
    if uv:
        w_by_pass = [dict(zip(NAMES, engine.model_linears(models[t]))) for t in typs]
        want, bound = table_grad_want(passes, w_by_pass, inp["rays"], inp["grid"], 1)
        check_table_grad(emb.embedding_space_ftr.weight.grad, pre[k + 1], want, bound, case, shares)
    _report(f"train_step {case}", shares)


# ------------------------------------------------------------------------------------------------
# d. code gather / scatter
# ------------------------------------------------------------------------------------------------
def _gather(table, ids):
    L = _lib()
    out = torch.full((ids.numel(), 64), float("nan"), device=DEV)
    L.check(L.load().onerf_code_gather(_ctx(), table.data_ptr(), ids.data_ptr(), ids.numel(), table.shape[0],
                                       out.data_ptr(), L.stream()))
    return out


def _scatter(d_codes, ids, grad):
    L = _lib()
    L.check(L.load().onerf_code_scatter_add(_ctx(), d_codes.data_ptr(), ids.data_ptr(), ids.numel(), grad.shape[0],
                                            grad.data_ptr(), L.stream()))


@pytest.mark.parametrize("n", [1, 7, 4097])
def test_code_gather_is_exact(n):
    gen = torch.Generator(device=DEV).manual_seed(n)
    table = torch.randn(64, 64, device=DEV, generator=gen)
    ids = torch.randint(0, 64, (n,), device=DEV, generator=gen)
    out = _gather(table, ids)
    torch.cuda.synchronize()
    assert torch.equal(out, table[ids])


@pytest.mark.parametrize("n", [1, 300, 20000])
def test_code_scatter_exact_on_integers_and_bounded_on_random(n):
    """Integer-valued d_codes sum exactly in any order, so the scatter is bit-exact against float64 when rows repeat
    heavily (ids drawn from 3 rows) and with ids only 0 and n_codes - 1; random d_codes stay within the bound of m
    fp32 atomic adds per row: (m + 1) 2^-24 (|prefill| + sum |terms|)."""
    gen = torch.Generator(device=DEV).manual_seed(n)
    n_codes = 64
    for ids in (torch.randint(0, n_codes, (n,), device=DEV, generator=gen),
                torch.tensor([5, 9, 63], device=DEV)[torch.randint(0, 3, (n,), device=DEV, generator=gen)],
                torch.tensor([0, n_codes - 1], device=DEV)[torch.randint(0, 2, (n,), device=DEV, generator=gen)]):
        dci = torch.randint(-64, 65, (n, 64), device=DEV, generator=gen).float()
        pre = torch.randint(-1000, 1001, (n_codes, 64), device=DEV, generator=gen).float()
        grad = pre.clone()
        _scatter(dci, ids, grad)
        want = pre.double().index_add(0, ids, dci.double())
        torch.cuda.synchronize()
        assert torch.equal(grad.double(), want)
        dc = torch.randn(n, 64, device=DEV, generator=gen)
        pre = torch.randn(n_codes, 64, device=DEV, generator=gen)
        grad = pre.clone()
        _scatter(dc, ids, grad)
        want = pre.double().index_add(0, ids, dc.double())
        bound = pre.double().abs().index_add(0, ids, dc.double().abs())
        m = torch.bincount(ids, minlength=n_codes).double()[:, None]
        torch.cuda.synchronize()
        assert ((grad.double() - want).abs() <= (m + 1) * U * bound).all()


def test_code_scatter_sends_out_of_range_ids_to_the_row_the_gather_read():
    """The gather clamps an id outside [0, n_codes) to row 0 / n_codes - 1; the scatter must add that ray's gradient to
    the same row, so the code that was rendered is the code that learns."""
    gen = torch.Generator(device=DEV).manual_seed(3)
    n_codes = 8
    table = torch.randn(n_codes, 64, device=DEV, generator=gen)
    ids = torch.tensor([-5, -1, 0, 3, 7, 8, 1 << 40, 2], device=DEV)
    rows = ids.clamp(0, n_codes - 1)
    out = _gather(table, ids)
    torch.cuda.synchronize()
    assert torch.equal(out, table[rows])
    dc = torch.randint(-64, 65, (ids.numel(), 64), device=DEV, generator=gen).float()
    grad = torch.zeros(n_codes, 64, device=DEV)
    _scatter(dc, ids, grad)
    torch.cuda.synchronize()
    assert torch.equal(grad, torch.zeros_like(grad).index_add(0, rows, dc))


def test_code_gather_scatter_with_no_rays_launch_nothing():
    L = _lib()
    dev = torch.device(DEV)
    table = torch.randn(4, 64, device=DEV)
    ids = torch.zeros(1, dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    n0 = L.launch_count(dev)
    L.check(L.load().onerf_code_gather(_ctx(), table.data_ptr(), ids.data_ptr(), 0, 4, table.data_ptr(), L.stream()))
    L.check(L.load().onerf_code_scatter_add(_ctx(), table.data_ptr(), ids.data_ptr(), 0, 4, table.data_ptr(), L.stream()))
    assert L.launch_count(dev) == n0
