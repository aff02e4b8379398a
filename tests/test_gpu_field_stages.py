"""The field forward (onerf_field_fwd) layer by layer against float64 references of the same operation, on the operands
the kernel itself read: the tensor-core kernel (csrc/field_tc.cu) through its training dump (X, every layer's bf16
output, the LeakyReLU sign masks), the per-ray constants (ray_const_kernel), the heads, the inference modes, and the
FFMA kernel (csrc/field_fp32.cu) through its fp32 activation dump.

Each GEMM layer is checked on its own dumped input with a monotone interval gate: its epilogue f is non-decreasing in
the fp32 pre-activation t, so f(t64 - d) <= got <= f(t64 + d), t64 the float64 pre-activation and d = c K B,
B = sum |a| |w| + |bias or ray_const term|.  c = 2^-23 for wgmma (twice the textbook fp32 bound), 2^-24 with K + 2
terms for the sequential FFMA dot products.  The weights are the reference-layout fp32 weights mapped to kernel-K
order and rounded here, never read from the packed blob.  The references are checked in tests/test_field_stages_cpu.py.
Each check prints the largest share of its gate that a result used."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from tests import cases, helpers, synth
from tests.test_field_stages_cpu import (DIR_LAYER, GEMMS, MASK_WORD0, N_OUT, SIGMA_LAYER, bf16, ffma_epilogue,
                                         gate_share, kernel_weights, point_in_boxes32, positions, preact, ray_const_ref,
                                         tc_epilogue, voxel_features32, x_reference, x_reference_ffma)
from tests.test_gpu_train_stages import GRID, _edge_rays, _train_forward, _wgrad_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODELS = {"voxel": True, "plain": False}
# (n_rays, S) from the SM count: fewer tiles than SMs, one tile per CTA, three tiles per CTA, a partial last tile with
# rays straddling tiles, S = 1, rays spanning several tiles; big_features: voxel features up to |f| ~ 10 (positions up
# to |x| ~ 9 for the plain model), the range edge of __sincosf and of the double-angle steps
SHAPES = {"few_tiles": lambda m: (10, 64), "one_tile_per_cta": lambda m: (2 * m, 64),
          "three_tiles_per_cta": lambda m: (3 * m, 128), "partial_straddle": lambda m: (77, 63),
          "s1": lambda m: (3001, 1), "long_rays": lambda m: (13, 200), "big_features": lambda m: (77, 63)}


def _lib():
    from object_nerf_b200 import _lib
    return _lib


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _report(label, r):
    print(f"RATIO {label}: {r:.3e}")
    return r


def _launch(packed, grid, rays, z, S, codes=None, code_row=None, want_scene=1, want_object=1, rc=None, z_stride=None,
            outs=None, out_stride=None, xyz=None, mute=0, boxes=None, precision=None, activations=None):
    """One onerf_field_fwd launch (inference unless activations) -> (scene, obj, ray_const)."""
    L = _lib()
    n = rays.shape[0]
    out_stride = out_stride or S
    if outs is None:
        outs = (torch.empty(n, out_stride, 4, device=DEV) if want_scene else None,
                torch.empty(n, out_stride, 4, device=DEV) if want_object else None)
    rc = torch.empty(n, 448, device=DEV) if rc is None else rc
    a = L.FieldArgs()
    a.rays, a.z, a.z_stride = rays.data_ptr(), z.data_ptr(), z_stride or S
    a.codes = codes.data_ptr() if codes is not None else None
    a.code_row = code_row.data_ptr() if code_row is not None else None
    a.xyz = xyz.data_ptr() if xyz is not None else None
    a.n_rays, a.n_samples = n, S
    a.grid = C.pointer(grid.c) if grid is not None else None
    a.packed = packed.data_ptr()
    a.want_scene, a.want_object = int(want_scene), int(want_object)
    a.precision = L.PREC_BF16 if precision is None else precision
    a.mute_zero_rays = int(mute)
    a.boxes, a.n_boxes = (boxes.data_ptr(), boxes.shape[0]) if boxes is not None else (None, 0)
    a.scene_out = outs[0].data_ptr() if want_scene else None
    a.obj_out = outs[1].data_ptr() if want_object else None
    a.out_stride, a.ray_const = out_stride, rc.data_ptr()
    a.activations = activations
    L.check(L.load().onerf_field_fwd(L.ctx(torch.device(DEV)), C.byref(a), L.stream()))
    return outs[0], outs[1], rc


def _case_inputs(use_voxel, shape):
    """Weights, grid, rays, depths and per-ray codes of one case (host tensors) and the device model."""
    from object_nerf_b200 import engine
    n, S = SHAPES[shape](_sms())
    rng = np.random.default_rng(n * 1000 + S)
    inp = cases.build_render_case(dict(cases.RENDER_CASES["eval_voxel" if use_voxel else "eval_plain"], n_rays=n))
    rays = inp["rays"].clone()
    z = engine.sample_coarse(rays.to(DEV), S).cpu()
    if S == 1:
        z[:] = 1.6
    g = None
    if use_voxel:
        g = synth.make_grid(**dict(GRID, feat_scale=2.5 if shape == "big_features" else 1.0))
        rays[:n // 2], z[:n // 2] = _edge_rays(g, n // 2, S, rng)
    elif shape == "big_features":
        z = z * 3.0
    w = inp["weights"]["coarse"]
    model = helpers.make_model(w, use_voxel, DEV)
    packed = engine.packed_for(model, use_voxel)
    grid = engine.GridBuffers.from_module(helpers.GridModule(g).to(DEV)) if use_voxel else None
    return dict(w=w, g=g, n=n, S=S, rays=rays.to(DEV).contiguous(), z=z.to(DEV).contiguous(),
                codes=inp["codes"].to(DEV).contiguous(), packed=packed, grid=grid, use_voxel=use_voxel)


def _dump_run(c):
    """The training-dump launch of a case on a workspace filled with 0xFF (bf16 NaN) -> the case dict plus the slots."""
    ws, T, scene, obj, rc = _train_forward(c["rays"], c["z"], c["packed"], c["grid"], c["codes"], int(c["use_voxel"]), 1,
                                           fill=0xFF, outputs=True)
    torch.cuda.synchronize()
    nt = T["n_tiles"]
    acts = [helpers.from_atoms(ws, T["act_off"][s], nt, T["act_atoms"][s]) for s in range(17)]
    return dict(c, ws=ws, T=T, scene=scene, obj=obj, rc=rc, acts=acts, B=c["n"] * c["S"])


@functools.lru_cache(maxsize=1)
def _stage_run(model, shape):
    return _dump_run(_case_inputs(MODELS[model], shape))


# ------------------------------------------------------------------------------------------------
# stage checks of one dump launch
# ------------------------------------------------------------------------------------------------
def check_x(r, label):
    """X (slot 0) against the float64 encoding of the kernel's fp32 positions fmaf(d, z, o): bf16(ref - e) <= got <=
    bf16(ref + e) with the per-octave budget e of x_reference (derivation at pe_budget); pad columns exactly 0."""
    uv, B = r["use_voxel"], r["B"]
    x32 = positions(r["rays"], r["z"], fused=True)
    feats = voxel_features32(x32, r["g"]) if uv else None
    ref, e = x_reference(x32, feats, uv)
    got = r["acts"][0][:B, :ref.shape[1]].double()
    q = gate_share(ref, e, got, bf16)
    _report(f"X {label}", q.max().item())
    bad = (q > 1).nonzero()
    assert bad.numel() == 0, (label, "X columns failing:", bad[:, 1].unique().tolist()[:20], q.max().item())
    pads = [63] if not uv else [271] + list(range(376, 384))
    assert (got[:, pads] == 0).all()
    return feats


def check_layers(r, label):
    """Every GEMM layer (slots 1-16) on its own dumped input against the interval gate with c = 2^-23; each hidden
    layer has at least 5 % of its live outputs negative and 5 % positive."""
    uv, B, S = r["use_voxel"], r["B"], r["S"]
    kw = {g: (W.to(DEV), b.to(DEV)) for g, (W, b) in kernel_weights(r["w"], uv).items()}
    A = [a[:B].double() for a in r["acts"]]
    inputs = _wgrad_inputs(A, uv)
    ray = torch.arange(B, device=DEV) // S
    rc = r["rc"].double()
    worst = 0.0
    for i, g in enumerate(GEMMS):
        t, Bs = preact(g, inputs[g], kw, rc, ray)
        d = 2.0 ** -23 * kw[g][0].shape[1] * Bs
        got = A[i + 1][:, :N_OUT[g]]
        q = gate_share(t, d, got, tc_epilogue(g))
        worst = max(worst, q.max().item())
        assert (q <= 1).all(), (label, g, f"{int((q > 1).sum())} outputs outside the gate, worst share {q.max().item():.3g}")
        if i + 1 in MASK_WORD0:
            neg = (got < 0).double().mean().item()
            pos = (got > 0).double().mean().item()
            assert neg >= 0.05 and pos >= 0.05, (label, g, neg, pos)
    _report(f"layers {label}", worst)


def check_masks(r, label):
    """Sign masks: bit b of mask word w of a row = the dumped bf16 at column w CPW + b is non-negative (CPW = 32, 16 for
    the 64-wide layer), for every mask word of every row of every tile."""
    T = r["T"]
    nt = T["n_tiles"]
    words = helpers.read_masks(r["ws"], T)
    for slot, w0 in MASK_WORD0.items():
        N = N_OUT[GEMMS[slot - 1]]
        cpw = 32 if N >= 128 else 16
        nonneg = ~torch.signbit(r["acts"][slot][:, :N])
        bits = nonneg.view(nt, 128, N // cpw, cpw).long() << torch.arange(cpw, device=DEV)
        want = bits.sum(-1).permute(0, 2, 1)
        got = words[:, w0:w0 + N // cpw]
        assert torch.equal(got, want), (label, slot, int((got != want).sum()))


def check_dead_rows(r, label):
    """Rows past n_samples of the last tile are finite in every slot (the weight-gradient GEMM multiplies them by zero
    dZ); with the 0xFF fill, an unwritten row would be NaN."""
    for s, a in enumerate(r["acts"]):
        assert torch.isfinite(a[r["B"]:]).all(), (label, s)


def check_heads(r, label):
    """sigma / rgb against float64 recomputed from the dumped inputs of the sigma layers (S7 / O3) and dir layers
    (SDIR / ODIR, with ray_const): the head weights' share of the layer gate plus 2^-20 of sum |w h|; rgb on the
    pre-sigmoid value, scaled by 1/4, plus 2^-20 for __expf.  The rigorous gate is loose against rounding the head's
    input to bf16 (2^-9 relative per term), so the RMS error must also be below a quarter of that alternative's."""
    uv, B, S = r["use_voxel"], r["B"], r["S"]
    kw = {g: (W.to(DEV), b.to(DEV)) for g, (W, b) in kernel_weights(r["w"], uv).items()}
    A = [a[:B].double() for a in r["acts"]]
    inputs = _wgrad_inputs(A, uv)
    ray = torch.arange(B, device=DEV) // S
    rc = r["rc"].double()
    rms = lambda x: x.pow(2).mean().sqrt().item()
    worst = 0.0
    for layers, col in ((SIGMA_LAYER, 3), (DIR_LAYER, slice(0, 3))):
        for g, (name, br) in layers.items():
            t, Bs = preact(g, inputs[g], kw, rc, ray)
            d = 2.0 ** -23 * kw[g][0].shape[1] * Bs
            hw, hb = r["w"][name][0].double().to(DEV), r["w"][name][1].double().to(DEV)
            h = torch.where(t > 0, t, 0.01 * t)
            pre = h @ hw.t() + hb
            gate = d @ hw.abs().t() + 2.0 ** -20 * (h.abs() @ hw.abs().t() + hb.abs())
            alt = A[GEMMS.index(g) + 1][:, :hw.shape[1]] @ hw.t() + hb
            got = (r["obj"] if br else r["scene"]).reshape(B, 4)[:, col].double().reshape(B, -1)
            if col == 3:
                want = pre
            else:
                want, gate, alt = torch.sigmoid(pre), gate / 4 + 2.0 ** -20, torch.sigmoid(alt)
            ratio = ((got - want).abs() / gate).max().item()
            worst = max(worst, ratio)
            assert ratio <= 1, (label, name, ratio)
            assert rms(got - want) <= 0.25 * rms(alt - want), (label, name, rms(got - want), rms(alt - want))
    _report(f"heads {label}", worst)


STAGES = {"x": check_x, "layers": check_layers, "masks": check_masks, "dead_rows": check_dead_rows, "heads": check_heads}


def _check_all(r, label):
    for f in STAGES.values():
        f(r, label)


@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("stage", list(STAGES))
def test_tc_forward_stage(model, shape, stage):
    r = _stage_run(model, shape)
    out = STAGES[stage](r, f"{model} {shape}")
    if stage == "x" and shape == "big_features" and model == "voxel":
        assert out[0].abs().max().item() > 6.0


# ------------------------------------------------------------------------------------------------
# ray_const
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("n_rays", [1, 7, 9, 1001])
@pytest.mark.parametrize("codes_kind", ["per_ray", "code_row", "no_object"])
def test_ray_const_matches_float64(model, n_rays, codes_kind):
    """ray_const read back from the launch's buffer (rows past n_rays of an oversized NaN-filled buffer stay NaN)
    against float64; with want_object = 0 the OL0 / OL2 entries are the biases exactly."""
    c = _case_inputs(MODELS[model], "few_tiles")
    gen = torch.Generator(device=DEV).manual_seed(n_rays)
    rays = torch.cat([torch.randn(n_rays, 3, device=DEV, generator=gen),
                      torch.nn.functional.normalize(torch.randn(n_rays, 3, device=DEV, generator=gen), dim=1),
                      torch.tensor([[0.1, 3.0]], device=DEV).expand(n_rays, 2)], 1).contiguous()
    z = torch.full((n_rays, 2), 1.0, device=DEV)
    code_tab = torch.randn(n_rays, 64, device=DEV, generator=gen)
    rc = torch.full((n_rays + 5, 448), float("nan"), device=DEV)
    want_object = codes_kind != "no_object"
    kw = dict(codes=code_tab if codes_kind == "per_ray" else None,
              code_row=code_tab[0].contiguous() if codes_kind == "code_row" else None)
    _launch(c["packed"], c["grid"], rays, z, 2, want_object=int(want_object), rc=rc, **kw)
    torch.cuda.synchronize()
    codes = code_tab if codes_kind == "per_ray" else code_tab[:1].expand(n_rays, 64)
    ref, gate = ray_const_ref(rays, codes, c["w"], MODELS[model], want_object)
    got = rc[:n_rays].double()
    ratio = ((got - ref).abs() / gate).max().item()
    _report(f"ray_const {model} n={n_rays} {codes_kind}", ratio)
    assert ratio <= 1
    assert torch.isnan(rc[n_rays:]).all()
    if not want_object:
        for name, c0 in (("obj.l0", 192), ("obj.l2", 320)):
            assert torch.equal(rc[:n_rays, c0:c0 + 128], c["w"][name][1].to(DEV).expand(n_rays, 128)), name


# ------------------------------------------------------------------------------------------------
# inference modes against launches whose stages are verified
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", list(MODELS))
def test_inference_modes_bit_identical_to_verified_launches(model):
    """77 x 63 rays, every fifth ray with a zero last depth, stage-checked through the training dump; then each
    inference mode against it: the inference launch, object-only and scene-only launches, mute_zero_rays with two
    removed-object boxes (muted set = fp32 emulation of point_in_boxes), strided z / outputs, and the explicit-xyz path
    against an S = 1 launch (also stage-checked) with o = xyz and d = 0."""
    c = _case_inputs(MODELS[model], "partial_straddle")
    n, S = c["n"], c["S"]
    c["z"] = c["z"].clone()
    c["z"][::5, -1] = 0.0
    r = _dump_run(c)
    _check_all(r, f"{model} modes")
    P, G = c["packed"], c["grid"]
    args = (P, G, c["rays"], c["z"], S)
    scene, obj, rc = _launch(*args, codes=c["codes"])
    s_only, _, _ = _launch(*args, want_object=0)
    _, o_only, _ = _launch(*args, codes=c["codes"], want_scene=0)
    torch.cuda.synchronize()
    assert torch.equal(scene, r["scene"]) and torch.equal(obj, r["obj"]) and torch.equal(rc, r["rc"])
    assert torch.equal(s_only, scene) and torch.equal(o_only, obj)
    # muting
    x32 = positions(c["rays"], c["z"], fused=True)
    mid = x32[:, 0].median().item()
    ang = 0.7
    A = torch.tensor([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]], dtype=torch.float32)
    ctr = x32[len(x32) // 3].cpu()
    boxes = torch.stack([
        torch.cat([torch.eye(3).reshape(-1), torch.zeros(3), torch.tensor([-1e9, -1e9, -1e9, mid, 1e9, 1e9])]),
        torch.cat([A.reshape(-1), -(A @ ctr), torch.full((3,), -0.3), torch.full((3,), 0.3)])]).to(DEV).contiguous()
    ms, mo, _ = _launch(*args, codes=c["codes"], mute=1, boxes=boxes)
    torch.cuda.synchronize()
    zero_ray = (c["z"][:, -1] == 0).repeat_interleave(S)
    in_box = point_in_boxes32(x32, boxes) & ~zero_ray
    assert zero_ray.any() and in_box.any() and not (zero_ray | in_box).all()
    for got, base, muted in ((ms, scene, zero_ray | in_box), (mo, obj, zero_ray)):
        got, base = got.reshape(-1, 4), base.reshape(-1, 4)
        assert torch.equal(got[:, :3], base[:, :3])
        assert torch.equal(got[:, 3] == -1e5, muted)
        assert torch.equal(got[~muted, 3], base[~muted, 3])
    # strides: z and outputs as column blocks of wider arrays; the sentinel columns stay NaN
    zw = torch.full((n, S + 3), 1e30, device=DEV)
    zw[:, :S] = c["z"]
    outs = (torch.full((n, S + 2, 4), float("nan"), device=DEV), torch.full((n, S + 2, 4), float("nan"), device=DEV))
    _launch(P, G, c["rays"], zw, S, codes=c["codes"], z_stride=S + 3, outs=outs, out_stride=S + 2)
    torch.cuda.synchronize()
    for o, base in zip(outs, (scene, obj)):
        assert torch.equal(o[:, :S], base) and torch.isnan(o[:, S:]).all()
    # explicit xyz (rays with d = 0) against S = 1 rays at o = xyz, d = 0
    rays0 = c["rays"].clone()
    rays0[:, 3:6] = 0.0
    rays0[:, :3] = 100.0
    xs, xo, _ = _launch(P, G, rays0, c["z"], S, codes=c["codes"], xyz=x32.view(n, S, 3).contiguous())
    rays1 = torch.zeros(n * S, 8, device=DEV)
    rays1[:, :3] = x32
    rays1[:, 6:] = torch.tensor([0.1, 3.0], device=DEV)
    c1 = dict(c, rays=rays1, z=torch.full((n * S, 1), 0.5, device=DEV), codes=c["codes"].repeat_interleave(S, 0),
              n=n * S, S=1)
    r1 = _dump_run(c1)
    _check_all(r1, f"{model} xyz as S=1 rays")
    torch.cuda.synchronize()
    assert torch.equal(xs.reshape(-1, 4), r1["scene"].reshape(-1, 4))
    assert torch.equal(xo.reshape(-1, 4), r1["obj"].reshape(-1, 4))


# ------------------------------------------------------------------------------------------------
# the FFMA kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("shape", ["few_tiles", "partial_straddle", "s1"])
def test_ffma_forward_stages(model, shape):
    """The fp32 kernel's activation dump: X against the float64 encoding of its positions fl(o + fl(d z)) (identity
    columns exact, sinf / cosf within 2 ulp), every layer on its dumped fp32 input with c = 2^-24 over K + 2 terms, the
    heads within 2^-24 (K + 1) sum |terms| (rgb: 1/4 of that plus 2^-20 for expf)."""
    c = _case_inputs(MODELS[model], shape)
    uv, B, S = c["use_voxel"], c["n"] * c["S"], c["S"]
    KO = 384 if uv else 64
    acts = [torch.empty(B, KO, device=DEV)] + [torch.empty(B, N_OUT[g], device=DEV) for g in GEMMS]
    ptrs = (C.c_void_p * 17)(*[t.data_ptr() for t in acts])
    scene, obj, rc = _launch(c["packed"], c["grid"], c["rays"], c["z"], S, codes=c["codes"],
                             precision=_lib().PREC_FP32, activations=ptrs)
    torch.cuda.synchronize()
    label = f"ffma {model} {shape}"
    x32 = positions(c["rays"], c["z"], fused=False)
    ref, e = x_reference_ffma(x32, voxel_features32(x32, c["g"]) if uv else None, uv)
    err = (acts[0].double() - ref).abs()
    _report(f"X {label}", (err / e.clamp(min=1e-300)).max().item())
    assert (err <= e).all(), (label, "X", (err > e).nonzero()[:, 1].unique().tolist()[:20])
    kw = {g: (W.to(DEV), b.to(DEV)) for g, (W, b) in kernel_weights(c["w"], uv, bf16=False).items()}
    A = [a.double() for a in acts]
    inputs = _wgrad_inputs(A, uv)
    ray = torch.arange(B, device=DEV) // S
    worst = 0.0
    for i, g in enumerate(GEMMS):
        t, Bs = preact(g, inputs[g], kw, rc.double(), ray)
        q = gate_share(t, 2.0 ** -24 * (kw[g][0].shape[1] + 2) * Bs, A[i + 1], ffma_epilogue(g))
        worst = max(worst, q.max().item())
        assert (q <= 1).all(), (label, g, q.max().item())
    _report(f"layers {label}", worst)
    worst = 0.0
    for layers, col in ((SIGMA_LAYER, 3), (DIR_LAYER, slice(0, 3))):
        for g, (name, br) in layers.items():
            h = A[GEMMS.index(g) + 1]
            hw, hb = c["w"][name][0].double().to(DEV), c["w"][name][1].double().to(DEV)
            pre = h @ hw.t() + hb
            gate = 2.0 ** -24 * (hw.shape[1] + 1) * (h.abs() @ hw.abs().t() + hb.abs())
            got = (obj if br else scene).reshape(B, 4)[:, col].double().reshape(B, -1)
            want = pre if col == 3 else torch.sigmoid(pre)
            if col != 3:
                gate = gate / 4 + 2.0 ** -20
            ratio = ((got - want).abs() / gate).max().item()
            worst = max(worst, ratio)
            assert ratio <= 1, (label, name, ratio)
    _report(f"heads {label}", worst)
