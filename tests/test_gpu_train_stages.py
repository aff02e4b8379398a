"""The tensor-core training backward (onerf_render_rays_bwd, csrc/bwd_api.cu) stage by stage through the C stage entry
points, against float64 references of the same operation on the same bf16-rounded operands the kernels read:
voxel-table gradient (onerf_bwd_dx, onerf_encode_bwd), head / bias column sums (onerf_bwd_colsums, the GEMM bias
gradients of onerf_bwd_wgrad), per-ray sums (onerf_bwd_raysums), the chain and wgrad at want_object = 0 and on ragged
batches, the compositing backward in every mode, the seeded (Philox) noise path, and whole training steps the other
files do not run.  The references themselves are checked in tests/test_train_stages_cpu.py."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

from tests import cases, helpers, synth
from tests.test_gpu_train_plain import _torch_chain as _chain_plain
from tests.test_gpu_train_tc import GEMM_K, GEMM_N, GEMM_OF_DZ, _torch_chain as _chain_voxel, grad_layout
from tests.test_fp32_backward_cpu import ORACLE_TWO_CHUNKS
from tests.test_train_stages_cpu import (DX_LAYERS, dx_from_dz, edge_points, grid_coords, philox_normal, philox_uniform,
                                         table_grad_autograd, table_grad_matched)
from oracle import onerf_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WIDTHS = {1: [384] + [256] * 8 + [256, 128] + [128] * 4 + [128, 64], 0: [64] + [256] * 8 + [256, 128] + [128] * 4 + [128, 64]}
GEMM_K_PLAIN = dict(GEMM_K, S0=64, S4=320, O0=64, O2=192)
OBJ_DZ_SLOTS = range(10, 16)
# a grid whose voxel size and offset are exact binary fractions: points on a voxel face have u = 0 exactly in fp32
GRID = dict(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.0625)


def _lib():
    from object_nerf_b200 import _lib
    return _lib


def _ctx():
    return _lib().ctx(torch.device(DEV))


def bf(t):
    return t.to(torch.bfloat16).float()


def _grad_offsets(use_voxel):
    """Kernel-layout gradient buffer (layout.h GradLayout): per GEMM (w, b) offsets and the head offsets."""
    Kd = GEMM_K if use_voxel else GEMM_K_PLAIN
    off, w_off, b_off = 0, {}, {}
    for g in GEMM_OF_DZ:
        w_off[g] = off
        off += GEMM_N[g] * Kd[g]
        b_off[g] = off
        off = (off + GEMM_N[g] + 3) // 4 * 4
    heads = {}
    for name, n in (("sigma_w", 256), ("sigma_b", 1), ("rgb_w", 384), ("rgb_b", 3), ("osigma_w", 128), ("osigma_b", 1),
                    ("orgb_w", 192), ("orgb_b", 3)):
        heads[name] = off
        off += (n + 3) // 4 * 4
    assert _lib().load().onerf_grad_buffer_floats(use_voxel) == off
    if use_voxel:
        assert (w_off, b_off, heads, off) == grad_layout()
    return Kd, w_off, b_off, heads, off


def _train_forward(rays, z, packed, grid, codes, use_voxel, want_object, fill=0, outputs=False):
    """onerf_field_fwd with a training workspace -> (ws, layout), and with outputs=True also the scene / object field
    outputs and the ray_const buffer."""
    L = _lib()
    n, S = z.shape
    T = helpers.train_layout(bool(use_voxel), n * S)
    ws = helpers.aligned_u8(T["total"], DEV, fill=fill)
    a = L.FieldArgs()
    scene = torch.empty(n, S, 4, device=DEV)
    obj = torch.empty(n, S, 4, device=DEV)
    rc = torch.empty(n, 448, device=DEV)
    a.rays, a.z, a.z_stride, a.codes = rays.data_ptr(), z.data_ptr(), S, codes.data_ptr()
    a.n_rays, a.n_samples = n, S
    a.grid = C.pointer(grid.c) if grid is not None else None
    a.packed = packed.data_ptr()
    a.want_scene, a.want_object, a.precision = 1, int(want_object), L.PREC_BF16
    a.scene_out, a.obj_out, a.out_stride, a.ray_const = scene.data_ptr(), obj.data_ptr() if want_object else None, S, rc.data_ptr()
    a.train_ws = ws.data_ptr()
    L.check(L.load().onerf_field_fwd(_ctx(), C.byref(a), L.stream()))
    if outputs:
        return ws, T, scene, obj if want_object else None, rc
    return ws, T


def _edge_rays(g, n, S, rng):
    """Axis-aligned rays (o = 0 on the ray's axis, d a unit axis) whose samples land on the cases of edge_points: the
    positions o + d z are exact in fp32, fused or not.  The last quarter repeats ray 0: heavy atomic contention."""
    shape = g["shape"].numpy()
    vs, off = float(g["voxel_size"]), g["offset"].double().numpy()
    pool = edge_points(shape, 5 * max(S, 64), rng).astype(np.float64)
    rays = torch.zeros(n, 8)
    z = torch.zeros(n, S)
    for r in range(n):
        a = r % 3
        o = pool[rng.integers(len(pool))] * vs - off
        o[a] = 0.0
        rays[r, :3] = torch.from_numpy(o)
        rays[r, 3 + a] = 1.0
        rays[r, 6:8] = torch.tensor([0.1, 3.0])
        z[r] = torch.from_numpy(pool[rng.integers(len(pool), size=S), a] * vs - off[a])
    k = n - n // 4
    rays[k:], z[k:] = rays[:1], z[:1]
    return rays, z


def _dx_inputs(n_rays, S, want_object, seed):
    from object_nerf_b200 import engine
    rng = np.random.default_rng(seed)
    inp = cases.build_render_case(dict(cases.RENDER_CASES["eval_voxel"], n_rays=n_rays))
    g = synth.make_grid(**GRID)
    rays = inp["rays"].clone()
    z = engine.sample_coarse(rays.to(DEV), S).cpu()
    if S == 1:
        z[:] = 1.6          # the one sample near the middle of the grid
    n_edge = n_rays // 2
    if n_edge:
        rays[:n_edge], z[:n_edge] = _edge_rays(g, n_edge, S, rng)
    model = helpers.make_model(inp["weights"]["coarse"], True, DEV)
    grid = engine.GridBuffers.from_module(helpers.GridModule(g).to(DEV))
    rays_d, z_d = rays.to(DEV).contiguous(), z.to(DEV).contiguous()
    packed = engine.packed_for(model, True)
    ws, T = _train_forward(rays_d, z_d, packed, grid, inp["codes"].to(DEV), 1, want_object)
    return inp["weights"]["coarse"], g, rays, z, rays_d, z_d, packed, grid, ws, T


def _report(label, err, scale):
    r = (err / scale).max().item()
    print(f"{label}: max error / tolerance scale = {r:.3e}")
    return r


# ------------------------------------------------------------------------------------------------
# 1. voxel-table gradient
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_rays,S,want_object", [(1, 1, 1), (37, 61, 0), (37, 61, 1), (301, 128, 1)])
def test_bwd_dx_matches_float64_references(n_rays, S, want_object):
    """onerf_bwd_dx on the real training dump: dX = sum dZ W[:, X block] (wgmma), the PE chain rule on the dumped bf16
    sin / cos and the trilinear red.global.add scatter, added to a pre-filled table gradient.
    Matched reference (same bf16 operands, same fp32 corner weights): |err| <= 2e-4 (B + |prefill|), B the same
    computation over absolute values.  Semantic reference (float64 autograd of voxel_embed, unrounded weights): the
    bf16 rounding of W and of sin / cos is <= 2^-9 relative each, so |err| <= 2^-8 B' + the matched gate, B' with
    2^-6 of slack on every sin / cos for the fp32 feature and the __sincosf / double-angle error."""
    L = _lib()
    w, g, rays, z, rays_d, z_d, packed, grid, ws, T = _dx_inputs(n_rays, S, want_object, seed=n_rays * 1000 + S)
    B, n_tiles = n_rays * S, T["n_tiles"]
    gen = torch.Generator(device=DEV).manual_seed(7 + want_object)
    dz = {}
    for name, slot, _, width in DX_LAYERS:     # rows past B stay random: the kernel must not scatter them
        m = torch.randn(n_tiles * 128, 64 * T["dz_atoms"][slot], device=DEV, generator=gen)
        helpers.write_atoms(ws, T["dz_off"][slot], m)
        dz[name] = bf(m[:B, :width]).double().cpu()
    n_rows = g["table"].shape[0]
    prefill = torch.randn(n_rows, 24, device=DEV, generator=gen)
    tg = prefill.clone()
    L.check(L.load().onerf_bwd_dx(_ctx(), want_object, packed.data_ptr(), ws.data_ptr(), rays_d.data_ptr(), z_d.data_ptr(),
                                  n_rays, S, C.byref(grid.c), tg.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    got = (tg.double() - prefill.double()).cpu()
    X = helpers.from_atoms(ws, T["act_off"][0], n_tiles, 6)[:B].double().cpu()
    p = grid_coords(rays, z, g["offset"], g["voxel_size"], fused=True)
    w_bf = {k: (v[0].to(torch.bfloat16).double(), v[1]) for k, v in w.items()}
    w_abs = {k: (v[0].abs(), v[1]) for k, v in w_bf.items()}
    dz_abs = {k: v.abs() for k, v in dz.items()}
    want = table_grad_matched(dx_from_dz(dz, w_bf, want_object), X, p, g["idx_map"], n_rows, want_object)
    bound = table_grad_matched(dx_from_dz(dz_abs, w_abs, want_object), X.abs() + 2 ** -6, p, g["idx_map"], n_rows,
                               want_object, bound=True)
    assert want.abs().max() > 0
    tol = 2e-4 * (bound + prefill.double().abs().cpu()) + 1e-6
    _report(f"bwd_dx matched {n_rays}x{S} obj={want_object}", (got - want).abs(), tol)
    assert ((got - want).abs() <= tol).all(), (got - want).abs().max().item()
    sem = table_grad_autograd(dx_from_dz(dz, w, want_object), p, g["idx_map"], g["table"], want_object)
    tol_sem = 2 ** -8 * bound + tol
    _report(f"bwd_dx semantic {n_rays}x{S} obj={want_object}", (got - sem).abs(), tol_sem)
    assert ((got - sem).abs() <= tol_sem).all(), (got - sem).abs().max().item()
    if not want_object:
        assert torch.equal(tg[:, 16:], prefill[:, 16:])


def test_encode_bwd_matches_float64_references():
    """onerf_encode_bwd (the fp32 path's encoding backward) fed an fp32 X (the dumped one) and a random fp32 dX, in two
    chunks (sample0 = 0 and sample0 > 0) into one pre-filled table gradient; positions by multiply-then-add."""
    L = _lib()
    n_rays, S = 37, 61
    w, g, rays, z, rays_d, z_d, packed, grid, ws, T = _dx_inputs(n_rays, S, 1, seed=5)
    B = n_rays * S
    X = helpers.from_atoms(ws, T["act_off"][0], T["n_tiles"], 6)[:B].contiguous()
    gen = torch.Generator(device=DEV).manual_seed(3)
    dX = torch.randn(B, 384, device=DEV, generator=gen)
    n_rows = g["table"].shape[0]
    prefill = torch.randn(n_rows, 24, device=DEV, generator=gen)
    tg = prefill.clone()
    cut = 1000
    for s0, s1 in ((0, cut), (cut, B)):
        L.check(L.load().onerf_encode_bwd(_ctx(), C.byref(grid.c), rays_d.data_ptr(), z_d.data_ptr(), n_rays, S,
                                          X[s0:].data_ptr(), dX[s0:].data_ptr(), 384, s0, s1 - s0, tg.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    got = (tg.double() - prefill.double()).cpu()
    Xc, dXc = X.double().cpu(), dX.double().cpu()
    p = grid_coords(rays, z, g["offset"], g["voxel_size"], fused=False)
    want = table_grad_matched(dXc, Xc, p, g["idx_map"], n_rows, 1)
    bound = table_grad_matched(dXc.abs(), Xc.abs() + 2 ** -6, p, g["idx_map"], n_rows, 1, bound=True)
    tol = 2e-4 * (bound + prefill.double().abs().cpu()) + 1e-6
    _report("encode_bwd matched", (got - want).abs(), tol)
    assert ((got - want).abs() <= tol).all(), (got - want).abs().max().item()
    sem = table_grad_autograd(dXc, p, g["idx_map"], g["table"], 1)
    tol_sem = 2 ** -8 * bound + tol       # the sin / cos in X are bf16
    _report("encode_bwd semantic", (got - sem).abs(), tol_sem)
    assert ((got - sem).abs() <= tol_sem).all(), (got - sem).abs().max().item()


# ------------------------------------------------------------------------------------------------
# 2. head and bias column sums
# ------------------------------------------------------------------------------------------------
def _wgrad_inputs(acts, use_voxel):
    """Input block of every GEMM in kernel-K order from the activation slots (slot 0 = X): the X-fed layers read
    X[0, KX) (scene) / X[0, KO) (object), the skip layers S4 / O2 then the previous hidden layer, every other layer its
    one input slot."""
    X = acts[0]
    kx, ko = (288, 384) if use_voxel else (64, 64)
    inputs = {"S0": X[:, :kx], "S4": torch.cat([X[:, :kx], acts[4]], 1), "O0": X[:, :ko],
              "O2": torch.cat([X[:, :ko], acts[12]], 1), "SFIN": acts[8], "SDIR": acts[9], "O1": acts[11],
              "O3": acts[13], "OFIN": acts[14], "ODIR": acts[15]}
    inputs.update({f"S{l}": acts[l] for l in (1, 2, 3, 5, 6, 7)})
    return inputs


def _random_atoms(ws, T, slots, kind, B, gen, garbage=None):
    """Random bf16 atoms into activation (kind = "act") or dZ slots; rows past B set to `garbage` (None: random too).
    Returns {slot: (B, 64 atoms) float64 of the bf16 values}."""
    out = {}
    for s in slots:
        atoms = T[f"{kind}_atoms"][s]
        m = torch.randn(T["n_tiles"] * 128, 64 * atoms, device=DEV, generator=gen)
        if garbage is not None:
            m[B:] = garbage
        helpers.write_atoms(ws, T[f"{kind}_off"][s], m)
        out[s] = bf(m[:B]).double().cpu()
    return out


@pytest.mark.parametrize("use_voxel", [1, 0])
@pytest.mark.parametrize("want_object", [0, 1])
@pytest.mark.parametrize("n_samples", [128 * 19, 37 * 61])
def test_bwd_colsums_match_float64(use_voxel, want_object, n_samples):
    """onerf_bwd_colsums: sigma / rgb head weights (sum_s dA H) and the four head biases (sum_s dA) of both branches,
    against float64 sums; padding rows of the activation atoms hold large finite garbage.  |err| <= 1e-4 sum |terms|;
    at want_object = 0 the object heads keep their pre-filled values."""
    L = _lib()
    B = n_samples
    T = helpers.train_layout(bool(use_voxel), B)
    ws = helpers.aligned_u8(T["total"], DEV, fill=0)
    gen = torch.Generator(device=DEV).manual_seed(11)
    H = _random_atoms(ws, T, (8, 10, 14, 16), "act", B, gen, garbage=1e30)
    dA_s = torch.randn(B, 4, device=DEV, generator=gen)
    dA_o = torch.randn(B, 4, device=DEV, generator=gen)
    _, _, _, heads, total = _grad_offsets(use_voxel)
    prefill = torch.randn(total, device=DEV, generator=gen)
    grad = prefill.clone()
    L.check(L.load().onerf_bwd_colsums(_ctx(), use_voxel, want_object, ws.data_ptr(), B, dA_s.data_ptr(),
                                       dA_o.data_ptr() if want_object else None, grad.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    got = (grad.double() - prefill.double()).cpu()
    ds, do = dA_s.double().cpu(), dA_o.double().cpu()
    refs = {"sigma_w": (ds[:, 3:4], H[8]), "rgb_w": (ds[:, :3], H[10]), "sigma_b": (ds[:, 3:4], None),
            "rgb_b": (ds[:, :3], None), "osigma_w": (do[:, 3:4], H[14]), "orgb_w": (do[:, :3], H[16]),
            "osigma_b": (do[:, 3:4], None), "orgb_b": (do[:, :3], None)}
    for name, (d, h) in refs.items():
        h = torch.ones(B, 1, dtype=torch.float64) if h is None else h
        want = (d.t() @ h).reshape(-1)
        bound = (d.abs().t() @ h.abs()).reshape(-1)
        o = heads[name]
        if name.startswith("o") and not want_object:
            assert torch.equal(grad[o:o + want.numel()], prefill[o:o + want.numel()]), name
            continue
        err = (got[o:o + want.numel()] - want).abs()
        _report(f"colsums {name} voxel={use_voxel} obj={want_object} B={B}", err, 1e-4 * bound + 1e-6)
        assert (err <= 1e-4 * bound + 1e-6).all(), (name, err.max().item())


@pytest.mark.parametrize("want_object", [0, 1])
def test_wgrad_bias_gradients_and_scene_only_regions(want_object):
    """onerf_bwd_wgrad (voxel layout) on a ragged batch: the GEMM bias gradients db = sum_s dZ it forms from the dZ atoms
    (the padding rows are zero, as the chain leaves them; the activation padding rows hold large finite garbage) and
    the weight gradients, against float64; at want_object = 0 the object layers' regions keep their pre-filled
    values."""
    L = _lib()
    B = 37 * 61
    T = helpers.train_layout(True, B)
    ws = helpers.aligned_u8(T["total"], DEV, fill=0)
    gen = torch.Generator(device=DEV).manual_seed(12)
    acts = _random_atoms(ws, T, range(17), "act", B, gen, garbage=1e30)
    dzs = _random_atoms(ws, T, range(16), "dz", B, gen, garbage=0.0)
    Kd, w_off, b_off, heads, total = _grad_offsets(1)
    prefill = torch.randn(total, device=DEV, generator=gen)
    grad = prefill.clone()
    L.check(L.load().onerf_bwd_wgrad(_ctx(), 1, want_object, ws.data_ptr(), B, grad.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    assert torch.isfinite(grad).all()
    got = (grad.double() - prefill.double()).cpu()
    inputs = _wgrad_inputs(acts, 1)
    for d, gname in enumerate(GEMM_OF_DZ):
        N, K = GEMM_N[gname], Kd[gname]
        region = slice(w_off[gname], b_off[gname] + N)
        if gname.startswith("O") and not want_object:
            assert torch.equal(grad[region], prefill[region]), gname
            continue
        dz = dzs[d][:, :N]
        db_want, db_bound = dz.sum(0), dz.abs().sum(0)
        db_err = (got[b_off[gname]:b_off[gname] + N] - db_want).abs()
        _report(f"wgrad db {gname} obj={want_object}", db_err, 1e-4 * db_bound + 1e-6)
        assert (db_err <= 1e-4 * db_bound + 1e-6).all(), (gname, db_err.max().item())
        dw_want = dz.t() @ inputs[gname]
        dw_bound = dz.abs().t() @ inputs[gname].abs()
        dw_err = (got[w_off[gname]:w_off[gname] + N * K].view(N, K) - dw_want).abs()
        assert (dw_err <= 1e-4 * dw_bound + 1e-6).all(), (gname, dw_err.max().item())
    # the heads belong to onerf_bwd_colsums
    assert torch.equal(grad[heads["sigma_w"]:], prefill[heads["sigma_w"]:])


# ------------------------------------------------------------------------------------------------
# 3. per-ray sums
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_voxel", [1, 0])
@pytest.mark.parametrize("want_object", [0, 1])
@pytest.mark.parametrize("S", [1, 61, 128, 200])
def test_bwd_raysums_match_float64(use_voxel, want_object, S):
    """onerf_bwd_raysums over 37 rays (rays straddle tiles): per-ray sums of the bf16 dZ atoms of the scene dir layer,
    object dir layer, object layers 0 and 2 into RC_SDIR / RC_ODIR / RC_OL0 / RC_OL2 (layout.h); |err| <= 1e-5 sum |x|.
    At want_object = 0 columns 128-447 keep their sentinel."""
    L = _lib()
    n = 37
    B = n * S
    T = helpers.train_layout(bool(use_voxel), B)
    ws = helpers.aligned_u8(T["total"], DEV, fill=0)
    gen = torch.Generator(device=DEV).manual_seed(S)
    dz = _random_atoms(ws, T, (9, 10, 12, 15), "dz", B, gen)
    out = torch.full((n, 448), -7.25, device=DEV)
    L.check(L.load().onerf_bwd_raysums(_ctx(), use_voxel, want_object, ws.data_ptr(), n, S, out.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    got = out.double().cpu()
    cols = [(9, 0, 128)] + ([(15, 128, 64), (10, 192, 128), (12, 320, 128)] if want_object else [])
    for slot, c0, width in cols:
        x = dz[slot][:, :width].reshape(n, S, width)
        want, bound = x.sum(1), x.abs().sum(1)
        err = (got[:, c0:c0 + width] - want).abs()
        _report(f"raysums slot {slot} voxel={use_voxel} S={S}", err, 1e-5 * bound + 1e-6)
        assert (err <= 1e-5 * bound + 1e-6).all(), (slot, err.max().item())
    if not want_object:
        assert (out[:, 128:] == -7.25).all()


# ------------------------------------------------------------------------------------------------
# 4. chain and wgrad at want_object = 0 and on ragged batches
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_voxel", [1, 0])
@pytest.mark.parametrize("want_object", [0, 1])
def test_chain_and_wgrad_scene_only_and_ragged(use_voxel, want_object):
    """37 rays x 61 samples (a partial last tile) on a workspace filled with 0xFF (bf16 NaN) before the forward:
    the chain's scene dZ against the fp32 reference of the existing chain tests; every dZ row past n_samples exactly
    zero (wgrad reduces over whole 64-sample stages); at want_object = 0 the object dZ slots keep their poison bytes and
    wgrad leaves the object regions of the gradient buffer alone; wgrad's output finite and equal to float64 dZ^T In
    over the valid rows."""
    from object_nerf_b200 import engine
    L = _lib()
    case = "eval_voxel" if use_voxel else "eval_plain"
    n, S = 37, 61
    inp = cases.build_render_case(dict(cases.RENDER_CASES[case], n_rays=n))
    model = helpers.make_model(inp["weights"]["coarse"], bool(use_voxel), DEV)
    rays = inp["rays"].to(DEV)
    z = engine.sample_coarse(rays, S)
    packed = engine.packed_for(model, bool(use_voxel))
    grid = engine.GridBuffers.from_module(helpers.GridModule(inp["grid"]).to(DEV)) if use_voxel else None
    ws, T = _train_forward(rays, z, packed, grid, inp["codes"].to(DEV), use_voxel, want_object, fill=0xFF)
    B, nt = n * S, T["n_tiles"]
    if not want_object:
        for s in OBJ_DZ_SLOTS:
            ws[T["dz_off"][s]:T["dz_off"][s] + T["dz_atoms"][s] * nt * helpers.ATOM_BYTES] = 0x5A
    g = torch.Generator(device=DEV).manual_seed(1)
    dA_s = torch.randn(B, 4, device=DEV, generator=g)
    dA_o = torch.randn(B, 4, device=DEV, generator=g)
    L.check(L.load().onerf_bwd_chain(_ctx(), use_voxel, want_object, packed.data_ptr(), ws.data_ptr(), B, dA_s.data_ptr(),
                                     dA_o.data_ptr() if want_object else None, L.stream()))
    torch.cuda.synchronize()
    W = WIDTHS[use_voxel]
    acts = [helpers.from_atoms(ws, T["act_off"][s], nt, T["act_atoms"][s]) for s in range(17)]
    chain = _chain_voxel if use_voxel else _chain_plain
    want = chain([a[:B, :W[s]] for s, a in enumerate(acts)], inp["weights"]["coarse"], dA_s,
                 dA_o if want_object else torch.zeros_like(dA_o))
    dzs = []
    for d, gname in enumerate(GEMM_OF_DZ):
        full = helpers.from_atoms(ws, T["dz_off"][d], nt, T["dz_atoms"][d])
        dzs.append(full)
        if d in OBJ_DZ_SLOTS and not want_object:
            raw = ws[T["dz_off"][d]:T["dz_off"][d] + T["dz_atoms"][d] * nt * helpers.ATOM_BYTES]
            assert (raw == 0x5A).all(), gname
            continue
        assert (full[B:] == 0).all(), (gname, "padding rows of dZ not zero")
        got, ref = full[:B, :GEMM_N[gname]], want[gname]
        scale = ref.abs().mean().item() + 1e-12
        err = (got - ref).abs()
        assert err.mean().item() <= 2e-2 * scale, (gname, err.mean().item(), scale)
        assert (err > 0.25 * scale + 0.05 * ref.abs()).float().mean().item() < 5e-3, (gname, err.max().item(), scale)
    # weight gradients over the same workspace: the padding rows (zero dZ, whatever activations) contribute nothing
    Kd, w_off, b_off, heads, total = _grad_offsets(use_voxel)
    prefill = torch.full((total,), 3.5, device=DEV)
    grad = prefill.clone()
    L.check(L.load().onerf_bwd_wgrad(_ctx(), use_voxel, want_object, ws.data_ptr(), B, grad.data_ptr(), L.stream()))
    torch.cuda.synchronize()
    assert torch.isfinite(grad).all()
    got = (grad.double() - 3.5).cpu()
    inputs = _wgrad_inputs([a[:B].double().cpu() for a in acts], use_voxel)
    for d, gname in enumerate(GEMM_OF_DZ):
        N, K = GEMM_N[gname], Kd[gname]
        if gname.startswith("O") and not want_object:
            assert torch.equal(grad[w_off[gname]:b_off[gname] + N], prefill[w_off[gname]:b_off[gname] + N]), gname
            continue
        dz = dzs[d][:B, :N].double().cpu()
        err = (got[w_off[gname]:w_off[gname] + N * K].view(N, K) - dz.t() @ inputs[gname]).abs()
        bound = dz.abs().t() @ inputs[gname].abs()
        assert (err <= 1e-4 * bound + 1e-6).all(), (gname, err.max().item())
        db_err = (got[b_off[gname]:b_off[gname] + N] - dz.sum(0)).abs()
        assert (db_err <= 1e-4 * dz.abs().sum(0) + 1e-6).all(), (gname, db_err.max().item())


# ------------------------------------------------------------------------------------------------
# 5. compositing backward in every mode; the seeded noise path
# ------------------------------------------------------------------------------------------------
COMPOSITE_MODES = {
    "eval": dict(),
    "white_bbox": dict(white_back=True, rays_in_bbox=True),
    "zero_last_delta": dict(zero_last_delta=True),
    "train_noise_mask": dict(noise_std=1.0, is_eval=False, frustum_bound_th=0.05, pass_through_mask=True),
    "white_train_mask": dict(white_back=True, is_eval=False, frustum_bound_th=0.05),
    "zero_last_white_noise": dict(zero_last_delta=True, white_back=True, noise_std=1.0, is_eval=False),
    "scene_only": dict(forward_instance=False, white_back=True),
}


def _composite_inputs(n, S, seed):
    rng = np.random.default_rng(seed)
    rays = synth.random_rays(seed, n)
    near, far = rays[:, 6:7].double(), rays[:, 7:8].double()
    t = torch.from_numpy(np.sort(rng.random((n, S)), -1))
    z = (near + (far - near) * t).float()
    f = lambda *sh: torch.from_numpy(rng.standard_normal(sh).astype(np.float32))
    return dict(z=z, sigma=f(n, S) * 5, isigma=f(n, S) * 5, rgb=torch.sigmoid(f(n, S, 3)),
                irgb=torch.sigmoid(f(n, S, 3)), ns=f(n, S), no=f(n, S),
                ptm=torch.from_numpy(rng.random((n, 1)) < 0.5), gout=lambda *sh: f(*sh))


@pytest.mark.parametrize("S", [1, 31, 33, 128, 192, 2048])
@pytest.mark.parametrize("mode", list(COMPOSITE_MODES))
def test_composite_bwd_matches_float64_autograd(mode, S):
    """onerf_composite_bwd against float64 autograd of the oracle's composite_pass, for every flag set of the
    compositing forward test plus white_back / zero_last_delta with the object branch and the scene-only call, at
    sample counts around the warp width and up to the 2048 limit.  d rgb within 2e-5 and d sigma within 1e-3 of
    max(1, max |reference|) (fp32 transmittance products over S samples against float64)."""
    from object_nerf_b200 import engine
    kw = dict(COMPOSITE_MODES[mode])
    fi = kw.pop("forward_instance", True)
    use_ptm = kw.pop("pass_through_mask", False)
    c = _composite_inputs(9, S, seed=S + 17)
    noise = kw.get("noise_std", 0.0) > 0
    leaf = lambda t: t.double().clone().requires_grad_(True)
    sigma, isigma, rgb, irgb = leaf(c["sigma"]), leaf(c["isigma"]), leaf(c["rgb"]), leaf(c["irgb"])
    ref = {}
    O.composite_pass(ref, "x", sigma, rgb, isigma, irgb, c["z"].double(), forward_instance=fi,
                     pass_through_mask=c["ptm"] if use_ptm else None,
                     noise_scene=c["ns"].double() if noise else None, noise_obj=c["no"].double() if noise else None,
                     **{"is_eval": True, **kw})
    names = ["rgb", "depth", "opacity"] + (["rgb_instance", "depth_instance", "opacity_instance"] if fi else [])
    gout = {k: c["gout"](*ref[f"{k}_x"].shape) for k in names}
    sum((ref[f"{k}_x"] * gout[k].double()).sum() for k in names).backward()
    scene = torch.cat([c["rgb"], c["sigma"][..., None]], -1).contiguous().to(DEV)
    obj = torch.cat([c["irgb"], c["isigma"][..., None]], -1).contiguous().to(DEV) if fi else None
    dscene, dobj = engine.composite_bwd(
        c["z"].to(DEV), scene, obj, ref["depth_x"].detach().float().to(DEV), {k: v.to(DEV) for k, v in gout.items()},
        noise_std=kw.get("noise_std", 0.0), white_back=kw.get("white_back", False), is_eval=kw.get("is_eval", True),
        zero_last_delta=kw.get("zero_last_delta", False), frustum_bound_th=kw.get("frustum_bound_th", 0.0),
        pass_through_mask=c["ptm"].to(DEV) if use_ptm else None, noise_scene=c["ns"].to(DEV) if noise else None,
        noise_obj=c["no"].to(DEV) if noise else None)
    torch.cuda.synchronize()
    pairs = [(dscene, rgb.grad, sigma.grad, "scene")] + ([(dobj, irgb.grad, isigma.grad, "obj")] if fi else [])
    for got, want_rgb, want_sigma, nm in pairs:
        got = got.double().cpu()
        s_rgb = max(1.0, want_rgb.abs().max().item())
        s_sig = max(1.0, want_sigma.abs().max().item())
        e_rgb = (got[..., :3] - want_rgb).abs().max().item()
        e_sig = (got[..., 3] - want_sigma).abs().max().item()
        print(f"composite_bwd {mode} S={S} {nm}: d rgb {e_rgb / s_rgb:.2e}, d sigma {e_sig / s_sig:.2e} (relative)")
        assert e_rgb <= 2e-5 * s_rgb, (nm, e_rgb, s_rgb)
        assert e_sig <= 1e-3 * s_sig, (nm, e_sig, s_sig)


SEED = (0x5EED_0001 << 32) | 0x0000_BEEF     # >= 2^32: the high key word matters


def test_sample_coarse_seeded_jitter_is_numpy_philox():
    """onerf_sample_coarse(perturb = 1, no jitter buffer, seed) draws U[0, 1) from Philox stream 0 at index ray S + i:
    bit-identical to the same call fed numpy's uniforms as the jitter buffer, and different from another seed."""
    from object_nerf_b200 import engine
    n, S = 37, 64
    rays = synth.random_rays(3, n).to(DEV)
    u = torch.from_numpy(philox_uniform(SEED, 0, np.arange(n * S))).view(n, S).to(DEV)
    z_seed = engine.sample_coarse(rays, S, perturb=1.0, seed=SEED)
    z_buf = engine.sample_coarse(rays, S, perturb=1.0, jitter=u)
    z_other = engine.sample_coarse(rays, S, perturb=1.0, seed=SEED & 0xFFFFFFFF)
    torch.cuda.synchronize()
    assert torch.equal(z_seed, z_buf)
    assert not torch.equal(z_seed, z_other)


def test_composite_seeded_noise_forward_and_backward_match_numpy_philox():
    """noise_std = 1 with no noise buffers: the forward draws N(0, 1) from Philox stream 2 (scene) / 3 (object) at index
    ray S + i and the backward re-draws the same values.  Both must match the calls fed numpy's normals (which agree
    with the device's logf / cospif to an ulp or two), and differ from the noise-free calls."""
    from object_nerf_b200 import engine
    n, S = 29, 96
    c = _composite_inputs(n, S, seed=41)
    idx = np.arange(n * S)
    ns = torch.from_numpy(philox_normal(SEED, 2, idx)).view(n, S).to(DEV)
    no = torch.from_numpy(philox_normal(SEED, 3, idx)).view(n, S).to(DEV)
    z = c["z"].to(DEV)
    scene = torch.cat([c["rgb"], c["sigma"][..., None]], -1).contiguous().to(DEV)
    obj = torch.cat([c["irgb"], c["isigma"][..., None]], -1).contiguous().to(DEV)
    kw = dict(noise_std=1.0, is_eval=False, frustum_bound_th=0.05)
    f_seed = engine.composite(z, scene, obj, seed=SEED, **kw)
    f_buf = engine.composite(z, scene, obj, noise_scene=ns, noise_obj=no, **kw)
    f_none = engine.composite(z, scene, obj, **dict(kw, noise_std=0.0))
    for k in f_seed:
        assert (f_seed[k] - f_buf[k]).abs().max().item() <= 1e-5, k
    assert (f_seed["weights"] - f_none["weights"]).abs().max().item() > 1e-2
    grads = {k: c["gout"](*f_seed[k].shape).to(DEV) for k in ("rgb", "depth", "opacity", "rgb_instance", "depth_instance",
                                                               "opacity_instance")}
    common = (z, scene, obj, f_seed["depth"], grads)
    kw = dict(noise_std=1.0, frustum_bound_th=0.05)
    d_seed = engine.composite_bwd(*common, seed=SEED, **kw)
    d_buf = engine.composite_bwd(*common, noise_scene=ns, noise_obj=no, **kw)
    d_wrong = engine.composite_bwd(*common, noise_scene=no, noise_obj=ns, **kw)        # the two streams exchanged
    torch.cuda.synchronize()
    for a, b, nm in ((d_seed[0], d_buf[0], "scene"), (d_seed[1], d_buf[1], "obj")):
        scale = max(1.0, b.abs().max().item())
        err = (a - b).abs().max().item()
        print(f"seeded composite_bwd {nm}: max |seeded - numpy buffers| / scale = {err / scale:.2e}")
        assert err <= 1e-4 * scale, (nm, err, scale)
    assert (d_seed[0] - d_wrong[0]).abs().max().item() > 1e-2


# ------------------------------------------------------------------------------------------------
# 6. whole steps the other files do not run
# ------------------------------------------------------------------------------------------------
STEP_CASES = {
    "scene_only_voxel": dict(use_voxel=True, forward_instance=False),
    "scene_only_plain": dict(use_voxel=False, forward_instance=False),
    "ragged_41_rays_fine_32": dict(use_voxel=True, n_rays=41, n_importance=32),
    "white_back": dict(use_voxel=True, white_back=True),
    "coarse_only": dict(use_voxel=True, n_importance=0),
}


def _grad_case(ov):
    """GRAD_CASE (voxel) or GRAD_CASE_PLAIN with overrides: inputs sized for the overridden case, batch / codes as the
    fixtures' builders make them."""
    from tests import grad_plain
    uv = ov["use_voxel"]
    c = dict(cases.GRAD_CASE if uv else grad_plain.GRAD_CASE_PLAIN, **ov)
    inp = cases.build_render_case(c)
    extra = (cases.build_grad_case if uv else grad_plain.build_grad_case_plain)(n_rays=c["n_rays"])
    inp.update(instance_ids=extra["instance_ids"], code_table=extra["code_table"], batch=extra["batch"])
    return c, inp


def _loss(out, batch, typs, forward_instance):
    """cases.total_loss; without the object branch its instance terms are constants (zero maps)."""
    if not forward_instance:
        out = dict(out)
        for typ in typs:
            for k in ("rgb", "depth", "opacity"):
                out.setdefault(f"{k}_instance_{typ}", torch.zeros_like(out[f"{k}_{typ}"]).detach())
    return cases.total_loss(out, batch)


def _pool_key(precision, c):
    prec = _lib().PREC_BF16 if precision == "bf16" else _lib().PREC_FP32
    return (_lib().load().onerf_train_workspace_bytes_prec(prec, int(c["use_voxel"]), c["n_rays"], c["n_samples"],
                                                            c["n_importance"]), torch.device(DEV))


def _step(precision, c, inp, pool_fill=None):
    from object_nerf_b200 import Embedding, backward, render_rays
    uv = c["use_voxel"]
    models = {k: helpers.make_model(w, uv, DEV).train() for k, w in inp["weights"].items()}
    emb = helpers.GridModule(inp["grid"]).to(DEV) if uv else Embedding(3, 10)
    lib = helpers.CodeLib(inp["code_table"]).to(DEV)
    codes = lib.embedding_instance(inp["instance_ids"].view(-1).to(DEV))
    if pool_fill is not None:
        assert backward._pool.free.get(_pool_key(precision, c)), "no pooled workspace of this step's size to fill"
        for lst in backward._pool.free.values():
            for t in lst:
                t.fill_(pool_fill)
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    out = render_rays(models, {"xyz": emb, "dir": Embedding(3, 4)}, inp["rays"].to(DEV), N_samples=c["n_samples"],
                      perturb=c["perturb"], noise_std=c["noise_std"], N_importance=c["n_importance"],
                      white_back=c["white_back"], forward_instance=c["forward_instance"], embedding_instance=codes,
                      frustum_bound_th=c["frustum_bound_th"], pass_through_mask=inp["pass_through_mask"].to(DEV),
                      is_eval=False, precision=precision, _rand=rand)
    loss = _loss(out, {k: v.to(DEV) for k, v in inp["batch"].items()}, list(models), c["forward_instance"])
    loss.backward()
    named = [(f"{typ}.{k}", p) for typ, m in models.items() for k, p in m.named_parameters()]
    named.append(("codes", lib.embedding_instance.weight))
    if uv:
        named.append(("voxel", emb.embedding_space_ftr.weight))
    return loss.item(), {k: (p.grad.detach().clone() if p.grad is not None else None) for k, p in named}


def _is_object_param(name):
    return name == "codes" or ".inst" in name


@pytest.mark.parametrize("case", list(STEP_CASES))
def test_training_step_bf16_vs_fp32_untested_configurations(case):
    """Whole training steps on the tensor cores against the fp32 path: loss within 2 %, per tensor norm within 5 % and
    cosine >= 0.995; with forward_instance = False the object layers get no gradient on either path."""
    c, inp = _grad_case(STEP_CASES[case])
    loss, g16 = _step("bf16", c, inp)
    loss32, g32 = _step("fp32", c, inp)
    assert abs(loss - loss32) <= 2e-2 * abs(loss32), (loss, loss32)
    bad, report = [], []
    for name, a in g16.items():
        b = g32[name]
        zero = lambda t: t is None or not t.any()
        if zero(b):
            assert zero(a), (name, "gradient where the fp32 path has none")
            continue
        a, b = a.reshape(-1).double(), b.reshape(-1).double()
        ratio = (a.norm() / b.norm()).item()
        cos = (a @ b / (a.norm() * b.norm() + 1e-30)).item()
        report.append((name, ratio, cos))
        if not (0.95 <= ratio <= 1.05 and cos >= 0.995):
            bad.append((name, ratio, cos))
    print(case, "worst cosine", min(report, key=lambda r: r[2]))
    assert not bad, bad
    if not c["forward_instance"]:
        assert not any(_is_object_param(r[0]) for r in report), report


def test_pooled_training_workspace_garbage_does_not_reach_the_gradients():
    """The training workspace is pooled and not cleared between steps: a step on a pooled workspace filled with 0xFF
    (bf16 and fp32 NaN everywhere) gives finite gradients equal to a step on a zero-filled one, to run-to-run atomic
    noise, in either precision."""
    c, inp = _grad_case(dict(use_voxel=True, n_rays=41, n_importance=32))
    for precision in ("bf16", "fp32"):
        _step(precision, c, inp)                        # leaves the workspace in the pool
        _, g0 = _step(precision, c, inp, pool_fill=0)
        _, gf = _step(precision, c, inp, pool_fill=0xFF)
        for name, a in g0.items():
            b = gf[name]
            if a is None:
                assert b is None, (precision, name)
                continue
            assert torch.isfinite(b).all(), (precision, name)
            scale = a.abs().max().item() + 1e-30
            assert (a - b).abs().max().item() <= 1e-4 * scale, (precision, name, (a - b).abs().max().item(), scale)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_training_workspace_one_byte_short_is_refused(precision):
    """onerf_render_rays_fwd and onerf_render_rays_bwd with a training workspace one byte smaller than
    onerf_train_workspace_bytes_prec: ONERF_ERR_WORKSPACE and a message, before any kernel runs."""
    from object_nerf_b200 import engine
    c, inp = _grad_case(dict(use_voxel=True, n_rays=41, n_importance=32))
    packed = {k: engine.packed_for(helpers.make_model(w, True, DEV), True, fresh=True) for k, w in inp["weights"].items()}
    grid = engine.GridBuffers.from_module(helpers.GridModule(inp["grid"]).to(DEV))
    codes = inp["code_table"][inp["instance_ids"].view(-1)].to(DEV)
    ws = helpers.aligned_u8(_pool_key(precision, c)[0] - 1, DEV, fill=0)
    L = _lib()
    lib, ctx = L.load(), _ctx()
    plan = engine.RenderPlan(inp["rays"].to(DEV), packed["coarse"], packed["fine"], grid, codes=codes,
                             n_samples=c["n_samples"], n_importance=c["n_importance"], precision=precision, train_ws=ws)
    launches = L.launch_count(torch.device(DEV))
    assert lib.onerf_render_rays_fwd(ctx, C.byref(plan.args), L.stream()) == -4      # ONERF_ERR_WORKSPACE
    assert b"training workspace too small" in lib.onerf_last_error()
    b = L.RenderBwdArgs()
    ptrs = (C.c_void_p * 20)(*([ws.data_ptr()] * 20))
    b.W_coarse, b.dW_coarse, b.db_coarse, b.W_fine, b.dW_fine, b.db_fine = (ptrs,) * 6
    assert lib.onerf_render_rays_bwd(ctx, C.byref(plan.args), C.byref(b), L.stream()) == -4
    assert b"training workspace too small" in lib.onerf_last_error()
    assert L.launch_count(torch.device(DEV)) == launches


def _oracle_grads(c, inp, dtype):
    """The same step restated by the CPU oracle in `dtype`, as _oracle_grads_fp64 of test_gpu_train_plain does for the
    plain fixture, with a leaf voxel table: float64 is the exact reference, float32 shows how far fp32 rounding alone
    moves each entry.  -> (loss, {parameter name: flat gradient or None})."""
    cast = lambda t: t.to(dtype) if t is not None and t.is_floating_point() else t
    leaves = {}

    def leaf(name, t):
        leaves[name] = t.to(dtype).clone().requires_grad_(True)
        return leaves[name]

    weights = {typ: {k: (leaf(f"{typ}.{helpers.REF_NAMES[k]}.weight", W), leaf(f"{typ}.{helpers.REF_NAMES[k]}.bias", b))
                     for k, (W, b) in w.items()} for typ, w in inp["weights"].items()}
    codes = leaf("codes", inp["code_table"])[inp["instance_ids"].view(-1)]
    grid = None
    if c["use_voxel"]:
        g = inp["grid"]
        grid = O.VoxelGrid(cast(g["offset"]), cast(g["voxel_size"]), g["shape"].tolist(), g["idx_map"],
                           leaf("voxel", g["table"]))
    out = O.render_rays(weights, grid, cast(inp["rays"]), codes, n_samples=c["n_samples"], perturb=c["perturb"],
                        noise_std=c["noise_std"], n_importance=c["n_importance"], white_back=c["white_back"],
                        forward_instance=c["forward_instance"], frustum_bound_th=c["frustum_bound_th"],
                        pass_through_mask=inp["pass_through_mask"], is_eval=False,
                        rand={k: cast(v) for k, v in inp["rand"].items()})
    loss = _loss(out, {k: cast(v) for k, v in inp["batch"].items()}, list(inp["weights"]), c["forward_instance"])
    loss.backward()
    return loss.item(), {k: (t.grad.reshape(-1) if t.grad is not None else None) for k, t in leaves.items()}


# coarse_only_two_chunks: 1 030 rays x 64 samples, the smallest coarse-only batch the fp32 backward runs in two chunks
# (1 024 + 6 rays)
ORACLE_CASES = dict(STEP_CASES, coarse_only_two_chunks=ORACLE_TWO_CHUNKS)


@pytest.mark.parametrize("case", ["scene_only_voxel", "scene_only_plain", "coarse_only", "coarse_only_two_chunks"])
def test_training_step_fp32_matches_float64_oracle(case):
    """The fp32 path of the scene-only and coarse-only steps, and of a coarse-only step across a chunk boundary of the
    fp32 backward, against float64 autograd of the oracle (leaf table for the voxel grid), with the gates of the plain
    fixture's fp32 test: loss 2e-4, per-tensor norm 2e-3, sampled entries within 1 % of the tensor's RMS entry.  An
    entry that the oracle's own float32 restatement already moves by more than that cannot decide the gate: it is
    reported, not asserted, and at least 95 % of the entries must be decidable.  Without the object branch the object
    layers and codes get no gradient."""
    c, inp = _grad_case(ORACLE_CASES[case])
    loss, ours = _step("fp32", c, inp)
    t0 = time.perf_counter()
    loss64, exact = _oracle_grads(c, inp, torch.float64)
    _, rounded = _oracle_grads(c, inp, torch.float32)
    print(f"{case}: {c['n_rays']} rays, the float64 and float32 oracle steps took {time.perf_counter() - t0:.1f} s")
    assert abs(loss - loss64) <= 2e-4 * abs(loss64), (loss, loss64)
    checked, total, undecidable = 0, 0, []
    for name, ref in exact.items():
        g = ours[name]
        if ref is None:
            assert not c["forward_instance"] and _is_object_param(name), name
            assert g is None or not g.any(), name
            continue
        gr = g.detach().cpu().reshape(-1).double()
        ref_norm = ref.norm().item()
        assert abs(gr.norm().item() - ref_norm) <= 2e-3 * max(ref_norm, 1e-7), (name, gr.norm().item(), ref_norm)
        idx = cases.sample_indices(name, gr.numel())
        rms = max(ref_norm, 1e-7) / max(1.0, gr.numel() ** 0.5)
        gate = 1e-2 * rms + 1e-8
        decidable = (rounded[name][idx].double() - ref[idx]).abs() <= gate
        err = (gr[idx] - ref[idx]).abs()
        assert (err[decidable] <= gate).all(), (name, err[decidable].max().item() / rms)
        checked += int(decidable.sum())
        total += len(idx)
        if not decidable.all():
            undecidable.append((name, int((~decidable).sum()), round(err[~decidable].max().item() / rms, 4)))
    print(case, "fp32 vs float64 oracle: entries checked", checked, "of", total, "; not decidable:", undecidable)
    assert checked >= 0.95 * total
