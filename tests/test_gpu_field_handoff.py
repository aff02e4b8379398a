"""The fused forward's X hand-off: the encoder warps write tile t + gridDim.x while the consumers run tile t.

Each case runs the bf16 tensor-core kernel against the fp32 kernel (DESIGN.md §2 bf16 tolerances) and checks that two
identical launches are bit-identical, at tile counts that exercise the hand-off differently: fewer tiles than SMs,
exactly one tile per CTA, many tiles per CTA, a partial last tile, S = 1 and an odd S (tiles spanning many rays), scene-
and object-only launches, muted rows, for the voxel and the plain-PE model, and the training dump of X.
"""
import ctypes as C

import pytest
import torch

from tests import cases, helpers

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _setup(use_voxel):
    from object_nerf_b200 import engine
    inp = cases.build_render_case(dict(cases.RENDER_CASES["eval_voxel" if use_voxel else "eval_plain"], n_rays=8))
    model = helpers.make_model(inp["weights"]["coarse"], use_voxel, DEV)
    packed = engine.packed_for(model, use_voxel)
    grid = engine.GridBuffers.from_module(helpers.GridModule(inp["grid"]).to(DEV)) if use_voxel else None
    return packed, grid, inp["codes"][0].to(DEV)


def _inputs(n_rays, S, seed):
    from object_nerf_b200 import engine
    g = torch.Generator().manual_seed(seed)
    o = (torch.rand(n_rays, 3, generator=g) - 0.5) * 0.4 + torch.tensor([1.0, 1.0, 0.5])
    d = torch.nn.functional.normalize(torch.randn(n_rays, 3, generator=g), dim=1)
    rays = torch.cat([o, d, torch.full((n_rays, 1), 0.1), torch.full((n_rays, 1), 1.5)], 1).to(DEV)
    return rays, engine.sample_coarse(rays, S).contiguous()


def _field(packed, grid, rays, z, code, precision, **kw):
    from object_nerf_b200 import engine
    n = rays.shape[0]
    codes = code.expand(n, -1).contiguous()
    return engine.field(rays, z, packed, grid, codes=codes, precision=precision, **kw)


def _close(got, want):
    """bf16 field outputs against fp32: rgb within 3e-2, sigma within 3e-2 (1 + |sigma|); muted sigma exactly."""
    rgb_bad = ((got[..., :3] - want[..., :3]).abs() > 3e-2).float().mean().item()
    s_got, s_want = got[..., 3], want[..., 3]
    assert torch.equal(s_got == -1e5, s_want == -1e5)
    s_bad = ((s_got - s_want).abs() > 3e-2 * (1 + s_want.abs())).float().mean().item()
    assert rgb_bad < 2e-3 and s_bad < 2e-3, (rgb_bad, s_bad)


def _n_sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


# (n_rays, S): fewer tiles than SMs, one tile per CTA, many tiles per CTA, partial last tile with odd S, S = 1
SHAPES = {"few_tiles": lambda: (10, 64), "one_tile_per_cta": lambda: (2 * _n_sms(), 64),
          "many_tiles": lambda: (1000, 128), "odd_s_partial": lambda: (77, 63), "s1": lambda: (3001, 1)}


@pytest.mark.parametrize("use_voxel", [True, False], ids=["voxel", "plain"])
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("branches", [(True, True), (True, False), (False, True)], ids=["both", "scene", "object"])
def test_handoff_matches_fp32_and_repeats(use_voxel, shape, branches):
    packed, grid, code = _setup(use_voxel)
    n_rays, S = SHAPES[shape]()
    rays, z = _inputs(n_rays, S, seed=n_rays * 1000 + S)
    ws, wo = branches
    kw = dict(want_scene=ws, want_object=wo)
    a = _field(packed, grid, rays, z, code, "bf16", **kw)
    b = _field(packed, grid, rays, z, code, "bf16", **kw)
    ref = _field(packed, grid, rays, z, code, "fp32", **kw)
    torch.cuda.synchronize()
    for x, y, r in zip(a, b, ref):
        if r is None:
            continue
        assert torch.equal(x, y)
        _close(x, r)


@pytest.mark.parametrize("use_voxel", [True, False], ids=["voxel", "plain"])
def test_handoff_muted_rows(use_voxel):
    """mute_zero_rays (rays whose last depth is 0) and a removed-object box: the mute bits travel through meta[]."""
    packed, grid, code = _setup(use_voxel)
    rays, z = _inputs(900, 63, seed=7)
    z[::5, -1] = 0.0
    xyz = rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]
    mid = xyz[..., 0].median().item()
    box = torch.tensor([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, -1e9, -1e9, -1e9, mid, 1e9, 1e9], dtype=torch.float32,
                       device=DEV)[None]
    kw = dict(mute_zero_rays=True, boxes=box)
    a = _field(packed, grid, rays, z, code, "bf16", **kw)
    b = _field(packed, grid, rays, z, code, "bf16", **kw)
    ref = _field(packed, grid, rays, z, code, "fp32", **kw)
    torch.cuda.synchronize()
    assert (ref[0][..., 3] == -1e5).any() and (ref[1][..., 3] == -1e5).any()
    assert not (ref[0][..., 3] == -1e5).all()
    for x, y, r in zip(a, b, ref):
        assert torch.equal(x, y)
        _close(x, r)


@pytest.mark.parametrize("use_voxel", [True, False], ids=["voxel", "plain"])
def test_handoff_training_dump_x(use_voxel):
    """The training forward's X atoms (written by the consumers from the encoders' buffer) against the fp32 encoding,
    bit-identical between two launches, and the outputs equal to those of the inference launch."""
    from object_nerf_b200 import _lib as L
    packed, grid, code = _setup(use_voxel)
    n_rays, S = 700, 63               # 44 100 samples: 345 tiles, the last one partial
    rays, z = _inputs(n_rays, S, seed=11)
    B = n_rays * S
    T = helpers.train_layout(use_voxel, B)
    codes = code.expand(n_rays, -1).contiguous()

    def dump_launch():
        ws = helpers.aligned_u8(T["total"], DEV, fill=0)
        scene = torch.empty(n_rays, S, 4, device=DEV)
        obj = torch.empty(n_rays, S, 4, device=DEV)
        rc = torch.empty(n_rays, 448, device=DEV)
        a = L.FieldArgs()
        a.rays, a.z, a.z_stride, a.codes = rays.data_ptr(), z.data_ptr(), S, codes.data_ptr()
        a.n_rays, a.n_samples = n_rays, S
        a.grid = C.pointer(grid.c) if grid is not None else None
        a.packed = packed.data_ptr()
        a.want_scene, a.want_object, a.precision = 1, 1, L.PREC_BF16
        a.scene_out, a.obj_out, a.out_stride, a.ray_const = scene.data_ptr(), obj.data_ptr(), S, rc.data_ptr()
        a.train_ws = ws.data_ptr()
        L.check(L.load().onerf_field_fwd(L.ctx(torch.device(DEV)), C.byref(a), L.stream()))
        return scene, obj, ws

    s1, o1, ws1 = dump_launch()
    s2, o2, ws2 = dump_launch()
    s0, o0 = _field(packed, grid, rays, z, code, "bf16")
    kx = 384 if use_voxel else 64
    x_fp32 = torch.empty(B, kx, device=DEV)
    widths = ([384] + [256] * 8 + [256, 128] + [128] * 4 + [128, 64]) if use_voxel else \
        ([64] + [256] * 8 + [256, 128] + [128] * 4 + [128, 64])
    acts = [x_fp32] + [torch.empty(B, w, device=DEV) for w in widths[1:]]
    ptrs = (C.c_void_p * 17)(*[t.data_ptr() for t in acts])
    _field(packed, grid, rays, z, code, "fp32", activations=ptrs)
    torch.cuda.synchronize()
    assert torch.equal(s1, s0) and torch.equal(o1, o0) and torch.equal(s1, s2) and torch.equal(o1, o2)
    x1 = helpers.from_atoms(ws1, T["act_off"][0], T["n_tiles"], T["act_atoms"][0])
    x2 = helpers.from_atoms(ws2, T["act_off"][0], T["n_tiles"], T["act_atoms"][0])
    assert torch.equal(x1, x2)
    got = x1[:B, :kx]
    tol = 2e-2 + 2e-2 * x_fp32.abs()
    bad = ((got - x_fp32).abs() > tol).float().mean().item()
    assert bad < 2e-3, (bad, (got - x_fp32).abs().max().item())
