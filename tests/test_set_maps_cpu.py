"""CPU checks of the per-set maps of edited frames (include/onerf_ext.h: onerf_render_edit_frame_sets,
onerf_render_edit_sets_workspace_bytes; editing.set_keys):
  * the float64 reference (tests/set_maps_oracle.py) on the inputs of the reference's multi fixtures: its coarse per-set
    opacity and depth equal the fixture's own weights_coarse / z_vals_coarse summed by obj_ids_coarse, and summed over
    the sets every map of both passes gives the fixture's joint maps, within float32 reassociation;
  * the entry's export, declaration, struct layout, workspace arithmetic and refusals before any CUDA call;
  * editing.render_frame's key checks for the new keys."""
import ctypes
import os
import re

import pytest
import torch

from oracle import onerf_oracle as O
from tests import cases
from tests import set_maps_oracle as SO
from tests.multi_noise_cases import NOISE_CLIP_CASES, build_noise_clip_case
from tests.test_edit_frame_cpu import _Args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
a256 = lambda x: (x + 255) // 256 * 256
U24 = 2.0 ** -24
FIXTURES = sorted(cases.MULTI_CASES) + ["dup_tied", "clip_swallow", "clip_empty", "clip_far_zero"]


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def _oracle(name):
    if name in cases.MULTI_CASES:
        c = cases.MULTI_CASES[name]
        inp, extra = cases.build_multi_case(c), {}
    else:
        c = NOISE_CLIP_CASES[name]
        inp = build_noise_clip_case(c)
        extra = dict(perturb=c["perturb"], noise_std=c["noise_std"], rand=inp["rand"])
    g = inp["grid"]
    grid = O.VoxelGrid(g["offset"], g["voxel_size"], g["shape"].tolist(), g["idx_map"], g["table"])
    out = SO.render_rays_multi_sets(inp["weights"], grid, inp["code_table"], inp["rays_list"], c["obj_ids"],
                                    n_samples=c["n_samples"], n_importance=c["n_importance"], white_back=c["white_back"],
                                    skip_boxes=[cases.box_affine(b) for b in inp["boxes"]], **extra)
    return c, out


def _within(got, want, bound, label):
    err = (got - want).abs()
    assert (err <= bound).all(), (label, err.max().item(), bound.max().item())


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_sums_the_fixture_by_set(golden, name):
    """Float32 bound: the fixture's fp32 weights carry the rounding of T transmittance factors, each of which may be off by
    u in absolute terms (1 - alpha after an opaque sample), and a sum of T terms a few more roundings, so a set's map
    is off by at most (T + 8) u sum |w v| over the ray's samples."""
    c, out = _oracle(name)
    g = golden("multi_" + name)
    for k in g:                                   # the port under the maps is the reference's, bit for bit
        assert torch.equal(out[k], g[k]), k
    n_obj = len(c["obj_ids"])
    w, z, ids = g["weights_coarse"].double(), g["z_vals_coarse"].double(), g["obj_ids_coarse"]
    T = w.shape[1]
    for i in range(n_obj):
        wi = torch.where(ids == i, w, torch.zeros_like(w))
        for key, v in (("opacity_sets_coarse", 1.0), ("depth_sets_coarse", z)):
            ref = (wi * v).sum(1)
            _within(out[key][:, i], ref, (T + 8) * U24 * (w * v).abs().sum(1) + 1e-30, (key, i))
    typs = ("coarse", "fine") if c["n_importance"] > 0 else ("coarse",)
    for typ in typs:
        op = g[f"opacity_{typ}"].double()
        rgb = g[f"rgb_{typ}"].double() - ((1 - op)[:, None] if c["white_back"] else 0)
        T = g[f"weights_{typ}"].shape[1]
        for key, joint, tot in (("opacity_sets", op, out[f"opacity_sets_{typ}"]),
                                ("depth_sets", g[f"depth_{typ}"].double(), out[f"depth_sets_{typ}"]),
                                ("rgb_sets", rgb, out[f"rgb_sets_{typ}"])):
            s = tot.sum(1)
            scale = tot.abs().sum(1) + (2.0 if key == "rgb_sets" else 0.0)   # white back: two more roundings of 1 - op
            _within(s, joint, (T + 8) * U24 * scale + 1e-30, (key, typ))
        if n_obj == 1:
            for k in SO.SET_KEYS:
                assert out[f"{k}_{typ}"].shape[1] == 1
    # the missed object sets of the fixtures contribute exact zeros
    for i in range(n_obj):
        missed = ((ids == i) & (g["z_vals_coarse"] == 0)).any(1)
        for k in SO.SET_KEYS:
            assert (out[f"{k}_coarse"][missed, i] == 0).all(), (k, i)


def test_set_maps_of_one_set_are_the_joint_maps():
    """With one set the joint sort is the set's own order: the float64 per-set maps are the joint ones exactly."""
    g = torch.Generator().manual_seed(0)
    z = [torch.sort(torch.rand(5, 9, generator=g) * 4, -1).values]
    rgb, sig = [torch.rand(5, 9, 3, generator=g)], [torch.randn(5, 9, generator=g) * 5]
    m = SO.composite_multi_sets(z, rgb, sig)
    for k in ("opacity", "depth", "rgb"):
        assert torch.equal(m[f"{k}_sets"][:, 0], m[k]), k


# ------------------------------------------------------------------------------------------------
# C entry, without a device
# ------------------------------------------------------------------------------------------------
def _ext_declarations():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "onerf_ext.h")).read(), flags=re.S)
    return src, {m.group(1): [p.strip() for p in m.group(2).split(",")]
                 for m in re.finditer(r"\b(onerf_[a-z0-9_]+)\s*\(([^)]*)\)", src)}


def test_exports_declarations_and_struct(lib):
    from object_nerf_b200 import _lib
    src, decl = _ext_declarations()
    assert decl["onerf_render_edit_frame_sets"] == ["onerf_ctx* ctx", "const onerf_render_edit_args* args",
                                                    "const onerf_set_maps* coarse", "const onerf_set_maps* fine",
                                                    "void* stream"]
    assert decl["onerf_render_edit_sets_workspace_bytes"] == ["int chunk_rays", "int n_obj", "int n_samples",
                                                              "int n_importance"]
    for name in ("onerf_render_edit_frame_sets", "onerf_render_edit_sets_workspace_bytes"):
        assert name in _lib.EXPORTS_EXT and name not in _lib.EXPORTS and hasattr(lib, name), name
        assert len(getattr(lib, name).argtypes) == len(decl[name]), name
    body = re.search(r"typedef struct onerf_set_maps \{(.*?)\} onerf_set_maps;", src, flags=re.S).group(1)
    names = [d.split()[-1].lstrip("*") for d in body.split(";") if d.strip()]
    assert [f[0] for f in _lib.SetMaps._fields_] == names == ["opacity", "depth", "rgb"]
    assert ctypes.sizeof(_lib.SetMaps) == 24


def test_workspace_bytes(lib):
    """The sets entry's workspace is the frame's plus one (n_obj, chunk, S + K) float buffer for the fine pass's weights in
    set order; without a fine pass it is the frame's.  onerf_render_edit_workspace_bytes is unchanged."""
    f, base = lib.onerf_render_edit_sets_workspace_bytes, lib.onerf_render_edit_workspace_bytes
    assert f(0, 3, 64, 64) == 0 and f(4096, 0, 64, 64) == 0 and f(4096, 3, 64, -1) == 0
    for n, no, s, si in ((1, 1, 2, 0), (1000, 3, 64, 64), (4096, 3, 64, 0), (65536, 25, 64, 64), (77, 5, 32, 96)):
        extra = a256(no * n * (s + si) * 4) if si > 0 else 0
        assert f(n, no, s, si) == base(n, no, s, si) + extra, (n, no, s, si)


def _set_maps(lib, **arrays):
    from object_nerf_b200 import _lib
    m = _lib.SetMaps()
    for k, v in arrays.items():
        setattr(m, k, v)
    return m


def test_refusals_without_a_device(lib):
    """Refused before the context is touched (the fake one would fault): a fine array without a fine pass, misaligned
    arrays, and the frame's own refusals reported under the new entry's name."""
    def call(t, coarse=None, fine=None, ctx=True):
        fake_ctx = ctypes.c_void_p(1 << 21) if ctx else None
        t.a.workspace_bytes = lib.onerf_render_edit_sets_workspace_bytes(1000, 3, t.a.n_samples, t.a.n_importance)
        rc = lib.onerf_render_edit_frame_sets(fake_ctx, ctypes.byref(t.a), ctypes.byref(coarse) if coarse else None,
                                              ctypes.byref(fine) if fine else None, None)
        return rc, lib.onerf_last_error()

    good = 1 << 24
    t = _Args(lib)
    t.a.n_importance, t.a.packed_fine = 0, None
    for arr in ("opacity", "depth", "rgb"):
        rc, msg = call(t, _set_maps(lib, opacity=good), _set_maps(lib, **{arr: good}))
        assert rc == -1 and msg == b"onerf_render_edit_frame_sets: fine set maps without a fine pass", msg
    for which in ("coarse", "fine"):
        for arr in ("opacity", "depth", "rgb"):
            m = _set_maps(lib, **{arr: good + 2})
            rc, msg = call(_Args(lib), **{which: m})
            assert rc == -1 and msg == b"onerf_render_edit_frame_sets: set maps must be 4-byte aligned", (which, arr)
    t = _Args(lib)
    t.a.chunk_rays = 0
    rc, msg = call(t, _set_maps(lib, opacity=good))
    assert rc == -1 and msg.startswith(b"onerf_render_edit_frame_sets: chunk_rays < 1")
    rc, msg = call(_Args(lib), _set_maps(lib, opacity=good), ctx=False)
    assert rc == -1 and b"null argument" in msg
    # a set map needs the larger workspace when there is a fine pass
    t = _Args(lib)
    t.a.workspace_bytes = lib.onerf_render_edit_workspace_bytes(1000, 3, 64, 64)
    rc = lib.onerf_render_edit_frame_sets(ctypes.c_void_p(1 << 21), ctypes.byref(t.a), None,
                                          ctypes.byref(_set_maps(lib, rgb=good)), None)
    assert rc == -4 and b"workspace too small" in lib.onerf_last_error()


def test_render_frame_key_checks():
    from object_nerf_b200 import editing
    assert editing.set_keys(0) == ["opacity_sets_coarse", "depth_sets_coarse", "rgb_sets_coarse"]
    assert editing.set_keys(64) == editing.set_keys(0) + ["opacity_sets_fine", "depth_sets_fine", "rgb_sets_fine"]
    assert not set(editing.set_keys(64)) & set(editing.result_keys(64))
    for keys, ni in ((["opacity_sets_fine"], 0), (["rgb_sets_fine", "rgb_coarse"], 0), (["opacity_sets"], 64),
                     (["rgb_set_coarse"], 64)):
        with pytest.raises(KeyError):
            editing.render_frame({}, {"xyz": None}, None, 4, 4, 1.0, [], 0.1, 1.0, 1.0, keys=keys, N_importance=ni)
