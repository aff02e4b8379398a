"""CPU checks of edited frames that compose objects from several trained scenes (include/onerf_ext.h:
onerf_render_edit_frame_scenes, onerf_edit_scene, onerf_render_edit_scenes_workspace_bytes; editing.Scene,
editing.import_sets):
  * the entry's export, declarations, struct layout, workspace arithmetic and every refusal before any CUDA call;
  * the reference of tests/compose_oracle.py: with one scene and k = 1 it is the existing multi-set reference exactly, and
    (with oracle/_ref built) it equals the reference's own inference_from_model, sample_pdf and volume_rendering_multi
    called per set with each scene's modules and the depths / densities rescaled by k;
  * editing.import_sets' pose against a float64 restatement built on the reference's center_pose_from_avg."""
import ctypes
import os
import re
import sys
import types

import numpy as np
import pytest
import torch

from oracle import onerf_oracle as O
from oracle import ref_loader as R
from tests import cases
from tests import compose_oracle as CO
from tests import set_maps_oracle as SO
from tests.test_edit_frame_cpu import _Args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
a256 = lambda x: (x + 255) // 256 * 256


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def _header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "onerf_ext.h")).read(), flags=re.S)


def test_exports_declarations_and_struct(lib):
    from object_nerf_b200 import _lib
    src = _header()
    decl = {m.group(1): [p.strip() for p in m.group(2).split(",")]
            for m in re.finditer(r"\b(onerf_[a-z0-9_]+)\s*\(([^)]*)\)", src)}
    assert decl["onerf_render_edit_frame_scenes"] == [
        "onerf_ctx* ctx", "const onerf_render_edit_args* args", "const onerf_edit_scene* scenes_host", "int n_scenes",
        "const int* set_scene_host", "const onerf_set_maps* coarse", "const onerf_set_maps* fine", "void* stream"]
    assert decl["onerf_render_edit_scenes_workspace_bytes"] == ["int chunk_rays", "int n_obj", "int n_samples",
                                                                "int n_importance"]
    for name in ("onerf_render_edit_frame_scenes", "onerf_render_edit_scenes_workspace_bytes"):
        assert name in _lib.EXPORTS_EXT and name not in _lib.EXPORTS and hasattr(lib, name), name
        assert len(getattr(lib, name).argtypes) == len(decl[name]), name
    body = re.search(r"typedef struct onerf_edit_scene \{(.*?)\} onerf_edit_scene;", src, flags=re.S).group(1)
    names = [d.split()[-1].lstrip("*") for d in body.split(";") if d.strip()]
    assert [f[0] for f in _lib.EditScene._fields_] == names == ["grid", "packed_coarse", "packed_fine", "code_table",
                                                                "n_codes", "scale_factor"]
    S = _lib.EditScene
    assert [S.grid.offset, S.packed_coarse.offset, S.packed_fine.offset, S.code_table.offset, S.n_codes.offset,
            S.scale_factor.offset] == [0, 8, 16, 24, 32, 40]
    assert ctypes.sizeof(S) == 48
    assert ctypes.sizeof(_lib.EditSet) == 64                      # the set struct does not grow


def test_workspace_bytes(lib):
    """The scenes entry's workspace is the sets entry's plus one (n_obj, chunk, S + K) float buffer: a pass's depths on
    the frame's axis.  The other two sizes are unchanged."""
    f, sets = lib.onerf_render_edit_scenes_workspace_bytes, lib.onerf_render_edit_sets_workspace_bytes
    assert f(0, 3, 64, 64) == 0 and f(4096, 0, 64, 64) == 0 and f(4096, 3, 0, 64) == 0 and f(4096, 3, 64, -1) == 0
    for n, no, s, si in ((1, 1, 2, 0), (1000, 3, 64, 64), (4096, 3, 64, 0), (65536, 25, 64, 64), (77, 5, 32, 96)):
        assert f(n, no, s, si) == sets(n, no, s, si) + a256(no * n * (s + si) * 4), (n, no, s, si)


class _SceneArgs(_Args):
    """_Args's frame (sets [0, 4, 4], 8 codes) with two source scenes; set 2 comes from scene 1."""

    def __init__(self, lib):
        super().__init__(lib)
        from object_nerf_b200 import _lib
        self.grids = [_lib.Grid(1 << 20, 1 << 20, 1 << 20, 1 << 20, 1 << 20) for _ in range(2)]
        self.scenes = (_lib.EditScene * 2)()
        for j in range(2):
            sc = self.scenes[j]
            sc.grid = ctypes.pointer(self.grids[j])
            sc.packed_coarse = sc.packed_fine = sc.code_table = 1 << 20
            sc.n_codes, sc.scale_factor = 16, 16.0
        self.set_scene = (ctypes.c_int * 3)(-1, -1, 1)
        self.n_scenes = 2
        self.a.workspace_bytes = lib.onerf_render_edit_scenes_workspace_bytes(1000, 3, 64, 64)

    def call(self, ctx=True):
        fake_ctx = ctypes.c_void_p(1 << 21) if ctx else None
        rc = self.lib.onerf_render_edit_frame_scenes(fake_ctx, ctypes.byref(self.a), self.scenes, self.n_scenes,
                                                     self.set_scene, None, None, None)
        return rc, self.lib.onerf_last_error()


def _set(obj, **kw):
    for k, v in kw.items():
        setattr(obj, k, v)


SCENE_REFUSALS = {
    "null_grid": (lambda t: _set(t.scenes[1], grid=None), b"needs its grid, packed_coarse and code_table"),
    "null_grid_table": (lambda t: _set(t.grids[0], table=None), b"null / misaligned grid buffer in a source scene"),
    "misaligned_grid_table": (lambda t: _set(t.grids[1], table=(1 << 20) + 4), b"null / misaligned grid buffer"),
    "null_packed_coarse": (lambda t: _set(t.scenes[0], packed_coarse=None), b"needs its grid, packed_coarse"),
    "null_code_table": (lambda t: _set(t.scenes[1], code_table=None), b"needs its grid, packed_coarse and code_table"),
    "null_packed_fine": (lambda t: _set(t.scenes[1], packed_fine=None), b"needs a source scene's packed_fine"),
    "zero_scale": (lambda t: _set(t.scenes[1], scale_factor=0.0), b"scale_factor must be positive and finite"),
    "negative_scale": (lambda t: _set(t.scenes[0], scale_factor=-2.0), b"scale_factor must be positive and finite"),
    "nan_scale": (lambda t: _set(t.scenes[1], scale_factor=float("nan")), b"scale_factor must be positive and finite"),
    "inf_scale": (lambda t: _set(t.scenes[1], scale_factor=float("inf")), b"scale_factor must be positive and finite"),
    "ratio_overflows_float": (lambda t: _set(t.scenes[1], scale_factor=1e300), b"positive and finite"),
    "scene_index_high": (lambda t: t.set_scene.__setitem__(2, 2), b"set scene index outside [-1, n_scenes)"),
    "scene_index_low": (lambda t: t.set_scene.__setitem__(1, -2), b"set scene index outside [-1, n_scenes)"),
    "no_scenes_but_index": (lambda t: setattr(t, "n_scenes", 0), b"set scene index outside [-1, n_scenes)"),
    "negative_n_scenes": (lambda t: setattr(t, "n_scenes", -1), b"null or negative source scene list"),
    "null_scene_list": (lambda t: setattr(t, "scenes", None), b"null or negative source scene list"),
    "id_outside_its_codes": (lambda t: (_set(t.sets[2], obj_id=16)), b"object id outside its source scene's code table"),
    "negative_source_id": (lambda t: (_set(t.sets[2], obj_id=-3)), b"object id outside its source scene's code table"),
    "base_id_outside_base_codes": (lambda t: _set(t.sets[1], obj_id=8), b"object id outside the code table"),
    "workspace_of_the_sets_entry": (lambda t: setattr(t.a, "workspace_bytes", t.lib.onerf_render_edit_sets_workspace_bytes(
        1000, 3, 64, 64)), b"workspace too small"),
}


@pytest.mark.parametrize("case", sorted(SCENE_REFUSALS))
def test_refusals_without_a_device(lib, case):
    """Every refusal comes before the context is touched (the fake one would fault)."""
    t = _SceneArgs(lib)
    SCENE_REFUSALS[case][0](t)
    rc, msg = t.call()
    assert rc == (-4 if case == "workspace_of_the_sets_entry" else -1), (case, rc, msg)
    assert msg.startswith(b"onerf_render_edit_frame_scenes: ") and SCENE_REFUSALS[case][1] in msg, (case, msg)


def test_source_scene_set_and_frame_refusals_without_a_device(lib):
    t = _SceneArgs(lib)
    t.sets[2].obj_id, t.sets[2].box = 0, None                     # a scene set from a source scene
    rc, msg = t.call()
    assert rc == -2 and msg == (b"onerf_render_edit_frame_scenes: unsupported: a set of a source scene must be an "
                                b"object set (obj_id > 0)"), msg
    t = _SceneArgs(lib)                                           # an id valid in the source's table, not in the base's:
    t.sets[2].obj_id = 12                                         # accepted up to the (fake) context
    t.a.chunk_rays = 0
    rc, msg = t.call()
    assert rc == -1 and b"chunk_rays < 1" in msg
    t = _SceneArgs(lib)
    t.a.n_importance, t.a.packed_fine = 0, None
    t.scenes[1].packed_fine = None                                # no fine pass: packed_fine is not needed
    t.a.chunk_rays = 0
    rc, msg = t.call()
    assert rc == -1 and b"chunk_rays < 1" in msg
    rc, msg = _SceneArgs(lib).call(ctx=False)
    assert rc == -1 and b"null argument" in msg


def test_scene_refuses_a_plain_embedding_and_a_bad_scale():
    from object_nerf_b200 import Embedding, editing, synthetic as S
    g = S.GridModule(S.make_grid(seed=5, shape=(8, 8, 8)))
    with pytest.raises(RuntimeError, match="voxel embedding"):
        editing.Scene({}, {"xyz": Embedding(3, 10)}, None, 2.0)
    for s in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="scale_factor"):
            editing.Scene({}, {"xyz": g}, None, s)
    assert editing.Scene({}, {"xyz": g}, None, 16).scale_factor == 16.0


# ------------------------------------------------------------------------------------------------
# the reference of tests/compose_oracle.py
# ------------------------------------------------------------------------------------------------
def _grid(g):
    return O.VoxelGrid(g["offset"], g["voxel_size"], g["shape"].tolist(), g["idx_map"], g["table"])


@pytest.mark.parametrize("name", sorted(cases.MULTI_CASES))
def test_one_scene_at_k_one_is_the_multi_set_reference(name):
    c = cases.MULTI_CASES[name]
    inp = cases.build_multi_case(c)
    boxes = [cases.box_affine(b) for b in inp["boxes"]]
    kw = dict(n_samples=c["n_samples"], n_importance=c["n_importance"], white_back=c["white_back"], skip_boxes=boxes)
    want = SO.render_rays_multi_sets(inp["weights"], _grid(inp["grid"]), inp["code_table"], inp["rays_list"],
                                     c["obj_ids"], **kw)
    scene = dict(weights=inp["weights"], grid=_grid(inp["grid"]), code_table=inp["code_table"], k=CO.compose_k(2.0, 2.0))
    got = CO.render_rays_multi_scenes([scene], [0] * len(c["obj_ids"]), inp["rays_list"], c["obj_ids"], **kw)
    assert list(got) == list(want)
    for k in want:
        assert torch.equal(got[k], want[k]), k


def _two_scene_case(k_src):
    """The "edit_dup" fixture's scene as the base, plus a second scene (other weights, grid and codes) whose objects 4 and
    6 are sets 3 and 4 at depth scale k_src; set 2 is object 4 of the base."""
    from object_nerf_b200 import synthetic as S
    c = cases.MULTI_CASES["edit_dup"]
    inp = cases.build_multi_case(c)
    base = dict(weights=inp["weights"], grid=inp["grid"], code_table=inp["code_table"], k=1.0)
    src = dict(weights={"coarse": S.make_weights(310, True, 8.0, 1.0), "fine": S.make_weights(1310, True, 8.0, 1.0)},
               grid=S.make_grid(seed=11, shape=(36, 40, 24), occupancy=0.5, voxel_size=0.06), code_table=S.make_codes(312),
               k=k_src)
    rays = inp["rays_list"]
    src_rays = []
    for j, r in enumerate(rays[1:3]):
        r = r.clone()
        r[:, 6:8] = r[:, 6:8] / np.float32(k_src) if j == 0 else r[:, 6:8]   # the source's own depth range
        src_rays.append(r)
    return c, inp, [base, src], [0, 0, 0, 1, 1], rays + src_rays, [0, 4, 4, 4, 6]


@pytest.mark.skipif(not R.available(), reason="oracle/_ref not built (needs the reference checkout at build time)")
@pytest.mark.parametrize("k_src", [1.0, 8.0, 0.125])
def test_against_the_reference_called_per_set(k_src):
    """The reference's inference_from_model with each set's own scene modules, its sample_pdf on the set's coarse
    depths, and its volume_rendering_multi on [z_i * k_i], [sigma_i / k_i] (k a float32 scalar, the kernels' rounding):
    every key of both passes equal to tests/compose_oracle.py on the same fp32 inputs."""
    from tests import dropin_fixture as F
    c, inp, scenes, set_scene, rays_list, ids = _two_scene_case(k_src)
    boxes = [cases.box_affine(b) for b in inp["boxes"]]
    S_, K = c["n_samples"], c["n_importance"]
    want = CO.render_rays_multi_scenes([dict(s, grid=_grid(s["grid"])) for s in scenes], set_scene, rays_list, ids,
                                       n_samples=S_, n_importance=K, white_back=c["white_back"], skip_boxes=boxes)
    F.purge_reference_modules()
    R.install(cuda_noop=True)
    try:
        from models.rendering import sample_pdf
        from render_tools.multi_rendering import inference_from_model, volume_rendering_multi
        mods = []
        for s in scenes:
            models, emb = R.ref_render_setup(s["weights"], s["grid"])
            code_lib = types.SimpleNamespace(embedding_instance=torch.nn.Embedding.from_pretrained(s["code_table"]))
            mods.append((models, emb, code_lib))
        ks = [torch.tensor(scenes[j]["k"], dtype=torch.float32) for j in set_scene]
        z_steps = torch.linspace(0, 1, S_)
        z_c = [(r[:, 6:7] * (1 - z_steps) + r[:, 7:8] * z_steps).expand(r.shape[0], S_) for r in rays_list]

        def fields(typ, zs):
            rgbs, sigmas = [], []
            for i, z in enumerate(zs):
                models, emb, code_lib = mods[set_scene[i]]
                r = rays_list[i]
                xyz = r[:, None, 0:3] + r[:, None, 3:6] * z[:, :, None]
                with torch.no_grad():
                    rgb, sigma = inference_from_model(models[typ], emb["xyz"], emb["dir"](r[:, 3:6]), code_lib, xyz, z,
                                                      1 << 15, ids[i])
                if ids[i] == 0:
                    sigma[O.points_in_boxes(xyz, boxes)] = -1e5
                rgbs.append(rgb)
                sigmas.append(sigma)
            return rgbs, sigmas

        def frame_axis(zs, sigmas):
            scaled = [k != 1 for k in ks]
            return ([z * k if s else z for z, k, s in zip(zs, ks, scaled)],
                    [g / k if s else g for g, k, s in zip(sigmas, ks, scaled)])

        got = {}
        rgbs, sigmas = fields("coarse", z_c)
        zf, sf = frame_axis(z_c, sigmas)
        volume_rendering_multi(got, "coarse", zf, rgbs, sf, 0, c["white_back"],
                               [torch.ones_like(s) * i for i, s in enumerate(sf)])
        z_fine = []
        for i, z in enumerate(z_c):
            w_i = got["weights_coarse"][got["obj_ids_coarse"] == i].view(z.shape[0], S_)
            z_new = sample_pdf(0.5 * (z[:, :-1] + z[:, 1:]), w_i[:, 1:-1], K, det=True)
            z_fine.append(torch.sort(torch.cat([z, z_new], -1), -1)[0])
        rgbs, sigmas = fields("fine", z_fine)
        zf, sf = frame_axis(z_fine, sigmas)
        volume_rendering_multi(got, "fine", zf, rgbs, sf, 0, c["white_back"])
    finally:
        F.purge_reference_modules()
        R.cuda_noop(not torch.cuda.is_available())
    assert sorted(got) == sorted(k for k in want if "_sets_" not in k)
    for k in got:
        assert torch.equal(got[k], want[k]), (k, (got[k] - want[k]).abs().max().item())


def test_a_source_set_alone_keeps_its_opacity_at_a_power_of_two_k():
    """With k = 8 the rescale is exact (z * 8, sigma / 8 and their product sigma * delta are exact in float32): a source
    set alone on its rays gives bit for bit the weights, opacity and colour of the same set at k = 1, and 8 times its
    depths."""
    _, _, scenes, _, rays_list, _ = _two_scene_case(8.0)
    sc = dict(scenes[1], grid=_grid(scenes[1]["grid"]))
    at1 = CO.render_rays_multi_scenes([dict(sc, k=1.0)], [0], [rays_list[3]], [4], n_samples=32, n_importance=32)
    at8 = CO.render_rays_multi_scenes([dict(sc, k=1.0), dict(sc, k=8.0)], [1], [rays_list[3]], [4], n_samples=32,
                                      n_importance=32)
    assert (at1["opacity_fine"] > 0.1).any()
    for typ in ("coarse", "fine"):
        for k in ("weights", "opacity", "rgb", "opacity_sets", "rgb_sets"):
            assert torch.equal(at8[f"{k}_{typ}"], at1[f"{k}_{typ}"]), (k, typ)
        for k in ("z_vals", "depth", "depth_sets"):
            assert torch.equal(at8[f"{k}_{typ}"], 8 * at1[f"{k}_{typ}"]), (k, typ)


# ------------------------------------------------------------------------------------------------
# editing.import_sets: the pose of an object taken from another scene
# ------------------------------------------------------------------------------------------------
def _center_pose_from_avg():
    """The reference's center_pose_from_avg where oracle/_ref is built, else its float64 restatement."""
    if R.available():
        from tests import dropin_fixture as F
        F.purge_reference_modules()
        R.install(cuda_noop=True)
        try:
            from datasets.geo_utils import center_pose_from_avg
            return center_pose_from_avg
        finally:
            F.purge_reference_modules()
            R.cuda_noop(not torch.cuda.is_available())

    def center_pose_from_avg(pose_avg, pose):
        A, P = np.eye(4), np.eye(4)
        A[:3], P[:3] = pose_avg, pose[:3]
        return np.linalg.inv(A) @ P
    return center_pose_from_avg


def _rigid(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    T = np.eye(4)
    T[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                 [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                 [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
    T[:3, 3] = rng.normal(size=3) * 2
    return T


def test_import_sets_pose_against_a_float64_restatement(monkeypatch):
    from object_nerf_b200 import editing
    mod = types.ModuleType("fake_source_renderer")
    mod.center_pose_from_avg = _center_pose_from_avg()
    monkeypatch.setitem(sys.modules, mod.__name__, mod)

    class Source:
        pass
    Source.__module__ = mod.__name__
    rng = np.random.default_rng(3)
    sources = []
    for center, s in (([0.4, -1.2, 0.3], 2.0), ([3.0, 0.5, -0.7], 16.0)):
        src = Source()
        src.pose_avg = np.concatenate([np.eye(3), np.array(center)[:, None]], 1)   # editable_renderer.py:64-66
        src.scale_factor = s
        src.boxes = {4: object(), 6: object()}
        src.get_object_bbox_helper = src.boxes.__getitem__
        src.system = types.SimpleNamespace(models={}, embeddings={"xyz": None}, code_library=None)
        sources.append(src)
    monkeypatch.setattr(editing, "_is_voxel", lambda emb: True)
    Twc = _rigid(rng)
    places = [_rigid(rng) for _ in range(3)]
    imports = [(sources[0], 4, places[0]), (sources[1], 6, places[1]), (sources[1], 4, places[2])]
    sets = editing.import_sets(Twc[:3], imports, 0.05)
    assert len(sets) == 3
    for (obj_id, Toc, box, enl, scene), (src, oid, place) in zip(sets, imports):
        A = np.eye(4)
        A[:3] = src.pose_avg
        want = np.linalg.inv(A) @ np.linalg.inv(place) @ Twc
        want[:3, 3] /= src.scale_factor
        assert obj_id == oid and box is src.boxes[oid] and enl == 0.05
        assert Toc.dtype == torch.float32 and Toc.shape == (3, 4)
        assert torch.equal(Toc, torch.from_numpy(want[:3]).float()) or np.abs(Toc.numpy() - want[:3]).max() < 1e-6
        assert isinstance(scene, editing.Scene) and scene.scale_factor == src.scale_factor
    assert sets[1][4] is sets[2][4] and sets[0][4] is not sets[1][4]    # one Scene per source renderer
