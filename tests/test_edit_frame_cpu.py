"""CPU checks of the edited-frame entry (include/onerf_ext.h: onerf_render_edit_frame, onerf_render_edit_workspace_bytes)
and of object_nerf_b200.editing's host side: exports and declarations, the workspace arithmetic, argument refusals before
any CUDA call, and (with oracle/_ref built) the ray sets editing.render_edit / render_origin hand to render_frame against
what the unmodified EditableRenderer hands to get_rays / render_rays_multi."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import ref_loader as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
a256 = lambda x: (x + 255) // 256 * 256


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def _ext_declarations():
    src = open(os.path.join(ROOT, "include", "onerf_ext.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return {m.group(1): [p.strip() for p in m.group(2).split(",")]
            for m in re.finditer(r"\b(onerf_[a-z0-9_]+)\s*\(([^)]*)\)", src)}


def test_exports_and_declarations(lib):
    from object_nerf_b200 import _lib
    decl = _ext_declarations()
    assert decl["onerf_render_edit_frame"] == ["onerf_ctx* ctx", "const onerf_render_edit_args* args", "void* stream"]
    assert decl["onerf_render_edit_workspace_bytes"] == ["int chunk_rays", "int n_obj", "int n_samples", "int n_importance"]
    for name in ("onerf_render_edit_frame", "onerf_render_edit_workspace_bytes"):
        assert name in _lib.EXPORTS_EXT and name not in _lib.EXPORTS and hasattr(lib, name), name
        assert len(getattr(lib, name).argtypes) == len(decl[name]), name
    assert sorted(set(_lib.EXPORTS_EXT)) == sorted(decl)


def test_struct_layout_matches_the_header():
    """The ctypes structs list the header's members in order; their C sizes follow from the members' alignment."""
    from object_nerf_b200 import _lib
    src = open(os.path.join(ROOT, "include", "onerf_ext.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    for struct, cls in (("onerf_edit_set", _lib.EditSet), ("onerf_render_edit_args", _lib.RenderEditArgs)):
        body = re.search(r"typedef struct " + struct + r" \{(.*?)\} " + struct + ";", src, flags=re.S).group(1)
        names = []
        for decl in body.split(";"):
            decl = re.sub(r"\[[^\]]*\]", "", decl).strip()
            if decl:
                first, *rest = decl.split(",")
                names += [first.split()[-1].lstrip("*")] + [r.strip().lstrip("*") for r in rest]
        assert [f[0] for f in cls._fields_] == names, struct
    assert _lib.EditSet.box.offset == 56 and ctypes.sizeof(_lib.EditSet) == 64   # 4 + 48 bytes, padded to the pointer
    assert _lib.RenderEditArgs.pixel_begin.offset % 8 == 0 and _lib.RenderEditArgs.near.offset % 8 == 0


def test_workspace_bytes(lib):
    f = lib.onerf_render_edit_workspace_bytes
    assert f(0, 3, 64, 64) == 0 and f(-5, 3, 64, 64) == 0
    assert f(4096, 0, 64, 64) == 0 and f(4096, 3, 0, 64) == 0 and f(4096, 3, 64, -1) == 0
    for n, no, s, si in ((1, 1, 2, 0), (1000, 3, 64, 64), (4096, 3, 64, 0), (65536, 3, 64, 64), (77, 5, 32, 96)):
        tc, tf, nf = no * s, no * (s + si), n if si > 0 else 0
        rays = a256(no * n * 32)
        coarse = 3 * a256(n * tc * 4) + a256(n * 12) + 2 * a256(n * 4)
        fine = 2 * a256(nf * tf * 4) + a256(nf * 12) + 2 * a256(nf * 4)
        want = rays + coarse + fine + a256(lib.onerf_render_multi_workspace_bytes(n, no, s, si))
        assert f(n, no, s, si) == want, (n, no, s, si)
    grow = [f(n, 3, 64, 64) for n in (1, 1000, 4096, 65536)]
    assert grow == sorted(grow) and len(set(grow)) == len(grow)


class _Args:
    """A valid-looking argument block whose device pointers are never dereferenced (every refusal comes first)."""

    def __init__(self, lib):
        from object_nerf_b200 import _lib
        self.lib, self._lib = lib, _lib
        self.box = _lib.BoxHost()
        for i in range(3):
            self.box.pose_avg[5 * i] = self.box.axis_align[5 * i] = 1.0
        self.box.bounds[3] = self.box.bounds[4] = self.box.bounds[5] = 1.0
        self.sets = (_lib.EditSet * 3)()
        for i, oid in enumerate((0, 4, 4)):
            self.sets[i].obj_id = oid
            for r in range(3):
                self.sets[i].Toc[4 * r + r] = 1.0
            if oid:
                self.sets[i].box = ctypes.pointer(self.box)
        self.grid = _lib.Grid()
        a = self.a = _lib.RenderEditArgs()
        a.sets_host, a.n_obj, a.H, a.W, a.focal = self.sets, 3, 48, 64, 50.0
        a.pixel_begin, a.pixel_end = 0, 48 * 64
        a.near, a.far, a.scale_factor = 0.1, 6.0, 2.0
        a.n_samples, a.n_importance = 64, 64
        a.grid = ctypes.pointer(self.grid)
        a.packed_coarse = a.packed_fine = a.code_table = 1 << 20
        a.n_codes, a.precision, a.chunk_rays = 8, _lib.PREC_BF16, 1000
        a.workspace = 1 << 30
        a.workspace_bytes = lib.onerf_render_edit_workspace_bytes(1000, 3, 64, 64)

    def call(self, ctx=True):
        fake_ctx = ctypes.c_void_p(1 << 21) if ctx else None
        return self.lib.onerf_render_edit_frame(fake_ctx, ctypes.byref(self.a), None), self.lib.onerf_last_error()


REFUSALS = {
    "tile_negative": (lambda t: setattr(t.a, "pixel_begin", -1), b"tile outside the frame"),
    "tile_reversed": (lambda t: (setattr(t.a, "pixel_begin", 10), setattr(t.a, "pixel_end", 9)), b"tile outside the frame"),
    "tile_past_frame": (lambda t: setattr(t.a, "pixel_end", 48 * 64 + 1), b"tile outside the frame"),
    "chunk_zero": (lambda t: setattr(t.a, "chunk_rays", 0), b"chunk_rays < 1"),
    "chunk_negative": (lambda t: setattr(t.a, "chunk_rays", -4096), b"chunk_rays < 1"),
    "object_without_box": (lambda t: setattr(t.sets[1], "box", None), b"an object set needs its box"),
    "scene_with_box": (lambda t: setattr(t.sets[0], "box", ctypes.pointer(t.box)), b"the scene set takes no box"),
    "zero_height": (lambda t: setattr(t.a, "H", 0), b"bad camera"),
    "negative_width": (lambda t: setattr(t.a, "W", -64), b"bad camera"),
    "zero_focal": (lambda t: setattr(t.a, "focal", 0.0), b"bad camera"),
    "nan_focal": (lambda t: setattr(t.a, "focal", float("nan")), b"bad camera"),
    "scale_factor": (lambda t: setattr(t.a, "scale_factor", 0.0), b"scale_factor"),
    "no_sets": (lambda t: setattr(t.a, "n_obj", 0), b"bad shape"),
    "null_sets": (lambda t: setattr(t.a, "sets_host", None), b"null argument"),
    "one_sample": (lambda t: setattr(t.a, "n_samples", 1), b"bad shape"),
    "negative_importance": (lambda t: setattr(t.a, "n_importance", -1), b"bad shape"),
    "id_outside_codes": (lambda t: setattr(t.sets[2], "obj_id", 8), b"object id outside the code table"),
    "negative_id": (lambda t: setattr(t.sets[2], "obj_id", -1), b"object id outside the code table"),
    "no_packed_fine": (lambda t: setattr(t.a, "packed_fine", None), b"needs packed_fine"),
    "no_grid": (lambda t: setattr(t.a, "grid", None), b"null input"),
    "no_code_table": (lambda t: setattr(t.a, "code_table", None), b"null input"),
    "boxes_without_pointer": (lambda t: setattr(t.a, "n_boxes", 2), b"n_boxes > 0 with null boxes"),
    "misaligned_workspace": (lambda t: setattr(t.a, "workspace", (1 << 30) + 16), b"256-byte aligned"),
    "null_workspace": (lambda t: setattr(t.a, "workspace", None), b"256-byte aligned"),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_refusals_without_a_device(lib, case):
    t = _Args(lib)
    REFUSALS[case][0](t)
    rc, msg = t.call()
    assert rc == -1, (case, rc, msg)
    assert msg.startswith(b"onerf_render_edit_frame: ") and REFUSALS[case][1] in msg, (case, msg)


def test_limits_and_workspace_refusals_without_a_device(lib):
    t = _Args(lib)
    t.a.n_samples, t.a.n_importance = 1024, 1025
    t.a.workspace_bytes = 1 << 40
    rc, msg = t.call()
    assert rc == -2 and b"2048" in msg, msg
    t = _Args(lib)
    t.a.workspace_bytes -= 1
    rc, msg = t.call()
    assert rc == -4 and b"workspace too small" in msg, msg
    rc, msg = _Args(lib).call(ctx=False)
    assert rc == -1 and b"null argument" in msg


def test_render_frame_refuses_unknown_keys_before_the_library():
    from object_nerf_b200 import editing
    for keys, ni in ((["rgb_fine"], 0), (["obj_ids_fine"], 64), (["rgb"], 64)):
        with pytest.raises(KeyError):
            editing.render_frame({}, {"xyz": None}, None, 4, 4, 1.0, [], 0.1, 1.0, 1.0, keys=keys, N_importance=ni)
    assert editing.result_keys(0) == ["weights_coarse", "opacity_coarse", "z_vals_coarse", "rgb_coarse", "depth_coarse",
                                      "obj_ids_coarse"]
    assert editing.result_keys(64)[6:] == ["weights_fine", "opacity_fine", "z_vals_fine", "rgb_fine", "depth_fine"]


# ------------------------------------------------------------------------------------------------
# editing.render_edit / render_origin against the unmodified EditableRenderer, render paths recorded
# ------------------------------------------------------------------------------------------------
H, W = 6, 8


def _renderer(er, conf, paths, monkeypatch):
    """The reference's EditableRenderer on the dropin_fixture scene; load_model is skipped (nothing here renders)."""
    monkeypatch.setattr(er.EditableRenderer, "load_model", lambda self, *a: setattr(
        self, "system", type("Sys", (), {"models": "models", "embeddings": "embeddings", "code_library": "codes"})()))
    cfg = R.to_attr({"chunk": 4096, "img_wh": [W, H], "ckpt_path": paths["ckpt"], "ckpt_config_path": paths["snapshot"],
                     "ckpt_config": conf})
    r = er.EditableRenderer(config=cfg)
    r.load_frame_meta()
    return r


def _edit(r, obj_ids, moved):
    for obj_id in obj_ids:
        r.initialize_object_bbox(obj_id)
    r.remove_scene_object_by_ids(list(obj_ids))
    processed = []
    for obj_id in obj_ids:
        dup = int(np.sum(np.array(processed) == obj_id))
        pose = np.eye(4)
        if moved:
            c, s = np.cos(0.1 + 0.2 * dup), np.sin(0.1 + 0.2 * dup)
            pose[:2, :2] = [[c, -s], [s, c]]
            pose[:2, 3] = [0.05, 0.3] if dup == 0 else [-0.05, -0.2]
        r.set_object_pose_transform(obj_id, pose, dup)
        processed.append(obj_id)


CASES = {
    "plain_edit": dict(obj_ids=[4], moved=True, kw={}),
    "duplicate": dict(obj_ids=[4, 4], moved=True, kw={}),
    "two_objects": dict(obj_ids=[4, 6], moved=False, kw={}),
    "bg_only": dict(obj_ids=[4, 4], moved=True, kw={"render_bg_only": True}),
    "obj_only": dict(obj_ids=[4, 6], moved=True, kw={"render_obj_only": True}),
}


@pytest.mark.skipif(not R.available(), reason="oracle/_ref not built (needs the reference checkout at build time)")
@pytest.mark.parametrize("case", sorted(CASES) + ["origin"])
def test_ray_sets_match_the_unmodified_renderer(tmp_path, monkeypatch, case):
    from object_nerf_b200 import editing
    from tests import dropin_fixture as F
    F.purge_reference_modules()
    R.install(cuda_noop=True)
    try:
        conf, paths = F.write_scene(str(tmp_path))
        from render_tools import editable_renderer as er
        got_rays, got_multi = [], []

        def rec_get_rays(directions, c2w):
            got_rays.append(c2w.clone())
            return ref_get_rays(directions, c2w)
        ref_get_rays = er.get_rays
        monkeypatch.setattr(er, "get_rays", rec_get_rays)

        def rec_multi(**kw):
            got_multi.append(kw)
            n = kw["rays_list"][0].shape[0]
            return {"rgb_fine": torch.zeros(n, 3)}
        monkeypatch.setattr(er, "render_rays_multi", rec_multi)
        frames = []
        monkeypatch.setattr(editing, "render_frame", lambda *a, **k: frames.append((a, k)) or {"rgb_fine": torch.zeros(H * W, 3)})
        pose_idx = 1
        results = {}
        for side in ("reference", "editing"):
            r = _renderer(er, conf, paths, monkeypatch)
            spec = CASES.get(case, dict(obj_ids=[4], moved=True, kw={}))
            _edit(r, spec["obj_ids"], spec["moved"])
            r.bbox_enlarge = 0.02
            Twc = r.get_camera_pose_by_frame_idx(pose_idx)
            fov = r.fov_x_deg_dataset
            if side == "reference":
                if case == "origin":
                    monkeypatch.setattr(er.EditableRenderer, "scene_inference", lambda self, rays: rec_multi(
                        rays_list=[rays], obj_instance_ids=[0], background_skip_bbox=None))
                    out = er.EditableRenderer.render_origin(r, H, W, Twc.copy(), fov)
                else:
                    out = er.EditableRenderer.render_edit(r, H, W, Twc.copy(), fov, show_progress=False, **spec["kw"])
            else:
                out = (editing.render_origin(r, H, W, Twc.copy(), fov) if case == "origin" else
                       editing.render_edit(r, H, W, Twc.copy(), fov, show_progress=False, **spec["kw"]))
            results[side] = (r, out)
        (rr, ref_out), (er_, ed_out) = results["reference"], results["editing"]
        assert len(got_multi) == 1 and len(frames) == 1
        a, k = frames[0]
        sets = a[6]
        assert [s[0] for s in sets] == list(got_multi[0]["obj_instance_ids"])
        assert len(got_rays) == len(sets)
        for (obj_id, Toc, box, enl), want in zip(sets, got_rays):
            assert Toc.dtype == torch.float32 and torch.equal(Toc, want.float()), (obj_id, Toc, want)
            if obj_id == 0:
                assert box is None
            else:
                assert box is er_.object_bbox_ray_helpers[str(obj_id)] and enl == rr.bbox_enlarge
                assert np.array_equal(box.bbox_bounds, rr.object_bbox_ray_helpers[str(obj_id)].bbox_bounds)
        want_skip = got_multi[0]["background_skip_bbox"]
        got_skip = k["background_skip_bbox"]
        assert (want_skip is None) == (got_skip is None)
        if want_skip is not None:
            assert sorted(want_skip) == sorted(got_skip)
            for key in want_skip:
                assert got_skip[key] is er_.object_bbox_ray_helpers[key]
        assert rr.active_object_ids == er_.active_object_ids
        assert a[3:5] == (H, W) and a[5] == pytest.approx((W / 2) / np.tan(np.deg2rad(er_.fov_x_deg_dataset) / 2), rel=1e-12)
        assert a[7:10] == (rr.near, rr.far, rr.scale_factor)
        model = conf["model"]
        assert (k["N_samples"], k["N_importance"], k["use_disp"]) == (model["N_samples"], model["N_importance"],
                                                                     model["use_disp"])
        assert set(ed_out) == set(ref_out)
    finally:
        F.purge_reference_modules()
        R.cuda_noop(not torch.cuda.is_available())
