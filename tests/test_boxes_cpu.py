"""CPU checks of onerf_render_boxes (every object rendered inside its own box): its declarations, exports and struct
layout, the workspace arithmetic (independent of K and the image), every refusal (the checks run before any CUDA
call); frames.read_boxes on ScanNet-style files and a ToyDesk JSON against hand-computed boxes and, where oracle/_ref is
built, the reference's own BBoxRayHelper; and a use_bbox test split loading as without use_bbox."""
import ctypes
import json
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import ref_loader as R
from tests import dropin_fixture as DF
from tests import frames_cases as FC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = {
    "onerf_render_boxes_workspace_bytes": ["int chunk_rays", "int n_samples", "int n_importance"],
    "onerf_render_boxes": ["onerf_ctx* ctx", "const onerf_render_boxes_args* args", "void* stream"],
}


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def test_entries_are_exported_and_declared(lib):
    from object_nerf_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "onerf_ext.h")).read(), flags=re.S)
    decl = {m.group(1): [p.strip() for p in m.group(2).split(",")]
            for m in re.finditer(r"\b(onerf_[a-z0-9_]+)\s*\(([^)]*)\)", src)}
    for name, params in ENTRIES.items():
        assert decl[name] == params
        assert name in _lib.EXPORTS_EXT and name not in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == len(params)
    assert _lib.ABI_VERSION == 2 and lib.onerf_abi_version() == 2
    header = open(os.path.join(ROOT, "include", "onerf_ext.h")).read()
    assert int(re.search(r"#define ONERF_BOXES_MAX (\d+)", header).group(1)) == _lib.BOXES_MAX


@pytest.mark.parametrize("cls,cname", [("BoxMaps", "onerf_box_maps"), ("RenderBoxesArgs", "onerf_render_boxes_args")])
def test_struct_layout_matches_the_header(tmp_path, cls, cname):
    from object_nerf_b200 import _lib
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    cls = getattr(_lib, cls)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "onerf_ext.h"', "int main(void) {",
             f'printf("size %zu\\n", sizeof({cname}));']
    lines += [f'printf("{f[0]} %zu\\n", offsetof({cname}, {f[0]}));' for f in cls._fields_]
    lines.append("return 0; }")
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", str(tmp_path / "l")],
                   check=True)
    got = dict(line.rsplit(" ", 1) for line in subprocess.run([str(tmp_path / "l")], capture_output=True, text=True,
                                                              check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(cls)
    for f in cls._fields_:
        assert int(got[f[0]]) == getattr(cls, f[0]).offset, f[0]


def _a256(nbytes):
    return (nbytes + 255) // 256 * 256


def _ws_bytes(chunk, S, I):
    """The workspace layout restated, in bytes: the chunk's rays and hit bits, the list (one offset per 4096 rows, the
    count, the row of each slot), and per listed row its ray, coarse depths and weights, fine depths, code row, per-ray
    constants and object field."""
    SF, nf = S + I, chunk if I > 0 else 0
    blocks = (chunk + 4095) // 4096
    parts = [32 * chunk, chunk, 4 * blocks, 4, 4 * chunk, 32 * chunk, 4 * chunk * S, 4 * chunk * S, 4 * nf * SF,
             4 * chunk * 64, 4 * chunk * 448, 16 * chunk * SF]
    return sum(_a256(b) for b in parts)


@pytest.mark.parametrize("chunk,S,I", [(1, 2, 0), (1000, 64, 64), (4099, 64, 64), (777, 128, 0), (65536, 64, 1984)])
def test_workspace_arithmetic(lib, chunk, S, I):
    assert lib.onerf_render_boxes_workspace_bytes(chunk, S, I) == _ws_bytes(chunk, S, I)


def test_workspace_is_zero_for_a_bad_shape(lib):
    f = lib.onerf_render_boxes_workspace_bytes
    for args in ((0, 64, 0), (10, 1, 0), (10, 64, -1)):
        assert f(*args) == 0, args


def test_python_chunk_keeps_the_workspace_within_its_budget(lib):
    from object_nerf_b200 import rendering
    for S, I in ((64, 64), (128, 1920)):
        c = rendering._boxes_chunk(1 << 20, S, I)
        assert 1 <= c <= 1 << 20
        assert lib.onerf_render_boxes_workspace_bytes(c, S, I) <= rendering.BOXES_WORKSPACE_BUDGET
        assert lib.onerf_render_boxes_workspace_bytes(c + 1, S, I) > 0.9 * rendering.BOXES_WORKSPACE_BUDGET


_IDS = (ctypes.c_int * 64)(*([3, 0, 7] + [1] * 61))
_C2W = (ctypes.c_float * 12)(1, 0, 0, 0.5, 0, 1, 0, 0, 0, 0, 1, 2)


def _boxes_host():
    from object_nerf_b200 import _lib
    boxes = (_lib.BoxHost * 64)()
    for b in boxes:
        for i in range(3):
            b.pose_avg[5 * i] = b.axis_align[5 * i] = 1.0
            b.bounds[i], b.bounds[3 + i] = -0.5, 0.5
    return boxes


_BOXES = _boxes_host()


def _args(lib):
    """An argument block that passes every check; the pointers are never dereferenced by the refusals."""
    from object_nerf_b200 import _lib
    a = _lib.RenderBoxesArgs()
    a.packed_coarse, a.packed_fine, a.precision = 0x10000, 0x10000, _lib.PREC_BF16
    a.n_samples, a.n_importance = 64, 64
    a.H, a.W, a.focal, a.c2w_host = 24, 32, 30.0, _C2W
    a.boxes_host, a.n_boxes = _BOXES, 3
    a.scale_factor, a.near, a.far = 2.0, 0.3, 6.0
    a.ids_host, a.code_table, a.n_codes_table = ctypes.cast(_IDS, ctypes.POINTER(ctypes.c_int)), 0x10000, 8
    a.pixel_begin, a.pixel_end, a.chunk_rays = 10, 700, 32
    a.coarse.opacity = a.fine.rgb = 0x20000
    a.hit = 0x30001
    a.workspace, a.workspace_bytes = 0x100000, lib.onerf_render_boxes_workspace_bytes(32, 64, 64)
    return a


def _set(a, path, value):
    obj, _, field = path.rpartition("__")
    setattr(getattr(a, obj) if obj else a, field, value)


def _grid(**over):
    from object_nerf_b200 import _lib
    g = _lib.Grid()
    g.table, g.idx_map, g.voxel_offset, g.voxel_size, g.voxel_shape = 0x10000, 0x10000, 0x10000, 0x10000, 0x10000
    for k, v in over.items():
        setattr(g, k, v)
    return g


_BAD_C2W = (ctypes.c_float * 12)(1, 0, 0, float("nan"), 0, 1, 0, 0, 0, 0, 1, 2)


def _bad_box(field, i, value):
    boxes = _boxes_host()
    getattr(boxes[1], field)[i] = value
    return boxes


@pytest.mark.parametrize("change,msg,rc", [
    ({"n_boxes": 0}, b"n_boxes outside", -1),
    ({"n_boxes": 65}, b"n_boxes outside", -1),
    ({"boxes_host": None}, b"null boxes_host", -1),
    ({"ids_host": None}, b"null boxes_host / ids_host", -1),
    ({"code_table": None}, b"code_table", -1),
    ({"n_codes_table": 7}, b"outside the code table", -1),
    ({"boxes_host": _bad_box("bounds", 4, float("inf"))}, b"non-finite box", -1),
    ({"boxes_host": _bad_box("pose_avg", 3, float("nan"))}, b"non-finite box", -1),
    ({"boxes_host": _bad_box("axis_align", 11, float("-inf"))}, b"non-finite box", -1),
    ({"c2w_host": None}, b"null c2w_host", -1),
    ({"c2w_host": _BAD_C2W}, b"non-finite camera", -1),
    ({"focal": float("nan")}, b"bad camera", -1),
    ({"focal": 0.0}, b"bad camera", -1),
    ({"H": 0}, b"bad camera", -1),
    ({"scale_factor": 0.0}, b"scale_factor", -1),
    ({"scale_factor": float("inf")}, b"scale_factor", -1),
    ({"pixel_begin": -1}, b"pixel range", -1),
    ({"pixel_end": 24 * 32 + 1}, b"pixel range", -1),
    ({"pixel_begin": 50, "pixel_end": 49}, b"pixel range", -1),
    ({"chunk_rays": 0}, b"chunk_rays", -1),
    ({"n_samples": 1}, b"bad shape", -1),
    ({"n_importance": -1}, b"bad shape", -1),
    ({"n_importance": 1985}, b"S + K > 2048", -2),
    ({"packed_coarse": None}, b"packed_coarse", -1),
    ({"packed_fine": None}, b"packed_fine", -1),
    ({"grid": ctypes.pointer(_grid(table=None))}, b"grid buffer", -1),
    ({"grid": ctypes.pointer(_grid(table=0x10004))}, b"grid buffer", -1),
    ({"grid": ctypes.pointer(_grid(voxel_shape=None))}, b"grid buffer", -1),
    ({"precision": 7}, b"unknown precision", -1),
    ({"n_importance": 0}, b"fine maps without a fine pass", -1),
    ({"code_table": 0x10004}, b"16-byte aligned", -1),
    ({"coarse__rgb": 0x10002}, b"4-byte aligned", -1),
    ({"fine__depth": 0x10001}, b"4-byte aligned", -1),
    ({"workspace": None}, b"256-byte aligned", -1),
    ({"workspace": 0x100010}, b"256-byte aligned", -1),
    ({"workspace_bytes": 1000}, b"workspace too small", -1),
])
def test_refusals(lib, change, msg, rc):
    a = _args(lib)
    for path, value in change.items():
        _set(a, path, value)
    assert lib.onerf_render_boxes(ctypes.c_void_p(1), ctypes.byref(a), None) == rc
    err = lib.onerf_last_error()
    assert msg in err and err.startswith(b"onerf_render_boxes:"), (change, err)


def test_null_context_and_args(lib):
    a = _args(lib)
    assert lib.onerf_render_boxes(None, ctypes.byref(a), None) == -1
    assert b"null argument" in lib.onerf_last_error()
    assert lib.onerf_render_boxes(ctypes.c_void_p(1), None, None) == -1
    assert b"null argument" in lib.onerf_last_error()
    a.grid = ctypes.pointer(_grid())
    a.workspace_bytes = 1000               # a valid grid passes up to the workspace size
    assert lib.onerf_render_boxes(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
    assert b"workspace too small" in lib.onerf_last_error()


def test_near_far_are_not_read_and_a_coarse_only_render_takes_more_than_2048_samples(lib):
    """near / far do not enter box mode (each ray's come from its box), so non-finite ones pass; the S + K <= 2048 limit
    is the importance sampler's and applies, as in onerf_render_rays_fwd, only with a fine pass.  Both calls get as far
    as the workspace check."""
    for change in ({"near": float("inf"), "far": float("nan")},
                   {"n_samples": 4096, "n_importance": 0, "fine__rgb": None}):
        a = _args(lib)
        for path, value in change.items():
            _set(a, path, value)
        a.workspace_bytes = 1000
        assert lib.onerf_render_boxes(ctypes.c_void_p(1), ctypes.byref(a), None) == -1, change
        assert b"workspace too small" in lib.onerf_last_error(), change


def test_python_refusals():
    import torch

    from object_nerf_b200 import rendering
    models = {"coarse": torch.nn.Linear(1, 1)}
    box = object()        # the refusals come before any box is read
    kw = dict(N_samples=64, N_importance=0, use_disp=False, scale_factor=1.0, near=0.1, far=1.0)
    with pytest.raises(ValueError, match="1 to 64 boxes"):
        rendering.render_boxes(models, {}, None, 4, 4, 1.0, np.eye(4), [], [], **kw)
    with pytest.raises(ValueError, match="one id each"):
        rendering.render_boxes(models, {}, None, 4, 4, 1.0, np.eye(4), [box, box], [1], **kw)
    with pytest.raises(ValueError, match="chunk"):
        rendering.render_boxes(models, {}, None, 4, 4, 1.0, np.eye(4), [box], [1], chunk=0, **kw)
    with pytest.raises(KeyError, match="no such map"):
        rendering.render_boxes(models, {}, None, 4, 4, 1.0, np.eye(4), [box], [1], keys=("rgb",), **kw)
    with pytest.raises(KeyError, match="no such map"):
        rendering.render_boxes(models, {}, None, 4, 4, 1.0, np.eye(4), [box], [1], keys=("opacity_instance_fine",),
                               **kw)


# ------------------------------------------------------------------------------------------------
# frames.read_boxes
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scannet(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("boxes_scannet"))
    conf, _ = DF.write_scene(root)
    return conf


def test_read_boxes_scannet_matches_hand_computed_boxes(scannet):
    from object_nerf_b200 import frames
    extra = scannet["dataset_extra"]
    ang = 0.2
    A = np.eye(4)
    A[:3, :3] = [[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]]
    A[:3, 3] = [0.1, -0.05, 0.02]
    A = np.array([float(f"{v:.8f}") for v in A.reshape(-1)]).reshape(4, 4)     # as the file writes it
    b4, b6 = frames.read_boxes("scannet_base", extra, [4, 6])
    for b, c, size, i in ((b4, [0.25, 0.10, 0.05], [0.7, 0.6, 0.5], 4), (b6, [-0.35, -0.20, 0.0], [0.5, 0.5, 0.6], 6)):
        c, h = np.array(c), np.array(size) * 0.5
        assert np.array_equal(b.axis_align_mat, A)
        assert np.array_equal(b.bbox_bounds, np.array([c - h, c + h])) and np.array_equal(b.bbox_c, c)
        assert np.array_equal(b.pose_avg, np.eye(4)) and b.instance_id == i and b.scale_factor == 2.0
        assert b.scene_id == DF.SCENE_ID and b.dataset_name == "scannet_base"
    with pytest.raises(ValueError, match="no box for instance id 5"):
        frames.read_boxes("scannet_base", extra, [4, 5])
    with pytest.raises(ValueError, match="unknown dataset"):
        frames.read_boxes("replica", extra, [4])
    with pytest.raises(ValueError, match="needs scene_id"):
        frames.read_boxes("scannet_base", {k: v for k, v in extra.items() if k != "scene_id"}, [4])


def test_read_boxes_scannet_last_row_wins_and_the_strip_charset(tmp_path, scannet):
    from object_nerf_b200 import frames
    extra = dict(scannet["dataset_extra"], scans_dir=str(tmp_path / "scans"), bbox_dir=str(tmp_path / "bbox"))
    os.makedirs(tmp_path / "scans" / DF.SCENE_ID)
    os.makedirs(tmp_path / "bbox")
    # "e" and "a" are in the stripped character set: a trailing exponent digit stays, a leading "a" of a number goes
    vals = [1, 0, 0, 2e-5, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1]
    with open(tmp_path / "scans" / DF.SCENE_ID / f"{DF.SCENE_ID}.txt", "w") as f:
        f.write("colorHeight = 968\naxisAlignment = " + " ".join(repr(float(v)) for v in vals) + "  \n"
                "axisAlignment = 9 9 9 9 9 9 9 9 9 9 9 9 9 9 9 9\n")
    np.save(tmp_path / "bbox" / f"{DF.SCENE_ID}_bbox.npy",
            np.array([[0, 0, 0, 1, 1, 1, 4], [1, 2, 3, 2, 2, 2, 4], [5, 5, 5, 1, 1, 1, 6]], np.float64))
    (b,) = frames.read_boxes("scannet_base", extra, [4])
    assert np.array_equal(b.axis_align_mat, np.array(vals, np.float64).reshape(4, 4))
    assert np.array_equal(b.bbox_bounds, np.array([[0, 1, 2], [2, 3, 4]], np.float64))
    assert np.array_equal(b.bbox_c, np.array([1, 2, 3], np.float64))


def _toydesk(tmp_path):
    labels = [{"id": 2, "data": {"note": "no position"}},
              {"id": "2", "data": {"position": [0.1, -0.2, 0.3], "quaternion": [0.1, 0.2, -0.3, 0.9],
                                   "scale": [0.4, 0.5, 0.6]}},
              {"id": 2, "data": {"position": [9, 9, 9], "quaternion": [0, 0, 0, 1], "scale": [1, 1, 1]}},
              {"id": 5, "data": {"position": [0.0, 0.0, 0.0], "quaternion": [0, 0, 0, 1], "scale": [1, 2, 3]}}]
    path = tmp_path / "bbox.json"
    path.write_text(json.dumps({"labels": labels}))
    return {"bbox_dir": str(path), "scene_center": [0.2, -0.1, 0.05], "scale_factor": 16.0}


def test_read_boxes_toydesk_matches_hand_computed_boxes(tmp_path):
    from object_nerf_b200 import frames
    conf = _toydesk(tmp_path)
    b2, b5 = frames.read_boxes("toydesk", conf, [2, 5])
    q = np.array([0.1, 0.2, -0.3, 0.9])
    x, y, z, w = q / np.linalg.norm(q)
    Rm = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                   [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                   [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = Rm, [0.1, -0.2, 0.3]
    assert np.allclose(b2.axis_align_mat, np.linalg.inv(T), rtol=0, atol=1e-12)
    assert np.array_equal(b2.bbox_bounds, np.array([[-0.2, -0.25, -0.3], [0.2, 0.25, 0.3]]))
    assert np.array_equal(b2.bbox_c, np.array([0.1, -0.2, 0.3]))
    P = np.eye(4)
    P[:3, 3] = conf["scene_center"]
    assert np.array_equal(b2.pose_avg, P) and b2.scale_factor == 16.0 and b2.instance_id == 2
    assert np.array_equal(b5.axis_align_mat, np.eye(4))
    assert np.array_equal(b5.bbox_bounds, np.array([[-0.5, -1, -1.5], [0.5, 1, 1.5]]))
    with pytest.raises(ValueError, match="instance id 7"):
        frames.read_boxes("toydesk", conf, [7])


_ATTRS = ("scale_factor", "instance_id", "dataset_name", "axis_align_mat", "bbox_bounds", "bbox_c", "pose_avg")


def _same(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)
    return a == b and type(a) is type(b)


@pytest.mark.skipif(not R.available(), reason="oracle/_ref not built (needs the reference checkout at build time)")
def test_read_boxes_equals_the_references_bbox_ray_helper(tmp_path, scannet):
    """BBoxRayHelper(config, id) of the unmodified reference, attribute for attribute, bit for bit."""
    import yaml

    from object_nerf_b200 import frames
    R.install(cuda_noop=True)
    DF.purge_reference_modules()
    from utils.bbox_utils import BBoxRayHelper
    for name, extra, ids in (("scannet_base", scannet["dataset_extra"], [4, 6]), ("toydesk", _toydesk(tmp_path), [2, 5])):
        path = tmp_path / f"{name}.yml"
        path.write_text(yaml.safe_dump({"dataset_name": name, "dataset_extra": extra}))
        for i, got in zip(ids, frames.read_boxes(name, extra, ids)):
            ref = BBoxRayHelper(str(path), i)
            for k in _ATTRS + (("scene_id",) if name == "scannet_base" else ()):
                assert _same(getattr(got, k), getattr(ref, k)), (name, i, k)


# ------------------------------------------------------------------------------------------------
# a use_bbox test split
# ------------------------------------------------------------------------------------------------
def test_use_bbox_test_split_loads_as_without_it(tmp_path, monkeypatch):
    """FrameSet.load(..., split="test") with use_bbox (either use_bbox_only_for_test) builds the store from exactly the
    arrays of the same config without it; training with use_bbox and without use_bbox_only_for_test stays refused."""
    from object_nerf_b200 import frames
    monkeypatch.setattr(frames.FrameSet, "__init__", lambda self, device="cuda", **kw: self.__dict__.update(kw=kw))
    center = FC.write_scene(str(tmp_path))
    np.savetxt(os.path.join(tmp_path, "split", "test.txt"), [8, 0, 3], fmt="%d")
    kw = dict(FC.CONFIGS["i3_bg_obs"])
    plain = frames.FrameSet.load(FC.config(str(tmp_path), center, **kw), FC.IMG_WH, split="test").kw
    assert plain["poses"].shape[0] == 3
    for only_for_test in (True, False):
        conf = FC.config(str(tmp_path), center, **dict(kw, use_bbox=True, use_bbox_only_for_test=only_for_test))
        boxed = frames.FrameSet.load(conf, FC.IMG_WH, split="test").kw
        assert sorted(boxed) == sorted(plain)
        for k, v in plain.items():
            if isinstance(v, np.ndarray):
                assert v.dtype == boxed[k].dtype and np.array_equal(v, boxed[k]), k
            else:
                assert v == boxed[k], k
        assert conf["use_bbox"]                               # the caller's config is left as it was
    with pytest.raises(ValueError, match="use_bbox"):
        frames.FrameSet.load(FC.config(str(tmp_path), center, **dict(kw, use_bbox=True, use_bbox_only_for_test=False)),
                             FC.IMG_WH)
    assert math.isfinite(plain["focal"])
