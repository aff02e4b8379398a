"""CPU checks of the depth and mask metrics: the float64 restatement (tests/geometry_metrics_oracle.py) against
hand-computed cases, the entry points' declarations, exports and struct layout, and every refusal (no device needed:
the checks run before any CUDA call)."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests import geometry_metrics_oracle as GO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = {
    "onerf_depth_metrics": ["onerf_ctx* ctx", "const onerf_depth_metrics_args* args", "void* stream"],
    "onerf_depth_metrics_finalize": ["onerf_ctx* ctx", "const onerf_depth_metrics_args* args", "int slot",
                                     "void* stream"],
    "onerf_mask_metrics": ["onerf_ctx* ctx", "const onerf_mask_metrics_args* args", "void* stream"],
    "onerf_mask_metrics_finalize": ["onerf_ctx* ctx", "const onerf_mask_metrics_args* args", "int slot",
                                    "void* stream"],
}


# ---------------------------------------------------------------------------------------------------------------------
# the restatement against hand-computed cases
# ---------------------------------------------------------------------------------------------------------------------
def test_depth_by_hand():
    """Four pixels, scale 2: gt 1, 2, 0 (excluded), 0.5 -> g = 2, 4, -, 1; pred 1, 2.5, 9, 0.25 -> d = 2, 5, -, 0.5."""
    gt = np.array([1, 2, 0, 0.5], np.float32)
    pred = np.array([1, 2.5, 9, 0.25], np.float32)
    rec, out = GO.depth_metrics(pred, gt, scale=2.0)
    e, g = np.array([0, 1, -0.5]), np.array([2, 4, 1.0])
    want = [3, (np.abs(e) / g).sum(), (e * e / g).sum(), (e * e).sum(), np.log(2) ** 2 + np.log(1.25) ** 2, 1, 2, 2]
    # ratios 1, 1.25 (not < 1.25, < 1.25^2) and 2 (not < 1.25^3)
    assert np.allclose(rec[0], want, rtol=1e-15, atol=0)
    assert rec[0, 4] == pytest.approx(np.log(5 / 4) ** 2 + np.log(2) ** 2, rel=1e-15)
    assert np.allclose(out[0], [(0 + 0.25 + 0.5) / 3, (0 + 0.25 + 0.25) / 3, math.sqrt(1.25 / 3),
                                math.sqrt(rec[0, 4] / 3), 1 / 3, 2 / 3, 2 / 3], rtol=1e-15, atol=0)


def test_depth_clamp_and_ratio_boundaries():
    """d_min / d_max clamp 0, negative and large predictions; ratios exactly 1.25^i fall outside delta_i."""
    gt = np.array([1, 1, 1, 1, 1, 1, 1.25], np.float32)
    pred = np.array([0, -3, 50, 1.25, 1.5625, 1.953125, 1], np.float32)
    rec, out = GO.depth_metrics(pred, gt, depth_range=(0.5, 4.0))
    # d = 0.5, 0.5, 4, 1.25, 1.5625, 1.953125, 1; ratios 2, 2, 4, 1.25, 1.5625, 1.953125 and g / d = 1.25
    assert rec[0, 3] == 0.25 + 0.25 + 9 + 0.0625 + 0.31640625 + 0.908447265625 + 0.0625
    assert list(rec[0, 5:]) == [0, 2, 3]
    assert out[0, 4] == 0 and out[0, 5] == pytest.approx(2 / 7) and out[0, 6] == pytest.approx(3 / 7)


def test_depth_object_columns_and_empty_columns():
    gt = np.array([1, 1, 2, 0, 1], np.float32)
    valid = np.array([1, 1, 1, 1, 0], bool)
    scene = np.array([1, 1, 1, 1, 1], np.float32)
    obj = np.array([2, 1, 2, 2, 2], np.float32)
    labels = np.array([7, 3, 7, 7, 3], np.uint16)
    rec, out = GO.depth_metrics(scene, gt, valid, obj, labels, ids=(7, 3, 65535))
    assert list(rec[:, 0]) == [3, 2, 1, 0]         # pixel 3 has no depth, pixel 4 is not valid
    assert rec[1, 3] == 1 and rec[2, 3] == 0       # object 7: errors 1 and 0; object 3: 0
    assert np.isnan(out[3]).all() and np.isfinite(out[:3]).all()


def test_nan_prediction_makes_its_column_nan():
    gt = np.ones(3, np.float32)
    scene = np.array([1, np.nan, 1], np.float32)
    obj = np.ones(3, np.float32)
    _, out = GO.depth_metrics(scene, gt, None, obj, np.array([1, 1, 2]), ids=(1, 2))
    assert np.isnan(out[0]).all() and np.isfinite(out[1:]).all()


def test_mask_by_hand():
    o = np.array([0.9, 0.5, 0.49, 0.2, 1.0, 0.7], np.float32)
    labels = np.array([4, 4, 4, 0, 0, 4], np.uint16)
    valid = np.array([1, 1, 1, 1, 1, 0], bool)
    rec = GO.mask_sums(o, labels, 4, valid, threshold=0.5)
    # P = 1 1 0 0 1 (0.5 counts), G = 1 1 1 0 0 over the valid pixels
    assert list(rec[[0, 1, 3]]) == [2, 4, 5]
    f32 = lambda x: float(np.float32(x))
    assert rec[2] == pytest.approx((1 - f32(0.9)) + 0.5 + (1 - f32(0.49)) + f32(0.2) + 1.0, rel=1e-15)
    iou, l1 = GO.mask_outputs(rec)
    assert iou[0] == 0.5 and l1[0] == pytest.approx(rec[2] / 5)
    # no pixel of the object and none covered: empty union -> NaN iou, finite l1
    iou, l1 = GO.mask_outputs(GO.mask_sums(np.zeros(4, np.float32), np.zeros(4), 9))
    assert np.isnan(iou[0]) and l1[0] == 0
    iou, l1 = GO.mask_outputs(GO.mask_sums(o, labels, 4, np.zeros(6, bool)))
    assert np.isnan(iou[0]) and np.isnan(l1[0])


# ---------------------------------------------------------------------------------------------------------------------
# the C entries
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def test_entries_are_exported_and_declared(lib):
    from object_nerf_b200 import _lib, metrics
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "onerf_ext.h")).read(), flags=re.S)
    decl = {m.group(1): [p.strip() for p in m.group(2).split(",")]
            for m in re.finditer(r"\b(onerf_[a-z0-9_]+)\s*\(([^)]*)\)", src)}
    for name, params in ENTRIES.items():
        assert decl[name] == params
        assert name in _lib.EXPORTS_EXT and name not in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == len(params)
    assert _lib.ABI_VERSION == 2 and lib.onerf_abi_version() == 2
    header = open(os.path.join(ROOT, "include", "onerf_ext.h")).read()
    for macro, value in (("ONERF_DEPTH_METRICS", _lib.DEPTH_METRICS), ("ONERF_DEPTH_RECORD", _lib.DEPTH_RECORD),
                         ("ONERF_MASK_RECORD", _lib.MASK_RECORD)):
        assert int(re.search(rf"#define {macro} (\d+)", header).group(1)) == value
    assert metrics.DEPTH_METRICS == GO.DEPTH_METRICS and len(GO.DEPTH_METRICS) == _lib.DEPTH_METRICS


@pytest.mark.parametrize("cls,cname", [("DepthMetricsArgs", "onerf_depth_metrics_args"),
                                       ("MaskMetricsArgs", "onerf_mask_metrics_args")])
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


_IDS = (ctypes.c_int * 65)(*range(65))


def _depth_args():
    """An argument block that passes every check; the pointers are never dereferenced by the refusals."""
    from object_nerf_b200 import _lib
    a = _lib.DepthMetricsArgs()
    a.H, a.W, a.n_ids, a.scale, a.d_min, a.d_max = 12, 10, 2, 1.0, 1e-3, 10.0
    for k in ("pred_scene", "pred_object", "gt", "valid", "labels", "record", "out"):
        setattr(a, k, 0x10000)
    a.ids_host = ctypes.cast(_IDS, ctypes.POINTER(ctypes.c_int))
    return a


def _mask_args():
    from object_nerf_b200 import _lib
    a = _lib.MaskMetricsArgs()
    a.H, a.W, a.n_ids, a.column, a.id, a.threshold = 12, 10, 3, 2, 7, 0.5
    for k in ("opacity", "valid", "labels", "record", "iou_out", "opacity_l1_out"):
        setattr(a, k, 0x10000)
    return a


@pytest.mark.parametrize("mutate,msg", [
    (lambda a: setattr(a, "n_ids", 65), b"n_ids"),
    (lambda a: setattr(a, "n_ids", -1), b"n_ids"),
    (lambda a: setattr(a, "H", 0), b"H and W"),
    (lambda a: setattr(a, "W", -2), b"H and W"),
    (lambda a: (setattr(a, "H", 1 << 20), setattr(a, "W", 1 << 20)), b"2^40"),
    (lambda a: setattr(a, "d_min", 0.0), b"0 < d_min < d_max"),
    (lambda a: setattr(a, "d_min", -1.0), b"0 < d_min < d_max"),
    (lambda a: setattr(a, "d_min", 10.0), b"0 < d_min < d_max"),
    (lambda a: setattr(a, "d_max", 5e-4), b"0 < d_min < d_max"),
    (lambda a: setattr(a, "d_max", math.inf), b"finite"),
    (lambda a: setattr(a, "d_min", math.nan), b"finite"),
    (lambda a: setattr(a, "scale", math.nan), b"scale"),
    (lambda a: setattr(a, "scale", math.inf), b"scale"),
    (lambda a: setattr(a, "scale", 0.0), b"scale"),
    (lambda a: setattr(a, "scale", -1.0), b"scale"),
    (lambda a: setattr(a, "pred_scene", None), b"null pred_scene or gt"),
    (lambda a: setattr(a, "gt", None), b"null pred_scene or gt"),
    (lambda a: setattr(a, "labels", None), b"object columns need"),
    (lambda a: setattr(a, "pred_object", None), b"object columns need"),
    (lambda a: setattr(a, "ids_host", None), b"ids_host"),
    (lambda a: setattr(a, "record", None), b"record"),
    (lambda a: setattr(a, "record", 0x10004), b"record"),
    (lambda a: setattr(a, "gt", 0x10002), b"misaligned"),
    (lambda a: setattr(a, "pred_object", 0x10001), b"misaligned"),
    (lambda a: setattr(a, "labels", 0x10001), b"misaligned"),
])
def test_depth_refusals(lib, mutate, msg):
    a = _depth_args()
    mutate(a)
    assert lib.onerf_depth_metrics(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
    assert msg in lib.onerf_last_error() and lib.onerf_last_error().startswith(b"onerf_depth_metrics:")


def test_depth_id_refusals(lib):
    a = _depth_args()
    for ids, msg in (((3, 70000), b"65535"), ((-1, 2), b"65535"), ((5, 5), b"distinct")):
        arr = (ctypes.c_int * 2)(*ids)
        a.ids_host = ctypes.cast(arr, ctypes.POINTER(ctypes.c_int))
        assert lib.onerf_depth_metrics(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
        assert msg in lib.onerf_last_error()
    # without objects no object pointer is needed: K = 0 fails here only at the NULL record
    a = _depth_args()
    a.n_ids, a.labels, a.pred_object, a.ids_host, a.valid, a.record = 0, None, None, None, None, None
    a.H = a.W = 1
    assert lib.onerf_depth_metrics(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
    assert b"record" in lib.onerf_last_error()


@pytest.mark.parametrize("mutate,msg", [
    (lambda a: setattr(a, "n_ids", 65), b"n_ids"),
    (lambda a: setattr(a, "n_ids", 0), b"n_ids"),
    (lambda a: setattr(a, "column", 3), b"column"),
    (lambda a: setattr(a, "column", -1), b"column"),
    (lambda a: setattr(a, "id", 65536), b"65535"),
    (lambda a: setattr(a, "id", -1), b"65535"),
    (lambda a: setattr(a, "threshold", math.nan), b"threshold"),
    (lambda a: setattr(a, "threshold", math.inf), b"threshold"),
    (lambda a: setattr(a, "threshold", -math.inf), b"threshold"),
    (lambda a: setattr(a, "H", 0), b"H and W"),
    (lambda a: setattr(a, "opacity", None), b"null opacity or labels"),
    (lambda a: setattr(a, "labels", None), b"null opacity or labels"),
    (lambda a: setattr(a, "record", None), b"record"),
    (lambda a: setattr(a, "record", 0x10004), b"record"),
    (lambda a: setattr(a, "opacity", 0x10002), b"misaligned"),
    (lambda a: setattr(a, "labels", 0x10001), b"misaligned"),
])
def test_mask_refusals(lib, mutate, msg):
    a = _mask_args()
    mutate(a)
    assert lib.onerf_mask_metrics(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
    assert msg in lib.onerf_last_error() and lib.onerf_last_error().startswith(b"onerf_mask_metrics:")


def test_null_context_and_finalize_refusals(lib):
    d, m = _depth_args(), _mask_args()
    for name, a in (("onerf_depth_metrics", d), ("onerf_mask_metrics", m)):
        assert getattr(lib, name)(None, ctypes.byref(a), None) == -1
        assert b"null argument" in lib.onerf_last_error()
        assert getattr(lib, name)(ctypes.c_void_p(1), None, None) == -1
        assert b"null argument" in lib.onerf_last_error()
        fin = getattr(lib, name + "_finalize")
        assert fin(None, ctypes.byref(a), 0, None) == -1
        assert lib.onerf_last_error().startswith(name.encode() + b"_finalize: null argument")
        assert fin(ctypes.c_void_p(1), ctypes.byref(a), -1, None) == -1
        assert b"slot" in lib.onerf_last_error()
    d.out = 0x10002
    assert lib.onerf_depth_metrics_finalize(ctypes.c_void_p(1), ctypes.byref(d), 0, None) == -1
    assert b"misaligned output" in lib.onerf_last_error()
    d = _depth_args()
    d.record = 0x10004
    assert lib.onerf_depth_metrics_finalize(ctypes.c_void_p(1), ctypes.byref(d), 0, None) == -1
    assert b"record" in lib.onerf_last_error()
    d = _depth_args()
    d.n_ids = 65
    assert lib.onerf_depth_metrics_finalize(ctypes.c_void_p(1), ctypes.byref(d), 0, None) == -1
    assert b"n_ids" in lib.onerf_last_error()
    m.opacity_l1_out = 0x10001
    assert lib.onerf_mask_metrics_finalize(ctypes.c_void_p(1), ctypes.byref(m), 0, None) == -1
    assert b"misaligned output" in lib.onerf_last_error()
    m = _mask_args()
    m.n_ids = 0
    assert lib.onerf_mask_metrics_finalize(ctypes.c_void_p(1), ctypes.byref(m), 0, None) == -1
    assert b"n_ids" in lib.onerf_last_error()


def test_python_wrappers_refuse_mismatched_pixel_counts():
    import torch
    from object_nerf_b200 import metrics
    with pytest.raises(ValueError, match="one pixel count"):
        metrics.mask_metrics(torch.zeros(4), torch.zeros(5, dtype=torch.int16), 1)
    with pytest.raises(ValueError, match="one pixel count"):
        metrics.mask_metrics(torch.zeros(4), torch.zeros(4, dtype=torch.int16), 1,
                             valid=torch.ones(3, dtype=torch.bool))
