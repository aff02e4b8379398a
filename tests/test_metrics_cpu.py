"""CPU checks of the image metrics: the float64 restatement (tests/metrics_oracle.py) against closed forms, the entry
points' declarations, struct layout and refusals (no device needed: the checks run before any CUDA call), and the
Python wrappers' shape refusals."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests import metrics_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_identical_images_give_ssim_one_and_psnr_inf():
    rng = np.random.default_rng(0)
    img = rng.random((13, 17, 3))
    for w in (1, 3, 5, 11):
        rec, psnr, ssim = MO.metrics(img, img, 13, 17, window=w)
        assert psnr[0] == np.inf and abs(ssim[0] - 1) < 1e-12 and rec[0, 0] == 0


def test_constant_offset_matches_the_closed_form():
    """gt = a everywhere, pred = a + c: mse c^2; every window holds constants, so s_* = 0 and
    ssim = (2 a (a + c) + C1) / (a^2 + (a + c)^2 + C1)."""
    a, c = 0.3, 0.125
    gt = np.full((9, 12, 3), a)
    for w in (1, 3, 7):
        _, psnr, ssim = MO.metrics(gt + c, gt, 9, 12, window=w)
        assert abs(psnr[0] - (-10 * np.log10(c * c))) < 1e-12
        want = (2 * a * (a + c) + MO.C1) / (a * a + (a + c) ** 2 + MO.C1)
        assert abs(ssim[0] - want) < 1e-12


def test_window_one_is_the_pointwise_formula():
    rng = np.random.default_rng(1)
    p, g = rng.random((7, 5, 3)), rng.random((7, 5, 3))
    _, _, ssim = MO.metrics(p, g, 7, 5, window=1)
    point = (2 * p * g + MO.C1) / (p * p + g * g + MO.C1)
    assert abs(ssim[0] - np.clip(point, 0, 1).mean()) < 1e-12


def test_anticorrelated_images_hit_the_clamp():
    rng = np.random.default_rng(2)
    g = rng.random((20, 24, 3))
    p = 1 - g
    raw = np.stack([MO.ssim_map(p[..., c], g[..., c], 3) for c in range(3)], -1)
    assert (raw < 0).mean() > 0.3
    _, _, ssim = MO.metrics(p, g, 20, 24, window=3)
    assert abs(ssim[0] - np.clip(raw, 0, 1).mean()) < 1e-12 and ssim[0] > raw.mean()


def test_masked_columns_zero_outside_the_mask_and_empty_masks_give_nan():
    rng = np.random.default_rng(3)
    p, q, g = rng.random((10, 11, 3)), rng.random((10, 11, 3)), rng.random((10, 11, 3))
    labels = rng.integers(0, 3, size=(10, 11))
    valid = rng.random((10, 11)) > 0.2
    rec, psnr, ssim = MO.metrics(p, g, 10, 11, valid, q, labels, ids=(1, 7), window=5)
    m = valid & (labels == 1)
    assert rec[1, 2] == m.sum() and abs(rec[1, 0] - ((q - g) ** 2)[m].sum()) < 1e-12
    # a pixel outside the mask changes nothing once it is zeroed
    q2 = q.copy()
    q2[~m] = 5.0
    rec2, _, _ = MO.metrics(p, g, 10, 11, valid, q2, labels, ids=(1,), window=5)
    assert np.array_equal(rec2[1], rec[1])
    assert np.isnan(psnr[2]) and np.isnan(ssim[2]) and rec[2, 2] == 0


def test_reflect_padding_is_torch_reflect():
    img = np.random.default_rng(4).random((6, 7))
    t = torch.nn.functional.pad(torch.from_numpy(img)[None, None], (2, 2, 2, 2), mode="reflect")[0, 0].numpy()
    assert np.array_equal(np.pad(img, 2, mode="reflect"), t)


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
    from object_nerf_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "onerf_ext.h")).read(), flags=re.S)
    decl = {m.group(1): [p.strip() for p in m.group(2).split(",")]
            for m in re.finditer(r"\b(onerf_[a-z0-9_]+)\s*\(([^)]*)\)", src)}
    assert decl["onerf_image_metrics"] == ["onerf_ctx* ctx", "const onerf_metrics_args* args", "void* stream"]
    assert decl["onerf_image_metrics_finalize"] == ["onerf_ctx* ctx", "const onerf_metrics_args* args", "int slot",
                                                    "void* stream"]
    for name in ("onerf_image_metrics", "onerf_image_metrics_finalize"):
        assert name in _lib.EXPORTS_EXT and name not in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == len(decl[name])
    header = open(os.path.join(ROOT, "include", "onerf_ext.h")).read()
    assert int(re.search(r"#define ONERF_METRICS_MAX_WINDOW (\d+)", header).group(1)) == _lib.METRICS_MAX_WINDOW
    assert int(re.search(r"#define ONERF_METRICS_MAX_IDS (\d+)", header).group(1)) == _lib.METRICS_MAX_IDS


def test_struct_layout_matches_the_header(tmp_path):
    from object_nerf_b200 import _lib
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    cls = _lib.MetricsArgs
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "onerf_ext.h"', "int main(void) {",
             'printf("size %zu\\n", sizeof(onerf_metrics_args));']
    lines += [f'printf("{f[0]} %zu\\n", offsetof(onerf_metrics_args, {f[0]}));' for f in cls._fields_]
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


def _valid_args():
    """An argument block that passes every check; the pointers are never dereferenced by the refusals."""
    from object_nerf_b200 import _lib
    a = _lib.MetricsArgs()
    a.H, a.W, a.window, a.n_ids = 12, 10, 3, 2
    for k in ("pred_scene", "pred_object", "gt", "valid", "labels", "record", "psnr_out", "ssim_out"):
        setattr(a, k, 0x10000)
    a.ids_host = ctypes.cast(_IDS, ctypes.POINTER(ctypes.c_int))
    return a


@pytest.mark.parametrize("mutate,msg", [
    (lambda a: setattr(a, "window", 4), b"window"),
    (lambda a: setattr(a, "window", 13), b"window"),
    (lambda a: setattr(a, "window", 0), b"window"),
    (lambda a: (setattr(a, "window", 11), setattr(a, "H", 5)), b"exceed window / 2"),
    (lambda a: (setattr(a, "window", 7), setattr(a, "W", 3)), b"exceed window / 2"),
    (lambda a: setattr(a, "n_ids", 65), b"n_ids"),
    (lambda a: setattr(a, "n_ids", -1), b"n_ids"),
    (lambda a: setattr(a, "labels", None), b"object columns need"),
    (lambda a: setattr(a, "pred_object", None), b"object columns need"),
    (lambda a: setattr(a, "ids_host", None), b"ids_host"),
    (lambda a: setattr(a, "gt", None), b"null pred_scene or gt"),
    (lambda a: setattr(a, "record", None), b"record"),
    (lambda a: setattr(a, "record", 0x10004), b"record"),
    (lambda a: setattr(a, "labels", 0x10001), b"misaligned"),
])
def test_refusals(lib, mutate, msg):
    a = _valid_args()
    mutate(a)
    assert lib.onerf_image_metrics(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
    assert msg in lib.onerf_last_error() and lib.onerf_last_error().startswith(b"onerf_image_metrics:")


def test_column_set_decides_which_pointers_are_needed(lib):
    a = _valid_args()
    assert lib.onerf_image_metrics(None, ctypes.byref(a), None) == -1
    assert b"null argument" in lib.onerf_last_error()
    # an id no 16-bit label takes
    ids = (ctypes.c_int * 2)(3, 70000)
    a.ids_host = ctypes.cast(ids, ctypes.POINTER(ctypes.c_int))
    assert lib.onerf_image_metrics(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
    assert b"65535" in lib.onerf_last_error()
    # the window 1 frame needs no halo: 1 x 1 passes the checks (and here fails only at the NULL record below)
    a = _valid_args()
    a.n_ids, a.labels, a.pred_object, a.ids_host = 0, None, None, None
    a.H = a.W = 1
    a.window = 1
    a.record = None
    assert lib.onerf_image_metrics(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
    assert b"record" in lib.onerf_last_error()
    a.record = 0x10000
    a.psnr_out = 0x10002
    assert lib.onerf_image_metrics_finalize(ctypes.c_void_p(1), ctypes.byref(a), 0, None) == -1
    assert b"misaligned output" in lib.onerf_last_error()
    a.psnr_out = 0x10000
    assert lib.onerf_image_metrics_finalize(ctypes.c_void_p(1), ctypes.byref(a), -1, None) == -1
    assert b"slot" in lib.onerf_last_error()


def test_python_wrappers_refuse_bad_shapes():
    from object_nerf_b200 import metrics
    x = torch.zeros(1, 3, 8, 8)
    with pytest.raises(ValueError, match="reduction"):
        metrics.ssim(x, x, reduction="none")
    with pytest.raises(ValueError, match=r"\(1, 3, H, W\)"):
        metrics.ssim(x[0], x[0])
    with pytest.raises(ValueError, match=r"\(\.\.\., 3\)"):
        metrics.psnr(torch.zeros(4, 2), torch.zeros(4, 2))
    with pytest.raises(ValueError, match="valid_mask"):
        metrics.psnr(torch.zeros(4, 3), torch.zeros(4, 3), torch.ones(3, dtype=torch.bool))
