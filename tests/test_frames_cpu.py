"""CPU side of the frame store (object_nerf_b200/frames.py, include/onerf_ext.h: onerf_draw_frames): the host decode
of GenericDataset's train split against the reference's own GenericDataset (oracle/_ref, where it is built), the golden
fixtures' decoded inputs against today's decode, the refusals before any CUDA call, and the C entries' exports, struct
layout and argument checks."""
import contextlib
import ctypes
import io
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests import frames_cases as FC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
RAYS_D_TOL = 2.5e-7


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    root = tmp_path_factory.mktemp("frames")
    return root, FC.write_scene(str(root))


@pytest.fixture(scope="module")
def ref():
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("oracle/_ref is not built")
    ref_loader.install()
    from datasets.generic_dataset import GenericDataset
    return ref_loader, GenericDataset


@pytest.mark.parametrize("name", sorted(FC.CONFIGS))
def test_reference_buffers_equal_the_host_restatement(scene, ref, name):
    from object_nerf_b200 import frames
    ref_loader, GenericDataset = ref
    root, center = scene
    conf = ref_loader.to_attr(FC.config(str(root), center, **FC.CONFIGS[name]))
    with contextlib.redirect_stdout(io.StringIO()):
        ds = GenericDataset("train", FC.IMG_WH, conf)
        inp = frames.read_frames(conf, FC.IMG_WH)
        # the same frames in the same order, with the reference's f32 c2w and frame indices
        F = inp["poses"].shape[0]
        assert F == len(ds.meta["frames"])
        assert np.array_equal(inp["frame_idx"], np.arange(F))
        for f, fr in enumerate(ds.meta["frames"]):
            c2w = ds.read_frame_data(fr, ds.instance_ids[0])["c2w"]
            assert np.array_equal(inp["poses"][f], c2w.numpy()), f
    mine = FC.expand_host(inp)
    for k, v in mine.items():
        r = FC.as_sampler_dtypes(getattr(ds, k), k)
        assert r.shape == v.shape, (k, tuple(r.shape), tuple(v.shape))
        if k == "all_rays":
            assert torch.equal(r[:, [0, 1, 2, 6, 7]], v[:, [0, 1, 2, 6, 7]])
            assert (r[:, 3:6] - v[:, 3:6]).abs().max().item() <= RAYS_D_TOL
        else:
            assert torch.equal(r, v), k


def test_the_scene_exercises_every_filter(scene):
    """Frames 0 (before train_start_idx), 3 (validate_idx), 4 (NaN pose) and 6 (not in the split) never train; the
    observation check drops 1 (angle) and 8 (distance); skip and max size keep frames 1 and 5."""
    from object_nerf_b200 import frames
    root, center = scene
    kept = {}
    for name in ("i1_counts", "i3_bg_obs", "zero_later_skip"):
        inp = frames.read_frames(FC.config(str(root), center, **FC.CONFIGS[name]), FC.IMG_WH)
        kept[name] = inp["poses"].shape[0]
        assert inp["rgb"].shape[1:] == (FC.IMG_WH[1], FC.IMG_WH[0], 3)
    assert kept == {"i1_counts": 5, "i3_bg_obs": 3, "zero_later_skip": 2}
    inp = frames.read_frames(FC.config(str(root), center, **FC.CONFIGS["zero_later_skip"]), FC.IMG_WH)
    assert inp["instance_ids"] == [2, 5]          # an id 0 after the first column is dropped, as the reference does
    assert (inp["depths"] == 0).any() and inp["labels"].max() == 300


@pytest.mark.parametrize("name", ["i1_counts", "i3_bg_obs"])
def test_golden_inputs_are_todays_decode(scene, name):
    from object_nerf_b200 import frames
    root, center = scene
    g = np.load(os.path.join(GOLDEN, f"frames_{name}.npz"))
    inp = frames.read_frames(FC.config(str(root), center, **FC.CONFIGS[name]), FC.IMG_WH)
    for k, v in inp.items():
        if v is None:
            assert f"in_{k}" not in g.files
        else:
            assert np.array_equal(g[f"in_{k}"], np.asarray(v)), k


@pytest.fixture
def no_cuda(monkeypatch):
    def fail(*a, **k):
        pytest.fail("touched a device before refusing")
    monkeypatch.setattr(torch.Tensor, "to", fail)
    monkeypatch.setattr(torch.cuda, "current_device", fail)


def test_load_refusals_come_before_any_cuda_call(scene, no_cuda, tmp_path):
    from object_nerf_b200.frames import FrameSet
    root, center = scene
    with pytest.raises(ValueError, match="use_bbox"):
        FrameSet.load(FC.config(str(root), center, use_bbox=True, use_bbox_only_for_test=False), FC.IMG_WH)
    with pytest.raises(ValueError, match="distance_transform"):
        FrameSet.load(FC.config(str(root), center, mask_rebalance_strategy="distance_transform"), FC.IMG_WH)
    with pytest.raises(ValueError, match="mask_rebalance_strategy"):
        FrameSet.load(FC.config(str(root), center, mask_rebalance_strategy="none"), FC.IMG_WH)
    with pytest.raises(ValueError, match="pass-through"):
        FrameSet.load(FC.config(str(root), center, bg_instance_id=list(range(20))), FC.IMG_WH)
    gone = tmp_path / "gone"
    shutil.copytree(root, gone)
    os.remove(gone / "images" / "0005.png")
    with pytest.raises(ValueError, match="missing RGB"):
        FrameSet.load(FC.config(str(gone), center), FC.IMG_WH)


def test_constructor_refusals_come_before_any_cuda_call(no_cuda):
    from object_nerf_b200.frames import FrameSet
    F, H, W = 2, 5, 7
    kw = dict(focal=10.0, near=0.1, far=2.0, scale_factor=1.0, instance_ids=[3])
    poses, rgb = np.zeros((F, 3, 4), np.float32), np.zeros((F, H, W, 3), np.uint8)
    depths, labels = np.zeros((F, H, W), np.float32), np.zeros((F, H, W), np.uint16)
    with pytest.raises(ValueError, match="16 bits"):
        FrameSet(poses, rgb, depths, labels.astype(np.int32), **kw)
    with pytest.raises(ValueError, match="rgb"):
        FrameSet(poses, rgb.astype(np.float32), depths, labels, **kw)
    with pytest.raises(ValueError, match="depths"):
        FrameSet(poses, rgb, depths.astype(np.float64), labels, **kw)
    with pytest.raises(ValueError, match="label images"):
        FrameSet(poses, rgb, depths, None, **kw)
    with pytest.raises(ValueError, match="both"):
        FrameSet(poses, rgb, depths, labels, fg_weight=1.0, **kw)
    with pytest.raises(ValueError, match="border"):
        FrameSet(poses, rgb, depths, labels, border=-1, **kw)


def test_instance_tables():
    from object_nerf_b200.frames import instance_tables
    labels = np.array([[2, 2, 0, 1], [7, 7, 7, 7]], dtype=np.uint16)
    ids, ones, w, p = instance_tables(labels, [0, 2, 70000], bg_instance_ids=[1])
    assert ids.tolist() == [0, 2, 70000] and ones.tolist() == [1, 0, 0]
    assert p.tolist() == [[1, 0], [1, 2], [1, -1]]
    assert w[:, 0].tolist() == [[0, 0], [0, 0]]
    assert w[0, 1].tolist() == [1.0, 1.0] and w[1, 1].tolist() == [np.float32(1 / 4), 4.0]  # fg clamped to 1
    ids, ones, w, p = instance_tables(labels, [2], use_instance_mask=False)
    assert ones.tolist() == [1] and not w.any()


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
    assert decl["onerf_draw_frames"] == ["onerf_ctx* ctx", "const onerf_frame_dataset* frames",
                                         "const onerf_batch_args* args", "void* stream"]
    assert decl["onerf_draw_frames_dstep"] == ["onerf_ctx* ctx", "const onerf_frame_dataset* frames",
                                               "const onerf_batch_args* args", "uint64_t* step_dev", "void* stream"]
    for name in ("onerf_draw_frames", "onerf_draw_frames_dstep"):
        assert name in _lib.EXPORTS_EXT and name not in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == len(decl[name])
    m = re.search(r"#define ONERF_FRAME_MAX_PASS (\d+)", open(os.path.join(ROOT, "include", "onerf_ext.h")).read())
    assert int(m.group(1)) == _lib.FRAME_MAX_PASS


def test_struct_layout_matches_the_header(tmp_path):
    from object_nerf_b200 import _lib
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    cls = _lib.FrameDataset
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "onerf_ext.h"', "int main(void) {",
             'printf("size %zu\\n", sizeof(onerf_frame_dataset));']
    lines += [f'printf("{f[0]} %zu\\n", offsetof(onerf_frame_dataset, {f[0]}));' for f in cls._fields_]
    lines.append("return 0; }")
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", str(tmp_path / "l")],
                   check=True)
    got = dict(line.rsplit(" ", 1) for line in subprocess.run([str(tmp_path / "l")], capture_output=True, text=True,
                                                              check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(cls)
    for f in cls._fields_:
        assert int(got[f[0]]) == getattr(cls, f[0]).offset, f[0]


def _valid():
    """A frame store and argument block that pass every check; the pointers are never dereferenced by the refusals."""
    from object_nerf_b200 import _lib
    d = _lib.FrameDataset()
    d.n_frames, d.H, d.W, d.n_instances, d.border, d.n_pass = 3, 40, 50, 2, 20, 2
    for k in ("poses", "directions", "rgb", "depths", "labels", "frame_idx", "ids", "mask_all_ones", "weights",
              "pass_ids"):
        setattr(d, k, 0x10000)
    a = _lib.BatchArgs()
    for k in ("rays", "rgbs", "depths", "valid_mask", "instance_mask", "instance_mask_weight", "instance_ids",
              "pass_through_mask"):
        setattr(a, k, 0x20000)
    a.batch, a.rank, a.world = 2000, 1, 3
    return d, a


@pytest.mark.parametrize("mutate,msg", [
    (lambda d, a: setattr(d, "poses", None), b"null frame-store buffer"),
    (lambda d, a: setattr(d, "weights", None), b"null frame-store buffer"),
    (lambda d, a: setattr(d, "pass_ids", None), b"null frame-store buffer"),
    (lambda d, a: setattr(a, "rgbs", None), b"null output buffer"),
    (lambda d, a: setattr(d, "H", 0), b"H and W"),
    (lambda d, a: setattr(d, "border", -1), b"border"),
    (lambda d, a: setattr(d, "n_pass", 17), b"n_pass"),
    (lambda d, a: setattr(d, "n_pass", 0), b"n_pass"),
    (lambda d, a: setattr(d, "n_instances", 0), b"n_instances"),
    (lambda d, a: setattr(a, "rank", 3), b"rank outside"),
    (lambda d, a: setattr(a, "batch", 2001), b"no full batch"),
    (lambda d, a: setattr(d, "n_frames", 1 << 30), b"2^40"),
])
def test_refusals(lib, mutate, msg):
    d, a = _valid()
    mutate(d, a)
    ctx = ctypes.c_void_p(1)
    assert lib.onerf_draw_frames(ctx, ctypes.byref(d), ctypes.byref(a), None) == -1
    assert msg in lib.onerf_last_error() and lib.onerf_last_error().startswith(b"onerf_draw_frames:")
    assert lib.onerf_draw_frames_dstep(ctx, ctypes.byref(d), ctypes.byref(a), 0x1000, None) == -1
    assert msg in lib.onerf_last_error() and lib.onerf_last_error().startswith(b"onerf_draw_frames_dstep:")


def test_labels_may_be_null_and_step_pointer_checks(lib):
    d, a = _valid()
    ctx = ctypes.c_void_p(1)
    assert lib.onerf_draw_frames(None, ctypes.byref(d), ctypes.byref(a), None) == -1
    assert lib.onerf_draw_frames(ctx, None, ctypes.byref(a), None) == -1
    assert b"null argument" in lib.onerf_last_error()
    assert lib.onerf_draw_frames_dstep(ctx, ctypes.byref(d), ctypes.byref(a), None, None) == -1
    assert b"null step_dev" in lib.onerf_last_error()
    assert lib.onerf_draw_frames_dstep(ctx, ctypes.byref(d), ctypes.byref(a), 0x1004, None) == -1
    assert b"8-byte aligned" in lib.onerf_last_error()
    # without labels no column reads a mask: the per-column mask tables and n_pass are not needed
    d.labels, d.mask_all_ones, d.pass_ids, d.n_pass = None, None, None, 0
    d.n_frames = 1 << 30
    assert lib.onerf_draw_frames(ctx, ctypes.byref(d), ctypes.byref(a), None) == -1
    assert b"2^40" in lib.onerf_last_error()                          # every earlier check passed
