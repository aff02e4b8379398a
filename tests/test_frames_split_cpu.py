"""The frame store's test split (frames.read_frames(..., split="test")): the frames split/test.txt lists, in
transforms_full.json order, without non-finite poses and without any of the training split's filters, decoded exactly as
training frames; the default split unchanged; the refusals."""
import os

import numpy as np
import pytest

from tests import frames_cases as FC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
TEST_IDX = [8, 4, 0, 3, 6, 2]      # out of order; 4 has a NaN pose, 0 < train_start_idx, 3 = validate_idx, 6 not trained


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    root = tmp_path_factory.mktemp("frames_split")
    center = FC.write_scene(str(root))
    np.savetxt(os.path.join(root, "split", "test.txt"), TEST_IDX, fmt="%d")
    return root, center


def _conf(scene, name="i3_bg_obs", **over):
    root, center = scene
    kw = dict(FC.CONFIGS[name])
    kw.update(over)
    return FC.config(str(root), center, **kw)


@pytest.mark.parametrize("name", sorted(FC.CONFIGS))
def test_test_split_keeps_the_listed_frames_in_file_order(scene, name):
    """Frames 0, 2, 3, 6, 8 (transforms order), each decoded as the training split decodes it: every array of a frame
    equals that frame's arrays in a training read whose filters keep every finite frame."""
    from object_nerf_b200 import frames
    root, _ = scene
    test = frames.read_frames(_conf(scene, name), FC.IMG_WH, split="test")
    want = [0, 2, 3, 6, 8]
    assert test["poses"].shape[0] == len(want)
    assert np.array_equal(test["frame_idx"], np.arange(len(want)))
    # a training read of every finite frame: split file of all, no start / validate / observation / skip / size filter
    every = os.path.join(str(root), "split_every")
    os.makedirs(every, exist_ok=True)
    np.savetxt(os.path.join(every, "train.txt"), list(range(FC.N_FRAMES)), fmt="%d")
    train = frames.read_frames(_conf(scene, name, split=every, train_start_idx=0, validate_idx=-1, obs_check=False,
                                     train_skip_step=1, train_max_size=100), FC.IMG_WH)
    finite = [i for i in range(FC.N_FRAMES) if i != 4]
    rows = [finite.index(i) for i in want]
    for k in ("poses", "rgb", "depths", "labels"):
        if train[k] is None:
            assert test[k] is None, k
        else:
            assert np.array_equal(test[k], train[k][rows]), k
    for k in ("focal", "near", "far", "scale_factor", "instance_ids", "bg_instance_ids", "use_instance_mask",
              "fg_weight", "bg_weight", "border"):
        assert test[k] == train[k], k


@pytest.mark.parametrize("name", ["i1_counts", "i3_bg_obs"])
def test_default_split_is_unchanged(scene, name):
    """The train split, by default and by name, decodes bit for bit what the golden fixtures recorded."""
    from object_nerf_b200 import frames
    g = np.load(os.path.join(GOLDEN, f"frames_{name}.npz"))
    for inp in (frames.read_frames(_conf(scene, name), FC.IMG_WH),
                frames.read_frames(_conf(scene, name), FC.IMG_WH, split="train")):
        for k, v in inp.items():
            if v is None:
                assert f"in_{k}" not in g.files
            else:
                assert np.array_equal(g[f"in_{k}"], np.asarray(v)), k


def test_test_split_refusals(scene, tmp_path):
    import shutil

    from object_nerf_b200 import frames
    with pytest.raises(ValueError, match="use_bbox"):
        frames.read_frames(_conf(scene, use_bbox=True, use_bbox_only_for_test=True), FC.IMG_WH, split="test")
    frames.read_frames(_conf(scene, use_bbox=True, use_bbox_only_for_test=True), FC.IMG_WH)   # training rays unclipped
    with pytest.raises(ValueError, match="unknown split"):
        frames.read_frames(_conf(scene), FC.IMG_WH, split="val")
    with pytest.raises(ValueError, match="distance_transform"):
        frames.read_frames(_conf(scene, mask_rebalance_strategy="distance_transform"), FC.IMG_WH, split="test")
    root, _ = scene
    only_nan = tmp_path / "only_nan"
    shutil.copytree(root, only_nan)
    np.savetxt(only_nan / "split" / "test.txt", [4], fmt="%d")
    with pytest.raises(ValueError, match="finite pose"):
        frames.read_frames(_conf((only_nan, scene[1])), FC.IMG_WH, split="test")
    np.savetxt(only_nan / "split" / "test.txt", [4, 5], fmt="%d")
    os.remove(only_nan / "images" / "0005.png")
    with pytest.raises(ValueError, match="missing RGB"):
        frames.read_frames(_conf((only_nan, scene[1])), FC.IMG_WH, split="test")


def test_one_line_test_file(scene, tmp_path):
    import shutil

    from object_nerf_b200 import frames
    root, center = scene
    one = tmp_path / "one"
    shutil.copytree(root, one)
    np.savetxt(one / "split" / "test.txt", [7], fmt="%d")
    got = frames.read_frames(_conf((one, center)), FC.IMG_WH, split="test")
    full = frames.read_frames(_conf(scene), FC.IMG_WH, split="test")
    assert got["poses"].shape[0] == 1
    assert not any(np.array_equal(got["rgb"][0], r) for r in full["rgb"])      # 7 is not in the fixture's test.txt
