"""Write tests/golden/frames_<config>.npz: GenericDataset's training buffers for the tiny dataset of
tests/frames_cases.py, computed by the reference itself (oracle/_ref), with the decoded inputs FrameSet is built from.
tests/test_gpu_frames.py checks the device draw against them without the reference.

    python tools/make_frames_golden.py
"""
import contextlib
import io
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GOLDEN = ("i1_counts", "i3_bg_obs")
KEYS = ("all_rays", "all_rgbs", "all_depths", "all_valid_masks", "all_frame_indices", "all_instance_masks",
        "all_instance_masks_weight", "all_instance_ids", "all_pass_through_masks")


def main():
    from object_nerf_b200 import frames
    from oracle import ref_loader
    from tests import frames_cases as FC
    if not ref_loader.available():
        sys.exit("oracle/_ref is not built")
    ref_loader.install()
    from datasets.generic_dataset import GenericDataset
    with tempfile.TemporaryDirectory() as root:
        center = FC.write_scene(root)
        for name in GOLDEN:
            conf = ref_loader.to_attr(FC.config(root, center, **FC.CONFIGS[name]))
            with contextlib.redirect_stdout(io.StringIO()):
                ds = GenericDataset("train", FC.IMG_WH, conf)
            inp = frames.read_frames(conf, FC.IMG_WH)
            out = {f"ref_{k}": FC.as_sampler_dtypes(getattr(ds, k), k).numpy() for k in KEYS}
            for k, v in inp.items():
                if v is not None:
                    out[f"in_{k}"] = np.asarray(v)
            path = os.path.join(ROOT, "tests", "golden", f"frames_{name}.npz")
            np.savez_compressed(path, **out)
            print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
