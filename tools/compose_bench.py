"""What an object imported from another trained scene costs in an edited frame (editing.Scene sets,
onerf_render_edit_frame_scenes).

Renders tools/edit_bench.py's 640x480 camera frame (64 + 64 samples, bf16, two removed-object boxes) with the sets
[0, 4, 4] plus one more object set, two ways:
  native   the extra set is object 4 of the base scene;
  imported the extra set is object 4 of a second synthetic scene (other weights, grid and codes) at scale_factor
           s_base * k, with the same box and the same world pose (its Toc translation divided by s_src), so its rays hit
           the box on the same pixels and the box culling leaves the same rows.
For k = 1 the imported frame runs the native frame's launches; for k = 8 each pass adds one depth copy and one rescale
launch.  The object's hit fraction is checked equal first, then the two arms are timed alternately (CUDA events around
render_frame with rgb_fine, outputs left on the device), --reps frames each, and the whole alternation is repeated once.
One JSON line per k: median ms per frame of each arm and each repeat.  The card's name and power limit are printed with
the numbers.

  python tools/compose_bench.py [--reps 10]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from edit_bench import FrameBox, frame_setup, scene  # noqa: E402


def source_scene(dev, scale_factor, k):
    """the second scene: its grid covers the base grid's world region at scale_factor = s_base * k"""
    from object_nerf_b200 import Embedding, editing, synthetic as S
    wc = S.make_weights(20, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)
    wf = S.make_weights(1020, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)
    grid = S.make_grid(seed=9, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05 / k, n_rows=800000)
    models = {"coarse": S.make_model(wc, True, dev), "fine": S.make_model(wf, True, dev)}
    emb = {"xyz": S.GridModule(grid).to(dev), "dir": Embedding(3, 4)}
    return editing.Scene(models, emb, S.make_code_library(S.make_codes(7)).to(dev), scale_factor * k)


def extra_toc(s):
    """the extra object's camera-to-object pose at the NeRF scale of a scene with scale_factor s"""
    cam = np.array([-3.2, 0.2, 0.3])
    fwd = -cam / np.linalg.norm(cam)
    right = np.cross(fwd, [0.0, 0.0, 1.0])
    right /= np.linalg.norm(right)
    Twc = np.eye(4)
    Twc[:3, :3] = np.stack([right, np.cross(right, fwd), -fwd], 1)
    Twc[:3, 3] = cam
    transform = np.eye(4)
    transform[:3, 3] = [0.0, -0.1, 0.25]
    t = np.linalg.inv(transform) @ Twc
    t[:3, 3] /= s
    return torch.from_numpy(t).float()[:3, :4]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from object_nerf_b200 import editing
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    models, emb, lib = scene(dev)
    cam, sets3, removed = frame_setup()
    H, W, sf = cam["H"], cam["W"], cam["scale_factor"]
    box = FrameBox([0.3, 0.1, 0.05], 0.3, sf)
    q = subprocess.run(["nvidia-smi", "-i", str(dev.index), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    info = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q, "size": f"{W}x{H}", "samples": "64+64",
            "precision": "bf16", "base_sets": [0, 4, 4]}
    native = sets3 + [(4, extra_toc(sf), box, 0.0)]
    for k in (1.0, 8.0):
        src = source_scene(dev, sf, k)
        imported = sets3 + [(4, extra_toc(src.scale_factor), box, 0.0, src)]

        def frame(sets, keys):
            return editing.render_frame(models, emb, lib, H, W, cam["focal"], sets, cam["near"], cam["far"], sf,
                                        background_skip_bbox=removed, N_samples=64, N_importance=64, precision="bf16",
                                        keys=keys)
        hits = {}
        for arm, sets in (("native", native), ("imported", imported)):
            o = frame(sets, ["z_vals_coarse", "obj_ids_coarse"])
            hits[arm] = float((o["z_vals_coarse"][o["obj_ids_coarse"] == 3] > 0).float().mean())
        assert hits["native"] > 0 and abs(hits["native"] - hits["imported"]) < 1e-3, hits
        torch.cuda.synchronize()
        repeats = []
        for _ in range(2):
            ms = {"native": [], "imported": []}
            for _ in range(args.reps):
                for arm, sets in (("native", native), ("imported", imported)):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    frame(sets, ["rgb_fine"])
                    e1.record()
                    torch.cuda.synchronize()
                    ms[arm].append(e0.elapsed_time(e1))
            med = {arm: statistics.median(v) for arm, v in ms.items()}
            med["overhead_pct"] = 100.0 * (med["imported"] / med["native"] - 1.0)
            repeats.append(med)
        print(json.dumps({**info, "k": k, "extra_set_hit_fraction": hits, "ms_per_frame": repeats}), flush=True)


if __name__ == "__main__":
    main()
