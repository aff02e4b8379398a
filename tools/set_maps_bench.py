"""What the per-set maps of an edited frame cost (editing.render_frame with keys from editing.set_keys).

Renders tools/edit_bench.py's 640x480 camera frame (64 + 64 samples, bf16, two removed-object boxes) with two set lists:
  [0, 4, 4]        the scene and a moved duplicate;
  25 sets          the scene and 24 copies of object 4 spread around the frame's centre;
and two key lists:
  plain            rgb_fine;
  sets             rgb_fine, opacity_sets_fine, depth_sets_fine, rgb_sets_fine.
It first checks that rgb_fine is bit-identical between the two and that the set maps sum to the joint opacity, then
times the key lists alternately (CUDA events around render_frame, outputs left on the device), --reps frames each, and
repeats the whole alternation once.  One JSON line per set list: median ms per frame of each arm and each repeat, and,
computed from shapes, the device bytes of the per-sample route to the same masks (weights_{typ}, z_vals_{typ} and
obj_ids_{typ}, (H*W, T) float32 each; the fine pass has no obj_ids in the reference, so the coarse pass only there)
against the bytes of the set maps.  The card's name and power limit are printed with the numbers.

  python tools/set_maps_bench.py [--reps 10]
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

from edit_bench import frame_setup, scene  # noqa: E402

PLAIN = ["rgb_fine"]
SETS = PLAIN + ["opacity_sets_fine", "depth_sets_fine", "rgb_sets_fine"]


def many_sets(sets, k=24):
    """the scene set and k copies of object 4, moved around the frame centre"""
    box = sets[1][2]
    Toc = sets[1][1]
    out = [sets[0]]
    for j in range(k):
        a = 2 * np.pi * j / k
        t = Toc.clone()
        t[:, 3] += torch.tensor([0.35 * np.cos(a), 0.3 * np.sin(a), 0.02 * (j % 3)], dtype=torch.float32)
        out.append((4, t, box, 0.0))
    return out


def per_sample_bytes(n_pix, n_obj, S, K):
    """device bytes of weights / z_vals / obj_ids (float32, (H*W, T)) per pass: what summing by set needs per pixel"""
    return {"coarse": 3 * n_pix * n_obj * S * 4, "fine": 3 * n_pix * n_obj * (S + K) * 4}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from object_nerf_b200 import editing
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    models, emb, lib = scene(dev)
    cam, sets3, removed = frame_setup()
    H, W = cam["H"], cam["W"]
    q = subprocess.run(["nvidia-smi", "-i", str(dev.index), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    info = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q, "size": f"{W}x{H}", "samples": "64+64",
            "precision": "bf16"}
    for label, sets in (("[0,4,4]", sets3), ("25 sets", many_sets(sets3))):
        def frame(keys):
            return editing.render_frame(models, emb, lib, H, W, cam["focal"], sets, cam["near"], cam["far"],
                                        cam["scale_factor"], background_skip_bbox=removed, N_samples=64,
                                        N_importance=64, precision="bf16", keys=keys)
        a, b = frame(PLAIN), frame(SETS)
        full = frame(["opacity_fine"])
        assert torch.equal(a["rgb_fine"], b["rgb_fine"]), "rgb_fine changed with the set maps"
        err = (b["opacity_sets_fine"].double().sum(1) - full["opacity_fine"].double()).abs().max().item()
        torch.cuda.synchronize()
        repeats = []
        for _ in range(2):
            ms = {"plain": [], "sets": []}
            for _ in range(args.reps):
                for arm, keys in (("plain", PLAIN), ("sets", SETS)):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    frame(keys)
                    e1.record()
                    torch.cuda.synchronize()
                    ms[arm].append(e0.elapsed_time(e1))
            med = {arm: statistics.median(v) for arm, v in ms.items()}
            med["overhead_pct"] = 100.0 * (med["sets"] / med["plain"] - 1.0)
            repeats.append(med)
        n_obj, n_pix = len(sets), H * W
        ps = per_sample_bytes(n_pix, n_obj, 64, 64)
        print(json.dumps({**info, "sets": label, "n_obj": n_obj, "rgb_fine_bit_identical": True,
                          "max_abs_sum_over_sets_minus_opacity": err, "ms_per_frame": repeats,
                          "per_sample_route_bytes": ps, "set_maps_bytes_per_pass": n_pix * n_obj * 5 * 4}), flush=True)


if __name__ == "__main__":
    main()
