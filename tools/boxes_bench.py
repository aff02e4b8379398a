"""What scoring every object inside its own box costs: rendering.render_boxes (one call, the object branch on the rows
that hit their box only) against the K validate_frame renders of box-clipped rays it replaces.

The 640x480 voxel scene of tools/eval_geometry_bench.py (64 + 64 samples, bf16) and its first camera; K = 4, 16 and 64
axis-aligned boxes around the scene's centre, each box's share of the frame's pixels printed with the numbers.
  render    ms per frame of every object's fine opacity, depth and colour maps, alternated, --reps calls each, the
            alternation repeated twice:
              (a) K training.validate_frame renders (rays_in_bbox, code ids[k] on every pixel) over
                  ray_utils.camera_rays(box k), what a per-object loop over box-clipped rays runs;
              (b) render_boxes;
            and the hit pixels of (a) and (b) compared bit for bit at the timed size.
  kernel    per-kernel device time per frame of (b) from torch.profiler in a run of its own (so its total is not the
            event-timed frame above), and the share of the stages that still see every (object, pixel) row, hit or
            not: the box rays, the three list kernels and the missed-value fill of the maps (everything else runs on the hit
            rows only).
The card's name and power limit are read in the same run and printed with the numbers, one JSON line per measurement.

  python tools/boxes_bench.py [--reps 3] [--boxes 4 16 64]
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

import eval_geometry_bench as G  # noqa: E402

H, W = G.H, G.W
S, NI = 64, 64
KEYS = ("opacity_instance", "depth_instance", "rgb_instance")
# kernels that run on every (object, pixel) row of a chunk, hit or not; every other kernel runs on the hit rows only
DEAD_ROW_STAGES = ("box_rays_kernel", "list_count_kernel", "list_scan_kernel", "list_write_kernel", "fill_missed_kernel")
KERNELS = DEAD_ROW_STAGES + ("field_tc_multi_kernel", "ray_const_kernel", "box_codes_kernel", "sample_coarse_live_kernel",
                             "sample_pdf_merge_live_kernel", "composite_boxes_kernel")


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def make_boxes(K):
    """K boxes on a ring around the scene's centre (side 0.35, 0.2 at K = 16, 0.1 at K = 64), alternately raised and
    lowered."""
    from object_nerf_b200.frames import ObjectBox
    side = 0.35 if K <= 4 else (0.2 if K <= 16 else 0.1)
    out = []
    for k in range(K):
        a = 2 * np.pi * k / K
        c = np.array([0.3 * np.cos(a), 0.3 * np.sin(a), 0.1 * (-1) ** k])
        out.append(ObjectBox(pose_avg=np.eye(4), axis_align_mat=np.eye(4), bbox_bounds=np.array([c - side / 2,
                                                                                                  c + side / 2])))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--boxes", type=int, nargs="+", default=[4, 16, 64], help="box counts K to measure")
    args = ap.parse_args()
    from object_nerf_b200 import evaluation, ray_utils, rendering, training
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    info = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q, "size": f"{W}x{H}", "samples": "64+64",
            "precision": "bf16", "model": "voxel"}
    models, emb, lib, fs = G.scene(dev, 1)
    c2w = torch.from_numpy(fs.poses_host[0].reshape(3, 4))
    cam = dict(near=fs.near, far=fs.far, scale_factor=fs.scale_factor)
    base = evaluation.frame_batch(fs, 0)
    render = dict(N_samples=S, N_importance=NI, use_disp=False)

    n_codes = lib.embedding_instance.weight.shape[0]
    for K in args.boxes:
        boxes, ids = make_boxes(K), [(1 + k) % n_codes for k in range(K)]
        clipped = [ray_utils.camera_rays(H, W, fs.focal, c2w, fs.near, fs.far, fs.scale_factor, box=b, device=dev,
                                         return_mask=True) for b in boxes]

        def loop(keep=False):        # (a)
            out = []
            for (rays, _), i in zip(clipped, ids):
                batch = dict(base, rays=rays, instance_ids=torch.full((H * W,), i, dtype=torch.int64, device=dev))
                o = training.validate_frame(models, emb, lib, batch, evaluation._NO_LOSS, white_back=False,
                                            rays_in_bbox=True, keys=KEYS, **render)
                out.append({k: v.clone() for k, v in o.items()} if keep else o)
            return out

        def fused():                 # (b)
            return rendering.render_boxes(models, emb, lib, H, W, fs.focal, c2w, boxes, ids, keys=KEYS, **render,
                                          **cam)

        a = loop(keep=True)
        b = {k: v.clone() for k, v in fused().items()}
        torch.cuda.synchronize()
        same = all(torch.equal(b["hit"][:, k], clipped[k][1]) and
                   all(torch.equal(b[f"{kind}_fine"][:, k][clipped[k][1]], a[k][f"{kind}_fine"][clipped[k][1]])
                       for kind in KEYS) for k in range(K))
        cover = [round(float(h.float().mean()), 4) for _, h in clipped]
        print(json.dumps({**info, "K": K, "measure": "render_boxes_bit_identical_at_hit_pixels", "same": same,
                          "pixel_share_per_box": cover, "mean_pixel_share": round(sum(cover) / K, 4)}), flush=True)
        repeats = []
        for _ in range(2):
            ms = {"a_validate_frame_loop": [], "b_render_boxes": []}
            for _ in range(args.reps):
                ms["a_validate_frame_loop"].append(timed(loop))
                ms["b_render_boxes"].append(timed(fused))
            repeats.append({"median_ms": {k: statistics.median(v) for k, v in ms.items()}, "runs_ms": ms})
        print(json.dumps({**info, "K": K, "measure": "ms_per_frame_every_object_fine_map", "repeats": repeats}),
              flush=True)

        from torch.profiler import ProfilerActivity, profile
        fused()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                fused()
            torch.cuda.synchronize()
        us = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA":
                name = next((k for k in KERNELS if k in ev.name), "other")
                us[name] = us.get(name, 0.0) + ev.device_time / 3
        total = sum(us.values())
        dead = sum(us.get(k, 0.0) for k in DEAD_ROW_STAGES)
        print(json.dumps({**info, "K": K, "measure": "kernels_profiled", "device_us_per_frame": us,
                          "profiled_kernel_total_us_per_frame": total, "every_row_stages_us": dead,
                          "every_row_stages_share": dead / total}), flush=True)


if __name__ == "__main__":
    main()
