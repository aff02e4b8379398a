"""What every object's maps of a frame cost: rendering.render_instances (one render, the object branch once per code)
against the K renders it replaces.

The 640x480 voxel scene of tools/eval_geometry_bench.py (64 + 64 samples, bf16, K = 4 quarter-frame objects in its
label images) and its first camera; K = 4 (those objects) and K = 16 (code rows 1..16) object codes.  Every pixel is
rendered with every code, so the cost does not depend on the objects' sizes.
  render    ms per frame of every object's opacity, depth and colour maps, alternated, --reps calls each, the alternation
            repeated twice:
              (a) K training.validate_frame renders, every pixel with object k's code (what evaluate_frames(masks=True)
                  ran before render_instances);
              (b) the same work composed from the stage entries: coarse depths, the coarse scene field, its
                  compositing and the importance sampler once, then in the fine pass the scene field once and per code
                  one object-only field launch and one compositing launch (engine.sample_coarse / field / composite /
                  sample_pdf_merge);
              (c) render_instances, asked for the fine object maps only (so it runs no coarse object branch and no
                  fine scene branch);
            and the outputs of (a) and (c) compared bit for bit at the timed size.
  evaluate  ms per frame of evaluate_frames(masks=True) against evaluate_frames() (K = 4), alternated.
  kernel    per-kernel device time per frame from torch.profiler in a run of its own (so its total is not the event-
            timed frame above), for the fine object maps alone and for every map of both passes; the multi-code field
            kernel's time over its algorithmic FLOPs: 1.40 MFLOP per sample for the scene branch plus 0.376 MFLOP per
            sample and code for the object branch (SURVEY.md App. B), against the dense BF16 rate of the H100 SXM data
            sheet (989 TFLOP/s at 700 W).
The card's name and power limit are read in the same run and printed with the numbers, one JSON line per measurement.

  python tools/instances_bench.py [--frames 2] [--reps 3]
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

import torch  # noqa: E402

import eval_geometry_bench as G  # noqa: E402

H, W = G.H, G.W
S, NI = 64, 64
IDS4 = G.IDS
IDS16 = tuple(range(1, 17))
MFLOP_SCENE, MFLOP_OBJECT = 1.40, 0.376


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from object_nerf_b200 import engine, evaluation, rendering, training
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    info = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q, "size": f"{W}x{H}", "samples": "64+64",
            "precision": "bf16"}
    models, emb, lib, fs = G.scene(dev, args.frames)
    batch = evaluation.frame_batch(fs, 0)
    rays = batch["rays"]
    table = lib.embedding_instance.weight.detach()
    grid = engine.GridBuffers.from_module(emb["xyz"])
    packed = {t: engine.packed_for(models[t], True) for t in ("coarse", "fine")}
    render = dict(N_samples=S, N_importance=NI, use_disp=False, white_back=False)

    def loop(ids, keep=False):   # (a); validate_frame's maps are overwritten by its next call: keep copies them
        out = []
        for i in ids:
            o = training.validate_frame(models, emb, lib, evaluation.frame_batch(fs, 0, [i], rays), evaluation._NO_LOSS,
                                        keys=("opacity_instance", "depth_instance", "rgb_instance"), **render)
            out.append({k: v.clone() for k, v in o.items()} if keep else o)
        return out

    def staged(ids):         # (b)
        with torch.no_grad():
            out = {}
            z = engine.sample_coarse(rays, S)
            for typ in ("coarse", "fine"):
                scene, _ = engine.field(rays, z, packed[typ], grid, want_scene=True, want_object=False,
                                        precision="bf16")
                sc = engine.composite(z, scene, None, is_eval=True)
                for k, i in enumerate(ids if typ == "fine" else ()):
                    _, obj = engine.field(rays, z, packed[typ], grid, code_row=table[i], want_scene=False,
                                          want_object=True, precision="bf16")
                    out[(typ, k)] = engine.composite(z, scene, obj, is_eval=True)
                if typ == "coarse":
                    z = engine.sample_pdf_merge(z, sc["weights"], NI, det=True)
            return out

    def fused(ids):          # (c)
        return rendering.render_instances(models, emb, lib, rays, ids, keys=("opacity_instance", "depth_instance",
                                                                              "rgb_instance"), **render)

    for ids in (IDS4, IDS16):
        K = len(ids)
        a = loop(ids, keep=True)
        c = {k: v.clone() for k, v in fused(ids).items()}
        b = staged(ids)
        torch.cuda.synchronize()
        same = all(torch.equal(c[f"{kind}_fine"][:, k], a[k][f"{kind}_fine"])
                   for k in range(K) for kind in ("opacity_instance", "depth_instance", "rgb_instance"))
        same_b = all(torch.equal(c[f"{kind}_fine"][:, k], b[("fine", k)][kind])
                     for k in range(K) for kind in ("opacity_instance", "depth_instance", "rgb_instance"))
        print(json.dumps({**info, "K": K, "measure": "render_instances_bit_identical",
                          "vs_validate_frame_loop": same, "vs_staged": same_b}), flush=True)
        repeats = []
        for _ in range(2):
            ms = {"a_validate_frame_loop": [], "b_staged_per_code": [], "c_render_instances": []}
            for _ in range(args.reps):
                ms["a_validate_frame_loop"].append(timed(lambda: loop(ids)))
                ms["b_staged_per_code"].append(timed(lambda: staged(ids)))
                ms["c_render_instances"].append(timed(lambda: fused(ids)))
            repeats.append({"median_ms": {k: statistics.median(v) for k, v in ms.items()}, "runs_ms": ms})
        print(json.dumps({**info, "K": K, "measure": "ms_per_frame_every_object_map", "repeats": repeats}), flush=True)

    def evaluate(**kw):
        return evaluation.evaluate_frames(models, emb, lib, fs, G.CONF, object_ids=IDS4, **kw)

    evaluate(masks=True)
    repeats = []
    for _ in range(2):
        ms = {"evaluate_frames": [], "evaluate_frames_masks": []}
        for _ in range(args.reps):
            ms["evaluate_frames"].append(timed(evaluate) / args.frames)
            ms["evaluate_frames_masks"].append(timed(lambda: evaluate(masks=True)) / args.frames)
        med = {k: statistics.median(v) for k, v in ms.items()}
        med["extra_pct"] = 100.0 * (med["evaluate_frames_masks"] / med["evaluate_frames"] - 1.0)
        repeats.append({"median_ms": med, "runs_ms": ms})
    print(json.dumps({**info, "K": len(IDS4), "measure": "ms_per_frame_masks", "repeats": repeats}), flush=True)

    from torch.profiler import ProfilerActivity, profile
    every = tuple(f"{k}_{t}" for t in ("coarse", "fine") for k in rendering.INSTANCE_KEYS)
    for maps, keys in (("fine_object_maps", ("opacity_instance", "depth_instance", "rgb_instance")), ("every_map", every)):
        for ids in (IDS4, IDS16):
            K = len(ids)
            run = lambda: rendering.render_instances(models, emb, lib, rays, ids, keys=keys, **render)  # noqa: E731
            run()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    run()
                torch.cuda.synchronize()
            us = {}
            for ev in prof.events():
                if ev.device_type.name == "CUDA":
                    name = next((k for k in ("field_tc_multi_kernel", "field_tc_kernel", "composite_instances_kernel",
                                             "ray_const_kernel") if k in ev.name), "other")
                    us[name] = us.get(name, 0.0) + ev.device_time / 3
            # the multi-code kernel: fine pass only, object branch only (fine_object_maps), or both passes and branches
            samples = H * W * (S + NI) if maps == "fine_object_maps" else H * W * (S + S + NI)
            mflop = MFLOP_OBJECT * K if maps == "fine_object_maps" else MFLOP_SCENE + MFLOP_OBJECT * K
            t = us.get("field_tc_multi_kernel", float("nan")) * 1e-6
            print(json.dumps({**info, "K": K, "maps": maps, "measure": "kernels_profiled",
                              "device_us_per_frame": us, "profiled_kernel_total_us_per_frame": sum(us.values()),
                              "multi_kernel_samples_per_frame": samples, "multi_kernel_mflop_per_sample": mflop,
                              "multi_kernel_ns_per_sample": 1e9 * t / samples,
                              "multi_kernel_algorithmic_TFLOP_per_s": samples * mflop * 1e6 / t / 1e12,
                              "share_of_989_TFLOPs_datasheet": samples * mflop * 1e6 / t / 989e12}), flush=True)

if __name__ == "__main__":
    main()
