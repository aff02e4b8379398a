"""Frame time of render_rays_multi (the editing path) with many ray sets.

For each frame size and ray-set list, renders the whole frame in chunks of 4 096 rays (64 + 64 samples per set, bf16,
synthetic scene of bench.py) and prints one JSON line per configuration: ms per frame (CUDA events, median of --reps
frames after one warm-up frame) and the fraction of object rows the field kernel evaluated (the rays that hit the set's
box; before box culling every object row was evaluated).  Object set k gets an axis-aligned box of half-size 0.12 around
a point at depth 1 on a random pixel's ray; near / far come from the slab test, misses get near = far = 0 as in
EditableRenderer.  The scene set carries two removed-object boxes.  A configuration the library refuses prints its error.

  python tools/edit_bench.py                      # 320x240 and 640x480: [0,4,4] with bench.py's random near / far
                                                  # (30 % misses), and [0] + [4] * k with boxes, k in 2 8 24 40
  python tools/edit_bench.py --bench-leg          # only bench.py's edit leg configuration (640x480, [0,4,4], 30 % misses)
  python tools/edit_bench.py --bench-leg --noise-std 1   # the same with sigma noise drawn in the compositing kernels
  python tools/edit_bench.py --frame [--reps 5]   # a camera frame, three routes (below)
  torchrun --nproc-per-node N tools/edit_bench.py --frame    # ... plus the frame sharded over N GPUs

--frame renders a 640x480 pinhole camera on the same scene with sets [0, 4, 4] (the duplicate moved; both object boxes
in view) and two removed-object boxes, 64 + 64 samples, bf16, through three routes:
  A  what EditableRenderer.render_edit does over the drop-in: camera_rays per set, render_rays_multi in 4 096-ray
     chunks, .cpu() of every key of every chunk;
  B  editing.render_frame with every key, copied to the host;
  C  editing.render_frame with rgb_fine / depth_fine only, copied to the host.
It first asserts that the routes' outputs are bit-identical, then times them alternately (wall clock from a synchronised
start to the host copy, median of --reps).  Under torchrun every rank renders its tile of C and the tiles are all-gathered
inside the timed region; rank 0 prints the slowest rank's median and the scaling efficiency against one GPU rendering the
whole frame (t_1 / (N t_N)).  The card's name and power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

CHUNK = 4096


class Box:   # the attributes of BBoxRayHelper that the removed-object mask reads (as bench.py's edit leg)
    def __init__(self, b):
        self.scale_factor = 2.0
        self.pose_avg = np.eye(4)
        self.axis_align_mat = np.eye(4)
        self.axis_align_mat[:3, 3] = [0.05 * b, -0.1, 0.0]
        lo = np.array([-0.5, -0.4, -0.3]) + 0.1 * b
        self.bbox_bounds = np.array([lo, lo + 0.6])


def scene(dev):
    from object_nerf_b200 import Embedding, synthetic as S
    wc = S.make_weights(0, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)
    wf = S.make_weights(1000, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0)
    grid = S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05, n_rows=800000)
    models = {"coarse": S.make_model(wc, True, dev), "fine": S.make_model(wf, True, dev)}
    emb = {"xyz": S.GridModule(grid).to(dev), "dir": Embedding(3, 4)}
    return models, emb, S.make_code_library(S.make_codes(2)).to(dev)


def box_sets(rays, k, rng):
    """k object ray sets, each with near / far from the slab test against its own box"""
    o, d = rays[:, 0:3], rays[:, 3:6]
    sets, hit_frac = [], []
    for _ in range(k):
        p = int(rng.integers(rays.shape[0]))
        c = o[p] + d[p] * 1.0
        lo, hi = c - 0.12, c + 0.12
        inv = 1.0 / torch.where(d.abs() < 1e-9, torch.full_like(d, 1e-9), d)
        t1, t2 = (lo - o) * inv, (hi - o) * inv
        tmin = torch.minimum(t1, t2).amax(1).clamp(min=0)
        tmax = torch.maximum(t1, t2).amin(1)
        hit = tmax > tmin
        r = rays.clone()
        r[:, 6] = torch.where(hit, tmin, torch.zeros_like(tmin))
        r[:, 7] = torch.where(hit, tmax, torch.zeros_like(tmax))
        sets.append(r)
        hit_frac.append(hit.float().mean().item())
    return sets, hit_frac


def bench_sets(rays, rng):
    """bench.py's edit leg: two object sets with random near / far and 30 % misses"""
    n = rays.shape[0]
    sets, hit_frac = [], []
    for _ in range(2):
        r = rays.clone()
        near = torch.from_numpy(rng.uniform(0.4, 1.2, size=n).astype(np.float32)).to(rays.device)
        far = near + torch.from_numpy(rng.uniform(0.2, 0.9, size=n).astype(np.float32)).to(rays.device)
        miss = torch.from_numpy(rng.random(n) < 0.3).to(rays.device)
        near[miss], far[miss] = 0, 0
        r[:, 6], r[:, 7] = near, far
        sets.append(r)
        hit_frac.append(1.0 - miss.float().mean().item())
    return sets, hit_frac


def time_frame(models, emb, lib, sets, ids, reps, noise_std=0.0):
    from object_nerf_b200.multi_rendering import render_rays_multi
    boxes = {"4": Box(0), "6": Box(1)}
    n = sets[0].shape[0]

    def frame():
        with torch.no_grad():
            for i in range(0, n, CHUNK):
                render_rays_multi(models, emb, lib, [s[i:i + CHUNK] for s in sets], ids, N_samples=64, N_importance=64,
                                  noise_std=noise_std, chunk=CHUNK, white_back=False, background_skip_bbox=boxes,
                                  precision="bf16")

    frame()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        frame()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms)


class FrameBox:   # BBoxRayHelper's attributes for the camera frame: a box of half-size `half` around `center` (world units)
    def __init__(self, center, half, scale_factor):
        self.scale_factor = scale_factor
        self.pose_avg = np.eye(4)
        self.axis_align_mat = np.eye(4)
        self.bbox_bounds = np.array([np.asarray(center) - half, np.asarray(center) + half])


def frame_setup(h=480, w=640, scale_factor=2.0):
    """camera (focal, near, far, scale factor), sets [0, 4, 4] with the duplicate moved, two removed boxes"""
    cam = np.array([-3.2, 0.2, 0.3])
    fwd = -cam / np.linalg.norm(cam)
    right = np.cross(fwd, [0.0, 0.0, 1.0])
    right /= np.linalg.norm(right)
    Twc = np.eye(4)
    Twc[:3, :3] = np.stack([right, np.cross(right, fwd), -fwd], 1)
    Twc[:3, 3] = cam

    def toc(shift):
        transform = np.eye(4)
        transform[:3, 3] = shift
        t = np.linalg.inv(transform) @ Twc
        t[:3, 3] /= scale_factor
        return torch.from_numpy(t).float()[:3, :4]
    box4, box6 = FrameBox([0.3, 0.1, 0.05], 0.3, scale_factor), FrameBox([-0.35, -0.25, 0.0], 0.25, scale_factor)
    sets = [(0, toc([0, 0, 0]), None, 0.0), (4, toc([0.05, 0.35, 0.0]), box4, 0.0), (4, toc([-0.05, -0.5, 0.0]), box4, 0.0)]
    cam_args = dict(H=h, W=w, focal=0.5 * w / np.tan(np.radians(30.0)), near=0.3, far=6.0, scale_factor=scale_factor)
    return cam_args, sets, {"4": box4, "6": box6}


def frame_mode(args):
    import torch.distributed as dist
    from object_nerf_b200 import editing
    from object_nerf_b200.multi_rendering import render_rays_multi
    from object_nerf_b200.ray_utils import camera_rays
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    models, emb, lib = scene(dev)
    cam, sets, removed = frame_setup()
    H, W = cam["H"], cam["W"]
    kw = dict(background_skip_bbox=removed, N_samples=64, N_importance=64, precision="bf16")
    ids = [s[0] for s in sets]

    def route_a():
        rays = [camera_rays(H, W, cam["focal"], Toc, cam["near"], cam["far"], cam["scale_factor"], box=box,
                            bbox_enlarge=enl, device=dev) for _, Toc, box, enl in sets]
        parts = {}
        with torch.no_grad():
            for i in range(0, H * W, CHUNK):
                out = render_rays_multi(models, emb, lib, [r[i:i + CHUNK] for r in rays], ids, perturb=0, noise_std=0,
                                        chunk=CHUNK, **kw)
                for k, v in out.items():
                    parts.setdefault(k, []).append(v.detach().cpu())
        return {k: torch.cat(v, 0) for k, v in parts.items()}

    def route_frame(keys=None, group=None):
        out = editing.render_frame(models, emb, lib, H, W, cam["focal"], sets, cam["near"], cam["far"],
                                   cam["scale_factor"], keys=keys, group=group, **kw)
        return {k: v.cpu() for k, v in out.items()}

    routes = {"A": route_a, "B": route_frame, "C": lambda: route_frame(["rgb_fine", "depth_fine"])}
    q = subprocess.run(["nvidia-smi", "-i", str(dev.index), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    info = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q, "size": f"{W}x{H}", "ids": ids, "world": world}
    if rank == 0:
        outs = {name: fn() for name, fn in routes.items()}
        a, b, c = outs["A"], outs["B"], outs["C"]
        assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a), "routes A and B differ"
        assert list(c) == ["rgb_fine", "depth_fine"] and all(torch.equal(c[k], b[k]) for k in c), "route C differs"
        hit = [float((b["z_vals_coarse"][b["obj_ids_coarse"] == k] > 0).float().mean()) for k in (1, 2)]
        ms = {name: [] for name in routes}
        for _ in range(args.reps):
            for name, fn in routes.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ms[name].append((time.perf_counter() - t0) * 1e3)
        med = {name: statistics.median(v) for name, v in ms.items()}
        print(json.dumps({**info, "mode": "frame", "bit_identical": True, "object_set_hit_fraction": hit,
                          "ms_per_frame": med, "runs_ms": ms}), flush=True)
    if world > 1:
        group = dist.group.WORLD
        a, b = editing.parallel.shard_bounds(H * W, world, rank)
        full = route_frame(["rgb_fine", "depth_fine"])
        sharded = route_frame(["rgb_fine", "depth_fine"], group)
        assert all(torch.equal(full[k], sharded[k]) for k in full), "sharded frame differs"
        t1, tn = [], []
        for _ in range(args.reps):
            for arm, grp in (("n", group), ("1", None)):
                dist.barrier()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if grp is not None or rank == 0:
                    route_frame(["rgb_fine", "depth_fine"], grp)
                torch.cuda.synchronize()
                (tn if arm == "n" else t1).append((time.perf_counter() - t0) * 1e3)
        worst = torch.tensor([statistics.median(tn)], device=dev)
        dist.all_reduce(worst, op=dist.ReduceOp.MAX)
        if rank == 0:
            m1, mn = statistics.median(t1), worst.item()
            print(json.dumps({**info, "mode": "frame sharded C", "tile_rows_rank0": b - a, "ms_per_frame_1gpu": m1,
                              "ms_per_frame_sharded": mn, "scaling_efficiency": m1 / (world * mn)}), flush=True)
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="320x240,640x480")
    ap.add_argument("--counts", default="2,8,24,40", help="k of the set lists [0] + [4] * k")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--bench-leg", action="store_true")
    ap.add_argument("--frame", action="store_true")
    ap.add_argument("--noise-std", type=float, default=0.0,
                    help="sigma noise of render_rays_multi (drawn in the compositing kernels); 0 = the editing renderer's call")
    args = ap.parse_args()
    if args.frame:
        return frame_mode(args)
    from object_nerf_b200 import synthetic as S
    dev = torch.device("cuda:0")
    models, emb, lib = scene(dev)
    gpu = torch.cuda.get_device_name(dev)
    if args.bench_leg:
        rays = S.pinhole_rays(480, 640).to(dev)
        sets, hf = bench_sets(rays, np.random.default_rng(7))
        ms = time_frame(models, emb, lib, [rays] + sets, [0, 4, 4], args.reps, args.noise_std)
        print(json.dumps({"config": "bench edit leg", "size": "640x480", "ids": [0, 4, 4], "ms_per_frame": ms,
                          "noise_std": args.noise_std, "object_rows_evaluated": statistics.mean(hf), "gpu": gpu}))
        return
    for size in args.sizes.split(","):
        w, h = (int(x) for x in size.split("x"))
        rays = S.pinhole_rays(h, w).to(dev)
        lists = [("[0,4,4]", 2)] + [(f"[0]+[4]*{k}", int(k)) for k in args.counts.split(",")]
        for name, k in lists:
            rng = np.random.default_rng(100 + k)
            sets, hf = bench_sets(rays, rng) if name == "[0,4,4]" else box_sets(rays, k, rng)
            row = {"size": size, "ids": name, "n_sets": k + 1, "object_rows_evaluated": statistics.mean(hf), "gpu": gpu}
            try:
                row["ms_per_frame"] = time_frame(models, emb, lib, [rays] + sets, [0] + [4] * k, args.reps, args.noise_std)
            except RuntimeError as ex:
                row["error"] = str(ex)[:160]
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
