"""One validation image three ways: a 640 x 480 image, 64 + 64 samples, voxel model, bf16, synthetic scene.

  A  the reference-shaped validation_step over the drop-in (train.py:73-105, 182-223): render_rays in 32 768-ray
     chunks, every result key kept and torch.cat'ed, losses.TotalLoss, torch psnr with a boolean mask
  B  training.validate_frame, eager
  C  B replayed from a CUDA graph

A and B must agree first (maps bit-identical, loss within 1e-6).  Then the routes alternate image by image after a
warm-up of every shape.  Per route: median and spread of the device time (events) and of the wall time ending in a
synchronise, library launches per image, the peak of torch's allocator during the route, and the card's name and power
limit read in this run.  There is no CPU mode: without a GPU the script fails.

    python tools/validate_bench.py [--images 20] [--chunk 65536]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

LOSS_CONF = dict(color_loss_weight=1.0, depth_loss_weight=0.1, opacity_loss_weight=100.0,
                 instance_color_loss_weight=1.0, instance_depth_loss_weight=0.1)
RENDER = dict(N_samples=64, N_importance=64, use_disp=False, white_back=False)
KEYS = ("rgb", "depth", "rgb_instance", "depth_instance", "opacity_instance")


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, limit = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": limit}


def make_scene(dev, H, W):
    from object_nerf_b200 import Embedding, synthetic as S
    models = {"coarse": S.make_model(S.make_weights(0, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0), True, dev).eval(),
              "fine": S.make_model(S.make_weights(1000, True, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=24.0), True, dev).eval()}
    emb = S.GridModule(S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05, n_rows=800000)).to(dev)
    lib = S.make_code_library(S.make_codes(2)).to(dev)
    n = H * W
    rng = np.random.default_rng(11)
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a.astype(np.float32))).to(dev)[None]
    batch = {"rays": S.pinhole_rays(H, W).to(dev)[None], "rgbs": f(rng.random((n, 3))),
             "depths": f(np.where(rng.random(n) < 0.8, rng.uniform(0.3, 2.5, size=n), 0.0)),
             "valid_mask": torch.from_numpy(rng.random(n) < 0.9).to(dev)[None],
             "instance_mask": torch.from_numpy(rng.random(n) < 0.3).to(dev)[None],
             "instance_mask_weight": f(np.where(rng.random(n) < 0.5, 1.0, 0.05)),
             "instance_ids": torch.from_numpy(rng.choice([4, 6], size=n)).to(dev).view(1, n, 1)}
    return models, {"xyz": emb, "dir": Embedding(3, 4)}, lib, batch


def route_a(scene):
    from object_nerf_b200 import render_rays
    from object_nerf_b200.losses import TotalLoss
    models, embeddings, lib, batch = scene
    with torch.no_grad():
        mask = (batch["valid_mask"] * batch["instance_mask"]).view(-1, 1).repeat(1, 3)
        rays, rgbs = batch["rays"].squeeze(), batch["rgbs"].squeeze()
        codes = lib(batch)["embedding_instance"]
        parts = {}
        for i in range(0, rays.shape[0], 32768):
            out = render_rays(models, embeddings, rays[i:i + 32768], embedding_instance=codes[i:i + 32768], perturb=0,
                              noise_std=0, chunk=32768, is_eval=True, rays_in_bbox=False, frustum_bound_th=0.025,
                              precision="bf16", **RENDER)
            for k, v in out.items():
                parts.setdefault(k, []).append(v)
        results = {k: torch.cat(v, 0) for k, v in parts.items()}
        loss_sum, loss_dict = TotalLoss(LOSS_CONF)(results, batch)
        value = ((results["rgb_fine"] - rgbs) ** 2)[mask]
        psnr = -10 * torch.log10(torch.mean(value))
    return dict(results, loss_sum=loss_sum, psnr=psnr, loss_dict=loss_dict)


def route_b(scene, chunk):
    from object_nerf_b200 import training
    models, embeddings, lib, batch = scene
    return training.validate_frame(models, embeddings, lib, batch, LOSS_CONF, chunk=chunk, keys=KEYS, precision="bf16",
                                   **RENDER)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=20)
    ap.add_argument("--chunk", type=int, default=65536)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("validate_bench.py measures on a CUDA device; none is available")
    from object_nerf_b200 import _lib
    dev = torch.device("cuda:0")
    info = card()
    scene = make_scene(dev, args.height, args.width)

    # agreement, which is also the warm-up of every shape
    a = route_a(scene)
    b = {k: v.clone() for k, v in route_b(scene, args.chunk).items()}
    torch.cuda.synchronize()
    for k in KEYS:
        assert torch.equal(a[f"{k}_fine"], b[f"{k}_fine"]), f"{k}_fine differs between routes A and B"
    rel = abs(a["loss_sum"].item() - b["loss_sum"].item()) / abs(a["loss_sum"].item())
    assert rel <= 1e-6, ("loss_sum", a["loss_sum"].item(), b["loss_sum"].item())
    assert abs(a["psnr"].item() - b["psnr"].item()) <= 1e-4 * abs(a["psnr"].item()), (a["psnr"].item(), b["psnr"].item())
    del a
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            held = route_b(scene, args.chunk)
    graph.replay()
    torch.cuda.synchronize()
    for k in KEYS:
        assert torch.equal(held[f"{k}_fine"], b[f"{k}_fine"]), f"{k}_fine differs between routes B and C"
    assert torch.allclose(held["loss_sum"], b["loss_sum"], rtol=1e-6, atol=0), "loss_sum differs between routes B and C"
    torch.cuda.empty_cache()

    routes = {"A": lambda: route_a(scene), "B": lambda: route_b(scene, args.chunk), "C": graph.replay}
    dev_ms, wall_ms, launches, peak = ({r: [] for r in routes} for _ in range(4))
    for _ in range(args.images):
        for name, fn in routes.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            before = _lib.launch_count(dev)
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            start.record()
            out = fn()
            end.record()
            torch.cuda.synchronize()
            wall_ms[name].append((time.perf_counter() - t0) * 1e3)
            dev_ms[name].append(start.elapsed_time(end))
            launches[name].append(_lib.launch_count(dev) - before)
            peak[name].append(torch.cuda.max_memory_allocated())
            del out

    def stats(v):
        return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}

    # memory the process holds whichever route runs (models, grid, batch, B's plan and workspace, C's graph pool)
    result = {"image": [args.height, args.width], "samples": [64, 64], "chunk": args.chunk, "images": args.images, **info,
              "resident_bytes_between_images": torch.cuda.memory_allocated(), "routes": {}}
    for name in routes:
        result["routes"][name] = {"device_ms": stats(dev_ms[name]), "wall_ms": stats(wall_ms[name]),
                                  "library_launches_per_image": statistics.median(launches[name]),
                                  "peak_allocated_bytes": max(peak[name])}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
