"""What scoring held-out views costs (evaluation.evaluate_frames, onerf_image_metrics).

A synthetic 640x480 voxel scene (64 + 64 samples, bf16) seen by 10 cameras, with label images holding K = 4 objects.
  frame    ms per frame of evaluate_frames (rays, one render, metrics) against validate_frame alone on the same frames
           (rays and the one render, no metrics), alternated, --reps passes of all frames each, the alternation repeated
           once;
  kernel   device time of one frame's onerf_image_metrics + finalize (K + 1 = 5 columns, window 3 and 11) against a torch
           fp32 restatement of the same definition (masking, F.pad reflect, depthwise conv2d of the five moments,
           ssim_map, clamp, masked means), CUDA events over --launches calls each, alternated; the two results are
           compared first.
The card's name and power limit are read in the same run and printed with the numbers, one JSON line per measurement.

  python tools/eval_bench.py [--reps 3] [--launches 50]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as Fn  # noqa: E402

H, W, N_FRAMES, IDS = 480, 640, 10, (3, 5, 7, 9)
CONF = {"model": {"N_samples": 64, "N_importance": 64, "use_disp": False}}


def scene(dev):
    from object_nerf_b200 import Embedding, frames, synthetic as S
    models = {"coarse": S.make_model(S.make_weights(20, True, 8.0, 1.0, rgb_gain=24.0), True, dev),
              "fine": S.make_model(S.make_weights(1020, True, 8.0, 1.0, rgb_gain=24.0), True, dev)}
    emb = {"xyz": S.GridModule(S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05,
                                           n_rows=800000)).to(dev), "dir": Embedding(3, 4)}
    lib = S.make_code_library(S.make_codes(7)).to(dev)
    rng = np.random.default_rng(0)
    poses = []
    for _ in range(N_FRAMES):
        cam = np.array([-1.6, 0.1, 0.15]) + rng.normal(size=3) * 0.1
        fwd = -cam / np.linalg.norm(cam)
        right = np.cross(fwd, [0, 0, 1.0])
        right /= np.linalg.norm(right)
        poses.append(np.concatenate([np.stack([right, np.cross(right, fwd), -fwd], 1), cam[:, None]], 1))
    labels = np.zeros((N_FRAMES, H, W), np.uint16)
    for k, i in enumerate(IDS):                        # one block per object, a quarter of the frame each
        labels[:, (k // 2) * H // 2:(k // 2 + 1) * H // 2, (k % 2) * W // 2:(k % 2 + 1) * W // 2] = i
    fs = frames.FrameSet(np.stack(poses).astype(np.float32), rng.integers(0, 256, (N_FRAMES, H, W, 3), dtype=np.uint8),
                         np.zeros((N_FRAMES, H, W), np.float32), labels, focal=0.5 * W / math.tan(math.radians(30)),
                         near=0.15, far=3.0, scale_factor=1.0, instance_ids=(IDS[0],), device=dev)
    return models, emb, lib, fs


def torch_metrics(pred_s, pred_o, gt, valid, labels, ids, window):
    """The definition in fp32 torch (metrics.py): (psnr (K+1,), ssim (K+1,))."""
    r = window // 2
    g1 = torch.exp(-(torch.arange(window, device=gt.device, dtype=torch.float64) - r) ** 2 / (2 * 1.5 ** 2))
    g1 = g1 / g1.sum()
    g = torch.outer(g1, g1).float()[None, None].expand(15, 1, window, window)
    lab = labels.to(torch.int32) & 0xFFFF
    masks = torch.stack([valid.bool()] + [valid.bool() & (lab == i) for i in ids]).view(-1, 1, H, W)
    preds = torch.stack([pred_s] + [pred_o] * len(ids)).view(-1, H, W, 3).permute(0, 3, 1, 2)
    p = preds * masks
    q = gt.view(1, H, W, 3).permute(0, 3, 1, 2) * masks
    x = torch.cat([p, q, p * p, q * q, p * q], 1)
    f = Fn.conv2d(Fn.pad(x, (r, r, r, r), mode="reflect"), g, groups=15)
    mp, mq, pp, qq, pq = f.split(3, 1)
    s = ((2 * mp * mq + 1e-4) * (2 * (pq - mp * mq) + 9e-4)) / ((mp * mp + mq * mq + 1e-4) * (pp - mp * mp + qq - mq * mq
                                                                                              + 9e-4))
    n = 3 * masks.sum((1, 2, 3))
    ssim = (s.clamp(0, 1) * masks).sum((1, 2, 3)) / n
    psnr = -10 * torch.log10(((p - q) ** 2).sum((1, 2, 3)) / n)
    return psnr, ssim


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    args = ap.parse_args()
    from object_nerf_b200 import evaluation, metrics, training
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    info = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q, "size": f"{W}x{H}", "frames": N_FRAMES,
            "K": len(IDS), "samples": "64+64", "precision": "bf16"}
    models, emb, lib, fs = scene(dev)

    def evaluate():
        evaluation.evaluate_frames(models, emb, lib, fs, CONF, object_ids=IDS)

    def render_only():
        rays = torch.empty(H * W, 8, device=dev)
        for f in range(N_FRAMES):
            batch = evaluation.frame_batch(fs, f, IDS, rays)
            training.validate_frame(models, emb, lib, batch, evaluation._NO_LOSS, N_samples=64, N_importance=64,
                                    use_disp=False, white_back=False, keys=("rgb", "rgb_instance"))

    evaluate()
    render_only()
    torch.cuda.synchronize()
    repeats = []
    for _ in range(2):
        ms = {"evaluate_frames": [], "validate_frame_only": []}
        for _ in range(args.reps):
            ms["evaluate_frames"].append(timed(evaluate) / N_FRAMES)
            ms["validate_frame_only"].append(timed(render_only) / N_FRAMES)
        med = {k: statistics.median(v) for k, v in ms.items()}
        med["metrics_share_pct"] = 100.0 * (med["evaluate_frames"] / med["validate_frame_only"] - 1.0)
        repeats.append(med)
    print(json.dumps({**info, "measure": "ms_per_frame", "repeats": repeats}), flush=True)

    # the metrics kernel alone on one rendered frame
    batch = evaluation.frame_batch(fs, 0, IDS)
    out = training.validate_frame(models, emb, lib, batch, evaluation._NO_LOSS, N_samples=64, N_importance=64,
                                  use_disp=False, white_back=False, keys=("rgb", "rgb_instance"))
    pred_s, pred_o = out["rgb_fine"].clone(), out["rgb_instance_fine"].clone()
    gt, valid, labels = batch["rgbs"], batch["valid_mask"], fs.tensors["labels"][0]
    for window in (3, 11):
        plan = metrics.MetricsPlan(H, W, IDS, window, 1, dev)

        def kernel():
            for _ in range(args.launches):
                plan.accumulate(pred_s, gt, valid, pred_o, labels)
                plan.finalize(0)

        def reference():
            for _ in range(args.launches):
                torch_metrics(pred_s, pred_o, gt, valid, labels, IDS, window)

        kernel()
        tp, ts = torch_metrics(pred_s, pred_o, gt, valid, labels, IDS, window)
        agree = {"max_abs_psnr_diff_db": float((plan.psnr[0] - tp).abs().max()),
                 "max_abs_ssim_diff": float((plan.ssim[0] - ts).abs().max())}
        reference()
        us = {"onerf_image_metrics": [], "torch_fp32_conv2d": []}
        for _ in range(3):
            us["onerf_image_metrics"].append(1000 * timed(kernel) / args.launches)
            us["torch_fp32_conv2d"].append(1000 * timed(reference) / args.launches)
        print(json.dumps({**info, "measure": "metrics_us_per_frame", "window": window, "columns": len(IDS) + 1,
                          "median_us": {k: statistics.median(v) for k, v in us.items()}, "runs_us": us,
                          "agreement_vs_fp32_torch": agree}), flush=True)


if __name__ == "__main__":
    main()
