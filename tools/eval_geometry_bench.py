"""What scoring depth and object masks of held-out views costs (evaluation.evaluate_frames(depth=, masks=),
onerf_depth_metrics, onerf_mask_metrics).

A synthetic 640x480 voxel scene (64 + 64 samples, bf16) seen by --frames cameras, with label images holding K = 4
objects and ground-truth depths.
  frame    ms per frame of evaluate_frames(depth=True) against evaluate_frames() on the same frames, alternated, --reps
           calls each, the alternation repeated once; then the same for masks=True (K more renders per frame);
  kernel   device time of one frame's onerf_depth_metrics + finalize (K + 1 = 5 columns) and of K onerf_mask_metrics +
           finalize, called from Python and replayed from a CUDA graph, against a torch fp64 restatement of the same
           definitions (column masks, clamp, the sums, the ratios), CUDA events over --launches calls each,
           alternated; the results are compared first.
The card's name and power limit are read in the same run and printed with the numbers, one JSON line per measurement.

  python tools/eval_geometry_bench.py [--frames 10] [--reps 3] [--launches 200]
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

H, W, IDS, SCALE = 480, 640, (3, 5, 7, 9), 1.0
CONF = {"model": {"N_samples": 64, "N_importance": 64, "use_disp": False}}


def scene(dev, n_frames):
    from object_nerf_b200 import Embedding, frames, synthetic as S
    models = {"coarse": S.make_model(S.make_weights(20, True, 8.0, 1.0, rgb_gain=24.0), True, dev),
              "fine": S.make_model(S.make_weights(1020, True, 8.0, 1.0, rgb_gain=24.0), True, dev)}
    emb = {"xyz": S.GridModule(S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05,
                                           n_rows=800000)).to(dev), "dir": Embedding(3, 4)}
    lib = S.make_code_library(S.make_codes(7)).to(dev)
    rng = np.random.default_rng(0)
    poses = []
    for _ in range(n_frames):
        cam = np.array([-1.6, 0.1, 0.15]) + rng.normal(size=3) * 0.1
        fwd = -cam / np.linalg.norm(cam)
        right = np.cross(fwd, [0, 0, 1.0])
        right /= np.linalg.norm(right)
        poses.append(np.concatenate([np.stack([right, np.cross(right, fwd), -fwd], 1), cam[:, None]], 1))
    labels = np.zeros((n_frames, H, W), np.uint16)
    for k, i in enumerate(IDS):                        # one block per object, a quarter of the frame each
        labels[:, (k // 2) * H // 2:(k // 2 + 1) * H // 2, (k % 2) * W // 2:(k % 2 + 1) * W // 2] = i
    depths = rng.uniform(0.5, 3.0, (n_frames, H, W)).astype(np.float32)
    depths[rng.random((n_frames, H, W)) < 0.05] = 0
    fs = frames.FrameSet(np.stack(poses).astype(np.float32), rng.integers(0, 256, (n_frames, H, W, 3), dtype=np.uint8),
                         depths, labels, focal=0.5 * W / math.tan(math.radians(30)), near=0.15, far=3.0,
                         scale_factor=SCALE, instance_ids=(IDS[0],), device=dev)
    return models, emb, lib, fs


def torch_depth(pred_s, pred_o, gt, valid, labels, ids, scale, d_min, d_max):
    """The depth definition in fp64 torch: (K+1, 7)."""
    lab = labels.to(torch.int32) & 0xFFFF
    m0 = valid.bool() & (gt > 0)
    masks = torch.stack([m0] + [m0 & (lab == i) for i in ids]).double()
    g = gt.double() * scale
    d = torch.stack([pred_s] + [pred_o] * len(ids)).double() * scale
    d = torch.where(d.isnan(), d, d.clamp(d_min, d_max))
    gs = torch.where(masks > 0, g, torch.ones_like(g))        # keeps the excluded pixels finite
    e = d - gs
    r = torch.maximum(d / gs, gs / d)
    n = masks.sum(1)
    cnt = [(torch.where(r.isnan(), r, (r < 1.25 ** i).double()) * masks).sum(1) for i in (1, 2, 3)]
    return torch.stack([(e.abs() / gs * masks).sum(1) / n, (e * e / gs * masks).sum(1) / n,
                        ((e * e * masks).sum(1) / n).sqrt(), ((((d.log() - gs.log()) ** 2) * masks).sum(1) / n).sqrt(),
                        cnt[0] / n, cnt[1] / n, cnt[2] / n], 1)


def torch_masks(opacities, labels, valid, ids, tau):
    """The mask definition in fp64 torch: (iou (K,), opacity_l1 (K,))."""
    lab = labels.to(torch.int32) & 0xFFFF
    v = valid.bool()
    o = torch.stack(opacities)
    G = torch.stack([lab == i for i in ids])
    P = o >= tau
    inter = (P & G & v).double().sum(1)
    union = ((P | G) & v).double().sum(1)
    l1 = ((o.double() - G.double()).abs() * v).sum(1) / v.double().sum()
    return inter / union, l1


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    from object_nerf_b200 import evaluation, metrics, training
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    info = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q, "size": f"{W}x{H}", "frames": args.frames,
            "K": len(IDS), "samples": "64+64", "precision": "bf16"}
    models, emb, lib, fs = scene(dev, args.frames)
    F = args.frames

    def evaluate(**kw):
        return evaluation.evaluate_frames(models, emb, lib, fs, CONF, object_ids=IDS, **kw)

    # the colour scores must not move with the new flags
    base, full = evaluate(), evaluate(depth=True, masks=True)
    torch.cuda.synchronize()
    same = all(torch.equal(base[k].nan_to_num(), full[k].nan_to_num()) for k in base)
    print(json.dumps({**info, "measure": "colour_scores_bit_identical_with_depth_and_masks", "value": same,
                      "mean_depth_metrics": full["mean_depth_metrics"].tolist(),
                      "mean_iou_objects": full["mean_iou_objects"].tolist()}), flush=True)

    for flag in ("depth", "masks"):
        repeats = []
        for _ in range(2):
            ms = {"evaluate_frames": [], f"evaluate_frames_{flag}": []}
            for _ in range(args.reps):
                ms["evaluate_frames"].append(timed(evaluate) / F)
                ms[f"evaluate_frames_{flag}"].append(timed(lambda: evaluate(**{flag: True})) / F)
            med = {k: statistics.median(v) for k, v in ms.items()}
            med["extra_pct"] = 100.0 * (med[f"evaluate_frames_{flag}"] / med["evaluate_frames"] - 1.0)
            repeats.append({"median_ms": med, "runs_ms": ms})
        print(json.dumps({**info, "measure": f"ms_per_frame_{flag}", "repeats": repeats}), flush=True)

    # the kernels alone on one rendered frame
    batch = evaluation.frame_batch(fs, 0, IDS)
    out = training.validate_frame(models, emb, lib, batch, evaluation._NO_LOSS, N_samples=64, N_importance=64,
                                  use_disp=False, white_back=False, keys=("depth", "depth_instance"))
    pred_s, pred_o = out["depth_fine"].clone(), out["depth_instance_fine"].clone()
    gt, valid, labels = fs.tensors["depths"][0], batch["valid_mask"], fs.tensors["labels"][0]
    ops = []
    for i in IDS:
        o = training.validate_frame(models, emb, lib, evaluation.frame_batch(fs, 0, [i]), evaluation._NO_LOSS,
                                    N_samples=64, N_importance=64, use_disp=False, white_back=False,
                                    keys=("opacity_instance",))
        ops.append(o["opacity_instance_fine"].clone())
    d_min, d_max = 1e-3, 10.0
    dplan = metrics.DepthMetricsPlan(H, W, IDS, SCALE, (d_min, d_max), 1, dev)
    mplan = metrics.MaskMetricsPlan(H, W, IDS, 0.5, 1, dev)

    def depth_kernel():
        for _ in range(args.launches):
            dplan.accumulate(pred_s, gt, valid, pred_o, labels)
            dplan.finalize(0)

    def depth_torch():
        for _ in range(args.launches):
            torch_depth(pred_s, pred_o, gt, valid, labels, IDS, SCALE, d_min, d_max)

    def mask_kernel():
        for _ in range(args.launches):
            for k in range(len(IDS)):
                mplan.accumulate(k, ops[k], labels, valid)
            mplan.finalize(0)

    def mask_torch():
        for _ in range(args.launches):
            torch_masks(ops, labels, valid, IDS, 0.5)

    def depth_once():
        dplan.accumulate(pred_s, gt, valid, pred_o, labels)
        dplan.finalize(0)

    def mask_once():
        for k in range(len(IDS)):
            mplan.accumulate(k, ops[k], labels, valid)
        mplan.finalize(0)

    def graphed(once):
        """--launches calls captured in one CUDA graph: device time without the Python and launch overhead."""
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            once()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(args.launches):
                once()
        return g.replay

    depth_kernel()
    mask_kernel()
    depth_graph, mask_graph = graphed(depth_once), graphed(mask_once)
    td = torch_depth(pred_s, pred_o, gt, valid, labels, IDS, SCALE, d_min, d_max)
    ti, tl = torch_masks(ops, labels, valid, IDS, 0.5)
    agree = {"max_rel_depth_diff": float(((dplan.out[0].double() - td).abs() / td.abs().clamp_min(1e-30)).max()),
             "max_abs_iou_diff": float((mplan.iou[0].double() - ti).abs().max()),
             "max_abs_opacity_l1_diff": float((mplan.opacity_l1[0].double() - tl).abs().max())}
    moved = H * W * (4 + 4 + 4 + 1 + 2)                           # scene, object, gt, valid, labels
    for name, kern, graph, ref in (("depth", depth_kernel, depth_graph, depth_torch),
                                   ("masks", mask_kernel, mask_graph, mask_torch)):
        ref()
        graph()
        us = {f"onerf_{name}_metrics": [], f"onerf_{name}_metrics_graph": [], "torch_fp64": []}
        for _ in range(3):
            us[f"onerf_{name}_metrics"].append(1000 * timed(kern) / args.launches)
            us[f"onerf_{name}_metrics_graph"].append(1000 * timed(graph) / args.launches)
            us["torch_fp64"].append(1000 * timed(ref) / args.launches)
        med = {k: statistics.median(v) for k, v in us.items()}
        rec = {**info, "measure": f"{name}_metrics_us_per_frame", "median_us": med, "runs_us": us,
               "agreement_vs_fp64_torch": agree}
        if name == "depth":
            rec["bytes_read"] = moved
            rec["achieved_GBps_graph"] = moved / (med["onerf_depth_metrics_graph"] * 1e3)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
