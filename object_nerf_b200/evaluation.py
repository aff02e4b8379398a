"""Held-out views scored on the device: per-frame PSNR and SSIM of the scene and of each object over a frame store
(frames.FrameSet, typically `FrameSet.load(conf.dataset_extra, img_wh, split="test")`), and on request their depth
errors and each object's mask agreement.

For each frame, `evaluate_frames`
  - builds the frame's (H*W, 8) rays on the device with the arithmetic of onerf_draw_frames' training rows
    (onerf_camera_rays: the rays GenericDataset holds for that pose) and the ground truth u8 / 255 in float32;
  - renders the frame once through training.validate_frame (is_eval, nothing random) with keys ("rgb", "rgb_instance")
    of the last pass.  The codes come from per-pixel instance ids: the pixel's label when it is one of object_ids, else
    object_ids[0] (0 without objects).  One render serves every object column: after zeroing outside its mask, object
    column k reads only pixels labelled object_ids[k-1], and each of those was rendered with that object's code;
  - scores the maps with onerf_image_metrics (metrics.py's definition; column 0 the scene over the valid pixels, column k
    the object prediction over the valid pixels labelled object_ids[k-1]) and finalises row f of the outputs.
With depth=True the one render also gives the last pass's depth and depth_instance, scored with onerf_depth_metrics
(metrics.py's definition) against the store's processed depths at scale frames.scale_factor: column 0 the scene over
the valid pixels with a depth, column k the object depth over those labelled object_ids[k-1].  The same argument as for
the colours makes the one render exact for every object column.  With masks=True one more render per frame,
rendering.render_instances over object_ids, gives every object's opacity_instance with its own code at every pixel
(what validate_frame gives for frame_batch(frames, f, [k]), bit for bit); column k is scored against the pixels
labelled object_ids[k] by onerf_mask_metrics.  Neither flag changes the colour render or its scores.
With boxes (one per object id, e.g. frames.read_boxes of the dataset's own files), the object columns follow a
use_bbox dataset's evaluation instead (GenericDataset's test split: rays clipped to the object's box, instance_mask *
bbox_mask, rays_in_bbox): one rendering.render_boxes call per frame gives every object's maps over its box-clipped
rays, and object k is scored over the valid pixels labelled object_ids[k] whose ray hits box k, for colour, depth and
(masks=True: G = label object_ids[k] and hit_k, from the same call's opacity) masks.  The scene columns are unchanged.
Valid pixels are those frames.BORDER or more pixels from every edge, the training split's valid_mask.  The loop reads
nothing back to the host; the per-frame outputs stay on the device.

group: a torch.distributed process group, passed to validate_frame, which renders one tile of each frame per rank and
gathers the maps; every rank then scores the whole frame, so every rank returns the same numbers.
"""
from __future__ import annotations

from typing import Any, Dict, Sequence

import torch

from . import _lib, metrics, rendering, training
from .losses import TERMS
from .ray_utils import _c2w_host

__all__ = ["evaluate_frames", "frame_batch", "valid_mask"]

_NO_LOSS = {f"{t}_weight": 0.0 for t in TERMS}          # validate_frame's loss terms are not used here


def _model_conf(conf):
    m = conf["model"] if "model" in conf else conf
    return int(m["N_samples"]), int(m["N_importance"]), bool(m["use_disp"])


def valid_mask(frames) -> torch.Tensor:
    """(H*W,) uint8: 1 for the pixels frames.border or more pixels from every edge (the training rows' valid_mask)."""
    H, W, b, dev = frames.H, frames.W, frames.border, frames.device
    y, x = torch.arange(H, device=dev).view(H, 1), torch.arange(W, device=dev).view(1, W)
    return ((y >= b) & (y < H - b) & (x >= b) & (x < W - b)).reshape(H * W).to(torch.uint8)


def frame_batch(frames, f: int, object_ids: Sequence[int] = (), rays=None) -> Dict[str, torch.Tensor]:
    """What evaluate_frames renders frame f of `frames` from, as a validate_frame batch: rays (H*W, 8) (written into
    `rays` when given), rgbs = the frame's u8 / 255, depths, valid_mask, and instance_ids = the pixel's label where it
    is one of object_ids, else object_ids[0] (0 without objects)."""
    H, W, dev, t = frames.H, frames.W, frames.device, frames.tensors
    if rays is None:
        rays = torch.empty(H * W, 8, dtype=torch.float32, device=dev)
    c2w = _c2w_host(frames.poses_host[f].reshape(3, 4))
    _lib.call("onerf_camera_rays", dev, H, W, frames.focal, c2w, None, frames.scale_factor, frames.near, frames.far,
              rays.data_ptr(), None)
    if object_ids:
        ids = torch.tensor([int(i) for i in object_ids], dtype=torch.int32, device=dev)
        lab = t["labels"][f].to(torch.int32) & 0xFFFF
        inst = torch.where(torch.isin(lab, ids), lab, ids[0]).to(torch.int64)
    else:
        inst = torch.zeros(H * W, dtype=torch.int64, device=dev)
    return {"rays": rays, "rgbs": t["rgb"][f].float() / 255, "depths": t["depths"][f], "valid_mask": valid_mask(frames),
            "instance_ids": inst}


def _box_columns(labels, ids, hit, outside: int):
    """Box mode's per-pixel inputs of the metrics kernels: the labels with every pixel whose object missed its box
    relabelled `outside` (so object k reads the pixels labelled ids[k] with hit_k, GenericDataset's
    instance_mask * bbox_mask), and each pixel's column: the position of its label in ids, else 0."""
    lab = labels.to(torch.int32) & 0xFFFF
    match = lab.view(-1, 1) == ids.view(1, -1)
    pick = match.to(torch.uint8).argmax(1)
    keep = (match & hit).any(1)
    return metrics._labels16(torch.where(keep, lab, outside)), pick


def evaluate_frames(models: Dict[str, Any], embeddings: Dict[str, Any], code_library, frames, conf, *,
                    object_ids: Sequence[int] = (), window: int = 3, chunk: int = 65536, precision: str = "bf16",
                    group=None, depth: bool = False, masks: bool = False, mask_threshold: float = 0.5,
                    depth_range=(1e-3, 10.0), boxes=None) -> Dict[str, torch.Tensor]:
    """PSNR and SSIM of every frame of `frames` (a frames.FrameSet) rendered by the trained model (module docstring).
    conf: the reference's config (conf.model's N_samples, N_importance and use_disp), or that model section itself.
    object_ids: up to 64 object ids to score, each a label of the store's label images and a row of the code table.
    window: the SSIM window (odd, 1 to 11; the reference's utils/metrics.ssim uses 3).  chunk, precision, group: as
    training.validate_frame.

    Returns device tensors: "psnr", "ssim" (F,) of the scene; "psnr_objects", "ssim_objects" (F, K); "mean_psnr",
    "mean_ssim" () and "mean_psnr_objects", "mean_ssim_objects" (K,), the means over frames ignoring NaN (a frame in
    which an object has no valid pixel scores NaN for it).

    depth=True adds "depth_metrics" (F, 7) of the scene and "depth_metrics_objects" (F, K, 7), columns in
    metrics.DEPTH_METRICS order, and their NaN-ignoring means over frames "mean_depth_metrics" (7,) and
    "mean_depth_metrics_objects" (K, 7).  depth_range: the (d_min, d_max) clamp of the predictions in metres.
    masks=True adds "iou_objects" and "opacity_l1_objects" (F, K) and "mean_iou_objects", "mean_opacity_l1_objects"
    (K,); it costs one more render per frame, whose object branch runs once per object.  mask_threshold: the opacity
    at which a pixel counts as covered.
    boxes: None, or one box per object id (objects with BBoxRayHelper's pose_avg, axis_align_mat and bbox_bounds): the
    object columns then come from one render_boxes call per frame (module docstring), masks=True included."""
    ids = [int(i) for i in object_ids]
    K = len(ids)
    if K > _lib.METRICS_MAX_IDS:
        raise ValueError(f"evaluate_frames: at most {_lib.METRICS_MAX_IDS} object ids, got {K}")
    if len(set(ids)) != K:
        raise ValueError(f"evaluate_frames: object_ids repeat an id: {ids}")
    n_codes = code_library.embedding_instance.weight.shape[0]
    if any(not 0 <= i < min(n_codes, 1 << 16) for i in ids):
        raise ValueError(f"evaluate_frames: object ids must be code-table rows in [0, {n_codes}) and 16-bit labels")
    t = frames.tensors
    if K and "labels" not in t:
        raise ValueError("evaluate_frames: object columns need the store's label images (load it with an instance "
                         "column that reads a mask)")
    if boxes is not None and len(boxes) != K:
        raise ValueError(f"evaluate_frames: one box per object id, got {len(boxes)} boxes for {K} ids")
    in_boxes = boxes is not None and K > 0
    N_samples, N_importance, use_disp = _model_conf(conf)
    F, H, W, dev = frames.n_frames, frames.H, frames.W, frames.device
    HW, typ = H * W, "fine" if N_importance > 0 else "coarse"
    keys = ("rgb", "rgb_instance") if K and not in_boxes else ("rgb",)
    if depth:
        keys += ("depth", "depth_instance") if K and not in_boxes else ("depth",)
    box_keys = ("rgb_instance",) + (("depth_instance",) if depth else ()) + (("opacity_instance",) if masks else ())
    render = dict(N_samples=N_samples, N_importance=N_importance, use_disp=use_disp, white_back=False, chunk=chunk,
                  precision=precision, group=group)

    plan = metrics.MetricsPlan(H, W, ids, window, F, dev)
    dplan = metrics.DepthMetricsPlan(H, W, ids, frames.scale_factor, depth_range, F, dev) if depth else None
    mplan = metrics.MaskMetricsPlan(H, W, ids, mask_threshold, F, dev) if masks else None
    rays = torch.empty(HW, 8, dtype=torch.float32, device=dev)
    if in_boxes:
        ids_dev = torch.tensor(ids, dtype=torch.int32, device=dev)
        outside = min(set(range(K + 1)) - set(ids))        # a label no object column reads
    for f in range(F):
        batch = frame_batch(frames, f, ids, rays)
        out = training.validate_frame(models, embeddings, code_library, batch, _NO_LOSS, keys=keys, **render)
        labels = t["labels"][f] if K else None
        if in_boxes:
            out.update(rendering.render_boxes(models, embeddings, code_library, H, W, frames.focal,
                                              torch.from_numpy(frames.poses_host[f].reshape(3, 4)), boxes, ids,
                                              N_samples=N_samples, N_importance=N_importance, use_disp=use_disp,
                                              scale_factor=frames.scale_factor, near=frames.near, far=frames.far,
                                              chunk=chunk, keys=box_keys, precision=precision, group=group))
            labels, pick = _box_columns(labels, ids_dev, out["hit"], outside)
            for key in box_keys[:1 + depth]:         # colour and depth: each pixel's own object's column
                v = out[f"{key}_{typ}"]
                out[f"{key}_{typ}"] = v.gather(1, pick.view(HW, 1, *([1] * (v.dim() - 2))).expand(HW, 1, *v.shape[2:]))
        plan.accumulate(out[f"rgb_{typ}"], batch["rgbs"], batch["valid_mask"], out.get(f"rgb_instance_{typ}"), labels)
        plan.finalize(f)
        if depth:
            dplan.accumulate(out[f"depth_{typ}"], t["depths"][f], batch["valid_mask"], out.get(f"depth_instance_{typ}"),
                             labels)
            dplan.finalize(f)
        if masks and in_boxes:
            o = out[f"opacity_instance_{typ}"]
            for k in range(K):
                mplan.accumulate(k, o[:, k], labels, batch["valid_mask"])
            mplan.finalize(f)
        elif masks and K:
            out = rendering.render_instances(models, embeddings, code_library, rays, ids, keys=("opacity_instance",),
                                             **render)
            for k in range(K):
                mplan.accumulate(k, out[f"opacity_instance_{typ}"][:, k], labels, batch["valid_mask"])
            mplan.finalize(f)
    P, S = plan.psnr, plan.ssim
    res = {"psnr": P[:, 0], "ssim": S[:, 0], "psnr_objects": P[:, 1:], "ssim_objects": S[:, 1:],
           "mean_psnr": P[:, 0].nanmean(), "mean_ssim": S[:, 0].nanmean(),
           "mean_psnr_objects": P[:, 1:].nanmean(0), "mean_ssim_objects": S[:, 1:].nanmean(0)}
    if depth:
        D = dplan.out
        res.update({"depth_metrics": D[:, 0], "depth_metrics_objects": D[:, 1:],
                    "mean_depth_metrics": D[:, 0].nanmean(0), "mean_depth_metrics_objects": D[:, 1:].nanmean(0)})
    if masks:
        res.update({"iou_objects": mplan.iou, "opacity_l1_objects": mplan.opacity_l1,
                    "mean_iou_objects": mplan.iou.nanmean(0), "mean_opacity_l1_objects": mplan.opacity_l1.nanmean(0)})
    return res
