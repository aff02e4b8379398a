"""Training frames kept as pixels on the device (GenericDataset's train split, datasets/generic_dataset.py:120-308,
without expanding every frame into one row per pixel).

GenericDataset holds 57 + 14*I bytes per training ray (rays, colours, depth, border mask, frame index and four fields per
instance column), nearly all of it derived from a handful of per-frame values.  `FrameSet` holds what those rows are
derived from: per pixel an 8-bit RGB triple, the processed float32 depth and a 16-bit label (9 bytes), and per frame
its pose, frame index and instance-column weights.  `RaySampler.from_frames` draws training batches from it, each row
rebuilt on the device (include/onerf_ext.h: onerf_draw_frames), bit-identical to the row RaySampler draws from the
expanded buffers with the same seed.

Decoding stays on the host, as in the reference: PNG reads, PIL LANCZOS for colour, cv2 INTER_NEAREST for depth and
labels, and the depth arithmetic with the reference's own torch ops.

`read_frames(..., split="test")` / `FrameSet.load(..., split="test")` keep the held-out frames instead: those whose idx
split/test.txt lists, in transforms_full.json order, without the frames whose pose is not finite, decoded exactly as the
training frames (evaluation.evaluate_frames renders and scores them).  `FrameSet.load` takes a test split with use_bbox
too: its frames decode exactly as without it, since the clipping to each object's box belongs to the render
(rendering.render_boxes over the boxes `read_boxes` reads, evaluate_frames(boxes=...)).

Refused rather than approximated (ValueError, before any device work):
  - training rays clipped to a box (use_bbox without use_bbox_only_for_test), and read_frames of a test split with
    use_bbox (its rays would be clipped to the object box; FrameSet.load leaves that clipping to the render);
  - mask_rebalance_strategy other than fg_bg_reweight (distance_transform crashes in the reference itself);
  - a frame whose RGB image is missing (the reference then misaligns its per-instance buffers against all_rays);
  - label images wider than 16 bits, and more than FRAME_MAX_PASS pass-through labels per instance column.
"""
from __future__ import annotations

import json
import os
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import _lib, ray_utils

__all__ = ["FrameSet", "read_frames", "read_boxes", "ObjectBox", "BORDER"]

BORDER = 20                     # black border of undistorted images, masked out of training (generic_dataset.py:44-52)
MAX_PASS = _lib.FRAME_MAX_PASS


def _host_directions(H: int, W: int, focal: float) -> torch.Tensor:
    """(H*W, 3) camera-space directions on the host, datasets/ray_utils.py:5-25 (only their norm is used: it scales
    the depths, generic_dataset.py:146, 395)."""
    j, i = torch.meshgrid(torch.linspace(0, H - 1, H), torch.linspace(0, W - 1, W), indexing="ij")
    d = torch.stack([(i - W / 2) / focal, -(j - H / 2) / focal, -torch.ones_like(i)], -1)
    return d.reshape(-1, 3)


def _obs_check(frame, conf, center) -> bool:
    """generic_dataset.py:175-185 with geo_utils.observe_angle_distance."""
    T = np.array(frame["transform_matrix"])
    if np.isnan(T.sum()) or np.isinf(T.sum()):
        return False
    if not conf["enable_observation_check"]:
        return True
    view_dir = T[:3, :3] @ np.array([0, 0, 1])
    c2o = center - T[:3, 3]
    dist = np.linalg.norm(c2o)
    c2o /= dist
    angle = np.arccos(c2o.dot(view_dir)) * 180 / np.pi
    return angle < conf["max_obs_angle"] and dist < conf["max_obs_distance"]


def _c2w(frame, pose_avg, scale_factor) -> np.ndarray:
    """generic_dataset.py:358-367: fix_rot, centring on pose_avg, scale; -> (3, 4) float32."""
    fix_rot = np.array([1, 0, 0, 0, -1, 0, 0, 0, -1]).reshape(3, 3)
    pose = np.array(frame["transform_matrix"])
    pose[:3, :3] = pose[:3, :3] @ fix_rot
    avg = np.eye(4)
    avg[:3] = pose_avg
    homo = np.eye(4)
    homo[:3] = pose[:3]
    pose = np.linalg.inv(avg) @ homo
    pose[:, 3] /= scale_factor
    return torch.FloatTensor(pose)[:3, :4].numpy()


def _columns(conf):
    """The instance columns GenericDataset stacks: instance_id in order, except that an id 0 after the first column is
    dropped (generic_dataset.py:247-249 skips it once the frame is registered)."""
    ids = list(conf["instance_id"])
    if not ids:
        raise ValueError("FrameSet: instance_id lists no instance column")
    return [ids[0]] + [i for i in ids[1:] if i != 0]


def read_frames(conf, img_wh, split: str = "train") -> Dict[str, object]:
    """Decode GenericDataset's train split on the host: the FrameSet constructor's keyword arguments (arrays on the
    host, frames in GenericDataset's order).  split="test": the frames split/test.txt lists instead, in
    transforms_full.json order, dropping only those whose pose is not finite (no train_start_idx, validate_idx,
    observation check, train_skip_step or train_max_size), decoded the same way."""
    import cv2
    from PIL import Image

    w, h = img_wh
    if split not in ("train", "test"):
        raise ValueError(f"FrameSet: unknown split {split!r} (train or test)")
    if split == "test" and conf["use_bbox"]:
        raise ValueError("FrameSet: test rays clipped to the object box (use_bbox) are not supported")
    if conf["use_bbox"] and not conf["use_bbox_only_for_test"]:
        raise ValueError("FrameSet: training rays clipped to the object box (use_bbox with use_bbox_only_for_test "
                         "false) are not supported")
    ids = _columns(conf)
    use_mask = bool(conf["use_instance_mask"]) and any(i != 0 for i in ids)
    fg_weight = bg_weight = None
    if use_mask:
        strategy = conf["mask_rebalance_strategy"]
        if strategy == "distance_transform":
            raise ValueError("FrameSet: mask_rebalance_strategy distance_transform is not supported (the reference "
                             "passes it fg_weight / bg_weight, which compute_distance_transfrom_weights does not take)")
        if strategy != "fg_bg_reweight":
            raise ValueError(f"FrameSet: unknown mask_rebalance_strategy {strategy!r}")
        fg_weight, bg_weight = conf.get("fg_weight"), conf.get("bg_weight")

    root = conf["root_dir"]
    with open(os.path.join(root, "transforms_full.json")) as f:
        meta = json.load(f)
    focal = 0.5 * w / np.tan(0.5 * meta["camera_angle_x"])
    focal *= img_wh[0] / w
    scale = conf["scale_factor"]
    pose_avg = np.concatenate([np.eye(3), np.array(conf["scene_center"])[:, None]], 1)

    split_inds = np.loadtxt(os.path.join(conf["split"], f"{split}.txt"))
    split_inds = (split_inds.reshape(-1) if split == "test" else split_inds).tolist()    # a one-line test.txt
    frames = [x for x in meta["frames"] if x["idx"] in split_inds]
    if split == "test":
        frames = [x for x in frames if np.isfinite(np.array(x["transform_matrix"], dtype=np.float64)).all()]
        if not frames:
            raise ValueError("FrameSet: split/test.txt lists no frame with a finite pose")
    else:
        frames = [x for x in frames if x["idx"] >= conf["train_start_idx"] and x["idx"] != conf["validate_idx"]]
        frames = [x for x in frames if _obs_check(x, conf, pose_avg[:3, 3])]
        frames = [frames[i] for i in np.arange(0, len(frames), conf["train_skip_step"])]
        frames = frames[:min(conf["train_max_size"], len(frames))]
        if not frames:
            raise ValueError("FrameSet: no training frame passes the split and observation filters")
    for fr in frames:
        p = os.path.join(root, f"{fr['file_path']}.png")
        if not os.path.exists(p):
            raise ValueError(f"FrameSet: missing RGB image {p} (GenericDataset would misalign its instance buffers)")

    norm = torch.norm(_host_directions(h, w, focal), dim=-1)
    poses, rgb, depths, labels = [], [], [], []
    for fr in frames:
        base = os.path.join(root, fr["file_path"])
        poses.append(_c2w(fr, pose_avg, scale))
        img = Image.open(base + ".png")
        img = np.asarray(img.resize(img_wh, Image.LANCZOS))
        if img.shape != (h, w, 3) or img.dtype != np.uint8:
            raise ValueError(f"FrameSet: {base}.png is not an 8-bit RGB image")
        rgb.append(img)
        depth = cv2.imread(base + ".depth.png", cv2.IMREAD_ANYDEPTH)
        if depth is None:
            depth = np.zeros((h, w))
        else:
            depth = cv2.resize(depth, img_wh, interpolation=cv2.INTER_NEAREST) * 1e-3
            depth[depth > 4] = 0
        d = torch.from_numpy(np.ascontiguousarray(depth)).float().view(-1)
        d /= scale
        d *= norm
        depths.append(d.numpy())
        if use_mask:
            path = f"{base}.{conf['inst_seg_tag']}.png"
            lab = cv2.imread(path, cv2.IMREAD_ANYDEPTH)
            if lab is None:
                raise ValueError(f"FrameSet: cannot read label image {path}")
            if lab.dtype not in (np.uint8, np.uint16):
                raise ValueError(f"FrameSet: label image {path} is {lab.dtype}; labels wider than 16 bits are not "
                                 "supported")
            labels.append(cv2.resize(lab, img_wh, interpolation=cv2.INTER_NEAREST).astype(np.uint16))
    return dict(poses=np.stack(poses), rgb=np.stack(rgb), depths=np.stack(depths).reshape(len(frames), h, w),
                labels=np.stack(labels) if use_mask else None, focal=float(focal), near=conf["near"],
                far=conf["far"], scale_factor=scale, instance_ids=ids,
                bg_instance_ids=list(conf.get("bg_instance_id", [])), use_instance_mask=use_mask,
                fg_weight=fg_weight, bg_weight=bg_weight, frame_idx=np.arange(len(frames)), border=BORDER)


def instance_tables(labels: Optional[np.ndarray], instance_ids: Sequence[int], bg_instance_ids: Sequence[int] = (),
                    use_instance_mask: bool = True, fg_weight=None, bg_weight=None):
    """Per-column tables of the frame store: ids (I,) int64, mask_all_ones (I,) uint8, weights (F,I,2) float32
    ([background, foreground] weight per frame, rebalance_mask of datasets/image_utils.py:8-25: fixed weights, or with
    both None the count ratio of the frame's label image) and pass_ids (I,K) int32 (bg_instance_ids + [id], -1 padded).
    labels: (F, H*W) uint16, or None when no column reads a mask."""
    I = len(instance_ids)
    ids = np.array([int(i) for i in instance_ids], dtype=np.int64)
    all_ones = np.array([not use_instance_mask or i == 0 for i in ids], dtype=np.uint8)
    if (fg_weight is None) != (bg_weight is None):
        raise ValueError("FrameSet: fg_weight and bg_weight are both given or both None")
    passes = [list(bg_instance_ids) + [int(i)] for i in ids]
    K = max(len(p) for p in passes)
    if K > MAX_PASS:
        raise ValueError(f"FrameSet: {K} pass-through labels per instance column; at most {MAX_PASS} are supported")
    pass_ids = np.full((I, K), -1, dtype=np.int32)
    for c, p in enumerate(passes):
        pass_ids[c, :len(p)] = [v if 0 <= v <= 0xFFFF else -1 for v in p]   # a value no 16-bit label takes
    if not all_ones.all() and labels is None:
        raise ValueError("FrameSet: instance columns with masks need label images")
    F = labels.shape[0] if labels is not None else None
    weights = np.zeros((F or 1, I, 2), dtype=np.float32)
    for c in range(I):
        if all_ones[c]:
            continue
        if fg_weight is not None:
            weights[:, c] = [np.float32(bg_weight), np.float32(fg_weight)]
            continue
        fg = np.maximum((labels == ids[c]).sum(1), 1)
        bg = np.maximum(labels.shape[1] - (labels == ids[c]).sum(1), 1)
        weights[:, c, 0] = [np.float32(float(f) / b) for f, b in zip(fg, bg)]
        weights[:, c, 1] = [np.float32(float(b) / f) for f, b in zip(fg, bg)]
    return ids, all_ones, weights, pass_ids


def _host(a, dtype=None) -> np.ndarray:
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return a.astype(dtype, copy=False) if dtype is not None else a


class FrameSet:
    """A training frame store on the device.

    poses         (F,3,4) or (F,12) float32 c2w, centred and scaled as GenericDataset's (generic_dataset.py:358-367)
    rgb           (F,H,W,3) uint8
    depths        (F,H,W) float32, processed (* 1e-3, > 4 -> 0, / scale_factor, * the direction norm)
    labels        (F,H,W) uint8 or uint16 instance labels, or None when no column reads a mask
    focal, near, far, scale_factor   the camera and GenericDataset's conf values
    instance_ids, bg_instance_ids, use_instance_mask, fg_weight, bg_weight   the instance columns (instance_tables)
    frame_idx     (F,) int64, default 0..F-1
    border        pixels nearer than this to an edge have valid_mask 0

    n_rays = F*H*W rays; ray f*H*W + y*W + x is pixel (x, y) of frame f, row for row the ray GenericDataset's
    all_* buffers hold."""

    def __init__(self, poses, rgb, depths, labels, *, focal: float, near: float, far: float, scale_factor: float,
                 instance_ids: Sequence[int] = (0,), bg_instance_ids: Sequence[int] = (), use_instance_mask=True,
                 fg_weight=None, bg_weight=None, frame_idx=None, border: int = BORDER, device="cuda"):
        rgb = _host(rgb)
        if rgb.ndim != 4 or rgb.shape[-1] != 3 or rgb.dtype != np.uint8:
            raise ValueError(f"FrameSet: rgb must be (F,H,W,3) uint8, got {rgb.shape} {rgb.dtype}")
        F, H, W = rgb.shape[:3]
        poses = _host(poses, np.float32).reshape(F, -1)
        depths = _host(depths)
        if poses.shape != (F, 12):
            raise ValueError(f"FrameSet: poses must be (F,3,4), got {F} frames of {poses.shape[1]} values")
        if depths.dtype != np.float32 or depths.reshape(F, -1).shape != (F, H * W):
            raise ValueError(f"FrameSet: depths must be (F,H,W) float32, got {depths.shape} {depths.dtype}")
        if labels is not None:
            labels = _host(labels)
            if labels.dtype not in (np.uint8, np.uint16):
                raise ValueError(f"FrameSet: labels are {labels.dtype}; labels wider than 16 bits are not supported")
            if labels.reshape(F, -1).shape != (F, H * W):
                raise ValueError(f"FrameSet: labels must be (F,H,W), got {labels.shape}")
            labels = labels.reshape(F, H * W).astype(np.uint16)
        if frame_idx is None:
            frame_idx = np.arange(F)
        frame_idx = _host(frame_idx, np.int64).reshape(-1)
        if frame_idx.shape != (F,):
            raise ValueError(f"FrameSet: frame_idx must have {F} entries")
        if int(border) < 0 or not focal > 0 or not scale_factor > 0:
            raise ValueError("FrameSet: border must be >= 0, focal and scale_factor positive")
        ids, all_ones, weights, pass_ids = instance_tables(labels, instance_ids, bg_instance_ids, use_instance_mask,
                                                           fg_weight, bg_weight)
        if all_ones.all():
            labels = None                      # no column reads a label
        if weights.shape[0] != F:
            weights = np.broadcast_to(weights, (F,) + weights.shape[1:])
        I = len(ids)
        if F * H * W >= 1 << 40:
            raise ValueError("FrameSet: at most 2^40 - 1 rays are supported")

        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.device, self.n_frames, self.H, self.W, self.n_instances = dev, F, H, W, I
        self.n_rays = F * H * W
        self.focal, self.near, self.far, self.scale_factor = float(focal), float(near), float(far), float(scale_factor)
        self.border = int(border)
        self.poses_host = poses.copy()
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        t = {"poses": up(poses), "rgb": up(rgb.reshape(F, H * W, 3)), "depths": up(depths.reshape(F, H * W)),
             "frame_idx": up(frame_idx), "ids": up(ids), "mask_all_ones": up(all_ones), "weights": up(weights),
             "pass_ids": up(pass_ids),
             "directions": ray_utils.get_ray_directions(H, W, self.focal, device=dev).reshape(H * W, 3)}
        if labels is not None:
            t["labels"] = up(labels.view(np.int16))    # the 16-bit pattern (the kernel reads it as uint16)
        self.tensors = t
        a = _lib.FrameDataset()
        a.n_frames, a.H, a.W, a.n_instances = F, H, W, I
        a.near_s, a.far_s = float(np.float32(near / scale_factor)), float(np.float32(far / scale_factor))
        a.border, a.n_pass = self.border, pass_ids.shape[1]
        for k in ("poses", "directions", "rgb", "depths", "labels", "frame_idx", "ids", "mask_all_ones", "weights",
                  "pass_ids"):
            setattr(a, k, t[k].data_ptr() if k in t else None)
        self.args = a

    @classmethod
    def load(cls, dataset_extra, img_wh=(640, 480), device="cuda", split: str = "train") -> "FrameSet":
        """GenericDataset(split="train", img_wh, dataset_extra)'s training frames, kept as pixels (read_frames);
        split="test": the held-out frames of split/test.txt.  A test split with use_bbox decodes exactly as without it:
        GenericDataset clips its rays to the object's box, which render_boxes does at render time."""
        if split == "test" and dataset_extra["use_bbox"]:
            dataset_extra = dict(dataset_extra, use_bbox=False)
        return cls(**read_frames(dataset_extra, tuple(img_wh), split), device=device)

    @property
    def nbytes(self) -> int:
        """Device bytes the store holds."""
        return sum(t.numel() * t.element_size() for t in self.tensors.values())

    def expand(self) -> Dict[str, torch.Tensor]:
        """The all_* buffers GenericDataset would hold for these frames, built on the device (camera_rays per frame):
        what RaySampler(...) takes, for tests and comparisons."""
        F, H, W, I, dev = self.n_frames, self.H, self.W, self.n_instances, self.device
        HW, t = H * W, self.tensors
        rays = torch.cat([ray_utils.camera_rays(H, W, self.focal, torch.from_numpy(self.poses_host[f].reshape(3, 4)),
                                                self.near, self.far, self.scale_factor, device=dev)
                          for f in range(F)])
        lut = torch.arange(256, dtype=torch.uint8).float().div(255).to(dev)     # torchvision ToTensor
        y = torch.arange(H, device=dev).view(H, 1)
        x = torch.arange(W, device=dev).view(1, W)
        b = self.border
        valid = ((y >= b) & (y < H - b) & (x >= b) & (x < W - b)).reshape(HW).repeat(F)
        f_of = torch.arange(F, device=dev).repeat_interleave(HW)
        labels = (t["labels"].to(torch.int32) & 0xFFFF).reshape(-1) if "labels" in t else None
        masks, weights, ids, passes = [], [], [], []
        for c in range(I):
            id_c = t["ids"][c]
            if labels is None or bool(t["mask_all_ones"][c]):
                m = torch.ones(F * HW, dtype=torch.bool, device=dev)
                p = m.clone()
            else:
                m = labels == id_c
                p = torch.isin(labels, t["pass_ids"][c].to(torch.int32))
            masks.append(m)
            passes.append(p)
            weights.append(t["weights"][f_of, c, m.long()])
            ids.append(id_c.expand(F * HW))
        return {"all_rays": rays, "all_rgbs": lut[t["rgb"].reshape(-1, 3).long()],
                "all_depths": t["depths"].reshape(-1).clone(), "all_valid_masks": valid,
                "all_frame_indices": t["frame_idx"][f_of], "all_instance_masks": torch.stack(masks, -1),
                "all_instance_masks_weight": torch.stack(weights, -1), "all_instance_ids": torch.stack(ids, -1),
                "all_pass_through_masks": torch.stack(passes, -1)}


# ------------------------------------------------------------------------------------------------
# object boxes
# ------------------------------------------------------------------------------------------------
class ObjectBox:
    """One object's box with the attributes of the reference's BBoxRayHelper (utils/bbox_utils.py:9-99) that describe
    it: dataset_name, conf (the dataset_extra section), scale_factor, instance_id, scene_id (scannet_base only),
    axis_align_mat (4, 4), bbox_bounds (2, 3) = [lo, hi], bbox_c (3,) and pose_avg (4, 4), all float64.  What
    ray_utils.camera_rays(box=...) and rendering.render_boxes take."""

    def __init__(self, **attrs):
        self.__dict__.update(attrs)


def _scannet_box(conf, instance_id):
    """BBoxRayHelper.read_bbox_info_scannet (utils/bbox_utils.py:64-84): the first axisAlignment line of
    scans_dir/<scene_id>/<scene_id>.txt, parsed with the reference's str.strip("axisAlignment = ") (a character set),
    and the last row of bbox_dir/<scene_id>_bbox.npy whose column 6 is the id."""
    if "scene_id" not in conf:
        raise ValueError("read_boxes: a scannet_base dataset_extra needs scene_id (BBoxRayHelper reads conf['scene_id'])")
    scene_id = conf["scene_id"]
    with open(os.path.join(conf["scans_dir"], f"{scene_id}/{scene_id}.txt")) as f:
        lines = f.readlines()
    align = None
    for line in lines:
        if "axisAlignment" in line:
            align = [float(x) for x in line.rstrip().strip("axisAlignment = ").split(" ")]
            break
    if align is None:
        raise ValueError(f"read_boxes: no axisAlignment line in {scene_id}.txt")
    center = bounds = None
    for b in np.load(os.path.join(conf["bbox_dir"], f"{scene_id}_bbox.npy")):
        if b[6] != instance_id:
            continue
        length = np.array([b[3], b[4], b[5]]) * 0.5
        center = np.array([b[0], b[1], b[2]])
        bounds = np.array([center - length, center + length])
    if bounds is None:
        raise ValueError(f"read_boxes: {scene_id}_bbox.npy has no box for instance id {instance_id}")
    return dict(scene_id=scene_id, axis_align_mat=np.array(align).reshape(4, 4), bbox_bounds=bounds, bbox_c=center)


def _toydesk_box(conf, instance_id):
    """BBoxRayHelper.read_bbox_info_desk (utils/bbox_utils.py:86-96): the first label of the bbox_dir JSON with this id
    and a position; axis_align_mat = inv([R(quaternion) | position]), bbox_bounds = [-scale / 2, scale / 2]."""
    from scipy.spatial.transform import Rotation

    with open(conf["bbox_dir"]) as f:
        labels = json.load(f)["labels"]
    for lab in labels:
        if int(lab["id"]) != instance_id or "position" not in lab["data"]:
            continue
        pos, scale = np.array(lab["data"]["position"]), np.array(lab["data"]["scale"])
        align = np.eye(4)
        align[:3, :3] = Rotation.from_quat(lab["data"]["quaternion"]).as_matrix()
        align[:3, 3] = pos
        return dict(axis_align_mat=np.linalg.inv(align), bbox_bounds=np.array([-scale / 2, scale / 2]), bbox_c=pos)
    raise ValueError(f"read_boxes: the bbox JSON has no box with a position for instance id {instance_id}")


def read_boxes(dataset_name: str, conf, ids: Sequence[int]):
    """The boxes of objects `ids` as the reference's BBoxRayHelper(config, id) reads them from the dataset's own files
    (utils/bbox_utils.py:41-99), for dataset_name "scannet_base" or "toydesk"; conf is the dataset_extra section.
    pose_avg = [I | scene_center].  An id without a box raises ValueError (the reference would reuse a stale centre
    or fail with a NameError).  Returns one ObjectBox per id, in order."""
    if dataset_name not in ("scannet_base", "toydesk"):
        raise ValueError(f"read_boxes: unknown dataset {dataset_name!r} (scannet_base or toydesk)")
    out = []
    for i in ids:
        i = int(i)
        attrs = _scannet_box(conf, i) if dataset_name == "scannet_base" else _toydesk_box(conf, i)
        pose_avg = np.eye(4)
        pose_avg[:3, 3] = np.array(conf["scene_center"])
        out.append(ObjectBox(dataset_name=dataset_name, conf=conf, scale_factor=conf["scale_factor"], instance_id=i,
                             pose_avg=pose_avg, **attrs))
    return out
