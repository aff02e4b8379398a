"""A tiny on-disk dataset in GenericDataset's layout, the configs the frame-store tests load it with, and a host
restatement of FrameSet.expand() (torch on the CPU, written from the reference's definitions: datasets/ray_utils.py,
datasets/generic_dataset.py:212-308, datasets/image_utils.py:8-25)."""
import json
import os

import cv2
import numpy as np
import torch
from PIL import Image

IMG_WH = (48, 44)           # frames are written at SRC_WH, so LANCZOS and INTER_NEAREST both resample
SRC_WH = (61, 37)
N_FRAMES = 9


def _pose(rng, center):
    """A camera 1-3 m from `center`, looking near it ('right down forward' axes, as the reference's poses)."""
    eye = center + rng.normal(size=3) * [1.2, 1.2, 0.4] + [0, 0, 1.2]
    fwd = center + rng.normal(size=3) * 0.3 - eye
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, [0, 0, 1.0])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    T = np.eye(4)
    T[:3, :3] = np.stack([right, down, fwd], 1)
    T[:3, 3] = eye
    return T


def write_scene(root, seed=0):
    """N_FRAMES frames (idx 0..8): RGB at SRC_WH, 16-bit depth in mm (some above 4 m), labels as uint8 PNGs on even
    frames and uint16 on odd ones (values 0..5, plus 300 on the uint16 ones).  Frame 4's pose is NaN; the split file
    drops frame 6."""
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    center = np.array([0.3, -0.2, 0.5])
    frames = []
    w, h = SRC_WH
    for i in range(N_FRAMES):
        T = _pose(rng, center)
        if i == 4:
            T[0, 3] = np.nan
        base = os.path.join("images", f"{i:04d}")
        frames.append({"idx": i, "file_path": base, "transform_matrix": T.tolist()})
        rgb = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        Image.fromarray(rgb, "RGB").save(os.path.join(root, base + ".png"))
        depth = rng.integers(0, 6000, size=(h, w)).astype(np.uint16)
        cv2.imwrite(os.path.join(root, base + ".depth.png"), depth)
        lab = rng.integers(0, 6, size=(h, w))
        lab[: h // 3, : w // 2] = 2                      # a large block: the count-based weights are far from 1
        if i % 2:
            lab[-4:, -5:] = 300
            lab = lab.astype(np.uint16)
        else:
            lab = lab.astype(np.uint8)
        cv2.imwrite(os.path.join(root, base + ".instance.png"), lab)
    # JSON cannot hold NaN strictly; json.dump writes it as NaN, which json.load reads back
    with open(os.path.join(root, "transforms_full.json"), "w") as f:
        json.dump({"camera_angle_x": 0.9, "frames": frames}, f)
    os.makedirs(os.path.join(root, "split"), exist_ok=True)
    np.savetxt(os.path.join(root, "split", "train.txt"), [i for i in range(N_FRAMES) if i != 6], fmt="%d")
    return center


def config(root, center, *, instance_id=(2,), bg_instance_id=(), obs_check=False, fg_weight=None, bg_weight=None,
           use_instance_mask=True, **over):
    c = {"root_dir": str(root), "split": os.path.join(str(root), "split"), "scale_factor": 2.5, "near": 0.1,
         "far": 6.0, "scene_center": center.tolist(), "use_bbox": False, "use_bbox_only_for_test": True,
         "train_start_idx": 1, "validate_idx": 3, "train_skip_step": 1, "train_max_size": 100,
         "enable_observation_check": obs_check, "max_obs_angle": 30, "max_obs_distance": 2.0,
         "bg_instance_id": list(bg_instance_id), "instance_id": list(instance_id),
         "use_instance_mask": use_instance_mask, "inst_seg_tag": "instance",
         "mask_rebalance_strategy": "fg_bg_reweight", "fg_weight": fg_weight, "bg_weight": bg_weight,
         "val_instance_id": instance_id[0]}
    c.update(over)
    return c


# the configs the tests and the golden fixtures use: name -> config keywords
CONFIGS = {
    "i1_counts": dict(instance_id=[2]),
    "i3_bg_obs": dict(instance_id=[2, 5, 300], bg_instance_id=[0, 1], obs_check=True),
    "i3_fixed": dict(instance_id=[0, 2, 4], bg_instance_id=[0], fg_weight=1.5, bg_weight=0.3),
    "no_mask": dict(instance_id=[2, 3], use_instance_mask=False),
    "zero_later_skip": dict(instance_id=[2, 0, 5], train_skip_step=2, train_max_size=2),
}


def expand_host(inp):
    """FrameSet.expand() restated on the host from read_frames' output: the all_* buffers, with GenericDataset's
    dtypes (masks bool, weights float32, ids and frame indices int64)."""
    poses, rgb, depths, labels = inp["poses"], inp["rgb"], inp["depths"], inp["labels"]
    F, H, W = rgb.shape[:3]
    HW = H * W
    focal, sf = inp["focal"], inp["scale_factor"]
    ys, xs = torch.meshgrid(torch.linspace(0, H - 1, H), torch.linspace(0, W - 1, W), indexing="ij")
    dirs = torch.stack([(xs - W / 2) / focal, -(ys - H / 2) / focal, -torch.ones_like(xs)], -1).reshape(-1, 3)
    rays = []
    for f in range(F):
        c2w = torch.from_numpy(np.asarray(poses[f], dtype=np.float32).reshape(3, 4))
        d = dirs @ c2w[:, :3].T
        d = d / torch.norm(d, dim=-1, keepdim=True)
        o = c2w[:, 3].expand(d.shape)
        near = inp["near"] / sf * torch.ones_like(o[:, :1])
        far = inp["far"] / sf * torch.ones_like(o[:, :1])
        rays.append(torch.cat([o, d, near, far], 1))
    b = inp["border"]
    y, x = torch.arange(H).view(H, 1), torch.arange(W).view(1, W)
    valid = ((y >= b) & (y < H - b) & (x >= b) & (x < W - b)).reshape(-1).repeat(F)
    lab = torch.from_numpy(labels.astype(np.int64)).reshape(F, HW) if labels is not None else None
    masks, weights, ids, passes = [], [], [], []
    for iid in inp["instance_ids"]:
        if not inp["use_instance_mask"] or iid == 0:
            m = torch.ones(F, HW, dtype=torch.bool)
            wgt = torch.zeros(F, HW)
            p = m.clone()
        else:
            m = lab == iid
            if inp["fg_weight"] is not None:
                wgt = torch.where(m, torch.tensor(np.float32(inp["fg_weight"])), torch.tensor(np.float32(inp["bg_weight"])))
            else:
                fg = m.sum(1, keepdim=True).clamp(min=1).double()
                bg = (~m).sum(1, keepdim=True).clamp(min=1).double()
                wgt = torch.where(m, (bg / fg).float(), (fg / bg).float())
            p = torch.zeros_like(m)
            for v in list(inp["bg_instance_ids"]) + [iid]:
                p |= lab == v
        masks.append(m.reshape(-1))
        weights.append(wgt.reshape(-1))
        ids.append(torch.full((F * HW,), int(iid), dtype=torch.int64))
        passes.append(p.reshape(-1))
    return {"all_rays": torch.cat(rays), "all_rgbs": torch.from_numpy(rgb).reshape(-1, 3).float().div(255),
            "all_depths": torch.from_numpy(np.asarray(depths, dtype=np.float32)).reshape(-1),
            "all_valid_masks": valid,
            "all_frame_indices": torch.from_numpy(np.asarray(inp["frame_idx"], dtype=np.int64)).repeat_interleave(HW),
            "all_instance_masks": torch.stack(masks, -1), "all_instance_masks_weight": torch.stack(weights, -1),
            "all_instance_ids": torch.stack(ids, -1), "all_pass_through_masks": torch.stack(passes, -1)}


def as_sampler_dtypes(t: torch.Tensor, key: str) -> torch.Tensor:
    """A buffer in the dtype RaySampler keeps it (masks bool, floats float32, ids int64)."""
    if key in ("all_valid_masks", "all_instance_masks", "all_pass_through_masks"):
        return t != 0
    if key in ("all_instance_ids", "all_frame_indices"):
        return t.long()
    return t.float()
