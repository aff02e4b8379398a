"""Camera rays and per-object ray assembly on the device (SURVEY.md section 8f rows 1-2).

Mirrors, with the reference's names and argument meaning:
  get_ray_directions, get_rays            datasets/ray_utils.py:5-51
  get_ray_bbox_intersections              utils/bbox_utils.py:132-156 (a BBoxRayHelper method; here a function of the helper)
  generate_rays                           render_tools/editable_renderer.py:153-181 (an EditableRenderer method)
plus `camera_rays`, the three fused into one kernel (pixel grid + pose + box -> (H*W, 8) rays).
The reference does the box part on the host (numpy float64 + numba) per frame and object and uploads the result;
these run as HBM-bound kernels of libonerf_sm100.so on the current CUDA stream.  There is no CPU path.
"""
import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib


def _device(device=None) -> torch.device:
    return torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())


def _c2w_host(c2w):
    a = np.ascontiguousarray(torch.as_tensor(c2w).detach().cpu().numpy()[:3, :4], dtype=np.float32)
    return (C.c_float * 12)(*a.reshape(-1).tolist())


def _box_host(box, bbox_enlarge: float) -> _lib.BoxHost:
    """box: anything with the BBoxRayHelper attributes pose_avg, axis_align_mat, bbox_bounds (utils/bbox_utils.py)."""
    b = _lib.BoxHost()
    P = np.asarray(box.pose_avg, dtype=np.float64).squeeze()
    A = np.asarray(box.axis_align_mat, dtype=np.float64)
    bounds = np.array(box.bbox_bounds, dtype=np.float64, copy=True)
    if bbox_enlarge > 0:                      # utils/bbox_utils.py:140-145
        bounds[0] -= bbox_enlarge
        bounds[1] += bbox_enlarge
    for i in range(3):
        for j in range(4):
            b.pose_avg[4 * i + j] = P[i, j]
            b.axis_align[4 * i + j] = A[i, j]
    for i in range(6):
        b.bounds[i] = bounds.reshape(-1)[i]
    return b


def get_ray_directions(H: int, W: int, focal: float, device=None) -> torch.Tensor:
    """(H, W, 3) camera-space directions, datasets/ray_utils.py:5-25 (returned on the GPU)."""
    dev = _device(device)
    out = torch.empty(H, W, 3, dtype=torch.float32, device=dev)
    _lib.call("onerf_ray_directions", dev, H, W, float(focal), out.data_ptr())
    return out


def get_rays(directions: torch.Tensor, c2w):
    """datasets/ray_utils.py:28-51: world-space (rays_o, rays_d), (H*W, 3) each, rays_d unit-norm."""
    d = directions.contiguous().float()
    n = d.numel() // 3
    rays_o = torch.empty(n, 3, dtype=torch.float32, device=d.device)
    rays_d = torch.empty(n, 3, dtype=torch.float32, device=d.device)
    _lib.call("onerf_get_rays", d.device, d.data_ptr(), n, _c2w_host(c2w), rays_o.data_ptr(), rays_d.data_ptr())
    return rays_o, rays_d


def generate_rays(obj_id: int, rays_o: torch.Tensor, rays_d: torch.Tensor, near: float, far: float, scale_factor: float,
                  box=None, bbox_enlarge: float = 0.0, return_mask: bool = False):
    """render_tools/editable_renderer.py:153-181: the (N, 8) rays of one object.  obj_id == 0: scene near / far;
    otherwise `box` (the object's BBoxRayHelper) gives per-ray near / far (0 / 0 where the ray misses the box)."""
    rays_o, rays_d = rays_o.contiguous().float(), rays_d.contiguous().float()
    n, dev = rays_o.shape[0], rays_o.device
    out = torch.empty(n, 8, dtype=torch.float32, device=dev)
    hit = torch.empty(n, dtype=torch.uint8, device=dev) if return_mask else None
    bh = None
    if obj_id != 0:
        if box is None:
            raise ValueError("generate_rays: an object (obj_id != 0) needs its bounding-box helper")
        bh = C.byref(_box_host(box, bbox_enlarge))
    _lib.call("onerf_generate_rays", dev, rays_o.data_ptr(), rays_d.data_ptr(), n, bh, float(scale_factor), float(near),
              float(far), out.data_ptr(), _lib.ptr(hit))
    return (out, hit.bool()) if return_mask else out


def get_ray_bbox_intersections(box, rays_o: torch.Tensor, rays_d: torch.Tensor, scale_factor: Optional[float] = None,
                               bbox_enlarge: float = 0.0):
    """utils/bbox_utils.py:132-156: (bbox_mask (N,) bool, batch_near (N,1), batch_far (N,1)), near / far already divided
    by the scale factor.  (The reference leaves the slab test's zeros in the missed rays' near / far; so do we.)"""
    sf = float(scale_factor if scale_factor is not None else box.scale_factor)
    rays, mask = generate_rays(1, rays_o, rays_d, 0.0, 0.0, sf, box=box, bbox_enlarge=bbox_enlarge, return_mask=True)
    return mask, rays[:, 6:7].contiguous(), rays[:, 7:8].contiguous()


def camera_rays(H: int, W: int, focal: float, c2w, near: float, far: float, scale_factor: float, box=None,
                bbox_enlarge: float = 0.0, device=None, return_mask: bool = False):
    """get_ray_directions + get_rays + generate_rays in one kernel: (H*W, 8) rays for the scene (box None) or an object."""
    dev = _device(device)
    out = torch.empty(H * W, 8, dtype=torch.float32, device=dev)
    hit = torch.empty(H * W, dtype=torch.uint8, device=dev) if return_mask else None
    bh = C.byref(_box_host(box, bbox_enlarge)) if box is not None else None
    _lib.call("onerf_camera_rays", dev, H, W, float(focal), _c2w_host(c2w), bh, float(scale_factor), float(near),
              float(far), out.data_ptr(), _lib.ptr(hit))
    return (out, hit.bool()) if return_mask else out
