"""Held-out view metrics on the device (utils/metrics.py, include/onerf_ext.h: onerf_image_metrics, onerf_depth_metrics,
onerf_mask_metrics).

`image_metrics` gives the PSNR and SSIM of a frame for the scene and for each object: column 0 compares the scene
prediction with the ground truth over the valid pixels, column k >= 1 compares the object prediction with it over the
valid pixels labelled ids[k-1].  `psnr` and `ssim` keep the signatures of the reference's utils/metrics.py.

The definition this library implements (the kernel's contract, restated in float64 by the tests):
  - both images are set to 0 outside the column's mask m;
  - each channel is filtered with g = outer(g1, g1), g1[i] = exp(-(i - w//2)^2 / (2 * 1.5^2)) normalised to sum 1, for an
    odd window w in [1, 11], with reflect padding of w//2 (F.pad(mode="reflect"): mirror without repeating the edge), so
    the filtered image is H x W;
  - mu_p, mu_g, s_pp = E[p^2] - mu_p^2, s_gg and s_pg are the filtered moments, and
    ssim_map = ((2 mu_p mu_g + C1)(2 s_pg + C2)) / ((mu_p^2 + mu_g^2 + C1)(s_pp + s_gg + C2)), C1 = 0.01^2, C2 = 0.03^2;
  - SSIM is the mean of clamp(ssim_map, 0, 1) over the 3 channels of the pixels in m;
  - PSNR is -10 log10 of the mean squared error over the 3 channels of the pixels in m (utils/metrics.py's psnr);
  - an empty mask gives NaN for both, as the mean of an empty tensor does.
The Gaussian with sigma 1.5, the reflect border of filter2D, odd windows only and the reading of losses.ssim(pred, gt, w)
as 1 - 2 * mean(clamp(1 - ssim_map, 0, 1) / 2) = mean(clamp(ssim_map, 0, 1)) are restated from kornia 0.4.1, which the
reference's utils/metrics.ssim calls with w = 3; with m all ones the SSIM here is that function.  Zeroing outside the
mask is this library's definition for masked columns: the reference defines none.  Window sums, ssim_map and the error
sums are fp64 on the device; the returned values are float32.

`depth_metrics` gives the depth errors DEPTH_METRICS of a frame for the scene and for each object: column 0 compares
the scene depth with the ground truth over the pixels with valid and gt > 0, column k >= 1 compares the object depth
(depth_instance) with it over those pixels that are also labelled ids[k-1].  Inputs are float32 and all arithmetic is
fp64.  With s = scale (the store's scale_factor: gt and the predictions are in its units), per pixel of a column
  - g = gt s, in metres along the ray; d = clamp(pred s, d_min, d_max) with (d_min, d_max) = depth_range;
  - the sums n, sum |d - g| / g, sum (d - g)^2 / g, sum (d - g)^2, sum (ln d - ln g)^2 and, for i = 1, 2, 3, the
    counts of max(d / g, g / d) < 1.25^i;
  - abs_rel = sum |d - g| / g / n, sq_rel = sum (d - g)^2 / g / n, rmse = sqrt(sum (d - g)^2 / n),
    rmse_log = sqrt(sum (ln d - ln g)^2 / n), delta_i = count_i / n.
An empty column gives NaN; a NaN prediction makes every output of its column NaN.

`mask_metrics` scores one object's opacity map (opacity_instance rendered with that object's code everywhere) against
its instance mask over the valid pixels: with G = (label == obj_id) and P = (opacity >= threshold) (float32),
  - iou = |P & G| / |P | G|, NaN when P | G is empty;
  - opacity_l1 = sum |opacity - [G]| / n_valid (the object branch's OpacityLoss target is [G]).
The counts are exact; the sums are fp64.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import torch

from . import _lib

__all__ = ["image_metrics", "psnr", "ssim", "MetricsPlan", "DEPTH_METRICS", "depth_metrics", "mask_metrics",
           "DepthMetricsPlan", "MaskMetricsPlan"]

DEPTH_METRICS = ("abs_rel", "sq_rel", "rmse", "rmse_log", "delta1", "delta2", "delta3")


def _pixels(t: torch.Tensor, n: int, name: str, width: int = 3, dtype=torch.float32) -> torch.Tensor:
    t = t.reshape(n, width) if width > 1 else t.reshape(n)
    if t.dtype == torch.bool and dtype == torch.uint8:
        t = t.view(torch.uint8)
    if t.device.type != "cuda":
        raise RuntimeError(f"metrics: {name} must be on a CUDA device (there is no CPU path); got {t.device}")
    return t.to(dtype).contiguous()


class MetricsPlan:
    """The record and argument block of one (H, W, ids, window) configuration, and F rows of psnr / ssim outputs.
    `accumulate(...)` adds one frame to the record, `finalize(slot)` writes row `slot` and zeroes the record."""

    def __init__(self, H: int, W: int, ids: Sequence[int] = (), window: int = 3, n_frames: int = 1, device="cuda"):
        ids = [int(i) for i in ids]
        self.K, self.device = len(ids), torch.device(device)
        self.record = torch.zeros(self.K + 1, 3, dtype=torch.float64, device=self.device)
        self.psnr = torch.empty(n_frames, self.K + 1, dtype=torch.float32, device=self.device)
        self.ssim = torch.empty_like(self.psnr)
        self._ids = (C.c_int * max(1, self.K))(*ids)
        a = self.args = _lib.MetricsArgs()
        a.H, a.W, a.n_ids, a.window = int(H), int(W), self.K, int(window)
        a.ids_host = C.cast(self._ids, C.POINTER(C.c_int))
        a.record, a.psnr_out, a.ssim_out = self.record.data_ptr(), self.psnr.data_ptr(), self.ssim.data_ptr()

    def accumulate(self, pred_scene, gt, valid=None, pred_object=None, labels=None):
        """Add one frame's sums to the record (onerf_image_metrics).  Inputs as image_metrics'; the converted tensors
        are returned so that a caller capturing the call can keep them alive."""
        a, n = self.args, self.args.H * self.args.W
        held = [_pixels(pred_scene, n, "pred_scene"), _pixels(gt, n, "gt"),
                _pixels(valid, n, "valid", 1, torch.uint8) if valid is not None else None,
                _pixels(pred_object, n, "pred_object") if pred_object is not None else None,
                _pixels(labels, n, "labels", 1, torch.int16) if labels is not None else None]
        a.pred_scene, a.gt, a.valid, a.pred_object, a.labels = (_lib.ptr(t) for t in held)
        _lib.call("onerf_image_metrics", self.device, C.byref(a))
        return held

    def finalize(self, slot: int = 0):
        _lib.call("onerf_image_metrics_finalize", self.device, C.byref(self.args), int(slot))


def _labels16(labels: torch.Tensor) -> torch.Tensor:
    """Labels as the 16-bit pattern the kernel reads (uint8 / uint16 / int16 / int32 / int64 values in [0, 65535])."""
    if labels.dtype in (torch.int16, torch.uint16):
        return labels.view(torch.int16)
    return labels.to(torch.int32).to(torch.int16)       # two's-complement wrap: the low 16 bits


def image_metrics(pred_scene: torch.Tensor, gt: torch.Tensor, H: int, W: int, valid=None, pred_object=None, labels=None,
                  ids: Sequence[int] = (), window: int = 3):
    """PSNR and SSIM (module docstring) of one H x W frame: returns device tensors (psnr, ssim), each (K+1,) float32 for
    the scene column and the K = len(ids) object columns.
      pred_scene, gt  (H*W, 3) (or anything of H*W*3 values, row-major pixels) float tensors on one CUDA device
      valid           (H*W) bool / uint8, or None: every pixel
      pred_object     (H*W, 3), required with ids
      labels          (H*W) integer labels in [0, 65535], required with ids
    The call reads nothing back to the host."""
    plan = MetricsPlan(H, W, ids, window, 1, pred_scene.device)
    plan.accumulate(pred_scene, gt, valid, pred_object, _labels16(labels) if labels is not None else None)
    plan.finalize(0)
    return plan.psnr[0], plan.ssim[0]


def psnr(image_pred: torch.Tensor, image_gt: torch.Tensor, valid_mask=None, reduction: str = "mean") -> torch.Tensor:
    """utils/metrics.py's psnr: -10 log10 of the mean squared error over the elements valid_mask selects.  The images
    are (..., 3) (pixels of 3 channels), valid_mask of the pixel shape image_pred.shape[:-1].  Returns a 0-d float32
    device tensor (NaN for an empty mask)."""
    if reduction != "mean":
        raise ValueError("metrics.psnr: only reduction='mean' is supported")
    if image_pred.shape != image_gt.shape or image_pred.shape[-1] != 3:
        raise ValueError(f"metrics.psnr: images must be (..., 3) of one shape, got {tuple(image_pred.shape)} and "
                         f"{tuple(image_gt.shape)}")
    n = image_pred.numel() // 3
    if valid_mask is not None and tuple(valid_mask.shape) != tuple(image_pred.shape[:-1]):
        raise ValueError(f"metrics.psnr: valid_mask must be {tuple(image_pred.shape[:-1])}, got {tuple(valid_mask.shape)}")
    return image_metrics(image_pred, image_gt, 1, n, valid=valid_mask, window=1)[0][0]


def ssim(image_pred: torch.Tensor, image_gt: torch.Tensor, reduction: str = "mean") -> torch.Tensor:
    """utils/metrics.py's ssim: image_pred and image_gt (1, 3, H, W); the mean of clamp(ssim_map, 0, 1) with window 3
    (module docstring).  Returns a 0-d float32 device tensor."""
    if reduction != "mean":
        raise ValueError("metrics.ssim: only reduction='mean' is supported")
    if image_pred.dim() != 4 or image_pred.shape[:2] != (1, 3) or image_gt.shape != image_pred.shape:
        raise ValueError(f"metrics.ssim: images must be (1, 3, H, W) of one shape, got {tuple(image_pred.shape)} and "
                         f"{tuple(image_gt.shape)}")
    H, W = image_pred.shape[2:]
    hwc = lambda t: t[0].permute(1, 2, 0).reshape(H * W, 3)
    return image_metrics(hwc(image_pred), hwc(image_gt), H, W, window=3)[1][0]


class DepthMetricsPlan:
    """The record and argument block of one (H, W, ids, scale, depth_range) configuration, and F rows of depth metrics
    (F, K+1, 7).  `accumulate(...)` adds one frame to the record, `finalize(slot)` writes row `slot` and zeroes the
    record."""

    def __init__(self, H: int, W: int, ids: Sequence[int] = (), scale: float = 1.0, depth_range=(1e-3, 10.0),
                 n_frames: int = 1, device="cuda"):
        ids = [int(i) for i in ids]
        self.K, self.device = len(ids), torch.device(device)
        self.record = torch.zeros(self.K + 1, _lib.DEPTH_RECORD, dtype=torch.float64, device=self.device)
        self.out = torch.empty(n_frames, self.K + 1, _lib.DEPTH_METRICS, dtype=torch.float32, device=self.device)
        self._ids = (C.c_int * max(1, self.K))(*ids)
        a = self.args = _lib.DepthMetricsArgs()
        a.H, a.W, a.n_ids = int(H), int(W), self.K
        a.ids_host = C.cast(self._ids, C.POINTER(C.c_int))
        a.scale, a.d_min, a.d_max = float(scale), float(depth_range[0]), float(depth_range[1])
        a.record, a.out = self.record.data_ptr(), self.out.data_ptr()

    def accumulate(self, pred_scene, gt, valid=None, pred_object=None, labels=None):
        """Add one frame's sums to the record (onerf_depth_metrics).  Inputs as depth_metrics'; the converted tensors
        are returned so that a caller capturing the call can keep them alive."""
        a, n = self.args, self.args.H * self.args.W
        held = [_pixels(pred_scene, n, "pred_scene", 1), _pixels(gt, n, "gt", 1),
                _pixels(valid, n, "valid", 1, torch.uint8) if valid is not None else None,
                _pixels(pred_object, n, "pred_object", 1) if pred_object is not None else None,
                _pixels(_labels16(labels), n, "labels", 1, torch.int16) if labels is not None else None]
        a.pred_scene, a.gt, a.valid, a.pred_object, a.labels = (_lib.ptr(t) for t in held)
        _lib.call("onerf_depth_metrics", self.device, C.byref(a))
        return held

    def finalize(self, slot: int = 0):
        _lib.call("onerf_depth_metrics_finalize", self.device, C.byref(self.args), int(slot))


class MaskMetricsPlan:
    """The record and argument block of one (H, W, ids, threshold) configuration, and F rows of iou / opacity_l1
    (F, K).  `accumulate(k, ...)` adds one frame's opacity map of object ids[k] to the record, `finalize(slot)` writes
    row `slot` and zeroes the record."""

    def __init__(self, H: int, W: int, ids: Sequence[int], threshold: float = 0.5, n_frames: int = 1, device="cuda"):
        self.ids = [int(i) for i in ids]
        self.K, self.device = len(self.ids), torch.device(device)
        self.record = torch.zeros(max(1, self.K), _lib.MASK_RECORD, dtype=torch.float64, device=self.device)
        self.iou = torch.empty(n_frames, self.K, dtype=torch.float32, device=self.device)
        self.opacity_l1 = torch.empty_like(self.iou)
        a = self.args = _lib.MaskMetricsArgs()
        a.H, a.W, a.n_ids, a.threshold = int(H), int(W), self.K, float(threshold)
        a.record, a.iou_out, a.opacity_l1_out = self.record.data_ptr(), self.iou.data_ptr(), self.opacity_l1.data_ptr()

    def accumulate(self, k: int, opacity, labels, valid=None):
        """Add the sums of object ids[k]'s opacity map to row k of the record (onerf_mask_metrics).  Inputs as
        mask_metrics'; the converted tensors are returned so that a caller capturing the call can keep them alive."""
        a, n = self.args, self.args.H * self.args.W
        held = [_pixels(opacity, n, "opacity", 1), _pixels(_labels16(labels), n, "labels", 1, torch.int16),
                _pixels(valid, n, "valid", 1, torch.uint8) if valid is not None else None]
        a.opacity, a.labels, a.valid = (_lib.ptr(t) for t in held)
        a.column = int(k)
        a.id = self.ids[k] if 0 <= k < self.K else -1          # a column outside [0, K) is refused by the call
        _lib.call("onerf_mask_metrics", self.device, C.byref(a))
        return held

    def finalize(self, slot: int = 0):
        _lib.call("onerf_mask_metrics_finalize", self.device, C.byref(self.args), int(slot))


def depth_metrics(pred_scene: torch.Tensor, gt: torch.Tensor, H: int, W: int, valid=None, pred_object=None,
                  labels=None, ids: Sequence[int] = (), scale: float = 1.0, depth_range=(1e-3, 10.0)) -> torch.Tensor:
    """Depth errors (module docstring) of one H x W frame: a (K+1, 7) float32 device tensor, row 0 the scene and row k
    object ids[k-1], columns in DEPTH_METRICS order.
      pred_scene, gt  (H*W) (or anything of H*W values, row-major pixels) float tensors on one CUDA device, in the
                      store's units (depth_fine and the frame store's processed depths)
      valid           (H*W) bool / uint8, or None: every pixel
      pred_object     (H*W) object depth (depth_instance), required with ids
      labels          (H*W) integer labels in [0, 65535], required with ids
      ids             up to 64 distinct object ids
      scale           metres per unit of gt and the predictions (the store's scale_factor)
      depth_range     (d_min, d_max) in metres, 0 < d_min < d_max: the clamp of the predictions
    The call reads nothing back to the host."""
    plan = DepthMetricsPlan(H, W, ids, scale, depth_range, 1, pred_scene.device)
    plan.accumulate(pred_scene, gt, valid, pred_object, labels)
    plan.finalize(0)
    return plan.out[0]


def mask_metrics(opacity: torch.Tensor, labels: torch.Tensor, obj_id: int, valid=None, threshold: float = 0.5):
    """Instance-mask agreement (module docstring) of one object's opacity map: device tensors (iou, opacity_l1), each
    0-d float32.  opacity (N,) float, labels (N,) integer labels in [0, 65535], valid (N,) bool / uint8 or None: every
    pixel.  The call reads nothing back to the host."""
    n = opacity.numel()
    if labels.numel() != n or (valid is not None and valid.numel() != n):
        raise ValueError(f"metrics.mask_metrics: opacity, labels and valid need one pixel count, got {n}, "
                         f"{labels.numel()} and {None if valid is None else valid.numel()}")
    if not 0 < n < 2 ** 31:
        raise ValueError(f"metrics.mask_metrics: 1 to 2^31 - 1 pixels, got {n}")
    plan = MaskMetricsPlan(1, n, [obj_id], threshold, 1, opacity.device)
    plan.accumulate(0, opacity, labels, valid)
    plan.finalize(0)
    return plan.iou[0, 0], plan.opacity_l1[0, 0]
