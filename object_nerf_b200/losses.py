"""TotalLoss of the training step on the device (SURVEY.md section 8f row 3).

Mirror of models/losses.py:5-135 (`TotalLoss`, `get_loss`): same config keys, same `forward(inputs, batch, epoch)`
signature, same `(loss_sum, loss_dict)` result - `loss_dict` holds the unweighted value of every term that is present
(a term whose mask is empty is absent, as in the reference).  Loss and d(loss_sum)/d(maps) come from two kernels of
libonerf_sm100.so (`csrc/loss.cu`) instead of ~120 torch kernels and several host syncs; `loss_sum` carries autograd
into the rendered maps (and from there through `backward.RenderRaysFn`).  `loss_dict` values are detached (the
reference only ever logs them, train.py:182-191).
"""
import ctypes as C
from typing import Dict

import torch
from torch import nn

from . import _lib

TERMS = ("color_loss", "depth_loss", "opacity_loss", "instance_color_loss", "instance_depth_loss")
MAPS = ("rgb", "depth", "opacity_instance", "rgb_instance", "depth_instance")


def fill_loss_args(a, weights, out: torch.Tensor, present: torch.Tensor) -> None:
    """Set onerf_loss_args' five term weights (TERMS order) and its outputs: out (6,) = loss_sum then the five terms,
    present (5,) int32."""
    (a.color_weight, a.depth_weight, a.opacity_weight, a.instance_color_weight, a.instance_depth_weight) = weights
    a.loss_sum_out, a.terms_out, a.present_out = out.data_ptr(), out[1:].data_ptr(), present.data_ptr()


class _TotalLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, weights, batch, has_fine, *maps):
        dev = maps[0].device
        n = maps[0].shape[0]
        maps = [m.detach().contiguous().float() for m in maps]
        grads = [torch.empty_like(m) for m in maps]
        out = torch.empty(1 + 5, dtype=torch.float32, device=dev)          # loss_sum, 5 terms
        present = torch.empty(5, dtype=torch.int32, device=dev)
        ws = torch.empty(_lib.load().onerf_total_loss_workspace_bytes() // 8, dtype=torch.float64, device=dev)
        keep = [batch["rgbs"].reshape(n, 3).contiguous().float(), batch["depths"].reshape(n).contiguous().float(),
                batch["valid_mask"].reshape(n).to(torch.uint8).contiguous(),
                batch["instance_mask"].reshape(n).to(torch.uint8).contiguous(),
                batch["instance_mask_weight"].reshape(n).contiguous().float()]
        a = _lib.LossArgs()
        a.n_rays, a.has_fine = n, int(has_fine)
        for i, typ in enumerate(("coarse", "fine") if has_fine else ("coarse",)):
            for j, k in enumerate(MAPS):
                setattr(getattr(a, typ), k, maps[5 * i + j].data_ptr())
                setattr(getattr(a, "grad_" + typ), k, grads[5 * i + j].data_ptr())
        a.rgbs, a.depths, a.valid_mask, a.instance_mask, a.instance_mask_weight = (t.data_ptr() for t in keep)
        fill_loss_args(a, weights, out, present)
        a.workspace = ws.data_ptr()
        _lib.call("onerf_total_loss", dev, C.byref(a))
        ctx.grads = grads
        ctx.mark_non_differentiable(present)
        return out[0], out[1:].detach(), present

    @staticmethod
    def backward(ctx, g_sum, _g_terms, _g_present):
        return (None, None, None) + tuple(g * g_sum for g in ctx.grads)


class TotalLoss(nn.Module):
    """models/losses.py:101-133."""

    def __init__(self, conf):
        super().__init__()
        self.conf = conf

    def forward(self, inputs: Dict[str, torch.Tensor], batch: Dict[str, torch.Tensor], epoch: int = -1):
        has_fine = "rgb_fine" in inputs
        maps = [inputs[f"{k}_{typ}"] for typ in (("coarse", "fine") if has_fine else ("coarse",)) for k in MAPS]
        weights = tuple(float(self.conf[f"{t}_weight"]) for t in TERMS)
        loss_sum, terms, present = _TotalLossFn.apply(weights, batch, has_fine, *maps)
        flags = present.tolist()                       # the one host read (the reference syncs per term)
        loss_dict = {t: terms[i] for i, t in enumerate(TERMS) if flags[i]}
        return loss_sum, loss_dict


def get_loss(config):
    """models/losses.py:136-137."""
    return TotalLoss(config.loss)
