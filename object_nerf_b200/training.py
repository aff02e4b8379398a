"""One training step in one library call (train.py:147-180 up to loss.backward(), reference models/losses.py and
models/rendering.py): `train_step` runs onerf_train_step, which renders both passes, evaluates TotalLoss, back-propagates
through compositing (fused into the compositing kernels) and the two MLPs, and accumulates the gradients into the
`.grad` of the reference-named parameters, the code table and the voxel table.

Unlike render_rays -> TotalLoss -> loss.backward() it reads nothing back to the host and, after the first call for a
given configuration, allocates no device memory: buffers, packed weights and the training workspace belong to a plan
cached per coarse model and configuration (the plans go when the model does).  A step can therefore be captured in a
CUDA graph together with `torch.optim.Adam(..., capturable=True)` and replayed.  Keep the gradients allocated between
steps (`optimizer.zero_grad(set_to_none=False)`): a missing `.grad` is created (zero-filled) on the call that finds it
missing.

A replay repeats what the capture saw on the host, in particular the voxel grid's buffers.  Grid maintenance
(EmbeddingVoxel.voxel_subdivision, .self_pruning_empty_voxels) replaces or reshapes them, so recapture the graph after
it; eager calls pick the current grid up on every call.

The random draws (stratified jitter, importance u, sigma noise) are fresh on every replay.  An eager call draws a new
Philox seed from torch's generator (`engine.new_seed`) and passes it by value (onerf_train_step).  A call made while
the current stream is capturing runs onerf_train_step_dseed instead: its kernels read the seed from the plan's device
counter `seed_dev` when they run, and the step's last compositing kernel adds 4 to it.  Replay k of a graph captured
with the counter at s0 therefore draws exactly what an eager step with seed s0 + 4k draws.  The counter is written once,
when the plan is made, with the seed of that (eager) first call plus 4; `step_seed` reads it.  The first call for a
configuration must therefore run eagerly (the usual warm-up before a capture): a plan made inside a capture would have
its counter reset on every replay, so that is refused.  Injected `_rand` buffers take precedence over either seed.

The returned tensors are the plan's output buffers and are overwritten by the next step of the same plan.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Any, Dict

import torch

from . import _lib, backward, engine
from .losses import TERMS

__all__ = ["train_step", "step_seed"]

_RAND_KEYS = ("jitter", "u", "noise_scene_coarse", "noise_obj_coarse", "noise_scene_fine", "noise_obj_fine")
# coarse model -> {configuration: plan}; a plan references no module, so it lives exactly as long as the model
_plans: "weakref.WeakKeyDictionary[Any, Dict[tuple, _StepPlan]]" = weakref.WeakKeyDictionary()


def _is_voxel(emb) -> bool:
    return hasattr(emb, "voxel_idx_map")


class _StepPlan:
    """Every buffer one configuration of the step needs, allocated once."""

    def __init__(self, models, emb_xyz, n, cfg, rand, dev, seed):
        lib = _lib.load()
        self.n, self.dev, self.cfg = n, dev, cfg
        # the device seed of captured steps (onerf_train_step_dseed), continuing from the creating call's host seed
        self.seed_dev = torch.full((1,), seed + 4, dtype=torch.int64, device=dev)
        self.model_order = ["coarse"] + (["fine"] if cfg["N_importance"] > 0 else [])
        self.use_voxel = _is_voxel(emb_xyz)
        f = lambda *shape, dtype=torch.float32: torch.empty(*shape, dtype=dtype, device=dev)
        self.rays, self.ids, self.codes, self.d_codes = f(n, 8), f(n, dtype=torch.int64), f(n, 64), f(n, 64)
        self.rgbs, self.depths, self.weight = f(n, 3), f(n), f(n)
        self.valid, self.inst, self.ptm = (f(n, dtype=torch.uint8) for _ in range(3))
        self.out, self.present, self.psnr = f(1 + len(TERMS)), f(len(TERMS), dtype=torch.int32), f(1)
        nbytes = lib.onerf_packed_weights_bytes(int(self.use_voxel))
        self.packed = {}
        for typ in self.model_order:
            engine.check_architecture(models[typ], self.use_voxel)
            blob = torch.empty(nbytes + 1024, dtype=torch.uint8, device=dev)
            off = (-blob.data_ptr()) % 1024
            self.packed[typ] = blob[off:off + nbytes]
        prec = engine.PRECISIONS[cfg["precision"]]
        self.ws = backward._pool.take(lib.onerf_train_step_workspace_bytes(
            prec, int(self.use_voxel), n, cfg["N_samples"], cfg["N_importance"]), dev)
        # the grid is set on every call (train_step): grid maintenance replaces its buffers between steps
        self.render = engine.RenderPlan(
            self.rays, self.packed["coarse"], self.packed.get("fine"), None, codes=self.codes,
            n_samples=cfg["N_samples"], n_importance=cfg["N_importance"], use_disp=cfg["use_disp"],
            perturb=cfg["perturb"], noise_std=cfg["noise_std"], white_back=cfg["white_back"], forward_instance=True,
            is_eval=cfg["is_eval"], zero_last_delta=cfg["zero_last_delta"], rays_in_bbox=cfg["rays_in_bbox"],
            frustum_bound_th=cfg["frustum_bound_th"], pass_through_mask=self.ptm if cfg["has_ptm"] else None,
            precision=cfg["precision"], rand=rand, train_ws=self.ws)
        la = _lib.LossArgs()
        la.n_rays, la.has_fine = n, int(len(self.model_order) == 2)
        la.rgbs, la.depths, la.valid_mask = self.rgbs.data_ptr(), self.depths.data_ptr(), self.valid.data_ptr()
        la.instance_mask, la.instance_mask_weight = self.inst.data_ptr(), self.weight.data_ptr()
        (la.color_weight, la.depth_weight, la.opacity_weight, la.instance_color_weight,
         la.instance_depth_weight) = cfg["loss_weights"]
        la.loss_sum_out, la.terms_out, la.present_out = self.out.data_ptr(), self.out[1:].data_ptr(), self.present.data_ptr()
        self.loss_args = la


def _capturing(dev) -> bool:
    return dev.type == "cuda" and torch.cuda.is_current_stream_capturing()


def step_seed(models: Dict[str, Any]) -> torch.Tensor:
    """A copy of the device seed counter of the model's train_step plan (one int64 on the device): the Philox seed the
    next captured step's replay draws with.  Taken inside a captured region, the copy is made on every replay.  The
    model must have exactly one plan (one train_step configuration)."""
    plans = list(_plans.get(models["coarse"], {}).values())
    if len(plans) != 1:
        raise ValueError(f"step_seed needs exactly one train_step plan for this model, found {len(plans)}")
    return plans[0].seed_dev.clone()


def _grad_of(p: torch.Tensor) -> torch.Tensor:
    if p.grad is None:
        p.grad = torch.zeros_like(p, memory_format=torch.contiguous_format)
    g = p.grad
    if g.dtype != torch.float32 or not g.is_contiguous():
        raise RuntimeError("train_step accumulates into contiguous fp32 .grad tensors")
    return g


def _f32_param(p: torch.Tensor) -> torch.Tensor:
    if p.dtype != torch.float32 or not p.is_contiguous():
        raise RuntimeError("train_step trains contiguous fp32 parameters")
    return p.detach()


def train_step(models: Dict[str, Any], embeddings: Dict[str, Any], code_library, batch: Dict[str, torch.Tensor],
               loss_conf, N_samples: int = 64, use_disp: bool = False, perturb: float = 0, noise_std: float = 1,
               N_importance: int = 0, white_back: bool = False, forward_instance: bool = True,
               frustum_bound_th: float = 0, pass_through_mask=None, rays_in_bbox: bool = False, **render_kwargs):
    """render_rays(models, embeddings, batch["rays"], ...) with the codes code_library(batch) looks up, then
    TotalLoss(loss_conf) and its backward, as one call.  Takes render_rays' keyword arguments (train.py:84-98, 155-165;
    is_eval, use_zero_as_last_delta, precision and _rand included, the rest ignored as render_rays ignores them).

    Returns (loss_sum, terms, present, psnr) as device tensors: loss_sum (), the five unweighted terms (5,) in
    losses.TERMS order (0 where skipped), present (5,) int32 flags (TotalLoss's loss_dict holds term i iff present[i]),
    and the PSNR of the fine pass's rgb (coarse without a fine pass) over the valid rays (train.py:171-172)."""
    if not forward_instance:
        raise NotImplementedError("TotalLoss needs the object branch's maps: train_step runs with forward_instance=True")
    lib = _lib.load()
    rays = batch["rays"].reshape(-1, 8)
    dev = rays.device
    n = rays.shape[0]
    emb_xyz = embeddings["xyz"]
    precision = render_kwargs.get("precision") or engine.default_precision()
    rand = render_kwargs.get("_rand") or {}
    cfg = dict(N_samples=int(N_samples), N_importance=int(N_importance), use_disp=bool(use_disp), perturb=float(perturb),
               noise_std=float(noise_std), white_back=bool(white_back), is_eval=bool(render_kwargs.get("is_eval", False)),
               zero_last_delta=bool(render_kwargs.get("use_zero_as_last_delta", False)),
               rays_in_bbox=bool(rays_in_bbox), frustum_bound_th=float(frustum_bound_th),
               has_ptm=pass_through_mask is not None, precision="bf16" if precision == "bf16" else "fp32",
               loss_weights=tuple(float(loss_conf[f"{t}_weight"]) for t in TERMS))
    use_voxel = _is_voxel(emb_xyz)
    table = emb_xyz.embedding_space_ftr.weight if use_voxel else None
    key = (dev, n, use_voxel, tuple(sorted(cfg.items())),
           tuple(rand[k].data_ptr() if rand.get(k) is not None else 0 for k in _RAND_KEYS))
    capturing = _capturing(dev)
    seed = engine.new_seed() if not capturing and (cfg["perturb"] > 0 or cfg["noise_std"] > 0) else 0
    plans = _plans.setdefault(models["coarse"], {})
    plan = plans.get(key)
    if plan is None:
        if capturing:
            raise RuntimeError("train_step: the first call for a configuration must run before the CUDA-graph capture "
                               "(warm up eagerly): its plan's device seed counter would be reset on every replay")
        plan = plans[key] = _StepPlan(models, emb_xyz, n, cfg, rand, dev, seed)
    # the grid as it is now (host-side argument block only)
    plan.grid = engine.GridBuffers.from_module(emb_xyz) if use_voxel else None
    plan.render.args.grid = C.pointer(plan.grid.c) if use_voxel else None
    # the batch into the plan's buffers (device copies only)
    plan.rays.copy_(rays)
    plan.ids.copy_(batch["instance_ids"].reshape(-1))
    plan.rgbs.copy_(batch["rgbs"].reshape(n, 3))
    plan.depths.copy_(batch["depths"].reshape(n))
    plan.valid.copy_(batch["valid_mask"].reshape(n))
    plan.inst.copy_(batch["instance_mask"].reshape(n))
    plan.weight.copy_(batch["instance_mask_weight"].reshape(n))
    if pass_through_mask is not None:
        plan.ptm.copy_(pass_through_mask.reshape(n))
    plan.d_codes.zero_()
    code_table = code_library.embedding_instance.weight
    ctx, stream = _lib.ctx(dev), _lib.stream()
    keep = []
    with torch.cuda.device(dev):
        _lib.check(lib.onerf_code_gather(ctx, _f32_param(code_table).data_ptr(), plan.ids.data_ptr(), n,
                                         code_table.shape[0], plan.codes.data_ptr(), stream))
        b = _lib.RenderBwdArgs()
        for typ in plan.model_order:
            lin = engine.model_linears(models[typ])
            Wp = (C.c_void_p * 20)(*[_f32_param(w).data_ptr() for w, _ in lin])
            Bp = (C.c_void_p * 20)(*[_f32_param(bb).data_ptr() for _, bb in lin])
            dWp = (C.c_void_p * 20)(*[_grad_of(w).data_ptr() for w, _ in lin])
            dbp = (C.c_void_p * 20)(*[_grad_of(bb).data_ptr() for _, bb in lin])
            keep += [Wp, Bp, dWp, dbp]
            _lib.check(lib.onerf_pack_weights(ctx, int(plan.use_voxel), Wp, Bp, plan.packed[typ].data_ptr(),
                                              plan.packed[typ].numel(), stream))
            setattr(b, "W_" + typ, Wp)
            setattr(b, "dW_" + typ, dWp)
            setattr(b, "db_" + typ, dbp)
        b.d_codes = plan.d_codes.data_ptr()
        b.table_grad = _grad_of(table).data_ptr() if table is not None else None
        a = plan.render.args
        if capturing:
            _lib.check(lib.onerf_train_step_dseed(ctx, C.byref(a), C.byref(plan.loss_args), C.byref(b),
                                                  plan.psnr.data_ptr(), plan.seed_dev.data_ptr(), stream))
        else:
            a.seed = seed
            _lib.check(lib.onerf_train_step(ctx, C.byref(a), C.byref(plan.loss_args), C.byref(b), plan.psnr.data_ptr(),
                                            stream))
        _lib.check(lib.onerf_code_scatter_add(ctx, plan.d_codes.data_ptr(), plan.ids.data_ptr(), n, code_table.shape[0],
                                              _grad_of(code_table).data_ptr(), stream))
    return plan.out[0], plan.out[1:], plan.present, plan.psnr[0]
