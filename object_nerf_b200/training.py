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

Data-parallel training (`group=`, a torch.distributed process group; DDP's semantics without DDP's hooks, which never
fire because the step writes `.grad` without autograd):
  - the plan made by the first call with a group allocates one fp32 gradient bucket and points the `.grad` of every
    trained tensor at a view of it: the 40 tensors of each model in engine.model_linears order (fine model first), the
    code table, the voxel table last, every offset 16-byte aligned.  Values already in `.grad` are copied in.  Keep
    them there: a later call whose `.grad` no longer aliases the bucket (`zero_grad(set_to_none=True)`, a replaced
    parameter) is refused;
  - after the step, one all-reduce (SUM, then a scale by 1/W: the mean over ranks, as DDP) of the bucket's prefix runs
    on the current stream.  The prefix ends after voxel-table row n_used: only rows the index map references,
    [0, n_used), can receive gradient, so the rows above are zero on every rank.  The whole prefix is reduced, including
    what `.grad` held before the step (as DDP without no_sync): zero the gradients before each step.  With NCCL the
    reduction captures in the step's CUDA graph;
  - `sync_replicas` must have run since the last change to the grid: it broadcasts rank 0's parameters and grid (DDP's
    construction-time broadcast and broadcast_buffers) and counts n_used.  Call it before training and after every
    grid maintenance (pruning without `group=` draws its jitter per rank, so the ranks' grids differ after it; with
    `group=` they stay identical, and the rule still holds);
  - rank r draws with the seed a group-less call would use plus r * 2^52 (mod 2^62), both the host seed and the start of
    the device counter.  A deliberate difference from the reference: its ranks start from identical torch generators
    and would draw the same jitter and noise at the same batch positions.  Injected `_rand` buffers still win;
  - the returned loss, terms, flags and PSNR are this rank's (train.py logs them per rank).

Through autograd (`TrainStepFn`, `install_training`): for host loops that call loss.backward() themselves (Lightning,
DDP, GradScaler).  The step writes its gradients into a bucket its plan owns (`grad_sink=True`, the `group=` bucket's
layout) and leaves `.grad` alone; the backward hands copies of them, times the incoming gradient, to autograd.
`install_training(ObjectNeRFSystem)` binds this as the reference's `training_step`.

Validation (`validate_frame`, `install_validation`): the other half of train.py's loop, one validation image per call
(onerf_validate_frame, include/onerf_ext.h).  The image runs through render_rays' passes (is_eval, perturb = 0,
noise_std = 0: nothing is random) in chunks of `chunk` rays; each pass's compositing kernel also adds the ray's squared
errors of the five TotalLoss terms and of the validation PSNR to an 18-double record, and one more launch turns the
record into the loss outputs.  Only the requested maps of the last pass are image-sized; weights and z_vals exist for
one chunk at a time.  Like the step it reads nothing back, allocates nothing after the first call for a shape (a plan
per coarse model and configuration owns the buffers; the returned tensors are overwritten by the next call of the same
plan) and can be captured: the batch tensors are read in place when they already have the kernels' types (float32,
int64 ids, bool or uint8 masks, 8 ray columns), so a replay validates whatever they hold by then, with the weights
re-packed from the parameters as they are by then.  With `group=` rank r renders parallel.shard_bounds(n_rays, W, r),
the records are all-reduced (SUM, float64) before the finalising launch, so every rank returns the loss and PSNR of the
whole image, and the maps are all-gathered (parallel.gather_tiles, which allocates the gathered tensors).
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Any, Dict

import torch

from . import _lib, backward, engine, parallel
from .losses import TERMS, fill_loss_args
from .rendering import _is_voxel

__all__ = ["train_step", "step_seed", "sync_replicas", "TrainStepFn", "install_training", "validate_frame",
           "install_validation"]

_RAND_KEYS = ("jitter", "u", "noise_scene_coarse", "noise_obj_coarse", "noise_scene_fine", "noise_obj_fine")
# coarse model -> {configuration: plan}; a plan references no module, so it lives exactly as long as the model
_plans: "weakref.WeakKeyDictionary[Any, Dict[tuple, _StepPlan]]" = weakref.WeakKeyDictionary()
# coarse model -> (grid stamp or None, n_used) of its last sync_replicas
_synced: "weakref.WeakKeyDictionary[Any, tuple]" = weakref.WeakKeyDictionary()
RANK_SEED_STRIDE = 1 << 52
# EmbeddingVoxel's grid state besides the table (voxel_occupancy and voxel_count are absent from bare grid modules)
GRID_BUFFERS = ("voxel_shape", "voxel_size", "voxel_offset", "voxel_count", "voxel_idx_map", "voxel_occupancy")


def _grid_stamp(emb) -> tuple:
    """What grid maintenance changes, readable without the device: the index map's address, shape and in-place
    version (pruning writes it in place, subdivision replaces it)."""
    m = emb.voxel_idx_map
    return m.data_ptr(), tuple(m.shape), m._version


def _trained_tensors(models, model_order, code_table, table) -> list:
    """The tensors a step writes gradients for, in bucket order."""
    out = []
    for typ in reversed(model_order):            # fine first
        for w, b in engine.model_linears(models[typ]):
            out += [w, b]
    out.append(code_table)
    if table is not None:
        out.append(table)
    return out


def _grad_ptrs(tensors) -> list:
    return [t.grad.data_ptr() if t.grad is not None else 0 for t in tensors]


class _GradBucket:
    """One fp32 buffer with a gradient view per trained tensor (layout: _trained_tensors, each offset rounded up to 4
    floats): either the `.grad` of every trained tensor views it (`adopt`), so that a step's gradients are reduced by one
    all-reduce, or it is the step's own gradient sink (train_step(grad_sink=True))."""

    def __init__(self, tensors, has_table, dev):
        self.flat, self.views, self.offsets = engine.grad_buffer(tensors, dev)
        self.table_offset = self.offsets[-1] if has_table else None
        self.table_row = tensors[-1].shape[1] if has_table else 0
        self.shapes = [tuple(t.shape) for t in tensors]
        self.ptrs = None

    def adopt(self, tensors) -> "_GradBucket":
        """Point the `.grad` of `tensors` at the views, keeping the values they held."""
        for t, view in zip(tensors, self.views):
            if t.grad is not None:
                view.copy_(t.grad)
            t.grad = view
        self.ptrs = _grad_ptrs(tensors)
        return self

    def prefix(self, n_used: int) -> int:
        """Floats up to the end of voxel-table row n_used (all of them without a table): the only ones a step can write
        when the index map references rows [0, n_used)."""
        return self.flat.numel() if self.table_offset is None else self.table_offset + self.table_row * n_used


class _StepPlan:
    """Every buffer one configuration of the step needs, allocated once."""

    def __init__(self, models, emb_xyz, n, cfg, rand, dev, seed):
        lib = _lib.load()
        self.n, self.dev, self.cfg = n, dev, cfg
        self.bucket = None              # _GradBucket of a plan made with a process group
        self.sink = None                # _GradBucket of a plan made with grad_sink=True
        # table rows the sink may hold gradient in (the most the grid has referenced) and the grid they were counted on
        self.sink_rows, self.sink_grid = 0, None
        # the device seed of captured steps (onerf_train_step_dseed), continuing from the creating call's host seed
        self.seed_dev = torch.full((1,), seed + 4, dtype=torch.int64, device=dev)
        self.model_order = ["coarse"] + (["fine"] if cfg["N_importance"] > 0 else [])
        self.use_voxel = _is_voxel(emb_xyz)
        f = lambda *shape, dtype=torch.float32: torch.empty(*shape, dtype=dtype, device=dev)
        self.rays, self.ids, self.codes, self.d_codes = f(n, 8), f(n, dtype=torch.int64), f(n, 64), f(n, 64)
        self.rgbs, self.depths, self.weight = f(n, 3), f(n), f(n)
        self.valid, self.inst, self.ptm = (f(n, dtype=torch.uint8) for _ in range(3))
        self.out, self.present, self.psnr = f(1 + len(TERMS)), f(len(TERMS), dtype=torch.int32), f(1)
        self.packed = _packed_blobs(models, self.model_order, self.use_voxel, dev)
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
        fill_loss_args(la, cfg["loss_weights"], self.out, self.present)
        self.loss_args = la


def _packed_blobs(models, model_order, use_voxel, dev) -> dict:
    """One packed-weights blob per model of a plan, filled by every call (a captured graph replays their addresses)."""
    nbytes = _lib.load().onerf_packed_weights_bytes(int(use_voxel))
    for typ in model_order:
        engine.check_architecture(models[typ], use_voxel)
    return {typ: engine.aligned_bytes(nbytes, dev) for typ in model_order}


def _pack(models, typ, use_voxel, packed) -> list:
    """Re-pack model `typ`'s current weights into the plan's blob; returns its (W, b) pairs."""
    lin = [(_f32_param(w), _f32_param(b)) for w, b in engine.model_linears(models[typ])]
    engine.pack_weights(lin, use_voxel, out=packed[typ])
    return lin


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


def sync_replicas(models: Dict[str, Any], embeddings: Dict[str, Any], code_library, group) -> None:
    """Make every rank's replica rank 0's: broadcast the parameters of `models`, `embeddings` and `code_library` and the
    voxel grid's buffers (GRID_BUFFERS; a rank whose index map has another shape gets new buffers of rank 0's shape), then
    count the table rows the index map references (one host read).  The eager counterpart of DDP's construction-time
    broadcast and broadcast_buffers: call it before the first train_step(group=...) and after every grid maintenance,
    before recapturing."""
    import torch.distributed as dist

    def bcast(t):
        dist.broadcast(t.view(torch.uint8) if t.dtype == torch.bool else t, group_src=0, group=group)

    emb = embeddings["xyz"]
    use_voxel = _is_voxel(emb)
    n_used = 0
    with torch.no_grad():
        if use_voxel:
            bcast(emb.voxel_shape)
            shape = tuple(int(v) for v in emb.voxel_shape.tolist())
            for name in ("voxel_idx_map", "voxel_occupancy"):
                t = getattr(emb, name, None)
                if t is not None and tuple(t.shape) != shape:
                    setattr(emb, name, torch.empty(shape, dtype=t.dtype, device=t.device))
            for name in GRID_BUFFERS[1:]:
                if getattr(emb, name, None) is not None:
                    bcast(getattr(emb, name))
        seen = set()
        for m in list(models.values()) + list(embeddings.values()) + [code_library]:
            for p in m.parameters() if m is not None else ():
                if id(p) not in seen:
                    seen.add(id(p))
                    bcast(p.detach())
        if use_voxel:
            n_used = _rows_used(emb)
    _synced[models["coarse"]] = (_grid_stamp(emb) if use_voxel else None, n_used)


def _rows_used(emb) -> int:
    """Voxel-table rows the index map references, [0, n_used): the only rows a step can write gradient to (one host
    read)."""
    m = emb.voxel_idx_map
    return min(int(m.max().item()) + 1, emb.embedding_space_ftr.weight.shape[0]) if m.numel() else 0


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
               frustum_bound_th: float = 0, pass_through_mask=None, rays_in_bbox: bool = False, group=None,
               grad_sink: bool = False, **render_kwargs):
    """render_rays(models, embeddings, batch["rays"], ...) with the codes code_library(batch) looks up, then
    TotalLoss(loss_conf) and its backward, as one call.  Takes render_rays' keyword arguments (train.py:84-98, 155-165;
    is_eval, use_zero_as_last_delta, precision and _rand included, the rest ignored as render_rays ignores them).
    group: a torch.distributed process group; the gradients are then averaged over its ranks (module docstring).
    grad_sink: write the gradients into an fp32 bucket the plan owns instead of `.grad` (which stays untouched), and
    return them (TrainStepFn hands them to autograd).  The call zeroes the bucket first (with the voxel model only up
    to the last table row the grid has referenced; the rows above were never written).

    Returns (loss_sum, terms, present, psnr) as device tensors: loss_sum (), the five unweighted terms (5,) in
    losses.TERMS order (0 where skipped), present (5,) int32 flags (TotalLoss's loss_dict holds term i iff present[i]),
    and the PSNR of the fine pass's rgb (coarse without a fine pass) over the valid rays (train.py:171-172).  With
    grad_sink a fifth element follows: the gradients as views of the bucket, one per tensor of _trained_tensors (fine
    model first, then coarse, each in engine.model_linears order with weight before bias; the code table; the voxel
    table), overwritten by the next call of the same plan."""
    if not forward_instance:
        raise NotImplementedError("TotalLoss needs the object branch's maps: train_step runs with forward_instance=True")
    if grad_sink and group is not None:
        raise ValueError("train_step: grad_sink returns the gradients for the caller to reduce (DDP does it through "
                         "autograd); group= reduces .grad itself: choose one")
    rays = batch["rays"].reshape(-1, 8)
    dev = rays.device
    n = rays.shape[0]
    emb_xyz = embeddings["xyz"]
    rand = render_kwargs.get("_rand") or {}
    cfg = dict(N_samples=int(N_samples), N_importance=int(N_importance), use_disp=bool(use_disp), perturb=float(perturb),
               noise_std=float(noise_std), white_back=bool(white_back), is_eval=bool(render_kwargs.get("is_eval", False)),
               zero_last_delta=bool(render_kwargs.get("use_zero_as_last_delta", False)),
               rays_in_bbox=bool(rays_in_bbox), frustum_bound_th=float(frustum_bound_th),
               has_ptm=pass_through_mask is not None, precision=engine.train_precision(render_kwargs.get("precision")),
               loss_weights=tuple(float(loss_conf[f"{t}_weight"]) for t in TERMS))
    use_voxel = _is_voxel(emb_xyz)
    table = emb_xyz.embedding_space_ftr.weight if use_voxel else None
    key = (dev, n, use_voxel, tuple(sorted(cfg.items())),
           tuple(rand[k].data_ptr() if rand.get(k) is not None else 0 for k in _RAND_KEYS), group, bool(grad_sink))
    capturing = _capturing(dev)
    seed = engine.new_seed() if not capturing and (cfg["perturb"] > 0 or cfg["noise_std"] > 0) else 0
    code_table = code_library.embedding_instance.weight
    if group is not None:
        import torch.distributed as dist
        synced = _synced.get(models["coarse"])
        if synced is None:
            raise RuntimeError("train_step(group=...): call training.sync_replicas(models, embeddings, code_library, "
                               "group) before the first step, so that every rank starts from rank 0's replica")
        if use_voxel and synced[0] != _grid_stamp(emb_xyz):
            raise RuntimeError("train_step(group=...): the voxel grid changed since the last sync_replicas (grid "
                               "maintenance); call training.sync_replicas again, then recapture")
        world = dist.get_world_size(group)
        seed = (seed + dist.get_rank(group) * RANK_SEED_STRIDE) % (1 << 62)
    plans = _plans.setdefault(models["coarse"], {})
    plan = plans.get(key)
    made = plan is None
    if made:
        if capturing:
            raise RuntimeError("train_step: the first call for a configuration must run before the CUDA-graph capture "
                               "(warm up eagerly): its plan's device seed counter would be reset on every replay")
        plan = _StepPlan(models, emb_xyz, n, cfg, rand, dev, seed)
    trained = _trained_tensors(models, plan.model_order, code_table, table)
    if made:
        if group is not None:
            ptrs = _grad_ptrs(trained)
            # another configuration's bucket, if the gradients still view it
            plan.bucket = next((p.bucket for p in plans.values() if p.bucket is not None and p.bucket.ptrs == ptrs),
                               None) or _GradBucket(trained, table is not None, dev).adopt(trained)
        if grad_sink:
            plan.sink = _GradBucket(trained, table is not None, dev)
        plans[key] = plan
    if group is not None and _grad_ptrs(trained) != plan.bucket.ptrs:
        raise RuntimeError("train_step(group=...): a .grad no longer views the gradient bucket this step all-reduces "
                           "(zero_grad(set_to_none=True) or a replaced parameter?); zero the gradients with "
                           "set_to_none=False")
    if grad_sink:
        if [tuple(t.shape) for t in trained] != plan.sink.shapes:
            raise RuntimeError("train_step(grad_sink=True): a trained tensor changed shape since this configuration's "
                               "first call")
        if use_voxel and plan.sink_grid != _grid_stamp(emb_xyz):
            # one host read after each grid change; pruning can lower n_used, so keep the most rows ever referenced
            plan.sink_rows, plan.sink_grid = max(plan.sink_rows, _rows_used(emb_xyz)), _grid_stamp(emb_xyz)
        plan.sink.flat[:plan.sink.prefix(plan.sink_rows)].zero_()
        grads = plan.sink.views
    else:
        grads = [_grad_of(t) for t in trained]
    first = {typ: 40 * k for k, typ in enumerate(reversed(plan.model_order))}     # grads: fine model first
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
    _lib.call("onerf_code_gather", dev, _f32_param(code_table).data_ptr(), plan.ids.data_ptr(), n, code_table.shape[0],
              plan.codes.data_ptr())
    b = _lib.RenderBwdArgs()
    for typ in plan.model_order:
        g = grads[first[typ]:first[typ] + 40]
        setattr(b, "W_" + typ, engine.pointer_tables(_pack(models, typ, plan.use_voxel, plan.packed))[0])
        dW, db = engine.pointer_tables(zip(g[0::2], g[1::2]))
        setattr(b, "dW_" + typ, dW)
        setattr(b, "db_" + typ, db)
    b.d_codes = plan.d_codes.data_ptr()
    b.table_grad = grads[-1].data_ptr() if table is not None else None
    a = plan.render.args
    if capturing:
        _lib.call("onerf_train_step_dseed", dev, C.byref(a), C.byref(plan.loss_args), C.byref(b), plan.psnr.data_ptr(),
                  plan.seed_dev.data_ptr())
    else:
        a.seed = seed
        _lib.call("onerf_train_step", dev, C.byref(a), C.byref(plan.loss_args), C.byref(b), plan.psnr.data_ptr())
    _lib.call("onerf_code_scatter_add", dev, plan.d_codes.data_ptr(), plan.ids.data_ptr(), n, code_table.shape[0],
              grads[40 * len(plan.model_order)].data_ptr())
    if group is not None:
        reduced = plan.bucket.flat[:plan.bucket.prefix(synced[1])]
        dist.all_reduce(reduced, op=dist.ReduceOp.SUM, group=group)     # gloo has no AVG
        reduced.mul_(1.0 / world)
    if grad_sink:
        return plan.out[0], plan.out[1:], plan.present, plan.psnr[0], grads
    return plan.out[0], plan.out[1:], plan.present, plan.psnr[0]


class TrainStepFn(torch.autograd.Function):
    """train_step as an autograd node, for host loops that own the backward (Lightning, DDP, GradScaler, gradient
    accumulation).  The inputs are the trained tensors in _trained_tensors order; forward runs the whole step into the
    plan's gradient sink (train_step(grad_sink=True)), so `.grad` is only written by autograd, through AccumulateGrad,
    where DDP's reducer hooks fire.  Returns (loss_sum, terms, present, psnr) as fresh tensors; only loss_sum is
    differentiable.  backward returns each sink gradient times grad_output as a new tensor (never a view of the sink:
    autograd may adopt a returned gradient as `.grad`, and the next step would overwrite it), so `(loss / N).backward()`
    and a GradScaler's scaled loss come out right.  Run backward before the next step of the same configuration: that
    step zeroes the sink, and a backward after it is refused.  Call through `run`."""

    @staticmethod
    def forward(ctx, step, *trained):
        models, embeddings, code_library, batch, loss_conf, kwargs = step
        loss_sum, terms, present, psnr, grads = train_step(models, embeddings, code_library, batch, loss_conf,
                                                           grad_sink=True, **kwargs)
        ctx.grads = grads
        ctx.sink_version = grads[0]._version if grads else None      # the views share the sink's version counter
        out = loss_sum.clone(), terms.clone(), present.clone(), psnr.clone()
        ctx.mark_non_differentiable(*out[1:])
        return out

    @staticmethod
    def backward(ctx, g_loss, *_):
        if ctx.grads and ctx.grads[0]._version != ctx.sink_version:
            raise RuntimeError("TrainStepFn: a later step of the same configuration has overwritten this step's "
                               "gradients; run backward before the next step")
        return (None,) + tuple(g * g_loss for g in ctx.grads)

    @classmethod
    def run(cls, models: Dict[str, Any], embeddings: Dict[str, Any], code_library, batch: Dict[str, torch.Tensor],
            loss_conf, **kwargs):
        """train_step(models, embeddings, code_library, batch, loss_conf, **kwargs) through autograd (group= is not
        taken: DDP reduces the gradients).  Refused when grad mode is off or no trained tensor requires grad: the
        step's backward would have nowhere to go."""
        emb_xyz = embeddings["xyz"]
        model_order = ["coarse"] + (["fine"] if int(kwargs.get("N_importance", 0)) > 0 else [])
        trained = _trained_tensors(models, model_order, code_library.embedding_instance.weight,
                                   emb_xyz.embedding_space_ftr.weight if _is_voxel(emb_xyz) else None)
        if not torch.is_grad_enabled():
            raise RuntimeError("TrainStepFn: grad mode is off (torch.no_grad() / inference_mode); the step exists for "
                               "its gradients: call training.train_step for a step that writes .grad directly")
        if not any(t.requires_grad for t in trained):
            raise RuntimeError("TrainStepFn: no trained tensor (model linears, code table, voxel table) requires grad")
        return cls.apply((models, embeddings, code_library, batch, loss_conf, kwargs), *trained)


def install_training(system_cls, *, precision=None):
    """Replace `training_step` of `system_cls` (the reference's ObjectNeRFSystem, train.py:147-180) by one that runs the
    step through TrainStepFn with the arguments the reference passes to render_rays: is_eval=False, the batch's
    pass_through_mask, rays_in_bbox from train_dataset.is_rays_in_bbox(), frustum_bound_th = config.model.frustum_bound
    / config.dataset_extra.scale_factor, N_samples, N_importance, use_disp, perturb and noise_std from config.model,
    white_back from train_dataset, and the codes of the batch's instance ids.  It makes the same `self.log` calls (lr,
    train/loss, train/<term> for each present term, train/psnr) and returns loss_sum, whose backward hands the step's
    gradients to autograd (and so to Lightning's gradient accumulation, AMP scaling and DDP).  Leaving absent terms out
    of the log needs the five flags on the host: one 20-byte read per step, the only one.  Grid maintenance in
    on_epoch_start needs nothing: each step reads the current grid.
    precision: the step's arithmetic (None = the library default)."""
    import sys
    get_learning_rate = sys.modules[system_cls.__module__].get_learning_rate      # train.py's own import

    def training_step(self, batch, batch_nb):
        conf, m = self.config, self.config.model
        loss_sum, terms, present, psnr = TrainStepFn.run(
            self.models, self.embeddings, self.code_library, batch, conf.loss, N_samples=m.N_samples,
            use_disp=m.use_disp, perturb=m.perturb, noise_std=m.noise_std, N_importance=m.N_importance,
            white_back=self.train_dataset.white_back, is_eval=False, pass_through_mask=batch["pass_through_mask"],
            rays_in_bbox=getattr(self.train_dataset, "is_rays_in_bbox", lambda: False)(),
            frustum_bound_th=m.frustum_bound / conf["dataset_extra"]["scale_factor"], precision=precision)
        flags = present.tolist()
        self.log("lr", get_learning_rate(self.optimizer))
        self.log("train/loss", loss_sum)
        for i, t in enumerate(TERMS):
            if flags[i]:
                self.log(f"train/{t}", terms[i])
        self.log("train/psnr", psnr, prog_bar=True)
        return loss_sum

    system_cls.training_step = training_step
    return system_cls


# ------------------------------------------------------------------------------------------------
# validation
# ------------------------------------------------------------------------------------------------
# what utils/train_helper.visualize_val_image reads of the last pass
VAL_KEYS = ("rgb", "depth", "rgb_instance", "depth_instance", "opacity_instance")
_VAL_WIDTHS = {"opacity": 1, "rgb": 3, "depth": 1, "rgb_instance": 3, "depth_instance": 1, "opacity_instance": 1}
_val_plans: "weakref.WeakKeyDictionary[Any, Dict[tuple, _ValPlan]]" = weakref.WeakKeyDictionary()


class _ValPlan:
    """Every buffer one configuration of validate_frame owns: the record, the outputs, the packed weights, the tile's
    maps and, for a batch without instance_mask, the all-zero mask and weight."""

    def __init__(self, models, n, tile, cfg, keys, dev, use_voxel):
        self.model_order = ["coarse"] + (["fine"] if cfg["N_importance"] > 0 else [])
        self.typ = self.model_order[-1]
        f = lambda *shape, dtype=torch.float32: torch.empty(*shape, dtype=dtype, device=dev)
        self.record = torch.zeros(_lib.VALIDATE_RECORD_DOUBLES, dtype=torch.float64, device=dev)
        self.out, self.present, self.psnr = f(1 + len(TERMS)), f(len(TERMS), dtype=torch.int32), f(1)
        self.no_inst = self.no_weight = None
        if not cfg["has_instance_mask"]:
            self.no_inst = torch.zeros(n, dtype=torch.uint8, device=dev)
            self.no_weight = torch.zeros(n, dtype=torch.float32, device=dev)
        self.packed = _packed_blobs(models, self.model_order, use_voxel, dev)
        self.maps = {f"{k}_{self.typ}": f(tile, 3) if _VAL_WIDTHS[k] == 3 else f(tile) for k in keys}
        self.weights = (C.c_float * len(TERMS))(*cfg["loss_weights"])
        a = self.args = _lib.ValidateArgs()
        r, la = a.render, a.loss
        r.n_rays, r.n_samples, r.n_importance = n, cfg["N_samples"], cfg["N_importance"]
        r.precision = engine.PRECISIONS[cfg["precision"]]
        r.use_disp, r.white_back, r.rays_in_bbox = int(cfg["use_disp"]), int(cfg["white_back"]), int(cfg["rays_in_bbox"])
        r.forward_instance, r.is_eval = 1, 1
        r.packed_coarse = self.packed["coarse"].data_ptr()
        r.packed_fine = self.packed["fine"].data_ptr() if "fine" in self.packed else None
        for k in keys:
            setattr(getattr(r, self.typ), k, self.maps[f"{k}_{self.typ}"].data_ptr())
        la.n_rays, la.has_fine = n, int(self.typ == "fine")
        fill_loss_args(la, cfg["loss_weights"], self.out, self.present)
        a.chunk_rays = cfg["chunk"]
        a.psnr_mask = _lib.PSNR_VALID_INSTANCE if cfg["has_instance_mask"] else _lib.PSNR_ALL_RAYS
        a.record, a.psnr_out = self.record.data_ptr(), self.psnr.data_ptr()


def _batch_rows(t: torch.Tensor, n: int, width: int, dtype) -> torch.Tensor:
    """batch[key] with the loader's leading dimension of 1 dropped, in the kernels' type; the tensor itself when it has
    that type already."""
    t = t.reshape((n, width) if width > 1 else (n,))
    if t.dtype == torch.bool and dtype == torch.uint8:
        t = t.view(torch.uint8)
    return t.to(dtype).contiguous()


def validate_frame(models: Dict[str, Any], embeddings: Dict[str, Any], code_library, batch: Dict[str, torch.Tensor],
                   loss_conf, *, N_samples: int, N_importance: int, use_disp: bool, white_back: bool,
                   rays_in_bbox: bool = False, chunk: int = 65536, keys=VAL_KEYS, precision: str = "bf16", group=None):
    """One validation image as train.py's validation_step computes it (train.py:182-223): render_rays over batch["rays"]
    with is_eval=True and the codes of batch["instance_ids"], TotalLoss(loss_conf) on the maps and the PSNR of the last
    pass's rgb, as one library call.  `batch` is what val_dataloader yields (leading dimension 1; the first 8 ray columns
    are used).  The PSNR averages over valid_mask * instance_mask, or over every ray when the batch has no
    instance_mask; such a batch is taken as one without instance pixels (mask and weight 0).

    Returns {"loss_sum": (), "terms": (5,) unweighted in losses.TERMS order (0 where skipped), "present": (5,) int32,
    "psnr": ()} plus, for every k in `keys` (of opacity, rgb, depth, rgb_instance, depth_instance, opacity_instance),
    the image-sized map f"{k}_fine" (f"{k}_coarse" without a fine pass), all on the device.  The default keys are what
    utils/train_helper.visualize_val_image reads.  group: see the module docstring."""
    keys = tuple(keys)
    unknown = [k for k in keys if k not in _VAL_WIDTHS]
    if unknown:
        raise KeyError(f"validate_frame: no such map {unknown} (choose from {sorted(_VAL_WIDTHS)})")
    if int(chunk) < 1:
        raise ValueError("validate_frame: chunk must be at least 1 ray")
    rays = batch["rays"]
    if rays.shape[-1] < 8:
        raise ValueError(f"validate_frame: rays need 8 columns (o, d, near, far), got {rays.shape[-1]}")
    rays = rays.reshape(-1, rays.shape[-1])[:, :8]
    n, dev = rays.shape[0], rays.device
    emb_xyz = embeddings["xyz"]
    use_voxel = _is_voxel(emb_xyz)
    has_mask = "instance_mask" in batch
    cfg = dict(N_samples=int(N_samples), N_importance=int(N_importance), use_disp=bool(use_disp),
               white_back=bool(white_back), rays_in_bbox=bool(rays_in_bbox), chunk=int(chunk),
               precision=engine.train_precision(precision), has_instance_mask=has_mask,
               loss_weights=tuple(float(loss_conf[f"{t}_weight"]) for t in TERMS))
    begin, end = parallel.tile_bounds(n, group)
    key = (dev, n, begin, end, use_voxel, tuple(sorted(cfg.items())), keys)
    plan = engine.cached_plan(_val_plans, models["coarse"], key,
                              lambda: _ValPlan(models, n, end - begin, cfg, keys, dev, use_voxel))
    a = plan.args
    code_table = _f32_param(code_library.embedding_instance.weight)
    # what the call reads, alive until it has been enqueued (a captured call reads the same tensors on every replay)
    held = [_batch_rows(rays, n, 8, torch.float32), _batch_rows(batch["rgbs"], n, 3, torch.float32),
            _batch_rows(batch["depths"], n, 1, torch.float32), _batch_rows(batch["valid_mask"], n, 1, torch.uint8),
            _batch_rows(batch["instance_mask"], n, 1, torch.uint8) if has_mask else plan.no_inst,
            _batch_rows(batch["instance_mask_weight"], n, 1, torch.float32) if has_mask else plan.no_weight,
            _batch_rows(batch["instance_ids"], n, 1, torch.int64)]
    (a.render.rays, a.loss.rgbs, a.loss.depths, a.loss.valid_mask, a.loss.instance_mask, a.loss.instance_mask_weight,
     a.instance_ids) = (t.data_ptr() for t in held)
    a.code_table, a.n_codes = code_table.data_ptr(), code_table.shape[0]
    grid = engine.GridBuffers.from_module(emb_xyz) if use_voxel else None
    a.render.grid = C.pointer(grid.c) if use_voxel else None
    a.ray_begin, a.ray_end, a.finalize = begin, end, int(group is None)
    ws = engine.workspace(_lib.load().onerf_validate_workspace_bytes(cfg["chunk"], cfg["N_samples"], cfg["N_importance"]),
                          dev)
    a.render.workspace, a.render.workspace_bytes = ws.data_ptr(), ws.numel()
    for typ in plan.model_order:
        _pack(models, typ, use_voxel, plan.packed)
    _lib.call("onerf_validate_frame", dev, C.byref(a))
    maps = dict(plan.maps)
    if group is not None:
        import torch.distributed as dist
        dist.all_reduce(plan.record, op=dist.ReduceOp.SUM, group=group)
        _lib.call("onerf_validate_finalize", dev, plan.record.data_ptr(), plan.weights, a.loss.has_fine,
                  plan.out.data_ptr(), plan.out[1:].data_ptr(), plan.present.data_ptr(), plan.psnr.data_ptr())
        maps = parallel.gather_tile_maps(maps, n, group)
    return {"loss_sum": plan.out[0], "terms": plan.out[1:], "present": plan.present, "psnr": plan.psnr[0], **maps}


def install_validation(system_cls, *, chunk: int = 65536, group=None):
    """Replace `validation_step` of `system_cls` (the reference's ObjectNeRFSystem, train.py:182-223) by one that runs
    validate_frame: the same `log` dict (val_loss, the present terms under the reference's names, val_psnr), the same
    `self.log("val/...")` calls, and visualize_val_image for the first image.  The image renders without jitter and
    sigma noise whatever config.model.perturb / noise_std say.  Leaving absent terms out of the dict needs the five
    flags on the host: one 20-byte read per image, the only one.  The logged values are copies (validation_epoch_end
    stacks them over the images; validate_frame's own outputs are overwritten by the next image).
    chunk, group: as validate_frame."""
    import sys

    def validation_step(self, batch, batch_nb):
        conf = self.config
        res = validate_frame(self.models, self.embeddings, self.code_library, batch, conf.loss,
                             N_samples=conf.model.N_samples, N_importance=conf.model.N_importance,
                             use_disp=conf.model.use_disp, white_back=self.val_dataset.white_back,
                             rays_in_bbox=getattr(self.val_dataset, "is_rays_in_bbox", lambda: False)(),
                             chunk=chunk, group=group)
        flags = res["present"].tolist()
        terms = res["terms"].clone()
        loss_dict = {t: terms[i] for i, t in enumerate(TERMS) if flags[i]}
        for k, v in loss_dict.items():
            self.log(f"val/{k}", v)
        log = {"val_loss": res["loss_sum"].clone()}
        log.update(loss_dict)
        typ = "fine" if conf.model.N_importance > 0 else "coarse"
        if batch_nb == 0:
            visualize = sys.modules[system_cls.__module__].visualize_val_image
            stack_image = visualize(conf.img_wh, batch, res, typ=typ)
            self.logger.experiment.add_images("val/GT_pred_depth", stack_image, self.global_step)
        log["val_psnr"] = res["psnr"].clone()
        return log

    system_cls.validation_step = validation_step
    return system_cls
