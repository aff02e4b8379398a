"""Drop-in for the reference's `models/rendering.py` call surface: render_rays(), inference_model(),
sample_pdf() with identical signatures and result keys (reference models/rendering.py:11-17, 64-83,
233-250).  Every stage runs as a CUDA kernel of libonerf_sm100.so; there is no PyTorch or CPU
implementation behind these functions.

Extra keyword-only knobs (absorbed by **dummy_kwargs in the reference, so call sites stay valid):
  precision="bf16"|"fp32"   arithmetic of the fused encode+MLP kernel (default: env ONERF_PRECISION or bf16)
  _rand=dict(...)           test hook: pre-drawn random buffers (jitter, u, noise_*), see tests/synth.py
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Any, Dict, Optional, Sequence

import torch

from . import _lib, engine

__all__ = ["render_rays", "sample_pdf", "inference_model", "render_instances", "render_boxes"]


def _is_voxel(embedding_xyz) -> bool:
    return hasattr(embedding_xyz, "voxel_idx_map")


def _grid_of(embedding_xyz):
    return engine.GridBuffers.from_module(embedding_xyz) if _is_voxel(embedding_xyz) else None


def _store_pass(results: Dict[str, Any], typ: str, out: Dict[str, torch.Tensor], z_vals, forward_instance: bool):
    """One pass's maps into the result dict under the reference's keys (models/rendering.py:210-230)."""
    for k in ("weights", "opacity", "rgb", "depth") + (("rgb_instance", "depth_instance", "opacity_instance")
                                                          if forward_instance else ()):
        results[f"{k}_{typ}"] = out[k]
    results[f"z_vals_{typ}"] = z_vals


def _needs_grad(model, *tensors) -> bool:
    if not torch.is_grad_enabled():
        return False
    return any(p.requires_grad for p in model.parameters()) or any(
        t is not None and t.requires_grad for t in tensors)


def sample_pdf(bins, weights, N_importance, det=False, eps=1e-5, _u=None):
    """Reference models/rendering.py:11-61: draw N_importance depths from the piecewise-constant pdf
    `weights` (N, M) over `bins` (N, M+1).  eps is fixed at the reference default 1e-5 in the kernel."""
    if eps != 1e-5:
        raise RuntimeError("sample_pdf kernel is built with eps = 1e-5")
    seed = 0 if (det or _u is not None) else engine.new_seed()
    return engine.sample_pdf(bins, weights, N_importance, det, u=_u, seed=seed)


def inference_model(results: Dict[str, Any], model, embeddings: Dict[str, Any], typ: str, xyz, rays_d, z_vals,
                    chunk: int, noise_std: float, white_back: bool, is_eval: bool = False,
                    use_zero_as_last_delta: bool = False, forward_instance: bool = True,
                    embedding_instance: Optional[torch.Tensor] = None, frustum_bound_th: float = 0,
                    pass_through_mask: Optional[torch.Tensor] = None, rays_in_bbox: bool = False,
                    precision: Optional[str] = None, _rand: Optional[dict] = None, _rays=None, _seed=None,
                    **dummy_kwargs):
    """Encode + two-branch MLP + compositing for one pass; fills `results` in place with the reference's
    keys (models/rendering.py:64-230).  `chunk` is accepted and ignored: the kernels tile internally.
    Under grad (parameters, codes or the voxel table requiring it) the maps carry autograd to the model's Linear
    tensors, embedding_instance and the voxel table (field_query); weights_* and z_vals_* are non-differentiable and
    xyz, rays_d and z_vals get no gradient."""
    n, s = z_vals.shape
    emb_xyz = embeddings["xyz"]
    use_voxel = _is_voxel(emb_xyz)
    table = emb_xyz.embedding_space_ftr.weight if use_voxel else None
    if _needs_grad(model, embedding_instance if forward_instance else None, table):
        return _inference_model_grad(results, model, emb_xyz if use_voxel else None, typ, xyz, rays_d, z_vals,
                                     noise_std, white_back, is_eval, use_zero_as_last_delta, forward_instance,
                                     embedding_instance, frustum_bound_th, pass_through_mask, rays_in_bbox, precision,
                                     _rand, _rays, _seed)
    packed = engine.packed_for(model, use_voxel)
    grid = _grid_of(emb_xyz)
    if _rays is None:  # explicit-xyz call surface: only the direction columns of `rays` are used
        _rays = torch.zeros(n, 8, dtype=torch.float32, device=z_vals.device)
        _rays[:, 3:6] = rays_d.reshape(n, 3)
        xyz_arg = xyz
    else:
        xyz_arg = None
    z = z_vals.contiguous()
    scene, obj = engine.field(_rays, z, packed, grid, codes=embedding_instance if forward_instance else None,
                              want_scene=True, want_object=forward_instance, precision=precision, xyz=xyz_arg)
    rand = _rand or {}
    seed = _seed if _seed is not None else (engine.new_seed() if noise_std > 0 else 0)
    out = engine.composite(z, scene, obj, noise_std=noise_std, white_back=white_back, is_eval=is_eval,
                           zero_last_delta=use_zero_as_last_delta, rays_in_bbox=rays_in_bbox,
                           frustum_bound_th=frustum_bound_th, pass_through_mask=pass_through_mask,
                           noise_scene=rand.get(f"noise_scene_{typ}"), noise_obj=rand.get(f"noise_obj_{typ}"),
                           seed=seed)
    _store_pass(results, typ, out, z_vals, forward_instance)


def _inference_model_grad(results, model, grid_module, typ, xyz, rays_d, z_vals, noise_std, white_back, is_eval,
                          zero_last_delta, forward_instance, codes, frustum_bound_th, pass_through_mask, rays_in_bbox,
                          precision, _rand, _rays, _seed):
    from . import field_query
    n, s = z_vals.shape
    if any(t is not None and t.requires_grad for t in (xyz, rays_d, z_vals)):
        raise ValueError("inference_model() gives no gradient to xyz, rays_d or z_vals: detach them")
    if forward_instance and codes is None:
        raise ValueError("forward_instance needs embedding_instance")
    z = z_vals.detach().float().contiguous()
    if _rays is None:   # explicit positions: only the direction columns of the rays are read
        rays = torch.zeros(n, 8, dtype=torch.float32, device=z.device)
        rays[:, 3:6] = rays_d.detach().reshape(n, 3)
        pos = xyz.detach().float().reshape(n, s, 3).contiguous()
    else:
        rays, pos = _rays.detach().float().contiguous(), None
    reached = field_query.SCENE + (field_query.OBJECT if forward_instance else ())
    scene, obj = field_query.field_eval(model, grid_module, rays, z, pos, codes if forward_instance else None,
                                        forward_instance, engine.train_precision(precision), reached)
    rand = _rand or {}
    seed = _seed if _seed is not None else (engine.new_seed() if noise_std > 0 else 0)
    cfg = dict(noise_std=float(noise_std), white_back=white_back, is_eval=is_eval, zero_last_delta=zero_last_delta,
               rays_in_bbox=rays_in_bbox, frustum_bound_th=float(frustum_bound_th), pass_through_mask=pass_through_mask,
               noise_scene=rand.get(f"noise_scene_{typ}"), noise_obj=rand.get(f"noise_obj_{typ}"), seed=seed)
    out = dict(zip(field_query.CompositeFn.KEYS, field_query.CompositeFn.apply(cfg, z, scene, obj)))
    _store_pass(results, typ, out, z_vals, forward_instance)


def query_sigma(model, embedding_xyz, xyz: torch.Tensor, obj_code: Optional[torch.Tensor] = None,
                chunk: int = 1 << 22, precision: Optional[str] = None) -> torch.Tensor:
    """Density of the field at arbitrary points: the `sigma_only=True` consumers of the fused encode + MLP
    (SURVEY.md section 8f row 4).  Replaces, in one call per chunk, the loop body of tools/extract_mesh.py:83-109
    (`embedding_xyz(xyz)` then `nerf_fine.forward(..., sigma_only=True)["sigma"]`, or with `obj_id > 0`
    `forward_instance(..., sigma_only=True)["inst_sigma"]` fed by one code-library row) and the density query of
    EmbeddingVoxel.self_pruning_empty_voxels (models/embedding_helper.py:219-225).
    xyz (B,3); obj_code None -> scene sigma (models/nerf_model.py:108-112), else (64,) -> object sigma (:140-144).
    Returns raw sigma (B,) (no relu), fp32, on xyz's device."""
    use_voxel = _is_voxel(embedding_xyz)
    packed = engine.packed_for(model, use_voxel)
    grid = _grid_of(embedding_xyz)
    xyz = xyz.reshape(-1, 3).contiguous().float()
    out = torch.empty(xyz.shape[0], dtype=torch.float32, device=xyz.device)
    for i in range(0, xyz.shape[0], chunk):
        pts = xyz[i:i + chunk]
        n = pts.shape[0]
        rays = torch.zeros(n, 8, dtype=torch.float32, device=xyz.device)   # directions are irrelevant for sigma
        z = torch.zeros(n, 1, dtype=torch.float32, device=xyz.device)
        scene, obj = engine.field(rays, z, packed, grid, code_row=obj_code, want_scene=obj_code is None,
                                  want_object=obj_code is not None, precision=precision, xyz=pts.view(n, 1, 3))
        out[i:i + n] = (scene if obj_code is None else obj)[:, 0, 3]
    return out

def _render_forward(cfg, rays, codes):
    """The whole forward of render_rays on the CUDA kernels, staged through engine (inference)."""
    rand = cfg["rand"]
    perturb, noise_std = cfg["perturb"], cfg["noise_std"]
    fi = cfg["forward_instance"]
    emb_xyz = cfg["embeddings"]["xyz"]
    use_voxel = _is_voxel(emb_xyz)
    grid = _grid_of(emb_xyz)
    seed = engine.new_seed() if (perturb > 0 or noise_std > 0) else 0
    z = engine.sample_coarse(rays, cfg["N_samples"], cfg["use_disp"], perturb, rand.get("jitter"), seed)
    results: Dict[str, Any] = {}

    def one_pass(typ, z_vals, seed_off):
        model = cfg["models"][typ]
        packed = engine.packed_for(model, use_voxel)
        scene, obj = engine.field(rays, z_vals, packed, grid, codes=codes if fi else None, want_scene=True,
                                  want_object=fi, precision=cfg["precision"])
        out = engine.composite(z_vals, scene, obj, noise_std=noise_std, white_back=cfg["white_back"],
                               is_eval=cfg["is_eval"], zero_last_delta=cfg["zero_last_delta"],
                               rays_in_bbox=cfg["rays_in_bbox"], frustum_bound_th=cfg["frustum_bound_th"],
                               pass_through_mask=cfg["pass_through_mask"], noise_scene=rand.get(f"noise_scene_{typ}"),
                               noise_obj=rand.get(f"noise_obj_{typ}"), seed=seed + seed_off)
        _store_pass(results, typ, out, z_vals, fi)

    one_pass("coarse", z, 1)
    if cfg["N_importance"] > 0:
        z_fine = engine.sample_pdf_merge(z, results["weights_coarse"], cfg["N_importance"], det=(perturb == 0),
                                         u=rand.get("u"), seed=seed + 2)
        one_pass("fine", z_fine, 3)
    return results


def render_rays(models: Dict[str, Any], embeddings: Dict[str, Any], rays: torch.Tensor, N_samples: int = 64,
                use_disp: bool = False, perturb: float = 0, noise_std: float = 1, N_importance: int = 0,
                chunk: int = 1024 * 32, white_back: bool = False, forward_instance: bool = True,
                embedding_instance: Optional[torch.Tensor] = None, frustum_bound_th: float = 0,
                pass_through_mask: Optional[torch.Tensor] = None, rays_in_bbox: bool = False,
                **dummy_kwargs):
    """Reference models/rendering.py:233-337: stratified sampling -> coarse pass -> importance resampling
    -> fine pass.  rays (N,8) = [o, d, near, far]; returns the reference's result dict.  When parameters (or the
    object codes) require grad under torch.enable_grad(), the result carries autograd through backward.py."""
    rays = rays.contiguous().float()
    emb_xyz = embeddings["xyz"]
    cfg = dict(models=models, embeddings=embeddings, N_samples=N_samples, use_disp=use_disp, perturb=float(perturb),
               noise_std=float(noise_std), N_importance=N_importance, white_back=white_back,
               forward_instance=forward_instance, frustum_bound_th=float(frustum_bound_th),
               pass_through_mask=pass_through_mask, rays_in_bbox=rays_in_bbox,
               is_eval=bool(dummy_kwargs.get("is_eval", False)),
               zero_last_delta=bool(dummy_kwargs.get("use_zero_as_last_delta", False)),
               precision=dummy_kwargs.get("precision"), rand=dummy_kwargs.get("_rand") or {})
    codes = embedding_instance
    model_order = ["coarse"] + (["fine"] if N_importance > 0 else [])
    trainable = [p for typ in model_order for p in models[typ].parameters()]
    has_table = _is_voxel(emb_xyz)
    needs_grad = torch.is_grad_enabled() and (
        any(p.requires_grad for p in trainable) or (codes is not None and codes.requires_grad)
        or (has_table and emb_xyz.embedding_space_ftr.weight.requires_grad))
    if not needs_grad:
        return _render_forward(cfg, rays, codes)
    # Training.  rays_in_bbox only swaps which weights feed the (detached) importance sampling and the returned
    # weights_* (models/rendering.py:228-229, :307): the gradients are unaffected.
    from . import backward
    cfg["has_table"], cfg["model_order"] = has_table, model_order
    cfg["precision"] = engine.train_precision(cfg["precision"])
    params = ([emb_xyz.embedding_space_ftr.weight] if has_table else [])
    for typ in model_order:
        for w, b in engine.model_linears(models[typ]):
            params += [w, b]
    tensors = backward.RenderRaysFn.apply(cfg, rays, codes, *params)
    keys = sorted(_result_keys(model_order, forward_instance))
    return dict(zip(keys, tensors))


def _result_keys(model_order, forward_instance):
    base = ["weights", "opacity", "z_vals", "rgb", "depth"] + (
        ["rgb_instance", "depth_instance", "opacity_instance"] if forward_instance else [])
    return [f"{k}_{typ}" for typ in model_order for k in base]


def _fit_chunk(chunk: int, ws_bytes, budget: int) -> int:
    """The largest chunk <= `chunk` whose workspace ws_bytes(chunk) fits `budget` bytes, or 1."""
    while chunk > 1 and ws_bytes(chunk) > budget:
        chunk = max(1, min(chunk - 1, chunk * budget // ws_bytes(chunk)))
    return chunk


def _pass_maps(fn: str, keys: Sequence[str], names: Sequence[str], N_importance: int) -> tuple:
    """The distinct (map, pass) pairs `keys` ask for: a name of `names` for the last pass, or with a "_coarse" / "_fine"
    suffix for that pass."""
    last = "fine" if N_importance > 0 else "coarse"
    maps = []
    for key in keys:
        base, _, typ = key.rpartition("_")
        base, typ = (base, typ) if typ in ("coarse", "fine") else (key, last)
        if base not in names or (typ == "fine" and N_importance == 0):
            raise KeyError(f"{fn}: no such map {key!r} (choose from {names}, optionally with _coarse or _fine)")
        maps.append((base, typ))
    return tuple(dict.fromkeys(maps))


# ------------------------------------------------------------------------------------------------
# every object's maps in one render
# ------------------------------------------------------------------------------------------------
INSTANCE_KEYS = ("rgb", "depth", "opacity", "opacity_instance", "depth_instance", "rgb_instance")
# render_instances keeps its per-chunk workspace (the field rows of K codes) within this many bytes by shrinking chunk
INSTANCES_WORKSPACE_BUDGET = 1 << 30
_instance_plans: "weakref.WeakKeyDictionary[Any, Dict[tuple, _InstancesPlan]]" = weakref.WeakKeyDictionary()


def _instances_chunk(chunk: int, K: int, n_samples: int, n_importance: int) -> int:
    """The largest chunk <= `chunk` whose onerf_render_instances workspace fits INSTANCES_WORKSPACE_BUDGET, or 1."""
    ws = _lib.load().onerf_render_instances_workspace_bytes
    return _fit_chunk(chunk, lambda c: ws(c, K, n_samples, n_importance), INSTANCES_WORKSPACE_BUDGET)


class _InstancesPlan:
    """Every buffer one configuration of render_instances owns: the packed weights, the tile's maps and the argument
    block."""

    def __init__(self, models, n, tile, cfg, maps, ids, dev, use_voxel):
        from . import training
        self.model_order = ["coarse"] + (["fine"] if cfg["N_importance"] > 0 else [])
        self.packed = training._packed_blobs(models, self.model_order, use_voxel, dev)
        K = len(ids)
        widths = {"rgb": (3,), "depth": (), "opacity": (), "opacity_instance": (K,), "depth_instance": (K,),
                  "rgb_instance": (K, 3)}
        self.maps = {f"{k}_{typ}": torch.empty((tile,) + widths[k], dtype=torch.float32, device=dev) for k, typ in maps}
        self.ids = (C.c_int * K)(*ids)
        a = self.args = _lib.InstancesArgs()
        r = a.render
        r.n_rays, r.n_samples, r.n_importance = n, cfg["N_samples"], cfg["N_importance"]
        r.precision = engine.PRECISIONS[cfg["precision"]]
        r.use_disp, r.white_back, r.is_eval = int(cfg["use_disp"]), int(cfg["white_back"]), 1
        r.packed_coarse = self.packed["coarse"].data_ptr()
        r.packed_fine = self.packed["fine"].data_ptr() if "fine" in self.packed else None
        for k, typ in maps:
            setattr(getattr(a, typ), k, self.maps[f"{k}_{typ}"].data_ptr())
        a.ids_host, a.n_ids = C.cast(self.ids, C.POINTER(C.c_int)), K
        a.chunk_rays = _instances_chunk(cfg["chunk"], K, cfg["N_samples"], cfg["N_importance"])


def render_instances(models: Dict[str, Any], embeddings: Dict[str, Any], code_library, rays: torch.Tensor,
                     ids: Sequence[int], *, N_samples: int, N_importance: int, use_disp: bool, white_back: bool = False,
                     chunk: int = 65536, keys: Sequence[str] = INSTANCE_KEYS, precision: str = "bf16", group=None):
    """Every object's own maps of `rays` (N, 8) in one render (onerf_render_instances).  Not a reference function:
    it returns, for K = len(ids) object codes code_library rows ids[k] (1 <= K <= 64, repeats allowed), what the
    reference's render_rays(..., embedding_instance=code of ids[k] on every ray, forward_instance=True, is_eval=True,
    perturb=0, noise_std=0, rays_in_bbox=False) returns, in one pass: the samples, the scene branch and each sample's
    encoding, which do not depend on the code, are computed once, and only the object branch runs per code.
    Column k of each object map is bit for bit that render's map at the same precision, and the scene maps are its
    scene maps.

    keys: of INSTANCE_KEYS, for the last pass (f"{key}_fine", or f"{key}_coarse" without a fine pass); a key written
    f"{key}_coarse" (or "_fine") selects that pass, so both passes' maps can be asked for.  Only the branches the asked
    maps need run: a pass without an object map skips the object branch, the fine pass without a scene map the scene
    branch.  Returns {name: device tensor}: rgb (N, 3), depth and opacity (N,), opacity_instance and depth_instance
    (N, K), rgb_instance (N, K, 3).  The tensors belong to a plan cached per configuration and are overwritten by the
    next call with it.
    chunk: rays per kernel chunk, lowered so that the workspace stays within INSTANCES_WORKSPACE_BUDGET bytes.  The
    workspace is cached per (device, size) for the life of the process, as validate_frame's and render_frame's are, so
    that a captured call keeps valid addresses: each distinct (K, chunk, samples) configuration holds up to
    INSTANCES_WORKSPACE_BUDGET bytes (1 GiB) of device memory.  Lower the budget (or chunk) to hold less.
    group: a torch.distributed process group; rank r renders parallel.shard_bounds(N, W, r) and the maps are
    all-gathered, so every rank returns the whole of them."""
    from . import parallel, training
    ids = [int(i) for i in ids]
    K = len(ids)
    if not 1 <= K <= _lib.INSTANCES_MAX_CODES:
        raise ValueError(f"render_instances: 1 to {_lib.INSTANCES_MAX_CODES} object ids, got {K}")
    if int(chunk) < 1:
        raise ValueError("render_instances: chunk must be at least 1 ray")
    maps = _pass_maps("render_instances", keys, INSTANCE_KEYS, N_importance)
    rays = rays.reshape(-1, rays.shape[-1])[:, :8].float().contiguous()
    n, dev = rays.shape[0], rays.device
    emb_xyz = embeddings["xyz"]
    use_voxel = _is_voxel(emb_xyz)
    cfg = dict(N_samples=int(N_samples), N_importance=int(N_importance), use_disp=bool(use_disp),
               white_back=bool(white_back), chunk=int(chunk), precision=engine.train_precision(precision))
    begin, end = parallel.tile_bounds(n, group)
    key = (dev, n, begin, end, use_voxel, tuple(sorted(cfg.items())), maps, tuple(ids))
    plan = engine.cached_plan(_instance_plans, models["coarse"], key,
                              lambda: _InstancesPlan(models, n, end - begin, cfg, maps, ids, dev, use_voxel))
    a = plan.args
    code_table = training._f32_param(code_library.embedding_instance.weight)
    a.render.rays = rays.data_ptr()
    a.code_table, a.n_codes_table = code_table.data_ptr(), code_table.shape[0]
    grid = engine.GridBuffers.from_module(emb_xyz) if use_voxel else None
    a.render.grid = C.pointer(grid.c) if use_voxel else None
    a.ray_begin, a.ray_end = begin, end
    ws = engine.workspace(_lib.load().onerf_render_instances_workspace_bytes(a.chunk_rays, K, cfg["N_samples"],
                                                                            cfg["N_importance"]), dev)
    a.render.workspace, a.render.workspace_bytes = ws.data_ptr(), ws.numel()
    for typ in plan.model_order:
        training._pack(models, typ, use_voxel, plan.packed)
    if end > begin:                  # an empty tile renders nothing (and its rays may have no storage)
        _lib.call("onerf_render_instances", dev, C.byref(a))
    return parallel.gather_tile_maps(plan.maps, n, group)


# ------------------------------------------------------------------------------------------------
# every object inside its own box
# ------------------------------------------------------------------------------------------------
BOX_KEYS = ("opacity_instance", "depth_instance", "rgb_instance")
# render_boxes keeps its per-chunk workspace within this many bytes by shrinking chunk
BOXES_WORKSPACE_BUDGET = 1 << 30
_box_plans: "weakref.WeakKeyDictionary[Any, Dict[tuple, _BoxesPlan]]" = weakref.WeakKeyDictionary()


def _boxes_chunk(chunk: int, n_samples: int, n_importance: int) -> int:
    """The largest chunk <= `chunk` whose onerf_render_boxes workspace fits BOXES_WORKSPACE_BUDGET, or 1."""
    ws = _lib.load().onerf_render_boxes_workspace_bytes
    return _fit_chunk(chunk, lambda c: ws(c, n_samples, n_importance), BOXES_WORKSPACE_BUDGET)


class _BoxesPlan:
    """Every buffer one configuration of render_boxes owns: the packed weights, the tile's maps and hit mask, and the
    argument block with its host arrays."""

    def __init__(self, models, H, W, tile, cfg, maps, K, dev, use_voxel):
        from . import training
        self.model_order = ["coarse"] + (["fine"] if cfg["N_importance"] > 0 else [])
        self.packed = training._packed_blobs(models, self.model_order, use_voxel, dev)
        widths = {"opacity_instance": (K,), "depth_instance": (K,), "rgb_instance": (K, 3)}
        self.maps = {f"{k}_{typ}": torch.empty((tile,) + widths[k], dtype=torch.float32, device=dev) for k, typ in maps}
        self.hit = torch.empty(tile, K, dtype=torch.uint8, device=dev)
        self.ids, self.boxes, self.c2w = (C.c_int * K)(), (_lib.BoxHost * K)(), (C.c_float * 12)()
        a = self.args = _lib.RenderBoxesArgs()
        a.packed_coarse = self.packed["coarse"].data_ptr()
        a.packed_fine = self.packed["fine"].data_ptr() if "fine" in self.packed else None
        a.precision = engine.PRECISIONS[cfg["precision"]]
        a.n_samples, a.n_importance, a.use_disp = cfg["N_samples"], cfg["N_importance"], int(cfg["use_disp"])
        a.H, a.W = H, W
        a.c2w_host, a.boxes_host, a.n_boxes = self.c2w, self.boxes, K
        a.ids_host = C.cast(self.ids, C.POINTER(C.c_int))
        fields = {"opacity_instance": "opacity", "depth_instance": "depth", "rgb_instance": "rgb"}
        for k, typ in maps:
            setattr(getattr(a, typ), fields[k], self.maps[f"{k}_{typ}"].data_ptr())
        a.hit = self.hit.data_ptr()
        a.chunk_rays = _boxes_chunk(cfg["chunk"], cfg["N_samples"], cfg["N_importance"])


def render_boxes(models: Dict[str, Any], embeddings: Dict[str, Any], code_library, H: int, W: int, focal: float, c2w,
                 boxes: Sequence[Any], ids: Sequence[int], *, N_samples: int, N_importance: int, use_disp: bool,
                 scale_factor: float, near: float, far: float, chunk: int = 65536, keys: Sequence[str] = BOX_KEYS,
                 precision: str = "bf16", group=None):
    """Every object rendered inside its own box from one camera (onerf_render_boxes): the object evaluation of a
    dataset with use_bbox, where GenericDataset clips each test ray to the object's box (near = far = 0 where it misses)
    and renders with rays_in_bbox, so the object's own weights drive the importance samples.  Not a reference function.

    For K = len(boxes) boxes (1 <= K <= 64; objects with BBoxRayHelper's pose_avg, axis_align_mat and bbox_bounds, such
    as frames.read_boxes returns) with code_library rows ids[k] (repeats allowed), object k's rays are
    ray_utils.camera_rays(H, W, focal, c2w, near, far, scale_factor, box=boxes[k]) and hit_k its return_mask:
      - at a hit pixel, column k of each map is bit for bit the opacity_instance / depth_instance / rgb_instance of the
        evaluation render of those rays (render_rays / training.validate_frame with is_eval, forward_instance,
        rays_in_bbox=True, perturb=0, noise_std=0) with code ids[k] on every ray, at the same precision;
      - at a missed pixel it is opacity +0, depth +0, rgb 1.  The reference's render evaluates those rays at z = 0
        instead; its metrics exclude them anyway (instance_mask * bbox_mask).
    No scene branch runs, and the object branch runs only on the rows that hit their box, so the field work follows
    the pixels the boxes cover.

    keys: of BOX_KEYS, for the last pass, or with a "_coarse" / "_fine" suffix for that pass.  Returns {name: device
    tensor}: opacity_instance and depth_instance (H*W, K), rgb_instance (H*W, K, 3), and "hit" (H*W, K) bool.  The
    tensors belong to a plan cached per configuration and are overwritten by the next call with it.
    chunk: (object, pixel) rows per kernel chunk, lowered so that the workspace stays within BOXES_WORKSPACE_BUDGET
    bytes; the workspace depends on neither K nor the image and is cached per (device, size) for the life of the
    process, as render_instances' is.
    group: a torch.distributed process group; rank r renders the pixels parallel.shard_bounds(H*W, W, r) and the maps
    are all-gathered, so every rank returns the whole of them."""
    from . import parallel, ray_utils, training
    ids = [int(i) for i in ids]
    K = len(ids)
    if not 1 <= K <= _lib.BOXES_MAX or len(boxes) != K:
        raise ValueError(f"render_boxes: 1 to {_lib.BOXES_MAX} boxes, one id each; got {len(boxes)} boxes, {K} ids")
    if int(chunk) < 1:
        raise ValueError("render_boxes: chunk must be at least 1 row")
    maps = _pass_maps("render_boxes", keys, BOX_KEYS, N_importance)
    H, W = int(H), int(W)
    n = H * W
    table = training._f32_param(code_library.embedding_instance.weight)
    dev = table.device
    emb_xyz = embeddings["xyz"]
    use_voxel = _is_voxel(emb_xyz)
    cfg = dict(N_samples=int(N_samples), N_importance=int(N_importance), use_disp=bool(use_disp), chunk=int(chunk),
               precision=engine.train_precision(precision))
    begin, end = parallel.tile_bounds(n, group)
    key = (dev, H, W, begin, end, use_voxel, tuple(sorted(cfg.items())), maps, K)
    plan = engine.cached_plan(_box_plans, models["coarse"], key,
                              lambda: _BoxesPlan(models, H, W, end - begin, cfg, maps, K, dev, use_voxel))
    a = plan.args
    for k in range(K):
        plan.ids[k] = ids[k]
        plan.boxes[k] = ray_utils._box_host(boxes[k], 0.0)
    C.memmove(plan.c2w, ray_utils._c2w_host(c2w), C.sizeof(plan.c2w))
    a.focal, a.scale_factor, a.near, a.far = float(focal), float(scale_factor), float(near), float(far)
    a.code_table, a.n_codes_table = table.data_ptr(), table.shape[0]
    grid = engine.GridBuffers.from_module(emb_xyz) if use_voxel else None
    a.grid = C.pointer(grid.c) if use_voxel else None
    a.pixel_begin, a.pixel_end = begin, end
    ws = engine.workspace(_lib.load().onerf_render_boxes_workspace_bytes(a.chunk_rays, cfg["N_samples"],
                                                                        cfg["N_importance"]), dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    for typ in plan.model_order:
        training._pack(models, typ, use_voxel, plan.packed)
    if end > begin:
        _lib.call("onerf_render_boxes", dev, C.byref(a))
    out = parallel.gather_tile_maps(dict(plan.maps, hit=plan.hit), n, group)
    out["hit"] = out["hit"].bool()
    return out
