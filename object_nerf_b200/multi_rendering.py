"""Drop-in for the reference's `render_tools/multi_rendering.py`: render_rays_multi() with the same
signature and result keys (reference render_tools/multi_rendering.py:160-175), used unchanged by
EditableRenderer.scene_inference / render_edit (render_tools/editable_renderer.py:125-140, 272-287).

Per ray set (scene id 0 or an object id): coarse depths -> one-branch field kernel (scene branch for id 0
with the removed-object box mask evaluated on the device, object branch with a constant code row
otherwise; zero-length rays muted) -> joint stable depth sort + compositing across all sets -> per-set
importance resampling -> fine pass.  No host round trips inside (the reference's check_in_any_boxes
goes device -> numpy -> device per chunk, utils/bbox_utils.py:119-130,170).

Everything the reference's function accepts runs on the device: perturb > 0 (per-set importance u), noise_std > 0
(N(0,1) * noise_std added to the jointly sorted sigmas of each pass, the coarse noise reaching the fine depths through the
coarse weights) and 10-column ray sets (N,10) = [o, d, near, far, near_box, far_box], whose fine depths strictly inside
(near_box, far_box) become far_box after the sorted merge; 8- and 10-column sets may be mixed.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Dict, Optional

import numpy as np
import torch

from . import _lib, engine
from .rendering import _grid_of, _is_voxel


def boxes_to_tensor(background_skip_bbox, device) -> Optional[torch.Tensor]:
    """Fold each BBoxRayHelper's xyz -> box-frame transform and bounds (utils/bbox_utils.py:119-130,
    158-186 with bbox_enlarge = 0, as check_in_any_boxes is called from multi_rendering.py:240) into
    rows [A (9) | t (3) | lo (3) | hi (3)] with p_box = A p + t."""
    if not background_skip_bbox:
        return None
    rows = []
    for _, box in background_skip_bbox.items():
        sf = float(box.scale_factor)
        P = np.asarray(box.pose_avg, dtype=np.float64).reshape(4, 4)
        Ax = np.asarray(box.axis_align_mat, dtype=np.float64).reshape(4, 4)
        A = Ax[:3, :3] @ P[:3, :3] * sf
        t = Ax[:3, :3] @ P[:3, 3] + Ax[:3, 3]
        bounds = np.asarray(box.bbox_bounds, dtype=np.float64)
        rows.append(np.concatenate([A.reshape(-1), t, bounds[0], bounds[1]]))
    return torch.from_numpy(np.stack(rows).astype(np.float32)).to(device)


def render_rays_multi(models: Dict[str, Any], embeddings: Dict[str, Any], code_library, rays_list: list,
                      obj_instance_ids: list, N_samples: int = 64, use_disp: bool = False, perturb: float = 0,
                      noise_std: float = 0, N_importance: int = 0, chunk: int = 1024 * 32,
                      white_back: bool = False, background_skip_bbox: Dict[str, Any] = None,
                      precision: Optional[str] = None, _staged: bool = False, *, _rand: Optional[dict] = None):
    """Reference render_tools/multi_rendering.py:160-175.  The whole forward is ONE C call (onerf_render_multi_fwd_ext);
    `_staged=True` runs the same kernels stage by stage from Python (tests: both routes are bit-identical).

    A ray set is (N,8) [o, d, near, far] or (N,10) with the box interval (near_box, far_box) appended: that set's fine
    depths strictly inside the interval become far_box (multi_rendering.py:278-287).  noise_std adds N(0,1) * noise_std to
    the jointly sorted sigmas of each pass (:131-132).  Random draws come from one seed of engine.new_seed() (taken when
    perturb != 0 or noise_std != 0) unless `_rand` injects them: dict(u=[per set (N, N_importance) or None],
    noise_coarse=(N, n_sets * N_samples), noise_fine=(N, n_sets * (N_samples + N_importance))), the noise in sorted order
    as the reference's randn_like draws it.  u is used only with perturb != 0, the noise only with noise_std != 0."""
    assert len(rays_list) == len(obj_instance_ids)
    emb_xyz = embeddings["xyz"]
    if not _is_voxel(emb_xyz):
        raise RuntimeError("render_rays_multi requires the voxel embedding, as the reference does "
                           "(render_tools/multi_rendering.py:55 unpacks a tuple)")
    if any(r.dim() != 2 or r.shape[1] not in (8, 10) for r in rays_list):
        raise ValueError("each ray set is (N,8) [o, d, near, far] or (N,10) with (near_box, far_box) appended")
    if not (np.isfinite(noise_std) and noise_std >= 0):
        raise ValueError(f"noise_std must be finite and >= 0, got {noise_std}")
    grid = _grid_of(emb_xyz)
    dev = rays_list[0].device
    n_obj, n, s = len(rays_list), rays_list[0].shape[0], N_samples
    clips = [r[:, 8:10].contiguous().float() if r.shape[1] == 10 else None for r in rays_list]
    rays_list = [r[:, :8].contiguous().float() for r in rays_list]
    rand = _check_rand(_rand or {}, n_obj, n, N_samples, N_importance, dev)
    u_list = rand.get("u") if (perturb != 0 and N_importance > 0) else None
    noise_c = rand.get("noise_coarse") if noise_std != 0 else None
    noise_f = rand.get("noise_fine") if (noise_std != 0 and N_importance > 0) else None
    seed = engine.new_seed() if (perturb != 0 or noise_std != 0) else 0
    boxes = boxes_to_tensor(background_skip_bbox, dev)
    code_table = engine._f32(code_library.embedding_instance.weight.detach())
    if not _staged:
        return _render_multi_one_call(models, grid, code_table, rays_list, [int(i) for i in obj_instance_ids], N_samples,
                                      use_disp, perturb, N_importance, white_back, boxes, precision, noise_std, seed,
                                      clips, u_list, noise_c, noise_f)

    def eval_pass(model, z_all):
        packed = engine.packed_for(model, True)
        s_ = z_all.shape[2]
        field_all = torch.empty(n_obj, n, s_, 4, dtype=torch.float32, device=dev)
        for i, iid in enumerate(obj_instance_ids):
            is_obj = iid > 0
            engine.field(rays_list[i], z_all[i], packed, grid, code_row=code_table[iid] if is_obj else None,
                         want_scene=not is_obj, want_object=is_obj, precision=precision, mute_zero_rays=True,
                         boxes=None if is_obj else boxes,
                         scene_out=None if is_obj else field_all[i], obj_out=field_all[i] if is_obj else None)
        return field_all

    results: Dict[str, Any] = {}
    with torch.no_grad():
        z_all = torch.empty(n_obj, n, s, dtype=torch.float32, device=dev)
        for i in range(n_obj):
            engine.sample_coarse(rays_list[i], s, use_disp, 0.0, out=z_all[i])
        out = engine.composite_multi(z_all, eval_pass(models["coarse"], z_all), white_back, want_ids=True,
                                     want_unsorted=N_importance > 0, noise_std=noise_std, noise=noise_c, seed=seed)
        for k in ("weights", "opacity", "z_vals", "rgb", "depth"):
            results[f"{k}_coarse"] = out[k]
        results["obj_ids_coarse"] = out["obj_ids"]
        if N_importance > 0:
            z_fine = torch.empty(n_obj, n, s + N_importance, dtype=torch.float32, device=dev)
            det = (perturb == 0)
            for i in range(n_obj):
                engine.sample_pdf_merge(z_all[i], out["weights_unsorted"][i], N_importance, det,
                                        u=u_list[i] if u_list is not None else None, seed=0 if det else seed + i,
                                        out=z_fine[i], clip=clips[i])
            out = engine.composite_multi(z_fine, eval_pass(models["fine"], z_fine), white_back, noise_std=noise_std,
                                         noise=noise_f, seed=seed, fine=True)
            for k in ("weights", "opacity", "z_vals", "rgb", "depth"):
                results[f"{k}_fine"] = out[k]
    return results


def _check_rand(rand: dict, n_obj: int, n: int, n_samples: int, n_importance: int, dev) -> dict:
    """`_rand` of render_rays_multi as contiguous fp32 device tensors of the shapes the passes draw."""
    unknown = set(rand) - {"u", "noise_coarse", "noise_fine"}
    if unknown:
        raise ValueError(f"unknown _rand keys {sorted(unknown)}")
    out = {}
    want = {"noise_coarse": (n, n_obj * n_samples), "noise_fine": (n, n_obj * (n_samples + n_importance))}
    for k, shape in want.items():
        if rand.get(k) is not None:
            if tuple(rand[k].shape) != shape:
                raise ValueError(f"_rand[{k!r}] is {tuple(rand[k].shape)}, expected {shape}")
            out[k] = rand[k].to(dev, torch.float32).contiguous()
    if rand.get("u") is not None:
        if len(rand["u"]) != n_obj:
            raise ValueError(f"_rand['u'] has {len(rand['u'])} entries for {n_obj} ray sets")
        out["u"] = []
        for u in rand["u"]:
            if u is not None and tuple(u.shape) != (n, n_importance):
                raise ValueError(f"_rand['u'] entry is {tuple(u.shape)}, expected {(n, n_importance)}")
            out["u"].append(u.to(dev, torch.float32).contiguous() if u is not None else None)
    return out


def _render_multi_one_call(models, grid, code_table, rays_list, obj_ids, n_samples, use_disp, perturb, n_importance,
                           white_back, boxes, precision, noise_std=0.0, seed=0, clips=None, u_list=None, noise_c=None,
                           noise_f=None):
    dev = rays_list[0].device
    n_obj, n = len(rays_list), rays_list[0].shape[0]
    f = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
    a = _lib.RenderMultiArgs()
    rays_p = (C.c_void_p * n_obj)(*[r.data_ptr() for r in rays_list])
    ids_p = (C.c_int * n_obj)(*obj_ids)
    a.rays_list_host, a.obj_ids_host = rays_p, ids_p
    a.n_obj, a.n_rays, a.n_samples, a.n_importance = n_obj, n, n_samples, n_importance
    a.grid = C.pointer(grid.c)
    packed_c = engine.packed_for(models["coarse"], True)
    packed_f = engine.packed_for(models["fine"], True) if n_importance > 0 else None
    a.packed_coarse = packed_c.data_ptr()
    a.packed_fine = packed_f.data_ptr() if packed_f is not None else None
    a.code_table, a.n_codes = code_table.data_ptr(), code_table.shape[0]
    a.precision = engine.PRECISIONS[precision or engine.default_precision()]
    a.use_disp, a.perturb = int(bool(use_disp)), float(perturb)
    a.seed = seed
    a.white_back = int(bool(white_back))
    a.boxes, a.n_boxes = _lib.ptr(boxes), (boxes.shape[0] if boxes is not None else 0)
    x = _lib.RenderMultiExt()
    x.noise_std = float(noise_std)
    x.noise_coarse, x.noise_fine = _lib.ptr(noise_c), _lib.ptr(noise_f)
    clip_p = u_p = None
    if clips is not None and any(c is not None for c in clips):
        clip_p = (C.c_void_p * n_obj)(*[_lib.ptr(c) for c in clips])
        x.clip_list_host = clip_p
    if u_list is not None:
        u_p = (C.c_void_p * n_obj)(*[_lib.ptr(u) for u in u_list])
        x.u_list_host = u_p
    results: Dict[str, Any] = {}
    for typ, s in (("coarse", n_samples), ("fine", n_samples + n_importance)):
        if typ == "fine" and n_importance == 0:
            continue
        t = n_obj * s
        m = dict(weights=f(n, t), opacity=f(n), z_vals=f(n, t), rgb=f(n, 3), depth=f(n))
        if typ == "coarse":
            m["obj_ids"] = f(n, t)
        cm = getattr(a, typ)
        for k, v in m.items():
            setattr(cm, k, v.data_ptr())
            results[f"{k}_{typ}"] = v
    ws = torch.empty(max(_lib.load().onerf_render_multi_workspace_bytes(n, n_obj, n_samples, n_importance), 256),
                     dtype=torch.uint8, device=dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    _lib.call("onerf_render_multi_fwd_ext", dev, C.byref(a), C.byref(x))
    return results
