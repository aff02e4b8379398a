"""Edited frames from a camera in one library call per frame (or per rank's tile of a frame).

    render_frame(models, embeddings, code_library, H, W, focal, sets, near, far, scale_factor, ...)
        One (obj_id, Toc, box, bbox_enlarge) per ray set -> the result dict of render_rays_multi for the whole H x W
        frame.  Rays are generated on the device, the frame runs through the multi path in chunks of chunk_rays pixels,
        and the maps are written straight into frame-sized buffers (onerf_render_edit_frame, include/onerf_ext.h).
    render_tile(..., pixel_begin, pixel_end, ...)
        The same for a contiguous range of pixels only.
    keys= may also name the per-set maps of set_keys(N_importance): opacity_sets_{typ}, depth_sets_{typ} (H*W, n_obj)
        and rgb_sets_{typ} (H*W, n_obj, 3), how much of each pixel each ray set shows in pass typ
        (onerf_render_edit_frame_sets).  They are never part of the default result.
    Scene(models, embeddings, code_library, scale_factor)
        Another trained scene.  A set (obj_id, Toc, box, bbox_enlarge, scene) renders object obj_id of that scene into
        the frame (onerf_render_edit_frame_scenes): its rays, fields and importance samples in the scene's own units,
        composited on the frame's depth axis.
    render_edit(renderer, ..., imports=None), render_origin(renderer, ...)
        EditableRenderer.render_edit / render_origin (render_tools/editable_renderer.py:183-294) for an instance of the
        reference's class: the same poses, duplicate counting, boxes and side effects, then one render_frame call.
        imports= adds objects of other EditableRenderer instances, each placed by a rigid transform in metres.
    install(EditableRenderer, keys=None, group=None)
        Binds those two as the class's methods, so the reference's demo loop renders through them unchanged.

With `group` (a torch.distributed process group) each rank renders its contiguous tile of the frame
(parallel.shard_bounds over the H*W pixels) and the tiles are all-gathered: every rank returns the whole frame.
A pixel's result does not depend on chunk_rays, the tile bounds or the number of ranks.
"""
from __future__ import annotations

import ctypes as C
import sys
from typing import Any, Dict, Optional, Sequence

import numpy as np
import torch

from . import _lib, engine, parallel
from .multi_rendering import boxes_to_tensor
from .ray_utils import _box_host, _c2w_host
from .rendering import _grid_of, _is_voxel

_MAPS = ("weights", "opacity", "z_vals", "rgb", "depth", "obj_ids")
_SET_MAPS = ("opacity_sets", "depth_sets", "rgb_sets")


def result_keys(N_importance: int):
    """The keys of render_rays_multi's result dict, in its order."""
    keys = [f"{k}_coarse" for k in _MAPS]
    if N_importance > 0:
        keys += [f"{k}_fine" for k in _MAPS[:-1]]
    return keys


def set_keys(N_importance: int):
    """The per-set map keys render_frame computes on request (keys=), for each pass: for pixel r and set position i,
    the sums over set i's samples of the pass's weights w, w * z and w * rgb (no white background).  Summed over the sets
    they give opacity_{typ}, depth_{typ} and rgb_{typ} without the white background."""
    typs = ("coarse", "fine") if N_importance > 0 else ("coarse",)
    return [f"{k}_{typ}" for typ in typs for k in _SET_MAPS]


class Scene:
    """A trained scene that edited frames take objects from: its models ("coarse", "fine"), embeddings (the voxel
    embedding under "xyz"), code library and scale_factor (world units per NeRF unit).  Its weights must have the frame's
    architecture; they are packed as engine.packed_for packs them."""

    def __init__(self, models: Dict[str, Any], embeddings: Dict[str, Any], code_library, scale_factor: float):
        if not _is_voxel(embeddings["xyz"]):
            raise RuntimeError("editing.Scene requires the voxel embedding, as render_frame does")
        scale_factor = float(scale_factor)
        if not (np.isfinite(scale_factor) and scale_factor > 0):
            raise ValueError(f"editing.Scene: scale_factor must be positive and finite, got {scale_factor}")
        self.models, self.embeddings, self.code_library, self.scale_factor = models, embeddings, code_library, scale_factor


def render_frame(models: Dict[str, Any], embeddings: Dict[str, Any], code_library, H: int, W: int, focal: float,
                 sets: Sequence, near: float, far: float, scale_factor: float, background_skip_bbox=None,
                 N_samples: int = 64, N_importance: int = 0, use_disp: bool = False, white_back: bool = False,
                 keys: Optional[Sequence[str]] = None, chunk_rays: int = 65536, group=None,
                 precision: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """Render the H x W frame of `sets`, a list of (obj_id, Toc, box_helper_or_None, bbox_enlarge): obj_id 0 is the scene
    set (no box), Toc its (3,4) or (4,4) camera-to-set pose at NeRF scale; an object set's box helper has BBoxRayHelper's
    pose_avg, axis_align_mat and bbox_bounds.  An object set may carry a fifth element, a Scene (None: this frame's
    scene): the set is then that scene's object, its Toc translation at that scene's NeRF scale and its box in that
    scene's frame; its depths are reported on this frame's axis.  background_skip_bbox: the removed objects' helpers
    (as render_rays_multi).
    Returns render_rays_multi's keys for the whole frame ((H*W, T) per-sample arrays, (H*W, ...) maps) on the device of
    the code table; `keys` restricts what is kept and returned (the rest goes to scratch).  perturb = 0 and noise_std = 0,
    as EditableRenderer renders."""
    n_pix = int(H) * int(W)
    begin, end = parallel.tile_bounds(n_pix, group)
    out = render_tile(models, embeddings, code_library, H, W, focal, sets, near, far, scale_factor, begin, end,
                      background_skip_bbox=background_skip_bbox, N_samples=N_samples, N_importance=N_importance,
                      use_disp=use_disp, white_back=white_back, keys=keys, chunk_rays=chunk_rays, precision=precision)
    return parallel.gather_tile_maps(out, n_pix, group)


def render_tile(models: Dict[str, Any], embeddings: Dict[str, Any], code_library, H: int, W: int, focal: float,
                sets: Sequence, near: float, far: float, scale_factor: float, pixel_begin: int, pixel_end: int,
                background_skip_bbox=None, N_samples: int = 64, N_importance: int = 0, use_disp: bool = False,
                white_back: bool = False, keys: Optional[Sequence[str]] = None, chunk_rays: int = 65536,
                precision: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """render_frame for pixels [pixel_begin, pixel_end) (row-major) of the frame only: (pixel_end - pixel_begin, ...)
    results, row for row those of the whole frame."""
    all_keys = result_keys(N_importance)
    keys = all_keys if keys is None else list(keys)
    all_keys = all_keys + set_keys(N_importance)
    unknown = [k for k in keys if k not in all_keys]
    if unknown:
        raise KeyError(f"render_frame: no such result key {unknown} (N_importance = {N_importance})")
    emb_xyz = embeddings["xyz"]
    if not _is_voxel(emb_xyz):
        raise RuntimeError("render_frame requires the voxel embedding, as render_rays_multi does")
    grid = _grid_of(emb_xyz)
    code_table = engine._f32(code_library.embedding_instance.weight.detach())
    dev = code_table.device
    begin, end = int(pixel_begin), int(pixel_end)
    n, n_obj = max(end - begin, 0), len(sets)
    a = _lib.RenderEditArgs()
    sets_c = (_lib.EditSet * max(n_obj, 1))()
    keep = []                                  # host structs the call reads
    scenes: list = []                          # the distinct source scenes, in order of first use
    set_scene = (C.c_int * max(n_obj, 1))()
    for i, s in enumerate(sets):
        obj_id, Toc, box, bbox_enlarge = s[:4]
        scene = s[4] if len(s) > 4 else None
        set_scene[i] = -1
        if scene is not None:
            j = next((j for j, sc in enumerate(scenes) if sc is scene), len(scenes))
            if j == len(scenes):
                scenes.append(scene)
            set_scene[i] = j
        sets_c[i].obj_id = int(obj_id)
        sets_c[i].Toc = _c2w_host(Toc)
        if box is not None:
            bh = _box_host(box, float(bbox_enlarge))
            keep.append(bh)
            sets_c[i].box = C.pointer(bh)
    a.sets_host, a.n_obj = sets_c, n_obj
    a.H, a.W, a.focal = int(H), int(W), float(focal)
    a.pixel_begin, a.pixel_end = begin, end
    a.near, a.far, a.scale_factor = float(near), float(far), float(scale_factor)
    a.n_samples, a.n_importance = int(N_samples), int(N_importance)
    a.grid = C.pointer(grid.c)
    with torch.no_grad():          # inference: the cached packed weights (held until the call has been enqueued)
        packed_c = engine.packed_for(models["coarse"], True)
        packed_f = engine.packed_for(models["fine"], True) if N_importance > 0 else None
        scenes_c = (_lib.EditScene * max(len(scenes), 1))()
        for j, sc in enumerate(scenes):
            g = _grid_of(sc.embeddings["xyz"])
            ct = engine._f32(sc.code_library.embedding_instance.weight.detach())
            if ct.device != dev:
                raise RuntimeError(f"render_frame: a source scene's code table is on {ct.device}, the frame on {dev}")
            pc = engine.packed_for(sc.models["coarse"], True)
            pf = engine.packed_for(sc.models["fine"], True) if N_importance > 0 else None
            keep += [g, ct, pc, pf]
            scenes_c[j].grid = C.pointer(g.c)
            scenes_c[j].packed_coarse, scenes_c[j].packed_fine = pc.data_ptr(), (pf.data_ptr() if pf is not None else None)
            scenes_c[j].code_table, scenes_c[j].n_codes = ct.data_ptr(), ct.shape[0]
            scenes_c[j].scale_factor = sc.scale_factor
    a.packed_coarse = packed_c.data_ptr()
    a.packed_fine = packed_f.data_ptr() if packed_f is not None else None
    a.code_table, a.n_codes = code_table.data_ptr(), code_table.shape[0]
    a.precision = engine.PRECISIONS[precision or engine.default_precision()]
    a.use_disp, a.white_back = int(bool(use_disp)), int(bool(white_back))
    boxes = boxes_to_tensor(background_skip_bbox, dev)
    a.boxes, a.n_boxes = _lib.ptr(boxes), (boxes.shape[0] if boxes is not None else 0)
    a.chunk_rays = int(chunk_rays)
    widths = {"rgb": 3, "opacity": 1, "depth": 1}
    out: Dict[str, torch.Tensor] = {}
    for typ, s in (("coarse", N_samples), ("fine", N_samples + N_importance)):
        for k in _MAPS:
            key = f"{k}_{typ}"
            if key in keys:
                w = widths.get(k, n_obj * s)
                out[key] = torch.empty((n, w) if w != 1 else (n,), dtype=torch.float32, device=dev)
                setattr(getattr(a, typ), k, out[key].data_ptr())
    set_maps = {"coarse": _lib.SetMaps(), "fine": _lib.SetMaps()}
    for key in set_keys(N_importance):
        if key in keys:
            k, typ = key.rsplit("_", 1)
            out[key] = torch.empty((n, n_obj, 3) if k == "rgb_sets" else (n, n_obj), dtype=torch.float32, device=dev)
            setattr(set_maps[typ], k.split("_")[0], out[key].data_ptr())
    lib = _lib.load()
    with_sets = any(k in keys for k in set_keys(N_importance))
    ws_bytes = (lib.onerf_render_edit_scenes_workspace_bytes if scenes else
                lib.onerf_render_edit_sets_workspace_bytes if with_sets else lib.onerf_render_edit_workspace_bytes)
    ws = engine.workspace(ws_bytes(a.chunk_rays, n_obj, a.n_samples, a.n_importance), dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    if scenes:
        _lib.call("onerf_render_edit_frame_scenes", dev, C.byref(a), scenes_c, len(scenes), set_scene,
                  C.byref(set_maps["coarse"]), C.byref(set_maps["fine"]))
    elif with_sets:
        _lib.call("onerf_render_edit_frame_sets", dev, C.byref(a), C.byref(set_maps["coarse"]), C.byref(set_maps["fine"]))
    else:
        _lib.call("onerf_render_edit_frame", dev, C.byref(a))
    return {k: out[k] for k in all_keys if k in out}


def _focal(w: int, fovx_deg: float) -> float:
    return (w / 2) / np.tan((fovx_deg / 2) / (180 / np.pi))          # editable_renderer.py:190, :214


def _center_pose_from_avg(renderer):
    """datasets/geo_utils.py's center_pose_from_avg, as the renderer's own module imported it."""
    return sys.modules[type(renderer).__module__].center_pose_from_avg


def _frame_of(renderer, h, w, focal, sets, background_skip_bbox, white_back, keys, group):
    model = renderer.ckpt_config.model
    s = renderer.system
    return render_frame(s.models, s.embeddings, s.code_library, h, w, focal, sets, renderer.near, renderer.far,
                        renderer.scale_factor, background_skip_bbox=background_skip_bbox, N_samples=model.N_samples,
                        N_importance=model.N_importance, use_disp=model.use_disp, white_back=white_back, keys=keys,
                        group=group)


def edit_sets(renderer, camera_pose_Twc, render_bg_only: bool = False, render_obj_only: bool = False):
    """The ray sets of EditableRenderer.render_edit (editable_renderer.py:216-263): [(obj_id, Toc, box, bbox_enlarge)],
    with its side effects on renderer.active_object_ids."""
    Twc = _center_pose_from_avg(renderer)(renderer.pose_avg, camera_pose_Twc)
    if render_bg_only:
        renderer.active_object_ids = [0]
    if render_obj_only:
        renderer.active_object_ids.remove(0)
    sets, processed_obj_id = [], []
    for obj_id in renderer.active_object_ids:
        obj_duplication_cnt = np.sum(np.array(processed_obj_id) == obj_id)
        box = None
        if obj_id == 0:
            Tow = np.eye(4)
        else:
            object_pose = renderer.object_pose_transform[f"{obj_id}_{obj_duplication_cnt}"]
            box = renderer.get_object_bbox_helper(obj_id)
            Tow_orig = box.get_world_to_object_transform()
            transform = np.linalg.inv(Tow_orig) @ object_pose @ Tow_orig
            Tow = np.linalg.inv(transform)
        processed_obj_id.append(obj_id)
        Toc = Tow @ Twc
        Toc[:, 3] /= renderer.scale_factor
        sets.append((obj_id, torch.from_numpy(Toc).float()[:3, :4], box, renderer.bbox_enlarge))
    return sets


def scene_of(renderer) -> Scene:
    """The trained scene an EditableRenderer instance holds, as a Scene."""
    s = renderer.system
    return Scene(s.models, s.embeddings, s.code_library, renderer.scale_factor)


def import_sets(camera_pose_Twc, imports, bbox_enlarge: float):
    """The ray sets of objects taken from other scenes: for each (source, obj_id, place) of `imports`, with source an
    EditableRenderer instance of the other scene and place the 4x4 rigid transform (metres) from the source's world (its
    transforms_full.json / bbox frame) to this frame's world, the set (obj_id, Toc, box, bbox_enlarge, Scene of source)
    with Toc = C_src @ inv(place) @ Twc and its translation divided by the source's scale_factor (C_src: the source's
    scene_center centring, center_pose_from_avg) and box = source.get_object_bbox_helper(obj_id)."""
    Twc = np.eye(4)
    Twc[:3] = np.asarray(camera_pose_Twc, dtype=np.float64)[:3]
    sets, scenes = [], {}
    for source, obj_id, place in imports:
        scene = scenes.setdefault(id(source), scene_of(source))
        Toc = _center_pose_from_avg(source)(source.pose_avg, np.linalg.inv(np.asarray(place, dtype=np.float64)) @ Twc)
        Toc[:, 3] /= source.scale_factor
        sets.append((int(obj_id), torch.from_numpy(Toc).float()[:3, :4], source.get_object_bbox_helper(obj_id),
                     bbox_enlarge, scene))
    return sets


def render_edit(renderer, h: int, w: int, camera_pose_Twc, fovx_deg: float = 70, show_progress: bool = True,
                render_bg_only: bool = False, render_obj_only: bool = False, white_back: bool = False, *, keys=None,
                group=None, imports=None) -> Dict[str, torch.Tensor]:
    """EditableRenderer.render_edit (editable_renderer.py:203-294) in one render_frame call; CPU tensors as the
    reference returns them.  show_progress is accepted and unused (there is no chunk loop to report on).
    imports: [(source_renderer, obj_id, place)] objects of other scenes added after the renderer's own sets (see
    import_sets; the renderer's bbox_enlarge applies), except with render_bg_only."""
    raw_Twc = np.array(camera_pose_Twc, dtype=np.float64)
    sets = edit_sets(renderer, camera_pose_Twc, render_bg_only, render_obj_only)
    if imports and not render_bg_only:
        sets += import_sets(raw_Twc, imports, renderer.bbox_enlarge)
    res = _frame_of(renderer, h, w, _focal(w, fovx_deg), sets, renderer.get_skipping_bbox_helper(), white_back, keys,
                    group)
    return {k: v.cpu() for k, v in res.items()}


def origin_sets(renderer, camera_pose_Twc):
    """The one scene ray set of EditableRenderer.render_origin (editable_renderer.py:190-199)."""
    Twc = _center_pose_from_avg(renderer)(renderer.pose_avg, camera_pose_Twc)
    Twc[:, 3] /= renderer.scale_factor
    Toc = np.linalg.inv(np.eye(4)) @ Twc
    return [(0, torch.from_numpy(Toc).float()[:3, :4], None, 0.0)]


def render_origin(renderer, h: int, w: int, camera_pose_Twc, fovx_deg: float = 70, *, group=None) -> Dict[str, torch.Tensor]:
    """EditableRenderer.render_origin (editable_renderer.py:183-201): the unedited scene (no removed boxes), device
    tensors as scene_inference keeps them."""
    return _frame_of(renderer, h, w, _focal(w, fovx_deg), origin_sets(renderer, camera_pose_Twc), None, False, None, group)


def install(editable_renderer_cls, keys=None, group=None):
    """Make `editable_renderer_cls` (the reference's EditableRenderer) render through render_edit / render_origin above.
    keys: what render_edit computes and returns (None: every key of the reference's dict; the per-set maps of set_keys
    only when named here); group: the process group whose ranks share each frame
    (None: one process renders it)."""
    def _render_edit(self, h, w, camera_pose_Twc, fovx_deg=70, show_progress=True, render_bg_only=False,
                     render_obj_only=False, white_back=False):
        return render_edit(self, h, w, camera_pose_Twc, fovx_deg, show_progress, render_bg_only, render_obj_only,
                           white_back, keys=keys, group=group)

    def _render_origin(self, h, w, camera_pose_Twc, fovx_deg=70):
        return render_origin(self, h, w, camera_pose_Twc, fovx_deg, group=group)

    editable_renderer_cls.render_edit = _render_edit
    editable_renderer_cls.render_origin = _render_origin
    return editable_renderer_cls
