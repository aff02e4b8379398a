"""Tensor-level wrappers over the C ABI: one function per stage kernel, plus the weight-pack cache.

All tensors are CUDA fp32 and stay on the device; nothing here computes on the host.  The reference
surface (render_rays / inference_model / render_rays_multi) is assembled from these in rendering.py
and multi_rendering.py.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import torch

from . import _lib

PRECISIONS = {"fp32": _lib.PREC_FP32, "bf16": _lib.PREC_BF16}

# bench.py's roofline pass sets this to a list; field() then brackets each field launch with CUDA events
# on the launching stream and appends (start, end, n_rays, n_samples).  None (default) = no events.
PROFILE_EVENTS = None


def default_precision() -> str:
    """bf16 = wgmma tensor-core path (product default); fp32 = FFMA verification arithmetic."""
    return os.environ.get("ONERF_PRECISION", "bf16")


def train_precision(precision: Optional[str]) -> str:
    """The arithmetic of a differentiable call: bf16 (None = the default) is the tensor-core forward and backward;
    anything else selects the fp32 verification arithmetic end to end."""
    return "bf16" if (precision or default_precision()) == "bf16" else "fp32"


def new_seed() -> int:
    """A fresh 63-bit seed from torch's CPU generator (so torch.manual_seed controls the render RNG)."""
    return int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).item())


def _f32(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


# ------------------------------------------------------------------------------------------------
# weights
# ------------------------------------------------------------------------------------------------
# reference attribute names (models/nerf_model.py:41-58, 77-95) in the C ABI's layer order
LINEAR_ATTRS = (
    [f"xyz_encoding_{i}.0" for i in range(1, 9)] + ["sigma", "xyz_encoding_final", "dir_encoding.0", "rgb.0"]
    + [f"instance_encoding_{i}.0" for i in range(1, 5)]
    + ["instance_sigma", "instance_encoding_final.0", "inst_dir_encoding.0", "inst_rgb.0"]
)


def _get(module, dotted):
    for part in dotted.split("."):
        module = module[int(part)] if part.isdigit() else getattr(module, part)
    return module


def model_linears(model) -> list:
    """The 20 (weight, bias) parameter pairs of an ObjectNeRF-shaped module, ABI order."""
    return [(_get(model, a).weight, _get(model, a).bias) for a in LINEAR_ATTRS]


def check_architecture(model, use_voxel: bool):
    lin = model_linears(model)
    xin = 271 if use_voxel else 63
    oin = xin + (104 if use_voxel else 0) + 64
    want = ([(256, xin)] + [(256, 256)] * 3 + [(256, xin + 256)] + [(256, 256)] * 3
            + [(1, 256), (256, 256), (128, 283), (3, 128)]
            + [(128, oin), (128, 128), (128, oin + 128), (128, 128)]
            + [(1, 128), (128, 128), (64, 155), (3, 64)])
    got = [tuple(w.shape) for w, _ in lin]
    if got != want:
        raise RuntimeError(
            "unsupported ObjectNeRF architecture for the sm_90a kernels (built for D=8, W=256, skips=[4], "
            f"inst_D=4, inst_W=128, inst_skips=[2]); layer shapes {got}")
    return lin


def pointer_tables(pairs: Sequence):
    """The two ABI pointer tables (c_void_p * 20) of 20 tensor pairs: (W, b) -> (W table, b table), and likewise
    (dW, db)."""
    return tuple((C.c_void_p * _lib.N_LINEAR)(*[t.data_ptr() for t in col]) for col in zip(*pairs))


def grad_buffer(tensors: Sequence, dev):
    """One zero-filled fp32 buffer with a gradient view shaped like each of `tensors`, each offset rounded up to 4 floats
    (16 bytes).  Returns (buffer, views, offsets in floats)."""
    offsets, off = [], 0
    for t in tensors:
        offsets.append(off)
        off += -(-t.numel() // 4) * 4
    flat = torch.zeros(off, dtype=torch.float32, device=dev)
    return flat, [flat[o:o + t.numel()].view(t.shape) for t, o in zip(tensors, offsets)], offsets


def aligned_bytes(nbytes: int, dev) -> torch.Tensor:
    """A uint8 tensor of nbytes (at least 1) starting on a 1024-byte boundary (packed weights, training dumps and
    workspaces)."""
    nbytes = max(int(nbytes), 1)
    t = torch.empty(nbytes + 1024, dtype=torch.uint8, device=dev)
    off = (-t.data_ptr()) % 1024
    return t[off:off + nbytes]


def pack_weights(linears: Sequence, use_voxel: bool, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Run the pack kernel into `out` (a new blob if None); returns the packed blob (uint8 tensor, 1024-byte aligned)."""
    dev = linears[0][0].device
    lin = [(_f32(w.detach()), _f32(b.detach())) for w, b in linears]
    if out is None:
        out = aligned_bytes(_lib.load().onerf_packed_weights_bytes(int(use_voxel)), dev)
    _lib.call("onerf_pack_weights", dev, int(use_voxel), *pointer_tables(lin), out.data_ptr(), out.numel())
    out._keepalive = lin  # sources must outlive the async pack kernels
    return out


_workspaces = {}   # (device index, bytes) -> workspace


def workspace(nbytes: int, dev: torch.device) -> torch.Tensor:
    """One workspace per (device, size), kept for the life of the process so that a captured call keeps valid addresses
    (calls on one stream are ordered)."""
    key = (dev.index, nbytes)
    ws = _workspaces.get(key)
    if ws is None:
        ws = _workspaces[key] = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
    return ws


def cached_plan(plans, owner, key: tuple, make):
    """plans[owner][key], made by make() on first use: the buffers of one configuration of a one-call render."""
    per_owner = plans.setdefault(owner, {})
    plan = per_owner.get(key)
    if plan is None:
        plan = per_owner[key] = make()
    return plan


_pack_cache = {}   # id(model) -> (weakref to the model, content fingerprint, blob)


def _fingerprint(lin) -> tuple:
    """Identity of the parameter CONTENT as far as it can be known without reading the device: storage address and
    in-place version counter of every tensor.  Updates made through `.data` (torch_optimizer's RAdam / Ranger) do not bump
    the version, which is why packed_for() never trusts this under autograd (see below) and exposes invalidate_packed()."""
    return tuple((w.data_ptr(), w._version, b.data_ptr(), b._version) for w, b in lin)


def invalidate_packed(model=None):
    """Drop the cached packed weights of `model` (all models if None).  Call after modifying parameters in a way
    autograd's version counter does not see (`p.data.copy_(...)`, `p.data.add_(...)`)."""
    if model is None:
        _pack_cache.clear()
    else:
        _pack_cache.pop(id(model), None)


def packed_for(model, use_voxel: bool, fresh: Optional[bool] = None) -> torch.Tensor:
    """Packed blob for an nn.Module.  Whenever gradients are enabled and a parameter requires grad (training: the
    optimizer changes the weights between calls, possibly through `.data`) the weights are re-packed on EVERY call: one
    kernel launch over 5 MB, far cheaper than a step.  Only inference calls (no_grad / frozen model) reuse a cached blob,
    keyed on a weak reference to the module (a new module on a recycled id() never hits) plus the fingerprint above."""
    lin = check_architecture(model, use_voxel)
    if fresh is None:
        fresh = torch.is_grad_enabled() and any(w.requires_grad or b.requires_grad for w, b in lin)
    if fresh:
        return pack_weights(lin, use_voxel)
    key = (_fingerprint(lin), bool(use_voxel))
    hit = _pack_cache.get(id(model))
    if hit is not None and hit[0]() is model and hit[1] == key:
        return hit[2]
    blob = pack_weights(lin, use_voxel)
    import weakref
    mid = id(model)
    _pack_cache[mid] = (weakref.ref(model, lambda _r, mid=mid: _pack_cache.pop(mid, None)), key, blob)
    return blob


# ------------------------------------------------------------------------------------------------
# grid
# ------------------------------------------------------------------------------------------------
class GridBuffers:
    """Device views of the EmbeddingVoxel buffers the kernels read
    (reference models/embedding_helper.py:107-133,189-200)."""

    def __init__(self, table, idx_map, voxel_offset, voxel_size, voxel_shape):
        self.table = _f32(table.detach())
        self.idx_map = idx_map.contiguous()
        assert self.idx_map.dtype == torch.int64
        self.voxel_offset = _f32(voxel_offset).reshape(3)
        self.voxel_size = _f32(voxel_size).reshape(1)
        self.voxel_shape = voxel_shape.to(torch.int64).contiguous()
        self.c = _lib.Grid(self.table.data_ptr(), self.idx_map.data_ptr(), self.voxel_offset.data_ptr(),
                           self.voxel_size.data_ptr(), self.voxel_shape.data_ptr())

    @classmethod
    def from_module(cls, emb):
        return cls(emb.embedding_space_ftr.weight, emb.voxel_idx_map, emb.voxel_offset, emb.voxel_size,
                   emb.voxel_shape)


# ------------------------------------------------------------------------------------------------
# stage kernels
# ------------------------------------------------------------------------------------------------
def sample_coarse(rays, n_samples, use_disp=False, perturb=0.0, jitter=None, seed=0, out=None):
    rays = _f32(rays)
    n = rays.shape[0]
    z = out if out is not None else torch.empty(n, n_samples, dtype=torch.float32, device=rays.device)
    assert z.is_contiguous() and z.shape == (n, n_samples)
    jitter = _f32(jitter) if jitter is not None else None
    _lib.call("onerf_sample_coarse", rays.device, rays.data_ptr(), n, n_samples, int(bool(use_disp)), float(perturb),
              _lib.ptr(jitter), seed, z.data_ptr())
    return z


def sample_pdf_merge(z_coarse, weights, n_importance, det, u=None, seed=0, out=None, clip=None):
    """clip (N,2) = (near_box, far_box) of a 10-column ray set: merged depths strictly inside the interval become far_box
    (onerf_sample_pdf_merge_clip)."""
    z_coarse, weights = _f32(z_coarse), _f32(weights.detach())
    n, s = z_coarse.shape
    if out is None:
        out = torch.empty(n, s + n_importance, dtype=torch.float32, device=z_coarse.device)
    assert out.is_contiguous() and out.shape == (n, s + n_importance)
    u = _f32(u) if u is not None else None
    args = (z_coarse.data_ptr(), weights.data_ptr(), n, s, n_importance, int(bool(det)), _lib.ptr(u), seed)
    if clip is None:
        _lib.call("onerf_sample_pdf_merge", z_coarse.device, *args, out.data_ptr())
    else:
        clip = _f32(clip)
        assert clip.shape == (n, 2)
        _lib.call("onerf_sample_pdf_merge_clip", z_coarse.device, *args, clip.data_ptr(), out.data_ptr())
    return out


def sample_pdf(bins, weights, n_importance, det, u=None, seed=0):
    bins, weights = _f32(bins), _f32(weights.detach())
    n, nb = bins.shape
    assert weights.shape == (n, nb - 1)
    out = torch.empty(n, n_importance, dtype=torch.float32, device=bins.device)
    u = _f32(u) if u is not None else None
    _lib.call("onerf_sample_pdf", bins.device, bins.data_ptr(), weights.data_ptr(), n, nb, n_importance, int(bool(det)),
              _lib.ptr(u), seed, out.data_ptr())
    return out


def encode(xyz, grid: Optional[GridBuffers]):
    xyz = _f32(xyz)
    n = xyz.shape[0]
    scene = torch.empty(n, 271 if grid is not None else 63, dtype=torch.float32, device=xyz.device)
    obj = torch.empty(n, 104, dtype=torch.float32, device=xyz.device) if grid is not None else None
    _lib.call("onerf_encode", xyz.device, C.byref(grid.c) if grid is not None else None, xyz.data_ptr(), n,
              scene.data_ptr(), _lib.ptr(obj))
    return scene, obj


def dir_encode(dirs):
    """PE4 of directions (B,3) -> (B,27) (onerf_dir_encode, the encoding the field kernel applies to rays[:, 3:6])."""
    n = dirs.shape[0]
    rays = torch.zeros(n, 8, dtype=torch.float32, device=dirs.device)
    rays[:, 3:6] = dirs
    out = torch.empty(n, 27, dtype=torch.float32, device=dirs.device)
    _lib.call("onerf_dir_encode", dirs.device, rays.data_ptr(), n, out.data_ptr())
    return out


def voxel_features(xyz, grid: GridBuffers):
    """Raw trilinear features (B,24) of the sparse voxel grid at xyz (no positional encoding)."""
    xyz = _f32(xyz).reshape(-1, 3)
    out = torch.empty(xyz.shape[0], 24, dtype=torch.float32, device=xyz.device)
    _lib.call("onerf_voxel_features", xyz.device, C.byref(grid.c), xyz.data_ptr(), xyz.shape[0], out.data_ptr())
    return out


def field(rays, z, packed, grid: Optional[GridBuffers], codes=None, code_row=None, want_scene=True,
          want_object=True, precision=None, xyz=None, mute_zero_rays=False, boxes=None, scene_out=None,
          obj_out=None, z_stride=None, out_stride=None, n_samples=None, activations=None, train_ws=None,
          _args_out=None):
    """Fused encode + MLP.  Returns (scene_out, obj_out), each (N,S,4) = rgb,sigma (or None).
    z / outputs may be column blocks of wider arrays (z_stride / out_stride, in samples).
    train_ws: a 1024-byte aligned uint8 tensor of onerf_field_train_bytes bytes receiving the tensor-core training dump.
    _args_out: a list that receives the argument block and the tensors it points into (field_bwd takes both)."""
    rays = _f32(rays)
    n = rays.shape[0]
    s = n_samples if n_samples is not None else z.shape[1]
    dev = rays.device
    z_stride = z_stride if z_stride is not None else s
    out_stride = out_stride if out_stride is not None else s
    if want_scene and scene_out is None:
        scene_out = torch.empty(n, s, 4, dtype=torch.float32, device=dev)
    if want_object and obj_out is None:
        obj_out = torch.empty(n, s, 4, dtype=torch.float32, device=dev)
    ray_const = torch.empty(n, _lib.RAY_CONST_FLOATS, dtype=torch.float32, device=dev)
    prec = PRECISIONS[precision or default_precision()]
    a = _lib.FieldArgs()
    a.rays = rays.data_ptr()
    xyz = _f32(xyz) if xyz is not None else None
    a.xyz = _lib.ptr(xyz)
    a.z = z.data_ptr()
    a.z_stride = z_stride
    codes = _f32(codes) if codes is not None else None
    code_row = _f32(code_row) if code_row is not None else None
    a.codes, a.code_row = _lib.ptr(codes), _lib.ptr(code_row)
    a.n_rays, a.n_samples = n, s
    a.grid = C.pointer(grid.c) if grid is not None else None
    a.packed = packed.data_ptr()
    a.want_scene, a.want_object, a.precision = int(want_scene), int(want_object), prec
    a.mute_zero_rays = int(mute_zero_rays)
    boxes = _f32(boxes) if boxes is not None and boxes.numel() > 0 else None
    a.boxes, a.n_boxes = _lib.ptr(boxes), (boxes.shape[0] if boxes is not None else 0)
    a.scene_out = scene_out.data_ptr() if want_scene else None
    a.obj_out = obj_out.data_ptr() if want_object else None
    a.out_stride = out_stride
    a.ray_const = ray_const.data_ptr()
    a.activations = activations      # (c_void_p * 17) array or None: FFMA kernel dumps per-layer activations (backward)
    a.train_ws = train_ws.data_ptr() if train_ws is not None else None
    if _args_out is not None:
        # (not the outputs: a caller that keeps them alive for the backward saves them itself)
        _args_out += [a, (rays, xyz, z, codes, code_row, boxes, ray_const, grid, packed, train_ws)]
    if PROFILE_EVENTS is not None:
        launch_stream = torch.cuda.current_stream(dev)      # the stream _lib.call enqueues the field kernel on
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(launch_stream)
    _lib.call("onerf_field_fwd", dev, C.byref(a))
    if PROFILE_EVENTS is not None:
        e1.record(launch_stream)
        PROFILE_EVENTS.append((e0, e1, n, s))
    return (scene_out if want_scene else None), (obj_out if want_object else None)


def field_bwd(args, d_scene, d_obj, linears, grads=None, d_codes=None, table_grad=None, workspace=None):
    """onerf_field_bwd for the evaluation `args` (from field(..., _args_out=...)): accumulates the 20 (dW, db) gradient
    pairs into `grads` (zeros shaped like `linears` if None) and returns them, ABI order; d_codes / table_grad are
    accumulated in place.  workspace: a 1024-byte aligned uint8 tensor of at least onerf_field_bwd_workspace_bytes
    (allocated if None)."""
    dev = linears[0][0].device
    if workspace is None:
        workspace = aligned_bytes(field_bwd_workspace_bytes(args.precision, bool(args.grid), args.n_rays, args.n_samples), dev)
    lin = [(_f32(w.detach()), b) for w, b in linears]
    if grads is None:
        views = grad_buffer([t for pair in linears for t in pair], dev)[1]
        grads = list(zip(views[0::2], views[1::2]))
    g = _lib.FieldBwdArgs()
    g.W = pointer_tables(lin)[0]
    g.dW, g.db = pointer_tables(grads)
    g.d_codes, g.table_grad = _lib.ptr(d_codes), _lib.ptr(table_grad)
    g.workspace, g.workspace_bytes = workspace.data_ptr(), workspace.numel()
    d_scene = _f32(d_scene) if d_scene is not None else None
    d_obj = _f32(d_obj) if d_obj is not None else None
    _lib.call("onerf_field_bwd", dev, C.byref(args), _lib.ptr(d_scene), _lib.ptr(d_obj), C.byref(g))
    return grads


def field_bwd_workspace_bytes(precision: int, use_voxel: bool, n_rays: int, n_samples: int) -> int:
    return int(_lib.load().onerf_field_bwd_workspace_bytes(precision, int(use_voxel), n_rays, n_samples))


def _composite_args(z, scene, obj, noise_std, white_back, is_eval, zero_last_delta, rays_in_bbox, frustum_bound_th,
                    pass_through_mask, noise_scene, noise_obj, seed):
    """Argument block of onerf_composite / onerf_composite_bwd (no outputs set) and the tensors it points into."""
    n, s = z.shape
    a = _lib.CompositeArgs()
    a.z, a.scene, a.obj = z.data_ptr(), scene.data_ptr(), _lib.ptr(obj)
    a.n_rays, a.n_samples = n, s
    a.noise_std = float(noise_std)
    noise_scene = _f32(noise_scene) if noise_scene is not None else None
    noise_obj = _f32(noise_obj) if noise_obj is not None else None
    a.noise_scene, a.noise_obj, a.seed = _lib.ptr(noise_scene), _lib.ptr(noise_obj), seed
    a.white_back, a.is_eval = int(bool(white_back)), int(bool(is_eval))
    a.zero_last_delta, a.rays_in_bbox = int(bool(zero_last_delta)), int(bool(rays_in_bbox))
    a.frustum_bound_th = float(frustum_bound_th)
    ptm = None
    if pass_through_mask is not None:
        ptm = pass_through_mask.reshape(-1).to(torch.uint8).contiguous()
    a.pass_through_mask = _lib.ptr(ptm)
    return a, (noise_scene, noise_obj, ptm)


def composite(z, scene, obj, noise_std=0.0, white_back=False, is_eval=False, zero_last_delta=False,
              rays_in_bbox=False, frustum_bound_th=0.0, pass_through_mask=None, noise_scene=None,
              noise_obj=None, seed=0):
    """Returns dict(weights, opacity, rgb, depth[, rgb_instance, depth_instance, opacity_instance])."""
    n, s = z.shape
    dev = z.device
    f = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
    out = {"weights": f(n, s), "opacity": f(n), "rgb": f(n, 3), "depth": f(n)}
    if obj is not None:
        out.update(rgb_instance=f(n, 3), depth_instance=f(n), opacity_instance=f(n))
    a, _keep = _composite_args(z, scene, obj, noise_std, white_back, is_eval, zero_last_delta, rays_in_bbox,
                               frustum_bound_th, pass_through_mask, noise_scene, noise_obj, seed)
    a.weights, a.opacity, a.rgb, a.depth = (out[k].data_ptr() for k in ("weights", "opacity", "rgb", "depth"))
    if obj is not None:
        a.rgb_instance = out["rgb_instance"].data_ptr()
        a.depth_instance = out["depth_instance"].data_ptr()
        a.opacity_instance = out["opacity_instance"].data_ptr()
    _lib.call("onerf_composite", dev, C.byref(a))
    return out


def composite_bwd(z, scene, obj, depth_scene, grads, noise_std=0.0, white_back=False, is_eval=False,
                  zero_last_delta=False, frustum_bound_th=0.0, pass_through_mask=None, noise_scene=None,
                  noise_obj=None, seed=0):
    """Gradient of composite() w.r.t. the fields -> (dscene, dobj | None), each (N,S,4); depth_scene: the forward's scene
    depth; grads: upstream gradients by map name (missing = 0).  Noise as the forward's (re-drawn from `seed` without
    buffers).  No rays_in_bbox: it only selects the returned weights, which carry no gradient."""
    n, s = z.shape
    dev = z.device
    dscene = torch.empty(n, s, 4, dtype=torch.float32, device=dev)
    dobj = torch.empty(n, s, 4, dtype=torch.float32, device=dev) if obj is not None else None
    a, _keep = _composite_args(z, scene, obj, noise_std, white_back, is_eval, zero_last_delta, False,
                               frustum_bound_th, pass_through_mask, noise_scene, noise_obj, seed)
    g = {k: (v.contiguous().float() if v is not None else None) for k, v in grads.items()}
    _lib.call("onerf_composite_bwd", dev, C.byref(a), _lib.ptr(depth_scene), _lib.ptr(g.get("rgb")),
              _lib.ptr(g.get("depth")), _lib.ptr(g.get("opacity")), _lib.ptr(g.get("rgb_instance")),
              _lib.ptr(g.get("depth_instance")), _lib.ptr(g.get("opacity_instance")), dscene.data_ptr(), _lib.ptr(dobj))
    return dscene, dobj


def composite_multi(z_all, field_all, white_back=False, want_ids=False, want_unsorted=False, merge=False, noise_std=0.0,
                    noise=None, seed=0, fine=False):
    """z_all (n_obj, N, S), field_all (n_obj, N, S, 4) -> sorted-order outputs (N, n_obj*S).  Any n_obj * S: the bitonic
    kernel up to 4096 samples per ray, the rank-merge path above (or always, with merge=True).
    noise_std != 0: sigma noise by sorted position, from `noise` (N, n_obj*S) or else Philox stream 7 (coarse) / 8
    (fine=True) keyed by `seed` (onerf_composite_multi_noise_ws / _merge)."""
    n_obj, n, s = z_all.shape
    t = n_obj * s
    dev = z_all.device
    f = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
    out = {"z_vals": f(n, t), "weights": f(n, t), "opacity": f(n), "rgb": f(n, 3), "depth": f(n)}
    ids = f(n, t) if want_ids else None
    unsorted = f(n_obj, n, s) if want_unsorted else None
    ws = None
    if merge or t > 4096:
        ws = torch.empty(max(_lib.load().onerf_composite_multi_workspace_bytes(n, n_obj, s), 256), dtype=torch.uint8, device=dev)
    head = (z_all.data_ptr(), field_all.data_ptr(), n, n_obj, s, int(bool(white_back)))
    if noise_std != 0 or noise is not None:
        noise = _f32(noise) if noise is not None else None
        assert noise is None or noise.shape == (n, t)
        entry = "onerf_composite_multi_noise_merge" if merge else "onerf_composite_multi_noise_ws"
        head += (float(noise_std), _lib.ptr(noise), seed, int(bool(fine)))
    else:
        entry = "onerf_composite_multi_merge" if merge else "onerf_composite_multi_ws"
    _lib.call(entry, dev, *head, out["z_vals"].data_ptr(), out["weights"].data_ptr(), _lib.ptr(ids), _lib.ptr(unsorted),
              out["opacity"].data_ptr(), out["rgb"].data_ptr(), out["depth"].data_ptr(), _lib.ptr(ws),
              ws.numel() if ws is not None else 0)
    if want_ids:
        out["obj_ids"] = ids
    if want_unsorted:
        out["weights_unsorted"] = unsorted
    return out


class RenderPlan:
    """Buffers + argument block of one onerf_render_rays_fwd() call (the whole forward of render_rays in ONE C call,
    models/rendering.py:233-337).  All outputs and the workspace are allocated once, so `run()` only enqueues kernels:
    it can be captured in a CUDA graph and replayed.  train_ws (a 1024-byte aligned uint8 tensor of
    onerf_train_workspace_bytes_prec bytes, owned by the caller) makes it the forward of a training step, whose
    backward (onerf_render_rays_bwd) takes `args`."""

    MAP_KEYS = ("weights", "opacity", "z_vals", "rgb", "depth", "rgb_instance", "depth_instance", "opacity_instance")

    def __init__(self, rays, packed_coarse, packed_fine, grid: Optional[GridBuffers], codes=None, n_samples=64,
                 n_importance=0, use_disp=False, perturb=0.0, noise_std=0.0, white_back=False, forward_instance=True,
                 is_eval=False, zero_last_delta=False, rays_in_bbox=False, frustum_bound_th=0.0,
                 pass_through_mask=None, precision=None, seed=0, rand=None, train_ws=None):
        lib = _lib.load()
        self.rays = _f32(rays)
        n, dev = self.rays.shape[0], self.rays.device
        rand = rand or {}
        self._keep = [self.rays, packed_coarse, packed_fine, grid]
        f = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        self.maps = {}
        a = _lib.RenderArgs()
        for typ, s in (("coarse", n_samples), ("fine", n_samples + n_importance)):
            if typ == "fine" and n_importance == 0:
                continue
            m = dict(weights=f(n, s), opacity=f(n), z_vals=f(n, s), rgb=f(n, 3), depth=f(n))
            if forward_instance:
                m.update(rgb_instance=f(n, 3), depth_instance=f(n), opacity_instance=f(n))
            self.maps[typ] = m
            cm = getattr(a, typ)
            for k, v in m.items():
                setattr(cm, k, v.data_ptr())
        ws_bytes = lib.onerf_render_rays_workspace_bytes(n, n_samples, n_importance)
        self.workspace = torch.empty(max(ws_bytes, 256), dtype=torch.uint8, device=dev)
        assert self.workspace.data_ptr() % 256 == 0
        codes = _f32(codes) if (codes is not None and forward_instance) else None
        mask = None
        if pass_through_mask is not None:
            mask = pass_through_mask.reshape(-1).to(torch.uint8).contiguous()
        opt = {k: (_f32(rand[k]) if rand.get(k) is not None else None)
               for k in ("jitter", "u", "noise_scene_coarse", "noise_obj_coarse", "noise_scene_fine", "noise_obj_fine")}
        self._keep += [codes, mask, opt]
        a.rays, a.codes = self.rays.data_ptr(), _lib.ptr(codes)
        a.n_rays, a.n_samples, a.n_importance = n, n_samples, n_importance
        a.grid = C.pointer(grid.c) if grid is not None else None
        a.packed_coarse = packed_coarse.data_ptr()
        a.packed_fine = packed_fine.data_ptr() if packed_fine is not None else None
        a.precision = PRECISIONS[precision or default_precision()]
        a.use_disp, a.perturb, a.noise_std, a.seed = int(use_disp), float(perturb), float(noise_std), seed
        a.jitter, a.u = _lib.ptr(opt["jitter"]), _lib.ptr(opt["u"])
        a.noise_scene_coarse, a.noise_obj_coarse = _lib.ptr(opt["noise_scene_coarse"]), _lib.ptr(opt["noise_obj_coarse"])
        a.noise_scene_fine, a.noise_obj_fine = _lib.ptr(opt["noise_scene_fine"]), _lib.ptr(opt["noise_obj_fine"])
        a.white_back, a.forward_instance, a.is_eval = int(white_back), int(forward_instance), int(is_eval)
        a.zero_last_delta, a.rays_in_bbox = int(zero_last_delta), int(rays_in_bbox)
        a.frustum_bound_th = float(frustum_bound_th)
        a.pass_through_mask = _lib.ptr(mask)
        a.workspace, a.workspace_bytes = self.workspace.data_ptr(), self.workspace.numel()
        if train_ws is not None:
            a.train_ws, a.train_ws_bytes = train_ws.data_ptr(), train_ws.numel()
        self.args = a

    def run(self, seed_dev: Optional[torch.Tensor] = None):
        """Enqueue the forward on the current stream; returns the reference's result dict (views of the plan's buffers).
        seed_dev: a one-element int64 tensor on the plan's device holding the Philox seed; the draws then use the value it
        holds when the kernels run instead of args.seed, and the call adds 4 to it (onerf_render_rays_fwd_dseed), so
        every replay of a captured run draws fresh numbers."""
        if seed_dev is None:
            _lib.call("onerf_render_rays_fwd", self.rays.device, C.byref(self.args))
        else:
            if seed_dev.dtype != torch.int64 or seed_dev.numel() != 1 or seed_dev.device != self.rays.device:
                raise ValueError("seed_dev must be a one-element int64 tensor on the plan's device")
            _lib.call("onerf_render_rays_fwd_dseed", self.rays.device, C.byref(self.args), seed_dev.data_ptr())
        return {f"{k}_{typ}": v for typ, m in self.maps.items() for k, v in m.items()}
