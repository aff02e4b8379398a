"""ctypes binding of libonerf_sm90.so (the C ABI declared in include/onerf.h).

There is no fallback: if the shared library is missing or the device is not sm_90 every entry point
raises.  PyTorch is used only for device memory and streams.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ONERF_LIB_PATH") or os.path.join(_HERE, "libonerf_sm90.so")   # override: A/B experiments
CSRC = os.path.join(_HERE, "csrc")

PREC_FP32, PREC_BF16 = 0, 1
ABI_VERSION = 2
RAY_CONST_FLOATS = 448
N_LINEAR = 20

EXPORTS = [
    "onerf_abi_version", "onerf_last_error", "onerf_ctx_create", "onerf_ctx_destroy",
    "onerf_ctx_launch_count", "onerf_packed_weights_bytes", "onerf_pack_weights", "onerf_sample_coarse",
    "onerf_sample_pdf_merge", "onerf_sample_pdf", "onerf_encode", "onerf_voxel_features", "onerf_field_fwd", "onerf_composite", "onerf_composite_multi",
    "onerf_render_rays_workspace_bytes", "onerf_render_rays_fwd",
    "onerf_ray_directions", "onerf_get_rays", "onerf_generate_rays", "onerf_camera_rays",
    "onerf_total_loss_workspace_bytes", "onerf_total_loss",
    "onerf_composite_bwd", "onerf_gemm", "onerf_leaky_bwd", "onerf_head_bwd", "onerf_segment_sum", "onerf_colsum",
    "onerf_dir_encode", "onerf_encode_bwd",
    "onerf_field_train_bytes", "onerf_train_workspace_bytes", "onerf_render_rays_bwd", "onerf_grad_buffer_floats",
    "onerf_unpack_grads", "onerf_bwd_chain", "onerf_bwd_wgrad", "onerf_bwd_colsums", "onerf_bwd_raysums", "onerf_bwd_dx",
    "onerf_code_gather", "onerf_code_scatter_add", "onerf_render_multi_workspace_bytes", "onerf_render_multi_fwd",
]
# additions to ABI version 2 declared in include/onerf_ext.h
EXPORTS_EXT = ["onerf_composite_multi_workspace_bytes", "onerf_composite_multi_ws", "onerf_composite_multi_merge",
               "onerf_train_workspace_bytes_prec", "onerf_train_step_workspace_bytes", "onerf_train_step",
               "onerf_render_rays_fwd_dseed", "onerf_train_step_dseed"]

_p = C.c_void_p


class Grid(C.Structure):
    _fields_ = [("table", _p), ("idx_map", _p), ("voxel_offset", _p), ("voxel_size", _p), ("voxel_shape", _p)]


class FieldArgs(C.Structure):
    _fields_ = [
        ("rays", _p), ("xyz", _p), ("z", _p), ("z_stride", C.c_int64), ("codes", _p), ("code_row", _p),
        ("n_rays", C.c_int), ("n_samples", C.c_int), ("grid", C.POINTER(Grid)), ("packed", _p),
        ("want_scene", C.c_int), ("want_object", C.c_int), ("precision", C.c_int),
        ("mute_zero_rays", C.c_int), ("boxes", _p), ("n_boxes", C.c_int),
        ("scene_out", _p), ("obj_out", _p), ("out_stride", C.c_int64), ("ray_const", _p),
        ("activations", C.POINTER(_p)), ("train_ws", _p),
    ]


class CompositeArgs(C.Structure):
    _fields_ = [
        ("z", _p), ("scene", _p), ("obj", _p), ("n_rays", C.c_int), ("n_samples", C.c_int),
        ("noise_std", C.c_float), ("noise_scene", _p), ("noise_obj", _p), ("seed", C.c_uint64),
        ("white_back", C.c_int), ("is_eval", C.c_int), ("zero_last_delta", C.c_int), ("rays_in_bbox", C.c_int),
        ("frustum_bound_th", C.c_float), ("pass_through_mask", _p),
        ("weights", _p), ("opacity", _p), ("rgb", _p), ("depth", _p),
        ("rgb_instance", _p), ("depth_instance", _p), ("opacity_instance", _p),
    ]


class LossMaps(C.Structure):
    _fields_ = [("rgb", _p), ("depth", _p), ("opacity_instance", _p), ("rgb_instance", _p), ("depth_instance", _p)]


class LossArgs(C.Structure):
    _fields_ = [
        ("n_rays", C.c_int64), ("has_fine", C.c_int), ("coarse", LossMaps), ("fine", LossMaps), ("rgbs", _p), ("depths", _p),
        ("valid_mask", _p), ("instance_mask", _p), ("instance_mask_weight", _p), ("color_weight", C.c_float),
        ("depth_weight", C.c_float), ("opacity_weight", C.c_float), ("instance_color_weight", C.c_float),
        ("instance_depth_weight", C.c_float), ("grad_coarse", LossMaps), ("grad_fine", LossMaps), ("loss_sum_out", _p),
        ("terms_out", _p), ("present_out", _p), ("workspace", _p),
    ]


class BoxHost(C.Structure):
    _fields_ = [("pose_avg", C.c_double * 16), ("axis_align", C.c_double * 16), ("bounds", C.c_double * 6)]


class RenderMaps(C.Structure):
    _fields_ = [("weights", _p), ("opacity", _p), ("z_vals", _p), ("rgb", _p), ("depth", _p),
                ("rgb_instance", _p), ("depth_instance", _p), ("opacity_instance", _p)]


class RenderArgs(C.Structure):
    _fields_ = [
        ("rays", _p), ("codes", _p), ("n_rays", C.c_int), ("n_samples", C.c_int), ("n_importance", C.c_int),
        ("grid", C.POINTER(Grid)), ("packed_coarse", _p), ("packed_fine", _p), ("precision", C.c_int),
        ("use_disp", C.c_int), ("perturb", C.c_float), ("noise_std", C.c_float), ("seed", C.c_uint64),
        ("jitter", _p), ("u", _p), ("noise_scene_coarse", _p), ("noise_obj_coarse", _p), ("noise_scene_fine", _p),
        ("noise_obj_fine", _p), ("white_back", C.c_int), ("forward_instance", C.c_int), ("is_eval", C.c_int),
        ("zero_last_delta", C.c_int), ("rays_in_bbox", C.c_int), ("frustum_bound_th", C.c_float),
        ("pass_through_mask", _p), ("coarse", RenderMaps), ("fine", RenderMaps), ("workspace", _p),
        ("workspace_bytes", C.c_size_t), ("train_ws", _p), ("train_ws_bytes", C.c_size_t),
    ]


class RenderMultiMaps(C.Structure):
    _fields_ = [("weights", _p), ("opacity", _p), ("z_vals", _p), ("rgb", _p), ("depth", _p), ("obj_ids", _p)]


class RenderMultiArgs(C.Structure):
    _fields_ = [
        ("rays_list_host", C.POINTER(_p)), ("obj_ids_host", C.POINTER(C.c_int)), ("n_obj", C.c_int), ("n_rays", C.c_int),
        ("n_samples", C.c_int), ("n_importance", C.c_int), ("grid", C.POINTER(Grid)), ("packed_coarse", _p),
        ("packed_fine", _p), ("code_table", _p), ("n_codes", C.c_int), ("precision", C.c_int), ("use_disp", C.c_int),
        ("perturb", C.c_float), ("seed", C.c_uint64), ("white_back", C.c_int), ("boxes", _p), ("n_boxes", C.c_int),
        ("coarse", RenderMultiMaps), ("fine", RenderMultiMaps), ("workspace", _p), ("workspace_bytes", C.c_size_t),
    ]


class MapGrads(C.Structure):
    _fields_ = [("rgb", _p), ("depth", _p), ("opacity", _p), ("rgb_instance", _p), ("depth_instance", _p),
                ("opacity_instance", _p)]


class RenderBwdArgs(C.Structure):
    _fields_ = [("coarse", MapGrads), ("fine", MapGrads), ("W_coarse", C.POINTER(_p)), ("W_fine", C.POINTER(_p)),
                ("dW_coarse", C.POINTER(_p)), ("db_coarse", C.POINTER(_p)), ("dW_fine", C.POINTER(_p)),
                ("db_fine", C.POINTER(_p)), ("d_codes", _p), ("table_grad", _p)]


def build(verbose: bool = False) -> str:
    """Compile the CUDA sources for sm_90a into libonerf_sm90.so (nvcc cross-compiles without a GPU)."""
    r = subprocess.run(["make", "-C", CSRC, "-j8"], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout[-4000:])
        print(r.stderr[-4000:])
    if r.returncode != 0:
        raise RuntimeError("building libonerf_sm90.so failed")
    return LIB_PATH


_lib = None
_lock = threading.Lock()


def load() -> C.CDLL:
    """dlopen the library and declare signatures.  Raises if it has not been built."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU or PyTorch fallback for the render path)")
        lib = C.CDLL(LIB_PATH)
        # ABI version 2 grows by additions only (include/onerf_ext.h): a library built before an addition has the right
        # version but lacks the symbol
        missing = [name for name in EXPORTS + EXPORTS_EXT if not hasattr(lib, name)]
        if missing:
            raise RuntimeError(f"{LIB_PATH} predates these entry points: {', '.join(missing)}; rebuild it "
                               "(`python -c 'import __graft_entry__ as g; g.build()'`)")
        lib.onerf_abi_version.restype = C.c_int
        lib.onerf_last_error.restype = C.c_char_p
        lib.onerf_ctx_create.argtypes = [C.c_int, C.POINTER(_p)]
        lib.onerf_ctx_destroy.argtypes = [_p]
        lib.onerf_ctx_launch_count.argtypes = [_p]
        lib.onerf_ctx_launch_count.restype = C.c_int64
        lib.onerf_packed_weights_bytes.argtypes = [C.c_int]
        lib.onerf_packed_weights_bytes.restype = C.c_size_t
        lib.onerf_pack_weights.argtypes = [_p, C.c_int, C.POINTER(_p), C.POINTER(_p), _p, C.c_size_t, _p]
        lib.onerf_sample_coarse.argtypes = [_p, _p, C.c_int, C.c_int, C.c_int, C.c_float, _p, C.c_uint64, _p, _p]
        lib.onerf_sample_pdf_merge.argtypes = [_p, _p, _p, C.c_int, C.c_int, C.c_int, C.c_int, _p, C.c_uint64, _p, _p]
        lib.onerf_sample_pdf.argtypes = [_p, _p, _p, C.c_int, C.c_int, C.c_int, C.c_int, _p, C.c_uint64, _p, _p]
        lib.onerf_encode.argtypes = [_p, C.POINTER(Grid), _p, C.c_int64, _p, _p, _p]
        lib.onerf_voxel_features.argtypes = [_p, C.POINTER(Grid), _p, C.c_int64, _p, _p]
        lib.onerf_field_fwd.argtypes = [_p, C.POINTER(FieldArgs), _p]
        lib.onerf_composite.argtypes = [_p, C.POINTER(CompositeArgs), _p]
        lib.onerf_render_rays_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        lib.onerf_render_rays_workspace_bytes.restype = C.c_size_t
        lib.onerf_render_rays_fwd.argtypes = [_p, C.POINTER(RenderArgs), _p]
        lib.onerf_ray_directions.argtypes = [_p, C.c_int, C.c_int, C.c_float, _p, _p]
        lib.onerf_get_rays.argtypes = [_p, _p, C.c_int64, C.POINTER(C.c_float), _p, _p, _p]
        lib.onerf_generate_rays.argtypes = [_p, _p, _p, C.c_int64, C.POINTER(BoxHost), C.c_double, C.c_double, C.c_double, _p, _p, _p]
        lib.onerf_camera_rays.argtypes = [_p, C.c_int, C.c_int, C.c_float, C.POINTER(C.c_float), C.POINTER(BoxHost), C.c_double,
                                          C.c_double, C.c_double, _p, _p, _p]
        lib.onerf_total_loss_workspace_bytes.restype = C.c_size_t
        lib.onerf_total_loss.argtypes = [_p, C.POINTER(LossArgs), _p]
        lib.onerf_composite_multi.argtypes = [_p, _p, _p, C.c_int, C.c_int, C.c_int, C.c_int, _p, _p, _p, _p, _p, _p, _p, _p]
        lib.onerf_composite_bwd.argtypes = [_p, C.POINTER(CompositeArgs), _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]
        lib.onerf_gemm.argtypes = [_p, _p, C.c_int, C.c_int, _p, C.c_int, _p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _p]
        lib.onerf_leaky_bwd.argtypes = [_p, _p, C.c_int, _p, C.c_int, C.c_int64, C.c_int, _p]
        lib.onerf_head_bwd.argtypes = [_p, _p, _p, _p, C.c_int64, _p]
        lib.onerf_segment_sum.argtypes = [_p, _p, C.c_int, _p, C.c_int, C.c_int, C.c_int, C.c_int, _p]
        lib.onerf_colsum.argtypes = [_p, _p, C.c_int, C.c_int64, C.c_int, _p, _p]
        lib.onerf_dir_encode.argtypes = [_p, _p, C.c_int, _p, _p]
        lib.onerf_encode_bwd.argtypes = [_p, C.POINTER(Grid), _p, _p, C.c_int, C.c_int, _p, _p, C.c_int, C.c_int64, C.c_int64, _p, _p]
        lib.onerf_field_train_bytes.argtypes = [C.c_int, C.c_int64]
        lib.onerf_field_train_bytes.restype = C.c_size_t
        lib.onerf_train_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
        lib.onerf_train_workspace_bytes.restype = C.c_size_t
        lib.onerf_render_rays_bwd.argtypes = [_p, C.POINTER(RenderArgs), C.POINTER(RenderBwdArgs), _p]
        lib.onerf_grad_buffer_floats.argtypes = [C.c_int]
        lib.onerf_grad_buffer_floats.restype = C.c_size_t
        lib.onerf_unpack_grads.argtypes = [_p, C.c_int, _p, C.POINTER(_p), C.POINTER(_p), _p]
        lib.onerf_bwd_chain.argtypes = [_p, C.c_int, C.c_int, _p, _p, C.c_int64, _p, _p, _p]
        lib.onerf_bwd_wgrad.argtypes = [_p, C.c_int, C.c_int, _p, C.c_int64, _p, _p]
        lib.onerf_bwd_colsums.argtypes = [_p, C.c_int, C.c_int, _p, C.c_int64, _p, _p, _p, _p]
        lib.onerf_bwd_raysums.argtypes = [_p, C.c_int, C.c_int, _p, C.c_int, C.c_int, _p, _p]
        lib.onerf_bwd_dx.argtypes = [_p, C.c_int, _p, _p, _p, _p, C.c_int, C.c_int, C.POINTER(Grid), _p, _p]
        lib.onerf_code_gather.argtypes = [_p, _p, _p, C.c_int, C.c_int, _p, _p]
        lib.onerf_code_scatter_add.argtypes = [_p, _p, _p, C.c_int, C.c_int, _p, _p]
        lib.onerf_render_multi_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
        lib.onerf_render_multi_workspace_bytes.restype = C.c_size_t
        lib.onerf_render_multi_fwd.argtypes = [_p, C.POINTER(RenderMultiArgs), _p]
        lib.onerf_composite_multi_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        lib.onerf_composite_multi_workspace_bytes.restype = C.c_size_t
        for name in ("onerf_composite_multi_ws", "onerf_composite_multi_merge"):
            getattr(lib, name).argtypes = lib.onerf_composite_multi.argtypes[:-1] + [_p, C.c_size_t, _p]
        lib.onerf_train_workspace_bytes_prec.argtypes = [C.c_int] * 5
        lib.onerf_train_workspace_bytes_prec.restype = C.c_size_t
        lib.onerf_train_step_workspace_bytes.argtypes = [C.c_int] * 5
        lib.onerf_train_step_workspace_bytes.restype = C.c_size_t
        lib.onerf_train_step.argtypes = [_p, C.POINTER(RenderArgs), C.POINTER(LossArgs), C.POINTER(RenderBwdArgs), _p, _p]
        lib.onerf_render_rays_fwd_dseed.argtypes = [_p, C.POINTER(RenderArgs), _p, _p]
        lib.onerf_train_step_dseed.argtypes = [_p, C.POINTER(RenderArgs), C.POINTER(LossArgs), C.POINTER(RenderBwdArgs), _p,
                                               _p, _p]
        if lib.onerf_abi_version() != ABI_VERSION:
            raise RuntimeError("libonerf_sm90.so ABI version mismatch")
        _lib = lib
        return lib


def check(rc: int):
    if rc != 0:
        raise RuntimeError(f"libonerf_sm90 error {rc}: {load().onerf_last_error().decode()}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL).  The tensor must be contiguous."""
    if t is None:
        return None
    assert t.is_contiguous(), "non-contiguous tensor passed to the C ABI"
    return t.data_ptr()


_ctx = {}


def ctx(device: torch.device):
    """One library context per (process, device)."""
    if device.type != "cuda":
        raise RuntimeError("object_nerf_b200 runs on CUDA (sm_90a) devices only; got tensor on " + str(device))
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _ctx:
        h = _p()
        check(load().onerf_ctx_create(idx, C.byref(h)))
        _ctx[idx] = h
    return _ctx[idx]


def stream():
    return torch.cuda.current_stream().cuda_stream


def launch_count(device: torch.device) -> int:
    return int(load().onerf_ctx_launch_count(ctx(device)))
