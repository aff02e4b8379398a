"""CPU-side checks of the C-ABI boundary: the library builds, loads, and exports every symbol that
include/onerf.h declares; argument validation fails loudly without a GPU."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def declared_functions():
    src = open(os.path.join(ROOT, "include", "onerf.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(onerf_[a-z0-9_]+)\s*\(", src)))


def test_exports_every_declared_symbol(lib):
    names = declared_functions()
    assert len(names) >= 13
    for n in names:
        assert hasattr(lib, n), f"libonerf_sm90.so does not export {n}"
    from object_nerf_b200 import _lib
    assert sorted(_lib.EXPORTS) == names


def test_abi_version_and_sizes(lib):
    from object_nerf_b200 import _lib
    assert lib.onerf_abi_version() == _lib.ABI_VERSION == 2
    v, p = lib.onerf_packed_weights_bytes(1), lib.onerf_packed_weights_bytes(0)
    # fp32 section + bf16 stage images; see object_nerf_b200/csrc/layout.h
    assert v > p > 4 * 704840
    assert v % 1024 == 0 and p % 1024 == 0


def test_ctx_create_fails_loudly_without_device(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = ctypes.c_void_p()
    rc = lib.onerf_ctx_create(0, ctypes.byref(h))
    assert rc != 0
    assert len(lib.onerf_last_error()) > 0


def test_product_refuses_cpu_tensors():
    import torch
    from object_nerf_b200 import engine
    with pytest.raises(RuntimeError):
        engine.sample_coarse(torch.zeros(4, 8), 8)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "object_nerf_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            assert "oracle" not in open(os.path.join(pkg, fn)).read(), fn


def test_every_entry_point_rejects_a_null_context_with_a_message(lib):
    """No GPU needed: argument validation runs before any CUDA call.  Every compute entry point must return a negative
    status (never crash, never silently succeed) and leave a message in onerf_last_error()."""
    from object_nerf_b200 import _lib
    null = None
    z = ctypes.c_void_p(0)
    calls = {
        "onerf_pack_weights": (null, 1, None, None, z, 0, z),
        "onerf_sample_coarse": (null, z, 4, 8, 0, 0.0, z, 0, z, z),
        "onerf_sample_pdf_merge": (null, z, z, 4, 8, 8, 1, z, 0, z, z),
        "onerf_sample_pdf": (null, z, z, 4, 8, 8, 1, z, 0, z, z),
        "onerf_encode": (null, None, z, 4, z, z, z),
        "onerf_voxel_features": (null, None, z, 4, z, z),
        "onerf_field_fwd": (null, None, z),
        "onerf_composite": (null, None, z),
        "onerf_composite_multi": (null, z, z, 4, 2, 8, 0, z, z, z, z, z, z, z, z),
        "onerf_render_rays_fwd": (null, None, z),
        "onerf_ray_directions": (null, 4, 4, 1.0, z, z),
        "onerf_get_rays": (null, z, 4, None, z, z, z),
        "onerf_generate_rays": (null, z, z, 4, None, 1.0, 0.1, 1.0, z, z, z),
        "onerf_camera_rays": (null, 4, 4, 1.0, None, None, 1.0, 0.1, 1.0, z, z, z),
        "onerf_total_loss": (null, None, z),
        "onerf_composite_bwd": (null, None, z, z, z, z, z, z, z, z, z, z),
        "onerf_gemm": (null, z, 4, 0, z, 4, z, 4, 4, 4, 4, 0, z),
        "onerf_leaky_bwd": (null, z, 4, z, 4, 4, 4, z),
        "onerf_head_bwd": (null, z, z, z, 4, z),
        "onerf_segment_sum": (null, z, 4, z, 4, 4, 4, 4, z),
        "onerf_colsum": (null, z, 4, 4, 4, z, z),
        "onerf_dir_encode": (null, z, 4, z, z),
        "onerf_encode_bwd": (null, None, z, z, 4, 4, z, z, 4, 0, 4, z, z),
        "onerf_render_rays_bwd": (null, None, None, z),
        "onerf_unpack_grads": (null, 1, z, None, None, z),
        "onerf_bwd_chain": (null, 1, 1, z, z, 128, z, z, z),
        "onerf_bwd_wgrad": (null, 1, 1, z, 128, z, z),
        "onerf_bwd_colsums": (null, 1, 1, z, 128, z, z, z, z),
        "onerf_bwd_raysums": (null, 1, 1, z, 2, 64, z, z),
        "onerf_bwd_dx": (null, 1, z, z, z, z, 2, 64, None, z, z),
        "onerf_code_gather": (null, z, z, 4, 64, z, z),
        "onerf_code_scatter_add": (null, z, z, 4, 64, z, z),
        "onerf_render_multi_fwd": (null, None, z),
    }
    helpers = {"onerf_abi_version", "onerf_last_error", "onerf_ctx_create", "onerf_ctx_destroy", "onerf_ctx_launch_count",
               "onerf_packed_weights_bytes", "onerf_render_rays_workspace_bytes", "onerf_total_loss_workspace_bytes",
               "onerf_field_train_bytes", "onerf_train_workspace_bytes", "onerf_grad_buffer_floats",
               "onerf_render_multi_workspace_bytes"}
    assert set(calls) | helpers == set(_lib.EXPORTS)
    for name, args in calls.items():
        rc = getattr(lib, name)(*args)
        assert rc < 0, name
        assert len(lib.onerf_last_error()) > 0, name
    assert lib.onerf_render_rays_workspace_bytes(1024, 64, 64) >= 1024 * (448 * 4 + 2 * 128 * 16)
    assert lib.onerf_total_loss_workspace_bytes() >= 16 * 8
    # training workspace: 104 operand tiles of 16 KB + 45 KB of masks per 128 samples, for both passes
    per_tile = 104 * 16384 + 88 * 128 * 4
    assert lib.onerf_field_train_bytes(1, 128 * 10) >= 10 * per_tile
    assert lib.onerf_train_workspace_bytes(1, 2048, 64, 64) >= (1024 + 2048) * per_tile
    assert lib.onerf_grad_buffer_floats(1) >= 891208 - 27 * 192 - 64 * 256


def test_train_workspace_bytes_for_either_precision(lib):
    """onerf_train_workspace_bytes_prec: 0 for an unknown precision or a bad shape; bf16 = onerf_train_workspace_bytes;
    fp32 = both passes' fields and field gradients, the directions' PE and one backward chunk (<= 65 536 samples of whole
    rays): 17 activation matrices, d(X), two 256-wide buffers, head gradients, fields, ray_const and per-ray sums."""
    from object_nerf_b200 import _lib
    f = lib.onerf_train_workspace_bytes_prec
    for prec in (_lib.PREC_FP32, _lib.PREC_BF16):
        assert f(prec, 1, -1, 64, 64) == 0 and f(prec, 1, 4, 0, 64) == 0 and f(prec, 0, 4, 64, -1) == 0
    assert f(2, 1, 4, 64, 64) == 0 and f(-1, 0, 4, 64, 64) == 0
    a1k = lambda x: (x + 1023) // 1024 * 1024
    tail = [256] * 8 + [256, 128] + [128] * 4 + [128, 64]
    for uv in (0, 1):
        for n, s, si in ((1, 2, 0), (41, 64, 32), (2048, 64, 128), (4096, 64, 0), (2, 70000, 0), (0, 64, 64)):
            assert f(_lib.PREC_BF16, uv, n, s, si) == lib.onerf_train_workspace_bytes(uv, n, s, si)
            sf = s + si
            rays = lambda S: min(n, max(1, 65536 // S))
            R, B = max(rays(s), rays(sf)), max(rays(s) * s, rays(sf) * sf)
            ko = 384 if uv else 64
            want = (2 * a1k(n * s * 16) + 4 * a1k(n * sf * 16) + a1k(R * 128 * 4) + a1k(n * 27 * 4)
                    + 2 * a1k(B * ko * 4) + sum(a1k(B * w * 4) for w in tail) + 2 * a1k(B * 256 * 4) + 3 * a1k(B * 16)
                    + a1k(R * 448 * 4))
            assert f(_lib.PREC_FP32, uv, n, s, si) == want, (uv, n, s, si)
