"""CPU checks of onerf_render_instances (every object's maps in one render): its declarations, export and struct
layout, the workspace arithmetic, every refusal (no device needed: the checks run before any CUDA call), and that the
multi-code field kernel's wgmma stream is pipelined in the built library; and, where oracle/_ref is built, that the
reference's render_rays run once per code gives the columns of a float64 restatement that shares the samples."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from oracle import ref_loader as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = {
    "onerf_render_instances_workspace_bytes": ["int chunk_rays", "int n_codes", "int n_samples", "int n_importance"],
    "onerf_render_instances": ["onerf_ctx* ctx", "const onerf_instances_args* args", "void* stream"],
}


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def test_entries_are_exported_and_declared(lib):
    from object_nerf_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "onerf_ext.h")).read(), flags=re.S)
    decl = {m.group(1): [p.strip() for p in m.group(2).split(",")]
            for m in re.finditer(r"\b(onerf_[a-z0-9_]+)\s*\(([^)]*)\)", src)}
    for name, params in ENTRIES.items():
        assert decl[name] == params
        assert name in _lib.EXPORTS_EXT and name not in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == len(params)
    assert _lib.ABI_VERSION == 2 and lib.onerf_abi_version() == 2
    header = open(os.path.join(ROOT, "include", "onerf_ext.h")).read()
    assert int(re.search(r"#define ONERF_INSTANCES_MAX_CODES (\d+)", header).group(1)) == _lib.INSTANCES_MAX_CODES


@pytest.mark.parametrize("cls,cname", [("InstanceMaps", "onerf_instance_maps"),
                                       ("InstancesArgs", "onerf_instances_args")])
def test_struct_layout_matches_the_header(tmp_path, cls, cname):
    from object_nerf_b200 import _lib
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    cls = getattr(_lib, cls)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "onerf_ext.h"', "int main(void) {",
             f'printf("size %zu\\n", sizeof({cname}));']
    lines += [f'printf("{f[0]} %zu\\n", offsetof({cname}, {f[0]}));' for f in cls._fields_]
    lines.append("return 0; }")
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", str(tmp_path / "l")],
                   check=True)
    got = dict(line.rsplit(" ", 1) for line in subprocess.run([str(tmp_path / "l")], capture_output=True, text=True,
                                                              check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(cls)
    for f in cls._fields_:
        assert int(got[f[0]]) == getattr(cls, f[0]).offset, f[0]


def _a256(nbytes):
    return (nbytes + 255) // 256 * 256


def _ws_bytes(chunk, K, S, I):
    """The workspace layout restated: K per-ray-constant blocks, the scene's and K codes' field rows (S + I samples),
    both passes' depths and weights, and one chunk of scene maps."""
    SF, nf = S + I, chunk if I > 0 else 0
    floats = [K * chunk * 448, chunk * SF * 4, K * chunk * SF * 4, chunk * S, chunk * S, nf * SF, nf * SF,
              chunk * 3, chunk, chunk]
    return sum(_a256(4 * f) for f in floats)


@pytest.mark.parametrize("chunk,K,S,I", [(1, 1, 2, 0), (1000, 5, 64, 64), (4099, 64, 64, 64), (777, 2, 128, 0),
                                         (65536, 4, 64, 1984)])
def test_workspace_arithmetic(lib, chunk, K, S, I):
    assert lib.onerf_render_instances_workspace_bytes(chunk, K, S, I) == _ws_bytes(chunk, K, S, I)


def test_workspace_is_zero_for_a_bad_shape(lib):
    f = lib.onerf_render_instances_workspace_bytes
    for args in ((0, 1, 64, 0), (10, 0, 64, 0), (10, 65, 64, 0), (10, 1, 1, 0), (10, 1, 64, -1)):
        assert f(*args) == 0, args


def test_python_chunk_keeps_the_workspace_within_its_budget(lib):
    from object_nerf_b200 import rendering
    for K in (1, 4, 16, 64):
        c = rendering._instances_chunk(65536, K, 64, 64)
        assert 1 <= c <= 65536
        assert lib.onerf_render_instances_workspace_bytes(c, K, 64, 64) <= rendering.INSTANCES_WORKSPACE_BUDGET
        assert c == 65536 or lib.onerf_render_instances_workspace_bytes(c + 1, K, 64, 64) > \
            0.9 * rendering.INSTANCES_WORKSPACE_BUDGET


_IDS = (ctypes.c_int * 64)(*([3, 0, 7] + [1] * 61))


def _args(lib):
    """An argument block that passes every check; the pointers are never dereferenced by the refusals."""
    from object_nerf_b200 import _lib
    a = _lib.InstancesArgs()
    r = a.render
    r.rays, r.n_rays, r.n_samples, r.n_importance = 0x10000, 100, 64, 64
    r.packed_coarse, r.packed_fine, r.precision, r.is_eval = 0x10000, 0x10000, _lib.PREC_BF16, 1
    r.workspace_bytes = lib.onerf_render_instances_workspace_bytes(32, 3, 64, 64)
    r.workspace = 0x100000
    a.code_table, a.n_codes_table = 0x10000, 8
    a.ids_host, a.n_ids = ctypes.cast(_IDS, ctypes.POINTER(ctypes.c_int)), 3
    a.ray_begin, a.ray_end, a.chunk_rays = 10, 90, 32
    a.coarse.opacity_instance = a.fine.rgb_instance = 0x20000
    return a


def _grid():
    from object_nerf_b200 import _lib
    g = _lib.Grid()
    g.table, g.idx_map, g.voxel_offset, g.voxel_size, g.voxel_shape = 0x10000, 0x10000, 0x10000, 0x10000, 0x10000
    return g



def _set(a, path, value):
    obj, _, field = path.rpartition("__")
    setattr(getattr(a, obj) if obj else a, field, value)


@pytest.mark.parametrize("change,msg,rc", [
    ({"n_ids": 0}, b"n_ids outside", -1),
    ({"n_ids": 65}, b"n_ids outside", -1),
    ({"ids_host": None}, b"null ids_host", -1),
    ({"code_table": None}, b"null ids_host / code_table", -1),
    ({"n_codes_table": 7}, b"outside the code table", -1),
    ({"render__is_eval": 0}, b"is_eval", -1),
    ({"render__rays_in_bbox": 1}, b"rays_in_bbox", -2),
    ({"render__perturb": 1.0}, b"perturb", -1),
    ({"render__noise_std": 0.5}, b"noise_std", -1),
    ({"render__train_ws": 0x10000}, b"training workspace", -1),
    ({"render__n_samples": 1}, b"bad shape", -1),
    ({"render__n_importance": -1}, b"bad shape", -1),
    ({"render__n_importance": 1985}, b"S + K > 2048", -2),
    ({"ray_begin": -1}, b"tile outside", -1),
    ({"ray_end": 101}, b"tile outside", -1),
    ({"ray_begin": 50, "ray_end": 49}, b"tile outside", -1),
    ({"chunk_rays": 0}, b"chunk_rays", -1),
    ({"render__rays": None}, b"null rays", -1),
    ({"render__packed_coarse": None}, b"packed_coarse", -1),
    ({"render__packed_fine": None}, b"packed_fine", -1),
    ({"render__precision": 7}, b"unknown precision", -1),
    ({"render__n_importance": 0}, b"fine maps without a fine pass", -1),
    ({"coarse__rgb": 0x10002}, b"4-byte aligned", -1),
    ({"fine__depth_instance": 0x10001}, b"4-byte aligned", -1),
    ({"render__workspace": None}, b"256-byte aligned", -1),
    ({"render__workspace": 0x100010}, b"256-byte aligned", -1),
    ({"render__workspace_bytes": 1000}, b"workspace too small", -1),
])
def test_refusals(lib, change, msg, rc):
    a = _args(lib)
    for path, value in change.items():
        _set(a, path, value)
    assert lib.onerf_render_instances(ctypes.c_void_p(1), ctypes.byref(a), None) == rc
    err = lib.onerf_last_error()
    assert msg in err and err.startswith(b"onerf_render_instances:"), (change, err)


def test_null_context_args_and_grid_refusals(lib):
    a = _args(lib)
    assert lib.onerf_render_instances(None, ctypes.byref(a), None) == -1
    assert b"null argument" in lib.onerf_last_error()
    assert lib.onerf_render_instances(ctypes.c_void_p(1), None, None) == -1
    assert b"null argument" in lib.onerf_last_error()
    g = _grid()
    a.render.grid = ctypes.pointer(g)
    a.render.workspace_bytes = 1000            # everything but the grid passes up to the workspace size
    assert lib.onerf_render_instances(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
    assert b"workspace too small" in lib.onerf_last_error()
    for field, value in (("table", None), ("table", 0x10004), ("voxel_shape", None)):
        g2 = _grid()
        setattr(g2, field, value)
        a.render.grid = ctypes.pointer(g2)
        assert lib.onerf_render_instances(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
        assert b"grid buffer" in lib.onerf_last_error(), field


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
            cand = os.path.join(home, "bin", "cuobjdump") if home else None
            if cand and os.path.exists(cand):
                return cand
    return exe


def test_multi_code_kernel_wgmma_is_pipelined(lib):
    """As tests/test_sass_pipeline_cpu.py checks field_tc_kernel: both field_tc_multi_kernel instances wait with one
    wgmma group in flight and wait for all groups only about once per layer."""
    from object_nerf_b200 import _lib
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found (CUDA toolkit bin/ not on PATH): cannot disassemble the library")
    sass = subprocess.run([exe, "-sass", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    counts, fn = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1) if "field_tc_multi_kernel" in m.group(1) else None
            if fn:
                counts[fn] = {"hgmma": 0, "wait_all": 0, "wait_one": 0}
            continue
        if fn is None:
            continue
        c = counts[fn]
        c["hgmma"] += bool(re.search(r"\bHGMMA\.", line))
        c["wait_all"] += "WARPGROUP.DEPBAR.LE gsb0, 0x0" in line
        c["wait_one"] += "WARPGROUP.DEPBAR.LE gsb0, 0x1" in line
    assert len(counts) == 2, sorted(counts)
    for fn, c in counts.items():
        assert c["hgmma"] > 0 and c["wait_one"] > 0, (fn, c)
        assert 4 * c["wait_all"] <= c["hgmma"], (fn, c)


# ------------------------------------------------------------------------------------------------
# the reference itself: one render_rays per code against a float64 restatement that shares the samples
# ------------------------------------------------------------------------------------------------
def _restated_instances(w, rays, table, ids, n_samples, n_importance):
    """The render onerf_render_instances computes, restated in float64 with the oracle's stages: the coarse depths, the
    scene branch and its weights and the fine depths once, then the object branch and its compositing once per code."""
    from oracle import onerf_oracle as O
    n = rays.shape[0]
    o, d = rays[:, 0:3], rays[:, 3:6]
    out = {}

    def one_pass(typ, z):
        s = z.shape[1]
        xyz = (o[:, None, :] + d[:, None, :] * z[:, :, None]).reshape(-1, 3)
        dirs = d[:, None, :].expand(n, s, 3).reshape(-1, 3)
        f = O.field_eval(w[typ], None, xyz, dirs, None, want_object=False)
        _, wts = O.alpha_weights(f["sigma"].view(n, s), z, 1e10)
        maps = O.composite(wts, f["rgb"].view(n, s, 3), z, False)
        out[f"opacity_{typ}"], out[f"rgb_{typ}"], out[f"depth_{typ}"] = maps
        out[f"weights_{typ}"] = wts
        cols = []
        for i in ids:
            codes = table[i].expand(n * s, table.shape[1])
            g = O.field_eval(w[typ], None, xyz, dirs, codes, want_scene=False)
            _, wi = O.alpha_weights(g["inst_sigma"].view(n, s), z, 0.0)
            cols.append(O.composite(wi, g["inst_rgb"].view(n, s, 3), z, True))
        out[f"opacity_instance_{typ}"] = torch.stack([c[0] for c in cols], 1)
        out[f"rgb_instance_{typ}"] = torch.stack([c[1] for c in cols], 1)
        out[f"depth_instance_{typ}"] = torch.stack([c[2] for c in cols], 1)
        return wts

    z = O.stratified_z(rays, n_samples)
    wc = one_pass("coarse", z)
    mid = 0.5 * (z[:, :-1] + z[:, 1:])
    one_pass("fine", O.merge_sorted(z, O.sample_pdf(mid, wc[:, 1:-1], n_importance, det=True)))
    return out



@pytest.mark.skipif(not R.available(), reason="oracle/_ref not built (needs the reference checkout at build time)")
def test_reference_per_code_renders_equal_a_float64_restatement_sharing_the_samples():
    """The reference's render_rays(forward_instance=True, is_eval=True, perturb=0, noise_std=0, rays_in_bbox=False), run
    once per code, draws the same fine samples for every code (they follow the scene's coarse weights), and its columns
    are those of one float64 render that shares the samples and the scene branch and runs the object branch per code."""
    from object_nerf_b200 import synthetic as S
    R.install(cuda_noop=True)
    from models.embedding_helper import Embedding as RefEmbedding
    from models.nerf_model import ObjectNeRF as RefNeRF
    from models.rendering import render_rays as ref_render_rays
    n, n_samples, n_importance, ids = 48, 64, 32, [3, 9, 3, 0]
    w = {"coarse": S.make_weights(31, False, 8.0, 1.0), "fine": S.make_weights(1031, False, 8.0, 1.0)}
    models = {}
    for typ, wt in w.items():
        m = RefNeRF(S.model_config(False))
        m.load_state_dict({f"{S.REF_NAMES[k]}.{p}": t for k, (W, b) in wt.items()
                           for p, t in (("weight", W), ("bias", b))})
        models[typ] = m.eval()
    embeddings = {"xyz": RefEmbedding(3, 10), "dir": RefEmbedding(3, 4)}
    rays, table = S.random_rays(104, n).float(), S.make_codes(105)
    refs = {}
    with torch.no_grad():
        for i in dict.fromkeys(ids):
            refs[i] = ref_render_rays(models, embeddings, rays, N_samples=n_samples, N_importance=n_importance,
                                      perturb=0, noise_std=0, forward_instance=True, rays_in_bbox=False, is_eval=True,
                                      embedding_instance=table[i].expand(n, 64))
    first = refs[ids[0]]
    for r in refs.values():                   # the samples and the scene do not depend on the code
        for key in ("z_vals_coarse", "z_vals_fine", "weights_coarse", "rgb_fine", "depth_fine", "opacity_fine"):
            assert torch.equal(r[key], first[key]), key
    w64 = {t: {k: (W.double(), b.double()) for k, (W, b) in wt.items()} for t, wt in w.items()}
    got = _restated_instances(w64, rays.double(), table.double(), ids, n_samples, n_importance)
    for typ in ("coarse", "fine"):
        for kind in ("rgb", "depth", "opacity"):
            want = first[f"{kind}_{typ}"].double()
            assert torch.allclose(want, got[f"{kind}_{typ}"], rtol=1e-4, atol=1e-4), (typ, kind)
        for k, i in enumerate(ids):
            for kind in ("opacity_instance", "depth_instance", "rgb_instance"):
                ref, col = refs[i][f"{kind}_{typ}"].double(), got[f"{kind}_{typ}"][:, k]
                assert torch.allclose(ref, col, rtol=1e-4, atol=1e-4), (typ, k, kind, (ref - col).abs().max().item())
