"""CPU side of the device batch sampler (include/onerf_ext.h: onerf_draw_batch, object_nerf_b200/batches.py): a numpy
restatement of the epoch permutation and the instance-column draw, their properties (bijection, independence of epochs
and seeds, shuffle quality, disjoint DDP strides), the exports and argument checks of the two entries, and RaySampler's
refusals before any CUDA call.  tests/test_gpu_batches.py compares the kernel with this restatement bit for bit."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests.test_train_stages_cpu import _MASK, _key, philox4x32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROUNDS, PERM_STREAM, COLUMN_STREAM = 6, 5, 4


def half_bits(R):
    """Half the bit width of the Feistel domain: m is the smallest even m >= 2 with 2^m >= R."""
    m = 2
    while (1 << m) < R:
        m += 2
    return m // 2


def feistel(x, half, seed, epoch):
    x = np.asarray(x, dtype=np.uint64)
    mask = np.uint64((1 << half) - 1)
    L, R = x >> np.uint64(half), x & mask
    key = _key(seed, x.size)
    for rnd in range(ROUNDS):
        ctr = np.stack([R, np.full_like(R, epoch & 0xFFFFFFFF), np.full_like(R, PERM_STREAM), np.full_like(R, rnd)], -1)
        f = philox4x32(ctr, key)[:, 0].astype(np.uint64) & mask
        L, R = R, L ^ f
    return (L << np.uint64(half)) | R


def permute(p, R, seed, epoch):
    """pi_{seed,epoch}(p) for positions p < R: the Feistel network applied until the value falls in [0, R)."""
    x = np.asarray(p, dtype=np.uint64).copy()
    half = half_bits(R)
    todo = np.ones(x.shape, dtype=bool)
    while todo.any():
        x[todo] = feistel(x[todo], half, seed, epoch)
        todo &= x >= np.uint64(R)
    return x.astype(np.int64)


def column(seed, n, I):
    """Instance column (w * I) >> 32 for element indices n (uint64): w = word n & 3 of Philox stream 4 at n >> 2."""
    n = np.asarray(n, dtype=np.uint64)
    ctr = np.stack([(n >> np.uint64(2)) & _MASK, n >> np.uint64(34), np.full_like(n, COLUMN_STREAM),
                    np.zeros_like(n)], -1)
    r = philox4x32(ctr, _key(seed, n.size))
    w = np.take_along_axis(r, (n & np.uint64(3)).astype(np.int64)[:, None], 1)[:, 0].astype(np.uint64)
    return ((w * np.uint64(I)) >> np.uint64(32)).astype(np.int64)


def draw_indices(R, I, B, W, rank, seed, step):
    """(ray, column) of every element of batch `step` on rank `rank`, as onerf_draw_batch draws them."""
    P = R // (B * W)
    epoch, j = divmod(step, P)
    b = np.arange(B, dtype=np.uint64)
    with np.errstate(over="ignore"):
        pos = (np.uint64(j * B) + b) * np.uint64(W) + np.uint64(rank)
        n = (np.uint64(step) * np.uint64(B) + b) * np.uint64(W) + np.uint64(rank)
    return permute(pos, R, seed, epoch), column(seed, n, I)


SEED = 0x0123_4567_89AB_CDEF


@pytest.mark.parametrize("R", [1, 2, 3, 4, 5, 17, 1000, 65537, (1 << 20) + 3])
def test_permutation_is_a_bijection(R):
    for epoch in (0, 7):
        pi = permute(np.arange(R), R, SEED, epoch)
        assert pi.min() >= 0 and pi.max() < R
        assert np.array_equal(np.sort(pi), np.arange(R)), (R, epoch)


def test_feistel_domain():
    assert [half_bits(R) for R in (1, 2, 4, 5, 16, 17, 1 << 20, (1 << 20) + 1)] == [1, 1, 1, 2, 2, 3, 10, 11]
    for R in (5, 17, 1000, 65537):
        assert (1 << 2 * half_bits(R)) < 4 * R


def test_epochs_and_seeds_give_different_permutations():
    R = 1000
    p = np.arange(R)
    base = permute(p, R, SEED, 0)
    for other in (permute(p, R, SEED, 1), permute(p, R, SEED, 2), permute(p, R, SEED + 1, 0), permute(p, R, 1, 0)):
        assert (other != base).mean() > 0.9


def test_shuffle_displacement_matches_a_uniform_shuffle():
    """E|pi(p) - p| / R = 1/3 for a uniform random permutation (R large)."""
    R = 100_000
    for seed, epoch in ((SEED, 0), (SEED, 3), (12345, 0)):
        d = np.abs(permute(np.arange(R), R, seed, epoch) - np.arange(R)).mean() / R
        assert abs(d - 1 / 3) <= 0.02 / 3, (seed, epoch, d)


@pytest.mark.parametrize("W", [2, 3])
def test_ranks_draw_disjoint_strides_of_one_epoch(W):
    R, B = 10_007, 64
    P = R // (B * W)
    for epoch in (0, 1):
        rays = [draw_indices(R, 2, B, W, r, SEED, epoch * P + j)[0] for r in range(W) for j in range(P)]
        allr = np.concatenate(rays)
        assert allr.size == P * B * W and np.unique(allr).size == P * B * W
        per_rank = [set(np.concatenate(rays[r * P:(r + 1) * P]).tolist()) for r in range(W)]
        for a in range(W):
            for b in range(a + 1, W):
                assert not per_rank[a] & per_rank[b]


def test_columns_cover_every_instance_and_differ_by_rank():
    ray0, col0 = draw_indices(5000, 3, 2048, 2, 0, SEED, 0)
    ray1, col1 = draw_indices(5000, 3, 2048, 2, 1, SEED, 0)
    assert set(col0.tolist()) == {0, 1, 2} and (col0 != col1).mean() > 0.5
    assert draw_indices(5000, 1, 2048, 2, 0, SEED, 0)[1].max() == 0


# ---------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def _ext_declarations():
    src = open(os.path.join(ROOT, "include", "onerf_ext.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return {m.group(1): [p.strip() for p in m.group(2).split(",")]
            for m in re.finditer(r"\b(onerf_[a-z0-9_]+)\s*\(([^)]*)\)", src)}


def test_entries_are_exported_and_declared(lib):
    from object_nerf_b200 import _lib
    decl = _ext_declarations()
    assert decl["onerf_draw_batch"] == ["onerf_ctx* ctx", "const onerf_batch_args* args", "void* stream"]
    assert decl["onerf_draw_batch_dstep"] == ["onerf_ctx* ctx", "const onerf_batch_args* args", "uint64_t* step_dev",
                                              "void* stream"]
    for name in ("onerf_draw_batch", "onerf_draw_batch_dstep"):
        assert name in _lib.EXPORTS_EXT and name not in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == len(decl[name])


def test_struct_layout_matches_the_header(tmp_path):
    """Field offsets and sizes of onerf_ray_dataset / onerf_batch_args as the C compiler lays them out."""
    from object_nerf_b200 import _lib
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    structs = {"onerf_ray_dataset": _lib.RayDataset, "onerf_batch_args": _lib.BatchArgs}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "onerf_ext.h"', "int main(void) {"]
    for cname, cls in structs.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for f in cls._fields_:
            lines.append(f'printf("{cname}.{f[0]} %zu\\n", offsetof({cname}, {f[0]}));')
    lines.append("return 0; }")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.rsplit(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True,
                                                              check=True).stdout.splitlines())
    for cname, cls in structs.items():
        assert int(got[cname]) == ctypes.sizeof(cls), cname
        for f in cls._fields_:
            assert int(got[f"{cname}.{f[0]}"]) == getattr(cls, f[0]).offset, (cname, f[0])


def _valid_args():
    """An argument block that passes every check; its device pointers are never dereferenced by the refusals."""
    from object_nerf_b200 import _lib
    a = _lib.BatchArgs()
    d = a.data
    d.n_rays, d.n_instances = 10_000, 2
    for k in ("rays", "rgbs", "depths", "valid_mask", "instance_mask", "instance_mask_weight", "instance_ids",
              "pass_through_mask"):
        setattr(d, k, 0x10000)
        setattr(a, k, 0x20000)
    a.batch, a.rank, a.world = 2048, 0, 2
    return a


@pytest.mark.parametrize("mutate,msg", [
    (lambda a: setattr(a.data, "rays", None), b"null dataset buffer"),
    (lambda a: setattr(a.data, "pass_through_mask", None), b"null dataset buffer"),
    (lambda a: setattr(a, "instance_ids", None), b"null output buffer"),
    (lambda a: setattr(a, "depths", None), b"null output buffer"),
    (lambda a: setattr(a, "batch", 0), b"batch must be >= 1"),
    (lambda a: setattr(a, "world", 0), b"world must be >= 1"),
    (lambda a: setattr(a, "rank", 2), b"rank outside"),
    (lambda a: setattr(a, "rank", -1), b"rank outside"),
    (lambda a: setattr(a.data, "n_instances", 0), b"n_instances"),
    (lambda a: setattr(a.data, "n_rays", 4095), b"no full batch"),
    (lambda a: setattr(a.data, "n_rays", 1 << 40), b"2^40"),
])
def test_refusals(lib, mutate, msg):
    a = _valid_args()
    mutate(a)
    ctx = ctypes.c_void_p(1)
    assert lib.onerf_draw_batch(ctx, ctypes.byref(a), None) == -1
    assert msg in lib.onerf_last_error() and lib.onerf_last_error().startswith(b"onerf_draw_batch:")
    assert lib.onerf_draw_batch_dstep(ctx, ctypes.byref(a), 0x1000, None) == -1
    assert msg in lib.onerf_last_error() and lib.onerf_last_error().startswith(b"onerf_draw_batch_dstep:")


def test_null_ctx_and_step_pointer(lib):
    a = _valid_args()
    assert lib.onerf_draw_batch(None, ctypes.byref(a), None) == -1
    assert b"null" in lib.onerf_last_error()
    assert lib.onerf_draw_batch_dstep(None, ctypes.byref(a), 0x1000, None) == -1
    assert b"null" in lib.onerf_last_error()
    assert lib.onerf_draw_batch(ctypes.c_void_p(1), None, None) == -1
    ctx = ctypes.c_void_p(1)
    assert lib.onerf_draw_batch_dstep(ctx, ctypes.byref(a), None, None) == -1
    assert b"null step_dev" in lib.onerf_last_error()
    assert lib.onerf_draw_batch_dstep(ctx, ctypes.byref(a), 0x1004, None) == -1
    assert b"8-byte aligned" in lib.onerf_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# RaySampler: checks that run before any upload
# ---------------------------------------------------------------------------------------------------------------------
def dataset(R, I, frame=True):
    g = torch.Generator().manual_seed(R)
    cols = (R, I) if I is not None else (R,)
    t = {"all_rays": torch.rand(R, 8, generator=g), "all_rgbs": torch.rand(R, 3, generator=g),
         "all_depths": torch.rand(R, generator=g), "all_valid_masks": torch.rand(R, generator=g) < 0.8,
         "all_instance_masks": torch.rand(cols, generator=g) < 0.5,
         "all_instance_masks_weight": torch.rand(cols, generator=g),
         "all_instance_ids": torch.randint(0, 64, cols, generator=g),
         "all_pass_through_masks": torch.rand(cols, generator=g) < 0.5}
    if frame:
        t["all_frame_indices"] = torch.arange(R) // 100
    return t


@pytest.fixture
def no_cuda(monkeypatch):
    """Any device transfer fails the test: the refusals come first."""
    def fail(*a, **k):
        pytest.fail("RaySampler touched a device before refusing")
    monkeypatch.setattr(torch.Tensor, "to", fail)
    monkeypatch.setattr(torch.cuda, "current_device", fail)


def test_sampler_refusals(no_cuda):
    from object_nerf_b200 import RaySampler
    t = dataset(5000, 2)
    for k in ("all_rgbs", "all_depths", "all_valid_masks", "all_instance_masks", "all_instance_ids",
              "all_frame_indices"):
        bad = dict(t)
        bad[k] = t[k][:-1]
        with pytest.raises(ValueError, match="rows"):
            RaySampler(bad, batch_size=1024, device="cuda:0")
    bad = dict(t)
    bad["all_instance_ids"] = t["all_instance_ids"][:, :1]
    with pytest.raises(ValueError, match="instance columns"):
        RaySampler(bad, batch_size=1024, device="cuda:0")
    zero = dataset(5000, 0)
    with pytest.raises(ValueError, match="I = 0"):
        RaySampler(zero, batch_size=1024, device="cuda:0")
    with pytest.raises(ValueError, match="no full batch"):
        RaySampler(t, batch_size=2048, world_size=3, rank=0, device="cuda:0")
    with pytest.raises(ValueError, match="no full batch"):
        RaySampler(t, batch_size=5001, device="cuda:0")
    with pytest.raises(ValueError, match="rank"):
        RaySampler(t, batch_size=1024, world_size=2, rank=2, device="cuda:0")
    missing = dict(t)
    del missing["all_depths"]
    with pytest.raises(ValueError, match="all_depths"):
        RaySampler(missing, batch_size=1024, device="cuda:0")


def test_from_dataset_reads_the_generic_dataset_attributes(monkeypatch):
    from object_nerf_b200 import batches
    seen = {}

    def fake_init(self, tensors, **kw):
        seen.update(tensors=tensors, kw=kw)
    monkeypatch.setattr(batches.RaySampler, "__init__", fake_init)

    class DS:
        pass
    ds = DS()
    for k, v in dataset(100, 2).items():
        setattr(ds, k, v)
    batches.RaySampler.from_dataset(ds, batch_size=10, seed=3)
    assert set(seen["tensors"]) == set(batches.DATASET_KEYS) | {"all_frame_indices"}
    assert seen["kw"] == {"batch_size": 10, "seed": 3}
    del ds.all_frame_indices
    batches.RaySampler.from_dataset(ds)
    assert set(seen["tensors"]) == set(batches.DATASET_KEYS)
