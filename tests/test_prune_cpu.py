"""CPU checks of the device pruning pass (include/onerf_ext.h: onerf_prune_workspace_bytes, onerf_prune_measure,
onerf_prune_apply; EmbeddingVoxel.self_pruning_empty_voxels): the entry points are exported as declared and refuse bad
arguments before any CUDA call, the method's host logic with the library stubbed (cells in torch.nonzero order, the
injected jitter concatenated, shard bounds, seed, the apply mask), two gloo ranks gathering their shards on the CPU, and
the compiled fused kernel's wgmma pipelining."""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch

from tests import cases
from tests.test_graph_rng_cpu import _ext_declarations
from tests.test_sass_pipeline_cpu import LIB
from tests.test_train_step_cpu import _FakeLib

S = 4096
TH = cases.MAINT_CASE["max_alpha_th"]


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def test_entry_points_are_exported_and_declared(lib):
    from object_nerf_b200 import _lib
    decl = _ext_declarations()
    assert decl["onerf_prune_workspace_bytes"] == ["int precision"]
    assert decl["onerf_prune_measure"] == ["onerf_ctx* ctx", "const onerf_prune_args* args", "void* stream"]
    assert decl["onerf_prune_apply"] == [
        "onerf_ctx* ctx", "const int64_t* cells", "int64_t n_cells", "const float* max_alpha", "float max_alpha_th",
        "int64_t dim_y", "int64_t dim_z", "uint8_t* occupancy", "int64_t* idx_map", "int64_t* n_pruned", "void* stream"]
    for name in decl:
        if name.startswith("onerf_prune"):
            assert name in _lib.EXPORTS_EXT and hasattr(lib, name), name
            assert len(getattr(lib, name).argtypes) == len(decl[name]), name
    header = open(os.path.join(os.path.dirname(LIB), "..", "include", "onerf_ext.h")).read()
    assert f"#define ONERF_PRUNE_SAMPLES {_lib.PRUNE_SAMPLES}\n" in header
    assert [f for f, _ in _lib.PruneArgs._fields_] == [
        "grid", "packed", "precision", "cells", "n_cells", "cell_begin", "cell_end", "jitter", "seed", "max_alpha_out",
        "workspace", "workspace_bytes"]


def test_workspace_is_one_fp32_chunk_and_nothing_for_bf16(lib):
    from object_nerf_b200 import _lib
    a256 = lambda x: (x + 255) // 256 * 256
    pts = 32 * S
    want = a256(pts * 12) + a256(pts * 4) + a256(32) + a256(448 * 4) + a256(pts * 16)
    assert lib.onerf_prune_workspace_bytes(_lib.PREC_FP32) == want
    assert lib.onerf_prune_workspace_bytes(_lib.PREC_BF16) == 0
    assert lib.onerf_prune_workspace_bytes(7) == 0 and lib.onerf_prune_workspace_bytes(-1) == 0


def test_refusals_come_before_any_cuda_call(lib):
    from object_nerf_b200 import _lib
    ctx = ctypes.c_void_p(1)
    grid = _lib.Grid(0x10000, 0x1000, 0x1000, 0x1000, 0x1000)

    def good(prec=_lib.PREC_FP32):
        a = _lib.PruneArgs()
        a.grid, a.packed, a.precision = ctypes.pointer(grid), 0x1000, prec
        a.cells, a.n_cells, a.cell_begin, a.cell_end = 0x1000, 10, 2, 8
        a.max_alpha_out = 0x2000
        a.workspace, a.workspace_bytes = 0x10000, lib.onerf_prune_workspace_bytes(_lib.PREC_FP32)
        return a

    def refused(message, code=-1, prec=_lib.PREC_FP32, **change):
        a = good(prec)
        for field, value in change.items():
            setattr(a, field, value)
        assert lib.onerf_prune_measure(ctx, ctypes.byref(a), None) == code, change
        assert message in lib.onerf_last_error(), (change, lib.onerf_last_error())

    assert lib.onerf_prune_measure(None, None, None) == -1 and b"null" in lib.onerf_last_error()
    assert lib.onerf_prune_measure(ctx, None, None) == -1
    refused(b"voxel model", grid=None)
    bad = _lib.Grid(0x10000, None, 0x1000, 0x1000, 0x1000)
    refused(b"grid buffer", grid=ctypes.pointer(bad))
    refused(b"packed", packed=None)
    refused(b"unknown precision", precision=2)
    refused(b"shard", cell_begin=-1)
    refused(b"shard", cell_end=11)
    refused(b"shard", cell_begin=5, cell_end=4)
    refused(b"shard", n_cells=-1, cell_begin=0, cell_end=0)
    refused(b"null cells", cells=None)
    refused(b"null max_alpha_out", max_alpha_out=None)
    refused(b"8-byte aligned", cells=0x1004)
    refused(b"4-byte aligned", jitter=0x1002)
    refused(b"4-byte aligned", max_alpha_out=0x2002)
    refused(b"256-byte aligned", workspace=None)
    refused(b"256-byte aligned", workspace=0x10010)
    refused(b"workspace too small", code=-4, workspace_bytes=good().workspace_bytes - 1)
    # bf16 needs no workspace; an empty shard (K = 0 included) needs no cells or output, and returns before any CUDA call
    a = good(_lib.PREC_BF16)
    a.workspace, a.workspace_bytes = None, 0
    a.cells, a.n_cells, a.cell_begin, a.cell_end, a.max_alpha_out = None, 0, 0, 0, None
    assert lib.onerf_prune_measure(ctx, ctypes.byref(a), None) == 0
    a.cells, a.n_cells, a.cell_begin, a.cell_end = 0x1000, 10, 4, 4
    assert lib.onerf_prune_measure(ctx, ctypes.byref(a), None) == 0

    args = [ctx, 0x1000, 10, 0x2000, 0.5, 4, 4, 0x3000, 0x4000, 0x5000, None]

    def apply_refused(message, **change):
        a = list(args)
        names = ["ctx", "cells", "n_cells", "max_alpha", "th", "dim_y", "dim_z", "occupancy", "idx_map", "n_pruned"]
        for k, v in change.items():
            a[names.index(k)] = v
        assert lib.onerf_prune_apply(*a) == -1, change
        assert message in lib.onerf_last_error(), (change, lib.onerf_last_error())

    apply_refused(b"null argument", ctx=None)
    apply_refused(b"null argument", occupancy=None)
    apply_refused(b"null argument", idx_map=None)
    apply_refused(b"null argument", n_pruned=None)
    apply_refused(b"null cells", cells=None)
    apply_refused(b"null cells", max_alpha=None)
    apply_refused(b"bad shape", n_cells=-1)
    apply_refused(b"bad shape", dim_y=0)
    apply_refused(b"bad shape", dim_z=0)
    apply_refused(b"misaligned", cells=0x1004)
    apply_refused(b"misaligned", idx_map=0x4004)
    apply_refused(b"misaligned", n_pruned=0x5004)
    apply_refused(b"misaligned", max_alpha=0x2002)


# ------------------------------------------------------------------------------------------------
# the method's host logic, library stubbed
# ------------------------------------------------------------------------------------------------
def _alpha_of(cell):
    """A per-voxel value the stub reports: a fixed function of the cell, about half of them below TH."""
    i, j, l = (int(v) for v in cell)
    return ((i * 7 + j * 13 + l * 29) % 10) / 10.0 * (2 * TH)


class _FakePruneLib(_FakeLib):
    def onerf_prune_workspace_bytes(self, prec):
        return 512 if prec == 0 else 0

    def onerf_prune_measure(self, ctx, a, stream):
        a = a._obj
        n, b, e = a.n_cells, a.cell_begin, a.cell_end
        cells = self.view(a.cells, 3 * n, ctypes.c_int64).reshape(n, 3).copy()
        jitter = self.view(a.jitter, 3 * n * S).reshape(-1, 3).copy() if a.jitter else None
        self.calls.append(("measure", dict(cells=cells, shard=(b, e), seed=a.seed, jitter=jitter, prec=a.precision,
                                           grid=bool(a.grid), ws=a.workspace_bytes)))
        if e > b:
            self.view(a.max_alpha_out, e - b)[:] = [_alpha_of(c) for c in cells[b:e]]
        return 0

    def onerf_prune_apply(self, ctx, cells, n, max_alpha, th, dim_y, dim_z, occ, idx, n_pruned, stream):
        c = self.view(cells, 3 * n, ctypes.c_int64).reshape(n, 3)
        m = self.view(max_alpha, n)
        self.calls.append(("apply", m.copy(), th, dim_y, dim_z))
        o = self.view(occ, self.numel, ctypes.c_uint8)
        ix = self.view(idx, self.numel, ctypes.c_int64)
        drop = m < np.float32(th)
        lin = (c[drop, 0] * dim_y + c[drop, 1]) * dim_z + c[drop, 2]
        o[lin], ix[lin] = 0, -1
        self.view(n_pruned, 1, ctypes.c_int64)[0] = int(drop.sum())
        return 0


def _stub(monkeypatch, emb):
    import contextlib

    from object_nerf_b200 import _lib
    fake = _FakePruneLib()
    fake.numel = emb.voxel_idx_map.numel()
    monkeypatch.setattr(_lib, "load", lambda: fake)
    monkeypatch.setattr(_lib, "ctx", lambda dev: None)
    monkeypatch.setattr(_lib, "stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    return fake


def _problem():
    from object_nerf_b200 import synthetic as Syn
    from tests.test_host_logic_cpu import _maint_embedding
    emb, inp = _maint_embedding()
    return emb, Syn.make_model(inp["weights"], True, "cpu")


def _expected(emb):
    """The grid after pruning every cell whose _alpha_of is below TH."""
    occ, idx = emb.voxel_occupancy.clone(), emb.voxel_idx_map.clone()
    cells = torch.nonzero(occ)
    drop = [c for c in cells.tolist() if np.float32(_alpha_of(c)) < np.float32(TH)]
    for i, j, l in drop:
        occ[i, j, l], idx[i, j, l] = False, -1
    return len(drop), occ, idx


def test_method_plumbing_with_the_library_stubbed(monkeypatch):
    from object_nerf_b200 import _lib, engine
    emb, model = _problem()
    fake = _stub(monkeypatch, emb)
    n_want, occ_want, idx_want = _expected(emb)
    cells = torch.nonzero(emb.voxel_occupancy)
    K = cells.shape[0]
    monkeypatch.setattr(engine, "new_seed", lambda: 0xABCDEF)
    version = emb.voxel_idx_map._version
    assert emb.self_pruning_empty_voxels(model, max_alpha_th=TH, precision="fp32") == n_want
    assert 0 < n_want < K
    assert torch.equal(emb.voxel_occupancy, occ_want) and torch.equal(emb.voxel_idx_map, idx_want)
    assert emb.voxel_idx_map._version > version                 # training._grid_stamp sees the change
    assert [c[0] for c in fake.calls] == ["pack", "measure", "apply"]
    m = fake.calls[1][1]
    assert np.array_equal(m["cells"], cells.numpy()) and m["shard"] == (0, K) and m["seed"] == 0xABCDEF
    assert m["jitter"] is None and m["prec"] == _lib.PREC_FP32 and m["grid"] and m["ws"] >= 512
    _, alpha, th, dy, dz = fake.calls[2]
    assert np.array_equal(alpha, np.array([_alpha_of(c) for c in cells.tolist()], dtype=np.float32))
    assert th == pytest.approx(TH) and (dy, dz) == tuple(emb.voxel_occupancy.shape[1:])


def test_injected_jitter_is_the_concatenated_chunks(monkeypatch):
    emb, model = _problem()
    fake = _stub(monkeypatch, emb)
    K = int(emb.voxel_occupancy.sum())
    rand = cases.maint_rand((K + 31) // 32 + 1)                 # one block too many: ignored
    emb.self_pruning_empty_voxels(model, max_alpha_th=TH, precision="bf16", _rand=rand, seed=5)
    m = fake.calls[1][1]
    want = torch.cat([r[:min(32, K - 32 * i) * S] for i, r in enumerate(rand[:(K + 31) // 32])]).numpy()
    assert np.array_equal(m["jitter"], want) and m["seed"] == 0 and m["prec"] == 1 and m["ws"] == 0
    with pytest.raises(ValueError, match="jitter rows"):
        emb.self_pruning_empty_voxels(model, max_alpha_th=TH, _rand=[r[:100] for r in rand])


def test_no_occupied_voxel_calls_nothing(monkeypatch):
    emb, model = _problem()
    fake = _stub(monkeypatch, emb)
    emb.voxel_occupancy.zero_()
    assert emb.self_pruning_empty_voxels(model) == 0 and fake.calls == []


def test_sharded_method_measures_its_shard_and_applies_the_gathered_mask(monkeypatch):
    import torch.distributed as dist

    from object_nerf_b200 import parallel
    emb, model = _problem()
    fake = _stub(monkeypatch, emb)
    n_want, occ_want, idx_want = _expected(emb)
    K = int(emb.voxel_occupancy.sum())
    sent = []
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 1)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 3)
    monkeypatch.setattr(dist, "broadcast", lambda t, group_src=None, group=None: (sent.append(int(t.item())), t.fill_(31))[1])
    cells = torch.nonzero(emb.voxel_occupancy)
    full = torch.tensor([_alpha_of(c) for c in cells.tolist()], dtype=torch.float32)
    monkeypatch.setattr(parallel, "gather_tiles", lambda local, n, group=None: (sent.append(("gather", local.clone(), n)), full)[1])
    assert emb.self_pruning_empty_voxels(model, max_alpha_th=TH, seed=9, group=object()) == n_want
    b, e = parallel.shard_bounds(K, 3, 1)
    m = fake.calls[1][1]
    assert m["shard"] == (b, e) and m["seed"] == 31 and sent[0] == 9
    assert sent[1][2] == K and torch.equal(sent[1][1], full[b:e])
    assert torch.equal(emb.voxel_occupancy, occ_want) and torch.equal(emb.voxel_idx_map, idx_want)
    with pytest.raises(ValueError, match="group"):
        emb.self_pruning_empty_voxels(model, _sigma_fn=lambda p: p[:, 0], group=object())


# ------------------------------------------------------------------------------------------------
# two gloo ranks, library stubbed
# ------------------------------------------------------------------------------------------------
def _gloo_worker(rank, world, port, ret):
    import torch.distributed as dist

    from object_nerf_b200 import _lib
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import contextlib
        emb, model = _problem()
        fake = _FakePruneLib()
        fake.numel = emb.voxel_idx_map.numel()
        _lib.load, _lib.ctx, _lib.stream = (lambda: fake), (lambda dev: None), (lambda: None)
        torch.cuda.device = lambda dev: contextlib.nullcontext()
        n = emb.self_pruning_empty_voxels(model, max_alpha_th=TH, seed=100 + rank, group=dist.group.WORLD)
        m = fake.calls[1][1]
        ret[rank] = (n, m["shard"], m["seed"], emb.voxel_occupancy.clone(), emb.voxel_idx_map.clone())
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_apply_the_same_gathered_mask():
    import torch.multiprocessing as mp

    from object_nerf_b200 import parallel
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    emb, _ = _problem()
    n_want, occ_want, idx_want = _expected(emb)
    K = int(emb.voxel_occupancy.sum())
    for rank in range(2):
        n, shard, seed, occ, idx = ret[rank]
        assert n == n_want and shard == parallel.shard_bounds(K, 2, rank) and seed == 100
        assert torch.equal(occ, occ_want) and torch.equal(idx, idx_want)
