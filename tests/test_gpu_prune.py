"""-m gpu: voxel pruning on the device (EmbeddingVoxel.self_pruning_empty_voxels -> onerf_prune_measure /
onerf_prune_apply, include/onerf_ext.h).

  - fp32 with the fixture's injected jitter reproduces the reference-generated grids bit for bit, through the method and
    through measure + apply called directly;
  - the fused bf16 pass gives per-voxel maxima bit-identical to the staged bf16 route (points built in torch in the
    reference's op order, rendering.query_sigma(precision="bf16"), torch alpha and max), on the maintenance case and on a
    2 000-voxel shard of the bench grid;
  - the Philox jitter is the documented mapping (the host restatement of tests/test_train_stages_cpu.py), in fp32 and
    bf16, also for sample indices past 2^31;
  - shapes: no occupied voxel, one voxel, an empty shard, voxels on the grid's edge;
  - two gloo ranks on one GPU with group= end with identical grids, equal to the single-process call's, and a grouped
    train_step still asks for sync_replicas after the pruning."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import cases, helpers
from tests.test_host_logic_cpu import _maint_embedding
from tests.test_train_stages_cpu import philox_uniform

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
S = 4096
TH = cases.MAINT_CASE["max_alpha_th"]


def _maint():
    emb, inp = _maint_embedding()
    return emb.to(DEV), helpers.make_model(inp["weights"], True, DEV)


def _bench():
    from object_nerf_b200 import synthetic as Syn
    import bench
    sc = bench.build_scene()
    return Syn.make_embedding(sc["grid"]).to(DEV), helpers.make_model(sc["weights"]["fine"], True, DEV)


def _measure(emb, model, cells, begin, end, precision, jitter=None, seed=0):
    """onerf_prune_measure on the shard [begin, end) of `cells` -> (end - begin,) max alpha."""
    from object_nerf_b200 import _lib, engine
    lib = _lib.load()
    prec = engine.PRECISIONS[precision]
    out = torch.full((end - begin,), 7.0, dtype=torch.float32, device=DEV)     # the call zeroes it first
    ws = torch.empty(max(lib.onerf_prune_workspace_bytes(prec), 256), dtype=torch.uint8, device=DEV)
    grid = emb.grid_buffers()
    cells = cells.contiguous()
    jitter = jitter.contiguous() if jitter is not None else None
    a = _lib.PruneArgs()
    a.grid, a.packed, a.precision = C.pointer(grid.c), engine.packed_for(model, True).data_ptr(), prec
    a.cells, a.n_cells, a.cell_begin, a.cell_end = cells.data_ptr(), cells.shape[0], begin, end
    a.jitter, a.seed, a.max_alpha_out = _lib.ptr(jitter), seed, out.data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    _lib.check(lib.onerf_prune_measure(_lib.ctx(DEV), C.byref(a), _lib.stream()))
    torch.cuda.synchronize()
    return out


def _staged(emb, model, cells, jitter_rows, precision="bf16"):
    """The route before the fused pass: points in torch with the reference's op order (embedding_helper.py:96, 116),
    query_sigma, torch alpha and per-voxel max.  jitter_rows (len(cells) * 4096, 3)."""
    from object_nerf_b200 import rendering
    centres = cells.float() * emb.voxel_size - emb.voxel_offset
    samples = centres[:, None, :].expand(-1, S, -1).reshape(-1, 3).clone()
    samples += jitter_rows * emb.voxel_size - emb.voxel_size / 2
    sigma = rendering.query_sigma(model, emb, samples, precision=precision)
    alpha = 1 - torch.exp(-torch.relu(sigma))
    return alpha.view(-1, S).max(-1)[0]


def _bits(t):
    return t.contiguous().view(torch.int32)


def _philox_rows(seed, k0, k1):
    """The documented jitter of voxels [k0, k1): component c of row k * 4096 + s is element (k * 4096 + s) * 3 + c of
    Philox stream 6."""
    idx = np.arange(k0 * S * 3, k1 * S * 3, dtype=np.int64)
    return torch.from_numpy(philox_uniform(seed, 6, idx).reshape(-1, 3))


# ------------------------------------------------------------------------------------------------
# 1. fp32 against the reference-generated fixture
# ------------------------------------------------------------------------------------------------
def test_fp32_method_matches_reference_golden(golden):
    gold = golden("maint_pruning")
    emb, model = _maint()
    n = int(gold["n_before"])
    rand = [r.to(DEV) for r in cases.maint_rand((n + 31) // 32)]
    pruned = emb.self_pruning_empty_voxels(model, max_alpha_th=TH, precision="fp32", _rand=rand)
    assert pruned == n - int(gold["pruned|voxel_occupancy"].sum())
    assert torch.equal(emb.voxel_occupancy.cpu(), gold["pruned|voxel_occupancy"].bool())
    assert torch.equal(emb.voxel_idx_map.cpu(), gold["pruned|voxel_idx_map"])


def test_fp32_measure_and_apply_match_reference_golden(golden):
    from object_nerf_b200 import _lib
    gold = golden("maint_pruning")
    emb, model = _maint()
    cells = torch.nonzero(emb.voxel_occupancy).contiguous()
    n = cells.shape[0]
    jitter = torch.cat(cases.maint_rand((n + 31) // 32))[:n * S].to(DEV)
    max_alpha = _measure(emb, model, cells, 0, n, "fp32", jitter)
    count = torch.full((1,), -5, dtype=torch.int64, device=DEV)
    occ, idx = emb.voxel_occupancy, emb.voxel_idx_map
    _lib.check(_lib.load().onerf_prune_apply(_lib.ctx(DEV), cells.data_ptr(), n, max_alpha.data_ptr(), TH, occ.shape[1],
                                             occ.shape[2], occ.data_ptr(), idx.data_ptr(), count.data_ptr(), _lib.stream()))
    assert int(count.item()) == n - int(gold["pruned|voxel_occupancy"].sum())
    assert torch.equal(occ.cpu(), gold["pruned|voxel_occupancy"].bool())
    assert torch.equal(idx.cpu(), gold["pruned|voxel_idx_map"])


# ------------------------------------------------------------------------------------------------
# 2. fused bf16 pass against the staged bf16 route
# ------------------------------------------------------------------------------------------------
def test_bf16_fused_pass_equals_staged_route_on_maintenance_case():
    emb, model = _maint()
    cells = torch.nonzero(emb.voxel_occupancy).contiguous()
    n = cells.shape[0]
    jitter = torch.cat(cases.maint_rand((n + 31) // 32))[:n * S].to(DEV)
    got = _measure(emb, model, cells, 0, n, "bf16", jitter)
    want = _staged(emb, model, cells, jitter)
    assert torch.equal(_bits(got), _bits(want)), (got - want).abs().max().item()
    assert (got > 0).any() and (got < 1).any()


def test_bf16_fused_pass_equals_staged_route_on_bench_grid_shard():
    emb, model = _bench()
    cells = torch.nonzero(emb.voxel_occupancy).contiguous()
    n = cells.shape[0]
    a, b = n // 3, n // 3 + 2000
    g = torch.Generator(device=DEV).manual_seed(11)
    jitter = torch.zeros(n * S, 3, device=DEV)
    jitter[a * S:b * S] = torch.rand(2000 * S, 3, device=DEV, generator=g)
    got = _measure(emb, model, cells, a, b, "bf16", jitter)
    want = _staged(emb, model, cells[a:b], jitter[a * S:b * S])
    assert torch.equal(_bits(got), _bits(want)), (got - want).abs().max().item()
    assert got.unique().numel() > 100


# ------------------------------------------------------------------------------------------------
# 3. the Philox mapping
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_seeded_jitter_is_the_documented_philox_mapping(precision):
    emb, model = _maint()
    cells = torch.nonzero(emb.voxel_occupancy).contiguous()
    n = cells.shape[0]
    seed = 0x5EED_1234_ABCD
    a, b = 5, 12
    jitter = torch.zeros(n * S, 3)
    jitter[a * S:b * S] = _philox_rows(seed, a, b)
    got = _measure(emb, model, cells, a, b, precision, seed=seed)
    want = _measure(emb, model, cells, a, b, precision, jitter.to(DEV))
    assert torch.equal(_bits(got), _bits(want))
    assert not torch.equal(got, _measure(emb, model, cells, a, b, precision, seed=seed + 1))


def test_seeded_jitter_past_2_pow_31_samples():
    """K = 600 000 cells (occupied cells repeated): rows of the last 40 voxels are indexed past 2^31 (and their jitter
    elements past 2^32); a jitter buffer that size would be 29 GB, so the seeded pass is checked against the staged route
    fed with the host's Philox rows."""
    emb, model = _maint()
    occ = torch.nonzero(emb.voxel_occupancy)
    K = 600_000
    cells = occ[torch.arange(K, device=DEV) % occ.shape[0]]
    assert (K - 40) * S * 3 > 2 ** 32
    seed = 987654321
    got = _measure(emb, model, cells, K - 40, K, "bf16", seed=seed)
    want = _staged(emb, model, cells[K - 40:], _philox_rows(seed, K - 40, K).to(DEV))
    assert torch.equal(_bits(got), _bits(want))


# ------------------------------------------------------------------------------------------------
# 4. shapes
# ------------------------------------------------------------------------------------------------
def test_no_occupied_voxel_launches_nothing():
    from object_nerf_b200 import _lib
    emb, model = _maint()
    emb.voxel_occupancy.zero_()
    before = emb.voxel_idx_map.clone()
    launches = _lib.launch_count(DEV)
    assert emb.self_pruning_empty_voxels(model, max_alpha_th=TH) == 0
    assert _lib.launch_count(DEV) == launches
    assert torch.equal(emb.voxel_idx_map, before) and not emb.voxel_occupancy.any()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_one_voxel_and_an_empty_shard(precision):
    emb, model = _maint()
    cells = torch.nonzero(emb.voxel_occupancy)[3:4]
    jitter = torch.rand(S, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    got = _measure(emb, model, cells, 0, 1, precision, jitter)
    want = _staged(emb, model, cells, jitter, precision)
    if precision == "bf16":
        assert torch.equal(_bits(got), _bits(want))
    else:
        assert torch.allclose(got, want, rtol=0, atol=1e-6)
    assert _measure(emb, model, cells, 1, 1, precision, jitter).numel() == 0


def test_voxels_on_the_grid_edge():
    """Cells on the grid's corners and faces: samples outside the grid read zero features, as the reference's."""
    emb, model = _maint()
    X, Y, Z = emb.voxel_shape.tolist()
    cells = torch.tensor([[0, 0, 0], [X - 1, Y - 1, Z - 1], [0, Y - 1, Z // 2], [X - 1, 0, 0]], device=DEV)
    jitter = torch.rand(4 * S, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    got = _measure(emb, model, cells, 0, 4, "bf16", jitter)
    assert torch.equal(_bits(got), _bits(_staged(emb, model, cells, jitter)))
    got32 = _measure(emb, model, cells, 0, 4, "fp32", jitter)
    assert torch.allclose(got32, _staged(emb, model, cells, jitter, "fp32"), rtol=0, atol=1e-6)


def test_seeded_method_is_reproducible_under_manual_seed():
    grids = []
    for _ in range(2):
        emb, model = _maint()
        torch.manual_seed(123)
        n = emb.self_pruning_empty_voxels(model, max_alpha_th=TH, precision="bf16")
        grids.append((n, emb.voxel_idx_map.clone()))
    assert grids[0][0] == grids[1][0] and torch.equal(grids[0][1], grids[1][1])


# ------------------------------------------------------------------------------------------------
# 5-6. two gloo ranks on one GPU
# ------------------------------------------------------------------------------------------------
def _gloo_worker(rank, world, port, ret):
    import torch.distributed as dist

    from tests.test_gpu_train_ddp import _batch, _kwargs, _setup
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(DEV)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from object_nerf_b200 import training
        res = {}
        for name in ("rand", "seed"):
            emb, model = _maint()
            n = int(emb.voxel_occupancy.sum())
            kw = dict(_rand=[r.to(DEV) for r in cases.maint_rand((n + 31) // 32)]) if name == "rand" else dict(seed=4242)
            pruned = emb.self_pruning_empty_voxels(model, max_alpha_th=TH, precision="bf16", group=dist.group.WORLD, **kw)
            res[name] = (pruned, emb.voxel_occupancy.cpu(), emb.voxel_idx_map.cpu())
        # rank 1's own seed is ignored: rank 0's is broadcast
        emb, model = _maint()
        emb.self_pruning_empty_voxels(model, max_alpha_th=TH, precision="bf16", group=dist.group.WORLD, seed=4242 + rank)
        res["rank_seed"] = emb.voxel_idx_map.cpu()

        # a grouped train_step after a grouped pruning
        from tests import cases as tc
        inp = tc.build_grad_case(96)
        mine = slice(rank * 48, rank * 48 + 48)
        emb, minp = _maint_embedding()
        emb = emb.to(DEV)
        models, embeddings, lib = _setup(inp, DEV, emb)
        training.sync_replicas(models, embeddings, lib, dist.group.WORLD)
        kw = _kwargs(inp, mine, DEV, "bf16")
        batch = _batch(inp, mine, DEV)
        training.train_step(models, embeddings, lib, batch, tc.LOSS_CONF, group=dist.group.WORLD, **kw)
        emb.self_pruning_empty_voxels(helpers.make_model(minp["weights"], True, DEV), max_alpha_th=TH,
                                      group=dist.group.WORLD, seed=77)
        try:
            training.train_step(models, embeddings, lib, batch, tc.LOSS_CONF, group=dist.group.WORLD, **kw)
            res["refusal"] = None
        except RuntimeError as e:
            res["refusal"] = str(e)
        training.sync_replicas(models, embeddings, lib, dist.group.WORLD)
        loss = training.train_step(models, embeddings, lib, batch, tc.LOSS_CONF, group=dist.group.WORLD, **kw)[0]
        res["after_sync"] = bool(torch.isfinite(loss).all())
        torch.cuda.synchronize()
        ret[rank] = res
    finally:
        dist.destroy_process_group()


@pytest.fixture(scope="module")
def gloo():
    from tests.test_gpu_train_ddp import _spawn
    return _spawn(_gloo_worker, 2)


@pytest.mark.parametrize("name", ["rand", "seed"])
def test_grouped_pruning_leaves_identical_grids_equal_to_one_process(gloo, name):
    emb, model = _maint()
    n = int(emb.voxel_occupancy.sum())
    kw = dict(_rand=[r.to(DEV) for r in cases.maint_rand((n + 31) // 32)]) if name == "rand" else dict(seed=4242)
    pruned = emb.self_pruning_empty_voxels(model, max_alpha_th=TH, precision="bf16", **kw)
    assert 0 < pruned < n
    for rank, res in gloo.items():
        got_n, occ, idx = res[name]
        assert got_n == pruned, rank
        assert torch.equal(occ, emb.voxel_occupancy.cpu()) and torch.equal(idx, emb.voxel_idx_map.cpu()), rank
    assert torch.equal(gloo[0]["rank_seed"], gloo[1]["rank_seed"])
    assert torch.equal(gloo[0]["rank_seed"], gloo[0]["seed"][2])


def test_grouped_train_step_still_asks_for_sync_after_grouped_pruning(gloo):
    for rank, res in gloo.items():
        assert res["refusal"] is not None and "grid changed" in res["refusal"], (rank, res["refusal"])
        assert res["after_sync"], rank
