"""CPU checks of data-parallel train_step (training.train_step(group=...), training.sync_replicas) with the library
stubbed: the gradient bucket's layout and the `.grad` views into it, the all-reduced prefix for the voxel and the plain
model, the per-rank seeds, every refusal, and sync_replicas over a two-process gloo group."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_graph_rng_cpu import _problem, _stubbed


class _FakeDist:
    """Stands in for torch.distributed's rank queries and collectives: all_reduce multiplies by the world size (W ranks
    holding identical gradients), broadcast keeps the local values."""

    def __init__(self, monkeypatch, rank=0, world=2):
        self.rank, self.world, self.reduced, self.broadcasts = rank, world, [], 0
        monkeypatch.setattr(dist, "get_rank", lambda group=None: self.rank)
        monkeypatch.setattr(dist, "get_world_size", lambda group=None: self.world)
        monkeypatch.setattr(dist, "all_reduce", self.all_reduce)
        monkeypatch.setattr(dist, "broadcast", self.broadcast)

    def all_reduce(self, t, op=None, group=None):
        assert op == dist.ReduceOp.SUM
        self.reduced.append((t.data_ptr(), t.numel()))
        t.mul_(self.world)

    def broadcast(self, t, group_src=None, group=None):
        assert group_src == 0
        self.broadcasts += 1


GROUP = object()


def _plain_problem():
    from object_nerf_b200 import Embedding
    from object_nerf_b200 import synthetic as S
    from tests import grad_plain, helpers
    inp = grad_plain.build_grad_case_plain()
    models = {k: S.make_model(w, False, "cpu") for k, w in inp["weights"].items()}
    batch = {k: v.clone() for k, v in inp["batch"].items()}
    batch["rays"], batch["instance_ids"] = inp["rays"], inp["instance_ids"]
    kw = dict(N_samples=64, N_importance=64, perturb=1.0, noise_std=1.0, pass_through_mask=inp["pass_through_mask"],
              frustum_bound_th=0.025, precision="bf16")
    return models, {"xyz": Embedding(3, 10), "dir": None}, helpers.CodeLib(inp["code_table"]), batch, kw


def _expected_layout(models, lib, emb):
    from object_nerf_b200 import engine
    tensors = [t for typ in ("fine", "coarse") for pair in engine.model_linears(models[typ]) for t in pair]
    tensors.append(lib.embedding_instance.weight)
    if emb is not None:
        tensors.append(emb.embedding_space_ftr.weight)
    offsets, off = [], 0
    for t in tensors:
        offsets.append(off)
        off += (t.numel() + 3) // 4 * 4
    return tensors, offsets, off


@pytest.mark.parametrize("use_voxel", [True, False])
def test_bucket_layout_views_and_reduced_prefix(monkeypatch, use_voxel):
    """Fine model's 40 tensors, coarse model's 40, code table, voxel table last, each at a 16-byte aligned offset of one
    fp32 bucket that its .grad views (earlier values copied in); the all-reduce covers the bucket up to voxel-table row
    n_used (the whole bucket without a table) and the 1/W scale gives back the single-rank gradients."""
    from object_nerf_b200 import engine, training
    from tests import cases
    _stubbed(monkeypatch)
    fd = _FakeDist(monkeypatch, rank=0, world=2)
    models, embeddings, lib, batch, kw = _problem() if use_voxel else _plain_problem()
    emb = embeddings["xyz"] if use_voxel else None
    first = engine.model_linears(models["coarse"])[3][0]
    first.grad = torch.full_like(first, 0.5)
    monkeypatch.setattr(engine, "new_seed", lambda: 1000)
    training.sync_replicas(models, embeddings, lib, GROUP)
    n_used = int(emb.voxel_idx_map.max()) + 1 if use_voxel else 0
    assert training._synced[models["coarse"]][1] == n_used
    if use_voxel:
        assert 0 < n_used < emb.embedding_space_ftr.weight.shape[0]
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, group=GROUP, **kw)
    (plan,) = training._plans[models["coarse"]].values()
    bucket = plan.bucket
    tensors, offsets, total = _expected_layout(models, lib, emb)
    assert bucket.offsets == offsets and bucket.flat.numel() == total and bucket.flat.dtype == torch.float32
    base = bucket.flat.data_ptr()
    for t, off in zip(tensors, offsets):
        assert t.grad.data_ptr() == base + 4 * off and (base + 4 * off) % 16 == 0
        assert t.grad.shape == t.shape and t.grad.is_contiguous()
    if use_voxel:
        assert bucket.table_offset == offsets[-1]
        assert fd.reduced == [(base, offsets[-1] + 24 * n_used)]
    else:
        assert bucket.table_offset is None and fd.reduced == [(base, total)]
    # the fake all-reduce multiplied by W; the scale divides it back: the stubbed step's values (layer i: i + 1)
    for typ in ("coarse", "fine"):
        for i, (w, b) in enumerate(engine.model_linears(models[typ])):
            was = 0.5 if (typ, i) == ("coarse", 3) else 0.0
            assert w.grad.reshape(-1)[0].item() == was + i + 1 and b.grad.reshape(-1)[0].item() == i + 1
    assert first.grad.reshape(-1)[1:].eq(0.5).all()
    # a second call reuses plan and bucket and reduces the same prefix
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, group=GROUP, **kw)
    assert list(training._plans[models["coarse"]].values()) == [plan] and fd.reduced[1] == fd.reduced[0]


def test_group_less_call_allocates_no_bucket_and_reduces_nothing(monkeypatch):
    from object_nerf_b200 import training
    from tests import cases
    _stubbed(monkeypatch)
    fd = _FakeDist(monkeypatch)
    models, embeddings, lib, batch, kw = _problem()
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    (plan,) = training._plans[models["coarse"]].values()
    assert plan.bucket is None and fd.reduced == [] and fd.broadcasts == 0


@pytest.mark.parametrize("rank,seed", [(0, 1000), (1, 1000), (3, 1000), (5, 2 ** 62 - 3)])
def test_rank_seeds(monkeypatch, rank, seed):
    """Rank r draws with the group-less seed + r * 2^52 (mod 2^62); the device counter starts 4 above it."""
    from object_nerf_b200 import engine, training
    from tests import cases
    fake = _stubbed(monkeypatch)
    _FakeDist(monkeypatch, rank=rank, world=8)
    models, embeddings, lib, batch, kw = _problem()
    monkeypatch.setattr(engine, "new_seed", lambda: seed)
    training.sync_replicas(models, embeddings, lib, GROUP)
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, group=GROUP, **kw)
    want = (seed + rank * 2 ** 52) % 2 ** 62
    assert [c for c in fake.calls if c[0] == "step"][-1][1]["seed"] == want
    assert training.step_seed(models).tolist() == [want + 4]


def _grouped(monkeypatch):
    from object_nerf_b200 import engine, training
    from tests import cases
    _stubbed(monkeypatch)
    fd = _FakeDist(monkeypatch)
    models, embeddings, lib, batch, kw = _problem()
    monkeypatch.setattr(engine, "new_seed", lambda: 1000)
    call = lambda: training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, group=GROUP, **kw)
    return models, embeddings, lib, call, fd


def test_refused_without_sync_replicas(monkeypatch):
    from object_nerf_b200 import training
    models, embeddings, lib, call, fd = _grouped(monkeypatch)
    with pytest.raises(RuntimeError, match="sync_replicas"):
        call()
    assert not training._plans.get(models["coarse"]) and fd.reduced == []


@pytest.mark.parametrize("change", ["pruned_in_place", "replaced", "reshaped"])
def test_refused_after_a_grid_change(monkeypatch, change):
    from object_nerf_b200 import training
    models, embeddings, lib, call, fd = _grouped(monkeypatch)
    emb = embeddings["xyz"]
    training.sync_replicas(models, embeddings, lib, GROUP)
    call()
    if change == "pruned_in_place":
        emb.voxel_idx_map[0, 0, 0] = -1
    elif change == "replaced":
        emb.voxel_idx_map = emb.voxel_idx_map.clone()
    else:
        emb.voxel_idx_map = emb.voxel_idx_map.reshape(-1, emb.voxel_idx_map.shape[-1]).contiguous()
    with pytest.raises(RuntimeError, match="grid changed"):
        call()
    assert len(fd.reduced) == 1
    training.sync_replicas(models, embeddings, lib, GROUP)
    if change != "reshaped":
        call()
        assert len(fd.reduced) == 2


@pytest.mark.parametrize("how", ["set_to_none", "new_grad", "replaced_parameter"])
def test_refused_when_a_grad_leaves_the_bucket(monkeypatch, how):
    from object_nerf_b200 import engine
    models, embeddings, lib, call, fd = _grouped(monkeypatch)
    from object_nerf_b200 import training
    training.sync_replicas(models, embeddings, lib, GROUP)
    call()
    w = engine.model_linears(models["fine"])[0][0]
    if how == "set_to_none":
        torch.optim.SGD([p for m in models.values() for p in m.parameters()], lr=1).zero_grad(set_to_none=True)
    elif how == "new_grad":
        w.grad = torch.zeros_like(w)
    else:
        models["fine"].xyz_encoding_1[0].weight = torch.nn.Parameter(w.detach().clone())
    with pytest.raises(RuntimeError, match="bucket"):
        call()
    assert len(fd.reduced) == 1


def test_first_grouped_call_inside_a_capture_is_refused(monkeypatch):
    from object_nerf_b200 import training
    models, embeddings, lib, call, fd = _grouped(monkeypatch)
    training.sync_replicas(models, embeddings, lib, GROUP)
    monkeypatch.setattr(training, "_capturing", lambda dev: True)
    with pytest.raises(RuntimeError, match="warm up"):
        call()
    assert not training._plans.get(models["coarse"]) and fd.reduced == []


def _sync_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from object_nerf_b200 import Embedding, training
        from object_nerf_b200 import synthetic as S
        from tests import cases, helpers
        from tests.test_host_logic_cpu import _maint_embedding
        inp = cases.build_grad_case()
        torch.manual_seed(rank)
        models = {k: S.make_model(w, True, "cpu") for k, w in inp["weights"].items()}
        emb, _ = _maint_embedding()
        lib = helpers.CodeLib(inp["code_table"])
        with torch.no_grad():        # every rank's replica differs, and rank 1's grid has another shape
            for p in [p for m in models.values() for p in m.parameters()] + [lib.embedding_instance.weight,
                                                                          emb.embedding_space_ftr.weight]:
                p.add_(torch.randn_like(p))
        for _ in range(1 + rank):
            emb.voxel_subdivision(_features_fn=lambda pts: torch.zeros(pts.shape[0], 24))
        if rank == 1:
            emb.voxel_offset += 0.25
        embeddings = {"xyz": emb, "dir": Embedding(3, 4)}
        training.sync_replicas(models, embeddings, lib, dist.group.WORLD)
        state = {f"{typ}.{k}": v.clone() for typ, m in models.items() for k, v in m.state_dict().items()}
        state.update({f"emb.{k}": v.clone() for k, v in emb.state_dict().items()})
        state["codes"] = lib.embedding_instance.weight.detach().clone()
        ret[rank] = (state, training._synced[models["coarse"]][1], int(emb.voxel_idx_map.max()) + 1,
                     training._synced[models["coarse"]][0] == training._grid_stamp(emb))
    finally:
        dist.destroy_process_group()


def test_sync_replicas_makes_every_rank_rank_0s_replica():
    """Two gloo ranks with different parameters, code tables, voxel tables and grids (rank 1's subdivided once more, so
    of another shape): after sync_replicas every parameter and grid buffer equals rank 0's, and both count rank 0's
    n_used."""
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_sync_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    (s0, n0, m0, ok0), (s1, n1, m1, ok1) = ret[0], ret[1]
    assert sorted(s0) == sorted(s1)
    for name in ("emb.voxel_idx_map", "emb.voxel_occupancy", "emb.voxel_shape", "emb.voxel_size", "emb.voxel_offset",
                 "emb.voxel_count", "emb.embedding_space_ftr.weight", "codes", "coarse.sigma.weight"):
        assert name in s0, name
    for k in s0:
        assert s0[k].dtype == s1[k].dtype and torch.equal(s0[k], s1[k]), k
    assert n0 == n1 == m0 > 0 and ok0 and ok1
