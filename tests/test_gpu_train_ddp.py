"""Data-parallel training on the device loop (training.train_step(group=...), training.sync_replicas).

gloo, two ranks sharing cuda:0 (as tests/test_gpu_ddp.py), 96 rays with injected random buffers, 48 per rank:
  - fp32 and bf16: every gradient on both ranks is the mean of the two single-process train_step gradients, the ranks'
    buckets are bit-identical, voxel-table rows at or above n_used are exactly zero, and the bf16 gradients agree with
    DDP around render_rays + loss.backward();
  - three eager steps with Adam leave bit-identical parameters on both ranks;
  - grids pruned with different jitter per rank are identical after sync_replicas, whose n_used the next step reduces
    up to; a step after voxel_subdivision without sync_replicas is refused;
  - rank r's maps equal a group-less call's with seed + r * 2^52.
NCCL: sampler + train_step(group=) + Adam captured in one graph on one GPU (world 1), replay k against eager step k; and
with two GPUs, the same over two ranks with bit-identical parameters after the replays."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import cases, helpers

pytestmark = pytest.mark.gpu
N_RAYS, HALF = 96, 48


def _port():
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        return sk.getsockname()[1]


def _spawn(target, world, *args):
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    port = _port()
    procs = [ctx.Process(target=target, args=(r, world, port, ret) + args) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0, p.exitcode
    return dict(ret)


def _setup(inp, dev, emb=None):
    from object_nerf_b200 import Embedding
    models = {k: helpers.make_model(w, True, dev).train() for k, w in inp["weights"].items()}
    emb = emb if emb is not None else helpers.GridModule(inp["grid"]).to(dev)
    lib = helpers.CodeLib(inp["code_table"]).to(dev)
    return models, {"xyz": emb, "dir": Embedding(3, 4)}, lib


def _named(models, embeddings, lib):
    named = [(f"{typ}.{k}", p) for typ, m in models.items() for k, p in m.named_parameters()]
    return named + [("codes", lib.embedding_instance.weight), ("voxel", embeddings["xyz"].embedding_space_ftr.weight)]


def _batch(inp, sl, dev):
    b = {k: v[sl].to(dev) for k, v in inp["batch"].items()}
    b["rays"], b["instance_ids"] = inp["rays"][sl].to(dev), inp["instance_ids"][sl].to(dev)
    return b


def _kwargs(inp, sl, dev, precision, rand=True):
    c = cases.GRAD_CASE
    kw = dict(N_samples=c["n_samples"], perturb=c["perturb"], noise_std=c["noise_std"], N_importance=c["n_importance"],
              frustum_bound_th=c["frustum_bound_th"], pass_through_mask=inp["pass_through_mask"][sl].to(dev),
              is_eval=False, precision=precision)
    if rand:
        kw["_rand"] = {k: v[sl].to(dev) for k, v in inp["rand"].items()}
    return kw


def _gathered_equal(t):
    """Whether every rank holds the same bits as this one (gloo gathers host copies)."""
    t = t.detach().reshape(-1).cpu()
    t = t.to(torch.uint8) if t.dtype == torch.bool else t
    out = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(out, t)
    return all(torch.equal(o.view(torch.int32) if o.is_floating_point() else o,
                           t.view(torch.int32) if t.is_floating_point() else t) for o in out)


def _flat_params(named):
    return torch.cat([p.detach().reshape(-1) for _, p in named])


def _rel(g, w):
    g, w = g.reshape(-1).double(), w.reshape(-1).double()
    return ((g - w).norm() / (w.norm() + 1e-30)).item() if w.norm() > 0 else g.norm().item()


def _gloo_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from object_nerf_b200 import engine, training
        from tests import test_gpu_ddp
        from tests.test_host_logic_cpu import _maint_embedding
        group = dist.group.WORLD
        inp = cases.build_grad_case(n_rays=N_RAYS)
        halves = [slice(r * HALF, (r + 1) * HALF) for r in range(world)]
        mine = halves[rank]
        res = {}
        reduced = []
        all_reduce = dist.all_reduce

        def recording_all_reduce(t, **kw):
            reduced.append(t.numel())
            return all_reduce(t, **kw)
        dist.all_reduce = recording_all_reduce

        # 1. gradients = mean of the single-process gradients
        for precision in ("fp32", "bf16"):
            singles = []
            for sl in halves:
                models, embeddings, lib = _setup(inp, dev)
                training.train_step(models, embeddings, lib, _batch(inp, sl, dev), cases.LOSS_CONF,
                                    **_kwargs(inp, sl, dev, precision))
                singles.append([p.grad.clone() for _, p in _named(models, embeddings, lib)])
            want = [(a + b) / 2 for a, b in zip(*singles)]
            models, embeddings, lib = _setup(inp, dev)
            training.sync_replicas(models, embeddings, lib, group)
            n_used = training._synced[models["coarse"]][1]
            reduced.clear()
            training.train_step(models, embeddings, lib, _batch(inp, mine, dev), cases.LOSS_CONF, group=group,
                                **_kwargs(inp, mine, dev, precision))
            torch.cuda.synchronize()
            named = _named(models, embeddings, lib)
            (plan,) = training._plans[models["coarse"]].values()
            table_grad = embeddings["xyz"].embedding_space_ftr.weight.grad
            res[precision] = dict(
                worst=max((_rel(p.grad, w), name) for (name, p), w in zip(named, want)),
                identical=_gathered_equal(plan.bucket.flat),
                n_used=n_used, rows=table_grad.shape[0], max_idx=int(embeddings["xyz"].voxel_idx_map.max()),
                above_zero=bool((table_grad[n_used:] == 0).all()),
                reduced=list(reduced), prefix=plan.bucket.table_offset + 24 * n_used)
            if precision == "bf16":
                system = test_gpu_ddp._system(inp, dev)
                ddp = torch.nn.parallel.DistributedDataParallel(system, device_ids=[dev.index],
                                                                broadcast_buffers=False)
                b, rand = test_gpu_ddp._batch(inp, mine, dev)
                ddp(b, rand).backward()
                ref = {f"{typ}.{k}": p.grad for typ in ("coarse", "fine")
                       for k, p in getattr(system, typ).named_parameters()}
                ref.update(codes=system.lib.embedding_instance.weight.grad, voxel=system.emb.embedding_space_ftr.weight.grad)
                res["vs_ddp"] = max(((p.grad - ref[name]).abs().max().item() / (ref[name].abs().max().item() + 1e-12),
                                     name) for name, p in named)

        # 2. three eager Adam steps: bit-identical parameters
        models, embeddings, lib = _setup(inp, dev)
        named = _named(models, embeddings, lib)
        training.sync_replicas(models, embeddings, lib, group)
        opt = torch.optim.Adam([p for _, p in named], lr=1e-3)
        batch, kw = _batch(inp, mine, dev), _kwargs(inp, mine, dev, "bf16")
        for _ in range(3):
            opt.zero_grad(set_to_none=False)
            training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, group=group, **kw)
            opt.step()
        res["adam_identical"] = _gathered_equal(_flat_params(named))
        res["adam_moved"] = bool((_flat_params(named) != _flat_params(_named(*_setup(inp, dev)))).any())

        # 3. rank seeds: rank r's maps are a group-less call's with seed + r * 2^52
        seed = 0x1234_5678_9AB
        maps = []
        for grouped in (True, False):
            models, embeddings, lib = _setup(inp, dev)
            if grouped:
                training.sync_replicas(models, embeddings, lib, group)
            engine.new_seed = (lambda: seed) if grouped else (lambda: seed + rank * 2 ** 52)
            training.train_step(models, embeddings, lib, _batch(inp, mine, dev), cases.LOSS_CONF,
                                group=group if grouped else None, **_kwargs(inp, mine, dev, "bf16", rand=False))
            (plan,) = training._plans[models["coarse"]].values()
            maps.append({f"{k}_{typ}": v.clone() for typ, m in plan.render.maps.items() for k, v in m.items()})
        res["seed_maps_equal"] = all(torch.equal(maps[0][k], maps[1][k]) for k in maps[0])
        res["z_identical_across_ranks"] = _gathered_equal(maps[0]["z_vals_coarse"])

        # 4. grid maintenance: pruning with per-rank jitter, sync_replicas, subdivision without it
        emb, minp = _maint_embedding()
        emb = emb.to(dev)
        models, embeddings, lib = _setup(inp, dev, emb)
        training.sync_replicas(models, embeddings, lib, group)
        kw = _kwargs(inp, mine, dev, "bf16")
        batch = _batch(inp, mine, dev)
        training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, group=group, **kw)
        n_occu = int(emb.voxel_occupancy.sum())
        pruned = emb.self_pruning_empty_voxels(
            helpers.make_model(minp["weights"], True, dev), max_alpha_th=cases.MAINT_CASE["max_alpha_th"],
            _rand=[r.to(dev) for r in cases.maint_rand((n_occu + 31) // 32, seed=100 + rank)])
        res["pruned"] = pruned
        res["grids_differed"] = not _gathered_equal(emb.voxel_idx_map)
        try:
            training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, group=group, **kw)
            res["prune_refusal"] = None
        except RuntimeError as e:
            res["prune_refusal"] = str(e)
        training.sync_replicas(models, embeddings, lib, group)
        res["grid_identical"] = all(_gathered_equal(getattr(emb, k)) for k in training.GRID_BUFFERS)
        n_used = training._synced[models["coarse"]][1]
        res["maint_n_used"] = (n_used, int(emb.voxel_idx_map.max()) + 1)
        reduced.clear()
        training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, group=group, **kw)
        (plan,) = training._plans[models["coarse"]].values()
        res["maint_reduced"] = (list(reduced), plan.bucket.table_offset + 24 * n_used)
        emb.voxel_subdivision()
        try:
            training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, group=group, **kw)
            res["subdiv_refusal"] = None
        except RuntimeError as e:
            res["subdiv_refusal"] = str(e)
        training.sync_replicas(models, embeddings, lib, group)
        reduced.clear()
        training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, group=group, **kw)
        n_used = training._synced[models["coarse"]][1]
        res["subdiv_reduced"] = (list(reduced), plan.bucket.table_offset + 24 * n_used, n_used,
                                 int(emb.voxel_idx_map.max()) + 1)
        torch.cuda.synchronize()
        ret[rank] = res
    finally:
        dist.destroy_process_group()


@pytest.fixture(scope="module")
def gloo():
    return _spawn(_gloo_worker, 2)


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5), ("bf16", 2e-3)])
def test_gradients_are_the_mean_of_the_single_process_gradients(gloo, precision, tol):
    for rank, res in gloo.items():
        r = res[precision]
        assert r["worst"][0] <= tol, (rank, r["worst"])
        assert r["identical"], rank
        assert r["n_used"] == r["max_idx"] + 1 and r["n_used"] <= r["rows"]
        assert r["above_zero"], rank
        assert r["reduced"] == [r["prefix"]], (r["reduced"], r["prefix"])


def test_bf16_gradients_agree_with_ddp_around_render_rays(gloo):
    """The tolerance of tests/test_gpu_ddp.py: largest difference over the largest magnitude, per tensor."""
    for rank, res in gloo.items():
        assert res["vs_ddp"][0] < 2e-3, (rank, res["vs_ddp"])


def test_adam_steps_leave_bit_identical_replicas(gloo):
    for rank, res in gloo.items():
        assert res["adam_identical"] and res["adam_moved"], rank


def test_rank_seeds_are_the_group_less_seed_plus_rank_stride(gloo):
    for rank, res in gloo.items():
        assert res["seed_maps_equal"], rank
        assert not res["z_identical_across_ranks"], rank       # the ranks do draw different jitter


def test_grid_maintenance_needs_sync_replicas(gloo):
    for rank, res in gloo.items():
        assert res["pruned"] > 0, rank
        assert res["prune_refusal"] and "sync_replicas" in res["prune_refusal"], rank
        assert res["grid_identical"], rank
        n_used, want = res["maint_n_used"]
        assert n_used == want
        got, prefix = res["maint_reduced"]
        assert got == [prefix], (got, prefix)
        assert res["subdiv_refusal"] and "grid changed" in res["subdiv_refusal"], rank
        got, prefix, n_used, want = res["subdiv_reduced"]
        assert got == [prefix] and n_used == want, res["subdiv_reduced"]
    assert gloo[0]["maint_n_used"] == gloo[1]["maint_n_used"]




# ------------------------------------------------------------------------------------------------
# NCCL: the sampler, the step and Adam in one CUDA graph
# ------------------------------------------------------------------------------------------------
def _nccl_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        import numpy as np

        from object_nerf_b200 import RaySampler, engine, training
        from object_nerf_b200 import synthetic as S
        from tests.test_batches_cpu import dataset
        group = dist.group.WORLD
        inp = cases.build_grad_case()
        R, B = 8192, 256
        t = dataset(R, 2)
        t["all_rays"] = S.random_rays(11, R)
        t["all_instance_ids"] = torch.from_numpy(np.random.default_rng(2).choice([4, 6], size=(R, 2)))
        c = cases.GRAD_CASE
        kw = dict(N_samples=c["n_samples"], perturb=1.0, noise_std=1.0, N_importance=c["n_importance"],
                  frustum_bound_th=c["frustum_bound_th"], is_eval=False, precision="bf16")
        warm_seed = 0x5EED

        def arm():
            models, embeddings, lib = _setup(inp, dev)
            named = _named(models, embeddings, lib)
            training.sync_replicas(models, embeddings, lib, group)
            sampler = RaySampler(t, batch_size=B, device=dev, seed=7, group=group)
            opt = torch.optim.Adam([p for _, p in named], lr=1e-3, capturable=True)

            def step():
                batch = sampler.next()
                opt.zero_grad(set_to_none=False)
                out = training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF,
                                          pass_through_mask=batch["pass_through_mask"], group=group, **kw)
                opt.step()
                return out

            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            engine.new_seed = lambda: warm_seed
            with torch.cuda.stream(side):
                step()          # warm-up: the plan, its bucket, Adam's state and the communicator
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            return dict(models=models, embeddings=embeddings, lib=lib, named=named, sampler=sampler, step=step)

        a = arm()
        s0 = training.step_seed(a["models"]).item()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out_g = a["step"]()
        (plan_g,) = training._plans[a["models"]["coarse"]].values()
        res = dict(s0=s0, want_s0=warm_seed + rank * 2 ** 52 + 4)
        if world == 1:
            # the same parameters and batch as each replay, one eager step with the replay's seed
            r = arm()
            (plan_r,) = training._plans[r["models"]["coarse"]].values()
            z_equal, loss_rel, after3 = [], [], None
            for k in range(4):
                with torch.no_grad():
                    for (_, pr), (_, pg) in zip(r["named"], a["named"]):
                        pr.copy_(pg)
                r["sampler"].set_step(a["sampler"].step)
                g.replay()
                torch.cuda.synchronize()
                loss_g = out_g[0].item()
                engine.new_seed = lambda: s0 + 4 * k
                batch = r["sampler"].next()
                for _, p in r["named"]:
                    p.grad.zero_()
                loss_r = training.train_step(r["models"], r["embeddings"], r["lib"], batch, cases.LOSS_CONF,
                                             pass_through_mask=batch["pass_through_mask"], group=group, **kw)[0].item()
                z_equal.append(all(torch.equal(plan_r.render.maps[typ]["z_vals"], plan_g.render.maps[typ]["z_vals"])
                                   for typ in ("coarse", "fine")))
                loss_rel.append(abs(loss_g - loss_r) / abs(loss_r))
                if k == 2:
                    after3 = _flat_params(a["named"]).clone()
            res.update(z_equal=z_equal, loss_rel=loss_rel, s_after=training.step_seed(a["models"]).item())
            # three eager Adam steps with the replays' seeds, from the graphed arm's starting point
            e = arm()
            start = _flat_params(e["named"]).clone()
            seeds = iter([s0, s0 + 4, s0 + 8])
            engine.new_seed = lambda: next(seeds)
            for _ in range(3):
                e["step"]()
            torch.cuda.synchronize()
            pe = _flat_params(e["named"])
            res["adam"] = ((after3 - pe).norm().item(), (pe - start).norm().item())
        else:
            start = _flat_params(a["named"]).clone()
            for _ in range(4):
                g.replay()
            torch.cuda.synchronize()
            p = _flat_params(a["named"])
            out = [torch.empty_like(p) for _ in range(world)]
            dist.all_gather(out, p)
            res["identical"] = all(torch.equal(o.view(torch.int32), p.view(torch.int32)) for o in out)
            res["moved"] = (p - start).norm().item()
        ret[rank] = res
    finally:
        dist.destroy_process_group()


def test_nccl_captured_loop_replays_match_eager_steps():
    """World 1: sampler + train_step(group=) + Adam in one graph.  Replay k draws what the eager step with seed
    s0 + 4k draws on the same parameters and batch (depths bit for bit, loss within 1e-6); after three replays the
    parameters match three eager Adam steps within 5 % of the distance moved (tests/test_gpu_graph_rng.py)."""
    (res,) = _spawn(_nccl_worker, 1).values()
    assert res["s0"] == res["want_s0"]
    assert all(res["z_equal"]), res["z_equal"]
    assert max(res["loss_rel"]) <= 1e-6, res["loss_rel"]
    assert res["s_after"] == res["s0"] + 16
    diff, moved = res["adam"]
    assert diff <= 5e-2 * moved, (diff, moved)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_nccl_captured_loop_keeps_two_ranks_bit_identical():
    ret = _spawn(_nccl_worker, 2)
    for rank, res in ret.items():
        assert res["s0"] == res["want_s0"], rank
        assert res["identical"] and res["moved"] > 0, (rank, res)
