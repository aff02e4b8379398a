"""training.install_training (TrainStepFn: the one-call step with its gradients handed to autograd) on the GPU:
  * the installed training_step + loss.backward() against the unmodified reference's training_step over
    dropin.install() + loss.backward(), voxel and plain-PE models, fp32 and bf16, on the same batch and injected `_rand`
    buffers: maps, loss, logged terms and PSNR, gradients under the gates of tests/test_gpu_train_step.py; and again
    after self_pruning_empty_voxels and after voxel_subdivision (needs oracle/_ref);
  * autograd semantics: gradients accumulate over steps, scale with the incoming gradient, never alias the plan's
    gradient sink, and the call is refused under torch.no_grad();
  * DistributedDataParallel around a module whose forward is the installed training_step, two gloo ranks on one GPU:
    each rank's gradients equal the single-process step on the concatenated batch."""
import functools
import os
import socket
import types

import pytest
import torch

from oracle import ref_loader as R
from tests import cases, helpers, synth
from tests.test_gpu_train_step import _assert_same_grads

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# (loss and terms, gradient relative norm, gradient cosine): tests/test_gpu_train_step.py's fp32 and bf16 gates
GATES = {"fp32": (1e-5, 1e-5, 0.99999), "bf16": (2e-2, 5e-2, 0.995)}
needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref not built (needs the reference at build time)")


# ------------------------------------------------------------------------------------------------
# the unmodified reference's training_step over the drop-in against the installed one
# ------------------------------------------------------------------------------------------------
def _fill(system, use_voxel, seed=7):
    """The same reference-shaped weights, codes and voxel table in every system (through the checkpoint keys)."""
    from object_nerf_b200 import synthetic as S
    sd = system.state_dict()
    for prefix, s in (("nerf_coarse.", seed), ("nerf_fine.", seed + 1000)):
        for k, (W, b) in S.make_weights(s, use_voxel, sigma_gain=8.0, sigma_bias=1.0, rgb_gain=16.0).items():
            sd[prefix + S.REF_NAMES[k] + ".weight"], sd[prefix + S.REF_NAMES[k] + ".bias"] = W, b
    g = torch.Generator().manual_seed(seed + 5)
    sd["code_library.embedding_instance.weight"] = torch.randn(64, 64, generator=g)
    if use_voxel:
        key = "embedding_xyz.embedding_space_ftr.weight"
        sd[key] = torch.randn(tuple(sd[key].shape), generator=g)
    system.load_state_dict(sd, strict=True)


@pytest.fixture
def pair(tmp_path, monkeypatch):
    """-> make(use_voxel, precision, max_voxels=None) -> (reference system over the drop-in, installed system, maps the
    reference route rendered last, batch).  Both draw from the same `_rand` buffers: jitter and sigma noise on."""
    import object_nerf_b200.dropin as dropin
    from object_nerf_b200 import rendering, training
    from tests import dropin_fixture as F

    def make(use_voxel, precision, max_voxels=None):
        monkeypatch.setenv("ONERF_PRECISION", precision)
        conf, _ = F.write_scene(str(tmp_path))
        conf["model"].update(use_voxel_embedding=use_voxel, perturb=1, noise_std=1)
        if max_voxels:
            conf["model"]["N_max_voxels"] = max_voxels
        n = 256
        batch = {k: v.to(DEV) for k, v in F.training_batch(n=n).items()}
        rand = {k: v.to(DEV) for k, v in synth.random_buffers(11, n, 64, 64).items()}
        systems = []
        for installed in (False, True):
            F.purge_reference_modules()
            R.install(cuda_noop=False)
            dropin.install()
            train, system = F.make_system(conf, DEV)
            _fill(system, use_voxel)
            system.train()
            if installed:
                training.install_training(train.ObjectNeRFSystem)
            systems.append((train, system))
        maps = {}

        def render_rays(*a, **kw):
            out = rendering.render_rays(*a, _rand=rand, **kw)
            maps.update(out)
            return out
        monkeypatch.setattr(systems[0][0], "render_rays", render_rays)
        monkeypatch.setattr(training, "train_step", functools.partial(training.train_step, _rand=rand))
        return systems[0][1], systems[1][1], maps, batch

    try:
        yield make
    finally:
        F.purge_reference_modules()
        R.cuda_noop(not torch.cuda.is_available())


def _step(system, batch):
    system.zero_grad(set_to_none=True)
    loss = system.training_step(dict(batch), 0)
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach()


def _assert_same_step(ref, ours, maps, batch, precision):
    from object_nerf_b200 import training
    loss_tol, norm_tol, cos_min = GATES[precision]
    loss_e, loss_f = _step(ref, batch), _step(ours, batch)
    assert abs(loss_f.item() - loss_e.item()) <= loss_tol * abs(loss_e.item()), (loss_f.item(), loss_e.item())
    assert list(ours.logged) == list(ref.logged)
    for k, v in ref.logged.items():
        if k.startswith("train/") and k not in ("train/loss", "train/psnr"):
            got, want = float(ours.logged[k].detach()), float(v.detach())
            assert abs(got - want) <= loss_tol * abs(want) + 1e-12, k
    psnr_e, psnr_f = float(ref.logged["train/psnr"]), float(ours.logged["train/psnr"])
    assert abs(psnr_f - psnr_e) <= 1e-4 * abs(psnr_e), (psnr_f, psnr_e)
    (plan,) = training._plans[ours.models["coarse"]].values()
    got = {f"{k}_{typ}": v for typ, m in plan.render.maps.items() for k, v in m.items()}
    for k, v in maps.items():
        assert torch.equal(got[k], v.detach()), k
    _assert_same_grads(list(ours.named_parameters()), list(ref.named_parameters()), norm_tol, cos_min)


@needs_ref
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("use_voxel", [True, False], ids=["voxel", "plain"])
def test_installed_step_matches_the_reference_step_over_dropin(pair, use_voxel, precision):
    ref, ours, maps, batch = pair(use_voxel, precision)
    _assert_same_step(ref, ours, maps, batch, precision)
    assert all(p.grad is not None and p.grad.norm() > 0 for p in ours.parameters())


@needs_ref
def test_installed_step_follows_pruning_and_subdivision(pair):
    """train.py:140-145 between steps: each step after self_pruning_empty_voxels and after voxel_subdivision matches
    the existing route on the new grid (the installed step's plan was made on the old one)."""
    ref, ours, maps, batch = pair(True, "fp32", max_voxels=65536)
    _assert_same_step(ref, ours, maps, batch, "fp32")
    # the synthetic fine model's scene density stays below the 0.5 alpha threshold everywhere, so pruning with it
    # would empty the grid: the same pass with a density that keeps the voxels at x > 0 (the same jitter on both)
    pruned = []
    for s in (ref, ours):
        torch.manual_seed(17)
        pruned.append(s.embedding_xyz.self_pruning_empty_voxels(
            s.models["fine"], _sigma_fn=lambda xyz: torch.where(xyz[:, 0] > 0, 10.0, 0.0)))
    assert pruned[0] == pruned[1] > 0 and (ours.embedding_xyz.voxel_idx_map >= 0).any()
    assert torch.equal(ref.embedding_xyz.voxel_idx_map, ours.embedding_xyz.voxel_idx_map)
    _assert_same_step(ref, ours, maps, batch, "fp32")
    assert ref.embedding_xyz.voxel_subdivision() == ours.embedding_xyz.voxel_subdivision() > 0
    _assert_same_step(ref, ours, maps, batch, "fp32")
    assert ours.embedding_xyz.embedding_space_ftr.weight.grad.norm() > 0


# ------------------------------------------------------------------------------------------------
# a module with what training_step reads (no reference needed)
# ------------------------------------------------------------------------------------------------
def get_learning_rate(optimizer):
    """The reference's utils.get_learning_rate, which install_training looks up in the system class's module."""
    return optimizer.param_groups[0]["lr"]


class LocalSystem(torch.nn.Module):
    """ObjectNeRFSystem's attributes that training_step reads, on tests/cases.py's gradient scene; forward is the
    training step (so that DDP can wrap it)."""

    def __init__(self, inp, dev):
        from object_nerf_b200 import Embedding
        super().__init__()
        self.nerf_coarse = helpers.make_model(inp["weights"]["coarse"], True, dev).train()
        self.nerf_fine = helpers.make_model(inp["weights"]["fine"], True, dev).train()
        self.embedding_xyz = helpers.GridModule(inp["grid"]).to(dev)
        self.code_library = helpers.CodeLib(inp["code_table"]).to(dev)
        self.models = {"coarse": self.nerf_coarse, "fine": self.nerf_fine}
        self.embeddings = {"xyz": self.embedding_xyz, "dir": Embedding(3, 4)}
        c = cases.GRAD_CASE
        self.config = R.to_attr({
            "model": {"N_samples": c["n_samples"], "N_importance": c["n_importance"], "use_disp": False,
                      "perturb": c["perturb"], "noise_std": c["noise_std"], "frustum_bound": 2 * c["frustum_bound_th"]},
            "dataset_extra": {"scale_factor": 2.0}, "loss": dict(cases.LOSS_CONF)})
        self.train_dataset = types.SimpleNamespace(white_back=False, is_rays_in_bbox=lambda: False)
        self.optimizer = torch.optim.SGD(self.parameters(), lr=1e-3)
        self.logged = {}

    def log(self, name, value, *a, **k):
        self.logged[name] = value

    def forward(self, batch):
        return self.training_step(batch, 0)


def _local_batch(inp, sl, dev):
    b = {k: v[sl].to(dev) for k, v in inp["batch"].items()}
    b.update(rays=inp["rays"][sl].to(dev), instance_ids=inp["instance_ids"][sl].to(dev),
             pass_through_mask=inp["pass_through_mask"][sl].to(dev))
    return b, {k: v[sl].to(dev) for k, v in inp["rand"].items()}


def _trained(system):
    from object_nerf_b200 import training
    t = training._trained_tensors(system.models, ["coarse", "fine"], system.code_library.embedding_instance.weight,
                                  system.embedding_xyz.embedding_space_ftr.weight)
    assert sorted(map(id, t)) == sorted(map(id, system.parameters()))
    return t


def _rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def test_autograd_semantics(monkeypatch):
    """fp32, the same batch and `_rand` buffers every step, so every step has the same gradients up to the order of
    the fp32 atomics."""
    from object_nerf_b200 import training
    monkeypatch.setenv("ONERF_PRECISION", "fp32")
    training.install_training(LocalSystem)
    inp = cases.build_grad_case()
    batch, rand = _local_batch(inp, slice(None), DEV)
    monkeypatch.setattr(training, "train_step", functools.partial(training.train_step, _rand=rand))
    s = LocalSystem(inp, DEV)
    trained = _trained(s)
    s(batch).backward()
    (plan,) = training._plans[s.models["coarse"]].values()
    sink = plan.sink.views
    taken = [t.grad for t in trained]
    g1 = [g.clone() for g in taken]
    assert all(g.norm() > 0 for g in g1)
    # the returned gradients are not views of the sink
    lo, hi = plan.sink.flat.data_ptr(), plan.sink.flat.data_ptr() + 4 * plan.sink.flat.numel()
    assert not any(lo <= g.data_ptr() < hi for g in taken)
    # a .grad taken after step 1 is left alone by step 2
    s.zero_grad(set_to_none=True)
    s(batch).backward()
    assert all(torch.equal(a, b) for a, b in zip(taken, g1))
    assert all(_rel(t.grad, g) < 1e-4 for t, g in zip(trained, g1))
    # two steps without zero_grad: the first step's gradients plus the second's
    first = [t.grad.clone() for t in trained]
    s(batch).backward()
    assert all(torch.equal(t.grad, f + v) for t, f, v in zip(trained, first, sink))
    assert all(_rel(t.grad, 2 * g) < 1e-4 for t, g in zip(trained, g1))
    # (0.5 * loss).backward() halves them
    s.zero_grad(set_to_none=True)
    (0.5 * s(batch)).backward()
    assert all(torch.equal(t.grad, 0.5 * v) for t, v in zip(trained, sink))
    assert all(_rel(t.grad, 0.5 * g) < 1e-4 for t, g in zip(trained, g1))
    assert s.logged["train/loss"].requires_grad and sorted(s.logged)[0] == "lr"
    with torch.no_grad(), pytest.raises(RuntimeError, match="grad mode"):
        s(batch)
    assert len(training._plans[s.models["coarse"]]) == 1


# ------------------------------------------------------------------------------------------------
# DDP around the installed step: two gloo ranks on one GPU
# ------------------------------------------------------------------------------------------------
N_DDP = 96


def _ddp_case():
    """The halves of the batch have the same valid and instance masks (and every target depth is positive), so every
    TotalLoss normaliser of a half is half the whole batch's: the mean of the halves' gradients is the gradient of the
    whole batch."""
    inp = cases.build_grad_case(n_rays=N_DDP)
    h = N_DDP // 2
    for k in ("valid_mask", "instance_mask"):
        inp["batch"][k][h:] = inp["batch"][k][:h]
    assert (inp["batch"]["depths"] > 0).all()
    return inp


def _ddp_worker(rank, world, port, ret):
    import torch.distributed as dist

    from object_nerf_b200 import training
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    os.environ["ONERF_PRECISION"] = "bf16"
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        training.install_training(LocalSystem)
        step = training.train_step
        inp = _ddp_case()
        whole, rand = _local_batch(inp, slice(None), dev)
        training.train_step = functools.partial(step, _rand=rand)
        single = LocalSystem(inp, dev)
        single(whole).backward()
        want = [p.grad.detach().clone() for p in single.parameters()]
        h = N_DDP // world
        part, rand = _local_batch(inp, slice(rank * h, (rank + 1) * h), dev)
        training.train_step = functools.partial(step, _rand=rand)
        s = LocalSystem(inp, dev)
        ddp = torch.nn.parallel.DistributedDataParallel(s, device_ids=[dev.index], broadcast_buffers=False)
        ddp(part).backward()
        errs = []
        for (name, p), w in zip(s.named_parameters(), want):
            scale = w.abs().max().item() + 1e-12
            errs.append(((p.grad - w).abs().max().item() / scale, name, p.grad.abs().max().item(), scale))
        errs.sort(reverse=True)
        ret[rank] = errs[:4]
    finally:
        dist.destroy_process_group()


def test_ddp_gradients_equal_the_single_process_step_on_the_whole_batch():
    import torch.multiprocessing as mp
    world = 2
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_ddp_worker, args=(r, world, port, ret)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    # tests/test_gpu_ddp.py's gate: equal up to the order of the fp32 accumulation
    assert len(ret) == world and max(v[0][0] for v in ret.values()) < 2e-3, dict(ret)
