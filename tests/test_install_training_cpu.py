"""CPU checks of the autograd route of the training step (training.train_step(grad_sink=True), TrainStepFn,
install_training):
  * the unmodified reference's training_step with render_rays replaced by a recorder, and the installed training_step
    with training.train_step replaced by a recorder, receive the same batch tensors and keyword values and make the same
    self.log calls (needs oracle/_ref);
  * with the library stubbed: the sink takes the gradients and `.grad` stays untouched, the sink is zeroed on every call
    (the voxel table up to the most rows the grid has referenced), and TrainStepFn's backward returns new tensors
    scaled by the incoming gradient, refuses a stale sink, and the call is refused without grad mode."""
import contextlib
import types

import pytest
import torch

from oracle import ref_loader as R
from tests import cases
from tests.test_train_step_cpu import _FakeLib, _FakeRenderPlan

# train.py:155-165 and ObjectNeRFSystem.forward (:84-97): what the reference passes to render_rays, besides models,
# embeddings, rays, chunk and the looked-up codes
STEP_KEYS = ("N_samples", "use_disp", "perturb", "noise_std", "N_importance", "white_back", "is_eval",
             "pass_through_mask", "rays_in_bbox", "frustum_bound_th")
CONFIGS = {
    # scannet_base_0192_multi.yml over default_conf.yml: two objects, frustum bound on
    "scannet_multi": dict(scale_factor=2.5, frustum_bound=0.05, perturb=1, noise_std=1, rays_in_bbox=False),
    # toy_desk_2.yml: frustum bound disabled; a dataset with use_bbox on, so rays_in_bbox is True
    "toydesk": dict(scale_factor=16.0, frustum_bound=-1, perturb=1, noise_std=1, rays_in_bbox=True),
}
MAP_KEYS = ("rgb", "depth", "opacity", "rgb_instance", "depth_instance", "opacity_instance")


def _maps(n, seed=5):
    g = torch.Generator().manual_seed(seed)
    return {f"{k}_{typ}": torch.rand((n, 3) if k.startswith("rgb") else (n,), generator=g) * (1 if "opacity" in k else 2)
            for typ in ("coarse", "fine") for k in MAP_KEYS}


def _system(conf, over):
    from tests import dropin_fixture as F
    F.purge_reference_modules()
    R.install(cuda_noop=True)
    train, system = F.make_system(conf, "cpu")
    system.train_dataset = types.SimpleNamespace(white_back=False, is_rays_in_bbox=lambda: over["rays_in_bbox"])
    return train, system


@pytest.mark.skipif(not R.available(), reason="oracle/_ref not built (needs the reference at build time)")
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_installed_training_step_passes_what_the_reference_passes(tmp_path, monkeypatch, name):
    from object_nerf_b200 import training
    from tests import dropin_fixture as F
    over = CONFIGS[name]
    conf, _ = F.write_scene(str(tmp_path))
    conf["dataset_extra"]["scale_factor"] = over["scale_factor"]
    conf["model"].update(frustum_bound=over["frustum_bound"], perturb=over["perturb"], noise_std=over["noise_std"])
    batch = F.training_batch(n=64)
    maps = _maps(64)
    try:
        # ---- the reference's own training_step, render_rays recorded ----
        train, ref_sys = _system(conf, over)
        F.fill_synthetic_weights(ref_sys)
        seen_ref = {}

        def render_rays(**kw):
            seen_ref.update(kw)
            return {k: v.clone().requires_grad_() for k, v in maps.items()}
        monkeypatch.setattr(train, "render_rays", render_rays)
        loss_ref = ref_sys.training_step({k: v.clone() for k, v in batch.items()}, 0)
        from utils.metrics import psnr as ref_psnr
        ref_loss_fn = ref_sys.loss
        sd = ref_sys.state_dict()

        # ---- the installed training_step, train_step recorded ----
        train2, sys = _system(conf, over)
        sys.load_state_dict(sd, strict=True)
        training.install_training(train2.ObjectNeRFSystem)
        seen = {}

        def train_step(models, embeddings, code_library, b, loss_conf, **kw):
            seen.update(kw, models=models, embeddings=embeddings, code_library=code_library, batch=b, loss_conf=loss_conf)
            # what the library computes, here from the recorded maps: the reference's TotalLoss and PSNR
            loss_sum, loss_dict = ref_loss_fn(maps, b)
            terms = torch.tensor([float(loss_dict[t]) if t in loss_dict else 0.0 for t in training.TERMS])
            present = torch.tensor([int(t in loss_dict) for t in training.TERMS], dtype=torch.int32)
            mask = b["valid_mask"].view(-1, 1).repeat(1, 3)
            return loss_sum.detach(), terms, present, ref_psnr(maps["rgb_fine"], b["rgbs"], mask), []
        monkeypatch.setattr(training, "train_step", train_step)
        gb = {k: v.clone() for k, v in batch.items()}
        loss = sys.training_step(gb, 0)
    finally:
        F.purge_reference_modules()
        R.cuda_noop(not torch.cuda.is_available())

    assert seen["batch"] is gb and seen["models"] is sys.models and seen["embeddings"] is sys.embeddings
    assert seen["code_library"] is sys.code_library and dict(seen["loss_conf"]) == dict(conf["loss"])
    assert sorted(seen) == sorted(STEP_KEYS + ("precision", "grad_sink", "models", "embeddings", "code_library", "batch",
                                      "loss_conf"))
    assert sorted(seen_ref) == sorted(STEP_KEYS + ("models", "embeddings", "rays", "chunk", "embedding_instance"))
    assert seen["precision"] is None and seen["grad_sink"] is True
    for k in STEP_KEYS:
        if isinstance(seen_ref[k], torch.Tensor):
            assert torch.equal(seen[k], seen_ref[k]), k
        else:
            assert seen[k] == seen_ref[k] and type(seen[k]) is type(seen_ref[k]), (k, seen[k], seen_ref[k])
    assert seen["frustum_bound_th"] == over["frustum_bound"] / over["scale_factor"]
    assert seen["rays_in_bbox"] is over["rays_in_bbox"] and seen["is_eval"] is False
    # the same rays, and the codes train_step gathers are the reference's lookup
    assert torch.equal(gb["rays"].reshape(-1, 8), seen_ref["rays"])
    codes = sys.code_library.embedding_instance.weight[gb["instance_ids"].reshape(-1)]
    assert torch.equal(codes, seen_ref["embedding_instance"].detach())
    # the same log calls with the same values; the returned loss carries autograd
    assert list(sys.logged) == list(ref_sys.logged)
    for k, v in ref_sys.logged.items():
        got, want = (float(torch.as_tensor(x).detach()) for x in (sys.logged[k], v))
        assert got == pytest.approx(want, rel=1e-6), k
    assert loss.requires_grad and loss.detach().item() == pytest.approx(loss_ref.detach().item(), rel=1e-6)


# ------------------------------------------------------------------------------------------------
# the gradient sink and TrainStepFn with the library stubbed
# ------------------------------------------------------------------------------------------------
class _SinkFakeLib(_FakeLib):
    """_FakeLib that also adds 1 to the first `table_rows` rows of the voxel-table gradient."""
    table_rows = 0

    def onerf_train_step(self, ctx, a, la, b, psnr, stream):
        rc = super().onerf_train_step(ctx, a, la, b, psnr, stream)
        if self.table_rows:
            self.view(b._obj.table_grad, self.table_rows * 24)[:] += 1.0
        return rc


def _stubbed(monkeypatch):
    from object_nerf_b200 import _lib, engine
    fake = _SinkFakeLib()
    monkeypatch.setattr(_lib, "load", lambda: fake)
    monkeypatch.setattr(_lib, "ctx", lambda dev: None)
    monkeypatch.setattr(_lib, "stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(engine, "RenderPlan", _FakeRenderPlan)
    from object_nerf_b200 import synthetic as S
    from tests import helpers
    inp = cases.build_grad_case()
    models = {k: S.make_model(w, True, "cpu") for k, w in inp["weights"].items()}
    emb = S.GridModule(inp["grid"])
    lib = helpers.CodeLib(inp["code_table"])
    batch = {k: v.clone() for k, v in inp["batch"].items()}
    batch["rays"], batch["instance_ids"] = inp["rays"], inp["instance_ids"]
    kw = dict(N_samples=64, N_importance=64, perturb=1.0, noise_std=1.0, pass_through_mask=inp["pass_through_mask"],
              frustum_bound_th=0.025, precision="bf16")
    return fake, models, {"xyz": emb, "dir": None}, lib, batch, kw


def test_sink_takes_the_gradients_and_is_zeroed_on_every_call(monkeypatch):
    from object_nerf_b200 import engine, training
    fake, models, embeddings, lib, batch, kw = _stubbed(monkeypatch)
    emb = embeddings["xyz"]
    n_used = int(emb.voxel_idx_map.max()) + 1
    fake.table_rows = n_used
    trained = training._trained_tensors(models, ["coarse", "fine"], lib.embedding_instance.weight,
                                        emb.embedding_space_ftr.weight)
    out = training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, grad_sink=True, **kw)
    assert all(t.grad is None for t in trained)
    (plan,) = training._plans[models["coarse"]].values()
    assert plan.bucket is None and plan.sink is not None
    grads = out[4]
    assert grads is plan.sink.views and [g.shape for g in grads] == [t.shape for t in trained]
    # bucket order: fine model first, 40 tensors per model, then the code table, then the voxel table
    (_, _, b), = [c for c in fake.calls if c[0] == "step"]
    for k, typ in enumerate(("fine", "coarse")):
        for i in range(20):
            assert getattr(b, "dW_" + typ)[i] == grads[40 * k + 2 * i].data_ptr()
            assert getattr(b, "db_" + typ)[i] == grads[40 * k + 2 * i + 1].data_ptr()
            assert grads[40 * k + 2 * i].reshape(-1)[0].item() == i + 1
    assert b.table_grad == grads[-1].data_ptr() and (grads[-1][:n_used] == 1).all() and not grads[-1][n_used:].any()
    n = batch["rays"].shape[0]
    want = torch.zeros_like(lib.embedding_instance.weight)
    want.index_add_(0, batch["instance_ids"].reshape(-1), torch.arange(n, dtype=torch.float32)[:, None].expand(n, 64))
    assert torch.equal(grads[80], want)
    assert all(o % 4 == 0 for o in plan.sink.offsets)
    # a second call starts from zero: the same values, not twice them
    before = [g.clone() for g in grads]
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, grad_sink=True, **kw)
    assert all(torch.equal(g, w) for g, w in zip(grads, before))
    assert all(t.grad is None for t in trained)
    # pruning lowers n_used: the rows the earlier grid referenced are still zeroed
    with torch.no_grad():
        emb.voxel_idx_map[emb.voxel_idx_map >= n_used // 2] = -1
    fake.table_rows = n_used // 2
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, grad_sink=True, **kw)
    assert (grads[-1][:n_used // 2] == 1).all() and not grads[-1][n_used // 2:].any()
    assert plan.sink_rows == n_used
    # .grad route unchanged: a plan of its own, gradients in .grad
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    assert len(training._plans[models["coarse"]]) == 2 and all(t.grad is not None for t in trained)
    assert engine.model_linears(models["coarse"])[3][0].grad.reshape(-1)[0].item() == 4
    with pytest.raises(ValueError, match="grad_sink"):
        training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, grad_sink=True, group=object(), **kw)


def test_train_step_fn_returns_scaled_copies_and_refuses_what_it_cannot_do(monkeypatch):
    from object_nerf_b200 import training
    fake, models, embeddings, lib, batch, kw = _stubbed(monkeypatch)
    fake.table_rows = 3
    emb = embeddings["xyz"]
    trained = training._trained_tensors(models, ["coarse", "fine"], lib.embedding_instance.weight,
                                        emb.embedding_space_ftr.weight)
    loss, terms, present, psnr = training.TrainStepFn.run(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    (plan,) = training._plans[models["coarse"]].values()
    assert loss.requires_grad and not terms.requires_grad and not present.requires_grad and not psnr.requires_grad
    assert loss.item() == 1 and terms.tolist() == [2, 3, 4, 5, 6] and present.tolist() == [1, 1, 0, 1, 0]
    assert loss.data_ptr() != plan.out.data_ptr()
    (0.5 * loss).backward()
    for t, g in zip(trained, plan.sink.views):
        assert torch.equal(t.grad, 0.5 * g), t.shape
        assert not (plan.sink.flat.data_ptr() <= t.grad.data_ptr() < plan.sink.flat.data_ptr() + 4 * plan.sink.flat.numel())
    kept = [t.grad.clone() for t in trained]
    loss, *_ = training.TrainStepFn.run(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    loss.backward()
    assert all(torch.equal(t.grad, 3 * k) for t, k in zip(trained, kept))
    # a backward after the next step of the same plan would read that step's gradients
    stale, *_ = training.TrainStepFn.run(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    training.TrainStepFn.run(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    with pytest.raises(RuntimeError, match="overwritten"):
        stale.backward()
    with torch.no_grad(), pytest.raises(RuntimeError, match="grad mode"):
        training.TrainStepFn.run(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    for t in trained:
        t.requires_grad_(False)
    with pytest.raises(RuntimeError, match="requires grad"):
        training.TrainStepFn.run(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
