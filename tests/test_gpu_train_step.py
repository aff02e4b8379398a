"""training.train_step (onerf_train_step: render, TotalLoss and backward in one call, loss and compositing backward fused
into the compositing kernels) against the existing route render_rays -> losses.TotalLoss -> loss.backward() on the same
seeded batch, and against the reference's own backward (fixtures)."""
import pytest
import torch

from tests import cases, grad_plain, helpers, synth
from tests.test_fp32_backward_cpu import FUSED_STEP_SHAPES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TERMS = ("color_loss", "depth_loss", "opacity_loss", "instance_color_loss", "instance_depth_loss")


def _setup(inp, use_voxel, fine=True):
    from object_nerf_b200 import Embedding
    models = {k: helpers.make_model(w, use_voxel, DEV).train() for k, w in inp["weights"].items() if fine or k == "coarse"}
    emb = helpers.GridModule(inp["grid"]).to(DEV) if use_voxel else Embedding(3, 10)
    lib = helpers.CodeLib(inp["code_table"]).to(DEV)
    return models, {"xyz": emb, "dir": Embedding(3, 4)}, lib


def _named(models, embeddings, lib):
    named = [(f"{typ}.{k}", p) for typ, m in models.items() for k, p in m.named_parameters()]
    named.append(("codes", lib.embedding_instance.weight))
    if hasattr(embeddings["xyz"], "embedding_space_ftr"):
        named.append(("voxel", embeddings["xyz"].embedding_space_ftr.weight))
    return named


def _kwargs(c, inp, precision, rand, **over):
    kw = dict(N_samples=c["n_samples"], perturb=c["perturb"], noise_std=c["noise_std"], N_importance=c["n_importance"],
              frustum_bound_th=c["frustum_bound_th"], pass_through_mask=inp["pass_through_mask"].to(DEV), is_eval=False,
              rays_in_bbox=False, precision=precision, _rand=rand)
    kw.update(over)
    return kw


def _batch(inp):
    b = {k: v.to(DEV) for k, v in inp["batch"].items()}
    b["rays"] = inp["rays"].to(DEV)
    b["instance_ids"] = inp["instance_ids"].to(DEV)
    return b


def _existing(inp, use_voxel, batch, kw):
    from object_nerf_b200 import render_rays
    from object_nerf_b200.losses import TotalLoss
    models, embeddings, lib = _setup(inp, use_voxel, kw["N_importance"] > 0)
    codes = lib.embedding_instance(batch["instance_ids"].view(-1))
    out = render_rays(models, embeddings, batch["rays"], embedding_instance=codes, **kw)
    loss_sum, loss_dict = TotalLoss(cases.LOSS_CONF)(out, batch)
    loss_sum.backward()
    return loss_sum.detach(), loss_dict, {k: v.detach() for k, v in out.items()}, _named(models, embeddings, lib)


def _fused(inp, use_voxel, batch, kw):
    from object_nerf_b200 import training
    models, embeddings, lib = _setup(inp, use_voxel, kw["N_importance"] > 0)
    loss_sum, terms, present, psnr = training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    torch.cuda.synchronize()
    (plan,) = training._plans[models["coarse"]].values()
    maps = {f"{k}_{typ}": v for typ, m in plan.render.maps.items() for k, v in m.items()}
    return (loss_sum.clone(), terms.clone(), present.clone(), psnr.clone()), maps, _named(models, embeddings, lib)


def _compare(inp, use_voxel, precision, rand, batch=None, loss_tol=1e-5, norm_tol=1e-5, cos_min=0.99999, **over):
    c = cases.GRAD_CASE if use_voxel else grad_plain.GRAD_CASE_PLAIN
    batch = batch or _batch(inp)
    kw = _kwargs(c, inp, precision, rand, **over)
    loss_e, dict_e, maps_e, named_e = _existing(inp, use_voxel, batch, kw)
    (loss_f, terms_f, present_f, psnr_f), maps_f, named_f = _fused(inp, use_voxel, batch, kw)
    assert abs(loss_f.item() - loss_e.item()) <= loss_tol * abs(loss_e.item()), (loss_f.item(), loss_e.item())
    flags = present_f.tolist()
    dict_f = {t: terms_f[i] for i, t in enumerate(TERMS) if flags[i]}
    assert sorted(dict_f) == sorted(dict_e), (dict_f, dict_e)
    for t in dict_e:
        assert abs(dict_f[t].item() - dict_e[t].item()) <= loss_tol * abs(dict_e[t].item()) + 1e-12, t
    for k, v in maps_e.items():
        assert torch.equal(maps_f[k], v), k
    _assert_same_grads(named_f, named_e, norm_tol, cos_min)
    return loss_f, psnr_f, maps_f, batch, named_f


def _assert_same_grads(named_f, named_e, norm_tol, cos_min):
    bad = []
    for (name, p), (_, q) in zip(named_f, named_e):
        assert p.grad is not None and q.grad is not None, name
        gf, ge = p.grad.reshape(-1).double(), q.grad.reshape(-1).double()
        rel = ((gf - ge).norm() / (ge.norm() + 1e-30)).item()
        cos = (gf @ ge / (gf.norm() * ge.norm() + 1e-30)).item()
        if ge.norm() == 0:
            if gf.norm() != 0:      # a gradient where the existing route has none
                bad.append((name, gf.norm().item(), 0.0))
        elif not (rel <= norm_tol and cos >= cos_min):
            bad.append((name, rel, cos))
    assert not bad, bad


def _voxel_case():
    inp = cases.build_grad_case()
    return inp, {k: v.to(DEV) for k, v in inp["rand"].items()}


def _plain_case():
    inp = grad_plain.build_grad_case_plain()
    return inp, {k: v.to(DEV) for k, v in inp["rand"].items()}


@pytest.mark.parametrize("use_voxel", [True, False])
def test_fp32_step_matches_existing_route(use_voxel):
    """Same fp32 kernels in both routes: loss / terms / flags within 1e-5, gradients within 1e-5 relative norm and
    cosine >= 0.99999 (only the order of accumulation differs), maps bit-identical."""
    inp, rand = _voxel_case() if use_voxel else _plain_case()
    _compare(inp, use_voxel, "fp32", rand)


@pytest.mark.parametrize("use_voxel", [True, False])
def test_bf16_step_matches_existing_route_and_reference(golden, use_voxel):
    """Tensor-core step against the existing route (loss 2e-2, norm 5e-2, cosine 0.995) and against the reference's own
    backward (fixture): loss within 2 %, per-tensor gradient norm within 5 %."""
    inp, rand = _voxel_case() if use_voxel else _plain_case()
    loss, _, _, _, named = _compare(inp, use_voxel, "bf16", rand, loss_tol=2e-2, norm_tol=5e-2, cos_min=0.995)
    g = golden("grad_train_step" if use_voxel else "grad_train_step_plain")
    assert abs(loss.item() - g["loss"].item()) <= 2e-2 * abs(g["loss"].item()), (loss.item(), g["loss"].item())
    bad = []
    for name, p in named:
        ref = g[name + "|norm"].item()
        ratio = p.grad.norm().item() / max(ref, 1e-12)
        if not 0.95 <= ratio <= 1.05:
            bad.append((name, ratio))
    assert not bad, bad


@pytest.mark.parametrize("empty", ["depth", "instance"])
def test_skipped_terms_match_total_loss(empty):
    """No target depth > 0, or an empty instance mask: the same present flags and loss_dict as TotalLoss."""
    inp, rand = _voxel_case()
    batch = _batch(inp)
    if empty == "depth":
        batch["depths"] = torch.zeros_like(batch["depths"])
    else:
        batch["instance_mask"] = torch.zeros_like(batch["instance_mask"])
    _compare(inp, True, "fp32", rand, batch=batch)


SHAPE_MODES = {"shape_33_30": (33, 30), "shape_3_1": (3, 1), "shape_2_1": (2, 1), "shape_1024_1024": (1024, 1024)}


@pytest.mark.parametrize("mode", ["rays_in_bbox", "no_pass_through", "is_eval", "coarse_only"] + list(SHAPE_MODES))
def test_modes_match_existing_route(mode):
    """rays_in_bbox, the occlusion mask without pass-through rays, is_eval and N_importance = 0 (the coarse pass writes
    the loss outputs and the PSNR); and (S, K) shapes off the 64 + 64 default on a few rays: a partial last warp chunk,
    the smallest sort buffers (S = 2: no pdf weight at all) and S + K = 2048, the shared-memory limit of the step's
    compositing kernel (4 warps x 4 S floats)."""
    inp, rand = _voxel_case()
    if mode in SHAPE_MODES:
        S, K = SHAPE_MODES[mode]
        n = 4 if S + K > 256 else 9
        inp = cases.build_grad_case(n_rays=n)
        inp["rand"] = synth.random_buffers(cases.GRAD_CASE["seed"] + 4, n, S, K)
        rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
        _compare(inp, True, "fp32", rand, N_samples=S, N_importance=K)
        return
    over = {"rays_in_bbox": dict(rays_in_bbox=True),
            "no_pass_through": dict(pass_through_mask=None),
            "is_eval": dict(is_eval=True),
            "coarse_only": dict(N_importance=0)}[mode]
    if mode == "coarse_only":
        rand = {k: v for k, v in rand.items() if not k.endswith("fine") and k != "u"}
    _compare(inp, True, "fp32", rand, **over)


@pytest.mark.parametrize("n_importance", [64, 0])
def test_psnr_is_the_reference_formula_on_the_returned_rgb(n_importance):
    """utils/metrics.py: psnr = -10 log10(mean over valid rays x 3 of (rgb - rgbs)^2) of the last pass (train.py:171)."""
    inp, rand = _voxel_case()
    if n_importance == 0:
        rand = {k: v for k, v in rand.items() if not k.endswith("fine") and k != "u"}
    _, psnr, maps, batch, _ = _compare(inp, True, "fp32", rand, N_importance=n_importance)
    typ = "fine" if n_importance else "coarse"
    mask = batch["valid_mask"].view(-1, 1).repeat(1, 3)
    mse = torch.mean((maps[f"rgb_{typ}"] - batch["rgbs"])[mask] ** 2)
    want = (-10 * torch.log10(mse)).item()
    assert abs(psnr.item() - want) <= 1e-4 * abs(want), (psnr.item(), want)


@pytest.mark.parametrize("shape", list(FUSED_STEP_SHAPES))
def test_fp32_step_at_batch_size_matches_existing_route(shape):
    """The fp32 comparison of test_fp32_step_matches_existing_route at batch size: 2 048 rays x 64 + 64 samples (512
    compositing blocks, more than the SMs, so the last block that finalises the loss runs in a later wave than the
    first; two fp32 chunks per pass) and 1 100 rays x 64 + 63 (ragged last chunks in both passes: 1 024 + 76 and
    516 + 516 + 68).  The PSNR output is the reference formula on the returned rgb."""
    n, S, K = FUSED_STEP_SHAPES[shape]
    inp = cases.build_grad_case(n_rays=n)
    inp["rand"] = synth.random_buffers(cases.GRAD_CASE["seed"] + 4, n, S, K)
    rand = {k: v.to(DEV) for k, v in inp["rand"].items()}
    _, psnr, maps, batch, _ = _compare(inp, True, "fp32", rand, N_samples=S, N_importance=K)
    mask = batch["valid_mask"].view(-1, 1).repeat(1, 3)
    want = (-10 * torch.log10(torch.mean((maps["rgb_fine"] - batch["rgbs"])[mask] ** 2))).item()
    assert abs(psnr.item() - want) <= 1e-4 * abs(want), (psnr.item(), want)


def test_step_and_adam_replay_in_a_cuda_graph():
    """One train_step + Adam(capturable=True) captured in a CUDA graph (the capture fails on any host read) and replayed
    three times: the parameters match three eager steps within the bf16 gate."""
    from object_nerf_b200 import training
    inp, rand = _voxel_case()
    batch = _batch(inp)
    kw = _kwargs(cases.GRAD_CASE, inp, "bf16", rand)
    runs = []
    for graphed in (False, True):
        models, embeddings, lib = _setup(inp, True)
        named = _named(models, embeddings, lib)
        params = [p for _, p in named]
        opt = torch.optim.Adam(params, lr=1e-3, capturable=True)

        def step():
            opt.zero_grad(set_to_none=False)
            training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
            opt.step()

        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()        # warm-up: the step's plan, the gradients and Adam's state are created here
        torch.cuda.current_stream().wait_stream(s)
        start = [p.detach().clone() for p in params]
        if graphed:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                step()
            for _ in range(3):
                g.replay()
        else:
            for _ in range(3):
                step()
        torch.cuda.synchronize()
        runs.append((named, start))
    (named_e, start_e), (named_g, _) = runs
    bad = []
    for (name, pe), (_, pg), p0 in zip(named_e, named_g, start_e):
        moved = (pe.detach() - p0).norm().item()
        diff = (pg.detach() - pe.detach()).norm().item()
        if diff > 5e-2 * moved + 1e-7:
            bad.append((name, diff, moved))
    assert not bad, bad


def test_step_follows_voxel_subdivision():
    """voxel_subdivision between two steps (train.py:140-145) replaces the index map and the voxel size and doubles the
    shape in place: the second step must run on the new grid, as the existing route (which reads the grid on every call)
    does.  Rays aimed through occupied voxels, fp32, compared as in the tests above."""
    from object_nerf_b200 import Embedding, render_rays, training
    from object_nerf_b200.losses import TotalLoss
    from tests.test_host_logic_cpu import _maint_embedding
    inp, rand = _voxel_case()
    n = inp["rays"].shape[0]
    kw = _kwargs(cases.GRAD_CASE, inp, "fp32", rand)
    embs = [_maint_embedding()[0].to(DEV) for _ in range(2)]
    _, centres = embs[0]._occupied()
    g = torch.Generator().manual_seed(11)
    pick = centres[torch.randint(0, centres.shape[0], (n,), generator=g).to(DEV)]
    d = torch.randn(n, 3, generator=g).to(DEV)
    d = d / d.norm(dim=1, keepdim=True)
    near, far = torch.full((n, 1), 0.5, device=DEV), torch.full((n, 1), 1.5, device=DEV)
    batch = _batch(inp)
    batch["rays"] = torch.cat([pick - d, d, near, far], 1).contiguous()

    def setup(emb):
        models = {k: helpers.make_model(w, True, DEV).train() for k, w in inp["weights"].items()}
        lib = helpers.CodeLib(inp["code_table"]).to(DEV)
        embeddings = {"xyz": emb, "dir": Embedding(3, 4)}
        return models, embeddings, lib, _named(models, embeddings, lib)

    models, embeddings, lib, named_f = setup(embs[0])
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)     # the plan is made on the old grid
    for emb in embs:
        assert emb.voxel_subdivision() > 0
    for _, p in named_f:
        p.grad.zero_()
    loss_f, _, _, _ = training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    torch.cuda.synchronize()
    (plan,) = training._plans[models["coarse"]].values()
    maps_f = {f"{k}_{typ}": v for typ, m in plan.render.maps.items() for k, v in m.items()}

    models_e, embeddings_e, lib_e, named_e = setup(embs[1])
    out = render_rays(models_e, embeddings_e, batch["rays"], embedding_instance=lib_e.embedding_instance(
        batch["instance_ids"].view(-1)), **kw)
    loss_e, _ = TotalLoss(cases.LOSS_CONF)(out, batch)
    loss_e.backward()
    assert abs(loss_f.item() - loss_e.item()) <= 1e-5 * abs(loss_e.item()), (loss_f.item(), loss_e.item())
    for k, v in out.items():
        assert torch.equal(maps_f[k], v.detach()), k
    assert embs[1].embedding_space_ftr.weight.grad.norm() > 0      # the rays do reach the grid
    _assert_same_grads(named_f, named_e, 1e-5, 0.99999)


def _step_and_validation(dev, precision):
    """One train_step and one validate_frame on the voxel case with every tensor on `dev`: their outputs, the gradients
    and the step's maps, copied to the host."""
    from object_nerf_b200 import Embedding, training
    torch.manual_seed(0)
    inp = cases.build_grad_case()
    models = {k: helpers.make_model(w, True, dev).train() for k, w in inp["weights"].items()}
    embeddings = {"xyz": helpers.GridModule(inp["grid"]).to(dev), "dir": Embedding(3, 4)}
    lib = helpers.CodeLib(inp["code_table"]).to(dev)
    batch = {k: v.to(dev) for k, v in inp["batch"].items()}
    batch["rays"], batch["instance_ids"] = inp["rays"].to(dev), inp["instance_ids"].to(dev)
    kw = _kwargs(cases.GRAD_CASE, inp, precision, {k: v.to(dev) for k, v in inp["rand"].items()},
                 pass_through_mask=inp["pass_through_mask"].to(dev))
    step = training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    (plan,) = training._plans[models["coarse"]].values()
    maps = [v for m in plan.render.maps.values() for v in m.values()]
    val = training.validate_frame(models, embeddings, lib, {k: v[None] for k, v in batch.items()}, cases.LOSS_CONF,
                                  N_samples=kw["N_samples"], N_importance=kw["N_importance"], use_disp=False,
                                  white_back=False, precision=precision)
    torch.cuda.synchronize(dev)
    grads = [p.grad for _, p in _named(models, embeddings, lib)]
    return [t.cpu() for t in list(step) + maps + grads + list(val.values())]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_step_and_validation_on_a_device_that_is_not_current(precision):
    """train_step and validate_frame on tensors of cuda:1 while cuda:0 is current compute bit for bit what they compute
    with cuda:1 current: every launch goes to the tensors' device and that device's current stream."""
    with torch.cuda.device(1):
        want = _step_and_validation("cuda:1", precision)
    assert torch.cuda.current_device() == 0
    got = _step_and_validation("cuda:1", precision)
    assert torch.cuda.current_device() == 0
    assert len(got) == len(want)
    bits = lambda t: t.reshape(-1).view(torch.uint8)
    assert all(torch.equal(bits(g), bits(w)) for g, w in zip(got, want))
