"""Device-side Philox seed (onerf_render_rays_fwd_dseed, onerf_train_step_dseed, training.train_step under CUDA-graph
capture): a call that reads its seed from device memory draws exactly what the host-seed call with that value draws,
advances the counter by 4, and so every replay of a captured step or forward draws fresh jitter, importance u and sigma
noise."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from tests import cases, grad_plain
from tests.test_gpu_train_step import _assert_same_grads, _batch, _kwargs, _named, _setup

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 0x1234_5678_9ABC


def _case(use_voxel):
    inp = cases.build_grad_case() if use_voxel else grad_plain.build_grad_case_plain()
    return inp, (cases.GRAD_CASE if use_voxel else grad_plain.GRAD_CASE_PLAIN)


def _step_once(monkeypatch, inp, use_voxel, kw, seed, device_seed):
    """One train_step after a plan-creating first call (its gradients are discarded): with host seed `seed`, or through
    onerf_train_step_dseed with the plan's counter set to `seed`.  Returns the loss outputs, maps, named parameters and
    the counter after the step."""
    from object_nerf_b200 import engine, training
    batch = _batch(inp)
    models, embeddings, lib = _setup(inp, use_voxel)
    named = _named(models, embeddings, lib)
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    for _, p in named:
        p.grad.zero_()
    (plan,) = training._plans[models["coarse"]].values()
    with monkeypatch.context() as m:
        if device_seed:
            plan.seed_dev.fill_(seed)
            m.setattr(training, "_capturing", lambda dev: True)
            m.setattr(engine, "new_seed", lambda: pytest.fail("the device-seed route drew a host seed"))
        else:
            m.setattr(engine, "new_seed", lambda: seed)
        out = training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    torch.cuda.synchronize()
    maps = {f"{k}_{typ}": v.clone() for typ, mp in plan.render.maps.items() for k, v in mp.items()}
    return [t.clone() for t in out], maps, named, plan.seed_dev.item()


def _assert_step_equal(res_h, res_d):
    (out_h, maps_h, named_h, _), (out_d, maps_d, named_d, _) = res_h, res_d
    for k in maps_h:
        assert torch.equal(maps_h[k], maps_d[k]), k
    loss_h, terms_h, present_h, psnr_h = out_h
    loss_d, terms_d, present_d, psnr_d = out_d
    assert torch.equal(present_h, present_d)
    for a, b in ((loss_h, loss_d), (psnr_h, psnr_d)):
        assert abs(a.item() - b.item()) <= 1e-6 * abs(b.item()), (a.item(), b.item())
    assert torch.allclose(terms_h, terms_d, rtol=1e-6, atol=0)
    _assert_same_grads(named_d, named_h, 1e-6, 0.999999)


@pytest.mark.parametrize("use_voxel,precision", [(True, "fp32"), (True, "bf16"), (False, "fp32"), (False, "bf16")])
def test_device_seed_step_draws_what_the_host_seed_step_draws(monkeypatch, use_voxel, precision):
    """onerf_train_step with seed s and onerf_train_step_dseed with *seed_dev = s: bit-identical maps, loss and PSNR
    within 1e-6 (fp64 block sums in a different order), gradients within fp32 accumulation order; the counter is s + 4."""
    inp, c = _case(use_voxel)
    kw = _kwargs(c, inp, precision, None)
    assert kw["perturb"] == 1 and kw["noise_std"] == 1
    res_h = _step_once(monkeypatch, inp, use_voxel, kw, SEED, False)
    res_d = _step_once(monkeypatch, inp, use_voxel, kw, SEED, True)
    _assert_step_equal(res_h, res_d)
    assert res_d[3] == SEED + 4


def test_injected_buffers_win_over_the_device_seed(monkeypatch):
    """With `_rand` buffers the seeds are unused: a device-seed step equals a host-seed step with another seed."""
    inp, c = _case(True)
    kw = _kwargs(c, inp, "fp32", {k: v.to(DEV) for k, v in inp["rand"].items()})
    res_h = _step_once(monkeypatch, inp, True, kw, 1, False)
    res_d = _step_once(monkeypatch, inp, True, kw, SEED, True)
    _assert_step_equal(res_h, res_d)
    assert res_d[3] == SEED + 4


def _render_plan(use_voxel, precision, perturb=1.0, noise_std=1.0):
    from object_nerf_b200 import Embedding, engine
    from object_nerf_b200.rendering import _grid_of
    from tests import helpers
    inp, c = _case(use_voxel)
    models = {k: helpers.make_model(w, use_voxel, DEV) for k, w in inp["weights"].items()}
    emb = helpers.GridModule(inp["grid"]).to(DEV) if use_voxel else Embedding(3, 10)
    plan = engine.RenderPlan(
        inp["rays"].to(DEV), engine.packed_for(models["coarse"], use_voxel), engine.packed_for(models["fine"], use_voxel),
        _grid_of(emb), codes=inp["codes"].to(DEV), n_samples=c["n_samples"], n_importance=c["n_importance"],
        use_disp=c["use_disp"], perturb=perturb, noise_std=noise_std, white_back=c["white_back"], forward_instance=True,
        is_eval=False, frustum_bound_th=c["frustum_bound_th"], pass_through_mask=inp["pass_through_mask"].to(DEV),
        precision=precision)
    return plan, inp, c, (models, emb)


@pytest.mark.parametrize("use_voxel,precision", [(True, "fp32"), (True, "bf16"), (False, "bf16")])
def test_device_seed_forward_draws_what_the_host_seed_forward_draws(use_voxel, precision):
    plan, _, _, _keep = _render_plan(use_voxel, precision)
    plan.args.seed = SEED
    host = {k: v.clone() for k, v in plan.run().items()}
    seed_dev = torch.full((1,), SEED, dtype=torch.int64, device=DEV)
    plan.args.seed = 7          # ignored by the device-seed entry
    dev = {k: v.clone() for k, v in plan.run(seed_dev).items()}
    torch.cuda.synchronize()
    for k in host:
        assert torch.equal(host[k], dev[k]), k
    assert seed_dev.item() == SEED + 4


def test_counter_advances_when_nothing_is_drawn():
    plan, _, _, _keep = _render_plan(True, "bf16", perturb=0.0, noise_std=0.0)
    seed_dev = torch.full((1,), 40, dtype=torch.int64, device=DEV)
    eager = {k: v.clone() for k, v in plan.run().items()}
    out = plan.run(seed_dev)
    torch.cuda.synchronize()
    assert seed_dev.item() == 44
    for k in eager:
        assert torch.equal(eager[k], out[k]), k


def test_train_step_replays_draw_fresh_numbers(monkeypatch):
    """train_step + Adam(capturable=True) captured after a warm-up, without `_rand`, replayed 4 times: the coarse depths
    differ between every pair of replays; replay k draws what an eager step with seed s0 + 4k draws (same depths bit for
    bit, loss within 1e-6 on the same parameters); after 3 replays the parameters match 3 eager Adam steps with seeds
    s0, s0 + 4, s0 + 8 within the bf16 gate of test_step_and_adam_replay_in_a_cuda_graph (5 % of the distance moved),
    taken over all parameters together: Adam turns the sign of a near-zero gradient element into a full lr step, so
    gradients that differ in their last bits (atomic accumulation order) can move single elements of one small tensor
    apart by several lr; over the whole model they are a small share of the motion."""
    from object_nerf_b200 import engine, training
    inp, c = _case(True)
    batch = _batch(inp)
    kw = _kwargs(c, inp, "bf16", None)
    warm_seed = 0x5EED

    def arm():
        models, embeddings, lib = _setup(inp, True)
        named = _named(models, embeddings, lib)
        opt = torch.optim.Adam([p for _, p in named], lr=1e-3, capturable=True)

        def step():
            opt.zero_grad(set_to_none=False)
            out = training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
            opt.step()
            return out

        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with monkeypatch.context() as m, torch.cuda.stream(s):
            m.setattr(engine, "new_seed", lambda: warm_seed)
            step()        # warm-up: the plan (its counter = warm_seed + 4), the gradients and Adam's state
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        return models, embeddings, lib, named, step

    # graphed arm
    models_g, _, _, named_g, step_g = arm()
    s0 = training.step_seed(models_g).item()
    assert s0 == warm_seed + 4
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step_g()
    (plan_g,) = training._plans[models_g["coarse"]].values()
    # same-parameter reference: before each replay its parameters are set to the graphed arm's, then one eager step
    models_r, emb_r, lib_r, named_r, _ = arm()
    (plan_r,) = training._plans[models_r["coarse"]].values()
    zs, after3 = [], None
    for k in range(4):
        with torch.no_grad():
            for (_, pr), (_, pg) in zip(named_r, named_g):
                pr.copy_(pg)
        g.replay()
        torch.cuda.synchronize()
        zs.append(plan_g.render.maps["coarse"]["z_vals"].clone())
        loss_g = plan_g.out[0].item()
        with monkeypatch.context() as m:
            m.setattr(engine, "new_seed", lambda: s0 + 4 * k)
            loss_r = training.train_step(models_r, emb_r, lib_r, batch, cases.LOSS_CONF, **kw)[0].item()
        torch.cuda.synchronize()
        assert torch.equal(plan_r.render.maps["coarse"]["z_vals"], zs[k]), k
        assert torch.equal(plan_r.render.maps["fine"]["z_vals"], plan_g.render.maps["fine"]["z_vals"]), k
        assert abs(loss_g - loss_r) <= 1e-6 * abs(loss_r), (k, loss_g, loss_r)
        if k == 2:
            after3 = [p.detach().clone() for _, p in named_g]
    assert training.step_seed(models_g).item() == s0 + 16
    for i, j in itertools.combinations(range(4), 2):
        assert not torch.equal(zs[i], zs[j]), (i, j)
    # eager Adam steps with the replays' seeds
    models_e, _, _, named_e, step_e = arm()
    start = [p.detach().clone() for _, p in named_e]
    seeds = iter([s0, s0 + 4, s0 + 8])
    with monkeypatch.context() as m:
        m.setattr(engine, "new_seed", lambda: next(seeds))
        for _ in range(3):
            step_e()
    torch.cuda.synchronize()
    flat = lambda ts: torch.cat([t.reshape(-1) for t in ts])
    pe = flat([p.detach() for _, p in named_e])
    moved = (pe - flat(start)).norm().item()
    diff = (flat(after3) - pe).norm().item()
    assert diff <= 5e-2 * moved, (diff, moved)


def test_forward_replays_draw_uniform_jitter():
    """32 replays of a captured onerf_render_rays_fwd_dseed (perturb = 1): the jitter u = (z - lower) / (upper - lower)
    implied by the coarse depths, with the stratified bins of rendering.py:268-277, pooled over the replays is U[0, 1)
    (Kolmogorov-Smirnov, p > 1e-3), and no two replays draw the same depths."""
    from scipy import stats
    plan, inp, c, _keep = _render_plan(True, "bf16", noise_std=0.0)
    seed_dev = torch.full((1,), SEED, dtype=torch.int64, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out = plan.run(seed_dev)                        # warm-up on the capture stream
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            out = plan.run(seed_dev)
    torch.cuda.current_stream().wait_stream(side)
    zs = []
    for _ in range(32):
        g.replay()
        torch.cuda.synchronize()
        zs.append(out["z_vals_coarse"].double().cpu())
    assert seed_dev.item() == SEED + 4 * 33
    assert len({z.numpy().tobytes() for z in zs}) == 32
    S = c["n_samples"]
    rays = inp["rays"].double()
    t = torch.linspace(0, 1, S, dtype=torch.float64)
    z = rays[:, 6:7] * (1 - t) + rays[:, 7:8] * t
    mids = 0.5 * (z[:, 1:] + z[:, :-1])
    upper, lower = torch.cat([mids, z[:, -1:]], 1), torch.cat([z[:, :1], mids], 1)
    u = torch.cat([((zz - lower) / (upper - lower)).reshape(-1) for zz in zs]).numpy()
    assert u.min() >= -1e-4 and u.max() < 1 + 1e-4, (u.min(), u.max())
    p = stats.kstest(np.clip(u, 0, 1), "uniform").pvalue
    assert p > 1e-3, p


def test_device_seed_entries_refuse_bad_arguments():
    """NULL seed_dev is ONERF_ERR_BAD_ARG on a live context; so is a training workspace on the forward-only entry."""
    from object_nerf_b200 import _lib
    lib = _lib.load()
    plan, _, _, _keep = _render_plan(True, "bf16")
    ctx, stream = _lib.ctx(torch.device(DEV)), _lib.stream()
    assert lib.onerf_render_rays_fwd_dseed(ctx, C.byref(plan.args), None, stream) == -1
    assert b"null" in lib.onerf_last_error()
    seed_dev = torch.zeros(1, dtype=torch.int64, device=DEV)
    ws = torch.empty(4096, dtype=torch.uint8, device=DEV)
    plan.args.train_ws, plan.args.train_ws_bytes = ws.data_ptr(), ws.numel()
    assert lib.onerf_render_rays_fwd_dseed(ctx, C.byref(plan.args), seed_dev.data_ptr(), stream) == -1
    assert b"train_ws" in lib.onerf_last_error()
    la, b = _lib.LossArgs(), _lib.RenderBwdArgs()
    psnr = torch.zeros(1, device=DEV)
    assert lib.onerf_train_step_dseed(ctx, C.byref(plan.args), C.byref(la), C.byref(b), psnr.data_ptr(), None, stream) == -1
    assert b"seed_dev" in lib.onerf_last_error()
    torch.cuda.synchronize()
    assert seed_dev.item() == 0


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")
def test_first_train_step_inside_a_capture_is_refused():
    """A plan made inside a capture would have its counter write captured and every replay would reset the seed."""
    from object_nerf_b200 import training
    inp, c = _case(True)
    batch = _batch(inp)
    kw = _kwargs(c, inp, "bf16", None)
    models, embeddings, lib = _setup(inp, True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="warm up"):
        with torch.cuda.graph(g, stream=s):
            training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    torch.cuda.current_stream().wait_stream(s)
    assert models["coarse"] not in training._plans or not training._plans[models["coarse"]]
