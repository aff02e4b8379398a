"""The rest of the render forward stage by stage against references of the same operation on the fp32 inputs the kernels
read: stratified coarse depths (onerf_sample_coarse), inverse-CDF importance sampling (onerf_sample_pdf) and its fused
form with the sorted merge (onerf_sample_pdf_merge), the importance draws' Philox stream, and the compositing forward
(onerf_composite) in every flag set, at shapes around the warp width, the power-of-two sort buffer, the 2048-sample
limit and the grid caps; then the two-coarse-sample forward and the S + K > 2048 refusal of the one-call entry points.
Coarse depths and the merged depths are compared bit for bit; importance samples and compositing within the a-priori
gates of tests/test_sampling_stages_cpu.py, where the references and gates themselves are checked.  Each check prints
the largest share of its gate that a result used (RATIO label: x)."""
import ctypes as C
from collections import Counter

import numpy as np
import pytest
import torch

from oracle import onerf_oracle as O
from tests import cases, synth
from tests.test_gpu_parity import _plan_for_case, _run_render_case, grid_obj
from tests.test_gpu_train_stages import COMPOSITE_MODES, SEED
from tests.test_sampling_stages_cpu import (COARSE_S, COMPOSITE_S, F32, MERGE_MANY_RAYS, MERGE_SHAPES, N_PLANT, PDF_SHAPES,
                                            ULP_64, coarse_depth32, coarse_depth64, coarse_jitter, coarse_rays,
                                            composite_inputs, composite_refs, disp_ok, gate_share, inside,
                                            linspace01_32, merge_inputs, merge_reference, occlusion_edge, pdf_gate,
                                            pdf_inputs)
from tests.test_train_stages_cpu import philox_uniform

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _report(label, r):
    print(f"RATIO {label}: {r:.3e}")
    return r


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _np(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _engine():
    from object_nerf_b200 import engine
    return engine


# ------------------------------------------------------------------------------------------------
# coarse depths
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", COARSE_S)
def test_sample_coarse_is_coarse_depth32_bit_for_bit(S):
    """onerf_sample_coarse on 1 ray, 37 rays (near = far and near = far = 0 planted) and enough rays that n S exceeds one
    grid (16 blocks x 256 threads x SMs), with and without use_disp, perturb 0 / 1 and injected jitter holding 0 and
    1 - 2^-24: bit-identical to coarse_depth32 (NaN = NaN on the near = 0 rays of use_disp, which divide by zero in the
    reference too), within ULP_64 ulp of the float64 formula.  The device-RNG jitter keeps every depth inside its stratum."""
    eng = _engine()
    worst = 0.0
    for n in (1, N_PLANT, 16 * 256 * _sms() // S + 1):
        rays = coarse_rays(n, S + n)
        jit = coarse_jitter(n, S, S + n + 1)
        R, J = _t(rays), _t(jit)
        for use_disp in (False, True):
            ok = disp_ok(rays) if use_disp else np.ones(n, bool)
            for perturb in (0.0, 1.0):
                got = _np(eng.sample_coarse(R, S, use_disp, perturb, J))
                want = coarse_depth32(rays, S, use_disp, perturb, jit)
                assert np.array_equal(got[ok], want[ok]), (n, use_disp, perturb)
                assert np.array_equal(got[~ok], want[~ok], equal_nan=True), (n, use_disp, perturb)
                z64 = coarse_depth64(rays, S, use_disp, perturb, jit)[ok]
                ulp = np.spacing(np.abs(z64).astype(F32)).astype(np.float64) + 1e-30
                worst = max(worst, float((np.abs(got[ok] - z64) / (ULP_64 * ulp)).max(initial=0.0)))
        z = _np(eng.sample_coarse(R, S, False, 1.0, None, seed=123))
        lo = coarse_depth32(rays, S, perturb=1.0, jitter=np.zeros((n, S), F32))
        hi = coarse_depth32(rays, S, perturb=1.0, jitter=np.ones((n, S), F32))
        # (near = far rays: the unjittered depths may wobble by an ulp, so a stratum's ends can come in either order)
        assert (z >= np.minimum(lo, hi)).all() and (z <= np.maximum(lo, hi)).all()
        assert (np.diff(z[rays[:, 7] > rays[:, 6]], axis=1) >= 0).all()
    _report(f"sample_coarse S={S} vs float64 ({ULP_64} ulp)", worst)
    assert worst <= 1.0


# ------------------------------------------------------------------------------------------------
# importance sampling
# ------------------------------------------------------------------------------------------------
def _pdf_check(label, got, bins, w, u):
    lo, ref, hi = pdf_gate(bins, w, u)
    share = gate_share(got, lo, ref, hi)
    interior = u < 0.999
    share_in = gate_share(got[interior], lo[interior], ref[interior], hi[interior])
    _report(label, share)
    _report(label + " (u < 0.999)", share_in)
    assert inside(got, lo, hi), (label, share)


@pytest.mark.parametrize("n_bins,K", PDF_SHAPES)
def test_sample_pdf_inside_the_float64_gate(n_bins, K):
    """onerf_sample_pdf on the planted rows of pdf_inputs (all-zero, one-hot, empty stretches, empty tail, zero-width
    bins), with injected u (0, 1 - 2^-24, mid guarded bin, draws away from the knots) and with det = 1 (u = 1 exactly):
    inside pdf_gate.  One bin (no weights) returns that bin for every draw."""
    eng = _engine()
    bins, w, u = pdf_inputs(N_PLANT, n_bins, K, n_bins * 1000 + K)
    B, W = _t(bins), _t(w)
    for det in (False, True):
        uu = np.broadcast_to(linspace01_32(K), u.shape).copy() if det else u
        got = _np(eng.sample_pdf(B, W, K, det, u=None if det else _t(u)))
        _pdf_check(f"sample_pdf bins={n_bins} K={K} det={det}", got, bins, w, uu)
        if n_bins == 1:
            assert np.array_equal(got, np.broadcast_to(bins, got.shape))


@pytest.mark.parametrize("S,K", MERGE_SHAPES)
def test_sample_pdf_merge_is_the_sorted_union(S, K):
    """onerf_sample_pdf_merge on 1 and 37 rays (9 000 past the grid cap for two small shapes), injected u and det = 1:
    bit-identical to sort(z_coarse u onerf_sample_pdf(fp32 mid-points, weights[:, 1:-1], u)), ascending, finite (no
    +inf padding of the power-of-two sort buffer leaks), S + K values per ray with every coarse depth at its
    multiplicity; the stand-alone samples inside pdf_gate.  S = 2: every sample is the one mid-point."""
    eng = _engine()
    for n in (1, N_PLANT) + ((9000,) if (S, K) in MERGE_MANY_RAYS else ()):
        z, w, u = merge_inputs(n, S, K, S * 1000 + K + n)
        mid, _ = merge_reference(z, w, np.zeros((n, 0), F32))
        Z, W, MID, WP = _t(z), _t(w), _t(mid), _t(w[:, 1:-1])
        for det in (False, True):
            uu = np.broadcast_to(linspace01_32(K), u.shape).copy() if det else u
            pdf = _np(eng.sample_pdf(MID, WP, K, det, u=None if det else _t(u)))
            got = _np(eng.sample_pdf_merge(Z, W, K, det, u=None if det else _t(u)))
            _, want = merge_reference(z, w, pdf)
            assert got.shape == (n, S + K)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (n, det)
            assert np.isfinite(got).all() and (np.diff(got, axis=1) >= 0).all(), (n, det)
            for r in range(min(n, 64)):
                have = Counter(got[r].tolist())
                assert all(have[v] >= c for v, c in Counter(z[r].tolist()).items()), (n, det, r)
            if S == 2:
                assert np.array_equal(pdf, np.broadcast_to(mid, pdf.shape))
            _pdf_check(f"sample_pdf_merge S={S} K={K} n={n} det={det}", pdf, mid, w[:, 1:-1], uu)


def test_importance_draws_are_numpy_philox():
    """Without u and det = 0, both importance-sampling entry points draw U[0, 1) from Philox stream 1 at index r K + k
    (seed >= 2^32, K = 30 not a multiple of 4, 9 000 rays over the grid-stride loop): bit-identical to the same calls fed
    numpy's uniforms, and different from the draws at index r S + k."""
    eng = _engine()
    n, S, K = 9000, 33, 30
    z, w, _ = merge_inputs(n, S, K, 77)
    mid, _ = merge_reference(z, w, np.zeros((n, 0), F32))
    u = philox_uniform(SEED, 1, np.arange(n * K)).reshape(n, K)
    u_wrong = philox_uniform(SEED, 1, (np.arange(n)[:, None] * S + np.arange(K)[None, :]).reshape(-1)).reshape(n, K)
    Z, W, MID, WP = _t(z), _t(w), _t(mid), _t(w[:, 1:-1])
    merged = eng.sample_pdf_merge(Z, W, K, False, seed=SEED)
    assert torch.equal(merged, eng.sample_pdf_merge(Z, W, K, False, u=_t(u)))
    assert not torch.equal(merged, eng.sample_pdf_merge(Z, W, K, False, u=_t(u_wrong)))
    alone = eng.sample_pdf(MID, WP, K, False, seed=SEED)
    assert torch.equal(alone, eng.sample_pdf(MID, WP, K, False, u=_t(u)))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# compositing forward
# ------------------------------------------------------------------------------------------------
def _composite_check(mode, S, n, seed):
    eng = _engine()
    c = composite_inputs(n, S, seed=seed)
    kw = dict(COMPOSITE_MODES[mode])
    fi = kw.pop("forward_instance", True)
    use_ptm = kw.pop("pass_through_mask", False)
    noise = kw.get("noise_std", 0.0) > 0
    scene = _t(np.concatenate([c["rgb"], c["sigma"][..., None]], -1))
    obj = _t(np.concatenate([c["irgb"], c["isigma"][..., None]], -1)) if fi else None
    got = eng.composite(_t(c["z"]), scene, obj, noise_scene=_t(c["ns"]) if noise else None,
                        noise_obj=_t(c["no"]) if noise else None, pass_through_mask=_t(c["ptm"]) if use_ptm else None,
                        **{"is_eval": True, **kw})
    got = {k: _np(v) for k, v in got.items()}
    refs = composite_refs(c, COMPOSITE_MODES[mode], got["depth"])
    assert set(refs) == set(got)
    shares = {}
    for k, (ref, g) in refs.items():
        shares[k] = float((np.abs(got[k].astype(np.float64) - ref) / g).max())
        assert shares[k] <= 1.0, (mode, S, k, shares[k])
    _report(f"composite {mode} S={S} n={n} weights", shares["weights"])
    _report(f"composite {mode} S={S} n={n} maps", max(v for k, v in shares.items() if k != "weights"))
    return c, got


@pytest.mark.parametrize("S", COMPOSITE_S)
@pytest.mark.parametrize("mode", list(COMPOSITE_MODES))
def test_composite_forward_inside_float64_gates(mode, S):
    """onerf_composite for every flag set of the compositing backward test, 37 rays with negative sigma, sigma = -1e5,
    opaque first samples, delta = 0 and transmittance running into the subnormals planted: every weight and every map
    inside composite_gate.  `weights` holds the object branch's weights with rays_in_bbox, the scene branch's
    otherwise (compared with that branch's reference)."""
    _composite_check(mode, S, N_PLANT, seed=S + 101)


def test_composite_forward_many_rays():
    """9 000 rays at S = 33 (partial last chunk, past the 8 warps x 8 blocks x SMs grid cap) in the training flag set."""
    _composite_check("train_noise_mask", 33, 9000, seed=33 + 202)


def test_composite_seeded_noise_forward_many_rays_matches_numpy_philox():
    """noise_std = 1 without noise buffers at S = 33 on 9 000 rays: the forward draws Philox streams 2 / 3 at index
    ray S + i over the grid-stride loop, within 1e-5 of the same call fed numpy's normals."""
    from tests.test_train_stages_cpu import philox_normal
    eng = _engine()
    n, S = 9000, 33
    c = composite_inputs(n, S, seed=5)
    idx = np.arange(n * S)
    ns, no = philox_normal(SEED, 2, idx).reshape(n, S), philox_normal(SEED, 3, idx).reshape(n, S)
    scene = _t(np.concatenate([c["rgb"], c["sigma"][..., None]], -1))
    obj = _t(np.concatenate([c["irgb"], c["isigma"][..., None]], -1))
    kw = dict(noise_std=1.0, is_eval=False, frustum_bound_th=0.05)
    f_seed = eng.composite(_t(c["z"]), scene, obj, seed=SEED, **kw)
    f_buf = eng.composite(_t(c["z"]), scene, obj, noise_scene=_t(ns), noise_obj=_t(no), **kw)
    torch.cuda.synchronize()
    for k in f_seed:
        assert (f_seed[k] - f_buf[k]).abs().max().item() <= 1e-5, k


def test_occlusion_mask_edge_is_strict():
    """Occlusion mask at its edge: for a threshold th with fl(depth + th) == z_k exactly (depth from a first call), sample
    k (positive object sigma and delta) keeps a nonzero object weight and every later sample with z > z_k gets exactly
    0; the scene depth is the first call's; pass-through rays are never masked (their object weights equal the unmasked
    call's bit for bit)."""
    eng = _engine()
    n, S = N_PLANT, 64
    c = composite_inputs(n, S, seed=9)
    rows = [8, 13, 21, 30]
    c["ptm"][:] = False
    c["ptm"][1::3] = True
    c["ptm"][rows] = False
    Z = _t(c["z"])
    scene = _t(np.concatenate([c["rgb"], c["sigma"][..., None]], -1))
    depth = _np(eng.composite(Z, scene, _t(np.concatenate([c["irgb"], c["isigma"][..., None]], -1)))["depth"])
    edges = {}
    for r in rows:
        k, th = occlusion_edge(depth[r], c["z"][r])
        c["isigma"][r, k] = 3.0
        edges[r] = (k, th)
    obj = _t(np.concatenate([c["irgb"], c["isigma"][..., None]], -1))
    free = _np(eng.composite(Z, scene, obj, is_eval=True, rays_in_bbox=True)["weights"])
    for r, (k, th) in edges.items():
        out = eng.composite(Z, scene, obj, is_eval=False, rays_in_bbox=True, frustum_bound_th=float(th),
                            pass_through_mask=_t(c["ptm"]))
        w, d = _np(out["weights"]), _np(out["depth"])
        assert np.array_equal(d, depth)
        assert F32(depth[r] + th) == c["z"][r, k]
        assert w[r, k] > 0, (r, k)
        later = c["z"][r] > c["z"][r, k]
        assert later.any() and (w[r, later] == 0).all(), (r, k)
        assert np.array_equal(w[c["ptm"][:, 0]], free[c["ptm"][:, 0]])


def test_former_oracle_cases():
    """The inputs of the earlier oracle comparisons at one comfortable shape, under the checks above: 77 camera rays at
    S = 64 (coarse depths bit for bit, with and without jitter and use_disp), 50 rays of 64 + 64 merged with weights
    rand^6 and three all-zero rows, and 37 rays of 128 merged depths (two stratified sets 0.01 apart) in four flag
    sets."""
    eng = _engine()
    rays = synth.random_rays(3, 77).numpy()
    jit = synth.random_buffers(4, 77, 64, 64)["jitter"].numpy()
    for use_disp in (False, True):
        for perturb in (0.0, 1.0):
            got = _np(eng.sample_coarse(_t(rays), 64, use_disp, perturb, _t(jit)))
            assert np.array_equal(got, coarse_depth32(rays, 64, use_disp, perturb, jit)), (use_disp, perturb)
    rng = np.random.default_rng(9)
    n = 50
    z = coarse_depth32(synth.random_rays(5, n).numpy(), 64)
    w = (rng.random((n, 64)) ** 6).astype(F32)
    w[:3] = 0
    u = rng.random((n, 64)).astype(F32)
    mid, _ = merge_reference(z, w, np.zeros((n, 0), F32))
    for det in (True, False):
        uu = np.broadcast_to(linspace01_32(64), u.shape).copy() if det else u
        pdf = _np(eng.sample_pdf(_t(mid), _t(w[:, 1:-1]), 64, det, u=None if det else _t(u)))
        got = _np(eng.sample_pdf_merge(_t(z), _t(w), 64, det, u=None if det else _t(u)))
        assert np.array_equal(got, merge_reference(z, w, pdf)[1])
        _pdf_check(f"former merge case det={det}", pdf, mid, w[:, 1:-1], uu)
    rng = np.random.default_rng(31)
    n, s = 37, 128
    zc = coarse_depth32(synth.random_rays(32, n).numpy(), 64)
    f = lambda *sh: rng.standard_normal(sh).astype(F32)
    c = dict(z=np.sort(np.concatenate([zc, zc + F32(0.01)], 1), 1), sigma=f(n, s) * F32(6), isigma=f(n, s) * F32(6))
    c.update(rgb=1 / (1 + np.exp(-f(n, s, 3))), irgb=1 / (1 + np.exp(-f(n, s, 3))), ns=f(n, s), no=f(n, s),
             ptm=rng.random((n, 1)) < 0.5)
    scene = _t(np.concatenate([c["rgb"], c["sigma"][..., None]], -1))
    obj = _t(np.concatenate([c["irgb"], c["isigma"][..., None]], -1))
    for kw in (dict(), dict(white_back=True, rays_in_bbox=True), dict(zero_last_delta=True),
               dict(noise_std=1.0, is_eval=False, frustum_bound_th=0.05, pass_through_mask=True)):
        kk = {k: v for k, v in kw.items() if k != "pass_through_mask"}
        got = eng.composite(_t(c["z"]), scene, obj, noise_scene=_t(c["ns"]), noise_obj=_t(c["no"]),
                            pass_through_mask=_t(c["ptm"]) if kw.get("pass_through_mask") else None,
                            **{"is_eval": True, **kk})
        got = {k: _np(v) for k, v in got.items()}
        for k, (ref, g) in composite_refs(c, kw, got["depth"]).items():
            share = float((np.abs(got[k].astype(np.float64) - ref) / g).max())
            assert share <= 1.0, (kw, k, share)


# ------------------------------------------------------------------------------------------------
# two coarse samples with importance sampling; S + K > 2048
# ------------------------------------------------------------------------------------------------
def _close_to_oracle(got, ref, train):
    for k, v in ref.items():
        tol = 5e-4 if k.startswith("weights") else (1e-3 if (train and k == "z_vals_fine") else 2e-4)
        err = (got[k].detach().cpu() - v.detach()).abs().max().item()
        assert err <= tol, (k, err)


def test_two_coarse_samples_with_importance_match_the_oracle():
    """n_samples = 2, n_importance = 1 (weights[:, 1:-1] is empty, every importance sample is the one mid-point bin):
    the one-call forward matches the oracle's render_rays in fp32 (tolerances of the golden render test) and equals the
    staged route bit for bit; the training step's maps match the oracle too."""
    from tests.test_gpu_train_step import _batch, _fused, _kwargs
    c = dict(cases.RENDER_CASES["train_voxel"], n_rays=37, n_samples=2, n_importance=1)
    inp = cases.build_render_case(c)
    plan, _models, _emb = _plan_for_case(c, "fp32")
    fused = plan.run()
    staged = _run_render_case(c, "fp32")
    torch.cuda.synchronize()
    for k in staged:
        assert torch.equal(fused[k], staged[k]), k
    ref = O.render_rays(inp["weights"], grid_obj(inp["grid"]), inp["rays"], inp["codes"], n_samples=2, n_importance=1,
                        perturb=c["perturb"], noise_std=c["noise_std"], white_back=c["white_back"],
                        frustum_bound_th=c["frustum_bound_th"], pass_through_mask=inp["pass_through_mask"],
                        is_eval=c["is_eval"], rand=inp["rand"])
    _close_to_oracle(fused, ref, train=True)
    g = dict(cases.GRAD_CASE, n_samples=2, n_importance=1)
    ginp = cases.build_grad_case()
    ginp["rand"] = synth.random_buffers(g["seed"] + 4, g["n_rays"], 2, 1)
    rand = {k: v.to(DEV) for k, v in ginp["rand"].items()}
    kw = _kwargs(cases.GRAD_CASE, ginp, "fp32", rand, N_samples=2, N_importance=1)
    (loss, _, _, _), maps, _ = _fused(ginp, True, _batch(ginp), kw)
    assert torch.isfinite(loss).all()
    codes = ginp["code_table"][ginp["instance_ids"].view(-1)]
    gref = O.render_rays(ginp["weights"], grid_obj(ginp["grid"]), ginp["rays"], codes, n_samples=2, n_importance=1,
                         perturb=g["perturb"], noise_std=g["noise_std"], frustum_bound_th=g["frustum_bound_th"],
                         pass_through_mask=ginp["pass_through_mask"], is_eval=False, rand=ginp["rand"])
    _close_to_oracle(maps, gref, train=True)


def test_more_than_2048_samples_are_refused_before_any_launch():
    """S + K = 2049: onerf_render_rays_fwd returns ONERF_ERR_UNSUPPORTED and launches nothing (before, the coarse pass ran
    first); the training step refuses the shape with the same status."""
    from object_nerf_b200 import _lib, training
    from tests.test_gpu_train_step import _batch, _kwargs, _setup
    c = dict(cases.RENDER_CASES["eval_voxel"], n_rays=4, n_samples=1025, n_importance=1024)
    plan, _models, _emb = _plan_for_case(c, "fp32")
    dev = torch.device(DEV)
    before = _lib.launch_count(dev)
    assert _lib.load().onerf_render_rays_fwd(_lib.ctx(dev), C.byref(plan.args), _lib.stream()) == -2
    assert b"2048" in _lib.load().onerf_last_error()
    assert _lib.launch_count(dev) == before
    ginp = cases.build_grad_case(n_rays=4)
    ginp["rand"] = synth.random_buffers(0, 4, 1025, 1024)
    rand = {k: v.to(DEV) for k, v in ginp["rand"].items()}
    models, embeddings, lib = _setup(ginp, True)
    kw = _kwargs(cases.GRAD_CASE, ginp, "fp32", rand, N_samples=1025, N_importance=1024)
    with pytest.raises(RuntimeError, match="error -2"):
        training.train_step(models, embeddings, lib, _batch(ginp), cases.LOSS_CONF, **kw)
