"""render_rays_multi with sigma noise, perturbed importance sampling and 10-column ray sets on the device (pytest -m gpu):
the reference's fixtures, the in-kernel Philox draws against numpy's, the staged route against the one call, the ext
entry against onerf_render_multi_fwd, and the refusals of the ext entry."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import helpers
from tests.multi_noise_cases import NOISE_CLIP_CASES, build_noise_clip_case
from tests.test_train_stages_cpu import philox_normal, philox_uniform

pytestmark = pytest.mark.gpu
DEV = "cuda"
PRECISIONS = ["fp32", "bf16"]


class _Box:   # the attributes of BBoxRayHelper that the removed-object mask reads
    pass


def _boxes(inp):
    if not inp["boxes"]:
        return None
    out = {}
    for k, b in enumerate(inp["boxes"]):
        h = _Box()
        h.scale_factor, h.pose_avg, h.axis_align_mat, h.bbox_bounds = (b["scale_factor"], b["pose_avg"], b["axis_align_mat"],
                                                                       b["bbox_bounds"])
        out[k] = h
    return out


_SETUPS = {}


def _setup(name, inp):
    from object_nerf_b200 import Embedding
    if name not in _SETUPS:
        models = {"coarse": helpers.make_model(inp["weights"]["coarse"], True, DEV),
                  "fine": helpers.make_model(inp["weights"]["fine"], True, DEV)}
        emb = {"xyz": helpers.GridModule(inp["grid"]).to(DEV), "dir": Embedding(3, 4)}
        _SETUPS[name] = (models, emb, helpers.CodeLib(inp["code_table"]).to(DEV))
    return _SETUPS[name]


def _render(name, precision="fp32", staged=False, rand="case", inp=None, **over):
    """rand: "case" injects the case's draws, None lets the kernels draw, a dict is injected as given."""
    from object_nerf_b200.multi_rendering import render_rays_multi
    c = dict(NOISE_CLIP_CASES[name], **over)
    inp = inp or build_noise_clip_case(NOISE_CLIP_CASES[name])
    models, emb, lib = _setup(name, inp)
    r = inp["rand"] if rand == "case" else rand
    if r is not None:
        r = {"u": [u.to(DEV) for u in r["u"]], "noise_coarse": r["noise_coarse"].to(DEV), "noise_fine": r["noise_fine"].to(DEV)}
    with torch.no_grad():
        return render_rays_multi(models, emb, lib, [x.to(DEV) for x in inp["rays_list"]], c["obj_ids"],
                                 N_samples=c["n_samples"], N_importance=c["n_importance"], perturb=c["perturb"],
                                 noise_std=c["noise_std"], white_back=c["white_back"], background_skip_bbox=_boxes(inp),
                                 precision=precision, _staged=staged, _rand=r)


def _equal(a, b):
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def _close(a, b, tol, name):
    err = (a.detach().cpu() - b).abs().max().item() if b.numel() else 0.0
    assert err <= tol, f"{name}: max abs err {err:.3e} > {tol:.1e}"


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(NOISE_CLIP_CASES))
def test_matches_reference_fixture(golden, name, precision):
    gold = golden("multi_" + name)
    out = _render(name, precision)
    assert set(out) == set(gold), (sorted(out), sorted(gold))
    _close(out["z_vals_coarse"], gold["z_vals_coarse"], 1e-6, "z_vals_coarse")
    # object tags only where the depth is untied (torch's CPU sort is not stable; tied samples carry equal fields)
    gz = gold["z_vals_coarse"]
    untied = torch.ones_like(gz, dtype=torch.bool)
    untied[:, 1:] &= gz[:, 1:] != gz[:, :-1]
    untied[:, :-1] &= gz[:, :-1] != gz[:, 1:]
    assert torch.equal(out["obj_ids_coarse"].cpu()[untied], gold["obj_ids_coarse"][untied])
    c = NOISE_CLIP_CASES[name]
    # fp32: as for render_rays' fixtures, the inverse CDF divides by pdf mass as small as 1e-5, which turns the ulps of
    # noised coarse weights into up to ~1e-3 of z_vals_fine (tests/test_gpu_parity.py)
    z_fine_tol = 1e-3 if (c["noise_std"] != 0 or c["perturb"] != 0) else 1e-4
    bad = []
    for k in gold:
        if k.startswith("weights"):
            tol = 5e-4 if precision == "fp32" else 3e-2
        elif k.startswith(("rgb", "opacity")):
            tol = 2e-4 if precision == "fp32" else 3e-2
            if precision == "bf16" and helpers.psnr(out[k].cpu(), gold[k]) < 45.0:
                bad.append(f"{k}: PSNR {helpers.psnr(out[k].cpu(), gold[k]):.1f} dB < 45")
        elif k.startswith("depth"):
            tol = 2e-4 if precision == "fp32" else 5e-2
        elif k.startswith("z_vals"):
            tol = (z_fine_tol if k == "z_vals_fine" else 1e-6) if precision == "fp32" else 5e-2
        else:
            continue
        err = (out[k].cpu() - gold[k]).abs().max().item()
        if err > tol:
            bad.append(f"{k}: max abs err {err:.3e} > {tol:.1e}")
    assert not bad, bad


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", ["mixed_clip", "dup_tied", "clip_far_zero"])
def test_staged_route_equals_the_one_call(name, precision):
    _equal(_render(name, precision), _render(name, precision, staged=True))
    # and with every draw made in the kernels, from one seed of the same torch generator state
    torch.manual_seed(11)
    one = _render(name, precision, rand=None)
    torch.manual_seed(11)
    _equal(one, _render(name, precision, staged=True, rand=None))


def test_same_seed_same_output_and_a_new_seed_differs():
    torch.manual_seed(5)
    a = _render("mixed_clip", rand=None)
    torch.manual_seed(5)
    b = _render("mixed_clip", rand=None)
    c = _render("mixed_clip", rand=None)
    _equal(a, b)
    assert not torch.equal(a["rgb_fine"], c["rgb_fine"]) and not torch.equal(a["rgb_coarse"], c["rgb_coarse"])


def _numpy_draws(seed, c):
    """What the kernels draw with `seed`: u of set i = Philox stream 1 keyed by seed + i at element r K + k; the noise of
    the coarse / fine pass = streams 7 / 8 at element r T + p."""
    n, s, k, no = c["n_rays"], c["n_samples"], c["n_importance"], len(c["obj_ids"])
    t = lambda a, *shape: torch.from_numpy(a).view(*shape)
    return {"u": [t(philox_uniform(seed + i, 1, np.arange(n * k)), n, k) for i in range(no)],
            "noise_coarse": t(philox_normal(seed, 7, np.arange(n * no * s)), n, no * s),
            "noise_fine": t(philox_normal(seed, 8, np.arange(n * no * (s + k))), n, no * (s + k))}


def test_one_call_draws_are_numpys_philox_draws():
    from object_nerf_b200 import engine
    c = NOISE_CLIP_CASES["mixed_clip"]
    torch.manual_seed(21)
    seed = engine.new_seed()
    want = _numpy_draws(seed, c)
    # u: integer Philox words scaled by 2^-24, exact on both sides: bit-identical without noise
    torch.manual_seed(21)
    _equal(_render("mixed_clip", rand=None, noise_std=0.0), _render("mixed_clip", rand=want, noise_std=0.0))
    # noise: numpy's float64 Box-Muller agrees with the device's logf / cospif to an ulp or two
    torch.manual_seed(21)
    got = _render("mixed_clip", rand=None)
    fed = _render("mixed_clip", rand=want)
    for k in fed:
        _close(got[k], fed[k].cpu(), 1e-4, k)
    swapped = dict(want, noise_coarse=want["noise_coarse"].flip(1))
    assert (_render("mixed_clip", rand=swapped)["rgb_coarse"] - got["rgb_coarse"]).abs().max().item() > 1e-2


def _composite_inputs(n_obj, n, s, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.sort(torch.rand(n_obj, n, s, generator=g) * 3.0, -1)[0]
    z[1 % n_obj, ::3] = z[0, ::3]                  # ties across sets
    z[n_obj - 1, 1::5] = 0.0                       # muted-looking rays (all zeros)
    f = torch.rand(n_obj, n, s, 4, generator=g)
    f[..., 3] = torch.randn(n_obj, n, s, generator=g) * 2.0
    return z.to(DEV), f.contiguous().to(DEV)


@pytest.mark.parametrize("path", ["bitonic", "merge_forced", "merge_large"])
def test_joint_compositing_noise_is_philox_by_sorted_position(path):
    from object_nerf_b200 import engine
    n_obj, n, s = (33, 48, 128) if path == "merge_large" else (3, 40, 96)
    t = n_obj * s
    assert (t > 4096) == (path == "merge_large")
    z, f = _composite_inputs(n_obj, n, s, seed=7 + n_obj)
    seed = 0x1234_5678_9ABC
    merge = path == "merge_forced"
    for fine, stream in ((False, 7), (True, 8)):
        nz = torch.from_numpy(philox_normal(seed, stream, np.arange(n * t))).view(n, t).to(DEV)
        kw = dict(want_ids=True, want_unsorted=True, merge=merge, noise_std=1.0, fine=fine)
        drawn = engine.composite_multi(z, f, seed=seed, **kw)
        fed = engine.composite_multi(z, f, noise=nz, **kw)
        for k in drawn:
            _close(drawn[k], fed[k].cpu(), 1e-5, f"{path} {k}")
        other = engine.composite_multi(z, f, noise=nz.flip(1), **kw)
        assert (other["weights"] - drawn["weights"]).abs().max().item() > 1e-2
        if path == "bitonic":   # the rank-merge path draws the same values for the same order: the same bits
            _equal(drawn, engine.composite_multi(z, f, seed=seed, **dict(kw, merge=True)))
            _equal(fed, engine.composite_multi(z, f, noise=nz, **dict(kw, merge=True)))


def _ext_call(monkeypatch, edit):
    """Run the one call with `edit(args, ext)` applied to its argument blocks; returns the status code."""
    from object_nerf_b200 import _lib
    lib = _lib.load()
    real = lib.onerf_render_multi_fwd_ext
    rcs = []

    def wrapped(ctx, a, x, stream):
        edit(a._obj, x._obj)
        rc = real(ctx, a, x, stream)
        rcs.append(rc)
        return 0

    monkeypatch.setattr(lib, "onerf_render_multi_fwd_ext", wrapped)
    try:
        _render("mixed_clip", rand="case")
    finally:
        monkeypatch.setattr(lib, "onerf_render_multi_fwd_ext", real)
    return rcs[0], lib.onerf_last_error()


def test_ext_entry_without_extensions_is_onerf_render_multi_fwd(monkeypatch):
    from object_nerf_b200 import _lib
    lib = _lib.load()
    inp = build_noise_clip_case(NOISE_CLIP_CASES["mixed_clip"])
    inp["rays_list"] = [r[:, :8].contiguous() for r in inp["rays_list"]]
    kw = dict(inp=inp, perturb=0.0, noise_std=0.0, rand=None)
    ext_zero = _render("mixed_clip", **kw)
    real = lib.onerf_render_multi_fwd_ext
    for call in (lambda ctx, a, x, s: lib.onerf_render_multi_fwd(ctx, a, s), lambda ctx, a, x, s: real(ctx, a, None, s)):
        monkeypatch.setattr(lib, "onerf_render_multi_fwd_ext", call)
        _equal(ext_zero, _render("mixed_clip", **kw))
    monkeypatch.setattr(lib, "onerf_render_multi_fwd_ext", real)


def _misalign(p, by):
    return C.c_void_p(p + by)


@pytest.mark.parametrize("case", ["clip_4_bytes", "noise_1_byte", "u_1_byte", "noise_with_zero_std", "negative_std",
                                  "nan_std", "noise_fine_without_fine_pass", "u_with_perturb_0"])
def test_ext_entry_refuses_bad_buffers(monkeypatch, case):
    def edit(a, x):
        if case == "clip_4_bytes":
            x.clip_list_host[1] = x.clip_list_host[1] + 4
        elif case == "noise_1_byte":
            x.noise_coarse = x.noise_coarse + 1
        elif case == "u_1_byte":
            x.u_list_host[2] = x.u_list_host[2] + 1
        elif case == "noise_with_zero_std":
            x.noise_std = 0.0
        elif case == "negative_std":
            x.noise_std = -1.0
        elif case == "nan_std":
            x.noise_std = float("nan")
        elif case == "noise_fine_without_fine_pass":
            a.n_importance = 0
            x.u_list_host = None
        elif case == "u_with_perturb_0":
            a.perturb = 0.0
    rc, err = _ext_call(monkeypatch, edit)
    assert rc == -1, (case, err)
    assert err.startswith(b"onerf_render_multi_fwd_ext: "), err


def test_python_refuses_bad_ray_sets_and_draws():
    inp = build_noise_clip_case(NOISE_CLIP_CASES["mixed_clip"])
    bad = dict(inp, rays_list=[inp["rays_list"][0], inp["rays_list"][1][:, :9].contiguous(), inp["rays_list"][2]])
    with pytest.raises(ValueError):
        _render("mixed_clip", inp=bad)
    with pytest.raises(ValueError):
        _render("mixed_clip", noise_std=-0.5)
    r = dict(inp["rand"], noise_fine=inp["rand"]["noise_fine"][:, :-1])
    with pytest.raises(ValueError):
        _render("mixed_clip", rand=r)
