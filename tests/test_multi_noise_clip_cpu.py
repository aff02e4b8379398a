"""render_rays_multi with sigma noise, perturbed importance sampling and 10-column ray sets: the CPU oracle against the
reference's own outputs (tests/golden/multi_<case>.npz from tools/make_golden.py, draws injected), and what each case
is there to cover.  The port is tests/multi_noise_oracle.py; without noise, perturb and clip it is
onerf_oracle.render_rays_multi bit for bit."""
import ctypes
import os

import pytest
import torch

from oracle import onerf_oracle as O
from tests import cases
from tests import multi_noise_oracle as M
from tests.multi_noise_cases import NOISE_CLIP_CASES, build_noise_clip_case


def grid_obj(g):
    return O.VoxelGrid(g["offset"], g["voxel_size"], g["shape"].tolist(), g["idx_map"], g["table"])


def run_oracle(c, inp, **over):
    kw = dict(n_samples=c["n_samples"], n_importance=c["n_importance"], white_back=c["white_back"],
              skip_boxes=[cases.box_affine(b) for b in inp["boxes"]], perturb=c["perturb"], noise_std=c["noise_std"],
              rand=inp["rand"])
    kw.update(over)
    rays_list = kw.pop("rays_list", inp["rays_list"])
    return M.render_rays_multi(inp["weights"], grid_obj(inp["grid"]), inp["code_table"], rays_list, c["obj_ids"], **kw)


@pytest.mark.parametrize("name", list(NOISE_CLIP_CASES))
def test_oracle_equals_reference_fixture(golden, name):
    c = NOISE_CLIP_CASES[name]
    g = golden("multi_" + name)
    out = run_oracle(c, build_noise_clip_case(c))
    assert set(out) == set(g), (sorted(out), sorted(g))
    for k in g:
        assert out[k].shape == g[k].shape, k
        assert torch.equal(out[k], g[k]), (k, (out[k] - g[k]).abs().max().item())


@pytest.mark.parametrize("name", ["edit_dup", "edit_scene_only", "edit_two_objs"])
def test_port_without_extensions_is_the_oracle(name):
    c = cases.MULTI_CASES[name]
    inp = cases.build_multi_case(c)
    kw = dict(n_samples=c["n_samples"], n_importance=c["n_importance"], white_back=c["white_back"],
              skip_boxes=[cases.box_affine(b) for b in inp["boxes"]])
    args = (inp["weights"], grid_obj(inp["grid"]), inp["code_table"], inp["rays_list"], c["obj_ids"])
    want, got = O.render_rays_multi(*args, **kw), M.render_rays_multi(*args, **kw)
    assert set(want) == set(got)
    for k in want:
        assert torch.equal(want[k], got[k]), k


def _differs(a, b, keys=("rgb_coarse", "rgb_fine", "z_vals_fine")):
    return {k: not torch.equal(a[k], b[k]) for k in keys}


def test_noise_changes_both_passes_and_the_fine_depths():
    c = NOISE_CLIP_CASES["noise_both"]
    inp = build_noise_clip_case(c)
    assert all(_differs(run_oracle(c, inp), run_oracle(c, inp, noise_std=0.0)).values())


def test_injected_u_changes_the_fine_depths():
    c = NOISE_CLIP_CASES["perturb_u"]
    inp = build_noise_clip_case(c)
    d = _differs(run_oracle(c, inp), run_oracle(c, inp, perturb=0.0))
    assert d["z_vals_fine"] and d["rgb_fine"] and not d["rgb_coarse"]


def test_mixed_sets_clip_only_the_ten_column_set_and_only_the_fine_pass():
    c = NOISE_CLIP_CASES["mixed_clip"]
    inp = build_noise_clip_case(c)
    assert [r.shape[1] for r in inp["rays_list"]] == [8, 10, 8]
    unclipped = run_oracle(c, inp, rays_list=[r[:, :8] for r in inp["rays_list"]])
    out = run_oracle(c, inp)
    for k in ("z_vals_coarse", "weights_coarse", "rgb_coarse", "obj_ids_coarse"):
        assert torch.equal(out[k], unclipped[k]), k
    assert not torch.equal(out["z_vals_fine"], unclipped["z_vals_fine"])


def _ties_at(z, far_box):
    return (z == far_box[:, None]).sum(1)


def test_swallowing_interval_sends_every_fine_sample_of_the_set_to_far_box(golden):
    c = NOISE_CLIP_CASES["clip_swallow"]
    inp = build_noise_clip_case(c)
    fb = inp["rays_list"][1][:, 9]
    sf = c["n_samples"] + c["n_importance"]
    assert (_ties_at(golden("multi_clip_swallow")["z_vals_fine"], fb) >= sf).all()
    # a missed ray (near = far = 0) is clipped to far + 0.1 too, so the fine pass no longer mutes it
    assert (inp["rays_list"][1][:, 7] == 0).any()


def test_empty_interval_clips_nothing():
    c = NOISE_CLIP_CASES["clip_empty"]
    inp = build_noise_clip_case(c)
    r1 = inp["rays_list"][1]
    assert (r1[:, 8] >= r1[:, 9]).all() and (r1[:, 8] == r1[:, 9]).any() and (r1[:, 8] > r1[:, 9]).any()
    trimmed = [r[:, :8] if i == 1 else r for i, r in enumerate(inp["rays_list"])]
    out, ref = run_oracle(c, inp), run_oracle(c, inp, rays_list=trimmed)
    for k in out:
        assert torch.equal(out[k], ref[k]), k


def test_far_box_zero_mutes_rays_whose_depths_clip_to_zero(golden):
    c = NOISE_CLIP_CASES["clip_far_zero"]
    inp = build_noise_clip_case(c)
    r1 = inp["rays_list"][1]
    assert (r1[:, 9] == 0).all()
    neg = r1[:, 7] < 0
    assert neg.any() and (~neg).any()
    sf = c["n_samples"] + c["n_importance"]
    g = golden("multi_clip_far_zero")
    fully = neg & (r1[:, 8] <= r1[:, 6])   # near_box <= near: every fine depth of the set is clipped to 0
    assert fully.any()
    # the set's fine depths are the row's first sf entries (the scene set's are positive); the last of them is 0, so the
    # fine pass mutes the set on those rays: none of its samples gets a weight, the one before the scene's first included
    assert (g["z_vals_fine"][fully, :sf] == 0).all() and (g["z_vals_fine"][fully, sf:] > 0).all()
    assert (g["weights_fine"][fully, :sf] == 0).all()
    # the coarse pass is not clipped: the same rays keep their negative depths there and are not muted
    assert (g["z_vals_coarse"][fully] < 0).any(1).all()


def test_duplicated_sets_tie_at_far_box_across_the_sets(golden):
    c = NOISE_CLIP_CASES["dup_tied"]
    inp = build_noise_clip_case(c)
    r1, r2 = inp["rays_list"][1], inp["rays_list"][2]
    assert torch.equal(r1[:, :6], r2[:, :6]) and torch.equal(r1[:, 8:], r2[:, 8:])
    assert c["obj_ids"][1] == c["obj_ids"][2]
    ties = _ties_at(golden("multi_dup_tied")["z_vals_fine"], r1[:, 9])
    both = (r1[:, 7] > 0) & (r2[:, 7] > 0)
    assert (ties[both] > 1).all()


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def test_stage_entries_refuse_bad_noise_and_clip_before_touching_the_device(lib):
    z = ctypes.c_void_p(0)
    odd = ctypes.c_void_p(0x1001)
    for name in ("onerf_composite_multi_noise_ws", "onerf_composite_multi_noise_merge"):
        f = getattr(lib, name)
        tail = (z, z, z, z, z, z, z, z, 0, z)
        cases_ = [((1.0, odd, 1, 0), b"4-byte aligned"), ((0.0, ctypes.c_void_p(0x1000), 1, 0), b"noise_std = 0"),
                  ((-1.0, z, 1, 0), b"finite and >= 0"), ((float("inf"), z, 1, 0), b"finite and >= 0"),
                  ((1.0, z, 1, 2), b"pass must be"), ((1.0, z, 1, 0), b"null")]
        for noise_args, msg in cases_:
            assert f(None, z, z, 4, 2, 8, 0, *noise_args, *tail) == -1, (name, noise_args)
            assert msg in lib.onerf_last_error(), (name, msg, lib.onerf_last_error())
    clip = lib.onerf_sample_pdf_merge_clip
    assert clip(None, z, z, 4, 8, 8, 1, z, 0, ctypes.c_void_p(0x1004), z, z) == -1
    assert b"aligned" in lib.onerf_last_error()
    assert clip(None, z, z, 4, 8, 8, 1, z, 0, ctypes.c_void_p(0x1008), z, z) == -1
    assert b"null" in lib.onerf_last_error()
    x = ctypes.c_void_p(0)
    assert lib.onerf_render_multi_fwd_ext(None, None, None, x) == -1
    assert b"null" in lib.onerf_last_error()
