"""CPU-side checks of the device-seed entry points (include/onerf_ext.h: onerf_render_rays_fwd_dseed,
onerf_train_step_dseed): exported, declared with the arguments the ctypes binding passes, argument validation before any
CUDA call, and train_step's choice between the host-seed and the device-seed entry with the library stubbed."""
import ctypes
import os
import re

import pytest

from tests.test_train_step_cpu import _FakeLib, _FakeRenderPlan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def _ext_declarations():
    src = open(os.path.join(ROOT, "include", "onerf_ext.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return {m.group(1): [p.strip() for p in m.group(2).split(",")]
            for m in re.finditer(r"\b(onerf_[a-z0-9_]+)\s*\(([^)]*)\)", src)}


def test_device_seed_entry_points_are_exported_and_declared(lib):
    from object_nerf_b200 import _lib
    decl = _ext_declarations()
    assert decl["onerf_render_rays_fwd_dseed"] == ["onerf_ctx* ctx", "const onerf_render_args* args",
                                                   "uint64_t* seed_dev", "void* stream"]
    assert decl["onerf_train_step_dseed"] == decl["onerf_train_step"][:5] + ["uint64_t* seed_dev", "void* stream"]
    for name in ("onerf_render_rays_fwd_dseed", "onerf_train_step_dseed"):
        assert name in _lib.EXPORTS_EXT and hasattr(lib, name), name
        assert len(getattr(lib, name).argtypes) == len(decl[name]), name
    assert lib.onerf_train_step_dseed.argtypes[:5] == lib.onerf_train_step.argtypes[:5]
    assert lib.onerf_render_rays_fwd_dseed.argtypes[:2] == lib.onerf_render_rays_fwd.argtypes[:2]


def test_device_seed_entries_validate_before_any_cuda_call(lib):
    """A null or misaligned seed_dev, and a training workspace on the forward-only entry, are ONERF_ERR_BAD_ARG with a
    message.  The context and the seed pointer are never dereferenced on these paths."""
    from object_nerf_b200 import _lib
    ctx = ctypes.c_void_p(1)
    a, la, b = _lib.RenderArgs(), _lib.LossArgs(), _lib.RenderBwdArgs()
    psnr = ctypes.c_float()
    assert lib.onerf_render_rays_fwd_dseed(ctx, ctypes.byref(a), None, None) == -1
    assert b"null" in lib.onerf_last_error()
    assert lib.onerf_render_rays_fwd_dseed(ctx, ctypes.byref(a), 0x1004, None) == -1
    assert b"8-byte aligned" in lib.onerf_last_error()
    a.train_ws = 0x10000
    assert lib.onerf_render_rays_fwd_dseed(ctx, ctypes.byref(a), 0x1000, None) == -1
    assert b"train_ws" in lib.onerf_last_error()
    for seed_dev, msg in ((None, b"null seed_dev"), (0x1004, b"8-byte aligned")):
        assert lib.onerf_train_step_dseed(ctx, ctypes.byref(a), ctypes.byref(la), ctypes.byref(b),
                                          ctypes.addressof(psnr), seed_dev, None) == -1
        assert msg in lib.onerf_last_error()
    # the host-seed checks still run on the device-seed entry
    a.train_ws = None
    assert lib.onerf_train_step_dseed(ctx, ctypes.byref(a), ctypes.byref(la), ctypes.byref(b), ctypes.addressof(psnr),
                                      0x1000, None) == -1
    assert b"training workspace" in lib.onerf_last_error()


class _FakeSeedLib(_FakeLib):
    def onerf_train_step_dseed(self, ctx, a, la, b, psnr, seed_dev, stream):
        self.calls.append(("dseed", seed_dev))
        return self.onerf_train_step(ctx, a, la, b, psnr, stream)


def _stubbed(monkeypatch):
    import contextlib

    import torch

    from object_nerf_b200 import _lib, engine
    fake = _FakeSeedLib()
    monkeypatch.setattr(_lib, "load", lambda: fake)
    monkeypatch.setattr(_lib, "ctx", lambda dev: None)
    monkeypatch.setattr(_lib, "stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(engine, "RenderPlan", _FakeRenderPlan)
    return fake


def _problem():
    from object_nerf_b200 import synthetic as S
    from tests import cases, helpers
    inp = cases.build_grad_case()
    models = {k: S.make_model(w, True, "cpu") for k, w in inp["weights"].items()}
    embeddings = {"xyz": S.GridModule(inp["grid"]), "dir": None}
    batch = {k: v.clone() for k, v in inp["batch"].items()}
    batch["rays"], batch["instance_ids"] = inp["rays"], inp["instance_ids"]
    kw = dict(N_samples=64, N_importance=64, perturb=1.0, noise_std=1.0, pass_through_mask=inp["pass_through_mask"],
              frustum_bound_th=0.025, precision="bf16")
    return models, embeddings, helpers.CodeLib(inp["code_table"]), batch, kw


def test_train_step_picks_the_entry_by_capture_state(monkeypatch):
    """Eager: onerf_train_step with a fresh host seed, and the plan's counter starts at that seed + 4.  Capturing:
    onerf_train_step_dseed with the plan's counter and no host draw.  step_seed returns a copy of the counter."""
    from object_nerf_b200 import engine, training
    from tests import cases
    fake = _stubbed(monkeypatch)
    models, embeddings, lib, batch, kw = _problem()
    monkeypatch.setattr(engine, "new_seed", lambda: 1000)
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    (plan,) = training._plans[models["coarse"]].values()
    assert [c[0] for c in fake.calls if c[0] in ("step", "dseed")] == ["step"]
    assert fake.calls[-1][1]["seed"] == 1000
    assert plan.seed_dev.tolist() == [1004]
    seed = training.step_seed(models)
    assert seed.tolist() == [1004] and seed.data_ptr() != plan.seed_dev.data_ptr()

    monkeypatch.setattr(training, "_capturing", lambda dev: True)
    monkeypatch.setattr(engine, "new_seed", lambda: pytest.fail("a captured step drew a host seed"))
    training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    assert [c[0] for c in fake.calls if c[0] in ("step", "dseed")] == ["step", "dseed", "step"]
    dseed = [c for c in fake.calls if c[0] == "dseed"][0]
    assert dseed[1] == plan.seed_dev.data_ptr()
    assert list(training._plans[models["coarse"]].values()) == [plan]


def test_first_train_step_while_capturing_is_refused(monkeypatch):
    from object_nerf_b200 import training
    from tests import cases
    fake = _stubbed(monkeypatch)
    models, embeddings, lib, batch, kw = _problem()
    monkeypatch.setattr(training, "_capturing", lambda dev: True)
    with pytest.raises(RuntimeError, match="warm up"):
        training.train_step(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    assert not [c for c in fake.calls if c[0] in ("step", "dseed")]
    assert not training._plans.get(models["coarse"])
    with pytest.raises(ValueError):
        training.step_seed(models)


def test_capture_state_is_not_queried_for_cpu_tensors():
    """torch.cuda.is_current_stream_capturing needs a CUDA device; train_step's CPU plumbing (tests above) never asks."""
    import torch

    from object_nerf_b200 import training
    assert training._capturing(torch.device("cpu")) is False
