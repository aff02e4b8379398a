"""CPU-side checks of the training-step entry points (include/onerf_ext.h: onerf_train_step,
onerf_train_step_workspace_bytes): exported, declared with the arguments the ctypes binding passes, sized as the
training workspace plus the coarse pass's field gradients and the loss accumulators, and argument validation that fails
loudly before any CUDA call."""
import ctypes
import os
import re

import pytest

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


def test_step_entry_points_are_exported_and_declared(lib):
    from object_nerf_b200 import _lib
    decl = _ext_declarations()
    for name in ("onerf_train_step", "onerf_train_step_workspace_bytes"):
        assert name in _lib.EXPORTS_EXT and name in decl and hasattr(lib, name), name
        assert len(getattr(lib, name).argtypes) == len(decl[name]), name
    assert decl["onerf_train_step"][1:4] == ["const onerf_render_args* fwd", "const onerf_loss_args* loss",
                                             "const onerf_render_bwd_args* bwd"]
    assert sorted(set(_lib.EXPORTS_EXT)) == sorted(decl)


def test_step_workspace_bytes(lib):
    from object_nerf_b200 import _lib
    f = lib.onerf_train_step_workspace_bytes
    a1k = lambda x: (x + 1023) // 1024 * 1024
    for prec in (_lib.PREC_FP32, _lib.PREC_BF16):
        assert f(prec, 1, -1, 64, 64) == 0 and f(prec, 1, 4, 0, 64) == 0 and f(prec, 0, 4, 64, -1) == 0
        for uv in (0, 1):
            for n, s, si in ((1, 2, 0), (41, 64, 32), (2048, 64, 64)):
                base = lib.onerf_train_workspace_bytes_prec(prec, uv, n, s, si)
                assert f(prec, uv, n, s, si) == base + 2 * a1k(n * s * 16) + 1024, (prec, uv, n, s, si)
    assert f(2, 1, 4, 64, 64) == 0


def test_step_rejects_bad_arguments_with_a_message(lib):
    from object_nerf_b200 import _lib
    z = ctypes.c_void_p(0)
    assert lib.onerf_train_step(None, None, None, None, z, z) < 0
    assert b"null" in lib.onerf_last_error()
    a, la, b = _lib.RenderArgs(), _lib.LossArgs(), _lib.RenderBwdArgs()
    dummy = ctypes.c_float()
    # no training workspace
    assert lib.onerf_train_step(ctypes.c_void_p(1), ctypes.byref(a), ctypes.byref(la), ctypes.byref(b),
                                ctypes.addressof(dummy), z) == -1
    assert b"training workspace" in lib.onerf_last_error()


def test_train_step_needs_the_object_branch():
    """TotalLoss reads the object branch's maps: forward_instance=False is refused before anything runs."""
    from object_nerf_b200 import training
    with pytest.raises(NotImplementedError):
        training.train_step({}, {}, None, {}, {}, forward_instance=False)


class _FakeLib:
    """Stands in for libonerf_sm90.so on the CPU: records what train_step passes and writes known values through the
    pointers it is given (all buffers are CPU tensors here, so the pointers are host addresses)."""

    def __init__(self):
        self.calls = []

    @staticmethod
    def view(ptr, n, ctype=ctypes.c_float):
        import numpy as np
        return np.ctypeslib.as_array((ctype * n).from_address(ptr))

    def onerf_packed_weights_bytes(self, use_voxel):
        return 4096

    def onerf_train_step_workspace_bytes(self, prec, use_voxel, n, s, k):
        return 8192

    def onerf_pack_weights(self, ctx, use_voxel, W, B, packed, nbytes, stream):
        self.calls.append(("pack", [W[i] for i in range(20)], [B[i] for i in range(20)], packed))
        return 0

    def onerf_code_gather(self, ctx, table, ids, n, n_codes, out, stream):
        t, i = self.view(table, n_codes * 64).reshape(n_codes, 64), self.view(ids, n, ctypes.c_int64)
        self.view(out, n * 64).reshape(n, 64)[:] = t[i]
        return 0

    def onerf_train_step(self, ctx, a, la, b, psnr, stream):
        import numpy as np
        a, la, b = a._obj, la._obj, b._obj
        n = la.n_rays
        rec = dict(n_rays=a.n_rays, grid=bool(a.grid), seed=a.seed, has_fine=la.has_fine,
                   weights=(la.color_weight, la.depth_weight, la.opacity_weight, la.instance_color_weight,
                            la.instance_depth_weight),
                   rgbs=self.view(la.rgbs, n * 3).copy(), valid=self.view(la.valid_mask, n, ctypes.c_uint8).copy(),
                   d_codes_before=self.view(b.d_codes, n * 64).copy())
        self.calls.append(("step", rec, b))
        # every dW / db tensor of layer i gets i + 1 added; d_codes = ray index; loss outputs 1..6, psnr 7
        for typ in ("coarse", "fine") if la.has_fine else ("coarse",):
            for i in range(20):
                for arr in (getattr(b, "dW_" + typ), getattr(b, "db_" + typ)):
                    self.view(arr[i], 1)[0] += i + 1      # first element only
        self.view(b.d_codes, n * 64).reshape(n, 64)[:] = np.arange(n, dtype=np.float32)[:, None]
        self.view(la.loss_sum_out, 6)[:] = [1, 2, 3, 4, 5, 6]
        self.view(la.present_out, 5, ctypes.c_int32)[:] = [1, 1, 0, 1, 0]
        self.view(psnr, 1)[0] = 7.0
        return 0

    def onerf_code_scatter_add(self, ctx, d_codes, ids, n, n_codes, table_grad, stream):
        import numpy as np
        g = self.view(table_grad, n_codes * 64).reshape(n_codes, 64)
        np.add.at(g, self.view(ids, n, ctypes.c_int64), self.view(d_codes, n * 64).reshape(n, 64))
        return 0


class _FakeRenderPlan:
    """engine.RenderPlan's argument block without the device workspace it allocates."""

    def __init__(self, rays, packed_coarse, packed_fine, grid, codes=None, **kw):
        from object_nerf_b200 import _lib
        self.args, self.kw = _lib.RenderArgs(), dict(kw, rays=rays, codes=codes, packed=(packed_coarse, packed_fine))
        self.args.n_rays = rays.shape[0]
        self.maps = {}


def test_train_step_plumbing_with_the_library_stubbed(monkeypatch):
    """train_step's Python side on CPU tensors against a stand-in library: the batch lands in the plan's buffers, the loss
    weights go in TERMS order, W / dW / db pointers are the parameters and their .grad (accumulated, created when
    missing), d_codes is zeroed before the step and scattered into the code table's .grad by instance id, the grid and
    the seed are set per call, and a second call reuses the plan."""
    import contextlib

    import torch

    from object_nerf_b200 import _lib, engine, training
    from object_nerf_b200 import synthetic as S
    from tests import cases, helpers

    fake = _FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: fake)
    monkeypatch.setattr(_lib, "ctx", lambda dev: None)
    monkeypatch.setattr(_lib, "stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(engine, "RenderPlan", _FakeRenderPlan)
    inp = cases.build_grad_case()
    n = inp["rays"].shape[0]
    models = {k: S.make_model(w, True, "cpu") for k, w in inp["weights"].items()}
    emb = S.GridModule(inp["grid"])
    lib = helpers.CodeLib(inp["code_table"])
    batch = {k: v.clone() for k, v in inp["batch"].items()}
    batch["rays"], batch["instance_ids"] = inp["rays"], inp["instance_ids"]
    lin = {typ: engine.model_linears(models[typ]) for typ in models}
    lin["coarse"][3][0].grad = torch.ones_like(lin["coarse"][3][0])        # accumulated into, not replaced
    kw = dict(N_samples=64, N_importance=64, perturb=1.0, noise_std=1.0, pass_through_mask=inp["pass_through_mask"],
              frustum_bound_th=0.025, precision="bf16")
    out = training.train_step(models, {"xyz": emb, "dir": None}, lib, batch, cases.LOSS_CONF, **kw)
    (plan,) = training._plans[models["coarse"]].values()
    step = [c for c in fake.calls if c[0] == "step"]
    assert len(step) == 1
    rec, b = step[0][1], step[0][2]
    f32 = lambda x: ctypes.c_float(x).value
    assert rec["weights"] == tuple(f32(cases.LOSS_CONF[f"{t}_weight"]) for t in training.TERMS)
    assert rec["has_fine"] == 1 and rec["n_rays"] == n and rec["grid"] and rec["seed"] != 0
    assert (rec["rgbs"] == batch["rgbs"].numpy().reshape(-1)).all()
    assert (rec["valid"] == batch["valid_mask"].numpy().astype("uint8")).all()
    assert (rec["d_codes_before"] == 0).all()
    assert torch.equal(plan.ids, batch["instance_ids"].reshape(-1))
    assert torch.equal(plan.codes, lib.embedding_instance.weight.detach()[batch["instance_ids"].reshape(-1)])
    assert plan.render.kw["pass_through_mask"] is plan.ptm
    assert torch.equal(plan.ptm, inp["pass_through_mask"].reshape(-1).to(torch.uint8))
    for typ in ("coarse", "fine"):
        for i, (w, bb) in enumerate(lin[typ]):
            assert getattr(b, "W_" + typ)[i] == w.data_ptr() and getattr(b, "dW_" + typ)[i] == w.grad.data_ptr()
            assert getattr(b, "db_" + typ)[i] == bb.grad.data_ptr()
            base = 1.0 if (typ, i) == ("coarse", 3) else 0.0
            assert w.grad.reshape(-1)[0].item() == base + i + 1 and bb.grad.reshape(-1)[0].item() == i + 1
            assert w.grad.reshape(-1)[1:].eq(base).all()
    assert b.table_grad == emb.embedding_space_ftr.weight.grad.data_ptr()
    want = torch.zeros_like(lib.embedding_instance.weight)
    want.index_add_(0, batch["instance_ids"].reshape(-1), torch.arange(n, dtype=torch.float32)[:, None].expand(n, 64))
    assert torch.equal(lib.embedding_instance.weight.grad, want)
    loss_sum, terms, present, psnr = out
    assert loss_sum.item() == 1 and terms.tolist() == [2, 3, 4, 5, 6] and present.tolist() == [1, 1, 0, 1, 0]
    assert psnr.item() == 7
    training.train_step(models, {"xyz": emb, "dir": None}, lib, batch, cases.LOSS_CONF, **kw)
    assert list(training._plans[models["coarse"]].values()) == [plan]
    assert not [c for c in fake.calls if c[0] == "step"][1][1]["d_codes_before"].any()


def test_a_library_without_the_step_entry_points_is_refused_by_name(monkeypatch, lib):
    """ABI version 2 grows by additions: a library built before them has the right version number, so load() names the
    missing entry points instead of failing later on an attribute."""
    from object_nerf_b200 import _lib

    class Stale:
        def __init__(self, path):
            self._real = lib

        def __getattr__(self, name):
            if name == "onerf_train_step":
                raise AttributeError(name)
            return getattr(self._real, name)

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib.C, "CDLL", Stale)
    with pytest.raises(RuntimeError, match="onerf_train_step"):
        _lib.load()
