"""CPU checks of the validation frame (include/onerf_ext.h: onerf_validate_frame, onerf_validate_finalize;
training.validate_frame): the entry points are exported as declared and validate before any CUDA call, the record
arithmetic "accumulate per tile, sum the records, finalise" restated in float64 equals the oracle's TotalLoss and the
reference PSNR on whole images, validate_frame's host logic with the library stubbed, and a two-process gloo reduction
of the record."""
import ctypes
import math
import os
import socket

import numpy as np
import pytest
import torch

from tests import cases
from tests.test_graph_rng_cpu import _ext_declarations
from tests.test_train_step_cpu import _FakeLib

TERMS = ("color_loss", "depth_loss", "opacity_loss", "instance_color_loss", "instance_depth_loss")


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def test_entry_points_are_exported_and_declared(lib):
    from object_nerf_b200 import _lib
    decl = _ext_declarations()
    assert decl["onerf_validate_workspace_bytes"] == ["int chunk_rays", "int n_samples", "int n_importance"]
    assert decl["onerf_validate_frame"] == ["onerf_ctx* ctx", "const onerf_validate_args* args", "void* stream"]
    assert decl["onerf_validate_finalize"] == [
        "onerf_ctx* ctx", "const double* record", "const float weights[5]", "int has_fine", "float* loss_sum_out",
        "float* terms_out", "int* present_out", "float* psnr_out", "void* stream"]
    for name in decl:
        if name.startswith("onerf_validate"):
            assert name in _lib.EXPORTS_EXT and hasattr(lib, name), name
            assert len(getattr(lib, name).argtypes) == len(decl[name]), name
    assert lib.onerf_abi_version() == 2
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "onerf_ext.h")).read()
    assert f"#define ONERF_VALIDATE_RECORD_DOUBLES {_lib.VALIDATE_RECORD_DOUBLES}\n" in header


def test_workspace_is_sized_by_the_chunk_alone(lib):
    f = lib.onerf_validate_workspace_bytes
    assert f(0, 64, 64) == 0 and f(-3, 64, 64) == 0 and f(1024, 1, 0) == 0 and f(1024, 64, -1) == 0
    a256 = lambda x: (x + 255) // 256 * 256
    for chunk, s, k in ((1, 2, 0), (1000, 64, 0), (32768, 64, 64), (65536, 64, 128)):
        maps = lambda rows, S: 2 * a256(rows * S * 4) + 4 * a256(rows * 4) + 2 * a256(rows * 12)
        want = (a256(chunk * 64 * 4) + maps(chunk, s) + maps(chunk if k else 0, s + k)
                + a256(lib.onerf_render_rays_workspace_bytes(chunk, s, k)))
        assert f(chunk, s, k) == want, (chunk, s, k)
    # per-sample arrays are chunk-sized: a 640 x 480 image in 32 768-ray chunks needs less than its weights and z_vals
    assert f(32768, 64, 64) < 640 * 480 * (64 + 128) * 2 * 4 + lib.onerf_render_rays_workspace_bytes(32768, 64, 64)


def test_refusals_come_before_any_cuda_call(lib):
    """ONERF_ERR_BAD_ARG with a message for every refusal; the context is never dereferenced on these paths."""
    from object_nerf_b200 import _lib
    ctx = ctypes.c_void_p(1)

    def good():
        a = _lib.ValidateArgs()
        r, la = a.render, a.loss
        r.n_rays, r.n_samples, r.n_importance, r.forward_instance, r.is_eval = 100, 64, 64, 1, 1
        r.rays = a.instance_ids = a.code_table = 0x1000
        la.n_rays = 100
        la.rgbs = la.depths = la.valid_mask = la.instance_mask = la.instance_mask_weight = 0x1000
        a.ray_begin, a.ray_end, a.chunk_rays, a.record = 0, 100, 32, 0x1000
        r.workspace, r.workspace_bytes = 0x10000, lib.onerf_validate_workspace_bytes(32, 64, 64)
        return a

    def refused(message, **change):
        a = good()
        for path, value in change.items():
            obj, _, field = path.rpartition("__")
            setattr(getattr(a, obj) if obj else a, field, value)
        assert lib.onerf_validate_frame(ctx, ctypes.byref(a), None) == -1, change
        assert message in lib.onerf_last_error(), (change, lib.onerf_last_error())

    assert lib.onerf_validate_frame(None, None, None) == -1 and b"null" in lib.onerf_last_error()
    refused(b"tile outside", ray_begin=-1)
    refused(b"tile outside", ray_end=101)
    refused(b"tile outside", ray_begin=7, ray_end=6)
    refused(b"chunk_rays", chunk_rays=0)
    refused(b"forward_instance", render__forward_instance=0)
    refused(b"is_eval", render__is_eval=0)
    refused(b"training workspace", render__train_ws=0x20000)
    refused(b"perturb", render__perturb=0.5)
    refused(b"noise_std", render__noise_std=1.0)
    refused(b"record", record=None)
    refused(b"record", record=0x1004)
    refused(b"256-byte aligned", render__workspace=0x10010)
    refused(b"256-byte aligned", render__workspace=None)
    refused(b"workspace too small", render__workspace_bytes=good().render.workspace_bytes - 1)
    refused(b"null batch buffer", loss__depths=None)
    refused(b"loss.n_rays", loss__n_rays=99)
    refused(b"psnr_mask", psnr_mask=7)
    refused(b"finalize", finalize=1)
    out = (ctypes.c_float * 8)()
    assert lib.onerf_validate_finalize(ctx, None, out, 1, out, out, out, out, None) == -1
    assert lib.onerf_validate_finalize(ctx, 0x1004, out, 1, out, out, out, out, None) == -1
    assert b"8-byte aligned" in lib.onerf_last_error()
    assert lib.onerf_validate_finalize(ctx, 0x1000, out, 1, out, out, out, None, None) == -1
    assert b"null output" in lib.onerf_last_error()


# ------------------------------------------------------------------------------------------------
# the record arithmetic, restated in float64
# ------------------------------------------------------------------------------------------------
def _tile_record(maps, batch, begin, end, psnr_all=False):
    """What batch_stats_kernel and the evaluation compositing add for rays [begin, end) (loss_terms.cuh)."""
    rec = np.zeros(18)
    sl = slice(begin, end)
    b = {k: v.numpy()[sl] for k, v in batch.items()}
    valid, inst, tpos, w = b["valid_mask"].astype(bool), b["instance_mask"].astype(bool), b["depths"] > 0, b["instance_mask_weight"].astype(np.float64)
    rec[0], rec[1], rec[2] = 3 * valid.sum(), (valid & tpos).sum(), valid.sum()
    rec[3], rec[4], rec[5] = 3 * (valid & inst).sum(), (valid & inst & tpos).sum(), tpos.sum()
    passes = ("coarse", "fine") if "rgb_fine" in maps else ("coarse",)
    for f, typ in enumerate(passes):
        m = {k: maps[f"{k}_{typ}"].numpy()[sl].astype(np.float64) for k in cases.LOSS_MAP_KEYS}
        e_rgb = ((m["rgb"] - b["rgbs"]) ** 2).sum(1)
        e_irgb = ((m["rgb_instance"] - b["rgbs"]) ** 2).sum(1)
        rec[6 + 0 + f] = e_rgb[valid].sum()
        rec[6 + 2 + f] = ((m["depth"] - b["depths"]) ** 2)[valid & tpos].sum()
        rec[6 + 4 + f] = (((np.clip(m["opacity_instance"], 0, 1) - inst) ** 2) * w)[valid].sum()
        rec[6 + 6 + f] = (e_irgb * w)[valid & inst].sum()
        rec[6 + 8 + f] = (((m["depth_instance"] - b["depths"]) ** 2) * w)[valid & inst & tpos].sum()
        if typ == passes[-1]:
            pm = np.ones_like(valid) if psnr_all else valid & inst
            rec[16], rec[17] = e_rgb[pm].sum(), 3 * pm.sum()
    return rec


def _finalize(rec, conf, has_fine):
    """validate_finalize_kernel: loss_sum, {present term: value}, psnr."""
    present = [True, rec[5] > 0, rec[2] > 0, rec[3] > 0, rec[5] > 0 and rec[4] > 0]
    terms, total = {}, 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        for t, name in enumerate(TERMS):
            if present[t]:
                v = rec[6 + 2 * t] / rec[t] + (rec[6 + 2 * t + 1] / rec[t] if has_fine else 0.0)
                terms[name] = v
                total += conf[name + "_weight"] * v
        psnr = -10.0 * np.log10(rec[16] / rec[17]) if rec[17] > 0 else float("nan")
    return total, terms, psnr


@pytest.mark.parametrize("tiles", [1, 2, 3])
@pytest.mark.parametrize("name", sorted(cases.LOSS_CASES))
def test_summed_tile_records_finalise_to_the_oracle_loss_and_psnr(name, tiles):
    from object_nerf_b200 import parallel
    from oracle import onerf_oracle as O
    c = cases.LOSS_CASES[name]
    maps, batch = cases.build_loss_case(c)
    n = c["n"]
    rec = sum(_tile_record(maps, batch, *parallel.shard_bounds(n, tiles, r)) for r in range(tiles))
    assert np.array_equal(rec[:6], _tile_record(maps, batch, 0, n)[:6])
    total, terms, psnr = _finalize(rec, cases.LOSS_CONF, c["fine"])
    m64 = {k: v.double() for k, v in maps.items()}
    b64 = {k: (v.double() if v.is_floating_point() else v) for k, v in batch.items()}
    want_sum, want_terms = O.total_loss(m64, b64, cases.LOSS_CONF)
    assert sorted(terms) == sorted(want_terms)
    for k, v in want_terms.items():
        assert terms[k] == pytest.approx(float(v), rel=1e-12), k
    assert total == pytest.approx(float(want_sum), rel=1e-12)
    typ = "fine" if c["fine"] else "coarse"
    mask = (batch["valid_mask"] * batch["instance_mask"]).view(-1, 1).repeat(1, 3)          # train.py:185-188
    value = ((m64[f"rgb_{typ}"] - b64["rgbs"]) ** 2)[mask]
    want_psnr = float(-10 * torch.log10(torch.mean(value)))                                # utils/metrics.py:5-15
    assert psnr == pytest.approx(want_psnr, rel=1e-12, nan_ok=True)
    assert math.isnan(psnr) == (c["p_inst"] == 0.0)
    every = sum(_tile_record(maps, batch, *parallel.shard_bounds(n, tiles, r), psnr_all=True) for r in range(tiles))
    want_all = float(-10 * torch.log10(torch.mean((m64[f"rgb_{typ}"] - b64["rgbs"]) ** 2)))
    assert _finalize(every, cases.LOSS_CONF, c["fine"])[2] == pytest.approx(want_all, rel=1e-12)


# ------------------------------------------------------------------------------------------------
# validate_frame's host logic
# ------------------------------------------------------------------------------------------------
class _FakeValidateLib(_FakeLib):
    def onerf_validate_workspace_bytes(self, chunk, s, k):
        return 1024 + chunk

    def onerf_validate_frame(self, ctx, a, stream):
        a = a._obj
        n = a.render.n_rays
        self.calls.append(("frame", dict(
            n=n, tile=(a.ray_begin, a.ray_end), chunk=a.chunk_rays, finalize=a.finalize, psnr_mask=a.psnr_mask,
            flags=(a.render.forward_instance, a.render.is_eval, a.render.perturb, a.render.noise_std, bool(a.render.train_ws)),
            rays=self.view(a.render.rays, n * 8).reshape(n, 8).copy(), ids=self.view(a.instance_ids, n, ctypes.c_int64).copy(),
            valid=self.view(a.loss.valid_mask, n, ctypes.c_uint8).copy(), inst=self.view(a.loss.instance_mask, n, ctypes.c_uint8).copy(),
            weights=(a.loss.color_weight, a.loss.depth_weight, a.loss.opacity_weight, a.loss.instance_color_weight,
                     a.loss.instance_depth_weight),
            maps={typ: {k: getattr(getattr(a.render, typ), k) for k in
                        ("weights", "z_vals", "opacity", "rgb", "depth", "rgb_instance", "depth_instance", "opacity_instance")}
                  for typ in ("coarse", "fine")}, grid=bool(a.render.grid), ws=(a.render.workspace, a.render.workspace_bytes))))
        self.view(a.record, 18, ctypes.c_double)[:] = np.arange(18) + 1.0 + a.ray_begin
        if a.finalize:
            self.view(a.loss.loss_sum_out, 6)[:] = [1, 2, 3, 4, 5, 6]
            self.view(a.loss.present_out, 5, ctypes.c_int32)[:] = [1, 1, 0, 1, 0]
            self.view(a.psnr_out, 1)[0] = 7.0
        return 0

    def onerf_validate_finalize(self, ctx, record, weights, has_fine, loss_sum, terms, present, psnr, stream):
        self.calls.append(("finalize", self.view(record, 18, ctypes.c_double).copy(), list(weights), has_fine))
        self.view(loss_sum, 1)[0] = 11.0
        self.view(psnr, 1)[0] = 12.0
        return 0


def _stub(monkeypatch):
    import contextlib

    from object_nerf_b200 import _lib
    fake = _FakeValidateLib()
    monkeypatch.setattr(_lib, "load", lambda: fake)
    monkeypatch.setattr(_lib, "ctx", lambda dev: None)
    monkeypatch.setattr(_lib, "stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    return fake


def _problem(n=40):
    from object_nerf_b200 import synthetic as S
    from tests import helpers
    inp = cases.build_grad_case(n)
    models = {k: S.make_model(w, True, "cpu") for k, w in inp["weights"].items()}
    batch = {k: v.clone()[None] for k, v in inp["batch"].items()}                            # the loader's leading 1
    batch["rays"] = torch.cat([inp["rays"], torch.full((n, 3), 9.0)], 1)[None]               # 11 dataset columns
    batch["instance_ids"] = inp["instance_ids"][None]
    return models, {"xyz": S.GridModule(inp["grid"]), "dir": None}, helpers.CodeLib(inp["code_table"]), batch, inp


KW = dict(N_samples=64, N_importance=64, use_disp=False, white_back=False)


def test_validate_frame_plumbing_with_the_library_stubbed(monkeypatch):
    """The leading dimension is dropped and the first 8 ray columns are passed; bool masks go as bytes; the loss weights
    in TERMS order; only the requested maps of the last pass get a buffer, per-sample arrays never; the render flags are
    validation's; the result has the reference's key names; a second call reuses plan and workspace."""
    from object_nerf_b200 import _lib, training
    fake = _stub(monkeypatch)
    models, embeddings, lib, batch, inp = _problem()
    out = training.validate_frame(models, embeddings, lib, batch, cases.LOSS_CONF, chunk=16, **KW)
    assert sorted(out) == sorted(["loss_sum", "terms", "present", "psnr", "rgb_fine", "depth_fine", "rgb_instance_fine",
                                  "depth_instance_fine", "opacity_instance_fine"])
    assert out["loss_sum"].item() == 1 and out["terms"].tolist() == [2, 3, 4, 5, 6] and out["psnr"].item() == 7
    assert out["present"].tolist() == [1, 1, 0, 1, 0] and out["present"].dtype == torch.int32
    assert out["rgb_fine"].shape == (40, 3) and out["depth_fine"].shape == (40,)
    assert [c[0] for c in fake.calls] == ["pack", "pack", "frame"]
    rec = fake.calls[-1][1]
    assert rec["n"] == 40 and rec["tile"] == (0, 40) and rec["chunk"] == 16 and rec["finalize"] == 1
    assert rec["psnr_mask"] == _lib.PSNR_VALID_INSTANCE and rec["flags"] == (1, 1, 0.0, 0.0, False) and rec["grid"]
    assert np.array_equal(rec["rays"], inp["rays"].numpy())
    assert np.array_equal(rec["ids"], inp["instance_ids"].view(-1).numpy())
    assert np.array_equal(rec["valid"], inp["batch"]["valid_mask"].numpy().astype(np.uint8))
    assert np.array_equal(rec["inst"], inp["batch"]["instance_mask"].numpy().astype(np.uint8))
    assert rec["weights"] == pytest.approx(tuple(cases.LOSS_CONF[t + "_weight"] for t in TERMS))
    assert not any(rec["maps"]["coarse"].values())
    assert rec["maps"]["fine"]["rgb"] == out["rgb_fine"].data_ptr() and rec["maps"]["fine"]["opacity"] is None
    assert rec["maps"]["fine"]["weights"] is None and rec["maps"]["fine"]["z_vals"] is None
    assert rec["ws"][1] >= 1024 + 16
    again = training.validate_frame(models, embeddings, lib, batch, cases.LOSS_CONF, chunk=16, **KW)
    assert again["rgb_fine"].data_ptr() == out["rgb_fine"].data_ptr() and fake.calls[-1][1]["ws"] == rec["ws"]
    assert len(training._val_plans[models["coarse"]]) == 1
    # typed, contiguous batch tensors are read in place (what a captured call replays on)
    typed = {k: (v.view(torch.uint8) if v.dtype == torch.bool else v) for k, v in batch.items()}
    typed["rays"] = batch["rays"][..., :8].contiguous()
    seen = {}
    real = fake.onerf_validate_frame
    fake.onerf_validate_frame = lambda ctx, a, stream: (seen.update(rays=a._obj.render.rays, valid=a._obj.loss.valid_mask,
                                                                    ids=a._obj.instance_ids), real(ctx, a, stream))[1]
    training.validate_frame(models, embeddings, lib, typed, cases.LOSS_CONF, chunk=16, **KW)
    assert seen == dict(rays=typed["rays"].data_ptr(), valid=typed["valid_mask"].data_ptr(), ids=typed["instance_ids"].data_ptr())


def test_validate_frame_keys_passes_and_refusals(monkeypatch):
    from object_nerf_b200 import _lib, training
    fake = _stub(monkeypatch)
    models, embeddings, lib, batch, _ = _problem()
    coarse = {"coarse": models["coarse"]}
    out = training.validate_frame(coarse, embeddings, lib, batch, cases.LOSS_CONF, keys=("opacity", "rgb"),
                                  **dict(KW, N_importance=0))
    assert sorted(k for k in out if k.endswith("_coarse")) == ["opacity_coarse", "rgb_coarse"]
    rec = fake.calls[-1][1]
    assert rec["maps"]["coarse"]["rgb"] == out["rgb_coarse"].data_ptr() and not any(rec["maps"]["fine"].values())
    assert sorted(training.validate_frame(models, embeddings, lib, batch, cases.LOSS_CONF, keys=(), **KW)) == [
        "loss_sum", "present", "psnr", "terms"]
    # a batch without instance_mask: every ray counts for the PSNR, no instance pixel for the loss
    bare = {k: v for k, v in batch.items() if not k.startswith("instance_mask")}
    training.validate_frame(models, embeddings, lib, bare, cases.LOSS_CONF, **KW)
    rec = fake.calls[-1][1]
    assert rec["psnr_mask"] == _lib.PSNR_ALL_RAYS and not rec["inst"].any()
    with pytest.raises(KeyError, match="weights"):
        training.validate_frame(models, embeddings, lib, batch, cases.LOSS_CONF, keys=("rgb", "weights"), **KW)
    with pytest.raises(ValueError, match="chunk"):
        training.validate_frame(models, embeddings, lib, batch, cases.LOSS_CONF, chunk=0, **KW)
    with pytest.raises(ValueError, match="8 columns"):
        training.validate_frame(models, embeddings, lib, dict(batch, rays=batch["rays"][..., :6]), cases.LOSS_CONF, **KW)


def test_cpu_tensors_are_refused_by_the_real_binding():
    from object_nerf_b200 import training
    models, embeddings, lib, batch, _ = _problem(8)
    with pytest.raises(RuntimeError, match="CUDA"):
        training.validate_frame(models, embeddings, lib, batch, cases.LOSS_CONF, **KW)


def test_sharded_frame_renders_its_tile_reduces_the_record_and_finalises(monkeypatch):
    import torch.distributed as dist

    from object_nerf_b200 import parallel, training
    fake = _stub(monkeypatch)
    models, embeddings, lib, batch, _ = _problem(41)
    reduced = []
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 1)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 3)
    monkeypatch.setattr(dist, "all_reduce", lambda t, op=None, group=None: (reduced.append((t.dtype, t.numel(), op)), t.mul_(3))[1])
    monkeypatch.setattr(parallel, "gather_tiles", lambda local, n, group=None: local.new_zeros((n,) + tuple(local.shape[1:])))
    out = training.validate_frame(models, embeddings, lib, batch, cases.LOSS_CONF, chunk=16, group=object(), **KW)
    frame, fin = fake.calls[-2], fake.calls[-1]
    assert frame[0] == "frame" and frame[1]["tile"] == parallel.shard_bounds(41, 3, 1) == (14, 28) and frame[1]["finalize"] == 0
    assert reduced == [(torch.float64, 18, dist.ReduceOp.SUM)]
    assert fin[0] == "finalize" and np.array_equal(fin[1], 3 * (np.arange(18) + 15.0)) and fin[3] == 1
    assert fin[2] == pytest.approx([cases.LOSS_CONF[t + "_weight"] for t in TERMS])
    assert out["loss_sum"].item() == 11 and out["psnr"].item() == 12 and out["rgb_fine"].shape == (41, 3)


# ------------------------------------------------------------------------------------------------
# two gloo ranks reduce their tiles' records to the single-process record
# ------------------------------------------------------------------------------------------------
def _reduce_worker(rank, world, port, ret):
    import torch.distributed as dist

    from object_nerf_b200 import parallel
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        c = cases.LOSS_CASES["loss_train"]
        maps, batch = cases.build_loss_case(c)
        rec = torch.from_numpy(_tile_record(maps, batch, *parallel.shard_bounds(c["n"], world, rank)))
        dist.all_reduce(rec, op=dist.ReduceOp.SUM, group=dist.group.WORLD)
        ret[rank] = rec.tolist()
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_reduce_to_the_single_process_record():
    import torch.multiprocessing as mp
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_reduce_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    c = cases.LOSS_CASES["loss_train"]
    maps, batch = cases.build_loss_case(c)
    whole = _tile_record(maps, batch, 0, c["n"])
    assert ret[0] == ret[1]
    assert np.allclose(np.array(ret[0]), whole, rtol=1e-13, atol=0) and np.array_equal(np.array(ret[0])[:6], whole[:6])
    assert _finalize(np.array(ret[0]), cases.LOSS_CONF, True)[0] == pytest.approx(_finalize(whole, cases.LOSS_CONF, True)[0], rel=1e-13)
