"""training.validate_frame (onerf_validate_frame: a validation image per call, TotalLoss and the validation PSNR summed
in the compositing kernels) against render_rays(is_eval=True) in 32 768-ray chunks, losses.TotalLoss and a float64
restatement on the same seeded image: maps, loss, skip rules, chunk / tile independence, sharding, graph replay and
every refusal."""
import ctypes as C
import math
import os
import socket
import types

import pytest
import torch

from tests import cases, grad_plain, helpers

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TERMS = ("color_loss", "depth_loss", "opacity_loss", "instance_color_loss", "instance_depth_loss")
ALL_KEYS = ("opacity", "rgb", "depth", "rgb_instance", "depth_instance", "opacity_instance")
RENDER = dict(N_samples=64, N_importance=64, use_disp=False, white_back=False)


def _scene(use_voxel, n, dev=DEV, fine=True):
    from object_nerf_b200 import Embedding
    inp = cases.build_grad_case(n) if use_voxel else grad_plain.build_grad_case_plain(n)
    models = {k: helpers.make_model(w, use_voxel, dev).eval() for k, w in inp["weights"].items() if fine or k == "coarse"}
    emb = helpers.GridModule(inp["grid"]).to(dev) if use_voxel else Embedding(3, 10)
    lib = helpers.CodeLib(inp["code_table"]).to(dev)
    batch = {k: v.to(dev)[None] for k, v in inp["batch"].items()}          # the loader's leading dimension
    batch["rays"] = torch.cat([inp["rays"], torch.zeros(n, 3)], 1).to(dev)[None]   # dataset rays carry extra columns
    batch["instance_ids"] = inp["instance_ids"].to(dev)[None]
    return models, {"xyz": emb, "dir": Embedding(3, 4)}, lib, batch


def _validate(scene, precision="bf16", **over):
    from object_nerf_b200 import training
    models, embeddings, lib, batch = scene
    kw = dict(RENDER, keys=ALL_KEYS, precision=precision)
    kw.update(over)
    if len(models) == 1:
        kw["N_importance"] = 0
    out = training.validate_frame(models, embeddings, lib, batch, cases.LOSS_CONF, **kw)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in out.items()}


def _plan(scene):
    from object_nerf_b200 import training
    return list(training._val_plans[scene[0]["coarse"]].values())[-1]


def _reference_maps(scene, precision):
    """render_rays(is_eval=True) over the image in 32 768-ray chunks, as ObjectNeRFSystem.forward runs it."""
    from object_nerf_b200 import render_rays
    models, embeddings, lib, batch = scene
    rays = batch["rays"][0][:, :8].contiguous()
    codes = lib.embedding_instance(batch["instance_ids"].view(-1)).detach()
    parts = []
    with torch.no_grad():
        for i in range(0, rays.shape[0], 32768):
            parts.append(render_rays(models, embeddings, rays[i:i + 32768], embedding_instance=codes[i:i + 32768],
                                     N_samples=64, N_importance=64 if "fine" in models else 0, perturb=0, noise_std=0,
                                     use_disp=False, white_back=False, is_eval=True, precision=precision))
    return {k: torch.cat([p[k] for p in parts], 0) for k in parts[0]}


def _flat(batch):
    return {k: v[0] for k, v in batch.items()}


def _psnr(rgb, batch, masked=True):
    """utils/metrics.psnr as validation_step calls it (train.py:185-190, :220)."""
    b = _flat(batch)
    value = (rgb - b["rgbs"]) ** 2
    if masked:
        value = value[(b["valid_mask"] * b["instance_mask"]).view(-1, 1).repeat(1, 3)]
    return -10 * torch.log10(torch.mean(value))


def _float64_loss(maps, batch):
    b = {k: (v.double() if v.is_floating_point() else v) for k, v in _flat(batch).items()}
    return cases.total_loss({k: v.double() for k, v in maps.items()}, b)


def _check_loss(out, maps, batch, rel):
    """loss_sum, terms and flags against losses.TotalLoss on `maps` (both sum in float64) and, where no term is skipped,
    against the float64 restatement."""
    from object_nerf_b200.losses import TotalLoss
    want_sum, want_dict = TotalLoss(cases.LOSS_CONF)(maps, _flat(batch))
    flags = out["present"].tolist()
    got = {t: out["terms"][i].item() for i, t in enumerate(TERMS) if flags[i]}
    assert sorted(got) == sorted(want_dict), (got, want_dict)
    for t, v in want_dict.items():
        assert got[t] == pytest.approx(v.item(), rel=1e-6, abs=1e-12, nan_ok=True), t
    assert out["loss_sum"].item() == pytest.approx(want_sum.item(), rel=1e-6, nan_ok=True)
    if all(flags) and not math.isnan(want_sum.item()):
        assert out["loss_sum"].item() == pytest.approx(_float64_loss(maps, batch).item(), rel=rel)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("use_voxel", [True, False])
def test_maps_loss_and_psnr_at_every_frame_size(use_voxel, precision):
    """Frames of 1, 127, 4 096 and 70 001 rays with chunk smaller than, equal to and larger than the frame: every map
    bit-identical to render_rays, the loss within 1e-6 of TotalLoss on those maps and 1e-5 of the float64 restatement,
    the PSNR the reference formula over valid_mask * instance_mask."""
    for n in (1, 127, 4096, 70001):
        scene = _scene(use_voxel, n)
        want = _reference_maps(scene, precision)
        chunks = (max(n // 3, 1), n, n + 5) if n < 70001 else ((32768,) if precision == "fp32" else (32768, n, 100000))
        for chunk in chunks:
            out = _validate(scene, precision, chunk=chunk)
            for k in ALL_KEYS:
                assert torch.equal(out[f"{k}_fine"], want[f"{k}_fine"]), (n, chunk, k)
            _check_loss(out, want, scene[3], 1e-5)
            ref_psnr = _psnr(want["rgb_fine"], scene[3])
            assert out["psnr"].item() == pytest.approx(ref_psnr.item(), rel=1e-5, nan_ok=True), (n, chunk)


def test_unrequested_maps_are_not_written_and_change_nothing():
    scene = _scene(True, 4096)
    full = _validate(scene, chunk=1000)
    record = _plan(scene).record.clone()
    none = _validate(scene, chunk=1000, keys=())
    assert sorted(none) == ["loss_sum", "present", "psnr", "terms"]
    again = _plan(scene).record          # float64 atomics: the order of the block sums differs from run to run
    assert torch.equal(again[:6], record[:6]) and again[17] == record[17]
    assert ((again - record).abs() <= 1e-12 * record.abs()).all()
    assert torch.equal(none["present"], full["present"])
    for k in ("loss_sum", "terms", "psnr"):
        assert torch.allclose(none[k], full[k], rtol=1e-6, atol=0), k
    some = _validate(scene, chunk=1000, keys=("depth",))
    assert torch.equal(some["depth_fine"], full["depth_fine"]) and "rgb_fine" not in some


def test_psnr_over_every_ray_without_an_instance_mask():
    """mask = None (train.py:189-190): every ray counts, valid or not; the batch is taken as one without instance
    pixels."""
    scene = _scene(True, 4096)
    models, embeddings, lib, batch = scene
    bare = {k: v for k, v in batch.items() if k not in ("instance_mask", "instance_mask_weight")}
    out = _validate((models, embeddings, lib, bare), chunk=1500)
    want = _reference_maps(scene, "bf16")
    assert torch.equal(out["rgb_fine"], want["rgb_fine"])
    assert out["psnr"].item() == pytest.approx(_psnr(want["rgb_fine"], batch, masked=False).item(), rel=1e-5)
    zero = dict(batch, instance_mask=torch.zeros_like(batch["instance_mask"]),
                instance_mask_weight=torch.zeros_like(batch["instance_mask_weight"]))
    _check_loss(out, want, zero, 1e-5)


@pytest.mark.parametrize("case", ["no_valid_ray", "no_depth", "no_instance", "no_fine"])
def test_skip_rules(case):
    """Flags as the reference's Nones, loss_sum over the present terms only, NaN exactly where the reference's mean of an
    empty set gives NaN (the color term without a valid ray, the PSNR with an empty mask)."""
    scene = _scene(True, 2048, fine=case != "no_fine")
    batch = scene[3]
    if case == "no_valid_ray":
        batch["valid_mask"] = torch.zeros_like(batch["valid_mask"])
    elif case == "no_depth":
        batch["depths"] = torch.zeros_like(batch["depths"])
    elif case == "no_instance":
        batch["instance_mask"] = torch.zeros_like(batch["instance_mask"])
    out = _validate(scene, chunk=700)
    want = _reference_maps(scene, "bf16")
    typ = "coarse" if case == "no_fine" else "fine"
    assert f"rgb_{typ}" in out and (typ == "fine" or "rgb_fine" not in out)
    assert torch.equal(out[f"rgb_{typ}"], want[f"rgb_{typ}"])
    _check_loss(out, want, batch, 1e-5)
    flags = out["present"].tolist()
    expect = {"no_valid_ray": [1, 1, 0, 0, 0], "no_depth": [1, 0, 1, 1, 0], "no_instance": [1, 1, 1, 0, 0],
              "no_fine": [1, 1, 1, 1, 1]}[case]
    assert flags == expect
    ref_psnr = _psnr(want[f"rgb_{typ}"], batch)
    assert math.isnan(ref_psnr.item()) == (case in ("no_valid_ray", "no_instance"))
    assert out["psnr"].item() == pytest.approx(ref_psnr.item(), rel=1e-5, nan_ok=True)
    assert math.isnan(out["loss_sum"].item()) == (case == "no_valid_ray")


def _tile_record(scene, begin, end, chunk):
    """The record of rays [begin, end) through the frame's plan (onerf_validate_frame without finalisation)."""
    from object_nerf_b200 import _lib
    plan = _plan(scene)
    a = plan.args
    a.ray_begin, a.ray_end, a.chunk_rays, a.finalize = begin, end, chunk, 0
    _lib.check(_lib.load().onerf_validate_frame(_lib.ctx(torch.device(DEV)), C.byref(a), _lib.stream()))
    torch.cuda.synchronize()
    return plan.record.clone()


def test_records_do_not_depend_on_chunks_or_tiles():
    """float64 sums in another order: chunk 1 000 against 65 536 within 1e-12; three tiles summed equal the frame."""
    n = 70001
    scene = _scene(True, n)
    _validate(scene, chunk=65536)
    whole = _plan(scene).record.clone()
    # the plan's buffers are alive for the raw calls below (the batch tensors are the scene's)
    small = _tile_record(scene, 0, n, 1000)
    assert whole[:6].eq(small[:6]).all() and whole[17] == small[17] and whole[17] > 0
    assert ((whole - small).abs() <= 1e-12 * whole.abs()).all()
    tiles = sum(_tile_record(scene, b, e, 65536) for b, e in ((0, 23333), (23333, 23334), (23334, n)))
    assert whole[:6].eq(tiles[:6]).all() and ((whole - tiles).abs() <= 1e-12 * whole.abs()).all()
    assert _tile_record(scene, 500, 500, 64).eq(0).all()


def test_graph_replay_validates_the_batch_as_it_is_then():
    """Capture one validate_frame, overwrite the batch tensors in place with a second image, replay: bit for bit the
    eager call on the second image."""
    n = 4096
    first, second = _scene(True, n), _scene(False, n)          # the plain case's rays and batch: another image
    models, embeddings, lib, batch = first
    batch = {k: (v.view(torch.uint8) if v.dtype == torch.bool else v).contiguous() for k, v in batch.items()}
    batch["rays"] = batch["rays"][..., :8].contiguous()
    image2 = {k: (v.view(torch.uint8) if v.dtype == torch.bool else v) for k, v in second[3].items()}
    image2["rays"] = image2["rays"][..., :8]
    scene = (models, embeddings, lib, batch)
    _validate(scene, chunk=1500)                                # warm-up: plan, workspace
    from object_nerf_b200 import training
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            held = training.validate_frame(models, embeddings, lib, batch, cases.LOSS_CONF, chunk=1500, keys=ALL_KEYS,
                                           **RENDER)
    for k in batch:
        batch[k].copy_(image2[k])
    graph.replay()
    torch.cuda.synchronize()
    replayed = {k: v.clone() for k, v in held.items()}
    eager = _validate((models, embeddings, lib, {k: v.clone() for k, v in image2.items()}), chunk=1500)
    assert sorted(replayed) == sorted(eager)
    for k in eager:                      # maps and flags bit for bit; the fp32 outputs of float64 atomic sums to an ulp
        if k.endswith("_fine") or k == "present":
            assert torch.equal(replayed[k], eager[k]), k
        else:
            assert torch.allclose(replayed[k], eager[k], rtol=1e-6, atol=0, equal_nan=True), k
    assert not torch.equal(replayed["rgb_fine"], _validate(first, chunk=1500)["rgb_fine"])


def test_every_refusal_is_bad_arg_with_a_message_and_launches_nothing():
    from object_nerf_b200 import _lib
    n = 127
    scene = _scene(True, n)
    _validate(scene, chunk=64)
    plan, lib, dev = _plan(scene), _lib.load(), torch.device(DEV)
    good = _lib.ValidateArgs.from_buffer_copy(plan.args)

    def refused(message, **change):
        a = _lib.ValidateArgs.from_buffer_copy(good)
        for path, value in change.items():
            obj, _, field = path.rpartition("__")
            setattr(getattr(a, obj) if obj else a, field, value)
        before = _lib.launch_count(dev)
        rc = lib.onerf_validate_frame(_lib.ctx(dev), C.byref(a), _lib.stream())
        assert rc == -1 and message in lib.onerf_last_error(), (change, rc, lib.onerf_last_error())
        assert _lib.launch_count(dev) == before, change

    ws, nbytes = good.render.workspace, good.render.workspace_bytes
    refused(b"tile outside", ray_begin=-1)
    refused(b"tile outside", ray_end=n + 1)
    refused(b"tile outside", ray_begin=5, ray_end=4)
    refused(b"chunk_rays", chunk_rays=0)
    refused(b"forward_instance", render__forward_instance=0)
    refused(b"is_eval", render__is_eval=0)
    refused(b"training workspace", render__train_ws=ws)
    refused(b"perturb", render__perturb=1.0)
    refused(b"noise_std", render__noise_std=1.0)
    refused(b"record", record=None)
    refused(b"record", record=good.record + 4)
    refused(b"256-byte aligned", render__workspace=ws + 16)
    refused(b"workspace too small", render__workspace_bytes=lib.onerf_validate_workspace_bytes(64, 64, 64) - 1)
    refused(b"null batch buffer", loss__valid_mask=None)
    refused(b"psnr_mask", psnr_mask=2)
    assert nbytes >= lib.onerf_validate_workspace_bytes(64, 64, 64)
    torch.cuda.synchronize()
    out = _validate(scene, chunk=64)                            # the good arguments still run
    assert torch.isfinite(out["loss_sum"])


# ------------------------------------------------------------------------------------------------
# sharding
# ------------------------------------------------------------------------------------------------
def _shard_worker(rank, world, port, backend, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        scene = _scene(True, 4099, dev=dev)
        single = _validate(scene, chunk=1000)
        shared = _validate(scene, chunk=1000, group=dist.group.WORLD)
        bad = [k for k in single if k.endswith("_fine") and not torch.equal(single[k], shared[k])]
        scalars = torch.cat([single["loss_sum"][None], single["terms"], single["psnr"][None]]).double()
        got = torch.cat([shared["loss_sum"][None], shared["terms"], shared["psnr"][None]]).double()
        ret[rank] = (sorted(shared) == sorted(single), bad, ((got - scalars).abs() / scalars.abs()).max().item(),
                     shared["present"].tolist() == single["present"].tolist(), got.tolist())
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_sharded_image_equals_the_single_process_image(backend):
    """Two ranks: maps bit-identical to the single-process call, the same loss, terms and PSNR on every rank (the fp32
    outputs of float64 records that agree within 1e-12)."""
    import torch.multiprocessing as mp
    world = 2
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("NCCL across devices needs two GPUs")
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, backend, ret)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    assert len(ret) == world
    for rank, (same_keys, bad, err, same_flags, _) in ret.items():
        assert same_keys and not bad and same_flags and err <= 1e-6, (rank, bad, err)
    assert ret[0][4] == ret[1][4]


# ------------------------------------------------------------------------------------------------
# the unmodified reference's validation_step
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_installed_validation_step_against_the_unmodified_reference(tmp_path, precision, monkeypatch):
    """ObjectNeRFSystem.validation_step of the unmodified reference on the CPU against the installed one on the GPU, on
    the drop-in fixture's scene (one 32 x 24 image): val_loss, every term and val_psnr within the training step's
    tolerances, and visualize_val_image's (7, 3, H, W) stack from the installed step's maps."""
    from oracle import ref_loader as R
    from tests import dropin_fixture as F
    if not R.available():
        pytest.skip("oracle/_ref not built")
    import object_nerf_b200.dropin as dropin
    from object_nerf_b200 import training
    batch = F.training_batch(n=32 * 24)
    del batch["pass_through_mask"]
    try:
        F.purge_reference_modules()
        R.install(cuda_noop=True)
        conf, paths = F.write_scene(str(tmp_path))
        train, ref_sys = F.make_system(conf, "cpu")
        F.fill_synthetic_weights(ref_sys)
        ref_sys.eval()
        with torch.no_grad():
            want = ref_sys.validation_step({k: v.clone() for k, v in batch.items()}, 1)
        sd = ref_sys.state_dict()
        F.purge_reference_modules()
        R.cuda_noop(False)
        dropin.install()
        train2, system = F.make_system(conf, "cuda:0")
        system.load_state_dict(sd, strict=True)
        system.eval()
        images = []
        system.logger = types.SimpleNamespace(experiment=types.SimpleNamespace(
            add_images=lambda tag, stack, step: images.append((tag, stack))))
        monkeypatch.setattr(training.validate_frame, "__kwdefaults__",
                            dict(training.validate_frame.__kwdefaults__, precision=precision))
        training.install_validation(train2.ObjectNeRFSystem, chunk=500)
        gpu_batch = {k: v.to("cuda:0") for k, v in batch.items()}
        got = system.validation_step(gpu_batch, 1)
        assert sorted(got) == sorted(want)
        tol = 2e-4 if precision == "fp32" else 2e-2
        for k in want:
            if k != "val_psnr":
                assert got[k].item() == pytest.approx(want[k].item(), rel=tol), k
        assert abs(got["val_psnr"].item() - want["val_psnr"].item()) < (1e-3 if precision == "fp32" else 0.05)
        try:
            import cv2  # noqa: F401  (visualize_depth's colour maps)
        except ImportError:
            return
        system.validation_step(gpu_batch, 0)
        (tag, stack), = images
        assert tag == "val/GT_pred_depth" and tuple(stack.shape) == (7, 3, 24, 32)
    finally:
        F.purge_reference_modules()
        R.cuda_noop(not torch.cuda.is_available())
