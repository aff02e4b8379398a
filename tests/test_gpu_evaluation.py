"""evaluation.evaluate_frames on a synthetic voxel scene: the one combined render per frame gives, at each object's
pixels, the bits of a render with that object's code everywhere; the numbers are the float64 restatement
(tests/metrics_oracle.py) of those maps; the rays are the frame store's training rays; two gloo ranks on one GPU return
what one process returns, bit for bit."""
import math
import os
import socket

import numpy as np
import pytest
import torch

from tests import metrics_oracle as MO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H, W, F = 48, 64, 3
IDS = (3, 5, 12)                 # 12 is absent from frame 1
CONF = {"model": {"N_samples": 32, "N_importance": 32, "use_disp": False}}


def _scene(dev=DEV):
    from object_nerf_b200 import Embedding, frames
    from object_nerf_b200 import synthetic as S
    models = {k: S.make_model(S.make_weights(seed, True, 8.0, 1.0), True, dev).eval()
              for k, seed in (("coarse", 103), ("fine", 1103))}
    emb = S.GridModule(S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05)).to(dev)
    lib = S.make_code_library(S.make_codes(105)).to(dev)
    rng = np.random.default_rng(11)
    focal = 0.5 * W / math.tan(math.radians(30))
    poses = []
    for f in range(F):
        cam = np.array([-1.6, 0.1, 0.15]) + rng.normal(size=3) * 0.1
        fwd = -cam / np.linalg.norm(cam)
        right = np.cross(fwd, [0, 0, 1.0])
        right /= np.linalg.norm(right)
        up = np.cross(right, fwd)
        poses.append(np.concatenate([np.stack([right, up, -fwd], 1), cam[:, None]], 1))
    labels = rng.choice([0, 3, 5, 12, 7], size=(F, H, W)).astype(np.uint16)
    labels[:, :H // 2, :W // 3] = 5                   # a block
    labels[1][labels[1] == 12] = 7
    fs = frames.FrameSet(np.stack(poses).astype(np.float32), rng.integers(0, 256, size=(F, H, W, 3), dtype=np.uint8),
                         np.zeros((F, H, W), np.float32), labels, focal=focal, near=0.15, far=3.0, scale_factor=1.0,
                         instance_ids=(3,), border=4, device=dev)
    return models, {"xyz": emb, "dir": Embedding(3, 4)}, lib, fs


def _render(scene, batch, **kw):
    from object_nerf_b200 import training
    from object_nerf_b200.evaluation import _NO_LOSS
    models, embeddings, lib, _ = scene
    out = training.validate_frame(models, embeddings, lib, batch, _NO_LOSS, N_samples=32, N_importance=32,
                                  use_disp=False, white_back=False, keys=("rgb", "rgb_instance"), chunk=1000, **kw)
    return {k: out[k].clone() for k in ("rgb_fine", "rgb_instance_fine")}


@pytest.fixture(scope="module")
def scene():
    return _scene()


def test_one_render_serves_every_object(scene):
    from object_nerf_b200 import evaluation
    fs = scene[3]
    for f in range(F):
        batch = evaluation.frame_batch(fs, f, IDS)
        both = _render(scene, batch)
        lab = fs.tensors["labels"][f].long() & 0xFFFF
        for k in IDS:
            alone = _render(scene, dict(batch, instance_ids=torch.full_like(batch["instance_ids"], k)))
            assert torch.equal(both["rgb_fine"], alone["rgb_fine"])
            m = lab == k
            assert torch.equal(both["rgb_instance_fine"][m], alone["rgb_instance_fine"][m]), (f, k)
        assert ((batch["instance_ids"] == lab) | ~torch.isin(lab, torch.tensor(IDS, device=DEV))).all()


def test_rays_are_the_stores_training_rays(scene):
    from object_nerf_b200 import evaluation
    fs = scene[3]
    expanded = fs.expand()["all_rays"].view(F, H * W, 8)
    for f in range(F):
        assert torch.equal(evaluation.frame_batch(fs, f)["rays"], expanded[f])


@pytest.mark.parametrize("window", [3, 7])
def test_numbers_are_the_float64_restatement_of_the_maps(scene, window):
    from object_nerf_b200 import evaluation
    models, embeddings, lib, fs = scene
    res = evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, object_ids=IDS, window=window, chunk=1000)
    res = {k: v.cpu().numpy() for k, v in res.items()}
    assert res["psnr"].shape == (F,) and res["psnr_objects"].shape == (F, len(IDS))
    P, S = [], []
    for f in range(F):
        batch = evaluation.frame_batch(fs, f, IDS)
        maps = {k: v.cpu().numpy() for k, v in _render(scene, batch).items()}
        _, psnr, ssim = MO.metrics(maps["rgb_fine"], batch["rgbs"].cpu().numpy(), H, W, batch["valid_mask"].cpu().numpy(),
                                   maps["rgb_instance_fine"], fs.tensors["labels"][f].cpu().numpy().view(np.uint16),
                                   IDS, window)
        P.append(psnr)
        S.append(ssim)
    P, S = np.array(P), np.array(S)
    assert np.isnan(P[1, 3]) and np.isnan(S[1, 3]) and np.isfinite(P[:, :3]).all()
    for got, want in ((res["psnr"], P[:, 0]), (res["ssim"], S[:, 0]), (res["psnr_objects"], P[:, 1:]),
                      (res["ssim_objects"], S[:, 1:])):
        assert np.array_equal(np.isnan(got), np.isnan(want))
        fin = np.isfinite(want)
        assert np.abs(got[fin] - want[fin]).max() <= 1e-6 * max(1, np.abs(want[fin]).max())
    assert abs(res["mean_psnr"] - P[:, 0].mean()) <= 1e-5
    assert np.allclose(res["mean_ssim_objects"], np.nanmean(S[:, 1:], 0), rtol=1e-6, atol=1e-7)
    # without objects: the scene column alone, the same numbers
    alone = evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, window=window, chunk=1000)
    assert torch.equal(alone["psnr"].cpu(), torch.from_numpy(res["psnr"]))
    assert alone["psnr_objects"].shape == (F, 0)


def test_refusals(scene):
    from object_nerf_b200 import evaluation
    models, embeddings, lib, fs = scene
    with pytest.raises(ValueError, match="at most 64"):
        evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, object_ids=range(65))
    with pytest.raises(ValueError, match="repeat"):
        evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, object_ids=(3, 3))
    with pytest.raises(ValueError, match="code-table rows"):
        evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, object_ids=(64,))


def _worker(rank, world, port, ret):
    import torch.distributed as dist
    from object_nerf_b200 import evaluation
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        models, embeddings, lib, fs = _scene()
        single = evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, object_ids=IDS, chunk=700)
        shared = evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, object_ids=IDS, chunk=700,
                                            group=dist.group.WORLD)
        ret[rank] = ({k: v.cpu().numpy() for k, v in single.items()}, {k: v.cpu().numpy() for k, v in shared.items()})
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_equal_one_process():
    import torch.multiprocessing as mp
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    for rank in range(2):
        single, shared = ret[rank]
        for k in single:
            assert np.array_equal(single[k], shared[k], equal_nan=True), (rank, k)
            assert np.array_equal(ret[0][1][k], shared[k], equal_nan=True), (rank, k)
