"""rendering.render_instances (onerf_render_instances: every object's maps in one render) against render_rays with each
column's code on every ray, bit for bit: both arithmetics, both models, K = 1, 2, 5 and 64, with and without a fine
pass, use_disp, chunks that do not divide the rays, N = 0 and 1; CUDA-graph replay, two gloo ranks, and
evaluate_frames(masks=True) against the loop of one validate_frame per object it replaces."""
import math
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KINDS = ("opacity_instance", "depth_instance", "rgb_instance")
SCENE_KINDS = ("rgb", "depth", "opacity")


def _scene(use_voxel, dev=DEV):
    from object_nerf_b200 import Embedding, synthetic as S
    models = {"coarse": S.make_model(S.make_weights(31, use_voxel, 8.0, 1.0), use_voxel, dev),
              "fine": S.make_model(S.make_weights(1031, use_voxel, 8.0, 1.0), use_voxel, dev)}
    xyz = (S.GridModule(S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05)).to(dev) if use_voxel
           else Embedding(3, 10))
    return models, {"xyz": xyz, "dir": Embedding(3, 4)}, S.make_code_library(S.make_codes(105)).to(dev)


def _rays(n, seed=104, dev=DEV):
    from object_nerf_b200 import synthetic as S
    return S.random_rays(seed, n).to(dev) if n else torch.zeros(0, 8, device=dev)


def _reference(scene, rays, i, n_importance, use_disp, precision):
    """render_rays with code row i on every ray, is_eval, nothing random."""
    from object_nerf_b200 import render_rays
    models, embeddings, lib = scene
    code = lib.embedding_instance.weight.detach()[i].expand(rays.shape[0], 64).contiguous()
    with torch.no_grad():
        return render_rays(models, embeddings, rays, N_samples=64, N_importance=n_importance, use_disp=use_disp,
                           perturb=0, noise_std=0, embedding_instance=code, is_eval=True, precision=precision)


def _instances(scene, rays, ids, n_importance, use_disp, precision, chunk, keys=None, group=None):
    from object_nerf_b200 import rendering
    models, embeddings, lib = scene
    passes = ("coarse", "fine") if n_importance else ("coarse",)
    keys = keys or tuple(f"{k}_{t}" for t in passes for k in KINDS + SCENE_KINDS)
    out = rendering.render_instances(models if n_importance else {"coarse": models["coarse"]}, embeddings, lib, rays,
                                     ids, N_samples=64, N_importance=n_importance, use_disp=use_disp, chunk=chunk,
                                     keys=keys, precision=precision, group=group)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in out.items()}


def _check(scene, rays, ids, n_importance=64, use_disp=False, precision="bf16", chunk=200):
    out = _instances(scene, rays, ids, n_importance, use_disp, precision, chunk)
    passes = ("coarse", "fine") if n_importance else ("coarse",)
    n, K = rays.shape[0], len(ids)
    for t in passes:
        assert out[f"opacity_instance_{t}"].shape == (n, K) and out[f"rgb_instance_{t}"].shape == (n, K, 3)
    refs = {}
    for k, i in enumerate(ids):
        if i not in refs:
            refs[i] = _reference(scene, rays, i, n_importance, use_disp, precision)
        ref = refs[i]
        for t in passes:
            for kind in KINDS:
                assert torch.equal(out[f"{kind}_{t}"][:, k], ref[f"{kind}_{t}"]), (k, i, t, kind)
            if k == 0:
                for kind in SCENE_KINDS:
                    assert torch.equal(out[f"{kind}_{t}"], ref[f"{kind}_{t}"]), (t, kind)
    return out


@pytest.mark.parametrize("use_voxel", [True, False], ids=["voxel", "plain"])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("K", [1, 2, 5, 64])
def test_columns_equal_one_render_per_code(use_voxel, precision, K):
    """Every column of both passes is the render with its code on every ray; 64 ids repeat one id."""
    ids = [3, 9, 0, 63, 17][:K] if K <= 5 else [(7 * k) % 64 for k in range(63)] + [9]
    _check(_scene(use_voxel), _rays(517), ids, precision=precision, chunk=200)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("use_voxel", [True, False], ids=["voxel", "plain"])
def test_coarse_only_and_use_disp(use_voxel, precision):
    _check(_scene(use_voxel), _rays(300), [4, 11, 4], n_importance=0, use_disp=True, precision=precision, chunk=128)


def test_chunk_that_does_not_divide_the_rays():
    _check(_scene(True), _rays(4099), [2, 5], chunk=1000)


def test_one_ray_and_no_ray():
    """One ray against the per-code renders; no ray (which render_rays itself does not take) gives empty maps."""
    scene = _scene(True)
    _check(scene, _rays(1), [1, 2, 3], chunk=64)
    out = _instances(scene, _rays(0), [1, 2, 3], 64, False, "bf16", 64)
    assert out["opacity_instance_fine"].shape == (0, 3) and out["rgb_instance_coarse"].shape == (0, 3, 3)
    assert out["rgb_fine"].shape == (0, 3)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_maps_asked_for_alone_equal_the_full_render(precision):
    """A pass without object maps skips the object branch, the fine pass without scene maps the scene branch (and a
    coarse-only render without scene maps the whole scene): the maps asked for keep the full render's bits."""
    scene, rays, ids = _scene(True), _rays(611), [7, 2, 7]
    for n_importance, key_sets in ((64, (("opacity_instance",), ("rgb_coarse",), ("depth_instance_coarse", "rgb_fine"),
                                         ("opacity_fine", "rgb_instance"))),
                                   (0, (("opacity_instance",), ("depth",)))):
        full = _instances(scene, rays, ids, n_importance, False, precision, 250)
        for keys in key_sets:
            part = _instances(scene, rays, ids, n_importance, False, precision, 250, keys=keys)
            assert len(part) == len(keys)
            for k, v in part.items():
                assert torch.equal(v, full[k]), (n_importance, keys, k)


def test_graph_replay_gives_the_eager_bits():
    """Capture one call, move the rays in place, replay: bit for bit the eager call on the new rays."""
    from object_nerf_b200 import rendering
    scene = _scene(True)
    rays, rays2 = _rays(777), _rays(777, seed=7)
    ids, kw = [6, 2], dict(N_samples=64, N_importance=64, use_disp=False, chunk=300)
    rendering.render_instances(*scene, rays, ids, **kw)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            held = rendering.render_instances(*scene, rays, ids, **kw)
    rays.copy_(rays2)
    graph.replay()
    torch.cuda.synchronize()
    replayed = {k: v.clone() for k, v in held.items()}
    eager = _instances(scene, rays2.clone(), ids, 64, False, "bf16", 300, keys=rendering.INSTANCE_KEYS)
    assert sorted(replayed) == sorted(eager)
    for k in eager:
        assert torch.equal(replayed[k], eager[k]), k


def _shard_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        scene, rays = _scene(True), _rays(1031)
        single = _instances(scene, rays, [5, 1, 5], 64, False, "bf16", 250)
        shared = _instances(scene, rays, [5, 1, 5], 64, False, "bf16", 250, group=dist.group.WORLD)
        ret[rank] = (sorted(single) == sorted(shared), [k for k in single if not torch.equal(single[k], shared[k])])
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_equal_one_process():
    import torch.multiprocessing as mp
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    assert len(ret) == 2
    for rank, (same_keys, bad) in ret.items():
        assert same_keys and not bad, (rank, bad)


# ------------------------------------------------------------------------------------------------
# evaluate_frames(masks=True)
# ------------------------------------------------------------------------------------------------
H, W, IDS = 64, 80, (3, 5, 9)
CONF = {"model": {"N_samples": 64, "N_importance": 64, "use_disp": False}}


def _frames(dev=DEV, n_frames=2):
    from object_nerf_b200 import frames
    rng = np.random.default_rng(0)
    poses = []
    for _ in range(n_frames):
        cam = np.array([-1.6, 0.1, 0.15]) + rng.normal(size=3) * 0.1
        fwd = -cam / np.linalg.norm(cam)
        right = np.cross(fwd, [0, 0, 1.0])
        right /= np.linalg.norm(right)
        poses.append(np.concatenate([np.stack([right, np.cross(right, fwd), -fwd], 1), cam[:, None]], 1))
    labels = rng.choice(np.array([0, *IDS], np.uint16), (n_frames, H, W))
    depths = rng.uniform(0.5, 3.0, (n_frames, H, W)).astype(np.float32)
    return frames.FrameSet(np.stack(poses).astype(np.float32), rng.integers(0, 256, (n_frames, H, W, 3), dtype=np.uint8),
                           depths, labels, focal=0.5 * W / math.tan(math.radians(30)), near=0.15, far=3.0,
                           scale_factor=1.0, instance_ids=(IDS[0],), device=dev)


def _old_mask_loop(scene, fs, chunk):
    """What evaluate_frames(masks=True) computed before render_instances: one validate_frame per object and frame,
    every pixel with that object's code, feeding MaskMetricsPlan."""
    from object_nerf_b200 import evaluation, metrics, training
    models, embeddings, lib = scene
    mplan = metrics.MaskMetricsPlan(H, W, IDS, 0.5, fs.n_frames, DEV)
    render = dict(N_samples=64, N_importance=64, use_disp=False, white_back=False, chunk=chunk, precision="bf16")
    for f in range(fs.n_frames):
        valid = evaluation.valid_mask(fs)
        for k, i in enumerate(IDS):
            out = training.validate_frame(models, embeddings, lib, evaluation.frame_batch(fs, f, [i]), evaluation._NO_LOSS,
                                          keys=("opacity_instance",), **render)
            mplan.accumulate(k, out["opacity_instance_fine"], fs.tensors["labels"][f], valid)
        mplan.finalize(f)
    return mplan.iou.clone(), mplan.opacity_l1.clone()


def test_evaluate_frames_masks_equal_the_per_object_loop():
    from object_nerf_b200 import evaluation
    scene, fs = _scene(True), _frames()
    models, embeddings, lib = scene
    kw = dict(object_ids=IDS, chunk=700)
    off = {k: v.clone() for k, v in evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, depth=True, **kw).items()}
    on = {k: v.clone() for k, v in evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, depth=True, masks=True,
                                                                **kw).items()}
    iou, l1 = _old_mask_loop(scene, fs, 700)
    assert torch.equal(on["iou_objects"].nan_to_num(-1), iou.nan_to_num(-1))
    assert torch.equal(on["opacity_l1_objects"].nan_to_num(-1), l1.nan_to_num(-1))
    assert torch.isfinite(iou).any()
    for k in off:
        assert torch.equal(off[k].nan_to_num(-1), on[k].nan_to_num(-1)), k
