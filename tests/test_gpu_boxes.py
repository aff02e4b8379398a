"""rendering.render_boxes (onerf_render_boxes: every object rendered inside its own box) against render_rays /
validate_frame with rays_in_bbox over onerf_camera_rays' box-clipped rays and the column's code on every ray: hit pixels
bit for bit, missed pixels exactly (+0, +0, 1), hit equal to camera_rays' mask.  Both arithmetics, both models, with
and without a fine pass, use_disp, K = 1, 2, 5 and 64 (a repeated id), an odd image with chunks that divide neither
H*W nor K*H*W, boxes that cover nothing, the whole frame or the camera; CUDA-graph replay, two gloo ranks, and
evaluate_frames(boxes=...) against the float64 metric restatements of the per-object validate_frame maps."""
import math
import os
import socket

import numpy as np
import pytest
import torch

from tests import geometry_metrics_oracle as GO
from tests import metrics_oracle as MO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KINDS = ("opacity_instance", "depth_instance", "rgb_instance")
H, W = 37, 53
NEAR, FAR, SCALE = 0.15, 3.0, 1.0


def _scene(use_voxel, dev=DEV):
    from object_nerf_b200 import Embedding, synthetic as S
    models = {"coarse": S.make_model(S.make_weights(31, use_voxel, 8.0, 1.0), use_voxel, dev),
              "fine": S.make_model(S.make_weights(1031, use_voxel, 8.0, 1.0), use_voxel, dev)}
    xyz = (S.GridModule(S.make_grid(seed=5, shape=(42, 42, 22), occupancy=0.6, voxel_size=0.05)).to(dev) if use_voxel
           else Embedding(3, 10))
    return models, {"xyz": xyz, "dir": Embedding(3, 4)}, S.make_code_library(S.make_codes(105)).to(dev)


def _pose(cam):
    cam = np.asarray(cam, np.float64)
    fwd = -cam / np.linalg.norm(cam)
    right = np.cross(fwd, [0, 0, 1.0])
    right /= np.linalg.norm(right)
    return np.concatenate([np.stack([right, np.cross(right, fwd), -fwd], 1), cam[:, None]], 1).astype(np.float32)


C2W = _pose([-1.6, 0.1, 0.15])
FOCAL = 0.5 * W / math.tan(math.radians(30))


def _box(center, size, angle=0.0, scene_center=(0.0, 0.0, 0.0)):
    """A BBoxRayHelper-like box: aligned frame = rotation about z by `angle` then a shift, bounds center +- size / 2."""
    from object_nerf_b200.frames import ObjectBox
    A = np.eye(4)
    A[:3, :3] = [[math.cos(angle), -math.sin(angle), 0], [math.sin(angle), math.cos(angle), 0], [0, 0, 1]]
    A[:3, 3] = [0.03, -0.02, 0.01]
    P = np.eye(4)
    P[:3, 3] = scene_center
    c, h = np.asarray(center, np.float64), np.asarray(size, np.float64) / 2
    return ObjectBox(pose_avg=P, axis_align_mat=A, bbox_bounds=np.array([c - h, c + h]))


BOXES = [_box([0.1, 0.05, 0.0], [0.5, 0.4, 0.5], 0.3), _box([-0.25, -0.2, 0.1], [0.3, 0.3, 0.4], -0.2),
         _box([0.0, 0.0, 0.0], [0.9, 0.9, 0.6]), _box([0.3, 0.3, -0.1], [0.2, 0.6, 0.3], 0.7),
         _box([-0.1, 0.25, 0.05], [0.35, 0.25, 0.5], 1.1)]
NOTHING = _box([6.0, 6.0, 6.0], [0.5, 0.5, 0.5])                         # behind the camera: covers no pixel
EVERYTHING = _box([0.4, 0.0, 0.0], [3.0, 20.0, 20.0])                    # fills the view, camera outside
AROUND_CAMERA = _box([-1.6, 0.1, 0.15], [0.4, 0.4, 0.4])                 # the camera inside: every ray misses


def _reference(scene, box, i, n_importance, use_disp, precision):
    """render_rays over camera_rays(box) with code row i on every ray, is_eval, rays_in_bbox, nothing random."""
    from object_nerf_b200 import ray_utils, render_rays
    models, embeddings, lib = scene
    rays, hit = ray_utils.camera_rays(H, W, FOCAL, torch.from_numpy(C2W), NEAR, FAR, SCALE, box=box, device=DEV,
                                      return_mask=True)
    code = lib.embedding_instance.weight.detach()[i].expand(H * W, 64).contiguous()
    with torch.no_grad():
        out = render_rays(models, embeddings, rays, N_samples=64, N_importance=n_importance, use_disp=use_disp,
                          perturb=0, noise_std=0, embedding_instance=code, is_eval=True, rays_in_bbox=True,
                          precision=precision)
    return out, hit, rays


def _boxes(scene, boxes, ids, n_importance=64, use_disp=False, precision="bf16", chunk=500, keys=None, group=None):
    from object_nerf_b200 import rendering
    models, embeddings, lib = scene
    passes = ("coarse", "fine") if n_importance else ("coarse",)
    keys = keys or tuple(f"{k}_{t}" for t in passes for k in KINDS)
    out = rendering.render_boxes(models if n_importance else {"coarse": models["coarse"]}, embeddings, lib, H, W,
                                 FOCAL, torch.from_numpy(C2W), boxes, ids, N_samples=64, N_importance=n_importance,
                                 use_disp=use_disp, scale_factor=SCALE, near=NEAR, far=FAR, chunk=chunk, keys=keys,
                                 precision=precision, group=group)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in out.items()}


def _check(scene, boxes, ids, n_importance=64, use_disp=False, precision="bf16", chunk=500):
    out = _boxes(scene, boxes, ids, n_importance, use_disp, precision, chunk)
    passes = ("coarse", "fine") if n_importance else ("coarse",)
    K = len(ids)
    assert out["hit"].shape == (H * W, K) and out["hit"].dtype == torch.bool
    for t in passes:
        assert out[f"opacity_instance_{t}"].shape == (H * W, K) and out[f"rgb_instance_{t}"].shape == (H * W, K, 3)
    for k, i in enumerate(ids):
        ref, hit, _ = _reference(scene, boxes[k], i, n_importance, use_disp, precision)
        assert torch.equal(out["hit"][:, k], hit), k
        for t in passes:
            for kind in KINDS:
                got = out[f"{kind}_{t}"][:, k]
                assert torch.equal(got[hit], ref[f"{kind}_{t}"][hit]), (k, i, t, kind)
                miss = got[~hit]
                want = 1.0 if kind == "rgb_instance" else 0.0
                assert (miss == want).all() and not torch.signbit(miss).any(), (k, t, kind)
    return out


@pytest.mark.parametrize("use_voxel", [True, False], ids=["voxel", "plain"])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("K", [1, 2, 5, 64])
def test_columns_equal_one_box_clipped_render_per_object(use_voxel, precision, K):
    """Hit pixels of every column of both passes are the rays_in_bbox render of box k with code ids[k]; 64 boxes
    repeat one id."""
    ids = [3, 9, 0, 63, 17][:K] if K <= 5 else [(7 * k) % 64 for k in range(63)] + [9]
    boxes = [BOXES[k % len(BOXES)] for k in range(K)]
    out = _check(_scene(use_voxel), boxes, ids, precision=precision, chunk=500)
    assert out["hit"].any() and not out["hit"].all()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("use_voxel", [True, False], ids=["voxel", "plain"])
def test_coarse_only_and_use_disp(use_voxel, precision):
    """Without a fine pass, and with use_disp (whose missed rows have no finite depth: their maps are still (+0, +0, 1))."""
    scene = _scene(use_voxel)
    _check(scene, BOXES[:3], [4, 11, 4], n_importance=0, use_disp=True, precision=precision, chunk=333)
    _check(scene, BOXES[:2], [4, 11], n_importance=64, use_disp=True, precision=precision, chunk=777)


def test_boxes_that_cover_nothing_everything_or_the_camera():
    out = _check(_scene(True), [NOTHING, EVERYTHING, AROUND_CAMERA, BOXES[0]], [5, 6, 7, 8], chunk=1000)
    assert not out["hit"][:, 0].any() and out["hit"][:, 1].all() and not out["hit"][:, 2].any()


def test_last_pass_equals_validate_frame():
    """The fine maps are validate_frame's (rays_in_bbox, box-clipped rays, the code on every pixel) at hit pixels."""
    from object_nerf_b200 import training
    from object_nerf_b200.evaluation import _NO_LOSS
    scene = _scene(True)
    models, embeddings, lib = scene
    ids = [2, 13]
    out = _boxes(scene, BOXES[:2], ids, chunk=4096)
    for k, i in enumerate(ids):
        _, hit, rays = _reference(scene, BOXES[k], i, 64, False, "bf16")
        batch = {"rays": rays, "rgbs": torch.zeros(H * W, 3, device=DEV), "depths": torch.zeros(H * W, device=DEV),
                 "valid_mask": torch.ones(H * W, dtype=torch.uint8, device=DEV),
                 "instance_ids": torch.full((H * W,), i, dtype=torch.int64, device=DEV)}
        ref = training.validate_frame(models, embeddings, lib, batch, _NO_LOSS, N_samples=64, N_importance=64,
                                      use_disp=False, white_back=False, rays_in_bbox=True, keys=KINDS, chunk=700)
        for kind in KINDS:
            assert torch.equal(out[f"{kind}_fine"][:, k][hit], ref[f"{kind}_fine"][hit]), (k, kind)


def test_maps_asked_for_alone_and_chunks_give_the_same_bits():
    scene, ids = _scene(True), [7, 2, 7]
    full = _boxes(scene, BOXES[:3], ids, chunk=500)
    for keys, chunk in ((("opacity_instance",), 500), (("depth_instance_coarse", "rgb_instance"), 1), (None, 5883)):
        part = _boxes(scene, BOXES[:3], ids, chunk=chunk, keys=keys)
        for k, v in part.items():
            assert torch.equal(v, full[k]), (keys, chunk, k)


def test_graph_replay_gives_the_eager_bits():
    """Capture one call, replay it after the code table changed in place: bit for bit the eager call."""
    from object_nerf_b200 import rendering
    scene = _scene(True)
    models, embeddings, lib = scene
    ids, kw = [6, 2], dict(N_samples=64, N_importance=64, use_disp=False, scale_factor=SCALE, near=NEAR, far=FAR,
                           chunk=700, keys=KINDS)
    args = (models, embeddings, lib, H, W, FOCAL, torch.from_numpy(C2W), BOXES[:2], ids)
    rendering.render_boxes(*args, **kw)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            held = rendering.render_boxes(*args, **kw)
    with torch.no_grad():
        lib.embedding_instance.weight.mul_(0.5)
    graph.replay()
    torch.cuda.synchronize()
    replayed = {k: v.clone() for k, v in held.items()}
    eager = _boxes(scene, BOXES[:2], ids, chunk=700, keys=KINDS)
    assert sorted(replayed) == sorted(eager)
    for k in eager:
        assert torch.equal(replayed[k], eager[k]), k


def _shard_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        scene = _scene(True)
        single = _boxes(scene, BOXES[:3], [5, 1, 5], chunk=600)
        shared = _boxes(scene, BOXES[:3], [5, 1, 5], chunk=600, group=dist.group.WORLD)
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
# evaluate_frames(boxes=...)
# ------------------------------------------------------------------------------------------------
IDS = (3, 5, 9)
CONF = {"model": {"N_samples": 64, "N_importance": 64, "use_disp": False}}


def _frames(n_frames=2):
    from object_nerf_b200 import frames
    rng = np.random.default_rng(0)
    poses = [_pose(np.array([-1.6, 0.1, 0.15]) + rng.normal(size=3) * 0.1) for _ in range(n_frames)]
    labels = rng.choice(np.array([0, *IDS], np.uint16), (n_frames, H, W))
    depths = rng.uniform(0.5, 3.0, (n_frames, H, W)).astype(np.float32)
    return frames.FrameSet(np.stack(poses), rng.integers(0, 256, (n_frames, H, W, 3), dtype=np.uint8), depths, labels,
                           focal=FOCAL, near=NEAR, far=FAR, scale_factor=SCALE, instance_ids=(IDS[0],), border=3,
                           device=DEV)


def test_evaluate_frames_in_boxes_is_the_restatement_of_the_per_object_renders():
    """Colour, depth and mask scores of every object over the valid pixels labelled with it whose ray hits its box,
    computed from one validate_frame(rays_in_bbox) per object over its box-clipped rays; the scene columns are those
    of the run without boxes."""
    from object_nerf_b200 import evaluation, ray_utils, training
    scene, fs = _scene(True), _frames()
    models, embeddings, lib = scene
    boxes = BOXES[:3]
    kw = dict(object_ids=IDS, chunk=900, depth=True, masks=True)
    plain = {k: v.clone() for k, v in evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, **kw).items()}
    res = {k: v.cpu().numpy() for k, v in
           evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, boxes=boxes, **kw).items()}
    for k in ("psnr", "ssim", "depth_metrics"):
        assert np.array_equal(res[k], plain[k].cpu().numpy(), equal_nan=True), k
    P, S, D, M = [], [], [], []
    valid = evaluation.valid_mask(fs).cpu().numpy()
    for f in range(fs.n_frames):
        batch = evaluation.frame_batch(fs, f, IDS)
        lab = fs.tensors["labels"][f].cpu().numpy().view(np.uint16).astype(np.int64)
        obj_rgb, obj_depth = np.ones((H * W, 3), np.float32), np.zeros(H * W, np.float32)
        keep = np.zeros(H * W, bool)
        opac = []
        for k, i in enumerate(IDS):
            rays, hit = ray_utils.camera_rays(H, W, fs.focal, torch.from_numpy(fs.poses_host[f].reshape(3, 4)), NEAR, FAR,
                                              SCALE, box=boxes[k], device=DEV, return_mask=True)
            b = dict(batch, rays=rays, instance_ids=torch.full((H * W,), i, dtype=torch.int64, device=DEV))
            out = training.validate_frame(models, embeddings, lib, b, evaluation._NO_LOSS, N_samples=64,
                                          N_importance=64, use_disp=False, white_back=False, rays_in_bbox=True,
                                          keys=KINDS, chunk=900)
            hit = hit.cpu().numpy()
            m = lab == i
            obj_rgb[m] = out["rgb_instance_fine"].cpu().numpy()[m]
            obj_depth[m] = out["depth_instance_fine"].cpu().numpy()[m]
            keep |= m & hit
            opac.append(np.where(hit, out["opacity_instance_fine"].cpu().numpy(), np.float32(0)))
        lab_box = np.where(keep, lab, 1)                  # 1 is none of IDS
        assert (~keep & np.isin(lab, IDS)).any() and keep.any()
        _, psnr, ssim = MO.metrics(np.zeros((H * W, 3), np.float32), batch["rgbs"].cpu().numpy(), H, W, valid, obj_rgb,
                                   lab_box, IDS, 3)
        _, dm = GO.depth_metrics(np.zeros(H * W, np.float32), fs.tensors["depths"][f].cpu().numpy(), valid, obj_depth,
                                 lab_box, IDS, SCALE)
        iou, l1 = GO.mask_outputs([GO.mask_sums(opac[k], lab_box, i, valid) for k, i in enumerate(IDS)])
        P.append(psnr[1:]), S.append(ssim[1:]), D.append(dm[1:]), M.append((iou, l1))
    for got, want in ((res["psnr_objects"], np.array(P)), (res["ssim_objects"], np.array(S)),
                      (res["depth_metrics_objects"], np.array(D)), (res["iou_objects"], np.array([m[0] for m in M])),
                      (res["opacity_l1_objects"], np.array([m[1] for m in M]))):
        assert np.array_equal(np.isnan(got), np.isnan(want))
        fin = np.isfinite(want)
        assert fin.any() and np.abs(got[fin] - want[fin]).max() <= 1e-5 * max(1, np.abs(want[fin]).max())
