"""onerf_depth_metrics and onerf_mask_metrics against the float64 restatement (tests/geometry_metrics_oracle.py): counts
exactly, the other fp64 record sums within 1e-9 relative, the float32 outputs as the float32 rounding of the
restatement; on random frames from 1x1 to 641x479 and on planted edges (no ground truth, predictions of 0, negative
and above d_max, ratios at 1.25^i, labels 0 and 65535, 64 ids, empty columns, NaN predictions, opacities at the
threshold); finalize zeroing the record; CUDA-graph replay; and evaluation.evaluate_frames(depth=, masks=) against the
restatement of validate_frame's own maps, with the colour scores unchanged and two gloo ranks equal to one process."""
import math
import os
import socket

import numpy as np
import pytest
import torch

from tests import geometry_metrics_oracle as GO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RANGE = (0.05, 3.0)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV) if a is not None else None


def _depth_frame(seed, H, W, ids, other=(0, 65535)):
    """Random depths in units where scale 2 gives metres, with planted edges at the first pixels: no ground truth,
    predictions of 0, negative, above d_max and below d_min, and ratios exactly 1.25, 1.25^2, 1.25^3 both ways."""
    rng = np.random.default_rng(seed)
    n = H * W
    gt = rng.uniform(0.02, 1.6, n).astype(np.float32)
    gt[rng.random(n) < 0.1] = 0
    pred, obj = ((gt * rng.uniform(0.5, 1.8, n)).astype(np.float32) for _ in range(2))
    plant = [(0.5, 0.0), (0.5, -1.0), (0.5, 4.0), (0.5, 0.01), (0.0, 1.0), (0.5, 0.625), (0.5, 0.78125),
             (0.5, 0.9765625), (0.625, 0.5), (0.78125, 0.5), (0.9765625, 0.5), (0.5, 0.5)]
    for i, (g, p) in enumerate(plant[:n]):
        gt[i], pred[i], obj[(i + 3) % n] = g, p, p
    valid = rng.random(n) > 0.15
    valid[:min(n, len(plant))] = True
    labels = rng.choice(list(ids) + list(other), size=n).astype(np.uint16)
    return pred, obj, gt, valid, labels


def _run_depth(pred, obj, gt, valid, labels, H, W, ids, scale=2.0, depth_range=RANGE):
    from object_nerf_b200 import metrics
    plan = metrics.DepthMetricsPlan(H, W, ids, scale, depth_range, 2, DEV)
    plan.accumulate(_t(pred), _t(gt), _t(valid), _t(obj) if ids else None,
                    _t(labels.view(np.int16)) if ids else None)
    torch.cuda.synchronize()
    rec = plan.record.cpu().numpy().copy()
    plan.finalize(1)
    torch.cuda.synchronize()
    return rec, plan.out[1].cpu().numpy(), plan.record.cpu().numpy()


def _close32(got, want):
    """float32 outputs: the same NaNs, and within 2 float32 ulps of the float64 value elsewhere."""
    assert np.array_equal(np.isnan(got), np.isnan(want))
    fin = np.isfinite(want)
    w32 = want[fin].astype(np.float32)
    assert (np.abs(got[fin] - w32) <= 2 * np.spacing(np.abs(w32))).all(), np.abs(got[fin] - w32).max()


def _check_depth(got, want):
    rec, out, after = got
    wrec, wout = want
    assert np.array_equal(rec[:, [0, 5, 6, 7]], wrec[:, [0, 5, 6, 7]], equal_nan=True)        # counts are exact
    assert np.allclose(rec[:, 1:5], wrec[:, 1:5], rtol=1e-9, atol=0, equal_nan=True)
    _close32(out, wout)
    assert not after.any()                                                                     # finalize zeroes it


SIZES = [(1, 1), (1, 1000), (999, 1), (17, 33), (480, 640), (479, 641)]


@pytest.mark.parametrize("H,W", SIZES)
def test_depth_kernel_matches_float64(H, W):
    ids = [3, 9, 65535, 0, 11]                        # 11 labels no pixel: an empty column
    pred, obj, gt, valid, labels = _depth_frame(H * 7 + W, H, W, ids[:4], other=(5, 70))
    want = GO.depth_metrics(pred, gt, valid, obj, labels, ids, 2.0, RANGE)
    assert want[0][5, 0] == 0 and np.isnan(want[1][5]).all()
    _check_depth(_run_depth(pred, obj, gt, valid, labels, H, W, ids), want)


def test_planted_edges_are_where_they_should_be():
    """The planted pixels of a 1 x 12 frame: gt 0 excluded, clamps to d_min / d_max, the ratio boundaries exact."""
    ids = [4]
    pred, obj, gt, valid, labels = _depth_frame(1, 1, 12, ids)
    labels[:] = 4
    rec, out = GO.depth_metrics(pred, gt, valid, obj, labels, ids, 2.0, RANGE)
    assert rec[0, 0] == 11                                       # the one planted pixel without ground truth is out
    got = _run_depth(pred, obj, gt, valid, labels, 1, 12, ids)
    _check_depth(got, (rec, out))
    # g = 1 with d = 0.02 -> 0.05, 8 -> 3; the last 7: ratios 1.25, 1.5625, 1.953125 both ways and 1
    assert list(rec[0, 5:]) == [1, 3, 5] and gt[3] * 2 == 1 and pred[3] * 2 < RANGE[0] and pred[2] * 2 > RANGE[1]


@pytest.mark.parametrize("K", [1, 64])
def test_depth_column_counts(K):
    H, W = 61, 47
    ids = [i * 1000 for i in range(K - 1)] + [65535]            # 0 and 65535 among them
    pred, obj, gt, valid, labels = _depth_frame(K, H, W, ids, other=(7, 65534))
    want = GO.depth_metrics(pred, gt, valid, obj, labels, ids, 2.0, RANGE)
    assert (want[0][:, 0] > 0).all()
    _check_depth(_run_depth(pred, obj, gt, valid, labels, H, W, ids), want)


def test_depth_without_objects_and_without_valid():
    H, W = 33, 65
    pred, _, gt, _, _ = _depth_frame(3, H, W, [1])
    want = GO.depth_metrics(pred, gt, None, scale=0.75, depth_range=(1e-3, 10.0))
    _check_depth(_run_depth(pred, None, gt, None, None, H, W, [], 0.75, (1e-3, 10.0)), want)


def test_nan_prediction_makes_its_column_nan():
    H, W = 40, 40
    ids = [1, 2]
    pred, obj, gt, valid, labels = _depth_frame(4, H, W, ids, other=())
    gt[:] = 1.0
    idx = int(np.nonzero((labels == 2) & valid)[0][0])
    obj[idx] = np.nan                                            # object 2's column only
    want = GO.depth_metrics(pred, gt, valid, obj, labels, ids, 2.0, RANGE)
    assert np.isnan(want[1][2]).all() and np.isfinite(want[1][:2]).all()
    _check_depth(_run_depth(pred, obj, gt, valid, labels, H, W, ids), want)


def test_depth_metrics_function():
    from object_nerf_b200 import metrics
    H, W = 20, 30
    ids = [5, 6]
    pred, obj, gt, valid, labels = _depth_frame(8, H, W, ids)
    got = metrics.depth_metrics(_t(pred), _t(gt), H, W, _t(valid), _t(obj), _t(labels.astype(np.int32)), ids,
                                scale=2.0, depth_range=RANGE)
    assert got.shape == (3, 7) and got.dtype == torch.float32
    _close32(got.cpu().numpy(), GO.depth_metrics(pred, gt, valid, obj, labels, ids, 2.0, RANGE)[1])


# ---------------------------------------------------------------------------------------------------------------------
# masks
# ---------------------------------------------------------------------------------------------------------------------
def _mask_frame(seed, n, ids, tau):
    rng = np.random.default_rng(seed)
    o = rng.random(n).astype(np.float32)
    o[rng.random(n) < 0.1] = np.float32(tau)                     # exactly at the threshold: covered
    o[rng.random(n) < 0.05] = np.nextafter(np.float32(tau), np.float32(0))
    labels = rng.choice(list(ids) + [0, 65535, 12], size=n).astype(np.uint16)
    valid = rng.random(n) > 0.2
    return o, labels, valid


@pytest.mark.parametrize("H,W", SIZES)
def test_mask_kernel_matches_float64(H, W):
    from object_nerf_b200 import metrics
    ids, tau = [4, 0, 65535, 99], 0.375                          # 99 labels no pixel
    plan = metrics.MaskMetricsPlan(H, W, ids, tau, 3, DEV)
    maps = [_mask_frame(H + W + k, H * W, ids[:3], tau) for k in range(len(ids))]
    for k, (o, labels, valid) in enumerate(maps):
        plan.accumulate(k, _t(o), _t(labels.view(np.int16)), _t(valid))
    torch.cuda.synchronize()
    rec = plan.record.cpu().numpy().copy()
    plan.finalize(2)
    want = np.stack([GO.mask_sums(o, labels, i, valid, tau) for i, (o, labels, valid) in zip(ids, maps)])
    assert np.array_equal(rec[:, [0, 1, 3]], want[:, [0, 1, 3]])
    assert np.allclose(rec[:, 2], want[:, 2], rtol=1e-9, atol=0)
    iou, l1 = GO.mask_outputs(want)
    _close32(plan.iou[2].cpu().numpy(), iou)
    _close32(plan.opacity_l1[2].cpu().numpy(), l1)
    assert not plan.record.any()


def test_mask_metrics_function_and_threshold():
    """Opacities exactly at tau count as covered; one below does not; no valid mask means every pixel."""
    from object_nerf_b200 import metrics
    o = torch.tensor([0.5, np.nextafter(np.float32(0.5), np.float32(0)), 1.0, 0.0], device=DEV)
    lab = torch.tensor([3, 3, 0, 3], dtype=torch.int64, device=DEV)
    iou, l1 = metrics.mask_metrics(o, lab, 3)
    assert iou.item() == 0.25                                    # P = {0, 2}, G = {0, 1, 3}
    want = (0.5 + (1 - float(np.nextafter(np.float32(0.5), np.float32(0)))) + 1 + 1) / 4
    assert abs(l1.item() - want) <= 1e-7
    iou, l1 = metrics.mask_metrics(o, lab, 3, valid=torch.tensor([1, 0, 1, 0], dtype=torch.bool, device=DEV),
                                   threshold=0.75)
    assert iou.item() == 0.0 and abs(l1.item() - 0.75) <= 1e-7
    iou, l1 = metrics.mask_metrics(torch.zeros(4, device=DEV), lab, 8)
    assert math.isnan(iou.item()) and l1.item() == 0.0


# ---------------------------------------------------------------------------------------------------------------------
# graph replay
# ---------------------------------------------------------------------------------------------------------------------
def test_graph_replay_equals_the_eager_call():
    from object_nerf_b200 import metrics
    H, W, ids = 120, 90, [2, 5]
    pred, obj, gt, valid, labels = _depth_frame(7, H, W, ids)
    o = np.random.default_rng(8).random(H * W).astype(np.float32)
    P, O, G, V, L, OP = _t(pred), _t(obj), _t(gt), _t(valid).view(torch.uint8), _t(labels.view(np.int16)), _t(o)

    def run(dplan, mplan, slot):
        dplan.accumulate(P, G, V, O, L)
        dplan.finalize(slot)
        for k in range(2):
            mplan.accumulate(k, OP, L, V)
        mplan.finalize(slot)

    eager = (metrics.DepthMetricsPlan(H, W, ids, 2.0, RANGE, 3, DEV), metrics.MaskMetricsPlan(H, W, ids, 0.5, 3, DEV))
    run(*eager, 2)
    plans = (metrics.DepthMetricsPlan(H, W, ids, 2.0, RANGE, 3, DEV), metrics.MaskMetricsPlan(H, W, ids, 0.5, 3, DEV))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(*plans, 0)                                           # warm-up
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run(*plans, 2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(plans[0].out[2], eager[0].out[2])
    assert torch.equal(plans[1].iou[2], eager[1].iou[2]) and torch.equal(plans[1].opacity_l1[2], eager[1].opacity_l1[2])
    O.mul_(0.5)                                                  # a replay scores what the buffers hold by then
    OP.mul_(0.5)
    g.replay()
    run(*eager, 1)
    torch.cuda.synchronize()
    assert torch.equal(plans[0].out[2], eager[0].out[1]) and not torch.equal(eager[0].out[1], eager[0].out[2])
    assert torch.equal(plans[1].iou[2], eager[1].iou[1]) and torch.equal(plans[1].opacity_l1[2], eager[1].opacity_l1[1])
    assert not plans[0].record.any() and not plans[1].record.any()


def test_refusals_through_python():
    from object_nerf_b200 import metrics
    x = torch.ones(16, device=DEV)
    with pytest.raises(RuntimeError, match="d_min"):
        metrics.depth_metrics(x, x, 4, 4, depth_range=(0.0, 1.0))
    with pytest.raises(RuntimeError, match="scale"):
        metrics.depth_metrics(x, x, 4, 4, scale=math.nan)
    with pytest.raises(RuntimeError, match="distinct"):
        metrics.depth_metrics(x, x, 4, 4, pred_object=x, labels=torch.zeros(16, dtype=torch.int16, device=DEV),
                              ids=[1, 1])
    with pytest.raises(RuntimeError, match="threshold"):
        metrics.mask_metrics(x, torch.zeros(16, dtype=torch.int16, device=DEV), 1, threshold=math.inf)


# ---------------------------------------------------------------------------------------------------------------------
# evaluate_frames
# ---------------------------------------------------------------------------------------------------------------------
H, W, F = 48, 64, 3
IDS = (3, 5, 12)                 # 12 is absent from frame 1
CONF = {"model": {"N_samples": 32, "N_importance": 32, "use_disp": False}}
SCALE = 1.0


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
    labels[:, :H // 2, :W // 3] = 5
    labels[1][labels[1] == 12] = 7
    depths = rng.uniform(0.8, 2.6, size=(F, H, W)).astype(np.float32)
    depths[rng.random((F, H, W)) < 0.1] = 0
    fs = frames.FrameSet(np.stack(poses).astype(np.float32), rng.integers(0, 256, size=(F, H, W, 3), dtype=np.uint8),
                         depths, labels, focal=focal, near=0.15, far=3.0, scale_factor=SCALE, instance_ids=(3,),
                         border=4, device=dev)
    return models, {"xyz": emb, "dir": Embedding(3, 4)}, lib, fs


@pytest.fixture(scope="module")
def scene():
    return _scene()


def _maps(scene, batch, keys):
    from object_nerf_b200 import training
    from object_nerf_b200.evaluation import _NO_LOSS
    models, embeddings, lib, _ = scene
    out = training.validate_frame(models, embeddings, lib, batch, _NO_LOSS, N_samples=32, N_importance=32,
                                  use_disp=False, white_back=False, keys=keys, chunk=1000)
    return {k: out[f"{k}_fine"].cpu().numpy().copy() for k in keys}


def test_evaluate_frames_depth_and_masks_are_the_restatement_of_the_maps(scene):
    from object_nerf_b200 import evaluation
    models, embeddings, lib, fs = scene
    plain = evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, object_ids=IDS, chunk=1000)
    res = evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, object_ids=IDS, chunk=1000, depth=True,
                                     masks=True, mask_threshold=0.25)
    plain = {k: v.cpu().numpy() for k, v in plain.items()}
    res = {k: v.cpu().numpy() for k, v in res.items()}
    for k in plain:                                              # the colour scores do not move
        assert np.array_equal(plain[k], res[k], equal_nan=True), k
    assert res["depth_metrics"].shape == (F, 7) and res["depth_metrics_objects"].shape == (F, len(IDS), 7)
    assert res["iou_objects"].shape == (F, len(IDS)) and res["opacity_l1_objects"].shape == (F, len(IDS))
    D, IOU, L1 = [], [], []
    for f in range(F):
        batch = evaluation.frame_batch(fs, f, IDS)
        maps = _maps(scene, batch, ("rgb", "rgb_instance", "depth", "depth_instance"))
        valid, labels = batch["valid_mask"].cpu().numpy(), fs.tensors["labels"][f].cpu().numpy().view(np.uint16)
        gt = fs.tensors["depths"][f].cpu().numpy()
        D.append(GO.depth_metrics(maps["depth"], gt, valid, maps["depth_instance"], labels, IDS, SCALE)[1])
        sums = np.stack([GO.mask_sums(_maps(scene, evaluation.frame_batch(fs, f, [i]), ("opacity_instance",))
                                      ["opacity_instance"], labels, i, valid, 0.25) for i in IDS])
        iou, l1 = GO.mask_outputs(sums)
        IOU.append(iou)
        L1.append(l1)
    D, IOU, L1 = np.array(D), np.array(IOU), np.array(L1)
    assert np.isnan(D[1, 3]).all() and np.isfinite(D[:, :3]).all()
    assert np.isnan(IOU[1, 2]) or IOU[1, 2] == 0                 # object 12 has no pixel in frame 1
    _close32(res["depth_metrics"], D[:, 0])
    _close32(res["depth_metrics_objects"], D[:, 1:])
    _close32(res["iou_objects"], IOU)
    _close32(res["opacity_l1_objects"], L1)
    assert np.allclose(res["mean_depth_metrics"], D[:, 0].mean(0), rtol=1e-6, atol=0)
    assert np.allclose(res["mean_depth_metrics_objects"], np.nanmean(D[:, 1:], 0), rtol=1e-6, atol=0)
    assert np.allclose(res["mean_iou_objects"], np.nanmean(IOU, 0), rtol=1e-6, atol=1e-7)
    assert np.allclose(res["mean_opacity_l1_objects"], np.nanmean(L1, 0), rtol=1e-6, atol=0)
    # the scene column alone, with depth
    alone = evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, chunk=1000, depth=True, masks=True)
    assert alone["depth_metrics_objects"].shape == (F, 0, 7) and alone["iou_objects"].shape == (F, 0)
    _close32(alone["depth_metrics"].cpu().numpy(), D[:, 0])


def _worker(rank, world, port, ret):
    import torch.distributed as dist
    from object_nerf_b200 import evaluation
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        models, embeddings, lib, fs = _scene()
        kw = dict(object_ids=IDS, chunk=700, depth=True, masks=True)
        single = evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, **kw)
        shared = evaluation.evaluate_frames(models, embeddings, lib, fs, CONF, group=dist.group.WORLD, **kw)
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
        assert "depth_metrics" in single and "iou_objects" in single
        for k in single:
            assert np.array_equal(single[k], shared[k], equal_nan=True), (rank, k)
            assert np.array_equal(ret[0][1][k], shared[k], equal_nan=True), (rank, k)
