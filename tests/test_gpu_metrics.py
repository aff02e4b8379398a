"""onerf_image_metrics against the float64 restatement (tests/metrics_oracle.py): the fp64 record within 1e-9 (SSIM) and
1e-9 dB (PSNR), the float32 outputs as the float32 rounding of the restatement, at every frame size from 2x2 to
641x479, windows 1 to 11, masks on corners, edges and single pixels, empty masks, K = 0, 1 and 64; metrics.psnr /
metrics.ssim; and CUDA-graph replay."""
import math

import numpy as np
import pytest
import torch

from tests import metrics_oracle as MO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _frame(seed, H, W, ids):
    """Random images, a random valid mask with its corners and edges set, and labels (uint16) that give ids[0] and
    ids[1] random pixels, ids[-2] the four corners, ids[-1] one pixel and ids[2] none."""
    rng = np.random.default_rng(seed)
    pred, obj, gt = (rng.random((H * W, 3), dtype=np.float32) for _ in range(3))
    valid = rng.random((H, W)) > 0.15
    valid[0, :] = valid[-1, :] = valid[:, 0] = valid[:, -1] = True
    labels = rng.choice([ids[0], ids[1], 0], size=(H, W))
    labels[H // 2, W // 2] = ids[-1]
    labels[0, 0] = labels[-1, -1] = labels[0, -1] = labels[-1, 0] = ids[-2]
    return pred, obj, gt, valid.reshape(-1), labels.reshape(-1).astype(np.uint16)


def _run(pred, obj, gt, valid, labels, H, W, ids, window):
    from object_nerf_b200 import metrics
    plan = metrics.MetricsPlan(H, W, ids, window, 2, DEV)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV) if a is not None else None
    lab = t(labels.view(np.int16)) if labels is not None else None
    plan.accumulate(t(pred), t(gt), t(valid), t(obj) if ids else None, lab)
    torch.cuda.synchronize()
    rec = plan.record.cpu().numpy().copy()
    plan.finalize(1)
    torch.cuda.synchronize()
    return rec, plan.psnr[1].cpu().numpy(), plan.ssim[1].cpu().numpy(), plan.record.cpu().numpy()


def _check(got, want):
    rec, psnr32, ssim32, after = got
    wrec, wpsnr, wssim = want
    assert np.array_equal(rec[:, 2], wrec[:, 2])                          # pixel counts are exact
    n = 3 * rec[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        psnr, ssim = -10 * np.log10(rec[:, 0] / n), rec[:, 1] / n
    for a, b, tol in ((psnr, wpsnr, 1e-9), (ssim, wssim, 1e-9)):
        assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isinf(a), np.isinf(b))
        fin = np.isfinite(b)
        assert np.abs(a[fin] - b[fin]).max(initial=0) <= tol, np.abs(a[fin] - b[fin]).max()
    for a, b in ((psnr32, wpsnr), (ssim32, wssim)):
        fin = np.isfinite(b)
        assert np.array_equal(np.isnan(a), np.isnan(b))
        assert np.abs(a[fin] - b[fin].astype(np.float32)).max(initial=0) <= 2 * np.spacing(np.float32(np.abs(b[fin]).max(initial=1)))
    assert not after.any()                                                 # finalize zeroes the record


SIZES = [(2, 2), (3, 2), (5, 7), (16, 32), (17, 33), (48, 31), (641, 479), (640, 480)]


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("window", [1, 3, 5, 11])
def test_kernel_matches_float64(H, W, window):
    if H <= window // 2 or W <= window // 2:
        pytest.skip("reflect padding is undefined (refused: tests/test_metrics_cpu.py)")
    ids = [3, 9, 4, 7, 1]
    pred, obj, gt, valid, labels = _frame(H * 1000 + W + window, H, W, ids)
    want = MO.metrics(pred, gt, H, W, valid, obj, labels, ids, window)
    assert want[0][3, 2] == 0 and np.isnan(want[1][3]) and np.isnan(want[2][3])      # the empty column
    _check(_run(pred, obj, gt, valid, labels, H, W, ids, window), want)


@pytest.mark.parametrize("K", [0, 1, 64])
def test_column_counts(K):
    H, W = 61, 47
    ids = list(range(K))
    rng = np.random.default_rng(K)
    pred, obj, gt = (rng.random((H * W, 3), dtype=np.float32) for _ in range(3))
    valid = (rng.random(H * W) > 0.1)
    labels = rng.integers(0, 70, size=H * W).astype(np.uint16) if K else None
    got = _run(pred, obj, gt, valid, labels, H, W, ids, 3)
    _check(got, MO.metrics(pred, gt, H, W, valid, obj, labels, ids, 3))


def test_identical_and_offset_images_on_the_device():
    from object_nerf_b200 import metrics
    rng = np.random.default_rng(5)
    g = torch.from_numpy(rng.random((40 * 30, 3), dtype=np.float32)).to(DEV)
    psnr, ssim = metrics.image_metrics(g, g, 40, 30, window=5)
    assert psnr.item() == math.inf and abs(ssim.item() - 1) < 1e-6
    a = torch.full((40 * 30, 3), 0.25, device=DEV)
    psnr, ssim = metrics.image_metrics(a + 0.125, a, 40, 30, window=3)
    assert abs(psnr.item() + 10 * math.log10(0.125 ** 2)) < 1e-5
    want = (2 * 0.25 * 0.375 + MO.C1) / (0.25 ** 2 + 0.375 ** 2 + MO.C1)
    assert abs(ssim.item() - want) < 1e-6


def test_reference_signatures():
    """metrics.ssim on (1, 3, H, W) and metrics.psnr with and without a mask against the restatement."""
    from object_nerf_b200 import metrics
    rng = np.random.default_rng(6)
    H, W = 37, 53
    g = rng.random((1, 3, H, W), dtype=np.float32)
    p = np.clip(g + 0.1 * rng.standard_normal(g.shape).astype(np.float32), 0, 1)
    hwc = lambda a: a[0].transpose(1, 2, 0).reshape(-1, 3)
    _, _, want = MO.metrics(hwc(p), hwc(g), H, W, window=3)
    got = metrics.ssim(torch.from_numpy(p).to(DEV), torch.from_numpy(g).to(DEV))
    assert got.shape == () and abs(got.item() - want[0]) <= 1e-6
    mask = rng.random((H * W,)) > 0.3
    for m in (None, mask):
        _, want, _ = MO.metrics(hwc(p), hwc(g), 1, H * W, m, window=1)
        got = metrics.psnr(torch.from_numpy(hwc(p)).to(DEV), torch.from_numpy(hwc(g)).to(DEV),
                           None if m is None else torch.from_numpy(m).to(DEV))
        assert abs(got.item() - want[0]) <= 1e-5
    empty = torch.zeros(H * W, dtype=torch.bool, device=DEV)
    assert math.isnan(metrics.psnr(torch.zeros(H * W, 3, device=DEV), torch.zeros(H * W, 3, device=DEV), empty).item())


def test_graph_replay_equals_the_eager_call():
    from object_nerf_b200 import metrics
    H, W, ids = 120, 90, [2, 5]
    pred, obj, gt, valid, labels = _frame(7, H, W, [2, 5, 6, 8])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    P, O, G, V, L = t(pred), t(obj), t(gt), t(valid).view(torch.uint8), t(labels.view(np.int16))
    eager = metrics.MetricsPlan(H, W, ids, 5, 3, DEV)
    eager.accumulate(P, G, V, O, L)
    eager.finalize(2)
    plan = metrics.MetricsPlan(H, W, ids, 5, 3, DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.accumulate(P, G, V, O, L)        # warm-up
        plan.finalize(0)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.accumulate(P, G, V, O, L)
        plan.finalize(2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(plan.psnr[2], eager.psnr[2]) and torch.equal(plan.ssim[2], eager.ssim[2])
    O.mul_(0.5)                                   # a replay scores what the buffers hold by then
    g.replay()
    eager.accumulate(P, G, V, O, L)
    eager.finalize(1)
    torch.cuda.synchronize()
    assert torch.equal(plan.psnr[2], eager.psnr[1]) and torch.equal(plan.ssim[2], eager.ssim[1])
    assert not torch.equal(eager.psnr[1], eager.psnr[2])


def test_refusals_through_python():
    from object_nerf_b200 import metrics
    x = torch.zeros(4 * 4, 3, device=DEV)
    with pytest.raises(RuntimeError, match="window"):
        metrics.image_metrics(x, x, 4, 4, window=4)
    with pytest.raises(RuntimeError, match="exceed window / 2"):
        metrics.image_metrics(x, x, 4, 4, window=11)
    with pytest.raises(RuntimeError, match="object columns need"):
        metrics.image_metrics(x, x, 4, 4, ids=[1])
