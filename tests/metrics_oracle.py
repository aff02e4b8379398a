"""The image metrics (object_nerf_b200/metrics.py, include/onerf_ext.h: onerf_image_metrics) restated in float64 numpy,
written from the definition: mask, 2-D Gaussian filter with reflect padding, moments, ssim_map, clamp, masked means."""
import numpy as np

C1, C2 = 0.01 ** 2, 0.03 ** 2


def gaussian(window: int) -> np.ndarray:
    """The 2-D kernel outer(g1, g1), g1 normalised to sum 1, sigma 1.5."""
    r = window // 2
    g1 = np.exp(-((np.arange(window) - r) ** 2) / (2 * 1.5 ** 2))
    g1 /= g1.sum()
    return np.outer(g1, g1)


def filter2d(img: np.ndarray, window: int) -> np.ndarray:
    """(H, W) float64 filtered with gaussian(window), reflect padding (numpy's "reflect" = F.pad's), output H x W."""
    r = window // 2
    H, W = img.shape
    P = np.pad(img, r, mode="reflect")
    g = gaussian(window)
    out = np.zeros((H, W))
    for i in range(window):
        for j in range(window):
            out += g[i, j] * P[i:i + H, j:j + W]
    return out


def ssim_map(p: np.ndarray, g: np.ndarray, window: int) -> np.ndarray:
    """Per-pixel ssim_map of one channel (no clamp)."""
    mu_p, mu_g = filter2d(p, window), filter2d(g, window)
    s_pp = filter2d(p * p, window) - mu_p ** 2
    s_gg = filter2d(g * g, window) - mu_g ** 2
    s_pg = filter2d(p * g, window) - mu_p * mu_g
    return ((2 * mu_p * mu_g + C1) * (2 * s_pg + C2)) / ((mu_p ** 2 + mu_g ** 2 + C1) * (s_pp + s_gg + C2))


def column(pred: np.ndarray, gt: np.ndarray, m: np.ndarray, window: int):
    """pred, gt (H, W, 3), m (H, W) bool -> (squared-error sum, clamped ssim_map sum, pixel count, psnr, ssim)."""
    p = np.where(m[..., None], pred.astype(np.float64), 0.0)
    g = np.where(m[..., None], gt.astype(np.float64), 0.0)
    ss = sum(np.clip(ssim_map(p[..., c], g[..., c], window), 0, 1)[m].sum() for c in range(3))
    se = ((p - g) ** 2)[m].sum()
    n = int(m.sum())
    with np.errstate(divide="ignore", invalid="ignore"):
        return se, ss, n, -10 * np.log10(se / (3 * n)) if n else np.nan, ss / (3 * n) if n else np.nan


def metrics(pred_scene, gt, H, W, valid=None, pred_object=None, labels=None, ids=(), window=3):
    """All K+1 columns: (record (K+1, 3) [se, ssim sum, count], psnr (K+1,), ssim (K+1,)), float64."""
    img = lambda a: np.asarray(a, dtype=np.float64).reshape(H, W, 3)
    v = np.ones((H, W), bool) if valid is None else np.asarray(valid).reshape(H, W).astype(bool)
    cols = [column(img(pred_scene), img(gt), v, window)]
    lab = None if labels is None else np.asarray(labels).astype(np.int64).reshape(H, W)
    for i in ids:
        cols.append(column(img(pred_object), img(gt), v & (lab == i), window))
    rec = np.array([c[:3] for c in cols], dtype=np.float64)
    return rec, np.array([c[3] for c in cols]), np.array([c[4] for c in cols])
