"""The depth and mask metrics (object_nerf_b200/metrics.py, include/onerf_ext.h: onerf_depth_metrics,
onerf_mask_metrics) restated in float64 numpy, written from the definition: column masks, scaled and clamped depths,
per-column sums, then the ratios."""
import numpy as np

DEPTH_METRICS = ("abs_rel", "sq_rel", "rmse", "rmse_log", "delta1", "delta2", "delta3")


def depth_sums(pred, gt, m, scale, d_min, d_max) -> np.ndarray:
    """The eight sums of one column: pred, gt float32 arrays, m bool -> [n, sum |e| / g, sum e^2 / g, sum e^2,
    sum (ln d - ln g)^2, count_1, count_2, count_3] (a NaN ratio makes the counts NaN)."""
    g = gt[m].astype(np.float64) * scale
    d = pred[m].astype(np.float64) * scale
    d = np.where(np.isnan(d), d, np.clip(d, d_min, d_max))
    e = d - g
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.maximum(d / g, g / d)
        counts = [np.where(np.isnan(r), np.nan, (r < 1.25 ** i).astype(np.float64)).sum() for i in (1, 2, 3)]
        return np.array([m.sum(), (np.abs(e) / g).sum(), (e * e / g).sum(), (e * e).sum(),
                         ((np.log(d) - np.log(g)) ** 2).sum(), *counts], dtype=np.float64)


def depth_outputs(rec) -> np.ndarray:
    """(C, 8) sums -> (C, 7) metrics in DEPTH_METRICS order (NaN for an empty column)."""
    rec = np.asarray(rec, dtype=np.float64)
    n = rec[:, 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.stack([rec[:, 1] / n, rec[:, 2] / n, np.sqrt(rec[:, 3] / n), np.sqrt(rec[:, 4] / n),
                         rec[:, 5] / n, rec[:, 6] / n, rec[:, 7] / n], 1)


def depth_metrics(pred_scene, gt, valid=None, pred_object=None, labels=None, ids=(), scale=1.0,
                  depth_range=(1e-3, 10.0)):
    """All K+1 columns of one frame: (record (K+1, 8), metrics (K+1, 7)), float64.  Arrays of one pixel count."""
    gt = np.asarray(gt, np.float32).reshape(-1)
    v = np.ones(gt.shape, bool) if valid is None else np.asarray(valid).reshape(-1).astype(bool)
    m0 = v & (gt > 0)
    d_min, d_max = depth_range
    rows = [depth_sums(np.asarray(pred_scene, np.float32).reshape(-1), gt, m0, scale, d_min, d_max)]
    if ids:
        lab = np.asarray(labels).astype(np.int64).reshape(-1) & 0xFFFF
        obj = np.asarray(pred_object, np.float32).reshape(-1)
        rows += [depth_sums(obj, gt, m0 & (lab == i), scale, d_min, d_max) for i in ids]
    rec = np.stack(rows)
    return rec, depth_outputs(rec)


def mask_sums(opacity, labels, obj_id, valid=None, threshold=0.5) -> np.ndarray:
    """[|P & G|, |P | G|, sum |o - [G]|, n_valid] of one object over the valid pixels (P: float32 o >= threshold)."""
    o = np.asarray(opacity, np.float32).reshape(-1)
    v = np.ones(o.shape, bool) if valid is None else np.asarray(valid).reshape(-1).astype(bool)
    G = (np.asarray(labels).astype(np.int64).reshape(-1) & 0xFFFF) == obj_id
    with np.errstate(invalid="ignore"):
        P = o >= np.float32(threshold)
    o, G, P = o[v], G[v], P[v]
    return np.array([(P & G).sum(), (P | G).sum(), np.abs(o.astype(np.float64) - G).sum(), v.sum()], np.float64)


def mask_outputs(rec):
    """(K, 4) sums -> (iou (K,), opacity_l1 (K,)) (NaN for an empty union / no valid pixel)."""
    rec = np.asarray(rec, dtype=np.float64).reshape(-1, 4)
    with np.errstate(divide="ignore", invalid="ignore"):
        return rec[:, 0] / rec[:, 1], rec[:, 2] / rec[:, 3]
