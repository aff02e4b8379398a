"""Float64 reference of the per-set maps of the editing path (onerf_render_edit_frame_sets, editing.set_keys).

For pass typ, ray r and set position i, with w the pass's joint-composited weights (multi_rendering.py:96-157, as
volume_rendering_multi forms them):
    opacity_sets[r, i] = sum w,  depth_sets[r, i] = sum w z,  rgb_sets[r, i] = sum w rgb   (over set i's samples)
with no white background.  composite_multi_sets restates volume_rendering_multi in float64 on the pass's fp32 per-set
inputs and sums by set; render_rays_multi_sets runs tests/multi_noise_oracle.py's port (bit-exact against the reference's
fixtures, so its depths are the reference's) and adds both passes' per-set maps.  set_maps64 / set_maps_verdict give the same
maps on the (n_obj, N, S) arrays of the device tests, with an a-priori error bound for the kernels built from
composite_gate's per-sample weight bound."""
import math

import numpy as np
import torch

from oracle import onerf_oracle as O
from tests import multi_noise_oracle as M
from tests.test_multi_stages_cpu import composite_multi64, scatter_to_sets
from tests.test_sampling_stages_cpu import TINY, U24

SET_KEYS = ("opacity_sets", "depth_sets", "rgb_sets")


def composite_multi_sets(z_list, rgb_list, sigma_list, noise=None, noise_std=0.0):
    """volume_rendering_multi in float64, summed by set.  z / sigma (N,S_i), rgb (N,S_i,3) per set; noise (N, T) in sorted
    order as M.composite_multi takes it.  -> dict of the per-set maps and the joint maps (rgb without white back)."""
    f64 = lambda t: t.to(torch.float64)
    z = f64(torch.cat(z_list, 1))
    z_sorted, order = torch.sort(torch.cat(z_list, 1), -1)                              # :112
    rgb = torch.gather(f64(torch.cat(rgb_list, 1)), 1, order[:, :, None].expand(-1, -1, 3))
    sigma = torch.gather(torch.cat(sigma_list, 1), 1, order)
    if noise is not None and noise_std != 0:
        sigma = sigma + noise * noise_std                                               # the fp32 roundings of :131-132
    ids = torch.cat([torch.full_like(s, i, dtype=torch.long) for i, s in enumerate(sigma_list)], -1)
    ids = torch.gather(ids, 1, order)
    _, w = O.alpha_weights(f64(sigma), f64(z_sorted), 0.0)
    n_obj = len(z_list)
    zs = torch.gather(z, 1, order)
    out = {"opacity_sets": torch.zeros(w.shape[0], n_obj, dtype=torch.float64)}
    out["depth_sets"] = torch.zeros_like(out["opacity_sets"])
    out["rgb_sets"] = torch.zeros(w.shape[0], n_obj, 3, dtype=torch.float64)
    for i in range(n_obj):
        wi = torch.where(ids == i, w, torch.zeros_like(w))
        out["opacity_sets"][:, i] = wi.sum(1)
        out["depth_sets"][:, i] = (wi * zs).sum(1)
        out["rgb_sets"][:, i] = (wi[..., None] * rgb).sum(1)
    out["opacity"], out["depth"], out["rgb"] = w.sum(1), (w * zs).sum(1), (w[..., None] * rgb).sum(1)
    return out


def render_rays_multi_sets(weights, grid, code_table, rays_list, obj_instance_ids, n_samples=64, use_disp=False,
                           n_importance=0, white_back=False, skip_boxes=None, perturb=0.0, noise_std=0.0, rand=None):
    """M.render_rays_multi's result dict plus f"{key}_{typ}" for key in SET_KEYS and each pass, float64."""
    rand = rand or {}
    out = M.render_rays_multi(weights, grid, code_table, rays_list, obj_instance_ids, n_samples=n_samples,
                              use_disp=use_disp, n_importance=n_importance, white_back=white_back,
                              skip_boxes=skip_boxes, perturb=perturb, noise_std=noise_std, rand=rand)
    # the per-set depths of each pass, as M.render_rays_multi forms them (its fp32 coarse weights feed the fine depths)
    z_c = [O.stratified_z(r, n_samples, use_disp) for r in rays_list]
    passes = {"coarse": z_c}
    if n_importance > 0:
        det = perturb == 0
        z_f = []
        for i, z in enumerate(z_c):
            n = z.shape[0]
            w_i = out["weights_coarse"][out["obj_ids_coarse"] == i].view(n, n_samples)
            z_new = O.sample_pdf(0.5 * (z[:, :-1] + z[:, 1:]), w_i[:, 1:-1], n_importance, det=det,
                                 u=None if det else rand["u"][i])
            z_f.append(M.clip_to_box(O.merge_sorted(z, z_new), rays_list[i]))
        passes["fine"] = z_f
    for typ, zs in passes.items():
        rgbs, sigmas = [], []
        for i, (z, iid) in enumerate(zip(zs, obj_instance_ids)):
            rays = rays_list[i]
            xyz = rays[:, None, 0:3] + rays[:, None, 3:6] * z[:, :, None]
            rgb, sigma = O.field_eval_single_branch(weights[typ], grid, xyz, z, O.posenc(rays[:, 3:6], 4),
                                                    code_table[iid] if iid > 0 else None, iid)
            if iid == 0 and skip_boxes:
                sigma[O.points_in_boxes(xyz, skip_boxes)] = -1e5
            rgbs.append(rgb)
            sigmas.append(sigma)
        noise = rand.get(f"noise_{typ}") if noise_std != 0 else None
        sets = composite_multi_sets(zs, rgbs, sigmas, noise, noise_std)
        for k in SET_KEYS:
            out[f"{k}_{typ}"] = sets[k]
    return out


def set_maps64(z_all, field_all):
    """The per-set maps in float64 of the kernels' inputs: z_all (n_obj, N, S) and field_all (n_obj, N, S, 4) fp32 numpy
    (the depths and fields one pass composites).  -> dict(opacity_sets (N, n_obj), depth_sets, rgb_sets (N, n_obj, 3),
    and their a-priori gates under the same keys + "_gate")."""
    n_obj, n, S = z_all.shape
    want = composite_multi64(z_all, field_all, False)
    with np.errstate(invalid="ignore", over="ignore"):
        w = scatter_to_sets(want["ref"]["w"], want["order"], n_obj, S)            # (n_obj, N, S) float64
        g = scatter_to_sets(want["gate"]["w"], want["order"], n_obj, S)
        z = z_all.astype(np.float64)
        c = field_all[..., :3].astype(np.float64)
        sum_r = (math.ceil(S / 32) + 6) * U24                                       # per-lane sums, butterfly, products
        wa = np.abs(w) + g
        out = dict(opacity_sets=w.sum(-1).T, depth_sets=(w * z).sum(-1).T,
                   rgb_sets=(w[..., None] * c).sum(-2).transpose(1, 0, 2))
        out["opacity_sets_gate"] = (g.sum(-1) + sum_r * wa.sum(-1)).T + TINY
        out["depth_sets_gate"] = ((g * np.abs(z)).sum(-1) + sum_r * (wa * np.abs(z)).sum(-1)).T + TINY
        out["rgb_sets_gate"] = ((g[..., None] * np.abs(c)).sum(-2) +
                                sum_r * (wa[..., None] * np.abs(c)).sum(-2)).transpose(1, 0, 2) + TINY
    return out


def set_maps_verdict(got, want, keys=SET_KEYS):
    """-> (failures, shares): each map NaN exactly where the float64 reference is, inside its gate elsewhere; shares =
    the largest share of its gate each map used."""
    fails, shares = [], {}
    for k in keys:
        g, ref, gate = np.asarray(got[k], np.float64), want[k], want[k + "_gate"]
        nan = np.isnan(ref)
        if not np.array_equal(np.isnan(g), nan):
            fails.append(k + " (NaN pattern)")
        err = np.abs(g[~nan] - ref[~nan]) / gate[~nan]
        shares[k] = float(err.max()) if err.size else 0.0
        if shares[k] > 1.0:
            fails.append(k)
    return fails, shares
