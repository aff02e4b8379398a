"""Reference of edited frames that compose objects from several trained scenes (onerf_render_edit_frame_scenes,
editing.Scene): render_rays_multi (multi_rendering.py:160-325) with each ray set evaluated from its own scene.

Set i belongs to scene set_scene[i] of `scenes`, each a dict of weights ({"coarse", "fine"}), grid, code_table and k =
compose_k(s_src, s_base) (1 for the base scene).  Everything up to the joint compositing is per set in the set's own
units (its coarse depths, its scene's field, its importance sampling from its own weights); volume_rendering_multi then
receives [z_i * k_i] and [sigma_i / k_i], and the per-set maps are tests/set_maps_oracle.py's sums on those inputs.  A set
with k == 1 is taken as it is.  With one scene and k = 1 this is set_maps_oracle.render_rays_multi_sets exactly; given
float64 inputs every step runs in float64."""
import numpy as np

from oracle import onerf_oracle as O
from tests import multi_noise_oracle as M
from tests import set_maps_oracle as SO


def compose_k(s_src, s_base):
    """k = float32(s_src / s_base), the ratio computed in double."""
    return float(np.float32(np.float64(s_src) / np.float64(s_base)))


def render_rays_multi_scenes(scenes, set_scene, rays_list, obj_instance_ids, n_samples=64, use_disp=False,
                             n_importance=0, white_back=False, skip_boxes=None):
    """-> render_rays_multi's result dict plus the per-set maps of both passes (f"{key}_{typ}", key in SO.SET_KEYS), all
    depths on the base scene's axis.  skip_boxes: the removed-object boxes of the base scene set (O.points_in_boxes)."""
    ks = [scenes[j]["k"] for j in set_scene]
    demb = [O.posenc(r[:, 3:6], 4) for r in rays_list]
    z_c = [O.stratified_z(r, n_samples, use_disp) for r in rays_list]

    def fields(typ, zs):
        rgbs, sigmas = [], []
        for i, (z, iid) in enumerate(zip(zs, obj_instance_ids)):
            sc, r = scenes[set_scene[i]], rays_list[i]
            xyz = r[:, None, 0:3] + r[:, None, 3:6] * z[:, :, None]
            rgb, sigma = O.field_eval_single_branch(sc["weights"][typ], sc["grid"], xyz, z, demb[i],
                                                    sc["code_table"][iid] if iid > 0 else None, iid)
            if iid == 0 and skip_boxes:
                sigma[O.points_in_boxes(xyz, skip_boxes)] = -1e5
            rgbs.append(rgb)
            sigmas.append(sigma)
        return rgbs, sigmas

    def frame_axis(zs, sigmas):
        return ([z if k == 1 else z * k for z, k in zip(zs, ks)],
                [s if k == 1 else s / k for s, k in zip(sigmas, ks)])

    out, composited = {}, {}
    rgbs, sigmas = fields("coarse", z_c)
    zf, sf = frame_axis(z_c, sigmas)
    M.composite_multi(out, "coarse", zf, rgbs, sf, white_back, tag_ids=True)
    composited["coarse"] = (zf, rgbs, sf)
    if n_importance > 0:
        z_fine = []
        for i, z in enumerate(z_c):                                      # in the set's own units
            n = z.shape[0]
            w_i = out["weights_coarse"][out["obj_ids_coarse"] == i].view(n, n_samples)
            z_new = O.sample_pdf(0.5 * (z[:, :-1] + z[:, 1:]), w_i[:, 1:-1], n_importance, det=True)
            z_fine.append(O.merge_sorted(z, z_new))
        rgbs, sigmas = fields("fine", z_fine)
        zf, sf = frame_axis(z_fine, sigmas)
        M.composite_multi(out, "fine", zf, rgbs, sf, white_back)
        composited["fine"] = (zf, rgbs, sf)
    for typ, (zs, rgbs, sigmas) in composited.items():
        sets = SO.composite_multi_sets(zs, rgbs, sigmas)
        for k in SO.SET_KEYS:
            out[f"{k}_{typ}"] = sets[k]
    return out
