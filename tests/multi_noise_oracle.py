"""CPU port of render_tools/multi_rendering.py:96-325 with what oracle.onerf_oracle.render_rays_multi leaves out: sigma
noise (:131-132), perturbed importance sampling (:272-274 with det = False) and 10-column ray sets clipped to their box
interval (:278-287).  Built from the oracle's stage functions in the reference's op order, so it is bit-exact against the
reference's outputs (tests/test_multi_noise_clip_cpu.py); with perturb = noise_std = 0 and 8-column sets it is
onerf_oracle.render_rays_multi."""
import torch

from oracle import onerf_oracle as O


def composite_multi(out, typ, z_list, rgb_list, sigma_list, white_back, tag_ids=False, noise=None, noise_std=0.0):
    """volume_rendering_multi (:96-157).  noise (N, T): the pass's randn_like draw over the SORTED sigmas, scaled by
    noise_std before it is added (:131-132); None adds nothing."""
    z, order = torch.sort(torch.cat(z_list, 1), -1)                                   # :112
    rgb = torch.gather(torch.cat(rgb_list, 1), 1, order[:, :, None].expand(-1, -1, 3))  # :114-115
    sigma = torch.gather(torch.cat(sigma_list, 1), 1, order)                          # :116
    if tag_ids:
        ids = torch.cat([torch.full_like(s, float(i)) for i, s in enumerate(sigma_list)], -1)
        out[f"obj_ids_{typ}"] = torch.gather(ids, 1, order)                           # :118-120
    _, wts = O.alpha_weights(sigma, z, 0.0, noise, noise_std)                         # :123-137, last delta 0
    opacity, rgb_map, depth = O.composite(wts, rgb, z, white_back)
    out[f"weights_{typ}"] = wts
    out[f"opacity_{typ}"] = opacity
    out[f"z_vals_{typ}"] = z
    out[f"rgb_{typ}"] = rgb_map
    out[f"depth_{typ}"] = depth


def clip_to_box(z, rays):
    """:278-287: for a 10-column set, depths with near_box < z < far_box (both strict) become far_box."""
    if rays.shape[1] != 10:
        return z
    near_box, far_box = rays[:, 8:9], rays[:, 9:10]
    return torch.where((z > near_box) & (z < far_box), far_box.expand_as(z), z)


def render_rays_multi(weights, grid, code_table, rays_list, obj_instance_ids, n_samples=64, use_disp=False,
                      n_importance=0, white_back=False, skip_boxes=None, perturb=0.0, noise_std=0.0, rand=None,
                      n_freq_xyz=10, n_freq_dir=4):
    """:160-325.  Ray sets are (N,8) or (N,10).  rand carries the injected draws: u (a list, one (N, K) per set, used
    when perturb != 0) and noise_coarse / noise_fine ((N, T) in sorted order, used when noise_std != 0)."""
    rand = rand or {}
    noise = {typ: rand.get(f"noise_{typ}") if noise_std != 0 else None for typ in ("coarse", "fine")}
    out = {}
    o_list = [r[:, 0:3] for r in rays_list]
    d_list = [r[:, 3:6] for r in rays_list]
    demb_list = [O.posenc(r[:, 3:6], n_freq_dir) for r in rays_list]                 # :194
    z_list = [O.stratified_z(r, n_samples, use_disp) for r in rays_list]             # :205-211

    def eval_all(typ, zs):
        rgbs, sigmas = [], []
        for i, (z, iid) in enumerate(zip(zs, obj_instance_ids)):
            xyz = o_list[i][:, None, :] + d_list[i][:, None, :] * z[:, :, None]
            rgb, sigma = O.field_eval_single_branch(weights[typ], grid, xyz, z, demb_list[i],
                                                    code_table[iid] if iid > 0 else None, iid, n_freq_xyz)
            if iid == 0 and skip_boxes:                                               # :239-241
                sigma[O.points_in_boxes(xyz, skip_boxes)] = -1e5
            rgbs.append(rgb)
            sigmas.append(sigma)
        return rgbs, sigmas

    rgbs, sigmas = eval_all("coarse", z_list)
    composite_multi(out, "coarse", z_list, rgbs, sigmas, white_back, tag_ids=True, noise=noise["coarse"],
                    noise_std=noise_std)
    if n_importance > 0:
        z_fine = []
        det = perturb == 0
        for i, z in enumerate(z_list):
            n = z.shape[0]
            mid = 0.5 * (z[:, :-1] + z[:, 1:])
            w_i = out["weights_coarse"][out["obj_ids_coarse"] == i].view(n, n_samples)   # :269-271
            z_new = O.sample_pdf(mid, w_i[:, 1:-1].detach(), n_importance, det=det, u=None if det else rand["u"][i])
            z_fine.append(clip_to_box(O.merge_sorted(z, z_new), rays_list[i]))
        rgbs, sigmas = eval_all("fine", z_fine)
        composite_multi(out, "fine", z_fine, rgbs, sigmas, white_back, noise=noise["fine"], noise_std=noise_std)
    return out
