"""CPU oracle for the object-compositional NeRF per-ray render path.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only `tests/`, `__graft_entry__.smoke()` and the
`cpu_baseline` / `--impl reference` legs of `bench.py` may import it.  The shipped path
(`object_nerf_b200/`) never does; it fails loudly if the CUDA library is missing.

It is a restatement, in plain functions over torch CPU tensors (torch is the reference's own array
library, so the arithmetic is op-for-op the same: fp32, same association order), of the algorithm in
zju3dv/object_nerf.  Every function cites the reference lines it follows (paths relative to
/root/reference).  Randomness is never drawn here: jitter / uniform / gaussian buffers are
*injected* by the caller so that the CUDA path and the oracle see the same numbers.

Parity pin: the reference ships no tests or golden vectors (SURVEY.md §4, §8c), so this oracle is
pinned against outputs of the reference itself, run in the build container by
`tools/make_golden.py` and committed under `tests/golden/` (`tests/test_oracle_golden.py` replays
them bit-for-bit on CPU).

Weight container: a flat dict name -> (W[out,in], b[out]) using the branch layout
  scene: l0..l7, sigma, final, dir, rgb        object: l0..l3, sigma, final, dir, rgb
(`weights_from_state_dict` maps the reference's nn.Module attribute names to it.)
"""
from __future__ import annotations

import itertools
from typing import Dict, Optional, Sequence

import torch

LEAKY_SLOPE = 0.01  # nn.LeakyReLU default, models/nerf_model.py:38


# --------------------------------------------------------------------------------------------
# weights
# --------------------------------------------------------------------------------------------
def weights_from_state_dict(sd: Dict[str, torch.Tensor], D: int = 8, inst_D: int = 4):
    """Reference attribute names (models/nerf_model.py:41-58, 77-95) -> oracle branch layout."""
    w = {}
    for i in range(D):
        w[f"scene.l{i}"] = (sd[f"xyz_encoding_{i+1}.0.weight"], sd[f"xyz_encoding_{i+1}.0.bias"])
    w["scene.final"] = (sd["xyz_encoding_final.weight"], sd["xyz_encoding_final.bias"])
    w["scene.sigma"] = (sd["sigma.weight"], sd["sigma.bias"])
    w["scene.dir"] = (sd["dir_encoding.0.weight"], sd["dir_encoding.0.bias"])
    w["scene.rgb"] = (sd["rgb.0.weight"], sd["rgb.0.bias"])
    for i in range(inst_D):
        w[f"obj.l{i}"] = (sd[f"instance_encoding_{i+1}.0.weight"], sd[f"instance_encoding_{i+1}.0.bias"])
    w["obj.final"] = (sd["instance_encoding_final.0.weight"], sd["instance_encoding_final.0.bias"])
    w["obj.sigma"] = (sd["instance_sigma.weight"], sd["instance_sigma.bias"])
    w["obj.dir"] = (sd["inst_dir_encoding.0.weight"], sd["inst_dir_encoding.0.bias"])
    w["obj.rgb"] = (sd["inst_rgb.0.weight"], sd["inst_rgb.0.bias"])
    return {k: (a.detach(), b.detach()) for k, (a, b) in w.items()}


def _affine(x, wb):
    W, b = wb
    return torch.addmm(b, x, W.t())  # nn.Linear


def _leaky(x):
    return torch.where(x > 0, x, x * LEAKY_SLOPE)


# --------------------------------------------------------------------------------------------
# encoding
# --------------------------------------------------------------------------------------------
def posenc(x: torch.Tensor, n_freqs: int) -> torch.Tensor:
    """[x, sin(2^0 x), cos(2^0 x), ..., sin(2^(F-1) x), cos(2^(F-1) x)], each block x.shape[-1] wide.
    models/embedding_helper.py:52-55 (bands = exact powers of two), :69-74 (order)."""
    parts = [x]
    for k in range(n_freqs):
        f = float(2 ** k)
        parts.append(torch.sin(f * x))
        parts.append(torch.cos(f * x))
    return torch.cat(parts, -1)


class VoxelGrid:
    """The buffers of the reference's EmbeddingVoxel that the per-ray path reads
    (models/embedding_helper.py:107-133, 189-200): offset (3,), voxel_size scalar, shape (3,) ints,
    idx_map (X,Y,Z) int64 with -1 = empty, table (n_rows, 24) fp32."""

    def __init__(self, offset, voxel_size, shape, idx_map, table, n_obj_channels: int = 8,
                 n_freq_voxel: int = 6, n_freq_xyz: int = 10):
        self.offset = offset
        self.voxel_size = voxel_size
        self.shape = [int(s) for s in shape]
        self.idx_map = idx_map
        self.table = table
        self.n_obj_channels = n_obj_channels
        self.n_freq_voxel = n_freq_voxel
        self.n_freq_xyz = n_freq_xyz


def voxel_features(xyz: torch.Tensor, g: VoxelGrid) -> torch.Tensor:
    """Trilinear blend of the 8 surrounding sparse-voxel feature rows; empty / out-of-range corners
    contribute zero.  models/embedding_helper.py:331-352 (lookup), :360-389 (corners, weights).
    Corner order is itertools.product([0,1], repeat=3) i.e. x-major; weights match that order."""
    n = xyz.shape[0]
    p = (xyz + g.offset) / g.voxel_size                       # :360
    q = torch.floor(p).long()                                 # :362
    frac = p - q.to(p.dtype)                                  # :371
    u, v, w = frac[:, 0], frac[:, 1], frac[:, 2]
    lu, lv, lw = 1 - u, 1 - v, 1 - w
    shape = torch.tensor(g.shape, dtype=torch.long)
    acc = None
    for (cx, cy, cz) in itertools.product((0, 1), repeat=3):  # :364-368
        c = q + torch.tensor([cx, cy, cz], dtype=torch.long)
        bad = ((c < 0).sum(1) > 0) | ((c >= shape).sum(1) > 0)  # :336-338
        c = torch.where(bad[:, None], torch.zeros_like(c), c)   # :339
        row = g.idx_map[c[:, 0], c[:, 1], c[:, 2]]              # :342-344
        bad = bad | (row < 0)                                   # :346-347
        row = torch.where(bad, torch.zeros_like(row), row)
        f = g.table[row]
        f = torch.where(bad[:, None], torch.zeros_like(f), f)   # :351
        wt = (u if cx else lu) * (v if cy else lv) * (w if cz else lw)   # :374-383
        term = f * wt[:, None]
        # reference stacks the 8 weighted corner tensors and sums over dim 0 (:386-388); torch's
        # sum over an 8-long leading dim is sequential in this order.
        acc = term if acc is None else acc + term
    return acc  # (n, 24)


def voxel_embed(xyz: torch.Tensor, g: VoxelGrid):
    """EmbeddingVoxel.forward: returns (scene input (n,271), object voxel input (n,104)).
    models/embedding_helper.py:325-329 and :401-409."""
    f = voxel_features(xyz, g)
    c = f.shape[1]
    scene_f, obj_f = f[:, : c - g.n_obj_channels], f[:, c - g.n_obj_channels:]
    scene_in = torch.cat([posenc(scene_f, g.n_freq_voxel), posenc(xyz, g.n_freq_xyz)], -1)
    return scene_in, posenc(obj_f, g.n_freq_voxel)


# --------------------------------------------------------------------------------------------
# the two-branch MLP
# --------------------------------------------------------------------------------------------
def scene_mlp(w, emb_xyz, emb_dir, D: int = 8, skips: Sequence[int] = (4,)):
    """ObjectNeRF.forward, models/nerf_model.py:97-121.  Returns sigma (n,), rgb (n,3)."""
    h = emb_xyz
    for i in range(D):
        if i in skips:
            h = torch.cat([emb_xyz, h], -1)                    # :105 (input first)
        h = _leaky(_affine(h, w[f"scene.l{i}"]))
    sigma = _affine(h, w["scene.sigma"])[:, 0]                 # :108 raw
    fin = _affine(h, w["scene.final"])                         # :114 no activation
    d = _leaky(_affine(torch.cat([fin, emb_dir], -1), w["scene.dir"]))   # :116-117
    rgb = torch.sigmoid(_affine(d, w["scene.rgb"]))            # :118
    return sigma, rgb


def object_mlp(w, emb_xyz, obj_voxel, obj_code, emb_dir, inst_D: int = 4, skips: Sequence[int] = (2,)):
    """ObjectNeRF.forward_instance, models/nerf_model.py:123-152."""
    parts = [emb_xyz] + ([obj_voxel] if obj_voxel is not None else []) + [obj_code]
    x = torch.cat(parts, -1)                                   # :130 / :132
    h = x
    for i in range(inst_D):
        if i in skips:
            h = torch.cat([x, h], -1)                          # :138
        h = _leaky(_affine(h, w[f"obj.l{i}"]))
    sigma = _affine(h, w["obj.sigma"])[:, 0]                   # :140
    fin = _affine(h, w["obj.final"])                           # :146
    d = _leaky(_affine(torch.cat([fin, emb_dir], -1), w["obj.dir"]))     # :147-148
    rgb = torch.sigmoid(_affine(d, w["obj.rgb"]))              # :149
    return sigma, rgb


def field_eval(w, grid: Optional[VoxelGrid], xyz, dirs, codes, n_freq_xyz=10, n_freq_dir=4,
               want_scene=True, want_object=True):
    """Encode + both branches for flat samples.  xyz (B,3); dirs (B,3) per-sample view direction;
    codes (B,C) per-sample object code.  models/rendering.py:106-130.
    Returns dict with sigma (B,), rgb (B,3), inst_sigma (B,), inst_rgb (B,3)."""
    emb_dir = posenc(dirs, n_freq_dir)
    if grid is not None:
        emb_xyz, obj_vox = voxel_embed(xyz, grid)
    else:
        emb_xyz, obj_vox = posenc(xyz, n_freq_xyz), None
    out = {}
    if want_scene:
        out["sigma"], out["rgb"] = scene_mlp(w, emb_xyz, emb_dir)
    if want_object:
        out["inst_sigma"], out["inst_rgb"] = object_mlp(w, emb_xyz, obj_vox, codes, emb_dir)
    return out


# --------------------------------------------------------------------------------------------
# sampling
# --------------------------------------------------------------------------------------------
def stratified_z(rays, n_samples, use_disp=False, perturb=0.0, jitter=None):
    """models/rendering.py:259-277.  rays (N,8) = [o, d, near, far]; jitter (N,S) in [0,1) replaces
    torch.rand_like(z_vals) (:276)."""
    near, far = rays[:, 6:7], rays[:, 7:8]
    t = torch.linspace(0, 1, n_samples, dtype=rays.dtype)
    if not use_disp:
        z = near * (1 - t) + far * t
    else:
        z = 1 / (1 / near * (1 - t) + 1 / far * t)
    if perturb > 0:
        mid = 0.5 * (z[:, :-1] + z[:, 1:])
        upper = torch.cat([mid, z[:, -1:]], -1)
        lower = torch.cat([z[:, :1], mid], -1)
        z = lower + (upper - lower) * (perturb * jitter)
    return z


def sample_pdf(bins, weights, n_importance, det=False, u=None, eps=1e-5):
    """Inverse-CDF sampling, models/rendering.py:11-61.  bins (N,M+1), weights (N,M); if not det the
    caller injects u (N,K) (replaces torch.rand, :40)."""
    n, m = weights.shape
    wts = weights + eps
    pdf = wts / wts.sum(-1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    # An extension of the reference, not a port: models/rendering.py prepends zeros_like(cdf[:, :1]), which is empty when
    # there are no weights (two coarse samples), and then gathers from an empty cdf.  A zero column of its own is the same
    # for m >= 1 and gives m = 0 the cdf [0]: every sample is the one bin, as the library's kernel gives it.
    cdf = torch.cat([torch.zeros(n, 1, dtype=cdf.dtype, device=cdf.device), cdf], -1)
    if det:
        u = torch.linspace(0, 1, n_importance, dtype=bins.dtype).expand(n, n_importance)
    u = u.contiguous()
    inds = torch.searchsorted(cdf, u, right=True)
    below = torch.clamp_min(inds - 1, 0)
    above = torch.clamp_max(inds, m)
    cdf_b, cdf_a = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    bin_b, bin_a = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    denom = cdf_a - cdf_b
    denom = torch.where(denom < eps, torch.ones_like(denom), denom)
    return bin_b + (u - cdf_b) / denom * (bin_a - bin_b)


def merge_sorted(z_coarse, z_new):
    """models/rendering.py:313 — sorted union of coarse and importance depths (values only)."""
    return torch.sort(torch.cat([z_coarse, z_new], -1), -1)[0]


# --------------------------------------------------------------------------------------------
# compositing
# --------------------------------------------------------------------------------------------
def alpha_weights(sigma, z, last_delta, noise=None, noise_std=0.0, zero_mask=None):
    """sigma (N,S), z (N,S) -> alpha (N,S), weights (N,S).  models/rendering.py:139-162.
    zero_mask: positions whose alpha is forced to 0 (occlusion mask, :202)."""
    deltas = z[:, 1:] - z[:, :-1]
    # An extension of the reference, not a port: models/rendering.py shapes the last delta from deltas[:, :1], which is
    # empty for one sample per ray and breaks there.  Shaped from z it is the same for S >= 2, and a lone sample gets
    # last_delta, as the library's kernels give it.
    deltas = torch.cat([deltas, torch.full_like(z[:, :1], last_delta)], -1)
    s = sigma if noise is None else sigma + noise * noise_std
    alpha = 1 - torch.exp(-deltas * torch.relu(s))
    if zero_mask is not None:
        alpha = torch.where(zero_mask, torch.zeros_like(alpha), alpha)
    shifted = torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], -1)
    weights = alpha * torch.cumprod(shifted[:, :-1], -1)
    return alpha, weights


def composite(weights, rgb, z, white_back):
    """opacity, rgb map, depth map.  models/rendering.py:164-182."""
    opacity = weights.sum(-1)
    rgb_map = (weights[:, :, None] * rgb).sum(1)
    depth = (weights * z).sum(-1)
    if white_back:
        rgb_map = rgb_map + 1 - opacity[:, None]
    return opacity, rgb_map, depth


def composite_pass(out, typ, sigma, rgb, inst_sigma, inst_rgb, z, noise_std=0.0, white_back=False,
                   is_eval=False, zero_last_delta=False, forward_instance=True, frustum_bound_th=0.0,
                   pass_through_mask=None, rays_in_bbox=False, noise_scene=None, noise_obj=None):
    """The tail of inference_model, models/rendering.py:139-229.  Fills out[...] like the reference."""
    _, wts = alpha_weights(sigma, z, 0.0 if zero_last_delta else 1e10, noise_scene, noise_std)
    opacity, rgb_map, depth = composite(wts, rgb, z, white_back)
    out[f"weights_{typ}"] = wts
    out[f"opacity_{typ}"] = opacity
    out[f"z_vals_{typ}"] = z
    out[f"rgb_{typ}"] = rgb_map
    out[f"depth_{typ}"] = depth
    if forward_instance:
        mask = None
        if (not is_eval) and frustum_bound_th > 0:           # :192-202
            mask = (depth[:, None] + frustum_bound_th) < z
            if pass_through_mask is not None:
                mask = mask & ~pass_through_mask.reshape(-1, 1).bool()
        _, wi = alpha_weights(inst_sigma, z, 0.0, noise_obj, noise_std, zero_mask=mask)   # :147-148
        oi, ri, di = composite(wi, inst_rgb, z, True)        # :223 always white
        out[f"rgb_instance_{typ}"] = ri
        out[f"depth_instance_{typ}"] = di
        out[f"opacity_instance_{typ}"] = oi
        if rays_in_bbox:                                      # :228-229
            out[f"weights_{typ}"] = wi


# --------------------------------------------------------------------------------------------
# full single-scene render (render_rays)
# --------------------------------------------------------------------------------------------
def render_rays(weights: Dict[str, dict], grid: Optional[VoxelGrid], rays, codes=None, n_samples=64,
                use_disp=False, perturb=0.0, noise_std=0.0, n_importance=0, white_back=False,
                forward_instance=True, frustum_bound_th=0.0, pass_through_mask=None, rays_in_bbox=False,
                is_eval=False, zero_last_delta=False, rand: Optional[dict] = None,
                n_freq_xyz=10, n_freq_dir=4):
    """models/rendering.py:233-337.  weights = {"coarse": w, "fine": w}.  rand carries the injected
    random buffers: jitter (N,S), u (N,K), noise_{scene,obj}_{coarse,fine}."""
    rand = rand or {}
    n = rays.shape[0]
    o, d = rays[:, 0:3], rays[:, 3:6]
    if codes is None:
        codes = torch.zeros(n, 64, dtype=rays.dtype)
    out = {}

    def one_pass(typ, z):
        s = z.shape[1]
        xyz = (o[:, None, :] + d[:, None, :] * z[:, :, None]).reshape(-1, 3)          # :279
        dirs = d[:, None, :].expand(n, s, 3).reshape(-1, 3)                           # :89-92
        cds = codes[:, None, :].expand(n, s, codes.shape[1]).reshape(n * s, -1)       # :94
        f = field_eval(weights[typ], grid, xyz, dirs, cds, n_freq_xyz, n_freq_dir,
                       want_object=forward_instance)
        composite_pass(out, typ, f["sigma"].view(n, s), f["rgb"].view(n, s, 3),
                       f["inst_sigma"].view(n, s) if forward_instance else None,
                       f["inst_rgb"].view(n, s, 3) if forward_instance else None, z,
                       noise_std=noise_std, white_back=white_back, is_eval=is_eval,
                       zero_last_delta=zero_last_delta, forward_instance=forward_instance,
                       frustum_bound_th=frustum_bound_th, pass_through_mask=pass_through_mask,
                       rays_in_bbox=rays_in_bbox, noise_scene=rand.get(f"noise_scene_{typ}"),
                       noise_obj=rand.get(f"noise_obj_{typ}"))

    z = stratified_z(rays, n_samples, use_disp, perturb, rand.get("jitter"))
    one_pass("coarse", z)
    if n_importance > 0:
        mid = 0.5 * (z[:, :-1] + z[:, 1:])                                            # :302-304
        z_new = sample_pdf(mid, out["weights_coarse"][:, 1:-1].detach(), n_importance,
                           det=(perturb == 0), u=rand.get("u"))                        # :305-310 (detached, :307)
        one_pass("fine", merge_sorted(z, z_new))                                      # :313
    return out


# --------------------------------------------------------------------------------------------
# multi-object (editing) render (render_rays_multi)
# --------------------------------------------------------------------------------------------
def field_eval_single_branch(w, grid, xyz, z, dir_emb_rays, code_row, instance_id, n_freq_xyz=10):
    """inference_from_model, render_tools/multi_rendering.py:16-93: scene branch if id == 0 else the
    object branch with one constant code row; rays whose last depth is 0 get sigma = -1e5 (:40,83,92)."""
    n, s = z.shape
    flat = xyz.reshape(-1, 3)
    emb_xyz, obj_vox = voxel_embed(flat, grid) if grid is not None else (posenc(flat, n_freq_xyz), None)
    emb_dir = dir_emb_rays[:, None, :].expand(n, s, dir_emb_rays.shape[1]).reshape(n * s, -1)
    if instance_id > 0:
        cds = code_row[None, :].expand(n * s, -1)
        sigma, rgb = object_mlp(w, emb_xyz, obj_vox, cds, emb_dir)
    else:
        sigma, rgb = scene_mlp(w, emb_xyz, emb_dir)
    sigma = sigma.view(n, s).clone()
    sigma[z[:, -1] == 0] = -1e5
    return rgb.view(n, s, 3), sigma


def composite_multi(out, typ, z_list, rgb_list, sigma_list, white_back, tag_ids=False):
    """volume_rendering_multi, render_tools/multi_rendering.py:96-157 (noise_std = 0 case: the
    editing renderer always passes 0, render_tools/editable_renderer.py:134-135,280-281)."""
    z = torch.cat(z_list, 1)
    rgb = torch.cat(rgb_list, 1)
    sigma = torch.cat(sigma_list, 1)
    z, order = torch.sort(z, -1)                                                      # :112 (stable? see tests)
    rgb = torch.gather(rgb, 1, order[:, :, None].expand(-1, -1, 3))                   # :114-115
    sigma = torch.gather(sigma, 1, order)                                             # :116
    if tag_ids:
        ids = torch.cat([torch.full_like(s, float(i)) for i, s in enumerate(sigma_list)], -1)
        out[f"obj_ids_{typ}"] = torch.gather(ids, 1, order)                           # :118-120
    _, wts = alpha_weights(sigma, z, 0.0)                                             # :125-128 last delta 0
    opacity, rgb_map, depth = composite(wts, rgb, z, white_back)
    out[f"weights_{typ}"] = wts
    out[f"opacity_{typ}"] = opacity
    out[f"z_vals_{typ}"] = z
    out[f"rgb_{typ}"] = rgb_map
    out[f"depth_{typ}"] = depth


def points_in_boxes(xyz, boxes):
    """check_in_any_boxes / BBoxRayHelper.check_xyz_in_bounds, utils/bbox_utils.py:119-130,158-207,
    with the per-box affine map pre-composed by the caller: boxes = list of (A (3,3), t (3,), lo (3,),
    hi (3,)) such that p_box = A @ p + t and inside <=> lo <= p_box <= hi (inclusive)."""
    inside = torch.zeros(xyz.shape[:-1], dtype=torch.bool)
    for (A, t, lo, hi) in boxes:
        p = xyz @ A.t() + t
        inside |= ((p >= lo) & (p <= hi)).all(-1)
    return inside


def render_rays_multi(weights, grid, code_table, rays_list, obj_instance_ids, n_samples=64,
                      use_disp=False, n_importance=0, white_back=False, skip_boxes=None,
                      n_freq_xyz=10, n_freq_dir=4):
    """render_tools/multi_rendering.py:160-325 with perturb = noise_std = 0 (the only way the
    EditableRenderer calls it).  skip_boxes: see points_in_boxes (the removed-object mask, :239-241)."""
    out = {}
    z_list, o_list, d_list, demb_list = [], [], [], []
    for rays in rays_list:
        o_list.append(rays[:, 0:3])
        d_list.append(rays[:, 3:6])
        demb_list.append(posenc(rays[:, 3:6], n_freq_dir))                            # :194
        z_list.append(stratified_z(rays, n_samples, use_disp))                        # :205-211

    def eval_all(typ, zs):
        rgbs, sigmas = [], []
        for i, (z, iid) in enumerate(zip(zs, obj_instance_ids)):
            xyz = o_list[i][:, None, :] + d_list[i][:, None, :] * z[:, :, None]
            rgb, sigma = field_eval_single_branch(weights[typ], grid, xyz, z, demb_list[i],
                                                  code_table[iid] if iid > 0 else None, iid, n_freq_xyz)
            if iid == 0 and skip_boxes:                                               # :239-241
                sigma[points_in_boxes(xyz, skip_boxes)] = -1e5
            rgbs.append(rgb)
            sigmas.append(sigma)
        return rgbs, sigmas

    rgbs, sigmas = eval_all("coarse", z_list)
    composite_multi(out, "coarse", z_list, rgbs, sigmas, white_back, tag_ids=True)
    if n_importance > 0:
        z_fine = []
        for i, z in enumerate(z_list):
            n = z.shape[0]
            mid = 0.5 * (z[:, :-1] + z[:, 1:])
            w_i = out["weights_coarse"][out["obj_ids_coarse"] == i].view(n, n_samples)   # :269-271
            z_new = sample_pdf(mid, w_i[:, 1:-1].detach(), n_importance, det=True)
            z_fine.append(merge_sorted(z, z_new))
        rgbs, sigmas = eval_all("fine", z_fine)
        composite_multi(out, "fine", z_fine, rgbs, sigmas, white_back)
    return out


# --------------------------------------------------------------------------------------------
# rays: camera ray generation and per-object ray assembly (SURVEY.md section 8f rows 1 and 2)
# --------------------------------------------------------------------------------------------
def ray_directions(H: int, W: int, focal: float) -> torch.Tensor:
    """datasets/ray_utils.py:5-25 (get_ray_directions).  kornia.create_meshgrid(H, W, normalized_coordinates=False)[0]
    is grid[y, x] = (x, y) with x = linspace(0, W-1, W), y = linspace(0, H-1, H) (kornia is not installed here: its
    published semantics are restated).  No +0.5 pixel centring (:19-20).  Returns (H, W, 3) fp32."""
    xs = torch.linspace(0, W - 1, W)
    ys = torch.linspace(0, H - 1, H)
    i = xs[None, :].expand(H, W)
    j = ys[:, None].expand(H, W)
    return torch.stack([(i - W / 2) / focal, -(j - H / 2) / focal, -torch.ones_like(i)], -1)


def get_rays(directions: torch.Tensor, c2w: torch.Tensor):
    """datasets/ray_utils.py:28-51: rotate by c2w[:, :3], normalise, origin = c2w[:, 3]; returns (H*W, 3) each."""
    rays_d = directions @ c2w[:, :3].T
    rays_d = rays_d / torch.norm(rays_d, dim=-1, keepdim=True)
    rays_o = c2w[:, 3].expand(rays_d.shape)
    return rays_o.reshape(-1, 3), rays_d.reshape(-1, 3)


def bbox_intersection(bounds, orig, dirn):
    """datasets/geo_utils.py:126-162 (slab test, float64): zero direction components become 1e-14 (:131), a ray whose
    origin is inside the box (tmin < 0 or tmax < 0) is a MISS (:158-160).  bounds (2,3); returns (hit, near, far)."""
    import numpy as np
    dirn = np.array(dirn, dtype=np.float64)
    dirn[dirn == 0] = 1.0e-14
    invdir = 1 / dirn
    sign = (invdir < 0).astype(np.int64)
    tmin = (bounds[sign[0]][0] - orig[0]) * invdir[0]
    tmax = (bounds[1 - sign[0]][0] - orig[0]) * invdir[0]
    tymin = (bounds[sign[1]][1] - orig[1]) * invdir[1]
    tymax = (bounds[1 - sign[1]][1] - orig[1]) * invdir[1]
    if tmin > tymax or tymin > tmax:
        return False, 0.0, 0.0
    tmin, tmax = max(tmin, tymin), min(tmax, tymax)
    tzmin = (bounds[sign[2]][2] - orig[2]) * invdir[2]
    tzmax = (bounds[1 - sign[2]][2] - orig[2]) * invdir[2]
    if tmin > tzmax or tzmin > tmax:
        return False, 0.0, 0.0
    tmin, tmax = max(tmin, tzmin), min(tmax, tzmax)
    if tmin < 0 or tmax < 0:
        return False, 0.0, 0.0
    return True, tmin, tmax


def ray_bbox_intersections(rays_o, rays_d, pose_avg, axis_align_mat, bbox_bounds, scale_factor, bbox_enlarge=0.0):
    """utils/bbox_utils.py:102-156: rays (fp32, NeRF scale) -> box frame -> slab test.  The unscale is an fp32 multiply
    (:109), the two rigid transforms are float64 (:111-116); the direction is rotated by the axis-alignment matrix ONLY
    (:116 uses rays_d, not the de-centred direction - kept).  Returns (mask bool (N,), near (N,1), far (N,1)) with
    near / far = fp32(t) / scale_factor (:151-155)."""
    import numpy as np
    o = rays_o.detach().cpu().numpy() * scale_factor
    d = rays_d.detach().cpu().numpy()
    Ta = np.asarray(pose_avg, dtype=np.float64).squeeze()
    Tb = np.asarray(axis_align_mat, dtype=np.float64)
    o_box = (Ta[:3, :3] @ o.T).T + Ta[:3, 3]
    o_box = (Tb[:3, :3] @ o_box.T).T + Tb[:3, 3]
    d_box = (Tb[:3, :3] @ d.T).T
    bounds = np.array(bbox_bounds, dtype=np.float64, copy=True)
    if bbox_enlarge > 0:
        bounds[0] -= bbox_enlarge
        bounds[1] += bbox_enlarge
    n = o.shape[0]
    hit, near, far = np.empty(n), np.empty(n), np.empty(n)
    for k in range(n):
        hit[k], near[k], far[k] = bbox_intersection(bounds, o_box[k], d_box[k])
    mask = torch.Tensor(hit).bool()
    near_t, far_t = torch.Tensor(near[..., None]), torch.Tensor(far[..., None])
    return mask, near_t / scale_factor, far_t / scale_factor


def generate_rays(obj_id, rays_o, rays_d, near, far, scale_factor, box=None, bbox_enlarge=0.0):
    """render_tools/editable_renderer.py:153-181: (N,8) rays of one object.  Scene (obj_id == 0): constant near / far
    divided by the scale factor; objects: box hit distances, 0 / 0 for rays that miss (:173-176).
    box = dict(pose_avg, axis_align_mat, bbox_bounds)."""
    if obj_id == 0:
        batch_near = near / scale_factor * torch.ones_like(rays_o[:, :1])
        batch_far = far / scale_factor * torch.ones_like(rays_o[:, :1])
        return torch.cat([rays_o, rays_d, batch_near, batch_far], 1)
    mask, bn, bf = ray_bbox_intersections(rays_o, rays_d, box["pose_avg"], box["axis_align_mat"], box["bbox_bounds"],
                                          scale_factor, bbox_enlarge)
    bn[~mask] = 0
    bf[~mask] = 0
    return torch.cat([rays_o, rays_d, bn, bf], 1)


# --------------------------------------------------------------------------------------------
# training loss (SURVEY.md section 8f row 3)
# --------------------------------------------------------------------------------------------
LOSS_TERMS = ("color_loss", "depth_loss", "opacity_loss", "instance_color_loss", "instance_depth_loss")


def total_loss(inputs, batch, conf):
    """models/losses.py:5-135 (TotalLoss): five masked-MSE terms, each summed over the coarse and fine maps, times its
    weight; a term whose mask is empty is skipped (returns None in the reference: :13-14, :46-47, :51-52, :80-81).
    Returns (loss_sum, {term: unweighted value}) like the reference (:121-133)."""
    mse = lambda a, b: (a - b) ** 2
    vm = batch["valid_mask"].view(-1)
    im = batch["instance_mask"].view(-1)
    imw = batch["instance_mask_weight"].view(-1)
    tgt_rgb, tgt_d = batch["rgbs"].view(-1, 3), batch["depths"].view(-1)
    fine = "rgb_fine" in inputs
    terms = {}
    # ColorLoss (:67-98), scene
    m3 = vm.view(-1, 1).repeat(1, 3)
    loss = mse(inputs["rgb_coarse"][m3], tgt_rgb[m3]).mean()
    if fine:
        loss = loss + mse(inputs["rgb_fine"][m3], tgt_rgb[m3]).mean()
    terms["color_loss"] = conf["color_loss_weight"] * loss
    # DepthLoss (:36-64), scene
    if (tgt_d > 0).sum() > 0:
        dm = (vm * (tgt_d > 0)).view(-1)
        loss = mse(inputs["depth_coarse"][dm], tgt_d[dm]).mean()
        if fine:
            loss = loss + mse(inputs["depth_fine"][dm], tgt_d[dm]).mean()
        terms["depth_loss"] = conf["depth_loss_weight"] * loss
    # OpacityLoss (:5-33)
    if vm.sum() > 0:
        w = imw[vm]
        loss = (mse(torch.clamp(inputs["opacity_instance_coarse"][vm], 0, 1), im[vm].float()) * w).mean()
        if "opacity_instance_fine" in inputs:
            loss = loss + (mse(torch.clamp(inputs["opacity_instance_fine"][vm], 0, 1), im[vm].float()) * w).mean()
        terms["opacity_loss"] = conf["opacity_loss_weight"] * loss
    # ColorLoss, instance only (:79-91)
    mi = m3 * im.view(-1, 1).repeat(1, 3)
    if mi.sum() > 0:
        w = imw.view(-1, 1).repeat(1, 3)[mi]
        loss = (mse(inputs["rgb_instance_coarse"][mi], tgt_rgb[mi]) * w).mean()
        if "rgb_instance_fine" in inputs:
            loss = loss + (mse(inputs["rgb_instance_fine"][mi], tgt_rgb[mi]) * w).mean()
        terms["instance_color_loss"] = conf["instance_color_loss_weight"] * loss
    # DepthLoss, instance only (:48-59)
    if (tgt_d > 0).sum() > 0:
        dmi = (vm * (tgt_d > 0)).view(-1) * im
        if dmi.sum() > 0:
            w = imw[dmi]
            loss = (mse(inputs["depth_instance_coarse"][dmi], tgt_d[dmi]) * w).mean()
            if "depth_instance_fine" in inputs:
                loss = loss + (mse(inputs["depth_instance_fine"][dmi], tgt_d[dmi]) * w).mean()
            terms["instance_depth_loss"] = conf["instance_depth_loss_weight"] * loss
    loss_sum = sum(terms.values())
    return loss_sum, {k: v / conf[f"{k}_weight"] for k, v in terms.items()}
