"""Host references and planted cases for the voxel grid's device kernels (tests/test_voxel_grid_cpu.py,
tests/test_gpu_voxel_grid.py):

  - voxel_features32: a float32 restatement of encode.cuh voxel_trilinear<..., EXACT = true> in the kernel's order
    (what onerf_voxel_features and onerf_encode compute), with a float64 sum and its error bound beside it;
  - planted positions for a grid: voxel coordinates px that are exact integers on one, two or three axes, px at -1,
    sx - 1 and sx and just below -1 and sx, far outside, non-finite, the 256 empty / occupied patterns of a cell's corners;
  - the grids the tests run on, as make_grid-style dicts (offset, voxel_size, shape, idx_map, table);
  - host restatements of the reference's voxel_subdivision (models/embedding_helper.py:247-302) and of the apply step of
    self_pruning_empty_voxels (:229-245).

Every restatement takes a `fault` argument that plants one known bug, so that the CPU tests can show the checks catch it."""
import itertools
import math

import numpy as np
import torch

from object_nerf_b200 import synthetic

FAULTS = ("trunc", "swap_yz", "reverse_corners", "guard")


# ------------------------------------------------------------------------------------------------
# the trilinear blend
# ------------------------------------------------------------------------------------------------
def voxel_coords(x, g):
    """fp32 voxel coordinates px = fl(fl(x + off) / vsize) of float32 positions x (B, 3), as the kernels form them."""
    return (x + g["offset"].to(x.device).float()) / g["voxel_size"].to(x.device).float()


def voxel_features32(x, g, fault=None):
    """Trilinear features at float32 positions x (B, 3) with the kernels' fp32 voxel coordinates and corner weights
    (encode.cuh voxel_trilinear): -> (float64 sum of the fp32-weighted corners, sum of |weighted corners|, the
    individually rounded fp32 sum of the kernels' EXACT path).

    In the kernel's order: px = fl(fl(x + off) / vsize), fx = floor(px), u = px - fx, lu = 1 - u; no corner is valid
    unless -1 <= fx < sx on every axis (the `any` guard: non-finite and far-outside positions give 0); corner c is
    (c >> 2, c >> 1, c & 1) with weight fl(fl(a b) c); out = fl(out + fl(f wt)) over the valid, occupied corners.
    fault plants one bug: 'trunc' (floor -> truncation), 'swap_yz' (the y / z strides of the index map swapped),
    'reverse_corners' (corners summed 7 .. 0), 'guard' (the guard tightened by one cell at both ends)."""
    assert fault in (None,) + FAULTS, fault
    dev = x.device
    p = voxel_coords(x, g)
    q = torch.trunc(p) if fault == "trunc" else torch.floor(p)
    u = p - q
    lu = 1.0 - u
    shape = g["shape"].to(dev)
    sx, sy, sz = (int(s) for s in g["shape"])
    lo, hi = (0.0, shape.float() - 1) if fault == "guard" else (-1.0, shape.float())
    live = ((q >= lo) & (q < hi)).all(1)
    q = torch.where(live[:, None], q, torch.full_like(q, -2.0)).long()
    idx_flat, table = g["idx_map"].to(dev).reshape(-1), g["table"].to(dev)
    ys, zs = (sy, sz) if fault != "swap_yz" else (sz, sy)
    f64 = torch.zeros(x.shape[0], table.shape[1], dtype=torch.float64, device=dev)
    bound = torch.zeros_like(f64)
    f32 = torch.zeros(x.shape[0], table.shape[1], dtype=torch.float32, device=dev)
    corners = range(7, -1, -1) if fault == "reverse_corners" else range(8)
    for corner in corners:
        cc = [(corner >> 2) & 1, (corner >> 1) & 1, corner & 1]
        ix = q + torch.tensor(cc, device=dev)
        ok = live & ((ix >= 0) & (ix < shape)).all(1)
        ixc = torch.where(ok[:, None], ix, torch.zeros_like(ix))
        row = idx_flat[((ixc[:, 0] * ys + ixc[:, 1]) * zs + ixc[:, 2]) % idx_flat.numel()]   # (wraps only when faulty)
        ok &= row >= 0
        wt = ((u[:, 0] if cc[0] else lu[:, 0]) * (u[:, 1] if cc[1] else lu[:, 1])) * (u[:, 2] if cc[2] else lu[:, 2])
        wt = torch.where(ok, wt, torch.zeros_like(wt))
        t = torch.where(ok[:, None], table[row.clamp(min=0)], torch.zeros(1, device=dev))
        term = t * wt[:, None]
        f32 = torch.where(ok[:, None], f32 + term, f32)
        f64 += t.double() * wt.double()[:, None]
        bound += (t.double() * wt.double()[:, None]).abs()
    return f64, bound, f32


def no_valid_corner(x, g):
    """(B,) True where no corner of the position's cell is inside the grid and occupied: the kernel writes 0 there."""
    p = voxel_coords(x, g)
    q = torch.floor(p)
    shape = g["shape"].to(x.device)
    live = ((q >= -1) & (q < shape.float())).all(1)
    q = torch.where(live[:, None], q, torch.full_like(q, -2.0)).long()
    idx = g["idx_map"].to(x.device)
    none = torch.ones(x.shape[0], dtype=torch.bool, device=x.device)
    for cc in itertools.product((0, 1), repeat=3):
        ix = q + torch.tensor(cc, device=x.device)
        ok = live & ((ix >= 0) & (ix < shape)).all(1)
        ixc = torch.where(ok[:, None], ix, torch.zeros_like(ix))
        none &= ~(ok & (idx[ixc[:, 0], ixc[:, 1], ixc[:, 2]] >= 0))
    return none


def gate(f32, f64, bound, k=16):
    """fp32 sums of at most 8 weighted corners, in any order, lie within k 2^-24 sum |f wt| of the float64 sum."""
    return (f32.double() - f64).abs() <= k * 2.0 ** -24 * bound


def bits(t):
    return t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------------
# planted positions
# ------------------------------------------------------------------------------------------------
def _ulp_walk(x0, steps):
    """float32 x0 (n,) -> (n, 2 steps + 1) of its neighbours x0 - steps ulp .. x0 + steps ulp."""
    up, dn = [x0], [x0]
    for _ in range(steps):
        up.append(torch.nextafter(up[-1], torch.full_like(x0, math.inf)))
        dn.append(torch.nextafter(dn[-1], torch.full_like(x0, -math.inf)))
    return torch.stack(dn[:0:-1] + up, 1)


def solve_axis(g, axis, targets, below=False, steps=96):
    """float32 positions on `axis` whose fp32 voxel coordinate equals each target exactly (below=True: the largest
    coordinate a position reaches that is < target, one ulp of px below it where the position's spacing allows), found
    by walking fp32 neighbours of the nearest position through the kernel's arithmetic.  NaN where the walk finds
    none."""
    t = torch.as_tensor(targets, dtype=torch.float32).reshape(-1)
    off, vs = float(g["offset"][axis]), float(g["voxel_size"])
    x0 = torch.tensor([k * vs - off for k in t.double().tolist()], dtype=torch.float64).float()
    cand = _ulp_walk(x0, steps)
    px = (cand + g["offset"][axis].float()) / g["voxel_size"].float()
    if below:
        ok = px < t[:, None]
        score = torch.where(ok, px, torch.full_like(px, -math.inf))
        j = score.argmax(1)
        found = ok.any(1)
    else:
        ok = px == t[:, None]
        j = ok.float().argmax(1)
        found = ok.any(1)
    out = cand[torch.arange(len(t)), j]
    return torch.where(found, out, torch.full_like(out, math.nan))


def interior(g, n, gen, margin=1.0):
    """n random float32 positions whose voxel coordinates lie in [-margin, s + margin) on every axis."""
    shape = g["shape"].double()
    px = -margin + (shape + 2 * margin) * torch.rand(n, 3, generator=gen, dtype=torch.float64)
    return (px * float(g["voxel_size"]) - g["offset"].double()).float()


def planted_points(g, seed=0):
    """(N, 3) float32 positions planted where the blend's cell choice and guard are decided:
      - px an exact integer on one, two or three axes (faces, edges, corners of cells), every integer in [-1, s];
      - px at -1, just below -1, at s - 1, at s and just below s on each axis;
      - far outside (+-1e30) and non-finite (+-inf, NaN) on each axis;
    the other axes of each position random in [-1, s + 1)."""
    gen = torch.Generator().manual_seed(seed)
    out = []
    ints = []
    for axis in range(3):
        s = int(g["shape"][axis])
        found = solve_axis(g, axis, np.arange(-1, s + 1))
        ints.append(found[~torch.isnan(found)])
        edges = torch.cat([solve_axis(g, axis, [-1.0, s - 1.0, float(s)]),
                           solve_axis(g, axis, [-1.0, float(s)], below=True)])
        vals = torch.cat([ints[-1], edges[~torch.isnan(edges)],
                          torch.tensor([1e30, -1e30, math.inf, -math.inf, math.nan])])
        pts = interior(g, len(vals), gen)
        pts[:, axis] = vals
        out.append(pts)
    # two and three planted axes: every combination of up to 6 of each axis's integer coordinates
    pick = [v[torch.linspace(0, len(v) - 1, min(len(v), 6)).round().long()] for v in ints]
    for axes in ((0, 1), (0, 2), (1, 2), (0, 1, 2)):
        grids = torch.meshgrid(*[pick[a] for a in axes], indexing="ij")
        pts = interior(g, grids[0].numel(), gen)
        for a, v in zip(axes, grids):
            pts[:, a] = v.reshape(-1)
        out.append(pts)
    return torch.cat(out)


def random_points(g, n, seed=1):
    """n random positions inside the grid and up to one cell outside it."""
    return interior(g, n, torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------------
# grids
# ------------------------------------------------------------------------------------------------
def grid_from_occupancy(occ, voxel_size, seed, extra_rows=0, offset=None):
    """A grid dict with the given occupancy: rows numbered in raster order (generate_voxel_idx_map), the last occupied
    cell on the table's last row unless extra_rows are appended, table rows ~ N(0, 1); offset: the volume centred on
    the origin by default."""
    occ = torch.as_tensor(occ, dtype=torch.bool)
    shape = torch.tensor(occ.shape, dtype=torch.int64)
    n = int(occ.sum())
    idx = torch.full(occ.shape, -1, dtype=torch.int64)
    idx[occ] = torch.arange(n)
    rng = np.random.default_rng(seed)
    table = torch.from_numpy(rng.standard_normal((n + extra_rows, synthetic.N_VOX_CH)).astype(np.float32))
    if offset is None:
        offset = (0.5 * shape.double() * voxel_size - voxel_size).float()
    return {"offset": torch.as_tensor(offset, dtype=torch.float32).reshape(3), "voxel_size": torch.tensor(voxel_size, dtype=torch.float32),
            "shape": shape, "idx_map": idx, "table": table}


def corner_pattern_grid(voxel_size=0.3):
    """256 2x2x2 blocks along z (separated by an empty plane), block p occupied in the bit pattern p of its corners
    (corner c = (c >> 2, c >> 1, c & 1) is bit c): the cell at the block's origin sees each empty / occupied pattern
    once.  The last occupied corner holds the table's last row."""
    occ = torch.zeros(2, 2, 3 * 256, dtype=torch.bool)
    for p in range(256):
        for c in range(8):
            if p >> c & 1:
                occ[c >> 2 & 1, c >> 1 & 1, 3 * p + (c & 1)] = True
    return grid_from_occupancy(occ, voxel_size, seed=256)


def corner_pattern_points(g, per_block=6, seed=2):
    """Positions inside the cell at each block's origin (px in (0, 1) on x, y, block z + (0, 1)), per_block each."""
    gen = torch.Generator().manual_seed(seed)
    frac = torch.rand(256, per_block, 3, generator=gen, dtype=torch.float64) * 0.98 + 0.01
    frac[:, :, 2] += 3 * torch.arange(256, dtype=torch.float64)[:, None]
    px = frac.reshape(-1, 3)
    return (px * float(g["voxel_size"]) - g["offset"].double()).float()


def six_face_grid(shape=(6, 9, 4), voxel_size=0.3, seed=61):
    """Random occupancy with every cell on the grid's six faces occupied."""
    occ = torch.from_numpy(np.random.default_rng(seed).random(shape) < 0.4)
    for a in range(3):
        occ.index_fill_(a, torch.tensor([0, shape[a] - 1]), True)
    return grid_from_occupancy(occ, voxel_size, seed)


def maint_grid():
    """The maintenance case's grid (tests/cases.py MAINT_CASE) as EmbeddingVoxel builds it from the point cloud."""
    from tests.test_host_logic_cpu import _maint_embedding
    emb, _ = _maint_embedding()
    return grid_of(emb)


def grid_of(emb):
    return {"offset": emb.voxel_offset.detach().clone(), "voxel_size": emb.voxel_size.detach().clone(),
            "shape": emb.voxel_shape.detach().clone(), "idx_map": emb.voxel_idx_map.detach().clone(),
            "table": emb.embedding_space_ftr.weight.detach().clone()}


def grids():
    """name -> grid dict: the maintenance case, a non-cubic grid, the bench-sized non-dyadic grid, a grid with all six
    faces occupied and the 256 corner patterns."""
    g = synthetic.make_grid(seed=11, shape=(42, 42, 22), voxel_size=0.05)
    n = int((g["idx_map"] >= 0).sum())
    g["table"] = g["table"][:n]                          # the last occupied cell holds the last row
    return {"maint": maint_grid(),
            "noncubic": grid_from_occupancy(np.random.default_rng(7).random((7, 5, 3)) < 0.6, 0.4, seed=7),
            "bench42": g,
            "six_faces": six_face_grid(),
            "corner_patterns": corner_pattern_grid()}


GRID_NAMES = ("maint", "noncubic", "bench42", "six_faces", "corner_patterns")


def points_for(name, g, n_random=20000):
    """The planted positions of a grid and n_random random ones (for the corner-pattern grid: positions in each
    block's cell too)."""
    pts = [planted_points(g), random_points(g, n_random)]
    if name == "corner_patterns":
        pts.append(corner_pattern_points(g))
    return torch.cat(pts)


# ------------------------------------------------------------------------------------------------
# grid maintenance
# ------------------------------------------------------------------------------------------------
def grid_state(emb):
    """The buffers voxel_subdivision / pruning rewrite, cloned (module -> dict)."""
    return {"voxel_size": emb.voxel_size.detach().clone(), "voxel_offset": emb.voxel_offset.detach().clone(),
            "voxel_shape": emb.voxel_shape.detach().clone(), "voxel_occupancy": emb.voxel_occupancy.detach().clone(),
            "voxel_idx_map": emb.voxel_idx_map.detach().clone(), "table": emb.embedding_space_ftr.weight.detach().clone()}


def state_grid(st):
    """A grid-state dict as the grid dict voxel_features32 reads."""
    return {"offset": st["voxel_offset"], "voxel_size": st["voxel_size"], "shape": st["voxel_shape"],
            "idx_map": st["voxel_idx_map"], "table": st["table"]}


def child_positions(st):
    """voxel_subdivision's child positions and their new integer coordinates, reference :248-264: occupied cells in
    torch.nonzero order, children in itertools.product([0, 1], repeat=3) order, blocks of all cells per child."""
    occ = st["voxel_occupancy"]
    idx = torch.nonzero(occ)
    xyz = idx.float() * st["voxel_size"] - st["voxel_offset"]
    target = st["voxel_size"] / 2
    new_xyz = torch.cat([xyz + torch.tensor(c, device=occ.device) * target for c in itertools.product([0, 1], repeat=3)])
    coord = ((new_xyz + st["voxel_offset"]) / target).round().long()
    return new_xyz, coord


def subdivide(st, features_fn=None):
    """Host restatement of voxel_subdivision (reference :247-302) on a grid-state dict -> the new state dict.
    features_fn(new_xyz) -> (n, 24): by default voxel_features32 of the old grid (the kernels' arithmetic).
    Raises RuntimeError when the children do not fit the table (the reference's assert in generate_voxel_idx_map)."""
    new_xyz, coord = child_positions(st)
    ftrs = features_fn(new_xyz) if features_fn else voxel_features32(new_xyz, state_grid(st))[2]
    shape = st["voxel_shape"] * 2
    occ = torch.zeros([int(s) for s in shape], dtype=torch.bool, device=coord.device)
    occ[coord[:, 0], coord[:, 1], coord[:, 2]] = True
    cells = torch.nonzero(occ)
    if cells.shape[0] > st["table"].shape[0]:
        raise RuntimeError("more occupied voxels than N_max_voxels")
    idx = torch.full(occ.shape, -1, dtype=torch.int64, device=coord.device)
    idx[cells[:, 0], cells[:, 1], cells[:, 2]] = torch.arange(cells.shape[0], device=coord.device)
    table = st["table"].clone()
    table[idx[coord[:, 0], coord[:, 1], coord[:, 2]]] = ftrs
    return {"voxel_size": st["voxel_size"] / 2, "voxel_offset": st["voxel_offset"], "voxel_shape": shape,
            "voxel_occupancy": occ, "voxel_idx_map": idx, "table": table}


def prune_apply(cells, max_alpha, th, occ, idx_map, fault=None):
    """Host restatement of the apply step of self_pruning_empty_voxels (reference :229-245): every cell k with
    max_alpha[k] < th (NaN is kept: the comparison is false) loses its occupancy and its index -> (occupancy, index
    map, number pruned), new tensors.  fault='le' plants `<=`."""
    th32 = torch.tensor(th, dtype=torch.float32)
    empty = max_alpha <= th32 if fault == "le" else max_alpha < th32
    gone = cells[empty]
    occ, idx_map = occ.clone(), idx_map.clone()
    occ[gone[:, 0], gone[:, 1], gone[:, 2]] = False
    idx_map[gone[:, 0], gone[:, 1], gone[:, 2]] = -1
    return occ, idx_map, int(gone.shape[0])


def planted_max_alpha(n, th, seed):
    """n per-voxel maxima in [0, 1] with th itself, one ulp below th, 0, NaN and +inf planted in the first rows (the
    rest uniform, so either side of th is populated)."""
    th32 = torch.tensor(th, dtype=torch.float32)
    planted = torch.stack([th32, torch.nextafter(th32, torch.tensor(-math.inf)), torch.tensor(0.0),
                           torch.tensor(math.nan), torch.tensor(math.inf)])
    m = torch.rand(n, generator=torch.Generator().manual_seed(seed))
    k = min(n, len(planted))
    m[:k] = planted[:k]
    return m
