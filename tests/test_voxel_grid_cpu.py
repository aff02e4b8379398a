"""The voxel grid's host references (tests/voxel_grid_cases.py) checked without a device, so that the device tests
(tests/test_gpu_voxel_grid.py) can compare the kernels with them bit for bit:

  - the float32 restatement of the trilinear blend equals the oracle's voxel_features on every finite planted and random
    position of five grids, and lies within its float64 gate; within the same gate of the unmodified reference's
    compute_voxel_features_sparse(..., positional_embedding=False) when oracle/_ref is built;
  - the planted positions hit what they claim (exact integer / boundary voxel coordinates, every corner pattern, the
    table's last row); non-finite and far positions give 0 (the reference gives NaN);
  - each planted fault of the restatement (floor -> truncation, swapped strides, reversed corners, the guard off by one,
    `<=` at the prune threshold) fails the equality or the gate the device tests use;
  - the restatements of voxel_subdivision and of the prune apply step reproduce the reference-generated fixtures;
  - EmbeddingVoxel.voxel_subdivision that would overflow the table raises and leaves every buffer bit-identical;
  - onerf_encode / onerf_voxel_features refuse a table that is not 16-byte aligned before any CUDA call."""
import ctypes
import math
import os

import pytest
import torch

from oracle import onerf_oracle as O
from oracle import ref_loader as R
from tests import cases
from tests import voxel_grid_cases as V


@pytest.fixture(scope="module")
def grids():
    return V.grids()


@pytest.fixture(scope="module")
def points(grids):
    return {name: V.points_for(name, g) for name, g in grids.items()}


def _oracle_grid(g, dtype=torch.float32):
    return O.VoxelGrid(g["offset"], g["voxel_size"], g["shape"].tolist(), g["idx_map"], g["table"].to(dtype))


def _moderate(x, g):
    """Positions the reference's floor().long() can hold: finite, voxel coordinates below 2^40."""
    p = V.voxel_coords(x, g)
    return (torch.isfinite(p) & (p.abs() < 2.0 ** 40)).all(1)


def _ref64(x, g):
    """The reference's blend in float64 at the fp32 voxel coordinates: exact corner choice, float64 weights."""
    p = V.voxel_coords(x, g).double()
    grid = O.VoxelGrid(torch.zeros(3, dtype=torch.float64), 1.0, g["shape"].tolist(), g["idx_map"], g["table"].double())
    return O.voxel_features(p, grid)


# ------------------------------------------------------------------------------------------------
# the restatement against the oracle and the reference
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", V.GRID_NAMES)
def test_restatement_equals_oracle_within_float64_gate(grids, points, name):
    g, x = grids[name], points[name]
    f64, bound, f32 = V.voxel_features32(x, g)
    ok = _moderate(x, g)
    assert torch.equal(f32[ok], O.voxel_features(x[ok], _oracle_grid(g)))
    assert V.gate(f32, f64, bound).all()
    ref = _ref64(x[ok], g)
    assert ((f32[ok].double() - ref).abs() <= 24 * 2.0 ** -24 * bound[ok]).all()
    none = V.no_valid_corner(x, g)
    assert (f32[none] == 0).all() and (bound[~none] > 0).any() and none.any() and (~none).any()


@pytest.mark.skipif(not R.available(), reason="oracle/_ref not built (needs the reference checkout at build time)")
@pytest.mark.parametrize("name", V.GRID_NAMES)
def test_restatement_within_gate_of_unmodified_reference(grids, points, name):
    """The reference sums its 8 weighted corners with sum(0), in no defined order: the gate, not bit equality."""
    g = grids[name]
    x = points[name]
    x = x[_moderate(x, g)]
    f64, bound, f32 = V.voxel_features32(x, g)
    restore = torch.Tensor.cuda is R._ORIG_CUDA[0]
    R.install(cuda_noop=True)
    try:
        emb = R.ref_voxel_embedding(g)
        with torch.no_grad():
            ref = emb.compute_voxel_features_sparse(x.clone(), trilinear_interpolate=True, positional_embedding=False)
    finally:
        if restore:
            R.cuda_noop(False)
    assert ref.dtype == torch.float32 and ref.shape == f32.shape
    assert V.gate(ref, f64, bound).all()
    assert V.gate(f32, ref.double(), bound).all()


@pytest.mark.parametrize("name", V.GRID_NAMES)
def test_far_and_non_finite_positions_give_zero(grids, name):
    """The `any` guard: +-1e30, +-inf and NaN on any axis have no valid corner and give 0; the reference's 0 * NaN
    weights give NaN for a NaN position instead (DESIGN.md section 7)."""
    g = grids[name]
    x = V.interior(g, 15, torch.Generator().manual_seed(5))
    for axis in range(3):
        x[5 * axis:5 * axis + 5, axis] = torch.tensor([1e30, -1e30, math.inf, -math.inf, math.nan])
    f64, bound, f32 = V.voxel_features32(x, g)
    assert torch.equal(V.bits(f32), torch.zeros_like(V.bits(f32))) and (f64 == 0).all() and (bound == 0).all()
    assert V.no_valid_corner(x, g).all()
    nan_rows = torch.isnan(x).any(1)
    assert torch.isnan(O.voxel_features(x[nan_rows], _oracle_grid(g))).all()


# ------------------------------------------------------------------------------------------------
# the planted cases are what they say
# ------------------------------------------------------------------------------------------------
def test_planted_coordinates_hit_their_targets(grids):
    """Every solved position reaches its voxel coordinate exactly (or the largest one below it); across the grids each
    axis sees px = -1, s - 1 and s exactly and just below -1 and s."""
    hit = {(a, k): 0 for a in range(3) for k in ("-1", "s-1", "s", "<-1", "<s")}
    for g in grids.values():
        for a in range(3):
            s = int(g["shape"][a])
            t = torch.arange(-1, s + 1, dtype=torch.float32)
            x = V.solve_axis(g, a, t)
            found = ~torch.isnan(x)
            px = (x[found] + g["offset"][a]) / g["voxel_size"]
            assert torch.equal(px, t[found])
            assert found.sum() >= (s + 2) // 2, (a, int(found.sum()), s + 2)
            for k, tv in (("-1", -1.0), ("s-1", s - 1.0), ("s", float(s))):
                hit[(a, k)] += int(found[int(tv) + 1])
            below = V.solve_axis(g, a, [-1.0, float(s)], below=True)
            pb = (below + g["offset"][a]) / g["voxel_size"]
            assert (pb < torch.tensor([-1.0, float(s)])).all()
            assert (pb > torch.tensor([-1.0 - 2e-5, s - 2e-5 * s])).all()
            hit[(a, "<-1")] += 1
            hit[(a, "<s")] += 1
    assert all(v > 0 for v in hit.values()), hit


def test_every_corner_pattern_and_the_last_row_are_planted(grids):
    g = grids["corner_patterns"]
    idx = g["idx_map"]
    assert int(idx.max()) == g["table"].shape[0] - 1
    x = V.corner_pattern_points(g)
    q = torch.floor(V.voxel_coords(x, g)).long()
    seen = set()
    for r in range(x.shape[0]):
        pattern = 0
        for c in range(8):
            i = q[r] + torch.tensor([c >> 2 & 1, c >> 1 & 1, c & 1])
            pattern |= int(idx[i[0], i[1], i[2]] >= 0) << c
        assert pattern == r // 6
        seen.add(pattern)
    assert seen == set(range(256))
    for name in ("bench42", "noncubic", "six_faces"):
        assert int(grids[name]["idx_map"].max()) == grids[name]["table"].shape[0] - 1
    six = grids["six_faces"]["idx_map"] >= 0
    for a in range(3):
        assert six.select(a, 0).all() and six.select(a, six.shape[a] - 1).all()


# ------------------------------------------------------------------------------------------------
# planted faults fail the checks the device tests use
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fault", V.FAULTS)
def test_planted_fault_in_the_blend_is_caught(grids, points, fault):
    """The device tests require the kernel's bits to equal the restatement's on these positions: each fault changes
    some bits; the faults that change what is computed (all but the summation order) also fail the float64 gate."""
    caught_bits = caught_gate = False
    for name, g in grids.items():
        x = points[name]
        f64, bound, f32 = V.voxel_features32(x, g)
        _, _, bad = V.voxel_features32(x, g, fault=fault)
        caught_bits |= not torch.equal(V.bits(bad), V.bits(f32))
        caught_gate |= not V.gate(bad, f64, bound).all()
    assert caught_bits
    assert caught_gate == (fault != "reverse_corners")


def test_planted_fault_at_the_prune_threshold_is_caught():
    th = 0.3
    g = grids_noncubic_full()
    occ = g["idx_map"] >= 0
    cells = torch.nonzero(occ)
    m = V.planted_max_alpha(cells.shape[0], th, seed=3)
    o1, i1, n1 = V.prune_apply(cells, m, th, occ, g["idx_map"])
    o2, i2, n2 = V.prune_apply(cells, m, th, occ, g["idx_map"], fault="le")
    kept = [bool(o1[tuple(cells[k])]) for k in range(5)]
    assert kept == [True, False, False, True, True]            # th kept, one ulp below pruned, 0 pruned, NaN / inf kept
    assert n2 == n1 + 1 and not torch.equal(o1, o2) and not torch.equal(i1, i2)


def grids_noncubic_full():
    """A fully occupied non-cubic grid (dim_y != dim_z)."""
    return V.grid_from_occupancy(torch.ones(7, 5, 3, dtype=torch.bool), 0.4, seed=9)


# ------------------------------------------------------------------------------------------------
# grid maintenance restatements against the reference-generated fixtures
# ------------------------------------------------------------------------------------------------
def _maint_state():
    from tests.test_host_logic_cpu import _maint_embedding
    emb, inp = _maint_embedding()
    return V.grid_state(emb), inp


def test_subdivision_restatement_matches_reference_golden(golden):
    gold = golden("maint_subdivision")
    st, _ = _maint_state()
    n = int(gold["before|table_rows"].shape[0])
    assert torch.equal(st["voxel_idx_map"], gold["before|voxel_idx_map"])
    old = _oracle_grid(V.state_grid(st))
    new = V.subdivide(st, features_fn=lambda p: O.voxel_features(p, old))
    for k in ("voxel_size", "voxel_shape", "voxel_idx_map"):
        assert torch.equal(new[k], gold["subdiv|" + k]), k
    assert torch.equal(new["voxel_occupancy"], gold["subdiv|voxel_occupancy"].bool())
    assert torch.equal(new["table"][:8 * n], gold["subdiv|table_rows"])
    # the kernels' arithmetic: the same rows within the gate of the reference's
    ours = V.subdivide(st)
    f64, bound, _ = V.voxel_features32(V.child_positions(st)[0], V.state_grid(st))
    assert torch.equal(ours["voxel_idx_map"], new["voxel_idx_map"])
    assert (ours["table"][:8 * n] - gold["subdiv|table_rows"]).abs().max() <= 1e-6
    assert bound.max() > 0 and f64.shape[0] == 8 * n


def test_prune_apply_restatement_matches_reference_golden(golden):
    """The per-voxel maxima of the reference's pruning loop (oracle density, the fixture's jitter), then the restated
    apply step: the reference's pruned grid."""
    gold = golden("maint_pruning")
    st, inp = _maint_state()
    grid = _oracle_grid(V.state_grid(st))
    cells = torch.nonzero(st["voxel_occupancy"])
    n = cells.shape[0]
    assert n == int(gold["n_before"])
    centres = cells.float() * st["voxel_size"] - st["voxel_offset"]
    rand = cases.maint_rand((n + 31) // 32)
    maxima = []
    for k, i in enumerate(range(0, n, 32)):
        s = centres[i:i + 32, None, :].expand(-1, 4096, -1).reshape(-1, 3).clone()
        s += rand[k][:s.shape[0]] * st["voxel_size"] - st["voxel_size"] / 2
        sigma = O.field_eval(inp["weights"], grid, s, torch.zeros_like(s), None, want_object=False)["sigma"]
        maxima.append((1 - torch.exp(-torch.relu(sigma.reshape(-1)))).view(-1, 4096).max(-1)[0])
    occ, idx, pruned = V.prune_apply(cells, torch.cat(maxima), cases.MAINT_CASE["max_alpha_th"], st["voxel_occupancy"],
                                     st["voxel_idx_map"])
    assert 0 < pruned < n
    assert torch.equal(occ, gold["pruned|voxel_occupancy"].bool())
    assert torch.equal(idx, gold["pruned|voxel_idx_map"])


# ------------------------------------------------------------------------------------------------
# voxel_subdivision that would overflow the table
# ------------------------------------------------------------------------------------------------
def _maint_module(max_voxels):
    from object_nerf_b200.embedding_helper import EmbeddingVoxel
    c, inp = cases.MAINT_CASE, cases.build_maint_case()
    torch.manual_seed(0)
    return EmbeddingVoxel(24, 6, max_voxels, c["extra"], points=inp["points"])


def _snapshot(emb):
    return {k: v.detach().clone() for k, v in list(emb.state_dict().items())}


@pytest.mark.parametrize("extra", [-1, 0])
def test_subdivision_overflow_leaves_every_buffer_unchanged(extra):
    """8 n - 1 table rows for n occupied voxels: the call raises, and every buffer and the table are bit-identical to
    before (the index map still matches the shape, so later kernels index inside it).  8 n rows: it succeeds and equals
    the restatement."""
    n = int(_maint_module(4096).voxel_occupancy.sum())
    emb = _maint_module(8 * n + extra)
    before = _snapshot(emb)
    st = V.grid_state(emb)
    fn = lambda p: V.voxel_features32(p, V.state_grid(st))[2]
    if extra < 0:
        with pytest.raises(RuntimeError, match="N_max_voxels"):
            emb.voxel_subdivision(_features_fn=fn)
        after = _snapshot(emb)
        assert after.keys() == before.keys()
        for k in before:
            assert before[k].dtype == after[k].dtype and before[k].shape == after[k].shape, k
            raw = lambda t: t.reshape(-1).view(torch.uint8) if t.dtype != torch.bool else t
            assert torch.equal(raw(before[k]), raw(after[k])), k
        with pytest.raises(RuntimeError, match="N_max_voxels"):
            V.subdivide(st)
    else:
        assert emb.voxel_subdivision(_features_fn=fn) == 8 * n
        want = V.subdivide(st)
        for k in ("voxel_size", "voxel_shape", "voxel_occupancy", "voxel_idx_map"):
            assert torch.equal(getattr(emb, k), want[k]), k
        assert torch.equal(V.bits(emb.embedding_space_ftr.weight.detach()), V.bits(want["table"]))


# ------------------------------------------------------------------------------------------------
# argument checks of the stand-alone encoders
# ------------------------------------------------------------------------------------------------
def test_encoders_refuse_a_misaligned_table_before_any_cuda_call():
    """Table rows are read as float4: a table 4 bytes off a 16-byte boundary is refused with a message (no GPU
    needed: the check runs before the context is touched)."""
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    lib = _lib.load()
    ctx = ctypes.c_void_p(1)
    grid = _lib.Grid(0x10004, 0x1000, 0x1000, 0x1000, 0x1000)
    assert lib.onerf_encode(ctx, ctypes.byref(grid), 0x2000, 4, 0x3000, 0x4000, None) == -1
    assert b"misaligned" in lib.onerf_last_error()
    assert lib.onerf_voxel_features(ctx, ctypes.byref(grid), 0x2000, 4, 0x3000, None) == -1
    assert b"misaligned" in lib.onerf_last_error()
    # no points: nothing to read or write (an empty tensor's data pointer is null) and nothing is launched
    grid = _lib.Grid(0x10000, 0x1000, 0x1000, 0x1000, 0x1000)
    assert lib.onerf_voxel_features(ctx, ctypes.byref(grid), None, 0, None, None) == 0
    assert lib.onerf_encode(ctx, ctypes.byref(grid), None, 0, None, None, None) == 0
    assert lib.onerf_encode(ctx, None, None, 0, None, None, None) == 0
