"""-m gpu: the voxel grid's device kernels against the host references of tests/voxel_grid_cases.py (checked on the
CPU by tests/test_voxel_grid_cpu.py):

  - onerf_voxel_features bit-identical to the float32 restatement on the planted positions of five grids (cell faces,
    edges and corners, the guard's boundaries, far and non-finite positions, all 256 corner patterns, the table's last
    row) and on 10^6 random positions; 0 exactly where no corner is valid; counts 0 (no launch), 1, 255, 257 and
    several grid-stride sweeps;
  - onerf_encode with and without a grid: identity columns bit-identical, every sin / cos column within 2^-22 of float64
    sin / cos of the exact fp32 argument, in the reference's column order; a table 4 bytes off alignment is refused
    before any launch;
  - EmbeddingVoxel.voxel_subdivision on the device: grid buffers equal to the host restatement, table rows
    bit-identical to it, rows past the new count untouched; on four grids, a pruned grid and two subdivisions in a row;
  - onerf_prune_apply with maxima planted at the threshold, one ulp below, 0, NaN and +inf on a non-cubic grid, and
    counts 0, 1 and a fully occupied 600 k-cell grid: the host restatement's occupancy, index map and count."""
import ctypes as C
import math
import time

import numpy as np
import pytest
import torch

from oracle import onerf_oracle as O
from tests import voxel_grid_cases as V

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def grids():
    return V.grids()


def _buffers(g):
    from object_nerf_b200 import engine
    return engine.GridBuffers(g["table"].to(DEV), g["idx_map"].to(DEV), g["offset"].to(DEV), g["voxel_size"].to(DEV),
                              g["shape"].to(DEV))


def _device_features(x, g):
    from object_nerf_b200 import engine
    out = engine.voxel_features(x.to(DEV), _buffers(g))
    torch.cuda.synchronize()
    return out.cpu()


def _launches():
    from object_nerf_b200 import _lib
    torch.cuda.synchronize()
    return _lib.launch_count(DEV)


def _same(got, want):
    """Bit-identical, NaN matching NaN."""
    return (V.bits(got) == V.bits(want)) | (torch.isnan(got) & torch.isnan(want))


def _sweeps():
    """A count past several grid-stride sweeps of the stand-alone kernels (num_sms * 16 blocks of 256 threads)."""
    return torch.cuda.get_device_properties(DEV).multi_processor_count * 16 * 256 * 2 + 17


# ------------------------------------------------------------------------------------------------
# onerf_voxel_features
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", V.GRID_NAMES)
def test_voxel_features_bit_identical_on_planted_points(grids, name):
    g = grids[name]
    x = V.points_for(name, g)
    got = _device_features(x, g)
    want = V.voxel_features32(x, g)[2]
    assert got.shape == want.shape
    diff = V.bits(got) != V.bits(want)
    assert not diff.any(), (int(diff.any(1).sum()), x[diff.any(1)][:4].tolist())
    none = V.no_valid_corner(x, g)
    assert (V.bits(got[none]) == 0).all() and (got[~none] != 0).any(1).any()
    far = ~torch.isfinite(x).all(1) | (x.abs() >= 1e30).any(1)
    assert far.sum() == 15 and (V.bits(got[far]) == 0).all()      # the kernel gives 0 where the reference gives NaN


def test_voxel_features_bit_identical_on_a_million_random_points(grids):
    g = grids["bench42"]
    x = V.random_points(g, 10 ** 6, seed=42)
    t0 = time.perf_counter()
    got = _device_features(x, g)
    t1 = time.perf_counter()
    want = V.voxel_features32(x, g)[2]
    print(f"10^6 points: device call {1e3 * (t1 - t0):.1f} ms, host restatement {time.perf_counter() - t1:.1f} s")
    assert torch.equal(V.bits(got), V.bits(want))
    none = V.no_valid_corner(x, g)
    assert none.any() and (~none).any() and (V.bits(got[none]) == 0).all()


@pytest.mark.parametrize("n", [0, 1, 255, 257, "sweeps"])
def test_voxel_features_at_every_count(grids, n):
    from object_nerf_b200 import engine
    n = _sweeps() if n == "sweeps" else n
    g = grids["noncubic"]
    x = V.random_points(g, n, seed=n)
    before = _launches()
    out = engine.voxel_features(x.to(DEV), _buffers(g))
    launched = _launches() - before
    assert out.shape == (n, 24) and launched == (0 if n == 0 else 1)
    want = V.voxel_features32(x, g)[2]
    assert torch.equal(V.bits(out.cpu()), V.bits(want))
    before = _launches()
    scene, obj = engine.encode(x.to(DEV), _buffers(g))
    assert scene.shape == (n, 271) and obj.shape == (n, 104) and _launches() - before == (0 if n == 0 else 1)
    assert torch.equal(V.bits(scene[:, :16].cpu()), V.bits(want[:, :16]))
    assert torch.equal(V.bits(obj[:, :8].cpu()), V.bits(want[:, 16:]))


# ------------------------------------------------------------------------------------------------
# onerf_encode
# ------------------------------------------------------------------------------------------------
def _check_pe(got, v32, n_freq, label):
    """got (B, C (2 n_freq + 1)) against [v, sin 2^k v, cos 2^k v]_k: v bit-identical, sin / cos within 2^-22 of the
    float64 functions at the exact fp32 argument 2^k v (NaN where that is NaN)."""
    c = v32.shape[1]
    assert got.shape[1] == c * (2 * n_freq + 1), label
    assert _same(got[:, :c], v32).all(), label
    want = O.posenc(v32.double(), n_freq)[:, c:]
    g = got[:, c:].double()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(g), nan), label
    err = (g - want).abs()[~nan]
    assert err.max() <= 2.0 ** -22, (label, err.max().item())


@pytest.mark.parametrize("name", [None, "bench42", "noncubic", "corner_patterns"])
def test_encode_columns_against_float64(grids, name):
    from object_nerf_b200 import engine
    g = grids[name or "bench42"]
    x = V.points_for(name or "bench42", g, n_random=5000)
    scene, obj = engine.encode(x.to(DEV), _buffers(g) if name else None)
    torch.cuda.synchronize()
    scene = scene.cpu()
    if name is None:
        assert obj is None and scene.shape == (x.shape[0], 63)
        _check_pe(scene, x, 10, "PE10(xyz)")
        return
    obj = obj.cpu()
    assert scene.shape == (x.shape[0], 271) and obj.shape == (x.shape[0], 104)    # 16 * 13 + 63, 8 * 13
    f = V.voxel_features32(x, g)[2]
    _check_pe(scene[:, :208], f[:, :16], 6, "scene voxel PE")
    _check_pe(obj, f[:, 16:], 6, "object voxel PE")
    _check_pe(scene[:, 208:], x, 10, "PE10(xyz)")


def test_encode_refuses_a_misaligned_table_before_any_launch(grids):
    """Rows are read as float4: a table view 4 bytes past a 16-byte boundary is refused with a message and nothing is
    launched (onerf_voxel_features likewise)."""
    from object_nerf_b200 import _lib
    g = dict(grids["noncubic"])
    rows = g["table"].shape[0]
    store = torch.zeros(rows * 24 + 4, dtype=torch.float32, device=DEV)
    g["table"] = store[1:1 + rows * 24].view(rows, 24)
    buf = _buffers(g)
    assert buf.table.data_ptr() % 16 == 4
    x = torch.zeros(8, 3, device=DEV)
    scene = torch.empty(8, 271, device=DEV)
    obj = torch.empty(8, 104, device=DEV)
    lib = _lib.load()
    before = _launches()
    rc = lib.onerf_encode(_lib.ctx(DEV), C.byref(buf.c), x.data_ptr(), 8, scene.data_ptr(), obj.data_ptr(), _lib.stream())
    assert rc == -1 and b"misaligned" in lib.onerf_last_error()
    rc = lib.onerf_voxel_features(_lib.ctx(DEV), C.byref(buf.c), x.data_ptr(), 8, scene.data_ptr(), _lib.stream())
    assert rc == -1 and b"misaligned" in lib.onerf_last_error()
    assert _launches() == before


# ------------------------------------------------------------------------------------------------
# voxel_subdivision
# ------------------------------------------------------------------------------------------------
def _module(g, spare_rows, seed):
    """EmbeddingVoxel holding grid g with its table extended by spare_rows random rows."""
    from object_nerf_b200 import synthetic
    g = dict(g)
    extra = torch.from_numpy(np.random.default_rng(seed).standard_normal((spare_rows, 24)).astype(np.float32))
    g["table"] = torch.cat([g["table"], extra])
    return synthetic.make_embedding(g)


SUBDIV_CASES = ("maint", "noncubic", "bench42", "six_faces", "pruned_six_faces", "noncubic_twice")


@pytest.mark.parametrize("case", SUBDIV_CASES)
def test_voxel_subdivision_on_device_matches_host_restatement(grids, case):
    from tests.test_host_logic_cpu import _maint_embedding
    times = 2 if case.endswith("_twice") else 1
    if case == "maint":
        emb = _maint_embedding()[0]
    else:
        g = dict(grids[case.replace("pruned_", "").replace("_twice", "")])
        if case.startswith("pruned_"):
            occ = g["idx_map"] >= 0
            cells = torch.nonzero(occ)
            m = V.planted_max_alpha(cells.shape[0], 0.5, seed=17)
            _, g["idx_map"], pruned = V.prune_apply(cells, m, 0.5, occ, g["idx_map"])
            assert 0 < pruned < cells.shape[0]                       # holes in the index map, rows not renumbered
        n = int((g["idx_map"] >= 0).sum())
        emb = _module(g, 8 ** times * n + 37 - g["table"].shape[0], seed=len(case))
    want = V.grid_state(emb)
    counts = []
    for _ in range(times):
        counts.append(int(want["voxel_occupancy"].sum()))
        want = V.subdivide(want)
    table0 = emb.embedding_space_ftr.weight.detach().clone()
    emb = emb.to(DEV)
    for k in range(times):
        n_after = emb.voxel_subdivision()
        assert n_after == 8 * counts[k]                             # every child has its own cell
    for k in ("voxel_size", "voxel_shape", "voxel_occupancy", "voxel_idx_map"):
        got = getattr(emb, k).cpu()
        assert got.dtype == want[k].dtype and torch.equal(got, want[k]), k
    table = emb.embedding_space_ftr.weight.detach().cpu()
    assert torch.equal(V.bits(table[:n_after]), V.bits(want["table"][:n_after]))
    assert torch.equal(V.bits(table[n_after:]), V.bits(table0[n_after:])) and table.shape[0] > n_after


# ------------------------------------------------------------------------------------------------
# onerf_prune_apply
# ------------------------------------------------------------------------------------------------
def _apply(cells, max_alpha, th, occ, idx_map):
    from object_nerf_b200 import _lib
    cells_d, m_d = cells.contiguous().to(DEV), max_alpha.to(DEV)
    occ_d, idx_d = occ.to(DEV), idx_map.to(DEV)
    count = torch.full((1,), -5, dtype=torch.int64, device=DEV)
    before = _launches()
    _lib.check(_lib.load().onerf_prune_apply(_lib.ctx(DEV), cells_d.data_ptr(), cells.shape[0], m_d.data_ptr(), th,
                                             occ.shape[1], occ.shape[2], occ_d.data_ptr(), idx_d.data_ptr(),
                                             count.data_ptr(), _lib.stream()))
    launched = _launches() - before
    return occ_d.cpu(), idx_d.cpu(), int(count.item()), launched


@pytest.mark.parametrize("case", ["noncubic", "noncubic_full", "empty", "one", "600k"])
def test_prune_apply_matches_host_restatement(grids, case):
    th = 0.3
    if case in ("noncubic", "noncubic_full", "empty", "one"):
        g = grids["noncubic"] if case == "noncubic" else V.grid_from_occupancy(torch.ones(7, 5, 3, dtype=torch.bool), 0.4, 9)
    else:
        g = V.grid_from_occupancy(torch.ones(100, 80, 75, dtype=torch.bool), 0.01, 600)
    occ = g["idx_map"] >= 0
    cells = torch.nonzero(occ)
    if case == "empty":
        cells = cells[:0]
    elif case == "one":
        cells = cells[37:38]
    m = V.planted_max_alpha(cells.shape[0], th, seed=cells.shape[0])
    if case == "one":
        m[:] = torch.nextafter(torch.tensor(th, dtype=torch.float32), torch.tensor(-math.inf))
    want_occ, want_idx, want_n = V.prune_apply(cells, m, th, occ, g["idx_map"])
    t0 = time.perf_counter()
    got_occ, got_idx, got_n, launched = _apply(cells, m, th, occ, g["idx_map"])
    print(f"{case}: {cells.shape[0]} cells, {want_n} pruned, call {1e3 * (time.perf_counter() - t0):.1f} ms")
    assert got_n == want_n and launched == (0 if cells.shape[0] == 0 else 1)
    assert torch.equal(got_occ, want_occ) and torch.equal(got_idx, want_idx)
    if case.startswith("noncubic"):
        assert [bool(got_occ[tuple(c)]) for c in cells[:5]] == [True, False, False, True, True]
    if case == "600k":
        assert cells.shape[0] > _sweeps() // 2 and 0 < want_n < cells.shape[0]
    if case == "one":
        assert want_n == 1
