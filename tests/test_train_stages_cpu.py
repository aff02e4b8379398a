"""Float64 references for the stage tests of the tensor-core training backward (tests/test_gpu_train_stages.py), and the
checks of those references that need no device:
  - a numpy Philox4x32-10 with the library's uniform / normal mappings (csrc/common.cuh), against Random123's
    published known-answer vectors;
  - the matched voxel-table gradient reference (PE chain rule on given sin / cos, trilinear scatter with index_add_)
    against float64 autograd of the oracle's voxel_embed, when it is given exact sin / cos."""
import numpy as np
import torch

from oracle import onerf_oracle as O
from tests import synth

# ------------------------------------------------------------------------------------------------
# Philox4x32-10 (Salmon et al., SC'11), the counter RNG of csrc/common.cuh
# ------------------------------------------------------------------------------------------------
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32(ctr, key):
    """ctr (..., 4), key (..., 2) uint32 -> (..., 4) uint32."""
    c = [np.asarray(ctr[..., i], dtype=np.uint64) for i in range(4)]
    k0, k1 = np.asarray(key[..., 0], dtype=np.uint64), np.asarray(key[..., 1], dtype=np.uint64)
    for _ in range(10):
        p0, p1 = np.uint64(_M0) * c[0], np.uint64(_M1) * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & _MASK, p1 >> np.uint64(32), p1 & _MASK
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + np.uint64(_W0)) & _MASK, (k1 + np.uint64(_W1)) & _MASK
    return np.stack(c, -1).astype(np.uint32)


def _key(seed, n):
    return np.broadcast_to(np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint64), (n, 2))


def philox_uniform(seed, stream_id, idx):
    """U[0, 1) with 24 random bits for elements idx (int64 array) of a stream: philox_uniform of common.cuh."""
    idx = np.asarray(idx, dtype=np.uint64)
    ctr = np.stack([idx >> np.uint64(2) & _MASK, idx >> np.uint64(34), np.full_like(idx, stream_id),
                    np.zeros_like(idx)], -1)
    r = philox4x32(ctr, _key(seed, idx.size))
    v = np.take_along_axis(r, (idx & np.uint64(3)).astype(np.int64)[:, None], 1)[:, 0]
    return ((v >> 8).astype(np.float32) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def philox_normal(seed, stream_id, idx):
    """N(0, 1) for elements idx of a stream: philox_normal of common.cuh (Box-Muller on one counter's two words),
    evaluated in float64 and rounded once (the device's logf / cospif may differ by an ulp or two)."""
    idx = np.asarray(idx, dtype=np.uint64)
    ctr = np.stack([idx >> np.uint64(1) & _MASK, idx >> np.uint64(33), np.full_like(idx, stream_id),
                    np.ones_like(idx)], -1)
    r = philox4x32(ctr, _key(seed, idx.size)).astype(np.uint64)
    odd = (idx & np.uint64(1)).astype(bool)
    a, b = np.where(odd, r[:, 2], r[:, 0]), np.where(odd, r[:, 3], r[:, 1])
    u1 = ((a >> np.uint64(8)) + np.uint64(1)).astype(np.float64) / 16777216.0
    u2 = (b >> np.uint64(8)).astype(np.float64) / 16777216.0
    return (np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)).astype(np.float32)


def test_philox_known_answer_vectors():
    """Random123 kat_vectors, philox4x32 with 10 rounds: (counter, key) -> output."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    ctr = np.array([k[0] for k in kat], dtype=np.uint64)
    key = np.array([k[1] for k in kat], dtype=np.uint64)
    want = np.array([k[2] for k in kat], dtype=np.uint32)
    assert np.array_equal(philox4x32(ctr, key), want)


def test_philox_mappings_use_every_word_and_the_high_key_word():
    """The uniform mapping reads word idx % 4 of counter idx / 4; the normal mapping pairs words (0, 1) / (2, 3) of
    counter idx / 2; the high half of a 64-bit seed changes the draw; the draws have the right first two moments."""
    seed = (0x1234_5678 << 32) | 0x9ABC_DEF0
    idx = np.arange(8, dtype=np.int64)
    r = philox4x32(np.array([[0, 0, 7, 0], [1, 0, 7, 0]], dtype=np.uint64), _key(seed, 2))
    want_u = (r.reshape(-1) >> 8).astype(np.float32) / np.float32(16777216.0)
    assert np.array_equal(philox_uniform(seed, 7, idx), want_u)
    assert not np.array_equal(philox_uniform(seed, 7, idx), philox_uniform(seed & 0xFFFFFFFF, 7, idx))
    n = philox_normal(seed, 2, np.arange(200000))
    assert abs(n.mean()) < 0.01 and abs(n.std() - 1.0) < 0.01
    u = philox_uniform(seed, 0, np.arange(200000))
    assert u.min() >= 0.0 and u.max() < 1.0 and abs(u.mean() - 0.5) < 0.005


# ------------------------------------------------------------------------------------------------
# voxel-table gradient references
# ------------------------------------------------------------------------------------------------
# the four layers that read the encoded input X (csrc/layout.h kernel-K order): their dZ slots and output widths
DX_LAYERS = (("S0", 0, "scene.l0", 256), ("S4", 4, "scene.l4", 256), ("O0", 10, "obj.l0", 128),
             ("O2", 12, "obj.l2", 128))
X_COLS = 384       # X layout: scene input [0, 271), pad 271, object voxel PE [272, 376), pad [376, 384)


def x_block(W, name):
    """The X-block columns of a reference weight [out, in] laid out on the 384 kernel columns of X (zero where the layer
    does not read a column)."""
    out = torch.zeros(W.shape[0], X_COLS, dtype=W.dtype)
    out[:, :271] = W[:, :271]
    if name.startswith("obj"):
        out[:, 272:376] = W[:, 271:375]
    return out


def dx_from_dz(dz, weights, want_object, dtype=torch.float64):
    """dX = sum over the X-fed layers of dZ_l W_l[:, X block]; weights: reference weight dict (the caller rounds)."""
    dX = 0
    for name, _, wname, _ in DX_LAYERS[: 4 if want_object else 2]:
        dX = dX + dz[name].to(dtype) @ x_block(weights[wname][0].to(dtype), wname)
    return dX


def grid_coords(rays, z, offset, voxel_size, fused):
    """The fp32 voxel coordinates the kernels form: p = (o + d z + offset) / voxel_size.  fused: o + d z by one fmaf
    (csrc/bwd_dx.cu); else multiply, then add (onerf_encode_bwd, csrc/backward.cu)."""
    n, S = z.shape
    o = rays[:, None, 0:3].expand(n, S, 3).reshape(-1, 3)
    d = rays[:, None, 3:6].expand(n, S, 3).reshape(-1, 3)
    zz = z.reshape(-1, 1).expand(-1, 3)
    if fused:   # an exact product in double, one rounding of the sum (ties of the double rounding are negligible)
        x = (d.double() * zz.double() + o.double()).float()
    else:
        x = o + d * zz
    return (x + offset.reshape(1, 3)) / voxel_size.reshape(1)


def pe_chain(dX, X, base, width, bound=False):
    """d f = dX[f] + sum_k 2^k (cos_k dX[sin_k] - sin_k dX[cos_k]) of the PE block at X column `base`, with sin / cos read
    from X.  bound=True: the same sum over absolute values (a scale for error estimates)."""
    blk = lambda t, j: t[:, base + width * j: base + width * (j + 1)]
    d = blk(dX, 0).abs() if bound else blk(dX, 0).clone()
    for k in range(6):
        s, c, ds, dc = blk(X, 1 + 2 * k), blk(X, 2 + 2 * k), blk(dX, 1 + 2 * k), blk(dX, 2 + 2 * k)
        if bound:
            d = d + 2 ** k * (c.abs() * ds.abs() + s.abs() * dc.abs())
        else:
            d = d + 2 ** k * (c * ds - s * dc)
    return d


def table_grad_matched(dX, X, p, idx_map, n_rows, want_object, bound=False):
    """(n_rows, 24) float64: PE chain rule, then the trilinear scatter; corner weights in p's dtype with the kernels'
    product order (cx ? u : 1 - u) (cy ? v : 1 - v) (cz ? w : 1 - w)."""
    df = [(pe_chain(dX, X, 0, 16, bound), 0)]
    if want_object:
        df.append((pe_chain(dX, X, 272, 8, bound), 16))
    out = torch.zeros(n_rows, 24, dtype=torch.float64)
    q = torch.floor(p)
    frac = p - q
    q = q.long()
    shape = torch.tensor(idx_map.shape)
    for corner in range(8):
        cc = torch.tensor([(corner >> 2) & 1, (corner >> 1) & 1, corner & 1])
        ix = q + cc
        ok = ((ix >= 0) & (ix < shape)).all(1)
        row = torch.full((p.shape[0],), -1, dtype=torch.long)
        row[ok] = idx_map[ix[ok, 0], ix[ok, 1], ix[ok, 2]]
        ok &= row >= 0
        wt = [frac[:, a] if cc[a] else 1 - frac[:, a] for a in range(3)]
        wt = (wt[0] * wt[1] * wt[2]).double()
        for d, ch0 in df:
            out[:, ch0:ch0 + d.shape[1]].index_add_(0, row[ok], wt[ok, None] * d[ok].double())
    return out


def table_grad_autograd(dX, p, idx_map, table, want_object):
    """float64 autograd of the oracle's voxel_embed with a leaf table, given dL/dX on the X layout.  The grid is stated in
    voxel units (offset 0, voxel size 1, xyz = p) so that the corners and weights are those of the same fp32 p."""
    leaf = table.double().clone().requires_grad_(True)
    g = O.VoxelGrid(torch.zeros(3, dtype=torch.float64), 1.0, list(idx_map.shape), idx_map, leaf)
    scene_in, obj_in = O.voxel_embed(p.double(), g)
    X = torch.cat([scene_in, torch.zeros_like(scene_in[:, :1]), obj_in, torch.zeros_like(scene_in[:, :8])], 1)
    mask = torch.zeros(X_COLS, dtype=torch.float64)
    mask[:208] = 1          # scene voxel PE: the xyz PE does not depend on the table
    if want_object:
        mask[272:376] = 1
    (X * dX * mask).sum().backward()
    return leaf.grad


def exact_X(p, idx_map, table):
    """The X layout of the encoded input in float64 (exact sin / cos)."""
    g = O.VoxelGrid(torch.zeros(3, dtype=torch.float64), 1.0, list(idx_map.shape), idx_map, table.double())
    scene_in, obj_in = O.voxel_embed(p.double(), g)
    return torch.cat([scene_in, torch.zeros_like(scene_in[:, :1]), obj_in, torch.zeros_like(scene_in[:, :8])], 1)


def edge_points(shape, n, rng):
    """Voxel coordinates hitting the cases a trilinear scatter gets wrong: interior, the outer half-cell shell
    (floor = -1 or shape - 1), fully outside, exact voxel faces (u = 0) and many points in one cell."""
    shape = np.asarray(shape)
    m = n // 5
    inner = rng.uniform(0, shape - 1, size=(m, 3))
    shell = rng.uniform(0, shape - 1, size=(m, 3))
    ax = rng.integers(0, 3, size=m)
    lo = rng.random(m) < 0.5
    shell[np.arange(m), ax] = np.where(lo, rng.uniform(-1, 0, m), shape[ax] - 1 + rng.uniform(0, 1, m))
    outside = rng.uniform(-3, shape + 2, size=(m, 3))
    face = rng.integers(-1, shape + 1, size=(m, 3)).astype(np.float64)
    face[: m // 2, 0] += rng.uniform(0, 1, m // 2)
    cell = np.floor(rng.uniform(0, shape - 1, size=(1, 3))) + rng.uniform(0, 1, size=(n - 4 * m, 3))
    return np.concatenate([inner, shell, outside, face, cell]).astype(np.float32)


def test_matched_table_grad_equals_autograd_with_exact_sin_cos():
    """The matched reference, fed exact sin / cos and float64 corner weights, is the float64 autograd of voxel_embed:
    both branches, and the object channels untouched at want_object = 0."""
    rng = np.random.default_rng(3)
    g = synth.make_grid(seed=11, shape=(7, 6, 5), occupancy=0.6, voxel_size=0.05)
    p = torch.from_numpy(edge_points((7, 6, 5), 2000, rng)).double()
    assert (p == torch.floor(p)).any(1).sum() > 100           # points on a face
    n_rows = g["table"].shape[0]
    X = exact_X(p, g["idx_map"], g["table"])
    for want_object in (0, 1):
        dX = torch.from_numpy(rng.standard_normal((p.shape[0], X_COLS)))
        want = table_grad_autograd(dX, p, g["idx_map"], g["table"], want_object)
        got = table_grad_matched(dX, X, p, g["idx_map"], n_rows, want_object)
        assert want.abs().max() > 1.0
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-10 * want.abs().max().item()), (got - want).abs().max()
        if not want_object:
            assert (got[:, 16:] == 0).all() and (want[:, 16:] == 0).all()


def test_dx_from_dz_is_the_x_gradient_of_the_four_layers():
    """dx_from_dz maps the reference weights' X columns to the kernel layout: d/dX of sum_l dZ_l . (x_l W_l^T), with x_l
    the reference input of layer l (scene input; object input [scene input | object voxel PE | code])."""
    rng = np.random.default_rng(4)
    w = synth.make_weights(5, True)
    n = 17
    Xk = torch.from_numpy(rng.standard_normal((n, X_COLS))).requires_grad_(True)
    h = torch.from_numpy(rng.standard_normal((n, 256)))
    ho = torch.from_numpy(rng.standard_normal((n, 128)))
    code = torch.from_numpy(rng.standard_normal((n, 64)))
    dz = {name: torch.from_numpy(rng.standard_normal((n, width))) for name, _, _, width in DX_LAYERS}
    scene_in, obj_vox = Xk[:, :271], Xk[:, 272:376]
    obj_in = torch.cat([scene_in, obj_vox, code], 1)
    W = {k: v[0].double() for k, v in w.items()}
    loss = ((scene_in @ W["scene.l0"].t()) * dz["S0"]).sum()
    loss = loss + ((torch.cat([scene_in, h], 1) @ W["scene.l4"].t()) * dz["S4"]).sum()
    loss = loss + ((obj_in @ W["obj.l0"].t()) * dz["O0"]).sum()
    loss = loss + ((torch.cat([obj_in, ho], 1) @ W["obj.l2"].t()) * dz["O2"]).sum()
    loss.backward()
    got = dx_from_dz(dz, w, 1)
    assert torch.allclose(got, Xk.grad, rtol=1e-12, atol=1e-12)
    assert (got[:, 271] == 0).all() and (got[:, 376:] == 0).all()
