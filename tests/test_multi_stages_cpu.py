"""Float64 references for the editing path's joint sort and compositing (tests/test_gpu_multi_stages.py), the inputs those
tests use, and the checks of the references and their gates that need no device:
  - multi_order: the stable order of each ray's concatenation [set 0 | set 1 | ...] by depth, -0.0 equal to +0.0 and
    NaN last (np.argsort(kind="stable"), which is torch.sort(stable=True)'s order);
  - composite_multi64: composite64 of tests/test_sampling_stages_cpu.py applied in that order (last delta 0, relu(sigma),
    no noise), with the object ids and the scatter of the weights back to set order (weights_unsorted);
  - multi_verdict: depths, ids and weights_unsorted bit for bit, weights and maps inside composite_gate at T = n_obj S
    samples (per-lane term ceil(T / 32) + 6), NaN exactly where the reference is NaN.
Soundness: torch's float32 compositing of O.composite_multi, given the stable order, passes multi_verdict on every input
set the device tests use.  Discrimination: mutants of the multi-object loaders and sinks (last delta 1e10, reversed
ties, no sort, no white background, object id off by one, weights_unsorted at the sorted index) fail it."""
import numpy as np
import pytest
import torch

from oracle import onerf_oracle as O
from tests.test_sampling_stages_cpu import F32, F64, N_PLANT, composite64, composite_gate, gate_share

# (n_obj, S) of the device tests: one-sample sets, the warp width, T = 32 / 33, the largest bitonic buffer (T = 4096),
# just past it (T = 4098, rank-merge only), many sets, and the 2048-sample set bound
MULTI_SHAPES = [(1, 1), (5, 1), (1, 2), (1, 33), (2, 16), (3, 11), (1, 2048), (2, 2048), (3, 1366), (41, 128), (3, 2048)]
MULTI_MANY_RAYS = [(2, 16), (3, 11)]      # 9 000 rays: past the 4 warps x 8 blocks x SMs grid cap
BITONIC_MAX_T = 4096
NAN_POS = np.array([0x7FC00000], np.uint32).view(F32)[0]
NAN_NEG = np.array([0xFFC00000], np.uint32).view(F32)[0]

# planted rows of multi_inputs
ROW_MUTED, ROW_BOX, ROW_TIES, ROW_DESC, ROW_UNSORTED, ROW_OPAQUE, ROW_SUBNORMAL, ROW_ZEROS, ROW_NAN, ROW_NAN_NEG = range(10)
MAP_KEYS = ("weights", "opacity", "rgb", "depth")
OUT_KEYS = ("z_vals", "obj_ids", "weights_unsorted") + MAP_KEYS


def ray_counts(n_obj, S):
    return (1, N_PLANT) + ((9000,) if (n_obj, S) in MULTI_MANY_RAYS else ())


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
def multi_inputs(n, n_obj, S, seed):
    """z_all (n_obj, n, S) and field_all (n_obj, n, S, 4) = (rgb, sigma), fp32.  Random rows: each set ascending in its
    own (near, far), sigma ~ 5 N(0, 1), rgb in (0, 1).  Planted rows, in inputs of at least N_PLANT rays (where they
    fit the shape):
      0 every set muted (z = 0, sigma = -1e5);
      1 a stretch of set 0 muted among live samples (the removed-object box), the last set missed (all zero, muted);
      2 ties: within set 0 pairs of equal depths, and set 1 a copy of set 0's depths; the sigmas differ, so the tie
        order decides which sample gets the non-zero delta;
      3 a descending set (near > far);
      4 an unsorted set;
      5 the ray's first sample opaque (sigma = 1e6);
      6 five opaque samples in a row of the joint order, spread over the sets: transmittance 1e-10, 1e-20, ... into the
        subnormals and to 0;
      7 -0.0 and +0.0 in one ray: set 0 starts +0.0, -0.0 and the last set starts -0.0;
      8 a positive NaN depth in set 0 (what the disparity form gives a missed ray); 9 a negative-signed NaN."""
    rng = np.random.default_rng(seed)
    near = rng.uniform(0.5, 2.0, (n_obj, n, 1))
    far = near + rng.uniform(0.5, 4.0, (n_obj, n, 1))
    z = (near + (far - near) * np.sort(rng.random((n_obj, n, S)), -1)).astype(F32)
    f = np.empty((n_obj, n, S, 4), F32)
    f[..., :3] = rng.random((n_obj, n, S, 3)).astype(F32)
    f[..., 3] = (rng.standard_normal((n_obj, n, S)) * 5).astype(F32)
    sig = f[..., 3]
    T = n_obj * S
    last = n_obj - 1
    if n < N_PLANT:
        return z, f
    z[:, ROW_MUTED] = 0.0
    sig[:, ROW_MUTED] = -1e5
    sig[0, ROW_BOX, S // 4: S // 4 + max(S // 3, 1)] = -1e5
    sig[0, ROW_BOX, S // 4 + max(S // 3, 1):] = np.abs(sig[0, ROW_BOX, S // 4 + max(S // 3, 1):])
    if n_obj > 1:
        z[last, ROW_BOX] = 0.0
        sig[last, ROW_BOX] = -1e5
    z[0, ROW_TIES, 1::2] = z[0, ROW_TIES, 0::2][: z[0, ROW_TIES, 1::2].shape[0]]
    sig[0, ROW_TIES, 0::2] = 0.0
    sig[0, ROW_TIES, 1::2] = 20.0
    if n_obj > 1:
        z[1, ROW_TIES] = z[0, ROW_TIES]
        sig[1, ROW_TIES, 0::2] = 5.0
        sig[1, ROW_TIES, 1::2] = 40.0
    if S > 1:        # evenly spaced from far down to near: strictly descending at every S
        k = n_obj // 2
        z[k, ROW_DESC] = np.linspace(far[k, ROW_DESC, 0], near[k, ROW_DESC, 0], S).astype(F32)
    if S > 2:
        z[0, ROW_UNSORTED] = rng.permutation(z[0, ROW_UNSORTED])
    cat = z[:, ROW_OPAQUE].reshape(T)
    first = int(np.argmin(cat))
    sig[first // S, ROW_OPAQUE, first % S] = 1e6
    cat = z[:, ROW_SUBNORMAL].reshape(T)
    order = np.argsort(cat, kind="stable")
    sig[:, ROW_SUBNORMAL] = np.abs(sig[:, ROW_SUBNORMAL]) * F32(0.1)
    for c in order[T // 3: T // 3 + 5]:
        if c != order[-1]:
            sig[c // S, ROW_SUBNORMAL, c % S] = 1e6
    if S > 1:
        z[0, ROW_ZEROS, :2] = [0.0, -0.0]
    else:
        z[0, ROW_ZEROS, 0] = 0.0
    if n_obj > 1:
        z[last, ROW_ZEROS, 0] = -0.0
    sig[:, ROW_ZEROS, :2] = np.abs(sig[:, ROW_ZEROS, :2]) + 1
    z[0, ROW_NAN, S // 2] = NAN_POS
    z[0, ROW_NAN_NEG, S // 2] = NAN_NEG
    return z, f


def descending_sets(z_all):
    """(n_obj, n) mask of strictly descending sets (S >= 2)."""
    d = np.diff(np.asarray(z_all, F32), axis=2)
    return (d < 0).all(2) & (z_all.shape[2] > 1)


def non_descending_sets(z_all):
    return (np.diff(np.asarray(z_all, F32), axis=2) >= 0).all(2)


# ------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------
def concat_sets(a):
    """(n_obj, n, S, ...) -> (n, n_obj S, ...): each ray's concatenation [set 0 | set 1 | ...]."""
    a = np.asarray(a)
    n_obj, n, S = a.shape[:3]
    return np.swapaxes(a, 0, 1).reshape((n, n_obj * S) + a.shape[3:])


def multi_order(z_all):
    """(n, T) stable order of each ray's concatenated depths by value: -0.0 == +0.0, NaN last (either sign), ties in
    concatenated-index order c = obj S + s."""
    return np.argsort(concat_sets(z_all), axis=1, kind="stable")


def reversed_tie_order(z_all):
    """The order by value with ties broken in reverse concatenated-index order (a mutant)."""
    cat = concat_sets(z_all)
    T = cat.shape[1]
    return T - 1 - np.argsort(cat[:, ::-1], axis=1, kind="stable")


def scatter_to_sets(w_sorted, order, n_obj, S):
    """weights in sorted order (n, T) -> (n_obj, n, S): entry (obj, r, s) is the weight of concatenated sample obj S + s."""
    n, T = order.shape
    out = np.empty((n, T), np.asarray(w_sorted).dtype)
    np.put_along_axis(out, order, w_sorted, 1)
    return np.swapaxes(out.reshape(n, n_obj, S), 0, 1)


def composite_multi64(z_all, field_all, white_back, order=None, last_delta=0.0):
    """volume_rendering_multi (O.composite_multi) in float64 on the fp32 inputs, in `order` (default multi_order):
    composite64 with last delta 0 and relu(sigma).  -> dict(order, z (fp32, sorted), obj_ids, ref (composite64's dict),
    gate (composite_gate), and the kernel's output names: z_vals, obj_ids, weights, weights_unsorted, opacity, rgb,
    depth)."""
    n_obj, n, S = z_all.shape
    order = multi_order(z_all) if order is None else order
    z = np.take_along_axis(concat_sets(z_all), order, 1)
    f = np.take_along_axis(concat_sets(field_all), order[..., None], 1)
    with np.errstate(invalid="ignore", over="ignore"):
        ref = composite64(z, f[..., 3], f[..., :3], last_delta)
        gate = composite_gate(ref, f[..., :3], z, white_back)
        rgb = ref["rgb"] + (1 - ref["opacity"][:, None] if white_back else 0)
    out = dict(order=order, ref=ref, gate=gate, z_vals=z, obj_ids=(order // S).astype(F32), weights=ref["w"],
               opacity=ref["opacity"], rgb=rgb, depth=ref["depth"])
    out["weights_unsorted"] = scatter_to_sets(ref["w"], order, n_obj, S)
    return out


def multi_verdict(got, want, keys=None):
    """-> (failures, shares).  got: the kernel's outputs (numpy, any subset of z_vals, obj_ids, weights, weights_unsorted,
    opacity, rgb, depth); want: composite_multi64's dict.  z_vals and obj_ids bit for bit; weights_unsorted bit for bit
    equal to got's own weights scattered back to set order in the reference's order (so every entry must have been
    written); weights and maps NaN exactly where the float64 reference is NaN and inside composite_gate elsewhere.
    shares: the largest share of its gate each map used."""
    fails, shares = [], {}
    keys = [k for k in (keys or OUT_KEYS) if k in got]
    for k in keys:
        g = np.asarray(got[k])
        if k == "z_vals":
            if not np.array_equal(g.astype(F32).view(np.uint32), np.asarray(want[k], F32).view(np.uint32)):
                fails.append(k)
        elif k == "obj_ids":
            if not np.array_equal(g, want[k]):
                fails.append(k)
        elif k == "weights_unsorted":
            n_obj, n, S = g.shape
            with np.errstate(over="ignore"):      # float64 weights of an unsorted mutant can exceed the fp32 range
                back = scatter_to_sets(np.asarray(got["weights"], F32), want["order"], n_obj, S)
                same = np.array_equal(g.astype(F32).view(np.uint32), back.view(np.uint32))
            if not same:
                fails.append(k)
        else:
            ref, gate = want[k], want["gate"]["w" if k == "weights" else k]
            g = g.astype(F64)
            nan = np.isnan(ref)
            if not np.array_equal(np.isnan(g), nan):
                fails.append(k + " (NaN pattern)")
            ref, gate, g = ref[~nan], gate[~nan], g[~nan]
            share = gate_share(g, ref - gate, ref, ref + gate)
            shares[k] = share
            if not share <= 1.0:
                fails.append(k)
    return fails, shares


def oracle_multi32(z_all, field_all, white_back):
    """torch's float32 compositing of O.composite_multi (O.alpha_weights with last delta 0, then O.composite) on the
    samples gathered in the stable order -> the kernel's output names."""
    order = multi_order(z_all)
    S = z_all.shape[2]
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    z = np.take_along_axis(concat_sets(z_all), order, 1)
    f = np.take_along_axis(concat_sets(field_all), order[..., None], 1)
    _, w = O.alpha_weights(T(f[..., 3]), T(z), 0.0)
    opacity, rgb, depth = O.composite(w, T(f[..., :3]), T(z), white_back)
    w = w.numpy()
    return dict(z_vals=z, obj_ids=(order // S).astype(F32), weights=w, opacity=opacity.numpy(), rgb=rgb.numpy(),
                depth=depth.numpy(), weights_unsorted=scatter_to_sets(w, order, z_all.shape[0], S))


# ------------------------------------------------------------------------------------------------
# checks of the references
# ------------------------------------------------------------------------------------------------
def test_multi_order_is_torch_stable_sort():
    """multi_order is torch.sort(stable=True) of the concatenation on finite depths with ties and zeros of both signs,
    and on the NaN rows it puts every NaN last, in index order, as torch does for a positive NaN."""
    z, _ = multi_inputs(N_PLANT, 3, 11, seed=1)
    cat = concat_sets(z)
    want = torch.sort(torch.from_numpy(cat), dim=1, stable=True).indices.numpy()
    assert np.array_equal(multi_order(z), want)
    r = ROW_ZEROS
    o = multi_order(z)[r]
    zeros = [c for c in o if cat[r, c] == 0]
    assert zeros == sorted(zeros) and np.signbit(cat[r, zeros[1]]) and not np.signbit(cat[r, zeros[0]])
    for r in (ROW_NAN, ROW_NAN_NEG):
        assert np.isnan(cat[r, multi_order(z)[r, -1]])
    # torch puts a negative-signed NaN last as well
    assert torch.isnan(torch.sort(torch.from_numpy(cat[ROW_NAN_NEG]), stable=True).values[-1])


def test_planted_rows_are_what_they_say():
    z, f = multi_inputs(N_PLANT, 3, 11, seed=2)
    sig = f[..., 3]
    assert (z[:, ROW_MUTED] == 0).all() and (sig[:, ROW_MUTED] == -1e5).all()
    assert (sig[0, ROW_BOX] == -1e5).any() and (sig[0, ROW_BOX] > 0).any() and (z[2, ROW_BOX] == 0).all()
    assert np.array_equal(z[0, ROW_TIES], z[1, ROW_TIES]) and (sig[0, ROW_TIES] != sig[1, ROW_TIES]).all()
    assert descending_sets(z)[1, ROW_DESC] and not descending_sets(z)[0, ROW_UNSORTED]
    assert not non_descending_sets(z)[0, ROW_UNSORTED]
    assert (sig[:, ROW_SUBNORMAL] == 1e6).sum() == 5 and (sig[:, ROW_OPAQUE] == 1e6).sum() == 1
    assert np.signbit(z[0, ROW_ZEROS, 1]) and np.signbit(z[2, ROW_ZEROS, 0]) and not np.signbit(z[0, ROW_ZEROS, 0])
    assert np.isnan(z[0, ROW_NAN]).sum() == 1 and not np.signbit(z[0, ROW_NAN][np.isnan(z[0, ROW_NAN])][0])
    assert np.signbit(z[0, ROW_NAN_NEG][np.isnan(z[0, ROW_NAN_NEG])][0])
    w = composite_multi64(z, f, False)["weights"]
    assert (w[ROW_SUBNORMAL] > 0).any() and (w[ROW_SUBNORMAL][w[ROW_SUBNORMAL] > 0].min() < 1e-38)


def test_reference_scatter_is_the_oracle_selection_on_non_descending_sets():
    """weights_unsorted[i] equals the reference's weights[obj_ids == i].view(n, S) (multi_rendering.py:269-271) wherever
    set i is non-descending, and its reverse on a strictly descending set: the sorted order reverses such a set, the
    set order keeps each weight with its own depth."""
    for n_obj, S in ((3, 11), (2, 16), (5, 1)):
        z, f = multi_inputs(N_PLANT, n_obj, S, seed=3)
        m = composite_multi64(z, f, False)
        w, ids = m["weights"], m["obj_ids"]
        asc, desc = non_descending_sets(z), descending_sets(z)
        for i in range(n_obj):
            sel = np.stack([w[r][ids[r] == i] for r in range(N_PLANT)])
            ok = asc[i]
            assert np.array_equal(m["weights_unsorted"][i][ok], sel[ok], equal_nan=True)
            assert np.array_equal(m["weights_unsorted"][i][desc[i]], sel[desc[i]][:, ::-1], equal_nan=True)
        if S > 1:
            assert desc.any()


@pytest.mark.parametrize("n_obj,S", MULTI_SHAPES)
def test_torch_fp32_composite_multi_passes_the_verdict(n_obj, S):
    """Soundness: torch's float32 compositing (O.composite_multi's arithmetic) in the stable order passes multi_verdict on
    every input set of the device tests, white background off and on; the NaN rows are NaN where the reference is."""
    worst = {}
    for n in ray_counts(n_obj, S):
        z, f = multi_inputs(n, n_obj, S, seed=n_obj * 10000 + S + n)
        for white in (False, True):
            got = oracle_multi32(z, f, white)
            fails, shares = multi_verdict(got, composite_multi64(z, f, white))
            assert not fails, (n, white, fails, shares)
            for k, v in shares.items():
                worst[k] = max(worst.get(k, 0.0), v)
    print(f"RATIO torch fp32 composite_multi n_obj={n_obj} S={S}: " +
          ", ".join(f"{k} {v:.2e}" for k, v in sorted(worst.items())))


def _mutants(z, f, white):
    n_obj, n, S = z.shape
    good = composite_multi64(z, f, white)
    out = {"last delta 1e10": composite_multi64(z, f, white, last_delta=1e10),
           "ties reversed": composite_multi64(z, f, white, order=reversed_tie_order(z)),
           "no sort": composite_multi64(z, f, white, order=np.broadcast_to(np.arange(n_obj * S), (n, n_obj * S)))}
    if white:
        out["no white background"] = composite_multi64(z, f, False)
    ids = dict(good)
    ids["obj_ids"] = ((good["order"] + 1) // S).astype(F32)
    out["obj id off by one"] = ids
    ws = dict(good)
    ws["weights_unsorted"] = np.swapaxes(good["weights"].reshape(n, n_obj, S), 0, 1)
    out["weights_unsorted at the sorted index"] = ws
    return good, out


@pytest.mark.parametrize("n_obj,S", [(3, 11), (2, 16), (41, 128)])
def test_verdict_rejects_the_mutants(n_obj, S):
    """Discrimination: each mutant of a loader or sink fails multi_verdict on the planted inputs, with white background
    on (and, but for the white-background mutant, off); the unmutated float64 reference passes with share 0."""
    z, f = multi_inputs(N_PLANT, n_obj, S, seed=n_obj * 10000 + S + N_PLANT)
    for white in (False, True):
        good, mutants = _mutants(z, f, white)
        fails, shares = multi_verdict(good, good)
        assert not fails and max(shares.values()) == 0.0
        for name, m in mutants.items():
            fails, _ = multi_verdict(m, good)
            assert fails, (name, white)
            # the map gates alone catch the arithmetic mutants (the depths and ids would not show them)
            if name in ("last delta 1e10", "ties reversed", "no white background"):
                assert set(fails) & set(MAP_KEYS), (name, white, fails)

