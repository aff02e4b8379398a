"""Float64 references for the depth-sampling and compositing stage tests (tests/test_gpu_sampling_stages.py), the inputs
those tests use, and the checks of the references and their gates that need no device:
  - coarse_depth32: the fp32 arithmetic of sample_coarse_kernel (csrc/sampling.cu), one rounding per operation, and
    coarse_depth64, the same formula in float64;
  - sample_pdf64 / pdf_gate: float64 inverse CDF with the reference's denominator guard, and the interval every fp32
    implementation of it must land in;
  - composite64 / composite_gate: the oracle's composite_pass in float64 on the fp32 inputs the kernel reads, and an
    a-priori bound per weight and per map.
Soundness: torch's own float32 oracle (a second fp32 implementation) lies inside every gate on every input set the device
tests use.  Discrimination: reference-level mutants (no guard, guard at <=, searchsorted left, one-sided linspace, <=
occlusion mask) fall outside the gates on the planted inputs."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import onerf_oracle as O
from tests import synth

F32, F64 = np.float32, np.float64
U24 = 2.0 ** -24
EPS32 = F32(1e-5)            # the kernel's eps (sample_pdf_merge_kernel), as float32
EPS = float(EPS32)

# ------------------------------------------------------------------------------------------------
# shapes of the device tests (the soundness checks below run the same inputs)
# ------------------------------------------------------------------------------------------------
COARSE_S = [1, 2, 3, 31, 32, 33, 64, 65, 1000, 2048]
PDF_BINS = [1, 2, 31, 32, 33, 63, 200, 1500]          # bin edges; n_bins - 1 weights
PDF_K = [1, 2, 31, 33, 64, 100]
PDF_SHAPES = [(b, k) for b in PDF_BINS for k in PDF_K if b + 1 + k <= 2048]
MERGE_SHAPES = [(2, 1), (3, 1), (3, 30), (33, 31), (33, 32), (40, 24), (64, 64), (64, 65), (100, 157), (1024, 1024),
                (2045, 3)]
MERGE_MANY_RAYS = [(3, 30), (33, 32)]                 # 9 000 rays: past the 8 warps x 8 blocks x SMs grid cap
COMPOSITE_S = [1, 2, 31, 32, 33, 128, 192, 2048]
N_PLANT = 37


# ------------------------------------------------------------------------------------------------
# coarse depths
# ------------------------------------------------------------------------------------------------
def linspace01_32(n, one_sided=False):
    """torch.linspace(0, 1, n) in fp32 as linspace01 (csrc/sampling.cu) forms it: step = 1 / (n - 1), step * i below
    n / 2, 1 - step * (n - 1 - i) from there (ATen's symmetric formula).  one_sided: step * i for all i (a mutant)."""
    i = np.arange(n)
    if n <= 1:
        return np.zeros(n, F32)
    step = F32(1) / F32(n - 1)
    lo = step * i.astype(F32)
    if one_sided:
        return lo
    hi = F32(1) - step * (n - 1 - i).astype(F32)
    return np.where(i < n // 2, lo, hi).astype(F32)


def linspace01_fma32(n):
    """torch.linspace(0, 1, n) as torch's CPU kernel forms it here: the same symmetric formula, but the upper half
    1 - step * (n - 1 - i) is one fused multiply-add (its vectorised path), so it is rounded once, not twice."""
    from fractions import Fraction
    t = linspace01_32(n)
    if n > 1:
        step = Fraction(float(F32(1) / F32(n - 1)))
        for i in range(n // 2, n):
            t[i] = F32(float(1 - step * (n - 1 - i)))
    return t


def coarse_depth32(rays, S, use_disp=False, perturb=0.0, jitter=None, one_sided=False, t=None):
    """sample_coarse_kernel in numpy float32: every + - * / rounded once, no fused multiply-add.  t overrides
    linspace01."""
    rays = np.asarray(rays, F32)
    near, far = rays[:, 6:7], rays[:, 7:8]
    t = (linspace01_32(S, one_sided) if t is None else np.asarray(t, F32))[None, :]
    omt = F32(1) - t
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if not use_disp:
            z = near * omt + far * t
        else:
            z = F32(1) / ((F32(1) / near) * omt + (F32(1) / far) * t)
        if perturb > 0:
            mid = F32(0.5) * (z[:, :-1] + z[:, 1:])
            lower = np.concatenate([z[:, :1], mid], 1)
            upper = np.concatenate([mid, z[:, -1:]], 1)
            z = lower + (upper - lower) * (F32(perturb) * np.asarray(jitter, F32))
    return z.astype(F32)


def coarse_depth64(rays, S, use_disp=False, perturb=0.0, jitter=None):
    """The same formula in float64 with t = i / (S - 1) exact."""
    rays = np.asarray(rays, F32).astype(F64)
    near, far = rays[:, 6:7], rays[:, 7:8]
    t = (np.arange(S) / max(S - 1, 1))[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        z = near * (1 - t) + far * t if not use_disp else 1 / (1 / near * (1 - t) + 1 / far * t)
        if perturb > 0:
            mid = 0.5 * (z[:, :-1] + z[:, 1:])
            lower = np.concatenate([z[:, :1], mid], 1)
            upper = np.concatenate([mid, z[:, -1:]], 1)
            z = lower + (upper - lower) * (perturb * np.asarray(jitter, F32).astype(F64))
    return z


# coarse_depth32 against coarse_depth64, in ulp of the depth: the disparity form rounds 1 / near, 1 / far, two products,
# their sum and the reciprocal (each relative u, the reciprocal passing on the sum's error) and t itself carries one
# rounding; the jitter adds the mid-points, upper - lower (which can cancel), the products and the add.  Up to eleven ulp
# were seen over the device test's 5 10^5 depths per shape; 16 leaves room.
ULP_64 = 16


def coarse_rays(n, seed):
    """Camera rays with random near < far, and planted rays: near = far (rows 1, 4) and near = far = 0 (rows 2, 5, the
    muted rays of the multi-object forward)."""
    rays = synth.random_rays(seed, n).numpy().astype(F32)
    rng = np.random.default_rng(seed)
    rays[:, 6] = rng.uniform(0.05, 2.0, n)
    rays[:, 7] = rays[:, 6] + rng.uniform(0.01, 6.0, n)
    for r in range(n):
        if r % 3 == 1 and r < 6:
            rays[r, 7] = rays[r, 6]
        elif r % 3 == 2 and r < 6:
            rays[r, 6:8] = 0.0
    return rays


def coarse_jitter(n, S, seed):
    """U[0, 1) jitter with 0 and 1 - 2^-24 planted."""
    j = np.random.default_rng(seed).random((n, S)).astype(F32)
    j.reshape(-1)[::7] = 0.0
    j.reshape(-1)[3::7] = F32(1 - U24)
    return j


def disp_ok(rays):
    """Rays the use_disp formula is defined on (near > 0; near = 0 divides by zero in the reference too)."""
    return np.asarray(rays)[:, 6] > 0


# ------------------------------------------------------------------------------------------------
# inverse CDF
# ------------------------------------------------------------------------------------------------
def cdf64_of(weights):
    """Float64 cdf of the pdf over fp32 weights + eps (that sum is rounded to fp32 first, as both fp32 implementations
    do): (N, M + 1), cdf[:, 0] = 0."""
    wts = (np.asarray(weights, F32) + EPS32).astype(F64)
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.cumsum(wts / wts.sum(-1, keepdims=True), -1)
    return np.concatenate([np.zeros((wts.shape[0], 1)), c], 1)


def pdf_delta(M):
    """Bound on |cdf_kernel - cdf64| for M weights.  With u = 2^-24 and every term positive:
      - the normaliser is summed in fp32 by 32 lanes of ceil(M / 32) sequential adds and a 5-level butterfly, so each
        term meets at most ceil(M / 32) + 5 roundings: total = W (1 + t), |t| <= (ceil(M / 32) + 5) u;
      - each quotient (w_j + eps) / total is rounded once more: relative error <= |t| + u;
      - the prefix sums are formed in double (relative 2^-53 per add, under u for M <= 2^29) and each is rounded to fp32
        once: another u.
    cdf64 <= 1, so |cdf_kernel - cdf64| <= (ceil(M / 32) + 8) u, with one u left over for the second-order terms."""
    return (math.ceil(M / 32) + 8) * U24


def _take(a, i):
    return np.take_along_axis(a, i, 1)


def sample_pdf64(bins, cdf, u, guard="lt", side="right", amb=None, amb_guard=None):
    """models/rendering.py:11-61 in float64 on a given cdf (N, M + 1): searchsorted(cdf, u, right=True), clamped gathers,
    denominator guard (denom < eps -> 1).  guard "le" / "none" and side "left" are the discrimination mutants.  amb (N, M)
    marks bins whose guard decision is forced to amb_guard."""
    bins, cdf, u = (np.asarray(x, F64) for x in (bins, cdf, u))
    M = cdf.shape[1] - 1
    inds = np.stack([np.searchsorted(cdf[r], u[r], side=side) for r in range(cdf.shape[0])])
    below, above = np.maximum(inds - 1, 0), np.minimum(inds, M)
    cb, ca, bb, ba = _take(cdf, below), _take(cdf, above), _take(bins, below), _take(bins, above)
    denom = ca - cb
    guarded = {"lt": denom < EPS, "le": denom <= EPS, "none": denom <= 0}[guard]
    if amb is not None:     # only where the sample is inside a bin (past the last knot below = above, denom = 0)
        amb_b = _take(np.concatenate([amb, np.zeros((amb.shape[0], 1), bool)], 1), below) & (above > below)
        guarded = np.where(amb_b, amb_guard, guarded)
    return bb + (u - cb) / np.where(guarded, 1.0, denom) * (ba - bb)


def pdf_gate(bins, weights, u, cdf=None, delta=None):
    """-> (lo, ref, hi).  The sample is non-decreasing in u and non-increasing in every cdf entry (d/dc_j and d/dc_j+1 of
    (u - c_j) / (c_j+1 - c_j) are <= 0 for u in the bin, and the guarded branch stays inside its bin), so with every entry
    within delta of cdf64: R(cdf64 + delta) - r <= got <= R(cdf64 - delta) + r.  A bin whose float64 denominator lies
    within 2 delta (+ the rounding of the difference) of eps may be guarded either way: lo / hi are taken over both
    decisions.  r: the last fp32 line bb + ((u - cb) / denom) (ba - bb) has five roundings (u - cb, ca - cb, the
    quotient, ba - bb, the product; relative u each on t (ba - bb), t <= 1) and the final add (u |result|)."""
    bins = np.asarray(bins, F32).astype(F64)
    cdf = cdf64_of(weights) if cdf is None else np.asarray(cdf, F64)
    M = cdf.shape[1] - 1
    delta = pdf_delta(M) if delta is None else delta
    amb = np.abs(np.diff(cdf, axis=1) - EPS) <= 2 * delta + 2 * U24 * EPS
    if delta == 0:          # an exact cdf (planted): every guard decision is determined
        amb[:] = False
    ends = [sample_pdf64(bins, cdf + s * delta, u, amb=amb, amb_guard=g) for s in (1, -1) for g in (True, False)]
    lo, hi = np.minimum.reduce(ends), np.maximum.reduce(ends)
    width = np.abs(np.diff(bins, axis=1)).max(1, initial=0.0)[:, None]
    # jittered depths of a near = far ray may descend by an ulp: the monotonicity in the cdf then holds up to the largest
    # drop of the bins
    drop = (np.maximum.accumulate(bins, 1) - bins).max(1)[:, None]
    r = U24 * (5 * width + np.abs(bins).max(1)[:, None]) + drop
    return lo - r, sample_pdf64(bins, cdf, u), hi + r


def gate_share(got, lo, ref, hi):
    """Largest share of its half-gate a result used (> 1: outside the gate)."""
    got = np.asarray(got, F64)
    up = np.where(got >= ref, (got - ref) / np.maximum(hi - ref, 1e-300), (ref - got) / np.maximum(ref - lo, 1e-300))
    return float(up.max()) if up.size else 0.0


def inside(got, lo, hi):
    got = np.asarray(got, F64)
    return bool(((got >= lo) & (got <= hi)).all())


def pdf_inputs(n, n_bins, K, seed):
    """bins (n, n_bins), weights (n, n_bins - 1), u (n, K), fp32.  Planted rows: 0 all zero, 1 one-hot, 2 summing to
    about 1 with empty stretches (the guard is active there), 3 an empty tail, 4 zero-width bins; planted u (cycling
    over rows and draws): 0, 1 - 2^-24, the middle of a guarded bin, and draws moved more than 4 delta away from every
    float64 cdf knot."""
    rng = np.random.default_rng(seed)
    M = n_bins - 1
    w = (rng.random((n, M)) ** 4).astype(F32)
    near = rng.uniform(0.1, 0.3, (n, 1))
    bins = (near + np.sort(rng.random((n, n_bins)), -1) * 2.5).astype(F32)
    if M > 0 and n >= 5:
        w[0] = 0.0
        w[1] = 0.0
        w[1, M // 2] = 1.0
        row = rng.random(M)
        row[M // 5: M // 5 + max(M // 4, 1)] = 0.0
        row[-max(M // 6, 1):] = 0.0
        w[2] = (row / max(row.sum(), 1e-30)).astype(F32)
        w[3, max(M // 3, 1):] = 0.0
    if n_bins > 1 and n >= 5:
        bins[4, 1::3] = bins[4, 0::3][: bins[4, 1::3].shape[0]]           # repeated edges: zero-width bins
        bins[4] = np.sort(bins[4])
    cdf = cdf64_of(w)
    delta = pdf_delta(M)
    u = rng.random((n, K)).astype(F32)
    for r in range(n):
        knots = cdf[r]
        guarded = np.nonzero(np.diff(knots) < EPS - 4 * delta)[0]
        for k in range(K):
            kind = (r + k) % 5
            if kind == 0:
                u[r, k] = 0.0
            elif kind == 1:
                u[r, k] = F32(1 - U24)
            elif kind == 2 and len(guarded):
                j = guarded[(r * 7 + k) % len(guarded)]
                u[r, k] = F32(0.5 * (knots[j] + knots[j + 1]))
            else:
                for _ in range(100):
                    if np.abs(knots - F64(u[r, k])).min() > 4 * delta:
                        break
                    u[r, k] = F32(rng.random())
    return bins, w, u


def merge_inputs(n, S, K, seed):
    """Coarse depths (jittered, ascending), coarse weights (n, S) with the planted pdf rows of pdf_inputs in
    weights[:, 1:-1], and injected u (n, K)."""
    rays = coarse_rays(n, seed)
    z = coarse_depth32(rays, S, perturb=1.0, jitter=coarse_jitter(n, S, seed + 1))
    _, w_in, u = pdf_inputs(n, S - 1, K, seed + 2)
    w = np.random.default_rng(seed + 3).random((n, S)).astype(F32)
    w[:, 1:S - 1] = w_in
    return z, w, u


def merge_reference(z, w, u_pdf):
    """The fused kernel's bins, fp32 mid-points __fmul_rn(0.5, a + b), and the sorted union of the coarse depths with
    a given set of importance samples: what the fused output must equal bit for bit."""
    z = np.asarray(z, F32)
    mid = (F32(0.5) * (z[:, :-1] + z[:, 1:])).astype(F32)
    return mid, np.sort(np.concatenate([z, np.asarray(u_pdf, F32)], 1), 1)


# ------------------------------------------------------------------------------------------------
# compositing
# ------------------------------------------------------------------------------------------------
# per-factor error of the kernel's t_j = (1 - alpha_j) + 1e-10, alpha_j = 1 - expf(-delta_j relu(s_j)), in units of
# 2^-22: the delta rounding and the product delta s are relative u each on x = delta s, which moves e^-x by at most
# 2 u x e^-x <= 2 u / e; expf is within 2 ulp (2^-23 absolute on [0, 1]); 1 - e, 1 - alpha and + 1e-10 round once
# each (<= 2^-25 absolute).  Sum: (2 / e + 2 + 3 / 2) u = 4.24 u = 1.06 2^-22; C_T = 1.25 leaves margin.
C_T = 1.25
E_T = C_T * 2.0 ** -22
TINY = 2.0 ** -140           # subnormal results round to 2^-149 absolute


def composite64(z, sigma, rgb, last_delta, noise=None, noise_std=0.0, mask=None):
    """alpha_weights + composite of the oracle in float64 on the fp32 inputs; the noised sigma s + n std is the kernel's
    two fp32 roundings.  -> dict(alpha, t, T, w, opacity, rgb (unscaled sums), depth)."""
    z = np.asarray(z, F32)
    s = np.asarray(sigma, F32)
    if noise_std > 0:
        s = s + np.asarray(noise, F32) * F32(noise_std)
    z64 = z.astype(F64)
    delta = np.concatenate([np.diff(z64, axis=1), np.full((z.shape[0], 1), float(last_delta))], 1)
    x = delta * np.maximum(s.astype(F64), 0.0)
    alpha = -np.expm1(-x)
    if mask is not None:
        alpha = np.where(mask, 0.0, alpha)
    t = 1.0 - alpha + 1e-10
    T = np.cumprod(np.concatenate([np.ones((z.shape[0], 1)), t[:, :-1]], 1), 1)
    w = alpha * T
    c = np.asarray(rgb, F32).astype(F64)
    return dict(alpha=alpha, t=t, T=T, w=w, opacity=w.sum(1), rgb=(w[..., None] * c).sum(1), depth=(w * z64).sum(1))


def composite_gate(ref, rgb, z, white):
    """A-priori error bounds of the kernel's weights and maps against composite64.
    Weights: each kernel factor is within E_T of t_j (all in [0, 1 + 1e-10]), so the product of the first i lies within
    U_i - T_i of T_i, U_i = prod (t_j + E_T) (the product is multilinear with non-negative coefficients; for transparent
    rays this is i E_T, the sum of the factor errors, and it shrinks where the ray turns opaque); the i products and
    alpha carry relative (i + 2) u.  So |w_i~ - w_i| <= (alpha_i + E_T)(U_i - T_i) + E_T T_i + (i + 2) u U_i (alpha_i + E_T).
    Maps sum_i w_i v_i (v = 1, rgb, z): sum_i g_i |v_i| for the weights, plus (ceil(S / 32) + 6) u sum_i (|w_i| + g_i)
    |v_i| for the per-lane sums, the butterfly and the products; the white background adds the opacity bound and two
    roundings."""
    t, T, a = ref["t"], ref["T"], ref["alpha"]
    n, S = t.shape
    Up = np.cumprod(np.concatenate([np.ones((n, 1)), t[:, :-1] + E_T], 1), 1)
    i = np.arange(S)[None, :]
    g = (a + E_T) * (Up - T) + E_T * T + (i + 2) * U24 * Up * (a + E_T) + TINY
    sum_r = (math.ceil(S / 32) + 6) * U24
    c = np.abs(np.asarray(rgb, F32).astype(F64))
    zz = np.abs(np.asarray(z, F32).astype(F64))
    wa = np.abs(ref["w"]) + g
    op = g.sum(1) + sum_r * wa.sum(1) + TINY
    out = dict(w=g, opacity=op,
               rgb=(g[..., None] * c).sum(1) + sum_r * (wa[..., None] * c).sum(1) + TINY,
               depth=(g * zz).sum(1) + sum_r * (wa * zz).sum(1) + TINY)
    if white:
        out["rgb"] = out["rgb"] + op[:, None] + 2 * U24 * (np.abs(ref["rgb"]) + 1 + np.abs(ref["opacity"])[:, None])
    return out


def composite_inputs(n, S, seed):
    """z ascending in (near, far), sigma / object sigma ~ 5 N(0, 1), rgb in (0, 1), noise N(0, 1), pass-through flags.
    Planted rows: 0 negative sigma, 1 sigma = -1e5, 2 opaque at its first sample, 3 equal neighbouring depths
    (delta = 0), 4 five opaque samples in a row (transmittance 1e-10, 1e-20, ... into the subnormals and to 0)."""
    rng = np.random.default_rng(seed)
    rays = synth.random_rays(seed, n).numpy()
    near, far = rays[:, 6:7].astype(F64), rays[:, 7:8].astype(F64)
    z = (near + (far - near) * np.sort(rng.random((n, S)), -1)).astype(F32)
    f = lambda *sh: rng.standard_normal(sh).astype(F32)
    sig, isig = f(n, S) * F32(5), f(n, S) * F32(5)
    for s in (sig, isig):
        s[0] = -np.abs(s[0])
        s[1] = -1e5
        s[2, 0] = 1e6
        s[4, S // 3: S // 3 + 5] = 1e6
    z[3, 1::2] = z[3, 0::2][: z[3, 1::2].shape[0]]         # (a no-op for S = 1)
    z[3] = np.sort(z[3])
    sig[4, 0] = isig[4, 0] = 0.5
    return dict(z=z, sigma=sig, isigma=isig, rgb=1 / (1 + np.exp(-f(n, S, 3))), irgb=1 / (1 + np.exp(-f(n, S, 3))),
                ns=f(n, S), no=f(n, S), ptm=rng.random((n, 1)) < 0.5)


def composite_refs(c, mode_kw, scene_depth):
    """composite64 of both branches for one COMPOSITE_MODES entry.  The occlusion mask is formed the kernel's way from
    the scene depth the kernel itself produced (fl(depth + th) < z, pass-through rays exempt): a depth within its gate
    may still sit on either side of a sample, so the mask is an input of the object branch here, not a result.
    -> {map name: (ref, gate)} plus "weights"."""
    kw = dict(mode_kw)
    fi = kw.get("forward_instance", True)
    noise = kw.get("noise_std", 0.0)
    white = kw.get("white_back", False)
    sc = composite64(c["z"], c["sigma"], c["rgb"], 0.0 if kw.get("zero_last_delta") else 1e10, c["ns"], noise)
    gs = composite_gate(sc, c["rgb"], c["z"], white)
    out = {"opacity": (sc["opacity"], gs["opacity"]), "depth": (sc["depth"], gs["depth"]),
           "rgb": (sc["rgb"] + (1 - sc["opacity"][:, None] if white else 0), gs["rgb"])}
    wmap = (sc["w"], gs["w"])
    if fi:
        mask = None
        th = kw.get("frustum_bound_th", 0.0)
        if not kw.get("is_eval", True) and th > 0:
            lim = (np.asarray(scene_depth, F32) + F32(th)).astype(F32)
            mask = lim[:, None] < c["z"]
            if kw.get("pass_through_mask"):
                mask &= ~c["ptm"]
        ob = composite64(c["z"], c["isigma"], c["irgb"], 0.0, c["no"], noise, mask)
        go = composite_gate(ob, c["irgb"], c["z"], True)
        out.update(opacity_instance=(ob["opacity"], go["opacity"]), depth_instance=(ob["depth"], go["depth"]),
                   rgb_instance=(ob["rgb"] + 1 - ob["opacity"][:, None], go["rgb"]))
        if kw.get("rays_in_bbox"):
            wmap = (ob["w"], go["w"])
    out["weights"] = wmap
    return out


def oracle_composite32(c, mode_kw):
    """torch's float32 composite_pass (the oracle) on the same inputs -> {kernel map name: array}."""
    kw = dict(mode_kw)
    fi = kw.pop("forward_instance", True)
    use_ptm = kw.pop("pass_through_mask", False)
    noise = kw.get("noise_std", 0.0) > 0
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    ref = {}
    O.composite_pass(ref, "x", T(c["sigma"]), T(c["rgb"]), T(c["isigma"]) if fi else None, T(c["irgb"]) if fi else None,
                     T(c["z"]), forward_instance=fi, pass_through_mask=T(c["ptm"]) if use_ptm else None,
                     noise_scene=T(c["ns"]) if noise else None, noise_obj=T(c["no"]) if noise else None,
                     **{"is_eval": True, **kw})
    return {k[:-2]: v.numpy() for k, v in ref.items() if k.endswith("_x") and not k.startswith("z_vals")}


def composite_modes():
    from tests.test_gpu_train_stages import COMPOSITE_MODES
    return COMPOSITE_MODES


# ------------------------------------------------------------------------------------------------
# checks of the references
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", COARSE_S)
def test_coarse_depth32_is_the_oracle_bit_for_bit(S):
    """coarse_depth32 equals O.stratified_z (torch's fp32 ops) bit for bit, with and without use_disp and jitter, given
    torch's linspace.  torch's CPU linspace itself is not linspace01: it fuses the upper half's multiply-add, so for
    S in {31, 64, 100, 128, 1000, 2048} some t above 1/2 differ by one ulp (5 of 64 at S = 64); linspace01_fma32
    reproduces it exactly, and both agree below n / 2 and wherever the two roundings happen to coincide.  The kernel
    keeps the two roundings (its depths are compared with coarse_depth32, not with torch).  The float64 formula is within
    a few ulp; the one-sided linspace differs from linspace01 for S >= 4 (for S <= 3 both formulas are exact)."""
    n = 37
    rays = coarse_rays(n, S)
    jit = coarse_jitter(n, S, S + 1)
    R, J = torch.from_numpy(rays), torch.from_numpy(jit)
    t_torch = torch.linspace(0, 1, S).numpy()
    assert np.array_equal(linspace01_fma32(S), t_torch)
    same = linspace01_32(S) == t_torch
    assert same[: S // 2].all() and (same.all() or S in (31, 64, 100, 128, 1000, 2048))
    for use_disp in (False, True):
        for perturb in (0.0, 1.0):
            got = coarse_depth32(rays, S, use_disp, perturb, jit)
            ref = O.stratified_z(R, S, use_disp, perturb, J).numpy()
            ok = disp_ok(rays) if use_disp else np.ones(n, bool)
            assert np.array_equal(coarse_depth32(rays, S, use_disp, perturb, jit, t=t_torch)[ok], ref[ok])
            cols = same if perturb == 0 else (same & np.roll(same, 1) & np.roll(same, -1))
            assert np.array_equal(got[ok][:, cols], ref[ok][:, cols]), (use_disp, perturb)
            z64 = coarse_depth64(rays, S, use_disp, perturb, jit)
            ulp = np.spacing(np.abs(z64[ok]).astype(F32)).astype(F64)
            assert (np.abs(got[ok] - z64[ok]) <= ULP_64 * ulp + 1e-30).all(), (use_disp, perturb)
    if S >= 4 and (S - 1) & (S - 2):        # 1 / (S - 1) is exact when S - 1 is a power of two: both formulas are
        assert not np.array_equal(linspace01_32(S, one_sided=True), linspace01_32(S))


def test_pdf_reference_is_the_oracle_in_float64():
    """sample_pdf64 on cdf64_of(weights) is O.sample_pdf run in float64 (on the fp32-rounded weights + eps)."""
    bins, w, u = pdf_inputs(N_PLANT, 63, 33, 5)
    wts = torch.from_numpy((w + EPS32).astype(F64) - EPS)       # + eps in float64 gives back the fp32 sum
    ref = O.sample_pdf(torch.from_numpy(bins.astype(F64)), wts, 33, u=torch.from_numpy(u.astype(F64)), eps=EPS).numpy()
    got = sample_pdf64(bins, cdf64_of(w), u)
    assert np.allclose(got, ref, rtol=0, atol=1e-12)


def _pdf_cases():
    for nb, k in PDF_SHAPES:
        yield f"pdf_{nb}x{k}", pdf_inputs(N_PLANT, nb, k, nb * 1000 + k)
    for S, K in MERGE_SHAPES:
        for n in (1, N_PLANT) + ((9000,) if (S, K) in MERGE_MANY_RAYS else ()):
            z, w, u = merge_inputs(n, S, K, S * 1000 + K + n)
            mid, _ = merge_reference(z, w, np.zeros((n, 0), F32))
            yield f"merge_{S}x{K}_n{n}", (mid, w[:, 1:-1], u)


def test_torch_fp32_sample_pdf_lies_inside_the_gates():
    """Soundness: torch's float32 sample_pdf (a second fp32 implementation: vectorised normaliser, cumsum in double)
    inside pdf_gate on every pdf and merge input set of the device tests, with injected u and with det = 1."""
    worst = 0.0
    for name, (bins, w, u) in _pdf_cases():
        K = u.shape[1]
        B, W = torch.from_numpy(bins), torch.from_numpy(w)
        for det in (False, True):
            uu = np.broadcast_to(linspace01_32(K), u.shape).copy() if det else u
            got = O.sample_pdf(B, W, K, det=det, u=torch.from_numpy(uu)).numpy()
            lo, ref, hi = pdf_gate(bins, w, uu)
            share = gate_share(got, lo, ref, hi)
            worst = max(worst, share)
            assert inside(got, lo, hi), (name, det, share)
    print(f"RATIO torch fp32 sample_pdf in pdf_gate: {worst:.3e}")


def test_pdf_gate_rejects_the_mutants():
    """Discrimination: without the denominator guard the planted rows' samples leave the gate.  searchsorted left and a
    guard at <= differ from the reference only where u equals a cdf knot, or a denominator equals eps, exactly; the gate
    has to leave those ties undecided whenever the cdf carries rounding (u = 1 against a last knot of 1 +- 1 ulp is the
    reference's own knife edge).  They are checked on a planted exact cdf (delta = 0): a guarded bin ending at a knot
    that u hits, and a bin exactly eps wide."""
    bins, w, u = pdf_inputs(N_PLANT, 200, 64, 11)
    cdf = cdf64_of(w)
    lo, ref, hi = pdf_gate(bins, w, u)
    assert inside(ref, lo, hi)
    assert not inside(sample_pdf64(bins, cdf, u, guard="none"), lo, hi)
    # bins: [0, 0.5 - eps) normal, [0.5 - eps, 0.5) exactly eps wide (0.5 - eps is exact in float64), then a guarded
    # bin 0.4 eps wide whose end knot u hits exactly
    ex_cdf = np.array([[0.0, 0.5 - EPS, 0.5, 0.5 + 0.4 * EPS, 0.75, 1.0]])
    assert ex_cdf[0, 2] - ex_cdf[0, 1] == EPS
    ex_bins = np.array([[0.0, 1.0, 2.0, 3.0, 4.0, 5.0]], F32)
    ex_u = np.array([[0.5 - EPS / 2, 0.5 + 0.4 * EPS, 0.5 + 0.2 * EPS]])
    lo, ref, hi = pdf_gate(ex_bins, None, ex_u, cdf=ex_cdf, delta=0.0)
    assert inside(ref, lo, hi)
    assert not inside(sample_pdf64(ex_bins, ex_cdf, ex_u, guard="le"), lo, hi)
    assert not inside(sample_pdf64(ex_bins, ex_cdf, ex_u, side="left"), lo, hi)


def test_one_sided_linspace_is_rejected_bit_for_bit():
    """The one-sided linspace mutant changes coarse depths that the bit-for-bit comparison of the device test rejects."""
    rays = coarse_rays(N_PLANT, 3)
    for S in (64, 1000, 2048):
        assert not np.array_equal(coarse_depth32(rays, S), coarse_depth32(rays, S, one_sided=True))


@pytest.mark.parametrize("S", COMPOSITE_S)
def test_torch_fp32_composite_lies_inside_the_gates(S):
    """Soundness: torch's float32 composite_pass inside composite_gate, per weight and per map, for every
    COMPOSITE_MODES entry on the device test's inputs (object mask from torch's own scene depth)."""
    c = composite_inputs(N_PLANT, S, seed=S + 101)
    worst = {}
    for mode, kw in composite_modes().items():
        got = oracle_composite32(c, kw)
        refs = composite_refs(c, kw, got["depth"])
        for k, (ref, g) in refs.items():
            share = float((np.abs(got[k].astype(F64) - ref) / g).max())
            worst[k] = max(worst.get(k, 0.0), share)
            assert share <= 1.0, (mode, k, share)
    print(f"RATIO torch fp32 composite S={S}: " + ", ".join(f"{k} {v:.2e}" for k, v in sorted(worst.items())))


def test_torch_fp32_composite_lies_inside_the_gates_many_rays():
    """Soundness on the device test's 9 000-ray input set (S = 33, training flags)."""
    c = composite_inputs(9000, 33, seed=33 + 202)
    kw = composite_modes()["train_noise_mask"]
    got = oracle_composite32(c, kw)
    for k, (ref, g) in composite_refs(c, kw, got["depth"]).items():
        assert (np.abs(got[k].astype(F64) - ref) <= g).all(), k


def test_composite_gate_rejects_a_non_strict_occlusion_mask():
    """Discrimination: on a planted occlusion edge (fl(depth + th) == z_k exactly, sample k with positive object sigma
    and delta), masking with <= zeroes sample k's object weight, which the gate refuses."""
    c = composite_inputs(N_PLANT, 64, seed=9)
    r = 10
    depth = composite64(c["z"], c["sigma"], c["rgb"], 1e10)["depth"].astype(F32)
    k, th = occlusion_edge(depth[r], c["z"][r])
    c["isigma"][r, k] = 3.0
    lim = (depth + F32(th)).astype(F32)
    good = composite64(c["z"], c["isigma"], c["irgb"], 0.0, mask=lim[:, None] < c["z"])
    bad = composite64(c["z"], c["isigma"], c["irgb"], 0.0, mask=lim[:, None] <= c["z"])
    g = composite_gate(good, c["irgb"], c["z"], True)["w"]
    assert good["w"][r, k] > 0 and bad["w"][r, k] == 0
    assert abs(bad["w"][r, k] - good["w"][r, k]) > g[r, k]


def occlusion_edge(depth, z):
    """A sample k beyond the scene depth and a threshold th > 0 with fl(depth + th) == z_k exactly in fp32, such that
    z_k has a positive delta to the next sample.  -> (k, th as float32)."""
    depth = F32(depth)
    z = np.asarray(z, F32)
    for k in range(len(z) - 2, -1, -1):
        if not (z[k] > depth and z[k + 1] > z[k]):
            continue
        th = F32(z[k] - depth)
        for _ in range(8):
            s = F32(depth + th)
            if s == z[k] and th > 0:
                return k, th
            th = np.nextafter(th, F32(np.inf) if s < z[k] else F32(-np.inf))
    raise AssertionError("no sample with an exact occlusion edge")


# ------------------------------------------------------------------------------------------------
# argument checks of the library, reachable without a device
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def test_render_forward_refuses_more_than_2048_samples_up_front(lib):
    """onerf_render_rays_fwd with S + K = 2049 returns ONERF_ERR_UNSUPPORTED before it looks at anything else (here:
    dummy pointers and a dummy context, so any later step would fail differently); without importance samples the
    fine-pass limit does not apply and the call goes on to the next check."""
    from object_nerf_b200 import _lib
    a = _lib.RenderArgs()
    a.rays, a.packed_coarse, a.packed_fine = 16, 16, 16
    a.n_rays, a.n_samples, a.n_importance = 4, 1025, 1024
    assert lib.onerf_render_rays_fwd(ctypes.c_void_p(1), ctypes.byref(a), None) == -2
    assert b"2048" in lib.onerf_last_error()
    a.n_samples, a.n_importance = 2049, 0
    assert lib.onerf_render_rays_fwd(ctypes.c_void_p(1), ctypes.byref(a), None) == -1
    assert b"null coarse output map" in lib.onerf_last_error()


def test_train_step_refuses_more_than_2048_samples_before_any_cuda_call(lib):
    """onerf_train_step with S + K = 2049 and otherwise complete (dummy) arguments: ONERF_ERR_UNSUPPORTED before the
    first CUDA call (there is no device here)."""
    from object_nerf_b200 import _lib
    a, la, b = _lib.RenderArgs(), _lib.LossArgs(), _lib.RenderBwdArgs()
    a.rays, a.packed_coarse, a.packed_fine, a.codes, a.train_ws = 16, 16, 16, 16, 1024
    a.n_rays, a.n_samples, a.n_importance, a.forward_instance = 4, 1025, 1024, 1
    a.precision = _lib.PREC_FP32
    la.n_rays, la.has_fine = 4, 1
    la.rgbs = la.depths = la.valid_mask = la.instance_mask = la.instance_mask_weight = 16
    la.loss_sum_out = la.terms_out = la.present_out = 16
    ptrs = (ctypes.c_void_p * 20)(*([16] * 20))
    b.W_coarse, b.dW_coarse, b.db_coarse, b.W_fine, b.dW_fine, b.db_fine = (ptrs,) * 6
    psnr = ctypes.c_float()
    args = (ctypes.c_void_p(1), ctypes.byref(a), ctypes.byref(la), ctypes.byref(b), ctypes.addressof(psnr), None)
    assert lib.onerf_train_step(*args) == -2
    assert b"2048" in lib.onerf_last_error()
