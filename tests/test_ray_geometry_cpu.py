"""References for camera rays and the ray-box slab test (tests/test_gpu_ray_geometry.py), the planted geometry those tests
use, and the checks of the references that need no device.

  - exact_ray: one ray through utils/bbox_utils.py:102-156 and datasets/geo_utils.py:126-162 in exact rational arithmetic
    (fractions.Fraction) from the fp32 inputs: the unscale is the fp32 product, the float64 matrices and bounds are exact
    values, a box-frame direction component that is exactly zero becomes 1e-14 (its inverse the float64 1 / 1e-14).
    Next to every value it carries a bound beta on how far ANY float64 evaluation of the same formula can be from it
    (any association, with or without FMA contraction: numpy / numba on the reference's side, DFMA on the kernel's),
    and 0 where every evaluation is exact;
  - slab64: the same path vectorised in float64 in one fixed order, with the same bounds, flagging every ray on which a
    decision or an fp32 rounding is closer than 2 beta; it also takes the mutants of the discrimination checks;
  - reference: slab64 for every ray, exact_ray for the flagged ones and a sample;
  - slab_verdict: on a decidable ray (every decision's margin above its bounds, or an exact tie computed exactly, and
    neither t within beta of an fp32 rounding boundary) the hit and near / far = fp32(fp32(t) / fp32(scale)) bit for bit,
    sign of zero included; a knife-edge ray may take either decision or either neighbouring value.
Camera rays: directions bit for bit against a numpy float32 restatement, rays_o = c2w[:, 3] bit for bit, rays_d inside
ROT_C 2^-24 (|d_i| + sum_j |r_ij x_j| / ||w||) of the float64 rotate-and-normalise."""
import math
from fractions import Fraction as Fr

import numpy as np
import pytest
import torch

from oracle import onerf_oracle as O
from oracle import ref_loader
from tests import cases

F32, F64 = np.float32, np.float64
U64 = 2.0 ** -53                         # float64 unit roundoff
INFL = 1 + 2.0 ** -40                    # bounds are evaluated in float64: this covers their own rounding
ZERO_DIR = 1.0e-14                       # geo_utils.py:131
INV_ZERO = Fr(1 / ZERO_DIR)              # the float64 value of 1 / 1e-14
F32_OVERFLOW = Fr(2 ** 128 - 2 ** 103)   # fp32 rounding gives inf from here (FLT_MAX and 2^128's midpoint, ties to even)
MUTANTS = ("slab_fp32", "reject_ge", "inside_le", "zero_plus_only", "dir_pose_avg")


def gamma(n):
    """gamma_n = n u / (1 - n u): a float64 sum of n products (or exact terms) evaluated in any association, with or
    without FMA contraction, is within gamma_n sum |terms| of the exact sum (Higham, Accuracy and Stability of Numerical
    Algorithms, 2nd ed., section 3.1; an FMA removes roundings, so it only tightens the count)."""
    return n * U64 / (1 - n * U64)


class Box:
    """A box as BBoxRayHelper holds it (utils/bbox_utils.py): pose_avg and axis_align_mat (4, 4) float64, bbox_bounds
    (2, 3) float64 before the enlarge, the scale factor and the enlarge the caller passes."""

    def __init__(self, pose_avg, axis_align_mat, bbox_bounds, scale_factor, bbox_enlarge=0.0):
        self.pose_avg = np.asarray(pose_avg, F64)
        self.axis_align_mat = np.asarray(axis_align_mat, F64)
        self.bbox_bounds = np.array(bbox_bounds, F64)
        self.scale_factor = float(scale_factor)
        self.bbox_enlarge = float(bbox_enlarge)

    def bounds(self):
        b = self.bbox_bounds.copy()
        if self.bbox_enlarge > 0:                 # utils/bbox_utils.py:140-145, in float64
            b[0] -= self.bbox_enlarge
            b[1] += self.bbox_enlarge
        return b


def rigid(R=None, t=(0.0, 0.0, 0.0)):
    T = np.eye(4)
    if R is not None:
        T[:3, :3] = R
    T[:3, 3] = t
    return T


def yaw(theta):
    c, s = math.cos(theta), math.sin(theta)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


# ------------------------------------------------------------------------------------------------
# exact reference, one ray
# ------------------------------------------------------------------------------------------------
def _is_f64(x):
    try:
        return Fr(float(x)) == x
    except OverflowError:
        return False


def _exact_sum(terms):
    """True when every partial sum of every subset of `terms` is a float64, so any association and any FMA contraction
    evaluates the sum exactly: dyadic terms whose magnitudes add up to less than 2^53 units of the finest one."""
    nz = [t for t in terms if t]
    if not nz:
        return True
    den = max(t.denominator for t in nz)
    if den & (den - 1) or den > 2 ** 1022:
        return False
    return sum(abs(t.numerator) * (den // t.denominator) for t in nz) < 2 ** 53


def _dot(c, x, xe, const=None):
    """sum_j c_j x_j (+ const) where x_j is known to within xe_j: exact value and its bound.  c and const are exact
    float64 values; the evaluated inputs x^_j then give terms c_j x^_j whose magnitudes are at most |c_j| (|x_j| + xe_j)."""
    terms = [ci * xi for ci, xi in zip(c, x)] + ([const] if const is not None else [])
    v = sum(terms, Fr(0))
    if not any(xe) and _exact_sum(terms):
        return v, 0.0
    cf, xf = [abs(float(ci)) for ci in c], [abs(float(xi)) for xi in x]
    prop = sum(ci * ei for ci, ei in zip(cf, xe))
    mag = sum(ci * (xi + ei) for ci, xi, ei in zip(cf, xf, xe)) + (abs(float(const)) if const is not None else 0.0)
    return v, (prop + gamma(len(terms)) * mag) * INFL


def round32(x, negzero=False):
    """The fp32 nearest to the rational x (ties to even), -0.0 for a zero that carries a negative sign."""
    if x == 0:
        return F32(-0.0) if negzero else F32(0.0)
    if abs(x) >= F32_OVERFLOW:
        return F32(np.inf) if x > 0 else F32(-np.inf)
    f = F32(float(x))
    best = None
    for c in (np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))):
        if not np.isfinite(c):
            continue
        key = (abs(Fr(float(c)) - x), int(np.array(c).view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return best[1]


def bits(x):
    return int(np.array(x, F32).view(np.uint32))


class _T:
    """A float64 quantity of the slab test: exact value v (Fraction), bound e (float, 0 when every evaluation is exact),
    and the sign of an exact zero."""
    __slots__ = ("v", "e", "neg")

    def __init__(self, v, e, neg=False):
        self.v, self.e, self.neg = v, e, neg


def _gt(x, y):
    """x > y as float64 computes it: True / False when certain, None on a knife edge; with the margin."""
    m = x.v - y.v
    if (x.e == 0 and y.e == 0) or abs(m) > x.e + y.e:
        return m > 0, m
    return None, m


def _or(a, b):
    if a is True or b is True:
        return True
    return None if (a is None or b is None) else False


class ExactBox:
    def __init__(self, box: Box):
        P, A, b = box.pose_avg, box.axis_align_mat, box.bounds()
        self.Ra = [[Fr(float(P[i, j])) for j in range(3)] for i in range(3)]
        self.ta = [Fr(float(P[i, 3])) for i in range(3)]
        self.Rb = [[Fr(float(A[i, j])) for j in range(3)] for i in range(3)]
        self.tb = [Fr(float(A[i, 3])) for i in range(3)]
        self.lo = [Fr(float(b[0, i])) for i in range(3)]
        self.hi = [Fr(float(b[1, i])) for i in range(3)]
        self.s32 = F32(box.scale_factor)


def exact_ray(eb: ExactBox, o, d):
    """One ray (fp32 o, d at NeRF scale) through the box: dict(hit_sure, hit, sure, near, far, near_lo, near_hi, far_lo,
    far_hi, tmin, tmax, decisions).  decisions: (name, outcome or None, exact margin, bound) in evaluation order."""
    dec = []
    knife = dict(hit_sure=False, hit=False, sure=False, decisions=dec)
    os_ = [Fr(float(F32(o[i]) * eb.s32)) for i in range(3)]            # fp32 unscale (:108), exact once formed
    p = [_dot(eb.Ra[i], os_, (0, 0, 0), eb.ta[i]) for i in range(3)]   # de-centre (:111)
    pv, pe = [x[0] for x in p], [x[1] for x in p]
    q = [_dot(eb.Rb[i], pv, pe, eb.tb[i]) for i in range(3)]           # to the box frame (:115)
    dd = [Fr(float(d[i])) for i in range(3)]
    db = [_dot(eb.Rb[i], dd, (0, 0, 0)) for i in range(3)]             # the direction by axis_align only (:116)
    slabs = []
    for i in range(3):
        di, Ed = db[i]
        if di == 0:
            if Ed:                       # the evaluated component may be a tiny non-zero: the 1e-14 rule is undecided
                dec.append((f"d{i} == 0", None, Fr(0), Ed))
                return knife
            inv, Ei, neg = INV_ZERO, 0.0, False
        else:
            ok = abs(di) > Ed
            dec.append((f"sign d{i}", (di < 0) if ok else None, abs(di), Ed))
            if not ok:
                return knife
            inv, neg = 1 / di, di < 0
            rho = Ed / abs(float(di)) * INFL
            # 1 / d^ = (1 / d) / (1 + (d^ - d) / d): relative error rho / (1 - rho), then one rounding of the quotient
            Ei = 0.0 if (Ed == 0 and _is_f64(inv)) else (rho + U64) / (1 - rho) * abs(float(inv)) * INFL
        qv, Eq = q[i]
        ts = []
        for B in ((eb.hi[i], eb.lo[i]) if neg else (eb.lo[i], eb.hi[i])):
            a = B - qv
            Ea = 0.0 if (Eq == 0 and _is_f64(a)) else (Eq + U64 * (abs(float(a)) + Eq)) * INFL
            t = a * inv
            if Ea == 0 and Ei == 0 and _is_f64(t):
                Et = 0.0
            else:
                af, invf = abs(float(a)), abs(float(inv))
                Et = (af * Ei + Ea * invf + Ea * Ei + U64 * (af + Ea) * (invf + Ei)) * INFL
            ts.append(_T(t, Et, neg=(t == 0 and neg)))   # (B - q) is +0 when equal; times a negative inverse: -0.0
        slabs.append(ts)
    tmin, tmax = slabs[0]
    for k, name in ((1, "y"), (2, "z")):
        lo_k, hi_k = slabs[k]
        r1, m1 = _gt(tmin, hi_k)
        r2, m2 = _gt(lo_k, tmax)
        dec += [(f"tmin > t{name}max", r1, m1, tmin.e + hi_k.e), (f"t{name}min > tmax", r2, m2, lo_k.e + tmax.e)]
        rej = _or(r1, r2)
        if rej is True:
            return dict(hit_sure=True, hit=False, sure=True, near=F32(0), far=F32(0), decisions=dec)
        if rej is None:
            return knife
        # max / min: |max(x^, y^) - max(x, y)| <= max(ex, ey) whichever way a close comparison goes
        g, _ = _gt(lo_k, tmin)
        tmin = lo_k if g is True else (tmin if g is False else _T(max(tmin.v, lo_k.v), max(tmin.e, lo_k.e)))
        g, _ = _gt(tmax, hi_k)
        tmax = hi_k if g is True else (tmax if g is False else _T(min(tmax.v, hi_k.v), max(tmax.e, hi_k.e)))
    zero = _T(Fr(0), 0.0)
    r1, m1 = _gt(zero, tmin)
    r2, m2 = _gt(zero, tmax)
    dec += [("tmin < 0", r1, -m1, tmin.e), ("tmax < 0", r2, -m2, tmax.e)]
    inside = _or(r1, r2)
    out = dict(tmin=tmin, tmax=tmax, decisions=dec)
    if inside is True:
        return dict(out, hit_sure=True, hit=False, sure=True, near=F32(0), far=F32(0))
    if inside is None:
        return dict(out, hit_sure=False, hit=False, sure=False)
    out.update(hit_sure=True, hit=True)
    for k, t in (("near", tmin), ("far", tmax)):
        if t.e == 0:
            lo = hi = round32(t.v, t.neg)
        else:
            lo, hi = round32(t.v - Fr(t.e)), round32(t.v + Fr(t.e))
        out[k + "_lo"], out[k + "_hi"] = F32(lo / eb.s32), F32(hi / eb.s32)
        out[k] = out[k + "_lo"]
    out["sure"] = bits(out["near_lo"]) == bits(out["near_hi"]) and bits(out["far_lo"]) == bits(out["far_hi"])
    return out


# ------------------------------------------------------------------------------------------------
# float64 pass, vectorised (and the mutants)
# ------------------------------------------------------------------------------------------------
def _row(R, i, x, y, z):
    return (R[i, 0] * x + R[i, 1] * y) + R[i, 2] * z


def _f32_boundary_dist(t):
    """Distance from each float64 t to the nearest fp32 rounding boundary (a midpoint of adjacent fp32 values, or the
    overflow threshold)."""
    big = float(F32_OVERFLOW)
    with np.errstate(over="ignore", invalid="ignore"):
        f = t.astype(F32)
        lo = np.nextafter(f, F32(-np.inf)).astype(F64)
        hi = np.nextafter(f, F32(np.inf)).astype(F64)
        f64 = f.astype(F64)
        lo = np.where(np.isinf(lo), -2.0 ** 128, lo)
        hi = np.where(np.isinf(hi), 2.0 ** 128, hi)
        d = np.minimum(np.abs(t - (f64 + lo) / 2), np.abs(t - (f64 + hi) / 2))
        d = np.where(np.isinf(f), np.abs(t) - big, d)
    return np.where(np.isfinite(d), d, 0.0)


def slab64(o, d, box: Box, mutant=None):
    """The slab test for (n, 3) fp32 o, d in float64, sums left to right, no FMA; returns dict(hit, near, far) as the
    kernel writes them, tmin / tmax and their bounds, and `flag`: rays with a decision or an fp32 rounding closer than
    2 beta, which exact_ray settles.  The bounds are exact_ray's, evaluated in float64 and inflated by 2^-30 for their own
    rounding.  `mutant` (one of MUTANTS) changes the arithmetic for the discrimination checks."""
    o, d = np.asarray(o, F32), np.asarray(d, F32)
    n = o.shape[0]
    s32 = F32(box.scale_factor)
    P, A, b = box.pose_avg, box.axis_align_mat, box.bounds()
    Ra, ta, Rb, tb = P[:3, :3], P[:3, 3], A[:3, :3], A[:3, 3]
    g3, g4 = 3 * U64 / (1 - 3 * U64), 4 * U64 / (1 - 4 * U64)
    os_ = (o * s32).astype(F64)
    p = [_row(Ra, i, *os_.T) + ta[i] for i in range(3)]
    Ep = [g4 * ((np.abs(Ra[i]) * np.abs(os_)).sum(1) + abs(ta[i])) for i in range(3)]
    q = [_row(Rb, i, *p) + tb[i] for i in range(3)]
    Eq = [sum(abs(Rb[i, j]) * Ep[j] for j in range(3))
          + g4 * (sum(abs(Rb[i, j]) * (np.abs(p[j]) + Ep[j]) for j in range(3)) + abs(tb[i])) for i in range(3)]
    dd = d.astype(F64)
    if mutant == "dir_pose_avg":
        dd = np.stack([_row(Ra, i, *dd.T) for i in range(3)], 1)
    db = [_row(Rb, i, *dd.T) for i in range(3)]
    Ed = [g3 * (np.abs(Rb[i]) * np.abs(dd)).sum(1) for i in range(3)]
    flag = np.zeros(n, bool)
    ts, Es = [], []
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for i in range(3):
            zero = (db[i] == 0) & ~np.signbit(db[i]) if mutant == "zero_plus_only" else db[i] == 0
            flag |= np.abs(db[i]) <= 2 * Ed[i] * (1 + 2.0 ** -30)
            dz = np.where(zero, ZERO_DIR, db[i])
            if mutant == "slab_fp32":
                inv = (F32(1) / dz.astype(F32))
                qq, lo, hi = q[i].astype(F32), F32(b[0, i]), F32(b[1, i])
            else:
                inv, qq, lo, hi = 1 / dz, q[i], b[0, i], b[1, i]
            neg = inv < 0
            t0, t1 = (np.where(neg, hi, lo) - qq) * inv, (np.where(neg, lo, hi) - qq) * inv
            rho = np.where(zero, 0.0, Ed[i] / np.abs(dz))
            Ei = np.where(zero, 0.0, (rho + U64) / (1 - rho) * np.abs(1 / dz))
            aE = []
            for t, B in ((t0, np.where(neg, hi, lo)), (t1, np.where(neg, lo, hi))):
                a = np.abs(B - q[i])
                Ea = Eq[i] + U64 * (a + Eq[i])
                aE.append((a * Ei + Ea * np.abs(1 / dz) + Ea * Ei + U64 * (a + Ea) * (np.abs(1 / dz) + Ei)) * (1 + 2.0 ** -30))
            ts.append((t0, t1))
            Es.append(aE)
        (tmin, tmax), (Emin, Emax) = ts[0], Es[0]
        miss = np.zeros(n, bool)
        for k in (1, 2):
            (lo_k, hi_k), (Elo, Ehi) = ts[k], Es[k]
            flag |= (np.abs(tmin - hi_k) <= 2 * (Emin + Ehi)) | (np.abs(lo_k - tmax) <= 2 * (Elo + Emax))
            if mutant == "reject_ge":
                miss |= (tmin >= hi_k) | (lo_k >= tmax)
            else:
                miss |= (tmin > hi_k) | (lo_k > tmax)
            tmin = np.where(lo_k > tmin, lo_k, tmin)
            tmax = np.where(hi_k < tmax, hi_k, tmax)
            Emin, Emax = np.maximum(Emin, Elo), np.maximum(Emax, Ehi)
        flag |= (np.abs(tmin) <= 2 * Emin) | (np.abs(tmax) <= 2 * Emax)
        miss |= ((tmin <= 0) | (tmax <= 0)) if mutant == "inside_le" else ((tmin < 0) | (tmax < 0))
        flag |= ~miss & ((_f32_boundary_dist(tmin) <= 2 * Emin) | (_f32_boundary_dist(tmax) <= 2 * Emax))
        near = np.where(miss, F32(0), tmin.astype(F32) / s32).astype(F32)
        far = np.where(miss, F32(0), tmax.astype(F32) / s32).astype(F32)
    flag |= ~np.isfinite(tmin) | ~np.isfinite(tmax)
    return dict(hit=~miss, near=near, far=far, tmin=tmin, tmax=tmax, Emin=Emin, Emax=Emax, flag=flag)


def reference(o, d, box: Box, sample=0, seed=0, check_beta=False):
    """Expected result of every ray: slab64 where nothing is close, exact_ray on every flagged ray and on `sample` more.
    Returns dict(hit, near, far, sure, hit_sure, near_lo, near_hi, far_lo, far_hi, n_exact, n_knife, beta_ratio) where
    beta_ratio is the largest |slab64's t - exact t| / beta over the exactly checked hits (check_beta)."""
    o, d = np.asarray(o, F32), np.asarray(d, F32)
    r = slab64(o, d, box)
    n = o.shape[0]
    out = dict(hit=r["hit"].copy(), near=r["near"].copy(), far=r["far"].copy(), sure=np.ones(n, bool),
               hit_sure=np.ones(n, bool))
    for k in ("near", "far"):
        out[k + "_lo"], out[k + "_hi"] = out[k].copy(), out[k].copy()
    idx = np.flatnonzero(r["flag"])
    if sample:
        rng = np.random.default_rng(seed)
        idx = np.union1d(idx, rng.choice(n, size=min(sample, n), replace=False))
    eb = ExactBox(box)
    ratio = 0.0
    for i in idx:
        e = exact_ray(eb, o[i], d[i])
        if not r["flag"][i]:       # a ray the float64 pass calls safe: the exact path must agree with it
            assert e["sure"] and e["hit"] == r["hit"][i], (i, e)
            assert bits(e["near"]) == bits(r["near"][i]) and bits(e["far"]) == bits(r["far"][i]), (i, e, r["near"][i])
        if check_beta and e.get("hit") and e["sure"]:
            for t, k in (("tmin", "tmin"), ("tmax", "tmax")):
                T = e[t]
                err = abs(Fr(float(r[k][i])) - T.v) if np.isfinite(r[k][i]) else Fr(0)
                if T.e:
                    ratio = max(ratio, float(err) / T.e)
                else:
                    assert err == 0, (i, t)
        out["hit_sure"][i], out["sure"][i], out["hit"][i] = e["hit_sure"], e["sure"], e["hit"]
        if e["hit"]:
            for k in ("near", "far", "near_lo", "near_hi", "far_lo", "far_hi"):
                out[k][i] = e[k]
        else:
            for k in ("near", "far", "near_lo", "near_hi", "far_lo", "far_hi"):
                out[k][i] = F32(0)
    out["n_exact"], out["n_knife"], out["beta_ratio"] = len(idx), int((~out["sure"]).sum()), ratio
    return out


def slab_verdict(hit, near, far, want):
    """hit (n,) bool, near / far (n,) fp32 of the code under test against reference(): decidable rays bit for bit, sign
    of zero included; knife-edge rays either decision, a hit inside the neighbouring values; a miss is (+0, +0).
    Returns the number of decidable rays."""
    hit, near, far = np.asarray(hit, bool), np.asarray(near, F32), np.asarray(far, F32)
    nb, fb = near.view(np.uint32), far.view(np.uint32)
    sure, hs = want["sure"], want["hit_sure"]
    bad = sure & ((hit != want["hit"]) | (nb != want["near"].view(np.uint32)) | (fb != want["far"].view(np.uint32)))
    bad |= hs & (hit != want["hit"])
    with np.errstate(invalid="ignore"):
        for k, got in (("near", near), ("far", far)):
            bad |= ~sure & hs & hit & ~((got >= want[k + "_lo"]) & (got <= want[k + "_hi"]))
    bad |= ~hit & ((nb != 0) | (fb != 0))
    if bad.any():
        i = np.flatnonzero(bad)[:8]
        raise AssertionError(f"{int(bad.sum())} rays wrong, e.g. rows {i.tolist()}: hit {hit[i].tolist()} want "
                             f"{want['hit'][i].tolist()}; near {near[i].tolist()} want {want['near'][i].tolist()}; far "
                             f"{far[i].tolist()} want {want['far'][i].tolist()}")
    return int(sure.sum())


def scene_near_far(near, far, scale_factor):
    """editable_renderer.py:157-158: near / scale_factor in float64 (python floats), then the fp32 the tensor holds."""
    return F32(float(near) / float(scale_factor)), F32(float(far) / float(scale_factor))


# ------------------------------------------------------------------------------------------------
# camera rays
# ------------------------------------------------------------------------------------------------
# rays_d gate ROT_C 2^-24 (|d_i| + sum_j |r_ij x_j| / ||w||).  The kernel forms w in fp32 (3 products: gamma_3 ~ 3 u32 of
# sum_j |r_ij x_j|); the norm inherits that error: | ||w^|| - ||w|| | <= gamma_3 || |R| |x| || <= 3 sqrt(3) u32 ||w|| for a
# rotation (|| |R| ||_2 <= ||R||_F = sqrt 3); the norm's rounding to fp32 and the quotient's add 2 u32 |d_i|.  So 3 on
# the second term and 3 sqrt(3) + 2 = 7.2 on the first, plus the float64 reference's own 2^-50: ROT_C = 8 covers both.
ROT_C = 8.0


def directions_f32(H, W, focal):
    """datasets/ray_utils.py:17-23 restated in numpy float32: ((x - W/2) / focal, -((y - H/2) / focal), -1), no +0.5."""
    x = np.arange(W, dtype=F32)[None, :].repeat(H, 0)
    y = np.arange(H, dtype=F32)[:, None].repeat(W, 1)
    f = F32(focal)
    return np.stack([(x - F32(W / 2)) / f, -((y - F32(H / 2)) / f), -np.ones((H, W), F32)], -1)


def rays_d64(x, c2w):
    """float64 rotate-and-normalise of (n, 3) fp32 directions by the fp32 c2w[:, :3], and the gate of each component."""
    R = np.asarray(c2w, F32)[:3, :3].astype(F64)
    x = np.asarray(x, F32).reshape(-1, 3).astype(F64)
    w = x @ R.T
    with np.errstate(invalid="ignore", divide="ignore"):
        nrm = np.linalg.norm(w, axis=1, keepdims=True)
        d = w / nrm
        gate = ROT_C * 2.0 ** -24 * (np.abs(d) + (np.abs(x)[:, None, :] * np.abs(R)[None]).sum(-1) / nrm)
    return d, gate


def rays_d_ratio(got, x, c2w):
    """Largest share of the rays_d gate used; NaN exactly where the reference is NaN (a zero-length direction)."""
    want, gate = rays_d64(x, c2w)
    got = np.asarray(got, F32).reshape(-1, 3).astype(F64)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    err, g = np.abs(got - want)[~nan], gate[~nan]
    assert (err[g == 0] == 0).all()          # a component the rotation makes exactly zero stays zero
    return float((err[g > 0] / g[g > 0]).max()) if (g > 0).any() else 0.0


def level_c2w(yaw_deg, t):
    """A level camera: right = (cos a, sin a, 0), up = world +z, back = right x up.  Its third row is (0, 1, 0), so the
    world dz of a ray is its camera dy: exactly zero on row H / 2 of an even-height frame."""
    a = math.radians(yaw_deg)
    R = np.array([[math.cos(a), 0.0, math.sin(a)], [math.sin(a), 0.0, -math.cos(a)], [0.0, 1.0, 0.0]])
    return torch.from_numpy(np.concatenate([R, np.asarray(t, F64)[:, None]], 1).astype(F32))


# ------------------------------------------------------------------------------------------------
# inputs: planted geometry and random boxes
# ------------------------------------------------------------------------------------------------
UNIT = [[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]]
PERM = np.array([[0.0, 0.0, -1.0], [1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])
ROT90 = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
YAW_34 = np.array([[0.6, -0.8, 0.0], [0.8, 0.6, 0.0], [0.0, 0.0, 1.0]])   # the float64 0.6, 0.8: taken as exact values
SUB = 2.0 ** -140                                                          # an fp32 subnormal
INF = float("inf")

# name: (Box, rays).  Each ray: (origin, direction, expected) with expected None for a miss or (t_near, t_far) in box
# units (near = fp32(fp32(t) / scale)).  Origins are box-frame points q for the dyadic setups, world points ("w") for
# yaw; directions are world directions.
PLANTED = {
    # q = 2 o + (0.75, -0.25, -0.625); identity axis alignment: the direction is the box-frame direction
    "unit": (Box(rigid(None, (0.25, -0.5, 0.125)), rigid(None, (0.5, 0.25, -0.75)), UNIT, 2.0), [
        ((-1, .5, .5), (1, 0, 0), (1, 2)),                  # parallel to two axes, inside both slabs
        ((-1, .5, .5), (1, -0.0, -0.0), (1, 2)),            # the same with -0.0
        ((-1, -.5, -.25), (1, .5, .25), (1, 2)),            # three-way tie of the entry distances
        ((-.5, .25, .75), (.5, .25, -.25), (1, 3)),         # interior crossing, a negative component
        ((-1, 0, .5), (1, 0, 0), (1, 2)),                   # face graze, q == lo: a hit
        ((-1, 1, .5), (1, 0, 0), None),                     # face graze, q == hi: a miss
        ((-1, .5, 0), (1, 0, 0), (1, 2)),                   # z == lo
        ((-1, .5, 1), (1, 0, 0), None),                     # z == hi
        ((-1, 1.5, .5), (1, 0, 0), None),                   # parallel, outside the slab
        ((-1, -.5, .5), (1, -0.0, 0), None),                # parallel (-0.0), below the slab
        ((-1, 0, .5), (1, 1, 0), (1, 1)),                   # edge touch: tmin == tymax, near == far
        ((-1, 0, 0), (1, 1, 1), (1, 1)),                    # corner touch
        ((-1, .5, -2), (1, 0, 1), (2, 2)),                  # edge touch: tzmin == tmax
        ((0, .5, .5), (1, 0, 0), (0, 1)),                   # origin on the lower face, pointing in: near +0
        ((1, .5, .5), (-1, 0, 0), (-0.0, 1)),               # origin on the upper face, pointing in: near -0.0
        ((1, .5, .5), (1, 0, 0), None),                     # on a face, pointing out
        ((0, .5, .5), (-1, 0, 0), None),
        ((.5, .5, .5), (1, .5, .25), None),                 # origin inside: a miss by the reference's rule
        ((2, .5, .5), (1, 0, 0), None),                     # box wholly behind
        ((-1, 2, .5), (1, .25, 0), None),                   # first rejection
        ((-1, .5, -3), (1, 0, 1), None),                    # second rejection
        ((2, 1, 2), (-1, -0.0, -1), None),                  # box-frame dy is -0.0 in every order, q == hi: a miss
        ((2, 0, 2), (-1, -0.0, -1), (1, 2)),                # ... q == lo: a hit
        ((.5, .5, 2), (0, 0, -1), (1, 2)),                  # parallel to x and y, down through the box
        ((-1, .5, .5), (1, SUB, 0), (1, 2)),                # subnormal component: inverse 2^140, no restriction
        ((-1, -1, -1), (SUB, SUB, SUB), (2.0 ** 140, 2.0 ** 141)),   # t past the fp32 range: near = far = inf
    ]),
    # signed axis permutation, scale 0.5: the direction is given in the box frame and mapped back (d_w = Rb^T d_box)
    "perm": (Box(rigid(None, (0.125, 0.25, -0.5)), rigid(PERM, (1.0, -0.5, 0.75)), UNIT, 0.5), [
        ((-1, .5, .5), (1, 0, 0), (1, 2)),
        ((-1, 0, .5), (1, 1, 0), (1, 1)),
        ((1, .5, .5), (-1, 0, 0), (-0.0, 1)),
        ((-1, 1, .5), (1, 0, 0), None),
        ((.25, .5, -.5), (.25, 0, .5), (1, 3)),
        ((.5, .5, .5), (0, 0, 1), None),
    ]),
    # rotated pose_avg: origins rotate by it, directions do not (utils/bbox_utils.py:116)
    "pose_rot": (Box(rigid(ROT90, (0.5, 0.0, 0.25)), rigid(None), UNIT, 0.5), [
        ((-1, .5, .5), (1, 0, 0), (1, 2)),
        ((.5, -1, .5), (0, .5, 0), (2, 4)),
        ((.5, .5, -1), (0, 0, 1), (1, 2)),
    ]),
    # yaw-only axis alignment (third row 0 0 1): q = YAW_34 (2 o) + (0, -0.5, 0.25); world origins
    "yaw": (Box(rigid(None), rigid(YAW_34, (0.0, -0.5, 0.25)), [[0, 0, 0], [1, 1, 0.5]], 2.0), [
        (("w", 0, 0, 0), (1, 0, 0), (0.625, Fr(5, 3))),     # horizontal: box-frame dz exactly 0, q_z inside
        (("w", 0, 0, -0.125), (1, 0, 0), (0.625, Fr(5, 3))),  # ... q_z == lo: a hit
        (("w", 0, 0, 0.125), (1, 0, 0), None),              # ... q_z == hi: a miss
        (("w", 0.625, 0.125, 1), (0, 0, -1), (1.75, 2.25)),  # vertical: box-frame dx, dy exactly 0, inside the footprint
        (("w", 0, 0, 0.5), (0, 0, -1), None),               # vertical, outside the footprint
    ]),
    "flat": (Box(rigid(None), rigid(None), [[0, 0, .5], [1, 1, .5]], 2.0), [
        ((.5, .5, 1), (0, 0, -1), (.5, .5)),
        ((-1, .5, .5), (1, 0, 0), None),                    # in the flat box's plane: tzmin == tzmax == 0 < tmin
        ((-1, .5, 0), (1, 0, .5), (1, 1)),
    ]),
    "enlarged": (Box(rigid(None), rigid(None), UNIT, 2.0, bbox_enlarge=0.25), [
        ((-1, 1.125, .5), (1, 0, 0), (.75, 2.25)),
        ((-1, 1.25, .5), (1, 0, 0), None),
        ((-1, -.25, .5), (1, 0, 0), (.75, 2.25)),
    ]),
}


def planted_rays(name):
    """(o, d, expected) fp32 world rays of PLANTED[name]."""
    box, rays = PLANTED[name]
    P, A, s = box.pose_avg, box.axis_align_mat, box.scale_factor
    o, d, exp = [], [], []
    for q, dd, e in rays:
        if q[0] == "w":
            ow = np.array(q[1:], F64)
        else:                                      # q = Rb (Ra 2o + ta) + tb, both rotations orthogonal and dyadic
            p = A[:3, :3].T @ (np.array(q, F64) - A[:3, 3])
            ow = P[:3, :3].T @ (p - P[:3, 3]) / s
        dw = np.array(dd, F64)
        if name == "perm":
            dw = A[:3, :3].T @ dw
        assert np.array_equal(ow.astype(F32).astype(F64), ow) and np.array_equal((ow.astype(F32) * F32(s)), ow * s)
        o.append(ow.astype(F32))
        d.append(dw.astype(F32))
        exp.append(e)
    return np.stack(o), np.stack(d), exp


def random_box(kind, seed):
    """Box variants of build_bbox_case: 'yaw' (axis alignment about z only), 'perm' (signed axis permutation),
    'pose_rot' (a rotated pose_avg and a general axis alignment)."""
    rng = np.random.default_rng(seed)
    lo = np.array([-0.6, -0.4, -0.3]) + rng.uniform(-0.05, 0.05, 3)
    hi = np.array([0.5, 0.7, 0.4]) + rng.uniform(-0.05, 0.05, 3)
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    q *= np.sign(np.linalg.det(q))
    ta, tb = rng.uniform(-0.5, 0.5, 3), rng.uniform(-0.5, 0.5, 3)
    if kind == "yaw":
        return Box(rigid(None, ta), rigid(yaw(rng.uniform(-3, 3)), tb), np.stack([lo, hi]), 2.0)
    if kind == "perm":
        return Box(rigid(None, ta), rigid(PERM, tb), np.stack([lo, hi]), 0.5, bbox_enlarge=0.03)
    q2, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    q2 *= np.sign(np.linalg.det(q2))
    return Box(rigid(q2, ta), rigid(q, tb), np.stack([lo, hi]), 4.0)


def box_rays(box: Box, n, seed):
    """n fp32 rays at NeRF scale, as build_bbox_case: aimed at the box from ~3 box sizes away, 10 % starting inside it,
    5 % with one exactly-zero world component of either sign."""
    rng = np.random.default_rng(seed)
    b = box.bounds()
    centre, half = (b[0] + b[1]) / 2, (b[1] - b[0]) / 2
    P, A, s = box.pose_avg, box.axis_align_mat, box.scale_factor
    tgt = centre + rng.uniform(-1.4, 1.4, size=(n, 3)) * half
    org = centre + rng.normal(size=(n, 3)) * 3.0
    inside = rng.uniform(size=n) < 0.1
    org[inside] = centre + rng.uniform(-0.9, 0.9, size=(int(inside.sum()), 3)) * half
    Ainv, Pinv = np.linalg.inv(A[:3, :3]), np.linalg.inv(P[:3, :3])
    o = (((org - A[:3, 3]) @ Ainv.T - P[:3, 3]) @ Pinv.T / s).astype(F32)
    d = (tgt - org) @ Ainv.T                               # the reference rotates the direction by axis_align only
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(F32)
    zero = np.flatnonzero(rng.uniform(size=n) < 0.05)
    d[zero, rng.integers(0, 3, size=zero.size)] = np.where(rng.uniform(size=zero.size) < 0.5, F32(0.0), F32(-0.0))
    return o, d


def golden_box(name):
    inp = cases.build_bbox_case(cases.BBOX_CASES[name])
    box = Box(inp["pose_avg"], inp["axis_align_mat"], inp["bbox_bounds"], inp["scale_factor"], inp["bbox_enlarge"])
    return box, np.ascontiguousarray(inp["rays_o"].numpy()), np.ascontiguousarray(inp["rays_d"].numpy())


RANDOM_BOXES = {"yaw": 501, "perm": 502, "pose_rot": 503}


# ------------------------------------------------------------------------------------------------
# checks of the references
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(PLANTED))
def test_planted_geometry_expectations(name):
    """The exact reference gives every planted ray the result written next to it, decidably, and so does slab64."""
    box = PLANTED[name][0]
    o, d, exp = planted_rays(name)
    want = reference(o, d, box, sample=len(o))
    assert want["sure"].all(), np.flatnonzero(~want["sure"])
    s = F32(box.scale_factor)
    for i, e in enumerate(exp):
        assert want["hit"][i] == (e is not None), (name, i)
        if e is None:
            assert bits(want["near"][i]) == 0 and bits(want["far"][i]) == 0
            continue
        for k, t in zip(("near", "far"), e):
            t32 = round32(Fr(t), negzero=isinstance(t, float) and t == 0 and math.copysign(1, t) < 0)
            assert bits(want[k][i]) == bits(F32(t32 / s)), (name, i, k, want[k][i], t32 / s)
    slab_verdict(*(slab64(o, d, box)[k] for k in ("hit", "near", "far")), want)


def test_planted_set_covers_the_rules():
    """The planted rays reach what they are for: exact ties at the rejections and the inside rule, -0.0 near, a -0.0
    box-frame direction component, the 1e-14 rule on both signs, a subnormal direction, infinite near / far."""
    o, d, _ = planted_rays("unit")
    box = PLANTED["unit"][0]
    eb = ExactBox(box)
    res = [exact_ray(eb, o[i], d[i]) for i in range(len(o))]
    ties = [n for r in res for (n, out, m, e) in r["decisions"] if m == 0 and e == 0]
    assert any(n.startswith("tmin > t") for n in ties) and any(n.startswith("t") and "min > tmax" in n for n in ties)
    assert "tmin < 0" in ties
    near = np.array([r.get("near", F32(0)) for r in res], F32)
    assert (np.signbit(near) & (near == 0)).any() and np.isinf(near).any()
    r = slab64(o, d, box)
    assert r["hit"].sum() == sum(x["hit"] for x in res)
    db = _row(box.axis_align_mat, 1, *d.astype(F64).T)
    assert ((db == 0) & np.signbit(db)).any() and ((db == 0) & ~np.signbit(db)).any()


@pytest.mark.parametrize("name", list(cases.BBOX_CASES))
def test_references_reproduce_the_golden_fixtures(golden, name):
    """(b) exact_ray / slab64 give the reference's own fixture results, bit for bit on decidable rays."""
    box, o, d = golden_box(name)
    gold = golden("rays_" + name)
    want = reference(o, d, box, sample=256, seed=1, check_beta=True)
    n_sure = slab_verdict(gold["mask"].numpy().astype(bool), gold["near"].numpy().reshape(-1),
                          gold["far"].numpy().reshape(-1), want)
    print(f"{name}: {n_sure} decidable, {want['n_knife']} knife-edge, {want['n_exact']} exact; "
          f"RATIO beta {name}: {want['beta_ratio']:.3e}")
    assert want["beta_ratio"] <= 1
    assert n_sure >= len(o) - 2


@pytest.mark.parametrize("kind", list(RANDOM_BOXES))
def test_beta_bounds_the_float64_pass(kind):
    """slab64's t values stay inside beta of the exact ones on the random box variants; the zero rule is reached."""
    box = random_box(kind, RANDOM_BOXES[kind])
    o, d = box_rays(box, 3000, RANDOM_BOXES[kind] + 1)
    want = reference(o, d, box, sample=600, seed=2, check_beta=True)
    print(f"{kind}: {want['n_knife']} knife-edge of {len(o)}; RATIO beta {kind}: {want['beta_ratio']:.3e}")
    assert want["beta_ratio"] <= 1 and want["n_knife"] == 0
    assert want["hit"].any() and (~want["hit"]).any()
    db = np.stack([_row(box.axis_align_mat, i, *d.astype(F64).T) for i in range(3)], 1)
    if kind != "pose_rot":
        assert (db == 0).sum() > 20


def test_camera_references_reproduce_the_golden_fixtures(golden):
    """(b) directions bit for bit, rays_o bit for bit, the reference's own rays_d inside the rays_d gate; a zero-length
    direction gives NaN in the float64 reference as in the reference's torch code."""
    for name, c in cases.CAMERA_CASES.items():
        inp = cases.build_camera_case(c)
        gold = golden("rays_" + name)
        dirs = directions_f32(inp["H"], inp["W"], inp["focal"])
        assert np.array_equal(dirs.view(np.uint32), gold["directions"].numpy().view(np.uint32))
        assert np.array_equal(dirs.view(np.uint32), O.ray_directions(inp["H"], inp["W"], inp["focal"]).numpy().view(np.uint32))
        c2w = inp["c2w"].numpy()
        assert np.array_equal(gold["rays_o"].numpy(), np.broadcast_to(c2w[:, 3], gold["rays_o"].shape))
        r = rays_d_ratio(gold["rays_d"].numpy(), dirs, c2w)
        print(f"RATIO rays_d golden {name}: {r:.3e}")
        assert r <= 1
    x = np.zeros((2, 3), F32)
    x[1] = (0.25, -0.5, -1)
    c2w = cases.build_camera_case(cases.CAMERA_CASES["cam_small"])["c2w"]
    _, rd = O.get_rays(torch.from_numpy(x), c2w)
    assert torch.isnan(rd[0]).all() and not torch.isnan(rd[1]).any()
    assert rays_d_ratio(rd.numpy(), x, c2w.numpy()) <= 1


def test_scene_near_far_reference():
    for near, far, s in ((0.3, 7.0, 3.0), (0.3, 6.0, 2.0), (0.1, 5.0, 0.5)):
        o = torch.zeros(2, 3)
        rays = O.generate_rays(0, o, o, near, far, s)
        n32, f32 = scene_near_far(near, far, s)
        assert bits(rays[0, 6].item()) == bits(n32) and bits(rays[0, 7].item()) == bits(f32)
    assert F32(0.3 / 3.0) != F32(0.1) or Fr(float(F32(0.3 / 3.0))) != Fr(3, 30)   # not exactly representable


def _mutant_cases():
    out = [(name, PLANTED[name][0]) + planted_rays(name)[:2] for name in PLANTED]
    for name in cases.BBOX_CASES:
        out.append((name,) + golden_box(name))
    for kind, seed in RANDOM_BOXES.items():
        box = random_box(kind, seed)
        out.append((kind, box) + box_rays(box, 3000, seed + 1))
    return out


def test_slab64_passes_its_own_verdict():
    """Soundness: the unmutated float64 pass, in its own evaluation order, passes the verdict on every input set."""
    for name, box, o, d in _mutant_cases():
        want = reference(o, d, box)
        r = slab64(o, d, box)
        slab_verdict(r["hit"], r["near"], r["far"], want)


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutants_fail_the_verdict(mutant):
    """(c) Discrimination: each mutant of the slab test fails the verdict on at least one input set."""
    failed = []
    for name, box, o, d in _mutant_cases():
        want = reference(o, d, box)
        r = slab64(o, d, box, mutant=mutant)
        try:
            slab_verdict(r["hit"], r["near"], r["far"], want)
        except AssertionError:
            failed.append(name)
    print(f"{mutant}: fails on {failed}")
    assert failed, mutant


# ------------------------------------------------------------------------------------------------
# (a) the reference's own code
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref_modules():
    if not ref_loader.available():
        pytest.skip("oracle/_ref not built")
    pytest.importorskip("numba")
    ref_loader.install()
    from datasets import geo_utils
    from utils import bbox_utils
    return geo_utils, bbox_utils


def _ref_intersections(bbox_utils, box: Box, o, d):
    h = object.__new__(bbox_utils.BBoxRayHelper)
    h.pose_avg, h.axis_align_mat, h.bbox_bounds = box.pose_avg, box.axis_align_mat, box.bbox_bounds
    h.scale_factor = box.scale_factor
    mask, near, far = h.get_ray_bbox_intersections(torch.from_numpy(o), torch.from_numpy(d), box.scale_factor,
                                                   box.bbox_enlarge)
    return mask.cpu().numpy(), near.cpu().numpy().reshape(-1), far.cpu().numpy().reshape(-1)


def test_reference_code_slab_rules(ref_modules):
    """geo_utils.bbox_intersection itself on the [0, 1]^3 box: a graze at z == lo hits at (1, 2), at z == hi misses, an
    origin on the upper face pointing in gives near = -0.0; exact_ray says the same."""
    geo_utils, _ = ref_modules
    bounds = np.array(UNIT)
    eb = ExactBox(Box(rigid(None), rigid(None), UNIT, 1.0))
    for o, d, want in (((-1, .5, 0), (1, 0, 0), (True, 1.0, 2.0)), ((-1, .5, 1), (1, 0, 0), (False, 0.0, 0.0)),
                       ((1, .5, .5), (-1, 0, 0), (True, -0.0, 1.0))):
        hit, near, far = geo_utils.bbox_intersection(bounds, np.array(o, F64), np.array(d, F64))
        assert (bool(hit), near, far) == want and math.copysign(1, near) == math.copysign(1, want[1])
        e = exact_ray(eb, np.array(o, F32), np.array(d, F32))
        assert e["sure"] and e["hit"] == want[0]
        if want[0]:
            assert bits(e["near"]) == bits(F32(want[1])) and bits(e["far"]) == bits(F32(want[2]))


def test_references_agree_with_the_reference_code(ref_modules):
    """(a) BBoxRayHelper.get_ray_bbox_intersections on every planted ray and the random boxes: the reference's own code
    passes the verdict (bit for bit on decidable rays)."""
    _, bbox_utils = ref_modules
    sets = [(name, PLANTED[name][0]) + planted_rays(name)[:2] for name in PLANTED]
    for kind, seed in RANDOM_BOXES.items():
        box = random_box(kind, seed)
        sets.append((kind, box) + box_rays(box, 2000, seed + 7))
    for name, box, o, d in sets:
        want = reference(o, d, box, sample=200 if len(o) > 200 else 0, seed=3)
        hit, near, far = _ref_intersections(bbox_utils, box, o, d)
        n = slab_verdict(hit, near, far, want)
        print(f"reference code {name}: {n} decidable of {len(o)}")
