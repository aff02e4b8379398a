"""Float64 references for the stage tests of the field forward (tests/test_gpu_field_stages.py), and the checks of those
references that need no device:
  - the layer-by-layer reference in kernel-K order (weights mapped from the reference layout, never read from the
    packed blob), with exact encodings and no rounding, reproduces the oracle's scene / object MLP; pad columns unused;
  - fmaf emulation with one rounding, the epilogue emulations, and the error budget of the positional encoding's
    double-angle recurrence against a float32 emulation of it."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import onerf_oracle as O
from tests import synth
from tests.test_gpu_train_stages import _wgrad_inputs
from tests.voxel_grid_cases import voxel_features32  # noqa: F401  (the kernels' trilinear blend, re-exported)

# GEMM layers in GemmId order (csrc/layout.h); the output of GEMMS[i] is activation slot i + 1
GEMMS = ("S0", "S1", "S2", "S3", "S4", "S5", "S6", "S7", "SFIN", "SDIR", "O0", "O1", "O2", "O3", "OFIN", "ODIR")
REF = {**{f"S{i}": f"scene.l{i}" for i in range(8)}, "SFIN": "scene.final", "SDIR": "scene.dir",
       **{f"O{i}": f"obj.l{i}" for i in range(4)}, "OFIN": "obj.final", "ODIR": "obj.dir"}
N_OUT = {g: (256 if g.startswith("S") and g != "SDIR" else 64 if g == "ODIR" else 128) for g in GEMMS}
RC_BASE = {"SDIR": 0, "ODIR": 128, "O0": 192, "O2": 320}      # layout.h RC_*: bias + direction / code terms
SIGMA_LAYER = {"S7": ("scene.sigma", 0), "O3": ("obj.sigma", 1)}  # layer feeding a sigma head, branch
DIR_LAYER = {"SDIR": ("scene.rgb", 0), "ODIR": ("obj.rgb", 1)}
MASK_WORD0 = {**{s: (s - 1) * 8 for s in range(1, 9)}, 10: 64, **{s: 68 + (s - 11) * 4 for s in range(11, 15)}, 16: 84}
SLOPE_BF16 = 0.010009765625          # bf16(0.01f): the slope of the packed-bf16 LeakyReLU
SLOPE_F32 = float(np.float32(0.01))


def dims(use_voxel):
    """(reference scene-input width, object voxel PE width, KX, KO)."""
    return (271, 104, 288, 384) if use_voxel else (63, 0, 64, 64)


def kernel_weights(w, use_voxel, bf16=True):
    """{GEMM: (W [N, K] float64 in kernel-K order, bias float64)} from the reference weights [out, in].  The X-fed
    layers read X[0, KX) / X[0, KO) (scene input at 0, object voxel PE at 272), the skip layers S4 / O2 then the
    previous hidden layer at KX / KO; code and direction columns are left out (they reach the layer through
    ray_const).  bf16: W rounded as the tensor cores read it."""
    xin, ovx, KX, KO = dims(use_voxel)
    oin = xin + ovx + synth.N_CODE
    segs = {"S0": (KX, [(0, xin, 0)]), "S4": (KX + 256, [(0, xin, 0), (KX, 256, xin)]),
            "O0": (KO, [(0, xin, 0), (272, ovx, xin)]), "O2": (KO + 128, [(0, xin, 0), (272, ovx, xin), (KO, 128, oin)]),
            "SDIR": (256, [(0, 256, 0)]), "ODIR": (128, [(0, 128, 0)])}
    out = {}
    for g in GEMMS:
        W, b = w[REF[g]]
        K, seg = segs.get(g, (W.shape[1], [(0, W.shape[1], 0)]))
        Wk = torch.zeros(W.shape[0], K, dtype=torch.float64)
        for dst, n, src in seg:
            Wk[:, dst:dst + n] = W[:, src:src + n].double()
        if bf16:
            Wk = Wk.to(torch.bfloat16).double()
        out[g] = (Wk, b.double())
    return out


def ray_const_ref(rays, codes, w, use_voxel, want_object=True):
    """float64 ray_const (n, 448) of ray_const_kernel (csrc/field_fp32.cu) from the fp32 weights, and its error gate:
    the fp32 dot products (K terms after the bias) within 2^-24 (K + 2) sum |terms|, plus 2^-22 (2 ulp of sinf) per
    direction-encoding input times |w|."""
    xin, ovx, _, _ = dims(use_voxel)
    dev = rays.device
    pe = O.posenc(rays[:, 3:6].double(), 4)
    code = codes.double() if want_object else torch.zeros(rays.shape[0], synth.N_CODE, dtype=torch.float64, device=dev)
    blocks = [("scene.dir", pe, slice(256, 283)), ("obj.dir", pe, slice(128, 155)),
              ("obj.l0", code, slice(xin + ovx, xin + ovx + 64)), ("obj.l2", code, slice(xin + ovx, xin + ovx + 64))]
    ref, gate = [], []
    for name, x, cols in blocks:
        W, b = w[name][0][:, cols].double().to(dev), w[name][1].double().to(dev)
        ref.append(x @ W.t() + b)
        bound = x.abs() @ W.abs().t() + b.abs()
        sin_err = 2.0 ** -22 * W.abs().sum(1) if x is pe else 0.0
        gate.append(2.0 ** -24 * (x.shape[1] + 2) * bound + sin_err)
    return torch.cat(ref, 1), torch.cat(gate, 1)


def preact(g, inp, kw, rc=None, ray=None):
    """Pre-activation t = inp W^T + (bias or the row's ray_const block) of GEMM g, and B = the same over |terms|."""
    W, b = kw[g]
    term = rc[ray, RC_BASE[g]:RC_BASE[g] + W.shape[0]] if g in RC_BASE else b
    return inp @ W.t() + term, inp.abs() @ W.abs().t() + term.abs()


# ------------------------------------------------------------------------------------------------
# epilogues: each a non-decreasing function of the fp32 pre-activation (evaluated on float64 tensors)
# ------------------------------------------------------------------------------------------------
def bf16(x):
    return x.to(torch.bfloat16).to(x.dtype)


def epi_hidden(t):
    """EPI_HIDDEN / EPI_HIDDEN_RC: one rounding to bf16, then __hmax2(v, __hmul2(v, bf16(0.01))) (one rounding of the
    product)."""
    v = bf16(t)
    return torch.maximum(v, bf16(v * SLOPE_BF16))


def epi_fp32_leaky(t):
    """EPI_HIDDEN_SIGMA / EPI_DIR: fmaxf(t, t * 0.01f) in fp32, then one rounding to bf16."""
    t32 = t.float()
    return bf16(torch.maximum(t32, t32 * SLOPE_F32).double())


def epi_final(t):
    return bf16(t)


def tc_epilogue(g):
    if g in SIGMA_LAYER or g in DIR_LAYER:
        return epi_fp32_leaky
    return epi_final if g in ("SFIN", "OFIN") else epi_hidden


def ffma_epilogue(g):
    """field_fp32.cu: t > 0 ? t : t * 0.01f in fp32 (no activation for the final layers), fp32 output."""
    if g in ("SFIN", "OFIN"):
        return lambda t: t.float().double()

    def leaky(t):
        t32 = t.float()
        return torch.where(t32 > 0, t32, t32 * SLOPE_F32).double()
    return leaky


def gate_share(t, d, got, f, iters=32):
    """Smallest q with f(t - q d) <= got <= f(t + q d) for a non-decreasing f (bisection on log2 q in [-40, 40]): the
    share of the error budget d a result uses.  0 where got == f(t); > 1 fails the gate (inf: outside even at 2^40)."""
    q = torch.zeros_like(t)
    idx = (f(t) != got).nonzero(as_tuple=True)
    if idx[0].numel() == 0:
        return q
    tt, dd, gg = t[idx], d[idx], got[idx]
    ok = lambda e: (f(tt - 2.0 ** e * dd) <= gg) & (gg <= f(tt + 2.0 ** e * dd))
    lo, hi = torch.full_like(tt, -40.0), torch.full_like(tt, 40.0)
    never = ~ok(hi)
    for _ in range(iters):
        mid = (lo + hi) / 2
        m = ok(mid)
        hi, lo = torch.where(m, mid, hi), torch.where(m, lo, mid)
    q[idx] = torch.where(never, torch.full_like(hi, math.inf), 2.0 ** hi)
    return q


# ------------------------------------------------------------------------------------------------
# encoding: the kernels' fp32 positions and voxel features, and the budget of the tensor-core X
# ------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fmaf(a, b, c) for float32 tensors: the product is exact in float64; the double sum's rounding error (TwoSum)
    breaks the ties its second rounding to float32 would otherwise resolve to even."""
    p, cd = a.double() * b.double(), c.double()
    s = p + cd
    bb = s - p
    err = (p - (s - bb)) + (cd - bb)
    r = s.float()
    up = torch.nextafter(r, torch.full_like(r, math.inf))
    dn = torch.nextafter(r, torch.full_like(r, -math.inf))
    r = torch.where((s == (r.double() + up.double()) / 2) & (err > 0), up, r)
    return torch.where((s == (r.double() + dn.double()) / 2) & (err < 0), dn, r)


def positions(rays, z, fused):
    """(n S, 3) float32 sample positions: fmaf(d, z, o) (tensor-core kernel, fused) or o + d z with two roundings
    (FFMA kernel)."""
    n, S = z.shape
    o = rays[:, None, 0:3].expand(n, S, 3).reshape(-1, 3)
    d = rays[:, None, 3:6].expand(n, S, 3).reshape(-1, 3)
    zz = z.reshape(-1, 1).expand(-1, 3)
    return fma32(d, zz, o) if fused else o + d * zz


def pe_budget(v, dv, e0, n_freq):
    """Absolute error budgets of [v, sin 2^k v, cos 2^k v]_k as the tensor-core encoder forms them (field_pe.cuh):
    v carries an error <= dv; sin / cos of octave 0 come from sincosf / __sincosf with absolute error <= e0; octave
    k + 1 from octave k by s' = fl(2 s c), c' = fl(1 - 2 s^2) (fmaf).

    Write the computed point of octave k as (1 + rho) e^{i(a + phi)} with a = 2^k v: an error vector of length <= e
    splits into |rho|, |phi| <= e, and each component of the error is <= |rho| + |phi|.  The step maps the exact
    point (1 + rho) e^{ib} to e^{2ib} (1 + eta (2 sin^2 b + i sin 2b)), eta = 2 rho + rho^2, so the phase error
    doubles plus eta |sin 2b| and the radial error becomes 2 eta sin^2 b; each fp32 rounding adds <= 2^-24 per
    component (|s'|, |c'| <= 1), i.e. <= 2^-23.5 to either.  b = a + phi, so sin^2 b and |sin 2b| are bounded with
    |phi| added to the exact angle.  The value error dv is a phase error 2^k dv at octave k.  1 % slack covers the
    second-order terms of the polar split.
    -> list of (values, budgets), one per column block [v, sin_0, cos_0, sin_1, ...]."""
    out = [(v, dv)]
    P = math.sqrt(2) * e0 + dv
    R = math.sqrt(2) * e0 + torch.zeros_like(v)
    for k in range(n_freq):
        a = v * 2.0 ** k
        e = 1.01 * (P + R)
        out += [(torch.sin(a), e), (torch.cos(a), e)]
        s2 = torch.clamp(torch.sin(a).abs() + P, max=1.0) ** 2
        s2b = torch.clamp(torch.sin(2 * a).abs() + 2 * P, max=1.0)
        eta = 2 * R + R * R
        R, P = 2 * eta * s2 + 2.0 ** -23.5, 2 * P + eta * s2b + 2.0 ** -23.5
    return out


# absolute error of octave 0: sincosf is within 2 ulp (<= 2^-23 on [-1, 1]); __sincosf evaluates MUFU.SIN / COS at
# fl(x fl(1 / 2 pi)): its documented bound 2^-21.41 on [-pi, pi], plus the angle error of those two roundings,
# |x| 2^-24 each, taken as |x| 2^-22 (twice that) beyond pi
E0_SINCOSF = 2.0 ** -23


def e0_fast_sincos(f):
    return 2.0 ** -21.41 + f.abs() * 2.0 ** -22


def x_reference(x32, feats, use_voxel):
    """float64 X (B, KO) of the tensor-core encoder at fp32 positions x32 and its budget; pad columns have budget 0
    and value 0.  feats = voxel_features32(...) (voxel model)."""
    v = x32.double()
    blocks = []
    if use_voxel:
        f64, fb = feats[0], feats[1] * 16 * 2.0 ** -24    # 8 fp32 roundings (or fused FMAs) of running sums
        blocks += pe_budget(f64[:, :16], fb[:, :16], e0_fast_sincos(f64[:, :16]), 6)
    blocks += pe_budget(v, torch.zeros_like(v), E0_SINCOSF, 10)
    zero = lambda n: (torch.zeros(v.shape[0], n, dtype=torch.float64, device=v.device),) * 2
    blocks.append(zero(1))
    if use_voxel:
        blocks += pe_budget(f64[:, 16:], fb[:, 16:], e0_fast_sincos(f64[:, 16:]), 6)
        blocks.append(zero(8))
    return torch.cat([b[0] for b in blocks], 1), torch.cat([b[1] for b in blocks], 1)


def x_reference_ffma(x32, feats, use_voxel):
    """float64 X of the FFMA encoder: the fp32 identity columns exact, sinf / cosf of the exact fp32 2^k f within 2 ulp
    (2^-22 absolute)."""
    def pe(vals, n_freq):
        v = vals.double()
        blocks = [(v, torch.zeros_like(v))]
        for k in range(n_freq):
            blocks += [(torch.sin(v * 2.0 ** k), torch.full_like(v, 2.0 ** -22)),
                       (torch.cos(v * 2.0 ** k), torch.full_like(v, 2.0 ** -22))]
        return blocks
    zero = lambda n: (torch.zeros(x32.shape[0], n, dtype=torch.float64, device=x32.device),) * 2
    blocks = pe(feats[2][:, :16], 6) if use_voxel else []
    blocks += pe(x32, 10) + [zero(1)]
    if use_voxel:
        blocks += pe(feats[2][:, 16:], 6) + [zero(8)]
    return torch.cat([b[0] for b in blocks], 1), torch.cat([b[1] for b in blocks], 1)


def point_in_boxes32(x, boxes):
    """point_in_boxes (field_common.cuh) step by step in fp32: row r of A p + t as ((x A0 + y A1) + z A2) + t, each
    product and sum rounded; inside = lo <= v <= hi on all three rows of any box."""
    inside = torch.zeros(x.shape[0], dtype=torch.bool, device=x.device)
    for B in boxes.float():
        inb = torch.ones_like(inside)
        for r in range(3):
            v = x[:, 0] * B[r * 3]
            v = v + x[:, 1] * B[r * 3 + 1]
            v = v + x[:, 2] * B[r * 3 + 2]
            v = v + B[9 + r]
            inb &= (v >= B[12 + r]) & (v <= B[15 + r])
        inside |= inb
    return inside


# ------------------------------------------------------------------------------------------------
# checks of the references
# ------------------------------------------------------------------------------------------------
def layer_chain(X, rc, ray, kw, use_voxel, act):
    """Run the 16 GEMM layers in kernel-K order from X with activation act(g, t) -> list of the 17 slots, and the
    pre-activations."""
    acts = [X] + [torch.zeros(X.shape[0], N_OUT[g], dtype=X.dtype) for g in GEMMS]
    pre = {}
    for i, g in enumerate(GEMMS):
        t, _ = preact(g, _wgrad_inputs(acts, use_voxel)[g], kw, rc, ray)
        pre[g] = t
        acts[i + 1] = act(g, t)
    return acts, pre


def heads(acts, pre, w):
    """sigma / rgb of both branches from the layer outputs (float64, unrounded)."""
    leaky = lambda t: torch.where(t > 0, t, 0.01 * t)
    out = {}
    for g, (name, br) in SIGMA_LAYER.items():
        out[f"sigma{br}"] = leaky(pre[g]) @ w[name][0].double().t()[:, 0] + w[name][1].double()
    for g, (name, br) in DIR_LAYER.items():
        out[f"rgb{br}"] = torch.sigmoid(leaky(pre[g]) @ w[name][0].double().t() + w[name][1].double())
    return out


@pytest.mark.parametrize("use_voxel", [True, False], ids=["voxel", "plain"])
def test_layer_chain_in_kernel_order_reproduces_the_oracle_mlp(use_voxel):
    """With exact encodings and no rounding, the kernel-K-order chain (weights mapped by kernel_weights, per-ray terms
    by ray_const_ref) is the oracle's scene_mlp / object_mlp to 1e-12; garbage in the pad columns of X changes
    nothing, and the pad columns carry zero weights in every X-fed layer."""
    rng = np.random.default_rng(21)
    w = synth.make_weights(31, use_voxel, 8.0, 1.0)
    kw = kernel_weights(w, use_voxel, bf16=False)
    n = 300
    p = torch.from_numpy(rng.uniform(-1, 8, (n, 3)))
    d = torch.nn.functional.normalize(torch.from_numpy(rng.standard_normal((n, 3))), dim=1)
    rays = torch.cat([torch.zeros(n, 3, dtype=torch.float64), d, torch.ones(n, 2, dtype=torch.float64)], 1)
    codes = torch.from_numpy(rng.standard_normal((n, synth.N_CODE)))
    emb_dir = O.posenc(d, 4)
    if use_voxel:
        g = synth.make_grid(seed=12, shape=(8, 9, 7), occupancy=0.6, voxel_size=1.0)
        grid = O.VoxelGrid(torch.zeros(3, dtype=torch.float64), 1.0, list(g["idx_map"].shape), g["idx_map"],
                           g["table"].double())
        scene_in, obj_in = O.voxel_embed(p, grid)
        X = torch.cat([scene_in, torch.full((n, 1), 1e3, dtype=torch.float64), obj_in,
                       torch.full((n, 8), -1e3, dtype=torch.float64)], 1)
    else:
        scene_in, obj_in = O.posenc(p, 10), None
        X = torch.cat([scene_in, torch.full((n, 1), 1e3, dtype=torch.float64)], 1)
    rc, _ = ray_const_ref(rays, codes, w, use_voxel)
    ray = torch.arange(n)
    acts, pre = layer_chain(X, rc, ray, kw, use_voxel, lambda g, t: t if g in ("SFIN", "OFIN") else
                            torch.where(t > 0, t, 0.01 * t))
    got = heads(acts, pre, w)
    w64 = {k: (a.double(), b.double()) for k, (a, b) in w.items()}
    s_sigma, s_rgb = O.scene_mlp(w64, scene_in, emb_dir)
    o_sigma, o_rgb = O.object_mlp(w64, scene_in, obj_in, codes, emb_dir)
    for name, a, b in (("sigma0", got["sigma0"], s_sigma), ("rgb0", got["rgb0"], s_rgb), ("sigma1", got["sigma1"], o_sigma),
                       ("rgb1", got["rgb1"], o_rgb)):
        assert b.abs().max() > 0.1, name
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-12 * b.abs().max().item()), (name, (a - b).abs().max().item())
    pads = [271] + list(range(376, 384)) if use_voxel else [63]
    for g in ("S0", "S4", "O0", "O2"):
        cols = [c for c in pads if c < kw[g][0].shape[1] and (c < 288 or g.startswith("O"))]
        assert (kw[g][0][:, cols] == 0).all(), g
    if use_voxel:      # the scene layers' columns over the object voxel PE
        assert (kw["S0"][0][:, 272:288] == 0).all() and (kw["S4"][0][:, 272:288] == 0).all()
        assert (kw["O0"][0][:, 272:288] != 0).any()


def _round_f32(x: Fraction):
    """Round a non-zero rational to the nearest float32 (ties to even), normal range."""
    e = math.floor(math.log2(abs(x)))
    while abs(x) >= Fraction(2) ** (e + 1):
        e += 1
    while abs(x) < Fraction(2) ** e:
        e -= 1
    m = round(x / Fraction(2) ** (e - 23))     # Python rounds halves to even
    return float(m * Fraction(2) ** (e - 23))


def test_fma32_rounds_once():
    """fma32 equals the exactly rounded a b + c on random operands and on sums whose float64 rounding lands on a
    float32 tie (where rounding twice goes the wrong way)."""
    rng = np.random.default_rng(5)
    a = rng.standard_normal(500).astype(np.float32)
    b = rng.standard_normal(500).astype(np.float32)
    c = rng.standard_normal(500).astype(np.float32)
    one = np.float32(1 + 2.0 ** -23)
    tie = (np.float32(1 + 2.0 ** -23), np.float32(2.0 ** -24 * (1 - 2.0 ** -23)), one)
    a, b, c = np.append(a, tie[0]), np.append(b, tie[1]), np.append(c, tie[2])
    got = fma32(*(torch.from_numpy(v) for v in (a, b, c))).numpy()
    want = [_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)]
    assert np.array_equal(got, np.array(want, dtype=np.float32))
    assert got[-1] == one and np.float32(float(a[-1]) * float(b[-1]) + float(c[-1])) != one


def test_epilogue_emulations():
    """The epilogues are non-decreasing; the bf16 LeakyReLU rounds the product once; the fp32 one rounds t * 0.01f."""
    t = torch.sort(torch.cat([torch.linspace(-3, 3, 20001, dtype=torch.float64),
                              torch.randn(20000, dtype=torch.float64) * 1e-3]))[0]
    for f in (epi_hidden, epi_fp32_leaky, epi_final, ffma_epilogue("S0"), ffma_epilogue("SFIN")):
        y = f(t)
        assert (y[1:] >= y[:-1]).all()
    assert SLOPE_BF16 == torch.tensor(0.01).to(torch.bfloat16).item()
    v = torch.tensor([-1.0, -0.375, 2.0 ** -3, -300.0], dtype=torch.float64)
    assert torch.equal(epi_hidden(v), torch.tensor([-0.010009765625, -0.003753662109375, 0.125, -3.0]).double())
    assert epi_fp32_leaky(torch.tensor([-1.0], dtype=torch.float64)).item() == bf16(torch.tensor([-SLOPE_F32])).item()


def test_gate_share():
    t = torch.tensor([1.0, 1.0, 1.0, 1.0], dtype=torch.float64)
    d = torch.full_like(t, 1e-3)
    got = torch.tensor([1.0, 1.0005, 1.002, 0.999], dtype=torch.float64)
    q = gate_share(t, d, got, lambda x: x)
    assert q[0] == 0 and 0.49 < q[1] <= 0.51 and 1.99 < q[2] <= 2.01 and 0.99 < q[3] <= 1.01


def test_pe_budget_covers_the_float32_double_angle_recurrence():
    """The double-angle recurrence emulated in fp32 (s' = fl(2 s c), c' = fmaf(-2 s, s, 1)) from an octave-0 pair
    perturbed by +-e0 in each component stays within pe_budget at every octave, for angles up to 8 (voxel features,
    __sincosf bound) and xyz positions (sincosf bound, 10 octaves)."""
    rng = np.random.default_rng(9)
    for vmax, n_freq, fast in ((8.0, 6, True), (4.0, 10, False)):
        v32 = torch.from_numpy(rng.uniform(-vmax, vmax, 40000).astype(np.float32))
        v = v32.double()
        e0 = e0_fast_sincos(v) if fast else torch.full_like(v, E0_SINCOSF)
        sgn = lambda: torch.from_numpy(rng.choice([-1.0, 1.0], v.shape[0]))
        s = (torch.sin(v) + sgn() * e0).float()
        c = (torch.cos(v) + sgn() * e0).float()
        budget = pe_budget(v, torch.zeros_like(v), e0, n_freq)
        worst = 0.0
        for k in range(n_freq):
            for val, (ref, e) in ((s, budget[1 + 2 * k]), (c, budget[2 + 2 * k])):
                r = ((val.double() - ref).abs() / e).max().item()
                worst = max(worst, r)
                assert r <= 1.0, (vmax, k, r)
            s, c = (2.0 * s) * c, fma32(-2.0 * s, s, torch.ones_like(s))
        print(f"pe budget, |v| <= {vmax}: worst error / budget {worst:.3f}")


def test_voxel_features32_is_the_trilinear_blend():
    """voxel_features32's float64 sum is the oracle's voxel_features (float64 corner weights) to the fp32 rounding of
    the corner weights, and its individually rounded fp32 sum is within the stated budget of it."""
    rng = np.random.default_rng(7)
    g = synth.make_grid(seed=3, shape=(6, 5, 7), occupancy=0.6, voxel_size=0.25, feat_scale=3.0)
    x = torch.from_numpy(rng.uniform(-1.2, 1.2, (4000, 3)).astype(np.float32))
    f64, bound, f32 = voxel_features32(x, g)
    p = ((x + g["offset"]) / g["voxel_size"]).double()
    grid = O.VoxelGrid(torch.zeros(3, dtype=torch.float64), 1.0, g["shape"].tolist(), g["idx_map"], g["table"].double())
    ref = O.voxel_features(p, grid)
    assert bound.max() > 5
    assert ((f64 - ref).abs() <= 2.0 ** -21 * bound + 1e-300).all()
    assert ((f32.double() - f64).abs() <= 16 * 2.0 ** -24 * bound).all()
