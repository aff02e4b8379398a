"""Float64 restatement of how the tensor-core backward (csrc/bwd_api.cu::bwd_pass_tc) assembles the reference-layout
gradients from the operands it keeps, for tests/test_gpu_grad_assembly.py, and the checks of it that need no device:
  - the restatement is built from the reference model's input definitions (which input feeds which reference column of
    models/nerf_model.py, as oracle/onerf_oracle.py restates them), never from pack.cu's column maps, and equals float64
    autograd of the reference-layout MLP;
  - the per-entry gate |got - want| <= c * sum|terms| (+ 2^-24 |got| for the one += into a prefilled tensor) rejects
    each layout fault a kernel could make: a shifted column segment, two swapped direction or code columns, the two
    code ray sums exchanged, = in place of +=, a kernel padding column written into a reference column;
  - a Python mirror of the training workspace offsets the GPU test reads (csrc/train_ws.h) against the library's
    sizes."""
import math

import pytest
import torch

from object_nerf_b200 import synthetic
from oracle import onerf_oracle as O
from tests import helpers
from tests.test_field_stages_cpu import GEMMS, N_OUT, REF, dims
from tests.test_gpu_train_stages import GEMM_K_PLAIN
from tests.test_gpu_train_tc import GEMM_K as GEMM_K_VOXEL

U = 2.0 ** -24
NAMES = [name for name, _, _ in synthetic.layer_dims()]          # ABI order of the 20 Linear layers
OBJ = [n for n in NAMES if n.startswith("obj.")]
# activation slot that feeds each reference layer (slot 0 = X; the output of GEMMS[i] is slot i + 1)
HEAD_IN = {"scene.sigma": 8, "scene.rgb": 10, "obj.sigma": 14, "obj.rgb": 16}
PRODUCERS = ("wgrad_w", "wgrad_b", "ray", "head_w", "head_b", "d_codes")


# ------------------------------------------------------------------------------------------------
# the restatement
# ------------------------------------------------------------------------------------------------
def ref_inputs(acts, pe, codes, use_voxel, S):
    """Per reference layer: its input segments in reference column order, each (per-sample matrix, producer), from the
    kernel-order activation slots (models/nerf_model.py:97-152: skip concats put the input first, dir concats put the
    direction last, the object input is [emb_xyz | obj_voxel | code])."""
    xin, ovx, _, _ = dims(use_voxel)
    X = acts[0]
    exyz, ovox = X[:, :xin], X[:, 272:272 + ovx]
    pe_s, code_s = pe.repeat_interleave(S, 0), codes.repeat_interleave(S, 0)
    W, R, H = "wgrad_w", "ray", "head_w"
    obj_in = [(exyz, W)] + ([(ovox, W)] if ovx else []) + [(code_s, R)]
    ins = {"scene.l0": [(exyz, W)], "scene.l4": [(exyz, W), (acts[4], W)], "scene.final": [(acts[8], W)],
           "scene.dir": [(acts[9], W), (pe_s, R)], "obj.l0": obj_in, "obj.l1": [(acts[11], W)],
           "obj.l2": obj_in + [(acts[12], W)], "obj.l3": [(acts[13], W)], "obj.final": [(acts[14], W)],
           "obj.dir": [(acts[15], W), (pe_s, R)]}
    for l in (1, 2, 3, 5, 6, 7):
        ins[f"scene.l{l}"] = [(acts[l], W)]
    for name, slot in HEAD_IN.items():
        ins[name] = [(acts[slot], H)]
    return ins


def ref_dz(dz, dA_s, dA_o):
    """Per reference layer: the gradient w.r.t. its output (GEMM layers: the dZ slot; heads: d rgb_pre / d sigma)."""
    out = {REF[g]: dz[i] for i, g in enumerate(GEMMS)}
    out.update({"scene.sigma": dA_s[:, 3:4], "scene.rgb": dA_s[:, :3], "obj.sigma": dA_o[:, 3:4], "obj.rgb": dA_o[:, :3]})
    return out


def assemble(ops, w, use_voxel, want_object, S):
    """float64 gradients of one model from the operands of one pass.
    ops: acts (17 per-sample matrices, kernel order, X with its padding columns), dz (16, GEMM order), dA_s / dA_o
    (B, 4) = d(rgb_pre, sigma_pre), pe (R, 27), codes (R, 64); w: {name: (W, b)} the fp32 reference weights.
    -> {name: (dW, db)}, {name: (bound of dW, bound of db)} (sum of |terms| per entry), {name: (producer of each dW
    entry, producer of db)} as indices into PRODUCERS, and d_codes (R, 64) with its bound; the object tensors and d_codes
    are zero with a zero bound at want_object = 0 (they must come back unchanged)."""
    ins = ref_inputs(ops["acts"], ops["pe"], ops["codes"], use_voxel, S)
    dzs = ref_dz(ops["dz"], ops["dA_s"], ops["dA_o"])
    val, bnd, prod = {}, {}, {}
    for name in NAMES:
        Wt = w[name][0]
        if name in OBJ and not want_object:
            z = torch.zeros(Wt.shape, dtype=torch.float64, device=ops["pe"].device)
            val[name], bnd[name] = (z, z[:, 0].clone()), (z, z[:, 0].clone())
            prod[name] = (torch.zeros(Wt.shape, dtype=torch.long), torch.zeros(Wt.shape[0], dtype=torch.long))
            continue
        d = dzs[name]
        segs = ins[name]
        In = torch.cat([x for x, _ in segs], 1)
        assert In.shape[1] == Wt.shape[1], name
        val[name] = (d.t() @ In, d.sum(0))
        bnd[name] = (d.abs().t() @ In.abs(), d.abs().sum(0))
        pw = torch.cat([torch.full((x.shape[1],), PRODUCERS.index(p), dtype=torch.long) for x, p in segs])
        head = name in HEAD_IN
        prod[name] = (pw.expand(Wt.shape[0], -1).clone(),
                      torch.full((Wt.shape[0],), PRODUCERS.index("head_b" if head else "wgrad_b"), dtype=torch.long))
    R = ops["pe"].shape[0]
    dc = torch.zeros(R, 64, dtype=torch.float64, device=ops["pe"].device)
    dcb = torch.zeros_like(dc)
    if want_object:
        xin, ovx, _, _ = dims(use_voxel)
        cols = slice(xin + ovx, xin + ovx + 64)
        for name in ("obj.l0", "obj.l2"):
            Wc = w[name][0][:, cols].double().to(dc.device)
            d = dzs[name]
            dc += d.view(R, S, -1).sum(1) @ Wc
            dcb += d.abs().view(R, S, -1).sum(1) @ Wc.abs()
    return val, bnd, prod, (dc, dcb)


# ------------------------------------------------------------------------------------------------
# the gate
# ------------------------------------------------------------------------------------------------
def gate_constants(B, R, S, n_sms=132):
    """c per producer, from its accumulation order (the first-order rounding bound of each sum):
      wgrad_w  per (layer, column) one wgmma accumulator per stream-K segment, one tensor-core accumulate per 16
               samples (each within 2^-22 of the running magnitude: bf16 products are exact, the tensor core's
               alignment truncates), then red.global across at most 2 x n_sms segments in fp32;
      wgrad_b  a sequential fp32 column sum per segment, atomics across segments;
      ray      the fp32 ray sums over S (S - 1 adds), then onerf_gemm over the R rays: (kps + splits + 1) 2^-24 with
               kps + splits <= R + 1 (DESIGN.md §4.4);
      head_w   atom_colsum_kernel: per-thread fmaf over at most 4 rows per tile, 32 partial rows in shared memory, atomics
               over at most min(n_tiles, 8 n_sms) CTAs;
      head_b   vec4_sum_kernel: a strided per-thread sum, 5 shuffle levels, atomics over 8 warps x 4 n_sms CTAs;
      d_codes  the ray sums, then two onerf_gemm over the 128 outputs of object layers 0 and 2, the second adding to the
               first."""
    n_tiles = (B + 127) // 128
    threads = min((B + 255) // 256, 4 * n_sms) * 256
    c = {"wgrad_w": (math.ceil(B / 16) + 1) * 4 * U + 2 * n_sms * U,
         "wgrad_b": (B + 2 * n_sms) * U,
         "ray": (S - 1 + R + 2) * U,
         "head_w": (4 * n_tiles + 32 + min(n_tiles, 8 * n_sms) + 1) * U,
         "head_b": (math.ceil(B / threads) + 5 + 8 * 4 * n_sms) * U,
         "d_codes": (S - 1 + 2 * (128 + 2) + 1) * U}
    return torch.tensor([c[p] for p in PRODUCERS], dtype=torch.float64)


def prefill_adds(R, passes=1):
    """Per producer: how many fp32 additions round onto a prefilled entry.  The kernel-layout buffer is added once
    (onerf_unpack_grads); the hoisted direction and code columns are added by onerf_gemm's atomics, once per split of its
    K = R reduction (the planner splits only K >= 256, into pieces of at least 32 rays, at most 256 of them); d_codes
    by two onerf_gemm calls (K = 128, unsplit) per pass."""
    splits = 1 if R < 256 else min(256, R // 32)
    adds = {"wgrad_w": 1, "wgrad_b": 1, "ray": splits, "head_w": 1, "head_b": 1, "d_codes": 2 * passes}
    return torch.tensor([adds[p] for p in PRODUCERS], dtype=torch.float64)


def gate_share(got, prefill, want, bound, prod, c, adds=None):
    """Share of its gate each entry uses: |got - (prefill + want)| / (c[prod] bound + adds[prod] 2^-24 max(|got|,
    |prefill| + bound) for a prefilled tensor where the bound is not 0; adds: prefill_adds, default one add).  No
    absolute floor: an entry whose gate is 0 must equal its prefill bit for bit (share 0, else inf)."""
    got, want, bound = got.double(), want.double(), bound.double()
    pre = prefill.double() if prefill is not None else torch.zeros_like(got)
    err = (got - (pre + want)).abs()
    prod = prod.to(got.device)
    tol = c.to(got.device)[prod] * bound
    if prefill is not None:     # each add onto the prefill rounds within 2^-24 of the running value
        n = adds.to(got.device)[prod] if adds is not None else 1.0
        tol = tol + torch.where(bound > 0, n * U * torch.maximum(got.abs(), pre.abs() + bound), torch.zeros_like(tol))
    share = torch.where(tol > 0, err / torch.where(tol > 0, tol, torch.ones_like(tol)), torch.zeros_like(err))
    exact = (got == pre) if prefill is not None else (got == 0)
    return torch.where((tol == 0) & ~exact, torch.full_like(err, math.inf), share)


# ------------------------------------------------------------------------------------------------
# float64 autograd of the reference-layout MLP, with the operands the kernels keep
# ------------------------------------------------------------------------------------------------
def _leaky(x):
    return torch.where(x > 0, x, x * O.LEAKY_SLOPE)


def reference_autograd(w, use_voxel, want_object, R, S, seed):
    """Random per-sample inputs through oracle.scene_mlp / object_mlp in float64 with a random linear loss on (sigma,
    rgb) -> (ops in kernel order as the backward keeps them, autograd gradients of the 40 tensors, d(codes))."""
    g = torch.Generator().manual_seed(seed)
    xin, ovx, KX, KO = dims(use_voxel)
    B = R * S
    W64 = {k: (a.double().clone().requires_grad_(), b.double().clone().requires_grad_()) for k, (a, b) in w.items()}
    emb_xyz = torch.randn(B, xin, generator=g, dtype=torch.float64)
    obj_voxel = torch.randn(B, ovx, generator=g, dtype=torch.float64) if ovx else None
    pe = torch.randn(R, 27, generator=g, dtype=torch.float64)
    codes = torch.randn(R, 64, generator=g, dtype=torch.float64).requires_grad_()
    rec = {}
    affine = O._affine

    def spy(x, wb):
        z = affine(x, wb)
        z.retain_grad()
        rec[next(k for k, v in W64.items() if v[0] is wb[0])] = z
        return z
    O._affine = spy
    try:
        sig, rgb = O.scene_mlp(W64, emb_xyz, pe.repeat_interleave(S, 0))
        loss = (torch.randn(B, generator=g, dtype=torch.float64) * sig).sum()
        loss = loss + (torch.randn(B, 3, generator=g, dtype=torch.float64) * rgb).sum()
        if want_object:
            osig, orgb = O.object_mlp(W64, emb_xyz, obj_voxel, codes.repeat_interleave(S, 0), pe.repeat_interleave(S, 0))
            loss = loss + (torch.randn(B, generator=g, dtype=torch.float64) * osig).sum()
            loss = loss + (torch.randn(B, 3, generator=g, dtype=torch.float64) * orgb).sum()
    finally:
        O._affine = affine
    loss.backward()
    X = torch.zeros(B, KO if use_voxel else KX, dtype=torch.float64)
    X[:, :xin] = emb_xyz
    if ovx:
        X[:, 272:272 + ovx] = obj_voxel
    zero = lambda n: torch.zeros(B, n, dtype=torch.float64)
    z = lambda name: rec[name].detach() if name in rec else zero(N_OUT.get(next((k for k, v in REF.items() if v == name), ""), 128))
    acts = [X] + [_leaky(z(f"scene.l{l}")) for l in range(8)] + [z("scene.final"), _leaky(z("scene.dir"))]
    acts += [_leaky(z(f"obj.l{l}")) for l in range(4)] + [z("obj.final"), _leaky(z("obj.dir"))[:, :64]]
    gz = lambda name, n: rec[name].grad if name in rec else zero(n)
    dz = [gz(REF[gm], N_OUT[gm]) for gm in GEMMS]
    dA = lambda br: torch.cat([gz(f"{br}.rgb", 3), gz(f"{br}.sigma", 1)], 1)
    ops = dict(acts=acts, dz=dz, dA_s=dA("scene"), dA_o=dA("obj"), pe=pe, codes=codes.detach())
    grads = {k: (a.grad, b.grad) for k, (a, b) in W64.items()}
    return ops, grads, codes.grad


@pytest.mark.parametrize("use_voxel", [1, 0])
@pytest.mark.parametrize("want_object", [1, 0])
def test_restatement_equals_float64_autograd_of_the_reference_mlp(use_voxel, want_object):
    w = synthetic.make_weights(31 + use_voxel, bool(use_voxel))
    R, S = 5, 7
    ops, grads, d_codes = reference_autograd(w, use_voxel, want_object, R, S, seed=3)
    val, bnd, prod, (dc, dcb) = assemble(ops, w, use_voxel, want_object, S)
    for name in NAMES:
        for i in range(2):
            want = grads[name][i]
            if want is None:          # an object tensor at want_object = 0: autograd never reached it
                assert name in OBJ and not want_object and not val[name][i].any() and not bnd[name][i].any()
                continue
            assert val[name][i].shape == want.shape, name
            assert (val[name][i] - want).abs().max().item() <= 1e-12 * max(1.0, bnd[name][i].max().item()), name
            assert (bnd[name][i] >= val[name][i].abs() * (1 - 1e-12)).all(), name
    if want_object:
        assert (dc - d_codes).abs().max().item() <= 1e-12 * max(1.0, dcb.max().item())
    else:
        assert d_codes is None and not dc.any()


# ------------------------------------------------------------------------------------------------
# planted faults: each must fail the gate at the GPU test's shapes
# ------------------------------------------------------------------------------------------------
def random_ops(use_voxel, R, S, seed):
    """Operands shaped as the GPU test reads them, bf16-valued activations and dZ, X padding columns non-zero (what a
    padding column would carry if a kernel read one)."""
    g = torch.Generator().manual_seed(seed)
    B = R * S
    widths = [384 if use_voxel else 64] + [256] * 9 + [128] * 6 + [64]
    bf = lambda t: t.to(torch.bfloat16).double()
    acts = [bf(torch.randn(B, n, generator=g, dtype=torch.float64)) for n in widths]
    dz = [bf(torch.randn(B, N_OUT[gm], generator=g, dtype=torch.float64)) for gm in GEMMS]
    return dict(acts=acts, dz=dz, dA_s=torch.randn(B, 4, generator=g, dtype=torch.float64),
                dA_o=torch.randn(B, 4, generator=g, dtype=torch.float64),
                pe=torch.randn(R, 27, generator=g, dtype=torch.float64).float().double(),
                codes=torch.randn(R, 64, generator=g, dtype=torch.float64).float().double())


def prefill_like(want, bound, gen):
    """Random fp32 prefill at the scale of the tensor's bound, so that = in place of += cannot hide under the gate."""
    return (torch.randn(want.shape, generator=gen, dtype=torch.float64) * max(1.0, bound.max().item())).float()


def _fails(got, pre, want, bound, prod, c, adds=None):
    return gate_share(got, pre, want, bound, prod, c, adds).max().item() > 1.0


# the GPU test's shapes (rays, samples per pass): 2048 x 128 is the bench batch's fine pass, where the weight-gradient
# gate is loosest
FAULT_SHAPES = [(1, 1), (37, 61), (13, 200), (2048, 64), (2048, 128)]


@pytest.mark.parametrize("use_voxel", [1, 0])
@pytest.mark.parametrize("R,S", FAULT_SHAPES)
def test_planted_layout_faults_fail_the_gate(use_voxel, R, S):
    w = synthetic.make_weights(7, bool(use_voxel))
    ops = random_ops(use_voxel, R, S, seed=R + S)
    val, bnd, prod, (dc, dcb) = assemble(ops, w, use_voxel, 1, S)
    c, adds = gate_constants(R * S, R, S), prefill_adds(R)
    g = torch.Generator().manual_seed(1)
    pre = {n: tuple(prefill_like(val[n][i], bnd[n][i], g) for i in range(2)) for n in NAMES}
    emu = {n: ((pre[n][0] + val[n][0].float()), (pre[n][1] + val[n][1].float())) for n in NAMES}   # fp32 +=
    # the emulated kernel result passes everywhere
    for n in NAMES:
        for i in range(2):
            assert not _fails(emu[n][i], pre[n][i], val[n][i], bnd[n][i], prod[n][i], c, adds), n
    assert not _fails(dc.float(), None, dc, dcb, torch.full(dc.shape, PRODUCERS.index("d_codes")), c)

    def check(name, got, label):
        assert _fails(got, pre[name][0], val[name][0], bnd[name][0], prod[name][0], c, adds), (label, name)

    xin, ovx, KX, KO = dims(use_voxel)
    oin = xin + ovx + 64
    code0 = xin + ovx
    # reference column segments fed by one kernel column block (models/nerf_model.py input definitions)
    segments = {"scene.l0": [(0, xin)], "scene.l4": [(0, xin), (xin, 256)], "obj.l0": [(0, xin), (xin, ovx)],
                "obj.l2": [(0, xin), (xin, ovx), (oin, 128)], "scene.dir": [(0, 256)], "obj.dir": [(0, 128)],
                **{f"scene.l{l}": [(0, 256)] for l in (1, 2, 3, 5, 6, 7)}, "scene.final": [(0, 256)],
                **{f"obj.l{l}": [(0, 128)] for l in (1, 3)}, "obj.final": [(0, 128)]}
    # 1. a one-column shift of any segment, either way
    for name, segs in segments.items():
        for a, n in segs:
            if n < 2:
                continue
            for sh in (1, -1):
                got = emu[name][0].clone()
                src = torch.arange(a, a + n)
                dst = (src + sh).clamp(a, a + n - 1)
                got[:, a:a + n] = pre[name][0][:, a:a + n]
                got[:, dst] = (pre[name][0][:, dst] + val[name][0][:, src].float())
                check(name, got, f"shift {sh} of [{a}, {a + n})")
    # 2. two adjacent direction or code columns swapped (in the weight gradients and in d_codes)
    for name, first, n in (("scene.dir", 256, 27), ("obj.dir", 128, 27), ("obj.l0", code0, 64), ("obj.l2", code0, 64)):
        for j in (first, first + n // 2, first + n - 2):
            got = emu[name][0].clone()
            got[:, [j, j + 1]] = pre[name][0][:, [j, j + 1]] + val[name][0][:, [j + 1, j]].float()
            check(name, got, f"columns {j}, {j + 1} swapped")
    for j in (0, 31, 62):
        got = dc.float().clone()
        got[:, [j, j + 1]] = got[:, [j + 1, j]]
        assert _fails(got, None, dc, dcb, torch.full(dc.shape, PRODUCERS.index("d_codes")), c), j
    # 3. the ray sums of object layers 0 and 2 exchanged (RC_OL0 <-> RC_OL2) on the code columns and in d_codes
    rs = {nm: ops["dz"][GEMMS.index(gm)].view(R, S, -1).sum(1) for nm, gm in (("obj.l0", "O0"), ("obj.l2", "O2"))}
    for name, other in (("obj.l0", "obj.l2"), ("obj.l2", "obj.l0")):
        got = emu[name][0].clone()
        got[:, code0:code0 + 64] = pre[name][0][:, code0:code0 + 64] + (rs[other].t() @ ops["codes"]).float()
        check(name, got, "RC_OL0 / RC_OL2 swapped")
    wc = {nm: w[nm][0][:, code0:code0 + 64].double() for nm in ("obj.l0", "obj.l2")}
    got = (rs["obj.l2"] @ wc["obj.l0"] + rs["obj.l0"] @ wc["obj.l2"]).float()
    assert _fails(got, None, dc, dcb, torch.full(dc.shape, PRODUCERS.index("d_codes")), c), "d_codes with RC_OL0 / RC_OL2"
    # 4. = in place of += (every tensor, weights and biases)
    for name in NAMES:
        assert _fails(val[name][0].float(), pre[name][0], val[name][0], bnd[name][0], prod[name][0], c, adds), name
        assert _fails(val[name][1].float(), pre[name][1], val[name][1], bnd[name][1], prod[name][1], c, adds), name
    # 5. a kernel padding column added to the reference column next to it: X columns [xin, KX) and [272 + ovx, KO)
    #    (voxel: also 271), the pad of the object voxel block, and the last kernel column of X read for the next one
    X = ops["acts"][0]
    pads = [("scene.l0", xin - 1, xin, "S0"), ("scene.l4", xin - 1, xin, "S4"), ("obj.l0", xin - 1, xin, "O0"),
            ("obj.l2", xin - 1, xin, "O2")]
    if use_voxel:
        pads += [("obj.l0", xin + ovx - 1, 272 + ovx, "O0"), ("obj.l2", xin + ovx - 1, 272 + ovx, "O2")]
    for name, ref_col, kcol, gm in pads:
        got = emu[name][0].clone()
        got[:, ref_col] += (ops["dz"][GEMMS.index(gm)].t() @ X[:, kcol]).float()
        check(name, got, f"padding column {kcol} into {ref_col}")


def test_gate_rejects_changes_to_untouched_entries():
    """An entry whose bound is 0 must be its prefill bit for bit: one ulp off fails."""
    c = gate_constants(128, 2, 64)
    pre = torch.tensor([1.5, -2.0, 0.25])
    z = torch.zeros(3, dtype=torch.float64)
    prod = torch.zeros(3, dtype=torch.long)
    assert gate_share(pre.clone(), pre, z, z, prod, c).max().item() == 0.0
    off = pre.clone()
    off[1] = torch.nextafter(off[1], torch.tensor(0.0))
    assert gate_share(off, pre, z, z, prod, c)[1].item() == math.inf


# ------------------------------------------------------------------------------------------------
# the workspace offsets the GPU test reads (csrc/train_ws.h)
# ------------------------------------------------------------------------------------------------
GEMM_K = {1: GEMM_K_VOXEL, 0: GEMM_K_PLAIN}      # kernel K per GEMM layer (csrc/layout.h)
RAY_CONST_FLOATS = 448


def grad_buffer_floats(use_voxel):
    off = 0
    for g in GEMMS:
        off = (off + N_OUT[g] * GEMM_K[use_voxel][g] + N_OUT[g] + 3) // 4 * 4
    for n in (256, 1, 384, 3, 128, 1, 192, 3):
        off += (n + 3) // 4 * 4
    return off


def train_ws(use_voxel, n_rays, n_samples, n_importance):
    """TrainWs of the bf16 path: byte offsets of every buffer, then TrainStepWs after it."""
    a1k = lambda x: (x + 1023) // 1024 * 1024
    sf = n_samples + n_importance
    Bc, Bf = n_rays * n_samples, n_rays * sf
    o, W = 0, {}
    for name, nbytes in (("tl_coarse", helpers.train_layout(bool(use_voxel), Bc)["total"]),
                         ("tl_fine", helpers.train_layout(bool(use_voxel), Bf)["total"] if n_importance else 0),
                         ("scene_c", Bc * 16), ("obj_c", Bc * 16), ("scene_f", Bf * 16), ("obj_f", Bf * 16),
                         ("dscene", Bf * 16), ("dobj", Bf * 16), ("dA_s", Bf * 16), ("dA_o", Bf * 16),
                         ("rs", n_rays * RAY_CONST_FLOATS * 4), ("pe", n_rays * 27 * 4),
                         ("gk", grad_buffer_floats(use_voxel) * 4)):
        W[name] = o
        o += a1k(nbytes)
    W["total"] = o
    for name, nbytes in (("dscene_c", Bc * 16), ("dobj_c", Bc * 16), ("loss", 256)):
        W[name] = o
        o += a1k(nbytes)
    W["step_total"] = o
    return W


@pytest.fixture(scope="module")
def lib():
    from object_nerf_b200 import _lib
    import os
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.load()


def test_train_workspace_mirror_matches_the_library(lib):
    from object_nerf_b200 import _lib
    for uv in (0, 1):
        assert lib.onerf_grad_buffer_floats(uv) == grad_buffer_floats(uv)
        for n, s, si in ((1, 1, 0), (1, 1, 1), (37, 61, 0), (37, 61, 64), (13, 200, 0), (2048, 64, 64), (4096, 64, 0),
                         (3, 2048, 0), (0, 64, 64), (129, 1, 127)):
            W = train_ws(uv, n, s, si)
            assert lib.onerf_train_workspace_bytes_prec(_lib.PREC_BF16, uv, n, s, si) == W["total"], (uv, n, s, si)
            assert lib.onerf_train_step_workspace_bytes(_lib.PREC_BF16, uv, n, s, si) == W["step_total"], (uv, n, s, si)
            assert lib.onerf_field_train_bytes(uv, n * s) == helpers.train_layout(bool(uv), n * s)["total"]
