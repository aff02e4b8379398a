"""The fp32 training backward (precision="fp32", csrc/bwd_api.cu::bwd_pass_fp32) at batch size, where it runs in
chunks of onerf_fp32_chunk_rays rays:
  1. its building blocks (csrc/backward.cu) against exact references: onerf_gemm bit-exact on integer operands in every
     split regime, with wide leading dimensions, odd offsets and canaries around every block, and within the rigorous
     rounding bound on random operands; onerf_colsum and onerf_segment_sum on integer operands; onerf_leaky_bwd and
     onerf_head_bwd bit-exact against fp32 torch; onerf_dir_encode within 2 ulp of float64 sin / cos;
  2. the chunked field backward by additivity: for a loss linear in the maps, the gradients of a multi-chunk batch equal
     the float64 sum of the gradients of single-chunk sub-batches (the principle is checked on the float64 oracle in
     tests/test_fp32_backward_cpu.py, which also holds the shapes and the restated planning).
Each gate check prints the largest share of its gate that a result used (RATIO label: x)."""
import numpy as np
import pytest
import torch

from tests import helpers
from tests.test_fp32_backward_cpu import (ADDITIVITY_CASES, COLSUM_SHAPES, GEMM_RANDOM_MAX_K, GEMM_REGIMES, GEMM_SHAPES,
                                          INT_RANGE, SEGSUM_SHAPES, chunk_list, colsum_strips, gemm_plan, gemm_regimes,
                                          grad_case, map_keys, map_weights)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CANARY = 0x7FC0DEAD          # a quiet-NaN bit pattern around every block a kernel reads or writes


def _lib():
    from object_nerf_b200 import _lib
    return _lib


def _call(name, *args):
    L = _lib()
    L.check(getattr(L.load(), name)(L.ctx(torch.device(DEV)), *args, L.stream()))
    torch.cuda.synchronize()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ratio(label, err, gate):
    r = (err / gate).max().item() if err.numel() else 0.0
    print(f"RATIO {label}: {r:.3e}")
    return r


def _ints(gen, *shape):
    return torch.randint(-INT_RANGE, INT_RANGE + 1, shape, generator=gen, device=DEV).float()


class Embedded:
    """A [rows x cols] fp32 block at float offset `off` of a canary-filled buffer, rows `ld` floats apart."""

    def __init__(self, fill, ld=None, off=0):
        rows, cols = fill.shape
        self.ld = cols if ld is None else ld
        n = off + (rows - 1) * self.ld + cols
        self.buf = torch.full((n + 5,), CANARY, dtype=torch.int32, device=DEV).view(torch.float32)
        self.mask = torch.zeros(n + 5, dtype=torch.bool, device=DEV)
        view = lambda t: t.as_strided((rows, cols), (self.ld, 1), off)
        self.block = view(self.buf)
        view(self.mask).fill_(True)
        self.block.copy_(fill)

    def ptr(self):
        return self.block.data_ptr()

    def canaries_intact(self):
        return bool((self.buf.view(torch.int32)[~self.mask] == CANARY).all())


def _padded(fill, padded):
    """Rows 7 floats wider than the block and an odd float offset when `padded`."""
    return Embedded(fill, ld=fill.shape[1] + 7, off=3) if padded else Embedded(fill)


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ------------------------------------------------------------------------------------------------
# 1. building blocks
# ------------------------------------------------------------------------------------------------
def _gemm_id(s):
    M, N, K, ta, acc, padded = s
    return f"M{M}_N{N}_K{K}_ta{ta}_acc{acc}" + ("_padded" if padded else "")


def _gemm(a, b, c0, ta, acc, padded):
    """onerf_gemm on a, b into c0's values, every operand embedded in canaries -> C's embedding."""
    M, N = c0.shape
    K = b.shape[0]
    A, B, Cm = _padded(a, padded), _padded(b, padded), _padded(c0, padded)
    _call("onerf_gemm", A.ptr(), A.ld, ta, B.ptr(), B.ld, Cm.ptr(), Cm.ld, M, N, K, acc)
    return Cm


def test_gemm_shapes_hit_every_split_regime_on_this_device():
    sms = _sms()
    hit = set().union(*(gemm_regimes(M, N, K, acc, sms) for M, N, K, _, acc, _ in GEMM_SHAPES))
    print(f"{sms} SMs: regimes {sorted(hit)}")
    assert hit == GEMM_REGIMES, GEMM_REGIMES - hit


@pytest.mark.parametrize("shape", GEMM_SHAPES, ids=_gemm_id)
def test_gemm_integer_operands_bit_exact(shape):
    """C (+)= op(A) B on integers in {-3..3}: every partial sum is an exact fp32 integer, so the result must equal the
    float64 product whatever the split or the order of the atomics.  Every element of the buffers around A, B and C is
    a NaN canary: a read outside A or B poisons C, a write outside C (the memset of a split that overwrites included)
    changes a canary."""
    M, N, K, ta, acc, padded = shape
    gen = torch.Generator(device=DEV).manual_seed(M * 7919 + N * 31 + K)
    a = _ints(gen, *((K, M) if ta else (M, K)))
    b, c0 = _ints(gen, K, N), _ints(gen, M, N)
    p = gemm_plan(M, N, K, acc, _sms())
    Cm = _gemm(a, b, c0, ta, acc, padded)
    want = (a.double().t() if ta else a.double()) @ b.double() + (c0.double() if acc else 0.0)
    assert torch.equal(Cm.block.double(), want), (p, (Cm.block.double() - want).abs().max().item())
    assert Cm.canaries_intact(), p


@pytest.mark.parametrize("shape", [s for s in GEMM_SHAPES if s[2] <= GEMM_RANDOM_MAX_K], ids=_gemm_id)
def test_gemm_random_operands_within_the_rounding_bound(shape):
    """Random normal operands: |got - ref64| <= (kps + splits + 1) 2^-24 (sum |a||b| + |C0|): at most kps fused
    multiply-adds in a split and `splits` atomic additions lie on any path to an output."""
    M, N, K, ta, acc, padded = shape
    gen = torch.Generator(device=DEV).manual_seed(K * 131 + M)
    a = torch.randn(*((K, M) if ta else (M, K)), generator=gen, device=DEV)
    b, c0 = torch.randn(K, N, generator=gen, device=DEV), torch.randn(M, N, generator=gen, device=DEV)
    p = gemm_plan(M, N, K, acc, _sms())
    Cm = _gemm(a, b, c0, ta, acc, padded)
    a64 = a.double().t() if ta else a.double()
    want = a64 @ b.double() + (c0.double() if acc else 0.0)
    mag = a64.abs() @ b.double().abs() + (c0.double().abs() if acc else 0.0)
    gate = (p["kps"] + p["splits"] + 1) * 2.0 ** -24 * mag + 1e-300
    err = (Cm.block.double() - want).abs()
    _ratio(f"gemm {_gemm_id(shape)} (kps {p['kps']}, splits {p['splits']})", err, gate)
    assert (err <= gate).all(), (p, (err / gate).max().item())
    assert Cm.canaries_intact()


@pytest.mark.parametrize("shape", COLSUM_SHAPES, ids=lambda s: f"rows{s[0]}_cols{s[1]}_ld{s[2]}")
def test_colsum_integer_operands_exact(shape):
    """out[c] += sum over rows of in[r][c], into a preset out, on integers: exact.  The input block sits in canaries
    (ld wider than cols where the shape says so), so a row past a strip's end or a padding column poisons the sum."""
    rows, cols, ld = shape
    gen = torch.Generator(device=DEV).manual_seed(rows + cols)
    x, preset = _ints(gen, rows, cols), _ints(gen, 1, cols)
    In, Out = Embedded(x, ld=ld, off=5), Embedded(preset, off=3)
    _call("onerf_colsum", In.ptr(), In.ld, rows, cols, Out.ptr())
    want = preset.double() + x.double().sum(0, keepdim=True)
    print(f"colsum {shape}: blocks, rows per block, empty strips = {colsum_strips(rows, _sms())}")
    assert torch.equal(Out.block.double(), want), (Out.block.double() - want).abs().max().item()
    assert Out.canaries_intact()


@pytest.mark.parametrize("shape", SEGSUM_SHAPES, ids=lambda s: "_".join(map(str, s)))
def test_segment_sum_integer_operands_exact(shape):
    """out[r][c] = sum over the S rows of ray r of in[r S + s][c], overwriting a preset out: exact on integers, nothing
    written between or around the output rows, nothing read outside the input block."""
    n, S, cols, ld_in, ld_out = shape
    gen = torch.Generator(device=DEV).manual_seed(n * S + cols)
    x, preset = _ints(gen, n * S, cols), _ints(gen, n, cols)
    In, Out = Embedded(x, ld=ld_in, off=1), Embedded(preset, ld=ld_out, off=3)
    _call("onerf_segment_sum", In.ptr(), In.ld, Out.ptr(), Out.ld, n, S, cols)
    want = x.double().view(n, S, cols).sum(1)
    assert torch.equal(Out.block.double(), want), (Out.block.double() - want).abs().max().item()
    assert Out.canaries_intact()


_F = lambda v: float(np.float32(v))
LEAKY_SPECIALS = [0.0, -0.0, 1e-40, -1e-40, 1.4e-45, -1.4e-45, float("nan"), -float("nan"), float("inf"), -float("inf"),
                  _F(1.1754944e-38), -_F(1.1754944e-38), 1.0, -1.0]


@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (37, 5, 9, 6), (1000, 128, 256, 128), (70000, 64, 256, 64)],
                         ids=lambda s: "_".join(map(str, s)))
def test_leaky_bwd_bit_exact(shape):
    """d <- d * (h > 0 ? 1 : 0.01) in place, bit for bit the fp32 torch expression, on strided d and h, with h = +0, -0,
    subnormals of both signs, NaN of both signs, infinities and the smallest normals planted (only h > 0, positive
    subnormals included, keeps slope 1, as in torch's LeakyReLU backward); some d subnormal too."""
    rows, cols, ld_d, ld_h = shape
    gen = torch.Generator(device=DEV).manual_seed(rows + cols)
    h = torch.randn(rows, cols, generator=gen, device=DEV)
    d = torch.randn(rows, cols, generator=gen, device=DEV)
    sp = torch.tensor(LEAKY_SPECIALS, device=DEV)
    hf, df = h.view(-1), d.view(-1)
    hf[::3] = sp.repeat(hf[::3].numel() // sp.numel() + 1)[:hf[::3].numel()]
    df[1::7] = 3e-39
    D, H = Embedded(d, ld=ld_d, off=1), Embedded(h, ld=ld_h, off=2)
    _call("onerf_leaky_bwd", D.ptr(), D.ld, H.ptr(), H.ld, rows, cols)
    hc, dc = h.cpu(), d.cpu()
    want = dc * torch.where(hc > 0, 1.0, 0.01)
    assert _bits_equal(D.block.cpu(), want)
    assert D.canaries_intact() and H.canaries_intact()


@pytest.mark.parametrize("n", [1, 1001, 700001])
def test_head_bwd_bit_exact(n):
    """dA = ((g f) (1 - f) for rgb, g for sigma) bit for bit the fp32 torch expression, with f = 0 and f = 1 planted and
    muted samples (sigma = -1e5, whose sigma gradient passes through unchanged); nothing written around dA."""
    gen = torch.Generator(device=DEV).manual_seed(n)
    g = torch.randn(n, 4, generator=gen, device=DEV)
    f = torch.rand(n, 4, generator=gen, device=DEV)
    f[::5, :3] = 0.0
    f[1::5, :3] = 1.0
    f[:, 3] = torch.randn(n, generator=gen, device=DEV) * 10
    f[2::3, 3] = -1e5
    out = Embedded(torch.zeros(n, 4, device=DEV), ld=4, off=4)         # float4 stores: keep 16-byte alignment
    _call("onerf_head_bwd", g.data_ptr(), f.data_ptr(), out.ptr(), n)
    gc, fc = g.cpu(), f.cpu()
    got = out.block.cpu()
    assert _bits_equal(got[:, :3], (gc[:, :3] * fc[:, :3]) * (1 - fc[:, :3]))
    assert _bits_equal(got[:, 3], gc[:, 3])
    assert out.canaries_intact()


@pytest.mark.parametrize("n", [1, 85, 86, 100003])
def test_dir_encode_within_two_ulp(n):
    """PE4 of the ray directions: column c is d exactly; sin / cos of d 2^k (exact arguments) within 2 fp32 ulp of
    float64, the documented accuracy of sinf / cosf.  Ray counts around the 256-thread block (3 threads per ray)."""
    gen = torch.Generator(device=DEV).manual_seed(n)
    rays = torch.randn(n, 8, generator=gen, device=DEV)
    rays[:, 3:6] /= rays[:, 3:6].norm(dim=1, keepdim=True)
    planted = torch.tensor([0.0, -0.0, 1.0, -1.0, _F(np.pi / 8), _F(np.pi / 4), _F(-np.pi / 2), _F(3 * np.pi / 8),
                            1e-30, -2e-42], device=DEV)
    d = rays[:, 3:6].reshape(-1).clone()
    d[: min(d.numel(), planted.numel())] = planted[: d.numel()]
    rays[:, 3:6] = d.view(n, 3)
    out = Embedded(torch.zeros(n, 27, device=DEV), off=3)
    _call("onerf_dir_encode", rays.data_ptr(), n, out.ptr())
    got = out.block.cpu()
    dc = rays[:, 3:6].cpu()
    assert _bits_equal(got[:, :3], dc)
    worst = 0.0
    for k in range(4):
        arg = dc.double().numpy() * 2.0 ** k
        for col, fn in ((3 * (1 + 2 * k), np.sin), (3 * (2 + 2 * k), np.cos)):
            ref = fn(arg)
            ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
            err = np.abs(got[:, col:col + 3].double().numpy() - ref)
            worst = max(worst, float((err / ulp).max()))
            assert (err <= 2 * ulp).all(), (k, fn.__name__, float((err / ulp).max()))
    print(f"RATIO dir_encode n={n}: {worst / 2:.3e}")
    assert out.canaries_intact()


# ------------------------------------------------------------------------------------------------
# 2. the chunked field backward by additivity
# ------------------------------------------------------------------------------------------------
def _setup(c, inp):
    from object_nerf_b200 import Embedding
    uv = c["use_voxel"]
    models = {k: helpers.make_model(w, uv, DEV).train() for k, w in inp["weights"].items()}
    emb = helpers.GridModule(inp["grid"]).to(DEV) if uv else Embedding(3, 10)
    lib = helpers.CodeLib(inp["code_table"]).to(DEV)
    named = [(f"{typ}.{k}", p) for typ, m in models.items() for k, p in m.named_parameters()]
    named.append(("codes", lib.embedding_instance.weight))
    if uv:
        named.append(("voxel", emb.embedding_space_ftr.weight))
    return models, emb, lib, named


def _linear_step(c, inp, setup, G, a, b):
    """render_rays(precision="fp32") on rays [a, b) with every injected input sliced, then backward of sum(map * G):
    -> (returned maps, {parameter: gradient as float64 or None})."""
    from object_nerf_b200 import Embedding, render_rays
    models, emb, lib, named = setup
    for _, p in named:
        p.grad = None
    sl = slice(a, b)
    codes = lib.embedding_instance(inp["instance_ids"].view(-1)[sl].to(DEV))
    out = render_rays(models, {"xyz": emb, "dir": Embedding(3, 4)}, inp["rays"][sl].to(DEV), N_samples=c["n_samples"],
                      perturb=c["perturb"], noise_std=c["noise_std"], N_importance=c["n_importance"],
                      white_back=c["white_back"], forward_instance=c["forward_instance"], embedding_instance=codes,
                      frustum_bound_th=c["frustum_bound_th"], pass_through_mask=inp["pass_through_mask"][sl].to(DEV),
                      is_eval=False, precision="fp32", _rand={k: v[sl].to(DEV) for k, v in inp["rand"].items()})
    sum((out[k] * G[k][sl]).sum() for k in G).backward()
    torch.cuda.synchronize()
    return ({k: v.detach().clone() for k, v in out.items()},
            {name: (p.grad.detach().double().clone() if p.grad is not None else None) for name, p in named})


@pytest.mark.parametrize("case", list(ADDITIVITY_CASES))
def test_chunked_backward_is_additive_over_sub_batches(case):
    """L = sum over every returned rgb / depth / opacity map (scene and instance, coarse and fine) of sum(map * G) is
    linear in the maps and every op of render_rays is per ray, so the gradients of a batch are exactly the sums of the
    gradients of a partition of its rays.  The full batch runs in several fp32 chunks per pass, the last one ragged;
    each sub-batch is one chunk per pass.  Maps: bit-identical to the concatenated sub-batch maps.  Gradients (80 MLP
    tensors, code table, voxel table): |full - float64 sum of parts| <= 1e-5 relative in norm, and every entry within
    1e-3 of the tensor's RMS entry (a chunk-offset bug moves entries by O(RMS)).  The head biases (sigma, rgb and their
    object twins, 1 or 3 entries) have a norm gate of 1e-4 instead: each entry is one column sum of ~10^5 per-sample
    terms that largely cancel, and the order of the fp32 atomics alone moves the scene-only fine sigma bias by 1.3e-5
    between two identical full-batch runs (H100)."""
    spec = ADDITIVITY_CASES[case]
    c, inp = grad_case(spec)
    n, cuts = c["n_rays"], spec["cuts"]
    order = ["coarse"] + (["fine"] if c["n_importance"] else [])
    print(case, "chunks per pass:", [chunk_list(n, s) for s in [c["n_samples"], c["n_samples"] + c["n_importance"]][:len(order)]])
    G = {k: v.to(DEV) for k, v in map_weights(n, map_keys(order, c["forward_instance"]), seed=33).items()}
    setup = _setup(c, inp)
    maps, full = _linear_step(c, inp, setup, G, 0, n)
    parts = [_linear_step(c, inp, setup, G, a, b) for a, b in zip(cuts[:-1], cuts[1:])]
    assert set(maps) == set(parts[0][0])
    for k, v in maps.items():
        assert _bits_equal(v, torch.cat([p[0][k] for p in parts])), k
    worst_norm, worst_head, worst_entry, n_checked = (0.0, ""), (0.0, ""), (0.0, ""), 0
    for name, g in full.items():
        sub = [p[1][name] for p in parts]
        if all(s is None or not s.any() for s in sub):
            assert g is None or not g.any(), (name, "gradient where no sub-batch has one")
            assert c["forward_instance"] is False and (name == "codes" or ".inst" in name), name
            continue
        ref = sum(s for s in sub if s is not None)
        rel = ((g - ref).norm() / ref.norm()).item()
        rms = ref.norm().item() / g.numel() ** 0.5
        ent = (g - ref).abs().max().item() / rms
        head_bias = g.numel() <= 3
        norm_gate = 1e-4 if head_bias else 1e-5
        worst_head = max(worst_head, (rel / norm_gate, name)) if head_bias else worst_head
        worst_norm = worst_norm if head_bias else max(worst_norm, (rel / norm_gate, name))
        worst_entry = max(worst_entry, (ent / 1e-3, name))
        n_checked += 1
        assert rel <= norm_gate, (name, rel)
        assert ent <= 1e-3, (name, ent)
    print(f"RATIO additivity {case} norm gate 1e-5: {worst_norm[0]:.3e} ({worst_norm[1]})")
    print(f"RATIO additivity {case} head-bias norm gate 1e-4: {worst_head[0]:.3e} ({worst_head[1]})")
    print(f"RATIO additivity {case} entry gate: {worst_entry[0]:.3e} ({worst_entry[1]})")
    # per model 24 scene tensors (12 linears) and 16 object tensors (8 linears)
    fi = int(c["forward_instance"])
    assert n_checked == len(order) * (24 + 16 * fi) + fi + int(c["use_voxel"]), n_checked
