"""Shapes and references for the tests of the fp32 training backward at batch size (tests/test_gpu_fp32_backward.py),
and the checks of them that need no device:
  - Python restatements of onerf_fp32_chunk_rays (csrc/train_ws.h), of onerf_gemm's split planning and of onerf_colsum's
    strips (csrc/backward.cu), with their constants parsed from the sources so the restatements fail if those drift;
  - the chunk lists of every multi-chunk case, and that each sub-batch of the additivity cases is one chunk per pass;
  - that the GEMM shape list reaches every split regime on 132 and on 114 SMs (H100 SXM and PCIe);
  - that every integer-operand GEMM, column sum and segment sum stays below 2^24 in every partial sum, so any order of
    summation is exact;
  - the additivity principle the GPU test rests on, on the float64 oracle: the parameter gradients of a loss that is
    linear in the maps equal the sum of the gradients of any partition of the rays into sub-batches."""
import math
import os
import re

import pytest
import torch

from oracle import onerf_oracle as O
from tests import cases, grad_plain, helpers

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "object_nerf_b200", "csrc")
SM_COUNTS = (132, 114)      # H100 SXM, H100 PCIe


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


CHUNK_SAMPLES = int(re.search(r"#define ONERF_FP32_CHUNK_SAMPLES (\d+)", _source("train_ws.h")).group(1))
_gb = re.search(r"constexpr int GB = (\d+), GK = (\d+);", _source("backward.cu"))
GB, GK = int(_gb.group(1)), int(_gb.group(2))


# ------------------------------------------------------------------------------------------------
# restatements of the host-side planning
# ------------------------------------------------------------------------------------------------
def chunk_rays(n_rays, n_samples):
    """onerf_fp32_chunk_rays: whole rays of at most CHUNK_SAMPLES samples per chunk, at least one ray."""
    r = max(1, CHUNK_SAMPLES // n_samples) if n_samples > 0 else 1
    return min(r, n_rays)


def chunk_list(n_rays, n_samples):
    """Ray counts of the chunks bwd_pass_fp32 walks."""
    c = chunk_rays(n_rays, n_samples)
    return [min(c, n_rays - r0) for r0 in range(0, n_rays, c)]


def gemm_plan(M, N, K, accumulate, sms):
    """onerf_gemm's launch: (gx, gy) output tiles, the split count before (`capped`) and after the minimum-rows loop
    (`looped`), then kps rows per split rounded up to GK and the final split count; `memset` when the split overwrites."""
    gx, gy = -(-N // GB), -(-M // GB)
    splits, want, capped, looped = 1, None, None, None
    if K >= 256 and gx * gy < 2 * sms:
        want = -(-(4 * sms) // (gx * gy))
        capped = min(max(want, 1), 256)
        min_k = 512 if K >= 4096 else 32
        splits = capped
        while splits > 1 and K // splits < min_k:
            splits -= 1
        looped = splits
    kps = -(-(-(-K // splits)) // GK) * GK
    splits = -(-K // kps)
    return dict(gx=gx, gy=gy, want=want, capped=capped, looped=looped, kps=kps, splits=splits,
                memset=splits > 1 and not accumulate)


def gemm_regimes(M, N, K, accumulate, sms):
    """The planning regimes a call takes on `sms` SMs."""
    p = gemm_plan(M, N, K, accumulate, sms)
    r = set()
    if K < 256:
        r.add("k_below_256")
    elif p["want"] is None:
        r.add("grid_fills_machine")
    elif p["looped"] < p["capped"]:
        r.add("min_32_rows" if K < 4096 else "min_512_rows")
    if p["want"] is not None and p["want"] > 256 and p["splits"] == 256:
        r.add("cap_256_splits")
    if p["memset"]:
        r.add("memset_then_split")
    return r


GEMM_REGIMES = {"k_below_256", "grid_fills_machine", "min_32_rows", "min_512_rows", "cap_256_splits",
                "memset_then_split"}


def colsum_strips(rows, sms):
    """onerf_colsum's launch: (blocks, rows per block, blocks whose strip is empty)."""
    blocks = min(rows // 256 + 1, 4 * sms)
    per = -(-rows // blocks)
    return blocks, per, sum(1 for b in range(blocks) if b * per >= rows)


# ------------------------------------------------------------------------------------------------
# shapes of the kernel tests
# ------------------------------------------------------------------------------------------------
# M, N, K, trans_a, accumulate, padded.  padded: lda, ldb and ldc wider than the matrix and A, B, C at odd float offsets
# inside larger buffers, as the fp32 backward addresses a column block of dW or of a weight matrix.
GEMM_SHAPES = [
    (1, 1, 1, 0, 0, False),
    (1, 1, 1, 1, 1, True),
    (70, 50, 33, 0, 1, True),
    (127, 27, 200, 1, 0, True),
    (128, 27, 1100, 1, 1, True),        # dir columns of a dW over a 1 100-ray batch
    (64, 64, 1000, 1, 0, True),
    (1100, 64, 128, 0, 1, True),        # d_codes: per-ray sums times a column block of W
    (256, 271, 9000, 1, 1, True),
    (1, 300, 20000, 1, 0, True),
    (33, 17, 131072, 1, 0, True),
    (1100, 1100, 300, 0, 0, True),
]
GEMM_RANDOM_MAX_K = 4096     # the rigorous random-operand bound is only tight enough to mean something up to here
INT_RANGE = 3                # integer operands and initial C drawn from {-3..3}

# rows, cols, ld.  140 000 rows: the strip count is capped at 4 SMs and the last strips are empty on 132 and 114 SMs;
# 1 000 003 rows: far more than 4 SMs x 256.
COLSUM_SHAPES = [(1, 1, 1), (100, 3, 4), (255, 300, 301), (1000, 1, 1), (140000, 2, 3), (1000003, 5, 7)]
# rays, samples per ray, cols, ld_in, ld_out.  (1100, 127, 128, 256, 128) is the fp32 backward's call on the per-ray
# sums of a 256-wide dZ buffer; the last shape has more elements than the grid-stride launch has threads.
SEGSUM_SHAPES = [(1, 1, 1, 1, 1), (37, 1, 128, 256, 128), (5, 7, 1, 3, 2), (1100, 127, 128, 256, 128),
                 (5000, 3, 130, 131, 133)]

# The chunked field backward by additivity: cases and sub-batch cuts (ray indices)
ADDITIVITY_CASES = {
    "ragged_both": dict(use_voxel=True, n_rays=1100, n_samples=64, n_importance=63, forward_instance=True,
                        cuts=(0, 300, 777, 1100)),
    "ragged_plain": dict(use_voxel=False, n_rays=1100, n_samples=64, n_importance=63, forward_instance=True,
                         cuts=(0, 300, 777, 1100)),
    "long_rays": dict(use_voxel=True, n_rays=70, n_samples=2048, n_importance=0, forward_instance=True,
                      cuts=(0, 20, 45, 70)),
    "scene_only": dict(use_voxel=True, n_rays=1100, n_samples=64, n_importance=63, forward_instance=False,
                       cuts=(0, 300, 777, 1100)),
}
# the one float64 oracle step across a chunk boundary, and the fused steps at batch size
ORACLE_TWO_CHUNKS = dict(use_voxel=True, n_rays=1030, n_importance=0)
FUSED_STEP_SHAPES = {"batch_2048_64_64": (2048, 64, 64), "ragged_1100_64_63": (1100, 64, 63)}

EXPECTED_CHUNKS = {   # (rays, samples per ray) -> chunk list
    (1100, 64): [1024, 76], (1100, 127): [516, 516, 68], (70, 2048): [32, 32, 6], (1030, 64): [1024, 6],
    (2048, 64): [1024, 1024], (2048, 128): [512] * 4,
}


# ------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------
def test_restated_planning_reads_the_sources():
    """The parsed constants, and the lines of onerf_gemm / onerf_colsum the restatements copy, as the sources hold them."""
    assert CHUNK_SAMPLES == 65536 and (GB, GK) == (64, 16)
    src = _source("backward.cu")
    for line in ("if (K >= 256 && gx * gy < 2 * ctx->num_sms) {",
                 "const int want = (4 * ctx->num_sms + gx * gy - 1) / (gx * gy);",
                 "splits = want < 1 ? 1 : (want > 256 ? 256 : want);",
                 "const int min_k = K >= 4096 ? 512 : 32;",
                 "while (splits > 1 && K / splits < min_k) --splits;",
                 "int kps = ((K + splits - 1) / splits + GK - 1) / GK * GK;",
                 "splits = (K + kps - 1) / kps;",
                 "if (splits > 1 && !accumulate) {",
                 "int blocks = (int)(rows / 256 + 1 < (int64_t)ctx->num_sms * 4 ? rows / 256 + 1 : (int64_t)ctx->num_sms * 4);",
                 "const int64_t rows_per_block = (rows + gridDim.x - 1) / gridDim.x;"):
        assert line in src, line
    assert "r = n_samples > 0 ? ONERF_FP32_CHUNK_SAMPLES / n_samples : 1;" in _source("train_ws.h")


def test_chunk_lists_of_the_multi_chunk_cases():
    for (n, s), want in EXPECTED_CHUNKS.items():
        assert chunk_list(n, s) == want, (n, s, chunk_list(n, s))
    assert chunk_list(3, 70000) == [1, 1, 1]           # one ray when a single ray has more samples than a chunk
    for name, c in ADDITIVITY_CASES.items():
        passes = [c["n_samples"]] + ([c["n_samples"] + c["n_importance"]] if c["n_importance"] else [])
        assert all(len(chunk_list(c["n_rays"], s)) > 1 for s in passes), name
        assert min(chunk_list(c["n_rays"], s)[-1] for s in passes) < chunk_rays(c["n_rays"], passes[0]), name   # ragged
        cuts = c["cuts"]
        assert cuts[0] == 0 and cuts[-1] == c["n_rays"] and list(cuts) == sorted(set(cuts)), name
        for a, b in zip(cuts[:-1], cuts[1:]):
            for s in passes:
                assert chunk_list(b - a, s) == [b - a], (name, a, b, s)
    assert chunk_list(ORACLE_TWO_CHUNKS["n_rays"], cases.GRAD_CASE["n_samples"]) == [1024, 6]
    for n, s, k in FUSED_STEP_SHAPES.values():
        assert len(chunk_list(n, s)) > 1 and len(chunk_list(n, s + k)) > 1


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_gemm_shapes_reach_every_split_regime(sms):
    hit = set()
    for M, N, K, _, acc, _ in GEMM_SHAPES:
        hit |= gemm_regimes(M, N, K, acc, sms)
    assert hit == GEMM_REGIMES, GEMM_REGIMES - hit
    shapes = [(M, N, K, ta) for M, N, K, ta, _, _ in GEMM_SHAPES]
    assert {ta for *_, ta in shapes} == {0, 1} and {1} <= {M for M, *_ in shapes} and {1} <= {N for _, N, *_ in shapes}
    assert any(M % 64 and N % 64 and K % 16 for M, N, K, _ in shapes)
    assert {0, 1} == {acc for _, _, _, _, acc, _ in GEMM_SHAPES}


def test_gemm_plan_examples():
    """A few plans worked out by hand (132 SMs)."""
    p = gemm_plan(64, 64, 1000, 0, 132)       # want 528 -> 256, then 1000 / s >= 32 -> 31, kps 48 -> 21 splits
    assert (p["capped"], p["looped"], p["kps"], p["splits"], p["memset"]) == (256, 31, 48, 21, True)
    p = gemm_plan(33, 17, 131072, 0, 132)
    assert (p["want"], p["kps"], p["splits"]) == (528, 512, 256)
    p = gemm_plan(256, 271, 9000, 1, 132)     # 20 tiles: want 27, 9000 / s >= 512 -> 17, kps 544
    assert (p["want"], p["looped"], p["kps"], p["splits"], p["memset"]) == (27, 17, 544, 17, False)
    assert gemm_plan(1100, 1100, 300, 0, 132)["splits"] == 1


def test_colsum_shapes_cover_empty_strips_and_long_columns():
    for sms in SM_COUNTS:
        empties = [colsum_strips(rows, sms)[2] for rows, _, _ in COLSUM_SHAPES]
        assert any(e > 0 for e in empties), sms
        assert max(rows for rows, _, _ in COLSUM_SHAPES) >= 7 * 4 * sms * 256
    assert colsum_strips(140000, 132) == (528, 266, 1)
    rows = [r for r, _, _ in COLSUM_SHAPES]
    assert min(rows) < 256 and any(c == 1 for _, c, _ in COLSUM_SHAPES) and any(ld > c for _, c, ld in COLSUM_SHAPES)
    assert any(s == 1 for _, s, _, _, _ in SEGSUM_SHAPES) and any(c == 1 for _, _, c, _, _ in SEGSUM_SHAPES)
    assert any(li > c and lo > c for _, _, c, li, lo in SEGSUM_SHAPES)


def test_integer_operands_are_exact_in_fp32():
    """Every partial sum of an integer GEMM (|a|, |b|, |C| <= 3), column sum (entries and preset <= 3) and segment sum
    (entries <= 3) is an integer below 2^24, so fp32 represents it exactly whatever the order of summation."""
    limit = 2 ** 24
    for M, N, K, *_ in GEMM_SHAPES:
        assert INT_RANGE + K * INT_RANGE * INT_RANGE < limit, (M, N, K)
    for rows, _, _ in COLSUM_SHAPES:
        assert INT_RANGE + rows * INT_RANGE < limit, rows
    for _, S, *_ in SEGSUM_SHAPES:
        assert S * INT_RANGE < limit


# ------------------------------------------------------------------------------------------------
# additivity on the float64 oracle
# ------------------------------------------------------------------------------------------------
def map_keys(model_order, forward_instance):
    names = ["rgb", "depth", "opacity"] + (["rgb_instance", "depth_instance", "opacity_instance"] if forward_instance else [])
    return [f"{k}_{typ}" for typ in model_order for k in names]


def map_weights(n_rays, keys, seed):
    """A fixed random weight G per map: L = sum over maps of sum(map * G) is linear in the maps."""
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn((n_rays, 3) if k.startswith("rgb") else (n_rays,), generator=g) for k in keys}


def grad_case(c):
    """GRAD_CASE (voxel) or GRAD_CASE_PLAIN with `c`'s model, sizes and branches; inputs built from their seeds."""
    base = cases.GRAD_CASE if c["use_voxel"] else grad_plain.GRAD_CASE_PLAIN
    cc = dict(base, **{k: c[k] for k in ("use_voxel", "n_rays", "n_samples", "n_importance", "forward_instance")})
    inp = cases.build_render_case(cc)
    extra = (cases.build_grad_case if c["use_voxel"] else grad_plain.build_grad_case_plain)(n_rays=cc["n_rays"])
    inp.update(instance_ids=extra["instance_ids"], code_table=extra["code_table"])
    return cc, inp


def _oracle_linear_grads(c, inp, G, sl):
    """float64 oracle on rays[sl]: gradients of sum(map * G) for every leaf (weights, code table, voxel table)."""
    leaves = {}

    def leaf(name, t):
        leaves[name] = t.double().clone().requires_grad_(True)
        return leaves[name]

    weights = {typ: {k: (leaf(f"{typ}.{helpers.REF_NAMES[k]}.weight", W), leaf(f"{typ}.{helpers.REF_NAMES[k]}.bias", b))
                     for k, (W, b) in w.items()} for typ, w in inp["weights"].items()}
    codes = leaf("codes", inp["code_table"])[inp["instance_ids"].view(-1)[sl]]
    grid = None
    if c["use_voxel"]:
        g = inp["grid"]
        grid = O.VoxelGrid(g["offset"].double(), g["voxel_size"].double(), g["shape"].tolist(), g["idx_map"],
                           leaf("voxel", g["table"]))
    out = O.render_rays(weights, grid, inp["rays"][sl].double(), codes, n_samples=c["n_samples"], perturb=c["perturb"],
                        noise_std=c["noise_std"], n_importance=c["n_importance"], white_back=c["white_back"],
                        forward_instance=c["forward_instance"], frustum_bound_th=c["frustum_bound_th"],
                        pass_through_mask=inp["pass_through_mask"][sl], is_eval=False,
                        rand={k: v[sl].double() for k, v in inp["rand"].items()})
    sum((out[k] * G[k][sl].double()).sum() for k in G).backward()
    return {k: (t.grad.clone() if t.grad is not None else torch.zeros_like(t)) for k, t in leaves.items()}


@pytest.mark.parametrize("use_voxel", [True, False])
def test_additivity_holds_on_the_float64_oracle(use_voxel):
    """12 rays, 16 + 15 samples, both branches, training noise, jitter and the occlusion mask with pass-through rays:
    the full-batch gradient of sum(map * G) equals the sum over the partition [0, 5), [5, 6), [6, 12) to 1e-12
    relative, for every parameter tensor."""
    c, inp = grad_case(dict(use_voxel=use_voxel, n_rays=12, n_samples=16, n_importance=15, forward_instance=True))
    assert c["perturb"] > 0 and c["noise_std"] > 0 and c["frustum_bound_th"] > 0 and inp["pass_through_mask"].any()
    G = map_weights(12, map_keys(["coarse", "fine"], True), seed=21)
    full = _oracle_linear_grads(c, inp, G, slice(0, 12))
    parts = [_oracle_linear_grads(c, inp, G, slice(a, b)) for a, b in ((0, 5), (5, 6), (6, 12))]
    assert len(full) == 80 + 1 + int(use_voxel)
    for name, g in full.items():
        s = sum(p[name] for p in parts)
        assert g.norm() > 0, name
        rel = ((g - s).norm() / g.norm()).item()
        assert rel <= 1e-12, (name, rel)
