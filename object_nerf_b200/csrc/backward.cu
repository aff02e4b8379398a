// Backward building blocks of the render path (SURVEY.md §8 row a14: the autograd the reference gets for free
// from PyTorch, models/rendering.py + models/nerf_model.py + models/embedding_helper.py under loss.backward()).
//
// fp32 throughout (the reference trains in fp32).  The field backward is organised as matrices over a chunk of
// samples: the FFMA field kernel re-runs the forward and dumps every layer's activations ([B x width] row-major,
// field_fp32.cu), then per layer  dZ = dH * act'(H),  dW += dZ^T In (split over samples, atomics),  db += colsum(dZ),
// dIn = dZ W  with the generic GEMM below; concatenations are handled with leading dimensions / column offsets.
// Orchestration: bwd_api.cu (onerf_render_rays_bwd with ONERF_PREC_FP32).
#include "composite_core.cuh"
#include "encode.cuh"
#include "field_common.cuh"
#include "../../include/onerf_ext.h"

namespace {

// ------------------------------------------------------------------------------------------------
// compositing backward: one warp per ray
// ------------------------------------------------------------------------------------------------
struct BranchGrad {
  const float* g_rgb;      // (N,3) or null
  const float* g_depth;    // (N,) or null
  const float* g_opacity;  // (N,) or null
};

struct CompositeBwdArgs {
  onerf_composite_args fwd;   // same inputs as the forward (outputs unused)
  const float* depth_scene;   // (N,) forward scene depth (for the occlusion mask)
  BranchGrad gs, go;
  float* dscene;              // (N,S,4)
  float* dobj;                // (N,S,4) or null
};

// Per branch: composite_branch recomputes the forward's alpha / transmittance / noised sigma (the caller's noise buffer
// or the same Philox draw) into the warp's shared memory, then composite_branch_grad back-propagates, the sequence
// composite_kernel<true> (composite.cu) runs.  smem (per warp): alpha[S], trans[S], sig[S], gw[S]
__global__ void __launch_bounds__(128) composite_bwd_kernel(CompositeBwdArgs a) {
  extern __shared__ float smem_c[];
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = a.fwd.n_samples;
  float* s_alpha = smem_c + (size_t)warp * 4 * S;
  float* s_trans = s_alpha + S;
  float* s_sig = s_trans + S;
  float* s_gw = s_sig + S;
  for (int r = blockIdx.x * warps_per_block + warp; r < a.fwd.n_rays; r += gridDim.x * warps_per_block) {
    const float* z = a.fwd.z + (int64_t)r * S;
    auto g3 = [&](const float* p, int c) { return p ? __ldg(p + (int64_t)r * 3 + c) : 0.0f; };
    auto g1 = [&](const float* p) { return p ? __ldg(p + r) : 0.0f; };
    const float4* scene = reinterpret_cast<const float4*>(a.fwd.scene) + (int64_t)r * S;
    const float scene_last_delta = a.fwd.zero_last_delta ? 0.0f : 1e10f;
    composite_branch(z, scene, S, scene_last_delta, a.fwd.noise_std,
                     a.fwd.noise_scene ? a.fwd.noise_scene + (int64_t)r * S : nullptr, a.fwd.seed, 2u, r, false, 0.0f,
                     nullptr, lane, s_alpha, s_trans, s_sig);
    __syncwarp();
    composite_branch_grad(z, scene, S, scene_last_delta, false, 0.0f, a.fwd.white_back != 0, g3(a.gs.g_rgb, 0),
                          g3(a.gs.g_rgb, 1), g3(a.gs.g_rgb, 2), g1(a.gs.g_depth), g1(a.gs.g_opacity),
                          reinterpret_cast<float4*>(a.dscene) + (int64_t)r * S, s_alpha, s_trans, s_sig, s_gw, lane);
    __syncwarp();
    if (a.fwd.obj != nullptr) {
      bool use_mask = (!a.fwd.is_eval) && (a.fwd.frustum_bound_th > 0.0f);
      if (use_mask && a.fwd.pass_through_mask && a.fwd.pass_through_mask[r]) use_mask = false;
      const float z_limit = __fadd_rn(__ldg(a.depth_scene + r), a.fwd.frustum_bound_th);
      const float4* obj = reinterpret_cast<const float4*>(a.fwd.obj) + (int64_t)r * S;
      composite_branch(z, obj, S, 0.0f, a.fwd.noise_std, a.fwd.noise_obj ? a.fwd.noise_obj + (int64_t)r * S : nullptr,
                       a.fwd.seed, 3u, r, use_mask, z_limit, nullptr, lane, s_alpha, s_trans, s_sig);
      __syncwarp();
      composite_branch_grad(z, obj, S, 0.0f, use_mask, z_limit, true, g3(a.go.g_rgb, 0), g3(a.go.g_rgb, 1),
                            g3(a.go.g_rgb, 2), g1(a.go.g_depth), g1(a.go.g_opacity),
                            reinterpret_cast<float4*>(a.dobj) + (int64_t)r * S, s_alpha, s_trans, s_sig, s_gw, lane);
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// generic fp32 GEMM:  C[M x N] (+)= op(A) . B,  B [K x N] row-major (ldb), C row-major (ldc)
//   trans_a = 0: A [M x K] row-major (lda);  trans_a = 1: A [K x M] row-major (lda)  (reduction over rows of A)
//   grid.z splits K; with more than one split (or accumulate) results are added atomically.
// 64 x 64 x 16 tiles, 256 threads, 4 x 4 outputs per thread, fully bounds-checked.
// ------------------------------------------------------------------------------------------------
constexpr int GB = 64, GK = 16;

__global__ void __launch_bounds__(256)
gemm_kernel(const float* __restrict__ A, int lda, int trans_a, const float* __restrict__ B, int ldb, float* __restrict__ C,
            int ldc, int M, int N, int K, int k_per_split, int atomic) {
  __shared__ float As[GK][GB + 4];
  __shared__ float Bs[GK][GB + 4];
  const int m0 = blockIdx.y * GB, n0 = blockIdx.x * GB;
  const int kbeg = blockIdx.z * k_per_split, kend = min(K, kbeg + k_per_split);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;   // 16 x 16 threads, each 4 x 4
  float acc[4][4] = {};
  for (int k0 = kbeg; k0 < kend; k0 += GK) {
    // A tile -> As[k][m]
    for (int e = threadIdx.x; e < GB * GK; e += 256) {
      int m, k;
      if (trans_a) { m = e % GB; k = e / GB; }    // A[k][m]: consecutive threads walk m (contiguous)
      else { k = e % GK; m = e / GK; }            // A[m][k]: consecutive threads walk k (contiguous)
      const int gm = m0 + m, gk = k0 + k;
      float v = 0.0f;
      if (gm < M && gk < kend) v = trans_a ? __ldg(A + (int64_t)gk * lda + gm) : __ldg(A + (int64_t)gm * lda + gk);
      As[k][m] = v;
    }
    for (int e = threadIdx.x; e < GB * GK; e += 256) {
      const int n = e % GB, k = e / GB;
      const int gn = n0 + n, gk = k0 + k;
      Bs[k][n] = (gn < N && gk < kend) ? __ldg(B + (int64_t)gk * ldb + gn) : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float* c = C + (int64_t)gm * ldc + gn;
      if (atomic) atomicAdd(c, acc[i][j]);
      else *c = acc[i][j];
    }
  }
}

// dH <- dH * (H > 0 ? 1 : 0.01) on a [rows x cols] block (row strides ld_d, ld_h)
__global__ void leaky_bwd_kernel(float* __restrict__ d, int ld_d, const float* __restrict__ h, int ld_h, int64_t rows, int cols) {
  const int64_t total = rows * cols;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / cols;
    const int c = (int)(e - r * cols);
    const float hv = __ldg(h + r * ld_h + c);
    float* p = d + r * ld_d + c;
    *p = *p * (hv > 0.0f ? 1.0f : 0.01f);
  }
}

// head gradients of one branch: dA[b] = (d_rgb * rgb (1 - rgb), d_sigma)  from dfield and the forward field output
__global__ void head_bwd_kernel(const float4* __restrict__ dfield, const float4* __restrict__ field, float4* __restrict__ dA,
                                int64_t n) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const float4 g = __ldg(dfield + e), f = __ldg(field + e);
    // a muted sample (sigma forced to -1e5) passes no gradient to sigma; its composited weight is 0 anyway
    dA[e] = make_float4(g.x * f.x * (1.0f - f.x), g.y * f.y * (1.0f - f.y), g.z * f.z * (1.0f - f.z), g.w);
  }
}

// out[r][c] (+)= sum over the S consecutive rows of ray r of in[(r S + s)][c]
__global__ void segment_sum_kernel(const float* __restrict__ in, int ld_in, float* __restrict__ out, int ld_out, int n_rays,
                                   int S, int cols) {
  const int64_t total = (int64_t)n_rays * cols;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / cols), c = (int)(e - (int64_t)r * cols);
    float acc = 0.0f;
    for (int s = 0; s < S; ++s) acc += __ldg(in + ((int64_t)r * S + s) * ld_in + c);
    out[(int64_t)r * ld_out + c] = acc;
  }
}

// out[c] += sum over rows of in[r][c]   (one CTA handles a strip of rows; atomics per column)
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ in, int ld, int64_t rows, int cols,
                                                     float* __restrict__ out) {
  const int64_t rows_per_block = (rows + gridDim.x - 1) / gridDim.x;
  const int64_t r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    float acc = 0.0f;
    for (int64_t r = r0; r < r1; ++r) acc += __ldg(in + r * ld + c);
    atomicAdd(out + c, acc);
  }
}

// PE4 of the ray directions: (N,8) rays -> (N,27)
__global__ void dir_encode_kernel(const float* __restrict__ rays, int n, float* __restrict__ out) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n * 3; e += gridDim.x * blockDim.x) {
    const int r = e / 3, c = e % 3;
    const float d = __ldg(rays + (int64_t)r * 8 + 3 + c);
    float* o = out + (int64_t)r * 27;
    o[c] = d;
    for (int k = 0; k < 4; ++k) {
      const float a = d * (float)(1 << k);
      o[3 * (1 + 2 * k) + c] = sinf(a);
      o[3 * (2 + 2 * k) + c] = cosf(a);
    }
  }
}

// Encoding backward: dX (B x ldx; X layout of layout.h) -> scatter-add into the voxel table gradient.
//   d f_c = dX[f_c] + sum_k 2^k ( cos(2^k f_c) dX[sin_k c] - sin(2^k f_c) dX[cos_k c] ),  sin / cos taken from X itself;
//   table_grad[row_corner][c] += trilinear weight * d f_c   (reference: embedding_helper.py:354-409 under autograd)
// One thread per (sample, group of 8 channels): groups 0,1 = scene channels 0-7, 8-15; group 2 = object channels.
// The sample's position is o + d z of its ray, or with XYZ row `gs` of p.xyz.
template <bool XYZ>
__global__ void __launch_bounds__(256)
encode_bwd_kernel(FieldParams p, const float* __restrict__ X, const float* __restrict__ dX, int ldx, int64_t sample0,
                  int64_t n_samples, float* __restrict__ table_grad) {
  const GridView g = load_grid_view(p.grid);
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_samples * 3; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t sl = e / 3;              // sample index inside the chunk
    const int grp = (int)(e - sl * 3);
    const int64_t gs = sample0 + sl;       // global sample index
    float x, y, z;
    if (XYZ) {
      const float* q = p.xyz + gs * 3;
      x = __ldg(q); y = __ldg(q + 1); z = __ldg(q + 2);
    } else {
      const int ray = (int)(gs / p.S), si = (int)(gs - (int64_t)ray * p.S);
      const float* rr = p.rays + (int64_t)ray * 8;
      const float zz = __ldg(p.z + (int64_t)ray * p.z_stride + si);
      x = __fadd_rn(__ldg(rr + 0), __fmul_rn(__ldg(rr + 3), zz));
      y = __fadd_rn(__ldg(rr + 1), __fmul_rn(__ldg(rr + 4), zz));
      z = __fadd_rn(__ldg(rr + 2), __fmul_rn(__ldg(rr + 5), zz));
    }
    const int base = (grp < 2) ? 0 : 272, width = (grp < 2) ? 16 : 8, ch0 = (grp == 1) ? 8 : 0;
    const float* xr = X + sl * ldx + base;
    const float* dr = dX + sl * ldx + base;
    float df[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float acc = __ldg(dr + ch0 + c);
      for (int k = 0; k < 6; ++k) {
        const float sn = __ldg(xr + width * (1 + 2 * k) + ch0 + c), cs = __ldg(xr + width * (2 + 2 * k) + ch0 + c);
        const float scale = (float)(1 << k);
        acc += scale * (cs * __ldg(dr + width * (1 + 2 * k) + ch0 + c) - sn * __ldg(dr + width * (2 + 2 * k) + ch0 + c));
      }
      df[c] = acc;
    }
    // corners and weights as in the forward
    const float px = __fdiv_rn(__fadd_rn(x, g.off[0]), g.vsize), py = __fdiv_rn(__fadd_rn(y, g.off[1]), g.vsize),
                pz = __fdiv_rn(__fadd_rn(z, g.off[2]), g.vsize);
    const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
    const float u = px - fx, v = py - fy, w = pz - fz;
    const bool any = (fx >= -1.0f) && (fy >= -1.0f) && (fz >= -1.0f) && (fx < (float)g.sx) && (fy < (float)g.sy) && (fz < (float)g.sz);
    if (!any) continue;
    const int qx = (int)fx, qy = (int)fy, qz = (int)fz;
    const int tch = (grp < 2) ? ch0 : 16;   // first table channel of this group
    for (int corner = 0; corner < 8; ++corner) {
      const int cx = (corner >> 2) & 1, cy = (corner >> 1) & 1, cz = corner & 1;
      const int ix = qx + cx, iy = qy + cy, iz = qz + cz;
      if (ix < 0 || iy < 0 || iz < 0 || ix >= g.sx || iy >= g.sy || iz >= g.sz) continue;
      const long long row = __ldg(g.idx_map + ((int64_t)ix * g.sy + iy) * g.sz + iz);
      if (row < 0) continue;
      const float wt = (cx ? u : 1.0f - u) * (cy ? v : 1.0f - v) * (cz ? w : 1.0f - w);
      float* dst = table_grad + row * 24 + tch;
#pragma unroll
      for (int c = 0; c < 8; ++c) atomicAdd(dst + c, wt * df[c]);
    }
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------
extern "C" int onerf_composite_bwd(onerf_ctx* ctx, const onerf_composite_args* fwd, const float* depth_scene,
                                   const float* g_rgb, const float* g_depth, const float* g_opacity,
                                   const float* g_rgb_inst, const float* g_depth_inst, const float* g_opacity_inst,
                                   float* dscene, float* dobj, void* stream) {
  ONERF_CHECK_ARG(ctx && fwd && fwd->z && fwd->scene && dscene, "null argument");
  ONERF_CHECK_ARG(!fwd->obj || (dobj && depth_scene), "object branch needs dobj and depth_scene");
  ONERF_UNSUPPORTED(fwd->n_samples > 2048, "S > 2048");
  if (fwd->n_rays == 0) return ONERF_OK;
  CompositeBwdArgs a;
  a.fwd = *fwd;
  a.depth_scene = depth_scene;
  a.gs = BranchGrad{g_rgb, g_depth, g_opacity};
  a.go = BranchGrad{g_rgb_inst, g_depth_inst, g_opacity_inst};
  a.dscene = dscene;
  a.dobj = dobj;
  const int warps = 4;
  const size_t smem = (size_t)warps * 4 * fwd->n_samples * sizeof(float);
  ONERF_CUDA(cudaFuncSetAttribute(composite_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  composite_bwd_kernel<<<composite_blocks(ctx, fwd->n_rays, warps), warps * 32, smem, (cudaStream_t)stream>>>(a);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_gemm(onerf_ctx* ctx, const float* A, int lda, int trans_a, const float* B, int ldb, float* C, int ldc,
                          int M, int N, int K, int accumulate, void* stream) {
  ONERF_CHECK_ARG(ctx && A && B && C, "null argument");
  ONERF_CHECK_ARG(M >= 0 && N >= 0 && K >= 0, "bad shape");
  if (M == 0 || N == 0 || K == 0) return ONERF_OK;
  const int gx = (N + GB - 1) / GB, gy = (M + GB - 1) / GB;
  // split the reduction when the output grid alone cannot fill the machine (weight gradients: K = samples)
  int splits = 1;
  if (K >= 256 && gx * gy < 2 * ctx->num_sms) {
    const int want = (4 * ctx->num_sms + gx * gy - 1) / (gx * gy);
    splits = want < 1 ? 1 : (want > 256 ? 256 : want);
    // long reductions (weight gradients over samples) keep >= 512 rows per CTA; short ones (per-ray sums, K = rays of
    // one batch) would otherwise run on one or two CTAs: let them go down to 32 rows
    const int min_k = K >= 4096 ? 512 : 32;
    while (splits > 1 && K / splits < min_k) --splits;
  }
  int kps = ((K + splits - 1) / splits + GK - 1) / GK * GK;
  splits = (K + kps - 1) / kps;
  ONERF_CHECK_ARG(gy <= 65535 && splits <= 65535, "grid too large");
  const int atomic = (accumulate || splits > 1) ? 1 : 0;
  if (splits > 1 && !accumulate) {
    // overwrite semantics with a split reduction: clear C first
    ONERF_CUDA(cudaMemset2DAsync(C, (size_t)ldc * sizeof(float), 0, (size_t)N * sizeof(float), (size_t)M, (cudaStream_t)stream));
  }
  gemm_kernel<<<dim3(gx, gy, splits), 256, 0, (cudaStream_t)stream>>>(A, lda, trans_a, B, ldb, C, ldc, M, N, K, kps, atomic);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_leaky_bwd(onerf_ctx* ctx, float* d, int ld_d, const float* h, int ld_h, int64_t rows, int cols, void* stream) {
  ONERF_CHECK_ARG(ctx && d && h, "null argument");
  if (rows == 0 || cols == 0) return ONERF_OK;
  int blocks = (int)((rows * cols + 255) / 256 < (int64_t)ctx->num_sms * 16 ? (rows * cols + 255) / 256 : (int64_t)ctx->num_sms * 16);
  leaky_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(d, ld_d, h, ld_h, rows, cols);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_head_bwd(onerf_ctx* ctx, const float* dfield, const float* field, float* dA, int64_t n, void* stream) {
  ONERF_CHECK_ARG(ctx && dfield && field && dA, "null argument");
  if (n == 0) return ONERF_OK;
  int blocks = (int)((n + 255) / 256 < (int64_t)ctx->num_sms * 16 ? (n + 255) / 256 : (int64_t)ctx->num_sms * 16);
  head_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(dfield),
                                                            reinterpret_cast<const float4*>(field),
                                                            reinterpret_cast<float4*>(dA), n);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_segment_sum(onerf_ctx* ctx, const float* in, int ld_in, float* out, int ld_out, int n_rays, int n_samples,
                                 int cols, void* stream) {
  ONERF_CHECK_ARG(ctx && in && out, "null argument");
  if (n_rays == 0 || cols == 0) return ONERF_OK;
  const int64_t total = (int64_t)n_rays * cols;
  int blocks = (int)((total + 255) / 256 < (int64_t)ctx->num_sms * 16 ? (total + 255) / 256 : (int64_t)ctx->num_sms * 16);
  segment_sum_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(in, ld_in, out, ld_out, n_rays, n_samples, cols);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_colsum(onerf_ctx* ctx, const float* in, int ld, int64_t rows, int cols, float* out, void* stream) {
  ONERF_CHECK_ARG(ctx && in && out, "null argument");
  if (rows == 0 || cols == 0) return ONERF_OK;
  int blocks = (int)(rows / 256 + 1 < (int64_t)ctx->num_sms * 4 ? rows / 256 + 1 : (int64_t)ctx->num_sms * 4);
  colsum_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(in, ld, rows, cols, out);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_dir_encode(onerf_ctx* ctx, const float* rays, int n_rays, float* out, void* stream) {
  ONERF_CHECK_ARG(ctx && rays && out, "null argument");
  if (n_rays == 0) return ONERF_OK;
  dir_encode_kernel<<<(n_rays * 3 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(rays, n_rays, out);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_encode_bwd(onerf_ctx* ctx, const onerf_grid* grid, const float* rays, const float* z, int n_rays,
                                int n_samples, const float* X, const float* dX, int ldx, int64_t sample0, int64_t n_chunk,
                                float* table_grad, void* stream) {
  ONERF_CHECK_ARG(ctx && grid && rays && z && X && dX && table_grad, "null argument");
  if (n_chunk == 0) return ONERF_OK;
  FieldParams p;
  memset(&p, 0, sizeof(p));
  p.rays = rays; p.z = z; p.z_stride = n_samples; p.n_rays = n_rays; p.S = n_samples; p.grid = *grid;
  int blocks = (int)((n_chunk * 3 + 255) / 256 < (int64_t)ctx->num_sms * 16 ? (n_chunk * 3 + 255) / 256 : (int64_t)ctx->num_sms * 16);
  encode_bwd_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(p, X, dX, ldx, sample0, n_chunk, table_grad);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_encode_bwd_xyz(onerf_ctx* ctx, const onerf_grid* grid, const float* xyz, const float* X, const float* dX,
                                    int ldx, int64_t sample0, int64_t n_chunk, float* table_grad, void* stream) {
  ONERF_CHECK_ARG(ctx && grid && xyz && X && dX && table_grad, "null argument");
  if (n_chunk == 0) return ONERF_OK;
  FieldParams p;
  memset(&p, 0, sizeof(p));
  p.xyz = xyz; p.grid = *grid;
  int blocks = (int)((n_chunk * 3 + 255) / 256 < (int64_t)ctx->num_sms * 16 ? (n_chunk * 3 + 255) / 256 : (int64_t)ctx->num_sms * 16);
  encode_bwd_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(p, X, dX, ldx, sample0, n_chunk, table_grad);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
