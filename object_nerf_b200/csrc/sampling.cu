// Depth sampling kernels: stratified coarse depths and inverse-CDF importance sampling fused with
// the sorted merge.  HBM-bound, one pass over the data; see DESIGN.md §kernels.
//
// Reference behaviour: models/rendering.py:259-277 (stratified), :11-61 (sample_pdf), :301-313 (merge).
#include "common.cuh"
#include "train_ws.h"

namespace {

// torch.linspace(0, 1, S)[i] in fp32: symmetric two-sided formula (ATen RangeFactories), every
// operation individually rounded (no FMA contraction) so the CPU oracle and the GPU agree.
__device__ __forceinline__ float linspace01(int i, int n) {
  if (n <= 1) return 0.0f;
  const float step = __fdiv_rn(1.0f, (float)(n - 1));
  return (i < n / 2) ? __fmul_rn(step, (float)i) : __fsub_rn(1.0f, __fmul_rn(step, (float)(n - 1 - i)));
}

__device__ __forceinline__ float coarse_depth(float near, float far, int i, int n, bool use_disp) {
  const float t = linspace01(i, n);
  const float omt = __fsub_rn(1.0f, t);
  if (!use_disp) return __fadd_rn(__fmul_rn(near, omt), __fmul_rn(far, t));
  const float a = __fmul_rn(__fdiv_rn(1.0f, near), omt);
  const float b = __fmul_rn(__fdiv_rn(1.0f, far), t);
  return __fdiv_rn(1.0f, __fadd_rn(a, b));
}

// seed_dev != null: the draws use seed + *seed_dev (the caller passes only the offset in `seed`); see onerf_ext.h
__global__ void __launch_bounds__(256)
sample_coarse_kernel(const float* __restrict__ rays, int n_rays, int S, int use_disp, float perturb,
                     const float* __restrict__ jitter, uint64_t seed, const uint64_t* seed_dev, float* __restrict__ z_out) {
  if (seed_dev && perturb > 0.0f && !jitter) seed += *seed_dev;
  const int64_t total = (int64_t)n_rays * S;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / S), i = (int)(e - (int64_t)r * S);
    const float near = __ldg(rays + (int64_t)r * 8 + 6), far = __ldg(rays + (int64_t)r * 8 + 7);
    float z = coarse_depth(near, far, i, S, use_disp);
    if (perturb > 0.0f) {
      const float zl = (i > 0) ? coarse_depth(near, far, i - 1, S, use_disp) : z;
      const float zu = (i < S - 1) ? coarse_depth(near, far, i + 1, S, use_disp) : z;
      const float lower = (i > 0) ? __fmul_rn(0.5f, __fadd_rn(zl, z)) : z;
      const float upper = (i < S - 1) ? __fmul_rn(0.5f, __fadd_rn(z, zu)) : z;
      const float u = jitter ? __ldg(jitter + e) : philox_uniform(seed, 0u, (uint64_t)e);
      z = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), __fmul_rn(perturb, u)));
    }
    z_out[e] = z;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// inclusive additive warp scan in double: torch's CPU cumsum accumulates fp32 rows in double and rounds
// each prefix to fp32 (ATen cumsum_cpu_kernel, acc_type<float> = double); doing the same keeps cdf[M]
// on the same side of 1.0 as the reference, which decides where the u = 1 sample lands when the tail
// bins are empty (denominator guard, models/rendering.py:54-56).
__device__ __forceinline__ double warp_scan_add(double v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    double t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// One warp per ray.  Shared memory per warp: bins[S-1] | cdf[S-1] | merged[P], P = pow2 >= S+K.
__global__ void __launch_bounds__(256)
sample_pdf_merge_kernel(const float* __restrict__ z_coarse, const float* __restrict__ weights, int n_rays,
                        int S, int K, int P, int det, const float* __restrict__ u_in, uint64_t seed,
                        const uint64_t* seed_dev, float* __restrict__ z_out, const float* __restrict__ bins_in) {
  // bins_in != null: stand-alone sample_pdf on explicit bins (N, S-1) and weights (N, S-2): no merge,
  // z_out (N, K) in draw order.  Otherwise the fused form on coarse depths / full coarse weights.
  // seed_dev != null: as in sample_coarse_kernel.
  extern __shared__ float smem[];
  if (seed_dev && !det && !u_in) seed += *seed_dev;
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per_warp = 2 * S + P;
  float* bins = smem + (size_t)warp * per_warp;   // S-1 used
  float* cdf = bins + S;                          // S-1 used: cdf[0..M], M = S-2
  float* merged = cdf + S;                        // P
  const float eps = 1e-5f;
  const int M = S - 2;

  for (int r = blockIdx.x * warps_per_block + warp; r < n_rays; r += gridDim.x * warps_per_block) {
    // w points one before the first pdf weight (the fused form skips weights[:, 0])
    const float* w = bins_in ? weights + (int64_t)r * M - 1 : weights + (int64_t)r * S;
    if (bins_in) {
      for (int i = lane; i < S - 1; i += 32) bins[i] = __ldg(bins_in + (int64_t)r * (S - 1) + i);
    } else {
      // coarse depths into the merge buffer; mid-point bins
      const float* zc = z_coarse + (int64_t)r * S;
      for (int i = lane; i < S; i += 32) merged[i] = __ldg(zc + i);
      __syncwarp();
      for (int i = lane; i < S - 1; i += 32) bins[i] = __fmul_rn(0.5f, __fadd_rn(merged[i], merged[i + 1]));
    }
    // pdf normaliser over weights[1:-1] + eps
    float part = 0.0f;
    for (int i = lane; i < M; i += 32) part += __fadd_rn(__ldg(w + 1 + i), eps);
    const float total = warp_sum(part);
    // cdf[0] = 0, cdf[j+1] = cdf[j] + pdf_j
    double carry = 0.0;
    if (lane == 0) cdf[0] = 0.0f;
    for (int base = 0; base < M; base += 32) {
      const int i = base + lane;
      const float p = (i < M) ? __fdiv_rn(__fadd_rn(__ldg(w + 1 + i), eps), total) : 0.0f;
      const double s = warp_scan_add((double)p, lane) + carry;
      if (i < M) cdf[i + 1] = (float)s;
      carry = __shfl_sync(0xffffffffu, s, 31);
    }
    __syncwarp();
    // inverse CDF
    for (int k = lane; k < K; k += 32) {
      float u;
      if (det) u = linspace01(k, K);
      else if (u_in) u = __ldg(u_in + (int64_t)r * K + k);
      else u = philox_uniform(seed, 1u, (uint64_t)r * K + k);
      // searchsorted(cdf[0..M], u, right=True): first index with cdf > u, in [0, M+1]
      int lo = 0, hi = M + 1;
      while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (cdf[mid] > u) hi = mid; else lo = mid + 1;
      }
      const int below = max(lo - 1, 0), above = min(lo, M);
      const float cb = cdf[below], ca = cdf[above];
      const float bb = bins[below], ba = bins[above];
      float denom = __fsub_rn(ca, cb);
      if (denom < eps) denom = 1.0f;
      merged[S + k] = __fadd_rn(bb, __fmul_rn(__fdiv_rn(__fsub_rn(u, cb), denom), __fsub_rn(ba, bb)));
    }
    __syncwarp();
    if (bins_in) {
      for (int k = lane; k < K; k += 32) z_out[(int64_t)r * K + k] = merged[S + k];
      __syncwarp();
      continue;
    }
    for (int i = S + K + lane; i < P; i += 32) merged[i] = __int_as_float(0x7f800000);
    __syncwarp();
    // bitonic sort (ascending) of P values by one warp
    for (int k2 = 2; k2 <= P; k2 <<= 1) {
      for (int j = k2 >> 1; j > 0; j >>= 1) {
        for (int t = lane; t < (P >> 1); t += 32) {
          const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // index with bit j cleared
          const int l = i | j;
          const bool up = ((i & k2) == 0);
          const float a = merged[i], b = merged[l];
          if ((a > b) == up) { merged[i] = b; merged[l] = a; }
        }
        __syncwarp();
      }
    }
    float* out = z_out + (int64_t)r * (S + K);
    for (int i = lane; i < S + K; i += 32) out[i] = merged[i];
    __syncwarp();
  }
}

}  // namespace

int onerf_launch_sample_coarse(onerf_ctx* ctx, const float* rays, int n_rays, int n_samples, int use_disp, float perturb,
                               const float* jitter, uint64_t seed, const uint64_t* seed_dev, float* z_out, void* stream) {
  ONERF_CHECK_ARG(ctx && rays && z_out, "null argument");
  ONERF_CHECK_ARG(n_rays >= 0 && n_samples >= 1, "bad shape");
  if (n_rays == 0) return ONERF_OK;
  const int64_t total = (int64_t)n_rays * n_samples;
  int blocks = (int)((total + 255) / 256);
  const int cap = ctx->num_sms * 16;
  if (blocks > cap) blocks = cap;
  sample_coarse_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(rays, n_rays, n_samples, use_disp, perturb,
                                                                 jitter, seed, seed_dev, z_out);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_sample_coarse(onerf_ctx* ctx, const float* rays, int n_rays, int n_samples,
                                   int use_disp, float perturb, const float* jitter, uint64_t seed,
                                   float* z_out, void* stream) {
  return onerf_launch_sample_coarse(ctx, rays, n_rays, n_samples, use_disp, perturb, jitter, seed, nullptr, z_out, stream);
}

extern "C" int onerf_sample_pdf_merge(onerf_ctx* ctx, const float* z_coarse, const float* weights,
                                      int n_rays, int n_samples, int n_importance, int det, const float* u,
                                      uint64_t seed, float* z_out, void* stream) {
  return onerf_launch_sample_pdf_merge(ctx, z_coarse, weights, n_rays, n_samples, n_importance, det, u, seed, nullptr, z_out,
                                       stream);
}

int onerf_launch_sample_pdf_merge(onerf_ctx* ctx, const float* z_coarse, const float* weights, int n_rays, int n_samples,
                                  int n_importance, int det, const float* u, uint64_t seed, const uint64_t* seed_dev,
                                  float* z_out, void* stream) {
  ONERF_CHECK_ARG(ctx && z_coarse && weights && z_out, "null argument");
  ONERF_CHECK_ARG(n_rays >= 0 && n_samples >= 3 && n_importance >= 1, "bad shape (need S >= 3, K >= 1)");
  ONERF_UNSUPPORTED(n_samples + n_importance > 2048, "S + K > 2048");
  if (n_rays == 0) return ONERF_OK;
  int P = 1;
  while (P < n_samples + n_importance) P <<= 1;
  const int warps = 8;
  const size_t smem = (size_t)warps * (2 * n_samples + P) * sizeof(float);
  ONERF_CUDA(cudaFuncSetAttribute(sample_pdf_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int blocks = (n_rays + warps - 1) / warps;
  const int cap = ctx->num_sms * 8;
  if (blocks > cap) blocks = cap;
  sample_pdf_merge_kernel<<<blocks, warps * 32, smem, (cudaStream_t)stream>>>(
      z_coarse, weights, n_rays, n_samples, n_importance, P, det, u, seed, seed_dev, z_out, nullptr);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_sample_pdf(onerf_ctx* ctx, const float* bins, const float* weights, int n_rays, int n_bins,
                                int n_importance, int det, const float* u, uint64_t seed, float* out,
                                void* stream) {
  ONERF_CHECK_ARG(ctx && bins && weights && out, "null argument");
  ONERF_CHECK_ARG(n_rays >= 0 && n_bins >= 2 && n_importance >= 1, "bad shape (need >= 2 bins, K >= 1)");
  ONERF_UNSUPPORTED(n_bins + 1 + n_importance > 2048, "bins + K > 2047");
  if (n_rays == 0) return ONERF_OK;
  const int S = n_bins + 1;  // the kernel's "S": S-1 bins, S-2 weights
  int P = 1;
  while (P < S + n_importance) P <<= 1;
  const int warps = 8;
  const size_t smem = (size_t)warps * (2 * S + P) * sizeof(float);
  ONERF_CUDA(cudaFuncSetAttribute(sample_pdf_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int blocks = (n_rays + warps - 1) / warps;
  const int cap = ctx->num_sms * 8;
  if (blocks > cap) blocks = cap;
  sample_pdf_merge_kernel<<<blocks, warps * 32, smem, (cudaStream_t)stream>>>(
      nullptr, weights, n_rays, S, n_importance, P, det, u, seed, nullptr, out, bins);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
