// TotalLoss of the training step and its gradient w.r.t. the rendered maps in two small kernels (SURVEY.md section 8f
// row 3).  Reference: models/losses.py:5-135 - five masked-MSE terms (color, depth, opacity, instance color, instance
// depth), each over the coarse and the fine maps; under autograd the reference runs ~120 elementwise / index / reduce
// kernels and several host syncs (`mask.sum() == 0`) for 2 048 rays.  Here: one reduction pass (counts and weighted
// squared-error sums, fp64 accumulators) and one pass that writes d(loss_sum)/d(map) for all ten maps and the loss values.
#include <string.h>

#include "loss_terms.cuh"
#include "train_ws.h"

namespace {

using namespace loss_terms;

struct LossParams {
  onerf_loss_args a;
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// Sums acc[0, n) over the block (256 threads) and adds the non-zero totals to ws[0, n).
template <int n>
__device__ __forceinline__ void block_accumulate(const double* acc, double* __restrict__ ws) {
  __shared__ double sh[8][n];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < n; ++i) {
    const double v = warp_sum(acc[i]);
    if (lane == 0) sh[warp][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < n) {
    double v = 0.0;
    for (int w8 = 0; w8 < 8; ++w8) v += sh[w8][threadIdx.x];
    if (v != 0.0) atomicAdd(ws + threadIdx.x, v);
  }
}

__global__ void __launch_bounds__(256) loss_reduce_kernel(LossParams P, double* __restrict__ ws) {
  const onerf_loss_args& a = P.a;
  double acc[WS_DOUBLES];
#pragma unroll
  for (int i = 0; i < WS_DOUBLES; ++i) acc[i] = 0.0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < a.n_rays; r += (int64_t)gridDim.x * blockDim.x) {
    const Target g = load_target(a, r);
    add_counts(g, acc);
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      const onerf_loss_maps& m = f ? a.fine : a.coarse;
      if (f && !a.has_fine) break;
      add_scene_sq(g, m.rgb + 3 * r, m.depth[r], acc + WS_SUM + f, 2);
      add_object_sq(g, m.opacity_instance[r], m.rgb_instance + 3 * r, m.depth_instance[r], acc + WS_SUM + f, 2);
    }
  }
  block_accumulate<WS_DOUBLES>(acc, ws);
}

// The counts half of loss_reduce_kernel: everything TotalLoss normalises by and skips on, from the batch alone.
__global__ void __launch_bounds__(256) batch_stats_kernel(LossParams P, double* __restrict__ ws) {
  const onerf_loss_args& a = P.a;
  double acc[WS_SUM];
#pragma unroll
  for (int i = 0; i < WS_SUM; ++i) acc[i] = 0.0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < a.n_rays; r += (int64_t)gridDim.x * blockDim.x)
    add_counts(load_target(a, r), acc);
  block_accumulate<WS_SUM>(acc, ws);
}

__global__ void __launch_bounds__(256) loss_grad_kernel(LossParams P, const double* __restrict__ ws) {
  const onerf_loss_args& a = P.a;
  float scale[N_TERMS];
  grad_scales(a, ws, scale);
  if (blockIdx.x == 0 && threadIdx.x == 0) write_outputs(a, ws);
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < a.n_rays; r += (int64_t)gridDim.x * blockDim.x) {
    const Target g = load_target(a, r);
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      if (f && !a.has_fine) break;
      const onerf_loss_maps& m = f ? a.fine : a.coarse;
      const onerf_loss_maps& gm = f ? a.grad_fine : a.grad_coarse;
      float gc[3], gi[3], gd, go, gid;
      scene_grads(g, m.rgb + 3 * r, m.depth[r], scale, gc, gd);
      object_grads(g, m.opacity_instance[r], m.rgb_instance + 3 * r, m.depth_instance[r], scale, go, gi, gid);
      float* grgb = const_cast<float*>(gm.rgb);
      float* girgb = const_cast<float*>(gm.rgb_instance);
      grgb[3 * r] = gc[0]; grgb[3 * r + 1] = gc[1]; grgb[3 * r + 2] = gc[2];
      girgb[3 * r] = gi[0]; girgb[3 * r + 1] = gi[1]; girgb[3 * r + 2] = gi[2];
      const_cast<float*>(gm.depth)[r] = gd;
      const_cast<float*>(gm.opacity_instance)[r] = go;
      const_cast<float*>(gm.depth_instance)[r] = gid;
    }
  }
}

// A validation record (onerf_validate_frame) to the loss outputs, with loss_grad_kernel's arithmetic (write_outputs), and
// the validation PSNR.  One thread: 18 doubles in, 12 values out.
__global__ void validate_finalize_kernel(LossParams P, const double* __restrict__ record, float* __restrict__ psnr_out) {
  if (threadIdx.x != 0) return;
  write_outputs(P.a, record);
  *psnr_out = (float)(-10.0 * log10(record[VR_PSNR_SUM] / record[VR_PSNR_COUNT]));   // 0 / 0: NaN, as mean([])
}

int loss_grid(onerf_ctx* ctx, int64_t n_rays) {
  const int64_t want = (n_rays + 255) / 256;
  return (int)(want < (int64_t)ctx->num_sms * 4 ? want : (int64_t)ctx->num_sms * 4);
}

bool maps_ok(const onerf_loss_maps& m) { return m.rgb && m.depth && m.opacity_instance && m.rgb_instance && m.depth_instance; }

}  // namespace

extern "C" size_t onerf_total_loss_workspace_bytes(void) { return WS_DOUBLES * sizeof(double); }

extern "C" int onerf_total_loss(onerf_ctx* ctx, const onerf_loss_args* a, void* stream_) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  ONERF_CHECK_ARG(a->n_rays > 0, "n_rays must be positive");
  ONERF_CHECK_ARG(a->rgbs && a->depths && a->valid_mask && a->instance_mask && a->instance_mask_weight, "null batch buffer");
  ONERF_CHECK_ARG(maps_ok(a->coarse) && maps_ok(a->grad_coarse), "null coarse map / gradient");
  ONERF_CHECK_ARG(!a->has_fine || (maps_ok(a->fine) && maps_ok(a->grad_fine)), "null fine map / gradient");
  ONERF_CHECK_ARG(a->loss_sum_out && a->terms_out && a->present_out && a->workspace, "null output / workspace");
  ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(a->workspace) & 7u) == 0, "workspace must be 8-byte aligned");
  cudaStream_t stream = (cudaStream_t)stream_;
  double* ws = reinterpret_cast<double*>(a->workspace);
  ONERF_CUDA(cudaMemsetAsync(ws, 0, WS_DOUBLES * sizeof(double), stream));
  LossParams P;
  P.a = *a;
  const int grid = loss_grid(ctx, a->n_rays);
  loss_reduce_kernel<<<grid, 256, 0, stream>>>(P, ws);
  ONERF_LAUNCH_CHECK(ctx);
  loss_grad_kernel<<<grid, 256, 0, stream>>>(P, ws);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int onerf_launch_batch_stats(onerf_ctx* ctx, const onerf_loss_args* a, double* ws, cudaStream_t stream) {
  LossParams P;
  P.a = *a;
  batch_stats_kernel<<<loss_grid(ctx, a->n_rays), 256, 0, stream>>>(P, ws);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_validate_finalize(onerf_ctx* ctx, const double* record, const float weights[5], int has_fine,
                                       float* loss_sum_out, float* terms_out, int* present_out, float* psnr_out,
                                       void* stream) {
  ONERF_CHECK_ARG(ctx && record && weights, "null argument");
  ONERF_CHECK_ARG(loss_sum_out && terms_out && present_out && psnr_out, "null output");
  ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(record) & 7u) == 0, "record must be 8-byte aligned");
  LossParams P;
  memset(&P, 0, sizeof(P));
  P.a.has_fine = has_fine;
  P.a.color_weight = weights[0]; P.a.depth_weight = weights[1]; P.a.opacity_weight = weights[2];
  P.a.instance_color_weight = weights[3]; P.a.instance_depth_weight = weights[4];
  P.a.loss_sum_out = loss_sum_out; P.a.terms_out = terms_out; P.a.present_out = present_out;
  validate_finalize_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(P, record, psnr_out);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
