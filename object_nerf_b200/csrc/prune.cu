// Voxel pruning entry points (include/onerf_ext.h: onerf_prune_measure, onerf_prune_apply).  The bf16 measure is one
// launch of the fused tensor-core pass (field_tc.cu: prune_tc_kernel); the fp32 measure stages each chunk of voxels
// through the FFMA field kernel: points -> scene-only field -> per-voxel maximum of alpha.

#include "prune.cuh"
#include "../../include/onerf_ext.h"

namespace {

constexpr int kChunkVoxels = 32;                                  // voxels per fp32 chunk (the reference's batch)
constexpr int64_t kChunkPoints = (int64_t)kChunkVoxels * kPruneSamples;

struct PruneWs {
  float *xyz, *z, *rays, *ray_const, *out;
  size_t total;
};

PruneWs prune_ws_layout(char* base) {
  PruneWs w;
  WsCarver c{base};
  w.xyz = c.floats(kChunkPoints * 3);
  w.z = c.floats(kChunkPoints);                       // zero depths and one zero ray: the field reads xyz
  w.rays = c.floats(8);
  w.ray_const = c.floats(ONERF_RAY_CONST_FLOATS);
  w.out = c.floats(kChunkPoints * 4);
  w.total = c.off;
  return w;
}

// points of voxels [k0, k0 + nk) -> xyz rows (k - k0) * 4096 + s
__global__ void __launch_bounds__(256) prune_points_kernel(PruneSource src, onerf_grid grid, int64_t k0, int nk,
                                                           float* __restrict__ xyz) {
  const GridView g = load_grid_view(grid);
  const int64_t n = (int64_t)nk * kPruneSamples;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    float p[3];
    prune_point(src, g, k0 + e / kPruneSamples, (int)(e % kPruneSamples), p);
    xyz[e * 3 + 0] = p[0];
    xyz[e * 3 + 1] = p[1];
    xyz[e * 3 + 2] = p[2];
  }
}

// one block per voxel: max over its 4096 (rgb, sigma) rows of alpha
__global__ void __launch_bounds__(256) prune_max_kernel(const float4* __restrict__ field, float* __restrict__ max_alpha) {
  __shared__ float red[8];
  const float4* f = field + (int64_t)blockIdx.x * kPruneSamples;
  float m = 0.0f;
  for (int s = threadIdx.x; s < kPruneSamples; s += blockDim.x) m = fmaxf(m, prune_alpha(f[s].w));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    max_alpha[blockIdx.x] = m;
  }
}

__global__ void __launch_bounds__(256) prune_apply_kernel(const int64_t* __restrict__ cells, int64_t n_cells,
                                                          const float* __restrict__ max_alpha, float th, int64_t dim_y,
                                                          int64_t dim_z, uint8_t* occupancy, int64_t* idx_map,
                                                          unsigned long long* n_pruned) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_cells; k += (int64_t)gridDim.x * blockDim.x) {
    if (!(max_alpha[k] < th)) continue;
    const int64_t cell = (cells[3 * k] * dim_y + cells[3 * k + 1]) * dim_z + cells[3 * k + 2];
    occupancy[cell] = 0;
    idx_map[cell] = -1;
    atomicAdd(n_pruned, 1ull);
  }
}

int blocks_for(onerf_ctx* ctx, int64_t n) {
  const int64_t b = (n + 255) / 256, cap = (int64_t)ctx->num_sms * 16;
  return (int)(b < cap ? b : cap);
}

}  // namespace

extern "C" size_t onerf_prune_workspace_bytes(int precision) {
  return precision == ONERF_PREC_FP32 ? prune_ws_layout(nullptr).total : 0;
}

extern "C" int onerf_prune_measure(onerf_ctx* ctx, const onerf_prune_args* a, void* stream_) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  ONERF_CHECK_ARG(a->grid, "the pruning pass needs the voxel model's grid");
  int rc = onerf_check_grid(__func__, a->grid);
  if (rc != ONERF_OK) return rc;
  ONERF_CHECK_ARG(a->packed, "null packed weights");
  ONERF_CHECK_ARG(a->precision == ONERF_PREC_FP32 || a->precision == ONERF_PREC_BF16, "unknown precision");
  ONERF_CHECK_ARG(a->n_cells >= 0 && a->cell_begin >= 0 && a->cell_begin <= a->cell_end && a->cell_end <= a->n_cells,
                  "shard outside [0, n_cells]");
  const int64_t nk = a->cell_end - a->cell_begin;
  ONERF_CHECK_ARG(a->n_cells == 0 || a->cells, "null cells");
  ONERF_CHECK_ARG(nk == 0 || a->max_alpha_out, "null max_alpha_out");
  ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(a->cells) & 7u) == 0, "cells must be 8-byte aligned");
  ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(a->jitter) & 3u) == 0 && (reinterpret_cast<uintptr_t>(a->max_alpha_out) & 3u) == 0,
                  "jitter / max_alpha_out must be 4-byte aligned");
  const size_t need = onerf_prune_workspace_bytes(a->precision);
  if (need > 0) {
    rc = onerf_check_workspace(__func__, a->workspace, a->workspace_bytes, need, ONERF_ERR_WORKSPACE);
    if (rc != ONERF_OK) return rc;
  }
  if (nk == 0) return ONERF_OK;
  cudaStream_t stream = (cudaStream_t)stream_;
  ONERF_CUDA(cudaMemsetAsync(a->max_alpha_out, 0, (size_t)nk * sizeof(float), stream));
  FieldParams p = onerf_field_params(a->grid, a->packed);
  p.want_scene = 1;
  const PruneSource src{a->cells, a->jitter, a->seed};
  if (a->precision == ONERF_PREC_BF16)
    return onerf_launch_prune_bf16(ctx, p, src, a->cell_begin, nk, a->max_alpha_out, stream);

  // fp32: one ray of up to kChunkPoints samples per chunk, with the points as explicit xyz
  const PruneWs w = prune_ws_layout(reinterpret_cast<char*>(a->workspace));
  ONERF_CUDA(cudaMemsetAsync(w.z, 0, (reinterpret_cast<char*>(w.ray_const) - reinterpret_cast<char*>(w.z)), stream));
  p.rays = w.rays; p.z = w.z; p.xyz = w.xyz;
  p.n_rays = 1;
  p.ray_const = w.ray_const;
  p.scene_out = w.out;
  rc = onerf_launch_ray_const(ctx, p, stream);   // (the direction layers run after sigma; their input is defined)
  if (rc != ONERF_OK) return rc;
  for (int64_t k0 = a->cell_begin; k0 < a->cell_end; k0 += kChunkVoxels) {
    const int n = (int)(a->cell_end - k0 < kChunkVoxels ? a->cell_end - k0 : kChunkVoxels);
    prune_points_kernel<<<blocks_for(ctx, (int64_t)n * kPruneSamples), 256, 0, stream>>>(src, *a->grid, k0, n, w.xyz);
    ONERF_LAUNCH_CHECK(ctx);
    p.S = n * kPruneSamples;
    p.z_stride = p.out_stride = p.S;
    rc = onerf_launch_field_fp32(ctx, p, stream);
    if (rc != ONERF_OK) return rc;
    prune_max_kernel<<<n, 256, 0, stream>>>(reinterpret_cast<const float4*>(w.out), a->max_alpha_out + (k0 - a->cell_begin));
    ONERF_LAUNCH_CHECK(ctx);
  }
  return ONERF_OK;
}

extern "C" int onerf_prune_apply(onerf_ctx* ctx, const int64_t* cells, int64_t n_cells, const float* max_alpha,
                                 float max_alpha_th, int64_t dim_y, int64_t dim_z, uint8_t* occupancy, int64_t* idx_map,
                                 int64_t* n_pruned, void* stream_) {
  ONERF_CHECK_ARG(ctx && occupancy && idx_map && n_pruned, "null argument");
  ONERF_CHECK_ARG(n_cells >= 0 && dim_y >= 1 && dim_z >= 1, "bad shape");
  ONERF_CHECK_ARG(n_cells == 0 || (cells && max_alpha), "null cells / max_alpha");
  ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(cells) & 7u) == 0 && (reinterpret_cast<uintptr_t>(idx_map) & 7u) == 0 &&
                      (reinterpret_cast<uintptr_t>(n_pruned) & 7u) == 0 && (reinterpret_cast<uintptr_t>(max_alpha) & 3u) == 0,
                  "misaligned buffer");
  cudaStream_t stream = (cudaStream_t)stream_;
  ONERF_CUDA(cudaMemsetAsync(n_pruned, 0, sizeof(int64_t), stream));
  if (n_cells == 0) return ONERF_OK;
  prune_apply_kernel<<<blocks_for(ctx, n_cells), 256, 0, stream>>>(cells, n_cells, max_alpha, max_alpha_th, dim_y, dim_z,
                                                                   occupancy, idx_map,
                                                                   reinterpret_cast<unsigned long long*>(n_pruned));
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
