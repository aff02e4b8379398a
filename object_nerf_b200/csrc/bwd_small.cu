// HBM-bound helpers of the tensor-core backward (SURVEY.md §8 row a14) and the device-side code library (row a6):
//   atom_colsum_kernel   column sums of bf16 atoms over all samples, optionally weighted per row by a component of a
//                        float4 array: bias gradients (db_l = sum_s dZ_l), sigma / rgb head weight gradients
//                        (dw_sigma = sum_s dsigma_s H_s, dW_rgb[c] = sum_s drgb_c,s Hdir_s)
//   ray_sum_kernel       per-ray sums of the dZ atoms whose layers take per-ray-constant inputs (direction encoding,
//                        object code): one warp per (ray, atom), no atomics
//   vec4_sum_kernel      head bias gradients: sum over samples of the float4 (d rgb_pre, d sigma)
//   code_gather / code_scatter_add   CodeLibrary.forward (models/code_library.py:18-28) and its gradient
#include "common.cuh"
#include "layout.h"

#include <cuda_bf16.h>

namespace {

struct ColsumJob {
  int64_t atom_off;     // byte offset of (tile 0, this atom)
  int atoms_slot;       // atoms per tile of the slot (tile stride = atoms_slot * 16 KB)
  int weight;           // 0: none; 1: scene .w; 2: scene .xyz (3 outputs); 3: object .w; 4: object .xyz
  int64_t out_off;      // float offset of column 0 (weight xyz: output c at out_off + c * out_cstride)
  int out_cstride;
};

constexpr int CS_MAX_JOBS = 64;
struct ColsumParams {
  const uint8_t* ws;
  const float4* dA_scene;
  const float4* dA_obj;
  float* out;
  int n_tiles;
  int64_t total;        // samples (rows beyond carry zero weight)
  int n_jobs;
  ColsumJob jobs[CS_MAX_JOBS];
};

__device__ __forceinline__ void unpack8(const uint4& q, float* f) {
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}

// block = 256 threads: lc = t & 7 owns columns 8 lc .. 8 lc + 7, rr = t >> 3 owns rows rr, rr + 32, rr + 64, rr + 96
__global__ void __launch_bounds__(256) atom_colsum_kernel(const __grid_constant__ ColsumParams P) {
  __shared__ float red[3][32][64 + 1];
  const ColsumJob j = P.jobs[blockIdx.y];
  const int lc = threadIdx.x & 7, rr = threadIdx.x >> 3;
  const int nw = (j.weight == 2 || j.weight == 4) ? 3 : 1;
  float acc[3][8];
#pragma unroll
  for (int w = 0; w < 3; ++w)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[w][c] = 0.0f;
  for (int tile = blockIdx.x; tile < P.n_tiles; tile += gridDim.x) {
    const uint8_t* atom = P.ws + j.atom_off + (size_t)tile * j.atoms_slot * ONERF_ATOM_BYTES;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = rr + 32 * i;
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(atom + row * 128 + ((lc ^ (row & 7)) << 4)));
      float f[8];
      unpack8(q, f);
      if (j.weight == 0) {
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[0][c] += f[c];
      } else {
        const int64_t e = (int64_t)tile * 128 + row;
        float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
        if (e < P.total) d = __ldg((j.weight <= 2 ? P.dA_scene : P.dA_obj) + e);
        if (nw == 1) {
#pragma unroll
          for (int c = 0; c < 8; ++c) acc[0][c] = fmaf(d.w, f[c], acc[0][c]);
        } else {
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            acc[0][c] = fmaf(d.x, f[c], acc[0][c]);
            acc[1][c] = fmaf(d.y, f[c], acc[1][c]);
            acc[2][c] = fmaf(d.z, f[c], acc[2][c]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int w = 0; w < 3; ++w)
#pragma unroll
    for (int c = 0; c < 8; ++c) red[w][rr][lc * 8 + c] = acc[w][c];
  __syncthreads();
  for (int o = threadIdx.x; o < nw * 64; o += 256) {
    const int w = o >> 6, col = o & 63;
    float s = 0.0f;
    for (int r = 0; r < 32; ++r) s += red[w][r][col];
    atomicAdd(P.out + j.out_off + (int64_t)w * j.out_cstride + col, s);
  }
}

// out[ray][col0 + lane * 2 + {0,1}] = sum over the ray's S samples of atom columns; one warp per (ray, job)
struct RaySumJob {
  int64_t atom_off;
  int atoms_slot;
  int out_col0;
};
struct RaySumParams {
  const uint8_t* ws;
  float* out;           // (n_rays, out_ld)
  int out_ld, n_rays, S, n_jobs;
  RaySumJob jobs[8];
};
__global__ void __launch_bounds__(256) ray_sum_kernel(const __grid_constant__ RaySumParams P) {
  const int lane = threadIdx.x & 31;
  const int64_t wid = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= (int64_t)P.n_rays * P.n_jobs) return;
  const int ray = (int)(wid / P.n_jobs), jb = (int)(wid - (int64_t)ray * P.n_jobs);
  const RaySumJob j = P.jobs[jb];
  float a0 = 0.0f, a1 = 0.0f;
  const int64_t e0 = (int64_t)ray * P.S;
  for (int s = 0; s < P.S; ++s) {
    const int64_t e = e0 + s;
    const int64_t tile = e >> 7;
    const int row = (int)(e & 127);
    const uint8_t* p = P.ws + j.atom_off + (size_t)tile * j.atoms_slot * ONERF_ATOM_BYTES + row * 128 +
                       ((((lane >> 2) ^ (row & 7))) << 4) + (lane & 3) * 4;
    const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(p));
    a0 += __uint_as_float(w << 16);
    a1 += __uint_as_float(w & 0xffff0000u);
  }
  float* o = P.out + (int64_t)ray * P.out_ld + j.out_col0 + lane * 2;
  o[0] = a0;
  o[1] = a1;
}

// out[0..3] += sum_e v[e]  (x, y, z to out_xyz[0..2], w to out_w[0])
__global__ void __launch_bounds__(256) vec4_sum_kernel(const float4* __restrict__ v, int64_t n, float* __restrict__ out_xyz,
                                                       float* __restrict__ out_w) {
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const float4 d = __ldg(v + e);
    a.x += d.x; a.y += d.y; a.z += d.z; a.w += d.w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a.x += __shfl_xor_sync(0xffffffffu, a.x, o);
    a.y += __shfl_xor_sync(0xffffffffu, a.y, o);
    a.z += __shfl_xor_sync(0xffffffffu, a.z, o);
    a.w += __shfl_xor_sync(0xffffffffu, a.w, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(out_xyz + 0, a.x);
    atomicAdd(out_xyz + 1, a.y);
    atomicAdd(out_xyz + 2, a.z);
    atomicAdd(out_w, a.w);
  }
}

// The table row of an instance id: ids outside [0, n_codes) are clamped to the nearest row (the ids are device data, so
// checking them on the host would cost a sync).  Gather and scatter share the rule, so a ray's code gradient goes to
// the row its code was read from.
__device__ __forceinline__ int64_t code_row(int64_t id, int n_codes) {
  return id < 0 ? 0 : (id >= n_codes ? n_codes - 1 : id);
}
__global__ void code_gather_kernel(const float* __restrict__ table, const int64_t* __restrict__ ids, int n, int n_codes,
                                   float* __restrict__ out) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n * 16; e += gridDim.x * blockDim.x) {
    const int r = e >> 4, c4 = e & 15;
    const int64_t id = code_row(ids[r], n_codes);
    reinterpret_cast<float4*>(out)[e] = __ldg(reinterpret_cast<const float4*>(table) + id * 16 + c4);
  }
}
__global__ void code_scatter_kernel(const float* __restrict__ d_codes, const int64_t* __restrict__ ids, int n, int n_codes,
                                    float* __restrict__ table_grad) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n * 64; e += gridDim.x * blockDim.x) {
    const int r = e >> 6, c = e & 63;
    atomicAdd(table_grad + code_row(ids[r], n_codes) * 64 + c, d_codes[e]);
  }
}

}  // namespace

// head weight / bias gradients into the kernel-layout gradient buffer (the GEMM layers' bias gradients are formed by the
// weight-gradient kernel, bwd_wgrad.cu, from the dZ tiles it streams)
int onerf_launch_bwd_colsums(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int64_t n_samples,
                             const float* dA_scene, const float* dA_obj, float* grad, cudaStream_t stream) {
  const GradLayout G = onerf_make_grad_layout(use_voxel);
  const TrainLayout T = onerf_make_train_layout(use_voxel, n_samples);
  ColsumParams P;
  memset(&P, 0, sizeof(P));
  P.ws = reinterpret_cast<const uint8_t*>(ws);
  P.dA_scene = reinterpret_cast<const float4*>(dA_scene);
  P.dA_obj = reinterpret_cast<const float4*>(dA_obj);
  P.out = grad;
  P.n_tiles = T.n_tiles;
  P.total = n_samples;
  const int gemm_of[ONERF_DZ_SLOTS] = {G_S0, G_S1, G_S2, G_S3, G_S4, G_S5, G_S6, G_S7, G_SFIN, G_SDIR,
                                       G_O0, G_O1, G_O2, G_O3, G_OFIN, G_ODIR};
  int n = 0;
  (void)gemm_of;
  auto head = [&](int act, int weight, int64_t out, int cstride) {
    for (int a = 0; a < T.act_atoms[act]; ++a)
      P.jobs[n++] = ColsumJob{T.act_off[act] + (int64_t)a * ONERF_ATOM_BYTES, T.act_atoms[act], weight, out + a * 64, cstride};
  };
  head(8, 1, G.sigma_w, 0);        // sigma head reads hidden 8
  head(10, 2, G.rgb_w, 128);       // rgb head reads the dir layer
  if (want_object) {
    head(14, 3, G.osigma_w, 0);
    head(16, 4, G.orgb_w, 64);
  }
  P.n_jobs = n;
  int gx = (8 * ctx->num_sms + n - 1) / n;     // ~8 CTAs per SM in flight: the kernel is a pure HBM stream
  if (gx > T.n_tiles) gx = T.n_tiles;
  if (gx < 1) gx = 1;
  atom_colsum_kernel<<<dim3(gx, n), 256, 0, stream>>>(P);
  ONERF_LAUNCH_CHECK(ctx);
  int blocks = (int)((n_samples + 255) / 256 < 4 * ctx->num_sms ? (n_samples + 255) / 256 : 4 * ctx->num_sms);
  vec4_sum_kernel<<<blocks, 256, 0, stream>>>(P.dA_scene, n_samples, grad + G.rgb_b, grad + G.sigma_b);
  ONERF_LAUNCH_CHECK(ctx);
  if (want_object) {
    vec4_sum_kernel<<<blocks, 256, 0, stream>>>(P.dA_obj, n_samples, grad + G.orgb_b, grad + G.osigma_b);
    ONERF_LAUNCH_CHECK(ctx);
  }
  return ONERF_OK;
}

// per-ray sums of dZ_dir (128) | dZ_odir (64) | dZ_o0 (128) | dZ_o2 (128) in the ray_const column layout (layout.h)
int onerf_launch_bwd_raysums(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int n_rays, int S, float* out,
                             cudaStream_t stream) {
  const TrainLayout T = onerf_make_train_layout(use_voxel, (int64_t)n_rays * S);
  RaySumParams P;
  memset(&P, 0, sizeof(P));
  P.ws = reinterpret_cast<const uint8_t*>(ws);
  P.out = out; P.out_ld = ONERF_RAY_CONST_FLOATS; P.n_rays = n_rays; P.S = S;
  int n = 0;
  auto add = [&](int dz, int col0) {
    for (int a = 0; a < T.dz_atoms[dz]; ++a)
      P.jobs[n++] = RaySumJob{T.dz_off[dz] + (int64_t)a * ONERF_ATOM_BYTES, T.dz_atoms[dz], col0 + a * 64};
  };
  add(9, RC_SDIR);
  if (want_object) { add(15, RC_ODIR); add(10, RC_OL0); add(12, RC_OL2); }
  P.n_jobs = n;
  const int64_t warps = (int64_t)n_rays * n;
  ray_sum_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(P);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_code_gather(onerf_ctx* ctx, const float* table, const int64_t* ids, int n, int n_codes, float* out,
                                 void* stream) {
  ONERF_CHECK_ARG(ctx && table && ids && out, "null argument");
  ONERF_CHECK_ARG(onerf_aligned16(table) && onerf_aligned16(out), "misaligned buffer");
  ONERF_CHECK_ARG(n >= 0 && (n == 0 || n_codes >= 1), "an empty code table has no row to read");
  if (n == 0) return ONERF_OK;
  code_gather_kernel<<<(n * 16 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(table, ids, n, n_codes, out);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_code_scatter_add(onerf_ctx* ctx, const float* d_codes, const int64_t* ids, int n, int n_codes,
                                      float* table_grad, void* stream) {
  ONERF_CHECK_ARG(ctx && d_codes && ids && table_grad, "null argument");
  ONERF_CHECK_ARG(n >= 0 && (n == 0 || n_codes >= 1), "an empty code table has no row to add to");
  if (n == 0) return ONERF_OK;
  code_scatter_kernel<<<(n * 64 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(d_codes, ids, n, n_codes, table_grad);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
