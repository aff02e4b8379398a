// FFMA (fp32) implementation of the fused encode + two-branch MLP, the per-ray-constant kernel shared
// with the tensor-core path, and the stand-alone encode entry point.
//
// This is the verification / gradient-check arithmetic (ONERF_PREC_FP32): same fusion and data flow as
// the wgmma kernel in field_tc.cu, fp32 end to end, accurate sinf/cosf.  A CTA owns 32 consecutive
// samples; activations live in shared memory as [k][32 samples]; each layer is a register-tiled
// 32 x N GEMM (thread = 4 samples x N/32 outputs) streaming W^T rows from L1/L2.
//
// Reference: models/rendering.py:85-137, models/nerf_model.py:97-152, models/embedding_helper.py:325-411,
// render_tools/multi_rendering.py:16-93.
#include "encode.cuh"
#include "field_common.cuh"

namespace {

constexpr int TS = 32;        // samples per CTA
constexpr float kLeaky = 0.01f;

template <int NO>
__device__ __forceinline__ void load_w(const float* __restrict__ p, float* w) {
  if constexpr (NO == 8) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p));
    const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
  } else if constexpr (NO == 4) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p));
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
  } else {
    const float2 a = __ldg(reinterpret_cast<const float2*>(p));
    w[0] = a.x; w[1] = a.y;
  }
}

// acc[4][NO] += A[K][32](this thread's 4 samples) . Wt[koff.., og*NO..]
template <int NO>
__device__ __forceinline__ void gemm_seg(const float* __restrict__ A, int K, const float* __restrict__ Wt,
                                         int N, int sg, int og, float (&acc)[4][NO]) {
  const float* wp = Wt + og * NO;
#pragma unroll 4
  for (int k = 0; k < K; ++k) {
    const float4 a = *reinterpret_cast<const float4*>(A + k * TS + 4 * sg);
    float w[NO];
    load_w<NO>(wp + (int64_t)k * N, w);
#pragma unroll
    for (int o = 0; o < NO; ++o) {
      acc[0][o] = fmaf(a.x, w[o], acc[0][o]);
      acc[1][o] = fmaf(a.y, w[o], acc[1][o]);
      acc[2][o] = fmaf(a.z, w[o], acc[2][o]);
      acc[3][o] = fmaf(a.w, w[o], acc[3][o]);
    }
  }
}

// One layer: out[n][s] = act( sum_seg A_seg . Wt + bias ), bias per column (bias != null) or per
// ray (rc_base >= 0: ray_const[ray(s)][rc_base + n]).  dump != null: also store the outputs as rows of a
// [samples x N] row-major matrix (backward support), first row = sample e0 of the tile.
template <int NO>
__device__ __forceinline__ void layer(const float* A0, int K0, const float* A1, int K1,
                                      const float* __restrict__ Wt, const float* __restrict__ bias,
                                      const float* __restrict__ ray_const, const int* s_ray, int rc_base,
                                      bool leaky, float* out, float* dump = nullptr, int64_t e0 = 0, int64_t total = 0) {
  const int N = 32 * NO;
  const int sg = threadIdx.x >> 5, og = threadIdx.x & 31;
  float acc[4][NO];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int o = 0; o < NO; ++o) acc[i][o] = 0.0f;
  gemm_seg<NO>(A0, K0, Wt, N, sg, og, acc);
  if (K1 > 0) gemm_seg<NO>(A1, K1, Wt + (int64_t)K0 * N, N, sg, og, acc);
#pragma unroll
  for (int o = 0; o < NO; ++o) {
    const int n = og * NO + o;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float bv = (rc_base >= 0)
                           ? __ldg(ray_const + (int64_t)s_ray[4 * sg + i] * ONERF_RAY_CONST_FLOATS + rc_base + n)
                           : __ldg(bias + n);
      float t = acc[i][o] + bv;
      if (leaky) t = t > 0.0f ? t : t * kLeaky;
      acc[i][o] = t;
    }
    *reinterpret_cast<float4*>(out + n * TS + 4 * sg) = make_float4(acc[0][o], acc[1][o], acc[2][o], acc[3][o]);
  }
  if (dump) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t e = e0 + 4 * sg + i;
      if (e < total) {
        float* d = dump + e * N + og * NO;   // a warp writes one contiguous row of N floats
#pragma unroll
        for (int o = 0; o < NO; ++o) d[o] = acc[i][o];
      }
    }
  }
}

// PE of NCH channels held in registers, written to X rows (reference order: [f, sin(2^0 f), cos(2^0 f), ...])
template <int NCH>
__device__ __forceinline__ void write_pe(float* X, int row0, int group_width, int ch0, const float* f,
                                         int n_freqs, int s) {
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    X[(row0 + ch0 + c) * TS + s] = f[c];
    for (int k = 0; k < n_freqs; ++k) {
      const float a = f[c] * (float)(1 << k);  // exact power-of-two scaling
      X[(row0 + group_width * (1 + 2 * k) + ch0 + c) * TS + s] = sinf(a);
      X[(row0 + group_width * (2 + 2 * k) + ch0 + c) * TS + s] = cosf(a);
    }
  }
}

template <bool VOXEL>
__global__ void __launch_bounds__(256) field_fp32_kernel(FieldParams p) {
  extern __shared__ __align__(16) float smem[];
  const PackLayout& L = p.L;
  const int KX = VOXEL ? 288 : 64, KO = VOXEL ? 384 : 64;
  float* X = smem;                 // [KO][32]
  float* H0 = X + KO * TS;         // [256][32]
  float* H1 = H0 + 256 * TS;       // [256][32]
  __shared__ int s_ray[TS];
  __shared__ float s_mute[TS];     // 1 -> scene sigma forced to -1e5 (box / zero ray); 2 bit -> object too
  const float* Pf = reinterpret_cast<const float*>(p.packed);
  const int64_t total = (int64_t)field_rays(p) * p.S;

  for (int64_t tile = blockIdx.x; tile * TS < total; tile += gridDim.x) {
    const int64_t e0 = tile * TS;
    // ---------------- encode ----------------
    {
      const int s = threadIdx.x & 31, role = threadIdx.x >> 5;
      const int64_t e = e0 + s;
      const bool live = e < total;
      const int ray = live ? (int)(e / p.S) : 0;
      const int i = live ? (int)(e - (int64_t)ray * p.S) : 0;
      const float* rr = p.rays + (int64_t)ray * 8;
      const float zz = live ? __ldg(p.z + (int64_t)ray * p.z_stride + i) : 0.0f;
      // xyz = o + d * z, individually rounded like the reference's broadcasted mul + add (rendering.py:279)
      float x = __fadd_rn(__ldg(rr + 0), __fmul_rn(__ldg(rr + 3), zz));
      float y = __fadd_rn(__ldg(rr + 1), __fmul_rn(__ldg(rr + 4), zz));
      float z = __fadd_rn(__ldg(rr + 2), __fmul_rn(__ldg(rr + 5), zz));
      if (p.xyz && live) {
        const float* q = p.xyz + ((int64_t)ray * p.S + i) * 3;
        x = __ldg(q); y = __ldg(q + 1); z = __ldg(q + 2);
      }
      if (VOXEL) {
        const GridView g = load_grid_view(p.grid);
        if (role < 4) {
          float f[4];
          if (role == 0) voxel_trilinear<0, 4, true>(g, x, y, z, f);
          else if (role == 1) voxel_trilinear<4, 4, true>(g, x, y, z, f);
          else if (role == 2) voxel_trilinear<8, 4, true>(g, x, y, z, f);
          else voxel_trilinear<12, 4, true>(g, x, y, z, f);
          write_pe<4>(X, 0, 16, role * 4, f, 6, s);
        } else if (role < 6) {
          float f[4];
          if (role == 4) voxel_trilinear<16, 4, true>(g, x, y, z, f);
          else voxel_trilinear<20, 4, true>(g, x, y, z, f);
          write_pe<4>(X, 272, 8, (role - 4) * 4, f, 6, s);
        } else if (role == 6) {
          const float f[3] = {x, y, z};
          write_pe<3>(X, 208, 3, 0, f, 10, s);
        } else {
          X[271 * TS + s] = 0.0f;
          for (int k = 376; k < 384; ++k) X[k * TS + s] = 0.0f;
        }
      } else {
        if (role == 0) {
          const float f[3] = {x, y, z};
          write_pe<3>(X, 0, 3, 0, f, 10, s);
          X[63 * TS + s] = 0.0f;
        }
      }
      if (role == 7) {
        s_ray[s] = ray;
        float m = 0.0f;
        if (live && p.mute_zero_rays && __ldg(p.z + (int64_t)ray * p.z_stride + (p.S - 1)) == 0.0f) m = 3.0f;
        if (live && m == 0.0f && point_in_boxes(p.boxes, p.n_boxes, x, y, z)) m = 1.0f;
        s_mute[s] = m;
      }
    }
    __syncthreads();
    if (p.dump_x) {
      for (int idx = threadIdx.x; idx < KO * TS; idx += blockDim.x) {
        const int k = idx / TS, sidx = idx % TS;
        if (e0 + sidx < total) p.dump_x[(e0 + sidx) * KO + k] = X[k * TS + sidx];
      }
    }
    const float* rc = p.ray_const;
    // ---------------- scene branch (models/nerf_model.py:97-121) ----------------
    if (p.want_scene) {
      layer<8>(X, KX, nullptr, 0, Pf + L.g[G_S0].wt_off, Pf + L.g[G_S0].bias_off, rc, s_ray, -1, true, H0, p.dump_s[0], e0, total); __syncthreads();
      layer<8>(H0, 256, nullptr, 0, Pf + L.g[G_S1].wt_off, Pf + L.g[G_S1].bias_off, rc, s_ray, -1, true, H1, p.dump_s[1], e0, total); __syncthreads();
      layer<8>(H1, 256, nullptr, 0, Pf + L.g[G_S2].wt_off, Pf + L.g[G_S2].bias_off, rc, s_ray, -1, true, H0, p.dump_s[2], e0, total); __syncthreads();
      layer<8>(H0, 256, nullptr, 0, Pf + L.g[G_S3].wt_off, Pf + L.g[G_S3].bias_off, rc, s_ray, -1, true, H1, p.dump_s[3], e0, total); __syncthreads();
      layer<8>(X, KX, H1, 256, Pf + L.g[G_S4].wt_off, Pf + L.g[G_S4].bias_off, rc, s_ray, -1, true, H0, p.dump_s[4], e0, total); __syncthreads();
      layer<8>(H0, 256, nullptr, 0, Pf + L.g[G_S5].wt_off, Pf + L.g[G_S5].bias_off, rc, s_ray, -1, true, H1, p.dump_s[5], e0, total); __syncthreads();
      layer<8>(H1, 256, nullptr, 0, Pf + L.g[G_S6].wt_off, Pf + L.g[G_S6].bias_off, rc, s_ray, -1, true, H0, p.dump_s[6], e0, total); __syncthreads();
      layer<8>(H0, 256, nullptr, 0, Pf + L.g[G_S7].wt_off, Pf + L.g[G_S7].bias_off, rc, s_ray, -1, true, H1, p.dump_s[7], e0, total); __syncthreads();
      float sigma = 0.0f;
      if (threadIdx.x < TS) {
        const int s = threadIdx.x;
        sigma = __ldg(Pf + L.sigma_b);
        for (int k = 0; k < 256; ++k) sigma = fmaf(H1[k * TS + s], __ldg(Pf + L.sigma_w + k), sigma);
      }
      layer<8>(H1, 256, nullptr, 0, Pf + L.g[G_SFIN].wt_off, Pf + L.g[G_SFIN].bias_off, rc, s_ray, -1, false, H0, p.dump_s[8], e0, total); __syncthreads();
      layer<4>(H0, 256, nullptr, 0, Pf + L.g[G_SDIR].wt_off, nullptr, rc, s_ray, RC_SDIR, true, H1, p.dump_s[9], e0, total); __syncthreads();
      if (threadIdx.x < TS) {
        const int s = threadIdx.x;
        const int64_t e = e0 + s;
        if (e < total) {
          float c[3];
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            float a = __ldg(Pf + L.rgb_b + j);
            for (int k = 0; k < 128; ++k) a = fmaf(H1[k * TS + s], __ldg(Pf + L.rgb_w + j * 128 + k), a);
            c[j] = 1.0f / (1.0f + expf(-a));
          }
          if (s_mute[s] != 0.0f) sigma = -1e5f;
          const int ray = s_ray[s];
          const int i = (int)(e - (int64_t)ray * p.S);
          reinterpret_cast<float4*>(p.scene_out)[(int64_t)ray * p.out_stride + i] = make_float4(c[0], c[1], c[2], sigma);
        }
      }
      __syncthreads();
    }
    // ---------------- object branch (models/nerf_model.py:123-152) ----------------
    if (p.want_object) {
      layer<4>(X, KO, nullptr, 0, Pf + L.g[G_O0].wt_off, nullptr, rc, s_ray, RC_OL0, true, H0, p.dump_o[0], e0, total); __syncthreads();
      layer<4>(H0, 128, nullptr, 0, Pf + L.g[G_O1].wt_off, Pf + L.g[G_O1].bias_off, rc, s_ray, -1, true, H1, p.dump_o[1], e0, total); __syncthreads();
      layer<4>(X, KO, H1, 128, Pf + L.g[G_O2].wt_off, nullptr, rc, s_ray, RC_OL2, true, H0, p.dump_o[2], e0, total); __syncthreads();
      layer<4>(H0, 128, nullptr, 0, Pf + L.g[G_O3].wt_off, Pf + L.g[G_O3].bias_off, rc, s_ray, -1, true, H1, p.dump_o[3], e0, total); __syncthreads();
      float sigma = 0.0f;
      if (threadIdx.x < TS) {
        const int s = threadIdx.x;
        sigma = __ldg(Pf + L.osigma_b);
        for (int k = 0; k < 128; ++k) sigma = fmaf(H1[k * TS + s], __ldg(Pf + L.osigma_w + k), sigma);
      }
      layer<4>(H1, 128, nullptr, 0, Pf + L.g[G_OFIN].wt_off, Pf + L.g[G_OFIN].bias_off, rc, s_ray, -1, false, H0, p.dump_o[4], e0, total); __syncthreads();
      layer<2>(H0, 128, nullptr, 0, Pf + L.g[G_ODIR].wt_off, nullptr, rc, s_ray, RC_ODIR, true, H1, p.dump_o[5], e0, total); __syncthreads();
      if (threadIdx.x < TS) {
        const int s = threadIdx.x;
        const int64_t e = e0 + s;
        if (e < total) {
          float c[3];
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            float a = __ldg(Pf + L.orgb_b + j);
            for (int k = 0; k < 64; ++k) a = fmaf(H1[k * TS + s], __ldg(Pf + L.orgb_w + j * 64 + k), a);
            c[j] = 1.0f / (1.0f + expf(-a));
          }
          if (s_mute[s] >= 2.0f) sigma = -1e5f;
          const int ray = s_ray[s];
          const int i = (int)(e - (int64_t)ray * p.S);
          reinterpret_cast<float4*>(p.obj_out)[(int64_t)ray * p.out_stride + i] = make_float4(c[0], c[1], c[2], sigma);
        }
      }
      __syncthreads();
    }
  }
}

// Per-ray constants: direction encoding through the dir layers' direction columns, object code through
// object layers 0 / 2 code columns, plus those layers' biases.  8 rays per CTA, 128 threads.
__global__ void __launch_bounds__(128) ray_const_kernel(FieldParams p) {
  __shared__ float s_dir[8][ONERF_NDIR + 1];
  __shared__ float s_code[8][ONERF_NCODE];
  const PackLayout& L = p.L;
  const float* Pf = reinterpret_cast<const float*>(p.packed);
  const int n_rays = field_rays(p);
  const int r0 = blockIdx.x * 8;
  if (r0 >= n_rays) return;
  for (int t = threadIdx.x; t < 8 * 3; t += blockDim.x) {
    const int lr = t / 3, c = t % 3;
    const int ray = min(r0 + lr, n_rays - 1);
    const float d = __ldg(p.rays + (int64_t)ray * 8 + 3 + c);
    s_dir[lr][c] = d;
    for (int k = 0; k < 4; ++k) {
      const float a = d * (float)(1 << k);
      s_dir[lr][3 * (1 + 2 * k) + c] = sinf(a);
      s_dir[lr][3 * (2 + 2 * k) + c] = cosf(a);
    }
  }
  for (int t = threadIdx.x; t < 8 * ONERF_NCODE; t += blockDim.x) {
    const int lr = t / ONERF_NCODE, c = t % ONERF_NCODE;
    const int ray = min(r0 + lr, n_rays - 1);
    float v = 0.0f;
    if (p.want_object) v = p.codes ? __ldg(p.codes + (int64_t)ray * ONERF_NCODE + c) : __ldg(p.code_row + c);
    s_code[lr][c] = v;
  }
  __syncthreads();
  const int n = threadIdx.x;  // output column 0..127
  float a_sdir[8], a_odir[8], a_ol0[8], a_ol2[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    a_sdir[r] = __ldg(Pf + L.b_sdir + n);
    a_odir[r] = (n < 64) ? __ldg(Pf + L.b_odir + n) : 0.0f;
    a_ol0[r] = __ldg(Pf + L.b_ol0 + n);
    a_ol2[r] = __ldg(Pf + L.b_ol2 + n);
  }
  for (int k = 0; k < ONERF_NDIR; ++k) {
    const float ws = __ldg(Pf + L.h_sdir + k * 128 + n);
    const float wo = (n < 64) ? __ldg(Pf + L.h_odir + k * 64 + n) : 0.0f;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      a_sdir[r] = fmaf(s_dir[r][k], ws, a_sdir[r]);
      a_odir[r] = fmaf(s_dir[r][k], wo, a_odir[r]);
    }
  }
  if (p.want_object) {
    for (int k = 0; k < ONERF_NCODE; ++k) {
      const float w0 = __ldg(Pf + L.h_ol0 + k * 128 + n);
      const float w2 = __ldg(Pf + L.h_ol2 + k * 128 + n);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        a_ol0[r] = fmaf(s_code[r][k], w0, a_ol0[r]);
        a_ol2[r] = fmaf(s_code[r][k], w2, a_ol2[r]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int ray = r0 + r;
    if (ray >= n_rays) break;
    float* o = p.ray_const + (int64_t)ray * ONERF_RAY_CONST_FLOATS;
    o[RC_SDIR + n] = a_sdir[r];
    if (n < 64) o[RC_ODIR + n] = a_odir[r];
    o[RC_OL0 + n] = a_ol0[r];
    o[RC_OL2 + n] = a_ol2[r];
  }
}

// Stand-alone encoder (test / ncu entry): fp32 outputs in the reference's column order.
__global__ void __launch_bounds__(256)
encode_kernel(onerf_grid grid, int has_grid, const float* __restrict__ xyz, int64_t n, float* __restrict__ scene_in,
              float* __restrict__ obj_in) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const float x = xyz[e * 3 + 0], y = xyz[e * 3 + 1], z = xyz[e * 3 + 2];
    const int width = has_grid ? 271 : 63;
    float* so = scene_in + e * width;
    int base = 0;
    if (has_grid) {
      const GridView g = load_grid_view(grid);
      float f[24];
      voxel_trilinear<0, 24, true>(g, x, y, z, f);
      for (int c = 0; c < 16; ++c) {
        so[c] = f[c];
        for (int k = 0; k < 6; ++k) {
          const float a = f[c] * (float)(1 << k);
          so[16 * (1 + 2 * k) + c] = sinf(a);
          so[16 * (2 + 2 * k) + c] = cosf(a);
        }
      }
      float* oo = obj_in + e * 104;
      for (int c = 0; c < 8; ++c) {
        oo[c] = f[16 + c];
        for (int k = 0; k < 6; ++k) {
          const float a = f[16 + c] * (float)(1 << k);
          oo[8 * (1 + 2 * k) + c] = sinf(a);
          oo[8 * (2 + 2 * k) + c] = cosf(a);
        }
      }
      base = 208;
    }
    const float v[3] = {x, y, z};
    for (int c = 0; c < 3; ++c) {
      so[base + c] = v[c];
      for (int k = 0; k < 10; ++k) {
        const float a = v[c] * (float)(1 << k);
        so[base + 3 * (1 + 2 * k) + c] = sinf(a);
        so[base + 3 * (2 + 2 * k) + c] = cosf(a);
      }
    }
  }
}

}  // namespace

int onerf_launch_ray_const(onerf_ctx* ctx, const FieldParams& p, cudaStream_t stream) {
  ray_const_kernel<<<(p.n_rays + 7) / 8, 128, 0, stream>>>(p);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int onerf_launch_field_fp32(onerf_ctx* ctx, const FieldParams& p, cudaStream_t stream) {
  const int64_t total = (int64_t)p.n_rays * p.S;
  const int64_t tiles = (total + TS - 1) / TS;
  int blocks = (int)(tiles < (int64_t)ctx->num_sms * 8 ? tiles : (int64_t)ctx->num_sms * 8);
  if (p.L.use_voxel) {
    const size_t smem = (size_t)(384 + 512) * TS * sizeof(float);
    ONERF_CUDA(cudaFuncSetAttribute(field_fp32_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    field_fp32_kernel<true><<<blocks, 256, smem, stream>>>(p);
  } else {
    const size_t smem = (size_t)(64 + 512) * TS * sizeof(float);
    ONERF_CUDA(cudaFuncSetAttribute(field_fp32_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    field_fp32_kernel<false><<<blocks, 256, smem, stream>>>(p);
  }
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_encode(onerf_ctx* ctx, const onerf_grid* grid, const float* xyz, int64_t n_points,
                            float* scene_in, float* obj_in, void* stream) {
  ONERF_CHECK_ARG(ctx && (n_points == 0 || (xyz && scene_in)), "null argument");   // (empty tensors have no data)
  ONERF_CHECK_ARG(n_points >= 0, "bad shape");
  if (grid) ONERF_CHECK_ARG((n_points == 0 || obj_in) && grid->table && grid->idx_map && grid->voxel_offset && grid->voxel_size && grid->voxel_shape, "null grid buffer");
  if (grid) ONERF_CHECK_ARG(onerf_aligned16(grid->table), "misaligned grid table (rows are read as float4)");
  if (n_points == 0) return ONERF_OK;
  onerf_grid g = grid ? *grid : onerf_grid{nullptr, nullptr, nullptr, nullptr, nullptr};
  int blocks = (int)((n_points + 255) / 256);
  if (blocks > ctx->num_sms * 16) blocks = ctx->num_sms * 16;
  encode_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(g, grid ? 1 : 0, xyz, n_points, scene_in, obj_in);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

// Raw trilinear voxel features (no positional encoding): compute_voxel_features_sparse(xyz, trilinear_interpolate=True,
// positional_embedding=False), models/embedding_helper.py:354-411 - what voxel_subdivision (:250-252) samples to
// initialise the refined grid.  Same individually rounded arithmetic as the stand-alone encoder.
namespace {
__global__ void __launch_bounds__(256)
voxel_features_kernel(onerf_grid grid, const float* __restrict__ xyz, int64_t n, float* __restrict__ out) {
  const GridView g = load_grid_view(grid);
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    float f[24];
    voxel_trilinear<0, 24, true>(g, xyz[e * 3 + 0], xyz[e * 3 + 1], xyz[e * 3 + 2], f);
    float4* o = reinterpret_cast<float4*>(out + e * 24);
#pragma unroll
    for (int q = 0; q < 6; ++q) o[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
  }
}
}  // namespace

extern "C" int onerf_voxel_features(onerf_ctx* ctx, const onerf_grid* grid, const float* xyz, int64_t n_points, float* out,
                                    void* stream) {
  ONERF_CHECK_ARG(ctx && grid && (n_points == 0 || (xyz && out)), "null argument");   // (empty tensors have no data)
  ONERF_CHECK_ARG(grid->table && grid->idx_map && grid->voxel_offset && grid->voxel_size && grid->voxel_shape, "null grid buffer");
  ONERF_CHECK_ARG(n_points >= 0 && onerf_aligned16(out) && onerf_aligned16(grid->table), "bad count or misaligned buffer");
  if (n_points == 0) return ONERF_OK;
  int blocks = (int)((n_points + 255) / 256);
  if (blocks > ctx->num_sms * 16) blocks = ctx->num_sms * 16;
  voxel_features_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(*grid, xyz, n_points, out);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
