// wgmma (Hopper tensor core) implementation of the fused encode + two-branch MLP for sm_90a.
//
// One persistent CTA per SM; a CTA owns one 128-sample tile at a time (tc_chain.cuh).
//   warpgroups 0 / 1 (256 thr)  encode rows [0, 64) / [64, 128) of the tile into shared memory (X, bf16, K-major
//                               SWIZZLE_128B atoms) and run every layer on them: wgmma M = 64 with the accumulator in
//                               registers, then the epilogue (bias / per-ray constant -> LeakyReLU -> bf16 pairs) leaves
//                               the output in registers as the NEXT layer's A operand.  Hidden activations never touch
//                               shared or global memory.  Heads (sigma, rgb) are CUDA-core dot products on the fp32
//                               values, reduced over the four lanes that share a row.
//   warpgroup 2                 its first warp streams the weights global -> shared with cp.async.bulk (pre-swizzled
//                               SWIZZLE_64B stage images written by pack.cu) through an mbarrier ring running ahead across
//                               layers and tiles; the warpgroup hands most of its registers to warpgroups 0 / 1.
// Skip / dir / code concatenations never materialise: a skip layer takes K-slabs from both X and H, and the
// per-ray-constant terms arrive through ray_const (see layout.h).
//
// Reference semantics: models/rendering.py:85-137, models/nerf_model.py:97-152,
// models/embedding_helper.py:325-411, render_tools/multi_rendering.py:16-93.
#include <cuda_bf16.h>

#include "encode.cuh"
#include "field_common.cuh"
#include "tc_chain.cuh"
#include "field_pe.cuh"

namespace {

using namespace tc;

constexpr float kLeaky = 0.01f;

enum Epi { EPI_HIDDEN = 0, EPI_HIDDEN_RC = 1, EPI_HIDDEN_SIGMA = 2, EPI_FINAL = 3, EPI_DIR = 4 };

struct TcParams {
  FieldParams f;
  WLayer layers[MAX_LAYERS];   // producer program (same order as the consumers' layer sequence)
  int n_layers;
  // training forward (DUMP): every layer's output activations (bf16 atoms), the encoded input X and the LeakyReLU sign
  // masks are left in the training workspace for the tensor-core backward (layout.h: TrainLayout)
  uint8_t* dump;
  TrainLayout TL;
  uint32_t* diag;   // mbarrier timeout record (onerf_ctx)
};

struct RowMeta {
  int ray, si, mute, live;   // mute bit 0: scene sigma muted, bit 1: object sigma muted
};

// the two rows of one thread in the accumulator fragment (tc_common.cuh)
struct Rows {
  int row[2];       // tile rows
  int live[2];
  int ray[2], si[2], mute[2];
  const float* rc[2];
  int64_t tile;
};

__device__ __forceinline__ uint32_t leaky_bf16x2(uint32_t x) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&x);
  const __nv_bfloat162 slope = __floats2bfloat162_rn(kLeaky, kLeaky);
  v = __hmax2(v, __hmul2(v, slope));
  return *reinterpret_cast<uint32_t*>(&v);
}

// store the packed output of one layer and (mask_word0 >= 0) its sign masks in the training dump
template <int N>
__device__ __forceinline__ void dump_layer(const TcParams& P, const Rows& R, int slot, int mask_word0, const uint32_t* pk) {
  const int q = threadIdx.x & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = R.row[r];
    uint8_t* base = P.dump + P.TL.act_off[slot] + ((size_t)R.tile * P.TL.act_atoms[slot]) * ATOM_BYTES + (size_t)row * 128 + q * 4;
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
      *reinterpret_cast<uint32_t*>(base + (size_t)(j >> 3) * ATOM_BYTES + (((j & 7) ^ (row & 7)) << 4)) = pk[2 * j + r];
  }
  if (mask_word0 < 0) return;
  // bit b of mask word w = the bf16 at column w * CPW + b is non-negative (CPW = 32, or 16 for the 64-wide layer)
  constexpr int CPW = N >= 128 ? 32 : 16, NW = N / CPW, BPW = CPW / 8;
  uint32_t* mrow = reinterpret_cast<uint32_t*>(P.dump + P.TL.mask_off) + ((size_t)R.tile * ONERF_MASK_WORDS + mask_word0) * 128;
#pragma unroll
  for (int w = 0; w < NW; ++w) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      uint32_t m = 0;
#pragma unroll
      for (int jj = 0; jj < BPW; ++jj) {
        const uint32_t v = pk[2 * (w * BPW + jj) + r];
        const uint32_t bits = (((v >> 15) & 1u) ^ 1u) | ((((v >> 31) & 1u) ^ 1u) << 1);
        m |= bits << (8 * jj + 2 * q);
      }
      m |= __shfl_xor_sync(0xffffffffu, m, 1);
      m |= __shfl_xor_sync(0xffffffffu, m, 2);
      if (q == 0) mrow[w * 128 + R.row[r]] = m;
    }
  }
}

// Epilogue of one layer for one thread: t = acc + bias (fp32), then
//   HIDDEN / HIDDEN_RC / FINAL: one rounding to bf16, LeakyReLU on packed bf16 pairs (not for FINAL);
//   HIDDEN_SIGMA: LeakyReLU in fp32, sigma head dot product on the un-rounded values (models/nerf_model.py:108,140);
//   DIR: LeakyReLU in fp32 feeding the 3-wide rgb head (fp32 dots).
// part[r] accumulates the row's head partial sums (sigma, r, g, b) over this thread's columns.
template <int N, int EPI>
__device__ __forceinline__ void epilogue(const float (&acc)[N / 2], uint32_t* pk, const float* bias, const Rows& R,
                                         int rc_base, const float* headw, float (&part)[2][4]) {
  const int q = threadIdx.x & 3;
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int c = 8 * j + 2 * q;
    float2 b[2];
    if (EPI == EPI_HIDDEN_RC || EPI == EPI_DIR) {
      b[0] = __ldg(reinterpret_cast<const float2*>(R.rc[0] + rc_base + c));
      b[1] = __ldg(reinterpret_cast<const float2*>(R.rc[1] + rc_base + c));
    } else {
      b[0] = b[1] = *reinterpret_cast<const float2*>(bias + c);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float t0 = acc[4 * j + 2 * r] + b[r].x, t1 = acc[4 * j + 2 * r + 1] + b[r].y;
      uint32_t p;
      if (EPI == EPI_HIDDEN || EPI == EPI_HIDDEN_RC) {
        p = leaky_bf16x2(pack_bf16(t0, t1));
      } else if (EPI == EPI_FINAL) {
        p = pack_bf16(t0, t1);
      } else {
        t0 = fmaxf(t0, t0 * kLeaky);
        t1 = fmaxf(t1, t1 * kLeaky);
        if (EPI == EPI_HIDDEN_SIGMA) {
          const float2 w = __ldg(reinterpret_cast<const float2*>(headw + c));
          part[r][0] = fmaf(t1, w.y, fmaf(t0, w.x, part[r][0]));
        } else {
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const float2 w = __ldg(reinterpret_cast<const float2*>(headw + k * N + c));
            part[r][1 + k] = fmaf(t1, w.y, fmaf(t0, w.x, part[r][1 + k]));
          }
        }
        p = pack_bf16(t0, t1);
      }
      pk[2 * j + r] = p;
    }
  }
}

// finish the heads of one branch: sum the four lanes of each row, add the head biases, write (rgb, sigma)
__device__ __forceinline__ void write_heads(const FieldParams& p, const Rows& R, int branch, float (&part)[2][4]) {
  const float* Pf = reinterpret_cast<const float*>(p.packed);
  const float* hb = Pf + (branch ? p.L.orgb_b : p.L.rgb_b);
  const float sb = __ldg(Pf + (branch ? p.L.osigma_b : p.L.sigma_b));
#pragma unroll
  for (int r = 0; r < 2; ++r) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      part[r][k] += __shfl_xor_sync(0xffffffffu, part[r][k], 1);
      part[r][k] += __shfl_xor_sync(0xffffffffu, part[r][k], 2);
    }
    if ((threadIdx.x & 3) == 0 && R.live[r]) {
      float sg = part[r][0] + sb;
      const float cr = 1.0f / (1.0f + __expf(-(part[r][1] + __ldg(hb + 0))));
      const float cg = 1.0f / (1.0f + __expf(-(part[r][2] + __ldg(hb + 1))));
      const float cb = 1.0f / (1.0f + __expf(-(part[r][3] + __ldg(hb + 2))));
      if (R.mute[r] & (branch ? 2 : 1)) sg = -1e5f;
      float* outp = branch ? p.obj_out : p.scene_out;
      reinterpret_cast<float4*>(outp)[(int64_t)R.ray[r] * p.out_stride + R.si[r]] = make_float4(cr, cg, cb, sg);
    }
  }
}

template <bool VOXEL, bool DUMP>
__global__ void __launch_bounds__(NUM_THREADS, 1) field_tc_kernel(const __grid_constant__ TcParams P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const FieldParams& p = P.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int X_ATOMS = VOXEL ? 6 : 1;
  constexpr int XS = VOXEL ? 9 : 2, XO = VOXEL ? 12 : 2;   // K slabs of X read by the scene / object branch (KX, KO)

  // ---- shared memory carve-up (base is 1024-byte aligned: required by the 128B swizzle) ----
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sX = sbase;
  const uint32_t sB = sX + X_ATOMS * ATOM_BYTES;
  const uint32_t sBias = sB + NSTAGE * STAGE_BYTES;                 // [G_COUNT][256] floats
  const uint32_t sMeta = sBias + G_COUNT * 256 * 4;                 // [128] RowMeta
  const uint32_t sBar = sMeta + TM * sizeof(RowMeta);
  uint8_t* gen_base = smem_raw + (sbase - smem_u32(smem_raw));
  float* bias_tab = reinterpret_cast<float*>(gen_base + (sBias - sbase));
  RowMeta* meta = reinterpret_cast<RowMeta*>(gen_base + (sMeta - sbase));
  const float* Pf = reinterpret_cast<const float*>(p.packed);
  Ring ring{sB, sBar, sBar + 8 * NSTAGE, 0u, 0u, P.diag};

  if (threadIdx.x == 0) ring_init_bars(ring.full, ring.empty);
  // per-column biases of every GEMM -> shared memory (layers with a per-ray constant read ray_const instead)
  for (int i = threadIdx.x; i < G_COUNT * 256; i += NUM_THREADS) {
    const int g = i >> 8, c = i & 255;
    bias_tab[i] = (c < p.L.g[g].N) ? __ldg(Pf + p.L.g[g].bias_off + c) : 0.0f;
  }
  __syncthreads();

  const int64_t total = (int64_t)p.n_rays * p.S;
  const int64_t n_tiles = (total + TM - 1) / TM;

  if (warp >= PRODUCER_WARP) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == PRODUCER_WARP)
      tc_producer_loop(P.layers, P.n_layers, reinterpret_cast<const uint8_t*>(p.packed), ring, n_tiles);
    return;
  }
  setmaxnreg_inc<CONSUMER_REGS>();

  // =============================== encode + MMA + epilogue warpgroups ===============================
  const int wg = warp >> 2, tid = threadIdx.x & 127;
  const uint32_t sXw = sX + (uint32_t)wg * 64u * 128u;
  Rows R;
  R.row[0] = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  R.row[1] = R.row[0] + 8;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    R.tile = tile;
    // ---- encode this warpgroup's 64 rows of X: (row, column quarter) jobs ----
#pragma unroll 1
    for (int job = tid; job < 256; job += 128) {
      const int row = wg * 64 + (job & 63), cq = job >> 6;
      const int64_t e = tile * TM + row;
      const bool live = e < total;
      const int ray = live ? (int)(e / p.S) : 0;
      const int si = live ? (int)(e - (int64_t)ray * p.S) : 0;
      const float* rr = p.rays + (int64_t)ray * 8;
      const float zz = live ? __ldg(p.z + (int64_t)ray * p.z_stride + si) : 0.0f;
      float x = fmaf(__ldg(rr + 3), zz, __ldg(rr + 0));
      float y = fmaf(__ldg(rr + 4), zz, __ldg(rr + 1));
      float z = fmaf(__ldg(rr + 5), zz, __ldg(rr + 2));
      if (p.xyz && live) {
        const float* qq = p.xyz + ((int64_t)ray * p.S + si) * 3;
        x = __ldg(qq); y = __ldg(qq + 1); z = __ldg(qq + 2);
      }
      if (!live) { x = 0.f; y = 0.f; z = 0.f; }
      if (cq == 0) {
        int mute = 0;
        if (live && p.mute_zero_rays && __ldg(p.z + (int64_t)ray * p.z_stride + (p.S - 1)) == 0.0f) mute = 3;
        if (live && mute == 0 && p.n_boxes > 0 && point_in_boxes(p.boxes, p.n_boxes, x, y, z)) mute = 1;
        meta[row] = RowMeta{ray, si, mute, live ? 1 : 0};
      }
      if (VOXEL) {
        const GridView g = load_grid_view(p.grid);
        float f[8];
        if (cq == 0) {
          voxel_trilinear<0, 8, false>(g, x, y, z, f);
          pe8_to_chunks(sX, row, 0, 2, f);        // scene channels 0-7 : chunks 0, 2, 4, ...
        } else if (cq == 1) {
          voxel_trilinear<8, 8, false>(g, x, y, z, f);
          pe8_to_chunks(sX, row, 1, 2, f);        // scene channels 8-15: chunks 1, 3, 5, ...
        } else if (cq == 2) {
          voxel_trilinear<16, 8, false>(g, x, y, z, f);
          pe8_to_chunks(sX, row, 34, 1, f);       // object voxel block starts at column 272 = chunk 34
        } else {
          pe_xyz_to_chunks(sX, row, 26, x, y, z); // columns 208..271
          st_chunk(a_chunk_addr(sX, row, 47), 0u, 0u, 0u, 0u);  // columns 376..383
        }
      } else {
        if (cq == 0) pe_xyz_to_chunks(sX, row, 0, x, y, z);
      }
    }
    fence_async_smem();
    wg_sync(wg);
    if (DUMP) {   // this warpgroup's rows of the X atoms, byte for byte
#pragma unroll 1
      for (int a = 0; a < X_ATOMS; ++a) {
        const uint4* src = reinterpret_cast<const uint4*>(gen_base + (size_t)a * ATOM_BYTES + (size_t)wg * 8192);
        uint4* dst = reinterpret_cast<uint4*>(P.dump + P.TL.act_off[0] + ((size_t)tile * X_ATOMS + a) * ATOM_BYTES + (size_t)wg * 8192);
        for (int i = tid; i < 512; i += 128) dst[i] = src[i];
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const RowMeta m = meta[R.row[r]];
      R.live[r] = m.live; R.ray[r] = m.ray; R.si[r] = m.si; R.mute[r] = m.mute;
      R.rc[r] = p.ray_const + (int64_t)m.ray * ONERF_RAY_CONST_FLOATS;
    }

    if (p.want_scene) {
      float acc[128];
      uint32_t h[64];
      float part[2][4] = {};
      const float* sw = Pf + p.L.sigma_w;
      mma_layer<256, XS, 0>(acc, h, sXw, ring);
      epilogue<256, EPI_HIDDEN>(acc, h, bias_tab + G_S0 * 256, R, 0, nullptr, part);
      if (DUMP) dump_layer<256>(P, R, 1, onerf_mask_word0(1), h);
#pragma unroll 1
      for (int l = 1; l < 4; ++l) {
        mma_layer<256, 0, 8>(acc, h, sXw, ring);
        epilogue<256, EPI_HIDDEN>(acc, h, bias_tab + (G_S0 + l) * 256, R, 0, nullptr, part);
        if (DUMP) dump_layer<256>(P, R, 1 + l, onerf_mask_word0(1 + l), h);
      }
      mma_layer<256, XS, 8>(acc, h, sXw, ring);   // skip layer: [X | h3]
      epilogue<256, EPI_HIDDEN>(acc, h, bias_tab + G_S4 * 256, R, 0, nullptr, part);
      if (DUMP) dump_layer<256>(P, R, 5, onerf_mask_word0(5), h);
#pragma unroll 1
      for (int l = 5; l < 7; ++l) {
        mma_layer<256, 0, 8>(acc, h, sXw, ring);
        epilogue<256, EPI_HIDDEN>(acc, h, bias_tab + (G_S0 + l) * 256, R, 0, nullptr, part);
        if (DUMP) dump_layer<256>(P, R, 1 + l, onerf_mask_word0(1 + l), h);
      }
      mma_layer<256, 0, 8>(acc, h, sXw, ring);
      epilogue<256, EPI_HIDDEN_SIGMA>(acc, h, bias_tab + G_S7 * 256, R, 0, sw, part);
      if (DUMP) dump_layer<256>(P, R, 8, onerf_mask_word0(8), h);
      mma_layer<256, 0, 8>(acc, h, sXw, ring);
      epilogue<256, EPI_FINAL>(acc, h, bias_tab + G_SFIN * 256, R, 0, nullptr, part);
      if (DUMP) dump_layer<256>(P, R, 9, -1, h);
      float accd[64];
      uint32_t hd[32];
      mma_layer<128, 0, 8>(accd, h, sXw, ring);
      epilogue<128, EPI_DIR>(accd, hd, nullptr, R, RC_SDIR, Pf + p.L.rgb_w, part);
      if (DUMP) dump_layer<128>(P, R, 10, onerf_mask_word0(10), hd);
      write_heads(p, R, 0, part);
    }
    if (p.want_object) {
      float acc[64];
      uint32_t h[32];
      float part[2][4] = {};
      mma_layer<128, XO, 0>(acc, h, sXw, ring);
      epilogue<128, EPI_HIDDEN_RC>(acc, h, nullptr, R, RC_OL0, nullptr, part);
      if (DUMP) dump_layer<128>(P, R, 11, onerf_mask_word0(11), h);
      mma_layer<128, 0, 4>(acc, h, sXw, ring);
      epilogue<128, EPI_HIDDEN>(acc, h, bias_tab + G_O1 * 256, R, 0, nullptr, part);
      if (DUMP) dump_layer<128>(P, R, 12, onerf_mask_word0(12), h);
      mma_layer<128, XO, 4>(acc, h, sXw, ring);   // [X | h1], object code through ray_const
      epilogue<128, EPI_HIDDEN_RC>(acc, h, nullptr, R, RC_OL2, nullptr, part);
      if (DUMP) dump_layer<128>(P, R, 13, onerf_mask_word0(13), h);
      mma_layer<128, 0, 4>(acc, h, sXw, ring);
      epilogue<128, EPI_HIDDEN_SIGMA>(acc, h, bias_tab + G_O3 * 256, R, 0, Pf + p.L.osigma_w, part);
      if (DUMP) dump_layer<128>(P, R, 14, onerf_mask_word0(14), h);
      mma_layer<128, 0, 4>(acc, h, sXw, ring);
      epilogue<128, EPI_FINAL>(acc, h, bias_tab + G_OFIN * 256, R, 0, nullptr, part);
      if (DUMP) dump_layer<128>(P, R, 15, -1, h);
      float accd[32];
      uint32_t hd[16];
      mma_layer<64, 0, 4>(accd, h, sXw, ring);
      epilogue<64, EPI_DIR>(accd, hd, nullptr, R, RC_ODIR, Pf + p.L.orgb_w, part);
      if (DUMP) dump_layer<64>(P, R, 16, onerf_mask_word0(16), hd);
      write_heads(p, R, 1, part);
    }
    // the next tile's encode overwrites X and the row metadata: both warpgroups' reads of them are done
    wg_sync(wg);
  }
}

}  // namespace

int onerf_launch_field_bf16(onerf_ctx* ctx, const FieldParams& fp, cudaStream_t stream) {
  const PackLayout& L = fp.L;
  TcParams P;
  memset(&P, 0, sizeof(P));
  P.f = fp;
  int n = 0;
  auto add = [&](int g) { P.layers[n++] = WLayer{L.g[g].img_off, L.g[g].N, L.g[g].K / 32}; };
  if (fp.want_scene)
    for (int g = G_S0; g <= G_SDIR; ++g) add(g);
  if (fp.want_object)
    for (int g = G_O0; g <= G_ODIR; ++g) add(g);
  P.n_layers = n;
  P.diag = ctx->tc_diag;
  const int64_t total = (int64_t)fp.n_rays * fp.S;
  const int64_t tiles = (total + TM - 1) / TM;
  if (fp.train_ws) {
    P.dump = reinterpret_cast<uint8_t*>(fp.train_ws);
    P.TL = onerf_make_train_layout(L.use_voxel, total);
  }
  const int blocks = (int)(tiles < ctx->num_sms ? tiles : ctx->num_sms);
  const int x_atoms = L.use_voxel ? 6 : 1;
  const size_t smem = 1024 + (size_t)x_atoms * ATOM_BYTES + NSTAGE * STAGE_BYTES + G_COUNT * 256 * 4 + TM * sizeof(RowMeta) +
                      16 * NSTAGE;
  auto launch = [&](auto kernel) -> int {
    ONERF_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<blocks, NUM_THREADS, smem, stream>>>(P);
    ONERF_LAUNCH_CHECK(ctx);
    return ONERF_OK;
  };
  if (L.use_voxel) return fp.train_ws ? launch(field_tc_kernel<true, true>) : launch(field_tc_kernel<true, false>);
  return fp.train_ws ? launch(field_tc_kernel<false, true>) : launch(field_tc_kernel<false, false>);
}
