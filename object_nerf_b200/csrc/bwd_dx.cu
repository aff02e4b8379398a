// Gradient w.r.t. the sparse-voxel feature table on wgmma tensor cores (SURVEY.md §8 row a14; autograd of
// models/embedding_helper.py:354-409 fed by the four layers that read the encoded input X):
//   dX[128 x 384] = [dZ_s0 | dZ_s4 | dZ_o0 | dZ_o2] (K = 768) . [W_s0 ; W_s4 ; W_o0 ; W_o2][:, X block]      (wgmma)
//   d f_c = dX[f_c] + sum_k 2^k ( cos(2^k f_c) dX[sin_k c] - sin(2^k f_c) dX[cos_k c] )                       (PE chain rule,
//           sin / cos taken from the X atoms the forward dumped)
//   table_grad[row_corner][c] += trilinear weight * d f_c                                                     (red.global.add)
// One persistent CTA per SM; per 128-sample tile the producer streams dZ atoms (K-major operand, straight from the
// workspace) and the matching transposed X-block weight images (layout.h: ximg_off) through a 4-stage ring, in two
// passes that keep the accumulator within the register file:
//   pass 0: dX columns [0, 256) (the scene voxel channels' PE block, 208 columns) from all 8 / 12 dZ atoms
//   pass 1: dX columns [256, 384) (the object voxel channels' PE block at 272) from the 4 object dZ atoms: the scene
//           layers carry zero weights there
// Warpgroups 0 / 1 own rows [0, 64) / [64, 128): wgmma, then the PE chain rule and the scatter on the register
// fragment (each thread holds whole channels: every PE column of a channel lands in the same lane).  Warp 8: producer.
#include "encode.cuh"
#include "field_common.cuh"
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int DX_STAGES = 4;
constexpr int DX_IMG_BYTES = ONERF_DX_N * 64;              // one 32-K image: 384 rows x 64 B
constexpr int DX_STAGE_BYTES = ATOM_BYTES + 2 * 256 * 64;  // dZ atom + two images' rows of one pass (48 KB)
constexpr int DX_THREADS = 288;

struct DxParams {
  const uint8_t* packed;
  int64_t ximg_off;
  const uint8_t* ws;
  TrainLayout TL;
  const float* rays;      // (N,8)
  const float* z;         // (N,S)
  int S;
  int64_t total;
  onerf_grid grid;
  float* table_grad;      // (n_rows, 24)
  int want_object;
  uint32_t* diag;         // mbarrier timeout record (onerf_ctx)
  const float* xyz;       // (total,3) explicit positions (XYZ instance); appended so the fields above keep their offsets
};

__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// operand atom qa of a tile: dZ slots 0 (S0), 4 (S4), 10 (O0), 12 (O2), four atoms each
__device__ __forceinline__ const uint8_t* dz_atom(const DxParams& P, int64_t tile, int qa) {
  const int slot = qa < 4 ? 0 : qa < 8 ? 4 : qa < 10 ? 10 : 12;
  const int atom = qa < 4 ? qa : qa < 8 ? qa - 4 : qa < 10 ? qa - 8 : qa - 10;
  return P.ws + P.TL.dz_off[slot] + ((size_t)tile * P.TL.dz_atoms[slot] + atom) * ATOM_BYTES;
}

// d f of the channel pair held by this thread: acc entries of column block j0 (the feature itself), the sin / cos
// blocks j0 + jstep (1 + 2 k) / j0 + jstep (2 + 2 k); sin / cos values from the dumped X row (atoms from xatom0 on)
template <int NACC>
__device__ __forceinline__ void pe_chain(const float (&acc)[NACC], int r, int j0, int jstep, const uint8_t* xrow, int xatom0,
                                         int swz, float& d0, float& d1) {
  const int q = threadIdx.x & 3;
  d0 = acc[4 * j0 + 2 * r];
  d1 = acc[4 * j0 + 2 * r + 1];
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const int js = j0 + jstep * (1 + 2 * k), jc = j0 + jstep * (2 + 2 * k);
    const uint32_t sn = __ldg(reinterpret_cast<const uint32_t*>(xrow + (size_t)(xatom0 + (js >> 3)) * ATOM_BYTES + (((js & 7) ^ swz) << 4) + q * 4));
    const uint32_t cs = __ldg(reinterpret_cast<const uint32_t*>(xrow + (size_t)(xatom0 + (jc >> 3)) * ATOM_BYTES + (((jc & 7) ^ swz) << 4) + q * 4));
    const float scale = (float)(1 << k);
    d0 += scale * (bf16_lo(cs) * acc[4 * js + 2 * r] - bf16_lo(sn) * acc[4 * jc + 2 * r]);
    d1 += scale * (bf16_hi(cs) * acc[4 * js + 2 * r + 1] - bf16_hi(sn) * acc[4 * jc + 2 * r + 1]);
  }
}

// trilinear scatter of NP channel pairs (d[2 p], d[2 p + 1] into table channels ch[p], ch[p] + 1) of sample e, whose
// position is o + d z of its ray (the forward's fmaf) or, with XYZ, row e of P.xyz
template <bool XYZ, int NP>
__device__ __forceinline__ void scatter(const DxParams& P, const GridView& g, int64_t e, const int* ch, const float* d) {
  float x, y, z;
  if (XYZ) {
    const float* q = P.xyz + e * 3;
    x = __ldg(q); y = __ldg(q + 1); z = __ldg(q + 2);
  } else {
    const int ray = (int)(e / P.S), si = (int)(e - (int64_t)ray * P.S);
    const float* rr = P.rays + (int64_t)ray * 8;
    const float zz = __ldg(P.z + (int64_t)ray * P.S + si);
    x = fmaf(__ldg(rr + 3), zz, __ldg(rr + 0)); y = fmaf(__ldg(rr + 4), zz, __ldg(rr + 1));
    z = fmaf(__ldg(rr + 5), zz, __ldg(rr + 2));
  }
  const float px = __fdiv_rn(__fadd_rn(x, g.off[0]), g.vsize), py = __fdiv_rn(__fadd_rn(y, g.off[1]), g.vsize),
              pz = __fdiv_rn(__fadd_rn(z, g.off[2]), g.vsize);
  const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
  const float u = px - fx, v = py - fy, w = pz - fz;
  const bool any = (fx >= -1.0f) && (fy >= -1.0f) && (fz >= -1.0f) && (fx < (float)g.sx) && (fy < (float)g.sy) && (fz < (float)g.sz);
  if (!any) return;
  const int qx = (int)fx, qy = (int)fy, qz = (int)fz;
#pragma unroll 1
  for (int corner = 0; corner < 8; ++corner) {
    const int cx = (corner >> 2) & 1, cy = (corner >> 1) & 1, cz = corner & 1;
    const int ix = qx + cx, iy = qy + cy, iz = qz + cz;
    if (ix < 0 || iy < 0 || iz < 0 || ix >= g.sx || iy >= g.sy || iz >= g.sz) continue;
    const long long trow = __ldg(g.idx_map + ((int64_t)ix * g.sy + iy) * g.sz + iz);
    if (trow < 0) continue;
    const float wt = (cx ? u : 1.0f - u) * (cy ? v : 1.0f - v) * (cz ? w : 1.0f - w);
#pragma unroll
    for (int p = 0; p < NP; ++p) red_add_v2(P.table_grad + trow * 24 + ch[p], wt * d[2 * p], wt * d[2 * p + 1]);
  }
}

template <bool XYZ>
__global__ void __launch_bounds__(DX_THREADS, 1) bwd_dx_kernel(const __grid_constant__ DxParams P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sStage = sbase;
  const uint32_t sBar = sStage + DX_STAGES * DX_STAGE_BYTES;
  const uint32_t bar_full = sBar, bar_empty = sBar + 8 * DX_STAGES;
  if (threadIdx.x == 0) {
    for (int s = 0; s < DX_STAGES; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 8);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int64_t n_tiles = (P.total + TM - 1) / TM;
  // pass 0 reads dZ atoms [0, n_src), pass 1 atoms [8, 12)
  const int n_src = P.want_object ? 12 : 8;
  uint32_t stage = 0, phase = 0;

  if (warp == 8) {
    // =============================== producer ===============================
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      for (int pass = 0; pass < (P.want_object ? 2 : 1); ++pass) {
        const uint32_t rows_off = pass ? 256u * 64u : 0u, rows_bytes = pass ? 128u * 64u : 256u * 64u;
        for (int qa = pass ? 8 : 0; qa < (pass ? 12 : n_src); ++qa) {
          mbar_wait(bar_empty + 8 * stage, phase ^ 1, P.diag);
          if (elect_one()) {
            mbar_expect_tx(bar_full + 8 * stage, ATOM_BYTES + 2 * rows_bytes);
            const uint32_t dst = sStage + stage * DX_STAGE_BYTES;
            tma_bulk_g2s(dst, dz_atom(P, tile, qa), ATOM_BYTES, bar_full + 8 * stage);
            for (int i = 0; i < 2; ++i)
              tma_bulk_g2s(dst + ATOM_BYTES + i * rows_bytes, P.packed + P.ximg_off + (size_t)(2 * qa + i) * DX_IMG_BYTES + rows_off,
                           rows_bytes, bar_full + 8 * stage);
          }
          __syncwarp();
          if (++stage == DX_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // =============================== consumers ===============================
  const int wg = warp >> 2, q = lane & 3;
  const GridView g = load_grid_view(P.grid);
  int row[2];
  row[0] = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  row[1] = row[0] + 8;
  float acc[128];
  // one pass: acc[64 x 64 NB] = sum over dZ atoms [qa0, qa1) of atom . image rows
  auto run_pass = [&](int qa0, int qa1, auto nb_tag) {
    constexpr int NB = decltype(nb_tag)::value;
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.0f;
    uint32_t prev = 0;
    for (int qa = qa0; qa < qa1; ++qa) {
      mbar_wait(bar_full + 8 * stage, phase, P.diag);
      const uint32_t sa = sStage + stage * DX_STAGE_BYTES + (uint32_t)wg * 8192u, sb = sStage + stage * DX_STAGE_BYTES + ATOM_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k16 = 0; k16 < 4; ++k16) {
        const uint64_t ad = desc_k_sw128(sa + (uint32_t)k16 * 32u);
#pragma unroll
        for (int nb = 0; nb < NB; ++nb)
          wgmma_ss_n64<0, 0>(acc + 32 * nb, ad,
                             desc_k_sw64(sb + (uint32_t)(k16 >> 1) * (uint32_t)(NB * 64 * 64) + (uint32_t)nb * 4096u + (uint32_t)(k16 & 1) * 32u));
      }
      wgmma_commit();
      if (qa > qa0) {
        wgmma_wait<1>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
      }
      prev = stage;
      if (++stage == DX_STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
    fence_regs<128>(acc);
  };

  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const uint8_t* xtile = P.ws + P.TL.act_off[0] + ((size_t)tile * P.TL.act_atoms[0]) * ATOM_BYTES;
    // pass 0: scene channels.  Column 16 b + ch of X is PE block b of scene channel ch: this thread holds channels
    // 2 q, 2 q + 1 (column blocks j = 2 b) and 8 + 2 q, 9 + 2 q (j = 2 b + 1) of all 13 blocks
    run_pass(0, n_src, std::integral_constant<int, 4>());
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int64_t e = tile * TM + row[r];
      const uint8_t* xrow = xtile + (size_t)row[r] * 128;
      float d[4];
      pe_chain(acc, r, 0, 2, xrow, 0, row[r] & 7, d[0], d[1]);
      pe_chain(acc, r, 1, 2, xrow, 0, row[r] & 7, d[2], d[3]);
      const int ch[2] = {2 * q, 8 + 2 * q};
      if (e < P.total) scatter<XYZ, 2>(P, g, e, ch, d);
    }
    if (!P.want_object) continue;
    // pass 1: object channels.  Column 272 + 8 b + c = local column 16 + 8 b + c: channels 2 q, 2 q + 1, block j = 2 + b
    run_pass(8, 12, std::integral_constant<int, 2>());
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int64_t e = tile * TM + row[r];
      const uint8_t* xrow = xtile + (size_t)row[r] * 128;
      float d[2];
      pe_chain(acc, r, 2, 1, xrow, 4, row[r] & 7, d[0], d[1]);
      const int ch[1] = {16 + 2 * q};
      if (e < P.total) scatter<XYZ, 1>(P, g, e, ch, d);
    }
  }
}

}  // namespace

// xyz != NULL: sample e sits at xyz[3 e] (rays / z unused)
int onerf_launch_bwd_dx(onerf_ctx* ctx, int want_object, const void* packed, const void* ws, int64_t n_samples,
                        const float* rays, const float* z, int n_samples_per_ray, const float* xyz, const onerf_grid* grid,
                        float* table_grad, cudaStream_t stream) {
  DxParams P;
  memset(&P, 0, sizeof(P));
  P.diag = ctx->tc_diag;
  const PackLayout L = onerf_make_layout(1);
  P.packed = reinterpret_cast<const uint8_t*>(packed);
  P.ximg_off = L.ximg_off;
  P.ws = reinterpret_cast<const uint8_t*>(ws);
  P.TL = onerf_make_train_layout(1, n_samples);
  P.rays = rays; P.z = z; P.S = n_samples_per_ray; P.total = n_samples; P.xyz = xyz;
  P.grid = *grid;
  P.table_grad = table_grad;
  P.want_object = want_object;
  const int64_t tiles = (n_samples + TM - 1) / TM;
  const int blocks = (int)(tiles < ctx->num_sms ? tiles : ctx->num_sms);
  const size_t smem = 1024 + DX_STAGES * DX_STAGE_BYTES + 256;
  const auto kernel = xyz ? bwd_dx_kernel<true> : bwd_dx_kernel<false>;
  ONERF_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<blocks, DX_THREADS, smem, stream>>>(P);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
