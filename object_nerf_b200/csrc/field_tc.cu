// wgmma (Hopper tensor core) implementation of the fused encode + two-branch MLP for sm_90a.
//
// One persistent CTA per SM; a CTA owns one 128-sample tile at a time (tc_chain.cuh).
//   warpgroups 0 / 1 (256 thr)  run every layer on rows [0, 64) / [64, 128) of the tile, object branch first: wgmma
//                               M = 64 with the accumulator in registers, then the epilogue (bias / per-ray constant ->
//                               LeakyReLU -> bf16 pairs) leaves the output in registers as the NEXT layer's A operand.
//                               Hidden activations never touch shared or global memory.  Heads (sigma, rgb) are CUDA-core
//                               dot products on the fp32 values, reduced over the four lanes that share a row.
//   warpgroup 2                 its first warp streams the weights global -> shared with cp.async.bulk (pre-swizzled
//                               SWIZZLE_64B stage images written by pack.cu) through an mbarrier ring running ahead across
//                               layers and tiles; its other three warps (encoder_loop) encode the next tile into shared
//                               memory (X, bf16, K-major SWIZZLE_128B atoms) while the consumers run the layers after the
//                               last X-fed one.  The warpgroup hands most of its registers to warpgroups 0 / 1.
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
#include "prune.cuh"

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
#ifdef ONERF_FIELD_TIMELINE
  uint64_t* tl;     // phase stamps (below)
#endif
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
#ifdef ONERF_FIELD_TIMELINE
  uint64_t* tl;     // this warpgroup's stamp record of this tile, or null
#endif
};

__device__ __forceinline__ void fragment_rows(int (&row)[2], int warp, int lane) {
  row[0] = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
  row[1] = row[0] + 8;
}

#ifdef ONERF_FIELD_TIMELINE
// Phase timeline, built only by tools/field_timeline.py: lane 0 of each warpgroup stores clock64 stamps of the first
// TL_TILES tiles of CTAs [0, TL_CTAS) at tl[((cta * 3 + warpgroup) * TL_TILES + k) * TL_SLOTS + slot] (slot meanings in
// the tool).  The store is predicated inside one asm statement, so no branch lands between two wgmmas.
constexpr int TL_CTAS = 8, TL_TILES = 16, TL_SLOTS = 80;
uint64_t* g_timeline = nullptr;
__device__ __forceinline__ void tl_put(uint64_t* tl, int slot, uint64_t v) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u64 p, %0, 0;\n\t@p st.global.u64 [%1], %2;\n\t}" ::"l"(tl), "l"(tl + slot),
               "l"(v)
               : "memory");
}
__device__ __forceinline__ uint64_t* tl_record(const TcParams& P, int64_t tile, int wg, bool lead) {
  const int64_t k = (tile - blockIdx.x) / gridDim.x;
  if (!P.tl || !lead || blockIdx.x >= TL_CTAS || k >= TL_TILES) return nullptr;
  return P.tl + (((int64_t)blockIdx.x * 3 + wg) * TL_TILES + k) * TL_SLOTS;
}
#define TL_AT(tl, slot) tl_put((tl), (slot), clock64())
#define TL_PUT(tl, slot, v) tl_put((tl), (slot), (v))
#else
#define TL_AT(tl, slot)
#define TL_PUT(tl, slot, v)
#endif

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

// sum of the partial sums that the four lanes of a row hold (every lane gets it)
__device__ __forceinline__ float row_sum(float part) {
  part += __shfl_xor_sync(0xffffffffu, part, 1);
  part += __shfl_xor_sync(0xffffffffu, part, 2);
  return part;
}

// finish the heads of one branch: sum the four lanes of each row, add the head biases, write (rgb, sigma) to outp
__device__ __forceinline__ void write_heads(const FieldParams& p, const Rows& R, int branch, float (&part)[2][4],
                                            float* outp) {
  const float* Pf = reinterpret_cast<const float*>(p.packed);
  const float* hb = Pf + (branch ? p.L.orgb_b : p.L.rgb_b);
  const float sb = __ldg(Pf + (branch ? p.L.osigma_b : p.L.sigma_b));
#pragma unroll
  for (int r = 0; r < 2; ++r) {
#pragma unroll
    for (int k = 0; k < 4; ++k) part[r][k] = row_sum(part[r][k]);
    if ((threadIdx.x & 3) == 0 && R.live[r]) {
      float sg = part[r][0] + sb;
      const float cr = 1.0f / (1.0f + __expf(-(part[r][1] + __ldg(hb + 0))));
      const float cg = 1.0f / (1.0f + __expf(-(part[r][2] + __ldg(hb + 1))));
      const float cb = 1.0f / (1.0f + __expf(-(part[r][3] + __ldg(hb + 2))));
      if (R.mute[r] & (branch ? 2 : 1)) sg = -1e5f;
      reinterpret_cast<float4*>(outp)[(int64_t)R.ray[r] * p.out_stride + R.si[r]] = make_float4(cr, cg, cb, sg);
    }
  }
}

// consumers -> encoders: lane 0 of each consumer warp arrives on x_free when `on` (a predicate, not a branch)
__device__ __forceinline__ void x_release(uint32_t x_free, bool on) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, %1, 1;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}" ::"r"(x_free),
      "r"((uint32_t)on & (uint32_t)((threadIdx.x & 31) == 0))
      : "memory");
}

// One layer of one warpgroup: MMAs, epilogue, and in the training forward the dump of its output to activation slot
// `slot` (= GEMM index + 1) with its sign masks (mask_word0 >= 0).  An X-fed layer with free_x set hands X to the
// encoder warps once its MMAs have completed.
template <int N, int NX, int NH, int EPI, bool DUMP>
__device__ __forceinline__ void run_layer(const TcParams& P, const Rows& R, Ring& ring, uint32_t sXw, float (&acc)[N / 2],
                                          const uint32_t* hin, uint32_t* hout, const float* bias, int rc_base,
                                          const float* headw, float (&part)[2][4], int slot, int mask_word0,
                                          uint32_t x_free = 0, bool free_x = false) {
  TL_AT(R.tl, 3 * slot);
  mma_layer<N, NX, NH>(acc, hin, sXw, ring);
  if constexpr (NX > 0) x_release(x_free, free_x);
  TL_AT(R.tl, 3 * slot + 1);
#ifdef ONERF_FIELD_TIMELINE
  TL_PUT(R.tl, 55 + slot, ring.full_wait);
  ring.full_wait = 0;
#endif
  epilogue<N, EPI>(acc, hout, bias, R, rc_base, headw, part);
  if (DUMP) dump_layer<N>(P, R, slot, mask_word0, hout);
  TL_AT(R.tl, 3 * slot + 2);
}

// The scene branch up to its sigma head (models/nerf_model.py:97-112): layers S0..S7, XS K slabs of X into S0 and the
// skip layer.  Leaves S7's output in h and the sigma partial sums in part[r][0].
template <int XS, bool DUMP>
__device__ __forceinline__ void scene_trunk(const TcParams& P, const Rows& R, Ring& ring, uint32_t sXw, float (&acc)[128],
                                            uint32_t (&h)[64], const float* bias_tab, float (&part)[2][4],
                                            uint32_t x_free) {
  const float* sw = reinterpret_cast<const float*>(P.f.packed) + P.f.L.sigma_w;
  run_layer<256, XS, 0, EPI_HIDDEN, DUMP>(P, R, ring, sXw, acc, h, h, bias_tab + G_S0 * 256, 0, nullptr, part, 1,
                                          onerf_mask_word0(1), x_free, false);
#pragma unroll 1
  for (int l = 1; l < 4; ++l)
    run_layer<256, 0, 8, EPI_HIDDEN, DUMP>(P, R, ring, sXw, acc, h, h, bias_tab + (G_S0 + l) * 256, 0, nullptr, part,
                                           1 + l, onerf_mask_word0(1 + l));
  // skip layer [X | h3]: the last reader of X
  run_layer<256, XS, 8, EPI_HIDDEN, DUMP>(P, R, ring, sXw, acc, h, h, bias_tab + G_S4 * 256, 0, nullptr, part, 5,
                                          onerf_mask_word0(5), x_free, true);
#pragma unroll 1
  for (int l = 5; l < 7; ++l)
    run_layer<256, 0, 8, EPI_HIDDEN, DUMP>(P, R, ring, sXw, acc, h, h, bias_tab + (G_S0 + l) * 256, 0, nullptr, part,
                                           1 + l, onerf_mask_word0(1 + l));
  run_layer<256, 0, 8, EPI_HIDDEN_SIGMA, DUMP>(P, R, ring, sXw, acc, h, h, bias_tab + G_S7 * 256, 0, sw, part, 8,
                                               onerf_mask_word0(8));
}

// =============================== encoder warps (warps 1-3 of the producer warpgroup) ===============================
// They write X (bf16, K-major SWIZZLE_128B atoms) and the row metadata of tile t + gridDim.x while the consumers still
// run tile t: (row, column quarter) jobs, each gathering before it waits for X to be free, so the first job's loads
// overlap the consumers' last X-fed layer.  Hand-off through two CTA-local mbarriers:
//   x_full  encoders -> consumers: X and meta[] of the tile are written (one arrival per encoder thread, after
//           fence.proxy.async so that wgmma sees the stores)
//   x_free  consumers -> encoders: the last X-fed layer's MMAs have completed and meta[] has been read (one arrival
//           per consumer warp)
// Channel order and arithmetic are those of the in-line encode they replace, so X is bit for bit the same.
constexpr int NUM_ENCODER = 3 * 32;

__device__ __forceinline__ void prefetch_l2(const void* ptr) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr));
}

// L2 prefetch of the 128-byte lines [bytes0, bytes0 + nbytes) of rows [r0, r1] (row pitch `pitch` bytes) of `base`
__device__ __forceinline__ void prefetch_rows(const void* base, int64_t pitch, int64_t bytes0, int nbytes, int r0,
                                              int r1, int et) {
  const int lines = (nbytes + 127) >> 7;
  for (int i = et; i < (r1 - r0 + 1) * lines; i += NUM_ENCODER)
    prefetch_l2(reinterpret_cast<const char*>(base) + (r0 + i / lines) * pitch + bytes0 + (int64_t)(i % lines) * 128);
}

// Column quarter cq (0..3) of row `row` of a voxel-model tile, for the point (x, y, z).  Each quarter gathers before it
// waits for X to be free (`parity` of x_free), so the first job's loads overlap the consumers' last X-fed layer.
__device__ __forceinline__ void voxel_encode_job(const GridView& g, uint32_t sX, int row, int cq, float x, float y,
                                                 float z, uint32_t x_free, uint32_t parity, uint32_t* diag) {
  if (cq < 3) {
    float f[8];
    // scene channels 0-7: chunks 0, 2, 4, ...; 8-15: chunks 1, 3, 5, ...; object channels: chunk 34 (column 272) on
    if (cq == 0) voxel_trilinear<0, 8, false>(g, x, y, z, f);
    else if (cq == 1) voxel_trilinear<8, 8, false>(g, x, y, z, f);
    else voxel_trilinear<16, 8, false>(g, x, y, z, f);
    mbar_wait(x_free, parity, diag);
    pe8_to_chunks(sX, row, cq < 2 ? cq : 34, cq < 2 ? 2 : 1, f);
  } else if (cq == 3) {
    mbar_wait(x_free, parity, diag);
    pe_xyz_to_chunks(sX, row, 26, x, y, z);                     // columns 208..271
    st_chunk(a_chunk_addr(sX, row, 47), 0u, 0u, 0u, 0u);        // columns 376..383
  }
}

template <bool VOXEL>
__device__ __forceinline__ void encoder_loop(const TcParams& P, uint32_t sX, RowMeta* meta, uint32_t x_full,
                                             uint32_t x_free, int64_t n_tiles, int64_t total) {
  const FieldParams& p = P.f;
  const int et = threadIdx.x - NUM_CONSUMER - 32;
  constexpr int JOBS = VOXEL ? 4 * TM : TM;
  uint32_t it = 0;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
#ifdef ONERF_FIELD_TIMELINE
    uint64_t* tl = tl_record(P, tile, 2, et == 0);
#endif
    TL_AT(tl, 0);
    {  // rows the consumers' per-ray-constant epilogues read for this tile, and the next tile's rays and depths
      const int64_t e0 = tile * TM, e1 = min(e0 + TM, total) - 1;
      prefetch_rows(p.ray_const, ONERF_RAY_CONST_FLOATS * 4, 0, ONERF_RAY_CONST_FLOATS * 4, (int)(e0 / p.S),
                    (int)(e1 / p.S), et);
      const int64_t n0 = e0 + (int64_t)gridDim.x * TM, n1 = min(n0 + TM, total) - 1;
      if (n0 < total) {
        prefetch_rows(p.rays, 32, 0, 32, (int)(n0 / p.S), (int)(n1 / p.S), et);
        prefetch_rows(p.z, p.z_stride * 4, 0, p.S * 4, (int)(n0 / p.S), (int)(n1 / p.S), et);
      }
    }
#pragma unroll 1
    for (int job = et; job < JOBS; job += NUM_ENCODER) {
      const int row = job & (TM - 1), cq = job / TM;
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
        mbar_wait(x_free, (it & 1) ^ 1, P.diag);
        meta[row] = RowMeta{ray, si, mute, live ? 1 : 0};
      }
      if (VOXEL) {
        voxel_encode_job(load_grid_view(p.grid), sX, row, cq, x, y, z, x_free, (it & 1) ^ 1, P.diag);
      } else if (cq == 0) {
        mbar_wait(x_free, (it & 1) ^ 1, P.diag);
        pe_xyz_to_chunks(sX, row, 0, x, y, z);
      }
    }
    mbar_wait(x_free, (it & 1) ^ 1, P.diag);   // (a no-op after the first job: keeps one arrival per phase)
    TL_AT(tl, 1);
    fence_async_smem();
    mbar_arrive(x_full);
    TL_AT(tl, 2);
  }
}

// Dynamic shared memory of a CTA as offsets from its 1024-byte aligned base (the 128B swizzle of X needs the
// alignment): the X atoms at 0, the weight ring, [G_COUNT][256] bias floats, [TM] RowMeta where the kernel keeps row
// metadata, then the barriers (ring full[], empty[], x_full, x_free).  `bytes` is what a launch asks for.
struct FieldSmem {
  uint32_t sB, sBias, sMeta, sBar, x_full, x_free, bytes;
};
__host__ __device__ constexpr FieldSmem field_smem(int x_atoms, bool has_meta) {
  FieldSmem s{};
  s.sB = x_atoms * ATOM_BYTES;
  s.sBias = s.sB + NSTAGE * STAGE_BYTES;
  s.sMeta = s.sBias + G_COUNT * 256 * 4;
  s.sBar = s.sMeta + (has_meta ? TM * (uint32_t)sizeof(RowMeta) : 0u);
  s.x_full = s.sBar + 16 * NSTAGE;
  s.x_free = s.x_full + 8;
  s.bytes = 1024 + s.x_free + 8;
  return s;
}

// Every thread of the CTA, once: the barriers of plan S at base sX, the bias table, __syncthreads().  Returns the ring.
__device__ __forceinline__ Ring cta_prologue(const FieldSmem& S, const TcParams& P, uint32_t sX, float* bias_tab) {
  const FieldParams& p = P.f;
  const float* Pf = reinterpret_cast<const float*>(p.packed);
  Ring ring{sX + S.sB, sX + S.sBar, sX + S.sBar + 8 * NSTAGE, 0u, 0u, P.diag};
  if (threadIdx.x == 0) {
    mbar_init(sX + S.x_full, NUM_ENCODER);
    mbar_init(sX + S.x_free, NUM_CONSUMER / 32);
    ring_init_bars(ring.full, ring.empty);   // (its fence covers the two above)
  }
  // per-column biases of every GEMM -> shared memory (layers with a per-ray constant read ray_const instead)
  for (int i = threadIdx.x; i < G_COUNT * 256; i += NUM_THREADS) {
    const int g = i >> 8, c = i & 255;
    bias_tab[i] = (c < p.L.g[g].N) ? __ldg(Pf + p.L.g[g].bias_off + c) : 0.0f;
  }
  __syncthreads();
  return ring;
}

// The code loop of the multi-code instance (field_tc_multi_kernel): the object branch runs once per code c in [0, n),
// with that code's per-ray constants at ray_const + c * rc_stride and its outputs at obj_out + c * obj_stride (floats).
// Every code's block carries the same direction terms (RC_SDIR, RC_ODIR).  The single-code instances run {1, 0, 0}.
struct CodeLoop {
  int n;
  int64_t rc_stride, obj_stride;
};

// Body of the field kernels.  MULTI: the object branch once per code of `cl` on the tile's one encoding X, then the
// scene branch; X is released after S4, or after the last code's O2 in an object-only launch.
template <bool VOXEL, bool DUMP, bool MULTI>
__device__ __forceinline__ void field_tc_body(const TcParams& P, const CodeLoop& cl) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const FieldParams& p = P.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int X_ATOMS = VOXEL ? 6 : 1;
  constexpr int XS = VOXEL ? 9 : 2, XO = VOXEL ? 12 : 2;   // K slabs of X read by the scene / object branch (KX, KO)
  constexpr FieldSmem S = field_smem(X_ATOMS, true);
  const uint32_t sX = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (sX - smem_u32(smem_raw));
  float* bias_tab = reinterpret_cast<float*>(gen_base + S.sBias);
  RowMeta* meta = reinterpret_cast<RowMeta*>(gen_base + S.sMeta);
  const uint32_t x_full = sX + S.x_full, x_free = sX + S.x_free;
  const float* Pf = reinterpret_cast<const float*>(p.packed);
  Ring ring = cta_prologue(S, P, sX, bias_tab);

  const int64_t total = (int64_t)field_rays(p) * p.S;
  const int64_t n_tiles = (total + TM - 1) / TM;

  if (warp >= PRODUCER_WARP) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == PRODUCER_WARP) {
      // a multi-code program leads with the six object layers, streamed once per code
      if constexpr (MULTI)
        tc_producer_loop(P.layers, P.n_layers, reinterpret_cast<const uint8_t*>(p.packed), ring, n_tiles,
                         G_ODIR - G_O0 + 1, cl.n);
      else
        tc_producer_loop(P.layers, P.n_layers, reinterpret_cast<const uint8_t*>(p.packed), ring, n_tiles);
    } else
      encoder_loop<VOXEL>(P, sX, meta, x_full, x_free, n_tiles, total);
    return;
  }
  setmaxnreg_inc<CONSUMER_REGS>();

  // =============================== MMA + epilogue warpgroups ===============================
  // Object branch first, then scene: the last X-fed layer is then the scene skip layer S4 (O2 in an object-only
  // launch), and the encoders write the next tile's X during the layers after it.
  const int wg = warp >> 2, tid = threadIdx.x & 127;
  const uint32_t sXw = sX + (uint32_t)wg * 64u * 128u;
  const bool free_after_o2 = !p.want_scene;
  Rows R;
  fragment_rows(R.row, warp, lane);
  uint32_t it = 0;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    R.tile = tile;
#ifdef ONERF_FIELD_TIMELINE
    R.tl = tl_record(P, tile, wg, tid == 0);
#endif
    TL_AT(R.tl, 0);
    mbar_wait(x_full, it & 1, P.diag);
    TL_AT(R.tl, 1);
    if (DUMP) {   // this warpgroup's rows of the X atoms, byte for byte
#pragma unroll 1
      for (int a = 0; a < X_ATOMS; ++a) {
        const uint4* src = reinterpret_cast<const uint4*>(gen_base + (size_t)a * ATOM_BYTES + (size_t)wg * 8192);
        uint4* dst = reinterpret_cast<uint4*>(P.dump + P.TL.act_off[0] + ((size_t)tile * X_ATOMS + a) * ATOM_BYTES + (size_t)wg * 8192);
        for (int i = tid; i < 512; i += 128) dst[i] = src[i];
      }
    }
    // the row metadata is read before this warp releases X (x_free covers meta[] too)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const RowMeta m = meta[R.row[r]];
      R.live[r] = m.live; R.ray[r] = m.ray; R.si[r] = m.si; R.mute[r] = m.mute;
      R.rc[r] = p.ray_const + (int64_t)m.ray * ONERF_RAY_CONST_FLOATS;
    }
    TL_AT(R.tl, 2);

    if (p.want_object) {
      // one pass of the object branch per code (one in the single-code instances) on the tile's X
      const float* rc0[2] = {R.rc[0], R.rc[1]};
      for (int c = 0; c < (MULTI ? cl.n : 1); ++c) {
        if constexpr (MULTI) {
          R.rc[0] = rc0[0] + c * cl.rc_stride;
          R.rc[1] = rc0[1] + c * cl.rc_stride;
        }
        float acc[64];
        uint32_t h[32];
        float part[2][4] = {};
        run_layer<128, XO, 0, EPI_HIDDEN_RC, DUMP>(P, R, ring, sXw, acc, h, h, nullptr, RC_OL0, nullptr, part, 11,
                                                   onerf_mask_word0(11), x_free, false);
        run_layer<128, 0, 4, EPI_HIDDEN, DUMP>(P, R, ring, sXw, acc, h, h, bias_tab + G_O1 * 256, 0, nullptr, part, 12,
                                               onerf_mask_word0(12));
        // [X | h1], object code through ray_const
        run_layer<128, XO, 4, EPI_HIDDEN_RC, DUMP>(P, R, ring, sXw, acc, h, h, nullptr, RC_OL2, nullptr, part, 13,
                                                   onerf_mask_word0(13), x_free, MULTI ? free_after_o2 && c == cl.n - 1 : free_after_o2);
        run_layer<128, 0, 4, EPI_HIDDEN_SIGMA, DUMP>(P, R, ring, sXw, acc, h, h, bias_tab + G_O3 * 256, 0,
                                                     Pf + p.L.osigma_w, part, 14, onerf_mask_word0(14));
        run_layer<128, 0, 4, EPI_FINAL, DUMP>(P, R, ring, sXw, acc, h, h, bias_tab + G_OFIN * 256, 0, nullptr, part, 15, -1);
        float accd[32];
        uint32_t hd[16];
        run_layer<64, 0, 4, EPI_DIR, DUMP>(P, R, ring, sXw, accd, h, hd, nullptr, RC_ODIR, Pf + p.L.orgb_w, part, 16,
                                           onerf_mask_word0(16));
        write_heads(p, R, 1, part, MULTI ? p.obj_out + c * cl.obj_stride : p.obj_out);
      }
      if constexpr (MULTI) {
        R.rc[0] = rc0[0];
        R.rc[1] = rc0[1];
      }
    }
    if (p.want_scene) {
      float acc[128];
      uint32_t h[64];
      float part[2][4] = {};
      scene_trunk<XS, DUMP>(P, R, ring, sXw, acc, h, bias_tab, part, x_free);
      run_layer<256, 0, 8, EPI_FINAL, DUMP>(P, R, ring, sXw, acc, h, h, bias_tab + G_SFIN * 256, 0, nullptr, part, 9, -1);
      float accd[64];
      uint32_t hd[32];
      run_layer<128, 0, 8, EPI_DIR, DUMP>(P, R, ring, sXw, accd, h, hd, nullptr, RC_SDIR, Pf + p.L.rgb_w, part, 10,
                                          onerf_mask_word0(10));
      write_heads(p, R, 0, part, p.scene_out);
    }
    TL_AT(R.tl, 51);
    TL_AT(R.tl, 52);
  }
}

template <bool VOXEL, bool DUMP>
__global__ void __launch_bounds__(NUM_THREADS, 1) field_tc_kernel(const __grid_constant__ TcParams P) {
  field_tc_body<VOXEL, DUMP, false>(P, CodeLoop{1, 0, 0});
}

// Every object code of a render in one pass over the samples (onerf_render_instances): X is encoded once per tile and
// the object branch runs once per code.  Inference only.
struct MultiTcParams {
  TcParams t;
  CodeLoop codes;
};

template <bool VOXEL>
__global__ void __launch_bounds__(NUM_THREADS, 1) field_tc_multi_kernel(const __grid_constant__ MultiTcParams Q) {
  field_tc_body<VOXEL, false, true>(Q.t, Q.codes);
}

// =============================== pruning pass (sigma only, voxel model) ===============================
// EmbeddingVoxel.self_pruning_empty_voxels (reference models/embedding_helper.py:202-245) on the tensor cores: the
// samples are generated in the encoder warps (prune.cuh), only the scene branch's layers S0..S7 and the sigma head run,
// and each warp folds the alpha of its 16 rows into the voxel's maximum with one atomicMax.  A 128-row tile lies inside
// one voxel (4096 % 128 == 0): tile t of the launch is tiles [32 k, 32 k + 32) of voxel k = cell_begin + t / 32.
struct PruneTcParams {
  TcParams t;              // t.f: grid, packed, L; t.layers: G_S0..G_S7
  PruneSource src;
  int64_t cell_begin, n_cells;   // the shard [cell_begin, cell_begin + n_cells) of src.cells
  uint32_t* max_alpha;     // (n_cells,) float bits, zeroed by the caller
};
constexpr int kPruneTilesPerVoxel = kPruneSamples / TM;
static_assert(kPruneSamples % TM == 0, "a tile must lie inside one voxel");

// The encoder warps of the pruning pass: the points come from prune_point instead of rays and depths.  No row
// metadata: every row is live.
__device__ __forceinline__ void prune_encoder_loop(const PruneTcParams& Q, uint32_t sX, uint32_t x_full, uint32_t x_free,
                                                   int64_t n_tiles) {
  const int et = threadIdx.x - NUM_CONSUMER - 32;
  const GridView g = load_grid_view(Q.t.f.grid);
  uint32_t it = 0;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    const int64_t k = Q.cell_begin + tile / kPruneTilesPerVoxel;
    const int s0 = (int)(tile % kPruneTilesPerVoxel) * TM;
#pragma unroll 1
    for (int job = et; job < 4 * TM; job += NUM_ENCODER) {
      const int row = job & (TM - 1);
      float p[3];
      prune_point(Q.src, g, k, s0 + row, p);
      voxel_encode_job(g, sX, row, job / TM, p[0], p[1], p[2], x_free, (it & 1) ^ 1, Q.t.diag);
    }
    mbar_wait(x_free, (it & 1) ^ 1, Q.t.diag);
    fence_async_smem();
    mbar_arrive(x_full);
  }
}

__global__ void __launch_bounds__(NUM_THREADS, 1) prune_tc_kernel(const __grid_constant__ PruneTcParams Q) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const TcParams& P = Q.t;
  const FieldParams& p = P.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr FieldSmem S = field_smem(6, false);
  const uint32_t sX = (smem_u32(smem_raw) + 1023u) & ~1023u;
  float* bias_tab = reinterpret_cast<float*>(smem_raw + (sX - smem_u32(smem_raw)) + S.sBias);
  const uint32_t x_full = sX + S.x_full, x_free = sX + S.x_free;
  Ring ring = cta_prologue(S, P, sX, bias_tab);

  const int64_t n_tiles = Q.n_cells * kPruneTilesPerVoxel;
  if (warp >= PRODUCER_WARP) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == PRODUCER_WARP)
      tc_producer_loop(P.layers, P.n_layers, reinterpret_cast<const uint8_t*>(p.packed), ring, n_tiles);
    else
      prune_encoder_loop(Q, sX, x_full, x_free, n_tiles);
    return;
  }
  setmaxnreg_inc<CONSUMER_REGS>();

  const uint32_t sXw = sX + (uint32_t)(warp >> 2) * 64u * 128u;
  const float sb = __ldg(reinterpret_cast<const float*>(p.packed) + p.L.sigma_b);
  Rows R;   // scene_trunk without DUMP reads row and tile only (and tl): the per-ray fields stay unset
  fragment_rows(R.row, warp, lane);
#ifdef ONERF_FIELD_TIMELINE
  R.tl = nullptr;
#endif
  uint32_t it = 0;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    R.tile = tile;
    mbar_wait(x_full, it & 1, P.diag);
    float acc[128];
    uint32_t h[64];
    float part[2][4] = {};
    scene_trunk<9, false>(P, R, ring, sXw, acc, h, bias_tab, part, x_free);
    // the warp's largest alpha
    float m = 0.0f;
#pragma unroll
    for (int r = 0; r < 2; ++r) m = fmaxf(m, prune_alpha(row_sum(part[r][0]) + sb));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    // lane 0 folds it into the voxel's slot; the lane test is a predicate inside the asm statement (see ring_release)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.eq.u32 p, %2, 0;\n\t@p red.global.max.u32 [%0], %1;\n\t}" ::"l"(
                     Q.max_alpha + tile / kPruneTilesPerVoxel),
                 "r"(__float_as_uint(m)), "r"(lane)
                 : "memory");
  }
}

// appends GEMMs [g0, g1] of the packed layout to the producer program
void add_layers(TcParams& P, int g0, int g1) {
  for (int g = g0; g <= g1; ++g) P.layers[P.n_layers++] = WLayer{P.f.L.g[g].img_off, P.f.L.g[g].N, P.f.L.g[g].K / 32};
}

// persistent grid: one CTA per SM, or per tile where there are fewer
template <class Params>
int launch_persistent(onerf_ctx* ctx, void (*kernel)(Params), const Params& P, int64_t tiles, size_t smem,
                      cudaStream_t stream) {
  const int blocks = (int)(tiles < ctx->num_sms ? tiles : ctx->num_sms);
  ONERF_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<blocks, NUM_THREADS, smem, stream>>>(P);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

}  // namespace

int onerf_launch_field_bf16(onerf_ctx* ctx, const FieldParams& fp, cudaStream_t stream) {
  TcParams P;
  memset(&P, 0, sizeof(P));
  P.f = fp;
  if (fp.want_object) add_layers(P, G_O0, G_ODIR);
  if (fp.want_scene) add_layers(P, G_S0, G_SDIR);
  P.diag = ctx->tc_diag;
#ifdef ONERF_FIELD_TIMELINE
  P.tl = g_timeline;
#endif
  const bool voxel = fp.L.use_voxel, train = fp.train_ws != nullptr;
  const int64_t total = (int64_t)fp.n_rays * fp.S;
  if (train) {
    P.dump = reinterpret_cast<uint8_t*>(fp.train_ws);
    P.TL = onerf_make_train_layout(voxel, total);
  }
  auto* kernel = voxel ? (train ? field_tc_kernel<true, true> : field_tc_kernel<true, false>)
                       : (train ? field_tc_kernel<false, true> : field_tc_kernel<false, false>);
  return launch_persistent(ctx, kernel, P, (total + TM - 1) / TM, field_smem(voxel ? 6 : 1, true).bytes, stream);
}

int onerf_launch_field_bf16_codes(onerf_ctx* ctx, const FieldParams& fp, int n_codes, int64_t rc_stride,
                                  int64_t obj_stride, cudaStream_t stream) {
  ONERF_CHECK_ARG(fp.want_object && !fp.train_ws && n_codes >= 1, "a multi-code launch is an object-branch inference");
  MultiTcParams Q;
  memset(&Q, 0, sizeof(Q));
  Q.t.f = fp;
  add_layers(Q.t, G_O0, G_ODIR);
  if (fp.want_scene) add_layers(Q.t, G_S0, G_SDIR);
  Q.t.diag = ctx->tc_diag;
#ifdef ONERF_FIELD_TIMELINE
  Q.t.tl = g_timeline;
#endif
  Q.codes = CodeLoop{n_codes, rc_stride, obj_stride};
  const bool voxel = fp.L.use_voxel;
  const int64_t total = (int64_t)fp.n_rays * fp.S;
  return launch_persistent(ctx, voxel ? field_tc_multi_kernel<true> : field_tc_multi_kernel<false>, Q,
                           (total + TM - 1) / TM, field_smem(voxel ? 6 : 1, true).bytes, stream);
}

int onerf_launch_prune_bf16(onerf_ctx* ctx, const FieldParams& fp, const PruneSource& src, int64_t cell_begin,
                            int64_t n_cells, float* max_alpha, cudaStream_t stream) {
  PruneTcParams Q;
  memset(&Q, 0, sizeof(Q));
  Q.t.f = fp;
  add_layers(Q.t, G_S0, G_S7);
  Q.t.diag = ctx->tc_diag;
  Q.src = src;
  Q.cell_begin = cell_begin;
  Q.n_cells = n_cells;
  Q.max_alpha = reinterpret_cast<uint32_t*>(max_alpha);
  return launch_persistent(ctx, prune_tc_kernel, Q, n_cells * kPruneTilesPerVoxel,
                           field_smem(6, false).bytes, stream);
}

#ifdef ONERF_FIELD_TIMELINE
// device buffer of TL_CTAS * 3 * TL_TILES * TL_SLOTS uint64 stamps that later field launches fill; null = off
extern "C" void onerf_field_timeline(void* buf) { g_timeline = static_cast<uint64_t*>(buf); }
#endif
