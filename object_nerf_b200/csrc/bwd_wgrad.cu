// Weight-gradient GEMMs of the two-branch MLP on wgmma tensor cores (SURVEY.md §8 row a14; what autograd does for
// every nn.Linear of models/nerf_model.py:97-152:  dW_l += dZ_l^T . In_l, reduction over ALL samples).
//
// Operands are the bf16 "atoms" the training forward and the input-gradient chain leave in the training workspace
// (layout.h: [128 samples x 64 columns] SWIZZLE_128B images).  For this GEMM the reduction (K) dimension is the
// SAMPLE axis, so both operands are MN-major (transposed) wgmma operands: the very same atom image that the chain
// consumed K-major.
//   D[M = outputs of layer l  x  N = inputs of layer l] += A[M x K] . B[N x K]^T,  K = samples
//   A: dZ atoms (64 output columns each), B: activation atoms (64 input columns each)
// One persistent CTA per SM.  The (layer, 128-output block, input column block) work items are laid end to end, each
// weighted by the bytes it streams per 64-sample stage (the kernel is HBM-bound), and the byte axis is cut into
// gridDim.x equal pieces: a CTA owns one contiguous piece = a few (item, stage range) segments.  Per segment each of the
// two consumer warpgroups accumulates 64 outputs x up to 256 inputs in registers and flushes them once with vector
// reductions (red.global.add.v2.f32) into the kernel-layout gradient buffer (layout.h: GradLayout).
//   warp 8: producer (cp.async.bulk, 4-stage ring of 64-sample stages)
//   warpgroups 0 / 1: wgmma on dZ atom 0 / 1 of the item; while the ring streams, the first warp of each also forms the
//   bias gradients db_l = sum_s dZ_l from the dZ tiles that are passing through shared memory anyway (first column
//   block of every layer)
#include "common.cuh"
#include "layout.h"
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int WG_STAGES = 4;
constexpr int HALF_ATOM = 8192;                 // 64 samples x 128 B
constexpr int WG_STAGE_BYTES = 6 * HALF_ATOM;   // 2 A half-atoms + up to 4 B half-atoms
constexpr int WG_THREADS = 288;
constexpr int WG_MAX_ITEMS = 40;

struct WgItem {
  int64_t a_off;      // byte offset of the A slot (dZ) in the workspace
  int64_t b_off;      // byte offset of the B slot (activations)
  int a_atoms_slot;   // atoms per tile of the A slot
  int b_atoms_slot;
  int a_atom0;        // M block: atoms a_atom0, a_atom0 + 1 (128 outputs)
  int b_atom0, b_atoms;   // N block: 1..4 atoms
  int64_t out_off;    // float offset of D[0][0] in the gradient buffer
  int out_ld;
  int m_valid, n_valid;   // outputs of the layer, valid input columns of the block
  int cost;           // 2 + b_atoms (8 KB units per stage)
  int64_t db_off;     // float offset of the layer's bias gradient, or -1: this item does not form it
};

struct WgParams {
  const uint8_t* ws;
  float* grad;
  int n_stages;       // 64-sample stages = 2 * tiles
  int n_items;
  uint32_t* diag;     // mbarrier timeout record (onerf_ctx)
  WgItem items[WG_MAX_ITEMS];
};

__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// segment s of this CTA: item index and stage range; returns false when there is no further segment
struct Segment {
  int item, s0, s1;
};
__device__ __forceinline__ bool next_segment(const WgParams& P, int64_t lo, int64_t hi, int& item, int64_t& item_start, Segment& seg) {
  while (item < P.n_items) {
    const int64_t c = P.items[item].cost;
    const int64_t item_end = item_start + c * P.n_stages;
    if (item_end > lo && item_start < hi) {
      const int64_t a = lo > item_start ? lo - item_start : 0, b = (hi < item_end ? hi : item_end) - item_start;
      seg.item = item;
      seg.s0 = (int)((a + c - 1) / c);
      seg.s1 = (int)((b + c - 1) / c);
      const bool last_of_item = hi >= item_end;
      if (last_of_item) { ++item; item_start = item_end; }
      else { item = P.n_items; }   // the CTA's range ends inside this item
      if (seg.s1 > seg.s0) return true;
      continue;
    }
    if (item_start >= hi) return false;
    ++item;
    item_start = item_end;
  }
  return false;
}

__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_kernel(const __grid_constant__ WgParams P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sStage = sbase;
  const uint32_t sBar = sStage + WG_STAGES * WG_STAGE_BYTES;
  const uint32_t bar_full = sBar, bar_empty = sBar + 8 * WG_STAGES;

  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 8);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  // this CTA's piece of the byte axis
  int64_t total = 0;
  for (int i = 0; i < P.n_items; ++i) total += (int64_t)P.items[i].cost * P.n_stages;
  const int64_t lo = total * blockIdx.x / gridDim.x, hi = total * (blockIdx.x + 1) / gridDim.x;
  int item = 0;
  int64_t item_start = 0;
  Segment seg;
  uint32_t stage = 0, phase = 0;

  if (warp == 8) {
    // =============================== producer ===============================
    while (next_segment(P, lo, hi, item, item_start, seg)) {
      const WgItem& it = P.items[seg.item];
      for (int s = seg.s0; s < seg.s1; ++s) {
        const int tile = s >> 1, half = s & 1;
        mbar_wait(bar_empty + 8 * stage, phase ^ 1, P.diag);
        if (elect_one()) {
          mbar_expect_tx(bar_full + 8 * stage, (uint32_t)(2 + it.b_atoms) * HALF_ATOM);
          const uint32_t dst = sStage + stage * WG_STAGE_BYTES;
          const uint8_t* a = P.ws + it.a_off + ((size_t)tile * it.a_atoms_slot + it.a_atom0) * ATOM_BYTES + (size_t)half * HALF_ATOM;
          for (int i = 0; i < 2; ++i)
            tma_bulk_g2s(dst + i * HALF_ATOM, a + (size_t)i * ATOM_BYTES, HALF_ATOM, bar_full + 8 * stage);
          const uint8_t* b = P.ws + it.b_off + ((size_t)tile * it.b_atoms_slot + it.b_atom0) * ATOM_BYTES + (size_t)half * HALF_ATOM;
          for (int i = 0; i < it.b_atoms; ++i)
            tma_bulk_g2s(dst + (2 + i) * HALF_ATOM, b + (size_t)i * ATOM_BYTES, HALF_ATOM, bar_full + 8 * stage);
        }
        __syncwarp();
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // =============================== consumers: wgmma + bias gradients + flush ===============================
  const int wg = warp >> 2, wi = warp & 3, q = lane & 3;
  while (next_segment(P, lo, hi, item, item_start, seg)) {
    const WgItem& it = P.items[seg.item];
    const int nb = it.b_atoms;
    // the first warp of a warpgroup owns dZ columns 2 lane, 2 lane + 1 of its atom: word `lane` of every sample row
    const bool cs = it.db_off >= 0 && wi == 0;
    float c0 = 0.0f, c1 = 0.0f;
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.0f;
    uint32_t prev = 0;
    for (int s = seg.s0; s < seg.s1; ++s) {
      mbar_wait(bar_full + 8 * stage, phase, P.diag);
      const uint32_t sa = sStage + stage * WG_STAGE_BYTES + (uint32_t)wg * HALF_ATOM, sb = sStage + stage * WG_STAGE_BYTES + 2 * HALF_ATOM;
      wgmma_fence();
#pragma unroll
      for (int k16 = 0; k16 < 4; ++k16) {
        const uint64_t ad = desc_mn_sw128(sa + (uint32_t)k16 * 2048u, HALF_ATOM);
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (i < nb) wgmma_ss_n64<1, 1>(acc + 32 * i, ad, desc_mn_sw128(sb + (uint32_t)i * HALF_ATOM + (uint32_t)k16 * 2048u, HALF_ATOM));
      }
      wgmma_commit();
      if (cs) {
        const uint32_t base = sa + (uint32_t)(lane & 3) * 4u;
#pragma unroll 8
        for (int r = 0; r < 64; ++r) {
          uint32_t w;
          asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(base + (uint32_t)r * 128u + ((((uint32_t)lane >> 2) ^ ((uint32_t)r & 7u)) << 4)));
          c0 += bf16_lo(w);
          c1 += bf16_hi(w);
        }
      }
      if (s > seg.s0) {   // the previous stage's MMAs have completed
        wgmma_wait<1>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
      }
      prev = stage;
      if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
    fence_regs<128>(acc);
    const int m0 = (it.a_atom0 + wg) * 64;
    if (cs && m0 + 2 * lane < it.m_valid) {
      atomicAdd(P.grad + it.db_off + m0 + 2 * lane, c0);
      atomicAdd(P.grad + it.db_off + m0 + 2 * lane + 1, c1);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int m = m0 + wi * 16 + (lane >> 2) + 8 * r;
      if (m >= it.m_valid) continue;
      float* out = P.grad + it.out_off + (int64_t)m * it.out_ld;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i < nb) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = 64 * i + 8 * j + 2 * q;
            if (c < it.n_valid) red_add_v2(out + c, acc[32 * i + 4 * j + 2 * r], acc[32 * i + 4 * j + 2 * r + 1]);
          }
        }
      }
    }
  }
}

}  // namespace

// Item list of one model.  dZ slot d belongs to GEMM layer gemm_of[d]; its inputs are activation slots in kernel-K order.
int onerf_launch_wgrad(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int64_t n_samples, float* grad,
                       cudaStream_t stream) {
  const PackLayout L = onerf_make_layout(use_voxel);
  const GradLayout G = onerf_make_grad_layout(use_voxel);
  const TrainLayout T = onerf_make_train_layout(use_voxel, n_samples);
  WgParams P;
  memset(&P, 0, sizeof(P));
  P.diag = ctx->tc_diag;
  P.ws = reinterpret_cast<const uint8_t*>(ws);
  P.grad = grad;
  P.n_stages = 2 * T.n_tiles;
  // dZ slot -> GEMM layer
  const int gemm_of[ONERF_DZ_SLOTS] = {G_S0, G_S1, G_S2, G_S3, G_S4, G_S5, G_S6, G_S7, G_SFIN, G_SDIR,
                                       G_O0, G_O1, G_O2, G_O3, G_OFIN, G_ODIR};
  int n = 0;
  bool db_done[ONERF_DZ_SLOTS][2] = {};
  // input blocks of a layer: (activation slot, first atom, atoms, first kernel-K column, valid columns); one item per
  // 128 outputs
  auto add = [&](int dz, int act, int b_atom0, int b_atoms, int col0, int n_valid) {
    const int g = gemm_of[dz];
    const int out_n = L.g[g].N;                 // 256 / 128 / 64
    for (int mb = 0; mb < (out_n + 127) / 128; ++mb) {
      WgItem& it = P.items[n++];
      it.a_off = T.dz_off[dz]; it.a_atoms_slot = T.dz_atoms[dz];
      it.b_off = T.act_off[act]; it.b_atoms_slot = T.act_atoms[act];
      it.a_atom0 = 2 * mb;   // the 64-wide object dir layer reads one atom past its slot
      it.b_atom0 = b_atom0; it.b_atoms = b_atoms;
      it.out_off = G.w_off[g] + col0; it.out_ld = L.g[g].K;
      it.m_valid = out_n; it.n_valid = n_valid;
      it.cost = 2 + it.b_atoms;
      it.db_off = db_done[dz][mb] ? -1 : G.b_off[g];   // the first column block of a layer also forms its bias gradient
      db_done[dz][mb] = true;
    }
  };
  const int xa = use_voxel ? 4 : 1;             // leading X atoms (256 / 64 columns)
  auto x_blocks = [&](int dz, int kx) {         // X[0, kx)
    add(dz, 0, 0, xa, 0, use_voxel ? 256 : 64);
    if (use_voxel) add(dz, 0, 4, (kx - 256 + 63) / 64, 256, kx - 256);
  };
  x_blocks(0, L.KX);
  for (int l = 1; l < 8; ++l) {
    if (l == 4) x_blocks(4, L.KX);
    add(l, l, 0, 4, l == 4 ? L.KX : 0, 256);   // hidden input = output of layer l - 1 = activation slot l
  }
  add(8, 8, 0, 4, 0, 256);      // final: input = hidden 8
  add(9, 9, 0, 4, 0, 256);      // dir: input = final (the 27 direction columns are per-ray constants)
  if (want_object) {
    x_blocks(10, L.KO);
    add(11, 11, 0, 2, 0, 128);
    x_blocks(12, L.KO);
    add(12, 12, 0, 2, L.KO, 128);
    add(13, 13, 0, 2, 0, 128);
    add(14, 14, 0, 2, 0, 128);   // object final: input = object hidden 4
    add(15, 15, 0, 2, 0, 128);   // object dir: input = object final
  }
  P.n_items = n;
  const size_t smem = 1024 + WG_STAGES * WG_STAGE_BYTES + 256;
  ONERF_CUDA(cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  wgrad_kernel<<<ctx->num_sms, WG_THREADS, smem, stream>>>(P);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
