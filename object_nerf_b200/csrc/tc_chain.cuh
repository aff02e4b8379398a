// Layer-chain machinery shared by the fused forward (field_tc.cu) and the input-gradient chain (bwd_chain.cu):
// a persistent CTA walks a static list of GEMM "layers" per 128-row tile.
//   warp PRODUCER_WARP streams the layers' weight stage images into a shared-memory ring with cp.async.bulk;
//   warpgroups 0 and 1 own rows [0, 64) and [64, 128) of the tile and issue wgmma (M = 64) on them: A from shared-memory
//   X atoms (K-major SWIZZLE_128B) or from registers (the previous layer's packed output), B from the ring (K-major
//   SWIZZLE_64B stage images, layout.h).  Accumulators and hidden activations never leave the registers.
// Barrier protocol (CTA-local mbarriers):
//   full[s]   producer -> consumers: ring stage s filled (transaction bytes)
//   empty[s]  consumers -> producer: the MMAs that read stage s have completed (one arrival per consumer warp)
// The producer and the consumers walk the same stage sequence: per layer, its 32-wide K slabs in order, 256 / N slabs
// (16 KB) per stage.
#pragma once
#include "tc_common.cuh"

namespace tc {

constexpr int NSTAGE = 6;            // weight ring depth
constexpr int STAGE_BYTES = 16384;   // 32 K-slab rows of N = 256, or 2 / 4 slabs of N = 128 / 64
constexpr int NUM_WG = 2;
constexpr int NUM_CONSUMER = NUM_WG * 128;
// first warp of the third warpgroup; its other three warps encode X in the forward (field_tc.cu) and exit in bwd_chain
constexpr int PRODUCER_WARP = NUM_CONSUMER / 32;
constexpr int NUM_THREADS = NUM_CONSUMER + 128;
// Register split: a 64 x 256 fp32 accumulator plus the 256-wide register A operand need more than the 168 registers a
// 384-thread CTA gets per thread, so the producer warpgroup hands registers to the two consumer warpgroups
// (40 x 128 + 232 x 256 = 64 512 <= 65 536).
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr int MAX_LAYERS = 16;

struct WLayer {
  int64_t img_off;   // byte offset of the layer's stage images in the packed blob (nslab images of N * 64 bytes)
  int N;             // outputs: 256, 128 or 64
  int nslab;         // 32-wide K slabs
};

struct Ring {
  uint32_t sB, full, empty;
  uint32_t stage, phase;
  uint32_t* diag;   // timeout record of mbar_wait (onerf_ctx)
#ifdef ONERF_FIELD_TIMELINE
  uint64_t full_wait = 0;   // cycles spent waiting on full barriers since the last reset (tools/field_timeline.py)
#endif
};

__device__ __forceinline__ void ring_init_bars(uint32_t full, uint32_t empty) {
  for (int s = 0; s < NSTAGE; ++s) {
    mbar_init(full + 8 * s, 1);
    mbar_init(empty + 8 * s, NUM_CONSUMER / 32);
  }
  fence_barrier_init();
}

// =============================== weight producer (bulk copies) ===============================
// The whole warp runs the (uniform) loop; one elected lane talks to the barriers.  Per tile the program is layers
// [0, lead) lead_repeat times, then the rest of the list (the multi-code field kernel repeats its object layers once
// per code; MAX_LAYERS leaves no room to list them again).
__device__ __forceinline__ void tc_producer_loop(const WLayer* layers, int n_layers, const uint8_t* blob, Ring r,
                                                 int64_t n_tiles, int lead = 0, int lead_repeat = 1) {
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    for (int l = 0, rep = 1; l < n_layers; ++l) {
      const WLayer& Ly = layers[l];
      const int spp = 256 / Ly.N;
      const uint32_t slab_bytes = (uint32_t)Ly.N * 64u;
      for (int s0 = 0; s0 < Ly.nslab; s0 += spp) {
        const int cnt = (Ly.nslab - s0 < spp) ? Ly.nslab - s0 : spp;
        mbar_wait(r.empty + 8 * r.stage, r.phase ^ 1, r.diag);
        if (elect_one()) {
          mbar_expect_tx(r.full + 8 * r.stage, (uint32_t)cnt * slab_bytes);
          tma_bulk_g2s(r.sB + r.stage * STAGE_BYTES, blob + Ly.img_off + (size_t)s0 * slab_bytes, (uint32_t)cnt * slab_bytes,
                       r.full + 8 * r.stage);
        }
        __syncwarp();
        if (++r.stage == NSTAGE) { r.stage = 0; r.phase ^= 1; }
      }
      if (rep < lead_repeat && l == lead - 1) {   // the leading group again, from layer 0
        ++rep;
        l = -1;
      }
    }
  }
}

// One arrival per consumer warp, from lane 0.  The lane test is a predicate inside the asm statement, not a branch:
// a divergent path between two wgmmas makes ptxas serialise every wgmma of the kernel.  wgmma.wait_group is
// warp-synchronous, so when lane 0 arrives the whole warp has seen its MMAs complete.
__device__ __forceinline__ void ring_release(const Ring& r, uint32_t stage) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}" ::"r"(
          r.empty + 8 * stage),
      "r"(threadIdx.x & 31)
      : "memory");
}

// =============================== one layer of one warpgroup ===============================
// acc[64 x N] = X[:, 0 : 32 NX] . W_x^T  +  H[:, 0 : 32 NH] . W_h^T, with X in shared memory (sXw: this warpgroup's
// first row of the X atoms) and H in registers (hin: 2 NH m64k16 A fragments).  Returns with every MMA complete and
// every stage of the layer released.  Each stage's MMAs form one commit group; the wait for the previous group leaves
// this one in flight.  W is the MMA width: N / W m64nWk16 MMAs per k16 step (W = N: one MMA, since a stage image
// spans all N rows of B with one descriptor).  The first k16 MMA of each output block runs with scale-d = 0 and so
// starts the sum: acc needs no zeroing.
template <int N, int NX, int NH, int W = N>
__device__ __forceinline__ void mma_layer(float (&acc)[N / 2], const uint32_t* hin, uint32_t sXw, Ring& r) {
  constexpr int SPP = 256 / N, NS = NX + NH;
  uint32_t prev = 0;
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    if (s % SPP == 0) {
#ifdef ONERF_FIELD_TIMELINE
      const uint64_t t0 = clock64();
#endif
      mbar_wait(r.full + 8 * r.stage, r.phase, r.diag);
#ifdef ONERF_FIELD_TIMELINE
      r.full_wait += clock64() - t0;
#endif
    }
    const uint32_t b0 = r.sB + r.stage * STAGE_BYTES + (uint32_t)(s % SPP) * (uint32_t)N * 64u;
    wgmma_fence();
#pragma unroll
    for (int k16 = 0; k16 < 2; ++k16) {
#pragma unroll
      for (int nb = 0; nb < N / W; ++nb) {
        const uint64_t bd = desc_k_sw64(b0 + (uint32_t)nb * (uint32_t)W * 64u + (uint32_t)k16 * 32u);
        const int scale_d = (s == 0 && k16 == 0) ? 0 : 1;
        if (s < NX)
          wgmma_ss<W>(acc + nb * (W / 2),
                      desc_k_sw128(sXw + (uint32_t)(s >> 1) * ATOM_BYTES + (uint32_t)(s & 1) * 64u + (uint32_t)k16 * 32u), bd,
                      scale_d);
        else
          wgmma_rs<W>(acc + nb * (W / 2), hin + ((s - NX) * 2 + k16) * 4, bd, scale_d);
      }
    }
    if (s % SPP == SPP - 1 || s == NS - 1) {
      wgmma_commit();
      if (s >= SPP) {   // the previous stage's MMAs have completed: hand it back to the producer
        wgmma_wait<1>();
        ring_release(r, prev);
      }
      prev = r.stage;
      if (++r.stage == NSTAGE) { r.stage = 0; r.phase ^= 1; }
    }
  }
  wgmma_wait<0>();
  ring_release(r, prev);
  fence_regs<N / 2>(acc);
}

}  // namespace tc
