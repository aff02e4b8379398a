// Input-gradient chain of the two-branch MLP on wgmma tensor cores (SURVEY.md §8 row a14): for every sample tile,
//   dZ_dir = (dL/d rgb_pre . W_rgb) * leaky'(H_dir)                                    (CUDA cores, 3-wide head)
//   dZ_l-1 = (dZ_l . W_l[:, hidden block]  [+ dL/d sigma . w_sigma]) * leaky'(H_l-1)    (wgmma, fp32 accumulate)
// walking the layers of models/nerf_model.py:97-152 backwards, scene branch then object branch.  It is the forward
// machinery (tc_chain.cuh: bulk-copy weight ring, register-resident operand chain) run on the TRANSPOSED weight images
// (layout.h: bimg_off); the LeakyReLU derivative comes from the 1-bit sign masks the training forward left behind.
// Every dZ_l is also written to the training workspace as bf16 atoms: the weight-gradient GEMM (bwd_wgrad.cu), the
// encoding gradient (bwd_dx.cu) and the bias / per-ray sums (bwd_small.cu) read them from there.
#include "field_common.cuh"
#include "tc_chain.cuh"

namespace {

using namespace tc;

enum BwdEpi { BE_PLAIN = 0, BE_MASK = 1, BE_MASK_SIG = 2 };

struct ChainParams {
  const uint8_t* packed;      // packed weights (bwd images + fp32 head vectors)
  PackLayout L;
  uint8_t* ws;                // training workspace (masks in, dZ atoms out)
  TrainLayout TL;
  const float4* dA_scene;     // (B) d(rgb_pre, sigma) of the scene branch
  const float4* dA_obj;       // (B) or null
  int64_t total;              // samples
  int want_object;
  WLayer layers[MAX_LAYERS];
  int n_layers;
  uint32_t* diag;             // mbarrier timeout record (onerf_ctx)
};

struct Rows {
  int row[2];
  float4 dAs[2], dAo[2];
  const uint32_t* mrow;       // &masks[tile][0][0]
  int64_t tile;
};

// store the packed fragment (N columns, rows R.row[0..1]) into dZ slot `slot` of the tile
template <int N>
__device__ __forceinline__ void store_dz(const ChainParams& P, const Rows& R, int slot, const uint32_t* pk) {
  const int q = threadIdx.x & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = R.row[r];
    uint8_t* base = P.ws + P.TL.dz_off[slot] + ((size_t)R.tile * P.TL.dz_atoms[slot]) * ATOM_BYTES + (size_t)row * 128 + q * 4;
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
      *reinterpret_cast<uint32_t*>(base + (size_t)(j >> 3) * ATOM_BYTES + (((j & 7) ^ (row & 7)) << 4)) = pk[2 * j + r];
  }
}

// dZ of a direction layer from the 3-wide rgb head: N = 128 (scene, mask words 64..67) or 64 (object, 84..87)
template <int N>
__device__ __forceinline__ void dir_dz(const Rows& R, const float* rgb_w, int branch, uint32_t* pk) {
  constexpr int CPW = N >= 128 ? 32 : 16;
  const int word0 = branch ? 84 : 64, q = threadIdx.x & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float4 d = branch ? R.dAo[r] : R.dAs[r];
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      const int c = 8 * j + 2 * q;
      const uint32_t m = R.mrow[(word0 + c / CPW) * 128 + R.row[r]];
      float v0 = d.x * rgb_w[c] + d.y * rgb_w[N + c] + d.z * rgb_w[2 * N + c];
      float v1 = d.x * rgb_w[c + 1] + d.y * rgb_w[N + c + 1] + d.z * rgb_w[2 * N + c + 1];
      v0 *= ((m >> (c % CPW)) & 1u) ? 1.0f : 0.01f;
      v1 *= ((m >> ((c + 1) % CPW)) & 1u) ? 1.0f : 0.01f;
      pk[2 * j + r] = pack_bf16(v0, v1);
    }
  }
}

// chain epilogue: v = acc [+ dsigma . w_sigma]  [* leaky'(mask of activation slot `act`)], bf16 pairs
template <int N, int EPI>
__device__ __forceinline__ void chain_epi(const float (&acc)[N / 2], uint32_t* pk, const Rows& R, int branch, int act,
                                          const float* wsig) {
  const int q = threadIdx.x & 3;
  const int word0 = EPI == BE_PLAIN ? 0 : onerf_mask_word0(act);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float dsig = branch ? R.dAo[r].w : R.dAs[r].w;
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      const int c = 8 * j + 2 * q;
      float v0 = acc[4 * j + 2 * r], v1 = acc[4 * j + 2 * r + 1];
      if (EPI == BE_MASK_SIG) {
        v0 = fmaf(dsig, wsig[c], v0);
        v1 = fmaf(dsig, wsig[c + 1], v1);
      }
      if (EPI != BE_PLAIN) {
        const uint32_t m = R.mrow[(word0 + (c >> 5)) * 128 + R.row[r]];
        v0 *= ((m >> (c & 31)) & 1u) ? 1.0f : 0.01f;
        v1 *= ((m >> ((c + 1) & 31)) & 1u) ? 1.0f : 0.01f;
      }
      pk[2 * j + r] = pack_bf16(v0, v1);
    }
  }
}

__global__ void __launch_bounds__(NUM_THREADS, 1) bwd_chain_kernel(const __grid_constant__ ChainParams P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sB = sbase;
  const uint32_t sHead = sB + NSTAGE * STAGE_BYTES;                  // 960 floats: rgb_w 384 | sigma_w 256 | orgb_w 192 | osigma_w 128
  const uint32_t sBar = sHead + 960 * 4;
  uint8_t* gen_base = smem_raw + (sbase - smem_u32(smem_raw));
  float* head = reinterpret_cast<float*>(gen_base + (sHead - sbase));
  const float* Pf = reinterpret_cast<const float*>(P.packed);
  Ring ring{sB, sBar, sBar + 8 * NSTAGE, 0u, 0u, P.diag};

  if (threadIdx.x == 0) ring_init_bars(ring.full, ring.empty);
  for (int i = threadIdx.x; i < 960; i += NUM_THREADS) {
    float v;
    if (i < 384) v = __ldg(Pf + P.L.rgb_w + i);
    else if (i < 640) v = __ldg(Pf + P.L.sigma_w + (i - 384));
    else if (i < 832) v = __ldg(Pf + P.L.orgb_w + (i - 640));
    else v = __ldg(Pf + P.L.osigma_w + (i - 832));
    head[i] = v;
  }
  __syncthreads();
  const int64_t n_tiles = (P.total + TM - 1) / TM;

  if (warp >= PRODUCER_WARP) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == PRODUCER_WARP)
      tc_producer_loop(P.layers, P.n_layers, P.packed, ring, n_tiles);
    return;
  }
  setmaxnreg_inc<CONSUMER_REGS>();

  const float* rgb_w = head, *sigma_w = head + 384, *orgb_w = head + 640, *osigma_w = head + 832;
  const int wg = warp >> 2;
  Rows R;
  R.row[0] = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  R.row[1] = R.row[0] + 8;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    R.tile = tile;
    R.mrow = reinterpret_cast<const uint32_t*>(P.ws + P.TL.mask_off) + (size_t)tile * ONERF_MASK_WORDS * 128;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int64_t e = tile * TM + R.row[r];
      const bool live = e < P.total;
      R.dAs[r] = live ? __ldg(P.dA_scene + e) : make_float4(0.f, 0.f, 0.f, 0.f);
      R.dAo[r] = (live && P.want_object) ? __ldg(P.dA_obj + e) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    // m64n64k16 MMAs: with full-width ones the chain's register demand (dZ fragments, per-row head gradients) does not
    // fit the consumer budget and ptxas spills several KB per thread.
    {
      // ---- scene: dZ_dir (128) -> dZ_final -> dZ_7 (+ sigma head) -> ... -> dZ_0 ----
      uint32_t a[32];
      dir_dz<128>(R, rgb_w, 0, a);
      store_dz<128>(P, R, 9, a);
      float acc[128];
      uint32_t h[64];
      mma_layer<256, 0, 4, 64>(acc, a, 0u, ring);
      chain_epi<256, BE_PLAIN>(acc, h, R, 0, 9, nullptr);
      store_dz<256>(P, R, 8, h);
      mma_layer<256, 0, 8, 64>(acc, h, 0u, ring);
      chain_epi<256, BE_MASK_SIG>(acc, h, R, 0, 8, sigma_w);
      store_dz<256>(P, R, 7, h);
#pragma unroll 1
      for (int l = 7; l >= 1; --l) {
        mma_layer<256, 0, 8, 64>(acc, h, 0u, ring);
        chain_epi<256, BE_MASK>(acc, h, R, 0, l, nullptr);
        store_dz<256>(P, R, l - 1, h);
      }
    }
    if (P.want_object) {
      // ---- object: dZ_odir (64) -> dZ_ofinal -> dZ_o3 (+ sigma head) -> ... -> dZ_o0 ----
      uint32_t a[16];
      dir_dz<64>(R, orgb_w, 1, a);
      store_dz<64>(P, R, 15, a);
      float acc[64];
      uint32_t h[32];
      mma_layer<128, 0, 2, 64>(acc, a, 0u, ring);
      chain_epi<128, BE_PLAIN>(acc, h, R, 1, 15, nullptr);
      store_dz<128>(P, R, 14, h);
      mma_layer<128, 0, 4, 64>(acc, h, 0u, ring);
      chain_epi<128, BE_MASK_SIG>(acc, h, R, 1, 14, osigma_w);
      store_dz<128>(P, R, 13, h);
#pragma unroll 1
      for (int l = 3; l >= 1; --l) {
        mma_layer<128, 0, 4, 64>(acc, h, 0u, ring);
        chain_epi<128, BE_MASK>(acc, h, R, 1, 10 + l, nullptr);
        store_dz<128>(P, R, 10 + l - 1, h);
      }
    }
  }
}

}  // namespace

int onerf_launch_bwd_chain(onerf_ctx* ctx, int use_voxel, int want_object, const void* packed, void* ws, int64_t n_samples,
                           const float* dA_scene, const float* dA_obj, cudaStream_t stream) {
  ChainParams P;
  memset(&P, 0, sizeof(P));
  const PackLayout L = onerf_make_layout(use_voxel);
  P.packed = reinterpret_cast<const uint8_t*>(packed);
  P.L = L;
  P.ws = reinterpret_cast<uint8_t*>(ws);
  P.TL = onerf_make_train_layout(use_voxel, n_samples);
  P.dA_scene = reinterpret_cast<const float4*>(dA_scene);
  P.dA_obj = reinterpret_cast<const float4*>(dA_obj);
  P.total = n_samples;
  P.want_object = want_object;
  P.diag = ctx->tc_diag;
  int n = 0;
  // chain layer of GEMM g: operand = dZ of g (its N outputs = K of this layer), result = the hid_n inputs of g
  auto add = [&](int g) { P.layers[n++] = WLayer{L.g[g].bimg_off, L.g[g].hid_n, L.g[g].N / 32}; };
  add(G_SDIR);
  add(G_SFIN);
  for (int l = 7; l >= 1; --l) add(G_S0 + l);
  if (want_object) {
    add(G_ODIR);
    add(G_OFIN);
    for (int l = 3; l >= 1; --l) add(G_O0 + l);
  }
  P.n_layers = n;
  const int64_t tiles = (n_samples + TM - 1) / TM;
  const int blocks = (int)(tiles < ctx->num_sms ? tiles : ctx->num_sms);
  const size_t smem = 1024 + NSTAGE * STAGE_BYTES + 960 * 4 + 16 * NSTAGE;
  ONERF_CUDA(cudaFuncSetAttribute(bwd_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  bwd_chain_kernel<<<blocks, NUM_THREADS, smem, stream>>>(P);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
