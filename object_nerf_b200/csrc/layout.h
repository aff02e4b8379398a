// Packed-weight layout shared by the pack kernels and both field kernels (host + device).
//
// One ObjectNeRF (reference models/nerf_model.py:18-95) is re-laid into one blob:
//   [fp32 section]  every GEMM layer as W^T [K][N] (K-major, kernel-K order), head vectors, biases and
//                   the per-ray-constant ("hoisted") column blocks
//   [bf16 section]  the tensor-core stage images: per GEMM layer, per 32-wide K slab, an N x 32 bf16 tile
//                   in the K-major SWIZZLE_64B shared-memory layout, in program order
//
// Kernel-K order ("X layout").  The encoded input of a sample is kept as one vector X:
//   voxel model:  X[0..271)   = scene input  [PE6(scene voxel ftr 16) | PE10(xyz)]  (reference order)
//                 X[271]      = 0 (pad)   (scene GEMMs read X[0..288): their weights for 271..287 are 0)
//                 X[272..376) = PE6(object voxel ftr 8)
//                 X[376..384) = 0 (pad to a multiple of 32/64)
//   plain model:  X[0..63) = PE10(xyz), X[63] = 0
// The scene branch consumes X[0..KX), the object branch X[0..KO).  Terms that are constant along a ray
// (direction encoding into the two dir layers, object code into object layers 0 and 2) are hoisted
// into a per-ray vector (ONERF_RAY_CONST_FLOATS) that also carries those layers' biases.
#pragma once
#include <stdint.h>

#define ONERF_W 256
#define ONERF_IW 128
#define ONERF_NCODE 64
#define ONERF_NDIR 27

// ray_const layout (floats)
#define RC_SDIR 0     // 128: b_dir  + W_dir [:,256:283] . PE4(d)
#define RC_ODIR 128   // 64 : b_odir + W_odir[:,128:155] . PE4(d)
#define RC_OL0 192    // 128: b_o0   + W_o0[:, code cols] . code
#define RC_OL2 320    // 128: b_o2   + W_o2[:, code cols] . code

enum GemmId {
  G_S0 = 0, G_S1, G_S2, G_S3, G_S4, G_S5, G_S6, G_S7, G_SFIN, G_SDIR,
  G_O0, G_O1, G_O2, G_O3, G_OFIN, G_ODIR, G_COUNT
};

struct GemmDesc {
  int K;            // kernel K (rows of W^T), multiple of 32
  int N;            // outputs
  int64_t wt_off;   // fp32 W^T [K][N], float offset into the blob
  int64_t bias_off; // fp32 [N] (for hoisted layers this bias is folded into ray_const and unused)
  int64_t img_off;  // bf16 stage images, BYTE offset into the blob; K/32 images of N*64 bytes
  // backward (input-gradient chain, bwd_tc.cu): stage images of the TRANSPOSED hidden block of W,
  //   B[n][k] = W[k][hid_col0 + n], n < hid_n (inputs taken from the previous hidden layer), k < N (outputs):
  //   N/32 images of hid_n*64 bytes.  hid_n = 0: the layer has no hidden input (S0, O0).
  int hid_n, hid_col0;     // hid_col0: first kernel-K column of the hidden block
  int64_t bimg_off;
};

struct PackLayout {
  int use_voxel;
  int KX, KO;       // scene / object widths of X (288/384 voxel, 64/64 plain)
  int n_obj_vox;    // 104 or 0
  GemmDesc g[G_COUNT];
  int64_t sigma_w, sigma_b;     // [256], [1]
  int64_t rgb_w, rgb_b;         // [3][128], [3]
  int64_t osigma_w, osigma_b;   // [128], [1]
  int64_t orgb_w, orgb_b;       // [3][64], [3]
  int64_t h_sdir, h_odir;       // [27][128], [27][64]   (K-major)
  int64_t h_ol0, h_ol2;         // [64][128] each
  int64_t b_sdir, b_odir, b_ol0, b_ol2;  // biases folded into ray_const
  int64_t fp32_floats;          // size of the fp32 section
  // backward: images of the X blocks of the four X-fed layers (S0, S4, O0, O2), transposed, rows = X column
  // (ONERF_DX_N rows, zero where a layer does not read the column), K = the layer's outputs:
  //   per layer N/32 images of ONERF_DX_N*64 bytes, in the order S0, S4, O0, O2 (24 images)
  int64_t ximg_off;
  int64_t total_bytes;
};

#define ONERF_DX_N 384

static inline PackLayout onerf_make_layout(int use_voxel) {
  PackLayout L;
  L.use_voxel = use_voxel;
  L.KX = use_voxel ? 288 : 64;  // 272 rounded up to a 32-wide K slab (columns 272..287 carry zero scene weights)
  L.KO = use_voxel ? 384 : 64;
  L.n_obj_vox = use_voxel ? 104 : 0;
  const int K[G_COUNT] = {L.KX, 256, 256, 256, L.KX + 256, 256, 256, 256, 256, 256,
                          L.KO, 128, L.KO + 128, 128, 128, 128};
  const int N[G_COUNT] = {256, 256, 256, 256, 256, 256, 256, 256, 256, 128, 128, 128, 128, 128, 128, 64};
  int64_t f = 0;
  for (int i = 0; i < G_COUNT; ++i) {
    L.g[i].K = K[i];
    L.g[i].N = N[i];
    L.g[i].wt_off = f;
    f += (int64_t)K[i] * N[i];
    L.g[i].bias_off = f;
    f += N[i];
  }
  auto take = [&](int64_t n) { int64_t o = f; f += (n + 3) & ~3ll; return o; };
  L.sigma_w = take(256); L.sigma_b = take(1);
  L.rgb_w = take(3 * 128); L.rgb_b = take(3);
  L.osigma_w = take(128); L.osigma_b = take(1);
  L.orgb_w = take(3 * 64); L.orgb_b = take(3);
  L.h_sdir = take(27 * 128); L.h_odir = take(27 * 64);
  L.h_ol0 = take(64 * 128); L.h_ol2 = take(64 * 128);
  L.b_sdir = take(128); L.b_odir = take(64); L.b_ol0 = take(128); L.b_ol2 = take(128);
  L.fp32_floats = f;
  int64_t bytes = (f * 4 + 1023) & ~1023ll;
  for (int i = 0; i < G_COUNT; ++i) {
    L.g[i].img_off = bytes;
    bytes += (int64_t)(K[i] / 32) * N[i] * 64;
  }
  // hidden input block of every layer (kernel-K columns): width and first column
  const int hid_n[G_COUNT] = {0, 256, 256, 256, 256, 256, 256, 256, 256, 256, 0, 128, 128, 128, 128, 128};
  const int hid_c[G_COUNT] = {0, 0, 0, 0, L.KX, 0, 0, 0, 0, 0, 0, 0, L.KO, 0, 0, 0};
  for (int i = 0; i < G_COUNT; ++i) {
    L.g[i].hid_n = hid_n[i];
    L.g[i].hid_col0 = hid_c[i];
    L.g[i].bimg_off = bytes;
    bytes += (int64_t)(N[i] / 32) * hid_n[i] * 64;
  }
  L.ximg_off = bytes;
  bytes += (int64_t)((256 + 256 + 128 + 128) / 32) * ONERF_DX_N * 64;
  L.total_bytes = bytes;
  return L;
}

// ---------------------------------------------------------------------------------------------------
// Training dump ("atoms"): what the bf16 forward leaves behind for the tensor-core backward.
// An atom is a [128 samples x 64 columns] bf16 block in the SWIZZLE_128B shared-memory layout
// (row r at r*128 B, 16-byte chunk c of the row stored at chunk position c ^ (r & 7)); 16 KB.  The same image
// serves as a K-major operand (K = columns: input-gradient GEMMs) and as an MN-major operand (K = samples:
// weight-gradient GEMMs), so one bulk copy brings a ready-to-use tile into shared memory.
//   activation slots: 0 = X (6 atoms voxel / 1 plain), 1..8 scene hidden 1..8, 9 scene final, 10 scene dir,
//                     11..14 object hidden 1..4, 15 object final, 16 object dir    (same order as the fp32 dump)
//   dZ slots        : gradient w.r.t. the pre-activation of the layer whose output is activation slot i + 1
//   masks           : per tile ONERF_MASK_WORDS x 128 uint32: bit j of word w of row r = (output column > 0)
// Slot-major: atom a of tile t of a slot lives at slot_off + (t * atoms + a) * 16 KB.
// ---------------------------------------------------------------------------------------------------
#define ONERF_ACT_SLOTS 17
#define ONERF_DZ_SLOTS 16
#define ONERF_MASK_WORDS 88      // scene hidden 8 x 8, scene dir 4, object hidden 4 x 4, object dir 4
#define ONERF_ATOM_BYTES 16384

struct TrainLayout {
  int n_tiles;
  int act_atoms[ONERF_ACT_SLOTS];
  int dz_atoms[ONERF_DZ_SLOTS];
  int64_t act_off[ONERF_ACT_SLOTS];   // byte offsets into the training workspace
  int64_t dz_off[ONERF_DZ_SLOTS];
  int64_t mask_off;
  int64_t total_bytes;
};

#ifdef __CUDACC__
__host__ __device__
#endif
static inline int onerf_mask_word0(int act_slot) {   // first mask word of the layer whose output is `act_slot`
  if (act_slot >= 1 && act_slot <= 8) return (act_slot - 1) * 8;
  if (act_slot == 10) return 64;
  if (act_slot >= 11 && act_slot <= 14) return 68 + (act_slot - 11) * 4;
  if (act_slot == 16) return 84;
  return -1;   // final layers have no activation
}

static inline TrainLayout onerf_make_train_layout(int use_voxel, int64_t n_samples) {
  TrainLayout T;
  T.n_tiles = (int)((n_samples + 127) / 128);
  const int aw[ONERF_ACT_SLOTS] = {use_voxel ? 6 : 1, 4, 4, 4, 4, 4, 4, 4, 4, 4, 2, 2, 2, 2, 2, 2, 1};
  int64_t bytes = 0;
  for (int i = 0; i < ONERF_ACT_SLOTS; ++i) {
    T.act_atoms[i] = aw[i];
    T.act_off[i] = bytes;
    bytes += (int64_t)aw[i] * T.n_tiles * ONERF_ATOM_BYTES;
  }
  for (int i = 0; i < ONERF_DZ_SLOTS; ++i) {
    T.dz_atoms[i] = aw[i + 1];
    T.dz_off[i] = bytes;
    bytes += (int64_t)aw[i + 1] * T.n_tiles * ONERF_ATOM_BYTES;
  }
  bytes += ONERF_ATOM_BYTES;   // the weight-gradient GEMM reads one atom past the 64-wide object-dir dZ slot
  T.mask_off = bytes;
  bytes += (int64_t)T.n_tiles * ONERF_MASK_WORDS * 128 * 4;
  T.total_bytes = (bytes + 1023) & ~1023ll;
  return T;
}

// Kernel-layout gradient buffer of one model (fp32), written by the tensor-core backward and mapped back to the
// reference's [out,in] tensors by onerf_unpack_grads: per GEMM layer dW [N][K] (kernel-K columns) and db [N], then
// the four heads.
struct GradLayout {
  int64_t w_off[G_COUNT], b_off[G_COUNT];
  int64_t sigma_w, sigma_b, rgb_w, rgb_b, osigma_w, osigma_b, orgb_w, orgb_b;
  int64_t total_floats;
};
GradLayout onerf_make_grad_layout(int use_voxel);
