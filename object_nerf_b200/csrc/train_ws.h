// Layout of the training workspace of onerf_render_rays_fwd / onerf_render_rays_bwd (one caller-owned blob).
#pragma once
#include <cuda_runtime.h>

#include "../../include/onerf.h"
#include "layout.h"

// The model a training call trains: voxel when it carries a grid, plain PE otherwise.  The forward and the backward
// both derive the workspace layout from it and from the call's precision.
static inline int onerf_train_use_voxel(const onerf_render_args* a) { return a->grid ? 1 : 0; }

// The fp32 backward re-runs the FFMA forward over chunks of whole rays holding at most this many samples (one ray when
// a single ray has more).
#define ONERF_FP32_CHUNK_SAMPLES 65536
static inline int onerf_fp32_chunk_rays(int n_rays, int n_samples) {
  int r = n_samples > 0 ? ONERF_FP32_CHUNK_SAMPLES / n_samples : 1;
  if (r < 1) r = 1;
  return r < n_rays ? r : n_rays;
}
// widths of the fp32 activation dump (onerf_field_args::activations) after X (384 voxel / 64 plain)
static constexpr int ONERF_ACT_WIDTHS_TAIL[16] = {256, 256, 256, 256, 256, 256, 256, 256, 256, 128, 128, 128, 128, 128, 128, 64};

struct TrainWs {
  int64_t tl_coarse, tl_fine;                   // bf16: field training workspaces (layout.h: TrainLayout) of the two passes
  int64_t scene_c, obj_c, scene_f, obj_f;       // per-sample fields (rgb, sigma) of both passes, kept for the backward
  int64_t dscene, dobj, dA_s, dA_o;             // per-sample gradients (one pass at a time); dA_*: bf16 only
  int64_t rs, pe;                               // per-ray sums (bf16: N x 448; fp32: chunk rays x 128), PE4 of the directions (N,27)
  int64_t gk;                                   // bf16: kernel-layout gradient buffer (one pass at a time)
  // fp32: one chunk of the backward (onerf_fp32_chunk_rays rays of either pass)
  int64_t act[17];                              // the FFMA forward's activation dump: X, then ONERF_ACT_WIDTHS_TAIL
  int64_t dX, bufA, bufB, dA;                   // d(X), two 256-wide input-gradient buffers, head gradients (B,4)
  int64_t field_s, field_o, ray_const;          // the re-run's fields (B,4) and per-ray hoisted terms
  int64_t total;
};

static inline TrainWs onerf_make_train_ws(int precision, int use_voxel, int n_rays, int n_samples, int n_importance) {
  TrainWs W = {};
  int64_t o = 0;
  auto take = [&](int64_t bytes) { int64_t r = o; o += (bytes + 1023) & ~1023ll; return r; };
  const bool tc = precision == ONERF_PREC_BF16;
  const int sf = n_samples + n_importance;
  const int64_t Bc = (int64_t)n_rays * n_samples, Bf = (int64_t)n_rays * sf;
  const int rc = onerf_fp32_chunk_rays(n_rays, n_samples), rf = onerf_fp32_chunk_rays(n_rays, sf);
  const int R = tc ? 0 : (rc > rf ? rc : rf);                                      // fp32 chunk: rays, samples
  const int64_t B = tc ? 0 : ((int64_t)rc * n_samples > (int64_t)rf * sf ? (int64_t)rc * n_samples : (int64_t)rf * sf);
  W.tl_coarse = take(tc ? onerf_make_train_layout(use_voxel, Bc).total_bytes : 0);
  W.tl_fine = take(tc && n_importance > 0 ? onerf_make_train_layout(use_voxel, Bf).total_bytes : 0);
  W.scene_c = take(Bc * 16); W.obj_c = take(Bc * 16);
  W.scene_f = take(Bf * 16); W.obj_f = take(Bf * 16);
  W.dscene = take(Bf * 16); W.dobj = take(Bf * 16); W.dA_s = take(tc ? Bf * 16 : 0); W.dA_o = take(tc ? Bf * 16 : 0);
  W.rs = take(tc ? (int64_t)n_rays * ONERF_RAY_CONST_FLOATS * 4 : (int64_t)R * 128 * 4);
  W.pe = take((int64_t)n_rays * 27 * 4);
  W.gk = take(tc ? onerf_make_grad_layout(use_voxel).total_floats * 4 : 0);
  if (!tc) {
    W.act[0] = take(B * (use_voxel ? 384 : 64) * 4);
    for (int i = 0; i < 16; ++i) W.act[1 + i] = take(B * ONERF_ACT_WIDTHS_TAIL[i] * 4);
    W.dX = take(B * (use_voxel ? 384 : 64) * 4);
    W.bufA = take(B * 256 * 4); W.bufB = take(B * 256 * 4);
    W.dA = take(B * 16);
    W.field_s = take(B * 16); W.field_o = take(B * 16);
    W.ray_const = take((int64_t)R * ONERF_RAY_CONST_FLOATS * 4);
  }
  W.total = o;
  return W;
}

// onerf_train_step appends to the training workspace: the coarse pass's per-sample field gradients (the fine pass uses
// TrainWs::dscene / dobj; both are written during the forward, before either field backward runs) and the loss
// accumulators (loss_terms.cuh: WS_DOUBLES doubles, then the block counter of the last compositing kernel).
struct TrainStepWs {
  int64_t dscene_c, dobj_c, loss;
  int64_t total;
};
#define ONERF_STEP_LOSS_BYTES 256

static inline TrainStepWs onerf_make_train_step_ws(const TrainWs& W, int n_rays, int n_samples) {
  TrainStepWs T;
  int64_t o = W.total;
  auto take = [&](int64_t bytes) { int64_t r = o; o += (bytes + 1023) & ~1023ll; return r; };
  const int64_t Bc = (int64_t)n_rays * n_samples;
  T.dscene_c = take(Bc * 16); T.dobj_c = take(Bc * 16);
  T.loss = take(ONERF_STEP_LOSS_BYTES);
  T.total = o;
  return T;
}

// The training step's compositing kernel (composite.cu): forward, the loss terms this pass owns and the compositing
// backward, per ray.
struct onerf_step_composite {
  onerf_loss_args loss;   // batch, term weights and (finalize) outputs; map and gradient pointers unused
  double* acc;            // loss accumulators + block counter, counts already summed (onerf_launch_batch_stats)
  int fine;               // 0 coarse, 1 fine: which squared-error sums this pass adds to
  int finalize;           // last compositing kernel of the step: its last block writes the loss outputs and psnr
  float* psnr_out;
  float* dscene;          // (N,S,4) d(r, g, b, sigma) of the scene branch
  float* dobj;            // (N,S,4) of the object branch
};
// Device seed (onerf_ext.h: onerf_render_rays_fwd_dseed, onerf_train_step_dseed): every launcher below that takes
// `seed_dev` draws with seed + *seed_dev read when its kernel runs if seed_dev != NULL (the caller then passes only the
// per-draw offset in `seed`), and with `seed` alone otherwise.  With finalize set, the step's compositing kernel adds
// ONERF_SEED_ADVANCE to *seed_dev once every block has read it.
#define ONERF_SEED_ADVANCE 4
int onerf_launch_composite_step(onerf_ctx* ctx, const onerf_composite_args* c, const onerf_step_composite* t,
                                uint64_t* seed_dev, cudaStream_t stream);
int onerf_launch_composite(onerf_ctx* ctx, const onerf_composite_args* c, uint64_t* seed_dev, cudaStream_t stream);
int onerf_launch_seed_advance(onerf_ctx* ctx, uint64_t* seed_dev, cudaStream_t stream);   // one thread: *seed_dev += 4
int onerf_launch_sample_coarse(onerf_ctx* ctx, const float* rays, int n_rays, int n_samples, int use_disp, float perturb,
                               const float* jitter, uint64_t seed, const uint64_t* seed_dev, float* z_out, void* stream);
int onerf_launch_sample_pdf_merge(onerf_ctx* ctx, const float* z_coarse, const float* weights, int n_rays, int n_samples,
                                  int n_importance, int det, const float* u, uint64_t seed, const uint64_t* seed_dev,
                                  float* z_out, void* stream);
int onerf_launch_batch_stats(onerf_ctx* ctx, const onerf_loss_args* a, double* acc, cudaStream_t stream);
// onerf_render_rays_fwd with an optional training step: step == NULL is the plain forward; otherwise both passes'
// compositing runs onerf_launch_composite_step with `step` (fine / finalize / dscene / dobj set per pass from ws_step),
// and the finalizing one advances *seed_dev.  seed_dev as above; a->seed is ignored when it is set.
int onerf_render_fwd_impl(onerf_ctx* ctx, const onerf_render_args* a, const onerf_step_composite* step, uint64_t* seed_dev,
                          void* stream);
