// Orchestration of the tensor-core training path behind the C ABI: workspace layout, the training variant of
// onerf_render_rays_fwd's passes, and onerf_render_rays_bwd (SURVEY.md §8 rows a14 / b).
#include <string.h>

#include "field_common.cuh"
#include "train_ws.h"

int onerf_launch_bwd_chain(onerf_ctx* ctx, int use_voxel, int want_object, const void* packed, void* ws, int64_t n_samples,
                           const float* dA_scene, const float* dA_obj, cudaStream_t stream);
int onerf_launch_wgrad(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int64_t n_samples, float* grad,
                       cudaStream_t stream);
int onerf_launch_bwd_dx(onerf_ctx* ctx, int want_object, const void* packed, const void* ws, int64_t n_samples,
                        const float* rays, const float* z, int n_samples_per_ray, const onerf_grid* grid, float* table_grad,
                        cudaStream_t stream);
int onerf_launch_bwd_colsums(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int64_t n_samples,
                             const float* dA_scene, const float* dA_obj, float* grad, cudaStream_t stream);
int onerf_launch_bwd_raysums(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int n_rays, int S, float* out,
                             cudaStream_t stream);

extern "C" size_t onerf_field_train_bytes(int use_voxel, int64_t n_samples) {
  return (size_t)onerf_make_train_layout(use_voxel ? 1 : 0, n_samples).total_bytes;
}

extern "C" size_t onerf_train_workspace_bytes(int use_voxel, int n_rays, int n_samples, int n_importance) {
  if (n_rays < 0 || n_samples < 1 || n_importance < 0) return 0;
  return (size_t)onerf_make_train_ws(use_voxel ? 1 : 0, n_rays, n_samples, n_importance).total;
}

// ---- stage entry points (tests, ncu) ----
extern "C" int onerf_bwd_chain(onerf_ctx* ctx, int use_voxel, int want_object, const void* packed, void* ws, int64_t n_samples,
                               const float* dA_scene, const float* dA_obj, void* stream) {
  ONERF_CHECK_ARG(ctx && packed && ws && dA_scene && (!want_object || dA_obj), "null argument");
  if (n_samples == 0) return ONERF_OK;
  return onerf_launch_bwd_chain(ctx, use_voxel ? 1 : 0, want_object, packed, ws, n_samples, dA_scene, dA_obj, (cudaStream_t)stream);
}
extern "C" int onerf_bwd_wgrad(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int64_t n_samples, float* grad,
                               void* stream) {
  ONERF_CHECK_ARG(ctx && ws && grad && onerf_aligned16(grad), "null / misaligned argument");
  if (n_samples == 0) return ONERF_OK;
  return onerf_launch_wgrad(ctx, use_voxel ? 1 : 0, want_object, ws, n_samples, grad, (cudaStream_t)stream);
}
extern "C" int onerf_bwd_colsums(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int64_t n_samples,
                                 const float* dA_scene, const float* dA_obj, float* grad, void* stream) {
  ONERF_CHECK_ARG(ctx && ws && grad && dA_scene && (!want_object || dA_obj), "null argument");
  if (n_samples == 0) return ONERF_OK;
  return onerf_launch_bwd_colsums(ctx, use_voxel ? 1 : 0, want_object, ws, n_samples, dA_scene, dA_obj, grad, (cudaStream_t)stream);
}
extern "C" int onerf_bwd_raysums(onerf_ctx* ctx, int use_voxel, int want_object, const void* ws, int n_rays, int n_samples,
                                 float* out, void* stream) {
  ONERF_CHECK_ARG(ctx && ws && out, "null argument");
  if (n_rays == 0) return ONERF_OK;
  return onerf_launch_bwd_raysums(ctx, use_voxel ? 1 : 0, want_object, ws, n_rays, n_samples, out, (cudaStream_t)stream);
}
extern "C" int onerf_bwd_dx(onerf_ctx* ctx, int want_object, const void* packed, const void* ws, const float* rays,
                            const float* z, int n_rays, int n_samples, const onerf_grid* grid, float* table_grad, void* stream) {
  ONERF_CHECK_ARG(ctx && packed && ws && rays && z && grid && table_grad && onerf_aligned16(table_grad), "null / misaligned argument");
  if (n_rays == 0) return ONERF_OK;
  return onerf_launch_bwd_dx(ctx, want_object, packed, ws, (int64_t)n_rays * n_samples, rays, z, n_samples, grid, table_grad,
                             (cudaStream_t)stream);
}

// ---- backward of one pass ----
static int bwd_pass(onerf_ctx* ctx, const onerf_render_args* f, const onerf_render_bwd_args* b, const TrainWs& W, int use_voxel,
                    bool fine, char* ws, const float* pe, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const int fi = f->forward_instance ? 1 : 0;
  const int S = fine ? f->n_samples + f->n_importance : f->n_samples;
  const int R = f->n_rays;
  const int64_t B = (int64_t)R * S;
  const onerf_render_maps& m = fine ? f->fine : f->coarse;
  const onerf_map_grads& g = fine ? b->fine : b->coarse;
  const void* packed = fine ? f->packed_fine : f->packed_coarse;
  const float* const* Wref = fine ? b->W_fine : b->W_coarse;
  float* const* dW = fine ? b->dW_fine : b->dW_coarse;
  float* const* db = fine ? b->db_fine : b->db_coarse;
  char* tl = ws + (fine ? W.tl_fine : W.tl_coarse);
  float* scene = reinterpret_cast<float*>(ws + (fine ? W.scene_f : W.scene_c));
  float* obj = reinterpret_cast<float*>(ws + (fine ? W.obj_f : W.obj_c));
  float* dscene = reinterpret_cast<float*>(ws + W.dscene);
  float* dobj = reinterpret_cast<float*>(ws + W.dobj);
  float* dA_s = reinterpret_cast<float*>(ws + W.dA_s);
  float* dA_o = reinterpret_cast<float*>(ws + W.dA_o);
  float* rs = reinterpret_cast<float*>(ws + W.rs);
  float* gk = reinterpret_cast<float*>(ws + W.gk);
  int rc;
#define TRY(x) do { rc = (x); if (rc != ONERF_OK) return rc; } while (0)
  // 1. compositing backward (same arguments / seeds as the forward's render_pass)
  onerf_composite_args c;
  memset(&c, 0, sizeof(c));
  c.z = m.z_vals; c.scene = scene; c.obj = fi ? obj : nullptr;
  c.n_rays = R; c.n_samples = S;
  c.noise_std = f->noise_std;
  c.noise_scene = fine ? f->noise_scene_fine : f->noise_scene_coarse;
  c.noise_obj = fine ? f->noise_obj_fine : f->noise_obj_coarse;
  c.seed = f->seed + (fine ? 3 : 1);
  c.white_back = f->white_back; c.is_eval = f->is_eval; c.zero_last_delta = f->zero_last_delta;
  c.rays_in_bbox = f->rays_in_bbox; c.frustum_bound_th = f->frustum_bound_th;
  c.pass_through_mask = f->pass_through_mask;
  TRY(onerf_composite_bwd(ctx, &c, m.depth, g.rgb, g.depth, g.opacity, g.rgb_instance, g.depth_instance, g.opacity_instance,
                          dscene, fi ? dobj : nullptr, stream_));
  // 2. sigmoid / raw-sigma heads
  TRY(onerf_head_bwd(ctx, dscene, scene, dA_s, B, stream_));
  if (fi) TRY(onerf_head_bwd(ctx, dobj, obj, dA_o, B, stream_));
  // 3. input-gradient chain: dZ of every layer -> workspace atoms
  TRY(onerf_launch_bwd_chain(ctx, use_voxel, fi, packed, tl, B, dA_s, fi ? dA_o : nullptr, stream));
  // 4. weight / bias / head gradients in kernel layout
  const GradLayout G = onerf_make_grad_layout(use_voxel);
  ONERF_CUDA(cudaMemsetAsync(gk, 0, (size_t)G.total_floats * sizeof(float), stream));
  TRY(onerf_launch_bwd_colsums(ctx, use_voxel, fi, tl, B, dA_s, fi ? dA_o : nullptr, gk, stream));
  TRY(onerf_launch_wgrad(ctx, use_voxel, fi, tl, B, gk, stream));
  TRY(onerf_unpack_grads(ctx, use_voxel, gk, dW, db, stream_));
  // 5. encoding -> voxel table (voxel model only: the plain model has nothing trainable in front of X)
  if (b->table_grad) TRY(onerf_launch_bwd_dx(ctx, fi, packed, tl, B, f->rays, m.z_vals, S, f->grid, b->table_grad, stream));
  // 6. per-ray-constant columns: direction encoding into the two dir layers, object code into object layers 1 and 3
  TRY(onerf_launch_bwd_raysums(ctx, use_voxel, fi, tl, R, S, rs, stream));
  // reference input widths: scene input [voxel PE | xyz PE] or [xyz PE], object voxel block, object input [.. | code]
  const int xin = use_voxel ? 271 : 63, ovx = use_voxel ? 104 : 0, oin = xin + ovx + ONERF_NCODE;
  TRY(onerf_gemm(ctx, rs + RC_SDIR, ONERF_RAY_CONST_FLOATS, 1, pe, 27, dW[10] + 256, 256 + 27, 128, 27, R, 1, stream_));
  if (fi) {
    TRY(onerf_gemm(ctx, rs + RC_ODIR, ONERF_RAY_CONST_FLOATS, 1, pe, 27, dW[18] + 128, 128 + 27, 64, 27, R, 1, stream_));
    TRY(onerf_gemm(ctx, rs + RC_OL0, ONERF_RAY_CONST_FLOATS, 1, f->codes, 64, dW[12] + xin + ovx, oin, 128, 64, R, 1, stream_));
    TRY(onerf_gemm(ctx, rs + RC_OL2, ONERF_RAY_CONST_FLOATS, 1, f->codes, 64, dW[14] + xin + ovx, oin + 128, 128, 64, R, 1, stream_));
    if (b->d_codes) {
      TRY(onerf_gemm(ctx, rs + RC_OL0, ONERF_RAY_CONST_FLOATS, 0, Wref[12] + xin + ovx, oin, b->d_codes, 64, R, 64, 128, 1, stream_));
      TRY(onerf_gemm(ctx, rs + RC_OL2, ONERF_RAY_CONST_FLOATS, 0, Wref[14] + xin + ovx, oin + 128, b->d_codes, 64, R, 64, 128, 1, stream_));
    }
  }
#undef TRY
  return ONERF_OK;
}

extern "C" int onerf_render_rays_bwd(onerf_ctx* ctx, const onerf_render_args* f, const onerf_render_bwd_args* b, void* stream) {
  ONERF_CHECK_ARG(ctx && f && b, "null argument");
  ONERF_CHECK_ARG(f->train_ws, "the forward was not run with a training workspace");
  ONERF_UNSUPPORTED(f->precision != ONERF_PREC_BF16, "the tensor-core backward is built for bf16");
  ONERF_CHECK_ARG(b->W_coarse && b->dW_coarse && b->db_coarse, "null coarse gradient arguments");
  ONERF_CHECK_ARG(f->n_importance == 0 || (b->W_fine && b->dW_fine && b->db_fine), "null fine gradient arguments");
  const int use_voxel = onerf_train_use_voxel(f);
  ONERF_CHECK_ARG(use_voxel || !b->table_grad, "table_grad given for the plain-PE model, which has no voxel table");
  ONERF_CHECK_ARG(!b->table_grad || onerf_aligned16(b->table_grad), "table_grad misaligned");
  const TrainWs W = onerf_make_train_ws(use_voxel, f->n_rays, f->n_samples, f->n_importance);
  if (f->train_ws_bytes < (size_t)W.total) {
    onerf_set_error("onerf_render_rays_bwd: training workspace too small (%zu < %lld)", f->train_ws_bytes, (long long)W.total);
    return ONERF_ERR_WORKSPACE;
  }
  if (f->n_rays == 0) return ONERF_OK;
  char* ws = reinterpret_cast<char*>(f->train_ws);
  float* pe = reinterpret_cast<float*>(ws + W.pe);
  int rc = onerf_dir_encode(ctx, f->rays, f->n_rays, pe, stream);
  if (rc != ONERF_OK) return rc;
  if (f->n_importance > 0) {
    rc = bwd_pass(ctx, f, b, W, use_voxel, true, ws, pe, stream);
    if (rc != ONERF_OK) return rc;
  }
  return bwd_pass(ctx, f, b, W, use_voxel, false, ws, pe, stream);
}
