// Orchestration of the training path behind the C ABI: workspace size, the stage entry points of the tensor-core
// backward, and onerf_render_rays_bwd for both arithmetics (SURVEY.md §8 rows a14 / b).
#include <string.h>

#include <initializer_list>

#include "field_common.cuh"
#include "train_ws.h"
#include "../../include/onerf_ext.h"

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

extern "C" size_t onerf_train_workspace_bytes_prec(int precision, int use_voxel, int n_rays, int n_samples, int n_importance) {
  if (precision != ONERF_PREC_FP32 && precision != ONERF_PREC_BF16) return 0;
  if (n_rays < 0 || n_samples < 1 || n_importance < 0) return 0;
  return (size_t)onerf_make_train_ws(precision, use_voxel ? 1 : 0, n_rays, n_samples, n_importance).total;
}

extern "C" size_t onerf_train_workspace_bytes(int use_voxel, int n_rays, int n_samples, int n_importance) {
  return onerf_train_workspace_bytes_prec(ONERF_PREC_BF16, use_voxel, n_rays, n_samples, n_importance);
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
#define TRY(x) do { rc = (x); if (rc != ONERF_OK) return rc; } while (0)

// Compositing backward of one pass, both precisions: the arguments and seeds of the forward's render_pass (api.cu), the
// fields it kept in the training workspace.
static int composite_bwd_pass(onerf_ctx* ctx, const onerf_render_args* f, const onerf_render_bwd_args* b, const TrainWs& W,
                              bool fine, char* ws, void* stream) {
  const int fi = f->forward_instance ? 1 : 0;
  const onerf_render_maps& m = fine ? f->fine : f->coarse;
  const onerf_map_grads& g = fine ? b->fine : b->coarse;
  onerf_composite_args c;
  memset(&c, 0, sizeof(c));
  c.z = m.z_vals;
  c.scene = reinterpret_cast<const float*>(ws + (fine ? W.scene_f : W.scene_c));
  c.obj = fi ? reinterpret_cast<const float*>(ws + (fine ? W.obj_f : W.obj_c)) : nullptr;
  c.n_rays = f->n_rays; c.n_samples = fine ? f->n_samples + f->n_importance : f->n_samples;
  c.noise_std = f->noise_std;
  c.noise_scene = fine ? f->noise_scene_fine : f->noise_scene_coarse;
  c.noise_obj = fine ? f->noise_obj_fine : f->noise_obj_coarse;
  c.seed = f->seed + (fine ? 3 : 1);
  c.white_back = f->white_back; c.is_eval = f->is_eval; c.zero_last_delta = f->zero_last_delta;
  c.rays_in_bbox = f->rays_in_bbox; c.frustum_bound_th = f->frustum_bound_th;
  c.pass_through_mask = f->pass_through_mask;
  return onerf_composite_bwd(ctx, &c, m.depth, g.rgb, g.depth, g.opacity, g.rgb_instance, g.depth_instance, g.opacity_instance,
                             reinterpret_cast<float*>(ws + W.dscene), fi ? reinterpret_cast<float*>(ws + W.dobj) : nullptr,
                             stream);
}

// bf16: the tensor-core chain, weight-gradient and encoding-gradient GEMMs on the operands the forward kept
static int bwd_pass_tc(onerf_ctx* ctx, const onerf_render_args* f, const onerf_render_bwd_args* b, const TrainWs& W,
                       int use_voxel, bool fine, char* ws, const float* pe, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const int fi = f->forward_instance ? 1 : 0;
  const int S = fine ? f->n_samples + f->n_importance : f->n_samples;
  const int R = f->n_rays;
  const int64_t B = (int64_t)R * S;
  const onerf_render_maps& m = fine ? f->fine : f->coarse;
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
  return ONERF_OK;
}

namespace {
// One input of an nn.Linear for the fp32 backward: In [B x width] (leading dimension ld) feeds the columns col..col+width
// of W; its gradient goes to d (leading dimension ld_d), accumulated or overwritten.  width 0 = absent (plain model).
struct LinearInput { const float* in; int ld; float* d; int ld_d, width, col, accumulate; };
}  // namespace

// fp32: per chunk of rays, the FFMA forward re-run with its activation dump, then every layer last to first
// (dZ = dH * act'(H), db += colsum dZ, dW += dZ^T In, dIn = dZ W) with the fp32 GEMM; per-ray-constant columns through
// per-ray sums; the encoding gradient scattered into the voxel table.  Accumulates into the reference-layout outputs.
static int bwd_pass_fp32(onerf_ctx* ctx, const onerf_render_args* f, const onerf_render_bwd_args* b, const TrainWs& W,
                         int use_voxel, bool fine, char* ws, const float* pe, void* stream) {
  const int fi = f->forward_instance ? 1 : 0;
  const int S = fine ? f->n_samples + f->n_importance : f->n_samples;
  const int N = f->n_rays;
  const float* z = fine ? f->fine.z_vals : f->coarse.z_vals;
  const void* packed = fine ? f->packed_fine : f->packed_coarse;
  const float* const* Wref = fine ? b->W_fine : b->W_coarse;
  float* const* dW = fine ? b->dW_fine : b->dW_coarse;
  float* const* db = fine ? b->db_fine : b->db_coarse;
  const float* dscene = reinterpret_cast<const float*>(ws + W.dscene);
  const float* dobj = reinterpret_cast<const float*>(ws + W.dobj);
  auto buf = [&](int64_t off) { return reinterpret_cast<float*>(ws + off); };
  float* act[17];
  for (int i = 0; i < 17; ++i) act[i] = buf(W.act[i]);
  float *X = act[0], *dX = buf(W.dX), *bufA = buf(W.bufA), *bufB = buf(W.bufB), *dA = buf(W.dA), *rs = buf(W.rs);
  float *field_s = buf(W.field_s), *field_o = buf(W.field_o);
  // reference input widths: scene input [voxel PE | xyz PE] or [xyz PE], object voxel block, object input [.. | code];
  // X holds the scene input at column 0 and the object voxel block at column 272
  const int xin = use_voxel ? 271 : 63, ovx = use_voxel ? 104 : 0, oin = xin + ovx + ONERF_NCODE, KO = use_voxel ? 384 : 64;
  const int in_width[ONERF_N_LINEAR] = {xin, 256, 256, 256, xin + 256, 256, 256, 256, 256, 256, 256 + 27, 128,
                                        oin, 128, oin + 128, 128, 128, 128, 128 + 27, 64};
  const int chunk = onerf_fp32_chunk_rays(N, S);
  int rc;
  for (int r0 = 0; r0 < N; r0 += chunk) {
    const int R = N - r0 < chunk ? N - r0 : chunk;
    const int B = R * S;
    const float* rays_c = f->rays + (int64_t)r0 * 8;
    const float* z_c = z + (int64_t)r0 * S;
    const float* codes_c = fi ? f->codes + (int64_t)r0 * ONERF_NCODE : nullptr;
    const float* pe_c = pe + (int64_t)r0 * 27;
    // layer idx: colsum, then dW for every input, then dIn for every input (in that order)
    auto linear = [&](const float* dZ, int ldz, int n_out, int idx, std::initializer_list<LinearInput> inputs) {
      int rc = onerf_colsum(ctx, dZ, ldz, B, n_out, db[idx], stream);
      for (const LinearInput& i : inputs)
        if (rc == ONERF_OK && i.width)
          rc = onerf_gemm(ctx, dZ, ldz, 1, i.in, i.ld, dW[idx] + i.col, in_width[idx], n_out, i.width, B, 1, stream);
      for (const LinearInput& i : inputs)
        if (rc == ONERF_OK && i.width)
          rc = onerf_gemm(ctx, dZ, ldz, 0, Wref[idx] + i.col, in_width[idx], i.d, i.ld_d, B, i.width, n_out, i.accumulate, stream);
      return rc;
    };
    // columns col..col+width of W[idx] fed by a per-ray constant [R x width]: dW += (sum over the ray's samples of dZ)^T
    // per_ray, and d_per_ray += (sum dZ) W
    auto ray_columns = [&](const float* dZ, int n_out, int idx, int col, const float* per_ray, int width, float* d_per_ray) {
      int rc = onerf_segment_sum(ctx, dZ, 256, rs, 128, R, S, n_out, stream);
      if (rc == ONERF_OK)
        rc = onerf_gemm(ctx, rs, 128, 1, per_ray, width, dW[idx] + col, in_width[idx], n_out, width, R, 1, stream);
      if (rc == ONERF_OK && d_per_ray)
        rc = onerf_gemm(ctx, rs, 128, 0, Wref[idx] + col, in_width[idx], d_per_ray, width, R, width, n_out, 1, stream);
      return rc;
    };
    // forward re-run with the activation dump: [0] X, [1..8] scene hidden, [9] final, [10] dir, [11..14] object hidden,
    // [15] object final, [16] object dir
    onerf_field_args a;
    memset(&a, 0, sizeof(a));
    a.rays = rays_c; a.z = z_c; a.z_stride = S; a.codes = codes_c;
    a.n_rays = R; a.n_samples = S;
    a.grid = f->grid; a.packed = packed;
    a.want_scene = 1; a.want_object = fi; a.precision = ONERF_PREC_FP32;
    a.scene_out = field_s; a.obj_out = fi ? field_o : nullptr; a.out_stride = S;
    a.ray_const = buf(W.ray_const);
    a.activations = act;
    TRY(onerf_field_fwd(ctx, &a, stream));
    ONERF_CUDA(cudaMemsetAsync(dX, 0, (size_t)B * KO * sizeof(float), (cudaStream_t)stream));
    // scene branch (models/nerf_model.py:97-121)
    TRY(onerf_head_bwd(ctx, dscene + (int64_t)r0 * S * 4, field_s, dA, B, stream));
    TRY(linear(dA, 4, 3, 11, {{act[10], 128, bufA, 256, 128, 0, 0}}));                 // rgb head, input = dir layer
    TRY(onerf_leaky_bwd(ctx, bufA, 256, act[10], 128, B, 128, stream));
    TRY(linear(bufA, 256, 128, 10, {{act[9], 256, bufB, 256, 256, 0, 0}}));            // dir layer: [final 256 | dir 27]
    TRY(ray_columns(bufA, 128, 10, 256, pe_c, 27, nullptr));
    TRY(linear(bufB, 256, 256, 9, {{act[8], 256, bufA, 256, 256, 0, 0}}));             // final layer, no activation
    TRY(linear(dA + 3, 4, 1, 8, {{act[8], 256, bufA, 256, 256, 0, 1}}));               // sigma head adds to d(h8)
    float *dH = bufA, *other = bufB;
    for (int l = 7; l >= 0; --l) {
      TRY(onerf_leaky_bwd(ctx, dH, 256, act[1 + l], 256, B, 256, stream));
      if (l == 0)
        TRY(linear(dH, 256, 256, 0, {{X, KO, dX, KO, xin, 0, 1}}));
      else if (l == 4)                                                                  // skip: [xyz input | h4]
        TRY(linear(dH, 256, 256, 4, {{X, KO, dX, KO, xin, 0, 1}, {act[4], 256, other, 256, 256, xin, 0}}));
      else
        TRY(linear(dH, 256, 256, l, {{act[l], 256, other, 256, 256, 0, 0}}));
      float* t = dH; dH = other; other = t;
    }
    // object branch (models/nerf_model.py:123-152)
    if (fi) {
      TRY(onerf_head_bwd(ctx, dobj + (int64_t)r0 * S * 4, field_o, dA, B, stream));
      TRY(linear(dA, 4, 3, 19, {{act[16], 64, bufA, 256, 64, 0, 0}}));
      TRY(onerf_leaky_bwd(ctx, bufA, 256, act[16], 64, B, 64, stream));
      TRY(linear(bufA, 256, 64, 18, {{act[15], 128, bufB, 256, 128, 0, 0}}));
      TRY(ray_columns(bufA, 64, 18, 128, pe_c, 27, nullptr));
      TRY(linear(bufB, 256, 128, 17, {{act[14], 128, bufA, 256, 128, 0, 0}}));
      TRY(linear(dA + 3, 4, 1, 16, {{act[14], 128, bufA, 256, 128, 0, 1}}));
      float* d_codes = b->d_codes ? b->d_codes + (int64_t)r0 * ONERF_NCODE : nullptr;
      dH = bufA; other = bufB;
      for (int l = 3; l >= 0; --l) {
        TRY(onerf_leaky_bwd(ctx, dH, 256, act[11 + l], 128, B, 128, stream));
        if (l == 0 || l == 2) {                                     // [xyz input | voxel block | code | h2 (layer 2 only)]
          const LinearInput x = {X, KO, dX, KO, xin, 0, 1}, vox = {X + 272, KO, dX + 272, KO, ovx, xin, 1};
          if (l == 2) TRY(linear(dH, 256, 128, 14, {x, vox, {act[12], 128, other, 256, 128, oin, 0}}));
          else TRY(linear(dH, 256, 128, 12, {x, vox}));
          TRY(ray_columns(dH, 128, 12 + l, xin + ovx, codes_c, ONERF_NCODE, d_codes));
        } else {
          TRY(linear(dH, 256, 128, 12 + l, {{act[10 + l], 128, other, 256, 128, 0, 0}}));
        }
        float* t = dH; dH = other; other = t;
      }
    }
    // encoding (models/embedding_helper.py:354-409)
    if (b->table_grad) TRY(onerf_encode_bwd(ctx, f->grid, rays_c, z_c, R, S, X, dX, KO, 0, B, b->table_grad, stream));
  }
  return ONERF_OK;
}
#undef TRY

static int check_bwd_args(const onerf_render_args* f, const onerf_render_bwd_args* b) {
  ONERF_CHECK_ARG(f->train_ws, "the forward was not run with a training workspace");
  ONERF_CHECK_ARG(f->precision == ONERF_PREC_FP32 || f->precision == ONERF_PREC_BF16, "unknown precision");
  ONERF_CHECK_ARG(b->W_coarse && b->dW_coarse && b->db_coarse, "null coarse gradient arguments");
  ONERF_CHECK_ARG(f->n_importance == 0 || (b->W_fine && b->dW_fine && b->db_fine), "null fine gradient arguments");
  const int use_voxel = onerf_train_use_voxel(f);
  ONERF_CHECK_ARG(use_voxel || !b->table_grad, "table_grad given for the plain-PE model, which has no voxel table");
  ONERF_CHECK_ARG(!b->table_grad || onerf_aligned16(b->table_grad), "table_grad misaligned");
  return ONERF_OK;
}

// The backward of both passes, fine first as autograd runs it.  step == NULL: each pass starts with the compositing
// backward of b's map gradients; otherwise the training step's compositing kernels have already written the field
// gradients (fine pass at W.dscene / W.dobj, coarse pass at step->dscene_c / dobj_c) and the field backward starts there.
static int render_bwd(onerf_ctx* ctx, const onerf_render_args* f, const onerf_render_bwd_args* b, const TrainWs& W,
                      const TrainStepWs* step, void* stream) {
  const int use_voxel = onerf_train_use_voxel(f);
  char* ws = reinterpret_cast<char*>(f->train_ws);
  float* pe = reinterpret_cast<float*>(ws + W.pe);
  int rc = onerf_dir_encode(ctx, f->rays, f->n_rays, pe, stream);
  const auto field_bwd = f->precision == ONERF_PREC_BF16 ? bwd_pass_tc : bwd_pass_fp32;
  for (const bool fine : {true, false}) {
    if (rc != ONERF_OK || (fine && f->n_importance == 0)) continue;
    TrainWs Wp = W;
    if (!step) rc = composite_bwd_pass(ctx, f, b, W, fine, ws, stream);
    else if (!fine) { Wp.dscene = step->dscene_c; Wp.dobj = step->dobj_c; }
    if (rc == ONERF_OK) rc = field_bwd(ctx, f, b, Wp, use_voxel, fine, ws, pe, stream);
  }
  return rc;
}

extern "C" int onerf_render_rays_bwd(onerf_ctx* ctx, const onerf_render_args* f, const onerf_render_bwd_args* b, void* stream) {
  ONERF_CHECK_ARG(ctx && f && b, "null argument");
  int rc = check_bwd_args(f, b);
  if (rc != ONERF_OK) return rc;
  const TrainWs W = onerf_make_train_ws(f->precision, onerf_train_use_voxel(f), f->n_rays, f->n_samples, f->n_importance);
  if (f->train_ws_bytes < (size_t)W.total) {
    onerf_set_error("onerf_render_rays_bwd: training workspace too small (%zu < %lld)", f->train_ws_bytes, (long long)W.total);
    return ONERF_ERR_WORKSPACE;
  }
  if (f->n_rays == 0) return ONERF_OK;
  return render_bwd(ctx, f, b, W, nullptr, stream);
}

// ---- the training step ----
extern "C" size_t onerf_train_step_workspace_bytes(int precision, int use_voxel, int n_rays, int n_samples, int n_importance) {
  if (precision != ONERF_PREC_FP32 && precision != ONERF_PREC_BF16) return 0;
  if (n_rays < 0 || n_samples < 1 || n_importance < 0) return 0;
  const TrainWs W = onerf_make_train_ws(precision, use_voxel ? 1 : 0, n_rays, n_samples, n_importance);
  return (size_t)onerf_make_train_step_ws(W, n_rays, n_samples).total;
}

static int train_step(onerf_ctx* ctx, const onerf_render_args* f, const onerf_loss_args* l, const onerf_render_bwd_args* b,
                      float* psnr_out, uint64_t* seed_dev, void* stream) {
  ONERF_CHECK_ARG(ctx && f && l && b && psnr_out, "null argument");
  int rc = check_bwd_args(f, b);
  if (rc != ONERF_OK) return rc;
  ONERF_CHECK_ARG(f->n_rays > 0 && l->n_rays == f->n_rays, "n_rays must be positive and equal in the render and loss arguments");
  ONERF_CHECK_ARG(f->forward_instance, "the loss needs the object branch's maps (forward_instance)");
  ONERF_CHECK_ARG(l->has_fine == (f->n_importance > 0 ? 1 : 0), "has_fine must say whether there is a fine pass");
  ONERF_CHECK_ARG(l->rgbs && l->depths && l->valid_mask && l->instance_mask && l->instance_mask_weight, "null batch buffer");
  ONERF_CHECK_ARG(l->loss_sum_out && l->terms_out && l->present_out, "null loss output");
  ONERF_UNSUPPORTED(f->n_samples + f->n_importance > 2048, "S > 2048");
  ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(f->train_ws) & 1023u) == 0, "train_ws must be 1024-byte aligned");
  const TrainWs W = onerf_make_train_ws(f->precision, onerf_train_use_voxel(f), f->n_rays, f->n_samples, f->n_importance);
  const TrainStepWs T = onerf_make_train_step_ws(W, f->n_rays, f->n_samples);
  if (f->train_ws_bytes < (size_t)T.total) {
    onerf_set_error("onerf_train_step: training workspace too small (%zu < %lld)", f->train_ws_bytes, (long long)T.total);
    return ONERF_ERR_WORKSPACE;
  }
  double* acc = reinterpret_cast<double*>(reinterpret_cast<char*>(f->train_ws) + T.loss);
  ONERF_CUDA(cudaMemsetAsync(acc, 0, ONERF_STEP_LOSS_BYTES, (cudaStream_t)stream));
  rc = onerf_launch_batch_stats(ctx, l, acc, (cudaStream_t)stream);
  if (rc != ONERF_OK) return rc;
  onerf_step_composite step;
  memset(&step, 0, sizeof(step));
  step.loss = *l;
  step.acc = acc;
  step.psnr_out = psnr_out;
  // the finalizing compositing kernel advances *seed_dev: the field backward draws nothing
  rc = onerf_render_fwd_impl(ctx, f, &step, seed_dev, stream);
  if (rc != ONERF_OK) return rc;
  return render_bwd(ctx, f, b, W, &T, stream);
}

extern "C" int onerf_train_step(onerf_ctx* ctx, const onerf_render_args* f, const onerf_loss_args* l,
                                const onerf_render_bwd_args* b, float* psnr_out, void* stream) {
  return train_step(ctx, f, l, b, psnr_out, nullptr, stream);
}

extern "C" int onerf_train_step_dseed(onerf_ctx* ctx, const onerf_render_args* f, const onerf_loss_args* l,
                                      const onerf_render_bwd_args* b, float* psnr_out, uint64_t* seed_dev, void* stream) {
  ONERF_CHECK_ARG(seed_dev, "null seed_dev");
  ONERF_CHECK_ARG((reinterpret_cast<uintptr_t>(seed_dev) & 7u) == 0, "seed_dev must be 8-byte aligned");
  return train_step(ctx, f, l, b, psnr_out, seed_dev, stream);
}
