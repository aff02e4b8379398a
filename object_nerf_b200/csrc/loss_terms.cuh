// Per-ray arithmetic of TotalLoss (models/losses.py:5-135) shared by the stand-alone loss kernels (loss.cu) and the
// fused compositing kernel of the training step (composite.cu): batch counts, squared errors and d(loss_sum)/d(map) of
// one ray.  The scene maps (rgb, depth) carry the color and depth terms, the object maps the other three.
#pragma once
#include "common.cuh"
#include "../../include/onerf_ext.h"

namespace loss_terms {

enum { T_COLOR = 0, T_DEPTH, T_OPACITY, T_ICOLOR, T_IDEPTH, N_TERMS };
// accumulators (doubles): [0..5) mask counts per term (elements of the masked mean), [5] number of targets > 0,
// [6..16) squared-error sums: term * 2 + (0 coarse / 1 fine)
enum { WS_COUNT = 0, WS_TPOS = 5, WS_SUM = 6, WS_DOUBLES = 16 };
// the validation record (onerf_validate_frame) is the accumulators followed by the validation PSNR's masked
// squared-error sum and element count (train.py:185-190, :220)
enum { VR_PSNR_SUM = WS_DOUBLES, VR_PSNR_COUNT, VR_DOUBLES };
static_assert(VR_DOUBLES == ONERF_VALIDATE_RECORD_DOUBLES, "record size declared in onerf_ext.h");

__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }

// what the batch says about one ray
struct Target {
  bool valid, inst, tpos;
  float t, w, rgb[3];
};

__device__ __forceinline__ Target load_target(const onerf_loss_args& a, int64_t r) {
  Target g;
  g.valid = a.valid_mask[r] != 0;
  g.inst = a.instance_mask[r] != 0;
  g.t = a.depths[r];
  g.w = a.instance_mask_weight[r];
  g.tpos = g.t > 0.0f;
  g.rgb[0] = a.rgbs[3 * r]; g.rgb[1] = a.rgbs[3 * r + 1]; g.rgb[2] = a.rgbs[3 * r + 2];
  return g;
}

// the ray's share of the counts acc[WS_COUNT .. WS_TPOS]: they depend on the batch only, never on the render
__device__ __forceinline__ void add_counts(const Target& g, double* acc) {
  if (g.tpos) acc[WS_TPOS] += 1.0;
  if (g.valid) {
    acc[WS_COUNT + T_COLOR] += 3.0;
    acc[WS_COUNT + T_OPACITY] += 1.0;
    if (g.tpos) acc[WS_COUNT + T_DEPTH] += 1.0;
    if (g.inst) acc[WS_COUNT + T_ICOLOR] += 3.0;
    if (g.inst && g.tpos) acc[WS_COUNT + T_IDEPTH] += 1.0;
  }
}

// squared errors of one pass's maps, added to sum[term * stride]
__device__ __forceinline__ void add_scene_sq(const Target& g, const float* rgb, float depth, double* sum, int stride) {
  if (!g.valid) return;
  const float e0 = rgb[0] - g.rgb[0], e1 = rgb[1] - g.rgb[1], e2 = rgb[2] - g.rgb[2];
  sum[stride * T_COLOR] += (double)(e0 * e0) + (double)(e1 * e1) + (double)(e2 * e2);
  if (g.tpos) { const float e = depth - g.t; sum[stride * T_DEPTH] += (double)(e * e); }
}

__device__ __forceinline__ void add_object_sq(const Target& g, float opacity, const float* rgb, float depth, double* sum,
                                              int stride) {
  if (!g.valid) return;
  { const float e = clamp01(opacity) - (g.inst ? 1.0f : 0.0f); sum[stride * T_OPACITY] += (double)(e * e * g.w); }
  if (g.inst) {
    const float e0 = rgb[0] - g.rgb[0], e1 = rgb[1] - g.rgb[1], e2 = rgb[2] - g.rgb[2];
    sum[stride * T_ICOLOR] += (double)(e0 * e0 * g.w) + (double)(e1 * e1 * g.w) + (double)(e2 * e2 * g.w);
    if (g.tpos) { const float e = depth - g.t; sum[stride * T_IDEPTH] += (double)(e * e * g.w); }
  }
}

// the validation PSNR's share of one ray: psnr = 0 (this pass is not the one measured), 1 + ONERF_PSNR_VALID_INSTANCE
// (mask = valid_mask * instance_mask) or 1 + ONERF_PSNR_ALL_RAYS (mask = None: every ray, valid or not)
__device__ __forceinline__ void add_psnr_sq(const Target& g, int psnr, const float* rgb, double* acc) {
  if (psnr == 0 || (psnr == 1 + ONERF_PSNR_VALID_INSTANCE && !(g.valid && g.inst))) return;
  const float e0 = rgb[0] - g.rgb[0], e1 = rgb[1] - g.rgb[1], e2 = rgb[2] - g.rgb[2];
  acc[0] += (double)(e0 * e0) + (double)(e1 * e1) + (double)(e2 * e2);
  acc[1] += 3.0;
}

// term present (the reference returns None otherwise): models/losses.py:13-14, :46-47, :51-52, :80-81
__device__ __forceinline__ bool term_present(const double* ws, int t) {
  switch (t) {
    case T_COLOR: return true;                                                   // never skipped (mean of an empty set = NaN)
    case T_DEPTH: return ws[WS_TPOS] > 0;                                        // skipped only if no target depth at all
    case T_OPACITY: return ws[WS_COUNT + T_OPACITY] > 0;
    case T_ICOLOR: return ws[WS_COUNT + T_ICOLOR] > 0;
    default: return ws[WS_TPOS] > 0 && ws[WS_COUNT + T_IDEPTH] > 0;
  }
}

// d(weighted mean)/d(squared error) = weight / count of every term, 0 where the term is skipped
__device__ __forceinline__ void grad_scales(const onerf_loss_args& a, const double* ws, float* scale) {
  const float wt[N_TERMS] = {a.color_weight, a.depth_weight, a.opacity_weight, a.instance_color_weight, a.instance_depth_weight};
#pragma unroll
  for (int t = 0; t < N_TERMS; ++t) scale[t] = term_present(ws, t) ? (float)((double)wt[t] / ws[WS_COUNT + t]) : 0.0f;
}

// d(loss_sum)/d(map) of one ray: scene rgb (3) and depth; object opacity, rgb (3) and depth
__device__ __forceinline__ void scene_grads(const Target& g, const float* rgb, float depth, const float* scale, float* gc,
                                            float& gd) {
  gc[0] = gc[1] = gc[2] = gd = 0.0f;
  if (!g.valid) return;
  gc[0] = 2.0f * (rgb[0] - g.rgb[0]) * scale[T_COLOR];
  gc[1] = 2.0f * (rgb[1] - g.rgb[1]) * scale[T_COLOR];
  gc[2] = 2.0f * (rgb[2] - g.rgb[2]) * scale[T_COLOR];
  if (g.tpos) gd = 2.0f * (depth - g.t) * scale[T_DEPTH];
}

__device__ __forceinline__ void object_grads(const Target& g, float o, const float* rgb, float depth, const float* scale,
                                             float& go, float* gi, float& gid) {
  go = gi[0] = gi[1] = gi[2] = gid = 0.0f;
  if (!g.valid) return;
  if (o >= 0.0f && o <= 1.0f) go = 2.0f * (o - (g.inst ? 1.0f : 0.0f)) * g.w * scale[T_OPACITY];   // clamp backward
  if (g.inst) {
    gi[0] = 2.0f * (rgb[0] - g.rgb[0]) * g.w * scale[T_ICOLOR];
    gi[1] = 2.0f * (rgb[1] - g.rgb[1]) * g.w * scale[T_ICOLOR];
    gi[2] = 2.0f * (rgb[2] - g.rgb[2]) * g.w * scale[T_ICOLOR];
    if (g.tpos) gid = 2.0f * (depth - g.t) * g.w * scale[T_IDEPTH];
  }
}

// loss_sum, the five unweighted terms and the present flags from the accumulators (one thread)
__device__ __forceinline__ void write_outputs(const onerf_loss_args& a, const double* ws) {
  const float wt[N_TERMS] = {a.color_weight, a.depth_weight, a.opacity_weight, a.instance_color_weight, a.instance_depth_weight};
  double total = 0.0;
  for (int t = 0; t < N_TERMS; ++t) {
    const bool present = term_present(ws, t);
    // mean over the mask in fp32 like torch (sum / count), coarse + fine, times the weight
    float v = 0.0f;
    if (present) {
      v = (float)(ws[WS_SUM + 2 * t] / ws[WS_COUNT + t]);
      if (a.has_fine) v += (float)(ws[WS_SUM + 2 * t + 1] / ws[WS_COUNT + t]);
    }
    a.terms_out[t] = v;                     // unweighted, as the reference's loss_dict (:129-131)
    a.present_out[t] = present ? 1 : 0;
    if (present) total += (double)(wt[t] * v);
  }
  *a.loss_sum_out = (float)total;
}

}  // namespace loss_terms
