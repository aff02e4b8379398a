// Held-out geometry metrics (include/onerf_ext.h: onerf_depth_metrics, onerf_mask_metrics and their _finalize): the
// depth errors of a frame's scene column and of each object column, and one object's opacity-versus-mask agreement,
// accumulated in fp64.
//
// Both kernels are one grid-stride pass over the pixels, about 15 bytes read per pixel for the depth kernel.  A depth
// warp walks 32 consecutive pixels at a time, so every lane runs the same number of iterations and the warp-wide votes
// and shuffles see all 32 lanes.  The scene column and the mask sums stay in registers until the end; the depth
// kernel's object columns are summed over the warp per distinct column and kept in a per-warp shared-memory slice, so
// no shared atomics are needed (with per-lane atomics, the warps that mix object pixels with pixels without depth, most
// of them in a frame with scattered missing depths, serialised on the same addresses).  Each CTA then adds every
// non-zero sum to the record with one fp64 atomicAdd.
#include <cmath>

#include "common.cuh"
#include "../../include/onerf_ext.h"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kCtasPerSm = 4;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kDR = ONERF_DEPTH_RECORD, kMR = ONERF_MASK_RECORD;

struct DepthParams {
  int64_t n;
  int n_ids;
  const float* pred_scene;
  const float* pred_object;
  const float* gt;
  const uint8_t* valid;
  const uint16_t* labels;
  double scale, d_min, d_max;
  double* record;
  int ids[ONERF_METRICS_MAX_IDS];
};

struct MaskParams {
  int64_t n;
  const float* opacity;
  const uint8_t* valid;
  const uint16_t* labels;
  int id;
  float threshold;
  double* record;              // the object's row
};

// The eight per-pixel terms of one column (header): d = clamp(pred s, d_min, d_max) with NaN kept, g = gt s > 0.
__device__ __forceinline__ void depth_terms(float pred, double g, double log_g, const DepthParams& a, double v[kDR]) {
  double d = (double)pred * a.scale;
  d = isnan(d) ? d : fmin(fmax(d, a.d_min), a.d_max);
  const double e = d - g, q = d / g, qi = g / d;
  const double r = q > qi ? q : qi;                      // max(d / g, g / d), NaN when d is
  const double l = log(d) - log_g;
  v[0] = 1.0;
  v[1] = fabs(e) / g;
  v[2] = e * e / g;
  v[3] = e * e;
  v[4] = l * l;
  // 1.25, 1.25^2 and 1.25^3 are exact in binary
  v[5] = isnan(r) ? r : (r < 1.25 ? 1.0 : 0.0);
  v[6] = isnan(r) ? r : (r < 1.5625 ? 1.0 : 0.0);
  v[7] = isnan(r) ? r : (r < 1.953125 ? 1.0 : 0.0);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

__global__ void __launch_bounds__(kThreads) depth_metrics_kernel(DepthParams a) {
  constexpr int kRow = (ONERF_METRICS_MAX_IDS + 1) * kDR;
  __shared__ int s_ids[ONERF_METRICS_MAX_IDS];
  __shared__ double s_acc[kWarps][kRow];                   // one slice per warp: written by its lane 0 only
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, n_sums = (a.n_ids + 1) * kDR;
  for (int i = t; i < kWarps * kRow; i += kThreads) (&s_acc[0][0])[i] = 0.0;
  if (t < a.n_ids) s_ids[t] = a.ids[t];
  __syncthreads();

  double acc[kDR];
#pragma unroll
  for (int j = 0; j < kDR; ++j) acc[j] = 0.0;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t base = (int64_t)blockIdx.x * kThreads + warp * 32; base < a.n; base += stride) {
    const int64_t p = base + lane;
    double g = 0.0;
    bool in = p < a.n && (a.valid == nullptr || __ldg(a.valid + p) != 0);
    if (in) {
      const float gt = __ldg(a.gt + p);
      in = gt > 0.0f;
      g = (double)gt * a.scale;
    }
    int col = 0;                                          // the pixel's object column, 0: none
    if (in && a.n_ids > 0) {
      const int lab = __ldg(a.labels + p);
      for (int k = 0; k < a.n_ids; ++k)
        if (s_ids[k] == lab) {
          col = k + 1;
          break;
        }
    }
    double v[kDR];
    if (in) {
      const double log_g = log(g);
      depth_terms(__ldg(a.pred_scene + p), g, log_g, a, v);
#pragma unroll
      for (int j = 0; j < kDR; ++j) acc[j] += v[j];
      if (col > 0) depth_terms(__ldg(a.pred_object + p), g, log_g, a, v);
    }
    // object columns: one warp sum per distinct column among the 32 pixels (one inside an object, two or three on its
    // edge), added by lane 0 to the warp's slice
    for (unsigned pending = __ballot_sync(kFull, col > 0); pending;) {
      const int c = __shfl_sync(kFull, col, __ffs(pending) - 1);
      const bool mine = col == c;
#pragma unroll
      for (int j = 0; j < kDR; ++j) {
        const double s = warp_sum_d(mine ? v[j] : 0.0);
        if (lane == 0) s_acc[warp][c * kDR + j] += s;
      }
      pending &= ~__ballot_sync(kFull, mine);
    }
  }
#pragma unroll
  for (int j = 0; j < kDR; ++j) {
    const double s = warp_sum_d(acc[j]);
    if (lane == 0) s_acc[warp][j] = s;
  }
  __syncthreads();
  for (int i = t; i < n_sums; i += kThreads) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += s_acc[w][i];
    if (s != 0.0) atomicAdd(a.record + i, s);             // NaN is != 0 and is added
  }
}

__global__ void __launch_bounds__(kThreads) mask_metrics_kernel(MaskParams a) {
  __shared__ double s_red[kMR][kWarps];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  double acc[kMR] = {0.0, 0.0, 0.0, 0.0};
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t p = (int64_t)blockIdx.x * kThreads + t; p < a.n; p += stride) {
    if (a.valid != nullptr && __ldg(a.valid + p) == 0) continue;
    const float o = __ldg(a.opacity + p);
    const bool G = (int)__ldg(a.labels + p) == a.id, P = o >= a.threshold;
    acc[0] += (P && G) ? 1.0 : 0.0;
    acc[1] += (P || G) ? 1.0 : 0.0;
    acc[2] += fabs((double)o - (G ? 1.0 : 0.0));
    acc[3] += 1.0;
  }
#pragma unroll
  for (int j = 0; j < kMR; ++j) {
    const double s = warp_sum_d(acc[j]);
    if (lane == 0) s_red[j][warp] = s;
  }
  __syncthreads();
  if (t < kMR) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += s_red[t][w];
    if (s != 0.0) atomicAdd(a.record + t, s);
  }
}

// record -> the seven depth metrics of row `slot` for every column, then the record back to zero for the next frame
__global__ void depth_finalize_kernel(double* record, int n_cols, float* out, int slot) {
  const int col = threadIdx.x;
  if (col >= n_cols) return;
  double* r = record + col * kDR;
  const double n = r[0];
  if (out) {
    float* o = out + ((int64_t)slot * n_cols + col) * ONERF_DEPTH_METRICS;
    o[0] = (float)(r[1] / n);
    o[1] = (float)(r[2] / n);
    o[2] = (float)sqrt(r[3] / n);
    o[3] = (float)sqrt(r[4] / n);
    o[4] = (float)(r[5] / n);
    o[5] = (float)(r[6] / n);
    o[6] = (float)(r[7] / n);
  }
  for (int j = 0; j < kDR; ++j) r[j] = 0.0;
}

// record -> iou / opacity_l1 of row `slot` for every object, then the record back to zero
__global__ void mask_finalize_kernel(double* record, int n_ids, float* iou_out, float* l1_out, int slot) {
  const int k = threadIdx.x;
  if (k >= n_ids) return;
  double* r = record + k * kMR;
  if (iou_out) iou_out[(int64_t)slot * n_ids + k] = (float)(r[0] / r[1]);
  if (l1_out) l1_out[(int64_t)slot * n_ids + k] = (float)(r[2] / r[3]);
  for (int j = 0; j < kMR; ++j) r[j] = 0.0;
}

int grid_size(const onerf_ctx* ctx, int64_t n) {
  const int64_t ctas = (n + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)kCtasPerSm * (ctx->num_sms > 0 ? ctx->num_sms : 1);
  return (int)(ctas < cap ? ctas : cap);
}

#define GEOM_CHECK(cond, msg)                 \
  do {                                        \
    if (!(cond)) {                            \
      onerf_set_error("%s: %s", fn, msg);     \
      return ONERF_ERR_BAD_ARG;               \
    }                                         \
  } while (0)

// The frame shape and record refusals both accumulating entries share.
int check_frame(const char* fn, int H, int W, const double* record) {
  GEOM_CHECK(H >= 1 && W >= 1 && (int64_t)H * W < (int64_t(1) << 40), "H and W must be >= 1 and H * W < 2^40");
  GEOM_CHECK(record && onerf_aligned8(record), "record must be a non-null 8-byte aligned buffer");
  return ONERF_OK;
}

int check_depth(const char* fn, onerf_ctx* ctx, const onerf_depth_metrics_args* a) {
  GEOM_CHECK(ctx && a, "null argument");
  GEOM_CHECK(a->n_ids >= 0 && a->n_ids <= ONERF_METRICS_MAX_IDS, "n_ids outside [0, ONERF_METRICS_MAX_IDS]");
  const int rc = check_frame(fn, a->H, a->W, a->record);
  if (rc != ONERF_OK) return rc;
  GEOM_CHECK(std::isfinite(a->scale) && a->scale > 0.0, "scale must be finite and > 0");
  GEOM_CHECK(std::isfinite(a->d_min) && std::isfinite(a->d_max), "d_min and d_max must be finite");
  GEOM_CHECK(a->d_min > 0.0 && a->d_min < a->d_max, "the depth range needs 0 < d_min < d_max");
  GEOM_CHECK(a->pred_scene && a->gt, "null pred_scene or gt");
  GEOM_CHECK(a->n_ids == 0 || (a->pred_object && a->labels), "object columns need pred_object and labels");
  GEOM_CHECK(a->n_ids == 0 || a->ids_host, "null ids_host with n_ids > 0");
  GEOM_CHECK(onerf_aligned4(a->pred_scene) && onerf_aligned4(a->pred_object) && onerf_aligned4(a->gt) &&
                 (reinterpret_cast<uintptr_t>(a->labels) & 1u) == 0,
             "misaligned depth or label buffer");
  for (int i = 0; i < a->n_ids; ++i) {
    GEOM_CHECK(a->ids_host[i] >= 0 && a->ids_host[i] <= 0xFFFF, "an id outside [0, 65535] matches no 16-bit label");
    for (int j = 0; j < i; ++j) GEOM_CHECK(a->ids_host[j] != a->ids_host[i], "ids must be distinct");
  }
  return ONERF_OK;
}

int check_mask(const char* fn, onerf_ctx* ctx, const onerf_mask_metrics_args* a) {
  GEOM_CHECK(ctx && a, "null argument");
  GEOM_CHECK(a->n_ids >= 1 && a->n_ids <= ONERF_METRICS_MAX_IDS, "n_ids outside [1, ONERF_METRICS_MAX_IDS]");
  GEOM_CHECK(a->column >= 0 && a->column < a->n_ids, "column outside [0, n_ids)");
  const int rc = check_frame(fn, a->H, a->W, a->record);
  if (rc != ONERF_OK) return rc;
  GEOM_CHECK(a->id >= 0 && a->id <= 0xFFFF, "an id outside [0, 65535] matches no 16-bit label");
  GEOM_CHECK(std::isfinite(a->threshold), "threshold must be finite");
  GEOM_CHECK(a->opacity && a->labels, "null opacity or labels");
  GEOM_CHECK(onerf_aligned4(a->opacity) && (reinterpret_cast<uintptr_t>(a->labels) & 1u) == 0,
             "misaligned opacity or label buffer");
  return ONERF_OK;
}

int check_finalize(const char* fn, onerf_ctx* ctx, const void* a, int n_ids, int min_ids, const double* record,
                   int slot, const float* out0, const float* out1) {
  GEOM_CHECK(ctx && a, "null argument");
  GEOM_CHECK(n_ids >= min_ids && n_ids <= ONERF_METRICS_MAX_IDS, "n_ids outside the entry's range");
  GEOM_CHECK(record && onerf_aligned8(record), "record must be a non-null 8-byte aligned buffer");
  GEOM_CHECK(slot >= 0, "slot must be >= 0");
  GEOM_CHECK(onerf_aligned4(out0) && onerf_aligned4(out1), "misaligned output");
  return ONERF_OK;
}

#undef GEOM_CHECK

}  // namespace

extern "C" int onerf_depth_metrics(onerf_ctx* ctx, const onerf_depth_metrics_args* a, void* stream) {
  const int rc = check_depth(__func__, ctx, a);
  if (rc != ONERF_OK) return rc;
  DepthParams p;
  p.n = (int64_t)a->H * a->W;
  p.n_ids = a->n_ids;
  p.pred_scene = a->pred_scene;
  p.pred_object = a->pred_object;
  p.gt = a->gt;
  p.valid = a->valid;
  p.labels = a->labels;
  p.scale = a->scale;
  p.d_min = a->d_min;
  p.d_max = a->d_max;
  p.record = a->record;
  for (int i = 0; i < ONERF_METRICS_MAX_IDS; ++i) p.ids[i] = i < a->n_ids ? a->ids_host[i] : -1;
  depth_metrics_kernel<<<grid_size(ctx, p.n), kThreads, 0, (cudaStream_t)stream>>>(p);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_depth_metrics_finalize(onerf_ctx* ctx, const onerf_depth_metrics_args* a, int slot, void* stream) {
  const int rc = check_finalize(__func__, ctx, a, a ? a->n_ids : 0, 0, a ? a->record : nullptr, slot,
                                a ? a->out : nullptr, nullptr);
  if (rc != ONERF_OK) return rc;
  depth_finalize_kernel<<<1, ONERF_METRICS_MAX_IDS + 1, 0, (cudaStream_t)stream>>>(a->record, a->n_ids + 1, a->out,
                                                                                  slot);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_mask_metrics(onerf_ctx* ctx, const onerf_mask_metrics_args* a, void* stream) {
  const int rc = check_mask(__func__, ctx, a);
  if (rc != ONERF_OK) return rc;
  MaskParams p;
  p.n = (int64_t)a->H * a->W;
  p.opacity = a->opacity;
  p.valid = a->valid;
  p.labels = a->labels;
  p.id = a->id;
  p.threshold = a->threshold;
  p.record = a->record + (int64_t)a->column * kMR;
  mask_metrics_kernel<<<grid_size(ctx, p.n), kThreads, 0, (cudaStream_t)stream>>>(p);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_mask_metrics_finalize(onerf_ctx* ctx, const onerf_mask_metrics_args* a, int slot, void* stream) {
  const int rc = check_finalize(__func__, ctx, a, a ? a->n_ids : 0, 1, a ? a->record : nullptr, slot,
                                a ? a->iou_out : nullptr, a ? a->opacity_l1_out : nullptr);
  if (rc != ONERF_OK) return rc;
  mask_finalize_kernel<<<1, ONERF_METRICS_MAX_IDS, 0, (cudaStream_t)stream>>>(a->record, a->n_ids, a->iou_out,
                                                                             a->opacity_l1_out, slot);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
