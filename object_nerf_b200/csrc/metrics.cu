// Held-out image metrics (include/onerf_ext.h: onerf_image_metrics, onerf_image_metrics_finalize): the masked PSNR and
// SSIM of a frame's scene column and of each object column, accumulated in fp64.
//
// One CTA owns a kTileX x kTileY tile of output pixels and one column (blockIdx.z).  It stages the column's mask for the
// tile plus its reflect halo once, then per channel: the masked prediction and ground truth of tile plus halo into shared
// memory, the horizontal Gaussian pass of the five window sums (p, g, p^2, g^2, p g) in fp64 for every halo row, the
// vertical pass and ssim_map for each output pixel in the mask.  The squared errors, the clamped ssim_map values and the
// pixel count are reduced within warps and added to the column's record with one fp64 atomicAdd per CTA per sum.
#include "common.cuh"
#include "../../include/onerf_ext.h"

namespace {

constexpr int kTileX = 32, kTileY = 16;
constexpr int kThreads = 256;
constexpr int kMaxR = ONERF_METRICS_MAX_WINDOW / 2;
constexpr int kExtX = kTileX + 2 * kMaxR, kExtY = kTileY + 2 * kMaxR;
constexpr double kC1 = 0.01 * 0.01, kC2 = 0.03 * 0.03;

struct MetricsParams {
  int H, W, r, n_cols;
  const float* pred_scene;
  const float* pred_object;
  const float* gt;
  const uint8_t* valid;
  const uint16_t* labels;
  double* record;
  int ids[ONERF_METRICS_MAX_IDS];
  double g1[ONERF_METRICS_MAX_WINDOW];
};

// F.pad(mode="reflect"): mirror without repeating the edge; one bounce suffices for i in [-r, n - 1 + r], r < n.  The
// rows and columns of a partial tile beyond that range feed only outputs outside the image: clamped into it, they are
// read but never used.
__device__ __forceinline__ int reflect(int i, int n) {
  i = i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i);
  return min(max(i, 0), n - 1);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kThreads) image_metrics_kernel(MetricsParams a) {
  __shared__ uint8_t s_m[kExtY * kExtX];
  __shared__ float s_p[kExtY * kExtX], s_g[kExtY * kExtX];
  __shared__ double s_h[5][kExtY * kTileX];
  __shared__ double s_red[3][kThreads / 32];
  const int col = blockIdx.z, r = a.r, ex = kTileX + 2 * r, ey = kTileY + 2 * r;
  const int x0 = blockIdx.x * kTileX, y0 = blockIdx.y * kTileY, t = threadIdx.x;
  const int id = col > 0 ? a.ids[col - 1] : -1;
  const float* pred = col > 0 ? a.pred_object : a.pred_scene;

  // the column's mask over tile plus halo (reflected coordinates); does any output pixel of the tile lie in it?
  int any = 0;
  for (int i = t; i < ey * ex; i += kThreads) {
    const int ty = i / ex, tx = i - ty * ex;
    const int y = reflect(y0 + ty - r, a.H), x = reflect(x0 + tx - r, a.W);
    const int64_t p = (int64_t)y * a.W + x;
    uint8_t m = a.valid ? (__ldg(a.valid + p) != 0) : 1;
    if (col > 0) m &= (int)__ldg(a.labels + p) == id ? 1 : 0;
    s_m[ty * kExtX + tx] = m;
    const int oy = y0 + ty - r, ox = x0 + tx - r;
    if (m && ty >= r && ty < r + kTileY && tx >= r && tx < r + kTileX && oy < a.H && ox < a.W) any = 1;
  }
  if (!__syncthreads_or(any)) return;

  double se = 0.0, ss = 0.0, cnt = 0.0;
  for (int c = 0; c < 3; ++c) {
    for (int i = t; i < ey * ex; i += kThreads) {
      const int ty = i / ex, tx = i - ty * ex;
      const int y = reflect(y0 + ty - r, a.H), x = reflect(x0 + tx - r, a.W);
      const int64_t p = ((int64_t)y * a.W + x) * 3 + c;
      const bool m = s_m[ty * kExtX + tx];
      s_p[ty * kExtX + tx] = m ? __ldg(pred + p) : 0.0f;
      s_g[ty * kExtX + tx] = m ? __ldg(a.gt + p) : 0.0f;
    }
    __syncthreads();
    // horizontal pass: every halo row, every output column
    for (int i = t; i < ey * kTileX; i += kThreads) {
      const int ty = i / kTileX, tx = i - ty * kTileX;
      double h0 = 0.0, h1 = 0.0, h2 = 0.0, h3 = 0.0, h4 = 0.0;
      for (int k = 0; k <= 2 * r; ++k) {
        const double w = a.g1[k];
        const double p = s_p[ty * kExtX + tx + k], g = s_g[ty * kExtX + tx + k];
        const double wp = w * p, wg = w * g;
        h0 += wp;
        h1 += wg;
        h2 = fma(wp, p, h2);
        h3 = fma(wg, g, h3);
        h4 = fma(wp, g, h4);
      }
      s_h[0][i] = h0; s_h[1][i] = h1; s_h[2][i] = h2; s_h[3][i] = h3; s_h[4][i] = h4;
    }
    __syncthreads();
    // vertical pass and ssim_map for the output pixels in the mask
    for (int i = t; i < kTileY * kTileX; i += kThreads) {
      const int ty = i / kTileX, tx = i - ty * kTileX;
      if (y0 + ty >= a.H || x0 + tx >= a.W || !s_m[(ty + r) * kExtX + tx + r]) continue;
      double v0 = 0.0, v1 = 0.0, v2 = 0.0, v3 = 0.0, v4 = 0.0;
      for (int k = 0; k <= 2 * r; ++k) {
        const double w = a.g1[k];
        const int j = (ty + k) * kTileX + tx;
        v0 = fma(w, s_h[0][j], v0);
        v1 = fma(w, s_h[1][j], v1);
        v2 = fma(w, s_h[2][j], v2);
        v3 = fma(w, s_h[3][j], v3);
        v4 = fma(w, s_h[4][j], v4);
      }
      const double spp = v2 - v0 * v0, sgg = v3 - v1 * v1, spg = v4 - v0 * v1;
      const double s = ((2.0 * v0 * v1 + kC1) * (2.0 * spg + kC2)) / ((v0 * v0 + v1 * v1 + kC1) * (spp + sgg + kC2));
      ss += fmin(fmax(s, 0.0), 1.0);
      const double d = (double)s_p[(ty + r) * kExtX + tx + r] - (double)s_g[(ty + r) * kExtX + tx + r];
      se = fma(d, d, se);
      if (c == 0) cnt += 1.0;
    }
    __syncthreads();
  }
  se = warp_sum_d(se);
  ss = warp_sum_d(ss);
  cnt = warp_sum_d(cnt);
  const int warp = t >> 5, lane = t & 31;
  if (lane == 0) {
    s_red[0][warp] = se;
    s_red[1][warp] = ss;
    s_red[2][warp] = cnt;
  }
  __syncthreads();
  if (t < 3) {
    double v = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) v += s_red[t][w];
    atomicAdd(a.record + col * 3 + t, v);
  }
}

// record -> psnr / ssim of row `slot`, then the record back to zero for the next frame
__global__ void metrics_finalize_kernel(double* record, int n_cols, float* psnr_out, float* ssim_out, int slot) {
  const int col = threadIdx.x;
  if (col >= n_cols) return;
  const double se = record[col * 3], ss = record[col * 3 + 1], n = 3.0 * record[col * 3 + 2];
  if (psnr_out) psnr_out[(int64_t)slot * n_cols + col] = (float)(-10.0 * log10(se / n));
  if (ssim_out) ssim_out[(int64_t)slot * n_cols + col] = (float)(ss / n);
  record[col * 3] = record[col * 3 + 1] = record[col * 3 + 2] = 0.0;
}

// The refusals both entries share.
int check_metrics(const char* fn, onerf_ctx* ctx, const onerf_metrics_args* a) {
#define METRICS_CHECK(cond, msg)                \
  do {                                          \
    if (!(cond)) {                              \
      onerf_set_error("%s: %s", fn, msg);       \
      return ONERF_ERR_BAD_ARG;                 \
    }                                           \
  } while (0)
  METRICS_CHECK(ctx && a, "null argument");
  METRICS_CHECK(a->window >= 1 && a->window <= ONERF_METRICS_MAX_WINDOW && (a->window & 1),
                "window must be odd and in [1, ONERF_METRICS_MAX_WINDOW]");
  METRICS_CHECK(a->n_ids >= 0 && a->n_ids <= ONERF_METRICS_MAX_IDS, "n_ids outside [0, ONERF_METRICS_MAX_IDS]");
  METRICS_CHECK(a->H > a->window / 2 && a->W > a->window / 2,
                "H and W must exceed window / 2 (reflect padding is undefined otherwise)");
  METRICS_CHECK((int64_t)a->H * a->W < (int64_t(1) << 40) && a->H <= 65535 * kTileY, "H * W must be < 2^40 and H <= 1048560");
  METRICS_CHECK(a->pred_scene && a->gt, "null pred_scene or gt");
  METRICS_CHECK(a->n_ids == 0 || (a->pred_object && a->labels), "object columns need pred_object and labels");
  METRICS_CHECK(a->n_ids == 0 || a->ids_host, "null ids_host with n_ids > 0");
  METRICS_CHECK(a->record && onerf_aligned8(a->record), "record must be a non-null 8-byte aligned buffer");
  METRICS_CHECK(onerf_aligned4(a->pred_scene) && onerf_aligned4(a->pred_object) && onerf_aligned4(a->gt) &&
                    (reinterpret_cast<uintptr_t>(a->labels) & 1u) == 0,
                "misaligned image buffer");
  for (int i = 0; i < a->n_ids; ++i)
    METRICS_CHECK(a->ids_host[i] >= 0 && a->ids_host[i] <= 0xFFFF, "an id outside [0, 65535] matches no 16-bit label");
  return ONERF_OK;
#undef METRICS_CHECK
}

}  // namespace

extern "C" int onerf_image_metrics(onerf_ctx* ctx, const onerf_metrics_args* a, void* stream) {
  const int rc = check_metrics(__func__, ctx, a);
  if (rc != ONERF_OK) return rc;
  MetricsParams p;
  p.H = a->H;
  p.W = a->W;
  p.r = a->window / 2;
  p.n_cols = a->n_ids + 1;
  p.pred_scene = a->pred_scene;
  p.pred_object = a->pred_object;
  p.gt = a->gt;
  p.valid = a->valid;
  p.labels = a->labels;
  p.record = a->record;
  for (int i = 0; i < ONERF_METRICS_MAX_IDS; ++i) p.ids[i] = i < a->n_ids ? a->ids_host[i] : -1;
  // g1[i] = exp(-(i - r)^2 / (2 sigma^2)) / sum, sigma = 1.5, in double on the host
  double sum = 0.0;
  for (int i = 0; i < ONERF_METRICS_MAX_WINDOW; ++i) {
    const double d = (double)(i - p.r);
    p.g1[i] = i < a->window ? exp(-d * d / (2.0 * 1.5 * 1.5)) : 0.0;
    sum += p.g1[i];
  }
  for (int i = 0; i < ONERF_METRICS_MAX_WINDOW; ++i) p.g1[i] /= sum;
  const dim3 grid((a->W + kTileX - 1) / kTileX, (a->H + kTileY - 1) / kTileY, p.n_cols);
  image_metrics_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(p);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_image_metrics_finalize(onerf_ctx* ctx, const onerf_metrics_args* a, int slot, void* stream) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  ONERF_CHECK_ARG(a->n_ids >= 0 && a->n_ids <= ONERF_METRICS_MAX_IDS, "n_ids outside [0, ONERF_METRICS_MAX_IDS]");
  ONERF_CHECK_ARG(a->record && onerf_aligned8(a->record), "record must be a non-null 8-byte aligned buffer");
  ONERF_CHECK_ARG(slot >= 0, "slot must be >= 0");
  ONERF_CHECK_ARG(onerf_aligned4(a->psnr_out) && onerf_aligned4(a->ssim_out), "misaligned output");
  metrics_finalize_kernel<<<1, ONERF_METRICS_MAX_IDS + 1, 0, (cudaStream_t)stream>>>(a->record, a->n_ids + 1,
                                                                                    a->psnr_out, a->ssim_out, slot);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
