// Every object rendered inside its own box from a camera (onerf_render_boxes, include/onerf_ext.h): the object
// evaluation of a use_bbox dataset, with work proportional to the pixels the boxes cover.  The rows are the (object,
// pixel) pairs of a tile, object-major.  Per chunk of rows: box-clipped rays and hit bits (rays.cu), then the rows that
// hit their box are listed in row order and their rays gathered (a three-kernel scan: per-block counts, block offsets,
// ordered writes).  Every map starts as (+0, +0, 1), what a missed row keeps.  Every later stage runs on the listed
// rows only and stops at the device-side count: coarse depths, code rows, per-ray constants, the object-only field, the object
// compositing with rays_in_bbox semantics (whose coarse weights feed the importance sampler), the fine pass.  Same
// arithmetic as onerf_render_rays_fwd for every stage a hit row goes through, so a hit row's maps are bit for bit that
// call's object maps.
#include <math.h>
#include <string.h>

#include <algorithm>

#include "composite_core.cuh"
#include "field_common.cuh"
#include "train_ws.h"
#include "../../include/onerf_ext.h"

namespace {

constexpr int kListThreads = 256, kListIters = 16;
constexpr int kListRows = kListThreads * kListIters;   // rows one block of the list kernels covers

// Every entry of one (T,K) map set as a missed row leaves it: opacity +0, depth +0, rgb 1.  Runs once per call, before
// any chunk; the hit rows' compositing overwrites its own entries afterwards.  Coalesced, where writing each missed
// row's entries from its own (object-major) row would scatter them K entries apart.
__global__ void __launch_bounds__(256)
fill_missed_kernel(float* __restrict__ opacity, float* __restrict__ depth, float* __restrict__ rgb, int64_t n) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    if (opacity) opacity[e] = 0.0f;
    if (depth) depth[e] = 0.0f;
    if (rgb) rgb[3 * e] = rgb[3 * e + 1] = rgb[3 * e + 2] = 1.0f;
  }
}

// block b: block_count[b] = hit rows among rows [b * kListRows, (b + 1) * kListRows) of the chunk
__global__ void __launch_bounds__(kListThreads)
list_count_kernel(const uint8_t* __restrict__ hit, int n, int* __restrict__ block_count) {
  const int64_t base = (int64_t)blockIdx.x * kListRows;
  int c = 0;
  for (int i = 0; i < kListIters; ++i) {
    const int64_t r = base + i * kListThreads + threadIdx.x;
    c += __syncthreads_count(r < n && hit[r] != 0);
  }
  if (threadIdx.x == 0) block_count[blockIdx.x] = c;
}

// one block: block_off[b] = exclusive prefix sum of the counts (in place), *count = their total
__global__ void __launch_bounds__(1024) list_scan_kernel(int* __restrict__ block_off, int n_blocks, int* __restrict__ count) {
  __shared__ int warp_tot[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int carry = 0;
  for (int b0 = 0; b0 < n_blocks; b0 += 1024) {
    const int b = b0 + threadIdx.x;
    const int v = b < n_blocks ? block_off[b] : 0;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      const int w = warp_tot[lane];
      int wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += t;
      }
      warp_tot[lane] = wi - w;
    }
    __syncthreads();
    const int excl = carry + warp_tot[warp] + incl - v;
    if (b < n_blocks) block_off[b] = excl;
    carry = __shfl_sync(0xffffffffu, excl + v, 31);   // lane 31 of the last warp holds the running total
    __syncthreads();
    if (threadIdx.x == 1023) warp_tot[0] = carry;
    __syncthreads();
    carry = warp_tot[0];
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = carry;
}

// The ordered list: hit row r of the chunk gets slot block_off[block] + (hit rows before it in its block), live[slot] = r
// and rays_l[slot] = rays[r].
__global__ void __launch_bounds__(kListThreads)
list_write_kernel(const uint8_t* __restrict__ hit, const float* __restrict__ rays, int n, const int* __restrict__ block_off,
                  int* __restrict__ live, float* __restrict__ rays_l) {
  __shared__ int warp_cnt[kListThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = (int64_t)blockIdx.x * kListRows;
  int next = block_off[blockIdx.x];
  for (int i = 0; i < kListIters; ++i) {
    const int64_t r = base + i * kListThreads + threadIdx.x;
    const bool h = r < n && hit[r] != 0;
    const unsigned ball = __ballot_sync(0xffffffffu, h);
    if (lane == 0) warp_cnt[warp] = __popc(ball);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kListThreads / 32; ++w) {
      before += w < warp ? warp_cnt[w] : 0;
      total += warp_cnt[w];
    }
    if (h) {
      const int j = next + before + __popc(ball & ((1u << lane) - 1u));
      live[j] = (int)r;
      const float4* src = reinterpret_cast<const float4*>(rays + r * 8);
      float4* dst = reinterpret_cast<float4*>(rays_l + (int64_t)j * 8);
      dst[0] = src[0];
      dst[1] = src[1];
    }
    next += total;
    __syncthreads();
  }
}

struct BoxIds {
  int ids[ONERF_BOXES_MAX];   // code-table row of each box
  int64_t T, g0;              // tile pixels; first row of the chunk
};

// codes[j] = code_table row of listed row live[j] (row g0 + live[j] belongs to box (g0 + live[j]) / T), j < *count
__global__ void __launch_bounds__(256) box_codes_kernel(const float* __restrict__ table, const BoxIds q,
                                                        const int* __restrict__ live, const int* __restrict__ count,
                                                        float* __restrict__ codes) {
  const int n = *count;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n * 16; e += gridDim.x * blockDim.x) {
    const int j = e >> 4, c4 = e & 15;
    const int k = (int)((q.g0 + __ldg(live + j)) / q.T);
    reinterpret_cast<float4*>(codes)[e] = __ldg(reinterpret_cast<const float4*>(table) + (int64_t)q.ids[k] * 16 + c4);
  }
}

// One warp per listed row j < *count: its object branch composited exactly as composite_kernel composites it with
// is_eval, rays_in_bbox and no noise (last delta 0, no occlusion mask, on white), its weights to weights[j] when given.
// The maps go to column k = g / T of pixel row g % T, g = g0 + live[j].
__global__ void __launch_bounds__(256)
composite_boxes_kernel(const float* __restrict__ z_all, const float* __restrict__ obj, const int* __restrict__ live,
                       const int* __restrict__ count, int S, float* __restrict__ weights, int64_t g0, int64_t T, int K,
                       float* __restrict__ opacity, float* __restrict__ depth, float* __restrict__ rgb) {
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_rows = *count;
  for (int r = blockIdx.x * warps_per_block + warp; r < n_rows; r += gridDim.x * warps_per_block) {
    const float* z = z_all + (int64_t)r * S;
    const float4* f = reinterpret_cast<const float4*>(obj) + (int64_t)r * S;
    const Acc ob = warp_sum(composite_branch(z, f, S, 0.0f, 0.0f, nullptr, 0, 3u, r, false, 0.0f,
                                             weights ? weights + (int64_t)r * S : nullptr, lane));
    if (lane == 0) {
      const int64_t g = g0 + __ldg(live + r);
      const int k = (int)(g / T);
      const int64_t l = (g - (int64_t)k * T) * K + k;
      if (opacity) opacity[l] = ob.opacity;
      if (depth) depth[l] = ob.depth;
      if (rgb) {
        rgb[l * 3 + 0] = __fadd_rn(__fadd_rn(ob.r, 1.0f), -ob.opacity);
        rgb[l * 3 + 1] = __fadd_rn(__fadd_rn(ob.g, 1.0f), -ob.opacity);
        rgb[l * 3 + 2] = __fadd_rn(__fadd_rn(ob.b, 1.0f), -ob.opacity);
      }
    }
  }
}

// Per-chunk scratch of n = chunk_rays rows; nothing in it depends on K or the image.  Every per-row array past the
// first two is indexed by list slot.
struct BoxesWs {
  float* rays;                         // (n,8) the chunk's rays
  uint8_t* hit;                        // (n,) hit bit of each row
  int *block_off, *count, *live;       // list: per-block offsets, number of hit rows, row of each slot
  float *rays_l, *z_c, *w_c, *z_f;     // listed rows' rays, coarse depths and weights (n,S), fine depths (n,S+I)
  float *codes, *ray_const, *field;    // listed rows' code rows, per-ray constants and object field (n,S+I,4)
  size_t total;
};

BoxesWs boxes_ws_layout(char* base, int chunk, int n_samples, int n_importance) {
  const size_t n = chunk, S = n_samples, SF = (size_t)n_samples + n_importance, nf = n_importance > 0 ? n : 0;
  const size_t n_blocks = (n + kListRows - 1) / kListRows;
  BoxesWs w;
  WsCarver c{base};
  w.rays = c.floats(n * 8);
  w.hit = static_cast<uint8_t*>(c.take(n));
  w.block_off = static_cast<int*>(c.take(n_blocks * sizeof(int)));
  w.count = static_cast<int*>(c.take(sizeof(int)));
  w.live = static_cast<int*>(c.take(n * sizeof(int)));
  w.rays_l = c.floats(n * 8);
  w.z_c = c.floats(n * S);
  w.w_c = c.floats(n * S);
  w.z_f = c.floats(nf * SF);
  w.codes = c.floats(n * ONERF_NCODE);
  w.ray_const = c.floats(n * ONERF_RAY_CONST_FLOATS);
  w.field = c.floats(n * SF * 4);
  w.total = c.off;
  return w;
}

bool finite_all(const double* v, int n) {
  for (int i = 0; i < n; ++i)
    if (!isfinite(v[i])) return false;
  return true;
}

bool box_maps_aligned(const onerf_box_maps& m) {
  return onerf_aligned4(m.opacity) && onerf_aligned4(m.depth) && onerf_aligned4(m.rgb);
}

// One pass over the listed rows of a chunk of n rows (rows g0.. of the tile) on their depths z (n,S): per-ray constants
// and object field of the listed rows, compositing (weights to w_out when given, maps to m).
int boxes_pass(onerf_ctx* ctx, const onerf_render_boxes_args* a, const BoxesWs& w, int n, int64_t g0, const void* packed,
               const float* z, int S, float* w_out, const onerf_box_maps& m, cudaStream_t stream) {
  FieldParams p = onerf_field_params(a->grid, packed);
  p.rays = w.rays_l; p.z = z; p.z_stride = S;
  p.codes = w.codes;
  p.n_rays = n; p.S = S;
  p.want_object = 1;
  p.obj_out = w.field; p.out_stride = S;
  p.ray_const = w.ray_const;
  p.n_live = w.count;
  int rc = onerf_launch_ray_const(ctx, p, stream);
  if (rc != ONERF_OK) return rc;
  rc = a->precision == ONERF_PREC_BF16 ? onerf_launch_field_bf16_codes(ctx, p, 1, 0, 0, stream)
                                       : onerf_launch_field_fp32(ctx, p, stream);
  if (rc != ONERF_OK) return rc;
  composite_boxes_kernel<<<composite_blocks(ctx, n, 8), 256, 0, stream>>>(
      z, w.field, w.live, w.count, S, w_out, g0, a->pixel_end - a->pixel_begin, a->n_boxes, m.opacity, m.depth, m.rgb);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

// List the hit rows of a chunk of n rows in row order and gather their rays; then the listed rows' code rows.
int boxes_list(onerf_ctx* ctx, const onerf_render_boxes_args* a, const BoxesWs& w, int n, int64_t g0,
               cudaStream_t stream) {
  const int n_blocks = (n + kListRows - 1) / kListRows;
  const int64_t T = a->pixel_end - a->pixel_begin;
  list_count_kernel<<<n_blocks, kListThreads, 0, stream>>>(w.hit, n, w.block_off);
  ONERF_LAUNCH_CHECK(ctx);
  list_scan_kernel<<<1, 1024, 0, stream>>>(w.block_off, n_blocks, w.count);
  ONERF_LAUNCH_CHECK(ctx);
  list_write_kernel<<<n_blocks, kListThreads, 0, stream>>>(w.hit, w.rays, n, w.block_off, w.live, w.rays_l);
  ONERF_LAUNCH_CHECK(ctx);
  BoxIds q;
  memset(&q, 0, sizeof(q));
  for (int k = 0; k < a->n_boxes; ++k) q.ids[k] = a->ids_host[k];
  q.T = T; q.g0 = g0;
  const int blocks = (int)std::min<int64_t>(((int64_t)n * 16 + 255) / 256, (int64_t)ctx->num_sms * 8);
  box_codes_kernel<<<blocks, 256, 0, stream>>>(a->code_table, q, w.live, w.count, w.codes);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

}  // namespace

extern "C" size_t onerf_render_boxes_workspace_bytes(int chunk_rays, int n_samples, int n_importance) {
  if (chunk_rays < 1 || n_samples < 2 || n_importance < 0) return 0;
  return boxes_ws_layout(nullptr, chunk_rays, n_samples, n_importance).total;
}

extern "C" int onerf_render_boxes(onerf_ctx* ctx, const onerf_render_boxes_args* a, void* stream_) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  const int K = a->n_boxes;
  ONERF_CHECK_ARG(K >= 1 && K <= ONERF_BOXES_MAX, "n_boxes outside [1, 64]");
  ONERF_CHECK_ARG(a->boxes_host && a->ids_host && a->code_table, "null boxes_host / ids_host / code_table");
  for (int k = 0; k < K; ++k) {
    ONERF_CHECK_ARG(a->ids_host[k] >= 0 && a->ids_host[k] < a->n_codes_table, "object id outside the code table");
    const onerf_box_host& b = a->boxes_host[k];
    ONERF_CHECK_ARG(finite_all(b.pose_avg, 12) && finite_all(b.axis_align, 12) && finite_all(b.bounds, 6),
                    "non-finite box");
  }
  ONERF_CHECK_ARG(a->c2w_host, "null c2w_host");
  for (int i = 0; i < 12; ++i) ONERF_CHECK_ARG(isfinite(a->c2w_host[i]), "non-finite camera");
  ONERF_CHECK_ARG(a->H >= 1 && a->W >= 1 && isfinite(a->focal) && a->focal > 0, "bad camera");
  ONERF_CHECK_ARG(isfinite(a->scale_factor) && a->scale_factor > 0, "scale_factor must be finite and positive");
  ONERF_CHECK_ARG(a->pixel_begin >= 0 && a->pixel_begin <= a->pixel_end && a->pixel_end <= (int64_t)a->H * a->W,
                  "pixel range outside the image");
  ONERF_CHECK_ARG(a->chunk_rays >= 1, "chunk_rays < 1");
  ONERF_CHECK_ARG(a->n_samples >= 2 && a->n_importance >= 0, "bad shape");
  // the importance sampler sorts S + K depths per ray in shared memory (onerf_render_rays_fwd's limit)
  ONERF_UNSUPPORTED(a->n_importance > 0 && (int64_t)a->n_samples + a->n_importance > 2048, "S + K > 2048");
  ONERF_CHECK_ARG(a->packed_coarse, "null packed_coarse");
  ONERF_CHECK_ARG(a->n_importance == 0 || a->packed_fine, "n_importance > 0 needs packed_fine");
  int rc = onerf_check_grid(__func__, a->grid);
  if (rc != ONERF_OK) return rc;
  ONERF_CHECK_ARG(a->precision == ONERF_PREC_FP32 || a->precision == ONERF_PREC_BF16, "unknown precision");
  ONERF_CHECK_ARG(a->n_importance > 0 || !(a->fine.opacity || a->fine.depth || a->fine.rgb),
                  "fine maps without a fine pass");
  ONERF_CHECK_ARG(onerf_aligned16(a->code_table), "code_table must be 16-byte aligned");
  ONERF_CHECK_ARG(box_maps_aligned(a->coarse) && box_maps_aligned(a->fine), "maps must be 4-byte aligned");
  const int chunk = a->chunk_rays;
  rc = onerf_check_workspace(__func__, a->workspace, a->workspace_bytes,
                             onerf_render_boxes_workspace_bytes(chunk, a->n_samples, a->n_importance), ONERF_ERR_BAD_ARG);
  if (rc != ONERF_OK) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  const BoxesWs w = boxes_ws_layout(reinterpret_cast<char*>(a->workspace), chunk, a->n_samples, a->n_importance);
  const int S = a->n_samples, SF = a->n_samples + a->n_importance;
  const int64_t T = a->pixel_end - a->pixel_begin, rows = T * K;
  if (rows > 0)
    for (const onerf_box_maps* m : {&a->coarse, &a->fine}) {
      if (!(m->opacity || m->depth || m->rgb)) continue;
      const int blocks = (int)std::min<int64_t>((rows + 255) / 256, (int64_t)ctx->num_sms * 16);
      fill_missed_kernel<<<blocks, 256, 0, stream>>>(m->opacity, m->depth, m->rgb, rows);
      ONERF_LAUNCH_CHECK(ctx);
    }
  for (int64_t g0 = 0; g0 < rows; g0 += chunk) {
    const int n = (int)(rows - g0 < chunk ? rows - g0 : chunk);
    rc = onerf_launch_box_rays(ctx, a->H, a->W, a->focal, a->c2w_host, a->boxes_host, K, a->scale_factor,
                                   a->pixel_begin, T, g0, n, w.rays, w.hit, a->hit, stream);
    if (rc != ONERF_OK) return rc;
    rc = boxes_list(ctx, a, w, n, g0, stream);
    if (rc != ONERF_OK) return rc;
    rc = onerf_launch_sample_coarse_live(ctx, w.rays_l, w.count, n, S, a->use_disp, w.z_c, stream);
    if (rc != ONERF_OK) return rc;
    rc = boxes_pass(ctx, a, w, n, g0, a->packed_coarse, w.z_c, S, a->n_importance > 0 ? w.w_c : nullptr, a->coarse,
                    stream);
    if (rc != ONERF_OK) return rc;
    if (a->n_importance == 0) continue;
    rc = onerf_launch_sample_pdf_merge_live(ctx, w.z_c, w.w_c, w.count, n, S, a->n_importance, w.z_f, stream);
    if (rc != ONERF_OK) return rc;
    rc = boxes_pass(ctx, a, w, n, g0, a->packed_fine, w.z_f, SF, nullptr, a->fine, stream);
    if (rc != ONERF_OK) return rc;
  }
  return ONERF_OK;
}
