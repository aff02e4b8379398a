// Shared helpers for libonerf_sm90.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/onerf.h"

struct onerf_ctx {
  int device;
  int num_sms;
  int64_t launches;
  void* pack_tables;   // pack.cu: per-layout job tables in device memory (created on first use)
  // Mapped host memory the tensor-core kernels' bounded mbarrier wait (tc_common.cuh: mbar_wait) writes
  // {1, block, barrier, parity} to before it traps.  Host memory stays readable after the trap has ended the CUDA
  // context, so the next launch check can say which wait timed out.
  uint32_t* tc_diag;
};
void onerf_free_pack_tables(onerf_ctx* ctx);

void onerf_set_error(const char* fmt, ...);

// rays.cu: pixels [p0, p0 + n) of onerf_camera_rays' H x W frame, written as rows 0 .. n-1 of rays_out (and hit_out).
// The camera and rays_out are the caller's to check.
int onerf_launch_camera_rays(onerf_ctx* ctx, int H, int W, float focal, const float* c2w_host, const onerf_box_host* box,
                             double scale_factor, double near, double far, int64_t p0, int64_t n, float* rays_out,
                             uint8_t* hit_out, cudaStream_t stream);
// rays.cu: rows [g0, g0 + n) of onerf_render_boxes' (object, pixel) rows of the tile of T pixels from p_begin (row g is
// pixel p_begin + g % T clipped to boxes[g / T], K boxes): their rays to rays_out (n,8) and hit bits to hit_rows (n,), and
// to hit_out[(g % T) * K + g / T] when hit_out is given.  The arguments are the caller's to check.
int onerf_launch_box_rays(onerf_ctx* ctx, int H, int W, float focal, const float* c2w_host, const onerf_box_host* boxes,
                          int K, double scale_factor, int64_t p_begin, int64_t T, int64_t g0, int n, float* rays_out,
                          uint8_t* hit_rows, uint8_t* hit_out, cudaStream_t stream);

// composite.cu: the per-set maps of one joint compositing from its weights in set order (weights_unsorted of
// onerf_composite_multi_ws), depths z_all (n_obj,N,S) and fields field_all (n_obj,N,S,4); NULL outputs are skipped.
int onerf_launch_set_maps(onerf_ctx* ctx, const float* z_all, const float* field_all, const float* weights_unsorted,
                          int n_rays, int n_obj, int n_samples, float* opacity, float* depth, float* rgb,
                          cudaStream_t stream);

// composite.cu: the object maps of n_codes object fields of the same rays and depths z (n_rays,S): field k is the
// (n_rays,S,4) block at obj + k * obj_stride floats, composited as onerf_composite composites the object branch with
// is_eval set.  opacity / depth (n_rays,n_codes), rgb (n_rays,n_codes,3); NULL outputs are skipped.
int onerf_launch_composite_instances(onerf_ctx* ctx, const float* z, const float* obj, int64_t obj_stride, int n_rays,
                                     int n_samples, int n_codes, float* opacity, float* depth, float* rgb,
                                     cudaStream_t stream);

// composite.cu: n samples of one set of a source scene onto the frame's depth axis: z_out = z * k, field sigma /= k in
// place (field: n float4).
int onerf_launch_rescale_set(onerf_ctx* ctx, const float* z, float* z_out, float* field, int64_t n, float k,
                             cudaStream_t stream);

#define ONERF_CHECK_ARG(cond, msg)                       \
  do {                                                   \
    if (!(cond)) {                                       \
      onerf_set_error("%s: %s", __func__, msg);          \
      return ONERF_ERR_BAD_ARG;                          \
    }                                                    \
  } while (0)

#define ONERF_UNSUPPORTED(cond, msg)                     \
  do {                                                   \
    if (cond) {                                          \
      onerf_set_error("%s: unsupported: %s", __func__, msg); \
      return ONERF_ERR_UNSUPPORTED;                      \
    }                                                    \
  } while (0)

#define ONERF_CUDA(call)                                                          \
  do {                                                                            \
    cudaError_t e_ = (call);                                                      \
    if (e_ != cudaSuccess) {                                                      \
      onerf_set_error("%s: %s failed: %s", __func__, #call, cudaGetErrorString(e_)); \
      return ONERF_ERR_CUDA;                                                      \
    }                                                                             \
  } while (0)

#define ONERF_LAUNCH_CHECK(ctx)                                                   \
  do {                                                                            \
    cudaError_t e_ = cudaGetLastError();                                          \
    if (e_ != cudaSuccess) {                                                      \
      const uint32_t* d_ = (ctx)->tc_diag;                                        \
      if (d_ && d_[0])                                                            \
        onerf_set_error("%s: kernel launch failed: %s (an earlier kernel timed out in an mbarrier wait: block %u, " \
                        "barrier 0x%x, parity %u)", __func__, cudaGetErrorString(e_), d_[1], d_[2], d_[3]); \
      else                                                                        \
        onerf_set_error("%s: kernel launch failed: %s", __func__, cudaGetErrorString(e_)); \
      return ONERF_ERR_CUDA;                                                      \
    }                                                                             \
    (ctx)->launches++;                                                            \
  } while (0)

// ONERF_CHECK_ARG / ONERF_UNSUPPORTED reported under the entry `fn` (a local of the caller) instead of __func__, for
// checks shared by several entry points.
#define FN_CHECK_ARG(cond, msg)                                                      \
  do {                                                                               \
    if (!(cond)) { onerf_set_error("%s: %s", fn, msg); return ONERF_ERR_BAD_ARG; }   \
  } while (0)
#define FN_UNSUPPORTED(cond, msg)                                                                 \
  do {                                                                                            \
    if (cond) { onerf_set_error("%s: unsupported: %s", fn, msg); return ONERF_ERR_UNSUPPORTED; }  \
  } while (0)

static inline bool onerf_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline bool onerf_aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }
static inline bool onerf_aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }

// The buffers of a voxel grid, refused under the entry `fn` with `where` ending the message.  NULL (the plain-PE model)
// passes.
static inline int onerf_check_grid(const char* fn, const onerf_grid* g, const char* where = "") {
  if (!g || (g->table && g->idx_map && g->voxel_offset && g->voxel_size && g->voxel_shape && onerf_aligned16(g->table)))
    return ONERF_OK;
  onerf_set_error("%s: null / misaligned grid buffer%s", fn, where);
  return ONERF_ERR_BAD_ARG;
}

// A caller's workspace of `bytes` bytes for an entry `fn` that needs `need`: NULL or misaligned is ONERF_ERR_BAD_ARG, too
// small is `small_code` (each entry's header names its own).
static inline int onerf_check_workspace(const char* fn, const void* ws, size_t bytes, size_t need, int small_code) {
  if (!ws || (reinterpret_cast<uintptr_t>(ws) & 255u) != 0) {
    onerf_set_error("%s: workspace null or not 256-byte aligned", fn);
    return ONERF_ERR_BAD_ARG;
  }
  if (bytes < need) {
    onerf_set_error("%s: workspace too small (%zu < %zu)", fn, bytes, need);
    return small_code;
  }
  return ONERF_OK;
}

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// Consecutive 256-byte aligned buffers of a workspace, in the order they are taken.  With a NULL base it only sizes the
// workspace: `off` is then its total size.
struct WsCarver {
  char* base;
  size_t off = 0;
  void* take(size_t bytes) {
    void* p = base + off;
    off += align256(bytes);
    return p;
  }
  float* floats(size_t n) { return static_cast<float*>(take(n * sizeof(float))); }
};

// ---------------------------------------------------------------------------------------------
// warp helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Ascending bitonic sort of keys[0, P) (P a power of two, shared memory) by the whole warp, after the warp's writes to
// keys.  Pad with keys that sort last.  The compare-exchange is (a > b) == up: float keys holding NaN end where that
// rule puts them.
template <typename T>
__device__ __forceinline__ void warp_bitonic_sort(T* keys, int P, int lane) {
  __syncwarp();
  for (int k2 = 2; k2 <= P; k2 <<= 1) {
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int t = lane; t < (P >> 1); t += 32) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // index with bit j cleared
        const int l = i | j;
        const bool up = ((i & k2) == 0);
        const T a = keys[i], b = keys[l];
        if ((a > b) == up) { keys[i] = b; keys[l] = a; }
      }
      __syncwarp();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 counter RNG (used only when the caller does not inject its own random buffers)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}

// uniform in [0,1) with 24 random bits (same granularity as torch.rand for fp32)
__device__ __forceinline__ float u01(uint32_t x) { return (x >> 8) * (1.0f / 16777216.0f); }

// one U[0,1) for element `idx` of random stream `stream_id`
__device__ __forceinline__ float philox_uniform(uint64_t seed, uint32_t stream_id, uint64_t idx) {
  uint4 r = philox4x32(make_uint4((uint32_t)(idx >> 2), (uint32_t)(idx >> 34), stream_id, 0u),
                       make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  uint32_t v = (idx & 3) == 0 ? r.x : (idx & 3) == 1 ? r.y : (idx & 3) == 2 ? r.z : r.w;
  return u01(v);
}

// one N(0,1) for element idx (Box-Muller on two uniforms of the same counter)
__device__ __forceinline__ float philox_normal(uint64_t seed, uint32_t stream_id, uint64_t idx) {
  uint4 r = philox4x32(make_uint4((uint32_t)(idx >> 1), (uint32_t)(idx >> 33), stream_id, 1u),
                       make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  uint32_t a = (idx & 1) ? r.z : r.x, b = (idx & 1) ? r.w : r.y;
  float u1 = ((a >> 8) + 1) * (1.0f / 16777216.0f);  // (0,1]
  float u2 = u01(b);
  return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}
