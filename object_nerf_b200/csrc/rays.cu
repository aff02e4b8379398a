// Camera ray generation and per-object (N,8) ray assembly: the steps directly in front of render_rays_multi()
// (SURVEY.md section 8f rows 1-2).  Reference: datasets/ray_utils.py:5-51 (get_ray_directions, get_rays),
// render_tools/editable_renderer.py:153-181 (generate_rays), utils/bbox_utils.py:102-156 (rays -> box frame) and
// datasets/geo_utils.py:111-162 (slab test; numba, float64).  The reference does the box part on the HOST per frame and
// per object (numpy + numba, then .cuda()); here it is one HBM-bound kernel: 24 B in, 32 (+1) B out per ray.
#include <string.h>

#include "camera.cuh"
#include "../../include/onerf_ext.h"

namespace {

struct BoxParams {           // passed by value; all float64 like the reference's numpy arrays
  double Ra[9], ta[3];       // pose_avg        (utils/bbox_utils.py:111-113)
  double Rb[9], tb[3];       // axis_align_mat  (:115-117)
  double lo[3], hi[3];       // bbox_bounds, already enlarged (:140-145)
  float scale_f;             // scale_factor as the fp32 scalar numpy / torch use in the fp32 ops (:109, :155)
  int has_box;
  float near_f, far_f;       // scene rays: fp32(near / scale_factor), fp32(far / scale_factor) (editable_renderer.py:157-158)
};

// utils/bbox_utils.py:102-156 + datasets/geo_utils.py:126-162 for one ray; returns hit, near / far already divided by
// the scale factor (fp32, :155) and zeroed for a miss (editable_renderer.py:173-176).
__device__ __forceinline__ bool box_near_far(const BoxParams& b, float ox, float oy, float oz, float dx, float dy, float dz,
                                             float& near, float& far) {
  // unscale in fp32 (numpy float32 array * python float), the rest in float64
  const double o0 = (double)__fmul_rn(ox, b.scale_f), o1 = (double)__fmul_rn(oy, b.scale_f), o2 = (double)__fmul_rn(oz, b.scale_f);
  double p[3], q[3], d[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) p[i] = (b.Ra[3 * i] * o0 + b.Ra[3 * i + 1] * o1 + b.Ra[3 * i + 2] * o2) + b.ta[i];
#pragma unroll
  for (int i = 0; i < 3; ++i) q[i] = (b.Rb[3 * i] * p[0] + b.Rb[3 * i + 1] * p[1] + b.Rb[3 * i + 2] * p[2]) + b.tb[i];
  // the direction is rotated by the axis-alignment matrix only (:116 uses rays_d, not the de-centred one)
#pragma unroll
  for (int i = 0; i < 3; ++i) d[i] = b.Rb[3 * i] * (double)dx + b.Rb[3 * i + 1] * (double)dy + b.Rb[3 * i + 2] * (double)dz;
  near = 0.0f;
  far = 0.0f;
  double inv[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) inv[i] = 1.0 / (d[i] == 0.0 ? 1.0e-14 : d[i]);   // geo_utils.py:131
  double tmin = ((inv[0] < 0 ? b.hi[0] : b.lo[0]) - q[0]) * inv[0];
  double tmax = ((inv[0] < 0 ? b.lo[0] : b.hi[0]) - q[0]) * inv[0];
  const double tymin = ((inv[1] < 0 ? b.hi[1] : b.lo[1]) - q[1]) * inv[1];
  const double tymax = ((inv[1] < 0 ? b.lo[1] : b.hi[1]) - q[1]) * inv[1];
  if (tmin > tymax || tymin > tmax) return false;
  if (tymin > tmin) tmin = tymin;
  if (tymax < tmax) tmax = tymax;
  const double tzmin = ((inv[2] < 0 ? b.hi[2] : b.lo[2]) - q[2]) * inv[2];
  const double tzmax = ((inv[2] < 0 ? b.lo[2] : b.hi[2]) - q[2]) * inv[2];
  if (tmin > tzmax || tzmin > tmax) return false;
  if (tzmin > tmin) tmin = tzmin;
  if (tzmax < tmax) tmax = tzmax;
  if (tmin < 0 || tmax < 0) return false;                                       // origin inside the box: a miss (:158-160)
  near = __fdiv_rn((float)tmin, b.scale_f);
  far = __fdiv_rn((float)tmax, b.scale_f);
  return true;
}

__device__ __forceinline__ void write_ray(float* __restrict__ out, uint8_t* __restrict__ hit_out, int64_t r, const BoxParams& b,
                                          float ox, float oy, float oz, float dx, float dy, float dz) {
  float near = b.near_f, far = b.far_f;
  bool hit = true;
  if (b.has_box) hit = box_near_far(b, ox, oy, oz, dx, dy, dz, near, far);
  float4* o4 = reinterpret_cast<float4*>(out + r * 8);
  o4[0] = make_float4(ox, oy, oz, dx);
  o4[1] = make_float4(dy, dz, near, far);
  if (hit_out) hit_out[r] = hit ? 1 : 0;
}

__global__ void __launch_bounds__(256) ray_directions_kernel(Cam c, float* __restrict__ directions) {
  const int64_t n = (int64_t)c.H * c.W;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(i / c.W), x = (int)(i - (int64_t)y * c.W);
    float dx, dy, dz;
    pixel_direction(c, x, y, dx, dy, dz);
    directions[3 * i] = dx; directions[3 * i + 1] = dy; directions[3 * i + 2] = dz;
  }
}

__global__ void __launch_bounds__(256) get_rays_kernel(Cam c, const float* __restrict__ directions, int64_t n,
                                                       float* __restrict__ rays_o, float* __restrict__ rays_d) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float ox, oy, oz;
    rotate_normalise(c, directions[3 * i], directions[3 * i + 1], directions[3 * i + 2], ox, oy, oz);
    rays_d[3 * i] = ox; rays_d[3 * i + 1] = oy; rays_d[3 * i + 2] = oz;
    rays_o[3 * i] = c.t[0]; rays_o[3 * i + 1] = c.t[1]; rays_o[3 * i + 2] = c.t[2];
  }
}

__global__ void __launch_bounds__(256) generate_rays_kernel(BoxParams b, const float* __restrict__ rays_o,
                                                            const float* __restrict__ rays_d, int64_t n,
                                                            float* __restrict__ out, uint8_t* __restrict__ hit_out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    write_ray(out, hit_out, i, b, rays_o[3 * i], rays_o[3 * i + 1], rays_o[3 * i + 2], rays_d[3 * i], rays_d[3 * i + 1],
              rays_d[3 * i + 2]);
}

// pixel -> (N,8) ray in one pass: get_ray_directions + get_rays + generate_rays.  Row i of out is pixel p0 + i (row-major),
// i < n: a tile of the frame gets the rays the whole frame has at those pixels.
__global__ void __launch_bounds__(256) camera_rays_kernel(Cam c, BoxParams b, int64_t p0, int64_t n, float* __restrict__ out,
                                                          uint8_t* __restrict__ hit_out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = p0 + i;
    const int y = (int)(p / c.W), x = (int)(p - (int64_t)y * c.W);
    float dx, dy, dz, wx, wy, wz;
    pixel_direction(c, x, y, dx, dy, dz);
    rotate_normalise(c, dx, dy, dz, wx, wy, wz);
    write_ray(out, hit_out, i, b, c.t[0], c.t[1], c.t[2], wx, wy, wz);
  }
}

// onerf_render_boxes: rows [g0, g0 + n) of the (object, pixel) rows of a tile of T pixels, object-major (row g is pixel
// p_begin + g % T of box g / T).  Row i of out / hit_rows is that row's ray as camera_rays_kernel writes it with the
// row's box; hit_out, when given, gets the hit bit at [(g % T) * K + g / T] as well.
struct BoxRaysParams {
  Cam c;
  BoxParams b[ONERF_BOXES_MAX];
  int64_t p_begin, T, g0;
  int n, K;
};

__global__ void __launch_bounds__(256) box_rays_kernel(const __grid_constant__ BoxRaysParams q, float* __restrict__ out,
                                                       uint8_t* __restrict__ hit_rows, uint8_t* __restrict__ hit_out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < q.n; i += gridDim.x * blockDim.x) {
    const int64_t g = q.g0 + i;
    const int k = (int)(g / q.T);
    const int64_t t = g - (int64_t)k * q.T, p = q.p_begin + t;
    const Cam& c = q.c;
    const int y = (int)(p / c.W), x = (int)(p - (int64_t)y * c.W);
    float dx, dy, dz, wx, wy, wz, near, far;
    pixel_direction(c, x, y, dx, dy, dz);
    rotate_normalise(c, dx, dy, dz, wx, wy, wz);
    const bool hit = box_near_far(q.b[k], c.t[0], c.t[1], c.t[2], wx, wy, wz, near, far);
    float4* o4 = reinterpret_cast<float4*>(out + (int64_t)i * 8);
    o4[0] = make_float4(c.t[0], c.t[1], c.t[2], wx);
    o4[1] = make_float4(wy, wz, near, far);
    hit_rows[i] = hit ? 1 : 0;
    if (hit_out) hit_out[t * q.K + k] = hit ? 1 : 0;
  }
}

int grid_for(const onerf_ctx* ctx, int64_t n) {
  const int64_t want = (n + 255) / 256, cap = (int64_t)ctx->num_sms * 8;   // grid-stride: a multiple of the SM count
  return (int)(want < cap ? (want > 0 ? want : 1) : cap);
}

Cam make_cam(int H, int W, float focal, const float* c2w_host) {
  Cam c;
  memset(&c, 0, sizeof(c));
  c.H = H; c.W = W;
  c.half_w = (float)(W / 2.0);   // python float W / 2, rounded to the fp32 scalar torch uses
  c.half_h = (float)(H / 2.0);
  c.focal = focal;
  if (c2w_host)
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) c.r[3 * i + j] = c2w_host[4 * i + j];
      c.t[i] = c2w_host[4 * i + 3];
    }
  return c;
}

int make_box(const onerf_box_host* box, double scale_factor, double near, double far, BoxParams& b) {
  memset(&b, 0, sizeof(b));
  ONERF_CHECK_ARG(scale_factor > 0, "scale_factor must be positive");
  b.scale_f = (float)scale_factor;
  b.near_f = (float)(near / scale_factor);
  b.far_f = (float)(far / scale_factor);
  if (box) {
    b.has_box = 1;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) {
        b.Ra[3 * i + j] = box->pose_avg[4 * i + j];
        b.Rb[3 * i + j] = box->axis_align[4 * i + j];
      }
      b.ta[i] = box->pose_avg[4 * i + 3];
      b.tb[i] = box->axis_align[4 * i + 3];
      b.lo[i] = box->bounds[i];
      b.hi[i] = box->bounds[3 + i];
    }
  }
  return ONERF_OK;
}

}  // namespace

extern "C" int onerf_ray_directions(onerf_ctx* ctx, int H, int W, float focal, float* directions, void* stream) {
  ONERF_CHECK_ARG(ctx && directions, "null argument");
  ONERF_CHECK_ARG(H > 0 && W > 0 && focal > 0, "bad camera");
  const Cam c = make_cam(H, W, focal, nullptr);
  ray_directions_kernel<<<grid_for(ctx, (int64_t)H * W), 256, 0, (cudaStream_t)stream>>>(c, directions);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_get_rays(onerf_ctx* ctx, const float* directions, int64_t n, const float* c2w_host, float* rays_o,
                              float* rays_d, void* stream) {
  ONERF_CHECK_ARG(ctx && directions && c2w_host && rays_o && rays_d, "null argument");
  ONERF_CHECK_ARG(n >= 0, "bad count");
  if (n == 0) return ONERF_OK;
  const Cam c = make_cam(1, 1, 1.0f, c2w_host);
  get_rays_kernel<<<grid_for(ctx, n), 256, 0, (cudaStream_t)stream>>>(c, directions, n, rays_o, rays_d);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_generate_rays(onerf_ctx* ctx, const float* rays_o, const float* rays_d, int64_t n,
                                   const onerf_box_host* box, double scale_factor, double near, double far, float* rays_out,
                                   uint8_t* hit_out, void* stream) {
  ONERF_CHECK_ARG(ctx && rays_o && rays_d && rays_out, "null argument");
  ONERF_CHECK_ARG(n >= 0 && onerf_aligned16(rays_out), "bad count or misaligned output");
  if (n == 0) return ONERF_OK;
  BoxParams b;
  const int rc = make_box(box, scale_factor, near, far, b);
  if (rc != ONERF_OK) return rc;
  generate_rays_kernel<<<grid_for(ctx, n), 256, 0, (cudaStream_t)stream>>>(b, rays_o, rays_d, n, rays_out, hit_out);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int onerf_launch_camera_rays(onerf_ctx* ctx, int H, int W, float focal, const float* c2w_host, const onerf_box_host* box,
                             double scale_factor, double near, double far, int64_t p0, int64_t n, float* rays_out,
                             uint8_t* hit_out, cudaStream_t stream) {
  BoxParams b;
  const int rc = make_box(box, scale_factor, near, far, b);
  if (rc != ONERF_OK) return rc;
  if (n == 0) return ONERF_OK;
  const Cam c = make_cam(H, W, focal, c2w_host);
  camera_rays_kernel<<<grid_for(ctx, n), 256, 0, stream>>>(c, b, p0, n, rays_out, hit_out);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int onerf_launch_box_rays(onerf_ctx* ctx, int H, int W, float focal, const float* c2w_host, const onerf_box_host* boxes,
                          int K, double scale_factor, int64_t p_begin, int64_t T, int64_t g0, int n, float* rays_out,
                          uint8_t* hit_rows, uint8_t* hit_out, cudaStream_t stream) {
  if (n == 0) return ONERF_OK;
  BoxRaysParams q;
  memset(&q, 0, sizeof(q));
  q.c = make_cam(H, W, focal, c2w_host);
  for (int k = 0; k < K; ++k) {
    const int rc = make_box(&boxes[k], scale_factor, 0.0, 0.0, q.b[k]);
    if (rc != ONERF_OK) return rc;
  }
  q.p_begin = p_begin; q.T = T; q.g0 = g0; q.n = n; q.K = K;
  box_rays_kernel<<<grid_for(ctx, n), 256, 0, stream>>>(q, rays_out, hit_rows, hit_out);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_camera_rays(onerf_ctx* ctx, int H, int W, float focal, const float* c2w_host, const onerf_box_host* box,
                                 double scale_factor, double near, double far, float* rays_out, uint8_t* hit_out,
                                 void* stream) {
  ONERF_CHECK_ARG(ctx && c2w_host && rays_out, "null argument");
  ONERF_CHECK_ARG(H > 0 && W > 0 && focal > 0 && onerf_aligned16(rays_out), "bad camera or misaligned output");
  return onerf_launch_camera_rays(ctx, H, W, focal, c2w_host, box, scale_factor, near, far, 0, (int64_t)H * W, rays_out,
                                  hit_out, (cudaStream_t)stream);
}
