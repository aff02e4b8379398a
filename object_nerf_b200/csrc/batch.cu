// Training batches drawn on the device (include/onerf_ext.h: onerf_draw_batch, onerf_draw_frames).  A block draws kElems
// consecutive batch elements: each thread first locates its element's ray in the epoch's permutation and draws its
// instance column, then the block copies every field with consecutive threads on consecutive output words, so the stores
// are coalesced.  Both kernels share that draw; they differ in where a row's fields come from (per-ray buffers, or a
// frame store the row is rebuilt from).
#include "camera.cuh"
#include "../../include/onerf_ext.h"

namespace {

constexpr int kElems = 128;                 // batch elements (and threads) per block
constexpr int kRounds = 6;                  // Feistel rounds
constexpr uint32_t kPermStream = 5u;        // Philox stream ids no other kernel of the library uses
constexpr uint32_t kColumnStream = 4u;
constexpr int64_t kMaxRays = int64_t(1) << 40;
constexpr int kMaxPass = ONERF_FRAME_MAX_PASS;

// One pass of the keyed Feistel network on [0, 2^(2*half)): a bijection for any round function.
__device__ __forceinline__ uint64_t feistel(uint64_t x, int half, uint2 key, uint64_t epoch) {
  const uint32_t mask = (1u << half) - 1u;
  uint32_t L = (uint32_t)(x >> half), R = (uint32_t)x & mask;
#pragma unroll
  for (uint32_t round = 0; round < kRounds; ++round) {
    const uint32_t f = philox4x32(make_uint4(R, (uint32_t)epoch, kPermStream, round), key).x & mask;
    const uint32_t next = L ^ f;
    L = R;
    R = next;
  }
  return ((uint64_t)L << half) | R;
}

// Position p < R of the permutation of [0, R): walk p's cycle until it re-enters [0, R) (2^(2*half) < 4R, so fewer
// than 4 passes are expected).
__device__ __forceinline__ int64_t permute(uint64_t p, uint64_t R, int half, uint2 key, uint64_t epoch) {
  uint64_t x = p;
  do {
    x = feistel(x, half, key, epoch);
  } while (x >= R);
  return (int64_t)x;
}

// Element b of the batch: its ray (position (j*B + b)*W + rank of epoch e's permutation of [0, R)) and its instance column.
__device__ __forceinline__ void draw_element(const onerf_batch_args& a, uint64_t R, int n_instances, int half, uint2 key,
                                             uint64_t step, uint64_t b, int64_t& ray, int64_t& col) {
  const uint64_t B = (uint64_t)a.batch, W = (uint64_t)a.world;
  const uint64_t P = R / (B * W);
  const uint64_t epoch = step / P, j = step % P;
  ray = permute((j * B + b) * W + (uint64_t)a.rank, R, half, key, epoch);
  const uint64_t e = (step * B + b) * W + (uint64_t)a.rank;
  const uint4 r = philox4x32(make_uint4((uint32_t)(e >> 2), (uint32_t)(e >> 34), kColumnStream, 0u), key);
  const uint32_t w = (e & 3) == 0 ? r.x : (e & 3) == 1 ? r.y : (e & 3) == 2 ? r.z : r.w;
  col = (int64_t)(((uint64_t)w * (uint64_t)n_instances) >> 32);
}

__global__ void __launch_bounds__(kElems) draw_batch_kernel(onerf_batch_args a, int half, const uint64_t* step_dev) {
  __shared__ int64_t s_ray[kElems], s_cell[kElems], s_col[kElems];
  const onerf_ray_dataset& d = a.data;
  const int64_t b0 = (int64_t)blockIdx.x * kElems;
  const int n = (int)min((int64_t)kElems, a.batch - b0);
  const uint2 key = make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32));
  const uint64_t step = step_dev ? *step_dev : a.step;
  const int t = threadIdx.x;
  if (t < n) {
    int64_t ray, col;
    draw_element(a, (uint64_t)d.n_rays, d.n_instances, half, key, step, (uint64_t)(b0 + t), ray, col);
    s_ray[t] = ray;
    s_col[t] = col;
    s_cell[t] = ray * d.n_instances + col;
  }
  __syncthreads();
  for (int f = t; f < n * 8; f += kElems) a.rays[b0 * 8 + f] = __ldg(d.rays + s_ray[f >> 3] * 8 + (f & 7));
  for (int f = t; f < n * 3; f += kElems) a.rgbs[b0 * 3 + f] = __ldg(d.rgbs + s_ray[f / 3] * 3 + f % 3);
  if (a.index_out)
    for (int f = t; f < n * 2; f += kElems) a.index_out[b0 * 2 + f] = (f & 1) ? s_col[f >> 1] : s_ray[f >> 1];
  if (t >= n) return;
  const int64_t i = s_ray[t], cell = s_cell[t], o = b0 + t;
  a.depths[o] = __ldg(d.depths + i);
  a.valid_mask[o] = __ldg(d.valid_mask + i);
  if (a.frame_idx) a.frame_idx[o] = d.frame_idx ? __ldg(d.frame_idx + i) : -1;
  a.instance_mask[o] = __ldg(d.instance_mask + cell);
  a.instance_mask_weight[o] = __ldg(d.instance_mask_weight + cell);
  a.instance_ids[o] = __ldg(d.instance_ids + cell);
  a.pass_through_mask[o] = __ldg(d.pass_through_mask + cell);
}

// A row rebuilt from the frame store (onerf_draw_frames).  Rays and colours go through shared memory so that their
// stores are coalesced as in draw_batch_kernel; every other field is one word per element, stored by its own thread.
__global__ void __launch_bounds__(kElems) draw_frames_kernel(onerf_frame_dataset d, onerf_batch_args a, int half,
                                                             const uint64_t* step_dev) {
  __shared__ float s_rays[kElems * 8], s_rgb[kElems * 3];
  __shared__ int64_t s_ray[kElems], s_col[kElems];
  const int64_t b0 = (int64_t)blockIdx.x * kElems;
  const int n = (int)min((int64_t)kElems, a.batch - b0);
  const uint2 key = make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32));
  const uint64_t step = step_dev ? *step_dev : a.step;
  const int64_t HW = (int64_t)d.H * d.W;
  const int t = threadIdx.x;
  if (t < n) {
    int64_t ray, col;
    draw_element(a, (uint64_t)(HW * d.n_frames), d.n_instances, half, key, step, (uint64_t)(b0 + t), ray, col);
    s_ray[t] = ray;
    s_col[t] = col;
    const int64_t f = ray / HW, p = ray - f * HW, o = b0 + t;
    const int y = (int)(p / d.W), x = (int)(p - (int64_t)y * d.W);
    Cam c;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
      for (int j = 0; j < 3; ++j) c.r[3 * i + j] = __ldg(d.poses + f * 12 + 4 * i + j);
      c.t[i] = __ldg(d.poses + f * 12 + 4 * i + 3);
    }
    float* r8 = s_rays + t * 8;
    rotate_normalise(c, __ldg(d.directions + 3 * p), __ldg(d.directions + 3 * p + 1), __ldg(d.directions + 3 * p + 2),
                     r8[3], r8[4], r8[5]);
    r8[0] = c.t[0]; r8[1] = c.t[1]; r8[2] = c.t[2];
    r8[6] = d.near_s; r8[7] = d.far_s;
#pragma unroll
    for (int k = 0; k < 3; ++k) s_rgb[t * 3 + k] = __fdiv_rn((float)__ldg(d.rgb + ray * 3 + k), 255.0f);
    a.depths[o] = __ldg(d.depths + ray);
    a.valid_mask[o] = (x >= d.border && x < d.W - d.border && y >= d.border && y < d.H - d.border) ? 1 : 0;
    if (a.frame_idx) a.frame_idx[o] = __ldg(d.frame_idx + f);
    const int64_t id = __ldg(d.ids + col);
    uint8_t m = 1, pass = 1;
    if (d.labels && !__ldg(d.mask_all_ones + col)) {
      const int l = __ldg(d.labels + ray);
      m = l == id ? 1 : 0;
      pass = 0;
      for (int k = 0; k < d.n_pass; ++k) pass |= __ldg(d.pass_ids + col * d.n_pass + k) == l ? 1 : 0;
    }
    a.instance_mask[o] = m;
    a.instance_mask_weight[o] = __ldg(d.weights + (f * d.n_instances + col) * 2 + m);
    a.instance_ids[o] = id;
    a.pass_through_mask[o] = pass;
  }
  __syncthreads();
  for (int f = t; f < n * 8; f += kElems) a.rays[b0 * 8 + f] = s_rays[f];
  for (int f = t; f < n * 3; f += kElems) a.rgbs[b0 * 3 + f] = s_rgb[f];
  if (a.index_out)
    for (int f = t; f < n * 2; f += kElems) a.index_out[b0 * 2 + f] = (f & 1) ? s_col[f >> 1] : s_ray[f >> 1];
}

// the _dstep entries' last device work
__global__ void step_advance_kernel(uint64_t* step_dev) { *step_dev += 1; }

#define BATCH_CHECK(cond, msg)                  \
  do {                                          \
    if (!(cond)) {                              \
      onerf_set_error("%s: %s", fn, msg);       \
      return ONERF_ERR_BAD_ARG;                 \
    }                                           \
  } while (0)

// The refusals every entry shares, after its dataset's own: outputs, batch, ranks and the ray count.
int check_draw(const char* fn, const onerf_batch_args* a, int64_t n_rays, int n_instances, int* half) {
  BATCH_CHECK(a->rays && a->rgbs && a->depths && a->valid_mask && a->instance_mask && a->instance_mask_weight &&
                  a->instance_ids && a->pass_through_mask,
              "null output buffer");
  BATCH_CHECK(a->batch >= 1, "batch must be >= 1");
  BATCH_CHECK(a->world >= 1, "world must be >= 1");
  BATCH_CHECK(a->rank >= 0 && a->rank < a->world, "rank outside [0, world)");
  BATCH_CHECK(n_instances >= 1, "n_instances must be >= 1");
  BATCH_CHECK(n_rays < kMaxRays, "n_rays must be < 2^40");
  BATCH_CHECK(n_rays >= (int64_t)a->batch * a->world, "n_rays < batch * world: no full batch per epoch");
  int m = 2;
  while ((int64_t(1) << m) < n_rays) m += 2;
  *half = m / 2;
  return ONERF_OK;
}

// The refusals of onerf_draw_batch / _dstep; `fn` names the entry in the error message.
int check_batch_args(const char* fn, onerf_ctx* ctx, const onerf_batch_args* a, int* half) {
  BATCH_CHECK(ctx && a, "null argument");
  const onerf_ray_dataset& d = a->data;
  BATCH_CHECK(d.rays && d.rgbs && d.depths && d.valid_mask && d.instance_mask && d.instance_mask_weight &&
                  d.instance_ids && d.pass_through_mask,
              "null dataset buffer");
  return check_draw(fn, a, d.n_rays, d.n_instances, half);
}

// The refusals of onerf_draw_frames / _dstep.
int check_frame_args(const char* fn, onerf_ctx* ctx, const onerf_frame_dataset* d, const onerf_batch_args* a,
                     int* half) {
  BATCH_CHECK(ctx && d && a, "null argument");
  BATCH_CHECK(d->poses && d->directions && d->rgb && d->depths && d->frame_idx && d->ids && d->weights &&
                  (!d->labels || (d->mask_all_ones && d->pass_ids)),
              "null frame-store buffer");
  BATCH_CHECK(d->n_frames >= 1 && d->H >= 1 && d->W >= 1, "n_frames, H and W must be >= 1");
  BATCH_CHECK(d->border >= 0, "border must be >= 0");
  BATCH_CHECK(!d->labels || (d->n_pass >= 1 && d->n_pass <= kMaxPass), "n_pass outside [1, ONERF_FRAME_MAX_PASS]");
  const int64_t hw = (int64_t)d->H * d->W;
  BATCH_CHECK(hw < kMaxRays, "n_rays must be < 2^40");
  return check_draw(fn, a, hw * d->n_frames, d->n_instances, half);
}

int launch_draw(onerf_ctx* ctx, const onerf_frame_dataset* frames, const onerf_batch_args* a, int half,
                const uint64_t* step_dev, cudaStream_t stream) {
  const int blocks = (int)(((int64_t)a->batch + kElems - 1) / kElems);
  if (frames)
    draw_frames_kernel<<<blocks, kElems, 0, stream>>>(*frames, *a, half, step_dev);
  else
    draw_batch_kernel<<<blocks, kElems, 0, stream>>>(*a, half, step_dev);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int draw_dstep(const char* fn, onerf_ctx* ctx, const onerf_frame_dataset* frames, const onerf_batch_args* a, int half,
               uint64_t* step_dev, cudaStream_t stream) {
  BATCH_CHECK(step_dev, "null step_dev");
  BATCH_CHECK((reinterpret_cast<uintptr_t>(step_dev) & 7u) == 0, "step_dev must be 8-byte aligned");
  const int rc = launch_draw(ctx, frames, a, half, step_dev, stream);
  if (rc != ONERF_OK) return rc;
  step_advance_kernel<<<1, 1, 0, stream>>>(step_dev);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
#undef BATCH_CHECK

}  // namespace

extern "C" int onerf_draw_batch(onerf_ctx* ctx, const onerf_batch_args* a, void* stream) {
  int half = 0;
  const int rc = check_batch_args(__func__, ctx, a, &half);
  if (rc != ONERF_OK) return rc;
  return launch_draw(ctx, nullptr, a, half, nullptr, (cudaStream_t)stream);
}

extern "C" int onerf_draw_batch_dstep(onerf_ctx* ctx, const onerf_batch_args* a, uint64_t* step_dev, void* stream) {
  int half = 0;
  const int rc = check_batch_args(__func__, ctx, a, &half);
  if (rc != ONERF_OK) return rc;
  return draw_dstep(__func__, ctx, nullptr, a, half, step_dev, (cudaStream_t)stream);
}

extern "C" int onerf_draw_frames(onerf_ctx* ctx, const onerf_frame_dataset* frames, const onerf_batch_args* a,
                                 void* stream) {
  int half = 0;
  const int rc = check_frame_args(__func__, ctx, frames, a, &half);
  if (rc != ONERF_OK) return rc;
  return launch_draw(ctx, frames, a, half, nullptr, (cudaStream_t)stream);
}

extern "C" int onerf_draw_frames_dstep(onerf_ctx* ctx, const onerf_frame_dataset* frames, const onerf_batch_args* a,
                                       uint64_t* step_dev, void* stream) {
  int half = 0;
  const int rc = check_frame_args(__func__, ctx, frames, a, &half);
  if (rc != ONERF_OK) return rc;
  return draw_dstep(__func__, ctx, frames, a, half, step_dev, (cudaStream_t)stream);
}
