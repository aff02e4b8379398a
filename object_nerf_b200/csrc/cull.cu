// Box culling of object ray sets on the editing path (api.cu: multi_fields).  A ray that misses an object's box has
// near = far = 0, so its depths end in 0 and the field kernel would only mute it (sigma = -1e5, mute_zero_rays).  These
// kernels list the other rays on the device, gather them into a dense set for the field kernel (which stops at the
// device-side count) and scatter the results back, filling the skipped rows with the muted value.  No host round trip.
#include <algorithm>

#include "field_common.cuh"

namespace {

constexpr int kCullThreads = 1024;

__device__ __forceinline__ bool ray_live(const float* __restrict__ z, int S, int r) {
  return __ldg(z + (int64_t)r * S + (S - 1)) != 0.0f;   // the criterion of mute_zero_rays
}

// One block: thread t owns rays [t * per, (t + 1) * per); a block scan of the per-thread counts gives each live ray its
// slot in ray order.  live[j] = ray of slot j, slot[r] = slot of ray r or -1, *count = number of live rays.
__global__ void __launch_bounds__(kCullThreads)
cull_list_kernel(const float* __restrict__ z, int n_rays, int S, int* __restrict__ live, int* __restrict__ slot,
                 int* __restrict__ count) {
  __shared__ int warp_tot[kCullThreads / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int per = (n_rays + kCullThreads - 1) / kCullThreads;
  const int r0 = min(t * per, n_rays), r1 = min(r0 + per, n_rays);
  int n = 0;
  for (int r = r0; r < r1; ++r) n += ray_live(z, S, r) ? 1 : 0;
  int incl = n;   // inclusive warp scan
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = warp_tot[lane], wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += v;
    }
    warp_tot[lane] = wi - w;   // exclusive
    if (lane == 31) *count = wi;
  }
  __syncthreads();
  int j = warp_tot[warp] + incl - n;
  for (int r = r0; r < r1; ++r) {
    if (ray_live(z, S, r)) {
      live[j] = r;
      slot[r] = j++;
    } else {
      slot[r] = -1;
    }
  }
}

// rays_c[j] = rays[live[j]], z_c[j] = z[live[j]] for j < *count; one warp per slot
__global__ void __launch_bounds__(256)
cull_gather_kernel(const float* __restrict__ rays, const float* __restrict__ z, int S, const int* __restrict__ live,
                   const int* __restrict__ count, float* __restrict__ rays_c, float* __restrict__ z_c) {
  const int n = *count;
  const int lane = threadIdx.x & 31;
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += (gridDim.x * blockDim.x) >> 5) {
    const int r = live[j];
    if (lane < 8) rays_c[(int64_t)j * 8 + lane] = __ldg(rays + (int64_t)r * 8 + lane);
    for (int s = lane; s < S; s += 32) z_c[(int64_t)j * S + s] = __ldg(z + (int64_t)r * S + s);
  }
}

// out[r][s] = field_c[slot[r]][s] for live rays, (0, 0, 0, -1e5) for the others
__global__ void __launch_bounds__(256)
cull_scatter_kernel(const float4* __restrict__ field_c, const int* __restrict__ slot, int n_rays, int S,
                    float4* __restrict__ out) {
  const int64_t total = (int64_t)n_rays * S;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / S), s = (int)(e - (int64_t)r * S);
    const int j = __ldg(slot + r);
    out[e] = j >= 0 ? __ldg(field_c + (int64_t)j * S + s) : make_float4(0.f, 0.f, 0.f, -1e5f);
  }
}

}  // namespace

int onerf_cull_rays(onerf_ctx* ctx, const float* rays, const float* z, int n_rays, int S, int* live, int* slot, int* count,
                    float* rays_c, float* z_c, cudaStream_t stream) {
  cull_list_kernel<<<1, kCullThreads, 0, stream>>>(z, n_rays, S, live, slot, count);
  ONERF_LAUNCH_CHECK(ctx);
  const int blocks = (int)std::min<int64_t>(((int64_t)n_rays + 7) / 8, (int64_t)ctx->num_sms * 8);
  cull_gather_kernel<<<blocks, 256, 0, stream>>>(rays, z, S, live, count, rays_c, z_c);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int onerf_uncull_field(onerf_ctx* ctx, const float* field_c, const int* slot, int n_rays, int S, float* out,
                       cudaStream_t stream) {
  const int64_t total = (int64_t)n_rays * S;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)ctx->num_sms * 16);
  cull_scatter_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const float4*>(field_c), slot, n_rays, S,
                                                  reinterpret_cast<float4*>(out));
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}
