// sigma -> alpha -> transmittance-weighted compositing, single-scene (scene + object branch) and the
// multi-object joint-sort variant.  One warp per ray, samples strided over lanes (coalesced float /
// float4 access); the scan itself is composite_core.cuh's composite_scan.
//
// Reference behaviour: models/rendering.py:139-229; render_tools/multi_rendering.py:96-157.
#include <float.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "composite_core.cuh"
#include "loss_terms.cuh"
#include "train_ws.h"
#include "../../include/onerf_ext.h"

namespace {

// kStep = false: the forward (onerf_composite).  kStep = true: the training step's compositing (onerf_train_step): the
// same forward, then per ray the squared errors of the loss terms this pass owns and their gradients w.r.t. the ray's
// maps (loss_terms.cuh; the normalisers depend on the batch only, so they are known before the render), then the
// compositing backward of both branches on the alpha / transmittance the forward left in shared memory
// (composite_core.cuh).  Per-block sums of the squared errors go to the fp64 accumulators; with `finalize` the last block
// to finish turns them into the loss outputs and the PSNR, and advances *seed_dev (train_ws.h: device seed), which every
// block has read by then.
// kEval (with kStep = false): the validation frame's compositing (onerf_validate_frame): the forward, then the ray's
// squared errors added to the same accumulators and, on the pass `st.psnr` selects, to the validation PSNR pair
// (loss_terms.cuh: VR_PSNR_*).  No gradients, no backward, no finalisation: the record is summed over chunks, tiles and
// ranks before validate_finalize_kernel (loss.cu) reads it.
template <bool kStep, bool kEval = false>
__global__ void __launch_bounds__(256) composite_kernel(onerf_composite_args a, onerf_step_composite st, uint64_t* seed_dev) {
  using namespace loss_terms;
  extern __shared__ float smem_c[];
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = a.n_samples;
  uint64_t seed = a.seed;
  if (seed_dev && a.noise_std > 0.0f) seed += *seed_dev;
  float *s_alpha = nullptr, *s_trans = nullptr, *s_sig = nullptr, *s_gw = nullptr;
  double sq[N_TERMS] = {0.0, 0.0, 0.0, 0.0, 0.0};   // lane 0: squared-error sums of this warp's rays
  double psnr[2] = {0.0, 0.0};                       // lane 0, kEval: masked squared-error sum and element count
  float scale[N_TERMS];
  if (kStep) {
    s_alpha = smem_c + (size_t)warp * 4 * S;
    s_trans = s_alpha + S;
    s_sig = s_trans + S;
    s_gw = s_sig + S;
    grad_scales(st.loss, st.acc, scale);
  }
  for (int r = blockIdx.x * warps_per_block + warp; r < a.n_rays; r += gridDim.x * warps_per_block) {
    const float* z = a.z + (int64_t)r * S;
    const bool obj_weights_out = (a.obj != nullptr) && a.rays_in_bbox;
    const float scene_last_delta = a.zero_last_delta ? 0.0f : 1e10f;
    const float4* scene = reinterpret_cast<const float4*>(a.scene) + (int64_t)r * S;
    const Acc sc = warp_sum(composite_branch(z, scene, S, scene_last_delta, a.noise_std,
                                             a.noise_scene ? a.noise_scene + (int64_t)r * S : nullptr, seed, 2u, r, false,
                                             0.0f, obj_weights_out ? nullptr : a.weights + (int64_t)r * S, lane, s_alpha,
                                             s_trans, s_sig));
    // white background: rgb + 1 - opacity, models/rendering.py:178-179
    const float rgb[3] = {a.white_back ? __fadd_rn(__fadd_rn(sc.r, 1.0f), -sc.opacity) : sc.r,
                          a.white_back ? __fadd_rn(__fadd_rn(sc.g, 1.0f), -sc.opacity) : sc.g,
                          a.white_back ? __fadd_rn(__fadd_rn(sc.b, 1.0f), -sc.opacity) : sc.b};
    if (lane == 0) {
      a.opacity[r] = sc.opacity;
      a.depth[r] = sc.depth;
      a.rgb[r * 3 + 0] = rgb[0];
      a.rgb[r * 3 + 1] = rgb[1];
      a.rgb[r * 3 + 2] = rgb[2];
    }
    Target tg;
    if (kEval) {
      tg = load_target(st.loss, r);
      if (lane == 0) {
        add_scene_sq(tg, rgb, sc.depth, sq, 1);
        add_psnr_sq(tg, st.psnr, rgb, psnr);
      }
    }
    if (kStep) {
      tg = load_target(st.loss, r);
      if (lane == 0) add_scene_sq(tg, rgb, sc.depth, sq, 1);
      float gc[3], gd;
      scene_grads(tg, rgb, sc.depth, scale, gc, gd);
      __syncwarp();
      composite_branch_grad(z, scene, S, scene_last_delta, false, 0.0f, a.white_back != 0, gc[0], gc[1], gc[2], gd, 0.0f,
                            reinterpret_cast<float4*>(st.dscene) + (int64_t)r * S, s_alpha, s_trans, s_sig, s_gw, lane);
      __syncwarp();
    }
    if (a.obj != nullptr) {
      bool use_mask = (!a.is_eval) && (a.frustum_bound_th > 0.0f);
      if (use_mask && a.pass_through_mask && a.pass_through_mask[r]) use_mask = false;
      const float z_limit = __fadd_rn(sc.depth, a.frustum_bound_th);
      const float4* obj = reinterpret_cast<const float4*>(a.obj) + (int64_t)r * S;
      const Acc ob = warp_sum(composite_branch(z, obj, S, 0.0f, a.noise_std,
                                               a.noise_obj ? a.noise_obj + (int64_t)r * S : nullptr, seed, 3u, r, use_mask,
                                               z_limit, obj_weights_out ? a.weights + (int64_t)r * S : nullptr, lane,
                                               s_alpha, s_trans, s_sig));
      // always composited on white, models/rendering.py:223
      const float irgb[3] = {__fadd_rn(__fadd_rn(ob.r, 1.0f), -ob.opacity), __fadd_rn(__fadd_rn(ob.g, 1.0f), -ob.opacity),
                             __fadd_rn(__fadd_rn(ob.b, 1.0f), -ob.opacity)};
      if (lane == 0) {
        a.opacity_instance[r] = ob.opacity;
        a.depth_instance[r] = ob.depth;
        a.rgb_instance[r * 3 + 0] = irgb[0];
        a.rgb_instance[r * 3 + 1] = irgb[1];
        a.rgb_instance[r * 3 + 2] = irgb[2];
      }
      if (kEval && lane == 0) add_object_sq(tg, ob.opacity, irgb, ob.depth, sq, 1);
      if (kStep) {
        if (lane == 0) add_object_sq(tg, ob.opacity, irgb, ob.depth, sq, 1);
        float go, gi[3], gid;
        object_grads(tg, ob.opacity, irgb, ob.depth, scale, go, gi, gid);
        __syncwarp();
        composite_branch_grad(z, obj, S, 0.0f, use_mask, z_limit, true, gi[0], gi[1], gi[2], gid, go,
                              reinterpret_cast<float4*>(st.dobj) + (int64_t)r * S, s_alpha, s_trans, s_sig, s_gw, lane);
        __syncwarp();
      }
    }
  }
  if (kEval) {
    __shared__ double red_e[8][N_TERMS + 2];
    if (lane == 0) {
      for (int t = 0; t < N_TERMS; ++t) red_e[warp][t] = sq[t];
      red_e[warp][N_TERMS] = psnr[0];
      red_e[warp][N_TERMS + 1] = psnr[1];
    }
    __syncthreads();
    if (threadIdx.x < N_TERMS + 2) {
      double v = 0.0;
      for (int w = 0; w < warps_per_block; ++w) v += red_e[w][threadIdx.x];
      double* dst = threadIdx.x < N_TERMS ? st.acc + WS_SUM + 2 * threadIdx.x + st.fine
                                          : st.acc + VR_PSNR_SUM + (threadIdx.x - N_TERMS);
      if (v != 0.0) atomicAdd(dst, v);
    }
    return;
  }
  if (!kStep) return;
  __shared__ double red[8][N_TERMS];
  if (lane == 0)
    for (int t = 0; t < N_TERMS; ++t) red[warp][t] = sq[t];
  __syncthreads();
  if (threadIdx.x < N_TERMS) {
    double v = 0.0;
    for (int w = 0; w < warps_per_block; ++w) v += red[w][threadIdx.x];
    if (v != 0.0) atomicAdd(st.acc + WS_SUM + 2 * threadIdx.x + st.fine, v);
    __threadfence();
  }
  if (!st.finalize) return;
  __shared__ bool last;
  __syncthreads();
  if (threadIdx.x == 0)
    last = atomicAdd(reinterpret_cast<unsigned int*>(st.acc + WS_DOUBLES), 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  double ws[WS_DOUBLES];
  for (int i = 0; i < WS_DOUBLES; ++i) ws[i] = __ldcg(st.acc + i);
  write_outputs(st.loss, ws);
  // train.py:171-172: psnr of the last pass's rgb over the valid rays = -10 log10 of that pass's colour term
  *st.psnr_out = (float)(-10.0 * log10(ws[WS_SUM + 2 * T_COLOR + st.fine] / ws[WS_COUNT + T_COLOR]));
  if (seed_dev) *seed_dev += ONERF_SEED_ADVANCE;
}

// One warp per (ray, code): code k's object field of ray r composited with exactly what composite_kernel passes for
// the object branch with is_eval set and no noise (last delta 0, no occlusion mask, no weights kept, on white), so
// column k is bit for bit that kernel's opacity_instance / depth_instance / rgb_instance of a render with code k.
__global__ void __launch_bounds__(256)
composite_instances_kernel(const float* __restrict__ z_all, const float* __restrict__ obj, int64_t obj_stride, int n_rays,
                           int S, int K, float* __restrict__ opacity, float* __restrict__ depth, float* __restrict__ rgb) {
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n_lists = (int64_t)n_rays * K;
  for (int64_t l = (int64_t)blockIdx.x * warps_per_block + warp; l < n_lists; l += (int64_t)gridDim.x * warps_per_block) {
    const int r = (int)(l / K), k = (int)(l % K);
    const float* z = z_all + (int64_t)r * S;
    const float4* f = reinterpret_cast<const float4*>(obj + k * obj_stride) + (int64_t)r * S;
    const Acc ob = warp_sum(composite_branch(z, f, S, 0.0f, 0.0f, nullptr, 0, 3u, r, false, 0.0f, nullptr, lane));
    if (lane == 0) {
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

// The forward-only call's last device work (onerf_render_rays_fwd_dseed).
__global__ void seed_advance_kernel(uint64_t* seed_dev) { *seed_dev += ONERF_SEED_ADVANCE; }

// ---------------------------------------------------------------------------------------------
// multi-object: joint stable sort by depth, then composite (last delta = 0)
// ---------------------------------------------------------------------------------------------
// Unsigned key ordered as the float's value.  -0.0 gets +0.0's key and every NaN, whatever its sign, the largest key, so
// with the concatenated index as the tie-break both paths give torch.sort(stable=True)'s order: zeros of either sign in
// index order, NaN last.
__device__ __forceinline__ uint32_t float_order_key(float f) {
  if (f != f) return 0xffffffffu;
  uint32_t u = __float_as_uint(f);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Offset of concatenated index c = obj * S + s of a ray in object-major storage [obj][ray][s] (obj_stride = n_rays * S),
// relative to sample 0 of the ray's first set.
__device__ __forceinline__ int64_t src_off(int c, int S, int64_t obj_stride) {
  return (int64_t)(c / S) * obj_stride + (c % S);
}

// lane 0 writes a multi-object ray's maps from the warp's sums
__device__ __forceinline__ void store_multi_maps(const Acc& acc, int white_back, int r, int lane, float* __restrict__ opacity,
                                                 float* __restrict__ rgb, float* __restrict__ depth) {
  if (lane == 0) {
    opacity[r] = acc.opacity;
    depth[r] = acc.depth;
    rgb[r * 3 + 0] = white_back ? __fadd_rn(__fadd_rn(acc.r, 1.0f), -acc.opacity) : acc.r;
    rgb[r * 3 + 1] = white_back ? __fadd_rn(__fadd_rn(acc.g, 1.0f), -acc.opacity) : acc.g;
    rgb[r * 3 + 2] = white_back ? __fadd_rn(__fadd_rn(acc.b, 1.0f), -acc.opacity) : acc.b;
  }
}

// Sigma noise of the joint compositing (render_tools/multi_rendering.py:131-132: one randn_like over the sorted sigmas):
// sorted sample p of ray r takes buf[r * T + p] if the caller gives a buffer, else Philox stream `stream_id`
// (ONERF_STREAM_MULTI_NOISE_COARSE / _FINE) at element r * T + p, keyed by `seed`.  Only read by the kNoise instances of
// the two compositing kernels; std == 0 launches the noise-free ones.
struct MultiNoise {
  float std;
  const float* buf;
  uint64_t seed;
  uint32_t stream_id;
};

// relu's argument sigma + noise * std, the multiply rounded first as the reference's (randn * std) + sigma
template <bool kNoise>
__device__ __forceinline__ float multi_sigma(float sigma, const MultiNoise& nz, int64_t e) {
  if (!kNoise) return sigma;
  const float v = nz.buf ? __ldg(nz.buf + e) : philox_normal(nz.seed, nz.stream_id, (uint64_t)e);
  return __fadd_rn(sigma, __fmul_rn(v, nz.std));
}

// One warp per ray.  Shared memory per warp: keys[P] (uint64: orderable z << 32 | concat index).
template <bool kNoise>
__global__ void __launch_bounds__(128)
composite_multi_kernel(const float* __restrict__ z_all, const float4* __restrict__ field_all, int n_rays,
                       int n_obj, int S, int P, int white_back, MultiNoise nz, float* __restrict__ z_sorted,
                       float* __restrict__ weights, float* __restrict__ obj_ids,
                       float* __restrict__ weights_unsorted, float* __restrict__ opacity,
                       float* __restrict__ rgb, float* __restrict__ depth) {
  extern __shared__ unsigned long long keys_all[];
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned long long* keys = keys_all + (size_t)warp * P;
  const int T = n_obj * S;
  for (int r = blockIdx.x * warps_per_block + warp; r < n_rays; r += gridDim.x * warps_per_block) {
    const int64_t obj_stride = (int64_t)n_rays * S;
    const float* z = z_all + (int64_t)r * S;
    const float4* fld = field_all + (int64_t)r * S;
    for (int i = lane; i < P; i += 32)
      keys[i] = (i < T) ? (((unsigned long long)float_order_key(__ldg(z + src_off(i, S, obj_stride))) << 32) | (unsigned)i)
                        : 0xffffffffffffffffull;
    warp_bitonic_sort(keys, P, lane);
    // composite in sorted order
    auto load = [&](int i) {
      const int src = (int)(keys[i] & 0xffffffffu);
      const float zi = __ldg(z + src_off(src, S, obj_stride));
      const float zn = (i + 1 < T) ? __ldg(z + src_off((int)(keys[i + 1] & 0xffffffffu), S, obj_stride)) : zi;
      const float delta = (i + 1 < T) ? __fsub_rn(zn, zi) : 0.0f;  // multi_rendering.py:125-128
      const float4 f = __ldg(fld + src_off(src, S, obj_stride));
      return Sample{zi, delta, multi_sigma<kNoise>(f.w, nz, (int64_t)r * T + i), f, false, src};
    };
    auto sink = [&](int i, const Sample& s, float, float, float w) {
      const int64_t o = (int64_t)r * T + i;
      z_sorted[o] = s.z;
      weights[o] = w;
      if (obj_ids) obj_ids[o] = (float)(s.src / S);
      if (weights_unsorted) weights_unsorted[(int64_t)r * S + src_off(s.src, S, obj_stride)] = w;
    };
    store_multi_maps(warp_sum(composite_scan(T, lane, load, sink)), white_back, r, lane, opacity, rgb, depth);
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------
// multi-object, any T: per-set sort, rank by binary search, composite in rank order.  Gives the same order as the
// bitonic kernel (a stable sort of the concatenation by float_order_key) without holding T keys in shared memory.
// Scratch (caller workspace), ray-major: skey[r][obj][p] = p-th smallest key of set obj of ray r, sidx[r][obj][p] = its
// sample index in the set.  The rank kernel leaves the concatenated index of sorted position i in weights[r][i] (as
// bits) and its depth in z_sorted[r][i]; the composite kernel reads both and overwrites weights[r][i] with the weight.
// ---------------------------------------------------------------------------------------------
constexpr int kMergeMaxS = 2048;   // per-set list sorted in shared memory; sidx is 16-bit

// One warp per (ray, set).  A set that is already ascending in key order (the usual case: unjittered coarse depths with
// near <= far, merged fine depths, all-zero muted rays) is copied; any other set is bitonic-sorted by (key, s).
__global__ void __launch_bounds__(128)
merge_sort_sets_kernel(const float* __restrict__ z_all, int n_rays, int n_obj, int S, int P,
                       uint32_t* __restrict__ skey, uint16_t* __restrict__ sidx) {
  extern __shared__ unsigned long long keys_all[];
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned long long* keys = keys_all + (size_t)warp * P;
  const int64_t n_lists = (int64_t)n_rays * n_obj;
  for (int64_t l = (int64_t)blockIdx.x * warps_per_block + warp; l < n_lists; l += (int64_t)gridDim.x * warps_per_block) {
    const int r = (int)(l / n_obj), obj = (int)(l % n_obj);
    const float* z = z_all + ((int64_t)obj * n_rays + r) * S;
    uint32_t* ko = skey + l * S;
    uint16_t* io = sidx + l * S;
    bool ascending = true;
    for (int s = lane; s + 1 < S; s += 32)
      ascending = ascending && (float_order_key(__ldg(z + s)) <= float_order_key(__ldg(z + s + 1)));
    if (__all_sync(0xffffffffu, ascending)) {
      for (int s = lane; s < S; s += 32) {
        ko[s] = float_order_key(__ldg(z + s));
        io[s] = (uint16_t)s;
      }
      continue;
    }
    for (int i = lane; i < P; i += 32)
      keys[i] = (i < S) ? (((unsigned long long)float_order_key(__ldg(z + i)) << 32) | (unsigned)i) : 0xffffffffffffffffull;
    warp_bitonic_sort(keys, P, lane);
    for (int s = lane; s < S; s += 32) {
      ko[s] = (uint32_t)(keys[s] >> 32);
      io[s] = (uint16_t)(keys[s] & 0xffffu);
    }
    __syncwarp();
  }
}

// number of entries of the ascending list k[0, n) that are < key (strict) or <= key
__device__ __forceinline__ int count_below(const uint32_t* __restrict__ k, int n, uint32_t key, bool strict) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const uint32_t v = __ldg(k + mid);
    if (strict ? (v < key) : (v <= key)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// One warp per (ray, set).  Sample p of sorted set obj goes to rank p + #(keys <= its key in sets before obj) +
// #(keys < its key in sets after obj): ties resolve in concatenated-index order, as the stable sort does.
__global__ void __launch_bounds__(128)
merge_rank_kernel(const float* __restrict__ z_all, int n_rays, int n_obj, int S, const uint32_t* __restrict__ skey,
                  const uint16_t* __restrict__ sidx, float* __restrict__ z_sorted, float* __restrict__ order) {
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n_lists = (int64_t)n_rays * n_obj;
  const int64_t T = (int64_t)n_obj * S;
  for (int64_t l = (int64_t)blockIdx.x * warps_per_block + warp; l < n_lists; l += (int64_t)gridDim.x * warps_per_block) {
    const int r = (int)(l / n_obj), obj = (int)(l % n_obj);
    const uint32_t* kr = skey + (int64_t)r * T;
    for (int p = lane; p < S; p += 32) {
      const uint32_t key = __ldg(kr + (int64_t)obj * S + p);
      const int s = __ldg(sidx + l * S + p);
      int rank = p;
      for (int q = 0; q < n_obj; ++q)
        if (q != obj) rank += count_below(kr + (int64_t)q * S, S, key, q > obj);
      const int64_t o = (int64_t)r * T + rank;
      z_sorted[o] = __ldg(z_all + ((int64_t)obj * n_rays + r) * S + s);
      order[o] = __uint_as_float((uint32_t)(obj * S + s));
    }
  }
}

// One warp per ray: composite_scan, as in composite_multi_kernel, over the order the rank kernel left in weights[] /
// z_sorted[].
template <bool kNoise>
__global__ void __launch_bounds__(128)
merge_composite_kernel(const float4* __restrict__ field_all, int n_rays, int n_obj, int S,
                       int white_back, MultiNoise nz, const float* __restrict__ z_sorted, float* __restrict__ weights,
                       float* __restrict__ obj_ids, float* __restrict__ weights_unsorted, float* __restrict__ opacity,
                       float* __restrict__ rgb, float* __restrict__ depth) {
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = n_obj * S;
  for (int r = blockIdx.x * warps_per_block + warp; r < n_rays; r += gridDim.x * warps_per_block) {
    const int64_t obj_stride = (int64_t)n_rays * S;
    const float4* fld = field_all + (int64_t)r * S;
    const float* zs = z_sorted + (int64_t)r * T;
    float* wr = weights + (int64_t)r * T;
    // each lane reads its order word wr[i] before its sink overwrites it with the weight
    auto load = [&](int i) {
      const int src = (int)__float_as_uint(wr[i]);
      const float zi = zs[i];
      const float zn = (i + 1 < T) ? zs[i + 1] : zi;
      const float delta = (i + 1 < T) ? __fsub_rn(zn, zi) : 0.0f;  // multi_rendering.py:125-128
      const float4 f = __ldg(fld + src_off(src, S, obj_stride));
      return Sample{zi, delta, multi_sigma<kNoise>(f.w, nz, (int64_t)r * T + i), f, false, src};
    };
    auto sink = [&](int i, const Sample& s, float, float, float w) {
      wr[i] = w;
      if (obj_ids) obj_ids[(int64_t)r * T + i] = (float)(s.src / S);
      if (weights_unsorted) weights_unsorted[(int64_t)r * S + src_off(s.src, S, obj_stride)] = w;
    };
    store_multi_maps(warp_sum(composite_scan(T, lane, load, sink)), white_back, r, lane, opacity, rgb, depth);
  }
}

// ---------------------------------------------------------------------------------------------
// Per-set maps of a joint compositing: for ray r and set i, the sums over set i's own samples of w, w z and w rgb, read in
// sample order from the weights scattered back to the sets (weights_unsorted, [obj][ray][s]) next to the set's depths
// and fields.  One warp per (ray, set): lane l sums samples l, l + 32, ... then warp_sum, an order fixed by S alone, so
// the maps do not depend on the sort path, the chunking or the tiling.  A zero weight adds nothing: a culled or muted
// sample's field value never reaches the maps (0 * inf would be NaN).  Outputs (n_rays, n_obj) / (n_rays, n_obj, 3),
// each skipped when NULL; no white background.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
set_maps_kernel(const float* __restrict__ z_all, const float4* __restrict__ field_all, const float* __restrict__ w_all,
                int n_rays, int n_obj, int S, float* __restrict__ opacity, float* __restrict__ depth,
                float* __restrict__ rgb) {
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n_lists = (int64_t)n_rays * n_obj;
  for (int64_t l = (int64_t)blockIdx.x * warps_per_block + warp; l < n_lists; l += (int64_t)gridDim.x * warps_per_block) {
    const int r = (int)(l / n_obj), obj = (int)(l % n_obj);
    const int64_t base = ((int64_t)obj * n_rays + r) * S;
    Acc acc = {0.f, 0.f, 0.f, 0.f, 0.f};
    for (int s = lane; s < S; s += 32) {
      const float w = __ldg(w_all + base + s);
      if (w != 0.0f) {
        const float4 f = __ldg(field_all + base + s);
        acc.opacity += w;
        acc.r += w * f.x;
        acc.g += w * f.y;
        acc.b += w * f.z;
        acc.depth += w * __ldg(z_all + base + s);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) {
      if (opacity) opacity[l] = acc.opacity;
      if (depth) depth[l] = acc.depth;
      if (rgb) {
        rgb[l * 3 + 0] = acc.r;
        rgb[l * 3 + 1] = acc.g;
        rgb[l * 3 + 2] = acc.b;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// One set of a source scene onto the frame's depth axis (k = s_src / s_base): z_out = z k for the joint compositing and
// the set maps, and the field's sigma / k in place, so that each interval keeps its optical depth sigma * delta.  z
// itself stays in the source's units for the set's importance sampling.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
rescale_set_kernel(const float* __restrict__ z, float* __restrict__ z_out, float4* __restrict__ field, int64_t n, float k) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    z_out[e] = z[e] * k;
    field[e].w = field[e].w / k;
  }
}

}  // namespace

int onerf_launch_rescale_set(onerf_ctx* ctx, const float* z, float* z_out, float* field, int64_t n, float k,
                             cudaStream_t stream) {
  if (n == 0) return ONERF_OK;
  const int threads = 256;
  const int blocks = (int)std::min((n + threads - 1) / threads, (int64_t)ctx->num_sms * 8);
  rescale_set_kernel<<<blocks, threads, 0, stream>>>(z, z_out, reinterpret_cast<float4*>(field), n, k);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int onerf_launch_set_maps(onerf_ctx* ctx, const float* z_all, const float* field_all, const float* weights_unsorted,
                          int n_rays, int n_obj, int n_samples, float* opacity, float* depth, float* rgb,
                          cudaStream_t stream) {
  if (n_rays == 0 || !(opacity || depth || rgb)) return ONERF_OK;
  const int warps = 4;
  const int64_t lists = (int64_t)n_rays * n_obj;
  const int blocks = (int)std::min((lists + warps - 1) / warps, (int64_t)ctx->num_sms * 16);
  set_maps_kernel<<<blocks, warps * 32, 0, stream>>>(z_all, reinterpret_cast<const float4*>(field_all), weights_unsorted,
                                                     n_rays, n_obj, n_samples, opacity, depth, rgb);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int onerf_launch_composite_instances(onerf_ctx* ctx, const float* z, const float* obj, int64_t obj_stride, int n_rays,
                                     int n_samples, int n_codes, float* opacity, float* depth, float* rgb,
                                     cudaStream_t stream) {
  if (n_rays == 0 || !(opacity || depth || rgb)) return ONERF_OK;
  const int warps = 8;
  const int64_t lists = (int64_t)n_rays * n_codes;
  const int blocks = (int)std::min((lists + warps - 1) / warps, (int64_t)ctx->num_sms * 8);
  composite_instances_kernel<<<blocks, warps * 32, 0, stream>>>(z, obj, obj_stride, n_rays, n_samples, n_codes, opacity,
                                                                depth, rgb);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

extern "C" int onerf_composite(onerf_ctx* ctx, const onerf_composite_args* a, void* stream) {
  return onerf_launch_composite(ctx, a, nullptr, (cudaStream_t)stream);
}

int onerf_launch_seed_advance(onerf_ctx* ctx, uint64_t* seed_dev, cudaStream_t stream) {
  seed_advance_kernel<<<1, 1, 0, stream>>>(seed_dev);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int onerf_launch_composite(onerf_ctx* ctx, const onerf_composite_args* a, uint64_t* seed_dev, cudaStream_t stream) {
  ONERF_CHECK_ARG(ctx && a, "null argument");
  ONERF_CHECK_ARG(a->z && a->scene && a->weights && a->opacity && a->rgb && a->depth, "null buffer");
  ONERF_CHECK_ARG(a->n_rays >= 0 && a->n_samples >= 1, "bad shape");
  ONERF_CHECK_ARG(onerf_aligned16(a->scene) && (!a->obj || onerf_aligned16(a->obj)), "field buffers must be 16-byte aligned");
  if (a->obj) ONERF_CHECK_ARG(a->rgb_instance && a->depth_instance && a->opacity_instance, "null instance output");
  if (a->n_rays == 0) return ONERF_OK;
  const int warps = 8;
  onerf_step_composite none;
  memset(&none, 0, sizeof(none));
  composite_kernel<false><<<composite_blocks(ctx, a->n_rays, warps), warps * 32, 0, stream>>>(*a, none, seed_dev);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int onerf_launch_composite_eval(onerf_ctx* ctx, const onerf_composite_args* a, const onerf_step_composite* t,
                                cudaStream_t stream) {
  if (a->n_rays == 0) return ONERF_OK;
  const int warps = 8;
  composite_kernel<false, true><<<composite_blocks(ctx, a->n_rays, warps), warps * 32, 0, stream>>>(*a, *t, nullptr);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

int onerf_launch_composite_step(onerf_ctx* ctx, const onerf_composite_args* a, const onerf_step_composite* t,
                                uint64_t* seed_dev, cudaStream_t stream) {
  ONERF_UNSUPPORTED(a->n_samples > 2048, "S > 2048");
  if (a->n_rays == 0) return ONERF_OK;
  const int warps = 4;
  const size_t smem = (size_t)warps * 4 * a->n_samples * sizeof(float);
  ONERF_CUDA(cudaFuncSetAttribute(composite_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  composite_kernel<true><<<composite_blocks(ctx, a->n_rays, warps), warps * 32, smem, stream>>>(*a, *t, seed_dev);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

// workspace of the rank-merge path: sorted keys (uint32) and in-set indices (uint16) of every sample
static size_t merge_ws_bytes(int64_t n_rays, int64_t T) { return ((n_rays * T * 4 + 255) & ~(int64_t)255) + n_rays * T * 2; }

extern "C" size_t onerf_composite_multi_workspace_bytes(int n_rays, int n_obj, int n_samples) {
  if (n_rays < 0 || n_obj < 1 || n_samples < 1) return 0;
  return merge_ws_bytes(n_rays, (int64_t)n_obj * n_samples);
}

// path: 0 = bitonic kernel (T <= 4096, no workspace), 1 = rank merge (any T up to the int32 / per-set bounds).
// nz.std == 0 runs the noise-free kernels.
static int composite_multi_run(onerf_ctx* ctx, int path, const float* z_all, const float* field_all, int n_rays, int n_obj,
                               int n_samples, int white_back, const MultiNoise& nz, float* z_sorted, float* weights,
                               float* obj_ids, float* weights_unsorted, float* opacity, float* rgb, float* depth,
                               void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  const int T = n_obj * n_samples;
  if (n_rays == 0) return ONERF_OK;
  const int warps = 4;
  const bool noise = nz.std != 0.0f;
  if (path == 0) {
    int P = 2;
    while (P < T) P <<= 1;
    const size_t smem = (size_t)warps * P * sizeof(unsigned long long);
    auto kernel = noise ? composite_multi_kernel<true> : composite_multi_kernel<false>;
    ONERF_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<composite_blocks(ctx, n_rays, warps), warps * 32, smem, stream>>>(
        z_all, reinterpret_cast<const float4*>(field_all), n_rays, n_obj, n_samples, P, white_back, nz, z_sorted,
        weights, obj_ids, weights_unsorted, opacity, rgb, depth);
    ONERF_LAUNCH_CHECK(ctx);
    return ONERF_OK;
  }
  uint32_t* skey = static_cast<uint32_t*>(workspace);
  uint16_t* sidx = reinterpret_cast<uint16_t*>(static_cast<char*>(workspace) + (((int64_t)n_rays * T * 4 + 255) & ~(int64_t)255));
  int P = 2;
  while (P < n_samples) P <<= 1;
  const size_t smem = (size_t)warps * P * sizeof(unsigned long long);
  ONERF_CUDA(cudaFuncSetAttribute(merge_sort_sets_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t lists = (int64_t)n_rays * n_obj;
  const int64_t cap = (int64_t)ctx->num_sms * 16;
  const int list_blocks = (int)std::min((lists + warps - 1) / warps, cap);
  merge_sort_sets_kernel<<<list_blocks, warps * 32, smem, stream>>>(z_all, n_rays, n_obj, n_samples, P, skey, sidx);
  ONERF_LAUNCH_CHECK(ctx);
  merge_rank_kernel<<<list_blocks, warps * 32, 0, stream>>>(z_all, n_rays, n_obj, n_samples, skey, sidx, z_sorted, weights);
  ONERF_LAUNCH_CHECK(ctx);
  auto kernel = noise ? merge_composite_kernel<true> : merge_composite_kernel<false>;
  kernel<<<composite_blocks(ctx, n_rays, warps), warps * 32, 0, stream>>>(
      reinterpret_cast<const float4*>(field_all), n_rays, n_obj, n_samples, white_back, nz, z_sorted, weights, obj_ids,
      weights_unsorted, opacity, rgb, depth);
  ONERF_LAUNCH_CHECK(ctx);
  return ONERF_OK;
}

static const MultiNoise kNoNoise = {0.0f, nullptr, 0, 0};

#define MULTI_ARGS_OK()                                                                                                 \
  ONERF_CHECK_ARG(ctx && z_all && field_all && z_sorted && weights && opacity && rgb && depth, "null argument");        \
  ONERF_CHECK_ARG(n_rays >= 0 && n_obj >= 1 && n_samples >= 1, "bad shape");                                            \
  ONERF_CHECK_ARG(onerf_aligned16(field_all), "field buffer must be 16-byte aligned")

extern "C" int onerf_composite_multi(onerf_ctx* ctx, const float* z_all, const float* field_all, int n_rays,
                                     int n_obj, int n_samples, int white_back, float* z_sorted,
                                     float* weights, float* obj_ids, float* weights_unsorted, float* opacity,
                                     float* rgb, float* depth, void* stream) {
  MULTI_ARGS_OK();
  ONERF_UNSUPPORTED((int64_t)n_obj * n_samples > 4096, "n_obj * n_samples > 4096 (onerf_composite_multi_ws has no such limit)");
  return composite_multi_run(ctx, 0, z_all, field_all, n_rays, n_obj, n_samples, white_back, kNoNoise, z_sorted, weights,
                             obj_ids, weights_unsorted, opacity, rgb, depth, nullptr, 0, (cudaStream_t)stream);
}

static int composite_multi_ws(onerf_ctx* ctx, int force_merge, const float* z_all, const float* field_all, int n_rays,
                              int n_obj, int n_samples, int white_back, const MultiNoise& nz, float* z_sorted,
                              float* weights, float* obj_ids, float* weights_unsorted, float* opacity, float* rgb,
                              float* depth, void* workspace, size_t workspace_bytes, void* stream) {
  MULTI_ARGS_OK();
  const int64_t T = (int64_t)n_obj * n_samples;
  const int path = (force_merge || T > 4096) ? 1 : 0;
  if (path == 1) {
    ONERF_UNSUPPORTED(T > INT32_MAX, "n_obj * n_samples >= 2^31");
    ONERF_UNSUPPORTED(n_samples > kMergeMaxS, "more than 2048 samples per ray set");
    const size_t need = onerf_composite_multi_workspace_bytes(n_rays, n_obj, n_samples);
    const int rc = onerf_check_workspace(__func__, workspace, workspace_bytes, need, ONERF_ERR_WORKSPACE);
    if (rc != ONERF_OK) return rc;
  }
  return composite_multi_run(ctx, path, z_all, field_all, n_rays, n_obj, n_samples, white_back, nz, z_sorted, weights,
                             obj_ids, weights_unsorted, opacity, rgb, depth, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int onerf_composite_multi_ws(onerf_ctx* ctx, const float* z_all, const float* field_all, int n_rays, int n_obj,
                                        int n_samples, int white_back, float* z_sorted, float* weights, float* obj_ids,
                                        float* weights_unsorted, float* opacity, float* rgb, float* depth, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  return composite_multi_ws(ctx, 0, z_all, field_all, n_rays, n_obj, n_samples, white_back, kNoNoise, z_sorted, weights,
                            obj_ids, weights_unsorted, opacity, rgb, depth, workspace, workspace_bytes, stream);
}

extern "C" int onerf_composite_multi_merge(onerf_ctx* ctx, const float* z_all, const float* field_all, int n_rays, int n_obj,
                                           int n_samples, int white_back, float* z_sorted, float* weights, float* obj_ids,
                                           float* weights_unsorted, float* opacity, float* rgb, float* depth, void* workspace,
                                           size_t workspace_bytes, void* stream) {
  return composite_multi_ws(ctx, 1, z_all, field_all, n_rays, n_obj, n_samples, white_back, kNoNoise, z_sorted, weights,
                            obj_ids, weights_unsorted, opacity, rgb, depth, workspace, workspace_bytes, stream);
}

// onerf_composite_multi_ws / _merge with sigma noise (include/onerf_ext.h)
static int composite_multi_noise(onerf_ctx* ctx, int force_merge, const float* z_all, const float* field_all, int n_rays,
                                 int n_obj, int n_samples, int white_back, float noise_std, const float* noise,
                                 uint64_t seed, int pass, float* z_sorted, float* weights, float* obj_ids,
                                 float* weights_unsorted, float* opacity, float* rgb, float* depth, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  ONERF_CHECK_ARG(noise_std >= 0.0f && noise_std <= FLT_MAX, "noise_std must be finite and >= 0");
  ONERF_CHECK_ARG(!noise || noise_std != 0.0f, "a noise buffer with noise_std = 0");
  ONERF_CHECK_ARG(onerf_aligned4(noise), "noise buffer must be 4-byte aligned");
  ONERF_CHECK_ARG(pass == 0 || pass == 1, "pass must be 0 (coarse) or 1 (fine)");
  const MultiNoise nz = {noise_std, noise, seed, pass ? ONERF_STREAM_MULTI_NOISE_FINE : ONERF_STREAM_MULTI_NOISE_COARSE};
  return composite_multi_ws(ctx, force_merge, z_all, field_all, n_rays, n_obj, n_samples, white_back, nz, z_sorted, weights,
                            obj_ids, weights_unsorted, opacity, rgb, depth, workspace, workspace_bytes, stream);
}

extern "C" int onerf_composite_multi_noise_ws(onerf_ctx* ctx, const float* z_all, const float* field_all, int n_rays,
                                              int n_obj, int n_samples, int white_back, float noise_std, const float* noise,
                                              uint64_t seed, int pass, float* z_sorted, float* weights, float* obj_ids,
                                              float* weights_unsorted, float* opacity, float* rgb, float* depth,
                                              void* workspace, size_t workspace_bytes, void* stream) {
  return composite_multi_noise(ctx, 0, z_all, field_all, n_rays, n_obj, n_samples, white_back, noise_std, noise, seed, pass,
                               z_sorted, weights, obj_ids, weights_unsorted, opacity, rgb, depth, workspace, workspace_bytes,
                               stream);
}

extern "C" int onerf_composite_multi_noise_merge(onerf_ctx* ctx, const float* z_all, const float* field_all, int n_rays,
                                                 int n_obj, int n_samples, int white_back, float noise_std,
                                                 const float* noise, uint64_t seed, int pass, float* z_sorted, float* weights,
                                                 float* obj_ids, float* weights_unsorted, float* opacity, float* rgb,
                                                 float* depth, void* workspace, size_t workspace_bytes, void* stream) {
  return composite_multi_noise(ctx, 1, z_all, field_all, n_rays, n_obj, n_samples, white_back, noise_std, noise, seed, pass,
                               z_sorted, weights, obj_ids, weights_unsorted, opacity, rgb, depth, workspace, workspace_bytes,
                               stream);
}
