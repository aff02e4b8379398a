// Volume-rendering arithmetic of one ray (one warp), forward and backward.  composite_scan is the only definition of
// alpha, the exclusive transmittance product and the weighted sums: composite_branch (the single-scene kernels of
// composite.cu and the recompute of composite_bwd_kernel in backward.cu) and both multi-object compositing kernels
// (composite.cu) call it and differ only in where their samples come from and where the weights go.
// composite_branch_grad is the compositing backward of one branch, shared by composite_bwd_kernel and the fused training
// compositing kernel.  models/rendering.py:139-229 (under autograd for the backward); render_tools/multi_rendering.py:96-157.
#pragma once
#include <algorithm>

#include "common.cuh"

__device__ __forceinline__ float alpha_from(float sigma, float delta) {
  // 1 - exp(-delta * relu(sigma))   (models/rendering.py:157)
  return __fsub_rn(1.0f, expf(__fmul_rn(-delta, fmaxf(sigma, 0.0f))));
}

struct Acc {
  float opacity, r, g, b, depth;
};

__device__ __forceinline__ Acc warp_sum(Acc a) {
  return Acc{warp_sum(a.opacity), warp_sum(a.r), warp_sum(a.g), warp_sum(a.b), warp_sum(a.depth)};
}

// inclusive multiplicative warp scan
__device__ __forceinline__ float warp_scan_mul(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v *= t;
  }
  return v;
}

// One sample as a loader of composite_scan hands it over: depth, distance to the next sample, rgb in f.xyz, the sigma
// alpha is taken from (noised or not), whether the occlusion mask zeroes its alpha, and where the caller found it.
struct Sample {
  float z, delta, sigma;
  float4 f;
  bool masked;
  int src;
};

// Composites samples [0, n) of one ray in 32-wide blocks, lane l taking sample base + l.  load(i) returns sample i;
// sink(i, sample, alpha, trans, w) receives its alpha, exclusive transmittance prod_{j < i} (1 - alpha_j + 1e-10) and
// weight alpha * trans; load(i) runs before sink(i) on the same lane.  Returns this lane's partial sums: warp_sum them
// for the ray's maps.  The operation order (rounding intrinsics, the weight grouped as alpha * (carry * excl), the
// transmittance taken before the carry advances) is what every caller's outputs are bit-identical to.
template <class Load, class Sink>
__device__ __forceinline__ Acc composite_scan(int n, int lane, Load load, Sink sink) {
  Acc acc = {0.f, 0.f, 0.f, 0.f, 0.f};
  float carry = 1.0f;  // prod_{j < block start} (1 - alpha_j + 1e-10)
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    Sample s = {0.f, 0.f, 0.f, make_float4(0.f, 0.f, 0.f, 0.f), false, 0};
    float alpha = 0.0f;
    if (i < n) {
      s = load(i);
      alpha = alpha_from(s.sigma, s.delta);
      if (s.masked) alpha = 0.0f;
    }
    const float t = (i < n) ? __fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f) : 1.0f;
    const float incl = warp_scan_mul(t, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.0f;
    const float trans = carry * excl;
    const float w = alpha * trans;
    carry *= __shfl_sync(0xffffffffu, incl, 31);
    if (i < n) {
      sink(i, s, alpha, trans, w);
      acc.opacity += w;
      acc.r += w * s.f.x;
      acc.g += w * s.f.y;
      acc.b += w * s.f.z;
      acc.depth += w * s.z;
    }
  }
  return acc;
}

// Composite one branch of one ray.  field = (S,4) rgb,sigma.  Returns this lane's partial sums (composite_scan).
// If w_out != nullptr the per-sample weights are stored; if s_alpha != nullptr, what composite_branch_grad reads
// (alpha, transmittance, noised sigma) goes to the warp's shared memory.  The noise is the caller's buffer or, without
// one, Philox stream `stream_id` at element ray * S + i, so a recompute with the same arguments replays the forward.
__device__ __forceinline__ Acc composite_branch(const float* __restrict__ z, const float4* __restrict__ field, int S,
                                                float last_delta, float noise_std, const float* __restrict__ noise,
                                                uint64_t seed, uint32_t stream_id, int64_t ray, bool use_mask,
                                                float z_limit, float* __restrict__ w_out, int lane,
                                                float* s_alpha = nullptr, float* s_trans = nullptr,
                                                float* s_sig = nullptr) {
  auto load = [&](int i) {
    const float zi = __ldg(z + i);
    const float delta = (i + 1 < S) ? __fsub_rn(__ldg(z + i + 1), zi) : last_delta;
    const float4 f = __ldg(field + i);
    float s = f.w;
    if (noise_std > 0.0f) {
      const float nz = noise ? __ldg(noise + i) : philox_normal(seed, stream_id, (uint64_t)ray * S + i);
      s = __fadd_rn(s, __fmul_rn(nz, noise_std));
    }
    // occlusion mask, models/rendering.py:192-202
    return Sample{zi, delta, s, f, use_mask && z_limit < zi, i};
  };
  auto sink = [&](int i, const Sample& s, float alpha, float trans, float w) {
    if (w_out) w_out[i] = w;
    if (s_alpha) {
      s_alpha[i] = alpha;
      s_trans[i] = trans;
      s_sig[i] = s.sigma;
    }
  };
  return composite_scan(S, lane, load, sink);
}

// inclusive suffix sum: v_i <- sum_{j >= i} v_j
__device__ __forceinline__ float composite_warp_suffix_add(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_down_sync(0xffffffffu, v, o);
    if (lane + o < 32) v += t;
  }
  return v;
}

// Per-warp shared memory of the forward, sample i of the branch: s_alpha[i] (after the occlusion mask), s_trans[i] (the
// exclusive transmittance product, weight = alpha * trans) and s_sig[i] (sigma with the noise added).  s_gw[S] is scratch.
// g_* = d(loss)/d(rgb, depth, opacity) of the branch's maps; dfield[i] <- d(r, g, b, sigma) of sample i.
__device__ __forceinline__ void composite_branch_grad(const float* __restrict__ z, const float4* __restrict__ field, int S,
                                                      float last_delta, bool use_mask, float z_limit, bool white, float g_r,
                                                      float g_g, float g_b, float g_d, float g_o, float4* __restrict__ dfield,
                                                      const float* s_alpha, const float* s_trans, const float* s_sig,
                                                      float* s_gw, int lane) {
  // dL/dw_i
  const float g_o_eff = g_o - (white ? (g_r + g_g + g_b) : 0.0f);
  for (int i = lane; i < S; i += 32) {
    const float4 f = __ldg(field + i);
    s_gw[i] = g_r * f.x + g_g * f.y + g_b * f.z + g_d * __ldg(z + i) + g_o_eff;
  }
  __syncwarp();
  // reverse pass: suffix sums of dL/dw_k * w_k for k > i
  float tail = 0.0f;
  const int nchunk = (S + 31) / 32;
  for (int c = nchunk - 1; c >= 0; --c) {
    const int i = c * 32 + lane;
    const bool in = i < S;
    const float alpha = in ? s_alpha[i] : 0.0f;
    const float T = in ? s_trans[i] : 0.0f;
    const float w = alpha * T;
    const float gw = in ? s_gw[i] : 0.0f;
    const float G = gw * w;
    const float incl = composite_warp_suffix_add(G, lane);
    const float after = incl - G + tail;          // sum over k > i
    tail += __shfl_sync(0xffffffffu, incl, 0);
    if (in) {
      const float zi = __ldg(z + i);
      const float delta = (i + 1 < S) ? __fsub_rn(__ldg(z + i + 1), zi) : last_delta;
      const float s = s_sig[i];
      const float t = __fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f);
      const float dalpha = gw * T - after / t;
      const bool masked = use_mask && z_limit < zi;
      // alpha = 1 - exp(-delta relu(s)):  d alpha / d s = delta exp(-delta s) for s > 0
      const float dsig = (masked || s <= 0.0f) ? 0.0f : dalpha * delta * expf(-delta * s);
      dfield[i] = make_float4(g_r * w, g_g * w, g_b * w, dsig);
    }
  }
}

// Grid of a one-warp-per-ray compositing launch: blocks of `warps` warps for every ray, at most 8 blocks per SM.
static inline int composite_blocks(const onerf_ctx* ctx, int n_rays, int warps) {
  return std::min((n_rays + warps - 1) / warps, ctx->num_sms * 8);
}
