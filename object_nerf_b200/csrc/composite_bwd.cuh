// Compositing backward of one branch of one ray (one warp), shared by composite_bwd_kernel (backward.cu), which first
// recomputes the forward, and the fused training compositing kernel (composite.cu), which runs it right after its own
// forward.  models/rendering.py:139-229 under autograd.
#pragma once
#include "common.cuh"

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
