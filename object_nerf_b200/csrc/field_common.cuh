// Parameters shared by the field kernels (FFMA and wgmma) and their launchers.
#pragma once
#include <string.h>

#include "common.cuh"
#include "layout.h"

struct FieldParams {
  const float* rays;      // (N,8)
  const float* xyz;       // optional (N,S,3)
  const float* z;         // depth of sample i of ray r at z[r * z_stride + i]
  int64_t z_stride;
  const float* codes;     // (N,64) or null
  const float* code_row;  // (64,) or null
  int n_rays, S;
  onerf_grid grid;        // device pointers (unused for the plain-PE model)
  const void* packed;
  PackLayout L;
  int want_scene, want_object;
  int mute_zero_rays;
  const float* boxes;     // (n_boxes, 18)
  int n_boxes;
  float* scene_out;       // float4 (rgb, sigma) of sample i of ray r at [r * out_stride + i]
  float* obj_out;
  int64_t out_stride;
  float* ray_const;       // (N, ONERF_RAY_CONST_FLOATS)
  // backward support (FFMA kernel only): dump every layer's activations as [samples x width] row-major matrices
  //   dump_x: X (KO wide);  dump_s[0..7] scene hidden (256), [8] final (256), [9] dir (128);
  //   dump_o[0..3] object hidden (128), [4] final (128), [5] dir (64).  All null = no dump.
  float* dump_x;
  float* dump_s[10];
  float* dump_o[6];
  // training forward of the tensor-core kernel: bf16 activation atoms, X atoms and LeakyReLU sign masks of every tile
  // go to this workspace (layout.h: onerf_make_train_layout(use_voxel, n_rays * S)); null = inference
  void* train_ws;
  // optional device-side ray count (<= n_rays): only rays [0, *n_live) are evaluated.  Set by the editing path for object
  // ray sets compacted on the device to the rays that hit the object's box (api.cu: multi_fields).
  const int* n_live;
};

// Field parameters with the grid (NULL: plain-PE model), the packed weights and their layout set and all else zero.
static inline FieldParams onerf_field_params(const onerf_grid* grid, const void* packed) {
  FieldParams p;
  memset(&p, 0, sizeof(p));
  if (grid) p.grid = *grid;
  p.packed = packed;
  p.L = onerf_make_layout(grid ? 1 : 0);
  return p;
}

// rays a field launch evaluates: n_rays, or the device-side count when there is one (read once at kernel start)
__device__ __forceinline__ int field_rays(const FieldParams& p) {
  return p.n_live ? min(*p.n_live, p.n_rays) : p.n_rays;
}

// removed-object mask: inside any box <=> lo <= A p + t <= hi (inclusive), utils/bbox_utils.py:158-207
__device__ __forceinline__ bool point_in_boxes(const float* __restrict__ boxes, int n_boxes, float x, float y, float z) {
  bool inside = false;
  for (int b = 0; b < n_boxes; ++b) {
    const float* B = boxes + b * 18;
    bool in = true;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      // row-by-row dot product in the order of the reference's xyz @ A.T + t
      float v = __fmul_rn(x, __ldg(B + r * 3 + 0));
      v = __fadd_rn(v, __fmul_rn(y, __ldg(B + r * 3 + 1)));
      v = __fadd_rn(v, __fmul_rn(z, __ldg(B + r * 3 + 2)));
      v = __fadd_rn(v, __ldg(B + 9 + r));
      in = in && (v >= __ldg(B + 12 + r)) && (v <= __ldg(B + 15 + r));
    }
    inside = inside || in;
  }
  return inside;
}

int onerf_launch_ray_const(onerf_ctx* ctx, const FieldParams& p, cudaStream_t stream);
int onerf_launch_field_fp32(onerf_ctx* ctx, const FieldParams& p, cudaStream_t stream);
int onerf_launch_field_bf16(onerf_ctx* ctx, const FieldParams& p, cudaStream_t stream);
// The tensor-core field with the object branch once per code c in [0, n_codes) on one encoding of each sample: code c's
// per-ray constants at p.ray_const + c * rc_stride, its outputs at p.obj_out + c * obj_stride (floats), then the scene
// branch when p.want_scene.  Needs want_object, no training dump.
int onerf_launch_field_bf16_codes(onerf_ctx* ctx, const FieldParams& p, int n_codes, int64_t rc_stride,
                                  int64_t obj_stride, cudaStream_t stream);

// box culling of an (N,8) ray set with depths z (N,S) (cull.cu): live[0, *count) = rays whose last depth is not 0, in ray
// order, slot[r] = position of ray r in that list or -1; rays_c / z_c = the listed rays' rows.  uncull writes the field
// rows of the listed rays from field_c (count,S,4) to out (N,S,4) and (0, 0, 0, -1e5) to the others.
int onerf_cull_rays(onerf_ctx* ctx, const float* rays, const float* z, int n_rays, int S, int* live, int* slot, int* count,
                    float* rays_c, float* z_c, cudaStream_t stream);
int onerf_uncull_field(onerf_ctx* ctx, const float* field_c, const int* slot, int n_rays, int S, float* out,
                       cudaStream_t stream);
