// Pinhole camera arithmetic shared by the ray kernels (rays.cu) and the frame-store batch draw (batch.cu): both must
// produce the same bits for the same pixel and pose.  Reference: datasets/ray_utils.py:5-51.
#pragma once
#include "common.cuh"

struct Cam {
  float r[9], t[3];          // c2w (3,4)
  float half_w, half_h, focal;
  int H, W;
};

// datasets/ray_utils.py:17-23: no +0.5 pixel centring
__device__ __forceinline__ void pixel_direction(const Cam& c, int x, int y, float& dx, float& dy, float& dz) {
  dx = __fdiv_rn(__fsub_rn((float)x, c.half_w), c.focal);
  dy = -__fdiv_rn(__fsub_rn((float)y, c.half_h), c.focal);
  dz = -1.0f;
}

// datasets/ray_utils.py:42-44: d_world = directions @ c2w[:, :3].T, then / ||.|| (torch.norm accumulates in double on CPU)
__device__ __forceinline__ void rotate_normalise(const Cam& c, float dx, float dy, float dz, float& ox, float& oy, float& oz) {
  const float wx = __fmaf_rn(dz, c.r[2], __fmaf_rn(dy, c.r[1], __fmul_rn(dx, c.r[0])));
  const float wy = __fmaf_rn(dz, c.r[5], __fmaf_rn(dy, c.r[4], __fmul_rn(dx, c.r[3])));
  const float wz = __fmaf_rn(dz, c.r[8], __fmaf_rn(dy, c.r[7], __fmul_rn(dx, c.r[6])));
  const double n2 = (double)wx * wx + (double)wy * wy + (double)wz * wz;
  const float n = (float)sqrt(n2);
  ox = __fdiv_rn(wx, n);
  oy = __fdiv_rn(wy, n);
  oz = __fdiv_rn(wz, n);
}
