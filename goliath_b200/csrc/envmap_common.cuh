// goliath_b200/csrc/envmap_common.cuh — environment-map lookups shared by envmap_compose.cu, envmap_spec.cu and
// envmap_prefilter.cu: the reference's dir2uv and grid_sample's bilinear tap location and fetch.
#pragma once
#include "common.cuh"

namespace gb {

// u = atan2(x, z) / pi, v = 2 acos(y) / pi - 1 (ca_code/utils/envmap.py:213-215, 242-244, 158-160, 289-291).  No
// clamp before acos: |y| > 1 gives NaN, as torch.acos does.
__device__ __forceinline__ float2 dir2uv(float x, float y, float z) {
  constexpr float kInvPi = (float)(1.0 / 3.14159265358979323846);  // (1 / np.pi) as torch rounds it for fp32
  const float u = __fmul_rn(kInvPi, atan2f(x, z));
  const float v = __fmul_rn(kInvPi, acosf(y));
  return make_float2(u, __fsub_rn(__fmul_rn(2.f, v), 1.f));
}

struct Bilin {
  int x0, y0, x1, y1;
  float fx, fy;     // fractional weights of (x1, y1)
  float mx, my;     // gradient multipliers of the border clip (0 where clipped)
};

// grid_sample coordinate handling: align_corners=False unnormalisation, padding_mode="border" clip.  fmaxf maps a NaN
// coordinate to 0, as torch's clip_coordinates does on both devices, so a NaN coordinate samples the first row/column.
__device__ __forceinline__ Bilin locate(float u, float v, int W, int H) {
  Bilin b;
  float ix = ((u + 1.f) * (float)W - 1.f) * 0.5f;
  float iy = ((v + 1.f) * (float)H - 1.f) * 0.5f;
  b.mx = (ix < 0.f || ix > (float)(W - 1)) ? 0.f : 1.f;
  b.my = (iy < 0.f || iy > (float)(H - 1)) ? 0.f : 1.f;
  ix = fminf(fmaxf(ix, 0.f), (float)(W - 1));
  iy = fminf(fmaxf(iy, 0.f), (float)(H - 1));
  const float x0f = floorf(ix), y0f = floorf(iy);
  b.x0 = (int)x0f; b.y0 = (int)y0f;
  b.x1 = b.x0 + 1; b.y1 = b.y0 + 1;
  b.fx = ix - x0f; b.fy = iy - y0f;
  return b;
}

// one channel plane: value and its derivatives w.r.t. the (unclipped-scale) pixel coordinates
__device__ __forceinline__ float fetch(const float* __restrict__ p, const Bilin& b, int W, int H, float& ddx, float& ddy) {
  const bool x1in = b.x1 < W, y1in = b.y1 < H;  // out-of-range neighbours contribute zero (their weight is zero too)
  const float v00 = p[(size_t)b.y0 * W + b.x0];
  const float v01 = x1in ? p[(size_t)b.y0 * W + b.x1] : 0.f;
  const float v10 = y1in ? p[(size_t)b.y1 * W + b.x0] : 0.f;
  const float v11 = (x1in && y1in) ? p[(size_t)b.y1 * W + b.x1] : 0.f;
  const float wx0 = 1.f - b.fx, wy0 = 1.f - b.fy;
  ddx = (v01 - v00) * wy0 + (v11 - v10) * b.fy;
  ddy = (v10 - v00) * wx0 + (v11 - v01) * b.fx;
  return v00 * wx0 * wy0 + v01 * b.fx * wy0 + v10 * wx0 * b.fy + v11 * b.fx * b.fy;
}

}  // namespace gb
