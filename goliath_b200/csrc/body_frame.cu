// goliath_b200/csrc/body_frame.cu — the two pieces of the body avatar's frame that no other kernel covers (sm_90a).
//
//   gb_depth_disc_mask                  geom.depth_discontuity_mask (ca_code/utils/geom.py:768-794): Sobel x / y of the
//                                       depth with zero padding, |grad| > threshold, then the 3x3 stride-1 avg_pool > 0
//                                       (an any-neighbour dilation over pixels inside the image), in one kernel over a
//                                       shared-memory tile with a halo of two.
//   gb_pixel_bias_fwd / _bwd            rgb + CameraPixelBias(idx) (ca_code/models/mesh_vae.py:51-69 and :335-339): the
//                                       per-camera low-resolution bias, bilinearly stretched to the image with torch's
//                                       half-pixel index (align_corners=False), added to every channel.  The backward
//                                       runs one thread per (camera, bias texel) and gathers its footprint in a fixed
//                                       order: no float atomics, the same bits on every call.
#include "common.cuh"

namespace {

constexpr int DD_TX = 32, DD_TY = 8;

__global__ void __launch_bounds__(DD_TX * DD_TY) depth_disc_kernel(int H, int W, const float* __restrict__ depth,
                                                                   double threshold, unsigned char* __restrict__ out) {
  __shared__ float d[DD_TY + 4][DD_TX + 4];          // depth, halo 2, zero outside the image (conv2d's padding)
  __shared__ unsigned char e[DD_TY + 2][DD_TX + 2];  // |grad| > threshold, halo 1, false outside the image
  const int tid = threadIdx.y * DD_TX + threadIdx.x;
  const int x0 = blockIdx.x * DD_TX, y0 = blockIdx.y * DD_TY;
  const size_t plane = (size_t)H * W;
  const float* D = depth + blockIdx.z * plane;
  for (int i = tid; i < (DD_TY + 4) * (DD_TX + 4); i += DD_TX * DD_TY) {
    const int r = i / (DD_TX + 4), c = i % (DD_TX + 4);
    const int gy = y0 - 2 + r, gx = x0 - 2 + c;
    d[r][c] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? D[(size_t)gy * W + gx] : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < (DD_TY + 2) * (DD_TX + 2); i += DD_TX * DD_TY) {
    const int r = i / (DD_TX + 2), c = i % (DD_TX + 2);
    const int gy = y0 - 1 + r, gx = x0 - 1 + c;
    bool v = false;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      const int a = r + 1, b = c + 1;  // the pixel in d
      const double sx = ((double)d[a - 1][b + 1] - d[a - 1][b - 1]) + 2.0 * ((double)d[a][b + 1] - d[a][b - 1]) +
                        ((double)d[a + 1][b + 1] - d[a + 1][b - 1]);
      const double sy = ((double)d[a + 1][b - 1] + 2.0 * d[a + 1][b] + d[a + 1][b + 1]) -
                        ((double)d[a - 1][b - 1] + 2.0 * d[a - 1][b] + d[a - 1][b + 1]);
      v = sqrt(sx * sx + sy * sy) > threshold;
    }
    e[r][c] = v;
  }
  __syncthreads();
  const int px = x0 + threadIdx.x, py = y0 + threadIdx.y;
  if (px >= W || py >= H) return;
  unsigned char any = 0;
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) any |= e[threadIdx.y + r][threadIdx.x + c];
  out[blockIdx.z * plane + (size_t)py * W + px] = any;
}

__global__ void __launch_bounds__(256) pixel_bias_fwd_kernel(int B, int C, int H, int W, int n_cams, int Hb, int Wb,
                                                             const float* __restrict__ rgb,
                                                             const float* __restrict__ bias,
                                                             const long long* __restrict__ idx,
                                                             float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y, b = blockIdx.z;
  if (x >= W) return;
  const long long n = idx[b];
  float v = 0.f;
  if (n >= 0 && n < n_cams) {
    const float* P = bias + (size_t)n * Hb * Wb;
    const gb::ResizeTap ty = gb::resize_tap(y, (float)Hb / (float)H, Hb);
    const gb::ResizeTap tx = gb::resize_tap(x, (float)Wb / (float)W, Wb);
    v = ty.l0 * (tx.l0 * P[ty.i0 * Wb + tx.i0] + tx.l1 * P[ty.i0 * Wb + tx.i1]) +
        ty.l1 * (tx.l0 * P[ty.i1 * Wb + tx.i0] + tx.l1 * P[ty.i1 * Wb + tx.i1]);
  }
  const size_t plane = (size_t)H * W, o = (size_t)y * W + x;
  for (int c = 0; c < C; ++c) out[((size_t)b * C + c) * plane + o] = rgb[((size_t)b * C + c) * plane + o] + v;
}

__global__ void __launch_bounds__(256) pixel_bias_bwd_kernel(int B, int C, int H, int W, int n_cams, int Hb, int Wb,
                                                             const long long* __restrict__ idx,
                                                             const float* __restrict__ g_out,
                                                             float* __restrict__ g_bias) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_cams * Hb * Wb) return;
  const int n = t / (Hb * Wb), by = (t / Wb) % Hb, bx = t % Wb;
  const float sy = (float)Hb / (float)H, sx = (float)Wb / (float)W;
  int ylo, yhi, xlo, xhi;
  gb::resize_footprint(by, sy, H, ylo, yhi);
  gb::resize_footprint(bx, sx, W, xlo, xhi);
  const size_t plane = (size_t)H * W;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) {  // batch order
    if (idx[b] != n) continue;
    const float* G = g_out + (size_t)b * C * plane;
    float item = 0.f;
    for (int y = ylo; y <= yhi; ++y) {
      const float wy = gb::resize_tap_weight(gb::resize_tap(y, sy, Hb), by);
      if (wy == 0.f) continue;
      float row = 0.f;
      for (int x = xlo; x <= xhi; ++x) {
        const float wx = gb::resize_tap_weight(gb::resize_tap(x, sx, Wb), bx);
        if (wx == 0.f) continue;
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += G[c * plane + (size_t)y * W + x];
        row += wx * s;
      }
      item += wy * row;
    }
    acc += item;
  }
  g_bias[t] = acc;
}

}  // namespace

GB_API int gb_depth_disc_mask(int B, int H, int W, const float* depth, float threshold, unsigned char* mask,
                              void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  const dim3 grid(gb::cdiv(W, DD_TX), gb::cdiv(H, DD_TY), B);
  return gb::launch<depth_disc_kernel>(grid, dim3(DD_TX, DD_TY), 0, (cudaStream_t)stream, H, W, depth,
                                       (double)threshold, mask);
}

GB_API int gb_pixel_bias_fwd(int B, int C, int H, int W, int n_cams, int Hb, int Wb, const float* rgb,
                             const float* bias, const long long* idx, float* out, void* stream) {
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0) return 0;
  if (n_cams <= 0 || Hb <= 0 || Wb <= 0) return 1;
  const dim3 grid(gb::cdiv(W, 256), H, B);
  return gb::launch<pixel_bias_fwd_kernel>(grid, 256, 0, (cudaStream_t)stream, B, C, H, W, n_cams, Hb, Wb, rgb, bias,
                                           idx, out);
}

GB_API int gb_pixel_bias_bwd(int B, int C, int H, int W, int n_cams, int Hb, int Wb, const long long* idx,
                             const float* g_out, float* g_bias, void* stream) {
  if (n_cams <= 0 || Hb <= 0 || Wb <= 0) return 0;
  if (H <= 0 || W <= 0) return 1;
  const int n = n_cams * Hb * Wb;
  return gb::launch<pixel_bias_bwd_kernel>(gb::cdiv(n, 256), 256, 0, (cudaStream_t)stream, B, C, H, W, n_cams, Hb, Wb,
                                           idx, g_out, g_bias);
}
