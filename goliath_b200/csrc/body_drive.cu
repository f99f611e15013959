// goliath_b200/csrc/body_drive.cu — the pieces of the drivable body avatar (ca_code/models/mesh_vae_drivable.py) that
// the mesh_vae kernels do not cover (sm_90a, fp32).
//
//   gb_face_tex_tail_fwd                the last layer of FaceDecoderFrontal.texmod (ca_code/nn/face.py:58, a k4 s2 p1
//                                       ConvTranspose2dWNUB with Cin <= 32 and Cout <= 4) with its untied bias, and in
//                                       the same pass the face bias and 255 (. + 0.5) of face.py:80-82: one thread per
//                                       output texel computes every output channel, the weights sit in shared memory.
//   gb_face_tex_cond_fwd                FaceEncoder's conditioning (mesh_vae_drivable.py:721-724): bilinear resize with
//                                       torch's fp32 half-pixel index, / 255 - 0.5, times the mask.
//   gb_pose_shadow_fwd / _bwd           PoseToShadow's sigmoid(x + beta) and bilinear resize (ca_code/nn/shadow.py:
//                                       466-470).  The forward evaluates the sigmoid at its four taps, so the
//                                       low-resolution map is never written; the backward runs one thread per
//                                       low-resolution texel, gathers its footprint in a fixed order and multiplies by
//                                       the sigmoid's derivative: no float atomics, the same bits on every call.
#include "common.cuh"

namespace {

constexpr int TT_X = 32, TT_Y = 8, TT_MAX_CIN = 32, TT_MAX_COUT = 4;

template <int COUT>
__global__ void __launch_bounds__(TT_X * TT_Y) face_tex_tail_kernel(int Cin, int Hi, int Wi, const float* __restrict__ x,
                                                                    const float* __restrict__ v,
                                                                    const float* __restrict__ scale,
                                                                    const float* __restrict__ ub,
                                                                    const float* __restrict__ face_bias,
                                                                    float* __restrict__ raw, float* __restrict__ tex) {
  __shared__ float w[TT_MAX_CIN * COUT * 16];  // weight_v [Cin, COUT, 4, 4]
  const int tid = threadIdx.y * TT_X + threadIdx.x;
  for (int i = tid; i < Cin * COUT * 16; i += TT_X * TT_Y) w[i] = v[i];
  __syncthreads();
  const int Ho = 2 * Hi, Wo = 2 * Wi;
  const int ox = blockIdx.x * TT_X + threadIdx.x, oy = blockIdx.y * TT_Y + threadIdx.y, b = blockIdx.z;
  if (ox >= Wo || oy >= Ho) return;
  // ConvTranspose2d(k=4, s=2, p=1): oy = 2 iy - 1 + ky, so ky has the parity of oy + 1 and there are two taps per axis
  const int ky0 = (oy + 1) & 1, kx0 = (ox + 1) & 1;
  int iy[2], ix[2];
  bool vy[2], vx[2];
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    iy[t] = (oy + 1 - ky0 - 2 * t) / 2;
    ix[t] = (ox + 1 - kx0 - 2 * t) / 2;
    vy[t] = iy[t] >= 0 && iy[t] < Hi;
    vx[t] = ix[t] >= 0 && ix[t] < Wi;
  }
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
  const size_t plane_in = (size_t)Hi * Wi;
  const float* X = x + (size_t)b * Cin * plane_in;
  for (int ci = 0; ci < Cin; ++ci) {
    const float* P = X + ci * plane_in;
#pragma unroll
    for (int ty = 0; ty < 2; ++ty) {
      if (!vy[ty]) continue;
#pragma unroll
      for (int tx = 0; tx < 2; ++tx) {
        if (!vx[tx]) continue;
        const float xv = __ldg(P + (size_t)iy[ty] * Wi + ix[tx]);
        const int k = (ky0 + 2 * ty) * 4 + kx0 + 2 * tx;
#pragma unroll
        for (int c = 0; c < COUT; ++c) acc[c] = fmaf(xv, w[(ci * COUT + c) * 16 + k], acc[c]);
      }
    }
  }
  const size_t plane = (size_t)Ho * Wo, o = (size_t)oy * Wo + ox;
#pragma unroll
  for (int c = 0; c < COUT; ++c) {
    const float r = acc[c] * scale[c] + ub[c * plane + o];
    raw[((size_t)b * COUT + c) * plane + o] = r;
    tex[((size_t)b * COUT + c) * plane + o] = 255.f * ((r + face_bias[c * plane + o]) + 0.5f);
  }
}

__global__ void __launch_bounds__(256) face_tex_cond_kernel(int C, int Hs, int Ws, int H, int W,
                                                            const float* __restrict__ x,
                                                            const float* __restrict__ mask, float* __restrict__ out) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y, b = blockIdx.z;
  if (px >= W) return;
  const gb::ResizeTap ty = gb::resize_tap(py, (float)Hs / (float)H, Hs);
  const gb::ResizeTap tx = gb::resize_tap(px, (float)Ws / (float)W, Ws);
  const float m = mask[(size_t)py * W + px];
  const size_t plane_in = (size_t)Hs * Ws, plane = (size_t)H * W;
  for (int c = 0; c < C; ++c) {
    const float* P = x + ((size_t)b * C + c) * plane_in;
    const float v = ty.l0 * (tx.l0 * P[(size_t)ty.i0 * Ws + tx.i0] + tx.l1 * P[(size_t)ty.i0 * Ws + tx.i1]) +
                    ty.l1 * (tx.l0 * P[(size_t)ty.i1 * Ws + tx.i0] + tx.l1 * P[(size_t)ty.i1 * Ws + tx.i1]);
    out[((size_t)b * C + c) * plane + (size_t)py * W + px] = (v / 255.f - 0.5f) * m;
  }
}

__device__ __forceinline__ float sigmoid_f(float v) { return 1.f / (1.f + expf(-v)); }

__global__ void __launch_bounds__(256) pose_shadow_fwd_kernel(int h, int w, int H, int W, const float* __restrict__ x,
                                                              float beta, float* __restrict__ out) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y, n = blockIdx.z;
  if (px >= W) return;
  const gb::ResizeTap ty = gb::resize_tap(py, (float)h / (float)H, h);
  const gb::ResizeTap tx = gb::resize_tap(px, (float)w / (float)W, w);
  const float* P = x + (size_t)n * h * w;
  const float s00 = sigmoid_f(P[ty.i0 * w + tx.i0] + beta), s01 = sigmoid_f(P[ty.i0 * w + tx.i1] + beta);
  const float s10 = sigmoid_f(P[ty.i1 * w + tx.i0] + beta), s11 = sigmoid_f(P[ty.i1 * w + tx.i1] + beta);
  out[(size_t)n * H * W + (size_t)py * W + px] =
      ty.l0 * (tx.l0 * s00 + tx.l1 * s01) + ty.l1 * (tx.l0 * s10 + tx.l1 * s11);
}

__global__ void __launch_bounds__(256) pose_shadow_bwd_kernel(int N, int h, int w, int H, int W,
                                                              const float* __restrict__ x, float beta,
                                                              const float* __restrict__ g_out,
                                                              float* __restrict__ g_x) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= N * h * w) return;
  const int n = t / (h * w), iy = (t / w) % h, ix = t % w;
  const float sy = (float)h / (float)H, sx = (float)w / (float)W;
  int ylo, yhi, xlo, xhi;
  gb::resize_footprint(iy, sy, H, ylo, yhi);
  gb::resize_footprint(ix, sx, W, xlo, xhi);
  const float* G = g_out + (size_t)n * H * W;
  float acc = 0.f;
  for (int y = ylo; y <= yhi; ++y) {
    const float wy = gb::resize_tap_weight(gb::resize_tap(y, sy, h), iy);
    if (wy == 0.f) continue;
    float row = 0.f;
    for (int px = xlo; px <= xhi; ++px) {
      const float wx = gb::resize_tap_weight(gb::resize_tap(px, sx, w), ix);
      if (wx != 0.f) row = fmaf(wx, G[(size_t)y * W + px], row);
    }
    acc = fmaf(wy, row, acc);
  }
  const float s = sigmoid_f(x[t] + beta);
  g_x[t] = acc * (1.f - s) * s;
}

}  // namespace

GB_API int gb_face_tex_tail_fwd(int B, int Cin, int Cout, int Hi, int Wi, const float* x, const float* weight_v,
                                const float* scale, const float* bias, const float* face_bias, float* tex_raw,
                                float* tex, void* stream) {
  if (B <= 0 || Hi <= 0 || Wi <= 0) return 0;
  if (Cin <= 0 || Cin > TT_MAX_CIN || Cout <= 0 || Cout > TT_MAX_COUT) return 1;
  const dim3 grid(gb::cdiv(2 * Wi, TT_X), gb::cdiv(2 * Hi, TT_Y), B), block(TT_X, TT_Y);
  cudaStream_t s = (cudaStream_t)stream;
#define GB_TAIL(C)                                                                                                     \
  GB_CUDA(gb::launch<face_tex_tail_kernel<C>>(grid, block, 0, s, Cin, Hi, Wi, x, weight_v, scale, bias, face_bias,     \
                                              tex_raw, tex))
  switch (Cout) {
    case 1: GB_TAIL(1); break;
    case 2: GB_TAIL(2); break;
    case 3: GB_TAIL(3); break;
    default: GB_TAIL(4); break;
  }
#undef GB_TAIL
  return 0;
}

GB_API int gb_face_tex_cond_fwd(int B, int C, int Hs, int Ws, int H, int W, const float* x, const float* mask,
                                float* out, void* stream) {
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0) return 0;
  if (Hs <= 0 || Ws <= 0) return 1;
  const dim3 grid(gb::cdiv(W, 256), H, B);
  return gb::launch<face_tex_cond_kernel>(grid, 256, 0, (cudaStream_t)stream, C, Hs, Ws, H, W, x, mask, out);
}

GB_API int gb_pose_shadow_fwd(int N, int h, int w, int H, int W, const float* x, float beta, float* out,
                              void* stream) {
  if (N <= 0 || H <= 0 || W <= 0) return 0;
  if (h <= 0 || w <= 0) return 1;
  const dim3 grid(gb::cdiv(W, 256), H, N);
  return gb::launch<pose_shadow_fwd_kernel>(grid, 256, 0, (cudaStream_t)stream, h, w, H, W, x, beta, out);
}

GB_API int gb_pose_shadow_bwd(int N, int h, int w, int H, int W, const float* x, float beta, const float* g_out,
                              float* g_x, void* stream) {
  if (N <= 0 || h <= 0 || w <= 0) return 0;
  if (H <= 0 || W <= 0) return 1;
  const int n = N * h * w;
  return gb::launch<pose_shadow_bwd_kernel>(gb::cdiv(n, 256), 256, 0, (cudaStream_t)stream, N, h, w, H, W, x, beta,
                                            g_out, g_x);
}
