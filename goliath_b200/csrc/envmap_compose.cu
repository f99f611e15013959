// goliath_b200/csrc/envmap_compose.cu — environment-map background and mirror-ball composite of the relighting frame
// (sm_90a).
//
// Replaces ca_code/utils/envmap.py:
//   rotate_envmap_mat (:141-166)  texel grid -> R * dir -> clamp -> dir2uv -> bilinear grid_sample (border,
//                                 align_corners=False); one thread per output texel, batched over B.
//   compose_envmap    (:325-345)  envmap_to_image (:169-227): camera rays -> R^T * dir -> normalise -> dir2uv ->
//                                 bicubic grid_sample (border, align_corners=True) -> 101x101 Gaussian blur (zero
//                                 padding 50); render + (1 - alpha) * clamp(bg, 0, 1); envmap_to_mirrorball (:230-248)
//                                 pasted at rows / columns [-200:] with its zsq < 1 mask.
// The blur kernel k (x) k / sum(k (x) k) is separable, so it runs as two 101-tap passes (exact in real arithmetic):
// 202 instead of 10,201 multiply-adds per pixel and channel.  Kernel 1 samples a row segment plus its 50-pixel halos
// into shared memory and runs the horizontal pass; kernel 2 runs the vertical pass on a column tile with its halos
// and composites (render, alpha, mirror ball) in the same pass.  The environment map (<= a few hundred KB) stays in
// L1/L2, so both kernels are bound by the blur arithmetic and one read + one write of the image per pass.
#include "envmap_common.cuh"

namespace {

constexpr float kPiGrid = 3.1415926f;                     // rotate_envmap_mat's texel grid uses this literal
constexpr float kA = -0.75f;                              // torch's bicubic convolution constant
constexpr float kFocalScale = 0.2f;                       // envmap_to_image(focal_scale=0.2)
constexpr int kBall = 200;                                // envmap_to_mirrorball(200, 200, ...)
constexpr int kR = 50, kTaps = 2 * kR + 1;                // 101-tap blur, padding 50

constexpr int kRowTile = 256;                             // kernel 1: outputs per block (one row segment)
constexpr int kColTile = 32, kRowsPer = 8, kColRows = 8 * kRowsPer;  // kernel 2: 32 columns x 64 rows per block

using gb::dir2uv;

// grid_sample's border padding applied to one tap (clip_coordinates + the in-bounds cast).  fmaxf maps a NaN
// coordinate to 0, so the fetch stays in bounds; the NaN weights still make the sample NaN, as in torch.
__device__ __forceinline__ int border_index(float c, int n) { return (int)fminf(fmaxf(c, 0.f), (float)(n - 1)); }

__device__ __forceinline__ float cubic1(float x) { return ((kA + 2.f) * x - (kA + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x) { return ((kA * x - 5.f * kA) * x + 8.f * kA) * x - 4.f * kA; }

// torch's bicubic rule (align_corners=True, padding_mode="border"): unnormalise, take the 4x4 taps around floor(i),
// clamp EACH tap to the border on its own (get_value_bounded), weights from the unclamped fraction.
struct Bicubic {
  int x[4], y[4];
  float wx[4], wy[4];
};

__device__ __forceinline__ void cubic_weights(float t, float w[4]) {
  w[0] = cubic2(t + 1.f);
  w[1] = cubic1(t);
  w[2] = cubic1(1.f - t);
  w[3] = cubic2(2.f - t);
}

__device__ __forceinline__ Bicubic bicubic_taps(float2 uv, int W, int H) {
  Bicubic b;
  const float ix = __fmul_rn(__fadd_rn(uv.x, 1.f), 0.5f * (float)(W - 1));
  const float iy = __fmul_rn(__fadd_rn(uv.y, 1.f), 0.5f * (float)(H - 1));
  const float fx = floorf(ix), fy = floorf(iy);
  cubic_weights(ix - fx, b.wx);
  cubic_weights(iy - fy, b.wy);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    b.x[k] = border_index(fx + (float)(k - 1), W);
    b.y[k] = border_index(fy + (float)(k - 1), H);
  }
  return b;
}

__device__ __forceinline__ float bicubic_fetch(const float* __restrict__ plane, const Bicubic& b, int W) {
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float* row = plane + (size_t)b.y[i] * W;
    const float r = row[b.x[0]] * b.wx[0] + row[b.x[1]] * b.wx[1] + row[b.x[2]] * b.wx[2] + row[b.x[3]] * b.wx[3];
    acc += r * b.wy[i];
  }
  return acc;
}

// torch.linspace(-1, 1, 200)[i] (float): start + step * i for the first half, end - step * (n - 1 - i) after.
__device__ __forceinline__ float ball_linspace(int i) {
  const float step = 2.f / (float)(kBall - 1);
  return i < kBall / 2 ? __fadd_rn(-1.f, __fmul_rn(step, (float)i)) : __fsub_rn(1.f, __fmul_rn(step, (float)(kBall - 1 - i)));
}

// envmap_to_mirrorball pixel (i, j) of the 200x200 ball: zsq < 1 mask and the unclamped bicubic lookup along the
// reflected view direction, rotated by R^T (einsum "bxy,bhwx->bhwy").  Returns the mask; col gets the colour.
__device__ __forceinline__ float mirror_pixel(int i, int j, const float* R, const float* __restrict__ env, int He,
                                              int We, float col[3]) {
  const float px = ball_linspace(j), py = ball_linspace(i);
  const float zsq = __fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py));
  const float nz = -sqrtf(fmaxf(__fsub_rn(1.f, zsq), 0.f));
  const float a = -2.f * nz;
  const float rx = __fmul_rn(a, px), ry = __fmul_rn(a, py), rz = __fadd_rn(1.f, __fmul_rn(a, nz));
  const float x = R[0] * rx + R[3] * ry + R[6] * rz;
  const float y = R[1] * rx + R[4] * ry + R[7] * rz;
  const float z = R[2] * rx + R[5] * ry + R[8] * rz;
  const Bicubic b = bicubic_taps(dir2uv(x, y, z), We, He);
  const size_t plane = (size_t)He * We;
#pragma unroll
  for (int c = 0; c < 3; ++c) col[c] = bicubic_fetch(env + c * plane, b, We);
  return zsq < 1.f ? 1.f : 0.f;
}

// torch.clamp(v, 0, 1): NaN stays NaN (fminf / fmaxf would drop it)
__device__ __forceinline__ float clamp01(float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); }

// the separable factor of the blur: k = exp(-linspace(-4, 4, 101)^2), normalised to sum 1 (its outer product is the
// reference's k (x) k / sum(k (x) k)).  Computed per block in double and rounded once.
__device__ void blur_weights(float* w) {
  __shared__ double kd[kTaps];
  const int t = threadIdx.x + threadIdx.y * blockDim.x;
  if (t < kTaps) {
    const float step = 8.f / (float)(kTaps - 1);
    const float x = t < kTaps / 2 ? __fadd_rn(-4.f, __fmul_rn(step, (float)t))
                                  : __fsub_rn(4.f, __fmul_rn(step, (float)(kTaps - 1 - t)));
    kd[t] = exp(-(double)x * (double)x);
  }
  __syncthreads();
  if (t < kTaps) {
    double s = 0.0;
    for (int k = 0; k < kTaps; ++k) s += kd[k];
    w[t] = (float)(kd[t] / s);
  }
  __syncthreads();
}

struct ComposeArgs {
  int B, H, W, He, We, rt_rows, rt_cols;
  const float *render, *alpha, *envbg, *K, *Rt;
  float *hblur, *out;
};

// R = Rt[b, :3, :3] as a row-major 3x3 in registers
__device__ __forceinline__ void load_rot(const ComposeArgs& a, int b, float R[9]) {
  const float* p = a.Rt + (size_t)b * a.rt_rows * a.rt_cols;
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) R[3 * r + c] = p[r * a.rt_cols + c];
}

// kernel 1: envmap_to_image's bicubic lookup for a row segment and its halos, then the horizontal blur pass.
// grid (cdiv(W, 256), H, B), block 256.
__global__ void __launch_bounds__(kRowTile) envmap_image_hblur_kernel(ComposeArgs a) {
  __shared__ float w[kTaps];
  __shared__ float s[3][kRowTile + 2 * kR];
  const int b = blockIdx.z, y = blockIdx.y, x0 = blockIdx.x * kRowTile;
  blur_weights(w);
  float R[9];
  load_rot(a, b, R);
  const float* Kb = a.K + 9 * b;
  const float fxs = __fmul_rn(Kb[0], kFocalScale), fys = __fmul_rn(Kb[4], kFocalScale);
  const float dy = __fdiv_rn(__fsub_rn((float)y, Kb[5]), fys);
  const float* env = a.envbg + (size_t)b * 3 * a.He * a.We;
  const size_t plane = (size_t)a.He * a.We;
  for (int k = threadIdx.x; k < kRowTile + 2 * kR; k += kRowTile) {
    const int x = x0 - kR + k;
    float col[3] = {0.f, 0.f, 0.f};  // the blur's zero padding
    if (x >= 0 && x < a.W) {
      const float dx = __fdiv_rn(__fsub_rn((float)x, Kb[2]), fxs);
      // R^T (dx, dy, 1), then F.normalize (eps 1e-12)
      float X = R[0] * dx + R[3] * dy + R[6];
      float Y = R[1] * dx + R[4] * dy + R[7];
      float Z = R[2] * dx + R[5] * dy + R[8];
      const float n = fmaxf(sqrtf(X * X + Y * Y + Z * Z), 1e-12f);
      X = __fdiv_rn(X, n); Y = __fdiv_rn(Y, n); Z = __fdiv_rn(Z, n);
      const Bicubic bc = bicubic_taps(dir2uv(X, Y, Z), a.We, a.He);
#pragma unroll
      for (int c = 0; c < 3; ++c) col[c] = bicubic_fetch(env + c * plane, bc, a.We);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) s[c][k] = col[c];
  }
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= a.W) return;
  float acc[3] = {0.f, 0.f, 0.f};
  for (int t = 0; t < kTaps; ++t) {
    const float wt = w[t];
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += wt * s[c][threadIdx.x + t];
  }
  const size_t hw = (size_t)a.H * a.W;
#pragma unroll
  for (int c = 0; c < 3; ++c) a.hblur[((size_t)b * 3 + c) * hw + (size_t)y * a.W + x] = acc[c];
}

// kernel 2: vertical blur pass on a 32 x 64 tile (+ 50-row halos, zero padding), then
// out = (1 - m) * (render + (1 - alpha) * clamp(bg, 0, 1)) + m * mirror  (m = 0 outside the 200x200 corner).
// grid (cdiv(W, 32), cdiv(H, 64), B), block (32, 8); each thread owns 8 consecutive rows of one column.
__global__ void __launch_bounds__(kColTile * 8) envmap_vblur_compose_kernel(ComposeArgs a) {
  __shared__ float w[kTaps];
  __shared__ float s[(kColRows + 2 * kR) * kColTile];
  const int b = blockIdx.z, tx = threadIdx.x, ty = threadIdx.y;
  const int x = blockIdx.x * kColTile + tx, y0 = blockIdx.y * kColRows;
  blur_weights(w);
  const size_t hw = (size_t)a.H * a.W;
  float acc[3][kRowsPer];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* src = a.hblur + ((size_t)b * 3 + c) * hw;
    if (c) __syncthreads();  // the previous channel's reads are done
    for (int r = ty; r < kColRows + 2 * kR; r += 8) {
      const int y = y0 - kR + r;
      s[r * kColTile + tx] = (x < a.W && y >= 0 && y < a.H) ? src[(size_t)y * a.W + x] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < kRowsPer; ++r) acc[c][r] = 0.f;
    const float* col = s + (ty * kRowsPer) * kColTile + tx;
#pragma unroll 4
    for (int t = 0; t < kTaps; ++t) {
      const float wt = w[t];
#pragma unroll
      for (int r = 0; r < kRowsPer; ++r) acc[c][r] += wt * col[(r + t) * kColTile];
    }
  }
  if (x >= a.W) return;
  float R[9];
  load_rot(a, b, R);
  const float* env = a.envbg + (size_t)b * 3 * a.He * a.We;
  const int by = a.H - kBall, bx = a.W - kBall;
#pragma unroll
  for (int r = 0; r < kRowsPer; ++r) {
    const int y = y0 + ty * kRowsPer + r;
    if (y >= a.H) break;
    const size_t p = (size_t)y * a.W + x;
    const float om = 1.f - a.alpha[(size_t)b * hw + p];
    float m = 0.f, mc[3] = {0.f, 0.f, 0.f};
    const bool in_ball = y >= by && x >= bx;
    if (in_ball) m = mirror_pixel(y - by, x - bx, R, env, a.He, a.We, mc);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const size_t o = ((size_t)b * 3 + c) * hw + p;
      const float comp = a.render[o] + om * clamp01(acc[c][r]);
      // the reference's (1 - mirror_alpha) * render + mirror_alpha * mirror_img; outside the corner m = 0 and the
      // mirror image is 0, so the output is the composite itself
      a.out[o] = in_ball ? (1.f - m) * comp + m * mc[c] : comp;
    }
  }
}

// g_render = (1 - m) * g: the mirror mask is the only path from the output back to `render`.
__global__ void envmap_compose_bwd_kernel(int B, int H, int W, const float* __restrict__ g, float* __restrict__ g_render) {
  const size_t hw = (size_t)H * W;
  const size_t n = (size_t)B * 3 * hw;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int p = (int)(i % hw);
    const int y = p / W, x = p - y * W;
    const int i_b = y - (H - kBall), j_b = x - (W - kBall);
    float v = g[i];
    if (i_b >= 0 && j_b >= 0) {
      const float px = ball_linspace(j_b), py = ball_linspace(i_b);
      const float m = __fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)) < 1.f ? 1.f : 0.f;
      v = (1.f - m) * v;
    }
    g_render[i] = v;
  }
}

// rotate_envmap_mat: one thread per output texel.  grid (cdiv(He * We, 256), B).
__global__ void __launch_bounds__(256) envmap_rotate_kernel(int B, int He, int We, const float* __restrict__ image,
                                                            const float* __restrict__ rot, float* __restrict__ out) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= He * We) return;
  const int i = t / We, j = t - i * We;
  // meshgrid((arange(H) + 0.5) * 3.1415926 / H, (arange(-W//2, W//2) + 0.5) * 3.1415926 * 2 / W), fp32 step by step
  const int j0 = -((We + 1) / 2);  // Python's -W // 2
  const float theta = __fdiv_rn(__fmul_rn(__fadd_rn((float)i, 0.5f), kPiGrid), (float)He);
  const float phi = __fdiv_rn(__fmul_rn(__fmul_rn(__fadd_rn((float)(j + j0), 0.5f), kPiGrid), 2.f), (float)We);
  const float st = sinf(theta);
  const float v0 = __fmul_rn(st, sinf(phi)), v1 = cosf(theta), v2 = __fmul_rn(st, cosf(phi));
  // vec @ R^T = R * vec, clamped to [-1, 1] per component
  const float* R = rot + 9 * b;
  const float x = fminf(fmaxf(R[0] * v0 + R[1] * v1 + R[2] * v2, -1.f), 1.f);
  const float y = fminf(fmaxf(R[3] * v0 + R[4] * v1 + R[5] * v2, -1.f), 1.f);
  const float z = fminf(fmaxf(R[6] * v0 + R[7] * v1 + R[8] * v2, -1.f), 1.f);
  const float2 uv = dir2uv(x, y, z);
  // bilinear grid_sample, align_corners=False, padding_mode="border": clip the coordinate, then the two neighbours
  // (the upper one only contributes when it is inside; its weight is 0 when the clip is active)
  const float ix = fminf(fmaxf(__fsub_rn(__fmul_rn(__fadd_rn(uv.x, 1.f), 0.5f * (float)We), 0.5f), 0.f), (float)(We - 1));
  const float iy = fminf(fmaxf(__fsub_rn(__fmul_rn(__fadd_rn(uv.y, 1.f), 0.5f * (float)He), 0.5f), 0.f), (float)(He - 1));
  const int x0 = (int)floorf(ix), y0 = (int)floorf(iy);
  const int x1 = min(x0 + 1, We - 1), y1 = min(y0 + 1, He - 1);
  const float fx = ix - (float)x0, fy = iy - (float)y0;
  const float w00 = (1.f - fx) * (1.f - fy), w01 = fx * (1.f - fy), w10 = (1.f - fx) * fy, w11 = fx * fy;
  const size_t plane = (size_t)He * We;
  const float* src = image + (size_t)b * 3 * plane;
  float* dst = out + (size_t)b * 3 * plane;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* p = src + c * plane;
    dst[c * plane + t] = p[y0 * We + x0] * w00 + p[y0 * We + x1] * w01 + p[y1 * We + x0] * w10 + p[y1 * We + x1] * w11;
  }
}

}  // namespace

GB_API int gb_envmap_rotate(int B, int He, int We, const float* image, const float* rot_mat, float* out, void* stream) {
  if (B <= 0) return 0;
  if (He < 1 || We < 1) return (int)cudaErrorInvalidValue;
  return gb::launch<envmap_rotate_kernel>(dim3(gb::cdiv(He * We, 256), B), 256, 0, (cudaStream_t)stream, B, He, We,
                                          image, rot_mat, out);
}

GB_API int gb_envmap_compose_fwd(int B, int H, int W, int He, int We, const float* render, const float* alpha,
                                 const float* envbg, const float* K, const float* Rt, int rt_rows, int rt_cols,
                                 float* hblur, float* out, void* stream) {
  if (B <= 0) return 0;
  if (H < kBall || W < kBall || He < 1 || We < 1 || rt_rows < 3 || rt_cols < 3) return (int)cudaErrorInvalidValue;
  ComposeArgs a = {B, H, W, He, We, rt_rows, rt_cols, render, alpha, envbg, K, Rt, hblur, out};
  const cudaStream_t st = (cudaStream_t)stream;
  GB_CUDA(gb::launch<envmap_image_hblur_kernel>(dim3(gb::cdiv(W, kRowTile), H, B), kRowTile, 0, st, a));
  return gb::launch<envmap_vblur_compose_kernel>(dim3(gb::cdiv(W, kColTile), gb::cdiv(H, kColRows), B),
                                                 dim3(kColTile, 8), 0, st, a);
}

GB_API int gb_envmap_compose_bwd(int B, int H, int W, const float* g_out, float* g_render, void* stream) {
  if (B <= 0) return 0;
  if (H < kBall || W < kBall) return (int)cudaErrorInvalidValue;
  const size_t n = (size_t)B * 3 * H * W;
  const int blocks = (int)(n < (size_t)gb::kNumSMs * 8 * 256 ? gb::cdiv64((int64_t)n, 256) : gb::kNumSMs * 8);
  return gb::launch<envmap_compose_bwd_kernel>(blocks, 256, 0, (cudaStream_t)stream, B, H, W, g_out, g_render);
}
