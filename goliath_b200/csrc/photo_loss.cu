// goliath_b200/csrc/photo_loss.cu — post-render chain + photometric losses of the RGCA train step, fused (sm_90a).
// SURVEY.md section 8f-2.  Replaces, per frame, the eager chain
//   rgb = cal(rgb, cam)                          ca_code/nn/color_cal.py:211-241  (CalV5: w * img + b; grey cameras: sum_c)
//   rgb = rgb + (1 - alpha) * bg                 ca_code/models/rgca.py:226-230
//   rgb = w0 rgb + w1 G3(rgb) + w2 G7(rgb)       ca_code/nn/dof_cal.py:44-56      (torchvision gaussian_blur, reflect pad)
//   l1   = mean(|(rgb - image) * mask|)          ca_code/loss/__init__.py:391-410
//   ssim = sum(ssim_map(image, rgb) * mask) / clamp(sum(mask), 1)   ca_code/loss/__init__.py:479-494, utils/ssim.py:25-63
// (11x11 Gaussian window, sigma 1.5, zero padding, C1 = 1e-4, C2 = 9e-4) and everything autograd derives from it
// (~60 launches and ~40 full-image passes) by four kernels:
//   post_render_fwd   cal + background composite + learnable blur, one pass, separable blurs in shared memory
//   ssim_l1_fwd       per 32x32 tile: the five windowed statistics by separable convolution in shared memory, the
//                     masked SSIM / L1 sums (one atomic triple per CTA) and the three derivative maps of the map
//   ssim_l1_bwd       dL/dpred = window * D_mu + 2 pred (window * D_pp) + target (window * D_tp) + L1 sign term
//   post_render_bwd   adjoint of the reflect-padded blurs (border-aware weights), adjoint of cal; gradients of the
//                     image, of the calibration (w, b) and of the blur weights (block reduction + atomics)
// The result of post_render_bwd is dL/d(rendered rgb): what the blend backward consumes as v_out.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kTile = 32;          // pixels per CTA side
constexpr int kThreads = 256;
constexpr int kR7 = 3, kR3 = 1;    // blur radii
constexpr int kRS = 5;             // SSIM window radius (11 taps)
constexpr float kC1 = 0.01f * 0.01f, kC2 = 0.03f * 0.03f;

struct Taps {
  float g3[3], g7[7], gs[11];
};

__device__ __forceinline__ int reflect(int i, int n) {  // torch "reflect" padding, radius < n
  i = i < 0 ? -i : i;
  i = i >= n ? 2 * n - 2 - i : i;
  return min(max(i, 0), n - 1);  // (only reached by tile pixels that lie outside a very small image; never stored)
}

struct PostArgs {
  int B, H, W;
  const float *rgb, *alpha, *bg, *cal_w, *cal_b, *blur_w;  // rgb [B,3,H,W]; alpha [B,1,H,W]; bg [B,3,H,W] or null;
  const int* grey;                                          // cal_w / cal_b [B,3] or null; blur_w [B,3] or null; grey [B] or null
  float* pred;                                              // [B,3,H,W]
  // backward
  const float* g_pred;
  float *g_rgb, *g_cal_w, *g_cal_b, *g_blur_w;  // g_rgb [B,3,H,W]; the parameter gradients [B,3], accumulated (zeroed by the caller)
};

// x2 = cal(rgb) + (1 - alpha) * bg for one pixel (all three channels)
__device__ __forceinline__ void cal_compose(const PostArgs& a, int b, int y, int x, float out[3]) {
  const size_t plane = (size_t)a.H * a.W, p = (size_t)y * a.W + x;
  const float* src = a.rgb + (size_t)b * 3 * plane + p;
  float v[3] = {src[0], src[plane], src[2 * plane]};
  if (a.cal_w) {
    const float w0 = a.cal_w[3 * b], w1 = a.cal_w[3 * b + 1], w2 = a.cal_w[3 * b + 2];
    const float b0 = a.cal_b[3 * b], b1 = a.cal_b[3 * b + 1], b2 = a.cal_b[3 * b + 2];
    if (a.grey && a.grey[b]) {
      const float s = v[0] * w0 + v[1] * w1 + v[2] * w2 + (b0 + b1 + b2);
      v[0] = v[1] = v[2] = s;
    } else {
      v[0] = v[0] * w0 + b0; v[1] = v[1] * w1 + b1; v[2] = v[2] * w2 + b2;
    }
  }
  if (a.bg) {
    const float t = 1.f - a.alpha[(size_t)b * plane + p];
    const float* g = a.bg + (size_t)b * 3 * plane + p;
    v[0] += t * g[0]; v[1] += t * g[plane]; v[2] += t * g[2 * plane];
  }
  out[0] = v[0]; out[1] = v[1]; out[2] = v[2];
}

// shared tile of x2 with a halo of 3 (reflect-indexed at the image border), one channel at a time
constexpr int kHaloB = kR7, kSideB = kTile + 2 * kHaloB;  // 38

__device__ __forceinline__ void load_x2_tile(const PostArgs& a, int b, int ty0, int tx0, float (*s)[kSideB][kSideB + 1]) {
  for (int i = threadIdx.x; i < kSideB * kSideB; i += kThreads) {
    const int ly = i / kSideB, lx = i - ly * kSideB;
    const int gy = reflect(ty0 + ly - kHaloB, a.H), gx = reflect(tx0 + lx - kHaloB, a.W);
    float v[3];
    cal_compose(a, b, gy, gx, v);
    s[0][ly][lx] = v[0]; s[1][ly][lx] = v[1]; s[2][ly][lx] = v[2];
  }
}

// blurred values (G3, G7) of channel c at tile pixel (ly, lx) from the shared x2 tile
__device__ __forceinline__ void blur_at(const float (*s)[kSideB + 1], const Taps& t, int ly, int lx, float& b3, float& b7) {
  const int cy = ly + kHaloB, cx = lx + kHaloB;
  float acc7 = 0.f, acc3 = 0.f;
#pragma unroll
  for (int dy = -kR7; dy <= kR7; ++dy) {
    float row7 = 0.f, row3 = 0.f;
#pragma unroll
    for (int dx = -kR7; dx <= kR7; ++dx) {
      const float v = s[cy + dy][cx + dx];
      row7 += t.g7[dx + kR7] * v;
      if (dx >= -kR3 && dx <= kR3) row3 += t.g3[dx + kR3] * v;
    }
    acc7 += t.g7[dy + kR7] * row7;
    if (dy >= -kR3 && dy <= kR3) acc3 += t.g3[dy + kR3] * row3;
  }
  b3 = acc3; b7 = acc7;
}

__global__ void __launch_bounds__(kThreads) post_render_fwd_kernel(PostArgs a, Taps t) {
  __shared__ float s_x2[3][kSideB][kSideB + 1];
  const int b = blockIdx.z, ty0 = blockIdx.y * kTile, tx0 = blockIdx.x * kTile;
  const size_t plane = (size_t)a.H * a.W;
  if (!a.blur_w) {  // no blur: purely per pixel
    for (int i = threadIdx.x; i < kTile * kTile; i += kThreads) {
      const int y = ty0 + i / kTile, x = tx0 + i % kTile;
      if (y >= a.H || x >= a.W) continue;
      float v[3];
      cal_compose(a, b, y, x, v);
      float* dst = a.pred + (size_t)b * 3 * plane + (size_t)y * a.W + x;
      dst[0] = v[0]; dst[plane] = v[1]; dst[2 * plane] = v[2];
    }
    return;
  }
  load_x2_tile(a, b, ty0, tx0, s_x2);
  __syncthreads();
  const float w0 = a.blur_w[3 * b], w1 = a.blur_w[3 * b + 1], w2 = a.blur_w[3 * b + 2];
  for (int i = threadIdx.x; i < kTile * kTile; i += kThreads) {
    const int ly = i / kTile, lx = i % kTile, y = ty0 + ly, x = tx0 + lx;
    if (y >= a.H || x >= a.W) continue;
    float* dst = a.pred + (size_t)b * 3 * plane + (size_t)y * a.W + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float b3, b7;
      blur_at(s_x2[c], t, ly, lx, b3, b7);
      dst[c * plane] = w0 * s_x2[c][ly + kHaloB][lx + kHaloB] + w1 * b3 + w2 * b7;
    }
  }
}

// 1-D adjoint weight of a reflect-padded convolution: contribution of output y to input x (even taps w, radius r)
__device__ __forceinline__ float adj_w(const float* w, int r, int x, int y, int n) {
  float s = 0.f;
  const int d0 = x - y;
  if (d0 >= -r && d0 <= r) s += w[d0 + r];
  if (x >= 1) { const int d1 = -x - y; if (d1 >= -r) s += w[d1 + r]; }                     // via the left mirror (z = -x)
  if (x <= n - 2) { const int d2 = 2 * n - 2 - x - y; if (d2 <= r) s += w[d2 + r]; }       // via the right mirror
  return s;
}

__device__ __forceinline__ float block_sum(float v, float* s_red) {
  v = gb::warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float r = 0.f;
  if (warp == 0) {
    r = lane < kThreads / 32 ? s_red[lane] : 0.f;
    r = gb::warp_sum(r);
  }
  return r;  // valid in warp 0
}

__global__ void __launch_bounds__(kThreads) post_render_bwd_kernel(PostArgs a, Taps t) {
  __shared__ float s_x2[3][kSideB][kSideB + 1];   // forward recomputation (blur-weight gradients)
  __shared__ float s_g[3][kSideB][kSideB + 1];    // dL/dpred with a halo of 3 (zero outside the image)
  __shared__ float s_red[kThreads / 32];
  const int b = blockIdx.z, ty0 = blockIdx.y * kTile, tx0 = blockIdx.x * kTile;
  const size_t plane = (size_t)a.H * a.W;
  const bool blur = a.blur_w != nullptr;
  float w0 = 1.f, w1 = 0.f, w2 = 0.f;
  if (blur) {
    w0 = a.blur_w[3 * b]; w1 = a.blur_w[3 * b + 1]; w2 = a.blur_w[3 * b + 2];
    load_x2_tile(a, b, ty0, tx0, s_x2);
    for (int i = threadIdx.x; i < kSideB * kSideB; i += kThreads) {
      const int ly = i / kSideB, lx = i - ly * kSideB, gy = ty0 + ly - kHaloB, gx = tx0 + lx - kHaloB;
      const bool in = gy >= 0 && gy < a.H && gx >= 0 && gx < a.W;
      const float* g = a.g_pred + (size_t)b * 3 * plane + (size_t)gy * a.W + gx;
      s_g[0][ly][lx] = in ? g[0] : 0.f; s_g[1][ly][lx] = in ? g[plane] : 0.f; s_g[2][ly][lx] = in ? g[2 * plane] : 0.f;
    }
    __syncthreads();
  }
  float acc_bw[3] = {0.f, 0.f, 0.f}, acc_w[3] = {0.f, 0.f, 0.f}, acc_b[3] = {0.f, 0.f, 0.f};
  const bool grey = a.grey && a.grey[b];
  for (int i = threadIdx.x; i < kTile * kTile; i += kThreads) {
    const int ly = i / kTile, lx = i % kTile, y = ty0 + ly, x = tx0 + lx;
    if (y >= a.H || x >= a.W) continue;
    const size_t p = (size_t)y * a.W + x;
    float gx2[3];  // dL/dx2 at this pixel
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (!blur) {
        gx2[c] = a.g_pred[(size_t)b * 3 * plane + c * plane + p];
        continue;
      }
      // forward values at this pixel for the blur-weight gradients
      float b3, b7;
      blur_at(s_x2[c], t, ly, lx, b3, b7);
      const float gc = s_g[c][ly + kHaloB][lx + kHaloB];
      acc_bw[0] += gc * s_x2[c][ly + kHaloB][lx + kHaloB];
      acc_bw[1] += gc * b3;
      acc_bw[2] += gc * b7;
      // adjoint of the reflect-padded separable blurs
      float a7 = 0.f, a3 = 0.f;
#pragma unroll
      for (int dy = -kR7; dy <= kR7; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= a.H) continue;
        const float wy7 = adj_w(t.g7, kR7, y, yy, a.H);
        const float wy3 = (dy >= -kR3 && dy <= kR3) ? adj_w(t.g3, kR3, y, yy, a.H) : 0.f;
        float r7 = 0.f, r3 = 0.f;
#pragma unroll
        for (int dx = -kR7; dx <= kR7; ++dx) {
          const int xx = x + dx;
          if (xx < 0 || xx >= a.W) continue;
          const float g = s_g[c][ly + kHaloB + dy][lx + kHaloB + dx];
          r7 += adj_w(t.g7, kR7, x, xx, a.W) * g;
          if (dx >= -kR3 && dx <= kR3) r3 += adj_w(t.g3, kR3, x, xx, a.W) * g;
        }
        a7 += wy7 * r7;
        a3 += wy3 * r3;
      }
      gx2[c] = w0 * gc + w1 * a3 + w2 * a7;
    }
    // adjoint of cal (the background term is additive and alpha is detached upstream)
    float* dst = a.g_rgb + (size_t)b * 3 * plane + p;
    if (a.cal_w) {
      const float* src = a.rgb + (size_t)b * 3 * plane + p;
      const float v0 = src[0], v1 = src[plane], v2 = src[2 * plane];
      const float cw0 = a.cal_w[3 * b], cw1 = a.cal_w[3 * b + 1], cw2 = a.cal_w[3 * b + 2];
      if (grey) {
        const float gs = gx2[0] + gx2[1] + gx2[2];
        dst[0] = gs * cw0; dst[plane] = gs * cw1; dst[2 * plane] = gs * cw2;
        acc_w[0] += gs * v0; acc_w[1] += gs * v1; acc_w[2] += gs * v2;
        acc_b[0] += gs; acc_b[1] += gs; acc_b[2] += gs;
      } else {
        dst[0] = gx2[0] * cw0; dst[plane] = gx2[1] * cw1; dst[2 * plane] = gx2[2] * cw2;
        acc_w[0] += gx2[0] * v0; acc_w[1] += gx2[1] * v1; acc_w[2] += gx2[2] * v2;
        acc_b[0] += gx2[0]; acc_b[1] += gx2[1]; acc_b[2] += gx2[2];
      }
    } else {
      dst[0] = gx2[0]; dst[plane] = gx2[1]; dst[2 * plane] = gx2[2];
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (blur && a.g_blur_w) {
      const float r = block_sum(acc_bw[c], s_red);
      if (threadIdx.x == 0) atomicAdd(a.g_blur_w + 3 * b + c, r);
    }
    if (a.cal_w && a.g_cal_w) {
      const float rw = block_sum(acc_w[c], s_red);
      if (threadIdx.x == 0) atomicAdd(a.g_cal_w + 3 * b + c, rw);
      const float rb = block_sum(acc_b[c], s_red);
      if (threadIdx.x == 0) atomicAdd(a.g_cal_b + 3 * b + c, rb);
    }
  }
}

// ------------------------------------------------------------------ SSIM + L1
struct LossArgs {
  int B, H, W;
  const float *pred, *target, *mask;  // [B,3,H,W] [B,3,H,W] [B,1,H,W]
  float *d_mu, *d_pp, *d_tp;          // derivative maps [B,3,H,W] (mask already applied)
  double* sums;                       // [3]: sum |delta * mask|, sum ssim * mask, sum mask (x3 channels)
  // backward: g_pred = g_loss * (l1_coef * sign * mask - ssim_w / clamp(sums[2], 1) * d(sum ssim * mask)/d pred)
  const float* g_loss;                // device scalar (upstream gradient of the loss) or null (= 1)
  float l1_coef, ssim_w;              // l1_weight / (B*3*H*W), ssim_weight
  float* g_pred;
};

constexpr int kSideS = kTile + 2 * kRS;  // 42

__global__ void __launch_bounds__(kThreads) ssim_l1_fwd_kernel(LossArgs a, Taps t) {
  // one channel plane per blockIdx.z; zero padding outside the image (F.conv2d padding = 5)
  __shared__ float s_p[kSideS][kSideS + 1], s_t[kSideS][kSideS + 1];
  __shared__ float s_h[5][kSideS][kTile + 1];  // horizontally filtered: t, p, tt, pp, tp
  __shared__ float s_red[kThreads / 32];
  const int bc = blockIdx.z, b = bc / 3, ty0 = blockIdx.y * kTile, tx0 = blockIdx.x * kTile;
  const size_t plane = (size_t)a.H * a.W;
  const float* P = a.pred + (size_t)bc * plane;
  const float* T = a.target + (size_t)bc * plane;
  for (int i = threadIdx.x; i < kSideS * kSideS; i += kThreads) {
    const int ly = i / kSideS, lx = i - ly * kSideS, gy = ty0 + ly - kRS, gx = tx0 + lx - kRS;
    const bool in = gy >= 0 && gy < a.H && gx >= 0 && gx < a.W;
    s_p[ly][lx] = in ? P[(size_t)gy * a.W + gx] : 0.f;
    s_t[ly][lx] = in ? T[(size_t)gy * a.W + gx] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kSideS * kTile; i += kThreads) {
    const int ly = i / kTile, lx = i - ly * kTile;
    float st = 0.f, sp = 0.f, stt = 0.f, spp = 0.f, stp = 0.f;
#pragma unroll
    for (int k = 0; k < 11; ++k) {
      const float w = t.gs[k], pv = s_p[ly][lx + k], tv = s_t[ly][lx + k];
      st += w * tv; sp += w * pv; stt += w * tv * tv; spp += w * pv * pv; stp += w * tv * pv;
    }
    s_h[0][ly][lx] = st; s_h[1][ly][lx] = sp; s_h[2][ly][lx] = stt; s_h[3][ly][lx] = spp; s_h[4][ly][lx] = stp;
  }
  __syncthreads();
  float acc_l1 = 0.f, acc_ss = 0.f, acc_m = 0.f;
  for (int i = threadIdx.x; i < kTile * kTile; i += kThreads) {
    const int ly = i / kTile, lx = i - ly * kTile, y = ty0 + ly, x = tx0 + lx;
    if (y >= a.H || x >= a.W) continue;
    float mt = 0.f, mp = 0.f, ett = 0.f, epp = 0.f, etp = 0.f;
#pragma unroll
    for (int k = 0; k < 11; ++k) {
      const float w = t.gs[k];
      mt += w * s_h[0][ly + k][lx]; mp += w * s_h[1][ly + k][lx]; ett += w * s_h[2][ly + k][lx];
      epp += w * s_h[3][ly + k][lx]; etp += w * s_h[4][ly + k][lx];
    }
    const float st2 = ett - mt * mt, sp2 = epp - mp * mp, stp = etp - mt * mp;
    const float A1 = 2.f * mt * mp + kC1, A2 = 2.f * stp + kC2, B1 = mt * mt + mp * mp + kC1, B2 = st2 + sp2 + kC2;
    const float iB1 = 1.f / B1, iB2 = 1.f / B2;
    const float S = A1 * A2 * iB1 * iB2;
    const size_t p = (size_t)y * a.W + x;
    const float m = a.mask[(size_t)b * plane + p];
    // derivatives of S with the window outputs mu_p, E[pp], E[tp] taken as independent variables
    const float dS_dtp = 2.f * A1 * iB1 * iB2;
    const float dS_dpp = -S * iB2;
    const float dS_dmu = 2.f * mt * (A2 - A1) * iB1 * iB2 - 2.f * mp * S * (iB1 - iB2);
    a.d_mu[(size_t)bc * plane + p] = m * dS_dmu;
    a.d_pp[(size_t)bc * plane + p] = m * dS_dpp;
    a.d_tp[(size_t)bc * plane + p] = m * dS_dtp;
    acc_ss += S * m;
    acc_m += m;
    acc_l1 += fabsf((s_p[ly + kRS][lx + kRS] - s_t[ly + kRS][lx + kRS]) * m);
  }
  const float r0 = block_sum(acc_l1, s_red);
  const float r1 = block_sum(acc_ss, s_red);
  const float r2 = block_sum(acc_m, s_red);
  if (threadIdx.x == 0) {
    atomicAdd(a.sums + 0, (double)r0);
    atomicAdd(a.sums + 1, (double)r1);
    atomicAdd(a.sums + 2, (double)r2);
  }
}

__global__ void __launch_bounds__(kThreads) ssim_l1_bwd_kernel(LossArgs a, Taps t) {
  __shared__ float s_d[3][kSideS][kSideS + 1];       // the three derivative maps with a halo of 5 (zero outside)
  __shared__ float s_h[3][kSideS][kTile + 1];
  const int bc = blockIdx.z, b = bc / 3, ty0 = blockIdx.y * kTile, tx0 = blockIdx.x * kTile;
  const size_t plane = (size_t)a.H * a.W;
  const float gl = a.g_loss ? *a.g_loss : 1.f;
  const float scale_l1 = gl * a.l1_coef;
  const float scale_ssim = -gl * a.ssim_w / (float)fmax(a.sums[2], 1.0);
  const float* D[3] = {a.d_mu + (size_t)bc * plane, a.d_pp + (size_t)bc * plane, a.d_tp + (size_t)bc * plane};
  for (int i = threadIdx.x; i < kSideS * kSideS; i += kThreads) {
    const int ly = i / kSideS, lx = i - ly * kSideS, gy = ty0 + ly - kRS, gx = tx0 + lx - kRS;
    const bool in = gy >= 0 && gy < a.H && gx >= 0 && gx < a.W;
#pragma unroll
    for (int q = 0; q < 3; ++q) s_d[q][ly][lx] = in ? D[q][(size_t)gy * a.W + gx] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kSideS * kTile; i += kThreads) {
    const int ly = i / kTile, lx = i - ly * kTile;
    float r[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 11; ++k) {
#pragma unroll
      for (int q = 0; q < 3; ++q) r[q] += t.gs[k] * s_d[q][ly][lx + k];
    }
    s_h[0][ly][lx] = r[0]; s_h[1][ly][lx] = r[1]; s_h[2][ly][lx] = r[2];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kTile * kTile; i += kThreads) {
    const int ly = i / kTile, lx = i - ly * kTile, y = ty0 + ly, x = tx0 + lx;
    if (y >= a.H || x >= a.W) continue;
    float c[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 11; ++k) {
#pragma unroll
      for (int q = 0; q < 3; ++q) c[q] += t.gs[k] * s_h[q][ly + k][lx];
    }
    const size_t p = (size_t)y * a.W + x;
    const float pv = a.pred[(size_t)bc * plane + p], tv = a.target[(size_t)bc * plane + p];
    const float m = a.mask[(size_t)b * plane + p];
    const float d = (pv - tv) * m;
    const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
    a.g_pred[(size_t)bc * plane + p] = scale_ssim * (c[0] + 2.f * pv * c[1] + tv * c[2]) + scale_l1 * sgn * m;
  }
}

void make_taps(Taps& t) {
  auto fill = [](float* w, int n, double sigma) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) {
      const double x = i - (n - 1) * 0.5;
      w[i] = (float)exp(-x * x / (2.0 * sigma * sigma));
      s += w[i];
    }
    for (int i = 0; i < n; ++i) w[i] = (float)(w[i] / s);
  };
  // torchvision gaussian_blur default sigma = 0.3 * ((k - 1) * 0.5 - 1) + 0.8 -> 0.8 (k = 3), 1.4 (k = 7)
  fill(t.g3, 3, 0.8);
  fill(t.g7, 7, 1.4);
  fill(t.gs, 11, 1.5);  // utils/ssim.py:14-20
}

}  // namespace

// pred = blur(cal(rgb) + (1 - alpha) * bg).  Optional stages are skipped when their pointers are NULL: cal_w / cal_b [B,3]
// (grey [B] int32 marks grey cameras), bg [B,3,H,W] (needs alpha [B,1,H,W]), blur_w [B,3] (softmaxed weights).
GB_API int gb_post_render_fwd(int B, int H, int W, const float* rgb, const float* alpha, const float* bg, const float* cal_w,
                              const float* cal_b, const int32_t* grey, const float* blur_w, float* pred, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  if (H <= kR7 || W <= kR7) return (int)cudaErrorInvalidValue;  // reflect padding needs radius < size
  PostArgs a = {};
  a.B = B; a.H = H; a.W = W; a.rgb = rgb; a.alpha = alpha; a.bg = bg; a.cal_w = cal_w; a.cal_b = cal_b; a.grey = grey;
  a.blur_w = blur_w; a.pred = pred;
  Taps t;
  make_taps(t);
  return gb::launch<post_render_fwd_kernel>(dim3(gb::cdiv(W, kTile), gb::cdiv(H, kTile), B), kThreads, 0,
                                            (cudaStream_t)stream, a, t);
}

// g_pred [B,3,H,W] -> g_rgb [B,3,H,W] (overwritten); g_cal_w / g_cal_b / g_blur_w [B,3] accumulated (caller zero-fills;
// may be NULL).
GB_API int gb_post_render_bwd(int B, int H, int W, const float* rgb, const float* alpha, const float* bg, const float* cal_w,
                              const float* cal_b, const int32_t* grey, const float* blur_w, const float* g_pred, float* g_rgb,
                              float* g_cal_w, float* g_cal_b, float* g_blur_w, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  if (H <= kR7 || W <= kR7) return (int)cudaErrorInvalidValue;
  PostArgs a = {};
  a.B = B; a.H = H; a.W = W; a.rgb = rgb; a.alpha = alpha; a.bg = bg; a.cal_w = cal_w; a.cal_b = cal_b; a.grey = grey;
  a.blur_w = blur_w; a.g_pred = g_pred; a.g_rgb = g_rgb; a.g_cal_w = g_cal_w; a.g_cal_b = g_cal_b; a.g_blur_w = g_blur_w;
  Taps t;
  make_taps(t);
  return gb::launch<post_render_bwd_kernel>(dim3(gb::cdiv(W, kTile), gb::cdiv(H, kTile), B), kThreads, 0,
                                            (cudaStream_t)stream, a, t);
}

// Masked L1 and SSIM sums of pred vs target (ca_code/loss/__init__.py:391-410, 479-494): sums[0] = sum |(pred - target) * mask|,
// sums[1] = sum ssim_map * mask, sums[2] = sum of the mask expanded to 3 channels (fp64, zeroed by the caller);
// d_mu / d_pp / d_tp [B,3,H,W]: derivative maps kept for the backward.
GB_API int gb_ssim_l1_fwd(int B, int H, int W, const float* pred, const float* target, const float* mask, float* d_mu,
                          float* d_pp, float* d_tp, double* sums, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  LossArgs a = {};
  a.B = B; a.H = H; a.W = W; a.pred = pred; a.target = target; a.mask = mask; a.d_mu = d_mu; a.d_pp = d_pp; a.d_tp = d_tp;
  a.sums = sums;
  Taps t;
  make_taps(t);
  return gb::launch<ssim_l1_fwd_kernel>(dim3(gb::cdiv(W, kTile), gb::cdiv(H, kTile), 3 * B), kThreads, 0,
                                        (cudaStream_t)stream, a, t);
}

// Gradient of loss = l1_weight * l1 + ssim_weight * (1 - ssim) w.r.t. pred, times the upstream gradient *g_loss (device
// scalar, NULL = 1); `sums` are the forward's sums (read on the device: no host round trip).
GB_API int gb_ssim_l1_bwd(int B, int H, int W, const float* pred, const float* target, const float* mask, const float* d_mu,
                          const float* d_pp, const float* d_tp, const double* sums, const float* g_loss, float l1_weight,
                          float ssim_weight, float* g_pred, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  LossArgs a = {};
  a.B = B; a.H = H; a.W = W; a.pred = pred; a.target = target; a.mask = mask;
  a.d_mu = const_cast<float*>(d_mu); a.d_pp = const_cast<float*>(d_pp); a.d_tp = const_cast<float*>(d_tp);
  a.sums = const_cast<double*>(sums); a.g_loss = g_loss; a.l1_coef = l1_weight / ((float)B * 3.f * (float)H * (float)W);
  a.ssim_w = ssim_weight; a.g_pred = g_pred;
  Taps t;
  make_taps(t);
  return gb::launch<ssim_l1_bwd_kernel>(dim3(gb::cdiv(W, kTile), gb::cdiv(H, kTile), 3 * B), kThreads, 0,
                                        (cudaStream_t)stream, a, t);
}
