// goliath_b200/csrc/mesh_raster.cu — triangle rasterisation, UV texture sampling and their gradients (sm_90a).
//
// Replaces the drtk calls of the body avatar's RenderLayer (ca_code/utils/render_drtk.py:45-73): rasterize, render,
// interpolate, the grid_sample of the texture with the mask multiply, and edge_grad_estimator.  drtk is a third-party
// package outside the reference tree, so the conventions below are this project's (DESIGN.md R9'', PARITY UNPINNED):
//   * pixel (x, y) samples the screen point (x, y) + kPixelOffset;
//   * a face is drawn only if its three vertices have z > 0 (no near clipping, no backface culling) and its screen
//     area is non-zero;
//   * the inside test is inclusive (every screen-space barycentric lambda_k >= 0) for either winding;
//   * perspective-correct barycentrics b_k = (lambda_k / z_k) / sum_j lambda_j / z_j, depth = 1 / sum_j lambda_j / z_j;
//   * the visible face of a pixel is the smallest 64-bit key (float_bits(depth) << 32) | face_id, so ties go to the
//     smaller depth and then to the smaller face id, whatever the launch order.
// The file is compiled with -fmad=false (build.py): the index image is a bit-exact contract with the C oracle
// (oracle/mesh_oracle.c), which evaluates the same fp32 expressions in the same order.
//
// Rasteriser: one thread per (item, face) writes the keys of a face whose clipped pixel box holds at most
// kLargeFacePixels samples; bigger faces are appended to a list that a second kernel walks with one CTA per face.
//
// Backward (gradient from `render` only), with no float atomics, so two calls give bitwise-equal results:
//   * every covered pixel folds its interior gradient (sampled UV -> perspective-correct barycentrics -> the three
//     vertices' x, y, z) and the edge terms of the neighbour pairs it occludes into one 9-float record;
//   * the pixels are stably sorted by face and by the texel of their top-left bilinear tap (gb_sort_intersects);
//   * one warp per face sums its records in a fixed order; each vertex gathers its incident (face, corner) entries
//     from a CSR list the caller builds once per `vi`; one thread per texel gathers the four neighbouring pixel lists.
#include "common.cuh"
#include "../../include/goliath_b200.h"

namespace {

constexpr float kPixelOffset = 0.5f;   // PARITY UNPINNED: drtk's sample offset is not checked here
constexpr int kLargeFacePixels = 256;  // pixel-box size above which a face goes to the CTA-per-face kernel
constexpr int kBlock = 256;

struct Tri {
  float x[3], y[3], z[3];
};

__device__ __forceinline__ float edge_fn(float ax, float ay, float bx, float by, float px, float py) {
  return (bx - ax) * (py - ay) - (by - ay) * (px - ax);
}

__device__ __forceinline__ Tri load_tri(const float* __restrict__ vp, const int* __restrict__ vi, int f) {
  Tri t;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int v = vi[3 * f + k];
    t.x[k] = vp[3 * v];
    t.y[k] = vp[3 * v + 1];
    t.z[k] = vp[3 * v + 2];
  }
  return t;
}

// the cull rule: all z > 0, finite coordinates, non-zero (finite) screen area
__device__ __forceinline__ bool drawable(const Tri& t, float& area) {
#pragma unroll
  for (int k = 0; k < 3; ++k)
    if (!(t.z[k] > 0.f) || !isfinite(t.x[k]) || !isfinite(t.y[k]) || !isfinite(t.z[k])) return false;
  area = edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], t.x[2], t.y[2]);
  return area != 0.f && isfinite(area);
}

__device__ __forceinline__ void screen_bary(const Tri& t, float area, float px, float py, float l[3]) {
  l[0] = edge_fn(t.x[1], t.y[1], t.x[2], t.y[2], px, py) / area;
  l[1] = edge_fn(t.x[2], t.y[2], t.x[0], t.y[0], px, py) / area;
  l[2] = edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], px, py) / area;
}

__device__ __forceinline__ bool inside(const float l[3]) { return l[0] >= 0.f && l[1] >= 0.f && l[2] >= 0.f; }

// perspective-correct interpolation: q_k = lambda_k / z_k, returns sum_k q_k (1 / depth)
__device__ __forceinline__ float persp(const Tri& t, const float l[3], float q[3]) {
  q[0] = l[0] / t.z[0];
  q[1] = l[1] / t.z[1];
  q[2] = l[2] / t.z[2];
  return q[0] + q[1] + q[2];
}

struct Box {
  int x0, x1, y0, y1;
};

// the pixels whose sample point lies in the face's screen bounding box, clipped to the image
__device__ __forceinline__ bool face_box(const Tri& t, int H, int W, Box& b) {
  const float xmin = fminf(fminf(t.x[0], t.x[1]), t.x[2]), xmax = fmaxf(fmaxf(t.x[0], t.x[1]), t.x[2]);
  const float ymin = fminf(fminf(t.y[0], t.y[1]), t.y[2]), ymax = fmaxf(fmaxf(t.y[0], t.y[1]), t.y[2]);
  const float fx0 = fmaxf(ceilf(xmin - kPixelOffset), 0.f), fx1 = fminf(floorf(xmax - kPixelOffset), (float)(W - 1));
  const float fy0 = fmaxf(ceilf(ymin - kPixelOffset), 0.f), fy1 = fminf(floorf(ymax - kPixelOffset), (float)(H - 1));
  if (!(fx0 <= fx1) || !(fy0 <= fy1)) return false;
  b.x0 = (int)fx0;
  b.x1 = (int)fx1;
  b.y0 = (int)fy0;
  b.y1 = (int)fy1;
  return true;
}

__device__ __forceinline__ void raster_px(unsigned long long* __restrict__ zb, int W, const Tri& t, float area,
                                          int f, int x, int y) {
  float l[3], q[3];
  screen_bary(t, area, (float)x + kPixelOffset, (float)y + kPixelOffset, l);
  if (!inside(l)) return;
  const float depth = 1.f / persp(t, l, q);
  const unsigned long long key = ((unsigned long long)__float_as_uint(depth) << 32) | (unsigned)f;
  atomicMin(zb + (size_t)y * W + x, key);
}

__global__ void __launch_bounds__(kBlock) raster_init_kernel(long long n, unsigned long long* __restrict__ zb,
                                                             int* __restrict__ n_large) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i == 0) *n_large = 0;
  if (i < n) zb[i] = ~0ull;
}

__global__ void __launch_bounds__(kBlock) raster_small_kernel(int B, int V, int F, int H, int W,
                                                              const float* __restrict__ v_pix,
                                                              const int* __restrict__ vi,
                                                              unsigned long long* __restrict__ zb,
                                                              int* __restrict__ n_large, int* __restrict__ large) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= (long long)B * F) return;
  const int b = (int)(i / F), f = (int)(i % F);
  const Tri t = load_tri(v_pix + (size_t)b * V * 3, vi, f);
  float area;
  Box bx;
  if (!drawable(t, area) || !face_box(t, H, W, bx)) return;
  if ((long long)(bx.x1 - bx.x0 + 1) * (bx.y1 - bx.y0 + 1) > kLargeFacePixels) {
    large[atomicAdd(n_large, 1)] = (int)i;  // the list order does not matter: atomicMin is order-independent
    return;
  }
  unsigned long long* zbb = zb + (size_t)b * H * W;
  for (int y = bx.y0; y <= bx.y1; ++y)
    for (int x = bx.x0; x <= bx.x1; ++x) raster_px(zbb, W, t, area, f, x, y);
}

__global__ void __launch_bounds__(kBlock) raster_large_kernel(int V, int F, int H, int W,
                                                              const float* __restrict__ v_pix,
                                                              const int* __restrict__ vi,
                                                              unsigned long long* __restrict__ zb,
                                                              const int* __restrict__ n_large,
                                                              const int* __restrict__ large) {
  const int n = *n_large;
  for (int it = blockIdx.x; it < n; it += gridDim.x) {
    const int i = large[it], b = i / F, f = i % F;
    const Tri t = load_tri(v_pix + (size_t)b * V * 3, vi, f);
    float area;
    Box bx;
    if (!drawable(t, area) || !face_box(t, H, W, bx)) continue;
    const int bw = bx.x1 - bx.x0 + 1;
    const long long npx = (long long)bw * (bx.y1 - bx.y0 + 1);
    unsigned long long* zbb = zb + (size_t)b * H * W;
    for (long long p = threadIdx.x; p < npx; p += kBlock)
      raster_px(zbb, W, t, area, f, bx.x0 + (int)(p % bw), bx.y0 + (int)(p / bw));
  }
}

__global__ void __launch_bounds__(kBlock) raster_resolve_kernel(long long n, const unsigned long long* __restrict__ zb,
                                                                int* __restrict__ index_img) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = zb[i];
  index_img[i] = k == ~0ull ? -1 : (int)(unsigned)(k & 0xffffffffull);
}

// ------------------------------------------------------------------ texture sampling (grid_sample, align_corners=False)

struct Tap {
  float ix, iy;  // unnormalised sample position in texels
  int x0, y0;    // top-left tap
  bool any;      // at least one tap inside the texture
};

__device__ __forceinline__ Tap sample_pos(float u, float v, int Ht, int Wt) {
  Tap s;
  s.ix = ((u + 1.f) * (float)Wt - 1.f) / 2.f;
  s.iy = ((v + 1.f) * (float)Ht - 1.f) / 2.f;
  s.any = s.ix > -1.f && s.ix < (float)Wt && s.iy > -1.f && s.iy < (float)Ht;
  s.x0 = s.any ? (int)floorf(s.ix) : 0;
  s.y0 = s.any ? (int)floorf(s.iy) : 0;
  return s;
}

// the four taps (y0 + dy, x0 + dx) in the order (0,0), (0,1), (1,0), (1,1); taps outside read zero
__device__ __forceinline__ void taps(const float* __restrict__ tc, int Ht, int Wt, const Tap& s, float v[4]) {
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    const int x = s.x0 + (d & 1), y = s.y0 + (d >> 1);
    v[d] = (s.any && x >= 0 && x < Wt && y >= 0 && y < Ht) ? tc[(size_t)y * Wt + x] : 0.f;
  }
}

__device__ __forceinline__ void tap_weights(const Tap& s, float w[4]) {
  const float wx1 = s.ix - (float)s.x0, wx0 = (float)(s.x0 + 1) - s.ix;
  const float wy1 = s.iy - (float)s.y0, wy0 = (float)(s.y0 + 1) - s.iy;
  w[0] = wy0 * wx0;
  w[1] = wy0 * wx1;
  w[2] = wy1 * wx0;
  w[3] = wy1 * wx1;
}

__device__ __forceinline__ void face_uv(const int* __restrict__ vti, const float* __restrict__ vt, int f, float u[3],
                                        float v[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int j = vti[3 * f + k];
    u[k] = 2.f * vt[2 * j] - 1.f;
    v[k] = 2.f * vt[2 * j + 1] - 1.f;
  }
}

__global__ void __launch_bounds__(kBlock) render_fwd_kernel(
    int B, int V, int H, int W, int C, int Ht, int Wt, const float* __restrict__ v_pix, const int* __restrict__ vi,
    const int* __restrict__ vti, const float* __restrict__ vt, const float* __restrict__ tex,
    const int* __restrict__ index_img, float* __restrict__ depth_img, float* __restrict__ bary_img,
    float* __restrict__ vt_img, float* __restrict__ mask, float* __restrict__ render) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  const long long HW = (long long)H * W;
  if (i >= (long long)B * HW) return;
  const int b = (int)(i / HW);
  const long long p = i - b * HW;
  const int f = index_img[i];
  float* bary = bary_img + (size_t)b * 3 * HW + p;
  float* uvo = vt_img + (size_t)b * 2 * HW + p;
  float* out = render + (size_t)b * C * HW + p;
  if (f < 0) {
    depth_img[i] = 0.f;
    mask[i] = 0.f;
    bary[0] = bary[HW] = bary[2 * HW] = 0.f;
    uvo[0] = uvo[HW] = 0.f;
    for (int c = 0; c < C; ++c) out[(size_t)c * HW] = 0.f;
    return;
  }
  const int y = (int)(p / W), x = (int)(p % W);
  const Tri t = load_tri(v_pix + (size_t)b * V * 3, vi, f);
  float area, l[3], q[3];
  drawable(t, area);
  screen_bary(t, area, (float)x + kPixelOffset, (float)y + kPixelOffset, l);
  const float zi = persp(t, l, q);
  const float bk[3] = {q[0] / zi, q[1] / zi, q[2] / zi};
  float u[3], v[3];
  face_uv(vti, vt, f, u, v);
  const float U = bk[0] * u[0] + bk[1] * u[1] + bk[2] * u[2];
  const float Vv = bk[0] * v[0] + bk[1] * v[1] + bk[2] * v[2];
  depth_img[i] = 1.f / zi;
  mask[i] = 1.f;
  bary[0] = bk[0];
  bary[HW] = bk[1];
  bary[2 * HW] = bk[2];
  uvo[0] = U;
  uvo[HW] = Vv;
  const Tap s = sample_pos(U, Vv, Ht, Wt);
  float w[4];
  tap_weights(s, w);
  const size_t tHW = (size_t)Ht * Wt;
  for (int c = 0; c < C; ++c) {
    float tv[4];
    taps(tex + ((size_t)b * C + c) * tHW, Ht, Wt, s, tv);
    out[(size_t)c * HW] = w[0] * tv[0] + w[1] * tv[1] + w[2] * tv[2] + w[3] * tv[3];
  }
}

// ------------------------------------------------------------------ backward

// gradient of edge_fn(v_a, v_b, p) with respect to v_a and v_b (p fixed), scaled by g
__device__ __forceinline__ void edge_bwd(const Tri& t, int a, int b, float px, float py, float g, float gx[3],
                                         float gy[3]) {
  gx[a] += g * (t.y[b] - py);
  gy[a] += g * (px - t.x[b]);
  gx[b] += g * (py - t.y[a]);
  gy[b] -= g * (px - t.x[a]);
}

__device__ __forceinline__ bool share_edge(const int* __restrict__ vi, int f, int g) {
  int n = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) n += vi[3 * f + a] == vi[3 * g + b];
  return n >= 2;
}

// One record per covered pixel: the 9 v_pix gradients (corner-major x, y, z) of its face from this pixel's interior
// term and from the edge terms of the neighbour pairs it occludes; plus the two sort keys and the pixel's index.
__global__ void __launch_bounds__(kBlock) render_bwd_record_kernel(
    int B, int V, int F, int H, int W, int C, int Ht, int Wt, const float* __restrict__ v_pix,
    const int* __restrict__ vi, const int* __restrict__ vti, const float* __restrict__ vt,
    const float* __restrict__ tex, const int* __restrict__ index_img, const float* __restrict__ vt_img,
    const float* __restrict__ render, const float* __restrict__ g_render, int edge_grad, float* __restrict__ rec,
    long long* __restrict__ key_face, long long* __restrict__ key_tex, int* __restrict__ pix) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  const long long HW = (long long)H * W;
  if (i >= (long long)B * HW) return;
  pix[i] = (int)i;
  const int f = index_img[i];
  if (f < 0) {
    key_face[i] = (long long)B * F;
    key_tex[i] = (long long)B * (Ht + 1) * (Wt + 1);
    return;
  }
  const int b = (int)(i / HW);
  const long long p = i - b * HW;
  const int y = (int)(p / W), x = (int)(p % W);
  const float px = (float)x + kPixelOffset, py = (float)y + kPixelOffset;
  const float* vpb = v_pix + (size_t)b * V * 3;
  const Tri t = load_tri(vpb, vi, f);
  float area, l[3], q[3];
  drawable(t, area);
  screen_bary(t, area, px, py, l);
  const float zi = persp(t, l, q);
  const float bk[3] = {q[0] / zi, q[1] / zi, q[2] / zi};
  float u[3], v[3];
  face_uv(vti, vt, f, u, v);
  const float* gr = g_render + (size_t)b * C * HW + p;
  const float* img = render + (size_t)b * C * HW + p;

  // interior: render_c = sum_d w_d(ix, iy) tex_c[tap_d]; d/dix and d/diy of the bilinear weights
  const Tap s = sample_pos(vt_img[(size_t)b * 2 * HW + p], vt_img[(size_t)b * 2 * HW + HW + p], Ht, Wt);
  const float wx1 = s.ix - (float)s.x0, wx0 = (float)(s.x0 + 1) - s.ix;
  const float wy1 = s.iy - (float)s.y0, wy0 = (float)(s.y0 + 1) - s.iy;
  float gix = 0.f, giy = 0.f;
  const size_t tHW = (size_t)Ht * Wt;
  for (int c = 0; c < C; ++c) {
    float tv[4];
    taps(tex + ((size_t)b * C + c) * tHW, Ht, Wt, s, tv);
    const float g = gr[(size_t)c * HW];
    gix += g * (wy0 * (tv[1] - tv[0]) + wy1 * (tv[3] - tv[2]));
    giy += g * (wx0 * (tv[2] - tv[0]) + wx1 * (tv[3] - tv[1]));
  }
  const float gU = gix * (float)Wt / 2.f, gV = giy * (float)Ht / 2.f;
  float gb[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) gb[k] = gU * u[k] + gV * v[k];
  const float sb = gb[0] * bk[0] + gb[1] * bk[1] + gb[2] * bk[2];
  float gx[3] = {0.f, 0.f, 0.f}, gy[3] = {0.f, 0.f, 0.f}, gz[3];
  float gw[3], gA = 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float gq = (gb[k] - sb) / zi;
    const float gl = gq / t.z[k];
    gz[k] = -gq * q[k] / t.z[k];
    gw[k] = gl / area;
    gA -= gl * l[k];
  }
  gA /= area;
  edge_bwd(t, 1, 2, px, py, gw[0], gx, gy);
  edge_bwd(t, 2, 0, px, py, gw[1], gx, gy);
  edge_bwd(t, 0, 1, px, py, gw[2], gx, gy);
  edge_bwd(t, 0, 1, t.x[2], t.y[2], gA, gx, gy);  // area = edge_fn(v0, v1, v2): the third point is a vertex too
  gx[2] -= gA * (t.y[1] - t.y[0]);
  gy[2] += gA * (t.x[1] - t.x[0]);

  if (edge_grad) {
    const int* ib = index_img + (size_t)b * HW;
    const float depth_p = 1.f / zi;
#pragma unroll 1
    for (int nb = 0; nb < 4; ++nb) {  // right, below, left, above
      const int dx = nb == 0 ? 1 : (nb == 2 ? -1 : 0), dy = nb == 1 ? 1 : (nb == 3 ? -1 : 0);
      const int qx = x + dx, qy = y + dy;
      if (qx < 0 || qx >= W || qy < 0 || qy >= H) continue;
      const long long pq = (long long)qy * W + qx;
      const int fq = ib[pq];
      if (fq == f) continue;
      const float qpx = (float)qx + kPixelOffset, qpy = (float)qy + kPixelOffset;
      float lo[3];  // this face's barycentrics at the other pixel's sample point
      screen_bary(t, area, qpx, qpy, lo);
      if (fq >= 0) {
        if (share_edge(vi, f, fq)) continue;
        const Tri tq = load_tri(vpb, vi, fq);
        float aq, lq[3], qq[3];
        drawable(tq, aq);
        screen_bary(tq, aq, px, py, lq);
        const bool in_p = inside(lo), in_q = inside(lq);
        if (in_p && in_q) continue;  // interpenetration
        if (in_p) continue;          // the other face is the occluder
        if (!in_q) {                 // neither contains the other's point: the nearer one occludes
          screen_bary(tq, aq, qpx, qpy, lq);
          const float depth_q = 1.f / persp(tq, lq, qq);
          if (!(depth_p < depth_q || (depth_p == depth_q && f < fq))) continue;
        }
      }
      // this pixel's face T occludes: s = where T's edge crosses the segment toward the other pixel
      int ks = -1;
      float smin = 0.f;
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (lo[k] < 0.f) {
          const float sk = l[k] / (l[k] - lo[k]);
          if (ks < 0 || sk < smin) {
            ks = k;
            smin = sk;
          }
        }
      if (ks < 0) continue;
      float dLds = 0.f;
      for (int c = 0; c < C; ++c)
        dLds += (gr[(size_t)c * HW] + gr[(size_t)c * HW + pq - p]) * (img[(size_t)c * HW] - img[(size_t)c * HW + pq - p]);
      dLds *= 0.5f;
      const int a = ks == 0 ? 1 : (ks == 1 ? 2 : 0), e = ks == 0 ? 2 : (ks == 1 ? 0 : 1);
      const float ex = fabsf(t.x[e] - t.x[a]), ey = fabsf(t.y[e] - t.y[a]);
      const float wgt = (dx != 0 ? ey : ex) / (ex + ey);
      // s = w_o / (w_o - w_t), with w the unnormalised edge function of edge ks at own / other sample point
      const float wo = edge_fn(t.x[a], t.y[a], t.x[e], t.y[e], px, py);
      const float wt = edge_fn(t.x[a], t.y[a], t.x[e], t.y[e], qpx, qpy);
      const float den = wo - wt, gs = wgt * dLds / (den * den);
      edge_bwd(t, a, e, px, py, -gs * wt, gx, gy);
      edge_bwd(t, a, e, qpx, qpy, gs * wo, gx, gy);
    }
  }
  float* r = rec + (size_t)i * 9;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    r[3 * k] = gx[k];
    r[3 * k + 1] = gy[k];
    r[3 * k + 2] = gz[k];
  }
  key_face[i] = (long long)b * F + f;
  key_tex[i] = s.any ? ((long long)b * (Ht + 1) + (s.y0 + 1)) * (Wt + 1) + (s.x0 + 1) : (long long)B * (Ht + 1) * (Wt + 1);
}

// [start, end) of every key in a sorted key array (bins zeroed by the caller); the sentinel key is not binned
__global__ void __launch_bounds__(kBlock) bin_edges_kernel(long long n, const long long* __restrict__ keys,
                                                           long long sentinel, int2* __restrict__ bins) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const long long k = keys[i];
  if (k == sentinel) return;
  if (i == 0 || keys[i - 1] != k) bins[k].x = (int)i;
  if (i == n - 1 || keys[i + 1] != k) bins[k].y = (int)(i + 1);
}

// one warp per (item, face): lane-strided sums of its records in pixel order, then a butterfly
__global__ void __launch_bounds__(kBlock) face_reduce_kernel(long long nf, const int2* __restrict__ bins,
                                                             const int* __restrict__ sorted_pix,
                                                             const float* __restrict__ rec,
                                                             float* __restrict__ face_grad) {
  const long long e = ((long long)blockIdx.x * kBlock + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (e >= nf) return;
  const int2 r = bins[e];
  float a[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) a[j] = 0.f;
  for (int k = r.x + lane; k < r.y; k += 32) {
    const float* src = rec + (size_t)sorted_pix[k] * 9;
#pragma unroll
    for (int j = 0; j < 9; ++j) a[j] += src[j];
  }
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    const float v = gb::warp_sum(a[j]);
    if (lane == j) face_grad[(size_t)e * 9 + j] = v;
  }
}

// one thread per (item, vertex): its incident (face, corner) entries in list order
__global__ void __launch_bounds__(kBlock) vertex_gather_kernel(int B, int V, int F, const int* __restrict__ inc_ptr,
                                                               const int* __restrict__ inc,
                                                               const float* __restrict__ face_grad,
                                                               float* __restrict__ g_v_pix) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= (long long)B * V) return;
  const int b = (int)(i / V), v = (int)(i % V);
  float gx = 0.f, gy = 0.f, gz = 0.f;
  for (int k = inc_ptr[v]; k < inc_ptr[v + 1]; ++k) {
    const int fc = inc[k];
    const float* src = face_grad + ((size_t)b * F + fc / 3) * 9 + (fc % 3) * 3;
    gx += src[0];
    gy += src[1];
    gz += src[2];
  }
  g_v_pix[3 * i] = gx;
  g_v_pix[3 * i + 1] = gy;
  g_v_pix[3 * i + 2] = gz;
}

// one thread per (item, texel) and group of up to 4 channels: the pixels whose top-left tap is (ty - dy, tx - dx),
// for (dy, dx) = (0,0), (0,1), (1,0), (1,1), each list in pixel order
__global__ void __launch_bounds__(kBlock) texel_gather_kernel(int B, int H, int W, int C, int Ht, int Wt,
                                                              const int2* __restrict__ bins,
                                                              const int* __restrict__ sorted_pix,
                                                              const float* __restrict__ vt_img,
                                                              const float* __restrict__ g_render,
                                                              float* __restrict__ g_tex) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  const long long tHW = (long long)Ht * Wt, HW = (long long)H * W;
  if (i >= (long long)B * tHW) return;
  const int b = (int)(i / tHW);
  const long long tp = i - b * tHW;
  const int ty = (int)(tp / Wt), tx = (int)(tp % Wt);
  for (int c0 = 0; c0 < C; c0 += 4) {
    const int nc = C - c0 < 4 ? C - c0 : 4;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const int dy = d >> 1, dx = d & 1;
      const int2 r = bins[((long long)b * (Ht + 1) + (ty - dy + 1)) * (Wt + 1) + (tx - dx + 1)];
      for (int k = r.x; k < r.y; ++k) {
        const int pi = sorted_pix[k];
        const long long p = pi - (long long)b * HW;
        const Tap s = sample_pos(vt_img[(size_t)b * 2 * HW + p], vt_img[(size_t)b * 2 * HW + HW + p], Ht, Wt);
        float w[4];
        tap_weights(s, w);
        const float* gr = g_render + ((size_t)b * C + c0) * HW + p;
        for (int c = 0; c < nc; ++c) acc[c] += gr[(size_t)c * HW] * w[d];
      }
    }
    for (int c = 0; c < nc; ++c) g_tex[((size_t)b * C + c0 + c) * tHW + tp] = acc[c];
  }
}

inline unsigned grid1(long long n) { return (unsigned)gb::cdiv64(n, kBlock); }
inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
inline int bits_for(long long v) {  // bits needed to hold keys 0..v
  int n = 1;
  while ((1ll << n) <= v) ++n;
  return n;
}

struct BwdLayout {
  size_t rec, key_face, key_tex, pix, key_sorted, pix_face, pix_tex, bins_face, bins_tex, face_grad, sort_ws, total;
};

BwdLayout bwd_layout(int B, int F, int H, int W, int Ht, int Wt) {
  const size_t n = (size_t)B * H * W, nf = (size_t)B * F, nt = (size_t)B * (Ht + 1) * (Wt + 1);
  BwdLayout L;
  size_t o = 0;
  L.rec = o;        o += align256(n * 9 * 4);
  L.key_face = o;   o += align256(n * 8);
  L.key_tex = o;    o += align256(n * 8);
  L.pix = o;        o += align256(n * 4);
  L.key_sorted = o; o += align256(n * 8);
  L.pix_face = o;   o += align256(n * 4);
  L.pix_tex = o;    o += align256(n * 4);
  L.bins_face = o;  o += align256(nf * 8);
  L.bins_tex = o;   o += align256(nt * 8);
  L.face_grad = o;  o += align256(nf * 9 * 4);
  L.sort_ws = o;    o += align256(gb_sort_workspace_bytes((int64_t)n));
  L.total = o;
  return L;
}

bool sizes_ok(int B, int H, int W, int F) {
  return B > 0 && H > 0 && W > 0 && F >= 0 && (long long)B * H * W < (1ll << 31) && (long long)B * F < (1ll << 31);
}

}  // namespace

GB_API size_t gb_mesh_raster_workspace_bytes(int B, int F, int H, int W) {
  if (!sizes_ok(B, H, W, F)) return 0;
  return align256((size_t)B * H * W * 8) + 256 + (size_t)B * F * 4;
}

GB_API int gb_mesh_raster(int B, int V, int F, int H, int W, const float* v_pix, const int32_t* vi,
                          int32_t* index_img, void* workspace, void* stream) {
  if (!sizes_ok(B, H, W, F)) return B == 0 ? 0 : (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const long long n = (long long)B * H * W;
  char* ws = (char*)workspace;
  unsigned long long* zb = (unsigned long long*)ws;
  int* n_large = (int*)(ws + align256((size_t)n * 8));
  int* large = n_large + 64;
  GB_CUDA(gb::launch<raster_init_kernel>(grid1(n), kBlock, 0, s, n, zb, n_large));
  if (F > 0) {
    GB_CUDA(gb::launch<raster_small_kernel>(grid1((long long)B * F), kBlock, 0, s, B, V, F, H, W, v_pix, vi, zb,
                                            n_large, large));
    GB_CUDA(gb::launch<raster_large_kernel>(gb::kNumSMs * 8, kBlock, 0, s, V, F, H, W, v_pix, vi, zb, n_large, large));
  }
  return gb::launch<raster_resolve_kernel>(grid1(n), kBlock, 0, s, n, zb, index_img);
}

GB_API int gb_mesh_render_fwd(int B, int V, int F, int H, int W, int C, int Ht, int Wt, const float* v_pix,
                              const int32_t* vi, const int32_t* vti, const float* vt, const float* tex,
                              const int32_t* index_img, float* depth_img, float* bary_img, float* vt_img, float* mask,
                              float* render, void* stream) {
  if (!sizes_ok(B, H, W, F) || C < 0 || Ht <= 0 || Wt <= 0) return B == 0 ? 0 : (int)cudaErrorInvalidValue;
  const long long n = (long long)B * H * W;
  return gb::launch<render_fwd_kernel>(grid1(n), kBlock, 0, (cudaStream_t)stream, B, V, H, W, C, Ht, Wt, v_pix, vi, vti,
                                       vt, tex, index_img, depth_img, bary_img, vt_img, mask, render);
}

GB_API size_t gb_mesh_render_bwd_workspace_bytes(int B, int F, int H, int W, int Ht, int Wt) {
  if (!sizes_ok(B, H, W, F) || Ht <= 0 || Wt <= 0) return 0;
  return bwd_layout(B, F, H, W, Ht, Wt).total;
}

GB_API int gb_mesh_render_bwd(int B, int V, int F, int H, int W, int C, int Ht, int Wt, const float* v_pix,
                              const int32_t* vi, const int32_t* vti, const float* vt, const float* tex,
                              const int32_t* index_img, const float* vt_img, const float* render,
                              const float* g_render, int edge_grad, const int32_t* inc_ptr, const int32_t* inc,
                              float* g_v_pix, float* g_tex, void* workspace, void* stream) {
  if (!sizes_ok(B, H, W, F) || C < 0 || Ht <= 0 || Wt <= 0 || (long long)B * (Ht + 1) * (Wt + 1) >= (1ll << 40))
    return B == 0 ? 0 : (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const BwdLayout L = bwd_layout(B, F, H, W, Ht, Wt);
  char* ws = (char*)workspace;
  const long long n = (long long)B * H * W, nf = (long long)B * F, nt = (long long)B * (Ht + 1) * (Wt + 1);
  float* rec = (float*)(ws + L.rec);
  long long* key_face = (long long*)(ws + L.key_face);
  long long* key_tex = (long long*)(ws + L.key_tex);
  int* pix = (int*)(ws + L.pix);
  long long* key_sorted = (long long*)(ws + L.key_sorted);
  int* pix_face = (int*)(ws + L.pix_face);
  int* pix_tex = (int*)(ws + L.pix_tex);
  int2* bins_face = (int2*)(ws + L.bins_face);
  int2* bins_tex = (int2*)(ws + L.bins_tex);
  float* face_grad = (float*)(ws + L.face_grad);
  void* sort_ws = ws + L.sort_ws;

  GB_CUDA(gb::launch<render_bwd_record_kernel>(grid1(n), kBlock, 0, s, B, V, F, H, W, C, Ht, Wt, v_pix, vi, vti, vt,
                                               tex, index_img, vt_img, render, g_render, edge_grad, rec, key_face,
                                               key_tex, pix));
  // g_v_pix: pixels by face, one warp per face, then the vertex gather
  GB_CUDA(cudaMemsetAsync(bins_face, 0, (size_t)nf * 8, s));
  int err = gb_sort_intersects(n, (const int64_t*)key_face, pix, (int64_t*)key_sorted, pix_face, bits_for(nf), sort_ws, stream);
  if (err) return err;
  if (nf > 0) {
    GB_CUDA(gb::launch<bin_edges_kernel>(grid1(n), kBlock, 0, s, n, key_sorted, nf, bins_face));
    GB_CUDA(gb::launch<face_reduce_kernel>(grid1(nf * 32), kBlock, 0, s, nf, bins_face, pix_face, rec, face_grad));
  }
  if (V > 0) {
    GB_CUDA(gb::launch<vertex_gather_kernel>(grid1((long long)B * V), kBlock, 0, s, B, V, F, inc_ptr, inc, face_grad,
                                             g_v_pix));
  }
  // g_tex: pixels by the texel of their top-left tap, one thread per texel
  GB_CUDA(cudaMemsetAsync(bins_tex, 0, (size_t)nt * 8, s));
  err = gb_sort_intersects(n, (const int64_t*)key_tex, pix, (int64_t*)key_sorted, pix_tex, bits_for(nt), sort_ws, stream);
  if (err) return err;
  GB_CUDA(gb::launch<bin_edges_kernel>(grid1(n), kBlock, 0, s, n, key_sorted, nt, bins_tex));
  if (C > 0)
    GB_CUDA(gb::launch<texel_gather_kernel>(grid1((long long)B * Ht * Wt), kBlock, 0, s, B, H, W, C, Ht, Wt, bins_tex,
                                            pix_tex, vt_img, g_render, g_tex));
  return 0;
}
