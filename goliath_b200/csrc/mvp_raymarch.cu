// goliath_b200/csrc/mvp_raymarch.cu — Mixture-of-Volumetric-Primitives raymarcher, fwd + bwd, and the
// fixed-order BVH bounds (sm_90a).
//
// Replaces the reference extension extensions/mvpraymarch:
//   raymarch_subset_forward_kernel   mvpraymarch_subset_kernel.h:7-112
//   raymarch_subset_backward_kernel  mvpraymarch_subset_kernel.h:114-228
//   compute_aabb_kernel              bvh.cu:157-201
// with the policies the reference hard-wires (mvpraymarch_kernel.cu:39,113-115,201-203): fixed-order BVH subset
// per WARP (utils.h:949-1045), SRT primitive transform (primtransf.h:105-180), channels-last trilinear sampler
// with optional warp field (primsampler.h:36-92, utils.h:523-758), additive alpha accumulation with saturation
// (primaccum.h:63-98), optional shadow splat (primsplatter.h:29-36).  Compiled with -use_fast_math like the
// reference (extensions/mvpraymarch/setup.py:31) and written in its per-sample operation order, so rays agree with
// the reference kernels to the last bits; the launch geometry (block (bx,by), 32 consecutive linear thread ids
// per warp, edge threads clamped) is kept because hit lists are per-warp unions.
//
// What is different:
//  * every hit primitive carries the warp-level [t_in, t_out] of its box; while marching, a primitive is
//    touched only when the warp's current t-window overlaps that interval (warp-uniform test, no ballot), so
//    the per-step cost follows the primitives actually overlapping the sample, not the whole hit list;
//  * backward: template / warp gradients use one 16-byte vector RED per trilinear corner
//    (red.global.add.v4.f32) instead of 4 scalar atomics; the 15 transform gradients are reduced across the warp
//    with a recursive-halving exchange (16 shuffles instead of 75) and issued as one RED per value by 15 lanes;
//  * current stream / current device everywhere; bounds scratch comes from the caller (no cudaMalloc per call,
//    bvh.cu:261-293).
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace {

constexpr int kMaxHit = 512;

struct RMArgs {
  int N, H, W, K;
  const float* raypos; const float* raydir; float stepsize; const float2* tminmax;
  const float* nodeaabb;                       // [N, 2K-1, 2, 3]
  const float* primpos; const float* primrot; const float* primscale;
  int TD, TH, TW; const float4* tplate;        // [N,K,TD,TH,TW,4]
  int WD, WH, WW; const float* warp;           // [N,K,WD,WH,WW,3] or null
  float fadescale, fadeexp;
  float4* rayrgba; float* raysat; float* shadow;                 // forward outputs (raysat/shadow nullable)
  const float4* grad_rayrgba;                                     // backward
  float* grad_primpos; float* grad_primrot; float* grad_primscale; float* grad_tplate; float* grad_warp;
  int L;                                       // views per item (shadow march): transforms / bounds at n / L; 0 = 1
  int U; const float* slab; const float* valid;  // shadow march: alpha slab [N/L,TD,U,U], valid mask [K] or null
};

__device__ __forceinline__ float3 ld3(const float* p) { return make_float3(p[0], p[1], p[2]); }
__device__ __forceinline__ float3 operator+(float3 a, float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 operator-(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 operator*(float3 a, float3 b) { return make_float3(a.x * b.x, a.y * b.y, a.z * b.z); }
__device__ __forceinline__ float3 operator*(float3 a, float s) { return make_float3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float3 min3(float3 a, float3 b) { return make_float3(fminf(a.x, b.x), fminf(a.y, b.y), fminf(a.z, b.z)); }
__device__ __forceinline__ float3 max3(float3 a, float3 b) { return make_float3(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z)); }
__device__ __forceinline__ float maxc(float3 a) { return fmaxf(fmaxf(a.x, a.y), a.z); }
__device__ __forceinline__ float minc(float3 a) { return fminf(fminf(a.x, a.y), a.z); }

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ bool aabb_hit(const float* a, float3 rp, float3 ird) {  // utils.h:912-919
  const float3 t0 = (ld3(a) - rp) * ird, t1 = (ld3(a + 3) - rp) * ird;
  return maxc(min3(t0, t1)) <= minc(max3(t0, t1));
}

// DFS over the implicit heap, warp-any semantics (utils.h:949-1045).  hit[] / ivl[] are this warp's shared arrays.
__device__ int build_hitlist(int K, float3 raypos, float3 raydir, const float* nodeaabb, const float* pp,
                             const float* pr, const float* ps, int* hit, float2* ivl, float& rtmin, float& rtmax) {
  const unsigned full = 0xffffffffu;
  const int lane = (int)((threadIdx.y * blockDim.x + threadIdx.x) & 31);
  const float3 ird = make_float3(1.0f / raydir.x, 1.0f / raydir.y, 1.0f / raydir.z);
  int stack[64];
  int sp = 0;
  stack[sp++] = -1;
  int node = 0, num = 0;
  do {
    if (node >= K - 1) {
      const int k = node - (K - 1);
      // forward2 (primtransf.h:134-153)
      const float3 pt = ld3(pp + 3 * (size_t)k);
      const float3 r0v = ld3(pr + 9 * (size_t)k), r1v = ld3(pr + 9 * (size_t)k + 3), r2v = ld3(pr + 9 * (size_t)k + 6);
      const float3 sc = ld3(ps + 3 * (size_t)k);
      const float3 xmt = raypos - pt, dmt = raydir;
      float3 rx = r0v * xmt.x, rd = r0v * dmt.x;
      rx = rx + r1v * xmt.y; rd = rd + r1v * dmt.y;
      rx = rx + r2v * xmt.z; rd = rd + r2v * dmt.z;
      const float3 r0 = rx * sc, d0 = rd * sc;
      const float3 id = make_float3(1.0f / d0.x, 1.0f / d0.y, 1.0f / d0.z);
      const float3 t0 = (make_float3(-1.f, -1.f, -1.f) - r0) * id, t1 = (make_float3(1.f, 1.f, 1.f) - r0) * id;
      const float trmin = maxc(min3(t0, t1)), trmax = minc(max3(t0, t1));
      const bool inter = trmin <= trmax;
      if (inter) { rtmin = fminf(rtmin, trmin); rtmax = fmaxf(rtmax, trmax); }
      if (__any_sync(full, inter)) {
        const float wmin = warp_min(inter ? trmin : INFINITY), wmax = warp_max(inter ? trmax : -INFINITY);
        if (num < kMaxHit) {
          if (lane == 0) { hit[num] = k; ivl[num] = make_float2(wmin, wmax); }
          ++num;
        }
      }
      node = stack[--sp];
    } else {
      const int cl = 2 * node + 1, cr = 2 * node + 2;
      const bool tl = __any_sync(full, aabb_hit(nodeaabb + (size_t)cl * 6, raypos, ird));
      const bool tr = __any_sync(full, aabb_hit(nodeaabb + (size_t)cr * 6, raypos, ird));
      if (!tl && !tr) node = stack[--sp];
      else {
        node = tl ? cl : cr;
        if (tl && tr) stack[sp++] = cr;
      }
    }
  } while (node != -1);
  __syncwarp();
  return num;
}

// trilinear setup shared by sampler / splatter (utils.h:523-560)
struct Tri {
  int ix, iy, iz;
  float fx, fy, fz;
};
template <bool CLAMP>
__device__ __forceinline__ Tri tri_setup(int D, int H, int W, float3 pos) {
  Tri t;
  if (CLAMP) {
    t.fx = fmaxf(-100.f, fminf(100.f, ((pos.x + 1.f) / 2))) * (W - 1);
    t.fy = fmaxf(-100.f, fminf(100.f, ((pos.y + 1.f) / 2))) * (H - 1);
    t.fz = fmaxf(-100.f, fminf(100.f, ((pos.z + 1.f) / 2))) * (D - 1);
  } else {
    t.fx = ((pos.x + 1.f) / 2) * (W - 1);
    t.fy = ((pos.y + 1.f) / 2) * (H - 1);
    t.fz = ((pos.z + 1.f) / 2) * (D - 1);
  }
  t.ix = (int)floorf(t.fx); t.iy = (int)floorf(t.fy); t.iz = (int)floorf(t.fz);
  return t;
}
// weights in the reference's corner order: tnw tne tsw tse bnw bne bsw bse
__device__ __forceinline__ void tri_weights(const Tri& t, float (&w)[8]) {
  const float x1 = (t.ix + 1) - t.fx, x0 = t.fx - t.ix, y1 = (t.iy + 1) - t.fy, y0 = t.fy - t.iy;
  const float z1 = (t.iz + 1) - t.fz, z0 = t.fz - t.iz;
  w[0] = x1 * y1 * z1; w[1] = x0 * y1 * z1; w[2] = x1 * y0 * z1; w[3] = x0 * y0 * z1;
  w[4] = x1 * y1 * z0; w[5] = x0 * y1 * z0; w[6] = x1 * y0 * z0; w[7] = x0 * y0 * z0;
}
__device__ __forceinline__ bool corner(const Tri& t, int c, int D, int H, int W, int& off) {
  const int w = t.ix + (c & 1), h = t.iy + ((c >> 1) & 1), d = t.iz + ((c >> 2) & 1);
  off = (d * H + h) * W + w;
  return d >= 0 && d < D && h >= 0 && h < H && w >= 0 && w < W;
}

__device__ __forceinline__ float4 sample4(int D, int H, int W, const float4* vals, float3 pos) {
  const Tri t = tri_setup<true>(D, H, W, pos);
  float w[8];
  tri_weights(t, w);
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    int off;
    if (corner(t, c, D, H, W, off)) {
      const float4 v = vals[off];
      r.x += v.x * w[c]; r.y += v.y * w[c]; r.z += v.z * w[c]; r.w += v.w * w[c];
    }
  }
  return r;
}
__device__ __forceinline__ float3 sample3(int D, int H, int W, const float* vals, float3 pos) {
  const Tri t = tri_setup<true>(D, H, W, pos);
  float w[8];
  tri_weights(t, w);
  float3 r = make_float3(0.f, 0.f, 0.f);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    int off;
    if (corner(t, c, D, H, W, off)) {
      r.x += vals[3 * off] * w[c]; r.y += vals[3 * off + 1] * w[c]; r.z += vals[3 * off + 2] * w[c];
    }
  }
  return r;
}

// d weight / d (x, y, z) for the 8 corners, reference sign conventions (utils.h:700-756)
__device__ __forceinline__ void tri_dweights(const Tri& t, float (&dx)[8], float (&dy)[8], float (&dz)[8]) {
  const float x1 = (t.ix + 1) - t.fx, x0 = t.fx - t.ix, y1 = (t.iy + 1) - t.fy, y0 = t.fy - t.iy;
  const float z1 = (t.iz + 1) - t.fz, z0 = t.fz - t.iz;
  dx[0] = -(y1 * z1); dx[1] = y1 * z1; dx[2] = -(y0 * z1); dx[3] = y0 * z1;
  dx[4] = -(y1 * z0); dx[5] = y1 * z0; dx[6] = -(y0 * z0); dx[7] = y0 * z0;
  dy[0] = -(x1 * z1); dy[1] = -(x0 * z1); dy[2] = x1 * z1; dy[3] = x0 * z1;
  dy[4] = -(x1 * z0); dy[5] = -(x0 * z0); dy[6] = x1 * z0; dy[7] = x0 * z0;
  dz[0] = -(x1 * y1); dz[1] = -(x0 * y1); dz[2] = -(x1 * y0); dz[3] = -(x0 * y0);
  dz[4] = x1 * y1; dz[5] = x0 * y1; dz[6] = x1 * y0; dz[7] = x0 * y0;
}

__device__ __forceinline__ float3 sample4_bwd(int D, int H, int W, const float4* vals, float* grad_vals, float3 pos,
                                              float4 g, bool scatter) {
  const Tri t = tri_setup<true>(D, H, W, pos);
  float w[8], dx[8], dy[8], dz[8];
  tri_weights(t, w);
  tri_dweights(t, dx, dy, dz);
  float gix = 0.f, giy = 0.f, giz = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    int off;
    if (corner(t, c, D, H, W, off)) {
      if (scatter) gb::red_add_v4(grad_vals + 4 * (size_t)off, w[c] * g.x, w[c] * g.y, w[c] * g.z, w[c] * g.w);
      const float4 v = vals[off];
      const float dt = v.x * g.x + v.y * g.y + v.z * g.z + v.w * g.w;
      gix += dx[c] * dt; giy += dy[c] * dt; giz += dz[c] * dt;
    }
  }
  return make_float3((W - 1.f) / 2 * gix, (H - 1.f) / 2 * giy, (D - 1.f) / 2 * giz);
}
__device__ __forceinline__ float3 sample3_bwd(int D, int H, int W, const float* vals, float* grad_vals, float3 pos,
                                              float3 g, bool scatter) {
  const Tri t = tri_setup<true>(D, H, W, pos);
  float w[8], dx[8], dy[8], dz[8];
  tri_weights(t, w);
  tri_dweights(t, dx, dy, dz);
  float gix = 0.f, giy = 0.f, giz = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    int off;
    if (corner(t, c, D, H, W, off)) {
      if (scatter) {
        gb::red_add(grad_vals + 3 * (size_t)off, w[c] * g.x);
        gb::red_add(grad_vals + 3 * (size_t)off + 1, w[c] * g.y);
        gb::red_add(grad_vals + 3 * (size_t)off + 2, w[c] * g.z);
      }
      const float dt = vals[3 * off] * g.x + vals[3 * off + 1] * g.y + vals[3 * off + 2] * g.z;
      gix += dx[c] * dt; giy += dy[c] * dt; giz += dz[c] * dt;
    }
  }
  return make_float3((W - 1.f) / 2 * gix, (H - 1.f) / 2 * giy, (D - 1.f) / 2 * giz);
}

__device__ __forceinline__ void splat_shadow(int D, int H, int W, float vis, float* vals, float3 pos) {  // utils.h:773-876
  const Tri t = tri_setup<false>(D, H, W, pos);
  float w[8];
  tri_weights(t, w);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    int off;
    if (corner(t, c, D, H, W, off)) gb::red_add_v2(vals + 2 * (size_t)off, w[c] * vis, w[c]);
  }
}

// ------------------------------------------------------------------ common ray / warp setup
struct RaySetup {
  int n, h, w;
  bool validthread;
  float3 raypos, raydir, pos;
  float t, rtmin, rtmax;
  int nhit, item;
  int* hit;
  float2* ivl;
  const float *pp, *pr, *ps;
};

__device__ __forceinline__ RaySetup setup_ray(const RMArgs& a, int* s_hit, float2* s_ivl) {
  RaySetup r;
  int w = blockIdx.x * blockDim.x + threadIdx.x;
  int h = blockIdx.y * blockDim.y + threadIdx.y;
  r.n = min(a.N - 1, (int)blockIdx.z);
  r.validthread = (w < a.W) && (h < a.H);
  r.h = h = min(a.H - 1, h);
  r.w = w = min(a.W - 1, w);
  const int warpid = (threadIdx.y * blockDim.x + threadIdx.x) >> 5;
  r.hit = s_hit + warpid * kMaxHit;
  r.ivl = s_ivl + warpid * kMaxHit;
  const size_t o = ((size_t)r.n * a.H + h) * a.W + w;
  r.raypos = ld3(a.raypos + 3 * o);
  r.raydir = ld3(a.raydir + 3 * o);
  const float2 tmm = a.tminmax[o];
  r.item = a.L > 1 ? r.n / a.L : r.n;
  r.pp = a.primpos + (size_t)r.item * a.K * 3;
  r.pr = a.primrot + (size_t)r.item * a.K * 9;
  r.ps = a.primscale + (size_t)r.item * a.K * 3;
  float rtmin = INFINITY, rtmax = -INFINITY;
  r.nhit = build_hitlist(a.K, r.raypos, r.raydir, a.nodeaabb + (size_t)r.item * (2 * a.K - 1) * 6, r.pp, r.pr, r.ps, r.hit,
                         r.ivl, rtmin, rtmax);
  r.rtmin = fmaxf(rtmin, tmm.x);
  r.rtmax = fminf(rtmax, tmm.y);
  r.t = tmm.x;
  r.pos = r.raypos + r.raydir * tmm.x;
  const int incs = (int)floorf((r.rtmin - r.t) / a.stepsize);  // saturating cvt, like the reference's int = floor()
  r.t += incs * a.stepsize;
  r.pos = r.pos + r.raydir * (float)incs * a.stepsize;
  return r;
}

// per-(ray, primitive) local frame (primtransf.h:119-132)
struct Local {
  float3 xmt, rxmt, y0, pr0, pr1, pr2, ps;
};
__device__ __forceinline__ Local prim_local(const RaySetup& r, int k, float3 x) {
  Local L;
  const float3 pt = ld3(r.pp + 3 * (size_t)k);
  L.pr0 = ld3(r.pr + 9 * (size_t)k); L.pr1 = ld3(r.pr + 9 * (size_t)k + 3); L.pr2 = ld3(r.pr + 9 * (size_t)k + 6);
  L.ps = ld3(r.ps + 3 * (size_t)k);
  L.xmt = x - pt;
  L.rxmt = L.pr0 * L.xmt.x + L.pr1 * L.xmt.y + L.pr2 * L.xmt.z;
  L.y0 = L.rxmt * L.ps;
  return L;
}
__device__ __forceinline__ bool inside_unit(float3 p) {
  return p.x > -1.f && p.x < 1.f && p.y > -1.f && p.y < 1.f && p.z > -1.f && p.z < 1.f;
}

// ------------------------------------------------------------------ forward
template <bool WARP, bool SHADOW>
__global__ void raymarch_fwd_kernel(RMArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int nwarps = (blockDim.x * blockDim.y + 31) >> 5;
  int* s_hit = reinterpret_cast<int*>(smem);
  float2* s_ivl = reinterpret_cast<float2*>(smem + (size_t)nwarps * kMaxHit * sizeof(int));
  RaySetup r = setup_ray(a, s_hit, s_ivl);
  const unsigned full = 0xffffffffu;
  const size_t tsz = (size_t)a.TD * a.TH * a.TW, wsz = (size_t)a.WD * a.WH * a.WW;
  const float stepsize = a.stepsize;

  float4 rgba = make_float4(0.f, 0.f, 0.f, 0.f);
  float3 raysat = make_float3(-1.f, -1.f, -1.f);
  bool sat = false;
  float t = r.t;
  float3 pos = r.pos;
  // warp-uniform window of the t values still marching
  const bool live0 = !(t > r.rtmax + 1e-5f);
  float tlo = warp_min(live0 ? t : INFINITY), thi = warp_max(live0 ? t : -INFINITY);
  const float margin = 2.f * stepsize + 1e-3f;

  while (!__all_sync(full, t > r.rtmax + 1e-5f || sat)) {
    for (int ks = 0; ks < r.nhit; ++ks) {
      const float2 iv = r.ivl[ks];
      if (thi + margin < iv.x || tlo - margin > iv.y) continue;  // warp-uniform: nobody is inside this box now
      const int k = r.hit[ks];
      Local L = prim_local(r, k, pos);
      if (inside_unit(L.y0) && !sat && t < r.rtmax + 1e-5f) {
        const float3 y0 = L.y0;
        const float fade = __expf(-a.fadescale * (__powf(fabsf(y0.x), a.fadeexp) + __powf(fabsf(y0.y), a.fadeexp) +
                                                  __powf(fabsf(y0.z), a.fadeexp)));
        float3 y1 = y0;
        if (WARP) y1 = sample3(a.WD, a.WH, a.WW, a.warp + ((size_t)r.n * a.K + k) * 3 * wsz, y0);
        float4 s = sample4(a.TD, a.TH, a.TW, a.tplate + ((size_t)r.n * a.K + k) * tsz, y1);
        s.w *= fade;
        if (SHADOW) splat_shadow(a.TD, a.TH, a.TW, 1.f - rgba.w, a.shadow + ((size_t)r.n * a.K + k) * 2 * tsz, y1);
        // PrimAccumAdditive::forward_prim (primaccum.h:63-79)
        const float newalpha = rgba.w + s.w * stepsize;
        const float contrib = fminf(newalpha, 1.f) - rgba.w;
        rgba.x += s.x * contrib; rgba.y += s.y * contrib; rgba.z += s.z * contrib; rgba.w += 1.f * contrib;
        if (newalpha >= 1.f) {
          if (!sat) raysat = make_float3(s.x, s.y, s.z);
          sat = true;
        }
      }
    }
    t += stepsize;
    pos = pos + r.raydir * stepsize;
    tlo += stepsize;
    thi += stepsize;
  }
  // every thread writes (edge duplicates write the same value, as in the reference)
  const size_t o = ((size_t)r.n * a.H + r.h) * a.W + r.w;
  a.rayrgba[o] = rgba;
  if (a.raysat) { a.raysat[3 * o] = raysat.x; a.raysat[3 * o + 1] = raysat.y; a.raysat[3 * o + 2] = raysat.z; }
}

// ------------------------------------------------------------------ deep shadow march over a shared alpha template
// The relightable hand teacher (hand_teacher_mvp.py:274-358) marches, from each of L lights, a template whose rgb is the
// constant 255 and whose alpha is the geometry decoder's slab, copied once per light, and keeps only the splat volume.
// This kernel is raymarch_fwd_kernel<false, true> with the rgb and raysat work removed: the alpha accumulation,
// saturation stop, fade and splat_shadow are the same expressions in the same order, so the splat volume depends on
// the alpha channel alone, exactly as there.  View n reads the transforms and bounds of item n / L, and samples the
// alpha slab [TD, U, U] of that item in place: primitive k = hy * (U / TW) + wx covers rows hy*TH.., columns wx*TW..
// of the slab, so template voxel (z, y, x) of k is slab texel (z, hy*TH + y, wx*TW + x) (hand_teacher_mvp.py:289-311),
// times valid[k].  Reading in place needs no per-item re-layout pass and no [B, K, TD, TH, TW] copy; the corners of a
// trilinear lookup are U floats apart in y instead of TW, which costs cache lines, not extra passes.
__device__ __forceinline__ float sample_alpha_slab(int D, int H, int W, int U, const float* base, float valid, float3 pos) {
  const Tri t = tri_setup<true>(D, H, W, pos);
  float w[8];
  tri_weights(t, w);
  float r = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int x = t.ix + (c & 1), y = t.iy + ((c >> 1) & 1), z = t.iz + ((c >> 2) & 1);
    if (z >= 0 && z < D && y >= 0 && y < H && x >= 0 && x < W) r += (valid * base[((size_t)z * U + y) * U + x]) * w[c];
  }
  return r;
}

__global__ void shadow_march_kernel(RMArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int nwarps = (blockDim.x * blockDim.y + 31) >> 5;
  int* s_hit = reinterpret_cast<int*>(smem);
  float2* s_ivl = reinterpret_cast<float2*>(smem + (size_t)nwarps * kMaxHit * sizeof(int));
  RaySetup r = setup_ray(a, s_hit, s_ivl);
  const unsigned full = 0xffffffffu;
  const size_t tsz = (size_t)a.TD * a.TH * a.TW;
  const int nx = a.U / a.TW;
  const float* slab = a.slab + (size_t)r.item * a.TD * a.U * a.U;
  const float stepsize = a.stepsize;

  float alpha = 0.f;
  bool sat = false;
  float t = r.t;
  float3 pos = r.pos;
  const bool live0 = !(t > r.rtmax + 1e-5f);
  float tlo = warp_min(live0 ? t : INFINITY), thi = warp_max(live0 ? t : -INFINITY);
  const float margin = 2.f * stepsize + 1e-3f;

  while (!__all_sync(full, t > r.rtmax + 1e-5f || sat)) {
    for (int ks = 0; ks < r.nhit; ++ks) {
      const float2 iv = r.ivl[ks];
      if (thi + margin < iv.x || tlo - margin > iv.y) continue;
      const int k = r.hit[ks];
      Local L = prim_local(r, k, pos);
      if (inside_unit(L.y0) && !sat && t < r.rtmax + 1e-5f) {
        const float3 y0 = L.y0;
        const float fade = __expf(-a.fadescale * (__powf(fabsf(y0.x), a.fadeexp) + __powf(fabsf(y0.y), a.fadeexp) +
                                                  __powf(fabsf(y0.z), a.fadeexp)));
        const int hy = k / nx, wx = k - hy * nx;
        float sw = sample_alpha_slab(a.TD, a.TH, a.TW, a.U, slab + (size_t)hy * a.TH * a.U + (size_t)wx * a.TW,
                                     a.valid ? a.valid[k] : 1.f, y0);
        sw *= fade;
        splat_shadow(a.TD, a.TH, a.TW, 1.f - alpha, a.shadow + ((size_t)r.n * a.K + k) * 2 * tsz, y0);
        const float newalpha = alpha + sw * stepsize;
        const float contrib = fminf(newalpha, 1.f) - alpha;
        alpha += 1.f * contrib;
        if (newalpha >= 1.f) sat = true;
      }
    }
    t += stepsize;
    pos = pos + r.raydir * stepsize;
    tlo += stepsize;
    thi += stepsize;
  }
}

// ------------------------------------------------------------------ forward, lane-compacted sampling (algo 0, no shadow)
// In the kernel above the sampling block — fade (3 pow + exp), trilinear setup, 8 corner loads — runs with few of the
// 32 lanes active, because a primitive overlaps only a few rays of the warp's 8x4
// footprint at a given step.  Here the warp ENQUEUES the (ray, primitive) pairs that are inside a primitive (local
// coordinate + primitive id, compacted with a ballot) and SAMPLES them 32 at a time with every lane busy, whichever
// ray or primitive an item belongs to; the results are then APPLIED in the original order — group by group (one group =
// one (step, primitive), at most one item per ray), each ray picking its own result — so the additive accumulation
// with saturation sees exactly the sequence of the kernel above: rays stay bit-identical (same expressions on the same
// values, executed by another lane).  `sat` is only known at apply time: enqueueing uses the value of the last flush
// (a superset; the apply step ignores items of saturated rays).
constexpr int kQueue = 64;  // items per warp: < 32 pending + one group of up to 32
struct RMQueue {
  float4 q[kQueue];        // y0.xyz, primitive id (int bits)
  float4 s[kQueue];        // sampled rgba (alpha already faded)
  unsigned g[kQueue];      // ballot of each pending group
};

__global__ void raymarch_fwd_queue_kernel(RMArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int nwarps = (blockDim.x * blockDim.y + 31) >> 5;
  int* s_hit = reinterpret_cast<int*>(smem);
  float2* s_ivl = reinterpret_cast<float2*>(smem + (size_t)nwarps * kMaxHit * sizeof(int));
  RMQueue* s_q = reinterpret_cast<RMQueue*>(smem + (size_t)nwarps * kMaxHit * (sizeof(int) + sizeof(float2)));
  RaySetup r = setup_ray(a, s_hit, s_ivl);
  const unsigned full = 0xffffffffu;
  const int lane = (threadIdx.y * blockDim.x + threadIdx.x) & 31;
  RMQueue& Q = s_q[(threadIdx.y * blockDim.x + threadIdx.x) >> 5];
  const unsigned lt = (1u << lane) - 1u;
  const size_t tsz = (size_t)a.TD * a.TH * a.TW;
  const float stepsize = a.stepsize;
  const float4* tbase = a.tplate + (size_t)r.n * a.K * tsz;

  float4 rgba = make_float4(0.f, 0.f, 0.f, 0.f);
  float3 raysat = make_float3(-1.f, -1.f, -1.f);
  bool sat = false;
  float t = r.t;
  float3 pos = r.pos;
  const bool live0 = !(t > r.rtmax + 1e-5f);
  float tlo = warp_min(live0 ? t : INFINITY), thi = warp_max(live0 ? t : -INFINITY);
  const float margin = 2.f * stepsize + 1e-3f;
  int qn = 0, ng = 0;  // pending items / groups (warp-uniform)

  auto flush = [&]() {
    __syncwarp();
    for (int base = 0; base < qn; base += 32) {  // sample: every lane takes one item
      const int i = base + lane;
      if (i < qn) {
        const float4 it = Q.q[i];
        const float3 y0 = make_float3(it.x, it.y, it.z);
        const int k = __float_as_int(it.w);
        const float fade = __expf(-a.fadescale * (__powf(fabsf(y0.x), a.fadeexp) + __powf(fabsf(y0.y), a.fadeexp) +
                                                  __powf(fabsf(y0.z), a.fadeexp)));
        float4 sv = sample4(a.TD, a.TH, a.TW, tbase + (size_t)k * tsz, y0);
        sv.w *= fade;
        Q.s[i] = sv;
      }
    }
    __syncwarp();
    int off = 0;
    for (int g = 0; g < ng; ++g) {  // apply: original order, each ray picks its own result
      const unsigned m = Q.g[g];
      if (((m >> lane) & 1u) && !sat) {
        const float4 sv = Q.s[off + __popc(m & lt)];
        // PrimAccumAdditive::forward_prim (primaccum.h:63-79)
        const float newalpha = rgba.w + sv.w * stepsize;
        const float contrib = fminf(newalpha, 1.f) - rgba.w;
        rgba.x += sv.x * contrib; rgba.y += sv.y * contrib; rgba.z += sv.z * contrib; rgba.w += 1.f * contrib;
        if (newalpha >= 1.f) {
          raysat = make_float3(sv.x, sv.y, sv.z);
          sat = true;
        }
      }
      off += __popc(m);
    }
    qn = 0;
    ng = 0;
    __syncwarp();
  };

  while (!__all_sync(full, t > r.rtmax + 1e-5f || sat)) {
    for (int ks = 0; ks < r.nhit; ++ks) {
      const float2 iv = r.ivl[ks];
      if (thi + margin < iv.x || tlo - margin > iv.y) continue;  // warp-uniform: nobody is inside this box now
      const int k = r.hit[ks];
      const Local L = prim_local(r, k, pos);
      const bool in = inside_unit(L.y0) && !sat && t < r.rtmax + 1e-5f;
      const unsigned m = __ballot_sync(full, in);
      if (m == 0u) continue;
      if (in) Q.q[qn + __popc(m & lt)] = make_float4(L.y0.x, L.y0.y, L.y0.z, __int_as_float(k));
      if (lane == 0) Q.g[ng] = m;
      qn += __popc(m);
      ++ng;
      if (qn >= 32) flush();
    }
    t += stepsize;
    pos = pos + r.raydir * stepsize;
    tlo += stepsize;
    thi += stepsize;
    if (qn >= 16) flush();  // keeps `sat` fresh: a saturated ray stops enqueueing (and the loop may end) a step later at most
  }
  flush();
  const size_t o = ((size_t)r.n * a.H + r.h) * a.W + r.w;
  a.rayrgba[o] = rgba;
  if (a.raysat) { a.raysat[3 * o] = raysat.x; a.raysat[3 * o + 1] = raysat.y; a.raysat[3 * o + 2] = raysat.z; }
}

// ------------------------------------------------------------------ backward
// recursive-halving reduction of 16 per-lane values: 8+4+2+1+1 = 16 shuffles; afterwards the lane with index L
// (even) holds the warp total of slot (L >> 1)
__device__ __forceinline__ float reduce16(float (&v)[16], int lane) {
  const bool h4 = lane & 16, h3 = lane & 8, h2 = lane & 4, h1 = lane & 2;
  float a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float send = h4 ? v[i] : v[8 + i], keep = h4 ? v[8 + i] : v[i];
    a[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
  float b[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float send = h3 ? a[i] : a[4 + i], keep = h3 ? a[4 + i] : a[i];
    b[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
  float c[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float send = h2 ? b[i] : b[2 + i], keep = h2 ? b[2 + i] : b[i];
    c[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  const float send = h1 ? c[0] : c[1], keep = h1 ? c[1] : c[0];
  float d = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  d += __shfl_xor_sync(0xffffffffu, d, 1);
  return d;
}

template <bool WARP>
__global__ void raymarch_bwd_kernel(RMArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int nwarps = (blockDim.x * blockDim.y + 31) >> 5;
  int* s_hit = reinterpret_cast<int*>(smem);
  float2* s_ivl = reinterpret_cast<float2*>(smem + (size_t)nwarps * kMaxHit * sizeof(int));
  RaySetup r = setup_ray(a, s_hit, s_ivl);
  const unsigned full = 0xffffffffu;
  const int lane = (threadIdx.y * blockDim.x + threadIdx.x) & 31;
  const size_t tsz = (size_t)a.TD * a.TH * a.TW, wsz = (size_t)a.WD * a.WH * a.WW;
  const float stepsize = a.stepsize;
  const size_t o = ((size_t)r.n * a.H + r.h) * a.W + r.w;

  float4 rgba = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 dL = a.grad_rayrgba[o];
  const float3 raysat = ld3(a.raysat + 3 * o);
  bool sat = false;
  float t = r.t;
  float3 pos = r.pos;
  const bool live0 = (t < r.rtmax + 1e-5f);
  float tlo = warp_min(live0 ? t : INFINITY), thi = warp_max(live0 ? t : -INFINITY);
  const float margin = 2.f * stepsize + 1e-3f;

  while (__any_sync(full, (t < r.rtmax + 1e-5f) && !sat)) {
    for (int ks = 0; ks < r.nhit; ++ks) {
      const float2 iv = r.ivl[ks];
      if (thi + margin < iv.x || tlo - margin > iv.y) continue;
      const int k = r.hit[ks];
      Local L = prim_local(r, k, pos);
      const bool evalprim = inside_unit(L.y0) && !sat && t < r.rtmax + 1e-5f;
      float3 dLy0 = make_float3(0.f, 0.f, 0.f);
      if (evalprim) {
        const float3 y0 = L.y0;
        const float fade = __expf(-a.fadescale * (__powf(fabsf(y0.x), a.fadeexp) + __powf(fabsf(y0.y), a.fadeexp) +
                                                  __powf(fabsf(y0.z), a.fadeexp)));
        float3 y1 = y0;
        const float* wptr = WARP ? a.warp + ((size_t)r.n * a.K + k) * 3 * wsz : nullptr;
        if (WARP) y1 = sample3(a.WD, a.WH, a.WW, wptr, y0);
        const float4* tptr = a.tplate + ((size_t)r.n * a.K + k) * tsz;
        float4 s = sample4(a.TD, a.TH, a.TW, tptr, y1);
        s.w *= fade;
        // PrimAccumAdditive::forwardbackward_prim (primaccum.h:81-98)
        const float aw = s.w * stepsize;
        const bool thissat = rgba.w + aw >= 1.f;
        sat = sat || thissat;
        const float weight = sat ? (1.f - rgba.w) : aw;
        float4 dLs;
        dLs.x = weight * dL.x; dLs.y = weight * dL.y; dLs.z = weight * dL.z;
        const bool hs = raysat.x > -1.f;
        const float4 ref = hs ? make_float4(raysat.x, raysat.y, raysat.z, 1.f) : make_float4(0.f, 0.f, 0.f, 0.f);
        dLs.w = sat ? 0.f
                    : stepsize * ((s.x - ref.x) * dL.x + (s.y - ref.y) * dL.y + (s.z - ref.z) * dL.z + (1.f - ref.w) * dL.w);
        rgba.x += s.x * weight; rgba.y += s.y * weight; rgba.z += s.z * weight; rgba.w += 1.f * weight;
        // PrimSamplerTW::backward (primsampler.h:69-92); with a warp field the fade/warp-grid gradients are taken
        // at the WARPED coordinate, like the reference
        const float3 yq = WARP ? y1 : y0;
        float3 dfade = make_float3(__powf(fabsf(yq.x), a.fadeexp - 1.f) * (yq.x > 0.f ? 1.f : -1.f),
                                   __powf(fabsf(yq.y), a.fadeexp - 1.f) * (yq.y > 0.f ? 1.f : -1.f),
                                   __powf(fabsf(yq.z), a.fadeexp - 1.f) * (yq.z > 0.f ? 1.f : -1.f));
        dfade = dfade * (-(a.fadescale * a.fadeexp));
        dLy0 = dfade * s.w * dLs.w;
        dLs.w *= fade;
        const float4 gs = r.validthread ? dLs : make_float4(0.f, 0.f, 0.f, 0.f);
        const float3 dLy1 = sample4_bwd(a.TD, a.TH, a.TW, tptr, a.grad_tplate + ((size_t)r.n * a.K + k) * 4 * tsz, y1, gs,
                                        r.validthread);
        if (WARP) {
          const float3 g3 = r.validthread ? dLy1 : make_float3(0.f, 0.f, 0.f);
          dLy0 = dLy0 + sample3_bwd(a.WD, a.WH, a.WW, wptr, a.grad_warp + ((size_t)r.n * a.K + k) * 3 * wsz, yq, g3,
                                    r.validthread);
        } else {
          dLy0 = dLy0 + dLy1;
        }
      }
      if (__any_sync(full, evalprim)) {
        // PrimTransfSRT::backward (primtransf.h:155-179): 15 sums over the warp, one RED each
        const bool vt = r.validthread && evalprim;
        float v[16];
        const float3 gsc = L.rxmt * dLy0;
        const float3 d = dLy0 * L.ps;
        v[0] = vt ? -dot3(L.pr0, d) : 0.f; v[1] = vt ? -dot3(L.pr1, d) : 0.f; v[2] = vt ? -dot3(L.pr2, d) : 0.f;
        v[3] = vt ? L.xmt.x * d.x : 0.f; v[4] = vt ? L.xmt.x * d.y : 0.f; v[5] = vt ? L.xmt.x * d.z : 0.f;
        v[6] = vt ? L.xmt.y * d.x : 0.f; v[7] = vt ? L.xmt.y * d.y : 0.f; v[8] = vt ? L.xmt.y * d.z : 0.f;
        v[9] = vt ? L.xmt.z * d.x : 0.f; v[10] = vt ? L.xmt.z * d.y : 0.f; v[11] = vt ? L.xmt.z * d.z : 0.f;
        v[12] = vt ? gsc.x : 0.f; v[13] = vt ? gsc.y : 0.f; v[14] = vt ? gsc.z : 0.f; v[15] = 0.f;
        const float tot = reduce16(v, lane);
        const int slot = lane >> 1;
        if (!(lane & 1) && slot < 15) {
          const size_t nk = (size_t)r.n * a.K + k;
          float* dst = slot < 3 ? a.grad_primpos + nk * 3 + slot
                                : (slot < 12 ? a.grad_primrot + nk * 9 + (slot - 3) : a.grad_primscale + nk * 3 + (slot - 12));
          gb::red_add(dst, tot);
        }
      }
    }
    t += stepsize;
    pos = pos + r.raydir * stepsize;
    tlo += stepsize;
    thi += stepsize;
  }
}

// ------------------------------------------------------------------ backward, lane-compacted (algo 0)
// Same idea as raymarch_fwd_queue_kernel, four phases per flush:
//   1 (lanes = items)  fade + trilinear sample of every queued (ray, primitive) pair
//   2 (lanes = rays)   the ordered recurrence of PrimAccumAdditive::forwardbackward_prim (primaccum.h:81-98): each ray walks
//                      its own items group by group, updates (rgba, sat) and leaves dL/d(sample) of every item in shared memory
//   3 (lanes = items)  PrimSamplerTW::backward (primsampler.h:69-92): fade gradient, template-gradient REDs (one 16-byte RED per
//                      trilinear corner), gradient of the local coordinate
//   4 (lanes = items)  PrimTransfSRT::backward (primtransf.h:155-179): the 15 transform sums, reduced over runs of consecutive
//                      items of the SAME primitive with a segmented shuffle scan, one RED per value and run
// Per ray the arithmetic and its order are those of raymarch_bwd_kernel<false>; sums over the rays of a warp are re-associated
// (different reduction tree), as they already are between the reference and round 1.
struct RMQueueB {
  float4 q[kQueue];   // y0.xyz, primitive id (bit-inverted for the clamped duplicate threads of an edge block)
  float4 x[kQueue];   // xmt.xyz (sample position minus primitive centre), fade
  float4 s[kQueue];   // sampled rgba, alpha already faded
  float4 d[kQueue];   // dL/d(sample) rgba (alpha part before the fade factor)
  unsigned g[kQueue];
};

__global__ void raymarch_bwd_queue_kernel(RMArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int nwarps = (blockDim.x * blockDim.y + 31) >> 5;
  int* s_hit = reinterpret_cast<int*>(smem);
  float2* s_ivl = reinterpret_cast<float2*>(smem + (size_t)nwarps * kMaxHit * sizeof(int));
  RMQueueB* s_q = reinterpret_cast<RMQueueB*>(smem + (size_t)nwarps * kMaxHit * (sizeof(int) + sizeof(float2)));
  RaySetup r = setup_ray(a, s_hit, s_ivl);
  const unsigned full = 0xffffffffu;
  const int lane = (threadIdx.y * blockDim.x + threadIdx.x) & 31;
  RMQueueB& Q = s_q[(threadIdx.y * blockDim.x + threadIdx.x) >> 5];
  const unsigned lt = (1u << lane) - 1u;
  const size_t tsz = (size_t)a.TD * a.TH * a.TW;
  const float stepsize = a.stepsize;
  const size_t o = ((size_t)r.n * a.H + r.h) * a.W + r.w;
  const float4* tbase = a.tplate + (size_t)r.n * a.K * tsz;
  float* gtbase = a.grad_tplate + (size_t)r.n * a.K * 4 * tsz;

  float4 rgba = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 dL = a.grad_rayrgba[o];
  const float3 raysat = ld3(a.raysat + 3 * o);
  const bool hs = raysat.x > -1.f;
  const float4 ref = hs ? make_float4(raysat.x, raysat.y, raysat.z, 1.f) : make_float4(0.f, 0.f, 0.f, 0.f);
  bool sat = false;
  float t = r.t;
  float3 pos = r.pos;
  const bool live0 = (t < r.rtmax + 1e-5f);
  float tlo = warp_min(live0 ? t : INFINITY), thi = warp_max(live0 ? t : -INFINITY);
  const float margin = 2.f * stepsize + 1e-3f;
  int qn = 0, ng = 0;

  auto flush = [&]() {
    __syncwarp();
    for (int base = 0; base < qn; base += 32) {  // phase 1
      const int i = base + lane;
      if (i < qn) {
        const float4 it = Q.q[i];
        const float3 y0 = make_float3(it.x, it.y, it.z);
        const int kv = __float_as_int(it.w), k = kv < 0 ? ~kv : kv;
        const float fade = __expf(-a.fadescale * (__powf(fabsf(y0.x), a.fadeexp) + __powf(fabsf(y0.y), a.fadeexp) +
                                                  __powf(fabsf(y0.z), a.fadeexp)));
        float4 sv = sample4(a.TD, a.TH, a.TW, tbase + (size_t)k * tsz, y0);
        sv.w *= fade;
        Q.s[i] = sv;
        Q.x[i].w = fade;
      }
    }
    __syncwarp();
    int off = 0;
    for (int g = 0; g < ng; ++g) {  // phase 2
      const unsigned m = Q.g[g];
      if ((m >> lane) & 1u) {
        const int i = off + __popc(m & lt);
        float4 dLs = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!sat) {
          const float4 sv = Q.s[i];
          const float aw = sv.w * stepsize;
          const bool thissat = rgba.w + aw >= 1.f;
          sat = sat || thissat;
          const float weight = sat ? (1.f - rgba.w) : aw;
          dLs.x = weight * dL.x; dLs.y = weight * dL.y; dLs.z = weight * dL.z;
          dLs.w = sat ? 0.f
                      : stepsize * ((sv.x - ref.x) * dL.x + (sv.y - ref.y) * dL.y + (sv.z - ref.z) * dL.z + (1.f - ref.w) * dL.w);
          rgba.x += sv.x * weight; rgba.y += sv.y * weight; rgba.z += sv.z * weight; rgba.w += 1.f * weight;
        }
        Q.d[i] = dLs;
      }
      off += __popc(m);
    }
    __syncwarp();
    for (int base = 0; base < qn; base += 32) {  // phases 3 and 4
      const int i = base + lane;
      const bool act = i < qn;
      int kv = -1 - 0x7fffffff;  // never equal to a real id
      float v[15];
#pragma unroll
      for (int c = 0; c < 15; ++c) v[c] = 0.f;
      if (act) {
        const float4 it = Q.q[i];
        kv = __float_as_int(it.w);
        const bool valid = kv >= 0;
        const int k = valid ? kv : ~kv;
        kv = k;  // runs are formed on the primitive id alone
        const float4 dl = Q.d[i];
        if (valid && (dl.x != 0.f || dl.y != 0.f || dl.z != 0.f || dl.w != 0.f)) {
          const float3 y0 = make_float3(it.x, it.y, it.z);
          const float4 xm = Q.x[i];
          const float4 sv = Q.s[i];
          float3 dfade = make_float3(__powf(fabsf(y0.x), a.fadeexp - 1.f) * (y0.x > 0.f ? 1.f : -1.f),
                                     __powf(fabsf(y0.y), a.fadeexp - 1.f) * (y0.y > 0.f ? 1.f : -1.f),
                                     __powf(fabsf(y0.z), a.fadeexp - 1.f) * (y0.z > 0.f ? 1.f : -1.f));
          dfade = dfade * (-(a.fadescale * a.fadeexp));
          float3 dLy0 = dfade * sv.w * dl.w;
          const float4 gs = make_float4(dl.x, dl.y, dl.z, dl.w * xm.w);
          const float3 dLy1 = sample4_bwd(a.TD, a.TH, a.TW, tbase + (size_t)k * tsz, gtbase + (size_t)k * 4 * tsz, y0, gs, true);
          dLy0 = dLy0 + dLy1;
          const float3 xmt = make_float3(xm.x, xm.y, xm.z);
          const float3 pr0 = ld3(r.pr + 9 * (size_t)k), pr1 = ld3(r.pr + 9 * (size_t)k + 3), pr2 = ld3(r.pr + 9 * (size_t)k + 6);
          const float3 ps = ld3(r.ps + 3 * (size_t)k);
          const float3 rxmt = pr0 * xmt.x + pr1 * xmt.y + pr2 * xmt.z;
          const float3 gsc = rxmt * dLy0;
          const float3 d = dLy0 * ps;
          v[0] = -dot3(pr0, d); v[1] = -dot3(pr1, d); v[2] = -dot3(pr2, d);
          v[3] = xmt.x * d.x; v[4] = xmt.x * d.y; v[5] = xmt.x * d.z;
          v[6] = xmt.y * d.x; v[7] = xmt.y * d.y; v[8] = xmt.y * d.z;
          v[9] = xmt.z * d.x; v[10] = xmt.z * d.y; v[11] = xmt.z * d.z;
          v[12] = gsc.x; v[13] = gsc.y; v[14] = gsc.z;
        }
      }
      // segmented inclusive scan over runs of equal primitive id; the last lane of a run adds the run's sums
      const int kprev = __shfl_up_sync(full, kv, 1);
      const bool head = (lane == 0) || (kprev != kv);
      const unsigned hm = __ballot_sync(full, head);
      const int myhead = 31 - __clz(hm & (lt | (1u << lane)));
      const int dist = lane - myhead;
#pragma unroll
      for (int sh = 1; sh < 32; sh <<= 1) {
#pragma unroll
        for (int c = 0; c < 15; ++c) {
          const float up = __shfl_up_sync(full, v[c], sh);
          if (dist >= sh) v[c] += up;
        }
      }
      const bool tail = act && (lane == 31 || ((hm >> (lane + 1)) & 1u));
      if (tail) {
        bool any = false;
#pragma unroll
        for (int c = 0; c < 15; ++c) any = any || (v[c] != 0.f);
        if (any) {
          const size_t nk = (size_t)r.n * a.K + kv;
#pragma unroll
          for (int c = 0; c < 3; ++c) gb::red_add(a.grad_primpos + nk * 3 + c, v[c]);
#pragma unroll
          for (int c = 0; c < 9; ++c) gb::red_add(a.grad_primrot + nk * 9 + c, v[3 + c]);
#pragma unroll
          for (int c = 0; c < 3; ++c) gb::red_add(a.grad_primscale + nk * 3 + c, v[12 + c]);
        }
      }
    }
    qn = 0;
    ng = 0;
    __syncwarp();
  };

  while (__any_sync(full, (t < r.rtmax + 1e-5f) && !sat)) {
    for (int ks = 0; ks < r.nhit; ++ks) {
      const float2 iv = r.ivl[ks];
      if (thi + margin < iv.x || tlo - margin > iv.y) continue;
      const int k = r.hit[ks];
      const Local L = prim_local(r, k, pos);
      const bool in = inside_unit(L.y0) && !sat && t < r.rtmax + 1e-5f;
      const unsigned m = __ballot_sync(full, in);
      if (m == 0u) continue;
      if (in) {
        const int i = qn + __popc(m & lt);
        Q.q[i] = make_float4(L.y0.x, L.y0.y, L.y0.z, __int_as_float(r.validthread ? k : ~k));
        Q.x[i] = make_float4(L.xmt.x, L.xmt.y, L.xmt.z, 0.f);
      }
      if (lane == 0) Q.g[ng] = m;
      qn += __popc(m);
      ++ng;
      if (qn >= 32) flush();
    }
    t += stepsize;
    pos = pos + r.raydir * stepsize;
    tlo += stepsize;
    thi += stepsize;
    if (qn >= 16) flush();
  }
  flush();
}

// ------------------------------------------------------------------ BVH bounds (any binary tree, Karras bottom-up)
__global__ void __launch_bounds__(256) compute_aabb_kernel(int N, int K, const float* __restrict__ primpos,
                                                           const float* __restrict__ primrot,
                                                           const float* __restrict__ primscale,
                                                           const int* __restrict__ sortedobjid,
                                                           const int2* __restrict__ nodechildren,
                                                           const int* __restrict__ nodeparent, float* nodeaabb,
                                                           int* flags /* [N, K-1] zeroed */) {
  const int NN = 2 * K - 1;
  for (int index = blockIdx.x * blockDim.x + threadIdx.x; index < N * K; index += blockDim.x * gridDim.x) {
    const int k = index % K, n = index / K;
    const int kk = sortedobjid[(size_t)n * K + k];
    const float3 pt = ld3(primpos + ((size_t)n * K + kk) * 3);
    const float* R = primrot + ((size_t)n * K + kk) * 9;
    const float3 r0 = ld3(R), r1 = ld3(R + 3), r2 = ld3(R + 6);
    const float3 ps = ld3(primscale + ((size_t)n * K + kk) * 3);
    float3 pmin, pmax;
#pragma unroll
    for (int c = 0; c < 8; ++c) {  // corner order of compute_aabb_srt (primtransf.h:12-63)
      float3 p = make_float3(((c & 1) ? 1.f : -1.f) / ps.x, ((c & 2) ? 1.f : -1.f) / ps.y, ((c & 4) ? 1.f : -1.f) / ps.z);
      p = make_float3(dot3(p, r0), dot3(p, r1), dot3(p, r2)) + pt;
      if (c == 0) { pmin = p; pmax = p; } else { pmin = min3(pmin, p); pmax = max3(pmax, p); }
    }
    float* A = nodeaabb + (size_t)n * NN * 6;
    float* leaf = A + (size_t)(K - 1 + k) * 6;
    leaf[0] = pmin.x; leaf[1] = pmin.y; leaf[2] = pmin.z; leaf[3] = pmax.x; leaf[4] = pmax.y; leaf[5] = pmax.z;
    int node = nodeparent[(size_t)n * NN + (K - 1 + k)];
    while (node != -1) {
      __threadfence();  // publish this subtree's box before announcing arrival
      if (atomicAdd(&flags[(size_t)n * (K - 1) + node], 1) == 0) break;  // first child to arrive stops here
      __threadfence();
      const int2 ch = nodechildren[(size_t)n * NN + node];
      const volatile float* l = A + (size_t)ch.x * 6;
      const volatile float* rr = A + (size_t)ch.y * 6;
      float* me = A + (size_t)node * 6;
#pragma unroll
      for (int c = 0; c < 3; ++c) { me[c] = fminf(l[c], rr[c]); me[3 + c] = fmaxf(l[3 + c], rr[3 + c]); }
      node = nodeparent[(size_t)n * NN + node];
    }
  }
}

// bit 0: lane-compacted sampling queue in the forward march, bit 1: in the backward march (algo 0, no shadow splat).
// Default 2 = queue in the BACKWARD only, from measurement: bench.py --config hand_mvp (decode + raymarch fwd+bwd) on an
// H100 SXM at a 400 W power limit, two runs each: queue in the backward 34.72 / 34.72 ms per step, no queue 37.85 /
// 37.96, both 35.65 / 35.90, forward only 38.94 / 38.93.  The backward, whose per-item block carries the template-gradient
// REDs and the fade / position gradients, gains; the forward does not — it is bound by dependent-load latency (BVH walk,
// template corners), not by issue slots, and the queue adds shared-memory round trips.
int g_raymarch_mode = -1;
int raymarch_mode() {
  if (g_raymarch_mode < 0) {
    const char* e = getenv("GOLIATH_B200_RAYMARCH");
    g_raymarch_mode = !e ? 2 : strcmp(e, "queue") == 0 ? 3 : strcmp(e, "queue-fwd") == 0 ? 1 : strcmp(e, "queue-bwd") == 0 ? 2 : 0;
  }
  return g_raymarch_mode;
}

int fill_and_launch_check(const RMArgs& a, int bx, int by) {
  if (a.N <= 0 || a.H <= 0 || a.W <= 0) return 1;
  // whole warps only: the hit list is a warp-wide union built with full-mask votes (the reference asserts the
  // same through its 0xffffffff warpmask, mvpraymarch_subset_kernel.h:38)
  if (a.K < 1 || bx < 1 || by < 1 || bx * by > 1024 || (bx * by) % 32 != 0) return -1;
  return 0;
}

}  // namespace

// bit 0 / bit 1: lane-compacted sampling queue in the forward / backward march (default 2: backward only);
// rays identical, transform gradients to re-association (A/B, tests).
GB_API int gb_get_raymarch_mode(void) { return raymarch_mode(); }
GB_API void gb_set_raymarch_mode(int mode) { g_raymarch_mode = mode & 3; }

// scratch for gb_mvp_compute_aabb: N*(K-1) int flags (zeroed by the call itself)
GB_API size_t gb_mvp_aabb_workspace_bytes(int N, int K) { return (size_t)N * (K > 1 ? K - 1 : 1) * sizeof(int); }

// replaces mvpraymarchlib.compute_aabb (mvpraymarch.cpp compute_aabb -> bvh.cu:157-201,249-294).
// nodeaabb [N,2K-1,2,3] out; sortedobjid [N,K], nodechildren [N,2K-1,2], nodeparent [N,2K-1] as built by
// mvpraymarch.py:44-82.
GB_API int gb_mvp_compute_aabb(int N, int K, const float* primpos, const float* primrot, const float* primscale,
                               const int32_t* sortedobjid, const int32_t* nodechildren, const int32_t* nodeparent,
                               float* nodeaabb, void* workspace, void* stream) {
  if (N <= 0 || K <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  GB_CUDA(cudaMemsetAsync(workspace, 0, gb_mvp_aabb_workspace_bytes(N, K), s));
  const int blocks = min(gb::cdiv(N * K, 256), gb::kNumSMs * 8);
  return gb::launch<compute_aabb_kernel>(blocks, 256, 0, s, N, K, primpos, primrot, primscale, sortedobjid,
                                         (const int2*)nodechildren, nodeparent, nodeaabb, (int*)workspace);
}

// replaces mvpraymarchlib.raymarch_forward (mvpraymarch.cpp:179-283 -> mvpraymarch_kernel.cu:41-130).
// Only the arguments the reference kernels actually read are part of the ABI (SURVEY.md §0.9): algo in {0,1}
// (warp field off/on), fadescale, fadeexp, block size, optional raysat / shadow outputs.
GB_API int gb_mvp_raymarch_fwd(int N, int H, int W, int K, const float* raypos, const float* raydir, float stepsize,
                               const float* tminmax, const float* nodeaabb, const float* primpos,
                               const float* primrot, const float* primscale, int TD, int TH, int TW,
                               const float* tplate, int WD, int WH, int WW, const float* warp, float* rayrgba,
                               float* raysat, float* shadow, int algo, float fadescale, float fadeexp, int blocksizex,
                               int blocksizey, void* stream) {
  RMArgs a = {};
  a.N = N; a.H = H; a.W = W; a.K = K; a.raypos = raypos; a.raydir = raydir; a.stepsize = stepsize;
  a.tminmax = (const float2*)tminmax; a.nodeaabb = nodeaabb; a.primpos = primpos; a.primrot = primrot;
  a.primscale = primscale; a.TD = TD; a.TH = TH; a.TW = TW; a.tplate = (const float4*)tplate; a.WD = WD; a.WH = WH;
  a.WW = WW; a.warp = warp; a.fadescale = fadescale; a.fadeexp = fadeexp; a.rayrgba = (float4*)rayrgba;
  a.raysat = raysat; a.shadow = shadow;
  const int chk = fill_and_launch_check(a, blocksizex, blocksizey);
  if (chk > 0) return 0;
  if (chk < 0 || (algo != 0 && algo != 1) || (algo == 1 && !warp)) return (int)cudaErrorInvalidValue;
  dim3 block(blocksizex, blocksizey);
  dim3 grid(gb::cdiv(W, blocksizex), gb::cdiv(H, blocksizey), N);
  const int nwarps = (blocksizex * blocksizey + 31) / 32;
  const size_t smem = (size_t)nwarps * kMaxHit * (sizeof(int) + sizeof(float2));
  cudaStream_t s = (cudaStream_t)stream;
  if (algo == 1) {
    if (shadow) return gb::launch<raymarch_fwd_kernel<true, true>>(grid, block, smem, s, a);
    return gb::launch<raymarch_fwd_kernel<true, false>>(grid, block, smem, s, a);
  }
  if (shadow) return gb::launch<raymarch_fwd_kernel<false, true>>(grid, block, smem, s, a);
  if (raymarch_mode() & 1)  // lane-compacted sampling (option, algo 0 without the shadow splat)
    return gb::launch<raymarch_fwd_queue_kernel>(grid, block, smem + (size_t)nwarps * sizeof(RMQueue), s, a);
  return gb::launch<raymarch_fwd_kernel<false, false>>(grid, block, smem, s, a);
}

// replaces mvpraymarchlib.raymarch_backward (mvpraymarch.cpp:285-399 -> mvpraymarch_kernel.cu:132-221).
// All gradient buffers are accumulated into (the caller zero-fills them, mvpraymarch.py:256-263);
// grad_warp is only touched when algo == 1.
GB_API int gb_mvp_raymarch_bwd(int N, int H, int W, int K, const float* raypos, const float* raydir, float stepsize,
                               const float* tminmax, const float* nodeaabb, const float* primpos,
                               const float* primrot, const float* primscale, int TD, int TH, int TW,
                               const float* tplate, int WD, int WH, int WW, const float* warp, const float* raysat,
                               const float* grad_rayrgba, float* grad_primpos, float* grad_primrot,
                               float* grad_primscale, float* grad_tplate, float* grad_warp, int algo, float fadescale,
                               float fadeexp, int blocksizex, int blocksizey, void* stream) {
  RMArgs a = {};
  a.N = N; a.H = H; a.W = W; a.K = K; a.raypos = raypos; a.raydir = raydir; a.stepsize = stepsize;
  a.tminmax = (const float2*)tminmax; a.nodeaabb = nodeaabb; a.primpos = primpos; a.primrot = primrot;
  a.primscale = primscale; a.TD = TD; a.TH = TH; a.TW = TW; a.tplate = (const float4*)tplate; a.WD = WD; a.WH = WH;
  a.WW = WW; a.warp = warp; a.fadescale = fadescale; a.fadeexp = fadeexp; a.raysat = const_cast<float*>(raysat);
  a.grad_rayrgba = (const float4*)grad_rayrgba; a.grad_primpos = grad_primpos; a.grad_primrot = grad_primrot;
  a.grad_primscale = grad_primscale; a.grad_tplate = grad_tplate; a.grad_warp = grad_warp;
  const int chk = fill_and_launch_check(a, blocksizex, blocksizey);
  if (chk > 0) return 0;
  if (chk < 0 || (algo != 0 && algo != 1) || (algo == 1 && (!warp || !grad_warp)) || !raysat)
    return (int)cudaErrorInvalidValue;
  dim3 block(blocksizex, blocksizey);
  dim3 grid(gb::cdiv(W, blocksizex), gb::cdiv(H, blocksizey), N);
  const int nwarps = (blocksizex * blocksizey + 31) / 32;
  const size_t smem = (size_t)nwarps * kMaxHit * (sizeof(int) + sizeof(float2));
  cudaStream_t s = (cudaStream_t)stream;
  if (algo == 1) return gb::launch<raymarch_bwd_kernel<true>>(grid, block, smem, s, a);
  if (raymarch_mode() & 2)  // lane-compacted backward (option, algo 0)
    return gb::launch<raymarch_bwd_queue_kernel>(grid, block, smem + (size_t)nwarps * sizeof(RMQueueB), s, a);
  return gb::launch<raymarch_bwd_kernel<false>>(grid, block, smem, s, a);
}

// Deep shadow march of the relightable hand teacher (hand_teacher_mvp.py:274-358 with mvpraymarch(with_shadow=True)):
// N = B * L light views, transforms [B,K,3] / [B,K,3,3] / [B,K,3] and bounds [B,2K-1,2,3] (gb_mvp_compute_aabb with
// N = B) of item n / L, alpha slab [B,TD,U,U] sampled in place (U = n_prim_x * TW = n_prim_y * TH, K = n_prim_x *
// n_prim_y), valid [K] or NULL.  Only output: the un-normalised splat volume shadow [N,K,TD,TH,TW,2], accumulated
// into (the caller zero-fills it).  No rayrgba, no raysat.
GB_API int gb_mvp_shadow_march(int N, int L, int H, int W, int K, const float* raypos, const float* raydir,
                               float stepsize, const float* tminmax, const float* nodeaabb, const float* primpos,
                               const float* primrot, const float* primscale, int TD, int TH, int TW, int U,
                               const float* alpha_slab, const float* valid, float* shadow, float fadescale,
                               float fadeexp, int blocksizex, int blocksizey, void* stream) {
  RMArgs a = {};
  a.N = N; a.H = H; a.W = W; a.K = K; a.raypos = raypos; a.raydir = raydir; a.stepsize = stepsize;
  a.tminmax = (const float2*)tminmax; a.nodeaabb = nodeaabb; a.primpos = primpos; a.primrot = primrot;
  a.primscale = primscale; a.TD = TD; a.TH = TH; a.TW = TW; a.fadescale = fadescale; a.fadeexp = fadeexp;
  a.shadow = shadow; a.L = L; a.U = U; a.slab = alpha_slab; a.valid = valid;
  const int chk = fill_and_launch_check(a, blocksizex, blocksizey);
  if (chk > 0) return 0;
  if (chk < 0 || L < 1 || N % L != 0 || TD < 1 || TH < 1 || TW < 1 || U % TW != 0 || U % TH != 0 ||
      (U / TW) * (U / TH) != K || !alpha_slab || !shadow)
    return (int)cudaErrorInvalidValue;
  dim3 block(blocksizex, blocksizey);
  dim3 grid(gb::cdiv(W, blocksizex), gb::cdiv(H, blocksizey), N);
  const int nwarps = (blocksizex * blocksizey + 31) / 32;
  const size_t smem = (size_t)nwarps * kMaxHit * (sizeof(int) + sizeof(float2));
  cudaStream_t s = (cudaStream_t)stream;
  return gb::launch<shadow_march_kernel>(grid, block, smem, s, a);
}
