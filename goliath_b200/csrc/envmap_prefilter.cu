// goliath_b200/csrc/envmap_prefilter.cu — environment-spin lighting of the relighting loop (sm_90a).
//
// Replaces ca_code/utils/envmap.py and ca_code/utils/light_decorator.py:
//   prefilterEnvmapSG (envmap.py:305-323) with importance_sample_sg (:251-281) and sample_uv (:295-302): per texel the
//     mean of S bilinear lookups (border, align_corners=False) along directions drawn around v from a spherical
//     Gaussian of width sigma.  One warp per texel, the lanes split the samples and a fixed xor-shuffle tree sums
//     them, so a seed gives bit-identical output; every mip level of a call runs in one launch (the level textures,
//     <= 1.5 MB each, stay in L2).  The pdf the reference computes and discards is not computed.
//   EnvSpinDecorator.forward (light_decorator.py:102-164), per batch item: rvec_to_R of (0, angle, 0) (envmap.py:20-50),
//     rotate_envmap_mat of the probe (gb_envmap_rotate), envbg = rotated / perc90 * 255 / 255, the 16x32 antialiased
//     bilinear downsample (torch's _upsample_bilinear2d_aa: triangle filter of half-width in / out, horizontal pass
//     first), envmap = env_scale * down / sum(down * sin(theta_row)), light_intensity = envmap as [512,3], norm_scale.
//     Three kernels plus one rotate launch per item; no host synchronisation, no copy.
#include <curand_philox4x32_x.h>

#include "envmap_common.cuh"

GB_API int gb_envmap_rotate(int B, int He, int We, const float* image, const float* rot_mat, float* out, void* stream);

namespace {

using gb::Bilin;
using gb::dir2uv;
using gb::fetch;
using gb::locate;

constexpr int kMaxLevels = 8;
constexpr int kWarps = 8;  // prefilter: texels (warps) per block

struct PrefilterArgs {
  int B, q, S;
  int H[kMaxLevels], W[kMaxLevels], He[kMaxLevels], We[kMaxLevels];
  long long first[kMaxLevels + 1];  // first texel (b, y, x flattened) of each level in the launch
  float ks[kMaxLevels], kerf[kMaxLevels];  // float(sqrt(2) sigma), float(erf(pi / (sqrt(2) sigma)))
  const float* v[kMaxLevels];              // [B,3,H,W]
  const float* env[kMaxLevels];            // [B,3,He,We]
  const float* xi[kMaxLevels];             // [S,B,2,H,W] or NULL (Philox)
  float* out[kMaxLevels];                  // [B,3,H,W]
  uint2 key;                               // the seed
};

__device__ __forceinline__ float3 cross3(float3 a, float3 b) {  // th.cross
  return make_float3(__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)),
                     __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
                     __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}

__device__ __forceinline__ float3 normalize3(float3 a) {  // F.normalize(dim=1), eps 1e-12
  const float n = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(a.x, a.x), __fmul_rn(a.y, a.y)), __fmul_rn(a.z, a.z))), 1e-12f);
  return make_float3(__fdiv_rn(a.x, n), __fdiv_rn(a.y, n), __fdiv_rn(a.z, n));
}

// uniform in [0, 1) from 24 random bits, the resolution of torch.rand in fp32
__device__ __forceinline__ float unit(unsigned r) { return (float)(r >> 8) * 0x1p-24f; }

// one warp per texel.  grid cdiv(first[q], kWarps), block 32 * kWarps.
__global__ void __launch_bounds__(32 * kWarps) envmap_prefilter_sg_kernel(PrefilterArgs a) {
  const long long t = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (t >= a.first[a.q]) return;
  int l = 0;
  while (t >= a.first[l + 1]) ++l;
  const int lane = threadIdx.x & 31;
  const int H = a.H[l], W = a.W[l], He = a.He[l], We = a.We[l];
  const long long hw = (long long)H * W, r = t - a.first[l];
  const int b = (int)(r / hw);
  const long long p = r - b * hw;
  const float* vb = a.v[l] + (size_t)b * 3 * hw + p;
  const float3 n = make_float3(vb[0], vb[hw], vb[2 * hw]);
  // up = (0,0,1) where n_z < 0.999, else (1,0,0); t = normalize(up x n), b = n x t
  const float3 up = n.z < 0.999f ? make_float3(0.f, 0.f, 1.f) : make_float3(1.f, 0.f, 0.f);
  const float3 tg = normalize3(cross3(up, n));
  const float3 bt = cross3(n, tg);
  const float ks = a.ks[l], kerf = a.kerf[l];
  constexpr float k2Pi = (float)(2.0 * 3.14159265358979323846);  // 2.0 * np.pi as an fp32 scalar
  const size_t plane = (size_t)He * We;
  const float* env = a.env[l] + (size_t)b * 3 * plane;
  const float* xi = a.xi[l];
  float acc[3] = {0.f, 0.f, 0.f};

  auto sample = [&](float xi0, float xi1) {
    const float phi = __fmul_rn(k2Pi, xi0);
    const float th = __fmul_rn(ks, erfinvf(__fmul_rn(xi1, kerf)));
    const float st = sinf(th), ct = cosf(th);
    float sp, cp;
    sincosf(phi, &sp, &cp);
    const float hx = __fmul_rn(cp, st), hy = __fmul_rn(sp, st);
    // t * Hx + b * Hy + n * Hz, left to right as torch evaluates it
    const float3 s = normalize3(make_float3(
        __fadd_rn(__fadd_rn(__fmul_rn(tg.x, hx), __fmul_rn(bt.x, hy)), __fmul_rn(n.x, ct)),
        __fadd_rn(__fadd_rn(__fmul_rn(tg.y, hx), __fmul_rn(bt.y, hy)), __fmul_rn(n.y, ct)),
        __fadd_rn(__fadd_rn(__fmul_rn(tg.z, hx), __fmul_rn(bt.z, hy)), __fmul_rn(n.z, ct))));
    const float2 uv = dir2uv(s.x, s.y, s.z);
    const Bilin bl = locate(uv.x, uv.y, We, He);
    float dx, dy;
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += fetch(env + c * plane, bl, We, He, dx, dy);
  };

  if (xi) {
    const size_t bstride = (size_t)2 * hw;
    for (int s = lane; s < a.S; s += 32) {
      const float* x = xi + ((size_t)s * a.B + b) * bstride + p;
      sample(x[0], x[hw]);
    }
  } else {
    // counter (sample pair, texel, item, level) under the seed: four 32-bit draws give two samples
    for (int k = lane; 2 * k < a.S; k += 32) {
      const uint4 rnd = curand_Philox4x32_10(make_uint4((unsigned)k, (unsigned)p, (unsigned)b, (unsigned)l), a.key);
      sample(unit(rnd.x), unit(rnd.y));
      if (2 * k + 1 < a.S) sample(unit(rnd.z), unit(rnd.w));
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) acc[c] = gb::warp_sum(acc[c]);
  if (lane < 3) {
    const float v = lane == 0 ? acc[0] : (lane == 1 ? acc[1] : acc[2]);
    a.out[l][(size_t)b * 3 * hw + lane * hw + p] = __fdiv_rn(v, (float)a.S);
  }
}

// ------------------------------------------------------------------------------------------------ per-frame light table
constexpr int kOutH = 16, kOutW = 32;  // the decorator's 16x32 = 512 lights
constexpr int kRowWarps = 4;          // horizontal pass: rows (warps) per block
constexpr int kMaxRotB = 64;          // angles per rotation launch (kernel parameter space)

struct RotArgs {
  int n;
  float angle[kMaxRotB];
};

// rvec_to_R (envmap.py:20-50) of rvec = normalize((0, 1, 0)) * angle, in fp32: n = max(|angle|, 1e-6), r = angle / n,
// R = I + sin(n) N + ((1 - cos(n)) N) @ N with N = [[0, 0, r], [0, 0, 0], [-r, 0, 0]].  angle 0 gives the identity.
__global__ void envmap_spin_rot_kernel(RotArgs a, float* __restrict__ R) {
  const int i = threadIdx.x;
  if (i >= a.n) return;
  const float ang = a.angle[i];
  const float n = fmaxf(sqrtf(__fmul_rn(ang, ang)), 1e-6f);
  const float r = __fdiv_rn(ang, n);
  const float s = sinf(n), omc = __fsub_rn(1.f, cosf(n));
  const float d = __fmul_rn(__fmul_rn(omc, r), -r);  // ((1 - cos) N @ N)[0][0] = [2][2]
  const float sr = __fmul_rn(s, r);
  float* o = R + 9 * i;
  o[0] = __fadd_rn(1.f, d); o[1] = 0.f; o[2] = sr;
  o[3] = 0.f;               o[4] = 1.f; o[5] = 0.f;
  o[6] = -sr;               o[7] = 0.f; o[8] = __fadd_rn(1.f, d);
}

// one output of torch's antialiased bilinear resize along one axis (_compute_weights_aa, align_corners=False,
// antialias=True, in >= out): the triangle filter of half-width scale = in / out over the window [xmin, xmin + xsize),
// weights normalised by their sum, mixed precision as aten evaluates it
struct AaWindow {
  int xmin, xsize;
  float center, invscale, total;
};

__device__ __forceinline__ float aa_filter(float x) {
  x = fabsf(x);
  return x < 1.f ? 1.f - x : 0.f;
}

__device__ __forceinline__ float aa_raw(const AaWindow& w, int j) {
  return aa_filter((float)(((double)((float)(j + w.xmin) - w.center) + 0.5) * (double)w.invscale));
}

__device__ __forceinline__ AaWindow aa_window(int i, int in, int out) {
  AaWindow w;
  const float scale = __fdiv_rn((float)in, (float)out);
  const float support = scale;  // bilinear: interp_size / 2 * scale
  const int max_size = (int)ceilf(support) * 2 + 1;
  w.center = (float)((double)scale * (i + 0.5));
  w.invscale = (float)(1.0 / scale);
  w.xmin = max((int)((double)(w.center - support) + 0.5), 0);
  w.xsize = min(max(min((int)((double)(w.center + support) + 0.5), in) - w.xmin, 0), max_size);
  w.total = 0.f;
  for (int j = 0; j < w.xsize; ++j) w.total += aa_raw(w, j);
  return w;
}

__device__ __forceinline__ float aa_weight(const AaWindow& w, int j) {
  const float x = aa_raw(w, j);
  return w.total != 0.f ? __fdiv_rn(x, w.total) : x;
}

// each warp owns one row (b, c, y) of the rotated probe in envbg: stages it in shared memory, rewrites it in place as
// envbg = row / perc90 * 255 / 255, and lane x writes column x of the horizontal pass hpass [B,3,He,32].
// grid cdiv(B * 3 * He, kRowWarps), block 32 * kRowWarps, dynamic shared kRowWarps * We floats.
__global__ void __launch_bounds__(32 * kRowWarps) envmap_spin_hpass_kernel(int rows, int We, float perc90,
                                                                           float* __restrict__ envbg,
                                                                           float* __restrict__ hpass) {
  extern __shared__ float srow[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * kRowWarps + warp;
  if (row >= rows) return;
  float* s = srow + warp * We;
  float* g = envbg + (size_t)row * We;
  for (int x = lane; x < We; x += 32) {
    const float v = g[x];
    s[x] = v;
    g[x] = __fdiv_rn(__fmul_rn(__fdiv_rn(v, perc90), 255.f), 255.f);
  }
  __syncwarp();
  const AaWindow w = aa_window(lane, We, kOutW);
  const float* src = s + w.xmin;
  float acc = 0.f;
  for (int j = 0; j < w.xsize; ++j) acc = __fadd_rn(acc, __fmul_rn(src[j], aa_weight(w, j)));
  hpass[(size_t)row * kOutW + lane] = acc;
}

// one block per item: the vertical pass of the 16x32 downsample, then the sin-weighted sum (a fixed-order block
// reduction), envmap = env_scale * down / sum, light_intensity[k][c] = envmap[c][k], norm_scale = (1 / sum) * env_scale
// (torch's scalar / tensor is reciprocal * scalar).  grid B, block 512 (one thread per light).
__global__ void __launch_bounds__(kOutH * kOutW) envmap_spin_table_kernel(int He, float env_scale,
                                                                          const float* __restrict__ hpass,
                                                                          float* __restrict__ envmap,
                                                                          float* __restrict__ light_intensity,
                                                                          float* __restrict__ norm_scale) {
  __shared__ float part[kOutH * kOutW / 32];
  __shared__ float total;
  const int b = blockIdx.x, k = threadIdx.x, oy = k / kOutW, ox = k - oy * kOutW;
  const AaWindow w = aa_window(oy, He, kOutH);
  float down[3];
  float sum = 0.f;
  // sin((arange(16) + 0.5) * np.pi / 16) in fp32
  const float sw = sinf(__fdiv_rn(__fmul_rn((float)oy + 0.5f, (float)3.14159265358979323846), (float)kOutH));
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* src = hpass + (((size_t)b * 3 + c) * He + w.xmin) * kOutW + ox;
    float acc = 0.f;
    for (int j = 0; j < w.xsize; ++j) acc = __fadd_rn(acc, __fmul_rn(src[(size_t)j * kOutW], aa_weight(w, j)));
    down[c] = acc;
    sum += __fmul_rn(acc, sw);
  }
  sum = gb::warp_sum(sum);
  if ((k & 31) == 0) part[k >> 5] = sum;
  __syncthreads();
  if (k == 0) {
    float t = 0.f;
    for (int i = 0; i < kOutH * kOutW / 32; ++i) t += part[i];
    total = t;
    norm_scale[b] = __fmul_rn(__frcp_rn(t), env_scale);
  }
  __syncthreads();
  const float t = total;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float e = __fdiv_rn(__fmul_rn(env_scale, down[c]), t);
    envmap[((size_t)b * 3 + c) * kOutH * kOutW + k] = e;
    light_intensity[((size_t)b * kOutH * kOutW + k) * 3 + c] = e;
  }
}

}  // namespace

GB_API int gb_envmap_prefilter_sg(int B, int q, const int32_t* level_hw, const float* sigma, const float* const* v,
                                  const float* const* env_tex, const float* const* xi, int num_samples,
                                  unsigned long long seed, float* const* out, void* stream) {
  if (B <= 0 || q == 0) return 0;
  if (q < 0 || q > kMaxLevels || num_samples < 1 || !level_hw || !sigma || !v || !env_tex || !out)
    return (int)cudaErrorInvalidValue;
  PrefilterArgs a = {};
  a.B = B; a.q = q; a.S = num_samples;
  a.key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  a.first[0] = 0;
  for (int l = 0; l < q; ++l) {
    a.H[l] = level_hw[4 * l]; a.W[l] = level_hw[4 * l + 1];
    a.He[l] = level_hw[4 * l + 2]; a.We[l] = level_hw[4 * l + 3];
    if (a.H[l] < 1 || a.W[l] < 1 || a.He[l] < 1 || a.We[l] < 1 || !(sigma[l] > 0.f) || !v[l] || !env_tex[l] || !out[l])
      return (int)cudaErrorInvalidValue;
    // importance_sample_sg's host scalars: math.sqrt(2.0) * sigma and math.erf(np.pi / sqrt2sigma), in double
    const double s2 = 1.4142135623730951 * (double)sigma[l];
    a.ks[l] = (float)s2;
    a.kerf[l] = (float)erf(3.141592653589793 / s2);
    a.v[l] = v[l]; a.env[l] = env_tex[l]; a.out[l] = out[l];
    a.xi[l] = xi ? xi[l] : nullptr;
    a.first[l + 1] = a.first[l] + (long long)B * a.H[l] * a.W[l];
  }
  const long long blocks = gb::cdiv64(a.first[q], kWarps);
  if (blocks > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  return gb::launch<envmap_prefilter_sg_kernel>((unsigned)blocks, 32 * kWarps, 0, (cudaStream_t)stream, a);
}

GB_API int gb_envmap_spin_table(int B, int He, int We, const float* angles, const float* image, float perc90,
                                float env_scale, float* lightrot, float* envbg, float* hpass, float* envmap,
                                float* light_intensity, float* norm_scale, void* stream) {
  if (B <= 0) return 0;
  if (He < kOutH || We < kOutW || (size_t)We * kRowWarps * sizeof(float) > 48 * 1024 || !(perc90 > 0.f) || !angles)
    return (int)cudaErrorInvalidValue;
  const cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < B; b0 += kMaxRotB) {
    RotArgs r;
    r.n = B - b0 < kMaxRotB ? B - b0 : kMaxRotB;
    for (int i = 0; i < r.n; ++i) r.angle[i] = angles[b0 + i];
    GB_CUDA(gb::launch<envmap_spin_rot_kernel>(1, kMaxRotB, 0, st, r, lightrot + 9 * (size_t)b0));
  }
  const size_t plane = (size_t)He * We;
  for (int b = 0; b < B; ++b) {  // one probe for every item: the rotation's batch stride is one image
    const int e = gb_envmap_rotate(1, He, We, image, lightrot + 9 * (size_t)b, envbg + 3 * plane * b, stream);
    if (e) return e;
  }
  const int rows = B * 3 * He;
  GB_CUDA(gb::launch<envmap_spin_hpass_kernel>(gb::cdiv(rows, kRowWarps), 32 * kRowWarps, kRowWarps * We * sizeof(float),
                                               st, rows, We, perc90, envbg, hpass));
  return gb::launch<envmap_spin_table_kernel>(B, kOutH * kOutW, 0, st, He, env_scale, hpass, envmap, light_intensity,
                                              norm_scale);
}
