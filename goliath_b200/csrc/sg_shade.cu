// goliath_b200/csrc/sg_shade.cu — spherical-Gaussian specular shade, forward + backward (sm_90a).
//
// Replaces the reference kernels extensions/sgutils/sg.cu:27-76 (fwd) and :78-175 (bwd) behind the
// same argument meaning (C ABI in include/goliath_b200.h: gb_sg_evaluate_fwd / gb_sg_evaluate_bwd).
//
// Design: one thread per Gaussian, the batch item's light table (position + value, 24 B/light)
// staged once per CTA in shared memory in chunks of kLightChunk, so the inner loop reads lights as
// conflict-free broadcasts instead of the reference's per-pair global loads.  For L >= 4 the kernel is
// FP32/SFU bound (acos + ex2 + rsqrt per pair), for L <= 2 it is a streaming HBM kernel (40 B in,
// 12 B out per Gaussian).  grad_light_values (optional) is reduced warp -> CTA (shared) -> one RED per
// (CTA, light, channel) instead of the reference's 3 global atomics per (Gaussian, light).
//
// Numerics: this translation unit is compiled with -use_fast_math exactly like the reference's extension
// (extensions/sgutils/setup.py:31) and evaluates each (Gaussian, light) pair with the reference's formula in
// the reference's operation order (clamped cosine -> acosf -> __expf, divisions where sg.cu divides), and
// accumulates over lights sequentially per thread, so forward values and grad_dirs / grad_sigmas agree with
// the reference kernels to the last bits; the -20 clamp-edge derivative (sg.cu:129,139) is kept.
#include "common.cuh"

namespace {

constexpr float TWOPI = 6.28318530718f;
constexpr float INV2PI = 0.15915494309f;
constexpr float SQRT2PI23 = 3.03352966508f;
constexpr float INVSQRT2PI23 = 0.32964899322f;
constexpr int kBlock = 128;
constexpr int kLightChunk = 256;  // 256 lights * 24 B = 6 KB of shared memory

__device__ __forceinline__ float sq(float v) { return v * v; }

// ---- the fused (shade_compose) pass, w_type 0: the per-pair arithmetic regrouped for the FP32 / SFU pipes.
// The drop-in binding above keeps the reference's operation order (bit parity with sg.cu); the fused pass has the
// oracle's 1e-4 bar instead and evaluates a pair with 3 SFU operations and ~33 instructions (was 4 / 53):
//   cos    = (l . dir) * rsqrt(l . l)                      (no normalised light vector, no division)
//   angle  = acos(cos) = sqrt(1 - |c|) * P7(|c|), reflected for c < 0   (Abramowitz & Stegun 4.4.46, |err| <= 2e-8)
//   weight = ex2(-0.5 log2e (angle / sigma)^2) / (sigma K)   with 1 / sigma and 1 / (sigma K) hoisted per Gaussian and the
//            normalisation applied once to the light sum.
__device__ __forceinline__ float rsqrt_approx(float x) {
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float sqrt_approx(float x) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
// acos of c in [-1, 1]; `a` = |c|, `s` = 1 - a are shared with the caller
__device__ __forceinline__ float acos_as(float c, float a, float s) {
  float p = -0.0012624911f;
  p = p * a + 0.0066700901f;
  p = p * a - 0.0170881256f;
  p = p * a + 0.0308918810f;
  p = p * a - 0.0501743046f;
  p = p * a + 0.0889789874f;
  p = p * a - 0.2145988016f;
  p = p * a + 1.5707963050f;
  const float r = sqrt_approx(s) * p;
  return c < 0.f ? 3.14159265358979f - r : r;
}
constexpr float kHalfLog2e = 0.72134752044448f;  // 0.5 * log2(e)

// Optional fusion of the shade's surroundings in ca_code/models/rgca.py:557-575 (and F.normalize of
// extensions/sgutils/sgutils.py:74-75) into the same pass: lobe direction normalised in-kernel, specular = integral *
// spec_vis, colour = clamp(clamp(diffuse, 0) + specular, 0).  The per-(Gaussian, light) arithmetic is untouched.
// The stored colour carries the sign of the pre-clamp value in its sign bit (-0.0f where it was negative) so that the
// backward can apply torch's clamp rule (gradient passes where pre >= 0) without a second pass over the lights.
struct Compose {
  const float* diff_color;  // [N,D,3]
  const float* spec_vis;    // [N,D]
  float* color;             // [N,D,3] out (fwd) / saved (bwd)
  float* spec_color;        // [N,D,3] out or null
  // backward only
  const float* g_color;       // [N,D,3]
  const float* g_spec_color;  // [N,D,3] or null
  float* g_diff;              // [N,D,3]
  float* g_vis;               // [N,D]
};

__device__ __forceinline__ float3 normalize_rn(float3 r, float& len_out) {  // F.normalize(eps = 1e-12), exact div/sqrt
  const float len = fmaxf(__fsqrt_rn(r.x * r.x + r.y * r.y + r.z * r.z), 1e-12f);
  len_out = len;
  return make_float3(__fdiv_rn(r.x, len), __fdiv_rn(r.y, len), __fdiv_rn(r.z, len));
}

template <int WT, bool FUSED>
__global__ void __launch_bounds__(kBlock) sg_fwd_kernel(const float* __restrict__ lobe_dirs,
                                                        const float* __restrict__ lobe_sigmas,
                                                        const float* __restrict__ light_values,
                                                        const float* __restrict__ light_pts,
                                                        const float* __restrict__ prim_pts,
                                                        const int* __restrict__ n_lights,
                                                        float* __restrict__ integral, int D, int L, Compose cz) {
  __shared__ float s_lp[kLightChunk * 3];
  __shared__ float s_lv[kLightChunk * 3];
  const int n = blockIdx.y;
  const int d = blockIdx.x * kBlock + threadIdx.x;
  const bool active = d < D;
  const size_t o = (size_t)n * D + (active ? d : 0);
  float3 dir = make_float3(0.f, 0.f, 0.f), pp = dir;
  float sigma = 1.f;
  if (active) {
    dir = make_float3(lobe_dirs[3 * o], lobe_dirs[3 * o + 1], lobe_dirs[3 * o + 2]);
    pp = make_float3(prim_pts[3 * o], prim_pts[3 * o + 1], prim_pts[3 * o + 2]);
    sigma = lobe_sigmas[o];
    if (FUSED) { float len; dir = normalize_rn(dir, len); }
  }
  const int nL = min(n_lights[n], L);
  float3 sum = make_float3(0.f, 0.f, 0.f);
  for (int l0 = 0; l0 < nL; l0 += kLightChunk) {
    const int cnt = min(kLightChunk, nL - l0);
    __syncthreads();
    for (int i = threadIdx.x; i < cnt * 3; i += kBlock) {
      s_lp[i] = light_pts[((size_t)n * L + l0) * 3 + i];
      s_lv[i] = light_values[((size_t)n * L + l0) * 3 + i];
    }
    __syncthreads();
    if (FUSED && WT == 0) {
      const float inv_sigma = 1.f / sigma;
#pragma unroll 4
      for (int l = 0; l < cnt; ++l) {
        const float lx = s_lp[3 * l] - pp.x, ly = s_lp[3 * l + 1] - pp.y, lz = s_lp[3 * l + 2] - pp.z;
        const float rinv = rsqrt_approx(lx * lx + ly * ly + lz * lz);
        const float c = fminf(fmaxf((lx * dir.x + ly * dir.y + lz * dir.z) * rinv, -1.f), 1.f);
        const float a = fabsf(c);
        const float t = acos_as(c, a, 1.f - a) * inv_sigma;
        const float w = ex2_approx(-kHalfLog2e * (t * t));
        sum.x += s_lv[3 * l] * w; sum.y += s_lv[3 * l + 1] * w; sum.z += s_lv[3 * l + 2] * w;
      }
    } else {
#pragma unroll 4
    for (int l = 0; l < cnt; ++l) {
      float lx = s_lp[3 * l] - pp.x, ly = s_lp[3 * l + 1] - pp.y, lz = s_lp[3 * l + 2] - pp.z;
      const float len = sqrtf(lx * lx + ly * ly + lz * lz);
      lx /= len; ly /= len; lz /= len;
      const float cos_dot = fminf(fmaxf(lx * dir.x + ly * dir.y + lz * dir.z, -1.f), 1.f);
      float w;
      if (WT == 0) {
        const float angle = acosf(cos_dot);
        w = __expf(-0.5f * sq(angle / sigma)) / (sigma * SQRT2PI23);
      } else if (WT == 1) {
        const float angle = acosf(cos_dot);
        w = __expf(-0.5f * sq(angle / sigma));
      } else if (WT == 2) {
        w = __expf((cos_dot - 1.f) / sigma) / (sigma * TWOPI);
      } else {
        w = __expf((cos_dot - 1.f) / sigma);
      }
      sum.x += s_lv[3 * l] * w; sum.y += s_lv[3 * l + 1] * w; sum.z += s_lv[3 * l + 2] * w;
    }
    }
  }
  if (FUSED && WT == 0) {  // the hoisted 1 / (sigma K)
    const float norm = INVSQRT2PI23 / sigma;
    sum.x *= norm; sum.y *= norm; sum.z *= norm;
  }
  if (active && !FUSED) {
    integral[3 * o] = sum.x; integral[3 * o + 1] = sum.y; integral[3 * o + 2] = sum.z;
  }
  if (active && FUSED) {
    const float vis = cz.spec_vis[o];
    const float sp[3] = {sum.x * vis, sum.y * vis, sum.z * vis};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float pre = fmaxf(cz.diff_color[3 * o + c], 0.f) + sp[c];
      cz.color[3 * o + c] = pre >= 0.f ? pre : -0.f;
      if (cz.spec_color) cz.spec_color[3 * o + c] = sp[c];
    }
  }
}

template <int WT, bool LIGHT_GRAD, bool FUSED>
__global__ void __launch_bounds__(kBlock) sg_bwd_kernel(const float* __restrict__ lobe_dirs,
                                                        const float* __restrict__ lobe_sigmas,
                                                        const float* __restrict__ light_values,
                                                        const float* __restrict__ light_pts,
                                                        const float* __restrict__ prim_pts,
                                                        const int* __restrict__ n_lights,
                                                        const float* __restrict__ grad_integral,
                                                        float* __restrict__ grad_dirs,
                                                        float* __restrict__ grad_sigmas,
                                                        float* __restrict__ grad_light_values, int D, int L,
                                                        Compose cz) {
  __shared__ float s_lp[kLightChunk * 3];
  __shared__ float s_lv[kLightChunk * 3];
  __shared__ float s_gl[LIGHT_GRAD ? kLightChunk * 3 : 1];
  const int n = blockIdx.y;
  const int d = blockIdx.x * kBlock + threadIdx.x;
  const bool active = d < D;
  const size_t o = (size_t)n * D + (active ? d : 0);
  float3 dir = make_float3(0.f, 0.f, 0.f), pp = dir, gi = dir;
  float sigma = 1.f;
  float3 raw = dir, gsp = dir, integ = dir;  // fused: un-normalised direction, dL/d(spec_color), recomputed integral
  float rawlen = 1.f, vis = 0.f;
  if (active) {
    dir = make_float3(lobe_dirs[3 * o], lobe_dirs[3 * o + 1], lobe_dirs[3 * o + 2]);
    pp = make_float3(prim_pts[3 * o], prim_pts[3 * o + 1], prim_pts[3 * o + 2]);
    sigma = lobe_sigmas[o];
    if (!FUSED) {
      gi = make_float3(grad_integral[3 * o], grad_integral[3 * o + 1], grad_integral[3 * o + 2]);
    } else {
      raw = dir;
      dir = normalize_rn(raw, rawlen);
      vis = cz.spec_vis[o];
      float g[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float gpre = signbit(cz.color[3 * o + c]) ? 0.f : cz.g_color[3 * o + c];  // outer clamp(min=0)
        cz.g_diff[3 * o + c] = cz.diff_color[3 * o + c] >= 0.f ? gpre : 0.f;            // inner clamp(min=0)
        g[c] = gpre + (cz.g_spec_color ? cz.g_spec_color[3 * o + c] : 0.f);
      }
      gsp = make_float3(g[0], g[1], g[2]);
      gi = make_float3(g[0] * vis, g[1] * vis, g[2] * vis);
    }
  }
  const int nL = min(n_lights[n], L);
  float3 gdir = make_float3(0.f, 0.f, 0.f);
  float gsig = 0.f;
  for (int l0 = 0; l0 < nL; l0 += kLightChunk) {
    const int cnt = min(kLightChunk, nL - l0);
    __syncthreads();
    for (int i = threadIdx.x; i < cnt * 3; i += kBlock) {
      s_lp[i] = light_pts[((size_t)n * L + l0) * 3 + i];
      s_lv[i] = light_values[((size_t)n * L + l0) * 3 + i];
      if (LIGHT_GRAD) s_gl[i] = 0.f;
    }
    __syncthreads();
    if (FUSED && WT == 0 && !LIGHT_GRAD) {
      // un-normalised accumulators: gsig_un = sum dLw ev (t^2 - 1), gdir_un = sum dLw ev t rs rinv l, integ_un = sum e ev
      // (t = angle / sigma, rs = 1 / sqrt(1 - c^2)); the factors K^-1 sigma^-2 and K^-1 sigma^-1 are applied after the loop
      const float inv_sigma = 1.f / sigma;
#pragma unroll 4
      for (int l = 0; l < cnt; ++l) {
        const float lx = s_lp[3 * l] - pp.x, ly = s_lp[3 * l + 1] - pp.y, lz = s_lp[3 * l + 2] - pp.z;
        const float e0 = s_lv[3 * l], e1 = s_lv[3 * l + 1], e2 = s_lv[3 * l + 2];
        const float rinv = rsqrt_approx(lx * lx + ly * ly + lz * lz);
        const float cu = (lx * dir.x + ly * dir.y + lz * dir.z) * rinv;
        const float c = fminf(fmaxf(cu, -1.f), 1.f);
        const float a = fabsf(c), s1 = 1.f - a;
        const float t = acos_as(c, a, s1) * inv_sigma;
        const float t2 = t * t;
        const float ev = ex2_approx(-kHalfLog2e * t2);
        const float dLw = (gi.x * e0 + gi.y * e1 + gi.z * e2) * ev;
        gsig += dLw * (t2 - 1.f);
        // d angle / d cos = -1 / sqrt(1 - c^2) inside (-1, 1); the reference's -20 at the clamp edges (sg.cu:129)
        const float rs = (fabsf(cu) < 1.f) ? rsqrt_approx(s1 * (1.f + a)) : 20.f;
        const float k = dLw * t * rs * rinv;
        gdir.x += k * lx; gdir.y += k * ly; gdir.z += k * lz;
        integ.x += e0 * ev; integ.y += e1 * ev; integ.z += e2 * ev;
      }
    } else {
#pragma unroll 2
    for (int l = 0; l < cnt; ++l) {
      float lx = s_lp[3 * l] - pp.x, ly = s_lp[3 * l + 1] - pp.y, lz = s_lp[3 * l + 2] - pp.z;
      const float len = sqrtf(lx * lx + ly * ly + lz * lz);
      lx /= len; ly /= len; lz /= len;
      const float e0 = s_lv[3 * l], e1 = s_lv[3 * l + 1], e2 = s_lv[3 * l + 2];
      const float cos_dot = lx * dir.x + ly * dir.y + lz * dir.z;
      const float cc = fminf(fmaxf(cos_dot, -1.f), 1.f);
      const float dLw = gi.x * e0 + gi.y * e1 + gi.z * e2;
      float weight, dL_cos;
      if (WT == 0) {
        const float angle = acosf(cc);
        const float ev = __expf(-0.5f * sq(angle / sigma));
        weight = ev / (sigma * SQRT2PI23);
        gsig += dLw * ((ev * INVSQRT2PI23 * (sq(angle) - sq(sigma))) / (sq(sigma) * sq(sigma)));
        const float dL_angle = dLw * -((INVSQRT2PI23 * angle * ev) / (sq(sigma) * sigma));
        dL_cos = dL_angle * ((cos_dot > -1.f && cos_dot < 1.f) ? (-1.f / sqrtf(1.f - sq(cos_dot))) : -20.f);
      } else if (WT == 1) {
        const float angle = acosf(cc);
        const float ev = __expf(-0.5f * sq(angle / sigma));
        weight = ev;
        gsig += dLw * ((ev * sq(angle)) / (sigma * sq(sigma)));
        const float dL_angle = dLw * -((angle * ev) / sq(sigma));
        dL_cos = dL_angle * ((cos_dot > -1.f && cos_dot < 1.f) ? (-1.f / sqrtf(1.f - sq(cos_dot))) : -20.f);
      } else if (WT == 2) {
        const float ev = __expf((cc - 1.f) / sigma);
        weight = ev / (sigma * TWOPI);
        gsig += dLw * ((ev * INV2PI * ((1.f - cc) - sigma)) / (sigma * sq(sigma)));
        dL_cos = dLw * INV2PI * ev / sq(sigma);
      } else {
        const float ev = __expf((cc - 1.f) / sigma);
        weight = ev;
        gsig += dLw * ((ev * (1.f - cc) / sq(sigma)));
        dL_cos = dLw * ev / sigma;
      }
      gdir.x += dL_cos * lx; gdir.y += dL_cos * ly; gdir.z += dL_cos * lz;
      if (FUSED) { integ.x += e0 * weight; integ.y += e1 * weight; integ.z += e2 * weight; }
      if (LIGHT_GRAD) {
        const float wa = active ? weight : 0.f;
        const float r0 = gb::warp_sum(gi.x * wa), r1 = gb::warp_sum(gi.y * wa), r2 = gb::warp_sum(gi.z * wa);
        if (gb::lane_id() == 0) {
          atomicAdd(&s_gl[3 * l], r0); atomicAdd(&s_gl[3 * l + 1], r1); atomicAdd(&s_gl[3 * l + 2], r2);
        }
      }
    }
    }
    if (LIGHT_GRAD) {
      __syncthreads();
      for (int i = threadIdx.x; i < cnt * 3; i += kBlock)
        gb::red_add(grad_light_values + ((size_t)n * L + l0) * 3 + i, s_gl[i]);
    }
  }
  if (FUSED && WT == 0 && !LIGHT_GRAD) {  // the hoisted factors of the regrouped loop
    const float inv_sigma = 1.f / sigma;
    const float fw = INVSQRT2PI23 * inv_sigma, fg = fw * inv_sigma;
    gsig *= fg;
    gdir.x *= fg; gdir.y *= fg; gdir.z *= fg;
    integ.x *= fw; integ.y *= fw; integ.z *= fw;
  }
  if (active) {
    grad_sigmas[o] = gsig;
    if (FUSED) {
      cz.g_vis[o] = gsp.x * integ.x + gsp.y * integ.y + gsp.z * integ.z;
      // backward of x / max(|x|, eps): (g - n (n . g)) / |x| on the regular branch, g / eps below it
      const float nd = dir.x * gdir.x + dir.y * gdir.y + dir.z * gdir.z;
      const bool regular = rawlen > 1e-12f;
      gdir = regular ? make_float3(__fdiv_rn(gdir.x - dir.x * nd, rawlen), __fdiv_rn(gdir.y - dir.y * nd, rawlen),
                                   __fdiv_rn(gdir.z - dir.z * nd, rawlen))
                     : make_float3(gdir.x * 1e12f, gdir.y * 1e12f, gdir.z * 1e12f);
    }
    grad_dirs[3 * o] = gdir.x; grad_dirs[3 * o + 1] = gdir.y; grad_dirs[3 * o + 2] = gdir.z;
  }
}

}  // namespace

// reference binding replaced: sgutilslib.evaluate_gaussian_fwd (extensions/sgutils/sg.cu:177-224)
GB_API int gb_sg_evaluate_fwd(const float* lobe_dirs, const float* lobe_sigmas, const float* light_values,
                              const float* light_pts, const float* prim_pts, const int32_t* n_lights,
                              float* integral, int N, int D, int L, int w_type, void* stream) {
  if (N <= 0 || D <= 0) return 0;
  if (w_type < 0 || w_type > 3) return (int)cudaErrorInvalidValue;
  dim3 grid(gb::cdiv(D, kBlock), N);
  cudaStream_t s = (cudaStream_t)stream;
#define GB_SG_FWD(WT)                                                                                                  \
  GB_CUDA(gb::launch<sg_fwd_kernel<WT, false>>(grid, kBlock, 0, s, lobe_dirs, lobe_sigmas, light_values, light_pts,    \
                                               prim_pts, n_lights, integral, D, L, Compose{}))
  switch (w_type) {
    case 0: GB_SG_FWD(0); break;
    case 1: GB_SG_FWD(1); break;
    case 2: GB_SG_FWD(2); break;
    default: GB_SG_FWD(3); break;
  }
#undef GB_SG_FWD
  return 0;
}

// reference binding replaced: sgutilslib.evaluate_gaussian_bwd (extensions/sgutils/sg.cu:226-277).
// grad_dirs / grad_sigmas are overwritten; grad_light_values (nullable) is accumulated into (caller zeroes it).
GB_API int gb_sg_evaluate_bwd(const float* lobe_dirs, const float* lobe_sigmas, const float* light_values,
                              const float* light_pts, const float* prim_pts, const int32_t* n_lights,
                              const float* grad_integral, float* grad_dirs, float* grad_sigmas,
                              float* grad_light_values, int N, int D, int L, int w_type, void* stream) {
  if (N <= 0 || D <= 0) return 0;
  if (w_type < 0 || w_type > 3) return (int)cudaErrorInvalidValue;
  dim3 grid(gb::cdiv(D, kBlock), N);
  cudaStream_t s = (cudaStream_t)stream;
#define GB_SG_BWD(WT, LG)                                                                                              \
  GB_CUDA(gb::launch<sg_bwd_kernel<WT, LG, false>>(grid, kBlock, 0, s, lobe_dirs, lobe_sigmas, light_values,           \
                                                   light_pts, prim_pts, n_lights, grad_integral, grad_dirs,            \
                                                   grad_sigmas, grad_light_values, D, L, Compose{}))
  if (grad_light_values) {
    switch (w_type) {
      case 0: GB_SG_BWD(0, true); break;
      case 1: GB_SG_BWD(1, true); break;
      case 2: GB_SG_BWD(2, true); break;
      default: GB_SG_BWD(3, true); break;
    }
  } else {
    switch (w_type) {
      case 0: GB_SG_BWD(0, false); break;
      case 1: GB_SG_BWD(1, false); break;
      case 2: GB_SG_BWD(2, false); break;
      default: GB_SG_BWD(3, false); break;
    }
  }
#undef GB_SG_BWD
  return 0;
}

// Fused shade + compose (rgca.py:557-575 with sgutils.py:74-75 folded in): lobe_dirs are the UN-normalised reflection
// directions, diff_color [N,D,3], spec_vis [N,D]; color [N,D,3] = clamp(clamp(diff,0) + integral*spec_vis, 0) (sign bit
// keeps the pre-clamp sign for the backward), spec_color [N,D,3] optional (NULL to skip).
GB_API int gb_sg_shade_compose_fwd(const float* lobe_dirs, const float* lobe_sigmas, const float* light_values,
                                   const float* light_pts, const float* prim_pts, const int32_t* n_lights,
                                   const float* diff_color, const float* spec_vis, float* color, float* spec_color,
                                   int N, int D, int L, int w_type, void* stream) {
  if (N <= 0 || D <= 0) return 0;
  if (w_type < 0 || w_type > 3) return (int)cudaErrorInvalidValue;
  dim3 grid(gb::cdiv(D, kBlock), N);
  cudaStream_t s = (cudaStream_t)stream;
  Compose cz{};
  cz.diff_color = diff_color; cz.spec_vis = spec_vis; cz.color = color; cz.spec_color = spec_color;
#define GB_SG_FWD(WT)                                                                                                  \
  GB_CUDA(gb::launch<sg_fwd_kernel<WT, true>>(grid, kBlock, 0, s, lobe_dirs, lobe_sigmas, light_values, light_pts,     \
                                              prim_pts, n_lights, nullptr, D, L, cz))
  switch (w_type) {
    case 0: GB_SG_FWD(0); break;
    case 1: GB_SG_FWD(1); break;
    case 2: GB_SG_FWD(2); break;
    default: GB_SG_FWD(3); break;
  }
#undef GB_SG_FWD
  return 0;
}

// Backward of the above.  color is the forward's output (unmodified), g_color [N,D,3], g_spec_color [N,D,3] or NULL;
// writes g_dirs [N,D,3] (w.r.t. the un-normalised directions), g_sigmas [N,D], g_diff [N,D,3], g_vis [N,D];
// g_light_values (nullable) is accumulated into (caller zeroes it).
GB_API int gb_sg_shade_compose_bwd(const float* lobe_dirs, const float* lobe_sigmas, const float* light_values,
                                   const float* light_pts, const float* prim_pts, const int32_t* n_lights,
                                   const float* diff_color, const float* spec_vis, const float* color,
                                   const float* g_color, const float* g_spec_color, float* g_dirs, float* g_sigmas,
                                   float* g_diff, float* g_vis, float* g_light_values, int N, int D, int L, int w_type,
                                   void* stream) {
  if (N <= 0 || D <= 0) return 0;
  if (w_type < 0 || w_type > 3) return (int)cudaErrorInvalidValue;
  dim3 grid(gb::cdiv(D, kBlock), N);
  cudaStream_t s = (cudaStream_t)stream;
  Compose cz{};
  cz.diff_color = diff_color; cz.spec_vis = spec_vis; cz.color = const_cast<float*>(color);
  cz.g_color = g_color; cz.g_spec_color = g_spec_color; cz.g_diff = g_diff; cz.g_vis = g_vis;
#define GB_SG_BWD(WT, LG)                                                                                              \
  GB_CUDA(gb::launch<sg_bwd_kernel<WT, LG, true>>(grid, kBlock, 0, s, lobe_dirs, lobe_sigmas, light_values,            \
                                                  light_pts, prim_pts, n_lights, nullptr, g_dirs, g_sigmas,            \
                                                  g_light_values, D, L, cz))
  if (g_light_values) {
    switch (w_type) {
      case 0: GB_SG_BWD(0, true); break;
      case 1: GB_SG_BWD(1, true); break;
      case 2: GB_SG_BWD(2, true); break;
      default: GB_SG_BWD(3, true); break;
    }
  } else {
    switch (w_type) {
      case 0: GB_SG_BWD(0, false); break;
      case 1: GB_SG_BWD(1, false); break;
      case 2: GB_SG_BWD(2, false); break;
      default: GB_SG_BWD(3, false); break;
    }
  }
#undef GB_SG_BWD
  return 0;
}
