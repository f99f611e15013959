// goliath_b200/csrc/envmap_spec.cu — environment-map specular branch of the RGCA PrimDecoder (sm_90a).
//
// Replaces /root/reference/ca_code/models/rgca.py:548-556 (run_vis_relight.py's second loop, EnvSpinDecorator):
//   ref_dirs = einsum("bxy,bny->bnx", lightrot, ref_dirs)                       rotate the reflection vector
//   ref_uv   = dir2uv(ref_dirs)            (ca_code/utils/envmap.py:284-292)     u = atan2(x,z)/pi, v = 2 acos(y)/pi - 1
//   spec     = mipmap_grid_sample(preconv_envmap, ref_uv, sigma * 5)            (ca_code/utils/mipmap_sampler.py:13-66)
//   spec     = spec.clamp(max=1) * spec_vis
// i.e. per Gaussian two bilinear texture fetches (border padding, align_corners=False) from adjacent levels of a
// pre-convolved mip pyramid, blended by the fractional level.  The eager formulation samples EVERY level for every
// Gaussian (q grid_sample launches + stack + gather + lerp, ~q * 12 B * G of temporaries); here one thread per
// Gaussian touches 8 texels per channel and writes 12 bytes.  HBM/L2 gather kernel: 40 B in, 12 B out per Gaussian
// plus the texel reads (the pyramid, 8 MB at 512x1024, stays in L2).
//
// Backward: gradients to ref_dirs (through the rotation, dir2uv and the bilinear weights; zero where the border
// clip is active, as grid_sample does) and to spec_vis.  The mip level is computed under no_grad upstream, so sigma
// receives none; the environment map itself is a constant of the relighting loop (no gradient is produced for it).
#include "envmap_common.cuh"

namespace {

constexpr int kMaxLevels = 8;
constexpr float kInvPi = 0.31830988618379067154f;

struct EnvArgs {
  int B, G, q;
  const float* level[kMaxLevels];  // [B,3,H_l,W_l] each
  int H[kMaxLevels], W[kMaxLevels];
  const float *ref_dirs, *sigma, *spec_vis, *lightrot;  // [B,G,3] [B,G] [B,G] [B,3,3]
  float level_scale;                                    // miplevel = sigma * level_scale (5 upstream)
  float* spec;                                          // [B,G,3]
  const float* g_spec;
  float *g_ref_dirs, *g_spec_vis;
};

using gb::Bilin;
using gb::fetch;
using gb::locate;

__device__ __forceinline__ float lerp_torch(float s, float e, float w) {  // th.lerp's two-sided formula
  return (w < 0.5f) ? s + w * (e - s) : e - (e - s) * (1.f - w);
}

template <bool BWD>
__global__ void __launch_bounds__(256) envmap_spec_kernel(EnvArgs a) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (g >= a.G) return;
  const size_t o = (size_t)b * a.G + g;
  const float* R = a.lightrot + 9 * b;
  const float r0 = a.ref_dirs[3 * o], r1 = a.ref_dirs[3 * o + 1], r2 = a.ref_dirs[3 * o + 2];
  const float x = R[0] * r0 + R[1] * r1 + R[2] * r2;
  const float y = R[3] * r0 + R[4] * r1 + R[5] * r2;
  const float z = R[6] * r0 + R[7] * r1 + R[8] * r2;
  const float u = kInvPi * atan2f(x, z);
  const float yc = fminf(fmaxf(y, -1.f), 1.f);
  const float v = 2.f * kInvPi * acosf(yc) - 1.f;
  float lam = fminf(fmaxf(a.sigma[o] * a.level_scale, 0.f), (float)(a.q - 1) - 1e-6f);
  if (a.q == 1) lam = 0.f;
  const int d1 = (int)floorf(lam);
  const float w = lam - (float)d1;
  const int d2 = min(d1 + 1, a.q - 1);
  const Bilin b1 = locate(u, v, a.W[d1], a.H[d1]);
  const Bilin b2 = locate(u, v, a.W[d2], a.H[d2]);
  const size_t plane1 = (size_t)a.H[d1] * a.W[d1], plane2 = (size_t)a.H[d2] * a.W[d2];
  const float* L1 = a.level[d1] + (size_t)b * 3 * plane1;
  const float* L2 = a.level[d2] + (size_t)b * 3 * plane2;
  const float vis = a.spec_vis[o];
  float gu = 0.f, gv = 0.f, gvis = 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float dx1, dy1, dx2, dy2;
    const float s1 = fetch(L1 + c * plane1, b1, a.W[d1], a.H[d1], dx1, dy1);
    const float s2 = (a.q == 1) ? s1 : fetch(L2 + c * plane2, b2, a.W[d2], a.H[d2], dx2, dy2);
    const float s = (a.q == 1) ? s1 : lerp_torch(s1, s2, w);
    const float sc = fminf(s, 1.f);
    if (!BWD) {
      a.spec[3 * o + c] = sc * vis;
    } else {
      const float gc = a.g_spec[3 * o + c];
      gvis += gc * sc;
      const float gs = (s <= 1.f) ? gc * vis : 0.f;  // clamp(max=1) passes the gradient where s <= 1
      const float g1 = (a.q == 1) ? gs : gs * (1.f - w), g2 = (a.q == 1) ? 0.f : gs * w;
      // d(ix)/du = W/2, d(iy)/dv = H/2, times the border-clip multipliers
      gu += g1 * dx1 * b1.mx * 0.5f * (float)a.W[d1];
      gv += g1 * dy1 * b1.my * 0.5f * (float)a.H[d1];
      if (a.q > 1) {
        gu += g2 * dx2 * b2.mx * 0.5f * (float)a.W[d2];
        gv += g2 * dy2 * b2.my * 0.5f * (float)a.H[d2];
      }
    }
  }
  if (BWD) {
    a.g_spec_vis[o] = gvis;
    // u = atan2(x, z) / pi: du/dx = z / (x^2 + z^2) / pi, du/dz = -x / (x^2 + z^2) / pi
    const float den = x * x + z * z;
    const float iu = den > 0.f ? kInvPi / den : 0.f;
    const float gx = gu * z * iu, gz = -gu * x * iu;
    // v = 2 acos(y) / pi - 1: dv/dy = -2 / (pi sqrt(1 - y^2))  (zero outside the clamp)
    const float om = 1.f - yc * yc;
    const float gy = (y > -1.f && y < 1.f && om > 0.f) ? -2.f * kInvPi * gv * rsqrtf(om) : 0.f;
    // r' = R r  ->  g_r = R^T g_r'
    a.g_ref_dirs[3 * o + 0] = R[0] * gx + R[3] * gy + R[6] * gz;
    a.g_ref_dirs[3 * o + 1] = R[1] * gx + R[4] * gy + R[7] * gz;
    a.g_ref_dirs[3 * o + 2] = R[2] * gx + R[5] * gy + R[8] * gz;
  }
}

int fill(EnvArgs& a, int B, int G, int q, const float* const* levels, const int32_t* level_hw) {
  if (q < 1 || q > kMaxLevels) return (int)cudaErrorInvalidValue;
  a.B = B; a.G = G; a.q = q;
  for (int i = 0; i < q; ++i) {
    a.level[i] = levels[i];
    a.H[i] = level_hw[2 * i];
    a.W[i] = level_hw[2 * i + 1];
    if (!levels[i] || a.H[i] < 1 || a.W[i] < 1) return (int)cudaErrorInvalidValue;
  }
  return 0;
}

}  // namespace

// levels: q host-side device pointers to [B,3,H_l,W_l] fp32 mip levels, level_hw: q (H, W) pairs (host memory).
// ref_dirs [B,G,3], sigma [B,G], spec_vis [B,G], lightrot [B,3,3] -> spec [B,G,3].
GB_API int gb_envmap_spec_fwd(int B, int G, int q, const float* const* levels, const int32_t* level_hw,
                              const float* ref_dirs, const float* sigma, const float* spec_vis, const float* lightrot,
                              float level_scale, float* spec, void* stream) {
  if (B <= 0 || G <= 0) return 0;
  EnvArgs a = {};
  const int e = fill(a, B, G, q, levels, level_hw);
  if (e) return e;
  a.ref_dirs = ref_dirs; a.sigma = sigma; a.spec_vis = spec_vis; a.lightrot = lightrot; a.level_scale = level_scale;
  a.spec = spec;
  return gb::launch<envmap_spec_kernel<false>>(dim3(gb::cdiv(G, 256), B), 256, 0, (cudaStream_t)stream, a);
}

// g_spec [B,G,3] -> g_ref_dirs [B,G,3], g_spec_vis [B,G] (both overwritten).
GB_API int gb_envmap_spec_bwd(int B, int G, int q, const float* const* levels, const int32_t* level_hw,
                              const float* ref_dirs, const float* sigma, const float* spec_vis, const float* lightrot,
                              float level_scale, const float* g_spec, float* g_ref_dirs, float* g_spec_vis,
                              void* stream) {
  if (B <= 0 || G <= 0) return 0;
  EnvArgs a = {};
  const int e = fill(a, B, G, q, levels, level_hw);
  if (e) return e;
  a.ref_dirs = ref_dirs; a.sigma = sigma; a.spec_vis = spec_vis; a.lightrot = lightrot; a.level_scale = level_scale;
  a.g_spec = g_spec; a.g_ref_dirs = g_ref_dirs; a.g_spec_vis = g_spec_vis;
  return gb::launch<envmap_spec_kernel<true>>(dim3(gb::cdiv(G, 256), B), 256, 0, (cudaStream_t)stream, a);
}
