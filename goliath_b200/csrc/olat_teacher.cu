// goliath_b200/csrc/olat_teacher.cu — per-texel OLAT features and the OLAT compose of the relightable hand teacher
// (hand_teacher_mvp.py:359-493, OLATRGBDecoder.forward_rgb), sm_90a.
//
// Features: one pass writes the U-Net input [B*L, 7Z, U, U] in its NCHW channel order (light vector Z*3, view
// direction Z*3, 1 - shadow Z) from the primitive transforms and the raw splat volume of gb_mvp_shadow_march, and the
// chunk's light mean of the shadow into primshadow.  The reference computes these under no_grad: there is no backward.
// Compose: rgb = sum_l s * relu(25 t + 100) * I over the decoder's [B, L, Z, 4, U, U] output, forward and backward.
//
// Compiled without fast-math: the shadow normalisation, F.normalize and the sigmoid keep IEEE division / sqrt / exp.
#include "common.cuh"

namespace {

// torch.linspace(-1, 1, n)[i] (the two-sided formula of torch's linspace kernel)
__device__ __forceinline__ float lin11(int i, int n) {
  if (n == 1) return -1.f;
  const float step = 2.f / (float)(n - 1);
  return i < n / 2 ? -1.f + step * (float)i : 1.f - step * (float)(n - 1 - i);
}

// F.normalize(v, dim) = v / max(|v|, 1e-12)
__device__ __forceinline__ float3 normalize3(float3 v) {
  const float n = fmaxf(sqrtf(v.x * v.x + v.y * v.y + v.z * v.z), 1e-12f);
  return make_float3(v.x / n, v.y / n, v.z / n);
}

// One thread per (item b, depth slice z, texel u, v), looping over the chunk's L lights.  Texel (u, v) lies in
// primitive k = (u / TH) * (U / TW) + v / TW at in-primitive (y', x') = (u % TH, v % TW).
//
// Index arithmetic of hand_teacher_mvp.py:379-401, as written there: the stack of meshgrid([intervz, intervy,
// intervx]) is transposed (1, 3) and flattened, so flat index f = xi*(TH*TD) + yi*TD + zi carries the local point
// (intervz[zi], intervy[yi], intervx[xi]); `.view(B, ny, nx, 3, TD, TH, TW)` then re-reads f as (z', y', x') with
// f = z'*(TH*TW) + y'*TW + x'.  So the texel (z', u, v) of primitive k uses
//     f  = z'*TH*TW + y'*TW + x',  xi = f / (TH*TD),  yi = (f / TD) % TH,  zi = f % TD,
//     q  = (lin(zi, TD), lin(yi, TH), lin(xi, TW)) / primscale[k]          (component-wise)
//     p  = volradius * (primpos[k] + primrot[k] q)                         (world point)
//     light = valid[k] * primrot[k]^T normalize(light_pos[b, l] - p)     channels  3z' + c
//     view  = valid[k] * primrot[k]^T normalize(campos[b] - p)           channels  3Z + 3z' + c
//     1 - shadow[b*L + l, k, z', y', x', 0] / (shadow[.., 1] + 1e-5)      channel   6Z + z'
// the shadow in its true (TD, TH, TW) layout (hand_teacher_mvp.py:359-377).
__global__ void __launch_bounds__(256) olat_features_kernel(
    int B, int L, int K, int TD, int TH, int TW, int U, float volradius, const float* __restrict__ primpos,
    const float* __restrict__ primrot, const float* __restrict__ primscale, const float* __restrict__ valid,
    const float* __restrict__ light_pos, const float* __restrict__ campos, const float2* __restrict__ shadow,
    float* __restrict__ feat, float* __restrict__ primshadow, int accumulate, float* __restrict__ shadow_feat) {
  const size_t UU = (size_t)U * U;
  const size_t total = (size_t)B * TD * UU;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t uv = idx % UU;
    const int z = (int)((idx / UU) % TD), b = (int)(idx / (UU * TD));
    const int u = (int)(uv / U), v = (int)(uv % U);
    const int nx = U / TW;
    const int hy = u / TH, yl = u % TH, wx = v / TW, xl = v % TW;
    const int k = hy * nx + wx;
    const int f = (z * TH + yl) * TW + xl;
    const int xi = f / (TH * TD), yi = (f / TD) % TH, zi = f % TD;
    const size_t bk = (size_t)b * K + k;
    const float* R = primrot + bk * 9;
    const float3 sc = make_float3(primscale[bk * 3], primscale[bk * 3 + 1], primscale[bk * 3 + 2]);
    const float3 q = make_float3(lin11(zi, TD) / sc.x, lin11(yi, TH) / sc.y, lin11(xi, TW) / sc.z);
    const float3 rq = make_float3(R[0] * q.x + R[1] * q.y + R[2] * q.z, R[3] * q.x + R[4] * q.y + R[5] * q.z,
                                  R[6] * q.x + R[7] * q.y + R[8] * q.z);
    const float3 p = make_float3(volradius * (primpos[bk * 3] + rq.x), volradius * (primpos[bk * 3 + 1] + rq.y),
                                 volradius * (primpos[bk * 3 + 2] + rq.z));
    const float vk = valid ? valid[k] : 1.f;
    // R^T d: out_f = sum_e R[e][f] d_e (einsum "bhwef,...e...->...f...")
    auto rot_t = [&](float3 d) {
      return make_float3(vk * (R[0] * d.x + R[3] * d.y + R[6] * d.z), vk * (R[1] * d.x + R[4] * d.y + R[7] * d.z),
                         vk * (R[2] * d.x + R[5] * d.y + R[8] * d.z));
    };
    const float3 vd = rot_t(normalize3(make_float3(campos[3 * b] - p.x, campos[3 * b + 1] - p.y, campos[3 * b + 2] - p.z)));
    const size_t tsz = (size_t)TD * TH * TW;
    float ssum = 0.f;
    for (int l = 0; l < L; ++l) {
      const size_t n = (size_t)b * L + l;
      const float* lp = light_pos + n * 3;
      const float3 ld = rot_t(normalize3(make_float3(lp[0] - p.x, lp[1] - p.y, lp[2] - p.z)));
      float* o = feat + n * 7 * TD * UU + uv;
      o[(size_t)(3 * z + 0) * UU] = ld.x;
      o[(size_t)(3 * z + 1) * UU] = ld.y;
      o[(size_t)(3 * z + 2) * UU] = ld.z;
      o[(size_t)(3 * TD + 3 * z + 0) * UU] = vd.x;
      o[(size_t)(3 * TD + 3 * z + 1) * UU] = vd.y;
      o[(size_t)(3 * TD + 3 * z + 2) * UU] = vd.z;
      const float2 sv = shadow[(n * K + k) * tsz + ((size_t)z * TH + yl) * TW + xl];
      const float sf = sv.x / (sv.y + 1e-5f);
      o[(size_t)(6 * TD + z) * UU] = 1.f - sf;
      if (shadow_feat) shadow_feat[(n * TD + z) * UU + uv] = sf;
      ssum += sf;
    }
    const float mean = ssum / (float)L;
    float* ps = primshadow + ((size_t)b * TD + z) * 3 * UU + uv;
#pragma unroll
    for (int c = 0; c < 3; ++c) ps[c * UU] = accumulate ? ps[c * UU] + mean : mean;
  }
}

// tex [B*L, 4Z, U, U] read as [B, L, Z, 4, U, U]; s = sigmoid(t0), or the shadow feature [B*L, Z, U, U] when given.
// One thread per (b, z, texel), summing the L lights in order.
__global__ void __launch_bounds__(256) olat_compose_fwd_kernel(int B, int L, int Z, int U,
                                                               const float* __restrict__ tex,
                                                               const float* __restrict__ intensity,
                                                               const float* __restrict__ shadow_feat,
                                                               float* __restrict__ rgb, int accumulate,
                                                               float* __restrict__ texolat) {
  const size_t UU = (size_t)U * U;
  const size_t total = (size_t)B * Z * UU;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t uv = idx % UU;
    const int z = (int)((idx / UU) % Z), b = (int)(idx / (UU * Z));
    float acc[3] = {0.f, 0.f, 0.f};
    for (int l = 0; l < L; ++l) {
      const size_t n = (size_t)b * L + l;
      const float* t = tex + (n * Z + z) * 4 * UU + uv;
      const float s = shadow_feat ? shadow_feat[(n * Z + z) * UU + uv] : 1.f / (1.f + expf(-t[0]));
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float to = 25.f * t[(c + 1) * UU] + 100.f;
        if (texolat) texolat[((n * Z + z) * 3 + c) * UU + uv] = to;
        acc[c] += s * fmaxf(to, 0.f) * intensity[n * 3 + c];
      }
    }
    float* o = rgb + ((size_t)b * Z + z) * 3 * UU + uv;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c * UU] = accumulate ? o[c * UU] + acc[c] : acc[c];
  }
}

// d rgb / d tex plus, when g_texolat is given, 25 g_texolat; t0 gets no gradient when the shadow feature stands in
// for the sigmoid.
__global__ void __launch_bounds__(256) olat_compose_bwd_kernel(int B, int L, int Z, int U,
                                                               const float* __restrict__ tex,
                                                               const float* __restrict__ intensity,
                                                               const float* __restrict__ shadow_feat,
                                                               const float* __restrict__ g_rgb,
                                                               const float* __restrict__ g_texolat,
                                                               float* __restrict__ g_tex) {
  const size_t UU = (size_t)U * U;
  const size_t total = (size_t)B * Z * UU;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t uv = idx % UU;
    const int z = (int)((idx / UU) % Z), b = (int)(idx / (UU * Z));
    const float* gr = g_rgb + ((size_t)b * Z + z) * 3 * UU + uv;
    const float g[3] = {gr[0], gr[UU], gr[2 * UU]};
    for (int l = 0; l < L; ++l) {
      const size_t n = (size_t)b * L + l;
      const float* t = tex + (n * Z + z) * 4 * UU + uv;
      float* gt = g_tex + (n * Z + z) * 4 * UU + uv;
      const float s = shadow_feat ? shadow_feat[(n * Z + z) * UU + uv] : 1.f / (1.f + expf(-t[0]));
      float gs = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float to = 25.f * t[(c + 1) * UU] + 100.f;
        const float gi = g[c] * intensity[n * 3 + c];
        float gto = to > 0.f ? gi * s : 0.f;
        if (g_texolat) gto += g_texolat[((n * Z + z) * 3 + c) * UU + uv];
        gt[(c + 1) * UU] = 25.f * gto;
        gs += gi * fmaxf(to, 0.f);
      }
      gt[0] = shadow_feat ? 0.f : gs * (1.f - s) * s;
    }
  }
}

int grid_for(size_t total) { return (int)min((total + 255) / 256, (size_t)gb::kNumSMs * 16); }

}  // namespace

// replaces the no_grad feature block of OLATRGBDecoder.forward_rgb (hand_teacher_mvp.py:359-439): see the kernel
// comment for the per-texel formula.  primpos / primrot / primscale [B,K,3] / [B,K,3,3] / [B,K,3] (world units),
// valid [K] or NULL, light_pos [B,L,3], campos [B,3], shadow [B*L,K,TD,TH,TW,2] (gb_mvp_shadow_march).  Writes
// feat [B*L,7*TD,U,U], primshadow [B,TD,3,U,U] (+= the light mean when accumulate, else =), and shadow_feat
// [B*L,TD,U,U] when not NULL.
GB_API int gb_olat_features(int B, int L, int K, int TD, int TH, int TW, int U, float volradius, const float* primpos,
                            const float* primrot, const float* primscale, const float* valid, const float* light_pos,
                            const float* campos, const float* shadow, float* feat, float* primshadow, int accumulate,
                            float* shadow_feat, void* stream) {
  if (B <= 0 || L <= 0 || U <= 0) return 0;
  if (TD < 1 || TH < 1 || TW < 1 || U % TW || U % TH || (U / TW) * (U / TH) != K) return (int)cudaErrorInvalidValue;
  const size_t total = (size_t)B * TD * U * U;
  return gb::launch<olat_features_kernel>(grid_for(total), 256, 0, (cudaStream_t)stream,
      B, L, K, TD, TH, TW, U, volradius, primpos, primrot, primscale, valid, light_pos, campos, (const float2*)shadow,
      feat, primshadow, accumulate, shadow_feat);
}

// replaces the compose of OLATRGBDecoder.forward_rgb (hand_teacher_mvp.py:468-479): tex [B*L,4Z,U,U], intensity
// [B,L,3], shadow_feat [B*L,Z,U,U] (training warm-up) or NULL (sigmoid of channel 0).  rgb [B,Z,3,U,U] (+= when
// accumulate, else =); texolat [B,L,Z,3,U,U] = 25 tex[..., 1:] + 100 when not NULL.
GB_API int gb_olat_compose_fwd(int B, int L, int Z, int U, const float* tex, const float* intensity,
                               const float* shadow_feat, float* rgb, int accumulate, float* texolat, void* stream) {
  if (B <= 0 || L <= 0 || Z <= 0 || U <= 0) return 0;
  const size_t total = (size_t)B * Z * U * U;
  return gb::launch<olat_compose_fwd_kernel>(grid_for(total), 256, 0, (cudaStream_t)stream, B, L, Z, U, tex, intensity,
                                             shadow_feat, rgb, accumulate, texolat);
}

// gradient of gb_olat_compose_fwd w.r.t. tex: g_tex [B*L,4Z,U,U] (written) from g_rgb [B,Z,3,U,U] and g_texolat
// [B,L,Z,3,U,U] or NULL.
GB_API int gb_olat_compose_bwd(int B, int L, int Z, int U, const float* tex, const float* intensity,
                               const float* shadow_feat, const float* g_rgb, const float* g_texolat, float* g_tex,
                               void* stream) {
  if (B <= 0 || L <= 0 || Z <= 0 || U <= 0) return 0;
  const size_t total = (size_t)B * Z * U * U;
  return gb::launch<olat_compose_bwd_kernel>(grid_for(total), 256, 0, (cudaStream_t)stream, B, L, Z, U, tex, intensity,
                                             shadow_feat, g_rgb, g_texolat, g_tex);
}
