// goliath_b200/csrc/rgca_heads.cu — RGCA Gaussian heads + SH diffuse + reflection direction, fused (sm_90a).
//
// Replaces the ~60 eager element-wise PyTorch ops of PrimDecoder.forward,
// /root/reference/ca_code/models/rgca.py:506-546 (row R2 of SURVEY.md §8a; channel map SURVEY.md Appendix C),
// including the materialised [B,G,3,81] SH tensor (rgca.py:514,540; 1.02 GB per frame at G = 1024^2).
//
// One thread per texel / Gaussian g = y*W + x.  The decoder's outputs are read directly as NCHW planes
// (plane c of batch b at [b][c][g]: every load is a fully coalesced 128-byte warp request), the 3x81 light SH
// table of the batch item sits in shared memory, and the 13 per-Gaussian results are written once in the [B,G,*]
// layouts the rest of the path consumes.  An optional second light-SH table (the training-mode random back light of
// rgca.py:590-618) is evaluated in the same pass (shsum2 = diff_color_rand before the clamp).  Pure HBM kernel: 129 planes * 4 B + 36 B in, ~130 B out per Gaussian
// (~680 B vs ~5-6 KB of traffic in the eager formulation).  Backward mirrors it: one pass that writes the 129
// gradient planes coalesced.
#include "common.cuh"

namespace {

constexpr int kBlock = 128;
constexpr int NCOL = 16, NMONO = 65, NDIFF = 3 * NCOL + NMONO;  // 113
constexpr int NVN = NDIFF + 12;                                  // 125 planes in f_vnocond
constexpr float kEps = 1e-12f;                                   // F.normalize eps

struct HeadsArgs {
  int B, G;
  const float *f_vnocond, *f_vcond, *postex, *tn, *albedo, *light_sh, *campos;
  float scale_lo, scale_hi;
  // forward outputs
  float *primpos, *primqvec, *primscale, *primscale_preclip, *opacity, *sigma, *spec_vis, *spec_dnml, *spec_nml,
      *diff_color, *ref_dirs, *primnmlbase, *shsum;
  // backward: upstream gradients (any may be null) and results
  const float *g_primpos, *g_primqvec, *g_primscale, *g_primscale_preclip, *g_opacity, *g_sigma, *g_spec_vis,
      *g_spec_dnml, *g_spec_nml, *g_diff_color, *g_ref_dirs, *g_primnmlbase;
  float *g_f_vnocond, *g_f_vcond, *g_postex, *g_tn, *g_albedo;  // g_albedo [B,G,3] (summed over B by the caller)
  // optional second light-SH table [B,3,81] (training-mode random back light, rgca.py:590-618): its SH sums come out
  // of the same pass over the 113 diffuse planes (shsum2 [B,G,3], no albedo); g_shsum2 is their upstream gradient
  const float* light_sh2;
  float* shsum2;
  const float* g_shsum2;
};

__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }  // F.softplus
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ void st3(float* p, size_t i, float a, float b, float c) { p[3 * i] = a; p[3 * i + 1] = b; p[3 * i + 2] = c; }
__device__ __forceinline__ float3 ld3n(const float* p, size_t i) { return p ? make_float3(p[3 * i], p[3 * i + 1], p[3 * i + 2]) : make_float3(0.f, 0.f, 0.f); }

template <bool SECOND>
__global__ void __launch_bounds__(kBlock) heads_fwd_kernel(HeadsArgs a) {
  __shared__ float s_L[3 * 81];
  __shared__ float s_L2[SECOND ? 3 * 81 : 1];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < 243; i += kBlock) {
    s_L[i] = a.light_sh[(size_t)b * 243 + i];
    if (SECOND) s_L2[i] = a.light_sh2[(size_t)b * 243 + i];
  }
  __syncthreads();
  const int g = blockIdx.x * kBlock + threadIdx.x;
  if (g >= a.G) return;
  const size_t G = a.G;
  const float* fn = a.f_vnocond + (size_t)b * NVN * G + g;
  const float* fv = a.f_vcond + (size_t)b * 4 * G + g;
  const size_t o = (size_t)b * G + g;

  // ---- SH diffuse: S_c = sum_{k<16} sh[c*16+k] L[c][k] + sum_{16<=k<81} sh[48+k-16] L[c][k]
  float S[3] = {0.f, 0.f, 0.f}, S2[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
#pragma unroll 8
    for (int k = 0; k < NCOL; ++k) {
      const float v = fn[(size_t)(c * NCOL + k) * G];
      S[c] += v * s_L[c * 81 + k];
      if (SECOND) S2[c] += v * s_L2[c * 81 + k];
    }
  }
#pragma unroll 5
  for (int k = 0; k < NMONO; ++k) {
    const float v = fn[(size_t)(3 * NCOL + k) * G];
    S[0] += v * s_L[NCOL + k];
    S[1] += v * s_L[81 + NCOL + k];
    S[2] += v * s_L[162 + NCOL + k];
    if (SECOND) {
      S2[0] += v * s_L2[NCOL + k];
      S2[1] += v * s_L2[81 + NCOL + k];
      S2[2] += v * s_L2[162 + NCOL + k];
    }
  }
  if (SECOND) st3(a.shsum2, (size_t)b * G + g, S2[0], S2[1], S2[2]);
  const float al0 = a.albedo[3 * (size_t)g], al1 = a.albedo[3 * (size_t)g + 1], al2 = a.albedo[3 * (size_t)g + 2];
  st3(a.diff_color, o, al0 * S[0], al1 * S[1], al2 * S[2]);
  st3(a.shsum, o, S[0], S[1], S[2]);

  // ---- Gaussian parameters
  const float* fg = fn + (size_t)NDIFF * G;
  const float px = fg[0] + a.postex[((size_t)b * 3 + 0) * G + g];
  const float py = fg[G] + a.postex[((size_t)b * 3 + 1) * G + g];
  const float pz = fg[2 * G] + a.postex[((size_t)b * 3 + 2) * G + g];
  st3(a.primpos, o, px, py, pz);
  const float q0 = fg[3 * G], q1 = fg[4 * G], q2 = fg[5 * G], q3 = fg[6 * G];
  const float qi = 1.f / fmaxf(sqrtf(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3), kEps);
  reinterpret_cast<float4*>(a.primqvec)[o] = make_float4(q0 * qi, q1 * qi, q2 * qi, q3 * qi);
  const float s0 = softplus_f(fg[7 * G]), s1 = softplus_f(fg[8 * G]), s2 = softplus_f(fg[9 * G]);
  st3(a.primscale_preclip, o, s0, s1, s2);
  st3(a.primscale, o, fminf(fmaxf(s0, a.scale_lo), a.scale_hi), fminf(fmaxf(s1, a.scale_lo), a.scale_hi),
      fminf(fmaxf(s2, a.scale_lo), a.scale_hi));
  a.opacity[o] = sigmoid_f(fg[10 * G]);
  a.sigma[o] = fmaxf(expf(fg[11 * G]) * 0.1f, 0.01f);

  // ---- view-dependent part
  a.spec_vis[o] = sigmoid_f(fv[0]);
  const float d0 = fv[G], d1 = fv[2 * G], d2 = fv[3 * G];
  st3(a.spec_dnml, o, d0, d1, d2);
  const float t0 = a.tn[((size_t)b * 3 + 0) * G + g], t1 = a.tn[((size_t)b * 3 + 1) * G + g], t2 = a.tn[((size_t)b * 3 + 2) * G + g];
  st3(a.primnmlbase, o, t0, t1, t2);
  const float w0 = d0 + t0, w1 = d1 + t1, w2 = d2 + t2;
  const float wi = 1.f / fmaxf(sqrtf(w0 * w0 + w1 * w1 + w2 * w2), kEps);
  const float m0 = w0 * wi, m1 = w1 * wi, m2 = w2 * wi;
  st3(a.spec_nml, o, m0, m1, m2);
  const float u0 = px - a.campos[3 * b], u1 = py - a.campos[3 * b + 1], u2 = pz - a.campos[3 * b + 2];
  const float ui = 1.f / fmaxf(sqrtf(u0 * u0 + u1 * u1 + u2 * u2), kEps);
  const float v0 = u0 * ui, v1 = u1 * ui, v2 = u2 * ui;
  const float s = v0 * m0 + v1 * m1 + v2 * m2;
  st3(a.ref_dirs, o, v0 - 2.f * s * m0, v1 - 2.f * s * m1, v2 - 2.f * s * m2);
}

template <bool SECOND>
__global__ void __launch_bounds__(kBlock) heads_bwd_kernel(HeadsArgs a) {
  __shared__ float s_L[3 * 81];
  __shared__ float s_L2[SECOND ? 3 * 81 : 1];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < 243; i += kBlock) {
    s_L[i] = a.light_sh[(size_t)b * 243 + i];
    if (SECOND) s_L2[i] = a.light_sh2[(size_t)b * 243 + i];
  }
  __syncthreads();
  const int g = blockIdx.x * kBlock + threadIdx.x;
  if (g >= a.G) return;
  const size_t G = a.G;
  const float* fn = a.f_vnocond + (size_t)b * NVN * G + g;
  const float* fv = a.f_vcond + (size_t)b * 4 * G + g;
  float* gn = a.g_f_vnocond + (size_t)b * NVN * G + g;
  float* gv = a.g_f_vcond + (size_t)b * 4 * G + g;
  const size_t o = (size_t)b * G + g;

  // ---- diffuse: diff_c = albedo_c * S_c
  const float3 gdiff = ld3n(a.g_diff_color, o);
  const float al0 = a.albedo[3 * (size_t)g], al1 = a.albedo[3 * (size_t)g + 1], al2 = a.albedo[3 * (size_t)g + 2];
  const float S0 = a.shsum[3 * o], S1 = a.shsum[3 * o + 1], S2 = a.shsum[3 * o + 2];
  st3(a.g_albedo, o, gdiff.x * S0, gdiff.y * S1, gdiff.z * S2);
  const float gS[3] = {gdiff.x * al0, gdiff.y * al1, gdiff.z * al2};
  const float3 g2v = SECOND ? ld3n(a.g_shsum2, o) : make_float3(0.f, 0.f, 0.f);
  const float g2[3] = {g2v.x, g2v.y, g2v.z};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
#pragma unroll 8
    for (int k = 0; k < NCOL; ++k) {
      float v = gS[c] * s_L[c * 81 + k];
      if (SECOND) v += g2[c] * s_L2[c * 81 + k];
      gn[(size_t)(c * NCOL + k) * G] = v;
    }
  }
#pragma unroll 5
  for (int k = 0; k < NMONO; ++k) {
    float v = gS[0] * s_L[NCOL + k] + gS[1] * s_L[81 + NCOL + k] + gS[2] * s_L[162 + NCOL + k];
    if (SECOND) v += g2[0] * s_L2[NCOL + k] + g2[1] * s_L2[81 + NCOL + k] + g2[2] * s_L2[162 + NCOL + k];
    gn[(size_t)(3 * NCOL + k) * G] = v;
  }

  // ---- recompute the forward quantities needed below
  const float* fg = fn + (size_t)NDIFF * G;
  float* gg = gn + (size_t)NDIFF * G;
  const float px = fg[0] + a.postex[((size_t)b * 3 + 0) * G + g];
  const float py = fg[G] + a.postex[((size_t)b * 3 + 1) * G + g];
  const float pz = fg[2 * G] + a.postex[((size_t)b * 3 + 2) * G + g];
  const float d0 = fv[G], d1 = fv[2 * G], d2 = fv[3 * G];
  const float t0 = a.tn[((size_t)b * 3 + 0) * G + g], t1 = a.tn[((size_t)b * 3 + 1) * G + g], t2 = a.tn[((size_t)b * 3 + 2) * G + g];
  const float w0 = d0 + t0, w1 = d1 + t1, w2 = d2 + t2;
  const float wn = fmaxf(sqrtf(w0 * w0 + w1 * w1 + w2 * w2), kEps), wi = 1.f / wn;
  const float m0 = w0 * wi, m1 = w1 * wi, m2 = w2 * wi;
  const float u0 = px - a.campos[3 * b], u1 = py - a.campos[3 * b + 1], u2 = pz - a.campos[3 * b + 2];
  const float un = fmaxf(sqrtf(u0 * u0 + u1 * u1 + u2 * u2), kEps), ui = 1.f / un;
  const float v0 = u0 * ui, v1 = u1 * ui, v2 = u2 * ui;
  const float s = v0 * m0 + v1 * m1 + v2 * m2;

  // ---- reflection direction r = v - 2 (v.m) m
  const float3 gr = ld3n(a.g_ref_dirs, o);
  const float grm = gr.x * m0 + gr.y * m1 + gr.z * m2;
  float gvx = gr.x - 2.f * grm * m0, gvy = gr.y - 2.f * grm * m1, gvz = gr.z - 2.f * grm * m2;
  const float3 gmu = ld3n(a.g_spec_nml, o);
  float gm0 = gmu.x - 2.f * (grm * v0 + s * gr.x), gm1 = gmu.y - 2.f * (grm * v1 + s * gr.y), gm2 = gmu.z - 2.f * (grm * v2 + s * gr.z);
  // v = u / |u|
  const float vgv = v0 * gvx + v1 * gvy + v2 * gvz;
  const float gu0 = (gvx - v0 * vgv) * ui, gu1 = (gvy - v1 * vgv) * ui, gu2 = (gvz - v2 * vgv) * ui;
  const float3 gpp = ld3n(a.g_primpos, o);
  const float gp0 = gpp.x + gu0, gp1 = gpp.y + gu1, gp2 = gpp.z + gu2;
  gg[0] = gp0; gg[G] = gp1; gg[2 * G] = gp2;
  a.g_postex[((size_t)b * 3 + 0) * G + g] = gp0;
  a.g_postex[((size_t)b * 3 + 1) * G + g] = gp1;
  a.g_postex[((size_t)b * 3 + 2) * G + g] = gp2;
  // m = w / |w|
  const float mgm = m0 * gm0 + m1 * gm1 + m2 * gm2;
  const float gw0 = (gm0 - m0 * mgm) * wi, gw1 = (gm1 - m1 * mgm) * wi, gw2 = (gm2 - m2 * mgm) * wi;
  const float3 gdn = ld3n(a.g_spec_dnml, o);
  gv[G] = gw0 + gdn.x; gv[2 * G] = gw1 + gdn.y; gv[3 * G] = gw2 + gdn.z;
  const float3 gnb = ld3n(a.g_primnmlbase, o);
  a.g_tn[((size_t)b * 3 + 0) * G + g] = gw0 + gnb.x;
  a.g_tn[((size_t)b * 3 + 1) * G + g] = gw1 + gnb.y;
  a.g_tn[((size_t)b * 3 + 2) * G + g] = gw2 + gnb.z;
  // spec_vis = sigmoid
  {
    const float sv = sigmoid_f(fv[0]);
    gv[0] = (a.g_spec_vis ? a.g_spec_vis[o] : 0.f) * sv * (1.f - sv);
  }
  // quaternion: qv = q / |q|
  {
    const float q0 = fg[3 * G], q1 = fg[4 * G], q2 = fg[5 * G], q3 = fg[6 * G];
    const float qn = fmaxf(sqrtf(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3), kEps), qi = 1.f / qn;
    const float4 gq = a.g_primqvec ? reinterpret_cast<const float4*>(a.g_primqvec)[o] : make_float4(0.f, 0.f, 0.f, 0.f);
    const float n0 = q0 * qi, n1 = q1 * qi, n2 = q2 * qi, n3 = q3 * qi;
    const float dq = n0 * gq.x + n1 * gq.y + n2 * gq.z + n3 * gq.w;
    gg[3 * G] = (gq.x - n0 * dq) * qi; gg[4 * G] = (gq.y - n1 * dq) * qi;
    gg[5 * G] = (gq.z - n2 * dq) * qi; gg[6 * G] = (gq.w - n3 * dq) * qi;
  }
  // scales: pre = softplus(x); out = clamp(pre, lo, hi)
  {
    const float3 gpre = ld3n(a.g_primscale_preclip, o), gcl = ld3n(a.g_primscale, o);
    const float gpre_[3] = {gpre.x, gpre.y, gpre.z}, gcl_[3] = {gcl.x, gcl.y, gcl.z};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float x = fg[(size_t)(7 + c) * G];
      const float pre = softplus_f(x);
      const float pass = (pre >= a.scale_lo && pre <= a.scale_hi) ? 1.f : 0.f;
      const float dsp = x > 20.f ? 1.f : sigmoid_f(x);
      gg[(size_t)(7 + c) * G] = (gpre_[c] + gcl_[c] * pass) * dsp;
    }
  }
  // opacity = sigmoid
  {
    const float op = sigmoid_f(fg[10 * G]);
    gg[10 * G] = (a.g_opacity ? a.g_opacity[o] : 0.f) * op * (1.f - op);
  }
  // sigma = max(0.1 exp(x), 0.01)
  {
    const float e = expf(fg[11 * G]) * 0.1f;
    gg[11 * G] = (e >= 0.01f) ? (a.g_sigma ? a.g_sigma[o] : 0.f) * e : 0.f;
  }
}

}  // namespace

// Row R2 forward: replaces rgca.py:506-546 (no native boundary exists in the reference; the Python-side mirror is
// goliath_b200.rgca_heads.gaussian_heads).  Planes are [B,C,G] with G = H*W; outputs are [B,G,*] (opacity, sigma,
// spec_vis: [B,G]); shsum [B,G,3] is saved for the backward.
GB_API int gb_rgca_heads_fwd(int B, int G, const float* f_vnocond, const float* f_vcond, const float* postex,
                             const float* tn, const float* albedo, const float* light_sh, const float* campos,
                             float scale_lo, float scale_hi, float* primpos, float* primqvec, float* primscale,
                             float* primscale_preclip, float* opacity, float* sigma, float* spec_vis, float* spec_dnml,
                             float* spec_nml, float* diff_color, float* ref_dirs, float* primnmlbase, float* shsum,
                             const float* light_sh2, float* shsum2, void* stream) {
  if (B <= 0 || G <= 0) return 0;
  HeadsArgs a = {};
  a.B = B; a.G = G; a.f_vnocond = f_vnocond; a.f_vcond = f_vcond; a.postex = postex; a.tn = tn; a.albedo = albedo;
  a.light_sh = light_sh; a.campos = campos; a.scale_lo = scale_lo; a.scale_hi = scale_hi; a.primpos = primpos;
  a.primqvec = primqvec; a.primscale = primscale; a.primscale_preclip = primscale_preclip; a.opacity = opacity;
  a.sigma = sigma; a.spec_vis = spec_vis; a.spec_dnml = spec_dnml; a.spec_nml = spec_nml; a.diff_color = diff_color;
  a.ref_dirs = ref_dirs; a.primnmlbase = primnmlbase; a.shsum = shsum;
  a.light_sh2 = light_sh2; a.shsum2 = shsum2;
  if ((light_sh2 == nullptr) != (shsum2 == nullptr)) return (int)cudaErrorInvalidValue;
  if (light_sh2)
    GB_CUDA(gb::launch<heads_fwd_kernel<true>>(dim3(gb::cdiv(G, kBlock), B), kBlock, 0, (cudaStream_t)stream, a));
  else
    GB_CUDA(gb::launch<heads_fwd_kernel<false>>(dim3(gb::cdiv(G, kBlock), B), kBlock, 0, (cudaStream_t)stream, a));
  return 0;
}

// Row R2 backward.  Upstream gradients may be NULL (treated as zero).  Writes g_f_vnocond [B,125,G],
// g_f_vcond [B,4,G], g_postex [B,3,G], g_tn [B,3,G], g_albedo [B,G,3] (the caller sums over B).
GB_API int gb_rgca_heads_bwd(int B, int G, const float* f_vnocond, const float* f_vcond, const float* postex,
                             const float* tn, const float* albedo, const float* light_sh, const float* campos,
                             float scale_lo, float scale_hi, const float* shsum, const float* g_primpos,
                             const float* g_primqvec, const float* g_primscale, const float* g_primscale_preclip,
                             const float* g_opacity, const float* g_sigma, const float* g_spec_vis,
                             const float* g_spec_dnml, const float* g_spec_nml, const float* g_diff_color,
                             const float* g_ref_dirs, const float* g_primnmlbase, float* g_f_vnocond, float* g_f_vcond,
                             float* g_postex, float* g_tn, float* g_albedo, const float* light_sh2, const float* g_shsum2,
                             void* stream) {
  if (B <= 0 || G <= 0) return 0;
  HeadsArgs a = {};
  a.B = B; a.G = G; a.f_vnocond = f_vnocond; a.f_vcond = f_vcond; a.postex = postex; a.tn = tn; a.albedo = albedo;
  a.light_sh = light_sh; a.campos = campos; a.scale_lo = scale_lo; a.scale_hi = scale_hi;
  a.shsum = const_cast<float*>(shsum);
  a.g_primpos = g_primpos; a.g_primqvec = g_primqvec; a.g_primscale = g_primscale;
  a.g_primscale_preclip = g_primscale_preclip; a.g_opacity = g_opacity; a.g_sigma = g_sigma; a.g_spec_vis = g_spec_vis;
  a.g_spec_dnml = g_spec_dnml; a.g_spec_nml = g_spec_nml; a.g_diff_color = g_diff_color; a.g_ref_dirs = g_ref_dirs;
  a.g_primnmlbase = g_primnmlbase; a.g_f_vnocond = g_f_vnocond; a.g_f_vcond = g_f_vcond; a.g_postex = g_postex;
  a.g_tn = g_tn; a.g_albedo = g_albedo;
  a.light_sh2 = light_sh2; a.g_shsum2 = g_shsum2;
  if (light_sh2 && g_shsum2)
    GB_CUDA(gb::launch<heads_bwd_kernel<true>>(dim3(gb::cdiv(G, kBlock), B), kBlock, 0, (cudaStream_t)stream, a));
  else
    GB_CUDA(gb::launch<heads_bwd_kernel<false>>(dim3(gb::cdiv(G, kBlock), B), kBlock, 0, (cudaStream_t)stream, a));
  return 0;
}
