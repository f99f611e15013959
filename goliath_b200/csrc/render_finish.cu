// goliath_b200/csrc/render_finish.cu — post-processing of one rendered view, one kernel each way (sm_90a).
//
// Replaces the ~20 small PyTorch kernels (and their autograd twins) of rgca.AutoEncoder.render after the rasteriser
// (ca_code/models/rgca.py:136-151 with ca_code/utils/render_gsplat.py:79-108): HWC -> CHW of the colour image,
// alpha = 1 - final_T (detached), depth normalised by alpha.clamp(0.05, 1).  Input is the fused rasteriser's 4-channel
// image [H,W,4] = rgb + depth-as-colour and its alpha [H,W].
#include "common.cuh"

namespace {

__global__ void __launch_bounds__(256) finish_fwd_kernel(int P, const float4* __restrict__ out4,
                                                         const float* __restrict__ alpha, float* __restrict__ rgb,
                                                         float* __restrict__ alpha_img, float* __restrict__ depth) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const float4 v = out4[i];
  const float a = alpha[i];
  rgb[i] = v.x; rgb[P + i] = v.y; rgb[2 * P + i] = v.z;
  alpha_img[i] = a;
  depth[i] = v.w / fminf(fmaxf(a, 0.05f), 1.f);
}

__global__ void __launch_bounds__(256) finish_bwd_kernel(int P, const float* __restrict__ alpha,
                                                         const float* __restrict__ g_rgb /* [3,P] or null */,
                                                         const float* __restrict__ g_depth /* [P] or null */,
                                                         float4* __restrict__ g_out4) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  if (g_rgb) { g.x = g_rgb[i]; g.y = g_rgb[P + i]; g.z = g_rgb[2 * P + i]; }
  if (g_depth) g.w = g_depth[i] / fminf(fmaxf(alpha[i], 0.05f), 1.f);
  g_out4[i] = g;
}

}  // namespace

// out4 [H,W,4], alpha [H,W] -> rgb [3,H,W], alpha_img [1,H,W] (a copy: the reference detaches it), depth [1,H,W].
GB_API int gb_render_finish_fwd(int img_h, int img_w, const float* out4, const float* alpha, float* rgb,
                                float* alpha_img, float* depth, void* stream) {
  const int P = img_h * img_w;
  if (P <= 0) return 0;
  return gb::launch<finish_fwd_kernel>(gb::cdiv(P, 256), 256, 0, (cudaStream_t)stream, P,
                                       reinterpret_cast<const float4*>(out4), alpha, rgb, alpha_img, depth);
}

// g_rgb [3,H,W] / g_depth [1,H,W] (either may be NULL) -> g_out4 [H,W,4]; alpha receives no gradient (detached upstream).
GB_API int gb_render_finish_bwd(int img_h, int img_w, const float* alpha, const float* g_rgb, const float* g_depth,
                                float* g_out4, void* stream) {
  const int P = img_h * img_w;
  if (P <= 0) return 0;
  return gb::launch<finish_bwd_kernel>(gb::cdiv(P, 256), 256, 0, (cudaStream_t)stream, P, alpha, g_rgb, g_depth,
                                       reinterpret_cast<float4*>(g_out4));
}
