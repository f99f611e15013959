// goliath_b200/csrc/conv_wnub.cu — stride-1 KxK (K = 1 | 3, "same" padding) convolution with the reference's
// weight-norm scale, tied or untied bias and LeakyReLU fused into the epilogue (sm_90a), forward and backward, on the
// kernels of wn_conv.cuh.
//
// This is the layer the hand-MVP decoders are made of besides the transposed convolutions:
//   TransDecoder       5 x la.Conv2dWNUB(.., 64, 64, 3, 1, 1) + LeakyReLU(0.2)   ca_code/models/hand_mvp.py:297-321
//   PoseEncoder        2 x blocks.ConvBlock = Conv2dWN 1x1 (tied bias) + 2 x Conv2dWNUB  hand_mvp.py:269-294, blocks.py:232-280
// replacing per layer cuDNN conv2d (layers.py:303-317), the `output + bias[None]` pass (layers.py:319-327), the
// LeakyReLU pass and the weight-norm reparametrisation w = g * v / ||v||_F (layers.py:200-204; g per OUTPUT channel,
// weight [Cout,Cin,K,K]) which is folded into a per-output-channel scale.
//
// The body texture branch (ShadowUNet, the UNetWB and UpscaleNet 1x1 layers) and mesh_vae.ConvDecoder's verts_conv /
// tex_conv, which read a channel slice of a wider map in place through x's batch stride, run on it too.
#include "wn_conv.cuh"

namespace {

// output channels per CTA: 8, or 4 for the narrow layers (the decoder's 3-channel verts_conv / tex_conv), where one
// CTA covers every channel either way and the narrower tile does half the arithmetic
int co_tile(int n) { return n <= 4 ? 4 : 8; }

template <int CO_T, int K>
[[nodiscard]] int launch_fwd(int B, int Cin, int Cout, const InMap& x, const float* v, const float* scale, const float* bias,
                             int bias_mode, float slope, int apply_act, float* out, cudaStream_t s) {
  dim3 grid(gb::cdiv(x.H, TP) * gb::cdiv(x.W, TP), gb::cdiv(Cout, CO_T), B);
  return gb::launch<wn_conv_fwd_kernel<CO_T, K, 1, false, 0, IN_PLAIN>>(grid, TP * TP, 0, s,
      Cin, Cout, 1, x, x.H, x.W, v, scale, bias, bias_mode, apply_act, slope, x, nullptr, nullptr, nullptr, out, nullptr);
}

template <int CO_T, int K>
[[nodiscard]] int launch_dgrad(int B, int Cin, int Cout, int H, int W, const float* gz, const float* v,
                               const float* scale, float* gx, long long x_bs, cudaStream_t s) {
  dim3 grid(gb::cdiv(H, TP) * gb::cdiv(W, TP), gb::cdiv(Cin, CO_T), B);
  return gb::launch<wn_conv_dgrad_kernel<CO_T, K, 1, false, 0>>(grid, TP * TP, 0, s,
      Cin, Cout, 1, H, W, gz, v, scale, nullptr, 1.f, 0, nullptr, nullptr, nullptr, gx, x_bs);
}

constexpr int kWgradPerSM = 3;

bool bad_shape(int Cin, int H, int W, int K, long long x_bs) {
  return (K != 1 && K != 3) || x_bs < (long long)Cin * H * W;
}

}  // namespace

// Fused Conv2dWN / Conv2dWNUB (stride 1, K = 1 or 3, padding (K-1)/2) [+ LeakyReLU] forward.
// x [B,Cin,H,W] with items x_bs floats apart; v = weight_v [Cout,Cin,K,K]; scale [Cout] = weight_g / ||weight_v||_F;
// bias_mode 0 none, 1 tied [Cout] (th.nn.Conv2d bias, blocks.py:252), 2 untied [Cout,H,W] (layers.py:276-327);
// out [B,Cout,H,W].
GB_API int gb_conv2d_wnub_fwd(int B, int Cin, int Cout, int H, int W, int K, const float* x, long long x_bs,
                              const float* v, const float* scale, const float* bias, int bias_mode, float slope,
                              int apply_act, float* out, void* stream) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || H <= 0 || W <= 0) return 0;
  if (bad_shape(Cin, H, W, K, x_bs)) return (int)cudaErrorInvalidValue;
  if (!bias) bias_mode = 0;
  cudaStream_t s = (cudaStream_t)stream;
  const InMap xm = plain_map(x, x_bs, H, W);
  if (co_tile(Cout) == 8) {
    if (K == 1) return launch_fwd<8, 1>(B, Cin, Cout, xm, v, scale, bias, bias_mode, slope, apply_act, out, s);
    return launch_fwd<8, 3>(B, Cin, Cout, xm, v, scale, bias, bias_mode, slope, apply_act, out, s);
  }
  if (K == 1) return launch_fwd<4, 1>(B, Cin, Cout, xm, v, scale, bias, bias_mode, slope, apply_act, out, s);
  return launch_fwd<4, 3>(B, Cin, Cout, xm, v, scale, bias, bias_mode, slope, apply_act, out, s);
}

GB_API size_t gb_conv2d_wnub_bwd_workspace_bytes(int B, int Cin, int Cout, int H, int W, int K) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || H <= 0 || W <= 0 || (K != 1 && K != 3)) return 0;
  return sizeof(float) * wgrad_part_floats(B, Cin, Cout, 1, K, H, W, kWgradPerSM);
}

// Backward of gb_conv2d_wnub_fwd.  gz [B,Cout,H,W]: scratch for the pre-activation gradient when apply_act, else unused
// (gout is that gradient); g_bias written ([Cout,H,W] for bias_mode 2, [Cout] for 1) or NULL; gx [B,Cin,H,W] with items
// x_bs floats apart, or NULL; gw [Cout,Cin,K,K] written = gradient of the effective weight at unit scale — the caller
// finishes the weight-norm chain rule on the small tensors.  workspace: gb_conv2d_wnub_bwd_workspace_bytes(..) bytes.
GB_API int gb_conv2d_wnub_bwd(int B, int Cin, int Cout, int H, int W, int K, const float* x, long long x_bs,
                              const float* v, const float* scale, const float* out, const float* gout, float slope,
                              int apply_act, int bias_mode, float* gz, float* g_bias, float* gx, float* gw,
                              void* workspace, void* stream) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || H <= 0 || W <= 0) return 0;
  if (bad_shape(Cin, H, W, K, x_bs)) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const long long per_item = (long long)Cout * H * W;
  const unsigned grid = (unsigned)gb::cdiv64(per_item, 256);
  const float* g = gout;
  if (apply_act) {
    GB_CUDA(gb::launch<act_bwd_kernel>(grid, 256, 0, s, B, per_item, gout, nullptr, out, slope, gz,
                                       bias_mode == 2 ? g_bias : nullptr));
    g = gz;
  } else if (bias_mode == 2 && g_bias) {
    GB_CUDA(gb::launch<batch_sum_kernel>(grid, 256, 0, s, B, per_item, gout, g_bias));
  }
  if (bias_mode == 1 && g_bias) GB_CUDA(gb::launch<chan_sum_kernel>(Cout, 256, 0, s, B, Cout, H * W, g, g_bias));
  if (gx) {
    if (co_tile(Cin) == 8) {
      if (K == 1) GB_CUDA(launch_dgrad<8, 1>(B, Cin, Cout, H, W, g, v, scale, gx, x_bs, s));
      else GB_CUDA(launch_dgrad<8, 3>(B, Cin, Cout, H, W, g, v, scale, gx, x_bs, s));
    } else {
      if (K == 1) GB_CUDA(launch_dgrad<4, 1>(B, Cin, Cout, H, W, g, v, scale, gx, x_bs, s));
      else GB_CUDA(launch_dgrad<4, 3>(B, Cin, Cout, H, W, g, v, scale, gx, x_bs, s));
    }
  }
  const InMap xm = plain_map(x, x_bs, H, W);
  float* part = (float*)workspace;
  if (K == 1) return launch_wgrad<1, 1>(B, Cin, Cout, 1, xm, H, W, g, gw, part, kWgradPerSM, s);
  return launch_wgrad<3, 1>(B, Cin, Cout, 1, xm, H, W, g, gw, part, kWgradPerSM, s);
}
