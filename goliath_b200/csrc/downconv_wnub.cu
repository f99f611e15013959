// goliath_b200/csrc/downconv_wnub.cu — the body encoders' downsampling residual block (blocks.ConvDownBlock) with
// grouped, weight-normalised convolutions and untied biases (sm_90a, fp32 SIMT), forward and backward, on the kernels
// of wn_conv.cuh.
//
//   h1  = lrelu(conv1(x) + b1)                                   kernel 1: 3x3, stride 1, "same"
//   out = lrelu(conv2(h1) + b2) + conv_resize(x) + br            kernel 2: 3x3, stride 2, pad 1; the 1x1 stride-2 skip
//                                                                is computed from x[:, :, ::2, ::2] in the epilogue
//
// The skip is never written.  The first block of mesh_vae.Encoder reads its input through an IN_RESIZE map: the resize
// (align_corners = False) of a strided window of the UV position map, times verts_scale and the encoder's boolean
// mask, evaluated while a tile is staged, so the conditioned [B,3,512,512] map is never written either.
//
// As in upconv_wnub.cu the backward needs the sign of conv2's pre-activation, which cannot be read back from `out`
// because the skip is added after the activation; the forward writes it as one byte per output element (`mask`) when
// the caller asks for it.  h1 is kept by the caller.
#include "wn_conv.cuh"

namespace {

struct BlockArgs {
  int B, Cin, Cout, groups, H, W;
  const float* x;
  long long x_bs, x_cs;
  int x_rs, Hs, Ws;
  const unsigned char* cond_mask;
  float cond_scale;
};

bool bad_block(const BlockArgs& a) {
  if (a.B <= 0 || a.Cin <= 0 || a.Cout <= 0 || a.groups <= 0 || a.Cin % a.groups || a.Cout % a.groups) return true;
  if (a.H <= 0 || a.W <= 0 || a.H % 2 || a.W % 2 || a.Hs <= 0 || a.Ws <= 0 || a.x_rs < a.Ws) return true;
  return !a.cond_mask && (a.Hs != a.H || a.Ws != a.W);
}

InMap x_map(const BlockArgs& a) {
  InMap m{};
  m.p = a.x, m.bs = a.x_bs, m.cs = a.x_cs, m.rs = a.x_rs, m.H = a.H, m.W = a.W;
  m.kind = a.cond_mask ? IN_RESIZE : IN_PLAIN;
  m.mask = a.cond_mask, m.Hs = a.Hs, m.Ws = a.Ws;
  m.sy = (float)a.Hs / (float)a.H, m.sx = (float)a.Ws / (float)a.W, m.vscale = a.cond_scale;
  return m;
}

template <int CO_T>
[[nodiscard]] int launch_conv1(const BlockArgs& a, const InMap& x, const float* v1, const float* s1, const float* b1,
                               float slope, float* h1, cudaStream_t s) {
  const int cin_g = a.Cin / a.groups;
  dim3 grid(gb::cdiv(a.H, TP) * gb::cdiv(a.W, TP), a.groups * gb::cdiv(cin_g, CO_T), a.B);
  return gb::launch<wn_conv_fwd_kernel<CO_T, 3, 1, false, 2>>(grid, TP * TP, 0, s, cin_g, cin_g, a.groups, x, a.H, a.W,
                                                              v1, s1, b1, 2, 1, slope, x, nullptr, nullptr, nullptr, h1,
                                                              nullptr);
}

template <int CO_T>
[[nodiscard]] int launch_conv2(const BlockArgs& a, const InMap& x, const float* h1, const float* v2, const float* s2,
                               const float* b2, const float* vr, const float* sr, const float* br, float slope,
                               float* out, unsigned char* mask, cudaStream_t s) {
  const int cin_g = a.Cin / a.groups, cout_g = a.Cout / a.groups, Ho = a.H / 2, Wo = a.W / 2;
  dim3 grid(gb::cdiv(Ho, TP) * gb::cdiv(Wo, TP), a.groups * gb::cdiv(cout_g, CO_T), a.B);
  return gb::launch<wn_conv_fwd_kernel<CO_T, 3, 2, true, 2>>(grid, TP * TP, 0, s,
      cin_g, cout_g, a.groups, plain_map(h1, (long long)a.Cin * a.H * a.W, a.H, a.W), Ho, Wo, v2, s2, b2, 2, 1, slope,
      x, vr, sr, br, out, mask);
}

// gz1 = conv2^T(gz2) * lrelu'(h1), or (ACT = false) gx = conv1^T(gz1) + conv_resize^T(gout)
template <int CO_T, int S, bool ACT, int SKIP>
[[nodiscard]] int launch_dgrad(int B, int Cin, int n_sum_g, int groups, int H, int W, const float* gz, const float* v,
                               const float* scale, const float* h1, float slope, int n_skip_g, const float* gs,
                               const float* vr, const float* sr, float* out, cudaStream_t s) {
  const int cin_g = Cin / groups;
  dim3 grid(gb::cdiv(H, TP) * gb::cdiv(W, TP), groups * gb::cdiv(cin_g, CO_T), B);
  return gb::launch<wn_conv_dgrad_kernel<CO_T, 3, S, ACT, SKIP>>(grid, TP * TP, 0, s,
      cin_g, n_sum_g, groups, H, W, gz, v, scale, h1, slope, n_skip_g, gs, vr, sr, out, (long long)Cin * H * W);
}

constexpr int kWgradPerSM = 4;

}  // namespace

GB_API int gb_downconv_block_fwd(int B, int Cin, int Cout, int groups, int H, int W, const float* x, long long x_bs,
                                 long long x_cs, int x_rs, int Hs, int Ws, const unsigned char* cond_mask,
                                 float cond_scale, const float* v1, const float* s1, const float* b1, const float* v2,
                                 const float* s2, const float* b2, const float* vr, const float* sr, const float* br,
                                 float slope, float* h1, float* out, unsigned char* mask, void* stream) {
  const BlockArgs a{B, Cin, Cout, groups, H, W, x, x_bs, x_cs, x_rs, Hs, Ws, cond_mask, cond_scale};
  if (bad_block(a)) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const InMap xm = x_map(a);
  if ((Cin / groups) % 8 == 0)
    GB_CUDA(launch_conv1<8>(a, xm, v1, s1, b1, slope, h1, s));
  else
    GB_CUDA(launch_conv1<4>(a, xm, v1, s1, b1, slope, h1, s));
  if ((Cout / groups) % 8 == 0) return launch_conv2<8>(a, xm, h1, v2, s2, b2, vr, sr, br, slope, out, mask, s);
  return launch_conv2<4>(a, xm, h1, v2, s2, b2, vr, sr, br, slope, out, mask, s);
}

GB_API size_t gb_downconv_block_bwd_workspace_bytes(int B, int Cin, int Cout, int groups, int H, int W) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || groups <= 0 || Cin % groups || Cout % groups || H <= 0 || W <= 0) return 0;
  const size_t w2 = wgrad_part_floats(B, Cin, Cout, groups, 3, H / 2, W / 2, kWgradPerSM);
  const size_t w1 = wgrad_part_floats(B, Cin, Cin, groups, 3, H, W, kWgradPerSM);
  const size_t wr = wgrad_part_floats(B, Cin, Cout, groups, 1, H / 2, W / 2, kWgradPerSM);
  return sizeof(float) * max(w2, max(w1, wr));
}

GB_API int gb_downconv_block_bwd(int B, int Cin, int Cout, int groups, int H, int W, const float* x, long long x_bs,
                                 long long x_cs, int x_rs, int Hs, int Ws, const unsigned char* cond_mask,
                                 float cond_scale, const float* v1, const float* s1, const float* v2, const float* s2,
                                 const float* vr, const float* sr, const float* h1, const unsigned char* mask,
                                 const float* gout, float slope, float* gz2, float* gz1, float* gb1, float* gb2,
                                 float* gbr, float* gw1, float* gw2, float* gwr, float* gx, void* workspace,
                                 void* stream) {
  const BlockArgs a{B, Cin, Cout, groups, H, W, x, x_bs, x_cs, x_rs, Hs, Ws, cond_mask, cond_scale};
  if (bad_block(a) || (gx && cond_mask)) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const InMap xm = x_map(a);
  const int cin_g = Cin / groups, cout_g = Cout / groups, Ho = H / 2, Wo = W / 2;
  const long long n_out = (long long)Cout * Ho * Wo, n_in = (long long)Cin * H * W;
  float* part = (float*)workspace;
  GB_CUDA(gb::launch<act_bwd_kernel>((unsigned)gb::cdiv64(n_out, 256), 256, 0, s, B, n_out, gout, mask, nullptr, slope,
                                     gz2, gb2));
  GB_CUDA(gb::launch<chan_sum_kernel>(Cout, 256, 0, s, B, Cout, Ho * Wo, gout, gbr));
  if (cin_g % 8 == 0)
    GB_CUDA(launch_dgrad<8, 2, true, 0>(B, Cin, cout_g, groups, H, W, gz2, v2, s2, h1, slope, 0, nullptr, nullptr,
                                        nullptr, gz1, s));
  else
    GB_CUDA(launch_dgrad<4, 2, true, 0>(B, Cin, cout_g, groups, H, W, gz2, v2, s2, h1, slope, 0, nullptr, nullptr,
                                        nullptr, gz1, s));
  GB_CUDA(gb::launch<batch_sum_kernel>((unsigned)gb::cdiv64(n_in, 256), 256, 0, s, B, n_in, gz1, gb1));
  GB_CUDA(launch_wgrad<3, 2>(B, Cin, Cout, groups, plain_map(h1, n_in, H, W), Ho, Wo, gz2, gw2, part, kWgradPerSM, s));
  GB_CUDA(launch_wgrad<3, 1>(B, Cin, Cin, groups, xm, H, W, gz1, gw1, part, kWgradPerSM, s));
  GB_CUDA(launch_wgrad<1, 2>(B, Cin, Cout, groups, xm, Ho, Wo, gout, gwr, part, kWgradPerSM, s));
  if (!gx) return 0;
  if (cin_g % 8 == 0)
    return launch_dgrad<8, 1, false, 2>(B, Cin, cin_g, groups, H, W, gz1, v1, s1, nullptr, slope, cout_g, gout, vr, sr,
                                        gx, s);
  return launch_dgrad<4, 1, false, 2>(B, Cin, cin_g, groups, H, W, gz1, v1, s1, nullptr, slope, cout_g, gout, vr, sr,
                                      gx, s);
}
