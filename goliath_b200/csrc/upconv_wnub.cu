// goliath_b200/csrc/upconv_wnub.cu — the body decoder's upsampling residual block (blocks.UpConvBlockDeep) with
// grouped, weight-normalised 3x3 convolutions and untied biases, fused with its bilinear x2 upsample and its 1x1 skip
// (sm_90a, fp32 SIMT), forward and backward, on the kernels of wn_conv.cuh; and the sparse gathers of the seam sampler
// and of GeometryModule.from_uv.
//
//   u   = UpsamplingBilinear2d(2 Hi)(x)                                   (align_corners = True)
//   h1  = lrelu(conv1(u) + b1)                                            kernel 1: u is built in shared memory
//   out = lrelu(conv2(h1) + b2) + conv_resize(u) + br                     kernel 2: the skip is recomputed from x
//
// Neither u nor the skip is written to memory: both convolutions read u through an IN_UP2 map of x.  The trunk blocks of
// mesh_vae.ConvDecoder run at 128^2..1024^2 with 4-64 channels per group and untied biases [C,H,W].
//
// The backward needs the sign of conv2's pre-activation, which cannot be read back from `out` because the skip is
// added after the activation; the forward writes it as one byte per output element (`mask`, a quarter of `out`'s
// bytes) when the caller asks for it (training).  h1 is kept by the caller.
#include "wn_conv.cuh"

namespace {

// gx = transpose of the upsample applied to gu, as a gather: low-resolution texel (yi, xi) sums gu over the output
// pixels whose bilinear footprint covers it, with the forward's weights; no atomics, fixed order.
__global__ void __launch_bounds__(256) up_transpose_kernel(long long n, InMap gm, const float* __restrict__ gu,
                                                           float* __restrict__ gx) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int H = gm.H, W = gm.W, Hi = gm.Hs, Wi = gm.Ws;
  const int xi = (int)(t % Wi), yi = (int)((t / Wi) % Hi);
  const long long bc = t / ((long long)Hi * Wi);
  // output rows whose i0 or i1 is yi: src = s*y in [yi-1, yi+1); one row of slack either side for rounding
  int ylo = 0, yhi = H - 1, xlo = 0, xhi = W - 1;
  if (gm.sy > 0.f) {
    ylo = max(0, (int)floorf((yi - 1) / gm.sy) - 1);
    yhi = min(H - 1, (int)ceilf((yi + 1) / gm.sy) + 1);
  }
  if (gm.sx > 0.f) {
    xlo = max(0, (int)floorf((xi - 1) / gm.sx) - 1);
    xhi = min(W - 1, (int)ceilf((xi + 1) / gm.sx) + 1);
  }
  const float* g = gu + bc * H * W;
  float acc = 0.f;
  for (int y = ylo; y <= yhi; ++y) {
    int y0, y1;
    float ly;
    up_index(y, Hi, gm.sy, y0, y1, ly);
    if (y0 != yi && y1 != yi) continue;
    const float wy = (y0 == yi ? 1.f - ly : 0.f) + (y1 == yi ? ly : 0.f);
    float row = 0.f;
    for (int x = xlo; x <= xhi; ++x) {
      int x0, x1;
      float lx;
      up_index(x, Wi, gm.sx, x0, x1, lx);
      if (x0 != xi && x1 != xi) continue;
      const float wx = (x0 == xi ? 1.f - lx : 0.f) + (x1 == xi ? lx : 0.f);
      row += wx * g[(size_t)y * W + x];
    }
    acc += wy * row;
  }
  gx[t] = acc;
}

// out[b, c, r] = sum_{e in [ptr[r], ptr[r+1])} coef[e] * in[b, c, col[e]]  — element strides per tensor
constexpr int SP_C = 8;
__global__ void __launch_bounds__(256)
    sparse_rows_kernel(int B, int C, int n_rows, const int* __restrict__ ptr, const int* __restrict__ col,
                       const float* __restrict__ coef, const float* __restrict__ in, long long in_bs, long long in_cs,
                       long long in_rs, float* __restrict__ out, long long out_bs, long long out_cs, long long out_rs) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)B * n_rows) return;
  const int r = (int)(t % n_rows), b = (int)(t / n_rows);
  const int e0 = ptr[r], e1 = ptr[r + 1];
  const float* inb = in + b * in_bs;
  float* outb = out + b * out_bs + r * out_rs;
  for (int c0 = 0; c0 < C; c0 += SP_C) {
    float acc[SP_C];
#pragma unroll
    for (int c = 0; c < SP_C; ++c) acc[c] = 0.f;
    for (int e = e0; e < e1; ++e) {
      const float w = __ldg(coef + e);
      const float* p = inb + __ldg(col + e) * in_rs;
#pragma unroll
      for (int c = 0; c < SP_C; ++c)
        if (c0 + c < C) acc[c] += w * p[(c0 + c) * in_cs];
    }
#pragma unroll
    for (int c = 0; c < SP_C; ++c)
      if (c0 + c < C) outb[(c0 + c) * out_cs] = acc[c];
  }
}

template <int CO_T>
void launch_fwd_pair(int B, int Cin, int Cout, int groups, const InMap& u, const float* v1,
                     const float* s1, const float* b1, const float* v2, const float* s2, const float* b2,
                     const float* vr, const float* sr, const float* br, float slope, float* h1, float* out,
                     unsigned char* mask, cudaStream_t s) {
  const int cin_g = Cin / groups, cout_g = Cout / groups;
  const int tiles = gb::cdiv(u.H, TP) * gb::cdiv(u.W, TP);
  dim3 g1(tiles, groups * gb::cdiv(cin_g, CO_T), B), g2(tiles, groups * gb::cdiv(cout_g, CO_T), B);
  wn_conv_fwd_kernel<CO_T, 3, 1, false, 2, IN_UP2, IN_UP2><<<g1, TP * TP, 0, s>>>(cin_g, cin_g, groups, u, u.H, u.W, v1, s1, b1, 2, 1,
                                                                slope, u, nullptr, nullptr, nullptr, h1, nullptr);
  wn_conv_fwd_kernel<CO_T, 3, 1, true, 2, IN_PLAIN, IN_UP2><<<g2, TP * TP, 0, s>>>(
      cin_g, cout_g, groups, plain_map(h1, (long long)Cin * u.H * u.W, u.H, u.W), u.H, u.W, v2, s2, b2, 2, 1, slope, u,
      vr, sr, br, out, mask);
}

// gz1 = conv2^T(gz2) * lrelu'(h1), or (ACT = false) gu = conv1^T(gz1) + conv_resize^T(gout)
template <int CO_T, bool ACT, int SKIP>
void launch_dgrad(int B, int Cin, int n_sum_g, int groups, int H, int W, const float* gz, const float* v,
                  const float* scale, const float* h1, float slope, int n_skip_g, const float* gs, const float* vr,
                  const float* sr, float* out, cudaStream_t s) {
  const int cin_g = Cin / groups;
  dim3 grid(gb::cdiv(H, TP) * gb::cdiv(W, TP), groups * gb::cdiv(cin_g, CO_T), B);
  wn_conv_dgrad_kernel<CO_T, 3, 1, ACT, SKIP><<<grid, TP * TP, 0, s>>>(
      cin_g, n_sum_g, groups, H, W, gz, v, scale, h1, slope, n_skip_g, gs, vr, sr, out, (long long)Cin * H * W);
}

constexpr int kWgradPerSM = 4;

bool bad_shape(int B, int Cin, int Cout, int groups, int Hi, int Wi) {
  return B <= 0 || Cin <= 0 || Cout <= 0 || Hi <= 0 || Wi <= 0 || groups <= 0 || Cin % groups || Cout % groups;
}

}  // namespace

GB_API int gb_upconv_block_fwd(int B, int Cin, int Cout, int groups, int Hi, int Wi, const float* x, const float* v1,
                               const float* s1, const float* b1, const float* v2, const float* s2, const float* b2,
                               const float* vr, const float* sr, const float* br, float slope, float* h1, float* out,
                               unsigned char* mask, void* stream) {
  if (bad_shape(B, Cin, Cout, groups, Hi, Wi)) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const InMap u = up2_map(x, Cin, Hi, Wi);
  if ((Cin / groups) % 8 == 0 && (Cout / groups) % 8 == 0)
    launch_fwd_pair<8>(B, Cin, Cout, groups, u, v1, s1, b1, v2, s2, b2, vr, sr, br, slope, h1, out, mask, s);
  else
    launch_fwd_pair<4>(B, Cin, Cout, groups, u, v1, s1, b1, v2, s2, b2, vr, sr, br, slope, h1, out, mask, s);
  gb::count_launches(2);
  GB_CHECK_LAUNCH();
  return 0;
}

GB_API size_t gb_upconv_block_bwd_workspace_bytes(int B, int Cin, int Cout, int groups, int Hi, int Wi) {
  if (bad_shape(B, Cin, Cout, groups, Hi, Wi)) return 0;
  const int H = 2 * Hi, W = 2 * Wi;
  const size_t w2 = wgrad_part_floats(B, Cin, Cout, groups, 3, H, W, kWgradPerSM);
  const size_t w1 = wgrad_part_floats(B, Cin, Cin, groups, 3, H, W, kWgradPerSM);
  const size_t wr = wgrad_part_floats(B, Cin, Cout, groups, 1, H, W, kWgradPerSM);
  return sizeof(float) * max(w2, max(w1, wr));
}

GB_API int gb_upconv_block_bwd(int B, int Cin, int Cout, int groups, int Hi, int Wi, const float* x, const float* v1,
                               const float* s1, const float* v2, const float* s2, const float* vr, const float* sr,
                               const float* h1, const unsigned char* mask, const float* gout, float slope, float* gz2,
                               float* gz1, float* gu, float* gb1, float* gb2, float* gbr, float* gw1, float* gw2,
                               float* gwr, float* gx, void* workspace, void* stream) {
  if (bad_shape(B, Cin, Cout, groups, Hi, Wi)) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const InMap u = up2_map(x, Cin, Hi, Wi);
  const int H = u.H, W = u.W, HW = H * W;
  const int cin_g = Cin / groups, cout_g = Cout / groups;
  const long long n_out = (long long)Cout * HW, n_in = (long long)Cin * HW;
  float* part = (float*)workspace;
  act_bwd_kernel<<<(unsigned)gb::cdiv64(n_out, 256), 256, 0, s>>>(B, n_out, gout, mask, nullptr, slope, gz2, gb2);
  chan_sum_kernel<<<Cout, 256, 0, s>>>(B, Cout, HW, gout, gbr);
  if (cin_g % 8 == 0)
    launch_dgrad<8, true, 0>(B, Cin, cout_g, groups, H, W, gz2, v2, s2, h1, slope, 0, nullptr, nullptr, nullptr,
                                 gz1, s);
  else
    launch_dgrad<4, true, 0>(B, Cin, cout_g, groups, H, W, gz2, v2, s2, h1, slope, 0, nullptr, nullptr, nullptr,
                                 gz1, s);
  batch_sum_kernel<<<(unsigned)gb::cdiv64(n_in, 256), 256, 0, s>>>(B, n_in, gz1, gb1);
  launch_wgrad<3, 1>(B, Cin, Cout, groups, plain_map(h1, n_in, H, W), H, W, gz2, gw2, part, kWgradPerSM, s);
  launch_wgrad<3, 1>(B, Cin, Cin, groups, u, H, W, gz1, gw1, part, kWgradPerSM, s);
  launch_wgrad<1, 1>(B, Cin, Cout, groups, u, H, W, gout, gwr, part, kWgradPerSM, s);
  int n = 10;
  if (gx) {
    if (cin_g % 8 == 0)
      launch_dgrad<8, false, 1>(B, Cin, cin_g, groups, H, W, gz1, v1, s1, nullptr, slope, cout_g, gout, vr, sr, gu,
                                   s);
    else
      launch_dgrad<4, false, 1>(B, Cin, cin_g, groups, H, W, gz1, v1, s1, nullptr, slope, cout_g, gout, vr, sr, gu,
                                   s);
    const long long nx = (long long)B * Cin * Hi * Wi;
    up_transpose_kernel<<<(unsigned)gb::cdiv64(nx, 256), 256, 0, s>>>(nx, u, gu, gx);
    n += 2;
  }
  gb::count_launches(n);
  GB_CHECK_LAUNCH();
  return 0;
}

GB_API int gb_sparse_rows_apply(int B, int C, int n_rows, const int* row_ptr, const int* col, const float* coef,
                                const float* in, long long in_bs, long long in_cs, long long in_rs, float* out,
                                long long out_bs, long long out_cs, long long out_rs, void* stream) {
  if (B <= 0 || C <= 0 || n_rows <= 0) return 0;
  const long long n = (long long)B * n_rows;
  sparse_rows_kernel<<<(unsigned)gb::cdiv64(n, 256), 256, 0, (cudaStream_t)stream>>>(
      B, C, n_rows, row_ptr, col, coef, in, in_bs, in_cs, in_rs, out, out_bs, out_cs, out_rs);
  gb::count_launches(1);
  GB_CHECK_LAUNCH();
  return 0;
}
