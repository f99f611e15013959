// goliath_b200/csrc/conv_wnub.cu — stride-1 KxK (K = 1 | 3, "same" padding) convolution with the reference's
// weight-norm scale, tied or untied bias and LeakyReLU fused into the epilogue (sm_90a), forward and backward.
//
// This is the layer the hand-MVP decoders are made of besides the transposed convolutions:
//   TransDecoder       5 x la.Conv2dWNUB(.., 64, 64, 3, 1, 1) + LeakyReLU(0.2)   ca_code/models/hand_mvp.py:297-321
//   PoseEncoder        2 x blocks.ConvBlock = Conv2dWN 1x1 (tied bias) + 2 x Conv2dWNUB  hand_mvp.py:269-294, blocks.py:232-280
// replacing per layer cuDNN conv2d (layers.py:303-317), the `output + bias[None]` pass (layers.py:319-327), the
// LeakyReLU pass and the weight-norm reparametrisation w = g * v / ||v||_F (layers.py:200-204; g per OUTPUT channel,
// weight [Cout,Cin,K,K]) which is folded into a per-output-channel scale.
//
// All maps on this path are 64x64 with <= 128 channels (<= 2 MB per tensor): the layers are launch/latency-bound,
// so one fused fp32 SIMT kernel per layer (and three for its backward) is the whole optimisation; no tensor cores.
#include "common.cuh"

namespace {

constexpr int TP = 16;       // pixels per CTA edge
constexpr int CO_T = 8;      // output channels per CTA
constexpr int CI_CHUNK = 8;  // input channels staged per step

// One kernel serves the forward and the data gradient (a convolution of gz with the flipped, channel-swapped kernel):
//   TRANSPOSED = false:  out[o,y,x] = act(scale[o] * sum_i sum_k in[i, y+ky-P, x+kx-P] * v[o,i,ky,kx] + bias)
//   TRANSPOSED = true :  out[o,y,x] =            sum_i sum_k in[i, y+ky-P, x+kx-P] * scale[i] * v[i,o,K-1-ky,K-1-kx]
// (n_in / n_out are the channel counts of `in` / `out` in this launch; v is always [Cout, Cin, K, K].)
template <int K, bool TRANSPOSED>
__global__ void __launch_bounds__(TP* TP) conv_s1_kernel(int n_in, int n_out, int H, int W, const float* __restrict__ in,
                                                         const float* __restrict__ v, const float* __restrict__ scale,
                                                         const float* __restrict__ bias, int bias_mode, float slope,
                                                         int apply_act, float* __restrict__ out) {
  constexpr int P = (K - 1) / 2, HALO = TP + 2 * P, KK = K * K;
  __shared__ float s_x[CI_CHUNK][HALO][HALO + 1];
  __shared__ float s_w[CI_CHUNK][CO_T][KK];
  const int tiles_x = (W + TP - 1) / TP;
  const int ty0 = (blockIdx.x / tiles_x) * TP, tx0 = (blockIdx.x % tiles_x) * TP;
  const int o0 = blockIdx.y * CO_T, b = blockIdx.z;
  const int tid = threadIdx.x, py = tid / TP, px = tid % TP;
  const float* inb = in + (size_t)b * n_in * H * W;
  float acc[CO_T];
#pragma unroll
  for (int c = 0; c < CO_T; ++c) acc[c] = 0.f;

  for (int i0 = 0; i0 < n_in; i0 += CI_CHUNK) {
    __syncthreads();
    for (int i = tid; i < CI_CHUNK * HALO * HALO; i += TP * TP) {
      const int ci = i / (HALO * HALO), r = (i / HALO) % HALO, c = i % HALO;
      const int yy = ty0 - P + r, xx = tx0 - P + c;
      float val = 0.f;
      if (i0 + ci < n_in && yy >= 0 && yy < H && xx >= 0 && xx < W) val = inb[((size_t)(i0 + ci) * H + yy) * W + xx];
      s_x[ci][r][c] = val;
    }
    for (int i = tid; i < CI_CHUNK * CO_T * KK; i += TP * TP) {
      const int ci = i / (CO_T * KK), co = (i / KK) % CO_T, k = i % KK;
      float val = 0.f;
      if (i0 + ci < n_in && o0 + co < n_out) {
        if (!TRANSPOSED) val = v[((size_t)(o0 + co) * n_in + (i0 + ci)) * KK + k];
        else val = v[((size_t)(i0 + ci) * n_out + (o0 + co)) * KK + (KK - 1 - k)] * scale[i0 + ci];
      }
      s_w[ci][co][k] = val;
    }
    __syncthreads();
#pragma unroll 2
    for (int ci = 0; ci < CI_CHUNK; ++ci) {
      float a[KK];
#pragma unroll
      for (int ky = 0; ky < K; ++ky)
#pragma unroll
        for (int kx = 0; kx < K; ++kx) a[ky * K + kx] = s_x[ci][py + ky][px + kx];
#pragma unroll
      for (int c = 0; c < CO_T; ++c) {
        float s = acc[c];
#pragma unroll
        for (int k = 0; k < KK; ++k) s += a[k] * s_w[ci][c][k];
        acc[c] = s;
      }
    }
  }
  const int y = ty0 + py, x = tx0 + px;
  if (y >= H || x >= W) return;
#pragma unroll
  for (int c = 0; c < CO_T; ++c) {
    const int o = o0 + c;
    if (o >= n_out) break;
    float r = acc[c];
    if (!TRANSPOSED) {
      r *= scale[o];
      if (bias_mode == 1) r += bias[o];
      else if (bias_mode == 2) r += bias[((size_t)o * H + y) * W + x];
      if (apply_act) r = r > 0.f ? r : r * slope;
    }
    out[(((size_t)b * n_out + o) * H + y) * W + x] = r;
  }
}

// gz = gout * act'(out);  untied bias gradient = sum over the batch (bias_mode 2);  the tied one (mode 1) is a
// per-channel sum over batch and pixels, accumulated with one RED per warp.
__global__ void __launch_bounds__(256) conv_act_bwd_kernel(int B, int C, int HW, const float* __restrict__ gout,
                                                           const float* __restrict__ out, float slope, int apply_act,
                                                           int bias_mode, float* __restrict__ gz,
                                                           float* __restrict__ gbias) {
  const long long per_item = (long long)C * HW;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float acc = 0.f;
  if (i < per_item) {
    for (int b = 0; b < B; ++b) {
      const size_t o = (size_t)b * per_item + i;
      float g = gout[o];
      if (apply_act) g = out[o] > 0.f ? g : g * slope;
      gz[o] = g;
      acc += g;
    }
    if (gbias && bias_mode == 2) gbias[i] = acc;
  }
  if (gbias && bias_mode == 1) {
    // HW is a multiple of 32 on this path or not: lanes of one warp may straddle two channels, so reduce per lane
    // group with match_any on the channel index
    const int ch = i < per_item ? (int)(i / HW) : -1;
    const unsigned grp = __match_any_sync(0xffffffffu, ch);
    float tot = 0.f;
    for (int l = 0; l < 32; ++l) {
      const float vv = __shfl_sync(0xffffffffu, acc, l);
      if (grp & (1u << l)) tot += vv;
    }
    if (ch >= 0 && (int)(__ffs(grp) - 1) == (int)(threadIdx.x & 31)) gb::red_add(gbias + ch, tot);
  }
}

// weight gradient gw[co,ci,ky,kx] = sum_{b,y,x} gz[b,co,y,x] * x[b,ci,y+ky-P,x+kx-P]   (effective weight, unit scale)
constexpr int BW_TX = 16, BW_TY = 8;
constexpr int BW_CI = 16, BW_CO = 8;

template <int K>
__global__ void __launch_bounds__(256) conv_s1_bwd_weight_kernel(int B, int Cin, int Cout, int H, int W,
                                                                 const float* __restrict__ x,
                                                                 const float* __restrict__ gz,
                                                                 float* __restrict__ gw /* [Cout,Cin,K,K] accumulated */) {
  constexpr int P = (K - 1) / 2, KK = K * K, XW = BW_TX + 2 * P, XH = BW_TY + 2 * P;
  __shared__ float s_x[BW_CI][XH][XW + 1];
  __shared__ float s_g[BW_CO][BW_TX * BW_TY];
  const int ci0 = blockIdx.y * BW_CI, co0 = blockIdx.z * BW_CO;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cig = lane >> 3, col = lane & 7;
  const int tiles_x = (W + BW_TX - 1) / BW_TX, tiles_y = (H + BW_TY - 1) / BW_TY;
  const int total = B * tiles_x * tiles_y;
  float acc[4][KK];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int k = 0; k < KK; ++k) acc[a][k] = 0.f;

  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    const int b = t / (tiles_x * tiles_y), tt = t % (tiles_x * tiles_y);
    const int ty0 = (tt / tiles_x) * BW_TY, tx0 = (tt % tiles_x) * BW_TX;
    __syncthreads();
    for (int i = tid; i < BW_CI * XH * XW; i += 256) {
      const int ci = i / (XH * XW), r = (i / XW) % XH, c = i % XW;
      const int yy = ty0 - P + r, xx = tx0 - P + c;
      float val = 0.f;
      if (ci0 + ci < Cin && yy >= 0 && yy < H && xx >= 0 && xx < W) val = x[(((size_t)b * Cin + ci0 + ci) * H + yy) * W + xx];
      s_x[ci][r][c] = val;
    }
    for (int i = tid; i < BW_CO * BW_TX * BW_TY; i += 256) {
      const int co = i / (BW_TX * BW_TY), p = i % (BW_TX * BW_TY);
      const int yy = ty0 + p / BW_TX, xx = tx0 + p % BW_TX;
      float val = 0.f;
      if (co0 + co < Cout && yy < H && xx < W) val = gz[(((size_t)b * Cout + co0 + co) * H + yy) * W + xx];
      s_g[co][p] = val;
    }
    __syncthreads();
    for (int pp = 0; pp < (BW_TX * BW_TY) / 8; ++pp) {  // this warp's row of the tile
      const int p = warp * ((BW_TX * BW_TY) / 8) + pp, py = p / BW_TX, px = p % BW_TX;
      const float g = s_g[col][p];
#pragma unroll
      for (int ky = 0; ky < K; ++ky)
#pragma unroll
        for (int kx = 0; kx < K; ++kx)
#pragma unroll
          for (int a = 0; a < 4; ++a) acc[a][ky * K + kx] += s_x[cig * 4 + a][py + ky][px + kx] * g;
    }
  }
  const int co = co0 + col;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int ci = ci0 + cig * 4 + a;
    if (ci < Cin && co < Cout) {
#pragma unroll
      for (int k = 0; k < KK; ++k) gb::red_add(gw + ((size_t)co * Cin + ci) * KK + k, acc[a][k]);
    }
  }
}

template <int K>
int launch_fwd(int B, int Cin, int Cout, int H, int W, const float* x, const float* v, const float* scale,
               const float* bias, int bias_mode, float slope, int apply_act, float* out, cudaStream_t s) {
  dim3 grid(gb::cdiv(H, TP) * gb::cdiv(W, TP), gb::cdiv(Cout, CO_T), B);
  conv_s1_kernel<K, false><<<grid, TP * TP, 0, s>>>(Cin, Cout, H, W, x, v, scale, bias, bias_mode, slope, apply_act, out);
  return 1;
}

template <int K>
int launch_bwd(int B, int Cin, int Cout, int H, int W, const float* x, const float* v, const float* scale,
               const float* gz, float* gx, float* gw, cudaStream_t s) {
  int n = 0;
  if (gx) {
    dim3 grid(gb::cdiv(H, TP) * gb::cdiv(W, TP), gb::cdiv(Cin, CO_T), B);
    conv_s1_kernel<K, true><<<grid, TP * TP, 0, s>>>(Cout, Cin, H, W, gz, v, scale, nullptr, 0, 1.f, 0, gx);
    ++n;
  }
  if (gw) {
    const int total = B * gb::cdiv(H, BW_TY) * gb::cdiv(W, BW_TX);
    const int pairs = gb::cdiv(Cin, BW_CI) * gb::cdiv(Cout, BW_CO);
    int split = gb::cdiv(gb::kNumSMs * 3, pairs);
    split = max(1, min(split, total));
    dim3 grid(split, gb::cdiv(Cin, BW_CI), gb::cdiv(Cout, BW_CO));
    conv_s1_bwd_weight_kernel<K><<<grid, 256, 0, s>>>(B, Cin, Cout, H, W, x, gz, gw);
    ++n;
  }
  return n;
}

}  // namespace

// Fused Conv2dWN / Conv2dWNUB (stride 1, K = 1 or 3, padding (K-1)/2) [+ LeakyReLU] forward.
// x [B,Cin,H,W]; v = weight_v [Cout,Cin,K,K]; scale [Cout] = weight_g / ||weight_v||_F; bias_mode 0 none,
// 1 tied [Cout] (th.nn.Conv2d bias, blocks.py:252), 2 untied [Cout,H,W] (layers.py:276-327); out [B,Cout,H,W].
GB_API int gb_conv2d_wnub_fwd(int B, int Cin, int Cout, int H, int W, int K, const float* x, const float* v,
                              const float* scale, const float* bias, int bias_mode, float slope, int apply_act,
                              float* out, void* stream) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || H <= 0 || W <= 0) return 0;
  if (K != 1 && K != 3) return (int)cudaErrorInvalidValue;
  if (!bias) bias_mode = 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int n = K == 1 ? launch_fwd<1>(B, Cin, Cout, H, W, x, v, scale, bias, bias_mode, slope, apply_act, out, s)
                       : launch_fwd<3>(B, Cin, Cout, H, W, x, v, scale, bias, bias_mode, slope, apply_act, out, s);
  gb::count_launches(n);
  GB_CHECK_LAUNCH();
  return 0;
}

// Backward of gb_conv2d_wnub_fwd.  gz [B,Cout,H,W] scratch (gradient at the pre-activation); g_bias ([Cout,H,W]
// written for bias_mode 2; [Cout] ACCUMULATED for bias_mode 1, caller zeroes it) or NULL; gx [B,Cin,H,W] or NULL;
// gw [Cout,Cin,K,K] ACCUMULATED (caller zeroes it) = gradient of the effective weight at unit scale — the caller
// finishes the weight-norm chain rule on the small tensors.
GB_API int gb_conv2d_wnub_bwd(int B, int Cin, int Cout, int H, int W, int K, const float* x, const float* v,
                              const float* scale, const float* out, const float* gout, float slope, int apply_act,
                              int bias_mode, float* gz, float* g_bias, float* gx, float* gw, void* stream) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || H <= 0 || W <= 0) return 0;
  if (K != 1 && K != 3) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const long long per_item = (long long)Cout * H * W;
  conv_act_bwd_kernel<<<(unsigned)gb::cdiv64(per_item, 256), 256, 0, s>>>(B, Cout, H * W, gout, out, slope, apply_act,
                                                                          bias_mode, gz, g_bias);
  int n = 1;
  n += K == 1 ? launch_bwd<1>(B, Cin, Cout, H, W, x, v, scale, gz, gx, gw, s)
              : launch_bwd<3>(B, Cin, Cout, H, W, x, v, scale, gz, gx, gw, s);
  gb::count_launches(n);
  GB_CHECK_LAUNCH();
  return 0;
}
