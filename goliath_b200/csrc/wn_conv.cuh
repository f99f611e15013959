// goliath_b200/csrc/wn_conv.cuh — the grouped, weight-normalised KxK convolution (K = 1 | 3, pad (K-1)/2, stride
// S = 1 | 2) that the stride-1 layer (conv_wnub.cu) and the body's residual blocks (upconv_wnub.cu, downconv_wnub.cu)
// are made of, fp32 SIMT (sm_90a): the forward with its epilogue fused, the data gradient, the weight gradient and the
// activation / bias backward.  Those files hold only launchers and the C ABI.  The stride-2 4x4 layers (deconv_wnub.cu)
// keep their own tiles and use the activation backward, the batch sum and the ordered weight-gradient reduction.
//
// The weight-norm scale is per output channel and applied in the epilogue (forward) or to the staged weights (data
// gradient); the weight gradient is that of the effective weight at unit scale, and the caller finishes the chain rule.
// The maps are bound by the bytes they move and the channel counts are small (1..128 per group), so the fusion (one
// pass per convolution, the input resampled while a tile is staged) is the optimisation; tensor cores are not used.
//
// The backward is gather-only and every sum runs in a fixed order, so two runs give the same bits: the data gradient
// visits, per input pixel, the taps that reach an output pixel; the weight gradients are summed across warps and then
// across CTAs in index order through a workspace; the bias gradients are batch sums and per-channel trees.
#pragma once
#include "common.cuh"

namespace {

constexpr int TP = 16;       // output pixels per CTA edge
constexpr int CI_CHUNK = 8;  // input channels staged per step

// A convolution's input x [B, C, H, W] as the kernels read it; channel (b, c) starts at p + b bs + c cs.
//   IN_PLAIN : x[b, c, y, x] = p[y rs + x]
//   IN_RESIZE: p addresses a [Hs, Ws] window (row stride rs), and
//              x[b, c, y, x] = vscale * bilinear(window -> H x W, align_corners = False)[y, x] * mask[y, x]
//   IN_UP2   : p addresses a [Hs, Ws] plane (row stride rs), and x = bilinear(plane -> H x W, align_corners = True)
enum InKind { IN_PLAIN, IN_RESIZE, IN_UP2 };
struct InMap {
  const float* p;
  long long bs, cs;
  int rs, H, W, kind;
  const unsigned char* mask;
  int Hs, Ws;
  float sy, sx, vscale;
};

// items bs floats apart, channels contiguous [H, W] planes
InMap plain_map(const float* p, long long bs, int H, int W) {
  InMap m{};
  m.p = p, m.bs = bs, m.cs = (long long)H * W, m.rs = W, m.H = H, m.W = W, m.kind = IN_PLAIN;
  return m;
}

// the bilinear x2 upsample (align_corners = True) of a contiguous x [B, C, Hi, Wi]
InMap up2_map(const float* p, int C, int Hi, int Wi) {
  InMap m{};
  m.p = p, m.bs = (long long)C * Hi * Wi, m.cs = (long long)Hi * Wi, m.rs = Wi, m.H = 2 * Hi, m.W = 2 * Wi;
  m.kind = IN_UP2, m.Hs = Hi, m.Ws = Wi;
  m.sy = (float)(Hi - 1) / (float)(m.H - 1);
  m.sx = (float)(Wi - 1) / (float)(m.W - 1);
  return m;
}

// torch's align_corners=False source index (UpSample.h area_pixel_compute_source_index, scale = in / out)
__device__ __forceinline__ void resize_index(int d, int n_in, float scale, int& i0, int& i1, float& l1) {
  const float src = fmaxf(scale * ((float)d + 0.5f) - 0.5f, 0.f);
  const int f = (int)src;
  l1 = src - (float)f;
  i0 = min(f, n_in - 1);
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
}

// torch's align_corners=True source index (UpSampleKernel: scale = (in-1)/(out-1), i1 clamped at the last row)
__device__ __forceinline__ void up_index(int d, int n_in, float scale, int& i0, int& i1, float& l1) {
  const float src = scale * (float)d;
  i0 = min((int)src, n_in - 1);
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  l1 = fminf(fmaxf(src - (float)i0, 0.f), 1.f);
}

__device__ __forceinline__ float in_at(const InMap& m, int b, int c, int y, int x) {
  const float* p = m.p + b * m.bs + c * m.cs;
  if (m.kind == IN_PLAIN) return p[(size_t)y * m.rs + x];
  int y0, y1, x0, x1;
  float ly, lx;
  if (m.kind == IN_UP2) {
    up_index(y, m.Hs, m.sy, y0, y1, ly);
    up_index(x, m.Ws, m.sx, x0, x1, lx);
  } else {
    resize_index(y, m.Hs, m.sy, y0, y1, ly);
    resize_index(x, m.Ws, m.sx, x0, x1, lx);
  }
  const float a = (1.f - lx) * __ldg(p + (size_t)y0 * m.rs + x0) + lx * __ldg(p + (size_t)y0 * m.rs + x1);
  const float c1 = (1.f - lx) * __ldg(p + (size_t)y1 * m.rs + x0) + lx * __ldg(p + (size_t)y1 * m.rs + x1);
  const float r = (1.f - ly) * a + ly * c1;
  return m.kind == IN_UP2 ? r : r * m.vscale * (float)m.mask[(size_t)y * m.W + x];
}

// in_at with the map's kind fixed at compile time (KIND < 0: read it from the map).  The forward's staging loop is its
// hot loop outside the FMAs; a kind known at compile time keeps the other readers' code out of it.
template <int KIND>
__device__ __forceinline__ float in_at_k(InMap m, int b, int c, int y, int x) {
  if (KIND >= 0) m.kind = KIND;
  return in_at(m, b, c, y, x);
}

// Forward KxK grouped convolution with pad (K-1)/2 and stride S, then the epilogue per output element:
//   r = acc scale[o] + bias, the bias none (bias_mode 0), tied [Cout] (1) or untied [Cout,Ho,Wo] (2);
//   mask (may be NULL) receives r > 0;  act: r = LeakyReLU(r, slope);
//   SKIP: r += scale_r[o] sum_i vr[o,i] xs[b, g cin_g + i, S y, S x] + bias_r[o] (a grouped 1x1 stride-S conv, tied bias).
// Per pixel the sum runs over channel chunks, then taps in (ky, kx) order.  KI / KX: the kinds of `in` / `xs` when
// known at compile time (-1: read from the map).  MIN_CTAS is the launch bound's CTAs per SM:
// 2 for the blocks (up to 128 registers), 0 (no bound) for the single layer, where ptxas then keeps 3 CTAs per SM.
// grid (tiles, groups * cdiv(cout_g, CO_T), B)
template <int CO_T, int K, int S, bool SKIP, int MIN_CTAS, int KI = -1, int KX = -1>
__global__ void __launch_bounds__(TP* TP, MIN_CTAS)
    wn_conv_fwd_kernel(int cin_g, int cout_g, int groups, InMap in, int Ho, int Wo, const float* __restrict__ v,
                       const float* __restrict__ scale, const float* __restrict__ bias, int bias_mode, int act,
                       float slope, InMap xs, const float* __restrict__ vr, const float* __restrict__ scale_r,
                       const float* __restrict__ bias_r, float* __restrict__ out, unsigned char* __restrict__ mask) {
  constexpr int P = (K - 1) / 2, KK = K * K, HALO = (TP - 1) * S + K;
  __shared__ float s_x[CI_CHUNK][HALO][HALO + 1];
  __shared__ float s_w[CI_CHUNK][CO_T][KK];
  const int tiles_x = (Wo + TP - 1) / TP;
  const int ty0 = (blockIdx.x / tiles_x) * TP, tx0 = (blockIdx.x % tiles_x) * TP;
  const int nblk = (cout_g + CO_T - 1) / CO_T;
  const int g = blockIdx.y / nblk, oc0 = (blockIdx.y % nblk) * CO_T, b = blockIdx.z;
  const int Cout = groups * cout_g;
  const int tid = threadIdx.x, py = tid / TP, px = tid % TP;
  float acc[CO_T];
#pragma unroll
  for (int c = 0; c < CO_T; ++c) acc[c] = 0.f;

  for (int i0 = 0; i0 < cin_g; i0 += CI_CHUNK) {
    const int nci = min(CI_CHUNK, cin_g - i0);
    __syncthreads();
#pragma unroll 1
    for (int i = tid; i < nci * HALO * HALO; i += TP * TP) {
      const int ci = i / (HALO * HALO), r = (i / HALO) % HALO, c = i % HALO;
      const int yy = ty0 * S - P + r, xx = tx0 * S - P + c;
      float val = 0.f;
      if (yy >= 0 && yy < in.H && xx >= 0 && xx < in.W) val = in_at_k<KI>(in, b, g * cin_g + i0 + ci, yy, xx);
      s_x[ci][r][c] = val;
    }
    for (int i = tid; i < nci * CO_T * KK; i += TP * TP) {
      const int ci = i / (CO_T * KK), co = (i / KK) % CO_T, k = i % KK;
      float val = 0.f;
      if (oc0 + co < cout_g) val = v[((size_t)(g * cout_g + oc0 + co) * cin_g + (i0 + ci)) * KK + k];
      s_w[ci][co][k] = val;
    }
    __syncthreads();
#pragma unroll 2
    for (int ci = 0; ci < CI_CHUNK; ++ci) {
      if (ci == nci) break;
      float a[KK];
#pragma unroll
      for (int ky = 0; ky < K; ++ky)
#pragma unroll
        for (int kx = 0; kx < K; ++kx) a[ky * K + kx] = s_x[ci][py * S + ky][px * S + kx];
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
  if (y >= Ho || x >= Wo) return;
  float sk[CO_T];
  if (SKIP) {
#pragma unroll
    for (int c = 0; c < CO_T; ++c) sk[c] = 0.f;
    for (int i = 0; i < cin_g; ++i) {
      const float u = in_at_k<KX>(xs, b, g * cin_g + i, y * S, x * S);
#pragma unroll
      for (int c = 0; c < CO_T; ++c) {
        const int oc = min(oc0 + c, cout_g - 1);
        sk[c] += u * __ldg(vr + (size_t)(g * cout_g + oc) * cin_g + i);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < CO_T; ++c) {
    if (oc0 + c >= cout_g) break;
    const int o = g * cout_g + oc0 + c;
    float r = acc[c] * scale[o];
    if (bias_mode == 1) r += bias[o];
    else if (bias_mode == 2) r += bias[((size_t)o * Ho + y) * Wo + x];
    const size_t oi = (((size_t)b * Cout + o) * Ho + y) * Wo + x;
    if (mask) mask[oi] = r > 0.f;
    if (act) r = r > 0.f ? r : r * slope;
    if (SKIP) r += sk[c] * scale_r[o] + bias_r[o];
    out[oi] = r;
  }
}

// Data gradient of a grouped KxK convolution with pad P = (K-1)/2 and stride S, as a gather over the H x W input pixels:
//   out[i,y,x] = sum_{o in group(i)} sum_{ky,kx : S | y+P-ky, S | x+P-kx} gz[o, (y+P-ky)/S, (x+P-kx)/S] scale[o] v[o,i,ky,kx]
//   ACT : multiplied by lrelu'(act_ref[i,y,x]) (act_ref = h1 of a block, so out is conv1's pre-activation gradient)
//   SKIP: (> 0) plus, where SKIP divides y and x, sum_o scale_r[o] vr[o,i] gs[o, y/SKIP, x/SKIP] (the data gradient of
//         a grouped 1x1 stride-SKIP conv with n_skip_g output channels per group)
// With S = 2 a warp holds pixels of one (row, column) parity, so the taps it visits are the same for all its lanes.
// n_res_g / n_sum_g: channels per group of `out` / of gz [B, groups n_sum_g, H/S, W/S].  Items of out and act_ref are
// out_bs floats apart.
template <int CO_T, int K, int S, bool ACT, int SKIP>
__global__ void __launch_bounds__(TP* TP)
    wn_conv_dgrad_kernel(int n_res_g, int n_sum_g, int groups, int H, int W, const float* __restrict__ gz,
                         const float* __restrict__ v, const float* __restrict__ scale,
                         const float* __restrict__ act_ref, float slope, int n_skip_g,
                         const float* __restrict__ gs, const float* __restrict__ vr,
                         const float* __restrict__ scale_r, float* __restrict__ out, long long out_bs) {
  static_assert(S == 1 || K == 3, "a stride-2 data gradient is a 3x3 one");
  constexpr int P = (K - 1) / 2, KK = K * K;
  constexpr int GT = S == 1 ? TP + K - 1 : TP / 2 + 1;
  __shared__ float s_g[CI_CHUNK][GT][GT + 1];
  __shared__ float s_w[CI_CHUNK][CO_T][KK];
  const int Hg = H / S, Wg = W / S;
  const int tiles_x = (W + TP - 1) / TP;
  const int ty0 = (blockIdx.x / tiles_x) * TP, tx0 = (blockIdx.x % tiles_x) * TP;
  const int oy0 = S == 1 ? ty0 - P : ty0 / 2, ox0 = S == 1 ? tx0 - P : tx0 / 2;
  const int nblk = (n_res_g + CO_T - 1) / CO_T;
  const int g = blockIdx.y / nblk, ic0 = (blockIdx.y % nblk) * CO_T, b = blockIdx.z;
  const int n_sum = groups * n_sum_g;
  const int tid = threadIdx.x;
  int py, px;
  if (S == 1) {
    py = tid / TP, px = tid % TP;
  } else {
    const int warp = tid >> 5, q = (warp >> 2) * 32 + (tid & 31);
    py = 2 * (q / 8) + ((warp >> 1) & 1), px = 2 * (q % 8) + (warp & 1);
  }
  const size_t gplane = (size_t)Hg * Wg;
  const float* gzb = gz + ((size_t)b * n_sum + (size_t)g * n_sum_g) * gplane;
  float acc[CO_T];
#pragma unroll
  for (int c = 0; c < CO_T; ++c) acc[c] = 0.f;

  for (int o0 = 0; o0 < n_sum_g; o0 += CI_CHUNK) {
    const int noc = min(CI_CHUNK, n_sum_g - o0);
    __syncthreads();
    for (int i = tid; i < noc * GT * GT; i += TP * TP) {
      const int oc = i / (GT * GT), r = (i / GT) % GT, c = i % GT;
      const int yy = oy0 + r, xx = ox0 + c;
      float val = 0.f;
      if (yy >= 0 && yy < Hg && xx >= 0 && xx < Wg) val = gzb[(size_t)(o0 + oc) * gplane + (size_t)yy * Wg + xx];
      s_g[oc][r][c] = val;
    }
    for (int i = tid; i < noc * CO_T * KK; i += TP * TP) {
      const int oc = i / (CO_T * KK), ic = (i / KK) % CO_T, k = i % KK;
      float val = 0.f;
      if (ic0 + ic < n_res_g) {
        const int o = g * n_sum_g + o0 + oc;
        val = v[((size_t)o * n_res_g + ic0 + ic) * KK + k] * scale[o];
      }
      s_w[oc][ic][k] = val;
    }
    __syncthreads();
    // unrolled x4 at S = 1 (no spills at CO_T = 4), not at S = 2 (spills)
#pragma unroll (S == 1 ? 4 : 1)
    for (int oc = 0; oc < noc; ++oc) {
#pragma unroll
      for (int ky = 0; ky < K; ++ky) {
        // row of gz this tap reads, relative to the staged tile: S = 1: y+P-ky - (ty0-P); S = 2: (y+1-ky)/2 - ty0/2
        const int t = S == 1 ? py + 2 * P - ky : py + 1 - ky;
        if (S == 2 && (t & 1)) continue;
        const int iy = S == 1 ? t : t >> 1;
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
          const int u = S == 1 ? px + 2 * P - kx : px + 1 - kx;
          if (S == 2 && (u & 1)) continue;
          const float gv = s_g[oc][iy][S == 1 ? u : u >> 1];
#pragma unroll
          for (int c = 0; c < CO_T; ++c) acc[c] += gv * s_w[oc][c][ky * K + kx];
        }
      }
    }
  }
  const int y = ty0 + py, x = tx0 + px;
  if (y >= H || x >= W) return;
  if (SKIP && y % SKIP == 0 && x % SKIP == 0) {
    const int Hs = H / SKIP, Ws = W / SKIP;
    const size_t splane = (size_t)Hs * Ws;
    const float* gsb = gs + ((size_t)b * groups * n_skip_g + (size_t)g * n_skip_g) * splane + (size_t)(y / SKIP) * Ws + x / SKIP;
    for (int o = 0; o < n_skip_g; ++o) {
      const int og = g * n_skip_g + o;
      const float gv = gsb[(size_t)o * splane] * scale_r[og];
#pragma unroll
      for (int c = 0; c < CO_T; ++c) {
        const int ic = min(ic0 + c, n_res_g - 1);
        acc[c] += gv * __ldg(vr + (size_t)og * n_res_g + ic);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < CO_T; ++c) {
    if (ic0 + c >= n_res_g) break;
    const size_t oi = (size_t)b * out_bs + ((size_t)(g * n_res_g + ic0 + c) * H + y) * W + x;
    float r = acc[c];
    if (ACT) r = act_ref[oi] > 0.f ? r : r * slope;
    out[oi] = r;
  }
}

// gz = gout * lrelu'(pre-activation), the sign read from the forward's mask or, where none was kept, from the layer's
// output (the same sign when nothing is added after the activation); gbias (may be NULL) = the batch sum of gz, in
// batch order: the untied bias gradient.
__global__ void __launch_bounds__(256)
    act_bwd_kernel(int B, long long per_item, const float* __restrict__ gout, const unsigned char* __restrict__ mask,
                   const float* __restrict__ out, float slope, float* __restrict__ gz, float* __restrict__ gbias) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= per_item) return;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) {
    const size_t o = (size_t)b * per_item + i;
    const float g = gout[o];
    const bool pos = mask ? mask[o] != 0 : out[o] > 0.f;
    const float z = pos ? g : g * slope;
    gz[o] = z;
    acc += z;
  }
  if (gbias) gbias[i] = acc;
}

// the batch sum of g, in batch order: an untied bias gradient
__global__ void __launch_bounds__(256) batch_sum_kernel(int B, long long per_item, const float* __restrict__ g,
                                                        float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= per_item) return;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) acc += g[(size_t)b * per_item + i];
  out[i] = acc;
}

// a tied bias gradient: out[c] = sum_{b,p} g[b,c,p]; one CTA per channel, strided partial sums and a tree in shared
// memory, so the order is fixed
__global__ void __launch_bounds__(256) chan_sum_kernel(int B, int C, int HW, const float* __restrict__ g,
                                                       float* __restrict__ out) {
  __shared__ float s[256];
  const int c = blockIdx.x;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) {
    const float* p = g + ((size_t)b * C + c) * HW;
    for (int i = threadIdx.x; i < HW; i += 256) acc += p[i];
  }
  s[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[c] = s[0];
}

// The end of a weight-gradient CTA of 8 warps whose lanes each hold acc[4][KK] (4 input channels x KK taps of one
// output channel): the warps are added in warp order through s_r [32][4 KK + 1], then every (lane, a, k) sum is handed
// to store(lane, a, k, value), which maps it to its place in the CTA's partial.  The first step begins while other
// warps may still be in their main loop, so s_r must not alias anything they read.
template <int KK, class Store>
__device__ __forceinline__ void store_warp_ordered_sums(const float (&acc)[4][KK], float* s_r, Store store) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int w = 0; w < 8; ++w) {
    if (warp == w) {
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int k = 0; k < KK; ++k) {
          float& r = s_r[lane * (4 * KK + 1) + a * KK + k];
          r = (w ? r : 0.f) + acc[a][k];
        }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < 32 * 4 * KK; i += 256) {
    const int l = i / (4 * KK), a = (i / KK) % 4, k = i % KK;
    store(l, a, k, s_r[l * (4 * KK + 1) + a * KK + k]);
  }
}

// Weight gradient of a grouped KxK convolution with stride S and pad (K-1)/2, at unit scale:
//   gw[o, i_local, ky, kx] = sum_{b,y,x} gz[b,o,y,x] * in[b, g*cin_g + i_local, S y + ky - P, S x + kx - P]
// CTA blockIdx.x sums its share of the (item, tile) list; its eight warps are added in warp order through shared
// memory and the result goes to part[blockIdx.x] ([Cout, cin_g, K, K]); split_sum_kernel adds the parts in order.
// grid (split, cdiv(cin_g, BW_CI), groups * cdiv(cout_g, BW_CO))
constexpr int BW_TX = 16, BW_TY = 8;
constexpr int BW_CI = 16, BW_CO = 8;

template <int K, int S>
__global__ void __launch_bounds__(256)
    wn_conv_wgrad_kernel(int B, int cin_g, int cout_g, int groups, InMap in, int Ho, int Wo,
                         const float* __restrict__ gz, float* __restrict__ part) {
  constexpr int P = (K - 1) / 2, KK = K * K, XW = (BW_TX - 1) * S + K, XH = (BW_TY - 1) * S + K;
  __shared__ float s_x[BW_CI][XH][XW + 1];
  __shared__ float s_g[BW_CO][BW_TX * BW_TY];
  __shared__ float s_r[32][4 * KK + 1];
  const int nblk = (cout_g + BW_CO - 1) / BW_CO;
  const int g = blockIdx.z / nblk, co0 = (blockIdx.z % nblk) * BW_CO, ci0 = blockIdx.y * BW_CI;
  const int Cout = groups * cout_g;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cig = lane >> 3, col = lane & 7;
  const int tiles_x = (Wo + BW_TX - 1) / BW_TX, tiles_y = (Ho + BW_TY - 1) / BW_TY;
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
      const int yy = ty0 * S - P + r, xx = tx0 * S - P + c;
      float val = 0.f;
      if (ci0 + ci < cin_g && yy >= 0 && yy < in.H && xx >= 0 && xx < in.W)
        val = in_at(in, b, g * cin_g + ci0 + ci, yy, xx);
      s_x[ci][r][c] = val;
    }
    for (int i = tid; i < BW_CO * BW_TX * BW_TY; i += 256) {
      const int co = i / (BW_TX * BW_TY), p = i % (BW_TX * BW_TY);
      const int yy = ty0 + p / BW_TX, xx = tx0 + p % BW_TX;
      float val = 0.f;
      if (co0 + co < cout_g && yy < Ho && xx < Wo)
        val = gz[(((size_t)b * Cout + g * cout_g + co0 + co) * Ho + yy) * Wo + xx];
      s_g[co][p] = val;
    }
    __syncthreads();
    for (int pp = 0; pp < (BW_TX * BW_TY) / 8; ++pp) {
      const int p = warp * ((BW_TX * BW_TY) / 8) + pp, py = p / BW_TX, px = p % BW_TX;
      const float gv = s_g[col][p];
#pragma unroll
      for (int ky = 0; ky < K; ++ky)
#pragma unroll
        for (int kx = 0; kx < K; ++kx)
#pragma unroll
          for (int a = 0; a < 4; ++a) acc[a][ky * K + kx] += s_x[cig * 4 + a][py * S + ky][px * S + kx] * gv;
    }
  }
  float* dst = part + (size_t)blockIdx.x * Cout * cin_g * KK;
  store_warp_ordered_sums<KK>(acc, &s_r[0][0], [&](int l, int a, int k, float r) {
    const int ci = ci0 + (l >> 3) * 4 + a, co = co0 + (l & 7);
    if (ci < cin_g && co < cout_g) dst[((size_t)(g * cout_g + co) * cin_g + ci) * KK + k] = r;
  });
}

__global__ void __launch_bounds__(256) split_sum_kernel(int n_split, int n, const float* __restrict__ part,
                                                        float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float acc = 0.f;
  for (int s = 0; s < n_split; ++s) acc += part[(size_t)s * n + i];
  out[i] = acc;
}

// CTAs per (input, output) channel block of the weight gradient: about `per_sm` CTAs per SM in all
int wgrad_split(int B, int cin_g, int cout_g, int groups, int Ho, int Wo, int per_sm) {
  const int total = B * gb::cdiv(Ho, BW_TY) * gb::cdiv(Wo, BW_TX);
  const int pairs = gb::cdiv(cin_g, BW_CI) * groups * gb::cdiv(cout_g, BW_CO);
  return max(1, min(gb::cdiv(gb::kNumSMs * per_sm, pairs), total));
}

// floats of workspace launch_wgrad needs for one weight gradient
size_t wgrad_part_floats(int B, int Cin, int Cout, int groups, int K, int Ho, int Wo, int per_sm) {
  const int cin_g = Cin / groups, cout_g = Cout / groups;
  return (size_t)wgrad_split(B, cin_g, cout_g, groups, Ho, Wo, per_sm) * Cout * cin_g * K * K;
}

// gw [Cout, Cin/groups, K, K] written
template <int K, int S>
[[nodiscard]] int launch_wgrad(int B, int Cin, int Cout, int groups, const InMap& in, int Ho, int Wo, const float* gz, float* gw,
                  float* part, int per_sm, cudaStream_t s) {
  const int cin_g = Cin / groups, cout_g = Cout / groups;
  const int split = wgrad_split(B, cin_g, cout_g, groups, Ho, Wo, per_sm);
  dim3 grid(split, gb::cdiv(cin_g, BW_CI), groups * gb::cdiv(cout_g, BW_CO));
  GB_CUDA(gb::launch<wn_conv_wgrad_kernel<K, S>>(grid, 256, 0, s, B, cin_g, cout_g, groups, in, Ho, Wo, gz, part));
  const int n = Cout * cin_g * K * K;
  return gb::launch<split_sum_kernel>(gb::cdiv(n, 256), 256, 0, s, split, n, part, gw);
}

}  // namespace
