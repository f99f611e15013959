// goliath_b200/csrc/downconv_wnub.cu — the body encoders' downsampling residual block (blocks.ConvDownBlock) with
// grouped, weight-normalised convolutions and untied biases (sm_90a, fp32 SIMT), forward and backward.
//
//   h1  = lrelu(conv1(x) + b1)                                   kernel 1: 3x3, stride 1, "same"
//   out = lrelu(conv2(h1) + b2) + conv_resize(x) + br            kernel 2: 3x3, stride 2, pad 1; the 1x1 stride-2 skip
//                                                                is computed from x[:, :, ::2, ::2] in the epilogue
//
// The skip is never written.  The first block of mesh_vae.Encoder reads its input through `InMap`: the bilinear resize
// (align_corners = False) of a strided window of the UV position map, times verts_scale and the encoder's boolean
// mask, evaluated while a tile is staged, so the conditioned [B,3,512,512] map is never written either.
//
// As in upconv_wnub.cu the backward needs the sign of conv2's pre-activation, which cannot be read back from `out`
// because the skip is added after the activation; the forward writes it as one byte per output element (`mask`) when
// the caller asks for it.  h1 is kept by the caller.
//
// The backward is gather-only and sums in a fixed order, so two runs give the same bits: the data gradient of the
// stride-2 convolution visits, per input pixel, the taps whose parity reaches an output pixel; the weight gradients are
// reduced across warps and across CTAs in index order through a workspace, not with atomics.
#include "common.cuh"

namespace {

constexpr int TP = 16;       // output pixels per CTA edge
constexpr int CI_CHUNK = 8;  // input channels staged per step

// A block's input x [B, C, H, W] as the kernels read it.  Plain: element (b, c, y, x) is p[b bs + c cs + y rs + x].
// Conditioned (mask != NULL): p addresses a [B, C, Hs, Ws] window with the same strides, and
//   x[b, c, y, x] = vscale * bilinear(window -> H x W)[b, c, y, x] * mask[y, x]
struct InMap {
  const float* p;
  long long bs, cs;
  int rs, H, W;
  const unsigned char* mask;
  int Hs, Ws;
  float sy, sx, vscale;
};

// torch's align_corners=False source index (UpSample.h area_pixel_compute_source_index, scale = in / out)
__device__ __forceinline__ void resize_index(int d, int n_in, float scale, int& i0, int& i1, float& l1) {
  const float src = fmaxf(scale * ((float)d + 0.5f) - 0.5f, 0.f);
  const int f = (int)src;
  l1 = src - (float)f;
  i0 = min(f, n_in - 1);
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
}

__device__ __forceinline__ float in_at(const InMap& m, int b, int c, int y, int x) {
  const float* p = m.p + b * m.bs + c * m.cs;
  if (!m.mask) return p[(size_t)y * m.rs + x];
  int y0, y1, x0, x1;
  float ly, lx;
  resize_index(y, m.Hs, m.sy, y0, y1, ly);
  resize_index(x, m.Ws, m.sx, x0, x1, lx);
  const float a = (1.f - lx) * __ldg(p + (size_t)y0 * m.rs + x0) + lx * __ldg(p + (size_t)y0 * m.rs + x1);
  const float c1 = (1.f - lx) * __ldg(p + (size_t)y1 * m.rs + x0) + lx * __ldg(p + (size_t)y1 * m.rs + x1);
  return ((1.f - ly) * a + ly * c1) * m.vscale * (float)m.mask[(size_t)y * m.W + x];
}

// Forward 3x3 grouped convolution with pad 1 and stride S, weight-norm scale, untied bias [Cout,Ho,Wo], LeakyReLU.
//   SKIP: the epilogue adds the grouped 1x1 stride-S conv_resize of xs and its tied bias (conv2).
//   mask (may be NULL) receives pre-activation > 0 per output element.
// grid (tiles, groups * cdiv(cout_g, CO_T), B)
template <int CO_T, int S, bool SKIP>
__global__ void __launch_bounds__(TP* TP, 2)
    down_fwd_kernel(int cin_g, int cout_g, int groups, InMap in, int Ho, int Wo, const float* __restrict__ v,
                    const float* __restrict__ scale, const float* __restrict__ bias, float slope, InMap xs,
                    const float* __restrict__ vr, const float* __restrict__ scale_r,
                    const float* __restrict__ bias_r, float* __restrict__ out, unsigned char* __restrict__ mask) {
  constexpr int HALO = (TP - 1) * S + 3;
  __shared__ float s_x[CI_CHUNK][HALO][HALO + 1];
  __shared__ float s_w[CI_CHUNK][CO_T][9];
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
      const int yy = ty0 * S - 1 + r, xx = tx0 * S - 1 + c;
      float val = 0.f;
      if (yy >= 0 && yy < in.H && xx >= 0 && xx < in.W) val = in_at(in, b, g * cin_g + i0 + ci, yy, xx);
      s_x[ci][r][c] = val;
    }
    for (int i = tid; i < nci * CO_T * 9; i += TP * TP) {
      const int ci = i / (CO_T * 9), co = (i / 9) % CO_T, k = i % 9;
      float val = 0.f;
      if (oc0 + co < cout_g) val = v[((size_t)(g * cout_g + oc0 + co) * cin_g + (i0 + ci)) * 9 + k];
      s_w[ci][co][k] = val;
    }
    __syncthreads();
#pragma unroll 2
    for (int ci = 0; ci < nci; ++ci) {
      float a[9];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) a[ky * 3 + kx] = s_x[ci][py * S + ky][px * S + kx];
#pragma unroll
      for (int c = 0; c < CO_T; ++c) {
        float s = acc[c];
#pragma unroll
        for (int k = 0; k < 9; ++k) s += a[k] * s_w[ci][c][k];
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
      const float u = in_at(xs, b, g * cin_g + i, y * S, x * S);
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
    float r = acc[c] * scale[o] + bias[((size_t)o * Ho + y) * Wo + x];
    const size_t oi = (((size_t)b * Cout + o) * Ho + y) * Wo + x;
    if (mask) mask[oi] = r > 0.f;
    r = r > 0.f ? r : r * slope;
    if (SKIP) r += sk[c] * scale_r[o] + bias_r[o];
    out[oi] = r;
  }
}

// Data gradient of a grouped 3x3 convolution with pad 1 and stride S, as a gather over the H x W input pixels:
//   out[i,y,x] = sum_{o in group(i)} sum_{ky,kx : S | y+1-ky, S | x+1-kx} gz[o, (y+1-ky)/S, (x+1-kx)/S] scale[o] v[o,i,ky,kx]
//   ACT : multiplied by lrelu'(act_ref[i,y,x]) (act_ref = h1, so out is conv1's pre-activation gradient)
//   SKIP: plus, at even (y, x), sum_o scale_r[o] vr[o,i] gs[o, y/2, x/2] (the 1x1 stride-2 skip's data gradient)
// With S = 2 a warp holds pixels of one (row, column) parity, so the taps it visits are the same for all its lanes.
// n_res_g / n_sum_g: channels per group of `out` / of `gz` [B, groups n_sum_g, H/S, W/S].
template <int CO_T, int S, bool ACT, bool SKIP>
__global__ void __launch_bounds__(TP* TP)
    down_dgrad_kernel(int n_res_g, int n_sum_g, int groups, int H, int W, const float* __restrict__ gz,
                      const float* __restrict__ v, const float* __restrict__ scale,
                      const float* __restrict__ act_ref, float slope, int n_skip_g, const float* __restrict__ gs,
                      const float* __restrict__ vr, const float* __restrict__ scale_r, float* __restrict__ out) {
  constexpr int GT = S == 1 ? TP + 2 : TP / 2 + 1;
  __shared__ float s_g[CI_CHUNK][GT][GT + 1];
  __shared__ float s_w[CI_CHUNK][CO_T][9];
  const int Hg = H / S, Wg = W / S;
  const int tiles_x = (W + TP - 1) / TP;
  const int ty0 = (blockIdx.x / tiles_x) * TP, tx0 = (blockIdx.x % tiles_x) * TP;
  const int oy0 = S == 1 ? ty0 - 1 : ty0 / 2, ox0 = S == 1 ? tx0 - 1 : tx0 / 2;
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
    for (int i = tid; i < noc * CO_T * 9; i += TP * TP) {
      const int oc = i / (CO_T * 9), ic = (i / 9) % CO_T, k = i % 9;
      float val = 0.f;
      if (ic0 + ic < n_res_g) {
        const int o = g * n_sum_g + o0 + oc;
        val = v[((size_t)o * n_res_g + ic0 + ic) * 9 + k] * scale[o];
      }
      s_w[oc][ic][k] = val;
    }
    __syncthreads();
    for (int oc = 0; oc < noc; ++oc) {
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        // row of gz this tap reads, relative to the staged tile: S = 1: y+1-ky - (ty0-1); S = 2: (y+1-ky)/2 - ty0/2
        const int t = S == 1 ? py + 2 - ky : py + 1 - ky;
        if (S == 2 && (t & 1)) continue;
        const int iy = S == 1 ? t : t >> 1;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const int u = S == 1 ? px + 2 - kx : px + 1 - kx;
          if (S == 2 && (u & 1)) continue;
          const float gv = s_g[oc][iy][S == 1 ? u : u >> 1];
#pragma unroll
          for (int c = 0; c < CO_T; ++c) acc[c] += gv * s_w[oc][c][ky * 3 + kx];
        }
      }
    }
  }
  const int y = ty0 + py, x = tx0 + px;
  if (y >= H || x >= W) return;
  if (SKIP && !(y & 1) && !(x & 1)) {
    const size_t splane = (size_t)(H / 2) * (W / 2);
    const float* gsb = gs + ((size_t)b * groups * n_skip_g + (size_t)g * n_skip_g) * splane + (size_t)(y / 2) * (W / 2) + x / 2;
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
    const size_t oi = (((size_t)b * groups * n_res_g + g * n_res_g + ic0 + c) * H + y) * W + x;
    float r = acc[c];
    if (ACT) r = act_ref[oi] > 0.f ? r : r * slope;
    out[oi] = r;
  }
}

// gz2 = gout * lrelu'(pre-activation) from the forward's mask; untied bias gradient = sum over the batch of gz2
__global__ void __launch_bounds__(256)
    mask_act_bwd_kernel(int B, long long per_item, const float* __restrict__ gout,
                        const unsigned char* __restrict__ mask, float slope, float* __restrict__ gz,
                        float* __restrict__ gbias) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= per_item) return;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) {
    const size_t o = (size_t)b * per_item + i;
    const float g = gout[o];
    const float z = mask[o] ? g : g * slope;
    gz[o] = z;
    acc += z;
  }
  gbias[i] = acc;
}

// the skip's tied bias gradient: out[c] = sum_{b,p} g[b,c,p]; one CTA per channel, strided partial sums and a tree in
// shared memory, so the order is fixed
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

// untied bias gradient of conv1: the batch sum of its pre-activation gradient, in batch order
__global__ void __launch_bounds__(256) batch_sum_kernel(int B, long long per_item, const float* __restrict__ g,
                                                        float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= per_item) return;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) acc += g[(size_t)b * per_item + i];
  out[i] = acc;
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
    down_wgrad_kernel(int B, int cin_g, int cout_g, int groups, InMap in, int Ho, int Wo,
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
  for (int w = 0; w < 8; ++w) {
    if (warp == w) {
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int k = 0; k < KK; ++k) s_r[lane][a * KK + k] = (w ? s_r[lane][a * KK + k] : 0.f) + acc[a][k];
    }
    __syncthreads();
  }
  float* dst = part + (size_t)blockIdx.x * Cout * cin_g * KK;
  for (int i = tid; i < 32 * 4 * KK; i += 256) {
    const int l = i / (4 * KK), a = (i / KK) % 4, k = i % KK;
    const int ci = ci0 + (l >> 3) * 4 + a, co = co0 + (l & 7);
    if (ci < cin_g && co < cout_g) dst[((size_t)(g * cout_g + co) * cin_g + ci) * KK + k] = s_r[l][a * KK + k];
  }
}

__global__ void __launch_bounds__(256) split_sum_kernel(int n_split, int n, const float* __restrict__ part,
                                                        float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float acc = 0.f;
  for (int s = 0; s < n_split; ++s) acc += part[(size_t)s * n + i];
  out[i] = acc;
}

int wgrad_split(int B, int cin_g, int cout_g, int groups, int Ho, int Wo) {
  const int total = B * gb::cdiv(Ho, BW_TY) * gb::cdiv(Wo, BW_TX);
  const int pairs = gb::cdiv(cin_g, BW_CI) * groups * gb::cdiv(cout_g, BW_CO);
  return max(1, min(gb::cdiv(gb::kNumSMs * 4, pairs), total));
}

template <int K, int S>
void launch_wgrad(int B, int Cin, int Cout, int groups, const InMap& in, int Ho, int Wo, const float* gz, float* gw,
                  float* part, cudaStream_t s) {
  const int cin_g = Cin / groups, cout_g = Cout / groups;
  const int split = wgrad_split(B, cin_g, cout_g, groups, Ho, Wo);
  dim3 grid(split, gb::cdiv(cin_g, BW_CI), groups * gb::cdiv(cout_g, BW_CO));
  down_wgrad_kernel<K, S><<<grid, 256, 0, s>>>(B, cin_g, cout_g, groups, in, Ho, Wo, gz, part);
  const int n = Cout * cin_g * K * K;
  split_sum_kernel<<<gb::cdiv(n, 256), 256, 0, s>>>(split, n, part, gw);
}

InMap plain_map(const float* p, int C, int H, int W) {
  InMap m{};
  m.p = p, m.bs = (long long)C * H * W, m.cs = (long long)H * W, m.rs = W, m.H = H, m.W = W;
  return m;
}

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
  m.mask = a.cond_mask, m.Hs = a.Hs, m.Ws = a.Ws;
  m.sy = (float)a.Hs / (float)a.H, m.sx = (float)a.Ws / (float)a.W, m.vscale = a.cond_scale;
  return m;
}

template <int CO_T>
void launch_conv1(const BlockArgs& a, const InMap& x, const float* v1, const float* s1, const float* b1, float slope,
                  float* h1, cudaStream_t s) {
  const int cin_g = a.Cin / a.groups;
  dim3 grid(gb::cdiv(a.H, TP) * gb::cdiv(a.W, TP), a.groups * gb::cdiv(cin_g, CO_T), a.B);
  down_fwd_kernel<CO_T, 1, false><<<grid, TP * TP, 0, s>>>(cin_g, cin_g, a.groups, x, a.H, a.W, v1, s1, b1, slope, x,
                                                            nullptr, nullptr, nullptr, h1, nullptr);
}

template <int CO_T>
void launch_conv2(const BlockArgs& a, const InMap& x, const float* h1, const float* v2, const float* s2,
                  const float* b2, const float* vr, const float* sr, const float* br, float slope, float* out,
                  unsigned char* mask, cudaStream_t s) {
  const int cin_g = a.Cin / a.groups, cout_g = a.Cout / a.groups, Ho = a.H / 2, Wo = a.W / 2;
  dim3 grid(gb::cdiv(Ho, TP) * gb::cdiv(Wo, TP), a.groups * gb::cdiv(cout_g, CO_T), a.B);
  down_fwd_kernel<CO_T, 2, true><<<grid, TP * TP, 0, s>>>(cin_g, cout_g, a.groups, plain_map(h1, a.Cin, a.H, a.W), Ho,
                                                           Wo, v2, s2, b2, slope, x, vr, sr, br, out, mask);
}

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
    launch_conv1<8>(a, xm, v1, s1, b1, slope, h1, s);
  else
    launch_conv1<4>(a, xm, v1, s1, b1, slope, h1, s);
  if ((Cout / groups) % 8 == 0)
    launch_conv2<8>(a, xm, h1, v2, s2, b2, vr, sr, br, slope, out, mask, s);
  else
    launch_conv2<4>(a, xm, h1, v2, s2, b2, vr, sr, br, slope, out, mask, s);
  gb::count_launches(2);
  GB_CHECK_LAUNCH();
  return 0;
}

GB_API size_t gb_downconv_block_bwd_workspace_bytes(int B, int Cin, int Cout, int groups, int H, int W) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || groups <= 0 || Cin % groups || Cout % groups || H <= 0 || W <= 0) return 0;
  const int cin_g = Cin / groups, cout_g = Cout / groups;
  const size_t w2 = (size_t)wgrad_split(B, cin_g, cout_g, groups, H / 2, W / 2) * Cout * cin_g * 9;
  const size_t w1 = (size_t)wgrad_split(B, cin_g, cin_g, groups, H, W) * Cin * cin_g * 9;
  const size_t wr = (size_t)wgrad_split(B, cin_g, cout_g, groups, H / 2, W / 2) * Cout * cin_g;
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
  const int tiles = gb::cdiv(H, TP) * gb::cdiv(W, TP);
  float* part = (float*)workspace;
  mask_act_bwd_kernel<<<(unsigned)gb::cdiv64(n_out, 256), 256, 0, s>>>(B, n_out, gout, mask, slope, gz2, gb2);
  chan_sum_kernel<<<Cout, 256, 0, s>>>(B, Cout, Ho * Wo, gout, gbr);
  // gz1 = conv2^T(gz2) * lrelu'(h1)
  if (cin_g % 8 == 0)
    down_dgrad_kernel<8, 2, true, false><<<dim3(tiles, groups * (cin_g / 8), B), TP * TP, 0, s>>>(
        cin_g, cout_g, groups, H, W, gz2, v2, s2, h1, slope, 0, nullptr, nullptr, nullptr, gz1);
  else
    down_dgrad_kernel<4, 2, true, false><<<dim3(tiles, groups * gb::cdiv(cin_g, 4), B), TP * TP, 0, s>>>(
        cin_g, cout_g, groups, H, W, gz2, v2, s2, h1, slope, 0, nullptr, nullptr, nullptr, gz1);
  batch_sum_kernel<<<(unsigned)gb::cdiv64(n_in, 256), 256, 0, s>>>(B, n_in, gz1, gb1);
  launch_wgrad<3, 2>(B, Cin, Cout, groups, plain_map(h1, Cin, H, W), Ho, Wo, gz2, gw2, part, s);
  launch_wgrad<3, 1>(B, Cin, Cin, groups, xm, H, W, gz1, gw1, part, s);
  launch_wgrad<1, 2>(B, Cin, Cout, groups, xm, Ho, Wo, gout, gwr, part, s);
  int n = 10;
  if (gx) {
    // gx = conv1^T(gz1) + conv_resize^T(gout)
    if (cin_g % 8 == 0)
      down_dgrad_kernel<8, 1, false, true><<<dim3(tiles, groups * (cin_g / 8), B), TP * TP, 0, s>>>(
          cin_g, cin_g, groups, H, W, gz1, v1, s1, nullptr, slope, cout_g, gout, vr, sr, gx);
    else
      down_dgrad_kernel<4, 1, false, true><<<dim3(tiles, groups * gb::cdiv(cin_g, 4), B), TP * TP, 0, s>>>(
          cin_g, cin_g, groups, H, W, gz1, v1, s1, nullptr, slope, cout_g, gout, vr, sr, gx);
    ++n;
  }
  gb::count_launches(n);
  GB_CHECK_LAUNCH();
  return 0;
}
