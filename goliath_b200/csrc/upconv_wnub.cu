// goliath_b200/csrc/upconv_wnub.cu — the body decoder's upsampling residual block (blocks.UpConvBlockDeep) with
// grouped, weight-normalised 3x3 convolutions and untied biases, fused with its bilinear x2 upsample and its 1x1 skip
// (sm_90a, fp32 SIMT), forward and backward; and the sparse gathers of the seam sampler and of GeometryModule.from_uv.
//
//   u   = UpsamplingBilinear2d(2 Hi)(x)                                   (align_corners = True)
//   h1  = lrelu(conv1(u) + b1)                                            kernel 1: u is built in shared memory
//   out = lrelu(conv2(h1) + b2) + conv_resize(u) + br                     kernel 2: the skip is recomputed from x
//
// Neither u nor the skip is written to memory.  The trunk blocks of mesh_vae.ConvDecoder run at 128^2..1024^2 with 4-64
// channels per group and untied biases [C,H,W]: the block is bound by the bytes it moves, so the fusion (one pass per
// convolution, no upsample / skip / bias / activation passes) is the optimisation; tensor cores are not used.
//
// The backward needs the sign of conv2's pre-activation, which cannot be read back from `out` because the skip is
// added after the activation; the forward writes it as one byte per output element (`mask`, a quarter of `out`'s
// bytes) when the caller asks for it (training).  h1 is kept by the caller.
#include "common.cuh"

namespace {

constexpr int TP = 16;       // output pixels per CTA edge
constexpr int CI_CHUNK = 8;  // input channels staged per step
constexpr int HALO = TP + 2;

// torch's align_corners=True source index (UpSampleKernel: scale = (in-1)/(out-1), i1 clamped at the last row)
__device__ __forceinline__ void up_index(int d, int n_in, float scale, int& i0, int& i1, float& l1) {
  const float src = scale * (float)d;
  i0 = min((int)src, n_in - 1);
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  l1 = fminf(fmaxf(src - (float)i0, 0.f), 1.f);
}

// one upsampled value u[y,x] of the low-resolution plane xp [Hi,Wi]
__device__ __forceinline__ float up_sample(const float* __restrict__ xp, int Hi, int Wi, float sy, float sx, int y,
                                           int x) {
  int y0, y1, x0, x1;
  float ly, lx;
  up_index(y, Hi, sy, y0, y1, ly);
  up_index(x, Wi, sx, x0, x1, lx);
  const float a = (1.f - lx) * __ldg(xp + y0 * Wi + x0) + lx * __ldg(xp + y0 * Wi + x1);
  const float c = (1.f - lx) * __ldg(xp + y1 * Wi + x0) + lx * __ldg(xp + y1 * Wi + x1);
  return (1.f - ly) * a + ly * c;
}

struct UpGeom {
  int H, W, Hi, Wi;
  float sy, sx;
};

// Forward 3x3 grouped convolution, "same" padding, weight-norm scale, untied bias, LeakyReLU.
//   UP_IN: the input is the low-resolution x, upsampled while it is staged (conv1); else it is h1 at full size (conv2).
//   SKIP : the epilogue adds the grouped 1x1 conv_resize of u (recomputed from x) and its tied bias (conv2).
//   mask (may be NULL) receives pre-activation > 0 per output element.
// grid (tiles, groups * cdiv(cout_g, CO_T), B)
template <int CO_T, bool UP_IN, bool SKIP>
__global__ void __launch_bounds__(TP* TP, 2)
    upconv_fwd_kernel(int cin_g, int cout_g, int groups, UpGeom gm, const float* __restrict__ in,
                      const float* __restrict__ v, const float* __restrict__ scale, const float* __restrict__ bias,
                      float slope, const float* __restrict__ xs, const float* __restrict__ vr,
                      const float* __restrict__ scale_r, const float* __restrict__ bias_r, float* __restrict__ out,
                      unsigned char* __restrict__ mask, size_t in_bs) {
  __shared__ float s_x[CI_CHUNK][HALO][HALO + 1];
  __shared__ float s_w[CI_CHUNK][CO_T][9];
  const int H = gm.H, W = gm.W, Hi = gm.Hi, Wi = gm.Wi;
  const int tiles_x = (W + TP - 1) / TP;
  const int ty0 = (blockIdx.x / tiles_x) * TP, tx0 = (blockIdx.x % tiles_x) * TP;
  const int nblk = (cout_g + CO_T - 1) / CO_T;
  const int g = blockIdx.y / nblk, oc0 = (blockIdx.y % nblk) * CO_T, b = blockIdx.z;
  const int Cin = groups * cin_g, Cout = groups * cout_g;
  const int tid = threadIdx.x, py = tid / TP, px = tid % TP;
  const size_t in_plane = UP_IN ? (size_t)Hi * Wi : (size_t)H * W;
  const float* inb = in + (size_t)b * in_bs + (size_t)g * cin_g * in_plane;
  float acc[CO_T];
#pragma unroll
  for (int c = 0; c < CO_T; ++c) acc[c] = 0.f;

  for (int i0 = 0; i0 < cin_g; i0 += CI_CHUNK) {
    __syncthreads();
#pragma unroll 1
    for (int i = tid; i < CI_CHUNK * HALO * HALO; i += TP * TP) {
      const int ci = i / (HALO * HALO), r = (i / HALO) % HALO, c = i % HALO;
      const int yy = ty0 - 1 + r, xx = tx0 - 1 + c;
      float val = 0.f;
      if (i0 + ci < cin_g && yy >= 0 && yy < H && xx >= 0 && xx < W) {
        const float* p = inb + (size_t)(i0 + ci) * in_plane;
        val = UP_IN ? up_sample(p, Hi, Wi, gm.sy, gm.sx, yy, xx) : p[(size_t)yy * W + xx];
      }
      s_x[ci][r][c] = val;
    }
    for (int i = tid; i < CI_CHUNK * CO_T * 9; i += TP * TP) {
      const int ci = i / (CO_T * 9), co = (i / 9) % CO_T, k = i % 9;
      float val = 0.f;
      if (i0 + ci < cin_g && oc0 + co < cout_g) val = v[((size_t)(g * cout_g + oc0 + co) * cin_g + (i0 + ci)) * 9 + k];
      s_w[ci][co][k] = val;
    }
    __syncthreads();
#pragma unroll 2
    for (int ci = 0; ci < CI_CHUNK; ++ci) {
      float a[9];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) a[ky * 3 + kx] = s_x[ci][py + ky][px + kx];
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
  if (y >= H || x >= W) return;
  float sk[CO_T];
  if (SKIP) {
#pragma unroll
    for (int c = 0; c < CO_T; ++c) sk[c] = 0.f;
    const float* xb = xs + ((size_t)b * Cin + (size_t)g * cin_g) * Hi * Wi;
    for (int i = 0; i < cin_g; ++i) {
      const float u = up_sample(xb + (size_t)i * Hi * Wi, Hi, Wi, gm.sy, gm.sx, y, x);
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
    float r = acc[c] * scale[o] + bias[((size_t)o * H + y) * W + x];
    const size_t oi = (((size_t)b * Cout + o) * H + y) * W + x;
    if (mask) mask[oi] = r > 0.f;
    r = r > 0.f ? r : r * slope;
    if (SKIP) r += sk[c] * scale_r[o] + bias_r[o];
    out[oi] = r;
  }
}

// Data gradient of a grouped 3x3 convolution (the transposed convolution of gz with the flipped kernel):
//   out[i,y,x] = sum_{o in group(i)} sum_k gz[o, y-ky+1, x-kx+1] * scale[o] * v[o, i_local, ky, kx]
//   ACT : multiplied by lrelu'(act_ref[i,y,x]) (act_ref = h1, so out is conv1's pre-activation gradient)
//   SKIP: plus sum_{o in group(i)} scale_r[o] vr[o, i_local] gs[o,y,x] (the 1x1 skip's data gradient)
// n_res_g / n_sum_g: channels per group of `out` / of `gz`; the skip has n_skip_g output channels per group.
template <int CO_T, bool ACT, bool SKIP>
__global__ void __launch_bounds__(TP* TP)
    upconv_dgrad_kernel(int n_res_g, int n_sum_g, int groups, int H, int W, const float* __restrict__ gz,
                        const float* __restrict__ v, const float* __restrict__ scale,
                        const float* __restrict__ act_ref, float slope, int n_skip_g, const float* __restrict__ gs,
                        const float* __restrict__ vr, const float* __restrict__ scale_r, float* __restrict__ out,
                        size_t out_bs) {
  __shared__ float s_x[CI_CHUNK][HALO][HALO + 1];
  __shared__ float s_w[CI_CHUNK][CO_T][9];
  const int tiles_x = (W + TP - 1) / TP;
  const int ty0 = (blockIdx.x / tiles_x) * TP, tx0 = (blockIdx.x % tiles_x) * TP;
  const int nblk = (n_res_g + CO_T - 1) / CO_T;
  const int g = blockIdx.y / nblk, ic0 = (blockIdx.y % nblk) * CO_T, b = blockIdx.z;
  const int n_sum = groups * n_sum_g;
  const int tid = threadIdx.x, py = tid / TP, px = tid % TP;
  const size_t plane = (size_t)H * W;
  const float* gzb = gz + ((size_t)b * n_sum + (size_t)g * n_sum_g) * plane;
  float acc[CO_T];
#pragma unroll
  for (int c = 0; c < CO_T; ++c) acc[c] = 0.f;

  for (int o0 = 0; o0 < n_sum_g; o0 += CI_CHUNK) {
    __syncthreads();
    for (int i = tid; i < CI_CHUNK * HALO * HALO; i += TP * TP) {
      const int oc = i / (HALO * HALO), r = (i / HALO) % HALO, c = i % HALO;
      const int yy = ty0 - 1 + r, xx = tx0 - 1 + c;
      float val = 0.f;
      if (o0 + oc < n_sum_g && yy >= 0 && yy < H && xx >= 0 && xx < W) val = gzb[(size_t)(o0 + oc) * plane + yy * W + xx];
      s_x[oc][r][c] = val;
    }
    for (int i = tid; i < CI_CHUNK * CO_T * 9; i += TP * TP) {
      const int oc = i / (CO_T * 9), ic = (i / 9) % CO_T, k = i % 9;
      float val = 0.f;
      if (o0 + oc < n_sum_g && ic0 + ic < n_res_g) {
        const int o = g * n_sum_g + o0 + oc;
        val = v[((size_t)o * n_res_g + ic0 + ic) * 9 + (8 - k)] * scale[o];
      }
      s_w[oc][ic][k] = val;
    }
    __syncthreads();
#pragma unroll 2
    for (int oc = 0; oc < CI_CHUNK; ++oc) {
      float a[9];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) a[ky * 3 + kx] = s_x[oc][py + ky][px + kx];
#pragma unroll
      for (int c = 0; c < CO_T; ++c) {
        float s = acc[c];
#pragma unroll
        for (int k = 0; k < 9; ++k) s += a[k] * s_w[oc][c][k];
        acc[c] = s;
      }
    }
  }
  const int y = ty0 + py, x = tx0 + px;
  if (y >= H || x >= W) return;
  if (SKIP) {
    const float* gsb = gs + ((size_t)b * groups * n_skip_g + (size_t)g * n_skip_g) * plane + (size_t)y * W + x;
    for (int o = 0; o < n_skip_g; ++o) {
      const int og = g * n_skip_g + o;
      const float gv = gsb[(size_t)o * plane] * scale_r[og];
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

// gz2 = gout * lrelu'(pre-activation) from the forward's mask; untied bias gradient = sum over the batch of gz2; the
// skip's tied bias gradient = per-channel sum of gout (one RED per channel run of a warp).
__global__ void __launch_bounds__(256)
    mask_act_bwd_kernel(int B, int C, int HW, const float* __restrict__ gout, const unsigned char* __restrict__ mask,
                        float slope, float* __restrict__ gz, float* __restrict__ gbias, float* __restrict__ gbias_r) {
  const long long per_item = (long long)C * HW;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float acc = 0.f, acc_r = 0.f;
  if (i < per_item) {
    for (int b = 0; b < B; ++b) {
      const size_t o = (size_t)b * per_item + i;
      const float g = gout[o];
      const float z = mask[o] ? g : g * slope;
      gz[o] = z;
      acc += z;
      acc_r += g;
    }
    gbias[i] = acc;
  }
  const int ch = i < per_item ? (int)(i / HW) : -1;
  const unsigned grp = __match_any_sync(0xffffffffu, ch);
  float tot = 0.f;
  for (int l = 0; l < 32; ++l) {
    const float vv = __shfl_sync(0xffffffffu, acc_r, l);
    if (grp & (1u << l)) tot += vv;
  }
  if (ch >= 0 && (int)(__ffs(grp) - 1) == (int)(threadIdx.x & 31)) gb::red_add(gbias_r + ch, tot);
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

// Weight gradient of a grouped KxK convolution at unit scale, accumulated with REDs:
//   gw[o, i_local, ky, kx] = sum_{b,y,x} gz[b,o,y,x] * in[b, g*cin_g + i_local, y+ky-P, x+kx-P]
// UP_IN: `in` is u, recomputed from the low-resolution x while it is staged.
// grid (split, cdiv(cin_g, BW_CI), groups * cdiv(cout_g, BW_CO))
constexpr int BW_TX = 16, BW_TY = 8;
constexpr int BW_CI = 16, BW_CO = 8;

template <int K, bool UP_IN>
__global__ void __launch_bounds__(256)
    upconv_wgrad_kernel(int B, int cin_g, int cout_g, int groups, UpGeom gm, const float* __restrict__ in,
                        const float* __restrict__ gz, float* __restrict__ gw, size_t in_bs) {
  constexpr int P = (K - 1) / 2, KK = K * K, XW = BW_TX + 2 * P, XH = BW_TY + 2 * P;
  __shared__ float s_x[BW_CI][XH][XW + 1];
  __shared__ float s_g[BW_CO][BW_TX * BW_TY];
  const int H = gm.H, W = gm.W, Hi = gm.Hi, Wi = gm.Wi;
  const int nblk = (cout_g + BW_CO - 1) / BW_CO;
  const int g = blockIdx.z / nblk, co0 = (blockIdx.z % nblk) * BW_CO, ci0 = blockIdx.y * BW_CI;
  const int Cout = groups * cout_g;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cig = lane >> 3, col = lane & 7;
  const int tiles_x = (W + BW_TX - 1) / BW_TX, tiles_y = (H + BW_TY - 1) / BW_TY;
  const int total = B * tiles_x * tiles_y;
  const size_t in_plane = UP_IN ? (size_t)Hi * Wi : (size_t)H * W;
  float acc[4][KK];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int k = 0; k < KK; ++k) acc[a][k] = 0.f;

  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    const int b = t / (tiles_x * tiles_y), tt = t % (tiles_x * tiles_y);
    const int ty0 = (tt / tiles_x) * BW_TY, tx0 = (tt % tiles_x) * BW_TX;
    const float* inb = in + (size_t)b * in_bs + (size_t)g * cin_g * in_plane;
    __syncthreads();
    for (int i = tid; i < BW_CI * XH * XW; i += 256) {
      const int ci = i / (XH * XW), r = (i / XW) % XH, c = i % XW;
      const int yy = ty0 - P + r, xx = tx0 - P + c;
      float val = 0.f;
      if (ci0 + ci < cin_g && yy >= 0 && yy < H && xx >= 0 && xx < W) {
        const float* p = inb + (size_t)(ci0 + ci) * in_plane;
        val = UP_IN ? up_sample(p, Hi, Wi, gm.sy, gm.sx, yy, xx) : p[(size_t)yy * W + xx];
      }
      s_x[ci][r][c] = val;
    }
    for (int i = tid; i < BW_CO * BW_TX * BW_TY; i += 256) {
      const int co = i / (BW_TX * BW_TY), p = i % (BW_TX * BW_TY);
      const int yy = ty0 + p / BW_TX, xx = tx0 + p % BW_TX;
      float val = 0.f;
      if (co0 + co < cout_g && yy < H && xx < W)
        val = gz[(((size_t)b * Cout + g * cout_g + co0 + co) * H + yy) * W + xx];
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
          for (int a = 0; a < 4; ++a) acc[a][ky * K + kx] += s_x[cig * 4 + a][py + ky][px + kx] * gv;
    }
  }
  const int co = co0 + col;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int ci = ci0 + cig * 4 + a;
    if (ci < cin_g && co < cout_g) {
#pragma unroll
      for (int k = 0; k < KK; ++k) gb::red_add(gw + ((size_t)(g * cout_g + co) * cin_g + ci) * KK + k, acc[a][k]);
    }
  }
}

// gx = transpose of the upsample applied to gu, as a gather: low-resolution texel (yi, xi) sums gu over the output
// pixels whose bilinear footprint covers it, with the forward's weights; no atomics, fixed order.
__global__ void __launch_bounds__(256) up_transpose_kernel(long long n, UpGeom gm, const float* __restrict__ gu,
                                                           float* __restrict__ gx) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int H = gm.H, W = gm.W, Hi = gm.Hi, Wi = gm.Wi;
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
void launch_fwd_pair(int B, int Cin, int Cout, int groups, UpGeom gm, const float* x, const float* v1,
                     const float* s1, const float* b1, const float* v2, const float* s2, const float* b2,
                     const float* vr, const float* sr, const float* br, float slope, float* h1, float* out,
                     unsigned char* mask, cudaStream_t s) {
  const int cin_g = Cin / groups, cout_g = Cout / groups;
  const int tiles = gb::cdiv(gm.H, TP) * gb::cdiv(gm.W, TP);
  dim3 g1(tiles, groups * gb::cdiv(cin_g, CO_T), B), g2(tiles, groups * gb::cdiv(cout_g, CO_T), B);
  upconv_fwd_kernel<CO_T, true, false><<<g1, TP * TP, 0, s>>>(cin_g, cin_g, groups, gm, x, v1, s1, b1, slope, nullptr,
                                                                nullptr, nullptr, nullptr, h1, nullptr,
                                                                (size_t)Cin * gm.Hi * gm.Wi);
  upconv_fwd_kernel<CO_T, false, true><<<g2, TP * TP, 0, s>>>(cin_g, cout_g, groups, gm, h1, v2, s2, b2, slope, x, vr,
                                                                sr, br, out, mask,
                                                                (size_t)Cin * gm.H * gm.W);
}

template <int K, bool UP_IN>
void launch_wgrad(int B, int Cin, int Cout, int groups, UpGeom gm, const float* in, const float* gz, float* gw,
                  cudaStream_t s, size_t in_bs = 0) {
  if (!in_bs) in_bs = (size_t)Cin * (UP_IN ? (size_t)gm.Hi * gm.Wi : (size_t)gm.H * gm.W);
  const int cin_g = Cin / groups, cout_g = Cout / groups;
  const int total = B * gb::cdiv(gm.H, BW_TY) * gb::cdiv(gm.W, BW_TX);
  const int pairs = gb::cdiv(cin_g, BW_CI) * groups * gb::cdiv(cout_g, BW_CO);
  int split = gb::cdiv(gb::kNumSMs * 4, pairs);
  split = max(1, min(split, total));
  dim3 grid(split, gb::cdiv(cin_g, BW_CI), groups * gb::cdiv(cout_g, BW_CO));
  upconv_wgrad_kernel<K, UP_IN><<<grid, 256, 0, s>>>(B, cin_g, cout_g, groups, gm, in, gz, gw, in_bs);
}

UpGeom make_geom(int Hi, int Wi) {
  UpGeom gm;
  gm.Hi = Hi, gm.Wi = Wi, gm.H = 2 * Hi, gm.W = 2 * Wi;
  gm.sy = (float)(Hi - 1) / (float)(gm.H - 1);
  gm.sx = (float)(Wi - 1) / (float)(gm.W - 1);
  return gm;
}

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
  const UpGeom gm = make_geom(Hi, Wi);
  if ((Cin / groups) % 8 == 0 && (Cout / groups) % 8 == 0)
    launch_fwd_pair<8>(B, Cin, Cout, groups, gm, x, v1, s1, b1, v2, s2, b2, vr, sr, br, slope, h1, out, mask, s);
  else
    launch_fwd_pair<4>(B, Cin, Cout, groups, gm, x, v1, s1, b1, v2, s2, b2, vr, sr, br, slope, h1, out, mask, s);
  gb::count_launches(2);
  GB_CHECK_LAUNCH();
  return 0;
}

GB_API int gb_upconv_block_bwd(int B, int Cin, int Cout, int groups, int Hi, int Wi, const float* x, const float* v1,
                               const float* s1, const float* v2, const float* s2, const float* vr, const float* sr,
                               const float* h1, const unsigned char* mask, const float* gout, float slope, float* gz2,
                               float* gz1, float* gu, float* gb1, float* gb2, float* gbr, float* gw1, float* gw2,
                               float* gwr, float* gx, void* stream) {
  if (bad_shape(B, Cin, Cout, groups, Hi, Wi)) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const UpGeom gm = make_geom(Hi, Wi);
  const int cin_g = Cin / groups, cout_g = Cout / groups;
  const int HW = gm.H * gm.W;
  const int tiles = gb::cdiv(gm.H, TP) * gb::cdiv(gm.W, TP);
  const long long n_out = (long long)Cout * HW, n_in = (long long)Cin * HW;
  mask_act_bwd_kernel<<<(unsigned)gb::cdiv64(n_out, 256), 256, 0, s>>>(B, Cout, HW, gout, mask, slope, gz2, gb2, gbr);
  // gz1 = conv2^T(gz2) * lrelu'(h1)
  if (cin_g % 8 == 0)
    upconv_dgrad_kernel<8, true, false><<<dim3(tiles, groups * (cin_g / 8), B), TP * TP, 0, s>>>(
        cin_g, cout_g, groups, gm.H, gm.W, gz2, v2, s2, h1, slope, 0, nullptr, nullptr, nullptr, gz1, n_in);
  else
    upconv_dgrad_kernel<4, true, false><<<dim3(tiles, groups * gb::cdiv(cin_g, 4), B), TP * TP, 0, s>>>(
        cin_g, cout_g, groups, gm.H, gm.W, gz2, v2, s2, h1, slope, 0, nullptr, nullptr, nullptr, gz1, n_in);
  batch_sum_kernel<<<(unsigned)gb::cdiv64(n_in, 256), 256, 0, s>>>(B, n_in, gz1, gb1);
  launch_wgrad<3, false>(B, Cin, Cout, groups, gm, h1, gz2, gw2, s);
  launch_wgrad<3, true>(B, Cin, Cin, groups, gm, x, gz1, gw1, s);
  launch_wgrad<1, true>(B, Cin, Cout, groups, gm, x, gout, gwr, s);
  int n = 6;
  if (gx) {
    // gu = conv1^T(gz1) + conv_resize^T(gout), then gx = upsample^T(gu)
    if (cin_g % 8 == 0)
      upconv_dgrad_kernel<8, false, true><<<dim3(tiles, groups * (cin_g / 8), B), TP * TP, 0, s>>>(
          cin_g, cin_g, groups, gm.H, gm.W, gz1, v1, s1, nullptr, slope, cout_g, gout, vr, sr, gu, n_in);
    else
      upconv_dgrad_kernel<4, false, true><<<dim3(tiles, groups * gb::cdiv(cin_g, 4), B), TP * TP, 0, s>>>(
          cin_g, cin_g, groups, gm.H, gm.W, gz1, v1, s1, nullptr, slope, cout_g, gout, vr, sr, gu, n_in);
    const long long nx = (long long)B * Cin * Hi * Wi;
    up_transpose_kernel<<<(unsigned)gb::cdiv64(nx, 256), 256, 0, s>>>(nx, gm, gu, gx);
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

// Conv2dWNUB 3x3 "same" with untied bias and no activation, reading a channel range of a wider map: item b of x (and of
// gx in the backward) starts at b * x_bs floats.  mesh_vae.ConvDecoder's verts_conv / tex_conv read channels [0,4) /
// [4,8) of the seam-sampled 8-channel map this way, with no copy of the slice.
GB_API int gb_conv3x3_ub_slice_fwd(int B, int Cin, int Cout, int H, int W, const float* x, long long x_bs,
                                   const float* v, const float* scale, const float* bias, float* out, void* stream) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || H <= 0 || W <= 0) return (int)cudaErrorInvalidValue;
  UpGeom gm = make_geom(H, W);
  gm.H = H, gm.W = W;
  const int tiles = gb::cdiv(H, TP) * gb::cdiv(W, TP);
  upconv_fwd_kernel<4, false, false><<<dim3(tiles, gb::cdiv(Cout, 4), B), TP * TP, 0, (cudaStream_t)stream>>>(
      Cin, Cout, 1, gm, x, v, scale, bias, 1.f, nullptr, nullptr, nullptr, nullptr, out, nullptr, (size_t)x_bs);
  gb::count_launches(1);
  GB_CHECK_LAUNCH();
  return 0;
}

// backward of the above: g_bias [Cout,H,W] written (batch sum of gout); gw [Cout,Cin,3,3] ACCUMULATED at unit scale;
// gx (items x_bs floats apart) written for channels [0,Cin) of each item, or NULL.
GB_API int gb_conv3x3_ub_slice_bwd(int B, int Cin, int Cout, int H, int W, const float* x, long long x_bs,
                                   const float* v, const float* scale, const float* gout, float* g_bias, float* gx,
                                   float* gw, void* stream) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || H <= 0 || W <= 0) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  UpGeom gm = make_geom(H, W);
  gm.H = H, gm.W = W;
  const long long per_item = (long long)Cout * H * W;
  batch_sum_kernel<<<(unsigned)gb::cdiv64(per_item, 256), 256, 0, s>>>(B, per_item, gout, g_bias);
  launch_wgrad<3, false>(B, Cin, Cout, 1, gm, x, gout, gw, s, (size_t)x_bs);
  int n = 2;
  if (gx) {
    const int tiles = gb::cdiv(H, TP) * gb::cdiv(W, TP);
    upconv_dgrad_kernel<4, false, false><<<dim3(tiles, gb::cdiv(Cin, 4), B), TP * TP, 0, s>>>(
        Cin, Cout, 1, H, W, gout, v, scale, nullptr, 1.f, 0, nullptr, nullptr, nullptr, gx, (size_t)x_bs);
    ++n;
  }
  gb::count_launches(n);
  GB_CHECK_LAUNCH();
  return 0;
}
