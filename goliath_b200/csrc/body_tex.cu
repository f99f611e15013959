// goliath_b200/csrc/body_tex.cu — the 2048^2 texture composite of the body avatar (sm_90a), forward and backward.
//
// Replaces the middle of mesh_vae.AutoEncoder.forward_tex (ca_code/models/mesh_vae.py:211-222) together with the end of
// UpscaleNet.forward (mesh_vae.py:670-678):
//   P = ((U(T1) + PS(out_block(h))) * tex_std + tex_mean) * S3
// with T1 [B,3,H,W] the seam-sampled low-resolution texture, U torch's bilinear x2 upsample (align_corners=False),
// h [B,4,H,W] the output of UpscaleNet.conv_block, out_block a 4 -> 12 1x1 weight-normalised convolution with an untied
// bias [12,H,W], PS = PixelShuffle(2), tex_mean [1,3,2H,2W] and S3 [B,1,2H,2W] the seam-sampled shadow map.  In
// torch this is a dozen passes over [B,3,2H,2W] maps; here neither z = out_block(h), nor U(T1), nor the pre-shadow
// texture is written.
//
// Layout: one thread per low-resolution texel (i, j), looping over the batch.  The thread owns the 2x2 block of
// high-resolution texels (2i+dy, 2j+dx) that PixelShuffle fills from z[:, 4c+2dy+dx, i, j], so it reads h and the 12
// biases once, reads the 12 tex_mean values once for all items, and writes each output row as float2.  CTAs are
// 32 x 8 texel tiles: a warp covers 32 consecutive texels of one row, so the 3x3 neighbourhood of T1 that the upsample
// reads is shared through L1 by the lanes and the warps of the tile.
//
// Backward: the same thread recomputes the pre-shadow value of its 2x2 block from T1, h and the weights (nothing of
// size [B,3,2H,2W] is kept for autograd) and writes g_S3, g_h and the batch-summed g_bias.  g_T1 is a gather over the
// upsample's footprint: the 2H rows that read low-resolution row i are 2i-1 .. 2i+2 (the same along x), so the thread
// reads g_P * S3 on that 4x4 window and weights each texel with the coefficients the forward gave it — no atomics.
// g_w [12,4] (gradient of the effective weight at unit scale) is a reduction over B*H*W terms: per-thread sums in
// batch order, then a fixed-order warp and CTA reduction into one partial per CTA, then one ordered pass over the
// partials, so two backward calls are bitwise equal.
#include "common.cuh"

namespace {

constexpr int TX = 32, TY = 8, NT = TX * TY;  // CTA tile of low-resolution texels
constexpr int NC = 3, NK = 4, NO = 12;         // texture channels, conv_block features, out_block channels

struct Lerp {
  int i0, i1;
  float l;  // weight of i1
};

// torch's upsample_bilinear2d source index for scale 2, align_corners=False (area_pixel_compute_source_index)
__device__ __forceinline__ Lerp up_src(int o, int n) {
  float r = 0.5f * ((float)o + 0.5f) - 0.5f;
  r = r < 0.f ? 0.f : r;
  Lerp s;
  s.i0 = (int)r;
  s.i1 = s.i0 + (s.i0 < n - 1 ? 1 : 0);
  s.l = r - (float)s.i0;
  return s;
}

// weight with which high-resolution row o reads low-resolution row i
__device__ __forceinline__ float up_weight(int o, int n, int i) {
  const Lerp s = up_src(o, n);
  return (s.i0 == i ? 1.f - s.l : 0.f) + (s.i1 == i ? s.l : 0.f);
}

__device__ __forceinline__ void load_weights(const float* __restrict__ v, const float* __restrict__ scale,
                                             float* s_w /* [NO][NK] effective */) {
  for (int t = threadIdx.y * TX + threadIdx.x; t < NO * NK; t += NT) s_w[t] = v[t] * scale[t / NK];
}

// pre-shadow value of the 2x2 block of (i, j) for item b: pre[c][dy][dx]
__device__ __forceinline__ void pre_shadow(int H, int W, int i, int j, const float* __restrict__ t1b,
                                           const float* __restrict__ hb, const float* __restrict__ s_w,
                                           const float* bias_r, const float* mean_r, float tex_std,
                                           float pre[NC][2][2]) {
  const size_t HW = (size_t)H * W, p = (size_t)i * W + j;
  float hv[NK];
#pragma unroll
  for (int k = 0; k < NK; ++k) hv[k] = hb[k * HW + p];
  Lerp ly[2], lx[2];
#pragma unroll
  for (int d = 0; d < 2; ++d) {
    ly[d] = up_src(2 * i + d, H);
    lx[d] = up_src(2 * j + d, W);
  }
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const float* t = t1b + c * HW;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const float* r0 = t + (size_t)ly[dy].i0 * W;
      const float* r1 = t + (size_t)ly[dy].i1 * W;
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const Lerp& sx = lx[dx];
        const float top = (1.f - sx.l) * r0[sx.i0] + sx.l * r0[sx.i1];
        const float bot = (1.f - sx.l) * r1[sx.i0] + sx.l * r1[sx.i1];
        const float u = (1.f - ly[dy].l) * top + ly[dy].l * bot;
        const int o = 4 * c + 2 * dy + dx;
        float z = bias_r[o];
#pragma unroll
        for (int k = 0; k < NK; ++k) z += s_w[o * NK + k] * hv[k];
        pre[c][dy][dx] = (u + z) * tex_std + mean_r[o];
      }
    }
  }
}

__global__ void __launch_bounds__(NT, 2) body_tex_compose_fwd_kernel(
    int B, int H, int W, const float* __restrict__ t1, const float* __restrict__ h, const float* __restrict__ v,
    const float* __restrict__ scale, const float* __restrict__ bias, float tex_std, const float* __restrict__ tex_mean,
    const float* __restrict__ s3, float* __restrict__ out) {
  __shared__ float s_w[NO * NK];
  load_weights(v, scale, s_w);
  __syncthreads();
  const int j = blockIdx.x * TX + threadIdx.x, i = blockIdx.y * TY + threadIdx.y;
  if (i >= H || j >= W) return;
  const size_t HW = (size_t)H * W, W2 = 2 * (size_t)W, HW4 = 4 * HW;
  float bias_r[NO], mean_r[NO];
#pragma unroll
  for (int o = 0; o < NO; ++o) bias_r[o] = bias[o * HW + (size_t)i * W + j];
#pragma unroll
  for (int c = 0; c < NC; ++c)
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const float2 m = *reinterpret_cast<const float2*>(tex_mean + c * HW4 + (2 * i + dy) * W2 + 2 * j);
      mean_r[4 * c + 2 * dy] = m.x;
      mean_r[4 * c + 2 * dy + 1] = m.y;
    }
  for (int b = 0; b < B; ++b) {
    float pre[NC][2][2];
    pre_shadow(H, W, i, j, t1 + (size_t)b * NC * HW, h + (size_t)b * NK * HW, s_w, bias_r, mean_r, tex_std, pre);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const size_t q = (2 * i + dy) * W2 + 2 * j;
      const float2 s = *reinterpret_cast<const float2*>(s3 + b * HW4 + q);
#pragma unroll
      for (int c = 0; c < NC; ++c)
        *reinterpret_cast<float2*>(out + ((size_t)b * NC + c) * HW4 + q) =
            make_float2(pre[c][dy][0] * s.x, pre[c][dy][1] * s.y);
    }
  }
}

__global__ void __launch_bounds__(NT, 1) body_tex_compose_bwd_kernel(
    int B, int H, int W, const float* __restrict__ t1, const float* __restrict__ h, const float* __restrict__ v,
    const float* __restrict__ scale, const float* __restrict__ bias, float tex_std, const float* __restrict__ tex_mean,
    const float* __restrict__ s3, const float* __restrict__ gp, float* __restrict__ g_t1, float* __restrict__ g_h,
    float* __restrict__ g_bias, float* __restrict__ g_s3, float* __restrict__ partials /* [nCTA][NO*NK] */) {
  __shared__ float s_w[NO * NK];
  __shared__ float s_red[NT / 32][NO * NK];
  load_weights(v, scale, s_w);
  __syncthreads();
  const int j = blockIdx.x * TX + threadIdx.x, i = blockIdx.y * TY + threadIdx.y;
  const bool live = i < H && j < W;
  const size_t HW = (size_t)H * W, W2 = 2 * (size_t)W, HW4 = 4 * HW;
  float gw[NO][NK];
#pragma unroll
  for (int o = 0; o < NO; ++o)
#pragma unroll
    for (int k = 0; k < NK; ++k) gw[o][k] = 0.f;

  if (live) {
    const size_t p = (size_t)i * W + j;
    float bias_r[NO], mean_r[NO], gb[NO];
#pragma unroll
    for (int o = 0; o < NO; ++o) {
      bias_r[o] = bias[o * HW + p];
      gb[o] = 0.f;
    }
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int dy = 0; dy < 2; ++dy) {
        const float2 m = *reinterpret_cast<const float2*>(tex_mean + c * HW4 + (2 * i + dy) * W2 + 2 * j);
        mean_r[4 * c + 2 * dy] = m.x;
        mean_r[4 * c + 2 * dy + 1] = m.y;
      }
    // the footprint of (i, j) in the upsample: rows / cols 2i-1 .. 2i+2 inside the map, and their weights
    float wy[4], wx[4];
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const int y = 2 * i - 1 + d, x = 2 * j - 1 + d;
      wy[d] = (y >= 0 && y < 2 * H) ? up_weight(y, H, i) : 0.f;
      wx[d] = (x >= 0 && x < 2 * W) ? up_weight(x, W, j) : 0.f;
    }
    for (int b = 0; b < B; ++b) {
      const float* hb = h + (size_t)b * NK * HW;
      float pre[NC][2][2];
      pre_shadow(H, W, i, j, t1 + (size_t)b * NC * HW, hb, s_w, bias_r, mean_r, tex_std, pre);
      float gz[NO];
#pragma unroll
      for (int dy = 0; dy < 2; ++dy) {
        const size_t q = (2 * i + dy) * W2 + 2 * j;
        const float2 s = *reinterpret_cast<const float2*>(s3 + b * HW4 + q);
        float gs0 = 0.f, gs1 = 0.f;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const float2 g = *reinterpret_cast<const float2*>(gp + ((size_t)b * NC + c) * HW4 + q);
          gs0 += g.x * pre[c][dy][0];
          gs1 += g.y * pre[c][dy][1];
          gz[4 * c + 2 * dy] = g.x * s.x * tex_std;
          gz[4 * c + 2 * dy + 1] = g.y * s.y * tex_std;
        }
        *reinterpret_cast<float2*>(g_s3 + b * HW4 + q) = make_float2(gs0, gs1);
      }
      float hv[NK];
#pragma unroll
      for (int k = 0; k < NK; ++k) hv[k] = hb[k * HW + p];
#pragma unroll
      for (int k = 0; k < NK; ++k) {
        float a = 0.f;
#pragma unroll
        for (int o = 0; o < NO; ++o) a += s_w[o * NK + k] * gz[o];
        g_h[((size_t)b * NK + k) * HW + p] = a;
      }
#pragma unroll
      for (int o = 0; o < NO; ++o) {
        gb[o] += gz[o];
#pragma unroll
        for (int k = 0; k < NK; ++k) gw[o][k] += gz[o] * hv[k];
      }
      // g_T1: gather of g_P * S3 * tex_std over the 4x4 footprint
      float gt[NC] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int dy = 0; dy < 4; ++dy) {
        if (wy[dy] == 0.f) continue;
        const size_t row = (size_t)(2 * i - 1 + dy) * W2;
        float acc[NC] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int dx = 0; dx < 4; ++dx) {
          if (wx[dx] == 0.f) continue;
          const size_t q = row + (2 * j - 1 + dx);
          const float s = s3[b * HW4 + q] * wx[dx];
#pragma unroll
          for (int c = 0; c < NC; ++c) acc[c] += gp[((size_t)b * NC + c) * HW4 + q] * s;
        }
#pragma unroll
        for (int c = 0; c < NC; ++c) gt[c] += wy[dy] * acc[c];
      }
#pragma unroll
      for (int c = 0; c < NC; ++c) g_t1[((size_t)b * NC + c) * HW + p] = gt[c] * tex_std;
    }
#pragma unroll
    for (int o = 0; o < NO; ++o) g_bias[o * HW + p] = gb[o];
  }

  // fixed-order reduction of gw: butterfly within the warp, then warps in index order
  const int tid = threadIdx.y * TX + threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int o = 0; o < NO; ++o)
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      float a = gw[o][k];
#pragma unroll
      for (int m = 16; m > 0; m >>= 1) a += __shfl_xor_sync(0xffffffffu, a, m);
      if (lane == 0) s_red[warp][o * NK + k] = a;
    }
  __syncthreads();
  if (tid < NO * NK) {
    float a = 0.f;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) a += s_red[w][tid];
    partials[(size_t)(blockIdx.y * gridDim.x + blockIdx.x) * (NO * NK) + tid] = a;
  }
}

// one warp per weight entry: lanes sum strided partials in index order, then a butterfly; g_w accumulated
__global__ void __launch_bounds__(NO * NK * 32 / 4) body_tex_gw_reduce_kernel(int n_cta, const float* __restrict__ partials,
                                                                              float* __restrict__ g_w) {
  const int lane = threadIdx.x & 31;
  const int e = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (e >= NO * NK) return;
  float a = 0.f;
  for (int c = lane; c < n_cta; c += 32) a += partials[(size_t)c * (NO * NK) + e];
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) a += __shfl_xor_sync(0xffffffffu, a, m);
  if (lane == 0) g_w[e] += a;
}

inline dim3 grid_of(int H, int W) { return dim3(gb::cdiv(W, TX), gb::cdiv(H, TY)); }

}  // namespace

GB_API size_t gb_body_tex_compose_workspace_bytes(int H, int W) {
  if (H <= 0 || W <= 0) return 0;
  const dim3 g = grid_of(H, W);
  return (size_t)g.x * g.y * NO * NK * sizeof(float);
}

GB_API int gb_body_tex_compose_fwd(int B, int H, int W, const float* t1, const float* h, const float* v,
                                   const float* scale, const float* bias, float tex_std, const float* tex_mean,
                                   const float* s3, float* out, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  return gb::launch<body_tex_compose_fwd_kernel>(grid_of(H, W), dim3(TX, TY), 0, (cudaStream_t)stream,
      B, H, W, t1, h, v, scale, bias, tex_std, tex_mean, s3, out);
}

GB_API int gb_body_tex_compose_bwd(int B, int H, int W, const float* t1, const float* h, const float* v,
                                   const float* scale, const float* bias, float tex_std, const float* tex_mean,
                                   const float* s3, const float* g_out, float* g_t1, float* g_h, float* g_bias,
                                   float* g_w, float* g_s3, float* workspace, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 g = grid_of(H, W);
  GB_CUDA(gb::launch<body_tex_compose_bwd_kernel>(g, dim3(TX, TY), 0, s, B, H, W, t1, h, v, scale, bias, tex_std,
                                                  tex_mean, s3, g_out, g_t1, g_h, g_bias, g_s3, workspace));
  constexpr int warps = NO * NK / 4;  // 4 CTAs of 12 warps
  return gb::launch<body_tex_gw_reduce_kernel>(gb::cdiv(NO * NK, warps), warps * 32, 0, s, (int)(g.x * g.y), workspace,
                                               g_w);
}
