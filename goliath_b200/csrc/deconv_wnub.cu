// goliath_b200/csrc/deconv_wnub.cu — stride-2 4x4 transposed convolution with weight-norm scale, untied
// (per-pixel) bias and LeakyReLU fused into the epilogue (sm_90a), forward.
//
// Replaces, for the layer type every RGCA / hand-MVP decoder tower is made of
// (make_conv_trans(.., 4, 2, 1, "wn", LeakyReLU(0.2), ub=(H,W)), ca_code/models/rgca.py:408-456,
// ca_code/nn/layers.py:27-47), the reference's three kernels per layer: cuDNN conv_transpose2d
// (layers.py:380-391), the `output + bias[None]` add (layers.py:392-396) and the in-place LeakyReLU, plus the
// weight-norm reparametrisation w = g * v / ||v||_F (whole-tensor norm, layers.py:200-204, SURVEY.md §0.6), which is
// folded into a per-output-channel scale applied to the accumulator.
//
// Round-1 implementation: fp32 SIMT with the sub-pixel (4-phase) decomposition — each thread owns one input
// position, i.e. a 2x2 output quad, for 8 output channels (32 accumulators); the 3x3 input neighbourhood and the
// 8x16 weights of the current input channel come from shared memory (weights as broadcast float4).  The tensor-core
// phase-GEMM version (3xTF32, TMA-fed: csrc/deconv_tc.cu) serves the inference forward; the last layers are bound by the
// untied-bias + output traffic (1.07 GB for 16->125 @1024^2), not by FLOPs.
#include "wn_conv.cuh"

namespace {

constexpr int TQ = 16;        // quads (input positions) per CTA edge -> 32x32 output tile
constexpr int CO_T = 8;       // output channels per CTA pass
constexpr int TQ_CI = 8;      // input channels staged per step
constexpr int HALO = TQ + 2;

// SCALE_IN = false: the weight-norm scale belongs to the output channel and is applied to the accumulator.
// SCALE_IN = true : it belongs to the INPUT channel (the data gradient of the stride-2 convolution, where the conv's
//                   output channels are this kernel's inputs): the weights are scaled while they are staged.
template <bool SCALE_IN>
__global__ void __launch_bounds__(TQ* TQ) deconv4x4s2_fwd_kernel(
    int Cin, int Cout, int Hi, int Wi, const float* __restrict__ x /* [B,Cin,Hi,Wi] */,
    const float* __restrict__ v /* [Cin,Cout,4,4] */, const float* __restrict__ scale /* [Cout] */,
    const float* __restrict__ bias /* [Cout,2Hi,2Wi] or null */, float slope, int apply_act,
    float* __restrict__ out /* [B,Cout,2Hi,2Wi] */) {
  __shared__ float s_x[TQ_CI][HALO][HALO + 1];
  __shared__ __align__(16) float s_w[TQ_CI][CO_T][16];
  const int tiles_x = (Wi + TQ - 1) / TQ;
  const int tile = blockIdx.x;
  const int ty0 = (tile / tiles_x) * TQ, tx0 = (tile % tiles_x) * TQ;
  const int co0 = blockIdx.y * CO_T;
  const int b = blockIdx.z;
  const int tid = threadIdx.x;
  const int qy = tid / TQ, qx = tid % TQ;
  const int m = ty0 + qy, n = tx0 + qx;  // input position / output quad
  const int Ho = 2 * Hi, Wo = 2 * Wi;

  float acc[CO_T][4];
#pragma unroll
  for (int c = 0; c < CO_T; ++c) { acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f; }

  const float* xb = x + (size_t)b * Cin * Hi * Wi;
  for (int ci0 = 0; ci0 < Cin; ci0 += TQ_CI) {
    __syncthreads();
    // stage the input tile with a 1-pixel halo (zeros outside the image / beyond Cin)
    for (int i = tid; i < TQ_CI * HALO * HALO; i += TQ * TQ) {
      const int ci = i / (HALO * HALO), r = (i / HALO) % HALO, c = i % HALO;
      const int yy = ty0 - 1 + r, xx = tx0 - 1 + c;
      float val = 0.f;
      if (ci0 + ci < Cin && yy >= 0 && yy < Hi && xx >= 0 && xx < Wi) val = xb[((size_t)(ci0 + ci) * Hi + yy) * Wi + xx];
      s_x[ci][r][c] = val;
    }
    // stage the weights of (ci chunk) x (co block): v[ci][co][ky][kx]
    for (int i = tid; i < TQ_CI * CO_T * 16; i += TQ * TQ) {
      const int ci = i / (CO_T * 16), co = (i / 16) % CO_T, k = i % 16;
      float val = 0.f;
      if (ci0 + ci < Cin && co0 + co < Cout) {
        val = v[((size_t)(ci0 + ci) * Cout + (co0 + co)) * 16 + k];
        if (SCALE_IN) val *= scale[ci0 + ci];
      }
      s_w[ci][co][k] = val;
    }
    __syncthreads();
#pragma unroll 2
    for (int ci = 0; ci < TQ_CI; ++ci) {
      // 3x3 neighbourhood of the input position (rows m-1..m+1, cols n-1..n+1)
      const float a00 = s_x[ci][qy][qx], a01 = s_x[ci][qy][qx + 1], a02 = s_x[ci][qy][qx + 2];
      const float a10 = s_x[ci][qy + 1][qx], a11 = s_x[ci][qy + 1][qx + 1], a12 = s_x[ci][qy + 1][qx + 2];
      const float a20 = s_x[ci][qy + 2][qx], a21 = s_x[ci][qy + 2][qx + 1], a22 = s_x[ci][qy + 2][qx + 2];
#pragma unroll
      for (int c = 0; c < CO_T; ++c) {
        const float4 w0 = *reinterpret_cast<const float4*>(&s_w[ci][c][0]);   // ky = 0: kx 0..3
        const float4 w1 = *reinterpret_cast<const float4*>(&s_w[ci][c][4]);   // ky = 1
        const float4 w2 = *reinterpret_cast<const float4*>(&s_w[ci][c][8]);   // ky = 2
        const float4 w3 = *reinterpret_cast<const float4*>(&s_w[ci][c][12]);  // ky = 3
        // out(2m  ,2n  ) = x(m,n) w11 + x(m,n-1) w13 + x(m-1,n) w31 + x(m-1,n-1) w33
        acc[c][0] += a11 * w1.y + a10 * w1.w + a01 * w3.y + a00 * w3.w;
        // out(2m  ,2n+1) = x(m,n+1) w10 + x(m,n) w12 + x(m-1,n+1) w30 + x(m-1,n) w32
        acc[c][1] += a12 * w1.x + a11 * w1.z + a02 * w3.x + a01 * w3.z;
        // out(2m+1,2n  ) = x(m+1,n) w01 + x(m+1,n-1) w03 + x(m,n) w21 + x(m,n-1) w23
        acc[c][2] += a21 * w0.y + a20 * w0.w + a11 * w2.y + a10 * w2.w;
        // out(2m+1,2n+1) = x(m+1,n+1) w00 + x(m+1,n) w02 + x(m,n+1) w20 + x(m,n) w22
        acc[c][3] += a22 * w0.x + a21 * w0.z + a12 * w2.x + a11 * w2.z;
      }
    }
  }
  if (m >= Hi || n >= Wi) return;
#pragma unroll
  for (int c = 0; c < CO_T; ++c) {
    const int co = co0 + c;
    if (co >= Cout) break;
    const float sc = SCALE_IN ? 1.f : scale[co];
    float o00 = acc[c][0] * sc, o01 = acc[c][1] * sc, o10 = acc[c][2] * sc, o11 = acc[c][3] * sc;
    const size_t row0 = ((size_t)co * Ho + 2 * m) * Wo + 2 * n;
    if (bias) {
      const float2 b0 = *reinterpret_cast<const float2*>(bias + row0);
      const float2 b1 = *reinterpret_cast<const float2*>(bias + row0 + Wo);
      o00 += b0.x; o01 += b0.y; o10 += b1.x; o11 += b1.y;
    }
    if (apply_act) {
      o00 = o00 > 0.f ? o00 : o00 * slope; o01 = o01 > 0.f ? o01 : o01 * slope;
      o10 = o10 > 0.f ? o10 : o10 * slope; o11 = o11 > 0.f ? o11 : o11 * slope;
    }
    float* ob = out + (size_t)b * Cout * Ho * Wo;
    *reinterpret_cast<float2*>(ob + row0) = make_float2(o00, o01);
    *reinterpret_cast<float2*>(ob + row0 + Wo) = make_float2(o10, o11);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Wide variant for the high-resolution layers (Cin <= 32: 32->16 @512^2, 16->125 @1024^2 in the RGCA towers, every
// layer of the hand-MVP content decoders).  At 16->125 @1024^2 the kernel above spends most of its instructions on
// shared-memory operand loads and per-co-block input re-staging rather than FMAs, and the epilogue's untied-bias loads
// sit exposed at the end of every CTA.  Here:
//  * a thread owns TWO horizontally adjacent quads (4 consecutive output columns x 2 rows -> 16-byte bias loads/stores);
//  * output channels are processed in PAIRS (ffma2 below): the x operand is stored
//    duplicated in shared memory, the weights as [ci][tap][co] so that a channel pair is one 64-bit operand;
//  * the input tile is staged once per CTA and reused for several blocks of output channels;
//  * the bias of a block is loaded into registers BEFORE its FMA loop (4 channels per block keep that affordable)
//    and its lines are pulled into L2 one block ahead, so no warp waits on HBM in the epilogue.
constexpr int WQ_X = 32, WQ_Y = 16;       // input positions per CTA: 16 rows x 32 columns (256 threads x 2 quads)
constexpr int W_CO = 4, W_CI = 16;
constexpr int W_HX = WQ_X + 2, W_HY = WQ_Y + 2, W_HS = 36;  // halo tile; row stride in float2 (rows 16-byte aligned)

// Hopper has no packed fma.rn.f32x2: a channel pair is two scalar fma.rn on the halves of the 64-bit operands (the
// same rounding, so the results are identical to the packed form)
__device__ __forceinline__ unsigned long long ffma2(unsigned long long a, unsigned long long b, unsigned long long c) {
  unsigned long long d;
  asm("{\n\t.reg .f32 a0, a1, b0, b1, c0, c1;\n\t"
      "mov.b64 {a0, a1}, %1;\n\tmov.b64 {b0, b1}, %2;\n\tmov.b64 {c0, c1}, %3;\n\t"
      "fma.rn.f32 c0, a0, b0, c0;\n\tfma.rn.f32 c1, a1, b1, c1;\n\t"
      "mov.b64 %0, {c0, c1};\n\t}"
      : "=l"(d) : "l"(a), "l"(b), "l"(c));
  return d;
}
__device__ __forceinline__ void cp_async4_zfill(void* smem, const void* gmem, bool valid) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(sa), "l"(gmem), "r"(valid ? 4 : 0) : "memory");
}
__device__ __forceinline__ float2 unpack2(unsigned long long v) {
  float2 r;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v));
  return r;
}

__global__ void __launch_bounds__(256, 2) deconv4x4s2_fwd_wide_kernel(
    int Cin, int Cout, int Hi, int Wi, int co_blocks_per_cta, const float* __restrict__ x, const float* __restrict__ v,
    const float* __restrict__ scale, const float* __restrict__ bias, float slope, int apply_act,
    float* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char wsm[];
  float2* s_x = reinterpret_cast<float2*>(wsm);                                 // [W_CI][W_HY][W_HS] (a, a)
  float* s_w = reinterpret_cast<float*>(wsm + (size_t)W_CI * W_HY * W_HS * 8);  // [2][W_CI][16][W_CO]
  const int tiles_x = (Wi + WQ_X - 1) / WQ_X;
  const int ty0 = (blockIdx.x / tiles_x) * WQ_Y, tx0 = (blockIdx.x % tiles_x) * WQ_X;
  const int b = blockIdx.z;
  const int tid = threadIdx.x, qy = tid >> 4, qx = tid & 15;
  const int m = ty0 + qy, n = tx0 + 2 * qx;  // first of the thread's two positions
  const int Ho = 2 * Hi, Wo = 2 * Wi;
  const float* xb = x + (size_t)b * Cin * Hi * Wi;
  const int nblk = (Cout + W_CO - 1) / W_CO;
  const int blk0 = blockIdx.y * co_blocks_per_cta, blk1 = min(nblk, blk0 + co_blocks_per_cta);
  const bool single_chunk = Cin <= W_CI;
  const bool inside = m < Hi && n < Wi;  // Wi and n are even: both positions are inside together

  // all staging is asynchronous (cp.async, 4-byte granules: the layouts are transposed / duplicated on the fly), so
  // no warp holds registers across a global-memory round trip; out-of-range elements are zero-filled by src-size 0
  auto stage_x = [&](int ci0) {
    for (int i = tid; i < W_CI * W_HY * W_HX; i += 256) {
      const int ci = i / (W_HY * W_HX), r = (i / W_HX) % W_HY, c = i % W_HX;
      const int yy = ty0 - 1 + r, xx = tx0 - 1 + c;
      const bool ok = ci0 + ci < Cin && yy >= 0 && yy < Hi && xx >= 0 && xx < Wi;
      const float* src = ok ? xb + ((size_t)(ci0 + ci) * Hi + yy) * Wi + xx : xb;
      float2* dst = &s_x[(ci * W_HY + r) * W_HS + c];
      cp_async4_zfill(&dst->x, src, ok);
      cp_async4_zfill(&dst->y, src, ok);
    }
  };
  auto stage_w = [&](int buf, int co0, int ci0) {
    float* dstw = s_w + buf * (W_CI * 16 * W_CO);
    for (int i = tid; i < W_CI * 16 * W_CO; i += 256) {
      const int ci = i / (16 * W_CO), co = (i / 16) % W_CO, k = i % 16;  // consecutive lanes read consecutive taps
      const bool ok = ci0 + ci < Cin && co0 + co < Cout;
      const float* src = ok ? v + ((size_t)(ci0 + ci) * Cout + (co0 + co)) * 16 + k : v;
      cp_async4_zfill(dstw + (ci * 16 + k) * W_CO + co, src, ok);
    }
  };
  auto prefetch_bias = [&](int blk) {
    if (!bias || !inside || blk >= blk1) return;
#pragma unroll
    for (int c = 0; c < W_CO; ++c) {
      if (blk * W_CO + c < Cout) {
        const float* bp = bias + ((size_t)(blk * W_CO + c) * Ho + 2 * m) * Wo + 2 * n;
        asm volatile("prefetch.global.L2 [%0];" ::"l"(bp));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(bp + Wo));
      }
    }
  };
  prefetch_bias(blk0);
  if (single_chunk) {
    stage_x(0);
    stage_w(0, blk0 * W_CO, 0);
    gb::cp_async_commit();
  }

  for (int blk = blk0; blk < blk1; ++blk) {
    const int co0 = blk * W_CO;
    prefetch_bias(blk + 1);
    float4 b4[W_CO][2];  // this block's bias, in flight during the FMA loop
#pragma unroll
    for (int c = 0; c < W_CO; ++c)
#pragma unroll
      for (int row = 0; row < 2; ++row) {
        b4[c][row] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (bias && inside && co0 + c < Cout)
          b4[c][row] = gb::ld_nc_f4(reinterpret_cast<const float4*>(bias + ((size_t)(co0 + c) * Ho + 2 * m + row) * Wo + 2 * n));
      }
    unsigned long long acc[2][2][4];  // [co pair][quad][j], j = 2 * row + column inside the quad
#pragma unroll
    for (int cp = 0; cp < 2; ++cp)
#pragma unroll
      for (int q = 0; q < 2; ++q)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[cp][q][j] = 0ull;

    for (int ci0 = 0; ci0 < Cin; ci0 += W_CI) {
      int buf = 0;
      if (single_chunk) {
        // weights of this block were issued one block ago into buffer (blk - blk0) & 1; the x tile at kernel start
        buf = (blk - blk0) & 1;
        gb::cp_async_wait<0>();
        __syncthreads();  // everybody's copies have landed, everybody left the previous block's FMA loop
        if (blk + 1 < blk1) {
          stage_w(buf ^ 1, (blk + 1) * W_CO, 0);
          gb::cp_async_commit();
        }
      } else {
        __syncthreads();  // previous users of s_x / s_w are done
        stage_x(ci0);
        stage_w(0, co0, ci0);
        gb::cp_async_commit();
        gb::cp_async_wait<0>();
        __syncthreads();
      }
      const float* s_wb = s_w + buf * (W_CI * 16 * W_CO);
      const int nci = min(W_CI, Cin - ci0);
#pragma unroll 2
      for (int ci = 0; ci < nci; ++ci) {
        unsigned long long X[3][4];  // rows m-1..m+1, columns n-1..n+2, each value duplicated (a, a)
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const ulonglong2* xp = reinterpret_cast<const ulonglong2*>(&s_x[(ci * W_HY + qy + r) * W_HS + 2 * qx]);
          const ulonglong2 x01 = xp[0], x23 = xp[1];
          X[r][0] = x01.x; X[r][1] = x01.y; X[r][2] = x23.x; X[r][3] = x23.y;
        }
        const ulonglong2* wp = reinterpret_cast<const ulonglong2*>(s_wb + (size_t)ci * 16 * W_CO);
        // one tap = the weights of 4 output channels (one 16-byte broadcast load) feeding one output of each quad
#define GB_TAP(ky, kx, j, r, c)                                      \
  {                                                                  \
    const ulonglong2 wa = wp[(ky) * 4 + (kx)];                       \
    _Pragma("unroll") for (int q = 0; q < 2; ++q) {                  \
      acc[0][q][j] = ffma2(X[r][(c) + q], wa.x, acc[0][q][j]);       \
      acc[1][q][j] = ffma2(X[r][(c) + q], wa.y, acc[1][q][j]);       \
    }                                                                \
  }
        // out(2m  ,2n  ): x(m,n) w11 + x(m,n-1) w13 + x(m-1,n) w31 + x(m-1,n-1) w33
        GB_TAP(1, 1, 0, 1, 1) GB_TAP(1, 3, 0, 1, 0) GB_TAP(3, 1, 0, 0, 1) GB_TAP(3, 3, 0, 0, 0)
        // out(2m  ,2n+1): x(m,n+1) w10 + x(m,n) w12 + x(m-1,n+1) w30 + x(m-1,n) w32
        GB_TAP(1, 0, 1, 1, 2) GB_TAP(1, 2, 1, 1, 1) GB_TAP(3, 0, 1, 0, 2) GB_TAP(3, 2, 1, 0, 1)
        // out(2m+1,2n  ): x(m+1,n) w01 + x(m+1,n-1) w03 + x(m,n) w21 + x(m,n-1) w23
        GB_TAP(0, 1, 2, 2, 1) GB_TAP(0, 3, 2, 2, 0) GB_TAP(2, 1, 2, 1, 1) GB_TAP(2, 3, 2, 1, 0)
        // out(2m+1,2n+1): x(m+1,n+1) w00 + x(m+1,n) w02 + x(m,n+1) w20 + x(m,n) w22
        GB_TAP(0, 0, 3, 2, 2) GB_TAP(0, 2, 3, 2, 1) GB_TAP(2, 0, 3, 1, 2) GB_TAP(2, 2, 3, 1, 1)
#undef GB_TAP
      }
    }
    if (inside) {
      float* ob = out + (size_t)b * Cout * Ho * Wo;
#pragma unroll
      for (int cp = 0; cp < 2; ++cp) {
        float o[2][2][4];  // [co parity][row][x]
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 pr = unpack2(acc[cp][q][j]);
            o[0][j >> 1][2 * q + (j & 1)] = pr.x;
            o[1][j >> 1][2 * q + (j & 1)] = pr.y;
          }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int c = 2 * cp + h, co = co0 + c;
          if (co >= Cout) continue;
          const float sc = scale[co];
#pragma unroll
          for (int row = 0; row < 2; ++row) {
            float4 r4 = make_float4(o[h][row][0] * sc + b4[c][row].x, o[h][row][1] * sc + b4[c][row].y,
                                    o[h][row][2] * sc + b4[c][row].z, o[h][row][3] * sc + b4[c][row].w);
            if (apply_act) {
              r4.x = r4.x > 0.f ? r4.x : r4.x * slope; r4.y = r4.y > 0.f ? r4.y : r4.y * slope;
              r4.z = r4.z > 0.f ? r4.z : r4.z * slope; r4.w = r4.w > 0.f ? r4.w : r4.w * slope;
            }
            *reinterpret_cast<float4*>(ob + ((size_t)co * Ho + 2 * m + row) * Wo + 2 * n) = r4;
          }
        }
      }
    }
  }
}

// The round-1 forward kernel's launch (also the stride-2 convolution's data gradient, SCALE_IN = true)
template <bool SCALE_IN>
[[nodiscard]] int launch_deconv_fwd(int B, int Cin, int Cout, int Hi, int Wi, const float* x, const float* v,
                                    const float* scale, const float* bias, float slope, int apply_act, float* out,
                                    cudaStream_t s) {
  dim3 grid(gb::cdiv(Hi, TQ) * gb::cdiv(Wi, TQ), gb::cdiv(Cout, CO_T), B);
  return gb::launch<deconv4x4s2_fwd_kernel<SCALE_IN>>(grid, TQ * TQ, 0, s, Cin, Cout, Hi, Wi, x, v, scale, bias, slope,
                                                      apply_act, out);
}

}  // namespace

// Fused ConvTranspose2dWNUB(k=4, s=2, p=1) [+ LeakyReLU] forward.  x [B,Cin,Hi,Wi], v = weight_v [Cin,Cout,4,4],
// scale [Cout] = weight_g / ||weight_v||_F, bias [Cout,2Hi,2Wi] or NULL, out [B,Cout,2Hi,2Wi].
// Replaces layers.py:380-396 (+ the activation that follows it in make_conv_trans, layers.py:27-47).
GB_API int gb_deconv4x4s2_wnub_fwd(int B, int Cin, int Cout, int Hi, int Wi, const float* x, const float* v,
                                   const float* scale, const float* bias, float slope, int apply_act, float* out,
                                   void* stream) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || Hi <= 0 || Wi <= 0) return 0;
  if (Cin <= 32 && Wi % 2 == 0 && Wi >= 32 && Hi >= 16) {
    // high-resolution layers: wide kernel, several blocks of output channels per staged input tile
    const int tiles = gb::cdiv(Hi, WQ_Y) * gb::cdiv(Wi, WQ_X);
    const int nblk = gb::cdiv(Cout, W_CO);
    int per_cta = 1;  // grow while the grid still fills the machine a few times over
    while (per_cta < nblk && (long long)tiles * B * gb::cdiv(nblk, per_cta * 2) >= 4LL * 2 * gb::kNumSMs) per_cta *= 2;
    const size_t smem = (size_t)W_CI * W_HY * W_HS * 8 + (size_t)2 * W_CI * 16 * W_CO * 4;
    dim3 grid(tiles, gb::cdiv(nblk, per_cta), B);
    return gb::launch<deconv4x4s2_fwd_wide_kernel>(grid, 256, smem, (cudaStream_t)stream, Cin, Cout, Hi, Wi, per_cta, x,
                                                   v, scale, bias, slope, apply_act, out);
  }
  return launch_deconv_fwd<false>(B, Cin, Cout, Hi, Wi, x, v, scale, bias, slope, apply_act, out, (cudaStream_t)stream);
}

// =====================================================================================================
// Backward (training), all hand-written (no cuDNN), gather-only, every sum in a fixed order:
//   1. act_bwd_kernel (wn_conv.cuh): gz = gout * act'(out) and g_bias = sum_b gz; without an activation gz is gout and
//      g_bias its batch sum (batch_sum_kernel)
//   2. deconv4x4s2_bwd_data_kernel   : gx[ci,y,x] = sum_co scale[co] sum_{ky,kx} gz[co,2y-1+ky,2x-1+kx] v[ci,co,ky,kx]
//   3. deconv4x4s2_bwd_weight_kernel : gw[ci,co,ky,kx] = sum_{b,y,x} x[ci,y,x] gz[co,2y-1+ky,2x-1+kx], as per-CTA
//      partials that split_sum_kernel adds in CTA order
// (gw is the gradient of the EFFECTIVE weight divided by nothing: the weight-norm chain rule on the tiny
//  [Cin,Cout,4,4] tensors is finished by the caller.)
namespace {

constexpr int BD_T = 16;          // input pixels per CTA edge
constexpr int BD_CO = 8;          // output channels staged per step
constexpr int BD_CI = 8;          // input channels per CTA
constexpr int BD_G = 2 * BD_T + 2;  // gz tile edge (34)

// The same gather is the forward of the stride-2 4x4 convolution (gb_conv4x4s2_wnub_fwd): with CONV_FWD the kernel
// reads the conv's input as `gz` (Cout here = the conv's Cin), v [Cin,Cout,4,4] as the conv weight [Cout_conv,Cin_conv,4,4]
// and writes the conv's output as `gx` (Cin here = the conv's Cout).  The weight-norm scale then belongs to the
// OUTPUT channel ci: it is applied to the accumulator, followed by the untied bias [Cin,Hi,Wi] and the activation.
__device__ __forceinline__ float wn_bias_act(float a, float sc, float b, float slope, int apply_act) {
  const float r = a * sc + b;
  return apply_act ? (r > 0.f ? r : r * slope) : r;
}

template <bool CONV_FWD>
__global__ void __launch_bounds__(BD_T* BD_T) deconv4x4s2_bwd_data_kernel(
    int Cin, int Cout, int Hi, int Wi, const float* __restrict__ gz /* [B,Cout,2Hi,2Wi] */,
    const float* __restrict__ v, const float* __restrict__ scale, const float* __restrict__ bias, float slope,
    int apply_act, float* __restrict__ gx /* [B,Cin,Hi,Wi] */) {
  __shared__ float s_g[BD_CO][BD_G][BD_G + 1];
  __shared__ __align__(16) float s_w[BD_CO][BD_CI][16];
  const int tiles_x = (Wi + BD_T - 1) / BD_T;
  const int ty0 = (blockIdx.x / tiles_x) * BD_T, tx0 = (blockIdx.x % tiles_x) * BD_T;
  const int ci0 = blockIdx.y * BD_CI;
  const int b = blockIdx.z;
  const int tid = threadIdx.x, py = tid / BD_T, px = tid % BD_T;
  const int Ho = 2 * Hi, Wo = 2 * Wi;
  const float* gzb = gz + (size_t)b * Cout * Ho * Wo;
  float acc[BD_CI];
#pragma unroll
  for (int c = 0; c < BD_CI; ++c) acc[c] = 0.f;
  for (int co0 = 0; co0 < Cout; co0 += BD_CO) {
    __syncthreads();
    // gz tile: rows 2*ty0-1 .. 2*ty0+2*BD_T, i.e. BD_G rows
    for (int i = tid; i < BD_CO * BD_G * BD_G; i += BD_T * BD_T) {
      const int co = i / (BD_G * BD_G), r = (i / BD_G) % BD_G, c = i % BD_G;
      const int Y = 2 * ty0 - 1 + r, X = 2 * tx0 - 1 + c;
      float val = 0.f;
      if (co0 + co < Cout && Y >= 0 && Y < Ho && X >= 0 && X < Wo) val = gzb[((size_t)(co0 + co) * Ho + Y) * Wo + X];
      s_g[co][r][c] = val;
    }
    for (int i = tid; i < BD_CO * BD_CI * 16; i += BD_T * BD_T) {
      const int co = i / (BD_CI * 16), ci = (i / 16) % BD_CI, k = i % 16;
      float val = 0.f;
      if (co0 + co < Cout && ci0 + ci < Cin) {
        val = v[((size_t)(ci0 + ci) * Cout + (co0 + co)) * 16 + k];
        if (!CONV_FWD) val *= scale[co0 + co];
      }
      s_w[co][ci][k] = val;
    }
    __syncthreads();
#pragma unroll 2
    for (int co = 0; co < BD_CO; ++co) {
      float g[16];  // 4x4 window: rows 2*py .. 2*py+3 of the tile (= 2y-1 .. 2y+2), cols 2*px .. 2*px+3
#pragma unroll
      for (int ky = 0; ky < 4; ++ky)
#pragma unroll
        for (int kx = 0; kx < 4; ++kx) g[ky * 4 + kx] = s_g[co][2 * py + ky][2 * px + kx];
#pragma unroll
      for (int ci = 0; ci < BD_CI; ++ci) {
        const float4 w0 = *reinterpret_cast<const float4*>(&s_w[co][ci][0]);
        const float4 w1 = *reinterpret_cast<const float4*>(&s_w[co][ci][4]);
        const float4 w2 = *reinterpret_cast<const float4*>(&s_w[co][ci][8]);
        const float4 w3 = *reinterpret_cast<const float4*>(&s_w[co][ci][12]);
        acc[ci] += g[0] * w0.x + g[1] * w0.y + g[2] * w0.z + g[3] * w0.w + g[4] * w1.x + g[5] * w1.y + g[6] * w1.z +
                   g[7] * w1.w + g[8] * w2.x + g[9] * w2.y + g[10] * w2.z + g[11] * w2.w + g[12] * w3.x + g[13] * w3.y +
                   g[14] * w3.z + g[15] * w3.w;
      }
    }
  }
  const int y = ty0 + py, x = tx0 + px;
  if (y >= Hi || x >= Wi) return;
#pragma unroll
  for (int ci = 0; ci < BD_CI; ++ci) {
    if (ci0 + ci >= Cin) continue;
    float r = acc[ci];
    if (CONV_FWD)
      r = wn_bias_act(r, scale[ci0 + ci], bias ? bias[((size_t)(ci0 + ci) * Hi + y) * Wi + x] : 0.f, slope, apply_act);
    gx[(((size_t)b * Cin + ci0 + ci) * Hi + y) * Wi + x] = r;
  }
}

// weight gradient: warp tile = 16 ci x 8 co (lane: cig = lane>>3 -> 4 ci, co = lane&7 -> 16 taps), 8 warps split the
// pixels of each staged 16x16 input tile; every CTA walks many tiles, adds its warps in order and writes its sums to
// part[blockIdx.x] ([Cin, Cout, 4, 4]).
constexpr int NW_TX = 16, NW_TY = 8;            // input tile staged per step: 8 rows x 16 columns = 128 pixels
constexpr int NW_CI = 16;
constexpr int NW_CO = 8;
constexpr int NW_GX = 2 * NW_TX + 2, NW_GY = 2 * NW_TY + 2;
static_assert(NW_TX == BW_TX && NW_TY == BW_TY && NW_CI == BW_CI && NW_CO == BW_CO,
              "wgrad_split sizes this kernel's grid with wn_conv.cuh's weight-gradient tile");

__global__ void __launch_bounds__(256) deconv4x4s2_bwd_weight_kernel(
    int B, int Cin, int Cout, int Hi, int Wi, const float* __restrict__ x, const float* __restrict__ gz,
    float* __restrict__ part /* [gridDim.x][Cin,Cout,4,4] */) {
  __shared__ float s_x[NW_CI][NW_TX * NW_TY];
  __shared__ float s_g[NW_CO][NW_GY][NW_GX + 1];
  __shared__ float s_r[32 * (4 * 16 + 1)];
  const int ci0 = blockIdx.y * NW_CI, co0 = blockIdx.z * NW_CO;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cig = lane >> 3, col = lane & 7;
  const int Ho = 2 * Hi, Wo = 2 * Wi;
  const int tiles_x = (Wi + NW_TX - 1) / NW_TX, tiles_y = (Hi + NW_TY - 1) / NW_TY;
  const int total = B * tiles_x * tiles_y;
  float acc[4][16];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int k = 0; k < 16; ++k) acc[a][k] = 0.f;

  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    const int b = t / (tiles_x * tiles_y), tt = t % (tiles_x * tiles_y);
    const int ty0 = (tt / tiles_x) * NW_TY, tx0 = (tt % tiles_x) * NW_TX;
    __syncthreads();
    for (int i = tid; i < NW_CI * NW_TX * NW_TY; i += 256) {
      const int ci = i / (NW_TX * NW_TY), p = i % (NW_TX * NW_TY);
      const int yy = ty0 + p / NW_TX, xx = tx0 + p % NW_TX;
      float val = 0.f;
      if (ci0 + ci < Cin && yy < Hi && xx < Wi) val = x[(((size_t)b * Cin + ci0 + ci) * Hi + yy) * Wi + xx];
      s_x[ci][p] = val;
    }
    for (int i = tid; i < NW_CO * NW_GY * NW_GX; i += 256) {
      const int co = i / (NW_GY * NW_GX), r = (i / NW_GX) % NW_GY, c = i % NW_GX;
      const int Y = 2 * ty0 - 1 + r, X = 2 * tx0 - 1 + c;
      float val = 0.f;
      if (co0 + co < Cout && Y >= 0 && Y < Ho && X >= 0 && X < Wo) val = gz[(((size_t)b * Cout + co0 + co) * Ho + Y) * Wo + X];
      s_g[co][r][c] = val;
    }
    __syncthreads();
    // this warp's 16 pixels of the tile (one row)
    for (int pp = 0; pp < (NW_TX * NW_TY) / 8; ++pp) {
      const int p = warp * ((NW_TX * NW_TY) / 8) + pp, py = p / NW_TX, px = p % NW_TX;
      float xv[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) xv[a] = s_x[cig * 4 + a][p];
#pragma unroll
      for (int ky = 0; ky < 4; ++ky)
#pragma unroll
        for (int kx = 0; kx < 4; ++kx) {
          const float g = s_g[col][2 * py + ky][2 * px + kx];
#pragma unroll
          for (int a = 0; a < 4; ++a) acc[a][ky * 4 + kx] += xv[a] * g;
        }
    }
  }
  float* dst = part + (size_t)blockIdx.x * Cin * Cout * 16;
  store_warp_ordered_sums<16>(acc, s_r, [&](int l, int a, int k, float r) {
    const int ci = ci0 + (l >> 3) * 4 + a, co = co0 + (l & 7);
    if (ci < Cin && co < Cout) dst[((size_t)ci * Cout + co) * 16 + k] = r;
  });
}

// ---------------------------------------------------------------------------------------------------------------
// Wide backward kernels for the high-resolution layers (Cin <= 32, the same layers as the wide forward).  The two
// kernels above move one shared-memory operand per 2.7 (data) / 3.2 (weight) FMAs and re-stage the gz tile with scalar
// loads; at 16->125 @1024^2 the layer's backward is 8.4 G FMA each way over a 524 MB gradient.  Here:
//  data:   a thread owns TWO horizontally adjacent input positions x 16 input channels in FMA pairs (32 sums in 16
//          64-bit registers); per output channel it reads its 4x6 window of gz (3 loads per row) once, and every 16-byte
//          weight load (two channel pairs of one tap) feeds 4 FMA pairs.  gz tiles (4 output channels x 34 x 66, 16-byte
//          cp.async for the interior, zero-filled halo) and the weights are double-buffered.
//  weight: lane = (4 input channels, 1 output channel, 16 taps) as above, but a step covers TWO adjacent positions: the
//          6-wide gz rows are shared between them (12 loads + 4 x-pair loads for 128 FMAs), tiles are staged with
//          cp.async and double-buffered.
constexpr int DW_Y = 16, DW_X = 32;                 // input positions per CTA (256 threads x 2 positions)
constexpr int DW_CO = 4, DW_CI = 16;
constexpr int DW_GY = 2 * DW_Y + 2, DW_GS = 72;     // gz tile rows, row stride in floats (global column 2*tx0 at index 4)
constexpr int DW_GBYTES = DW_CO * DW_GY * DW_GS * 4;   // 39168
constexpr int DW_WBYTES = DW_CO * 16 * DW_CI * 4;      // 4096, layout [co][tap][ci]
constexpr int DW_SMEM = 2 * (DW_GBYTES + DW_WBYTES);   // 86528

__device__ __forceinline__ void cp_async16_zfill(void* smem, const void* gmem, bool valid) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(sa), "l"(gmem), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ unsigned long long pack2(float a, float b) {
  unsigned long long r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
  return r;
}

// stage the gz tile of `nco` output channels starting at co0 into s_g [nco][rows][DW_GS]: rows 2*ty0-1 .. 2*ty0+rows-2,
// global columns 2*tx0-1 .. 2*tx0+64 at indices 3 .. 68.  Requires Wo % 4 == 0 (16-byte chunks are inside or outside).
template <int NCO, int ROWS, int PLANE>
__device__ __forceinline__ void stage_gz_tile(float* s_g, const float* __restrict__ gzb, int co0, int Cout, int Ho, int Wo,
                                              int ty0, int tx0, int tid) {
  constexpr int kChunks = 16;  // 64 interior floats per row
  for (int i = tid; i < NCO * ROWS * (kChunks + 2); i += 256) {
    const int co = i / (ROWS * (kChunks + 2)), r = (i / (kChunks + 2)) % ROWS, c = i % (kChunks + 2);
    const int Y = 2 * ty0 - 1 + r;
    const bool rok = co0 + co < Cout && Y >= 0 && Y < Ho;
    float* row = s_g + (size_t)co * PLANE + (size_t)r * DW_GS;
    const float* grow = gzb + ((size_t)(co0 + co) * Ho + (rok ? Y : 0)) * Wo;
    if (c < kChunks) {
      const int X = 2 * tx0 + 4 * c;
      const bool ok = rok && X < Wo;
      cp_async16_zfill(row + 4 + 4 * c, ok ? grow + X : gzb, ok);
    } else {
      const int X = (c == kChunks) ? 2 * tx0 - 1 : 2 * tx0 + 64;
      const bool ok = rok && X >= 0 && X < Wo;
      cp_async4_zfill(row + (c == kChunks ? 3 : 68), ok ? grow + X : gzb, ok);
    }
  }
}

template <bool CONV_FWD>  // as in deconv4x4s2_bwd_data_kernel
__global__ void __launch_bounds__(256, 2) deconv4x4s2_bwd_data_wide_kernel(
    int Cin, int Cout, int Hi, int Wi, const float* __restrict__ gz /* [B,Cout,2Hi,2Wi] */, const float* __restrict__ v,
    const float* __restrict__ scale, const float* __restrict__ bias, float slope, int apply_act,
    float* __restrict__ gx /* [B,Cin,Hi,Wi] */) {
  extern __shared__ __align__(16) unsigned char dsm[];
  const int tiles_x = (Wi + DW_X - 1) / DW_X;
  const int ty0 = (blockIdx.x / tiles_x) * DW_Y, tx0 = (blockIdx.x % tiles_x) * DW_X;
  const int ci0 = blockIdx.y * DW_CI;
  const int b = blockIdx.z;
  const int tid = threadIdx.x, qy = tid >> 4, qx = tid & 15;
  const int m = ty0 + qy, n = tx0 + 2 * qx;
  const int Ho = 2 * Hi, Wo = 2 * Wi;
  const float* gzb = gz + (size_t)b * Cout * Ho * Wo;
  auto g_buf = [&](int k) { return reinterpret_cast<float*>(dsm + (size_t)k * (DW_GBYTES + DW_WBYTES)); };
  auto w_buf = [&](int k) { return reinterpret_cast<float*>(dsm + (size_t)k * (DW_GBYTES + DW_WBYTES) + DW_GBYTES); };
  auto stage = [&](int k, int co0) {
    stage_gz_tile<DW_CO, DW_GY, DW_GY * DW_GS>(g_buf(k), gzb, co0, Cout, Ho, Wo, ty0, tx0, tid);
    float* sw = w_buf(k);
    for (int i = tid; i < DW_CO * 16 * DW_CI; i += 256) {
      const int ci = i / (DW_CO * 16), co = (i / 16) % DW_CO, t = i % 16;  // consecutive lanes read consecutive taps
      const bool ok = ci0 + ci < Cin && co0 + co < Cout;
      cp_async4_zfill(sw + (co * 16 + t) * DW_CI + ci, ok ? v + ((size_t)(ci0 + ci) * Cout + co0 + co) * 16 + t : v, ok);
    }
  };
  unsigned long long acc[2][DW_CI / 2];
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int c = 0; c < DW_CI / 2; ++c) acc[p][c] = 0ull;

  const int nblk = (Cout + DW_CO - 1) / DW_CO;
  stage(0, 0);
  gb::cp_async_commit();
  for (int blk = 0; blk < nblk; ++blk) {
    const int k = blk & 1;
    gb::cp_async_wait<0>();
    __syncthreads();  // this block's tile has landed for everybody; everybody has left the previous block's FMA loop
    if (blk + 1 < nblk) {
      stage(k ^ 1, (blk + 1) * DW_CO);
      gb::cp_async_commit();
    }
    const float* sg = g_buf(k);
    const float* sw = w_buf(k);
#pragma unroll 1
    for (int co = 0; co < DW_CO; ++co) {
      if (blk * DW_CO + co >= Cout) break;
      const float sc = CONV_FWD ? 1.f : scale[blk * DW_CO + co];
      unsigned long long G[4][6];  // rows 2m-1 .. 2m+2, columns 2n-1 .. 2n+4, scaled and duplicated
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float* rp = sg + ((size_t)co * DW_GY + 2 * qy + r) * DW_GS + 4 * qx + 3;
        const float g0 = rp[0];
        const float4 g14 = *reinterpret_cast<const float4*>(rp + 1);
        const float g5 = rp[5];
        const float gs[6] = {g0 * sc, g14.x * sc, g14.y * sc, g14.z * sc, g14.w * sc, g5 * sc};
#pragma unroll
        for (int c = 0; c < 6; ++c) G[r][c] = pack2(gs[c], gs[c]);
      }
      const ulonglong2* wp = reinterpret_cast<const ulonglong2*>(sw + (size_t)co * 16 * DW_CI);
#pragma unroll
      for (int ky = 0; ky < 4; ++ky)
#pragma unroll
        for (int kx = 0; kx < 4; ++kx) {
#pragma unroll
          for (int q = 0; q < DW_CI / 4; ++q) {
            const ulonglong2 w2 = wp[(ky * 4 + kx) * (DW_CI / 4) + q];  // channel pairs 2q, 2q+1 of this tap
            acc[0][2 * q] = ffma2(G[ky][kx], w2.x, acc[0][2 * q]);
            acc[0][2 * q + 1] = ffma2(G[ky][kx], w2.y, acc[0][2 * q + 1]);
            acc[1][2 * q] = ffma2(G[ky][kx + 2], w2.x, acc[1][2 * q]);
            acc[1][2 * q + 1] = ffma2(G[ky][kx + 2], w2.y, acc[1][2 * q + 1]);
          }
        }
    }
  }
  if (m >= Hi || n >= Wi) return;  // Wi and n are even: both positions are inside together
  float* gxb = gx + (size_t)b * Cin * Hi * Wi;
#pragma unroll
  for (int c = 0; c < DW_CI / 2; ++c) {
    const float2 a0 = unpack2(acc[0][c]), a1 = unpack2(acc[1][c]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int ch = ci0 + 2 * c + h;
      if (ch >= Cin) continue;
      const size_t off = ((size_t)ch * Hi + m) * Wi + n;
      float2 r = h ? make_float2(a0.y, a1.y) : make_float2(a0.x, a1.x);
      if (CONV_FWD) {
        const float sc = scale[ch];
        const float2 bb = bias ? *reinterpret_cast<const float2*>(bias + off) : make_float2(0.f, 0.f);
        r = make_float2(wn_bias_act(r.x, sc, bb.x, slope, apply_act), wn_bias_act(r.y, sc, bb.y, slope, apply_act));
      }
      *reinterpret_cast<float2*>(gxb + off) = r;
    }
  }
}

constexpr int WW_Y = 8, WW_X = 32;                 // input positions per staged tile
constexpr int WW_CO = 8, WW_CI = 16;
constexpr int WW_GY = 2 * WW_Y + 2;                // 18 gz rows
constexpr int WW_XS = 36;                          // x row stride in floats (32 + pad, rows 16-byte aligned)
// plane strides = 16 bytes mod 128: the 4 channel groups (x, 8-byte loads) and the 8 output channels (gz, 16-byte loads)
// that the lanes of a warp address in one instruction then fall into distinct banks (strides of 0 / 64 bytes mod 128
// would give 4-way conflicts on every operand load).
constexpr int WW_XP = WW_Y * WW_XS + 4;            // 292 floats
constexpr int WW_GP = WW_GY * DW_GS + 20;          // 1316 floats
constexpr int WW_XBYTES = WW_CI * WW_XP * 4;              // 18688
constexpr int WW_GBYTES = WW_CO * WW_GP * 4;              // 42112
constexpr int WW_SMEM = 2 * (WW_XBYTES + WW_GBYTES);      // 121600

__global__ void __launch_bounds__(256, 1) deconv4x4s2_bwd_weight_wide_kernel(
    int B, int Cin, int Cout, int Hi, int Wi, const float* __restrict__ x, const float* __restrict__ gz,
    float* __restrict__ part /* [gridDim.x][Cin,Cout,4,4] */) {
  extern __shared__ __align__(16) unsigned char dsm[];
  const int ci0 = blockIdx.y * WW_CI, co0 = blockIdx.z * WW_CO;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cig = lane >> 3, col = lane & 7;
  const int Ho = 2 * Hi, Wo = 2 * Wi;
  const int tiles_x = (Wi + WW_X - 1) / WW_X, tiles_y = (Hi + WW_Y - 1) / WW_Y;
  const int total = B * tiles_x * tiles_y;
  auto x_buf = [&](int k) { return reinterpret_cast<float*>(dsm + (size_t)k * (WW_XBYTES + WW_GBYTES)); };
  auto g_buf = [&](int k) { return reinterpret_cast<float*>(dsm + (size_t)k * (WW_XBYTES + WW_GBYTES) + WW_XBYTES); };
  auto stage = [&](int k, int t) {
    const int b = t / (tiles_x * tiles_y), tt = t % (tiles_x * tiles_y);
    const int ty0 = (tt / tiles_x) * WW_Y, tx0 = (tt % tiles_x) * WW_X;
    float* sx = x_buf(k);
    for (int i = tid; i < WW_CI * WW_Y * (WW_X / 4); i += 256) {  // 16-byte chunks: Wi % 4 == 0, tx0 % 32 == 0
      const int ci = i / (WW_Y * (WW_X / 4)), r = (i / (WW_X / 4)) % WW_Y, c = i % (WW_X / 4);
      const int yy = ty0 + r, xx = tx0 + 4 * c;
      const bool ok = ci0 + ci < Cin && yy < Hi && xx < Wi;
      cp_async16_zfill(sx + (size_t)ci * WW_XP + (size_t)r * WW_XS + 4 * c,
                       ok ? x + (((size_t)b * Cin + ci0 + ci) * Hi + yy) * Wi + xx : x, ok);
    }
    stage_gz_tile<WW_CO, WW_GY, WW_GP>(g_buf(k), gz + (size_t)b * Cout * Ho * Wo, co0, Cout, Ho, Wo, ty0, tx0, tid);
  };
  float acc[4][16];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int t = 0; t < 16; ++t) acc[a][t] = 0.f;

  int it = 0;
  if ((int)blockIdx.x < total) {
    stage(0, blockIdx.x);
    gb::cp_async_commit();
  }
  for (int t = blockIdx.x; t < total; t += gridDim.x, ++it) {
    const int k = it & 1;
    gb::cp_async_wait<0>();
    __syncthreads();
    if (t + (int)gridDim.x < total) {
      stage(k ^ 1, t + gridDim.x);
      gb::cp_async_commit();
    }
    const float* sx = x_buf(k);
    const float* sg = g_buf(k) + (size_t)col * WW_GP;
    // warp w: tile row w, 16 pairs of adjacent positions
#pragma unroll 2
    for (int pp = 0; pp < WW_X / 2; ++pp) {
      const int py = warp, px = 2 * pp;
      float2 xv[4];
#pragma unroll
      for (int a = 0; a < 4; ++a)  // lane's channels: a * 4 + cig (adjacent planes across the channel groups)
        xv[a] = *reinterpret_cast<const float2*>(sx + (size_t)(a * 4 + cig) * WW_XP + (size_t)py * WW_XS + px);
#pragma unroll
      for (int ky = 0; ky < 4; ++ky) {
        const float* rp = sg + (size_t)(2 * py + ky) * DW_GS + 2 * px + 3;  // global column 2*(tx0+px) - 1
        // 2*px + 3 = 4*pp + 3: one scalar, one aligned float4, one scalar
        const float g0 = rp[0];
        const float4 g14 = *reinterpret_cast<const float4*>(rp + 1);
        const float g5 = rp[5];
        const float g[6] = {g0, g14.x, g14.y, g14.z, g14.w, g5};
#pragma unroll
        for (int kx = 0; kx < 4; ++kx)
#pragma unroll
          for (int a = 0; a < 4; ++a) acc[a][ky * 4 + kx] += xv[a].x * g[kx] + xv[a].y * g[kx + 2];
      }
    }
  }
  // the staged tiles are dead: the reduction reuses their shared memory
  gb::cp_async_wait<0>();
  __syncthreads();
  float* dst = part + (size_t)blockIdx.x * Cin * Cout * 16;
  store_warp_ordered_sums<16>(acc, reinterpret_cast<float*>(dsm), [&](int l, int a, int k, float r) {
    const int ci = ci0 + a * 4 + (l >> 3), co = co0 + (l & 7);
    if (ci < Cin && co < Cout) dst[((size_t)ci * Cout + co) * 16 + k] = r;
  });
}

// The backward launches, shared by the transposed convolution and the stride-2 convolution (whose forward is this
// data gradient and whose weight gradient is this weight gradient with the roles of x and gz swapped).  `wide` picks
// the kernels for the high-resolution layers; the caller has checked Wi % 4 == 0, Wi >= 32, Hi >= 16.
template <bool CONV_FWD>
[[nodiscard]] int launch_bwd_data(bool wide, int B, int Cin, int Cout, int Hi, int Wi, const float* gz, const float* v,
                                  const float* scale, const float* bias, float slope, int apply_act, float* gx,
                                  cudaStream_t s) {
  if (wide) {
    dim3 grid(gb::cdiv(Hi, DW_Y) * gb::cdiv(Wi, DW_X), gb::cdiv(Cin, DW_CI), B);
    return gb::launch<deconv4x4s2_bwd_data_wide_kernel<CONV_FWD>>(grid, 256, DW_SMEM, s, Cin, Cout, Hi, Wi, gz, v,
                                                                  scale, bias, slope, apply_act, gx);
  }
  dim3 grid(gb::cdiv(Hi, BD_T) * gb::cdiv(Wi, BD_T), gb::cdiv(Cin, BD_CI), B);
  return gb::launch<deconv4x4s2_bwd_data_kernel<CONV_FWD>>(grid, BD_T * BD_T, 0, s, Cin, Cout, Hi, Wi, gz, v, scale,
                                                           bias, slope, apply_act, gx);
}

// The backward's kernels for a transposed convolution Cin -> Cout on an Hi x Wi input, and its weight gradient's split
// (CTAs per channel block, each writing one [Cin, Cout, 4, 4] partial).  The wide kernels need 16-byte rows and a full
// tile; the transposed convolution takes them for the layers of the wide forward (Cin <= 32), where its data gradient
// follows the same choice, and the stride-2 convolution (`conv`: its weight gradient, with the sides exchanged) at any
// channel count.  The launch and the workspace size both come from here.
struct BwdPlan {
  bool wide;
  int split;
  size_t part_bytes;
};

BwdPlan bwd_plan(bool conv, int B, int Cin, int Cout, int Hi, int Wi) {
  BwdPlan p;
  p.wide = (conv || Cin <= 32) && Wi % 4 == 0 && Wi >= 32 && Hi >= 16;
  if (p.wide) {
    // one CTA per SM at a time (120 KB of shared memory): two FULL waves
    const int total = B * gb::cdiv(Hi, WW_Y) * gb::cdiv(Wi, WW_X);
    const int pairs = gb::cdiv(Cin, WW_CI) * gb::cdiv(Cout, WW_CO);
    p.split = max(1, min((gb::kNumSMs * 2) / pairs, total));
  } else {
    p.split = wgrad_split(B, Cin, Cout, 1, Hi, Wi, 3);  // ~3 CTAs per SM in total
  }
  p.part_bytes = sizeof(float) * p.split * Cin * Cout * 16;
  return p;
}

// gw [Cin,Cout,4,4] written
[[nodiscard]] int launch_bwd_weight(const BwdPlan& p, int B, int Cin, int Cout, int Hi, int Wi, const float* x,
                                    const float* gz, float* gw, float* part, cudaStream_t s) {
  if (p.wide) {
    dim3 grid(p.split, gb::cdiv(Cin, WW_CI), gb::cdiv(Cout, WW_CO));
    GB_CUDA(gb::launch<deconv4x4s2_bwd_weight_wide_kernel>(grid, 256, WW_SMEM, s, B, Cin, Cout, Hi, Wi, x, gz, part));
  } else {
    dim3 grid(p.split, gb::cdiv(Cin, NW_CI), gb::cdiv(Cout, NW_CO));
    GB_CUDA(gb::launch<deconv4x4s2_bwd_weight_kernel>(grid, 256, 0, s, B, Cin, Cout, Hi, Wi, x, gz, part));
  }
  const int n = Cin * Cout * 16;
  return gb::launch<split_sum_kernel>(gb::cdiv(n, 256), 256, 0, s, p.split, n, part, gw);
}

// With an activation: gz = gout * act'(out) and the untied-bias gradient.  Without one, gz is gout and the bias
// gradient its batch sum (NULL at B == 1, where the caller aliases it to gout).
[[nodiscard]] int launch_act_bwd(int B, long long per_item, const float* out, const float* gout, float slope,
                                 int apply_act, float* gz, float* g_bias, cudaStream_t s) {
  const unsigned grid = (unsigned)gb::cdiv64(per_item, 256);
  if (apply_act) return gb::launch<act_bwd_kernel>(grid, 256, 0, s, B, per_item, gout, nullptr, out, slope, gz, g_bias);
  if (g_bias) return gb::launch<batch_sum_kernel>(grid, 256, 0, s, B, per_item, gout, g_bias);
  return 0;
}

}  // namespace

GB_API size_t gb_deconv4x4s2_wnub_bwd_workspace_bytes(int B, int Cin, int Cout, int Hi, int Wi) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || Hi <= 0 || Wi <= 0) return 0;
  return bwd_plan(false, B, Cin, Cout, Hi, Wi).part_bytes;
}

// Backward of gb_deconv4x4s2_wnub_fwd.  gz [B,Cout,2Hi,2Wi]: scratch for the pre-activation gradient when apply_act,
// else unused (gout is that gradient); g_bias [Cout,2Hi,2Wi] written, or NULL; gx [B,Cin,Hi,Wi] or NULL; gw
// [Cin,Cout,4,4] written, or NULL: the gradient w.r.t. the un-normalised direction tensor v at unit scale
// (d out / d (scale*v) contracted with v's slot), gw[ci,co,k] = sum x * gz; the caller applies the weight-norm chain
// rule.  workspace: gb_deconv4x4s2_wnub_bwd_workspace_bytes(..) bytes.
GB_API int gb_deconv4x4s2_wnub_bwd(int B, int Cin, int Cout, int Hi, int Wi, const float* x, const float* v,
                                   const float* scale, const float* out, const float* gout, float slope, int apply_act,
                                   float* gz, float* g_bias, float* gx, float* gw, void* workspace, void* stream) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || Hi <= 0 || Wi <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  GB_CUDA(launch_act_bwd(B, (long long)Cout * 4 * Hi * Wi, out, gout, slope, apply_act, gz, g_bias, s));
  const float* g = apply_act ? gz : gout;
  const BwdPlan p = bwd_plan(false, B, Cin, Cout, Hi, Wi);
  if (gx) GB_CUDA(launch_bwd_data<false>(p.wide, B, Cin, Cout, Hi, Wi, g, v, scale, nullptr, 1.f, 0, gx, s));
  if (gw) GB_CUDA(launch_bwd_weight(p, B, Cin, Cout, Hi, Wi, x, g, gw, (float*)workspace, s));
  return 0;
}

// =====================================================================================================
// Stride-2 4x4 convolution (k=4, s=2, p=1) with weight-norm scale, untied bias and LeakyReLU: the layer of the RGCA
// texture encoder (ca_code/models/rgca.py:281-298, la.Conv2dWNUB(cin, cout, h, w, 4, 2, 1), layers.py:276-327).
//   out[b,o,y,x] = act(scale[o] * sum_i sum_{ky,kx} x[b,i,2y-1+ky,2x-1+kx] v[o,i,ky,kx] + bias[o,y,x])
// This is the transposed convolution with its two sides exchanged, so it runs on the kernels above:
//   forward         = the deconv data gradient with the conv input as gz (CONV_FWD: scale on the output channel,
//                     bias + activation epilogue);
//   data gradient   = the (round-1) deconv forward of gz with v read as [Cin_d = Cout, Cout_d = Cin, 4, 4] (SCALE_IN:
//                     the scale belongs to its input channel o);
//   weight gradient = the deconv weight gradient with x and gz exchanged; its [Cin_d, Cout_d, 4, 4] output is the
//                     conv weight layout [Cout, Cin, 4, 4].
// Kernels are chosen by shape: the wide ones where the tile conditions hold and their grid still fills the machine.
namespace {

bool conv_wide_fwd(int B, int Cout, int Ho, int Wo) {
  return Wo % 4 == 0 && Wo >= 32 && Ho >= 16 &&
         (long long)gb::cdiv(Ho, DW_Y) * gb::cdiv(Wo, DW_X) * gb::cdiv(Cout, DW_CI) * B >= gb::kNumSMs;
}

}  // namespace

// x [B,Cin,2Ho,2Wo], v = weight_v [Cout,Cin,4,4], scale [Cout] = weight_g / ||weight_v||_F, bias [Cout,Ho,Wo] or
// NULL, out [B,Cout,Ho,Wo]; apply_act != 0 applies LeakyReLU(slope).
GB_API int gb_conv4x4s2_wnub_fwd(int B, int Cin, int Cout, int Ho, int Wo, const float* x, const float* v,
                                 const float* scale, const float* bias, float slope, int apply_act, float* out,
                                 void* stream) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || Ho <= 0 || Wo <= 0) return 0;
  return launch_bwd_data<true>(conv_wide_fwd(B, Cout, Ho, Wo), B, Cout, Cin, Ho, Wo, x, v, scale, bias, slope,
                               apply_act, out, (cudaStream_t)stream);
}

GB_API size_t gb_conv4x4s2_wnub_bwd_workspace_bytes(int B, int Cin, int Cout, int Ho, int Wo) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || Ho <= 0 || Wo <= 0) return 0;
  return bwd_plan(true, B, Cout, Cin, Ho, Wo).part_bytes;
}

// Backward of gb_conv4x4s2_wnub_fwd, with the conventions of gb_deconv4x4s2_wnub_bwd: gz [B,Cout,Ho,Wo] scratch when
// apply_act, else unused; g_bias [Cout,Ho,Wo] or NULL; gx [B,Cin,2Ho,2Wo] or NULL; gw [Cout,Cin,4,4] written at unit
// scale (gw[o,i,k] = sum gz * x), or NULL; the caller applies the weight-norm chain rule.  workspace:
// gb_conv4x4s2_wnub_bwd_workspace_bytes(..) bytes.
GB_API int gb_conv4x4s2_wnub_bwd(int B, int Cin, int Cout, int Ho, int Wo, const float* x, const float* v,
                                 const float* scale, const float* out, const float* gout, float slope, int apply_act,
                                 float* gz, float* g_bias, float* gx, float* gw, void* workspace, void* stream) {
  if (B <= 0 || Cin <= 0 || Cout <= 0 || Ho <= 0 || Wo <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  GB_CUDA(launch_act_bwd(B, (long long)Cout * Ho * Wo, out, gout, slope, apply_act, gz, g_bias, s));
  const float* g = apply_act ? gz : gout;
  if (gx) GB_CUDA(launch_deconv_fwd<true>(B, Cout, Cin, Ho, Wo, g, v, scale, nullptr, 1.f, 0, gx, s));
  if (gw)
    GB_CUDA(launch_bwd_weight(bwd_plan(true, B, Cout, Cin, Ho, Wo), B, Cout, Cin, Ho, Wo, g, x, gw, (float*)workspace,
                              s));
  return 0;
}
