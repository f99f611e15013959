// goliath_b200/csrc/deconv_tc.cu — stride-2 4x4 transposed convolution on the Hopper tensor cores
// (wgmma.mma_async, tf32, 3xTF32 split) fed by TMA, with the weight-norm scale, the untied bias and LeakyReLU in the
// epilogue (sm_90a).  Forward only (inference path; training uses csrc/deconv_wnub.cu).
//
// Replaces cuDNN conv_transpose2d + bias add + activation of the decoder towers
// (ca_code/nn/layers.py:380-396 called from ca_code/models/rgca.py:408-456) for layers with Cin % 32 == 0.
//
// Formulation: the k=4, s=2, p=1 transposed convolution splits into 4 output parities (py,px); each is a 2x2
// correlation, i.e. a GEMM  D[m, co] = sum_{tap,ci} A[m, (tap,ci)] * W[(tap,ci), co]  with
//   M = B*Hi*Wi output positions of that parity, N = Cout, K = 4*Cin.
// Activations live in HBM as NHWC (channels-last) so that A is K-major: a TMA box {32 ch, c px, r rows, 1 image}
// lands in shared memory as 128 rows of 128 bytes in the 128B-swizzled K-major layout wgmma reads; the tap
// offset (dy,dx) is just a coordinate shift and the image border is TMA out-of-bounds zero fill.
// 1e-4 parity with the fp32 reference needs more than one TF32 pass: every operand is carried as hi + lo (hi =
// round-to-tf32, lo = x - hi), D = Ahi*Bhi + Alo*Bhi + Ahi*Blo (3 MMAs per K slice), all accumulated in registers.
// One CTA = one 128-position tile of one parity: warp 8 = TMA producer, warps 0-7 = two consumer warpgroups (tile
// rows 0-63 and 64-127) that issue m64n16k8 wgmmas over the CTA's output channels, 2-4 stage mbarrier ring.  The
// accumulators are staged through the (then idle) stage buffers so that the epilogue owns one tile row and 16
// consecutive channels per thread (vector bias loads and NHWC stores).
#include <cuda.h>
#include <cudaTypedefs.h>

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kTileM = 128;
constexpr int kBlockK = 32;                 // fp32 elements per K block = one 128-byte swizzle row
constexpr int kMmaK = 8;                    // tf32
constexpr int kMmaN = 16;                   // output channels per wgmma (Nchunk is a multiple of 16)
constexpr int kMaxNT = 16;                  // Nchunk <= 256
constexpr int kConsumers = 256;             // two warpgroups
constexpr int kThreads = kConsumers + 32;   // + producer warp
constexpr int kABytes = kTileM * kBlockK * 4;  // 16 KB per A tile

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned phase) {
  unsigned ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(phase)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            unsigned long long* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, unsigned long long* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
               : "memory");
}
// wgmma shared-memory descriptor: K-major, 128B swizzle, rows 128 B apart, 8-row groups 1024 B apart
__device__ __forceinline__ unsigned long long wgmma_desc(unsigned smem_addr) {
  unsigned long long d = 0;
  d |= (unsigned long long)((smem_addr & 0x3FFFF) >> 4);   // start address, bits [0,14)
  d |= (unsigned long long)1 << 16;                         // leading byte offset (unused for swizzled K-major)
  d |= (unsigned long long)(1024 >> 4) << 32;               // stride byte offset, bits [32,46)
  d |= (unsigned long long)1 << 62;                         // SWIZZLE_128B
  return d;
}
// D[64 x 16] += A[64 x 8] * B[16 x 8]^T, tf32 inputs, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_tf32_n16(float (&d)[8], unsigned long long a, unsigned long long b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory"); }
__device__ __forceinline__ float to_tf32(float x) {
  unsigned r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

struct TcArgs {
  int B, Cin, Cout, Npad, Hi, Wi;  // Cin = padded channel count (multiple of 32); Npad = Cout rounded up to 16
  int Nchunk;                    // output channels per CTA (divides Npad, multiple of 16): grid.z = Npad / Nchunk
  int tile_r, tile_c;            // tile = tile_r rows x tile_c columns of input positions, tile_r * tile_c == 128
  int stages;
  const float* scale;            // [Cout]
  const float* bias;             // [Cout, 2Hi, 2Wi] or null
  float slope; int apply_act;
  float* out_hi; float* out_lo;  // NHWC [B,2Hi,2Wi,ldc] (next tensor-core layer), or null
  int ldc;                       // channel stride of out_hi / out_lo (>= Cout, multiple of 32)
  float* out_nchw;               // NCHW [B,Cout,2Hi,2Wi] fp32, or null
};

// row stride (floats) of the accumulator staging tile: 16-byte rows, conflict-free quarter-warp float4 reads
__host__ __device__ __forceinline__ int acc_stride(int npx, int nchunk) { return npx * nchunk + 4; }

__device__ __forceinline__ void ld_acc16(const float* p, float (&r)[16]) {
#pragma unroll
  for (int j = 0; j < 16; j += 4) {
    const float4 v = *reinterpret_cast<const float4*>(p + j);
    r[j] = v.x; r[j + 1] = v.y; r[j + 2] = v.z; r[j + 3] = v.w;
  }
}
__device__ __forceinline__ float2 ld_nc_f2(const float2* p) {
  float2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
  return r;
}
// 16 consecutive channels of one output pixel -> the NHWC hi/lo pair the next tensor-core layer reads
__device__ __forceinline__ void store_nhwc_split(const TcArgs& a, size_t base, const float (&v)[16]) {
  float hi[16], lo[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) { hi[j] = to_tf32(v[j]); lo[j] = v[j] - hi[j]; }
#pragma unroll
  for (int j = 0; j < 16; j += 4) {
    *reinterpret_cast<float4*>(a.out_hi + base + j) = make_float4(hi[j], hi[j + 1], hi[j + 2], hi[j + 3]);
    *reinterpret_cast<float4*>(a.out_lo + base + j) = make_float4(lo[j], lo[j + 1], lo[j + 2], lo[j + 3]);
  }
}

// NT = Nchunk / 16 wgmma column blocks, NPX = column parities per CTA (2 in pair mode)
template <int NT, int NPX>
__global__ void __launch_bounds__(kThreads, 1) deconv_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi,
                                                                 const __grid_constant__ CUtensorMap map_a_lo,
                                                                 const __grid_constant__ CUtensorMap map_b_hi,
                                                                 const __grid_constant__ CUtensorMap map_b_lo, TcArgs a) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  constexpr int kNchunk = NT * kMmaN;
  // carve: per stage [A_hi | A_lo | B_hi | B_lo], all 1024-byte aligned
  constexpr int b_bytes = kNchunk * kBlockK * 4;
  constexpr int stage_bytes = 2 * kABytes + 2 * b_bytes;
  const int nc0 = blockIdx.z * kNchunk;      // first output channel of this CTA
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) unsigned long long s_full[4], s_empty[4];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // output parity (py, px): one CTA per parity, or (pair mode) one CTA per row parity that computes px = 0 and 1 into
  // two accumulators, so that its epilogue owns pairs of adjacent output pixels (8-byte bias loads / stores)
  const int py = NPX == 2 ? (int)blockIdx.y : (int)(blockIdx.y >> 1);
  const int tiles_x = (a.Wi + a.tile_c - 1) / a.tile_c, tiles_y = (a.Hi + a.tile_r - 1) / a.tile_r;
  const int tile = blockIdx.x;
  const int b = tile / (tiles_x * tiles_y);
  const int ty = (tile / tiles_x) % tiles_y, tx = tile % tiles_x;
  const int m0 = ty * a.tile_r, n0 = tx * a.tile_c;
  const int kb_per_tap = a.Cin / kBlockK, num_kb = 4 * kb_per_tap;

  if (threadIdx.x == 0) {
    for (int s = 0; s < a.stages; ++s) { mbar_init(&s_full[s], 1); mbar_init(&s_empty[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kConsumers / 32) {
    // ===== TMA producer (one elected lane) =====
    if (lane == 0) {
      for (int g = 0; g < NPX * num_kb; ++g) {
        const int px = NPX == 2 ? g / num_kb : (int)(blockIdx.y & 1), kb = g % num_kb;
        const int phase_id = py * 2 + px;
        const int s = g % a.stages, it = g / a.stages;
        if (it > 0) mbar_wait(&s_empty[s], (unsigned)((it - 1) & 1));
        const int tap = kb / kb_per_tap, cblk = kb % kb_per_tap;
        const int tyy = tap >> 1, txx = tap & 1;
        // parity 0: taps (k=1, d=0), (k=3, d=-1); parity 1: taps (k=2, d=0), (k=0, d=+1)
        const int dy = (tyy == 0) ? 0 : (py ? 1 : -1), dx = (txx == 0) ? 0 : (px ? 1 : -1);
        unsigned char* st = smem + (size_t)s * stage_bytes;
        mbar_expect_tx(&s_full[s], (unsigned)stage_bytes);
        tma_load_4d(st, &map_a_hi, cblk * kBlockK, n0 + dx, m0 + dy, b, &s_full[s]);
        tma_load_4d(st + kABytes, &map_a_lo, cblk * kBlockK, n0 + dx, m0 + dy, b, &s_full[s]);
        const int krow = phase_id * a.Npad + nc0;    // weight matrix rows: [phase][co padded]
        const int kcol = tap * a.Cin + cblk * kBlockK;  // columns: [tap][ci]
        tma_load_2d(st + 2 * kABytes, &map_b_hi, kcol, krow, &s_full[s]);
        tma_load_2d(st + 2 * kABytes + b_bytes, &map_b_lo, kcol, krow, &s_full[s]);
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64) =====
  const int wg = threadIdx.x >> 7;
  float acc[NPX][NT][8];
#pragma unroll
  for (int p = 0; p < NPX; ++p)
#pragma unroll
    for (int t = 0; t < NT; ++t)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[p][t][j] = 0.f;
#pragma unroll
  for (int p = 0; p < NPX; ++p) {
    for (int kb = 0; kb < num_kb; ++kb) {
      const int g = p * num_kb + kb;
      const int s = g % a.stages, it = g / a.stages;
      mbar_wait(&s_full[s], (unsigned)(it & 1));
      const unsigned st = smem_u32(smem + (size_t)s * stage_bytes);
      const unsigned a_off = (unsigned)wg * 64u * 128u;
      const unsigned long long da_hi = wgmma_desc(st + a_off), da_lo = wgmma_desc(st + kABytes + a_off);
      const unsigned long long db_hi = wgmma_desc(st + 2 * kABytes), db_lo = wgmma_desc(st + 2 * kABytes + b_bytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / kMmaK; ++k) {
        const unsigned long long adv = (unsigned long long)((k * kMmaK * 4) >> 4);  // +32 bytes per K slice
#pragma unroll
        for (int t = 0; t < NT; ++t) {
          const unsigned long long bt = (unsigned long long)((t * kMmaN * 128) >> 4);  // 16 weight rows further
          // small terms first, then the main product
          wgmma_tf32_n16(acc[p][t], da_lo + adv, db_hi + bt + adv);
          wgmma_tf32_n16(acc[p][t], da_hi + adv, db_lo + bt + adv);
          wgmma_tf32_n16(acc[p][t], da_hi + adv, db_hi + bt + adv);
        }
      }
      wgmma_commit();
      // each stage's MMAs complete before the next stage is issued: keeping one stage in flight (wait_group 1,
      // releasing the previous stage) measured slower (decoder tower 1.19 vs 1.15 ms, H100 SXM at a 400 W limit)
      wgmma_wait0();
      if ((threadIdx.x & 127) == 0) mbar_arrive(&s_empty[s]);  // this warpgroup is done reading the stage
    }
  }

  // stage the accumulators through shared memory: [128 rows][NPX * Nchunk] (+4 padding floats per row).  Both
  // warpgroups must be done with the stage buffers first; every TMA load has landed (all full barriers were consumed).
  consumers_sync();
  float* sacc = reinterpret_cast<float*>(smem);
  const int ldS = acc_stride(NPX, kNchunk);
  {
    const int wl = (threadIdx.x >> 5) & 3, qr = lane >> 2, qc = lane & 3;
#pragma unroll
    for (int p = 0; p < NPX; ++p)
#pragma unroll
      for (int t = 0; t < NT; ++t)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < 2; ++i) {  // fragment: d[4h + 2i + {0,1}] = row 8i + qr, columns 8h + 2qc + {0,1}
            const int row = wg * 64 + wl * 16 + 8 * i + qr;
            const int col = p * kNchunk + t * kMmaN + 8 * h + 2 * qc;
            *reinterpret_cast<float2*>(sacc + (size_t)row * ldS + col) = make_float2(acc[p][t][4 * h + 2 * i], acc[p][t][4 * h + 2 * i + 1]);
          }
  }
  consumers_sync();

  // ===== epilogue: thread owns tile row (tid % 128) and every other 16-channel block starting at 16 * (tid / 128)
  const int row = threadIdx.x & 127;
  const int cstart = (threadIdx.x >> 7) * 16;
  const int ry = row / a.tile_c, rx = row % a.tile_c;
  const int m = m0 + ry, n = n0 + rx;
  if (m >= a.Hi || n >= a.Wi) return;
  const int Ho = 2 * a.Hi, Wo = 2 * a.Wi;
  const int Y = 2 * m + py;
  const float* srow = sacc + (size_t)row * ldS;
  if (NPX == 1) {
    const int px = (int)(blockIdx.y & 1), X = 2 * n + px;
    for (int c0 = cstart; c0 < kNchunk; c0 += 32) {
      float r[16];
      ld_acc16(srow + c0, r);
      float v[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int co = nc0 + c0 + j;
        float o = 0.f;
        if (co < a.Cout) {  // columns beyond Cout are zero padding of the N dimension
          o = r[j] * a.scale[co];
          if (a.bias) o += a.bias[((size_t)co * Ho + Y) * Wo + X];
          if (a.apply_act) o = o > 0.f ? o : o * a.slope;
        }
        v[j] = o;
      }
      if (a.out_nchw) {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (nc0 + c0 + j < a.Cout) a.out_nchw[(((size_t)b * a.Cout + nc0 + c0 + j) * Ho + Y) * Wo + X] = v[j];
      }
      if (a.out_hi) store_nhwc_split(a, (((size_t)b * Ho + Y) * Wo + X) * a.ldc + nc0 + c0, v);
    }
  } else {
    // both column parities: tile position (m, n) -> output columns 2n, 2n+1: a warp's 32 lanes cover 256 contiguous
    // bytes of a bias / output row per channel
    for (int c0 = cstart; c0 < kNchunk; c0 += 32) {
      float r0[16], r1[16];
      ld_acc16(srow + c0, r0);
      ld_acc16(srow + kNchunk + c0, r1);
      float2 bb[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        bb[j] = make_float2(0.f, 0.f);
        if (a.bias && nc0 + c0 + j < a.Cout)
          bb[j] = ld_nc_f2(reinterpret_cast<const float2*>(a.bias + ((size_t)(nc0 + c0 + j) * Ho + Y) * Wo + 2 * n));
      }
      float v0[16], v1[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int co = nc0 + c0 + j;
        float o0 = 0.f, o1 = 0.f;
        if (co < a.Cout) {
          const float sc = a.scale[co];
          o0 = r0[j] * sc + bb[j].x;
          o1 = r1[j] * sc + bb[j].y;
          if (a.apply_act) { o0 = o0 > 0.f ? o0 : o0 * a.slope; o1 = o1 > 0.f ? o1 : o1 * a.slope; }
        }
        v0[j] = o0; v1[j] = o1;
      }
      if (a.out_nchw) {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (nc0 + c0 + j < a.Cout)
            *reinterpret_cast<float2*>(a.out_nchw + (((size_t)b * a.Cout + nc0 + c0 + j) * Ho + Y) * Wo + 2 * n) = make_float2(v0[j], v1[j]);
      }
      if (a.out_hi) {
        const size_t base = (((size_t)b * Ho + Y) * Wo + 2 * n) * a.ldc + nc0 + c0;
        store_nhwc_split(a, base, v0);
        store_nhwc_split(a, base + a.ldc, v1);
      }
    }
  }
}

// ---- helpers: NCHW fp32 -> NHWC hi/lo (channel-padded), weights -> [4 phases][Cout][4 taps * Cin_pad] hi/lo
__global__ void __launch_bounds__(256) nchw_to_nhwc_split_kernel(int B, int C, int Cpad, int HW, const float* __restrict__ x,
                                                                 float* __restrict__ hi, float* __restrict__ lo) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over B*HW*Cpad
  if (i >= (long long)B * HW * Cpad) return;
  const int c = (int)(i % Cpad);
  const long long p = i / Cpad;
  const int b = (int)(p / HW), pix = (int)(p % HW);
  const float v = c < C ? x[((size_t)b * C + c) * HW + pix] : 0.f;
  const float h = to_tf32(v);
  hi[i] = h;
  lo[i] = v - h;
}

__global__ void __launch_bounds__(256) weight_prep_kernel(int Cin, int Cpad, int Cout, int Npad, const float* __restrict__ v,
                                                          float* __restrict__ w_hi, float* __restrict__ w_lo) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over 4*Cout*4*Cpad
  const long long total = 16ll * Npad * Cpad;
  if (i >= total) return;
  const int ci = (int)(i % Cpad);
  const int tap = (int)((i / Cpad) % 4);
  const int co = (int)((i / (4ll * Cpad)) % Npad);
  const int phase = (int)(i / (4ll * Cpad * Npad));
  const int py = phase >> 1, px = phase & 1, tyy = tap >> 1, txx = tap & 1;
  const int ky = (tyy == 0) ? (py ? 2 : 1) : (py ? 0 : 3);
  const int kx = (txx == 0) ? (px ? 2 : 1) : (px ? 0 : 3);
  const float val = (ci < Cin && co < Cout) ? v[(((size_t)ci * Cout + co) * 4 + ky) * 4 + kx] : 0.f;
  const float h = to_tf32(val);
  w_hi[i] = h;
  w_lo[i] = val - h;
}

PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult q;
    void* p = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (PFN_cuTensorMapEncodeTiled_v12000)p;
  }
  return fn;
}

template <int NT, int NPX>
[[nodiscard]] cudaError_t launch_tc(dim3 grid, size_t smem, cudaStream_t s, const CUtensorMap& ma_hi,
                                    const CUtensorMap& ma_lo, const CUtensorMap& mb_hi, const CUtensorMap& mb_lo,
                                    const TcArgs& a) {
  static_assert(NT * NPX <= kMaxNT, "accumulators per thread");
  return gb::launch<deconv_tc_kernel<NT, NPX>>(grid, kThreads, smem, s, ma_hi, ma_lo, mb_hi, mb_lo, a);
}

}  // namespace

// bytes of scratch for the weight matrices of one layer (hi + lo)
GB_API size_t gb_deconv_tc_weight_bytes(int Cin_pad, int Cout) {
  return (size_t)2 * 16 * ((Cout + 15) / 16 * 16) * Cin_pad * sizeof(float);
}

// NCHW fp32 -> NHWC hi/lo with the channel count padded to Cpad (multiple of 32): the tensor-core layers' input format
GB_API int gb_nchw_to_nhwc_split(int B, int C, int Cpad, int H, int W, const float* x, float* hi, float* lo, void* stream) {
  const long long total = (long long)B * H * W * Cpad;
  if (total <= 0) return 0;
  return gb::launch<nchw_to_nhwc_split_kernel>((unsigned)gb::cdiv64(total, 256), 256, 0, (cudaStream_t)stream, B, C,
                                               Cpad, H * W, x, hi, lo);
}

// Tensor-core forward of ConvTranspose2dWNUB(k=4,s=2,p=1) [+LeakyReLU].  x_hi/x_lo: NHWC [B,Hi,Wi,Cin_pad] (tf32 hi
// part and remainder), v [Cin,Cout,4,4], w_scratch of gb_deconv_tc_weight_bytes(Cin_pad, Cout) bytes, scale [Cout],
// bias [Cout,2Hi,2Wi] or NULL.  Outputs (either or both): out_hi/out_lo NHWC [B,2Hi,2Wi,ldc] for a following
// tensor-core layer, out_nchw [B,Cout,2Hi,2Wi] fp32.  Requires Cin_pad % 32 == 0 and Cout <= 256 (N is padded to 16).
// v == NULL skips the weight preparation: w_scratch must then hold the result of an earlier call with the same v.
GB_API int gb_deconv4x4s2_tc_fwd(int B, int Cin, int Cin_pad, int Cout, int Hi, int Wi, const float* x_hi,
                                 const float* x_lo, const float* v, float* w_scratch, const float* scale,
                                 const float* bias, float slope, int apply_act, float* out_hi, float* out_lo, int ldc,
                                 float* out_nchw, void* stream) {
  if (B <= 0 || Hi <= 0 || Wi <= 0) return 0;
  const int Npad = (Cout + 15) / 16 * 16;
  if (Cin_pad % 32 != 0 || Cin > Cin_pad || Cout < 1 || Npad > 256) return (int)cudaErrorInvalidValue;
  if (out_hi && (ldc < Cout || ldc % 4 != 0)) return (int)cudaErrorInvalidValue;
  PFN_cuTensorMapEncodeTiled_v12000 encode = get_encode();
  if (!encode) return (int)cudaErrorNotSupported;
  cudaStream_t s = (cudaStream_t)stream;
  float* w_hi = w_scratch;
  float* w_lo = w_scratch + (size_t)16 * Npad * Cin_pad;
  if (v) {  // v == NULL: w_scratch still holds the matrices prepared by an earlier call with the same weight_v
    const long long total = 16ll * Npad * Cin_pad;
    GB_CUDA(gb::launch<weight_prep_kernel>((unsigned)gb::cdiv64(total, 256), 256, 0, s, Cin, Cin_pad, Cout, Npad, v,
                                           w_hi, w_lo));
  }
  // tile geometry: 128 positions = tile_r rows x tile_c columns
  int tile_c = 128;
  while (tile_c > Wi && tile_c > 1) tile_c >>= 1;
  if (tile_c < 8) tile_c = 8;
  const int tile_r = kTileM / tile_c;

  const int tiles = B * gb::cdiv(Hi, tile_r) * gb::cdiv(Wi, tile_c);
  // pair mode holds two accumulators in registers (2 * Npad <= 256 floats per row) and needs enough tiles to fill the
  // machine with half as many CTAs
  const int pair = (2 * Npad <= 256 && tiles * 2 >= 2 * gb::kNumSMs && Wi % 2 == 0) ? 1 : 0;
  // the low-resolution layers have a handful of tiles: split the output channels over CTAs (grid.z) until the
  // machine is covered; every CTA then streams the same A tiles (L2 hits) against its own slice of the weights
  int Nchunk = Npad;
  while (tiles * (pair ? 2 : 4) * (Npad / Nchunk) < gb::kNumSMs && Nchunk >= 32 && (Nchunk / 2) % 16 == 0 &&
         Npad % (Nchunk / 2) == 0)
    Nchunk /= 2;
  const int ctas = tiles * (pair ? 2 : 4) * (Npad / Nchunk);

  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  {
    const cuuint64_t gdim[4] = {(cuuint64_t)Cin_pad, (cuuint64_t)Wi, (cuuint64_t)Hi, (cuuint64_t)B};
    const cuuint64_t gstr[3] = {(cuuint64_t)Cin_pad * 4, (cuuint64_t)Wi * Cin_pad * 4, (cuuint64_t)Hi * Wi * Cin_pad * 4};
    const cuuint32_t box[4] = {(cuuint32_t)kBlockK, (cuuint32_t)tile_c, (cuuint32_t)tile_r, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    if (encode(&ma_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)x_hi, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return (int)cudaErrorInvalidValue;
    if (encode(&ma_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)x_lo, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return (int)cudaErrorInvalidValue;
  }
  {
    const cuuint64_t gdim[2] = {(cuuint64_t)4 * Cin_pad, (cuuint64_t)4 * Npad};
    const cuuint64_t gstr[1] = {(cuuint64_t)4 * Cin_pad * 4};
    const cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)Nchunk};
    const cuuint32_t estr[2] = {1, 1};
    if (encode(&mb_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)w_hi, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return (int)cudaErrorInvalidValue;
    if (encode(&mb_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)w_lo, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return (int)cudaErrorInvalidValue;
  }
  TcArgs a = {};
  a.B = B; a.Cin = Cin_pad; a.Cout = Cout; a.Npad = Npad; a.Nchunk = Nchunk; a.Hi = Hi; a.Wi = Wi; a.tile_r = tile_r;
  a.tile_c = tile_c;
  a.scale = scale; a.bias = bias; a.slope = slope; a.apply_act = apply_act; a.out_hi = out_hi; a.out_lo = out_lo;
  a.ldc = ldc; a.out_nchw = out_nchw;
  // every CTA is a serial TMA -> MMA -> epilogue chain: with few CTAs give each a deep ring (up to 4 stages); with
  // many, keep the ring short so that the next CTA on the SM starts while this one drains its epilogue
  const int stage_bytes = 2 * kABytes + 2 * Nchunk * kBlockK * 4;
  const int num_kb_total = (pair ? 2 : 1) * 4 * (Cin_pad / kBlockK);
  int stages = ctas > gb::kNumSMs ? 2 : 4;
  while (stages > 2 && (size_t)stages * stage_bytes + 1024 > 200 * 1024) --stages;
  if (stages > num_kb_total) stages = num_kb_total;
  if (stages < 1) stages = 1;
  a.stages = stages;
  // the stage buffers also hold the accumulator tile for the epilogue
  const size_t acc_bytes = (size_t)kTileM * acc_stride(pair ? 2 : 1, Nchunk) * sizeof(float);
  const size_t smem = std::max((size_t)a.stages * stage_bytes, acc_bytes) + 1024;
  const dim3 grid(tiles, pair ? 2 : 4, Npad / Nchunk);
  const int nt = Nchunk / kMmaN;
  cudaError_t err = cudaErrorInvalidValue;
  switch (pair * 100 + nt) {
#define GB_TC_CASE(NPX, NT)                                                                                        \
  case (NPX - 1) * 100 + NT:                                                                                       \
    err = launch_tc<NT, NPX>(grid, smem, s, ma_hi, ma_lo, mb_hi, mb_lo, a);                                       \
    break;
    GB_TC_CASE(1, 1) GB_TC_CASE(1, 2) GB_TC_CASE(1, 3) GB_TC_CASE(1, 4) GB_TC_CASE(1, 5) GB_TC_CASE(1, 6)
    GB_TC_CASE(1, 7) GB_TC_CASE(1, 8) GB_TC_CASE(1, 9) GB_TC_CASE(1, 10) GB_TC_CASE(1, 11) GB_TC_CASE(1, 12)
    GB_TC_CASE(1, 13) GB_TC_CASE(1, 14) GB_TC_CASE(1, 15) GB_TC_CASE(1, 16)
    GB_TC_CASE(2, 1) GB_TC_CASE(2, 2) GB_TC_CASE(2, 3) GB_TC_CASE(2, 4) GB_TC_CASE(2, 5) GB_TC_CASE(2, 6)
    GB_TC_CASE(2, 7) GB_TC_CASE(2, 8)
#undef GB_TC_CASE
    default: break;
  }
  return err;
}
