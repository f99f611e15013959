// goliath_b200/csrc/splat_blend.cu — per-tile alpha blending of sorted 2-D Gaussians, fwd + bwd (sm_90a).
//
// Replaces (third-party, absent from the reference tree) gsplat 0.1.11 rasterize_forward /
// rasterize_backward_kernel as called from ca_code/utils/render_gsplat.py:65-78 (rgb) and :90-104
// (depth-as-colour); semantics restated in SURVEY.md Appendix A and oracle/splat_oracle.c.
//
// One CTA per 16x16 tile (block_width <= 16 supported; CTA = roundup(bw*bw, 32) threads).
// Design points:
//  * each warp owns a compact 8x4 pixel footprint (bw == 16), so "all lanes done" / "no lane hit"
//    tests prune far more often than with the reference's 16x2 rows;
//  * a batch of Gaussians (position, conic, opacity AND colours) is gathered once per CTA into shared
//    memory as float4 records read as conflict-free broadcasts; the gather of batch b+1 is issued into
//    registers before batch b is blended, so HBM/L2 latency hides under the blend loop;
//  * C = 3 (reference API) or C = 4 (fused rgb+depth single pass, SURVEY.md §8f-1) colour channels;
//  * backward: per-Gaussian gradients are reduced warp -> CTA (shared-memory accumulators for the
//    batch) -> ONE set of RED atomics per (tile, Gaussian) instead of one per (warp, Gaussian).
#include "common.cuh"

namespace {

constexpr int kMaxThreads = 256;
constexpr float kAlphaMaxFwd = 0.999f;
// contract constant of gsplat 0.1.x: the backward clamps alpha at 0.99 (oracle: ORC_BWD_ALPHA_CLAMP)
constexpr float kAlphaMaxBwd = 0.99f;
constexpr float kAlphaMin = 1.f / 255.f;
constexpr float kTEps = 1e-4f;

struct PixMap {
  int px, py;     // pixel coordinates
  bool inside;
};

__device__ __forceinline__ PixMap map_pixel(int bw, int img_w, int img_h) {
  const int t = threadIdx.x;
  int lx, ly;
  if (bw == 16) {  // warp w -> 8x4 footprint
    const int w = t >> 5, l = t & 31;
    lx = ((w & 1) << 3) + (l & 7);
    ly = ((w >> 1) << 2) + (l >> 3);
  } else {
    lx = t % bw;
    ly = t / bw;
  }
  PixMap m;
  m.px = blockIdx.x * bw + lx;
  m.py = blockIdx.y * bw + ly;
  m.inside = (t < bw * bw) && (m.px < img_w) && (m.py < img_h);
  return m;
}

// per-Gaussian record staged in shared memory
template <int C>
struct Batch {
  float4 a[kMaxThreads];  // x, y, conic.A, conic.B
  float4 b[kMaxThreads];  // conic.C, opacity, col0, col1
  float2 c[kMaxThreads];  // col2, col3 (C == 4)
};

template <int C>
struct Rec {
  float4 a, b;
  float2 c;
};

template <int C>
__device__ __forceinline__ Rec<C> gather(int g, const float2* __restrict__ xys, const float* __restrict__ conics,
                                         const float* __restrict__ colors, const float* __restrict__ opac) {
  Rec<C> r;
  const float2 xy = xys[g];
  const float cA = conics[3 * g], cB = conics[3 * g + 1], cC = conics[3 * g + 2];
  r.a = make_float4(xy.x, xy.y, cA, cB);
  if (C == 4) {
    const float4 col = reinterpret_cast<const float4*>(colors)[g];
    r.b = make_float4(cC, opac[g], col.x, col.y);
    r.c = make_float2(col.z, col.w);
  } else {
    r.b = make_float4(cC, opac[g], colors[3 * g], colors[3 * g + 1]);
    r.c = make_float2(colors[3 * g + 2], 0.f);
  }
  return r;
}

template <int C>
__global__ void __launch_bounds__(kMaxThreads) rasterize_fwd_kernel(
    int img_w, int img_h, int bw, const int* __restrict__ gids_sorted, const int2* __restrict__ tile_bins,
    const float2* __restrict__ xys, const float* __restrict__ conics, const float* __restrict__ colors,
    const float* __restrict__ opacities, const float* __restrict__ background, float* __restrict__ final_Ts,
    int* __restrict__ final_idx, float* __restrict__ out_img) {
  __shared__ Batch<C> sb;
  const int tile_id = blockIdx.y * gridDim.x + blockIdx.x;
  const PixMap pm = map_pixel(bw, img_w, img_h);
  const float px = (float)pm.px + 0.5f, py = (float)pm.py + 0.5f;
  const int2 range = tile_bins[tile_id];
  const int bs = blockDim.x;
  const int tr = threadIdx.x;
  const int num_batches = (range.y - range.x + bs - 1) / bs;

  bool done = !pm.inside;
  float T = 1.f;
  int cur_idx = 0;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};

  // prefetch batch 0 into registers
  Rec<C> nxt;
  bool have = false;
  if (num_batches > 0) {
    const int idx = range.x + tr;
    have = idx < range.y;
    if (have) nxt = gather<C>(gids_sorted[idx], xys, conics, colors, opacities);
  }
  for (int b = 0; b < num_batches; ++b) {
    // all pixels of the tile saturated -> stop (also orders smem reuse)
    if (__syncthreads_count(done) >= bs) break;
    if (have) { sb.a[tr] = nxt.a; sb.b[tr] = nxt.b; sb.c[tr] = nxt.c; }
    const int batch_start = range.x + bs * b;
    // issue the gather of the next batch now; it is consumed after this batch's blend loop
    {
      const int idx = batch_start + bs + tr;
      have = idx < range.y;
      if (have) nxt = gather<C>(gids_sorted[idx], xys, conics, colors, opacities);
    }
    __syncthreads();
    const int batch_size = min(bs, range.y - batch_start);
    if (!__all_sync(0xffffffffu, done)) {
      for (int t = 0; t < batch_size && !done; ++t) {
        const float4 ga = sb.a[t];
        const float4 gb_ = sb.b[t];
        const float dx = ga.x - px, dy = ga.y - py;
        const float sigma = 0.5f * (ga.z * dx * dx + gb_.x * dy * dy) + ga.w * dx * dy;
        const float alpha = fminf(kAlphaMaxFwd, gb_.y * __expf(-sigma));
        if (sigma < 0.f || alpha < kAlphaMin) continue;
        const float next_T = T * (1.f - alpha);
        if (next_T <= kTEps) { done = true; break; }
        const float vis = alpha * T;
        acc[0] += gb_.z * vis;
        acc[1] += gb_.w * vis;
        const float2 gc = sb.c[t];
        acc[2] += gc.x * vis;
        if (C == 4) acc[3] += gc.y * vis;
        T = next_T;
        cur_idx = batch_start + t;
      }
    }
  }
  if (pm.inside) {
    const size_t pix = (size_t)pm.py * img_w + pm.px;
    final_Ts[pix] = T;
    final_idx[pix] = cur_idx;
    if (C == 4) {
      reinterpret_cast<float4*>(out_img)[pix] =
          make_float4(acc[0] + T * background[0], acc[1] + T * background[1], acc[2] + T * background[2],
                      acc[3] + T * background[3]);
    } else {
      out_img[pix * 3 + 0] = acc[0] + T * background[0];
      out_img[pix * 3 + 1] = acc[1] + T * background[1];
      out_img[pix * 3 + 2] = acc[2] + T * background[2];
    }
  }
}

// ---------------------------------------------------------------------------------------- backward
template <int C>
__global__ void __launch_bounds__(kMaxThreads) rasterize_bwd_kernel(
    int img_w, int img_h, int bw, const int* __restrict__ gids_sorted, const int2* __restrict__ tile_bins,
    const float2* __restrict__ xys, const float* __restrict__ conics, const float* __restrict__ colors,
    const float* __restrict__ opacities, const float* __restrict__ background, const float* __restrict__ final_Ts,
    const int* __restrict__ final_idx, const float* __restrict__ v_output, const float* __restrict__ v_output_alpha,
    float* __restrict__ v_xy, float* __restrict__ v_conic, float* __restrict__ v_colors,
    float* __restrict__ v_opacity) {
  constexpr int NV = C + 6;  // colours, conic(3), xy(2), opacity
  __shared__ Batch<C> sb;
  __shared__ int s_id[kMaxThreads];
  __shared__ float s_grad[kMaxThreads][NV + (NV % 2 == 0 ? 1 : 0)];  // odd stride: conflict-free flush
  __shared__ int s_touched[kMaxThreads];

  const int tile_id = blockIdx.y * gridDim.x + blockIdx.x;
  const PixMap pm = map_pixel(bw, img_w, img_h);
  const float px = (float)pm.px + 0.5f, py = (float)pm.py + 0.5f;
  const int2 range = tile_bins[tile_id];
  if (range.y <= range.x) return;
  const int bs = blockDim.x;
  const int tr = threadIdx.x;
  const int lane = tr & 31;
  const int num_batches = (range.y - range.x + bs - 1) / bs;
  const size_t pix = pm.inside ? ((size_t)pm.py * img_w + pm.px) : 0;

  const float T_final = pm.inside ? final_Ts[pix] : 1.f;
  float T = T_final;
  float buffer[4] = {0.f, 0.f, 0.f, 0.f};
  const int bin_final = pm.inside ? final_idx[pix] : 0;
  float vo[4] = {0.f, 0.f, 0.f, 0.f};
  float voa = 0.f;
  if (pm.inside) {
#pragma unroll
    for (int c = 0; c < C; ++c) vo[c] = v_output[pix * C + c];
    voa = v_output_alpha ? v_output_alpha[pix] : 0.f;  // NULL = no gradient through alpha
  }
  float bgdot = 0.f;  // sum_c bg_c * v_out_c
#pragma unroll
  for (int c = 0; c < C; ++c) bgdot += background[c] * vo[c];

  // furthest-back index any lane of this warp / any warp of this CTA needs
  int warp_bin_final = bin_final;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) warp_bin_final = max(warp_bin_final, __shfl_xor_sync(0xffffffffu, warp_bin_final, o));
  __shared__ int s_cta_final;
  if (tr == 0) s_cta_final = 0;
  __syncthreads();
  if (lane == 0) atomicMax(&s_cta_final, warp_bin_final);
  __syncthreads();
  const int cta_bin_final = s_cta_final;

  // batches walk back to front; skip batches entirely behind every pixel's last contributor
  int b0 = 0;
  {
    const int last = range.y - 1;
    if (cta_bin_final < last) b0 = (last - cta_bin_final) / bs;
  }
  for (int b = b0; b < num_batches; ++b) {
    __syncthreads();
    const int batch_end = range.y - 1 - bs * b;
    const int batch_size = min(bs, batch_end + 1 - range.x);
    const int idx = batch_end - tr;
    if (idx >= range.x) {
      const int g = gids_sorted[idx];
      s_id[tr] = g;
      const Rec<C> r = gather<C>(g, xys, conics, colors, opacities);
      sb.a[tr] = r.a; sb.b[tr] = r.b; sb.c[tr] = r.c;
    }
#pragma unroll
    for (int k = 0; k < NV; ++k) s_grad[tr][k] = 0.f;
    s_touched[tr] = 0;
    __syncthreads();

    for (int t = max(0, batch_end - warp_bin_final); t < batch_size; ++t) {
      bool valid = pm.inside && (batch_end - t <= bin_final);
      float alpha = 0.f, opac = 0.f, vis = 0.f, dx = 0.f, dy = 0.f;
      float4 ga = make_float4(0.f, 0.f, 0.f, 0.f), gb_ = ga;
      if (valid) {
        ga = sb.a[t];
        gb_ = sb.b[t];
        opac = gb_.y;
        dx = ga.x - px; dy = ga.y - py;
        const float sigma = 0.5f * (ga.z * dx * dx + gb_.x * dy * dy) + ga.w * dx * dy;
        vis = __expf(-sigma);
        alpha = fminf(kAlphaMaxBwd, opac * vis);
        if (sigma < 0.f || alpha < kAlphaMin) valid = false;
      }
      if (!__any_sync(0xffffffffu, valid)) continue;
      float v[NV];
#pragma unroll
      for (int k = 0; k < NV; ++k) v[k] = 0.f;
      if (valid) {
        const float ra = 1.f / (1.f - alpha);
        T *= ra;
        const float fac = alpha * T;
        float col[4];
        const float2 gc = sb.c[t];
        col[0] = gb_.z; col[1] = gb_.w; col[2] = gc.x; col[3] = gc.y;
        float v_alpha = 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
          v[c] = fac * vo[c];
          v_alpha += (col[c] * T - buffer[c] * ra) * vo[c];
        }
        v_alpha += T_final * ra * voa;
        v_alpha += -T_final * ra * bgdot;
#pragma unroll
        for (int c = 0; c < C; ++c) buffer[c] += col[c] * fac;
        const float v_sigma = -opac * vis * v_alpha;
        v[C + 0] = 0.5f * v_sigma * dx * dx;
        v[C + 1] = v_sigma * dx * dy;
        v[C + 2] = 0.5f * v_sigma * dy * dy;
        v[C + 3] = v_sigma * (ga.z * dx + ga.w * dy);
        v[C + 4] = v_sigma * (ga.w * dx + gb_.x * dy);
        v[C + 5] = vis * v_alpha;
      }
#pragma unroll
      for (int k = 0; k < NV; ++k) v[k] = gb::warp_sum(v[k]);
      if (lane < NV) {
        float mine = v[0];
#pragma unroll
        for (int k = 1; k < NV; ++k) mine = (lane == k) ? v[k] : mine;
        atomicAdd(&s_grad[t][lane], mine);
        if (lane == 0) s_touched[t] = 1;
      }
    }
    __syncthreads();
    // flush: one thread per Gaussian of the batch -> one RED set per (tile, Gaussian)
    if (tr < batch_size && s_touched[tr]) {
      const int g = s_id[tr];
#pragma unroll
      for (int c = 0; c < C; ++c) gb::red_add(v_colors + (size_t)C * g + c, s_grad[tr][c]);
      gb::red_add(v_conic + 3 * (size_t)g + 0, s_grad[tr][C + 0]);
      gb::red_add(v_conic + 3 * (size_t)g + 1, s_grad[tr][C + 1]);
      gb::red_add(v_conic + 3 * (size_t)g + 2, s_grad[tr][C + 2]);
      gb::red_add_v2(v_xy + 2 * (size_t)g, s_grad[tr][C + 3], s_grad[tr][C + 4]);
      gb::red_add(v_opacity + g, s_grad[tr][C + 5]);
    }
  }
}

}  // namespace

// replaces gsplat._C.rasterize_forward (3 channels) — and, with channels == 4, the fused rgb+depth pass.
// out_img [H,W,C], final_Ts [H,W], final_idx [H,W] are fully overwritten.
GB_API int gb_rasterize_fwd(int img_h, int img_w, int block_width, int channels, const int32_t* gids_sorted,
                            const int32_t* tile_bins, const float* xys, const float* conics, const float* colors,
                            const float* opacities, const float* background, float* out_img, float* final_Ts,
                            int32_t* final_idx, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if (block_width < 2 || block_width > 16 || (channels != 3 && channels != 4)) return (int)cudaErrorInvalidValue;
  dim3 grid(gb::cdiv(img_w, block_width), gb::cdiv(img_h, block_width));
  const int threads = ((block_width * block_width + 31) / 32) * 32;
  cudaStream_t s = (cudaStream_t)stream;
  if (channels == 3)
    GB_CUDA(gb::launch<rasterize_fwd_kernel<3>>(grid, threads, 0, s, img_w, img_h, block_width, gids_sorted,
                                                (const int2*)tile_bins, (const float2*)xys, conics, colors, opacities,
                                                background, final_Ts, final_idx, out_img));
  else
    GB_CUDA(gb::launch<rasterize_fwd_kernel<4>>(grid, threads, 0, s, img_w, img_h, block_width, gids_sorted,
                                                (const int2*)tile_bins, (const float2*)xys, conics, colors, opacities,
                                                background, final_Ts, final_idx, out_img));
  return 0;
}

// replaces gsplat._C.rasterize_backward.  v_xy [G,2], v_conic [G,3], v_colors [G,C], v_opacity [G]
// are ACCUMULATED into (caller zeroes them), like the reference's atomics.
GB_API int gb_rasterize_bwd(int img_h, int img_w, int block_width, int channels, const int32_t* gids_sorted,
                            const int32_t* tile_bins, const float* xys, const float* conics, const float* colors,
                            const float* opacities, const float* background, const float* final_Ts,
                            const int32_t* final_idx, const float* v_output, const float* v_output_alpha,
                            float* v_xy, float* v_conic, float* v_colors, float* v_opacity, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if (block_width < 2 || block_width > 16 || (channels != 3 && channels != 4)) return (int)cudaErrorInvalidValue;
  dim3 grid(gb::cdiv(img_w, block_width), gb::cdiv(img_h, block_width));
  const int threads = ((block_width * block_width + 31) / 32) * 32;
  cudaStream_t s = (cudaStream_t)stream;
  if (channels == 3)
    GB_CUDA(gb::launch<rasterize_bwd_kernel<3>>(grid, threads, 0, s, img_w, img_h, block_width, gids_sorted,
                                                (const int2*)tile_bins, (const float2*)xys, conics, colors, opacities,
                                                background, final_Ts, final_idx, v_output, v_output_alpha, v_xy,
                                                v_conic, v_colors, v_opacity));
  else
    GB_CUDA(gb::launch<rasterize_bwd_kernel<4>>(grid, threads, 0, s, img_w, img_h, block_width, gids_sorted,
                                                (const int2*)tile_bins, (const float2*)xys, conics, colors, opacities,
                                                background, final_Ts, final_idx, v_output, v_output_alpha, v_xy,
                                                v_conic, v_colors, v_opacity));
  return 0;
}
