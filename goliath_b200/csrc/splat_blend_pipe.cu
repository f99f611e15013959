// goliath_b200/csrc/splat_blend_pipe.cu — warp-decoupled formulation of the packed blend (sm_90a).
//
// Same records, same per-(pixel, Gaussian) arithmetic and same outputs as csrc/splat_blend_packed.cu (which
// restates gsplat 0.1.11 rasterize_forward / rasterize_backward_kernel, call sites
// ca_code/utils/render_gsplat.py:65-78,90-104); what changes is how the 8 pixel warps of a tile are
// synchronised.  In the CTA-synchronous kernels the per-batch __syncthreads parks warps at the barrier: the warps of a tile see different numbers of footprint hits per batch, and every batch waits for
// the slowest.  Here the warps never meet at a CTA barrier inside the walk:
//
//  forward   records stream through a 4-stage ring of 128-record (6 KB) buffers filled by cp.async.bulk.
//            A 9th warp is the producer: it waits on a stage's "empty" mbarrier (one arrival per pixel warp)
//            and re-arms the "full" mbarrier with the next bulk copy.  Each pixel warp walks the ring at its
//            own pace, up to 3 batches ahead of the slowest.  A warp whose 32 pixels are saturated keeps
//            releasing the stages without touching them (every warp arrives exactly once per batch, so the
//            phases of the barriers stay aligned); when all 8 are saturated the tile is finished: the warps
//            and the producer notice the shared counter while they poll and stop, nothing more is fetched.
//  backward  3-stage ring; every stage has its own shared-memory gradient accumulator.  No producer warp: the
//            LAST warp to finish a stage (shared-memory ticket) flushes that stage's per-Gaussian sums with
//            RED atomics, clears it and issues the bulk copy that refills it, while the other 7 warps are
//            already blending the next stages.
//
// Pixels are bit-identical to the CTA-synchronous kernels (per pixel the records are visited in the same
// order); gradients agree to the order of the floating-point atomics.
//
// Both kernels can also draw their tile from an SM-affine schedule (gb_tile_schedule, draw_tile below) instead of
// taking order[blockIdx.x]; it is an option (GOLIATH_B200_BLEND=affine), not the default.
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "splat_blend_common.cuh"

namespace {

using namespace gbblend;

constexpr int kPixelWarps = 8;
constexpr int kStageRecs = 128;  // records per pipeline stage (6 KB)
constexpr int kFwdStages = 4;
constexpr int kFwdThreads = (kPixelWarps + 1) * 32;  // 8 pixel warps + the producer warp
constexpr int kBwdStages = 3;
constexpr int kBwdThreads = kPixelWarps * 32;

struct Tile {
  int tile_id, tx, ty;
};
__device__ __forceinline__ Tile make_tile(int tile_id, int tbx) {
  Tile t;
  t.tile_id = tile_id;
  t.ty = tile_id / tbx;
  t.tx = tile_id - t.ty * tbx;
  return t;
}

// ------------------------------------------------------------------ forward
template <int C>
__global__ void __launch_bounds__(kFwdThreads) blend_fwd_pipe_kernel(
    int img_w, int img_h, int tbx, const int* order, int sched, const int2* __restrict__ tile_bins,
    const float4* __restrict__ rec, const float* __restrict__ background, float* __restrict__ final_Ts,
    int* __restrict__ final_idx, float* __restrict__ out_img) {
  __shared__ __align__(128) float4 s_rec[kFwdStages][kStageRecs * 3];
  __shared__ __align__(8) unsigned long long s_full[kFwdStages];
  __shared__ __align__(8) unsigned long long s_empty[kFwdStages];
  __shared__ int s_ndone;  // pixel warps whose 32 pixels are saturated
  __shared__ int s_tile;

  const int tr = threadIdx.x, lane = tr & 31, warp = tr >> 5;
  if (tr == 0) {
    s_tile = draw_tile(order, sched, tbx * ((img_h + 15) >> 4));
#pragma unroll
    for (int s = 0; s < kFwdStages; ++s) {
      mbar_init(&s_full[s], 1);
      mbar_init(&s_empty[s], kPixelWarps);
    }
    s_ndone = 0;
    fence_mbar_init();
  }
  __syncthreads();  // the only CTA-wide barrier of this kernel
  if (s_tile < 0) return;
  const Tile tl = make_tile(s_tile, tbx);
  const int2 range = tile_bins[tl.tile_id];
  const int num_batches = (range.y - range.x + kStageRecs - 1) / kStageRecs;

  if (warp == kPixelWarps) {  // ------------------------------ producer warp (one lane)
    if (lane != 0) return;
    volatile int* ndone = &s_ndone;
    int issued = 0;
    for (int b = 0; b < num_batches; ++b) {
      const int s = b % kFwdStages;
      if (b >= kFwdStages) {  // stage s still holds batch b - kFwdStages: wait until all 8 warps have released it
        const unsigned par = (unsigned)(((b / kFwdStages) - 1) & 1);
        while (!mbar_try(&s_empty[s], par) && *ndone < kPixelWarps) {
        }
        if (*ndone >= kPixelWarps) break;  // every pixel of the tile is saturated: nothing more to fetch
      }
      const int start = range.x + b * kStageRecs;
      const unsigned bytes = (unsigned)min(kStageRecs, range.y - start) * kRecBytes;
      mbar_expect_tx(&s_full[s], bytes);
      bulk_g2s(&s_rec[s][0], rec + (size_t)start * 3, bytes, &s_full[s]);
      issued = b + 1;
    }
    // every issued copy must land before the CTA (and its shared memory) retires
    for (int b = max(0, issued - kFwdStages); b < issued; ++b)
      mbar_wait(&s_full[b % kFwdStages], (unsigned)((b / kFwdStages) & 1));
    return;
  }

  // ------------------------------------------------------------ pixel warps: warp w -> 8x4 pixel footprint
  const int wx0 = tl.tx * 16 + ((warp & 1) << 3), wy0 = tl.ty * 16 + ((warp >> 1) << 2);
  const int pxi = wx0 + (lane & 7), pyi = wy0 + (lane >> 3);
  const bool inside = (pxi < img_w) && (pyi < img_h);
  const float px = (float)pxi + 0.5f, py = (float)pyi + 0.5f;
  const float fx0 = (float)wx0 + 0.5f, fx1 = (float)wx0 + 7.5f, fy0 = (float)wy0 + 0.5f, fy1 = (float)wy0 + 3.5f;

  bool done = !inside;
  float T = 1.f;
  int cur_idx = 0;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};

  bool counted = false;  // this warp has been added to s_ndone
  for (int b = 0; b < num_batches; ++b) {
    const bool all_done = __all_sync(0xffffffffu, done);
    if (all_done && !counted) {
      counted = true;
      if (lane == 0) atomicAdd(&s_ndone, 1);
    }
    const int s = b % kFwdStages;
    const unsigned par = (unsigned)((b / kFwdStages) & 1);
    // lane 0 waits for batch b — or, once this warp is saturated, for the moment every warp of the tile is
    int st = 0;
    if (lane == 0) {
      volatile int* ndone = &s_ndone;
      for (;;) {
        if (mbar_try(&s_full[s], par)) { st = 1; break; }
        if (all_done && *ndone >= kPixelWarps) { st = 2; break; }
      }
    }
    st = __shfl_sync(0xffffffffu, st, 0);
    if (st == 2) break;  // tile finished
    if (all_done) {      // saturated warp: release the stage untouched, keep the barrier phases aligned
      if (lane == 0) mbar_arrive(&s_empty[s]);
      continue;
    }
    mbar_wait(&s_full[s], par);  // every lane acquires the landed bytes itself (returns at once)
    const float4* sr = s_rec[s];
    const int batch_start = range.x + b * kStageRecs;
    const int batch_size = min(kStageRecs, range.y - batch_start);
    for (int c0 = 0; c0 < batch_size; c0 += 32) {
      // 32 records' boxes against this warp's footprint
      const int ti = c0 + lane;
      unsigned hit = 0;
      if (ti < batch_size) {
        const float4 q = sr[ti * 3];
        hit = (q.x + q.z >= fx0) && (q.x - q.z <= fx1) && (q.y + q.w >= fy0) && (q.y - q.w <= fy1);
      }
      unsigned mask = __ballot_sync(0xffffffffu, hit);
      while (mask) {
        const int t = c0 + __ffs(mask) - 1;
        mask &= mask - 1;
        const float4 q0 = sr[t * 3], q1 = sr[t * 3 + 1];
        const float dx = q0.x - px, dy = q0.y - py;
        const float sigma = 0.5f * (q1.x * dx * dx + q1.z * dy * dy) + q1.y * dx * dy;
        const float alpha = fminf(kAlphaMaxFwd, q1.w * __expf(-sigma));
        if (done || sigma < 0.f || alpha < kAlphaMin) continue;
        const float next_T = T * (1.f - alpha);
        if (next_T <= kTEps) { done = true; continue; }
        const float4 q2 = sr[t * 3 + 2];
        const float vis = alpha * T;
        acc[0] += q2.x * vis;
        acc[1] += q2.y * vis;
        acc[2] += q2.z * vis;
        if (C == 4) acc[3] += q2.w * vis;
        T = next_T;
        cur_idx = batch_start + t;
      }
      if (__all_sync(0xffffffffu, done)) break;
    }
    __syncwarp();  // every lane's reads of the stage are complete (their values have been consumed)
    if (lane == 0) mbar_arrive(&s_empty[s]);
  }
  if (inside) {
    const size_t pix = (size_t)pyi * img_w + pxi;
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

// ------------------------------------------------------------------ backward
template <int C>
__global__ void __launch_bounds__(kBwdThreads, 4) blend_bwd_pipe_kernel(
    int img_w, int img_h, int tbx, const int* order, int sched, const int* __restrict__ gids_sorted,
    const int2* __restrict__ tile_bins, const float4* __restrict__ rec, const float* __restrict__ background,
    const float* __restrict__ final_Ts, const int* __restrict__ final_idx, const float* __restrict__ v_output,
    const float* __restrict__ v_output_alpha, float* __restrict__ v_xy, float* __restrict__ v_conic,
    float* __restrict__ v_colors, float* __restrict__ v_opacity) {
  constexpr int NV = C + 6;    // colours, conic(3), xy(2), opacity
  constexpr int kStride = 11;  // odd stride: conflict-free flush
  __shared__ __align__(128) float4 s_rec[kBwdStages][kStageRecs * 3];
  __shared__ __align__(8) unsigned long long s_full[kBwdStages];
  __shared__ float s_grad[kBwdStages][kStageRecs * kStride];
  __shared__ int s_touched[kBwdStages][kStageRecs];
  __shared__ int s_ticket[kBwdStages];  // warps that have finished the stage's current batch
  __shared__ int s_cta_final;
  __shared__ int s_tile;

  const int tr = threadIdx.x, lane = tr & 31, warp = tr >> 5;
  if (tr == 0) s_tile = draw_tile(order, sched, tbx * ((img_h + 15) >> 4));
  __syncthreads();
  if (s_tile < 0) return;
  const Tile tl = make_tile(s_tile, tbx);
  const int2 range = tile_bins[tl.tile_id];
  if (range.y <= range.x) return;
  const int wx0 = tl.tx * 16 + ((warp & 1) << 3), wy0 = tl.ty * 16 + ((warp >> 1) << 2);
  const int pxi = wx0 + (lane & 7), pyi = wy0 + (lane >> 3);
  const bool inside = (pxi < img_w) && (pyi < img_h);
  const float px = (float)pxi + 0.5f, py = (float)pyi + 0.5f;
  const float fx0 = (float)wx0 + 0.5f, fx1 = (float)wx0 + 7.5f, fy0 = (float)wy0 + 0.5f, fy1 = (float)wy0 + 3.5f;
  const size_t pix = inside ? ((size_t)pyi * img_w + pxi) : 0;

  const float T_final = inside ? final_Ts[pix] : 1.f;
  float T = T_final;
  float buffer[4] = {0.f, 0.f, 0.f, 0.f};
  const int bin_final = inside ? final_idx[pix] : 0;
  float vo[4] = {0.f, 0.f, 0.f, 0.f};
  float voa = 0.f;
  if (inside) {
#pragma unroll
    for (int c = 0; c < C; ++c) vo[c] = v_output[pix * C + c];
    voa = v_output_alpha ? v_output_alpha[pix] : 0.f;  // NULL = no gradient through alpha
  }
  float bgdot = 0.f;
#pragma unroll
  for (int c = 0; c < C; ++c) bgdot += background[c] * vo[c];

  int warp_bin_final = bin_final;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) warp_bin_final = max(warp_bin_final, __shfl_xor_sync(0xffffffffu, warp_bin_final, o));
  if (tr == 0) {
    s_cta_final = 0;
#pragma unroll
    for (int s = 0; s < kBwdStages; ++s) {
      mbar_init(&s_full[s], 1);
      s_ticket[s] = 0;
    }
    fence_mbar_init();
  }
  for (int i = tr; i < kBwdStages * kStageRecs * kStride; i += kBwdThreads) (&s_grad[0][0])[i] = 0.f;
  for (int i = tr; i < kBwdStages * kStageRecs; i += kBwdThreads) (&s_touched[0][0])[i] = 0;
  __syncthreads();
  if (lane == 0) atomicMax(&s_cta_final, warp_bin_final);
  __syncthreads();
  // the walk starts at the last index any pixel of the tile needs and goes down to range.x
  const int last = min(s_cta_final, range.y - 1);
  if (last < range.x) return;  // no pixel of this tile blended anything (CTA-uniform: nothing is in flight yet)
  const int num_batches = (last - range.x + kStageRecs) / kStageRecs;  // ceil((last - range.x + 1) / kStageRecs)
  // batch k (k = 0 is the furthest back) covers indices [hi_k - size_k + 1, hi_k], hi_k = last - k*kStageRecs
  auto issue = [&](int k) {  // one lane
    const int s = k % kBwdStages;
    const int hi = last - k * kStageRecs;
    const int lo = max(range.x, hi - kStageRecs + 1);
    const unsigned bytes = (unsigned)(hi - lo + 1) * kRecBytes;
    mbar_expect_tx(&s_full[s], bytes);
    bulk_g2s(&s_rec[s][0], rec + (size_t)lo * 3, bytes, &s_full[s]);
  };
  if (tr == 0)
    for (int k = 0; k < min(kBwdStages, num_batches); ++k) issue(k);
  // no CTA-wide barrier below this line

  for (int k = 0; k < num_batches; ++k) {
    const int s = k % kBwdStages;
    const int hi = last - k * kStageRecs;
    const int lo = max(range.x, hi - kStageRecs + 1);
    const int batch_size = hi - lo + 1;
    mbar_wait(&s_full[s], (unsigned)((k / kBwdStages) & 1));
    const float4* sr = s_rec[s];
    float* sgrad = s_grad[s];
    int* stouched = s_touched[s];
    // slot j of the stage holds sorted index lo + j; walk j downwards, 32 at a time
    const int j_top = min(batch_size - 1, warp_bin_final - lo);  // nothing above this index matters to the warp
    for (int c1 = (j_top & ~31); c1 >= 0 && j_top >= 0; c1 -= 32) {
      const int tj = c1 + lane;
      unsigned hit = 0;
      if (tj <= j_top) {
        const float4 q = sr[tj * 3];
        hit = (q.x + q.z >= fx0) && (q.x - q.z <= fx1) && (q.y + q.w >= fy0) && (q.y - q.w <= fy1);
      }
      unsigned mask = __ballot_sync(0xffffffffu, hit);
      while (mask) {
        const int bit = 31 - __clz(mask);
        mask &= ~(1u << bit);
        const int j = c1 + bit;
        bool valid = inside && (lo + j <= bin_final);
        const float4 q0 = sr[j * 3], q1 = sr[j * 3 + 1];
        const float dx = q0.x - px, dy = q0.y - py;
        const float sigma = 0.5f * (q1.x * dx * dx + q1.z * dy * dy) + q1.y * dx * dy;
        const float vis = __expf(-sigma);
        const float opac = q1.w;
        const float alpha = fminf(kAlphaMaxBwd, opac * vis);
        if (sigma < 0.f || alpha < kAlphaMin) valid = false;
        if (!__any_sync(0xffffffffu, valid)) continue;
        float v[10];
#pragma unroll
        for (int i = 0; i < 10; ++i) v[i] = 0.f;
        if (valid) {
          const float4 q2 = sr[j * 3 + 2];
          const float ra = 1.f / (1.f - alpha);
          T *= ra;
          const float fac = alpha * T;
          const float col[4] = {q2.x, q2.y, q2.z, q2.w};
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
          v[C + 3] = v_sigma * (q1.x * dx + q1.y * dy);
          v[C + 4] = v_sigma * (q1.y * dx + q1.z * dy);
          v[C + 5] = vis * v_alpha;
        }
        int slot;
        bool sv;
        const float r = reduce10(v, lane, slot, sv);
        if (!(lane & 1) && sv && slot < NV) atomicAdd(&sgrad[j * kStride + slot], r);
        if (lane == 0) stouched[j] = 1;
      }
    }
    // ticket: the last of the 8 warps through this stage flushes it and recycles it
    __syncwarp();
    int ticket = 0;
    if (lane == 0) {
      __threadfence_block();  // release: this warp's shared-memory sums and its reads of the stage
      ticket = atomicAdd(&s_ticket[s], 1);
    }
    ticket = __shfl_sync(0xffffffffu, ticket, 0);
    if (ticket == kPixelWarps - 1) {
      __threadfence_block();  // acquire: the other warps' sums
      for (int j = lane; j < batch_size; j += 32) {
        if (!stouched[j]) continue;
        stouched[j] = 0;
        const int g = gids_sorted[lo + j];
        float* sg = &sgrad[j * kStride];
#pragma unroll
        for (int c = 0; c < C; ++c) gb::red_add(v_colors + (size_t)C * g + c, sg[c]);
        gb::red_add(v_conic + 3 * (size_t)g + 0, sg[C + 0]);
        gb::red_add(v_conic + 3 * (size_t)g + 1, sg[C + 1]);
        gb::red_add(v_conic + 3 * (size_t)g + 2, sg[C + 2]);
        gb::red_add_v2(v_xy + 2 * (size_t)g, sg[C + 3], sg[C + 4]);
        gb::red_add(v_opacity + g, sg[C + 5]);
#pragma unroll
        for (int c = 0; c < NV; ++c) sg[c] = 0.f;
      }
      __syncwarp();
      if (lane == 0) {
        s_ticket[s] = 0;
        if (k + kBwdStages < num_batches) issue(k + kBwdStages);  // arrive.expect_tx releases the reset and the clears
      }
    }
  }
}

constexpr int kDefaultBlendMode = 3;  // round 2: hit-ILP forward + transposed-reduction backward (splat_blend_mom.cu)
int g_blend_mode = -1;  // 0: CTA-synchronous (splat_blend_packed.cu), 1: warp-decoupled pipeline, 2: + SM-affine schedule,
                        // 3: exact cull + 4-hit ILP forward + transposed (moment) backward (splat_blend_mom.cu),
                        // 4: mode 3 drawing its tiles from the SM-affine schedule

}  // namespace

// Blend formulation: 0 = CTA-synchronous double buffer, 1 = warp-decoupled pipeline, 2 = warp-decoupled pipeline
// over an SM-affine schedule, 3 = exact cull + hit-ILP forward + transposed-reduction backward (default).
// gb_rasterize_packed_fwd/bwd dispatch on it; callers that can provide a schedule (gb_tile_schedule: the fused
// render, bench.py) use gb_rasterize_sched_fwd/bwd in mode 2.  Default from the environment
// (GOLIATH_B200_BLEND=batch|pipe|affine|mom).  Pixels are identical bit for bit in every mode; gradients agree to
// the order of the atomics in modes 0-2 and to fp32 re-association (1e-5 relative) in mode 3.  The switch exists
// for A/B timing and the parity tests.
GB_API int gb_get_blend_mode(void) {
  if (g_blend_mode < 0) {
    const char* e = getenv("GOLIATH_B200_BLEND");
    g_blend_mode = !e ? kDefaultBlendMode
                   : strcmp(e, "batch") == 0 ? 0
                   : strcmp(e, "pipe") == 0  ? 1
                   : strcmp(e, "affine") == 0 ? 2
                   : strcmp(e, "mom") == 0    ? 3
                                              : 4;  // "mom-affine"
  }
  return g_blend_mode;
}
GB_API void gb_set_blend_mode(int mode) { g_blend_mode = mode < 0 ? 0 : (mode > 4 ? 4 : mode); }

// Blend over an SM-affine schedule (gb_tile_schedule): the warp-decoupled kernels, each CTA drawing its tile from
// the queue of the SM it runs on.  Same arguments and outputs as gb_rasterize_packed_fwd / _bwd.
GB_API int gb_rasterize_sched_fwd(int img_h, int img_w, int channels, const int32_t* tile_bins, int32_t* sched,
                                  const float* records, const float* background, float* out_img, float* final_Ts,
                                  int32_t* final_idx, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if (channels != 3 && channels != 4) return (int)cudaErrorInvalidValue;
  if (gb_get_blend_mode() >= 3)
    return gbblend::launch_fwd_mom(img_h, img_w, channels, tile_bins, sched, 1, records, background, out_img, final_Ts,
                                   final_idx, (cudaStream_t)stream);
  return gbblend::launch_fwd_pipe(img_h, img_w, channels, tile_bins, sched, 1, records, background, out_img, final_Ts,
                                  final_idx, (cudaStream_t)stream);
}
GB_API int gb_rasterize_sched_bwd(int img_h, int img_w, int channels, const int32_t* gids_sorted,
                                  const int32_t* tile_bins, int32_t* sched, const float* records,
                                  const float* background, const float* final_Ts, const int32_t* final_idx,
                                  const float* v_output, const float* v_output_alpha, float* v_xy, float* v_conic,
                                  float* v_colors, float* v_opacity, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if (channels != 3 && channels != 4) return (int)cudaErrorInvalidValue;
  if (gb_get_blend_mode() >= 3)
    return gbblend::launch_bwd_mom(img_h, img_w, channels, gids_sorted, tile_bins, sched, 1, records, background,
                                   final_Ts, final_idx, v_output, v_output_alpha, v_xy, v_conic, v_colors, v_opacity,
                                   (cudaStream_t)stream);
  return gbblend::launch_bwd_pipe(img_h, img_w, channels, gids_sorted, tile_bins, sched, 1, records, background,
                                  final_Ts, final_idx, v_output, v_output_alpha, v_xy, v_conic, v_colors, v_opacity,
                                  (cudaStream_t)stream);
}

namespace gbblend {

int launch_fwd_pipe(int img_h, int img_w, int channels, const int32_t* tile_bins, const int32_t* tile_order, int sched,
                    const float* records, const float* background, float* out_img, float* final_Ts,
                    int32_t* final_idx, cudaStream_t s) {
  const int tbx = gb::cdiv(img_w, 16), tby = gb::cdiv(img_h, 16);
  if (sched && !tile_order) return (int)cudaErrorInvalidValue;
  if (channels == 3)
    GB_CUDA(gb::launch<blend_fwd_pipe_kernel<3>>(tbx * tby, kFwdThreads, 0, s, img_w, img_h, tbx, tile_order, sched,
                                                 (const int2*)tile_bins, (const float4*)records, background, final_Ts,
                                                 final_idx, out_img));
  else
    GB_CUDA(gb::launch<blend_fwd_pipe_kernel<4>>(tbx * tby, kFwdThreads, 0, s, img_w, img_h, tbx, tile_order, sched,
                                                 (const int2*)tile_bins, (const float4*)records, background, final_Ts,
                                                 final_idx, out_img));
  return 0;
}

int launch_bwd_pipe(int img_h, int img_w, int channels, const int32_t* gids_sorted, const int32_t* tile_bins,
                    const int32_t* tile_order, int sched, const float* records, const float* background, const float* final_Ts,
                    const int32_t* final_idx, const float* v_output, const float* v_output_alpha, float* v_xy,
                    float* v_conic, float* v_colors, float* v_opacity, cudaStream_t s) {
  const int tbx = gb::cdiv(img_w, 16), tby = gb::cdiv(img_h, 16);
  if (sched && !tile_order) return (int)cudaErrorInvalidValue;
  if (channels == 3)
    GB_CUDA(gb::launch<blend_bwd_pipe_kernel<3>>(tbx * tby, kBwdThreads, 0, s,
        img_w, img_h, tbx, tile_order, sched, gids_sorted, (const int2*)tile_bins, (const float4*)records, background, final_Ts,
        final_idx, v_output, v_output_alpha, v_xy, v_conic, v_colors, v_opacity));
  else
    GB_CUDA(gb::launch<blend_bwd_pipe_kernel<4>>(tbx * tby, kBwdThreads, 0, s,
        img_w, img_h, tbx, tile_order, sched, gids_sorted, (const int2*)tile_bins, (const float4*)records, background, final_Ts,
        final_idx, v_output, v_output_alpha, v_xy, v_conic, v_colors, v_opacity));
  return 0;
}

}  // namespace gbblend
