// goliath_b200/csrc/splat_blend_common.cuh — constants and device primitives shared by the two packed blend
// formulations (csrc/splat_blend_packed.cu: CTA-synchronous double buffer; csrc/splat_blend_pipe.cu: warp-decoupled
// mbarrier pipeline with a producer warp).  Same arithmetic per (pixel, Gaussian) pair as csrc/splat_blend.cu.
#pragma once
#include "common.cuh"

namespace gbblend {

constexpr int kThreads = 256;
constexpr int kBatch = 256;
constexpr int kRecFloats = 12;  // x y ex ey | A B C opac | c0 c1 c2 c3
constexpr int kRecBytes = kRecFloats * 4;
constexpr float kAlphaMaxFwd = 0.999f;
constexpr float kAlphaMaxBwd = 0.99f;  // gsplat 0.1.x backward constant (oracle: ORC_BWD_ALPHA_CLAMP)
constexpr float kAlphaMin = 1.f / 255.f;
constexpr float kTEps = 1e-4f;
constexpr int kSchedQueues = gb::kNumSMs;  // work queues of the SM-affine tile schedule (gb_tile_schedule)

// ------------------------------------------------------------------ mbarrier / bulk-copy primitives
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
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

// one non-blocking probe of a phase (the instruction itself may suspend the thread for a bounded time)
__device__ __forceinline__ bool mbar_try(unsigned long long* bar, unsigned phase) {
  unsigned ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(phase)
      : "memory");
  return ok != 0;
}
// consumer side of a pipeline stage: one arrival per warp on the stage's "empty" barrier (release semantics)
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// Recursive-halving reduction of 10 per-lane values over the warp: 5+3+2+1+1 = 12 shuffles.
// On return the lane with index L holds the warp total of slot slot_of(L) in `r` (for lanes with an even
// index and a valid slot).  Slot mapping: slot = 5*b4 + 3*b3 + 2*b2 + b1 (bits of the lane index), valid
// when the partial sizes allow it (see slot_valid()).
__device__ __forceinline__ float reduce10(const float (&v)[10], int lane, int& slot, bool& valid) {
  const bool h4 = lane & 16, h3 = lane & 8, h2 = lane & 4, h1 = lane & 2;
  float a[5];
#pragma unroll
  for (int i = 0; i < 5; ++i) {  // xor 16: low half keeps v[0..4], high half keeps v[5..9]
    const float send = h4 ? v[i] : v[5 + i];
    const float keep = h4 ? v[5 + i] : v[i];
    a[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
  float b[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {  // xor 8: low keeps a[0..2], high keeps a[3..4] (+ a zero)
    const float hi_part = (i < 2) ? a[3 + i] : 0.f;
    const float send = h3 ? a[i] : hi_part;
    const float keep = h3 ? hi_part : a[i];
    b[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
  float c[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {  // xor 4: low keeps b[0..1], high keeps b[2] (+ zero)
    const float hi_part = (i < 1) ? b[2] : 0.f;
    const float send = h2 ? b[i] : hi_part;
    const float keep = h2 ? hi_part : b[i];
    c[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  float d;
  {  // xor 2: low keeps c[0], high keeps c[1]
    const float send = h1 ? c[0] : c[1];
    const float keep = h1 ? c[1] : c[0];
    d = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  d += __shfl_xor_sync(0xffffffffu, d, 1);
  // Which slot did this lane end up with?  10 -> (5|5) by b4; 5 -> (3|2) by b3; the (padded) 3 -> (2|1) by b2;
  // 2 -> (1|1) by b1.  Padding positions carry zeros and are reported invalid.
  const int off = (h2 ? 2 : 0) + (h1 ? 1 : 0);          // index inside the part selected by b3
  valid = !(h2 && h1) && (off < (h3 ? 2 : 3));
  slot = (h4 ? 5 : 0) + (h3 ? 3 : 0) + off;
  return d;
}


// Which tile does this CTA blend?  (one thread calls this.)
//  sched == 0: the launch order, order[blockIdx.x] (longest list first) or row-major when order is null.
//  sched == 1: `order` is a schedule written by gb_tile_schedule: position k*Q + q is the k-th item of queue q
//  (Q = kSchedQueues = SM count), Q draw counters and a draw count follow at order[T ..].  The CTA draws the
//  next item of the queue of the SM it runs on, so an SM blends the tiles of ITS queue whatever the block
//  scheduler does, and the queues were filled with near-equal work (with the plain launch order the SMs can finish far
//  apart).  A CTA whose queue
//  is exhausted takes from the following queues (a grid of T CTAs draws exactly T items, one scan finds
//  one), and the launch's last draw puts the counters back to zero for the next launch on this schedule.
__device__ __forceinline__ int draw_tile(const int* order, int sched, int T) {
  if (!sched) return order ? order[blockIdx.x] : (int)blockIdx.x;
  int* cursors = const_cast<int*>(order) + T;
  unsigned smid;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
  int q = (int)(smid % (unsigned)kSchedQueues);
  int tile = -1;
  for (int i = 0; i < kSchedQueues; ++i, q = (q + 1 == kSchedQueues) ? 0 : q + 1) {
    const int cnt = (T > q) ? (T - q + kSchedQueues - 1) / kSchedQueues : 0;
    if (cnt == 0 || *(volatile int*)&cursors[q] >= cnt) continue;  // empty or exhausted queue
    const int slot = atomicAdd(&cursors[q], 1);
    if (slot < cnt) {
      tile = order[slot * kSchedQueues + q];
      break;
    }
  }
  __threadfence();
  if (atomicAdd(&cursors[kSchedQueues], 1) == (int)gridDim.x - 1) {  // every CTA of the launch has drawn
    __threadfence();
    for (int i = 0; i <= kSchedQueues; ++i) cursors[i] = 0;
  }
  return tile;
}

// host-side launchers of the warp-decoupled kernels (csrc/splat_blend_pipe.cu)
// `sched` = 1: tile_order is a schedule written by gb_tile_schedule (CTAs draw their tile from per-SM queues)
int launch_fwd_pipe(int img_h, int img_w, int channels, const int32_t* tile_bins, const int32_t* tile_order, int sched,
                    const float* records, const float* background, float* out_img, float* final_Ts,
                    int32_t* final_idx, cudaStream_t s);
int launch_bwd_pipe(int img_h, int img_w, int channels, const int32_t* gids_sorted, const int32_t* tile_bins,
                    const int32_t* tile_order, int sched, const float* records, const float* background, const float* final_Ts,
                    const int32_t* final_idx, const float* v_output, const float* v_output_alpha, float* v_xy,
                    float* v_conic, float* v_colors, float* v_opacity, cudaStream_t s);

// host-side launchers of the hit-ILP forward / transposed-reduction backward (csrc/splat_blend_mom.cu)
int launch_fwd_mom(int img_h, int img_w, int channels, const int32_t* tile_bins, const int32_t* tile_order, int sched,
                   const float* records, const float* background, float* out_img, float* final_Ts, int32_t* final_idx,
                   cudaStream_t s);
int launch_bwd_mom(int img_h, int img_w, int channels, const int32_t* gids_sorted, const int32_t* tile_bins,
                   const int32_t* tile_order, int sched, const float* records, const float* background, const float* final_Ts,
                   const int32_t* final_idx, const float* v_output, const float* v_output_alpha, float* v_xy,
                   float* v_conic, float* v_colors, float* v_opacity, cudaStream_t s);

}  // namespace gbblend

GB_API int gb_get_blend_mode(void);
GB_API void gb_set_blend_mode(int mode);
