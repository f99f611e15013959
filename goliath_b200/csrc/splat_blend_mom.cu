// goliath_b200/csrc/splat_blend_mom.cu — third formulation of the packed blend (sm_90a), blend mode 3 (default).
//
// Same records, same per-(pixel, Gaussian) arithmetic in the forward and the same gradients as
// csrc/splat_blend_pipe.cu (gsplat 0.1.11 rasterize_forward / rasterize_backward_kernel, call sites
// ca_code/utils/render_gsplat.py:65-78,90-104).  The pipeline kernels are bound in both directions by the per-warp
// issue rate on the heaviest tile: a dependent chain of LDS -> FMA -> ex2 -> shuffles -> shared-memory CAS atomics
// per footprint hit in the backward.  What changes here:
//
//  cull      the 32-lane record test is the exact minimum of the Gaussian's quadratic form over the warp's 8x4
//            pixel rectangle (a convex QP on a box: the minimiser lies on one of the two faces visible from the
//            centre), compared with log(255 * opacity); the axis-aligned box of round 1 passed 10-45 % false hits.
//  forward   footprint hits are blended four at a time: the four alphas (loads, quadratic form, ex2) are
//            independent and issue back to back, only the transmittance recurrence is serial.  Pixels stay
//            bit-identical to the other formulations (same operations in the same order per pixel).
//  backward  TRANSPOSED reduction.  Hits are compacted into a per-warp list of entries (a copy of the record plus
//            its sorted index).  For a chunk of 16 entries, phase A runs with lanes = pixels: the serial
//            transmittance / colour-buffer recurrence, writing (fac, v_sigma) of every (hit, pixel) pair into a
//            16 x 32 shared-memory matrix (odd row stride).  Phase B runs with lanes = (hit, half of the
//            footprint): a lane reads ITS hit's row and accumulates v_colour = sum fac * v_out and the image
//            moments S0, Si, Sj, Sii, Sij of v_sigma over the pixels (pixel offsets are compile-time constants),
//            from which v_conic, v_xy and v_opacity follow in closed form (dx = u - i, dy = v - j).  One xor-16
//            shuffle of the 10 sums replaces the 12-shuffle recursive halving PER HIT of round 1, and the lane
//            that owns the hit adds it to the global gradient arrays with RED (vector RED for the colours): no
//            shared-memory float atomics (CAS loops in SASS), no per-stage accumulators, no flush tickets.
//            1 / (1 - alpha) uses rcp.approx (gradients have a 1e-4 bar, not bit parity).
//
// Stages are recycled as in the pipeline kernels (mbarrier ring, cp.async.bulk), but a warp has finished with a
// stage as soon as it has culled it — the entries carry what phases A and B need.
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "splat_blend_common.cuh"
#include "splat_tile_sort.cuh"

namespace {

using namespace gbblend;

constexpr int kPixelWarps = 8;
constexpr int kStageRecs = 128;  // records per pipeline stage (6 KB)
constexpr int kFwdStages = 4;
constexpr int kFwdThreads = (kPixelWarps + 1) * 32;
constexpr int kBwdStages = 3;
constexpr int kBwdThreads = kPixelWarps * 32;
constexpr int kChunk = 16;            // hits per transposed-reduction chunk
constexpr int kEntryCap = 48;         // pending entries per warp: < kChunk left over + up to 32 new
constexpr int kMStride = 33;          // float2 row stride of the (hit, pixel) matrix: odd -> conflict-free both ways
constexpr float kCullMargin = 2e-3f;  // slack of the exact cull test (ex2.approx / lg2.approx / rounding)

__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// __expf(-s) with flush-to-zero: ex2.approx of s * -log2(e) without the denormal range guard (3 instructions per hit).
// Results differ from __expf only where the result is below 2^-126, i.e. alpha < 1/255: skipped either way.
__device__ __forceinline__ float exp_neg(float s) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(s * -1.4426950408889634f));
  return r;
}

// RANKED staging: the tile's list is a list of sorted Gaussian ids (4 B) into the by-id record table [G,12] written
// once per Gaussian by the binning; a stage is filled by 16-byte cp.async gathers (three per record) instead of one
// bulk copy of materialised sorted records, which removes the binning's record gather (52 MB written + read per view).
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// arrival on `bar` once every cp.async this thread has issued so far has landed (the barrier's count includes it)
__device__ __forceinline__ void cp_async_arrive(unsigned long long* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// Does the record (centre (x, y), conic (A, B, Cc), opacity o) reach alpha >= 1/255 anywhere on the rectangle of pixel
// centres [fx0, fx1] x [fy0, fy1]?  d = centre - pixel ranges over [x - fx1, x - fx0] x [y - fy1, y - fy0]; sigma(d) is
// a positive-definite quadratic with its minimum at d = 0.  If 0 is outside the rectangle the minimiser lies on a face
// from which the segment to 0 leaves the rectangle, i.e. on the line d.x = ex0 or d.y = ey0 (ex0, ey0 = the
// coordinates of the rectangle nearest to 0); on each line the 1-D minimiser is clamped to the face.  Both candidates
// are feasible points, so min(f1, f2) >= the true minimum, and one of them attains it.  (ex, ey) is the round-1 box
// (kept as a cheap pre-test and as the "never cull" marker 3e38 for malformed conics).
__device__ __forceinline__ bool footprint_hit(const float4 q0, const float4* __restrict__ q1p, float fx0, float fx1,
                                              float fy0, float fy1) {
  if (!((q0.x + q0.z >= fx0) && (q0.x - q0.z <= fx1) && (q0.y + q0.w >= fy0) && (q0.y - q0.w <= fy1))) return false;
  if (q0.z > 1e30f) return true;  // malformed conic / opacity: the per-pixel test decides
  const float4 q1 = *q1p;         // A B C o
  const float dxlo = q0.x - fx1, dxhi = q0.x - fx0, dylo = q0.y - fy1, dyhi = q0.y - fy0;
  const float ex0 = fminf(fmaxf(0.f, dxlo), dxhi), ey0 = fminf(fmaxf(0.f, dylo), dyhi);
  const float dy1 = fminf(fmaxf(-q1.y * ex0 * rcp_approx(q1.z), dylo), dyhi);
  const float dx2 = fminf(fmaxf(-q1.y * ey0 * rcp_approx(q1.x), dxlo), dxhi);
  const float f1 = 0.5f * (q1.x * ex0 * ex0 + q1.z * dy1 * dy1) + q1.y * ex0 * dy1;
  const float f2 = 0.5f * (q1.x * dx2 * dx2 + q1.z * ey0 * ey0) + q1.y * dx2 * ey0;
  const float s = __logf(255.f * q1.w);
  return fminf(f1, f2) <= s + kCullMargin + 1e-4f * fabsf(s);
}

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
// LIST = false: a round takes up to four hits of the current 32-record cull step (a step with 9 hits costs 3 rounds, 12 slots).
// LIST = true : the warp first culls the whole stage (up to 128 records, four independent tests in flight) into a
//               per-warp list of hit indices, then blends the list four entries per round (one LDS.128 fetches the four
//               indices): rounds are full except the last one of a stage, and the mask walk (brev / flo / lop per hit
//               on the uniform path) is gone.  Same per-pixel operations in the same order -> identical pixels.
// HITS (with LIST): each pixel warp also stores its hit lists for blend_bwd_lists_kernel.  Warp w of a tile with list
//               range [x, y) appends the sorted indices of its hits, stage after stage, at hit_list[8x + w(y - x)] (a
//               warp cannot hit more than y - x records, so the segments never overlap and need no device-side count),
//               and writes hit_count[8 tile + w] = the number of leading entries the backward needs: up to and
//               including the last hit any pixel of the warp blended (the backward's `idx <= final_idx` walk).  Block 0
//               sets hit_count[8T], the backward's draw counter, to zero.  Only stores are added: pixels stay identical.
// SORT (with LIST, RANKED and HITS): the CTA first sorts its tile's bucket by (depth, id) with all its threads
//               (FwdSort::sort_tile, the algorithm of the binning's tile_sort_kernel): bucket holds the tile's ids in
//               arbitrary order and `sorted` their depth keys at the same slots (gb_bin_tiles_buckets); `sorted`
//               receives the ids in blend order, the array the backward's hit lists index, and the producer stages from
//               it.  The sort's buffers alias the stage ring and the hit lists, which are not live before the blend.
//               Pixels and hit lists are those of the HITS variant run on tile_sort_kernel's output.
// 15 entries per thread: the longest tile of the bench head (4223 entries) stays in shared memory; longer tiles take the
// chunked path through global memory inside the CTA.
using FwdSort = gbsort::TileSort<kFwdThreads, 15>;

template <bool LIST>
struct FwdRing {
  float4 rec[kFwdStages][kStageRecs * 3];
  int hits[LIST ? kPixelWarps : 1][LIST ? kStageRecs + 4 : 4];
};
template <bool LIST, bool SORT>
struct FwdSmem {
  FwdRing<LIST> f;
};
template <bool LIST>
struct FwdSmem<LIST, true> {
  union {
    FwdRing<LIST> f;
    struct {
      unsigned long long key[FwdSort::kCap];
      FwdSort::Smem s;
    } sort;
  };
};

template <int C, bool LIST, bool RANKED, bool HITS, bool SORT, bool FINISH = false>
__device__ __forceinline__ void blend_fwd_body(
    int img_w, int img_h, int tbx, const int* order, int sched, const int2* __restrict__ tile_bins,
    const float4* __restrict__ rec /* RANKED: the by-rank table */, const int* __restrict__ ranks /* RANKED only */,
    const float* __restrict__ background, float* __restrict__ final_Ts, int* __restrict__ final_idx,
    float* __restrict__ out_img, int* __restrict__ hit_list, int* __restrict__ hit_count,
    const unsigned* __restrict__ depth_keys /* SORT only */, int* bucket /* SORT only */,
    int* sorted /* SORT only: depth keys in, ids in blend order out */,
    float* __restrict__ alpha_img = nullptr /* FINISH only */, float* __restrict__ depth_img = nullptr /* FINISH only */) {
  static_assert(!HITS || LIST, "hit lists are the LIST variant's per-stage lists");
  static_assert(!SORT || (LIST && RANKED && HITS), "the sorting forward is the ranked hit-list forward");
  static_assert(!FINISH || C == 4, "the finished view is rgb + depth");
  __shared__ __align__(128) FwdSmem<LIST, SORT> sm;
  float4 (&s_rec)[kFwdStages][kStageRecs * 3] = sm.f.rec;
  auto& s_hits = sm.f.hits;
  __shared__ __align__(8) unsigned long long s_full[kFwdStages];
  __shared__ __align__(8) unsigned long long s_empty[kFwdStages];
  __shared__ int s_ndone;  // pixel warps whose 32 pixels are saturated
  __shared__ int s_tile;
  // SORT: the ids are read back from `sorted`, which this CTA has just written (plain loads, not the read-only path)
  const int* rk = SORT ? sorted : ranks;

  const int tr = threadIdx.x, lane = tr & 31, warp = tr >> 5;
  if (tr == 0) {
    s_tile = draw_tile(order, sched, tbx * ((img_h + 15) >> 4));
#pragma unroll
    for (int s = 0; s < kFwdStages; ++s) {
      mbar_init(&s_full[s], RANKED ? 32 : 1);
      mbar_init(&s_empty[s], kPixelWarps);
    }
    s_ndone = 0;
    fence_mbar_init();
  }
  __syncthreads();  // the only CTA-wide barrier of this kernel besides the sort's
  if (s_tile < 0) return;
  const Tile tl = make_tile(s_tile, tbx);
  const int2 range = tile_bins[tl.tile_id];
  if constexpr (SORT) {
    if (range.y > range.x) FwdSort::sort_tile(range, depth_keys, bucket, sorted, sm.sort.key, sm.sort.s);
  }
  const int num_batches = (range.y - range.x + kStageRecs - 1) / kStageRecs;

  if (RANKED && warp == kPixelWarps) {  // --------------------- producer warp, all lanes: gathers by rank
    volatile int* ndone = &s_ndone;
    // the ranks of stage b + 1 are loaded while the producer waits for stage b's slot: the per-stage chain is then one
    // L2 round trip (the gathers), not two
    int r[4];
    auto load_ranks = [&](int b) {
      const int start = range.x + b * kStageRecs;
      const int count = min(kStageRecs, range.y - start);
#pragma unroll
      for (int k = 0; k < 4; ++k) r[k] = (b < num_batches && lane + 32 * k < count) ? rk[start + lane + 32 * k] : -1;
    };
    load_ranks(0);
    for (int b = 0; b < num_batches; ++b) {
      const int s = b % kFwdStages;
      if (b >= kFwdStages) {
        int go = 1;
        if (lane == 0) {
          const unsigned par = (unsigned)(((b / kFwdStages) - 1) & 1);
          while (!mbar_try(&s_empty[s], par) && *ndone < kPixelWarps) {
        }
          go = *ndone < kPixelWarps;
        }
        go = __shfl_sync(0xffffffffu, go, 0);
        if (!go) break;
      }
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (r[k] >= 0) {
          const float4* src = rec + 3 * (size_t)r[k];
          float4* dst = &s_rec[s][3 * (lane + 32 * k)];
          cp_async16(dst, src);
          cp_async16(dst + 1, src + 1);
          cp_async16(dst + 2, src + 2);
        }
      cp_async_arrive(&s_full[s]);
      load_ranks(b + 1);
    }
    cp_async_wait_all();  // every issued copy lands before the CTA retires
    return;
  }
  if (warp == kPixelWarps) {  // ------------------------------ producer warp (one lane)
    if (lane != 0) return;
    volatile int* ndone = &s_ndone;
    int issued = 0;
    for (int b = 0; b < num_batches; ++b) {
      const int s = b % kFwdStages;
      if (b >= kFwdStages) {
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
    for (int b = max(0, issued - kFwdStages); b < issued; ++b)  // every issued copy lands before the CTA retires
      mbar_wait(&s_full[b % kFwdStages], (unsigned)((b / kFwdStages) & 1));
    return;
  }

  const int wx0 = tl.tx * 16 + ((warp & 1) << 3), wy0 = tl.ty * 16 + ((warp >> 1) << 2);
  const int pxi = wx0 + (lane & 7), pyi = wy0 + (lane >> 3);
  const bool inside = (pxi < img_w) && (pyi < img_h);
  const float px = (float)pxi + 0.5f, py = (float)pyi + 0.5f;
  const float fx0 = (float)wx0 + 0.5f, fx1 = (float)wx0 + 7.5f, fy0 = (float)wy0 + 0.5f, fy1 = (float)wy0 + 3.5f;

  bool done = !inside;
  float T = 1.f;
  int cur_idx = 0;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  // HITS: this warp's list segment, entries stored so far, and the list position of the pixel's last blended hit
  int* const seg = HITS ? hit_list + 8 * (size_t)range.x + (size_t)warp * (range.y - range.x) : nullptr;
  int written = 0, last_pos = -1;

  bool counted = false;
  for (int b = 0; b < num_batches; ++b) {
    const bool all_done = __all_sync(0xffffffffu, done);
    if (all_done && !counted) {
      counted = true;
      if (lane == 0) atomicAdd(&s_ndone, 1);
    }
    const int s = b % kFwdStages;
    const unsigned par = (unsigned)((b / kFwdStages) & 1);
    int st = 0;
    if (lane == 0) {
      volatile int* ndone = &s_ndone;
      for (;;) {
        if (mbar_try(&s_full[s], par)) { st = 1; break; }
        if (all_done && *ndone >= kPixelWarps) { st = 2; break; }
        // (many of this kernel's executed instructions are these single-lane probes, mostly saturated warps waiting
        // at the producer's frontier.  They are not parked with __nanosleep: the probes use issue slots nobody else
        // wants, while the wake-up latency of a parked warp lands on the critical path.)
      }
    }
    st = __shfl_sync(0xffffffffu, st, 0);
    if (st == 2) break;  // tile finished
    if (all_done) {      // saturated warp: release the stage untouched, keep the barrier phases aligned
      if (lane == 0) mbar_arrive(&s_empty[s]);
      continue;
    }
    mbar_wait(&s_full[s], par);
    const float4* sr = s_rec[s];
    const int batch_start = range.x + b * kStageRecs;
    const int batch_size = min(kStageRecs, range.y - batch_start);
    if (LIST) {
      int* hl = s_hits[LIST ? warp : 0];
      const unsigned lt = (1u << lane) - 1u;
      int cnt = 0;
#pragma unroll 4
      for (int c0 = 0; c0 < batch_size; c0 += 32) {
        const int ti = c0 + lane;
        bool hit = false;
        if (ti < batch_size) hit = footprint_hit(sr[ti * 3], &sr[ti * 3 + 1], fx0, fx1, fy0, fy1);
        const unsigned mask = __ballot_sync(0xffffffffu, hit);
        if (hit) hl[cnt + __popc(mask & lt)] = ti;
        cnt += __popc(mask);
      }
      __syncwarp();
      if (HITS) {
        for (int i = lane; i < cnt; i += 32) seg[written + i] = batch_start + hl[i];
        // a pixel that blends nothing keeps final_idx = 0, which the backward's walk still includes
        if (b == 0 && range.x == 0 && cnt > 0 && hl[0] == 0 && inside) last_pos = 0;
      }
      for (int i0 = 0; i0 < cnt; i0 += 16) {  // saturation is polled every four rounds
        const int i1 = min(i0 + 16, cnt);
        for (int i = i0; i < i1; i += 4) {
          const int4 e = *reinterpret_cast<const int4*>(hl + i);
          bool live[4];
          int t[4];
          live[0] = true; live[1] = i + 1 < cnt; live[2] = i + 2 < cnt; live[3] = i + 3 < cnt;
          t[0] = e.x; t[1] = live[1] ? e.y : e.x; t[2] = live[2] ? e.z : e.x; t[3] = live[3] ? e.w : e.x;
          float alpha[4], sig[4];
          float4 col[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float4 q0 = sr[t[u] * 3], q1 = sr[t[u] * 3 + 1];
            col[u] = sr[t[u] * 3 + 2];
            const float dx = q0.x - px, dy = q0.y - py;
            sig[u] = 0.5f * (q1.x * dx * dx + q1.z * dy * dy) + q1.y * dx * dy;
            alpha[u] = fminf(kAlphaMaxFwd, q1.w * exp_neg(sig[u]));
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const bool ok = live[u] && !done && !(sig[u] < 0.f) && !(alpha[u] < kAlphaMin);
            const float next_T = T * (1.f - alpha[u]);
            const bool stop = ok && (next_T <= kTEps);
            const bool take = ok && !stop;
            done = done || stop;
            if (take) {
              const float vis = alpha[u] * T;
              acc[0] += col[u].x * vis;
              acc[1] += col[u].y * vis;
              acc[2] += col[u].z * vis;
              if (C == 4) acc[3] += col[u].w * vis;
              T = next_T;
              cur_idx = batch_start + t[u];
              if (HITS) last_pos = written + i + u;
            }
          }
        }
        if (__all_sync(0xffffffffu, done)) break;
      }
      written += cnt;
    } else {
    for (int c0 = 0; c0 < batch_size; c0 += 32) {
        const int ti = c0 + lane;
        bool hit = false;
        if (ti < batch_size) hit = footprint_hit(sr[ti * 3], &sr[ti * 3 + 1], fx0, fx1, fy0, fy1);
        unsigned mask = __ballot_sync(0xffffffffu, hit);
        while (mask) {
          // up to four hits per round: independent alphas, serial transmittance
          int t[4];
          bool live[4];
  #pragma unroll
          for (int u = 0; u < 4; ++u) {
            live[u] = mask != 0;
            t[u] = live[u] ? c0 + __ffs(mask) - 1 : t[0];
            mask &= mask - 1;  // 0 & anything == 0
          }
          float alpha[4], sig[4];
          float4 col[4];
  #pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float4 q0 = sr[t[u] * 3], q1 = sr[t[u] * 3 + 1];
            col[u] = sr[t[u] * 3 + 2];
            const float dx = q0.x - px, dy = q0.y - py;
            sig[u] = 0.5f * (q1.x * dx * dx + q1.z * dy * dy) + q1.y * dx * dy;
            alpha[u] = fminf(kAlphaMaxFwd, q1.w * __expf(-sig[u]));
          }
  #pragma unroll
          for (int u = 0; u < 4; ++u) {
            const bool ok = live[u] && !done && !(sig[u] < 0.f) && !(alpha[u] < kAlphaMin);
            const float next_T = T * (1.f - alpha[u]);
            const bool stop = ok && (next_T <= kTEps);
            const bool take = ok && !stop;
            done = done || stop;
            if (take) {
              const float vis = alpha[u] * T;
              acc[0] += col[u].x * vis;
              acc[1] += col[u].y * vis;
              acc[2] += col[u].z * vis;
              if (C == 4) acc[3] += col[u].w * vis;
              T = next_T;
              cur_idx = batch_start + t[u];
            }
          }
        }
        if (__all_sync(0xffffffffu, done)) break;
      }
  }
    __syncwarp();
    if (lane == 0) mbar_arrive(&s_empty[s]);
  }
  if (HITS) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) last_pos = max(last_pos, __shfl_xor_sync(0xffffffffu, last_pos, o));
    if (lane == 0) hit_count[8 * tl.tile_id + warp] = last_pos + 1;
    if (blockIdx.x == 0 && tr == 0) hit_count[8 * tbx * ((img_h + 15) >> 4)] = 0;
  }
  if (inside) {
    const size_t pix = (size_t)pyi * img_w + pxi;
    final_Ts[pix] = T;
    final_idx[pix] = cur_idx;
    if (FINISH) {
      // render_finish.cu's finish_fwd_kernel on the pixel in registers, alpha = 1 - T as torch's rsub computes it:
      // out_img is rgb [3,H,W], the depth channel's background is background[0] (the 4-channel blend's bg[3])
      const size_t P = (size_t)img_w * img_h;
      out_img[pix] = acc[0] + T * background[0];
      out_img[P + pix] = acc[1] + T * background[1];
      out_img[2 * P + pix] = acc[2] + T * background[2];
      const float a = 1.f - T;
      alpha_img[pix] = a;
      depth_img[pix] = (acc[3] + T * background[0]) / fminf(fmaxf(a, 0.05f), 1.f);
    } else if (C == 4) {
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

template <int C, bool LIST, bool RANKED, bool HITS = false>
__global__ void __launch_bounds__(kFwdThreads) blend_fwd_ilp_kernel(
    int img_w, int img_h, int tbx, const int* order, int sched, const int2* __restrict__ tile_bins,
    const float4* __restrict__ rec, const int* __restrict__ ranks, const float* __restrict__ background,
    float* __restrict__ final_Ts, int* __restrict__ final_idx, float* __restrict__ out_img,
    int* __restrict__ hit_list = nullptr, int* __restrict__ hit_count = nullptr) {
  blend_fwd_body<C, LIST, RANKED, HITS, false>(img_w, img_h, tbx, order, sched, tile_bins, rec, ranks, background,
                                               final_Ts, final_idx, out_img, hit_list, hit_count, nullptr, nullptr,
                                               nullptr);
}

// The sorting forward.  The sort's 15 keys per thread need more than the 56 registers of four CTAs per SM: three CTAs
// (72 registers, 864 threads) hold 396 tiles at a time.  FINISH: the view's rgb [3,H,W], alpha [H,W] and depth [H,W]
// instead of the 4-channel image (background holds 3 floats).
template <int C, bool FINISH = false>
__global__ void __launch_bounds__(kFwdThreads, 3) blend_fwd_sort_kernel(
    int img_w, int img_h, int tbx, const int* order, const int2* __restrict__ tile_bins, const float4* __restrict__ rec,
    const float* __restrict__ background, float* __restrict__ final_Ts, int* __restrict__ final_idx,
    float* __restrict__ out_img, int* __restrict__ hit_list, int* __restrict__ hit_count,
    const unsigned* __restrict__ depth_keys, int* bucket, int* sorted, float* __restrict__ alpha_img = nullptr,
    float* __restrict__ depth_img = nullptr) {
  blend_fwd_body<C, true, true, true, true, FINISH>(img_w, img_h, tbx, order, 0, tile_bins, rec, nullptr, background,
                                                    final_Ts, final_idx, out_img, hit_list, hit_count, depth_keys,
                                                    bucket, sorted, alpha_img, depth_img);
}

// ------------------------------------------------------------------ backward
// dynamic shared memory layout (bytes): records ring | per-warp entries | per-warp (hit, pixel) matrix | per-warp v_out
constexpr int kSmRec = kBwdStages * kStageRecs * kRecBytes;                 // 18432
constexpr int kSmEntries = kPixelWarps * kEntryCap * 48;                    // 18432
constexpr int kSmM = kPixelWarps * kChunk * kMStride * 8;                   // 33792
constexpr int kSmVo = kPixelWarps * 32 * 16;                                // 4096
constexpr int kBwdSmem = kSmRec + kSmEntries + kSmM + kSmVo;                // 74752

template <int C, bool RANKED>
__global__ void __launch_bounds__(kBwdThreads, 3) blend_bwd_mom_kernel(
    int img_w, int img_h, int tbx, const int* order, int sched,
    const int* __restrict__ gids_sorted /* RANKED: unused */, const int* __restrict__ ranks /* RANKED only */,
    const int2* __restrict__ tile_bins, const float4* __restrict__ rec, const float* __restrict__ background,
    const float* __restrict__ final_Ts, const int* __restrict__ final_idx, const float* __restrict__ v_output,
    const float* __restrict__ v_output_alpha, float* __restrict__ v_xy, float* __restrict__ v_conic,
    float* __restrict__ v_colors, float* __restrict__ v_opacity) {
  extern __shared__ __align__(128) unsigned char smem[];
  float4* s_rec = reinterpret_cast<float4*>(smem);
  __shared__ __align__(8) unsigned long long s_full[kBwdStages];
  __shared__ int s_ticket[kBwdStages];  // warps that have finished culling the stage's current batch
  __shared__ int s_cta_final;
  __shared__ int s_tile;
  __shared__ int s_rk[RANKED ? kBwdStages : 1][RANKED ? kStageRecs : 1];  // RANKED: ranks of each slot's NEXT batch

  const int tr = threadIdx.x, lane = tr & 31, warp = tr >> 5;
  if (tr == 0) s_tile = draw_tile(order, sched, tbx * ((img_h + 15) >> 4));
  __syncthreads();
  if (s_tile < 0) return;
  float4* E = reinterpret_cast<float4*>(smem + kSmRec) + warp * kEntryCap * 3;           // pending entries
  float2* M = reinterpret_cast<float2*>(smem + kSmRec + kSmEntries) + warp * kChunk * kMStride;
  float4* VO = reinterpret_cast<float4*>(smem + kSmRec + kSmEntries + kSmM) + warp * 32;

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
  float bufv = 0.f;  // (colour accumulated behind the current Gaussian) . v_out
  const int bin_final = inside ? final_idx[pix] : -1;
  float vo[4] = {0.f, 0.f, 0.f, 0.f};
  float voa = 0.f;
  if (inside) {
#pragma unroll
    for (int c = 0; c < C; ++c) vo[c] = v_output[pix * C + c];
    voa = v_output_alpha ? v_output_alpha[pix] : 0.f;  // NULL = no gradient through alpha
  }
  VO[lane] = make_float4(vo[0], vo[1], vo[2], vo[3]);
  float bgdot = 0.f;
#pragma unroll
  for (int c = 0; c < C; ++c) bgdot += background[c] * vo[c];
  const float tfc = T_final * (voa - bgdot);  // the two T_final * ra terms of v_alpha share it

  int warp_bin_final = bin_final;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) warp_bin_final = max(warp_bin_final, __shfl_xor_sync(0xffffffffu, warp_bin_final, o));
  if (tr == 0) {
    s_cta_final = -1;
#pragma unroll
    for (int s = 0; s < kBwdStages; ++s) {
      mbar_init(&s_full[s], RANKED ? 32 : 1);
      s_ticket[s] = 0;
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (lane == 0) atomicMax(&s_cta_final, warp_bin_final);
  __syncthreads();
  // the walk starts at the last index any pixel of the tile needs and goes down to range.x
  const int last = min(s_cta_final, range.y - 1);
  if (last < range.x) return;  // no pixel of this tile blended anything (CTA-uniform: nothing is in flight yet)
  const int num_batches = (last - range.x + kStageRecs) / kStageRecs;
  auto issue = [&](int k) {  // one lane; batch k covers indices [hi_k - size_k + 1, hi_k], hi_k = last - k*kStageRecs
    const int s = k % kBwdStages;
    const int hi = last - k * kStageRecs;
    const int lo = max(range.x, hi - kStageRecs + 1);
    const unsigned bytes = (unsigned)(hi - lo + 1) * kRecBytes;
    mbar_expect_tx(&s_full[s], bytes);
    bulk_g2s(s_rec + s * kStageRecs * 3, rec + (size_t)lo * 3, bytes, &s_full[s]);
  };
  // One whole warp.  The ranks of batch k were copied into s_rk[slot] by the issue of batch k - kBwdStages (same slot;
  // its arrival on the stage's barrier covers that copy, and this warp has since waited on that phase), so the warp
  // that recycles a stage pays one L2 round trip (the gathers), not two.
  auto issue_ranked = [&](int k) {
    const int s = k % kBwdStages;
    const int hi = last - k * kStageRecs;
    const int lo = max(range.x, hi - kStageRecs + 1);
    const int count = hi - lo + 1;
    int r[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int j = lane + 32 * i;
      r[i] = (j < count) ? (k >= kBwdStages ? s_rk[s][j] : ranks[lo + j]) : -1;
    }
    float4* stage = s_rec + s * kStageRecs * 3;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (r[i] >= 0) {
        const float4* src = rec + 3 * (size_t)r[i];
        float4* dst = stage + 3 * (lane + 32 * i);
        cp_async16(dst, src);
        cp_async16(dst + 1, src + 1);
        cp_async16(dst + 2, src + 2);
      }
    const int k2 = k + kBwdStages;
    if (k2 < num_batches) {
      const int hi2 = last - k2 * kStageRecs;
      const int lo2 = max(range.x, hi2 - kStageRecs + 1);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = lane + 32 * i;
        if (j < hi2 - lo2 + 1) cp_async4(&s_rk[s][j], ranks + lo2 + j);
      }
    }
    cp_async_arrive(&s_full[s]);
  };
  if (RANKED) {
    if (warp == 0)
      for (int k = 0; k < min(kBwdStages, num_batches); ++k) issue_ranked(k);
  } else if (tr == 0) {
    for (int k = 0; k < min(kBwdStages, num_batches); ++k) issue(k);
  }
  // no CTA-wide barrier below this line

  // ---- one chunk of n <= 16 pending entries starting at entry `base`: phase A (lanes = pixels), phase B (lanes = hits)
  // (entries [base, base + n) with n rounded up to a multiple of 4 by invalid padding entries, see pad4 below)
  auto chunk = [&](int base, int n) {
#pragma unroll 1
    for (int h0 = 0; h0 < n; h0 += 4) {
      float al[4], ov[4], ra[4];
      float4 col[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int h = h0 + u;
        const float4 a0 = E[(base + h) * 3], a1 = E[(base + h) * 3 + 1];  // x y A B | C o idx -
        col[u] = E[(base + h) * 3 + 2];
        const float dx = a0.x - px, dy = a0.y - py;
        const float sigma = 0.5f * (a0.z * dx * dx + a1.x * dy * dy) + a0.w * dx * dy;
        const float vis = exp_neg(sigma);
        const float alpha = fminf(kAlphaMaxBwd, a1.y * vis);
        // pixels outside the image have bin_final = -1, padding entries have idx = INT_MAX
        const bool valid = (__float_as_int(a1.z) <= bin_final) && !(sigma < 0.f) && !(alpha < kAlphaMin);
        al[u] = valid ? alpha : 0.f;
        ov[u] = valid ? a1.y * vis : 0.f;
        ra[u] = rcp_approx(1.f - al[u]);  // exactly 1 for the pairs that do not take part
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        // v_alpha = sum_c (c_c T' - buffer_c ra) v_out_c + T_final ra (v_out_alpha - bg.v_out) with T' = T ra:
        // the common factor ra is applied once
        // sum_c (c_c T - buffer_c) v_out_c = T (c . v_out) - (buffer . v_out): only the SCALAR buffer . v_out is carried
        // (buffer_c += c_c fac  =>  buffer . v_out += fac (c . v_out)); c . v_out is off the serial chain
        const float cc[4] = {col[u].x, col[u].y, col[u].z, col[u].w};
        float cv = 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) cv += cc[c] * vo[c];
        const float v_alpha = ((cv * T - bufv) + tfc) * ra[u];
        T *= ra[u];
        const float fac = al[u] * T;
        bufv += cv * fac;
        M[(h0 + u) * kMStride + lane] = make_float2(fac, -ov[u] * v_alpha);  // (fac, v_sigma); zeros when not valid
      }
    }
    if (RANKED) cp_async_wait_all();  // this lane's rank copies into the entries have landed (then the warp barrier)
    __syncwarp();
    {
      const int hh = lane & 15, half = lane >> 4;
      const int he = min(hh, n - 1);
      const float4 a0 = E[(base + he) * 3], a1 = E[(base + he) * 3 + 1];
      // the Gaussian id is only needed by the REDs at the end: start its load now (padding entries: index 0 / id 0)
      const int e_idx = __float_as_int(a1.z);
      const int e_safe = e_idx == 0x7fffffff ? range.x : e_idx;
      const int g_id = RANKED ? __float_as_int(a1.w) : gids_sorted[e_safe];
      const float2* Mrow = M + hh * kMStride + half * 16;
      const float4* V = VO + half * 16;
      float g[4] = {0.f, 0.f, 0.f, 0.f};
      float r00 = 0.f, r01 = 0.f, r10 = 0.f, r11 = 0.f, sii = 0.f;
      float facmax = 0.f;  // fac = alpha * T > 0 exactly for the (hit, pixel) pairs that took a gradient
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const float2 m = Mrow[q];
        const float4 v = V[q];
        const float fi = (float)(q & 7);
        facmax = fmaxf(facmax, m.x);
        g[0] += m.x * v.x;
        g[1] += m.x * v.y;
        g[2] += m.x * v.z;
        if (C == 4) g[3] += m.x * v.w;
        if (q < 8) {
          r00 += m.y;
          r10 += m.y * fi;
        } else {
          r01 += m.y;
          r11 += m.y * fi;
        }
        sii += m.y * (fi * fi);
      }
      // pixel (i, j) of this half: dx = u - i, dy = v - j with j in {0, 1}
      const float u_ = a0.x - fx0, v_ = a0.y - (fy0 + (float)(2 * half));
      const float S0 = r00 + r01, Sj = r01, Si = r10 + r11, Sij = r11;
      const float sx = u_ * S0 - Si, sy = v_ * S0 - Sj;                      // sum v_sigma * dx, * dy
      const float sxx = u_ * (u_ * S0 - 2.f * Si) + sii;                     // sum v_sigma * dx^2
      const float sxy = u_ * (v_ * S0 - Sj) - v_ * Si + Sij;                 // sum v_sigma * dx * dy
      const float syy = v_ * (v_ * S0 - 2.f * Sj) + Sj;                      // sum v_sigma * dy^2  (j^2 == j)
      float o[10];
      o[0] = g[0]; o[1] = g[1]; o[2] = g[2]; o[3] = g[3];
      o[4] = 0.5f * sxx; o[5] = sxy; o[6] = 0.5f * syy;
      o[7] = a0.z * sx + a0.w * sy;   // v_xy.x = A sx + B sy
      o[8] = a0.w * sx + a1.x * sy;   // v_xy.y = B sx + C sy
      o[9] = S0;
#pragma unroll
      for (int i = 0; i < 10; ++i) o[i] += __shfl_xor_sync(0xffffffffu, o[i], 16);
      facmax = fmaxf(facmax, __shfl_xor_sync(0xffffffffu, facmax, 16));
      if (half == 0 && hh < n && facmax > 0.f) {  // false hits (no valid pixel) add nothing
        if (C == 4) {
          gb::red_add_v4(v_colors + 4 * (size_t)g_id, o[0], o[1], o[2], o[3]);
        } else {
          gb::red_add(v_colors + 3 * (size_t)g_id + 0, o[0]);
          gb::red_add(v_colors + 3 * (size_t)g_id + 1, o[1]);
          gb::red_add(v_colors + 3 * (size_t)g_id + 2, o[2]);
        }
        gb::red_add(v_conic + 3 * (size_t)g_id + 0, o[4]);
        gb::red_add(v_conic + 3 * (size_t)g_id + 1, o[5]);
        gb::red_add(v_conic + 3 * (size_t)g_id + 2, o[6]);
        gb::red_add_v2(v_xy + 2 * (size_t)g_id, o[7], o[8]);
        // v_opacity = sum vis * v_alpha = -sum v_sigma / o   (o >= 1/255 wherever a pair was valid)
        gb::red_add(v_opacity + g_id, -o[9] * rcp_approx(a1.y));
      }
    }
    __syncwarp();  // phase B's reads of M / E are complete before the next chunk or the compaction overwrites them
  };

  // pad the entry list [0, cnt) to a multiple of 4 with entries no pixel accepts (idx = INT_MAX)
  auto pad4 = [&](int cnt_) {
    const int padded = (cnt_ + 3) & ~3;
    if (lane < padded - cnt_) {
      E[(cnt_ + lane) * 3 + 0] = make_float4(0.f, 0.f, 1.f, 0.f);
      E[(cnt_ + lane) * 3 + 1] = make_float4(1.f, 0.f, __int_as_float(0x7fffffff), 0.f);
      E[(cnt_ + lane) * 3 + 2] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncwarp();
    return padded;
  };
  int cnt = 0;  // pending entries of this warp (warp-uniform)
  for (int k = 0; k < num_batches; ++k) {
    const int s = k % kBwdStages;
    const int hi = last - k * kStageRecs;
    const int lo = max(range.x, hi - kStageRecs + 1);
    const int batch_size = hi - lo + 1;
    while (!mbar_try(&s_full[s], (unsigned)((k / kBwdStages) & 1))) __nanosleep(64);  // warps far ahead park cheaply
    const float4* sr = s_rec + s * kStageRecs * 3;
    // slot j of the stage holds sorted index lo + j; walk j downwards, 32 at a time
    const int j_top = min(batch_size - 1, warp_bin_final - lo);  // nothing above this index matters to the warp
    for (int c1 = (j_top & ~31); c1 >= 0 && j_top >= 0; c1 -= 32) {
      const int tj = c1 + lane;
      bool hit = false;
      if (tj <= j_top) hit = footprint_hit(sr[tj * 3], &sr[tj * 3 + 1], fx0, fx1, fy0, fy1);
      const unsigned mask = __ballot_sync(0xffffffffu, hit);
      if (mask == 0) continue;
      if (hit) {  // back to front: the hit with the highest index goes first
        const int pos = cnt + __popc(mask & ~((2u << lane) - 1u));
        const float4 q0 = sr[tj * 3], q1 = sr[tj * 3 + 1], q2 = sr[tj * 3 + 2];
        E[pos * 3 + 0] = make_float4(q0.x, q0.y, q1.x, q1.y);
        if constexpr (RANKED) {
          // the entry's 4th word gets the hit's Gaussian id (the list entry), copied asynchronously (chunk() waits for
          // it before phase B), so phase B needs no dependent load to find it
          float* e1 = reinterpret_cast<float*>(&E[pos * 3 + 1]);
          *reinterpret_cast<float2*>(e1) = make_float2(q1.z, q1.w);
          e1[2] = __int_as_float(lo + tj);
          cp_async4(e1 + 3, ranks + lo + tj);
        } else {
          E[pos * 3 + 1] = make_float4(q1.z, q1.w, __int_as_float(lo + tj), 0.f);
        }
        E[pos * 3 + 2] = q2;
      }
      cnt += __popc(mask);
      __syncwarp();
      if (cnt >= kChunk) {
        int base = 0;
        while (cnt - base >= kChunk) {
          chunk(base, kChunk);
          base += kChunk;
        }
        const int left = cnt - base;  // < 16, source entries [base, cnt) with base >= 16: disjoint from [0, left)
        if (lane < left) {
          const float4 e0 = E[(base + lane) * 3], e1 = E[(base + lane) * 3 + 1], e2 = E[(base + lane) * 3 + 2];
          E[lane * 3 + 0] = e0;
          E[lane * 3 + 1] = e1;
          E[lane * 3 + 2] = e2;
        }
        cnt = left;
        __syncwarp();
      }
    }
    // this warp is finished with the stage: the last of the 8 through recycles it
    __syncwarp();
    int refill = 0;
    if (lane == 0) {
      __threadfence_block();  // release this warp's reads of the stage
      const int ticket = atomicAdd(&s_ticket[s], 1);
      if (ticket == kPixelWarps - 1) {
        __threadfence_block();
        s_ticket[s] = 0;
        if (k + kBwdStages < num_batches) {
          if (RANKED) refill = 1;
          else issue(k + kBwdStages);
        }
      }
    }
    if (RANKED) {
      refill = __shfl_sync(0xffffffffu, refill, 0);
      if (refill) issue_ranked(k + kBwdStages);
    }
  }
  if (cnt > 0) chunk(0, pad4(cnt));
  if (RANKED) cp_async_wait_all();
}

// ------------------------------------------------------------------ backward from the forward's hit lists
// The ranked backward above has every pixel warp of a tile cull every record of the tile again, through a stage ring
// that the slowest warp paces.  Here each (tile, pixel warp) is an independent work item: the warp walks the hit list
// the forward stored for it (blend_fwd_ilp_kernel<.., HITS>) back to front, 16 entries per chunk, and gathers the
// next chunk's records with cp.async straight from the by-id table into a double-buffered entry buffer while it runs
// phase B of the current one (the list and id loads behind them are issued a chunk earlier).  Phases A / B and the REDs are those of blend_bwd_mom_kernel (entries in
// record layout x y ex ey | A B C o | colour, index and id beside them), and the chunks hold the same hits in the same
// order, so per warp the gradients are the same numbers; only the order of the atomic adds across warps changes.
// Warps share nothing, so they draw items one at a time from a counter.  The kernel time is set by the warps with the
// most hits, and those are not the warps of the longest tiles, so order_items_kernel first puts the items with hits in
// descending order of their chunk count: the heaviest items start in the first wave, the light ones fill in behind.
//
// hit_count [16 T + 2]: per-item counts [8 T] (the forward) | draw counter (zeroed by the forward, reset by each
// backward) | number of items with hits | those items, heaviest first [8 T] (order_items_kernel).
constexpr int kListWarps = 4;
constexpr int kListThreads = kListWarps * 32;
constexpr int kOrderBuckets = 64;  // items are ordered by min(chunks, 63): bucket b holds items of 63 - b chunks

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }

// one CTA: a counting sort of the n_items counts into descending chunk-count buckets (order inside a bucket is free)
__global__ void __launch_bounds__(1024) order_items_kernel(int n_items, int* __restrict__ hit_count) {
  __shared__ int s_off[kOrderBuckets];
  const int tr = threadIdx.x, lane = tr & 31;
  auto bucket = [](int n) { return kOrderBuckets - 1 - min((n + kChunk - 1) / kChunk, kOrderBuckets - 1); };
  if (tr < kOrderBuckets) s_off[tr] = 0;
  __syncthreads();
  for (int i = tr; i < n_items; i += blockDim.x) {
    const int n = hit_count[i];
    if (n > 0) atomicAdd(&s_off[bucket(n)], 1);
  }
  __syncthreads();
  if (tr < 32) {  // exclusive scan of the 64 bucket sizes, two per lane
    const int a = s_off[2 * lane], b = s_off[2 * lane + 1];
    int incl = a + b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    const int excl = incl - a - b;
    s_off[2 * lane] = excl;
    s_off[2 * lane + 1] = excl + a;
    if (lane == 31) hit_count[n_items + 1] = incl;
  }
  __syncthreads();
  int* items = hit_count + n_items + 2;
  for (int i = tr; i < n_items; i += blockDim.x) {
    const int n = hit_count[i];
    if (n > 0) items[atomicAdd(&s_off[bucket(n)], 1)] = i;
  }
}

// FINISH: v_output is the gradient of the finished view's rgb [3,H,W] (may be NULL), g_depth [H,W] (may be NULL) that of
// its depth, and each pixel's 4-vector is formed in registers with render_finish.cu's finish_bwd_kernel arithmetic
// (alpha_img: the forward's alpha).  background holds 3 floats, the depth channel's is background[0].
template <int C, bool FINISH = false>
__global__ void __launch_bounds__(kListThreads, 6) blend_bwd_lists_kernel(
    int img_w, int img_h, int tbx, int n_items, const int2* __restrict__ tile_bins, const int* __restrict__ hit_list,
    const int* __restrict__ hit_count, int* draw /* hit_count + n_items */,
    const int* __restrict__ ranks, const float4* __restrict__ rec, const float* __restrict__ background,
    const float* __restrict__ final_Ts, const int* __restrict__ final_idx, const float* __restrict__ v_output,
    const float* __restrict__ v_output_alpha, float* __restrict__ v_xy, float* __restrict__ v_conic,
    float* __restrict__ v_colors, float* __restrict__ v_opacity, const float* __restrict__ g_depth = nullptr,
    const float* __restrict__ alpha_img = nullptr) {
  static_assert(!FINISH || C == 4, "the finished view is rgb + depth");
  __shared__ __align__(16) float4 s_e[kListWarps][2][kChunk * 3];  // entries: the gathered records
  __shared__ __align__(8) int2 s_ig[kListWarps][2][kChunk];        // (sorted index, Gaussian id) of each entry
  __shared__ float2 s_m[kListWarps][kChunk * kMStride];            // (fac, v_sigma) of each (hit, pixel)
  __shared__ float4 s_vo[kListWarps][32];

  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float2* M = s_m[wib];
  float4* VO = s_vo[wib];
  const int n_work = hit_count[n_items + 1];
  const int* items = hit_count + n_items + 2;
  const int n_draws = n_work + (int)gridDim.x * kListWarps;  // every warp's last draw finds the items exhausted
  for (;;) {
    int k = 0;
    if (lane == 0) {
      k = atomicAdd(draw, 1);
      if (k == n_draws - 1) *draw = 0;  // the launch's last draw: the counter is ready for the next launch
    }
    k = __shfl_sync(0xffffffffu, k, 0);
    if (k >= n_work) break;
    const int item = items[k], tile = item >> 3, warp = item & 7;
    const int n = hit_count[item];
    const int2 range = tile_bins[tile];
    const int* list = hit_list + 8 * (size_t)range.x + (size_t)warp * (range.y - range.x);
    const Tile tl = make_tile(tile, tbx);
    const int wx0 = tl.tx * 16 + ((warp & 1) << 3), wy0 = tl.ty * 16 + ((warp >> 1) << 2);
    const int pxi = wx0 + (lane & 7), pyi = wy0 + (lane >> 3);
    const bool inside = (pxi < img_w) && (pyi < img_h);
    const float px = (float)pxi + 0.5f, py = (float)pyi + 0.5f;
    const float fx0 = (float)wx0 + 0.5f, fy0 = (float)wy0 + 0.5f;
    const size_t pix = inside ? ((size_t)pyi * img_w + pxi) : 0;

    // chunk j holds list positions [top - cnt, top), top = n - 16 j, entry l = position top - 1 - l (back to front)
    const int nchunks = (n + kChunk - 1) / kChunk;
    int g_idx = 0, g_id = 0;  // this lane's entry of the next chunk to gather (lanes < 16)
    auto load_next = [&](int j) {
      const int top = n - kChunk * j;
      if (lane < min(kChunk, top)) {
        g_idx = list[top - 1 - lane];
        g_id = ranks[g_idx];
      }
    };
    // issue chunk j's gathers into buffer j & 1; pad its entry count up to a multiple of 4 with entries no pixel accepts
    auto gather = [&](int j) {
      const int cnt = min(kChunk, n - kChunk * j);
      float4* E = s_e[wib][j & 1];
      if (lane < cnt) {
        const float4* src = rec + 3 * (size_t)g_id;
        cp_async16(&E[lane * 3 + 0], src);
        cp_async16(&E[lane * 3 + 1], src + 1);
        cp_async16(&E[lane * 3 + 2], src + 2);
        s_ig[wib][j & 1][lane] = make_int2(g_idx, g_id);
      } else if (lane < ((cnt + 3) & ~3)) {
        E[lane * 3 + 0] = make_float4(0.f, 0.f, 0.f, 0.f);
        E[lane * 3 + 1] = make_float4(1.f, 0.f, 1.f, 0.f);
        E[lane * 3 + 2] = make_float4(0.f, 0.f, 0.f, 0.f);
        s_ig[wib][j & 1][lane] = make_int2(0x7fffffff, 0);
      }
      cp_async_commit();
    };
    // the pixel loads go out first: their latency hides behind the list -> id -> gather chain of chunk 0
    const float T_final = inside ? final_Ts[pix] : 1.f;
    float T = T_final;
    float bufv = 0.f;  // (colour accumulated behind the current Gaussian) . v_out
    const int bin_final = inside ? final_idx[pix] : -1;
    float vo[4] = {0.f, 0.f, 0.f, 0.f};
    float voa = 0.f, a_pix = 1.f;
    if (inside) {
      if (FINISH) {
        const size_t P = (size_t)img_w * img_h;
        if (v_output) {
          vo[0] = v_output[pix];
          vo[1] = v_output[P + pix];
          vo[2] = v_output[2 * P + pix];
        }
        if (g_depth) vo[3] = g_depth[pix];
        a_pix = alpha_img[pix];
      } else {
#pragma unroll
        for (int c = 0; c < C; ++c) vo[c] = v_output[pix * C + c];
      }
      voa = v_output_alpha ? v_output_alpha[pix] : 0.f;  // NULL = no gradient through alpha
    }
    load_next(0);
    gather(0);
    if (FINISH) vo[3] = vo[3] / fminf(fmaxf(a_pix, 0.05f), 1.f);  // 0 without g_depth
    VO[lane] = make_float4(vo[0], vo[1], vo[2], vo[3]);
    float bgdot = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) bgdot += background[FINISH && c == 3 ? 0 : c] * vo[c];
    const float tfc = T_final * (voa - bgdot);  // the two T_final * ra terms of v_alpha share it
    if (nchunks > 1) load_next(1);

    for (int j = 0; j < nchunks; ++j) {
      const int cnt = min(kChunk, n - kChunk * j);
      const int nn = j + 1 < nchunks ? kChunk : ((cnt + 3) & ~3);  // only the last chunk is short
      const float4* E = s_e[wib][j & 1];
      const int2* IG = s_ig[wib][j & 1];
      cp_async_wait_all();  // chunk j has landed (chunk j + 1 is issued below)
      __syncwarp();
      // ---- phase A, lanes = pixels: the serial transmittance / colour-buffer recurrence over the chunk's hits
#pragma unroll 1
      for (int h0 = 0; h0 < nn; h0 += 4) {
        float al[4], ov[4], ra[4];
        float4 col[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int h = h0 + u;
          const float4 q0 = E[h * 3], q1 = E[h * 3 + 1];  // x y - - | A B C o
          col[u] = E[h * 3 + 2];
          const float dx = q0.x - px, dy = q0.y - py;
          const float sigma = 0.5f * (q1.x * dx * dx + q1.z * dy * dy) + q1.y * dx * dy;
          const float vis = exp_neg(sigma);
          const float alpha = fminf(kAlphaMaxBwd, q1.w * vis);
          // pixels outside the image have bin_final = -1, padding entries have idx = INT_MAX
          const bool valid = (IG[h].x <= bin_final) && !(sigma < 0.f) && !(alpha < kAlphaMin);
          al[u] = valid ? alpha : 0.f;
          ov[u] = valid ? q1.w * vis : 0.f;
          ra[u] = rcp_approx(1.f - al[u]);  // exactly 1 for the pairs that do not take part
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float cc[4] = {col[u].x, col[u].y, col[u].z, col[u].w};
          float cv = 0.f;
#pragma unroll
          for (int c = 0; c < C; ++c) cv += cc[c] * vo[c];
          const float v_alpha = ((cv * T - bufv) + tfc) * ra[u];
          T *= ra[u];
          const float fac = al[u] * T;
          bufv += cv * fac;
          M[(h0 + u) * kMStride + lane] = make_float2(fac, -ov[u] * v_alpha);  // (fac, v_sigma); zeros when not valid
        }
      }
      if (j + 1 < nchunks) {  // the next chunk's gathers run under phase B and the next phase A's start
        gather(j + 1);
        if (j + 2 < nchunks) load_next(j + 2);
      }
      __syncwarp();
      // ---- phase B, lanes = (hit, half of the 8x4 footprint): colour sums and image moments of v_sigma, then RED
      {
        const int hh = lane & 15, half = lane >> 4;
        const int he = min(hh, nn - 1);
        const float4 q0 = E[he * 3], q1 = E[he * 3 + 1];
        const int e_id = IG[he].y;
        const float2* Mrow = M + hh * kMStride + half * 16;
        const float4* V = VO + half * 16;
        float g[4] = {0.f, 0.f, 0.f, 0.f};
        float r00 = 0.f, r01 = 0.f, r10 = 0.f, r11 = 0.f, sii = 0.f;
        float facmax = 0.f;  // fac = alpha * T > 0 exactly for the (hit, pixel) pairs that took a gradient
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          const float2 m = Mrow[q];
          const float4 v = V[q];
          const float fi = (float)(q & 7);
          facmax = fmaxf(facmax, m.x);
          g[0] += m.x * v.x;
          g[1] += m.x * v.y;
          g[2] += m.x * v.z;
          if (C == 4) g[3] += m.x * v.w;
          if (q < 8) {
            r00 += m.y;
            r10 += m.y * fi;
          } else {
            r01 += m.y;
            r11 += m.y * fi;
          }
          sii += m.y * (fi * fi);
        }
        // pixel (i, j) of this half: dx = u - i, dy = v - j with j in {0, 1}
        const float u_ = q0.x - fx0, v_ = q0.y - (fy0 + (float)(2 * half));
        const float S0 = r00 + r01, Sj = r01, Si = r10 + r11, Sij = r11;
        const float sx = u_ * S0 - Si, sy = v_ * S0 - Sj;       // sum v_sigma * dx, * dy
        const float sxx = u_ * (u_ * S0 - 2.f * Si) + sii;      // sum v_sigma * dx^2
        const float sxy = u_ * (v_ * S0 - Sj) - v_ * Si + Sij;  // sum v_sigma * dx * dy
        const float syy = v_ * (v_ * S0 - 2.f * Sj) + Sj;       // sum v_sigma * dy^2  (j^2 == j)
        float o[10];
        o[0] = g[0]; o[1] = g[1]; o[2] = g[2]; o[3] = g[3];
        o[4] = 0.5f * sxx; o[5] = sxy; o[6] = 0.5f * syy;
        o[7] = q1.x * sx + q1.y * sy;  // v_xy.x = A sx + B sy
        o[8] = q1.y * sx + q1.z * sy;  // v_xy.y = B sx + C sy
        o[9] = S0;
#pragma unroll
        for (int i = 0; i < 10; ++i) o[i] += __shfl_xor_sync(0xffffffffu, o[i], 16);
        facmax = fmaxf(facmax, __shfl_xor_sync(0xffffffffu, facmax, 16));
        if (half == 0 && hh < nn && facmax > 0.f) {  // false hits (no valid pixel) add nothing
          if (C == 4) {
            gb::red_add_v4(v_colors + 4 * (size_t)e_id, o[0], o[1], o[2], o[3]);
          } else {
            gb::red_add(v_colors + 3 * (size_t)e_id + 0, o[0]);
            gb::red_add(v_colors + 3 * (size_t)e_id + 1, o[1]);
            gb::red_add(v_colors + 3 * (size_t)e_id + 2, o[2]);
          }
          gb::red_add(v_conic + 3 * (size_t)e_id + 0, o[4]);
          gb::red_add(v_conic + 3 * (size_t)e_id + 1, o[5]);
          gb::red_add(v_conic + 3 * (size_t)e_id + 2, o[6]);
          gb::red_add_v2(v_xy + 2 * (size_t)e_id, o[7], o[8]);
          // v_opacity = sum vis * v_alpha = -sum v_sigma / o   (o >= 1/255 wherever a pair was valid)
          gb::red_add(v_opacity + e_id, -o[9] * rcp_approx(q1.w));
        }
      }
      __syncwarp();  // phase B's reads of M / VO / this buffer are complete before they are overwritten
    }
  }
}

// ================================================================== four lighting conditions per pass (OLAT)
// BASELINE config 3 (SURVEY.md section 8d): the 32 one-light-at-a-time conditions of a view share geometry, projection, tile
// lists AND every pixel's alphas / transmittances — only the colours differ.  These kernels blend FOUR colour sets in one
// walk: the quadratic form, ex2, the transmittance recurrence (forward) and the whole (fac, v_sigma) machinery, the cull
// and the hit compaction (backward) are paid once per hit instead of four times; per condition only 3 FMAs (forward) or
// the colour-buffer FMAs and the v_colour sums (backward) are added.  Records are "wide": 32 B of geometry + 4 x rgb =
// 80 B (5 x float4), colour part rewritten per group of conditions by gb_records_set_colors4.
constexpr int kMK = 4;                 // conditions per pass
constexpr int kMC = 3 * kMK;           // colour channels per pass
constexpr int kMRQ = 5;                // float4 per wide record
constexpr int kMRecBytes = kMRQ * 16;  // 80

__global__ void __launch_bounds__(kFwdThreads) blend_fwd_multi_kernel(
    int img_w, int img_h, int tbx, const int* order, int sched, const int2* __restrict__ tile_bins,
    const float4* __restrict__ rec, const float* __restrict__ background, float* __restrict__ out_planes /* [4][H][W][3] */) {
  __shared__ __align__(128) float4 s_rec[kFwdStages][kStageRecs * kMRQ];  // 40 KB
  __shared__ __align__(8) unsigned long long s_full[kFwdStages];
  __shared__ __align__(8) unsigned long long s_empty[kFwdStages];
  __shared__ int s_ndone;
  __shared__ __align__(16) int s_hits[kPixelWarps][kStageRecs + 4];
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
  __syncthreads();
  if (s_tile < 0) return;
  const Tile tl = make_tile(s_tile, tbx);
  const int2 range = tile_bins[tl.tile_id];
  const int num_batches = (range.y - range.x + kStageRecs - 1) / kStageRecs;

  if (warp == kPixelWarps) {  // producer warp (one lane)
    if (lane != 0) return;
    volatile int* ndone = &s_ndone;
    int issued = 0;
    for (int b = 0; b < num_batches; ++b) {
      const int s = b % kFwdStages;
      if (b >= kFwdStages) {
        const unsigned par = (unsigned)(((b / kFwdStages) - 1) & 1);
        while (!mbar_try(&s_empty[s], par) && *ndone < kPixelWarps) {
        }
        if (*ndone >= kPixelWarps) break;
      }
      const int start = range.x + b * kStageRecs;
      const unsigned bytes = (unsigned)min(kStageRecs, range.y - start) * kMRecBytes;
      mbar_expect_tx(&s_full[s], bytes);
      bulk_g2s(&s_rec[s][0], rec + (size_t)start * kMRQ, bytes, &s_full[s]);
      issued = b + 1;
    }
    for (int b = max(0, issued - kFwdStages); b < issued; ++b)
      mbar_wait(&s_full[b % kFwdStages], (unsigned)((b / kFwdStages) & 1));
    return;
  }

  const int wx0 = tl.tx * 16 + ((warp & 1) << 3), wy0 = tl.ty * 16 + ((warp >> 1) << 2);
  const int pxi = wx0 + (lane & 7), pyi = wy0 + (lane >> 3);
  const bool inside = (pxi < img_w) && (pyi < img_h);
  const float px = (float)pxi + 0.5f, py = (float)pyi + 0.5f;
  const float fx0 = (float)wx0 + 0.5f, fx1 = (float)wx0 + 7.5f, fy0 = (float)wy0 + 0.5f, fy1 = (float)wy0 + 3.5f;

  bool done = !inside;
  float T = 1.f;
  float acc[kMC];
#pragma unroll
  for (int c = 0; c < kMC; ++c) acc[c] = 0.f;

  bool counted = false;
  for (int b = 0; b < num_batches; ++b) {
    const bool all_done = __all_sync(0xffffffffu, done);
    if (all_done && !counted) {
      counted = true;
      if (lane == 0) atomicAdd(&s_ndone, 1);
    }
    const int s = b % kFwdStages;
    const unsigned par = (unsigned)((b / kFwdStages) & 1);
    int st = 0;
    if (lane == 0) {
      volatile int* ndone = &s_ndone;
      for (;;) {
        if (mbar_try(&s_full[s], par)) { st = 1; break; }
        if (all_done && *ndone >= kPixelWarps) { st = 2; break; }
        // (many of this kernel's executed instructions are these single-lane probes, mostly saturated warps waiting
        // at the producer's frontier.  They are not parked with __nanosleep: the probes use issue slots nobody else
        // wants, while the wake-up latency of a parked warp lands on the critical path.)
      }
    }
    st = __shfl_sync(0xffffffffu, st, 0);
    if (st == 2) break;
    if (all_done) {
      if (lane == 0) mbar_arrive(&s_empty[s]);
      continue;
    }
    mbar_wait(&s_full[s], par);
    const float4* sr = s_rec[s];
    const int batch_start = range.x + b * kStageRecs;
    const int batch_size = min(kStageRecs, range.y - batch_start);
    {  // cull the whole stage into the warp's hit list, then blend the list two entries per round (see the single pass)
      int* hl = s_hits[warp];
      const unsigned lt = (1u << lane) - 1u;
      int cnt = 0;
#pragma unroll 4
      for (int c0 = 0; c0 < batch_size; c0 += 32) {
        const int ti = c0 + lane;
        bool hit = false;
        if (ti < batch_size) hit = footprint_hit(sr[ti * kMRQ], &sr[ti * kMRQ + 1], fx0, fx1, fy0, fy1);
        const unsigned mask = __ballot_sync(0xffffffffu, hit);
        if (hit) hl[cnt + __popc(mask & lt)] = ti;
        cnt += __popc(mask);
      }
      __syncwarp();
      for (int i0 = 0; i0 < cnt; i0 += 16) {
        const int i1 = min(i0 + 16, cnt);
        for (int i = i0; i < i1; i += 2) {
          const int2 e = *reinterpret_cast<const int2*>(hl + i);
          bool live[2];
          int t[2];
          live[0] = true; live[1] = i + 1 < cnt;
          t[0] = e.x; t[1] = live[1] ? e.y : e.x;
          float alpha[2], sig[2];
          float4 col[2][3];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const float4 q0 = sr[t[u] * kMRQ], q1 = sr[t[u] * kMRQ + 1];
            col[u][0] = sr[t[u] * kMRQ + 2]; col[u][1] = sr[t[u] * kMRQ + 3]; col[u][2] = sr[t[u] * kMRQ + 4];
            const float dx = q0.x - px, dy = q0.y - py;
            sig[u] = 0.5f * (q1.x * dx * dx + q1.z * dy * dy) + q1.y * dx * dy;
            alpha[u] = fminf(kAlphaMaxFwd, q1.w * exp_neg(sig[u]));
          }
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const bool ok = live[u] && !done && !(sig[u] < 0.f) && !(alpha[u] < kAlphaMin);
            const float next_T = T * (1.f - alpha[u]);
            const bool stop = ok && (next_T <= kTEps);
            const bool take = ok && !stop;
            done = done || stop;
            if (take) {
              const float vis = alpha[u] * T;
              const float cc[kMC] = {col[u][0].x, col[u][0].y, col[u][0].z, col[u][0].w, col[u][1].x, col[u][1].y,
                                     col[u][1].z, col[u][1].w, col[u][2].x, col[u][2].y, col[u][2].z, col[u][2].w};
#pragma unroll
              for (int c = 0; c < kMC; ++c) acc[c] += cc[c] * vis;
              T = next_T;
            }
          }
        }
        if (__all_sync(0xffffffffu, done)) break;
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&s_empty[s]);
  }
  if (inside) {
    const size_t pix = (size_t)pyi * img_w + pxi, plane = (size_t)img_h * img_w * 3;
#pragma unroll
    for (int k = 0; k < kMK; ++k) {
      float* o = out_planes + k * plane + pix * 3;
      o[0] = acc[3 * k + 0] + T * background[0];
      o[1] = acc[3 * k + 1] + T * background[1];
      o[2] = acc[3 * k + 2] + T * background[2];
    }
  }
}

constexpr int kMSmRec = kBwdStages * kStageRecs * kMRecBytes;      // 30720
constexpr int kMSmEntries = kPixelWarps * kEntryCap * kMRecBytes;  // 30720  (entry: x y A B | C o idx - | 12 colours)
constexpr int kMSmM = kPixelWarps * kChunk * kMStride * 8;         // 33792
constexpr int kMSmVo = kPixelWarps * 32 * 48;                      // 12288
constexpr int kMBwdSmem = kMSmRec + kMSmEntries + kMSmM + kMSmVo;  // 107520: two CTAs per SM

__global__ void __launch_bounds__(kBwdThreads, 2) blend_bwd_multi_kernel(
    int img_w, int img_h, int tbx, const int* order, int sched, const int* __restrict__ gids_sorted,
    const int2* __restrict__ tile_bins, const float4* __restrict__ rec, const float* __restrict__ background,
    const float* __restrict__ final_Ts, const int* __restrict__ final_idx,
    const float* __restrict__ v_planes /* [4][H][W][3] */, float* __restrict__ v_xy, float* __restrict__ v_conic,
    float* __restrict__ v_colors12 /* [G,12] */, float* __restrict__ v_opacity) {
  extern __shared__ __align__(128) unsigned char smem[];
  float4* s_rec = reinterpret_cast<float4*>(smem);
  __shared__ __align__(8) unsigned long long s_full[kBwdStages];
  __shared__ int s_ticket[kBwdStages];
  __shared__ int s_cta_final;
  __shared__ int s_tile;

  const int tr = threadIdx.x, lane = tr & 31, warp = tr >> 5;
  if (tr == 0) s_tile = draw_tile(order, sched, tbx * ((img_h + 15) >> 4));
  __syncthreads();
  if (s_tile < 0) return;
  float4* E = reinterpret_cast<float4*>(smem + kMSmRec) + warp * kEntryCap * kMRQ;
  float2* M = reinterpret_cast<float2*>(smem + kMSmRec + kMSmEntries) + warp * kChunk * kMStride;
  float4* VO = reinterpret_cast<float4*>(smem + kMSmRec + kMSmEntries + kMSmM) + warp * 32 * 3;

  const Tile tl = make_tile(s_tile, tbx);
  const int2 range = tile_bins[tl.tile_id];
  if (range.y <= range.x) return;
  const int wx0 = tl.tx * 16 + ((warp & 1) << 3), wy0 = tl.ty * 16 + ((warp >> 1) << 2);
  const int pxi = wx0 + (lane & 7), pyi = wy0 + (lane >> 3);
  const bool inside = (pxi < img_w) && (pyi < img_h);
  const float px = (float)pxi + 0.5f, py = (float)pyi + 0.5f;
  const float fx0 = (float)wx0 + 0.5f, fx1 = (float)wx0 + 7.5f, fy0 = (float)wy0 + 0.5f, fy1 = (float)wy0 + 3.5f;
  const size_t pix = inside ? ((size_t)pyi * img_w + pxi) : 0, plane = (size_t)img_h * img_w * 3;

  const float T_final = inside ? final_Ts[pix] : 1.f;
  float T = T_final;
  const int bin_final = inside ? final_idx[pix] : -1;
  float vo[kMC];
  float bufv = 0.f;
  float bgdot = 0.f;
#pragma unroll
  for (int k = 0; k < kMK; ++k) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      vo[3 * k + c] = inside ? v_planes[k * plane + pix * 3 + c] : 0.f;
      bgdot += background[c] * vo[3 * k + c];
    }
  }
  VO[lane * 3 + 0] = make_float4(vo[0], vo[1], vo[2], vo[3]);
  VO[lane * 3 + 1] = make_float4(vo[4], vo[5], vo[6], vo[7]);
  VO[lane * 3 + 2] = make_float4(vo[8], vo[9], vo[10], vo[11]);
  const float tfc = -T_final * bgdot;  // no alpha gradient here: the view's alpha belongs to the pass that carries the depth

  int warp_bin_final = bin_final;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) warp_bin_final = max(warp_bin_final, __shfl_xor_sync(0xffffffffu, warp_bin_final, o));
  if (tr == 0) {
    s_cta_final = -1;
#pragma unroll
    for (int s = 0; s < kBwdStages; ++s) {
      mbar_init(&s_full[s], 1);
      s_ticket[s] = 0;
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (lane == 0) atomicMax(&s_cta_final, warp_bin_final);
  __syncthreads();
  const int last = min(s_cta_final, range.y - 1);
  if (last < range.x) return;
  const int num_batches = (last - range.x + kStageRecs) / kStageRecs;
  auto issue = [&](int k) {
    const int s = k % kBwdStages;
    const int hi = last - k * kStageRecs;
    const int lo = max(range.x, hi - kStageRecs + 1);
    const unsigned bytes = (unsigned)(hi - lo + 1) * kMRecBytes;
    mbar_expect_tx(&s_full[s], bytes);
    bulk_g2s(s_rec + s * kStageRecs * kMRQ, rec + (size_t)lo * kMRQ, bytes, &s_full[s]);
  };
  if (tr == 0)
    for (int k = 0; k < min(kBwdStages, num_batches); ++k) issue(k);

  auto chunk = [&](int base, int n) {  // n is a multiple of 2 (pad2 below)
#pragma unroll 1
    for (int h0 = 0; h0 < n; h0 += 2) {
      float al[2], ov[2], ra[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int h = h0 + u;
        const float4 a0 = E[(base + h) * kMRQ], a1 = E[(base + h) * kMRQ + 1];
        const float dx = a0.x - px, dy = a0.y - py;
        const float sigma = 0.5f * (a0.z * dx * dx + a1.x * dy * dy) + a0.w * dx * dy;
        const float vis = exp_neg(sigma);
        const float alpha = fminf(kAlphaMaxBwd, a1.y * vis);
        const bool valid = (__float_as_int(a1.z) <= bin_final) && !(sigma < 0.f) && !(alpha < kAlphaMin);
        al[u] = valid ? alpha : 0.f;
        ov[u] = valid ? a1.y * vis : 0.f;
        ra[u] = rcp_approx(1.f - al[u]);
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const float4 c0 = E[(base + h0 + u) * kMRQ + 2], c1 = E[(base + h0 + u) * kMRQ + 3], c2 = E[(base + h0 + u) * kMRQ + 4];
        const float cc[kMC] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w, c2.x, c2.y, c2.z, c2.w};
        float cv = 0.f;  // c . v_out over the 12 channels; only the scalar buffer . v_out is carried (see the single pass)
#pragma unroll
        for (int c = 0; c < kMC; ++c) cv += cc[c] * vo[c];
        const float v_alpha = ((cv * T - bufv) + tfc) * ra[u];
        T *= ra[u];
        const float fac = al[u] * T;
        bufv += cv * fac;
        M[(h0 + u) * kMStride + lane] = make_float2(fac, -ov[u] * v_alpha);
      }
    }
    __syncwarp();
    {
      const int hh = lane & 15, half = lane >> 4;
      const int he = min(hh, n - 1);
      const float4 a0 = E[(base + he) * kMRQ], a1 = E[(base + he) * kMRQ + 1];
      const int e_idx = __float_as_int(a1.z);
      const int g_id = gids_sorted[e_idx == 0x7fffffff ? 0 : e_idx];
      const float2* Mrow = M + hh * kMStride + half * 16;
      const float4* V = VO + half * 16 * 3;
      float g[kMC];
#pragma unroll
      for (int c = 0; c < kMC; ++c) g[c] = 0.f;
      float r00 = 0.f, r01 = 0.f, r10 = 0.f, r11 = 0.f, sii = 0.f, facmax = 0.f;
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const float2 m = Mrow[q];
        const float4 v0 = V[q * 3], v1 = V[q * 3 + 1], v2 = V[q * 3 + 2];
        const float fi = (float)(q & 7);
        facmax = fmaxf(facmax, m.x);
        g[0] += m.x * v0.x; g[1] += m.x * v0.y; g[2] += m.x * v0.z; g[3] += m.x * v0.w;
        g[4] += m.x * v1.x; g[5] += m.x * v1.y; g[6] += m.x * v1.z; g[7] += m.x * v1.w;
        g[8] += m.x * v2.x; g[9] += m.x * v2.y; g[10] += m.x * v2.z; g[11] += m.x * v2.w;
        if (q < 8) {
          r00 += m.y;
          r10 += m.y * fi;
        } else {
          r01 += m.y;
          r11 += m.y * fi;
        }
        sii += m.y * (fi * fi);
      }
      const float u_ = a0.x - fx0, v_ = a0.y - (fy0 + (float)(2 * half));
      const float S0 = r00 + r01, Sj = r01, Si = r10 + r11, Sij = r11;
      const float sx = u_ * S0 - Si, sy = v_ * S0 - Sj;
      const float sxx = u_ * (u_ * S0 - 2.f * Si) + sii;
      const float sxy = u_ * (v_ * S0 - Sj) - v_ * Si + Sij;
      const float syy = v_ * (v_ * S0 - 2.f * Sj) + Sj;
      float o[kMC + 6];
#pragma unroll
      for (int c = 0; c < kMC; ++c) o[c] = g[c];
      o[kMC + 0] = 0.5f * sxx; o[kMC + 1] = sxy; o[kMC + 2] = 0.5f * syy;
      o[kMC + 3] = a0.z * sx + a0.w * sy;
      o[kMC + 4] = a0.w * sx + a1.x * sy;
      o[kMC + 5] = S0;
#pragma unroll
      for (int i = 0; i < kMC + 6; ++i) o[i] += __shfl_xor_sync(0xffffffffu, o[i], 16);
      facmax = fmaxf(facmax, __shfl_xor_sync(0xffffffffu, facmax, 16));
      if (half == 0 && hh < n && facmax > 0.f) {
        float* vc = v_colors12 + (size_t)kMC * g_id;
        gb::red_add_v4(vc, o[0], o[1], o[2], o[3]);
        gb::red_add_v4(vc + 4, o[4], o[5], o[6], o[7]);
        gb::red_add_v4(vc + 8, o[8], o[9], o[10], o[11]);
        gb::red_add(v_conic + 3 * (size_t)g_id + 0, o[kMC + 0]);
        gb::red_add(v_conic + 3 * (size_t)g_id + 1, o[kMC + 1]);
        gb::red_add(v_conic + 3 * (size_t)g_id + 2, o[kMC + 2]);
        gb::red_add_v2(v_xy + 2 * (size_t)g_id, o[kMC + 3], o[kMC + 4]);
        gb::red_add(v_opacity + g_id, -o[kMC + 5] * rcp_approx(a1.y));
      }
    }
    __syncwarp();
  };

  auto pad2 = [&](int cnt_) {
    const int padded = (cnt_ + 1) & ~1;
    if (lane < padded - cnt_) {
      E[(cnt_ + lane) * kMRQ + 0] = make_float4(0.f, 0.f, 1.f, 0.f);
      E[(cnt_ + lane) * kMRQ + 1] = make_float4(1.f, 0.f, __int_as_float(0x7fffffff), 0.f);
      E[(cnt_ + lane) * kMRQ + 2] = make_float4(0.f, 0.f, 0.f, 0.f);
      E[(cnt_ + lane) * kMRQ + 3] = make_float4(0.f, 0.f, 0.f, 0.f);
      E[(cnt_ + lane) * kMRQ + 4] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncwarp();
    return padded;
  };
  int cnt = 0;
  for (int k = 0; k < num_batches; ++k) {
    const int s = k % kBwdStages;
    const int hi = last - k * kStageRecs;
    const int lo = max(range.x, hi - kStageRecs + 1);
    const int batch_size = hi - lo + 1;
    while (!mbar_try(&s_full[s], (unsigned)((k / kBwdStages) & 1))) __nanosleep(64);
    const float4* sr = s_rec + s * kStageRecs * kMRQ;
    const int j_top = min(batch_size - 1, warp_bin_final - lo);
    for (int c1 = (j_top & ~31); c1 >= 0 && j_top >= 0; c1 -= 32) {
      const int tj = c1 + lane;
      bool hit = false;
      if (tj <= j_top) hit = footprint_hit(sr[tj * kMRQ], &sr[tj * kMRQ + 1], fx0, fx1, fy0, fy1);
      const unsigned mask = __ballot_sync(0xffffffffu, hit);
      if (mask == 0) continue;
      if (hit) {
        const int pos = cnt + __popc(mask & ~((2u << lane) - 1u));
        const float4 q0 = sr[tj * kMRQ], q1 = sr[tj * kMRQ + 1];
        E[pos * kMRQ + 0] = make_float4(q0.x, q0.y, q1.x, q1.y);
        E[pos * kMRQ + 1] = make_float4(q1.z, q1.w, __int_as_float(lo + tj), 0.f);
        E[pos * kMRQ + 2] = sr[tj * kMRQ + 2];
        E[pos * kMRQ + 3] = sr[tj * kMRQ + 3];
        E[pos * kMRQ + 4] = sr[tj * kMRQ + 4];
      }
      cnt += __popc(mask);
      __syncwarp();
      if (cnt >= kChunk) {
        int base = 0;
        while (cnt - base >= kChunk) {
          chunk(base, kChunk);
          base += kChunk;
        }
        const int left = cnt - base;
        if (lane < left) {
          float4 e[kMRQ];
#pragma unroll
          for (int q = 0; q < kMRQ; ++q) e[q] = E[(base + lane) * kMRQ + q];
#pragma unroll
          for (int q = 0; q < kMRQ; ++q) E[lane * kMRQ + q] = e[q];
        }
        cnt = left;
        __syncwarp();
      }
    }
    __syncwarp();
    if (lane == 0) {
      __threadfence_block();
      const int ticket = atomicAdd(&s_ticket[s], 1);
      if (ticket == kPixelWarps - 1) {
        __threadfence_block();
        s_ticket[s] = 0;
        if (k + kBwdStages < num_batches) issue(k + kBwdStages);
      }
    }
  }
  if (cnt > 0) chunk(0, pad2(cnt));
}

// geometry part of the 48-byte records into the 80-byte wide records (once per view)
__global__ void __launch_bounds__(256) records_widen_kernel(long long cap, const int* __restrict__ n_dev,
                                                            const float4* __restrict__ rec12, float4* __restrict__ rec20) {
  const long long n = n_dev ? min((long long)*n_dev, cap) : cap;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  rec20[kMRQ * i + 0] = rec12[3 * i + 0];
  rec20[kMRQ * i + 1] = rec12[3 * i + 1];
}

// colour part of the wide records: up to four [G,3] colour tables (missing ones read as zero)
__global__ void __launch_bounds__(256) records_set_colors4_kernel(long long cap, const int* __restrict__ n_dev,
                                                                  const int* __restrict__ gids_sorted,
                                                                  const float* __restrict__ colors /* [nk][G][3] */, int nk,
                                                                  long long G, float4* __restrict__ rec20) {
  const long long n = n_dev ? min((long long)*n_dev, cap) : cap;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int g = gids_sorted[i];
  float c[kMC];
#pragma unroll
  for (int k = 0; k < kMK; ++k) {
    const float* src = colors + ((size_t)k * G + g) * 3;
    const bool on = k < nk;
    c[3 * k + 0] = on ? src[0] : 0.f; c[3 * k + 1] = on ? src[1] : 0.f; c[3 * k + 2] = on ? src[2] : 0.f;
  }
  rec20[kMRQ * i + 2] = make_float4(c[0], c[1], c[2], c[3]);
  rec20[kMRQ * i + 3] = make_float4(c[4], c[5], c[6], c[7]);
  rec20[kMRQ * i + 4] = make_float4(c[8], c[9], c[10], c[11]);
}

// [G,12] group gradients -> up to four [G,3] tables (overwritten), and the group buffer is cleared for the next pass
__global__ void __launch_bounds__(256) colors12_unpack_kernel(long long G, int nk, float4* __restrict__ v12,
                                                              float* __restrict__ v_colors /* [nk][G][3] */) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const float4 a = v12[3 * g], b = v12[3 * g + 1], c = v12[3 * g + 2];
  const float v[kMC] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w};
#pragma unroll
  for (int k = 0; k < kMK; ++k)
    if (k < nk) {
      float* dst = v_colors + ((size_t)k * G + g) * 3;
      dst[0] = v[3 * k]; dst[1] = v[3 * k + 1]; dst[2] = v[3 * k + 2];
    }
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  v12[3 * g] = z; v12[3 * g + 1] = z; v12[3 * g + 2] = z;
}

}  // namespace

namespace gbblend {

// GOLIATH_B200_BLEND_FWD = list (default) | rounds: hit list per stage vs up to four hits of one cull step per round
static bool fwd_list_variant() {
  const char* e = getenv("GOLIATH_B200_BLEND_FWD");
  return !(e && !strcmp(e, "rounds"));
}

// ranks == nullptr: `records` are the sorted 48-byte records; else `records` is the by-rank table and `ranks` the sorted ranks.
// hit_list != nullptr (ranked only): the forward also stores the hit lists for blend_bwd_lists_kernel.
static int launch_fwd_any(int img_h, int img_w, int channels, const int32_t* tile_bins, const int32_t* tile_order, int sched,
                          const float* records, const int32_t* ranks, const float* background, float* out_img,
                          float* final_Ts, int32_t* final_idx, cudaStream_t s, int32_t* hit_list = nullptr,
                          int32_t* hit_count = nullptr) {
  const int tbx = gb::cdiv(img_w, 16), tby = gb::cdiv(img_h, 16);
  if (sched && !tile_order) return (int)cudaErrorInvalidValue;
  static const bool list = fwd_list_variant();
#define GB_FWD_MOM(CC, LL, RR, ...)                                                                                     \
  GB_CUDA(gb::launch<blend_fwd_ilp_kernel<CC, LL, RR, ##__VA_ARGS__>>(tbx * tby, kFwdThreads, 0, s,                     \
      img_w, img_h, tbx, tile_order, sched, (const int2*)tile_bins, (const float4*)records, ranks, background, final_Ts, \
      final_idx, out_img, hit_list, hit_count))
  if (ranks && hit_list) {
    if (channels == 3) GB_FWD_MOM(3, true, true, true); else GB_FWD_MOM(4, true, true, true);
  } else if (ranks) {
    if (channels == 3) GB_FWD_MOM(3, true, true); else GB_FWD_MOM(4, true, true);
  } else if (channels == 3) {
    if (list) GB_FWD_MOM(3, true, false); else GB_FWD_MOM(3, false, false);
  } else {
    if (list) GB_FWD_MOM(4, true, false); else GB_FWD_MOM(4, false, false);
  }
#undef GB_FWD_MOM
  return 0;
}

// the sorting forward (SORT): gb_rasterize_ranked_fwd_sort_lists, and with alpha_img (4 channels only) the finishing
// one, gb_rasterize_ranked_fwd_sort_finish
static int launch_fwd_sort(int img_h, int img_w, int channels, const int32_t* tile_bins, const int32_t* tile_order,
                           const float* depths, int32_t* bucket, int32_t* ranks, const float* records,
                           const float* background, float* out_img, float* final_Ts, int32_t* final_idx,
                           int32_t* hit_list, int32_t* hit_count, cudaStream_t s, float* alpha_img = nullptr,
                           float* depth_img = nullptr) {
  const int tbx = gb::cdiv(img_w, 16), tby = gb::cdiv(img_h, 16);
#define GB_FWD_SORT(CC, FF)                                                                                             \
  GB_CUDA(gb::launch<blend_fwd_sort_kernel<CC, FF>>(tbx * tby, kFwdThreads, 0, s,                                       \
      img_w, img_h, tbx, tile_order, (const int2*)tile_bins, (const float4*)records, background, final_Ts, final_idx,   \
      out_img, hit_list, hit_count, (const unsigned*)depths, bucket, ranks, alpha_img, depth_img))
  if (alpha_img) GB_FWD_SORT(4, true); else if (channels == 3) GB_FWD_SORT(3, false); else GB_FWD_SORT(4, false);
#undef GB_FWD_SORT
  return 0;
}

static int launch_bwd_any(int img_h, int img_w, int channels, const int32_t* gids_sorted, const int32_t* ranks,
                          const int32_t* tile_bins, const int32_t* tile_order, int sched, const float* records,
                          const float* background, const float* final_Ts, const int32_t* final_idx, const float* v_output,
                          const float* v_output_alpha, float* v_xy, float* v_conic, float* v_colors, float* v_opacity,
                          cudaStream_t s) {
  const int tbx = gb::cdiv(img_w, 16), tby = gb::cdiv(img_h, 16);
  if (sched && !tile_order) return (int)cudaErrorInvalidValue;
#define GB_BWD_MOM(CC, RR)                                                                                              \
  GB_CUDA(gb::launch<blend_bwd_mom_kernel<CC, RR>>(tbx * tby, kBwdThreads, kBwdSmem, s,                                 \
      img_w, img_h, tbx, tile_order, sched, gids_sorted, ranks, (const int2*)tile_bins, (const float4*)records, background, \
      final_Ts, final_idx, v_output, v_output_alpha, v_xy, v_conic, v_colors, v_opacity))
  if (ranks) {
    if (channels == 3) GB_BWD_MOM(3, true); else GB_BWD_MOM(4, true);
  } else {
    if (channels == 3) GB_BWD_MOM(3, false); else GB_BWD_MOM(4, false);
  }
#undef GB_BWD_MOM
  return 0;
}

static int launch_bwd_lists(int img_h, int img_w, int channels, const int32_t* ranks, const int32_t* tile_bins,
                            const int32_t* hit_list, int32_t* hit_count, const float* records,
                            const float* background, const float* final_Ts, const int32_t* final_idx,
                            const float* v_output, const float* v_output_alpha, float* v_xy, float* v_conic,
                            float* v_colors, float* v_opacity, cudaStream_t s, bool finish = false,
                            const float* g_depth = nullptr, const float* alpha_img = nullptr) {
  const int tbx = gb::cdiv(img_w, 16), tby = gb::cdiv(img_h, 16);
  const int n_items = 8 * tbx * tby;
  int dev = 0;
  GB_CUDA(cudaGetDevice(&dev));
  // persistent grid: as many CTAs as fit on the device at once, each warp drawing items until they run out
  static int resident[64][3] = {};
  int uncached = 0;
  int& per_sm = (dev >= 0 && dev < 64) ? resident[dev][finish ? 2 : channels == 4] : uncached;
  if (per_sm == 0) {
    int n = 0, sms = 0;
    if (finish)
      GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, blend_bwd_lists_kernel<4, true>, kListThreads, 0));
    else if (channels == 4)
      GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, blend_bwd_lists_kernel<4>, kListThreads, 0));
    else
      GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, blend_bwd_lists_kernel<3>, kListThreads, 0));
    GB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    per_sm = max(1, n) * sms;
  }
  const int grid = min(per_sm, gb::cdiv(n_items, kListWarps));
  GB_CUDA(gb::launch<order_items_kernel>(1, 1024, 0, s, n_items, hit_count));
#define GB_BWD_LISTS(CC, FF)                                                                                            \
  GB_CUDA(gb::launch<blend_bwd_lists_kernel<CC, FF>>(grid, kListThreads, 0, s,                                          \
      img_w, img_h, tbx, n_items, (const int2*)tile_bins, hit_list, hit_count, hit_count + n_items, ranks,              \
      (const float4*)records, background, final_Ts, final_idx, v_output, v_output_alpha, v_xy, v_conic, v_colors,       \
      v_opacity, g_depth, alpha_img))
  if (finish) GB_BWD_LISTS(4, true); else if (channels == 3) GB_BWD_LISTS(3, false); else GB_BWD_LISTS(4, false);
#undef GB_BWD_LISTS
  return 0;
}

int launch_fwd_mom(int img_h, int img_w, int channels, const int32_t* tile_bins, const int32_t* tile_order, int sched,
                   const float* records, const float* background, float* out_img, float* final_Ts, int32_t* final_idx,
                   cudaStream_t s) {
  return launch_fwd_any(img_h, img_w, channels, tile_bins, tile_order, sched, records, nullptr, background, out_img, final_Ts,
                        final_idx, s);
}

int launch_bwd_mom(int img_h, int img_w, int channels, const int32_t* gids_sorted, const int32_t* tile_bins,
                   const int32_t* tile_order, int sched, const float* records, const float* background, const float* final_Ts,
                   const int32_t* final_idx, const float* v_output, const float* v_output_alpha, float* v_xy,
                   float* v_conic, float* v_colors, float* v_opacity, cudaStream_t s) {
  return launch_bwd_any(img_h, img_w, channels, gids_sorted, nullptr, tile_bins, tile_order, sched, records, background,
                        final_Ts, final_idx, v_output, v_output_alpha, v_xy, v_conic, v_colors, v_opacity, s);
}

}  // namespace gbblend

// ---------------------------------------------------------------- blend straight from the by-id record table, C ABI
// ranks_sorted [cap] (per tile: Gaussian ids in blend order), rec_by_rank [G,12] (by id), rank_to_gid [G] (identity,
// not read): outputs of gb_bin_tiles_ranked.  Same results as gb_rasterize_packed_fwd/bwd on the materialised records; final_idx indexes
// ranks_sorted.  channels 3 or 4; tile_order as for the packed kernels (launch order, may be NULL).
GB_API int gb_rasterize_ranked_fwd(int img_h, int img_w, int channels, const int32_t* tile_bins, const int32_t* tile_order,
                                   const int32_t* ranks_sorted, const float* rec_by_rank, const float* background,
                                   float* out_img, float* final_Ts, int32_t* final_idx, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if ((channels != 3 && channels != 4) || !ranks_sorted) return (int)cudaErrorInvalidValue;
  return gbblend::launch_fwd_any(img_h, img_w, channels, tile_bins, tile_order, 0, rec_by_rank, ranks_sorted, background,
                                 out_img, final_Ts, final_idx, (cudaStream_t)stream);
}
GB_API int gb_rasterize_ranked_bwd(int img_h, int img_w, int channels, const int32_t* rank_to_gid,
                                   const int32_t* ranks_sorted, const int32_t* tile_bins, const int32_t* tile_order,
                                   const float* rec_by_rank, const float* background, const float* final_Ts,
                                   const int32_t* final_idx, const float* v_output, const float* v_output_alpha,
                                   float* v_xy, float* v_conic, float* v_colors, float* v_opacity, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if ((channels != 3 && channels != 4) || !ranks_sorted) return (int)cudaErrorInvalidValue;
  return gbblend::launch_bwd_any(img_h, img_w, channels, rank_to_gid, ranks_sorted, tile_bins, tile_order, 0, rec_by_rank,
                                 background, final_Ts, final_idx, v_output, v_output_alpha, v_xy, v_conic, v_colors,
                                 v_opacity, (cudaStream_t)stream);
}
// The same pair with the backward walking per-warp hit lists the forward stores (blend_bwd_lists_kernel): hit_list
// [8 cap] and hit_count [16 T + 2] int32 (layout above order_items_kernel) are written by the forward and used by the
// backward, which may be run more than once on them.
GB_API int gb_rasterize_ranked_fwd_lists(int img_h, int img_w, int channels, const int32_t* tile_bins,
                                         const int32_t* tile_order, const int32_t* ranks_sorted, const float* rec_by_rank,
                                         const float* background, float* out_img, float* final_Ts, int32_t* final_idx,
                                         int32_t* hit_list, int32_t* hit_count, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if ((channels != 3 && channels != 4) || !ranks_sorted || !hit_list || !hit_count) return (int)cudaErrorInvalidValue;
  return gbblend::launch_fwd_any(img_h, img_w, channels, tile_bins, tile_order, 0, rec_by_rank, ranks_sorted, background,
                                 out_img, final_Ts, final_idx, (cudaStream_t)stream, hit_list, hit_count);
}
// gb_rasterize_ranked_fwd_lists on the unsorted buckets of gb_bin_tiles_buckets: each CTA sorts its tile's bucket
// (ids) by (depth key, id) before it blends, writing the sorted ids over the depth keys in ranks_keys [cap]: the same
// ranks_sorted as gb_bin_tiles_ranked's, read by the backward.  depths [G] are the depth keys the chunked path of tiles
// longer than the in-CTA sort's capacity reads by id.  Outputs identical to gb_bin_tiles_ranked +
// gb_rasterize_ranked_fwd_lists.
GB_API int gb_rasterize_ranked_fwd_sort_lists(int img_h, int img_w, int channels, const int32_t* tile_bins,
                                              const int32_t* tile_order, const float* depths, int32_t* bucket,
                                              int32_t* ranks_keys, const float* rec_by_rank, const float* background,
                                              float* out_img, float* final_Ts, int32_t* final_idx, int32_t* hit_list,
                                              int32_t* hit_count, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if ((channels != 3 && channels != 4) || !depths || !bucket || !ranks_keys || !hit_list || !hit_count)
    return (int)cudaErrorInvalidValue;
  return gbblend::launch_fwd_sort(img_h, img_w, channels, tile_bins, tile_order, depths, bucket, ranks_keys, rec_by_rank,
                                  background, out_img, final_Ts, final_idx, hit_list, hit_count, (cudaStream_t)stream);
}
// gb_rasterize_ranked_fwd_sort_lists (4 channels) that writes the finished view instead of the 4-channel image: rgb
// [3,H,W] = colour + T background, alpha [H,W] = 1 - T and depth [H,W] = (depth channel + T background[0]) /
// clamp(alpha, 0.05, 1), bit for bit what gb_render_finish_fwd makes of the 4-channel image and 1 - final_Ts.
// background holds 3 floats.  final_Ts, final_idx, ranks_keys, hit_list and hit_count are those of
// gb_rasterize_ranked_fwd_sort_lists.
GB_API int gb_rasterize_ranked_fwd_sort_finish(int img_h, int img_w, const int32_t* tile_bins,
                                               const int32_t* tile_order, const float* depths, int32_t* bucket,
                                               int32_t* ranks_keys, const float* rec_by_rank, const float* background,
                                               float* rgb, float* alpha, float* depth, float* final_Ts,
                                               int32_t* final_idx, int32_t* hit_list, int32_t* hit_count,
                                               void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if (!depths || !bucket || !ranks_keys || !hit_list || !hit_count || !rgb || !alpha || !depth)
    return (int)cudaErrorInvalidValue;
  return gbblend::launch_fwd_sort(img_h, img_w, 4, tile_bins, tile_order, depths, bucket, ranks_keys, rec_by_rank,
                                  background, rgb, final_Ts, final_idx, hit_list, hit_count, (cudaStream_t)stream,
                                  alpha, depth);
}
GB_API int gb_rasterize_ranked_bwd_lists(int img_h, int img_w, int channels, const int32_t* ranks_sorted,
                                         const int32_t* tile_bins, const int32_t* hit_list, int32_t* hit_count,
                                         const float* rec_by_rank, const float* background, const float* final_Ts,
                                         const int32_t* final_idx, const float* v_output, const float* v_output_alpha,
                                         float* v_xy, float* v_conic, float* v_colors, float* v_opacity, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if ((channels != 3 && channels != 4) || !ranks_sorted || !hit_list || !hit_count) return (int)cudaErrorInvalidValue;
  return gbblend::launch_bwd_lists(img_h, img_w, channels, ranks_sorted, tile_bins, hit_list, hit_count,
                                   rec_by_rank, background, final_Ts, final_idx, v_output, v_output_alpha, v_xy, v_conic,
                                   v_colors, v_opacity, (cudaStream_t)stream);
}
// gb_rasterize_ranked_bwd_lists behind gb_rasterize_ranked_fwd_sort_finish: g_rgb [3,H,W] and g_depth [H,W] (either
// may be NULL) are the gradients of the finished view, alpha [H,W] the forward's alpha (it takes no gradient).  The
// accumulated gradients are those of gb_render_finish_bwd + gb_rasterize_ranked_bwd_lists, up to the order of the
// atomic adds.  background holds 3 floats.
GB_API int gb_rasterize_ranked_bwd_lists_finish(int img_h, int img_w, const int32_t* ranks_sorted,
                                                const int32_t* tile_bins, const int32_t* hit_list, int32_t* hit_count,
                                                const float* rec_by_rank, const float* background,
                                                const float* final_Ts, const int32_t* final_idx, const float* alpha,
                                                const float* g_rgb, const float* g_depth, float* v_xy, float* v_conic,
                                                float* v_colors, float* v_opacity, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if (!ranks_sorted || !hit_list || !hit_count || !alpha) return (int)cudaErrorInvalidValue;
  return gbblend::launch_bwd_lists(img_h, img_w, 4, ranks_sorted, tile_bins, hit_list, hit_count, rec_by_rank,
                                   background, final_Ts, final_idx, g_rgb, nullptr, v_xy, v_conic, v_colors, v_opacity,
                                   (cudaStream_t)stream, true, g_depth, alpha);
}

// ---------------------------------------------------------------- four lighting conditions per pass (OLAT), C ABI
// wide records [cap, 20] fp32: geometry of the 48-byte records + 4 x rgb.
GB_API int gb_records_widen(int64_t cap, const int32_t* n_dev, const float* records, float* records_wide, void* stream) {
  if (cap <= 0) return 0;
  return gb::launch<records_widen_kernel>((unsigned)gb::cdiv64(cap, 256), 256, 0, (cudaStream_t)stream, cap, n_dev,
                                          (const float4*)records, (float4*)records_wide);
}
// colors: nk (1..4) consecutive [G,3] tables; missing conditions are blended as black.
GB_API int gb_records_set_colors4(int64_t cap, const int32_t* n_dev, const int32_t* gids_sorted, const float* colors, int nk,
                                  int64_t G, float* records_wide, void* stream) {
  if (cap <= 0) return 0;
  if (nk < 1 || nk > 4) return (int)cudaErrorInvalidValue;
  return gb::launch<records_set_colors4_kernel>((unsigned)gb::cdiv64(cap, 256), 256, 0, (cudaStream_t)stream, cap,
                                                n_dev, gids_sorted, colors, nk, G, (float4*)records_wide);
}
// out_planes [4][H][W][3]: the four conditions' images (background added); same tile_bins / order as the single pass.
GB_API int gb_rasterize_multi_fwd(int img_h, int img_w, const int32_t* tile_bins, const int32_t* tile_order, int sched,
                                  const float* records_wide, const float* background, float* out_planes, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if (sched && !tile_order) return (int)cudaErrorInvalidValue;
  const int tbx = gb::cdiv(img_w, 16), tby = gb::cdiv(img_h, 16);
  return gb::launch<blend_fwd_multi_kernel>(tbx * tby, kFwdThreads, 0, (cudaStream_t)stream,
      img_w, img_h, tbx, tile_order, sched, (const int2*)tile_bins, (const float4*)records_wide, background, out_planes);
}
// v_planes [4][H][W][3]; final_Ts / final_idx of the view (from the single-condition pass); v_xy / v_conic / v_opacity are
// accumulated into; v_colors12 [G,12] (zero-filled) receives the four colour gradients interleaved per Gaussian.
GB_API int gb_rasterize_multi_bwd(int img_h, int img_w, const int32_t* gids_sorted, const int32_t* tile_bins,
                                  const int32_t* tile_order, int sched, const float* records_wide, const float* background,
                                  const float* final_Ts, const int32_t* final_idx, const float* v_planes, float* v_xy,
                                  float* v_conic, float* v_colors12, float* v_opacity, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if (sched && !tile_order) return (int)cudaErrorInvalidValue;
  const int tbx = gb::cdiv(img_w, 16), tby = gb::cdiv(img_h, 16);
  return gb::launch<blend_bwd_multi_kernel>(tbx * tby, kBwdThreads, kMBwdSmem, (cudaStream_t)stream,
      img_w, img_h, tbx, tile_order, sched, gids_sorted, (const int2*)tile_bins, (const float4*)records_wide, background, final_Ts,
      final_idx, v_planes, v_xy, v_conic, v_colors12, v_opacity);
}
// v_colors12 [G,12] -> nk consecutive [G,3] tables (overwritten); clears v_colors12 for the next group.
GB_API int gb_colors12_unpack(int64_t G, int nk, float* v_colors12, float* v_colors, void* stream) {
  if (G <= 0) return 0;
  if (nk < 1 || nk > 4) return (int)cudaErrorInvalidValue;
  return gb::launch<colors12_unpack_kernel>((unsigned)gb::cdiv64(G, 256), 256, 0, (cudaStream_t)stream, G, nk,
                                            (float4*)v_colors12, v_colors);
}
