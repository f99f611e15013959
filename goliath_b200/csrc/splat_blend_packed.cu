// goliath_b200/csrc/splat_blend_packed.cu — the packed blend path: packed per-intersection records streamed
// with bulk async copies (TMA, cp.async.bulk + mbarrier), warp-level footprint culling, LPT tile order.
//
// Same arithmetic per (pixel, Gaussian) pair as csrc/splat_blend.cu (which restates gsplat 0.1.11
// rasterize_forward / rasterize_backward_kernel, call sites ca_code/utils/render_gsplat.py:65-78,90-104), so
// the outputs are bit-identical to that kernel's; only the work distribution changes:
//
//  1. gb_pack_records: after the sort, one thread per intersection gathers (xy, conic, opacity, colours) of
//     its Gaussian ONCE into a 48-byte record in sorted order, plus the half-extents (ex, ey) of the
//     axis-aligned box outside which alpha < 1/255 for every pixel.  Forward, backward and both colour
//     passes then stream the records linearly instead of gathering four arrays per tile batch.
//  2. a CTA owns one 16x16 tile; batches of 256 records (12 KB) land in shared memory through
//     cp.async.bulk (UBLKCP) completing on an mbarrier, double buffered: no per-thread gather
//     instructions, the next batch is in flight while the current one is blended.
//  3. each warp owns an 8x4 pixel footprint.  32 lanes test 32 records' boxes against the footprint in
//     one step (ballot), then the warp walks only the set bits in order.  At the RGCA operating point
//     (3-sigma radius ~6 px) this removes most of the per-pixel tests of the reference formulation, which
//     is issue-bound, not HBM-bound.
//  4. tiles are launched longest-list-first (gb_tile_order), so the tail of the grid is made of short tiles.
//  5. backward: the 10 per-Gaussian partial sums are reduced across the warp with a recursive-halving
//     exchange (12 shuffles instead of 50), accumulated per CTA in shared memory, and flushed with one set
//     of RED atomics per (tile, Gaussian).
#include "common.cuh"
#include "splat_blend_common.cuh"
#include "splat_record.cuh"

namespace {

using namespace gbblend;

// ------------------------------------------------------------------ record packing
template <int C>
__global__ void __launch_bounds__(256) pack_records_kernel(long long n, const int* __restrict__ gids_sorted,
                                                           const float2* __restrict__ xys,
                                                           const float* __restrict__ conics,
                                                           const float* __restrict__ colors,
                                                           const float* __restrict__ opac, float4* __restrict__ rec) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int g = gids_sorted[i];
  const float2 xy = xys[g];
  const float A = conics[3 * g], B = conics[3 * g + 1], Cc = conics[3 * g + 2];
  const float o = opac[g];
  float ex, ey;
  gb::cull_box(A, B, Cc, o, ex, ey);
  float c0, c1, c2, c3 = 0.f;
  if (C == 4) {
    const float4 col = reinterpret_cast<const float4*>(colors)[g];
    c0 = col.x; c1 = col.y; c2 = col.z; c3 = col.w;
  } else {
    c0 = colors[3 * g]; c1 = colors[3 * g + 1]; c2 = colors[3 * g + 2];
  }
  rec[3 * i + 0] = make_float4(xy.x, xy.y, ex, ey);
  rec[3 * i + 1] = make_float4(A, B, Cc, o);
  rec[3 * i + 2] = make_float4(c0, c1, c2, c3);
}

// Fused-render variant of the packing: the record's opacity is opacity * compensation and its 4th colour channel is
// the view-space depth, i.e. exactly what ca_code/utils/render_gsplat.py:72 and :97 feed to the two rasterise calls,
// without materialising those tensors.
__global__ void __launch_bounds__(256) pack_records_fused_kernel(long long n_cap, const int* __restrict__ n_dev,
                                                                 const int* __restrict__ gids_sorted,
                                                                 const float2* __restrict__ xys,
                                                                 const float* __restrict__ conics,
                                                                 const float* __restrict__ colors3,
                                                                 const float* __restrict__ depths,
                                                                 const float* __restrict__ opacity,
                                                                 const float* __restrict__ comp, float4* __restrict__ rec) {
  const long long n = n_dev ? min((long long)*n_dev, n_cap) : n_cap;  // count may live on the device (sync-free path)
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  gb::pack_record_fused(gids_sorted[i], xys, conics, colors3, depths, opacity, comp, rec + 3 * i);
}

// OLAT / multi-condition renders (SURVEY.md section 8d config 3): geometry, projection and tile lists of a view are shared by
// every lighting condition, only the colours change.  Rewrites the colour quarter (rgb + depth) of the packed records
// in place from a new [G,3] colour table: 16 B per intersection instead of a full re-pack.
__global__ void __launch_bounds__(256) records_set_colors_kernel(long long n_cap, const int* __restrict__ n_dev,
                                                                 const int* __restrict__ gids_sorted,
                                                                 const float* __restrict__ colors3,
                                                                 const float* __restrict__ depths, float4* __restrict__ rec) {
  const long long n = n_dev ? min((long long)*n_dev, n_cap) : n_cap;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int g = gids_sorted[i];
  rec[3 * i + 2] = make_float4(colors3[3 * g], colors3[3 * g + 1], colors3[3 * g + 2], depths[g]);
}

// Backward glue of the fused render: split the blend's per-Gaussian gradients back into the tensors the projection
// backward and the caller expect (product rule of opacity * compensation, depth = 4th colour channel).
__global__ void __launch_bounds__(256) splat_grad_unpack_kernel(int G, const float4* __restrict__ v_colors4,
                                                                const float* __restrict__ v_opac_eff,
                                                                const float* __restrict__ opacity,
                                                                const float* __restrict__ comp, float* __restrict__ v_colors3,
                                                                float* __restrict__ v_opacity, float* __restrict__ v_comp,
                                                                float* __restrict__ v_depth) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const float4 c = v_colors4[g];
  const float e = v_opac_eff[g];
  v_colors3[3 * g] = c.x; v_colors3[3 * g + 1] = c.y; v_colors3[3 * g + 2] = c.z;
  v_depth[g] = c.w;
  v_opacity[g] = e * comp[g];
  v_comp[g] = e * opacity[g];
}

// ------------------------------------------------------------------ LPT tile order (single CTA)
// order[] = tile ids sorted by descending list length (bucketed, stable); any tile count.
// With queues = Q > 0 the same array is a SCHEDULE (gb_tile_schedule): position p = k*Q + q is the k-th work item of
// queue q, the sorted sequence is dealt to the queues boustrophedon-wise (every other group of Q reversed), so the
// queues carry near-equal sums of list lengths, and Q + 1 draw counters follow at order[T .. T+Q] (zeroed here,
// restored to zero by every kernel launch that draws from them).
__global__ void __launch_bounds__(1024) tile_order_kernel(int T, const int2* __restrict__ tile_bins,
                                                          int* __restrict__ order, int queues) {
  constexpr int kBuckets = 1024;
  __shared__ int s_cnt[kBuckets];
  __shared__ int s_warp[33];
  for (int i = threadIdx.x; i < kBuckets; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  auto bucket = [](int len) { return kBuckets - 1 - min(len >> 3, kBuckets - 1); };  // long lists -> low bucket
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const int2 r = tile_bins[t];
    atomicAdd(&s_cnt[bucket(r.y - r.x)], 1);
  }
  __syncthreads();
  // exclusive scan of 1024 counters with 1024 threads
  {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int v = s_cnt[threadIdx.x];
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane], winc = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, winc, o);
        if (lane >= o) winc += t;
      }
      s_warp[lane] = winc - w;
    }
    __syncthreads();
    s_cnt[threadIdx.x] = s_warp[warp] + inc - v;
  }
  __syncthreads();
  // scatter; order inside a bucket is irrelevant for correctness (any permutation is a valid launch order)
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const int2 r = tile_bins[t];
    int pos = atomicAdd(&s_cnt[bucket(r.y - r.x)], 1);
    if (queues > 0) {
      const int grp = pos / queues;
      if ((grp & 1) && (grp + 1) * queues <= T) pos = grp * queues + (queues - 1 - (pos - grp * queues));
    }
    order[pos] = t;
  }
  for (int i = threadIdx.x; i <= queues && queues > 0; i += blockDim.x) order[T + i] = 0;
}

// ------------------------------------------------------------------ shared helpers
struct Tile {
  int tile_id, tx, ty;
};
__device__ __forceinline__ Tile pick_tile(const int* __restrict__ order, int tbx) {
  Tile t;
  t.tile_id = order ? order[blockIdx.x] : (int)blockIdx.x;
  t.ty = t.tile_id / tbx;
  t.tx = t.tile_id - t.ty * tbx;
  return t;
}

// ------------------------------------------------------------------ forward
template <int C>
__global__ void __launch_bounds__(kThreads) blend_fwd_packed_kernel(
    int img_w, int img_h, int tbx, const int* __restrict__ order, const int2* __restrict__ tile_bins,
    const float4* __restrict__ rec, const float* __restrict__ background, float* __restrict__ final_Ts,
    int* __restrict__ final_idx, float* __restrict__ out_img) {
  __shared__ __align__(128) float4 s_rec[2][kBatch * 3];
  __shared__ __align__(8) unsigned long long s_bar[2];

  const Tile tl = pick_tile(order, tbx);
  const int tr = threadIdx.x, lane = tr & 31, warp = tr >> 5;
  // warp w -> 8x4 pixel footprint
  const int wx0 = tl.tx * 16 + ((warp & 1) << 3), wy0 = tl.ty * 16 + ((warp >> 1) << 2);
  const int pxi = wx0 + (lane & 7), pyi = wy0 + (lane >> 3);
  const bool inside = (pxi < img_w) && (pyi < img_h);
  const float px = (float)pxi + 0.5f, py = (float)pyi + 0.5f;
  // footprint of pixel centres, for the box test
  const float fx0 = (float)wx0 + 0.5f, fx1 = (float)wx0 + 7.5f, fy0 = (float)wy0 + 0.5f, fy1 = (float)wy0 + 3.5f;

  const int2 range = tile_bins[tl.tile_id];
  const int num_batches = (range.y - range.x + kBatch - 1) / kBatch;

  if (tr == 0) {
    mbar_init(&s_bar[0], 1);
    mbar_init(&s_bar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto issue = [&](int b) {  // thread 0 only
    const int start = range.x + b * kBatch;
    const unsigned bytes = (unsigned)min(kBatch, range.y - start) * kRecBytes;
    mbar_expect_tx(&s_bar[b & 1], bytes);
    bulk_g2s(&s_rec[b & 1][0], rec + (size_t)start * 3, bytes, &s_bar[b & 1]);
  };
  if (tr == 0 && num_batches > 0) issue(0);

  bool done = !inside;
  float T = 1.f;
  int cur_idx = 0;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};

  for (int b = 0; b < num_batches; ++b) {
    // every thread is past batch b-1 here, so stage (b+1)&1 may be refilled; also the tile-done test
    if (__syncthreads_count(done) >= kThreads) {
      // batch b is already in flight: it must land before the CTA (and its shared memory) retires
      if (tr == 0) mbar_wait(&s_bar[b & 1], (unsigned)((b >> 1) & 1));
      break;
    }
    if (tr == 0 && b + 1 < num_batches) issue(b + 1);
    mbar_wait(&s_bar[b & 1], (unsigned)((b >> 1) & 1));
    const float4* sr = s_rec[b & 1];
    const int batch_start = range.x + b * kBatch;
    const int batch_size = min(kBatch, range.y - batch_start);
    if (__all_sync(0xffffffffu, done)) continue;
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
__global__ void __launch_bounds__(kThreads) blend_bwd_packed_kernel(
    int img_w, int img_h, int tbx, const int* __restrict__ order, const int* __restrict__ gids_sorted,
    const int2* __restrict__ tile_bins, const float4* __restrict__ rec, const float* __restrict__ background,
    const float* __restrict__ final_Ts, const int* __restrict__ final_idx, const float* __restrict__ v_output,
    const float* __restrict__ v_output_alpha, float* __restrict__ v_xy, float* __restrict__ v_conic,
    float* __restrict__ v_colors, float* __restrict__ v_opacity) {
  constexpr int NV = C + 6;  // colours, conic(3), xy(2), opacity
  constexpr int kStride = 11;  // odd stride: conflict-free flush
  __shared__ __align__(128) float4 s_rec[2][kBatch * 3];
  __shared__ __align__(8) unsigned long long s_bar[2];
  __shared__ float s_grad[kBatch * kStride];
  __shared__ int s_touched[kBatch];
  __shared__ int s_cta_final;

  const Tile tl = pick_tile(order, tbx);
  const int2 range = tile_bins[tl.tile_id];
  if (range.y <= range.x) return;
  const int tr = threadIdx.x, lane = tr & 31, warp = tr >> 5;
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
    mbar_init(&s_bar[0], 1);
    mbar_init(&s_bar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (lane == 0) atomicMax(&s_cta_final, warp_bin_final);
  __syncthreads();
  // the walk starts at the last index any pixel of the tile needs and goes down to range.x
  const int last = min(s_cta_final, range.y - 1);
  if (last < range.x) return;  // no pixel of this tile blended anything (CTA-uniform: nothing is in flight yet)
  const int num_batches = (last - range.x + kBatch) / kBatch;  // ceil((last - range.x + 1) / kBatch)
  // batch k (k = 0 is the furthest back) covers indices [hi_k - size_k + 1, hi_k], hi_k = last - k*kBatch
  auto issue = [&](int k) {
    const int hi = last - k * kBatch;
    const int lo = max(range.x, hi - kBatch + 1);
    const unsigned bytes = (unsigned)(hi - lo + 1) * kRecBytes;
    mbar_expect_tx(&s_bar[k & 1], bytes);
    bulk_g2s(&s_rec[k & 1][0], rec + (size_t)lo * 3, bytes, &s_bar[k & 1]);
  };
  if (tr == 0) issue(0);

  for (int k = 0; k < num_batches; ++k) {
    __syncthreads();  // previous batch fully consumed (records, s_grad flush)
    if (tr == 0 && k + 1 < num_batches) issue(k + 1);
    const int hi = last - k * kBatch;
    const int lo = max(range.x, hi - kBatch + 1);
    const int batch_size = hi - lo + 1;
    for (int i = tr; i < kBatch * kStride; i += kThreads) s_grad[i] = 0.f;
    s_touched[tr] = 0;
    mbar_wait(&s_bar[k & 1], (unsigned)((k >> 1) & 1));
    __syncthreads();
    const float4* sr = s_rec[k & 1];
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
        if (!(lane & 1) && sv && slot < NV) atomicAdd(&s_grad[j * kStride + slot], r);
        if (lane == 0) s_touched[j] = 1;
      }
    }
    __syncthreads();
    if (tr < batch_size && s_touched[tr]) {
      const int g = gids_sorted[lo + tr];
      const float* sg = &s_grad[tr * kStride];
#pragma unroll
      for (int c = 0; c < C; ++c) gb::red_add(v_colors + (size_t)C * g + c, sg[c]);
      gb::red_add(v_conic + 3 * (size_t)g + 0, sg[C + 0]);
      gb::red_add(v_conic + 3 * (size_t)g + 1, sg[C + 1]);
      gb::red_add(v_conic + 3 * (size_t)g + 2, sg[C + 2]);
      gb::red_add_v2(v_xy + 2 * (size_t)g, sg[C + 3], sg[C + 4]);
      gb::red_add(v_opacity + g, sg[C + 5]);
    }
  }
}

}  // namespace

// Gather the per-intersection blend records in sorted order.  records: [n, 12] fp32, 16-byte aligned.
GB_API int gb_pack_records(int64_t n, int channels, const int32_t* gids_sorted, const float* xys,
                           const float* conics, const float* colors, const float* opacities, float* records,
                           void* stream) {
  if (n <= 0) return 0;
  if (channels != 3 && channels != 4) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)gb::cdiv64(n, 256);
  if (channels == 3)
    GB_CUDA(gb::launch<pack_records_kernel<3>>(blocks, 256, 0, s, n, gids_sorted, (const float2*)xys, conics, colors,
                                               opacities, (float4*)records));
  else
    GB_CUDA(gb::launch<pack_records_kernel<4>>(blocks, 256, 0, s, n, gids_sorted, (const float2*)xys, conics, colors,
                                               opacities, (float4*)records));
  return 0;
}

// Fused-render packing: records carry opacity*compensation and (rgb, depth); see pack_records_fused_kernel.
static int pack_fused_impl(int64_t n, const int32_t* n_dev, const int32_t* gids_sorted, const float* xys,
                           const float* conics, const float* colors3, const float* depths, const float* opacity,
                           const float* compensation, float* records, void* stream) {
  if (n <= 0) return 0;
  return gb::launch<pack_records_fused_kernel>((unsigned)gb::cdiv64(n, 256), 256, 0, (cudaStream_t)stream,
      n, n_dev, gids_sorted, (const float2*)xys, conics, colors3, depths, opacity, compensation, (float4*)records);
}
GB_API int gb_pack_records_fused(int64_t n, const int32_t* gids_sorted, const float* xys, const float* conics,
                                 const float* colors3, const float* depths, const float* opacity,
                                 const float* compensation, float* records, void* stream) {
  return pack_fused_impl(n, nullptr, gids_sorted, xys, conics, colors3, depths, opacity, compensation, records, stream);
}
// sync-free variant: `cap` sizes the launch, the count is read from *n_dev on the device
GB_API int gb_pack_records_fused_dn(int64_t cap, const int32_t* n_dev, const int32_t* gids_sorted, const float* xys,
                                    const float* conics, const float* colors3, const float* depths,
                                    const float* opacity, const float* compensation, float* records, void* stream) {
  return pack_fused_impl(cap, n_dev, gids_sorted, xys, conics, colors3, depths, opacity, compensation, records, stream);
}

// Colour quarter of the fused-render records from another colour table (same geometry): records[i].c = (colors3[g], depths[g]).
// n_dev (device int32, may be NULL) = number of valid records; cap sizes the launch.
GB_API int gb_records_set_colors(int64_t cap, const int32_t* n_dev, const int32_t* gids_sorted, const float* colors3,
                                 const float* depths, float* records, void* stream) {
  if (cap <= 0) return 0;
  return gb::launch<records_set_colors_kernel>((unsigned)gb::cdiv64(cap, 256), 256, 0, (cudaStream_t)stream,
      cap, n_dev, gids_sorted, colors3, depths, (float4*)records);
}

// Backward glue of the fused render (all outputs overwritten): v_colors3 [G,3], v_opacity [G], v_comp [G], v_depth [G].
GB_API int gb_splat_grad_unpack(int G, const float* v_colors4, const float* v_opac_eff, const float* opacity,
                                const float* compensation, float* v_colors3, float* v_opacity, float* v_comp,
                                float* v_depth, void* stream) {
  if (G <= 0) return 0;
  return gb::launch<splat_grad_unpack_kernel>(gb::cdiv(G, 256), 256, 0, (cudaStream_t)stream,
      G, (const float4*)v_colors4, v_opac_eff, opacity, compensation, v_colors3, v_opacity, v_comp, v_depth);
}

// Launch order of the tiles: longest list first.  order: [T] int32.
GB_API int gb_tile_order(int num_tiles, const int32_t* tile_bins, int32_t* order, void* stream) {
  if (num_tiles <= 0) return 0;
  return gb::launch<tile_order_kernel>(1, 1024, 0, (cudaStream_t)stream, num_tiles, (const int2*)tile_bins, order, 0);
}

// SM-affine schedule of the tiles: `sched` holds gb_tile_schedule_ints(num_tiles) int32.  One queue per SM, filled
// boustrophedon-wise from the longest-first order so that the queues carry near-equal work; consumed by
// gb_rasterize_sched_fwd / _bwd, whose CTAs draw from the queue of the SM they run on (csrc/splat_blend_pipe.cu).
GB_API int gb_tile_schedule_ints(int num_tiles) { return (num_tiles > 0 ? num_tiles : 0) + gbblend::kSchedQueues + 1; }
GB_API int gb_tile_schedule(int num_tiles, const int32_t* tile_bins, int32_t* sched, void* stream) {
  if (num_tiles <= 0) return 0;
  return gb::launch<tile_order_kernel>(1, 1024, 0, (cudaStream_t)stream, num_tiles, (const int2*)tile_bins, sched,
                                       gbblend::kSchedQueues);
}

// Blend forward over packed records (block_width == 16).  tile_order may be NULL (row-major launch order).
GB_API int gb_rasterize_packed_fwd(int img_h, int img_w, int channels, const int32_t* tile_bins,
                                   const int32_t* tile_order, const float* records, const float* background,
                                   float* out_img, float* final_Ts, int32_t* final_idx, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if (channels != 3 && channels != 4) return (int)cudaErrorInvalidValue;
  const int tbx = gb::cdiv(img_w, 16), tby = gb::cdiv(img_h, 16);
  cudaStream_t s = (cudaStream_t)stream;
  if (gb_get_blend_mode() >= 3)  // exact cull + hit-ILP forward (csrc/splat_blend_mom.cu), identical pixels
    return gbblend::launch_fwd_mom(img_h, img_w, channels, tile_bins, tile_order, 0, records, background, out_img, final_Ts,
                                   final_idx, s);
  if (gb_get_blend_mode())  // warp-decoupled pipeline (csrc/splat_blend_pipe.cu), identical outputs
    return gbblend::launch_fwd_pipe(img_h, img_w, channels, tile_bins, tile_order, 0, records, background, out_img,
                                    final_Ts, final_idx, s);
  if (channels == 3)
    GB_CUDA(gb::launch<blend_fwd_packed_kernel<3>>(tbx * tby, kThreads, 0, s, img_w, img_h, tbx, tile_order,
                                                   (const int2*)tile_bins, (const float4*)records, background, final_Ts,
                                                   final_idx, out_img));
  else
    GB_CUDA(gb::launch<blend_fwd_packed_kernel<4>>(tbx * tby, kThreads, 0, s, img_w, img_h, tbx, tile_order,
                                                   (const int2*)tile_bins, (const float4*)records, background, final_Ts,
                                                   final_idx, out_img));
  return 0;
}

// Blend backward over packed records (block_width == 16); gradients are accumulated into (caller zeroes).
GB_API int gb_rasterize_packed_bwd(int img_h, int img_w, int channels, const int32_t* gids_sorted,
                                   const int32_t* tile_bins, const int32_t* tile_order, const float* records,
                                   const float* background, const float* final_Ts, const int32_t* final_idx,
                                   const float* v_output, const float* v_output_alpha, float* v_xy, float* v_conic,
                                   float* v_colors, float* v_opacity, void* stream) {
  if (img_h <= 0 || img_w <= 0) return 0;
  if (channels != 3 && channels != 4) return (int)cudaErrorInvalidValue;
  const int tbx = gb::cdiv(img_w, 16), tby = gb::cdiv(img_h, 16);
  cudaStream_t s = (cudaStream_t)stream;
  if (gb_get_blend_mode() >= 3)  // transposed-reduction backward (csrc/splat_blend_mom.cu)
    return gbblend::launch_bwd_mom(img_h, img_w, channels, gids_sorted, tile_bins, tile_order, 0, records, background,
                                   final_Ts, final_idx, v_output, v_output_alpha, v_xy, v_conic, v_colors, v_opacity, s);
  if (gb_get_blend_mode())
    return gbblend::launch_bwd_pipe(img_h, img_w, channels, gids_sorted, tile_bins, tile_order, 0, records, background,
                                    final_Ts, final_idx, v_output, v_output_alpha, v_xy, v_conic, v_colors, v_opacity,
                                    s);
  if (channels == 3)
    GB_CUDA(gb::launch<blend_bwd_packed_kernel<3>>(tbx * tby, kThreads, 0, s, img_w, img_h, tbx, tile_order,
                                                   gids_sorted, (const int2*)tile_bins, (const float4*)records,
                                                   background, final_Ts, final_idx, v_output, v_output_alpha, v_xy,
                                                   v_conic, v_colors, v_opacity));
  else
    GB_CUDA(gb::launch<blend_bwd_packed_kernel<4>>(tbx * tby, kThreads, 0, s, img_w, img_h, tbx, tile_order,
                                                   gids_sorted, (const int2*)tile_bins, (const float4*)records,
                                                   background, final_Ts, final_idx, v_output, v_output_alpha, v_xy,
                                                   v_conic, v_colors, v_opacity));
  return 0;
}
