// goliath_b200/csrc/splat_bin_tiles.cu — tile binning for the fused render path, sm_90a.
//
// Produces exactly what the key sort of csrc/splat_bin.cu produces for the fused render — per-tile
// [first,last) bins, the Gaussian ids of every tile in front-to-back order (ties: ascending id), and the
// packed blend records — i.e. the work gsplat 0.1.11 does in bin_and_sort_gaussians (called from
// rasterize_gaussians, call sites ca_code/utils/render_gsplat.py:65-78,90-104), but without ever sorting
// the I (tile, depth) intersection keys globally.  Ordering a tile only needs the (depth key, Gaussian id) pairs of
// that tile, and a tile holds a few hundred to a few thousand of them, so each tile is sorted by one CTA in shared
// memory:
//
//   1. tile_count_kernel     G threads: the per-tile intersection COUNT of every visible Gaussian.  Counts are
//                            privatised per CTA in shared memory and flushed with one RED per (CTA, non-empty tile):
//                            the hot tiles of a head scene take ~4000 hits each, which serialise on the L2 atomic
//                            unit when issued one by one.
//   2. tile_scan_kernel      one CTA: exclusive scan of the T counts -> tile_bins (clamped to the capacity),
//                            scatter cursors, total count, overflow flag.  Then the launch order of the tiles
//                            (gb_tile_order, longest first, or the SM-affine schedule of gb_tile_schedule).
//   3. tile_scatter_kernel   G threads: every (Gaussian, tile) pair drops the Gaussian's ID into the tile's bucket
//                            (order inside the bucket arbitrary) and its depth key at the same slot of the output
//                            array.  Slots are claimed per CTA: count in shared memory, one atomicAdd per (CTA, tile)
//                            on the global cursor; the pairs are staged tile by tile in shared memory and written out
//                            as runs of consecutive slots.  The same threads write the 48-byte blend record of their
//                            Gaussian into a table indexed BY ID (cull box computed once per Gaussian, not once per
//                            intersection), one contiguous span per warp.
//   4. tile_sort_kernel      one CTA per tile, in launch order, on the 64-bit key (depth bits - tile minimum) << id
//                            bits | (id - tile minimum), over the bits that vary inside the tile only (CTA min/max
//                            reduction).  Buckets of up to kSortCap entries are spread over all warps and sorted in
//                            registers + shared memory by stable LSD passes (9-bit digits) over the DEPTH bits only;
//                            the id bits only break ties, and ties come in short runs (at most 3 entries on the bench
//                            head), so the thread holding the first entry of each equal-depth run then sorts the run
//                            by the full key in place.  A tile with a run longer than kTieRun runs the passes over the
//                            full key instead.  Longer buckets run the full-key passes chunk by chunk through global
//                            memory (the bucket and the output array serve as the ping-pong pair, keys are gathered
//                            by id).  The sorted ids overwrite the keys in the output array.  The sort itself is
//                            TileSort::sort_tile (csrc/splat_tile_sort.cuh).  gb_bin_tiles_buckets stops before this
//                            kernel: the head step's forward (gb_rasterize_ranked_fwd_sort_lists) runs the same sort
//                            in each blend CTA before it blends the tile, so a light tile's sort runs underneath a heavy
//                            tile's blend instead of in a kernel of its own between the scatter and the blend.
//   5. gather_records_kernel (packed callers only) the sorted 48-byte records, copied from the by-id table.
//
// Integer/byte work with a BIT-EXACT contract: gids_sorted, tile_bins and records are identical to the
// key-sort path's (tests/test_splat_gpu.py::test_bin_tiles_matches_key_sort).

#include "common.cuh"
#include "splat_record.cuh"
#include "splat_tile_sort.cuh"

#include <algorithm>

extern "C" int gb_tile_order(int num_tiles, const int32_t* tile_bins, int32_t* order, void* stream);
extern "C" int gb_tile_schedule(int num_tiles, const int32_t* tile_bins, int32_t* sched, void* stream);
GB_API int gb_bin_tiles_pack_ev(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                                const float* colors3, const float* opacity, const float* compensation, int img_h,
                                int img_w, int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order,
                                int tile_sched, int32_t* gids_sorted, float* records, int32_t* n_out, int32_t* overflow,
                                void* workspace, void* colors_ready, void* stream);

namespace {

constexpr int kGaussBlock = 1024;                     // threads of the per-Gaussian kernels
constexpr int kScatItems = 3;                         // Gaussians per thread in tile_scatter_kernel, at most
constexpr int kMaxSmemTiles = 20 * 1024;              // per-CTA tile counters (x2 in the scatter) in shared memory
// Largest view the bucket binning takes (1.5 x 2^20 Gaussians, the native RGCA head has 2^20).  The sort itself has no
// such bound; the range is what gb_bin_tiles_supported reports to callers, and the fused render (gsplat/fused.py) uses
// the key sort of csrc/splat_bin.cu above it.
constexpr int kMaxGaussians = 3 << 19;

// Per-tile sort (csrc/splat_tile_sort.cuh).  kSortCap = 5120 entries are sorted in registers + shared memory (10 per
// thread: 64 registers without spills at two CTAs per SM).  The longest tile of the 300k-Gaussian bench head (1024x667,
// 16 ring cameras) holds 4223 entries; the 2^20-Gaussian head (test_fullpath_gpu.py, ring camera 2) reaches 13754, and
// 300 to 444 of its tiles (the counts above 6144 and above 4096) take the chunked path.
constexpr int kSortThreads = 512;
using Sort = gbsort::TileSort<kSortThreads, 10>;
constexpr int kSortCap = Sort::kCap;
using gbsort::block_exclusive_scan;

// Gaussians per CTA of tile_count_kernel: 2048 up to ~400k Gaussians, 4096 beyond (fewer counter flushes)
inline int count_items(int G) { return G <= 2048 * 192 ? 2 : 4; }

// tile rectangle of a Gaussian: same arithmetic as map_to_intersects_kernel (csrc/splat_bin.cu)
__device__ __forceinline__ void tile_bbox(float cx, float cy, float radius, int tbx, int tby, int bw, int& x0,
                                          int& y0, int& x1, int& y1) {
  const float fb = (float)bw;
  const float tcx = __fdiv_rn(cx, fb), tcy = __fdiv_rn(cy, fb), tr = __fdiv_rn(radius, fb);
  x0 = min(max(0, __float2int_rz(__fsub_rn(tcx, tr))), tbx);
  x1 = min(max(0, __float2int_rz(__fadd_rn(__fadd_rn(tcx, tr), 1.f))), tbx);
  y0 = min(max(0, __float2int_rz(__fsub_rn(tcy, tr))), tby);
  y1 = min(max(0, __float2int_rz(__fadd_rn(__fadd_rn(tcy, tr), 1.f))), tby);
}

// ------------------------------------------------------------------ 1. tile counts
// smem_tiles = T: per-CTA counters in dynamic shared memory; 0: global atomics (more tiles than fit).
// Few fat CTAs keep the number of counter flushes low, many threads per CTA keep enough loads in flight.
// rects [G]: the tile rectangle (x0, y0, x1, y1) of every Gaussian, x0 = -1 when it is culled, for the scatter.
// identity (may be null): written with identity[i] = i, the rank_to_gid table of gb_bin_tiles_ranked.
template <int kItems>
__global__ void __launch_bounds__(kGaussBlock) tile_count_kernel(int G, const float2* __restrict__ xys,
                                                                 const int* __restrict__ radii, int tbx, int tby,
                                                                 int block_width, int smem_tiles,
                                                                 int* __restrict__ tile_counts, int4* __restrict__ rects,
                                                                 int* __restrict__ identity) {
  extern __shared__ int s_cnt[];
  for (int t = threadIdx.x; t < smem_tiles; t += kGaussBlock) s_cnt[t] = 0;
  const int base = blockIdx.x * (kGaussBlock * kItems);
  int r[kItems];
  float2 c[kItems];
#pragma unroll
  for (int j = 0; j < kItems; ++j) {  // all loads first: independent, in flight together
    const int i = base + j * kGaussBlock + threadIdx.x;
    const bool in = i < G;
    r[j] = in ? radii[i] : 0;
    c[j] = in ? xys[i] : make_float2(0.f, 0.f);
    if (in && identity) identity[i] = i;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < kItems; ++j) {
    const int i = base + j * kGaussBlock + threadIdx.x;
    if (i >= G) continue;
    if (r[j] <= 0) {
      rects[i] = make_int4(-1, 0, 0, 0);
      continue;
    }
    int x0, y0, x1, y1;
    tile_bbox(c[j].x, c[j].y, (float)r[j], tbx, tby, block_width, x0, y0, x1, y1);
    rects[i] = make_int4(x0, y0, x1, y1);
    for (int ty = y0; ty < y1; ++ty)
      for (int tx = x0; tx < x1; ++tx) {
        if (smem_tiles) atomicAdd(&s_cnt[ty * tbx + tx], 1);
        else atomicAdd(&tile_counts[ty * tbx + tx], 1);
      }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < smem_tiles; t += kGaussBlock) {
    const int cnt = s_cnt[t];
    if (cnt) atomicAdd(&tile_counts[t], cnt);
  }
}

// ------------------------------------------------------------------ 2. bins from the tile counts (one CTA)
__global__ void __launch_bounds__(1024) tile_scan_kernel(int T, long long cap, const int* __restrict__ counts,
                                                         int2* __restrict__ tile_bins, int* __restrict__ cursor,
                                                         int* __restrict__ n_out, int* __restrict__ overflow) {
  __shared__ int s_warp[33];
  int carry = 0;
  for (int base = 0; base < T; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int v = (i < T) ? counts[i] : 0;
    int total;
    const int ex = block_exclusive_scan(v, s_warp, total);
    if (i < T) {
      const int s = carry + ex;
      cursor[i] = s;
      const int cs = (int)min((long long)s, cap), ce = (int)min((long long)s + v, cap);
      tile_bins[i] = (ce > cs) ? make_int2(cs, ce) : make_int2(0, 0);  // empty tiles read (0,0), as after torch.zeros
    }
    carry += total;
  }
  if (threadIdx.x == 0) {
    if (n_out) *n_out = carry;
    if (overflow && (long long)carry > cap) *overflow = 1;  // capacity exceeded: caller must re-run
  }
}

// ------------------------------------------------------------------ 3. ids + depth keys into the tile buckets, by-id records
// Every (Gaussian, tile) pair puts the Gaussian's id at a slot of the tile's bucket (tile_ids) and its 32-bit depth key
// at the same slot of `keys` (the caller's output array, which the sort overwrites with sorted ids), so the sort reads
// both contiguously instead of gathering depth_keys[id].
//
// smem_tiles = T: slots claimed per CTA through shared memory; 0: one global atomic per (Gaussian, tile).
// per_cta Gaussians per CTA (a multiple of 32, at most kScatItems x kGaussBlock; see scatter_per_cta).  The tile
// rectangles come from tile_count_kernel, so both kernels walk the same tiles by construction.
//
// The kernel's time went into stores, not atomics.  On the bench head (H100 80GB HBM3, 700 W, 1980 MHz max SM clock)
// the record pack took 17 us of 42 and the placement walk 20 us, and making the placement atomic non-returning changed
// nothing: one 4-byte store per pair scattered over the whole bucket, and 16-byte record parts at a 48-byte stride,
// cost about as much per store as full sectors would.  So with stage_cap > 0 both go through shared memory:
//   - each warp writes the records of its 32 consecutive Gaussians as one contiguous 1536-byte span;
//   - the CTA's pairs are placed tile by tile into a staging buffer of stage_cap (id, key, tile) entries, then written
//     out in that order: the CTA's entries of one tile are consecutive slots of the bucket, written by neighbouring
//     lanes.  A CTA with more pairs than the buffer holds writes each pair directly at the same slot instead.
// Dynamic shared memory: s_cnt [T] int | s_off [T] int | s_id [stage_cap] int | s_key [stage_cap] | s_tile [stage_cap]
// u16.  The record spans (kGaussBlock / 32 warps x 96 float4 = 48 KB) borrow s_id | s_key before the walks.
constexpr int kStageCap = 12 * 1024;                   // staged pairs per CTA: 8.3k on average on the bench head
constexpr int kStageMaxTiles = 10 * 1024;              // larger grids leave no room for the staging buffer
constexpr size_t kStageEntryBytes = 4 + 4 + 2;
static_assert(kStageCap * 8 >= (kGaussBlock / 32) * 96 * 16, "the record spans fit in s_id | s_key");

// Gaussians per scatter CTA: the view spread over one wave of CTAs (one CTA per SM: 1024 threads and the staging
// buffer).  A CTA runs its phases (loads, records, count walk, claims and scan, placement, write-out) one after the
// other between barriers, so a second, nearly empty wave costs almost as much as the first: at 2048 Gaussians per CTA
// the bench head's 300k took 147 CTAs on the 132 SMs of an H100 SXM, and one wave of 131 took the kernel from 31.9 to
// 23.7 us.
inline int scatter_per_cta(int G, int num_sms) {
  const int per_sm = gb::cdiv(G, num_sms > 0 ? num_sms : 1);
  return std::min(kScatItems * kGaussBlock, std::max(kGaussBlock, (per_sm + 31) & ~31));
}

inline int scatter_stage_cap(int smem_tiles) { return (smem_tiles > 0 && smem_tiles <= kStageMaxTiles) ? kStageCap : 0; }
inline size_t scatter_smem_bytes(int smem_tiles) {
  return (size_t)((smem_tiles + 3) & ~3) * 8 + (size_t)scatter_stage_cap(smem_tiles) * kStageEntryBytes;
}

__global__ void __launch_bounds__(kGaussBlock, 1) tile_scatter_kernel(
    int G, const int4* __restrict__ rects, const float2* __restrict__ xys, const float* __restrict__ conics,
    const float* __restrict__ colors3, const float* __restrict__ depths, const float* __restrict__ opacity,
    const float* __restrict__ comp, int tbx, long long cap, int per_cta, int smem_tiles, int stage_cap,
    int* __restrict__ cursor, int* __restrict__ tile_ids, unsigned* __restrict__ keys, float4* __restrict__ rec_by_id) {
  extern __shared__ int s_cnt[];
  __shared__ int s_warp[33];
  const int tpad = (smem_tiles + 3) & ~3;  // keeps the record spans 16-byte aligned
  int* s_off = s_cnt + tpad;
  int* s_id = s_off + tpad;
  unsigned* s_key = reinterpret_cast<unsigned*>(s_id + stage_cap);
  unsigned short* s_tile = reinterpret_cast<unsigned short*>(s_key + stage_cap);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = threadIdx.x; t < smem_tiles; t += kGaussBlock) s_cnt[t] = 0;
  const int base = blockIdx.x * per_cta, end = min(G, base + per_cta);
  int4 rc[kScatItems];
  unsigned dk[kScatItems];
#pragma unroll
  for (int j = 0; j < kScatItems; ++j) {  // all loads first: independent, in flight together
    const int i = base + j * kGaussBlock + threadIdx.x;
    rc[j] = (i < end) ? rects[i] : make_int4(-1, 0, 0, 0);
    dk[j] = (i < end) ? __float_as_uint(depths[i]) : 0u;
  }
  __syncthreads();
  unsigned bx[kScatItems], by[kScatItems];  // x0 | x1 << 16, y0 | y1 << 16 (tile coordinates < 65536)
#pragma unroll
  for (int j = 0; j < kScatItems; ++j) {
    const int i = base + j * kGaussBlock + threadIdx.x;
    const bool vis = rc[j].x >= 0;  // false: culled or past the CTA's Gaussians
    bx[j] = vis ? (unsigned)rc[j].x | ((unsigned)rc[j].z << 16) : 0u;
    by[j] = vis ? (unsigned)rc[j].y | ((unsigned)rc[j].w << 16) : 0u;
    if (stage_cap && j * kGaussBlock < per_cta) {  // the warp's 32 records through shared memory, then one span
      float4* span = reinterpret_cast<float4*>(s_id) + warp * 96;
      if (vis) gb::pack_record_fused(i, xys, conics, colors3, depths, opacity, comp, span + 3 * lane);
      const unsigned vmask = __ballot_sync(0xffffffffu, vis);
      __syncwarp();
      float4* dst = rec_by_id + 3 * (size_t)(i - lane);
#pragma unroll
      for (int f = lane; f < 96; f += 32) {
        const int r = f / 3, part = f - 3 * r;
        if (((vmask >> r) & 1u) && (part < 2 || colors3)) dst[f] = span[f];
      }
      __syncwarp();
    } else if (vis) {
      gb::pack_record_fused(i, xys, conics, colors3, depths, opacity, comp, rec_by_id + 3 * (size_t)i);
    }
  }
  if (!smem_tiles) {
#pragma unroll
    for (int j = 0; j < kScatItems; ++j) {
      const int i = base + j * kGaussBlock + threadIdx.x;
      const int x0 = bx[j] & 0xffffu, x1 = bx[j] >> 16, y0 = by[j] & 0xffffu, y1 = by[j] >> 16;
      for (int ty = y0; ty < y1; ++ty)
        for (int tx = x0; tx < x1; ++tx) {
          const int pos = atomicAdd(&cursor[ty * tbx + tx], 1);
          if ((long long)pos < cap) {
            tile_ids[pos] = i;
            keys[pos] = dk[j];
          }
        }
    }
    return;
  }
#pragma unroll
  for (int j = 0; j < kScatItems; ++j) {
    const int x0 = bx[j] & 0xffffu, x1 = bx[j] >> 16, y0 = by[j] & 0xffffu, y1 = by[j] >> 16;
    for (int ty = y0; ty < y1; ++ty)
      for (int tx = x0; tx < x1; ++tx) atomicAdd(&s_cnt[ty * tbx + tx], 1);
  }
  __syncthreads();
  // the CTA's slots of every tile on the global cursor, claims issued back to back
#pragma unroll 4
  for (int t = threadIdx.x; t < smem_tiles; t += kGaussBlock) {
    const int cnt = s_cnt[t];
    s_off[t] = cnt ? atomicAdd(&cursor[t], cnt) : 0;
  }
  // local slots: the CTA's pairs tile by tile (exclusive scan of the counts); global slot = s_off[t] + local slot
  int n_local = 0;
  for (int t0 = 0; t0 < smem_tiles; t0 += kGaussBlock) {
    const int t = t0 + threadIdx.x;
    const int cnt = (t < smem_tiles) ? s_cnt[t] : 0;
    int total;
    const int loc = n_local + block_exclusive_scan(cnt, s_warp, total);
    if (t < smem_tiles) {
      s_off[t] -= loc;
      s_cnt[t] = loc;  // from here: the next free local slot of the tile
    }
    n_local += total;
  }
  __syncthreads();
  const bool staged = n_local <= stage_cap;  // uniform over the CTA
#pragma unroll
  for (int j = 0; j < kScatItems; ++j) {
    const int i = base + j * kGaussBlock + threadIdx.x;
    const int x0 = bx[j] & 0xffffu, x1 = bx[j] >> 16, y0 = by[j] & 0xffffu, y1 = by[j] >> 16;
    for (int ty = y0; ty < y1; ++ty)
      for (int tx = x0; tx < x1; ++tx) {
        const int t = ty * tbx + tx;
        const int e = atomicAdd(&s_cnt[t], 1);
        if (staged) {
          s_id[e] = i;
          s_key[e] = dk[j];
          s_tile[e] = (unsigned short)t;
        } else {
          const int pos = s_off[t] + e;
          if ((long long)pos < cap) {
            tile_ids[pos] = i;
            keys[pos] = dk[j];
          }
        }
      }
  }
  if (!staged) return;
  __syncthreads();
  for (int e = threadIdx.x; e < n_local; e += kGaussBlock) {
    const int pos = s_off[s_tile[e]] + e;
    if ((long long)pos < cap) {
      tile_ids[pos] = s_id[e];
      keys[pos] = s_key[e];
    }
  }
}

// ------------------------------------------------------------------ 4. per-tile sort by (depth, id)
// One CTA per tile in launch order: Sort::sort_tile on the tile's bucket (ids) and output slots (depth keys in, sorted
// ids out).
__global__ void __launch_bounds__(kSortThreads, 2) tile_sort_kernel(const int* __restrict__ order,
                                                                    const int2* __restrict__ tile_bins,
                                                                    const unsigned* __restrict__ depth_keys,
                                                                    int* bucket, int* out) {
  extern __shared__ unsigned long long s_key[];  // kSortCap keys
  __shared__ Sort::Smem s;
  const int tile = order ? order[blockIdx.x] : (int)blockIdx.x;
  const int2 range = tile_bins[tile];
  if (range.y <= range.x) return;  // uniform over the CTA
  Sort::sort_tile(range, depth_keys, bucket, out, s_key, s);
}

// Late colours (gb_bin_tiles_pack_ev with an event): tile_scatter leaves the colour quarter of the by-id records
// empty and this kernel fills it once the colours exist — colours are the only input of the binning that comes from
// the shade, so everything before it can run beside the shade forward.
__global__ void __launch_bounds__(256) rec_colors_kernel(int G, const int* __restrict__ radii,
                                                         const float* __restrict__ colors3,
                                                         const float* __restrict__ depths, float4* __restrict__ rec_by_id) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G || radii[g] <= 0) return;
  rec_by_id[3 * (size_t)g + 2] = make_float4(colors3[3 * (size_t)g], colors3[3 * (size_t)g + 1],
                                             colors3[3 * (size_t)g + 2], depths[g]);
}

// ------------------------------------------------------------------ 5. sorted records (packed callers)
__global__ void __launch_bounds__(256) gather_records_kernel(long long cap, const int* __restrict__ n_dev,
                                                             const int* __restrict__ gids_sorted,
                                                             const float4* __restrict__ rec_by_id,
                                                             float4* __restrict__ rec) {
  const long long n = min((long long)*n_dev, cap);
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // float4 index: record j / 3, part j % 3
  if (j >= 3 * n) return;
  const long long i = j / 3;
  const int part = (int)(j - 3 * i);
  rec[j] = gb::ld_nc_f4(rec_by_id + 3 * (size_t)gids_sorted[i] + part);
}

struct Layout {
  size_t counts, sync, zero_bytes, cursor, rects, rec_by_id, bucket, total;
};
inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
inline Layout make_layout(int G, int T, int64_t cap) {
  const int g1 = G > 0 ? G : 1;
  Layout l;
  size_t o = 0;
  l.counts = o; o += align256((size_t)T * 4);
  l.sync = o;   o += 256;                 // [0]: the intersection count when the caller passes no n_out
  l.zero_bytes = o;                       // [counts | sync] are zeroed with one memset per call
  l.cursor = o; o += align256((size_t)T * 4);
  l.rects = o;  o += align256((size_t)g1 * 16);   // int4 tile rectangle per Gaussian
  l.rec_by_id = o; o += align256((size_t)g1 * 48);
  l.bucket = o; o += align256((size_t)(cap > 0 ? cap : 1) * 4);
  l.total = o;
  return l;
}

// SMs of the current device, queried once per device
int num_sms() {
  static int s_sms[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (dev < 0 || dev >= 64) return 0;
  if (!s_sms[dev] && cudaDeviceGetAttribute(&s_sms[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
  return s_sms[dev];
}

// opt in to a dynamic shared-memory window above 48 KB, once per device and kernel
template <typename K>
int opt_in_smem(K kernel, size_t bytes, bool* done) {
  int dev = 0;
  GB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !done[dev]) {
    GB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    if (dev >= 0 && dev < 64) done[dev] = true;
  }
  return 0;
}

}  // namespace

// There is one formulation of the binning; these report it as mode 0 and accept (and ignore) any setting, so callers
// that select or label modes keep working.
GB_API int gb_get_tile_sort_mode(void) { return 0; }
GB_API void gb_set_tile_sort_mode(int mode) { (void)mode; }
GB_API int gb_get_rank_sort_mode(void) { return 0; }
GB_API void gb_set_rank_sort_mode(int mode) { (void)mode; }

// 1 when gb_bin_tiles_pack supports G Gaussians (1 <= G <= kMaxGaussians)
GB_API int gb_bin_tiles_supported(int G) { return G >= 1 && G <= kMaxGaussians; }

GB_API size_t gb_bin_tiles_workspace_bytes(int G, int num_tiles, int64_t cap) {
  return make_layout(G, num_tiles, cap).total;
}

// Binning + record packing of the fused render (see the header of this file).  Outputs: tile_bins [T,2],
// tile_order [T] (longest list first; with tile_sched = 1 an SM-affine schedule of gb_tile_schedule_ints(T)
// int32, see gb_tile_schedule), gids_sorted [cap], records [cap,12]; n_out (device int32, may be
// null) receives the true intersection count, *overflow is set to 1 when it exceeds `cap` (the excess is
// dropped).  Never allocates, never synchronises; capturable in a CUDA graph.
GB_API int gb_bin_tiles_pack(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                             const float* colors3, const float* opacity, const float* compensation, int img_h,
                             int img_w, int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order,
                             int tile_sched, int32_t* gids_sorted, float* records, int32_t* n_out, int32_t* overflow,
                             void* workspace, void* stream) {
  return gb_bin_tiles_pack_ev(G, xys, depths, radii, conics, colors3, opacity, compensation, img_h, img_w, block_width, cap,
                              tile_bins, tile_order, tile_sched, gids_sorted, records, n_out, overflow, workspace, nullptr,
                              stream);
}

// Same, with the colours allowed to arrive late: `colors_ready` (a cudaEvent_t recorded on the stream that produces
// colors3, or NULL) is waited for on `stream` just before the small kernel that fills the colour quarter of the by-id
// records after the per-tile sort, so counts, buckets and the per-tile sort overlap the caller's shade.
static int bin_tiles_impl(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                          const float* colors3, const float* opacity, const float* compensation, int img_h, int img_w,
                          int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order, int tile_sched,
                          int32_t* gids_sorted, float* records, int32_t* n_out, int32_t* overflow, void* workspace,
                          void* colors_ready, void* stream, int32_t* ext_ids, float* ext_rec, int32_t* ext_identity,
                          int32_t* ext_bucket);

GB_API int gb_bin_tiles_pack_ev(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                                const float* colors3, const float* opacity, const float* compensation, int img_h,
                                int img_w, int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order,
                                int tile_sched, int32_t* gids_sorted, float* records, int32_t* n_out, int32_t* overflow,
                                void* workspace, void* colors_ready, void* stream) {
  return bin_tiles_impl(G, xys, depths, radii, conics, colors3, opacity, compensation, img_h, img_w, block_width, cap,
                        tile_bins, tile_order, tile_sched, gids_sorted, records, n_out, overflow, workspace, colors_ready,
                        stream, nullptr, nullptr, nullptr, nullptr);
}

// Binning WITHOUT the sorted-record gather, for the blend kernels that stage records from the per-Gaussian table
// (gb_rasterize_ranked_*): ranks_sorted [cap] receives, per tile, the sorted Gaussian ids; rec_by_rank [G,12] the
// 48-byte record of each visible Gaussian at its id; rank_to_gid [G] the identity.  All three are the CALLER's arrays
// (they must outlive the backward; the shared workspace does not).  Everything else as gb_bin_tiles_pack_ev.  Saves the
// 52 MB write + read of the sorted records and holds 14.4 + 4 I bytes per view for the backward instead of 52 I.
GB_API int gb_bin_tiles_ranked(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                               const float* colors3, const float* opacity, const float* compensation, int img_h,
                               int img_w, int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order,
                               int tile_sched, int32_t* ranks_sorted, float* rec_by_rank, int32_t* rank_to_gid,
                               int32_t* n_out, int32_t* overflow, void* workspace, void* colors_ready, void* stream) {
  if (!ranks_sorted || !rec_by_rank || !rank_to_gid) return (int)cudaErrorInvalidValue;
  return bin_tiles_impl(G, xys, depths, radii, conics, colors3, opacity, compensation, img_h, img_w, block_width, cap,
                        tile_bins, tile_order, tile_sched, nullptr, nullptr, n_out, overflow, workspace, colors_ready, stream,
                        ranks_sorted, rec_by_rank, rank_to_gid, nullptr);
}

// gb_bin_tiles_ranked up to the bucket scatter, for the forward that sorts each tile itself
// (gb_rasterize_ranked_fwd_sort_lists): every tile's ids in arbitrary order in bucket [cap] and their 32-bit depth keys
// at the same slots of ranks_keys [cap], which that forward overwrites with the sorted ids.  tile_bins, tile_order,
// rec_by_rank, rank_to_gid, n_out and overflow as gb_bin_tiles_ranked.  One launch fewer than gb_bin_tiles_ranked.
GB_API int gb_bin_tiles_buckets(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                                const float* colors3, const float* opacity, const float* compensation, int img_h,
                                int img_w, int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order,
                                int32_t* ranks_keys, int32_t* bucket, float* rec_by_rank, int32_t* rank_to_gid,
                                int32_t* n_out, int32_t* overflow, void* workspace, void* colors_ready, void* stream) {
  if (!ranks_keys || !bucket || !rec_by_rank || !rank_to_gid) return (int)cudaErrorInvalidValue;
  return bin_tiles_impl(G, xys, depths, radii, conics, colors3, opacity, compensation, img_h, img_w, block_width, cap,
                        tile_bins, tile_order, 0, nullptr, nullptr, n_out, overflow, workspace, colors_ready, stream,
                        ranks_keys, rec_by_rank, rank_to_gid, bucket);
}

static int bin_tiles_impl(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                          const float* colors3, const float* opacity, const float* compensation, int img_h, int img_w,
                          int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order, int tile_sched,
                          int32_t* gids_sorted, float* records, int32_t* n_out, int32_t* overflow, void* workspace,
                          void* colors_ready, void* stream, int32_t* ext_ids, float* ext_rec, int32_t* ext_identity,
                          int32_t* ext_bucket) {
  if (!gb_bin_tiles_supported(G) || block_width < 1 || cap < 0) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const int tbx = gb::cdiv(img_w, block_width), tby = gb::cdiv(img_h, block_width);
  const int T = tbx * tby;
  if (T < 1 || tbx > 65535 || tby > 65535) return (int)cudaErrorInvalidValue;
  const Layout l = make_layout(G, T, cap);
  char* ws = (char*)workspace;
  int* counts = (int*)(ws + l.counts);
  int* cursor = (int*)(ws + l.cursor);
  int* bucket = ext_bucket ? ext_bucket : (int*)(ws + l.bucket);
  int4* rects = (int4*)(ws + l.rects);
  const bool ranked = ext_ids != nullptr;  // outputs for the blend that stages records by id: no sorted-record gather
  float4* rec_by_id = ranked ? (float4*)ext_rec : (float4*)(ws + l.rec_by_id);
  int* ids_sorted = ranked ? ext_ids : gids_sorted;
  const int items = count_items(G);
  const int smem_tiles = (T <= kMaxSmemTiles) ? T : 0;
  const int stage_cap = scatter_stage_cap(smem_tiles);
  const size_t scat_smem = scatter_smem_bytes(smem_tiles);
  static bool s_opt_c2[64] = {}, s_opt_c4[64] = {}, s_opt_scat[64] = {}, s_opt_sort[64] = {};
  if ((size_t)smem_tiles * 4 > 40 * 1024) {
    constexpr size_t kCountSmem = (size_t)kMaxSmemTiles * 4;
    const int e = (items == 2) ? opt_in_smem(tile_count_kernel<2>, kCountSmem, s_opt_c2)
                               : opt_in_smem(tile_count_kernel<4>, kCountSmem, s_opt_c4);
    if (e) return e;
  }
  {  // the largest window any grid asks for: the tile arrays of kMaxSmemTiles, or those of kStageMaxTiles + staging
    const size_t a = scatter_smem_bytes(kMaxSmemTiles), b = scatter_smem_bytes(kStageMaxTiles);
    const int e = opt_in_smem(tile_scatter_kernel, a > b ? a : b, s_opt_scat);
    if (e) return e;
  }
  const size_t sort_smem = (size_t)kSortCap * 8;
  {
    const int e = opt_in_smem(tile_sort_kernel, sort_smem, s_opt_sort);
    if (e) return e;
  }

  GB_CUDA(cudaMemsetAsync(ws, 0, l.zero_bytes, s));
  const int ctas = gb::cdiv(G, kGaussBlock * items);
  if (items == 2)
    tile_count_kernel<2><<<ctas, kGaussBlock, (size_t)smem_tiles * 4, s>>>(G, (const float2*)xys, radii, tbx, tby,
                                                                          block_width, smem_tiles, counts, rects, ext_identity);
  else
    tile_count_kernel<4><<<ctas, kGaussBlock, (size_t)smem_tiles * 4, s>>>(G, (const float2*)xys, radii, tbx, tby,
                                                                          block_width, smem_tiles, counts, rects, ext_identity);
  int* n_total = n_out ? n_out : (int*)(ws + l.sync);  // the record gather below needs the count on the device
  tile_scan_kernel<<<1, 1024, 0, s>>>(T, (long long)cap, counts, (int2*)tile_bins, cursor, n_total, overflow);
  gb::count_launches(2);
  GB_CHECK_LAUNCH();
  const int e = tile_sched ? gb_tile_schedule(T, tile_bins, tile_order, stream)
                           : gb_tile_order(T, tile_bins, tile_order, stream);
  if (e) return e;
  const bool late = colors_ready != nullptr;  // the colour quarter of the by-id records is filled after the tile sort
  const int per_cta = scatter_per_cta(G, num_sms());
  tile_scatter_kernel<<<gb::cdiv(G, per_cta), kGaussBlock, scat_smem, s>>>(
      G, rects, (const float2*)xys, conics, late ? nullptr : colors3, depths, opacity, compensation, tbx, (long long)cap,
      per_cta, smem_tiles, stage_cap, cursor, bucket, (unsigned*)ids_sorted, rec_by_id);
  gb::count_launches(1);
  if (!ext_bucket) {  // else the caller's forward sorts each bucket
    tile_sort_kernel<<<T, kSortThreads, sort_smem, s>>>(tile_order, (const int2*)tile_bins, (const unsigned*)depths, bucket,
                                                        ids_sorted);
    gb::count_launches(1);
  }
  if (late) {
    GB_CUDA(cudaStreamWaitEvent(s, (cudaEvent_t)colors_ready, 0));
    rec_colors_kernel<<<gb::cdiv(G, 256), 256, 0, s>>>(G, radii, colors3, depths, rec_by_id);
    gb::count_launches(1);
  }
  if (cap > 0 && !ranked) {
    gather_records_kernel<<<(unsigned)gb::cdiv64(3 * cap, 256), 256, 0, s>>>((long long)cap, n_total, gids_sorted,
                                                                           rec_by_id, (float4*)records);
    gb::count_launches(1);
  }
  GB_CHECK_LAUNCH();
  return 0;
}
