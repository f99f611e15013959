// goliath_b200/csrc/splat_bin.cu — tile binning for the splat rasteriser (sm_90a):
//   inclusive int32 scan of num_tiles_hit -> (tile<<32 | depth-bits) intersection keys ->
//   stable LSD radix sort of (u64 key, i32 Gaussian id) -> per-tile [first,last) bin edges.
//
// Replaces (third-party, absent from the reference tree) gsplat 0.1.11's
// compute_cumulative_intersects / map_gaussian_to_intersects / torch.sort / get_tile_bin_edges, i.e. the
// work done inside rasterize_gaussians at ca_code/utils/render_gsplat.py:65-78,90-104.
// All of it is integer/byte work and a BIT-EXACT contract (SURVEY.md Appendix A "Binning"): the sort is
// stable, so equal keys keep emission order == ascending Gaussian id, exactly as the oracle.
//
// Radix sort design: 8-bit digits, only the significant low `key_bits` are sorted (32 depth bits +
// ceil(log2(#tiles))), and passes whose digit is identical for every key are skipped (typical for the
// top depth byte).  Each pass = per-CTA digit histogram -> single-CTA exclusive scan over the
// (digit-major) histogram table -> stable scatter with warp match-any ranking.  Everything stays in
// the 50 MB L2 at the sizes of this path (1 M keys = 12 MB).
#include "common.cuh"

namespace {

// ------------------------------------------------------------------ inclusive scan (int32)
constexpr int kScanBlock = 256;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanBlock * kScanItems;  // 2048

__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int& total) {
  // returns exclusive prefix of v over the CTA; total = CTA sum. kScanBlock threads.
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = (lane < (int)(blockDim.x >> 5)) ? s_warp[lane] : 0;
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    s_warp[lane] = winc - w;                 // exclusive warp offsets
    if (lane == 31) s_warp[32] = winc;       // total
  }
  __syncthreads();
  total = s_warp[32];
  const int r = s_warp[warp] + inc - v;
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(kScanBlock) scan_tile_sums_kernel(int n, const int* __restrict__ in,
                                                                     int* __restrict__ tile_sums) {
  __shared__ int s_warp[33];
  const int base = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
  int s = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) s += (base + k < n) ? in[base + k] : 0;
  int total;
  block_exclusive_scan(s, s_warp, total);
  if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

// single CTA: exclusive scan of tile_sums in place (any length)
__global__ void __launch_bounds__(kScanBlock) scan_small_kernel(int n, int* __restrict__ data) {
  __shared__ int s_warp[33];
  int carry = 0;
  for (int base = 0; base < n; base += kScanBlock) {
    const int i = base + threadIdx.x;
    const int v = (i < n) ? data[i] : 0;
    int total;
    const int ex = block_exclusive_scan(v, s_warp, total);
    if (i < n) data[i] = carry + ex;
    carry += total;
  }
}

__global__ void __launch_bounds__(kScanBlock) scan_apply_kernel(int n, const int* __restrict__ in,
                                                                 const int* __restrict__ tile_offsets,
                                                                 int* __restrict__ out) {
  __shared__ int s_warp[33];
  const int base = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
  int v[kScanItems];
  int s = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) { v[k] = (base + k < n) ? in[base + k] : 0; s += v[k]; }
  int total;
  int run = block_exclusive_scan(s, s_warp, total) + tile_offsets[blockIdx.x];
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    run += v[k];
    if (base + k < n) out[base + k] = run;
  }
}

// ------------------------------------------------------------------ intersection keys
__device__ __forceinline__ void tile_bbox(float cx, float cy, float radius, int tbx, int tby, int bw, int& x0,
                                          int& y0, int& x1, int& y1) {
  const float fb = (float)bw;
  const float tcx = __fdiv_rn(cx, fb), tcy = __fdiv_rn(cy, fb), tr = __fdiv_rn(radius, fb);
  x0 = min(max(0, __float2int_rz(__fsub_rn(tcx, tr))), tbx);
  x1 = min(max(0, __float2int_rz(__fadd_rn(__fadd_rn(tcx, tr), 1.f))), tbx);
  y0 = min(max(0, __float2int_rz(__fsub_rn(tcy, tr))), tby);
  y1 = min(max(0, __float2int_rz(__fadd_rn(__fadd_rn(tcy, tr), 1.f))), tby);
}

__global__ void __launch_bounds__(256) map_to_intersects_kernel(int G, const float2* __restrict__ xys,
                                                                const float* __restrict__ depths,
                                                                const int* __restrict__ radii,
                                                                const int* __restrict__ cum_tiles_hit, int tbx,
                                                                int tby, int block_width,
                                                                long long* __restrict__ isect_ids,
                                                                int* __restrict__ gaussian_ids, long long cap) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  const int r = radii[i];
  if (r <= 0) return;
  int x0, y0, x1, y1;
  const float2 c = xys[i];
  tile_bbox(c.x, c.y, (float)r, tbx, tby, block_width, x0, y0, x1, y1);
  int cur = (i == 0) ? 0 : cum_tiles_hit[i - 1];
  const long long depth_id = (long long)__float_as_int(depths[i]);
  for (int ty = y0; ty < y1; ++ty)
    for (int tx = x0; tx < x1; ++tx) {
      if (cur >= cap) return;  // capacity of the sync-free path (flagged by the bin-edges kernel)
      const long long tile_id = (long long)ty * tbx + tx;
      isect_ids[cur] = (tile_id << 32) | depth_id;
      gaussian_ids[cur] = i;
      ++cur;
    }
}

// The element count may live on the device (sync-free path): n = min(*n_dev, capacity) when n_dev != null.
__device__ __forceinline__ long long resolve_n(long long n_cap, const int* __restrict__ n_dev) {
  return n_dev ? min((long long)*n_dev, n_cap) : n_cap;
}

// ------------------------------------------------------------------ radix sort (u64 keys, i32 values)
constexpr int kSortBlock = 256;                      // 8 warps
constexpr int kSortItems = 16;                       // keys per thread
constexpr int kSortTile = kSortBlock * kSortItems;   // 4096 keys per CTA
constexpr int kRadix = 256;

// warp w of a CTA owns the contiguous chunk [tile_base + w*512, +512); lane-strided inside the chunk so
// that "earlier in memory" == (smaller item index j, then smaller lane) — needed for stability.
__global__ void __launch_bounds__(kSortBlock) sort_hist_kernel(long long n_cap, const int* __restrict__ n_dev,
                                                               const unsigned long long* __restrict__ keys,
                                                               int shift, int num_tiles,
                                                               unsigned* __restrict__ hist /* [256][num_tiles] */) {
  __shared__ unsigned s_hist[kRadix];
  const long long n = resolve_n(n_cap, n_dev);
  s_hist[threadIdx.x] = 0;
  __syncthreads();
  const long long base = (long long)blockIdx.x * kSortTile;
#pragma unroll 4
  for (int j = 0; j < kSortItems; ++j) {
    const long long i = base + (long long)j * kSortBlock + threadIdx.x;
    if (i < n) atomicAdd(&s_hist[(unsigned)(keys[i] >> shift) & 0xffu], 1u);
  }
  __syncthreads();
  hist[(size_t)threadIdx.x * num_tiles + blockIdx.x] = s_hist[threadIdx.x];
}

// one CTA per digit: exclusive scan of that digit's per-tile counts (in place) + the digit's total.
// 256 small independent scans run in parallel instead of one serial sweep over the 256*num_tiles table.
__global__ void __launch_bounds__(kScanBlock) sort_scan_kernel(unsigned* __restrict__ hist, int num_tiles,
                                                               unsigned* __restrict__ totals) {
  __shared__ int s_warp[33];
  unsigned* row = hist + (size_t)blockIdx.x * num_tiles;
  int carry = 0;
  for (int base = 0; base < num_tiles; base += kScanBlock) {
    const int i = base + threadIdx.x;
    const int v = (i < num_tiles) ? (int)row[i] : 0;
    int total;
    const int ex = block_exclusive_scan(v, s_warp, total);
    if (i < num_tiles) row[i] = (unsigned)(carry + ex);
    carry += total;
  }
  if (threadIdx.x == 0) totals[blockIdx.x] = (unsigned)carry;
}

__global__ void __launch_bounds__(kSortBlock) sort_scatter_kernel(
    long long n_cap, const int* __restrict__ n_dev, const unsigned long long* __restrict__ keys_in, const int* __restrict__ vals_in,
    unsigned long long* __restrict__ keys_out, int* __restrict__ vals_out, int shift, int num_tiles,
    const unsigned* __restrict__ offsets /* per-digit scanned [256][num_tiles] */,
    const unsigned* __restrict__ totals /* [256] keys per digit */) {
  constexpr int kWarps = kSortBlock / 32;
  __shared__ unsigned s_whist[kWarps][kRadix];  // per-warp digit counts -> per-warp running offsets (8 KB)
  __shared__ int s_scan[33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n = resolve_n(n_cap, n_dev);
  // digit bases = exclusive scan of the 256 digit totals (every CTA recomputes it: 256 loads from L2);
  // a digit holding every key makes the pass a no-op (typical for the top depth byte)
  const unsigned my_total = totals[threadIdx.x];
  const bool copy_only = __syncthreads_or(my_total == (unsigned)n) != 0;
  int tot_unused;
  const unsigned digit_base = (unsigned)block_exclusive_scan((int)my_total, s_scan, tot_unused);
  const long long tile_base = (long long)blockIdx.x * kSortTile;
  const long long warp_base = tile_base + (long long)warp * (32 * kSortItems);

  unsigned long long k[kSortItems];
  int v[kSortItems];
#pragma unroll
  for (int j = 0; j < kSortItems; ++j) {
    const long long i = warp_base + j * 32 + lane;
    k[j] = (i < n) ? keys_in[i] : ~0ull;
    v[j] = (i < n) ? vals_in[i] : 0;
  }
  if (copy_only) {  // digit identical for all keys: order is unchanged, just move the data
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
      const long long i = warp_base + j * 32 + lane;
      if (i < n) { keys_out[i] = k[j]; vals_out[i] = v[j]; }
    }
    return;
  }
  for (int d = lane; d < kRadix; d += 32) s_whist[warp][d] = 0;
  __syncwarp();
  // pass 1: per-warp digit counts
  unsigned rank[kSortItems];  // rank among equal digits inside this warp's chunk
#pragma unroll
  for (int j = 0; j < kSortItems; ++j) {
    const long long i = warp_base + j * 32 + lane;
    const bool valid = i < n;
    const unsigned dgt = (unsigned)(k[j] >> shift) & 0xffu;
    const unsigned peers = __match_any_sync(0xffffffffu, valid ? dgt : 0x100u + 0u);
    const unsigned lower = peers & ((1u << lane) - 1u);
    unsigned prev = 0;
    if (valid) prev = s_whist[warp][dgt];
    __syncwarp();
    rank[j] = prev + __popc(lower);
    if (valid && lower == 0u) s_whist[warp][dgt] = prev + __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  // exclusive scan across warps per digit + global base for (digit, tile)
  {
    const int d = threadIdx.x;  // 256 threads == 256 digits
    unsigned run = digit_base + offsets[(size_t)d * num_tiles + blockIdx.x];
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const unsigned c = s_whist[w][d];
      s_whist[w][d] = run;
      run += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < kSortItems; ++j) {
    const long long i = warp_base + j * 32 + lane;
    if (i < n) {
      const unsigned dgt = (unsigned)(k[j] >> shift) & 0xffu;
      const unsigned dst = s_whist[warp][dgt] + rank[j];
      keys_out[dst] = k[j];
      vals_out[dst] = v[j];
    }
  }
}

// ------------------------------------------------------------------ tile bin edges
__global__ void __launch_bounds__(256) tile_bin_edges_kernel(long long n_cap, const int* __restrict__ n_dev,
                                                             const long long* __restrict__ isect_sorted,
                                                             int2* __restrict__ tile_bins, int* __restrict__ overflow) {
  const long long n = resolve_n(n_cap, n_dev);
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 && overflow && n_dev && (long long)*n_dev > n_cap) *overflow = 1;  // capacity exceeded: caller must re-run
  if (i >= n) return;
  const int cur = (int)(isect_sorted[i] >> 32);
  if (i == 0) tile_bins[cur].x = 0;
  if (i == n - 1) tile_bins[cur].y = (int)n;
  if (i == 0) return;
  const int prev = (int)(isect_sorted[i - 1] >> 32);
  if (prev != cur) {
    tile_bins[prev].y = (int)i;
    tile_bins[cur].x = (int)i;
  }
}

}  // namespace

// workspace (bytes) for gb_cumsum_i32 over n elements
GB_API size_t gb_cumsum_workspace_bytes(int n) { return (size_t)(gb::cdiv(n > 0 ? n : 1, kScanTile) + 1) * sizeof(int); }

// inclusive scan, int32 (gsplat compute_cumulative_intersects: torch.cumsum(..., dtype=int32))
GB_API int gb_cumsum_i32(int n, const int32_t* in, int32_t* out, void* workspace, void* stream) {
  if (n <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int tiles = gb::cdiv(n, kScanTile);
  int* tile_sums = (int*)workspace;
  GB_CUDA(gb::launch<scan_tile_sums_kernel>(tiles, kScanBlock, 0, s, n, in, tile_sums));
  GB_CUDA(gb::launch<scan_small_kernel>(1, kScanBlock, 0, s, tiles, tile_sums));
  return gb::launch<scan_apply_kernel>(tiles, kScanBlock, 0, s, n, in, tile_sums, out);
}

// replaces gsplat._C.map_gaussian_to_intersects
static int map_impl(int G, const float* xys, const float* depths, const int32_t* radii, const int32_t* cum_tiles_hit,
                    int img_h, int img_w, int block_width, int64_t* isect_ids, int32_t* gaussian_ids, long long cap,
                    void* stream) {
  if (G <= 0) return 0;
  const int tbx = gb::cdiv(img_w, block_width), tby = gb::cdiv(img_h, block_width);
  return gb::launch<map_to_intersects_kernel>(gb::cdiv(G, 256), 256, 0, (cudaStream_t)stream,
      G, (const float2*)xys, depths, radii, cum_tiles_hit, tbx, tby, block_width, (long long*)isect_ids, gaussian_ids, cap);
}

GB_API int gb_map_gaussian_to_intersects(int G, const float* xys, const float* depths, const int32_t* radii,
                                         const int32_t* cum_tiles_hit, int img_h, int img_w, int block_width,
                                         int64_t* isect_ids, int32_t* gaussian_ids, void* stream) {
  return map_impl(G, xys, depths, radii, cum_tiles_hit, img_h, img_w, block_width, isect_ids, gaussian_ids,
                  0x7fffffffffffffffLL, stream);
}
// sync-free variant: the buffers hold `cap` intersections; writes beyond are dropped (and flagged by
// gb_get_tile_bin_edges_dn), the true count stays on the device (last element of cum_tiles_hit)
GB_API int gb_map_gaussian_to_intersects_dn(int G, const float* xys, const float* depths, const int32_t* radii,
                                            const int32_t* cum_tiles_hit, int img_h, int img_w, int block_width,
                                            int64_t cap, int64_t* isect_ids, int32_t* gaussian_ids, void* stream) {
  return map_impl(G, xys, depths, radii, cum_tiles_hit, img_h, img_w, block_width, isect_ids, gaussian_ids, cap, stream);
}

// workspace for gb_sort_intersects: ping-pong key/value buffers + histogram table + flag
GB_API size_t gb_sort_workspace_bytes(int64_t n) {
  const int64_t nn = n > 0 ? n : 1;
  const int64_t tiles = gb::cdiv64(nn, kSortTile);
  size_t b = 0;
  b += (size_t)nn * 8;                 // alt keys
  b += (size_t)nn * 4;                 // alt vals
  b = (b + 255) & ~(size_t)255;
  b += (size_t)kRadix * tiles * 4;     // histogram table
  b += kRadix * 4;                     // digit totals
  return b;
}

// replaces torch.sort(isect_ids) + gather(gaussian_ids) inside gsplat bin_and_sort_gaussians.
// Stable ascending sort on the low `key_bits` bits (keys are non-negative: depth > 0).
static int sort_impl(int64_t n, const int* n_dev, const int64_t* isect_ids, const int32_t* gaussian_ids,
                     int64_t* isect_sorted, int32_t* gids_sorted, int key_bits, void* workspace, void* stream) {
  if (n <= 0) return 0;
  if (key_bits < 1 || key_bits > 64) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const int tiles = (int)gb::cdiv64(n, kSortTile);
  char* ws = (char*)workspace;
  unsigned long long* alt_k = (unsigned long long*)ws;
  int* alt_v = (int*)(ws + (size_t)n * 8);
  size_t off = ((size_t)n * 12 + 255) & ~(size_t)255;
  unsigned* hist = (unsigned*)(ws + off);
  unsigned* totals = (unsigned*)(ws + off + (size_t)kRadix * tiles * 4);

  const int passes = (key_bits + 7) / 8;
  // ping-pong so that the LAST pass lands in the caller's output buffers
  const unsigned long long* src_k = (const unsigned long long*)isect_ids;
  const int* src_v = gaussian_ids;
  for (int p = 0; p < passes; ++p) {
    const bool to_out = ((passes - 1 - p) % 2) == 0;
    unsigned long long* dst_k = to_out ? (unsigned long long*)isect_sorted : alt_k;
    int* dst_v = to_out ? gids_sorted : alt_v;
    const int shift = 8 * p;
    GB_CUDA(gb::launch<sort_hist_kernel>(tiles, kSortBlock, 0, s, n, n_dev, src_k, shift, tiles, hist));
    GB_CUDA(gb::launch<sort_scan_kernel>(kRadix, kScanBlock, 0, s, hist, tiles, totals));
    GB_CUDA(gb::launch<sort_scatter_kernel>(tiles, kSortBlock, 0, s, n, n_dev, src_k, src_v, dst_k, dst_v, shift, tiles,
                                            hist, totals));
    src_k = dst_k;
    src_v = dst_v;
  }
  return 0;
}

GB_API int gb_sort_intersects(int64_t n, const int64_t* isect_ids, const int32_t* gaussian_ids,
                              int64_t* isect_sorted, int32_t* gids_sorted, int key_bits, void* workspace,
                              void* stream) {
  return sort_impl(n, nullptr, isect_ids, gaussian_ids, isect_sorted, gids_sorted, key_bits, workspace, stream);
}
// sync-free variant: `cap` sizes the launch and the workspace, the element count is read from *n_dev on the device
GB_API int gb_sort_intersects_dn(int64_t cap, const int32_t* n_dev, const int64_t* isect_ids,
                                 const int32_t* gaussian_ids, int64_t* isect_sorted, int32_t* gids_sorted, int key_bits,
                                 void* workspace, void* stream) {
  return sort_impl(cap, n_dev, isect_ids, gaussian_ids, isect_sorted, gids_sorted, key_bits, workspace, stream);
}

static int edges_impl(int64_t n, const int* n_dev, const int64_t* isect_sorted, int32_t* tile_bins, int* overflow,
                      void* stream) {
  if (n <= 0) return 0;
  return gb::launch<tile_bin_edges_kernel>((unsigned)gb::cdiv64(n, 256), 256, 0, (cudaStream_t)stream,
      n, n_dev, (const long long*)isect_sorted, (int2*)tile_bins, overflow);
}

// replaces gsplat._C.get_tile_bin_edges; tile_bins [T,2] int32 must be zeroed by the caller
GB_API int gb_get_tile_bin_edges(int64_t n, const int64_t* isect_sorted, int32_t* tile_bins, void* stream) {
  return edges_impl(n, nullptr, isect_sorted, tile_bins, nullptr, stream);
}
// sync-free variant; *overflow (int32, device) is set to 1 when the true count exceeds `cap`
GB_API int gb_get_tile_bin_edges_dn(int64_t cap, const int32_t* n_dev, const int64_t* isect_sorted, int32_t* tile_bins,
                                    int32_t* overflow, void* stream) {
  return edges_impl(cap, n_dev, isect_sorted, tile_bins, overflow, stream);
}
