// goliath_b200/csrc/splat_tile_sort.cuh — the per-tile (depth, id) sort of the tile binning, as a CTA-wide device
// function.  Two kernels run it: tile_sort_kernel (csrc/splat_bin_tiles.cu, 512 threads, one CTA per tile) and the
// sort-then-blend forward (csrc/splat_blend_mom.cu, the forward's 288 threads, before the tile is blended).  See the
// header of csrc/splat_bin_tiles.cu for the algorithm.
//
// TileSort<kThreads, kItems> sorts up to kThreads * kItems entries in registers + shared memory and longer buckets
// chunk by chunk through global memory.  Every thread of the CTA calls sort_tile; it returns after a CTA barrier.
#pragma once

#include "common.cuh"

namespace gbsort {

constexpr int kDigitBits = 9;
constexpr int kDigits = 1 << kDigitBits;
// Longest run of equal depth keys that one thread sorts by id in place after the depth passes.  The bench head's
// tiles tie in ~70 % of tiles but in runs of at most 3 entries; a tile with a longer run re-sorts on the full key.
constexpr int kTieRun = 16;

// exclusive prefix of v over the CTA (any multiple of 32 threads up to 1024); total = CTA sum
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int& total) {
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
    s_warp[lane] = winc - w;
    if (lane == 31) s_warp[32] = winc;
  }
  __syncthreads();
  total = s_warp[32];
  const int r = s_warp[warp] + inc - v;
  __syncthreads();
  return r;
}

__device__ __forceinline__ int bits_of(unsigned span) { return span ? 32 - __clz((int)span) : 0; }

template <int kThreads, int kItems>
struct TileSort {
  static constexpr int kWarps = kThreads / 32;
  static constexpr int kCap = kThreads * kItems;                     // entries sorted in shared memory
  static constexpr int kDpt = (kDigits + kThreads - 1) / kThreads;   // digits per thread in the scans
  static constexpr int kRunWords = (kItems + 11) / 12;               // tie-run lengths, 5 bits per item, 12 per word
  static_assert(kThreads % 32 == 0 && kThreads <= 1024, "whole warps");
  static_assert(kTieRun < 32, "run lengths are packed 5 bits per item");

  struct Smem {
    unsigned short whist[kWarps][kDigits];  // per-warp digit counts, then their exclusive prefix over the warps
    int base[kDigits];                      // scatter base of each digit
    int run[kDigits];                       // chunked path: running base of each digit over the chunks
    int warp[33];
    unsigned red[4];                        // min / max of the depth keys and of the ids
  };
  static constexpr size_t kKeyBytes = (size_t)kCap * 8;  // the caller's s_key buffer

  // With ipt items per thread (ipt <= kItems), entry e of a chunk is held by warp e / (32 ipt), item (e / 32) % ipt,
  // lane e % 32: "earlier in the chunk" == (smaller warp, then smaller item, then smaller lane), which the per-warp
  // ranking below preserves.
  static __device__ __forceinline__ int entry_of(int j, int ipt) {
    return (threadIdx.x >> 5) * (32 * ipt) + j * 32 + (threadIdx.x & 31);
  }

  // item j of this thread is one of the m entries of the chunk
  static __device__ __forceinline__ bool holds(int j, int ipt, int m) { return j < ipt && entry_of(j, ipt) < m; }

  // One stable counting pass on digit (key >> shift) & (kDigits - 1) over the m valid entries of a chunk held in
  // registers, ipt per thread: dst[j] = destination of item j.  whole: the chunk is the whole list (bases = exclusive
  // scan of this chunk's counts); else the bases come from s.run, which is advanced by this chunk's counts.
  static __device__ __forceinline__ void radix_positions(const unsigned long long (&k)[kItems], int m, int ipt,
                                                         int shift, bool whole, Smem& s, int (&dst)[kItems]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // items held by this warp and by this thread: item j is valid iff j < mine
    const int wbase = warp * (32 * ipt);
    const int ours = min(ipt, max(0, (m - wbase + 31) >> 5)), mine = min(ipt, max(0, (m - wbase - lane + 31) >> 5));
    for (int d = lane; d < kDigits; d += 32) s.whist[warp][d] = 0;
    __syncwarp();
#pragma unroll
    for (int j = 0; j < kItems; ++j) {  // dst[j] = rank among the equal digits of this warp's earlier entries
      dst[j] = 0;
      if (j >= ours) continue;  // warp-uniform
      const bool valid = j < mine;
      const unsigned dgt = (unsigned)(k[j] >> shift) & (kDigits - 1);
      // lanes holding the same digit: one ballot per digit bit (__match_any_sync serialises over the ~30 distinct
      // digits a warp holds)
      unsigned peers = __ballot_sync(0xffffffffu, valid);
#pragma unroll
      for (int b = 0; b < kDigitBits; ++b) {
        const unsigned bal = __ballot_sync(0xffffffffu, (dgt >> b) & 1u);
        peers &= ((dgt >> b) & 1u) ? bal : ~bal;
      }
      const unsigned lower = peers & ((1u << lane) - 1u);
      unsigned prev = 0;
      if (valid) prev = s.whist[warp][dgt];
      __syncwarp();
      dst[j] = (int)(prev + __popc(lower));
      if (valid && lower == 0u) s.whist[warp][dgt] = (unsigned short)(prev + __popc(peers));
      __syncwarp();
    }
    __syncthreads();
    {
      // thread t owns digits [t kDpt, (t + 1) kDpt): their counts summed over the warps, then scanned over the CTA
      int run[kDpt], sum = 0;
#pragma unroll
      for (int i = 0; i < kDpt; ++i) {
        const int d = (int)threadIdx.x * kDpt + i;
        run[i] = 0;
        if (d >= kDigits) continue;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
          const int c = s.whist[w][d];
          s.whist[w][d] = (unsigned short)run[i];
          run[i] += c;
        }
        sum += run[i];
      }
      if (whole) {
        int total;
        int b = block_exclusive_scan(sum, s.warp, total);
#pragma unroll
        for (int i = 0; i < kDpt; ++i) {
          const int d = (int)threadIdx.x * kDpt + i;
          if (d < kDigits) s.base[d] = b;
          b += run[i];
        }
      } else {
#pragma unroll
        for (int i = 0; i < kDpt; ++i) {
          const int d = (int)threadIdx.x * kDpt + i;
          if (d >= kDigits) continue;
          const int b = s.run[d];
          s.base[d] = b;
          s.run[d] = b + run[i];
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
      const unsigned dgt = (unsigned)(k[j] >> shift) & (kDigits - 1);
      dst[j] = (j < mine) ? s.base[dgt] + s.whist[warp][dgt] + dst[j] : -1;
    }
  }

  // One pass of the shared-memory sort: the n keys (ipt per thread) go to s_key in digit order, and every thread
  // reloads its items from there.
  static __device__ __forceinline__ void smem_pass(unsigned long long (&k)[kItems], int n, int ipt, int shift,
                                                   Smem& s, unsigned long long* s_key) {
    int dst[kItems];
    radix_positions(k, n, ipt, shift, true, s, dst);
#pragma unroll
    for (int j = 0; j < kItems; ++j)
      if (dst[j] >= 0) s_key[dst[j]] = k[j];
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kItems; ++j)
      if (holds(j, ipt, n)) k[j] = s_key[entry_of(j, ipt)];
    // the next pass overwrites s_key only after the barriers inside radix_positions
  }

  static __device__ __forceinline__ void minmax_to_smem(unsigned kmin, unsigned kmax, unsigned imin, unsigned imax,
                                                        Smem& s) {
    kmin = __reduce_min_sync(0xffffffffu, kmin);
    kmax = __reduce_max_sync(0xffffffffu, kmax);
    imin = __reduce_min_sync(0xffffffffu, imin);
    imax = __reduce_max_sync(0xffffffffu, imax);
    if ((threadIdx.x & 31) == 0) {
      atomicMin(&s.red[0], kmin);
      atomicMax(&s.red[1], kmax);
      atomicMin(&s.red[2], imin);
      atomicMax(&s.red[3], imax);
    }
  }

  // Sorts the n = range.y - range.x entries of one tile by (depth key, id).  bucket: the tile's ids in arbitrary order
  // and out: their depth keys at the same slots (tile_scatter_kernel); out receives the same ids sorted by (depth key,
  // id).  Both are [cap] arrays indexed by the tile's range.  The shared-memory path (n <= kCap) reads every key and id
  // of the tile before it writes out; the chunked path for longer buckets uses both arrays as scratch, and so takes its
  // keys from depth_keys[id].  s_key holds kCap keys.  Called by every thread of the CTA with n > 0; ends with a CTA
  // barrier, after which s_key and s may be reused and every write to out is visible to the CTA.
  static __device__ __forceinline__ void sort_tile(int2 range, const unsigned* __restrict__ depth_keys, int* bucket,
                                                   int* out, unsigned long long* s_key, Smem& s) {
    const int n = range.y - range.x;
    if (threadIdx.x == 0) {
      s.red[0] = s.red[2] = 0xffffffffu;
      s.red[1] = s.red[3] = 0u;
    }
    __syncthreads();

    if (n <= kCap) {
      const int ipt = (n + kThreads - 1) / kThreads;  // the tile spread over all warps
      int id[kItems];
      unsigned dk[kItems];
#pragma unroll
      for (int j = 0; j < kItems; ++j) {
        const bool h = holds(j, ipt, n);
        id[j] = h ? bucket[range.x + entry_of(j, ipt)] : -1;
        dk[j] = h ? (unsigned)out[range.x + entry_of(j, ipt)] : 0u;
      }
      unsigned kmin = 0xffffffffu, kmax = 0u, imin = 0xffffffffu, imax = 0u;
#pragma unroll
      for (int j = 0; j < kItems; ++j) {
        if (id[j] < 0) continue;
        kmin = min(kmin, dk[j]); kmax = max(kmax, dk[j]);
        imin = min(imin, (unsigned)id[j]); imax = max(imax, (unsigned)id[j]);
      }
      minmax_to_smem(kmin, kmax, imin, imax, s);
      __syncthreads();
      kmin = s.red[0];
      imin = s.red[2];
      const int bi = bits_of(s.red[3] - imin), bits = bits_of(s.red[1] - kmin) + bi;
      unsigned long long k[kItems];
#pragma unroll
      for (int j = 0; j < kItems; ++j)
        k[j] = ((unsigned long long)(dk[j] - kmin) << bi) | (unsigned long long)((unsigned)id[j] - imin);
      // stable passes over the depth bits only: s_key ends in depth order, equal depth keys in bucket order
      for (int shift = bi; shift < bits; shift += kDigitBits) smem_pass(k, n, ipt, shift, s, s_key);
      if (bits == bi) {  // one depth key over the whole tile: no pass ran
#pragma unroll
        for (int j = 0; j < kItems; ++j)
          if (holds(j, ipt, n)) s_key[entry_of(j, ipt)] = k[j];
        __syncthreads();
      }
      // ties: find every run of equal depth keys (read only), then the thread holding its first entry sorts the run by
      // id in place.  A run longer than kTieRun sends the whole tile through the passes on the full key instead.
      unsigned long long runs[kRunWords];  // 5 bits per item: length of the run it starts (0: none)
#pragma unroll
      for (int w = 0; w < kRunWords; ++w) runs[w] = 0ull;
      bool too_long = false;
#pragma unroll
      for (int j = 0; j < kItems; ++j) {
        const int e = j * kThreads + threadIdx.x;
        if (j >= ipt || e >= n) continue;
        const unsigned long long d = s_key[e] >> bi;
        if (e > 0 && (s_key[e - 1] >> bi) == d) continue;  // not the first entry of its run
        int len = 1;
        while (len <= kTieRun && e + len < n && (s_key[e + len] >> bi) == d) ++len;
        if (len > kTieRun) too_long = true;
        else runs[j / 12] |= (unsigned long long)len << (5 * (j % 12));
      }
      if (__syncthreads_or(too_long)) {
#pragma unroll
        for (int j = 0; j < kItems; ++j) k[j] = holds(j, ipt, n) ? s_key[entry_of(j, ipt)] : 0ull;
        for (int shift = 0; shift < bits; shift += kDigitBits) smem_pass(k, n, ipt, shift, s, s_key);
      } else {
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
          const int e = j * kThreads + threadIdx.x, len = (int)(runs[j / 12] >> (5 * (j % 12))) & 31;
          for (int a = e + 1; a < e + len; ++a) {  // insertion sort of s_key[e, e + len)
            const unsigned long long v = s_key[a];
            int b = a;
            for (; b > e && s_key[b - 1] > v; --b) s_key[b] = s_key[b - 1];
            s_key[b] = v;
          }
        }
        __syncthreads();
      }
      const unsigned long long imask = (1ull << bi) - 1ull;
      for (int e = threadIdx.x; e < n; e += kThreads) out[range.x + e] = (int)(imin + (unsigned)(s_key[e] & imask));
      __syncthreads();
      return;
    }

    // ---- long bucket: the full-key passes chunk by chunk (kCap entries in registers at a time) through global memory,
    // ids ping-ponging between bucket and out (each pass recomputes the keys from the ids); one CTA, slow but exact
    {
      unsigned kmin = 0xffffffffu, kmax = 0u, imin = 0xffffffffu, imax = 0u;
      for (int i = threadIdx.x; i < n; i += kThreads) {
        const int g = bucket[range.x + i];
        const unsigned d = depth_keys[g];
        kmin = min(kmin, d); kmax = max(kmax, d);
        imin = min(imin, (unsigned)g); imax = max(imax, (unsigned)g);
      }
      minmax_to_smem(kmin, kmax, imin, imax, s);
    }
    __syncthreads();
    const unsigned kmin = s.red[0], imin = s.red[2];
    const int bi = bits_of(s.red[3] - imin), bits = bits_of(s.red[1] - kmin) + bi;
    const unsigned long long imask = (1ull << bi) - 1ull;
    auto key_of = [&](int g) {
      return ((unsigned long long)(depth_keys[g] - kmin) << bi) | (unsigned long long)((unsigned)g - imin);
    };
    int* src = bucket + range.x;
    int* dstp = out + range.x;
    for (int shift = 0; shift < bits; shift += kDigitBits) {
      // digit histogram of the whole bucket -> running bases
      unsigned* s_cnt = reinterpret_cast<unsigned*>(s_key);
      for (int d = threadIdx.x; d < kDigits; d += kThreads) s_cnt[d] = 0u;
      __syncthreads();
      for (int i = threadIdx.x; i < n; i += kThreads)
        atomicAdd(&s_cnt[(unsigned)(key_of(src[i]) >> shift) & (kDigits - 1)], 1u);
      __syncthreads();
      {
        int c[kDpt], sum = 0;
#pragma unroll
        for (int i = 0; i < kDpt; ++i) {
          const int d = (int)threadIdx.x * kDpt + i;
          c[i] = (d < kDigits) ? (int)s_cnt[d] : 0;
          sum += c[i];
        }
        int total;
        int b = block_exclusive_scan(sum, s.warp, total);
#pragma unroll
        for (int i = 0; i < kDpt; ++i) {
          const int d = (int)threadIdx.x * kDpt + i;
          if (d < kDigits) s.run[d] = b;
          b += c[i];
        }
      }
      __syncthreads();
      for (int c0 = 0; c0 < n; c0 += kCap) {
        const int m = min(kCap, n - c0);
        unsigned long long k[kItems];
#pragma unroll
        for (int j = 0; j < kItems; ++j)
          k[j] = holds(j, kItems, m) ? key_of(src[c0 + entry_of(j, kItems)]) : 0ull;
        int dst[kItems];
        radix_positions(k, m, kItems, shift, false, s, dst);
#pragma unroll
        for (int j = 0; j < kItems; ++j)
          if (dst[j] >= 0) dstp[dst[j]] = (int)(imin + (unsigned)(k[j] & imask));
        __syncthreads();  // s.whist / s.base are reused by the next chunk; global writes visible to the CTA
      }
      int* t = src; src = dstp; dstp = t;
    }
    if (src != out + range.x) {  // an even number of passes (or none) left the result in the bucket
      for (int i = threadIdx.x; i < n; i += kThreads) out[range.x + i] = src[i];
    }
    __syncthreads();
  }
};

}  // namespace gbsort
