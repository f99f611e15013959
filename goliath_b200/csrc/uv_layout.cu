// goliath_b200/csrc/uv_layout.cu — UV index, face and barycentric images of a mesh's UV layout, and the
// nearest-valid-texel impaint (sm_90a).
//
// Replaces make_uv_face_index / make_uv_vert_index / make_uv_barys / index_image_impaint (ca_code/utils/geom.py:31-194),
// which run pytorch3d's rasterize_meshes and an sklearn KDTree on the host.  pytorch3d is third-party and outside the
// reference tree, so the rasteriser's conventions below are this project's (DESIGN.md R12, PARITY UNPINNED):
//   * the NDC vertex of UV coordinate (u, v) is x = 2 (1 - u) - 1, y = 2 (1 - v) - 1, or y = 2 (1 - (1 - v)) - 1 with
//     flip_uv, each operation rounded to fp32 in that order (the reference's `1 - vt`, the flip, `2 vt - 1`);
//   * texel (row i, column j) samples the NDC pixel centre x_j = 1 - (2 j + 1) / U, y_i = 1 - (2 i + 1) / U in fp32, so
//     it sits at u = (j + 0.5) / U, v = (i + 0.5) / U without the flip;
//   * a face whose NDC area |e(v0, v1, v2)| is at most 1e-8 is skipped, e(a, b, p) = (p.x - a.x)(b.y - a.y) -
//     (p.y - a.y)(b.x - a.x);
//   * the inside test is inclusive and accepts both windings: every edge function e(v1, v2, p), e(v2, v0, p),
//     e(v0, v1, p) >= 0 for a positive area, <= 0 for a negative one, so a texel centre exactly on an edge or a
//     vertex is covered;
//   * every vertex has z = 1, so all faces tie in depth and a texel takes the LOWEST covering face id (an int32
//     atomicMin into an image set to INT_MAX: order-independent, no ordering pass).
// The barycentric map is the reference's bary_coords (geom.py:86-106) on the UV triangle, with its +-1e-6 clamp of the
// denominator, at the sample grid the caller builds with the reference's own torch.linspace call.  The file is built
// with -fmad=false (build.py): the face image and the barycentrics are bit-exact with the same fp32 expressions
// evaluated one rounding at a time (tests/uv_raster_restate.py, and torch for the barycentrics).
//
// Raster: one thread per face over its texel box; a face whose box holds more than kLargeFaceTexels texels is appended
// to a list that a second kernel walks with one CTA per face.  A per-texel pass then writes the face image (-1 where
// uncovered), vi[face], the barycentrics and the valid mask.
//
// Impaint: an exact squared Euclidean distance transform in integer arithmetic (per column a warp-scanned nearest valid
// texel above and below; per row Meijster's lower envelope of parabolas), then, for each invalid texel with
// sqrt(d2) < threshold, the offsets of squared length exactly d2 from a host-built table sorted by (d2, di, dj): the
// first in-image valid one is the source, i.e. the smallest row-major index among the equidistant valid texels.  One
// gather applies the source table to up to three images.  No float atomics anywhere: two calls give the same bits.
#include <climits>

#include "common.cuh"
#include "../../include/goliath_b200.h"

namespace {

constexpr int kBlock = 256;
constexpr int kLargeFaceTexels = 256;  // texel-box size above which a face goes to the CTA-per-face kernel
constexpr float kZeroArea = 1e-8f;     // PARITY UNPINNED: |NDC area| at or below which a face is skipped
constexpr float kBaryEps = 1e-6f;      // geom.py:86
constexpr size_t kMaxRowSmem = 227 * 1024;  // the row pass keeps four int rows in shared memory: W <= 14528

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

struct UvTri {
  float x[3], y[3];
};

__device__ __forceinline__ float edge_fn(float ax, float ay, float bx, float by, float px, float py) {
  return (px - ax) * (by - ay) - (py - ay) * (bx - ax);
}

// the NDC triangle of face f: x = 2 (1 - u) - 1, y = 2 (1 - v) - 1 (flip: 2 (1 - (1 - v)) - 1), one rounding per op
__device__ __forceinline__ UvTri load_ndc(const float* __restrict__ vt, const int* __restrict__ vti, int f, int flip) {
  UvTri t;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int v = vti[3 * f + k];
    const float a = 1.f - vt[2 * v];
    float b = 1.f - vt[2 * v + 1];
    if (flip) b = 1.f - b;
    t.x[k] = 2.f * a - 1.f;
    t.y[k] = 2.f * b - 1.f;
  }
  return t;
}

__device__ __forceinline__ float pix_ndc(int k, int U) { return 1.f - (float)(2 * k + 1) / (float)U; }

struct Box {
  int j0, j1, i0, i1;
};

// the texels whose centre can lie in the face's NDC bounding box, with one texel of margin, clipped to the image;
// false for a zero-area (or non-finite) face and for a box outside the image
__device__ __forceinline__ bool face_box(const UvTri& t, int U, float& area, Box& b) {
  area = edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], t.x[2], t.y[2]);
  if (!(fabsf(area) > kZeroArea) || !isfinite(area)) return false;
  const float xmin = fminf(fminf(t.x[0], t.x[1]), t.x[2]), xmax = fmaxf(fmaxf(t.x[0], t.x[1]), t.x[2]);
  const float ymin = fminf(fminf(t.y[0], t.y[1]), t.y[2]), ymax = fmaxf(fmaxf(t.y[0], t.y[1]), t.y[2]);
  const float Uf = (float)U;
  // x_j = 1 - (2 j + 1) / U decreases with j: j = ((1 - x) U - 1) / 2
  const float j0 = fmaxf(ceilf(((1.f - xmax) * Uf - 1.f) * 0.5f) - 1.f, 0.f);
  const float j1 = fminf(floorf(((1.f - xmin) * Uf - 1.f) * 0.5f) + 1.f, Uf - 1.f);
  const float i0 = fmaxf(ceilf(((1.f - ymax) * Uf - 1.f) * 0.5f) - 1.f, 0.f);
  const float i1 = fminf(floorf(((1.f - ymin) * Uf - 1.f) * 0.5f) + 1.f, Uf - 1.f);
  if (!(j0 <= j1) || !(i0 <= i1)) return false;
  b.j0 = (int)j0;
  b.j1 = (int)j1;
  b.i0 = (int)i0;
  b.i1 = (int)i1;
  return true;
}

__device__ __forceinline__ void raster_texel(int* __restrict__ img, int U, const UvTri& t, float area, int f, int i,
                                             int j) {
  const float px = pix_ndc(j, U), py = pix_ndc(i, U);
  const float w0 = edge_fn(t.x[1], t.y[1], t.x[2], t.y[2], px, py);
  const float w1 = edge_fn(t.x[2], t.y[2], t.x[0], t.y[0], px, py);
  const float w2 = edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], px, py);
  const bool in = area > 0.f ? (w0 >= 0.f && w1 >= 0.f && w2 >= 0.f) : (w0 <= 0.f && w1 <= 0.f && w2 <= 0.f);
  if (in) atomicMin(img + (size_t)i * U + j, f);
}

__global__ void __launch_bounds__(kBlock) uv_raster_init_kernel(long long n, int* __restrict__ img,
                                                                int* __restrict__ n_large) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t == 0) *n_large = 0;
  if (t < n) img[t] = INT_MAX;
}

__global__ void __launch_bounds__(kBlock) uv_raster_small_kernel(int F, int U, int flip, const float* __restrict__ vt,
                                                                 const int* __restrict__ vti, int* __restrict__ img,
                                                                 int* __restrict__ n_large, int* __restrict__ large) {
  const int f = blockIdx.x * kBlock + threadIdx.x;
  if (f >= F) return;
  const UvTri t = load_ndc(vt, vti, f, flip);
  float area;
  Box b;
  if (!face_box(t, U, area, b)) return;
  if ((long long)(b.j1 - b.j0 + 1) * (b.i1 - b.i0 + 1) > kLargeFaceTexels) {
    large[atomicAdd(n_large, 1)] = f;  // the list order does not matter: atomicMin is order-independent
    return;
  }
  for (int i = b.i0; i <= b.i1; ++i)
    for (int j = b.j0; j <= b.j1; ++j) raster_texel(img, U, t, area, f, i, j);
}

__global__ void __launch_bounds__(kBlock) uv_raster_large_kernel(int U, int flip, const float* __restrict__ vt,
                                                                 const int* __restrict__ vti, int* __restrict__ img,
                                                                 const int* __restrict__ n_large,
                                                                 const int* __restrict__ large) {
  const int n = *n_large;
  for (int it = blockIdx.x; it < n; it += gridDim.x) {
    const int f = large[it];
    const UvTri t = load_ndc(vt, vti, f, flip);
    float area;
    Box b;
    if (!face_box(t, U, area, b)) continue;
    const int bw = b.j1 - b.j0 + 1;
    const long long n_tex = (long long)bw * (b.i1 - b.i0 + 1);
    for (long long p = threadIdx.x; p < n_tex; p += kBlock)
      raster_texel(img, U, t, area, f, b.i0 + (int)(p / bw), b.j0 + (int)(p % bw));
  }
}

// per texel: face (-1 where uncovered), vi[face] (-1 x 3), bary_coords on the UV triangle (0 x 3), valid = face >= 0
__global__ void __launch_bounds__(kBlock) uv_texel_kernel(int U, int flip, const float* __restrict__ vt,
                                                          const int* __restrict__ vti, const int* __restrict__ vi,
                                                          const float* __restrict__ grid, const int* __restrict__ img,
                                                          long long* __restrict__ face_out,
                                                          long long* __restrict__ vert_out,
                                                          float* __restrict__ bary_out,
                                                          unsigned char* __restrict__ valid_out) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= (long long)U * U) return;
  const int i = (int)(t / U), j = (int)(t % U);
  const int raw = img[t];
  const int f = raw == INT_MAX ? -1 : raw;
  if (face_out) face_out[t] = f;
  if (valid_out) valid_out[t] = f >= 0;
  if (vert_out) {
#pragma unroll
    for (int k = 0; k < 3; ++k) vert_out[3 * t + k] = f >= 0 ? (long long)vi[3 * f + k] : -1ll;
  }
  if (!bary_out) return;
  if (f < 0) {
    bary_out[3 * t] = 0.f;
    bary_out[3 * t + 1] = 0.f;
    bary_out[3 * t + 2] = 0.f;
    return;
  }
  float tx[3], ty[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int v = vti[3 * f + k];
    tx[k] = vt[2 * v];
    ty[k] = flip ? 1.f - vt[2 * v + 1] : vt[2 * v + 1];
  }
  // geom.py:89-104, term by term
  const float x = grid[j] - tx[2], x1 = tx[0] - tx[2], x2 = tx[1] - tx[2];
  const float y = grid[i] - ty[2], y1 = ty[0] - ty[2], y2 = ty[1] - ty[2];
  float denom = y2 * x1 - y1 * x2;
  const float n0 = y2 * x - x2 * y;
  const float n1 = x1 * y - y1 * x;
  denom = denom >= 0.f ? fmaxf(denom, kBaryEps) : fminf(denom, -kBaryEps);
  const float b0 = n0 / denom, b1 = n1 / denom;
  bary_out[3 * t] = b0;
  bary_out[3 * t + 1] = b1;
  bary_out[3 * t + 2] = 1.f - b0 - b1;
}

// ------------------------------------------------------------------------------------------------------- impaint

__device__ __forceinline__ bool texel_valid(const long long* __restrict__ index, int C, long long t) {
  for (int c = 0; c < C; ++c)
    if (index[t * C + c] != -1) return true;
  return false;
}


// one warp per column j: g[i, j] = |i - the nearest valid row of column j|, or inf = H + W when the column has none.
// Lane l owns rows [l R, l R + R); the nearest valid row above (below) a row outside its chunk comes from a warp max
// (min) scan of the chunks' last (first) valid rows.
__global__ void __launch_bounds__(32) edt_cols_kernel(int H, int W, int C, const long long* __restrict__ index,
                                                      int* __restrict__ g) {
  extern __shared__ int above[];  // [H] the nearest valid row <= i inside the lane's chunk, -1 if none
  const int j = blockIdx.x, lane = threadIdx.x, inf = H + W;
  const int R = (H + 31) / 32, r0 = min(lane * R, H), r1 = min(r0 + R, H);
  int last = -1;
  for (int i = r0; i < r1; ++i) {
    if (texel_valid(index, C, (long long)i * W + j)) last = i;
    above[i] = last;
  }
  int first = INT_MAX;
  for (int i = r1 - 1; i >= r0; --i)
    if (above[i] == i) first = i;
  int up = last, down = first;  // inclusive scans: max over lanes <= lane, min over lanes >= lane
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, up, o), b = __shfl_down_sync(0xffffffffu, down, o);
    if (lane >= o) up = max(up, a);
    if (lane + o < 32) down = min(down, b);
  }
  int carry_up = __shfl_up_sync(0xffffffffu, up, 1), below = __shfl_down_sync(0xffffffffu, down, 1);
  if (lane == 0) carry_up = -1;
  if (lane == 31) below = INT_MAX;
  for (int i = r1 - 1; i >= r0; --i) {
    if (above[i] == i) below = i;
    const int a = above[i] >= 0 ? above[i] : carry_up;
    int d = inf;
    if (a >= 0) d = i - a;
    if (below != INT_MAX) d = min(d, below - i);
    g[(size_t)i * W + j] = d;
  }
}

// one warp per row i: d2[i, j] = min_k (j - k)^2 + g[i, k]^2 by Meijster's lower envelope (lane 0 walks the row in
// shared memory; the warp loads and stores it).  Integer arithmetic throughout: the distances are exact.
__global__ void __launch_bounds__(32) edt_rows_kernel(int H, int W, const int* __restrict__ g, int* __restrict__ d2) {
  extern __shared__ int sm[];
  int* gr = sm;          // [W] the row of g
  int* s = sm + W;       // [W] the envelope's parabola apices
  int* t = sm + 2 * W;   // [W] the first column each one owns
  int* dt = sm + 3 * W;  // [W] the result row
  const int i = blockIdx.x, lane = threadIdx.x;
  for (int k = lane; k < W; k += 32) gr[k] = g[(size_t)i * W + k];
  __syncwarp();
  if (lane == 0) {
    auto f = [&](long long x, int k) { return (x - k) * (x - k) + (long long)gr[k] * gr[k]; };
    int q = 0;
    s[0] = 0;
    t[0] = 0;
    for (int u = 1; u < W; ++u) {
      while (q >= 0 && f(t[q], s[q]) > f(t[q], u)) --q;
      if (q < 0) {
        q = 0;
        s[0] = u;
      } else {
        // the first column where apex u is strictly closer than apex s[q]; the numerator is >= 0 because apex s[q] is
        // no farther than u at column t[q] >= 0, so C division is floor division here
        const long long a = s[q];
        const long long w = 1 + ((long long)u * u - a * a + (long long)gr[u] * gr[u] - (long long)gr[a] * gr[a]) /
                                    (2 * (u - a));
        if (w < W) {
          ++q;
          s[q] = u;
          t[q] = (int)w;
        }
      }
    }
    for (int u = W - 1; u >= 0; --u) {
      dt[u] = (int)f(u, s[q]);
      if (u == t[q]) --q;
    }
  }
  __syncwarp();
  for (int k = lane; k < W; k += 32) d2[(size_t)i * W + k] = dt[k];
}

// per texel: the source texel of the impaint, -1 for a valid texel and for one at sqrt(d2) >= the threshold.  The
// candidates are the offsets of squared length exactly d2, in (di, dj) order: the first in-image valid one is the
// valid texel at distance d with the smallest row-major index.
__global__ void __launch_bounds__(kBlock) impaint_select_kernel(int H, int W, const int* __restrict__ d2, int d2max,
                                                                const int* __restrict__ offsets,
                                                                const int* __restrict__ group_start,
                                                                int* __restrict__ src) {
  const long long p = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (p >= (long long)H * W) return;
  const int i = (int)(p / W), j = (int)(p % W), d = d2[p];
  int out = -1;
  if (d > 0 && d <= d2max) {
    for (int k = group_start[d], e = group_start[d + 1]; k < e; ++k) {
      const int ni = i + offsets[2 * k], nj = j + offsets[2 * k + 1];
      if (ni >= 0 && ni < H && nj >= 0 && nj < W && d2[(size_t)ni * W + nj] == 0) {
        out = ni * W + nj;
        break;
      }
    }
  }
  src[p] = out;
}

struct GatherImage {
  const unsigned* in;
  unsigned* out;
  int words;  // 32-bit words per texel
};

__device__ __forceinline__ void gather_words(const GatherImage& m, long long t, long long from) {
  if (!m.in) return;
  for (int c = 0; c < m.words; ++c) m.out[t * m.words + c] = m.in[from * m.words + c];
}

// out[t] = in[src[t]] where src[t] >= 0, in[t] elsewhere, for up to three images of any texel size
__global__ void __launch_bounds__(kBlock) impaint_gather_kernel(long long T, const int* __restrict__ src,
                                                                GatherImage a, GatherImage b, GatherImage c) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= T) return;
  const int s = src[t];
  const long long from = s >= 0 ? s : t;
  gather_words(a, t, from);
  gather_words(b, t, from);
  gather_words(c, t, from);
}

unsigned grid1(long long n) { return (unsigned)gb::cdiv64(n, kBlock); }

}  // namespace

GB_API size_t gb_uv_raster_workspace_bytes(int F, int U) {
  return align256((size_t)U * U * 4) + 256 + (size_t)(F > 0 ? F : 0) * 4;
}

GB_API int gb_uv_index_images(int F, int U, int flip, const float* vt, const int32_t* vti, const int32_t* vi,
                              const float* grid, void* workspace, int64_t* face, int64_t* vert_index, float* bary,
                              uint8_t* valid, void* stream) {
  if (U <= 0) return 0;
  if (F < 0 || (F > 0 && vert_index && !vi) || (bary && !grid)) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const long long n = (long long)U * U;
  char* ws = (char*)workspace;
  int* img = (int*)ws;
  int* n_large = (int*)(ws + align256((size_t)n * 4));
  int* large = n_large + 64;
  GB_CUDA(gb::launch<uv_raster_init_kernel>(grid1(n), kBlock, 0, s, n, img, n_large));
  if (F > 0) {
    GB_CUDA(gb::launch<uv_raster_small_kernel>(gb::cdiv(F, kBlock), kBlock, 0, s, F, U, flip, vt, vti, img, n_large,
                                               large));
    GB_CUDA(gb::launch<uv_raster_large_kernel>(gb::kNumSMs * 8, kBlock, 0, s, U, flip, vt, vti, img, n_large, large));
  }
  return gb::launch<uv_texel_kernel>(grid1(n), kBlock, 0, s, U, flip, vt, vti, vi, grid, img, (long long*)face,
                                     (long long*)vert_index, bary, (unsigned char*)valid);
}

GB_API size_t gb_uv_impaint_workspace_bytes(int H, int W) { return align256((size_t)H * W * 4); }

GB_API int gb_uv_impaint_sources(int H, int W, int C, const int64_t* index, int d2max, const int32_t* offsets,
                                 const int32_t* group_start, void* workspace, int32_t* d2, int32_t* src, void* stream) {
  if (H <= 0 || W <= 0) return 0;
  if (C <= 0 || (d2max >= 0 && (!offsets || !group_start)) || (size_t)W * 16 > kMaxRowSmem)
    return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  int* g = (int*)workspace;
  GB_CUDA(gb::launch<edt_cols_kernel>(W, 32, (size_t)H * 4, s, H, W, C, (const long long*)index, g));
  GB_CUDA(gb::launch<edt_rows_kernel>(H, 32, (size_t)W * 16, s, H, W, g, d2));
  return gb::launch<impaint_select_kernel>(grid1((long long)H * W), kBlock, 0, s, H, W, d2, d2max, offsets,
                                           group_start, src);
}

GB_API int gb_uv_impaint_gather(int64_t T, const int32_t* src, const void* in0, void* out0, int words0, const void* in1,
                                void* out1, int words1, const void* in2, void* out2, int words2, void* stream) {
  if (T <= 0) return 0;
  const GatherImage a{(const unsigned*)in0, (unsigned*)out0, words0}, b{(const unsigned*)in1, (unsigned*)out1, words1},
      c{(const unsigned*)in2, (unsigned*)out2, words2};
  return gb::launch<impaint_gather_kernel>(grid1(T), kBlock, 0, (cudaStream_t)stream, T, src, a, b, c);
}
