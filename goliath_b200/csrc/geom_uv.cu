// goliath_b200/csrc/geom_uv.cu — mesh front end of the decoders: vertex normals and vertex -> UV gather (sm_90a).
// SURVEY.md section 8f-4.  Replaces ca_code/utils/geom.py:308-346 as called by rgca.PrimDecoder.forward
// (ca_code/models/rgca.py:478-491: postex = to_uv(geom); tn = normalize(to_uv(vn(geom)))):
//   vert_normals   face normals (cross product, normalised with clamp(min=eps)) scatter-added to their three vertices,
//                  then normalised — the reference runs index_select, cross, norm, 3 scatter_add_ and a second norm;
//   values_to_uv   per texel: three vertex indices + barycentric weights -> interpolated value, zero where the texel
//                  is uncovered — the reference builds a boolean mask, two masked gathers and a masked scatter per call.
// Here: one kernel over the faces (atomics into a [B,V,3] accumulator), one over the vertices, one over the texels
// (any channel count; vertex tables are L2-resident, the texel maps stream: 24 B in + 4 C B out per texel), and
// their backward counterparts (the gather's backward and the face pass' backward are atomic scatters).
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

struct float3x { float x, y, z; };
__device__ __forceinline__ float3x ld3(const float* p) { return {p[0], p[1], p[2]}; }
__device__ __forceinline__ float3x sub(float3x a, float3x b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ float3x cross(float3x a, float3x b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
__device__ __forceinline__ float dot(float3x a, float3x b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// ---- face pass: n_f = cross(v1 - v0, v2 - v0) / max(|.|, eps), added to the three corners
__global__ void __launch_bounds__(kThreads) face_normals_scatter_kernel(int B, int V, int F, const float* __restrict__ v,
                                                                        const int* __restrict__ vi, float eps,
                                                                        float* __restrict__ acc /* [B,V,3] zeroed */) {
  const int f = blockIdx.x * kThreads + threadIdx.x, b = blockIdx.y;
  if (f >= F) return;
  const int i0 = vi[3 * f], i1 = vi[3 * f + 1], i2 = vi[3 * f + 2];
  const float* vb = v + (size_t)b * V * 3;
  const float3x p0 = ld3(vb + 3 * i0), p1 = ld3(vb + 3 * i1), p2 = ld3(vb + 3 * i2);
  const float3x n = cross(sub(p1, p0), sub(p2, p0));
  const float inv = 1.f / fmaxf(sqrtf(dot(n, n)), eps);
  float* ab = acc + (size_t)b * V * 3;
  const int idx[3] = {i0, i1, i2};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    gb::red_add(ab + 3 * idx[k] + 0, n.x * inv);
    gb::red_add(ab + 3 * idx[k] + 1, n.y * inv);
    gb::red_add(ab + 3 * idx[k] + 2, n.z * inv);
  }
}

// ---- vertex pass: vn = acc / max(|acc|, eps)
__global__ void __launch_bounds__(kThreads) normalize3_kernel(long long n, const float* __restrict__ acc, float eps,
                                                              float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const float3x a = ld3(acc + 3 * i);
  const float inv = 1.f / fmaxf(sqrtf(dot(a, a)), eps);
  out[3 * i] = a.x * inv; out[3 * i + 1] = a.y * inv; out[3 * i + 2] = a.z * inv;
}

// backward of y = a / max(|a|, eps): g_a = (g - y (y.g)) / |a| where |a| >= eps, g / eps below
__device__ __forceinline__ float3x normalize_bwd(float3x a, float3x g, float eps) {
  const float len = sqrtf(dot(a, a));
  if (len < eps) return {g.x / eps, g.y / eps, g.z / eps};
  const float inv = 1.f / len;
  const float3x y = {a.x * inv, a.y * inv, a.z * inv};
  const float yg = dot(y, g);
  return {(g.x - y.x * yg) * inv, (g.y - y.y * yg) * inv, (g.z - y.z * yg) * inv};
}

__global__ void __launch_bounds__(kThreads) normalize3_bwd_kernel(long long n, const float* __restrict__ acc,
                                                                  const float* __restrict__ g_out, float eps,
                                                                  float* __restrict__ g_acc) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const float3x r = normalize_bwd(ld3(acc + 3 * i), ld3(g_out + 3 * i), eps);
  g_acc[3 * i] = r.x; g_acc[3 * i + 1] = r.y; g_acc[3 * i + 2] = r.z;
}

// backward of the face pass: g_n = sum of the corners' g_acc; through the normalisation and the cross product
__global__ void __launch_bounds__(kThreads) face_normals_scatter_bwd_kernel(int B, int V, int F, const float* __restrict__ v,
                                                                            const int* __restrict__ vi, float eps,
                                                                            const float* __restrict__ g_acc,
                                                                            float* __restrict__ g_v /* [B,V,3] zeroed */) {
  const int f = blockIdx.x * kThreads + threadIdx.x, b = blockIdx.y;
  if (f >= F) return;
  const int i0 = vi[3 * f], i1 = vi[3 * f + 1], i2 = vi[3 * f + 2];
  const float* vb = v + (size_t)b * V * 3;
  const float* gb_ = g_acc + (size_t)b * V * 3;
  const float3x p0 = ld3(vb + 3 * i0), p1 = ld3(vb + 3 * i1), p2 = ld3(vb + 3 * i2);
  const float3x e0 = sub(p1, p0), e1 = sub(p2, p0);
  const float3x n = cross(e0, e1);
  const float3x g0 = ld3(gb_ + 3 * i0), g1 = ld3(gb_ + 3 * i1), g2 = ld3(gb_ + 3 * i2);
  const float3x gn = normalize_bwd(n, {g0.x + g1.x + g2.x, g0.y + g1.y + g2.y, g0.z + g1.z + g2.z}, eps);
  // n = e0 x e1: d/de0 = e1 x gn, d/de1 = gn x e0
  const float3x ge0 = cross(e1, gn), ge1 = cross(gn, e0);
  float* gv = g_v + (size_t)b * V * 3;
  gb::red_add(gv + 3 * i1 + 0, ge0.x); gb::red_add(gv + 3 * i1 + 1, ge0.y); gb::red_add(gv + 3 * i1 + 2, ge0.z);
  gb::red_add(gv + 3 * i2 + 0, ge1.x); gb::red_add(gv + 3 * i2 + 1, ge1.y); gb::red_add(gv + 3 * i2 + 2, ge1.z);
  gb::red_add(gv + 3 * i0 + 0, -(ge0.x + ge1.x)); gb::red_add(gv + 3 * i0 + 1, -(ge0.y + ge1.y));
  gb::red_add(gv + 3 * i0 + 2, -(ge0.z + ge1.z));
}

// ---- texel pass: out[b, c, t] = sum_k bary[t, k] * values[b, index[t, k], c]  (0 where any index is -1)
__global__ void __launch_bounds__(kThreads) values_to_uv_kernel(int B, int V, int C, long long T,
                                                                const float* __restrict__ values /* [B,V,C] */,
                                                                const int* __restrict__ index /* [T,3] */,
                                                                const float* __restrict__ bary /* [T,3] */,
                                                                float* __restrict__ out /* [B,C,T] */) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
  const int b = blockIdx.y;
  if (t >= T) return;
  const int i0 = index[3 * t], i1 = index[3 * t + 1], i2 = index[3 * t + 2];
  float* o = out + (size_t)b * C * T + t;
  if (i0 == -1 || i1 == -1 || i2 == -1) {
    for (int c = 0; c < C; ++c) o[(size_t)c * T] = 0.f;
    return;
  }
  const float w0 = bary[3 * t], w1 = bary[3 * t + 1], w2 = bary[3 * t + 2];
  const float* vb = values + (size_t)b * V * C;
  for (int c = 0; c < C; ++c)
    o[(size_t)c * T] = vb[(size_t)i0 * C + c] * w0 + vb[(size_t)i1 * C + c] * w1 + vb[(size_t)i2 * C + c] * w2;
}

__global__ void __launch_bounds__(kThreads) values_to_uv_bwd_kernel(int B, int V, int C, long long T,
                                                                    const int* __restrict__ index,
                                                                    const float* __restrict__ bary,
                                                                    const float* __restrict__ g_out /* [B,C,T] */,
                                                                    float* __restrict__ g_values /* [B,V,C] zeroed */) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
  const int b = blockIdx.y;
  if (t >= T) return;
  const int i0 = index[3 * t], i1 = index[3 * t + 1], i2 = index[3 * t + 2];
  if (i0 == -1 || i1 == -1 || i2 == -1) return;
  const float w0 = bary[3 * t], w1 = bary[3 * t + 1], w2 = bary[3 * t + 2];
  const float* g = g_out + (size_t)b * C * T + t;
  float* gv = g_values + (size_t)b * V * C;
  for (int c = 0; c < C; ++c) {
    const float x = g[(size_t)c * T];
    gb::red_add(gv + (size_t)i0 * C + c, x * w0);
    gb::red_add(gv + (size_t)i1 * C + c, x * w1);
    gb::red_add(gv + (size_t)i2 * C + c, x * w2);
  }
}

}  // namespace

// v [B,V,3], vi [F,3] int32 -> vn [B,V,3]; acc [B,V,3] is scratch the caller zero-fills and keeps for the backward.
GB_API int gb_vert_normals_fwd(int B, int V, int F, const float* v, const int32_t* vi, float eps, float* acc, float* vn,
                               void* stream) {
  if (B <= 0 || V <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  if (F > 0) GB_CUDA(gb::launch<face_normals_scatter_kernel>(dim3(gb::cdiv(F, kThreads), B), kThreads, 0, s, B, V, F, v,
                                                             vi, eps, acc));
  const long long n = (long long)B * V;
  return gb::launch<normalize3_kernel>((unsigned)gb::cdiv64(n, kThreads), kThreads, 0, s, n, acc, eps, vn);
}

// g_vn [B,V,3] -> g_v [B,V,3] (zero-filled by the caller, accumulated); g_acc [B,V,3] scratch.
GB_API int gb_vert_normals_bwd(int B, int V, int F, const float* v, const int32_t* vi, float eps, const float* acc,
                               const float* g_vn, float* g_acc, float* g_v, void* stream) {
  if (B <= 0 || V <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const long long n = (long long)B * V;
  GB_CUDA(gb::launch<normalize3_bwd_kernel>((unsigned)gb::cdiv64(n, kThreads), kThreads, 0, s, n, acc, g_vn, eps,
                                            g_acc));
  if (F > 0) GB_CUDA(gb::launch<face_normals_scatter_bwd_kernel>(dim3(gb::cdiv(F, kThreads), B), kThreads, 0, s, B, V,
                                                                 F, v, vi, eps, g_acc, g_v));
  return 0;
}

// values [B,V,C], index [T,3] int32 (-1 = uncovered texel), bary [T,3] -> out [B,C,T]   (T = uv_size^2)
GB_API int gb_values_to_uv_fwd(int B, int V, int C, int64_t T, const float* values, const int32_t* index, const float* bary,
                               float* out, void* stream) {
  if (B <= 0 || T <= 0 || C <= 0) return 0;
  return gb::launch<values_to_uv_kernel>(dim3((unsigned)gb::cdiv64(T, kThreads), B), kThreads, 0, (cudaStream_t)stream,
                                         B, V, C, T, values, index, bary, out);
}

// g_out [B,C,T] -> g_values [B,V,C] (zero-filled by the caller, accumulated)
GB_API int gb_values_to_uv_bwd(int B, int V, int C, int64_t T, const int32_t* index, const float* bary, const float* g_out,
                               float* g_values, void* stream) {
  if (B <= 0 || T <= 0 || C <= 0) return 0;
  return gb::launch<values_to_uv_bwd_kernel>(dim3((unsigned)gb::cdiv64(T, kThreads), B), kThreads, 0,
                                             (cudaStream_t)stream, B, V, C, T, index, bary, g_out, g_values);
}
