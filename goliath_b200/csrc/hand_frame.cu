// goliath_b200/csrc/hand_frame.cu — the glue of the hand avatar's frame around the MVP raymarcher (sm_90a).
//
//   gb_hand_valid_gather_fwd / _bwd     Raymarcher.forward's valid-primitive selection (ca_code/utils/
//                                       render_raymarcher.py:36-47): primpos / volradius and four boolean-mask
//                                       indexings, through a slot table built once on the host, so no launch depends
//                                       on a device-side count.  One CTA per (item, primitive); the backward writes
//                                       every element of the full-size gradients once (zero at invalid primitives).
//   gb_hand_finish_fwd / _bwd           the march output to the frame's images (render_raymarcher.py:69-70 and
//                                       hand_mvp.py:249-255): channels-last rayrgba -> CalV5 rows -> (training)
//                                       + (1 - alpha) * background, written as NCHW rgb and alpha.  The calibration
//                                       gradients are per-CTA partials reduced per view in a fixed order by a second
//                                       launch: no float atomics, the same bits on every call.
#include "common.cuh"

namespace {

constexpr int kGatherThreads = 256;
constexpr int kFinishThreads = 256;
constexpr int kFinishPixels = 8;  // pixels per thread of the finish kernels: one CTA covers 2048 pixels of a view

// one CTA per (b, k): the template's float4s and the 15 transform floats of primitive k
__global__ void __launch_bounds__(kGatherThreads)
    valid_gather_fwd_kernel(int K, int n_valid, int tpl4, const int* __restrict__ slot,
                            const float4* __restrict__ tpl, const float* __restrict__ pos,
                            const float* __restrict__ rot, const float* __restrict__ scale, float inv_radius,
                            float4* __restrict__ tpl_out, float* __restrict__ pos_out, float* __restrict__ rot_out,
                            float* __restrict__ scale_out) {
  const int k = blockIdx.x, b = blockIdx.y;
  const int j = slot[k];
  if (j < 0) return;
  const size_t src = (size_t)b * K + k, dst = (size_t)b * n_valid + j;
  const float4* s = tpl + src * tpl4;
  float4* d = tpl_out + dst * tpl4;
  for (int i = threadIdx.x; i < tpl4; i += kGatherThreads) d[i] = gb::ld_nc_f4(s + i);
  const int t = threadIdx.x;
  if (t < 3) pos_out[dst * 3 + t] = pos[src * 3 + t] * inv_radius;
  else if (t < 12) rot_out[dst * 9 + t - 3] = rot[src * 9 + t - 3];
  else if (t < 15) scale_out[dst * 3 + t - 12] = scale[src * 3 + t - 12];
}

__global__ void __launch_bounds__(kGatherThreads)
    valid_gather_bwd_kernel(int K, int n_valid, int tpl4, const int* __restrict__ slot,
                            const float4* __restrict__ g_tpl, const float* __restrict__ g_pos,
                            const float* __restrict__ g_rot, const float* __restrict__ g_scale, float inv_radius,
                            float4* __restrict__ g_tpl_full, float* __restrict__ g_pos_full,
                            float* __restrict__ g_rot_full, float* __restrict__ g_scale_full) {
  const int k = blockIdx.x, b = blockIdx.y;
  const int j = slot[k];
  const size_t dst = (size_t)b * K + k, src = (size_t)b * n_valid + (j < 0 ? 0 : j);
  float4* d = g_tpl_full + dst * tpl4;
  const int t = threadIdx.x;
  if (j < 0) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = t; i < tpl4; i += kGatherThreads) d[i] = z;
    if (t < 3) g_pos_full[dst * 3 + t] = 0.f;
    else if (t < 12) g_rot_full[dst * 9 + t - 3] = 0.f;
    else if (t < 15) g_scale_full[dst * 3 + t - 12] = 0.f;
    return;
  }
  const float4* s = g_tpl + src * tpl4;
  for (int i = t; i < tpl4; i += kGatherThreads) d[i] = gb::ld_nc_f4(s + i);
  if (t < 3) g_pos_full[dst * 3 + t] = g_pos[src * 3 + t] * inv_radius;
  else if (t < 12) g_rot_full[dst * 9 + t - 3] = g_rot[src * 9 + t - 3];
  else if (t < 15) g_scale_full[dst * 3 + t - 12] = g_scale[src * 3 + t - 12];
}

struct FinishArgs {
  int B, HW;
  const float4* rayrgba;                         // [B,H,W,4]
  const float *cal_w, *cal_b, *bg;               // [B,3], [B,3] (both NULL: no calibration); [B,3,H,W] or NULL
  const int* grey;                               // [B] or NULL
  float *rgb, *alpha;                            // [B,3,H,W], [B,1,H,W]
  const float *g_rgb, *g_alpha;                  // backward: [B,3,H,W], [B,1,H,W] (NULL: zero)
  float4* g_rayrgba;                             // [B,H,W,4]
  float* partial;                                // [B, n_blocks, 6]: per-CTA sums of g_w (3) and g_b (3)
};

__global__ void __launch_bounds__(kFinishThreads) hand_finish_fwd_kernel(FinishArgs a) {
  const int b = blockIdx.y;
  const size_t HW = (size_t)a.HW;
  const bool cal = a.cal_w != nullptr, grey = cal && a.grey && a.grey[b];
  float w[3] = {1.f, 1.f, 1.f}, c[3] = {0.f, 0.f, 0.f};
  if (cal)
    for (int i = 0; i < 3; ++i) w[i] = a.cal_w[3 * b + i], c[i] = a.cal_b[3 * b + i];
  const int p0 = blockIdx.x * kFinishThreads * kFinishPixels + threadIdx.x;
#pragma unroll
  for (int r = 0; r < kFinishPixels; ++r) {
    const int p = p0 + r * kFinishThreads;
    if (p >= a.HW) break;
    const float4 s = a.rayrgba[b * HW + p];
    float v[3] = {s.x, s.y, s.z};
    if (grey) {
      const float g = v[0] * w[0] + v[1] * w[1] + v[2] * w[2] + (c[0] + c[1] + c[2]);
      v[0] = v[1] = v[2] = g;
    } else if (cal) {
      for (int i = 0; i < 3; ++i) v[i] = v[i] * w[i] + c[i];
    }
    if (a.bg) {
      const float t = 1.f - s.w;
      for (int i = 0; i < 3; ++i) v[i] += t * a.bg[(b * 3 + i) * HW + p];
    }
    for (int i = 0; i < 3; ++i) a.rgb[(b * 3 + i) * HW + p] = v[i];
    a.alpha[b * HW + p] = s.w;
  }
}

__global__ void __launch_bounds__(kFinishThreads) hand_finish_bwd_kernel(FinishArgs a) {
  __shared__ float red[kFinishThreads / 32][6];
  const int b = blockIdx.y;
  const size_t HW = (size_t)a.HW;
  const bool cal = a.cal_w != nullptr, grey = cal && a.grey && a.grey[b];
  float w[3] = {1.f, 1.f, 1.f};
  if (cal)
    for (int i = 0; i < 3; ++i) w[i] = a.cal_w[3 * b + i];
  float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const int p0 = blockIdx.x * kFinishThreads * kFinishPixels + threadIdx.x;
#pragma unroll
  for (int r = 0; r < kFinishPixels; ++r) {
    const int p = p0 + r * kFinishThreads;
    if (p >= a.HW) break;
    const float4 s = a.rayrgba[b * HW + p];
    float g[3];
    for (int i = 0; i < 3; ++i) g[i] = a.g_rgb[(b * 3 + i) * HW + p];
    float ga = a.g_alpha ? a.g_alpha[b * HW + p] : 0.f;
    if (a.bg)  // d/d alpha of (1 - alpha) * bg: alpha is not detached (hand_mvp.py:252-255)
      for (int i = 0; i < 3; ++i) ga -= g[i] * a.bg[(b * 3 + i) * HW + p];
    const float v[3] = {s.x, s.y, s.z};
    float4 o;
    if (grey) {
      const float gs = g[0] + g[1] + g[2];
      o = make_float4(gs * w[0], gs * w[1], gs * w[2], ga);
      for (int i = 0; i < 3; ++i) acc[i] += gs * v[i], acc[3 + i] += gs;
    } else {
      o = make_float4(g[0] * w[0], g[1] * w[1], g[2] * w[2], ga);
      for (int i = 0; i < 3; ++i) acc[i] += g[i] * v[i], acc[3 + i] += g[i];
    }
    a.g_rayrgba[b * HW + p] = o;
  }
  if (!cal) return;
  // fixed-order CTA reduction: butterfly within each warp, then the warps in index order
  for (int i = 0; i < 6; ++i) acc[i] = gb::warp_sum(acc[i]);
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
    for (int i = 0; i < 6; ++i) red[warp][i] = acc[i];
  __syncthreads();
  if (threadIdx.x < 6) {
    float s = 0.f;
    for (int q = 0; q < kFinishThreads / 32; ++q) s += red[q][threadIdx.x];
    a.partial[((size_t)b * gridDim.x + blockIdx.x) * 6 + threadIdx.x] = s;
  }
}

// one CTA per view: the view's partials in a fixed order -> g_cal_w [B,3], g_cal_b [B,3] (written)
__global__ void __launch_bounds__(kFinishThreads)
    hand_finish_cal_reduce_kernel(int n_blocks, const float* __restrict__ partial, float* __restrict__ g_cal_w,
                                  float* __restrict__ g_cal_b) {
  __shared__ float red[kFinishThreads / 32][6];
  const int b = blockIdx.x;
  float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int q = threadIdx.x; q < n_blocks; q += kFinishThreads)
    for (int i = 0; i < 6; ++i) acc[i] += partial[((size_t)b * n_blocks + q) * 6 + i];
  for (int i = 0; i < 6; ++i) acc[i] = gb::warp_sum(acc[i]);
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
    for (int i = 0; i < 6; ++i) red[warp][i] = acc[i];
  __syncthreads();
  if (threadIdx.x < 6) {
    float s = 0.f;
    for (int q = 0; q < kFinishThreads / 32; ++q) s += red[q][threadIdx.x];
    (threadIdx.x < 3 ? g_cal_w : g_cal_b)[3 * b + threadIdx.x % 3] = s;
  }
}

int finish_blocks(int HW) { return gb::cdiv(HW, kFinishThreads * kFinishPixels); }

}  // namespace

GB_API int gb_hand_valid_gather_fwd(int B, int K, int n_valid, int tpl_elems, const int32_t* slot, const float* tpl,
                                    const float* pos, const float* rot, const float* scale, float inv_radius,
                                    float* tpl_out, float* pos_out, float* rot_out, float* scale_out, void* stream) {
  if (B <= 0 || K <= 0 || n_valid <= 0) return 0;
  if (tpl_elems <= 0 || tpl_elems % 4 != 0 || B > 65535) return 1;
  return gb::launch<valid_gather_fwd_kernel>(dim3(K, B), kGatherThreads, 0, (cudaStream_t)stream,
      K, n_valid, tpl_elems / 4, slot, (const float4*)tpl, pos, rot, scale, inv_radius, (float4*)tpl_out, pos_out,
      rot_out, scale_out);
}

GB_API int gb_hand_valid_gather_bwd(int B, int K, int n_valid, int tpl_elems, const int32_t* slot, const float* g_tpl,
                                    const float* g_pos, const float* g_rot, const float* g_scale, float inv_radius,
                                    float* g_tpl_full, float* g_pos_full, float* g_rot_full, float* g_scale_full,
                                    void* stream) {
  if (B <= 0 || K <= 0) return 0;
  if (tpl_elems <= 0 || tpl_elems % 4 != 0 || B > 65535) return 1;
  return gb::launch<valid_gather_bwd_kernel>(dim3(K, B), kGatherThreads, 0, (cudaStream_t)stream,
      K, n_valid, tpl_elems / 4, slot, (const float4*)g_tpl, g_pos, g_rot, g_scale, inv_radius, (float4*)g_tpl_full,
      g_pos_full, g_rot_full, g_scale_full);
}

GB_API size_t gb_hand_finish_workspace_bytes(int B, int H, int W) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  return (size_t)B * finish_blocks(H * W) * 6 * sizeof(float);
}

GB_API int gb_hand_finish_fwd(int B, int H, int W, const float* rayrgba, const float* cal_w, const float* cal_b,
                              const int32_t* grey, const float* bg, float* rgb, float* alpha, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  if ((cal_w == nullptr) != (cal_b == nullptr) || B > 65535) return 1;
  FinishArgs a = {};
  a.B = B; a.HW = H * W; a.rayrgba = (const float4*)rayrgba; a.cal_w = cal_w; a.cal_b = cal_b; a.grey = grey;
  a.bg = bg; a.rgb = rgb; a.alpha = alpha;
  return gb::launch<hand_finish_fwd_kernel>(dim3(finish_blocks(a.HW), B), kFinishThreads, 0, (cudaStream_t)stream, a);
}

GB_API int gb_hand_finish_bwd(int B, int H, int W, const float* rayrgba, const float* cal_w, const int32_t* grey,
                              const float* bg, const float* g_rgb, const float* g_alpha, float* g_rayrgba,
                              float* g_cal_w, float* g_cal_b, void* workspace, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  if (B > 65535 || (cal_w && (!g_cal_w || !g_cal_b || !workspace))) return 1;
  FinishArgs a = {};
  a.B = B; a.HW = H * W; a.rayrgba = (const float4*)rayrgba; a.cal_w = cal_w; a.grey = grey; a.bg = bg;
  a.g_rgb = g_rgb; a.g_alpha = g_alpha; a.g_rayrgba = (float4*)g_rayrgba; a.partial = (float*)workspace;
  const int nb = finish_blocks(a.HW);
  GB_CUDA(gb::launch<hand_finish_bwd_kernel>(dim3(nb, B), kFinishThreads, 0, (cudaStream_t)stream, a));
  if (cal_w) {
    GB_CUDA(gb::launch<hand_finish_cal_reduce_kernel>(B, kFinishThreads, 0, (cudaStream_t)stream, nb, a.partial,
                                                      g_cal_w, g_cal_b));
  }
  return 0;
}
