// goliath_b200/csrc/head_frame.cu — the per-frame light work of the head avatar's frame (ca_code/models/rgca.py:
// 175-193) in one launch (sm_90a).
//
//   gb_head_lights_fwd   one CTA per batch item: the head-relative camera (Rt @ [head_pose; 0 0 0 1]), camera
//                        position and light positions, the degree-8 SH light table headrel_light_sh [3,81] and, when
//                        given, lightrot @ R.  The arithmetic is double from the fp32 inputs; the SH basis is
//                        sh.dir2sh's (reference ordering, cos(acos(z)), the 1e-8 clamp of sin^2) on F.normalize's
//                        max(|v|, 1e-12) direction.  The lights go through shared memory in chunks of LT_CHUNK: the
//                        first threads evaluate one light's 81 basis values each, then thread (c, k) adds
//                        sh[l][k] * I[l][c] over the chunk's lights in index order into a double.  No atomics: the
//                        same bits on every call.
#include "common.cuh"

namespace {

constexpr int LT_THREADS = 256, LT_CHUNK = 128, LT_DEG = 8, LT_NSH = (LT_DEG + 1) * (LT_DEG + 1);
static_assert(3 * LT_NSH <= LT_THREADS, "one thread per (channel, coefficient)");
static_assert(LT_CHUNK <= LT_THREADS, "one thread per light of a chunk");

__global__ void __launch_bounds__(LT_THREADS) head_lights_kernel(int L, int C, const float* __restrict__ head_pose,
                                                                 const float* __restrict__ campos,
                                                                 const float* __restrict__ Rt,
                                                                 const float* __restrict__ light_pos,
                                                                 const float* __restrict__ light_intensity,
                                                                 const float* __restrict__ lightrot,
                                                                 float* __restrict__ headrel_Rt,
                                                                 float* __restrict__ headrel_campos,
                                                                 float* __restrict__ headrel_light_pos,
                                                                 float* __restrict__ headrel_light_sh,
                                                                 float* __restrict__ lightrot_out) {
  __shared__ float s_sh[LT_CHUNK][LT_NSH];
  __shared__ float s_int[LT_CHUNK][3];
  __shared__ double s_knorm[LT_NSH];  // K_n^|m|, times sqrt(2) for m != 0, at n^2 + n + m
  __shared__ double s_pose[12];       // head_pose [3,4]: R | t
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid < 12) s_pose[tid] = (double)head_pose[b * 12 + tid];
  if (tid < LT_NSH) {
    int n = 0;
    while ((n + 1) * (n + 1) <= tid) ++n;
    const int m = abs(tid - n * n - n);
    double r = 1.0;
    for (int i = n - m + 1; i <= n + m; ++i) r *= (double)i;
    double k = sqrt((2 * n + 1) / (4.0 * 3.14159265358979323846) / r);
    if (m != 0) k *= 1.4142135623730950488;
    s_knorm[tid] = k;
  }
  __syncthreads();
  const double* P = s_pose;  // R[i][j] = P[4 i + j], t[i] = P[4 i + 3]

  if (tid < 12) {  // headrel_Rt = Rt @ [head_pose; 0 0 0 1]
    const int i = tid / 4, j = tid % 4;
    const float* A = Rt + b * 12;
    double s = 0.0;
    for (int k = 0; k < 3; ++k) s += (double)A[4 * i + k] * P[4 * k + j];
    if (j == 3) s += (double)A[4 * i + 3];
    headrel_Rt[b * 12 + tid] = (float)s;
  } else if (tid < 15) {  // headrel_campos = (campos - t) @ R
    const int j = tid - 12;
    double s = 0.0;
    for (int i = 0; i < 3; ++i) s += ((double)campos[b * 3 + i] - P[4 * i + 3]) * P[4 * i + j];
    headrel_campos[b * 3 + j] = (float)s;
  } else if (lightrot != nullptr && tid >= 32 && tid < 41) {  // lightrot @ R
    const int i = (tid - 32) / 3, j = (tid - 32) % 3;
    double s = 0.0;
    for (int k = 0; k < 3; ++k) s += (double)lightrot[b * 9 + 3 * i + k] * P[4 * k + j];
    lightrot_out[b * 9 + 3 * i + j] = (float)s;
  }

  double acc = 0.0;  // thread (c, k) = (tid / 81, tid % 81)
  const int ac = tid / LT_NSH, ak = tid % LT_NSH;
  for (int l0 = 0; l0 < L; l0 += LT_CHUNK) {
    const int nl = min(LT_CHUNK, L - l0);
    if (tid < nl) {
      const int l = l0 + tid;
      const float* lp = light_pos + ((size_t)b * L + l) * 3;
      double p[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < 3; ++i) s += ((double)lp[i] - P[4 * i + 3]) * P[4 * i + j];
        p[j] = s;
      }
      float* out = headrel_light_pos + ((size_t)b * L + l) * 3;
      out[0] = (float)p[0];
      out[1] = (float)p[1];
      out[2] = (float)p[2];
      const double inv = 1.0 / fmax(sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]), 1e-12);
      const double x = p[0] * inv, y = p[1] * inv, z = fmin(fmax(p[2] * inv, -1.0), 1.0);
      const double ct = cos(acos(z));
      const double st = sqrt(fmax((1.0 + ct) * (1.0 - ct), 1e-8));
      const double phi = atan2(y, x), c1 = cos(phi), s1 = sin(phi);
      double pmm = 1.0, cm = 1.0, sm = 0.0;  // P_m^m, cos(m phi), sin(m phi)
      float* row = s_sh[tid];
      for (int m = 0; m <= LT_DEG; ++m) {
        if (m > 0) {
          pmm = -pmm * (2 * m - 1) * st;
          const double cn = cm * c1 - sm * s1;
          sm = sm * c1 + cm * s1;
          cm = cn;
        }
        double p_prev = 0.0, p_cur = pmm;
        for (int n = m; n <= LT_DEG; ++n) {
          if (n == m + 1) {
            p_prev = p_cur;
            p_cur = ct * (2 * m + 1) * p_cur;
          } else if (n > m + 1) {
            const double nx = (ct * (2 * n - 1) * p_cur - (n + m - 1) * p_prev) / (n - m);
            p_prev = p_cur;
            p_cur = nx;
          }
          const int base = n * n + n;
          if (m == 0) {
            row[base] = (float)(s_knorm[base] * p_cur);
          } else {
            row[base + m] = (float)(s_knorm[base + m] * cm * p_cur);
            row[base - m] = (float)(s_knorm[base - m] * sm * p_cur);
          }
        }
      }
      const float* li = light_intensity + ((size_t)b * L + l) * C;
#pragma unroll
      for (int c = 0; c < 3; ++c) s_int[tid][c] = li[C == 1 ? 0 : c];
    }
    __syncthreads();
    if (tid < 3 * LT_NSH)
      for (int i = 0; i < nl; ++i) acc += (double)s_sh[i][ak] * (double)s_int[i][ac];
    __syncthreads();
  }
  if (tid < 3 * LT_NSH) headrel_light_sh[(size_t)b * 3 * LT_NSH + tid] = (float)acc;
}

}  // namespace

GB_API int gb_head_lights_fwd(int B, int L, int C, const float* head_pose, const float* campos, const float* Rt,
                              const float* light_pos, const float* light_intensity, const float* lightrot,
                              float* headrel_Rt, float* headrel_campos, float* headrel_light_pos,
                              float* headrel_light_sh, float* lightrot_out, void* stream) {
  if (B <= 0) return 0;
  if (L < 0 || (C != 1 && C != 3) || ((lightrot == nullptr) != (lightrot_out == nullptr))) return 1;
  return gb::launch<head_lights_kernel>(B, LT_THREADS, 0, (cudaStream_t)stream, L, C, head_pose, campos, Rt, light_pos,
                                        light_intensity, lightrot, headrel_Rt, headrel_campos, headrel_light_pos,
                                        headrel_light_sh, lightrot_out);
}
