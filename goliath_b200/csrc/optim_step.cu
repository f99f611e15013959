// goliath_b200/csrc/optim_step.cu — gradient hygiene + global-norm clip + Adam/AdamW over a parameter list (sm_90a).
// SURVEY.md section 8f-3.  Replaces, per train step, ca_code/utils/train.py:209-215
//     p.grad[isnan(p.grad)] = 0; p.grad[isinf(p.grad)] = 0        (two masked writes per tensor)
//     torch.nn.utils.clip_grad_norm_(params, 1.0)                 (norm pass + scale pass)
//     optimizer.step()                                            (torch.optim.Adam / AdamW, config/*.yml)
// over the 163 M parameters of the RGCA model (131 M of them one untied-bias tensor) by TWO launches that touch every
// gradient twice and every parameter / moment once:
//   grad_sanitize_sqnorm   non-finite gradient entries -> 0 (written back only where needed), sum of squares in fp64
//   adam_step              clip coefficient from the device-side norm, moments, bias-corrected update, optional L2 /
//                          decoupled weight decay, per-tensor learning rate (the reference's per-module lr)
// Multi-tensor: a device table of {p, g, m, v, numel, lr, wd} rows and a chunk map (tensor, chunk) so that one grid
// covers tensors from 3 to 131 M elements.  HBM-bound: 4 B + 28 B per parameter.
#include "common.cuh"

namespace {

constexpr int kChunk = 16384;  // elements per CTA
constexpr int kThreads = 256;

struct TensorRow {  // 56 bytes, mirrored by goliath_b200/optim.py
  float* p;
  float* g;
  float* m;
  float* v;
  long long numel;
  float lr, wd;
  int missed;  // steps this parameter sat out (no gradient): torch keeps a step count per parameter
  int pad;
};

__device__ __forceinline__ bool finite_f(float x) { return fabsf(x) <= 3.402823466e38f; }  // false for NaN and +-Inf

__global__ void __launch_bounds__(kThreads) grad_sanitize_sqnorm_kernel(const TensorRow* __restrict__ rows,
                                                                        const int2* __restrict__ chunks,
                                                                        double* __restrict__ sqnorm) {
  __shared__ float s_red[kThreads / 32];
  const int2 ck = chunks[blockIdx.x];
  const TensorRow r = rows[ck.x];
  const long long base = (long long)ck.y * kChunk;
  const long long end = min(base + kChunk, r.numel);
  float acc = 0.f;
  if (r.g) {
    const bool vec = ((reinterpret_cast<uintptr_t>(r.g) & 15) == 0);
    if (vec) {
      const long long end4 = base + ((end - base) & ~3LL);
      for (long long i = base + 4 * threadIdx.x; i < end4; i += 4 * kThreads) {
        float4 x = *reinterpret_cast<const float4*>(r.g + i);
        const bool bad = !(finite_f(x.x) && finite_f(x.y) && finite_f(x.z) && finite_f(x.w));
        if (bad) {
          x.x = finite_f(x.x) ? x.x : 0.f; x.y = finite_f(x.y) ? x.y : 0.f;
          x.z = finite_f(x.z) ? x.z : 0.f; x.w = finite_f(x.w) ? x.w : 0.f;
          *reinterpret_cast<float4*>(r.g + i) = x;
        }
        acc += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
      }
      for (long long i = end4 + threadIdx.x; i < end; i += kThreads) {
        float x = r.g[i];
        if (!finite_f(x)) { x = 0.f; r.g[i] = 0.f; }
        acc += x * x;
      }
    } else {
      for (long long i = base + threadIdx.x; i < end; i += kThreads) {
        float x = r.g[i];
        if (!finite_f(x)) { x = 0.f; r.g[i] = 0.f; }
        acc += x * x;
      }
    }
  }
  acc = gb::warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < kThreads / 32 ? s_red[threadIdx.x] : 0.f;
    t = gb::warp_sum(t);
    if (threadIdx.x == 0 && t != 0.f) atomicAdd(sqnorm, (double)t);
  }
}

struct AdamArgs {
  const TensorRow* rows;
  const int2* chunks;
  const double* sqnorm;  // may be null (no clipping)
  float max_norm, beta1, beta2, eps;
  int step;  // global step count, this one included
  int adamw, write_grads;
};

__device__ __forceinline__ void adam_one(float& p, float& g, float& m, float& v, float coef, const AdamArgs& a, float lr,
                                         float wd, float bc1, float bc2_sqrt) {
  g *= coef;                                 // what clip_grad_norm_ leaves in p.grad (stored back when asked)
  float ge = g;                              // the gradient Adam sees
  if (a.adamw) p *= 1.f - lr * wd;           // decoupled decay (torch.optim.AdamW)
  else if (wd != 0.f) ge += wd * p;          // L2 (torch.optim.Adam weight_decay), not written back
  m = a.beta1 * m + (1.f - a.beta1) * ge;    // exp_avg.lerp_(grad, 1 - beta1)
  v = a.beta2 * v + (1.f - a.beta2) * ge * ge; // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
  const float denom = sqrtf(v) / bc2_sqrt + a.eps;
  p -= (lr / bc1) * (m / denom);
}

__global__ void __launch_bounds__(kThreads) adam_step_kernel(AdamArgs a) {
  const int2 ck = a.chunks[blockIdx.x];
  const TensorRow r = a.rows[ck.x];
  if (!r.g) return;  // parameter without a gradient this step: untouched, as torch skips it
  const long long base = (long long)ck.y * kChunk;
  const long long end = min(base + kChunk, r.numel);
  const double t = (double)max(a.step - r.missed, 1);  // this parameter's own step count (fp64 pow: matches the host formula)
  const float bc1 = (float)(1.0 - pow((double)a.beta1, t)), bc2_sqrt = (float)sqrt(1.0 - pow((double)a.beta2, t));
  float coef = 1.f;
  if (a.sqnorm && a.max_norm > 0.f) {  // clip_grad_norm_: coef = clamp(max_norm / (norm + 1e-6), max = 1)
    const float norm = (float)sqrt(*a.sqnorm);
    coef = fminf(a.max_norm / (norm + 1e-6f), 1.f);
  }
  const bool vec = (((reinterpret_cast<uintptr_t>(r.p) | reinterpret_cast<uintptr_t>(r.g) | reinterpret_cast<uintptr_t>(r.m) |
                      reinterpret_cast<uintptr_t>(r.v)) & 15) == 0);
  long long i0 = base;
  if (vec) {
    const long long end4 = base + ((end - base) & ~3LL);
    for (long long i = base + 4 * threadIdx.x; i < end4; i += 4 * kThreads) {
      float4 p = *reinterpret_cast<float4*>(r.p + i), g = *reinterpret_cast<float4*>(r.g + i);
      float4 m = *reinterpret_cast<float4*>(r.m + i), v = *reinterpret_cast<float4*>(r.v + i);
      adam_one(p.x, g.x, m.x, v.x, coef, a, r.lr, r.wd, bc1, bc2_sqrt);
      adam_one(p.y, g.y, m.y, v.y, coef, a, r.lr, r.wd, bc1, bc2_sqrt);
      adam_one(p.z, g.z, m.z, v.z, coef, a, r.lr, r.wd, bc1, bc2_sqrt);
      adam_one(p.w, g.w, m.w, v.w, coef, a, r.lr, r.wd, bc1, bc2_sqrt);
      *reinterpret_cast<float4*>(r.p + i) = p;
      *reinterpret_cast<float4*>(r.m + i) = m;
      *reinterpret_cast<float4*>(r.v + i) = v;
      if (a.write_grads) *reinterpret_cast<float4*>(r.g + i) = g;
    }
    i0 = end4;
  }
  for (long long i = i0 + threadIdx.x; i < end; i += kThreads) {
    float p = r.p[i], g = r.g[i], m = r.m[i], v = r.v[i];
    adam_one(p, g, m, v, coef, a, r.lr, r.wd, bc1, bc2_sqrt);
    r.p[i] = p; r.m[i] = m; r.v[i] = v;
    if (a.write_grads) r.g[i] = g;
  }
}

}  // namespace

GB_API int gb_optim_chunk_elems(void) { return kChunk; }
GB_API int gb_optim_row_bytes(void) { return (int)sizeof(TensorRow); }

// rows: device array of n TensorRow; chunks: device array of n_chunks (tensor index, chunk index) pairs covering every
// tensor in steps of gb_optim_chunk_elems(); *sqnorm (device fp64, zero-filled by the caller) += sum of squares of all
// gradients after non-finite entries were zeroed in place (rows with g == NULL are skipped).
GB_API int gb_grad_sanitize_sqnorm(const void* rows, const int32_t* chunks, int n_chunks, double* sqnorm, void* stream) {
  if (n_chunks <= 0) return 0;
  return gb::launch<grad_sanitize_sqnorm_kernel>(n_chunks, kThreads, 0, (cudaStream_t)stream, (const TensorRow*)rows,
                                                 (const int2*)chunks, sqnorm);
}

// One Adam (adamw = 0) / AdamW (adamw = 1) step over every row; gradients are scaled by clamp(max_norm / (sqrt(*sqnorm)
// + 1e-6), max = 1) when sqnorm != NULL and max_norm > 0; bias corrections 1 - beta^t with t = step - row.missed (torch
// counts steps per parameter); write_grads = 1 also stores the clipped gradients (what clip_grad_norm_ leaves in p.grad).
GB_API int gb_adam_step(const void* rows, const int32_t* chunks, int n_chunks, const double* sqnorm, float max_norm,
                        float beta1, float beta2, float eps, int step, int adamw, int write_grads, void* stream) {
  if (n_chunks <= 0) return 0;
  AdamArgs a;
  a.rows = (const TensorRow*)rows; a.chunks = (const int2*)chunks; a.sqnorm = sqnorm; a.max_norm = max_norm;
  a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.step = step; a.adamw = adamw;
  a.write_grads = write_grads;
  return gb::launch<adam_step_kernel>(n_chunks, kThreads, 0, (cudaStream_t)stream, a);
}
