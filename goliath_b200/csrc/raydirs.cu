// goliath_b200/csrc/raydirs.cu — camera rays + unit-cube slab interval (sm_90a).
//
// Replaces the reference kernel extensions/utils/utils_kernel.cu:11-51 (compute_raydirs_forward_kernel) behind
// utilslib.compute_raydirs_forward (extensions/utils/utils.cpp:46-82).  Pure bandwidth: 8 B in / 32 B out per
// ray.  Compiled WITHOUT fast-math, like the reference's utils extension (extensions/utils/setup.py), and
// written in the reference's operation order so the outputs agree bit for bit.
// The reference's backward kernel is an empty stub (utils_kernel.cu:53-94) and its Python backward returns
// None for every input (extensions/utils/utils.py:48-50); gb_compute_raydirs_bwd is the same no-op.
#include "common.cuh"

namespace {

__global__ void __launch_bounds__(256) raydirs_fwd_kernel(int N, int H, int W, const float* __restrict__ viewpos,
                                                          const float* __restrict__ viewrot,
                                                          const float2* __restrict__ focal,
                                                          const float2* __restrict__ princpt,
                                                          const float2* __restrict__ pixelcoords, float volradius,
                                                          float* __restrict__ raypos, float* __restrict__ raydir,
                                                          float2* __restrict__ tminmax) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  const int hn = blockIdx.y * blockDim.y + threadIdx.y;
  const int h = hn % H, n = hn / H;
  if (w >= W || n >= N) return;
  const size_t o = ((size_t)n * H + h) * W + w;
  const float3 rp = make_float3(viewpos[3 * n] / volradius, viewpos[3 * n + 1] / volradius, viewpos[3 * n + 2] / volradius);
  const float* R = viewrot + 9 * n;
  float2 pc = pixelcoords ? pixelcoords[o] : make_float2((float)w, (float)h);
  const float2 pp = princpt[n], fc = focal[n];
  pc.x = (pc.x - pp.x) / fc.x;
  pc.y = (pc.y - pp.y) / fc.y;
  // raydir = viewrot0 * x + viewrot1 * y + viewrot2 * 1
  float3 d;
  d.x = R[0] * pc.x + R[3] * pc.y + R[6] * 1.f;
  d.y = R[1] * pc.x + R[4] * pc.y + R[7] * 1.f;
  d.z = R[2] * pc.x + R[5] * pc.y + R[8] * 1.f;
  const float inv = rnorm3df(d.x, d.y, d.z);
  d.x *= inv; d.y *= inv; d.z *= inv;
  const float3 t1 = make_float3((-1.f - rp.x) / d.x, (-1.f - rp.y) / d.y, (-1.f - rp.z) / d.z);
  const float3 t2 = make_float3((1.f - rp.x) / d.x, (1.f - rp.y) / d.y, (1.f - rp.z) / d.z);
  const float tmin = fmaxf(fminf(t1.x, t2.x), fmaxf(fminf(t1.y, t2.y), fminf(t1.z, t2.z)));
  const float tmax = fminf(fmaxf(t1.x, t2.x), fminf(fmaxf(t1.y, t2.y), fmaxf(t1.z, t2.z)));
  raypos[3 * o] = rp.x; raypos[3 * o + 1] = rp.y; raypos[3 * o + 2] = rp.z;
  raydir[3 * o] = d.x; raydir[3 * o + 1] = d.y; raydir[3 * o + 2] = d.z;
  tminmax[o] = make_float2(fmaxf(tmin, 0.f), tmax);
}

}  // namespace

// replaces utilslib.compute_raydirs_forward (extensions/utils/utils.cpp:46-82).  pixelcoords may be NULL.
GB_API int gb_compute_raydirs_fwd(int N, int H, int W, const float* viewpos, const float* viewrot, const float* focal,
                                  const float* princpt, const float* pixelcoords, float volradius, float* raypos,
                                  float* raydir, float* tminmax, void* stream) {
  if (N <= 0 || H <= 0 || W <= 0) return 0;
  dim3 block(32, 8);
  dim3 grid(gb::cdiv(W, 32), gb::cdiv(N * H, 8));
  return gb::launch<raydirs_fwd_kernel>(grid, block, 0, (cudaStream_t)stream, N, H, W, viewpos, viewrot,
                                        (const float2*)focal, (const float2*)princpt, (const float2*)pixelcoords,
                                        volradius, raypos, raydir, (float2*)tminmax);
}

// replaces utilslib.compute_raydirs_backward (utils.cpp:84-132): the reference computes nothing here.
GB_API int gb_compute_raydirs_bwd(void) { return 0; }
