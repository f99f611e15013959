// goliath_b200/csrc/common.cuh — shared device/host helpers for the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <mutex>
#include <utility>

#define GB_API extern "C" __attribute__((visibility("default")))

// Every C-ABI entry point returns 0 or a cudaError_t value (never throws, never allocates).  Variadic so that a
// template argument list with commas passes through: GB_CUDA(gb::launch<k<4, false>>(...)).
#define GB_CUDA(...)                               \
  do {                                             \
    const int e__ = (int)(__VA_ARGS__);            \
    if (e__ != 0) return e__;                      \
  } while (0)

namespace gb {

// number of kernel launches issued by this library (bench.py reports it as gpu_launches)
extern unsigned long long g_launch_count;

constexpr int kNumSMs = 132;  // H100 SXM
constexpr int kMaxDevices = 64;

// Every kernel of the library is launched through here: Kernel<<<grid, block, smem, stream>>>(args...).
// Without an opt-in a kernel's dynamic shared memory is limited to 48 KB less its static shared memory.  The opt-in
// applies to the current device: it is made once per (kernel, device) for any dynamic shared memory and raised when a
// later call asks for more.  Returns cudaGetLastError(); only a launch that succeeded is counted in g_launch_count.
template <auto Kernel, class... Args>
[[nodiscard]] cudaError_t launch(dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  if (smem > 0) {
    static std::atomic<size_t> granted[kMaxDevices];
    static std::mutex mu;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
    if (granted[dev].load(std::memory_order_acquire) < smem) {
      std::lock_guard<std::mutex> lock(mu);
      if (granted[dev].load(std::memory_order_relaxed) < smem) {
        e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        granted[dev].store(smem, std::memory_order_release);
      }
    }
  }
  Kernel<<<grid, block, smem, stream>>>(std::forward<Args>(args)...);
  const cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) __atomic_fetch_add(&g_launch_count, 1ull, __ATOMIC_RELAXED);
  return e;
}

__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// no-return global float add (RED): one L2 atomic-ALU op, no round trip
__device__ __forceinline__ void red_add(float* addr, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}

// streaming loads/stores that do not pollute L1
__device__ __forceinline__ float4 ld_nc_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

// cp.async (LDGSTS) 4/8/16-byte global->shared copies
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem, const void* gmem) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// torch's upsample_bilinear2d source index (align_corners=False, no scale factor): src = in/out * (dst + 0.5) - 0.5 in
// fp32, clamped at 0; i0 = floor, i1 = i0 + 1 except at the last input index, l1 = src - i0.  `scale` is in/out.
struct ResizeTap {
  int i0, i1;
  float l0, l1;
};

__device__ __forceinline__ ResizeTap resize_tap(int dst, float scale, int n_in) {
  float s = scale * ((float)dst + 0.5f) - 0.5f;
  s = s < 0.f ? 0.f : s;
  ResizeTap t;
  t.i0 = (int)s;
  t.i1 = t.i0 + (t.i0 < n_in - 1 ? 1 : 0);
  t.l1 = s - (float)t.i0;
  t.l0 = 1.f - t.l1;
  return t;
}

// weight of input index `i` in an output index's taps (both taps count when they coincide at the border)
__device__ __forceinline__ float resize_tap_weight(const ResizeTap& t, int i) {
  return (t.i0 == i ? t.l0 : 0.f) + (t.i1 == i ? t.l1 : 0.f);
}

// range of output indices whose taps can reach input index i (a superset; resize_tap_weight decides)
__device__ __forceinline__ void resize_footprint(int i, float scale, int n_out, int& lo, int& hi) {
  lo = max(0, (int)floorf(((float)i - 0.5f) / scale - 0.5f) - 2);
  hi = min(n_out - 1, (int)ceilf(((float)i + 1.5f) / scale - 0.5f) + 2);
}

}  // namespace gb
