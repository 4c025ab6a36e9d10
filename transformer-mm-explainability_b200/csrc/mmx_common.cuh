// Shared helpers for libmmx (sm_90a only).
#pragma once
#include <utility>
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <atomic>

#include "../../include/mmx.h"

namespace mmx {

void set_error(const std::string& msg);
extern std::atomic<uint64_t> g_launches;
int sm_count();          // SM count of the CURRENT device (cached per device)

// One process may drive several GPUs (ClipEngine(device="cuda:1") after a cuda:0 engine): every piece of cached
// per-device state (function attributes, SM counts, memory-pool settings) is indexed by the device ordinal.
constexpr int MMX_MAX_DEVICES = 64;
inline int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MMX_MAX_DEVICES) dev = 0;
  return dev;
}

// Stream-ordered scratch (cudaMallocAsync) comes from the device's default pool; with the default release threshold (0) the
// pool hands its memory back to the driver at every synchronisation point and the next step pays for real allocations.
// Called once per device by every path that takes such scratch.
inline void keep_stream_scratch_cached() {
  static std::atomic<bool> pool_set[MMX_MAX_DEVICES];
  const int dev = current_device();
  if (pool_set[dev].load(std::memory_order_acquire)) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
    unsigned long long thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  pool_set[dev].store(true, std::memory_order_release);
}

// Programmatic dependent launch (sm_90+): the kernel is launched as a dependent of whatever precedes it in the stream, so
// its launch latency (and any prologue before pdl_wait()) overlaps that kernel's tail.  Every kernel launched this way
// calls pdl_wait() before it touches global memory.  MMX_PDL=0 switches the attribute off (pdl_wait() is then a no-op).
inline bool pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("MMX_PDL"); v = e ? atoi(e) != 0 : 1; }
  return v != 0;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t lc = {};
  lc.gridDim = grid; lc.blockDim = block; lc.dynamicSmemBytes = smem; lc.stream = st;
  lc.attrs = attr; lc.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&lc, kernel, std::forward<Args>(args)...);
}
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif

inline void count_launch(uint64_t n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define MMX_CHECK_CUDA(expr)                                                                     \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      ::mmx::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ +    \
                       ":" + std::to_string(__LINE__) + ")");                                    \
      return 1;                                                                                  \
    }                                                                                            \
  } while (0)

#define MMX_REQUIRE(cond, msg)                                                                   \
  do {                                                                                           \
    if (!(cond)) {                                                                               \
      ::mmx::set_error(std::string("requirement failed: ") + #cond + " - " + (msg));             \
      return 2;                                                                                  \
    }                                                                                            \
  } while (0)

#define MMX_LAUNCH_CHECK()                                                                       \
  do {                                                                                           \
    ::mmx::count_launch();                                                                       \
    cudaError_t _e = cudaPeekAtLastError();                                                      \
    if (_e != cudaSuccess) {                                                                     \
      ::mmx::set_error(std::string("kernel launch: ") + cudaGetErrorString(_e) + " (" +          \
                       __FILE__ + ":" + std::to_string(__LINE__) + ")");                         \
      return 1;                                                                                  \
    }                                                                                            \
  } while (0)

#define MMX_TRY(expr)                                                                            \
  do {                                                                                           \
    int _r = (expr);                                                                             \
    if (_r != 0) return _r;                                                                      \
  } while (0)

__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline int round_up(int a, int b) { return cdiv(a, b) * b; }

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// streaming 128-bit load that does not pollute L1 (data touched once)
__device__ __forceinline__ float4 ld_stream4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float ld_stream1(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Row max and sum of exp(x - max) of a softmax over the n columns of x, in the order torch's warp softmax uses for rows of
// up to 1024 columns: per-lane partials over columns lane, lane + 32, ..., then a butterfly.  Every lane of the warp gets
// both; prob[c] = expf(x[c] - m) / s.
__device__ __forceinline__ void warp_softmax_stats(const float* x, int n, int lane, float& m, float& s) {
  m = -INFINITY;
  for (int c = lane; c < n; c += 32) { const float v = x[c]; m = m > v ? m : v; }
  m = warp_max(m);
  s = 0.f;
  for (int c = lane; c < n; c += 32) s += expf(x[c] - m);
  s = warp_sum(s);
}

// clamp(min=0), min() and max() with torch's NaN semantics (NaN propagates; fmaxf / fminf would drop it): a numerical blow-up
// upstream must reach the caller (and trip the reference's `assert diag(R - I).min() >= 0`) instead of being masked.
__device__ __forceinline__ float relu_nan(float x) { return x < 0.f ? 0.f : x; }
__device__ __forceinline__ float min_nan(float m, float v) { return (v < m || v != v) ? v : m; }
__device__ __forceinline__ float max_nan(float m, float v) { return (v > m || v != v) ? v : m; }

// torch's max(-1) / argmax order (GreaterOrNan): a NaN beats any number, equal values keep the lower index; index -1 is
// "no candidate yet".
__device__ __forceinline__ bool argmax_better(float a, int ia, float b, int ib) {
  if (ib < 0) return ia >= 0;
  if (ia < 0) return false;
  if (a != a) return b != b ? ia < ib : true;
  if (b != b) return false;
  return a > b || (a == b && ia < ib);
}

// Source index of torch's legacy "nearest" resampling (F.interpolate(mode="nearest"), the same rule on CPU and CUDA):
// min(floor(dst * scale), in - 1) with scale = (float)in / (float)out.
__device__ __forceinline__ int nearest_src(int dst, float scale, int in) {
  return min((int)floorf((float)dst * scale), in - 1);
}

// ATen's area_pixel_compute_source_index (align_corners=False, linear): max(scale (dst + 0.5) - 0.5, 0), then the two taps
// and the weight of the second (UpSample.cuh; upsample_bilinear2d_out_frame).  The expression is written as ATen writes it,
// so nvcc contracts it the same way (one fma).
__device__ __forceinline__ void linear_taps(int dst, float scale, int in, int& i0, int& i1, float& l1) {
  const float src = scale * ((float)dst + 0.5f) - 0.5f;
  const float r = src < 0.f ? 0.f : src;
  i0 = (int)r;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = r - (float)i0;
}

__device__ __forceinline__ float act_fwd(float x, int act) {
  switch (act) {
    case MMX_ACT_QUICKGELU: return x / (1.f + expf(-1.702f * x));
    case MMX_ACT_GELU: return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
    case MMX_ACT_RELU: return relu_nan(x);      // F.relu(NaN) = NaN: an overflow upstream stays visible
    case MMX_ACT_TANH: return tanhf(x);
    case MMX_ACT_SIGMOID: return 1.f / (1.f + expf(-x));
    default: return x;
  }
}
__device__ __forceinline__ float act_bwd(float x, int act) {  // d act(x) / dx
  switch (act) {
    case MMX_ACT_QUICKGELU: {
      float s = 1.f / (1.f + expf(-1.702f * x));
      return s + 1.702f * x * s * (1.f - s);
    }
    case MMX_ACT_GELU: {
      float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
      float pdf = 0.39894228040143268f * expf(-0.5f * x * x);
      return cdf + x * pdf;
    }
    case MMX_ACT_RELU: return x <= 0.f ? 0.f : 1.f;   // torch's threshold_backward: a NaN pre passes the gradient
    case MMX_ACT_TANH: { const float t = tanhf(x); return 1.f - t * t; }
    case MMX_ACT_MUL: return x;   // the epilogue multiplies by `pre` itself (Linear.relprop)
    case MMX_ACT_SIGMOID: { const float s = 1.f / (1.f + expf(-x)); return s * (1.f - s); }
    default: return 1.f;
  }
}

}  // namespace mmx
