// Shared helpers for libgnnrag_b200.so (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/gnnrag_b200.h"

namespace gr {

constexpr int kNumSMs = 132;  // H100 SXM

void set_error(const char* fmt, ...);

#define GR_CHECK_ARG(cond, msg)                                                     \
  do {                                                                              \
    if (!(cond)) {                                                                  \
      gr::set_error("%s: invalid argument: %s", __func__, msg);                     \
      return GR_ERR_INVALID_ARG;                                                    \
    }                                                                               \
  } while (0)

#define GR_CHECK_CUDA(expr)                                                         \
  do {                                                                              \
    cudaError_t _e = (expr);                                                        \
    if (_e != cudaSuccess) {                                                        \
      gr::set_error("%s: CUDA error %s at %s:%d", __func__, cudaGetErrorString(_e), \
                    __FILE__, __LINE__);                                            \
      return GR_ERR_CUDA;                                                           \
    }                                                                               \
  } while (0)

#define GR_CHECK_LAUNCH() GR_CHECK_CUDA(cudaGetLastError())

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// number of SMs of the current device (132 on H100 SXM); cached
int sm_count();

// true the first time it is called for (flag array, current device): kernel attributes such as the dynamic
// shared-memory opt-in are per device, a process may drive several
inline bool first_use_on_device(bool (&done)[64]) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
  if (done[dev]) return false;
  done[dev] = true;
  return true;
}

// element-wise fp32x2 fma / mul, rounded to nearest like the scalar instructions they expand to
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }

// Bitonic network with all comparators ascending (virtual +inf padding beyond n): sorts arbitrary n.  The whole
// block calls it; `a` is shared or global memory.
template <typename T>
__device__ void bitonic_sort_block(T* a, int n) {
  for (int k = 2; (k >> 1) < n; k <<= 1) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      int l = i ^ (k - 1);
      if (l > i && l < n) {
        T x = a[i], y = a[l];
        if (x > y) { a[i] = y; a[l] = x; }
      }
    }
    __syncthreads();
    for (int j = k >> 2; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        int l = i ^ j;
        if (l > i && l < n) {
          T x = a[i], y = a[l];
          if (x > y) { a[i] = y; a[l] = x; }
        }
      }
      __syncthreads();
    }
  }
}

}  // namespace gr
