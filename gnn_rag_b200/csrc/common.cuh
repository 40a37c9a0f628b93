// Shared helpers for libgnnrag_b200.so (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <type_traits>

#include "../../include/gnnrag_b200.h"

namespace gr {

constexpr int kNumSMs = 132;  // H100 SXM

void set_error(const char* fmt, ...);

// The checks report the function they are written in; the _AS forms report `name` instead, so that a launcher
// shared by several entry points reports the entry point that called it.
#define GR_CHECK_ARG_AS(name, cond, msg)                                            \
  do {                                                                              \
    if (!(cond)) {                                                                  \
      gr::set_error("%s: invalid argument: %s", name, msg);                         \
      return GR_ERR_INVALID_ARG;                                                    \
    }                                                                               \
  } while (0)
#define GR_CHECK_ARG(cond, msg) GR_CHECK_ARG_AS(__func__, cond, msg)

#define GR_CHECK_CUDA_AS(name, expr)                                                \
  do {                                                                              \
    cudaError_t _e = (expr);                                                        \
    if (_e != cudaSuccess) {                                                        \
      gr::set_error("%s: CUDA error %s at %s:%d", name, cudaGetErrorString(_e),     \
                    __FILE__, __LINE__);                                            \
      return GR_ERR_CUDA;                                                           \
    }                                                                               \
  } while (0)
#define GR_CHECK_CUDA(expr) GR_CHECK_CUDA_AS(__func__, expr)

#define GR_CHECK_LAUNCH_AS(name) GR_CHECK_CUDA_AS(name, cudaGetLastError())
#define GR_CHECK_LAUNCH() GR_CHECK_CUDA(cudaGetLastError())

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// number of SMs of the current device (132 on H100 SXM); cached
int sm_count();

// Raises Kernel's dynamic shared-memory limit to `bytes` once per (Kernel, device): the attribute is per device and a
// process may drive several.  Keyed on the kernel itself, not its type, so kernels with the same signature keep
// separate flags.
template <auto Kernel>
int opt_in_smem(const char* fn, int bytes) {
  static bool done[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < 64) {
    if (done[dev]) return GR_OK;
    done[dev] = true;
  }
  GR_CHECK_CUDA_AS(fn, cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return GR_OK;
}

// GR_ERR_WORKSPACE unless `ws` is non-null and holds `need` bytes
static inline int check_workspace(const char* fn, const void* ws, size_t have, size_t need) {
  if (ws && have >= need) return GR_OK;
  set_error("%s: workspace too small (%zu < %zu)", fn, have, need);
  return GR_ERR_WORKSPACE;
}

// element-wise fp32x2 fma / mul, rounded to nearest like the scalar instructions they expand to
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}

// Node-sized training tensors ([B*N, D] outputs and their gradients) are fp32 or, under torch.autocast(bfloat16),
// bf16 (GR_IO_BF16).  A bf16 load widens exactly and a bf16 store rounds the fp32 value to nearest even; the kernels
// do the same fp32 operations in between for both types.
__device__ __forceinline__ float ldg_node(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ldg_node(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }
__device__ __forceinline__ float ld_node(const float* p) { return *p; }
__device__ __forceinline__ float ld_node(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ void st_node(float* p, float v) { *p = v; }
__device__ __forceinline__ void st_node(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// the io flags word of the *_ex entry points: only GR_IO_BF16 is defined
static inline bool io_bf16(uint32_t io) { return (io & GR_IO_BF16) != 0; }

static inline int check_io(const char* fn, uint32_t io) {
  GR_CHECK_ARG_AS(fn, (io & ~GR_IO_BF16) == 0, "unknown io flags");
  return GR_OK;
}

// ---- host dispatch: a runtime value selects a template instance.  f receives it as a std::integral_constant (use
// decltype(x)::value) or, in with_node_type, as a type_tag (use typename decltype(t)::type); the helper returns
// what f returns.
template <int V>
using int_c = std::integral_constant<int, V>;
template <typename T>
struct type_tag {
  using type = T;
};

// columns per lane of the warp-per-row kernels (column c = lane + 32 k, k < nc): D <= 512
static inline int nc_for(int D) { return D <= 32 ? 1 : D <= 64 ? 2 : D <= 128 ? 4 : D <= 256 ? 8 : 16; }

template <typename F>
auto with_nc(int D, F&& f) {
  switch (nc_for(D)) {
    case 1: return f(int_c<1>{});
    case 2: return f(int_c<2>{});
    case 4: return f(int_c<4>{});
    case 8: return f(int_c<8>{});
    default: return f(int_c<16>{});
  }
}

// instructions per launch, 1..4 (anything above 4 takes 4)
template <typename F>
auto with_ni(int I, F&& f) {
  switch (I) {
    case 1: return f(int_c<1>{});
    case 2: return f(int_c<2>{});
    case 3: return f(int_c<3>{});
    default: return f(int_c<4>{});
  }
}

// element type of the node-sized tensors: float, or __nv_bfloat16 under GR_IO_BF16
template <typename F>
auto with_node_type(uint32_t io, F&& f) {
  if (io_bf16(io)) return f(type_tag<__nv_bfloat16>{});
  return f(type_tag<float>{});
}

// ---- in-kernel dropout ----------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11) with key = the 64-bit seed and counter (c0, c1, c2, c3); returns the first output
// word.  A kernel's dropout keys each element by its own counter layout (documented at its entry point).
__device__ __forceinline__ uint32_t philox4x32_10_x0(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2,
                                                     uint32_t c3) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}

// an element survives dropout with probability 1 - p:  u = (x >> 8) * 2^-24 in [0, 1), kept iff u >= p
__device__ __forceinline__ bool philox_keep(uint32_t x, float p) {
  return (float)(x >> 8) * 5.9604644775390625e-8f >= p;
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

// ---- fixed-window segmented sums (the deterministic backward kernels) ---------------------------------------------
// A list of L entries sorted by segment (relation, question) is cut into windows of W consecutive entries, W a
// compile-time constant.  One warp per window adds each segment's entries in list order, starting from 0
// (__fadd_rn, so the order written is the order computed).  A segment that lies inside one window is owned by it:
// the warp adds its sum to the output row.  A segment that crosses a window edge leaves one partial per window it
// touches, in `part` [windows][2][width]: slot 0 holds the partial of the window's first segment, slot 1 that of its
// last; segwin_combine_kernel then sums those partials in window order and adds the total to the output row.  Every
// output element is therefore  out + ((p_first + p_next) + ... + p_last)  with the windows fixed by the data and W
// alone: no atomics, and nothing depends on the grid or on which block runs first.

// where the partial of segment `seg` of window [a, b) goes: -1 = the window owns it (add to the output row), else
// its slot in `part`.  `first`: seg is the window's first segment.
template <typename SegOf>
__device__ __forceinline__ int segwin_slot(int64_t a, int64_t b, int64_t L, int64_t seg, bool first, SegOf seg_of) {
  const bool before = first && a > 0 && seg_of(a - 1) == seg;
  const bool after = b < L && seg_of(b) == seg;
  return (before || after) ? (first ? 0 : 1) : -1;
}

// store one warp's NC-columns-per-lane partial (column c = lane + 32 k, c < D): out_row += acc or part_row = acc
template <int NC>
__device__ __forceinline__ void segwin_store(const float (&acc)[NC], int slot, float* part_row, float* out_row,
                                             int D) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const int c = lane + 32 * k;
    if (c < D) {
      if (slot < 0) out_row[c] = __fadd_rn(out_row[c], acc[k]);
      else part_row[c] = acc[k];
    }
  }
}

// one thread per (segment, column): segments that cross a window edge.  Segment s spans list entries
// [seg_ptr[s], seg_ptr[s + 1]), or [s * seg_len, (s + 1) * seg_len) without seg_ptr.  out[s * ld_out + c] +=.
template <int W>
__global__ void segwin_combine_kernel(const float* __restrict__ part, int64_t width, const int32_t* __restrict__ seg_ptr,
                                      int64_t seg_len, int64_t nseg, float* __restrict__ out, int64_t ld_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nseg * width) return;
  const int64_t s = i / width, c = i % width;
  const int64_t beg = seg_ptr ? seg_ptr[s] : s * seg_len, end = seg_ptr ? seg_ptr[s + 1] : beg + seg_len;
  if (end <= beg) return;
  const int64_t ws = beg / W, we = (end - 1) / W;
  if (ws == we) return;
  float v = part[(ws * 2 + (beg == ws * W ? 0 : 1)) * width + c];
#pragma unroll 8
  for (int64_t w = ws + 1; w <= we; ++w) v = __fadd_rn(v, part[w * 2 * width + c]);
  out[s * ld_out + c] = __fadd_rn(out[s * ld_out + c], v);
}

// bytes of `part` for a list of up to L entries and `width` floats per segment row
static inline size_t segwin_part_bytes(int64_t L, int64_t width, int W) {
  return align_up((size_t)2 * (size_t)ceil_div(L > 0 ? L : 1, W) * (size_t)width * sizeof(float), 256);
}

}  // namespace gr
