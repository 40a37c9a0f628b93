// wgmma / TMA / mbarrier / cluster PTX helpers and tensor-map builders shared by the tensor-core kernels
// (linear_tc.cu, fused_layer.cu).  sm_90a.
//
// Both kernels run the same consumer: two warpgroups per CTA, warpgroup w owns rows 64w .. 64w+63 of a 128-row tile
// and keeps its 64 x n_pad fp32 accumulator in registers as n_pad / 32 chunks of m64n32 (plus one m64n16 chunk when
// n_pad % 32 == 16).  Operand tiles are K-major bf16, written by TMA (or by the fused kernel's aggregation warps) with
// SWIZZLE_64B (BK = 32) or SWIZZLE_128B (BK = 64).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"

namespace gr {
namespace tc {

constexpr int BM = 128;          // rows per CTA tile: two consumer warpgroups of 64 rows
constexpr int WG_M = 64;         // rows per consumer warpgroup (wgmma M)
constexpr int MMA_K = 16;
constexpr int kMaxChunks = 8;    // 32-column accumulator chunks: n_pad <= 256

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D bf16 row-major [rows, cols] (row stride ld elements) -> tensor map with box {BK cols, box_rows},
// 128-byte (BK = 64) or 64-byte (BK = 32) swizzle, zero fill out of bounds.
inline bool make_tmap(CUtensorMap* m, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows,
               int bk) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// Output tensor map: row-major [rows, cols] of `elem_bytes`-wide elements, box {16 cols, 64 rows}, no swizzle
// (each consumer warpgroup stages 64x16 chunks densely in smem and TMA-stores them; out-of-range rows/cols are clipped).
inline bool make_out_tmap(CUtensorMap* m, const void* base, int64_t rows, int64_t cols, int64_t ld, int elem_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return false;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld * elem_bytes) % 16 != 0) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * elem_bytes};
  cuuint32_t box[2] = {16u, (cuuint32_t)WG_M};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                  const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// ---------------------------------------------------------------------------------------------------
// PTX helpers
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive on the barrier at the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// a consumer warp is done with a ring slot: with W multicast (CS = 2) the slot is refilled by both CTAs' producers,
// so the release goes to the barrier of every CTA of the cluster
template <int CS>
__device__ __forceinline__ void release_slot(uint64_t* bar) {
  if (CS == 1) {
    mbar_arrive(bar);
  } else {
#pragma unroll
    for (int r = 0; r < CS; ++r) mbar_arrive_cluster(bar, (uint32_t)r);
  }
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_mc(void* dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                               int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5}], [%2], %3;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

// wgmma shared-memory descriptor of a K-major swizzled operand tile whose rows are BK*2 bytes (= the swizzle span):
// 8-row groups are 8*BK*2 bytes apart (SBO), LBO unused (=1), layout SWIZZLE_128B (1) / SWIZZLE_64B (2).  The tile
// base must be aligned to the swizzle pattern (8 rows); a K step of 16 elements adds 32 bytes to the start address.
template <int BK>
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((8 * BK * 2) >> 4) << 32;
  d |= (uint64_t)(BK == 64 ? 1 : 2) << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator accesses across the asynchronous wgmma window
__device__ __forceinline__ void acc_fence(float (&d)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 32] += A[64 x 16] B[32 x 16]^T, bf16 operands from shared memory, fp32 accumulate
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b));
}
// the same for a 16-column chunk: D[64 x 16] in d[0 .. 7]
__device__ __forceinline__ void wgmma_n16(float (&d)[16], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b));
}

// One k-block of the 3-product split-bf16 contraction (or the single product A_hi W_hi) for one consumer warpgroup:
// acc[j] += A[64 rows, ksteps*16] W[32j .. 32j+31, ksteps*16]^T for j < nc.  `da_*` / `dw_*` are descriptors of the
// k-block's first column; the W tile holds n_pad rows of BK*2 bytes.  NC (template) sizes the register accumulator,
// nc <= NC chunks are live, `tail16`: chunk nc - 1 has 16 columns.
template <int NC, int BK>
__device__ __forceinline__ void mma_kblock(float (&acc)[NC][16], uint64_t da_hi, uint64_t da_lo, uint64_t dw_hi,
                                           uint64_t dw_lo, int ksteps, int nc, bool single, bool tail16) {
  constexpr uint64_t kChunkAdv = (uint64_t)((32 * BK * 2) >> 4);     // 32 W rows
#pragma unroll
  for (int j = 0; j < NC; ++j) acc_fence(acc[j]);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < BK / MMA_K; ++k) {
    if (k < ksteps) {
      const uint64_t adv = (uint64_t)((k * MMA_K * 2) >> 4);        // +32 B per K step inside the swizzle row
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        if (j >= nc) continue;
        const uint64_t wh = dw_hi + j * kChunkAdv + adv, wl = dw_lo + j * kChunkAdv + adv;
        if (j == nc - 1 && tail16) {
          wgmma_n16(acc[j], da_hi + adv, wh);
          if (!single) {
            wgmma_n16(acc[j], da_hi + adv, wl);
            wgmma_n16(acc[j], da_lo + adv, wh);
          }
        } else {
          wgmma_n32(acc[j], da_hi + adv, wh);
          if (!single) {
            wgmma_n32(acc[j], da_hi + adv, wl);
            wgmma_n32(acc[j], da_lo + adv, wh);
          }
        }
      }
    }
  }
  wgmma_commit();
#pragma unroll
  for (int j = 0; j < NC; ++j) acc_fence(acc[j]);
}

// Epilogue helpers.  Accumulator fragment of thread (warp w of the warpgroup, lane l), chunk j, element i:
// row 16w + l/4 + 8*((i >> 1) & 1), column 32j + 8*(i >> 2) + 2*(l % 4) + (i & 1).
struct EpiOut {
  const float* bias;        // [256] in shared memory, zero padded
  const float* w_score;     // [256] in shared memory, zero padded
  bool relu;
};

// bias + relu + score dot of 16-column half `h` of chunk j: v[0..7] = columns (8*(2h) | 8*(2h+1)) + 2c + {0,1}, rows
// r (v[0,1], v[4,5]) and r + 8 (v[2,3], v[6,7]); dot0 / dot1 accumulate the score dot of rows r / r + 8
__device__ __forceinline__ void epi_values(const float (&a)[16], int h, int c0, int cq, const EpiOut& e, float (&v)[8],
                                           float& dot0, float& dot1) {
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const int col = c0 + 8 * b + 2 * cq;
    const float2 bb = *reinterpret_cast<const float2*>(e.bias + col);
    const float2 ww = *reinterpret_cast<const float2*>(e.w_score + col);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float x = a[8 * h + 4 * b + i] + ((i & 1) ? bb.y : bb.x);
      if (e.relu) x = fmaxf(x, 0.f);
      v[4 * b + i] = x;
    }
    dot0 = fmaf(v[4 * b + 0], ww.x, dot0); dot0 = fmaf(v[4 * b + 1], ww.y, dot0);
    dot1 = fmaf(v[4 * b + 2], ww.x, dot1); dot1 = fmaf(v[4 * b + 3], ww.y, dot1);
  }
}

__device__ __forceinline__ uint32_t split_hi_lo(float x0, float x1, uint32_t& lo) {
  const __nv_bfloat162 h2 = __floats2bfloat162_rn(x0, x1);
  const float2 hf = __bfloat1622float2(h2);
  const __nv_bfloat162 l2 = __floats2bfloat162_rn(x0 - hf.x, x1 - hf.y);
  lo = *reinterpret_cast<const uint32_t*>(&l2);
  return *reinterpret_cast<const uint32_t*>(&h2);
}

// staged epilogue of one 64 x 16 chunk (columns c0 .. c0+15) of a warpgroup: values -> dense smem staging
// {fp32 64x16, hi 64x16, lo 64x16} -> TMA stores by one thread (clipping rows >= M and columns beyond the map).
constexpr int kStageOutBytes = WG_M * 16 * 4 + 2 * WG_M * 16 * 2;   // 8 KB per warpgroup
__device__ __forceinline__ void epi_store_tma(const float (&v)[8], uint8_t* stg, int r, int cq, bool issuer,
                                              int bar_id, const CUtensorMap* map_c, const CUtensorMap* map_hi,
                                              const CUtensorMap* map_lo, bool has_c, bool has_planes, int c0, int m0) {
  if (issuer) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // previous chunk's stores read stg
  named_bar_sync(bar_id, 128);
  float* s_c = reinterpret_cast<float*>(stg);
  uint32_t* s_h = reinterpret_cast<uint32_t*>(stg + WG_M * 16 * 4);
  uint32_t* s_l = reinterpret_cast<uint32_t*>(stg + WG_M * 16 * 4 + WG_M * 16 * 2);
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const int col = 8 * b + 2 * cq;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int row = r + 8 * hr;
      const float x0 = v[4 * b + 2 * hr], x1 = v[4 * b + 2 * hr + 1];
      if (has_c) *reinterpret_cast<float2*>(s_c + row * 16 + col) = make_float2(x0, x1);
      if (has_planes) {
        uint32_t lo;
        const uint32_t hi = split_hi_lo(x0, x1, lo);
        s_h[row * 8 + col / 2] = hi;
        s_l[row * 8 + col / 2] = lo;
      }
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  named_bar_sync(bar_id, 128);
  if (issuer) {
    if (has_c) tma_store_2d(map_c, stg, c0, m0);
    if (has_planes) {
      tma_store_2d(map_hi, stg + WG_M * 16 * 4, c0, m0);
      tma_store_2d(map_lo, stg + WG_M * 16 * 4 + WG_M * 16 * 2, c0, m0);
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
}

// score dot of rows r and r + 8 summed over the 4 lanes that share them; lane cq == 0 writes dots[row], dots[M + row]
__device__ __forceinline__ void epi_dots(float dot0, float dot1, float* dots, int64_t row0, int64_t M, int cq) {
  dot0 += __shfl_xor_sync(0xffffffffu, dot0, 1);
  dot0 += __shfl_xor_sync(0xffffffffu, dot0, 2);
  dot1 += __shfl_xor_sync(0xffffffffu, dot1, 1);
  dot1 += __shfl_xor_sync(0xffffffffu, dot1, 2);
  if (dots && cq == 0) {
    if (row0 < M) { dots[row0] = dot0; dots[M + row0] = 0.f; }
    if (row0 + 8 < M) { dots[row0 + 8] = dot1; dots[M + row0 + 8] = 0.f; }
  }
}

}  // namespace tc
}  // namespace gr
