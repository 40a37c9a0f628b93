// wgmma / TMA / mbarrier / cluster PTX helpers and tensor-map builders shared by the tensor-core kernels
// (linear_tc.cu, fused_layer.cu).  sm_90a.
//
// Both kernels run the same consumer: two warpgroups per CTA, warpgroup w owns rows 64w .. 64w+63 of a 128-row tile
// and keeps its 64 x NP fp32 accumulator in registers (NP / 2 per thread).  NP is the instantiated accumulator width
// (64, 128, 208, 224 or 256): the output width n_pad rounds up to it, the W rows beyond N come from the TMA zero fill.
// Every k-step issues ONE wgmma.mma_async.m64n{NP}k16 per product, and the k-steps of a k-block form one batch (one
// fence, the products back to back, one commit).  Operand tiles are K-major bf16, written by TMA (or by the fused
// kernel's aggregation warps) with SWIZZLE_64B (BK = 32) or SWIZZLE_128B (BK = 64).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"

namespace gr {
namespace tc {

constexpr int BM = 128;          // rows per CTA tile: two consumer warpgroups of 64 rows
constexpr int WG_M = 64;         // rows per consumer warpgroup (wgmma M)
constexpr int MMA_K = 16;

// Grouped K order of a dense ReaRev layer.  The layer input is T = 2I + 1 segments [h | nb_0-> | nb_0<- | nb_1-> | ...]
// of `pitch` columns each.  In grouped order K is walked in G = ceil(pitch / 32) column groups; group g holds the
// 32-column block g of every segment: k-block g*T + t is columns 32g .. 32g+31 of segment seg(t), seg(0) = 0 (h) and
// seg(t) = 1 + 2*((t-1) % I) + (t-1) / I (direction 0 for every instruction, then direction 1).  The W planes of this
// order are [N, G*T*32] bf16 hi/lo, k-block kb at columns 32 kb, zero beyond D inside each block.  When the last group
// of a segment holds 16 columns (ksteps_last == 1) its k-blocks are ONE k-step.  gr_fused_layer and
// gr_linear_tc_planes (GR_LINEAR_K_GROUPED) share this plan, these planes and therefore the fp32 accumulation order
// of every output element.  Defined in fused_layer.cu.
//
// Packed (GR_LINEAR_K_ORDER_PLANES, the A operand in the K-order layout of gr_aggregate_dual_abs_ex): the same k16 steps
// in the same order, with a 16-column last group packed as the h tail (one k-step, W block = 16 columns + 16 zeros)
// followed by I k-blocks of two k-steps, block i = the last group of neighbour slots 2i and 2i+1 (16 columns each).
// (G-1)*T + 1 + I k-blocks instead of G*T; without a 16-column last group the packed planes are the grouped ones.
struct GroupedK {
  int G, ksteps_last, nkb;       // nkb: k-blocks of the walk
  int64_t kp;                    // columns of the W planes: nkb * 32
  size_t w_plane_bytes;
};
GroupedK plan_grouped_k(int64_t pitch, int I, int64_t N_out, bool packed = false);
int grouped_w_split(const float* W, int64_t ldw, int64_t N_out, int D, int I, const GroupedK& k, __nv_bfloat16* hi,
                    __nv_bfloat16* lo, cudaStream_t stream);

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
// 128-byte (BK = 64) or 64-byte (BK = 32) swizzle, zero fill out of bounds.  L2 promotion 128 B: a 64-byte box row
// also brings its neighbour half line into L2, which the next k-block of the same row reads.  At cfg2 the dense-layer
// GEMM (A boxes of 64-byte rows streaming from HBM) takes 0.329 ms with it against 0.347 ms with 256-byte promotion and
// 0.367 ms with none or 64 B (H100 80GB HBM3 at 700 W, bench.py, two alternating runs each).
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
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
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
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] += A[64 x 16] B[N x 16]^T, bf16 operands from shared memory, fp32 accumulate in d[OFF .. OFF + N/2 - 1]
#define GR_ACC8(i) "+f"(d[OFF + (i)]), "+f"(d[OFF + (i) + 1]), "+f"(d[OFF + (i) + 2]), "+f"(d[OFF + (i) + 3]), \
                   "+f"(d[OFF + (i) + 4]), "+f"(d[OFF + (i) + 5]), "+f"(d[OFF + (i) + 6]), "+f"(d[OFF + (i) + 7])
#define GR_ACC32(i) GR_ACC8(i), GR_ACC8((i) + 8), GR_ACC8((i) + 16), GR_ACC8((i) + 24)
#define GR_REGS8 "%0, %1, %2, %3, %4, %5, %6, %7"
#define GR_REGS16 GR_REGS8 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define GR_REGS32 GR_REGS16 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define GR_REGS64 GR_REGS32 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, " \
                  "%49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define GR_REGS104 GR_REGS64 ", %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, " \
                   "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, " \
                   "%99, %100, %101, %102, %103"
#define GR_REGS128 GR_REGS104 ", %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, " \
                   "%117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
// REGS: the accumulator operands %0 .. %(N/2 - 1); the descriptors follow them as operands RA and RB
#define GR_WGMMA(N, REGS, RA, RB, ...)                                                                   \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"                                          \
               "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 {" REGS "}, %" #RA ", %" #RB  \
               ", p, 1, 1, 0, 0;\n\t}"                                                                   \
               : __VA_ARGS__                                                                             \
               : "l"(a), "l"(b))
template <int N, int OFF, int R>
__device__ __forceinline__ void wgmma_bf16(float (&d)[R], uint64_t a, uint64_t b) {
  static_assert(OFF + N / 2 <= R, "accumulator range");
  if constexpr (N == 16) {
    GR_WGMMA(16, GR_REGS8, 8, 9, GR_ACC8(0));
  } else if constexpr (N == 32) {
    GR_WGMMA(32, GR_REGS16, 16, 17, GR_ACC8(0), GR_ACC8(8));
  } else if constexpr (N == 64) {
    GR_WGMMA(64, GR_REGS32, 32, 33, GR_ACC32(0));
  } else if constexpr (N == 128) {
    GR_WGMMA(128, GR_REGS64, 64, 65, GR_ACC32(0), GR_ACC32(32));
  } else if constexpr (N == 208) {
    GR_WGMMA(208, GR_REGS104, 104, 105, GR_ACC32(0), GR_ACC32(32), GR_ACC32(64), GR_ACC8(96));
  } else {
    static_assert(N == 256, "instruction widths: 16, 32, 64, 128, 208, 256");
    GR_WGMMA(256, GR_REGS128, 128, 129, GR_ACC32(0), GR_ACC32(32), GR_ACC32(64), GR_ACC32(96));
  }
}
#undef GR_WGMMA
#undef GR_REGS128
#undef GR_REGS104
#undef GR_REGS64
#undef GR_REGS32
#undef GR_REGS16
#undef GR_REGS8
#undef GR_ACC32
#undef GR_ACC8

// one product over the NP accumulator columns: instructions of NI columns from column C0 on (the last one takes
// what is left), W rows C0 .. of the tile with BK*2-byte rows
template <int NP, int NI, int BK, int C0 = 0>
__device__ __forceinline__ void wgmma_product(float (&acc)[NP / 2], uint64_t a, uint64_t b) {
  constexpr int n = NP - C0 < NI ? NP - C0 : NI;
  wgmma_bf16<n, C0 / 2>(acc, a, b + (uint64_t)((C0 * BK * 2) >> 4));
  if constexpr (C0 + n < NP) wgmma_product<NP, NI, BK, C0 + n>(acc, a, b);
}

// One k-block of the 3-product split-bf16 contraction (or, SINGLE, the one product A_hi W_hi) for one consumer
// warpgroup: acc += A[64 rows, KSTEPS*16] W[NP rows, KSTEPS*16]^T.  `da_*` / `dw_*` are descriptors of the k-block's
// first column; the W tile holds NP rows of BK*2 bytes.  Each product is ONE m64n{NP}k16 instruction (NI = NP), or,
// where the kernel's register budget cannot hold the accumulator as one instruction operand, NP / NI instructions of
// NI columns (plus one for the rest).  KSTEPS and SINGLE are template parameters so that the batch is straight-line
// code: a runtime condition between two wgmma instructions makes ptxas wait for the accumulator (C7519) and split
// the batch.
template <int NP, int BK, int KSTEPS, bool SINGLE, int NI = NP>
__device__ __forceinline__ void mma_kblock(float (&acc)[NP / 2], uint64_t da_hi, uint64_t da_lo, uint64_t dw_hi,
                                           uint64_t dw_lo) {
  static_assert(KSTEPS >= 1 && KSTEPS <= BK / MMA_K, "k-steps of one k-block");
  acc_fence(acc);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k) {
    const uint64_t adv = (uint64_t)((k * MMA_K * 2) >> 4);          // +32 B per K step inside the swizzle row
    wgmma_product<NP, NI, BK>(acc, da_hi + adv, dw_hi + adv);
    if (!SINGLE) {
      wgmma_product<NP, NI, BK>(acc, da_hi + adv, dw_lo + adv);
      wgmma_product<NP, NI, BK>(acc, da_lo + adv, dw_hi + adv);
    }
  }
  wgmma_commit();
  acc_fence(acc);
}

// Epilogue helpers.  Accumulator fragment of thread (warp w of the warpgroup, lane l), element i of float[NP / 2]:
// row 16w + l/4 + 8*((i >> 1) & 1), column 8*(i >> 2) + 2*(l % 4) + (i & 1) (m64nN is the concatenation of its
// 8-column blocks), so the 16-column half q of the tile is elements 8q .. 8q+7.
struct EpiOut {
  const float* bias;        // [256] in shared memory, zero padded
  const float* w_score;     // [256] in shared memory, zero padded
  bool relu;
};

// bias + relu + score dot of 16-column half `q` (columns c0 = 16q .. 16q+15): v[0..7] = columns c0 + (0 | 8) + 2c +
// {0,1}, rows r (v[0,1], v[4,5]) and r + 8 (v[2,3], v[6,7]); dot0 / dot1 accumulate the score dot of rows r / r + 8
template <int R>
__device__ __forceinline__ void epi_values(const float (&a)[R], int q, int cq, const EpiOut& e, float (&v)[8],
                                           float& dot0, float& dot1) {
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const int col = 16 * q + 8 * b + 2 * cq;
    const float2 bb = *reinterpret_cast<const float2*>(e.bias + col);
    const float2 ww = *reinterpret_cast<const float2*>(e.w_score + col);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float x = a[8 * q + 4 * b + i] + ((i & 1) ? bb.y : bb.x);
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

// Launches a warp-specialised kernel as `grid` CTAs of `threads` threads in clusters of `cs` along x.  The kernel is
// opted in to 227 KB of dynamic shared memory once per device, and refused unless it was compiled with exactly
// `launch_regs` registers per thread: setmaxnreg only redistributes the registers the CTA was launched with, so the
// warpgroups' budgets add up to exactly threads x launch_regs.  Errors are reported as `fn`.
template <auto Kernel, typename... Args>
int launch_cluster(const char* fn, int launch_regs, int cs, int grid, int threads, size_t smem, cudaStream_t stream,
                   const Args&... args) {
  if (int rc = opt_in_smem<Kernel>(fn, 227 * 1024)) return rc;
  static int num_regs = 0;   // one per Kernel
  if (num_regs == 0) {
    cudaFuncAttributes fa{};
    GR_CHECK_CUDA_AS(fn, cudaFuncGetAttributes(&fa, Kernel));
    num_regs = fa.numRegs;
  }
  if (num_regs != launch_regs) {
    set_error("%s: kernel was compiled with %d registers per thread, the warpgroup budget needs %d", fn, num_regs,
              launch_regs);
    return GR_ERR_UNSUPPORTED;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3((unsigned)threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  GR_CHECK_CUDA_AS(fn, cudaLaunchKernelEx(&cfg, Kernel, args...));
  return GR_OK;
}

}  // namespace tc
}  // namespace gr
