// Aggregation kernel for the ReaRev hot shape (both directions, bf16-plane output), |v| variant.
//
// Same math and same CSR / tile decomposition as aggregate.cu (reference: ReasonGNNLayer.reason_layer /
// reason_layer_inv, gnn/modules/kg_reasoning/reasongnn.py:61-116), restructured around what the ncu source view of
// that kernel showed (profiles/README.md): at 333 warp instructions per (row, direction) only a third were the
// FFMA2s that do the work -- 14 % were FMNMX (relu of every gathered table element; 24 % of the stall samples) and
// ~38 % were address / predicate / loop scaffolding.
//
//   * relu(v) = (v + |v|) / 2, and |.| is a free source modifier of FFMA.
//     The edge loop accumulates  S = sum c*v  and  Q = sum c*|v|  -- 8 FFMA2 per gathered edge and lane, no FMNMX --
//     and the epilogue uses  sum c*relu(v) = (Q+S)/2,  sum c*relu(-v) = (Q-S)/2  (the 1/2 is folded into the staged
//     relu(+-ins)).  If every v of a row is >= 0 the two chains execute bit-identical operations, so Q-S == 0 exactly
//     (and Q+S == 0 exactly if every v <= 0): exact zeros stay exact zeros.
//     (First attempt, kept in the history: pre-split tables relu(P) | relu(-P).  It doubles the gathered bytes and the
//     gather is L2-bandwidth bound: 250 us instead of 154 us.)
//   * the table is copied once per layer to a 256-column zero-padded layout (gr_pad_table256, 1 KB rows): every
//     lane is in-bounds, so the loop has no clamping or predication, one 64-bit address per gathered edge and the
//     second column chunk is an immediate (+512 B) off it.
//   * ncu on the first version of this file (profiles/): l1tex__data_pipe_lsu_wavefronts at 76 % -- the LSU data pipe
//     (one 128-byte wavefront per clock per SM) was the limiter, with 40 of 115 wavefronts per (row, direction) spent
//     re-reading relu(+-ins) from shared memory, 36 on the gather (two padded 512-byte chunks per edge, odd rows
//     padded to an even edge count) and 16 on the stores.  Hence: relu(+-ins)/2 is staged in shared memory once per
//     tile but held in REGISTERS while a warp stays inside one question; the second column chunk is loaded only by the
//     lanes that own real columns (3 wavefronts instead of 4); edges are taken two at a time with an unpadded
//     single-edge tail.
//   * output: the split-bf16 planes of the e2e GEMM's A operand, segment pitch SEGP (32-byte sectors, see
//     aggregate.cu); columns D..SEGP-1 receive exact zeros (staged ins are zero there).  With GR_AGG_K_ORDER (template
//     flag KO of every kernel) the same values go to the K-order layout of the dense layer's GEMM (ko_lane).
#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace gr {

int g_opt_agg_abs_ws = 2;     // gr_set_option("agg_abs_ws", 0|1|2|3): kernel variant when a tile counter is given, see launch_pn

namespace {

constexpr int kRows = 64;         // destination rows per CTA tile
constexpr int kThreads = 256;     // consumer threads
constexpr int kWarps = kThreads / 32;
constexpr int kEdgeCap = 1024;    // staged edges per direction per tile; the rest takes the slow path
constexpr int kPnCols = 256;      // padded table width
constexpr int kPnRowBytes = kPnCols * 4;

struct PnDir {
  const int32_t* rowptr;
  const int32_t* src;
  const int32_t* rel;
  const float* w;
  const float* pn;      // [R1][256] zero-padded relation table
};

struct PnParams {
  PnDir dir[2];
  const float* prior;
  const float* ins;     // [B, I, D]
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  int64_t ld, out_col0, Nt;
  int B, N, I, j0;
  int32_t* tile_counter;   // persistent kernel: dynamic tile scheduler (zeroed before the launch)
  int64_t table_rows;      // rows of each padded relation table (R1); > 0 enables the staged-row variant (agg_abs_ws 3)
};

__device__ __forceinline__ float4 ldg4(const char* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }

__device__ __forceinline__ void fma4(float4& acc, float c, const float4& v) {          // acc += c * v
  const float2 cc = make_float2(c, c);
  const float2 lo = ffma2(cc, make_float2(v.x, v.y), make_float2(acc.x, acc.y));
  const float2 hi = ffma2(cc, make_float2(v.z, v.w), make_float2(acc.z, acc.w));
  acc = make_float4(lo.x, lo.y, hi.x, hi.y);
}
__device__ __forceinline__ void fma4_abs(float4& acc, float c, const float4& v) {      // acc += c * |v|
  const float2 cc = make_float2(c, c);
  const float2 lo = ffma2(cc, make_float2(fabsf(v.x), fabsf(v.y)), make_float2(acc.x, acc.y));
  const float2 hi = ffma2(cc, make_float2(fabsf(v.z), fabsf(v.w)), make_float2(acc.z, acc.w));
  acc = make_float4(lo.x, lo.y, hi.x, hi.y);
}

__device__ __forceinline__ float4 addsub4(const float4& q, const float4& s, float sign) {   // q + sign*s, packed
  const float2 ss = make_float2(sign, sign);
  const float2 lo = ffma2(make_float2(s.x, s.y), ss, make_float2(q.x, q.y));
  const float2 hi = ffma2(make_float2(s.z, s.w), ss, make_float2(q.z, q.w));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}

// y = xp*(Q+S) + xn*(Q-S)  (xp, xn already carry the 1/2) -> (hi, lo) bf16 pairs, 8-byte stores into both planes
template <bool LO = true>
__device__ __forceinline__ void emit4(__nv_bfloat16* ph, __nv_bfloat16* pl, bool pred, const float4& xp,
                                      const float4& xn, const float4& U, const float4& V) {
  float2 y01 = fmul2(make_float2(xp.x, xp.y), make_float2(U.x, U.y));
  float2 y23 = fmul2(make_float2(xp.z, xp.w), make_float2(U.z, U.w));
  y01 = ffma2(make_float2(xn.x, xn.y), make_float2(V.x, V.y), y01);
  y23 = ffma2(make_float2(xn.z, xn.w), make_float2(V.z, V.w), y23);
  const __nv_bfloat162 h01 = __floats2bfloat162_rn(y01.x, y01.y), h23 = __floats2bfloat162_rn(y23.x, y23.y);
  // bf16x2 -> float2 by hand: low half << 16, high half masked (2 ALU ops per pair; the library routine compiles to 4)
  const uint32_t u01 = *reinterpret_cast<const uint32_t*>(&h01), u23 = *reinterpret_cast<const uint32_t*>(&h23);
  const float2 f01 = make_float2(__uint_as_float(u01 << 16), __uint_as_float(u01 & 0xffff0000u));
  const float2 f23 = make_float2(__uint_as_float(u23 << 16), __uint_as_float(u23 & 0xffff0000u));
  if (!LO) {                                    // bf16 activation storage: the hi plane only
    if (pred) *reinterpret_cast<uint2*>(ph) = make_uint2(u01, u23);
    return;
  }
  const float2 m1 = make_float2(-1.f, -1.f);
  const float2 r01 = ffma2(f01, m1, y01), r23 = ffma2(f23, m1, y23);   // y - hi, exact, packed
  const __nv_bfloat162 l01 = __floats2bfloat162_rn(r01.x, r01.y);
  const __nv_bfloat162 l23 = __floats2bfloat162_rn(r23.x, r23.y);
  if (pred) {
    *reinterpret_cast<uint2*>(ph) = make_uint2(u01, u23);
    *reinterpret_cast<uint2*>(pl) =
        make_uint2(*reinterpret_cast<const uint32_t*>(&l01), *reinterpret_cast<const uint32_t*>(&l23));
  }
}

// relu(+-ins)/2 of one question for this lane's 2 x 4 columns: shared memory -> registers
template <int NI>
struct LaneIns {
  float4 xp[NI][2], xn[NI][2];
  __device__ __forceinline__ void load(const float* xq) {   // xq = &x[q][0][0][lane * 4]
#pragma unroll
    for (int j = 0; j < NI; ++j) {
      const float* xj = xq + j * 2 * kPnCols;
      xp[j][0] = *reinterpret_cast<const float4*>(xj);
      xp[j][1] = *reinterpret_cast<const float4*>(xj + 128);
      xn[j][0] = *reinterpret_cast<const float4*>(xj + kPnCols);
      xn[j][1] = *reinterpret_cast<const float4*>(xj + kPnCols + 128);
    }
  }
};

// K-order layout (GR_AGG_K_ORDER, KO): this lane's columns relative to the neighbour region.  Chunk 0 (columns lane*4 ..)
// of slot u lies at c0 + 32 u; chunk 1 (128 + lane*4 ..) at c1 + s1 u: s1 = 32 inside the full 32-column groups, 16 in
// the tail.  A lane's 4 columns never cross a 32-column group, so each store stays one 8-byte piece.
struct KoLane {
  int c0, c1, s1;
};
template <int SEGP>
__device__ __forceinline__ KoLane ko_lane(int lane, int I) {
  constexpr int GF = SEGP / 32;
  static_assert(SEGP % 16 == 0 && SEGP - 32 * GF <= 16, "a 16-column tail at most");
  const int k0 = lane * 4, k1 = 128 + lane * 4;
  KoLane l;
  l.c0 = (k0 >> 5) * 64 * I + (k0 & 31);
  if (k1 < 32 * GF) { l.c1 = (k1 >> 5) * 64 * I + (k1 & 31); l.s1 = 32; }
  else { l.c1 = GF * 64 * I + (k1 - 32 * GF); l.s1 = 16; }
  return l;
}

// One (destination row, direction) unit: gather + accumulate the row's in-edges, then emit the NI instruction
// segments.  rc: staged {table byte offset, coefficient} of the tile's edge slice; [beg, end) the row's range in it.
// KO: hrow / lrow point at the row's neighbour region and seg_d is the slot of the unit's first instruction
template <int NI, int DT, int SEGP, bool LO = true, bool KO = false>
__device__ __forceinline__ void row_unit(const int2* __restrict__ rc, int beg, int end, int ebase, const PnDir& dd,
                                         const float* __restrict__ prior, const char* tb, const LaneIns<NI>& x,
                                         __nv_bfloat16* hrow, __nv_bfloat16* lrow, int seg_d, bool ld1, bool wr1,
                                         KoLane ko = KoLane{}) {
  float4 S0 = zero4(), S1 = S0, Q0 = S0, Q1 = S0;
  float4 v01 = zero4(), v11 = zero4();                     // lanes without chunk-1 columns never overwrite these
  const int fast_end = min(end, kEdgeCap);
  int i = beg;
  for (; i + 1 < fast_end; i += 2) {                       // two edges per step: 4 x 16-byte loads in flight per lane
    const int2 m0 = rc[i], m1 = rc[i + 1];
    const char* a0 = tb + (uint32_t)m0.x;
    const char* a1 = tb + (uint32_t)m1.x;
    const float4 v00 = ldg4(a0), v10 = ldg4(a1);
    if (ld1) { v01 = ldg4(a0 + 512); v11 = ldg4(a1 + 512); }
    const float c0 = __int_as_float(m0.y), c1 = __int_as_float(m1.y);
    fma4(S0, c0, v00); fma4_abs(Q0, c0, v00); fma4(S1, c0, v01); fma4_abs(Q1, c0, v01);
    fma4(S0, c1, v10); fma4_abs(Q0, c1, v10); fma4(S1, c1, v11); fma4_abs(Q1, c1, v11);
  }
  if (i < fast_end) {                                      // odd tail: no padded slot
    const int2 m0 = rc[i];
    const char* a0 = tb + (uint32_t)m0.x;
    const float4 v00 = ldg4(a0);
    if (ld1) v01 = ldg4(a0 + 512);
    const float c0 = __int_as_float(m0.y);
    fma4(S0, c0, v00); fma4_abs(Q0, c0, v00); fma4(S1, c0, v01); fma4_abs(Q1, c0, v01);
  }
  for (i = max(beg, kEdgeCap); i < end; ++i) {             // slow path: slice overflowed the staging buffer
    const int64_t e = (int64_t)ebase + i;
    const float w = dd.w ? dd.w[e] : 1.0f;
    const float c = w * (w * prior[dd.src[e]]);
    const char* a = tb + (uint32_t)dd.rel[e] * (uint32_t)kPnRowBytes;
    const float4 v0 = ldg4(a);
    if (ld1) v01 = ldg4(a + 512);
    fma4(S0, c, v0); fma4_abs(Q0, c, v0); fma4(S1, c, v01); fma4_abs(Q1, c, v01);
  }
  const float4 U0 = addsub4(Q0, S0, 1.f), V0 = addsub4(Q0, S0, -1.f);   // 2 * sum c*relu(v), 2 * sum c*relu(-v)
  const float4 U1 = addsub4(Q1, S1, 1.f), V1 = addsub4(Q1, S1, -1.f);
#pragma unroll
  for (int j = 0; j < NI; ++j) {
    if constexpr (KO) {
      const int o0 = ko.c0 + 32 * (seg_d + j), o1 = ko.c1 + ko.s1 * (seg_d + j);
      emit4<LO>(hrow + o0, lrow + o0, true, x.xp[j][0], x.xn[j][0], U0, V0);
      emit4<LO>(hrow + o1, lrow + o1, wr1, x.xp[j][1], x.xn[j][1], U1, V1);
    } else {
      const int seg = seg_d + j * 2 * SEGP;
      emit4<LO>(hrow + seg, lrow + seg, true, x.xp[j][0], x.xn[j][0], U0, V0);
      emit4<LO>(hrow + seg + 128, lrow + seg + 128, wr1, x.xp[j][1], x.xn[j][1], U1, V1);
    }
  }
}

// relu(+-ins)/2 staging of the tile's two questions (float4 granularity), by `nthr` threads starting at `t`
template <int NI, int DT>
__device__ __forceinline__ void stage_ins(float (*x)[NI][2][kPnCols], const PnParams& p, int b0, int t, int nthr) {
  for (int i = t; i < 2 * NI * (kPnCols / 4); i += nthr) {
    const int c4 = i % (kPnCols / 4), j = (i / (kPnCols / 4)) % NI, q = i / ((kPnCols / 4) * NI);
    const int b = b0 + q;
    float4 v = zero4();
    if (4 * c4 < DT && b < p.B)
      v = __ldg(reinterpret_cast<const float4*>(p.ins + ((int64_t)b * p.I + p.j0 + j) * DT) + c4);
    reinterpret_cast<float4*>(&x[q][j][0][0])[c4] =
        make_float4(0.5f * fmaxf(v.x, 0.f), 0.5f * fmaxf(v.y, 0.f), 0.5f * fmaxf(v.z, 0.f), 0.5f * fmaxf(v.w, 0.f));
    reinterpret_cast<float4*>(&x[q][j][1][0])[c4] = make_float4(0.5f * fmaxf(-v.x, 0.f), 0.5f * fmaxf(-v.y, 0.f),
                                                                 0.5f * fmaxf(-v.z, 0.f), 0.5f * fmaxf(-v.w, 0.f));
  }
}

// ---------------------------------------------------------------------------------------------------------
// One CTA per 64-row tile (used when the caller passes no tile counter)
// ---------------------------------------------------------------------------------------------------------
template <int NI, int DT, int SEGP, bool KO = false>
__global__ void __launch_bounds__(kThreads, 2) agg_abs_kernel(const PnParams p) {
  static_assert(DT % 4 == 0 && DT > 128 && DT <= kPnCols, "two column chunks of 128");
  __shared__ int32_t s_rowptr[2][kRows + 1];
  __shared__ int2 s_rc[2][kEdgeCap];                        // {table byte offset rel*1024, float_as_int(c)}
  __shared__ unsigned char s_any[2][kRows];
  __shared__ __align__(16) float s_x[2][NI][2][kPnCols];    // [question of the tile][j][relu(+x)/2 | relu(-x)/2][col]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * kRows;
  const int nrows = (int)min((int64_t)kRows, p.Nt - r0);
  const int N = p.N;
  const int b0 = (int)(r0 / N);
  const int rem0 = (int)(r0 - (int64_t)b0 * N);

  // ---------------- phase 1: row pointers, edge slice -> (table offset, coefficient), instructions ----------
  if (tid <= nrows) {
    s_rowptr[0][tid] = p.dir[0].rowptr[r0 + tid];
    s_rowptr[1][tid] = p.dir[1].rowptr[r0 + tid];
  }
  stage_ins<NI, DT>(s_x, p, b0, tid, kThreads);
  __syncthreads();
#pragma unroll
  for (int d = 0; d < 2; ++d) {
    const PnDir& dd = p.dir[d];
    const int64_t eb = s_rowptr[d][0];
    const int ne = (int)min((int64_t)(s_rowptr[d][nrows] - eb), (int64_t)kEdgeCap);
    for (int i = tid; i < ne; i += kThreads) {
      const int s = dd.src[eb + i];
      const int r = dd.rel[eb + i];
      const float w = dd.w ? dd.w[eb + i] : 1.0f;
      const float c = w * (w * p.prior[s]);                  // reasongnn.py:80-84
      s_rc[d][i] = make_int2((int)((uint32_t)r * (uint32_t)kPnRowBytes), __float_as_int(c));
    }
  }
  __syncthreads();
  if (tid < 2 * kRows) {   // rows whose in-edges all carry c == 0 are pure zero stores
    const int d = tid / kRows, lr = tid % kRows;
    unsigned char any = 0;
    if (lr < nrows) {
      const int ebase = s_rowptr[d][0];
      const int beg = s_rowptr[d][lr] - ebase, end = s_rowptr[d][lr + 1] - ebase;
      if (end > kEdgeCap) any = 1;
      for (int i = beg; i < min(end, kEdgeCap) && !any; ++i) any = (s_rc[d][i].y << 1) != 0;
    }
    s_any[d][lr] = any;
  }
  __syncthreads();

  // ---------------- phase 2: one warp per destination row, lane = 4 columns in each of 2 chunks -----------
  const bool ld1 = 128 + lane * 4 < DT;                      // chunk 1: lanes that own real columns
  const bool wr1 = 128 + lane * 4 < SEGP;                    //          lanes that own segment columns (incl. zero pad)
  const char* tb[2];
#pragma unroll
  for (int d = 0; d < 2; ++d) tb[d] = reinterpret_cast<const char*>(p.dir[d].pn) + lane * 16;
  // KO: the row's neighbour region, the lane's columns come from ko
  __nv_bfloat16* const hi_lane = KO ? p.out_hi + r0 * p.ld + p.out_col0
                          : p.out_hi + r0 * p.ld + p.out_col0 + lane * 4 + (int64_t)p.j0 * 2 * SEGP;
  __nv_bfloat16* const lo_lane = KO ? p.out_lo + r0 * p.ld + p.out_col0
                          : p.out_lo + r0 * p.ld + p.out_col0 + lane * 4 + (int64_t)p.j0 * 2 * SEGP;
  const KoLane ko = KO ? ko_lane<SEGP>(lane, p.I) : KoLane{};
  const int lr_switch = N - rem0;                            // first tile row of question b0 + 1 (N >= kRows)
  LaneIns<NI> x;
  int cur_q = -1;
  for (int lr = warp; lr < nrows; lr += kWarps) {
    const int q = lr >= lr_switch ? 1 : 0;
    if (q != cur_q) {
      cur_q = q;
      x.load(&s_x[q][0][0][lane * 4]);
    }
    __nv_bfloat16* const hrow = hi_lane + (int64_t)lr * p.ld;
    __nv_bfloat16* const lrow = lo_lane + (int64_t)lr * p.ld;
#pragma unroll
    for (int d = 0; d < 2; ++d) {
      const int ebase = s_rowptr[d][0];
      const int beg = s_rowptr[d][lr] - ebase, end = s_rowptr[d][lr + 1] - ebase;
      if (!s_any[d][lr]) {
#pragma unroll
        for (int j = 0; j < NI; ++j) {
          const int u = d * p.I + p.j0 + j;
          const int seg = KO ? ko.c0 + 32 * u : d * SEGP + j * 2 * SEGP;
          const int seg1 = KO ? ko.c1 + ko.s1 * u : seg + 128;
          *reinterpret_cast<uint2*>(hrow + seg) = make_uint2(0u, 0u);
          *reinterpret_cast<uint2*>(lrow + seg) = make_uint2(0u, 0u);
          if (wr1) {
            *reinterpret_cast<uint2*>(hrow + seg1) = make_uint2(0u, 0u);
            *reinterpret_cast<uint2*>(lrow + seg1) = make_uint2(0u, 0u);
          }
        }
        continue;
      }
      row_unit<NI, DT, SEGP, true, KO>(s_rc[d], beg, end, ebase, p.dir[d], p.prior, tb[d], x, hrow, lrow,
                                       KO ? d * p.I + p.j0 : d * SEGP, ld1, wr1, ko);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// mbarrier helpers
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(b)), "r"(parity), "r"(20000u)     // suspend-time hint [ns]: a waiting role does not spin on the
        : "memory");                                       // issue port (measured: 129 us with, 141 us without)
  }
}

__device__ __forceinline__ bool mbar_test(uint64_t* b, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(b)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
template <int NI, int ROWS>
struct alignas(16) HBuf {
  int2 rc[2][kEdgeCap];
  float x[2][NI][2][kPnCols];
  int32_t rowptr[2][ROWS + 4];
  int32_t tile;
  int32_t pad_[3];
};

// Staging side of the persistent kernels: one warp stages a tile of <= ROWS destination rows (row pointers,
// relu(+-ins)/2 of its <= 2 questions, {table byte offset | relation row index, coefficient} per in-edge of both
// directions) into `bf`.  Tried and measured against this batch structure (128 edges of one direction per batch, 4
// per lane): both directions and 8 edges per lane per batch (3 dependent round trips per tile instead of ~10) -- the
// kernel got 1-5 % SLOWER; the staging warp is not what bounds it, and burstier index loads disturb the gather.
template <int NI, int DT, int ROWS, int CAP = kEdgeCap, bool REL_INDEX = false, class Buf>
__device__ __forceinline__ void produce_tile_rows(Buf& bf, const PnParams& p, int tile, int lane) {
  const int N = p.N;
  const int64_t r0 = (int64_t)tile * ROWS;
  const int nrows = (int)min((int64_t)ROWS, p.Nt - r0);
  const int b0 = (int)(r0 / N);
  if (lane == 0) bf.tile = tile;
  int eb[2], ne[2];
#pragma unroll
  for (int d = 0; d < 2; ++d) {
    const int32_t* rp = p.dir[d].rowptr + r0;
    const int e0 = __ldg(rp), e1 = __ldg(rp + nrows);
#pragma unroll
    for (int k = 0; k < (ROWS + 32) / 32; ++k) {
      const int i = lane + 32 * k;
      if (i <= nrows) bf.rowptr[d][i] = __ldg(rp + i);
    }
    eb[d] = e0;
    ne[d] = min(e1 - e0, CAP);
  }
  stage_ins<NI, DT>(bf.x, p, b0, lane, 32);
#pragma unroll
  for (int d = 0; d < 2; ++d) {
    const PnDir& dd = p.dir[d];
    for (int i0 = 0; i0 < ne[d]; i0 += 128) {
      int sidx[4], ridx[4];
      float wv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + lane + 32 * u;
        const bool ok = i < ne[d];
        sidx[u] = ok ? __ldg(dd.src + eb[d] + i) : 0;
        ridx[u] = ok ? __ldg(dd.rel + eb[d] + i) : 0;
        wv[u] = (ok && dd.w) ? __ldg(dd.w + eb[d] + i) : 1.0f;
      }
      float pr[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) pr[u] = __ldg(p.prior + sidx[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + lane + 32 * u;
        if (i < ne[d])
          bf.rc[d][i] = make_int2(REL_INDEX ? ridx[u] : (int)((uint32_t)ridx[u] * (uint32_t)kPnRowBytes),
                                  __float_as_int(wv[u] * (wv[u] * pr[u])));             // reasongnn.py:80-84
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Persistent, warp-specialised kernel (used when the caller passes a tile counter; gr_set_option("agg_abs_ws", 1|2)):
// each CTA lives for the whole launch; warp KW (the staging warp) stages tile t+1 (row pointers, {table offset,
// coefficient} per edge, relu(+-ins)/2) into the other half of a double buffer while warps 0..KW-1 (consumers, one row
// at a time) work on tile t; full/empty mbarriers per buffer; tiles are handed out by an atomic counter so the tail
// balances.  Consumer warps per CTA, rows per tile and resident CTAs per SM are template parameters.  The register
// file is split per scheduler (16 K registers each): with W warps per CTA and MINB CTAs per SM the busiest scheduler
// holds ceil(W * MINB / 4) warps, so 9-warp CTAs x 2 leave 96 registers per thread -- and so do 10-warp CTAs x 2 (5
// warps on all four schedulers): the default is 9 consumer warps + the staging warp and 72-row tiles (127 us at cfg2
// against 131 us for 8 + 1 / 64 rows).  More warps do not help: 11 + 1 at 80 registers 143 us, 19 + 1 in one CTA
// 164 us, 7 + 1 x 3 CTAs 148 us (profiles/r2_agg_modes.txt).
// ---------------------------------------------------------------------------------------------------------
template <int NI, int DT, int SEGP, int KW, int ROWS, int MINB, bool LO, bool KO = false>
__global__ void __launch_bounds__((KW + 1) * 32, MINB) agg_abs_wsg_kernel(const PnParams p, int ntiles) {
  using Buf = HBuf<NI, ROWS>;
  extern __shared__ __align__(16) unsigned char ws_smem[];
  Buf* bufs = reinterpret_cast<Buf*>(ws_smem);
  __shared__ __align__(8) uint64_t s_full[2], s_empty[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = p.N;
  if (tid == 0) {
    mbar_init(&s_full[0], 32); mbar_init(&s_full[1], 32);
    mbar_init(&s_empty[0], KW * 32); mbar_init(&s_empty[1], KW * 32);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == KW) {
    for (int it = 0;; ++it) {
      Buf& bf = bufs[it & 1];
      if (it >= 2) mbar_wait(&s_empty[it & 1], ((it >> 1) - 1) & 1);
      int tile = 0;
      if (lane == 0) tile = atomicAdd(p.tile_counter, 1);
      tile = __shfl_sync(0xffffffffu, tile, 0);
      if (tile >= ntiles) {
        if (lane == 0) bf.tile = -1;
        __syncwarp();
        mbar_arrive(&s_full[it & 1]);
        break;
      }
      produce_tile_rows<NI, DT, ROWS>(bf, p, tile, lane);
      __syncwarp();
      mbar_arrive(&s_full[it & 1]);
    }
    return;
  }
  const bool ld1 = 128 + lane * 4 < DT;
  const bool wr1 = 128 + lane * 4 < SEGP;
  const char* tb[2];
#pragma unroll
  for (int d = 0; d < 2; ++d) tb[d] = reinterpret_cast<const char*>(p.dir[d].pn) + lane * 16;
  const KoLane ko = KO ? ko_lane<SEGP>(lane, p.I) : KoLane{};
  LaneIns<NI> x;
  for (int it = 0;; ++it) {
    Buf& bf = bufs[it & 1];
    mbar_wait(&s_full[it & 1], (it >> 1) & 1);
    const int tile = bf.tile;
    if (tile < 0) break;
    const int64_t r0 = (int64_t)tile * ROWS;
    const int nrows = (int)min((int64_t)ROWS, p.Nt - r0);
    const int b0 = (int)(r0 / N);
    const int lr_switch = N - (int)(r0 - (int64_t)b0 * N);
    __nv_bfloat16* const hi_lane = KO ? p.out_hi + r0 * p.ld + p.out_col0
                          : p.out_hi + r0 * p.ld + p.out_col0 + lane * 4 + (int64_t)p.j0 * 2 * SEGP;
    __nv_bfloat16* const lo_lane = KO ? p.out_lo + r0 * p.ld + p.out_col0
                          : p.out_lo + r0 * p.ld + p.out_col0 + lane * 4 + (int64_t)p.j0 * 2 * SEGP;
    int cur_q = -1;
    for (int lr = warp; lr < nrows; lr += KW) {
      const int q = lr >= lr_switch ? 1 : 0;
      if (q != cur_q) {
        cur_q = q;
        x.load(&bf.x[q][0][0][lane * 4]);
      }
      __nv_bfloat16* const hrow = hi_lane + (int64_t)lr * p.ld;
      __nv_bfloat16* const lrow = lo_lane + (int64_t)lr * p.ld;
#pragma unroll
      for (int d = 0; d < 2; ++d) {
        const int ebase = bf.rowptr[d][0];
        const int beg = bf.rowptr[d][lr] - ebase, end = bf.rowptr[d][lr + 1] - ebase;
        row_unit<NI, DT, SEGP, LO, KO>(bf.rc[d], beg, end, ebase, p.dir[d], p.prior, tb[d], x, hrow, lrow,
                                       KO ? d * p.I + p.j0 : d * SEGP, ld1, wr1, ko);
      }
    }
    mbar_arrive(&s_empty[it & 1]);
  }
}

constexpr int kTmaCap = 512;       // staged edges per direction per tile of the gather4 kernel (mean 224); the rest -> slow path

__device__ __forceinline__ float4 lds4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ float lds1(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
  return v;
}

constexpr int kOobRow = 0x3fffffff;         // row coordinate outside any table: zero fill, no memory traffic

// four table rows r0..r3 (`slot_bytes` of each) into consecutive slots at dst, completion counted on `bar`: one 1-D
// bulk copy per row (16-byte aligned slots; a 2-D tensor copy would need 128-byte aligned destinations).  A row of
// kOobRow (a slot past the unit's edges, never read) copies row 0.
__device__ __forceinline__ void tma_gather4(uint32_t dst, const float* table, uint64_t* bar, int r0, int r1, int r2,
                                            int r3, uint32_t slot_bytes) {
  const int rows[4] = {r0, r1, r2, r3};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const char* src = reinterpret_cast<const char*>(table) + (size_t)(rows[i] == kOobRow ? 0 : rows[i]) * kPnRowBytes;
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     dst + (uint32_t)i * slot_bytes),
                 "l"(src), "r"(slot_bytes), "r"(smem_u32(bar))
                 : "memory");
  }
}

template <int NI, int ROWS>
struct alignas(16) G5Buf {
  int4 quad[2][ROWS][2];             // gather4 row coordinates of the unit's stage edges 0-3 / 4-7
  int2 rc[2][kTmaCap];               // {relation row index, coefficient}
  float x[2][NI][2][kPnCols];
  int32_t rowptr[2][ROWS + 4];
  uint32_t ud[2][ROWS];              // first staged edge | #stage edges << 16 | (unit has more edges than that) << 31
  int32_t tile;
  int32_t nrows;
  int32_t pad_[2];
};

// ---------------------------------------------------------------------------------------------------------
// staged-row kernel with a deeper prefetch (gr_set_option("agg_abs_ws", 3)).
// Three gather kernels with very different instruction counts (tma2 340, tma3 308, g4 303 per unit) all ran 157.5 us:
// 1730 units per SM / 14 warps x 1.27 us.  With the copies of unit k + 1 issued when unit k starts, a unit cannot
// take less than the latency of a TMA gather (issue -> bytes landed -> mbarrier flip -> waiter resumes), ~1.3 us here,
// three times the LDG round trip.  So the per-warp ring is cut into FOUR groups of four slots (one gather4 each): a
// unit takes one or two groups (its first <= 8 staged edges), its mbarrier is the one of its first group, and a flat
// prefetch cursor keeps issuing ahead (across the tile boundary) while groups are free: 2-3 units in flight.
// ---------------------------------------------------------------------------------------------------------
template <int NI, int DT, int SEGP, int KW, int RPW, bool KO = false>
__global__ void __launch_bounds__((KW + 2) * 32, 1)
agg_abs_g5_kernel(const PnParams p, int ntiles) {
  static_assert(DT % 4 == 0 && DT > 128 && DT <= kPnCols, "two column chunks of 128");
  constexpr int ROWS = KW * RPW;
  constexpr int kSlot = DT * 4;
  constexpr int kGroup = 4 * kSlot;            // bytes of one gather4 group
  using Buf = G5Buf<NI, ROWS>;
  extern __shared__ __align__(128) unsigned char ws_smem_raw[];
  unsigned char* const ring_all = ws_smem_raw + ((128u - (smem_u32(ws_smem_raw) & 127u)) & 127u);
  Buf* bufs = reinterpret_cast<Buf*>(ring_all + (size_t)KW * 4 * kGroup);
  __shared__ __align__(8) uint64_t s_full[2], s_empty[2];
  __shared__ __align__(8) uint64_t s_bar[KW][4];
  __shared__ volatile int s_turn;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = p.N;
  if (tid == 0) {
    mbar_init(&s_full[0], 32); mbar_init(&s_full[1], 32);
    mbar_init(&s_empty[0], KW * 32); mbar_init(&s_empty[1], KW * 32);
    for (int w = 0; w < KW; ++w)
      for (int b = 0; b < 4; ++b) mbar_init(&s_bar[w][b], 1);
    s_turn = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= KW) {
    // =============================== staging warps: warp KW -> even iterations, KW + 1 -> odd ===============
    const int par = warp - KW;
    Buf& bf = bufs[par];
    for (int it = par;; it += 2) {
      if (it >= 2) mbar_wait(&s_empty[par], ((it >> 1) - 1) & 1);
      int tile = 0;
      if (lane == 0) {
        while (s_turn != it) __nanosleep(20);                 // tiles are grabbed in hand-over order
        tile = atomicAdd(p.tile_counter, 1);
        __threadfence_block();
        s_turn = it + 1;
      }
      tile = __shfl_sync(0xffffffffu, tile, 0);
      if (tile >= ntiles) {
        if (lane == 0) bf.tile = -1;
        __syncwarp();
        mbar_arrive(&s_full[par]);
        break;
      }
      const int nrows = (int)min((int64_t)ROWS, p.Nt - (int64_t)tile * ROWS);
      if (lane == 0) bf.nrows = nrows;
      produce_tile_rows<NI, DT, ROWS, kTmaCap, true>(bf, p, tile, lane);
      __syncwarp();
      for (int un = lane; un < 2 * nrows; un += 32) {          // unit descriptors + gather4 coordinate quads
        const int d = un >= nrows ? 1 : 0, lr = un - d * nrows;
        const int ebase = bf.rowptr[d][0];
        const int beg = bf.rowptr[d][lr] - ebase, end = bf.rowptr[d][lr + 1] - ebase;
        const int n = max(0, min(min(end, kTmaCap) - beg, 8));
        int r[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) r[k] = k < n ? bf.rc[d][beg + k].x : kOobRow;
        bf.quad[d][lr][0] = make_int4(r[0], r[1], r[2], r[3]);
        bf.quad[d][lr][1] = make_int4(r[4], r[5], r[6], r[7]);
        bf.ud[d][lr] = (uint32_t)min(beg, kTmaCap) | ((uint32_t)n << 16) | (end - beg > n ? 0x80000000u : 0u);
      }
      __syncwarp();
      mbar_arrive(&s_full[par]);
    }
    return;
  }

  // =============================== consumer warps ===============================
  const bool ld1 = 128 + lane * 4 < DT;
  const bool wr1 = 128 + lane * 4 < SEGP;
  const KoLane ko = KO ? ko_lane<SEGP>(lane, p.I) : KoLane{};
  const uint32_t ring_s = smem_u32(ring_all) + (uint32_t)warp * 4u * kGroup;   // this warp's four groups
  const uint32_t ring_lane = ring_s + lane * 16;
  uint64_t* const bars = s_bar[warp];
  LaneIns<NI> x;
  // ring state (all warp-uniform)
  int gh = 0, gc = 0, gfree = 4;      // next group to fill / group of the unit being consumed / free groups
  uint32_t parbits = 0;               // phase parity of the four group barriers
  // prefetch cursor: next unit to issue = (tile iteration pit, row plr, direction pd); pnrows = rows of that tile
  int pit = -1, plr = 0, pd = 0, pnrows = 0;
  bool pend = false;                  // the cursor has seen the end marker

  for (int it = 0;; ++it) {
    Buf& bf = bufs[it & 1];
    mbar_wait(&s_full[it & 1], (it >> 1) & 1);
    const int tile = bf.tile;
    if (tile < 0) break;
    const int64_t r0 = (int64_t)tile * ROWS;
    const int nrows = bf.nrows;
    const int b0 = (int)(r0 / N);
    const int lr_switch = N - (int)(r0 - (int64_t)b0 * N);
    const int64_t ld = p.ld;
    __nv_bfloat16* hrow = KO ? p.out_hi + (r0 + warp) * ld + p.out_col0
                          : p.out_hi + (r0 + warp) * ld + p.out_col0 + lane * 4 + (int64_t)p.j0 * 2 * SEGP;
    __nv_bfloat16* lrow = KO ? p.out_lo + (r0 + warp) * ld + p.out_col0
                          : p.out_lo + (r0 + warp) * ld + p.out_col0 + lane * 4 + (int64_t)p.j0 * 2 * SEGP;
    if (pit < it) { pit = it; plr = warp; pd = 0; pnrows = nrows; }
    int cur_q = -1;
    for (int lr = warp; lr < nrows; lr += KW, hrow += KW * ld, lrow += KW * ld) {
      const int q = lr >= lr_switch ? 1 : 0;
      if (q != cur_q) {
        cur_q = q;
        x.load(&bf.x[q][0][0][lane * 4]);
      }
#pragma unroll
      for (int d = 0; d < 2; ++d) {
        // ---------------- keep the ring full ----------------
        for (;;) {
          if (plr >= pnrows) {                                // cursor at the end of its tile
            if (pend || pit > it) break;                      // never two tiles ahead (that buffer is this one)
            if (!mbar_test(&s_full[(it + 1) & 1], ((it + 1) >> 1) & 1)) break;
            const Buf& nb = bufs[(it + 1) & 1];
            pit = it + 1; plr = warp; pd = 0;
            if (nb.tile < 0) { pend = true; pnrows = 0; break; }
            pnrows = nb.nrows;
            continue;
          }
          const Buf& pb = bufs[pit & 1];
          const uint32_t pdesc = pb.ud[pd][plr];
          const int ng = (int)(((pdesc >> 16) & 0xffu) + 3u) >> 2;
          if (ng > gfree) break;
          if (ng > 0) {
            uint64_t* const bar = &bars[gh];
            if (lane == 0) mbar_expect_tx(bar, (uint32_t)(ng * kGroup));
            if (lane < ng) {
              const int4 qd = pb.quad[pd][plr][lane];
              tma_gather4(ring_s + (uint32_t)(((gh + lane) & 3) * kGroup), p.dir[pd].pn, bar, qd.x, qd.y, qd.z, qd.w,
                          (uint32_t)kSlot);
            }
            gh = (gh + ng) & 3;
            gfree -= ng;
          }
          pd ^= 1;
          if (pd == 0) plr += KW;
        }
        // ---------------- consume unit (lr, d) ----------------
        const uint32_t desc = bf.ud[d][lr];
        const int beg = (int)(desc & 0xffffu), n = (int)((desc >> 16) & 0xffu);
        float4 S0 = zero4(), S1 = S0, Q0 = S0, Q1 = S0;
        float4 v1 = zero4();                                  // lanes without chunk-1 columns never overwrite it
        if (n > 0) {
          mbar_wait(&bars[gc], (parbits >> gc) & 1u);
          parbits ^= 1u << gc;
          uint32_t cy = smem_u32(&bf.rc[d][0]) + (uint32_t)(beg * 8 + 4);
          uint32_t sl = ring_lane + (uint32_t)gc * kGroup;
          const int n0 = min(n, 4);
#pragma unroll 1
          for (int i = 0; i < n0; ++i, sl += kSlot, cy += 8) {
            const float c = lds1(cy);
            const float4 v0 = lds4(sl);
            if (ld1) v1 = lds4(sl + 512);
            fma4(S0, c, v0); fma4_abs(Q0, c, v0); fma4(S1, c, v1); fma4_abs(Q1, c, v1);
          }
          if (n > 4) {
            sl = ring_lane + (uint32_t)((gc + 1) & 3) * kGroup;
#pragma unroll 1
            for (int i = 4; i < n; ++i, sl += kSlot, cy += 8) {
              const float c = lds1(cy);
              const float4 v0 = lds4(sl);
              if (ld1) v1 = lds4(sl + 512);
              fma4(S0, c, v0); fma4_abs(Q0, c, v0); fma4(S1, c, v1); fma4_abs(Q1, c, v1);
            }
          }
          const int ngc = (n + 3) >> 2;
          gc = (gc + ngc) & 3;
          gfree += ngc;
        }
        if (desc >> 31) {                                     // long rows: staged edges beyond the ring, then the rest
          const char* tb = reinterpret_cast<const char*>(p.dir[d].pn) + lane * 16;
          const int ebase = bf.rowptr[d][0];
          const int rb = bf.rowptr[d][lr] - ebase, end = bf.rowptr[d][lr + 1] - ebase;
          const int fast_end = min(end, kTmaCap);
          for (int i = rb + n; i < fast_end; ++i) {
            const int2 m = bf.rc[d][i];
            const char* a0 = tb + (size_t)(uint32_t)m.x * kPnRowBytes;
            const float4 v0 = ldg4(a0);
            if (ld1) v1 = ldg4(a0 + 512);
            const float c = __int_as_float(m.y);
            fma4(S0, c, v0); fma4_abs(Q0, c, v0); fma4(S1, c, v1); fma4_abs(Q1, c, v1);
          }
          const PnDir& dd = p.dir[d];
          for (int i = max(rb + n, kTmaCap); i < end; ++i) {
            const int64_t e = (int64_t)ebase + i;
            const float w = dd.w ? dd.w[e] : 1.0f;
            const float c = w * (w * p.prior[dd.src[e]]);
            const char* a0 = tb + (size_t)(uint32_t)dd.rel[e] * kPnRowBytes;
            const float4 v0 = ldg4(a0);
            if (ld1) v1 = ldg4(a0 + 512);
            fma4(S0, c, v0); fma4_abs(Q0, c, v0); fma4(S1, c, v1); fma4_abs(Q1, c, v1);
          }
        }
        const float4 U0 = addsub4(Q0, S0, 1.f), V0 = addsub4(Q0, S0, -1.f);
        const float4 U1 = addsub4(Q1, S1, 1.f), V1 = addsub4(Q1, S1, -1.f);
#pragma unroll
        for (int j = 0; j < NI; ++j) {
          const int u = d * p.I + p.j0 + j;
          const int seg = KO ? ko.c0 + 32 * u : d * SEGP + j * 2 * SEGP;
          const int seg1 = KO ? ko.c1 + ko.s1 * u : seg + 128;
          emit4(hrow + seg, lrow + seg, true, x.xp[j][0], x.xn[j][0], U0, V0);
          emit4(hrow + seg1, lrow + seg1, wr1, x.xp[j][1], x.xn[j][1], U1, V1);
        }
      }
    }
    mbar_arrive(&s_empty[it & 1]);
  }
}

// table [rows, D] fp32 (row stride ldt) -> zero-padded [rows][256]
__global__ void pad_table_kernel(const float* __restrict__ table, int64_t ldt, int64_t rows, int D,
                                 float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // (row, 4-column group)
  if (i >= rows * (kPnCols / 4)) return;
  const int64_t r = i / (kPnCols / 4);
  const int g = (int)(i % (kPnCols / 4));
  float v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = 4 * g + k < D ? table[r * ldt + 4 * g + k] : 0.f;
  reinterpret_cast<float4*>(out + r * kPnCols)[g] = make_float4(v[0], v[1], v[2], v[3]);
}


template <int NI, int KW, int ROWS, int MINB, bool LO, bool KO>
int launch_wsg_lo(const PnParams& p, cudaStream_t stream) {
  constexpr auto kern = agg_abs_wsg_kernel<NI, 200, 208, KW, ROWS, MINB, LO, KO>;
  const size_t smem = 2 * sizeof(HBuf<NI, ROWS>);
  if (int rc = opt_in_smem<kern>(__func__, (int)smem)) return rc;
  GR_CHECK_CUDA(cudaMemsetAsync(p.tile_counter, 0, sizeof(int32_t), stream));
  const unsigned tiles = (unsigned)ceil_div(p.Nt, ROWS);
  const unsigned pgrid = std::min<unsigned>(tiles, (unsigned)MINB * (unsigned)sm_count());
  kern<<<pgrid, (KW + 1) * 32, smem, stream>>>(p, (int)tiles);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

template <int NI, int KW, int ROWS, int MINB, bool KO>
int launch_wsg(const PnParams& p, cudaStream_t stream) {
  // out_lo == NULL: bf16 activation storage (hi plane only; the K-order layout always has both planes)
  if constexpr (KO) return launch_wsg_lo<NI, KW, ROWS, MINB, true, true>(p, stream);
  return p.out_lo ? launch_wsg_lo<NI, KW, ROWS, MINB, true, false>(p, stream)
                  : launch_wsg_lo<NI, KW, ROWS, MINB, false, false>(p, stream);
}

template <int NI, int KW, int RPW, bool KO>
int launch_g4(const PnParams& p, cudaStream_t stream) {
  constexpr auto kern = agg_abs_g5_kernel<NI, 200, 208, KW, RPW, KO>;
  const size_t smem = 128 + (size_t)KW * 16 * 200 * 4 + 2 * sizeof(G5Buf<NI, KW * RPW>);
  if (int rc = opt_in_smem<kern>(__func__, (int)smem)) return rc;
  GR_CHECK_CUDA(cudaMemsetAsync(p.tile_counter, 0, sizeof(int32_t), stream));
  const unsigned tiles = (unsigned)ceil_div(p.Nt, KW * RPW);
  const unsigned pgrid = std::min<unsigned>(tiles, (unsigned)sm_count());
  kern<<<pgrid, (KW + 2) * 32, smem, stream>>>(p, (int)tiles);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

// agg_abs_ws: 0 one CTA per 64-row tile | 1 persistent, 8 + 1 warps, 64-row tiles (the round-1 shape) |
//             2 persistent, 9 + 1 warps, 72-row tiles (default) | 3 gather4 kernel (NI == 2 and table_rows given).
// KO: the neighbour segments in the K-order layout (GR_AGG_K_ORDER), every variant
template <int NI, bool KO>
int launch_pn(const PnParams& p, cudaStream_t stream) {
  if (p.tile_counter && g_opt_agg_abs_ws) {
    if constexpr (NI == 2) {
      if (g_opt_agg_abs_ws == 3 && p.table_rows > 0 && p.out_lo) return launch_g4<2, 14, 4, KO>(p, stream);
    }
    if (g_opt_agg_abs_ws == 1 || p.N < 72) return launch_wsg<NI, 8, 64, 2, KO>(p, stream);   // a tile spans <= 2 questions
    return launch_wsg<NI, 9, 72, 2, KO>(p, stream);
  }
  const unsigned grid = (unsigned)ceil_div(p.Nt, kRows);
  agg_abs_kernel<NI, 200, 208, KO><<<grid, kThreads, 0, stream>>>(p);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

}  // namespace
}  // namespace gr

extern "C" int gr_pad_table256(const float* table, int64_t ldt, int64_t rows, int D, float* pn, void* stream_) {
  using namespace gr;
  GR_CHECK_ARG(table && pn, "null pointer");
  GR_CHECK_ARG(rows > 0 && D > 0 && D <= kPnCols && ldt >= D, "bad shape (D <= 256)");
  GR_CHECK_ARG((reinterpret_cast<uintptr_t>(pn) & 15) == 0, "pn must be 16-byte aligned");
  const int64_t work = rows * (kPnCols / 4);
  pad_table_kernel<<<(unsigned)ceil_div(work, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      table, ldt, rows, D, pn);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_aggregate_dual_abs_supported(int N, int D, int64_t seg_pitch, int64_t R1) {
  return (D == 200 && seg_pitch == 208 && N >= gr::kRows && R1 > 0 && R1 < (1 << 21)) ? 1 : 0;
}

namespace gr {
namespace {
// both entry points; errors are reported as `fn`
int aggregate_dual_abs(const char* fn, const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                       const float* w_t, const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h,
                       const float* w_h, const float* prior, const float* pn_fwd, const float* pn_inv,
                       int64_t table_rows, const float* ins, void* out_hi, void* out_lo, int64_t ld_planes,
                       int64_t out_col0, int64_t seg_pitch, int B, int N, int D, int I, int64_t F,
                       int32_t* tile_counter, uint32_t flags, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG_AS(fn, rowptr_t && rowptr_h && prior && pn_fwd && pn_inv && ins && out_hi, "null pointer");
  GR_CHECK_ARG_AS(fn, (flags & ~GR_AGG_K_ORDER) == 0, "unknown flags");
  const bool ko = (flags & GR_AGG_K_ORDER) != 0;
  GR_CHECK_ARG_AS(fn, !ko || out_lo, "GR_AGG_K_ORDER needs both planes (no hi-only output: the dense layer keeps fp32-class A)");
  // the dense layer runs I <= 2; wider K-order builds would spill (as the segment-layout ones of 3 and 4 instructions do)
  GR_CHECK_ARG_AS(fn, !ko || I <= 2, "GR_AGG_K_ORDER is built for I <= 2");
  // only the persistent kernels have a hi-only form; agg_abs_kernel (no tile counter, or agg_abs_ws 0) always stores lo
  GR_CHECK_ARG_AS(fn, out_lo || (tile_counter && g_opt_agg_abs_ws != 0),
               "hi-only output (bf16 activation storage) needs a persistent kernel (a tile counter and agg_abs_ws != 0)");
  GR_CHECK_ARG_AS(fn, F == 0 || (src_t && rel_t && src_h && rel_h), "null edge arrays");
  GR_CHECK_ARG_AS(fn, B > 0 && N >= kRows && I > 0, "B, I must be positive and N >= 64");
  GR_CHECK_ARG_AS(fn, D == 200 && seg_pitch == 208, "this build specialises D = 200, seg_pitch = 208 (use gr_aggregate_dual)");
  GR_CHECK_ARG_AS(fn, ld_planes % 4 == 0 && out_col0 % 4 == 0 && ld_planes >= out_col0 + 2 * (int64_t)I * seg_pitch,
               "plane row pitch / column offset must be multiples of 4 and cover all segments");
  GR_CHECK_ARG_AS(fn, (reinterpret_cast<uintptr_t>(out_hi) & 7) == 0 && (reinterpret_cast<uintptr_t>(out_lo) & 7) == 0 &&   /* NULL ok */
                   (reinterpret_cast<uintptr_t>(pn_fwd) & 15) == 0 && (reinterpret_cast<uintptr_t>(pn_inv) & 15) == 0,
               "misaligned planes / padded tables");
  PnParams p{};
  p.dir[0] = PnDir{rowptr_t, src_t, rel_t, w_t, pn_fwd};
  p.dir[1] = PnDir{rowptr_h, src_h, rel_h, w_h, pn_inv};
  p.prior = prior; p.ins = ins;
  p.out_hi = reinterpret_cast<__nv_bfloat16*>(out_hi); p.out_lo = reinterpret_cast<__nv_bfloat16*>(out_lo);
  p.ld = ld_planes; p.out_col0 = out_col0; p.Nt = (int64_t)B * N;
  p.B = B; p.N = N; p.I = I; p.tile_counter = tile_counter;
  p.table_rows = table_rows;
  for (int j0 = 0; j0 < I; j0 += 4) {
    p.j0 = j0;
    const int ni = I - j0 < 4 ? I - j0 : 4;
    int rc = ko ? (ni == 1 ? launch_pn<1, true>(p, stream) : launch_pn<2, true>(p, stream))
                : (ni == 1 ? launch_pn<1, false>(p, stream) : ni == 2 ? launch_pn<2, false>(p, stream)
                   : ni == 3 ? launch_pn<3, false>(p, stream) : launch_pn<4, false>(p, stream));
    if (rc != GR_OK) return rc;
  }
  return GR_OK;
}

}  // namespace
}  // namespace gr

extern "C" int gr_aggregate_dual_abs_ex(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                                        const float* w_t, const int32_t* rowptr_h, const int32_t* src_h,
                                        const int32_t* rel_h, const float* w_h, const float* prior,
                                        const float* pn_fwd, const float* pn_inv, int64_t table_rows, const float* ins,
                                        void* out_hi, void* out_lo, int64_t ld_planes, int64_t out_col0,
                                        int64_t seg_pitch, int B, int N, int D, int I, int64_t F,
                                        int32_t* tile_counter, uint32_t flags, void* stream_) {
  return gr::aggregate_dual_abs(__func__, rowptr_t, src_t, rel_t, w_t, rowptr_h, src_h, rel_h, w_h, prior, pn_fwd,
                                pn_inv, table_rows, ins, out_hi, out_lo, ld_planes, out_col0, seg_pitch, B, N, D, I, F,
                                tile_counter, flags, stream_);
}

extern "C" int gr_aggregate_dual_abs(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                                    const float* w_t, const int32_t* rowptr_h, const int32_t* src_h,
                                    const int32_t* rel_h, const float* w_h, const float* prior,
                                    const float* pn_fwd, const float* pn_inv, int64_t table_rows, const float* ins, void* out_hi,
                                    void* out_lo, int64_t ld_planes, int64_t out_col0, int64_t seg_pitch, int B,
                                    int N, int D, int I, int64_t F, int32_t* tile_counter, void* stream_) {
  return gr::aggregate_dual_abs(__func__, rowptr_t, src_t, rel_t, w_t, rowptr_h, src_h, rel_h, w_h, prior, pn_fwd,
                                pn_inv, table_rows, ins, out_hi, out_lo, ld_planes, out_col0, seg_pitch, B, N, D, I, F,
                                tile_counter, 0u, stream_);
}
