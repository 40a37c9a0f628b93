// The aggregation kernel family: relation-typed neighbour aggregation over the destination-CSR subgraph.
//
// Replaces (reference paths): ReasonGNNLayer.reason_layer / reason_layer_inv
// (gnn/modules/kg_reasoning/reasongnn.py:61-116), NSMLayer.reason_layer (nsm_gnn.py:87-112) and the
// SpMM half of TypeLayer.forward (gnn/modules/layer_init.py:46-57).
//
// Math.  The reference computes, per fact f with relation r_f, question b_f and destination n,
//     msg_f = relu( (W_k rel[r_f] + b_k) * ins[b_f] ) * w_f * (w_f * p[src_f])      and  out[n] = sum_f msg_f.
// (W_k rel + b_k) only depends on the relation: it is hoisted to a table P[R1, D] (gr_linear).  With
// c_f = w_f*(w_f*p[src_f]) >= 0 and, per element,  relu(P*x) = x*relu(P) for x >= 0 and (-x)*relu(-P) for
// x < 0, the edge loop only needs two instruction-INDEPENDENT accumulators
//     A[n] = sum_f c_f relu(P[r_f]),   Bn[n] = sum_f c_f relu(-P[r_f]),
// and every instruction j is an epilogue  out_j[n] = x_j >= 0 ? x_j*A : (-x_j)*Bn.  The inner loop is
// therefore 2 FMNMX + 2 FFMA per element per edge for any number of instructions.
//
// Work decomposition.  One CTA = one tile of kRows consecutive destination rows.  Phase 1 stages the
// tile's row pointers and its contiguous edge slice (relation id + coefficient c_f, which needs the
// prior gather) into shared memory, either with plain coalesced loads or with 1-D bulk TMA copies
// (cp.async.bulk + mbarrier) of the raw src/rel slices.  Phase 2: one warp per row, lanes across the
// feature dimension (128-bit loads of the L2-resident table row, 128-bit stores of the output row).
// Reduction order inside a row = CSR slot order = original fact order: deterministic, atomic-free.
//
// Roofline: HBM-bound on the OUTPUT rows (SURVEY.md 8d): per (direction, instruction) unit
//   F*8 + (Nt+1)*4 + Nt*4 + R1*D*4 + B*D*4 + Nt*D*4 bytes.
#include <cuda_bf16.h>

#include "common.cuh"

namespace gr {

int g_opt_agg_tma = 0;   // set through gr_set_option("agg_tma", 0|1)

namespace {

constexpr int kRows = 64;        // destination rows per CTA tile
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kEdgeCap = 1024;   // staged edges per direction per tile; the rest takes the slow path

enum { MODE_MSG = 0, MODE_TYPE = 1 };

struct AggDir {
  const int32_t* rowptr;
  const int32_t* src;
  const int32_t* rel;
  const float* w;
  const float* table;
};

struct AggParams {
  AggDir dir[2];
  int ndir;
  const float* prior;
  const float* ins;     // [B, I, D]
  float* out;               // fp32 output (may be null when the bf16 planes are requested)
  __nv_bfloat16* out_hi;    // optional split-bf16 planes (hi + lo ~= value to 2^-18): the A operand layout of
  __nv_bfloat16* out_lo;    // the wgmma e2e GEMM (linear_tc.cu); same column indexing as `out`
  int64_t ld_planes;
  float* possible;
  int64_t out_row_stride, out_col0, seg_stride_j, seg_stride_dir;
  int B, N, D, I, j0;   // this launch handles instructions j0 .. j0+NI-1
  int64_t Nt, Fpad;
  __nv_bfloat16* out_bf;    // bf16 output instead of `out` (training under torch.autocast, GR_IO_BF16)
};

template <int VEC> struct Vec;
template <> struct Vec<4> { using T = float4; };
template <> struct Vec<2> { using T = float2; };
template <> struct Vec<1> { using T = float; };

template <int VEC>
__device__ __forceinline__ void ldg_vec(float (&v)[VEC], const void* p) {
  using T = typename Vec<VEC>::T;
  T t = __ldg(reinterpret_cast<const T*>(p));
  const float* f = reinterpret_cast<const float*>(&t);
#pragma unroll
  for (int i = 0; i < VEC; ++i) v[i] = f[i];
}

template <int VEC>
__device__ __forceinline__ void st_vec(float* p, const float (&v)[VEC]) {
  using T = typename Vec<VEC>::T;
  T t;
  float* f = reinterpret_cast<float*>(&t);
#pragma unroll
  for (int i = 0; i < VEC; ++i) f[i] = v[i];
  *reinterpret_cast<T*>(p) = t;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// y -> (hi, lo) bf16 pair per element, hi = bf16(y), lo = bf16(y - hi), with packed conversions
// (cvt.rn.bf16x2.f32); the caller predicates the store.
template <int VEC>
struct SplitVec {
  uint32_t h[(VEC + 1) / 2], l[(VEC + 1) / 2];
};

template <int VEC>
__device__ __forceinline__ SplitVec<VEC> split_vec(const float (&y)[VEC]) {
  SplitVec<VEC> r;
  if constexpr (VEC % 2 == 0) {
#pragma unroll
    for (int k = 0; k < VEC; k += 2) {
      const __nv_bfloat162 h2 = __floats2bfloat162_rn(y[k], y[k + 1]);
      const float2 hf = __bfloat1622float2(h2);
      const __nv_bfloat162 l2 = __floats2bfloat162_rn(y[k] - hf.x, y[k + 1] - hf.y);
      r.h[k / 2] = *reinterpret_cast<const uint32_t*>(&h2);
      r.l[k / 2] = *reinterpret_cast<const uint32_t*>(&l2);
    }
  } else {
    const __nv_bfloat16 h = __float2bfloat16_rn(y[0]);
    const __nv_bfloat16 l = __float2bfloat16_rn(y[0] - __bfloat162float(h));
    r.h[0] = *reinterpret_cast<const unsigned short*>(&h);
    r.l[0] = *reinterpret_cast<const unsigned short*>(&l);
  }
  return r;
}

// bf16 store of y rounded to nearest even (the packed conversions round each element like __float2bfloat16_rn)
template <int VEC>
__device__ __forceinline__ void st_bf16(__nv_bfloat16* p, const float (&y)[VEC]) {
  if constexpr (VEC == 4) {
    const __nv_bfloat162 a = __floats2bfloat162_rn(y[0], y[1]), b = __floats2bfloat162_rn(y[2], y[3]);
    *reinterpret_cast<uint2*>(p) =
        make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
  } else if constexpr (VEC == 2) {
    *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(y[0], y[1]);
  } else {
    *p = __float2bfloat16_rn(y[0]);
  }
}

template <int VEC>
__device__ __forceinline__ void st_split(__nv_bfloat16* ph, __nv_bfloat16* pl, const SplitVec<VEC>& r) {
  if constexpr (VEC == 4) {
    *reinterpret_cast<uint2*>(ph) = make_uint2(r.h[0], r.h[1]);
    *reinterpret_cast<uint2*>(pl) = make_uint2(r.l[0], r.l[1]);
  } else if constexpr (VEC == 2) {
    *reinterpret_cast<uint32_t*>(ph) = r.h[0];
    *reinterpret_cast<uint32_t*>(pl) = r.l[0];
  } else {
    *reinterpret_cast<unsigned short*>(ph) = (unsigned short)r.h[0];
    *reinterpret_cast<unsigned short*>(pl) = (unsigned short)r.l[0];
  }
}

// coefficient of one edge: c = w*(w*prior[src]) (reasongnn.py:80-84 applies the COO value twice when
// normalized_gnn is on); TypeLayer: c = w (layer_init.py:39-42,52-53)
template <int MODE>
__device__ __forceinline__ float edge_coeff(const AggParams& p, const AggDir& d, int64_t e, int s) {
  float w = d.w ? d.w[e] : 1.0f;
  if (MODE == MODE_TYPE) return w;
  float pr = p.prior[s];
  return w * (w * pr);
}

// Two running sums per feature element, independent of the instruction:
//   A = sum_e c_e * relu(v_e)     S = sum_e c_e * v_e       (=> sum_e c_e * relu(-v_e) = A - S)
// accumulated as fp32 pairs (ffma2) when VEC is even.  If every v_e >= 0 the two
// chains execute bit-identical operations, so A - S is exactly 0 where the true value is 0.
template <int VEC, int MODE>
__device__ __forceinline__ void accumulate(float (&A)[VEC], float (&S)[VEC], const float (&v)[VEC], float c) {
  if constexpr (VEC % 2 == 0) {
    const float2 cc = make_float2(c, c);
#pragma unroll
    for (int k = 0; k < VEC; k += 2) {
      const float2 vv = make_float2(v[k], v[k + 1]);
      float2 s2 = ffma2(cc, vv, make_float2(S[k], S[k + 1]));
      S[k] = s2.x; S[k + 1] = s2.y;
      if (MODE == MODE_MSG) {
        const float2 vp = make_float2(fmaxf(vv.x, 0.f), fmaxf(vv.y, 0.f));
        float2 a2 = ffma2(cc, vp, make_float2(A[k], A[k + 1]));
        A[k] = a2.x; A[k + 1] = a2.y;
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      S[k] = fmaf(c, v[k], S[k]);
      if (MODE == MODE_MSG) A[k] = fmaf(c, fmaxf(v[k], 0.f), A[k]);
    }
  }
}

// y = xp * A + xn * (A - S)   with xp = relu(x), xn = relu(-x)   (exactly one of xp, xn is non-zero)
template <int VEC>
__device__ __forceinline__ void msg_epilogue(float (&y)[VEC], const float (&xp)[VEC], const float (&xn)[VEC],
                                             const float (&A)[VEC], const float (&T)[VEC]) {
  if constexpr (VEC % 2 == 0) {
#pragma unroll
    for (int k = 0; k < VEC; k += 2) {
      float2 r = fmul2(make_float2(xp[k], xp[k + 1]), make_float2(A[k], A[k + 1]));
      r = ffma2(make_float2(xn[k], xn[k + 1]), make_float2(T[k], T[k + 1]), r);
      y[k] = r.x; y[k + 1] = r.y;
    }
  } else {
#pragma unroll
    for (int k = 0; k < VEC; ++k) y[k] = fmaf(xn[k], T[k], xp[k] * A[k]);
  }
}

// CH = feature chunks per lane (1 or 2): one pass covers 32*VEC*CH columns.
// PLANES: output goes to the split-bf16 planes (p.out_hi/p.out_lo) instead of fp32 p.out.
// DT / SEGP: compile-time feature dimension and output-segment pitch (0 = runtime p.D / p.seg_stride_*).  With
// both fixed every output-segment offset is an immediate, which removes the per-store address arithmetic the
// generic kernel spends most of its issue slots on; the dual-direction ReaRev layout (segment 2j+d at column
// (2j+d)*SEGP) is assumed when DT != 0.
// OUT_BF16: the fp32 values of `out` are stored rounded to bf16 in p.out_bf (same row stride / column indexing).
template <int VEC, int CH, int NI, int MODE, bool USE_TMA, bool PLANES, int DT, int SEGP, bool OUT_BF16 = false>
__global__ void __launch_bounds__(kThreads, 2) agg_kernel(const AggParams p) {
  __shared__ int32_t s_rowptr[2][kRows + 1];
  __shared__ int2 s_rc[2][kEdgeCap];                       // {table byte offset rel*D*4, float_as_int(c)}
  __shared__ __align__(16) int32_t s_src[USE_TMA ? 2 : 1][USE_TMA ? kEdgeCap + 8 : 1];
  __shared__ __align__(16) int32_t s_rel[USE_TMA ? 2 : 1][USE_TMA ? kEdgeCap + 8 : 1];
  __shared__ __align__(8) uint64_t s_bar;
  __shared__ unsigned char s_any[2][kRows];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * kRows;
  const int nrows = (int)min((int64_t)kRows, p.Nt - r0);
  const int D = DT ? DT : p.D, N = p.N;
  const int b0 = (int)(r0 / N);                 // one 64-bit division per thread per CTA
  const int rem0 = (int)(r0 - (int64_t)b0 * N);

  // ---------------- phase 1: stage row pointers + edge slice -----------------------------------------
  if (tid <= nrows) {
    s_rowptr[0][tid] = p.dir[0].rowptr[r0 + tid];
    if (p.ndir == 2) s_rowptr[1][tid] = p.dir[1].rowptr[r0 + tid];
  }
  if (USE_TMA && tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&s_bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (USE_TMA) {
    if (tid == 0) {
      uint32_t total = 0;
      uint32_t bytes[2];
      int64_t abeg[2];
      for (int d = 0; d < p.ndir; ++d) {
        int64_t eb = s_rowptr[d][0], ee = s_rowptr[d][nrows];
        int64_t ne = min(ee - eb, (int64_t)kEdgeCap);
        abeg[d] = eb & ~(int64_t)3;
        int64_t aend = min((eb + ne + 3) & ~(int64_t)3, p.Fpad);
        bytes[d] = ne > 0 ? (uint32_t)((aend - abeg[d]) * 4) : 0u;
        total += 2 * bytes[d];
      }
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&s_bar)),
                   "r"(total)
                   : "memory");
      for (int d = 0; d < p.ndir; ++d) {
        if (bytes[d] == 0) continue;
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
                "r"(smem_u32(&s_src[d][0])),
            "l"(p.dir[d].src + abeg[d]), "r"(bytes[d]), "r"(smem_u32(&s_bar))
            : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
                "r"(smem_u32(&s_rel[d][0])),
            "l"(p.dir[d].rel + abeg[d]), "r"(bytes[d]), "r"(smem_u32(&s_bar))
            : "memory");
      }
    }
    // everyone waits for the bulk copies (phase parity 0: the barrier is used once per CTA)
    uint32_t ok = 0;
    while (!ok) {
      asm volatile(
          "{\n\t.reg .pred p;\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
          "selp.u32 %0, 1, 0, p;\n\t}"
          : "=r"(ok)
          : "r"(smem_u32(&s_bar)), "r"(0)
          : "memory");
    }
  }
  for (int d = 0; d < p.ndir; ++d) {
    const AggDir& dd = p.dir[d];
    const int64_t eb = s_rowptr[d][0];
    const int ne = (int)min((int64_t)(s_rowptr[d][nrows] - eb), (int64_t)kEdgeCap);
    const int shift = (int)(eb & 3);
    for (int i = tid; i < ne; i += kThreads) {
      int s, r;
      if (USE_TMA) {
        s = s_src[d][shift + i];
        r = s_rel[d][shift + i];
      } else {
        s = dd.src ? dd.src[eb + i] : 0;
        r = dd.rel[eb + i];
      }
      float c = edge_coeff<MODE>(p, dd, eb + i, s);
      s_rc[d][i] = make_int2((int)((uint32_t)r * (uint32_t)D * 4u), __float_as_int(c));
    }
  }
  __syncthreads();
  // phase 1b: per (direction, row): does any edge carry a non-zero coefficient?  (first layer of every
  // iteration: the prior is the one-hot seed, almost every row is exactly zero -> pure zero store)
  if (tid < 2 * kRows) {
    const int d = tid / kRows, lr = tid % kRows;
    unsigned char any = 0;
    if (d < p.ndir && lr < nrows) {
      const int64_t ebase = s_rowptr[d][0];
      const int beg = (int)(s_rowptr[d][lr] - ebase), end = (int)(s_rowptr[d][lr + 1] - ebase);
      if (MODE == MODE_TYPE || end > kEdgeCap) any = 1;
      for (int i = beg; i < min(end, kEdgeCap) && !any; ++i) any = (s_rc[d][i].y << 1) != 0;   // c != +-0
    }
    s_any[d][lr] = any;
  }
  __syncthreads();

  // ---------------- phase 2: one warp per destination row, lanes across features ----------------------
  constexpr int PASS_COLS = 32 * VEC * CH;
  constexpr int CHW = 32 * VEC;                       // columns per chunk
  const int64_t ld = PLANES ? p.ld_planes : p.out_row_stride;
  for (int c0 = 0; c0 < D; c0 += PASS_COLS) {
    const int col0 = c0 + lane * VEC;                 // this lane's column in chunk 0
    // columns written per segment: the bf16 planes also get the zero padding up to the 16-column (32-byte)
    // boundary so that every store completes whole sectors (partial-sector writes halve HBM write throughput)
    const int seg_pitch_rt = (int)(p.seg_stride_dir > 0 ? p.seg_stride_dir : (p.seg_stride_j > 0 ? p.seg_stride_j : D));
    const int Dw = PLANES ? (DT ? SEGP : min((D + 15) / 16 * 16, MODE == MODE_TYPE ? (int)ld : max(seg_pitch_rt, D))) : D;
    bool act[CH], wr[CH];
    const char* tcol[2][CH];     // per-direction table column bases; inactive lanes are clamped to column 0
#pragma unroll
    for (int ch = 0; ch < CH; ++ch) {
      act[ch] = col0 + ch * CHW < D;
      wr[ch] = col0 + ch * CHW < Dw;
      const int lc = act[ch] ? col0 + ch * CHW : 0;
#pragma unroll
      for (int d = 0; d < 2; ++d)
        tcol[d][ch] = reinterpret_cast<const char*>(p.dir[d < p.ndir ? d : 0].table) + (size_t)lc * 4;
    }
    // warp-uniform element offsets of every (direction, instruction) segment inside an output row
    int seg[2][NI];
#pragma unroll
    for (int d = 0; d < 2; ++d)
#pragma unroll
      for (int j = 0; j < NI; ++j)
        seg[d][j] = DT ? (d * SEGP + j * 2 * SEGP)   // + j0 * 2 * SEGP folded into the lane base pointers
                       : (int)(d * p.seg_stride_dir + (int64_t)(p.j0 + j) * p.seg_stride_j);
    const int64_t j0off = DT ? (int64_t)p.j0 * 2 * SEGP : 0;

    int cur_b = -1;
    float xp[NI][CH][VEC], xn[NI][CH][VEC];   // relu(ins), relu(-ins) of the current question
#pragma unroll
    for (int j = 0; j < NI; ++j)
#pragma unroll
      for (int ch = 0; ch < CH; ++ch)
#pragma unroll
        for (int k = 0; k < VEC; ++k) xp[j][ch][k] = xn[j][ch][k] = 0.f;

    // per-lane base pointers of the tile (row 0, this lane's chunk-0 column)
    float* const out_lane = PLANES || OUT_BF16 ? nullptr : p.out + r0 * ld + p.out_col0 + col0 + j0off;
    __nv_bfloat16* const bf_lane = OUT_BF16 ? p.out_bf + r0 * ld + p.out_col0 + col0 + j0off : nullptr;
    __nv_bfloat16* const hi_lane = PLANES ? p.out_hi + r0 * ld + p.out_col0 + col0 + j0off : nullptr;
    __nv_bfloat16* const lo_lane = PLANES ? p.out_lo + r0 * ld + p.out_col0 + col0 + j0off : nullptr;

    const int lr_switch = N - rem0;      // first tile row that belongs to question b0 + 1 (N >= kRows assumed
                                         // for the fast path; the while loop below handles tiny N)
    for (int lr = warp; lr < nrows; lr += kWarps) {
      if (MODE == MODE_MSG) {
        int b = b0 + (lr >= lr_switch ? 1 : 0);
        if (N < kRows) {                 // rare: several questions inside one tile
          int q = rem0 + lr;
          b = b0;
          while (q >= N) { q -= N; ++b; }
        }
        if (b != cur_b) {
          cur_b = b;
#pragma unroll
          for (int j = 0; j < NI; ++j)
#pragma unroll
            for (int ch = 0; ch < CH; ++ch) {
              float x[VEC];
              ldg_vec<VEC>(x, p.ins + ((int64_t)b * p.I + p.j0 + j) * D + (act[ch] ? col0 + ch * CHW : 0));
#pragma unroll
              for (int k = 0; k < VEC; ++k) {   // lanes past D carry x = 0 -> they produce exact zeros
                xp[j][ch][k] = act[ch] ? fmaxf(x[k], 0.f) : 0.f;
                xn[j][ch][k] = act[ch] ? fmaxf(-x[k], 0.f) : 0.f;
              }
            }
        }
      }
      const int64_t rowoff = (int64_t)lr * ld;        // warp-uniform
      float* const orow = PLANES || OUT_BF16 ? nullptr : out_lane + rowoff;
      __nv_bfloat16* const brow = OUT_BF16 ? bf_lane + rowoff : nullptr;
      __nv_bfloat16* const hrow = PLANES ? hi_lane + rowoff : nullptr;
      __nv_bfloat16* const lrow = PLANES ? lo_lane + rowoff : nullptr;
      auto store = [&](int off, bool pred, const float (&y)[VEC]) {   // off: warp-uniform element offset
        if constexpr (PLANES) {
          const SplitVec<VEC> sv = split_vec<VEC>(y);
          if (pred) st_split<VEC>(hrow + off, lrow + off, sv);
        } else if constexpr (OUT_BF16) {
          if (pred) st_bf16<VEC>(brow + off, y);
        } else {
          if (pred) st_vec<VEC>(orow + off, y);
        }
      };
      auto store_zero = [&](int off, bool pred) {
        if constexpr (PLANES) {
          SplitVec<VEC> sv;
#pragma unroll
          for (int k = 0; k < (VEC + 1) / 2; ++k) sv.h[k] = sv.l[k] = 0u;
          if (pred) st_split<VEC>(hrow + off, lrow + off, sv);
        } else {
          float z[VEC];
#pragma unroll
          for (int k = 0; k < VEC; ++k) z[k] = 0.f;
          if constexpr (OUT_BF16) {
            if (pred) st_bf16<VEC>(brow + off, z);
          } else {
            if (pred) st_vec<VEC>(orow + off, z);
          }
        }
      };
      float tsum[CH][VEC];   // MODE_TYPE: sum over both directions
#pragma unroll
      for (int ch = 0; ch < CH; ++ch)
#pragma unroll
        for (int k = 0; k < VEC; ++k) tsum[ch][k] = 0.f;

#pragma unroll
      for (int d = 0; d < 2; ++d) {
        if (d >= p.ndir) break;
        const AggDir& dd = p.dir[d];
        const int ebase = s_rowptr[d][0];
        const int beg = s_rowptr[d][lr] - ebase, end = s_rowptr[d][lr + 1] - ebase;

        if (MODE == MODE_MSG && p.possible && c0 == 0 && d == 0 && p.j0 == 0) {   // nsm_gnn.py:101-103
          float cs = 0.f;
          for (int i = beg; i < min(end, kEdgeCap); ++i) cs += __int_as_float(s_rc[d][i].y);
          for (int i = max(beg, kEdgeCap); i < end; ++i)
            cs += edge_coeff<MODE>(p, dd, (int64_t)ebase + i, dd.src[(int64_t)ebase + i]);
          if (lane == 0) p.possible[r0 + lr] = cs > 1e-10f ? 1.f : 0.f;
        }

        if (MODE == MODE_MSG && !s_any[d][lr]) {
#pragma unroll
          for (int j = 0; j < NI; ++j)
#pragma unroll
            for (int ch = 0; ch < CH; ++ch) store_zero(seg[d][j] + ch * CHW, wr[ch]);
          continue;
        }

        float A[CH][VEC], S[CH][VEC];
#pragma unroll
        for (int ch = 0; ch < CH; ++ch)
#pragma unroll
          for (int k = 0; k < VEC; ++k) A[ch][k] = S[ch][k] = 0.f;

        // edges in branch-free blocks of 4: slots past the row end re-read the last edge with c forced to
        // 0 (fma(0, x, acc) == acc exactly for finite table values), so every block issues its loads together
        const int fast_end = min(end, kEdgeCap);
        for (int i = beg; i < fast_end; i += 4) {
          int2 m[4];
          float v[4][CH][VEC];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            m[u] = s_rc[d][min(i + u, fast_end - 1)];
            if (i + u >= fast_end) m[u].y = 0;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int ch = 0; ch < CH; ++ch) ldg_vec<VEC>(v[u][ch], tcol[d][ch] + (uint32_t)m[u].x);
#pragma unroll
          for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int ch = 0; ch < CH; ++ch)
              accumulate<VEC, MODE>(A[ch], S[ch], v[u][ch], __int_as_float(m[u].y));
        }
        for (int i = max(beg, kEdgeCap); i < end; ++i) {   // slow path: edge slice overflowed the staging buffer
          const int64_t e = (int64_t)ebase + i;
          const int s = dd.src ? dd.src[e] : 0;
          const uint32_t off = (uint32_t)dd.rel[e] * (uint32_t)D * 4u;
          const float c = edge_coeff<MODE>(p, dd, e, s);
#pragma unroll
          for (int ch = 0; ch < CH; ++ch) {
            float v[VEC];
            ldg_vec<VEC>(v, tcol[d][ch] + off);
            accumulate<VEC, MODE>(A[ch], S[ch], v, c);
          }
        }

        if (MODE == MODE_MSG) {
#pragma unroll
          for (int ch = 0; ch < CH; ++ch) {
            float T[VEC];   // A - S = sum c*relu(-v)
            if constexpr (VEC % 2 == 0) {
#pragma unroll
              for (int k = 0; k < VEC; k += 2) {
                float2 t2 = ffma2(make_float2(S[ch][k], S[ch][k + 1]), make_float2(-1.f, -1.f),
                                       make_float2(A[ch][k], A[ch][k + 1]));
                T[k] = t2.x; T[k + 1] = t2.y;
              }
            } else {
#pragma unroll
              for (int k = 0; k < VEC; ++k) T[k] = A[ch][k] - S[ch][k];
            }
#pragma unroll
            for (int j = 0; j < NI; ++j) {
              float y[VEC];
              msg_epilogue<VEC>(y, xp[j][ch], xn[j][ch], A[ch], T);
              store(seg[d][j] + ch * CHW, wr[ch], y);
            }
          }
        } else {
#pragma unroll
          for (int ch = 0; ch < CH; ++ch)
#pragma unroll
            for (int k = 0; k < VEC; ++k) tsum[ch][k] += S[ch][k];   // (sum_tail) + (sum_head), layer_init.py:57
        }
      }
      if (MODE == MODE_TYPE) {
#pragma unroll
        for (int ch = 0; ch < CH; ++ch) {
          float y[VEC];
#pragma unroll
          for (int k = 0; k < VEC; ++k) y[k] = act[ch] ? fmaxf(tsum[ch][k], 0.f) : 0.f;
          store(ch * CHW, wr[ch], y);
        }
      }
    }
  }
}

template <int VEC, int CH, int NI, int MODE, int DT, int SEGP>
int launch_agg3(const AggParams& p, bool tma, cudaStream_t stream) {
  unsigned grid = (unsigned)ceil_div(p.Nt, kRows);
  if (p.out) {
    if (tma && DT == 0)
      agg_kernel<VEC, CH, NI, MODE, (DT == 0), false, DT, SEGP><<<grid, kThreads, 0, stream>>>(p);
    else
      agg_kernel<VEC, CH, NI, MODE, false, false, DT, SEGP><<<grid, kThreads, 0, stream>>>(p);
    GR_CHECK_LAUNCH();
  }
  if constexpr (DT == 0) {   // bf16 output: single-direction training calls only, never the DT-specialised layout
    if (p.out_bf) {
      agg_kernel<VEC, CH, NI, MODE, false, false, DT, SEGP, true><<<grid, kThreads, 0, stream>>>(p);
      GR_CHECK_LAUNCH();
    }
  }
  if (p.out_hi) {   // split-bf16 planes (a second launch only if the caller asked for both formats)
    if (tma && DT == 0)
      agg_kernel<VEC, CH, NI, MODE, (DT == 0), true, DT, SEGP><<<grid, kThreads, 0, stream>>>(p);
    else
      agg_kernel<VEC, CH, NI, MODE, false, true, DT, SEGP><<<grid, kThreads, 0, stream>>>(p);
    GR_CHECK_LAUNCH();
  }
  return GR_OK;
}

template <int VEC, int CH, int NI, int MODE>
int launch_agg2(const AggParams& p, bool tma, cudaStream_t stream) {
  // specialised instance for the WebQSP-shape feature width (BASELINE cfg1/2/4: D = 200) in the
  // dual-direction ReaRev layout; everything else takes the runtime-D kernel
  if constexpr (VEC == 4 && CH == 2 && MODE == MODE_MSG) {
    if (p.D == 200 && p.ndir == 2 && !tma) {
      if (p.seg_stride_dir == 200 && p.seg_stride_j == 400)
        return launch_agg3<VEC, CH, NI, MODE, 200, 200>(p, tma, stream);
      if (p.seg_stride_dir == 208 && p.seg_stride_j == 416)   // 32-byte aligned bf16 plane segments
        return launch_agg3<VEC, CH, NI, MODE, 200, 208>(p, tma, stream);
    }
  }
  return launch_agg3<VEC, CH, NI, MODE, 0, 0>(p, tma, stream);
}

template <int MODE>
int launch_agg(AggParams p, cudaStream_t stream) {
  // vector width from alignment of D, strides and base pointers
  auto aligned = [&](int v) {
    size_t a = (size_t)v * 4;
    bool ok = p.D % v == 0 && p.out_row_stride % v == 0 && p.out_col0 % v == 0 &&
              p.seg_stride_j % v == 0 && p.seg_stride_dir % v == 0 &&
              (reinterpret_cast<size_t>(p.out) % a) == 0 && (reinterpret_cast<size_t>(p.ins) % a) == 0 &&
              p.ld_planes % v == 0 && (reinterpret_cast<size_t>(p.out_hi) % (a / 2)) == 0 &&
              (reinterpret_cast<size_t>(p.out_lo) % (a / 2)) == 0 &&
              (reinterpret_cast<size_t>(p.out_bf) % (a / 2)) == 0;
    for (int d = 0; d < p.ndir; ++d) ok = ok && (reinterpret_cast<size_t>(p.dir[d].table) % a) == 0;
    return ok;
  };
  const int vec = aligned(4) ? 4 : (aligned(2) ? 2 : 1);
  const int ch = p.D > 32 * vec ? 2 : 1;
  bool tma = g_opt_agg_tma != 0 && MODE == MODE_MSG;
  for (int d = 0; d < p.ndir && tma; ++d)
    tma = (reinterpret_cast<size_t>(p.dir[d].src) % 16) == 0 &&
          (reinterpret_cast<size_t>(p.dir[d].rel) % 16) == 0;
  // f(int_c<vec>{}, int_c<ch>{}): vec is 4, 2 or 1 and ch 1 or 2
  auto with_vec_ch = [&](auto f) {
    auto with_ch = [&](auto v) { return ch == 1 ? f(v, int_c<1>{}) : f(v, int_c<2>{}); };
    return vec == 4 ? with_ch(int_c<4>{}) : vec == 2 ? with_ch(int_c<2>{}) : with_ch(int_c<1>{});
  };
  if constexpr (MODE == MODE_TYPE) {
    return with_vec_ch([&](auto v, auto c) {
      return launch_agg2<decltype(v)::value, decltype(c)::value, 1, MODE_TYPE>(p, false, stream);
    });
  } else {
    for (int j0 = 0; j0 < p.I; j0 += 4) {   // instructions in groups of <= 4 (epilogue register budget)
      p.j0 = j0;
      const int rc = with_vec_ch([&](auto v, auto c) {
        return with_ni(std::min(4, p.I - j0), [&](auto ni) {
          return launch_agg2<decltype(v)::value, decltype(c)::value, decltype(ni)::value, MODE_MSG>(p, tma, stream);
        });
      });
      if (rc != GR_OK) return rc;
    }
    return GR_OK;
  }
}

}  // namespace
}  // namespace gr

namespace gr {
namespace {
// Store-pattern probe (scripts/agg_probe.py): writes zeros to the neighbour columns of the bf16 planes with
// the aggregation kernel's exact thread->address mapping (64-row CTA tiles, one warp per row, lanes across
// 2 chunks of 4 bf16, 8 stores per direction) but WITHOUT phase 1 / edge work.  mode 0: STG.64 per lane as the
// kernel does; mode 1: same bytes written as contiguous 16-byte lanes (row-major sweep of the 1600-byte span).
__global__ void __launch_bounds__(kThreads, 2)
agg_store_probe_kernel(__nv_bfloat16* hi, __nv_bfloat16* lo, int64_t Nt, int64_t ld, int col_start, int ncols,
                       int mode) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * kRows;
  const int nrows = (int)min((int64_t)kRows, Nt - r0);
  for (int lr = warp; lr < nrows; lr += kWarps) {
    __nv_bfloat16* h = hi + (r0 + lr) * ld + col_start;
    __nv_bfloat16* l = lo + (r0 + lr) * ld + col_start;
    if (mode == 0) {          // 8-byte lanes (what the planes kernel does)
      for (int c = lane * 4; c < ncols; c += 128) {
        *reinterpret_cast<uint2*>(h + c) = make_uint2(0u, 0u);
        *reinterpret_cast<uint2*>(l + c) = make_uint2(0u, 0u);
      }
    } else if (mode == 1) {   // 16-byte lanes
      for (int c = lane * 8; c < ncols; c += 256) {
        *reinterpret_cast<uint4*>(h + c) = make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(l + c) = make_uint4(0u, 0u, 0u, 0u);
      }
    } else {                  // single plane, 16-byte lanes, twice the columns (= one fp32-wide row)
      for (int c = lane * 8; c < 2 * ncols; c += 256)
        *reinterpret_cast<uint4*>(h + c) = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}
}  // namespace
}  // namespace gr

extern "C" int gr_debug_store_probe(void* hi, void* lo, int64_t Nt, int64_t ld, int col_start, int ncols,
                                    int mode, void* stream_) {
  using namespace gr;
  GR_CHECK_ARG(hi && lo && Nt > 0, "bad args");
  unsigned grid = (unsigned)ceil_div(Nt, kRows);
  agg_store_probe_kernel<<<grid, kThreads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<__nv_bfloat16*>(hi), reinterpret_cast<__nv_bfloat16*>(lo), Nt, ld, col_start, ncols, mode);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_aggregate_ex(const int32_t* rowptr, const int32_t* src, const int32_t* rel, const float* w,
                               const float* prior, const float* table, const float* ins, void* out,
                               int64_t out_row_stride, int64_t out_col0, int64_t seg_stride, float* possible, int B,
                               int N, int D, int I, int64_t F, uint32_t io, void* stream_) {
  using namespace gr;
  if (int rc = check_io(__func__, io)) return rc;
  GR_CHECK_ARG(rowptr && prior && table && ins && out, "null pointer");
  GR_CHECK_ARG(F == 0 || (src && rel), "null edge arrays");
  GR_CHECK_ARG(B > 0 && N > 0 && D > 0 && I > 0, "B, N, D, I must be positive");
  AggParams p{};
  p.dir[0] = AggDir{rowptr, src, rel, w, table};
  p.ndir = 1;
  p.prior = prior; p.ins = ins; p.possible = possible;
  if (io_bf16(io)) p.out_bf = static_cast<__nv_bfloat16*>(out);
  else p.out = static_cast<float*>(out);
  p.out_row_stride = out_row_stride; p.out_col0 = out_col0;
  p.seg_stride_j = seg_stride; p.seg_stride_dir = 0;
  p.B = B; p.N = N; p.D = D; p.I = I; p.j0 = 0;
  p.Nt = (int64_t)B * N; p.Fpad = gr_pad4(F);
  return launch_agg<MODE_MSG>(p, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_aggregate(const int32_t* rowptr, const int32_t* src, const int32_t* rel,
                            const float* w, const float* prior, const float* table, const float* ins,
                            float* out, int64_t out_row_stride, int64_t out_col0, int64_t seg_stride,
                            float* possible, int B, int N, int D, int I, int64_t F, void* stream_) {
  return gr_aggregate_ex(rowptr, src, rel, w, prior, table, ins, out, out_row_stride, out_col0, seg_stride, possible,
                         B, N, D, I, F, 0u, stream_);
}

extern "C" int gr_aggregate_dual(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                                 const float* w_t, const int32_t* rowptr_h, const int32_t* src_h,
                                 const int32_t* rel_h, const float* w_h, const float* prior,
                                 const float* table_fwd, const float* table_inv, const float* ins,
                                 float* out, int64_t out_row_stride, int64_t out_col0, int64_t seg_pitch,
                                 void* out_hi, void* out_lo, int64_t ld_planes, int B, int N, int D, int I,
                                 int64_t F, void* stream_) {
  using namespace gr;
  GR_CHECK_ARG(rowptr_t && rowptr_h && prior && table_fwd && table_inv && ins, "null pointer");
  GR_CHECK_ARG(out || (out_hi && out_lo), "no output requested");
  GR_CHECK_ARG(!out_hi || (out_lo && ld_planes > 0), "out_lo / ld_planes missing");
  GR_CHECK_ARG(F == 0 || (src_t && rel_t && src_h && rel_h), "null edge arrays");
  GR_CHECK_ARG(B > 0 && N > 0 && D > 0 && I > 0, "B, N, D, I must be positive");
  AggParams p{};
  p.dir[0] = AggDir{rowptr_t, src_t, rel_t, w_t, table_fwd};
  p.dir[1] = AggDir{rowptr_h, src_h, rel_h, w_h, table_inv};
  p.ndir = 2;
  p.prior = prior; p.ins = ins; p.out = out; p.possible = nullptr;
  p.out_hi = reinterpret_cast<__nv_bfloat16*>(out_hi); p.out_lo = reinterpret_cast<__nv_bfloat16*>(out_lo);
  p.ld_planes = out_hi ? ld_planes : 0;
  p.out_row_stride = out_row_stride; p.out_col0 = out_col0;
  if (seg_pitch <= 0) seg_pitch = D;
  GR_CHECK_ARG(seg_pitch >= D, "seg_pitch smaller than D");
  p.seg_stride_j = 2 * seg_pitch; p.seg_stride_dir = seg_pitch;
  p.B = B; p.N = N; p.D = D; p.I = I; p.j0 = 0;
  p.Nt = (int64_t)B * N; p.Fpad = gr_pad4(F);
  return launch_agg<MODE_MSG>(p, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_type_layer_ex(const int32_t* rowptr_t, const int32_t* rel_t, const float* w_t,
                                const int32_t* rowptr_h, const int32_t* rel_h, const float* w_h, const float* table,
                                void* out, int64_t out_row_stride, void* out_hi, void* out_lo, int64_t ld_planes,
                                int B, int N, int D, int64_t F, uint32_t io, void* stream_) {
  using namespace gr;
  if (int rc = check_io(__func__, io)) return rc;
  GR_CHECK_ARG(rowptr_t && rowptr_h && table, "null pointer");
  GR_CHECK_ARG(out || (out_hi && out_lo), "no output requested");
  GR_CHECK_ARG(F == 0 || (rel_t && rel_h), "null edge arrays");
  GR_CHECK_ARG(B > 0 && N > 0 && D > 0, "B, N, D must be positive");
  AggParams p{};
  p.dir[0] = AggDir{rowptr_t, nullptr, rel_t, w_t, table};
  p.dir[1] = AggDir{rowptr_h, nullptr, rel_h, w_h, table};
  p.ndir = 2;
  p.prior = nullptr; p.ins = nullptr; p.possible = nullptr;
  if (io_bf16(io)) p.out_bf = static_cast<__nv_bfloat16*>(out);
  else p.out = static_cast<float*>(out);
  p.out_hi = reinterpret_cast<__nv_bfloat16*>(out_hi); p.out_lo = reinterpret_cast<__nv_bfloat16*>(out_lo);
  p.ld_planes = out_hi ? ld_planes : 0;
  p.out_row_stride = out_row_stride; p.out_col0 = 0;
  p.seg_stride_j = 0; p.seg_stride_dir = 0;
  p.B = B; p.N = N; p.D = D; p.I = 1; p.j0 = 0;
  p.Nt = (int64_t)B * N; p.Fpad = gr_pad4(F);
  return launch_agg<MODE_TYPE>(p, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_type_layer(const int32_t* rowptr_t, const int32_t* rel_t, const float* w_t,
                             const int32_t* rowptr_h, const int32_t* rel_h, const float* w_h,
                             const float* table, float* out, int64_t out_row_stride, void* out_hi,
                             void* out_lo, int64_t ld_planes, int B, int N, int D, int64_t F,
                             void* stream_) {
  return gr_type_layer_ex(rowptr_t, rel_t, w_t, rowptr_h, rel_h, w_h, table, out, out_row_stride, out_hi, out_lo,
                          ld_planes, B, N, D, F, 0u, stream_);
}
