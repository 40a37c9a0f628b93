// Tensor-core linear layer for sm_90a:  C = act(A W^T + bias)  with fp32 in / fp32 out and fp32-class
// accuracy, via the 3-product split-bf16 scheme on wgmma:
//     x = hi + lo (hi = bf16(x), lo = bf16(x - hi));   A W^T ~= A_hi W_hi^T + A_hi W_lo^T + A_lo W_hi^T
// (dropped term A_lo W_lo^T <= 2^-18 relative).  All three products accumulate into one fp32 register
// accumulator.  This is the `e2e_linear` of ReasonGNNLayer.forward / NSMBaseLayer.forward
// (reference gnn/modules/kg_reasoning/reasongnn.py:163, nsm_gnn.py:63): a genuine dense contraction,
// M = B*N node rows, K = (2*num_ins+1)*D, N = D.
//
// Kernel: persistent, one 128-row tile of A at a time, full N (<= 256) per CTA.  Warpgroup 0 = TMA producer
// (cp.async.bulk.tensor, swizzled K-major tiles of the four bf16 planes into a ring of `stages` slots with
// full/empty mbarriers); warpgroups 1 and 2 = consumers, 64 rows each: one full-width wgmma.mma_async m64n{NP}k16
// from shared memory per product and K step (NP = n_pad rounded up to an instantiated width: 64, 128, 208 or 256),
// fp32 accumulator in registers, then the epilogue (bias + relu + score dot,
// fp32 and bf16 hi/lo plane outputs, staged TMA stores or direct stores).  With tc_cluster = 2, clusters of 2 CTAs
// share the W tiles by TMA multicast (single-CTA clusters measured faster and are the default).  GR_LINEAR_K_GROUPED
// walks a segmented K in the fused layer kernel's k-block order (GroupedK, wgmma.cuh) and so returns its bits, from the
// segment layout or (GR_LINEAR_K_ORDER_PLANES) from the K-order layout gr_aggregate_dual_abs_ex writes.
//
// Roofline: tensor-pipe work 3 * 2*M*N*K flop; HBM traffic ~ 2 planes * M*K*2 B = M*K*4 B (same as fp32 A).
#include "wgmma.cuh"

namespace gr {

int g_tc_cluster = 1;      // gr_set_option("tc_cluster", 1|2): 2 = CTA pairs share the W tiles by TMA multicast
int g_tc_bk = 32;          // gr_set_option("tc_bk", 32|64): k-block width (64B / 128B swizzle)
int g_tc_tma_store = 1;    // gr_set_option("tc_tma_store", 0|1): staged TMA-store epilogue vs direct per-row stores

namespace {

using namespace tc;
// k-block width BK (bf16 elements) is a template parameter: 64 (128-byte swizzle rows) or 32 (64-byte swizzle rows,
// twice as many, finer stages -> more TMA requests in flight)
constexpr int kThreads = 384;          // warpgroup 0: TMA producer; warpgroups 1, 2: consumers
constexpr int kConsumerWarps = 8;
// setmaxnreg budget: 384 threads x 168 registers at launch = 128 x 40 (producer) + 256 x 232 (consumers)
constexpr int kLaunchRegs = 168, kProducerRegs = 40, kConsumerRegs = 232;
static_assert(128 * kProducerRegs + 256 * kConsumerRegs <= kThreads * kLaunchRegs, "register budget");

// ---------------------------------------------------------------------------------------------------
// fp32 -> (hi, lo) bf16 planes
// ---------------------------------------------------------------------------------------------------
// W [N, nseg*seg] dense -> hi/lo planes [N, >= nseg*pitch] with segment s at columns [s*pitch, s*pitch+seg),
// zeros in the padding columns (matches the padded activation-plane layout)
__global__ void split_bf16_seg_kernel(const float* __restrict__ W, int64_t ldw, int64_t N, int64_t Kpad,
                                      int seg, int pitch, __nv_bfloat16* __restrict__ hi,
                                      __nv_bfloat16* __restrict__ lo, int64_t ldo) {
  const int64_t total = N * Kpad;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t n = i / Kpad, k = i - n * Kpad;
    const int sidx = (int)(k / pitch), c = (int)(k - (int64_t)sidx * pitch);
    float v = c < seg ? __ldg(W + n * ldw + (int64_t)sidx * seg + c) : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[n * ldo + k] = h;
    lo[n * ldo + k] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

__global__ void split_bf16_kernel(const float* __restrict__ A, int64_t lda, int64_t M, int64_t K,
                                  __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                  int64_t ldo, int vec_ok, int vec_st) {
  const int64_t kq = (K + 3) / 4;
  const int64_t total = M * kq;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t m = i / kq, k = (i - m * kq) * 4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    const float* src = A + m * lda + k;
    if (vec_ok && k + 3 < K) {
      float4 t = __ldg(reinterpret_cast<const float4*>(src));
      v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (k + q < K) v[q] = __ldg(src + q);
    }
    __nv_bfloat16 h[4], l[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      h[q] = __float2bfloat16_rn(v[q]);
      l[q] = __float2bfloat16_rn(v[q] - __bfloat162float(h[q]));
    }
    __nv_bfloat16* ph = hi + m * ldo + k;
    __nv_bfloat16* pl = lo + m * ldo + k;
    if (vec_st && k + 3 < ldo) {   // 8-byte aligned plane bases and ldo % 4 == 0
      *reinterpret_cast<uint2*>(ph) = *reinterpret_cast<uint2*>(h);
      *reinterpret_cast<uint2*>(pl) = *reinterpret_cast<uint2*>(l);
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (k + q < ldo) { ph[q] = h[q]; pl[q] = l[q]; }
    }
  }
}

struct TcParams {
  const float* bias;
  float* C;                 // fp32 output [M, N] (may be null)
  int64_t ldc;
  const float* c_rows;      // optional [M]: C receives only the rows m with c_rows[m] != 0 (direct stores), the other
                            //   rows keep what they held; every other output is written as without it
  __nv_bfloat16* c_hi;      // optional bf16 hi/lo planes of the output (next layer's A operand)
  __nv_bfloat16* c_lo;
  int64_t ldc16;
  const float* w_score;     // optional: score_func dot product (reasongnn.py:165): dots[m] = sum_n out[m,n] * w_score[n],
  float* dots;              //   dots[M + m] = 0 (the [2, M] partial-dot layout callers sum)
  int M, N, K, n_pad, n16, stages, num_tiles;   // n_pad = round16(N): the epilogue skips the columns beyond it
  uint32_t flags;
  int tma_store;            // 1: epilogue stages 64x16 chunks in smem and writes them with TMA stores
  // GR_LINEAR_K_GROUPED (the GROUPED instantiations; kg_T = 0 otherwise): T segments of kg_pitch columns walked in kg_G
  // column groups (GroupedK, wgmma.cuh), kg_nkb k-blocks of which kg_one0 .. kg_one1 - 1 are one k-step.  kg_nb0 > 0
  // (GR_LINEAR_K_ORDER_PLANES): the 2I neighbour segments lie in the K-order layout from column kg_nb0 on, kg_G counts
  // the full 32-column groups only and a 16-column last group follows as the h tail and I packed neighbour k-blocks
  int kg_T, kg_G, kg_pitch, kg_nkb, kg_one0, kg_one1, kg_nb0;
};

// ---------------------------------------------------------------------------------------------------
// the GEMM kernel: persistent over 128-row tiles.  Warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 =
// consumers: each issues wgmma for its 64 rows of the tile, holds the accumulator in registers and runs the epilogue.
// The producer runs up to `stages` k-blocks ahead, so the next tile's loads overlap this tile's epilogue.
// ---------------------------------------------------------------------------------------------------
// NP: accumulator width (W tile rows); CS: CTAs per cluster sharing W tiles by multicast; BK: k-block width;
// GROUPED: k-block kb = g*T + t reads A at column seg(t)*pitch + 32g and W at column 32 kb -- the k-block sequence, and
// so the per-element accumulation order, of fused_layer_kernel.  With kg_nb0 > 0 the same k16 steps come from the K-order
// layout: h boxes at column 32g, the neighbour boxes one after another from kg_nb0 (every box 64-byte aligned)
template <int NP, int CS, int BK, bool GROUPED>
__global__ void __launch_bounds__(kThreads, 1)
linear_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                 const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                 const __grid_constant__ CUtensorMap map_c, const __grid_constant__ CUtensorMap map_c_hi,
                 const __grid_constant__ CUtensorMap map_c_lo, const TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages] x {A_hi, A_lo, W_hi, W_lo}, epilogue staging, barriers, bias / score weights
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int a_bytes = BM * BK * 2;
  constexpr int w_bytes = NP * BK * 2;
  // GR_LINEAR_BF16_SINGLE: bf16 activation storage -- one product A_hi W_hi, stages hold {A_hi, W_hi} only
  const bool single = (p.flags & GR_LINEAR_BF16_SINGLE) != 0;
  const int w_off = single ? a_bytes : 2 * a_bytes;          // W_hi tile inside a stage
  const int stage_bytes = single ? a_bytes + w_bytes : 2 * a_bytes + 2 * w_bytes;
  uint8_t* s_out = smem + (size_t)p.stages * stage_bytes;    // [2 warpgroups] x kStageOutBytes (TMA-store source)
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_out + 2 * kStageOutBytes);
  uint64_t* full_bar = bars;                       // [stages]
  uint64_t* empty_bar = bars + p.stages;           // [stages]
  float* s_bias = reinterpret_cast<float*>(bars + 2 * p.stages);   // [256] zero padded
  float* s_ws = s_bias + 256;                                      // [256] zero padded
  for (int i = threadIdx.x; i < 256; i += kThreads) {
    s_bias[i] = (p.bias && i < p.N) ? p.bias[i] : 0.f;
    s_ws[i] = (p.w_score && i < p.N) ? p.w_score[i] : 0.f;
  }

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = GROUPED ? p.kg_nkb : (p.K + BK - 1) / BK;
  const int crank = CS > 1 ? (int)cluster_ctarank() : 0;
  const int ncluster = gridDim.x / CS, cid = blockIdx.x / CS;
  const int ngroups = (p.num_tiles + CS - 1) / CS;       // tile groups: CS consecutive 128-row tiles
  constexpr uint16_t kMask = (uint16_t)((1u << CS) - 1);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumerWarps * CS);     // every consumer warp of the cluster releases the slot
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (CS > 1) cluster_sync_all();                        // all barriers of the cluster are initialised

  if (warp < 4) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp == 0 && lane == 0) {
      uint32_t phase = 0;
      int s = 0;
      constexpr int w_rows = NP / CS;                    // W rows this CTA fetches (and multicasts)
      const int w_slice = w_rows * BK * 2;               // bytes
      for (int g = cid; g < ngroups; g += ncluster) {
        const int m0 = (g * CS + crank) * BM;            // may lie beyond M for the last group: zero-filled
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty_bar[s], phase ^ 1);
          uint8_t* st = smem + (size_t)s * stage_bytes;
          mbar_expect_tx(&full_bar[s], (uint32_t)stage_bytes);
          int a_col = kb * BK;
          if constexpr (GROUPED) {
            if (p.kg_nb0 == 0) {
              const int g = kb / p.kg_T, t = kb - g * p.kg_T, ni = p.kg_T >> 1;
              const int seg = t == 0 ? 0 : 1 + 2 * ((t - 1) % ni) + (t - 1) / ni;
              a_col = seg * p.kg_pitch + g * BK;
            } else {
              // K-order layout: group g (g = kg_G: the tail) is its h box, then its neighbour boxes, which continue the
              // ones of the groups before: kb - g - 1 neighbour boxes precede them
              const int g = min(kb / p.kg_T, p.kg_G), t = kb - g * p.kg_T;
              a_col = t == 0 ? g * BK : p.kg_nb0 + (kb - g - 1) * BK;
            }
          }
          tma_load_2d(st, &map_a_hi, &full_bar[s], a_col, m0);
          if (!single) tma_load_2d(st + a_bytes, &map_a_lo, &full_bar[s], a_col, m0);
          if (CS == 1) {
            tma_load_2d(st + w_off, &map_w_hi, &full_bar[s], kb * BK, 0);
            if (!single) tma_load_2d(st + w_off + w_bytes, &map_w_lo, &full_bar[s], kb * BK, 0);
          } else {
            tma_load_2d_mc(st + w_off + crank * w_slice, &map_w_hi, &full_bar[s], kb * BK,
                           crank * w_rows, kMask);
            if (!single)
              tma_load_2d_mc(st + w_off + w_bytes + crank * w_slice, &map_w_lo, &full_bar[s], kb * BK,
                             crank * w_rows, kMask);
          }
          if (++s == p.stages) { s = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: wgmma mainloop + epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    const int cw = (warp - 4) >> 2, wq = warp & 3;       // consumer warpgroup (row half), warp inside it
    const EpiOut e{s_bias, s_ws, (p.flags & GR_LINEAR_RELU) != 0};
    const int r = wq * 16 + (lane >> 2), cq = lane & 3;
    uint8_t* stg = s_out + (size_t)cw * kStageOutBytes;
    const bool issuer = wq == 0 && lane == 0;
    const bool vec_c = p.C && (p.ldc % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 7) == 0);
    const bool vec_h = p.c_hi && (p.ldc16 % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.c_hi) & 3) == 0) &&
                       ((reinterpret_cast<uintptr_t>(p.c_lo) & 3) == 0);
    uint32_t phase = 0;
    int s = 0;
    for (int g = cid; g < ngroups; g += ncluster) {
      const int tile = g * CS + crank;
      float acc[NP / 2];
#pragma unroll
      for (int i = 0; i < NP / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[s], phase);
        const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
        const uint32_t a_row = (uint32_t)(cw * WG_M * BK * 2);
        const uint64_t da_hi = make_smem_desc<BK>(sa + a_row), da_lo = make_smem_desc<BK>(sa + a_bytes + a_row);
        const uint64_t dw_hi = make_smem_desc<BK>(sa + w_off), dw_lo = make_smem_desc<BK>(sa + w_off + w_bytes);
        if constexpr (GROUPED) {
          // a 16-column h block (segment layout: every block of the last group) is one k-step: its own straight-line batch
          if (kb >= p.kg_one0 && kb < p.kg_one1) mma_kblock<NP, BK, 1, false>(acc, da_hi, da_lo, dw_hi, dw_lo);
          else mma_kblock<NP, BK, BK / MMA_K, false>(acc, da_hi, da_lo, dw_hi, dw_lo);
        } else if (single) {
          mma_kblock<NP, BK, BK / MMA_K, true>(acc, da_hi, da_lo, dw_hi, dw_lo);
        } else {
          mma_kblock<NP, BK, BK / MMA_K, false>(acc, da_hi, da_lo, dw_hi, dw_lo);
        }
        wgmma_wait<1>();                                 // the previous k-block's products are done: free its slot
        if (prev >= 0 && lane == 0) release_slot<CS>(&empty_bar[prev]);
        prev = s;
        if (++s == p.stages) { s = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) release_slot<CS>(&empty_bar[prev]);

      const int64_t row0 = (int64_t)tile * BM + cw * WG_M + r;
      // C rows r and r + 8 of this thread (all of them without c_rows)
      bool keep[2] = {true, true};
      if (p.c_rows) {
        keep[0] = row0 < p.M && p.c_rows[row0] != 0.f;
        keep[1] = row0 + 8 < p.M && p.c_rows[row0 + 8] != 0.f;
      }
      float dot0 = 0.f, dot1 = 0.f;
#pragma unroll
      for (int q = 0; q < NP / 16; ++q) {
        const int c0 = 16 * q;
        if (c0 >= p.n_pad) continue;
        float v[8];
        epi_values(acc, q, cq, e, v, dot0, dot1);
        if (p.tma_store) {
          // a row-selected C takes the direct stores below: a TMA store writes whole 64-row boxes
          epi_store_tma(v, stg, r, cq, issuer, 1 + cw, &map_c, &map_c_hi, &map_c_lo, p.C && !p.c_rows,
                        p.c_hi != nullptr, c0, tile * BM + cw * WG_M);
          if (!p.c_rows) continue;
        }
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int col = c0 + 8 * b + 2 * cq;
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int64_t row = row0 + 8 * hr;
            if (row >= p.M) continue;
            const float x0 = v[4 * b + 2 * hr], x1 = v[4 * b + 2 * hr + 1];
            if (p.C && keep[hr]) {
              float* c = p.C + row * p.ldc + col;
              if (vec_c && col + 1 < p.N) {
                *reinterpret_cast<float2*>(c) = make_float2(x0, x1);
              } else {
                if (col < p.N) c[0] = x0;
                if (col + 1 < p.N) c[1] = x1;
              }
            }
            if (p.c_hi && !p.tma_store) {
              // the planes also receive the (exactly zero) columns N .. n16
              uint32_t lo;
              const uint32_t hi = split_hi_lo(x0, x1, lo);
              unsigned short* ph = reinterpret_cast<unsigned short*>(p.c_hi + row * p.ldc16 + col);
              unsigned short* pl = reinterpret_cast<unsigned short*>(p.c_lo + row * p.ldc16 + col);
              if (vec_h && col + 1 < p.n16) {
                *reinterpret_cast<uint32_t*>(ph) = hi;
                *reinterpret_cast<uint32_t*>(pl) = lo;
              } else {
                if (col < p.n16) { ph[0] = (unsigned short)(hi & 0xFFFF); pl[0] = (unsigned short)(lo & 0xFFFF); }
                if (col + 1 < p.n16) { ph[1] = (unsigned short)(hi >> 16); pl[1] = (unsigned short)(lo >> 16); }
              }
            }
          }
        }
      }
      epi_dots(dot0, dot1, p.dots, row0, p.M, cq);
    }
    if (p.tma_store && issuer) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // stores complete
  }
  __syncthreads();
  if (CS > 1) cluster_sync_all();   // nobody exits while a peer may still multicast into / arrive on this CTA
}

struct TcPlan {
  int64_t kp;          // plane row stride (elements), multiple of 8
  int n_pad, np, stages, bk;   // np: instantiated accumulator width >= n_pad (W tile rows, zero filled beyond N)
  size_t a_plane_bytes, w_plane_bytes, total_bytes, w_only_bytes, smem_bytes;
  bool ok;
};

TcPlan plan_tc(int64_t M, int64_t N, int64_t K, bool single = false) {
  TcPlan t{};
  const int BK = g_tc_bk == 64 ? 64 : 32;
  t.ok = (N >= 8 && N <= 256 && K >= 8 && M >= 1);
  t.kp = (K + 7) / 8 * 8;
  t.n_pad = (int)((N + 15) / 16 * 16);
  t.np = t.n_pad <= 64 ? 64 : t.n_pad <= 128 ? 128 : t.n_pad <= 208 ? 208 : 256;
  const size_t stage = (single ? 1 : 2) * ((size_t)BM * BK * 2 + (size_t)t.np * BK * 2);
  // 227 KB usable smem minus alignment slack, bias/score arrays, barriers and the epilogue staging buffers
  int stages = (int)((227 * 1024 - 1024 - 2048 - 128 - 2 * kStageOutBytes) / stage);
  t.stages = stages > 8 ? 8 : stages;
  if (t.stages < 2) t.ok = false;
  t.bk = BK;
  t.smem_bytes = (size_t)t.stages * stage + 1024 /*align slack*/ + 2 * t.stages * 8 + 2 * 256 * 4 + 2 * kStageOutBytes;
  t.a_plane_bytes = align_up((size_t)M * t.kp * 2, 256);
  t.w_plane_bytes = align_up((size_t)N * t.kp * 2, 256);
  t.total_bytes = 2 * t.a_plane_bytes + 2 * t.w_plane_bytes;
  t.w_only_bytes = 2 * t.w_plane_bytes;
  return t;
}


int split_launch(const float* A, int64_t lda, int64_t M, int64_t K, __nv_bfloat16* hi, __nv_bfloat16* lo,
                 int64_t ldo, cudaStream_t stream) {
  int va = (lda % 4 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
  int64_t work = M * ((K + 3) / 4);
  int grid = (int)std::min<int64_t>(ceil_div(work, 256), 32LL * sm_count());
  int vs = (ldo % 4 == 0) && ((reinterpret_cast<uintptr_t>(hi) & 7) == 0) &&
           ((reinterpret_cast<uintptr_t>(lo) & 7) == 0);
  split_bf16_kernel<<<grid, 256, 0, stream>>>(A, lda, M, K, hi, lo, ldo, va, vs);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

template <int NP, int CS, int BK, bool GROUPED = false>
int launch_tc_cs(const CUtensorMap& m_a_hi, const CUtensorMap& m_a_lo, const CUtensorMap& m_w_hi,
                 const CUtensorMap& m_w_lo, const CUtensorMap& m_c, const CUtensorMap& m_c_hi,
                 const CUtensorMap& m_c_lo, const TcPlan& t, const TcParams& p, cudaStream_t stream) {
  const int ngroups = (p.num_tiles + CS - 1) / CS;
  const int nclusters = std::max(1, std::min(ngroups, sm_count() / CS));
  return launch_cluster<linear_tc_kernel<NP, CS, BK, GROUPED>>("gr_linear_tc", kLaunchRegs, CS, nclusters * CS, kThreads,
                                                               t.smem_bytes, stream, m_a_hi, m_a_lo, m_w_hi, m_w_lo,
                                                               m_c, m_c_hi, m_c_lo, p);
}

template <int NP>
int launch_tc_np(const CUtensorMap* const (&m)[7], int cs, const TcPlan& t, const TcParams& p, cudaStream_t stream) {
  if (p.kg_T) {
    if (cs == 2) return launch_tc_cs<NP, 2, 32, true>(*m[0], *m[1], *m[2], *m[3], *m[4], *m[5], *m[6], t, p, stream);
    return launch_tc_cs<NP, 1, 32, true>(*m[0], *m[1], *m[2], *m[3], *m[4], *m[5], *m[6], t, p, stream);
  }
  if (t.bk == 64) {
    if (cs == 2) return launch_tc_cs<NP, 2, 64>(*m[0], *m[1], *m[2], *m[3], *m[4], *m[5], *m[6], t, p, stream);
    return launch_tc_cs<NP, 1, 64>(*m[0], *m[1], *m[2], *m[3], *m[4], *m[5], *m[6], t, p, stream);
  }
  if (cs == 2) return launch_tc_cs<NP, 2, 32>(*m[0], *m[1], *m[2], *m[3], *m[4], *m[5], *m[6], t, p, stream);
  return launch_tc_cs<NP, 1, 32>(*m[0], *m[1], *m[2], *m[3], *m[4], *m[5], *m[6], t, p, stream);
}

int launch_tc(const __nv_bfloat16* a_hi, const __nv_bfloat16* a_lo, int64_t lda16,
              const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo, int64_t ldw16, const TcPlan& t,
              TcParams p, cudaStream_t stream) {
  p.n_pad = t.n_pad; p.stages = t.stages;
  p.num_tiles = (int)ceil_div(p.M, BM);
  // cluster multicast of W needs 8-row-aligned W slices and at least two tiles
  int cs = (g_tc_cluster >= 2 && (t.np / 2) % 8 == 0 && p.num_tiles >= 2) ? 2 : 1;
  CUtensorMap m_a_hi, m_a_lo, m_w_hi, m_w_lo;
  const int64_t w_cols = p.kg_T ? ldw16 : p.K;           // grouped order: dense planes of kg_nkb * 32 columns
  // K-order layout: the A map reaches the end of the neighbour region (past K), or the last tail box would be zero filled
  const int64_t a_cols = p.kg_nb0 ? p.kg_nb0 + (int64_t)(p.kg_T - 1) * p.kg_pitch : p.K;
  if (!make_tmap(&m_a_hi, a_hi, p.M, a_cols, lda16, BM, t.bk) || !make_tmap(&m_a_lo, a_lo, p.M, a_cols, lda16, BM, t.bk) ||
      !make_tmap(&m_w_hi, w_hi, p.N, w_cols, ldw16, t.np / cs, t.bk) ||
      !make_tmap(&m_w_lo, w_lo, p.N, w_cols, ldw16, t.np / cs, t.bk)) {
    set_error("gr_linear_tc: cuTensorMapEncodeTiled failed (pointers must be 16-byte aligned, row strides "
              "multiples of 8 elements)");
    return GR_ERR_CUDA;
  }
  // the planes also receive the (exactly zero) columns N .. round16(N): whole 32-byte sectors per row
  p.n16 = (int)std::min<int64_t>((p.N + 15) / 16 * 16, p.ldc16);
  // output tensor maps for the staged TMA-store epilogue (need 16-byte aligned bases and row pitches)
  CUtensorMap m_c, m_c_hi, m_c_lo;
  memset(&m_c, 0, sizeof(m_c)); memset(&m_c_hi, 0, sizeof(m_c_hi)); memset(&m_c_lo, 0, sizeof(m_c_lo));
  bool ok = g_tc_tma_store != 0;
  // with N % 4 != 0 the TMA-store epilogue wrote past column N of an fp32 column view whose pitch is 16-byte aligned
  // (observed on an H100: N = 50 wrote columns 50 and 51, the rest of the last 16-byte unit), so such an output takes
  // the direct stores
  if (ok && p.C) ok = p.N % 4 == 0 && make_out_tmap(&m_c, p.C, p.M, p.N, p.ldc, 4);
  if (ok && p.c_hi) ok = make_out_tmap(&m_c_hi, p.c_hi, p.M, p.n16, p.ldc16, 2) &&
                         make_out_tmap(&m_c_lo, p.c_lo, p.M, p.n16, p.ldc16, 2);
  p.tma_store = ok ? 1 : 0;
  const CUtensorMap* m[7] = {&m_a_hi, &m_a_lo, &m_w_hi, &m_w_lo, &m_c, &m_c_hi, &m_c_lo};
  switch (t.np) {
    case 64: return launch_tc_np<64>(m, cs, t, p, stream);
    case 128: return launch_tc_np<128>(m, cs, t, p, stream);
    case 208: return launch_tc_np<208>(m, cs, t, p, stream);
    default: return launch_tc_np<256>(m, cs, t, p, stream);
  }
}

}  // namespace

bool linear_tc_supported(int64_t M, int64_t N, int64_t K) {
  return plan_tc(M, N, K).ok && get_encode_fn() != nullptr;
}

}  // namespace gr

extern "C" size_t gr_linear_tc_workspace_bytes(int64_t M, int64_t N, int64_t K) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  return gr::plan_tc(M, N, K).total_bytes;
}

extern "C" size_t gr_linear_tc_planes_workspace_bytes(int64_t N, int64_t K) {
  if (N <= 0 || K <= 0) return 0;
  return gr::plan_tc(1, N, K).w_only_bytes;
}

extern "C" int gr_split_bf16(const float* A, int64_t lda, int64_t M, int64_t K, void* hi, void* lo,
                             int64_t ld_out, void* stream_) {
  using namespace gr;
  GR_CHECK_ARG(A && hi && lo, "null pointer");
  GR_CHECK_ARG(M > 0 && K > 0 && lda >= K && ld_out >= K && ld_out % 8 == 0, "bad shape / ld_out % 8 != 0");
  return split_launch(A, lda, M, K, reinterpret_cast<__nv_bfloat16*>(hi), reinterpret_cast<__nv_bfloat16*>(lo),
                      ld_out, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_linear_tc(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias,
                            float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, uint32_t flags,
                            void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(A && W && C && workspace, "null pointer");
  GR_CHECK_ARG(M > 0 && N > 0 && K > 0, "M, N, K must be positive");
  GR_CHECK_ARG(lda >= K && ldw >= K && ldc >= N, "leading dimension smaller than row length");
  GR_CHECK_ARG(M < (int64_t)0x7fffffff - BM, "M exceeds int32 range");
  TcPlan t = plan_tc(M, N, K);
  if (!t.ok) {
    set_error("gr_linear_tc: unsupported shape M=%lld N=%lld K=%lld (need 8 <= N <= 256, K >= 8)",
              (long long)M, (long long)N, (long long)K);
    return GR_ERR_UNSUPPORTED;
  }
  if (int rc = check_workspace(__func__, workspace, workspace_bytes, t.total_bytes)) return rc;
  if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) {
    set_error("gr_linear_tc: workspace must be 256-byte aligned");
    return GR_ERR_INVALID_ARG;
  }
  char* ws = reinterpret_cast<char*>(workspace);
  __nv_bfloat16* a_hi = reinterpret_cast<__nv_bfloat16*>(ws);
  __nv_bfloat16* a_lo = reinterpret_cast<__nv_bfloat16*>(ws + t.a_plane_bytes);
  __nv_bfloat16* w_hi = reinterpret_cast<__nv_bfloat16*>(ws + 2 * t.a_plane_bytes);
  __nv_bfloat16* w_lo = reinterpret_cast<__nv_bfloat16*>(ws + 2 * t.a_plane_bytes + t.w_plane_bytes);
  int rc = split_launch(A, lda, M, K, a_hi, a_lo, t.kp, stream);
  if (rc != GR_OK) return rc;
  rc = split_launch(W, ldw, N, K, w_hi, w_lo, t.kp, stream);
  if (rc != GR_OK) return rc;
  TcParams p{};
  p.bias = bias; p.C = C; p.ldc = ldc;
  p.M = (int)M; p.N = (int)N; p.K = (int)K; p.flags = flags;
  return launch_tc(a_hi, a_lo, t.kp, w_hi, w_lo, t.kp, t, p, stream);
}

namespace gr {
namespace {

// gr_linear_tc_planes and gr_linear_tc_planes_rows; errors name the entry point `fn`
int linear_tc_planes_entry(const char* fn, const void* A_hi, const void* A_lo, int64_t lda16, const float* W,
                           int64_t ldw, const float* bias, float* C, int64_t ldc, const float* c_rows, void* C_hi,
                           void* C_lo, int64_t ldc16, const float* w_score, float* dots, int64_t M, int64_t N,
                           int64_t K, int64_t k_seg, int64_t k_seg_pitch, uint32_t flags, void* workspace,
                           size_t workspace_bytes, cudaStream_t stream) {
  GR_CHECK_ARG_AS(fn, A_hi && (A_lo || (flags & GR_LINEAR_BF16_SINGLE)) && W && workspace, "null pointer");
  GR_CHECK_ARG_AS(fn, C || C_hi, "no output requested");
  GR_CHECK_ARG_AS(fn, !c_rows || C, "c_rows selects rows of C and needs C");
  GR_CHECK_ARG_AS(fn, M > 0 && N > 0 && K > 0, "M, N, K must be positive");
  const bool grouped = (flags & GR_LINEAR_K_GROUPED) != 0;
  const bool korder = (flags & GR_LINEAR_K_ORDER_PLANES) != 0;
  GR_CHECK_ARG_AS(fn, !korder || grouped, "GR_LINEAR_K_ORDER_PLANES modifies GR_LINEAR_K_GROUPED and needs it");
  if (grouped) {
    GR_CHECK_ARG_AS(fn, k_seg > 0 && k_seg_pitch >= k_seg && k_seg_pitch % 16 == 0,
                    "GR_LINEAR_K_GROUPED needs segmented K: k_seg > 0 and k_seg_pitch >= k_seg, a multiple of 16");
    GR_CHECK_ARG_AS(fn, K % k_seg_pitch == 0 && (K / k_seg_pitch) % 2 == 1,
                    "GR_LINEAR_K_GROUPED needs an odd number of segments (2 I + 1)");
    GR_CHECK_ARG_AS(fn, g_tc_bk != 64, "GR_LINEAR_K_GROUPED needs 32-column k-blocks (tc_bk = 32)");
    GR_CHECK_ARG_AS(fn, !(flags & GR_LINEAR_BF16_SINGLE),
                    "GR_LINEAR_K_GROUPED does not combine with GR_LINEAR_BF16_SINGLE");
  }
  const bool segmented = grouped || (k_seg > 0 && k_seg_pitch > k_seg);
  GR_CHECK_ARG_AS(fn, lda16 >= K && lda16 % 8 == 0, "lda16 must be >= K and a multiple of 8");
  GR_CHECK_ARG_AS(fn, !segmented || K % k_seg_pitch == 0, "K must be a multiple of k_seg_pitch");
  GR_CHECK_ARG_AS(fn, ldw >= (segmented ? K / k_seg_pitch * k_seg : K), "ldw smaller than the weight row length");
  GR_CHECK_ARG_AS(fn, !C || ldc >= N, "ldc smaller than N");
  GR_CHECK_ARG_AS(fn, !C_hi || (C_lo && ldc16 >= N), "C_lo missing or ldc16 smaller than N");
  GR_CHECK_ARG_AS(fn, !dots || w_score, "dots requested without w_score");
  GR_CHECK_ARG_AS(fn, M < (int64_t)0x7fffffff - BM, "M exceeds int32 range");
  TcPlan t = plan_tc(M, N, K, (flags & GR_LINEAR_BF16_SINGLE) != 0);
  if (!t.ok) {
    set_error("%s: unsupported shape M=%lld N=%lld K=%lld", fn, (long long)M, (long long)N, (long long)K);
    return GR_ERR_UNSUPPORTED;
  }
  // grouped order: the W planes gr_fused_layer keeps (same layout, same size: one workspace serves both); over K-order
  // planes the packed form of them, no larger
  const int num_ins = grouped ? (int)(K / k_seg_pitch / 2) : 0;
  const GroupedK gk = grouped ? plan_grouped_k(k_seg_pitch, num_ins, N, korder) : GroupedK{};
  const int64_t nb0 = (k_seg_pitch + 31) / 32 * 32;      // K-order layout: first column of the neighbour region
  GR_CHECK_ARG_AS(fn, !korder || lda16 >= nb0 + 2 * num_ins * k_seg_pitch,
                  "GR_LINEAR_K_ORDER_PLANES: lda16 must cover the neighbour region (round32(k_seg_pitch) + "
                  "(K - k_seg_pitch) columns)");
  const size_t w_plane_bytes = grouped ? gk.w_plane_bytes : t.w_plane_bytes;
  if (workspace_bytes < 2 * w_plane_bytes || (reinterpret_cast<uintptr_t>(workspace) & 255) != 0) {
    set_error("%s: workspace too small or not 256-byte aligned", fn);
    return GR_ERR_WORKSPACE;
  }
  char* ws = reinterpret_cast<char*>(workspace);
  __nv_bfloat16* w_hi = reinterpret_cast<__nv_bfloat16*>(ws);
  __nv_bfloat16* w_lo = reinterpret_cast<__nv_bfloat16*>(ws + w_plane_bytes);
  int rc = GR_OK;
  if (flags & GR_LINEAR_W_PRESPLIT) {
    // the caller kept the workspace of an earlier call with the same W / N / K / k_seg / k_seg_pitch
  } else if (grouped) {
    rc = grouped_w_split(W, ldw, N, (int)k_seg, num_ins, gk, w_hi, w_lo, stream);
  } else if (segmented) {
    int64_t work = N * K;
    int grid = (int)std::min<int64_t>(ceil_div(work, 256), 32LL * sm_count());
    split_bf16_seg_kernel<<<grid, 256, 0, stream>>>(W, ldw, N, K, (int)k_seg, (int)k_seg_pitch, w_hi, w_lo, t.kp);
    GR_CHECK_LAUNCH();
  } else {
    rc = split_launch(W, ldw, N, K, w_hi, w_lo, t.kp, stream);
  }
  if (rc != GR_OK) return rc;
  TcParams p{};
  p.bias = bias; p.C = C; p.ldc = ldc; p.c_rows = c_rows;
  p.c_hi = reinterpret_cast<__nv_bfloat16*>(C_hi); p.c_lo = reinterpret_cast<__nv_bfloat16*>(C_lo);
  p.ldc16 = ldc16; p.w_score = w_score; p.dots = dots;
  p.M = (int)M; p.N = (int)N; p.K = (int)K; p.flags = flags;
  if (grouped) {
    p.kg_T = 2 * num_ins + 1; p.kg_pitch = (int)k_seg_pitch; p.kg_nkb = gk.nkb;
    const bool tail = gk.ksteps_last == 1;
    if (!korder) {
      p.kg_G = gk.G;
      p.kg_one0 = tail ? (gk.G - 1) * p.kg_T : gk.nkb; p.kg_one1 = gk.nkb;
    } else {
      p.kg_G = tail ? gk.G - 1 : gk.G; p.kg_nb0 = (int)nb0;
      p.kg_one0 = tail ? p.kg_G * p.kg_T : gk.nkb; p.kg_one1 = tail ? p.kg_one0 + 1 : gk.nkb;
    }
  }
  return launch_tc(reinterpret_cast<const __nv_bfloat16*>(A_hi),
                   reinterpret_cast<const __nv_bfloat16*>(A_lo ? A_lo : A_hi), lda16, w_hi, w_lo,
                   grouped ? gk.kp : t.kp, t, p, stream);
}

}  // namespace
}  // namespace gr

extern "C" int gr_linear_tc_planes(const void* A_hi, const void* A_lo, int64_t lda16, const float* W,
                                   int64_t ldw, const float* bias, float* C, int64_t ldc, void* C_hi,
                                   void* C_lo, int64_t ldc16, const float* w_score, float* dots, int64_t M,
                                   int64_t N, int64_t K, int64_t k_seg, int64_t k_seg_pitch, uint32_t flags,
                                   void* workspace, size_t workspace_bytes, void* stream) {
  return gr::linear_tc_planes_entry(__func__, A_hi, A_lo, lda16, W, ldw, bias, C, ldc, nullptr, C_hi, C_lo, ldc16,
                                    w_score, dots, M, N, K, k_seg, k_seg_pitch, flags, workspace, workspace_bytes,
                                    reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int gr_linear_tc_planes_rows(const void* A_hi, const void* A_lo, int64_t lda16, const float* W,
                                        int64_t ldw, const float* bias, float* C, int64_t ldc, void* C_hi,
                                        void* C_lo, int64_t ldc16, const float* w_score, float* dots, int64_t M,
                                        int64_t N, int64_t K, int64_t k_seg, int64_t k_seg_pitch, uint32_t flags,
                                        void* workspace, size_t workspace_bytes, const float* c_rows,
                                        void* stream) {
  return gr::linear_tc_planes_entry(__func__, A_hi, A_lo, lda16, W, ldw, bias, C, ldc, c_rows, C_hi, C_lo, ldc16,
                                    w_score, dots, M, N, K, k_seg, k_seg_pitch, flags, workspace, workspace_bytes,
                                    reinterpret_cast<cudaStream_t>(stream));
}
