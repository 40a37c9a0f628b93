// GraftNet on the GPU: graft-tuple staging, query-conditioned fact attention and the per-layer PageRank aggregation.
//
// Reference: GraftLayer (gnn/modules/kg_reasoning/graft_gnn.py) on the batch of GraftSingleDataLoader.get_batch
// (gnn/dataset_load_graft.py:70-149), with the sparse operators of BaseGNNLayer.build_adj_facts (base_gnn.py:56-75).
//   gr_graft_stage      build_adj_facts: pairs the head list (b, f, head) and the tail list (b, tail, f) by fact slot
//                       and orders the facts by (b, f), so gr_csr_build's stable CSRs list every row in slot order --
//                       the order torch's CPU sparse bmm sums a row in.
//   gr_graft_attention  compute_attention, graft_gnn.py:64-87: W per slot, W~ = exp(W - max_f W), E = max(sum, 1e-10).
//   gr_graft_aggregate  reason_layer, graft_gnn.py:89-107 (the fact-side half): per tail row, in slot order,
//                       s_f = W~_f * (d[head] / E[head]), v_f = relu(self_tab[r_f] + head_tab[head]) * s_f, and the
//                       sums sum_f v_f, indeg, d' = lambda * sum_f s_f + (1 - lambda) * d.  No atomics: every output
//                       row is owned by one warp, so results are bit-reproducible and do not depend on the loader's
//                       permutation of the fact lists.
// Training (model(batch, training=True)): gr_graft_aggregate_train / gr_graft_aggregate_backward (the fact messages
// with kb_tail_linear moved after the per-node sum, in-kernel dropout keyed by fact slot), gr_graft_attention_backward
// and gr_graft_dropout_mask.
#include <cub/device/device_scan.cuh>
#include <cuda_bf16.h>

#include <algorithm>

#include "common.cuh"

namespace gr {
namespace {

constexpr float kVeryNeg = -100000000000.0f;   // VERY_NEG_NUMBER, graft_gnn.py:11
constexpr float kVerySmall = 1e-10f;           // VERY_SMALL_NUMBER, graft_gnn.py:10

// status bits
constexpr int kBadId = 1;         // batch / slot / node id out of range
constexpr int kBadRel = 2;        // relation id out of range
constexpr int kDupSlot = 4;       // a (b, f) slot listed twice in one list
constexpr int kUnpaired = 8;      // a slot with a head but no tail or the reverse

// ---- staging ------------------------------------------------------------------------------------------------------

// One of the two graft lists -> dense per-slot node table (global node id, -1 = absent).  ``live`` (optional device
// int32): only the first min(F, *live) entries are read -- F is then the capacity of a fixed-shape buffer whose tail
// holds whatever an earlier batch left there.
__global__ void graft_scatter_kernel(const int64_t* __restrict__ bid, const int64_t* __restrict__ fid,
                                     const int64_t* __restrict__ nid, int64_t F, const int32_t* __restrict__ live,
                                     int B, int N, int64_t max_fact, int32_t* __restrict__ node_of,
                                     int32_t* __restrict__ status) {
  if (live) F = min(F, (int64_t)max(*live, 0));
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < F; i += stride) {
    const int64_t b = bid[i], f = fid[i], e = nid[i];
    if (b < 0 || b >= B || f < 0 || f >= max_fact || e < 0 || e >= N) {
      atomicOr(status, kBadId);
      continue;
    }
    const int32_t old = atomicExch(&node_of[b * max_fact + f], (int32_t)(b * N + e));
    if (old != -1) atomicOr(status, kDupSlot);
  }
}

__global__ void graft_flags_kernel(const int32_t* __restrict__ head_of, const int32_t* __restrict__ tail_of,
                                   int64_t S, int32_t* __restrict__ flag, int32_t* __restrict__ status) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += stride) {
    const bool h = head_of[s] >= 0, t = tail_of[s] >= 0;
    if (h != t) atomicOr(status, kUnpaired);
    flag[s] = (h && t) ? 1 : 0;
  }
}

__global__ void graft_compact_kernel(const int32_t* __restrict__ head_of, const int32_t* __restrict__ tail_of,
                                     const int32_t* __restrict__ flag, const int32_t* __restrict__ pos,
                                     const int64_t* __restrict__ kb_fact_rel, int64_t S, int64_t R1, int64_t cap,
                                     int32_t* __restrict__ heads, int32_t* __restrict__ rels,
                                     int32_t* __restrict__ tails, int32_t* __restrict__ slot_of,
                                     int32_t* __restrict__ nfacts, int32_t* __restrict__ status) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += stride) {
    if (s == S - 1) *nfacts = (int32_t)min((int64_t)pos[s] + flag[s], cap);
    if (!flag[s]) continue;
    const int64_t p = pos[s];
    if (p >= cap) continue;
    int64_t r = kb_fact_rel[s];
    if (r < 0 || r >= R1) {
      atomicOr(status, kBadRel);
      r = 0;
    }
    heads[p] = head_of[s];
    tails[p] = tail_of[s];
    rels[p] = (int32_t)r;
    slot_of[p] = (int32_t)s;
  }
}

struct StageWs {
  size_t dense_bytes, scan_bytes, total;
};

StageWs stage_ws(int64_t S) {
  StageWs w{};
  w.dense_bytes = align_up((size_t)(S > 0 ? S : 1) * sizeof(int32_t), 256);
  size_t tmp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(S > 0 ? S : 1));
  w.scan_bytes = align_up(tmp, 256);
  w.total = 4 * w.dense_bytes + w.scan_bytes;
  return w;
}

// ---- fact attention -----------------------------------------------------------------------------------------------

template <int NC>
__device__ __forceinline__ float warp_dot(const float (&x)[NC], const float* __restrict__ row, int D) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const int c = lane + 32 * k;
    if (c < D) s = fmaf(x[k], __ldg(row + c), s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// One warp per fact slot (pads and dropped facts included: compute_attention runs over every slot, :71-81).
// sim_q = <qh[b,q], rel[r]> / div + (1 - mask_q) * VERY_NEG;  a = softmax_q(sim);  W = <sum_q a_q qh[b,q], rel[r]> / div.
template <int NC>
__global__ void __launch_bounds__(256) graft_w_kernel(const float* __restrict__ qh, const float* __restrict__ qmask,
                                                      int Q, const float* __restrict__ rel, int64_t ldr, int64_t R1,
                                                      const int64_t* __restrict__ kb_fact_rel, int64_t S,
                                                      int64_t max_fact, int D, float div, float* __restrict__ W,
                                                      int32_t* __restrict__ status) {
  const int lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (s >= S) return;
  const int64_t b = s / max_fact;
  int64_t r = kb_fact_rel[s];
  if (r < 0 || r >= R1) {
    if (lane == 0) atomicOr(status, kBadRel);
    r = 0;
  }
  float rv[NC];
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const int c = lane + 32 * k;
    rv[k] = c < D ? __ldg(rel + r * ldr + c) : 0.f;
  }
  const float* qb = qh + b * (int64_t)Q * D;
  const float* mb = qmask + b * (int64_t)Q;
  float mx = -INFINITY;
  for (int q = 0; q < Q; ++q) {
    const float sim = __fadd_rn(__fdiv_rn(warp_dot<NC>(rv, qb + (int64_t)q * D, D), div),
                                __fmul_rn(1.0f - __ldg(mb + q), kVeryNeg));
    mx = fmaxf(mx, sim);
  }
  float att[NC];
#pragma unroll
  for (int k = 0; k < NC; ++k) att[k] = 0.f;
  float den = 0.f;
  for (int q = 0; q < Q; ++q) {
    const float* row = qb + (int64_t)q * D;
    const float sim = __fadd_rn(__fdiv_rn(warp_dot<NC>(rv, row, D), div),
                                __fmul_rn(1.0f - __ldg(mb + q), kVeryNeg));
    const float e = expf(sim - mx);
    den += e;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int c = lane + 32 * k;
      if (c < D) att[k] = fmaf(e, __ldg(row + c), att[k]);
    }
  }
  const float inv = 1.0f / den;
#pragma unroll
  for (int k = 0; k < NC; ++k) att[k] *= inv;
  float w = 0.f;
#pragma unroll
  for (int k = 0; k < NC; ++k) w = fmaf(att[k], rv[k], w);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
  if (lane == 0) W[s] = __fdiv_rn(w, div);
}

// One block per question: W~[b, f] = exp(W[b, f] - max_f W[b, f]) over every slot (graft_gnn.py:82-83).
__global__ void __launch_bounds__(256) graft_wtilde_kernel(const float* __restrict__ W, int64_t max_fact,
                                                           float* __restrict__ Wt) {
  __shared__ float sm[32];
  const float* w = W + blockIdx.x * max_fact;
  float m = -INFINITY;
  for (int64_t f = threadIdx.x; f < max_fact; f += blockDim.x) m = fmaxf(m, w[f]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    float x = threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : -INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
    if (threadIdx.x == 0) sm[0] = x;
  }
  __syncthreads();
  m = sm[0];
  for (int64_t f = threadIdx.x; f < max_fact; f += blockDim.x) Wt[blockIdx.x * max_fact + f] = expf(w[f] - m);
}

// E[n] = max(sum_{graft f: head_f = n} W~_f, 1e-10), summed in slot order over the head CSR (graft_gnn.py:84-85).
__global__ void graft_e_kernel(const int32_t* __restrict__ rowptr_h, const int32_t* __restrict__ fact_h,
                               const int32_t* __restrict__ slot_of, const float* __restrict__ Wt, int64_t Nt,
                               float* __restrict__ E) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= Nt) return;
  float s = 0.f;
  for (int e = rowptr_h[n]; e < rowptr_h[n + 1]; ++e) s = __fadd_rn(s, Wt[slot_of[fact_h[e]]]);
  E[n] = fmaxf(s, kVerySmall);
}

// ---- layer aggregation --------------------------------------------------------------------------------------------

__device__ __forceinline__ void store_split(__nv_bfloat16* hi, __nv_bfloat16* lo, int64_t i, float y) {
  const __nv_bfloat16 h = __float2bfloat16_rn(y);
  hi[i] = h;
  lo[i] = __float2bfloat16_rn(y - __bfloat162float(h));
}

struct AggArgs {
  const int32_t *rowptr, *src, *rel, *fact, *slot_of;
  const float *Wt, *E, *prior, *self_tab, *head_tab, *q2e;
  int64_t ld_self, ld_head;
  float lam, one_minus_lam;
  float* sum_out;
  int64_t ld_sum;
  __nv_bfloat16 *hi, *lo;
  int64_t ld_planes, col_sum, col_indeg, col_q2e;
  float *indeg_out, *prior_next;
  int64_t Nt;
  int N, D;
};

// One warp per destination (tail CSR) row; the lane owns columns lane + 32k.  Facts are visited in slot order.
template <int NC>
__global__ void __launch_bounds__(256) graft_aggregate_kernel(const AggArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t n = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.Nt) return;
  const int D = a.D;
  float acc[NC];
#pragma unroll
  for (int k = 0; k < NC; ++k) acc[k] = 0.f;
  float dsum = 0.f;
  const int beg = a.rowptr[n], end = a.rowptr[n + 1];
  for (int e = beg; e < end; ++e) {
    const int h = __ldg(a.src + e);
    const int r = __ldg(a.rel + e);
    const int sl = __ldg(a.slot_of + __ldg(a.fact + e));
    // e2f_softmax_normalized = W~ * (curr_dist / E)[head]   (graft_gnn.py:97)
    const float s = __fmul_rn(__ldg(a.Wt + sl), __fdiv_rn(__ldg(a.prior + h), __ldg(a.E + h)));
    dsum = __fadd_rn(dsum, s);
    if (s == 0.f) continue;        // relu(x) * 0 == 0 for finite x: the fact adds nothing
    const float* st = a.self_tab + (int64_t)r * a.ld_self;
    const float* ht = a.head_tab + (int64_t)h * a.ld_head;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int c = lane + 32 * k;
      if (c < D) {
        const float x = fmaxf(__fadd_rn(__ldg(st + c), __ldg(ht + c)), 0.f);
        acc[k] = __fadd_rn(acc[k], __fmul_rn(x, s));
      }
    }
  }
  const int64_t b = n / a.N;
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const int c = lane + 32 * k;
    if (c < D) {
      if (a.sum_out) a.sum_out[n * a.ld_sum + c] = acc[k];
      if (a.hi) {
        store_split(a.hi, a.lo, n * a.ld_planes + a.col_sum + c, acc[k]);
        if (a.q2e) store_split(a.hi, a.lo, n * a.ld_planes + a.col_q2e + c, __ldg(a.q2e + b * D + c));
      }
    }
  }
  if (lane == 0) {
    const float deg = (float)(end - beg);
    if (a.indeg_out) a.indeg_out[n] = deg;
    if (a.hi) store_split(a.hi, a.lo, n * a.ld_planes + a.col_indeg, deg);
    // next_curr_dist = lambda * next + (1 - lambda) * curr_dist   (graft_gnn.py:101-102)
    a.prior_next[n] = __fadd_rn(__fmul_rn(a.lam, dsum), __fmul_rn(a.one_minus_lam, __ldg(a.prior + n)));
  }
}

// ---- training: dropout, aggregation forward / backward, attention backward ----------------------------------------

// Philox4x32-10 (common.cuh) with counter = (slot lo, slot hi, column, 0).  Keyed by fact SLOT (b * max_fact + f), so
// the mask of a fact does not depend on where the loader's permutation put it in the graft lists.
__device__ __forceinline__ bool drop_keep(uint64_t seed, int64_t slot, int col, float p) {
  return philox_keep(philox4x32_10_x0(seed, (uint32_t)(uint64_t)slot, (uint32_t)((uint64_t)slot >> 32), (uint32_t)col, 0u),
                     p);
}

__global__ void graft_dropout_mask_kernel(const int64_t* __restrict__ seed, float p, int64_t S, int D,
                                          uint8_t* __restrict__ mask) {
  const uint64_t sd = p > 0.f ? (uint64_t)__ldg(seed) : 0;
  const int64_t total = S * D, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride)
    mask[i] = p > 0.f ? (uint8_t)drop_keep(sd, i / D, (int)(i % D), p) : (uint8_t)1;
}

struct TrainArgs {
  // forward: the tail CSR (src = head); backward: the head CSR (src = tail)
  const int32_t *rowptr, *src, *rel, *fact, *slot_of;
  const float *s, *self_tab;
  const void* head_tab;     // [B*N, D] fp32 or bf16 (the node-sized operands: head_tab, sum_out, grad, grad_head)
  int64_t ld_self, ld_head;
  const int64_t* seed;      // NULL: no dropout
  float p, scale;
  void* sum_out;            // forward
  int64_t ld_sum;
  const void* grad;         // backward: dL/dsum_out
  int64_t ld_grad;
  float *grad_s, *grad_self;
  void* grad_head;
  int64_t ld_gself, ld_ghead;
  int64_t Nt;
  int D;
};

// sum_out[n] = sum_{f -> n} drop_f(relu(self_tab[r_f] + head_tab[head_f])) * s_f, one warp per tail-CSR row, slot order.
template <int NC, typename T>
__global__ void __launch_bounds__(256) graft_aggregate_train_kernel(const TrainArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t n = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.Nt) return;
  const int D = a.D;
  const bool drop = a.seed != nullptr;
  const uint64_t seed = drop ? (uint64_t)__ldg(a.seed) : 0;
  float acc[NC];
#pragma unroll
  for (int k = 0; k < NC; ++k) acc[k] = 0.f;
  const int beg = a.rowptr[n], end = a.rowptr[n + 1];
  for (int e = beg; e < end; ++e) {
    const int f = __ldg(a.fact + e);
    const float s = __ldg(a.s + f);
    if (s == 0.f) continue;        // the fact adds nothing (its relu term is finite)
    const int h = __ldg(a.src + e), r = __ldg(a.rel + e);
    const int64_t sl = __ldg(a.slot_of + f);
    const float* st = a.self_tab + (int64_t)r * a.ld_self;
    const T* ht = static_cast<const T*>(a.head_tab) + (int64_t)h * a.ld_head;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int c = lane + 32 * k;
      if (c < D) {
        float v = __fmul_rn(fmaxf(__fadd_rn(__ldg(st + c), ldg_node(ht + c)), 0.f), s);
        if (drop) v = drop_keep(seed, sl, c, a.p) ? __fmul_rn(v, a.scale) : 0.f;
        acc[k] = __fadd_rn(acc[k], v);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const int c = lane + 32 * k;
    if (c < D) st_node(static_cast<T*>(a.sum_out) + n * a.ld_sum + c, acc[k]);
  }
}

// Backward of graft_aggregate_train_kernel, one warp per HEAD-CSR row n (the out-facts of n).  With
// g_f = G[tail_f] * mask_f / (1 - p) and a_f = self_tab[r_f] + head_tab[n]:
//   grad_s[f] += <g_f, relu(a_f)>                 every fact, s_f = 0 included (lane 0, the fact is owned)
//   grad_head[n] += sum_f g_f s_f [a_f > 0]       registers, one read-modify-write per row (the row is owned)
//   grad_self[r_f] += g_f s_f [a_f > 0]           fp32 atomics into the R1 relation rows
template <int NC, bool kSelfAtomics, typename T>
__global__ void __launch_bounds__(256) graft_aggregate_bwd_kernel(const TrainArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t n = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.Nt) return;
  const int beg = a.rowptr[n], end = a.rowptr[n + 1];
  if (beg == end) return;
  const int D = a.D;
  const bool drop = a.seed != nullptr;
  const uint64_t seed = drop ? (uint64_t)__ldg(a.seed) : 0;
  float ht[NC], gh[NC];
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const int c = lane + 32 * k;
    ht[k] = c < D ? ldg_node(static_cast<const T*>(a.head_tab) + n * a.ld_head + c) : 0.f;
    gh[k] = 0.f;
  }
  for (int e = beg; e < end; ++e) {
    const int t = __ldg(a.src + e), r = __ldg(a.rel + e), f = __ldg(a.fact + e);
    const int64_t sl = __ldg(a.slot_of + f);
    const float s = __ldg(a.s + f);
    const float* st = a.self_tab + (int64_t)r * a.ld_self;
    const T* gt = static_cast<const T*>(a.grad) + (int64_t)t * a.ld_grad;
    float* gs_row = a.grad_self + (int64_t)r * a.ld_gself;
    float gs = 0.f;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int c = lane + 32 * k;
      if (c < D) {
        const float x = __fadd_rn(__ldg(st + c), ht[k]);
        float g = ldg_node(gt + c);
        if (drop) g = drop_keep(seed, sl, c, a.p) ? __fmul_rn(g, a.scale) : 0.f;
        gs = fmaf(g, fmaxf(x, 0.f), gs);
        if (s != 0.f && x > 0.f) {          // strict: relu'(0) = 0, as torch
          const float v = __fmul_rn(g, s);
          gh[k] = __fadd_rn(gh[k], v);
          if (kSelfAtomics && v != 0.f) atomicAdd(gs_row + c, v);
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) gs += __shfl_xor_sync(0xffffffffu, gs, o);
    if (lane == 0) a.grad_s[f] += gs;
  }
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const int c = lane + 32 * k;
    if (c < D) {
      T* q = static_cast<T*>(a.grad_head) + n * a.ld_ghead + c;
      st_node(q, ld_node(q) + gh[k]);
    }
  }
}

constexpr int kSlotsPerBlock = 64;     // attention backward: 8 warps x 8 slots, all of one question

// Backward of graft_w_kernel.  With z_q = <qh_q, rv>/div, a = softmax_q(z + mask) and W = sum_q a_q z_q:
//   dW/dqh_q = c_q rv,   dW/drv = sum_q c_q qh_q,   c_q = a_q (1 + z_q - W) / div
// One warp per slot recomputes the softmax (same operations as the forward); grad_rel goes out through fp32 atomics
// by relation; grad_qh of the block's question is accumulated in shared memory (or, when Q*D does not fit, straight
// into global memory) and flushed once per block.  Slots with grad_W == 0 contribute nothing and are skipped.
template <int NC>
__global__ void __launch_bounds__(256, 2) graft_w_bwd_kernel(const float* __restrict__ qh,
                                                          const float* __restrict__ qmask, int Q,
                                                          const float* __restrict__ rel, int64_t ldr, int64_t R1,
                                                          const int64_t* __restrict__ kb_fact_rel, int64_t max_fact,
                                                          int D, float div, const float* __restrict__ gW,
                                                          float* __restrict__ grad_qh, float* __restrict__ grad_rel,
                                                          int64_t ld_grel, bool smem_acc) {
  extern __shared__ float sacc[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int64_t b = blockIdx.y;
  const int64_t f0 = (int64_t)blockIdx.x * kSlotsPerBlock, f1 = min(f0 + kSlotsPerBlock, max_fact);
  const int64_t QD = (int64_t)Q * D;
  if (smem_acc) {
    for (int64_t i = threadIdx.x; i < QD; i += blockDim.x) sacc[i] = 0.f;
    __syncthreads();
  }
  float* acc = smem_acc ? sacc : grad_qh + b * QD;
  const float* qb = qh + b * QD;
  const float* mb = qmask + b * (int64_t)Q;
  const float inv_div = __frcp_rn(div);
  for (int64_t f = f0 + warp; f < f1; f += nwarps) {
    const int64_t s = b * max_fact + f;
    const float g = __ldg(gW + s);
    if (g == 0.f) continue;
    int64_t r = kb_fact_rel[s];
    if (r < 0 || r >= R1) r = 0;           // as the forward (which reports it)
    float rv[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int c = lane + 32 * k;
      rv[k] = c < D ? __ldg(rel + r * ldr + c) : 0.f;
    }
    float mx = -INFINITY;
    for (int q = 0; q < Q; ++q) {
      const float sim = __fadd_rn(__fdiv_rn(warp_dot<NC>(rv, qb + (int64_t)q * D, D), div),
                                  __fmul_rn(1.0f - __ldg(mb + q), kVeryNeg));
      mx = fmaxf(mx, sim);
    }
    float den = 0.f, wz = 0.f;
    for (int q = 0; q < Q; ++q) {
      const float z = __fdiv_rn(warp_dot<NC>(rv, qb + (int64_t)q * D, D), div);
      const float e = expf(__fadd_rn(z, __fmul_rn(1.0f - __ldg(mb + q), kVeryNeg)) - mx);
      den += e;
      wz = fmaf(e, z, wz);
    }
    const float inv = __frcp_rn(den), Wr = wz * inv, ginv = g * inv * inv_div;
    float gr[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) gr[k] = 0.f;
    for (int q = 0; q < Q; ++q) {
      const float* row = qb + (int64_t)q * D;
      const float z = __fdiv_rn(warp_dot<NC>(rv, row, D), div);
      const float e = expf(__fadd_rn(z, __fmul_rn(1.0f - __ldg(mb + q), kVeryNeg)) - mx);
      const float cq = e * ginv * (1.0f + z - Wr);
      if (cq == 0.f) continue;             // warp-uniform: masked tokens (a_q = 0)
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int c = lane + 32 * k;
        if (c < D) {
          atomicAdd(acc + (int64_t)q * D + c, cq * rv[k]);
          gr[k] = fmaf(cq, __ldg(row + c), gr[k]);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int c = lane + 32 * k;
      if (c < D && gr[k] != 0.f) atomicAdd(grad_rel + r * ld_grel + c, gr[k]);
    }
  }
  if (smem_acc) {
    __syncthreads();
    for (int64_t i = threadIdx.x; i < QD; i += blockDim.x) {
      const float v = sacc[i];
      if (v != 0.f) atomicAdd(grad_qh + b * QD + i, v);
    }
  }
}

// ---- deterministic backward (torch.use_deterministic_algorithms) --------------------------------------------------
// grad_s and grad_head of graft_aggregate_bwd_kernel are already owned sums; only grad_self and the attention
// gradients need a fixed order.  Both use the fixed-window segmented sums of common.cuh.

constexpr int kFactWin = 64;   // relation-index entries per window (grad_self, grad_rel)

// grad_self[r] += sum over the staged facts of relation r, in slot order, of  g_f s_f [a_f > 0]  (as the atomics of
// graft_aggregate_bwd_kernel; g_f = G[tail_f] * mask_f / (1 - p), a_f = self_tab[r] + head_tab[head_f]).
// Entry i of the relation index -> staged fact f = rix_fact[i].
template <int NC, typename T>
__global__ void __launch_bounds__(256) graft_self_det_kernel(const TrainArgs a, const int32_t* __restrict__ rix_ptr,
                                                             const int32_t* __restrict__ rix_fact,
                                                             const int32_t* __restrict__ heads,
                                                             const int32_t* __restrict__ rels,
                                                             const int32_t* __restrict__ tails,
                                                             float* __restrict__ part, int64_t R1) {
  const int lane = threadIdx.x & 31;
  const int64_t win = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t L = rix_ptr[R1];
  const int64_t lo = win * kFactWin, hi = min(L, lo + kFactWin);
  if (lo >= L) return;
  const int D = a.D;
  const bool drop = a.seed != nullptr;
  const uint64_t seed = drop ? (uint64_t)__ldg(a.seed) : 0;
  auto seg_of = [&](int64_t i) { return (int64_t)rels[rix_fact[i]]; };
  float st[NC], acc[NC];
  int64_t cur = -1;
  bool first = true;
  auto flush = [&]() {
    const int slot = segwin_slot(lo, hi, L, cur, first, seg_of);
    segwin_store<NC>(acc, slot, part + (win * 2 + (slot > 0)) * D, a.grad_self + cur * a.ld_gself, D);
    first = false;
  };
  for (int64_t i = lo; i < hi; ++i) {
    const int f = rix_fact[i];
    const int64_t r = rels[f];
    if (r != cur) {
      if (cur >= 0) flush();
      cur = r;
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int c = lane + 32 * k;
        st[k] = c < D ? __ldg(a.self_tab + r * a.ld_self + c) : 0.f;
        acc[k] = 0.f;
      }
    }
    const float s = __ldg(a.s + f);
    if (s == 0.f) continue;
    const int64_t h = heads[f], t = tails[f], sl = __ldg(a.slot_of + f);
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int c = lane + 32 * k;
      if (c < D && __fadd_rn(st[k], ldg_node(static_cast<const T*>(a.head_tab) + h * a.ld_head + c)) > 0.f) {
        float g = ldg_node(static_cast<const T*>(a.grad) + t * a.ld_grad + c);
        if (drop) g = drop_keep(seed, sl, c, a.p) ? __fmul_rn(g, a.scale) : 0.f;
        acc[k] = __fadd_rn(acc[k], __fmul_rn(g, s));
      }
    }
  }
  flush();
}

// relation of slot s as the forward reads it (out-of-range ids are reported by the forward and read as row 0)
__device__ __forceinline__ int64_t slot_rel(const int64_t* kb_fact_rel, int64_t s, int64_t R1) {
  const int64_t r = kb_fact_rel[s];
  return (r < 0 || r >= R1) ? 0 : r;
}

// c[s, q] = grad_W[s] a_{s,q} (1 + z_{s,q} - W_s) / div for every slot (0 where grad_W == 0 and for masked tokens),
// one warp per slot, the operations of graft_w_bwd_kernel.
template <int NC>
__global__ void __launch_bounds__(256) graft_w_coef_kernel(const float* __restrict__ qh,
                                                           const float* __restrict__ qmask, int Q,
                                                           const float* __restrict__ rel, int64_t ldr, int64_t R1,
                                                           const int64_t* __restrict__ kb_fact_rel, int64_t S,
                                                           int64_t max_fact, int D, float div,
                                                           const float* __restrict__ gW, float* __restrict__ coef) {
  const int lane = threadIdx.x & 31;
  const int64_t s = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (s >= S) return;
  float* cs = coef + s * Q;
  const float g = __ldg(gW + s);
  if (g == 0.f) {
    for (int q = lane; q < Q; q += 32) cs[q] = 0.f;
    return;
  }
  const int64_t b = s / max_fact, r = slot_rel(kb_fact_rel, s, R1);
  const float* qb = qh + b * (int64_t)Q * D;
  const float* mb = qmask + b * (int64_t)Q;
  float rv[NC];
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const int c = lane + 32 * k;
    rv[k] = c < D ? __ldg(rel + r * ldr + c) : 0.f;
  }
  float mx = -INFINITY;
#pragma unroll 1
  for (int q = 0; q < Q; ++q) {
    const float sim = __fadd_rn(__fdiv_rn(warp_dot<NC>(rv, qb + (int64_t)q * D, D), div),
                                __fmul_rn(1.0f - __ldg(mb + q), kVeryNeg));
    mx = fmaxf(mx, sim);
  }
  float den = 0.f, wz = 0.f;
#pragma unroll 1
  for (int q = 0; q < Q; ++q) {
    const float z = __fdiv_rn(warp_dot<NC>(rv, qb + (int64_t)q * D, D), div);
    const float e = expf(__fadd_rn(z, __fmul_rn(1.0f - __ldg(mb + q), kVeryNeg)) - mx);
    den += e;
    wz = fmaf(e, z, wz);
  }
  const float inv = __frcp_rn(den), Wr = wz * inv, ginv = g * inv * __frcp_rn(div);
#pragma unroll 1
  for (int q = 0; q < Q; ++q) {
    const float z = __fdiv_rn(warp_dot<NC>(rv, qb + (int64_t)q * D, D), div);
    const float e = expf(__fadd_rn(z, __fmul_rn(1.0f - __ldg(mb + q), kVeryNeg)) - mx);
    if (lane == 0) cs[q] = e * ginv * (1.0f + z - Wr);
  }
}

// grad_qh[b, q, c] += sum over the question's slots f, in slot order, of c[f, q] rel[r_f, c] (one thread per element)
__global__ void graft_qh_det_kernel(const float* __restrict__ coef, int Q, const float* __restrict__ rel,
                                    int64_t ldr, int64_t R1, const int64_t* __restrict__ kb_fact_rel, int B,
                                    int64_t max_fact, int D, float* __restrict__ grad_qh) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * Q * D) return;
  const int64_t c = i % D, q = (i / D) % Q, b = i / ((int64_t)Q * D);
  float v = 0.f;
  for (int64_t s = b * max_fact, e = s + max_fact; s < e; ++s) {
    const float cq = coef[s * Q + q];
    if (cq != 0.f) v = __fadd_rn(v, __fmul_rn(cq, __ldg(rel + slot_rel(kb_fact_rel, s, R1) * ldr + c)));
  }
  grad_qh[i] = __fadd_rn(grad_qh[i], v);
}

// grad_rel[r] += sum over the slots of relation r, in slot order, of sum_q c[s, q] qh[b_s, q] (q in order).
// Entry i of the slot-level relation index -> slot rix_slot[i].
template <int NC>
__global__ void __launch_bounds__(256) graft_rel_det_kernel(const float* __restrict__ coef, int Q,
                                                            const float* __restrict__ qh, int64_t R1,
                                                            const int64_t* __restrict__ kb_fact_rel,
                                                            int64_t max_fact, int D,
                                                            const int32_t* __restrict__ rix_ptr,
                                                            const int32_t* __restrict__ rix_slot,
                                                            float* __restrict__ grad_rel, int64_t ld_grel,
                                                            float* __restrict__ part) {
  const int lane = threadIdx.x & 31;
  const int64_t win = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t L = rix_ptr[R1];
  const int64_t lo = win * kFactWin, hi = min(L, lo + kFactWin);
  if (lo >= L) return;
  auto seg_of = [&](int64_t i) { return slot_rel(kb_fact_rel, rix_slot[i], R1); };
  float acc[NC];
  int64_t cur = -1;
  bool first = true;
  auto flush = [&]() {
    const int slot = segwin_slot(lo, hi, L, cur, first, seg_of);
    segwin_store<NC>(acc, slot, part + (win * 2 + (slot > 0)) * D, grad_rel + cur * ld_grel, D);
    first = false;
  };
  for (int64_t i = lo; i < hi; ++i) {
    const int64_t s = rix_slot[i], r = slot_rel(kb_fact_rel, s, R1);
    if (r != cur) {
      if (cur >= 0) flush();
      cur = r;
#pragma unroll
      for (int k = 0; k < NC; ++k) acc[k] = 0.f;
    }
    const float* qb = qh + (s / max_fact) * (int64_t)Q * D;
    float t[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) t[k] = 0.f;
#pragma unroll 1
    for (int q = 0; q < Q; ++q) {
      const float cq = coef[s * Q + q];
      if (cq == 0.f) continue;           // warp-uniform
#pragma unroll
      for (int k = 0; k < NC; ++k) {
        const int c = lane + 32 * k;
        if (c < D) t[k] = __fadd_rn(t[k], __fmul_rn(cq, __ldg(qb + (int64_t)q * D + c)));
      }
    }
#pragma unroll
    for (int k = 0; k < NC; ++k) acc[k] = __fadd_rn(acc[k], t[k]);
  }
  flush();
}

}  // namespace
}  // namespace gr

using namespace gr;

extern "C" size_t gr_graft_stage_workspace_bytes(int64_t B, int64_t max_fact) {
  return stage_ws(B * max_fact).total;
}

extern "C" int gr_graft_stage(const int64_t* e2f_b, const int64_t* e2f_f, const int64_t* e2f_e, int64_t F_e2f,
                              const int64_t* f2e_b, const int64_t* f2e_e, const int64_t* f2e_f, int64_t F_f2e,
                              const int64_t* kb_fact_rel, int B, int N, int64_t max_fact, int64_t R1, int32_t* heads,
                              int32_t* rels, int32_t* tails, int32_t* slot_of, int32_t* nfacts, int32_t* status,
                              const int32_t* live, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(B > 0 && N > 0 && max_fact >= 0 && R1 > 0 && F_e2f >= 0 && F_f2e >= 0, "bad sizes");
  GR_CHECK_ARG(nfacts && status && (max_fact == 0 || kb_fact_rel), "null pointer");   // max_fact == 0: no slots
  GR_CHECK_ARG((int64_t)B * N < 0x7fffffff && (int64_t)B * max_fact < 0x7fffffff, "B*N or B*max_fact exceeds int32");
  GR_CHECK_ARG(F_e2f == 0 || (e2f_b && e2f_f && e2f_e && heads && rels && tails && slot_of), "null pointer");
  GR_CHECK_ARG(F_f2e == 0 || (f2e_b && f2e_e && f2e_f), "null pointer");
  const int64_t S = (int64_t)B * max_fact;
  StageWs w = stage_ws(S);
  if (int rc = check_workspace(__func__, workspace, workspace_bytes, w.total)) return rc;
  char* ws = reinterpret_cast<char*>(workspace);
  int32_t* head_of = reinterpret_cast<int32_t*>(ws);
  int32_t* tail_of = reinterpret_cast<int32_t*>(ws + w.dense_bytes);
  int32_t* flag = reinterpret_cast<int32_t*>(ws + 2 * w.dense_bytes);
  int32_t* pos = reinterpret_cast<int32_t*>(ws + 3 * w.dense_bytes);
  void* tmp = ws + 4 * w.dense_bytes;
  GR_CHECK_CUDA(cudaMemsetAsync(head_of, 0xff, 2 * w.dense_bytes, stream));
  GR_CHECK_CUDA(cudaMemsetAsync(nfacts, 0, sizeof(int32_t), stream));
  // with live counts F_e2f / F_f2e are capacities: the launch shape depends on them only (fixed under graph capture)
  const int g1 = (int)std::min<int64_t>(ceil_div(std::max<int64_t>(std::max(F_e2f, F_f2e), 1), 256), 4096);
  if (F_e2f > 0) {
    graft_scatter_kernel<<<g1, 256, 0, stream>>>(e2f_b, e2f_f, e2f_e, F_e2f, live, B, N, max_fact, head_of,
                                                 status);
    GR_CHECK_LAUNCH();
  }
  if (S == 0) {           // no slots: every listed fact is out of range (reported by the scatter)
    if (F_f2e > 0) {
      graft_scatter_kernel<<<g1, 256, 0, stream>>>(f2e_b, f2e_f, f2e_e, F_f2e, live ? live + 1 : nullptr, B, N,
                                                 max_fact, tail_of, status);
      GR_CHECK_LAUNCH();
    }
    return GR_OK;
  }
  if (F_f2e > 0) {
    graft_scatter_kernel<<<g1, 256, 0, stream>>>(f2e_b, f2e_f, f2e_e, F_f2e, live ? live + 1 : nullptr, B, N,
                                                 max_fact, tail_of, status);
    GR_CHECK_LAUNCH();
  }
  const int g2 = (int)std::min<int64_t>(ceil_div(S, 256), 8192);
  graft_flags_kernel<<<g2, 256, 0, stream>>>(head_of, tail_of, S, flag, status);
  GR_CHECK_LAUNCH();
  size_t tmp_bytes = w.scan_bytes;
  GR_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, flag, pos, (int)S, stream));
  graft_compact_kernel<<<g2, 256, 0, stream>>>(head_of, tail_of, flag, pos, kb_fact_rel, S, R1, F_e2f, heads, rels,
                                               tails, slot_of, nfacts, status);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_graft_attention(const float* qh, const float* qmask, int Q, const float* rel, int64_t ldr,
                                  int64_t R1, const int64_t* kb_fact_rel, int B, int64_t max_fact, int D,
                                  const int32_t* rowptr_h, const int32_t* fact_h, const int32_t* slot_of, int N,
                                  float* W, float* Wt, float* E, int32_t* status, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(B > 0 && N > 0 && D > 0 && D <= 512 && Q >= 0 && max_fact >= 0 && R1 > 0 && ldr >= D,
               "bad sizes (need 0 < D <= 512)");
  GR_CHECK_ARG(rowptr_h && E && status, "null pointer");
  GR_CHECK_ARG(max_fact == 0 || (qh && qmask && rel && kb_fact_rel && W && Wt && fact_h && slot_of), "null pointer");
  GR_CHECK_ARG(Q > 0 || max_fact == 0, "Q must be positive");
  const int64_t S = (int64_t)B * max_fact, Nt = (int64_t)B * N;
  if (S > 0) {
    const float div = (float)sqrt((double)D);
    const int grid = (int)ceil_div(S, 8);
    with_nc(D, [&](auto nc) {
      graft_w_kernel<decltype(nc)::value><<<grid, 256, 0, stream>>>(qh, qmask, Q, rel, ldr, R1, kb_fact_rel, S,
                                                                     max_fact, D, div, W, status);
    });
    GR_CHECK_LAUNCH();
    graft_wtilde_kernel<<<B, 256, 0, stream>>>(W, max_fact, Wt);
    GR_CHECK_LAUNCH();
  }
  graft_e_kernel<<<(int)ceil_div(Nt, 256), 256, 0, stream>>>(rowptr_h, fact_h, slot_of, Wt, Nt, E);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_graft_aggregate(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                                  const int32_t* fact_t, const int32_t* slot_of, const float* Wt, const float* E,
                                  const float* prior, const float* self_tab, int64_t ld_self, const float* head_tab,
                                  int64_t ld_head, const float* q2e, double lambda, float* sum_out, int64_t ld_sum,
                                  void* out_hi, void* out_lo, int64_t ld_planes, int64_t col_sum, int64_t col_indeg,
                                  int64_t col_q2e, float* indeg_out, float* prior_next, int B, int N, int D,
                                  void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(B > 0 && N > 0 && D > 0 && D <= 512, "bad sizes (need 0 < D <= 512)");
  GR_CHECK_ARG(rowptr_t && src_t && rel_t && fact_t && slot_of && Wt && E && prior && self_tab && head_tab &&
                   prior_next, "null pointer");
  GR_CHECK_ARG(ld_self >= D && ld_head >= D && (!sum_out || ld_sum >= D), "leading dimension smaller than D");
  GR_CHECK_ARG(!out_hi || (out_lo && col_sum >= 0 && col_sum + D <= ld_planes && col_indeg >= 0 &&
                           col_indeg < ld_planes && (!q2e || (col_q2e >= 0 && col_q2e + D <= ld_planes))),
               "plane columns outside the row");
  AggArgs a{};
  a.rowptr = rowptr_t; a.src = src_t; a.rel = rel_t; a.fact = fact_t; a.slot_of = slot_of;
  a.Wt = Wt; a.E = E; a.prior = prior; a.self_tab = self_tab; a.head_tab = head_tab; a.q2e = out_hi ? q2e : nullptr;
  a.ld_self = ld_self; a.ld_head = ld_head;
  a.lam = (float)lambda;                     // pagerank_lambda * x and (1 - pagerank_lambda) * y with the python
  a.one_minus_lam = (float)(1.0 - lambda);   // double rounded once to fp32, as torch applies the scalars
  a.sum_out = sum_out; a.ld_sum = ld_sum;
  a.hi = reinterpret_cast<__nv_bfloat16*>(out_hi); a.lo = reinterpret_cast<__nv_bfloat16*>(out_lo);
  a.ld_planes = ld_planes; a.col_sum = col_sum; a.col_indeg = col_indeg; a.col_q2e = col_q2e;
  a.indeg_out = indeg_out; a.prior_next = prior_next;
  a.Nt = (int64_t)B * N; a.N = N; a.D = D;
  const int grid = (int)ceil_div(a.Nt, 8);
  with_nc(D, [&](auto nc) { graft_aggregate_kernel<decltype(nc)::value><<<grid, 256, 0, stream>>>(a); });
  GR_CHECK_LAUNCH();
  return GR_OK;
}

// ---- training entry points -----------------------------------------------------------------------------------------

namespace {

// dropout arguments shared by the training entry points: p in [0, 1); p > 0 needs the seed, p == 0 ignores it
int drop_args(const int64_t* seed, double p, TrainArgs& a) {
  GR_CHECK_ARG(p >= 0.0 && p < 1.0, "dropout probability outside [0, 1)");
  GR_CHECK_ARG(p == 0.0 || seed, "null seed with p > 0");
  a.seed = p > 0.0 ? seed : nullptr;
  a.p = (float)p;
  a.scale = (float)(1.0 / (1.0 - p));
  return GR_OK;
}

}  // namespace

extern "C" int gr_graft_dropout_mask(const int64_t* seed, double p, int64_t S, int D, uint8_t* mask, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(S >= 0 && D > 0 && D <= 512, "bad sizes (need S >= 0, 0 < D <= 512)");
  GR_CHECK_ARG(p >= 0.0 && p < 1.0, "dropout probability outside [0, 1)");
  GR_CHECK_ARG(S == 0 || mask, "null pointer");
  GR_CHECK_ARG(p == 0.0 || seed, "null seed with p > 0");
  if (S == 0) return GR_OK;
  const int grid = (int)std::min<int64_t>(ceil_div(S * D, 256), 8192);
  graft_dropout_mask_kernel<<<grid, 256, 0, stream>>>(seed, (float)p, S, D, mask);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_graft_aggregate_train_ex(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                                           const int32_t* fact_t, const int32_t* slot_of, const float* s,
                                           const float* self_tab, int64_t ld_self, const void* head_tab,
                                           int64_t ld_head, const int64_t* seed, double p, void* sum_out,
                                           int64_t ld_sum, int B, int N, int D, uint32_t io, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (int rc = check_io(__func__, io)) return rc;
  GR_CHECK_ARG(B > 0 && N > 0 && D > 0 && D <= 512, "bad sizes (need 0 < D <= 512)");
  GR_CHECK_ARG(rowptr_t && src_t && rel_t && fact_t && slot_of && s && self_tab && head_tab && sum_out,
               "null pointer");
  GR_CHECK_ARG(ld_self >= D && ld_head >= D && ld_sum >= D, "leading dimension smaller than D");
  TrainArgs a{};
  if (int rc = drop_args(seed, p, a)) return rc;
  a.rowptr = rowptr_t; a.src = src_t; a.rel = rel_t; a.fact = fact_t; a.slot_of = slot_of;
  a.s = s; a.self_tab = self_tab; a.head_tab = head_tab; a.ld_self = ld_self; a.ld_head = ld_head;
  a.sum_out = sum_out; a.ld_sum = ld_sum;
  a.Nt = (int64_t)B * N; a.D = D;
  const int grid = (int)ceil_div(a.Nt, 8);
  with_nc(D, [&](auto nc) {
    with_node_type(io, [&](auto t) {
      graft_aggregate_train_kernel<decltype(nc)::value, typename decltype(t)::type><<<grid, 256, 0, stream>>>(a);
    });
  });
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_graft_aggregate_train(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                                        const int32_t* fact_t, const int32_t* slot_of, const float* s,
                                        const float* self_tab, int64_t ld_self, const float* head_tab, int64_t ld_head,
                                        const int64_t* seed, double p, float* sum_out, int64_t ld_sum, int B, int N,
                                        int D, void* stream_) {
  return gr_graft_aggregate_train_ex(rowptr_t, src_t, rel_t, fact_t, slot_of, s, self_tab, ld_self, head_tab, ld_head,
                                     seed, p, sum_out, ld_sum, B, N, D, 0u, stream_);
}

// ---- deterministic training entry points ---------------------------------------------------------------------------

extern "C" size_t gr_graft_aggregate_backward_det_workspace_bytes(int64_t F, int D) {
  if (F < 0 || D <= 0) return 0;
  return segwin_part_bytes(F, D, kFactWin);
}

namespace {

// gr_graft_aggregate_backward_ex (det == false: grad_self by fp32 atomics) and gr_graft_aggregate_backward_det_ex
// (det == true: fixed-order grad_self, which also takes the arguments after D); `fn` is the entry point the argument
// checks report.
int graft_aggregate_backward(const char* fn, bool det, const int32_t* rowptr_h, const int32_t* src_h,
                             const int32_t* rel_h, const int32_t* fact_h, const int32_t* slot_of, const float* s,
                             const float* self_tab, int64_t ld_self, const void* head_tab, int64_t ld_head,
                             const int64_t* seed, double p, const void* grad_sum, int64_t ld_grad, float* grad_s,
                             float* grad_self, int64_t ld_gself, void* grad_head, int64_t ld_ghead, int B, int N, int D,
                             const int32_t* heads, const int32_t* rels, const int32_t* tails, const int32_t* rix_ptr,
                             const int32_t* rix_fact, int64_t R1, int64_t F, void* workspace, size_t workspace_bytes,
                             uint32_t io, cudaStream_t stream) {
  if (int rc = check_io(fn, io)) return rc;
  GR_CHECK_ARG_AS(fn, B > 0 && N > 0 && D > 0 && D <= 512 && (!det || (R1 > 0 && F >= 0)),
                  "bad sizes (need 0 < D <= 512)");
  GR_CHECK_ARG_AS(fn, rowptr_h && src_h && rel_h && fact_h && slot_of && s && self_tab && head_tab && grad_sum &&
                          grad_s && grad_self && grad_head && (!det || (heads && rels && tails && rix_ptr && rix_fact)),
                  "null pointer");
  GR_CHECK_ARG_AS(fn, ld_self >= D && ld_head >= D && ld_grad >= D && ld_gself >= D && ld_ghead >= D,
                  "leading dimension smaller than D");
  TrainArgs a{};
  if (int rc = drop_args(seed, p, a)) return rc;
  const size_t need = det ? segwin_part_bytes(F, D, kFactWin) : 0;
  if (det) {
    if (int rc = check_workspace("gr_graft_aggregate_backward_det", workspace, workspace_bytes, need)) return rc;
  }
  a.rowptr = rowptr_h; a.src = src_h; a.rel = rel_h; a.fact = fact_h; a.slot_of = slot_of;
  a.s = s; a.self_tab = self_tab; a.head_tab = head_tab; a.ld_self = ld_self; a.ld_head = ld_head;
  a.grad = grad_sum; a.ld_grad = ld_grad;
  a.grad_s = grad_s; a.grad_self = grad_self; a.grad_head = grad_head; a.ld_gself = ld_gself; a.ld_ghead = ld_ghead;
  a.Nt = (int64_t)B * N; a.D = D;
  const int grid = (int)ceil_div(a.Nt, 8);
  with_nc(D, [&](auto nc) {
    with_node_type(io, [&](auto t) {
      constexpr int NC = decltype(nc)::value;
      using T = typename decltype(t)::type;
      if (det) graft_aggregate_bwd_kernel<NC, false, T><<<grid, 256, 0, stream>>>(a);
      else graft_aggregate_bwd_kernel<NC, true, T><<<grid, 256, 0, stream>>>(a);
    });
  });
  GR_CHECK_LAUNCH_AS(fn);
  if (!det || F == 0) return GR_OK;
  float* part = reinterpret_cast<float*>(workspace);
  const int grid_w = (int)ceil_div(ceil_div(F, kFactWin), 8);
  with_nc(D, [&](auto nc) {
    with_node_type(io, [&](auto t) {
      graft_self_det_kernel<decltype(nc)::value, typename decltype(t)::type><<<grid_w, 256, 0, stream>>>(
          a, rix_ptr, rix_fact, heads, rels, tails, part, R1);
    });
  });
  GR_CHECK_LAUNCH_AS(fn);
  segwin_combine_kernel<kFactWin><<<(int)ceil_div(R1 * D, 256), 256, 0, stream>>>(part, D, rix_ptr, 0, R1, grad_self,
                                                                                  ld_gself);
  GR_CHECK_LAUNCH_AS(fn);
  return GR_OK;
}

}  // namespace

extern "C" int gr_graft_aggregate_backward_ex(const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h,
                                              const int32_t* fact_h, const int32_t* slot_of, const float* s,
                                              const float* self_tab, int64_t ld_self, const void* head_tab,
                                              int64_t ld_head, const int64_t* seed, double p, const void* grad_sum,
                                              int64_t ld_grad, float* grad_s, float* grad_self, int64_t ld_gself,
                                              void* grad_head, int64_t ld_ghead, int B, int N, int D, uint32_t io,
                                              void* stream_) {
  return graft_aggregate_backward(__func__, false, rowptr_h, src_h, rel_h, fact_h, slot_of, s, self_tab, ld_self,
                                  head_tab, ld_head, seed, p, grad_sum, ld_grad, grad_s, grad_self, ld_gself,
                                  grad_head, ld_ghead, B, N, D, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 0,
                                  nullptr, 0, io, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_graft_aggregate_backward(const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h,
                                           const int32_t* fact_h, const int32_t* slot_of, const float* s,
                                           const float* self_tab, int64_t ld_self, const float* head_tab,
                                           int64_t ld_head, const int64_t* seed, double p, const float* grad_sum,
                                           int64_t ld_grad, float* grad_s, float* grad_self, int64_t ld_gself,
                                           float* grad_head, int64_t ld_ghead, int B, int N, int D, void* stream_) {
  return gr_graft_aggregate_backward_ex(rowptr_h, src_h, rel_h, fact_h, slot_of, s, self_tab, ld_self, head_tab,
                                        ld_head, seed, p, grad_sum, ld_grad, grad_s, grad_self, ld_gself, grad_head,
                                        ld_ghead, B, N, D, 0u, stream_);
}

extern "C" int gr_graft_aggregate_backward_det_ex(const int32_t* rowptr_h, const int32_t* src_h,
                                                  const int32_t* rel_h, const int32_t* fact_h, const int32_t* slot_of,
                                                  const float* s, const float* self_tab, int64_t ld_self,
                                                  const void* head_tab, int64_t ld_head, const int64_t* seed, double p,
                                                  const void* grad_sum, int64_t ld_grad, float* grad_s,
                                                  float* grad_self, int64_t ld_gself, void* grad_head,
                                                  int64_t ld_ghead, int B, int N, int D, const int32_t* heads,
                                                  const int32_t* rels, const int32_t* tails, const int32_t* rix_ptr,
                                                  const int32_t* rix_fact, int64_t R1, int64_t F, void* workspace,
                                                  size_t workspace_bytes, uint32_t io, void* stream_) {
  return graft_aggregate_backward(__func__, true, rowptr_h, src_h, rel_h, fact_h, slot_of, s, self_tab, ld_self,
                                  head_tab, ld_head, seed, p, grad_sum, ld_grad, grad_s, grad_self, ld_gself,
                                  grad_head, ld_ghead, B, N, D, heads, rels, tails, rix_ptr, rix_fact, R1, F,
                                  workspace, workspace_bytes, io, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_graft_aggregate_backward_det(const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h,
                                               const int32_t* fact_h, const int32_t* slot_of, const float* s,
                                               const float* self_tab, int64_t ld_self, const float* head_tab,
                                               int64_t ld_head, const int64_t* seed, double p, const float* grad_sum,
                                               int64_t ld_grad, float* grad_s, float* grad_self, int64_t ld_gself,
                                               float* grad_head, int64_t ld_ghead, int B, int N, int D,
                                               const int32_t* heads, const int32_t* rels, const int32_t* tails,
                                               const int32_t* rix_ptr, const int32_t* rix_fact, int64_t R1, int64_t F,
                                               void* workspace, size_t workspace_bytes, void* stream_) {
  return gr_graft_aggregate_backward_det_ex(rowptr_h, src_h, rel_h, fact_h, slot_of, s, self_tab, ld_self, head_tab,
                                            ld_head, seed, p, grad_sum, ld_grad, grad_s, grad_self, ld_gself,
                                            grad_head, ld_ghead, B, N, D, heads, rels, tails, rix_ptr, rix_fact, R1, F,
                                            workspace, workspace_bytes, 0u, stream_);
}

extern "C" int gr_graft_attention_backward(const float* qh, const float* qmask, int Q, const float* rel, int64_t ldr,
                                           int64_t R1, const int64_t* kb_fact_rel, int B, int64_t max_fact, int D,
                                           const float* grad_W, float* grad_qh, float* grad_rel, int64_t ld_grel,
                                           void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(B > 0 && B <= 65535 && D > 0 && D <= 512 && Q > 0 && max_fact >= 0 && R1 > 0 && ldr >= D &&
                   ld_grel >= D, "bad sizes (need 0 < D <= 512, 0 < B <= 65535, Q > 0)");
  GR_CHECK_ARG(qh && qmask && rel && grad_qh && grad_rel && (max_fact == 0 || (kb_fact_rel && grad_W)),
               "null pointer");
  if (max_fact == 0) return GR_OK;
  const float div = (float)sqrt((double)D);
  const size_t acc_bytes = (size_t)Q * D * sizeof(float);
  const bool smem_acc = acc_bytes <= 48 * 1024;
  const size_t smem = smem_acc ? acc_bytes : 0;
  const dim3 grid((unsigned)ceil_div(max_fact, kSlotsPerBlock), (unsigned)B);
  with_nc(D, [&](auto nc) {
    graft_w_bwd_kernel<decltype(nc)::value><<<grid, 256, smem, stream>>>(qh, qmask, Q, rel, ldr, R1, kb_fact_rel,
                                                                          max_fact, D, div, grad_W, grad_qh, grad_rel,
                                                                          ld_grel, smem_acc);
  });
  GR_CHECK_LAUNCH();
  return GR_OK;
}

namespace {
struct AttnDetWs {
  size_t coef_bytes, total;
};
AttnDetWs attn_det_ws(int64_t S, int Q, int D) {
  AttnDetWs w;
  w.coef_bytes = align_up((size_t)(S > 0 ? S : 1) * (size_t)Q * sizeof(float), 256);
  w.total = w.coef_bytes + segwin_part_bytes(S, D, kFactWin);
  return w;
}
}  // namespace

extern "C" size_t gr_graft_attention_backward_det_workspace_bytes(int B, int64_t max_fact, int Q, int D) {
  if (B <= 0 || max_fact < 0 || Q <= 0 || D <= 0) return 0;
  return attn_det_ws((int64_t)B * max_fact, Q, D).total;
}

extern "C" int gr_graft_attention_backward_det(const float* qh, const float* qmask, int Q, const float* rel,
                                               int64_t ldr, int64_t R1, const int64_t* kb_fact_rel, int B,
                                               int64_t max_fact, int D, const float* grad_W, float* grad_qh,
                                               float* grad_rel, int64_t ld_grel, const int32_t* rix_ptr,
                                               const int32_t* rix_slot, void* workspace, size_t workspace_bytes,
                                               void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(B > 0 && D > 0 && D <= 512 && Q > 0 && max_fact >= 0 && R1 > 0 && ldr >= D && ld_grel >= D,
               "bad sizes (need 0 < D <= 512, Q > 0)");
  GR_CHECK_ARG(qh && qmask && rel && kb_fact_rel && grad_W && grad_qh && grad_rel && rix_ptr, "null pointer");
  GR_CHECK_ARG(max_fact == 0 || rix_slot, "null pointer");
  const int64_t S = (int64_t)B * max_fact;
  GR_CHECK_ARG(S < 0x7fffffff, "B*max_fact exceeds int32");
  if (S == 0) return GR_OK;
  const AttnDetWs ws = attn_det_ws(S, Q, D);
  if (int rc = check_workspace(__func__, workspace, workspace_bytes, ws.total)) return rc;
  float* coef = reinterpret_cast<float*>(workspace);
  float* part = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + ws.coef_bytes);
  const float div = (float)sqrt((double)D);
  with_nc(D, [&](auto nc) {
    graft_w_coef_kernel<decltype(nc)::value><<<(int)ceil_div(S, 8), 256, 0, stream>>>(
        qh, qmask, Q, rel, ldr, R1, kb_fact_rel, S, max_fact, D, div, grad_W, coef);
  });
  GR_CHECK_LAUNCH();
  graft_qh_det_kernel<<<(int)ceil_div((int64_t)B * Q * D, 256), 256, 0, stream>>>(coef, Q, rel, ldr, R1, kb_fact_rel,
                                                                                  B, max_fact, D, grad_qh);
  GR_CHECK_LAUNCH();
  with_nc(D, [&](auto nc) {
    graft_rel_det_kernel<decltype(nc)::value><<<(int)ceil_div(ceil_div(S, kFactWin), 8), 256, 0, stream>>>(
        coef, Q, qh, R1, kb_fact_rel, max_fact, D, rix_ptr, rix_slot, grad_rel, ld_grel, part);
  });
  GR_CHECK_LAUNCH();
  segwin_combine_kernel<kFactWin><<<(int)ceil_div(R1 * D, 256), 256, 0, stream>>>(part, D, rix_ptr, 0, R1, grad_rel,
                                                                                  ld_grel);
  GR_CHECK_LAUNCH();
  return GR_OK;
}
