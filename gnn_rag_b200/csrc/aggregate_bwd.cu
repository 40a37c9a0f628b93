// Backward of the relation-typed aggregation (SURVEY.md 8f row 4: the kernel Trainer_KBQA.train_epoch needs,
// gnn/train_model.py:209-233).  Forward (gr_aggregate; ReasonGNNLayer.reason_layer / reason_layer_inv,
// gnn/modules/kg_reasoning/reasongnn.py:61-116; NSMLayer.reason_layer, nsm_gnn.py:87-112):
//
//     out[n, j, :] = sum_{e -> n} c_e * relu(P[r_e, :] * x_j[b(n), :]),     c_e = w_e^2 * p[s_e]
//
// Given G = dL/dout the three gradients are reductions over the same edge list with three different keys:
//
//     dP[r, :]    = sum_{e: r_e = r}   c_e * sum_j  G[n_e, j, :] * x_j[b, :] * m_{e,j}       (key: relation)
//     dx_j[b, :]  = sum_{e in b}       c_e *        G[n_e, j, :] * P[r_e, :] * m_{e,j}       (key: question)
//     dp[s]       = sum_{e: s_e = s} w_e^2 * sum_j <G[n_e, j, :], relu(P[r_e, :] * x_j[b, :])>   (key: source node)
//
// with m_{e,j} = [P[r_e] * x_j[b] > 0] elementwise.  One warp per destination row walks the row's in-edges in the
// destination CSR the forward uses (so G[n] and x_j[b] are loaded once per row and stay in registers); dx_j is
// accumulated in registers across all rows a warp handles inside one question and flushed with one atomicAdd per
// column on a question change; dP and dp go out through fp32 atomics (relation rows / source nodes are random).  The
// gradient buffers are ACCUMULATED into (caller zeroes them): the two directions and the T x K layer calls of one
// backward pass add up in place.  Atomic accumulation order is not deterministic -- as in the reference, whose
// torch.sparse.mm backward on CUDA is an atomic scatter as well.
#include <algorithm>

#include "common.cuh"

namespace gr {
namespace {

constexpr int kBwdThreads = 256;
constexpr int kCPL = 8;                 // columns per lane: D <= 256

struct BwdParams {
  const int32_t* rowptr;
  const int32_t* src;
  const int32_t* rel;
  const float* w;
  const float* prior;
  const float* table;     // [R1, D]
  const float* ins;       // [B, I, D]
  const void* gout;       // [Nt, ld] fp32 or bf16: G[n, j, d] at n * ld + col0 + j * seg + d
  int64_t ld, col0, seg;
  float* gtable;          // [R1, D]   +=
  float* gins;            // [B, I, D] +=
  float* gprior;          // [Nt]      +=
  int64_t Nt;
  int N, D, I;
};

template <int NI, typename TG>
__global__ void __launch_bounds__(kBwdThreads) agg_bwd_kernel(const BwdParams p) {
  const TG* gout = static_cast<const TG*>(p.gout);
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  // contiguous row ranges per warp: a warp stays inside one question for ~all of its rows
  const int64_t per = (p.Nt + nwarps - 1) / nwarps;
  const int64_t row_beg = warp * per, row_end = min(p.Nt, row_beg + per);
  const int D = p.D;
  float x[NI][kCPL], dx[NI][kCPL];
  int cur_b = -1;
  auto flush = [&]() {
    if (cur_b < 0) return;
#pragma unroll
    for (int j = 0; j < NI; ++j)
#pragma unroll
      for (int k = 0; k < kCPL; ++k) {
        const int c = lane + 32 * k;
        if (c < D && dx[j][k] != 0.f) atomicAdd(p.gins + ((int64_t)cur_b * p.I + j) * D + c, dx[j][k]);
      }
  };
  for (int64_t n = row_beg; n < row_end; ++n) {
    const int b = (int)(n / p.N);
    if (b != cur_b) {
      flush();
      cur_b = b;
#pragma unroll
      for (int j = 0; j < NI; ++j)
#pragma unroll
        for (int k = 0; k < kCPL; ++k) {
          const int c = lane + 32 * k;
          x[j][k] = c < D ? __ldg(p.ins + ((int64_t)b * p.I + j) * D + c) : 0.f;
          dx[j][k] = 0.f;
        }
    }
    const int beg = p.rowptr[n], end = p.rowptr[n + 1];
    if (beg == end) continue;
    float g[NI][kCPL];
#pragma unroll
    for (int j = 0; j < NI; ++j)
#pragma unroll
      for (int k = 0; k < kCPL; ++k) {
        const int c = lane + 32 * k;
        g[j][k] = c < D ? ldg_node(gout + n * p.ld + p.col0 + (int64_t)j * p.seg + c) : 0.f;
      }
    for (int e = beg; e < end; ++e) {
      const int s = p.src[e], r = p.rel[e];
      const float w = p.w ? p.w[e] : 1.f;
      const float w2 = w * w;
      const float c_e = w2 * p.prior[s];
      const float* prow = p.table + (int64_t)r * D;
      float* gprow = p.gtable + (int64_t)r * D;
      float dot = 0.f;
#pragma unroll
      for (int k = 0; k < kCPL; ++k) {
        const int c = lane + 32 * k;
        if (c < D) {
          const float pv = __ldg(prow + c);
          float dp_c = 0.f;
#pragma unroll
          for (int j = 0; j < NI; ++j) {
            const float pre = pv * x[j][k];
            if (pre > 0.f) {
              dp_c = fmaf(g[j][k], x[j][k], dp_c);
              dx[j][k] = fmaf(c_e * g[j][k], pv, dx[j][k]);
              dot = fmaf(g[j][k], pre, dot);
            }
          }
          if (c_e != 0.f && dp_c != 0.f) atomicAdd(gprow + c, c_e * dp_c);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
      if (lane == 0 && dot != 0.f) atomicAdd(p.gprior + s, w2 * dot);
    }
  }
  flush();
}

}  // namespace
}  // namespace gr

// ---- deterministic variant (torch.use_deterministic_algorithms) ----------------------------------------------------
// The same three gradients, each a sum whose order is fixed by the data (common.cuh, fixed-window segmented sums):
//   dx_j[b]  windows of kRowWin destination rows walk the rows and their in-edges in CSR order; segment = question
//   dp[s]    the row walk stores q_e = w_e^2 * dot_e per fact; one thread per source node then adds the q_e of its
//            out-edges in the slot order of the OTHER destination CSR (which lists exactly the edges with that source)
//   dP[r]    windows of kRelWin entries of the relation index (this CSR's slots sorted by (relation, slot)) gather
//            G[n_e] and x_j[b_e] per edge; segment = relation
// Inside every term __fmul_rn / __fadd_rn, so nothing is contracted: dot_e = butterfly over lanes of the lane sums
// over (k, j) of g * (P * x), added in that order.
namespace gr {
namespace {

constexpr int kRowWin = 32;   // destination rows per window of the dx pass
constexpr int kRelWin = 64;   // relation-index entries per window of the dP / grad_table passes

struct DetParams {
  BwdParams p;
  const int32_t *fact, *rowptr_o, *fact_o, *rix_ptr, *rix_slot, *row_of;
  float* q;                 // [F] per-fact w^2 * dot, keyed by original fact id
  float* part;              // segmented-sum partials (dx, then dP)
  int64_t R1;
};

template <int NI, typename TG>
__global__ void __launch_bounds__(kBwdThreads) agg_bwd_det_rows_kernel(const DetParams d) {
  const BwdParams& p = d.p;
  const TG* gout = static_cast<const TG*>(p.gout);
  const int lane = threadIdx.x & 31;
  const int64_t win = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t a = win * kRowWin, bnd = min(p.Nt, a + kRowWin);
  if (a >= p.Nt) return;
  const int D = p.D, N = p.N;
  const int64_t width = (int64_t)p.I * D;
  auto seg_of = [N](int64_t n) { return n / N; };
  float x[NI][kCPL], dx[NI][kCPL];
  int64_t cur_b = -1;
  bool first = true;
  auto flush = [&]() {
    const int slot = segwin_slot(a, bnd, p.Nt, cur_b, first, seg_of);
#pragma unroll
    for (int j = 0; j < NI; ++j)
      segwin_store<kCPL>(dx[j], slot, d.part + (win * 2 + (slot > 0)) * width + j * D,
                         p.gins + cur_b * width + (int64_t)j * D, D);
    first = false;
  };
  for (int64_t n = a; n < bnd; ++n) {
    const int64_t b = n / N;
    if (b != cur_b) {
      if (cur_b >= 0) flush();
      cur_b = b;
#pragma unroll
      for (int j = 0; j < NI; ++j)
#pragma unroll
        for (int k = 0; k < kCPL; ++k) {
          const int c = lane + 32 * k;
          x[j][k] = c < D ? __ldg(p.ins + (b * p.I + j) * D + c) : 0.f;
          dx[j][k] = 0.f;
        }
    }
    const int beg = p.rowptr[n], end = p.rowptr[n + 1];
    if (beg == end) continue;
    float g[NI][kCPL];
#pragma unroll
    for (int j = 0; j < NI; ++j)
#pragma unroll
      for (int k = 0; k < kCPL; ++k) {
        const int c = lane + 32 * k;
        g[j][k] = c < D ? ldg_node(gout + n * p.ld + p.col0 + (int64_t)j * p.seg + c) : 0.f;
      }
    for (int e = beg; e < end; ++e) {
      const int s = p.src[e], r = p.rel[e];
      const float w = p.w ? p.w[e] : 1.f;
      const float w2 = __fmul_rn(w, w);
      const float c_e = __fmul_rn(w2, p.prior[s]);
      const float* prow = p.table + (int64_t)r * D;
      float dot = 0.f;
#pragma unroll
      for (int k = 0; k < kCPL; ++k) {
        const int c = lane + 32 * k;
        if (c < D) {
          const float pv = __ldg(prow + c);
#pragma unroll
          for (int j = 0; j < NI; ++j) {
            const float pre = __fmul_rn(pv, x[j][k]);
            if (pre > 0.f) {
              dx[j][k] = __fadd_rn(dx[j][k], __fmul_rn(__fmul_rn(c_e, g[j][k]), pv));
              dot = __fadd_rn(dot, __fmul_rn(g[j][k], pre));
            }
          }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dot = __fadd_rn(dot, __shfl_xor_sync(0xffffffffu, dot, o));
      if (lane == 0) d.q[d.fact[e]] = __fmul_rn(w2, dot);
    }
  }
  flush();
}

// dp[s] += sum of q over the out-edges of s, in the other CSR's slot order (one thread per node)
__global__ void agg_bwd_det_prior_kernel(const int32_t* __restrict__ rowptr_o, const int32_t* __restrict__ fact_o,
                                         const float* __restrict__ q, float* __restrict__ gprior, int64_t Nt) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= Nt) return;
  const int beg = rowptr_o[s], end = rowptr_o[s + 1];
  if (beg == end) return;
  float v = 0.f;
  for (int e = beg; e < end; ++e) v = __fadd_rn(v, q[fact_o[e]]);
  gprior[s] = __fadd_rn(gprior[s], v);
}

// dP[r] over the relation index: entry i -> CSR slot e = rix_slot[i] of relation rel[e], row row_of[e]
template <int NI, typename TG>
__global__ void __launch_bounds__(kBwdThreads) agg_bwd_det_rel_kernel(const DetParams d) {
  const BwdParams& p = d.p;
  const TG* gout = static_cast<const TG*>(p.gout);
  const int lane = threadIdx.x & 31;
  const int64_t win = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t L = d.rix_ptr[d.R1];
  const int64_t a = win * kRelWin, bnd = min(L, a + kRelWin);
  if (a >= L) return;
  const int D = p.D, N = p.N;
  auto seg_of = [&](int64_t i) { return (int64_t)p.rel[d.rix_slot[i]]; };
  float pv[kCPL], x[NI][kCPL], acc[kCPL];
  int64_t cur_r = -1, cur_b = -1;
  bool first = true;
  auto flush = [&]() {
    const int slot = segwin_slot(a, bnd, L, cur_r, first, seg_of);
    segwin_store<kCPL>(acc, slot, d.part + (win * 2 + (slot > 0)) * D, p.gtable + cur_r * D, D);
    first = false;
  };
  for (int64_t i = a; i < bnd; ++i) {
    const int e = d.rix_slot[i];
    const int64_t r = p.rel[e], n = d.row_of[e], b = n / N;
    if (r != cur_r) {
      if (cur_r >= 0) flush();
      cur_r = r;
#pragma unroll
      for (int k = 0; k < kCPL; ++k) {
        const int c = lane + 32 * k;
        pv[k] = c < D ? __ldg(p.table + r * D + c) : 0.f;
        acc[k] = 0.f;
      }
    }
    if (b != cur_b) {
      cur_b = b;
#pragma unroll
      for (int j = 0; j < NI; ++j)
#pragma unroll
        for (int k = 0; k < kCPL; ++k) {
          const int c = lane + 32 * k;
          x[j][k] = c < D ? __ldg(p.ins + (b * p.I + j) * D + c) : 0.f;
        }
    }
    const float w = p.w ? p.w[e] : 1.f;
    const float c_e = __fmul_rn(__fmul_rn(w, w), p.prior[p.src[e]]);
#pragma unroll
    for (int k = 0; k < kCPL; ++k) {
      const int c = lane + 32 * k;
      if (c < D) {
        float dp_c = 0.f;
#pragma unroll
        for (int j = 0; j < NI; ++j)
          if (__fmul_rn(pv[k], x[j][k]) > 0.f)
            dp_c = __fadd_rn(dp_c, __fmul_rn(ldg_node(gout + n * p.ld + p.col0 + (int64_t)j * p.seg + c), x[j][k]));
        acc[k] = __fadd_rn(acc[k], __fmul_rn(c_e, dp_c));
      }
    }
  }
  flush();
}

struct AggDetWs {
  size_t q_bytes, part_bytes, total;
};

AggDetWs agg_det_ws(int64_t Nt, int D, int I, int64_t F) {
  AggDetWs w;
  w.q_bytes = align_up((size_t)(F > 0 ? F : 1) * sizeof(float), 256);
  w.part_bytes = std::max(segwin_part_bytes(Nt, (int64_t)I * D, kRowWin), segwin_part_bytes(F, D, kRelWin));
  w.total = w.q_bytes + w.part_bytes;
  return w;
}

}  // namespace
}  // namespace gr

extern "C" size_t gr_aggregate_backward_det_workspace_bytes(int B, int N, int D, int I, int64_t F) {
  if (B <= 0 || N <= 0 || D <= 0 || I <= 0 || F < 0) return 0;
  return gr::agg_det_ws((int64_t)B * N, D, I, F).total;
}

namespace gr {
namespace {

// gr_aggregate_backward_ex (det == false: fp32 atomics) and gr_aggregate_backward_det_ex (det == true: the fixed-order
// kernels, which also take the arguments after F); `fn` is the entry point the argument checks report.
int agg_backward(const char* fn, bool det, const int32_t* rowptr, const int32_t* src, const int32_t* rel,
                 const int32_t* fact, const float* w, const float* prior, const float* table, const float* ins,
                 const void* grad_out, int64_t grad_row_stride, int64_t grad_col0, int64_t seg_stride,
                 float* grad_table, float* grad_ins, float* grad_prior, int B, int N, int D, int I, int64_t F,
                 const int32_t* rowptr_o, const int32_t* fact_o, const int32_t* rix_ptr, const int32_t* rix_slot,
                 const int32_t* row_of, int64_t R1, void* workspace, size_t workspace_bytes, uint32_t io,
                 cudaStream_t stream) {
  if (int rc = check_io(fn, io)) return rc;
  GR_CHECK_ARG_AS(fn, rowptr && prior && table && ins && grad_out && grad_table && grad_ins && grad_prior &&
                          (!det || (rowptr_o && rix_ptr)), "null pointer");
  GR_CHECK_ARG_AS(fn, F == 0 || (src && rel && (!det || (fact && fact_o && rix_slot && row_of))), "null edge arrays");
  GR_CHECK_ARG_AS(fn, B > 0 && N > 0 && D > 0 && D <= 32 * kCPL && I > 0 && I <= 4 && (!det || (F >= 0 && R1 > 0)),
                  "need 0 < D <= 256 and 0 < I <= 4");
  GR_CHECK_ARG_AS(fn, seg_stride >= D && grad_row_stride >= grad_col0 + (int64_t)(I - 1) * seg_stride + D,
                  "grad_out row stride / segment stride smaller than the rows it must hold");
  if (F == 0) return GR_OK;
  const int64_t Nt = (int64_t)B * N;
  DetParams d{};
  BwdParams& p = d.p;
  p.rowptr = rowptr; p.src = src; p.rel = rel; p.w = w; p.prior = prior; p.table = table; p.ins = ins;
  p.gout = grad_out; p.ld = grad_row_stride; p.col0 = grad_col0; p.seg = seg_stride;
  p.gtable = grad_table; p.gins = grad_ins; p.gprior = grad_prior;
  p.Nt = Nt; p.N = N; p.D = D; p.I = I;
  if (!det) {
    const int grid = (int)std::min<int64_t>(ceil_div(p.Nt * 32, kBwdThreads), 16LL * sm_count());
    with_ni(I, [&](auto ni) {
      with_node_type(io, [&](auto t) {
        agg_bwd_kernel<decltype(ni)::value, typename decltype(t)::type><<<grid, kBwdThreads, 0, stream>>>(p);
      });
    });
    GR_CHECK_LAUNCH_AS(fn);
    return GR_OK;
  }
  const AggDetWs ws = agg_det_ws(Nt, D, I, F);
  if (int rc = check_workspace("gr_aggregate_backward_det", workspace, workspace_bytes, ws.total)) return rc;
  d.fact = fact; d.rowptr_o = rowptr_o; d.fact_o = fact_o; d.rix_ptr = rix_ptr; d.rix_slot = rix_slot;
  d.row_of = row_of; d.R1 = R1;
  d.q = reinterpret_cast<float*>(workspace);
  d.part = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + ws.q_bytes);
  const int wpb = kBwdThreads / 32;
  const int grid_rows = (int)ceil_div(ceil_div(Nt, kRowWin), wpb);
  const int grid_rel = (int)ceil_div(ceil_div(F, kRelWin), wpb);
  const int64_t width = (int64_t)I * D;
  with_ni(I, [&](auto ni) {
    with_node_type(io, [&](auto t) {
      agg_bwd_det_rows_kernel<decltype(ni)::value, typename decltype(t)::type><<<grid_rows, kBwdThreads, 0, stream>>>(d);
    });
  });
  GR_CHECK_LAUNCH_AS(fn);
  segwin_combine_kernel<kRowWin><<<(int)ceil_div(B * width, 256), 256, 0, stream>>>(d.part, width, nullptr, N, B,
                                                                                   grad_ins, width);
  GR_CHECK_LAUNCH_AS(fn);
  agg_bwd_det_prior_kernel<<<(int)ceil_div(Nt, 256), 256, 0, stream>>>(rowptr_o, fact_o, d.q, grad_prior, Nt);
  GR_CHECK_LAUNCH_AS(fn);
  with_ni(I, [&](auto ni) {
    with_node_type(io, [&](auto t) {
      agg_bwd_det_rel_kernel<decltype(ni)::value, typename decltype(t)::type><<<grid_rel, kBwdThreads, 0, stream>>>(d);
    });
  });
  GR_CHECK_LAUNCH_AS(fn);
  segwin_combine_kernel<kRelWin><<<(int)ceil_div(R1 * D, 256), 256, 0, stream>>>(d.part, D, rix_ptr, 0, R1,
                                                                                 grad_table, D);
  GR_CHECK_LAUNCH_AS(fn);
  return GR_OK;
}

}  // namespace
}  // namespace gr

extern "C" int gr_aggregate_backward_det_ex(const int32_t* rowptr, const int32_t* src, const int32_t* rel,
                                            const int32_t* fact, const float* w, const float* prior,
                                            const float* table, const float* ins, const void* grad_out,
                                            int64_t grad_row_stride, int64_t grad_col0, int64_t seg_stride,
                                            float* grad_table, float* grad_ins, float* grad_prior, int B, int N, int D,
                                            int I, int64_t F, const int32_t* rowptr_o, const int32_t* fact_o,
                                            const int32_t* rix_ptr, const int32_t* rix_slot, const int32_t* row_of,
                                            int64_t R1, void* workspace, size_t workspace_bytes, uint32_t io,
                                            void* stream_) {
  return gr::agg_backward(__func__, true, rowptr, src, rel, fact, w, prior, table, ins, grad_out, grad_row_stride,
                          grad_col0, seg_stride, grad_table, grad_ins, grad_prior, B, N, D, I, F, rowptr_o, fact_o,
                          rix_ptr, rix_slot, row_of, R1, workspace, workspace_bytes, io,
                          reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_aggregate_backward_det(const int32_t* rowptr, const int32_t* src, const int32_t* rel,
                                         const int32_t* fact, const float* w, const float* prior, const float* table,
                                         const float* ins, const float* grad_out, int64_t grad_row_stride,
                                         int64_t grad_col0, int64_t seg_stride, float* grad_table, float* grad_ins,
                                         float* grad_prior, int B, int N, int D, int I, int64_t F,
                                         const int32_t* rowptr_o, const int32_t* fact_o, const int32_t* rix_ptr,
                                         const int32_t* rix_slot, const int32_t* row_of, int64_t R1, void* workspace,
                                         size_t workspace_bytes, void* stream_) {
  return gr_aggregate_backward_det_ex(rowptr, src, rel, fact, w, prior, table, ins, grad_out, grad_row_stride,
                                      grad_col0, seg_stride, grad_table, grad_ins, grad_prior, B, N, D, I, F, rowptr_o,
                                      fact_o, rix_ptr, rix_slot, row_of, R1, workspace, workspace_bytes, 0u, stream_);
}

extern "C" int gr_aggregate_backward_ex(const int32_t* rowptr, const int32_t* src, const int32_t* rel,
                                        const float* w, const float* prior, const float* table, const float* ins,
                                        const void* grad_out, int64_t grad_row_stride, int64_t grad_col0,
                                        int64_t seg_stride, float* grad_table, float* grad_ins, float* grad_prior,
                                        int B, int N, int D, int I, int64_t F, uint32_t io, void* stream_) {
  return gr::agg_backward(__func__, false, rowptr, src, rel, nullptr, w, prior, table, ins, grad_out, grad_row_stride,
                          grad_col0, seg_stride, grad_table, grad_ins, grad_prior, B, N, D, I, F, nullptr, nullptr,
                          nullptr, nullptr, nullptr, 0, nullptr, 0, io, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_aggregate_backward(const int32_t* rowptr, const int32_t* src, const int32_t* rel, const float* w,
                                     const float* prior, const float* table, const float* ins, const float* grad_out,
                                     int64_t grad_row_stride, int64_t grad_col0, int64_t seg_stride, float* grad_table,
                                     float* grad_ins, float* grad_prior, int B, int N, int D, int I, int64_t F,
                                     void* stream_) {
  return gr_aggregate_backward_ex(rowptr, src, rel, w, prior, table, ins, grad_out, grad_row_stride, grad_col0,
                                  seg_stride, grad_table, grad_ins, grad_prior, B, N, D, I, F, 0u, stream_);
}

// Backward of gr_type_layer (TypeLayer.forward, gnn/modules/layer_init.py:46-57):
//     out[n] = relu( sum_{tail CSR of n} w_e table[rel_e] + sum_{head CSR of n} w_e table[rel_e] )
//     grad_table[r] += sum_{tail CSR rows n} w_e Gm[n] + sum_{head CSR rows n} w_e Gm[n],   Gm = G * [out > 0]
// One warp per row holds Gm[n] in registers and walks both of the row's CSR lists; runs of equal relations are merged
// into one coefficient, then added to the R1 table rows with fp32 atomics (not bit-reproducible).
namespace gr {
namespace {

template <int NC, typename T>
__global__ void __launch_bounds__(kBwdThreads) type_bwd_kernel(const int32_t* __restrict__ rowptr_t,
                                                               const int32_t* __restrict__ rel_t,
                                                               const float* __restrict__ w_t,
                                                               const int32_t* __restrict__ rowptr_h,
                                                               const int32_t* __restrict__ rel_h,
                                                               const float* __restrict__ w_h,
                                                               const T* __restrict__ grad, int64_t ld_grad,
                                                               const T* __restrict__ out, int64_t ld_out,
                                                               float* __restrict__ gtable, int64_t ld_gt, int64_t Nt,
                                                               int D) {
  const int lane = threadIdx.x & 31;
  const int64_t n = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= Nt) return;
  const int bt = rowptr_t[n], et = rowptr_t[n + 1], bh = rowptr_h[n], eh = rowptr_h[n + 1];
  if (bt == et && bh == eh) return;
  float g[NC];
  bool any = false;
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const int c = lane + 32 * k;
    g[k] = (c < D && ldg_node(out + n * ld_out + c) > 0.f) ? ldg_node(grad + n * ld_grad + c) : 0.f;
    any |= g[k] != 0.f;
  }
  if (!__any_sync(0xffffffffu, any)) return;
  int cur = -1;
  float cw = 0.f;
  auto flush = [&]() {
    if (cur < 0 || cw == 0.f) return;
    float* row = gtable + (int64_t)cur * ld_gt;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int c = lane + 32 * k;
      if (c < D && g[k] != 0.f) atomicAdd(row + c, cw * g[k]);
    }
  };
  for (int i = 0, len = (et - bt) + (eh - bh); i < len; ++i) {
    const bool tail = i < et - bt;
    const int e = tail ? bt + i : bh + (i - (et - bt));
    const int r = __ldg((tail ? rel_t : rel_h) + e);
    const float* w = tail ? w_t : w_h;
    const float we = w ? __ldg(w + e) : 1.f;
    if (r != cur) {
      flush();
      cur = r;
      cw = 0.f;
    }
    cw += we;
  }
  flush();
}

}  // namespace
}  // namespace gr

// Deterministic variant of gr_type_layer_backward: two fixed-window segmented sums (common.cuh) over the relation
// indexes of the tail CSR and then of the head CSR.  Entry i -> CSR slot e of relation rel[e], row n = row_of[e]:
//     grad_table[r] = (grad_table[r] + sum_{tail-CSR slots of r} w_e Gm[n]) + sum_{head-CSR slots of r} w_e Gm[n]
// each sum in slot order, each term __fmul_rn(w_e, Gm[n]).
namespace gr {
namespace {

template <int NC, typename T>
__global__ void __launch_bounds__(kBwdThreads) type_bwd_det_kernel(const int32_t* __restrict__ rix_ptr,
                                                                   const int32_t* __restrict__ rix_slot,
                                                                   const int32_t* __restrict__ rel,
                                                                   const float* __restrict__ w,
                                                                   const int32_t* __restrict__ row_of,
                                                                   const T* __restrict__ grad, int64_t ld_grad,
                                                                   const T* __restrict__ out, int64_t ld_out,
                                                                   float* __restrict__ gtable, int64_t ld_gt,
                                                                   float* __restrict__ part, int64_t R1, int D) {
  const int lane = threadIdx.x & 31;
  const int64_t win = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t L = rix_ptr[R1];
  const int64_t a = win * kRelWin, bnd = min(L, a + kRelWin);
  if (a >= L) return;
  auto seg_of = [&](int64_t i) { return (int64_t)rel[rix_slot[i]]; };
  float acc[NC];
  int64_t cur = -1;
  bool first = true;
  auto flush = [&]() {
    const int slot = segwin_slot(a, bnd, L, cur, first, seg_of);
    segwin_store<NC>(acc, slot, part + (win * 2 + (slot > 0)) * D, gtable + cur * ld_gt, D);
    first = false;
  };
  for (int64_t i = a; i < bnd; ++i) {
    const int e = rix_slot[i];
    const int64_t r = rel[e], n = row_of[e];
    if (r != cur) {
      if (cur >= 0) flush();
      cur = r;
#pragma unroll
      for (int k = 0; k < NC; ++k) acc[k] = 0.f;
    }
    const float we = w ? __ldg(w + e) : 1.f;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const int c = lane + 32 * k;
      if (c < D) {
        const float gm = ldg_node(out + n * ld_out + c) > 0.f ? ldg_node(grad + n * ld_grad + c) : 0.f;
        acc[k] = __fadd_rn(acc[k], __fmul_rn(we, gm));
      }
    }
  }
  flush();
}

// one direction (tail / head CSR) of the TypeLayer's edges: the row pointers for the atomic kernel, the relation
// index (rix_ptr / rix_slot / row_of) for the deterministic one
struct TypeDir {
  const int32_t *rowptr, *rel;
  const float* w;
  const int32_t *rix_ptr, *rix_slot, *row_of;
};

// gr_type_layer_backward_ex (det == false: B, N and the row pointers) and gr_type_layer_backward_det_ex (det == true:
// R1, the relation indexes and the workspace); `fn` is the entry point the argument checks report.
int type_layer_backward(const char* fn, bool det, const TypeDir& t, const TypeDir& h, const void* grad_out,
                        int64_t ld_grad, const void* out, int64_t ld_out, float* grad_table, int64_t ld_gtable, int B,
                        int N, int64_t R1, int D, int64_t F, void* workspace, size_t workspace_bytes, uint32_t io,
                        cudaStream_t stream) {
  if (int rc = check_io(fn, io)) return rc;
  GR_CHECK_ARG_AS(fn, (det ? R1 > 0 : B > 0 && N > 0) && D > 0 && D <= 512 && F >= 0, "bad sizes (need 0 < D <= 512)");
  GR_CHECK_ARG_AS(fn, (det ? t.rix_ptr && h.rix_ptr : t.rowptr && h.rowptr) && grad_out && out && grad_table,
                  "null pointer");
  GR_CHECK_ARG_AS(fn, F == 0 || (t.rel && h.rel && (!det || (t.rix_slot && t.row_of && h.rix_slot && h.row_of))),
                  "null edge arrays");
  GR_CHECK_ARG_AS(fn, ld_grad >= D && ld_out >= D && ld_gtable >= D, "leading dimension smaller than D");
  if (F == 0) return GR_OK;
  if (!det) {
    const int64_t Nt = (int64_t)B * N;
    const int grid = (int)ceil_div(Nt, kBwdThreads / 32);
    with_nc(D, [&](auto nc) {
      with_node_type(io, [&](auto tag) {
        using T = typename decltype(tag)::type;
        type_bwd_kernel<decltype(nc)::value, T><<<grid, kBwdThreads, 0, stream>>>(
            t.rowptr, t.rel, t.w, h.rowptr, h.rel, h.w, static_cast<const T*>(grad_out), ld_grad,
            static_cast<const T*>(out), ld_out, grad_table, ld_gtable, Nt, D);
      });
    });
    GR_CHECK_LAUNCH_AS(fn);
    return GR_OK;
  }
  const size_t need = segwin_part_bytes(F, D, kRelWin);
  if (int rc = check_workspace("gr_type_layer_backward_det", workspace, workspace_bytes, need)) return rc;
  float* part = reinterpret_cast<float*>(workspace);
  const int grid = (int)ceil_div(ceil_div(F, kRelWin), kBwdThreads / 32);
  for (const TypeDir* dir : {&t, &h}) {
    with_nc(D, [&](auto nc) {
      with_node_type(io, [&](auto tag) {
        using T = typename decltype(tag)::type;
        type_bwd_det_kernel<decltype(nc)::value, T><<<grid, kBwdThreads, 0, stream>>>(
            dir->rix_ptr, dir->rix_slot, dir->rel, dir->w, dir->row_of, static_cast<const T*>(grad_out), ld_grad,
            static_cast<const T*>(out), ld_out, grad_table, ld_gtable, part, R1, D);
      });
    });
    GR_CHECK_LAUNCH_AS(fn);
    segwin_combine_kernel<kRelWin><<<(int)ceil_div(R1 * D, 256), 256, 0, stream>>>(part, D, dir->rix_ptr, 0, R1,
                                                                                   grad_table, ld_gtable);
    GR_CHECK_LAUNCH_AS(fn);
  }
  return GR_OK;
}

}  // namespace
}  // namespace gr

extern "C" int gr_type_layer_backward_ex(const int32_t* rowptr_t, const int32_t* rel_t, const float* w_t,
                                         const int32_t* rowptr_h, const int32_t* rel_h, const float* w_h,
                                         const void* grad_out, int64_t ld_grad, const void* out, int64_t ld_out,
                                         float* grad_table, int64_t ld_gtable, int B, int N, int D, int64_t F,
                                         uint32_t io, void* stream_) {
  return gr::type_layer_backward(__func__, false, {rowptr_t, rel_t, w_t}, {rowptr_h, rel_h, w_h}, grad_out, ld_grad,
                                 out, ld_out, grad_table, ld_gtable, B, N, 0, D, F, nullptr, 0, io,
                                 reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_type_layer_backward(const int32_t* rowptr_t, const int32_t* rel_t, const float* w_t,
                                      const int32_t* rowptr_h, const int32_t* rel_h, const float* w_h,
                                      const float* grad_out, int64_t ld_grad, const float* out, int64_t ld_out,
                                      float* grad_table, int64_t ld_gtable, int B, int N, int D, int64_t F,
                                      void* stream_) {
  return gr_type_layer_backward_ex(rowptr_t, rel_t, w_t, rowptr_h, rel_h, w_h, grad_out, ld_grad, out, ld_out,
                                   grad_table, ld_gtable, B, N, D, F, 0u, stream_);
}

extern "C" size_t gr_type_layer_backward_det_workspace_bytes(int64_t F, int D) {
  if (F < 0 || D <= 0) return 0;
  return gr::segwin_part_bytes(F, D, gr::kRelWin);
}

extern "C" int gr_type_layer_backward_det_ex(const int32_t* rel_t, const float* w_t, const int32_t* rix_ptr_t,
                                             const int32_t* rix_slot_t, const int32_t* row_of_t, const int32_t* rel_h,
                                             const float* w_h, const int32_t* rix_ptr_h, const int32_t* rix_slot_h,
                                             const int32_t* row_of_h, const void* grad_out, int64_t ld_grad,
                                             const void* out, int64_t ld_out, float* grad_table, int64_t ld_gtable,
                                             int64_t R1, int D, int64_t F, void* workspace, size_t workspace_bytes,
                                             uint32_t io, void* stream_) {
  return gr::type_layer_backward(__func__, true, {nullptr, rel_t, w_t, rix_ptr_t, rix_slot_t, row_of_t},
                                 {nullptr, rel_h, w_h, rix_ptr_h, rix_slot_h, row_of_h}, grad_out, ld_grad, out, ld_out,
                                 grad_table, ld_gtable, 0, 0, R1, D, F, workspace, workspace_bytes, io,
                                 reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_type_layer_backward_det(const int32_t* rel_t, const float* w_t, const int32_t* rix_ptr_t,
                                          const int32_t* rix_slot_t, const int32_t* row_of_t, const int32_t* rel_h,
                                          const float* w_h, const int32_t* rix_ptr_h, const int32_t* rix_slot_h,
                                          const int32_t* row_of_h, const float* grad_out, int64_t ld_grad,
                                          const float* out, int64_t ld_out, float* grad_table, int64_t ld_gtable,
                                          int64_t R1, int D, int64_t F, void* workspace, size_t workspace_bytes,
                                          void* stream_) {
  return gr_type_layer_backward_det_ex(rel_t, w_t, rix_ptr_t, rix_slot_t, row_of_t, rel_h, w_h, rix_ptr_h, rix_slot_h,
                                       row_of_h, grad_out, ld_grad, out, ld_out, grad_table, ld_gtable, R1, D, F,
                                       workspace, workspace_bytes, 0u, stream_);
}
