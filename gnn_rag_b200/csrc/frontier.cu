// Sparse-prior fast path for one ReaRev GNN layer (SURVEY.md 7, hard part 3: degenerate priors).
//
// In the first GNN layer of every iteration the prior is the seed distribution (reference
// gnn/models/ReaRev/rearev.py:208: `self.curr_dist = current_dist`), i.e. non-zero on a handful of nodes.  A
// destination row whose in-edges (either direction) all come from zero-prior nodes receives EXACTLY zero
// neighbour messages (relu(x) * 0 = 0), so for those rows
//     h_new = relu(e2e_k([h | 0 ... 0])) = relu(W[:, :D] h + b)
// which the tensor-core GEMM computes with K = one segment instead of 2I+1 -- no 410 MB of zeros written by the
// aggregation kernel and re-read by the GEMM.  The remaining "frontier" rows (those with at least one in-edge
// from a node with non-zero prior) are recomputed in full here and overwrite the GEMM's result:
//     gr_frontier_rows   : list the frontier rows (exact for ANY prior; just slower when the prior is dense)
//     gr_frontier_fixup  : per frontier row: both directions' aggregation for every instruction (same edge order
//                          and arithmetic as aggregate.cu), then the full e2e linear + relu + score dot in fp32,
//                          written to the next layer's bf16 planes / fp32 h / score dots.
// Mirrors ReasonGNNLayer.forward (gnn/modules/kg_reasoning/reasongnn.py:134-174) restricted to those rows.
#include <cuda_bf16.h>

#include "common.cuh"

namespace gr {
namespace {

constexpr int kFixRows = 8;        // frontier rows per CTA iteration (one warp per row in phase A)
constexpr int kFixThreads = 1024;  // 32 warps: phase B is latency-bound on the weight stream, so more warps = more loads in flight

// one thread per destination row: does any in-edge carry prior mass?
__global__ void frontier_rows_kernel(const int32_t* __restrict__ rp_t, const int32_t* __restrict__ src_t,
                                     const int32_t* __restrict__ rp_h, const int32_t* __restrict__ src_h,
                                     const float* __restrict__ prior, int64_t Nt, int32_t* __restrict__ list,
                                     int32_t* __restrict__ count) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool hit = false;
  if (row < Nt) {
    for (int e = rp_t[row]; e < rp_t[row + 1] && !hit; ++e) hit = prior[src_t[e]] != 0.f;
    for (int e = rp_h[row]; e < rp_h[row + 1] && !hit; ++e) hit = prior[src_h[e]] != 0.f;
  }
  // warp-aggregated append (order inside the list is irrelevant: rows are processed independently)
  const unsigned bal = __ballot_sync(0xffffffffu, hit);
  if (bal) {
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == 0) base = atomicAdd(count, __popc(bal));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (hit) list[base + __popc(bal & ((1u << lane) - 1))] = (int32_t)row;
  }
}

struct FixParams {
  const int32_t *rp_t, *src_t, *rel_t, *rp_h, *src_h, *rel_h;
  const float *w_t, *w_h;            // optional edge weights (normalized_gnn)
  const float* prior;
  const float *table_fwd, *table_inv; // [R1, D]
  const float* ins;                   // [B, I, D]
  const __nv_bfloat16 *cur_hi, *cur_lo;   // current planes (h in columns [0, D))
  int64_t ld_cur;
  const float* W;                     // [D, (2I+1)*D] torch Linear weight, row stride ldw
  int64_t ldw;
  const float *bias, *w_score;
  __nv_bfloat16 *nxt_hi, *nxt_lo;     // next planes: h_new written to columns [0, D)
  int64_t ld_nxt;
  float* h32;                         // optional fp32 h_new [Nt, D]
  float* dots;                        // optional [2*Nt]
  const int32_t *list, *count;
  int N, D, I;
  int64_t Nt;
};

template <bool V2>   // V2: Kd and ldw even, W 8-byte aligned -> each lane owns k pairs (float2 weight / x loads)
__global__ void __launch_bounds__(kFixThreads)
frontier_fixup_kernel(const FixParams p) {
  extern __shared__ __align__(16) float sx[];                  // [kFixRows][Kd]  layer input rows, fp32
  __shared__ float s_dot[kFixThreads / 32][kFixRows];
  __shared__ float s_cf[kFixThreads / 32][32];   // per-warp staged edge coefficients / relation ids
  __shared__ int s_ro[kFixThreads / 32][32];
  const int D = p.D, I = p.I, Kd = (2 * I + 1) * D;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int total = *p.count;
  for (int base = blockIdx.x * kFixRows; base < total; base += gridDim.x * kFixRows) {
    const int nr = min(kFixRows, total - base);
    // ---------------- phase A: warps 0-15 = (row, direction) aggregation, warps 16-23 = the row's h ----------
    if (warp >= 16 && warp < 16 + nr) {
      const int64_t row = p.list[base + warp - 16];
      float* x = sx + (size_t)(warp - 16) * Kd;
      for (int c = lane; c < D; c += 32)
        x[c] = __bfloat162float(p.cur_hi[row * p.ld_cur + c]) + __bfloat162float(p.cur_lo[row * p.ld_cur + c]);
    } else if (warp < 16 && (warp & 7) < nr) {
      const int r = warp & 7, d = warp >> 3;
      const int64_t row = p.list[base + r];
      const int b = (int)(row / p.N);
      float* x = sx + (size_t)r * Kd;
      const int32_t* rp = d ? p.rp_h : p.rp_t;
      const int32_t* src = d ? p.src_h : p.src_t;
      const int32_t* rel = d ? p.rel_h : p.rel_t;
      const float* wgt = d ? p.w_h : p.w_t;
      const float* table = d ? p.table_inv : p.table_fwd;
      const int beg = rp[row], end = rp[row + 1];
      for (int c0 = 0; c0 < D; c0 += 256) {         // 8 columns per lane held in registers
        float A[8], S[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) A[i] = S[i] = 0.f;
        for (int e0 = beg; e0 < end; e0 += 32) {
          // lanes fetch 32 edges' (coefficient, relation) in parallel: one latency per 32 edges, not per edge
          const int e = e0 + lane;
          float cf = 0.f;
          int ro = 0;
          if (e < end) {
            const float w = wgt ? wgt[e] : 1.f;
            cf = w * (w * p.prior[src[e]]);
            ro = rel[e];
          }
          __syncwarp();
          s_cf[warp][lane] = cf;
          s_ro[warp][lane] = ro;
          __syncwarp();
          const int cnt = min(32, end - e0);
          for (int q = 0; q < cnt; ++q) {           // edge order as in aggregate.cu; zero-prior edges add 0
            const float cq = s_cf[warp][q];
            if (cq == 0.f) continue;
            const float* tr = table + (int64_t)s_ro[warp][q] * D + c0 + lane;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              if (c0 + lane + 32 * i < D) {
                const float v = __ldg(tr + 32 * i);
                S[i] = fmaf(cq, v, S[i]);
                A[i] = fmaf(cq, fmaxf(v, 0.f), A[i]);
              }
            }
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c = c0 + lane + 32 * i;
          if (c < D) {
            const float T = fmaf(S[i], -1.f, A[i]);
            for (int j = 0; j < I; ++j) {
              const float xi = __ldg(p.ins + ((int64_t)b * I + j) * D + c);
              const float xp = fmaxf(xi, 0.f), xn = fmaxf(-xi, 0.f);
              x[(1 + 2 * j + d) * D + c] = fmaf(xn, T, xp * A[i]);
            }
          }
        }
      }
    }
    __syncthreads();
    // ---------------- phase B: out[r][n] = relu(b[n] + sum_k W[n][k] x[r][k]) ---------------------------------
    // warp w owns 2 output columns per pass (n = 2*(w + 32*pass) + t); lane owns k pairs; 16 weight values in
    // flight per lane per round.
    constexpr int kNT = 2, kU = 4, kKL = V2 ? 2 : 1;   // k values per lane per load
    float dotacc[kFixRows];
#pragma unroll
    for (int r = 0; r < kFixRows; ++r) dotacc[r] = 0.f;
    for (int n0 = warp * kNT; n0 < D; n0 += (kFixThreads / 32) * kNT) {
      float acc[kNT][kFixRows];
#pragma unroll
      for (int t = 0; t < kNT; ++t)
#pragma unroll
        for (int r = 0; r < kFixRows; ++r) acc[t][r] = 0.f;
      const float* wrow[kNT];
#pragma unroll
      for (int t = 0; t < kNT; ++t) wrow[t] = p.W + (int64_t)min(n0 + t, D - 1) * p.ldw;
      for (int k0 = 0; k0 < Kd; k0 += 32 * kKL * kU) {
        float wv[kNT][kU][kKL];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const int k = k0 + (u * 32 + lane) * kKL;
#pragma unroll
          for (int t = 0; t < kNT; ++t) {
            if constexpr (V2) {
              const float2 w2 = k < Kd ? __ldg(reinterpret_cast<const float2*>(wrow[t] + k)) : make_float2(0.f, 0.f);
              wv[t][u][0] = w2.x;
              wv[t][u][1] = w2.y;
            } else {
              wv[t][u][0] = k < Kd ? __ldg(wrow[t] + k) : 0.f;
            }
          }
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const int k = min(k0 + (u * 32 + lane) * kKL, Kd - kKL);
#pragma unroll
          for (int r = 0; r < kFixRows; ++r) {
            if constexpr (V2) {
              const float2 xv = *reinterpret_cast<const float2*>(sx + (size_t)r * Kd + k);
#pragma unroll
              for (int t = 0; t < kNT; ++t) acc[t][r] = fmaf(wv[t][u][1], xv.y, fmaf(wv[t][u][0], xv.x, acc[t][r]));
            } else {
              const float xv = sx[(size_t)r * Kd + k];
#pragma unroll
              for (int t = 0; t < kNT; ++t) acc[t][r] = fmaf(wv[t][u][0], xv, acc[t][r]);
            }
          }
        }
      }
#pragma unroll
      for (int t = 0; t < kNT; ++t)
#pragma unroll
        for (int r = 0; r < kFixRows; ++r) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) acc[t][r] += __shfl_xor_sync(0xffffffffu, acc[t][r], o);
        }
      if (lane == 0) {
#pragma unroll
        for (int t = 0; t < kNT; ++t) {
          const int n = n0 + t;
          if (n < D) {
            const float bn = p.bias ? p.bias[n] : 0.f, wsn = p.w_score ? p.w_score[n] : 0.f;
#pragma unroll
            for (int r = 0; r < kFixRows; ++r) {
              if (r < nr) {
                const float y = fmaxf(acc[t][r] + bn, 0.f);
                const int64_t row = p.list[base + r];
                const __nv_bfloat16 h = __float2bfloat16_rn(y);
                p.nxt_hi[row * p.ld_nxt + n] = h;
                p.nxt_lo[row * p.ld_nxt + n] = __float2bfloat16_rn(y - __bfloat162float(h));
                if (p.h32) p.h32[row * D + n] = y;
                dotacc[r] = fmaf(y, wsn, dotacc[r]);
              }
            }
          }
        }
      }
    }
    if (p.dots) {
      if (lane == 0) {
#pragma unroll
        for (int r = 0; r < kFixRows; ++r) s_dot[warp][r] = dotacc[r];
      }
      __syncthreads();
      if (threadIdx.x < nr) {
        float s = 0.f;
        for (int w = 0; w < kFixThreads / 32; ++w) s += s_dot[w][threadIdx.x];   // fixed order: deterministic
        const int64_t row = p.list[base + threadIdx.x];
        p.dots[row] = s;
        p.dots[p.Nt + row] = 0.f;
      }
    }
    __syncthreads();
  }
}

}  // namespace
}  // namespace gr

extern "C" int gr_frontier_rows(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rowptr_h,
                                const int32_t* src_h, const float* prior, int64_t Nt, int32_t* list,
                                int32_t* count, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(rowptr_t && rowptr_h && prior && list && count && Nt > 0, "null pointer / bad size");
  GR_CHECK_CUDA(cudaMemsetAsync(count, 0, sizeof(int32_t), stream));
  frontier_rows_kernel<<<(unsigned)ceil_div(Nt, 256), 256, 0, stream>>>(rowptr_t, src_t, rowptr_h, src_h, prior,
                                                                         Nt, list, count);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_frontier_fixup(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                                 const float* w_t, const int32_t* rowptr_h, const int32_t* src_h,
                                 const int32_t* rel_h, const float* w_h, const float* prior,
                                 const float* table_fwd, const float* table_inv, const float* ins,
                                 const void* cur_hi, const void* cur_lo, int64_t ld_cur, const float* W,
                                 int64_t ldw, const float* bias, const float* w_score, void* nxt_hi,
                                 void* nxt_lo, int64_t ld_nxt, float* h32, float* dots, const int32_t* list,
                                 const int32_t* count, int B, int N, int D, int I, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(rowptr_t && rowptr_h && prior && table_fwd && table_inv && ins && cur_hi && cur_lo && W &&
                   nxt_hi && nxt_lo && list && count,
               "null pointer");
  GR_CHECK_ARG(B > 0 && N > 0 && D > 0 && I > 0 && ldw >= (2 * I + 1) * (int64_t)D, "bad shape");
  const size_t smem = (size_t)kFixRows * (2 * I + 1) * D * sizeof(float);
  GR_CHECK_ARG(smem <= 200 * 1024, "(2I+1)*D too large for the fix-up kernel's shared memory");
  if (int rc = opt_in_smem<frontier_fixup_kernel<true>>(__func__, 200 * 1024)) return rc;
  if (int rc = opt_in_smem<frontier_fixup_kernel<false>>(__func__, 200 * 1024)) return rc;
  FixParams p{};
  p.rp_t = rowptr_t; p.src_t = src_t; p.rel_t = rel_t; p.rp_h = rowptr_h; p.src_h = src_h; p.rel_h = rel_h;
  p.w_t = w_t; p.w_h = w_h; p.prior = prior; p.table_fwd = table_fwd; p.table_inv = table_inv; p.ins = ins;
  p.cur_hi = reinterpret_cast<const __nv_bfloat16*>(cur_hi);
  p.cur_lo = reinterpret_cast<const __nv_bfloat16*>(cur_lo);
  p.ld_cur = ld_cur; p.W = W; p.ldw = ldw; p.bias = bias; p.w_score = w_score;
  p.nxt_hi = reinterpret_cast<__nv_bfloat16*>(nxt_hi); p.nxt_lo = reinterpret_cast<__nv_bfloat16*>(nxt_lo);
  p.ld_nxt = ld_nxt; p.h32 = h32; p.dots = dots; p.list = list; p.count = count;
  p.N = N; p.D = D; p.I = I; p.Nt = (int64_t)B * N;
  const bool v2 = ((2 * I + 1) * D) % 2 == 0 && ldw % 2 == 0 && (reinterpret_cast<uintptr_t>(W) & 7) == 0;
  if (v2)
    frontier_fixup_kernel<true><<<2 * sm_count(), kFixThreads, smem, stream>>>(p);
  else
    frontier_fixup_kernel<false><<<2 * sm_count(), kFixThreads, smem, stream>>>(p);
  GR_CHECK_LAUNCH();
  return GR_OK;
}
