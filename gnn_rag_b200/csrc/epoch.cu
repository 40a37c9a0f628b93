// Step bookkeeping of a training epoch replayed as CUDA graphs (graphed.GraphedTrainStep.start_epoch).
//
// The only input that changes from one replay to the next is a device cursor, the index of the step.  The epoch's
// question order (the loader's `batches`) and its per-question kept counts are uploaded once per epoch.
//
//   gr_epoch_step_begin   at the head of the graph: the step's question ids, gather rows and kept counts, the live
//                         fact count (`nfacts` of the CSR build) and the live kept total, from the cursor.
//   gr_epoch_graft_begin  right after it, for GraftNet: the step's graft kept counts and the live graft count
//                         (`live` of gr_graft_stage), from the ids gr_epoch_step_begin wrote.
//   gr_epoch_step_record  at the tail: loss, gradient norm, fact-order seed, hit@1 and F1 stored at the cursor, the
//                         step's status words OR-ed into the epoch's, the cursor advanced.
//
// An evaluation epoch (graphed.GraphedStep.start_eval) shares the head kernel and ends with
//   gr_eval_step_record   the evaluator's precision / recall / F1 / hit / EM of every question of the step against its
//                         answer list, and its ranked candidates appended to the split's flat records.
//
// One CTA each; integer and copy work only (gr_eval_step_record: plus float64 divisions), no atomics, so the records
// do not depend on scheduling.
#include <limits.h>

#include "common.cuh"

namespace gr {
namespace {

constexpr int kEpochThreads = 256;

// sum over the block of one int64 per thread (valid in every thread); s_red holds 33 entries
__device__ __forceinline__ int64_t epoch_block_sum(int64_t v, int64_t* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();                                   // s_red may still be read from a previous call
  if (lane_id() == 0) s_red[warp_id()] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w];
    s_red[32] = t;
  }
  __syncthreads();
  return s_red[32];
}

__global__ void __launch_bounds__(kEpochThreads)
epoch_step_begin_kernel(const int64_t* __restrict__ cursor, const int64_t* __restrict__ order, int64_t num_data,
                        int64_t batch_size, int B, const int64_t* __restrict__ kept_table,
                        const int64_t* __restrict__ q_off, const int32_t* __restrict__ q_ents, int64_t num_q,
                        int use_self_loop, int64_t capacity, int64_t* __restrict__ ids, int64_t* __restrict__ rows,
                        int64_t* __restrict__ kept, int32_t* __restrict__ nfacts, int64_t* __restrict__ kept_total,
                        int32_t* __restrict__ status) {
  __shared__ int64_t s_red[33];
  const int64_t c = *cursor;
  int64_t sum_k = 0, sum_f = 0, bad = 0;
  for (int j = threadIdx.x; j < B; j += blockDim.x) {
    const int64_t p = c * batch_size + j;
    const int64_t id = (c >= 0 && p < num_data) ? order[p] : -1;
    const bool ok = id >= 0 && id < num_q;
    const int64_t n = ok ? q_off[id + 1] - q_off[id] : 0;
    const int64_t k = kept_table && ok ? min(max(kept_table[id], (int64_t)0), n) : n;
    const int64_t e = ok && use_self_loop ? (int64_t)q_ents[id] : 0;
    ids[j] = id;
    rows[j] = ok ? id : 0;
    kept[j] = k;
    sum_k += k;
    sum_f += k + e;
    bad += ok ? 0 : 1;
  }
  sum_k = epoch_block_sum(sum_k, s_red);
  sum_f = epoch_block_sum(sum_f, s_red);
  bad = epoch_block_sum(bad, s_red);
  if (threadIdx.x == 0) {
    *nfacts = (int32_t)min(sum_f, capacity);
    *kept_total = sum_k;
    *status = (bad ? 1 : 0) | (sum_f > capacity ? 2 : 0);
  }
}

__global__ void __launch_bounds__(kEpochThreads)
epoch_graft_begin_kernel(const int64_t* __restrict__ ids, int B, const int64_t* __restrict__ kept_table,
                         const int64_t* __restrict__ g_off, int64_t num_q, int64_t capacity,
                         int64_t* __restrict__ kept_g, int32_t* __restrict__ graft_live, int32_t* __restrict__ status) {
  __shared__ int64_t s_red[33];
  int64_t sum_g = 0;
  for (int j = threadIdx.x; j < B; j += blockDim.x) {
    const int64_t id = ids[j];
    const bool ok = id >= 0 && id < num_q;
    const int64_t n = ok ? g_off[id + 1] - g_off[id] : 0;
    const int64_t k = kept_table && ok ? min(max(kept_table[id], (int64_t)0), n) : n;
    kept_g[j] = k;
    sum_g += k;
  }
  sum_g = epoch_block_sum(sum_g, s_red);
  if (threadIdx.x == 0) {
    const int32_t live = (int32_t)min(sum_g, capacity);
    graft_live[0] = live;
    graft_live[1] = live;
    *status = sum_g > capacity ? 2 : 0;
  }
}

__global__ void __launch_bounds__(kEpochThreads)
epoch_step_record_kernel(int64_t* __restrict__ cursor, int64_t steps, int64_t batch_size, int B, int64_t num_data,
                         const float* __restrict__ loss, const float* __restrict__ grad_norm,
                         const int64_t* __restrict__ seed, const float* __restrict__ h1, const float* __restrict__ f1,
                         const int32_t* __restrict__ split_status, const int32_t* __restrict__ csr_status,
                         float* __restrict__ losses, float* __restrict__ grad_norms, int64_t* __restrict__ seeds,
                         float* __restrict__ h1_all, float* __restrict__ f1_all, int32_t* __restrict__ epoch_status) {
  const int64_t c = *cursor;
  const bool in_epoch = c >= 0 && c < steps;
  if (in_epoch) {
    const int64_t p0 = c * batch_size;
    for (int j = threadIdx.x; j < B; j += blockDim.x) {
      if (p0 + j < num_data) {
        h1_all[p0 + j] = h1[j];
        f1_all[p0 + j] = f1[j];
      }
    }
  }
  __syncthreads();                                   // every thread has read the cursor
  if (threadIdx.x == 0) {
    if (in_epoch) {
      losses[c] = *loss;
      if (grad_norm) grad_norms[c] = *grad_norm;
      if (seed) seeds[c] = *seed;
    }
    epoch_status[0] |= *split_status | (in_epoch ? 0 : 2);
    epoch_status[1] |= *csr_status;
    *cursor = c + 1;
  }
}

// e in the ascending run a[lo, hi)
__device__ __forceinline__ bool eval_member(const int64_t* __restrict__ a, int64_t lo, int64_t hi, int64_t e) {
  int64_t l = lo, h = hi;
  while (l < h) {
    const int64_t mid = l + ((h - l) >> 1);
    if (a[mid] < e) l = mid + 1; else h = mid;
  }
  return l < hi && a[l] == e;
}

// One warp per question: a question's candidates are read in rounds of kEvalUnroll per lane, their loads issued
// before any membership search, so each lane keeps several independent gathers in flight.
constexpr int kEvalThreads = 1024;
constexpr int kEvalUnroll = 4;

__global__ void __launch_bounds__(kEvalThreads)
eval_step_record_kernel(int64_t* __restrict__ cursor, int64_t steps, int64_t batch_size, int B, int64_t num_data,
                        int N, const int64_t* __restrict__ ids, const int64_t* __restrict__ local_entity,
                        const float* __restrict__ pred_dist, const int32_t* __restrict__ cand_idx,
                        const int32_t* __restrict__ cand_count, const int64_t* __restrict__ a_off,
                        const int64_t* __restrict__ a_ids, int64_t num_a, const int64_t* __restrict__ seed,
                        const int32_t* __restrict__ split_status, const int32_t* __restrict__ csr_status,
                        double* __restrict__ metrics, int8_t* __restrict__ cases, int32_t* __restrict__ counts,
                        int64_t* __restrict__ cand_off, int64_t* __restrict__ cand, int64_t capacity,
                        int64_t* __restrict__ cand_total, int64_t* __restrict__ seeds,
                        int32_t* __restrict__ eval_status) {
  constexpr int kWarps = kEvalThreads / 32;
  __shared__ int64_t s_warp[kWarps];
  __shared__ int64_t s_base;
  __shared__ int s_over;
  const int64_t c = *cursor;
  const bool in_epoch = c >= 0 && c < steps;
  const int64_t p0 = c * batch_size;
  const int lane = lane_id(), warp = warp_id();
  if (threadIdx.x == 0) {
    s_base = *cand_total;
    s_over = 0;
  }
  __syncthreads();
  if (in_epoch) {
    // 1. where each recorded question's candidates start: an exclusive scan of the counts, kEvalThreads at a time
    for (int j0 = 0; j0 < B; j0 += kEvalThreads) {
      const int j = j0 + threadIdx.x;
      const bool rec = j < B && p0 + j < num_data;
      const int64_t n = rec ? (int64_t)min(max(cand_count[j], 0), N) : 0;
      int64_t v = n;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
      }
      if (lane == 31) s_warp[warp] = v;
      __syncthreads();
      int64_t before = s_base;
      for (int w = 0; w < warp; ++w) before += s_warp[w];
      if (rec) cand_off[p0 + j] = before + v - n;
      __syncthreads();                               // every thread has read s_base and s_warp
      if (threadIdx.x == kEvalThreads - 1) s_base = before + v;
      __syncthreads();
    }
    // 2. one warp per question: membership of every candidate, the metrics, the candidate records
    for (int j = warp; j < B; j += kWarps) {
      const int64_t p = p0 + j;
      if (p >= num_data) continue;
      const int C = min(max(cand_count[j], 0), N);
      const int64_t id = ids[j];
      const bool ok = id >= 0 && id < num_a;
      const int64_t lo = ok ? a_off[id] : 0, hi = ok ? a_off[id + 1] : 0;
      const int64_t off = cand_off[p];
      const bool fits = off + C <= capacity;
      const int64_t* le = local_entity + (int64_t)j * N;
      const float* pd = pred_dist + (int64_t)j * N;
      const int32_t* ci = cand_idx + (int64_t)j * N;
      int correct = 0;
      for (int k0 = lane; k0 < C; k0 += 32 * kEvalUnroll) {
        int32_t li[kEvalUnroll];
        int64_t e[kEvalUnroll];
        float pr[kEvalUnroll];
#pragma unroll
        for (int u = 0; u < kEvalUnroll; ++u) li[u] = k0 + 32 * u < C ? ci[k0 + 32 * u] : 0;
#pragma unroll
        for (int u = 0; u < kEvalUnroll; ++u) {
          e[u] = le[li[u]];
          pr[u] = pd[li[u]];
        }
#pragma unroll
        for (int u = 0; u < kEvalUnroll; ++u) {
          const int k = k0 + 32 * u;
          if (k < C) {
            correct += eval_member(a_ids, lo, hi, e[u]) ? 1 : 0;
            if (fits) {
              int64_t* r = cand + 2 * (off + k);
              r[0] = e[u];
              reinterpret_cast<int32_t*>(r + 1)[0] = li[u];
              reinterpret_cast<int32_t*>(r + 1)[1] = __float_as_int(pr[u]);
            }
          }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) correct += __shfl_xor_sync(0xffffffffu, correct, o);
      if (lane == 0) {
        if (!fits) s_over = 1;
        // f1_and_hits (gnn/evaluate.py:51-67), each float64 operation rounded as python rounds it
        const int64_t A = hi - lo;
        const double hit = eval_member(a_ids, lo, hi, C > 0 ? le[ci[0]] : -1) ? 1.0 : 0.0;
        double pr, rc, f1, h, em;
        int8_t cs;
        if (A == 0) {
          pr = C == 0 ? 1.0 : 0.0; rc = 1.0; f1 = pr; h = 1.0; em = 1.0; cs = C == 0 ? 0 : 1;
        } else if (C == 0) {
          pr = 1.0; rc = 0.0; f1 = 0.0; h = hit; em = hit; cs = 2;
        } else {
          pr = __ddiv_rn((double)correct, (double)C);
          rc = __ddiv_rn((double)correct, (double)A);
          f1 = pr != 0.0 && rc != 0.0 ? __ddiv_rn(2.0, __dadd_rn(__ddiv_rn(1.0, pr), __ddiv_rn(1.0, rc))) : 0.0;
          h = hit; em = correct > 0 ? 1.0 : 0.0; cs = 3;
        }
        double* m = metrics + 5 * p;
        m[0] = pr; m[1] = rc; m[2] = f1; m[3] = h; m[4] = em;
        cases[p] = cs;
        counts[p] = C;
      }
    }
  }
  __syncthreads();                                   // every thread has read the cursor, s_over is final
  if (threadIdx.x == 0) {
    if (in_epoch) {
      *cand_total = s_base;
      if (seed) seeds[c] = *seed;
    }
    eval_status[0] |= *split_status | (in_epoch ? 0 : 2);
    eval_status[1] |= *csr_status;
    eval_status[2] |= s_over;
    *cursor = c + 1;
  }
}

}  // namespace
}  // namespace gr

extern "C" int gr_epoch_step_begin(const int64_t* cursor, const int64_t* order, int64_t num_data, int64_t batch_size,
                                   int B, const int64_t* kept_table, const int64_t* q_off, const int32_t* q_ents,
                                   int64_t num_q, int use_self_loop, int64_t capacity, int64_t* ids, int64_t* rows,
                                   int64_t* kept, int32_t* nfacts, int64_t* kept_total, int32_t* status,
                                   void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(cursor && order && q_off && q_ents, "null pointer");
  GR_CHECK_ARG(ids && rows && kept && nfacts && kept_total && status, "null output");
  GR_CHECK_ARG(B > 0 && batch_size >= B && num_data >= 0 && num_q >= 0,
               "need 0 < B <= batch_size, num_data >= 0 and num_q >= 0");
  GR_CHECK_ARG(capacity >= 0 && capacity <= INT_MAX, "capacity must be in [0, INT_MAX]");
  epoch_step_begin_kernel<<<1, kEpochThreads, 0, stream>>>(cursor, order, num_data, batch_size, B, kept_table, q_off,
                                                           q_ents, num_q, use_self_loop, capacity, ids, rows, kept,
                                                           nfacts, kept_total, status);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_epoch_graft_begin(const int64_t* ids, int B, const int64_t* kept_table, const int64_t* g_off,
                                    int64_t num_q, int64_t capacity, int64_t* kept_g, int32_t* graft_live,
                                    int32_t* status, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(ids && g_off, "null pointer");
  GR_CHECK_ARG(kept_g && graft_live && status, "null output");
  GR_CHECK_ARG(B > 0 && num_q >= 0, "need B > 0 and num_q >= 0");
  GR_CHECK_ARG(capacity >= 0 && capacity <= INT_MAX, "capacity must be in [0, INT_MAX]");
  epoch_graft_begin_kernel<<<1, kEpochThreads, 0, stream>>>(ids, B, kept_table, g_off, num_q, capacity, kept_g,
                                                            graft_live, status);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_epoch_step_record(int64_t* cursor, int64_t steps, int64_t batch_size, int B, int64_t num_data,
                                    const float* loss, const float* grad_norm, const int64_t* seed, const float* h1,
                                    const float* f1, const int32_t* split_status, const int32_t* csr_status,
                                    float* losses, float* grad_norms, int64_t* seeds, float* h1_all, float* f1_all,
                                    int32_t* epoch_status, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(cursor && loss && h1 && f1 && split_status && csr_status, "null pointer");
  GR_CHECK_ARG(losses && h1_all && f1_all && epoch_status, "null output");
  GR_CHECK_ARG(!grad_norm == !grad_norms && !seed == !seeds, "grad_norm / seed and their records go together");
  GR_CHECK_ARG(B > 0 && batch_size >= B && steps >= 0 && num_data >= 0,
               "need 0 < B <= batch_size, steps >= 0 and num_data >= 0");
  epoch_step_record_kernel<<<1, kEpochThreads, 0, stream>>>(cursor, steps, batch_size, B, num_data, loss, grad_norm,
                                                            seed, h1, f1, split_status, csr_status, losses,
                                                            grad_norms, seeds, h1_all, f1_all, epoch_status);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_eval_step_record(int64_t* cursor, int64_t steps, int64_t batch_size, int B, int64_t num_data,
                                   int64_t N, const int64_t* ids, const int64_t* local_entity, const float* pred_dist,
                                   const int32_t* cand_idx, const int32_t* cand_count, const int64_t* a_off,
                                   const int64_t* a_ids, int64_t num_a, const int64_t* seed,
                                   const int32_t* split_status, const int32_t* csr_status, double* metrics,
                                   int8_t* cases, int32_t* counts, int64_t* cand_off, int64_t* cand, int64_t capacity,
                                   int64_t* cand_total, int64_t* seeds, int32_t* eval_status, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(cursor && ids && local_entity && pred_dist && cand_idx && cand_count && a_off && a_ids &&
               split_status && csr_status, "null pointer");
  GR_CHECK_ARG(metrics && cases && counts && cand_off && cand && cand_total && eval_status, "null output");
  GR_CHECK_ARG(!seed == !seeds, "seed and its record go together");
  GR_CHECK_ARG(B > 0 && batch_size >= B && steps >= 0 && num_data >= 0 && num_a >= 0,
               "need 0 < B <= batch_size, steps >= 0, num_data >= 0 and num_a >= 0");
  GR_CHECK_ARG(N > 0 && N <= INT_MAX, "N must be in [1, INT_MAX]");
  GR_CHECK_ARG(capacity >= 0, "capacity must be >= 0");
  eval_step_record_kernel<<<1, kEvalThreads, 0, stream>>>(cursor, steps, batch_size, B, num_data, (int)N, ids,
                                                           local_entity, pred_dist, cand_idx, cand_count, a_off,
                                                           a_ids, num_a, seed, split_status, csr_status, metrics,
                                                           cases, counts, cand_off, cand, capacity, cand_total,
                                                           seeds, eval_status);
  GR_CHECK_LAUNCH();
  return GR_OK;
}
