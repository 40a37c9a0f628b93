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
// One CTA each; integer and copy work only, no atomics, so the records do not depend on scheduling.
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
