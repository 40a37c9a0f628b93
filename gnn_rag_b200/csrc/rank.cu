// Candidate ranking: the "retrieved answer-node set" of the evaluator.
//
// Reference: Evaluator.evaluate (gnn/evaluate.py:156,188-209) builds candidate2prob by dropping seeds
// (s == 1 after the LongTensor cast at :173), pads (c == len(id2entity)) and p < (1-eps)/N; f1_and_hits
// (:25-50) sorts with python's STABLE sorted(..., reverse=True) (equal probabilities keep local-index
// order) and keeps the prefix up to and including the item where the running float64 sum exceeds eps.
// Here: one CTA per question, order-preserving compaction, a 64-bit key sort
// (key = desc_key(p) << 32 | local_index: ascending key == descending p, ascending index on ties), and the
// same sequential float64 running sum.  Integer/bit work end to end: bit-exact w.r.t. the reference
// given the same probabilities.
// Input domain: any fp32 p but NaN.  -0.0 ranks level with +0.0 and negative values rank below every other, as in
// python's sorted; they survive the (1-eps)/N cut only when eps >= 1 (e.g. eps = 1 to retrieve every candidate), and
// then the order is the whole output.  NaN is outside the contract: python's sorted has no order for NaN keys that
// could be restated.
#include <limits.h>
#include <math.h>

#include "common.cuh"

namespace gr {
namespace {

constexpr int kRankThreads = 512;
constexpr int kSmemKeys = 4096;

__device__ void bitonic_sort_u64(unsigned long long* a, int n) {
  // all-ascending bitonic network (virtual +inf padding): sorts arbitrary n
  for (int k = 2; (k >> 1) < n; k <<= 1) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      int l = i ^ (k - 1);
      if (l > i && l < n) {
        unsigned long long x = a[i], y = a[l];
        if (x > y) { a[i] = y; a[l] = x; }
      }
    }
    __syncthreads();
    for (int j = k >> 2; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        int l = i ^ j;
        if (l > i && l < n) {
          unsigned long long x = a[i], y = a[l];
          if (x > y) { a[i] = y; a[l] = x; }
        }
      }
      __syncthreads();
    }
  }
}

// 32-bit sort key of p: ascending key == descending p.  The standard order-preserving map of a float's bits (-0.0 made
// +0.0 first; a negative value gets all bits flipped, any other the sign bit set), inverted for descending order.
__device__ __forceinline__ unsigned desc_key(float p) {
  unsigned u = __float_as_uint(p);
  if (u == 0x80000000u) u = 0u;
  return ~((u & 0x80000000u) ? ~u : (u | 0x80000000u));
}

__device__ __forceinline__ float key_value(unsigned k) {   // inverse of desc_key (-0.0 comes back as +0.0)
  return __uint_as_float((k & 0x80000000u) ? k : ~(k | 0x80000000u));
}

__global__ void __launch_bounds__(kRankThreads)
rank_kernel(const float* __restrict__ dist, const int64_t* __restrict__ local_entity,
            const float* __restrict__ query_entities, int64_t pad_id, double eps, double ignore_prob,
            int32_t* __restrict__ cand_idx, int32_t* __restrict__ cand_count,
            int32_t* __restrict__ cand_total, int N, unsigned long long* __restrict__ ws, int exact_ok) {
  __shared__ unsigned long long s_keys[kSmemKeys];
  __shared__ int s_woff[kRankThreads / 32 + 1];
  __shared__ int s_base;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  constexpr int nw = kRankThreads / 32;
  const float* p = dist + (int64_t)b * N;
  const int64_t* le = local_entity + (int64_t)b * N;
  const float* qe = query_entities + (int64_t)b * N;
  unsigned long long* gkeys = ws + (int64_t)b * N;
  __shared__ int s_bad;      // a kept term > 1.0: not a probability -> no exactness argument, sequential sum
  if (tid == 0) { s_base = 0; s_bad = 0; }
  __syncthreads();
  // 1. order-preserving compaction of surviving candidates into gkeys
  for (int base = 0; base < N; base += kRankThreads) {
    int n = base + tid;
    bool keep = false;
    float pv = 0.f;
    if (n < N) {
      pv = p[n];
      bool is_seed = ((long long)qe[n]) == 1LL;          // evaluate.py:173,194
      bool is_pad = le[n] == pad_id;                      // :201
      bool small = (double)pv < ignore_prob;              // :203 (python float compare)
      keep = !is_seed && !is_pad && !small;
      if (keep && !(pv <= 1.0f)) s_bad = 1;
    }
    unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_woff[wid + 1] = __popc(bal);
    __syncthreads();
    if (tid == 0) {
      s_woff[0] = s_base;
      for (int i = 0; i < nw; ++i) s_woff[i + 1] += s_woff[i];
      s_base = s_woff[nw];
    }
    __syncthreads();
    if (keep) {
      int pos = s_woff[wid] + __popc(bal & ((1u << lane) - 1));
      gkeys[pos] = ((unsigned long long)desc_key(pv) << 32) | (unsigned)n;
    }
    __syncthreads();
  }
  const int total = s_base;
  __syncthreads();
  // 2. sort
  unsigned long long* keys = gkeys;
  if (total <= kSmemKeys) {
    for (int i = tid; i < total; i += kRankThreads) s_keys[i] = gkeys[i];
    __syncthreads();
    keys = s_keys;
  } else {
    __threadfence_block();
  }
  bitonic_sort_u64(keys, total);
  // 3. eps-mass prefix = first i with (sum_{k<=i} p_k in float64) > eps (f1_and_hits, evaluate.py:41-50).
  //    The reference adds sequentially in python floats (fp64).  Every surviving p_k is an fp32 value
  //    >= ignore_prob, so with exact_ok (host: 24 + ceil(log2(1/ignore_prob)) + 1 <= 53) every partial sum of
  //    any subset is exactly representable in fp64: the fp64 sum is ORDER-INDEPENDENT and a parallel scan is
  //    bit-identical to the sequential loop.  Otherwise fall back to the sequential loop.  exact_ok implies eps < 1,
  //    so ignore_prob > 0 and no zero or negative p is ever kept on this path: the argument holds as stated.
  if (exact_ok && !s_bad) {
    __shared__ double s_wsum[kRankThreads / 32];
    __shared__ double s_carry;
    __shared__ int s_first;
    if (tid == 0) { s_carry = 0.0; s_first = total; }
    __syncthreads();
    for (int base = 0; base < total && s_first == total; base += kRankThreads) {
      const int i = base + tid;
      double v = 0.0;
      if (i < total) v = (double)key_value((unsigned)(keys[i] >> 32));
      double x = v;                                   // inclusive warp scan
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        double y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (lane == 31) s_wsum[wid] = x;
      __syncthreads();
      double off = s_carry;
      for (int w = 0; w < wid; ++w) off += s_wsum[w];
      const double cum = off + x;
      if (i < total && cum > eps) atomicMin(&s_first, i);
      __syncthreads();
      if (tid == kRankThreads - 1) s_carry = cum;     // carry = inclusive sum of the whole chunk
      __syncthreads();
    }
    if (tid == 0) {
      cand_count[b] = s_first < total ? s_first + 1 : total;
      cand_total[b] = total;
    }
  } else if (tid == 0) {
    double tp = 0.0;
    int cnt = 0;
    for (int i = 0; i < total; ++i) {
      tp += (double)key_value((unsigned)(keys[i] >> 32));
      cnt = i + 1;
      if (tp > eps) break;
    }
    cand_count[b] = cnt;
    cand_total[b] = total;
  }
  // 4. ordered local indices
  for (int i = tid; i < N; i += kRankThreads)   // slots past `total` are zero-filled (defined output)
    cand_idx[(int64_t)b * N + i] = i < total ? (int32_t)(keys[i] & 0xFFFFFFFFull) : 0;
}

// ---- train-time metrics (get_eval_metric, base_model.py:236-298) ------------------------------------------------------
// One CTA per question.  hit@1: answer_dist > 1e-10 at the top-1 of pred_dist (torch.argmax: NaN counts as the maximum,
// ties go to the first index).  F1 (questions with hit@1 only): the candidates are the first cand_count[b] entries of
// cand_idx (gr_rank_candidates); the answers are the non-seed, non-pad nodes with answer mass, kept as a LIST of entity
// ids (duplicates count in the recall denominator); a candidate is correct when its entity id is among them (np.isin).
// The F1 is evaluated in float64 with the host's operations and rounded once to fp32, so it is bit-equal.
constexpr int kMetricThreads = 256;
constexpr int kSmemAnswers = 2048;    // answer ids kept in shared memory; more are matched from global memory

__device__ __forceinline__ bool argmax_before(float v, int i, float bv, int bi) {
  const bool vn = v != v, bn = bv != bv;
  if (vn != bn) return vn;
  if (!vn && v != bv) return v > bv;
  return i < bi;
}

__device__ __forceinline__ bool is_answer(const float* ad, const float* sd, const int64_t* le, int64_t pad_id, int n) {
  return ad[n] > 0.f && !(sd[n] > 0.f) && le[n] != pad_id;
}

__global__ void __launch_bounds__(kMetricThreads)
train_metrics_kernel(const float* __restrict__ pred_dist, const float* __restrict__ answer_dist,
                     const float* __restrict__ seed_dist, const int64_t* __restrict__ local_entity, int64_t pad_id,
                     const int32_t* __restrict__ cand_idx, const int32_t* __restrict__ cand_count,
                     float* __restrict__ h1, float* __restrict__ f1, int N) {
  constexpr int nw = kMetricThreads / 32;
  __shared__ float s_v[nw];
  __shared__ int s_i[nw];
  __shared__ int64_t s_ans[kSmemAnswers];
  __shared__ int s_hit, s_n_ans, s_correct;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const float* p = pred_dist + (int64_t)b * N;
  const float* ad = answer_dist + (int64_t)b * N;
  const float* sd = seed_dist + (int64_t)b * N;
  const int64_t* le = local_entity + (int64_t)b * N;
  // 1. top-1 and hit@1
  float bv = -INFINITY;
  int bi = INT_MAX;
  for (int n = tid; n < N; n += kMetricThreads) {
    const float v = p[n];
    if (argmax_before(v, n, bv, bi)) { bv = v; bi = n; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_down_sync(0xffffffffu, bv, o);
    const int oi = __shfl_down_sync(0xffffffffu, bi, o);
    if (argmax_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) { s_v[wid] = bv; s_i[wid] = bi; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < nw; ++w)
      if (argmax_before(s_v[w], s_i[w], bv, bi)) { bv = s_v[w]; bi = s_i[w]; }
    s_hit = ad[bi] > 1e-10f;           // (answer_dist > 1e-10) of an fp32 tensor compares in fp32
    s_n_ans = 0;
    s_correct = 0;
    h1[b] = s_hit ? 1.f : 0.f;
  }
  __syncthreads();
  if (!s_hit) {
    if (tid == 0) f1[b] = 0.f;
    return;
  }
  // 2. the answer list
  for (int n = tid; n < N; n += kMetricThreads) {
    if (is_answer(ad, sd, le, pad_id, n)) {
      const int pos = atomicAdd(&s_n_ans, 1);
      if (pos < kSmemAnswers) s_ans[pos] = le[n];
    }
  }
  __syncthreads();
  const int n_ans = s_n_ans;
  const int c = min(max(cand_count[b], 0), N);
  // 3. candidates whose entity id is an answer id
  int correct = 0;
  for (int i = tid; i < c; i += kMetricThreads) {
    const int ix = cand_idx[(int64_t)b * N + i];
    if ((unsigned)ix >= (unsigned)N) continue;
    const int64_t e = le[ix];
    bool found = false;
    if (n_ans <= kSmemAnswers) {
      for (int k = 0; k < n_ans && !found; ++k) found = s_ans[k] == e;
    } else {
      for (int n = 0; n < N && !found; ++n) found = le[n] == e && is_answer(ad, sd, le, pad_id, n);
    }
    correct += found;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) correct += __shfl_down_sync(0xffffffffu, correct, o);
  if (lane == 0 && correct) atomicAdd(&s_correct, correct);
  __syncthreads();
  if (tid == 0) {
    const int k = s_correct;
    double v;
    if (n_ans == 0) {
      v = c == 0 ? 1.0 : 0.0;
    } else if (c == 0 || k == 0) {
      v = 0.0;
    } else {                           // 2 / (1/p + 1/r) with p = k / c, r = k / n_ans, each op rounded as on the host
      const double pr = __ddiv_rn((double)k, (double)c), rc = __ddiv_rn((double)k, (double)n_ans);
      v = __ddiv_rn(2.0, __dadd_rn(__ddiv_rn(1.0, pr), __ddiv_rn(1.0, rc)));
    }
    f1[b] = __double2float_rn(v);
  }
}

}  // namespace
}  // namespace gr

extern "C" int gr_train_metrics(const float* pred_dist, const float* answer_dist, const float* seed_dist,
                                const int64_t* local_entity, int64_t pad_id, const int32_t* cand_idx,
                                const int32_t* cand_count, float* h1, float* f1, int B, int N, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(pred_dist && answer_dist && seed_dist && local_entity && cand_idx && cand_count && h1 && f1,
               "null pointer");
  GR_CHECK_ARG(B > 0 && N > 0, "B and N must be positive");
  train_metrics_kernel<<<B, kMetricThreads, 0, stream>>>(pred_dist, answer_dist, seed_dist, local_entity, pad_id,
                                                         cand_idx, cand_count, h1, f1, N);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" size_t gr_rank_workspace_bytes(int B, int N) {
  if (B <= 0 || N <= 0) return 0;
  return (size_t)B * (size_t)N * sizeof(unsigned long long);
}

extern "C" int gr_rank_candidates(const float* dist, const int64_t* local_entity,
                                  const float* query_entities, int64_t pad_id, double eps,
                                  int32_t* cand_idx, int32_t* cand_count, int32_t* cand_total, int B,
                                  int N, void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(dist && local_entity && query_entities && cand_idx && cand_count && cand_total,
               "null pointer");
  GR_CHECK_ARG(B > 0 && N > 0, "bad shape");
  if (workspace_bytes < gr_rank_workspace_bytes(B, N) || !workspace) {
    set_error("gr_rank_candidates: workspace too small");
    return GR_ERR_WORKSPACE;
  }
  double ignore_prob = (1 - eps) / N;   // evaluate.py:156
  // order-independence of the fp64 running sum (see rank_kernel step 3)
  int exact_ok = 0;
  if (ignore_prob > 0.0 && ignore_prob < 1.0) {
    int e_min;
    frexp(ignore_prob, &e_min);                       // ignore_prob = m * 2^e_min, m in [0.5, 1)
    // all terms are multiples of 2^(e_min - 24); terms are <= 1 (checked on device) and the scan only trusts
    // partial sums up to the first crossing of eps (< eps + 1 < 2): 24 + (1 - e_min) + 1 bits suffice
    int bits = 24 + (1 - e_min) + 1;
    exact_ok = bits <= 53 && eps < 1.0;
  }
  rank_kernel<<<B, kRankThreads, 0, stream>>>(dist, local_entity, query_entities, pad_id, eps,
                                              ignore_prob, cand_idx, cand_count, cand_total, N,
                                              reinterpret_cast<unsigned long long*>(workspace), exact_ok);
  GR_CHECK_LAUNCH();
  return GR_OK;
}
