// Device-resident split (loader.DeviceSplit): a split's per-question fact segments are uploaded once, and each batch is
// assembled on the device from B question ids.
//
//   gr_split_assemble        the kb_adj_mat fact arrays of SingleDataLoader._build_fact_mat (gnn/dataset_load.py:473-527)
//                            in stored fact order with the self-loops appended per question (loader.build_fact_mat with
//                            shuffle=False): row bias b*N, batch ids, fact ids, one pass.
//   gr_split_assemble_graft  both graft lists of GraftSingleDataLoader._build_fact_mat_maxfacts
//                            (gnn/dataset_load_graft.py:70-102) in stored order, and the kb_fact_rel rows.
//   gr_split_assemble_ordered / gr_split_assemble_graft_ordered   the same two with fact dropout (below): a question's
//                            facts are its kept count of a fact order, gathered through it.
//   gr_fact_weights          weight_list = 1/outdeg(head) and weight_rel_list = 1/count(head, rel) (:507-516).
//   gr_fact_weights_live     the same over the live prefix of capacity-length fact buffers, its length read on the
//                            device (the batch a captured training epoch assembles in place).
//
// Assembly: grid (X, B) with X = CTAs per question (a function of B alone).  Every CTA of question b adds up the fact
// counts of questions 0..b-1 itself (B ids, read from the resident offsets) to find where its question starts, so no
// host round trip and no second launch is needed; the host sizes the outputs from its own copy of the counts.
// Out-of-range question ids count as empty questions and set status bit 1; outputs that would run past the capacity
// the host passed are not written and set status bit 2.  One kernel per list serves both entry points of that list.
// Stored order reads every stored fact, fact k at k, after one block sum; ordered (kOrdered) the counts are kept[b]
// clamped to the stored ones and fact k is read at order[k], which adds the order's offsets (a second block sum for
// the kb facts), the bound K on the order and bit 1 for an entry that is not a stored index.  kOrdered is a template
// parameter, so the stored-order instance compiles to the stored-order code alone; the launcher picks it from `kept`,
// never from `order`: with every fact dropped, K = 0 and the order pointer is null.
//
// Weights: integer counting only.  outdeg(head) by atomicAdd on an int counter per row; count(head, rel) by an open-
// addressing hash table over the (head, rel) keys of the batch (linear probing, load <= 1/2) with an int counter per
// key.  The counts are exact whatever order the atomics land in, and each weight is 1.0 / count in float64 rounded
// once to fp32: bit-equal to fp32 of the host's float64 weights.
//
// Fact dropout (DeviceSplit with shuffle=True): the reference keeps the first floor(n (1 - p)) facts of a fresh
// np.random.permutation of each question's n facts (dataset_load.py:488-490, dataset_load_graft.py:88-90).
//   gr_split_fact_order      per question, the stored indices of the kept prefix of a uniform permutation: fact i of
//                            the question at batch position b gets a 64-bit Philox key, and the permutation is the
//                            ascending order of (key, i).  One CTA per question.  Up to kOrderSmem facts are keyed and
//                            bitonic-sorted in shared memory.  A larger question is bucketed by the top key bits (the
//                            keys are uniform, so the buckets are balanced, ~kOrderSmem / 4 each) into a global
//                            workspace; only the buckets that hold kept ranks are scattered and sorted, each in shared
//                            memory, or in the workspace when it overflows.  The sort is by a total order, so the
//                            result does not depend on the order the scatter's atomics land in.
#include <limits.h>

#include <algorithm>

#include "common.cuh"

namespace gr {
namespace {

constexpr int kSplitThreads = 256;
constexpr int kWeightThreads = 256;
constexpr unsigned long long kEmptyKey = ~0ull;

static int ctas_per_question(int B) {
  // enough CTAs to cover the SMs twice over at small B, one per question at large B
  return (int)std::max<int64_t>(1, std::min<int64_t>(64, ceil_div(2 * (int64_t)sm_count(), B)));
}

__device__ __forceinline__ bool valid_id(int64_t id, int64_t num_q) { return id >= 0 && id < num_q; }

// sum over the block of one int64 per thread (result valid in every thread)
__device__ __forceinline__ int64_t block_sum(int64_t v, int64_t* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
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

// per question: its facts (in stored order, or kOrdered: at the stored indices in its run of `order`), then the
// self-loops of its entities
template <typename IdxT, bool kOrdered>
__global__ void __launch_bounds__(kSplitThreads)
split_assemble_kernel(const int64_t* __restrict__ q_off, const int32_t* __restrict__ q_heads,
                      const int32_t* __restrict__ q_rels, const int32_t* __restrict__ q_tails,
                      const int32_t* __restrict__ q_ents, int64_t num_q, const int64_t* __restrict__ ids,
                      const int64_t* __restrict__ kept, const int32_t* __restrict__ order, int64_t K, int64_t N,
                      int64_t self_rel, int use_self_loop, int64_t F, IdxT* __restrict__ heads, IdxT* __restrict__ rels,
                      IdxT* __restrict__ tails, IdxT* __restrict__ bids, IdxT* __restrict__ fids,
                      int32_t* __restrict__ status) {
  __shared__ int64_t s_red[33];
  const int b = blockIdx.y;
  auto stored = [&](int64_t id) -> int64_t { return valid_id(id, num_q) ? q_off[id + 1] - q_off[id] : 0; };
  auto facts = [&](int j, int64_t n) -> int64_t { return kOrdered ? min(max(kept[j], (int64_t)0), n) : n; };
  auto ents = [&](int64_t id) -> int64_t { return use_self_loop && valid_id(id, num_q) ? (int64_t)q_ents[id] : 0; };
  int64_t before = 0, obefore = 0;
  for (int j = threadIdx.x; j < b; j += blockDim.x) {
    const int64_t idj = ids[j], kj = facts(j, stored(idj));
    obefore += kj;
    before += kj + ents(idj);
  }
  const int64_t pos = block_sum(before, s_red);
  const int64_t opos = kOrdered ? block_sum(obefore, s_red) : 0;
  const int64_t id = ids[b];
  const bool ok = valid_id(id, num_q);
  const int64_t base = ok ? q_off[id] : 0, nf = stored(id), k = facts(b, nf), tot = k + ents(id);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    if (!ok) atomicOr(status, 1);
    if (pos + tot > F || (kOrdered && opos + k > K)) atomicOr(status, 2);
  }
  const int64_t bias = (int64_t)b * N;
  const int64_t end = min(tot, F - pos);
  for (int64_t kk = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; kk < end; kk += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = pos + kk;
    int64_t h, r, t;
    if (kk < k) {
      int64_t s = kk;
      if (kOrdered) {
        if (opos + kk >= K) continue;          // past the order array (flagged above)
        s = order[opos + kk];
        if (s < 0 || s >= nf) {                // not a stored index of this question: not read, not written
          atomicOr(status, 1);
          continue;
        }
      }
      h = bias + q_heads[base + s];
      r = q_rels[base + s];
      t = bias + q_tails[base + s];
    } else {                                   // the self-loops of the question's entities (dataset_load.py:498-505)
      h = t = bias + (kk - k);
      r = self_rel;
    }
    heads[o] = (IdxT)h;
    rels[o] = (IdxT)r;
    tails[o] = (IdxT)t;
    bids[o] = (IdxT)b;
    fids[o] = (IdxT)o;
  }
}

// both graft lists (in stored order, or kOrdered: at the positions in `order`, the lists and the order sharing one
// layout) and the kb_fact_rel rows, stored either way
template <typename IdxT, bool kOrdered>
__global__ void __launch_bounds__(kSplitThreads)
split_assemble_graft_kernel(const int64_t* __restrict__ g_off, const int32_t* __restrict__ g_e2f_f,
                            const int32_t* __restrict__ g_e2f_e, const int32_t* __restrict__ g_f2e_e,
                            const int32_t* __restrict__ g_f2e_f, const int64_t* __restrict__ r_off,
                            const int32_t* __restrict__ r_vals, int64_t num_q, const int64_t* __restrict__ ids,
                            const int64_t* __restrict__ kept, const int32_t* __restrict__ order, int64_t K,
                            int64_t max_facts, int64_t rel_pad, int64_t G, IdxT* __restrict__ e2f_b,
                            IdxT* __restrict__ e2f_f, IdxT* __restrict__ e2f_e, float* __restrict__ e2f_v,
                            IdxT* __restrict__ f2e_b, IdxT* __restrict__ f2e_e, IdxT* __restrict__ f2e_f,
                            float* __restrict__ f2e_v, int64_t* __restrict__ kb_fact_rel,
                            int32_t* __restrict__ status) {
  __shared__ int64_t s_red[33];
  const int b = blockIdx.y;
  auto stored = [&](int64_t id) -> int64_t { return valid_id(id, num_q) ? g_off[id + 1] - g_off[id] : 0; };
  auto entries = [&](int j, int64_t n) -> int64_t { return kOrdered ? min(max(kept[j], (int64_t)0), n) : n; };
  int64_t before = 0;
  for (int j = threadIdx.x; j < b; j += blockDim.x) before += entries(j, stored(ids[j]));
  const int64_t pos = block_sum(before, s_red);
  const int64_t id = ids[b];
  const bool ok = valid_id(id, num_q);
  const int64_t base = ok ? g_off[id] : 0, n = stored(id), k = entries(b, n);
  const int64_t cap = kOrdered ? min(G, K) : G;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    if (!ok) atomicOr(status, 1);
    if (pos + k > cap) atomicOr(status, 2);
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x, k0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t end = min(k, cap - pos);
  for (int64_t kk = k0; kk < end; kk += stride) {
    const int64_t o = pos + kk;
    int64_t s = kk;
    if (kOrdered) {
      s = order[o];
      if (s < 0 || s >= n) {
        atomicOr(status, 1);
        continue;
      }
    }
    e2f_b[o] = (IdxT)b;
    e2f_f[o] = (IdxT)g_e2f_f[base + s];
    e2f_e[o] = (IdxT)g_e2f_e[base + s];
    e2f_v[o] = 1.0f;
    f2e_b[o] = (IdxT)b;
    f2e_e[o] = (IdxT)g_f2e_e[base + s];
    f2e_f[o] = (IdxT)g_f2e_f[base + s];
    f2e_v[o] = 1.0f;
  }
  // the kb_fact_rel row: the stored prefix of the question's row, then the pad relation
  const int64_t rbase = ok ? r_off[id] : 0, rlen = ok ? min(r_off[id + 1] - rbase, max_facts) : 0;
  int64_t* row = kb_fact_rel + (int64_t)b * max_facts;
  for (int64_t j = k0; j < max_facts; j += stride) row[j] = j < rlen ? (int64_t)r_vals[rbase + j] : rel_pad;
}

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {   // splitmix64 finaliser
  x ^= x >> 30;
  x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27;
  x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}

__device__ __forceinline__ int64_t ld_index(const void* p, int64_t i, int idx_bytes) {
  return idx_bytes == 8 ? reinterpret_cast<const int64_t*>(p)[i] : (int64_t)reinterpret_cast<const int32_t*>(p)[i];
}

// live facts of F slots: all of them, or the first min(F, max(*live, 0)) (as gr_csr_build reads nfacts)
__device__ __forceinline__ int64_t live_prefix(int64_t F, const int32_t* live) {
  return live ? min(F, (int64_t)max(*live, 0)) : F;
}

// pass 1: outdeg(head) and the (head, rel) counts; the hash slot of every fact is kept for pass 2
__global__ void __launch_bounds__(kWeightThreads)
fact_count_kernel(const void* __restrict__ heads, const void* __restrict__ rels, int idx_bytes, int64_t F, int64_t Nt,
                  unsigned long long* __restrict__ keys, uint32_t* __restrict__ counts, uint64_t table_mask,
                  uint32_t* __restrict__ deg, uint32_t* __restrict__ slot_of, int32_t* __restrict__ status,
                  const int32_t* __restrict__ live) {
  F = live_prefix(F, live);
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
    const int64_t h = ld_index(heads, f, idx_bytes), r = ld_index(rels, f, idx_bytes);
    if (h < 0 || h >= Nt || r < 0 || r > INT_MAX) {
      atomicOr(status, 1);
      slot_of[f] = 0xFFFFFFFFu;
      continue;
    }
    atomicAdd(&deg[h], 1u);
    const unsigned long long key = ((unsigned long long)h << 32) | (unsigned long long)r;
    uint64_t s = mix64(key) & table_mask;
    while (true) {
      const unsigned long long prev = atomicCAS(&keys[s], kEmptyKey, key);
      if (prev == kEmptyKey || prev == key) break;
      s = (s + 1) & table_mask;
    }
    atomicAdd(&counts[s], 1u);
    slot_of[f] = (uint32_t)s;
  }
}

// pass 2: weight = 1 / count, in float64, rounded once to fp32 (0 for a fact refused in pass 1)
__global__ void __launch_bounds__(kWeightThreads)
fact_weight_kernel(const void* __restrict__ heads, int idx_bytes, int64_t F, const uint32_t* __restrict__ counts,
                   const uint32_t* __restrict__ deg, const uint32_t* __restrict__ slot_of, float* __restrict__ w,
                   float* __restrict__ wr, const int32_t* __restrict__ live) {
  F = live_prefix(F, live);
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t s = slot_of[f];
    if (s == 0xFFFFFFFFu) {
      if (w) w[f] = 0.f;
      if (wr) wr[f] = 0.f;
      continue;
    }
    if (w) w[f] = __double2float_rn(__ddiv_rn(1.0, (double)deg[ld_index(heads, f, idx_bytes)]));
    if (wr) wr[f] = __double2float_rn(__ddiv_rn(1.0, (double)counts[s]));
  }
}

// ---- fact dropout: the kept prefix of a per-question permutation ----------------------------------------------------
constexpr int kOrderThreads = 1024;
constexpr int kOrderSmem = 8192;           // facts sorted in shared memory at once
constexpr int kOrderBucketMean = 2048;     // target facts per bucket of a question past kOrderSmem
constexpr int kOrderMaxBuckets = 2048;
constexpr size_t kOrderSmemBytes =
    (size_t)kOrderSmem * (sizeof(unsigned long long) + sizeof(uint32_t)) + (2 * kOrderMaxBuckets + 1) * sizeof(uint32_t);

// the sort key of stored fact i of the question at batch position b: Philox4x32-10 with key = seed and counter
// (i lo, i hi, b, perm) gives the high word, counter (i lo, i hi, b, perm | 2) the low word
__device__ __forceinline__ unsigned long long fact_key(uint64_t seed, int64_t i, int b, int perm) {
  const uint32_t lo = (uint32_t)i, hi = (uint32_t)((uint64_t)i >> 32);
  const uint32_t k1 = philox4x32_10_x0(seed, lo, hi, (uint32_t)b, (uint32_t)perm);
  const uint32_t k0 = philox4x32_10_x0(seed, lo, hi, (uint32_t)b, (uint32_t)perm | 2u);
  return ((unsigned long long)k1 << 32) | k0;
}

// bitonic_sort_block over (key, idx) pairs, ascending by key then idx; shared or global memory
__device__ void sort_pairs_block(unsigned long long* key, uint32_t* idx, int n) {
  auto cas = [&](int i, int l) {
    const unsigned long long a = key[i], c = key[l];
    const uint32_t x = idx[i], y = idx[l];
    if (a > c || (a == c && x > y)) {
      key[i] = c;
      key[l] = a;
      idx[i] = y;
      idx[l] = x;
    }
  };
  for (int k = 2; (k >> 1) < n; k <<= 1) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int l = i ^ (k - 1);
      if (l > i && l < n) cas(i, l);
    }
    __syncthreads();
    for (int j = k >> 2; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i && l < n) cas(i, l);
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(kOrderThreads)
split_fact_order_kernel(const int64_t* __restrict__ off, int64_t num_q, const int64_t* __restrict__ ids,
                        const int64_t* __restrict__ kept, const int64_t* __restrict__ seed_p, int perm, int64_t K,
                        int64_t n_total, int32_t* __restrict__ order, unsigned long long* __restrict__ w_key,
                        uint32_t* __restrict__ w_idx, int32_t* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int64_t s_red[33];
  auto* s_key = reinterpret_cast<unsigned long long*>(smem);
  auto* s_idx = reinterpret_cast<uint32_t*>(s_key + kOrderSmem);
  uint32_t* s_start = s_idx + kOrderSmem;            // [buckets + 1] first rank of each bucket
  uint32_t* s_cur = s_start + kOrderMaxBuckets + 1;  // [buckets] counts, then scatter cursors
  const int b = blockIdx.x;
  auto stored = [&](int64_t id) -> int64_t { return valid_id(id, num_q) ? off[id + 1] - off[id] : 0; };
  auto keep = [&](int j) -> int64_t { return min(max(kept[j], (int64_t)0), stored(ids[j])); };
  int64_t kb = 0, nb = 0;
  for (int j = threadIdx.x; j < b; j += blockDim.x) {
    kb += keep(j);
    nb += stored(ids[j]);
  }
  const int64_t opos = block_sum(kb, s_red);
  const int64_t wpos = block_sum(nb, s_red);
  const int64_t id = ids[b], n = stored(id), k = keep(b);
  const bool big = n > kOrderSmem;
  const bool fits = opos + k <= K && n <= INT_MAX && (!big || wpos + n <= n_total);
  if (threadIdx.x == 0) {
    if (!valid_id(id, num_q)) atomicOr(status, 1);
    if (!fits) atomicOr(status, 2);
  }
  if (!fits || k == 0) return;
  const uint64_t seed = (uint64_t)*seed_p;
  if (!big) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      s_key[i] = fact_key(seed, i, b, perm);
      s_idx[i] = (uint32_t)i;
    }
    __syncthreads();
    sort_pairs_block(s_key, s_idx, (int)n);
    for (int t = threadIdx.x; t < k; t += blockDim.x) order[opos + t] = (int32_t)s_idx[t];
    return;
  }
  int log_nb = 1;
  while ((1ll << log_nb) * kOrderBucketMean < n && (1 << log_nb) < kOrderMaxBuckets) ++log_nb;
  const int nbk = 1 << log_nb, shift = 64 - log_nb;
  for (int j = threadIdx.x; j < nbk; j += blockDim.x) s_cur[j] = 0;
  __syncthreads();
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) atomicAdd(&s_cur[fact_key(seed, i, b, perm) >> shift], 1u);
  __syncthreads();
  if (warp_id() == 0) {                              // exclusive scan of the bucket counts
    uint32_t carry = 0;
    for (int c = 0; c < nbk; c += 32) {
      const int j = c + lane_id();
      const uint32_t v = j < nbk ? s_cur[j] : 0u;
      uint32_t x = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane_id() >= o) x += y;
      }
      if (j < nbk) s_start[j] = s_cur[j] = carry + x - v;
      carry += __shfl_sync(0xffffffffu, x, 31);
    }
    if (lane_id() == 0) s_start[nbk] = carry;
  }
  __syncthreads();
  unsigned long long* wk = w_key + wpos;
  uint32_t* wi = w_idx + wpos;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {   // only the buckets that hold kept ranks
    const unsigned long long key = fact_key(seed, i, b, perm);
    const int j = (int)(key >> shift);
    if (s_start[j] < k) {
      const uint32_t p = atomicAdd(&s_cur[j], 1u);
      wk[p] = key;
      wi[p] = (uint32_t)i;
    }
  }
  __syncthreads();
  for (int j = 0; j < nbk && s_start[j] < k; ++j) {
    const int64_t s = s_start[j], c = s_start[j + 1] - s, take = min(c, k - s);
    if (c <= kOrderSmem) {
      for (int t = threadIdx.x; t < c; t += blockDim.x) {
        s_key[t] = wk[s + t];
        s_idx[t] = wi[s + t];
      }
      __syncthreads();
      sort_pairs_block(s_key, s_idx, (int)c);
      for (int t = threadIdx.x; t < take; t += blockDim.x) order[opos + s + t] = (int32_t)s_idx[t];
    } else {                                          // an overflowing bucket: sorted where it lies
      sort_pairs_block(wk + s, wi + s, (int)c);
      for (int64_t t = threadIdx.x; t < take; t += blockDim.x) order[opos + s + t] = (int32_t)wi[s + t];
    }
    __syncthreads();
  }
}

static size_t order_workspace_key_bytes(int64_t n_total) {
  return align_up((size_t)std::max<int64_t>(n_total, 1) * sizeof(unsigned long long), 256);
}

// hash table entries for F facts: the power of two >= 2F (at least 1024)
static uint64_t weight_table_size(int64_t F) {
  uint64_t t = 1024;
  while (t < 2 * (uint64_t)F) t <<= 1;
  return t;
}

struct WeightWorkspace {
  size_t keys, counts, deg, slot, total;
};

static WeightWorkspace weight_workspace(int64_t F, int64_t Nt) {
  WeightWorkspace w;
  const uint64_t T = weight_table_size(F);
  w.keys = 0;
  w.counts = align_up(T * sizeof(unsigned long long), 256);
  w.deg = w.counts + align_up(T * sizeof(uint32_t), 256);
  w.slot = w.deg + align_up((size_t)Nt * sizeof(uint32_t), 256);
  w.total = w.slot + align_up((size_t)std::max<int64_t>(F, 1) * sizeof(uint32_t), 256);
  return w;
}

// gr_split_assemble (kept and order null, K = 0: stored order) and gr_split_assemble_ordered: one validation and one
// launch, the messages reported as the calling entry point `fn`.  The ordered entry point refuses a null `kept` itself.
int split_assemble_launch(const char* fn, const int64_t* q_off, const int32_t* q_heads, const int32_t* q_rels,
                          const int32_t* q_tails, const int32_t* q_ents, int64_t num_q, const int64_t* ids,
                          const int64_t* kept, const int32_t* order, int64_t K, int B, int64_t N, int64_t self_rel,
                          int use_self_loop, int idx_bytes, int64_t F, void* heads, void* rels, void* tails,
                          void* batch_ids, void* fact_ids, int32_t* status, cudaStream_t stream) {
  GR_CHECK_ARG_AS(fn, q_off && ids && status, "null pointer");
  GR_CHECK_ARG_AS(fn, num_q >= 0 && B > 0 && N > 0 && F >= 0 && K >= 0,
                  kept ? "need num_q >= 0, B > 0, N > 0, F >= 0 and K >= 0"
                       : "need num_q >= 0, B > 0, N > 0 and F >= 0");
  GR_CHECK_ARG_AS(fn, idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
  GR_CHECK_ARG_AS(fn, idx_bytes == 8 || ((int64_t)B * N <= INT_MAX && F <= INT_MAX && self_rel <= INT_MAX),
                  "the batch overflows int32 indices");
  GR_CHECK_ARG_AS(fn, self_rel >= 0, "self_rel must be non-negative");
  GR_CHECK_ARG_AS(fn, F == 0 || (heads && rels && tails && batch_ids && fact_ids), "null output arrays");
  GR_CHECK_ARG_AS(fn, K == 0 || order, "null order");
  GR_CHECK_ARG_AS(fn, q_heads && q_rels && q_tails && q_ents, "null resident arrays");
  const dim3 grid(ctas_per_question(B), B);
  auto go = [&](auto t) {
    using IdxT = typename decltype(t)::type;
    const auto kernel = kept ? split_assemble_kernel<IdxT, true> : split_assemble_kernel<IdxT, false>;
    kernel<<<grid, kSplitThreads, 0, stream>>>(q_off, q_heads, q_rels, q_tails, q_ents, num_q, ids, kept, order, K, N,
                                               self_rel, use_self_loop, F, (IdxT*)heads, (IdxT*)rels, (IdxT*)tails,
                                               (IdxT*)batch_ids, (IdxT*)fact_ids, status);
  };
  idx_bytes == 8 ? go(type_tag<int64_t>{}) : go(type_tag<int32_t>{});
  GR_CHECK_LAUNCH_AS(fn);
  return GR_OK;
}

// gr_split_assemble_graft and gr_split_assemble_graft_ordered, as split_assemble_launch
int split_assemble_graft_launch(const char* fn, const int64_t* g_off, const int32_t* g_e2f_f, const int32_t* g_e2f_e,
                                const int32_t* g_f2e_e, const int32_t* g_f2e_f, const int64_t* r_off,
                                const int32_t* r_vals, int64_t num_q, const int64_t* ids, const int64_t* kept,
                                const int32_t* order, int64_t K, int B, int64_t max_facts, int64_t rel_pad,
                                int idx_bytes, int64_t G, void* e2f_b, void* e2f_f, void* e2f_e, float* e2f_v,
                                void* f2e_b, void* f2e_e, void* f2e_f, float* f2e_v, int64_t* kb_fact_rel,
                                int32_t* status, cudaStream_t stream) {
  GR_CHECK_ARG_AS(fn, g_off && r_off && ids && status, "null pointer");
  GR_CHECK_ARG_AS(fn, g_e2f_f && g_e2f_e && g_f2e_e && g_f2e_f && r_vals, "null resident arrays");
  GR_CHECK_ARG_AS(fn, num_q >= 0 && B > 0 && max_facts >= 0 && G >= 0 && K >= 0,
                  kept ? "need num_q >= 0, B > 0, max_facts >= 0, G >= 0 and K >= 0"
                       : "need num_q >= 0, B > 0, max_facts >= 0 and G >= 0");
  GR_CHECK_ARG_AS(fn, idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
  GR_CHECK_ARG_AS(fn, idx_bytes == 8 || (G <= INT_MAX && max_facts <= INT_MAX), "the batch overflows int32 indices");
  GR_CHECK_ARG_AS(fn, G == 0 || (e2f_b && e2f_f && e2f_e && e2f_v && f2e_b && f2e_e && f2e_f && f2e_v),
                  "null output arrays");
  GR_CHECK_ARG_AS(fn, K == 0 || order, "null order");
  GR_CHECK_ARG_AS(fn, max_facts == 0 || kb_fact_rel, "null kb_fact_rel");
  const dim3 grid(ctas_per_question(B), B);
  auto go = [&](auto t) {
    using IdxT = typename decltype(t)::type;
    const auto kernel = kept ? split_assemble_graft_kernel<IdxT, true> : split_assemble_graft_kernel<IdxT, false>;
    kernel<<<grid, kSplitThreads, 0, stream>>>(g_off, g_e2f_f, g_e2f_e, g_f2e_e, g_f2e_f, r_off, r_vals, num_q, ids,
                                               kept, order, K, max_facts, rel_pad, G, (IdxT*)e2f_b, (IdxT*)e2f_f,
                                               (IdxT*)e2f_e, e2f_v, (IdxT*)f2e_b, (IdxT*)f2e_e, (IdxT*)f2e_f, f2e_v,
                                               kb_fact_rel, status);
  };
  idx_bytes == 8 ? go(type_tag<int64_t>{}) : go(type_tag<int32_t>{});
  GR_CHECK_LAUNCH_AS(fn);
  return GR_OK;
}

}  // namespace
}  // namespace gr

extern "C" int gr_split_assemble(const int64_t* q_off, const int32_t* q_heads, const int32_t* q_rels,
                                 const int32_t* q_tails, const int32_t* q_ents, int64_t num_q, const int64_t* ids,
                                 int B, int64_t N, int64_t self_rel, int use_self_loop, int idx_bytes, int64_t F,
                                 void* heads, void* rels, void* tails, void* batch_ids, void* fact_ids,
                                 int32_t* status, void* stream_) {
  return gr::split_assemble_launch(__func__, q_off, q_heads, q_rels, q_tails, q_ents, num_q, ids, nullptr, nullptr, 0,
                                   B, N, self_rel, use_self_loop, idx_bytes, F, heads, rels, tails, batch_ids,
                                   fact_ids, status, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_split_assemble_graft(const int64_t* g_off, const int32_t* g_e2f_f, const int32_t* g_e2f_e,
                                       const int32_t* g_f2e_e, const int32_t* g_f2e_f, const int64_t* r_off,
                                       const int32_t* r_vals, int64_t num_q, const int64_t* ids, int B,
                                       int64_t max_facts, int64_t rel_pad, int idx_bytes, int64_t G, void* e2f_b,
                                       void* e2f_f, void* e2f_e, float* e2f_v, void* f2e_b, void* f2e_e, void* f2e_f,
                                       float* f2e_v, int64_t* kb_fact_rel, int32_t* status, void* stream_) {
  return gr::split_assemble_graft_launch(__func__, g_off, g_e2f_f, g_e2f_e, g_f2e_e, g_f2e_f, r_off, r_vals, num_q,
                                         ids, nullptr, nullptr, 0, B, max_facts, rel_pad, idx_bytes, G, e2f_b, e2f_f,
                                         e2f_e, e2f_v, f2e_b, f2e_e, f2e_f, f2e_v, kb_fact_rel, status,
                                         reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" size_t gr_fact_weights_workspace_bytes(int64_t F, int64_t Nt) {
  if (F < 0 || Nt <= 0) return 0;
  return gr::weight_workspace(F, Nt).total;
}

namespace gr {
namespace {

// gr_fact_weights (live = null) and gr_fact_weights_live: the table, the grid and the memsets are sized by the F slots,
// the kernels count and weigh the live prefix only, so the prefix is bit-equal to gr_fact_weights over it
int fact_weights_launch(const char* fn, const void* heads, const void* rels, int idx_bytes, int64_t F,
                        const int32_t* live, int64_t Nt, float* weight, float* weight_rel, int32_t* status,
                        void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  GR_CHECK_ARG_AS(fn, heads && rels && status, "null pointer");
  GR_CHECK_ARG_AS(fn, weight || weight_rel, "no output requested");
  GR_CHECK_ARG_AS(fn, idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
  GR_CHECK_ARG_AS(fn, F >= 0 && Nt > 0 && Nt <= UINT_MAX, "need F >= 0 and 0 < Nt <= 2^32 - 1");
  GR_CHECK_ARG_AS(fn, F <= (int64_t)INT_MAX, "F must fit int32 (hash slots are 32-bit)");
  const WeightWorkspace ws = weight_workspace(F, Nt);
  int rc = check_workspace(fn, workspace, workspace_bytes, ws.total);
  if (rc != GR_OK) return rc;
  if (F == 0) return GR_OK;
  char* base = static_cast<char*>(workspace);
  const uint64_t T = weight_table_size(F);
  auto* keys = reinterpret_cast<unsigned long long*>(base + ws.keys);
  auto* counts = reinterpret_cast<uint32_t*>(base + ws.counts);
  auto* deg = reinterpret_cast<uint32_t*>(base + ws.deg);
  auto* slot_of = reinterpret_cast<uint32_t*>(base + ws.slot);
  GR_CHECK_CUDA_AS(fn, cudaMemsetAsync(keys, 0xFF, T * sizeof(unsigned long long), stream));
  GR_CHECK_CUDA_AS(fn, cudaMemsetAsync(counts, 0, ws.slot - ws.counts, stream));        // counts and deg
  const int grid = (int)std::min<int64_t>(ceil_div(F, kWeightThreads), 8LL * sm_count());
  fact_count_kernel<<<grid, kWeightThreads, 0, stream>>>(heads, rels, idx_bytes, F, Nt, keys, counts, T - 1, deg,
                                                         slot_of, status, live);
  GR_CHECK_LAUNCH_AS(fn);
  fact_weight_kernel<<<grid, kWeightThreads, 0, stream>>>(heads, idx_bytes, F, counts, deg, slot_of, weight,
                                                          weight_rel, live);
  GR_CHECK_LAUNCH_AS(fn);
  return GR_OK;
}

}  // namespace
}  // namespace gr

extern "C" int gr_fact_weights(const void* heads, const void* rels, int idx_bytes, int64_t F, int64_t Nt,
                               float* weight, float* weight_rel, int32_t* status, void* workspace,
                               size_t workspace_bytes, void* stream_) {
  return gr::fact_weights_launch(__func__, heads, rels, idx_bytes, F, nullptr, Nt, weight, weight_rel, status,
                                 workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_fact_weights_live(const void* heads, const void* rels, int idx_bytes, int64_t capacity,
                                    const int32_t* nfacts, int64_t Nt, float* weight, float* weight_rel,
                                    int32_t* status, void* workspace, size_t workspace_bytes, void* stream_) {
  GR_CHECK_ARG(nfacts, "null nfacts");
  return gr::fact_weights_launch(__func__, heads, rels, idx_bytes, capacity, nfacts, Nt, weight, weight_rel, status,
                                 workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" size_t gr_split_fact_order_workspace_bytes(int64_t n_total) {
  if (n_total < 0) return 0;
  return gr::order_workspace_key_bytes(n_total) + gr::align_up((size_t)std::max<int64_t>(n_total, 1) * 4, 256);
}

extern "C" int gr_split_fact_order(const int64_t* off, int64_t num_q, const int64_t* ids, const int64_t* kept, int B,
                                   const int64_t* seed, int perm, int64_t n_total, int64_t K, int32_t* order,
                                   int32_t* status, void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(off && ids && kept && seed && status, "null pointer");
  GR_CHECK_ARG(num_q >= 0 && B > 0 && n_total >= 0 && K >= 0, "need num_q >= 0, B > 0, n_total >= 0 and K >= 0");
  GR_CHECK_ARG(K <= INT_MAX, "K must fit int32");
  GR_CHECK_ARG(perm == 0 || perm == 1, "perm must be 0 (kb facts) or 1 (graft lists)");
  GR_CHECK_ARG(K == 0 || order, "null order");
  const size_t need = gr_split_fact_order_workspace_bytes(n_total);
  int rc = check_workspace(__func__, workspace, workspace_bytes, need);
  if (rc != GR_OK) return rc;
  rc = opt_in_smem<split_fact_order_kernel>(__func__, (int)kOrderSmemBytes);
  if (rc != GR_OK) return rc;
  char* base = static_cast<char*>(workspace);
  split_fact_order_kernel<<<B, kOrderThreads, kOrderSmemBytes, stream>>>(
      off, num_q, ids, kept, seed, perm, K, n_total, order, reinterpret_cast<unsigned long long*>(base),
      reinterpret_cast<uint32_t*>(base + order_workspace_key_bytes(n_total)), status);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_split_assemble_ordered(const int64_t* q_off, const int32_t* q_heads, const int32_t* q_rels,
                                         const int32_t* q_tails, const int32_t* q_ents, int64_t num_q,
                                         const int64_t* ids, const int64_t* kept, const int32_t* order, int64_t K,
                                         int B, int64_t N, int64_t self_rel, int use_self_loop, int idx_bytes,
                                         int64_t F, void* heads, void* rels, void* tails, void* batch_ids,
                                         void* fact_ids, int32_t* status, void* stream_) {
  GR_CHECK_ARG(kept, "null pointer");
  return gr::split_assemble_launch(__func__, q_off, q_heads, q_rels, q_tails, q_ents, num_q, ids, kept, order, K, B,
                                   N, self_rel, use_self_loop, idx_bytes, F, heads, rels, tails, batch_ids, fact_ids,
                                   status, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_split_assemble_graft_ordered(const int64_t* g_off, const int32_t* g_e2f_f, const int32_t* g_e2f_e,
                                               const int32_t* g_f2e_e, const int32_t* g_f2e_f, const int64_t* r_off,
                                               const int32_t* r_vals, int64_t num_q, const int64_t* ids,
                                               const int64_t* kept, const int32_t* order, int64_t K, int B,
                                               int64_t max_facts, int64_t rel_pad, int idx_bytes, int64_t G,
                                               void* e2f_b, void* e2f_f, void* e2f_e, float* e2f_v, void* f2e_b,
                                               void* f2e_e, void* f2e_f, float* f2e_v, int64_t* kb_fact_rel,
                                               int32_t* status, void* stream_) {
  GR_CHECK_ARG(kept, "null pointer");
  return gr::split_assemble_graft_launch(__func__, g_off, g_e2f_f, g_e2f_e, g_f2e_e, g_f2e_f, r_off, r_vals, num_q,
                                         ids, kept, order, K, B, max_facts, rel_pad, idx_bytes, G, e2f_b, e2f_f,
                                         e2f_e, e2f_v, f2e_b, f2e_e, f2e_f, f2e_v, kb_fact_rel, status,
                                         reinterpret_cast<cudaStream_t>(stream_));
}
