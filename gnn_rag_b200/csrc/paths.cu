// Shortest-path node sets between seed entities and retrieved candidates (SURVEY.md 8f row 1).
//
// Reference: build_graph (llm/src/utils/graph_utils.py:10-21) makes an UNDIRECTED nx.Graph from the
// question's triples; get_truth_paths (:49-75) enumerates nx.all_shortest_paths(seed, answer) for every
// (seed, candidate) pair.  The set of nodes on those paths is {v : d(s,v) + d(v,t) = d(s,t)}.
//
// Two kernels serve every caller:
//   bfs_kernel   one CTA per (question, root), a root being one of the question's sources or targets: a
//                level-synchronous BFS over the union of the tail-CSR and head-CSR (which together are the undirected
//                adjacency) into the root's distance row of the workspace [B, S + T, N].  A row of N <= 12 288 is
//                expanded in shared memory and copied out once.
//   mark_kernel  one CTA per question: on_path and pair_dist from the distance rows.
// gr_eval_step_paths (an evaluation epoch's graphs, graphed.GraphedStep.start_eval with path_targets) selects the
// roots on the device before them, and after them scans the node counts into a running offset and compacts each
// question's on-path nodes into the split's node records.
// Pure integer work and no atomics: bit-exact and independent of scheduling.
#include <limits.h>

#include "common.cuh"

namespace gr {
namespace {

constexpr int kThreads = 512;
constexpr int kSmemDistBytes = 48 * 1024;          // the default dynamic shared-memory limit: no opt-in needed

// Level-synchronous BFS from `root` over both CSRs of the question whose global rows start at row0: dist (N entries,
// shared or global memory) receives the hop distances, -1 for unreachable.
__device__ void bfs_levels(int root, int32_t* dist, int N, int64_t row0, const int32_t* __restrict__ rp_t,
                           const int32_t* __restrict__ src_t, const int32_t* __restrict__ rp_h,
                           const int32_t* __restrict__ src_h) {
  for (int v = threadIdx.x; v < N; v += blockDim.x) dist[v] = (v == root) ? 0 : -1;
  __syncthreads();
  for (int level = 0; level < N; ++level) {
    int changed = 0;
    for (int v = threadIdx.x; v < N; v += blockDim.x) {
      if (dist[v] != level) continue;
      const int64_t g = row0 + v;
      for (int e = rp_t[g]; e < rp_t[g + 1]; ++e) {
        const int u = (int)(src_t[e] - row0);
        if (u >= 0 && u < N && dist[u] < 0) { dist[u] = level + 1; changed = 1; }
      }
      for (int e = rp_h[g]; e < rp_h[g + 1]; ++e) {
        const int u = (int)(src_h[e] - row0);
        if (u >= 0 && u < N && dist[u] < 0) { dist[u] = level + 1; changed = 1; }
      }
    }
    if (!__syncthreads_or(changed)) break;
  }
}

// Grid B * (S + T): CTA k runs the BFS of root r = k % (S + T) of question b = k / (S + T), source r (r < S) or
// target r - S, and writes its row of ws; a root past its question's count writes nothing.
template <bool kShared>
__global__ void __launch_bounds__(kThreads)
bfs_kernel(const int32_t* __restrict__ rp_t, const int32_t* __restrict__ src_t, const int32_t* __restrict__ rp_h,
           const int32_t* __restrict__ src_h, const int32_t* __restrict__ source_idx,
           const int32_t* __restrict__ source_cnt, int S, const int32_t* __restrict__ target_idx,
           const int32_t* __restrict__ target_cnt, int T, int N, int32_t* __restrict__ ws) {
  extern __shared__ int32_t s_dist[];
  const int b = blockIdx.x / (S + T), r = blockIdx.x % (S + T);
  int root;
  if (r < S) {
    if (r >= min(source_cnt[b], S)) return;
    root = source_idx[(int64_t)b * S + r];
  } else {
    if (r - S >= min(target_cnt[b], T)) return;
    root = target_idx[(int64_t)b * T + (r - S)];
  }
  const int64_t row0 = (int64_t)b * N;
  int32_t* row = ws + ((int64_t)b * (S + T) + r) * N;
  if (kShared) {
    bfs_levels(root, s_dist, N, row0, rp_t, src_t, rp_h, src_h);
    for (int v = threadIdx.x; v < N; v += blockDim.x) row[v] = s_dist[v];
  } else {
    bfs_levels(root, row, N, row0, rp_t, src_t, rp_h, src_h);
  }
}

// One CTA per question b: on_path[b, v] = 1 when d(s_i, v) + d(v, t_j) = d(s_i, t_j) for a connected pair (i, j),
// and the [S, T] block of pair distances (-1 past the counts) at row p of pair_dist.  p = b, or with `cursor` the
// position c * batch_size + b of an evaluation step, whose block is written only when c is in [0, steps) and
// p < num_data.  counts (optional): the number of on-path nodes of each question.
__global__ void __launch_bounds__(kThreads)
mark_kernel(const int32_t* __restrict__ source_cnt, int S, const int32_t* __restrict__ target_idx,
            const int32_t* __restrict__ target_cnt, int T, int N, const int32_t* __restrict__ ws,
            uint8_t* __restrict__ on_path, int32_t* __restrict__ pair_dist, int32_t* __restrict__ counts,
            const int64_t* __restrict__ cursor, int64_t steps, int64_t batch_size, int64_t num_data) {
  const int b = blockIdx.x;
  const int ns = max(min(source_cnt[b], S), 0), nt = max(min(target_cnt[b], T), 0);
  const int32_t* base = ws + (int64_t)b * (S + T) * N;
  const int32_t* tg = target_idx + (int64_t)b * T;
  bool write_pairs = true;
  int64_t p = b;
  if (cursor) {
    const int64_t c = *cursor;
    p = c * batch_size + b;
    write_pairs = c >= 0 && c < steps && p < num_data;
  }
  if (write_pairs) {
    for (int k = threadIdx.x; k < S * T; k += blockDim.x) {
      const int i = k / T, j = k % T;
      pair_dist[p * S * T + k] = (i < ns && j < nt) ? base[(int64_t)i * N + tg[j]] : -1;
    }
  }
  int total = 0;
  for (int v0 = 0; v0 < N; v0 += blockDim.x) {
    const int v = v0 + threadIdx.x;
    int on = 0;
    if (v < N) {
      for (int i = 0; i < ns && !on; ++i) {
        const int32_t* ds = base + (int64_t)i * N;
        const int dsv = ds[v];
        if (dsv < 0) continue;
        for (int j = 0; j < nt; ++j) {
          const int dst = ds[tg[j]];
          const int dtv = base[(int64_t)(S + j) * N + v];
          if (dst >= 0 && dtv >= 0 && dsv + dtv == dst) { on = 1; break; }
        }
      }
      on_path[(int64_t)b * N + v] = (uint8_t)on;
    }
    if (counts) total += __syncthreads_count(on);
  }
  if (counts && threadIdx.x == 0) counts[b] = total;
}

void launch_bfs(const int32_t* rp_t, const int32_t* src_t, const int32_t* rp_h, const int32_t* src_h,
                const int32_t* source_idx, const int32_t* source_cnt, int S, const int32_t* target_idx,
                const int32_t* target_cnt, int T, int B, int N, int32_t* ws, cudaStream_t stream) {
  const unsigned grid = (unsigned)((int64_t)B * (S + T));
  if ((int64_t)N * 4 <= kSmemDistBytes)
    bfs_kernel<true><<<grid, kThreads, N * 4, stream>>>(rp_t, src_t, rp_h, src_h, source_idx, source_cnt, S,
                                                        target_idx, target_cnt, T, N, ws);
  else
    bfs_kernel<false><<<grid, kThreads, 0, stream>>>(rp_t, src_t, rp_h, src_h, source_idx, source_cnt, S,
                                                     target_idx, target_cnt, T, N, ws);
}

// ---- an evaluation step's node sets (gr_eval_step_paths) --------------------------------------------------------

constexpr int kSelectThreads = 256;
constexpr int kScanThreads = 1024;
constexpr int kCompactThreads = 256;

// One warp per question j < B: the local indices with query_entities != 0 in increasing order (at most S of them)
// and the first min(cand_count, T) ranked candidates.  Outside [0, steps): no roots.
__global__ void __launch_bounds__(kSelectThreads)
eval_paths_select_kernel(const int64_t* __restrict__ cursor, int64_t steps, int B, int N,
                         const float* __restrict__ query_entities, const int32_t* __restrict__ cand_idx,
                         const int32_t* __restrict__ cand_count, int S, int T, int32_t* __restrict__ source_idx,
                         int32_t* __restrict__ source_cnt, int32_t* __restrict__ target_idx,
                         int32_t* __restrict__ target_cnt) {
  const int j = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = lane_id();
  if (j >= B) return;
  const int64_t c = *cursor;
  const bool in_epoch = c >= 0 && c < steps;
  const float* qe = query_entities + (int64_t)j * N;
  int found = 0;
  for (int v0 = 0; in_epoch && v0 < N && found < S; v0 += 32) {
    const int v = v0 + lane;
    const bool seed = v < N && qe[v] != 0.0f;
    const unsigned m = __ballot_sync(0xffffffffu, seed);
    const int at = found + __popc(m & ((1u << lane) - 1u));
    if (seed && at < S) source_idx[(int64_t)j * S + at] = v;
    found += __popc(m);
  }
  const int nt = in_epoch ? min(max(cand_count[j], 0), T) : 0;
  for (int k = lane; k < T; k += 32) target_idx[(int64_t)j * T + k] = k < nt ? cand_idx[(int64_t)j * N + k] : 0;
  if (lane == 0) {
    source_cnt[j] = min(found, S);
    target_cnt[j] = nt;
  }
}

// One CTA: node_off of the step's recorded questions is the exclusive scan of their counts in batch order from
// *node_total, node_count their counts; *node_total moves past them.  When the step's nodes do not all fit below
// capacity, bit 2 of *eval_status is set and *ok = 0, so the compaction writes none of them.
__global__ void __launch_bounds__(kScanThreads)
eval_paths_scan_kernel(const int64_t* __restrict__ cursor, int64_t steps, int64_t batch_size, int B,
                       int64_t num_data, const int32_t* __restrict__ counts, int64_t* __restrict__ node_off,
                       int32_t* __restrict__ node_count, int64_t* __restrict__ node_total, int64_t capacity,
                       int32_t* __restrict__ eval_status, int32_t* __restrict__ ok) {
  constexpr int kWarps = kScanThreads / 32;
  __shared__ int64_t s_warp[kWarps];
  __shared__ int64_t s_base;
  const int64_t c = *cursor;
  const bool in_epoch = c >= 0 && c < steps;
  const int64_t p0 = c * batch_size;
  const int lane = lane_id(), warp = warp_id();
  if (threadIdx.x == 0) s_base = *node_total;
  __syncthreads();
  const int64_t start = s_base;
  if (in_epoch) {
    for (int j0 = 0; j0 < B; j0 += kScanThreads) {
      const int j = j0 + threadIdx.x;
      const bool rec = j < B && p0 + j < num_data;
      const int64_t n = rec ? (int64_t)counts[j] : 0;
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
      if (rec) {
        node_off[p0 + j] = before + v - n;
        node_count[p0 + j] = (int32_t)n;
      }
      __syncthreads();                               // every thread has read s_base and s_warp
      if (threadIdx.x == kScanThreads - 1) s_base = before + v;
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) {
    const bool fits = s_base <= capacity;
    *ok = in_epoch && fits;
    if (in_epoch) {
      *node_total = s_base;
      if (!fits && s_base > start) *eval_status |= 2;
    }
  }
}

// One CTA per question: its on-path local indices, ascending, at node_off[p] of the node records (when *ok).
__global__ void __launch_bounds__(kCompactThreads)
eval_paths_compact_kernel(const int64_t* __restrict__ cursor, int64_t batch_size, int64_t num_data, int N,
                          const uint8_t* __restrict__ on_path, const int32_t* __restrict__ ok,
                          const int64_t* __restrict__ node_off, int32_t* __restrict__ nodes) {
  constexpr int kWarps = kCompactThreads / 32;
  __shared__ int s_warp[kWarps];
  const int b = blockIdx.x;
  const int64_t p = *cursor * batch_size + b;
  if (!*ok || p >= num_data) return;
  const int lane = lane_id(), warp = warp_id();
  int32_t* out = nodes + node_off[p];
  const uint8_t* on = on_path + (int64_t)b * N;
  int base = 0;
  for (int v0 = 0; v0 < N; v0 += kCompactThreads) {
    const int v = v0 + threadIdx.x;
    const bool f = v < N && on[v];
    const unsigned m = __ballot_sync(0xffffffffu, f);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int before = base, total = 0;
    for (int w = 0; w < kWarps; ++w) {
      before += w < warp ? s_warp[w] : 0;
      total += s_warp[w];
    }
    if (f) out[before + __popc(m & ((1u << lane) - 1u))] = v;
    base += total;
    __syncthreads();                                 // s_warp is rewritten by the next chunk
  }
}

struct EvalPathsWs {
  int32_t *dist, *source_idx, *source_cnt, *target_idx, *target_cnt, *counts, *ok;
  uint8_t* on_path;
  size_t bytes;
};

EvalPathsWs eval_paths_ws(void* base, int64_t B, int64_t N, int64_t S, int64_t T) {
  EvalPathsWs w;
  int32_t* p = reinterpret_cast<int32_t*>(base);
  w.dist = p;             p += B * (S + T) * N;
  w.source_idx = p;       p += B * S;
  w.source_cnt = p;       p += B;
  w.target_idx = p;       p += B * T;
  w.target_cnt = p;       p += B;
  w.counts = p;           p += B;
  w.ok = p;               p += 1;
  w.on_path = reinterpret_cast<uint8_t*>(p);
  w.bytes = (size_t)(p - reinterpret_cast<int32_t*>(base)) * sizeof(int32_t) + (size_t)(B * N) + 16;
  return w;
}

}  // namespace
}  // namespace gr

extern "C" size_t gr_paths_workspace_bytes(int B, int N, int max_sources, int max_targets) {
  if (B <= 0 || N <= 0 || max_sources < 0 || max_targets < 0) return 0;
  return (size_t)B * (size_t)(max_sources + max_targets) * (size_t)N * sizeof(int32_t) + 16;
}

extern "C" int gr_shortest_path_nodes(const int32_t* rowptr_t, const int32_t* src_t,
                                      const int32_t* rowptr_h, const int32_t* src_h,
                                      const int32_t* source_idx, const int32_t* source_cnt,
                                      int max_sources, const int32_t* target_idx,
                                      const int32_t* target_cnt, int max_targets, uint8_t* on_path,
                                      int32_t* pair_dist, int B, int N, void* workspace,
                                      size_t workspace_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(rowptr_t && rowptr_h && source_idx && source_cnt && target_idx && target_cnt &&
                   on_path && pair_dist,
               "null pointer");
  GR_CHECK_ARG(B > 0 && N > 0 && max_sources > 0 && max_targets > 0, "bad shape");
  if (!workspace || workspace_bytes < gr_paths_workspace_bytes(B, N, max_sources, max_targets)) {
    set_error("gr_shortest_path_nodes: workspace too small");
    return GR_ERR_WORKSPACE;
  }
  int32_t* ws = reinterpret_cast<int32_t*>(workspace);
  launch_bfs(rowptr_t, src_t, rowptr_h, src_h, source_idx, source_cnt, max_sources, target_idx, target_cnt,
             max_targets, B, N, ws, stream);
  GR_CHECK_LAUNCH();
  mark_kernel<<<B, kThreads, 0, stream>>>(source_cnt, max_sources, target_idx, target_cnt, max_targets, N, ws,
                                          on_path, pair_dist, nullptr, nullptr, 0, 0, 0);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" size_t gr_eval_paths_workspace_bytes(int B, int64_t N, int S, int T) {
  if (B <= 0 || N <= 0 || S < 0 || T <= 0) return 0;
  return gr::eval_paths_ws(nullptr, B, N, S, T).bytes;
}

extern "C" int gr_eval_step_paths(const int64_t* cursor, int64_t steps, int64_t batch_size, int B, int64_t num_data,
                                  int64_t N, const float* query_entities, const int32_t* cand_idx,
                                  const int32_t* cand_count, int S, int T, const int32_t* rowptr_t,
                                  const int32_t* src_t, const int32_t* rowptr_h, const int32_t* src_h,
                                  int64_t* node_off, int32_t* node_count, int32_t* pair_dist, int32_t* nodes,
                                  int64_t capacity, int64_t* node_total, int32_t* eval_status, void* workspace,
                                  size_t workspace_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(cursor && query_entities && cand_idx && cand_count && rowptr_t && src_t && rowptr_h && src_h,
               "null pointer");
  GR_CHECK_ARG(node_off && node_count && pair_dist && nodes && node_total && eval_status, "null output");
  GR_CHECK_ARG(B > 0 && batch_size >= B && steps >= 0 && num_data >= 0,
               "need 0 < B <= batch_size, steps >= 0 and num_data >= 0");
  GR_CHECK_ARG(N > 0 && N <= INT_MAX, "N must be in [1, INT_MAX]");
  GR_CHECK_ARG(S >= 0 && T > 0, "need S >= 0 and T > 0");
  GR_CHECK_ARG((int64_t)B * ((int64_t)S + T) * N <= INT_MAX, "B * (S + T) * N overflows int32 indexing");
  GR_CHECK_ARG(capacity >= 0, "capacity must be >= 0");
  const EvalPathsWs w = eval_paths_ws(workspace, B, N, S, T);
  if (int rc = check_workspace("gr_eval_step_paths", workspace, workspace_bytes, w.bytes)) return rc;
  const int n = (int)N;
  eval_paths_select_kernel<<<(unsigned)ceil_div((int64_t)B * 32, kSelectThreads), kSelectThreads, 0, stream>>>(
      cursor, steps, B, n, query_entities, cand_idx, cand_count, S, T, w.source_idx, w.source_cnt, w.target_idx,
      w.target_cnt);
  GR_CHECK_LAUNCH();
  launch_bfs(rowptr_t, src_t, rowptr_h, src_h, w.source_idx, w.source_cnt, S, w.target_idx, w.target_cnt, T, B, n,
             w.dist, stream);
  GR_CHECK_LAUNCH();
  mark_kernel<<<B, kThreads, 0, stream>>>(w.source_cnt, S, w.target_idx, w.target_cnt, T, n, w.dist, w.on_path,
                                          pair_dist, w.counts, cursor, steps, batch_size, num_data);
  GR_CHECK_LAUNCH();
  eval_paths_scan_kernel<<<1, kScanThreads, 0, stream>>>(cursor, steps, batch_size, B, num_data, w.counts, node_off,
                                                         node_count, node_total, capacity, eval_status, w.ok);
  GR_CHECK_LAUNCH();
  eval_paths_compact_kernel<<<B, kCompactThreads, 0, stream>>>(cursor, batch_size, num_data, n, w.on_path, w.ok,
                                                               node_off, nodes);
  GR_CHECK_LAUNCH();
  return GR_OK;
}
