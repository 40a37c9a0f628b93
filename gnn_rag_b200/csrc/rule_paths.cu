// Rule-guided reasoning paths: bfs_with_rule (llm/src/utils/graph_utils.py:24-47) for many (start node, rule) jobs,
// as PromptBuilder.apply_rules calls it (llm/src/qa_prediction/build_qa_input.py:58-64).  Walks, not simple paths
// (no visited set), never truncated (max_p is unused in the reference), in the reference's FIFO order.
// 1. gr_rule_adj_build: each node row of the two CSRs is merged, deduplicated by neighbour (first fact = place in
//    nx.Graph's adjacency, last fact = label) and sorted by (label, first fact), so the neighbours with one label are
//    one contiguous segment in graph.neighbors order.
// 2. Per level: segment lengths, an int64 scan, children emitted parent by parent in segment order (the FIFO order,
//    no sorting); finished jobs' entries are their paths, walked back into [P, len + 1] node blocks at the end.
// Integer-only, no atomics in output placement: bit-exact and run-to-run identical.  DESIGN.md section 4.5.
#include "common.cuh"

namespace gr {
namespace {

constexpr int kSmallRow = 16;      // merged rows up to this length: one thread, registers
constexpr int kSmemRow = 2048;     // up to this length: CTA sort in shared memory (2 x 16 KB of 64-bit keys)
constexpr int kRowThreads = 256;
constexpr int kThreads = 256;

constexpr int kScanThreads = 256;
constexpr int kScanItems = 4;
constexpr int kScanChunk = kScanThreads * kScanItems;

// first index in [lo, hi) with a[idx] >= x (a sorted ascending)
template <typename T>
__device__ __forceinline__ int64_t lower_bound(const T* a, int64_t lo, int64_t hi, T x) {
  while (lo < hi) {
    int64_t mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// first index in [lo, hi) with a[idx] > x
template <typename T>
__device__ __forceinline__ int64_t upper_bound(const T* a, int64_t lo, int64_t hi, T x) {
  while (lo < hi) {
    int64_t mid = (lo + hi) >> 1;
    if (a[mid] <= x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

struct Csr2 {
  const int32_t *rp_t, *src_t, *rel_t, *fact_t, *rp_h, *src_h, *rel_h, *fact_h;
};

// neighbour and label of fact f in row u (f is in the tail row or the head row of u; a self-loop is in both)
__device__ __forceinline__ void fact_entry(const Csr2& g, int64_t u, int32_t f, int32_t& nbr, int32_t& lab) {
  const int bt = g.rp_t[u], et = g.rp_t[u + 1];
  const int64_t k = lower_bound(g.fact_t, (int64_t)bt, (int64_t)et, f);
  if (k < et && g.fact_t[k] == f) {
    nbr = g.src_t[k];
    lab = g.rel_t[k];
    return;
  }
  const int64_t kh = lower_bound(g.fact_h, (int64_t)g.rp_h[u], (int64_t)g.rp_h[u + 1], f);
  nbr = g.src_h[kh];
  lab = g.rel_h[kh];
}

// Rows of <= kSmallRow merged entries, one thread each.  Also writes the row pointers of every row.
__global__ void adj_small_kernel(Csr2 g, int64_t Nt, int32_t* __restrict__ out_rp, int32_t* __restrict__ out_len,
                                 int32_t* __restrict__ out_nbr, int32_t* __restrict__ out_lab) {
  const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= Nt) return;
  const int bt = g.rp_t[u], dt = g.rp_t[u + 1] - bt;
  const int bh = g.rp_h[u], dh = g.rp_h[u + 1] - bh;
  const int deg = dt + dh, beg = bt + bh;
  out_rp[u] = beg;
  if (u == Nt - 1) out_rp[Nt] = g.rp_t[Nt] + g.rp_h[Nt];
  if (deg > kSmallRow) return;
  int nb[kSmallRow], fa[kSmallRow], lb[kSmallRow];
#pragma unroll
  for (int k = 0; k < kSmallRow; ++k) {
    if (k < dt) {
      nb[k] = g.src_t[bt + k]; fa[k] = g.fact_t[bt + k]; lb[k] = g.rel_t[bt + k];
    } else if (k < deg) {
      nb[k] = g.src_h[bh + k - dt]; fa[k] = g.fact_h[bh + k - dt]; lb[k] = g.rel_h[bh + k - dt];
    } else {
      nb[k] = -1; fa[k] = 0x7fffffff; lb[k] = 0;
    }
  }
  // per entry: is it the first fact of its neighbour (ties between the two copies of a self-loop: lower slot), and
  // the label of its neighbour's last fact
  unsigned first = 0;
#pragma unroll
  for (int i = 0; i < kSmallRow; ++i) {
    bool f = i < deg;
    int lastf = fa[i], lab = lb[i];
#pragma unroll
    for (int j = 0; j < kSmallRow; ++j) {
      if (j != i && j < deg && nb[j] == nb[i]) {
        if (fa[j] < fa[i] || (fa[j] == fa[i] && j < i)) f = false;
        if (fa[j] > lastf) { lastf = fa[j]; lab = lb[j]; }
      }
    }
    if (f) first |= 1u << i;
    lb[i] = lab;    // only read for first entries below, whose own label is no longer needed
  }
  // rank of each first entry among the first entries by (label, first fact); distinct neighbours have distinct facts
#pragma unroll
  for (int i = 0; i < kSmallRow; ++i) {
    if (!((first >> i) & 1u)) continue;
    int r = 0;
#pragma unroll
    for (int j = 0; j < kSmallRow; ++j)
      if (((first >> j) & 1u) && (lb[j] < lb[i] || (lb[j] == lb[i] && fa[j] < fa[i]))) ++r;
    out_nbr[beg + r] = nb[i];
    out_lab[beg + r] = lb[i];
  }
  out_len[u] = __popc(first);
}

// Rows of more than kSmallRow merged entries: one CTA per row (grid-stride over rows; the skip test is block-uniform).
//   a: keys (neighbour << 32 | fact), sorted -> one run per neighbour, its first and last fact at the run's ends
//   b: per run (label << 32 | first fact), other slots ~0, sorted -> the output row
__global__ void __launch_bounds__(kRowThreads)
adj_long_kernel(Csr2 g, int64_t Nt, int32_t* __restrict__ out_len, int32_t* __restrict__ out_nbr,
                int32_t* __restrict__ out_lab, uint64_t* __restrict__ ws_a, uint64_t* __restrict__ ws_b) {
  __shared__ uint64_t sa[kSmemRow], sb[kSmemRow];
  __shared__ int s_n;
  for (int64_t u = blockIdx.x; u < Nt; u += gridDim.x) {
    const int bt = g.rp_t[u], dt = g.rp_t[u + 1] - bt;
    const int bh = g.rp_h[u], dh = g.rp_h[u + 1] - bh;
    const int deg = dt + dh, beg = bt + bh;
    if (deg <= kSmallRow) continue;
    uint64_t* a = deg <= kSmemRow ? sa : ws_a + beg;
    uint64_t* b = deg <= kSmemRow ? sb : ws_b + beg;
    if (threadIdx.x == 0) s_n = 0;
    for (int k = threadIdx.x; k < deg; k += blockDim.x) {
      const int nbr = k < dt ? g.src_t[bt + k] : g.src_h[bh + k - dt];
      const int f = k < dt ? g.fact_t[bt + k] : g.fact_h[bh + k - dt];
      a[k] = ((uint64_t)(uint32_t)nbr << 32) | (uint32_t)f;
    }
    __syncthreads();
    bitonic_sort_block(a, deg);
    for (int k = threadIdx.x; k < deg; k += blockDim.x) {
      const uint64_t key = a[k];
      const uint64_t v = key >> 32;
      if (k > 0 && (a[k - 1] >> 32) == v) {
        b[k] = ~(uint64_t)0;
        continue;
      }
      const int64_t last = upper_bound(a, (int64_t)k, (int64_t)deg, (uint64_t)((v << 32) | 0xffffffffull)) - 1;
      int32_t nbr, lab;
      fact_entry(g, u, (int32_t)(uint32_t)a[last], nbr, lab);
      b[k] = ((uint64_t)(uint32_t)lab << 32) | (key & 0xffffffffull);
      atomicAdd(&s_n, 1);   // a count only: placement comes from the sort below
    }
    __syncthreads();
    bitonic_sort_block(b, deg);
    const int nd = s_n;
    for (int k = threadIdx.x; k < nd; k += blockDim.x) {
      int32_t nbr, lab;
      fact_entry(g, u, (int32_t)(uint32_t)b[k], nbr, lab);
      out_nbr[beg + k] = nbr;
      out_lab[beg + k] = (int32_t)(b[k] >> 32);
    }
    if (threadIdx.x == 0) out_len[u] = nd;
    __syncthreads();
  }
}

// ---- level expansion -----------------------------------------------------------------------------------------------

struct Jobs {
  const int32_t *rule_off, *rule_len, *rule_lab;
  int J;
};

// cnt[i] = length of the segment of node[i]'s row whose label is the job's rule element at this level (0 once the job
// is finished); cnt[n] = 0 so the scan leaves the level total there.
__global__ void count_kernel(const int32_t* __restrict__ adj_rp, const int32_t* __restrict__ adj_len,
                             const int32_t* __restrict__ adj_lab, Jobs jobs, int level,
                             const int32_t* __restrict__ node, const int32_t* __restrict__ job, int64_t n,
                             int32_t* __restrict__ seg_begin, int64_t* __restrict__ cnt) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += stride) {
    if (i == n) { cnt[n] = 0; continue; }
    const int j = job[i];
    int64_t c = 0, sb = 0;
    const int u = node[i];
    if (level < jobs.rule_len[j] && u >= 0) {
      const int32_t lab = jobs.rule_lab[jobs.rule_off[j] + level];
      if (lab >= 0) {
        const int64_t b = adj_rp[u], e = b + adj_len[u];
        sb = lower_bound(adj_lab, b, e, lab);
        c = upper_bound(adj_lab, sb, e, lab) - sb;
      }
    }
    seg_begin[i] = (int32_t)sb;
    cnt[i] = c;
  }
}

__device__ __forceinline__ int64_t block_exclusive_scan64(int64_t v, int64_t* smem, int64_t& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int64_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) smem[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int64_t s = lane < nw ? smem[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int64_t y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < nw) smem[lane] = s;
  }
  __syncthreads();
  const int64_t off = wid == 0 ? 0 : smem[wid - 1];
  total = smem[nw - 1];
  __syncthreads();
  return off + x - v;
}

__global__ void __launch_bounds__(kScanThreads) scan_local_kernel(int64_t* __restrict__ a, int64_t m,
                                                                  int64_t* __restrict__ sums) {
  __shared__ int64_t sm[32];
  const int64_t base = (int64_t)blockIdx.x * kScanChunk + (int64_t)threadIdx.x * kScanItems;
  int64_t v[kScanItems], s = 0;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    v[i] = base + i < m ? a[base + i] : 0;
    s += v[i];
  }
  int64_t total;
  int64_t ex = block_exclusive_scan64(s, sm, total);
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    if (base + i < m) a[base + i] = ex;
    ex += v[i];
  }
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) scan_sums_kernel(int64_t* __restrict__ sums, int64_t nblocks) {
  __shared__ int64_t sm[32];
  int64_t carry = 0;
  for (int64_t base = 0; base < nblocks; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    const int64_t v = i < nblocks ? sums[i] : 0;
    int64_t total;
    const int64_t ex = block_exclusive_scan64(v, sm, total);
    if (i < nblocks) sums[i] = carry + ex;
    carry += total;
  }
}

__global__ void __launch_bounds__(kScanThreads) scan_add_kernel(int64_t* __restrict__ a, int64_t m,
                                                                const int64_t* __restrict__ sums) {
  const int64_t add = sums[blockIdx.x];
  const int64_t base = (int64_t)blockIdx.x * kScanChunk + (int64_t)threadIdx.x * kScanItems;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i)
    if (base + i < m) a[base + i] += add;
}

// jobs finishing at this level: their entries are one contiguous run of the job-major frontier
__global__ void job_ranges_kernel(Jobs jobs, int level, const int32_t* __restrict__ job, int64_t n,
                                  int32_t* __restrict__ res_begin, int32_t* __restrict__ res_count) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= jobs.J || jobs.rule_len[j] != level) return;
  const int64_t b = lower_bound(job, (int64_t)0, n, j);
  const int64_t e = lower_bound(job, b, n, j + 1);
  res_begin[j] = (int32_t)b;
  res_count[j] = (int32_t)(e - b);
}

// child c of the level: parent i = the entry whose scanned range [off[i], off[i+1]) holds c
__global__ void emit_kernel(const int32_t* __restrict__ adj_nbr, const int32_t* __restrict__ job,
                            const int32_t* __restrict__ seg_begin, const int64_t* __restrict__ off, int64_t n,
                            int64_t total, int32_t* __restrict__ child_node, int32_t* __restrict__ child_parent,
                            int32_t* __restrict__ child_job) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += stride) {
    const int64_t i = upper_bound(off, (int64_t)0, n + 1, c) - 1;
    child_node[c] = adj_nbr[seg_begin[i] + (c - off[i])];
    child_parent[c] = (int32_t)i;
    child_job[c] = job[i];
  }
}

// path t (all jobs, job-major) -> its job by binary search over path_off; nodes written from the last level back
__global__ void write_paths_kernel(const int32_t* const* __restrict__ level_node,
                                   const int32_t* const* __restrict__ level_parent,
                                   const int32_t* __restrict__ rule_len, const int32_t* __restrict__ res_begin,
                                   const int64_t* __restrict__ path_off, const int64_t* __restrict__ elem_off, int J,
                                   int64_t P, int32_t* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < P; t += stride) {
    const int j = (int)(upper_bound(path_off, (int64_t)0, (int64_t)J + 1, t) - 1);
    const int64_t k = t - path_off[j];
    const int L = rule_len[j];
    int32_t* dst = out + elem_off[j] + k * (L + 1);
    int64_t e = res_begin[j] + k;
    for (int l = L; l >= 0; --l) {
      dst[l] = level_node[l][e];
      e = level_parent[l][e];
    }
  }
}

int grid_for(int64_t n, int threads) {
  return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, threads), 16LL * sm_count()));
}

}  // namespace
}  // namespace gr

extern "C" size_t gr_rule_adj_workspace_bytes(int64_t F) {
  if (F < 0) return 0;
  return gr::align_up(sizeof(uint64_t) * 2 * (size_t)F, 256) * 2 + 256;
}

extern "C" int gr_rule_adj_build(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                                 const int32_t* fact_t, const int32_t* rowptr_h, const int32_t* src_h,
                                 const int32_t* rel_h, const int32_t* fact_h, int64_t Nt, int64_t F,
                                 int32_t* adj_rowptr, int32_t* adj_len, int32_t* adj_nbr, int32_t* adj_lab,
                                 void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(Nt > 0 && F >= 0 && 2 * F < (int64_t)0x7fffffff && Nt < (int64_t)0x7fffffff, "bad shape");
  GR_CHECK_ARG(rowptr_t && rowptr_h && adj_rowptr && adj_len, "null pointer");
  GR_CHECK_ARG(F == 0 || (src_t && rel_t && fact_t && src_h && rel_h && fact_h && adj_nbr && adj_lab),
               "null edge array");
  if (int rc = check_workspace(__func__, workspace, workspace_bytes, gr_rule_adj_workspace_bytes(F))) return rc;
  Csr2 g{rowptr_t, src_t, rel_t, fact_t, rowptr_h, src_h, rel_h, fact_h};
  adj_small_kernel<<<(unsigned)ceil_div(Nt, kThreads), kThreads, 0, stream>>>(g, Nt, adj_rowptr, adj_len, adj_nbr,
                                                                             adj_lab);
  GR_CHECK_LAUNCH();
  if (F > kSmallRow / 2) {   // a row longer than kSmallRow needs more than kSmallRow / 2 facts
    uint64_t* a = reinterpret_cast<uint64_t*>(workspace);
    uint64_t* b = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(workspace) +
                                              align_up(sizeof(uint64_t) * 2 * (size_t)F, 256));
    adj_long_kernel<<<2 * sm_count(), kRowThreads, 0, stream>>>(g, Nt, adj_len, adj_nbr, adj_lab, a, b);
    GR_CHECK_LAUNCH();
  }
  return GR_OK;
}

extern "C" size_t gr_rule_level_workspace_bytes(int64_t n) {
  if (n < 0) return 0;
  return sizeof(int64_t) * (size_t)gr::ceil_div(n + 1, gr::kScanChunk) + 256;
}

extern "C" int gr_rule_level_count(const int32_t* adj_rowptr, const int32_t* adj_len, const int32_t* adj_lab,
                                   const int32_t* job_rule_off, const int32_t* job_rule_len, const int32_t* rule_lab,
                                   int J, int level, const int32_t* node, const int32_t* job, int64_t n,
                                   int32_t* seg_begin, int64_t* child_off, int32_t* res_begin, int32_t* res_count,
                                   void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(J >= 0 && level >= 0 && n >= 0 && n <= (int64_t)0x7fffffff, "bad shape");
  GR_CHECK_ARG(adj_rowptr && adj_len && child_off && res_begin && res_count, "null pointer");
  GR_CHECK_ARG(J == 0 || (job_rule_off && job_rule_len), "null job array");
  GR_CHECK_ARG(n == 0 || (node && job && seg_begin), "null frontier array");
  if (int rc = check_workspace(__func__, workspace, workspace_bytes, gr_rule_level_workspace_bytes(n))) return rc;
  Jobs jobs{job_rule_off, job_rule_len, rule_lab, J};
  count_kernel<<<grid_for(n + 1, kThreads), kThreads, 0, stream>>>(adj_rowptr, adj_len, adj_lab, jobs, level, node,
                                                                   job, n, seg_begin, child_off);
  GR_CHECK_LAUNCH();
  const int64_t m = n + 1, nblocks = ceil_div(m, kScanChunk);
  int64_t* sums = reinterpret_cast<int64_t*>(workspace);
  scan_local_kernel<<<(unsigned)nblocks, kScanThreads, 0, stream>>>(child_off, m, sums);
  GR_CHECK_LAUNCH();
  if (nblocks > 1) {
    scan_sums_kernel<<<1, 1024, 0, stream>>>(sums, nblocks);
    GR_CHECK_LAUNCH();
    scan_add_kernel<<<(unsigned)nblocks, kScanThreads, 0, stream>>>(child_off, m, sums);
    GR_CHECK_LAUNCH();
  }
  if (J > 0) {
    job_ranges_kernel<<<(unsigned)ceil_div(J, kThreads), kThreads, 0, stream>>>(jobs, level, job, n, res_begin,
                                                                                res_count);
    GR_CHECK_LAUNCH();
  }
  return GR_OK;
}

extern "C" int gr_rule_level_emit(const int32_t* adj_nbr, const int32_t* job, const int32_t* seg_begin,
                                  const int64_t* child_off, int64_t n, int64_t total, int32_t* child_node,
                                  int32_t* child_parent, int32_t* child_job, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(n >= 0 && total >= 0, "bad shape");
  if (total > (int64_t)0x7fffffff) {
    set_error("gr_rule_level_emit: the level has %lld paths, more than int32 indexing allows",
              (long long)total);
    return GR_ERR_UNSUPPORTED;
  }
  if (total == 0) return GR_OK;
  GR_CHECK_ARG(adj_nbr && job && seg_begin && child_off && child_node && child_parent && child_job, "null pointer");
  emit_kernel<<<grid_for(total, kThreads), kThreads, 0, stream>>>(adj_nbr, job, seg_begin, child_off, n, total,
                                                                  child_node, child_parent, child_job);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_rule_paths_write(const int32_t* const* level_node, const int32_t* const* level_parent,
                                   const int32_t* job_rule_len, const int32_t* res_begin, const int64_t* path_off,
                                   const int64_t* elem_off, int J, int64_t P, int32_t* paths, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(J >= 0 && P >= 0, "bad shape");
  if (P == 0) return GR_OK;
  GR_CHECK_ARG(level_node && level_parent && job_rule_len && res_begin && path_off && elem_off && paths,
               "null pointer");
  write_paths_kernel<<<grid_for(P, kThreads), kThreads, 0, stream>>>(level_node, level_parent, job_rule_len,
                                                                     res_begin, path_off, elem_off, J, P, paths);
  GR_CHECK_LAUNCH();
  return GR_OK;
}
