// CSR batching on device: batched COO fact list -> in-edge CSR by tail and by head.
//
// Replaces BaseGNNLayer.build_matrix (reference gnn/modules/kg_reasoning/base_gnn.py:19-51) and the index
// half of TypeLayer.forward (gnn/modules/layer_init.py:32-37).  The reference builds seven uncoalesced
// COO tensors from Python lists on the host; here one histogram + scan + placement produces two CSRs.
// Inside a row the edges are re-ordered to ORIGINAL FACT ORDER (the order torch.sparse.mm walks an
// uncoalesced COO operand), which makes every downstream per-row reduction a pure function of the
// row's fact sequence: run-to-run deterministic, and structurally symmetric nodes get identical
// floats (the ranking-tie contract, SURVEY.md 7 hard part 1).
#include "common.cuh"

namespace gr {
namespace {

constexpr int kSmallRow = 16;        // rows up to this degree are sorted by one thread
constexpr int kSmemSortCap = 4096;   // long rows up to this degree are sorted in shared memory

__device__ __forceinline__ int64_t ld_idx(const void* p, int64_t i, int idx_bytes) {
  return idx_bytes == 8 ? reinterpret_cast<const int64_t*>(p)[i]
                        : (int64_t) reinterpret_cast<const int32_t*>(p)[i];
}

// `nfacts` (optional, device): the first *nfacts of the F slots hold facts, the rest is capacity padding of a
// fixed-shape (CUDA-graph) buffer and is ignored.
__device__ __forceinline__ int64_t live_facts(int64_t F, const int32_t* nfacts) {
  return nfacts ? min(F, (int64_t)max(*nfacts, 0)) : F;
}

__global__ void hist_kernel(const void* __restrict__ heads, const void* __restrict__ rels,
                            const void* __restrict__ tails, int idx_bytes, int64_t F, int64_t Nt,
                            int64_t R1, int32_t* __restrict__ cnt_t, int32_t* __restrict__ cnt_h,
                            int32_t* __restrict__ status, const int32_t* __restrict__ nfacts) {
  F = live_facts(F, nfacts);
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += stride) {
    int64_t h = ld_idx(heads, f, idx_bytes), t = ld_idx(tails, f, idx_bytes);
    int64_t r = ld_idx(rels, f, idx_bytes);
    if (h < 0 || h >= Nt || t < 0 || t >= Nt || r < 0 || r >= R1) {
      atomicOr(status, 1);
      h = min(max(h, (int64_t)0), Nt - 1);
      t = min(max(t, (int64_t)0), Nt - 1);
    }
    atomicAdd(&cnt_t[t], 1);
    atomicAdd(&cnt_h[h], 1);
  }
}

// ---- exclusive scan over n = Nt+1 counters, two arrays at once (blockIdx.y) -------------------------
constexpr int kScanThreads = 512;
constexpr int kScanItems = 4;
constexpr int kScanChunk = kScanThreads * kScanItems;

__device__ __forceinline__ int block_exclusive_scan(int v, int* smem, int& total) {
  // smem: >= blockDim.x/32 ints.  Returns exclusive prefix of v over the block; total = block sum.
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) smem[wid] = x;
  __syncthreads();
  int nw = blockDim.x >> 5;
  if (wid == 0) {
    int s = lane < nw ? smem[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < nw) smem[lane] = s;  // inclusive over warps
  }
  __syncthreads();
  int warp_off = wid == 0 ? 0 : smem[wid - 1];
  total = smem[nw - 1];
  __syncthreads();
  return warp_off + x - v;
}

__global__ void scan_local_kernel(const int32_t* __restrict__ cnt0, const int32_t* __restrict__ cnt1,
                                  int32_t* __restrict__ out0, int32_t* __restrict__ out1,
                                  int32_t* __restrict__ sums, int64_t n, int nblocks) {
  __shared__ int sm[32];
  const int32_t* cnt = blockIdx.y ? cnt1 : cnt0;
  int32_t* out = blockIdx.y ? out1 : out0;
  int64_t base = (int64_t)blockIdx.x * kScanChunk + (int64_t)threadIdx.x * kScanItems;
  int v[kScanItems];
  int s = 0;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    v[i] = (base + i < n) ? cnt[base + i] : 0;
    s += v[i];
  }
  int total;
  int ex = block_exclusive_scan(s, sm, total);
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    if (base + i < n) out[base + i] = ex;
    ex += v[i];
  }
  if (threadIdx.x == 0) sums[(int64_t)blockIdx.y * nblocks + blockIdx.x] = total;
}

__global__ void scan_sums_kernel(int32_t* __restrict__ sums, int nblocks) {
  // one block per array; sequential over chunks of blockDim
  __shared__ int sm[32];
  int32_t* s = sums + (int64_t)blockIdx.x * nblocks;
  int carry = 0;
  for (int base = 0; base < nblocks; base += blockDim.x) {
    int i = base + threadIdx.x;
    int v = i < nblocks ? s[i] : 0;
    int total;
    int ex = block_exclusive_scan(v, sm, total);
    if (i < nblocks) s[i] = carry + ex;
    carry += total;
  }
}

__global__ void scan_add_kernel(int32_t* __restrict__ out0, int32_t* __restrict__ out1,
                                int32_t* __restrict__ cur0, int32_t* __restrict__ cur1,
                                const int32_t* __restrict__ sums, int64_t n, int nblocks) {
  int32_t* out = blockIdx.y ? out1 : out0;
  int32_t* cur = blockIdx.y ? cur1 : cur0;
  int add = sums[(int64_t)blockIdx.y * nblocks + blockIdx.x];
  int64_t base = (int64_t)blockIdx.x * kScanChunk + (int64_t)threadIdx.x * kScanItems;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    if (base + i < n) {
      int v = out[base + i] + add;
      out[base + i] = v;
      cur[base + i] = v;
    }
  }
}

__global__ void place_kernel(const void* __restrict__ heads, const void* __restrict__ tails,
                             int idx_bytes, int64_t F, int64_t Nt, int32_t* __restrict__ cur_t,
                             int32_t* __restrict__ cur_h, int32_t* __restrict__ fact_t,
                             int32_t* __restrict__ fact_h, const int32_t* __restrict__ nfacts) {
  F = live_facts(F, nfacts);
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += stride) {
    int64_t h = ld_idx(heads, f, idx_bytes), t = ld_idx(tails, f, idx_bytes);
    h = min(max(h, (int64_t)0), Nt - 1);
    t = min(max(t, (int64_t)0), Nt - 1);
    fact_t[atomicAdd(&cur_t[t], 1)] = (int32_t)f;
    fact_h[atomicAdd(&cur_h[h], 1)] = (int32_t)f;
  }
}

// Restore original fact order inside each row.  Small rows: one thread, insertion sort in registers.
// Longer rows are appended to a work list for sort_rows_long_kernel.
__global__ void sort_rows_small_kernel(const int32_t* __restrict__ rowptr_t,
                                       const int32_t* __restrict__ rowptr_h,
                                       int32_t* __restrict__ fact_t, int32_t* __restrict__ fact_h,
                                       int64_t Nt, int32_t* __restrict__ long_list,
                                       int32_t* __restrict__ long_count) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * Nt) return;
  int dir = i >= Nt;
  int64_t row = dir ? i - Nt : i;
  const int32_t* rp = dir ? rowptr_h : rowptr_t;
  int32_t* fact = dir ? fact_h : fact_t;
  int beg = rp[row], end = rp[row + 1];
  int deg = end - beg;
  if (deg <= 1) return;
  if (deg > kSmallRow) {
    int slot = atomicAdd(long_count, 1);
    long_list[slot] = (int32_t)i;   // encodes (dir,row) as dir*Nt+row; Nt*2 < 2^31 checked on host
    return;
  }
  int v[kSmallRow];
#pragma unroll
  for (int k = 0; k < kSmallRow; ++k) v[k] = k < deg ? fact[beg + k] : 0x7fffffff;
  // fixed-size odd-even transposition network: fully unrolled, stays in registers
#pragma unroll
  for (int pass = 0; pass < kSmallRow; ++pass) {
#pragma unroll
    for (int k = pass & 1; k + 1 < kSmallRow; k += 2) {
      int a = v[k], b = v[k + 1];
      v[k] = min(a, b);
      v[k + 1] = max(a, b);
    }
  }
#pragma unroll
  for (int k = 0; k < kSmallRow; ++k)
    if (k < deg) fact[beg + k] = v[k];
}

__global__ void sort_rows_long_kernel(const int32_t* __restrict__ rowptr_t,
                                      const int32_t* __restrict__ rowptr_h,
                                      int32_t* __restrict__ fact_t, int32_t* __restrict__ fact_h,
                                      int64_t Nt, const int32_t* __restrict__ long_list,
                                      const int32_t* __restrict__ long_count) {
  __shared__ int32_t buf[kSmemSortCap];
  int count = *long_count;
  for (int it = blockIdx.x; it < count; it += gridDim.x) {
    int64_t i = long_list[it];
    int dir = i >= Nt;
    int64_t row = dir ? i - Nt : i;
    const int32_t* rp = dir ? rowptr_h : rowptr_t;
    int32_t* fact = dir ? fact_h : fact_t;
    int beg = rp[row], n = rp[row + 1] - beg;
    if (n <= kSmemSortCap) {
      for (int k = threadIdx.x; k < n; k += blockDim.x) buf[k] = fact[beg + k];
      __syncthreads();
      bitonic_sort_block(buf, n);
      for (int k = threadIdx.x; k < n; k += blockDim.x) fact[beg + k] = buf[k];
      __syncthreads();
    } else {
      __syncthreads();
      bitonic_sort_block(fact + beg, n);   // in place in global memory (L2 resident)
    }
  }
}

__global__ void fill_kernel(const void* __restrict__ heads, const void* __restrict__ rels,
                            const void* __restrict__ tails, int idx_bytes, int64_t F, int64_t Fpad,
                            int64_t Nt, int64_t R1,
                            const int32_t* __restrict__ fact_t, const int32_t* __restrict__ fact_h,
                            int32_t* __restrict__ src_t, int32_t* __restrict__ rel_t,
                            int32_t* __restrict__ src_h, int32_t* __restrict__ rel_h,
                            const int32_t* __restrict__ nfacts) {
  F = live_facts(F, nfacts);
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < Fpad; e += stride) {
    if (e >= F) {   // padding slots: defined values so whole-chunk staging copies are benign
      src_t[e] = 0; rel_t[e] = 0; src_h[e] = 0; rel_h[e] = 0;
      continue;
    }
    int ft = fact_t[e], fh = fact_h[e];
    int64_t h = ld_idx(heads, ft, idx_bytes), r = ld_idx(rels, ft, idx_bytes);
    src_t[e] = (int32_t)min(max(h, (int64_t)0), Nt - 1);
    rel_t[e] = (int32_t)min(max(r, (int64_t)0), R1 - 1);
    int64_t t = ld_idx(tails, fh, idx_bytes), r2 = ld_idx(rels, fh, idx_bytes);
    src_h[e] = (int32_t)min(max(t, (int64_t)0), Nt - 1);
    rel_h[e] = (int32_t)min(max(r2, (int64_t)0), R1 - 1);
  }
}

__global__ void gather_f32_kernel(const float* __restrict__ in, const int32_t* __restrict__ fact,
                                  float* __restrict__ out, int64_t F) {
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < F; e += stride) {
    const int64_t f = fact[e];                     // slots beyond the live fact count (capacity padding) hold garbage
    out[e] = in[min(max(f, (int64_t)0), F - 1)];   // and are never read through the row pointers: keep the load in bounds
  }
}

struct CsrWs {
  int32_t *cur_t, *cur_h, *sums, *long_list, *long_count;
  size_t bytes;
};

CsrWs carve(void* base, int64_t F, int64_t Nt) {
  CsrWs w;
  size_t off = 0;
  auto take = [&](size_t nbytes) {
    size_t o = off;
    off = align_up(off + nbytes, 256);
    return reinterpret_cast<int32_t*>(reinterpret_cast<char*>(base) + o);
  };
  int64_t n = Nt + 1;
  int nblocks = (int)ceil_div(n, kScanChunk);
  w.cur_t = take(sizeof(int32_t) * n);
  w.cur_h = take(sizeof(int32_t) * n);
  w.sums = take(sizeof(int32_t) * 2 * nblocks);
  w.long_list = take(sizeof(int32_t) * (2 * (F / (kSmallRow + 1)) + 2));
  w.long_count = take(sizeof(int32_t));
  w.bytes = off;
  return w;
}

}  // namespace
}  // namespace gr

extern "C" size_t gr_csr_build_workspace_bytes(int64_t F, int64_t Nt) {
  if (F < 0 || Nt < 0) return 0;
  return gr::carve(nullptr, F, Nt).bytes;
}

extern "C" int gr_csr_build(const void* heads, const void* rels, const void* tails, int idx_bytes,
                            int64_t F, int64_t Nt, int64_t num_rel_rows, int32_t* rowptr_t,
                            int32_t* src_t, int32_t* rel_t, int32_t* fact_t, int32_t* rowptr_h,
                            int32_t* src_h, int32_t* rel_h, int32_t* fact_h, int32_t* status,
                            const int32_t* nfacts, void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(idx_bytes == 4 || idx_bytes == 8, "idx_bytes must be 4 or 8");
  GR_CHECK_ARG(F >= 0 && Nt > 0 && num_rel_rows > 0, "F >= 0, Nt > 0, num_rel_rows > 0");
  GR_CHECK_ARG(2 * Nt < (int64_t)0x7fffffff && F < (int64_t)0x7fffffff, "Nt / F exceed int32 range");
  GR_CHECK_ARG(F == 0 || (heads && rels && tails), "null fact arrays");
  GR_CHECK_ARG(rowptr_t && rowptr_h && status && workspace, "null output");
  GR_CHECK_ARG(F == 0 || (src_t && rel_t && fact_t && src_h && rel_h && fact_h), "null edge output");
  CsrWs w = carve(workspace, F, Nt);
  if (int rc = check_workspace(__func__, workspace, workspace_bytes, w.bytes)) return rc;
  int64_t n = Nt + 1;
  int nblocks = (int)ceil_div(n, kScanChunk);
  GR_CHECK_CUDA(cudaMemsetAsync(w.cur_t, 0, sizeof(int32_t) * n, stream));
  GR_CHECK_CUDA(cudaMemsetAsync(w.cur_h, 0, sizeof(int32_t) * n, stream));
  GR_CHECK_CUDA(cudaMemsetAsync(w.long_count, 0, sizeof(int32_t), stream));
  GR_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), stream));
  const int threads = 256;
  int grid_f = (int)std::min<int64_t>(std::max<int64_t>(ceil_div(F, threads), 1), 8LL * sm_count());
  if (F > 0) {
    hist_kernel<<<grid_f, threads, 0, stream>>>(heads, rels, tails, idx_bytes, F, Nt, num_rel_rows,
                                                w.cur_t, w.cur_h, status, nfacts);
    GR_CHECK_LAUNCH();
  }
  scan_local_kernel<<<dim3(nblocks, 2), kScanThreads, 0, stream>>>(w.cur_t, w.cur_h, rowptr_t,
                                                                   rowptr_h, w.sums, n, nblocks);
  GR_CHECK_LAUNCH();
  scan_sums_kernel<<<2, 1024, 0, stream>>>(w.sums, nblocks);
  GR_CHECK_LAUNCH();
  scan_add_kernel<<<dim3(nblocks, 2), kScanThreads, 0, stream>>>(rowptr_t, rowptr_h, w.cur_t, w.cur_h,
                                                                 w.sums, n, nblocks);
  GR_CHECK_LAUNCH();
  if (F > 0) {
    place_kernel<<<grid_f, threads, 0, stream>>>(heads, tails, idx_bytes, F, Nt, w.cur_t, w.cur_h,
                                                 fact_t, fact_h, nfacts);
    GR_CHECK_LAUNCH();
    int64_t rows2 = 2 * Nt;
    sort_rows_small_kernel<<<(unsigned)ceil_div(rows2, threads), threads, 0, stream>>>(
        rowptr_t, rowptr_h, fact_t, fact_h, Nt, w.long_list, w.long_count);
    GR_CHECK_LAUNCH();
    sort_rows_long_kernel<<<2 * sm_count(), 512, 0, stream>>>(rowptr_t, rowptr_h, fact_t, fact_h, Nt,
                                                              w.long_list, w.long_count);
    GR_CHECK_LAUNCH();
    int64_t Fpad = gr_pad4(F);
    fill_kernel<<<grid_f, threads, 0, stream>>>(heads, rels, tails, idx_bytes, F, Fpad, Nt,
                                                num_rel_rows, fact_t, fact_h, src_t, rel_t, src_h, rel_h, nfacts);
    GR_CHECK_LAUNCH();
  }
  return GR_OK;
}

extern "C" int gr_gather_f32(const float* in, const int32_t* fact, float* out, int64_t F,
                             void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(F >= 0, "F >= 0");
  if (F == 0) return GR_OK;
  GR_CHECK_ARG(in && fact && out, "null pointer");
  int grid = (int)std::min<int64_t>(ceil_div(F, 256), 8LL * sm_count());
  gather_f32_kernel<<<grid, 256, 0, stream>>>(in, fact, out, F);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

namespace gr {
namespace {

__global__ void csr_row_of_kernel(const int32_t* __restrict__ rowptr, int64_t Nt, int32_t* __restrict__ row_of) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= Nt) return;
  for (int e = rowptr[n], end = rowptr[n + 1]; e < end; ++e) row_of[e] = (int32_t)n;
}

}  // namespace
}  // namespace gr

extern "C" int gr_csr_row_of(const int32_t* rowptr, int64_t Nt, int32_t* row_of, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(Nt > 0 && Nt < (int64_t)0x7fffffff, "need 0 < Nt < 2^31");
  GR_CHECK_ARG(rowptr && row_of, "null pointer");
  csr_row_of_kernel<<<(int)ceil_div(Nt, 256), 256, 0, stream>>>(rowptr, Nt, row_of);
  GR_CHECK_LAUNCH();
  return GR_OK;
}
