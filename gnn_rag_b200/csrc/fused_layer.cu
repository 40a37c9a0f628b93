// One ReaRev GNN layer with a dense prior as ONE kernel: relation-typed aggregation of both directions and all
// instructions  ->  e2e linear (+ bias, relu, score dot)  (ReasonGNNLayer.forward, gnn/modules/kg_reasoning/
// reasongnn.py:134-174: reason_layer / reason_layer_inv :61-116, the torch.cat + e2e_linear of :158-163, the
// score_func dot of :165).
//
// The unfused pair (aggregate_abs.cu -> linear_tc.cu) writes the 2*I neighbour segments of the layer-input matrix to
// HBM (0.41 GB per layer at cfg2) and reads them straight back as the GEMM's A operand.  Here the neighbour k-blocks
// never leave the SM: aggregation warps produce them directly into the wgmma shared-memory operand slots (K-major,
// SWIZZLE_64B, bf16 hi/lo planes -- the layout TMA would have written), only the h segment and W come from memory.
//
// Per 128-row tile the K dimension is walked in G column groups of 32; group g holds, in this order,
//     H, Y(dir 0, j = 0..I-1), Y(dir 1, j = 0..I-1)              (T = 2*I + 1 k-blocks of 32 columns)
// i.e. column block g of every segment of [h | nb_0^fwd | nb_0^inv | nb_1^fwd | ...].  The S = sum c*v / Q = sum c*|v|
// accumulation of aggregate_abs.cu is instruction independent, so one pass over a row's in-edges restricted to the 32
// columns of group g yields the I blocks Y(dir, 0..I-1) together.  W is pre-formatted once per weight version in this
// K order (fused_w_split_kernel).  Arithmetic per element is the one of aggregate_abs.cu (same edge order, same FMA
// sequence, same hi/lo split), so the A operand is bit-identical to the unfused path; only the order in which the
// tensor core accumulates k-blocks differs (fp32 rounding, ~1e-7).
//
// Edge data: once per batch both CSRs are re-laid out slot-major per quad of 4 rows ("quad ELL",
// fused_ell_build_kernel); the kernel's stagers move a tile's entries into shared memory with ONE bulk copy per
// direction and turn {table offset, source node} into {table offset, c_f} there (weighted graphs: fused_coef_kernel), so
// no per-edge index arithmetic runs inside the fused kernel.
//
// The pair can walk K in this kernel's order (gr_linear_tc_planes with GR_LINEAR_K_GROUPED, same W planes:
// plan_grouped_k / grouped_w_split below) and then returns this kernel's bits; at accumulator widths above 128 columns
// it is the faster of the two (see the end of this comment) and ops.dense_layer runs it.  This kernel is the
// reference it is held to, and the dense layer of the widths it can issue as one instruction.
//
// Warp roles (512 threads, one CTA per SM, clusters of 2 share W by TMA multicast):
//   warp 0      TMA producer: W k-blocks into a 3-stage ring, the H block of every group into its operand slot (the
//               next tile's h blocks are L2-prefetched a tile ahead)
//   warps 2, 3  stagers: bulk copies of the tile's ELL entries + quad offsets, relu(+-ins)/2 of its <= 2 questions
//               -> double-buffered tile descriptor
//   warps 4-11  two consumer warpgroups, 64 tile rows each: wgmma.mma_async (3 products per k-step: one m64n{NP}k16
//               each up to NP = 128, 32-column instructions above, see "Registers" below) with the fp32 accumulator in
//               registers, then the epilogue: bias + relu + score dot -> fp32 h / bf16 planes via TMA stores
//   warps 12-15 aggregation: warp a owns tile rows 32a .. 32a+31 = eight quads; a quarter-warp owns a row, lane = 4
//               columns of the 32-column group, so one warp-wide 16-byte load gathers one in-edge of each row of the
//               quad (one 128-byte table line per row); 8 such loads in flight per lane, no predicates (slots past a
//               quad's block read a {0, 0} entry)
// Registers: 512 x 128 at launch; setmaxnreg shrinks the control (40) and aggregation (72) warpgroups and grows the
// consumers (200), whose register accumulators (128 rows x n_pad fp32 per tile) take the place of tensor memory.
// Operand slots are dedicated: slot t < 2I is always written by the aggregation warps, slot 2I always by TMA, so every
// slot barrier flips once per group and the parity is the group counter.
//
// Registers: ptxas places a wgmma accumulator operand within the 128 registers per thread of the launch, so an
// m64n208k16 (130 needed) does not compile here: accumulators wider than 128 columns are issued as 32-column
// instructions, one straight-line batch per k-block.
// Performance on one H100 80GB HBM3 at 700 W, cfg2 (scripts/dense_layer_probe.py): 1.02 ms per dense layer; the pair
// in this kernel's K order 0.23 + 0.49 ms, in segment order 0.23 + 0.34 ms.
#include <algorithm>
#include <cstddef>

#include "wgmma.cuh"

namespace gr {

// gr_set_option("fused_debug", bits): timing decomposition of the fused kernel (results are WRONG with any bit set).
// 1: aggregation warps skip the gather / emit work; 2: the stager skips the edge staging; 4: the epilogue skips its stores
int g_fused_debug = 0;

// bit 32 of fused_debug: per-CTA cycle counters of every role's waits (gr_fused_profile_read), 16 slots per CTA:
// 0 MMA loop total, 1 MMA wait W, 2 MMA wait aggregated operand, 3 MMA wait h operand, 4 MMA wait accumulator,
// 5 producer wait W slot, 6 producer wait h slot, 7 aggregation warp 0 total, 8 its wait for operand slots, 9 its wait
// for the tile descriptor, 10 its aggregation work, 11 stager (direction 0) wait for a descriptor buffer, 12 its staging
// work, 13 epilogue warp 0 wait for the accumulator, 14 epilogue total
__device__ unsigned long long g_fused_prof[160 * 16];

namespace {

using namespace tc;

constexpr int BK = 32;                       // k-block width: 64-byte rows, SWIZZLE_64B
constexpr int kAggWarps = 4;
constexpr int kConsWarps = 8;                // two consumer warpgroups
constexpr int kFirstCons = 4, kFirstAgg = 12;
constexpr int kThreads = (kFirstAgg + kAggWarps) * 32;      // 512
constexpr int kQuadsPerWarp = BM / 4 / kAggWarps;           // 8: an aggregation warp owns 32 tile rows
// setmaxnreg budget: 512 x 128 at launch = 128 x 40 (control) + 256 x 200 (consumers) + 128 x 72 (aggregation)
constexpr int kLaunchRegs = 128, kControlRegs = 40, kConsRegs = 200, kAggRegs = 72;
static_assert(kControlRegs <= kLaunchRegs && kAggRegs <= kLaunchRegs && kConsRegs >= kLaunchRegs,
              "setmaxnreg: control and aggregation warpgroups shrink (.dec), consumers grow (.inc)");
static_assert(128 * (kControlRegs + kAggRegs) + 256 * kConsRegs <= kThreads * kLaunchRegs, "register budget");
constexpr int kNW = 3;                       // W ring stages
constexpr int kECap = 1024;                  // staged in-edges per direction per tile (mean 512 at cfg2); rest: slow path
constexpr int kXCols = 224;                  // instruction columns kept per question: 7 groups of 32 (zero padded)
constexpr int kPnRowBytes = 1024;            // padded relation table: 256 fp32 per row (gr_pad_table256)
constexpr int kABytes = BM * BK * 2;         // one bf16 plane of an A slot: 8 KB
constexpr int kOutBytes = 2 * kStageOutBytes;               // epilogue staging: 8 KB per consumer warpgroup

struct FDir {
  const int32_t* rowptr;
  const int32_t* src;
  const int32_t* rel;
  const float* w;          // optional per-edge weights (normalized_gnn)
  const char* pn;          // zero-padded relation table [R1, 256] fp32
};

// Slot-major "quad ELL" form of both CSRs, built ONCE per batch (fused_ell_build_kernel): for every 128-row tile and
// direction a block of entries, quad Q (4 consecutive rows) owning m_Q = max in-degree of its rows slots, slot k of row r
// at block offset qoff[Q] + 4k + r.  Static per batch: source node, relation table byte offset and edge weight of every
// entry (padding entries: node -1, offset 0, weight 0).  The fused kernel's stagers move a tile's entries into shared
// memory with one bulk copy per direction and replace the node by c_f = prior[node] there (26 independent L2 gathers per
// lane and tile); graphs with edge weights (c_f = w (w prior[src]), normalized_gnn) take one streaming pass per layer
// instead (fused_coef_kernel) -- no per-layer index arithmetic inside the fused kernel either way.
constexpr int kQRow = BM / 4 + 4;     // per (direction, tile): 32 quad offsets, [32] = entries of the tile, [33] = block base
struct EllView {
  int32_t* counters;                  // [2] entries allocated per direction (atomic bump allocator of the build)
  int32_t* qrow;                      // [2][ntiles][kQRow]
  int2* ent;                          // [2][cap] static {table byte offset, source node | -1 for a padding entry}
  float* w;                           // [2][cap] edge weights (graphs with normalized_gnn weights only)
  int2* rc;                           // [2][cap] per-layer {off, c} (weighted graphs: fused_coef_kernel)
  int weighted;                       // 0: c_f = prior[src], computed by the kernel's stagers from `ent`
  int64_t cap;
  int ntiles;
};

struct FParams {
  FDir dir[2];
  EllView ell;
  const float* prior;      // [Nt]
  const float* ins;        // [B, I, D]
  const float* bias;
  float* C;                // optional fp32 output [Nt, N]
  int64_t ldc;
  const float* w_score;
  float* dots;             // [2 * Nt]: dots[m] = score dot, dots[Nt + m] = 0 (layout of gr_linear_tc_planes)
  int M, N, n_pad, D, B, Nq, G, ksteps_last, num_tiles;
  int has_planes;
  uint32_t flags;
  int debug;
};

// Tile descriptor the edge stager hands to the aggregation warps.  The in-edges are staged SLOT-MAJOR per quad of 4
// consecutive rows: quad Q (rows 4Q .. 4Q+3) owns m_Q = max in-degree of its rows slots; slot k of row r sits at entry
// qbase[Q] + 4k + r and is {table byte offset rel * 1024, c_f}, or {0, 0} when row r has fewer than k+1 in-edges (a
// gather of table row 0 weighted by zero).  A quarter-warp (8 lanes x 4 columns) owns a row, one warp-wide 16-byte load
// gathers one in-edge of each row of the quad, and the loop over slots has a warp-uniform trip count with no predicates.
template <int NI>
struct alignas(16) ETile {
  int2 rc[2][kECap];
  float x[2][NI][2][kXCols];          // relu(+x)/2 | relu(-x)/2 of the instruction vectors of the tile's two questions
  int32_t rowptr[2][BM + 4];          // global edge indices (slow path, and the stager's own row lookup)
  int32_t qbase[2][kQRow];            // entry offset of each quad's block, [BM/4] = total entries (bulk copy of the ELL row)
  int32_t nrows, lr_switch, fits[2];
  int2 zero_entry[2];                 // {0, 0}: what the slots beyond a quad's block read (c = 0: contributes nothing)
};

template <int NI>
constexpr size_t fused_smem_bytes(int np) {
  return 1024 /*align slack*/ + (size_t)(2 * NI + 1) * 2 * kABytes + (size_t)kNW * 2 * np * BK * 2 + kOutBytes +
         2 * sizeof(ETile<NI>) + 64 * 8 + 2 * 256 * 4;
}

// W [N, (2I+1)*D] fp32 -> hi/lo planes [N, nkb*32] in the kernel's K order (see the header comment); nkb < G*T: the
// packed walk of GroupedK (wgmma.cuh), whose last I k-blocks hold the last group of two neighbour slots each
__global__ void fused_w_split_kernel(const float* __restrict__ W, int64_t ldw, int N, int D, int I, int G, int nkb,
                                     __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int T = 2 * I + 1;
  const int64_t Kp = (int64_t)nkb * BK;
  const int64_t total = (int64_t)N * Kp;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / Kp;
    const int k = (int)(i - n * Kp);
    int blk = k / BK, c = k % BK;
    if (nkb != G * T && blk > (G - 1) * T) {                 // packed tail block i: slots 2i | 2i + 1 of the last group
      blk = (G - 1) * T + 1 + 2 * (blk - (G - 1) * T - 1) + c / 16;
      c %= 16;
    }
    const int g = blk / T, t = blk % T;
    // t == 0: the h segment;  t >= 1: Y(dir = (t-1) / I, j = (t-1) % I) -> segment 1 + 2j + dir
    const int seg = t == 0 ? 0 : 1 + 2 * ((t - 1) % I) + (t - 1) / I;
    const int col = g * BK + c;
    const float v = col < D ? __ldg(W + n * ldw + (int64_t)seg * D + col) : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

#ifndef GR_FUSED_WATCHDOG
#define GR_FUSED_WATCHDOG 0          // debug aid: a wait that lasts > 2 s reports its barrier and traps instead of hanging
#endif

__device__ __forceinline__ uint64_t global_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// `tag` identifies the waiting site in the watchdog report
#ifndef GR_FUSED_PROFILE
#define GR_FUSED_PROFILE 0           // 1: compile the per-role wait-cycle counters in (fused_debug bit 32; costs registers)
#endif
struct Prof {                                   // cycle accumulation for one role (only when debug bit 32 is set)
#if GR_FUSED_PROFILE
  bool on;
  long long acc[4];
  __device__ __forceinline__ void init(bool enable) { on = enable; acc[0] = acc[1] = acc[2] = acc[3] = 0; }
  __device__ __forceinline__ long long t() const { return on ? clock64() : 0; }
  __device__ __forceinline__ void add(int i, long long t0) { if (on) acc[i] += clock64() - t0; }
  __device__ __forceinline__ void store(int slot0, int n) const {
    if (on) for (int i = 0; i < n; ++i) g_fused_prof[(blockIdx.x % 160) * 16 + slot0 + i] = (unsigned long long)acc[i];
  }
  __device__ __forceinline__ void total(int slot, long long t0) const {
    if (on) g_fused_prof[(blockIdx.x % 160) * 16 + slot] = (unsigned long long)(clock64() - t0);
  }
#else
  __device__ __forceinline__ void init(bool) {}
  __device__ __forceinline__ long long t() const { return 0; }
  __device__ __forceinline__ void add(int, long long) {}
  __device__ __forceinline__ void store(int, int) const {}
  __device__ __forceinline__ void total(int, long long) const {}
#endif
};

__device__ __forceinline__ void mbar_wait_sleep(uint64_t* bar, uint32_t parity, int tag = 0, unsigned backoff_ns = 0) {
  uint32_t ok = 0;
#if GR_FUSED_WATCHDOG
  uint64_t t0 = 0;
  uint32_t spins = 0;
#endif
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(20000u)
        : "memory");
    // the hardware suspend returns after ~100 cycles whatever the hint says: back off explicitly so that waiting roles
    // do not spend the issue slots the working warps need
    if (!ok && backoff_ns) __nanosleep(backoff_ns);
#if GR_FUSED_WATCHDOG
    if (!ok && (++spins & 1023u) == 0) {
      const uint64_t t = global_ns();
      if (t0 == 0) t0 = t;
      else if (t - t0 > 2000000000ull) {
        printf("fused_layer watchdog: block %d warp %d lane %d tag %d parity %u\n", (int)blockIdx.x,
               (int)(threadIdx.x >> 5), (int)(threadIdx.x & 31), tag, parity);
        __trap();
      }
    }
#endif
  }
}

__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(c0), "r"(c1)
               : "memory");
}
// explicit shared-state-space accesses (the carve-up of the dynamic buffer goes through integer alignment, after
// which the compiler would fall back to generic loads / stores)
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}

// ---------------------------------------------------------------------------------------------------------
// edge stager (one warp): tile descriptor of tile `tile` into `et`
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// Stager warp `d` (0: also the tile header and the instruction vectors) fills direction d of the tile descriptor: the
// quad offsets and the tile's {offset, c} entries are bulk-copied from the per-layer ELL arrays; completion is counted
// on the descriptor's full barrier (expect_tx), on which lane 0 arrives once for the warp.
template <int NI>
__device__ __forceinline__ void stage_tile(ETile<NI>& et, const FParams& p, int tile, int lane, int d, uint64_t* full,
                                           uint64_t* own, uint32_t& own_uses) {
  const int64_t r0 = (int64_t)tile * BM;
  const int nrows = tile < p.num_tiles ? (int)min((int64_t)BM, (int64_t)p.M - r0) : 0;
  int total = 0, base = 0;
  if (nrows > 0 && lane == 0) {
    const int32_t* qr = p.ell.qrow + ((int64_t)d * p.ell.ntiles + tile) * kQRow;
    total = __ldg(qr + BM / 4);
    base = __ldg(qr + BM / 4 + 1);
  }
  total = __shfl_sync(0xffffffffu, total, 0);
  base = __shfl_sync(0xffffffffu, base, 0);
  const bool fits = total <= kECap && base >= 0 && !(p.debug & 2);
  if (lane == 0) {
    et.fits[d] = fits ? 1 : 0;
    if (d == 0) {
      et.nrows = nrows;
      const int b0 = nrows > 0 ? (int)(r0 / p.Nq) : 0;
      et.lr_switch = p.Nq - (int)(r0 - (int64_t)b0 * p.Nq);       // first tile row of question b0 + 1 (Nq >= BM)
      et.zero_entry[0] = make_int2(0, 0);
    }
  }
  uint32_t tx = 0;
  if (nrows > 0) {
    if (d == 0) {
      const int b0 = (int)(r0 / p.Nq);
      for (int i = lane; i < 2 * NI * kXCols; i += 32) {
        const int c = i % kXCols, j = (i / kXCols) % NI, q = i / (kXCols * NI);
        const int b = b0 + q;
        const float v = (c < p.D && b < p.B) ? __ldg(p.ins + ((int64_t)b * NI + j) * p.D + c) : 0.f;
        et.x[q][j][0][c] = 0.5f * fmaxf(v, 0.f);
        et.x[q][j][1][c] = 0.5f * fmaxf(-v, 0.f);
      }
    }
    if (!fits) {
      // slow path of this tile / direction: the aggregation warps walk the CSR themselves, they need the row pointers
      const int32_t* rp = p.dir[d].rowptr + r0;
#pragma unroll
      for (int k = 0; k < (BM + 32) / 32; ++k) {
        const int i = lane + 32 * k;
        if (i <= BM) et.rowptr[d][i] = __ldg(rp + min(i, nrows));
      }
    }
  }
  __syncwarp();                                                  // the lanes' descriptor stores precede lane 0's arrival
  if (nrows > 0 && fits && !p.ell.weighted) {
    // unweighted graph: copy the static {offset, node} entries to this warp's own barrier, then c_f = prior[node] in place
    if (lane == 0) {
      const int32_t* qr = p.ell.qrow + ((int64_t)d * p.ell.ntiles + tile) * kQRow;
      mbar_expect_tx(own, (uint32_t)(kQRow * 4) + (uint32_t)total * 8u);
      bulk_g2s(smem_u32(&et.qbase[d][0]), qr, (uint32_t)(kQRow * 4), own);
      if (total > 0) bulk_g2s(smem_u32(&et.rc[d][0]), p.ell.ent + (int64_t)d * p.ell.cap + base, (uint32_t)total * 8u, own);
    }
    mbar_wait_sleep(own, own_uses & 1, 8, 100);
    ++own_uses;
    const uint32_t rc_s = smem_u32(&et.rc[d][0]) + 4u;           // the node / coefficient word of entry 0
    for (int i0 = 0; i0 < total; i0 += 256) {
      int node[8];
      float c[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int i = i0 + lane + 32 * u;
        node[u] = i < total ? (int)lds_u32(rc_s + (uint32_t)i * 8u) : -1;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) c[u] = node[u] >= 0 ? __ldg(p.prior + node[u]) : 0.f;   // w = 1: c_f = 1 * (1 * prior)
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int i = i0 + lane + 32 * u;
        if (i < total) asm volatile("st.shared.f32 [%0], %1;" ::"r"(rc_s + (uint32_t)i * 8u), "f"(c[u]) : "memory");
      }
    }
    __syncwarp();
  } else if (lane == 0 && nrows > 0 && fits) {
    const int32_t* qr = p.ell.qrow + ((int64_t)d * p.ell.ntiles + tile) * kQRow;
    tx = (uint32_t)(kQRow * 4) + (uint32_t)total * 8u;
    mbar_expect_tx(full, tx);
    bulk_g2s(smem_u32(&et.qbase[d][0]), qr, (uint32_t)(kQRow * 4), full);
    if (total > 0) bulk_g2s(smem_u32(&et.rc[d][0]), p.ell.rc + (int64_t)d * p.ell.cap + base, (uint32_t)total * 8u, full);
  }
  if (lane == 0 && tx == 0) mbar_arrive(full);                   // (with tx > 0 the expect_tx above was the arrival)
}

// ---------------------------------------------------------------------------------------------------------
// aggregation: one pass = (direction d, column group g) for this warp's 8 rows (2 quads) -> I A-operand blocks
// ---------------------------------------------------------------------------------------------------------
// (ld.global.nc.L1::no_allocate for this gather was measured: 489 us instead of 270 -- even the ~28 KB of L1 left next to
// 226 KB of shared memory serve enough of the quads' repeated table lines to matter)
// (also measured: an L2 evict_last policy on this gather (createpolicy + ld.global.nc.L2::cache_hint) to keep the 12.5 MB
// of relation tables resident against the 212 MB of h planes streaming through L2 -- 276 us instead of 270, no gain)
__device__ __forceinline__ float4 ldg4(const char* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 lds_f4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ uint2 lds_u2(uint32_t a) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts_u2(uint32_t a, uint32_t x, uint32_t y) {
  asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory");
}

struct Acc4 {                                   // S = sum c*v, Q = sum c*|v| for this lane's 4 columns
  float2 s0, s1, q0, q1;
  __device__ __forceinline__ void clear() { s0 = s1 = q0 = q1 = make_float2(0.f, 0.f); }
  __device__ __forceinline__ void add(float c, const float4& v) {
    const float2 cc = make_float2(c, c);
    s0 = ffma2(cc, make_float2(v.x, v.y), s0);
    s1 = ffma2(cc, make_float2(v.z, v.w), s1);
    q0 = ffma2(cc, make_float2(fabsf(v.x), fabsf(v.y)), q0);
    q1 = ffma2(cc, make_float2(fabsf(v.z), fabsf(v.w)), q1);
  }
};

// y = xp * (Q + S) + xn * (Q - S) for 4 columns (xp = relu(x)/2, xn = relu(-x)/2), split into bf16 hi / lo, 8-byte
// stores into the K-major SWIZZLE_64B operand tile
__device__ __forceinline__ void emit_quad(uint32_t slot, const float4& xp, const float4& xn, const float2& U0,
                                          const float2& U1, const float2& V0, const float2& V1) {
  const float2 xp0 = make_float2(xp.x, xp.y), xp1 = make_float2(xp.z, xp.w);
  const float2 xn0 = make_float2(xn.x, xn.y), xn1 = make_float2(xn.z, xn.w);
  float2 y0 = fmul2(xp0, U0), y1 = fmul2(xp1, U1);
  y0 = ffma2(xn0, V0, y0);
  y1 = ffma2(xn1, V1, y1);
  const __nv_bfloat162 h0 = __floats2bfloat162_rn(y0.x, y0.y), h1 = __floats2bfloat162_rn(y1.x, y1.y);
  const uint32_t u0 = *reinterpret_cast<const uint32_t*>(&h0), u1 = *reinterpret_cast<const uint32_t*>(&h1);
  const float2 f0 = make_float2(__uint_as_float(u0 << 16), __uint_as_float(u0 & 0xffff0000u));
  const float2 f1 = make_float2(__uint_as_float(u1 << 16), __uint_as_float(u1 & 0xffff0000u));
  const float2 m1 = make_float2(-1.f, -1.f);
  const float2 r0 = ffma2(f0, m1, y0), r1 = ffma2(f1, m1, y1);
  const __nv_bfloat162 l0 = __floats2bfloat162_rn(r0.x, r0.y), l1 = __floats2bfloat162_rn(r1.x, r1.y);
  sts_u2(slot, u0, u1);
  sts_u2(slot + kABytes, *reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
}

template <int NI>
__device__ __forceinline__ void agg_pass(const ETile<NI>& et, const FParams& p, int d, int g, int wa, int lane,
                                         uint32_t a_slots) {
  const int r = lane >> 3, c8 = lane & 7;                    // row of the quad, 4-column group of the 32-column block
  const uint32_t et_s = smem_u32(&et);
  const int nrows = (int)lds_u32(et_s + (uint32_t)offsetof(ETile<NI>, nrows));
  const int lr_switch = (int)lds_u32(et_s + (uint32_t)offsetof(ETile<NI>, lr_switch));
  const bool fits = lds_u32(et_s + (uint32_t)offsetof(ETile<NI>, fits) + (uint32_t)d * 4u) != 0;
  const FDir& dd = p.dir[d];
  const char* tb = dd.pn + (g * BK + 4 * c8) * 4;
  const uint32_t qb_s = et_s + (uint32_t)offsetof(ETile<NI>, qbase) + (uint32_t)d * (BM / 4 + 4) * 4u;
  const uint32_t rc_s = et_s + (uint32_t)d * kECap * 8u + (uint32_t)r * 8u;
  const uint32_t xs = et_s + (uint32_t)offsetof(ETile<NI>, x) + (uint32_t)((g * BK + 4 * c8) * 4);
  const float2 one = make_float2(1.f, 1.f), mone = make_float2(-1.f, -1.f);
#pragma unroll 1
  for (int qd = 0; qd < kQuadsPerWarp; ++qd) {
    const int quad = wa * kQuadsPerWarp + qd;
    const int lr = quad * 4 + r;
    if (quad * 4 >= nrows) break;                            // warp uniform
    Acc4 acc;
    acc.clear();
    if (fits) {
      const int qb = (int)lds_u32(qb_s + (uint32_t)quad * 4u);
      int m = ((int)lds_u32(qb_s + (uint32_t)quad * 4u + 4u) - qb) >> 2;     // slots of this quad (warp uniform)
      uint32_t es = rc_s + (uint32_t)qb * 8u;
      const uint32_t zs = et_s + (uint32_t)offsetof(ETile<NI>, zero_entry);
      for (; m > 0; m -= 8, es += 8 * 32) {
        // 8 slots per round, no predicates: slots past the quad's block read the zero entry (table row 0 x 0)
        float4 v[8];
        float c[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint2 e = lds_u2(k < m ? es + (uint32_t)k * 32u : zs);
          c[k] = __uint_as_float(e.y);
          v[k] = ldg4(tb + e.x);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) acc.add(c[k], v[k]);
      }
    } else if (lr < nrows) {
      // slow path (the tile's slot-major blocks overflow the staging buffer): every lane walks its own row in the CSR
      const uint32_t rp_s = et_s + (uint32_t)offsetof(ETile<NI>, rowptr) + (uint32_t)d * (BM + 4) * 4u;
      const int beg = (int)lds_u32(rp_s + (uint32_t)lr * 4u), end = (int)lds_u32(rp_s + (uint32_t)lr * 4u + 4u);
      for (int e = beg; e < end; ++e) {
        const float w = dd.w ? dd.w[e] : 1.0f;
        const float c = w * (w * p.prior[dd.src[e]]);
        acc.add(c, ldg4(tb + (uint32_t)dd.rel[e] * (uint32_t)kPnRowBytes));
      }
    }
    if (lr < nrows) {
      const float2 U0 = ffma2(acc.s0, one, acc.q0), V0 = ffma2(acc.s0, mone, acc.q0);
      const float2 U1 = ffma2(acc.s1, one, acc.q1), V1 = ffma2(acc.s1, mone, acc.q1);
      const int q = lr >= lr_switch ? 1 : 0;
      const uint32_t off = (uint32_t)lr * 64u + ((uint32_t)((c8 >> 1) ^ ((lr >> 1) & 3)) << 4) + (uint32_t)(c8 & 1) * 8u;
#pragma unroll
      for (int j = 0; j < NI; ++j) {
        const float4 xp = lds_f4(xs + (uint32_t)(((q * NI + j) * 2) * kXCols * 4));
        const float4 xn = lds_f4(xs + (uint32_t)(((q * NI + j) * 2 + 1) * kXCols * 4));
        emit_quad(a_slots + (uint32_t)((d * NI + j) * 2 * kABytes) + off, xp, xn, U0, U1, V0, V1);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------------------------------------
template <int NI, int NP, int CS>   // NP: accumulator width (W tile rows), n_pad rounded up to 64, 128, 208 or 224
__global__ void __launch_bounds__(kThreads, 1)
fused_layer_kernel(const __grid_constant__ CUtensorMap map_h_hi, const __grid_constant__ CUtensorMap map_h_lo,
                   const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                   const __grid_constant__ CUtensorMap map_c, const __grid_constant__ CUtensorMap map_c_hi,
                   const __grid_constant__ CUtensorMap map_c_lo, const FParams p) {
  constexpr int T = 2 * NI + 1;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int w_bytes = NP * BK * 2;
  uint8_t* a_slots = smem;                                        // [T] x {hi 8 KB, lo 8 KB}
  uint8_t* w_ring = a_slots + (size_t)T * 2 * kABytes;            // [kNW] x {W_hi, W_lo}
  uint8_t* s_out = w_ring + (size_t)kNW * 2 * w_bytes;            // epilogue staging: [2 consumer warpgroups]
  ETile<NI>* etile = reinterpret_cast<ETile<NI>*>(s_out + kOutBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(etile) + 2 * sizeof(ETile<NI>));
  uint64_t* wfull = bars;                 // [kNW]
  uint64_t* wempty = wfull + kNW;         // [kNW]
  uint64_t* afull = wempty + kNW;         // [T]
  uint64_t* aempty = afull + T;           // [T]
  uint64_t* efull = aempty + T;           // [2]
  uint64_t* eempty = efull + 2;           // [2]
  uint64_t* sbar = eempty + 2;            // [2] one per stager warp: its own bulk copies
  float* s_bias = reinterpret_cast<float*>(bars + 64);            // [256]
  float* s_ws = s_bias + 256;                                     // [256]
  for (int i = threadIdx.x; i < 256; i += kThreads) {
    s_bias[i] = (p.bias && i < p.N) ? p.bias[i] : 0.f;
    s_ws[i] = (p.w_score && i < p.N) ? p.w_score[i] : 0.f;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int crank = CS > 1 ? (int)cluster_ctarank() : 0;
  const int ncluster = gridDim.x / CS, cid = blockIdx.x / CS;
  const int ngroups = (p.num_tiles + CS - 1) / CS;
  constexpr uint16_t kMask = (uint16_t)((1u << CS) - 1);
  const int G = p.G;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kNW; ++s) { mbar_init(&wfull[s], 1); mbar_init(&wempty[s], kConsWarps * CS); }
    for (int t = 0; t < T; ++t) { mbar_init(&afull[t], t == T - 1 ? 1 : kAggWarps); mbar_init(&aempty[t], kConsWarps); }
    for (int a = 0; a < 2; ++a) { mbar_init(&efull[a], 2); mbar_init(&eempty[a], kAggWarps); mbar_init(&sbar[a], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (CS > 1) cluster_sync_all();

  // register file: kThreads x kLaunchRegs at launch = the CTA's pool; the control and aggregation warpgroups hand back
  // what the two consumer warpgroups (register accumulators) take.  setmaxnreg.inc only draws on registers released
  // inside the CTA.  (The instruction sits at the top of each role's branch: ptxas
  // budgets the code it dominates.)
  if (warp < kFirstCons) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kControlRegs));
    if (warp == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      Prof pf; pf.init(p.debug & 32);
      uint32_t wphase = 0, grp = 0;
      int ws = 0;
      constexpr int w_rows = NP / CS;
      constexpr int w_slice = w_rows * BK * 2;
      for (int tg = cid; tg < ngroups; tg += ncluster) {
        const int m0 = (tg * CS + crank) * BM;
        // the h planes come from HBM: pull the NEXT tile's blocks into L2 now, so that their TMA loads (issued only
        // ~3 k-blocks ahead of the MMA) see L2 latency
        if (tg + ncluster < ngroups) {
          const int m1 = ((tg + ncluster) * CS + crank) * BM;
          for (int g = 0; g < G; ++g) {
            tma_prefetch_2d(&map_h_hi, g * BK, m1);
            tma_prefetch_2d(&map_h_lo, g * BK, m1);
          }
        }
        for (int g = 0; g < G; ++g, ++grp) {
          for (int t = 0; t < T; ++t) {
            const int kcol = (g * T + t) * BK;
            { const long long t0 = pf.t(); mbar_wait_sleep(&wempty[ws], wphase ^ 1, 1); pf.add(0, t0); }
            uint8_t* st = w_ring + (size_t)ws * 2 * w_bytes;
            if (p.debug & 8) {                                   // timing experiment: no W traffic
              mbar_arrive(&wfull[ws]);
            } else {
            mbar_expect_tx(&wfull[ws], (uint32_t)(2 * w_bytes));
            if (CS == 1) {
              tma_load_2d(st, &map_w_hi, &wfull[ws], kcol, 0);
              tma_load_2d(st + w_bytes, &map_w_lo, &wfull[ws], kcol, 0);
            } else {
              tma_load_2d_mc(st + crank * w_slice, &map_w_hi, &wfull[ws], kcol, crank * w_rows, kMask);
              tma_load_2d_mc(st + w_bytes + crank * w_slice, &map_w_lo, &wfull[ws], kcol, crank * w_rows, kMask);
            }
            }
            if (++ws == kNW) { ws = 0; wphase ^= 1; }
            if (t == 0) {                                          // the h block leads its group (operand slot T-1)
              { const long long t0 = pf.t(); mbar_wait_sleep(&aempty[T - 1], (grp & 1) ^ 1, 2); pf.add(1, t0); }
              uint8_t* as = a_slots + (size_t)(T - 1) * 2 * kABytes;
              mbar_expect_tx(&afull[T - 1], (uint32_t)(2 * kABytes));
              tma_load_2d(as, &map_h_hi, &afull[T - 1], g * BK, m0);
              tma_load_2d(as + kABytes, &map_h_lo, &afull[T - 1], g * BK, m0);
            }
          }
        }
      }
      pf.store(5, 2);
    }
  } else if (warp >= 2) {
    // ===================== edge stagers: warp 3 direction 0 (+ header, instructions), warp 2 direction 1 ==========
    Prof pf; pf.init((p.debug & 32) && warp == 3 && lane == 0);
    uint32_t own_uses = 0;
    int it = 0;
    for (int tg = cid; tg < ngroups; tg += ncluster, ++it) {
      const int eb = it & 1;
      long long t0 = pf.t();
      if (it >= 2) mbar_wait_sleep(&eempty[eb], ((it >> 1) - 1) & 1, 5, 500);
      pf.add(0, t0);
      t0 = pf.t();
      stage_tile<NI>(etile[eb], p, tg * CS + crank, lane, 3 - warp, &efull[eb], &sbar[3 - warp], own_uses);
      pf.add(1, t0);
    }
    pf.store(11, 2);
  }
  } else if (warp >= kFirstAgg) {
    // ===================== aggregation warps =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kAggRegs));   // kAggRegs < kLaunchRegs
    const int wa = warp - kFirstAgg;
    Prof pf; pf.init((p.debug & 32) && wa == 0 && lane == 0);
    const long long t_all = pf.t();
    uint32_t grp = 0;
    int it = 0;
    for (int tg = cid; tg < ngroups; tg += ncluster, ++it) {
      const int eb = it & 1;
      { const long long t0 = pf.t(); mbar_wait_sleep(&efull[eb], (it >> 1) & 1, 6, 200); pf.add(1, t0); }
      const ETile<NI>& et = etile[eb];
      for (int g = 0; g < G; ++g, ++grp) {
#pragma unroll
        for (int d = 0; d < 2; ++d) {
          long long t0 = pf.t();
#pragma unroll
          for (int j = 0; j < NI; ++j) mbar_wait_sleep(&aempty[d * NI + j], (grp & 1) ^ 1, 20 + d * NI + j, 0);
          pf.add(0, t0);
          t0 = pf.t();
          if (!(p.debug & 1)) agg_pass<NI>(et, p, d, g, wa, lane, smem_u32(a_slots));
          pf.add(2, t0);
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) {
#pragma unroll
            for (int j = 0; j < NI; ++j) mbar_arrive(&afull[d * NI + j]);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&eempty[eb]);
    }
    pf.total(7, t_all);
    pf.store(8, 3);
  } else {
    // ===================== consumers: wgmma over the tile's k-blocks, then the epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsRegs));
    const int cw = (warp - kFirstCons) >> 2, wq = warp & 3;     // consumer warpgroup (row half), warp inside it
    // 512 threads launch with 128 registers each, and ptxas allocates every role within that (setmaxnreg only moves
    // registers at run time): an accumulator operand wider than 128 columns does not fit one wgmma instruction
    constexpr int kInstrCols = NP <= 128 ? NP : 32;
    const EpiOut e{s_bias, s_ws, (p.flags & GR_LINEAR_RELU) != 0};
    const int r = wq * 16 + (lane >> 2), cq = lane & 3;
    uint8_t* stg = s_out + (size_t)cw * kStageOutBytes;
    const bool issuer = wq == 0 && lane == 0;
    Prof pf; pf.init((p.debug & 32) && cw == 0 && issuer);
    const long long t_all = pf.t();
    uint32_t wphase = 0, grp = 0;
    int ws = 0;
    for (int tg = cid; tg < ngroups; tg += ncluster) {
      const int tile = tg * CS + crank;
      float acc[NP / 2];
#pragma unroll
      for (int i = 0; i < NP / 2; ++i) acc[i] = 0.f;
      int prev_ws = -1, prev_sl = -1;
      for (int g = 0; g < G; ++g, ++grp) {
        // the last column group of a 16-column-padded segment holds one k-step: its own straight-line batch
        static_assert(BK / MMA_K == 2, "a k-block is one or two k-steps");
        const bool half = g == G - 1 && p.ksteps_last == 1;
        for (int t = 0; t < T; ++t) {
          const int sl = t == 0 ? T - 1 : t - 1;              // operand slot of block t (slot T-1 = the h block)
          { const long long t0 = pf.t(); mbar_wait_sleep(&wfull[ws], wphase, 4); pf.add(0, t0); }
          { const long long t0 = pf.t(); mbar_wait_sleep(&afull[sl], grp & 1, 10 + sl); pf.add(t == 0 ? 2 : 1, t0); }
          const uint32_t sa = smem_u32(a_slots + (size_t)sl * 2 * kABytes) + (uint32_t)(cw * WG_M * BK * 2);
          const uint32_t sw = smem_u32(w_ring + (size_t)ws * 2 * w_bytes);
          const uint64_t da_hi = make_smem_desc<BK>(sa), da_lo = make_smem_desc<BK>(sa + kABytes);
          const uint64_t dw_hi = make_smem_desc<BK>(sw), dw_lo = make_smem_desc<BK>(sw + w_bytes);
          if (half) mma_kblock<NP, BK, 1, false, kInstrCols>(acc, da_hi, da_lo, dw_hi, dw_lo);
          else mma_kblock<NP, BK, 2, false, kInstrCols>(acc, da_hi, da_lo, dw_hi, dw_lo);
          wgmma_wait<1>();                                     // the previous k-block is done: free its W and A slots
          if (prev_ws >= 0 && lane == 0) { release_slot<CS>(&wempty[prev_ws]); mbar_arrive(&aempty[prev_sl]); }
          prev_ws = ws; prev_sl = sl;
          if (++ws == kNW) { ws = 0; wphase ^= 1; }
        }
      }
      wgmma_wait<0>();
      if (prev_ws >= 0 && lane == 0) { release_slot<CS>(&wempty[prev_ws]); mbar_arrive(&aempty[prev_sl]); }

      const int64_t row0 = (int64_t)tile * BM + cw * WG_M + r;
      float dot0 = 0.f, dot1 = 0.f;
      const bool store = !(p.debug & 4);
#pragma unroll
      for (int q = 0; q < NP / 16; ++q) {
        const int c0 = 16 * q;
        if (c0 >= p.n_pad) continue;
        float v[8];
        epi_values(acc, q, cq, e, v, dot0, dot1);
        epi_store_tma(v, stg, r, cq, issuer, 1 + cw, &map_c, &map_c_hi, &map_c_lo, store && p.C != nullptr,
                      store && p.has_planes, c0, tile * BM + cw * WG_M);
      }
      epi_dots(dot0, dot1, p.dots, row0, p.M, cq);
    }
    if (issuer) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    pf.total(0, t_all);
    pf.store(1, 4);
  }
  __syncthreads();
  if (CS > 1) cluster_sync_all();
}

// ---------------------------------------------------------------------------------------------------------
// per batch: quad-ELL build.  grid = (ntiles, 2 directions), 128 threads = the rows of the tile
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BM) fused_ell_build_kernel(FDir d0, FDir d1, EllView ell, int64_t Nt) {
  const int tile = blockIdx.x, d = blockIdx.y;
  const FDir dd = d == 0 ? d0 : d1;
  const int64_t r0 = (int64_t)tile * BM;
  const int r = threadIdx.x, lane = r & 31, warp = r >> 5;
  const int64_t row = r0 + r;
  int beg = 0, deg = 0;
  if (row < Nt) {
    beg = dd.rowptr[row];
    deg = dd.rowptr[row + 1] - beg;
  }
  int m = max(deg, __shfl_xor_sync(0xffffffffu, deg, 1));
  m = max(m, __shfl_xor_sync(0xffffffffu, m, 2));                 // slots of this row's quad
  __shared__ int s_q[BM / 4 + 1];
  __shared__ int s_base;
  if ((r & 3) == 0) s_q[r >> 2] = 4 * m;
  __syncthreads();
  if (warp == 0) {                                                // exclusive scan over the 32 quads
    const int v = s_q[lane];
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    s_q[lane] = incl - v;
    if (lane == 31) {
      s_q[32] = incl;
      int base = -1;
      if (incl <= kECap) {                                        // larger tiles take the fused kernel's slow path
        base = atomicAdd(ell.counters + d, incl);
        if ((int64_t)base + incl > ell.cap) base = -1;            // arrays full (cannot happen with cap >= 4 F): slow path
      }
      s_base = base;
    }
  }
  __syncthreads();
  int32_t* qr = ell.qrow + ((int64_t)d * ell.ntiles + tile) * kQRow;
  if (r <= 32) qr[r] = s_q[r];
  if (r == 33) qr[33] = s_base;
  if (r > 33 && r < kQRow) qr[r] = 0;
  const int base = s_base;
  if (base < 0) return;
  const int64_t o = (int64_t)d * ell.cap + base + s_q[r >> 2] + (r & 3);
  for (int k = 0; k < m; ++k) {
    int sn = 0;
    uint32_t off = 0;
    float w = 0.f;
    if (k < deg) {
      sn = dd.src[beg + k];
      off = (uint32_t)dd.rel[beg + k] * (uint32_t)kPnRowBytes;
      w = dd.w ? dd.w[beg + k] : 1.0f;
    }
    ell.ent[o + 4 * k] = make_int2((int)off, k < deg ? sn : -1);
    if (ell.weighted) ell.w[o + 4 * k] = w;
  }
}

// per layer: rc[e] = {off[e], w (w prior[src[e]])} for the allocated entries of both directions (reasongnn.py:80-84)
__global__ void fused_coef_kernel(EllView ell, const float* __restrict__ prior) {
  const int d = blockIdx.y;
  const int n = min((int64_t)ell.counters[d], ell.cap);
  const int64_t o = (int64_t)d * ell.cap;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float w = ell.w[o + i];
    const int2 e = ell.ent[o + i];
    ell.rc[o + i] = make_int2(e.x, __float_as_int(w * (w * __ldg(prior + max(e.y, 0)))));      // padding: w = 0
  }
}

struct EllPlan {
  int64_t cap;
  int ntiles;
  size_t o_qrow, o_ent, o_w, o_rc, bytes;
};

EllPlan plan_ell(int64_t Nt, int64_t F) {
  EllPlan e{};
  e.ntiles = (int)ceil_div(Nt, BM);
  // sum over quads of 4 * max degree <= 4 F; typical graphs need ~1.6 F.  2 F + 4 Nt covers them, tiles that do not
  // fit any more fall back to the slow path of the fused kernel
  e.cap = (int64_t)align_up((size_t)(2 * F + 4 * Nt + 64), 64);
  size_t o = 256;
  e.o_qrow = o; o += align_up((size_t)2 * e.ntiles * kQRow * 4, 256);
  e.o_ent = o;  o += align_up((size_t)2 * e.cap * 8, 256);
  e.o_w = o;    o += align_up((size_t)2 * e.cap * 4, 256);
  e.o_rc = o;   o += align_up((size_t)2 * e.cap * 8, 256);
  e.bytes = o;
  return e;
}

EllView ell_view(void* blob, const EllPlan& e) {
  char* b = reinterpret_cast<char*>(blob);
  EllView v{};
  v.counters = reinterpret_cast<int32_t*>(b);
  v.qrow = reinterpret_cast<int32_t*>(b + e.o_qrow);
  v.ent = reinterpret_cast<int2*>(b + e.o_ent);
  v.w = reinterpret_cast<float*>(b + e.o_w);
  v.rc = reinterpret_cast<int2*>(b + e.o_rc);
  v.cap = e.cap;
  v.ntiles = e.ntiles;
  return v;
}

struct FusedPlan {
  bool ok;
  int n_pad, np, G, ksteps_last;   // np: instantiated accumulator width >= n_pad (W tile rows, zero filled beyond N)
  int64_t kp;                 // columns of the pre-formatted W planes
  size_t w_plane_bytes, smem_bytes;
};

FusedPlan plan_fused(int64_t Nq, int64_t D, int64_t pitch, int I, int64_t N_out) {
  FusedPlan f{};
  f.n_pad = (int)((N_out + 15) / 16 * 16);
  f.np = f.n_pad <= 64 ? 64 : f.n_pad <= 128 ? 128 : f.n_pad <= 208 ? 208 : 224;
  const GroupedK k = plan_grouped_k(pitch, I, N_out);
  f.G = k.G; f.ksteps_last = k.ksteps_last; f.kp = k.kp; f.w_plane_bytes = k.w_plane_bytes;
  f.smem_bytes = I == 2 ? fused_smem_bytes<2>(f.np) : fused_smem_bytes<1>(f.np);
  f.ok = (I == 1 || I == 2) && Nq >= BM && D >= 8 && D <= pitch && pitch % 16 == 0 && (pitch + BK - 1) / BK * BK <= kXCols &&
         N_out >= 8 && f.n_pad <= 224 && f.smem_bytes <= 227 * 1024 && get_encode_fn() != nullptr;
  return f;
}

template <int NI, int NP, int CS>
int launch_fused(const CUtensorMap& m_h_hi, const CUtensorMap& m_h_lo, const CUtensorMap& m_w_hi,
                 const CUtensorMap& m_w_lo, const CUtensorMap& m_c, const CUtensorMap& m_c_hi,
                 const CUtensorMap& m_c_lo, const FusedPlan& f, const FParams& p, cudaStream_t stream) {
  const int ngroups = (p.num_tiles + CS - 1) / CS;
  const int nclusters = std::max(1, std::min(ngroups, sm_count() / CS));
  return launch_cluster<fused_layer_kernel<NI, NP, CS>>("gr_fused_layer", kLaunchRegs, CS, nclusters * CS, kThreads,
                                                        f.smem_bytes, stream, m_h_hi, m_h_lo, m_w_hi, m_w_lo, m_c,
                                                        m_c_hi, m_c_lo, p);
}

template <int NP>
int launch_fused_np(const CUtensorMap* const (&m)[7], int I, int cs, const FusedPlan& f, const FParams& p,
                    cudaStream_t stream) {
  if (I == 2) {
    if (cs == 2) return launch_fused<2, NP, 2>(*m[0], *m[1], *m[2], *m[3], *m[4], *m[5], *m[6], f, p, stream);
    return launch_fused<2, NP, 1>(*m[0], *m[1], *m[2], *m[3], *m[4], *m[5], *m[6], f, p, stream);
  }
  if (cs == 2) return launch_fused<1, NP, 2>(*m[0], *m[1], *m[2], *m[3], *m[4], *m[5], *m[6], f, p, stream);
  return launch_fused<1, NP, 1>(*m[0], *m[1], *m[2], *m[3], *m[4], *m[5], *m[6], f, p, stream);
}

}  // namespace

namespace tc {

GroupedK plan_grouped_k(int64_t pitch, int I, int64_t N_out, bool packed) {
  GroupedK k{};
  k.G = (int)((pitch + BK - 1) / BK);
  k.ksteps_last = (int)((pitch - (int64_t)(k.G - 1) * BK) / MMA_K);
  k.nkb = packed && k.ksteps_last == 1 ? (k.G - 1) * (2 * I + 1) + 1 + I : k.G * (2 * I + 1);
  k.kp = (int64_t)k.nkb * BK;
  k.w_plane_bytes = align_up((size_t)N_out * k.kp * 2, 256);
  return k;
}

int grouped_w_split(const float* W, int64_t ldw, int64_t N_out, int D, int I, const GroupedK& k, __nv_bfloat16* hi,
                    __nv_bfloat16* lo, cudaStream_t stream) {
  const int64_t work = N_out * k.kp;
  const int grid = (int)std::min<int64_t>(ceil_div(work, 256), 32LL * sm_count());
  fused_w_split_kernel<<<grid, 256, 0, stream>>>(W, ldw, (int)N_out, D, I, k.G, k.nkb, hi, lo);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

}  // namespace tc
}  // namespace gr

extern "C" int gr_fused_profile_read(unsigned long long* out, int n) {
  using namespace gr;
  GR_CHECK_ARG(out && n > 0 && n <= 160 * 16, "bad buffer");
  GR_CHECK_CUDA(cudaMemcpyFromSymbol(out, g_fused_prof, sizeof(unsigned long long) * (size_t)n));
  return GR_OK;
}

extern "C" int gr_fused_layer_supported(int64_t N_nodes, int64_t D, int64_t seg_pitch, int I, int64_t N_out) {
  return gr::plan_fused(N_nodes, D, seg_pitch, I, N_out).ok ? 1 : 0;
}

extern "C" size_t gr_fused_layer_workspace_bytes(int64_t D, int64_t seg_pitch, int I, int64_t N_out) {
  if (D <= 0 || seg_pitch <= 0 || I <= 0 || N_out <= 0) return 0;
  return 2 * gr::plan_fused(gr::tc::BM, D, seg_pitch, I, N_out).w_plane_bytes;
}

extern "C" size_t gr_fused_ell_bytes(int B, int N_nodes, int64_t F) {
  if (B <= 0 || N_nodes <= 0 || F < 0) return 0;
  return gr::plan_ell((int64_t)B * N_nodes, F).bytes;
}

extern "C" int gr_fused_ell_build(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t, const float* w_t,
                                  const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h, const float* w_h,
                                  int B, int N_nodes, int64_t F, void* ell, size_t ell_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(rowptr_t && rowptr_h && ell, "null pointer");
  GR_CHECK_ARG(F == 0 || (src_t && rel_t && src_h && rel_h), "null edge arrays");
  GR_CHECK_ARG(B > 0 && N_nodes > 0, "sizes must be positive");
  const int64_t Nt = (int64_t)B * N_nodes;
  const EllPlan e = plan_ell(Nt, F);
  if (ell_bytes < e.bytes || (reinterpret_cast<uintptr_t>(ell) & 255) != 0) {
    set_error("gr_fused_ell_build: buffer too small (%zu < %zu) or not 256-byte aligned", ell_bytes, e.bytes);
    return GR_ERR_WORKSPACE;
  }
  EllView v = ell_view(ell, e);
  v.weighted = (w_t || w_h) ? 1 : 0;
  GR_CHECK_CUDA(cudaMemsetAsync(v.counters, 0, 256, stream));
  FDir d0{rowptr_t, src_t, rel_t, w_t, nullptr}, d1{rowptr_h, src_h, rel_h, w_h, nullptr};
  fused_ell_build_kernel<<<dim3((unsigned)e.ntiles, 2), BM, 0, stream>>>(d0, d1, v, Nt);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_fused_layer(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t, const float* w_t,
                              const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h, const float* w_h,
                              const float* prior, const float* pn_fwd, const float* pn_inv, const float* ins,
                              const void* h_hi, const void* h_lo, int64_t ldh16, int64_t seg_pitch, const float* W,
                              int64_t ldw, const float* bias, float* C, int64_t ldc, void* C_hi, void* C_lo,
                              int64_t ldc16, const float* w_score, float* dots, int B, int N_nodes, int D, int I,
                              int64_t N_out, int64_t F, uint32_t flags, void* workspace, size_t workspace_bytes,
                              void* ell, size_t ell_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(rowptr_t && rowptr_h && prior && pn_fwd && pn_inv && ins && h_hi && h_lo && W && workspace && ell,
               "null pointer");
  GR_CHECK_ARG(F == 0 || (src_t && rel_t && src_h && rel_h), "null edge arrays");
  GR_CHECK_ARG(C || C_hi, "no output requested");
  GR_CHECK_ARG(!C_hi || (C_lo && ldc16 >= N_out), "C_lo missing or ldc16 smaller than N_out");
  GR_CHECK_ARG(!C || ldc >= N_out, "ldc smaller than N_out");
  GR_CHECK_ARG(!dots || w_score, "dots requested without w_score");
  GR_CHECK_ARG(B > 0 && N_nodes > 0 && D > 0 && I > 0 && N_out > 0, "sizes must be positive");
  GR_CHECK_ARG(ldh16 >= seg_pitch && ldh16 % 8 == 0, "ldh16 must be >= seg_pitch and a multiple of 8");
  GR_CHECK_ARG(ldw >= (int64_t)(2 * I + 1) * D, "ldw smaller than the weight row length");
  const int64_t M = (int64_t)B * N_nodes;
  GR_CHECK_ARG(M < (int64_t)0x7fffffff - BM, "B * N exceeds int32 range");
  FusedPlan f = plan_fused(N_nodes, D, seg_pitch, I, N_out);
  if (!f.ok) {
    set_error("gr_fused_layer: unsupported shape N=%d D=%d pitch=%lld I=%d N_out=%lld (need I <= 2, N >= 128, "
              "pitch %% 16 == 0, pitch <= 224, N_out <= 224 and the stages must fit shared memory)",
              N_nodes, D, (long long)seg_pitch, I, (long long)N_out);
    return GR_ERR_UNSUPPORTED;
  }
  if (workspace_bytes < 2 * f.w_plane_bytes || (reinterpret_cast<uintptr_t>(workspace) & 255) != 0) {
    set_error("gr_fused_layer: workspace too small or not 256-byte aligned");
    return GR_ERR_WORKSPACE;
  }
  const EllPlan ep = plan_ell(M, F);
  if (ell_bytes < ep.bytes || (reinterpret_cast<uintptr_t>(ell) & 255) != 0) {
    set_error("gr_fused_layer: quad-ELL buffer too small or not 256-byte aligned (gr_fused_ell_bytes / gr_fused_ell_build)");
    return GR_ERR_WORKSPACE;
  }
  char* ws = reinterpret_cast<char*>(workspace);
  __nv_bfloat16* w_hi = reinterpret_cast<__nv_bfloat16*>(ws);
  __nv_bfloat16* w_lo = reinterpret_cast<__nv_bfloat16*>(ws + f.w_plane_bytes);
  if (!(flags & GR_LINEAR_W_PRESPLIT)) {
    if (int rc = grouped_w_split(W, ldw, N_out, D, I, plan_grouped_k(seg_pitch, I, N_out), w_hi, w_lo, stream)) return rc;
  }
  FParams p{};
  p.dir[0] = FDir{rowptr_t, src_t, rel_t, w_t, reinterpret_cast<const char*>(pn_fwd)};
  p.dir[1] = FDir{rowptr_h, src_h, rel_h, w_h, reinterpret_cast<const char*>(pn_inv)};
  p.ell = ell_view(ell, ep);
  p.ell.weighted = (w_t || w_h) ? 1 : 0;        // must match the build (same graph, same weights)
  if (p.ell.weighted) {
    // per layer: the entries' coefficients c_f = w (w prior[src]) next to their table offsets, one streaming pass
    fused_coef_kernel<<<dim3((unsigned)(2 * sm_count()), 2), 256, 0, stream>>>(p.ell, prior);
    GR_CHECK_LAUNCH();
  }
  p.prior = prior; p.ins = ins; p.bias = bias; p.C = C; p.ldc = ldc; p.w_score = w_score; p.dots = dots;
  p.M = (int)M; p.N = (int)N_out; p.n_pad = f.n_pad; p.D = D; p.B = B; p.Nq = N_nodes; p.G = f.G;
  p.ksteps_last = f.ksteps_last; p.num_tiles = (int)ceil_div(M, BM);
  p.has_planes = C_hi ? 1 : 0;
  p.flags = flags;
  p.debug = g_fused_debug;
  const int cs = ((f.np / 2) % 8 == 0 && p.num_tiles >= 2) ? 2 : 1;
  CUtensorMap m_h_hi, m_h_lo, m_w_hi, m_w_lo, m_c, m_c_hi, m_c_lo;
  // the h planes are exposed with seg_pitch columns only: the box of the last column group is zero filled beyond them
  if (!make_tmap(&m_h_hi, h_hi, M, seg_pitch, ldh16, BM, BK) || !make_tmap(&m_h_lo, h_lo, M, seg_pitch, ldh16, BM, BK) ||
      !make_tmap(&m_w_hi, w_hi, N_out, f.kp, f.kp, f.np / cs, BK) ||
      !make_tmap(&m_w_lo, w_lo, N_out, f.kp, f.kp, f.np / cs, BK)) {
    set_error("gr_fused_layer: cuTensorMapEncodeTiled failed (plane pointers must be 16-byte aligned)");
    return GR_ERR_CUDA;
  }
  memset(&m_c, 0, sizeof(m_c)); memset(&m_c_hi, 0, sizeof(m_c_hi)); memset(&m_c_lo, 0, sizeof(m_c_lo));
  bool ok = true;
  // TMA stores only: with N_out % 4 != 0 they write past column N_out to the end of its 16-byte unit (gr_linear_tc_planes
  // takes direct stores there).  The model's C is a contiguous h32 [M, N_out], whose pitch refuses such a map.
  if (C) ok = make_out_tmap(&m_c, C, M, N_out, ldc, 4);
  const int64_t n16 = std::min<int64_t>((N_out + 15) / 16 * 16, ldc16);
  if (ok && C_hi) ok = make_out_tmap(&m_c_hi, C_hi, M, n16, ldc16, 2) && make_out_tmap(&m_c_lo, C_lo, M, n16, ldc16, 2);
  if (!ok) {
    set_error("gr_fused_layer: output pointers / pitches must be 16-byte aligned (TMA-store epilogue)");
    return GR_ERR_INVALID_ARG;
  }
  const CUtensorMap* m[7] = {&m_h_hi, &m_h_lo, &m_w_hi, &m_w_lo, &m_c, &m_c_hi, &m_c_lo};
  switch (f.np) {
    case 64: return launch_fused_np<64>(m, I, cs, f, p, stream);
    case 128: return launch_fused_np<128>(m, I, cs, f, p, stream);
    case 208: return launch_fused_np<208>(m, I, cs, f, p, stream);
    default: return launch_fused_np<224>(m, I, cs, f, p, stream);
  }
}
