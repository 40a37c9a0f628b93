// Question-side updates of the retrieval forward, one CTA per question.
//
// These are the O(B*D^2) pieces between the graph layers: the instruction generator, the instruction reform
// after every iteration and the evaluation loss / argmax.  In the reference each is a chain of 10-20 tiny torch
// ops on [B, D] tensors; on a GPU the chain is pure launch latency (~230 launches per forward), so each
// chain is one kernel here.
//   gr_instructions   BaseInstruction.get_instruction x num_ins
//                     (gnn/modules/question_encoding/base_encoder.py:73-114, lstm_encoder.py:38-45)
//   gr_query_reform   QueryReform.forward + Fusion.forward for every instruction
//                     (gnn/modules/query_update.py:6-16,18-44; called from gnn/models/ReaRev/rearev.py:214-221)
//   gr_kl_loss_pred   BaseModel.calc_loss_label (kl) + torch.max(pred_dist, dim=1)
//                     (gnn/models/base_model.py:186-215, gnn/models/ReaRev/rearev.py:156-160,228-232)
#include <math.h>

#include "common.cuh"

namespace gr {
namespace {

constexpr float kVeryNegQ = -100000000000.0f;   // VERY_NEG_NUMBER, base_encoder.py:7
constexpr int kQThreads = 1024;                 // 32 warps: the per-question GEMVs are weight-stream latency bound
constexpr int kMaxIns = 8;

// G independent GEMVs of the same shape in one sweep: y[g][n] = (bias[g] ? bias[g][n] : 0) + sum_k W[g][n*ldw + k] * x[g][k]
// for g < G, n < N;  x[g], y[g] in shared memory.  One warp per 4 output rows of the stacked [G*N] row space (lanes
// across k: coalesced weight reads, 4 x 4 independent loads in flight per lane), so all 32 warps stay busy even when
// one GEMV has only D = 200 rows.
struct GemvGroup {
  const float* W;
  const float* bias;
  const float* x;
  float* y;
};

// y_g[n] = W_g[n, :] . x_g (+ bias_g[n]) for every group g < ng and output row n in [n0, n1) (default: all N rows);
// four rows per warp pass, lanes across K.  The dot order of a row does not depend on the row range, so a range split
// over several CTAs gives the bits of the unsplit call.
template <int G>
__device__ __forceinline__ void block_gemv(const GemvGroup (&grp)[G], int ng, int64_t ldw, int N, int K, int n0 = 0,
                                           int n1 = -1) {
  constexpr int NT = 4;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (n1 < 0) n1 = N;
  const int Nr = n1 - n0;
  const int rows = ng * Nr;
  for (int m0 = warp * NT; m0 < rows; m0 += nw * NT) {
    float acc[NT];
    const float* wr[NT];
    const float* xs[NT];
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const int m = min(m0 + t, rows - 1);
      const int g = m / Nr, n = n0 + (m - g * Nr);
      acc[t] = 0.f;
      wr[t] = grp[g].W + (int64_t)n * ldw;
      xs[t] = grp[g].x;
    }
#pragma unroll 4
    for (int k = lane; k < K; k += 32) {
#pragma unroll
      for (int t = 0; t < NT; ++t) acc[t] = fmaf(__ldg(wr[t] + k), xs[t][k], acc[t]);
    }
#pragma unroll
    for (int t = 0; t < NT; ++t) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[t] += __shfl_xor_sync(0xffffffffu, acc[t], o);
      const int m = m0 + t;
      if (lane == 0 && m < rows) {
        const int g = m / Nr, n = n0 + (m - g * Nr);
        grp[g].y[n] = acc[t] + (grp[g].bias ? grp[g].bias[n] : 0.f);
      }
    }
  }
}

struct InsParams {
  const float* hidden;      // [B, Q, D] token states
  const float* qnode;       // [B, D]    last LSTM state
  const int64_t* qtext;     // [B, Q]    token ids (mask = id != pad)
  int64_t pad;
  const float* Wq[kMaxIns]; // question_linear_i.weight [D, D]
  const float* bq[kMaxIns];
  const float *Wcq, *bcq;   // cq_linear [D, 4D]
  const float *wca, *bca;   // ca_linear [1, D], [1]
  float* out;               // [B, I, D]
  float* attn_out;          // optional [B, I, Q]
  int B, Q, D, I;
};

__global__ void __launch_bounds__(kQThreads) instructions_kernel(const InsParams p) {
  extern __shared__ __align__(16) float smq[];
  const int D = p.D, Q = p.Q, I = p.I, b = blockIdx.x, tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  float* s_hid = smq;                    // [Q][D]
  float* s_qn = s_hid + (size_t)Q * D;   // [D]
  float* s_qi = s_qn + D;                // [I][D]
  float* s_ri = s_qi + (size_t)I * D;    // [D]
  float* s_z = s_ri + D;                 // [4D]
  float* s_cq = s_z + 4 * D;             // [D]
  float* s_ca = s_cq + D;                // [Q]
  float* s_mask = s_ca + Q;              // [Q]
  for (int i = tid; i < Q * D; i += blockDim.x) s_hid[i] = p.hidden[(int64_t)b * Q * D + i];
  for (int i = tid; i < D; i += blockDim.x) {
    s_qn[i] = p.qnode[(int64_t)b * D + i];
    s_ri[i] = 0.f;                       // relational_ins starts at zero (base_encoder.py:62)
  }
  for (int q = tid; q < Q; q += blockDim.x) s_mask[q] = p.qtext[(int64_t)b * Q + q] != p.pad ? 1.f : 0.f;
  __syncthreads();
  {
    GemvGroup grp[kMaxIns];                               // q_i = question_linear_i(qnode) for every i at once
    for (int i = 0; i < I; ++i) grp[i] = GemvGroup{p.Wq[i], p.bq[i], s_qn, s_qi + (size_t)i * D};
    block_gemv(grp, I, D, D, D);
  }
  __syncthreads();
  for (int i = 0; i < I; ++i) {
    const float* qi = s_qi + (size_t)i * D;
    for (int d = tid; d < D; d += blockDim.x) {           // cat(ri, q_i, q_i - ri, q_i * ri)
      const float r = s_ri[d], q = qi[d];
      s_z[d] = r;
      s_z[D + d] = q;
      s_z[2 * D + d] = q - r;
      s_z[3 * D + d] = q * r;
    }
    __syncthreads();
    {
      GemvGroup grp[1] = {GemvGroup{p.Wcq, p.bcq, s_z, s_cq}};
      block_gemv(grp, 1, 4 * D, D, 4 * D);
    }
    __syncthreads();
    for (int q = warp; q < Q; q += nw) {                   // ca[q] = ca_linear(cq * hidden[q])
      float s = 0.f;
      for (int d = lane; d < D; d += 32) s = fmaf(__ldg(p.wca + d), s_cq[d] * s_hid[(size_t)q * D + d], s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) s_ca[q] = (s + p.bca[0]) + (1.f - s_mask[q]) * kVeryNegQ;
    }
    __syncthreads();
    if (warp == 0) {                                       // softmax over the Q tokens
      float mx = -INFINITY;
      for (int q = lane; q < Q; q += 32) mx = fmaxf(mx, s_ca[q]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float sum = 0.f;
      for (int q = lane; q < Q; q += 32) sum += expf(s_ca[q] - mx);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      for (int q = lane; q < Q; q += 32) {
        const float a = expf(s_ca[q] - mx) / sum;
        s_ca[q] = a;
        if (p.attn_out) p.attn_out[((int64_t)b * I + i) * Q + q] = a;
      }
    }
    __syncthreads();
    for (int d = tid; d < D; d += blockDim.x) {            // relational_ins = sum_q attn[q] * hidden[q]
      float s = 0.f;
      for (int q = 0; q < Q; ++q) s = fmaf(s_ca[q], s_hid[(size_t)q * D + d], s);
      s_ri[d] = s;
      p.out[((int64_t)b * I + i) * D + d] = s;
    }
    __syncthreads();
  }
}

struct ReformParams {
  const float* seed;        // [B, N] seed weights (query_entities)
  const float* h;           // [B*N, ldh] node embeddings
  int64_t ldh;
  const float* ins_in;      // [B, I, D]
  const float* Wr[kMaxIns]; // reform_j.fusion.r.weight [D, 3D]
  const float* Wg[kMaxIns]; // reform_j.fusion.g.weight [D, 3D]
  float* ins_out;           // [B, I, D]
  float* seed_out;          // optional [B, D]
  int B, N, D, I;
};

__global__ void __launch_bounds__(kQThreads) query_reform_kernel(const ReformParams p) {
  extern __shared__ __align__(16) float smq[];
  __shared__ int s_list[kQThreads];
  __shared__ float s_val[kQThreads];
  __shared__ int s_woff[kQThreads / 32 + 1];
  // grid (B, S): CTA (b, s) owns output columns [d0, d1) of question b's new instructions (the seed pick is cheap and
  // repeated by every slice); 4 x as many CTAs as questions: the one-CTA-per-question version left most SMs idle
  const int D = p.D, N = p.N, b = blockIdx.x, tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int dper = (D + gridDim.y - 1) / gridDim.y;
  const int d0 = min(D, (int)blockIdx.y * dper), d1 = min(D, d0 + dper);
  float* s_y = smq;            // [D]        seed_retrieve
  float* s_z = s_y + D;        // [I][3D]
  float* s_g = s_z + (size_t)p.I * 3 * D;   // [I][D]
  float* s_r = s_g + (size_t)p.I * D;       // [I][D]
  // ---- seed_retrieve = seed_info[b] @ h[b]  (query_update.py:40); seeds visited in index order ----
  const float* sd = p.seed + (int64_t)b * N;
  float acc = 0.f;             // thread d owns column d (D <= 1024)
  for (int base = 0; base < N; base += blockDim.x) {
    const int n = base + tid;
    const float v = n < N ? sd[n] : 0.f;
    const bool nz = v != 0.f;
    const unsigned bal = __ballot_sync(0xffffffffu, nz);
    if (lane == 0) s_woff[warp + 1] = __popc(bal);
    __syncthreads();
    if (tid == 0) {
      s_woff[0] = 0;
      for (int i = 0; i < nw; ++i) s_woff[i + 1] += s_woff[i];
    }
    __syncthreads();
    if (nz) {
      const int pos = s_woff[warp] + __popc(bal & ((1u << lane) - 1));
      s_list[pos] = n;
      s_val[pos] = v;
    }
    __syncthreads();
    const int cnt = s_woff[nw];
    if (tid < D)
      for (int i = 0; i < cnt; ++i) acc = fmaf(s_val[i], p.h[((int64_t)b * N + s_list[i]) * p.ldh + tid], acc);
    __syncthreads();
  }
  if (tid < D) {
    s_y[tid] = acc;
    if (p.seed_out && blockIdx.y == 0) p.seed_out[(int64_t)b * D + tid] = acc;
  }
  __syncthreads();
  // ---- Fusion per instruction: z = [x, y, x-y]; g = sigmoid(G z); out = g * (R z) + (1-g) * x ----
  // (the 2*I GEMVs are independent: one sweep over the stacked rows)
  for (int i = tid; i < p.I * D; i += blockDim.x) {
    const int j = i / D, d = i - j * D;
    const float xv = p.ins_in[((int64_t)b * p.I + j) * D + d], yv = s_y[d];
    float* z = s_z + (size_t)j * 3 * D;
    z[d] = xv;
    z[D + d] = yv;
    z[2 * D + d] = xv - yv;
  }
  __syncthreads();
  {
    GemvGroup grp[2 * kMaxIns];
    for (int j = 0; j < p.I; ++j) {
      grp[2 * j] = GemvGroup{p.Wg[j], nullptr, s_z + (size_t)j * 3 * D, s_g + (size_t)j * D};
      grp[2 * j + 1] = GemvGroup{p.Wr[j], nullptr, s_z + (size_t)j * 3 * D, s_r + (size_t)j * D};
    }
    block_gemv(grp, 2 * p.I, 3 * D, D, 3 * D, d0, d1);
  }
  __syncthreads();
  for (int i = tid; i < p.I * (d1 - d0); i += blockDim.x) {
    const int j = i / (d1 - d0), d = d0 + (i - j * (d1 - d0));
    const float g = 1.f / (1.f + expf(-s_g[(size_t)j * D + d]));
    p.ins_out[((int64_t)b * p.I + j) * D + d] = g * s_r[(size_t)j * D + d] + (1.f - g) * s_z[(size_t)j * 3 * D + d];
  }
}

__device__ __forceinline__ float block_sum(float v, float* sm) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) sm[wid] = v;
  __syncthreads();
  float r = 0.f;
  if (wid == 0) {
    r = lane < nw ? sm[lane] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    if (lane == 0) sm[0] = r;
  }
  __syncthreads();
  r = sm[0];
  __syncthreads();
  return r;
}

// one CTA per question: KL(teacher/len || pred) row sum (x case_valid) and argmax (lowest index on ties)
__global__ void kl_loss_pred_kernel(const float* __restrict__ dist, const float* __restrict__ teacher,
                                    float* __restrict__ loss_q, int64_t* __restrict__ pred, int N) {
  __shared__ float sm[32];
  __shared__ float s_bv[32];
  __shared__ int s_bi[32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
  const float* p = dist + (int64_t)b * N;
  const float* t = teacher + (int64_t)b * N;
  float len = 0.f;
  for (int n = tid; n < N; n += blockDim.x) len += t[n];
  len = block_sum(len, sm);
  const float valid = len > 0.f ? 1.f : 0.f;               // case_valid (rearev.py:228)
  if (len == 0.f) len = 1.f;                               // base_model.py:207
  float kl = 0.f, bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int n = tid; n < N; n += blockDim.x) {
    const float pv = p[n];
    const float tv = t[n] / len;
    // F.kl_div(log(p + 1e-8), t, 'none') = xlogy(t, t) - t * log(p + 1e-8)
    const float inp = logf(pv + 1e-8f);
    const float term = (tv > 0.f ? tv * logf(tv) : 0.f) - tv * inp;
    kl += term * valid;
    if (pv > bv) {
      bv = pv;
      bi = n;
    }
  }
  kl = block_sum(kl, sm);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) {
      bv = ov;
      bi = oi;
    }
  }
  if (lane == 0) {
    s_bv[wid] = bv;
    s_bi[wid] = bi;
  }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < nw; ++w)
      if (s_bv[w] > bv || (s_bv[w] == bv && s_bi[w] < bi)) {
        bv = s_bv[w];
        bi = s_bi[w];
      }
    loss_q[b] = kl;
    pred[b] = bi == 0x7fffffff ? 0 : bi;
  }
}

// loss = sum_b loss_q[b] / B, fixed order
__global__ void loss_finalize_kernel(const float* __restrict__ loss_q, float* __restrict__ loss, int B) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += loss_q[b];
    loss[0] = s / (float)B;
  }
}

}  // namespace
}  // namespace gr

extern "C" int gr_instructions(const float* hidden, const float* qnode, const int64_t* qtext, int64_t pad_id,
                               const float* const* Wq_host, const float* const* bq_host, const float* Wcq,
                               const float* bcq, const float* wca, const float* bca, float* out,
                               float* attn_out, int B, int Q, int D, int I, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(hidden && qnode && qtext && Wq_host && bq_host && Wcq && bcq && wca && bca && out,
               "null pointer");
  GR_CHECK_ARG(B > 0 && Q > 0 && D > 0 && I > 0 && I <= kMaxIns, "bad shape (num_ins <= 8)");
  InsParams p{};
  p.hidden = hidden; p.qnode = qnode; p.qtext = qtext; p.pad = pad_id;
  for (int i = 0; i < I; ++i) {
    GR_CHECK_ARG(Wq_host[i] && bq_host[i], "null question_linear pointer");
    p.Wq[i] = Wq_host[i];
    p.bq[i] = bq_host[i];
  }
  p.Wcq = Wcq; p.bcq = bcq; p.wca = wca; p.bca = bca; p.out = out; p.attn_out = attn_out;
  p.B = B; p.Q = Q; p.D = D; p.I = I;
  const size_t smem = ((size_t)Q * D + (size_t)(I + 7) * D + 2 * (size_t)Q) * sizeof(float);
  GR_CHECK_ARG(smem <= 200 * 1024, "question length x entity_dim too large for shared memory");
  if (int rc = opt_in_smem<instructions_kernel>(__func__, 200 * 1024)) return rc;
  instructions_kernel<<<B, kQThreads, smem, stream>>>(p);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_query_reform(const float* seed_info, const float* h, int64_t ldh, const float* ins_in,
                               const float* const* Wr_host, const float* const* Wg_host, float* ins_out,
                               float* seed_out, int B, int N, int D, int I, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(seed_info && h && ins_in && Wr_host && Wg_host && ins_out, "null pointer");
  GR_CHECK_ARG(B > 0 && N > 0 && D > 0 && D <= kQThreads && ldh >= D && I > 0 && I <= kMaxIns,
               "bad shape (D <= 1024, num_ins <= 8)");
  ReformParams p{};
  p.seed = seed_info; p.h = h; p.ldh = ldh; p.ins_in = ins_in; p.ins_out = ins_out; p.seed_out = seed_out;
  for (int j = 0; j < I; ++j) {
    GR_CHECK_ARG(Wr_host[j] && Wg_host[j], "null fusion weight pointer");
    p.Wr[j] = Wr_host[j];
    p.Wg[j] = Wg_host[j];
  }
  p.B = B; p.N = N; p.D = D; p.I = I;
  const size_t smem = ((size_t)1 + 5 * (size_t)I) * D * sizeof(float);
  GR_CHECK_ARG(smem <= 48 * 1024, "num_ins x entity_dim too large for shared memory");
  // the kernel's static seed list (s_list / s_val / s_woff, ~8 KB) comes on top of the dynamic area: without the
  // opt-in, static + dynamic is capped at 48 KB and every admitted shape with (5I+1)*D > ~10200 fails to launch
  if (int rc = opt_in_smem<query_reform_kernel>(__func__, 48 * 1024)) return rc;
  const int slices = D >= 128 ? 4 : (D >= 64 ? 2 : 1);
  query_reform_kernel<<<dim3((unsigned)B, (unsigned)slices), kQThreads, smem, stream>>>(p);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_kl_loss_pred(const float* dist, const float* teacher, float* loss_q, float* loss,
                               int64_t* pred, int B, int N, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(dist && teacher && loss_q && loss && pred, "null pointer");
  GR_CHECK_ARG(B > 0 && N > 0, "bad shape");
  kl_loss_pred_kernel<<<B, 256, 0, stream>>>(dist, teacher, loss_q, pred, N);
  GR_CHECK_LAUNCH();
  loss_finalize_kernel<<<1, 32, 0, stream>>>(loss_q, loss, B);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

// ---------------------------------------------------------------------------------------------------------
// gr_lstm_forward: the recurrent half of the question encoder (nn.LSTM, one layer, batch_first, zero initial state;
// gnn/modules/question_encoding/lstm_encoder.py:27-36).  cuDNN runs it as 2 launches per token (GEMM + cell); here
// the whole sequence is ONE launch: a cluster of 8 CTAs serves 8 questions, CTA r keeps the W_hh rows of hidden
// units [r*U, (r+1)*U) (all four gates) resident in shared memory for every time step, computes those units for the
// cluster's questions and broadcasts the new h slice to the 7 peers through distributed shared memory; one cluster
// barrier per token.
// ---------------------------------------------------------------------------------------------------------
#include <cooperative_groups.h>
#include <cuda_pipeline.h>

namespace gr {
namespace {
namespace cg = cooperative_groups;

constexpr int kLstmCluster = 8;   // CTAs per cluster (portable maximum)
constexpr int kLstmQB = 8;        // questions per cluster
constexpr int kLstmThreads = 256;

__global__ void __cluster_dims__(kLstmCluster, 1, 1) __launch_bounds__(kLstmThreads)
lstm_kernel(const float* __restrict__ gx, const float* __restrict__ Whh, const float* __restrict__ bhh,
            float* __restrict__ hidden, int B, int Q, int D) {
  extern __shared__ __align__(16) float sml[];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int qb0 = (blockIdx.x / kLstmCluster) * kLstmQB;
  const int U = (D + kLstmCluster - 1) / kLstmCluster;
  const int u0 = rank * U;
  const int nu = max(0, min(U, D - u0));
  const int pitch = D | 1;                              // odd row pitch: conflict-free row-per-lane reads
  float* sW = sml;                                      // [4U][pitch]
  float* sH = reinterpret_cast<float*>(                  // [2][D][QB], 16-byte aligned (float4 reads)
      (reinterpret_cast<uintptr_t>(sW + (size_t)4 * U * pitch) + 15) & ~(uintptr_t)15);
  float* sG = sH + (size_t)2 * D * kLstmQB;             // [4U][QB]
  const int tid = threadIdx.x;
  for (int i = tid; i < 4 * U * D; i += blockDim.x) {   // async copies: all of a thread's loads are in flight at once
    const int r = i / D, k = i - r * D;
    const int g = r / U, u = r - g * U;
    if (u < nu)
      __pipeline_memcpy_async(sW + (size_t)r * pitch + k, Whh + ((int64_t)g * D + u0 + u) * D + k, sizeof(float));
    else
      sW[(size_t)r * pitch + k] = 0.f;
  }
  __pipeline_commit();
  for (int i = tid; i < 2 * D * kLstmQB; i += blockDim.x) sH[i] = 0.f;
  __pipeline_wait_prior(0);
  cluster.sync();
  // gate/cell role: thread -> (hidden unit u, question q); matvec role: thread -> (gate row r, 4 questions)
  const int gu = tid / kLstmQB, gq = tid % kLstmQB;
  const bool cell = gu < nu && qb0 + gq < B;
  const int ug = u0 + gu;
  const int64_t bq = (int64_t)(qb0 + gq);
  float c = 0.f;
  float bias[4] = {0.f, 0.f, 0.f, 0.f};
  if (cell && bhh)
#pragma unroll
    for (int g = 0; g < 4; ++g) bias[g] = bhh[g * D + ug];
  const int r = tid & 127, qh = tid >> 7;
  float gin[4] = {0.f, 0.f, 0.f, 0.f}, gnext[4] = {0.f, 0.f, 0.f, 0.f};
  if (cell) {
#pragma unroll
    for (int g = 0; g < 4; ++g) gin[g] = __ldg(gx + (bq * Q) * 4 * D + (int64_t)g * D + ug);
  }
  for (int t = 0; t < Q; ++t) {
    const int cur = t & 1, nxt = cur ^ 1;
    if (cell && t + 1 < Q) {                             // next token's input projection: a full step of slack
      const float* gp = gx + (bq * Q + t + 1) * 4 * D + ug;
#pragma unroll
      for (int g = 0; g < 4; ++g) gnext[g] = __ldg(gp + (int64_t)g * D);
    }
    if (r < 4 * U) {
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      const float* w = sW + (size_t)r * pitch;
      const float* hb = sH + (size_t)cur * D * kLstmQB + 4 * qh;
#pragma unroll 4
      for (int k = 0; k < D; ++k) {
        const float wv = w[k];
        const float4 h4 = *reinterpret_cast<const float4*>(hb + (size_t)k * kLstmQB);
        a0 = fmaf(wv, h4.x, a0);
        a1 = fmaf(wv, h4.y, a1);
        a2 = fmaf(wv, h4.z, a2);
        a3 = fmaf(wv, h4.w, a3);
      }
      float* gdst = sG + (size_t)r * kLstmQB + 4 * qh;
      gdst[0] = a0; gdst[1] = a1; gdst[2] = a2; gdst[3] = a3;
    }
    __syncthreads();
    if (cell) {
      const float gi = sG[(size_t)(0 * U + gu) * kLstmQB + gq] + gin[0] + bias[0];
      const float gf = sG[(size_t)(1 * U + gu) * kLstmQB + gq] + gin[1] + bias[1];
      const float gg = sG[(size_t)(2 * U + gu) * kLstmQB + gq] + gin[2] + bias[2];
      const float go = sG[(size_t)(3 * U + gu) * kLstmQB + gq] + gin[3] + bias[3];
      const float iv = 1.f / (1.f + expf(-gi)), fv = 1.f / (1.f + expf(-gf));
      const float ov = 1.f / (1.f + expf(-go)), gv = tanhf(gg);
      c = fmaf(fv, c, iv * gv);
      const float h = ov * tanhf(c);
      hidden[(bq * Q + t) * D + ug] = h;
      const size_t off = (size_t)nxt * D * kLstmQB + (size_t)ug * kLstmQB + gq;
#pragma unroll
      for (int rk = 0; rk < kLstmCluster; ++rk) cluster.map_shared_rank(sH, rk)[off] = h;
#pragma unroll
      for (int g = 0; g < 4; ++g) gin[g] = gnext[g];
    }
    cluster.sync();                                      // new h visible everywhere; sG / old h free for reuse
  }
}

}  // namespace
}  // namespace gr

extern "C" size_t gr_lstm_max_hidden(void) { return 256; }

extern "C" int gr_lstm_forward(const float* gates_x, const float* W_hh, const float* b_hh, float* hidden, int B,
                               int Q, int D, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(gates_x && W_hh && hidden, "null pointer");
  GR_CHECK_ARG(B > 0 && Q > 0 && D > 0 && D <= 256, "bad shape (hidden size <= 256)");
  const int U = (D + kLstmCluster - 1) / kLstmCluster;
  const size_t smem = ((size_t)4 * U * (D | 1) + 8 + (size_t)2 * D * kLstmQB + (size_t)4 * U * kLstmQB) * sizeof(float);
  if (int rc = opt_in_smem<lstm_kernel>(__func__, 200 * 1024)) return rc;
  GR_CHECK_ARG(smem <= 200 * 1024, "hidden size too large for shared memory");
  const int clusters = (B + kLstmQB - 1) / kLstmQB;
  lstm_kernel<<<clusters * kLstmCluster, kLstmThreads, smem, stream>>>(gates_x, W_hh, b_hh, hidden, B, Q, D);
  GR_CHECK_LAUNCH();
  return GR_OK;
}
