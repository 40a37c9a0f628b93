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

#include <algorithm>

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
  const int64_t* seed;      // training dropout (kDrop): device int64[1]
  float p, scale;           // drop probability and 1 / (1 - p)
};

// The three linear_drop sites of get_instruction (base_encoder.py:85-98) at step i: 0 = qnode before
// question_linear_i (column c < D), 1 = [ri, q_i, q_i - ri, q_i * ri] before cq_linear (c < 4D), 2 = cq * hidden[q]
// before ca_linear (token q, c < D).  Counter = (question, 4 * step + site, token (0 for sites 0 / 1), column).
enum { kSiteQnode = 0, kSiteCq = 1, kSiteCa = 2 };

__device__ __forceinline__ bool ins_keep(uint64_t seed, float p, int b, int i, int site, int q, int c) {
  return philox_keep(philox4x32_10_x0(seed, (uint32_t)b, (uint32_t)(4 * i + site), (uint32_t)q, (uint32_t)c), p);
}

// v dropped at one site: v * scale if kept, else 0
__device__ __forceinline__ float ins_drop(float v, bool keep, float scale) { return keep ? __fmul_rn(v, scale) : 0.f; }

// kDrop = false: gr_instructions (eval) and gr_instructions_train with p = 0.  kDrop = true: the three dropout sites;
// q_i is then formed per step from that step's dropped qnode (same GEMV rows, same dot order).
template <bool kDrop>
__global__ void __launch_bounds__(kQThreads) instructions_kernel(const InsParams p) {
  extern __shared__ __align__(16) float smq[];
  const int D = p.D, Q = p.Q, I = p.I, b = blockIdx.x, tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const uint64_t seed = kDrop ? (uint64_t)__ldg(p.seed) : 0;
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
  if constexpr (!kDrop) {
    GemvGroup grp[kMaxIns];                               // q_i = question_linear_i(qnode) for every i at once
    for (int i = 0; i < I; ++i) grp[i] = GemvGroup{p.Wq[i], p.bq[i], s_qn, s_qi + (size_t)i * D};
    block_gemv(grp, I, D, D, D);
    __syncthreads();
  }
  for (int i = 0; i < I; ++i) {
    const float* qi = s_qi + (size_t)i * D;
    if constexpr (kDrop) {                                // q_i = question_linear_i(drop(qnode)), s_z as scratch
      for (int d = tid; d < D; d += blockDim.x)
        s_z[d] = ins_drop(s_qn[d], ins_keep(seed, p.p, b, i, kSiteQnode, 0, d), p.scale);
      __syncthreads();
      GemvGroup grp[1] = {GemvGroup{p.Wq[i], p.bq[i], s_z, s_qi + (size_t)i * D}};
      block_gemv(grp, 1, D, D, D);
      __syncthreads();
    }
    for (int d = tid; d < D; d += blockDim.x) {           // cat(ri, q_i, q_i - ri, q_i * ri)
      const float r = s_ri[d], q = qi[d];
      float z[4] = {r, q, q - r, q * r};
      if constexpr (kDrop) {
#pragma unroll
        for (int k = 0; k < 4; ++k) z[k] = ins_drop(z[k], ins_keep(seed, p.p, b, i, kSiteCq, 0, k * D + d), p.scale);
      }
      s_z[d] = z[0];
      s_z[D + d] = z[1];
      s_z[2 * D + d] = z[2];
      s_z[3 * D + d] = z[3];
    }
    __syncthreads();
    {
      GemvGroup grp[1] = {GemvGroup{p.Wcq, p.bcq, s_z, s_cq}};
      block_gemv(grp, 1, 4 * D, D, 4 * D);
    }
    __syncthreads();
    for (int q = warp; q < Q; q += nw) {                   // ca[q] = ca_linear(cq * hidden[q])
      float s = 0.f;
      for (int d = lane; d < D; d += 32) {
        float e = s_cq[d] * s_hid[(size_t)q * D + d];
        if constexpr (kDrop) e = ins_drop(e, ins_keep(seed, p.p, b, i, kSiteCa, q, d), p.scale);
        s = fmaf(__ldg(p.wca + d), e, s);
      }
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

struct InsBwdParams {
  InsParams f;              // the forward's inputs (out / attn_out unused), seed, p, scale
  const float* ri;          // [B, I, D] the forward's instructions
  const float* attn;        // [B, I, Q] the forward's attention
  const float* grad_out;    // [B, I, D]
  float* grad_hidden;       // [B, Q, D]
  float* grad_qnode;        // [B, D]
  float *g_q, *x_q;         // [B, I, D]: question_linear_i pre-activation gradient and its (dropped) input
  float *g_cq, *x_cq;       // [B, I, D], [B, I, 4D]: cq_linear
  float *g_ca, *x_ca;       // [B, I, Q], [B, I, Q, D]: ca_linear (the masked logit's gradient)
};

// y[k] = sum_n W[n * ldw + k] * x[n] for k < K, n in order: one thread per output column (coalesced across k)
__device__ __forceinline__ void block_gemv_t(const float* __restrict__ W, int64_t ldw, const float* x, float* y,
                                             int N, int K) {
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float s = 0.f;
    for (int n = 0; n < N; ++n) s = fmaf(__ldg(W + (int64_t)n * ldw + k), x[n], s);
    y[k] = s;
  }
}

// gr_instructions_backward: one CTA per question walks the steps in reverse.  Step i is recomputed from the saved
// inputs, the forward's ri[i-1] and attention and the seed (the mask is redrawn, never stored), with the forward
// kernel's operations, so the recomputed q_i, cq and dropped operands are the forward's bits.  Every output element is
// owned by this CTA and written by one thread per step, in a fixed order: no atomics.
template <bool kDrop>
__global__ void __launch_bounds__(kQThreads) instructions_bwd_kernel(const InsBwdParams a) {
  extern __shared__ __align__(16) float smq[];
  const InsParams& p = a.f;
  const int D = p.D, Q = p.Q, I = p.I, b = blockIdx.x, tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const uint64_t seed = kDrop ? (uint64_t)__ldg(p.seed) : 0;
  float* s_hid = smq;                    // [Q][D]
  float* s_qn = s_hid + (size_t)Q * D;   // [D]
  float* s_q = s_qn + D;                 // [D]   q_i
  float* s_cq = s_q + D;                 // [D]   cq, then its gradient
  float* s_gr = s_cq + D;                // [D]   gradient of ri[i]
  float* s_g4 = s_gr + D;                // [4D]  gradient of the dropped cq_linear input, then of q_i (first D)
  float* s_gca = s_g4 + 4 * D;           // [Q]   dattn, then the logit gradient (pads: attn = 0, so 0)
  const int64_t bq = (int64_t)b * Q * D;
  for (int i = tid; i < Q * D; i += blockDim.x) {
    s_hid[i] = p.hidden[bq + i];
    a.grad_hidden[bq + i] = 0.f;
  }
  for (int d = tid; d < D; d += blockDim.x) {
    s_qn[d] = p.qnode[(int64_t)b * D + d];
    s_gr[d] = a.grad_out[((int64_t)b * I + I - 1) * D + d];
    a.grad_qnode[(int64_t)b * D + d] = 0.f;
  }
  __syncthreads();
  for (int i = I - 1; i >= 0; --i) {
    const int64_t bi = (int64_t)b * I + i;
    const float* ri_prev = i > 0 ? a.ri + (bi - 1) * D : nullptr;   // ri[-1] = 0
    float* xq = a.x_q + bi * D;
    float* xcq = a.x_cq + bi * 4 * D;
    const float* at = a.attn + bi * Q;
    // ---- recompute q_i and cq of step i (the forward's operations) ----
    for (int d = tid; d < D; d += blockDim.x)
      xq[d] = kDrop ? ins_drop(s_qn[d], ins_keep(seed, p.p, b, i, kSiteQnode, 0, d), p.scale) : s_qn[d];
    __syncthreads();
    {
      GemvGroup grp[1] = {GemvGroup{p.Wq[i], p.bq[i], xq, s_q}};
      block_gemv(grp, 1, D, D, D);
    }
    __syncthreads();
    for (int d = tid; d < D; d += blockDim.x) {
      const float r = ri_prev ? ri_prev[d] : 0.f, q = s_q[d];
      float z[4] = {r, q, q - r, q * r};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (kDrop) z[k] = ins_drop(z[k], ins_keep(seed, p.p, b, i, kSiteCq, 0, k * D + d), p.scale);
        xcq[k * D + d] = z[k];
      }
    }
    __syncthreads();
    {
      GemvGroup grp[1] = {GemvGroup{p.Wcq, p.bcq, xcq, s_cq}};
      block_gemv(grp, 1, 4 * D, D, 4 * D);
    }
    // ---- ri[i] = sum_q attn[q] hidden[q]:  dattn[q] = <hidden[q], g_ri> ----
    for (int q = warp; q < Q; q += nw) {
      float s = 0.f;
      for (int d = lane; d < D; d += 32) s = fmaf(s_hid[(size_t)q * D + d], s_gr[d], s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) s_gca[q] = s;
    }
    __syncthreads();
    // ---- softmax: g_ca[q] = attn[q] (dattn[q] - sum_q' attn[q'] dattn[q']), q' in order ----
    if (warp == 0) {
      float s = 0.f;
      for (int q = lane; q < Q; q += 32) s = fmaf(__ldg(at + q), s_gca[q], s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      for (int q = lane; q < Q; q += 32) {
        const float g = __ldg(at + q) * (s_gca[q] - s);
        s_gca[q] = g;
        a.g_ca[bi * Q + q] = g;
      }
    }
    __syncthreads();
    // ---- ca[q] = <wca, drop(cq * hidden[q])> + bca:  one thread per column d walks the tokens in order ----
    for (int d = tid; d < D; d += blockDim.x) {
      const float cq = s_cq[d], w = __ldg(p.wca + d), gr = s_gr[d];
      float gcq = 0.f;
      for (int q = 0; q < Q; ++q) {
        const float h = s_hid[(size_t)q * D + d];
        float e = cq * h, ge = s_gca[q] * w;
        if (kDrop) {
          const bool keep = ins_keep(seed, p.p, b, i, kSiteCa, q, d);
          e = ins_drop(e, keep, p.scale);
          ge = ins_drop(ge, keep, p.scale);
        }
        a.x_ca[(bi * Q + q) * D + d] = e;
        float* gh = a.grad_hidden + bq + (int64_t)q * D + d;
        *gh = *gh + fmaf(ge, cq, __ldg(at + q) * gr);
        gcq = fmaf(ge, h, gcq);
      }
      s_cq[d] = gcq;                                      // cq is dead in this column from here on
      a.g_cq[bi * D + d] = gcq;
    }
    __syncthreads();
    // ---- cq = Wcq drop(z) + bcq:  g_z = drop'(Wcq^T g_cq) ----
    block_gemv_t(p.Wcq, 4 * D, s_cq, s_g4, D, 4 * D);
    __syncthreads();
    for (int d = tid; d < D; d += blockDim.x) {
      float gz[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        gz[k] = s_g4[k * D + d];
        if (kDrop) gz[k] = ins_drop(gz[k], ins_keep(seed, p.p, b, i, kSiteCq, 0, k * D + d), p.scale);
      }
      const float r = ri_prev ? ri_prev[d] : 0.f, q = s_q[d];
      const float gq = fmaf(gz[3], r, gz[1] + gz[2]);     // z = [ri, q, q - ri, q * ri]
      const float gri = fmaf(gz[3], q, gz[0] - gz[2]);
      s_g4[d] = gq;                                       // this thread's own columns only
      a.g_q[bi * D + d] = gq;
      s_gr[d] = i > 0 ? a.grad_out[(bi - 1) * D + d] + gri : 0.f;
    }
    __syncthreads();
    // ---- q_i = Wq_i drop(qnode) + bq_i:  grad_qnode += drop'(Wq_i^T g_q) ----
    for (int k = tid; k < D; k += blockDim.x) {
      float s = 0.f;
      for (int n = 0; n < D; ++n) s = fmaf(__ldg(p.Wq[i] + (int64_t)n * D + k), s_g4[n], s);
      if (kDrop) s = ins_drop(s, ins_keep(seed, p.p, b, i, kSiteQnode, 0, k), p.scale);
      a.grad_qnode[(int64_t)b * D + k] += s;
    }
    __syncthreads();
  }
}

// the dropout masks of gr_instructions_train: one thread per element of the three sites
__global__ void instructions_dropout_mask_kernel(const int64_t* __restrict__ seed, float p, int B, int Q, int D, int I,
                                                 uint8_t* __restrict__ m_q, uint8_t* __restrict__ m_cq,
                                                 uint8_t* __restrict__ m_ca) {
  const uint64_t sd = (uint64_t)__ldg(seed);
  const int64_t nq = (int64_t)B * I * D, ncq = 4 * nq, nca = (int64_t)Q * nq;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nq + ncq + nca; t += stride) {
    if (t < nq) {
      const int64_t bi = t / D;
      m_q[t] = ins_keep(sd, p, (int)(bi / I), (int)(bi % I), kSiteQnode, 0, (int)(t % D));
    } else if (t < nq + ncq) {
      const int64_t u = t - nq, bi = u / (4 * D);
      m_cq[u] = ins_keep(sd, p, (int)(bi / I), (int)(bi % I), kSiteCq, 0, (int)(u % (4 * D)));
    } else {
      const int64_t u = t - nq - ncq, biq = u / D, bi = biq / Q;
      m_ca[u] = ins_keep(sd, p, (int)(bi / I), (int)(bi % I), kSiteCa, (int)(biq % Q), (int)(u % D));
    }
  }
}

struct ReformParams {
  const float* seed;        // [B, N] seed weights (query_entities)
  const void* h;            // [B*N, ldh] node embeddings, fp32 or (GR_IO_BF16) bf16
  int64_t ldh;
  const float* ins_in;      // [B, I, D]
  const float* Wr[kMaxIns]; // reform_j.fusion.r.weight [D, 3D]
  const float* Wg[kMaxIns]; // reform_j.fusion.g.weight [D, 3D]
  float* ins_out;           // [B, I, D]
  float* seed_out;          // optional [B, D]
  int B, N, D, I;
};

// The non-zero seeds of one question in index order, a block-wide walk: chunks of blockDim.x nodes are compacted into
// (s_list, s_val) and f(cnt) is called by every thread after each chunk, with the chunk's cnt seeds in index order.
struct SeedList {
  int list[kQThreads];
  float val[kQThreads];
  int woff[kQThreads / 32 + 1];
};

template <typename F>
__device__ __forceinline__ void for_each_seed_chunk(const float* sd, int N, SeedList& sl, F&& f) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  for (int base = 0; base < N; base += blockDim.x) {
    const int n = base + tid;
    const float v = n < N ? sd[n] : 0.f;
    const bool nz = v != 0.f;
    const unsigned bal = __ballot_sync(0xffffffffu, nz);
    if (lane == 0) sl.woff[warp + 1] = __popc(bal);
    __syncthreads();
    if (tid == 0) {
      sl.woff[0] = 0;
      for (int i = 0; i < nw; ++i) sl.woff[i + 1] += sl.woff[i];
    }
    __syncthreads();
    if (nz) {
      const int pos = sl.woff[warp] + __popc(bal & ((1u << lane) - 1));
      sl.list[pos] = n;
      sl.val[pos] = v;
    }
    __syncthreads();
    f(sl.woff[nw]);
    __syncthreads();
  }
}

// seed_retrieve = seed_info[b] @ h[b] (query_update.py:40) for column tid < D, seeds in index order
template <typename T>
__device__ __forceinline__ float seed_retrieve_col(const float* sd, const T* h, int64_t ldh, int b, int N, int D,
                                                   SeedList& sl) {
  const int tid = threadIdx.x;
  float acc = 0.f;             // thread d owns column d (D <= 1024)
  for_each_seed_chunk(sd, N, sl, [&](int cnt) {
    if (tid < D)
      for (int i = 0; i < cnt; ++i) acc = fmaf(sl.val[i], ldg_node(h + ((int64_t)b * N + sl.list[i]) * ldh + tid), acc);
  });
  return acc;
}

template <typename T>
__global__ void __launch_bounds__(kQThreads) query_reform_kernel(const ReformParams p) {
  extern __shared__ __align__(16) float smq[];
  __shared__ SeedList sl;
  // grid (B, S): CTA (b, s) owns output columns [d0, d1) of question b's new instructions (the seed pick is cheap and
  // repeated by every slice); 4 x as many CTAs as questions: the one-CTA-per-question version left most SMs idle
  const int D = p.D, N = p.N, b = blockIdx.x, tid = threadIdx.x;
  const int dper = (D + gridDim.y - 1) / gridDim.y;
  const int d0 = min(D, (int)blockIdx.y * dper), d1 = min(D, d0 + dper);
  float* s_y = smq;            // [D]        seed_retrieve
  float* s_z = s_y + D;        // [I][3D]
  float* s_g = s_z + (size_t)p.I * 3 * D;   // [I][D]
  float* s_r = s_g + (size_t)p.I * D;       // [I][D]
  // ---- seed_retrieve = seed_info[b] @ h[b]  (query_update.py:40); seeds visited in index order ----
  const float acc = seed_retrieve_col(p.seed + (int64_t)b * N, static_cast<const T*>(p.h), p.ldh, b, N, D, sl);
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

struct ReformBwdParams {
  ReformParams f;           // the forward's inputs (ins_out / seed_out unused)
  const float* grad_out;    // [B, I, D]
  float* grad_ins;          // [B, I, D]
  void* grad_h;             // [B*N, ldg] in h's type: the seed rows are added to, nothing else is touched
  int64_t ldg;
  float *g_r, *g_g;         // [B, I, D] pre-activation gradients of fusion.r / fusion.g
  float* x_z;               // [B, I, 3D] their input z = [x, y, x - y]
};

// gr_query_reform_backward: one CTA per question recomputes y, z, g and r with the forward's operations (the same
// seed walk and GEMV rows), then
//   g_r = G g,  g_g = G (r - x) g (1 - g),  g_z = Wr^T g_r + Wg^T g_g   (each transposed GEMV over n in order),
//   grad_x = (G (1 - g) + g_z[x]) + g_z[x - y],   g_y = sum_j (g_z[y] - g_z[x - y]) in j order,
//   grad_h[seed n] = fma(s_n, g_y, grad_h[seed n]) over the forward's seed list.
template <typename T>
__global__ void __launch_bounds__(kQThreads) query_reform_bwd_kernel(const ReformBwdParams a) {
  extern __shared__ __align__(16) float smq[];
  __shared__ SeedList sl;
  const ReformParams& p = a.f;
  const int D = p.D, N = p.N, I = p.I, b = blockIdx.x, tid = threadIdx.x;
  float* s_y = smq;                         // [D]      y, then g_y
  float* s_z = s_y + D;                     // [I][3D]  z, then g_z
  float* s_g = s_z + (size_t)I * 3 * D;     // [I][D]   G z, then g_g
  float* s_r = s_g + (size_t)I * D;         // [I][D]   R z, then g_r
  const float* sd = p.seed + (int64_t)b * N;
  const float acc = seed_retrieve_col(sd, static_cast<const T*>(p.h), p.ldh, b, N, D, sl);
  if (tid < D) s_y[tid] = acc;
  __syncthreads();
  for (int i = tid; i < I * D; i += blockDim.x) {
    const int j = i / D, d = i - j * D;
    const float xv = p.ins_in[((int64_t)b * I + j) * D + d], yv = s_y[d];
    float* z = s_z + (size_t)j * 3 * D;
    float* xz = a.x_z + ((int64_t)b * I + j) * 3 * D;
    z[d] = xz[d] = xv;
    z[D + d] = xz[D + d] = yv;
    z[2 * D + d] = xz[2 * D + d] = xv - yv;
  }
  __syncthreads();
  {
    GemvGroup grp[2 * kMaxIns];
    for (int j = 0; j < I; ++j) {
      grp[2 * j] = GemvGroup{p.Wg[j], nullptr, s_z + (size_t)j * 3 * D, s_g + (size_t)j * D};
      grp[2 * j + 1] = GemvGroup{p.Wr[j], nullptr, s_z + (size_t)j * 3 * D, s_r + (size_t)j * D};
    }
    block_gemv(grp, 2 * I, 3 * D, D, 3 * D);
  }
  __syncthreads();
  for (int i = tid; i < I * D; i += blockDim.x) {   // out = g r + (1 - g) x
    const int j = i / D, d = i - j * D;
    const int64_t o = ((int64_t)b * I + j) * D + d;
    const float G = a.grad_out[o];
    const float g = 1.f / (1.f + expf(-s_g[i])), r = s_r[i], x = s_z[(size_t)j * 3 * D + d];
    const float gr = G * g, gg = G * (r - x) * (g * (1.f - g));
    s_r[i] = gr;
    s_g[i] = gg;
    a.g_r[o] = gr;
    a.g_g[o] = gg;
    a.grad_ins[o] = G * (1.f - g);
  }
  __syncthreads();
  for (int i = tid; i < I * 3 * D; i += blockDim.x) {   // g_z = Wr^T g_r + Wg^T g_g  (z is in x_z from here on)
    const int j = i / (3 * D), k = i - j * 3 * D;
    float sr = 0.f, sg = 0.f;
    for (int n = 0; n < D; ++n) {
      sr = fmaf(__ldg(p.Wr[j] + (int64_t)n * 3 * D + k), s_r[(size_t)j * D + n], sr);
      sg = fmaf(__ldg(p.Wg[j] + (int64_t)n * 3 * D + k), s_g[(size_t)j * D + n], sg);
    }
    s_z[i] = sr + sg;
  }
  __syncthreads();
  for (int i = tid; i < I * D; i += blockDim.x) {
    const int j = i / D, d = i - j * D;
    const float* gz = s_z + (size_t)j * 3 * D;
    const int64_t o = ((int64_t)b * I + j) * D + d;
    a.grad_ins[o] = (a.grad_ins[o] + gz[d]) + gz[2 * D + d];
  }
  for (int d = tid; d < D; d += blockDim.x) {
    float gy = 0.f;
    for (int j = 0; j < I; ++j) gy += s_z[(size_t)j * 3 * D + D + d] - s_z[(size_t)j * 3 * D + 2 * D + d];
    s_y[d] = gy;
  }
  __syncthreads();
  T* gh = static_cast<T*>(a.grad_h);
  for_each_seed_chunk(sd, N, sl, [&](int cnt) {
    for (int i = 0; i < cnt; ++i)
      for (int d = tid; d < D; d += blockDim.x) {
        T* e = gh + ((int64_t)b * N + sl.list[i]) * a.ldg + d;
        st_node(e, fmaf(sl.val[i], s_y[d], ld_node(e)));
      }
  });
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

namespace gr {
namespace {

// InsParams of the three instruction entry points: the forward's inputs and the dropout (p in [0, 1); p = 0 ignores
// the seed).  Admits exactly the shapes of gr_instructions: I <= 8 and (Q D + (I + 7) D + 2 Q) floats <= 200 KB.
int ins_params(const char* fn, InsParams& p, const float* hidden, const float* qnode, const int64_t* qtext,
               int64_t pad_id, const float* const* Wq_host, const float* const* bq_host, const float* Wcq,
               const float* bcq, const float* wca, const float* bca, const int64_t* seed, double drop, int B, int Q,
               int D, int I, size_t* smem) {
  GR_CHECK_ARG_AS(fn, hidden && qnode && qtext && Wq_host && bq_host && Wcq && bcq && wca && bca, "null pointer");
  GR_CHECK_ARG_AS(fn, B > 0 && Q > 0 && D > 0 && I > 0 && I <= kMaxIns, "bad shape (num_ins <= 8)");
  GR_CHECK_ARG_AS(fn, drop >= 0.0 && drop < 1.0, "dropout probability outside [0, 1)");
  GR_CHECK_ARG_AS(fn, drop == 0.0 || seed, "null seed with p > 0");
  p.hidden = hidden; p.qnode = qnode; p.qtext = qtext; p.pad = pad_id;
  for (int i = 0; i < I; ++i) {
    GR_CHECK_ARG_AS(fn, Wq_host[i] && bq_host[i], "null question_linear pointer");
    p.Wq[i] = Wq_host[i];
    p.bq[i] = bq_host[i];
  }
  p.Wcq = Wcq; p.bcq = bcq; p.wca = wca; p.bca = bca;
  p.B = B; p.Q = Q; p.D = D; p.I = I;
  p.seed = drop > 0.0 ? seed : nullptr;
  p.p = (float)drop;
  p.scale = (float)(1.0 / (1.0 - drop));
  *smem = ((size_t)Q * D + (size_t)(I + 7) * D + 2 * (size_t)Q) * sizeof(float);
  GR_CHECK_ARG_AS(fn, *smem <= 200 * 1024, "question length x entity_dim too large for shared memory");
  return GR_OK;
}

int launch_instructions(const char* fn, const InsParams& p, size_t smem, cudaStream_t stream) {
  auto go = [&](auto drop) -> int {
    constexpr bool kDrop = decltype(drop)::value;
    if (int rc = opt_in_smem<instructions_kernel<kDrop>>(fn, 200 * 1024)) return rc;
    instructions_kernel<kDrop><<<p.B, kQThreads, smem, stream>>>(p);
    GR_CHECK_LAUNCH_AS(fn);
    return GR_OK;
  };
  return p.p > 0.f ? go(std::true_type{}) : go(std::false_type{});
}

// the backward keeps Q D + 8 D + Q floats in shared memory: never more than the forward's Q D + (I + 7) D + 2 Q
int launch_instructions_bwd(const char* fn, const InsBwdParams& a, cudaStream_t stream) {
  const InsParams& p = a.f;
  const size_t smem = ((size_t)p.Q * p.D + 8 * (size_t)p.D + (size_t)p.Q) * sizeof(float);
  auto go = [&](auto drop) -> int {
    constexpr bool kDrop = decltype(drop)::value;
    if (int rc = opt_in_smem<instructions_bwd_kernel<kDrop>>(fn, 200 * 1024)) return rc;
    instructions_bwd_kernel<kDrop><<<p.B, kQThreads, smem, stream>>>(a);
    GR_CHECK_LAUNCH_AS(fn);
    return GR_OK;
  };
  return p.p > 0.f ? go(std::true_type{}) : go(std::false_type{});
}

// ReformParams of the reform entry points.  Admits exactly the shapes of gr_query_reform: D <= 1024, I <= 8 and
// (5I + 1) D floats <= 48 KB.
int reform_params(const char* fn, ReformParams& p, const float* seed_info, const void* h, int64_t ldh,
                  const float* ins_in, const float* const* Wr_host, const float* const* Wg_host, int B, int N, int D,
                  int I, uint32_t io, size_t* smem) {
  if (int rc = check_io(fn, io)) return rc;
  GR_CHECK_ARG_AS(fn, seed_info && h && ins_in && Wr_host && Wg_host, "null pointer");
  GR_CHECK_ARG_AS(fn, B > 0 && N > 0 && D > 0 && D <= kQThreads && ldh >= D && I > 0 && I <= kMaxIns,
                  "bad shape (D <= 1024, num_ins <= 8)");
  p.seed = seed_info; p.h = h; p.ldh = ldh; p.ins_in = ins_in;
  for (int j = 0; j < I; ++j) {
    GR_CHECK_ARG_AS(fn, Wr_host[j] && Wg_host[j], "null fusion weight pointer");
    p.Wr[j] = Wr_host[j];
    p.Wg[j] = Wg_host[j];
  }
  p.B = B; p.N = N; p.D = D; p.I = I;
  *smem = ((size_t)1 + 5 * (size_t)I) * D * sizeof(float);
  GR_CHECK_ARG_AS(fn, *smem <= 48 * 1024, "num_ins x entity_dim too large for shared memory");
  return GR_OK;
}

// The kernels' static seed list (SeedList, ~8 KB) comes on top of the dynamic area: without the opt-in, static +
// dynamic is capped at 48 KB and every admitted shape with (5I+1)*D > ~10200 fails to launch.
int launch_query_reform(const char* fn, const ReformParams& p, size_t smem, uint32_t io, cudaStream_t stream) {
  const int slices = p.D >= 128 ? 4 : (p.D >= 64 ? 2 : 1);
  return with_node_type(io, [&](auto t) -> int {
    using T = typename decltype(t)::type;
    if (int rc = opt_in_smem<query_reform_kernel<T>>(fn, 48 * 1024)) return rc;
    query_reform_kernel<T><<<dim3((unsigned)p.B, (unsigned)slices), kQThreads, smem, stream>>>(p);
    GR_CHECK_LAUNCH_AS(fn);
    return GR_OK;
  });
}

int launch_query_reform_bwd(const char* fn, const ReformBwdParams& a, size_t smem, uint32_t io, cudaStream_t stream) {
  return with_node_type(io, [&](auto t) -> int {
    using T = typename decltype(t)::type;
    if (int rc = opt_in_smem<query_reform_bwd_kernel<T>>(fn, 48 * 1024)) return rc;
    query_reform_bwd_kernel<T><<<a.f.B, kQThreads, smem, stream>>>(a);
    GR_CHECK_LAUNCH_AS(fn);
    return GR_OK;
  });
}

}  // namespace
}  // namespace gr

extern "C" int gr_instructions(const float* hidden, const float* qnode, const int64_t* qtext, int64_t pad_id,
                               const float* const* Wq_host, const float* const* bq_host, const float* Wcq,
                               const float* bcq, const float* wca, const float* bca, float* out,
                               float* attn_out, int B, int Q, int D, int I, void* stream_) {
  using namespace gr;
  InsParams p{};
  size_t smem = 0;
  if (int rc = ins_params(__func__, p, hidden, qnode, qtext, pad_id, Wq_host, bq_host, Wcq, bcq, wca, bca, nullptr,
                          0.0, B, Q, D, I, &smem))
    return rc;
  GR_CHECK_ARG(out, "null pointer");
  p.out = out; p.attn_out = attn_out;
  return launch_instructions(__func__, p, smem, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_instructions_train(const float* hidden, const float* qnode, const int64_t* qtext, int64_t pad_id,
                                     const float* const* Wq_host, const float* const* bq_host, const float* Wcq,
                                     const float* bcq, const float* wca, const float* bca, const int64_t* seed,
                                     double p_drop, float* out, float* attn_out, int B, int Q, int D, int I,
                                     void* stream_) {
  using namespace gr;
  InsParams p{};
  size_t smem = 0;
  if (int rc = ins_params(__func__, p, hidden, qnode, qtext, pad_id, Wq_host, bq_host, Wcq, bcq, wca, bca, seed,
                          p_drop, B, Q, D, I, &smem))
    return rc;
  GR_CHECK_ARG(out && attn_out, "null pointer");
  p.out = out; p.attn_out = attn_out;
  return launch_instructions(__func__, p, smem, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_instructions_backward(const float* hidden, const float* qnode, const int64_t* qtext, int64_t pad_id,
                                        const float* const* Wq_host, const float* const* bq_host, const float* Wcq,
                                        const float* bcq, const float* wca, const float* bca, const int64_t* seed,
                                        double p_drop, const float* ri, const float* attn, const float* grad_out,
                                        float* grad_hidden, float* grad_qnode, float* g_q, float* x_q, float* g_cq,
                                        float* x_cq, float* g_ca, float* x_ca, int B, int Q, int D, int I,
                                        void* stream_) {
  using namespace gr;
  InsBwdParams a{};
  size_t smem = 0;
  if (int rc = ins_params(__func__, a.f, hidden, qnode, qtext, pad_id, Wq_host, bq_host, Wcq, bcq, wca, bca, seed,
                          p_drop, B, Q, D, I, &smem))
    return rc;
  GR_CHECK_ARG(ri && attn && grad_out && grad_hidden && grad_qnode && g_q && x_q && g_cq && x_cq && g_ca && x_ca,
               "null pointer");
  a.ri = ri; a.attn = attn; a.grad_out = grad_out; a.grad_hidden = grad_hidden; a.grad_qnode = grad_qnode;
  a.g_q = g_q; a.x_q = x_q; a.g_cq = g_cq; a.x_cq = x_cq; a.g_ca = g_ca; a.x_ca = x_ca;
  return launch_instructions_bwd(__func__, a, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int gr_instructions_dropout_mask(const int64_t* seed, double p, int B, int Q, int D, int I, uint8_t* mask_q,
                                            uint8_t* mask_cq, uint8_t* mask_ca, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(seed && mask_q && mask_cq && mask_ca, "null pointer");
  GR_CHECK_ARG(B > 0 && Q > 0 && D > 0 && I > 0 && I <= kMaxIns, "bad shape (num_ins <= 8)");
  GR_CHECK_ARG(p > 0.0 && p < 1.0, "dropout probability outside (0, 1)");
  const int64_t total = (int64_t)B * I * D * (5 + (int64_t)Q);
  const int grid = (int)std::min<int64_t>(ceil_div(total, 256), 8192);
  instructions_dropout_mask_kernel<<<grid, 256, 0, stream>>>(seed, (float)p, B, Q, D, I, mask_q, mask_cq, mask_ca);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

namespace gr {
namespace {

// gr_query_reform and gr_query_reform_ex; errors name the entry point `fn`
int query_reform_entry(const char* fn, const float* seed_info, const void* h, int64_t ldh, const float* ins_in,
                       const float* const* Wr_host, const float* const* Wg_host, float* ins_out, float* seed_out,
                       int B, int N, int D, int I, uint32_t io, void* stream_) {
  ReformParams p{};
  size_t smem = 0;
  if (int rc = reform_params(fn, p, seed_info, h, ldh, ins_in, Wr_host, Wg_host, B, N, D, I, io, &smem)) return rc;
  GR_CHECK_ARG_AS(fn, ins_out, "null pointer");
  p.ins_out = ins_out; p.seed_out = seed_out;
  return launch_query_reform(fn, p, smem, io, reinterpret_cast<cudaStream_t>(stream_));
}

}  // namespace
}  // namespace gr

extern "C" int gr_query_reform(const float* seed_info, const float* h, int64_t ldh, const float* ins_in,
                               const float* const* Wr_host, const float* const* Wg_host, float* ins_out,
                               float* seed_out, int B, int N, int D, int I, void* stream_) {
  return gr::query_reform_entry(__func__, seed_info, h, ldh, ins_in, Wr_host, Wg_host, ins_out, seed_out, B, N, D, I,
                                0u, stream_);
}

extern "C" int gr_query_reform_ex(const float* seed_info, const void* h, int64_t ldh, const float* ins_in,
                                  const float* const* Wr_host, const float* const* Wg_host, float* ins_out,
                                  float* seed_out, int B, int N, int D, int I, uint32_t io, void* stream_) {
  return gr::query_reform_entry(__func__, seed_info, h, ldh, ins_in, Wr_host, Wg_host, ins_out, seed_out, B, N, D, I,
                                io, stream_);
}

extern "C" int gr_query_reform_backward(const float* seed_info, const void* h, int64_t ldh, const float* ins_in,
                                        const float* const* Wr_host, const float* const* Wg_host,
                                        const float* grad_out, float* grad_ins, void* grad_h, int64_t ldg, float* g_r,
                                        float* g_g, float* x_z, int B, int N, int D, int I, uint32_t io,
                                        void* stream_) {
  using namespace gr;
  ReformBwdParams a{};
  size_t smem = 0;
  if (int rc = reform_params(__func__, a.f, seed_info, h, ldh, ins_in, Wr_host, Wg_host, B, N, D, I, io, &smem))
    return rc;
  GR_CHECK_ARG(grad_out && grad_ins && grad_h && g_r && g_g && x_z, "null pointer");
  GR_CHECK_ARG(ldg >= D, "bad grad_h row stride");
  a.grad_out = grad_out; a.grad_ins = grad_ins; a.grad_h = grad_h; a.ldg = ldg; a.g_r = g_r; a.g_g = g_g; a.x_z = x_z;
  return launch_query_reform_bwd(__func__, a, smem, io, reinterpret_cast<cudaStream_t>(stream_));
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
