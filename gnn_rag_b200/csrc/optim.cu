// Gradient clipping + Adam over fp32 tensor lists (the tail of a training iteration, gnn/train_model.py:221-230):
// torch.nn.utils.clip_grad_norm_ followed by torch.optim.Adam.step() on torch's default CUDA path
// (torch.optim.adam._multi_tensor_adam: foreach, not capturable), one launch for the norm and one for the update.
//
// The work is cut into chunks of kChunk elements of one tensor each, listed by the caller; one CTA per chunk.
// gr_grad_sumsq writes each chunk's sum of g^2 (float64) to its own slot.  gr_clip_adam reduces the slots in one
// fixed order in every CTA (the same sum everywhere, no atomics, no second pass), forms torch's clip coefficient and
// then clips and updates its chunk element by element, with torch's rounding for each foreach op.
#include "common.cuh"

namespace gr {
namespace {

constexpr int kChunk = 8192;     // elements per chunk (a multiple of 4: float4 chunks stay aligned)
constexpr int kOptThreads = 256;

// one row of the tensor table (int64 [T][6])
struct AdamTensor {
  float* param;
  float* grad;
  float* exp_avg;      // null: clip only (a parameter the optimizer does not hold)
  float* exp_avg_sq;
  int64_t numel;
  int64_t flags;       // GR_ADAM_ALIGNED16: every pointer of the row is 16-byte aligned
};
static_assert(sizeof(AdamTensor) == 6 * sizeof(int64_t), "tensor table row");

// one row of the per-tensor scalars (fp32 [T][8]), each the fp32 value torch hands its foreach kernel
struct AdamScalars {
  float lerp_w;        // 1 - beta1                    (_foreach_lerp_ weight)
  float beta2;         // beta2                        (_foreach_mul_)
  float one_m_beta2;   // 1 - beta2                    (_foreach_addcmul_ value)
  float eps;           // eps                          (_foreach_add_)
  float wd;            // weight_decay                 (_foreach_add alpha)
  float step_size;     // -(lr / (1 - beta1^t))        (_foreach_addcdiv_ value)
  float bc2_sqrt;      // (1 - beta2^t) ** 0.5         (_foreach_div_)
  float pad;
};
static_assert(sizeof(AdamScalars) == 8 * sizeof(float), "scalar table row");

// ATen/native/Lerp.h in fp32: the branch on |weight| < 0.5, each form with one contraction
__device__ __forceinline__ float lerp_rn(float self, float end, float w) {
  const float d = __fsub_rn(end, self);
  return fabsf(w) < 0.5f ? __fmaf_rn(w, d, self) : __fmaf_rn(-d, __fsub_rn(1.0f, w), end);
}

// one element: clip (g *= coef when clip), then Adam in _multi_tensor_adam's op order.  g is written back to p.grad
// by the caller; weight decay makes a new gradient for the moments only (_foreach_add, not in place).
template <bool WD>
__device__ __forceinline__ void adam_elem(float& p, float g, float& m, float& v, const AdamScalars& s) {
  if (WD && s.wd != 0.0f) g = __fmaf_rn(s.wd, p, g);                 // grad + wd * p
  m = lerp_rn(m, g, s.lerp_w);                                        // exp_avg.lerp_(grad, 1 - beta1)
  v = __fmul_rn(v, s.beta2);                                          // exp_avg_sq.mul_(beta2)
  const float gg = __fmul_rn(g, g);                                   // addcmul_(grad, grad, 1 - beta2)
  v = s.one_m_beta2 == 1.0f ? __fmaf_rn(g, g, v) : __fmaf_rn(s.one_m_beta2, gg, v);
  float d = __fsqrt_rn(v);                                            // sqrt
  d = __fdiv_rn(d, s.bc2_sqrt);                                       // / bias_correction2_sqrt
  d = __fadd_rn(d, s.eps);                                            // + eps
  p = __fmaf_rn(s.step_size, __fdiv_rn(m, d), p);                     // addcdiv_(exp_avg, denom, step_size)
}

// the chunk [beg, end) of tensor `t` of chunk c
__device__ __forceinline__ void chunk_range(const int32_t* chunks, const AdamTensor* table, int c, int& t,
                                            int64_t& beg, int64_t& end) {
  t = chunks[2 * c];
  beg = (int64_t)chunks[2 * c + 1] * kChunk;
  end = min(beg + (int64_t)kChunk, table[t].numel);
}

// fixed-order block sum of one double per thread (warp shuffles, then the warps in order); thread 0 holds the result
__device__ __forceinline__ double block_sum(double x, double* s_warp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
  if (lane_id() == 0) s_warp[warp_id()] = x;
  __syncthreads();
  if (threadIdx.x == 0) {
    x = s_warp[0];
    for (int w = 1; w < kOptThreads / 32; ++w) x += s_warp[w];
  }
  return x;
}

__global__ void __launch_bounds__(kOptThreads) grad_sumsq_kernel(const AdamTensor* __restrict__ table,
                                                                  const int32_t* __restrict__ chunks,
                                                                  double* __restrict__ slots) {
  __shared__ double s_warp[kOptThreads / 32];
  int t;
  int64_t beg, end;
  chunk_range(chunks, table, blockIdx.x, t, beg, end);
  const AdamTensor e = table[t];
  double acc = 0.0;
  int64_t i = beg;
  if (e.flags & GR_ADAM_ALIGNED16) {
    const int64_t n4 = (end - beg) >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(e.grad + beg);
    for (int64_t k = threadIdx.x; k < n4; k += kOptThreads) {
      const float4 g = g4[k];
      acc += (double)g.x * g.x;
      acc += (double)g.y * g.y;
      acc += (double)g.z * g.z;
      acc += (double)g.w * g.w;
    }
    i = beg + 4 * n4;
  }
  for (int64_t k = i + threadIdx.x; k < end; k += kOptThreads) {
    const double g = e.grad[k];
    acc += g * g;
  }
  acc = block_sum(acc, s_warp);
  if (threadIdx.x == 0) slots[blockIdx.x] = acc;
}

template <bool CLIP, bool WD>
__global__ void __launch_bounds__(kOptThreads) clip_adam_kernel(const AdamTensor* __restrict__ table,
                                                                 const AdamScalars* __restrict__ scalars,
                                                                 const int32_t* __restrict__ chunks, int C,
                                                                 const double* __restrict__ slots, float max_norm,
                                                                 float* __restrict__ grad_norm) {
  __shared__ double s_warp[kOptThreads / 32];
  __shared__ float s_coef;
  float coef = 1.0f;
  if (CLIP) {
    double x = 0.0;
    for (int k = threadIdx.x; k < C; k += kOptThreads) x += slots[k];
    x = block_sum(x, s_warp);
    if (threadIdx.x == 0) {
      const float norm = __double2float_rn(__dsqrt_rn(x));
      // clip_grads_with_norm_: clamp(max_norm / (norm + 1e-6), max=1), where float / tensor is
      // tensor.reciprocal() * float; clamp keeps a NaN
      const float c = __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), max_norm);
      s_coef = isnan(c) ? c : fminf(c, 1.0f);
      if (blockIdx.x == 0 && grad_norm) *grad_norm = norm;
    }
    __syncthreads();
    coef = s_coef;
  }
  if ((int)blockIdx.x >= C) return;          // the one CTA of an empty list only writes the norm
  int t;
  int64_t beg, end;
  chunk_range(chunks, table, blockIdx.x, t, beg, end);
  const AdamTensor e = table[t];
  const bool adam = e.exp_avg != nullptr;
  const AdamScalars s = scalars[t];
  int64_t i = beg;
  if (e.flags & GR_ADAM_ALIGNED16) {
    const int64_t n4 = (end - beg) >> 2;
    float4* g4 = reinterpret_cast<float4*>(e.grad + beg);
    float4* p4 = reinterpret_cast<float4*>(e.param + beg);
    float4* m4 = reinterpret_cast<float4*>(e.exp_avg + beg);
    float4* v4 = reinterpret_cast<float4*>(e.exp_avg_sq + beg);
    for (int64_t k = threadIdx.x; k < n4; k += kOptThreads) {
      float4 g = g4[k];
      if (CLIP) {
        g = make_float4(__fmul_rn(g.x, coef), __fmul_rn(g.y, coef), __fmul_rn(g.z, coef), __fmul_rn(g.w, coef));
        g4[k] = g;
      }
      if (adam) {
        float4 p = p4[k], m = m4[k], v = v4[k];
        adam_elem<WD>(p.x, g.x, m.x, v.x, s);
        adam_elem<WD>(p.y, g.y, m.y, v.y, s);
        adam_elem<WD>(p.z, g.z, m.z, v.z, s);
        adam_elem<WD>(p.w, g.w, m.w, v.w, s);
        p4[k] = p;
        m4[k] = m;
        v4[k] = v;
      }
    }
    i = beg + 4 * n4;
  }
  for (int64_t k = i + threadIdx.x; k < end; k += kOptThreads) {
    float g = e.grad[k];
    if (CLIP) {
      g = __fmul_rn(g, coef);
      e.grad[k] = g;
    }
    if (adam) {
      float p = e.param[k], m = e.exp_avg[k], v = e.exp_avg_sq[k];
      adam_elem<WD>(p, g, m, v, s);
      e.param[k] = p;
      e.exp_avg[k] = m;
      e.exp_avg_sq[k] = v;
    }
  }
}

}  // namespace
}  // namespace gr

extern "C" int gr_adam_chunk_elems(void) { return gr::kChunk; }

extern "C" int gr_grad_sumsq(const int64_t* table, const int32_t* chunks, int C, double* slots, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(C >= 0, "C must be >= 0");
  if (C == 0) return GR_OK;
  GR_CHECK_ARG(table && chunks && slots, "null pointer");
  grad_sumsq_kernel<<<C, kOptThreads, 0, stream>>>(reinterpret_cast<const AdamTensor*>(table), chunks, slots);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_clip_adam(const int64_t* table, const float* scalars, const int32_t* chunks, int C,
                            const double* slots, double max_norm, float* grad_norm, uint32_t flags, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(C >= 0, "C must be >= 0");
  GR_CHECK_ARG((flags & ~GR_ADAM_WEIGHT_DECAY) == 0, "unknown flags");
  const bool clip = slots != nullptr;
  GR_CHECK_ARG(!clip || max_norm > 0.0, "max_norm must be > 0 when clipping");
  GR_CHECK_ARG(clip || grad_norm == nullptr, "grad_norm needs the slots of gr_grad_sumsq");
  if (C == 0 && !clip) return GR_OK;
  GR_CHECK_ARG(C == 0 || (table && scalars && chunks), "null pointer");
  const bool wd = (flags & GR_ADAM_WEIGHT_DECAY) != 0;
  auto launch = [&](auto kernel) {
    kernel<<<C > 0 ? C : 1, kOptThreads, 0, stream>>>(reinterpret_cast<const AdamTensor*>(table),
                                                      reinterpret_cast<const AdamScalars*>(scalars), chunks, C,
                                                      slots, (float)max_norm, grad_norm);
  };
  if (clip) {
    if (wd) launch(clip_adam_kernel<true, true>);
    else launch(clip_adam_kernel<true, false>);
  } else {
    if (wd) launch(clip_adam_kernel<false, true>);
    else launch(clip_adam_kernel<false, false>);
  }
  GR_CHECK_LAUNCH();
  return GR_OK;
}
