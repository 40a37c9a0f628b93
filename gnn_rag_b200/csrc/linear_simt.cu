// fp32 SIMT linear layer: C = act(A W^T + bias) (+ addend).  Exact-fp32 path of gr_linear: used for the
// hoisted relation projection rel_linear_k(rel_features) (reference reasongnn.py:79,105 applies the same
// Linear to F gathered rows), for small problems, and as the validator of the split-bf16 wgmma path
// (linear_tc.cu).  Classic 128x64x16 shared-memory tiling, 8x4 outputs per thread.
#include "common.cuh"

namespace gr {
namespace {

constexpr int BM = 128, BN = 64, BK = 16, TM = 8, TN = 4;
constexpr int kThreads = (BM / TM) * (BN / TN);   // 256

__global__ void __launch_bounds__(kThreads)
linear_simt_kernel(const float* __restrict__ A, int64_t lda, const float* __restrict__ W, int64_t ldw,
                   const float* __restrict__ bias, const float* __restrict__ addend,
                   int64_t ld_addend, int64_t addend_rows, float* __restrict__ C, int64_t ldc,
                   int64_t M, int64_t N, int64_t K, uint32_t flags, int vec_ok) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Ws[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int64_t m0 = (int64_t)blockIdx.x * BM, n0 = (int64_t)blockIdx.y * BN;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int64_t k0 = 0; k0 < K; k0 += BK) {
    // A tile: 128 x 16 -> each thread 2 x (4 consecutive k)
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      int r = tid / 4 + it * 64, kk = (tid % 4) * 4;
      int64_t m = m0 + r, k = k0 + kk;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (m < M) {
        const float* src = A + m * lda + k;
        if (vec_ok && k + 3 < K) {
          float4 t = __ldg(reinterpret_cast<const float4*>(src));
          v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (k + q < K) v[q] = __ldg(src + q);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) As[kk + q][r] = v[q];
    }
    // W tile: 64 x 16 -> each thread 1 x (4 consecutive k)
    {
      int r = tid / 4, kk = (tid % 4) * 4;
      int64_t n = n0 + r, k = k0 + kk;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (n < N) {
        const float* src = W + n * ldw + k;
        if (vec_ok && k + 3 < K) {
          float4 t = __ldg(reinterpret_cast<const float4*>(src));
          v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (k + q < K) v[q] = __ldg(src + q);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) Ws[kk + q][r] = v[q];
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
      float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * TM]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * TM + 4]);
      float4 b0 = *reinterpret_cast<const float4*>(&Ws[kk][tx * TN]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w;
      a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  const bool relu = flags & GR_LINEAR_RELU;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int64_t m = m0 + ty * TM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int64_t n = n0 + tx * TN + j;
      if (n >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[n];
      if (addend && m < addend_rows) v += addend[m * ld_addend + n];
      if (relu) v = fmaxf(v, 0.f);
      C[m * ldc + n] = v;
    }
  }
}

}  // namespace

int linear_simt(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias,
                const float* addend, int64_t ld_addend, int64_t addend_rows, float* C, int64_t ldc,
                int64_t M, int64_t N, int64_t K, uint32_t flags, cudaStream_t stream) {
  int vec_ok = (lda % 4 == 0) && (ldw % 4 == 0) && (reinterpret_cast<size_t>(A) % 16 == 0) &&
               (reinterpret_cast<size_t>(W) % 16 == 0);
  dim3 grid((unsigned)ceil_div(M, BM), (unsigned)ceil_div(N, BN));
  linear_simt_kernel<<<grid, kThreads, 0, stream>>>(A, lda, W, ldw, bias, addend, ld_addend,
                                                    addend_rows, C, ldc, M, N, K, flags, vec_ok);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

}  // namespace gr
