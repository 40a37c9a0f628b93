// Micro-benchmark: how fast can 800-byte rows of a 12.5 MB table (L2 resident) be gathered at random by all SMs?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o gather_bw gather_bw.cu && ./gather_bw
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <vector>

template <int U>
__global__ void gather_ldg(const float* __restrict__ tab, const int* __restrict__ rel, int nedges, float* out) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  float4 acc0 = make_float4(0, 0, 0, 0), acc1 = acc0;
  const bool ld1 = 128 + lane * 4 < 200;
  for (int e = gw * U; e + U <= nedges; e += nw * U) {
    float4 v0[U], v1[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const char* a = reinterpret_cast<const char*>(tab) + (size_t)__ldg(rel + e + u) * 1024 + lane * 16;
      v0[u] = __ldg(reinterpret_cast<const float4*>(a));
      v1[u] = ld1 ? __ldg(reinterpret_cast<const float4*>(a + 512)) : make_float4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      acc0.x += v0[u].x; acc0.y += v0[u].y; acc0.z += v0[u].z; acc0.w += v0[u].w;
      acc1.x += v1[u].x; acc1.y += v1[u].y; acc1.z += v1[u].z; acc1.w += v1[u].w;
    }
  }
  if (acc0.x + acc0.y + acc0.z + acc0.w + acc1.x + acc1.y + acc1.z + acc1.w == 12345.678f) out[0] = 1.f;
}

// one bulk copy per row into a per-warp smem ring, NS slots, completion per slot group via mbarrier
__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
template <int NS>
__global__ void gather_bulk(const float* __restrict__ tab, const int* __restrict__ rel, int nedges, float* out) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwb = blockDim.x >> 5;
  __shared__ __align__(8) unsigned long long bars[32][2];
  unsigned char* ring = smem + (size_t)warp * 2 * NS * 800;
  if (lane == 0) {
    for (int b = 0; b < 2; ++b) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(&bars[warp][b])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  const int gw = blockIdx.x * nwb + warp, nw = gridDim.x * nwb;
  float4 acc0 = make_float4(0, 0, 0, 0), acc1 = acc0;
  const bool ld1 = 128 + lane * 4 < 200;
  int it = 0;
  auto issue = [&](int e, int stage) {
    if (lane == 0)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(&bars[warp][stage])), "r"(NS * 800) : "memory");
    __syncwarp();
    if (lane < NS) {
      const char* a = reinterpret_cast<const char*>(tab) + (size_t)__ldg(rel + e + lane) * 1024;
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                       s32(ring + (stage * NS + lane) * 800)),
                   "l"(a), "r"(800), "r"(s32(&bars[warp][stage]))
                   : "memory");
    }
  };
  int e = gw * NS;
  if (e + NS <= nedges) issue(e, 0);
  for (; e + NS <= nedges; e += nw * NS, ++it) {
    const int stage = it & 1;
    if (e + nw * NS + NS <= nedges) issue(e + nw * NS, stage ^ 1);
    uint32_t ok = 0;
    while (!ok)
      asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                   : "=r"(ok) : "r"(s32(&bars[warp][stage])), "r"((it >> 1) & 1) : "memory");
#pragma unroll
    for (int u = 0; u < NS; ++u) {
      const unsigned char* a = ring + (stage * NS + u) * 800 + lane * 16;
      const float4 v0 = *reinterpret_cast<const float4*>(a);
      const float4 v1 = ld1 ? *reinterpret_cast<const float4*>(a + 512) : make_float4(0, 0, 0, 0);
      acc0.x += v0.x; acc0.y += v0.y; acc0.z += v0.z; acc0.w += v0.w;
      acc1.x += v1.x; acc1.y += v1.y; acc1.z += v1.z; acc1.w += v1.w;
    }
  }
  if (acc0.x + acc0.y + acc0.z + acc0.w + acc1.x + acc1.y + acc1.z + acc1.w == 12345.678f) out[0] = 1.f;
}

int main() {
  const int R = 12214, E = 1 << 20;
  float* tab; int* rel; float* out;
  cudaMalloc(&tab, (size_t)R * 1024); cudaMalloc(&rel, E * 4); cudaMalloc(&out, 4);
  cudaMemset(tab, 0, (size_t)R * 1024);
  std::vector<int> h(E);
  srand(1);
  for (int i = 0; i < E; ++i) h[i] = rand() % R;
  cudaMemcpy(rel, h.data(), E * 4, cudaMemcpyHostToDevice);
  cudaEvent_t s, e; cudaEventCreate(&s); cudaEventCreate(&e);
  auto time = [&](auto launch, const char* name) {
    for (int i = 0; i < 3; ++i) launch();
    float best = 1e9;
    for (int i = 0; i < 10; ++i) {
      cudaEventRecord(s); launch(); cudaEventRecord(e); cudaEventSynchronize(e);
      float ms; cudaEventElapsedTime(&ms, s, e); best = ms < best ? ms : best;
    }
    printf("%-40s %8.1f us  %6.2f TB/s  (%s)\n", name, best * 1e3, (double)E * 800 / (best * 1e-3) / 1e12,
           cudaGetErrorString(cudaGetLastError()));
  };
  for (int wps : {16, 32, 48, 64}) {
    const int threads = 256, blocks = 132 * wps / 8;   // one wave on the 132 SMs of an H100 SXM
    char nm[64];
    snprintf(nm, 64, "ldg U=1 warps/SM=%d", wps); time([&] { gather_ldg<1><<<blocks, threads>>>(tab, rel, E, out); }, nm);
    snprintf(nm, 64, "ldg U=2 warps/SM=%d", wps); time([&] { gather_ldg<2><<<blocks, threads>>>(tab, rel, E, out); }, nm);
    snprintf(nm, 64, "ldg U=4 warps/SM=%d", wps); time([&] { gather_ldg<4><<<blocks, threads>>>(tab, rel, E, out); }, nm);
    snprintf(nm, 64, "ldg U=8 warps/SM=%d", wps); time([&] { gather_ldg<8><<<blocks, threads>>>(tab, rel, E, out); }, nm);
  }
  for (int wpb : {8, 16}) {
    {
      const size_t smem = (size_t)wpb * 2 * 4 * 800;
      cudaFuncSetAttribute(gather_bulk<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      char nm[64]; snprintf(nm, 64, "bulk NS=4 x2 stages, %d warps/CTA, 2 CTA/SM", wpb);
      time([&] { gather_bulk<4><<<296, wpb * 32, smem>>>(tab, rel, E, out); }, nm);
    }
    {
      const size_t smem = (size_t)wpb * 2 * 8 * 800;
      cudaFuncSetAttribute(gather_bulk<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      char nm[64]; snprintf(nm, 64, "bulk NS=8 x2 stages, %d warps/CTA, 1-2 CTA/SM", wpb);
      time([&] { gather_bulk<8><<<296, wpb * 32, smem>>>(tab, rel, E, out); }, nm);
    }
  }
  return 0;
}
