// Library-wide entry points: version, error string, options, gr_linear dispatch.
#include <stdarg.h>

#include "common.cuh"

namespace gr {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached = 0;
  if (cached) return cached;
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) == cudaSuccess &&
      cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
    cached = n;
  else
    cached = kNumSMs;
  return cached;
}

extern int g_opt_agg_tma;
extern int g_tc_cluster;
extern int g_tc_bk;
extern int g_tc_tma_store;
extern int g_opt_agg_abs_ws;
extern int g_fused_debug;

int linear_simt(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias,
                const float* addend, int64_t ld_addend, int64_t addend_rows, float* C, int64_t ldc,
                int64_t M, int64_t N, int64_t K, uint32_t flags, cudaStream_t stream);

}  // namespace gr

extern "C" int gr_abi_version(void) { return GR_ABI_VERSION; }

extern "C" const char* gr_last_error(void) { return gr::g_err; }

extern "C" int gr_set_option(const char* name, int64_t value) {
  using namespace gr;
  GR_CHECK_ARG(name != nullptr, "null option name");
  if (!strcmp(name, "agg_tma")) { g_opt_agg_tma = (int)value; return GR_OK; }
  if (!strcmp(name, "tc_cluster")) { g_tc_cluster = (int)value; return GR_OK; }
  if (!strcmp(name, "tc_bk")) { g_tc_bk = (int)value; return GR_OK; }
  if (!strcmp(name, "tc_tma_store")) { g_tc_tma_store = (int)value; return GR_OK; }
  if (!strcmp(name, "agg_abs_ws")) { g_opt_agg_abs_ws = (int)value; return GR_OK; }
  if (!strcmp(name, "fused_debug")) { g_fused_debug = (int)value; return GR_OK; }
  set_error("gr_set_option: unknown option '%s'", name);
  return GR_ERR_INVALID_ARG;
}

extern "C" int gr_linear(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias,
                         const float* addend, int64_t ld_addend, int64_t addend_rows, float* C,
                         int64_t ldc, int64_t M, int64_t N, int64_t K, uint32_t flags,
                         void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(A && W && C, "null pointer");
  GR_CHECK_ARG(M > 0 && N > 0 && K > 0, "M, N, K must be positive");
  GR_CHECK_ARG(lda >= K && ldw >= K && ldc >= N, "leading dimension smaller than row length");
  GR_CHECK_ARG(!addend || ld_addend >= N, "ld_addend smaller than N");
  return linear_simt(A, lda, W, ldw, bias, addend, ld_addend, addend_rows, C, ldc, M, N, K, flags,
                     stream);
}
