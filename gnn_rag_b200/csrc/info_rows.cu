// The `.info` file of an evaluation epoch (graphed.EvalRun.info): one JSONL row per question, formatted on the device
// from the epoch's records, byte for byte what evaluate.Evaluator writes with json.dumps.
//
// A row of position p (question q = order[p]) is
//   prefix[q]  "precison": P, "recall": R, "f1": F, "hit": H, "em": E, "cand": [["name", prob], ...]}\n
// The host builds prefix[q] (everything up to and including `"answers": [...], `) and the JSON-escaped name of every
// entity the split can rank once per split; the numbers are Python reprs of float64 values (float_repr.cuh), em an
// int in case 3, each prob the float64 of the fp32 candidate record.
//
//   gr_info_rows_size   one warp per row sizes it (the candidates spread over the lanes), then one CTA scans the sizes
//                       into row offsets.
//   gr_info_rows_write  one warp per row copies the prefix, writes the metrics (lane 0), then the candidates 32 at a
//                       time, each lane at its place from a warp scan of their lengths.
// No atomics: the bytes do not depend on scheduling.
#include "common.cuh"
#include "float_repr.cuh"

namespace gr {
namespace {

constexpr int kRowThreads = 256;
constexpr int kScanThreads = 1024;

// the fixed text of a row around its numbers
__device__ const char kKeyPrecision[] = "\"precison\": ";
__device__ const char kKeyRecall[] = ", \"recall\": ";
__device__ const char kKeyF1[] = ", \"f1\": ";
__device__ const char kKeyHit[] = ", \"hit\": ";
__device__ const char kKeyEm[] = ", \"em\": ";
__device__ const char kKeyCand[] = ", \"cand\": [";
__device__ const char kRowEnd[] = "]}\n";
constexpr int kMetricKeyBytes = 12 + 12 + 8 + 9 + 8 + 11;
constexpr int kRowEndBytes = 3;

// per-row flags (gr_info_rows_size's summary[1])
constexpr int kBadRecord = 2;   // question id outside [0, num_q), or candidates outside the records in use
constexpr int kNoName = 4;      // a candidate entity without a name

struct Row {
  int64_t q, off;   // question id, first candidate record
  int count;        // candidates
  int flags;
};

__device__ __forceinline__ Row load_row(int64_t p, const int32_t* counts, const int64_t* cand_off,
                                        const int64_t* cand_total, int64_t capacity, const int64_t* order,
                                        int64_t num_q) {
  Row r;
  r.q = order[p];
  r.off = cand_off[p];
  r.count = counts[p];
  const int64_t used = min(*cand_total, capacity);
  r.flags = (r.q < 0 || r.q >= num_q || r.count < 0 || r.off < 0 || r.off > used - r.count) ? kBadRecord : 0;
  if (r.flags) r.count = 0;
  return r;
}

// metric k of the row as printed: em of case 3 is an int
__device__ __forceinline__ bool em_is_int(int k, int8_t cs) { return k == 4 && cs == 3; }

__device__ __forceinline__ int metrics_len(const double* m, int8_t cs) {
  int n = kMetricKeyBytes;
#pragma unroll 1
  for (int k = 0; k < 5; ++k) n += em_is_int(k, cs) ? 1 : fr::repr_len(fr::shortest(m[k]));
  return n;
}

// candidate k of a row: its entity and probability
__device__ __forceinline__ void load_cand(const int64_t* cand, int64_t rec, int64_t& ent, double& prob) {
  const longlong2 v = *reinterpret_cast<const longlong2*>(cand + 2 * rec);
  ent = v.x;
  prob = (double)__int_as_float((int)((uint64_t)v.y >> 32));
}

__device__ __forceinline__ int name_slot_of(int64_t ent, const int32_t* name_slot, int64_t num_entity,
                                            int64_t num_names) {
  const int s = ent >= 0 && ent < num_entity ? name_slot[ent] : -1;
  return s < num_names ? s : -1;
}

// bytes of candidate k: ", " (k > 0) "[" name ", " repr "]"
__device__ __forceinline__ int cand_len(int k, int64_t name_bytes, const fr::Decimal& d) {
  return (k > 0 ? 2 : 0) + 4 + (int)name_bytes + fr::repr_len(d);
}

__global__ void __launch_bounds__(kRowThreads)
info_rows_size_kernel(const double* __restrict__ metrics, const int8_t* __restrict__ cases,
                      const int32_t* __restrict__ counts, const int64_t* __restrict__ cand_off,
                      const int64_t* __restrict__ cand_total, int64_t num_data, const int64_t* __restrict__ cand,
                      int64_t capacity, const int64_t* __restrict__ order, const int64_t* __restrict__ prefix_off,
                      int64_t num_q, const int32_t* __restrict__ name_slot, int64_t num_entity,
                      const int64_t* __restrict__ name_off, int64_t num_names, int64_t* __restrict__ row_off) {
  const int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (p >= num_data) return;
  const int lane = lane_id();
  const Row r = load_row(p, counts, cand_off, cand_total, capacity, order, num_q);
  int64_t bytes = 0;
  int flags = r.flags;
  for (int k = lane; k < r.count; k += 32) {
    int64_t ent;
    double prob;
    load_cand(cand, r.off + k, ent, prob);
    const int s = name_slot_of(ent, name_slot, num_entity, num_names);
    if (s < 0) flags |= kNoName;
    const int64_t nb = s < 0 ? 0 : name_off[s + 1] - name_off[s];
    bytes += cand_len(k, nb, fr::shortest(prob));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, o);
  flags = __reduce_or_sync(0xffffffffu, flags);
  if (lane == 0) {
    if (!flags) bytes += prefix_off[r.q + 1] - prefix_off[r.q] + metrics_len(metrics + 5 * p, cases[p]) + kRowEndBytes;
    row_off[p + 1] = flags ? -(int64_t)flags : bytes;      // the scan turns a negative entry into the flags
  }
}

// row_off[1 .. n] holds the row sizes (or -flags): scanned in place into the offsets, row_off[0] = 0.
// summary = (total bytes, flags): flags 1 when a status word of the run is nonzero, else the rows' flags OR-ed; the
// total is 0 when any flag is set.
__global__ void __launch_bounds__(kScanThreads)
info_rows_scan_kernel(const int32_t* __restrict__ eval_status, int64_t num_data, int64_t* __restrict__ row_off,
                      int64_t* __restrict__ summary) {
  constexpr int kWarps = kScanThreads / 32;
  __shared__ int64_t s_warp[kWarps];
  __shared__ int64_t s_base;
  __shared__ int s_flags[kWarps];
  const int lane = lane_id(), warp = warp_id();
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  int flags = 0;
  for (int64_t j0 = 0; j0 < num_data; j0 += kScanThreads) {
    const int64_t j = j0 + threadIdx.x;
    int64_t n = j < num_data ? row_off[j + 1] : 0;
    if (n < 0) {
      flags |= (int)-n;
      n = 0;
    }
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
    if (j < num_data) row_off[j + 1] = before + v;
    __syncthreads();                                 // every thread has read s_base and s_warp
    if (threadIdx.x == kScanThreads - 1) s_base = before + v;
    __syncthreads();
  }
  flags = __reduce_or_sync(0xffffffffu, flags);
  if (lane == 0) s_flags[warp] = flags;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kWarps; ++w) flags |= s_flags[w];
    const int status = eval_status[0] | eval_status[1] | eval_status[2] | eval_status[3];
    if (status) flags = 1;
    row_off[0] = 0;
    summary[0] = flags ? 0 : s_base;
    summary[1] = flags;
  }
}

template <int N>
__device__ __forceinline__ uint8_t* put_text(uint8_t* o, const char (&s)[N]) {
#pragma unroll
  for (int i = 0; i < N - 1; ++i) o[i] = (uint8_t)s[i];
  return o + N - 1;
}

__device__ __forceinline__ uint8_t* put_metric(uint8_t* o, double v, bool as_int) {
  if (as_int) {
    *o = v != 0.0 ? '1' : '0';
    return o + 1;
  }
  const fr::Decimal d = fr::shortest(v);
  fr::write_repr(d, o);
  return o + fr::repr_len(d);
}

__global__ void __launch_bounds__(kRowThreads)
info_rows_write_kernel(const double* __restrict__ metrics, const int8_t* __restrict__ cases,
                       const int32_t* __restrict__ counts, const int64_t* __restrict__ cand_off,
                       const int64_t* __restrict__ cand_total, int64_t num_data, const int64_t* __restrict__ cand,
                       int64_t capacity, const int64_t* __restrict__ order, const uint8_t* __restrict__ prefix,
                       const int64_t* __restrict__ prefix_off, int64_t num_q, const int32_t* __restrict__ name_slot,
                       int64_t num_entity, const uint8_t* __restrict__ names, const int64_t* __restrict__ name_off,
                       int64_t num_names, const int64_t* __restrict__ row_off, const int64_t* __restrict__ summary,
                       uint8_t* __restrict__ out, int64_t out_bytes) {
  const int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (p >= num_data || summary[1] != 0 || summary[0] > out_bytes) return;
  const int lane = lane_id();
  const Row r = load_row(p, counts, cand_off, cand_total, capacity, order, num_q);
  uint8_t* o = out + row_off[p];
  const int64_t pb = prefix_off[r.q], plen = prefix_off[r.q + 1] - pb;
  for (int64_t i = lane; i < plen; i += 32) o[i] = prefix[pb + i];
  o += plen;
  int mlen = 0;
  if (lane == 0) {
    const double* m = metrics + 5 * p;
    const int8_t cs = cases[p];
    uint8_t* w = put_text(o, kKeyPrecision);
    w = put_metric(w, m[0], false);
    w = put_text(w, kKeyRecall);
    w = put_metric(w, m[1], false);
    w = put_text(w, kKeyF1);
    w = put_metric(w, m[2], false);
    w = put_text(w, kKeyHit);
    w = put_metric(w, m[3], false);
    w = put_text(w, kKeyEm);
    w = put_metric(w, m[4], em_is_int(4, cs));
    w = put_text(w, kKeyCand);
    mlen = (int)(w - o);
  }
  o += __shfl_sync(0xffffffffu, mlen, 0);
  for (int k0 = 0; k0 < r.count; k0 += 32) {
    const int k = k0 + lane;
    int len = 0;
    int64_t nb = 0, ns = 0;
    fr::Decimal d;
    if (k < r.count) {
      int64_t ent;
      double prob;
      load_cand(cand, r.off + k, ent, prob);
      const int s = name_slot_of(ent, name_slot, num_entity, num_names);   // >= 0: the size pass checked it
      ns = name_off[s];
      nb = name_off[s + 1] - ns;
      d = fr::shortest(prob);
      len = cand_len(k, nb, d);
    }
    int at = len;                                    // inclusive scan of the lengths over the lanes
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, at, off);
      if (lane >= off) at += t;
    }
    if (k < r.count) {
      uint8_t* w = o + at - len;
      if (k > 0) {
        *w++ = ',';
        *w++ = ' ';
      }
      *w++ = '[';
      for (int64_t i = 0; i < nb; ++i) w[i] = names[ns + i];
      w += nb;
      *w++ = ',';
      *w++ = ' ';
      fr::write_repr(d, w);
      w[fr::repr_len(d)] = ']';
    }
    o += __shfl_sync(0xffffffffu, at, 31);
  }
  if (lane == 0) put_text(o, kRowEnd);
}

}  // namespace
}  // namespace gr

extern "C" int gr_info_rows_size(const double* metrics, const int8_t* cases, const int32_t* counts,
                                 const int64_t* cand_off, const int64_t* cand_total, const int32_t* eval_status,
                                 int64_t num_data, const int64_t* cand, int64_t capacity, const int64_t* order,
                                 const int64_t* prefix_off, int64_t num_q, const int32_t* name_slot,
                                 int64_t num_entity, const int64_t* name_off, int64_t num_names, int64_t* row_off,
                                 int64_t* summary, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(metrics && cases && counts && cand_off && cand_total && eval_status && cand && order && prefix_off &&
               name_slot && name_off, "null pointer");
  GR_CHECK_ARG(row_off && summary, "null output");
  GR_CHECK_ARG(num_data >= 0 && capacity >= 0 && num_q >= 0 && num_entity >= 0 && num_names >= 0,
               "need num_data, capacity, num_q, num_entity and num_names >= 0");
  if (num_data > 0) {
    info_rows_size_kernel<<<(unsigned)ceil_div(num_data * 32, kRowThreads), kRowThreads, 0, stream>>>(
        metrics, cases, counts, cand_off, cand_total, num_data, cand, capacity, order, prefix_off, num_q, name_slot,
        num_entity, name_off, num_names, row_off);
    GR_CHECK_LAUNCH();
  }
  info_rows_scan_kernel<<<1, kScanThreads, 0, stream>>>(eval_status, num_data, row_off, summary);
  GR_CHECK_LAUNCH();
  return GR_OK;
}

extern "C" int gr_info_rows_write(const double* metrics, const int8_t* cases, const int32_t* counts,
                                  const int64_t* cand_off, const int64_t* cand_total, int64_t num_data,
                                  const int64_t* cand, int64_t capacity, const int64_t* order, const uint8_t* prefix,
                                  const int64_t* prefix_off, int64_t num_q, const int32_t* name_slot,
                                  int64_t num_entity, const uint8_t* names, const int64_t* name_off,
                                  int64_t num_names, const int64_t* row_off, const int64_t* summary, uint8_t* out,
                                  int64_t out_bytes, void* stream_) {
  using namespace gr;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GR_CHECK_ARG(metrics && cases && counts && cand_off && cand_total && cand && order && prefix && prefix_off &&
               name_slot && names && name_off && row_off && summary, "null pointer");
  GR_CHECK_ARG(out, "null output");
  GR_CHECK_ARG(num_data >= 0 && capacity >= 0 && num_q >= 0 && num_entity >= 0 && num_names >= 0 && out_bytes >= 0,
               "need num_data, capacity, num_q, num_entity, num_names and out_bytes >= 0");
  if (num_data == 0) return GR_OK;
  info_rows_write_kernel<<<(unsigned)ceil_div(num_data * 32, kRowThreads), kRowThreads, 0, stream>>>(
      metrics, cases, counts, cand_off, cand_total, num_data, cand, capacity, order, prefix, prefix_off, num_q,
      name_slot, num_entity, names, name_off, num_names, row_off, summary, out, out_bytes);
  GR_CHECK_LAUNCH();
  return GR_OK;
}
