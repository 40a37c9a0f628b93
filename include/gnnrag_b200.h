/*
 * gnnrag_b200.h -- C ABI of libgnnrag_b200.so: the H100 (sm_90a) implementation of GNN-RAG's GNN
 * retrieval hot path (ReaRev / NSM multi-hop message passing + answer scoring + candidate ranking).
 *
 * The reference (cmavro/GNN-RAG) has no FFI; its boundary is the Python nn.Module contract that
 * gnn/train_model.py:49-57,222 and gnn/evaluate.py:160 call.  The Python mirror in gnn_rag_b200/ keeps
 * that contract and calls the entry points below through ctypes.  Each entry point names the
 * reference code it replaces (paths relative to the reference checkout).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - the CALLER allocates every input, output and workspace; the library never allocates, frees
 *     or retains a pointer; it is stateless and re-entrant per stream;
 *   - `stream` is a cudaStream_t passed as void* (e.g. torch.cuda.current_stream().cuda_stream);
 *   - all work is enqueued asynchronously on `stream`; nothing synchronises;
 *   - return value: 0 = GR_OK, negative = error (see gr_status); never throws;
 *     gr_last_error() returns a thread-local message for the last failing call;
 *   - node ids are GLOBAL rows b*N + local (gnn/dataset_load.py:483); index arrays produced by the
 *     library are int32; floating point is fp32 unless stated;
 *   - edge arrays (src/rel/w/fact) must be allocated with capacity gr_pad4(F) elements and row
 *     pointer arrays with capacity gr_pad4(Nt + 1) elements (the staging copies read whole 16-byte
 *     chunks).
 */
#ifndef GNNRAG_B200_H_
#define GNNRAG_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GR_ABI_VERSION 1

typedef enum gr_status {
  GR_OK = 0,
  GR_ERR_INVALID_ARG = -1,   /* null pointer, bad size, unsupported combination            */
  GR_ERR_CUDA = -2,          /* a CUDA runtime call failed (message in gr_last_error)        */
  GR_ERR_WORKSPACE = -3,     /* workspace too small                                          */
  GR_ERR_UNSUPPORTED = -4    /* shape/dtype not handled by this build                        */
} gr_status;

/* flags for gr_linear */
#define GR_LINEAR_RELU 1u        /* C = relu(A W^T + b)                                      */
#define GR_LINEAR_EXACT_FP32 2u  /* force the fp32 SIMT kernel (no split-bf16 tensor-core path) */
#define GR_LINEAR_BF16_SINGLE 8u /* gr_linear_tc_planes: bf16 activation storage -- ONE product A_hi W_hi (A_lo ignored, may
                                    be NULL); bf16-input / fp32-accumulate accuracy, a third of the tensor work   */
#define GR_LINEAR_W_PRESPLIT 4u  /* gr_linear_tc_planes: the workspace still holds the bf16 hi/lo split of the same
                                  * W (same N, K, k_seg, k_seg_pitch) from an earlier call: skip the conversion pass.
                                  * For inference with fixed weights (weight pre-formatting, done once per weight
                                  * version by the caller). */

#define GR_LINEAR_K_GROUPED 16u /* gr_linear_tc_planes: walk the T = K / k_seg_pitch segments of A column group by
                                  * column group, k-block g*T + t = columns 32g.. of segment seg(t) -- the k-block
                                  * order of gr_fused_layer, so that every output element sees the same sequence of
                                  * fp32 accumulations and the outputs equal gr_fused_layer's bit for bit.  Needs
                                  * k_seg > 0, k_seg_pitch >= k_seg and a multiple of 16, T odd (2 I + 1) and "tc_bk"
                                  * 32; not with GR_LINEAR_BF16_SINGLE.  The workspace is the one of gr_fused_layer
                                  * (gr_fused_layer_workspace_bytes(k_seg, k_seg_pitch, I, N)): same W planes, so
                                  * GR_LINEAR_W_PRESPLIT carries over between the two entry points. */
#define GR_LINEAR_K_ORDER_PLANES 32u /* with GR_LINEAR_K_GROUPED: the 2I neighbour segments of A are not at
                                  * k_seg_pitch * (1 + s) but in the K-order layout gr_aggregate_dual_abs_ex writes
                                  * (GR_AGG_K_ORDER), from column NB0 = round32(k_seg_pitch) on; the h segment stays at
                                  * column 0.  The k-blocks are aligned 64-byte boxes: per 32-column group the h box
                                  * and 2I consecutive neighbour boxes, then for a 16-column last group the h tail (one
                                  * k-step) and I boxes of two neighbour slots each.  The k16 steps, and so the output
                                  * bits, are those of GR_LINEAR_K_GROUPED.  lda16 must reach NB0 + (K - k_seg_pitch).
                                  * The W planes are packed to match: another format than gr_fused_layer's (keep a
                                  * separate workspace; gr_fused_layer_workspace_bytes is large enough). */

int gr_abi_version(void);
const char* gr_last_error(void);
/* runtime switches: "agg_tma" (0|1: stage CSR slices with bulk TMA copies), "tc_cluster" (1|2, default 1: CTAs per cluster
 * that share the W tiles of the wgmma GEMM through TMA multicast), "tc_bk" (32|64: k-block width of the wgmma GEMM),
 * "tc_tma_store" (0|1: TMA-store epilogue of the wgmma GEMM where the outputs are 16-byte aligned), "agg_abs_ws"
 * (0|1|2|3: build of the |v| aggregation kernel, see gr_aggregate_dual_abs), "fused_debug" (bits: timing decomposition
 * of gr_fused_layer, see csrc/fused_layer.cu).  Process-wide; set before launching work.  Any other name returns
 * GR_ERR_INVALID_ARG. */
int gr_set_option(const char* name, int64_t value);
static inline int64_t gr_pad4(int64_t n) { return (n + 3) & ~(int64_t)3; }

/* ------------------------------------------------------------------------------------------------
 * CSR batching.  Replaces BaseGNNLayer.build_matrix (gnn/modules/kg_reasoning/base_gnn.py:19-51: seven
 * uncoalesced COO tensors) and the index part of TypeLayer.forward (gnn/modules/layer_init.py:32-37).
 * Input: the batched fact list of SingleDataLoader._build_fact_mat (gnn/dataset_load.py:473-527),
 * copied to the device as-is (idx_bytes = 8 for the reference's int64 arrays, 4 for int32).
 * Output: in-edges grouped by TAIL (forward messages: src = head) and by HEAD (inverse messages:
 * src = tail); inside a row, edges keep the ORIGINAL FACT ORDER (stable), so per-row reductions are a
 * pure function of the row's own fact sequence (deterministic; ties stay ties).
 *   rowptr_*: int32[Nt+1]; src_*, rel_*, fact_*: int32[F] (fact_* = original fact id of each slot).
 *   status: int32[1], set non-zero on device if an id is out of range (ids are clamped).
 *   nfacts: optional device int32[1].  When given, only the first min(F, *nfacts) fact slots are read: F is then the
 *   CAPACITY of fixed-shape input buffers (CUDA-graph replay over batches of different fact counts); everything
 *   downstream sees the live facts only, through the row pointers.
 * Workspace: gr_csr_build_workspace_bytes(F, Nt).
 */
size_t gr_csr_build_workspace_bytes(int64_t F, int64_t Nt);
int gr_csr_build(const void* heads, const void* rels, const void* tails, int idx_bytes,
                 int64_t F, int64_t Nt, int64_t num_rel_rows,
                 int32_t* rowptr_t, int32_t* src_t, int32_t* rel_t, int32_t* fact_t,
                 int32_t* rowptr_h, int32_t* src_h, int32_t* rel_h, int32_t* fact_h,
                 int32_t* status, const int32_t* nfacts, void* workspace, size_t workspace_bytes, void* stream);

/* out[e] = in[fact[e]] -- permute a per-fact fp32 array (weight_list / weight_rel_list of
 * gnn/dataset_load.py:509-517) into CSR slot order. */
int gr_gather_f32(const float* in, const int32_t* fact, float* out, int64_t F, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense linear layer  C[m, n] = act( sum_k A[m,k] W[n,k] + bias[n] ) (+ addend[m, n] for m < addend_rows)
 * A: [M,K] row stride lda; W: [N,K] row stride ldw (torch nn.Linear layout); C: row stride ldc.
 * Used for the HOISTED relation projection rel_linear_k(rel_features) (reasongnn.py:79,105 apply it to
 * F gathered rows; the R1 distinct rows suffice), `addend` = pos_emb rows (reasongnn.py:75-77), and for
 * e2e_linear (reasongnn.py:163, nsm_gnn.py:63).  bias / addend may be NULL.
 */
int gr_linear(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias,
              const float* addend, int64_t ld_addend, int64_t addend_rows,
              float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, uint32_t flags, void* stream);

/* Tensor-core variant of gr_linear for the big e2e_linear GEMMs (reasongnn.py:163, nsm_gnn.py:63):
 * fp32 in / fp32 out with fp32-class accuracy through the 3-product split-bf16 scheme on wgmma
 * (x = hi + lo in bf16; A W^T ~= A_hi W_hi^T + A_hi W_lo^T + A_lo W_hi^T, fp32 accumulation in registers,
 * dropped term <= 2^-18 relative).  Persistent, TMA-fed 128 x N tiles over 32- or 64-column k-blocks ("tc_bk"),
 * W shared across a CTA pair by TMA multicast ("tc_cluster"), TMA-store epilogue ("tc_tma_store").  Requires
 * 8 <= N <= 256.  The workspace (256-byte aligned, gr_linear_tc_workspace_bytes) holds the bf16 planes.
 * flags: GR_LINEAR_RELU. */
size_t gr_linear_tc_workspace_bytes(int64_t M, int64_t N, int64_t K);
int gr_linear_tc(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias,
                 float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, uint32_t flags,
                 void* workspace, size_t workspace_bytes, void* stream);
/* Same GEMM with the A operand already in split-bf16 planes (written by gr_aggregate_dual / gr_type_layer /
 * a previous call): no conversion pass over A.  Outputs (each optional, at least one): fp32 C; bf16 planes
 * C_hi/C_lo (row stride ldc16) = the node-embedding columns of the NEXT layer's A operand; and
 * dots (float[2*M]): the score_func dot product (reasongnn.py:165) fused into the epilogue as two partial
 * sums over the lower / upper half of the output columns, dots[m] + dots[M+m] = sum_n C[m,n] * w_score[n]
 * (gr_masked_softmax adds them).  Persistent kernel, register accumulators (the producer loads the next tile during the epilogue).
 * Segmented K: when k_seg_pitch > k_seg > 0 the A planes hold K/k_seg_pitch segments of k_seg valid columns
 * at pitch k_seg_pitch (zero padding in between) while W is the dense [N, (K/k_seg_pitch)*k_seg] torch weight;
 * the W planes are built in the padded layout.  K is the padded length.
 * Workspace: gr_linear_tc_planes_workspace_bytes(N, K) (the W planes), 256-byte aligned.
 * flags: GR_LINEAR_RELU, GR_LINEAR_W_PRESPLIT (the workspace still holds this W's planes: skip the conversion). */
size_t gr_linear_tc_planes_workspace_bytes(int64_t N, int64_t K);
int gr_linear_tc_planes(const void* A_hi, const void* A_lo, int64_t lda16, const float* W, int64_t ldw,
                        const float* bias, float* C, int64_t ldc, void* C_hi, void* C_lo, int64_t ldc16,
                        const float* w_score, float* dots, int64_t M, int64_t N, int64_t K,
                        int64_t k_seg, int64_t k_seg_pitch,
                        uint32_t flags, void* workspace, size_t workspace_bytes, void* stream);
/* gr_linear_tc_planes with a row predicate on the fp32 output (its arguments, then c_rows): C receives only the rows m with c_rows[m] != 0
 * (c_rows: float[M], e.g. a question batch's seed weights query_entities [B, N] viewed as [B*N]); the other rows
 * of C keep what they held.  C_hi / C_lo and dots are written as by gr_linear_tc_planes, bit for bit.  c_rows == NULL
 * is gr_linear_tc_planes; c_rows without C is refused. */
int gr_linear_tc_planes_rows(const void* A_hi, const void* A_lo, int64_t lda16, const float* W, int64_t ldw,
                             const float* bias, float* C, int64_t ldc, void* C_hi, void* C_lo, int64_t ldc16,
                             const float* w_score, float* dots, int64_t M, int64_t N, int64_t K,
                             int64_t k_seg, int64_t k_seg_pitch,
                             uint32_t flags, void* workspace, size_t workspace_bytes, const float* c_rows,
                             void* stream);
/* fp32 [M,K] (row stride lda) -> bf16 hi/lo planes (row stride ld_out, multiple of 8). */
int gr_split_bf16(const float* A, int64_t lda, int64_t M, int64_t K, void* hi, void* lo, int64_t ld_out,
                  void* stream);

/* ------------------------------------------------------------------------------------------------
 * The aggregation kernel family (SURVEY.md 8a rows 3, 5, 6, 10).
 *
 * gr_aggregate: one direction.  For every destination row n and instruction j < I
 *     out[n, out_col0 + j*seg_stride + d] = sum_{e in row n} relu(table[rel_e, d] * ins[b(n), j, d]) * c_e
 *     c_e = w_e * (w_e * prior[src_e])        (w_e = 1 when w == NULL)
 * = ReasonGNNLayer.reason_layer (reasongnn.py:61-89) with the tail CSR, reason_layer_inv (:91-116) with
 * the head CSR, NSMLayer.reason_layer (nsm_gnn.py:87-112) with I = 1.  `table` is the hoisted
 * rel_linear(rel_features) [R1, D].  ins: [B, I, D] contiguous.  b(n) = n / N.
 * possible (optional, float[Nt]): 1.0 where sum_e c_e > 1e-10 (nsm_gnn.py:101-103).
 * Edges with c_e == 0 are skipped exactly (relu(x)*0 = 0 for finite x).
 *
 * gr_aggregate_dual: both directions of one ReaRev GNN layer in one launch; instruction j writes
 *     forward  (tail CSR, table_fwd) -> columns out_col0 + (2j  )*D
 *     inverse  (head CSR, table_inv) -> columns out_col0 + (2j+1)*D
 * which is the concat order of ReasonGNNLayer.forward (reasongnn.py:150-161).  seg_pitch (0 = D) is the
 * column distance between consecutive segments: the bf16 planes use a pitch rounded up to 16 columns so that
 * every segment starts on a 32-byte sector (a 16-byte-misaligned segment start splits the
 * achievable write bandwidth, scripts/agg_probe.py).
 *
 * Split-bf16 planes (optional, gr_aggregate_dual / gr_type_layer): when out_hi/out_lo are non-NULL the
 * result is ALSO (or, with out == NULL, only) written as two bf16 matrices with row stride ld_planes and
 * the same column indexing as `out`: hi = bf16(y), lo = bf16(y - hi), so hi + lo = y to 2^-18 relative.
 * That is the A-operand layout gr_linear_tc_planes consumes, so the fp32 concat buffer of
 * reasongnn.py:158-161 never has to exist.
 *
 * gr_type_layer: out[n,:] = relu( sum_{tail CSR} w_e table[rel_e] + sum_{head CSR} w_e table[rel_e] ),
 * TypeLayer.forward (layer_init.py:46-57) with table = kb_self_linear(rel_features).
 */
int gr_aggregate(const int32_t* rowptr, const int32_t* src, const int32_t* rel, const float* w,
                 const float* prior, const float* table, const float* ins,
                 float* out, int64_t out_row_stride, int64_t out_col0, int64_t seg_stride,
                 float* possible, int B, int N, int D, int I, int64_t F, void* stream);

/* Backward of gr_aggregate (csrc/aggregate_bwd.cu; the kernel behind model(batch, training=True), gnn/train_model.py:222):
 * given grad_out[n, grad_col0 + j*seg_stride + d] = dL/dout it ACCUMULATES (+=, caller zeroes)
 *     grad_table[r, :] += sum_{e: rel_e = r} c_e sum_j grad_out[n_e, j, :] * ins[b, j, :] * [table[r] * ins[b, j] > 0]
 *     grad_ins[b, j, :] += sum_{e in b} c_e grad_out[n_e, j, :] * table[rel_e, :] * [table[rel_e] * ins[b, j] > 0]
 *     grad_prior[s]     += sum_{e: src_e = s} w_e^2 sum_j <grad_out[n_e, j, :], relu(table[rel_e] * ins[b, j])>
 * over the same destination CSR as the forward call.  D <= 256, I <= 4.  fp32 atomics: summation order is not
 * deterministic (neither is the reference's sparse.mm backward on CUDA). */
int gr_aggregate_backward(const int32_t* rowptr, const int32_t* src, const int32_t* rel, const float* w,
                          const float* prior, const float* table, const float* ins, const float* grad_out,
                          int64_t grad_row_stride, int64_t grad_col0, int64_t seg_stride, float* grad_table,
                          float* grad_ins, float* grad_prior, int B, int N, int D, int I, int64_t F, void* stream);

int gr_aggregate_dual(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                      const float* w_t, const int32_t* rowptr_h, const int32_t* src_h,
                      const int32_t* rel_h, const float* w_h, const float* prior,
                      const float* table_fwd, const float* table_inv, const float* ins,
                      float* out, int64_t out_row_stride, int64_t out_col0, int64_t seg_pitch,
                      void* out_hi, void* out_lo, int64_t ld_planes,
                      int B, int N, int D, int I, int64_t F, void* stream);

/* Specialised variant of gr_aggregate_dual for the hot shape (csrc/aggregate_abs.cu).  The hoisted relation table is
 * copied once per layer into a zero-padded 256-column layout (gr_pad_table256: table [rows, D] fp32, row stride ldt
 * -> out [rows][256] fp32, 16-byte aligned) so every lane of the gather is in-bounds, and the edge loop accumulates
 * sum c*v and sum c*|v| (|.| is a free FFMA source modifier) instead of taking relu of every gathered
 * element: sum c*relu(+-v) = (Q +- S)/2.  Output: the split-bf16 planes only.  This build specialises D = 200,
 * seg_pitch = 208, N >= 64 (gr_aggregate_dual_abs_supported); other shapes use gr_aggregate_dual.
 * Same reference lines: reasongnn.py:61-116. */
int gr_pad_table256(const float* table, int64_t ldt, int64_t rows, int D, float* pn, void* stream);
int gr_aggregate_dual_abs_supported(int N, int D, int64_t seg_pitch, int64_t R1);
int gr_aggregate_dual_abs(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t, const float* w_t,
                         const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h, const float* w_h,
                         const float* prior, const float* pn_fwd, const float* pn_inv, int64_t table_rows,
                         const float* ins, void* out_hi, void* out_lo, int64_t ld_planes, int64_t out_col0,
                         int64_t seg_pitch, int B, int N, int D, int I, int64_t F, int32_t* tile_counter, void* stream);
/* gr_aggregate_dual_abs_ex: the same with a flags word before the stream (0 = gr_aggregate_dual_abs).
 * GR_AGG_K_ORDER writes the 2I neighbour segments in the K-order layout that gr_linear_tc_planes reads with
 * GR_LINEAR_K_ORDER_PLANES: slot u = d*I + j (direction d, instruction j; the K order of gr_fused_layer), Gf =
 * seg_pitch / 32 full column groups, and column c of slot u at
 *     out_col0 + (c >> 5) * 64 I + 32 u + (c & 31)           c < 32 Gf
 *     out_col0 + Gf * 64 I + 16 u + (c - 32 Gf)              c >= 32 Gf (the 16-column tail)
 * so the region spans 2 I seg_pitch columns, like the segment layout.  The dense layer calls it with out_col0 =
 * round32(seg_pitch); columns outside the region are not touched.  Needs both planes (out_lo != NULL) and I <= 2. */
#define GR_AGG_K_ORDER 1u
int gr_aggregate_dual_abs_ex(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t, const float* w_t,
                             const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h, const float* w_h,
                             const float* prior, const float* pn_fwd, const float* pn_inv, int64_t table_rows,
                             const float* ins, void* out_hi, void* out_lo, int64_t ld_planes, int64_t out_col0,
                             int64_t seg_pitch, int B, int N, int D, int I, int64_t F, int32_t* tile_counter,
                             uint32_t flags, void* stream);
/* table_rows: rows (R1) of each padded table.
 * tile_counter: 4 bytes of device scratch (zeroed by the call) -> the persistent, warp-specialised kernel (a staging
 * warp prepares the next tile of rows while the consumer warps aggregate the current one; dynamic tile scheduler);
 * NULL -> one CTA per 64-row tile.  gr_set_option("agg_abs_ws", v) picks the persistent variant: 1 = 8 consumer warps /
 * 64-row tiles, 2 (default) = 9 consumer warps / 72-row tiles, 3 = gather through TMA tile::gather4 copies into
 * shared-memory rings (bit-identical results; slower at cfg2, kept as the measured alternative, DESIGN.md 4.1);
 * 0 = one CTA per 64-row tile even when a tile counter is given.
 * out_lo NULL (bf16 activation storage: the hi plane only) is accepted only by the persistent kernels 1 and 2, so it
 * needs a tile counter and agg_abs_ws != 0 (GR_ERR_INVALID_ARG otherwise); with agg_abs_ws 3 it runs variant 2. */

/* One dense-prior ReaRev layer as ONE kernel (csrc/fused_layer.cu): the aggregation of both directions and all
 * instructions (reason_layer / reason_layer_inv, reasongnn.py:61-116) is produced straight into the shared-memory
 * operand slots of the wgmma e2e GEMM (torch.cat + e2e_linear + relu, reasongnn.py:158-163; score_func dot :165), so
 * the 2*I neighbour segments never reach HBM.  Replaces the pair gr_aggregate_dual_abs -> gr_linear_tc_planes.
 *   h_hi / h_lo    bf16 planes of the layer input h: [B*N, >= seg_pitch] with row stride ldh16 (only the first
 *                  seg_pitch columns are read; columns D .. seg_pitch-1 must be zero)
 *   pn_fwd/pn_inv  zero-padded 256-column relation tables of this layer (gr_pad_table256)
 *   W              e2e_linear weight [N_out, (2I+1)*D] fp32 (row stride ldw); it is re-ordered and split into bf16 hi/lo
 *                  planes inside `workspace` (gr_fused_layer_workspace_bytes, 256-byte aligned) unless flags carries
 *                  GR_LINEAR_W_PRESPLIT (workspace kept from an earlier call with the same W)
 *   outputs        any of C (fp32 [B*N, N_out]), C_hi / C_lo (bf16 planes, row stride ldc16), dots [2*B*N]
 *                  (dots[m] = <out[m], w_score>, dots[B*N + m] = 0: the layout gr_masked_softmax takes)
 * Supported (gr_fused_layer_supported): I <= 2, N >= 128, seg_pitch % 16 == 0, seg_pitch <= 224, N_out <= 256 and the
 * operand stages must fit shared memory (D = N_out = 200 does).  The A operand is bit-identical to the unfused pair;
 * the tensor core accumulates the k-blocks in another order than the pair's default (fp32 rounding), and in the same
 * order as the pair with GR_LINEAR_K_GROUPED, whose outputs equal this kernel's bit for bit. */
/* Diagnostic: per-CTA wait-cycle counters of the last gr_fused_layer launch made with gr_set_option("fused_debug", 32)
 * (16 uint64 per CTA, slot meaning in csrc/fused_layer.cu). */
int gr_fused_profile_read(unsigned long long* out, int n);
int gr_fused_layer_supported(int64_t N_nodes, int64_t D, int64_t seg_pitch, int I, int64_t N_out);
size_t gr_fused_layer_workspace_bytes(int64_t D, int64_t seg_pitch, int I, int64_t N_out);
/* Once per batch: both CSRs of gr_csr_build re-laid out slot-major per quad of 4 rows ("quad ELL", csrc/fused_layer.cu)
 * into `ell` (gr_fused_ell_bytes, 256-byte aligned); gr_fused_layer reads it and keeps its per-layer {table offset,
 * coefficient} scratch inside the same buffer. */
size_t gr_fused_ell_bytes(int B, int N_nodes, int64_t F);
int gr_fused_ell_build(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t, const float* w_t,
                       const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h, const float* w_h,
                       int B, int N_nodes, int64_t F, void* ell, size_t ell_bytes, void* stream);
int gr_fused_layer(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t, const float* w_t,
                   const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h, const float* w_h,
                   const float* prior, const float* pn_fwd, const float* pn_inv, const float* ins,
                   const void* h_hi, const void* h_lo, int64_t ldh16, int64_t seg_pitch, const float* W,
                   int64_t ldw, const float* bias, float* C, int64_t ldc, void* C_hi, void* C_lo,
                   int64_t ldc16, const float* w_score, float* dots, int B, int N_nodes, int D, int I,
                   int64_t N_out, int64_t F, uint32_t flags, void* workspace, size_t workspace_bytes,
                   void* ell, size_t ell_bytes, void* stream);

/* Diagnostic only (scripts/agg_probe.py): replays the aggregation kernel's store pattern without any edge work. */
int gr_debug_store_probe(void* hi, void* lo, int64_t Nt, int64_t ld, int col_start, int ncols, int mode,
                         void* stream);

int gr_type_layer(const int32_t* rowptr_t, const int32_t* rel_t, const float* w_t,
                  const int32_t* rowptr_h, const int32_t* rel_h, const float* w_h,
                  const float* table, float* out, int64_t out_row_stride,
                  void* out_hi, void* out_lo, int64_t ld_planes,
                  int B, int N, int D, int64_t F, void* stream);

/* ------------------------------------------------------------------------------------------------
 * GraftNet (csrc/graft.cu): GraftLayer, gnn/modules/kg_reasoning/graft_gnn.py, on the batch of
 * GraftSingleDataLoader.get_batch (gnn/dataset_load_graft.py:113-149).
 *
 * gr_graft_stage: BaseGNNLayer.build_adj_facts (gnn/modules/kg_reasoning/base_gnn.py:56-75).  Input: the two lists
 * of kb_adj_mat_graft as int64 device arrays -- head list (e2f_b, e2f_f, e2f_e) = (b, fact slot f, local head) and
 * tail list (f2e_b, f2e_e, f2e_f) = (b, local tail, fact slot f) (dataset_load_graft.py:70-102) -- and kb_fact_rel
 * int64 [B, max_fact].  Pairs head and tail by slot and writes the facts ordered by (b, f): heads / tails (global rows
 * b*N + local), rels = kb_fact_rel[b, f], slot_of = b*max_fact + f, each int32 with capacity gr_pad4(F_e2f), and the
 * count to nfacts (device int32[1]).  Feed them to gr_csr_build(F = F_e2f, nfacts): its stable CSRs then list every
 * row in slot order, the order torch's sparse bmm sums a row in.  status (int32[1], OR-ed): 1 = batch / slot / node
 * id out of range, 2 = relation id outside [0, R1), 4 = a slot listed twice, 8 = a slot with a head but no tail or the
 * reverse.  Offending entries are dropped or clamped, never read out of bounds.
 * live (optional device int32[2], NULL = the whole lists): the live entries of the head list and of the tail list.
 * F_e2f / F_f2e are then capacities of fixed-shape buffers and only the first min(F, live[k]) entries are read, so a
 * stale capacity tail is never staged; the launch shape depends on the capacities only (CUDA-graph capture).
 * Workspace: gr_graft_stage_workspace_bytes(B, max_fact) (depends on B * max_fact only).
 *
 * gr_graft_attention: GraftLayer.compute_attention (graft_gnn.py:64-87).  For EVERY slot (pads and dropped facts
 * included) with r = kb_fact_rel[b, f]:
 *     a_q = softmax_q(<qh[b,q], rel[r]>/sqrt(D) + (1 - qmask[b,q]) * -1e11),  W[b,f] = <sum_q a_q qh[b,q], rel[r]>/sqrt(D)
 *     Wt[b,f] = exp(W[b,f] - max_f W[b,f]);   E[n] = max(sum_{graft f: head_f = n} Wt[f], 1e-10)  (head CSR, slot order)
 * qh [B,Q,D], qmask float [B,Q], rel [R1, D] row stride ldr; W / Wt float [B*max_fact]; E float [B*N].
 * rowptr_h / fact_h: the head CSR of gr_csr_build on the staged facts; slot_of from gr_graft_stage.  D <= 512.
 *
 * gr_graft_aggregate: the fact side of GraftLayer.reason_layer (graft_gnn.py:89-107) for one layer.  One destination
 * row per tail-CSR row; its facts in slot order:
 *     s_f = Wt[slot_f] * (prior[head_f] / E[head_f]),   v_f = relu(self_tab[r_f] + head_tab[head_f]) * s_f
 *     sum[n] = sum_f v_f,   indeg[n] = number of facts,   prior_next[n] = lambda * sum_f s_f + (1 - lambda) * prior[n]
 * self_tab = kb_self_linear_i(rel) [R1, D], head_tab = kb_head_linear_i(h) [B*N, D].  Outputs: prior_next (required);
 * sum_out fp32 (optional); split-bf16 planes (optional, row stride ld_planes) with sum at columns col_sum.., indeg at
 * column col_indeg and, when q2e [B, D] is given, the row's question vector q2e[b] at col_q2e.. -- the A operands of
 * the f2e and e2e GEMMs; indeg_out fp32 [B*N] (optional).  No atomics: bit-reproducible.  D <= 512.
 */
size_t gr_graft_stage_workspace_bytes(int64_t B, int64_t max_fact);
int gr_graft_stage(const int64_t* e2f_b, const int64_t* e2f_f, const int64_t* e2f_e, int64_t F_e2f,
                   const int64_t* f2e_b, const int64_t* f2e_e, const int64_t* f2e_f, int64_t F_f2e,
                   const int64_t* kb_fact_rel, int B, int N, int64_t max_fact, int64_t R1, int32_t* heads,
                   int32_t* rels, int32_t* tails, int32_t* slot_of, int32_t* nfacts, int32_t* status,
                   const int32_t* live, void* workspace, size_t workspace_bytes, void* stream);
int gr_graft_attention(const float* qh, const float* qmask, int Q, const float* rel, int64_t ldr, int64_t R1,
                       const int64_t* kb_fact_rel, int B, int64_t max_fact, int D, const int32_t* rowptr_h,
                       const int32_t* fact_h, const int32_t* slot_of, int N, float* W, float* Wt, float* E,
                       int32_t* status, void* stream);
int gr_graft_aggregate(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t, const int32_t* fact_t,
                       const int32_t* slot_of, const float* Wt, const float* E, const float* prior,
                       const float* self_tab, int64_t ld_self, const float* head_tab, int64_t ld_head,
                       const float* q2e, double lambda, float* sum_out, int64_t ld_sum, void* out_hi, void* out_lo,
                       int64_t ld_planes, int64_t col_sum, int64_t col_indeg, int64_t col_q2e, float* indeg_out,
                       float* prior_next, int B, int N, int D, void* stream);

/* ------------------------------------------------------------------------------------------------
 * GraftNet training (csrc/graft.cu; model(batch, training=True), gnn/train_model.py:222).  The per-fact scalars
 * (W~, E, s_f, d') stay in torch autograd on [F] vectors; these kernels do the per-fact work of width D, so no [F, D]
 * tensor exists.  Every gradient output is ACCUMULATED (+=, caller zeroes).  D <= 512.
 *
 * Dropout (linear_dropout on the fact messages, graft_gnn.py:105): element (slot, column) is kept iff
 * u = (Philox4x32-10(key = *seed, counter = (slot lo, slot hi, column, 0))[0] >> 8) * 2^-24 >= p, and kept elements
 * are scaled by 1/(1-p).  slot = b*max_fact + f (slot_of), so the mask does not depend on the loader's permutation of
 * the graft lists.  seed: device int64[1]; p in [0, 1); p == 0 ignores the seed and computes without dropout.
 *
 * gr_graft_dropout_mask: mask[slot*D + c] = 1 if (slot, c) is kept, for slot < S (the same device function).
 *
 * gr_graft_aggregate_train: graft_gnn.py:89-107 (the fact messages, kb_tail_linear moved after the sum by
 * linearity).  One warp per tail-CSR row n, facts in slot order:
 *     sum_out[n] = sum_{f -> n} drop_f(relu(self_tab[r_f] + head_tab[head_f])) * s_f
 * s: fp32 per staged fact (gr_graft_stage order); facts with s_f == 0 are skipped.  No atomics.
 *
 * gr_graft_aggregate_backward: given G = dL/dsum_out, g_f = G[tail_f] * mask_f/(1-p), a_f = self_tab[r_f] +
 * head_tab[head_f]:
 *     grad_s[f] += <g_f, relu(a_f)>  (every fact, s_f = 0 included)
 *     grad_self[r] += sum_{f: r_f = r} g_f s_f [a_f > 0]      (fp32 atomics into the R1 rows)
 *     grad_head[n] += sum_{f: head_f = n} g_f s_f [a_f > 0]   (one warp per head-CSR row, no atomics)
 * Takes the HEAD CSR of the staged facts (rowptr_h, src_h = tails, rel_h, fact_h).
 *
 * gr_graft_attention_backward: graft_gnn.py:64-87.  Given grad_W [B*max_fact] (dL/dW of gr_graft_attention's W),
 *     grad_qh[b, q] += sum_f c_{f,q} rel[r_f],   grad_rel[r] += sum_{f: r_f = r} sum_q c_{f,q} qh[b, q],
 *     c_{f,q} = grad_W[f] a_{f,q} (1 + z_{f,q} - W_f) / sqrt(D),   z_{f,q} = <qh[b,q], rel[r_f]> / sqrt(D)
 * with the softmax a recomputed per slot.  Slots with grad_W == 0 are skipped.  fp32 atomics.
 *
 * gr_type_layer_backward: TypeLayer.forward (layer_init.py:46-57) given G = dL/dout and gr_type_layer's fp32 output:
 *     grad_table[r] += sum_{tail CSR} w_e (G * [out > 0])[n] + sum_{head CSR} w_e (G * [out > 0])[n]
 * One warp per row, fp32 atomics into the R1 table rows.  Same CSRs and weights as the forward call.
 */
int gr_graft_dropout_mask(const int64_t* seed, double p, int64_t S, int D, uint8_t* mask, void* stream);
int gr_graft_aggregate_train(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                             const int32_t* fact_t, const int32_t* slot_of, const float* s, const float* self_tab,
                             int64_t ld_self, const float* head_tab, int64_t ld_head, const int64_t* seed, double p,
                             float* sum_out, int64_t ld_sum, int B, int N, int D, void* stream);
int gr_graft_aggregate_backward(const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h,
                                const int32_t* fact_h, const int32_t* slot_of, const float* s,
                                const float* self_tab, int64_t ld_self, const float* head_tab, int64_t ld_head,
                                const int64_t* seed, double p, const float* grad_sum, int64_t ld_grad, float* grad_s,
                                float* grad_self, int64_t ld_gself, float* grad_head, int64_t ld_ghead, int B, int N,
                                int D, void* stream);
int gr_graft_attention_backward(const float* qh, const float* qmask, int Q, const float* rel, int64_t ldr,
                                int64_t R1, const int64_t* kb_fact_rel, int B, int64_t max_fact, int D,
                                const float* grad_W, float* grad_qh, float* grad_rel, int64_t ld_grel, void* stream);
int gr_type_layer_backward(const int32_t* rowptr_t, const int32_t* rel_t, const float* w_t,
                           const int32_t* rowptr_h, const int32_t* rel_h, const float* w_h,
                           const float* grad_out, int64_t ld_grad, const float* out, int64_t ld_out,
                           float* grad_table, int64_t ld_gtable, int B, int N, int D, int64_t F, void* stream);

/* Deterministic backward (torch.use_deterministic_algorithms): the gradients of the four entry points above, each
 * output element a sum whose order is fixed by the data alone -- fact, slot and row ids and compile-time window sizes,
 * never the grid, the SM count or block arrival.  No floating-point atomics; every term and sum is rounded with
 * __fmul_rn / __fadd_rn.  Same accumulate-into-the-caller's-buffers convention as the atomic versions.
 *
 * The relation-keyed sums walk a relation index: gr_csr_build called with heads = rels = tails = the relation id of
 * each list entry and Nt = num_rel_rows = R1, whose tail CSR (rix_ptr [R1+1], rix_slot) lists each relation's entries
 * in increasing entry order.  row_of (gr_csr_row_of) maps a CSR slot to its row.  Partial sums go to `workspace`
 * (size from the *_workspace_bytes helper, allocated by the caller): windows of 32 rows / 64 entries each add their
 * entries in list order; sums that cross a window edge are then added in window order (csrc/common.cuh).
 *
 * gr_aggregate_backward_det: gr_aggregate_backward's arguments, plus fact (this CSR's slot -> fact id), the OTHER
 *   destination CSR (rowptr_o, fact_o: it lists every source's out-edges in slot order) and this CSR's relation index
 *   (rix_ptr, rix_slot over this CSR's slots, row_of).  dx per question over windows of 32 destination rows; dp[s] adds
 *   q_e = w_e^2 <G[n_e], relu(P[r_e] x_j[b])> over the other CSR's row s; dP per relation over windows of 64 entries.
 * gr_type_layer_backward_det: the relation indexes of both CSRs; grad_table[r] = (grad_table[r] + tail-CSR sum) +
 *   head-CSR sum, each over the relation's slots in slot order.  No rowptr / B / N: the row comes from row_of.
 * gr_graft_aggregate_backward_det: gr_graft_aggregate_backward's arguments, plus the staged facts (heads, rels, tails
 *   of gr_graft_stage) and their relation index (rix_ptr, rix_fact over staged fact ids; F = the fact capacity).
 *   grad_s and grad_head are the owned sums of the atomic version; grad_self per relation in slot order.
 * gr_graft_attention_backward_det: a slot-level relation index over all B*max_fact slots (relation ids out of range
 *   read as 0, as the forward does).  The coefficients c_{s,q} go to the workspace; grad_qh[b, q] sums the question's
 *   slots in slot order, grad_rel[r] the relation's slots in slot order (each term summed over q in order).
 */
int gr_csr_row_of(const int32_t* rowptr, int64_t Nt, int32_t* row_of, void* stream);
size_t gr_aggregate_backward_det_workspace_bytes(int B, int N, int D, int I, int64_t F);
int gr_aggregate_backward_det(const int32_t* rowptr, const int32_t* src, const int32_t* rel, const int32_t* fact,
                              const float* w, const float* prior, const float* table, const float* ins,
                              const float* grad_out, int64_t grad_row_stride, int64_t grad_col0, int64_t seg_stride,
                              float* grad_table, float* grad_ins, float* grad_prior, int B, int N, int D, int I,
                              int64_t F, const int32_t* rowptr_o, const int32_t* fact_o, const int32_t* rix_ptr,
                              const int32_t* rix_slot, const int32_t* row_of, int64_t R1, void* workspace,
                              size_t workspace_bytes, void* stream);
size_t gr_type_layer_backward_det_workspace_bytes(int64_t F, int D);
int gr_type_layer_backward_det(const int32_t* rel_t, const float* w_t, const int32_t* rix_ptr_t,
                               const int32_t* rix_slot_t, const int32_t* row_of_t, const int32_t* rel_h,
                               const float* w_h, const int32_t* rix_ptr_h, const int32_t* rix_slot_h,
                               const int32_t* row_of_h, const float* grad_out, int64_t ld_grad, const float* out,
                               int64_t ld_out, float* grad_table, int64_t ld_gtable, int64_t R1, int D, int64_t F,
                               void* workspace, size_t workspace_bytes, void* stream);
size_t gr_graft_aggregate_backward_det_workspace_bytes(int64_t F, int D);
int gr_graft_aggregate_backward_det(const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h,
                                    const int32_t* fact_h, const int32_t* slot_of, const float* s,
                                    const float* self_tab, int64_t ld_self, const float* head_tab, int64_t ld_head,
                                    const int64_t* seed, double p, const float* grad_sum, int64_t ld_grad,
                                    float* grad_s, float* grad_self, int64_t ld_gself, float* grad_head,
                                    int64_t ld_ghead, int B, int N, int D, const int32_t* heads, const int32_t* rels,
                                    const int32_t* tails, const int32_t* rix_ptr, const int32_t* rix_fact, int64_t R1,
                                    int64_t F, void* workspace, size_t workspace_bytes, void* stream);
size_t gr_graft_attention_backward_det_workspace_bytes(int B, int64_t max_fact, int Q, int D);
int gr_graft_attention_backward_det(const float* qh, const float* qmask, int Q, const float* rel, int64_t ldr,
                                    int64_t R1, const int64_t* kb_fact_rel, int B, int64_t max_fact, int D,
                                    const float* grad_W, float* grad_qh, float* grad_rel, int64_t ld_grel,
                                    const int32_t* rix_ptr, const int32_t* rix_slot, void* workspace,
                                    size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Mixed-precision training (torch.autocast(bfloat16)): *_ex variants of the training entry points with an io flags
 * word before the stream.  io = 0 is the entry point without the suffix.  io = GR_IO_BF16 makes the node-sized
 * tensors ([B*N, D] rows) bf16; their pointers are then __nv_bfloat16 data with strides still counted in elements:
 *   gr_aggregate_ex                  out
 *   gr_aggregate_backward(_det)_ex   grad_out
 *   gr_type_layer_ex                 out (the split-bf16 planes are unchanged)
 *   gr_type_layer_backward(_det)_ex  grad_out and out (the forward's output, read for the relu mask)
 *   gr_graft_aggregate_train_ex      head_tab, sum_out
 *   gr_graft_aggregate_backward(_det)_ex  head_tab, grad_sum, grad_head (read, added to, stored: owned rows)
 * Everything else keeps its fp32 type: relation tables, ins, priors, s, weights, every gradient accumulator and the
 * workspaces, whose sizes (*_workspace_bytes) do not depend on io.
 * Rounding contract: a bf16 load is widened to fp32 (exact), the kernel then does the fp32 kernel's operations in the
 * same order, and a bf16 store is the round-to-nearest-even of the value the fp32 kernel would store.  So the forward
 * and the deterministic backward in bf16 mode equal the fp32 call on the upcast inputs followed by a conversion to
 * bf16, bit for bit; the atomic backward differs from it only by its summation order.  Shape limits are those of the
 * fp32 entry points.  Other io bits are refused. */
#define GR_IO_BF16 1u
int gr_aggregate_ex(const int32_t* rowptr, const int32_t* src, const int32_t* rel, const float* w, const float* prior,
                    const float* table, const float* ins, void* out, int64_t out_row_stride, int64_t out_col0,
                    int64_t seg_stride, float* possible, int B, int N, int D, int I, int64_t F, uint32_t io,
                    void* stream);
int gr_aggregate_backward_ex(const int32_t* rowptr, const int32_t* src, const int32_t* rel, const float* w,
                             const float* prior, const float* table, const float* ins, const void* grad_out,
                             int64_t grad_row_stride, int64_t grad_col0, int64_t seg_stride, float* grad_table,
                             float* grad_ins, float* grad_prior, int B, int N, int D, int I, int64_t F, uint32_t io,
                             void* stream);
int gr_aggregate_backward_det_ex(const int32_t* rowptr, const int32_t* src, const int32_t* rel, const int32_t* fact,
                                 const float* w, const float* prior, const float* table, const float* ins,
                                 const void* grad_out, int64_t grad_row_stride, int64_t grad_col0, int64_t seg_stride,
                                 float* grad_table, float* grad_ins, float* grad_prior, int B, int N, int D, int I,
                                 int64_t F, const int32_t* rowptr_o, const int32_t* fact_o, const int32_t* rix_ptr,
                                 const int32_t* rix_slot, const int32_t* row_of, int64_t R1, void* workspace,
                                 size_t workspace_bytes, uint32_t io, void* stream);
int gr_type_layer_ex(const int32_t* rowptr_t, const int32_t* rel_t, const float* w_t, const int32_t* rowptr_h,
                     const int32_t* rel_h, const float* w_h, const float* table, void* out, int64_t out_row_stride,
                     void* out_hi, void* out_lo, int64_t ld_planes, int B, int N, int D, int64_t F, uint32_t io,
                     void* stream);
int gr_type_layer_backward_ex(const int32_t* rowptr_t, const int32_t* rel_t, const float* w_t,
                              const int32_t* rowptr_h, const int32_t* rel_h, const float* w_h, const void* grad_out,
                              int64_t ld_grad, const void* out, int64_t ld_out, float* grad_table, int64_t ld_gtable,
                              int B, int N, int D, int64_t F, uint32_t io, void* stream);
int gr_type_layer_backward_det_ex(const int32_t* rel_t, const float* w_t, const int32_t* rix_ptr_t,
                                  const int32_t* rix_slot_t, const int32_t* row_of_t, const int32_t* rel_h,
                                  const float* w_h, const int32_t* rix_ptr_h, const int32_t* rix_slot_h,
                                  const int32_t* row_of_h, const void* grad_out, int64_t ld_grad, const void* out,
                                  int64_t ld_out, float* grad_table, int64_t ld_gtable, int64_t R1, int D, int64_t F,
                                  void* workspace, size_t workspace_bytes, uint32_t io, void* stream);
int gr_graft_aggregate_train_ex(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t,
                                const int32_t* fact_t, const int32_t* slot_of, const float* s, const float* self_tab,
                                int64_t ld_self, const void* head_tab, int64_t ld_head, const int64_t* seed, double p,
                                void* sum_out, int64_t ld_sum, int B, int N, int D, uint32_t io, void* stream);
int gr_graft_aggregate_backward_ex(const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h,
                                   const int32_t* fact_h, const int32_t* slot_of, const float* s,
                                   const float* self_tab, int64_t ld_self, const void* head_tab, int64_t ld_head,
                                   const int64_t* seed, double p, const void* grad_sum, int64_t ld_grad,
                                   float* grad_s, float* grad_self, int64_t ld_gself, void* grad_head,
                                   int64_t ld_ghead, int B, int N, int D, uint32_t io, void* stream);
int gr_graft_aggregate_backward_det_ex(const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h,
                                       const int32_t* fact_h, const int32_t* slot_of, const float* s,
                                       const float* self_tab, int64_t ld_self, const void* head_tab, int64_t ld_head,
                                       const int64_t* seed, double p, const void* grad_sum, int64_t ld_grad,
                                       float* grad_s, float* grad_self, int64_t ld_gself, void* grad_head,
                                       int64_t ld_ghead, int B, int N, int D, const int32_t* heads,
                                       const int32_t* rels, const int32_t* tails, const int32_t* rix_ptr,
                                       const int32_t* rix_fact, int64_t R1, int64_t F, void* workspace,
                                       size_t workspace_bytes, uint32_t io, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Sparse-prior fast path for one ReaRev layer (the first layer of every iteration sees the seed distribution,
 * rearev.py:208).  Rows none of whose in-edges carries prior mass get exactly zero neighbour messages, so
 * h_new = relu(W[:, :D] h + b) there (gr_linear_tc_planes with K = one segment).  gr_frontier_rows lists the
 * other rows (exact for any prior); gr_frontier_fixup recomputes those rows in full -- aggregation of both
 * directions for every instruction (same edge order/arithmetic as gr_aggregate_dual), e2e linear, relu, score
 * dot -- and overwrites h_new in the next planes / fp32 h / dots.  list: int32[Nt], count: int32[1] (device).
 */
int gr_frontier_rows(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rowptr_h,
                     const int32_t* src_h, const float* prior, int64_t Nt, int32_t* list, int32_t* count,
                     void* stream);
int gr_frontier_fixup(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t, const float* w_t,
                      const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h, const float* w_h,
                      const float* prior, const float* table_fwd, const float* table_inv, const float* ins,
                      const void* cur_hi, const void* cur_lo, int64_t ld_cur, const float* W, int64_t ldw,
                      const float* bias, const float* w_score, void* nxt_hi, void* nxt_lo, int64_t ld_nxt,
                      float* h32, float* dots, const int32_t* list, const int32_t* count,
                      int B, int N, int D, int I, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Scoring: logits[b,n] = dot(h[b,n,:], w_score) + b_score + (1 - mask[b,n]) * (-1e11);
 * dist = softmax_n(logits).  reasongnn.py:165-169 / nsm_gnn.py:67-74.  One CTA per question.
 * h row stride ldh.  mask: float[B*N] (local_entity != num_entity, times possible_tail for NSM
 * reason_kb).  logits_out optional.
 */
int gr_score_softmax(const float* h, int64_t ldh, const float* w_score, const float* b_score,
                     const float* mask, float* dist, float* logits_out, int B, int N, int D,
                     void* stream);
/* Same, starting from precomputed score dots (gr_linear_tc_planes epilogue): logit = dots[n] (+ dots2[n] if
 * dots2 != NULL) + b_score + (1-mask)*VERY_NEG. */
int gr_masked_softmax(const float* dots, const float* dots2, const float* b_score, const float* mask,
                      float* dist, int B, int N, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Question-side updates, one CTA per question (csrc/question.cu).  In the reference each is a chain of 10-20
 * tiny torch ops on [B, D] tensors; fused here because on a GPU they are pure launch latency.
 * Pointer arrays named *_host are HOST arrays of device pointers (one per instruction, <= 8).
 *
 * gr_instructions: LSTMInstruction.forward after the encoder (gnn/modules/question_encoding/
 * base_encoder.py:73-114): for i < I:  q_i = question_linear_i(qnode);  cq = cq_linear([ri, q_i, q_i-ri, q_i*ri]);
 * attn = softmax_q(ca_linear(cq * hidden[q]) + (1-mask[q])*VERY_NEG);  ri = sum_q attn[q]*hidden[q];
 * out[b,i,:] = ri (ri starts at 0).  hidden [B,Q,D], qnode [B,D], qtext int64 [B,Q] (mask = qtext != pad_id).
 * attn_out optional [B,I,Q]. */
int gr_instructions(const float* hidden, const float* qnode, const int64_t* qtext, int64_t pad_id,
                    const float* const* Wq_host, const float* const* bq_host, const float* Wcq,
                    const float* bcq, const float* wca, const float* bca, float* out, float* attn_out,
                    int B, int Q, int D, int I, void* stream);
/* gr_query_reform: the instruction update after every iteration (gnn/models/ReaRev/rearev.py:214-221 ->
 * QueryReform.forward, gnn/modules/query_update.py:18-44, Fusion :6-16): y = seed_info[b] @ h[b] (seed rows
 * only, index order); for j < I: z = [x_j, y, x_j - y]; g = sigmoid(G_j z); out_j = g * (R_j z) + (1-g) * x_j.
 * ins_in/ins_out [B,I,D] (may not alias); Wr/Wg: fusion.r / fusion.g weights [D,3D]; seed_out optional [B,D]. */
int gr_query_reform(const float* seed_info, const float* h, int64_t ldh, const float* ins_in,
                    const float* const* Wr_host, const float* const* Wg_host, float* ins_out,
                    float* seed_out, int B, int N, int D, int I, void* stream);
/* gr_query_reform_ex: gr_query_reform with an io flags word (see the *_ex entry points): GR_IO_BF16 makes h bf16
 * (widened on load; everything else fp32).  io = 0 is gr_query_reform. */
int gr_query_reform_ex(const float* seed_info, const void* h, int64_t ldh, const float* ins_in,
                       const float* const* Wr_host, const float* const* Wg_host, float* ins_out, float* seed_out,
                       int B, int N, int D, int I, uint32_t io, void* stream);

/* Question-side training (model(batch, training=True), gnn/train_model.py:222).  Same shapes as the forward entry
 * points above (gr_instructions: I <= 8 and (Q D + (I+7) D + 2 Q) * 4 bytes <= 200 KB; gr_query_reform: D <= 1024,
 * I <= 8 and (5I+1) D * 4 bytes <= 48 KB).  One CTA per question in every backward; each output element is owned by
 * one question and written in a fixed order: no atomics, bit-reproducible.  The weight gradients are left to the
 * caller as one GEMM per weight over the per-question operands written here (G = the pre-activation gradient, X =
 * the layer's dropped input): grad_W = G^T X over the rows (b, i) (ca_linear: rows (b, i, q)), grad_b = column sums.
 *
 * gr_instructions_train: gr_instructions with the three linear_drop sites of get_instruction (base_encoder.py:85-98)
 * drawn in the kernel.  Element (question b, step i, site s, token q, column c) is kept iff
 * u = (Philox4x32-10(key = *seed, counter = (b, 4 i + s, q, c))[0] >> 8) * 2^-24 >= p, and kept elements are scaled
 * by 1/(1-p).  Sites: s = 0 qnode before question_linear_i (q = 0, c < D); s = 1 [ri, q_i, q_i - ri, q_i * ri]
 * before cq_linear (q = 0, c < 4D); s = 2 cq * hidden[q] before ca_linear (c < D).  seed: device int64[1]; p in
 * [0, 1); p == 0 ignores the seed and runs gr_instructions' kernel (the same bits).  attn_out [B,I,Q] is required:
 * the backward reads it.
 * gr_instructions_dropout_mask: the masks of the three sites (1 = kept) for 0 < p < 1: mask_q [B,I,D],
 * mask_cq [B,I,4D], mask_ca [B,I,Q,D] (the same device function).
 * gr_instructions_backward: the forward's inputs, seed and p, its outputs ri [B,I,D] and attn [B,I,Q], and
 * grad_out = dL/dri [B,I,D].  Writes (overwrites) grad_hidden [B,Q,D], grad_qnode [B,D] and the operands g_q, x_q
 * [B,I,D] (question_linear_i), g_cq [B,I,D], x_cq [B,I,4D] (cq_linear), g_ca [B,I,Q], x_ca [B,I,Q,D] (ca_linear).
 * The mask is redrawn from the seed, never stored.
 * gr_query_reform_backward: the forward's inputs (h fp32, or bf16 with GR_IO_BF16) and grad_out = dL/dins_out
 * [B,I,D].  Writes grad_ins [B,I,D] and the operands g_r, g_g [B,I,D] (fusion.r / fusion.g) and x_z [B,I,3D]
 * (their input z = [x, y, x - y]); adds s_n * dL/dy to each seed row n of grad_h (row stride ldg, h's type), seeds
 * in index order as in the forward.  No other row of grad_h is read or written. */
int gr_instructions_train(const float* hidden, const float* qnode, const int64_t* qtext, int64_t pad_id,
                          const float* const* Wq_host, const float* const* bq_host, const float* Wcq,
                          const float* bcq, const float* wca, const float* bca, const int64_t* seed, double p,
                          float* out, float* attn_out, int B, int Q, int D, int I, void* stream);
int gr_instructions_dropout_mask(const int64_t* seed, double p, int B, int Q, int D, int I, uint8_t* mask_q,
                                 uint8_t* mask_cq, uint8_t* mask_ca, void* stream);
int gr_instructions_backward(const float* hidden, const float* qnode, const int64_t* qtext, int64_t pad_id,
                             const float* const* Wq_host, const float* const* bq_host, const float* Wcq,
                             const float* bcq, const float* wca, const float* bca, const int64_t* seed, double p,
                             const float* ri, const float* attn, const float* grad_out, float* grad_hidden,
                             float* grad_qnode, float* g_q, float* x_q, float* g_cq, float* x_cq, float* g_ca,
                             float* x_ca, int B, int Q, int D, int I, void* stream);
int gr_query_reform_backward(const float* seed_info, const void* h, int64_t ldh, const float* ins_in,
                             const float* const* Wr_host, const float* const* Wg_host, const float* grad_out,
                             float* grad_ins, void* grad_h, int64_t ldg, float* g_r, float* g_g, float* x_z, int B,
                             int N, int D, int I, uint32_t io, void* stream);
/* gr_kl_loss_pred: BaseModel.calc_loss_label with loss_type "kl" (gnn/models/base_model.py:186-215,
 * rearev.py:156-160,228-232) and pred = argmax_n dist[b,n] (lowest index on ties):
 * loss = sum_b valid_b * sum_n kl_div(log(dist+1e-8), teacher/len_b) / B.  loss_q: float[B] scratch/output. */
int gr_kl_loss_pred(const float* dist, const float* teacher, float* loss_q, float* loss, int64_t* pred,
                    int B, int N, void* stream);

/* gr_lstm_forward: recurrence of the one-layer LSTM question encoder (gnn/modules/question_encoding/
 * lstm_encoder.py:27-36: nn.LSTM(batch_first=True), h0 = c0 = 0, gate order i,f,g,o) for all Q tokens in ONE
 * launch (8-CTA clusters, W_hh slices resident in shared memory, h exchanged through distributed shared memory).
 * gates_x [B,Q,4D] = x_t W_ih^T + b_ih (computed by the caller); W_hh [4D,D]; b_hh [4D] or NULL;
 * hidden [B,Q,D] out (h_n = hidden[:, Q-1]).  D <= gr_lstm_max_hidden() (256). */
size_t gr_lstm_max_hidden(void);
int gr_lstm_forward(const float* gates_x, const float* W_hh, const float* b_hh, float* hidden, int B, int Q,
                    int D, void* stream);

/* seed_retrieve[b,:] = sum_n seed_info[b,n] * h[b,n,:]  (torch.bmm in QueryReform.forward,
 * gnn/modules/query_update.py:40); only rows with seed_info != 0 are read, in index order. */
int gr_seed_retrieve(const float* seed_info, const float* h, int64_t ldh, float* out,
                     int B, int N, int D, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Candidate ranking = the retrieved answer-node set, Evaluator.evaluate + f1_and_hits
 * (gnn/evaluate.py:156, 188-209, 25-50).  Per question: drop seeds (query_entities truncated to an
 * integer == 1), pads (local_entity == pad_id) and p < (1-eps)/N (compared in double); stable sort by
 * p descending (ties keep local-index order, -0.0 ties with +0.0, negative p last); keep the prefix up
 * to and including the item at which the sequential float64 running sum exceeds eps.  Any eps; p may
 * be any fp32 value but NaN.
 *   cand_idx:  int32[B, N]  local indices in retrieval order (first cand_count[b] valid, 0 past cand_total[b])
 *   cand_count:int32[B]; cand_total:int32[B] = number of candidates before the eps cut.
 * Workspace: gr_rank_workspace_bytes(B, N).
 */
size_t gr_rank_workspace_bytes(int B, int N);
int gr_rank_candidates(const float* dist, const int64_t* local_entity, const float* query_entities,
                       int64_t pad_id, double eps, int32_t* cand_idx, int32_t* cand_count,
                       int32_t* cand_total, int B, int N, void* workspace, size_t workspace_bytes,
                       void* stream);

/* Train-time metrics, get_eval_metric (gnn/models/base_model.py:236-298), per question, no host involvement:
 *   h1[b] = 1 when answer_dist > 1e-10 (fp32 compare) at the top-1 of pred_dist (torch.argmax: first maximal index,
 *           NaN counts as maximal), else 0;
 *   f1[b] = for h1 = 1: F1 of the retrieval = the first cand_count[b] local indices of cand_idx (gr_rank_candidates
 *           with query_entities = (seed_dist > 0)) against the answers = nodes with answer_dist > 0, seed_dist <= 0 and
 *           local_entity != pad_id, matched by ENTITY ID (np.isin; a repeated id counts once per answer node in the
 *           recall denominator and once per candidate in the count of correct ones).  No answers: 1 if no candidates
 *           else 0; no candidates or none correct: 0.  Evaluated in float64 and rounded once to fp32.  0 for h1 = 0.
 *   pred_dist, answer_dist, seed_dist: fp32 [B, N]; local_entity: int64 [B, N]; cand_idx: int32 [B, N];
 *   cand_count: int32 [B]; h1, f1: fp32 [B].  Refused: null pointers, B or N not positive. */
int gr_train_metrics(const float* pred_dist, const float* answer_dist, const float* seed_dist,
                     const int64_t* local_entity, int64_t pad_id, const int32_t* cand_idx, const int32_t* cand_count,
                     float* h1, float* f1, int B, int N, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Gradient clipping + Adam over fp32 tensor lists (csrc/optim.cu): torch.nn.utils.clip_grad_norm_(params, max_norm)
 * followed by torch.optim.Adam.step() (gnn/train_model.py:91-92, 221-230), bit for bit as torch's default CUDA path,
 * torch.optim.adam._multi_tensor_adam (foreach, not capturable, no amsgrad / maximize / decoupled weight decay).
 * Deterministic, no atomics.
 *
 * table: int64 [T][6], one row per tensor: {param, grad, exp_avg, exp_avg_sq, numel, flags} (device pointers as
 *   integers; exp_avg = 0: the row is clipped but not updated; flags: GR_ADAM_ALIGNED16 when every pointer of the row
 *   is 16-byte aligned).  Tensors are contiguous fp32; numel may be 0.
 * scalars: fp32 [T][8], per tensor, each rounded from the float64 value torch computes on the host:
 *   {1 - beta1, beta2, 1 - beta2, eps, weight_decay, step_size = -(lr / (1 - beta1^t)), (1 - beta2^t) ** 0.5, 0}.
 * chunks: int32 [C][2] = {tensor row, chunk index k}: the elements [k E, min((k + 1) E, numel)) of that tensor,
 *   E = gr_adam_chunk_elems().  One CTA per chunk.
 * gr_grad_sumsq: slots[c] (float64 [C]) = sum of grad^2 over chunk c.
 * gr_clip_adam: with slots (clipping): total = sqrt of the sum of slots[0 .. C) in one fixed order, in float64, rounded
 *   once to fp32 and written to grad_norm[0] (fp32, may be NULL); coef = min(fp32(1 / (total + 1e-6)) * max_norm, 1)
 *   in fp32 (clip_grads_with_norm_: a NaN total gives NaN, an infinite one 0); grad *= coef, written back.  Then
 *   for every row with exp_avg: g = grad (+ weight_decay * param when weight_decay != 0, not written back);
 *   exp_avg.lerp_(g, 1 - beta1) (ATen/native/Lerp.h); exp_avg_sq = exp_avg_sq * beta2, then + (1 - beta2) g g
 *   (addcmul); param += step_size * (exp_avg / (sqrt(exp_avg_sq) / bc2_sqrt + eps)) (addcdiv); one fp32 rounding
 *   per foreach op.  slots = NULL: no clipping (max_norm and grad_norm unused; grad_norm must be NULL).
 *   flags: GR_ADAM_WEIGHT_DECAY when any row has weight_decay != 0 (without it the weight decay is not read).
 */
#define GR_ADAM_ALIGNED16 1
#define GR_ADAM_WEIGHT_DECAY 1u
int gr_adam_chunk_elems(void);
int gr_grad_sumsq(const int64_t* table, const int32_t* chunks, int C, double* slots, void* stream);
int gr_clip_adam(const int64_t* table, const float* scalars, const int32_t* chunks, int C, const double* slots,
                 double max_norm, float* grad_norm, uint32_t flags, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Device-resident split (loader.DeviceSplit, csrc/split.cu): a split's per-question facts are uploaded once and
 * every batch is assembled on the device from B question ids (the int64 device array `ids`, B > 0).
 * A question id outside [0, num_q) counts as an empty question and sets bit 1 of `status` (int32[1], OR-ed); a batch
 * whose entries would run past the capacity passed (F, G) is cut there and sets bit 2.  Nothing is read or written
 * outside the arrays.  Index outputs are int64 (idx_bytes = 8) or int32 (idx_bytes = 4; refused when B*N, the
 * capacity or self_rel exceed INT_MAX).  Launch shape: (CTAs per question, B), a function of B alone.
 *
 * gr_split_assemble: the kb_adj_mat arrays of SingleDataLoader._build_fact_mat (gnn/dataset_load.py:473-527) in
 * STORED fact order (loader.build_fact_mat with shuffle=False): question b = ids[b] contributes its facts
 * q_heads/q_rels/q_tails[q_off[id] .. q_off[id+1]) (int32 local ids) with heads/tails + b*N, then, with use_self_loop,
 * one self-loop (b*N + k, self_rel, b*N + k) for each k < q_ents[id]; batch_ids = b, fact_ids = position.
 * q_off: int64 [num_q+1]; q_ents: int32 [num_q]; outputs: [F], F = the batch's fact count computed by the caller. */
int gr_split_assemble(const int64_t* q_off, const int32_t* q_heads, const int32_t* q_rels, const int32_t* q_tails,
                      const int32_t* q_ents, int64_t num_q, const int64_t* ids, int B, int64_t N, int64_t self_rel,
                      int use_self_loop, int idx_bytes, int64_t F, void* heads, void* rels, void* tails,
                      void* batch_ids, void* fact_ids, int32_t* status, void* stream);

/* gr_split_assemble_graft: the graft lists of GraftSingleDataLoader._build_fact_mat_maxfacts
 * (gnn/dataset_load_graft.py:70-102) in stored order: question b = ids[b] contributes entries g_off[id] .. g_off[id+1]
 * to e2f = (b, g_e2f_f, g_e2f_e, 1.0) and f2e = (b, g_f2e_e, g_f2e_f, 1.0); the lists have G entries.  kb_fact_rel
 * int64 [B, max_facts]: row b = r_vals[r_off[id] .. r_off[id+1]) (at most max_facts entries), then rel_pad. */
int gr_split_assemble_graft(const int64_t* g_off, const int32_t* g_e2f_f, const int32_t* g_e2f_e,
                            const int32_t* g_f2e_e, const int32_t* g_f2e_f, const int64_t* r_off,
                            const int32_t* r_vals, int64_t num_q, const int64_t* ids, int B, int64_t max_facts,
                            int64_t rel_pad, int idx_bytes, int64_t G, void* e2f_b, void* e2f_f, void* e2f_e,
                            float* e2f_v, void* f2e_b, void* f2e_e, void* f2e_f, float* f2e_v, int64_t* kb_fact_rel,
                            int32_t* status, void* stream);

/* gr_fact_weights: weight_list / weight_rel_list of _build_fact_mat (gnn/dataset_load.py:507-516) for F facts with
 * global head rows in [0, Nt): weight[f] = 1 / #facts with head[f], weight_rel[f] = 1 / #facts with (head[f], rel[f]),
 * each 1.0 / count in float64 rounded once to fp32 (bit-equal to fp32 of the host's float64 values).  Integer
 * counting only (no float atomics).  Either output may be null (not both).  A fact whose head is outside [0, Nt) or
 * whose relation is negative sets status bit 1, is left out of the counts and gets weight 0.  F <= INT_MAX.
 * Workspace: gr_fact_weights_workspace_bytes(F, Nt). */
size_t gr_fact_weights_workspace_bytes(int64_t F, int64_t Nt);
int gr_fact_weights(const void* heads, const void* rels, int idx_bytes, int64_t F, int64_t Nt, float* weight,
                    float* weight_rel, int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* gr_fact_weights_live: gr_fact_weights over the live prefix of capacity-length fact buffers, the live count read
 * from the device: F = min(capacity, max(*nfacts, 0)) (nfacts: int32[1], as gr_csr_build reads it).  Slots
 * [F, capacity) (a previous batch's facts) are neither counted nor flagged, and their weights are not written; the
 * live prefix is bit-equal to gr_fact_weights over F facts.  Workspace: gr_fact_weights_workspace_bytes(capacity, Nt). */
int gr_fact_weights_live(const void* heads, const void* rels, int idx_bytes, int64_t capacity, const int32_t* nfacts,
                         int64_t Nt, float* weight, float* weight_rel, int32_t* status, void* workspace,
                         size_t workspace_bytes, void* stream);

/* Fact dropout on a resident split (loader.DeviceSplit with shuffle=True): the reference keeps the first
 * floor(n (1 - p)) facts of a fresh np.random.permutation of each question's n stored facts.  `kept` (int64 [B], from
 * the host) holds those counts; a count is clamped to [0, n] (n = 0 for an id out of range).
 *
 * gr_split_fact_order: order (int32 [K]) = per question b, in batch order, the stored indices (0 .. n-1) of the first
 * kept[b] facts of the permutation that sorts the question's facts by (key, index) ascending, where fact i's key is
 * the 64-bit value whose high word is philox4x32_10_x0(*seed, i lo, i hi, b, perm) and whose low word is
 * philox4x32_10_x0(*seed, i lo, i hi, b, perm | 2).  perm = 0 for the kb facts, 1 for the graft lists.  off is the
 * question offsets (q_off or g_off, int64 [num_q+1]); seed is one int64 on the device.  Deterministic for a seed.
 * n_total >= the sum of the stored counts of the B questions sizes the workspace
 * (gr_split_fact_order_workspace_bytes(n_total)).  A question whose kept prefix would run past K, or that holds more
 * than INT_MAX facts, is not written and sets status bit 2.  One CTA per question, any question size. */
size_t gr_split_fact_order_workspace_bytes(int64_t n_total);
int gr_split_fact_order(const int64_t* off, int64_t num_q, const int64_t* ids, const int64_t* kept, int B,
                        const int64_t* seed, int perm, int64_t n_total, int64_t K, int32_t* order, int32_t* status,
                        void* workspace, size_t workspace_bytes, void* stream);

/* gr_split_assemble_ordered: gr_split_assemble with question b contributing the facts order[o_b .. o_b + kept[b])
 * (stored indices; o_b = the kept counts before b) instead of all of its facts, then its self-loops.  F = the sum of
 * kept[b] (+ q_ents with use_self_loop).  An order entry outside [0, n) sets status bit 1 and its fact is not
 * written; reading past K sets bit 2. */
int gr_split_assemble_ordered(const int64_t* q_off, const int32_t* q_heads, const int32_t* q_rels,
                              const int32_t* q_tails, const int32_t* q_ents, int64_t num_q, const int64_t* ids,
                              const int64_t* kept, const int32_t* order, int64_t K, int B, int64_t N,
                              int64_t self_rel, int use_self_loop, int idx_bytes, int64_t F, void* heads, void* rels,
                              void* tails, void* batch_ids, void* fact_ids, int32_t* status, void* stream);

/* gr_split_assemble_graft_ordered: gr_split_assemble_graft with both graft lists taking question b's entries at the
 * positions order[o_b .. o_b + kept[b]) (G = the sum of kept[b]); the kb_fact_rel rows are the stored ones. */
int gr_split_assemble_graft_ordered(const int64_t* g_off, const int32_t* g_e2f_f, const int32_t* g_e2f_e,
                                    const int32_t* g_f2e_e, const int32_t* g_f2e_f, const int64_t* r_off,
                                    const int32_t* r_vals, int64_t num_q, const int64_t* ids, const int64_t* kept,
                                    const int32_t* order, int64_t K, int B, int64_t max_facts, int64_t rel_pad,
                                    int idx_bytes, int64_t G, void* e2f_b, void* e2f_f, void* e2f_e, float* e2f_v,
                                    void* f2e_b, void* f2e_e, void* f2e_f, float* f2e_v, int64_t* kb_fact_rel,
                                    int32_t* status, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Step bookkeeping of a training epoch replayed as CUDA graphs (csrc/epoch.cu, graphed.GraphedTrainStep.start_epoch).
 * cursor: int64[1] on the device, the step index c; step c covers positions [c * batch_size, min((c + 1) * batch_size,
 * num_data)) of order (int64 [num_data], the epoch's question ids); B is that step's batch size.  One CTA each, no
 * atomics.
 *
 * gr_epoch_step_begin: for j < B, id = order[c * batch_size + j] (-1 past num_data); an id outside [0, num_q) sets
 *   status bit 1 and counts as an empty question.  ids[j] = id (for the gr_split_* kernels), rows[j] = id or 0 when
 *   out of range (for row gathers), kept[j] = kept_table[id] clamped to [0, n] (n = the stored facts, q_off[id + 1] -
 *   q_off[id]; kept_table NULL: n).  kept_total[0] = sum of kept; nfacts[0] = min(sum of kept + q_ents (with
 *   use_self_loop), capacity); a sum past capacity sets status bit 2.  status[0] is written, not OR-ed.
 * gr_epoch_graft_begin: GraftNet's half of the head, after gr_epoch_step_begin, from the ids it wrote (int64 [B]): for
 *   j < B, kept_g[j] = kept_table[ids[j]] clamped to [0, n] (n = the stored graft entries, g_off[id + 1] - g_off[id];
 *   kept_table NULL: n; an id outside [0, num_q) counts as an empty question, n = 0).  graft_live[0] = graft_live[1]
 *   = min(G, capacity) with G the sum of kept_g (the `live` gr_graft_stage reads); status[0] = 2 when G > capacity,
 *   else 0 (written, not OR-ed).  g_off: int64 [num_q+1]; kept_table: int64 [num_q] or NULL.
 * gr_epoch_step_record: with c in [0, steps): losses[c] = *loss, grad_norms[c] = *grad_norm and seeds[c] = *seed (both
 *   optional, each with its record array), h1_all / f1_all[c * batch_size + j] = h1 / f1[j] for j < B (positions
 *   below num_data).  epoch_status[0] |= *split_status, epoch_status[1] |= *csr_status; a cursor outside [0, steps)
 *   records nothing and sets bit 2 of epoch_status[0].  Then cursor = c + 1. */
int gr_epoch_step_begin(const int64_t* cursor, const int64_t* order, int64_t num_data, int64_t batch_size, int B,
                        const int64_t* kept_table, const int64_t* q_off, const int32_t* q_ents, int64_t num_q,
                        int use_self_loop, int64_t capacity, int64_t* ids, int64_t* rows, int64_t* kept,
                        int32_t* nfacts, int64_t* kept_total, int32_t* status, void* stream);
int gr_epoch_graft_begin(const int64_t* ids, int B, const int64_t* kept_table, const int64_t* g_off, int64_t num_q,
                         int64_t capacity, int64_t* kept_g, int32_t* graft_live, int32_t* status, void* stream);
int gr_epoch_step_record(int64_t* cursor, int64_t steps, int64_t batch_size, int B, int64_t num_data,
                         const float* loss, const float* grad_norm, const int64_t* seed, const float* h1,
                         const float* f1, const int32_t* split_status, const int32_t* csr_status, float* losses,
                         float* grad_norms, int64_t* seeds, float* h1_all, float* f1_all, int32_t* epoch_status,
                         void* stream);

/* gr_eval_step_record: the tail of an evaluation epoch step (graphed.GraphedStep.start_eval), after
 * gr_epoch_step_begin, the serving forward and gr_rank_candidates.  With c in [0, steps), for every j < B whose
 * position p = c * batch_size + j is below num_data: C = cand_count[j] clamped to [0, N], the candidates
 * e_k = local_entity[j, cand_idx[j, k]] (k < C; cand_idx entries in [0, N)) and the answers of ids[j], the ascending
 * run a_ids[a_off[id] .. a_off[id + 1]) of length A (A = 0 for an id outside [0, num_a)).  As f1_and_hits
 * (evaluate.f1_and_hits): correct = #{k : e_k among the answers}, hit = (e_0, or -1 when C = 0, among the answers),
 * case 0 (A = 0, C = 0), 1 (A = 0), 2 (C = 0) or 3, with p = correct / C, r = correct / A and
 * f1 = 2 / (1/p + 1/r) (0 when p or r is 0) in IEEE round-to-nearest float64.  Writes metrics[p] = (precision,
 * recall, f1, hit, em) (float64 [num_data, 5]), cases[p] (int8), counts[p] = C (int32) and cand_off[p] (int64), the
 * offset of its candidates in the flat records: cand_off of the step's recorded questions is the exclusive scan of
 * their C in batch order, starting at *cand_total.  Candidate k of position p goes to record cand_off[p] + k of cand
 * (int64 [capacity, 2]: the entity id, then the int32 pair (local index, fp32 bits of pred_dist[j, local index])) when
 * all C of them fit below capacity; a question that does not fit is not written and sets bit 1 of eval_status[2].
 * Then *cand_total = cand_off past the step's last record and seeds[c] = *seed (both optional together).
 * eval_status[0] |= *split_status, eval_status[1] |= *csr_status; a cursor outside [0, steps) records nothing and sets
 * bit 2 of eval_status[0].  Then cursor = c + 1.  pred_dist fp32, local_entity int64, cand_idx int32: [B, N]. */
int gr_eval_step_record(int64_t* cursor, int64_t steps, int64_t batch_size, int B, int64_t num_data, int64_t N,
                        const int64_t* ids, const int64_t* local_entity, const float* pred_dist,
                        const int32_t* cand_idx, const int32_t* cand_count, const int64_t* a_off,
                        const int64_t* a_ids, int64_t num_a, const int64_t* seed, const int32_t* split_status,
                        const int32_t* csr_status, double* metrics, int8_t* cases, int32_t* counts, int64_t* cand_off,
                        int64_t* cand, int64_t capacity, int64_t* cand_total, int64_t* seeds, int32_t* eval_status,
                        void* stream);

/* ------------------------------------------------------------------------------------------------
 * The `.info` file of an evaluation epoch (csrc/info_rows.cu, graphed.EvalRun.info): one JSONL row per position p of
 * the run, byte for byte the json.dumps row evaluate.Evaluator writes:
 *   prefix[q]  "precison": P, "recall": R, "f1": F, "hit": H, "em": E, "cand": [["name", prob], ...]}\n
 * with q = order[p] (int64 [num_data]).  The records are gr_eval_step_record's: metrics float64 [num_data, 5], cases
 * int8, counts int32 and cand_off int64 [num_data], cand_total int64[1], eval_status int32[4] (the run's status words)
 * and cand int64 [capacity, 2].  The numbers are Python reprs of float64 values (shortest round trip, csrc/float_repr.cuh)
 * -- em an int (0 / 1) in case 3 -- and each prob is the float64 of the candidate record's fp32.  Host-built tables:
 * prefix (bytes) with prefix_off int64 [num_q + 1], question q's text up to and including `"answers": [...], `;
 * names (bytes) with name_off int64 [num_names + 1], JSON strings with their quotes; name_slot int32 [num_entity],
 * the name of each entity id or -1.
 *
 * gr_info_rows_size: row_off int64 [num_data + 1] = the rows' byte offsets (row_off[0] = 0) and summary int64[2] =
 *   (total bytes, flags).  flags: 1 a status word is nonzero; else the OR over the rows of 2 (q outside [0, num_q), or
 *   candidates outside [0, min(*cand_total, capacity))) and 4 (a candidate entity without a name).  With flags the
 *   total is 0.  Two launches, no workspace.
 * gr_info_rows_write: the rows into out (out_bytes >= summary[0]) at row_off; writes nothing when summary[1] != 0 or
 *   summary[0] > out_bytes.  Same records and tables as the size call. */
int gr_info_rows_size(const double* metrics, const int8_t* cases, const int32_t* counts, const int64_t* cand_off,
                      const int64_t* cand_total, const int32_t* eval_status, int64_t num_data, const int64_t* cand,
                      int64_t capacity, const int64_t* order, const int64_t* prefix_off, int64_t num_q,
                      const int32_t* name_slot, int64_t num_entity, const int64_t* name_off, int64_t num_names,
                      int64_t* row_off, int64_t* summary, void* stream);
int gr_info_rows_write(const double* metrics, const int8_t* cases, const int32_t* counts, const int64_t* cand_off,
                       const int64_t* cand_total, int64_t num_data, const int64_t* cand, int64_t capacity,
                       const int64_t* order, const uint8_t* prefix, const int64_t* prefix_off, int64_t num_q,
                       const int32_t* name_slot, int64_t num_entity, const uint8_t* names, const int64_t* name_off,
                       int64_t num_names, const int64_t* row_off, const int64_t* summary, uint8_t* out,
                       int64_t out_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Shortest-path node sets (SURVEY.md 8f row 1): nodes lying on any shortest path between any seed and
 * any retrieved candidate in the UNDIRECTED subgraph -- build_graph + get_truth_paths,
 * llm/src/utils/graph_utils.py:10-21,49-75.  Uses both CSRs of a question batch.  One CTA per (question, root) runs a
 * level-synchronous BFS from one of the question's sources or targets; one CTA per question then marks the nodes.
 *   source_idx int32 [B, max_sources] / target_idx int32 [B, max_targets]: local indices in [0, N), the first
 *   source_cnt[b] / target_cnt[b] of each row used.  on_path: uint8 [B, N] output, 1 on a shortest path of a connected
 *   (source, target) pair.  pair_dist: int32 [B, max_sources, max_targets] hop distances, -1 unreachable and past the
 *   counts.  The workspace keeps the BFS distances int32 [B, max_sources + max_targets, N] (sources first, -1
 *   unreachable); rows past the counts are not written.
 */
size_t gr_paths_workspace_bytes(int B, int N, int max_sources, int max_targets);
int gr_shortest_path_nodes(const int32_t* rowptr_t, const int32_t* src_t,
                           const int32_t* rowptr_h, const int32_t* src_h,
                           const int32_t* source_idx, const int32_t* source_cnt, int max_sources,
                           const int32_t* target_idx, const int32_t* target_cnt, int max_targets,
                           uint8_t* on_path, int32_t* pair_dist, int B, int N,
                           void* workspace, size_t workspace_bytes, void* stream);

/* gr_eval_step_paths: the shortest-path node sets of an evaluation epoch step (graphed.GraphedStep.start_eval with
 * path_targets), after gr_rank_candidates and before gr_eval_step_record, which advances the cursor.  With c = *cursor
 * in [0, steps), for every j < B whose position p = c * batch_size + j is below num_data: the sources are the local
 * indices with query_entities[j, v] != 0 in increasing order (the first S of them), the targets the first
 * min(cand_count[j], T) entries of cand_idx[j] (cand_idx int32 [B, N]); BFS over both CSRs of the step's batch as in
 * gr_shortest_path_nodes.  Writes pair_dist[p] (int32 [num_data, S, T], -1 unreachable and past the counts),
 * node_count[p] (int32 [num_data]) = the number of on-path nodes, and node_off[p] (int64 [num_data]): the exclusive
 * scan of the step's counts in batch order from *node_total.  The nodes of position p, ascending local indices, go
 * to nodes[node_off[p] ..] (int32 [capacity]) when all of the step's nodes fit below capacity; otherwise the step
 * writes no node and sets bit 2 of *eval_status.  Then *node_total moves past the step's nodes.  A cursor outside
 * [0, steps) writes nothing.  No atomics.  Refused: B * (S + T) * N above INT_MAX.  query_entities fp32 [B, N].
 * Workspace: gr_eval_paths_workspace_bytes(B, N, S, T). */
size_t gr_eval_paths_workspace_bytes(int B, int64_t N, int S, int T);
int gr_eval_step_paths(const int64_t* cursor, int64_t steps, int64_t batch_size, int B, int64_t num_data, int64_t N,
                       const float* query_entities, const int32_t* cand_idx, const int32_t* cand_count, int S, int T,
                       const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rowptr_h, const int32_t* src_h,
                       int64_t* node_off, int32_t* node_count, int32_t* pair_dist, int32_t* nodes, int64_t capacity,
                       int64_t* node_total, int32_t* eval_status, void* workspace, size_t workspace_bytes,
                       void* stream);

/* ------------------------------------------------------------------------------------------------
 * Rule-guided reasoning paths (csrc/rule_paths.cu): bfs_with_rule over the undirected graph of build_graph
 * (llm/src/utils/graph_utils.py:10-47) for many (start node, relation rule) jobs at once -- the calls
 * PromptBuilder.apply_rules makes (llm/src/qa_prediction/build_qa_input.py:58-64).  Exact: every walk whose i-th edge
 * label equals rule[i] (nodes may repeat), in the reference's FIFO order, never truncated.  Integer-only, bit-exact.
 *
 * gr_rule_adj_build: label-grouped adjacency from the two CSRs of gr_csr_build called with rels = per-triple LABEL ids
 * (the stripped relation strings interned by the caller).  Row u lists each distinct neighbour once (nx.Graph),
 * sorted by (label of the pair's LAST triple, the pair's FIRST triple), so the neighbours with one label form a
 * contiguous segment in graph.neighbors(u) order.
 *   adj_rowptr: int32[Nt+1] = rowptr_t + rowptr_h (row capacity); adj_len: int32[Nt] = entries used in each row;
 *   adj_nbr, adj_lab: int32[2F].  Workspace: gr_rule_adj_workspace_bytes(F).
 *
 * Level expansion.  Jobs j < J: rule = rule_lab[job_rule_off[j] .. + job_rule_len[j]) (label ids; -1 = a label absent
 * from the graph, which matches nothing).  The caller orders the jobs (apply_rules: source-major, rule-minor) and
 * builds level 0 = one entry (node, job) per job, job ascending: node = the start node, or -1 for a start that is not
 * in the graph (kept only when the rule is empty: the reference returns one empty path then).  Level l (l = 0, 1, ...):
 *   gr_rule_level_count: for every entry, the length of its node's segment with label rule[l] (0 when the job's rule
 *     is shorter), scanned in place into child_off: int64[n+1], child_off[n] = the next level's size (read it back
 *     and allocate the next level).  seg_begin: int32[n].  Jobs whose rule length is l are finished: their entries
 *     are their result paths, res_begin[j] / res_count[j] (int32[J]) receive that run of the level.  Workspace:
 *     gr_rule_level_workspace_bytes(n).
 *   gr_rule_level_emit: writes the next level, int32[total] each: child_node, child_parent (entry index in level l),
 *     child_job; children of one entry are consecutive, in segment order.  A level of more than INT32_MAX entries is
 *     refused with GR_ERR_UNSUPPORTED and the count in gr_last_error (never clamped).
 * gr_rule_paths_write: after the last level; level_node / level_parent are DEVICE arrays of the per-level device
 * pointers (level 0's parents are not read).  path_off: int64[J+1] exclusive sums of res_count; elem_off: int64[J]
 * exclusive sums of res_count[j] * (job_rule_len[j] + 1).  Path k of job j is written to
 * paths[elem_off[j] + k*(len+1) ...] as its len+1 node ids, start first; P = path_off[J].
 */
size_t gr_rule_adj_workspace_bytes(int64_t F);
int gr_rule_adj_build(const int32_t* rowptr_t, const int32_t* src_t, const int32_t* rel_t, const int32_t* fact_t,
                      const int32_t* rowptr_h, const int32_t* src_h, const int32_t* rel_h, const int32_t* fact_h,
                      int64_t Nt, int64_t F, int32_t* adj_rowptr, int32_t* adj_len, int32_t* adj_nbr,
                      int32_t* adj_lab, void* workspace, size_t workspace_bytes, void* stream);
size_t gr_rule_level_workspace_bytes(int64_t n);
int gr_rule_level_count(const int32_t* adj_rowptr, const int32_t* adj_len, const int32_t* adj_lab,
                        const int32_t* job_rule_off, const int32_t* job_rule_len, const int32_t* rule_lab, int J,
                        int level, const int32_t* node, const int32_t* job, int64_t n, int32_t* seg_begin,
                        int64_t* child_off, int32_t* res_begin, int32_t* res_count, void* workspace,
                        size_t workspace_bytes, void* stream);
int gr_rule_level_emit(const int32_t* adj_nbr, const int32_t* job, const int32_t* seg_begin, const int64_t* child_off,
                       int64_t n, int64_t total, int32_t* child_node, int32_t* child_parent, int32_t* child_job,
                       void* stream);
int gr_rule_paths_write(const int32_t* const* level_node, const int32_t* const* level_parent,
                        const int32_t* job_rule_len, const int32_t* res_begin, const int64_t* path_off,
                        const int64_t* elem_off, int J, int64_t P, int32_t* paths, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GNNRAG_B200_H_ */
