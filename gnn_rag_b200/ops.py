"""Tensor-level wrappers over the C ABI (include/gnnrag_b200.h): torch CUDA tensors in, torch CUDA tensors
out.  torch is used for device memory and streams only; every op below launches our own sm_90a kernels.
All ops raise if handed a CPU tensor -- there is no CPU fallback on the product path.

Each kernel's shape rule (``*_ok``) sits next to its wrapper: the training path asks it to choose between a kernel and
its torch restatement, and tests/test_entry_refusals_host.py holds it to the entry point's own refusals."""
import contextlib
import ctypes
import functools
import weakref

import numpy as np
import torch

from . import _lib

LINEAR_RELU = 1
LINEAR_EXACT_FP32 = 2
LINEAR_W_PRESPLIT = 4
LINEAR_BF16_SINGLE = 8
LINEAR_K_GROUPED = 16
LINEAR_K_ORDER_PLANES = 32
AGG_K_ORDER = 1

# bf16 ACTIVATION STORAGE (BASELINE configs[2], "bf16"): the layer-input matrix keeps its hi plane only -- the aggregation
# kernel skips the lo plane (half the output bytes) and the e2e GEMM runs ONE bf16 product instead of three.  Tables,
# accumulation, scores and softmax stay fp32.  Off by default (cfg2's contract is fp32); bench.py --config cfg3 turns it on.
ACT_BF16 = False


class _Stats:
    """Launch accounting (bench.py's ``gpu_launches``) and optional CUDA-event timing of the aggregation
    launches (bench.py's live roofline measurement).  Events are recorded on the launching stream."""

    def __init__(self):
        self.launches = 0
        self.time_agg = False
        self.agg_events = []      # (start_event, end_event, tag)
        self.time_ops = False     # bench.py's per-kernel-class share table: events around every wrapper below
        self.op_events = []       # (start_event, end_event, class tag, info)

    def reset(self):
        self.launches = 0
        self.agg_events = []
        self.op_events = []


STATS = _Stats()


class _Timer:
    """CUDA events (on the launching stream) around one wrapper call: into ``STATS.op_events`` as op class ``op`` with
    ``info`` when ``STATS.time_ops`` is on.  An aggregation tag ``agg`` makes the class "aggregation" with the tag as
    info, and also goes into ``STATS.agg_events`` when ``STATS.time_agg`` is on.  Neither given: untimed."""

    def __init__(self, op=None, info=None, agg=None):
        if agg is not None:
            op, info = "aggregation", agg
        self.op, self.info, self.agg = op, info, agg

    def __enter__(self):
        self.to_ops = self.op is not None and STATS.time_ops
        self.to_agg = self.agg is not None and STATS.time_agg
        if self.to_ops or self.to_agg:
            self.s = torch.cuda.Event(enable_timing=True)
            self.e = torch.cuda.Event(enable_timing=True)
            self.s.record()
        return self

    def __exit__(self, *a):
        if self.to_ops or self.to_agg:
            self.e.record()
            if self.to_agg:
                STATS.agg_events.append((self.s, self.e, self.agg))
            if self.to_ops:
                STATS.op_events.append((self.s, self.e, self.op, self.info))


def _L():
    return _lib.load()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _launch(name, *args, io=0, launches=1, op=None, info=None, agg=None):
    """Call C entry point ``name`` with ``args`` and the current stream; with io flags its ``*_ex`` form, which takes
    the flags before the stream.  Timed as :class:`_Timer` says (``op``, ``info``, ``agg``); raises on any refusal and
    adds ``launches`` to ``STATS.launches``."""
    fn = getattr(_L(), name + "_ex" if io else name)
    args = (*args, io, _stream()) if io else (*args, _stream())
    if (op is None and agg is None) or not (STATS.time_ops or STATS.time_agg):     # untimed: no per-call timer object
        rc = fn(*args)
    else:
        with _Timer(op, info, agg):
            rc = fn(*args)
    _lib.check(rc)
    STATS.launches += launches


def _workspace(device, sizer, *sizes):
    """(workspace, nbytes): an uninitialised device buffer of the bytes the size entry point ``sizer`` asks for."""
    nbytes = getattr(_L(), sizer)(*sizes)
    return torch.empty(nbytes, dtype=torch.uint8, device=device), nbytes


def _p(t):
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def _cuda(t, dtype=None, name="tensor"):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor (no CPU fallback on this path)" % name)
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError("%s must be %s, got %s" % (name, dtype, t.dtype))
    return t


def pad4(n):
    return (n + 3) & ~3


IO_BF16 = 1     # GR_IO_BF16: the node-sized tensors of a training entry point are bf16 (include/gnnrag_b200.h)


def _node_io(**tensors):
    """io flags of the training entry points for their node-sized tensors (name -> tensor, None skipped): 0 when they
    are torch.float32, IO_BF16 when they are torch.bfloat16 (training under torch.autocast).  Any other dtype, or a
    mix of the two, is refused."""
    ts = {k: _cuda(v, name=k) for k, v in tensors.items() if v is not None}
    for k, t in ts.items():
        if t.dtype not in (torch.float32, torch.bfloat16):
            raise RuntimeError("%s must be torch.float32 or torch.bfloat16, got %s" % (k, t.dtype))
    if len({t.dtype for t in ts.values()}) > 1:
        raise RuntimeError("%s must share one dtype, got %s" % (", ".join(ts), ", ".join(str(t.dtype) for t in ts.values())))
    return IO_BF16 if any(t.dtype == torch.bfloat16 for t in ts.values()) else 0


def set_option(name, value):
    _lib.check(_L().gr_set_option(name.encode(), int(value)))


class CsrGraph:
    """Both destination-CSRs of one batched subgraph (device resident).

    ``*_t``: in-edges grouped by tail (forward messages, src = head); ``*_h``: grouped by head (inverse
    messages, src = tail).  ``fact_*`` maps a CSR slot back to the original fact id, so per-fact arrays
    (weights) can be permuted with :func:`gather_f32`.
    """

    def __init__(self, B, N, F, R1, device):
        self.B, self.N, self.F, self.R1 = B, N, F, R1
        Nt = B * N
        i32 = dict(dtype=torch.int32, device=device)
        self.rowptr_t = torch.empty(pad4(Nt + 1), **i32)
        self.rowptr_h = torch.empty(pad4(Nt + 1), **i32)
        Fp = max(pad4(F), 4)
        self.src_t = torch.empty(Fp, **i32)
        self.rel_t = torch.empty(Fp, **i32)
        self.fact_t = torch.empty(Fp, **i32)
        self.src_h = torch.empty(Fp, **i32)
        self.rel_h = torch.empty(Fp, **i32)
        self.fact_h = torch.empty(Fp, **i32)
        self.status = torch.zeros(1, **i32)
        self.w_t = self.w_h = None        # normalized_gnn edge weights (1/outdeg(head))
        self.wr_t = self.wr_h = None      # norm_rel edge weights (1/count(head, rel))
        self.nfacts = None                # device int32[1] live fact count when F is a capacity
        self.rel_index = {}               # direction -> relation index of that CSR (deterministic backward)

    def csr(self, direction):
        """(rowptr, src, rel, fact) of one destination CSR: 'fwd' = the tail CSR, 'inv' = the head CSR."""
        if direction == "fwd":
            return self.rowptr_t, self.src_t, self.rel_t, self.fact_t
        return self.rowptr_h, self.src_h, self.rel_h, self.fact_h

    def check_status(self):
        if int(self.status.item()) != 0:
            raise RuntimeError("fact list contains node/relation ids outside the batch (clamped)")


def csr_build(heads, rels, tails, B, N, R1, nfacts=None):
    """heads/rels/tails: 1-D int64 or int32 CUDA tensors (global rows b*N+local) -> CsrGraph.
    ``nfacts``: optional int32[1] device tensor -- only the first ``nfacts`` slots are facts, the rest is capacity
    padding of fixed-shape buffers (GraphedStep)."""
    heads, rels, tails = _cuda(heads, name="heads"), _cuda(rels, name="rels"), _cuda(tails, name="tails")
    if heads.dtype not in (torch.int64, torch.int32) or rels.dtype != heads.dtype or tails.dtype != heads.dtype:
        raise RuntimeError("fact arrays must share dtype int64 or int32")
    F = heads.numel()
    g = CsrGraph(B, N, F, R1, heads.device)
    ws, ws_bytes = _workspace(heads.device, "gr_csr_build_workspace_bytes", F, B * N)
    # memsets excluded: hist, 3x scan, place, 2x sort, fill (+gather)
    _launch("gr_csr_build", _p(heads.contiguous()), _p(rels.contiguous()), _p(tails.contiguous()),
            heads.element_size(), F, B * N, R1,
            _p(g.rowptr_t), _p(g.src_t), _p(g.rel_t), _p(g.fact_t),
            _p(g.rowptr_h), _p(g.src_h), _p(g.rel_h), _p(g.fact_h),
            _p(g.status), _p(nfacts), _p(ws), ws_bytes, launches=9 if F > 0 else 5, op="csr_build")
    g.nfacts = nfacts
    return g


def _relation_index(keys, R1, nfacts=None):
    """(rix_ptr int32 [R1+1], rix_slot): the positions of ``keys`` (a relation id per list entry, int32 or int64,
    all in [0, R1)) grouped by relation, in increasing position inside each relation -- gr_csr_build keyed on the
    relation.  The list order the deterministic backward kernels sum in."""
    g = csr_build(keys, keys, keys, 1, R1, R1, nfacts=nfacts)
    return g.rowptr_t, g.fact_t


def csr_relation_index(g, direction):
    """Relation index of one destination CSR of ``g`` ('fwd': tail CSR, 'inv': head CSR), built once and cached on
    the graph: (rix_ptr [R1+1], rix_slot = that CSR's slots sorted by (relation, slot), row_of = the row of every
    slot)."""
    if direction not in g.rel_index:
        rp, _src, rel, _fact = g.csr(direction)
        rix_ptr, rix_slot = _relation_index(rel[: g.F], g.R1, g.nfacts)
        row_of = torch.empty(max(pad4(g.F), 4), dtype=torch.int32, device=rp.device)
        _launch("gr_csr_row_of", _p(rp), g.B * g.N, _p(row_of))
        g.rel_index[direction] = (rix_ptr, rix_slot, row_of)
    return g.rel_index[direction]


def gather_f32(values, fact):
    values = _cuda(values, torch.float32, "values")
    F = values.numel()
    out = torch.empty(max(pad4(F), 4), dtype=torch.float32, device=values.device)
    _launch("gr_gather_f32", _p(values), _p(fact), _p(out), F)
    return out


def linear(A, W, bias=None, relu=False, out=None, addend=None, addend_rows=0, exact=False):
    """out[M,N] = act(A[M,K] @ W[N,K]^T + bias) (+ addend rows).  A/out may be strided row views."""
    A, W = _cuda(A, torch.float32, "A"), _cuda(W, torch.float32, "W")
    M, K = A.shape
    N = W.shape[0]
    assert W.shape[1] == K and A.stride(1) == 1 and W.stride(1) == 1
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32, device=A.device)
    assert out.shape == (M, N) and out.stride(1) == 1
    flags = (LINEAR_RELU if relu else 0) | (LINEAR_EXACT_FP32 if exact else 0)
    _launch("gr_linear", _p(A), A.stride(0), _p(W), W.stride(0), _p(bias), _p(addend),
            addend.stride(0) if addend is not None else 0, addend_rows, _p(out), out.stride(0), M, N, K, flags)
    return out


TC_LINEAR = True       # route the big e2e linears through the wgmma split-bf16 kernel (models use this)
TC_MAX_N = 256         # output columns of one wgmma GEMM launch (the register accumulator of a consumer warpgroup)
TC_MAX_N_SPLIT = 512   # wider outputs are tiled over N: one launch per <= 256-column slice of W


def tc_linear_ok(N, K):
    """True when ``TC_LINEAR`` is on and gr_linear_tc admits an [N, K] weight: 8 <= N <= 256, K >= 8."""
    return bool(TC_LINEAR) and 8 <= N <= TC_MAX_N and K >= 8


def tc_planes_ok(N, K):
    """True when ``TC_LINEAR`` is on and :func:`linear_tc_planes` takes an [N, K] weight: 8 <= N <= 512 (wider than
    256 through column slices), K >= 8."""
    return bool(TC_LINEAR) and 8 <= N <= TC_MAX_N_SPLIT and K >= 8


def linear_tc(A, W, bias=None, relu=False, out=None):
    """Tensor-core (wgmma, split-bf16 x3) version of :func:`linear` for the shapes :func:`tc_linear_ok` admits."""
    A, W = _cuda(A, torch.float32, "A"), _cuda(W, torch.float32, "W")
    M, K = A.shape
    N = W.shape[0]
    assert W.shape[1] == K and A.stride(1) == 1 and W.stride(1) == 1
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32, device=A.device)
    assert out.shape == (M, N) and out.stride(1) == 1
    ws, nbytes = _workspace(A.device, "gr_linear_tc_workspace_bytes", M, N, K)
    _launch("gr_linear_tc", _p(A), A.stride(0), _p(W), W.stride(0), _p(bias), _p(out), out.stride(0),
            M, N, K, LINEAR_RELU if relu else 0, _p(ws), nbytes, launches=3)
    return out


def rel_linear(A, W, bias=None, addend=None, addend_rows=0):
    """Hoisted relation projection table = A W^T + b (+ pos_emb rows): wgmma split-bf16 path when enabled
    (fp32-class accuracy, ~3x faster than the SIMT kernel at [6107 x 200 x 200]); the optional pos_emb addend
    keeps the exact SIMT kernel."""
    if addend is None and tc_linear_ok(*W.shape):
        return linear_tc(A, W, bias, relu=False)
    return linear(A, W, bias, addend=addend, addend_rows=addend_rows)


def e2e_linear(A, W, bias, out):
    """relu(A W^T + b) for the node-update GEMM: wgmma path when enabled and the shape fits."""
    if tc_linear_ok(*W.shape):
        return linear_tc(A, W, bias, relu=True, out=out)
    return linear(A, W, bias, relu=True, out=out)


def aggregate(g, direction, prior, table, ins, out=None, out_col0=0, seg_stride=None, w=None,
              possible=None, dtype=torch.float32):
    """One direction of the relation-typed aggregation.  direction: 'fwd' (tail CSR) | 'inv' (head CSR).
    prior [B,N]; table [R1,D]; ins [B,I,D]; out [B*N, >= out_col0 + I*seg_stride] row-major view, fp32 or bf16
    (``dtype`` when ``out`` is None): bf16 holds the fp32 result rounded to nearest even."""
    prior = _cuda(prior, torch.float32, "prior").contiguous()
    table = _cuda(table, torch.float32, "table").contiguous()
    ins = _cuda(ins, torch.float32, "ins").contiguous()
    B, I, D = ins.shape
    N = g.N
    if seg_stride is None:
        seg_stride = D
    if out is None:
        out = torch.empty(B * N, I * seg_stride + out_col0, dtype=dtype, device=prior.device)
    io = _node_io(out=out)
    assert out.stride(1) == 1
    rp, src, rel, _fact = g.csr(direction)
    _launch("gr_aggregate", _p(rp), _p(src), _p(rel), _p(w), _p(prior), _p(table), _p(ins), _p(out), out.stride(0),
            out_col0, seg_stride, _p(possible), B, N, D, I, g.F, io=io, launches=(I + 3) // 4, agg=("single", I))
    return out


def aggregate_backward_ok(D, I):
    """True when gr_aggregate_backward (and its _det form) admits width D and I instructions: 0 < D <= 256,
    0 < I <= 4."""
    return 0 < D <= 256 and 0 < I <= 4


def aggregate_backward(g, direction, prior, table, ins, grad_out, grad_table, grad_ins, grad_prior, w=None,
                       deterministic=False):
    """Accumulate the gradients of :func:`aggregate` (same ``direction`` / CSR) into grad_table [R1,D], grad_ins
    [B,I,D], grad_prior [B,N]; grad_out [B*N, I*D] contiguous rows, fp32 or bf16 (csrc/aggregate_bwd.cu).
    ``deterministic``: the fixed-order kernels (gr_aggregate_backward_det) instead of the fp32 atomics."""
    prior = _cuda(prior, torch.float32, "prior").contiguous()
    table = _cuda(table, torch.float32, "table").contiguous()
    ins = _cuda(ins, torch.float32, "ins").contiguous()
    io = _node_io(grad_out=grad_out)
    B, I, D = ins.shape
    assert grad_out.stride(1) == 1 and grad_table.is_contiguous() and grad_ins.is_contiguous() and grad_prior.is_contiguous()
    rp, src, rel, fact = g.csr(direction)
    if deterministic:
        assert grad_table.shape[0] >= g.R1
        rix_ptr, rix_slot, row_of = csr_relation_index(g, direction)
        rp_o, _src, _rel, fact_o = g.csr("inv" if direction == "fwd" else "fwd")
        ws, nbytes = _workspace(prior.device, "gr_aggregate_backward_det_workspace_bytes", B, g.N, D, I, g.F)
        _launch("gr_aggregate_backward_det", _p(rp), _p(src), _p(rel), _p(fact), _p(w), _p(prior), _p(table), _p(ins),
                _p(grad_out), grad_out.stride(0), 0, D, _p(grad_table), _p(grad_ins), _p(grad_prior), B, g.N, D, I,
                g.F, _p(rp_o), _p(fact_o), _p(rix_ptr), _p(rix_slot), _p(row_of), g.R1, _p(ws), nbytes, io=io,
                launches=5 if g.F > 0 else 0, op="aggregation_bwd_det")
        return
    _launch("gr_aggregate_backward", _p(rp), _p(src), _p(rel), _p(w), _p(prior), _p(table), _p(ins), _p(grad_out),
            grad_out.stride(0), 0, D, _p(grad_table), _p(grad_ins), _p(grad_prior), B, g.N, D, I, g.F, io=io,
            op="aggregation_bwd")


def aggregate_dual(g, prior, table_fwd, table_inv, ins, out, out_col0, w_t=None, w_h=None, planes=None,
                   seg_pitch=0):
    """Both directions of one ReaRev layer: out[:, out_col0 + (2j+dir)*D : +D] (reasongnn.py:150-161).
    ``planes`` = (hi, lo) bf16 [B*N, ld] tensors: write the split-bf16 A-operand planes (``out`` may be
    None)."""
    prior = _cuda(prior, torch.float32, "prior").contiguous()
    ins = _cuda(ins, torch.float32, "ins").contiguous()
    B, I, D = ins.shape
    assert table_fwd.is_contiguous() and table_inv.is_contiguous()
    assert out is None or out.stride(1) == 1
    hi, lo = planes if planes is not None else (None, None)
    _launch("gr_aggregate_dual", _p(g.rowptr_t), _p(g.src_t), _p(g.rel_t), _p(w_t),
            _p(g.rowptr_h), _p(g.src_h), _p(g.rel_h), _p(w_h),
            _p(prior), _p(table_fwd), _p(table_inv), _p(ins), _p(out),
            out.stride(0) if out is not None else 0, out_col0, seg_pitch,
            _p(hi), _p(lo), hi.stride(0) if hi is not None else 0,
            B, g.N, D, I, g.F, launches=(I + 3) // 4, agg=("dual", I))
    return out


AGG_ABS = True          # |v|-accumulating aggregation kernel (csrc/aggregate_abs.cu) for the shapes it specialises


def pad_table256(table):
    """[rows, D] fp32 relation table -> zero-padded [rows, 256] copy (1 KB rows: every lane of the gather is
    in-bounds) for :func:`aggregate_dual_abs`."""
    table = _cuda(table, torch.float32, "table")
    rows, D = table.shape
    assert table.stride(1) == 1
    pn = torch.empty(rows, 256, dtype=torch.float32, device=table.device)
    _launch("gr_pad_table256", _p(table), table.stride(0), rows, D, _p(pn), op="table_prep")
    return pn


def aggregate_dual_abs_supported(N, D, seg_pitch, R1):
    return bool(AGG_ABS) and bool(_L().gr_aggregate_dual_abs_supported(N, D, seg_pitch, R1))


_TILE_COUNTER = {}


def k_order_nb0(seg_pitch):
    """First column of the neighbour region of the K-order layout (:func:`aggregate_dual_abs` with ``k_order``)."""
    return (seg_pitch + 31) // 32 * 32


def aggregate_dual_abs(g, prior, pn_fwd, pn_inv, ins, planes, out_col0, seg_pitch, w_t=None, w_h=None, k_order=False):
    """Both directions of one ReaRev layer into the split-bf16 planes, |v|-accumulating kernel (reasongnn.py:150-161).
    ``k_order``: the 2I neighbour segments go to the K-order layout from ``out_col0`` on (GR_AGG_K_ORDER), the A operand
    :func:`linear_tc_planes` reads with ``k_order``."""
    prior = _cuda(prior, torch.float32, "prior").contiguous()
    ins = _cuda(ins, torch.float32, "ins").contiguous()
    B, I, D = ins.shape
    hi, lo = planes
    assert pn_fwd.is_contiguous() and pn_inv.is_contiguous() and hi.stride(0) == lo.stride(0)
    if ACT_BF16:
        lo = None
    dev = prior.device
    if dev not in _TILE_COUNTER:
        _TILE_COUNTER[dev] = torch.zeros(1, dtype=torch.int32, device=dev)
    _launch("gr_aggregate_dual_abs_ex", _p(g.rowptr_t), _p(g.src_t), _p(g.rel_t), _p(w_t),
            _p(g.rowptr_h), _p(g.src_h), _p(g.rel_h), _p(w_h),
            _p(prior), _p(pn_fwd), _p(pn_inv), pn_fwd.shape[0], _p(ins), _p(hi), _p(lo), hi.stride(0),
            out_col0, seg_pitch, B, g.N, D, I, g.F, _p(_TILE_COUNTER[dev]), AGG_K_ORDER if k_order else 0,
            launches=(I + 3) // 4, agg=("dual", I))


FUSED_LAYER = True      # dense-prior ReaRev layers run in grouped K order (the k-block order of csrc/fused_layer.cu)
# Which kernels run such a layer (ops.dense_layer).  gr_fused_layer issues an accumulator wider than 128 columns as
# 32-column wgmma instructions; for those widths (D = 200: 208 columns) the aggregation kernel followed by the full-width
# GEMM in the same K order gives the same bits faster (scripts/dense_layer_probe.py).  False: gr_fused_layer at every width.
DENSE_WIDE_AS_PAIR = True
FUSED_MIN_ROWS = 132 * 128   # below one 128-row tile per SM the fused kernel's serial per-tile chain (35 dependent k-blocks)
                             # loses to the two wide kernels


def fused_layer_supported(N, D, seg_pitch, I, n_out):
    return bool(_L().gr_fused_layer_supported(N, D, seg_pitch, I, n_out))


def fused_ell(g, w_t=None, w_h=None):
    """Quad-ELL form of the batch's CSRs for the fused layer kernel, built once per batch and cached on the graph
    (keyed on whether edge weights are used: they are part of the static entries)."""
    key = "_ell_w" if w_t is not None else "_ell"
    ell = getattr(g, key, None)
    if ell is None:
        ell, nbytes = _workspace(g.rowptr_t.device, "gr_fused_ell_bytes", g.B, g.N, g.F)
        _launch("gr_fused_ell_build", _p(g.rowptr_t), _p(g.src_t), _p(g.rel_t), _p(w_t),
                _p(g.rowptr_h), _p(g.src_h), _p(g.rel_h), _p(w_h), g.B, g.N, g.F, _p(ell), nbytes, op="csr_build")
        setattr(g, key, ell)
    return ell


def fused_layer(g, prior, pn_fwd, pn_inv, ins, h_planes, seg_pitch, W, bias, out=None, out_planes=None,
                w_score=None, dots=None, relu=True, w_t=None, w_h=None):
    """One dense-prior ReaRev layer in one kernel (reasongnn.py:134-165): both directions and all instructions are
    aggregated straight into the tensor-core operand stages of ``relu(e2e([h | nb...]))``.  ``h_planes`` = (hi, lo)
    bf16 planes whose first ``seg_pitch`` columns hold h; writes any of fp32 ``out``, ``out_planes``, ``dots``."""
    prior = _cuda(prior, torch.float32, "prior").contiguous()
    ins = _cuda(ins, torch.float32, "ins").contiguous()
    B, I, D = ins.shape
    hi, lo = h_planes
    n_out = W.shape[0]
    assert pn_fwd.is_contiguous() and pn_inv.is_contiguous() and hi.stride(0) == lo.stride(0)
    assert W.stride(1) == 1 and W.shape[1] == (2 * I + 1) * D
    nbytes = _L().gr_fused_layer_workspace_bytes(D, seg_pitch, I, n_out)
    ws, presplit = _weight_ws(W, n_out, W.shape[1], "fused", seg_pitch, nbytes)
    ell = fused_ell(g, w_t, w_h)
    chi, clo = out_planes if out_planes is not None else (None, None)
    flags = (LINEAR_RELU if relu else 0) | (LINEAR_W_PRESPLIT if presplit else 0)
    _launch("gr_fused_layer", _p(g.rowptr_t), _p(g.src_t), _p(g.rel_t), _p(w_t),
            _p(g.rowptr_h), _p(g.src_h), _p(g.rel_h), _p(w_h),
            _p(prior), _p(pn_fwd), _p(pn_inv), _p(ins), _p(hi), _p(lo), hi.stride(0), seg_pitch,
            _p(W), W.stride(0), _p(bias), _p(out), out.stride(0) if out is not None else 0,
            _p(chi), _p(clo), chi.stride(0) if chi is not None else 0, _p(w_score), _p(dots),
            B, g.N, D, I, n_out, g.F, flags, _p(ws), ws.numel(), _p(ell), ell.numel(),
            launches=2 if (w_t is not None or w_h is not None) else 1,     # weighted graphs: + the coefficient pass
            op="fused_layer")
    return out


def dense_layer(g, prior, pn_fwd, pn_inv, ins, planes, seg_pitch, W, bias, out=None, out_planes=None, w_score=None,
                dots=None, w_t=None, w_h=None, out_rows=None):
    """One dense-prior ReaRev layer in grouped K order: ``relu(e2e([h | nb...]))`` with the score dot.  ``planes`` =
    (hi, lo) layer-input planes [M, >= k_order_nb0(seg_pitch) + 2I * seg_pitch] whose first segment holds h.
    Accumulators of more than 128 columns run as :func:`aggregate_dual_abs` into the K-order neighbour region of
    ``planes`` + :func:`linear_tc_planes` walking it in grouped order, the others as :func:`fused_layer`; the outputs
    are the same bits either way.  ``out_rows`` (fp32 [M]): only the rows m of ``out`` with out_rows[m] != 0 need be
    written; the pair writes just those (:func:`linear_tc_planes`), the fused kernel every row."""
    I, n_out = ins.shape[1], W.shape[0]
    if DENSE_WIDE_AS_PAIR and (n_out + 15) // 16 * 16 > 128:
        aggregate_dual_abs(g, prior, pn_fwd, pn_inv, ins, planes, k_order_nb0(seg_pitch), seg_pitch, w_t, w_h,
                           k_order=True)
        return linear_tc_planes(planes[0], planes[1], (2 * I + 1) * seg_pitch, W, bias, out=out, out_planes=out_planes,
                                w_score=w_score, dots=dots, relu=True, k_seg=ins.shape[2], k_seg_pitch=seg_pitch,
                                k_grouped=True, k_order=True, **({} if out_rows is None else {"out_rows": out_rows}))
    return fused_layer(g, prior, pn_fwd, pn_inv, ins, planes, seg_pitch, W, bias, out=out, out_planes=out_planes,
                       w_score=w_score, dots=dots, relu=True, w_t=w_t, w_h=w_h)


def type_layer(g, table, out, w_t=None, w_h=None, planes=None):
    """out[:, :D] = relu(sum_tail w*table[rel] + sum_head w*table[rel]) (layer_init.py:46-57); optional
    split-bf16 planes of the same values.  ``out``: fp32, or bf16 (the fp32 values rounded to nearest even)."""
    table = _cuda(table, torch.float32, "table").contiguous()
    D = table.shape[1]
    io = _node_io(out=out)
    assert out is None or out.stride(1) == 1
    hi, lo = planes if planes is not None else (None, None)
    _launch("gr_type_layer", _p(g.rowptr_t), _p(g.rel_t), _p(w_t), _p(g.rowptr_h), _p(g.rel_h), _p(w_h), _p(table),
            _p(out), out.stride(0) if out is not None else 0, _p(hi), _p(lo), hi.stride(0) if hi is not None else 0,
            g.B, g.N, D, g.F, io=io, op="type_layer")
    return out


def split_bf16(A, hi, lo):
    """fp32 [M,K] -> bf16 hi/lo planes (first K columns of hi/lo)."""
    A = _cuda(A, torch.float32, "A")
    M, K = A.shape
    assert A.stride(1) == 1 and hi.stride(1) == 1 and hi.stride(0) == lo.stride(0)
    _launch("gr_split_bf16", _p(A), A.stride(0), M, K, _p(hi), _p(lo), hi.stride(0))


WEIGHT_CACHE = True    # keep pre-formatted weights (bf16 hi/lo splits) until their tensor version changes
_CACHE = {}            # key -> [buffers (tuple of tensors), owner version, weakref(owner tensor)]
_PRIVATE = None        # inside graph_private_weights: the buffers handed to the capture


@contextlib.contextmanager
def graph_private_weights():
    """A CUDA graph captured inside this context formats every weight it reads (the split-bf16 workspaces of the wgmma
    GEMM and the fused layer, :func:`param_planes`) into buffers of its own on every replay, instead of reading the
    cache's copies formatted at capture time.  Such a graph stays valid across in-place parameter updates
    (``optimizer.step()``, ``load_state_dict``) at the cost of those formatting kernels per replay.  Yields the list
    of those buffers: the graph's owner keeps it alive with the graph.  Nothing changes outside a capture."""
    global _PRIVATE
    prev, _PRIVATE = _PRIVATE, []
    try:
        yield _PRIVATE
    finally:
        _PRIVATE = prev


def _base(t):
    return t._base if t._base is not None else t


def _cached(key, owner, fits, make):
    """(buffers, current): device buffers pre-formatted from tensor ``owner`` (conversion runs once per VERSION, so an
    in-place update / load_state_dict re-formats on the next call).  The entry of ``key`` is reused while it belongs
    to the same ``owner`` object and ``fits(buffers)``; ``current`` says whether it still holds owner's ``_version``
    (False: the caller rewrites the buffers).  Otherwise ``make()`` gives new buffers.  While a CUDA graph is being
    captured nothing is inserted or refreshed: a stale or missing entry gets new buffers the cache does not keep.
    Inside :func:`graph_private_weights` a capture always gets new buffers with ``current`` False."""
    capturing = torch.cuda.is_current_stream_capturing()
    if capturing and _PRIVATE is not None:
        buffers = make()
        _PRIVATE.extend(buffers)
        return buffers, False
    ent = _CACHE.get(key) if WEIGHT_CACHE else None
    if ent is not None and ent[2]() is owner and fits(ent[0]):
        if ent[1] == owner._version:
            return ent[0], True
        if not capturing:
            ent[1] = owner._version
            return ent[0], False          # same buffers, re-formatted by the caller
    buffers = make()
    if WEIGHT_CACHE and not capturing:
        if len(_CACHE) > 512:            # models that were dropped: release the buffers of dead tensors
            for k in [k for k, e in _CACHE.items() if e[2]() is None]:
                del _CACHE[k]
        _CACHE[key] = [buffers, owner._version, weakref.ref(owner)]
    return buffers, False


def _weight_ws(W, N, K, k_seg, k_seg_pitch, nbytes):
    """Workspace holding W's split planes + whether it is still valid (weight pre-formatting)."""
    (ws,), presplit = _cached(("ws", W.data_ptr(), W.stride(0), N, K, k_seg, k_seg_pitch), _base(W),
                              lambda b: b[0].numel() >= nbytes,
                              lambda: (torch.empty(nbytes, dtype=torch.uint8, device=W.device),))
    return ws, presplit


def param_planes(P):
    """bf16 hi/lo planes [M, round_up(K, 64)] of a parameter matrix used as a GEMM A operand (relation embedding
    tables), cached per tensor version like the weight split."""
    M, K = P.shape
    Kp = (K + 63) // 64 * 64
    (hi, lo), current = _cached(("planes", P.data_ptr()), P, lambda b: b[0].shape[0] == M,
                                lambda: tuple(torch.zeros(M, Kp, dtype=torch.bfloat16, device=P.device)
                                              for _ in range(2)))
    if not current:
        split_bf16(P.detach(), hi, lo)
    return hi, lo


def clear_weight_cache():
    """Drop the cached pre-formatted weights.  Captured CUDA graphs keep their own references to the workspaces they
    read (:func:`live_weight_workspaces`), so clearing the cache never frees memory a graph replay still uses.
    Note: the cache is validated by ``tensor._version``; in-place writes through ``.data`` (``p.data.copy_``,
    ``p.data.mul_``) do not bump it -- call this function after such updates."""
    _CACHE.clear()


def live_weight_workspaces():
    """Strong references to every cached pre-formatted weight buffer (held by GraphedStep entries)."""
    return [t for e in _CACHE.values() for t in e[0]]


def linear_tc_planes(a_hi, a_lo, K, W, bias, out=None, out_planes=None, w_score=None, dots=None, relu=True,
                     k_seg=0, k_seg_pitch=0, single_ok=False, k_grouped=False, k_order=False, out_rows=None):
    """wgmma split-bf16 GEMM whose A operand already lives in bf16 hi/lo planes [M, >=K] (shapes:
    :func:`tc_planes_ok`).
    ``single_ok``: this call may run as ONE bf16 product when ``ACT_BF16`` is on (the node-update GEMMs; the small
    relation-table GEMMs always keep the three-product fp32-class path).
    Writes any of: fp32 ``out`` [M,N]; ``out_planes`` (hi, lo) [M, >=N] (next layer's h columns);
    ``dots`` [2*M] = the two column-half partial sums of out @ w_score.
    ``k_grouped``: walk the K segments column group by column group (GR_LINEAR_K_GROUPED): the accumulation order, the
    W planes and the cached workspace of :func:`fused_layer`; always the three-product path.
    ``k_order`` (with ``k_grouped``): the neighbour segments lie in the K-order layout of :func:`aggregate_dual_abs`
    (GR_LINEAR_K_ORDER_PLANES): the same k16 steps from aligned boxes, W packed to match under a cache key of its own.
    ``out_rows``: fp32 [M]; ``out`` then receives only the rows m with out_rows[m] != 0 and keeps its other rows
    (gr_linear_tc_planes_rows); the other outputs are unchanged by it.
    N > 256 (cfg5: entity_dim 400) is tiled over the output columns: one launch per slice of W rows."""
    N = W.shape[0]
    if N > TC_MAX_N:
        nsl = (N + TC_MAX_N - 1) // TC_MAX_N
        step = ((N + nsl - 1) // nsl + 15) // 16 * 16
        part = None
        for n0 in range(0, N, step):
            n1 = min(N, n0 + step)
            d = torch.empty_like(dots) if (dots is not None and n0 > 0) else dots
            linear_tc_planes(a_hi, a_lo, K, W[n0:n1], None if bias is None else bias[n0:n1],
                             out=None if out is None else out[:, n0:n1],
                             out_planes=None if out_planes is None else (out_planes[0][:, n0:n1], out_planes[1][:, n0:n1]),
                             w_score=None if w_score is None else w_score[n0:n1], dots=d, relu=relu, k_seg=k_seg,
                             k_seg_pitch=k_seg_pitch, single_ok=single_ok, k_grouped=k_grouped, k_order=k_order,
                             **({} if out_rows is None else {"out_rows": out_rows}))
            if dots is not None and n0 > 0:
                part = d if part is None else part + d
        if part is not None:
            dots += part
        return out
    M = a_hi.shape[0]
    assert a_hi.dtype == torch.bfloat16 and a_hi.stride(1) == 1 and a_hi.stride(0) == a_lo.stride(0)
    if k_seg and k_seg_pitch > k_seg:
        assert K % k_seg_pitch == 0 and W.shape[1] == K // k_seg_pitch * k_seg
    else:
        assert W.shape[1] == K
    assert W.stride(1) == 1
    assert k_grouped or not k_order
    if k_grouped:                   # fused_layer's W planes, under fused_layer's cache key (packed: a key of its own)
        nbytes = _L().gr_fused_layer_workspace_bytes(k_seg, k_seg_pitch, K // k_seg_pitch // 2, N)
        ws, presplit = _weight_ws(W, N, W.shape[1], "korder" if k_order else "fused", k_seg_pitch, nbytes)
    else:
        nbytes = _L().gr_linear_tc_planes_workspace_bytes(N, K)
        ws, presplit = _weight_ws(W, N, K, k_seg, k_seg_pitch, nbytes)
    chi, clo = out_planes if out_planes is not None else (None, None)
    if out_rows is not None:
        out_rows = _cuda(out_rows, torch.float32, "out_rows")
        if out is None or not out_rows.is_contiguous() or out_rows.numel() != M:
            raise ValueError("out_rows must be a contiguous fp32 [M] row predicate of out (M = %d)" % M)
    flags = (LINEAR_RELU if relu else 0) | (LINEAR_W_PRESPLIT if presplit else 0) | \
        (LINEAR_K_GROUPED if k_grouped else LINEAR_BF16_SINGLE if (ACT_BF16 and single_ok) else 0) | \
        (LINEAR_K_ORDER_PLANES if k_order else 0)
    _launch("gr_linear_tc_planes_rows", _p(a_hi), _p(a_lo), a_hi.stride(0), _p(W), W.stride(0), _p(bias),
            _p(out), out.stride(0) if out is not None else 0,
            _p(chi), _p(clo), chi.stride(0) if chi is not None else 0,
            _p(w_score), _p(dots), M, N, K, k_seg, k_seg_pitch, flags, _p(ws), nbytes, _p(out_rows),
            launches=1 if presplit else 2, op="gemm_tc", info=(M, N, K))
    return out


class RelFeatures:
    """Relation features (ReaRev.get_rel_feature / NSM.get_rel_feature) for all directions, stacked row-wise
    [n_dir * R1, D]: as split-bf16 planes (A operand of the per-layer relation-table GEMMs) and/or fp32."""

    _buf = {}

    def __init__(self, R1, D, n_dir, device, planes):
        self.R1, self.D, self.n_dir = R1, D, n_dir
        self.hi = self.lo = self.f32 = None
        if planes:
            Kp = (D + 63) // 64 * 64
            key = (str(device), n_dir * R1, Kp)
            if key not in RelFeatures._buf:
                RelFeatures._buf[key] = (torch.zeros(n_dir * R1, Kp, dtype=torch.bfloat16, device=device),
                                         torch.zeros(n_dir * R1, Kp, dtype=torch.bfloat16, device=device))
            self.hi, self.lo = RelFeatures._buf[key]
        else:
            self.f32 = torch.empty(n_dir * R1, D, dtype=torch.float32, device=device)

    def rows(self, d):
        return slice(d * self.R1, (d + 1) * self.R1)


def rel_features_from_embeddings(embs, W, bias):
    """relation_linear applied to the relation embedding table(s) (rearev.py:91-99 / nsm.py:97-104):
    one wgmma GEMM per direction straight into the stacked planes (no fp32 round trip)."""
    R1, K = embs[0].shape
    D = W.shape[0]
    planes = tc_planes_ok(D, K) and tc_planes_ok(D, D)
    rf = RelFeatures(R1, D, len(embs), W.device, planes)
    for d, E in enumerate(embs):
        if planes:
            ahi, alo = param_planes(E)
            linear_tc_planes(ahi, alo, K, W, bias, out_planes=(rf.hi[rf.rows(d)], rf.lo[rf.rows(d)]), relu=False)
        else:
            linear(E, W, bias, out=rf.f32[rf.rows(d)])
    return rf


def rel_features_from_tensors(feats):
    """Relation features computed elsewhere in fp32 (relation-text encoder, rearev.py:100-111)."""
    R1, D = feats[0].shape
    planes = tc_planes_ok(D, D)
    rf = RelFeatures(R1, D, len(feats), feats[0].device, planes)
    for d, f in enumerate(feats):
        if planes:
            split_bf16(f.contiguous(), rf.hi[rf.rows(d)], rf.lo[rf.rows(d)])
        else:
            rf.f32[rf.rows(d)].copy_(f)
    return rf


def rel_table(rf, W, bias, dirs=None, addends=None):
    """Hoisted relation projection table(s) = rel_features W^T + b for the stacked directions in ONE GEMM
    (reasongnn.py:79,105 / nsm_gnn.py:95 / layer_init.py:41 applied to R1 relation rows instead of F facts).
    Returns the list of per-direction [R1, D] tables.  ``addends``: optional per-direction pos_emb rows."""
    n = rf.n_dir if dirs is None else dirs
    rows = n * rf.R1
    out = torch.empty(rows, W.shape[0], dtype=torch.float32, device=W.device)
    if rf.hi is not None:
        linear_tc_planes(rf.hi[:rows], rf.lo[:rows], rf.D, W, bias, out=out, relu=False)
    else:
        linear(rf.f32[:rows], W, bias, out=out)
    tabs = [out[d * rf.R1:(d + 1) * rf.R1] for d in range(n)]
    if addends is not None:
        for t, a in zip(tabs, addends):
            if a is not None:
                t[: a.shape[0]] += a
    return tabs


SPARSE_PRIOR_FASTPATH = True   # first layer of every ReaRev iteration (seed prior): K=1-segment GEMM + frontier fix-up


def frontier_rows(g, prior, rows, count):
    """rows/count <- destination rows with at least one in-edge (either direction) from a node with prior != 0."""
    prior = _cuda(prior, torch.float32, "prior").contiguous()
    _launch("gr_frontier_rows", _p(g.rowptr_t), _p(g.src_t), _p(g.rowptr_h), _p(g.src_h), _p(prior), g.B * g.N,
            _p(rows), _p(count), op="frontier")


def frontier_fixup(g, prior, table_fwd, table_inv, ins, cur_planes, W, bias, w_score, nxt_planes, h32, dots,
                   rows, count, w_t=None, w_h=None):
    """Recompute the listed rows of one ReaRev layer in full (aggregation + e2e linear + relu + score dot)."""
    prior = _cuda(prior, torch.float32, "prior").contiguous()
    ins = _cuda(ins, torch.float32, "ins").contiguous()
    B, I, D = ins.shape
    chi, clo = cur_planes
    nhi, nlo = nxt_planes
    assert W.stride(1) == 1 and table_fwd.is_contiguous() and table_inv.is_contiguous()
    _launch("gr_frontier_fixup", _p(g.rowptr_t), _p(g.src_t), _p(g.rel_t), _p(w_t), _p(g.rowptr_h), _p(g.src_h),
            _p(g.rel_h), _p(w_h), _p(prior), _p(table_fwd), _p(table_inv), _p(ins),
            _p(chi), _p(clo), chi.stride(0), _p(W), W.stride(0), _p(bias), _p(w_score),
            _p(nhi), _p(nlo), nhi.stride(0), _p(h32), _p(dots), _p(rows), _p(count), B, g.N, D, I, op="frontier")


def masked_softmax(dots, b_score, mask, B, N):
    """dist[b,:] = softmax(dots[0,b,:] + dots[1,b,:] + b + (1-mask)*VERY_NEG)  (reasongnn.py:168-169);
    ``dots`` = the [2, B*N] partial score dots of :func:`linear_tc_planes`."""
    dist = torch.empty(B, N, dtype=torch.float32, device=dots.device)
    d = dots.view(2, -1)
    _launch("gr_masked_softmax", _p(d[0]), _p(d[1]), _p(b_score), _p(mask.contiguous()), _p(dist), B, N,
            op="softmax")
    return dist


def score_softmax(h, w_score, b_score, mask, B, N, logits_out=None):
    """h: [B*N, >=D] row view (stride(0) = ldh); returns dist [B,N]."""
    h = _cuda(h, torch.float32, "h")
    D = w_score.numel()
    assert h.stride(1) == 1
    dist = torch.empty(B, N, dtype=torch.float32, device=h.device)
    _launch("gr_score_softmax", _p(h), h.stride(0), _p(w_score.contiguous()), _p(b_score),
            _p(mask.contiguous()), _p(dist), _p(logits_out), B, N, D, launches=2)
    return dist


def seed_retrieve(seed_info, h, B, N, D):
    seed_info = _cuda(seed_info, torch.float32, "seed_info").contiguous()
    out = torch.empty(B, D, dtype=torch.float32, device=h.device)
    assert h.stride(1) == 1
    _launch("gr_seed_retrieve", _p(seed_info), _p(h), h.stride(0), _p(out), B, N, D)
    return out


def _ptr_array(tensors):
    for t in tensors:
        _cuda(t, torch.float32, "weight")
        assert t.is_contiguous()
    return (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def instructions_ok(Q, D, I):
    """True when gr_instructions (and its _train / _backward forms) admits Q tokens of width D and I instructions:
    I <= 8 and (Q D + (I + 7) D + 2 Q) floats of shared memory <= 200 KB."""
    return I <= 8 and (Q * D + (I + 7) * D + 2 * Q) * 4 <= 200 * 1024


def _ins_args(hidden, qnode, qtext, pad_id, Wq, bq, Wcq, bcq, wca, bca):
    hidden = _cuda(hidden, torch.float32, "hidden").contiguous()
    qnode = _cuda(qnode, torch.float32, "qnode").contiguous()
    qtext = _cuda(qtext, torch.int64, "qtext").contiguous()
    wca = wca.reshape(-1).contiguous()
    return (hidden, qnode, qtext, [_p(hidden), _p(qnode), _p(qtext), int(pad_id), _ptr_array(Wq), _ptr_array(bq),
                                   _p(Wcq.contiguous()), _p(bcq), _p(wca), _p(bca)])


def instructions(hidden, qnode, qtext, pad_id, Wq, bq, Wcq, bcq, wca, bca):
    """All ``num_ins`` instruction vectors of one question batch in one launch (base_encoder.py:73-114).
    hidden [B,Q,D], qnode [B,D], qtext int64 [B,Q]; Wq/bq: lists of question_linear_i weight/bias.
    Returns ins [B, I, D]."""
    hidden, _qn, _qt, args = _ins_args(hidden, qnode, qtext, pad_id, Wq, bq, Wcq, bcq, wca, bca)
    B, Q, D = hidden.shape
    I = len(Wq)
    out = torch.empty(B, I, D, dtype=torch.float32, device=hidden.device)
    _launch("gr_instructions", *args, _p(out), None, B, Q, D, I, op="question_side")
    return out


@functools.lru_cache(maxsize=None)
def _lstm_max_hidden():
    return int(_L().gr_lstm_max_hidden())


def lstm_ok(D):
    """True when gr_lstm_forward admits hidden size D: D <= gr_lstm_max_hidden()."""
    return D <= _lstm_max_hidden()


def lstm_forward(gates_x, W_hh, b_hh):
    """hidden [B,Q,D] of a one-layer LSTM with zero initial state, given gates_x = x W_ih^T + b_ih [B,Q,4D]
    (lstm_encoder.py:27-36); one launch for the whole sequence."""
    gates_x = _cuda(gates_x, torch.float32, "gates_x").contiguous()
    B, Q, G = gates_x.shape
    D = G // 4
    assert W_hh.shape == (4 * D, D) and W_hh.is_contiguous()
    hidden = torch.empty(B, Q, D, dtype=torch.float32, device=gates_x.device)
    _launch("gr_lstm_forward", _p(gates_x), _p(W_hh), _p(b_hh), _p(hidden), B, Q, D, op="question_side")
    return hidden


def query_reform_ok(D, I):
    """True when gr_query_reform (and its _ex / _backward forms) admits width D and I instructions: D <= 1024, I <= 8
    and (5 I + 1) D floats of shared memory <= 48 KB."""
    return D <= 1024 and I <= 8 and (5 * I + 1) * D * 4 <= 48 * 1024


def _reform_h(h):
    h = _cuda(h, name="h")
    assert h.stride(1) == 1 and h.dtype in (torch.float32, torch.bfloat16), (h.stride(), h.dtype)
    return h, IO_BF16 if h.dtype == torch.bfloat16 else 0


def query_reform(seed_info, h, ins, Wr, Wg, B, N, op="query_reform"):
    """ins_new[b,j] = Fusion_j(ins[b,j], seed_info[b] @ h[b]) for every instruction (query_update.py:6-44).  h is
    read in its own dtype: fp32, or bf16 under autocast (gr_query_reform_ex).  ``op``: the op class the call is
    timed under."""
    seed_info = _cuda(seed_info, torch.float32, "seed_info").contiguous()
    ins = _cuda(ins, torch.float32, "ins").contiguous()
    h, io = _reform_h(h)
    _, I, D = ins.shape
    out = torch.empty_like(ins)
    _launch("gr_query_reform", _p(seed_info), _p(h), h.stride(0), _p(ins), _ptr_array(Wr), _ptr_array(Wg),
            _p(out), None, B, N, D, I, io=io, op=op)
    return out


def instructions_train(hidden, qnode, qtext, pad_id, Wq, bq, Wcq, bcq, wca, bca, seed=None, p=0.0):
    """Training forward of :func:`instructions` with the three linear_drop sites drawn in the kernel
    (gr_instructions_train).  ``seed``: device int64 [1] (read when p > 0).  Returns (ins [B, I, D], attn [B, I, Q])."""
    hidden, _qn, _qt, args = _ins_args(hidden, qnode, qtext, pad_id, Wq, bq, Wcq, bcq, wca, bca)
    seed, p = _seed_p(seed, p)
    B, Q, D = hidden.shape
    I = len(Wq)
    out = torch.empty(B, I, D, dtype=torch.float32, device=hidden.device)
    attn = torch.empty(B, I, Q, dtype=torch.float32, device=hidden.device)
    _launch("gr_instructions_train", *args, _p(seed), p, _p(out), _p(attn), B, Q, D, I, op="question_train")
    return out, attn


def instructions_dropout_mask(seed, p, B, Q, D, I):
    """uint8 masks (1 = kept) of :func:`instructions_train`'s three dropout sites for 0 < p < 1:
    (qnode [B, I, D], cq_linear input [B, I, 4D], ca_linear input [B, I, Q, D])."""
    seed = _cuda(seed, torch.int64, "seed")
    m = [torch.empty(s, dtype=torch.uint8, device=seed.device) for s in ((B, I, D), (B, I, 4 * D), (B, I, Q, D))]
    _launch("gr_instructions_dropout_mask", _p(seed), float(p), B, Q, D, I, *(_p(t) for t in m))
    return m


def instructions_backward(hidden, qnode, qtext, pad_id, Wq, bq, Wcq, bcq, wca, bca, seed, p, ri, attn, grad_out):
    """Backward of :func:`instructions_train` (same inputs, seed and p; its outputs ri and attn) given
    grad_out = dL/dri [B, I, D] (gr_instructions_backward).  Returns grad_hidden [B, Q, D], grad_qnode [B, D] and the
    weight-gradient operands (g_q, x_q [B, I, D]; g_cq [B, I, D], x_cq [B, I, 4D]; g_ca [B, I, Q], x_ca [B, I, Q, D])."""
    hidden, _qn, _qt, args = _ins_args(hidden, qnode, qtext, pad_id, Wq, bq, Wcq, bcq, wca, bca)
    seed, p = _seed_p(seed, p)
    B, Q, D = hidden.shape
    I = len(Wq)
    ri = _cuda(ri, torch.float32, "ri").contiguous()
    attn = _cuda(attn, torch.float32, "attn").contiguous()
    grad_out = _cuda(grad_out, torch.float32, "grad_out").contiguous()
    e = lambda *s: torch.empty(s, dtype=torch.float32, device=hidden.device)   # noqa: E731
    outs = [e(B, Q, D), e(B, D), e(B, I, D), e(B, I, D), e(B, I, D), e(B, I, 4 * D), e(B, I, Q), e(B, I, Q, D)]
    _launch("gr_instructions_backward", *args, _p(seed), p, _p(ri), _p(attn), _p(grad_out), *(_p(t) for t in outs),
            B, Q, D, I, op="question_train")
    return outs


def query_reform_backward(seed_info, h, ins, Wr, Wg, B, N, grad_out, grad_h):
    """Backward of :func:`query_reform` (gr_query_reform_backward): adds s_n dL/dy to the seed rows of grad_h
    ([B*N, D], h's dtype; no other row is touched) and returns grad_ins [B, I, D] and the weight-gradient operands
    g_r, g_g [B, I, D] and z [B, I, 3D]."""
    seed_info = _cuda(seed_info, torch.float32, "seed_info").contiguous()
    ins = _cuda(ins, torch.float32, "ins").contiguous()
    h, io = _reform_h(h)
    grad_out = _cuda(grad_out, torch.float32, "grad_out").contiguous()
    assert grad_h.dtype == h.dtype and grad_h.stride(1) == 1 and grad_h.shape[0] == B * N
    _, I, D = ins.shape
    e = lambda *s: torch.empty(s, dtype=torch.float32, device=ins.device)   # noqa: E731
    outs = [e(B, I, D), e(B, I, D), e(B, I, D), e(B, I, 3 * D)]
    _launch("gr_query_reform_backward", _p(seed_info), _p(h), h.stride(0), _p(ins), _ptr_array(Wr), _ptr_array(Wg),
            _p(grad_out), _p(outs[0]), _p(grad_h), grad_h.stride(0), *(_p(t) for t in outs[1:]), B, N, D, I, io,
            op="question_train")
    return outs


def kl_loss_pred(dist, teacher):
    """-> (loss 0-dim fp32, pred int64[B]) : calc_loss_label('kl') with case_valid, and argmax (base_model.py:186)."""
    dist = _cuda(dist, torch.float32, "dist").contiguous()
    teacher = _cuda(teacher, torch.float32, "teacher").contiguous()
    B, N = dist.shape
    loss_q = torch.empty(B, dtype=torch.float32, device=dist.device)
    loss = torch.empty((), dtype=torch.float32, device=dist.device)
    pred = torch.empty(B, dtype=torch.int64, device=dist.device)
    _launch("gr_kl_loss_pred", _p(dist), _p(teacher), _p(loss_q), _p(loss), _p(pred), B, N, launches=2,
            op="loss_rank")
    return loss, pred


def rank_candidates_ok(B, N):
    """True when gr_rank_candidates admits B questions of N nodes: B > 0 and N > 0."""
    return B > 0 and N > 0


def rank_candidates(dist, local_entity, query_entities, pad_id, eps):
    """-> (cand_idx int32[B,N], cand_count int32[B], cand_total int32[B]) on device.  dist, local_entity and
    query_entities are all [B, N]: the kernel reads N entries of each per question."""
    if dist.dim() != 2 or not rank_candidates_ok(*dist.shape):
        raise RuntimeError("rank_candidates: dist must be [B, N] with B > 0 and N > 0, got %s" % list(dist.shape))
    for name, t in (("local_entity", local_entity), ("query_entities", query_entities)):
        if t.shape != dist.shape:
            raise RuntimeError("rank_candidates: %s must be %s like dist, got %s"
                               % (name, list(dist.shape), list(t.shape)))
    dist = _cuda(dist, torch.float32, "dist").contiguous()
    local_entity = _cuda(local_entity, torch.int64, "local_entity").contiguous()
    query_entities = _cuda(query_entities, torch.float32, "query_entities").contiguous()
    B, N = dist.shape
    dev = dist.device
    cand_idx = torch.empty(B, N, dtype=torch.int32, device=dev)
    cand_count = torch.empty(B, dtype=torch.int32, device=dev)
    cand_total = torch.empty(B, dtype=torch.int32, device=dev)
    ws, nbytes = _workspace(dev, "gr_rank_workspace_bytes", B, N)
    _launch("gr_rank_candidates", _p(dist), _p(local_entity), _p(query_entities), int(pad_id), float(eps),
            _p(cand_idx), _p(cand_count), _p(cand_total), B, N, _p(ws), nbytes, op="loss_rank")
    return cand_idx, cand_count, cand_total


def train_metrics_ok(B, N):
    """True when gr_train_metrics admits B questions of N nodes: B > 0 and N > 0."""
    return B > 0 and N > 0


def train_metrics(pred_dist, answer_dist, seed_dist, local_entity, cand_idx, cand_count, pad_id):
    """-> (h1, f1) fp32 [B] on the device: the train-time hit@1 and F1 of autograd_path.eval_metric
    (gr_train_metrics), with the candidates of :func:`rank_candidates` run on query_entities = (seed_dist > 0)."""
    f32 = lambda t, n: _cuda(t, torch.float32, n).contiguous()   # noqa: E731
    pred_dist, answer_dist, seed_dist = f32(pred_dist, "pred_dist"), f32(answer_dist, "answer_dist"), \
        f32(seed_dist, "seed_dist")
    local_entity = _cuda(local_entity, torch.int64, "local_entity").contiguous()
    cand_idx = _cuda(cand_idx, torch.int32, "cand_idx").contiguous()
    cand_count = _cuda(cand_count, torch.int32, "cand_count").contiguous()
    B, N = pred_dist.shape
    if not train_metrics_ok(B, N):
        raise RuntimeError("train_metrics: need B > 0 and N > 0, got B=%d N=%d" % (B, N))
    for name, t in (("answer_dist", answer_dist), ("seed_dist", seed_dist), ("local_entity", local_entity),
                    ("cand_idx", cand_idx)):
        if t.shape != (B, N):
            raise RuntimeError("train_metrics: %s must be [%d, %d], got %s" % (name, B, N, list(t.shape)))
    if cand_count.shape != (B,):
        raise RuntimeError("train_metrics: cand_count must be [%d], got %s" % (B, list(cand_count.shape)))
    h1 = torch.empty(B, dtype=torch.float32, device=pred_dist.device)
    f1 = torch.empty(B, dtype=torch.float32, device=pred_dist.device)
    _launch("gr_train_metrics", _p(pred_dist), _p(answer_dist), _p(seed_dist), _p(local_entity), int(pad_id),
            _p(cand_idx), _p(cand_count), _p(h1), _p(f1), B, N, op="loss_rank")
    return h1, f1


ADAM_ALIGNED16 = 1          # GR_ADAM_ALIGNED16: a tensor-table row whose pointers are all 16-byte aligned
ADAM_WEIGHT_DECAY = 1       # GR_ADAM_WEIGHT_DECAY: some row of the table has weight_decay != 0


@functools.lru_cache(maxsize=None)
def adam_chunk_elems():
    """Elements per chunk of :func:`clip_adam` (gr_adam_chunk_elems): a tensor of n elements takes ceil(n / E)."""
    return int(_L().gr_adam_chunk_elems())


def clip_adam(table, scalars, chunks, slots=None, max_norm=0.0, grad_norm=None, weight_decay=False):
    """clip_grad_norm_ + Adam.step() over a tensor list (gr_grad_sumsq, then gr_clip_adam; csrc/optim.cu).

    ``table`` int64 [T, 6], ``scalars`` fp32 [T, 8] and ``chunks`` int32 [C, 2] are device tensors laid out as the
    header says; ``slots`` float64 [C] turns clipping to ``max_norm`` on, and ``grad_norm`` (fp32, one element) then
    receives the total norm.  ``weight_decay``: some row has weight_decay != 0.  Nothing here waits on the host, so a
    CUDA graph can capture the two launches."""
    table = _cuda(table, torch.int64, "table")
    scalars = _cuda(scalars, torch.float32, "scalars")
    chunks = _cuda(chunks, torch.int32, "chunks")
    slots = _cuda(slots, torch.float64, "slots")
    grad_norm = _cuda(grad_norm, torch.float32, "grad_norm")
    T, C = table.shape[0], chunks.shape[0]
    assert table.shape == (T, 6) and scalars.shape == (T, 8) and chunks.shape == (C, 2)
    if slots is not None:
        assert slots.numel() >= C
        _launch("gr_grad_sumsq", _p(table), _p(chunks), C, _p(slots), op="optimizer")
    _launch("gr_clip_adam", _p(table), _p(scalars), _p(chunks), C, _p(slots), float(max_norm), _p(grad_norm),
            ADAM_WEIGHT_DECAY if weight_decay else 0, op="optimizer")


_INT32_MAX = 2 ** 31 - 1
_INDEX_BYTES = {torch.int32: 4, torch.int64: 8}


def split_assemble_ok(B, N, F, index_dtype):
    """True when gr_split_assemble admits a batch of B questions of N nodes and F facts: B > 0, N > 0, F >= 0, an
    int32 or int64 index dtype, and with int32 B*N and F within the int32 range."""
    if index_dtype not in _INDEX_BYTES or B <= 0 or N <= 0 or F < 0:
        return False
    return index_dtype == torch.int64 or (B * N <= _INT32_MAX and F <= _INT32_MAX)


def _split_out(out, F, index_dtype, dev):
    """The five [F] index outputs of a split assembly: the tensors of ``out`` (None entries are made here)."""
    out = [None] * 5 if out is None else list(out)
    for i, t in enumerate(out):
        if t is None:
            out[i] = torch.empty(F, dtype=index_dtype, device=dev)
        elif not (t.is_cuda and t.dtype == index_dtype and t.is_contiguous() and t.numel() == F):
            raise RuntimeError("split assembly: out[%d] must be a contiguous %s [%d] CUDA tensor" % (i, index_dtype, F))
    return out


def _split_order(fn, kept, order, B):
    """(kept, order) of an assembly through a fact order, checked: both or neither; kept int64 [B], order int32."""
    if (kept is None) != (order is None):
        raise RuntimeError("%s: kept and order come together, got only %s" % (fn, "order" if kept is None else "kept"))
    if kept is None:
        return None, None
    kept = _cuda(kept, torch.int64, "kept").contiguous()
    if kept.numel() != B:
        raise RuntimeError("%s: need kept [B], got B=%d kept %s" % (fn, B, list(kept.shape)))
    return kept, _cuda(order, torch.int32, "order").contiguous()


def split_assemble(q_off, q_heads, q_rels, q_tails, q_ents, ids, N, F, self_rel, use_self_loop, index_dtype, out=None,
                   kept=None, order=None):
    """-> (heads, rels, tails, batch_ids, fact_ids, status): the fact arrays of the questions ``ids`` (int64 [B] on the
    device) of a resident split (gr_split_assemble), each [F] in ``index_dtype``; ``status`` int32[1] on the device
    (bit 1: an id out of range, bit 2: more facts than F).  q_off int64 [num_q+1]; q_heads/q_rels/q_tails int32 (local
    ids, by question); q_ents int32 [num_q].  ``out``: optional five [F] tensors (None entries allocated) written in
    place of new ones.  ``kept`` (int64 [B]) and ``order`` (int32, :func:`split_fact_order`), given together: question
    b contributes the facts at the stored indices of its ``kept[b]`` entries of ``order``, then its self-loops
    (gr_split_assemble_ordered; an order entry that is not a stored index of its question also sets bit 1)."""
    q_off = _cuda(q_off, torch.int64, "q_off").contiguous()
    q_heads, q_rels, q_tails, q_ents = (_cuda(t, torch.int32, n).contiguous() for t, n in
                                        ((q_heads, "q_heads"), (q_rels, "q_rels"), (q_tails, "q_tails"),
                                         (q_ents, "q_ents")))
    ids = _cuda(ids, torch.int64, "ids").contiguous()
    B, num_q = ids.numel(), q_ents.numel()
    kept, order = _split_order("split_assemble", kept, order, B)
    if not split_assemble_ok(B, N, F, index_dtype):
        raise RuntimeError("split_assemble: need B > 0, N > 0, F >= 0 and an int32 / int64 index dtype whose range "
                           "holds B*N and F, got B=%d N=%d F=%d %s" % (B, N, F, index_dtype))
    dev = ids.device
    out = _split_out(out, F, index_dtype, dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    through = () if kept is None else (_p(kept), _p(order) if order.numel() else None, order.numel())
    _launch("gr_split_assemble" if kept is None else "gr_split_assemble_ordered", _p(q_off), _p(q_heads), _p(q_rels),
            _p(q_tails), _p(q_ents), num_q, _p(ids), *through, B, int(N), int(self_rel), int(bool(use_self_loop)),
            _INDEX_BYTES[index_dtype], int(F), *(_p(t) if F else None for t in out), _p(status), op="split_assemble")
    return (*out, status)


def split_assemble_graft_ok(B, max_facts, G, index_dtype):
    """True when gr_split_assemble_graft admits B questions, rows of max_facts and G graft entries: B > 0,
    max_facts >= 0, G >= 0, an int32 or int64 index dtype, and with int32 G and max_facts within the int32 range."""
    if index_dtype not in _INDEX_BYTES or B <= 0 or max_facts < 0 or G < 0:
        return False
    return index_dtype == torch.int64 or (G <= _INT32_MAX and max_facts <= _INT32_MAX)


def _graft_out(out, B, max_facts, G, index_dtype, dev):
    """(the six [G] index lists, the two fp32 [G] value lists, kb_fact_rel int64 [B, max_facts]) of a graft assembly:
    the tensors of ``out`` = ((e2f_b, e2f_f, e2f_e, e2f_v), (f2e_b, f2e_e, f2e_f, f2e_v), kb_fact_rel), checked, or
    new ones without it."""
    if out is None:
        idx = [torch.empty(G, dtype=index_dtype, device=dev) for _ in range(6)]
        vals = [torch.empty(G, dtype=torch.float32, device=dev) for _ in range(2)]
        return idx, vals, torch.empty(B, max_facts, dtype=torch.int64, device=dev)
    (e2f, f2e), kfr = out[:2], out[2]
    idx, vals = [*e2f[:3], *f2e[:3]], [e2f[3], f2e[3]]
    for i, t in enumerate(idx):
        if not (t.is_cuda and t.dtype == index_dtype and t.is_contiguous() and t.numel() == G):
            raise RuntimeError("split_assemble_graft: out index list %d must be a contiguous %s [%d] CUDA tensor"
                               % (i, index_dtype, G))
    for i, t in enumerate(vals):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == G):
            raise RuntimeError("split_assemble_graft: out value list %d must be a contiguous fp32 [%d] CUDA tensor"
                               % (i, G))
    if not (kfr.is_cuda and kfr.dtype == torch.int64 and kfr.is_contiguous() and tuple(kfr.shape) == (B, max_facts)):
        raise RuntimeError("split_assemble_graft: out kb_fact_rel must be a contiguous int64 [%d, %d] CUDA tensor"
                           % (B, max_facts))
    return idx, vals, kfr


def _graft_index_dtype(out, index_dtype):
    """The index dtype of a graft assembly: ``out``'s (its six index lists share one), else ``index_dtype``."""
    if out is None:
        return index_dtype
    dts = {t.dtype for t in (*out[0][:3], *out[1][:3])}
    if len(dts) != 1 or (index_dtype is not None and dts != {index_dtype}):
        raise RuntimeError("split_assemble_graft: the out index lists must share one dtype%s, got %s"
                           % ("" if index_dtype is None else " (%s)" % index_dtype, sorted(map(str, dts))))
    return dts.pop()


def split_assemble_graft(g_off, g_e2f_f, g_e2f_e, g_f2e_e, g_f2e_f, r_off, r_vals, ids, max_facts, rel_pad, G,
                         index_dtype=None, out=None, kept=None, order=None):
    """-> ((e2f_b, e2f_f, e2f_e, e2f_v), (f2e_b, f2e_e, f2e_f, f2e_v)), kb_fact_rel, status: the graft lists ([G], the
    index entries in ``index_dtype``, the values fp32 1.0) and kb_fact_rel int64 [B, max_facts] of the questions
    ``ids`` of a resident split (gr_split_assemble_graft); ``status`` as :func:`split_assemble`.  ``out``: optional
    tensors in the layout returned, ``((e2f_b, e2f_f, e2f_e, e2f_v), (f2e_b, f2e_e, f2e_f, f2e_v), kb_fact_rel)``,
    written in place of new ones; the index dtype is then theirs, and G their length (a capacity: the batch's entries
    fill the front, and entries past G are not written and set status bit 2).  ``kept`` / ``order`` as in
    :func:`split_assemble`: both graft lists take question b's entries at its ``kept[b]`` positions of ``order``
    (gr_split_assemble_graft_ordered); the kb_fact_rel rows are the stored ones."""
    g_off, r_off = _cuda(g_off, torch.int64, "g_off").contiguous(), _cuda(r_off, torch.int64, "r_off").contiguous()
    lists = [_cuda(t, torch.int32, n).contiguous() for t, n in
             ((g_e2f_f, "g_e2f_f"), (g_e2f_e, "g_e2f_e"), (g_f2e_e, "g_f2e_e"), (g_f2e_f, "g_f2e_f"),
              (r_vals, "r_vals"))]
    ids = _cuda(ids, torch.int64, "ids").contiguous()
    B, num_q = ids.numel(), g_off.numel() - 1
    kept, order = _split_order("split_assemble_graft", kept, order, B)
    index_dtype = _graft_index_dtype(out, index_dtype)
    if not split_assemble_graft_ok(B, max_facts, G, index_dtype):
        raise RuntimeError("split_assemble_graft: need B > 0, max_facts >= 0, G >= 0 and an int32 / int64 index dtype "
                           "whose range holds G and max_facts, got B=%d max_facts=%d G=%d %s"
                           % (B, max_facts, G, index_dtype))
    dev = ids.device
    idx, vals, kfr = _graft_out(out, B, max_facts, G, index_dtype, dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    p = (lambda t: _p(t) if t.numel() else None)     # noqa: E731
    through = () if kept is None else (_p(kept), p(order), order.numel())
    _launch("gr_split_assemble_graft" if kept is None else "gr_split_assemble_graft_ordered", _p(g_off),
            *(_p(t) for t in lists[:4]), _p(r_off), _p(lists[4]), num_q, _p(ids), *through, B, int(max_facts),
            int(rel_pad), _INDEX_BYTES[index_dtype], int(G), p(idx[0]), p(idx[1]), p(idx[2]), p(vals[0]), p(idx[3]),
            p(idx[4]), p(idx[5]), p(vals[1]), p(kfr), _p(status), op="split_assemble")
    return ((idx[0], idx[1], idx[2], vals[0]), (idx[3], idx[4], idx[5], vals[1])), kfr, status


def split_fact_order_ok(B, n_total, K):
    """True when gr_split_fact_order admits B questions holding n_total stored facts with K kept in all: B > 0,
    n_total >= 0 and 0 <= K <= 2^31 - 1."""
    return B > 0 and n_total >= 0 and 0 <= K <= _INT32_MAX


def split_fact_order(off, ids, kept, seed, perm, n_total, K):
    """-> (order, status): order int32 [K], per question of ``ids`` in batch order the stored indices of the first
    ``kept[b]`` facts of the question's permutation drawn from ``seed`` (gr_split_fact_order); ``status`` as
    :func:`split_assemble`.  off int64 [num_q+1] (q_off or g_off); ids, kept int64 [B]; seed int64 [1], all on the
    device; perm 0 (kb facts) or 1 (graft lists); n_total >= the stored facts of the B questions."""
    off = _cuda(off, torch.int64, "off").contiguous()
    ids, kept = _cuda(ids, torch.int64, "ids").contiguous(), _cuda(kept, torch.int64, "kept").contiguous()
    seed = _cuda(seed, torch.int64, "seed").contiguous()
    B, num_q = ids.numel(), off.numel() - 1
    if not split_fact_order_ok(B, n_total, K) or kept.numel() != B or seed.numel() != 1:
        raise RuntimeError("split_fact_order: need B > 0, kept [B], one seed, n_total >= 0 and 0 <= K <= 2^31 - 1, "
                           "got B=%d kept %s n_total=%d K=%d" % (B, list(kept.shape), n_total, K))
    dev = ids.device
    order = torch.empty(K, dtype=torch.int32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    ws, nbytes = _workspace(dev, "gr_split_fact_order_workspace_bytes", int(n_total))
    _launch("gr_split_fact_order", _p(off), num_q, _p(ids), _p(kept), B, _p(seed), int(perm), int(n_total), int(K),
            _p(order) if K else None, _p(status), _p(ws), nbytes, op="split_assemble")
    return order, status


def fact_weights_ok(F, Nt):
    """True when gr_fact_weights admits F facts over Nt node rows: 0 <= F <= 2^31 - 1 and 0 < Nt < 2^32."""
    return 0 <= F <= _INT32_MAX and 0 < Nt < 2 ** 32


def fact_weights(heads, rels, Nt, weight=True, weight_rel=True):
    """-> (weight_list, weight_rel_list, status): fp32 [F] 1/outdeg(head) and 1/count(head, rel) of a fact list
    (gr_fact_weights), each bit-equal to fp32 of the host's float64 value; None for an output not asked for.
    heads/rels: int32 or int64 [F] on the device, heads global rows in [0, Nt)."""
    heads, rels = _cuda(heads, name="heads").contiguous(), _cuda(rels, name="rels").contiguous()
    if heads.dtype not in _INDEX_BYTES or rels.dtype != heads.dtype:
        raise RuntimeError("fact_weights: heads and rels must share dtype int32 or int64")
    F = heads.numel()
    if not fact_weights_ok(F, Nt) or not (weight or weight_rel):
        raise RuntimeError("fact_weights: need 0 <= F <= 2^31 - 1, 0 < Nt < 2^32 and an output, got F=%d Nt=%d"
                           % (F, Nt))
    dev = heads.device
    w = torch.empty(F, dtype=torch.float32, device=dev) if weight else None
    wr = torch.empty(F, dtype=torch.float32, device=dev) if weight_rel else None
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    if F == 0:
        return w, wr, status
    ws, nbytes = _workspace(dev, "gr_fact_weights_workspace_bytes", F, Nt)
    _launch("gr_fact_weights", _p(heads), _p(rels), _INDEX_BYTES[heads.dtype], F, int(Nt), _p(w), _p(wr),
            _p(status), _p(ws), nbytes, launches=2, op="split_assemble")
    return w, wr, status


def fact_weights_live(heads, rels, nfacts, Nt, weight=None, weight_rel=None):
    """1/outdeg(head) into ``weight`` and 1/count(head, rel) into ``weight_rel`` (fp32, the capacity of ``heads``; either
    may be None, not both) over the live prefix of capacity-length fact buffers, ``nfacts`` (int32[1] on the device)
    long (gr_fact_weights_live): bit-equal there to :func:`fact_weights` of the prefix; entries past it are not
    written.  -> status int32[1] (as :func:`fact_weights`).  Shape rule: :func:`fact_weights_ok` of the capacity."""
    heads, rels = _cuda(heads, name="heads").contiguous(), _cuda(rels, name="rels").contiguous()
    nfacts = _cuda(nfacts, torch.int32, "nfacts")
    if heads.dtype not in _INDEX_BYTES or rels.dtype != heads.dtype:
        raise RuntimeError("fact_weights_live: heads and rels must share dtype int32 or int64")
    cap = heads.numel()
    for name, t in (("weight", weight), ("weight_rel", weight_rel)):
        if t is not None and not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == cap):
            raise RuntimeError("fact_weights_live: %s must be a contiguous fp32 [%d] CUDA tensor" % (name, cap))
    if not fact_weights_ok(cap, Nt) or (weight is None and weight_rel is None) or nfacts.numel() != 1:
        raise RuntimeError("fact_weights_live: need 0 <= capacity <= 2^31 - 1, 0 < Nt < 2^32, one nfacts and an "
                           "output, got capacity=%d Nt=%d" % (cap, Nt))
    status = torch.zeros(1, dtype=torch.int32, device=heads.device)
    if cap == 0:
        return status
    ws, nbytes = _workspace(heads.device, "gr_fact_weights_workspace_bytes", cap, Nt)
    _launch("gr_fact_weights_live", _p(heads), _p(rels), _INDEX_BYTES[heads.dtype], cap, _p(nfacts), int(Nt),
            _p(weight), _p(weight_rel), _p(status), _p(ws), nbytes, launches=2, op="split_assemble")
    return status


def epoch_step_begin(cursor, order, batch_size, kept_table, q_off, q_ents, use_self_loop, capacity, ids, rows, kept,
                     nfacts, kept_total, status):
    """The head of a graphed epoch step (gr_epoch_step_begin): from the device ``cursor`` (int64[1]) and the epoch's
    ``order`` (int64 [num_data]), the step's ``ids`` / ``rows`` / ``kept`` (int64 [B], B their length), ``nfacts``
    (int32[1]), ``kept_total`` (int64[1]) and ``status`` (int32[1]), all written in place.  ``kept_table``: int64
    [num_q] kept counts, or None for every stored fact."""
    B = ids.numel()
    for name, t, dt, n in (("cursor", cursor, torch.int64, 1), ("order", order, torch.int64, None),
                           ("kept_table", kept_table, torch.int64, None), ("q_off", q_off, torch.int64, None),
                           ("q_ents", q_ents, torch.int32, None), ("ids", ids, torch.int64, B),
                           ("rows", rows, torch.int64, B), ("kept", kept, torch.int64, B),
                           ("nfacts", nfacts, torch.int32, 1), ("kept_total", kept_total, torch.int64, 1),
                           ("status", status, torch.int32, 1)):
        if t is not None and (not t.is_contiguous() or (n is not None and t.numel() != n)):
            raise RuntimeError("epoch_step_begin: %s must be contiguous%s" % (name, "" if n is None else " [%d]" % n))
        _cuda(t, dt, name)
    _launch("gr_epoch_step_begin", _p(cursor), _p(order), order.numel(), int(batch_size), B, _p(kept_table),
            _p(q_off), _p(q_ents), q_ents.numel(), int(bool(use_self_loop)), int(capacity), _p(ids), _p(rows),
            _p(kept), _p(nfacts), _p(kept_total), _p(status), op="split_assemble")


def epoch_graft_begin(ids, kept_table, g_off, capacity, kept_g, graft_live, status):
    """GraftNet's half of the head of a graphed epoch step (gr_epoch_graft_begin), after :func:`epoch_step_begin` and
    from the ``ids`` (int64 [B]) it wrote: the graft kept counts ``kept_g`` (int64 [B]), ``graft_live`` (int32[2], both
    the live graft count clamped to ``capacity``) and ``status`` (int32[1]; bit 2: more entries than ``capacity``),
    all written in place.  ``kept_table``: int64 [num_q] kept counts, or None for every stored entry; ``g_off`` int64
    [num_q+1]."""
    B = ids.numel()
    for name, t, dt, n in (("ids", ids, torch.int64, B), ("kept_table", kept_table, torch.int64, None),
                           ("g_off", g_off, torch.int64, None), ("kept_g", kept_g, torch.int64, B),
                           ("graft_live", graft_live, torch.int32, 2), ("status", status, torch.int32, 1)):
        if t is not None and (not t.is_contiguous() or (n is not None and t.numel() != n)):
            raise RuntimeError("epoch_graft_begin: %s must be contiguous%s" % (name, "" if n is None else " [%d]" % n))
        _cuda(t, dt, name)
    _launch("gr_epoch_graft_begin", _p(ids), B, _p(kept_table), _p(g_off), g_off.numel() - 1, int(capacity),
            _p(kept_g), _p(graft_live), _p(status), op="split_assemble")


def epoch_step_record(cursor, batch_size, num_data, loss, grad_norm, seed, h1, f1, split_status, csr_status, losses,
                      grad_norms, seeds, h1_all, f1_all, epoch_status):
    """The tail of a graphed epoch step (gr_epoch_step_record): the step's fp32 ``loss``, ``grad_norm`` and int64
    ``seed`` (each one element; the last two optional, with their records ``grad_norms`` / ``seeds``) stored at the
    cursor, ``h1`` / ``f1`` (fp32 [B]) at its batch's positions of ``h1_all`` / ``f1_all`` (fp32 [num_data]), the int32
    status words OR-ed into ``epoch_status`` (int32[2]), the cursor advanced.  ``losses`` holds one entry per step."""
    for name, t, dt in (("cursor", cursor, torch.int64), ("loss", loss, torch.float32),
                        ("grad_norm", grad_norm, torch.float32), ("seed", seed, torch.int64),
                        ("h1", h1, torch.float32), ("f1", f1, torch.float32), ("split_status", split_status, torch.int32),
                        ("csr_status", csr_status, torch.int32), ("losses", losses, torch.float32),
                        ("grad_norms", grad_norms, torch.float32), ("seeds", seeds, torch.int64),
                        ("h1_all", h1_all, torch.float32), ("f1_all", f1_all, torch.float32),
                        ("epoch_status", epoch_status, torch.int32)):
        if t is not None and not t.is_contiguous():
            raise RuntimeError("epoch_step_record: %s must be contiguous" % name)
        _cuda(t, dt, name)
    B, steps = h1.numel(), losses.numel()
    if f1.numel() != B or h1_all.numel() != num_data or f1_all.numel() != num_data or epoch_status.numel() != 2:
        raise RuntimeError("epoch_step_record: need h1, f1 [B], h1_all, f1_all [num_data] and epoch_status [2]")
    _launch("gr_epoch_step_record", _p(cursor), steps, int(batch_size), B, int(num_data), _p(loss), _p(grad_norm),
            _p(seed), _p(h1), _p(f1), _p(split_status), _p(csr_status), _p(losses), _p(grad_norms), _p(seeds),
            _p(h1_all), _p(f1_all), _p(epoch_status), op="optimizer")


def eval_step_record(cursor, batch_size, steps, ids, local_entity, pred_dist, cand_idx, cand_count, a_off, a_ids, seed,
                     split_status, csr_status, metrics, cases, counts, cand_off, cand, cand_total, seeds, eval_status):
    """The tail of a graphed evaluation step (gr_eval_step_record): the evaluator's metrics of the step's questions
    (``ids`` int64 [B]; ``local_entity`` int64, ``pred_dist`` fp32, ``cand_idx`` int32 [B, N] and ``cand_count``
    int32 [B] of :func:`rank_candidates`) against their answers (``a_off`` int64 [num_a + 1], ``a_ids`` int64, each
    question's run ascending) stored at the cursor's positions of ``metrics`` (float64 [num_data, 5]), ``cases``
    (int8), ``counts`` (int32) and ``cand_off`` (int64, all [num_data]); the candidates appended to ``cand`` (int64
    [capacity, 2]) at ``cand_total`` (int64[1]); ``seed`` (int64[1] or None) at the cursor of ``seeds``; the status
    words OR-ed into ``eval_status`` (int32[3]); the cursor advanced.  See include/gnnrag_b200.h."""
    for name, t, dt in (("cursor", cursor, torch.int64), ("ids", ids, torch.int64),
                        ("local_entity", local_entity, torch.int64), ("pred_dist", pred_dist, torch.float32),
                        ("cand_idx", cand_idx, torch.int32), ("cand_count", cand_count, torch.int32),
                        ("a_off", a_off, torch.int64), ("a_ids", a_ids, torch.int64), ("seed", seed, torch.int64),
                        ("split_status", split_status, torch.int32), ("csr_status", csr_status, torch.int32),
                        ("metrics", metrics, torch.float64), ("cases", cases, torch.int8),
                        ("counts", counts, torch.int32), ("cand_off", cand_off, torch.int64),
                        ("cand", cand, torch.int64), ("cand_total", cand_total, torch.int64),
                        ("seeds", seeds, torch.int64), ("eval_status", eval_status, torch.int32)):
        if t is not None and not t.is_contiguous():
            raise RuntimeError("eval_step_record: %s must be contiguous" % name)
        _cuda(t, dt, name)
    B, N = local_entity.shape
    num_data = cases.numel()
    if (ids.numel() != B or pred_dist.shape != (B, N) or cand_idx.shape != (B, N) or cand_count.numel() != B
            or metrics.shape != (num_data, 5) or counts.numel() != num_data or cand_off.numel() != num_data
            or cand.dim() != 2 or cand.shape[1] != 2 or eval_status.numel() != 3):
        raise RuntimeError("eval_step_record: need ids, cand_count [B], pred_dist, cand_idx [B, N] like local_entity, "
                           "metrics [num_data, 5], counts, cand_off [num_data] like cases, cand [capacity, 2] and "
                           "eval_status [3]")
    _launch("gr_eval_step_record", _p(cursor), int(steps), int(batch_size), B, num_data, N, _p(ids),
            _p(local_entity), _p(pred_dist), _p(cand_idx), _p(cand_count), _p(a_off), _p(a_ids), a_off.numel() - 1,
            _p(seed), _p(split_status), _p(csr_status), _p(metrics), _p(cases), _p(counts), _p(cand_off), _p(cand),
            cand.shape[0], _p(cand_total), _p(seeds), _p(eval_status), op="loss_rank")


def eval_step_paths(cursor, batch_size, steps, num_data, g, query_entities, cand_idx, cand_count, S, T, node_off,
                    node_count, pair_dist, nodes, node_total, eval_status):
    """The shortest-path node sets of a graphed evaluation step (gr_eval_step_paths), before :func:`eval_step_record`
    moves the cursor: the sources of each question of the step are its local indices with ``query_entities`` (fp32
    [B, N]) nonzero, ascending, at most ``S``; its targets the first ``min(cand_count, T)`` of ``cand_idx`` (int32
    [B, N]); the BFS runs over the CsrGraph ``g``.  At the cursor's positions: ``node_off`` (int64 [num_data]),
    ``node_count`` (int32 [num_data]) and ``pair_dist`` (int32 [num_data, S, T]); the ascending on-path nodes appended
    to ``nodes`` (int32 [capacity]) at ``node_total`` (int64[1]), or none of the step's with bit 2 of ``eval_status``
    (int32[1]) set when they do not fit.  See include/gnnrag_b200.h."""
    for name, t, dt in (("cursor", cursor, torch.int64), ("query_entities", query_entities, torch.float32),
                        ("cand_idx", cand_idx, torch.int32), ("cand_count", cand_count, torch.int32),
                        ("node_off", node_off, torch.int64), ("node_count", node_count, torch.int32),
                        ("pair_dist", pair_dist, torch.int32), ("nodes", nodes, torch.int32),
                        ("node_total", node_total, torch.int64), ("eval_status", eval_status, torch.int32)):
        if not t.is_contiguous():
            raise RuntimeError("eval_step_paths: %s must be contiguous" % name)
        _cuda(t, dt, name)
    B, N = query_entities.shape
    if (cand_idx.shape != (B, N) or cand_count.numel() != B or node_off.numel() != num_data
            or node_count.numel() != num_data or pair_dist.shape != (num_data, S, T) or node_total.numel() != 1
            or eval_status.numel() != 1 or (g.B, g.N) != (B, N)):
        raise RuntimeError("eval_step_paths: need cand_idx [B, N] like query_entities and the graph's B, N, cand_count "
                           "[B], node_off, node_count [num_data], pair_dist [num_data, S, T], node_total and "
                           "eval_status [1]")
    ws, nbytes = _workspace(cursor.device, "gr_eval_paths_workspace_bytes", B, N, int(S), int(T))
    _launch("gr_eval_step_paths", _p(cursor), int(steps), int(batch_size), B, int(num_data), N, _p(query_entities),
            _p(cand_idx), _p(cand_count), int(S), int(T), _p(g.rowptr_t), _p(g.src_t), _p(g.rowptr_h), _p(g.src_h),
            _p(node_off), _p(node_count), _p(pair_dist), _p(nodes), nodes.numel(), _p(node_total), _p(eval_status),
            _p(ws), nbytes, launches=5, op="paths")


def _info_rows_args(name, metrics, cases, counts, cand_off, cand_total, cand, order, tables):
    """The checked record and table arguments of the two ``.info`` row entry points."""
    for arg, t, dt in (("metrics", metrics, torch.float64), ("cases", cases, torch.int8), ("counts", counts, torch.int32),
                       ("cand_off", cand_off, torch.int64), ("cand_total", cand_total, torch.int64),
                       ("cand", cand, torch.int64), ("order", order, torch.int64),
                       ("prefix", tables.prefix, torch.uint8), ("prefix_off", tables.prefix_off, torch.int64),
                       ("name_slot", tables.name_slot, torch.int32), ("names", tables.names, torch.uint8),
                       ("name_off", tables.name_off, torch.int64)):
        if not t.is_contiguous():
            raise RuntimeError("%s: %s must be contiguous" % (name, arg))
        _cuda(t, dt, arg)
    n = cases.numel()
    if (metrics.shape != (n, 5) or counts.numel() != n or cand_off.numel() != n or order.numel() != n
            or cand_total.numel() != 1 or cand.dim() != 2 or cand.shape[1] != 2):
        raise RuntimeError("%s: need metrics [num_data, 5], counts, cand_off, order [num_data] like cases, cand_total "
                           "[1] and cand [capacity, 2]" % name)
    return n, (tables.prefix_off.numel() - 1, tables.name_slot.numel(), tables.name_off.numel() - 1)


def info_rows_size(metrics, cases, counts, cand_off, cand_total, eval_status, cand, order, tables, row_off, summary):
    """Sizes of the ``.info`` rows of an evaluation's records (gr_info_rows_size): ``row_off`` (int64 [num_data + 1])
    receives the rows' byte offsets and ``summary`` (int64[2]) the total and the flags.  The records are
    gr_eval_step_record's (``metrics`` float64 [num_data, 5], ``cases`` int8, ``counts`` int32, ``cand_off`` int64
    [num_data], ``cand_total`` int64[1], ``eval_status`` int32[4], ``cand`` int64 [capacity, 2]); ``order``: the
    question id of each position; ``tables``: an ``evaluate.InfoTables``.  See include/gnnrag_b200.h."""
    n, (num_q, num_entity, num_names) = _info_rows_args("info_rows_size", metrics, cases, counts, cand_off, cand_total,
                                                        cand, order, tables)
    for arg, t, dt in (("eval_status", eval_status, torch.int32), ("row_off", row_off, torch.int64),
                       ("summary", summary, torch.int64)):
        if not t.is_contiguous():
            raise RuntimeError("info_rows_size: %s must be contiguous" % arg)
        _cuda(t, dt, arg)
    if eval_status.numel() != 4 or row_off.numel() != n + 1 or summary.numel() != 2:
        raise RuntimeError("info_rows_size: need eval_status [4], row_off [num_data + 1] and summary [2]")
    _launch("gr_info_rows_size", _p(metrics), _p(cases), _p(counts), _p(cand_off), _p(cand_total), _p(eval_status), n,
            _p(cand), cand.shape[0], _p(order), _p(tables.prefix_off), num_q, _p(tables.name_slot), num_entity,
            _p(tables.name_off), num_names, _p(row_off), _p(summary), launches=2, op="info_rows")


def info_rows_write(metrics, cases, counts, cand_off, cand_total, cand, order, tables, row_off, summary, out):
    """The ``.info`` rows of an evaluation's records into ``out`` (uint8, at least ``summary[0]`` bytes) at the
    offsets :func:`info_rows_size` wrote into ``row_off`` (gr_info_rows_write); nothing when ``summary`` holds
    flags.  Same records and tables as :func:`info_rows_size`."""
    n, (num_q, num_entity, num_names) = _info_rows_args("info_rows_write", metrics, cases, counts, cand_off, cand_total,
                                                        cand, order, tables)
    for arg, t, dt in (("row_off", row_off, torch.int64), ("summary", summary, torch.int64), ("out", out, torch.uint8)):
        if not t.is_contiguous():
            raise RuntimeError("info_rows_write: %s must be contiguous" % arg)
        _cuda(t, dt, arg)
    if row_off.numel() != n + 1 or summary.numel() != 2:
        raise RuntimeError("info_rows_write: need row_off [num_data + 1] and summary [2]")
    _launch("gr_info_rows_write", _p(metrics), _p(cases), _p(counts), _p(cand_off), _p(cand_total), n, _p(cand),
            cand.shape[0], _p(order), _p(tables.prefix), _p(tables.prefix_off), num_q, _p(tables.name_slot),
            num_entity, _p(tables.names), _p(tables.name_off), num_names, _p(row_off), _p(summary), _p(out),
            out.numel(), op="info_rows")


def shortest_path_nodes(g, source_idx, source_cnt, target_idx, target_cnt, return_distances=False):
    """source_idx int32[B,S], target_idx int32[B,T] local indices (+counts) ->
    (on_path uint8[B,N], pair_dist int32[B,S,T]); with ``return_distances`` also the BFS distance arrays the kernel
    leaves in its workspace: int32 [B, S+T, N] (sources first), -1 = unreachable."""
    B, N = g.B, g.N
    S, T = source_idx.shape[1], target_idx.shape[1]
    dev = source_idx.device
    on_path = torch.empty(B, N, dtype=torch.uint8, device=dev)
    pair_dist = torch.empty(B, S, T, dtype=torch.int32, device=dev)
    ws, nbytes = _workspace(dev, "gr_paths_workspace_bytes", B, N, S, T)
    _launch("gr_shortest_path_nodes", _p(g.rowptr_t), _p(g.src_t), _p(g.rowptr_h), _p(g.src_h),
            _p(source_idx.contiguous()), _p(source_cnt.contiguous()), S,
            _p(target_idx.contiguous()), _p(target_cnt.contiguous()), T,
            _p(on_path), _p(pair_dist), B, N, _p(ws), nbytes, launches=0, op="paths")
    if return_distances:
        return on_path, pair_dist, ws[: B * (S + T) * N * 4].view(torch.int32).view(B, S + T, N)
    return on_path, pair_dist


class RuleAdjacency:
    """Label-grouped undirected adjacency (gr_rule_adj_build): row u = [rowptr[u], rowptr[u] + len[u]) of nbr / lab,
    sorted by (label, first fact) -- every label's neighbours form one segment in nx.Graph neighbour order."""

    def __init__(self, rowptr, length, nbr, lab):
        self.rowptr, self.len, self.nbr, self.lab = rowptr, length, nbr, lab


def rule_adjacency(g):
    """CsrGraph built with rels = per-triple label ids -> RuleAdjacency (global node ids, like the CSR)."""
    Nt, F = g.B * g.N, g.F
    dev = g.rowptr_t.device
    i32 = dict(dtype=torch.int32, device=dev)
    adj = RuleAdjacency(torch.empty(Nt + 1, **i32), torch.empty(Nt, **i32), torch.empty(max(2 * F, 1), **i32),
                        torch.empty(max(2 * F, 1), **i32))
    ws, nbytes = _workspace(dev, "gr_rule_adj_workspace_bytes", F)
    _launch("gr_rule_adj_build", _p(g.rowptr_t), _p(g.src_t), _p(g.rel_t), _p(g.fact_t), _p(g.rowptr_h), _p(g.src_h),
            _p(g.rel_h), _p(g.fact_h), Nt, F, _p(adj.rowptr), _p(adj.len), _p(adj.nbr), _p(adj.lab), _p(ws), nbytes,
            launches=2, op="rule_paths")
    return adj


def rule_walks(adj, start, rule_off, rule_len, rule_lab):
    """All rule walks of J jobs (gr_rule_level_count / _emit per level, then gr_rule_paths_write).
    Host numpy int32 inputs: start[J] (node id, -1 = not in the graph), rule_off[J] / rule_len[J] into rule_lab
    (label ids, -1 = absent label).  Returns (paths, counts, elem_off): paths = int32 device tensor holding, for job j,
    counts[j] rows of rule_len[j] + 1 node ids from elem_off[j] on (host int64 arrays)."""
    with _Timer("rule_paths"):
        return _rule_walks(adj, start, rule_off, rule_len, rule_lab)


def _rule_walks(adj, start, rule_off, rule_len, rule_lab):
    dev = adj.nbr.device
    J = len(start)
    start, rule_len = np.asarray(start, np.int32), np.asarray(rule_len, np.int32)
    i32 = dict(dtype=torch.int32, device=dev)
    keep = np.nonzero((rule_len == 0) | (start >= 0))[0]
    node = torch.from_numpy(start[keep]).to(dev)
    job = torch.from_numpy(keep.astype(np.int32)).to(dev)
    d_off = torch.from_numpy(np.asarray(rule_off, np.int32)).to(dev)
    d_len = torch.from_numpy(rule_len).to(dev)
    d_lab = torch.from_numpy(np.append(np.asarray(rule_lab, np.int32), np.int32(-1))).to(dev)
    res_begin = torch.zeros(max(J, 1), **i32)
    res_count = torch.zeros(max(J, 1), **i32)
    levels_node, levels_parent = [node], [torch.full_like(node, -1)]
    for level in range(int(rule_len.max()) + 1 if J else 0):
        n = node.numel()
        seg = torch.empty(max(n, 1), **i32)
        off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        ws, nbytes = _workspace(dev, "gr_rule_level_workspace_bytes", n)
        _launch("gr_rule_level_count", _p(adj.rowptr), _p(adj.len), _p(adj.lab), _p(d_off), _p(d_len), _p(d_lab),
                J, level, _p(node), _p(job), n, _p(seg), _p(off), _p(res_begin), _p(res_count), _p(ws), nbytes,
                launches=0)
        if level == rule_len.max():
            break
        total = int(off[n].item())              # the one read-back per level: the next level is allocated exactly
        fits = total <= 0x7fffffff              # a level that int32 cannot index is refused by gr_rule_level_emit
        nxt = [torch.empty(max(total if fits else 0, 1), **i32) for _ in range(3)]
        _launch("gr_rule_level_emit", _p(adj.nbr), _p(job), _p(seg), _p(off), n, total, _p(nxt[0]), _p(nxt[1]),
                _p(nxt[2]), launches=0)
        node, job = nxt[0][:total], nxt[2][:total]
        levels_node.append(node)
        levels_parent.append(nxt[1][:total])
    counts = res_count[:J].cpu().numpy().astype(np.int64)
    path_off = np.zeros(J + 1, dtype=np.int64)
    np.cumsum(counts, out=path_off[1:])
    elems = counts * (rule_len.astype(np.int64) + 1)
    elem_off = np.zeros(J + 1, dtype=np.int64)
    np.cumsum(elems, out=elem_off[1:])
    paths = torch.empty(max(int(elem_off[-1]), 1), **i32)
    if path_off[-1] > 0:
        lv_node = torch.tensor([t.data_ptr() for t in levels_node], dtype=torch.int64, device=dev)
        lv_parent = torch.tensor([t.data_ptr() for t in levels_parent], dtype=torch.int64, device=dev)
        d_path_off, d_elem_off = torch.from_numpy(path_off).to(dev), torch.from_numpy(elem_off).to(dev)
        _launch("gr_rule_paths_write", _p(lv_node), _p(lv_parent), _p(d_len), _p(res_begin), _p(d_path_off),
                _p(d_elem_off), J, int(path_off[-1]), _p(paths), launches=0)
    return paths[: int(elem_off[-1])], counts, elem_off[:J]


class GraftGraph:
    """The graft facts of one batch (kb_adj_mat_graft, gnn/dataset_load_graft.py:70-102) staged on the device: facts
    paired by slot and ordered by (b, f), their CSRs (``graph``: tail CSR = in-facts of every node, head CSR =
    out-facts), ``slot_of`` = b*max_fact + f of each staged fact, and ``kb_fact_rel`` int64 [B, max_fact]."""

    def __init__(self, B, N, max_fact, cap, device):
        self.B, self.N, self.max_fact, self.cap = B, N, max_fact, cap
        i32 = dict(dtype=torch.int32, device=device)
        Fp = max(pad4(cap), 4)
        self.heads, self.rels, self.tails, self.slot_of = (torch.empty(Fp, **i32) for _ in range(4))
        self.nfacts = torch.zeros(1, **i32)
        self.status = torch.zeros(1, **i32)
        self.graph = None
        self.kb_fact_rel = None
        self.rel_index = {}      # (kind, R1) -> relation index of the staged facts / of all slots (deterministic backward)

    def fact_relation_index(self, R1):
        """(rix_ptr, rix_fact): the staged facts grouped by relation, in slot order inside each relation."""
        if ("facts", R1) not in self.rel_index:
            self.rel_index[("facts", R1)] = _relation_index(self.rels[: self.cap], R1, self.nfacts)
        return self.rel_index[("facts", R1)]

    def slot_relation_index(self, R1):
        """(rix_ptr, rix_slot): all B*max_fact slots grouped by relation (ids outside [0, R1) read as 0, as the
        attention kernels read them), in slot order inside each relation."""
        if ("slots", R1) not in self.rel_index:
            r = self.kb_fact_rel.reshape(-1)
            r = torch.where((r < 0) | (r >= R1), torch.zeros_like(r), r)
            self.rel_index[("slots", R1)] = _relation_index(r, R1)
        return self.rel_index[("slots", R1)]

    _MESSAGES = {1: "a batch, fact-slot or node id outside the batch", 2: "a relation id outside the relation table",
                 4: "a fact slot listed twice", 8: "a fact slot with a head but no tail (or a tail but no head)"}

    @classmethod
    def raise_status(cls, st):
        """Raise for a non-zero staging status word ``st`` (an int read back from ``status``)."""
        if st:
            why = "; ".join(m for bit, m in sorted(cls._MESSAGES.items()) if st & bit)
            raise RuntimeError("graft fact lists rejected: %s (offending entries were dropped or clamped)" % why)

    def check_status(self):
        self.raise_status(int(self.status.item()))
        self.graph.check_status()


def _i64(x, name):
    x = _cuda(x, torch.int64, name)
    return x.contiguous()


def graft_stage(e2f, f2e, kb_fact_rel, B, N, R1, live=None):
    """e2f = (b, f, head), f2e = (b, tail, f): int64 CUDA tensors of kb_adj_mat_graft (the 1.0 values are not needed);
    kb_fact_rel int64 [B, max_fact] -> GraftGraph (gr_graft_stage, then gr_csr_build over the staged facts).
    ``live``: optional int32[2] device tensor with the live entries of the head and the tail list when the lists are
    fixed-capacity buffers (GraphedStep); only those front parts are staged."""
    e2f = [_i64(t, "e2f") for t in e2f]
    f2e = [_i64(t, "f2e") for t in f2e]
    kb_fact_rel = _i64(kb_fact_rel, "kb_fact_rel")
    if live is not None:
        live = _cuda(live, torch.int32, "live")
        assert live.numel() >= 2 and live.is_contiguous()
    max_fact = kb_fact_rel.shape[1] if kb_fact_rel.dim() == 2 else 0
    assert kb_fact_rel.shape[0] == B
    F0, F1 = e2f[0].numel(), f2e[0].numel()
    assert all(t.numel() == F0 for t in e2f) and all(t.numel() == F1 for t in f2e)
    dev = kb_fact_rel.device
    gg = GraftGraph(B, N, max_fact, F0, dev)
    gg.kb_fact_rel = kb_fact_rel
    ws, nbytes = _workspace(dev, "gr_graft_stage_workspace_bytes", B, max_fact)
    _launch("gr_graft_stage", _p(e2f[0]), _p(e2f[1]), _p(e2f[2]), F0, _p(f2e[0]), _p(f2e[1]), _p(f2e[2]), F1,
            _p(kb_fact_rel), B, N, max_fact, R1, _p(gg.heads), _p(gg.rels), _p(gg.tails),
            _p(gg.slot_of), _p(gg.nfacts), _p(gg.status), _p(live), _p(ws), nbytes, launches=5, op="csr_build")
    gg.graph = csr_build(gg.heads[:F0], gg.rels[:F0], gg.tails[:F0], B, N, R1, nfacts=gg.nfacts)
    return gg


def graft_attention(gg, qh, qmask, rel, out_w=False):
    """Fact attention of GraftLayer.compute_attention (graft_gnn.py:64-87) -> (W or None, W~ [B, max_fact], E [B*N]).
    qh [B,Q,D], qmask float [B,Q], rel [R1, D] (row view allowed)."""
    qh = _cuda(qh, torch.float32, "qh").contiguous()
    qmask = _cuda(qmask, torch.float32, "qmask").contiguous()
    rel = _cuda(rel, torch.float32, "rel")
    assert rel.stride(1) == 1
    B, Q, D = qh.shape
    dev = qh.device
    S = B * gg.max_fact
    W = torch.empty(max(S, 1), dtype=torch.float32, device=dev)
    Wt = torch.empty(max(S, 1), dtype=torch.float32, device=dev)
    E = torch.empty(B * gg.N, dtype=torch.float32, device=dev)
    g = gg.graph
    _launch("gr_graft_attention", _p(qh), _p(qmask), Q, _p(rel), rel.stride(0), rel.shape[0], _p(gg.kb_fact_rel),
            B, gg.max_fact, D, _p(g.rowptr_h), _p(g.fact_h), _p(gg.slot_of), gg.N, _p(W), _p(Wt), _p(E),
            _p(gg.status), launches=3 if S > 0 else 1, op="graft_attention")
    return (W[:S] if out_w else None), Wt[:S], E


def graft_aggregate(gg, Wt, E, prior, self_tab, head_tab, lam, q2e=None, sum_out=None, planes=None, col_sum=0,
                    col_indeg=0, col_q2e=0, indeg_out=None, prior_next=None):
    """Fact side of one GraftLayer layer (graft_gnn.py:89-107, gr_graft_aggregate): returns prior_next [B, N] and
    writes the per-row sum of v_f (fp32 ``sum_out`` and/or the split-bf16 ``planes`` at ``col_sum``), the in-degree and
    the question vector ``q2e`` [B, D] into the planes."""
    g = gg.graph
    B, N = gg.B, gg.N
    prior = _cuda(prior, torch.float32, "prior").contiguous()
    self_tab = _cuda(self_tab, torch.float32, "self_tab")
    head_tab = _cuda(head_tab, torch.float32, "head_tab")
    D = self_tab.shape[1]
    assert self_tab.stride(1) == 1 and head_tab.stride(1) == 1 and head_tab.shape[0] == B * N
    if prior_next is None:
        prior_next = torch.empty(B, N, dtype=torch.float32, device=prior.device)
    if sum_out is not None:
        assert sum_out.stride(1) == 1
    if q2e is not None:
        q2e = _cuda(q2e, torch.float32, "q2e").contiguous()
    hi, lo = planes if planes is not None else (None, None)
    _launch("gr_graft_aggregate", _p(g.rowptr_t), _p(g.src_t), _p(g.rel_t), _p(g.fact_t), _p(gg.slot_of),
            _p(Wt), _p(E), _p(prior), _p(self_tab), self_tab.stride(0), _p(head_tab),
            head_tab.stride(0), _p(q2e), float(lam), _p(sum_out),
            sum_out.stride(0) if sum_out is not None else 0, _p(hi), _p(lo),
            hi.stride(0) if hi is not None else 0, col_sum, col_indeg, col_q2e,
            _p(indeg_out), _p(prior_next), B, N, D, agg=("graft", 1))
    return prior_next


def _seed_p(seed, p):
    """(seed pointer or None, p) of the dropout arguments: p == 0 takes the no-dropout path and ignores the seed."""
    p = float(p)
    if p == 0.0:
        return None, 0.0
    seed = _cuda(seed, torch.int64, "seed")
    assert seed.numel() >= 1
    return seed, p


def graft_dropout_mask(seed, p, S, D):
    """uint8 [S, D]: 1 where (slot, column) survives the fact-message dropout of :func:`graft_aggregate_train`
    (same Philox keying, gr_graft_dropout_mask); all ones for p == 0."""
    seed, p = _seed_p(seed, p)
    dev = seed.device if seed is not None else torch.device("cuda")
    mask = torch.empty(max(S, 1), D, dtype=torch.uint8, device=dev)
    _launch("gr_graft_dropout_mask", _p(seed), p, S, D, _p(mask), launches=1 if S > 0 else 0)
    return mask[:S]


def fact_train_ok(D):
    """True when the TypeLayer and GraftNet training kernels (gr_type_layer_backward, gr_graft_aggregate_train /
    _backward, gr_graft_attention_backward) admit width D: D <= 512."""
    return D <= 512


def graft_aggregate_train(gg, s, self_tab, head_tab, seed=None, p=0.0, sum_out=None):
    """Training forward of the fact messages (gr_graft_aggregate_train): sum_out [B*N, D] with
    sum_out[n] = sum_{f -> n} drop_f(relu(self_tab[r_f] + head_tab[head_f])) * s_f.  ``s``: fp32 per staged fact;
    ``seed``: device int64 [1] (read when p > 0).  head_tab and sum_out: both fp32 or both bf16 (sum_out, when not
    given, takes head_tab's dtype; bf16 holds the fp32 sums rounded to nearest even)."""
    g = gg.graph
    self_tab = _cuda(self_tab, torch.float32, "self_tab")
    head_tab = _cuda(head_tab, name="head_tab")
    s = _cuda(s, torch.float32, "s").contiguous()
    D = self_tab.shape[1]
    assert self_tab.stride(1) == 1 and head_tab.stride(1) == 1 and head_tab.shape[0] == gg.B * gg.N
    seed, p = _seed_p(seed, p)
    if sum_out is None:
        sum_out = torch.empty(gg.B * gg.N, D, dtype=head_tab.dtype, device=self_tab.device)
    io = _node_io(head_tab=head_tab, sum_out=sum_out)
    assert sum_out.stride(1) == 1
    if s.numel() == 0:               # no staged facts (every question's subgraph empty): every row sums nothing
        return sum_out.zero_()
    _launch("gr_graft_aggregate_train", _p(g.rowptr_t), _p(g.src_t), _p(g.rel_t), _p(g.fact_t), _p(gg.slot_of), _p(s),
            _p(self_tab), self_tab.stride(0), _p(head_tab), head_tab.stride(0), _p(seed), p, _p(sum_out),
            sum_out.stride(0), gg.B, gg.N, D, io=io, agg=("graft_train", 1))
    return sum_out


def graft_aggregate_backward(gg, s, self_tab, head_tab, grad_sum, grad_s, grad_self, grad_head, seed=None, p=0.0,
                             deterministic=False):
    """Accumulate the gradients of :func:`graft_aggregate_train` (same s, tables, seed and p) into grad_s [F],
    grad_self [R1, D] and grad_head [B*N, D] (gr_graft_aggregate_backward, over the head CSR).  ``deterministic``:
    grad_self in relation order instead of fp32 atomics (gr_graft_aggregate_backward_det).  head_tab, grad_sum and
    grad_head: all fp32 or all bf16 (grad_head is read, added to and stored rounded to nearest even)."""
    g = gg.graph
    self_tab = _cuda(self_tab, torch.float32, "self_tab")
    io = _node_io(head_tab=head_tab, grad_sum=grad_sum, grad_head=grad_head)
    s = _cuda(s, torch.float32, "s").contiguous()
    D = self_tab.shape[1]
    assert all(t.stride(1) == 1 for t in (self_tab, head_tab, grad_sum, grad_self, grad_head))
    assert grad_s.is_contiguous() and grad_s.dtype == torch.float32
    seed, p = _seed_p(seed, p)
    if s.numel() == 0:               # no staged facts: nothing to add
        return
    args = (_p(g.rowptr_h), _p(g.src_h), _p(g.rel_h), _p(g.fact_h), _p(gg.slot_of), _p(s), _p(self_tab),
            self_tab.stride(0), _p(head_tab), head_tab.stride(0), _p(seed), p, _p(grad_sum), grad_sum.stride(0),
            _p(grad_s), _p(grad_self), grad_self.stride(0), _p(grad_head), grad_head.stride(0), gg.B, gg.N, D)
    if deterministic:
        R1 = self_tab.shape[0]
        rix_ptr, rix_fact = gg.fact_relation_index(R1)
        ws, nbytes = _workspace(s.device, "gr_graft_aggregate_backward_det_workspace_bytes", gg.cap, D)
        _launch("gr_graft_aggregate_backward_det", *args, _p(gg.heads), _p(gg.rels), _p(gg.tails), _p(rix_ptr),
                _p(rix_fact), R1, gg.cap, _p(ws), nbytes, io=io, launches=3, op="aggregation_bwd_det")
        return
    _launch("gr_graft_aggregate_backward", *args, io=io, op="aggregation_bwd")


def graft_attention_backward(gg, qh, qmask, rel, grad_W, grad_qh, grad_rel, deterministic=False):
    """Accumulate dL/dqh [B, Q, D] and dL/drel [R1, D] of :func:`graft_attention`'s W given grad_W [B*max_fact]
    (gr_graft_attention_backward).  ``deterministic``: per-slot coefficients, then fixed-order sums by question and
    by relation (gr_graft_attention_backward_det)."""
    qh = _cuda(qh, torch.float32, "qh").contiguous()
    qmask = _cuda(qmask, torch.float32, "qmask").contiguous()
    rel = _cuda(rel, torch.float32, "rel")
    grad_W = _cuda(grad_W, torch.float32, "grad_W").contiguous()
    assert rel.stride(1) == 1 and grad_rel.stride(1) == 1 and grad_qh.is_contiguous()
    B, Q, D = qh.shape
    if deterministic:
        if gg.max_fact == 0:
            return
        R1 = rel.shape[0]
        rix_ptr, rix_slot = gg.slot_relation_index(R1)
        ws, nbytes = _workspace(qh.device, "gr_graft_attention_backward_det_workspace_bytes", B, gg.max_fact, Q, D)
        _launch("gr_graft_attention_backward_det", _p(qh), _p(qmask), Q, _p(rel), rel.stride(0), R1,
                _p(gg.kb_fact_rel), B, gg.max_fact, D, _p(grad_W), _p(grad_qh), _p(grad_rel), grad_rel.stride(0),
                _p(rix_ptr), _p(rix_slot), _p(ws), nbytes, launches=4, op="graft_attention_bwd_det")
        return
    _launch("gr_graft_attention_backward", _p(qh), _p(qmask), Q, _p(rel), rel.stride(0), rel.shape[0],
            _p(gg.kb_fact_rel), B, gg.max_fact, D, _p(grad_W), _p(grad_qh), _p(grad_rel), grad_rel.stride(0),
            launches=1 if gg.max_fact > 0 else 0, op="graft_attention_bwd")


def type_layer_backward(g, grad_out, out, grad_table, w_t=None, w_h=None, deterministic=False):
    """Accumulate dL/dtable [R1, D] of :func:`type_layer` given grad_out and the forward's ``out`` [B*N, D], both fp32
    or both bf16 (gr_type_layer_backward).  ``deterministic``: relation-ordered sums instead of fp32 atomics
    (gr_type_layer_backward_det)."""
    io = _node_io(grad_out=grad_out, out=out)
    assert grad_out.stride(1) == 1 and out.stride(1) == 1 and grad_table.stride(1) == 1
    D = out.shape[1]
    if deterministic:
        assert grad_table.shape[0] >= g.R1
        ptr_t, slot_t, row_t = csr_relation_index(g, "fwd")
        ptr_h, slot_h, row_h = csr_relation_index(g, "inv")
        ws, nbytes = _workspace(out.device, "gr_type_layer_backward_det_workspace_bytes", g.F, D)
        _launch("gr_type_layer_backward_det", _p(g.rel_t), _p(w_t), _p(ptr_t), _p(slot_t), _p(row_t),
                _p(g.rel_h), _p(w_h), _p(ptr_h), _p(slot_h), _p(row_h), _p(grad_out), grad_out.stride(0),
                _p(out), out.stride(0), _p(grad_table), grad_table.stride(0), g.R1, D, g.F, _p(ws), nbytes, io=io,
                launches=4 if g.F > 0 else 0, op="type_layer_bwd_det")
        return
    _launch("gr_type_layer_backward", _p(g.rowptr_t), _p(g.rel_t), _p(w_t), _p(g.rowptr_h), _p(g.rel_h), _p(w_h),
            _p(grad_out), grad_out.stride(0), _p(out), out.stride(0), _p(grad_table), grad_table.stride(0),
            g.B, g.N, D, g.F, io=io, op="type_layer_bwd")
