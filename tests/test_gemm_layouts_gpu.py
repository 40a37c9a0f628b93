"""GPU: the split-bf16 wgmma GEMM (gr_linear_tc_planes / gr_linear_tc, csrc/linear_tc.cu) against float64 element by
element, in every layout the models call it with -- segmented K with padded segments, column windows of the A planes
and of the output planes, output row pitches that force the direct-store epilogue, column-sliced weights, N > 256 in
column slices, the stacked relation tables -- plus the weight pre-split cache, and the layers the GEMM completes: the
dense ReaRev layer off the fused hot shape, the NSM layer, and every GEMM of full ReaRev, NSM and GraftNet forwards.

Bound (u = 2^-24).  With A the values the kernel reads (hi + lo of the planes in float64; the fp32 A for gr_linear_tc)
and s = |W| |A| + |b| per output element, as derived in test_dense_layer_gpu.py:
  * the W split, 2^-17 |W|, and the dropped A_lo W_lo product, 2^-16 (|A_lo| |W_lo| <= 2^-18 |A| |W|: generous);
  * the accumulation.  wgmma's internal accumulation order and rounding are not documented.  ASSUMED (not measured):
    each of the 3K products is added with one rounding of at most 2^-23 of the running sum, plus the bias add:
    (3K + 2) 2^-23 of s;
  * gr_linear_tc splits an fp32 A itself: + 2^-17 of s.
One bf16 product (ACT_BF16) is held to bf16(A_hi) bf16(W_hi) in float64 with (K + 2) 2^-23 of its own scale.  relu
does not enlarge an error.  Output planes are the bf16 split of the fp32 output bit for bit (within the bound plus
2^-17 |y| when no fp32 output is asked for), their pad columns N .. round16(N) are written as 0 and nothing past
round16(N) or row M is written.  dots[:M] + dots[M:] is within (N + 2) u |y| |w_score| plus |w_score| times y's bound.

A dropped product, a misaddressed segment, column or k-block, an unzeroed weight pad or a stale cached weight moves an
element by a sizeable fraction of its scale, far outside these bounds."""
import contextlib
import math

import numpy as np
import pytest
import torch

from gnn_rag_b200 import batching, modules, ops, optim
from gnn_rag_b200 import synthetic as S

import fp64_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
F64 = torch.float64
BF16 = torch.bfloat16
SENT = 7.0                          # what every output buffer holds before the call: unwritten elements keep it
SPLIT = 2.0 ** -17 + 2.0 ** -16     # the W split and the dropped A_lo W_lo product
VERY_NEG = -100000000000.0


def _r16(n):
    return (n + 15) // 16 * 16


def _r64(n):
    return (n + 63) // 64 * 64


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def _bits(p):
    return p.view(torch.int16 if p.dtype == BF16 else torch.int32)


def _bf(x):
    return x.to(BF16).to(F64)


@contextlib.contextmanager
def _options(cluster=1, bk=32, tma_store=1, single=False):
    try:
        ops.set_option("tc_cluster", cluster)
        ops.set_option("tc_bk", bk)
        ops.set_option("tc_tma_store", tma_store)
        ops.ACT_BF16 = single
        yield
    finally:
        ops.set_option("tc_cluster", 1)
        ops.set_option("tc_bk", 32)
        ops.set_option("tc_tma_store", 1)
        ops.ACT_BF16 = False


def _planes(X, width=None):
    """Split-bf16 planes [M, width] of fp32 X [M, K] (zero beyond K)."""
    M, K = X.shape
    hi = torch.zeros(M, width or _r64(K), dtype=BF16, device=DEV)
    lo = torch.zeros_like(hi)
    ops.split_bf16(X, hi, lo)
    return hi, lo


def _operand(hi, lo, K, k_seg=0, pitch=0, single=False):
    """The float64 A the kernel multiplies: hi + lo (hi alone for one product) of the first K columns, only the
    k_seg data columns of every segment when K is segmented (W's pad columns are zero)."""
    a = hi[:, :K].to(F64)
    if not single:
        a = a + lo[:, :K].to(F64)
    if k_seg and pitch > k_seg:
        a = a.reshape(a.shape[0], K // pitch, pitch)[:, :, :k_seg].reshape(a.shape[0], -1)
    return a


def _ref(A, W, bias, relu, K, single=False, extra=0.0):
    """(y, bound) in float64 for y = act(A W^T + b) from the operand A [M, Kw]."""
    W64 = _bf(W) if single else W.detach().to(F64)
    pre = A @ W64.t()
    s = A.abs() @ W64.abs().t()
    if bias is not None:
        pre = pre + bias.detach().to(F64)
        s = s + bias.detach().to(F64).abs()
    y = torch.relu(pre) if relu else pre
    f = (K + 2) * 2.0 ** -23 if single else SPLIT + (3 * K + 2) * 2.0 ** -23 + extra
    return y, f * s + 1e-30


def _dots_check(dots, M, y, bound, wsc):
    aw = wsc.detach().to(F64).abs()
    dbound = bound @ aw + (y.shape[1] + 2) * U * ((y.abs() + bound) @ aw) + 1e-30
    derr = (dots[:M].to(F64) + dots[M:2 * M].to(F64) - y @ wsc.detach().to(F64)).abs()
    assert (derr <= dbound).all(), (derr / dbound).max().item()
    return (derr / dbound).max().item()


def _out_checks(out, planes, dots, y, bound, wsc):
    """out / planes / dots (any may be None) against float64; returns the largest err/bound of out-or-planes and of
    the dots."""
    ratio = [0.0, 0.0]
    N = y.shape[1]
    if out is not None:
        err = (out.to(F64) - y).abs()
        assert (err <= bound).all(), (err / bound).max().item()
        ratio[0] = (err / bound).max().item()
    if planes is not None:
        hi, lo = planes[0][:, :N], planes[1][:, :N]
        if out is not None:
            hw = out.to(BF16)
            assert torch.equal(_bits(hi), _bits(hw))
            assert torch.equal(_bits(lo), _bits((out - hw.float()).to(BF16)))
        else:
            b2 = bound + 2.0 ** -17 * y.abs()
            err = (hi.to(F64) + lo.to(F64) - y).abs()
            assert (err <= b2).all(), (err / b2).max().item()
            ratio[0] = max(ratio[0], (err / b2).max().item())
    if dots is not None:
        ratio[1] = _dots_check(dots, y.shape[0], y, bound, wsc)
    return ratio


def _run(hi, lo, K, W, bias, wsc, M, relu=True, outs="cpd", k_seg=0, pitch=0, single=False,
         c_width=None, c_col0=0, p_width=None, p_col0=0):
    """One ops.linear_tc_planes call into sentinel-filled buffers with two spare rows and spare columns: fp32 out
    (view at c_col0 of a c_width-column buffer), planes (view at p_col0 of p_width columns), dots ([2M] of 2M + 8)."""
    N = W.shape[0]
    cbuf = torch.full((M + 2, c_width or N + 8), SENT, device=DEV)
    pbuf = [torch.full((M + 2, p_width or _r16(N) + 16), SENT, dtype=BF16, device=DEV) for _ in range(2)]
    dbuf = torch.full((2 * M + 8,), SENT, device=DEV)
    out = cbuf[:M, c_col0:c_col0 + N] if "c" in outs else None
    planes = tuple(p[:M, p_col0:p_col0 + N] for p in pbuf) if "p" in outs else None
    dots = dbuf[:2 * M] if "d" in outs else None
    ops.linear_tc_planes(hi, lo, K, W, bias, out=out, out_planes=planes, w_score=wsc if dots is not None else None,
                         dots=dots, relu=relu, k_seg=k_seg, k_seg_pitch=pitch, single_ok=single)
    torch.cuda.synchronize()
    return dict(cbuf=cbuf, pbuf=pbuf, dbuf=dbuf, out=out, planes=planes, dots=dots, M=M, N=N, c0=c_col0, p0=p_col0)


def _check(r, y, bound, wsc):
    """A :func:`_run` result against float64, and nothing written outside the requested views; returns the ratios."""
    M, N, c0, p0 = r["M"], r["N"], r["c0"], r["p0"]
    n16 = _r16(N)
    ratio = _out_checks(r["out"], r["planes"], r["dots"], y, bound, wsc)
    cbuf = r["cbuf"].clone()
    if r["out"] is not None:
        cbuf[:M, c0:c0 + N] = SENT
    bad = (cbuf != SENT).nonzero()
    assert bad.numel() == 0, ("written outside the fp32 view", bad[:8].tolist(), cbuf.shape, c0, N)
    for pb in r["pbuf"]:
        if r["planes"] is None:
            assert (pb == SENT).all()
            continue
        assert (pb[:M, p0 + N:p0 + n16] == 0).all()               # pad columns N .. round16(N) written as 0
        assert (pb[:M, :p0] == SENT).all() and (pb[:M, p0 + n16:] == SENT).all() and (pb[M:] == SENT).all()
    assert (r["dbuf"][2 * M:] == SENT).all()
    if r["dots"] is None:
        assert (r["dbuf"] == SENT).all()
    return ratio


def _same_bits(a, b):
    """Every output both runs wrote is equal bit for bit."""
    for k in ("out", "dots"):
        if a[k] is not None and b[k] is not None:
            assert torch.equal(_bits(a[k]), _bits(b[k])), k
    if a["planes"] is not None and b["planes"] is not None:
        for pa, pb in zip(a["pbuf"], b["pbuf"]):
            assert torch.equal(_bits(pa), _bits(pb))


def _segmented_inputs(rs, M, T, D, N, garbage=True):
    """(hi, lo) planes of T segments of D data columns at pitch round16(D) -- finite non-zero garbage in the pad
    columns when ``garbage`` -- the same planes with zero pads, W [N, T D], bias, w_score."""
    P = _r16(D)
    X = rs.randn(M, T, P).astype(np.float32)
    X0 = X.copy()
    X0[:, :, D:] = 0
    if garbage:
        X[:, :, D:] = rs.choice([-1.0, 1.0], size=X[:, :, D:].shape) * rs.uniform(50, 100, size=X[:, :, D:].shape)
    hi, lo = _planes(_t(X.reshape(M, T * P)))
    hi0, lo0 = _planes(_t(X0.reshape(M, T * P)))
    W = _t(rs.randn(N, T * D) / np.sqrt(T * D))
    return (hi, lo), (hi0, lo0), W, _t(rs.randn(N) * 0.1), _t(rs.randn(N))


def _launch_ws(ws, hi, lo, K, W, bias, out, k_seg, pitch, relu):
    """gr_linear_tc_planes on a caller-owned W workspace (split afresh: no W_PRESPLIT)."""
    ops._launch("gr_linear_tc_planes", ops._p(hi), ops._p(lo), hi.stride(0), ops._p(W), W.stride(0), ops._p(bias),
                ops._p(out), out.stride(0), None, None, 0, None, None, out.shape[0], W.shape[0], K, k_seg, pitch,
                ops.LINEAR_RELU if relu else 0, ops._p(ws), ws.numel())


# ---- segmented K ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("D", [8, 50, 72, 100, 120, 136, 200, 256])
@pytest.mark.parametrize("T", [1, 2, 3, 5, 7])
def test_segmented_layout_vs_fp64(T, D, relu):
    """T segments of D columns at pitch round16(D) (pad width 0, 8, 12 or 14), the layout of the dense ReaRev / NSM
    layers.  A's pad columns hold finite non-zero garbage: with W's pads zero the result equals the zero-pad run bit for
    bit.  Every output alone equals the run that writes all three.  A W workspace that first held a larger, different
    W's planes gives the same bits (the pads of a reused buffer are zeroed)."""
    rs = np.random.RandomState(100 * T + D + 7 * relu)
    M, N, P = 300, D, _r16(D)
    K = T * P
    (hi, lo), (hi0, lo0), W, bias, wsc = _segmented_inputs(rs, M, T, D, N)
    y, bound = _ref(_operand(hi, lo, K, D, P), W, bias, relu, K)
    kw = dict(relu=relu, k_seg=D, pitch=P)
    full = _run(hi, lo, K, W, bias, wsc, M, **kw)
    ratio = _check(full, y, bound, wsc)
    _same_bits(_run(hi0, lo0, K, W, bias, wsc, M, **kw), full)
    for outs in ("c", "p", "pd"):                 # dots alone is refused: they come with an output
        r = _run(hi, lo, K, W, bias, wsc, M, outs=outs, **kw)
        _check(r, y, bound, wsc)
        _same_bits(r, full)
    big = _t(rs.randn(256, K) * 3.0)
    ws = torch.empty(ops._L().gr_linear_tc_planes_workspace_bytes(256, K), dtype=torch.uint8, device=DEV)
    scratch = torch.empty(M, 256, device=DEV)
    _launch_ws(ws, hi, lo, K, big, None, scratch, 0, 0, False)            # ws now holds the larger W's planes
    reused = torch.full((M, N), SENT, device=DEV)
    _launch_ws(ws, hi, lo, K, W, bias, reused, D, P, relu)
    torch.cuda.synchronize()
    assert torch.equal(_bits(reused), _bits(full["out"]))
    print("segmented T=%d D=%d relu=%d: max err/bound out %.3g dots %.3g" % (T, D, relu, *ratio))


@pytest.mark.parametrize("T,D", [(1, 200), (3, 50), (5, 200), (7, 72), (2, 136)])
def test_single_product_vs_fp64(T, D):
    """ACT_BF16: one product A_hi W_hi over the segmented layout (cfg3), held to bf16(A_hi) bf16(W_hi) in float64."""
    rs = np.random.RandomState(T * 1000 + D)
    M, N, P = 1000, D, _r16(D)
    K = T * P
    (hi, lo), _zero, W, bias, wsc = _segmented_inputs(rs, M, T, D, N)
    with _options(single=True):
        r = _run(hi, lo, K, W, bias, wsc, M, k_seg=D, pitch=P, single=True)
    y, bound = _ref(_operand(hi, lo, K, D, P, single=True), W, bias, True, K, single=True)
    ratio = _check(r, y, bound, wsc)
    print("single product T=%d D=%d: max err/bound out %.3g dots %.3g" % (T, D, *ratio))


# ---- tiles and kernel options ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("tma_store", [1, 0])
@pytest.mark.parametrize("bk", [32, 64])
@pytest.mark.parametrize("cluster", [1, 2])
def test_tiles_and_kernel_options_vs_fp64(cluster, bk, tma_store):
    """M = 1, 127, 128, 129 (one and two tiles), 1100 (9 tiles: odd for CTA pairs) and enough rows that every persistent
    CTA (or CTA pair) takes at least 3 tiles, an odd count.  K = 3 x 112 is not a multiple of either k-block width, so
    the last k-block is partial."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    big = 128 * (3 * sms + 2) + 37
    tiles = math.ceil(big / 128)
    assert tiles % 2 == 1 and math.ceil(tiles / 2) >= 3 * (sms // 2) and tiles >= 3 * sms
    T, D = 3, 100
    P = _r16(D)
    K = T * P
    assert K % 32 and K % 64
    rs = np.random.RandomState(cluster + 2 * bk + tma_store)
    worst = [0.0, 0.0]
    with _options(cluster=cluster, bk=bk, tma_store=tma_store):
        for M in (1, 127, 128, 129, 1100, big):
            (hi, lo), _zero, W, bias, wsc = _segmented_inputs(rs, M, T, D, D)
            y, bound = _ref(_operand(hi, lo, K, D, P), W, bias, True, K)
            ratio = _check(_run(hi, lo, K, W, bias, wsc, M, k_seg=D, pitch=P), y, bound, wsc)
            worst = [max(a, b) for a, b in zip(worst, ratio)]
    print("tiles cluster=%d bk=%d tma_store=%d: max err/bound out %.3g dots %.3g" % (cluster, bk, tma_store, *worst))


# ---- output views and A windows ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("D", [50, 200])
def test_output_views_and_a_windows_vs_fp64(D):
    """GraftLayer's geometry: planes of five segments at pitch Dp.  The A operand is a column window hi[:, k Dp:] (the
    head GEMM: k = 2, K = Dp; the e2e GEMM: k = 2, K = 3 Dp; the f2e GEMM: k = 0, K = 3 Dp), the output planes go to a
    window at column 2 Dp or 4 Dp of a wider buffer.  The fp32 output is a view whose row pitch is not a multiple of
    16 bytes (and a base 4 bytes off: direct, unvectorised stores) or is one.  At D = 50 the second view's rows end
    mid 16-byte unit: the TMA-store epilogue would write two columns past N there, so it must take the direct stores."""
    rs = np.random.RandomState(D)
    M, P = 700, _r16(D)
    Kp = _r64(5 * P)
    X = rs.randn(M, 5, P).astype(np.float32)
    X[:, :, D:] = 0
    hi, lo = _planes(_t(X.reshape(M, 5 * P)), Kp)
    worst = [0.0, 0.0]
    for col, T in ((2, 1), (2, 3), (0, 3)):
        ahi, alo = hi[:, col * P:], lo[:, col * P:]
        K = T * P
        W = _t(rs.randn(D, T * D) / np.sqrt(T * D))
        bias, wsc = _t(rs.randn(D) * 0.1), _t(rs.randn(D))
        y, bound = _ref(_operand(ahi, alo, K, D, P), W, bias, True, K)
        for c_width, c_col0 in ((D + 3, 1), (_r16(D) + 16, 4)):
            for p_col0 in (2 * P, 4 * P):
                r = _run(ahi, alo, K, W, bias, wsc, M, k_seg=D, pitch=P, c_width=c_width, c_col0=c_col0,
                         p_width=Kp, p_col0=p_col0)
                ratio = _check(r, y, bound, wsc)
                worst = [max(a, b) for a, b in zip(worst, ratio)]
    print("views and windows D=%d: max err/bound out %.3g dots %.3g" % (D, *worst))


# ---- N > 256 ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("segmented", [False, True])
@pytest.mark.parametrize("N", [257, 300, 400, 512])
def test_column_slices_vs_fp64(N, segmented):
    """N > 256 runs as launches over column slices of W (a step rounded to 16): out, the planes across the seam
    between slices, and the dots summed over the slices."""
    rs = np.random.RandomState(N + segmented)
    M = 1000
    if segmented:
        T, D = 3, 100
        P = _r16(D)
        K = T * P
        (hi, lo), _zero, _w, _b, _s = _segmented_inputs(rs, M, T, D, 8)
        W = _t(rs.randn(N, T * D) / np.sqrt(T * D))
        kw = dict(k_seg=D, pitch=P)
        A = _operand(hi, lo, K, D, P)
    else:
        K = 200
        hi, lo = _planes(_t(rs.randn(M, K)))
        W = _t(rs.randn(N, K) / np.sqrt(K))
        kw = {}
        A = _operand(hi, lo, K)
    bias, wsc = _t(rs.randn(N) * 0.1), _t(rs.randn(N))
    y, bound = _ref(A, W, bias, True, K)
    ratio = _check(_run(hi, lo, K, W, bias, wsc, M, **kw), y, bound, wsc)
    print("column slices N=%d segmented=%d: max err/bound out %.3g dots %.3g" % (N, segmented, *ratio))


# ---- the weight pre-split cache -------------------------------------------------------------------------------------

def _layer_planes(rs, M, I, D):
    """[h | 2I neighbour segments] planes at pitch Dp, the fp32 values, and the dense [M, (2I+1) D] planes."""
    P = _r16(D)
    T = 2 * I + 1
    X = rs.randn(M, T, D).astype(np.float32)
    Xp = np.zeros((M, T, P), np.float32)
    Xp[:, :, :D] = X
    return _planes(_t(Xp.reshape(M, T * P))), _planes(_t(X.reshape(M, T * D)))


def test_weight_cache_layouts_and_slices_alternate():
    """One e2e weight seen as ``e2e.weight`` (segmented, plain and grouped-order layouts) and as ``e2e.weight[:, :D]``
    (the sparse-prior GEMM's h-segment weight, row stride (2I+1) D), called in turn twice over: each call gives its own
    float64 result, so no layout or view is served another one's cached planes."""
    rs = np.random.RandomState(3)
    M, I, D = 500, 2, 50
    P, T = _r16(D), 2 * I + 1
    lin = torch.nn.Linear(T * D, D).to(DEV)
    W, bias = lin.weight, lin.bias
    wsc = _t(rs.randn(D))
    (hi, lo), (dhi, dlo) = _layer_planes(rs, M, I, D)
    calls = {
        "segmented": (hi, lo, T * P, W, dict(k_seg=D, k_seg_pitch=P)),
        "h segment": (hi, lo, P, W[:, :D], dict(k_seg=D, k_seg_pitch=P)),
        "plain": (dhi, dlo, T * D, W, {}),
        "grouped": (hi, lo, T * P, W, dict(k_seg=D, k_seg_pitch=P, k_grouped=True)),
    }
    assert calls["h segment"][3].stride(0) == T * D
    worst = 0.0
    with torch.no_grad():
        for _round in range(2):
            for name, (ahi, alo, K, Wv, kw) in calls.items():
                out = torch.full((M, D), SENT, device=DEV)
                dots = torch.full((2 * M,), SENT, device=DEV)
                ops.linear_tc_planes(ahi, alo, K, Wv, bias, out=out, w_score=wsc, dots=dots, relu=True, **kw)
                torch.cuda.synchronize()
                seg = kw.get("k_seg", 0), kw.get("k_seg_pitch", 0)
                y, bound = _ref(_operand(ahi, alo, K, *seg), Wv, bias, True, K)
                worst = max(worst, _out_checks(out, None, dots, y, bound, wsc)[0])
    print("weight cache, alternating layouts: max err/bound %.3g" % worst)


def test_weight_cache_korder_alternates_with_the_other_layouts():
    """The dense-layer weight at D = 200 (the width the K-order layout serves) called in turn, twice over: segmented,
    the h-segment view, grouped order over the segment layout and grouped order over the K-order layout
    (GR_LINEAR_K_ORDER_PLANES, W packed under a cache key of its own).  The first three are held to float64; the
    K-order call reads the same A values in the same k16 steps and so must equal the grouped call bit for bit."""
    NR, B, N, I, D, P = 30, 3, 600, 2, 200, 208
    T, M = 2 * I + 1, B * N
    db, _facts, _w, _dt, _dh = _stage(11, B, N, 6 * N, NR, False)
    rs = np.random.RandomState(11)
    pn = ops.pad_table256(_t(rs.randn(2 * (NR + 1), D)))
    ins, h = _t(rs.randn(B, I, D)), _t(rs.randn(M, D))
    prior = torch.softmax(_t(rs.randn(B, N)), 1)
    nb0 = ops.k_order_nb0(P)
    width = _r64(nb0 + 2 * I * P)
    seg, ko = _planes(h, width), _planes(h, width)
    ops.aggregate_dual_abs(db.graph, prior, pn[:NR + 1], pn[NR + 1:], ins, seg, P, P)
    ops.aggregate_dual_abs(db.graph, prior, pn[:NR + 1], pn[NR + 1:], ins, ko, nb0, P, k_order=True)
    lin = torch.nn.Linear(T * D, D).to(DEV)
    W, bias, wsc = lin.weight, lin.bias, _t(rs.randn(D))
    calls = {
        "segmented": (seg, T * P, W, dict(k_seg=D, k_seg_pitch=P)),
        "h segment": (seg, P, W[:, :D], dict(k_seg=D, k_seg_pitch=P)),
        "grouped": (seg, T * P, W, dict(k_seg=D, k_seg_pitch=P, k_grouped=True)),
        "k-order": (ko, T * P, W, dict(k_seg=D, k_seg_pitch=P, k_grouped=True, k_order=True)),
    }
    worst = 0.0
    with torch.no_grad():
        for _round in range(2):
            got = {}
            for name, ((ahi, alo), K, Wv, kw) in calls.items():
                out = torch.full((M, D), SENT, device=DEV)
                dots = torch.full((2 * M,), SENT, device=DEV)
                ops.linear_tc_planes(ahi, alo, K, Wv, bias, out=out, w_score=wsc, dots=dots, relu=True, **kw)
                torch.cuda.synchronize()
                got[name] = (out, dots)
                if name != "k-order":
                    y, bound = _ref(_operand(ahi, alo, K, D, P), Wv, bias, True, K)
                    worst = max(worst, _out_checks(out, None, dots, y, bound, wsc)[0])
            for a, b in zip(got["k-order"], got["grouped"]):
                assert torch.equal(_bits(a), _bits(b))
    print("weight cache, K-order alternating: max err/bound %.3g" % worst)


def test_weight_cache_follows_updates():
    """In-place updates (``mul_`` under no_grad, an optimizer step, the fused clip + Adam step that writes through raw
    pointers) are seen by the next call; a per-call weight freed and re-created at the same address gives its new
    values; a write through ``.data`` is documented not to bump the version, and after clear_weight_cache() the result
    is right again."""
    rs = np.random.RandomState(4)
    M, I, D = 400, 1, 72
    P, T = _r16(D), 2 * I + 1
    (hi, lo), _dense = _layer_planes(rs, M, I, D)
    A = _operand(hi, lo, T * P, D, P)
    lin = torch.nn.Linear(T * D, D).to(DEV)
    W, bias = lin.weight, lin.bias
    ops.clear_weight_cache()

    def call(Wv):
        out = torch.full((M, D), SENT, device=DEV)
        ops.linear_tc_planes(hi, lo, T * P, Wv, bias, out=out, relu=False, k_seg=D, k_seg_pitch=P)
        torch.cuda.synchronize()
        return out

    def check(Wv):
        y, bound = _ref(A, Wv, bias, False, T * P)
        return _out_checks(call(Wv), None, None, y, bound, None)[0]

    worst = check(W)
    with torch.no_grad():
        W.mul_(-0.5)
    worst = max(worst, check(W))
    opt = torch.optim.SGD([W], lr=1.0)
    W.grad = torch.randn_like(W)
    opt.step()
    worst = max(worst, check(W))
    W.grad = torch.randn_like(W)
    optim.ClipAdam(torch.optim.Adam([W], lr=1e-2), [W], [W.grad], max_norm=1.0).step()
    worst = max(worst, check(W))
    ptrs = []
    for k in range(4):
        Wc = torch.zeros(D, T * D, device=DEV)
        Wc[:, (k % T) * D:(k % T + 1) * D] = _t(rs.randn(D, D))     # another block every call: a stale split shows
        ptrs.append(Wc.data_ptr())
        worst = max(worst, check(Wc))
        del Wc
    assert len(set(ptrs)) < len(ptrs)                      # the allocator handed an address back
    W.data.mul_(2.0)
    ops.clear_weight_cache()
    worst = max(worst, check(W))
    print("weight cache, updates: max err/bound %.3g" % worst)


# ---- gr_linear_tc (fp32 A) and the relation tables -------------------------------------------------------------------

@pytest.mark.parametrize("M,N,K", [(1, 8, 8), (129, 200, 1000), (1000, 50, 250), (300, 256, 300)])
def test_linear_tc_fp32_a_vs_fp64(M, N, K):
    """gr_linear_tc splits an fp32 A (a strided row view) itself: + 2^-17 of the scale."""
    rs = np.random.RandomState(M + N + K)
    A = _t(rs.randn(M, K + 4))[:, 4:]
    W = _t(rs.randn(N, K) / np.sqrt(K))
    bias = _t(rs.randn(N) * 0.1)
    cbuf = torch.full((M + 2, N + 8), SENT, device=DEV)
    ops.linear_tc(A, W, bias, relu=True, out=cbuf[:M, :N])
    torch.cuda.synchronize()
    y, bound = _ref(A.to(F64), W, bias, True, K, extra=2.0 ** -17)
    ratio = _out_checks(cbuf[:M, :N], None, None, y, bound, None)[0]
    cbuf[:M, :N] = SENT
    assert (cbuf == SENT).all()
    print("gr_linear_tc M=%d N=%d K=%d: max err/bound %.3g" % (M, N, K, ratio))


@pytest.mark.parametrize("R1", [1, 127, 6107])
def test_relation_tables_vs_fp64(R1):
    """rel_features_from_embeddings: relation_linear over the word-dim embeddings (K = 300, from param_planes) into
    the stacked planes, both directions; rel_table: the per-layer projection of those planes, with and without the
    pos_emb addends (added in fp32 afterwards), and one direction only (NSM)."""
    rs = np.random.RandomState(R1)
    Kw, D = 300, 200
    embs = [_t(rs.randn(R1, Kw)) for _ in range(2)]
    Wr, br = _t(rs.randn(D, Kw) / np.sqrt(Kw)), _t(rs.randn(D) * 0.1)
    rf = ops.rel_features_from_embeddings(embs, Wr, br)
    torch.cuda.synchronize()
    worst = 0.0
    for d, E in enumerate(embs):
        ehi, elo = ops.param_planes(E)
        y, bound = _ref(_operand(ehi, elo, Kw), Wr, br, False, Kw)
        worst = max(worst, _out_checks(None, (rf.hi[rf.rows(d)], rf.lo[rf.rows(d)]), None, y, bound, None)[0])
    assert (rf.hi[:, D:_r16(D)] == 0).all() and (rf.lo[:, D:_r16(D)] == 0).all()
    W2, b2 = _t(rs.randn(D, D) / np.sqrt(D)), _t(rs.randn(D) * 0.1)
    adds = [_t(rs.randn(R1, D)), _t(rs.randn(R1, D))]
    for addends, dirs in ((None, None), (adds, None), (None, 1)):
        tabs = ops.rel_table(rf, W2, b2, dirs=dirs, addends=addends)
        torch.cuda.synchronize()
        for d, tab in enumerate(tabs):
            y, bound = _ref(_operand(rf.hi[rf.rows(d)], rf.lo[rf.rows(d)], D), W2, b2, False, D)
            if addends is not None:
                y = y + addends[d].to(F64)
                bound = bound + U * y.abs()
            worst = max(worst, _out_checks(tab, None, None, y, bound, None)[0])
    print("relation tables R1=%d: max err/bound %.3g" % (R1, worst))


# ---- the layers the GEMM completes ------------------------------------------------------------------------------------

def _stage(seed, B, N, E, R, normalized):
    b = S.make_batch(seed, B=B, N=N, E=E, num_entity=5000, num_relation=R, num_word=50, n_real="ragged",
                     powerlaw=True)
    db = batching.stage_batch(b, torch.device(DEV), R + 1, normalized, False)
    kb = b[2]
    facts = tuple(_t(np.asarray(a), torch.int64) for a in (kb[0], kb[1], kb[2]))
    w = _t(np.asarray(kb[5], np.float32)).to(F64) if normalized else None
    Nt = B * N
    heads, tails = np.asarray(kb[0]), np.asarray(kb[2])
    deg_t, deg_h = np.bincount(tails, minlength=Nt), np.bincount(heads, minlength=Nt)
    return db, facts, w, deg_t, deg_h


def _put_h(layer, h):
    """The layer-input h into the first D columns of the current planes (the pads stay zero)."""
    hi, lo = layer.P[layer.cur]
    ops.split_bf16(h, hi, lo)
    return _operand(hi, lo, h.shape[1])


def _softmax_check(dist, s, sb, mask, dbound, B, N):
    """dist against the float64 masked softmax of s + sb, s off by at most ``dbound``."""
    z = (s + float(sb) + (1 - mask.to(F64)) * VERY_NEG).view(B, N)
    p = torch.softmax(z, 1)
    delta = (dbound + U * z.abs().view(-1) * (mask.view(-1) > 0)).view(B, N).max(1, keepdim=True)[0]
    zmax = z.max(1, keepdim=True)[0]
    bound = p * (2.01 * delta + (128 + 8 * (zmax - z).clamp_max(200)) * U) + 1e-30
    err = (dist.view(B, N).to(F64) - p).abs()
    assert (err <= bound).all(), (err / bound).max().item()
    return (err / bound).max().item()


@pytest.mark.parametrize("single", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("D,I,B,N", [(50, 2, 4, 300), (50, 3, 4, 300), (72, 2, 3, 500), (120, 2, 3, 500),
                                     (200, 2, 4, 2000)])
def test_dense_rearev_layer_vs_fp64(D, I, B, N, weighted, single):
    """ReasonGNNLayer.forward(sparse_prior=False) off the fused hot shape: the aggregation into the segmented planes,
    then the segmented GEMM with the score dot, then the masked softmax.  D = 50, 72, 120 run the generic aggregation
    kernel; D = 200 with B N below FUSED_MIN_ROWS the |v|-accumulating one.  Power-law tails give hub rows.  A operand:
    (2n + 8) u of the aggregation scale (test_aggregate_edges_gpu.py), n the row's larger in-degree.  ACT_BF16: the
    planes keep hi only and the GEMM is one bf16 product, + 2^-8 of the scale."""
    if D == 200:
        assert B * N < ops.FUSED_MIN_ROWS
    NR = 30
    db, facts, w, deg_t, deg_h = _stage(D + I + 10 * weighted, B, N, 6 * N, NR, weighted)
    assert max(deg_t.max(), deg_h.max()) > 64
    rs = np.random.RandomState(D + I + weighted + single)
    layer = modules.ReasonGNNLayer(dict(num_ins=I, num_gnn=1, pos_emb=False, normalized_gnn=weighted), 5000, NR, D,
                                   "bfs").to(DEV)
    M, P = B * N, _r16(D)
    K = (2 * I + 1) * P
    with torch.no_grad(), _options(single=single):
        rf = ops.rel_features_from_tensors([_t(rs.randn(NR + 1, D)), _t(rs.randn(NR + 1, D))])
        layer.init_reason(db, rf)
        h64 = _put_h(layer, _t(rs.randn(M, D)))
        if single:
            hi = layer.P[layer.cur][0]
            h64 = hi[:, :D].to(F64)
        prior = torch.softmax(_t(rs.randn(B, N)), 1)
        ins = _t(rs.randn(B, I, D))
        dist, h32 = layer.forward(prior, ins, step=0, need_h=True, sparse_prior=False)
        torch.cuda.synchronize()
    tf, ti, _pn = layer.tables[0]
    e2e = layer.e2e_linear0
    W, b = e2e.weight.detach(), e2e.bias.detach()
    sw, sb = layer.score_func.weight.detach().view(-1), layer.score_func.bias.detach()
    args = (h64, prior.to(F64), tf.to(F64), ti.to(F64), ins.to(F64), (_bf(W) if single else W.to(F64)), b.to(F64))
    y, s = R.rearev_layer(*args, sw.to(F64), facts, w)
    scale = R.rearev_layer_scale(*args, facts, w)
    n = _t(np.maximum(deg_t, deg_h), F64)[:, None]
    f = (2 * n + 8) * U + ((2.0 ** -8 + 2.0 ** -16 + (K + 2) * 2.0 ** -23) if single else
                           (2.0 ** -15 + (3 * K + 2) * 2.0 ** -23))
    bound = f * scale + 1e-30
    nhi, nlo = layer.P[layer.cur]
    ratio = _out_checks(h32, (nhi, nlo), layer.dots, y, bound, sw)
    assert (nhi[:, D:P] == 0).all() and (nlo[:, D:P] == 0).all()
    dbound = bound @ sw.to(F64).abs() + (D + 2) * U * ((y.abs() + bound) @ sw.to(F64).abs()) + 1e-30
    rd = _softmax_check(dist, s, sb, layer.local_entity_mask, dbound, B, N)
    print("ReaRev layer D=%d I=%d weighted=%d single=%d: max err/bound h %.3g dots %.3g dist %.3g"
          % (D, I, weighted, single, *ratio, rd))


@pytest.mark.parametrize("reason_kb", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("D", [50, 200])
def test_nsm_layer_vs_fp64(D, weighted, reason_kb):
    """NSMLayer.forward: the one-direction aggregation in fp32, split into the neighbour segment at column Dp, the
    two-segment GEMM (an even segment count), the score dot and the masked softmax (with ``possible`` under
    reason_kb), against fp64_ref.nsm_layer."""
    NR, B, N = 30, 4, 400
    db, facts, w, deg_t, _deg_h = _stage(D + 3 * weighted + reason_kb, B, N, 6 * N, NR, weighted)
    rs = np.random.RandomState(D + weighted)
    layer = modules.NSMLayer(dict(num_step=1, reason_kb=reason_kb, normalized_gnn=weighted), 5000, NR, D).to(DEV)
    M, P = B * N, _r16(D)
    with torch.no_grad():
        layer.init_reason(db, ops.rel_features_from_tensors([_t(rs.randn(NR + 1, D))]))
        h64 = _put_h(layer, _t(rs.randn(M, D)))
        prior = torch.softmax(_t(rs.randn(B, N)), 1)
        prior[:, ::3] = 0                          # rows whose every in-edge carries no mass: possible = 0
        prior /= prior.sum(1, keepdim=True)
        ins = _t(rs.randn(B, D))
        dist = layer.forward(prior, ins, step=0)
        torch.cuda.synchronize()
    e2e = layer.e2e_linear0
    W, b = e2e.weight.detach().to(F64), e2e.bias.detach().to(F64)
    sw, sb = layer.score_func.weight.detach().view(-1), layer.score_func.bias.detach()
    args = (h64, prior.to(F64), layer.tables[0].to(F64), ins.to(F64), W, b)
    y, s, poss = R.nsm_layer(*args, sw.to(F64), facts, w)
    scale = R.nsm_layer_scale(*args, facts, w)
    n = _t(deg_t, F64)[:, None]
    bound = ((2 * n + 8) * U + 2.0 ** -17 + SPLIT + (3 * 2 * P + 2) * 2.0 ** -23) * scale + 1e-30
    assert torch.equal(layer.possible.to(F64), poss)
    assert (poss == 0).any() and (poss == 1).any()
    nhi, nlo = layer.P[layer.cur]
    ratio = _out_checks(None, (nhi, nlo), layer.dots, y, bound, sw)
    mask = layer.local_entity_mask * layer.possible if reason_kb else layer.local_entity_mask
    dbound = bound @ sw.to(F64).abs() + (D + 2) * U * ((y.abs() + bound) @ sw.to(F64).abs()) + 1e-30
    rd = _softmax_check(dist, s, sb, mask, dbound, B, N)
    print("NSM layer D=%d weighted=%d reason_kb=%d: max err/bound h %.3g dots %.3g dist %.3g"
          % (D, weighted, reason_kb, *ratio, rd))


class _HoldEveryCall:
    """Stands in for ops.linear_tc_planes: the A operand, W, bias and w_score of every call are captured before it
    runs, and what it wrote is held to float64 right after.  Column slices of a wide call are held as part of it, and
    grouped-order calls (the fused-layer order) by test_dense_pair_gpu.py / test_dense_layer_gpu.py."""

    def __init__(self, monkeypatch):
        self.orig = ops.linear_tc_planes
        self.inner = False
        self.ratios = []
        self.a_max = []
        monkeypatch.setattr(ops, "linear_tc_planes", self)

    def __call__(self, a_hi, a_lo, K, W, bias, out=None, out_planes=None, w_score=None, dots=None, relu=True,
                 k_seg=0, k_seg_pitch=0, single_ok=False, k_grouped=False, k_order=False):
        kw = dict(out=out, out_planes=out_planes, w_score=w_score, dots=dots, relu=relu, k_seg=k_seg,
                  k_seg_pitch=k_seg_pitch, single_ok=single_ok, k_grouped=k_grouped, k_order=k_order)
        if self.inner or k_grouped:
            return self.orig(a_hi, a_lo, K, W, bias, **kw)
        single = bool(ops.ACT_BF16 and single_ok)
        A = _operand(a_hi, a_lo, K, k_seg, k_seg_pitch, single)
        W0 = W.detach().clone()
        b0 = None if bias is None else bias.detach().clone()
        s0 = None if w_score is None else w_score.detach().clone()
        self.inner = True
        try:
            res = self.orig(a_hi, a_lo, K, W, bias, **kw)
        finally:
            self.inner = False
        torch.cuda.synchronize()
        y, bound = _ref(A, W0, b0, relu, K, single)
        self.ratios.append(_out_checks(out, out_planes, dots, y, bound, s0))
        self.a_max.append(A.abs().max(0)[0])
        return res


@pytest.mark.parametrize("name,single", [("rearev_d50_pads", False), ("rearev_posemb", False), ("rearev_hub", False),
                                         ("rearev_d50_pads", True), ("nsm_small", False), ("nsm_reason_kb", False)])
def test_every_gemm_of_rearev_and_nsm_forwards_vs_fp64(name, single, monkeypatch):
    """Full ReaRev and NSM forwards of the reference goldens: every split-bf16 GEMM (relation features, relation
    tables, sparse-prior GEMM, dense layers, NSM's two-segment GEMM) held to float64 of the operand it read."""
    from golden_io import Golden
    from test_parity_gpu import build_model
    g = Golden(name)
    m = build_model(g)
    hold = _HoldEveryCall(monkeypatch)
    with _options(single=single):
        m(g.batch)
    assert len(hold.ratios) >= 3
    worst = np.max(np.array(hold.ratios), 0)
    print("%s single=%d: %d GEMMs, max err/bound out %.3g dots %.3g" % (name, single, len(hold.ratios), *worst))


@pytest.mark.parametrize("name", ["graft_small", "graft_d50_sharp", "graft_hub_clamp"])
def test_every_gemm_of_graftnet_forwards_vs_fp64(name, monkeypatch):
    """GraftNet forwards of the reference goldens: per layer the head GEMM over the h window, the f2e GEMM over
    [sum_v | indeg | h] with the per-call weight [W_tail | b_tail e_0 | W_self] writing planes into segment 4, and the
    e2e GEMM over the [h | q2e | f2e] window with fact_scale folded into its per-call weight, each held to float64 of
    the planes as gr_graft_aggregate left them.  graft_hub_clamp's hub has more than 2048 in-facts: the indeg column
    exceeds 256, so its value needs the lo plane."""
    from test_graftnet_host import load_model
    m, g = load_model(name, "cuda")
    m = m.cuda()
    hold = _HoldEveryCall(monkeypatch)
    m(g.batch)
    D = m.entity_dim
    assert len(hold.ratios) >= 3 * m.num_layer
    if name == "graft_hub_clamp":
        assert max(float(a[D]) for a in hold.a_max if a.numel() == 3 * D) > 256
    worst = np.max(np.array(hold.ratios), 0)
    print("%s: %d GEMMs, max err/bound out %.3g dots %.3g" % (name, len(hold.ratios), *worst))


@pytest.mark.parametrize("name", ["graft_small", "graft_d50_sharp", "graft_hub_clamp"])
def test_graftnet_layer_vs_fp64(name, monkeypatch):
    """Every GraftLayer.forward of a GraftNet forward held to fp64_ref.graft_layer (graft_gnn.py:111-153) from the
    inputs the layer read: h from its planes, the prior, the query, the relation features and the attention W_tilde and
    E the kernels left.  So the per-call weights are checked as well as the GEMMs: [W_tail | b_tail e_0 | W_self] (the
    per-fact bias through the indeg column) and fact_scale folded into e2e's f2e block.  Checked: h' (fp32 and the next
    planes, bit for bit their split), the score dots, the score softmax, the next prior d' and query_emb.  graft_hub_clamp
    has a hub with more than 256 in-facts, whose indeg column needs the lo plane.

    Bound: every rounding along the layer is relative to the elementwise envelope fp64_ref.graft_layer_scale, and an
    error of e times the envelope of an intermediate stays within e times the envelope downstream.  Summed over the
    stages: the graft aggregation's sums of at most n terms and the divisions, (2n + 16) u; three GEMMs (test bound of
    this file, K <= 3 Dp); the bf16 splits of h, f2e and the aggregated planes, 4 x 2^-17; the query's seed_retrieve
    and SIMT e2q linear over 3 D + N terms, (3 D + N + 8) u."""
    from test_graftnet_host import load_model
    from test_gemm_layouts_host import graft_lin
    m, g = load_model(name, "cuda")
    m = m.cuda()
    local_entity, _qe, _kb, graft, _q, kb_fact_rel = g.batch[:6]
    B, N = local_entity.shape
    D = m.entity_dim
    layer = m.reasoning
    Dp = _r16(D)
    (e2f_b, e2f_f, e2f_e, _v0), (f2e_b, f2e_e, f2e_f, _v1) = graft
    n = max(np.bincount(np.asarray(f2e_b) * N + np.asarray(f2e_e)).max(),
            np.bincount(np.asarray(e2f_b) * np.asarray(kb_fact_rel).shape[1] + np.asarray(e2f_f)).max())
    if name == "graft_hub_clamp":
        assert n > 256
    K = 3 * Dp
    eps = (2 * n + 16) * U + 3 * (SPLIT + (3 * K + 2) * 2.0 ** -23) + 4 * 2.0 ** -17 + (3 * D + N + 8) * U
    rel_seen = {}
    ratios = []
    init, fwd = modules.GraftLayer.init_reason, modules.GraftLayer.forward

    def init_reason(self, db, rel, *a):
        rel_seen["rel"] = rel.detach().to(F64)
        return init(self, db, rel, *a)

    def forward(self, dist, query_node, step, last):
        hi, lo = self.P[self.cur]
        h = hi[:, 2 * Dp:2 * Dp + D].to(F64) + lo[:, 2 * Dp:2 * Dp + D].to(F64)
        args = (h, dist.to(F64), query_node.reshape(B, D).to(F64),
                rel_seen["rel"][torch.as_tensor(np.asarray(kb_fact_rel), device=DEV)], self.W_tilde.reshape(B, -1).to(F64),
                self.E.to(F64), (e2f_b, e2f_f, e2f_e), (f2e_b, f2e_e, f2e_f))
        args = tuple(a.cpu() if isinstance(a, torch.Tensor) else a for a in args)
        rest = (graft_lin(self, step), self.score_func.weight.detach().to(F64).view(-1), self.pagerank_lambda,
                self.fact_scale)
        rest = ({k: (W.cpu(), b.cpu()) for k, (W, b) in rest[0].items()}, rest[1].cpu()) + rest[2:]
        score, d_next, query_emb = fwd(self, dist, query_node, step, last)
        torch.cuda.synchronize()
        y, s, nd, q = (t.to(DEV) for t in R.graft_layer(*args, *rest))
        sy, ss, snd, sq = (t.to(DEV) for t in R.graft_layer_scale(*args, *rest))
        sw = self.score_func.weight.detach().view(-1)
        bound = eps * sy + 1e-30
        nhi, nlo = self.P[self.cur]
        r = _out_checks(self.h32, (nhi[:, 2 * Dp:], nlo[:, 2 * Dp:]), self.dots, y, bound, sw)
        derr = (d_next.to(F64) - nd).abs()
        dbound = eps * snd + 1e-30
        assert (derr <= dbound).all(), (derr / dbound).max().item()
        rr = [*r, (derr / dbound).max().item()]
        if query_emb is not None:
            qerr = (query_emb.to(F64) - q).abs()
            qbound = eps * sq + 1e-30
            assert (qerr <= qbound).all(), (qerr / qbound).max().item()
            rr.append((qerr / qbound).max().item())
        dots_bound = bound @ sw.to(F64).abs() + (D + 2) * U * ((y.abs() + bound) @ sw.to(F64).abs()) + 1e-30
        rr.append(_softmax_check(score, s, self.score_func.bias.detach(), self.local_entity_mask, dots_bound, B, N))
        ratios.append(max(rr))
        return score, d_next, query_emb

    monkeypatch.setattr(modules.GraftLayer, "init_reason", init_reason)
    monkeypatch.setattr(modules.GraftLayer, "forward", forward)
    m(g.batch)
    assert len(ratios) == m.num_layer
    print("%s: GraftLayer.forward x %d, max err/bound %.3g" % (name, len(ratios), max(ratios)))
