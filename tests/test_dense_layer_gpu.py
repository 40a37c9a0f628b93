"""GPU: the two kernels every dense-prior ReaRev layer at D = 200 runs on -- gr_aggregate_dual_abs
(csrc/aggregate_abs.cu, in every agg_abs_ws mode, two planes and hi-only) and gr_fused_layer (csrc/fused_layer.cu)
-- against the float64 references of tests/fp64_ref.py, element by element, at their edge shapes: question
boundaries inside tiles, the slow paths of overflowing edge slices, and several tiles per persistent CTA.

Bounds (u = 2^-24).

Aggregation.  Per (row, direction, column) the kernel sums the row's n in-edges into two fp32 FMA chains,
S = sum c v and Q = sum c |v|, with c = w (w p) rounded twice, and emits y = (x+/2)(Q + S) + (x-/2)(Q - S) where
x+ = relu(x), x- = relu(-x).  One of x+, x- is 0, so y is one product: with A = sum |c| |v| the two chains are each
off by n u A, the two roundings of c move S and Q by 2 u A each, the add Q +- S rounds once (u 2A) and the product
once (u |y|): |y - ref| <= (n + 4) u |x| A (1 + O(n u)), where |x| A is fp64_ref.aggregate_abs.  The tests use
(2n + 8) u of aggregate_abs, twice that.  The hi/lo planes are hi = bf16(y), lo = bf16(y - hi), y - hi exact: with
2^e <= |y| < 2^(e+1), |lo| < 2^(e-8) (half an ulp of hi) and lo rounds by at most half its own ulp, 2^(e-17), so hi + lo
is off y by at most 2^-17 |y|; the tests add 2^-17 |ref|.  This term is tight: it sets the largest error / bound
ratios (0.88-0.94 on an H100 80GB HBM3).  Where the fp64 value is exactly 0 every term is c = 0 or has
v x <= 0; then the two chains run negated operations (or add exact zeros), Q + S or Q - S is exactly 0, and so is
the output.

Fused layer.  pre = sum_k A_k W_k over K = (2I + 1) pitch columns as A_hi W_hi + A_hi W_lo + A_lo W_hi, fp32
accumulation on the tensor core, then + bias and relu.  Against s = fp64_ref.rearev_layer_scale = |W| |A| + |b|:
  * the A operand: the aggregated columns as above, ((2n + 8) u + 2^-17) of their scale with n the larger in-degree of
    the row; the h columns are split into bf16 hi/lo, 2^-17 |h|;
  * the W split, 2^-17 |W|, and the dropped A_lo W_lo term, 2^-8 |A| 2^-8 |W|;
  * the accumulation.  wgmma's internal accumulation order and rounding are not documented.  ASSUMED (not measured):
    each of the 3K products (exact in fp32) is added with one rounding of at most 2^-23 relative to the running sum
    (one ulp: truncation allowed), so the sum is off by at most 3K 2^-23 of the sum of |terms| <= s;
  * the bias add, u |pre|.
So |y - ref| <= ((2n + 8) u + 2^-15 + (3K + 2) 2^-23) s; relu does not enlarge an error.  The planes are the bf16
split of the fp32 output, bit for bit.  The score dot sums N_out fp32 products in an FMA chain and a 2-step shuffle
tree: (N_out + 2) u of |y| |w_score|, plus |w_score| times the bound on y.

A dropped, repeated or misplaced edge, a wrong question's instructions, a stale accumulator or a stale coefficient
moves an element by a sizeable fraction of its scale, far outside these bounds; at the hub rows one planted edge with
a dominant coefficient sits exactly where a slow path starts."""
import math

import numpy as np
import pytest
import torch

from gnn_rag_b200 import ops

import fp64_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
F64 = torch.float64
BF16 = torch.bfloat16
SEGP = 208             # segment pitch of the hot shape (gr_aggregate_dual_abs specialises D = 200, pitch 208)
SENT = 7.0             # what every output buffer holds before the call: unwritten elements keep it
BIG = 30.0             # weight of a planted hub edge
HUB = 0                # the hub row: the first row of tile 0 in every tile geometry (64, 72 and 56 rows)
BM = 128               # rows per fused-layer tile
ABS_TILE_ROWS = {1: 64, 2: 72, 3: 56}      # persistent abs kernels: rows per tile (mode 2 at N < 72 uses 64)
ABS_CTAS_PER_SM = {1: 2, 2: 2, 3: 1}


def _r16(n):
    return (n + 15) // 16 * 16


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def _graph(rs, B, N, E, R1):
    """E random facts inside every question: numpy (heads, rels, tails) with global node rows."""
    h = (rs.randint(0, N, size=(B, E)) + np.arange(B)[:, None] * N).ravel()
    t = (rs.randint(0, N, size=(B, E)) + np.arange(B)[:, None] * N).ravel()
    r = rs.randint(0, R1 - 1, size=len(h))          # relation R1 - 1 is reserved for planted edges
    return h, r, t


def _build(h, r, t, B, N, R1):
    g = ops.csr_build(*(_t(a, torch.int64) for a in (h, r, t)), B, N, R1)
    g.check_status()
    Nt = B * N
    deg_t = np.bincount(t, minlength=Nt)
    deg_h = np.bincount(h, minlength=Nt)
    return g, deg_t, deg_h


def _weights(rs, g, F, planted=()):
    w = rs.uniform(0.2, 1.5, size=F).astype(np.float32)
    w[rs.rand(F) < 0.1] = 0.0                       # exact zeros: rows whose edges all carry c = 0
    w[list(planted)] = BIG
    wd = _t(w)
    return wd, ops.gather_f32(wd, g.fact_t), ops.gather_f32(wd, g.fact_h)


def _priors(rs, B, N):
    dense = torch.softmax(_t(rs.randn(B, N)), 1)
    onehot = np.zeros((B, N), np.float32)
    onehot[np.arange(B), rs.randint(0, N, size=B)] = 1.0
    return {"dense": dense, "onehot": _t(onehot)}


def _tables(rs, R1, D):
    tf, ti = _t(rs.randn(R1, D)), _t(rs.randn(R1, D))
    for tab in (tf, ti):                            # the planted relation's row is not small anywhere
        tab[R1 - 1] = torch.where(tab[R1 - 1] < 0, -1.0, 1.0) * tab[R1 - 1].abs().clamp_min(0.5)
    return tf, ti


# ---- gr_aggregate_dual_abs -------------------------------------------------------------------------------------------

def _abs_ref(tf, ti, ins, prior, facts, w, deg_t, deg_h):
    """fp64 [Nt, I, 2, D] value and bound of every aggregated element (direction 0 = fwd, 1 = inv)."""
    B, I, D = ins.shape
    Nt = prior.numel()
    w64 = None if w is None else w.to(F64)
    wants, bounds = [], []
    for tab, direction, deg in ((tf, "fwd", deg_t), (ti, "inv", deg_h)):
        args = (tab.to(F64), ins.to(F64), prior.to(F64), *facts, w64, direction)
        want = R.aggregate(*args).view(Nt, I, D)
        scale = R.aggregate_abs(*args).view(Nt, I, D)
        n = _t(deg, F64).view(Nt, 1, 1)
        wants.append(want)
        bounds.append((2 * n + 8) * U * scale + 2.0 ** -17 * want.abs())
    return torch.stack(wants, 2), torch.stack(bounds, 2)


def _run_abs(g, prior, pf, pi, ins, w_t, w_h, mode, hi_only, out_col0, ld):
    Nt = g.B * g.N
    hi = torch.full((Nt, ld), SENT, dtype=BF16, device=DEV)
    lo = hi.clone()
    ops.set_option("agg_abs_ws", mode)
    ops.ACT_BF16 = hi_only
    try:
        ops.aggregate_dual_abs(g, prior, pf, pi, ins, (hi, lo), out_col0, SEGP, w_t, w_h)
        torch.cuda.synchronize()
    finally:
        ops.ACT_BF16 = False
        ops.set_option("agg_abs_ws", 2)
    return hi, lo


def _check_abs(hi, lo, want, bound, out_col0):
    """Every segment of hi + lo against fp64; pads 200..207 zero, exact zeros exact, h segment and tail untouched.
    Returns the largest error / bound."""
    Nt, I, _, D = want.shape
    end = out_col0 + 2 * I * SEGP
    for p in (hi, lo):
        assert (p[:, :out_col0] == SENT).all() and (p[:, end:] == SENT).all()
        assert (p[:, out_col0:end].view(Nt, I, 2, SEGP)[..., D:] == 0).all()
    got = (hi[:, out_col0:end].to(F64) + lo[:, out_col0:end].to(F64)).view(Nt, I, 2, SEGP)[..., :D]
    err = (got - want).abs()
    assert (err <= bound).all(), (err / bound.clamp_min(1e-300)).max().item()
    zero = want == 0
    assert zero.any() and (~zero).any()
    assert (got[zero] == 0).all()
    return (err[~zero] / bound[~zero]).max().item()


def _bits(p):
    return p.view(torch.int16)


def _abs_all_modes(g, prior, pf, pi, ins, w_t, w_h, want, bound, modes, out_col0, ld):
    """Two-plane runs of every mode in `modes` (all bit-identical and within the fp64 bound), then hi-only runs of
    the persistent modes: the hi plane bit for bit the two-plane one, the lo plane untouched."""
    first, ratio = None, 0.0
    for mode in modes:
        hi, lo = _run_abs(g, prior, pf, pi, ins, w_t, w_h, mode, False, out_col0, ld)
        ratio = max(ratio, _check_abs(hi, lo, want, bound, out_col0))
        if first is None:
            first = (hi, lo)
        assert torch.equal(_bits(hi), _bits(first[0])) and torch.equal(_bits(lo), _bits(first[1])), mode
    for mode in (m for m in modes if m != 0):
        hi, lo = _run_abs(g, prior, pf, pi, ins, w_t, w_h, mode, True, out_col0, ld)
        assert torch.equal(_bits(hi), _bits(first[0])), ("hi-only", mode)     # mode 3 falls back to mode 2's kernel
        assert (lo == SENT).all()
    return ratio


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("N", [64, 65, 67, 71, 72, 73])
@pytest.mark.parametrize("I", [1, 2, 3, 5])
def test_aggregate_dual_abs_vs_fp64(I, N, weighted):
    """B = 16 questions of N nodes: 72-row tiles would span three questions at N = 65 and 67 (so N < 72 takes the
    64-row tiles), 56-row tiles of mode 3 span two.  Row 0 is a hub with 1100 more in-edges per direction; with
    weights, its in-edges at positions 512 (mode 3's staging cap) and 1024 (the others') carry a dominant coefficient.
    I = 5 runs as two launches (4 + 1 instructions)."""
    rs = np.random.RandomState(1000 * I + 10 * N + weighted)
    B, E, R1, D = 16, 150, 23, 200
    h, r, t = _graph(rs, B, N, E, R1)
    src = rs.randint(1, N, size=1100)                            # question 0, never the hub itself
    h = np.concatenate([h, src, np.full(1100, HUB)])
    t = np.concatenate([t, np.full(1100, HUB), src])
    r = np.concatenate([r, rs.randint(0, R1 - 1, size=2200)])
    planted = [np.flatnonzero(ends == HUB)[k] for ends in (t, h) for k in (512, 1024)]   # fwd: tail CSR, inv: head
    r[planted] = R1 - 1
    g, deg_t, deg_h = _build(h, r, t, B, N, R1)
    assert deg_t[HUB] > 1024 and deg_h[HUB] > 1024
    wd = w_t = w_h = None
    if weighted:
        wd, w_t, w_h = _weights(rs, g, len(h), planted)
    tf, ti = _tables(rs, R1, D)
    pf, pi = ops.pad_table256(tf), ops.pad_table256(ti)
    ins = _t(rs.randn(B, I, D))
    facts = tuple(_t(a, torch.int64) for a in (h, r, t))
    out_col0 = SEGP                                              # the h segment leads the row
    ld = out_col0 + 2 * I * SEGP + 16
    for kind, prior in _priors(rs, B, N).items():
        want, bound = _abs_ref(tf, ti, ins, prior, facts, wd, deg_t, deg_h)
        if weighted and kind == "dense":
            for k, f in enumerate(planted):
                d = k // 2
                s = (h, t)[d][f]
                edge = BIG * BIG * float(prior.view(-1)[s]) * torch.relu((tf, ti)[d][R1 - 1].to(F64) * ins[0].to(F64))
                assert (edge > 100 * bound[HUB, :, d]).any()   # one planted edge is far outside the bound
        ratio = _abs_all_modes(g, prior, pf, pi, ins, w_t, w_h, want, bound, (0, 1, 2, 3), out_col0, ld)
        print("gr_aggregate_dual_abs I=%d N=%d weighted=%d %s: max err/bound %.3g" % (I, N, weighted, kind, ratio))


# ---- gr_fused_layer ----------------------------------------------------------------------------------------------------

def _quad_total(deg, tile):
    """Entries of one tile and direction in the quad-ELL form: 4 x the largest in-degree of each 4-row quad."""
    d = np.zeros(BM, np.int64)
    seg = deg[tile * BM:(tile + 1) * BM]
    d[:len(seg)] = seg
    return 4 * int(d.reshape(BM // 4, 4).max(1).sum())


def _controlled_facts(rs, B, N, R1, tiles):
    """Random facts, except that the rows of each (tile, hub) in `tiles` (question 0) get exactly these in-degrees in
    both directions: `hub` on the tile's first row, (row % 3) on the others -- so every other quad's largest in-degree is
    2 and the tile's quad-ELL total is 4 (hub + 62)."""
    h, r, t = _graph(rs, B, N, 3 * N, R1)
    ctrl = np.zeros(B * N, bool)
    for tile, _ in tiles:
        ctrl[tile * BM:(tile + 1) * BM] = True
    keep = ~ctrl[h] & ~ctrl[t]
    free = np.flatnonzero(~ctrl[:N])
    hs, ts = [h[keep]], [t[keep]]
    for tile, hub in tiles:
        deg = np.arange(BM) % 3
        deg[0] = hub
        dst = np.repeat(tile * BM + np.arange(BM), deg)
        src = rs.choice(free, size=len(dst))
        hs += [src, dst]                                         # in-edges of the tail CSR, then of the head CSR
        ts += [dst, src]
    h, t = np.concatenate(hs), np.concatenate(ts)
    return h, rs.randint(0, R1 - 1, size=len(h)), t


def _fused_ref(h, prior, tf, ti, ins, W, bias, wsc, facts, w, deg_t, deg_h, P):
    I = ins.shape[1]
    d64 = lambda x: None if x is None else x.to(F64)                     # noqa: E731
    args = (h.to(F64), prior.to(F64), tf.to(F64), ti.to(F64), ins.to(F64), W.to(F64), d64(bias))
    y, s = R.rearev_layer(*args, d64(wsc), facts, d64(w))
    scale = R.rearev_layer_scale(*args, facts, d64(w))
    n = _t(np.maximum(deg_t, deg_h), F64)[:, None]
    K = (2 * I + 1) * P
    bound = ((2 * n + 8) * U + 2.0 ** -15 + (3 * K + 2) * 2.0 ** -23) * scale + 1e-30
    return y, s, bound


def _check_fused(g, prior, tf, ti, pf, pi, ins, h, hp, W, bias, wsc, facts, wd, w_t, w_h, deg_t, deg_h, P):
    """One gr_fused_layer call (fp32 output, planes and dots) against fp64; returns the largest error / bound of the
    output and of the dots."""
    M, n_out = h.shape[0], W.shape[0]
    n16 = _r16(n_out)
    cbuf = torch.full((M, n_out + 8), SENT, device=DEV)
    out = cbuf[:, :n_out]
    chi = torch.full((M, n16 + 16), SENT, dtype=BF16, device=DEV)
    clo = chi.clone()
    dots = torch.full((2 * M,), SENT, device=DEV)
    ops.fused_layer(g, prior, pf, pi, ins, hp, P, W, bias, out=out, out_planes=(chi, clo), w_score=wsc, dots=dots,
                    relu=True, w_t=w_t, w_h=w_h)
    torch.cuda.synchronize()
    y, s, bound = _fused_ref(h, prior, tf, ti, ins, W, bias, wsc, facts, wd, deg_t, deg_h, P)
    assert (cbuf[:, n_out:] == SENT).all()                      # nothing past N_out in the fp32 output
    err = (out.to(F64) - y).abs()
    assert (err <= bound).all(), (err / bound).max().item()
    hi_want = out.to(BF16)                                       # the planes are the bf16 split of the fp32 output
    assert torch.equal(_bits(chi[:, :n_out]), _bits(hi_want))
    assert torch.equal(_bits(clo[:, :n_out]), _bits((out - hi_want.float()).to(BF16)))
    assert ((chi.to(F64) + clo.to(F64))[:, :n_out] - y).abs().le(bound + 2.0 ** -17 * y.abs()).all()
    for p in (chi, clo):
        assert (p[:, n_out:n16] == 0).all() and (p[:, n16:] == SENT).all()   # pad columns 0, nothing past round16
    aw = wsc.to(F64).abs()
    dbound = bound @ aw + (n_out + 2) * U * ((y.abs() + bound) @ aw) + 1e-30
    derr = (dots[:M].to(F64) + dots[M:].to(F64) - s).abs()
    assert (dots[M:] == 0).all()
    assert (derr <= dbound).all(), (derr / dbound).max().item()
    return (err / bound).max().item(), (derr / dbound).max().item()


def _layer_inputs(rs, M, D, P, I):
    h = _t(rs.randn(M, D))
    h_hi = torch.zeros(M, P + 48, dtype=BF16, device=DEV)
    h_lo = torch.zeros(M, P + 48, dtype=BF16, device=DEV)
    ops.split_bf16(h, h_hi, h_lo)
    h_hi[:, P:] = float("nan")                                   # past the segment pitch: never read
    h_lo[:, P:] = float("nan")
    W = _t(rs.randn(D, (2 * I + 1) * D) / np.sqrt(D))
    bias = _t(rs.randn(D) * 0.1)
    wsc = _t(rs.randn(D))
    return h, (h_hi, h_lo), W, bias, wsc


@pytest.mark.parametrize("N", [128, 129, 2000])
@pytest.mark.parametrize("D,P", [(200, 208), (72, 80)])
@pytest.mark.parametrize("I", [1, 2])
def test_fused_layer_vs_fp64(I, D, P, N):
    """N = 128: tiles are questions; N = 129: every tile but the first starts inside a question; N = 2000 (B = 3):
    tile 15 switches question at row 80, tile 1 has a quad-ELL total of exactly 1024 entries per direction (the
    staged fast path) and tile 3 has 1028 (the CSR slow path).  One graph object is run unweighted, weighted, then
    weighted and unweighted again under a second prior (one-hot): a stale quad-ELL form or coefficient pass shows."""
    rs = np.random.RandomState(100 * I + D + N)
    R1 = 17
    if N == 2000:
        B = 3
        h, r, t = _controlled_facts(rs, B, N, R1, [(1, 194), (3, 195)])
    else:
        B = 5
        h, r, t = _graph(rs, B, N, 3 * N, R1)
    g, deg_t, deg_h = _build(h, r, t, B, N, R1)
    if N == 2000:
        for deg in (deg_t, deg_h):
            assert _quad_total(deg, 1) == 1024 and _quad_total(deg, 3) == 1028
    assert ops.fused_layer_supported(N, D, P, I, D)
    M = B * N
    wd, w_t, w_h = _weights(rs, g, len(h))
    tf, ti = _tables(rs, R1, D)
    pf, pi = ops.pad_table256(tf), ops.pad_table256(ti)
    ins = _t(rs.randn(B, I, D))
    facts = tuple(_t(a, torch.int64) for a in (h, r, t))
    h_in, hp, W, bias, wsc = _layer_inputs(rs, M, D, P, I)
    priors = _priors(rs, B, N)
    for weighted, kind in ((False, "dense"), (True, "dense"), (True, "onehot"), (False, "onehot")):
        ww = (wd, w_t, w_h) if weighted else (None, None, None)
        ratio = _check_fused(g, priors[kind], tf, ti, pf, pi, ins, h_in, hp, W, bias, wsc, facts, *ww, deg_t, deg_h, P)
        print("gr_fused_layer I=%d D=%d N=%d weighted=%d %s: max err/bound out %.3g dots %.3g"
              % (I, D, N, weighted, kind, *ratio))


# ---- several tiles per CTA -------------------------------------------------------------------------------------------

def test_several_tiles_per_cta_vs_fp64():
    """B = 32 questions of N = 2000 nodes and ~6000 facts each (the size of a cfg2 question): every persistent CTA of
    the fused kernel and of abs modes 1, 2, 3 works through at least 3 tiles, so the double-buffered descriptors wrap
    and every per-tile state is set up again.  Checked as above: the fused layer, and abs modes 1-3 with two planes
    and hi-only (bit-identical to each other)."""
    rs = np.random.RandomState(32)
    B, N, E, R1, D, P, I = 32, 2000, 6000, 61, 200, 208, 2
    M = B * N
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ngroups = math.ceil(math.ceil(M / BM) / 2)                  # clusters of 2 CTAs take pairs of tiles
    assert ngroups >= 3 * min(ngroups, sms // 2)
    for mode, rows in ABS_TILE_ROWS.items():
        tiles = math.ceil(M / rows)
        assert tiles >= 3 * min(tiles, ABS_CTAS_PER_SM[mode] * sms), mode
    h, r, t = _graph(rs, B, N, E, R1)
    g, deg_t, deg_h = _build(h, r, t, B, N, R1)
    tf, ti = _tables(rs, R1, D)
    pf, pi = ops.pad_table256(tf), ops.pad_table256(ti)
    ins = _t(rs.randn(B, I, D))
    facts = tuple(_t(a, torch.int64) for a in (h, r, t))
    prior = _priors(rs, B, N)["dense"]
    h_in, hp, W, bias, wsc = _layer_inputs(rs, M, D, P, I)
    ratio = _check_fused(g, prior, tf, ti, pf, pi, ins, h_in, hp, W, bias, wsc, facts, None, None, None, deg_t, deg_h,
                         P)
    print("gr_fused_layer B=%d N=%d: max err/bound out %.3g dots %.3g" % (B, N, *ratio))
    want, bound = _abs_ref(tf, ti, ins, prior, facts, None, deg_t, deg_h)
    out_col0 = SEGP
    ratio = _abs_all_modes(g, prior, pf, pi, ins, None, None, want, bound, (1, 2, 3), out_col0,
                           out_col0 + 2 * I * SEGP)
    print("gr_aggregate_dual_abs B=%d N=%d: max err/bound %.3g" % (B, N, ratio))
