"""GPU: the sparse-prior layer kernels (csrc/frontier.cu) and gr_masked_softmax against the float64 references of
tests/fp64_ref.py.

Error bounds.  For a listed row the fix-up sums, per direction, n in-edges of that row into two fp32 accumulators
(A = sum c relu(v), S = sum c v) and forms A - S, each edge coefficient c = w*(w*p) carrying two roundings: an
aggregated element is off by at most (2n + 8) u times its |.|-scale (u = 2^-24).  The e2e dot then sums Kd = (2I+1)D
products per output, ceil(Kd/32) per lane plus a 5-step shuffle tree and the bias: (Kd/32 + 8) u of |W| |x| + |b|.
Both are taken against ``fp64_ref.rearev_layer_scale``, which is exactly |W| [|h| | aggregate_abs] + |b|; relu does
not enlarge an error.  The score dot adds (D + 2) u of |y| |w_score| plus |w_score| times the bound on y.  A dropped
or doubled edge, a swapped direction segment or a wrong weight moves an element by a sizeable fraction of its scale,
far outside these bounds."""
import math

import numpy as np
import pytest
import torch

from gnn_rag_b200 import _lib, ops

import fp64_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
F64 = torch.float64


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _r16(n):
    return (n + 15) // 16 * 16


def _facts(rs, B, N, E, R1, n_real=None, hub=0, isolated=()):
    """Random facts inside every question (plus a self-loop on every real node, as the loader adds them).
    ``hub``: extra in-edges into local node 5 of question 0 (more than one 32-edge staging round).  ``isolated``:
    (question, local node) pairs that get no edge at all."""
    nr = N if n_real is None else n_real
    hs, rl, ts = [], [], []
    for b in range(B):
        h = rs.randint(0, nr, size=E)
        t = rs.randint(0, nr, size=E)
        loops = np.arange(nr)
        h, t = np.concatenate([h, loops]), np.concatenate([t, loops])
        if b == 0 and hub:
            hh = rs.randint(0, nr, size=hub)
            hh[::10] = 0                                          # the seed feeds the hub in every staging round
            h = np.concatenate([h, hh])
            t = np.concatenate([t, np.full(hub, 5)])
        r = rs.randint(0, R1, size=len(h))
        r[:2] = [0, R1 - 1]
        keep = np.ones(len(h), dtype=bool)
        for (qb, node) in isolated:
            if qb == b:
                keep &= (h != node) & (t != node)
        hs.append(h[keep] + b * N)
        ts.append(t[keep] + b * N)
        rl.append(r[keep])
    return np.concatenate(hs), np.concatenate(rl), np.concatenate(ts)


def _graph(heads, rels, tails, B, N, R1):
    g = ops.csr_build(*(torch.from_numpy(a).to(DEV) for a in (heads, rels, tails)), B, N, R1)
    g.check_status()
    return g


def _weights(rs, g, F, zeros=True):
    """Arbitrary per-fact weights (some exactly zero), permuted into both CSR orders with gather_f32."""
    w = rs.uniform(0.2, 1.5, size=F).astype(np.float32)
    if zeros:
        w[rs.rand(F) < 0.1] = 0.0
    wd = torch.from_numpy(w).to(DEV)
    w_t, w_h = ops.gather_f32(wd, g.fact_t), ops.gather_f32(wd, g.fact_h)
    assert torch.equal(w_t[:F], wd[g.fact_t[:F].long()]) and torch.equal(w_h[:F], wd[g.fact_h[:F].long()])
    return wd, w_t, w_h


def _frontier_set(heads, tails, prior):
    p = prior.reshape(-1)
    return set(tails[p[heads] != 0].tolist()) | set(heads[p[tails] != 0].tolist())


def _indeg(heads, tails, Nt):
    return np.maximum(np.bincount(tails, minlength=Nt), np.bincount(heads, minlength=Nt))


def _planes(h, pitch):
    Nt, D = h.shape
    hi = torch.zeros(Nt, pitch, dtype=torch.bfloat16, device=DEV)
    lo = torch.zeros_like(hi)
    ops.split_bf16(h, hi, lo)
    return hi, lo


def _priors(B, N, isolated_node):
    """q0: one-hot seed; q1: three seeds of 1/3; q2: no seed; q3: a seed on a node without edges; further
    questions: one-hot seeds again."""
    p = np.zeros((B, N), dtype=np.float32)
    p[:, 0] = 1.0
    p[1, :3] = 1.0 / 3
    p[2, :] = 0.0
    if B > 3:
        p[3, :] = 0.0
        p[3, isolated_node] = 1.0
    return p


def _run_rows(g, prior, Nt):
    rows = torch.full((Nt,), -7, dtype=torch.int32, device=DEV)
    count = torch.full((1,), 12345, dtype=torch.int32, device=DEV)
    ops.frontier_rows(g, prior, rows, count)
    return rows, count


def _check_rows(rows, count, want):
    c = int(count.item())
    listed = rows[:c].cpu().numpy()
    assert c == len(want)
    assert len(set(listed.tolist())) == c                         # no duplicates
    assert set(listed.tolist()) == want
    assert (rows[c:] == -7).all()                                 # nothing written past the count
    return listed


class _Layer:
    """Inputs of one sparse-prior layer and its float64 reference."""

    def __init__(self, seed, D, I, B=4, N=96, E=150, R1=37, weights=True, w_layout="plain", hub=100, n_real=None,
                 prior=None, bias=True):
        rs = np.random.RandomState(seed)
        self.B, self.N, self.D, self.I, self.Nt = B, N, D, I, B * N
        self.Kd = Kd = (2 * I + 1) * D
        iso = (3, N - 1)
        self.heads, self.rels, self.tails = _facts(rs, B, N, E, R1, n_real=n_real, hub=hub, isolated=(iso,))
        self.F = len(self.heads)
        self.g = _graph(self.heads, self.rels, self.tails, B, N, R1)
        self.w = self.w_t = self.w_h = None
        if weights:
            self.w, self.w_t, self.w_h = _weights(rs, self.g, self.F)
        p = _priors(B, N, iso[1]) if prior is None else prior
        self.prior = torch.from_numpy(p).to(DEV)
        f = lambda *s: torch.from_numpy(rs.randn(*s).astype(np.float32)).to(DEV)   # noqa: E731
        self.tf, self.ti = f(R1, D), f(R1, D)
        self.ins = f(B, I, D)
        h = f(self.Nt, D)
        self.hi, self.lo = _planes(h, _r16(D))
        if w_layout == "plain":
            self.W = f(D, Kd) / math.sqrt(Kd)
        elif w_layout == "strided":                               # ldw = Kd + 3 > Kd
            self.W = (f(D, Kd + 3) / math.sqrt(Kd))[:, :Kd]
        else:                                                     # one float past an 8-byte boundary: scalar loads
            self.W = (f(D * Kd + 1) / math.sqrt(Kd))[1:].view(D, Kd)
        self.bias = f(D) * 0.1 if bias else None
        self.ws = f(D) / math.sqrt(D)

    def ref(self):
        facts = tuple(torch.from_numpy(a).to(DEV) for a in (self.heads, self.rels, self.tails))
        h64 = self.hi[:, :self.D].to(F64) + self.lo[:, :self.D].to(F64)
        args = (h64, self.prior.to(F64), self.tf.to(F64), self.ti.to(F64), self.ins.to(F64), self.W.to(F64),
                None if self.bias is None else self.bias.to(F64))
        w = None if self.w is None else self.w.to(F64)
        y, s = R.rearev_layer(*args, self.ws.to(F64), facts, w)
        scale = R.rearev_layer_scale(*args, facts, w)
        n = torch.from_numpy(_indeg(self.heads, self.tails, self.Nt)).to(DEV, F64)
        gamma = (2 * n + 8 + math.ceil(self.Kd / 32) + 8) * U
        ybound = gamma[:, None] * scale + 1e-30
        sbound = (self.D + 2) * U * (y @ self.ws.to(F64).abs()) + ybound @ self.ws.to(F64).abs()
        return y, s, ybound, sbound

    def outputs(self, with_h32=True, with_dots=True):
        P = _r16(self.D)
        nhi = torch.full((self.Nt, P), 7.0, dtype=torch.bfloat16, device=DEV)
        nlo = torch.full((self.Nt, P), -5.0, dtype=torch.bfloat16, device=DEV)
        h32 = torch.full((self.Nt, self.D), -3.0, device=DEV) if with_h32 else None
        dots = torch.full((2 * self.Nt,), 9.0, device=DEV) if with_dots else None
        return nhi, nlo, h32, dots

    def fixup(self, rows, count, outs):
        nhi, nlo, h32, dots = outs
        ops.frontier_fixup(self.g, self.prior, self.tf, self.ti, self.ins, (self.hi, self.lo), self.W, self.bias,
                           self.ws, (nhi, nlo), h32, dots, rows, count, self.w_t, self.w_h)


def _check_fixup(L, listed, outs):
    nhi, nlo, h32, dots = outs
    y, s, ybound, sbound = L.ref()
    Nt, D = L.Nt, L.D
    li = torch.from_numpy(listed.astype(np.int64)).to(DEV)
    un = torch.ones(Nt, dtype=torch.bool, device=DEV)
    un[li] = False
    if h32 is not None:
        err = (h32[li].to(F64) - y[li]).abs()
        assert (err <= ybound[li]).all(), (err / ybound[li]).max().item()
        hi_want = h32[li].to(torch.bfloat16)
        assert torch.equal(nhi[li, :D].view(torch.int16), hi_want.view(torch.int16))
        lo_want = (h32[li] - hi_want.float()).to(torch.bfloat16)
        assert torch.equal(nlo[li, :D].view(torch.int16), lo_want.view(torch.int16))
        assert (h32[un] == -3.0).all()
    else:
        got = nhi[li, :D].to(F64) + nlo[li, :D].to(F64)
        err = (got - y[li]).abs()
        assert (err <= ybound[li] + 2.0 ** -17 * y[li]).all()
    assert (nhi[un] == 7.0).all() and (nlo[un] == -5.0).all()   # unlisted rows untouched
    assert (nhi[:, D:] == 7.0).all() and (nlo[:, D:] == -5.0).all()   # and no column past D
    if dots is not None:
        err = (dots[li].to(F64) - s[li]).abs()
        assert (err <= sbound[li] + 1e-30).all(), (err / sbound[li]).max().item()
        assert (dots[Nt + li] == 0).all()                        # the GEMM's second half is cleared
        assert (dots[:Nt][un] == 9.0).all() and (dots[Nt:][un] == 9.0).all()


# (D, I, weights, W layout).  33: odd D -> scalar weight loads; "offset": W one float off -> scalar loads at even Kd;
# "strided": ldw > Kd; 300 / 400: a second 256-column pass in the aggregation phase.
CASES = [
    (8, 1, True, "plain"), (8, 4, False, "strided"),
    (33, 2, True, "plain"), (33, 3, False, "offset"),
    (50, 1, True, "offset"), (50, 4, True, "plain"),
    (200, 2, True, "plain"), (200, 3, False, "strided"),
    (256, 1, False, "plain"), (256, 4, True, "offset"),
    (300, 2, True, "strided"), (300, 3, True, "plain"),
    (400, 1, True, "plain"), (400, 4, False, "offset"),
]


@pytest.mark.parametrize("D,I,weights,layout", CASES)
def test_frontier_rows_and_fixup_vs_fp64(D, I, weights, layout):
    """Per listed row: h32 and dots[row] within the bound of the module docstring, dots[Nt + row] == 0, the next
    planes are bf16_rn(h32) and bf16_rn(h32 - hi) bit for bit; unlisted rows and padding columns keep their
    sentinels.  The prior mixes a one-hot seed, a multi-seed, a question without seed and a seed without edges; the
    graph has a destination with 100+ in-edges (several 32-edge staging rounds)."""
    L = _Layer(D * 10 + I, D, I, weights=weights, w_layout=layout)
    rows, count = _run_rows(L.g, L.prior, L.Nt)
    want = _frontier_set(L.heads, L.tails, L.prior.cpu().numpy())
    assert 5 in want                                              # the hub row is on the frontier
    assert not any(2 * L.N <= r < 3 * L.N for r in want)          # no seed: no frontier row in question 2
    assert not any(3 * L.N <= r < 4 * L.N for r in want)          # isolated seed: none in question 3
    listed = _check_rows(rows, count, want)
    outs = L.outputs()
    L.fixup(rows, count, outs)
    _check_fixup(L, listed, outs)


def test_fixup_optional_outputs_absent():
    """h32 = None, dots = None, bias = None: the planes alone, bounded by the fp64 layer (+ the lo plane's 2^-17)."""
    L = _Layer(5, 50, 2, bias=False)
    rows, count = _run_rows(L.g, L.prior, L.Nt)
    listed = _check_rows(rows, count, _frontier_set(L.heads, L.tails, L.prior.cpu().numpy()))
    outs = L.outputs(with_h32=False, with_dots=False)
    L.fixup(rows, count, outs)
    _check_fixup(L, listed, outs)


def test_frontier_rows_dense_and_zero_prior():
    """A dense softmax prior lists every row with an in-edge; an all-zero prior lists nothing and writes nothing."""
    rs = np.random.RandomState(3)
    B, N = 3, 200
    heads, rels, tails = _facts(rs, B, N, 120, 20, n_real=150)
    g = _graph(heads, rels, tails, B, N, 20)
    dense = torch.softmax(torch.from_numpy(rs.randn(B, N).astype(np.float32)), 1).to(DEV)
    rows, count = _run_rows(g, dense, B * N)
    want = set(tails.tolist()) | set(heads.tolist())
    assert len(want) == 3 * 150
    _check_rows(rows, count, want)
    rows, count = _run_rows(g, torch.zeros(B, N, device=DEV), B * N)
    assert int(count.item()) == 0 and (rows == -7).all()
    # and the fix-up with count == 0 leaves every output untouched
    L = _Layer(4, 33, 2, prior=np.zeros((4, 96), dtype=np.float32))
    rows, count = _run_rows(L.g, L.prior, L.Nt)
    assert int(count.item()) == 0
    outs = L.outputs()
    L.fixup(rows, count, outs)
    _check_fixup(L, np.zeros(0, dtype=np.int64), outs)


def test_long_frontier_spans_several_grid_passes_and_is_order_independent():
    """More than 2 * SMs * 8 listed rows (the fix-up grid loops) and a last group of fewer than 8 rows; a second
    run over the reversed list gives bit-identical planes, h32 and dots."""
    n_real = 719
    B, N = 3, 720
    assert B * n_real > 2 * _sms() * 8 and (B * n_real) % 8 != 0
    rs = np.random.RandomState(8)
    dense = torch.softmax(torch.from_numpy(rs.randn(B, N).astype(np.float32)), 1).numpy()
    L = _Layer(9, 200, 2, B=B, N=N, E=900, n_real=n_real, prior=dense, hub=60)
    rows, count = _run_rows(L.g, L.prior, L.Nt)
    want = _frontier_set(L.heads, L.tails, dense)
    assert len(want) == B * n_real                                # every real node (all have a self-loop)
    listed = _check_rows(rows, count, want)
    outs = L.outputs()
    L.fixup(rows, count, outs)
    _check_fixup(L, listed, outs)
    c = int(count.item())
    rows2 = rows.clone()
    rows2[:c] = torch.flip(rows[:c], [0])
    outs2 = L.outputs()
    L.fixup(rows2, count, outs2)
    for a, b in zip(outs, outs2):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a,
                           b.view(torch.int16) if b.dtype == torch.bfloat16 else b)


def test_fixup_refuses_shapes_beyond_its_shared_memory():
    """8 rows of (2I+1)*D floats above 200 KB: GR_ERR_INVALID_ARG with a message, checked before any launch."""
    L = _Layer(6, 8, 1, B=4, N=16, E=10, hub=0)
    D, I = 512, 6
    Kd = (2 * I + 1) * D
    W = torch.zeros(D, Kd, device=DEV)
    ins = torch.zeros(L.B, I, D, device=DEV)
    tab = torch.zeros(37, D, device=DEV)
    hi, lo = _planes(torch.zeros(L.Nt, D, device=DEV), D)
    rows, count = _run_rows(L.g, L.prior, L.Nt)
    with pytest.raises(_lib.GrError, match="too large for the fix-up kernel"):
        ops.frontier_fixup(L.g, L.prior, tab, tab, ins, (hi, lo), W, None, None, (hi.clone(), lo.clone()), None,
                           None, rows, count)
    assert b"too large" in _lib.load().gr_last_error()


def _dense_model_inputs(L, mask_rs):
    """Multi-seed prior and 1/outdeg(head) weights (normalized_gnn), as the model's first layer sees them."""
    outdeg = np.bincount(L.heads, minlength=L.Nt).astype(np.float32)
    w = (1.0 / outdeg[L.heads]).astype(np.float32)
    L.w = torch.from_numpy(w).to(DEV)
    L.w_t, L.w_h = ops.gather_f32(L.w, L.g.fact_t), ops.gather_f32(L.w, L.g.fact_h)
    mask = (mask_rs.rand(L.Nt) > 0.1).astype(np.float32)
    return torch.from_numpy(mask).to(DEV)


@pytest.mark.parametrize("D", [50, 400])
def test_sparse_prior_layer_sequence_vs_fp64(D):
    """The sequence of ReasonGNNLayer._forward_sparse_prior -- frontier_rows, the K = D GEMM over the h segment,
    frontier_fixup, masked_softmax -- against fp64 rearev_layer + softmax over ALL rows.  Rows off the frontier
    come from the split-bf16 GEMM (three bf16 products: 2^-15 of |W| |h| + |b| on top of the fp32 sum).  D = 400 is
    the N-tiled GEMM whose two dots halves the fix-up overwrites.  The distribution is bounded per question by
    twice the largest logit error plus the softmax's own (N + 16 + 2 * logit span) u, relative."""
    I = 2
    B, N = 4, 96
    seeds = np.zeros((B, N), dtype=np.float32)
    seeds[:, :3] = 1.0 / 3
    L = _Layer(40 + D, D, I, B=B, N=N, prior=seeds)
    mask = _dense_model_inputs(L, np.random.RandomState(D))
    P = _r16(D)
    Kp = ((2 * I + 1) * P + 63) // 64 * 64
    cur_hi = torch.zeros(L.Nt, Kp, dtype=torch.bfloat16, device=DEV)
    cur_lo = torch.zeros_like(cur_hi)
    cur_hi[:, :P], cur_lo[:, :P] = L.hi, L.lo
    L.hi, L.lo = cur_hi, cur_lo
    nhi, nlo = torch.zeros_like(cur_hi), torch.zeros_like(cur_hi)
    h32 = torch.empty(L.Nt, D, device=DEV)
    dots = torch.empty(2 * L.Nt, device=DEV)
    sb = torch.tensor([0.3], device=DEV)
    rows = torch.empty(L.Nt, dtype=torch.int32, device=DEV)
    count = torch.zeros(1, dtype=torch.int32, device=DEV)
    ops.frontier_rows(L.g, L.prior, rows, count)
    ops.linear_tc_planes(cur_hi, cur_lo, P, L.W[:, :D], L.bias, out=h32, out_planes=(nhi, nlo), w_score=L.ws,
                         dots=dots, relu=True, k_seg=D, k_seg_pitch=P)
    ops.frontier_fixup(L.g, L.prior, L.tf, L.ti, L.ins, (cur_hi, cur_lo), L.W, L.bias, L.ws, (nhi, nlo), h32, dots,
                       rows, count, L.w_t, L.w_h)
    dist = ops.masked_softmax(dots, sb, mask, B, N)

    y, s, ybound, sbound = L.ref()
    h64 = cur_hi[:, :D].to(F64) + cur_lo[:, :D].to(F64)
    gemm_scale = h64.abs() @ L.W[:, :D].to(F64).abs().t() + L.bias.to(F64).abs()
    ybound = torch.maximum(ybound, (2.0 ** -15 + (D + 8) * U) * gemm_scale)
    c = int(count.item())
    assert 0 < c < L.Nt // 2
    got = nhi[:, :D].to(F64) + nlo[:, :D].to(F64)
    err = (got - y).abs()
    assert (err <= ybound + 2.0 ** -17 * y).all(), (err / ybound).max().item()
    assert (nhi[:, D:] == 0).all()
    sbound = torch.maximum(sbound, (D + 2) * U * (y @ L.ws.to(F64).abs()) + ybound @ L.ws.to(F64).abs())
    logits = torch.where(mask > 0, s + 0.3, torch.full_like(s, -1e11)).view(B, N)
    want = torch.softmax(logits, 1)
    live = (mask > 0).view(B, N)
    span = (logits.max(1, keepdim=True)[0] - torch.where(live, logits, logits.max(1, keepdim=True)[0])).max(1)[0]
    delta = torch.where(live, sbound.view(B, N), torch.zeros_like(logits)).max(1)[0]
    rel = 2 * delta + (N + 16 + 2 * span) * U
    err = (dist.to(F64) - want).abs()
    assert (err <= rel[:, None] * want + 1e-38).all(), (err / (rel[:, None] * want + 1e-38)).max().item()
    assert (dist[~live] == 0).all()


# --------------------------------------------------------------------------------------------------------------
# gr_masked_softmax
# --------------------------------------------------------------------------------------------------------------
def _softmax_ref(d0, d1, b, mask):
    l32 = (d0 + d1 + b) + (1.0 - mask) * -100000000000.0        # the kernel's fp32 logits, same operations
    return torch.softmax(l32.to(F64), 1), l32.to(F64)


@pytest.mark.parametrize("B,N,scale,masked", [
    (3, 1, 1.0, 0.0), (4, 17, 1.0, 0.3), (2, 63, 5.0, 0.2), (3, 64, 1.0, 0.0), (2, 300, 1.0, 0.5),
    (2, 1500, 2.0, 0.3), (2, 2049, 1.0, 0.1), (2, 256, 60.0, 0.2),
])
def test_masked_softmax_vs_fp64(B, N, scale, masked):
    """Both dots halves non-zero, N below / at / not a multiple of the block size, logits up to +-180 (scale 60).
    Bound: |got - want| <= (N + 16 + 2 * span) u * want, span = the largest logit distance to the maximum (expf of an
    fp32 difference is relatively off by that difference times u)."""
    rs = np.random.RandomState(N)
    d = torch.from_numpy((rs.randn(2, B * N) * scale).astype(np.float32)).to(DEV)
    mask = torch.from_numpy((rs.rand(B * N) >= masked).astype(np.float32)).to(DEV)
    mask.view(B, N)[:, 0] = 1.0
    b = torch.tensor([0.25], device=DEV)
    dist = ops.masked_softmax(d.reshape(-1), b, mask, B, N)
    want, l64 = _softmax_ref(d[0].view(B, N), d[1].view(B, N), b, mask.view(B, N))
    live = mask.view(B, N) > 0
    mx = l64.max(1, keepdim=True)[0]
    span = torch.where(live, mx - l64, torch.zeros_like(l64)).max(1, keepdim=True)[0]
    bound = (N + 16 + 2 * span) * U * want + 1e-40
    assert ((dist.to(F64) - want).abs() <= bound).all()
    assert (dist.view(B, N)[~live] == 0).all()


def test_masked_softmax_all_masked_question_is_uniform():
    """Every node masked: all logits round to the same -1e11, so the question gets exactly 1/N everywhere."""
    B, N = 3, 77
    rs = np.random.RandomState(2)
    d = torch.from_numpy(rs.randn(2, B * N).astype(np.float32)).to(DEV)
    mask = torch.ones(B * N, device=DEV)
    mask[N:2 * N] = 0.0
    dist = ops.masked_softmax(d.reshape(-1), torch.tensor([0.1], device=DEV), mask, B, N)
    assert ((dist[1].to(F64) - 1.0 / N).abs() <= U / N).all()
    want, _ = _softmax_ref(d[0].view(B, N), d[1].view(B, N), torch.tensor([0.1], device=DEV), mask.view(B, N))
    assert ((dist.to(F64) - want).abs() <= (N + 24) * U * want).all()



@pytest.mark.parametrize("I", range(1, 9))
def test_query_reform_refuses_every_width_the_fixup_refuses(I):
    """The fix-up stages 8 rows of (2I+1)*D floats (<= 200 KB, i.e. (2I+1)*D <= 6400); the instruction update that
    follows the first layer of every iteration stages (5I+1)*D floats (<= 48 KB, (5I+1)*D <= 12288).  Since
    5I+1 >= 2(2I+1), every ReaRev shape the fix-up refuses is refused by gr_query_reform as well, so the model has no
    shape at which the sparse-prior layer would need a dense fallback.  Checked at the smallest refused D per
    num_ins (1..8, the question kernels' limit), with real buffers."""
    D = 6400 // (2 * I + 1) + 1
    B, N = 2, 8
    rs = np.random.RandomState(I)
    f = lambda *s: torch.from_numpy(rs.randn(*s).astype(np.float32)).to(DEV)   # noqa: E731
    seed = torch.zeros(B, N, device=DEV)
    seed[:, 0] = 1.0
    Wr = [f(D, 3 * D) for _ in range(I)]
    Wg = [f(D, 3 * D) for _ in range(I)]
    with pytest.raises(_lib.GrError, match="gr_query_reform: invalid argument"):
        ops.query_reform(seed, f(B * N, D), f(B, I, D), Wr, Wg, B, N)
