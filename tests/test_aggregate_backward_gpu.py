"""GPU: gr_aggregate_backward (csrc/aggregate_bwd.cu) against float64 autograd of fp64_ref.aggregate.

Error bounds, per element, u = 2^-24, against the matching gradient of fp64_ref.aggregate_abs (|P|, |x|, |p|, |G|):
  * grad_table[r, d]: per edge an I-term fma chain, one product with c = w*(w*p) (two roundings), then one atomic
    add per edge of relation r: (n_r + I + 6) u, n_r = edges with relation r.
  * grad_ins[b, j, d]: an fma chain over the edges of question b (register accumulation, atomic flush per warp),
    the product c*G and c's own two roundings: (n_b + 5) u, n_b = edges of question b.
  * grad_prior[s]: per edge a dot of I*D terms (8*I per lane + a 5-step shuffle tree), times w^2, one atomic add per
    edge leaving s: (n_s + 8 I + 8) u.
Buffers that start non-zero add one rounding and their own magnitude to the scale.  The relu mask at exactly zero
matters here: ins and the table carry planted zeros, where P * x == 0 and the gradient must not flow."""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import _lib, autograd_path, ops

import fp64_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
F64 = torch.float64


def _facts(rs, B, N, E, R1, kind):
    """Fact lists (global node rows) for the graph kinds of the tests."""
    if kind == "mixed":
        # question 2 has no facts at all; nodes >= 40 of every question have no edge (empty rows); self-loops,
        # duplicated facts and relation ids 0 and R1 - 1 appear
        hs, rl, ts = [], [], []
        for b in range(B):
            if b == 2:
                continue
            h, t = rs.randint(0, 40, size=E), rs.randint(0, 40, size=E)
            h[:5] = t[:5]
            r = rs.randint(0, R1, size=E)
            r[5], r[6] = 0, R1 - 1
            dup = rs.randint(0, E, size=E // 10)
            hs += [h + b * N, h[dup] + b * N]
            ts += [t + b * N, t[dup] + b * N]
            rl += [r, r[dup]]
        return np.concatenate(hs), np.concatenate(rl), np.concatenate(ts)
    if kind == "hub":
        # node 7 of question 1 receives about 5000 edges as tail and 5000 as head
        h = rs.randint(0, N, size=(B, E)) + np.arange(B)[:, None] * N
        t = rs.randint(0, N, size=(B, E)) + np.arange(B)[:, None] * N
        hub = N + 7
        h, t = h.ravel(), t.ravel()
        h = np.concatenate([h, N + rs.randint(0, N, size=5000), np.full(5000, hub)])
        t = np.concatenate([t, np.full(5000, hub), N + rs.randint(0, N, size=5000)])
    else:   # random facts inside every question, vectorised (up to 100 000 questions / nodes)
        h = (rs.randint(0, N, size=(B, E)) + np.arange(B)[:, None] * N).ravel()
        t = (rs.randint(0, N, size=(B, E)) + np.arange(B)[:, None] * N).ravel()
    r = rs.randint(0, R1, size=len(h))
    r[:2] = [0, R1 - 1]
    return h.astype(np.int64), r.astype(np.int64), t.astype(np.int64)


class _Case:
    def __init__(self, seed, D, I, direction, weights, kind="mixed", B=4, N=50, E=120, R1=23):
        rs = np.random.RandomState(seed)
        self.B, self.N, self.D, self.I, self.Nt, self.R1 = B, N, D, I, B * N, R1
        self.direction = direction
        self.heads, self.rels, self.tails = _facts(rs, B, N, E, R1, kind)
        self.F = len(self.heads)
        dev = lambda a: torch.from_numpy(a).to(DEV)   # noqa: E731
        self.g = ops.csr_build(dev(self.heads), dev(self.rels), dev(self.tails), B, N, R1)
        self.g.check_status()
        self.w = self.w_csr = None
        if weights:
            w = rs.uniform(0.1, 1.7, size=self.F).astype(np.float32)
            w[rs.rand(self.F) < 0.1] = 0.0
            self.w = dev(w)
            self.w_csr = ops.gather_f32(self.w, self.g.fact_t if direction == "fwd" else self.g.fact_h)
        table = rs.randn(R1, D).astype(np.float32)
        table[rs.rand(R1, D) < 0.15] = 0.0                       # P == 0: mask closed for every sign of x
        ins = rs.randn(B, I, D).astype(np.float32)
        ins[rs.rand(B, I, D) < 0.15] = 0.0                       # x == 0: mask closed for every P
        prior = rs.rand(B, N).astype(np.float32)
        prior[rs.rand(B, N) < 0.2] = 0.0
        self.table, self.ins, self.prior = dev(table), dev(ins), dev(prior)
        self.G = dev(rs.randn(self.Nt, I * D).astype(np.float32))

    def run(self, gt=None, gi=None, gp=None):
        gt = torch.zeros(self.R1, self.D, device=DEV) if gt is None else gt
        gi = torch.zeros(self.B, self.I, self.D, device=DEV) if gi is None else gi
        gp = torch.zeros(self.B, self.N, device=DEV) if gp is None else gp
        ops.aggregate_backward(self.g, self.direction, self.prior, self.table, self.ins, self.G, gt, gi, gp,
                               w=self.w_csr)
        return gt, gi, gp

    def _facts_dev(self):
        return tuple(torch.from_numpy(a).to(DEV) for a in (self.heads, self.rels, self.tails))

    def ref(self, G=None):
        """(gradients, scales, gammas) of fp64 autograd through fp64_ref.aggregate / aggregate_abs."""
        G = self.G if G is None else G
        facts = self._facts_dev()
        w = None if self.w is None else self.w.to(F64)
        outs = []
        for fn, g in ((R.aggregate, G.to(F64)), (R.aggregate, G.to(F64).abs())):
            absv = len(outs) == 1
            t, x, p = (a.to(F64).abs() if absv else a.to(F64) for a in (self.table, self.ins, self.prior))
            for a in (t, x, p):
                a.requires_grad_(True)
            out = fn(t, x, p, *facts, w, self.direction)
            out.backward(g)
            outs.append((t.grad, x.grad, p.grad))
        src, dst = (self.heads, self.tails) if self.direction == "fwd" else (self.tails, self.heads)
        n_r = np.bincount(self.rels, minlength=self.R1)
        n_b = np.bincount(dst // self.N, minlength=self.B)
        n_s = np.bincount(src, minlength=self.Nt)
        I = self.I
        gam = [torch.from_numpy((n_r + I + 6) * U).to(DEV)[:, None],
               torch.from_numpy((n_b + 5) * U).to(DEV)[:, None, None],
               torch.from_numpy((n_s + 8 * I + 8) * U).to(DEV).view(self.B, self.N)]
        return outs[0], outs[1], gam


def _check(case, got, prefill=None):
    want, scale, gam = case.ref()
    names = ("grad_table", "grad_ins", "grad_prior")
    for k in range(3):
        w, s, g = want[k], scale[k], gam[k]
        if prefill is not None:
            w = w + prefill[k].to(F64)
            s = s + prefill[k].to(F64).abs()
            g = g + U
        err = (got[k].to(F64) - w).abs()
        bound = g * s + 1e-35
        assert (err <= bound).all(), "%s: worst err/bound %.3g" % (names[k], (err / bound).max().item())
    return want


CASES = [   # (D, I, direction, weights)
    (1, 1, "fwd", False), (1, 4, "inv", True),
    (8, 2, "inv", True), (8, 3, "fwd", False),
    (31, 3, "fwd", True), (31, 1, "inv", False),
    (32, 4, "inv", False), (32, 2, "fwd", True),
    (33, 1, "inv", True), (33, 4, "fwd", True),
    (200, 2, "fwd", True), (200, 3, "inv", False),
    (255, 3, "inv", True), (255, 2, "fwd", False),
    (256, 4, "fwd", False), (256, 1, "inv", True),
]


@pytest.mark.parametrize("D,I,direction,weights", CASES)
def test_backward_vs_fp64_autograd(D, I, direction, weights):
    """Every gradient element within the bound of the module docstring, on a graph with empty rows, an all-empty
    question, self-loops, duplicated facts and the relation ids 0 and R1 - 1."""
    case = _Case(D * 7 + I, D, I, direction, weights)
    want = _check(case, case.run())
    assert (want[1] == 0).any() and (want[1] != 0).any()
    assert (want[1][2] == 0).all()                              # the all-empty question gets no gradient


@pytest.mark.parametrize("kind,B,N,E,D,I,direction,weights", [
    ("hub", 2, 300, 400, 33, 2, "fwd", True),
    ("hub", 2, 300, 400, 64, 3, "inv", False),
    ("random", 1, 1, 3, 8, 1, "fwd", True),                       # B = 1, N = 1: self-loops only
    ("random", 20000, 5, 6, 32, 2, "fwd", True),                  # warp row ranges cross many question boundaries
    ("random", 20000, 5, 6, 31, 4, "inv", False),
    ("random", 1, 100000, 200000, 31, 3, "inv", True),            # one question spread over every warp
])
def test_backward_graph_shapes(kind, B, N, E, D, I, direction, weights):
    """Hub rows with ~5000 in-edges; B = N = 1; N = 5 with B = 20 000 (rows per warp > N once the grid is capped at
    16 CTAs per SM, so a warp's range crosses question boundaries and must flush dx at each); B = 1 with N = 100 000
    (many warps add into the same question).  Same bound as above."""
    case = _Case(B + N + D, D, I, direction, weights, kind=kind, B=B, N=N, E=E)
    _check(case, case.run())


def test_backward_accumulates_into_buffers_and_f0_is_a_no_op():
    """The ABI adds to the gradient buffers (both directions and all layers of a backward share them): random
    pre-filled buffers end as prefill + gradient.  A graph without facts leaves them bit-identical."""
    case = _Case(5, 33, 2, "inv", True)
    rs = np.random.RandomState(1)
    pre = [torch.from_numpy(rs.randn(*s).astype(np.float32)).to(DEV)
           for s in ((case.R1, case.D), (case.B, case.I, case.D), (case.B, case.N))]
    got = case.run(*(p.clone() for p in pre))
    _check(case, got, prefill=pre)
    g0 = ops.csr_build(*(torch.zeros(0, dtype=torch.int64, device=DEV) for _ in range(3)), case.B, case.N, case.R1)
    assert g0.F == 0
    bufs = [p.clone() for p in pre]
    ops.aggregate_backward(g0, "fwd", case.prior, case.table, case.ins, case.G, *bufs)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(bufs, pre))


def _raw(case, G, ld, col0, seg, D=None, I=None):
    L = _lib.load()
    gt = torch.zeros(case.R1, case.D, device=DEV)
    gi = torch.zeros(case.B, case.I, case.D, device=DEV)
    gp = torch.zeros(case.B, case.N, device=DEV)
    g = case.g
    rp, src, rel = (g.rowptr_t, g.src_t, g.rel_t) if case.direction == "fwd" else (g.rowptr_h, g.src_h, g.rel_h)
    p = ops._p
    rc = L.gr_aggregate_backward(p(rp), p(src), p(rel), p(case.w_csr), p(case.prior), p(case.table), p(case.ins), p(G),
                                 ld, col0, seg, p(gt), p(gi), p(gp), case.B, case.N,
                                 case.D if D is None else D, case.I if I is None else I, case.F, ops._stream())
    return rc, (gt, gi, gp)


def test_backward_refuses_unsupported_shapes():
    """D = 257, I = 5 and a segment stride below D are refused with GR_ERR_INVALID_ARG (-1), before any launch."""
    case = _Case(3, 8, 2, "fwd", False)
    G = case.G
    assert _raw(case, G, 2 * 8, 0, 8)[0] == 0
    assert _raw(case, G, 2 * 257, 0, 257, D=257)[0] == -1
    assert b"D <= 256" in _lib.load().gr_last_error()
    assert _raw(case, G, 5 * 8, 0, 8, I=5)[0] == -1
    assert _raw(case, G, 2 * 8, 0, 7)[0] == -1
    assert b"segment stride" in _lib.load().gr_last_error()
    torch.cuda.synchronize()


def test_backward_reads_a_column_window_of_a_wider_grad_buffer():
    """grad_out as a window of a wider buffer (grad_col0 > 0, seg_stride > D): a layout the ABI accepts although
    ops never passes it.  Same bound as the contiguous case."""
    case = _Case(11, 40, 3, "fwd", True)
    col0, seg = 5, 40 + 7
    ld = col0 + (case.I - 1) * seg + case.D + 3
    rs = np.random.RandomState(2)
    wide = torch.from_numpy(rs.randn(case.Nt, ld).astype(np.float32)).to(DEV)
    case.G = torch.cat([wide[:, col0 + j * seg: col0 + j * seg + case.D] for j in range(case.I)], 1).contiguous()
    rc, got = _raw(case, wide, ld, col0, seg)
    assert rc == 0
    _check(case, got)


def test_autograd_function_with_noncontiguous_table_and_prior_grad():
    """_AggregateFn.apply (forward gr_aggregate, backward gr_aggregate_backward) with a transposed table and a prior
    that requires grad, against fp64 autograd: forward within (2n + 8) u of aggregate_abs, gradients as above."""
    case = _Case(13, 48, 2, "inv", True)
    table_t = case.table.t().contiguous().requires_grad_(True)   # storage of the transposed view
    table = table_t.t()
    assert not table.is_contiguous()
    ins = case.ins.clone().requires_grad_(True)
    prior = case.prior.clone().requires_grad_(True)
    out = autograd_path._AggregateFn.apply(table, ins, prior, case.g, "inv", case.w_csr)
    out.backward(case.G)
    facts = case._facts_dev()
    w = case.w.to(F64)
    want = R.aggregate(*(a.to(F64) for a in (case.table, case.ins, case.prior)), *facts, w, "inv")
    scale = R.aggregate_abs(*(a.to(F64) for a in (case.table, case.ins, case.prior)), *facts, w, "inv")
    n = torch.from_numpy(np.bincount(case.heads, minlength=case.Nt)).to(DEV, F64)[:, None]
    assert ((out.to(F64) - want).abs() <= (2 * n + 8) * U * scale + 1e-35).all()
    _check(case, (table_t.grad.t(), ins.grad, prior.grad))


def test_large_shapes_take_the_torch_path_and_match_fp64():
    """D = 400 or I = 5 is beyond the backward kernel: _kernel_graph returns None and the layer's messages come from
    torch index_add (fp32 atomics); forward and gradients still match fp64 within the same per-element bounds."""
    assert autograd_path._kernel_graph(None, None, torch.device(DEV), 400, 2) is None
    assert autograd_path._kernel_graph(None, None, torch.device(DEV), 200, 5) is None
    D, I, B, N = 400, 5, 3, 40
    rs = np.random.RandomState(4)
    heads, rels, tails = _facts(rs, B, N, 100, 17, "random")
    F = len(heads)
    w = rs.uniform(0.1, 1.5, size=F).astype(np.float32)
    kb = (heads, rels, tails, heads // N, np.arange(F), w.tolist(), None)
    facts = autograd_path._Facts(kb, torch.device(DEV), True, False)
    f = lambda *s: torch.from_numpy(rs.randn(*s).astype(np.float32)).to(DEV)   # noqa: E731
    tf, ti, ins = f(17, D), f(17, D), f(B, I, D)
    ins[:, :, ::9] = 0.0
    prior = torch.from_numpy(rs.rand(B, N).astype(np.float32)).to(DEV)
    leaves = [t.clone().requires_grad_(True) for t in (tf, ti, ins, prior)]
    out = autograd_path._neighbours(leaves[0], leaves[1], leaves[2], leaves[3], facts, None, B * N)
    G = f(*out.shape)
    out.backward(G)
    fd = tuple(torch.from_numpy(a).to(DEV) for a in (heads, rels, tails))
    wd = torch.from_numpy(w).to(DEV, F64)
    ref = [t.to(F64).requires_grad_(True) for t in (tf, ti, ins, prior)]
    outs = [R.aggregate(ref[0], ref[2], ref[3], *fd, wd, "fwd").view(B * N, I, 1, D),
            R.aggregate(ref[1], ref[2], ref[3], *fd, wd, "inv").view(B * N, I, 1, D)]
    want = torch.cat(outs, 2)
    want.backward(G.to(F64))
    absr = [t.to(F64).abs().requires_grad_(True) for t in (tf, ti, ins, prior)]
    sc = torch.cat([R.aggregate(absr[0], absr[2], absr[3], *fd, wd, "fwd").view(B * N, I, 1, D),
                    R.aggregate(absr[1], absr[2], absr[3], *fd, wd, "inv").view(B * N, I, 1, D)], 2)
    sc.backward(G.to(F64).abs())
    gam = (2 * F + 8 * I + 8) * U                                  # no per-element count: torch's order is opaque
    assert ((out.to(F64) - want).abs() <= gam * sc + 1e-35).all()
    for got, r, a in zip(leaves, ref, absr):
        assert ((got.grad.to(F64) - r.grad).abs() <= gam * a.grad + 1e-35).all()
