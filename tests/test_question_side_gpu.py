"""GPU: the question-side and scoring kernels (csrc/question.cu, csrc/score.cu) against the float64 restatements of
tests/question_ref.py, at the shapes the kernels are written around.

Every output buffer the kernel should fill is pre-filled with NaN and the C entry point is called directly, so an
element the kernel never writes fails ``err <= bound`` instead of passing by accident.

Error bounds (u = 2^-24; the library is built without fast-math, so ``expf`` / ``tanhf`` are within 2 ulp, ``logf``
within 1 ulp, and divisions are IEEE).  Each bound below is a first-order forward error analysis of the kernel's own
operation order, carried through in float64 next to the reference values:
  * a warp GEMV row of length K (lanes over k, ceil(K/32) fmas per lane, a 5-step shuffle tree, the bias):
    G(K) = (ceil(K/32) + 8) u of sum |w| |x| + |b|, plus |W| times the error already in x;
  * sigmoid as 1 / (1 + expf(-x)): 8 u absolute plus 1/4 of the argument's error; tanhf: 4 u plus the argument's
    error;
  * a softmax over n entries whose logits are each off by at most delta: relative (e^(2 delta) - 1) +
    (n + 16 + 2 span) u, span = the largest live logit distance to the maximum (expf of an fp32 difference is off by
    that difference times u); masked entries of a row with a live entry are exactly 0;
  * a sequential sum of n terms: n u of sum |term|.
The LSTM bound is carried over all tokens (the recurrence contracts); the instruction steps are checked one at a time,
each from the kernel's own previous instruction (see ``_Ins.ref``).  A dropped or doubled term, a wrong column slice, a skipped token or a wrong maximum moves an element by a sizeable
fraction of its scale (or leaves the NaN in place), far outside these bounds."""
import math

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import _lib, ops, synthetic as S
from oracle import kgqa_oracle as O

import question_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
F64 = torch.float64
NAN = float("nan")


def _gemv(K):
    return (math.ceil(K / 32) + 8) * U


def _sig_err(e):
    return e / 4 + 8 * U


def _nan(*shape):
    return torch.full(shape, NAN, device=DEV)


def _p(t):
    return ops._p(t)


def _check(got, want, bound, what):
    err = (got.to(F64) - want).abs()
    ok = err <= bound                                        # NaN (an unwritten element) is never <= anything
    assert ok.all(), "%s: %d bad, worst err/bound %g" % (what, int((~ok).sum()), (err / bound).max().item())


def _softmax_rel(logits, mask, delta, n):
    """Per-row relative bound of a softmax over fp32 logits each off by at most ``delta`` (per row)."""
    live = mask > 0
    mx = torch.where(live, logits, torch.full_like(logits, -math.inf)).max(1, keepdim=True)[0]
    span = torch.where(live, mx - logits, torch.zeros_like(logits)).max(1, keepdim=True)[0]
    span = torch.where(live.any(1, keepdim=True), span, torch.zeros_like(span))
    return torch.expm1(2 * delta) + (n + 16 + 2 * span) * U


# --------------------------------------------------------------------------------------------------------------
# gr_lstm_forward
# --------------------------------------------------------------------------------------------------------------
def _lstm_bound(gx, W, b):
    """The float64 LSTM and a per-element bound on the kernel's hidden states, by recursion over t.

    Step t: the gate pre-activation a = sum_k W[r,k] h[k] (one sequential fma chain of D terms) + gx + b has D + 2
    roundings of S = |W| (|h| + e_h) + |gx| + |b|, plus |W| e_h from the previous state's error e_h.  The sigmoid gates
    are then off by da/4 + 8u, the tanh gate by da + 4u.  c = fma(f, c, i * g) adds the gates' errors times the other
    factors and 2u (|f c| + |i g|); h = o * tanhf(c) adds e_o |tanh c| + (|o| + e_o)(e_c + 4u) + u |h|.  The tests
    draw W_hh entries as N(0, 1) * 0.5 / D, so a row's sum |W| is about 0.4: the previous error enters each gate
    scaled by well under 1 (and a sigmoid gate by a quarter of that), the recursion contracts, and the bound stays a
    small multiple of one step's roundings over 40 tokens instead of growing geometrically."""
    gx, W = gx.to(F64), W.to(F64)
    B, Q, G4 = gx.shape
    D = G4 // 4
    b = torch.zeros(G4, dtype=F64, device=gx.device) if b is None else b.to(F64)
    aW = W.abs()
    h = torch.zeros(B, D, dtype=F64, device=gx.device)
    c, eh, ec = torch.zeros_like(h), torch.zeros_like(h), torch.zeros_like(h)
    hs, bounds = [], []
    for t in range(Q):
        a = gx[:, t] + h @ W.t() + b
        S_ = (h.abs() + eh) @ aW.t() + gx[:, t].abs() + b.abs()
        da = (D + 2) * U * S_ + eh @ aW.t()
        i, f, o = torch.sigmoid(a[:, :D]), torch.sigmoid(a[:, D:2 * D]), torch.sigmoid(a[:, 3 * D:])
        g = torch.tanh(a[:, 2 * D:3 * D])
        di, df, do = _sig_err(da[:, :D]), _sig_err(da[:, D:2 * D]), _sig_err(da[:, 3 * D:])
        dg = da[:, 2 * D:3 * D] + 4 * U
        cn = f * c + i * g
        ec = (f + df) * ec + df * c.abs() + di * (g.abs() + dg) + i * dg + 2 * U * ((f * c).abs() + (i * g).abs())
        c = cn
        tc = torch.tanh(c)
        h = o * tc
        eh = do * tc.abs() + (o + do) * (ec + 4 * U) + U * h.abs()
        hs.append(h)
        bounds.append(eh)
    return torch.stack(hs, 1), torch.stack(bounds, 1)


def _lstm_run(gx, W, b):
    B, Q, G4 = gx.shape
    out = _nan(B, Q, G4 // 4)
    _lib.check(_lib.load().gr_lstm_forward(_p(gx), _p(W), _p(b), _p(out), B, Q, G4 // 4, ops._stream()))
    return out


# D < 8: CTAs without hidden units; B = 7 / 9 / 17: partial clusters of 8 questions
LSTM_CASES = [(1, 1, 1, True), (7, 2, 7, True), (8, 40, 8, False), (9, 2, 9, True), (17, 40, 33, True),
              (1, 40, 64, False), (9, 40, 200, True), (17, 2, 255, True), (8, 40, 256, True), (7, 1, 256, False),
              (17, 1, 1, False), (9, 40, 7, True)]


@pytest.mark.parametrize("B,Q,D,bias", LSTM_CASES)
def test_lstm_forward_vs_fp64(B, Q, D, bias):
    """Every token's hidden state of every question, against the float64 LSTM, within the bound of _lstm_bound."""
    rs = np.random.RandomState(B * 1000 + Q * 10 + D)
    gx = torch.from_numpy(rs.randn(B, Q, 4 * D).astype(np.float32)).to(DEV)
    W = torch.from_numpy((rs.randn(4 * D, D) * 0.5 / D).astype(np.float32)).to(DEV)   # a contracting recurrence
    b = torch.from_numpy((rs.randn(4 * D) * 0.5).astype(np.float32)).to(DEV) if bias else None
    got = _lstm_run(gx, W, b)
    torch.cuda.synchronize()
    want, bound = _lstm_bound(gx, W, b)
    assert torch.allclose(want, R.lstm(gx, W, b), rtol=0, atol=1e-12)             # the restatement, independently
    _check(got, want, bound + 1e-30, "hidden")


def test_lstm_forward_refuses_hidden_257():
    B, Q, D = 2, 3, 257
    gx = torch.zeros(B, Q, 4 * D, device=DEV)
    W = torch.zeros(4 * D, D, device=DEV)
    out = _nan(B, Q, D)
    with pytest.raises(_lib.GrError, match="gr_lstm_forward: invalid argument"):
        _lib.check(_lib.load().gr_lstm_forward(_p(gx), _p(W), None, _p(out), B, Q, D, ops._stream()))
    assert torch.isnan(out).all()


# --------------------------------------------------------------------------------------------------------------
# gr_instructions
# --------------------------------------------------------------------------------------------------------------
class _Ins:
    PAD = 90

    def __init__(self, seed, B, Q, D, I, peaked=None):
        rs = np.random.RandomState(seed)
        f = lambda *s, sc=1.0: torch.from_numpy((rs.randn(*s) * sc).astype(np.float32)).to(DEV)   # noqa: E731
        self.B, self.Q, self.D, self.I = B, Q, D, I
        self.hid = f(B, Q, D, sc=0.5)
        self.qn = f(B, D, sc=0.5)
        self.Wq = [f(D, D, sc=1 / math.sqrt(D)) for _ in range(I)]
        self.bq = [f(D, sc=0.1) for _ in range(I)]
        self.Wcq, self.bcq = f(D, 4 * D, sc=1 / math.sqrt(4 * D)), f(D, sc=0.1)
        self.wca, self.bca = f(D, sc=1 / math.sqrt(D)), f(1, sc=0.1)
        text = rs.randint(0, self.PAD, size=(B, Q))
        if Q >= 3:
            text[0, Q // 2] = self.PAD                          # a pad token inside the question
            text[0, -1] = self.PAD                              # and one in the tail
        if B > 1:
            text[B - 1] = self.PAD                              # an all-pad question
        self.text = torch.from_numpy(text).to(DEV)
        if peaked is not None:
            self._peak(peaked)

    def _peak(self, k):
        """Make token k of question 0 win the first attention step by a logit margin above 100 over every other
        token: hidden[0, k] = alpha * sign(wca * cq), where cq is the step-0 cq_linear output."""
        D = self.D
        q0 = self.qn[0].to(F64) @ self.Wq[0].to(F64).t() + self.bq[0].to(F64)
        z = torch.cat([torch.zeros_like(q0), q0, q0, torch.zeros_like(q0)])
        cq = self.Wcq.to(F64) @ z + self.bcq.to(F64)
        v = self.wca.to(F64) * cq
        others = (self.hid[0].to(F64) @ v).max().item()
        alpha = (max(others, 0.0) + 100.0) / v.abs().sum().item() + 1.0
        self.hid[0, k] = (alpha * torch.sign(v)).float()
        self.text[0, k] = 1

    def run(self, attn=True, I=None):
        I = self.I if I is None else I
        out = _nan(self.B, I, self.D)
        at = _nan(self.B, I, self.Q) if attn else None
        rc = _lib.load().gr_instructions(_p(self.hid), _p(self.qn), _p(self.text), self.PAD, ops._ptr_array(self.Wq),
                                         ops._ptr_array(self.bq), _p(self.Wcq), _p(self.bcq), _p(self.wca),
                                         _p(self.bca), _p(out), _p(at), self.B, self.Q, self.D, I, ops._stream())
        _lib.check(rc)
        return out, at

    def ref(self, out=None):
        """float64 instructions / attention of every step and their bounds (module docstring).

        Step i starts from the relational instruction the kernel itself produced at step i - 1 (``out``, which is
        exactly the fp32 value the kernel carries on in shared memory), so each bound covers one step's roundings.
        Chaining worst-case bounds instead multiplies them by |Wcq| |wca| |hidden| (about 100 at D = 256) per step
        through the softmax and overflows by the eighth instruction.  Step 0 starts from zero, as the model does;
        every later step is then checked against an exact restatement of its own inputs.  Without ``out`` (a kernel
        run not yet made) the steps chain from zero."""
        D, Q, I = self.D, self.Q, self.I
        hid = self.hid.to(F64)
        aH = hid.abs()
        mask = (self.text != self.PAD).to(F64)
        live = mask > 0
        Wcq, bcq, wca, bca = (t.to(F64) for t in (self.Wcq, self.bcq, self.wca, self.bca))
        qn = self.qn.to(F64)
        ri = torch.zeros(self.B, D, dtype=F64, device=DEV)
        wants, eouts, attns, eattns, cas = [], [], [], [], []
        for i in range(I):
            W, b = self.Wq[i].to(F64), self.bq[i].to(F64)
            qi = qn @ W.t() + b
            eqi = _gemv(D) * (qn.abs() @ W.abs().t() + b.abs())
            z = torch.cat([ri, qi, qi - ri, qi * ri], 1)
            ez = torch.cat([torch.zeros_like(ri), eqi, eqi + U * (qi - ri).abs(),
                            ri.abs() * eqi + U * (qi * ri).abs()], 1)
            cq = z @ Wcq.t() + bcq
            ecq = _gemv(4 * D) * ((z.abs() + ez) @ Wcq.abs().t() + bcq.abs()) + ez @ Wcq.abs().t()
            ca = (cq.unsqueeze(1) * hid) @ wca + bca
            eca = (_gemv(D) + U) * (((cq.abs() + ecq).unsqueeze(1) * aH) @ wca.abs() + bca.abs()) \
                + (ecq.unsqueeze(1) * aH) @ wca.abs()
            assert (ca.abs() < 4096).all()                          # masked logits collapse to VERY_NEG (question_ref)
            delta = torch.where(live, eca, torch.zeros_like(eca)).max(1, keepdim=True)[0]
            attn = torch.softmax(torch.where(live, ca, torch.full_like(ca, R.VERY_NEG)), 1)
            eattn = _softmax_rel(ca, mask, delta, Q) * attn
            ri_new = (attn.unsqueeze(2) * hid).sum(1)
            eri = Q * U * (attn.unsqueeze(2) * aH).sum(1) + ((eattn.unsqueeze(2)) * aH).sum(1)
            want, att = R.instructions(self.hid, self.qn, self.text, self.PAD, [self.Wq[i]], [self.bq[i]], self.Wcq,
                                       self.bcq, self.wca, self.bca, ri0=ri)
            assert torch.allclose(ri_new, want[:, 0], rtol=0, atol=1e-9 * (1 + ri_new.abs().max().item()))
            wants.append(want[:, 0]), eouts.append(eri), attns.append(att[:, 0]), eattns.append(eattn), cas.append(ca)
            ri = ri_new if out is None else out[:, i].to(F64)
        return (torch.stack(wants, 1), torch.stack(eouts, 1), torch.stack(attns, 1), torch.stack(eattns, 1),
                torch.stack(cas, 1))


def _check_ins(L, out, at):
    assert not torch.isnan(out).any()                           # every element written (before conditioning on it)
    want, bound, att, abound, _ = L.ref(out)
    _check(out, want, bound + 1e-30, "instructions")
    if at is not None:
        _check(at, att, abound + 1e-38, "attention")
        if L.B > 1:                                             # the all-pad question: exactly uniform attention
            assert (at[L.B - 1] == at[L.B - 1, 0, 0]).all()
            assert abs(at[L.B - 1, 0, 0].item() - 1.0 / L.Q) <= U / L.Q
        live = (L.text != L.PAD)
        if L.B > 1:
            assert (at[:L.B - 1][~live[:L.B - 1].unsqueeze(1).expand(-1, L.I, -1)] == 0).all()


@pytest.mark.parametrize("B,Q,D,I", [(3, 1, 1, 1), (3, 31, 33, 2), (3, 32, 200, 4), (3, 33, 256, 8), (2, 100, 400, 8),
                                     (3, 100, 200, 1), (3, 33, 1, 8), (2, 32, 400, 2), (4, 31, 256, 4)])
def test_instructions_vs_fp64(B, Q, D, I):
    """Instruction vectors and attention of every step; a pad inside question 0, an all-pad last question."""
    L = _Ins(Q * 100 + D + I, B, Q, D, I)
    out, at = L.run()
    torch.cuda.synchronize()
    _check_ins(L, out, at)


@pytest.mark.parametrize("Q,k", [(41, 40), (100, 77), (33, 32)])
def test_instructions_peaked_attention_past_the_first_warp(Q, k):
    """Token k >= 32 outscores every earlier token by more than 88 at the first step, so an expf that did not
    subtract the true maximum (e.g. one taken over the first 32 tokens only) overflows.  Without the optional
    attention output as well."""
    L = _Ins(Q + k, 2, Q, 64, 1, peaked=k)
    _, _, att, _, ca = L.ref()
    live = L.text[0] != L.PAD
    assert ca[0, 0, k] - ca[0, 0, :k][live[:k]].max() > 88 and att[0, 0, k] > 0.999   # the precondition
    out, at = L.run()
    torch.cuda.synchronize()
    _check_ins(L, out, at)
    out2, _ = L.run(attn=False)
    assert torch.equal(out, out2)


def _q_max(D, I):
    """The largest Q gr_instructions admits: (Q D + (I + 7) D + 2 Q) * 4 bytes <= 200 KB."""
    return (200 * 1024 // 4 - (I + 7) * D) // (D + 2)


@pytest.mark.parametrize("D,I", [(200, 2), (400, 8), (33, 1)])
def test_instructions_largest_admitted_question_runs_and_next_is_refused(D, I):
    Q = _q_max(D, I)
    assert (Q * D + (I + 7) * D + 2 * Q) * 4 <= 200 * 1024 < ((Q + 1) * D + (I + 7) * D + 2 * (Q + 1)) * 4
    L = _Ins(D + I, 2, Q, D, I)
    out, at = L.run()
    torch.cuda.synchronize()
    _check_ins(L, out, at)
    L2 = _Ins(D + I, 2, Q + 1, D, I)
    with pytest.raises(_lib.GrError, match="gr_instructions: invalid argument.*too large"):
        L2.run()


def test_instructions_refuses_nine_instructions():
    L = _Ins(9, 2, 5, 16, 9)
    with pytest.raises(_lib.GrError, match="gr_instructions: invalid argument"):
        L.run()


# --------------------------------------------------------------------------------------------------------------
# gr_query_reform and gr_seed_retrieve
# --------------------------------------------------------------------------------------------------------------
def _seeds(rs, B, N):
    """q0: one seed; q1: several seeds across 1024- (and 256-) node chunk edges; q2: none; q3: dense (every node
    non-zero); further questions: one seed each."""
    s = np.zeros((B, N), dtype=np.float32)
    s[:, min(3, N - 1)] = 1.0
    if B > 1:
        s[1] = 0.0
        idx = sorted({i for i in (0, 255, 256, 1023, 1024, 2047, 2048, N - 1) if i < N})
        s[1, idx] = rs.uniform(0.1, 1.0, size=len(idx))
    if B > 2:
        s[2] = 0.0
    if B > 3:
        s[3] = rs.uniform(0.01, 1.0, size=N) / N
    return torch.from_numpy(s).to(DEV)


def _seed_bound(seed, h, B, N):
    """A sequential fma sum over each question's non-zero seeds: nnz u of |s| |h|."""
    s = seed.to(F64)
    nnz = (s != 0).sum(1, keepdim=True).to(F64)
    return nnz * U * torch.bmm(s.abs().view(B, 1, N), h.to(F64).abs().reshape(B, N, -1)).squeeze(1)


class _Reform:
    def __init__(self, seed, B, N, D, I, ldh_pad=0):
        rs = np.random.RandomState(seed)
        f = lambda *s, sc=1.0: torch.from_numpy((rs.randn(*s) * sc).astype(np.float32)).to(DEV)   # noqa: E731
        self.B, self.N, self.D, self.I = B, N, D, I
        self.h = f(B * N, D + ldh_pad)[:, :D]                  # ldh = D + ldh_pad
        self.seed = _seeds(rs, B, N)
        self.ins = f(B, I, D)
        self.Wr = [f(D, 3 * D, sc=1 / math.sqrt(3 * D)) for _ in range(I)]
        self.Wg = [f(D, 3 * D, sc=1 / math.sqrt(3 * D)) for _ in range(I)]

    def run(self):
        out, sout = _nan(self.B, self.I, self.D), _nan(self.B, self.D)
        rc = _lib.load().gr_query_reform(_p(self.seed), _p(self.h), self.h.stride(0), _p(self.ins),
                                         ops._ptr_array(self.Wr), ops._ptr_array(self.Wg), _p(out), _p(sout),
                                         self.B, self.N, self.D, self.I, ops._stream())
        _lib.check(rc)
        return out, sout

    def check(self, out, sout):
        B, N, D = self.B, self.N, self.D
        want, y = R.query_reform(self.seed, self.h, self.ins, self.Wr, self.Wg, B, N)
        ey = _seed_bound(self.seed, self.h, B, N)
        _check(sout, y, ey + 1e-30, "seed_retrieve")
        x = self.ins.to(F64)
        for j in range(self.I):
            xj = x[:, j]
            z = torch.cat([xj, y, xj - y], 1)
            ez = torch.cat([torch.zeros_like(ey), ey, ey + U * (xj - y).abs()], 1)
            Wr, Wg = self.Wr[j].to(F64), self.Wg[j].to(F64)
            r, g = z @ Wr.t(), torch.sigmoid(z @ Wg.t())
            er = _gemv(3 * D) * ((z.abs() + ez) @ Wr.abs().t()) + ez @ Wr.abs().t()
            eg = _sig_err(_gemv(3 * D) * ((z.abs() + ez) @ Wg.abs().t()) + ez @ Wg.abs().t())
            bound = eg * (r.abs() + er + xj.abs()) + g * er + 4 * U * ((g * r).abs() + ((1 - g) * xj).abs())
            _check(out[:, j], want[:, j], bound + 1e-30, "instruction %d" % j)


# D: 1-column slices below 64, 2 up to 127, 4 from 128; 65 / 129 / 130 leave a short last slice
REFORM_CASES = [(1, 1, 1), (63, 3, 1023), (64, 8, 1024), (65, 2, 1025), (127, 5, 3000), (128, 4, 1024),
                (129, 7, 1025), (130, 6, 1023), (200, 2, 3000), (1024, 1, 1025), (1024, 2, 300), (65, 8, 1)]


@pytest.mark.parametrize("D,I,N", REFORM_CASES)
@pytest.mark.parametrize("ldh_pad", [0, 3])
def test_query_reform_vs_fp64(D, I, N, ldh_pad):
    """New instructions of all I Fusions and the optional seed_retrieve output, for seeds none / one / across the
    1024-node chunk edges / dense, with h a plain or strided (ldh > D) view."""
    L = _Reform(D * 10 + I + N, 4, N, D, I, ldh_pad)
    out, sout = L.run()
    torch.cuda.synchronize()
    L.check(out, sout)
    assert torch.equal(L.seed[2], torch.zeros_like(L.seed[2])) and (sout[2] == 0).all()


def _reform_d_max(I):
    """The widest D gr_query_reform admits: D <= 1024 and (5I + 1) D floats of shared memory <= 48 KB."""
    return min(1024, 48 * 1024 // (4 * (5 * I + 1)))


@pytest.mark.parametrize("I", range(1, 9))
def test_query_reform_largest_admitted_width_runs(I):
    """Every shape the entry point admits must launch and compute: the widest D for each num_ins (1024, 1024, 768,
    585, 472, 396, 341, 299), and the next width is refused."""
    D = _reform_d_max(I)
    L = _Reform(I, 2, 300, D, I, ldh_pad=1)
    out, sout = L.run()
    torch.cuda.synchronize()
    L.check(out, sout)
    L2 = _Reform(I, 2, 8, D + 1, I)
    with pytest.raises(_lib.GrError, match="gr_query_reform: invalid argument"):
        L2.run()


def _seed_retrieve_run(seed, h, B, N, D):
    out = _nan(B, D)
    _lib.check(_lib.load().gr_seed_retrieve(_p(seed), _p(h), h.stride(0), _p(out), B, N, D, ops._stream()))
    return out


@pytest.mark.parametrize("D", [1, 255, 256, 257, 768, 769, 1024])
@pytest.mark.parametrize("N,ldh_pad", [(1, 0), (257, 5), (700, 0), (2049, 2)])
def test_seed_retrieve_vs_fp64(D, N, ldh_pad):
    """One to four columns per thread (D <= 1024 with 256 threads), seeds across the 256-node chunks, dense seeds."""
    rs = np.random.RandomState(D + N)
    B = 5
    h = torch.from_numpy(rs.randn(B * N, D + ldh_pad).astype(np.float32)).to(DEV)[:, :D]
    seed = _seeds(rs, B, N)
    out = _seed_retrieve_run(seed, h, B, N, D)
    torch.cuda.synchronize()
    _check(out, R.seed_retrieve(seed, h, B, N), _seed_bound(seed, h, B, N) + 1e-30, "seed_retrieve")
    assert (out[2] == 0).all()


def test_seed_retrieve_refuses_1025_columns():
    B, N, D = 2, 4, 1025
    h, seed, out = torch.zeros(B * N, D, device=DEV), torch.ones(B, N, device=DEV), _nan(B, D)
    with pytest.raises(_lib.GrError, match="gr_seed_retrieve: invalid argument"):
        _lib.check(_lib.load().gr_seed_retrieve(_p(seed), _p(h), D, _p(out), B, N, D, ops._stream()))


# --------------------------------------------------------------------------------------------------------------
# gr_score_softmax
# --------------------------------------------------------------------------------------------------------------
def _score_inputs(rs, B, N, D, layout):
    """h [B*N, D] as: "vec" (D % 4 == 0, ldh % 4 == 0, 16-byte aligned: the float4 path), "ldh" (ldh = D + 2),
    "offset" (one float past an aligned base) or "odd" (D % 4 != 0): the scalar path."""
    ld = D + (2 if layout == "ldh" else 0)
    buf = torch.from_numpy(rs.randn(B * N * ld + 4).astype(np.float32)).to(DEV)
    off = 1 if layout == "offset" else 0
    h = buf[off:off + B * N * ld].view(B * N, ld)[:, :D]
    w = torch.from_numpy((rs.randn(D) / math.sqrt(D)).astype(np.float32)).to(DEV)
    return h, w


SCORE_CASES = [(1, 200, "vec", True), (63, 201, "odd", True), (64, 200, "ldh", False), (255, 200, "offset", True),
               (256, 200, "vec", False), (1023, 33, "odd", True), (1024, 200, "vec", True), (1025, 200, "offset", True),
               (1025, 64, "ldh", True), (63, 4, "vec", False), (256, 1, "odd", True), (1024, 7, "offset", False)]


@pytest.mark.parametrize("N,D,layout,bias", SCORE_CASES)
def test_score_softmax_vs_fp64(N, D, layout, bias):
    """Block sizes 64 / 256 / 1024 (by N), the float4 and scalar dot paths, b_score None, logits_out given.
    Question 0 has masked nodes, question 1 is all padding (exactly uniform), question 2 is all live."""
    B = 3
    rs = np.random.RandomState(N * 7 + D)
    h, w = _score_inputs(rs, B, N, D, layout)
    b = torch.tensor([0.3], device=DEV) if bias else None
    mask = torch.from_numpy((rs.rand(B, N) > 0.3).astype(np.float32)).to(DEV)
    mask[0, 0] = 1.0
    mask[1] = 0.0
    mask[2] = 1.0
    dist, logits = _nan(B, N), _nan(B, N)
    rc = _lib.load().gr_score_softmax(_p(h), h.stride(0), _p(w), _p(b), _p(mask), _p(dist), _p(logits), B, N, D,
                                      ops._stream())
    _lib.check(rc)
    torch.cuda.synchronize()
    want, wl = R.score_softmax(h, w, b, mask.view(-1), B, N)
    live = mask > 0
    dots = h.to(F64) @ w.to(F64)
    scale = (h.to(F64).abs() @ w.to(F64).abs()).view(B, N) + (abs(b.item()) if bias else 0.0)
    assert (dots.abs() < 4096).all()
    delta = _gemv(D) * scale
    _check(logits[live], wl[live], delta[live] + 1e-30, "logits")
    assert (logits[~live] == R.VERY_NEG).all()
    dmax = torch.where(live, delta, torch.zeros_like(delta)).max(1, keepdim=True)[0]
    rel = _softmax_rel(wl, mask.to(F64), dmax, N)
    _check(dist, want, rel * want + 1e-38, "dist")
    assert (dist[0][~live[0]] == 0).all()                        # masked entries of a row with a live node
    assert (dist[1] == dist[1, 0]).all() and abs(dist[1, 0].item() - 1.0 / N) <= U / N   # all-pad: uniform
    # and without logits_out (the logits are staged in dist): the same distribution bit for bit
    d2 = ops.score_softmax(h, w, b, mask.view(-1), B, N)
    assert torch.equal(d2, dist)


# --------------------------------------------------------------------------------------------------------------
# gr_kl_loss_pred
# --------------------------------------------------------------------------------------------------------------
def _tie(dist, b, kind, N):
    """Two or three exact maxima in row b (256 threads: n and n + 256 are one thread's strided chunk, 5 and 17 two
    lanes of warp 0, 40 and 200 two warps); returns the index the argmax must give (the lowest), or None when the
    row is too short for the tie."""
    idx = {"lanes": (17, 5), "chunk": (3 + 512, 3 + 256, 3), "warps": (200, 40), "ends": (N - 1, 0)}[kind]
    idx = [i for i in idx if i < N]
    if len(set(idx)) < 2:
        return None
    v = dist[b].max() + 0.25
    dist[b, idx] = v
    return min(idx)


@pytest.mark.parametrize("B", [1, 1000])
@pytest.mark.parametrize("N", [1, 255, 256, 257, 5000])
def test_kl_loss_pred_vs_fp64(B, N):
    """Per-question KL and case_valid, the batch mean (a serial sum over B questions) and the argmax, bit-exact.
    Ties within one thread's strided chunk, across lanes, across warps and between index 0 and N - 1; fractional
    teachers, a teacher summing to 0 (loss_q exactly 0), dist = 0 under a positive teacher."""
    rs = np.random.RandomState(B + N)
    dist = torch.softmax(torch.from_numpy(rs.randn(B, N) * 3), 1).float()
    teacher = torch.zeros(B, N)
    for b in range(B):
        k = rs.randint(1, min(N, 6) + 1)
        teacher[b, torch.from_numpy(rs.choice(N, k, replace=False))] = torch.from_numpy(
            rs.uniform(0.1, 1.0, size=k).astype(np.float32))
    kinds = ["lanes", "chunk", "warps", "ends"]
    want_pred = {}
    for b in range(min(B, 8)):
        want_pred[b] = _tie(dist, b, kinds[b % 4], N)
    if B > 1:
        teacher[9] = 0.0                                          # no answer: case_valid 0
        teacher[10, :] = 0.0
        teacher[10, N - 1] = 0.7
        dist[10, N - 1] = 0.0                                     # dist = 0 where the teacher is > 0
        teacher[11] = torch.from_numpy(rs.uniform(0.0, 1.0, size=N).astype(np.float32))   # dense fractional
    dist, teacher = dist.to(DEV), teacher.to(DEV)
    loss_q, loss, pred = _nan(B), _nan(1), torch.full((B,), -5, dtype=torch.int64, device=DEV)
    _lib.check(_lib.load().gr_kl_loss_pred(_p(dist), _p(teacher), _p(loss_q), _p(loss), _p(pred), B, N,
                                           ops._stream()))
    torch.cuda.synchronize()
    wl, wq, valid, wpred = R.kl_loss_pred(dist, teacher)
    assert torch.equal(pred, wpred)
    for b, i in want_pred.items():
        assert i is None or pred[b].item() == i
    # bound: len and the KL sum are strided per-thread sums + a block tree (ceil(N/256) + 10 roundings each); t/len,
    # both logs and the products add a few u; all relative to sum tv (|log tv| + |log(p + 1e-8)| + 1)
    t, p = teacher.to(F64), dist.to(F64)
    tv = t / torch.where(t.sum(1, keepdim=True) > 0, t.sum(1, keepdim=True), torch.ones_like(t[:, :1]))
    A = (tv * (torch.log(torch.where(tv > 0, tv, torch.ones_like(tv))).abs() + torch.log(p + 1e-8).abs() + 1)).sum(1)
    eq = (2 * math.ceil(N / 256) + 32) * U * A * valid
    _check(loss_q, wq, eq + 1e-30, "loss_q")
    assert (loss_q[valid == 0] == 0).all()
    el = (eq.sum() + (B + 1) * U * wq.abs().sum()) / B + U * wl.abs()
    _check(loss, wl.view(1), el + 1e-30, "loss")


# --------------------------------------------------------------------------------------------------------------
# model level: the widest num_ins x entity_dim shapes the question kernels admit
# --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,I", [(400, 5), (256, 8)])
def test_rearev_eval_at_wide_instruction_shapes_vs_oracle(D, I):
    """ReaRev.eval() at (D = 400, I = 5) and (D = 256, I = 8): every question kernel runs at a width where
    (5I + 1) D is close to the query-reform limit; pred_dist within 1e-3 relative of the CPU oracle."""
    args = S.model_args("ReaRev", entity_dim=D, num_iter=2, num_ins=I, num_gnn=2, word_dim=32, use_cuda=True)
    torch.manual_seed(D + I)
    m = G.ReaRev(dict(args), 2000, 50, 100).eval()
    with torch.no_grad():
        m.reasoning.score_func.weight.mul_(20.0)
    b = S.make_batch(D + I, B=2, N=300, E=900, num_entity=2000, num_relation=50, num_word=100, multi_seed=True,
                     test=True)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    _, _, want = O.forward(sd, args, 2000, 100, b)
    _, _, dist, _ = m(b[:7])
    err = ((dist.cpu().double() - want.double()).abs() / want.double().clamp_min(1e-30)).max().item()
    assert err < 1e-3, err
