"""The GraftNet kernels (csrc/graft.cu, and the TypeLayer backward of csrc/aggregate_bwd.cu that GraftNet trains)
against the float64 restatement in tests/graft_edges_ref.py, element by element under each element's own bound, at
the shapes where they branch:

* every width instantiation (NC = 1, 2, 4, 8, 16 columns chunks per lane) and both sides of each NC boundary, for the
  attention forward, the inference aggregate, the training aggregate and its backward, the attention backward and
  the TypeLayer backward, atomic and deterministic forms, plus the bf16 ``_ex`` forms at NC = 4;
* slots per question past W~'s 256-thread stride and the attention backward's 64-slot blocks, a head hub for E and
  grad_head and a tail hub for the aggregates, the shared / global memory switch of the attention backward, and its
  largest grid;
* relation windows of the deterministic backward: relations ending on, starting at and spanning 64-entry window
  edges, one relation holding 50 000 facts, many one-fact relations, and the last rows of a 6 107-row table;
* question masks (a fully masked question, Q from 1 to 64) and row views with a leading dimension above D.

Caller-owned outputs start at a sentinel, so a write outside the documented extent fails; gradient buffers start
pre-filled, so the accumulating kernels must add."""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import _lib, ops
import graft_edges_ref as R

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
EPS24 = 2.0 ** -24
BF = torch.bfloat16
WIDTHS = [1, 32, 33, 64, 65, 96, 128, 129, 256, 257, 511, 512]
PLANE_SENT = 0x7FC1          # a bf16 NaN bit pattern: plane columns the aggregate must not write


def _d(a):
    return torch.as_tensor(np.asarray(a, dtype=np.int64)).to(dev)


def _f32(rs, *shape):
    return torch.from_numpy(rs.randn(*shape).astype(np.float32))


def _view(rs, rows, D, pad):
    """A [rows, D] row view (leading dimension D + pad) of a random fp32 CUDA buffer, and the buffer."""
    buf = _f32(rs, rows, D + pad).to(dev)
    return buf[:, :D], buf


def _le(got, want, bound, what):
    """|got - want| <= bound element-wise (NaN fails); reports the worst offender."""
    err = (got.detach().cpu().double() - want).abs()
    bad = ~(err <= bound + 1e-30)
    assert not bad.any(), (what, int(bad.sum()), float(err[bad].max()), float(bound[bad].min()),
                           tuple(int(i) for i in bad.nonzero()[0]))


def _within(got, want_scale_n, pre, what):
    """got = pre + value within n 2^-24 (scale + |pre|): a kernel that adds into the pre-filled buffer ``pre``."""
    v, scale, n = want_scale_n
    pre = pre.detach().cpu().double()
    _le(got, pre + v, n * EPS24 * (scale + pre.abs()), what)


def _same_bits(a, b, what=""):
    torch.cuda.synchronize()
    assert a.dtype == b.dtype and a.shape == b.shape, what
    view = {4: torch.int32, 2: torch.int16, 1: torch.uint8}[a.element_size()]
    eq = a.contiguous().view(view) == b.contiguous().view(view)
    assert bool(eq.all()), "%s: %d of %d elements differ" % (what, int((~eq).sum()), eq.numel())


# ---- graft batches --------------------------------------------------------------------------------------------------

class Batch:
    """Facts (b, f, head, tail) with kb_fact_rel [B, M] staged by gr_graft_stage (tail list permuted, as the loader
    permutes it); ``st`` holds the staged facts, checked against the restatement's staging."""

    def __init__(self, rs, B, N, M, R1, b, f, head, tail, kfr):
        self.B, self.N, self.M, self.R1, self.Nt, self.kfr = B, N, M, R1, B * N, kfr
        b, f, head, tail = (np.asarray(x, dtype=np.int64) for x in (b, f, head, tail))
        p = rs.permutation(len(b))
        self.gg = ops.graft_stage([_d(b), _d(f), _d(head)], [_d(b[p]), _d(tail[p]), _d(f[p])],
                                  _d(kfr).view(B, M), B, N, R1)
        self.gg.check_status()
        n = int(self.gg.nfacts.item())
        self.st = {k: getattr(self.gg, k)[:n].long().cpu() for k in ("heads", "tails", "rels", "slot_of")}
        want = R.stage((b, f, head), (b[p], tail[p], f[p]), kfr, N)
        for k, v in want.items():
            assert torch.equal(self.st[k], v), k
        self.F = n


def random_batch(seed, B, N, M, R1, per_q, head_hub=0, tail_hub=0):
    """per_q[b] facts on random slots of question b (the others are pads of relation R1 - 1); question 0 may hold a
    head hub (node 0) and a tail hub (node N - 1)."""
    rs = np.random.RandomState(seed)
    kfr = np.full((B, M), R1 - 1, dtype=np.int64)
    cols = [[], [], [], []]
    for q, n in enumerate(per_q):
        slots = rs.permutation(M)[:n]
        kfr[q, slots] = rs.randint(0, R1 - 1, n)
        heads, tails = rs.randint(0, N, n), rs.randint(0, N, n)
        if q == 0:
            heads[:head_hub] = 0
            tails[n - tail_hub:] = N - 1
        for c, v in zip(cols, (np.full(n, q), slots, heads, tails)):
            c.append(v)
    b, f, h, t = (np.concatenate(c) if c else np.zeros(0, np.int64) for c in cols)
    return Batch(rs, B, N, M, R1, b, f, h, t, kfr)


@pytest.fixture(scope="module")
def wide():
    """The width cases' batch: question 0 holds 4 300 facts with a head hub and a tail hub of 4 100 facts each,
    question 1 has no facts (all pads), question 2 has 150 facts and every token masked."""
    g = random_batch(0, 3, 40, 4400, 12, [4300, 0, 150], head_hub=4100, tail_hub=4100)
    assert int(torch.bincount(g.st["heads"]).max()) >= 4097 and int(torch.bincount(g.st["tails"]).max()) >= 4097
    return g


def _question(rs, B, Q, D, masked=(2,)):
    qh = _f32(rs, B, Q, D)
    qmask = torch.from_numpy((rs.rand(B, Q) < 0.7).astype(np.float32))
    qmask[:, 0] = 1
    for b in masked:
        if b < B:
            qmask[b] = 0                                   # every token masked: the -1e11 offset everywhere
    return qh, qmask


# ---- attention forward ----------------------------------------------------------------------------------------------

def _check_attention(g, qh, qmask, rel):
    Q, D = qh.shape[1], qh.shape[2]
    W, Wt, E = ops.graft_attention(g.gg, qh.to(dev), qmask.to(dev), rel, out_w=True)
    if g.M == 0:                                     # no slots: E is the clamp on every node
        assert W.numel() == 0 and Wt.numel() == 0 and bool((E == np.float32(R.VERY_SMALL)).all())
        return None
    rel_c = rel.cpu()
    at = R.attention(qh, qmask, rel_c, g.kfr)
    n = 3 * Q * D + D + 8
    B, M = g.B, g.M
    _le(W.view(B, M), at["W"], n * EPS24 * (at["Wabs"] + at["W"].abs()), "W")
    rWt = R.w_tilde(at["W"])
    wb = R.w_tilde_bound(at["W"], at["Wabs"], Q, D)
    _le(Wt.view(B, M), rWt, wb, "W~")
    rE, raw, cnt = R.e_sum(rWt, g.st, g.Nt)
    # the errors of the summed W~ plus a serial sum's (terms + 2) roundings of the (non-negative) total
    # (and the clamp constant 1e-10 rounded to fp32)
    Eb = R._rows(g.st["heads"], wb.reshape(-1)[g.st["slot_of"]], g.Nt) + (cnt + 2) * EPS24 * raw + EPS24 * rE
    _le(E, rE, Eb, "E")
    g.gg.check_status()
    return at


@pytest.mark.parametrize("D", WIDTHS)
def test_attention_forward_widths(wide, D):
    rs = np.random.RandomState(D)
    qh, qmask = _question(rs, 3, 7, D)
    rel, _ = _view(rs, wide.R1, D, 3)
    at = _check_attention(wide, qh, qmask, rel)
    assert torch.equal(at["a"][2], torch.full_like(at["a"][2], 1 / 7))


@pytest.mark.parametrize("M", [0, 1, 63, 64, 65, 129, 255, 256, 257, 4096, 17_960])
def test_slots_per_question(M):
    """Forward and both attention backwards at max_fact around W~'s 256-thread stride and the backward's 64-slot
    blocks; 17 960 slots is 2 * max_tuples + N at a cfg2-like question.  Question 0 is full, question 1 has no
    facts."""
    B, N, R1, Q, D = 2, 30, 9, 5, 48
    g = random_batch(M, B, N, M, R1, [M, 0])
    rs = np.random.RandomState(M + 1)
    qh, qmask = _question(rs, B, Q, D, masked=())
    rel, _ = _view(rs, R1, D, 2)
    _check_attention(g, qh, qmask, rel)
    _check_attention_backward(g, qh, qmask, rel, rs)


@pytest.mark.parametrize("Q,D", [(1, 64), (31, 64), (32, 64), (33, 64), (64, 64), (32, 384), (33, 384), (24, 512)])
def test_tokens_per_question(Q, D):
    """Q from 1 to 64 with a fully masked question; Q * D = 12 288 (32 x 384, 24 x 512) is the last shape whose
    grad_qh accumulates in 48 KB of shared memory, 33 x 384 the first that accumulates in global memory."""
    g = random_batch(Q * 1000 + D, 3, 20, 200, 11, [180, 60, 90])
    rs = np.random.RandomState(Q + D)
    qh, qmask = _question(rs, 3, Q, D)
    rel, _ = _view(rs, 11, D, 5)
    _check_attention(g, qh, qmask, rel)
    _check_attention_backward(g, qh, qmask, rel, rs)


# ---- inference aggregate --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("D", WIDTHS)
def test_inference_aggregate_widths(wide, D):
    """sum_out (fp32 row view and the split-bf16 planes at col_sum = 0), the in-degree (at col_indeg = Dp), q2e (at
    col_q2e = 3 Dp) and prior_next; every other plane column, the rows past B*N and the view's padding keep their
    sentinels."""
    g, rs = wide, np.random.RandomState(100 + D)
    B, N, Nt = g.B, g.N, g.Nt
    Wt = torch.from_numpy(rs.rand(B * g.M).astype(np.float32)).to(dev)
    Wt[::5] = 0.0
    E = torch.from_numpy((rs.rand(Nt) + 0.1).astype(np.float32)).to(dev)
    E[::3] = 1e-10
    prior = torch.from_numpy((rs.rand(B, N) * (rs.rand(B, N) < 0.5)).astype(np.float32)).to(dev)
    self_tab, _ = _view(rs, g.R1, D, 3)
    head_tab, _ = _view(rs, Nt, D, 5)
    q2e = _f32(rs, B, D).to(dev)
    Dp = (D + 15) // 16 * 16
    hi = torch.full((Nt + 2, 5 * Dp), PLANE_SENT, dtype=torch.int16, device=dev).view(BF)
    lo = hi.clone()
    sum_buf = torch.full((Nt + 2, D + 4), float("nan"), device=dev)
    indeg = torch.full((Nt + 3,), float("nan"), device=dev)
    pn_buf = torch.full((Nt + 3,), float("nan"), device=dev)
    lam = 0.8
    ops.graft_aggregate(g.gg, Wt, E, prior, self_tab, head_tab, lam, q2e=q2e, sum_out=sum_buf[:Nt, :D],
                        planes=(hi[:Nt], lo[:Nt]), col_sum=0, col_indeg=Dp, col_q2e=3 * Dp, indeg_out=indeg[:Nt],
                        prior_next=pn_buf[:Nt].view(B, N))
    ag = R.aggregate(Wt.cpu(), E.cpu(), prior.cpu(), self_tab.cpu(), head_tab.cpu(), g.st, lam, Nt)
    n = 4 * (ag["indeg"].unsqueeze(1) + 3)
    bound = n * EPS24 * ag["sabs"]
    _le(sum_buf[:Nt, :D], ag["sum_out"], bound, "sum_out")
    assert bool(sum_buf[:Nt, D:].isnan().all()) and bool(sum_buf[Nt:].isnan().all())
    assert torch.equal(indeg[:Nt].cpu().double(), ag["indeg"]) and bool(indeg[Nt:].isnan().all())
    planes = (hi[:Nt].float() + lo[:Nt].float()).cpu().double()
    _le(planes[:, :D], ag["sum_out"], bound + 2.0 ** -17 * (ag["sum_out"].abs() + bound), "planes sum")
    assert torch.equal(planes[:, Dp], ag["indeg"])
    q2e_rows = q2e.cpu().double().repeat_interleave(N, 0)
    _le(planes[:, 3 * Dp:3 * Dp + D], q2e_rows, 2.0 ** -17 * q2e_rows.abs(), "planes q2e")
    written = torch.zeros(5 * Dp, dtype=torch.bool)
    written[:D] = written[Dp] = True
    written[3 * Dp:3 * Dp + D] = True
    for p in (hi, lo):
        bits = p.view(torch.int16).cpu()
        assert bool((bits[:Nt, ~written] == PLANE_SENT).all()) and bool((bits[Nt:] == PLANE_SENT).all())
    _le(pn_buf[:Nt], ag["prior_next"], (ag["indeg"] + 4) * 4 * EPS24 * ag["pn_scale"] + 1e-38, "prior_next")
    assert bool(pn_buf[Nt:].isnan().all())


# ---- training aggregate and its backward ----------------------------------------------------------------------------

def _train_inputs(g, D, rs, p, seed_val=1234):
    s = torch.from_numpy(rs.rand(g.F).astype(np.float32))
    s[torch.from_numpy(rs.rand(g.F) < 0.3)] = 0.0                   # facts with s = 0 still get a gradient
    self_tab, self_buf = _view(rs, g.R1, D, 3)
    head_tab, _ = _view(rs, g.Nt, D, 5)
    if g.F:                                                          # self + head == 0 exactly: relu'(0) = 0
        h0, r0 = int(g.st["heads"][0]), int(g.st["rels"][0])
        head_tab[h0, : (D + 1) // 2] = -self_tab[r0, : (D + 1) // 2]
    G, _ = _view(rs, g.Nt, D, 1)
    seed = torch.tensor([seed_val], dtype=torch.int64, device=dev)
    mask = ops.graft_dropout_mask(seed, p, g.B * g.M, D).cpu() if p > 0 else None
    return dict(s=s.to(dev), self_tab=self_tab, head_tab=head_tab, G=G, seed=seed, p=p, mask=mask)


def _train_backward(g, c, deterministic, rs, pads=(3, 2)):
    """One backward into pre-filled buffers (grad_self and grad_head as row views) -> (buffers, pre-filled copies)."""
    D = c["self_tab"].shape[1]
    gs = _f32(rs, g.F).to(dev)
    gself, gself_buf = _view(rs, g.R1, D, pads[0])
    ghead, ghead_buf = _view(rs, g.Nt, D, pads[1])
    pre = (gs.clone(), gself_buf.clone(), ghead_buf.clone())
    ops.graft_aggregate_backward(g.gg, c["s"], c["self_tab"], c["head_tab"], c["G"], gs, gself, ghead, c["seed"],
                                 c["p"], deterministic=deterministic)
    return (gs, gself_buf, ghead_buf), pre


def _check_train_backward(g, c, bufs, pre, ref):
    D = c["self_tab"].shape[1]
    gs, gself_buf, ghead_buf = bufs
    _within(gs, ref["grad_s"], pre[0], "grad_s")
    _within(gself_buf[:, :D], ref["grad_self"], pre[1][:, :D], "grad_self")
    _within(ghead_buf[:, :D], ref["grad_head"], pre[2][:, :D], "grad_head")
    _same_bits(gself_buf[:, D:], pre[1][:, D:], "grad_self padding")
    _same_bits(ghead_buf[:, D:], pre[2][:, D:], "grad_head padding")


def _train_ref(g, c):
    cpu = {k: c[k].cpu() for k in ("self_tab", "head_tab", "s", "G")}
    return R.train_aggregate_backward(cpu["self_tab"], cpu["head_tab"], cpu["s"], cpu["G"], g.st, g.Nt, c["mask"],
                                      c["p"])


@pytest.mark.parametrize("D", WIDTHS)
def test_train_aggregate_widths(wide, D):
    """Forward (into a NaN-filled row view) and the atomic and deterministic backward with dropout p = 0.2, the mask
    taken from gr_graft_dropout_mask."""
    g, rs = wide, np.random.RandomState(200 + D)
    c = _train_inputs(g, D, rs, 0.2)
    out_buf = torch.full((g.Nt + 1, D + 3), float("nan"), device=dev)
    ops.graft_aggregate_train(g.gg, c["s"], c["self_tab"], c["head_tab"], c["seed"], c["p"],
                              sum_out=out_buf[:g.Nt, :D])
    cpu = {k: c[k].cpu() for k in ("self_tab", "head_tab", "s")}
    want = R.train_aggregate(cpu["self_tab"].double(), cpu["head_tab"].double(), cpu["s"].double(), g.st, g.Nt,
                             c["mask"], c["p"])
    scale, n = R.train_aggregate_scale(cpu["self_tab"], cpu["head_tab"], cpu["s"], g.st, g.Nt, c["mask"], c["p"])
    _le(out_buf[:g.Nt, :D], want, n * EPS24 * scale, "sum_out")
    assert bool(out_buf[:g.Nt, D:].isnan().all()) and bool(out_buf[g.Nt:].isnan().all())
    ref = _train_ref(g, c)
    for det in (False, True):
        _check_train_backward(g, c, *_train_backward(g, c, det, rs), ref)


# ---- attention backward ---------------------------------------------------------------------------------------------

def _check_attention_backward(g, qh, qmask, rel, rs, deterministic=(False, True)):
    B, Q, D = qh.shape
    gW = _f32(rs, B, g.M)
    gW[torch.from_numpy(g.kfr == g.R1 - 1)] = 0.0                  # pad slots: no gradient (skipped) ...
    gW[0, : min(5, g.M)] = _f32(rs, min(5, g.M))                    # ... except a few, which must count
    ref = R.attention_backward(qh, qmask, rel.cpu(), g.kfr, gW)
    out = {}
    for det in deterministic:
        gq = _f32(rs, B, Q, D).to(dev)
        gr, gr_buf = _view(rs, g.R1, D, 3)
        pre_q, pre_r = gq.clone(), gr_buf.clone()
        ops.graft_attention_backward(g.gg, qh.to(dev), qmask.to(dev), rel, gW.to(dev).view(-1), gq, gr,
                                     deterministic=det)
        _within(gq, ref["grad_qh"], pre_q, "grad_qh det=%s" % det)
        _within(gr, ref["grad_rel"], pre_r[:, :D], "grad_rel det=%s" % det)
        _same_bits(gr_buf[:, D:], pre_r[:, D:], "grad_rel padding")
        partly = (qmask == 0) & (qmask.sum(1, keepdim=True) > 0)
        assert torch.equal(gq.cpu()[partly], pre_q.cpu()[partly])   # masked tokens of a live question get nothing
        out[det] = (gq, gr_buf)
    return out


@pytest.mark.parametrize("D", WIDTHS)
def test_attention_backward_widths(wide, D):
    rs = np.random.RandomState(300 + D)
    qh, qmask = _question(rs, 3, 7, D)
    rel, _ = _view(rs, wide.R1, D, 3)
    _check_attention_backward(wide, qh, qmask, rel, rs)


def test_attention_backward_batch_limit():
    """B = 65 535 (the largest grid.y) is accepted and correct; B = 65 536 is refused by the atomic kernel and run
    correctly by the deterministic one."""
    for B in (65535, 65536):
        rs = np.random.RandomState(B)
        g = Batch(rs, B, 1, 2, 3, [], [], [], [], rs.randint(0, 2, (B, 2)))     # no facts, no pad slots
        qh, qmask = _question(rs, B, 2, 3, masked=(7,))
        rel, _ = _view(rs, 3, 3, 1)
        if B == 65535:
            _check_attention_backward(g, qh, qmask, rel, rs)
            continue
        gq = torch.zeros(B, 2, 3, device=dev)
        with pytest.raises(_lib.GrError, match="B <= 65535"):
            ops.graft_attention_backward(g.gg, qh.to(dev), qmask.to(dev), rel, torch.ones(B * 2, device=dev), gq,
                                         torch.zeros(3, 3, device=dev))
        _check_attention_backward(g, qh, qmask, rel, rs, deterministic=(True,))


# ---- TypeLayer backward ---------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def typed():
    """A TypeLayer batch: B = 2, N = 50, 6 000 facts over 13 relations with a 4 200-fact head hub, weighted."""
    rs = np.random.RandomState(7)
    B, N, R1, F_ = 2, 50, 13, 6000
    q = rs.randint(0, B, F_)
    heads, tails, rels = q * N + rs.randint(0, N, F_), q * N + rs.randint(0, N, F_), rs.randint(0, R1, F_)
    heads[:4200] = 0
    heads, tails, rels = (torch.from_numpy(x.astype(np.int64)) for x in (heads, tails, rels))
    g = ops.csr_build(heads.to(dev), rels.to(dev), tails.to(dev), B, N, R1)
    w = torch.from_numpy(rs.uniform(0.1, 1.7, F_).astype(np.float32)).to(dev)
    return dict(g=g, heads=heads, rels=rels, tails=tails, w=w, w_t=ops.gather_f32(w, g.fact_t),
                w_h=ops.gather_f32(w, g.fact_h), R1=R1, Nt=B * N)


@pytest.mark.parametrize("D", WIDTHS)
def test_type_layer_backward_widths(typed, D):
    """grad_table (a pre-filled row view) from the relu mask of ``out`` (which holds exact zeros), atomic and
    deterministic."""
    t, rs = typed, np.random.RandomState(400 + D)
    G, _ = _view(rs, t["Nt"], D, 2)
    out, _ = _view(rs, t["Nt"], D, 1)
    out[torch.from_numpy(rs.rand(t["Nt"], D) < 0.2).to(dev)] = 0.0
    ref = R.type_layer_backward(G.cpu(), out.cpu(), t["heads"], t["rels"], t["tails"], t["R1"], t["w"].cpu())
    for det in (False, True):
        gt, gt_buf = _view(rs, t["R1"], D, 3)
        pre = gt_buf.clone()
        ops.type_layer_backward(t["g"], G, out, gt, t["w_t"], t["w_h"], deterministic=det)
        _within(gt, ref, pre[:, :D], "grad_table det=%s" % det)
        _same_bits(gt_buf[:, D:], pre[:, D:], "grad_table padding")


# ---- bf16 node tensors at NC = 4 ------------------------------------------------------------------------------------

def test_bf16_ex_forms_at_nc4(wide):
    """D = 96: the bf16 forward equals the fp32 kernel's output rounded to bf16; the backward's owned sums (grad_s,
    grad_head) and the deterministic grad_self and grad_table equal the fp32 kernels on the upcast inputs."""
    D, g, rs = 96, wide, np.random.RandomState(96)
    c = _train_inputs(g, D, rs, 0.2)
    head16 = c["head_tab"].to(BF)
    G16 = c["G"].to(BF)
    out16 = ops.graft_aggregate_train(g.gg, c["s"], c["self_tab"], head16, c["seed"], c["p"])
    out32 = ops.graft_aggregate_train(g.gg, c["s"], c["self_tab"], head16.float(), c["seed"], c["p"])
    _same_bits(out16, out32.to(BF), "sum_out")
    pre = [_f32(rs, g.F).to(dev), _f32(rs, g.R1, D).to(dev), _f32(rs, g.Nt, D).to(BF).float().to(dev)]
    for det in (False, True):
        res = []
        for head, G, dt in ((head16, G16, BF), (head16.float(), G16.float(), torch.float32)):
            gs, gself, ghead = pre[0].clone(), pre[1].clone(), pre[2].to(dt, copy=True)
            ops.graft_aggregate_backward(g.gg, c["s"], c["self_tab"], head, G, gs, gself, ghead, c["seed"], c["p"],
                                         deterministic=det)
            res.append((gs, gself, ghead))
        _same_bits(res[0][0], res[1][0], "grad_s")
        _same_bits(res[0][2], res[1][2].to(BF), "grad_head")
        if det:
            _same_bits(res[0][1], res[1][1], "grad_self")
    t = _typed_bf16(rs, D)
    _same_bits(t[0], t[1], "grad_table")


def _typed_bf16(rs, D):
    B, N, R1, F_ = 2, 30, 7, 500
    q = rs.randint(0, B, F_)
    g = ops.csr_build(_d(q * N + rs.randint(0, N, F_)), _d(rs.randint(0, R1, F_)), _d(q * N + rs.randint(0, N, F_)),
                      B, N, R1)
    out16 = _f32(rs, B * N, D).to(dev).to(BF)
    out16[torch.from_numpy(rs.rand(B * N, D) < 0.2).to(dev)] = 0
    G16 = _f32(rs, B * N, D).to(dev).to(BF)
    pre = _f32(rs, R1, D).to(dev)
    got, want = pre.clone(), pre.clone()
    ops.type_layer_backward(g, G16, out16, got, deterministic=True)
    ops.type_layer_backward(g, G16.float(), out16.float(), want, deterministic=True)
    return got, want


# ---- relation windows of the deterministic backward -----------------------------------------------------------------

# facts (= slots) per relation, in relation order: relation 0 ends on the window edge 64, relation 2 crosses 128 and
# ends on 192, relation 3 starts on 192 and spans three windows, then 100 one-fact relations share windows 5 and 6,
# and 129, 63, 64, 65 facts cross the edges after them
EDGE_COUNTS = [64, 63, 65, 129] + [1] * 100 + [129, 63, 64, 65, 1, 1]


def _window_batch(case):
    rs = np.random.RandomState(len(case))
    if case == "edges":
        rels = np.repeat(np.arange(len(EDGE_COUNTS)), EDGE_COUNTS)
        B, N, R1 = 2, 30, len(EDGE_COUNTS) + 1
    elif case == "one_relation":                 # every fact of a 50 000-fact batch in relation 0
        rels = np.zeros(50_000, dtype=np.int64)
        B, N, R1 = 2, 40, 3
    else:                                        # relation ids in the last rows of a WebQSP-sized table
        R1, B, N = 6107, 3, 25
        rels = rs.randint(R1 - 7, R1, 3 * 250)
    T = len(rels)
    M = T // B
    assert M * B == T
    slots = rs.permutation(T)                    # every slot holds a fact: the slot index sees the same counts
    kfr = np.empty(T, dtype=np.int64)
    kfr[slots] = rels
    b, f = slots // M, slots % M
    return Batch(rs, B, N, M, R1, b, f, rs.randint(0, N, T), rs.randint(0, N, T), kfr.reshape(B, M))


@pytest.mark.parametrize("case", ["edges", "one_relation", "last_rows"])
@pytest.mark.parametrize("D", [33, 96])
def test_relation_windows(case, D):
    """grad_self of the aggregate backward and grad_rel of the attention backward in their deterministic forms,
    against float64 and bit-identical between two runs; relation rows no fact uses keep their pre-filled bits."""
    g = _window_batch(case)
    counts = torch.bincount(g.st["rels"], minlength=g.R1)
    if case == "edges":
        assert counts[:len(EDGE_COUNTS)].tolist() == EDGE_COUNTS
    rs = np.random.RandomState(D)
    c = _train_inputs(g, D, rs, 0.2 if case == "edges" else 0.0)
    ref = _train_ref(g, c)
    runs = []
    for _ in range(2):
        bufs, pre = _train_backward(g, c, True, np.random.RandomState(5))
        _check_train_backward(g, c, bufs, pre, ref)
        runs.append(bufs)
    for a, b in zip(*runs):
        _same_bits(a, b, "repeat")
    unused = (counts == 0).nonzero().view(-1).to(dev)
    _same_bits(runs[0][1][unused], pre[1][unused], "unused relation rows")
    qh, qmask = _question(rs, g.B, 4, D)
    rel, _ = _view(rs, g.R1, D, 3)
    rs_a = np.random.RandomState(9)
    first = _check_attention_backward(g, qh, qmask, rel, rs_a, deterministic=(True,))[True]
    second = _check_attention_backward(g, qh, qmask, rel, np.random.RandomState(9), deterministic=(True,))[True]
    for a, b in zip(first, second):
        _same_bits(a, b, "repeat")
