"""GraftNet training on the GPU kernels (csrc/graft.cu, csrc/aggregate_bwd.cu): the fact-message aggregation and its
backward, the fact-attention backward, the TypeLayer backward and the in-kernel dropout against float64 autograd of
the restatements below; the model's kernel path against its per-fact torch path; no per-fact activations saved for
backward; and a short training loop."""
import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import _lib, autograd_path, batching, ops, synthetic as S
from graft_train_ref import ref_aggregate as _ref_aggregate, ref_attention as _ref_attention

pytestmark = pytest.mark.gpu
EPS24 = 2.0 ** -24
dev = torch.device("cuda")


def _graft(B, N, maxF, R1, rs, per_q, head_hub=0, tail_hub=0):
    """Graft lists in the loader layout (permuted) with pad slots; question 0 may hold a head hub (node 0) and a tail hub
    (node N-1); node N-2 of question 0 has no facts -> GraftGraph and the staged facts as int64 host arrays."""
    kfr = np.full((B, maxF), R1 - 1, dtype=np.int64)
    hb, hf, he, tb, te, tf = ([] for _ in range(6))
    for b in range(B):
        n = min(per_q[b], maxF)
        slots = rs.permutation(maxF)[:n]
        kfr[b, slots] = rs.randint(0, R1 - 1, size=n)
        heads, tails = rs.randint(0, N, size=n), rs.randint(0, N, size=n)
        if b == 0:
            heads[:head_hub] = 0
            tails[n - tail_hub:] = N - 1
            heads[heads == N - 2] = 1
            tails[tails == N - 2] = 1
        hb += [b] * n; hf += list(slots); he += list(heads)
        perm = rs.permutation(n)
        tb += [b] * n; te += list(tails[perm]); tf += list(slots[perm])
    t = lambda a: torch.tensor(np.asarray(a, dtype=np.int64), device=dev)  # noqa: E731
    gg = ops.graft_stage([t(hb), t(hf), t(he)], [t(tb), t(te), t(tf)], t(kfr).view(B, maxF), B, N, R1)
    gg.check_status()
    n = int(gg.nfacts.item())
    st = {k: getattr(gg, k)[:n].long().cpu() for k in ("heads", "tails", "rels", "slot_of")}
    return gg, kfr, st


def _leaf(x):
    return x.detach().cpu().double().requires_grad_(True)


def _check(got, want, n, scale, what):
    """|got - want| <= n * 2^-24 * scale, element-wise (n: terms summed per element, scale: sum of their |.|)."""
    err = (got.detach().cpu().double() - want).abs()
    bound = n * EPS24 * scale + 1e-30
    bad = err > bound
    assert not bad.any(), (what, float(err[bad].max()), float(bound[bad].min()), int(bad.sum()))


def _run_aggregate(D, p, seed_val=1234, plant_zero=True):
    rs = np.random.RandomState(D)
    B, N, R1, maxF = 3, 40, 9, 3600
    gg, kfr, st = _graft(B, N, maxF, R1, rs, [3400, 0, 70], head_hub=2500, tail_hub=2500)   # question 1: no facts
    Nt, F_ = B * N, st["heads"].numel()
    self_tab = torch.tensor(rs.randn(R1, D), dtype=torch.float32)
    head_tab = torch.tensor(rs.randn(Nt, D), dtype=torch.float32)
    if plant_zero:                                     # self + head == 0 exactly: relu'(0) = 0 on both sides
        h0, r0 = int(st["heads"][0]), int(st["rels"][0])
        head_tab[h0, : (D + 1) // 2] = -self_tab[r0, : (D + 1) // 2]
    s = torch.tensor(rs.rand(F_), dtype=torch.float32)
    s[torch.as_tensor(rs.rand(F_) < 0.3)] = 0.0          # facts with s = 0 still get a gradient
    G_ = torch.tensor(rs.randn(Nt, D), dtype=torch.float32)
    seed = torch.tensor([seed_val], dtype=torch.int64, device=dev)
    mask = ops.graft_dropout_mask(seed, p, B * maxF, D).cpu() if p > 0 else None
    # forward
    sum_out = ops.graft_aggregate_train(gg, s.cuda(), self_tab.cuda(), head_tab.cuda(), seed, p)
    lt, lh, ls = _leaf(self_tab), _leaf(head_tab), _leaf(s)
    ref = _ref_aggregate(lt, lh, ls, st, Nt, mask, p)
    (ref * G_.double()).sum().backward()
    # backward into pre-filled buffers
    pre_s, pre_self, pre_head = (torch.tensor(rs.randn(*sh), dtype=torch.float32)
                                 for sh in ((F_,), (R1, D), (Nt, D)))
    gs, gself, ghead = pre_s.cuda(), pre_self.cuda(), pre_head.cuda()
    ops.graft_aggregate_backward(gg, s.cuda(), self_tab.cuda(), head_tab.cuda(), G_.cuda(), gs, gself, ghead, seed, p)
    # |.|-scales and term counts
    keep = (mask[st["slot_of"]].double() / (1 - p)) if mask is not None else torch.ones(F_, D, dtype=torch.float64)
    absa = self_tab.double()[st["rels"]].abs() + head_tab.double()[st["heads"]].abs()
    a = self_tab.double()[st["rels"]] + head_tab.double()[st["heads"]]
    Gt = G_.double()[st["tails"]] * keep
    sd = s.double().unsqueeze(1)
    deg_t = torch.bincount(st["tails"], minlength=Nt).double().unsqueeze(1)
    deg_h = torch.bincount(st["heads"], minlength=Nt).double().unsqueeze(1)
    deg_r = torch.bincount(st["rels"], minlength=R1).double().unsqueeze(1)
    sabs = torch.zeros(Nt, D, dtype=torch.float64).index_add(0, st["tails"], absa * sd * keep)
    _check(sum_out, ref.detach(), deg_t + 4, sabs, "sum_out")
    gterm = Gt.abs() * sd * (a > 0)
    _check(gs, pre_s.double() + ls.grad, D + 4, (Gt.abs() * absa).sum(1) + pre_s.double().abs(), "grad_s")
    _check(gself, pre_self.double() + lt.grad, deg_r + 3,
           torch.zeros(R1, D, dtype=torch.float64).index_add(0, st["rels"], gterm) + pre_self.double().abs(),
           "grad_self")
    _check(ghead, pre_head.double() + lh.grad, deg_h + 3,
           torch.zeros(Nt, D, dtype=torch.float64).index_add(0, st["heads"], gterm) + pre_head.double().abs(),
           "grad_head")
    return dict(s=s, grad_s=ls.grad, sum_out=sum_out, st=st, gg=gg)


@pytest.mark.parametrize("D", [1, 31, 50, 200, 256, 512])
def test_aggregate_forward_and_backward_match_fp64(D):
    """Per element |kernel - fp64| <= n 2^-24 * (sum of the |.| of the n terms summed): each term is formed with at
    most 3 fp32 roundings (self + head, * s, * 1/(1-p)) and the running sum adds one rounding per term, so n = (terms) +
    4 for the sums and D + 4 for grad_s (a D-term dot product).  The gradient buffers start pre-filled and the kernels
    add into them (one more rounding), so the pre-filled |.| joins the scale.  The relu mask agrees exactly: a
    rounded fp32 sum has the sign of the exact sum and is 0 only where it is exactly 0."""
    r = _run_aggregate(D, 0.0)
    zero_s = r["s"] == 0
    assert zero_s.any() and (r["grad_s"][zero_s] != 0).any()
    rp = r["gg"].graph.rowptr_t.cpu()
    assert (rp[1:41] - rp[:40]).max() >= 2500 and int(rp[39] - rp[38]) == 0      # tail hub, node without facts
    assert float(r["sum_out"][40:80].abs().max()) == 0.0                        # the question without facts


@pytest.mark.parametrize("D", [50, 200])
def test_aggregate_with_dropout_matches_fp64_with_the_same_mask(D):
    _run_aggregate(D, 0.2)


@pytest.mark.parametrize("D", [1, 200])
def test_aggregate_with_no_staged_facts(D):
    """F = 0 (no graft fact in the whole batch, e.g. one question without a subgraph): the forward is all zeros and
    the backward leaves the pre-filled gradient buffers as they were."""
    B, N, R1, maxF = 2, 5, 4, 6
    t = lambda a: torch.tensor(a, dtype=torch.int64, device=dev)  # noqa: E731
    kfr = torch.full((B, maxF), R1 - 1, dtype=torch.int64, device=dev)
    gg = ops.graft_stage([t([]), t([]), t([])], [t([]), t([]), t([])], kfr, B, N, R1)
    assert int(gg.nfacts.item()) == 0
    s = torch.empty(0, device=dev)
    self_tab, head_tab = torch.randn(R1, D, device=dev), torch.randn(B * N, D, device=dev)
    seed = torch.tensor([3], dtype=torch.int64, device=dev)
    for sd, p in ((None, 0.0), (seed, 0.2)):
        out = ops.graft_aggregate_train(gg, s, self_tab, head_tab, sd, p)
        assert out.shape == (B * N, D) and float(out.abs().max()) == 0.0
        gs, gself, ghead = torch.empty(0, device=dev), torch.randn(R1, D, device=dev), torch.randn(B * N, D, device=dev)
        keep = (gself.clone(), ghead.clone())
        ops.graft_aggregate_backward(gg, s, self_tab, head_tab, torch.randn(B * N, D, device=dev), gs, gself, ghead,
                                     sd, p)
        assert torch.equal(gself, keep[0]) and torch.equal(ghead, keep[1])
    gg.check_status()


@pytest.mark.parametrize("D,Q", [(1, 5), (31, 1), (50, 6), (200, 9), (256, 4), (512, 7), (512, 40)])
def test_attention_backward_matches_fp64(D, Q):
    """grad_qh[b,q] = sum_f c_fq rel[r_f], grad_rel[r] = sum_f sum_q c_fq qh[b,q], c_fq = g_f a_fq (1 + z_fq - W_f)/sqrt(D).

    Per element |kernel - fp64| <= (n_sum + n_term) 2^-24 * S, S = sum over the element's terms of
    |g| a (1 + |z| + |W|)(1 + Z_f) |x| / sqrt(D), with Z_f = max_q sum_c |qh_q||rel_r|/sqrt(D) the |.|-scale of z.
    * n_term, the roundings inside one term: the kernel recomputes z as a warp dot product (ceil(D/32) fused
      multiply-adds per lane and a 5-level shuffle tree, then the division), so |dz| <= (ceil(D/32) + 7) 2^-24 Z_f.  That
      error enters a_q twice through exp(z - max) and (1 + z - W) twice more (z and the recomputed W); the softmax sum
      over Q tokens, the exp, the reciprocal and the products forming c_q x add 2Q + 20 roundings relative to
      |.|(1 + |z| + |W|).  So n_term = 4 (ceil(D/32) + 7) + 2Q + 20.
    * n_sum, the summation: grad_qh[b] adds one term per slot of question b with grad_W != 0 (cnt_b) in shared memory,
      then one flush per block (ceil(max_fact/64)) into the pre-filled buffer; grad_rel[r] sums Q tokens per slot in
      registers, then one atomic per slot with relation r (cnt_r) into the pre-filled buffer.
    Q = 40 at D = 512 accumulates grad_qh in global memory (Q*D too large for shared memory)."""
    rs = np.random.RandomState(D + Q)
    B, N, R1, maxF = 4, 30, 11, 300
    gg, kfr, _st = _graft(B, N, maxF, R1, rs, [280, 0, 150, 1])
    qh = torch.tensor(rs.randn(B, Q, D), dtype=torch.float32)
    qmask = torch.tensor((rs.rand(B, Q) < 0.6).astype(np.float32))
    qmask[:, 0] = 1
    rel = torch.tensor(rs.randn(R1, D), dtype=torch.float32)
    gW = torch.tensor(rs.randn(B, maxF), dtype=torch.float32)
    gW[torch.as_tensor(kfr == R1 - 1)] = 0.0                     # pad slots: no gradient (skipped) ...
    gW[2, :5] = torch.tensor(rs.randn(5), dtype=torch.float32)   # ... except a few, which must count
    pre_q, pre_r = torch.tensor(rs.randn(B, Q, D), dtype=torch.float32), torch.tensor(rs.randn(R1, D), dtype=torch.float32)
    gq, gr = pre_q.cuda(), pre_r.cuda()
    ops.graft_attention_backward(gg, qh.cuda(), qmask.cuda(), rel.cuda(), gW.cuda().view(-1), gq, gr)
    lq, lr = _leaf(qh), _leaf(rel)
    W, a = _ref_attention(lq, qmask.double(), lr, kfr)
    (W * gW.double()).sum().backward()
    with torch.no_grad():
        qd, rd = qh.double(), rel.double()
        fe = rd[torch.as_tensor(kfr)]                                           # [B, maxF, D]
        z = torch.bmm(qd, fe.transpose(1, 2)) / np.sqrt(D)                      # [B, Q, maxF]
        Zf = (torch.bmm(qd.abs(), fe.abs().transpose(1, 2)) / np.sqrt(D)).amax(1, keepdim=True)
        coef = gW.double().abs().unsqueeze(1) * a * (1 + z.abs() + W.abs().unsqueeze(1)) * (1 + Zf) / np.sqrt(D)
        scale_q = torch.bmm(coef, fe.abs()) + pre_q.double().abs()              # [B, Q, D]
        scale_r = torch.zeros(R1, D, dtype=torch.float64).index_add(
            0, torch.as_tensor(kfr).view(-1), torch.bmm(coef.transpose(1, 2), qd.abs()).view(-1, D)) + pre_r.double().abs()
        live = (gW != 0)
        cnt_b = live.sum(1).double().view(B, 1, 1)
        cnt_r = torch.zeros(R1, dtype=torch.float64).index_add(0, torch.as_tensor(kfr).view(-1),
                                                               live.view(-1).double()).view(R1, 1)
    n_term = 4 * (-(-D // 32) + 7) + 2 * Q + 20
    _check(gq, pre_q.double() + lq.grad, cnt_b + -(-maxF // 64) + 2 + n_term, scale_q, "grad_qh")
    _check(gr, pre_r.double() + lr.grad, cnt_r + Q + 2 + n_term, scale_r, "grad_rel")
    masked = qmask == 0
    assert torch.equal(gq.cpu()[masked], pre_q[masked])           # masked tokens get nothing
    gq1 = torch.zeros(B, Q, D, device=dev)
    ops.graft_attention_backward(gg, qh.cuda(), qmask.cuda(), rel.cuda(), gW.cuda().view(-1), gq1, torch.zeros_like(gr))
    assert float(gq1[1].abs().max()) == 0.0                       # question 1 has no facts: all its slots are pads


@pytest.mark.parametrize("D", [1, 31, 50, 200, 256, 512])
@pytest.mark.parametrize("weighted", [False, True])
def test_type_layer_backward_matches_fp64(D, weighted):
    """grad_table[r] = sum over both CSR lists of w_e (G * [out > 0])[n]: n = terms per relation + 2 (runs of equal
    relations inside a row are merged into one coefficient first), scale = sum of |w G| plus the pre-filled value.
    The relu mask is taken from the given ``out`` (strictly > 0), which holds exact zeros here."""
    rs = np.random.RandomState(D + 7 * weighted)
    B, N, R1 = 3, 50, 13
    b = S.make_batch(D, B=B, N=N, E=400, num_entity=500, num_relation=R1 - 1, num_word=20, powerlaw=True,
                     n_real="ragged", with_weights=True)
    db = batching.stage_batch(b, dev, R1, False, weighted)
    g = db.graph
    heads, rels, tails = (torch.as_tensor(np.asarray(x, dtype=np.int64)) for x in b[2][:3])
    w = torch.as_tensor(np.asarray(b[2][6], dtype=np.float64)) if weighted else torch.ones(len(heads), dtype=torch.float64)
    Nt = B * N
    G_ = torch.tensor(rs.randn(Nt, D), dtype=torch.float32)
    out = torch.tensor(rs.randn(Nt, D), dtype=torch.float32)
    out[torch.as_tensor(rs.rand(Nt, D) < 0.2)] = 0.0
    pre = torch.tensor(rs.randn(R1, D), dtype=torch.float32)
    gt = pre.cuda()
    ops.type_layer_backward(g, G_.cuda(), out.cuda(), gt, g.wr_t if weighted else None, g.wr_h if weighted else None)
    Gm = G_.double() * (out > 0)
    contrib = (Gm[tails] + Gm[heads]) * w.unsqueeze(1)
    want = pre.double() + torch.zeros(R1, D, dtype=torch.float64).index_add(0, rels, contrib)
    scale = torch.zeros(R1, D, dtype=torch.float64).index_add(0, rels, (Gm[tails].abs() + Gm[heads].abs())
                                                              * w.unsqueeze(1)) + pre.double().abs()
    cnt = 2 * torch.bincount(rels, minlength=R1).double().unsqueeze(1)
    _check(gt, want, cnt + 2, scale, "grad_table")


def test_type_layer_through_autograd_matches_fp64():
    """_TypeLayerFn (gr_type_layer forward, gr_type_layer_backward) against float64 autograd of the per-fact sum."""
    D, B, N, R1 = 64, 2, 40, 9
    b = S.make_batch(3, B=B, N=N, E=300, num_entity=500, num_relation=R1 - 1, num_word=20)
    g = batching.stage_batch(b, dev, R1).graph
    rs = np.random.RandomState(0)
    table = torch.tensor(rs.randn(R1, D), dtype=torch.float32, device=dev, requires_grad=True)
    out = autograd_path._TypeLayerFn.apply(table, g, None, None)
    Gr = torch.tensor(rs.randn(B * N, D), dtype=torch.float32, device=dev)
    (out * Gr).sum().backward()
    heads, rels, tails = (torch.as_tensor(np.asarray(x, dtype=np.int64)) for x in b[2][:3])
    t64 = table.detach().cpu().double().requires_grad_(True)
    fv = t64[rels]
    ref = torch.relu(torch.zeros(B * N, D, dtype=torch.float64).index_add(0, tails, fv).index_add(0, heads, fv))
    (ref * Gr.cpu().double()).sum().backward()
    assert torch.allclose(out.detach().cpu().double(), ref.detach(), rtol=1e-5, atol=1e-5)
    assert torch.allclose(table.grad.cpu().double(), t64.grad, rtol=1e-5, atol=1e-4)


def test_refusals():
    L = _lib.load()
    assert L.gr_graft_dropout_mask(None, 0.5, 10, 8, None, None) == -1
    assert L.gr_graft_dropout_mask(None, 1.0, 10, 8, None, None) == -1
    x = torch.zeros(16, device=dev)
    xp = x.data_ptr()
    assert L.gr_graft_aggregate_train(xp, xp, xp, xp, xp, xp, xp, 8, xp, 8, None, 0.0, xp, 8, 1, 2, 600, None) == -1
    assert L.gr_graft_aggregate_train(xp, xp, xp, xp, xp, xp, xp, 8, xp, 8, None, 0.3, xp, 8, 1, 2, 8, None) == -1
    assert L.gr_graft_aggregate_train(xp, xp, xp, xp, xp, xp, xp, 4, xp, 8, None, 0.0, xp, 8, 1, 2, 8, None) == -1
    assert L.gr_graft_aggregate_backward(xp, xp, xp, xp, xp, xp, xp, 8, xp, 8, None, 0.0, xp, 8, None, xp, 8, xp, 8,
                                         1, 2, 8, None) == -1
    assert L.gr_graft_attention_backward(xp, xp, 0, xp, 8, 3, xp, 1, 4, 8, xp, xp, xp, 8, None) == -1
    assert L.gr_graft_attention_backward(xp, xp, 2, xp, 8, 3, xp, 1, 4, 8, None, xp, xp, 8, None) == -1
    assert L.gr_type_layer_backward(xp, xp, None, xp, xp, None, xp, 8, xp, 8, xp, 4, 1, 2, 8, 3, None) == -1
    assert b"leading dimension" in L.gr_last_error()
    with pytest.raises(_lib.GrError):
        ops.graft_dropout_mask(torch.zeros(1, dtype=torch.int64, device=dev), 0.2, 10, 1000)


# ---- dropout --------------------------------------------------------------------------------------------------------

def test_dropout_keep_fraction_and_seeds():
    S_, D, p = 5000, 256, 0.2                                   # 1.28e6 elements
    sa = torch.tensor([7], dtype=torch.int64, device=dev)
    m = ops.graft_dropout_mask(sa, p, S_, D)
    n = m.numel()
    frac = float(m.double().mean())
    assert abs(frac - (1 - p)) <= 5 * np.sqrt(p * (1 - p) / n), frac
    m2 = ops.graft_dropout_mask(torch.tensor([8], dtype=torch.int64, device=dev), p, S_, D)
    assert float((m != m2).double().mean()) > 0.2                # independent masks differ in ~2p(1-p) = 32%
    assert torch.equal(m, ops.graft_dropout_mask(sa, p, S_, D))  # same seed, same mask
    assert torch.equal(m[:100], ops.graft_dropout_mask(sa, p, 100, D))   # keyed by slot, not by the call's size
    assert bool((ops.graft_dropout_mask(sa, 0.0, 10, D) == 1).all())


def test_p_zero_is_the_no_dropout_path_bit_for_bit():
    """p = 0 (seed given or not) equals the kernel without dropout and the inference kernel's sum, bit for bit."""
    rs = np.random.RandomState(3)
    B, N, R1, maxF, D = 2, 30, 7, 200, 96
    gg, _kfr, st = _graft(B, N, maxF, R1, rs, [150, 90])
    Wt = torch.tensor(rs.rand(B * maxF), dtype=torch.float32, device=dev)
    E = torch.tensor(rs.rand(B * N) + 0.1, dtype=torch.float32, device=dev)
    prior = torch.tensor(rs.rand(B, N), dtype=torch.float32, device=dev)
    self_tab = torch.tensor(rs.randn(R1, D), dtype=torch.float32, device=dev)
    head_tab = torch.tensor(rs.randn(B * N, D), dtype=torch.float32, device=dev)
    slot, head = st["slot_of"].to(dev), st["heads"].to(dev)
    s = Wt[slot] * (prior.view(-1) / E)[head]                  # the training path's s (graft_gnn.py:97)
    seed = torch.tensor([99], dtype=torch.int64, device=dev)
    a = ops.graft_aggregate_train(gg, s, self_tab, head_tab)
    b = ops.graft_aggregate_train(gg, s, self_tab, head_tab, seed, 0.0)
    ref = torch.empty(B * N, D, device=dev)
    ops.graft_aggregate(gg, Wt, E, prior, self_tab, head_tab, 0.8, sum_out=ref)
    assert torch.equal(a, b) and torch.equal(a, ref)
    c = ops.graft_aggregate_train(gg, s, self_tab, head_tab, seed, 0.5)
    assert not torch.equal(a, c)


def _graft_model(D, dropout, num_relation=40, num_word=100, num_entity=1000, seed=0, **over):
    args = S.model_args("GraftNet", entity_dim=D, num_layer=3, use_cuda=True, linear_dropout=dropout, lm_dropout=0.0,
                        **over)
    torch.manual_seed(seed)
    return G.GraftNet(args, num_entity, num_relation, num_word).cuda()


def test_eval_mode_passes_p_zero(monkeypatch):
    m = _graft_model(32, 0.3)
    b = S.make_graft_batch(1, B=3, N=40, E=120, num_entity=1000, num_relation=40, num_word=100)
    seen = []
    orig = ops.graft_aggregate_train

    def spy(gg, s, self_tab, head_tab, seed=None, p=0.0, sum_out=None):
        seen.append((seed, p))
        return orig(gg, s, self_tab, head_tab, seed, p, sum_out)
    monkeypatch.setattr(ops, "graft_aggregate_train", spy)
    m.train()
    m(b, training=True)
    assert len(seen) == 3 and all(sd is not None and p == pytest.approx(0.3) for sd, p in seen)
    assert len({int(sd.item()) for sd, _ in seen}) == 3          # one seed per layer
    seen.clear()
    m.reasoning.linear_drop_train.eval()
    m(b, training=True)
    assert len(seen) == 3 and all(sd is None and p == 0.0 for sd, p in seen)


def test_permuted_graft_lists_keep_masks_and_loss():
    m = _graft_model(64, 0.2)
    m.train()
    b = S.make_graft_batch(5, B=4, N=60, E=300, num_entity=1000, num_relation=40, num_word=100, n_real="ragged")
    (hb, hf, he, v0), (tb, te, tf, v1) = b[3]
    rs = np.random.RandomState(1)
    p, q = rs.permutation(len(hb)), rs.permutation(len(tb))
    bp = list(b)
    bp[3] = ((hb[p], hf[p], he[p], v0), (tb[q], te[q], tf[q], v1))
    bp = tuple(bp)
    g1 = batching.stage_graft_batch(b, dev, 41).graft
    g2 = batching.stage_graft_batch(bp, dev, 41).graft
    n = int(g1.nfacts.item())
    assert n == int(g2.nfacts.item()) and torch.equal(g1.slot_of[:n], g2.slot_of[:n])
    seed = torch.tensor([5], dtype=torch.int64, device=dev)
    mask = ops.graft_dropout_mask(seed, 0.2, g1.B * g1.max_fact, 64)
    assert torch.equal(mask[g1.slot_of[:n].long()], mask[g2.slot_of[:n].long()])
    losses = []
    for batch in (b, bp):
        torch.manual_seed(123)
        losses.append(float(m(batch, training=True)[0].detach()))
    assert abs(losses[0] - losses[1]) <= 1e-6 * abs(losses[0]), losses


# ---- model level ----------------------------------------------------------------------------------------------------

def test_kernel_path_equals_torch_path_at_d200():
    """USE_KERNELS True vs False on one batch (dropout off, D = 200, power-law graft facts, ragged questions): loss and
    every parameter gradient within 2e-4 of the tensor's scale."""
    m = _graft_model(200, 0.0, num_entity=3000)
    m.train()
    b = S.make_graft_batch(61, B=6, N=300, E=1500, num_entity=3000, num_relation=40, num_word=100, powerlaw=True,
                           n_real="ragged")
    res = {}
    for mode in (True, False):
        autograd_path.USE_KERNELS = mode
        try:
            m.zero_grad()
            with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):    # keep cuDNN's LSTM in fp32: with
                loss = m(b, training=True)[0]                                    # TF32 its gradients alone differ
                loss.backward()                                                  # by ~1e-4 between two runs
        finally:
            autograd_path.USE_KERNELS = True
        res[mode] = (float(loss.detach()), {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None})
    assert abs(res[True][0] - res[False][0]) <= 2e-4 * abs(res[False][0])
    assert set(res[True][1]) == set(res[False][1])
    for k, r in res[False][1].items():
        a = res[True][1][k]
        assert (a - r).abs().max().item() <= 2e-4 * r.abs().max().item() + 1e-9, k


def _train_step_grads(m, b, kernels):
    autograd_path.USE_KERNELS = kernels
    try:
        m.zero_grad()
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            loss = m(b, training=True)[0]
            loss.backward()
    finally:
        autograd_path.USE_KERNELS = True
    return float(loss.detach()), {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}


def _assert_same_training(a, r):
    assert abs(a[0] - r[0]) <= 2e-4 * abs(r[0]) + 1e-12
    assert set(a[1]) == set(r[1])
    # plus 1e-5 of the model's largest gradient: the score bias has a mathematically zero gradient (softmax is shift
    # invariant), both paths hold rounding noise there
    gmax = max(g.abs().max().item() for g in r[1].values())
    for k, g in r[1].items():
        assert torch.isfinite(a[1][k]).all(), k
        assert (a[1][k] - g).abs().max().item() <= 2e-4 * g.abs().max().item() + 1e-5 * gmax + 1e-12, k


def test_training_on_a_batch_without_graft_facts():
    """No graft fact in the batch (F = 0) but kb facts for the TypeLayer, and a batch whose questions are all empty:
    the kernel path trains like the per-fact torch path."""
    m = _graft_model(64, 0.0)
    m.train()
    b = list(S.make_graft_batch(4, B=3, N=40, E=150, num_entity=1000, num_relation=40, num_word=100))
    z = np.zeros(0, dtype=np.int64)
    b[3] = ((z, z, z, np.ones(0)), (z, z, z, np.ones(0)))
    b = tuple(b)
    a, r = _train_step_grads(m, b, True), _train_step_grads(m, b, False)
    assert a[0] > 0
    _assert_same_training(a, r)
    e = S.make_graft_batch(4, B=2, N=20, E=50, num_entity=1000, num_relation=40, num_word=100, empty_questions=(0, 1))
    assert len(e[3][0][0]) == 0 and len(e[2][0]) == 0
    _assert_same_training(_train_step_grads(m, e, True), _train_step_grads(m, e, False))


def test_widths_beyond_the_kernels_keep_the_torch_path():
    """D > 512: the TypeLayer of ReaRev / NSM and GraftNet's fact-level work stay on the per-fact torch ops in
    training (as before the training kernels existed), so backward runs and matches USE_KERNELS = False."""
    D = 520
    assert not autograd_path._fact_kernels(dev, D) and autograd_path._fact_kernels(dev, 512)
    m = _graft_model(D, 0.0)
    m.train()
    b = S.make_graft_batch(6, B=2, N=30, E=90, num_entity=1000, num_relation=40, num_word=100)
    _assert_same_training(_train_step_grads(m, b, True), _train_step_grads(m, b, False))
    for name, cls in (("ReaRev", G.ReaRev), ("NSM", G.NSM)):
        args = S.model_args(name, entity_dim=D, num_iter=1, num_ins=1, num_gnn=1, num_step=1, use_cuda=True,
                            linear_dropout=0.0, lm_dropout=0.0)
        torch.manual_seed(0)
        mr = cls(args, 1000, 40, 100).cuda()
        mr.train()
        assert mr.encode_type
        br = S.make_batch(7, B=2, N=30, E=90, num_entity=1000, num_relation=40, num_word=100)
        _assert_same_training(_train_step_grads(mr, br, True), _train_step_grads(mr, br, False))


def _saved_numels(m, b):
    sizes = []

    def pack(t):
        sizes.append(t.numel())
        return t
    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        loss = m(b, training=True)[0]
    loss.backward()
    return sizes


def test_no_per_fact_activation_is_saved_for_backward():
    """B = 4, N = 500, 8000 graft facts per question, D = 64: nothing saved for backward on the kernel path has
    min(F_kb, F_graft, B*max_fact) * D / 2 elements; the per-fact torch path saves such tensors."""
    D = 64
    m = _graft_model(D, 0.2, num_relation=40, num_word=50, num_entity=600)
    m.train()
    b = S.make_graft_batch(2, B=4, N=500, E=8000, num_entity=600, num_relation=40, num_word=50)
    F_kb = len(b[2][0])
    F_graft = len(b[3][0][0])
    S_ = b[5].size
    assert F_graft >= 4 * 7000
    thresh = min(F_kb, F_graft, S_) * D // 2
    assert max(p.numel() for p in m.parameters()) < thresh
    big = [n for n in _saved_numels(m, b) if n >= thresh]
    assert not big, (big, thresh)
    autograd_path.USE_KERNELS = False
    try:
        assert any(n >= thresh for n in _saved_numels(m, b))
    finally:
        autograd_path.USE_KERNELS = True


def test_three_adam_steps_with_dropout_reduce_the_loss():
    m = _graft_model(64, 0.2)
    b = S.make_graft_batch(9, B=8, N=80, E=400, num_entity=1000, num_relation=40, num_word=100, n_real="ragged")
    m.train()
    torch.manual_seed(0)
    opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=5e-3)
    losses = []
    for _ in range(3):
        opt.zero_grad()
        loss, _, _, tp_list = m(b, training=True)
        loss.backward()
        torch.nn.utils.clip_grad_norm_([p for p in m.parameters()], 1.0)
        opt.step()
        losses.append(float(loss))
        assert len(tp_list) == 2 and len(tp_list[0]) == 8
    m.eval()
    final = float(m(b, training=True)[0])
    assert final < losses[0], (losses, final)
