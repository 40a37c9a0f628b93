"""GraftNet on the GPU: the new kernels (csrc/graft.cu) against float64 restatements at their edge shapes, the full
forward against the reference goldens (tests/golden/graft/*.npz), the evaluator's lists, ties, determinism, refusal of
out-of-range ids, and the training path against the reference's gradients."""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import autograd_path, batching, evaluate, ops, synthetic as S
from test_graftnet_host import CASES, NUM_ENTITY, TRAIN_CASES, GraftGolden, load_model

pytestmark = pytest.mark.gpu
EPS24 = 2.0 ** -24
dev = torch.device("cuda")


def _graph(B, N, maxF, R1, rs, facts_per_q, hub=None):
    """Random graft lists (loader layout, permuted) + kb_fact_rel with pad slots -> (GraftGraph, host arrays)."""
    kfr = np.full((B, maxF), R1 - 1, dtype=np.int64)
    hb, hf, he, tb, te, tf = ([] for _ in range(6))
    for b in range(B):
        n = min(facts_per_q[b], maxF)
        slots = rs.permutation(maxF)[:n]
        kfr[b, slots] = rs.randint(0, R1 - 1, size=n)                  # R1 - 1: the pad relation
        heads = rs.randint(0, N, size=n)
        tails = rs.randint(0, N, size=n)
        if hub is not None and b == 0:
            tails[: hub] = N - 1
        hb += [b] * n; hf += list(slots); he += list(heads)
        perm = rs.permutation(n)
        tb += [b] * n; te += list(tails[perm]); tf += list(slots[perm])
    t = lambda a: torch.tensor(np.asarray(a, dtype=np.int64), device=dev)  # noqa: E731
    gg = ops.graft_stage([t(hb), t(hf), t(he)], [t(tb), t(te), t(tf)], t(kfr).view(B, maxF), B, N, R1)
    facts = dict(b=np.array(hb), f=np.array(hf), head=np.array(he))
    return gg, kfr, facts


def _fp64_attention(qh, qmask, rel, kfr, facts, B, N):
    qh, rel = qh.double(), rel.double()
    D = rel.shape[1]
    fe = rel[torch.as_tensor(kfr)]
    sim = torch.bmm(qh, fe.transpose(1, 2)) / np.sqrt(D) + (1 - qmask.double().unsqueeze(2)) * -1e11
    a = torch.softmax(sim, 1)
    W = (torch.bmm(a.transpose(1, 2), qh) * fe).sum(2) / np.sqrt(D)
    Wt = torch.exp(W - W.max(1, keepdim=True)[0])
    E = torch.zeros(B * N, dtype=torch.float64)
    E.index_add_(0, torch.as_tensor(facts["b"] * N + facts["head"]), Wt[facts["b"], facts["f"]])
    # |.|-scale of W: sum_q a_q |qh| . |rel| / sqrt(D)
    Wabs = (torch.bmm(a.transpose(1, 2), qh.abs()) * fe.abs()).sum(2) / np.sqrt(D)
    return W, Wt, E.clamp(min=1e-10), Wabs


@pytest.mark.parametrize("D", [1, 7, 32, 50, 96, 200, 256, 400])
def test_attention_kernel_matches_fp64(D):
    rs = np.random.RandomState(D)
    B, N, Q, R1, maxF = 3, 17, 6, 9, 40
    gg, kfr, facts = _graph(B, N, maxF, R1, rs, [30, 0, 12])        # question 1: no facts
    qh = torch.tensor(rs.randn(B, Q, D), dtype=torch.float32)
    qmask = torch.tensor((rs.rand(B, Q) < 0.7).astype(np.float32))
    qmask[:, 0] = 1
    rel = torch.tensor(rs.randn(R1, D), dtype=torch.float32)
    W, Wt, E = ops.graft_attention(gg, qh.cuda(), qmask.cuda(), rel.cuda(), out_w=True)
    rW, rWt, rE, Wabs = _fp64_attention(qh, qmask, rel, kfr, facts, B, N)
    n = 3 * Q * D + D + 8
    assert (W.view(B, maxF).cpu().double() - rW).abs().le(n * EPS24 * (Wabs + rW.abs()) + 1e-30).all()
    # W~ = exp(W - max): the error of W enters the exponent
    bound = (n * EPS24 * (Wabs + Wabs.max(1, keepdim=True)[0]) * 2 + 4 * EPS24) * rWt + 1e-38
    assert (Wt.view(B, maxF).cpu().double() - rWt).abs().le(bound).all()
    cnt = np.bincount(facts["b"] * N + facts["head"], minlength=B * N)
    Eb = torch.as_tensor(cnt + 1.0) * (bound.max() + 4 * EPS24) + 1e-30
    assert (E.cpu().double() - rE).abs().le(Eb).all()
    gg.check_status()


def test_attention_max_includes_pad_slots_and_clamps_e():
    rs = np.random.RandomState(5)
    B, N, Q, R1, maxF, D = 2, 9, 4, 6, 20, 16
    gg, kfr, facts = _graph(B, N, maxF, R1, rs, [8, 8])
    qh = torch.tensor(rs.randn(B, Q, D), dtype=torch.float32)
    qmask = torch.ones(B, Q)
    rel = torch.tensor(rs.randn(R1, D), dtype=torch.float32)
    rel[R1 - 1] = 500.0 * qh[0].mean(0) / qh[0].mean(0).norm()         # the pad relation dominates question 0
    _W, Wt, E = ops.graft_attention(gg, qh.cuda(), qmask.cuda(), rel.cuda())
    rW, rWt, rE, _ = _fp64_attention(qh, qmask, rel, kfr, facts, B, N)
    Wt = Wt.view(B, maxF).cpu()
    pad0 = torch.as_tensor(kfr[0] == R1 - 1)
    assert (Wt[0][pad0] == 1.0).all()                                  # the maximum sits on a pad slot
    assert (Wt[0][~pad0] == 0.0).all()                                 # every real fact underflows ...
    E0 = E.view(B, N)[0].cpu()
    assert (E0 == np.float32(1e-10)).all()                             # ... so E clamps on every node of question 0
    assert torch.allclose(E.view(B, N)[1].cpu().double(), rE.view(B, N)[1], rtol=1e-5)


def _fp64_aggregate(gg, Wt, E, prior, self_tab, head_tab, lam, B, N):
    Wt, E, prior = Wt.double().cpu(), E.double().cpu(), prior.double().cpu().view(-1)
    self_tab, head_tab = self_tab.double().cpu(), head_tab.double().cpu()
    n = int(gg.nfacts.item())
    heads = gg.heads[:n].long().cpu(); tails = gg.tails[:n].long().cpu()
    rels = gg.rels[:n].long().cpu(); slot = gg.slot_of[:n].long().cpu()
    s = Wt[slot] * prior[heads] / E[heads]
    x = torch.relu(self_tab[rels] + head_tab[heads])
    v = x * s.unsqueeze(1)
    Nt, D = B * N, self_tab.shape[1]
    sv = torch.zeros(Nt, D, dtype=torch.float64).index_add_(0, tails, v)
    sabs = torch.zeros(Nt, D, dtype=torch.float64).index_add_(0, tails, (self_tab[rels].abs() + head_tab[heads].abs())
                                                               * s.abs().unsqueeze(1))
    ds = torch.zeros(Nt, dtype=torch.float64).index_add_(0, tails, s)
    deg = torch.bincount(tails, minlength=Nt).double()
    dn = lam * ds + (1 - lam) * prior
    return sv, sabs, deg, dn, ds


@pytest.mark.parametrize("D,B,N,hub,zero_prior", [(1, 1, 1, None, False), (7, 2, 13, None, False),
                                                  (50, 3, 40, None, False), (200, 2, 300, 3000, False),
                                                  (256, 2, 30, None, True), (400, 2, 25, None, False),
                                                  (33, 1, 5, None, False)])
def test_aggregate_kernel_matches_fp64(D, B, N, hub, zero_prior):
    rs = np.random.RandomState(D + N)
    R1, maxF = 7, 4000 if hub else 3 * N + 2
    per_q = [3500 if (hub and b == 0) else (0 if b == 1 and B > 2 else rs.randint(1, 3 * N)) for b in range(B)]
    gg, kfr, facts = _graph(B, N, maxF, R1, rs, per_q, hub=hub)
    Nt = B * N
    Wt = torch.tensor(rs.rand(B * maxF), dtype=torch.float32, device=dev)
    Wt[:: 5] = 0.0                                                    # some facts carry no mass at all
    E = torch.tensor(rs.rand(Nt) + 0.1, dtype=torch.float32, device=dev)
    E[::3] = 1e-10                                                     # clamped E
    prior = torch.tensor(rs.rand(B, N) * (rs.rand(B, N) < 0.5), dtype=torch.float32, device=dev)
    if zero_prior:
        prior.zero_()
    self_tab = torch.tensor(rs.randn(R1, D), dtype=torch.float32, device=dev)
    head_tab = torch.tensor(rs.randn(Nt, D), dtype=torch.float32, device=dev)
    q2e = torch.tensor(rs.randn(B, D), dtype=torch.float32, device=dev)
    Dp = (D + 15) // 16 * 16
    hi = torch.zeros(Nt, 5 * Dp, dtype=torch.bfloat16, device=dev)
    lo = torch.zeros_like(hi)
    sum_out = torch.empty(Nt, D, device=dev)
    indeg = torch.empty(Nt, device=dev)
    lam = 0.8
    dn = ops.graft_aggregate(gg, Wt, E, prior, self_tab, head_tab, lam, q2e=q2e, sum_out=sum_out, planes=(hi, lo),
                             col_sum=0, col_indeg=Dp, col_q2e=3 * Dp, indeg_out=indeg)
    sv, sabs, deg, rdn, ds = _fp64_aggregate(gg, Wt, E, prior, self_tab, head_tab, lam, B, N)
    n = deg.unsqueeze(1) + 3
    assert (sum_out.cpu().double() - sv).abs().le(n * 4 * EPS24 * sabs + 1e-30).all()
    assert torch.equal(indeg.cpu().double(), deg)
    planes = hi.float() + lo.float()
    assert torch.equal(planes[:, Dp].cpu().double(), deg)
    assert (planes[:, :D].cpu().double() - sv).abs().le(n * 4 * EPS24 * sabs + 2.0 ** -17 * sv.abs() + 1e-30).all()
    q2e_rows = q2e.repeat_interleave(N, 0).cpu().double()
    assert (planes[:, 3 * Dp:3 * Dp + D].cpu().double() - q2e_rows).abs().le(2.0 ** -17 * q2e_rows.abs()).all()
    assert (planes[:, D:Dp].abs().sum() == 0) and (planes[:, Dp + 1:2 * Dp].abs().sum() == 0)
    pa = prior.view(-1).cpu().double()
    bound = (deg + 4) * 4 * EPS24 * (lam * ds.abs() + (1 - lam) * pa) + 1e-38
    assert (dn.view(-1).cpu().double() - rdn).abs().le(bound).all()
    if zero_prior:
        assert float(sum_out.abs().max()) == 0.0 and float(dn.abs().max()) == 0.0
    gg.check_status()


def test_empty_fact_list_and_tiny_batch():
    t = lambda a: torch.tensor(a, dtype=torch.int64, device=dev)  # noqa: E731
    gg = ops.graft_stage([t([]), t([]), t([])], [t([]), t([]), t([])], t([[3, 3]]), 1, 1, 4)
    qh = torch.randn(1, 2, 8, device=dev)
    _W, Wt, E = ops.graft_attention(gg, qh, torch.ones(1, 2, device=dev), torch.randn(4, 8, device=dev))
    assert float(E.item()) == np.float32(1e-10)
    prior = torch.ones(1, 1, device=dev)
    dn = ops.graft_aggregate(gg, Wt, E, prior, torch.randn(4, 8, device=dev), torch.randn(1, 8, device=dev), 0.8)
    assert float(dn.item()) == np.float32(np.float32(1 - 0.8) * np.float32(1.0))
    gg.check_status()


@pytest.mark.parametrize("bad", ["node", "slot", "batch", "rel", "dup", "unpaired"])
def test_out_of_range_inputs_are_refused(bad):
    t = lambda a: torch.tensor(a, dtype=torch.int64, device=dev)  # noqa: E731
    hb, hf, he = [0, 0, 1], [0, 2, 1], [1, 2, 0]
    tb, te, tf = [0, 0, 1], [2, 0, 1], [0, 2, 1]
    kfr = [[1, 2, 0, 3], [3, 1, 3, 3]]
    if bad == "node":
        he[1] = 7
    elif bad == "slot":
        hf[1] = tf[1] = 9
    elif bad == "batch":
        hb[2] = tb[2] = 5
    elif bad == "rel":
        kfr[0][2] = 11
    elif bad == "dup":
        hf[1] = 0
    else:
        tf[1] = 3
    gg = ops.graft_stage([t(hb), t(hf), t(he)], [t(tb), t(te), t(tf)], t(kfr), 2, 3, 4)
    ops.graft_attention(gg, torch.randn(2, 2, 8, device=dev), torch.ones(2, 2, device=dev),
                        torch.randn(4, 8, device=dev))
    with pytest.raises(RuntimeError, match="graft fact lists rejected"):
        gg.check_status()


def test_model_refuses_out_of_range_batch():
    m, g = load_model("graft_small", "cuda")
    m = m.cuda()
    b = list(g.batch)
    (e2f_b, e2f_f, e2f_e, v0), f2e = b[3]
    e2f_e = e2f_e.copy()
    e2f_e[0] = 10 ** 6
    b[3] = ((e2f_b, e2f_f, e2f_e, v0), f2e)
    with pytest.raises(RuntimeError, match="node id outside the batch"):
        m(tuple(b))


RESULTS = {}


@pytest.mark.parametrize("name", CASES)
def test_forward_matches_reference_golden(name):
    m, g = load_model(name, "cuda")
    m = m.cuda()
    loss, pred, pred_dist, tp = m(g.batch)
    assert tp is None
    want = g.out["pred_dist"]
    got = pred_dist.cpu().numpy()
    rel_err = float(np.abs(got - want).max() / np.abs(want).max())
    RESULTS[name] = rel_err
    print("%s: pred_dist max relative error %.3g" % (name, rel_err))
    assert rel_err < 1e-3
    pr = torch.stack(m.pagerank_history[1:]).cpu().numpy()
    prw = g.out["pagerank_history"]
    assert np.abs(pr - prw).max() <= 1e-3 * np.abs(prw).max()
    hist = torch.stack(m.dist_history[1:]).cpu().numpy()
    assert np.abs(hist - g.out["dist_history"]).max() <= 1e-3 * np.abs(g.out["dist_history"]).max()
    assert abs(float(loss) - float(g.out["loss"])) <= 1e-3 * abs(float(g.out["loss"]))
    peaked = want.max(1) > 2 * np.sort(want, 1)[:, -2]
    assert np.array_equal(pred.cpu().numpy()[peaked], g.out["pred"][peaked])


@pytest.mark.parametrize("name", ["graft_d50_sharp", "graft_hub_clamp"])
def test_evaluator_lists_equal_reference(name):
    m, g = load_model(name, "cuda")
    m = m.cuda()
    _l, _p, pred_dist, _ = m(g.batch)
    retrieved, _ = evaluate.retrieve(pred_dist, m.last_batch, NUM_ENTITY, g.args["eps"])
    ids = [r.ent.tolist() for r in retrieved]
    peaked = [b for b in range(len(ids)) if g.out["pred_dist"][b].max() > 0.5]     # near-uniform rows hold near-ties
    assert len(peaked) >= 1
    assert [ids[b] for b in peaked] == [g.cand_lists()[b] for b in peaked]


def test_twins_tie_exactly():
    m, g = load_model("graft_d50_sharp", "cuda")
    m = m.cuda()
    _l, _p, pred_dist, _ = m(g.batch)
    pd = pred_dist.cpu()
    assert torch.equal(pd[:, 4], pd[:, 5])
    for h in m.pagerank_history[1:]:
        assert torch.equal(h[:, 4], h[:, 5])


@pytest.mark.parametrize("name", ["graft_small", "graft_dropout_padmax", "graft_hub_clamp"])
def test_bit_identical_runs_and_permutation_invariance(name):
    m, g = load_model(name, "cuda")
    m = m.cuda()
    a = m(g.batch)[2].clone()
    b = m(g.batch)[2].clone()
    assert torch.equal(a, b)
    (hb, hf, he, v0), (tb, te, tf, v1) = g.batch[3]
    rs = np.random.RandomState(0)
    p, q = rs.permutation(len(hb)), rs.permutation(len(tb))
    batch = list(g.batch)
    batch[3] = ((hb[p], hf[p], he[p], v0), (tb[q], te[q], tf[q], v1))
    c = m(tuple(batch))[2]
    assert torch.equal(a, c)


def test_staged_facts_are_in_slot_order():
    g = GraftGolden("graft_inverse")
    db = batching.stage_graft_batch(g.batch, dev, 41)
    n = int(db.graft.nfacts.item())
    slots = db.graft.slot_of[:n].cpu().numpy()
    assert n == len(g.batch[3][0][0]) and (np.diff(slots) > 0).all()
    gr = db.graft.graph
    rp, fact = gr.rowptr_t.cpu().numpy(), gr.fact_t.cpu().numpy()
    for r in range(db.B * db.N):
        assert (np.diff(slots[fact[rp[r]:rp[r + 1]]]) > 0).all()


@pytest.mark.parametrize("name", TRAIN_CASES)
def test_training_on_gpu_matches_reference_gradients(name):
    assert not autograd_path.HOST_CHECK
    m, g = load_model(name, "cuda")
    m = m.cuda()
    m.train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.eval()
    if hasattr(m.instruction, "node_encoder") and not isinstance(m.instruction.node_encoder, torch.nn.LSTM):
        m.instruction.node_encoder.eval()
    batch = list(g.batch)
    batch[8] = g.train["answer_dist"]
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        loss, pred, pred_dist, tp_list = m(tuple(batch), training=True)
        assert abs(float(loss.detach()) - float(g.train["loss"])) <= 2e-5 * abs(float(g.train["loss"]))
        assert tp_list[0] == g.train["h1"].tolist()
        loss.backward()
    gmax = max(float(np.abs(v).max()) for v in g.grads.values())
    checked = 0
    for k, p in m.named_parameters():
        if k not in g.grads:
            continue
        want = g.grads[k]
        got = p.grad.cpu().numpy() if p.grad is not None else np.zeros_like(want)
        assert np.abs(got - want).max() <= 5e-3 * np.abs(want).max() + 1e-5 * gmax + 1e-7, k
        checked += 1
    assert checked >= 15
