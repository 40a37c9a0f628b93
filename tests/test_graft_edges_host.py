"""The float64 restatement of the GraftNet kernels (tests/graft_edges_ref.py) pinned on the CPU: against the torch-CPU
oracle and the reference's own outputs on the shipped graft goldens, and its closed-form gradients against float64
autograd of its forward statements."""
import numpy as np
import pytest
import torch

import graft_edges_ref as R
from graft_train_ref import graftnet_fp64
from test_graftnet_host import CASES, NUM_ENTITY, load_model

F64 = torch.float64


def _close(got, want, rtol, what):
    got, want = torch.as_tensor(np.asarray(got)).double(), torch.as_tensor(np.asarray(want)).double()
    err = (got - want).abs()
    bound = rtol * want.abs() + rtol * 1e-3 * want.abs().max() + 1e-30
    assert bool((err <= bound).all()), (what, float((err - bound).max()))


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_the_oracle_on_the_goldens(name):
    """The model's forward built from the restatement (staging, attention, W~, E and the per-layer aggregate with
    kb_tail_linear moved after the per-node sum) gives the oracle's PageRank history and prediction, and the
    reference's own W~ and E."""
    from oracle import graft_oracle
    m, g = load_model(name)
    with torch.no_grad():
        out = graft_oracle.forward(m, g.batch)
        logit, pr = graftnet_fp64(m, g.batch)
        mask = torch.as_tensor(g.batch[0] != NUM_ENTITY).double()
        pred = torch.softmax(logit + (1 - mask) * R.VERY_NEG, dim=1)
        _close(pred, out["pred_dist"], 1e-4, "pred_dist")
        _close(pr, out["pagerank_history"], 1e-4, "pagerank_history")
        # the attention alone, against the reference's first-layer W~ and E
        enc = m.instruction
        enc.encode_question_train(torch.as_tensor(g.batch[4]))
        B, N = g.batch[0].shape
        kfr = g.batch[5]
        at = R.attention(enc.query_hidden_emb, enc.query_mask_train, m.get_rel_feature_train(), kfr)
        Wt = R.w_tilde(at["W"])
        st = R.stage(g.batch[3][0][:3], g.batch[3][1][:3], kfr, N)
        E = R.e_sum(Wt, st, B * N)[0]
    _close(Wt, g.out["w_tilde"], 1e-4, "w_tilde")
    _close(E.view(B, N), g.out["e2f_softmax"], 1e-4, "E")


def test_stage_pairs_permuted_lists_in_slot_order():
    rs = np.random.RandomState(0)
    B, N, M = 3, 7, 11
    slots = [rs.permutation(M)[:n] for n in (5, 0, 9)]
    kfr = rs.randint(0, 4, size=(B, M))
    hb = np.concatenate([np.full(len(s), b) for b, s in enumerate(slots)])
    hf = np.concatenate(slots)
    he, te = rs.randint(0, N, len(hf)), rs.randint(0, N, len(hf))
    p = rs.permutation(len(hf))
    st = R.stage((hb, hf, he), (hb[p], te[p], hf[p]), kfr, N)
    order = np.argsort(hb * M + hf)
    assert st["slot_of"].tolist() == (hb * M + hf)[order].tolist()
    assert st["heads"].tolist() == (hb * N + he)[order].tolist()
    assert st["tails"].tolist() == (hb * N + te)[order].tolist()
    assert st["rels"].tolist() == kfr.reshape(-1)[(hb * M + hf)[order]].tolist()


def test_fully_masked_question_shares_its_softmax_evenly():
    rs = np.random.RandomState(1)
    B, Q, D, R1, M = 2, 5, 8, 4, 6
    qh = torch.tensor(rs.randn(B, Q, D))
    qmask = torch.tensor([[1, 0, 1, 1, 0], [0, 0, 0, 0, 0]], dtype=F64)
    at = R.attention(qh, qmask, torch.tensor(rs.randn(R1, D)), rs.randint(0, R1, (B, M)))
    assert torch.equal(at["a"][1], torch.full((Q, M), 1.0 / Q, dtype=F64))
    assert float(at["a"][0][[1, 4]].abs().max()) == 0.0
    torch.testing.assert_close(at["W"][1], at["z"][1].mean(0), rtol=1e-14, atol=0)


def _graph(rs, B, N, M, R1, per_q):
    kfr = np.full((B, M), R1 - 1, dtype=np.int64)
    hb, hf, he, te = [], [], [], []
    for b, n in enumerate(per_q):
        s = rs.permutation(M)[:n]
        kfr[b, s] = rs.randint(0, R1 - 1, n)
        hb += [b] * n; hf += list(s); he += list(rs.randint(0, N, n)); te += list(rs.randint(0, N, n))
    hb, hf = np.array(hb), np.array(hf)
    return kfr, R.stage((hb, hf, np.array(he)), (hb, np.array(te), hf), kfr, N)


@pytest.mark.parametrize("Q", [1, 4])
def test_attention_backward_equals_autograd(Q):
    """Closed-form grad_qh and grad_rel against float64 autograd of sum(W * gW), pads and a fully masked question
    included."""
    rs = np.random.RandomState(Q)
    B, D, R1, M = 3, 6, 5, 9
    qh = torch.tensor(rs.randn(B, Q, D), requires_grad=True)
    rel = torch.tensor(rs.randn(R1, D), requires_grad=True)
    qmask = torch.tensor((rs.rand(B, Q) < 0.6).astype(np.float64))
    qmask[0, 0], qmask[2] = 1, 0
    kfr = rs.randint(0, R1, (B, M))
    gW = torch.tensor(rs.randn(B, M))
    gW[1, ::2] = 0
    (R.attention(qh, qmask, rel, kfr)["W"] * gW).sum().backward()
    got = R.attention_backward(qh.detach(), qmask, rel.detach(), kfr, gW)
    torch.testing.assert_close(got["grad_qh"][0], qh.grad, rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(got["grad_rel"][0], rel.grad, rtol=1e-12, atol=1e-14)
    for k in ("grad_qh", "grad_rel"):
        v, scale, n = got[k]
        assert bool((scale >= v.abs()).all()) and bool((n > 0).all())


@pytest.mark.parametrize("p", [0.0, 0.3])
def test_train_aggregate_backward_equals_autograd(p):
    rs = np.random.RandomState(int(p * 10))
    B, N, M, R1, D = 2, 9, 40, 6, 7
    kfr, st = _graph(rs, B, N, M, R1, [35, 12])
    F_, Nt = len(st["heads"]), B * N
    self_tab = torch.tensor(rs.randn(R1, D), requires_grad=True)
    head_tab = torch.tensor(rs.randn(Nt, D))
    h0, r0 = int(st["heads"][0]), int(st["rels"][0])
    head_tab[h0, :3] = -self_tab.detach()[r0, :3]                       # relu'(0) = 0
    head_tab.requires_grad_(True)
    s = torch.tensor(rs.rand(F_))
    s[::4] = 0
    s.requires_grad_(True)
    mask = torch.tensor((rs.rand(B * M, D) >= p).astype(np.uint8)) if p > 0 else None
    G = torch.tensor(rs.randn(Nt, D))
    out = R.train_aggregate(self_tab, head_tab, s, st, Nt, mask, p)
    (out * G).sum().backward()
    got = R.train_aggregate_backward(self_tab.detach(), head_tab.detach(), s.detach(), G, st, Nt, mask, p)
    for k, ref in (("grad_s", s.grad), ("grad_self", self_tab.grad), ("grad_head", head_tab.grad)):
        torch.testing.assert_close(got[k][0], ref, rtol=1e-12, atol=1e-14)
        assert bool((got[k][1] >= got[k][0].abs() - 1e-12).all())
    scale, n = R.train_aggregate_scale(self_tab.detach(), head_tab.detach(), s.detach(), st, Nt, mask, p)
    assert bool((scale >= out.detach().abs() - 1e-12).all())
    assert n[:, 0].tolist() == (torch.bincount(st["tails"], minlength=Nt) + 4).double().tolist()


def test_type_layer_backward_equals_autograd():
    rs = np.random.RandomState(3)
    Nt, R1, D, F_ = 20, 6, 5, 70
    heads, tails = torch.tensor(rs.randint(0, Nt, F_)), torch.tensor(rs.randint(0, Nt, F_))
    rels = torch.tensor(rs.randint(0, R1, F_))
    w = torch.tensor(rs.uniform(0.1, 2.0, F_))
    table = torch.tensor(rs.randn(R1, D), requires_grad=True)
    fv = table[rels] * w.unsqueeze(1)
    out = torch.relu(torch.zeros(Nt, D, dtype=F64).index_add(0, tails, fv).index_add(0, heads, fv))
    G = torch.tensor(rs.randn(Nt, D))
    (out * G).sum().backward()
    v, scale, n = R.type_layer_backward(G, out.detach(), heads, rels, tails, R1, w)
    torch.testing.assert_close(v, table.grad, rtol=1e-12, atol=1e-14)
    assert bool((scale >= v.abs()).all())


def test_inference_aggregate_restates_its_terms():
    """sum_out, in-degree and prior_next of the restatement against a per-fact loop."""
    rs = np.random.RandomState(4)
    B, N, M, R1, D, lam = 2, 6, 20, 5, 3, 0.8
    kfr, st = _graph(rs, B, N, M, R1, [18, 7])
    Nt = B * N
    Wt, E, prior = torch.tensor(rs.rand(B * M)), torch.tensor(rs.rand(Nt) + 0.1), torch.tensor(rs.rand(Nt))
    self_tab, head_tab = torch.tensor(rs.randn(R1, D)), torch.tensor(rs.randn(Nt, D))
    ag = R.aggregate(Wt, E, prior, self_tab, head_tab, st, lam, Nt)
    so, ds, deg = np.zeros((Nt, D)), np.zeros(Nt), np.zeros(Nt)
    for h, t, r, sl in zip(*(st[k].tolist() for k in ("heads", "tails", "rels", "slot_of"))):
        s = float(Wt[sl]) * float(prior[h]) / float(E[h])
        so[t] += np.maximum(self_tab[r].numpy() + head_tab[h].numpy(), 0) * s
        ds[t] += s
        deg[t] += 1
    np.testing.assert_allclose(ag["sum_out"].numpy(), so, rtol=1e-12, atol=1e-15)
    np.testing.assert_array_equal(ag["indeg"].numpy(), deg)
    np.testing.assert_allclose(ag["prior_next"].numpy(), lam * ds + (1 - lam) * prior.numpy(), rtol=1e-12)
    Et, raw, cnt = R.e_sum(Wt, st, Nt)
    assert float(Et.min()) >= R.VERY_SMALL and cnt.sum() == len(st["heads"])
