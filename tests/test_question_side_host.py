"""CPU: the float64 restatements of tests/question_ref.py against the reference's own operations run in float64 --
torch's nn.LSTM, ``modules.LSTMInstruction.get_instruction``, ``modules.Fusion`` and the oracle's
``LstmQuestion.get_instruction``, ``query_reform`` and ``kl_loss`` (oracle/kgqa_oracle.py).  Both sides are float64
and compute the same expressions in a different order, so they agree to a few float64 ulps of each element's scale;
1e-12 relative to the scale leaves room for that and for nothing else."""
import numpy as np
import pytest
import torch

from gnn_rag_b200.modules import Fusion, LSTMInstruction
from oracle import kgqa_oracle as O

import question_ref as R

F64 = torch.float64
TOL = 1e-12


def _close(got, want):
    got, want = got.to(F64), want.to(F64)
    scale = want.abs().max().item() + 1e-300
    assert got.shape == want.shape
    assert ((got - want).abs().max().item()) <= TOL * scale


@pytest.mark.parametrize("B,Q,D,W,bias", [(3, 5, 7, 4, True), (2, 1, 1, 3, True), (4, 9, 16, 6, False)])
def test_lstm_matches_torch_lstm(B, Q, D, W, bias):
    torch.manual_seed(B * Q + D)
    lstm = torch.nn.LSTM(W, D, batch_first=True, bias=bias).double()
    x = torch.randn(B, Q, W, dtype=F64)
    with torch.no_grad():
        want, (hn, _) = lstm(x)
        gx = x @ lstm.weight_ih_l0.t()
        if bias:
            gx = gx + lstm.bias_ih_l0
        got = R.lstm(gx, lstm.weight_hh_l0, lstm.bias_hh_l0 if bias else None)
    _close(got, want)
    _close(got[:, -1], hn[0])


def _instruction_inputs(B, Q, D, I, seed):
    rs = np.random.RandomState(seed)
    f = lambda *s: torch.from_numpy(rs.randn(*s)).to(F64)          # noqa: E731
    pad = 50
    text = torch.from_numpy(rs.randint(0, pad, size=(B, Q)))
    text[0, Q // 2] = pad                                            # a pad token inside the question
    text[0, -1] = pad
    text[B - 1] = pad                                                # an all-pad question
    return f(B, Q, D), f(B, D), text, pad


@pytest.mark.parametrize("B,Q,D,I", [(3, 6, 5, 3), (2, 1, 4, 1), (3, 4, 8, 8)])
def test_instructions_match_lstm_instruction_module(B, Q, D, I):
    hid, qn, text, pad = _instruction_inputs(B, Q, D, I, D + I)
    torch.manual_seed(I)
    emb = torch.nn.Embedding(pad + 1, 3, padding_idx=pad)
    mod = LSTMInstruction(dict(num_ins=I, entity_dim=D, word_dim=3), emb, pad).double().eval()
    mod.query_hidden_emb, mod.query_node_emb, mod._query_text = hid, qn.unsqueeze(1), text
    lins = [getattr(mod, "question_linear%d" % i) for i in range(I)]
    args = ([l.weight for l in lins], [l.bias for l in lins], mod.cq_linear.weight, mod.cq_linear.bias,
            mod.ca_linear.weight, mod.ca_linear.bias)
    with torch.no_grad():
        got, attn = R.instructions(hid, qn, text, pad, *args)
        ri = torch.zeros(B, D, dtype=F64)
        for i in range(I):
            ri, a = mod.get_instruction(ri, step=i)
            _close(got[:B - 1, i], ri[:B - 1])
            _close(attn[:B - 1, i], a[:B - 1].squeeze(2))
        # the all-pad question: float64 keeps the ca differences under VERY_NEG, the reference's fp32 does not --
        # against the module run in fp32, the attention is exactly uniform
        mod.float()
        mod.query_hidden_emb, mod.query_node_emb = hid.float(), qn.unsqueeze(1).float()
        ri = torch.zeros(B, D)
        for i in range(I):
            ri, a = mod.get_instruction(ri, step=i)
            assert torch.equal(a[B - 1].squeeze(1), torch.full((Q,), 1.0 / Q))
    assert torch.equal(attn[B - 1], torch.full((I, Q), 1.0 / Q, dtype=F64))
    _close(got[B - 1], hid[B - 1].mean(0).expand(I, D))


def test_instructions_match_oracle_get_instruction():
    B, Q, D, I = 3, 7, 6, 4
    hid, qn, text, pad = _instruction_inputs(B, Q, D, I, 9)
    rs = np.random.RandomState(10)
    f = lambda *s: torch.from_numpy(rs.randn(*s)).to(F64)          # noqa: E731
    p = "instruction."
    sd = {p + "cq_linear.weight": f(D, 4 * D), p + "cq_linear.bias": f(D), p + "ca_linear.weight": f(1, D),
          p + "ca_linear.bias": f(1)}
    for i in range(I):
        sd[p + "question_linear%d.weight" % i], sd[p + "question_linear%d.bias" % i] = f(D, D), f(D)
    q = O.LstmQuestion.__new__(O.LstmQuestion)                       # the encoder's outputs, set in float64
    q.sd, q.D = sd, D
    q.query_hidden_emb, q.query_node_emb, q.query_mask = hid, qn.unsqueeze(1), (text != pad).to(F64)
    ri = torch.zeros(B, D, dtype=F64)
    want = []
    for i in range(I):
        ri = q.get_instruction(ri, i)
        want.append(ri)
    got, _ = R.instructions(hid, qn, text, pad, [sd[p + "question_linear%d.weight" % i] for i in range(I)],
                            [sd[p + "question_linear%d.bias" % i] for i in range(I)], sd[p + "cq_linear.weight"],
                            sd[p + "cq_linear.bias"], sd[p + "ca_linear.weight"], sd[p + "ca_linear.bias"])
    _close(got[:B - 1], torch.stack(want, 1)[:B - 1])        # the all-pad question: see the test above


@pytest.mark.parametrize("I", [1, 3])
def test_query_reform_matches_oracle_and_fusion(I):
    B, N, D = 3, 11, 5
    rs = np.random.RandomState(I)
    f = lambda *s: torch.from_numpy(rs.randn(*s)).to(F64)          # noqa: E731
    h = f(B * N, D)
    seed = torch.zeros(B, N, dtype=F64)
    seed[0, 0] = 1.0
    seed[1, [2, 5, 10]] = torch.tensor([0.2, 0.3, 0.5], dtype=F64)    # question 2: no seed
    ins = f(B, I, D)
    sd = {}
    for j in range(I):
        sd["reform%d.fusion.r.weight" % j], sd["reform%d.fusion.g.weight" % j] = f(D, 3 * D), f(D, 3 * D)
    Wr = [sd["reform%d.fusion.r.weight" % j] for j in range(I)]
    Wg = [sd["reform%d.fusion.g.weight" % j] for j in range(I)]
    got, y = R.query_reform(seed, h, ins, Wr, Wg, B, N)
    _close(y, torch.stack([(seed[b].view(N, 1) * h.view(B, N, D)[b]).sum(0) for b in range(B)]))
    assert (y[2] == 0).all()
    for j in range(I):
        _close(got[:, j], O.query_reform(sd, "reform%d." % j, ins[:, j], h.view(B, N, D), seed))
        fu = Fusion(D).double()
        with torch.no_grad():
            fu.r.weight.copy_(Wr[j])
            fu.g.weight.copy_(Wg[j])
            _close(got[:, j], fu(ins[:, j], y))


def test_score_softmax_matches_torch_chain():
    B, N, D = 3, 9, 4
    rs = np.random.RandomState(4)
    h = torch.from_numpy(rs.randn(B * N, D + 3))[:, :D]
    w, b = torch.from_numpy(rs.randn(D)), torch.from_numpy(rs.randn(1))
    mask = torch.from_numpy((rs.rand(B * N) > 0.3).astype(np.float64))
    mask[N:2 * N] = 0.0                                              # an all-pad question
    dist, logits = R.score_softmax(h, w, b, mask, B, N)
    want_l = (h @ w + b).view(B, N) + (1 - mask.view(B, N)) * O.VERY_NEG_NUMBER
    live = mask.view(B, N) > 0
    _close(logits[live], want_l[live])
    assert (logits[~live] == R.VERY_NEG).all()
    rows = [0, 2]
    _close(dist[rows], torch.softmax(want_l[rows], 1))
    assert (dist[rows][~live[rows]] == 0).all()
    # the all-pad question is uniform, as in the reference's fp32 chain
    want32 = torch.softmax((h.float() @ w.float() + b.float()).view(B, N) + (1 - mask.float().view(B, N))
                           * O.VERY_NEG_NUMBER, 1)
    assert torch.equal(want32[1], torch.full((N,), 1.0 / N))
    assert torch.equal(dist[1], torch.full((N,), 1.0 / N, dtype=F64))
    _, l0 = R.score_softmax(h, w, None, mask, B, N)
    _close(l0[live], (want_l - b)[live])


def test_kl_loss_pred_matches_oracle_kl_loss_and_lowest_index_argmax():
    B, N = 5, 40
    rs = np.random.RandomState(5)
    dist = torch.softmax(torch.from_numpy(rs.randn(B, N)), 1)
    dist[0, 3] = dist[0, 30] = dist[0].max() + 0.1                   # tie: lowest index wins
    dist[2, 0] = dist[2, N - 1] = dist[2].max() + 0.1
    dist[4, 7] = 0.0
    t = torch.zeros(B, N, dtype=F64)
    t[0, [3, 4]] = 1.0
    t[1, :] = torch.from_numpy(rs.rand(N))                            # fractional teacher weights
    t[4, 7] = 0.5                                                     # dist = 0 under a positive teacher
    # question 2 and 3: no answer -> case_valid 0, loss_q exactly 0
    loss, loss_q, valid, pred = R.kl_loss_pred(dist, t)
    _close(loss, O.kl_loss(dist, t))
    assert valid.tolist() == [1.0, 1.0, 0.0, 0.0, 1.0]
    assert loss_q[2].item() == 0.0 and loss_q[3].item() == 0.0
    tn = t / t.sum(1, keepdim=True).clamp_min(1e-300)
    for b in (0, 1, 4):
        _close(loss_q[b], torch.nn.functional.kl_div(torch.log(dist[b] + 1e-8), tn[b], reduction="sum"))
    assert pred.tolist() == [3, int(np.argmax(dist[1].numpy())), 0, int(np.argmax(dist[3].numpy())),
                             int(np.argmax(dist[4].numpy()))]
