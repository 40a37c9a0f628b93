"""Plain float64 restatements of the question-side and scoring kernels (csrc/question.cu, csrc/score.cu).

These are the references ``tests/test_question_side_gpu.py`` holds the kernels to.  Each one follows the math of the
reference model as written -- lstm_encoder.py:27-36 (nn.LSTM), base_encoder.py:73-114 (get_instruction),
query_update.py:6-44 (QueryReform / Fusion), reasongnn.py:165-169 (score + masked softmax) and
base_model.py:186-215 / rearev.py:156-160,228-232 (kl loss, case_valid, argmax) -- with none of the shortcuts the
kernels take: no seed compaction, no column slices, no online maximum, every sum a dense float64 reduction.  Like
``fp64_ref`` they do not import ``gnn_rag_b200``; ``tests/test_question_side_host.py`` checks them against the torch
modules and the oracle in float64 first.

Inputs may be fp32 or fp64 tensors; everything is computed in float64 on the device of the inputs.

Masked logits.  The model adds (1 - mask) * VERY_NEG_NUMBER in fp32, where the sum rounds every |logit| < 4096 (half
an fp32 ulp of 1e11) to VERY_NEG_NUMBER itself: an all-pad question gets exactly uniform attention / distribution.
A float64 sum would keep the logit and make that row non-uniform, which the reference never is, so a masked logit is
exactly ``VERY_NEG`` (the fp32 value of -1e11) here; callers keep live logits below 4096 in magnitude.
"""
import torch

F64 = torch.float64
VERY_NEG = float(torch.tensor(-100000000000.0, dtype=torch.float32))   # VERY_NEG_NUMBER in fp32: -99999997952


def _d(t):
    return None if t is None else torch.as_tensor(t).to(F64)


def _masked(logits, mask):
    return torch.where(mask > 0, logits, torch.full_like(logits, VERY_NEG))


def lstm(gates_x, W_hh, b_hh=None):
    """One-layer LSTM, zero initial state, gate order (i, f, g, o) as in torch.  gates_x [B, Q, 4D] is the input
    projection x W_ih^T + b_ih; W_hh [4D, D]; b_hh [4D] or None.  Returns every token's hidden state [B, Q, D]."""
    gx, W = _d(gates_x), _d(W_hh)
    B, Q, G = gx.shape
    D = G // 4
    b = torch.zeros(G, dtype=F64, device=gx.device) if b_hh is None else _d(b_hh)
    h = torch.zeros(B, D, dtype=F64, device=gx.device)
    c = torch.zeros_like(h)
    out = []
    for t in range(Q):
        a = gx[:, t] + h @ W.t() + b
        i, f, g, o = a[:, :D], a[:, D:2 * D], a[:, 2 * D:3 * D], a[:, 3 * D:]
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        out.append(h)
    return torch.stack(out, 1)


def instructions(hidden, qnode, qtext, pad, Wq, bq, Wcq, bcq, wca, bca, ri0=None):
    """``get_instruction`` applied len(Wq) times from relational_ins = ri0, zero by default (base_encoder.py:73-114).
    hidden [B, Q, D] token states, qnode [B, D] last state, qtext [B, Q] token ids; Wq / bq: the question_linear_i
    weights and biases; Wcq [D, 4D], bcq [D]; wca [D] (ca_linear.weight flattened), bca [1].
    Returns (instructions [B, I, D], attention [B, I, Q])."""
    hid, qn = _d(hidden), _d(qnode)
    B, Q, D = hid.shape
    mask = (torch.as_tensor(qtext) != pad).to(F64)
    Wcq, bcq, wca, bca = _d(Wcq), _d(bcq), _d(wca).reshape(-1), _d(bca).reshape(-1)
    ri = torch.zeros(B, D, dtype=F64, device=hid.device) if ri0 is None else _d(ri0)
    outs, attns = [], []
    for W, b in zip(Wq, bq):
        qi = qn @ _d(W).t() + _d(b)
        cq = torch.cat([ri, qi, qi - ri, qi * ri], 1) @ Wcq.t() + bcq
        ca = (cq.unsqueeze(1) * hid) @ wca + bca
        attn = torch.softmax(_masked(ca, mask), 1)
        ri = (attn.unsqueeze(2) * hid).sum(1)
        outs.append(ri)
        attns.append(attn)
    return torch.stack(outs, 1), torch.stack(attns, 1)


def seed_retrieve(seed, h, B, N):
    """bmm(seed.unsqueeze(1), h.view(B, N, D)): the seed-weighted row sum (query_update.py:40).  seed [B, N],
    h [B*N, D] (any row stride).  Returns [B, D]."""
    s, x = _d(seed), _d(h)
    return torch.bmm(s.view(B, 1, N), x.reshape(B, N, -1)).squeeze(1)


def fusion(x, y, Wr, Wg):
    """Fusion.forward (query_update.py:6-16): z = [x, y, x - y]; g = sigmoid(Wg z); g * (Wr z) + (1 - g) * x.
    Returns (out, r = Wr z, g)."""
    x, y = _d(x), _d(y)
    z = torch.cat([x, y, x - y], -1)
    r = z @ _d(Wr).t()
    g = torch.sigmoid(z @ _d(Wg).t())
    return g * r + (1 - g) * x, r, g


def query_reform(seed, h, ins, Wr, Wg, B, N):
    """QueryReform.forward for every instruction j: Fusion_j(ins[:, j], seed_retrieve).  ins [B, I, D];
    Wr / Wg: lists of the fusion.r / fusion.g weights [D, 3D].  Returns (new instructions [B, I, D], seed_retrieve
    [B, D])."""
    y = seed_retrieve(seed, h, B, N)
    x = _d(ins)
    out = [fusion(x[:, j], y, Wr[j], Wg[j])[0] for j in range(x.shape[1])]
    return torch.stack(out, 1), y


def score_softmax(h, w, b, mask, B, N):
    """logits = h w + b (VERY_NEG where masked) and softmax over each question's N nodes (reasongnn.py:165-169).
    h [B*N, D] (any row stride), w [D], b [1] or None, mask [B*N].  Returns (dist [B, N], logits [B, N])."""
    x = _d(h) @ _d(w).reshape(-1)
    if b is not None:
        x = x + _d(b).reshape(-1)
    logits = _masked(x, _d(mask).reshape(-1)).view(B, N)
    return torch.softmax(logits, 1), logits


def kl_loss_pred(dist, teacher):
    """calc_loss_label with loss_type 'kl' (base_model.py:193-215, rearev.py:228-232) and the argmax.
    Per question: len = sum t; case_valid = len > 0; a zero len becomes 1; loss_q = case_valid * sum_n
    [xlogy(t/len, t/len) - t/len * log(p + 1e-8)].  loss = sum_b loss_q / B.  pred = the lowest index of each row's
    maximum.  Returns (loss, loss_q [B], case_valid [B], pred int64 [B])."""
    p, t = _d(dist), _d(teacher)
    length = t.sum(1, keepdim=True)
    valid = (length > 0).to(F64)
    length = torch.where(length == 0, torch.ones_like(length), length)
    tv = t / length
    term = torch.xlogy(tv, tv) - tv * torch.log(p + 1e-8)
    loss_q = (term * valid).sum(1)
    mx = p.max(1, keepdim=True)[0]
    n = torch.arange(p.shape[1], device=p.device).expand_as(p)
    pred = torch.where(p == mx, n, torch.full_like(n, p.shape[1])).min(1)[0]
    return loss_q.sum() / p.shape[0], loss_q, valid.view(-1), pred
