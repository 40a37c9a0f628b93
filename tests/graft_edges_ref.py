"""float64 restatement of the GraftNet kernels' contracts (csrc/graft.cu, and the TypeLayer backward GraftNet trains),
with the |.|-scale and the term count of every output element, for per-element bounds n * 2^-24 * scale.

torch on the CPU in float64.  It does not import gnn_rag_b200: it states the operations apart from the code it checks.
Staged facts ``st`` are a dict of int64 tensors in slot order: heads and tails (global rows b * N + node), rels, and
slot_of (b * max_fact + f)."""
import numpy as np
import torch

VERY_NEG = -1e11          # VERY_NEG_NUMBER of the reference
VERY_SMALL = 1e-10        # VERY_SMALL_NUMBER: the clamp of E
F64 = torch.float64


def _i64(x):
    return torch.as_tensor(np.asarray(x), dtype=torch.int64)


def _rows(idx, v, n):
    """index_add of v's rows (or values) into n zero rows."""
    return torch.zeros((n,) + tuple(v.shape[1:]), dtype=F64).index_add(0, idx, v.double())


def stage(e2f, f2e, kfr, N):
    """The graft lists e2f = (b, f, head) and f2e = (b, tail, f) paired by slot and put in slot order -> staged facts.
    Every slot must be listed once in each list (the staging kernel reports anything else)."""
    kfr = _i64(kfr)
    M = kfr.shape[1]
    hb, hf, he = (_i64(x) for x in e2f)
    tb, te, tf = (_i64(x) for x in f2e)
    hs, ts = hb * M + hf, tb * M + tf
    ho, to = torch.argsort(hs), torch.argsort(ts)
    assert torch.equal(hs[ho], ts[to]), "head and tail lists do not pair"
    slot = hs[ho]
    return dict(heads=(hb * N + he)[ho], tails=(tb * N + te)[to], rels=kfr.reshape(-1)[slot], slot_of=slot)


# ---- attention ------------------------------------------------------------------------------------------------------

def attention(qh, qmask, rel, kfr):
    """compute_attention for every slot (pads included) -> dict W [B, M], a [B, Q, M] (softmax over the question's
    tokens), z [B, Q, M] = <qh_q, rel_r> / sqrt(D), fe [B, M, D] (the slot's relation row) and Wabs [B, M], the
    |.|-scale of W (sum_q a_q |qh_q| . |rel_r| / sqrt(D)).

    The mask offset is added in fp32, as the reference adds it: a masked token's logit is the fp32 value of
    z - 1e11, which is -1e11 itself for |z| < 4096.  So a question whose every token is masked shares its softmax
    evenly, a_q = 1 / Q.  The cast keeps the gradient (autograd differentiates the softmax at those values, as the
    reference's backward does).  Relation ids must lie in [0, R1)."""
    qh, rel, qmask = qh.double(), rel.double(), qmask.double()
    D = rel.shape[1]
    fe = rel[_i64(kfr)]
    div = np.sqrt(D)
    z = torch.bmm(qh, fe.transpose(1, 2)) / div
    off = ((1 - qmask) * VERY_NEG).unsqueeze(2)
    sim = z + off
    fp32 = (sim.float().double() - z).detach()                # the offset as the fp32 sum applies it
    sim = torch.where((off != 0).expand_as(sim), z + fp32, sim)
    a = torch.softmax(sim, 1)
    W = (torch.bmm(a.transpose(1, 2), qh) * fe).sum(2) / div
    Wabs = (torch.bmm(a.transpose(1, 2), qh.abs()) * fe.abs()).sum(2) / div
    return dict(W=W, a=a, z=z, fe=fe, Wabs=Wabs)


def w_tilde(W):
    """W~ = exp(W - max over every slot of the question, pads included)."""
    return torch.exp(W - W.max(1, keepdim=True)[0])


def w_tilde_bound(W, Wabs, Q, D):
    """Per-slot bound on |W~ - fp64| for W computed with n = 3QD + D + 8 roundings relative to its |.|-scale: the
    error of W and of the question's maximum enters the exponent, plus the exp and the subtraction."""
    n = 3 * Q * D + D + 8
    eW = n * 2.0 ** -24 * (Wabs + W.abs())
    return ((eW + eW.max(1, keepdim=True)[0]) * 2 + 4 * 2.0 ** -24) * w_tilde(W) + 1e-38


def e_sum(Wt, st, Nt):
    """E [Nt] = max(sum over the node's staged out-facts (head CSR) of W~[slot], 1e-10), the unclamped sum (its terms
    are >= 0, so it is its own |.|-scale) and the term count per node."""
    v = Wt.double().reshape(-1)[st["slot_of"]]
    s = _rows(st["heads"], v, Nt)
    return s.clamp(min=VERY_SMALL), s, torch.bincount(st["heads"], minlength=Nt).double()


# ---- inference aggregate --------------------------------------------------------------------------------------------

def aggregate(Wt, E, prior, self_tab, head_tab, st, lam, Nt):
    """One layer's fact side (gr_graft_aggregate): s_f = W~[slot] * prior[head] / E[head] and, per tail row,
    sum_out = sum_f relu(self_tab[r_f] + head_tab[head_f]) * s_f, the in-degree, and
    prior_next = lam * sum_f s_f + (1 - lam) * prior.  Returns a dict with those, ``sabs`` (|.|-scale of sum_out) and
    ``pn_scale`` (of prior_next)."""
    Wt, E, prior = Wt.double().reshape(-1), E.double().reshape(-1), prior.double().reshape(-1)
    self_tab, head_tab = self_tab.double(), head_tab.double()
    h, t, r = st["heads"], st["tails"], st["rels"]
    s = Wt[st["slot_of"]] * prior[h] / E[h]
    x = torch.relu(self_tab[r] + head_tab[h])
    ds = _rows(t, s, Nt)
    return dict(s=s, sum_out=_rows(t, x * s.unsqueeze(1), Nt),
                sabs=_rows(t, (self_tab[r].abs() + head_tab[h].abs()) * s.abs().unsqueeze(1), Nt),
                indeg=torch.bincount(t, minlength=Nt).double(), ds=ds,
                prior_next=lam * ds + (1 - lam) * prior, pn_scale=lam * ds.abs() + (1 - lam) * prior.abs())


# ---- training aggregate and its backward ----------------------------------------------------------------------------

def _keep(st, mask, p, F, D):
    """Dropout factor per staged fact and column: mask[slot] / (1 - p), or 1 without a mask."""
    if mask is None:
        return torch.ones(F, D, dtype=F64)
    return mask[st["slot_of"]].double() / (1 - p)


def train_aggregate(self_tab, head_tab, s, st, Nt, mask=None, p=0.0):
    """sum_out[n] = sum_{f -> n} drop_f(relu(self_tab[r_f] + head_tab[head_f])) * s_f.  ``mask`` [slots, D] is the
    dropout keep mask (an input here).  Differentiable with torch autograd."""
    a = self_tab[st["rels"]] + head_tab[st["heads"]]
    v = torch.relu(a) * s.unsqueeze(1)
    if mask is not None:
        v = v * mask[st["slot_of"]].double() / (1 - p)
    return torch.zeros(Nt, self_tab.shape[1], dtype=F64).index_add(0, st["tails"], v)


def train_aggregate_scale(self_tab, head_tab, s, st, Nt, mask=None, p=0.0):
    """(|.|-scale, term count) of every train_aggregate element: each term takes at most 3 roundings and the running
    sum one per term, so n = in-degree + 4."""
    self_tab, head_tab, s = self_tab.double(), head_tab.double(), s.double()
    D = self_tab.shape[1]
    keep = _keep(st, mask, p, len(s), D)
    absa = self_tab[st["rels"]].abs() + head_tab[st["heads"]].abs()
    return (_rows(st["tails"], absa * s.abs().unsqueeze(1) * keep, Nt),
            torch.bincount(st["tails"], minlength=Nt).double().unsqueeze(1) + 4)


def train_aggregate_backward(self_tab, head_tab, s, G, st, Nt, mask=None, p=0.0):
    """Gradients of sum(train_aggregate * G): with g_f = G[tail_f] * keep_f and a_f = self_tab[r_f] + head_tab[head_f],
        grad_s[f] = <g_f, relu(a_f)>,  grad_self[r] = sum_{f: r_f = r} g_f s_f [a_f > 0],
        grad_head[n] = sum_{f: head_f = n} g_f s_f [a_f > 0]          (relu'(0) = 0, as torch).
    Returns a dict of (value, |.|-scale, term count) triples under the keys grad_s, grad_self and grad_head; the
    counts are those of the kernels' sums (D + 4 for the dot product of grad_s, the fact count + 3 for the others)."""
    self_tab, head_tab, s, G = self_tab.double(), head_tab.double(), s.double(), G.double()
    R1, D = self_tab.shape
    keep = _keep(st, mask, p, len(s), D)
    h, t, r = st["heads"], st["tails"], st["rels"]
    a = self_tab[r] + head_tab[h]
    g = G[t] * keep
    term = g * s.unsqueeze(1) * (a > 0)
    absa = self_tab[r].abs() + head_tab[h].abs()
    cnt = lambda idx, n: torch.bincount(idx, minlength=n).double().unsqueeze(1) + 3  # noqa: E731
    return dict(grad_s=((g * torch.relu(a)).sum(1), (g.abs() * absa).sum(1), torch.full((len(s),), D + 4.0, dtype=F64)),
                grad_self=(_rows(r, term, R1), _rows(r, term.abs(), R1), cnt(r, R1)),
                grad_head=(_rows(h, term, Nt), _rows(h, term.abs(), Nt), cnt(h, Nt)))


# ---- attention backward ---------------------------------------------------------------------------------------------

def attention_backward(qh, qmask, rel, kfr, gW):
    """Gradients of sum(W * gW) for attention(): with c[b, q, f] = gW[b, f] a[b, q, f] (1 + z[b, q, f] - W[b, f]) / sqrt(D),
        grad_qh[b, q] = sum_f c[b, q, f] rel[r_f],    grad_rel[r] = sum_{(b, f): r_f = r} sum_q c[b, q, f] qh[b, q].
    Returns a dict of (value, |.|-scale, term count) triples under grad_qh [B, Q, D] and grad_rel [R1, D].

    The scale of a term is |gW| a (1 + |z| + |W|)(1 + Z_f) |x| / sqrt(D), Z_f = max_q sum_c |qh_q||rel_r| / sqrt(D)
    the |.|-scale of z.  The count is the roundings of the sum (one per slot with gW != 0, one flush per 64-slot
    block, the add into the caller's buffer) plus those inside one term: z is recomputed as a warp dot product
    (ceil(D/32) fused multiply-adds per lane and a 5-level shuffle tree, then the division), and its error enters a
    twice and (1 + z - W) twice more; the softmax over Q tokens, the exp, the reciprocal and the products add
    2Q + 20, so n_term = 4 (ceil(D/32) + 7) + 2Q + 20."""
    at = attention(qh, qmask, rel, kfr)
    qd, gW = qh.double(), gW.double().reshape(at["W"].shape)
    R1, D = rel.shape
    B, Q, _ = qd.shape
    M = at["W"].shape[1]
    div = np.sqrt(D)
    fe, a, z, W = at["fe"], at["a"], at["z"], at["W"]
    c = gW.unsqueeze(1) * a * (1 + z - W.unsqueeze(1)) / div                       # [B, Q, M]
    Zf = (torch.bmm(qd.abs(), fe.abs().transpose(1, 2)) / div).amax(1, keepdim=True)
    cabs = gW.abs().unsqueeze(1) * a * (1 + z.abs() + W.abs().unsqueeze(1)) * (1 + Zf) / div
    rix = _i64(kfr).reshape(-1)
    per_slot = lambda cc, x: torch.bmm(cc.transpose(1, 2), x).reshape(-1, D)     # noqa: E731
    live = (gW != 0).double()
    n_term = 4 * (-(-D // 32) + 7) + 2 * Q + 20
    cnt_q = (live.sum(1) + -(-M // 64) + 2 + n_term).view(B, 1, 1).expand(B, Q, D)
    cnt_r = (_rows(rix, live.reshape(-1), R1) + Q + 2 + n_term).view(R1, 1).expand(R1, D)
    return dict(grad_qh=(torch.bmm(c, fe), torch.bmm(cabs, fe.abs()), cnt_q),
                grad_rel=(_rows(rix, per_slot(c, qd), R1), _rows(rix, per_slot(cabs, qd.abs()), R1), cnt_r))


# ---- TypeLayer backward ---------------------------------------------------------------------------------------------

def type_layer_backward(G, out, heads, rels, tails, R1, w=None):
    """grad_table[r] = sum over the facts of relation r of w_f (Gm[tail_f] + Gm[head_f]), Gm = G * [out > 0] (the
    relu mask of the forward's output, strict) -> (value, |.|-scale, term count: 2 per fact + 2)."""
    Gm = G.double() * (out > 0)
    wf = torch.ones(len(rels), dtype=F64) if w is None else torch.as_tensor(w).double()
    wf = wf.unsqueeze(1)
    v = (Gm[tails] + Gm[heads]) * wf
    va = (Gm[tails].abs() + Gm[heads].abs()) * wf.abs()
    return _rows(rels, v, R1), _rows(rels, va, R1), 2 * torch.bincount(rels, minlength=R1).double().unsqueeze(1) + 2


def within(got, want, scale, n, what):
    """Assert |got - want| <= n 2^-24 scale + 1e-30 element-wise; reports the worst offender."""
    err = (got.detach().cpu().double() - want).abs()
    bound = n * 2.0 ** -24 * scale + 1e-30
    bad = ~(err <= bound)
    assert not bad.any(), (what, int(bad.sum()), float(err[bad].max()), float(bound[bad].min()),
                           tuple(int(i) for i in bad.nonzero()[0]))
