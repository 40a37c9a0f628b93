"""Plain float64 restatements of the aggregation-family kernels, one fact at a time.

These are the references the kernel-level tests compare with.  They follow the math of the reference model
(reasongnn.py:61-174, layer_init.py:44-59, nsm_gnn.py:101-103) written as per-fact gathers and ``index_add``, with no
shortcut the kernels take (no hoisted relu split, no CSR order), and they do not import ``gnn_rag_b200`` at all:
its torch training path is itself under test.  Gradients come from torch autograd on these functions in float64;
``relu'(0) = 0`` as in torch, which is what the reference's backward uses.

Conventions, shared with ``ops``:
  * node rows are global (``b * N + local``), facts are ``(heads, rels, tails)`` int64 vectors;
  * direction ``"fwd"`` sends messages head -> tail (the tail CSR), ``"inv"`` tail -> head (the head CSR);
  * ``w`` is the per-fact edge weight (normalized_gnn), applied twice, or None for 1.
"""
import torch

F64 = torch.float64
U32 = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)


def _d(t):
    return None if t is None else torch.as_tensor(t).to(F64)


def _i(t):
    return torch.as_tensor(t).to(torch.int64)


def _ends(heads, tails, direction):
    heads, tails = _i(heads), _i(tails)
    if direction == "fwd":
        return heads, tails
    if direction == "inv":
        return tails, heads
    raise ValueError(direction)


def aggregate(table, ins, prior, heads, rels, tails, w, direction):
    """out[n, j*D:(j+1)*D] = sum_{e -> n} w_e^2 * p[src_e] * relu(P[r_e] * x_j[b_e]).

    table [R1, D], ins [B, I, D], prior [B, N] (or [B*N] with N = Nt / B); returns [B*N, I*D] (the layout of
    ``ops.aggregate`` with seg_stride = D).  Differentiable in table, ins and prior."""
    B, I, D = ins.shape
    Nt = prior.numel()
    N = Nt // B
    src, dst = _ends(heads, tails, direction)
    r = _i(rels)
    b = dst // N
    c = prior.reshape(-1)[src]
    if w is not None:
        wd = _d(w)
        c = wd * wd * c
    msg = torch.relu(table[r].unsqueeze(1) * ins[b]) * c.view(-1, 1, 1)       # [F, I, D]
    out = torch.zeros(Nt, I, D, dtype=msg.dtype, device=msg.device).index_add_(0, dst, msg)
    return out.reshape(Nt, I * D)


def aggregate_abs(table, ins, prior, heads, rels, tails, w, direction):
    """The same sum with |P|, |x| and |p|: sum_e w_e^2 |p[src_e]| |P[r_e]| |x_j[b_e]|, the magnitude every
    rounding error of the kernel's sum is relative to.  Autograd of this function with grad_outputs = |G| gives the
    matching scale of each gradient element (|G| substituted for G)."""
    return aggregate(table.abs(), ins.abs(), prior.abs(), heads, rels, tails, w, direction)


def type_layer(table, heads, rels, tails, wr, Nt):
    """relu(sum_{facts into n as tail} wr * P[r] + sum_{facts into n as head} wr * P[r])  (layer_init.py:44-57).
    Returns [Nt, D]."""
    heads, tails, r = _i(heads), _i(tails), _i(rels)
    val = table[r]
    if wr is not None:
        val = val * _d(wr).view(-1, 1)
    z = torch.zeros(Nt, table.shape[1], dtype=val.dtype, device=val.device)
    return torch.relu(z.index_add(0, tails, val) + z.index_add(0, heads, val))


def type_layer_abs(table, heads, rels, tails, wr, Nt):
    """sum over both directions of |wr| |P[r]|: the error scale of :func:`type_layer` (before the relu)."""
    heads, tails, r = _i(heads), _i(tails), _i(rels)
    val = table[r].abs()
    if wr is not None:
        val = val * _d(wr).abs().view(-1, 1)
    z = torch.zeros(Nt, table.shape[1], dtype=val.dtype, device=val.device)
    return z.index_add(0, tails, val) + z.index_add(0, heads, val)


def layer_input(h, prior, tf, ti, ins, facts, w):
    """[h | nb_0,fwd | nb_0,inv | nb_1,fwd | ...]: the e2e_linear input of ReasonGNNLayer.forward
    (reasongnn.py:150-161).  h [Nt, D]; facts = (heads, rels, tails)."""
    heads, rels, tails = facts
    B, I, D = ins.shape
    Nt = h.shape[0]
    fwd = aggregate(tf, ins, prior, heads, rels, tails, w, "fwd").view(Nt, I, 1, D)
    inv = aggregate(ti, ins, prior, heads, rels, tails, w, "inv").view(Nt, I, 1, D)
    return torch.cat([h, torch.cat([fwd, inv], dim=2).reshape(Nt, 2 * I * D)], dim=1)


def rearev_layer(h, prior, tf, ti, ins, W, b, w_score, facts, w):
    """y = relu(W [h | nb...] + b) and the score dot y . w_score (no score bias): ReasonGNNLayer.forward
    (reasongnn.py:150-165).  W [D, (2I+1) D] as torch Linear; b / w_score may be None."""
    x = layer_input(h, prior, tf, ti, ins, facts, w)
    pre = x @ W.t()
    if b is not None:
        pre = pre + b
    y = torch.relu(pre)
    s = y @ w_score if w_score is not None else torch.zeros(y.shape[0], dtype=y.dtype, device=y.device)
    return y, s


def rearev_layer_scale(h, prior, tf, ti, ins, W, b, facts, w):
    """|W| [|h| | aggregate_abs...] + |b|: the per-element scale of :func:`rearev_layer`'s pre-activation."""
    x = layer_input(h.abs(), prior.abs(), tf.abs(), ti.abs(), ins.abs(), facts, w)
    pre = x @ W.abs().t()
    return pre + b.abs() if b is not None else pre


def nsm_layer(h, prior, table, ins, W, b, w_score, facts, w):
    """One NSM step, forward direction, one instruction (nsm_gnn.py:54-77, 87-112): y = relu(W [h | nb] + b) with
    nb[n] = sum_{e -> n} w_e^2 p[head_e] relu(P[r_e] * ins[b_e]), the score dot y . w_score (no score bias) and the
    ``possible`` mask reason_kb multiplies into the answer mask.  ins [B, D]; returns (y, s, possible)."""
    x = torch.cat([h, aggregate(table, ins.unsqueeze(1), prior, *facts, w, "fwd")], dim=1)
    y = torch.relu(x @ W.t() + b)
    return y, y @ w_score, possible(prior, facts, w, h.shape[0])[0]


def nsm_layer_scale(h, prior, table, ins, W, b, facts, w):
    """|W| [|h| | aggregate_abs] + |b|: the per-element scale of :func:`nsm_layer`'s pre-activation."""
    x = torch.cat([h.abs(), aggregate_abs(table, ins.unsqueeze(1), prior, *facts, w, "fwd")], dim=1)
    return x @ W.abs().t() + b.abs()


def _graft_layer(h, d, q, fact_rel, W_tilde, E, e2f, f2e, lin, score_w, lam, fact_scale, act):
    B, N = d.shape
    Mf, D = W_tilde.shape[1], h.shape[1]
    eb, ef, en = (_i(a) for a in e2f)
    fb, fn, ff = (_i(a) for a in f2e)
    eslot, enode = eb * Mf + ef, eb * N + en
    fslot, fnode = fb * Mf + ff, fb * N + fn

    def linear(x, name):
        W, b = lin[name]
        return x @ W.t() + b

    head = linear(h, "kb_head")
    e2f_emb = act(linear(fact_rel.reshape(B * Mf, D), "kb_self")
                  + torch.zeros(B * Mf, D, dtype=h.dtype).index_add_(0, eslot, head[enode]))          # :118-121
    norm = W_tilde.reshape(-1) * torch.zeros(B * Mf, dtype=h.dtype).index_add_(0, eslot, (d.reshape(-1) / E.reshape(-1))[enode])
    e2f_emb = e2f_emb * norm.unsqueeze(1)                                                              # :122-124
    tail = linear(e2f_emb, "kb_tail")                     # the bias enters once per (fact, tail) pair
    f2e_emb = act(linear(h, "kb_self") + torch.zeros(B * N, D, dtype=h.dtype).index_add_(0, fnode, tail[fslot]))
    nd = lam * torch.zeros(B * N, dtype=h.dtype).index_add_(0, fnode, norm[fslot]) + (1 - lam) * d.reshape(-1)
    node_b = torch.arange(B * N) // N
    x = torch.cat([h, linear(q, "q2e")[node_b], fact_scale * f2e_emb], dim=1)                          # :136-137
    query = torch.zeros(B, D, dtype=h.dtype).index_add_(0, node_b, nd.unsqueeze(1) * linear(x, "e2q"))
    y = act(linear(x, "e2e"))
    return y, y @ score_w, nd.view(B, N), query


def graft_layer(h, d, q, fact_rel, W_tilde, E, e2f, f2e, lin, score_w, lam, fact_scale):
    """One GraftNet layer (graft_gnn.py:111-153) as per-fact gathers and ``index_add``.  h [B*N, D] node embeddings,
    d [B, N] PageRank prior, q [B, D] query (query_node_emb at layer 0), fact_rel [B, M, D] = rel[kb_fact_rel],
    W_tilde [B, M] fact attention, E [B, N] its clamped per-head sum; e2f = (b, fact slot, head) and
    f2e = (b, tail, fact slot) index lists; lin: name -> (W, b) for q2e, e2q, e2e, kb_head, kb_tail, kb_self;
    score_w [D].  Returns (h' = relu(e2e(x)), its score dot (no score bias), the next prior d' [B, N], query_emb
    [B, D] = sum_n d'[n] e2q(x[n]))."""
    return _graft_layer(h, d, q, fact_rel, W_tilde, E, e2f, f2e, lin, score_w, lam, fact_scale, torch.relu)


def graft_layer_scale(h, d, q, fact_rel, W_tilde, E, e2f, f2e, lin, score_w, lam, fact_scale):
    """:func:`graft_layer` on |inputs| and |weights| with the relus dropped: an elementwise envelope of every
    pre-activation and output, the magnitude each rounding error along the layer is relative to.  An error of at
    most e times its envelope in any intermediate stays within e times the envelope of each result."""
    absl = {k: (W.abs(), b.abs()) for k, (W, b) in lin.items()}
    return _graft_layer(h.abs(), d.abs(), q.abs(), fact_rel.abs(), W_tilde.abs(), E.abs(), e2f, f2e, absl,
                        score_w.abs(), lam, abs(fact_scale), lambda t: t)


def possible(prior, facts, w, Nt):
    """sum_{e -> n} w_e^2 p[head_e] > 1e-10 per tail row n (nsm_gnn.py:101-103), as float 0/1."""
    heads, _rels, tails = facts
    heads, tails = _i(heads), _i(tails)
    c = prior.reshape(-1)[heads]
    if w is not None:
        wd = _d(w)
        c = wd * wd * c
    mass = torch.zeros(Nt, dtype=c.dtype, device=c.device).index_add_(0, tails, c)
    return (mass > 1e-10).to(F64), mass
