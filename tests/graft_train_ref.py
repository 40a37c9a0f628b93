"""float64 restatements of GraftNet's training forward in the decomposition the GPU kernels implement
(autograd_path.graftnet_forward's kernel path): fact attention per slot, the fact-message sum per node with
kb_tail_linear applied after it, and the TypeLayer as per-fact sums.  Differentiable with torch autograd."""
import numpy as np
import torch
import torch.nn.functional as F

import graft_edges_ref as R

ref_aggregate = R.train_aggregate


def ref_attention(qh, qmask, rel, kfr):
    """W [B, max_fact] of compute_attention (graft_gnn.py:64-87) for every slot, and the softmax a [B, Q, max_fact]."""
    at = R.attention(qh, qmask, rel, kfr)
    return at["W"], at["a"]


def graftnet_fp64(m, batch):
    """GraftNet's forward (graftnet.py:135-183) in float64 from the model's fp32 parameters (dropout off): returns
    (last-layer logits [B, N], PageRank history [layers, B, N])."""
    le, _qe, kb, graft, q_input, kfr, seed_dist = batch[:7]
    B, N = le.shape
    Nt, D = B * N, m.entity_dim
    layer = m.reasoning

    def lin(mod, x):
        return F.linear(x, mod.weight.double(), mod.bias.double() if mod.bias is not None else None)

    def L(name, i, x):
        return lin(layer.lin(name, i), x)
    rel = m.get_rel_feature_train().double()
    le_t = torch.as_tensor(le)
    if m.encode_type:
        heads, rels, tails = (torch.as_tensor(np.asarray(x, dtype=np.int64)) for x in kb[:3])
        fv = lin(m.type_layer.kb_self_linear, rel)[rels]
        if m.norm_rel:
            fv = fv * torch.as_tensor(np.asarray(kb[6], dtype=np.float64)).unsqueeze(1)
        z = torch.zeros(Nt, D, dtype=torch.float64)
        h = torch.relu(z.index_add(0, tails, fv) + z.index_add(0, heads, fv))
    else:
        h = lin(m.entity_linear, m.entity_embedding(le_t).double()).view(Nt, D)
    enc = m.instruction
    enc.encode_question_train(torch.as_tensor(q_input))
    qh, query, qmask = enc.query_hidden_emb.double(), enc.query_node_emb.double(), enc.query_mask_train.double()
    kfr = np.asarray(kfr, dtype=np.int64)
    st = R.stage(graft[0][:3], graft[1][:3], kfr, N)
    W, _a = ref_attention(qh, qmask, rel, kfr)
    Wt = R.w_tilde(W)
    E = R.e_sum(Wt, st, Nt)[0]
    d = torch.as_tensor(np.asarray(seed_dist, dtype=np.float64)).reshape(-1)
    lam = layer.pagerank_lambda
    pr = []
    for i in range(m.num_layer):
        q2e = L("q2e_linear", i, query).expand(B, N, D).reshape(Nt, D)
        kt = layer.lin("kb_tail_linear", i)
        ag = R.aggregate(Wt, E, d, L("kb_self_linear", i, rel), L("kb_head_linear", i, h), st, lam, Nt)
        sum_v, indeg = ag["sum_out"], ag["indeg"].unsqueeze(1)
        f2e = torch.relu(L("kb_self_linear", i, h) + sum_v @ kt.weight.double().t() + indeg * kt.bias.double())
        d = ag["prior_next"]
        x = torch.cat([h, q2e, layer.fact_scale * f2e], dim=1)
        query = torch.bmm(d.view(B, 1, N), L("e2q_linear", i, x).view(B, N, D))
        h = torch.relu(L("e2e_linear", i, x))
        logit = lin(layer.score_func, h).view(B, N)
        pr.append(d.view(B, N))
    return logit, torch.stack(pr)
