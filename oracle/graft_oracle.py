"""Torch-CPU restatement of GraftNet inference in the reference's op order (gnn/models/GraftNet/graftnet.py:105-183,
gnn/modules/kg_reasoning/graft_gnn.py:45-153, base_gnn.py:56-75): the CPU baseline of scripts/graftnet_probe.py and the
host-side check of tests/test_graftnet_host.py.  It reads the parameters of a ``gnn_rag_b200.GraftNet`` (same names as
the reference) and runs the same sparse ``bmm`` operators the reference builds, on CPU."""
import numpy as np
import torch
import torch.nn.functional as F

VERY_SMALL_NUMBER = 1e-10
VERY_NEG_NUMBER = -100000000000


def _sparse(idx, n, size):
    return torch.sparse_coo_tensor(torch.as_tensor(np.stack(idx), dtype=torch.long),
                                   torch.ones(n, dtype=torch.float32), size)


def _type_layer(lin, kb, rel_features, B, N, norm_rel):
    """layer_init.py:25-62."""
    heads, rels, tails = (torch.as_tensor(np.asarray(a), dtype=torch.long) for a in kb[:3])
    fact_val = lin(rel_features[rels])
    if norm_rel:
        fact_val = fact_val * torch.as_tensor(np.asarray(kb[6], dtype=np.float32)).unsqueeze(1)
    Nt, Fn = B * N, len(heads)
    f2t = torch.sparse_coo_tensor(torch.stack([tails, torch.arange(Fn)]), torch.ones(Fn), (Nt, Fn))
    f2h = torch.sparse_coo_tensor(torch.stack([heads, torch.arange(Fn)]), torch.ones(Fn), (Nt, Fn))
    return F.relu(torch.sparse.mm(f2t, fact_val) + torch.sparse.mm(f2h, fact_val)).view(B, N, -1)


@torch.no_grad()
def forward(model, batch):
    """-> dict(loss, pred, pred_dist, dist_history [L,B,N], pagerank_history [L,B,N]) as numpy / floats."""
    m = model
    local_entity, _qe, kb, graft, q_input, kb_fact_rel, seed_dist, _tb, answer_dist = batch[:9]
    local_entity = torch.as_tensor(local_entity, dtype=torch.long)
    B, N = local_entity.shape
    D = m.entity_dim
    layer = m.reasoning
    q_input = torch.as_tensor(q_input, dtype=torch.long)
    enc = m.instruction
    enc.encode_question_train(q_input)
    qh, qnode, qmask = enc.query_hidden_emb, enc.query_node_emb, enc.query_mask_train
    rel = m.get_rel_feature_train()
    if m.encode_type:
        h = _type_layer(m.type_layer.kb_self_linear, kb, rel, B, N, m.norm_rel)
    else:
        h = m.entity_linear(m.entity_embedding(local_entity))
    (e2f_b, e2f_f, e2f_e, _v0), (f2e_b, f2e_e, f2e_f, _v1) = graft
    kfr = torch.as_tensor(kb_fact_rel, dtype=torch.long)
    M = kfr.shape[1]
    e2f = _sparse([e2f_b, e2f_f, e2f_e], len(e2f_b), (B, M, N))            # entity2fact_mat [B, max_fact, N]
    f2e = _sparse([f2e_b, f2e_e, f2e_f], len(f2e_b), (B, N, M))            # fact2entity_mat [B, N, max_fact]
    fact_emb = rel[kfr]
    div = float(np.sqrt(D))
    sim = torch.bmm(qh, fact_emb.transpose(1, 2)) / div
    sim = torch.softmax(sim + (1 - qmask.unsqueeze(dim=2)) * VERY_NEG_NUMBER, dim=1)
    att = torch.sum(sim.unsqueeze(dim=3) * qh.unsqueeze(dim=2), dim=1)
    W = torch.sum(att * fact_emb, dim=2) / div
    W_tilde = torch.exp(W - torch.max(W, dim=1, keepdim=True)[0])
    E = torch.clamp(torch.bmm(e2f.transpose(1, 2), W_tilde.unsqueeze(dim=2)).squeeze(dim=2), min=VERY_SMALL_NUMBER)
    mask = (local_entity != m.num_entity).float()
    d = torch.as_tensor(seed_dist, dtype=torch.float32)
    query = qnode
    hist, pr = [], []
    for i in range(m.num_layer):
        lin = lambda n: layer.lin(n, i)  # noqa: E731
        q2e = lin("q2e_linear")(query).expand(B, N, D)
        e2f_emb = F.relu(lin("kb_self_linear")(fact_emb) + torch.bmm(e2f, lin("kb_head_linear")(h)))
        e2f_norm = W_tilde.unsqueeze(dim=2) * torch.bmm(e2f, (d / E).unsqueeze(dim=2))
        e2f_emb = e2f_emb * e2f_norm
        f2e_emb = F.relu(lin("kb_self_linear")(h) + torch.bmm(f2e, lin("kb_tail_linear")(e2f_emb)))
        nd = torch.bmm(f2e, e2f_norm).squeeze(dim=2)
        nd = layer.pagerank_lambda * nd + (1 - layer.pagerank_lambda) * d
        x = torch.cat((torch.cat((h, q2e), dim=2), layer.fact_scale * f2e_emb), dim=2)
        query = torch.bmm(nd.unsqueeze(dim=1), lin("e2q_linear")(x))
        h = F.relu(lin("e2e_linear")(x))
        logit = layer.score_func(h).squeeze(dim=2)
        hist.append(torch.softmax(logit + (1 - mask) * VERY_NEG_NUMBER, dim=1))
        d = nd
        pr.append(d)
    ans = torch.as_tensor(answer_dist, dtype=torch.float32)
    valid = (torch.sum(ans, dim=1, keepdim=True) > 0).float()
    loss = m.calc_loss_label(logit, ans, valid)
    pred_dist = hist[-1]
    return dict(loss=float(loss), pred=pred_dist.argmax(1).numpy(), pred_dist=pred_dist.numpy(),
                dist_history=torch.stack(hist).numpy(), pagerank_history=torch.stack(pr).numpy())


def candidate_lists(pred_dist, batch, num_entity, eps):
    """Evaluator.evaluate's candidate cut + f1_and_hits (gnn/evaluate.py:188-209, 25-67) -> per-question entity ids."""
    local_entity, query_entities = batch[0], batch[1]
    B, N = local_entity.shape
    out = []
    for b in range(B):
        cand = [(int(c), float(p)) for c, p, s in zip(local_entity[b], pred_dist[b], query_entities[b])
                if s != 1.0 and c != num_entity and p >= (1 - eps) / N]
        cand.sort(key=lambda x: x[1], reverse=True)
        ids, acc = [], 0.0
        for c, p in cand:
            ids.append(c)
            acc += p
            if acc > eps:
                break
        out.append(ids)
    return out
