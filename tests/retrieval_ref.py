"""Exact restatements of the reference's retrieval output, independent of every kernel and of the package:
candidate ranking (gnn/evaluate.py:155-209 and the sort / cut of f1_and_hits :34-50), the train-time metrics
(gnn/models/base_model.py:217-298: get_eval_metric, calc_h1, calc_f1_new, f1_and_hits) and the shortest-path node
sets behind the LLM stage's reasoning paths (llm/src/utils/graph_utils.py:10-21, 49-75).

Everything here runs on the CPU in Python floats (float64) or torch CPU tensors, in the reference's own order of
operations.  tests/test_retrieval_edges_gpu.py holds gr_rank_candidates, gr_train_metrics and gr_shortest_path_nodes
to these bit for bit; tests/test_retrieval_edges_host.py pins them to the oracle and to networkx."""
import numpy as np
import torch
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import shortest_path


# ---- candidate ranking ------------------------------------------------------------------------------------------------

def rank_full(local_entity, query_entities, pred_dist, pad_id, eps):
    """Per question: (every surviving candidate in retrieval order, the eps-mass cut).  A candidate is (local index,
    entity id, prob as a Python float); the cut is the number the evaluator keeps.

    Survivors: not a seed (``int(s) == 1``: the reference casts query_entities to a LongTensor, which truncates), not a
    pad (``c == pad_id``) and not ``p < (1 - eps) / N`` in float64.  Order: python's stable ``sorted(..., reverse=True)``
    on p, so equal p keep local-index order.  Cut: the prefix up to and including the item at which the sequential
    float64 running sum first exceeds eps; all of them when it never does."""
    local_entity = np.asarray(local_entity)
    B, N = local_entity.shape
    ignore_prob = (1 - eps) / N
    probs_all = np.asarray(pred_dist, dtype=np.float32)
    seeds_all = torch.from_numpy(np.asarray(query_entities, dtype=np.float32)).long()
    out = []
    for b in range(B):
        probs = probs_all[b].tolist()
        cands = local_entity[b].tolist()
        seeds = seeds_all[b].tolist()
        cand = []
        for n, (c, p, s) in enumerate(zip(cands, probs, seeds)):
            if s == 1:
                continue
            if c == pad_id:
                continue
            if p < ignore_prob:
                continue
            cand.append((n, c, p))
        cand = sorted(cand, key=lambda x: x[2], reverse=True)
        tp_prob = 0.0
        cut = 0
        for _n, _c, p in cand:
            tp_prob += p
            cut += 1
            if tp_prob > eps:
                break
        out.append((cand, cut))
    return out


def rank(local_entity, query_entities, pred_dist, pad_id, eps):
    """Per question: the retrieved list [(local index, entity id, prob), ...] in retrieval order (the
    ``oracle.kgqa_oracle.rank_candidates`` layout)."""
    return [cand[:cut] for cand, cut in rank_full(local_entity, query_entities, pred_dist, pad_id, eps)]


# ---- train-time metrics -----------------------------------------------------------------------------------------------

def _f1_and_hits(answers, candidate2prob, eps):
    """BaseModel.f1_and_hits (base_model.py:217-234): the F1 of the eps-mass prefix of the sorted candidates."""
    retrieved = []
    correct = 0
    cand_list = sorted(candidate2prob, key=lambda x: x[1], reverse=True)
    tp_prob = 0.0
    for c, prob in cand_list:
        retrieved.append((c, prob))
        tp_prob += prob
        if c in answers:
            correct += 1
        if tp_prob > eps:
            break
    if len(answers) == 0:
        return 1.0 if len(retrieved) == 0 else 0.0
    if len(retrieved) == 0:
        return 0.0
    p, r = correct / len(retrieved), correct / len(answers)
    return 2.0 / (1.0 / p + 1.0 / r) if p != 0 and r != 0 else 0.0


def train_metrics(pred_dist, answer_dist, seed_dist, local_entity, pad_id, eps):
    """get_eval_metric (base_model.py:281-298) -> (h1, f1), fp32 numpy [B].

    calc_h1: ``torch.argmax`` of the fp32 pred_dist on the CPU (the first maximal index, NaN counts as maximal) and
    ``answer_dist > 1e-10`` compared as the fp32 tensor compares it.  calc_f1_new, for hit@1 questions only: answers are
    the entity ids of the non-seed (``s > 0``), non-pad nodes with ``p_a > 0`` (a list: repeats count), candidates the
    non-seed, non-pad nodes with ``p >= (1 - eps) / N`` in float64; the F1 of their eps-mass prefix is computed in
    float64 and rounded once to fp32 (``torch.FloatTensor``)."""
    pd = torch.from_numpy(np.ascontiguousarray(pred_dist, dtype=np.float32))
    ad = torch.from_numpy(np.ascontiguousarray(answer_dist, dtype=np.float32))
    B, N = pd.shape
    top1 = pd.argmax(dim=-1, keepdim=True)
    dist_top1 = torch.zeros_like(pd).scatter_(1, top1, 1.0)
    h1 = (torch.sum(dist_top1 * (ad > 1e-10).float(), dim=-1) > 0).float()
    ignore_prob = (1 - eps) / N
    seeds_all = np.asarray(seed_dist, dtype=np.float32)
    le = np.asarray(local_entity)
    f1_list = []
    for b in range(B):
        if h1[b].item() == 0.0:
            f1_list.append(0.0)
            continue
        answer_list, candidate2prob = [], []
        for c, p, p_a, s in zip(le[b].tolist(), pd[b].tolist(), ad[b].tolist(), seeds_all[b].tolist()):
            if s > 0:
                continue
            if c == pad_id:
                continue
            if p_a > 0:
                answer_list.append(c)
            if p < ignore_prob:
                continue
            candidate2prob.append((c, p))
        f1_list.append(_f1_and_hits(answer_list, candidate2prob, eps))
    return h1.numpy(), torch.FloatTensor(f1_list).numpy()


# ---- shortest-path node sets ------------------------------------------------------------------------------------------

def path_nodes(heads, tails, N, sources, targets):
    """Hop distances on the undirected, unweighted graph of the (head, tail) pairs (self-loops ignored, as
    ``nx.Graph`` has no use for them; parallel edges are one edge) -> (dist_s int32 [S, N], dist_t int32 [T, N],
    pair_dist int32 [S, T], sorted node list).  -1 = unreachable.  The nodes are those on any shortest path of a
    connected (source, target) pair: {v : d(s, v) + d(v, t) = d(s, t)}."""
    h = np.asarray(heads, dtype=np.int64)
    t = np.asarray(tails, dtype=np.int64)
    keep = h != t
    h, t = h[keep], t[keep]
    adj = csr_matrix((np.ones(len(h)), (h, t)), shape=(N, N))

    def dists(roots):
        if len(roots) == 0:
            return np.zeros((0, N), dtype=np.int32)
        d = shortest_path(adj, directed=False, unweighted=True, indices=np.asarray(roots, dtype=np.int64))
        d = np.atleast_2d(d)
        return np.where(np.isinf(d), -1, d).astype(np.int32)

    ds, dt = dists(sources), dists(targets)
    pair = np.full((len(sources), len(targets)), -1, dtype=np.int32)
    on = np.zeros(N, dtype=bool)
    for i in range(len(sources)):
        for j, tg in enumerate(targets):
            d = ds[i, tg]
            pair[i, j] = d
            if d >= 0:
                on |= (ds[i] >= 0) & (dt[j] >= 0) & (ds[i] + dt[j] == d)
    return ds, dt, pair, np.nonzero(on)[0].tolist()
