"""Seeded synthetic KGQA batches in the exact ``SingleDataLoader.get_batch`` tuple layout.

The reference batches questions block-diagonally (gnn/dataset_load.py:473-527, 599-629): node
``local`` of question ``b`` is global row ``b*N + local``; every real node gets one self-loop fact
with relation id ``num_relation-1`` (dataset_load.py:499-506); pads carry entity id ``num_entity``
(dataset_load.py:250-257).  This module emits that tuple from a ``numpy.random.RandomState`` so the
oracle, the parity tests and bench.py all see the same inputs (SURVEY.md §8d).

Tuple layout (dataset_load.py:623-629):
  [0] local_entity   int64  [B,N]   global entity ids, pad = num_entity
  [1] query_entities float64[B,N]   1.0 on seed nodes
  [2] kb_adj_mat     (heads, rels, tails, batch_ids, fact_ids, weight_list, weight_rel_list)
  [3] q_input        int64  [B,Q]   token ids, pad = num_word
  [4] seed_dist      float64[B,N]   1/k on the k seeds
  [5] true_batch_id  None
  [6] answer_dist    float64[B,N]   1.0 on answer nodes
  ([7] answer_lists  object [B]     only with test=True)
"""
from collections import Counter

import numpy as np

# WebQSP-like vocabulary sizes (SURVEY.md §8d)
WEBQSP_NUM_RELATION = 6106  # relation ids incl. self-loop; table rows R1 = NUM_RELATION + 1
WEBQSP_NUM_ENTITY = 100_000
WEBQSP_NUM_WORD = 5_000


def _degree_weights(heads, rels):
    """1/outdeg(head) and 1/count(head,rel) exactly as dataset_load.py:509-517 (python lists)."""
    head_count = Counter(heads.tolist())
    weight_list = [1.0 / head_count[h] for h in heads.tolist()]
    hr = list(zip(heads.tolist(), rels.tolist()))
    hr_count = Counter(hr)
    weight_rel_list = [1.0 / hr_count[k] for k in hr]
    return weight_list, weight_rel_list


def make_batch(seed, B, N, E, num_entity=WEBQSP_NUM_ENTITY, num_relation=WEBQSP_NUM_RELATION,
               num_word=WEBQSP_NUM_WORD, Q=12, n_real=None, powerlaw=False, multi_seed=False,
               n_answers=2, with_weights=True, test=False, seeds_are_pad=False,
               empty_questions=()):
    """Build one batch.

    n_real:     number of real (non-pad) nodes per question; int, or None for N, or "ragged" to
                draw per-question sizes in [N//4, N].
    powerlaw:   tails drawn from a Zipf-like law so a few hub nodes get most in-edges.
    multi_seed: 2-3 seeds per question with 1/k mass (dataset_load.py:293-295).
    seeds_are_pad: reproduce the non-CWQ quirk that seed nodes keep the pad entity id
                (dataset_load.py:250-257) so their probability is forced to 0.
    empty_questions: question indices that get no real nodes and no facts (all-padding row).
    with_weights: build the two python weight lists (slow for large F; only needed by
                normalized_gnn / norm_rel).
    """
    rs = np.random.RandomState(seed)
    local_entity = np.full((B, N), num_entity, dtype=np.int64)
    query_entities = np.zeros((B, N), dtype=np.float64)
    seed_dist = np.zeros((B, N), dtype=np.float64)
    answer_dist = np.zeros((B, N), dtype=np.float64)
    q_input = np.full((B, Q), num_word, dtype=np.int64)
    heads, rels, tails, bids = [], [], [], []
    answer_lists = []
    for b in range(B):
        if b in empty_questions:
            answer_lists.append([])
            continue
        if n_real is None:
            nr = N
        elif n_real == "ragged":
            nr = int(rs.randint(max(2, N // 4), N + 1))
        else:
            nr = int(n_real)
        nr = max(2, min(nr, N))
        local_entity[b, :nr] = rs.randint(0, num_entity, size=nr)
        k = int(rs.randint(2, 4)) if multi_seed else 1
        k = min(k, nr - 1)
        seeds = np.arange(k)
        query_entities[b, seeds] = 1.0
        seed_dist[b, seeds] = 1.0 / k
        if seeds_are_pad:
            local_entity[b, seeds] = num_entity
        na = min(n_answers, nr - k)
        ans = k + rs.choice(nr - k, size=na, replace=False)
        answer_dist[b, ans] = 1.0
        answer_lists.append(local_entity[b, ans].tolist())
        qlen = int(rs.randint(3, Q + 1))
        q_input[b, :qlen] = rs.randint(0, num_word, size=qlen)
        e = int(E * nr / N) if n_real == "ragged" else E
        h = rs.randint(0, nr, size=e)
        if powerlaw:
            # Zipf-like destination choice: a handful of hubs soak up most in-edges
            # (hubs sit at the high local ids so they do not coincide with the seeds at 0..k-1)
            ranks = np.minimum((rs.pareto(1.1, size=e)).astype(np.int64), nr - 1)
            t = nr - 1 - ranks
        else:
            t = rs.randint(0, nr, size=e)
        # guarantee the seeds have out-edges so that mass can flow
        ns = min(e, 8 * k)
        h[:ns] = np.repeat(seeds, 8)[:ns]
        r = rs.randint(0, num_relation - 1, size=e)
        off = b * N
        heads.append(h + off)
        rels.append(r)
        tails.append(t + off)
        bids.append(np.full(e, b, dtype=np.int64))
        # self loops for every real node (dataset_load.py:499-506)
        ent = np.arange(nr, dtype=np.int64) + off
        heads.append(ent)
        tails.append(ent)
        rels.append(np.full(nr, num_relation - 1, dtype=np.int64))
        bids.append(np.full(nr, b, dtype=np.int64))
    if heads:
        batch_heads = np.concatenate(heads).astype(np.int64)
        batch_rels = np.concatenate(rels).astype(np.int64)
        batch_tails = np.concatenate(tails).astype(np.int64)
        batch_ids = np.concatenate(bids).astype(np.int64)
    else:
        batch_heads = batch_rels = batch_tails = batch_ids = np.zeros(0, dtype=np.int64)
    fact_ids = np.arange(len(batch_heads), dtype=np.int64)
    if with_weights:
        weight_list, weight_rel_list = _degree_weights(batch_heads, batch_rels)
    else:
        weight_list, weight_rel_list = None, None
    kb_adj_mat = (batch_heads, batch_rels, batch_tails, batch_ids, fact_ids, weight_list,
                  weight_rel_list)
    out = (local_entity, query_entities, kb_adj_mat, q_input, seed_dist, None, answer_dist)
    if test:
        al = np.empty(B, dtype=object)
        for i, a in enumerate(answer_lists):
            al[i] = a
        out = out + (al,)
    return out


def model_args(model_name="ReaRev", entity_dim=200, num_iter=3, num_ins=2, num_gnn=3, num_step=3, num_layer=3,
               data_folder="", use_cuda=False, **over):
    """The ``args`` dict the reference threads everywhere (gnn/parsing.py:13-125, main.py:33).

    ``kg_dim = entity_dim/2`` because with ``lm='lstm'`` ReaRev rebuilds ``relation_linear`` as
    Linear(D, D) (rearev.py:125) while relation embeddings have ``2*kg_dim`` columns
    (base_model.py:144) -- SURVEY.md §8c.
    """
    args = dict(
        model_name=model_name, name="synthetic", data_folder=data_folder, use_cuda=use_cuda,
        word2id="vocab.txt", relation2id="relations.txt", entity2id="entities.txt",
        entity_emb_file=None, relation_emb_file=None, relation_word_emb=False,
        word_emb_file=None, kge_frozen=0, lm="lstm", lm_frozen=1,
        entity_dim=entity_dim, kg_dim=entity_dim // 2, word_dim=300,
        lm_dropout=0.3, linear_dropout=0.2, eps=0.95, q_type="seq", loss_type="kl",
        use_self_loop=True, normalized_gnn=False, norm_rel=False, data_eff=False,
        test_batch_size=20, batch_size=20, fact_drop=0, is_eval=True,
        checkpoint_dir="checkpoint/", experiment_name="synthetic",
    )
    if model_name == "ReaRev":
        args.update(alg="bfs", num_iter=num_iter, num_ins=num_ins, num_gnn=num_gnn, pos_emb=False)
    elif model_name == "NSM":
        args.update(num_step=num_step, reason_kb=False, lambda_constrain=0.0, lambda_back=0.0,
                    use_inverse_relation=False)
    elif model_name == "GraftNet":                 # create_parser_graftnet, gnn/parsing.py:115-124; fact_scale :42
        args.update(num_layer=num_layer, pagerank_lambda=0.8, loss_type="bce", use_inverse_relation=False,
                    fact_scale=3)
    else:
        raise ValueError(model_name)
    args.update(over)
    return args


def make_graft_batch(seed, B, N, E, num_entity=WEBQSP_NUM_ENTITY, num_relation=WEBQSP_NUM_RELATION,
                     num_word=WEBQSP_NUM_WORD, fact_dropout=0.0, use_inverse_relation=False, test=False, **kw):
    """One batch in the ``GraftSingleDataLoader.get_batch`` layout (gnn/dataset_load_graft.py:113-149):

      [0] local_entity [1] query_entities [2] kb_adj_mat (as :func:`make_batch`, self-loops included)
      [3] kb_adj_mat_graft = ((b, f, head, 1.0), (b, tail, f, 1.0))   the tuples only, no self-loops
      [4] q_input [5] kb_fact_rel int64 [B, max_fact] [6] seed_dist [7] true_batch_id = None [8] answer_dist
      ([9] answer_lists with ``test=True``)

    The tuples of question b are the non-self-loop facts :func:`make_batch` draws for it.  As the loader does
    (dataset_load_graft.py:27-102, dataset_load.py:265-291): max_fact = 2 * max_tuples + N; kb_fact_rel slots past the
    tuples hold the pad relation ``num_relation`` (the last row of the [num_relation + 1, D] table); every question's
    facts are permuted and only floor(n * (1 - fact_dropout)) of them kept.  With ``use_inverse_relation`` the relation
    ids are drawn from the lower half, tuple i becomes graft facts 2i (head -> tail) and 2i+1 (tail -> head), and
    kb_fact_rel[b, i] holds the INVERSE relation of tuple i -- the loader's own layout, which the model reads as is."""
    base = make_batch(seed, B, N, E, num_entity=num_entity, num_relation=num_relation, num_word=num_word, test=test,
                      **kw)
    return graft_from_batch(base, seed, num_relation, fact_dropout, use_inverse_relation)


def graft_from_batch(base, seed, num_relation, fact_dropout=0.0, use_inverse_relation=False):
    """The graft tuple of :func:`make_graft_batch` around an existing ``make_batch`` tuple (its non-self-loop facts
    are the tuples)."""
    test = len(base) > 7
    B, N = base[0].shape
    local_entity, query_entities, kb, q_input, seed_dist, _tb, answer_dist = base[:7]
    heads, rels, tails, bids, fids, wl, wrl = kb
    loop = num_relation - 1
    half = (num_relation - 1) // 2
    rels = rels.copy()
    if use_inverse_relation:
        rels[rels != loop] %= half
    kb = (heads, rels, tails, bids, fids, wl, wrl)
    rs = np.random.RandomState(seed + 7919)
    per_q = []
    for b in range(B):
        sel = np.nonzero((bids == b) & (rels != loop))[0]
        per_q.append((heads[sel] - b * N, rels[sel], tails[sel] - b * N))
    max_tuples = max([len(t[0]) for t in per_q] + [0])
    max_fact = 2 * max_tuples + N
    kb_fact_rel = np.full((B, max_fact), num_relation, dtype=np.int64)
    lists = [[] for _ in range(6)]
    for b, (h, r, t) in enumerate(per_q):
        T = len(h)
        if use_inverse_relation:
            kb_fact_rel[b, :T] = r + half
            e_head = np.stack([h, t], 1).reshape(-1)
            e_tail = np.stack([t, h], 1).reshape(-1)
            slots = np.arange(2 * T, dtype=np.int64)
        else:
            kb_fact_rel[b, :T] = r
            e_head, e_tail, slots = h, t, np.arange(T, dtype=np.int64)
        n = len(slots)
        keep = rs.permutation(n)[: int(np.floor(n * (1 - fact_dropout)))]
        for lst, arr in zip(lists, (np.full(len(keep), b, dtype=np.int64), slots[keep], e_head[keep],
                                    np.full(len(keep), b, dtype=np.int64), e_tail[keep], slots[keep])):
            lst.append(arr.astype(np.int64))
    cat = [np.concatenate(x) if x else np.zeros(0, dtype=np.int64) for x in lists]
    ones = np.ones(len(cat[0]))
    graft = ((cat[0], cat[1], cat[2], ones), (cat[3], cat[4], cat[5], ones.copy()))
    out = (local_entity, query_entities, kb, graft, q_input, kb_fact_rel, seed_dist, None, answer_dist)
    if test:
        out = out + (base[7],)
    return out


# Named workloads from BASELINE.json:configs / SURVEY.md §8
CONFIGS = {
    "cfg1": dict(B=1, N=2000, E=6000, D=200, T=3, K=3, I=2),
    "cfg2": dict(B=64, N=2000, E=6000, D=200, T=3, K=3, I=2),
    "cfg3": dict(B=256, N=10_000, E=40_000, D=200, T=2, K=4, I=3),
    "cfg4": dict(B=1024, N=2000, E=6000, D=200, T=3, K=3, I=2),
    "cfg5": dict(B=1, N=100_000, E=1_000_000, D=400, T=3, K=3, I=2),
    # the shape of the published checkpoints (gnn/README.md:19, gnn/scripts/rearev_cwq.sh:14): entity_dim 50
    "d50": dict(B=64, N=2000, E=6000, D=50, T=3, K=3, I=2),
}


def seeded_state_dict(shapes, seed=0, sharpen=None):
    """Deterministic weights for a ``{name: shape}`` map, independent of module construction order and of torch's RNG:
    every tensor comes from its own ``numpy.random.RandomState(crc32(name) + seed)``.  Embeddings ~ N(0, 1) (torch's
    default), matrices ~ U(+-1/sqrt(fan_in)), vectors ~ U(+-0.05).  Lets the hot-shape goldens (tests/golden/
    make_golden_hot.py, generated from the unmodified reference) store OUTPUTS only: the test rebuilds the same
    weights.  ``sharpen = (e2e, rel, score)`` scales those weight groups like tests/golden/make_golden.py:sharpen."""
    import zlib
    out = {}
    for name in sorted(shapes):
        shape = tuple(shapes[name])
        rs = np.random.RandomState((zlib.crc32(name.encode()) + seed) % (2 ** 31))
        if "embedding" in name:
            w = rs.standard_normal(shape)
        elif len(shape) >= 2:
            w = rs.uniform(-1.0, 1.0, shape) / np.sqrt(shape[-1])
        else:
            w = rs.uniform(-0.05, 0.05, shape)
        if sharpen is not None:
            e2e, rel, score = sharpen
            if "e2e_linear" in name and name.endswith("weight"):
                w = w * e2e
            if "rel_linear" in name and name.endswith("weight"):
                w = w * rel
            if name.endswith("reasoning.score_func.weight"):
                w = w * score
        out[name] = w.astype(np.float32)
    return out
