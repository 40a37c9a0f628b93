"""Host-side drop-in for the batch assembly of the reference loader (SURVEY.md 8a row 1).

``build_fact_mat`` replaces ``BasicDataLoader._build_fact_mat`` (gnn/dataset_load.py:473-527): same arguments, same
seven return values, same consumption of ``np.random`` (one ``permutation`` per question, in order), therefore
bit-identical arrays for the same RNG state -- but assembled with one concatenate and two counting passes instead of
four ``np.append`` per question (quadratic in the batch) and two Python ``Counter`` passes over all facts.  At the
WebQSP-shape batch of BASELINE cfg2 (64 questions, 512 000 facts) the reference takes ~1 s per batch on one host core;
the device step this repo builds takes 2.8 ms, so without this the loader IS the end-to-end time.

    from gnn_rag_b200 import loader
    loader.install(SingleDataLoader)           # monkeypatches _build_fact_mat; get_batch (:599-629) is untouched

``weights``: ``"lists"`` (default) returns ``weight_list`` / ``weight_rel_list`` as Python lists of float exactly
like the reference; ``"arrays"`` returns float64 numpy arrays (what ``batching.stage_batch`` wants, no 512 000-item
list building); ``"none"`` skips the two counting passes and returns ``None`` for both (valid whenever the model
runs with ``normalized_gnn = norm_rel = False``, the reference's defaults).
``index_dtype``: ``np.int64`` (reference) or ``np.int32`` (halves the H2D bytes of the fact arrays; ``gr_csr_build``
takes either).
``shuffle=False`` (serving): keep every question's facts in stored order instead of drawing a permutation -- the
forward is invariant to the fact order up to fp32 summation order (SURVEY.md 7, hard part 1), the RNG is not touched,
and with :func:`preconvert` (SURVEY.md 8f row 3: the per-question arrays flattened once at load time) the batch
assembly is an offset concat.

GraftNet's loader (``GraftSingleDataLoader``, gnn/dataset_load_graft.py) additionally calls
``_build_fact_mat_maxfacts`` (:70-102) in every ``get_batch``: per question it re-parses the subgraph tuples
(``create_kb_adj_mats_facts``, :27-68, a Python loop with dictionary lookups) and grows eight arrays by ``np.append``.
:func:`build_fact_mat_maxfacts` is its drop-in -- same return values and dtypes, the same one ``permutation`` per
question in order (so it interleaves with either ``_build_fact_mat`` under one seed), one concatenate per array, and
the per-question triple taken from the loader's own ``create_kb_adj_mats_facts`` once per sample and cached:

    loader.install_graft(GraftSingleDataLoader)    # monkeypatches _build_fact_mat_maxfacts

Pure numpy on the host; nothing here touches the GPU.
"""
import numpy as np


def _per_question(self, sample_id):
    if getattr(self, "data_eff", False):
        return self.create_kb_adj_mats(sample_id)          # dataset_load.py:484-485
    return self.kb_adj_mats[sample_id]


def preconvert(self):
    """Flatten ``kb_adj_mats`` once (load time): int64 [sum facts] arrays + offsets, kept on the loader as
    ``_gr_flat``.  Used by ``build_fact_mat(..., shuffle=False)``."""
    n = len(self.kb_adj_mats)
    cnt = np.fromiter((len(self.kb_adj_mats[i][0]) for i in range(n)), dtype=np.int64, count=n)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(cnt, out=off[1:])

    def flat(k):
        parts = [np.asarray(self.kb_adj_mats[i][k], dtype=np.int64) for i in range(n)]
        return np.concatenate(parts) if parts else np.zeros(0, dtype=np.int64)

    ents = np.fromiter((len(m) for m in self.global2local_entity_maps), dtype=np.int64, count=n)
    self._gr_flat = dict(heads=flat(0), rels=flat(1), tails=flat(2), off=off, ents=ents)
    return self._gr_flat


def _assemble_unshuffled(self, sample_ids, index_dtype):
    """Offset concat of the pre-flattened per-question arrays (+ self loops), stored fact order."""
    fl = getattr(self, "_gr_flat", None) or preconvert(self)
    N, self_rel = self.max_local_entity, self.num_kb_relation - 1
    ids = np.asarray(sample_ids, dtype=np.int64)
    nf = fl["off"][ids + 1] - fl["off"][ids]
    ne = fl["ents"][ids] if self.use_self_loop else np.zeros(len(ids), dtype=np.int64)
    tot = nf + ne
    pos = np.zeros(len(ids) + 1, dtype=np.int64)
    np.cumsum(tot, out=pos[1:])
    F = int(pos[-1])
    heads, rels, tails = (np.empty(F, dtype=index_dtype) for _ in range(3))
    for i, sid in enumerate(ids.tolist()):
        a, b = int(fl["off"][sid]), int(fl["off"][sid + 1])
        p, bias = int(pos[i]), i * N
        k = b - a
        np.add(fl["heads"][a:b], bias, out=heads[p:p + k], casting="unsafe")
        np.add(fl["tails"][a:b], bias, out=tails[p:p + k], casting="unsafe")
        rels[p:p + k] = fl["rels"][a:b]
        m = int(ne[i])
        if m:
            ent = np.arange(bias, bias + m, dtype=index_dtype)
            heads[p + k:p + k + m] = ent
            tails[p + k:p + k + m] = ent
            rels[p + k:p + k + m] = self_rel
    bids = np.repeat(np.arange(len(ids), dtype=index_dtype), tot)
    return heads, rels, tails, bids


def build_fact_mat(self, sample_ids, fact_dropout, weights="lists", index_dtype=np.int64, shuffle=True):
    """-> (batch_heads, batch_rels, batch_tails, batch_ids, fact_ids, weight_list, weight_rel_list),
    dataset_load.py:473-527.  Global node row of question i = i * max_local_entity + local id (:483)."""
    if not shuffle:
        if fact_dropout != 0 or getattr(self, "data_eff", False):
            raise ValueError("shuffle=False needs fact_dropout == 0 and stored kb_adj_mats (data_eff off)")
        # the counting passes want int64 keys; without them assemble straight into the requested dtype
        h, r, t, b = _assemble_unshuffled(self, sample_ids, index_dtype if weights == "none" else np.int64)
        return _finish(h, r, t, b, weights, index_dtype)
    N = self.max_local_entity
    use_self_loop = self.use_self_loop
    self_rel = self.num_kb_relation - 1
    heads, rels, tails, bids = [], [], [], []
    for i, sample_id in enumerate(sample_ids):
        bias = i * N
        head_list, rel_list, tail_list = _per_question(self, sample_id)
        num_fact = len(head_list)
        num_keep = int(np.floor(num_fact * (1 - fact_dropout)))
        mask_index = np.random.permutation(num_fact)[:num_keep]          # same RNG stream as the reference (:489)
        heads.append(np.asarray(head_list)[mask_index] + bias)
        tails.append(np.asarray(tail_list)[mask_index] + bias)
        rels.append(np.asarray(rel_list)[mask_index])
        n_i = len(mask_index)
        if use_self_loop:                                                # :498-505
            num_ent_now = len(self.global2local_entity_maps[sample_id])
            ent = np.arange(num_ent_now, dtype=np.int64) + bias
            heads.append(ent)
            tails.append(ent)
            rels.append(np.full(num_ent_now, self_rel, dtype=np.int64))
            n_i += num_ent_now
        bids.append(np.full(n_i, i, dtype=np.int64))

    def cat(parts):
        if not parts:
            return np.array([], dtype=np.int64)
        return np.concatenate(parts).astype(np.int64, copy=False)

    return _finish(cat(heads), cat(rels), cat(tails), cat(bids), weights, index_dtype)


def _finish(batch_heads, batch_rels, batch_tails, batch_ids, weights, index_dtype):
    F = batch_heads.shape[0]
    fact_ids = np.arange(F, dtype=np.int64)

    weight_list = weight_rel_list = None
    if weights != "none":
        if F:
            # 1 / (#facts with this head)                      == [1.0 / Counter(batch_heads)[h] ...]   (:507-510)
            head_count = np.bincount(batch_heads)
            w = 1.0 / head_count[batch_heads]
            # 1 / (#facts with this (head, relation) pair)     == Counter(zip(heads, rels))             (:513-516)
            key = batch_heads * (int(batch_rels.max()) + 1) + batch_rels
            _, inverse, counts = np.unique(key, return_inverse=True, return_counts=True)
            wr = 1.0 / counts[inverse.reshape(-1)]
        else:
            w = wr = np.zeros(0, dtype=np.float64)
        if weights == "lists":
            weight_list, weight_rel_list = w.tolist(), wr.tolist()
        elif weights == "arrays":
            weight_list, weight_rel_list = w, wr
        else:
            raise ValueError("weights must be 'lists', 'arrays' or 'none'")
    if np.dtype(index_dtype) != np.dtype(np.int64):
        batch_heads, batch_rels, batch_tails, batch_ids, fact_ids = (
            a.astype(index_dtype) for a in (batch_heads, batch_rels, batch_tails, batch_ids, fact_ids))
    return batch_heads, batch_rels, batch_tails, batch_ids, fact_ids, weight_list, weight_rel_list


def install(loader, weights="lists", index_dtype=np.int64, shuffle=True):
    """Monkeypatch ``_build_fact_mat`` on a reference loader class (or a single instance).  ``get_batch`` and every
    other method keep working unchanged.  Returns the original function so it can be restored."""
    import types

    def patched(self, sample_ids, fact_dropout):
        return build_fact_mat(self, sample_ids, fact_dropout, weights=weights, index_dtype=index_dtype,
                              shuffle=shuffle)

    if isinstance(loader, type):
        orig = loader._build_fact_mat
        loader._build_fact_mat = patched
    else:
        orig = loader._build_fact_mat
        loader._build_fact_mat = types.MethodType(patched, loader)
    return orig


def _graft_per_question(self, sample_id):
    """``create_kb_adj_mats_facts(sample_id)`` of the loader itself, once per sample: the result is a pure function of
    the loaded data, so it is cached on the instance (``_gr_graft``)."""
    cache = self.__dict__.get("_gr_graft")
    if cache is None:
        cache = self._gr_graft = {}
    ent = cache.get(sample_id)
    if ent is None:
        ((m00, m01, v0), (m10, m11, v1)), kb_fact_rel = self.create_kb_adj_mats_facts(sample_id)
        assert len(v0) == len(v1)
        ent = cache[sample_id] = (m00, m01, v0, m10, m11, v1, kb_fact_rel)
    return ent


def build_fact_mat_maxfacts(self, sample_ids, fact_dropout):
    """-> ((mats0_batch, mats0_0, mats0_1, vals0), (mats1_batch, mats1_0, mats1_1, vals1)), kb_fact_rels,
    gnn/dataset_load_graft.py:70-102, bit for bit (dtypes included) for the same ``np.random`` state."""
    kb_fact_rels = np.full((len(sample_ids), self.max_facts), self.num_kb_relation, dtype=int)
    # the reference grows each array from these empties by np.append: starting every concatenate from them gives the
    # same dtype promotion
    parts = [[np.array([], dtype=int)] for _ in range(3)] + [[np.array([], dtype=float)]] + \
        [[np.array([], dtype=int)] for _ in range(3)] + [[np.array([], dtype=float)]]
    for i, sample_id in enumerate(sample_ids):
        m00, m01, v0, m10, m11, v1, kb_fact_rel = _graft_per_question(self, sample_id)
        kb_fact_rels[i] = kb_fact_rel
        num_fact = len(v0)
        num_keep_fact = int(np.floor(num_fact * (1 - fact_dropout)))
        mask_index = np.random.permutation(num_fact)[:num_keep_fact]      # same RNG stream as the reference (:90)
        bcol = np.full(len(mask_index), i, dtype=int)
        for lst, arr in zip(parts, (bcol, m00[mask_index], m01[mask_index], v0[mask_index],
                                    bcol, m10[mask_index], m11[mask_index], v1[mask_index])):
            lst.append(np.ravel(arr))
    out = [np.concatenate(lst) for lst in parts]
    return (tuple(out[:4]), tuple(out[4:])), kb_fact_rels


def install_graft(loader):
    """Monkeypatch ``_build_fact_mat_maxfacts`` on a reference graft loader class (or a single instance) with
    :func:`build_fact_mat_maxfacts`.  Returns the original function so it can be restored."""
    import types

    orig = loader._build_fact_mat_maxfacts
    if isinstance(loader, type):
        loader._build_fact_mat_maxfacts = build_fact_mat_maxfacts
    else:
        loader._build_fact_mat_maxfacts = types.MethodType(build_fact_mat_maxfacts, loader)
    return orig
