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

Everything above is pure numpy on the host.  :class:`DeviceSplit` goes one step further: it uploads a whole split
once and assembles each batch on the GPU from its question ids (csrc/split.cu), so per batch only B ids cross PCIe:

    split = loader.DeviceSplit(valid_data, torch.device("cuda"))
    evaluator.evaluate(split, test_batch_size=20)          # get_batch returns the loader's tuple, built from CUDA tensors

With ``shuffle=True`` it also draws the reference's fact dropout on the device, so ``train_epoch`` with
``fact_drop > 0`` trains from a resident split:

    train = loader.DeviceSplit(train_data, torch.device("cuda"), shuffle=True)
    batch = train.get_batch(iteration, batch_size, fact_dropout=args['fact_drop'])
"""
import time

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


_INT32_MAX = 2 ** 31 - 1


def same_device(a, b):
    """True when torch devices ``a`` and ``b`` are the same CUDA device (``cuda`` is the current one)."""
    import torch

    def index(d):
        return d.index if d.index is not None else torch.cuda.current_device()
    return a.type == b.type == "cuda" and index(a) == index(b)


def kept_counts(n, fact_dropout):
    """Facts kept per question under fact dropout: ``int(np.floor(n * (1 - fact_dropout)))`` of the reference
    (gnn/dataset_load.py:488, gnn/dataset_load_graft.py:88) for every count in ``n``, in float64 as there.  int64."""
    return np.floor(np.asarray(n, dtype=np.int64) * (1 - float(fact_dropout))).astype(np.int64)


def pack_answers(answer_lists):
    """Per-question answer lists (the loader's ``answer_lists``: global entity ids, possibly outside the subgraph and
    repeated) -> ``(off, ids)``: int64 [len(answer_lists) + 1] offsets and int64 ids, each question's run sorted
    ascending with repeats kept, so membership is a binary search and the run's length is ``len(answers)``.  ``ids``
    keeps one element when there are no answers at all.  Raises ``ValueError`` naming the question when an answer is
    not an integer or outside int64."""
    import numbers
    off = np.zeros(len(answer_lists) + 1, dtype=np.int64)
    runs = []
    for q in range(len(answer_lists)):
        answers = list(answer_lists[q])
        for a in answers:
            if not isinstance(a, numbers.Integral) or not -2 ** 63 <= int(a) < 2 ** 63:
                raise ValueError("DeviceSplit: question %d has an answer that is not an int64 entity id: %r" % (q, a))
        runs.append(np.sort(np.array([int(a) for a in answers], dtype=np.int64)))
        off[q + 1] = off[q] + len(answers)
    ids = np.concatenate(runs) if off[-1] else np.zeros(1, dtype=np.int64)       # a null pointer is refused
    return off, ids


def candidate_capacity(candidate_entities, pad_id):
    """Candidates an evaluation over a split can retrieve, at most: the entities of its questions'
    ``candidate_entities`` rows that are not the pad ``pad_id`` (the ranking drops pads and seeds)."""
    return int(np.count_nonzero(np.asarray(candidate_entities) != pad_id))


def seed_counts(query_entities):
    """Seeds of each question: its local entities whose ``query_entities`` entry is nonzero in fp32, the table the
    split uploads (the sources of ``evaluate.path_node_sets``).  int64 [num_q]."""
    qe = np.asarray(query_entities, dtype=np.float32)
    return np.count_nonzero(qe != 0, axis=1).astype(np.int64)


class DeviceSplit:
    """A split resident in device memory: ``get_batch`` assembles each batch on the GPU from its question ids.

    ``DeviceSplit(data_loader, device, weights="arrays", index_dtype=torch.int32)`` wraps a ``SingleDataLoader`` or a
    ``GraftSingleDataLoader`` (recognised by its ``create_kb_adj_mats_facts``) and uploads, once: the per-question
    fact segments (int32 local ids with int64 offsets), the entity counts, the [num_q, N] tables
    (``candidate_entities``, ``query_entities``, ``seed_distribution``, ``answer_dists``) and ``query_texts``; for
    GraftNet also both graft lists per question and the stored prefix of every ``kb_fact_rels`` row.

    ``get_batch(iteration, batch_size, fact_dropout, q_type=None, test=False)`` has the loader's signature and returns
    its tuple layout (7-tuple, or GraftNet's 9-tuple; ``answer_lists`` appended with ``test=True``, still the loader's
    host object array) built from CUDA tensors: ``local_entity`` int64 [B, N], ``query_entities`` / ``seed_dist`` /
    ``answer_dist`` fp32 [B, N], ``q_input`` int64 [B, Q], ``kb_adj_mat`` with its five index arrays in
    ``index_dtype`` and fp32 weights (``None`` with ``weights="none"``); GraftNet's graft lists in ``index_dtype``
    with fp32 1.0 values and ``kb_fact_rel`` int64 [B, max_facts].  The facts are in stored order with the self-loops
    appended per question, exactly :func:`build_fact_mat` with ``shuffle=False`` (and the graft lists
    :func:`build_fact_mat_maxfacts` under the identity permutation); the weights are bit-equal to fp32 of the host's
    float64 ones.  The question ids come from ``data_loader.batches`` as in the loader, so ``reset_batches`` works,
    and ``sample_ids`` is set on the loader.  The fact count of a batch comes from a host copy of the per-question
    counts, so assembling a batch never waits on the device.

    Refused (``ValueError``): fact dropout without ``shuffle`` (with it, one outside [0, 1]), ``data_eff``, a
    ``q_type`` other than ``"seq"``, and a batch whose facts would overflow int32 indices.  ``reset_batches``, ``num_data``, ``max_local_entity`` and ``get_quest`` pass
    through to the loader, so ``Evaluator.evaluate(split)`` and a ``train_epoch``-shaped loop run unchanged.

    ``shuffle=True`` samples facts as the reference's training batches do (:func:`build_fact_mat` with
    ``shuffle=True``, :func:`build_fact_mat_maxfacts`): ``get_batch(it, B, p)`` takes any ``p`` in [0, 1], and each
    question keeps :func:`kept_counts` of its facts, the first of a uniform random permutation, in permutation order,
    with its self-loops after them in entity order.  GraftNet's graft lists keep the same number of their entries
    from a second, independent permutation; ``kb_fact_rel`` rows stay as stored.  The permutations are drawn on the
    device (csrc/split.cu, gr_split_fact_order) from one seed per call taken from torch's CUDA generator, so
    ``torch.manual_seed`` makes a run reproducible and no call waits on the device.  ``np.random`` is not touched:
    the sampled facts differ from the host loader's for the same numpy seed.  The last batch's orders are kept in
    ``last_order``: ``kb`` / ``graft`` device int32 arrays of stored indices per question, in batch order, and
    ``kb_offsets`` / ``graft_offsets`` numpy int64 [B+1] where each question's run starts."""

    def __init__(self, data_loader, device, weights="arrays", index_dtype=None, shuffle=False):
        import torch
        index_dtype = torch.int32 if index_dtype is None else index_dtype
        if weights not in ("arrays", "none"):
            raise ValueError("DeviceSplit: weights must be 'arrays' or 'none', got %r" % (weights,))
        if index_dtype not in (torch.int32, torch.int64):
            raise ValueError("DeviceSplit: index_dtype must be torch.int32 or torch.int64, got %s" % (index_dtype,))
        if getattr(data_loader, "data_eff", False):
            raise ValueError("DeviceSplit: data_eff loaders build their facts per batch; the split needs stored "
                             "kb_adj_mats (data_eff off)")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise ValueError("DeviceSplit: the split lives on a CUDA device, got %s" % dev)
        self.loader, self.device, self.weights, self.index_dtype = data_loader, dev, weights, index_dtype
        self.shuffle, self.last_order = bool(shuffle), None
        self.graft = hasattr(data_loader, "create_kb_adj_mats_facts")
        L = data_loader
        N = int(L.max_local_entity)
        self.N, self.self_rel, self.use_self_loop = N, int(L.num_kb_relation) - 1, bool(L.use_self_loop)
        had_flat = getattr(L, "_gr_flat", None) is not None
        fl = L._gr_flat if had_flat else preconvert(L)
        num_q = len(fl["ents"])
        self.num_q = num_q
        for name in ("heads", "tails"):
            a = fl[name]
            if a.size and (a.min() < 0 or a.max() >= N):
                raise ValueError("DeviceSplit: kb_adj_mats %s hold local ids outside [0, %d)" % (name, N))
        if fl["rels"].size and (fl["rels"].min() < 0 or fl["rels"].max() > _INT32_MAX):
            raise ValueError("DeviceSplit: kb_adj_mats hold relation ids outside [0, 2^31)")
        if fl["ents"].size and fl["ents"].max() > N:
            raise ValueError("DeviceSplit: a question has more entities than max_local_entity = %d" % N)
        nf = np.diff(fl["off"])
        # host copies per question: stored facts, self-loops, and both together
        self._stored = nf
        self._ents = fl["ents"] if self.use_self_loop else np.zeros_like(nf)
        self._count = nf + self._ents

        t0 = time.perf_counter()
        self._res = {}
        self._put("q_off", fl["off"], np.int64)
        for name in ("heads", "rels", "tails"):
            self._put("q_" + name, fl[name], np.int32)
        self._put("q_ents", fl["ents"], np.int32)
        self._put("local_entity", L.candidate_entities, np.int64)
        for name, src in (("query_entities", L.query_entities), ("seed_dist", L.seed_distribution),
                          ("answer_dist", L.answer_dists)):
            self._put(name, src, np.float32)
        self._put("q_input", L.query_texts, np.int64)
        if self.graft:
            self._upload_graft(L, num_q)
        torch.cuda.synchronize(dev)
        self.build_seconds = time.perf_counter() - t0        # the upload; preconvert and the graft parse come before
        if not had_flat:
            del L._gr_flat                                    # flattened here for the upload only
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self._answers = None                                  # answer_table(), uploaded by the first evaluation
        self._seed_counts = None                              # seed_counts(), counted by the first evaluation with paths

    def _put(self, name, a, dtype):
        import torch
        a = np.ascontiguousarray(np.asarray(a).astype(dtype, copy=False))
        if a.size == 0:                 # a null pointer is refused: keep one element behind an empty array
            a = np.zeros(1, dtype=dtype)
        self._res[name] = torch.from_numpy(a).to(self.device)

    def _upload_graft(self, L, num_q):
        parts = [[] for _ in range(4)]
        cnt = np.zeros(num_q, dtype=np.int64)
        for q in range(num_q):
            ((m00, m01, v0), (m10, m11, v1)), _rel = L.create_kb_adj_mats_facts(q)
            if len(v0) != len(v1):
                raise ValueError("DeviceSplit: question %d has graft lists of different lengths" % q)
            if np.any(np.asarray(v0) != 1.0) or np.any(np.asarray(v1) != 1.0):
                raise ValueError("DeviceSplit: question %d has graft values other than 1.0" % q)
            cnt[q] = len(v0)
            for lst, a in zip(parts, (m00, m01, m10, m11)):
                lst.append(np.asarray(a, dtype=np.int64).ravel())
        flat = [np.concatenate(p) if p else np.zeros(0, dtype=np.int64) for p in parts]
        for a in flat:
            if a.size and (a.min() < 0 or a.max() > _INT32_MAX):
                raise ValueError("DeviceSplit: graft lists hold ids outside [0, 2^31)")
        off = np.zeros(num_q + 1, dtype=np.int64)
        np.cumsum(cnt, out=off[1:])
        self._graft_count = cnt
        self._put("g_off", off, np.int64)
        for name, a in zip(("g_e2f_f", "g_e2f_e", "g_f2e_e", "g_f2e_f"), flat):
            self._put(name, a, np.int32)
        # kb_fact_rels rows (what get_batch reads): keep each row up to its last entry that is not the pad relation
        kfr = np.asarray(L.kb_fact_rels)
        self.max_facts, self.rel_pad = int(kfr.shape[1]), int(L.num_kb_relation)
        live = kfr != self.rel_pad
        rlen = np.where(live.any(axis=1), kfr.shape[1] - np.argmax(live[:, ::-1], axis=1), 0).astype(np.int64)
        if kfr.size and (kfr.min() < 0 or kfr.max() > _INT32_MAX):
            raise ValueError("DeviceSplit: kb_fact_rels hold relation ids outside [0, 2^31)")
        roff = np.zeros(num_q + 1, dtype=np.int64)
        np.cumsum(rlen, out=roff[1:])
        vals = np.concatenate([kfr[q, :rlen[q]] for q in range(num_q)]) if num_q else np.zeros(0, dtype=np.int64)
        self._put("r_off", roff, np.int64)
        self._put("r_vals", vals, np.int32)

    # -- what Evaluator.evaluate and train_epoch read from their loader ------------------------------------------------
    @property
    def num_data(self):
        return self.loader.num_data

    @property
    def max_local_entity(self):
        return self.loader.max_local_entity

    def reset_batches(self, is_sequential=True):
        return self.loader.reset_batches(is_sequential=is_sequential)

    def get_quest(self, training=False):
        return self.loader.get_quest(training)

    def answer_table(self):
        """:func:`pack_answers` of the loader's ``answer_lists`` on the device, uploaded at the first call and kept:
        ``(a_off, a_ids)`` int64 tensors."""
        if self._answers is None:
            import torch
            self._answers = tuple(torch.from_numpy(a).to(self.device) for a in pack_answers(self.loader.answer_lists))
        return self._answers

    def seed_counts(self):
        """:func:`seed_counts` of the loader's ``query_entities``, counted at the first call and kept: int64 [num_q]."""
        if self._seed_counts is None:
            self._seed_counts = seed_counts(self.loader.query_entities)
        return self._seed_counts

    def max_seeds(self):
        """The largest seed count of any question of the split (0 without questions): the source capacity of the
        shortest-path node sets of an evaluation (``GraphedStep.start_eval(..., path_targets=T)``)."""
        c = self.seed_counts()
        return int(c.max()) if c.size else 0

    @property
    def resident_bytes(self):
        """Device bytes the split holds."""
        return int(sum(t.numel() * t.element_size() for t in self._res.values()))

    def check(self):
        """Raise when the last batch's assembly flagged an id out of range or an overflow (reads the device)."""
        self.raise_status(int(self.status.item()))

    @staticmethod
    def raise_status(s):
        """Raise for a nonzero assembly status word ``s`` (an int read from the device)."""
        if s:
            raise RuntimeError("DeviceSplit: batch assembly status %d (1: question id out of range, 2: more facts than "
                               "the batch's capacity)" % s)

    # -- one batch ---------------------------------------------------------------------------------------------------
    def assemble(self, ids, kept, seed, F, K, n_total, rows=None, out=None, nfacts=None):
        """The device part of :meth:`get_batch` for the kb side of B > 0 questions: the row gathers, the fact order
        (with ``shuffle``), the fact assembly and the fact weights (``weights="arrays"``).

        ``ids`` / ``kept`` int64 [B] and ``seed`` int64 [1] on the device (``kept`` and ``seed`` only read with
        ``shuffle``); ``rows``: the ids the row tables are gathered at (default ``ids``).  ``F``: the capacity of the
        fact arrays, ``K`` of the order, ``n_total`` >= the stored facts of the B questions (host ints).  ``out``: an
        object whose ``local_entity``, ``query_entities``, ``seed_dist``, ``answer_dist``, ``q_input``, ``heads``,
        ``rels``, ``tails``, ``weight_list`` and ``weight_rel_list`` are written in place (a weight that is None is not
        computed), with ``nfacts`` (int32[1] on the device) the live count of the F slots; without it new tensors of F
        facts.  Launch shapes and sizes come from these arguments alone, so a CUDA graph can capture the call.
        -> (le, qe, sd, ad, qi), (heads, rels, tails, batch_ids, fact_ids, w, wr), order (None without shuffle), status
        int32[1]."""
        import torch
        from . import ops
        r, N, idt = self._res, self.N, self.index_dtype
        B = ids.numel()
        rows = ids if rows is None else rows
        names = ("local_entity", "query_entities", "seed_dist", "answer_dist", "q_input")
        gathered = tuple(torch.index_select(r[n], 0, rows, out=None if out is None else getattr(out, n)) for n in names)
        fo = None if out is None else (out.heads, out.rels, out.tails, None, None)
        order = ost = None
        if self.shuffle:
            order, ost = ops.split_fact_order(r["q_off"], ids, kept, seed, 0, n_total, K)
        *kb, status = ops.split_assemble(r["q_off"], r["q_heads"], r["q_rels"], r["q_tails"], r["q_ents"], ids, N, F,
                                         self.self_rel, self.use_self_loop, idt, out=fo,
                                         kept=kept if self.shuffle else None, order=order)
        if ost is not None:
            status = status | ost
        w = wr = None
        if self.weights == "arrays":
            if out is not None:
                w, wr = out.weight_list, out.weight_rel_list
                if w is not None or wr is not None:
                    ops.fact_weights_live(kb[0], kb[1], nfacts, max(B * N, 1), w, wr)
            elif F:
                w, wr, _st = ops.fact_weights(kb[0], kb[1], max(B * N, 1))
            else:
                w, wr = (torch.empty(0, dtype=torch.float32, device=self.device) for _ in range(2))
        return gathered, (*kb, w, wr), order, status

    def assemble_graft(self, ids, kept_g, seed, G, n_total, out=None):
        """The device part of :meth:`get_batch` for GraftNet's graft side of B > 0 questions: the graft order (with
        ``shuffle``, from the same ``seed`` as the kb facts' order, as a second permutation) and the assembly of both
        graft lists and of ``kb_fact_rel``.

        ``ids`` / ``kept_g`` int64 [B] and ``seed`` int64 [1] on the device (``kept_g``, the graft entries each
        question keeps, and ``seed`` only read with ``shuffle``).  ``G``: the length of the lists and of the order,
        ``n_total`` >= the stored graft entries of the B questions (host ints).  ``out``: ``((e2f_b, e2f_f, e2f_e,
        e2f_v), (f2e_b, f2e_e, f2e_f, f2e_v), kb_fact_rel)`` written in place (G their capacity, the index dtype
        theirs: the live entries at the front, a batch past G cut there and flagged); without it new tensors of G
        entries in ``index_dtype``.  Launch shapes and sizes come from these arguments alone, so a CUDA graph can
        capture the call.  -> (graft lists, kb_fact_rel, order (None without shuffle), status int32[1])."""
        from . import ops
        r = self._res
        lists = (r["g_off"], r["g_e2f_f"], r["g_e2f_e"], r["g_f2e_e"], r["g_f2e_f"], r["r_off"], r["r_vals"])
        idt = None if out is not None else self.index_dtype
        order = ost = None
        if self.shuffle:
            order, ost = ops.split_fact_order(r["g_off"], ids, kept_g, seed, 1, n_total, G)
        graft, kfr, status = ops.split_assemble_graft(*lists, ids, self.max_facts, self.rel_pad, G, idt, out=out,
                                                      kept=kept_g if self.shuffle else None, order=order)
        if ost is not None:
            status = status | ost
        return graft, kfr, order, status

    def get_batch(self, iteration, batch_size, fact_dropout, q_type=None, test=False, seed=None):
        """The loader's ``get_batch`` from the resident split (see the class docstring).  ``seed``: with ``shuffle``,
        the fact-order seed to use (int64 [1] on the device, e.g. a seed an epoch recorded) instead of one drawn from
        torch's CUDA generator."""
        import torch
        L, r, dev = self.loader, self._res, self.device
        if not self.shuffle and fact_dropout != 0:
            raise ValueError("DeviceSplit.get_batch: fact_dropout must be 0 (facts come in stored order), got %r"
                             % (fact_dropout,))
        if self.shuffle and not 0 <= fact_dropout <= 1:
            raise ValueError("DeviceSplit.get_batch: fact_dropout must be in [0, 1], got %r" % (fact_dropout,))
        if q_type is None:
            q_type = getattr(L, "q_type", "seq")
        if q_type != "seq":
            raise ValueError("DeviceSplit.get_batch: q_type must be 'seq', got %r" % (q_type,))
        start = batch_size * iteration
        end = min(batch_size * (iteration + 1), L.num_data)
        sample_ids = L.batches[start:end]
        L.sample_ids = sample_ids                                  # get_quest / deal_q_type read it
        ids = np.asarray(sample_ids, dtype=np.int64).reshape(-1)
        if ids.size and (ids.min() < 0 or ids.max() >= self.num_q):
            raise ValueError("DeviceSplit.get_batch: question ids outside [0, %d)" % self.num_q)
        B, N = len(ids), self.N
        if self.shuffle:
            kept = kept_counts(self._stored[ids], fact_dropout)
            F = int(kept.sum() + self._ents[ids].sum())
        else:
            F = int(self._count[ids].sum())
        idt = self.index_dtype
        if idt == torch.int32 and (B * N > _INT32_MAX or F > _INT32_MAX):
            raise ValueError("DeviceSplit.get_batch: the batch overflows int32 indices (B*N = %d, %d facts); use "
                             "index_dtype=torch.int64" % (B * N, F))
        kept_dev = None
        if self.shuffle:
            kept_g = kept_counts(self._graft_count[ids], fact_dropout) if self.graft else kept[:0]
            # one upload: the ids, then the kept counts of the kb facts and of the graft lists
            up = torch.from_numpy(np.concatenate([ids, kept, kept_g])).to(dev, non_blocking=True)
            ids_dev, kept_dev, kept_g_dev = up[:B], up[B:2 * B], up[2 * B:]
            if seed is None:
                seed = torch.randint(0, 2 ** 62, (1,), device=dev)
            elif not (isinstance(seed, torch.Tensor) and same_device(seed.device, dev) and seed.dtype == torch.int64
                      and seed.numel() == 1):
                raise ValueError("DeviceSplit.get_batch: seed must be one int64 on %s" % dev)
            seed = seed.reshape(1)
        else:
            ids_dev = torch.from_numpy(ids).to(dev, non_blocking=True)
        if B:
            K = int(kept.sum()) if self.shuffle else 0
            n_total = int(self._stored[ids].sum()) if self.shuffle else 0
            (le, qe, sd, ad, qi), kb, order, self.status = self.assemble(ids_dev, kept_dev, seed, F, K, n_total)
            if self.shuffle:
                self.last_order = dict(kb=order, kb_offsets=np.concatenate([[0], np.cumsum(kept)]))
        else:
            le, qe, sd, ad, qi = (torch.index_select(r[n], 0, ids_dev) for n in (
                "local_entity", "query_entities", "seed_dist", "answer_dist", "q_input"))
            kb = tuple(torch.empty(0, dtype=idt, device=dev) for _ in range(5))
            kb += (None, None) if self.weights != "arrays" else \
                tuple(torch.empty(0, dtype=torch.float32, device=dev) for _ in range(2))
        tail = (L.answer_lists[sample_ids],) if test else ()
        if not self.graft:
            return (le, qe, kb, qi, sd, None, ad) + tail
        G = int(kept_g.sum()) if self.shuffle else int(self._graft_count[ids].sum())
        if idt == torch.int32 and G > _INT32_MAX:
            raise ValueError("DeviceSplit.get_batch: the graft lists overflow int32 indices (%d entries)" % G)
        if B:
            graft, kfr, gorder, gst = self.assemble_graft(ids_dev, kept_g_dev if self.shuffle else None, seed, G,
                                                          int(self._graft_count[ids].sum()))
            self.status = self.status | gst
            if self.shuffle:
                self.last_order.update(graft=gorder, graft_offsets=np.concatenate([[0], np.cumsum(kept_g)]))
        else:
            e = lambda dt: torch.empty(0, dtype=dt, device=dev)       # noqa: E731
            graft = ((e(idt), e(idt), e(idt), e(torch.float32)), (e(idt), e(idt), e(idt), e(torch.float32)))
            kfr = torch.empty(0, self.max_facts, dtype=torch.int64, device=dev)
        return (le, qe, kb, graft, qi, kfr, sd, None, ad) + tail
