"""Retrieved-answer-node sets and evaluation metrics, mirroring ``gnn/evaluate.py``.

``retrieve`` is the candidate loop of ``Evaluator.evaluate`` (gnn/evaluate.py:188-209) plus the sort / eps-mass
cut of ``f1_and_hits`` (:25-50), run on the device by csrc/rank.cu; only the short ordered candidate lists
come back to the host.  ``Evaluator`` keeps the reference's class interface and ``.info`` JSONL row schema
(:106-138, 210-219) so the downstream LLM stage (llm/src/qa_prediction) reads the output unchanged.
"""
import json
import math
import os

import numpy as np
import torch

from . import batching, ops


class Retrieved:
    """Retrieved candidates of one question, in retrieval order (numpy views, no per-item Python objects):
    ``idx`` local node indices, ``ent`` global entity ids, ``prob`` fp32 probabilities."""
    __slots__ = ("idx", "ent", "prob")

    def __init__(self, idx, ent, prob):
        self.idx, self.ent, self.prob = idx, ent, prob

    def __len__(self):
        return len(self.idx)

    def pairs(self):
        """[(entity_id, prob_as_python_float), ...] -- the reference's ``retrieved`` list layout."""
        return list(zip(self.ent.tolist(), self.prob.astype(np.float64).tolist()))


def retrieve(pred_dist, db, num_entity, eps):
    """Device ranking (csrc/rank.cu) + one D2H of the ordered lists.
    -> (list of :class:`Retrieved`, one per question; d2h_bytes)."""
    cand_idx, cand_count, _total = ops.rank_candidates(pred_dist, db.local_entity, db.query_entities,
                                                       num_entity, eps)
    return read_ranked(pred_dist, db, cand_idx, cand_count)


def read_ranked(pred_dist, db, cand_idx, cand_count):
    """The ordered candidate lists of a ranked batch (``cand_idx`` / ``cand_count`` of ``ops.rank_candidates``),
    read back to the host, the counts first -> (list of :class:`Retrieved`, one per question; d2h_bytes)."""
    counts_h = cand_count.cpu().numpy()
    maxc = int(counts_h.max()) if counts_h.size else 0
    empty_i, empty_f = np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.float32)
    if maxc == 0:
        return [Retrieved(empty_i, empty_i, empty_f) for _ in range(db.B)], counts_h.size * 4
    idx = cand_idx[:, :maxc].long()
    probs = torch.gather(pred_dist, 1, idx)
    ents = torch.gather(db.local_entity, 1, idx)
    idx_h, probs_h, ents_h = idx.cpu().numpy(), probs.cpu().numpy(), ents.cpu().numpy()
    out = [Retrieved(idx_h[b, :c], ents_h[b, :c], probs_h[b, :c]) for b, c in enumerate(counts_h.tolist())]
    d2h = counts_h.size * 4 + idx_h.size * 8 + probs_h.size * 4 + ents_h.size * 8
    return out, d2h


def f1_and_hits(answers, retrieved_ids):
    """Metric tail of gnn/evaluate.py:51-67 on an already ordered + cut candidate list.
    Returns (precision, recall, f1, hits, em, case)."""
    best = retrieved_ids[0] if retrieved_ids else -1
    correct = sum(1 for c in retrieved_ids if c in answers)
    em = 1 if correct > 0 else 0
    if len(answers) == 0:
        return (1.0, 1.0, 1.0, 1.0, 1.0, 0) if not retrieved_ids else (0.0, 1.0, 0.0, 1.0, 1.0, 1)
    hits = float(best in answers)
    if not retrieved_ids:
        return 1.0, 0.0, 0.0, hits, hits, 2
    p, r = correct / len(retrieved_ids), correct / len(answers)
    f1 = 2.0 / (1.0 / p + 1.0 / r) if p != 0 and r != 0 else 0.0
    return p, r, f1, hits, em, 3


class Evaluator:
    """Drop-in for ``gnn/evaluate.py:Evaluator`` (constructor :70-104, ``write_info`` :106-138, ``evaluate`` :140-240).

    ``step``: optionally a ``graphed.GraphedStep`` of ``model`` that ranks with this evaluator's pad id
    (``len(entity2id)``) and ``eps``.  With it, :meth:`evaluate` over a ``loader.DeviceSplit`` runs the whole split as
    one evaluation epoch (``GraphedStep.start_eval``: batch assembly, forward, ranking and metrics in CUDA graphs) and
    formats the ``.info`` rows from its records on the device (``EvalRun.info``); it returns the same values and
    writes the same file as the per-batch loop, which still serves host loaders and evaluators without a step."""

    def __init__(self, args, model, entity2id, relation2id, device, step=None):
        self.model, self.args, self.eps = model, args, args["eps"]
        self.model_name = args["model_name"]
        self.id2entity = {idx: ent for ent, idx in entity2id.items()}
        self.entity2name = None
        if "sr-" in args.get("data_folder", ""):                   # gnn/evaluate.py:81-84
            import pickle
            with open("ent2id.pickle", "rb") as f:
                self.entity2name = list(pickle.load(f).keys())
        id2relation = {idx: rel for rel, idx in relation2id.items()}   # :87-101
        num_rel_ori = len(relation2id)
        if args.get("use_inverse_relation", False):
            for i in range(len(id2relation)):
                id2relation[i + num_rel_ori] = id2relation[i] + "_rev"
        if args.get("use_self_loop", False):
            id2relation[len(id2relation)] = "self_loop"
        self.id2relation = id2relation
        self.device = device
        self.file_write = None
        if step is not None:
            from .graphed import GraphedStep
            if not isinstance(step, GraphedStep) or step.model is not model:
                raise ValueError("Evaluator: step must be a graphed.GraphedStep of this model")
            if step.num_entity != len(self.id2entity):
                raise ValueError("Evaluator: the step ranks with pad id %d, the evaluator with %d (len(entity2id))"
                                 % (step.num_entity, len(self.id2entity)))
            if step.eps != self.eps:
                raise ValueError("Evaluator: the step ranks with eps %r, the evaluator with %r" % (step.eps, self.eps))
        self.step = step
        self._tables = {}             # id(split) -> InfoTables

    def _name(self, ent):
        return self.id2entity[ent] if self.entity2name is None else self.entity2name[self.id2entity[ent]]

    def write_info(self, valid_data, tp_list, num_step):
        """One dict per question of the CURRENT batch (gnn/evaluate.py:106-138).  ``get_quest`` decodes the loader's
        ``sample_ids``, which ``get_batch`` sets (gnn/dataset_load.py:130-141, 602-603): call it after every
        ``get_batch`` and index the result by the position inside the batch."""
        question_list = valid_data.get_quest()
        obj_list = [{} for _ in question_list]
        actions = None if tp_list is None else [tp[0] for tp in tp_list]
        for j in range(num_step):
            act = None if actions is None else actions[j].cpu().numpy()
            for i, q in enumerate(question_list):
                obj = obj_list[i]
                obj["question"] = q
                obj[j] = {}
                if act is not None:
                    obj[j]["rel_action"] = self.id2relation[act[i]]
                    obj[j]["action"] = str(act[i])
        return obj_list

    def _info_path(self):
        return os.path.join(self.args["checkpoint_dir"], "{}_test.info".format(self.args["experiment_name"]))

    def _open_info(self):
        if self.file_write is None:
            self.file_write = open(self._info_path(), "w")

    def _row(self, obj, answers, p, r, f1, hit, em, cand):
        obj["answers"] = [self._name(a) for a in answers]
        obj["precison"] = p
        obj["recall"] = r
        obj["f1"] = f1
        obj["hit"] = hit
        obj["em"] = em
        obj["cand"] = [(self._name(c), pr) for c, pr in cand.pairs()]
        self.file_write.write(json.dumps(obj) + "\n")

    def evaluate(self, valid_data, test_batch_size=20, write_info=False):
        from .loader import DeviceSplit
        if self.step is not None and isinstance(valid_data, DeviceSplit):
            return self._evaluate_epoch(valid_data, test_batch_size)
        write_info = True                                          # the reference forces it (gnn/evaluate.py:141)
        self.model.eval()
        self.count = 0
        eps = self.eps
        f1s, hits, ems, precisions, recalls = [], [], [], [], []
        valid_data.reset_batches(is_sequential=True)
        num_epoch = math.ceil(valid_data.num_data / test_batch_size)
        if write_info:
            self._open_info()
        case_ct = {}
        num_entity = len(self.id2entity)
        for it in range(num_epoch):
            batch = valid_data.get_batch(it, test_batch_size, fact_dropout=0.0, test=True)
            answer_lists = batch[-1]
            with torch.no_grad():
                _loss, _pred, pred_dist, tp_list = self.model(batch[:-1])
            # the reference drops candidates below (1 - eps) / valid_data.max_local_entity (:154); the ranking kernel
            # uses the batch's own N, which is the loader's max_local_entity by construction (dataset_load.py:250)
            mle = getattr(valid_data, "max_local_entity", pred_dist.shape[1])
            if mle != pred_dist.shape[1]:
                raise ValueError("batch width %d != valid_data.max_local_entity %d" % (pred_dist.shape[1], mle))
            obj_list = self.write_info(valid_data, tp_list, self.model.num_iter) if write_info else None
            retrieved, _ = retrieve(pred_dist, self.model.last_batch, num_entity, eps)
            for b, ret in enumerate(retrieved):
                answers = list(answer_lists[b])
                p, r, f1, hit, em, case = f1_and_hits(answers, ret.ent.tolist())
                if write_info:
                    self._row(obj_list[b], answers, p, r, f1, hit, em, ret)
                case_ct[case] = case_ct.get(case, 0) + 1
                f1s.append(f1); hits.append(hit); ems.append(em); precisions.append(p); recalls.append(r)
        self.case_ct = case_ct
        if write_info and self.file_write is not None:
            self.file_write.close()
            self.file_write = None
        return float(np.mean(f1s)), float(np.mean(hits)), float(np.mean(ems))

    def _evaluate_epoch(self, split, test_batch_size):
        """:meth:`evaluate` over the resident split ``split`` as one evaluation epoch of ``self.step``: the means and
        ``case_ct`` come from the device records, the ``.info`` file from ``EvalRun.info`` with this evaluator's
        :meth:`info_tables` of the split (a malformed run raises before the file is opened)."""
        self.model.eval()
        self.count = 0
        tables = self.info_tables(split)
        run = self.step.start_eval(split, test_batch_size)
        metrics, cases = run.records()
        data = run.info(tables)
        case_ct = {}
        for case in cases.tolist():
            case_ct[case] = case_ct.get(case, 0) + 1
        self.case_ct = case_ct
        with open(self._info_path(), "wb") as f:
            f.write(data)
        return float(np.mean(metrics[:, 2])), float(np.mean(metrics[:, 3])), float(np.mean(metrics[:, 4]))

    def info_tables(self, split):
        """The :class:`InfoTables` of the resident split ``split`` for this evaluator's names, built on the first call
        and kept: the later evaluations of the split (between training epochs, say) reuse them."""
        t = self._tables.get(id(split))
        if t is None or t.split is not split:
            t = self._tables[id(split)] = InfoTables(self, split)
        return t


class InfoTables:
    """What the ``.info`` rows of an evaluation epoch (``graphed.EvalRun.info``) take from the host, on the split's
    device.  ``prefix`` (uint8) with ``prefix_off`` (int64 [num_q + 1]): question q's row up to and including
    ``"answers": [...], ``, cut from ``json.dumps`` of the dict :meth:`Evaluator.write_info` and the answer names
    make.  ``names`` (uint8) with ``name_off`` (int64 [num_names + 1]): ``json.dumps`` of the name
    (``Evaluator._name``) of every entity the split can rank, its ``candidate_entities`` other than the pad id;
    ``name_slot`` (int32, one per entity id up to the largest of them): the entity's name index, -1 for none."""

    def __init__(self, evaluator, split):
        import torch
        self.split = split
        for name, a in self.host_arrays(evaluator, split.loader, split.num_q).items():
            setattr(self, name, torch.from_numpy(a).to(split.device))

    @staticmethod
    def host_arrays(evaluator, data_loader, num_q):
        """The tables as numpy arrays (a dict of the attribute names) for the first ``num_q`` questions of
        ``data_loader``; its ``sample_ids`` are restored afterwards."""
        ev, L = evaluator, data_loader
        had_ids = hasattr(L, "sample_ids")
        saved = getattr(L, "sample_ids", None)
        L.sample_ids = np.arange(num_q)                         # get_quest decodes the questions of sample_ids
        try:
            objs = ev.write_info(L, None, ev.model.num_iter)      # an eval forward returns tp_list None
        finally:
            if had_ids:
                L.sample_ids = saved
            else:
                del L.sample_ids
        prefixes = []
        for obj, answers in zip(objs, L.answer_lists):
            obj["answers"] = [ev._name(a) for a in answers]
            prefixes.append(json.dumps(obj)[:-1].encode("ascii") + b", ")
        ents = np.unique(np.asarray(L.candidate_entities, dtype=np.int64))
        ents = ents[(ents >= 0) & (ents != len(ev.id2entity))]
        slot = np.full(int(ents[-1]) + 1 if ents.size else 1, -1, dtype=np.int32)
        names = []
        for e in ents.tolist():
            try:
                name = ev._name(e)
            except (KeyError, IndexError):
                continue
            slot[e] = len(names)
            names.append(json.dumps(name).encode("ascii"))

        def flat(chunks):
            off = np.zeros(len(chunks) + 1, dtype=np.int64)
            np.cumsum(np.array([len(c) for c in chunks], dtype=np.int64), out=off[1:])
            return np.frombuffer(b"".join(chunks) or b"\0", dtype=np.uint8).copy(), off
        out = dict(name_slot=slot)
        out["prefix"], out["prefix_off"] = flat(prefixes)
        out["names"], out["name_off"] = flat(names)
        return out


def merge_candidates(cand1, cand2):
    """Union of two GNNs' candidate lists as the LLM stage builds it (``load_gnn_rag``,
    llm/src/qa_prediction/predict_answer.py:61-75): an entity present in both keeps the larger score in place,
    new entities are appended in ``cand2`` order, then a STABLE sort by score, descending.  ``cand*`` are the
    ``[[entity, prob], ...]`` lists of two ``.info`` rows; returns a new list (inputs untouched).  O(n) with a dict
    instead of the reference's nested loop; same result including tie order."""
    out = [[c[0], c[1]] for c in cand1]
    pos = {}
    for i, c in enumerate(out):
        pos.setdefault(c[0], i)                   # the reference's inner loop stops at the FIRST match
    for e, p in cand2:
        i = pos.get(e)
        if i is None:
            pos[e] = len(out)
            out.append([e, p])
        elif p > out[i][1]:
            out[i][1] = p
    return sorted(out, key=lambda x: x[1], reverse=True)


def merge_info_rows(rows1, rows2):
    """Row-wise :func:`merge_candidates` of two ``.info`` row lists of the same questions (same order, as written by
    :class:`Evaluator` for two models): returns copies of ``rows1`` with the merged ``cand``."""
    assert len(rows1) == len(rows2)
    out = []
    for a, b in zip(rows1, rows2):
        r = dict(a)
        r["cand"] = merge_candidates(a["cand"], b["cand"])
        out.append(r)
    return out


def path_node_sets(db, retrieved, max_targets=32):
    """Shortest-path node sets seed -> retrieved candidates on the undirected subgraph
    (llm/src/utils/graph_utils.py:10-21,49-75), computed on device (csrc/paths.cu).
    Returns per-question sorted local-index lists and the [B,S,T] hop-distance tensor (host)."""
    B, N = db.B, db.N
    dev = db.local_entity.device
    qe = db.query_entities
    S = int(qe.sum(dim=1).max().item()) if B else 0
    S = max(S, 1)
    src_sorted = torch.argsort((qe != 0).to(torch.int8), dim=1, descending=True, stable=True)[:, :S]
    source_idx = src_sorted.to(torch.int32).contiguous()
    source_cnt = (qe != 0).sum(dim=1).to(torch.int32)
    T = max(1, min(max_targets, max((len(r) for r in retrieved), default=1)))
    tgt = np.zeros((B, T), dtype=np.int32)
    cnt = np.zeros(B, dtype=np.int32)
    for b, r in enumerate(retrieved):
        k = min(len(r), T)
        cnt[b] = k
        tgt[b, :k] = np.asarray(r.idx[:k] if isinstance(r, Retrieved) else [x[0] for x in r[:k]])
    target_idx = torch.from_numpy(tgt).to(dev)
    target_cnt = torch.from_numpy(cnt).to(dev)
    on_path, pair_dist = ops.shortest_path_nodes(db.graph, source_idx, source_cnt, target_idx, target_cnt)
    on = on_path.cpu().numpy()
    return [np.nonzero(on[b])[0].tolist() for b in range(B)], pair_dist.cpu().numpy()
